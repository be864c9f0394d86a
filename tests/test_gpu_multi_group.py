"""GPU tests (-m gpu) of multi-GPU groups (lpcnet_b200_multi_group_*): several models, each a Multi over the same devices, served by
one call that runs one group per device over the members' shards and gathers the PCM on devices[0] like a Multi does.

The contract: a multi-group call leaves every member exactly as the member's own Multi call on its rows of the inputs would, PCM
and state, bit for bit, from any member state.  So most cases drive two identically prepared sets of members, one through the
multi-group and one ("the twins") through their own Multi calls, and compare the PCM, every stream's exported state and a tail
afterwards.  The one-device cases run everywhere; the two-device cases skip on a one-GPU box."""
import ctypes

import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "EXACT_CVT", "FCW_NODES", "FLOAT_LANE_STREAM")
T = 20                          # 20 frames: two chunks, 16 + 4


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv("LPCNET_B200_" + k, raising=False)
    return monkeypatch


_SEEDED = {}


def seeded_blob(seed, flavour="int8"):
    """blob of gen_model.make_model(seed): the default model's shape with other weights"""
    import gen_model
    from lpcnet_b200 import api
    if (seed, flavour) not in _SEEDED:
        common, only8, onlyf = gen_model.make_model(seed)
        _SEEDED[(seed, flavour)] = api.write_blob([(n, t, a.tobytes()) for n, t, a in common + (onlyf if flavour == "float" else only8)])
    return _SEEDED[(seed, flavour)]


def shard_batch(eng, m, k):
    """shard k's batch of Multi m as a Batch (lpcnet_b200_multi_batch); the Multi owns it"""
    class Shard(eng.Batch):
        def close(self):
            self._h = None
        __del__ = close
    b = Shard.__new__(Shard)
    b._L = eng.lib()
    b._h = b._L.lpcnet_b200_multi_batch(m._h, k)
    b.n = m.shard(k)[2]
    return b


def set_codebooks(b, cb):
    assert b._L.lpcnet_b200_batch_set_codebooks(b._h, cb.ctypes.data, cb.size) == 0


def check(got, want, what):
    assert got.shape == want.shape, "%s: shape %s vs %s" % (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.flatnonzero((got != want).any(axis=1))
        t = int(np.flatnonzero(got[bad[0]] != want[bad[0]])[0])
        raise AssertionError("%s: %d of %d streams differ, first at stream %d sample %d (%d vs %d)"
                             % (what, bad.size, got.shape[0], bad[0], t, got[bad[0], t], want[bad[0], t]))


class Twins:
    """members (blob, n) twice over `devices`: `m` driven through a MultiGroup, `t` through their own Multi calls"""

    def __init__(self, eng, members, devices=(0,), codebooks=True):
        self.eng, self.devices, self.blobs = eng, list(devices), [b for b, _ in members]
        cb = H.codebooks() if codebooks else None
        mk = lambda: [eng.Multi(n, b, self.devices, config=H.model_config(""), codebooks=cb) for b, n in members]  # noqa: E731
        self.m, self.t = mk(), mk()
        self.mg = eng.MultiGroup(self.m)
        self.rows = np.cumsum([0] + [n for _, n in members])
        self.n = int(self.rows[-1])
        assert self.mg.n == self.n

    def split(self, a):
        return [a[self.rows[k]:self.rows[k + 1]] for k in range(len(self.m))]

    def synth(self, f, gather=False):
        got = self.mg.synthesize(f, gather=gather)
        want = np.concatenate([t.synthesize(x) for t, x in zip(self.t, self.split(f))])
        check(got, want, "multi-group synthesize%s" % (" (gather)" if gather else ""))
        return got

    def decode(self, pk, gather=False):
        got = self.mg.decode(pk, gather=gather)
        want = np.concatenate([t.decode(x) for t, x in zip(self.t, self.split(pk))])
        check(got, want, "multi-group decode%s" % (" (gather)" if gather else ""))
        return got

    def shards(self, side):
        """[(member, shard, batch)] of one side"""
        return [(j, k, shard_batch(self.eng, m, k)) for j, m in enumerate(side) for k in range(len(self.devices))]

    def both(self, fn):
        """a call made on both sides: fn(member, shard, batch) for every shard batch"""
        for side in (self.m, self.t):
            for j, k, b in self.shards(side):
                fn(j, k, b)

    def check_state(self):
        for (j, k, a), (_, _, b) in zip(self.shards(self.m), self.shards(self.t)):
            for s in range(a.n):
                assert np.array_equal(a.export_state(s).view(np.uint32), b.export_state(s).view(np.uint32)), \
                    "member %d shard %d stream %d: state differs" % (j, k, s)

    def check_tails(self, samples=90):
        for (j, k, a), (_, _, b) in zip(self.shards(self.m), self.shards(self.t)):
            check(a.synthesize_tail(samples), b.synthesize_tail(samples), "member %d shard %d tail" % (j, k))

    def oracle(self, got, f, kind="int8", rows=3):
        for j, (blob, x, y) in enumerate(zip(self.blobs, self.split(f), self.split(got))):
            check(y[:rows], H.oracle_synth(x[:rows], kind, model_blob=blob), "member %d vs the oracle" % j)

    def close(self):
        self.mg.close()
        for m in self.m + self.t:
            m.close()


def feats(n, base=0, nframes=T):
    return make_feature_batch(range(base, base + n), nframes)


# ---- one device ----
@pytest.mark.parametrize("sizes", [[37, 5], [37, 5, 64]], ids=["two", "three"])
def test_synthesis_equals_member_multis_and_oracle(eng, sizes):
    P = Twins(eng, [(seeded_blob(100 + i), n) for i, n in enumerate(sizes)])
    f = feats(P.n, 10)
    got = P.synth(f)
    P.oracle(got, f)
    g = P.mg.group(0)
    ms, launches = g.last_sample_kernel_ms()
    assert ms > 0 and launches > 0 and g.n == P.n
    P.check_state()
    P.check_tails()
    P.close()


def test_state_across_mixed_calls(eng):
    """multi-group calls between member Multi calls (gather on and off: the gather leaves a PCM sink on the shard batches), shard
    resets and a single-device group call over the shards"""
    P = Twins(eng, [(seeded_blob(110), 9), (H.blob("int8"), 6), (seeded_blob(111), 4)])
    f = feats(P.n, 200, 80)
    P.synth(f[:, 0:3])
    for j, (m, t) in enumerate(zip(P.m, P.t)):       # member calls on both sides: member 1 gathers, leaving its sink set
        x = P.split(f)[j][:, 3:5]
        check(m.synthesize(x, gather=j == 1), t.synthesize(x, gather=j == 1), "member %d Multi call" % j)
    P.synth(f[:, 5:23], gather=True)                 # not refused and not forwarded to member 1's leftover sink
    P.both(lambda j, k, b: b.reset_streams([0, 2]) if j != 1 else None)
    P.synth(f[:, 23:24])                             # inside FEATURES_DELAY for the reset streams
    P.synth(f[:, 24:41])
    P.check_tails()
    # a single-device group over the shards (the public group refuses the leftover sink: clear it first); the twins make the
    # members' own calls
    sh = [b for _, _, b in P.shards(P.m)]
    for b in sh:
        b.set_pcm_sink(None, 0, 0)
    grp = eng.Group(sh)
    x = f[:, 41:46]
    check(grp.synthesize(x), np.concatenate([t.synthesize(y) for t, y in zip(P.t, P.split(x))]), "group over the shards")
    grp.close()
    for j, (m, t) in enumerate(zip(P.m, P.t)):
        x = P.split(f)[j][:, 46:50]
        check(m.synthesize(x, gather=True), t.synthesize(x, gather=True), "member %d Multi call" % j)
    P.both(lambda j, k, b: b.reset_streams([b.n - 1]))
    P.synth(f[:, 50:80], gather=True)
    P.check_state()
    P.check_tails()
    P.close()


def test_gather_equals_host_and_touches_only_its_rows(eng):
    P = Twins(eng, [(seeded_blob(120), 7), (seeded_blob(121), 12)])
    L = eng.lib()
    f = feats(P.n, 300)
    want = P.synth(f)
    # a second, fresh set: the same call gathered into rows 2.. of a larger buffer
    Q = Twins(eng, [(seeded_blob(120), 7), (seeded_blob(121), 12)])
    before, after, TS = 2, 3, T * 160
    rows = before + Q.n + after
    fill = np.full((rows, TS), 0x5555, np.int16)
    L.lpcnet_b200_set_device(0)
    d = L.lpcnet_b200_device_alloc_on(0, fill.nbytes)
    L.lpcnet_b200_memcpy_h2d(d, fill.ctypes.data, fill.nbytes)
    fc = np.ascontiguousarray(f)
    assert L.lpcnet_b200_multi_group_synthesize_gather(Q.mg._h, fc.ctypes.data, T, 20, 160, d + 2 * before * TS) == 0, eng.api._err()
    got = np.zeros_like(fill)
    L.lpcnet_b200_memcpy_d2h(got.ctypes.data, d, got.nbytes)
    L.lpcnet_b200_device_free(d)
    check(got[before:before + Q.n], want, "gathered PCM")
    assert (got[:before] == 0x5555).all() and (got[before + Q.n:] == 0x5555).all(), "the gather wrote outside the job's rows"
    P.close()
    Q.close()


def test_decode_equals_member_multis(eng):
    import gen_model
    P = Twins(eng, [(H.blob("int8"), 5), (seeded_blob(130), 11)])
    other = np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=78)]).astype(np.float32)
    P.both(lambda j, k, b: set_codebooks(b, other) if j == 1 else None)     # member 1 decodes with codebooks of its own
    pk = np.stack([make_packets(s, 5) for s in range(P.n)])
    got = P.decode(pk[:, :2])
    check(P.split(got)[0], H.oracle_decode(P.split(pk)[0][:, :2], "int8"), "member 0 decode vs the oracle")
    P.synth(feats(P.n, 400, 3))
    P.decode(pk[:, 2:], gather=True)
    P.check_state()
    P.check_tails()
    P.close()


def test_decode_without_codebooks_is_refused_and_changes_nothing(eng):
    P = Twins(eng, [(H.blob("int8"), 4), (seeded_blob(140), 3)], codebooks=False)
    P.both(lambda j, k, b: set_codebooks(b, H.codebooks()) if j == 0 else None)
    f = feats(P.n, 500, 6)
    P.synth(f[:, :3])
    pk = np.stack([make_packets(s, 2) for s in range(P.n)])
    for gather in (False, True):
        with pytest.raises(eng.LPCNetB200Error, match="codebooks"):
            P.mg.decode(pk, gather=gather)
    P.check_state()                                   # member 0, which has codebooks, did not run either
    P.synth(f[:, 3:])
    P.check_state()
    P.close()


@pytest.mark.parametrize("case", ["neuron", "lane", "lane_env"])
def test_float_members(eng, clean_env, case):
    """small counts take the neuron-per-lane kernel, larger ones the lane == stream kernel, as does
    LPCNET_B200_FLOAT_LANE_STREAM set at create"""
    import torch
    sizes = [700, 900] if case == "lane" else [3, 6, 2]
    if case == "lane_env":
        clean_env.setenv("LPCNET_B200_FLOAT_LANE_STREAM", "1")
    P = Twins(eng, [(seeded_blob(150 + i, "float"), n) for i, n in enumerate(sizes)])
    clean_env.delenv("LPCNET_B200_FLOAT_LANE_STREAM", raising=False)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert eng.group_plan_float(sizes, sms, lane_stream=case == "lane_env")[0] == case.split("_")[0]
    f = feats(P.n, 600)
    got = np.concatenate([P.synth(f[:, :3]), P.synth(f[:, 3:], gather=True)], axis=1)
    P.oracle(got, f, "float", rows=2)
    P.check_state()
    P.check_tails()
    P.close()


def test_refusals(eng):
    L = eng.lib()
    a = eng.Multi(4, H.blob("int8"), [0], config=H.model_config(""))
    b = eng.Multi(3, seeded_blob(160), [0], config=H.model_config(""))
    c256 = eng.Multi(2, H.blob("int8", "na256"), [0], config=H.model_config("na256"))
    fl = eng.Multi(2, H.blob("float"), [0], config=H.model_config(""))

    def refused(hs, count, what):
        arr = (ctypes.c_void_p * max(1, len(hs)))(*hs) if hs is not None else None
        assert not L.lpcnet_b200_multi_group_create(arr, count)
        assert what in eng.api._err(), eng.api._err()
    refused(None, 1, "1..16")
    refused([a._h], 0, "1..16")
    refused([a._h, None], 2, "NULL")
    refused([a._h, b._h, a._h], 3, "twice")
    refused([a._h, c256._h], 2, "GRU_A")
    refused([a._h, fl._h], 2, "float")
    many = [eng.Multi(1, H.blob("int8"), [0], config=H.model_config("")) for _ in range(17)]
    refused([m._h for m in many], 17, "1..16")
    eng.MultiGroup(many[:16]).close()
    if eng.device_count() >= 2:
        d01 = eng.Multi(4, H.blob("int8"), [0, 1], config=H.model_config(""))
        d10 = eng.Multi(4, H.blob("int8"), [1, 0], config=H.model_config(""))
        refused([a._h, d01._h], 2, "devices")
        refused([d01._h, d10._h], 2, "devices")
        d01.close()
        d10.close()
    # the members are untouched by the refusals: a multi-group over a and b works
    mg = eng.MultiGroup([a, b])
    f = feats(7, 700, 3)
    got = mg.synthesize(f)
    mg.close()
    x = eng.Batch(4, H.blob("int8"), config=H.model_config(""))
    y = eng.Batch(3, seeded_blob(160), config=H.model_config(""))
    check(got, np.concatenate([x.synthesize(f[:4]), y.synthesize(f[4:])]), "after the refusals")
    for m in [a, b, c256, fl, x, y] + many:
        m.close()


# ---- two devices ----
def _need2(eng):
    if eng.device_count() < 2:
        pytest.skip("needs two GPUs")


@pytest.mark.parametrize("devices", [[0, 1], [1, 0]], ids=["01", "10"])
def test_two_devices_equal_single_device_batches(eng, devices):
    _need2(eng)
    members = [(seeded_blob(170), 11), (H.blob("int8"), 5), (seeded_blob(171), 64)]
    P = Twins(eng, members, devices)
    assert [P.m[0].shard(k)[2] for k in range(2)] == [6, 5]
    f = feats(P.n, 800)
    single = [eng.Batch(n, b, device=0, config=H.model_config("")) for b, n in members]
    want = np.concatenate([s.synthesize(x) for s, x in zip(single, P.split(f))])
    got = np.concatenate([P.synth(f[:, :17]), P.synth(f[:, 17:], gather=True)], axis=1)
    check(got, want, "two devices vs single-device batches")
    for s in single:
        s.close()
    P.check_state()
    P.close()


@pytest.mark.parametrize("devices", [[0, 1], [1, 0]], ids=["01", "10"])
def test_two_devices_decode_equals_single_device_batches(eng, devices):
    _need2(eng)
    members = [(H.blob("int8"), 9), (seeded_blob(180), 7)]
    P = Twins(eng, members, devices)
    pk = np.stack([make_packets(s, 3) for s in range(P.n)])
    single = [eng.Batch(n, b, device=0, config=H.model_config(""), codebooks=H.codebooks()) for b, n in members]
    want = np.concatenate([s.decode(x) for s, x in zip(single, P.split(pk))])
    check(P.decode(pk[:, :1], gather=True), want[:, :640], "two devices decode (gather)")
    check(P.decode(pk[:, 1:]), want[:, 640:], "two devices decode")
    for s in single:
        s.close()
    P.close()
