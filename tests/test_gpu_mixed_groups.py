"""GPU tests (-m gpu) of mixed groups (lpcnet_b200_mixed_group_*): batches of different GRU_A sizes and flavours in one call, one
ordinary group per (GRU_A size, flavour) class, each class's launches on a CUDA stream of its own.

The contract is the group's: a call leaves every member exactly as the member's own call on its rows of the inputs would, PCM and
state, bit for bit, from any member state.  Every case runs the same sequence twice on identically prepared batches, once with
mixed-group calls and once with member calls, and compares the PCM, the members' exported states and a tail afterwards; several
cases also compare each member with the CPU restatement of its model."""
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "EXACT_CVT", "FCW_NODES", "FLOAT_LANE_STREAM")
T1, T2 = 3, 18                  # calls of 3 + 18 frames: state carried across calls, the second crosses the 16-frame chunk
FOFF, POFF, GUARD = 12, 5, -12345            # `_device` buffers: features 12 floats in, PCM 5 samples in, guard value around the PCM
STATE_ALL = 48                  # members up to this size have every stream's state compared, larger ones a spread


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


@pytest.fixture(scope="module")
def sms(eng):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv("LPCNET_B200_" + k, raising=False)
    return monkeypatch


_SEEDED = {}


def seeded_blob(kind, seed, na=None):
    """int8 or float blob of gen_model.make_model(seed): the default model's shape (or `na` GRU_A units) with other weights"""
    import gen_model
    from lpcnet_b200 import api
    key = (kind, seed, na)
    if key not in _SEEDED:
        common, only8, onlyf = gen_model.make_model(seed, na=na)
        _SEEDED[key] = api.write_blob([(n, t, a.tobytes()) for n, t, a in common + (onlyf if kind == "float" else only8)])
    return _SEEDED[key]


class Member:
    """one member: blob, flavour, header tag of its switches (oracle), streams, VQ codebooks"""

    def __init__(self, blob, kind, tag="", n=8, codebooks=None):
        self.blob, self.kind, self.tag, self.n, self.codebooks = blob, kind, tag, n, codebooks

    def make(self, eng):
        return eng.Batch(self.n, self.blob, device=0, config=H.model_config(self.tag),
                         codebooks=H.codebooks() if self.codebooks is None else self.codebooks)


def m8(na=384, n=8, seed=None, tag=None):
    tag = ("na%d" % na if na != 384 else "") if tag is None else tag
    return Member(H.blob("int8", tag) if seed is None else seeded_blob("int8", seed, na), "int8", tag, n)


def mf(na=384, n=8, seed=None, tag=None):
    tag = ("na%d" % na if na != 384 else "") if tag is None else tag
    return Member(H.blob("float", tag) if seed is None else seeded_blob("float", seed, na), "float", tag, n)


def check(got, want, what):
    assert got.shape == want.shape, "%s: shape %s vs %s" % (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.flatnonzero((got != want).any(axis=1))
        t = int(np.flatnonzero(got[bad[0]] != want[bad[0]])[0])
        raise AssertionError("%s: %d of %d streams differ, first at stream %d sample %d (%d vs %d)"
                             % (what, bad.size, got.shape[0], bad[0], t, got[bad[0], t], want[bad[0], t]))


def state_rows(n):
    if n <= STATE_ALL:
        return range(n)
    return sorted(set(range(4)) | set(range(n - 4, n)) | set(np.linspace(0, n - 1, 9).astype(int).tolist()))


def device_synth(call, f, spf):
    """call(d_features, nframes, stride, d_pcm, spf) on buffers that start FOFF floats / POFF samples into their allocations; the
    guard samples around the PCM must stay untouched"""
    import torch
    n, nf, stride = f.shape
    d_f = torch.full((FOFF + f.size,), float("nan"), dtype=torch.float32, device="cuda")
    d_f[FOFF:] = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32).ravel()).cuda()
    d_p = torch.full((2 * POFF + n * nf * spf,), GUARD, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    call(d_f.data_ptr() + 4 * FOFF, nf, stride, d_p.data_ptr() + 2 * POFF, spf)
    out = d_p.cpu().numpy()
    assert (out[:POFF] == GUARD).all() and (out[-POFF:] == GUARD).all(), "the mixed group wrote outside its PCM buffer"
    return out[POFF:-POFF].reshape(n, nf * spf)


def device_decode(mg, pk):
    import torch
    n, P, _ = pk.shape
    d_k = torch.zeros((FOFF + pk.size,), dtype=torch.uint8, device="cuda")
    d_k[FOFF:] = torch.from_numpy(np.ascontiguousarray(pk).ravel()).cuda()
    d_p = torch.full((2 * POFF + n * P * 640,), GUARD, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    mg.decode_device(d_k.data_ptr() + FOFF, P, d_p.data_ptr() + 2 * POFF)
    out = d_p.cpu().numpy()
    assert (out[:POFF] == GUARD).all() and (out[-POFF:] == GUARD).all(), "the mixed group wrote outside its PCM buffer"
    return out[POFF:-POFF].reshape(n, P * 640)


class Pair:
    """the same members twice: `g` driven through a mixed group, `r` through member calls.  spc pins the streams per CTA;
    lane_stream sets LPCNET_B200_FLOAT_LANE_STREAM for the members and the mixed group."""

    def __init__(self, eng, mp, members, spc=None, lane_stream=False):
        self.members = members
        if lane_stream:
            mp.setenv("LPCNET_B200_FLOAT_LANE_STREAM", "1")
        self.g = [m.make(eng) for m in members]
        self.r = [m.make(eng) for m in members]
        if spc:
            mp.setenv("LPCNET_B200_STREAMS_PER_CTA", str(spc))
        self.mg = eng.MixedGroup(self.g)
        mp.delenv("LPCNET_B200_STREAMS_PER_CTA", raising=False)
        mp.delenv("LPCNET_B200_FLOAT_LANE_STREAM", raising=False)
        self.rows = np.cumsum([0] + [m.n for m in members])
        self.n = int(self.rows[-1])

    def split(self, a):
        return [a[self.rows[k]:self.rows[k + 1]] for k in range(len(self.members))]

    def synth(self, f, spf=160, device=False):
        got = device_synth(self.mg.synthesize_device, f, spf) if device else self.mg.synthesize(f, spf)
        want = np.concatenate([b.synthesize(x, spf) for b, x in zip(self.r, self.split(f))])
        check(got, want, "mixed group synthesize%s (spf %d)" % ("_device" if device else "", spf))
        return got

    def decode(self, p, device=False):
        got = device_decode(self.mg, p) if device else self.mg.decode(p)
        want = np.concatenate([b.decode(x) for b, x in zip(self.r, self.split(p))])
        check(got, want, "mixed group decode%s" % ("_device" if device else ""))
        return got

    def both(self, fn):
        """a member lifecycle call, made on both sides: fn(k, batch)"""
        for side in (self.g, self.r):
            for k, b in enumerate(side):
                fn(k, b)

    def check_state(self):
        for k, m in enumerate(self.members):
            for s in state_rows(m.n):
                a, b = self.g[k].export_state(s), self.r[k].export_state(s)
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "member %d stream %d: state differs" % (k, s)

    def check_tails(self, samples=90):
        for k in range(len(self.members)):
            check(self.g[k].synthesize_tail(samples), self.r[k].synthesize_tail(samples), "member %d tail" % k)

    def oracle(self, got, f):
        for k, (m, x) in enumerate(zip(self.members, self.split(f))):
            want = H.oracle_synth(np.ascontiguousarray(x[:, :, :20]), m.kind, tag=m.tag, model_blob=m.blob)
            check(self.split(got)[k], want, "member %d (%s %s) vs the oracle" % (k, m.kind, m.tag or "default"))

    def close(self):
        self.mg.close()
        for b in self.g + self.r:
            b.close()


def feats(n, T, base=0):
    return make_feature_batch(range(base, base + n), T)


def in_calls(P, f, **kw):
    return np.concatenate([P.synth(f[:, :T1], **kw), P.synth(f[:, T1:], **kw)], axis=1)


# ---- shapes ----
def test_int8_sizes_in_one_call(eng, clean_env):
    """int8 128 + 256 + 384: three classes, each its own group; per-class kernel times and the call's time are reported"""
    P = Pair(eng, clean_env, [m8(128, 5), m8(256, 9), m8(384, 7), m8(128, 11, seed=13)])
    assert P.mg.classes == 3
    f = feats(P.n, T1 + T2)
    P.oracle(in_calls(P, f), f)
    P.check_state()
    P.check_tails()
    assert P.mg.last_call_ms() > 0
    for c in range(P.mg.classes):
        ms, launches = P.mg.group(c).last_sample_kernel_ms()
        assert ms > 0 and launches > 0
    P.close()


@pytest.mark.parametrize("spc", [None, 4, 5])
def test_int8_and_float_together(eng, clean_env, spc):
    """int8 and float members of every size; at spc <= 4 the float classes take the neuron-per-lane kernel, above it the lane ==
    stream kernel"""
    P = Pair(eng, clean_env, [mf(384, 6), m8(384, 10), mf(128, 4), m8(256, 7), mf(256, 5, seed=17)], spc=spc)
    assert P.mg.classes == 5
    f = feats(P.n, T1 + T2, 100)
    P.oracle(in_calls(P, f), f)
    P.check_state()
    P.check_tails()
    P.close()


def test_float_kernels_automatic_plan(eng, clean_env, sms):
    """automatic plans on both float kernels: about 2 x SMs streams in all (neuron-per-lane) and about 8 x SMs (lane == stream)"""
    from lpcnet_b200 import api
    for total, want in ((2 * sms, "neuron"), (8 * sms, "lane")):
        sizes = [total // 2, total // 4, total - total // 2 - total // 4]
        _, _, classes = api.mixed_plan(sizes, [384, 384, 128], [0, 1, 1], sms)
        assert [k for k, _ in classes] == ["int8", want, want]
        P = Pair(eng, clean_env, [m8(384, sizes[0], seed=21), mf(384, sizes[1], seed=22), mf(128, sizes[2], seed=23)])
        f = make_feature_batch(np.arange(P.n) % 97 + 150, 3)
        P.synth(f)
        P.check_state()
        P.check_tails(40)
        P.close()


@pytest.mark.parametrize("kind", ["int8", "float"])
def test_stress_models_of_several_sizes(eng, clean_env, kind):
    """the stress models at 384, 256 and 128 units in one call, and the default models"""
    import gen_model
    ms = []
    for na in (384, 256, 128):
        tag = "na%d" % na if na != 384 else ""
        ms += [Member(H.stress_blob(name, kind, na=na), kind, tag, n=2 + i) for i, name in enumerate(gen_model.stress_names(na)[:5])]
    ms.append(m8(384, 4) if kind == "float" else mf(384, 4))      # and a member of the other flavour
    P = Pair(eng, clean_env, ms)
    f = feats(P.n, 7, 200)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


def test_sixteen_members_all_six_classes(eng, clean_env):
    ms = []
    for k in range(16):
        na = (128, 256, 384)[k % 3]
        make = mf if (k // 3) % 2 else m8
        ms.append(make(na, n=1 + k, seed=None if k < 6 else 40 + k))
    P = Pair(eng, clean_env, ms)
    assert P.mg.classes == 6
    f = feats(P.n, 5, 300)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.check_tails(40)
    P.close()


def test_variants_in_one_call(eng, clean_env):
    """FEATURES_DELAY 0, 1 and 2, END2END and LPC_GAMMA differ by member: the members' silent prefixes differ in length"""
    ms = [m8(384, 6, tag="e2e"), mf(384, 5, tag="delay0"), m8(384, 7, tag="delay1"), m8(256, 4, tag="na256e2e"),
          mf(384, 3, tag="e2e"), m8(384, 5), mf(256, 4, tag="na256e2e")]
    P = Pair(eng, clean_env, ms)
    f = feats(P.n, 19, 400)
    got = np.concatenate([P.synth(f[:, :1]), P.synth(f[:, 1:])], axis=1)
    P.oracle(got, f)
    P.check_state()
    P.check_tails()
    P.close()


# ---- geometry ----
@pytest.mark.parametrize("spc", [1, 4, 5, 16, 17, 32])
def test_pinned_spc(eng, clean_env, spc):
    P = Pair(eng, clean_env, [m8(384, 3), mf(384, 13, seed=31), m8(128, 21, seed=32), mf(256, 7)], spc=spc)
    f = feats(P.n, 4, 500)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


def test_more_than_one_wave(eng, clean_env, sms):
    half = 16 * sms
    P = Pair(eng, clean_env, [m8(384, half + 100), mf(384, 200, seed=51), m8(128, half - 99, seed=52)])
    f = make_feature_batch(np.arange(P.n) % 97 + 700, 3)
    P.synth(f)
    P.check_state()
    P.close()


# ---- call shapes ----
def shape_members():
    return [m8(384, 5), mf(384, 4), m8(128, 6, seed=33), mf(256, 3)]


@pytest.mark.parametrize("spf,path", [(80, "host"), (320, "device"), (1, "device")])
def test_samples_per_frame(eng, clean_env, spf, path):
    P = Pair(eng, clean_env, shape_members())
    f = feats(P.n, T1 + T2, 800)
    in_calls(P, f, spf=spf, device=path == "device")
    P.check_state()
    P.check_tails()
    P.close()


@pytest.mark.parametrize("path", ["host", "device"])
def test_feature_stride_36(eng, clean_env, path):
    """features of 36 floats per frame whose last 16 are NaN; the members' own calls take the same 36-float rows"""
    P = Pair(eng, clean_env, shape_members())
    f = feats(P.n, T1 + T2, 850)
    f36 = np.full(f.shape[:2] + (36,), np.nan, np.float32)
    f36[:, :, :20] = f
    P.oracle(in_calls(P, f36, device=path == "device"), f)
    P.check_state()
    P.check_tails()
    P.close()


@pytest.mark.parametrize("path", ["host", "device"])
def test_decode_across_a_chunk(eng, clean_env, path):
    """decode of 5 packets (20 frames: across the 16-frame chunk) with per-member codebooks, then synthesis, then 5 more packets"""
    import gen_model
    other = np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=78)]).astype(np.float32)
    P = Pair(eng, clean_env, [m8(384, 5), Member(seeded_blob("float", 34), "float", n=6, codebooks=other),
                              Member(seeded_blob("int8", 35, 128), "int8", "na128", n=4, codebooks=other), mf(384, 3)])
    pk = np.stack([make_packets(7700 + s, 10) for s in range(P.n)])
    got = P.decode(pk[:, :5], path == "device")
    for k, kind in ((0, "int8"), (3, "float")):      # default model and codebooks: the oracle decodes them
        check(P.split(got)[k], H.oracle_decode(P.split(pk)[k][:, :5], kind), "member %d decode vs the oracle" % k)
    P.synth(feats(P.n, 3, 7800), device=path == "device")
    P.check_tails()
    P.decode(pk[:, 5:], path == "device")
    P.check_state()
    P.check_tails()
    P.close()


# ---- state ----
def test_reset_streams_between_calls(eng, clean_env):
    """reset_streams on some members between calls: the silent prefixes differ by member and by stream"""
    P = Pair(eng, clean_env, [m8(384, 6), mf(384, 5, tag="delay1"), m8(128, 7), mf(256, 4)])
    f = feats(P.n, 30, 900)
    P.synth(f[:, 0:3])
    P.both(lambda k, b: b.reset_streams([1, 3]) if k in (0, 3) else None)
    P.synth(f[:, 3:4])                                                           # inside FEATURES_DELAY for the reset streams
    P.both(lambda k, b: b.reset_streams([0]) if k == 1 else None)
    P.synth(f[:, 4:6])
    P.check_tails()
    P.both(lambda k, b: b.reset() if k == 2 else None)
    P.synth(f[:, 6:9])
    st = {}
    P.both(lambda k, b: st.__setitem__(id(b), b.export_state(2)) if k == 3 else None)
    P.both(lambda k, b: b.import_state(0, st[id(b)]) if k == 3 else None)
    P.synth(f[:, 9:30])
    P.check_state()
    P.check_tails()
    P.close()


# ---- ordering ----
def test_device_calls_on_two_streams_mixed_with_member_and_group_calls(eng, clean_env):
    import torch
    P = Pair(eng, clean_env, [m8(384, 6), mf(256, 5), m8(384, 9, seed=81), m8(128, 4)])
    og = eng.Group([P.g[0], P.g[2]])                   # an ordinary group over two of the members
    T = 5
    fs = [feats(P.n, T, 1100 + 50 * i) for i in range(3)]
    d_f = [torch.from_numpy(x).cuda() for x in fs]
    d_p = [torch.zeros((P.n, T * 160), dtype=torch.int16, device="cuda") for _ in fs]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    extra = feats(6, 2, 1300)
    gx = feats(15, 3, 1350)
    P.mg.synthesize_device(d_f[0].data_ptr(), T, 20, d_p[0].data_ptr(), 160, s1.cuda_stream)
    got_m = P.g[0].synthesize(extra)                                            # member host call while mixed work is queued
    P.mg.synthesize_device(d_f[1].data_ptr(), T, 20, d_p[1].data_ptr(), 160, s2.cuda_stream)
    got_g = og.synthesize(gx)                                                   # group over two members
    P.g[1].reset_streams([0, 4])
    P.mg.synthesize_device(d_f[2].data_ptr(), T, 20, d_p[2].data_ptr(), 160, s1.cuda_stream)
    s1.synchronize(); s2.synchronize()
    want0 = np.concatenate([b.synthesize(x) for b, x in zip(P.r, P.split(fs[0]))])
    want_m = P.r[0].synthesize(extra)
    want1 = np.concatenate([b.synthesize(x) for b, x in zip(P.r, P.split(fs[1]))])
    want_g = np.concatenate([P.r[0].synthesize(gx[:6]), P.r[2].synthesize(gx[6:])])
    P.r[1].reset_streams([0, 4])
    want2 = np.concatenate([b.synthesize(x) for b, x in zip(P.r, P.split(fs[2]))])
    check(got_m, want_m, "member call between mixed-group calls")
    check(got_g, want_g, "group call between mixed-group calls")
    for i, w in enumerate((want0, want1, want2)):
        check(d_p[i].cpu().numpy(), w, "mixed-group _device call %d" % i)
    P.check_state()
    og.close()
    P.close()


# ---- refusals ----
def test_create_refusals(eng, clean_env):
    import lpcnet_b200
    a = m8(384, 2).make(eng)
    b = mf(128, 2).make(eng)
    many = [m8(128, 1).make(eng) for _ in range(17)]
    for members, what in [([], "1..16"), ([a, None], "NULL"), ([a, b, a], "twice"), (many, "1..16")]:
        with pytest.raises(lpcnet_b200.LPCNetB200Error, match=what):
            eng.MixedGroup(members)
    mg = eng.MixedGroup(many[:16])
    assert mg.classes == 1 and mg.n == 16
    mg.close()
    for x in [a, b] + many:
        x.close()


def test_members_on_different_devices_are_refused(eng, clean_env):
    import lpcnet_b200
    if lpcnet_b200.device_count() < 2:
        pytest.skip("needs two GPUs")
    a = m8(384, 2).make(eng)
    b = eng.Batch(2, H.blob("int8", "na128"), device=1, config=H.model_config("na128"))
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="device"):
        eng.MixedGroup([a, b])
    a.close(); b.close()


def test_call_refusals_change_nothing(eng, clean_env):
    """a member with a sink, a decode with a member lacking codebooks, bad strides and samples per frame: refused before anything
    is enqueued, so no member's state changed; the next good call matches the twins"""
    import lpcnet_b200
    import torch
    P = Pair(eng, clean_env, [m8(384, 3), mf(256, 4)])
    f = feats(P.n, 4, 1500)
    P.synth(f[:, :2])
    sink = torch.zeros((4, 160 * 4), dtype=torch.int16, device="cuda")
    P.g[1].set_pcm_sink(sink.data_ptr(), 160 * 4, 0)
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="sink"):
        P.mg.synthesize(f[:, 2:])
    P.g[1].set_pcm_sink(None, 0, 0)
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="feature_stride"):
        P.mg.synthesize(f[:, 2:, :19])
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="samples_per_frame"):
        P.mg.synthesize(f[:, 2:], samples_per_frame=0)
    P.check_state()
    P.synth(f[:, 2:])
    P.check_state()
    P.close()

    # decode with a member lacking codebooks: the first class may not have run either
    a, b = m8(384, 3).make(eng), eng.Batch(2, H.blob("float", "na128"), device=0, config=H.model_config("na128"))
    ra, rb = m8(384, 3).make(eng), eng.Batch(2, H.blob("float", "na128"), device=0, config=H.model_config("na128"))
    mg = eng.MixedGroup([a, b])
    pk = np.stack([make_packets(7900 + s, 2) for s in range(5)])
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="codebooks"):
        mg.decode(pk)
    for x, y in ((a, ra), (b, rb)):
        for s in range(x.n):
            assert np.array_equal(x.export_state(s).view(np.uint32), y.export_state(s).view(np.uint32)), "a refused decode changed state"
    mg.close()
    for x in (a, b, ra, rb):
        x.close()
