"""GPU tests (-m gpu) of float groups: the synthesize / decode calls of several float batches of one GRU_A size run as one call,
with one per-sample launch for all their streams, on the neuron-per-lane kernel (at most 4 streams per CTA) or the lane == stream
kernel.

The contract is the one of int8 groups (test_gpu_groups.py): a group call leaves every member exactly as the member's own call on
its rows of the inputs would, PCM and state, bit for bit, from any member state.  Every case runs the same sequence twice on
identically prepared batches, once with group calls and once with member calls, and compares the PCM, the members' exported
states (a spread of streams in large members) and a tail afterwards; most cases also compare each member's PCM with the float
CPU restatement of its model."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "EXACT_CVT", "FCW_NODES", "FLOAT_LANE_STREAM")
T1, T2 = 3, 18                  # calls of 3 + 18 frames: state carried across calls, the second crosses the 16-frame chunk
FOFF, POFF, GUARD = 12, 5, -12345            # `_device` buffers: features 12 floats in, PCM 5 samples in, guard value around the PCM
STATE_ALL = 64                  # members up to this size have every stream's state compared, larger ones a spread


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


def seeded_blob(seed, na=None):
    """float blob of gen_model.make_model(seed): the default model's shape with other weights"""
    import gen_model
    from lpcnet_b200 import api
    key = (seed, na)
    if key not in _SEEDED:
        common, _, onlyf = gen_model.make_model(seed, na=na)
        _SEEDED[key] = api.write_blob([(n, t, a.tobytes()) for n, t, a in common + onlyf])
    return _SEEDED[key]


class Member:
    """one member's float model: blob, header tag of its switches (oracle), streams, VQ codebooks"""

    def __init__(self, blob, tag="", n=8, codebooks=None):
        self.blob, self.tag, self.n, self.codebooks = blob, tag, n, codebooks

    def make(self, eng):
        return eng.Batch(self.n, self.blob, device=0, config=H.model_config(self.tag),
                         codebooks=H.codebooks() if self.codebooks is None else self.codebooks)


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
    """call(d_features, stride, d_pcm) on buffers that start FOFF floats / POFF samples into their allocations; the guard samples
    around the PCM must stay untouched"""
    import torch
    n, nf, stride = f.shape
    d_f = torch.full((FOFF + f.size,), float("nan"), dtype=torch.float32, device="cuda")
    d_f[FOFF:] = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32).ravel()).cuda()
    d_p = torch.full((2 * POFF + n * nf * spf,), GUARD, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    call(d_f.data_ptr() + 4 * FOFF, nf, stride, d_p.data_ptr() + 2 * POFF, spf)
    out = d_p.cpu().numpy()
    assert (out[:POFF] == GUARD).all() and (out[-POFF:] == GUARD).all(), "the group wrote outside its PCM buffer"
    return out[POFF:-POFF].reshape(n, nf * spf)


def device_decode(group, pk):
    import torch
    n, P, _ = pk.shape
    d_k = torch.zeros((FOFF + pk.size,), dtype=torch.uint8, device="cuda")
    d_k[FOFF:] = torch.from_numpy(np.ascontiguousarray(pk).ravel()).cuda()
    d_p = torch.full((2 * POFF + n * P * 640,), GUARD, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    group.decode_device(d_k.data_ptr() + FOFF, P, d_p.data_ptr() + 2 * POFF)
    out = d_p.cpu().numpy()
    assert (out[:POFF] == GUARD).all() and (out[-POFF:] == GUARD).all(), "the group wrote outside its PCM buffer"
    return out[POFF:-POFF].reshape(n, P * 640)


class Pair:
    """the same members twice: `g` driven through a group, `r` through member calls.  spc pins the group's streams per CTA;
    lane_stream sets LPCNET_B200_FLOAT_LANE_STREAM for the members and the group."""

    def __init__(self, eng, mp, members, spc=None, lane_stream=False):
        self.members = members
        if lane_stream:
            mp.setenv("LPCNET_B200_FLOAT_LANE_STREAM", "1")
        self.g = [m.make(eng) for m in members]
        self.r = [m.make(eng) for m in members]
        if spc:
            mp.setenv("LPCNET_B200_STREAMS_PER_CTA", str(spc))
        self.group = eng.Group(self.g)
        mp.delenv("LPCNET_B200_STREAMS_PER_CTA", raising=False)
        mp.delenv("LPCNET_B200_FLOAT_LANE_STREAM", raising=False)
        self.rows = np.cumsum([0] + [m.n for m in members])
        self.n = int(self.rows[-1])

    def split(self, a):
        return [a[self.rows[k]:self.rows[k + 1]] for k in range(len(self.members))]

    def synth(self, f, spf=160, device=False):
        got = device_synth(self.group.synthesize_device, f, spf) if device else self.group.synthesize(f, spf)
        want = np.concatenate([b.synthesize(x, spf) for b, x in zip(self.r, self.split(f))])
        check(got, want, "group synthesize%s (spf %d)" % ("_device" if device else "", spf))
        return got

    def decode(self, p, device=False):
        got = device_decode(self.group, p) if device else self.group.decode(p)
        want = np.concatenate([b.decode(x) for b, x in zip(self.r, self.split(p))])
        check(got, want, "group decode%s" % ("_device" if device else ""))
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

    def oracle(self, got, f, spf=160):
        for k, (m, x) in enumerate(zip(self.members, self.split(f))):
            want = H.oracle_synth(x[:, :, :20], "float", tag=m.tag, model_blob=m.blob) if spf == 160 else oracle_spf(x, m, spf)
            check(self.split(got)[k], want, "member %d vs the oracle" % k)

    def close(self):
        self.group.close()
        for b in self.g + self.r:
            b.close()


def oracle_spf(f, m, spf):
    """the float oracle's PCM of the rows `f` (fresh states), one feature vector per `spf` samples"""
    L = H.oracle_lib()
    model = H.oracle_model("float", m.tag, m.blob)
    f = np.ascontiguousarray(f[:, :, :20], dtype=np.float32)
    out = np.zeros((f.shape[0], f.shape[1] * spf), np.int16)

    def one(s):
        st = L.oracle_state_create(model)
        for t in range(f.shape[1]):
            L.oracle_synthesize(st, f[s, t].ctypes.data, out[s, t * spf:].ctypes.data, spf)
        L.oracle_state_destroy(st)
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:        # (ctypes releases the GIL)
        list(ex.map(one, range(f.shape[0])))
    return out


def feats(n, T, base=0):
    return make_feature_batch(range(base, base + n), T)


def in_calls(P, f, **kw):
    """3 + 18 frames: state across calls, the second call crosses a chunk"""
    return np.concatenate([P.synth(f[:, :T1], **kw), P.synth(f[:, T1:], **kw)], axis=1)


# ---- models ----
def test_seeded_models_match_members_and_oracle(eng, clean_env):
    P = Pair(eng, clean_env, [Member(H.blob("float"), n=5), Member(seeded_blob(11), n=40), Member(seeded_blob(12), n=17)])
    f = feats(P.n, T1 + T2)
    P.oracle(in_calls(P, f), f)
    P.check_state()
    P.check_tails()
    ms, launches = P.group.last_sample_kernel_ms()
    assert ms > 0 and launches > 0
    P.close()


def test_variants_in_one_group(eng, clean_env):
    """END2END, FEATURES_DELAY 0 and 1 and the default in one launch: the members' silent prefixes differ in length"""
    P = Pair(eng, clean_env, [Member(H.blob("float", t), tag=t, n=6 + i) for i, t in enumerate(["e2e", "delay0", "delay1", ""])])
    f = feats(P.n, 19, 300)
    got = np.concatenate([P.synth(f[:, :1]), P.synth(f[:, 1:])], axis=1)
    P.oracle(got, f)
    P.check_state()
    P.check_tails()
    P.close()


@pytest.mark.parametrize("spc", [None, 32])
@pytest.mark.parametrize("na", [256, 128])
def test_smaller_gru_a(eng, clean_env, na, spc):
    tag = "na%d" % na
    P = Pair(eng, clean_env, [Member(H.blob("float", tag), tag=tag, n=7), Member(seeded_blob(21, na), tag=tag, n=30),
                              Member(H.stress_blob("skew", "float", na=na), tag=tag, n=5)], spc=spc)
    f = feats(P.n, 5, 400)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


@pytest.mark.parametrize("spc", [1, 4, 32])
def test_stress_models(eng, clean_env, spc):
    """every float stress model (dense, split and evenly cut GRU_B lists, skewed GRU_A lists, weights at the limits) and the
    default model in one launch: members with and without the dense GRU_B chain share it"""
    import gen_model
    ms = [Member(H.stress_blob(name, "float"), n=3 + 2 * i) for i, name in enumerate(gen_model.stress_names())]
    ms.append(Member(H.blob("float"), n=6))
    P = Pair(eng, clean_env, ms, spc=spc)
    f = feats(P.n, 7, 200)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


# ---- geometry ----
@pytest.mark.parametrize("spc", [1, 2, 3, 4, 5, 17, 32])
def test_pinned_spc(eng, clean_env, spc):
    """both kernels at every S and past it; member boundaries inside what would otherwise be one CTA (sizes that are not
    multiples of the slots)"""
    P = Pair(eng, clean_env, [Member(H.blob("float"), n=3), Member(seeded_blob(31), n=13), Member(seeded_blob(32), n=21)], spc=spc)
    f = feats(P.n, 4, 500)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


@pytest.mark.parametrize("spc", [1, 2, 3, 4])
def test_pinned_small_spc_lane_stream(eng, clean_env, spc):
    """LPCNET_B200_FLOAT_LANE_STREAM: the lane == stream kernel at the spc that would take the neuron-per-lane kernel"""
    from lpcnet_b200 import api
    sizes = [3, 13, 21]
    assert api.group_plan_float(sizes, 132, spc, lane_stream=True)[0] == "lane"
    P = Pair(eng, clean_env, [Member(H.blob("float"), n=sizes[0]), Member(seeded_blob(31), n=sizes[1]),
                              Member(seeded_blob(32), n=sizes[2])], spc=spc, lane_stream=True)
    f = feats(P.n, 4, 550)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


@pytest.mark.parametrize("m", [1, 2, 4])
@pytest.mark.parametrize("extra", [0, 1])
def test_automatic_plan_switch_points(eng, clean_env, sms, m, extra):
    """m x SMs streams and one more, split unevenly over two members: spc 1 -> 2, 2 -> 3 (S 4), 4 -> 5 (lane == stream)"""
    from lpcnet_b200 import api
    total = m * sms + extra
    sizes = [m * (sms // 3), total - m * (sms // 3)]                   # (a multiple of m: the plan at spc m fits exactly when extra is 0)
    kernel, spc, _, _ = api.group_plan_float(sizes, sms)
    assert spc == m + extra and kernel == ("lane" if spc > 4 else "neuron")
    P = Pair(eng, clean_env, [Member(seeded_blob(41), n=sizes[0]), Member(seeded_blob(42), n=sizes[1])])
    f = make_feature_batch(np.arange(P.n) % 97 + 600, 3)
    P.synth(f)
    P.check_state()
    P.check_tails(40)
    P.close()


def test_more_than_one_wave(eng, clean_env, sms):
    half = 16 * sms
    P = Pair(eng, clean_env, [Member(H.blob("float"), n=half + 100), Member(seeded_blob(51), n=half - 99)])    # 32 x SMs + 1 streams
    f = make_feature_batch(np.arange(P.n) % 97 + 700, 3)
    P.synth(f)
    P.check_state()
    P.close()


def test_sixteen_members(eng, clean_env):
    ms = [Member(H.blob("float") if k % 4 == 0 else seeded_blob(60 + k), n=1 + k) for k in range(16)]
    P = Pair(eng, clean_env, ms)
    f = feats(P.n, 5, 750)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.check_tails(40)
    P.close()


# ---- call shapes ----
def shape_members():
    return [Member(H.blob("float"), n=5), Member(seeded_blob(33), n=9), Member(H.blob("float"), n=2)]


@pytest.mark.parametrize("spf,path", [(80, "host"), (320, "device"), (1, "device")])
def test_samples_per_frame(eng, clean_env, spf, path):
    """group synthesis at `spf` samples per feature vector (3 then 18 frames), host buffers or `_device` ones at non-zero
    offsets; the oracle synthesizes `spf` samples per vector too"""
    P = Pair(eng, clean_env, shape_members())
    f = feats(P.n, T1 + T2, 800)
    P.oracle(in_calls(P, f, spf=spf, device=path == "device"), f, spf)
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
    """group decode of 5 packets (20 frames: across the 16-frame chunk) with per-member codebooks, then synthesis, then 5 more
    packets"""
    import gen_model
    other = np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=78)]).astype(np.float32)
    P = Pair(eng, clean_env, [Member(H.blob("float"), n=5), Member(seeded_blob(34), n=6, codebooks=other), Member(H.blob("float"), n=3)])
    pk = np.stack([make_packets(7700 + s, 10) for s in range(P.n)])
    got = P.decode(pk[:, :5], path == "device")
    for k in (0, 2):      # default model and codebooks: the oracle decodes them
        check(P.split(got)[k], H.oracle_decode(P.split(pk)[k][:, :5], "float"), "member %d decode vs the oracle" % k)
    P.synth(feats(P.n, 3, 7800), device=path == "device")
    P.check_tails()
    P.decode(pk[:, 5:], path == "device")
    P.check_state()
    P.check_tails()
    P.close()


# ---- state ----
def test_lifecycle_between_group_calls(eng, clean_env):
    ms = [Member(H.blob("float"), n=6), Member(H.blob("float", "delay1"), tag="delay1", n=5), Member(seeded_blob(61), n=7)]
    P = Pair(eng, clean_env, ms)
    f = feats(P.n, 40, 900)
    P.synth(f[:, 0:3])
    P.both(lambda k, b: b.reset_streams([1, 3]) if k == 0 else None)             # reset inside some members only
    P.synth(f[:, 3:4])                                                           # inside FEATURES_DELAY for the reset streams
    P.synth(f[:, 4:6])
    P.check_tails()
    P.both(lambda k, b: b.reset() if k == 1 else None)
    P.synth(f[:, 6:9])
    st = {}
    P.both(lambda k, b: st.__setitem__((id(b), k), b.export_state(2)) if k == 2 else None)
    P.both(lambda k, b: b.import_state(0, st[(id(b), k)]) if k == 2 else None)
    P.synth(f[:, 9:11])
    snaps = {}
    P.both(lambda k, b: snaps.__setitem__(id(b), b.snapshot()) if k == 0 else None)
    P.synth(f[:, 11:13])
    P.both(lambda k, b: b.restore(snaps[id(b)]) if k == 0 else None)
    P.check_tails()
    P.synth(f[:, 13:15])
    P.both(lambda k, b: b.free_snapshot(snaps[id(b)]) if k == 0 else None)
    P.both(lambda k, b: b.frame_network_deferred(f[P.rows[k]:P.rows[k + 1], 15]) if k != 1 else None)
    P.both(lambda k, b: b.reset_streams([4]) if k == 2 else None)
    P.both(lambda k, b: b.frame_network_deferred(f[P.rows[k]:P.rows[k + 1], 16]) if k != 1 else None)
    P.both(lambda k, b: b.frame_network_flush() if k != 1 else None)
    P.check_tails()
    P.synth(f[:, 17:35])
    P.check_state()
    P.check_tails()
    P.close()


# ---- ordering and refusals ----
def test_device_calls_on_two_streams_mixed_with_member_calls(eng, clean_env):
    import torch
    P = Pair(eng, clean_env, [Member(H.blob("float"), n=6), Member(seeded_blob(81), n=10)])
    T = 5
    fs = [feats(P.n, T, 1100 + 50 * i) for i in range(3)]
    d_f = [torch.from_numpy(x).cuda() for x in fs]
    d_p = [torch.zeros((P.n, T * 160), dtype=torch.int16, device="cuda") for _ in fs]
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    extra = feats(6, 2, 1300)
    P.group.synthesize_device(d_f[0].data_ptr(), T, 20, d_p[0].data_ptr(), 160, s1.cuda_stream)
    got_m = P.g[0].synthesize(extra)                                            # member host call while group work is queued
    P.group.synthesize_device(d_f[1].data_ptr(), T, 20, d_p[1].data_ptr(), 160, s2.cuda_stream)
    P.g[1].reset_streams([0, 9])
    P.group.synthesize_device(d_f[2].data_ptr(), T, 20, d_p[2].data_ptr(), 160, s1.cuda_stream)
    s1.synchronize(); s2.synchronize()
    want0 = np.concatenate([b.synthesize(x) for b, x in zip(P.r, P.split(fs[0]))])
    want_m = P.r[0].synthesize(extra)
    want1 = np.concatenate([b.synthesize(x) for b, x in zip(P.r, P.split(fs[1]))])
    P.r[1].reset_streams([0, 9])
    want2 = np.concatenate([b.synthesize(x) for b, x in zip(P.r, P.split(fs[2]))])
    check(got_m, want_m, "member call between group calls")
    for i, w in enumerate((want0, want1, want2)):
        check(d_p[i].cpu().numpy(), w, "group _device call %d" % i)
    P.check_state()
    P.close()


def test_refusals(eng, clean_env):
    import lpcnet_b200
    import torch
    a = eng.Batch(2, H.blob("float"), device=0, config=H.model_config(""))
    b = eng.Batch(2, seeded_blob(91), device=0, config=H.model_config(""))
    i8 = eng.Batch(2, H.blob("int8"), device=0, config=H.model_config(""))
    f256 = eng.Batch(2, H.blob("float", "na256"), device=0, config=H.model_config("na256"))
    for members, what in [([a, i8], "float"), ([i8, a], "float"), ([a, b, i8], "float"), ([a, f256], "GRU_A")]:
        with pytest.raises(lpcnet_b200.LPCNetB200Error, match=what):
            eng.Group(members)
    g = eng.Group([a, b])
    sink = torch.zeros((2, 160 * 4), dtype=torch.int16, device="cuda")
    b.set_pcm_sink(sink.data_ptr(), 160 * 4, 0)
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="sink"):
        g.synthesize(feats(4, 2))
    b.set_pcm_sink(None, 0, 0)
    g.synthesize(feats(4, 2))
    g.close()
    for x in (a, b, i8, f256):
        x.close()
