"""GPU tests (-m gpu) of groups (lpcnet_b200_group_*): the synthesize / decode calls of several int8 batches of one GRU_A size
run as one call, with one per-sample launch for all their streams.

The contract: a group call leaves every member exactly as the member's own call on its rows of the inputs would, PCM and state,
bit for bit, from any member state.  So every case runs the same sequence twice on identically prepared batches, once with group
calls and once with member calls, and compares the PCM and every stream's exported state; several cases also compare with the
CPU restatement of each member's model."""
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "EXACT_CVT", "FCW_NODES")


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


def seeded_blob(seed, na=None):
    """int8 blob of gen_model.make_model(seed): the default model's shape with other weights"""
    import gen_model
    from lpcnet_b200 import api
    key = (seed, na)
    if key not in _SEEDED:
        common, only8, _ = gen_model.make_model(seed, na=na)
        _SEEDED[key] = api.write_blob([(n, t, a.tobytes()) for n, t, a in common + only8])
    return _SEEDED[key]


class Member:
    """one member's model: blob, header tag of its switches (oracle), create-time environment"""

    def __init__(self, blob, tag="", n=8, exact=False, codebooks=None):
        self.blob, self.tag, self.n, self.exact, self.codebooks = blob, tag, n, exact, codebooks

    def make(self, eng, mp):
        if self.exact:
            mp.setenv("LPCNET_B200_EXACT_CVT", "1")
        b = eng.Batch(self.n, self.blob, device=0, config=H.model_config(self.tag),
                      codebooks=H.codebooks() if self.codebooks is None else self.codebooks)
        mp.delenv("LPCNET_B200_EXACT_CVT", raising=False)
        return b


class Pair:
    """the same members twice: `g` driven through a group, `r` through member calls"""

    def __init__(self, eng, mp, members, spc=None):
        self.members = members
        self.g = [m.make(eng, mp) for m in members]
        self.r = [m.make(eng, mp) for m in members]
        if spc:
            mp.setenv("LPCNET_B200_STREAMS_PER_CTA", str(spc))
        self.group = eng.Group(self.g)
        mp.delenv("LPCNET_B200_STREAMS_PER_CTA", raising=False)
        self.rows = np.cumsum([0] + [m.n for m in members])
        self.n = int(self.rows[-1])

    def split(self, a):
        return [a[self.rows[k]:self.rows[k + 1]] for k in range(len(self.members))]

    def synth(self, f, spf=160):
        got = self.group.synthesize(f, spf)
        want = np.concatenate([b.synthesize(x, spf) for b, x in zip(self.r, self.split(f))])
        check(got, want, "group synthesize")
        return got

    def decode(self, p):
        got = self.group.decode(p)
        want = np.concatenate([b.decode(x) for b, x in zip(self.r, self.split(p))])
        check(got, want, "group decode")
        return got

    def both(self, fn):
        """a member lifecycle call, made on both sides: fn(k, batch)"""
        for side in (self.g, self.r):
            for k, b in enumerate(side):
                fn(k, b)

    def check_state(self):
        for k in range(len(self.members)):
            for s in range(self.members[k].n):
                a, b = self.g[k].export_state(s), self.r[k].export_state(s)
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "member %d stream %d: state differs" % (k, s)

    def check_tails(self, samples=90):
        for k in range(len(self.members)):
            check(self.g[k].synthesize_tail(samples), self.r[k].synthesize_tail(samples), "member %d tail" % k)

    def oracle(self, got, f):
        for k, (m, x) in enumerate(zip(self.members, self.split(f))):
            want = H.oracle_synth(x, "int8", tag=m.tag, model_blob=m.blob)
            check(self.split(got)[k], want, "member %d vs the oracle" % k)

    def close(self):
        self.group.close()
        for b in self.g + self.r:
            b.close()


def check(got, want, what):
    assert got.shape == want.shape, what
    if not np.array_equal(got, want):
        s, t = np.argwhere(got != want)[0]
        raise AssertionError("%s: first difference at stream %d sample %d (%d vs %d)" % (what, s, t, got[s, t], want[s, t]))


def feats(n, T, base=0):
    return make_feature_batch(range(base, base + n), T)


# ---- models ----
def test_seeded_models_match_members_and_oracle(eng, clean_env):
    P = Pair(eng, clean_env, [Member(H.blob("int8"), n=5), Member(seeded_blob(11), n=40), Member(seeded_blob(12), n=17)])
    f = feats(P.n, 21)
    got = np.concatenate([P.synth(f[:, :3]), P.synth(f[:, 3:])], axis=1)     # state across calls, the second crosses a chunk
    P.oracle(got, f)
    P.check_state()
    P.check_tails()
    ms, launches = P.group.last_sample_kernel_ms()
    assert ms > 0 and launches > 0
    P.close()


def test_same_blob_members(eng, clean_env):
    P = Pair(eng, clean_env, [Member(H.blob("int8"), n=9) for _ in range(4)])
    f = feats(P.n, 6, 100)
    P.oracle(P.synth(f), f)
    P.close()


def test_stress_models_mixed_rounding(eng, clean_env):
    """skewed block lists, fewer dual_fc rows in shared memory, and `hot`, whose range proof rules out the conversion-free
    rounding, next to members that allow it; one more member with the conversion unit forced"""
    import gen_model
    names = [n for n in gen_model.stress_names() if n != "overflow"]       # the loader refuses the int8 blob of "overflow"
    ms = [Member(H.stress_blob(name), n=3 + 2 * i) for i, name in enumerate(names)]
    ms.append(Member(seeded_blob(13), n=6, exact=True))
    P = Pair(eng, clean_env, ms)
    f = feats(P.n, 7, 200)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


def test_variants_in_one_group(eng, clean_env):
    """END2END, FEATURES_DELAY 0 and 1 and the default in one launch: the members' silent prefixes differ in length"""
    P = Pair(eng, clean_env, [Member(H.blob("int8", t), tag=t, n=6 + i) for i, t in enumerate(["e2e", "delay0", "delay1", ""])])
    f = feats(P.n, 19, 300)
    got = np.concatenate([P.synth(f[:, :1]), P.synth(f[:, 1:])], axis=1)
    P.oracle(got, f)
    P.check_tails()
    P.close()


@pytest.mark.parametrize("na", [256, 128])
def test_smaller_gru_a(eng, clean_env, na):
    tag = "na%d" % na
    P = Pair(eng, clean_env, [Member(H.blob("int8", tag), tag=tag, n=7), Member(seeded_blob(21, na), tag=tag, n=30),
                              Member(H.stress_blob("skew", na=na), tag=tag, n=5)])
    f = feats(P.n, 5, 400)
    P.oracle(P.synth(f), f)
    P.check_state()
    P.close()


# ---- geometry ----
@pytest.mark.parametrize("spc", [1, 5, 16, 17, 32])
def test_pinned_spc(eng, clean_env, spc):
    """both schedules; member boundaries inside what would otherwise be one CTA (sizes that are not multiples of spc)"""
    P = Pair(eng, clean_env, [Member(H.blob("int8"), n=3), Member(seeded_blob(31), n=13), Member(seeded_blob(32), n=21)], spc=spc)
    f = feats(P.n, 4, 500)
    P.oracle(P.synth(f), f)
    P.close()


@pytest.mark.parametrize("sizes", [[1, 2], [700, 900, 500]], ids=["small", "large"])
def test_automatic_plan(eng, clean_env, sizes):
    P = Pair(eng, clean_env, [Member(seeded_blob(41 + i), n=n) for i, n in enumerate(sizes)])
    f = feats(P.n, 4, 600)
    P.synth(f)
    P.check_tails(40)
    P.close()


def test_more_than_one_wave(eng, clean_env):
    P = Pair(eng, clean_env, [Member(H.blob("int8"), n=2500), Member(seeded_blob(51), n=2100)])    # 4600 > 32 x 132 streams
    f = feats(P.n, 3, 700)
    P.synth(f)
    P.close()


# ---- state ----
def test_lifecycle_between_group_calls(eng, clean_env):
    ms = [Member(H.blob("int8"), n=6), Member(H.blob("int8", "delay1"), tag="delay1", n=5), Member(seeded_blob(61), n=7)]
    P = Pair(eng, clean_env, ms)
    f = feats(P.n, 40, 800)
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


def test_reset_all_members_then_group(eng, clean_env):
    P = Pair(eng, clean_env, [Member(H.blob("int8", "delay0"), tag="delay0", n=4), Member(H.blob("int8"), n=4)])
    f = feats(P.n, 8, 900)
    P.synth(f[:, :4])
    P.both(lambda k, b: b.reset())
    P.synth(f[:, 4:])
    P.check_state()
    P.close()


# ---- decode ----
def test_decode_per_member_codebooks_mixed_with_synthesis(eng, clean_env):
    import gen_model
    other = np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=77)]).astype(np.float32)
    ms = [Member(H.blob("int8"), n=5), Member(seeded_blob(71), n=6, codebooks=other), Member(H.blob("int8"), n=3)]
    P = Pair(eng, clean_env, ms)
    pk = np.stack([make_packets(s, 4) for s in range(P.n)])
    got = P.decode(pk[:, :2])
    for k in (0, 2):      # default codebooks: the oracle decodes them
        check(P.split(got)[k], H.oracle_decode(P.split(pk)[k][:, :2], "int8"), "member %d decode vs the oracle" % k)
    P.synth(feats(P.n, 3, 1000))
    P.decode(pk[:, 2:])
    P.check_state()
    P.check_tails()
    P.close()


# ---- ordering and refusals ----
def test_device_calls_on_two_streams_mixed_with_member_calls(eng, clean_env):
    import torch
    P = Pair(eng, clean_env, [Member(H.blob("int8"), n=6), Member(seeded_blob(81), n=10)])
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
    a = eng.Batch(2, H.blob("int8"), device=0, config=H.model_config(""))
    b = eng.Batch(2, seeded_blob(91), device=0, config=H.model_config(""))
    c256 = eng.Batch(2, H.blob("int8", "na256"), device=0, config=H.model_config("na256"))
    fl = eng.Batch(2, H.blob("float"), device=0, config=H.model_config(""))
    for members, what in [([a, c256], "GRU_A"), ([a, fl], "float"), ([a, b, a], "twice")]:
        with pytest.raises(lpcnet_b200.LPCNetB200Error, match=what):
            eng.Group(members)
    many = [eng.Batch(1, H.blob("int8"), device=0, config=H.model_config("")) for _ in range(17)]
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="1..16"):
        eng.Group(many)
    eng.Group(many[:16]).close()
    for x in many:
        x.close()
    if eng.device_count() > 1:
        d1 = eng.Batch(2, H.blob("int8"), device=1, config=H.model_config(""))
        with pytest.raises(lpcnet_b200.LPCNetB200Error, match="device"):
            eng.Group([a, d1])
        d1.close()
    # a member with a PCM sink set
    import torch
    sink = torch.zeros((2, 160 * 4), dtype=torch.int16, device="cuda")
    g = eng.Group([a, b])
    a.set_pcm_sink(sink.data_ptr(), 160 * 4, 0)
    with pytest.raises(lpcnet_b200.LPCNetB200Error, match="sink"):
        g.synthesize(feats(4, 2))
    a.set_pcm_sink(None, 0, 0)
    g.synthesize(feats(4, 2))
    g.close()
    for x in (a, b, c256, fl):
        x.close()
