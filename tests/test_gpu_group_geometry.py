"""GPU tests (-m gpu) of groups (lpcnet_b200_group_*) at every launch geometry and call shape: each compiled group kernel
instance (GRU_A 384 / 256 / 128 x conversion-free / conversion-unit rounding x one half / two halves), every pinned
streams-per-CTA value (spc) with member boundaries where one CTA would otherwise hold two members, the automatic plan at its
switch points, past one wave, sixteen members (GROUP_MAX) with members compacted out of the launch while silent, stress
models, and the call shapes: samples per frame other than 160, a feature stride of 36, `_device` buffers at non-zero
offsets, and decode across a 16-frame chunk.

Every case runs each call twice on identically prepared members, once through the group and once through the members' own
calls, and compares the PCM, the exported state of every stream (a spread of streams in members of more than STATE_ALL) and
a tail after the calls, bit for bit; and each member's PCM with the CPU restatement of its model.

Input pool (as in test_gpu_geometry.py): group row r takes entry r mod K of a pool of K feature sequences, K prime, so that
rows 1..64 apart or a whole wave apart get different inputs, and the oracle runs once per model, on the pool only.  At each
size the members alternate between two blobs, the variant's default and a gen_model seed: a CTA that reads another member's
parameters shows up against the oracle as well as against the member calls."""
import functools
import os
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

gpu = pytest.mark.gpu

T1, T2 = 3, 18                  # calls of 3 + 18 frames: state carried across calls, the second crosses the 16-frame chunk
T = T1 + T2
SPC_MAX, HALF, GROUP_MAX = 32, 16, 16    # engine.h STREAMS_PER_CTA, HALF, GROUP_MAX
N_BIG = 32768
KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "EXACT_CVT", "FCW_NODES")
TAGS = {384: "", 256: "na256", 128: "na128"}
SEED = {384: 3101, 256: 3102, 128: 3103}     # gen_model seed of each size's second blob
STATE_ALL = 256
FOFF, POFF, GUARD = 12, 5, -12345            # `_device` buffers: features 12 floats in, PCM 5 samples in, guard value around the PCM


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


# ---- the input pool ----
def _is_prime(k):
    return k > 1 and all(k % d for d in range(2, int(k ** 0.5) + 1))


def pool_distinct(k, sms, n_max):
    wave = SPC_MAX * sms
    return all(d % k for d in list(range(1, 2 * SPC_MAX + 1)) + list(range(wave, n_max, wave)))


@pytest.fixture(scope="module")
def K(sms):
    k = 67
    while not (_is_prime(k) and pool_distinct(k, sms, N_BIG)):
        k += 1
    return k


@functools.lru_cache(None)
def pool_features(k):
    return make_feature_batch(range(7000, 7000 + k), T)


# ---- models ----
_SEEDED = {}


def seeded_blob(seed, na):
    """int8 blob of gen_model.make_model(seed) with `na` GRU_A units: the default model's shape with other weights"""
    import gen_model
    from lpcnet_b200 import api
    key = (seed, na)
    if key not in _SEEDED:
        common, only8, _ = gen_model.make_model(seed, na=None if na == 384 else na)
        _SEEDED[key] = api.write_blob([(n, t, a.tobytes()) for n, t, a in common + only8])
    return _SEEDED[key]


BEYOND_BIAS, BEYOND_RESET = 1024.0, -8.0


@functools.lru_cache(None)
def beyond_blob(na):
    """A model whose GRU_A accumulators really leave the conversion-free rounding's range, without saturating what they feed:
    the candidate-gate recurrent bias of neuron group 0 is +-BEYOND_BIAS (about 1.7e7 accumulator units, past 2^22 on every
    sample; the loader falls back to the conversion unit), and the same neurons' reset-gate bias BEYOND_RESET keeps r small, so
    that r times the candidate's recurrent part stays where tanh is not flat and a wrong conversion changes the state."""
    import gen_model
    from lpcnet_b200 import api
    common, only8, _ = gen_model.make_model(3400 + na, na=None if na == 384 else na)
    arrs = {n: a for n, _, a in common + only8}
    sign = np.where(np.arange(8) % 2, -1.0, 1.0).astype(np.float32)
    for name in ("sparse_gru_a_subias", "sparse_gru_a_bias"):
        arrs[name][1, 2 * na + np.arange(8)] = np.float32(BEYOND_BIAS) * sign
        arrs[name][1, na + np.arange(8)] = np.float32(BEYOND_RESET)
    assert 4 * 4194304.0 < gen_model.cvt_bound(arrs, na) < 2.0 ** 31
    return api.write_blob([(n, t, a.tobytes()) for n, t, a in common + only8])


def model_blob(na, name):
    """name: "default" (the size's own blob), "seed<k>" (gen_model.make_model(k)), "beyond" (beyond_blob) or a stress model's
    name"""
    if name == "default":
        return H.blob("int8", TAGS[na])
    if name.startswith("seed"):
        return seeded_blob(int(name[4:]), na)
    if name == "beyond":
        return beyond_blob(na)
    return H.stress_blob(name, na=na)


@functools.lru_cache(None)
def image_layout(na, name):
    """layout words of lpcnet_b200_debug_image of the blob (host only): [5] shared-memory footprint, [21] 1 = the loader's range
    proof allows the conversion-free rounding"""
    import lpcnet_b200
    import image_replay
    r, _, lay = image_replay.int8_image(lpcnet_b200.lib(), model_blob(na, name))
    assert r > 0, "the loader refused %s at %d units" % (name, na)
    return lay


@functools.lru_cache(None)
def pool_pcm(k, na, name):
    """the oracle's PCM of every pool entry over T frames from a fresh state"""
    return H.oracle_synth(pool_features(k), "int8", tag=TAGS[na], model_blob=model_blob(na, name))


def oracle_spf(f, na, name, spf):
    """the oracle's PCM of the rows `f` (fresh states), one feature vector per `spf` samples"""
    L = H.oracle_lib()
    m = H.oracle_model("int8", TAGS[na], model_blob(na, name))
    f = np.ascontiguousarray(f[:, :, :20], dtype=np.float32)
    out = np.zeros((f.shape[0], f.shape[1] * spf), np.int16)

    def one(s):
        st = L.oracle_state_create(m)
        for t in range(f.shape[1]):
            L.oracle_synthesize(st, f[s, t].ctypes.data, out[s, t * spf:].ctypes.data, spf)
        L.oracle_state_destroy(st)
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:        # (ctypes releases the GIL)
        list(ex.map(one, range(f.shape[0])))
    return out


class Member:
    """one member: GRU_A size, model name (model_blob), streams, created with LPCNET_B200_EXACT_CVT=1, VQ codebooks"""

    def __init__(self, na, name, n, exact=False, codebooks=None):
        self.na, self.name, self.n, self.exact, self.codebooks = na, name, n, exact, codebooks

    @property
    def blob(self):
        return model_blob(self.na, self.name)

    @property
    def tag(self):
        return TAGS[self.na]

    def fast_cvt(self):
        """the member's own launches take the conversion-free rounding"""
        return bool(image_layout(self.na, self.name)[21]) and not self.exact

    def make(self, eng, mp):
        if self.exact:
            mp.setenv("LPCNET_B200_EXACT_CVT", "1")
        b = eng.Batch(self.n, self.blob, device=0, config=H.model_config(self.tag),
                      codebooks=H.codebooks() if self.codebooks is None else self.codebooks)
        mp.delenv("LPCNET_B200_EXACT_CVT", raising=False)
        return b

    def __repr__(self):
        return "%s%s x%d" % (self.name, "/exact" if self.exact else "", self.n)


def check(got, want, what):
    assert got.shape == want.shape, "%s: shape %s vs %s" % (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        bad = np.flatnonzero((got != want).any(axis=1))
        t = int(np.flatnonzero(got[bad[0]] != want[bad[0]])[0])
        raise AssertionError("%s: %d of %d streams differ, first at stream %d sample %d (%d vs %d)"
                             % (what, bad.size, got.shape[0], bad[0], t, got[bad[0], t], want[bad[0], t]))


def check_pool(got, want_pool, entry, what):
    """stream s of `got` must equal row entry[s] of `want_pool` (per-stream digests; names the first stream and sample)"""
    assert got.shape == (len(entry), want_pool.shape[1]), "%s: shape %s" % (what, got.shape)
    bad = np.flatnonzero(H.stream_digests(got) != H.stream_digests(want_pool)[entry])
    if bad.size:
        s = int(bad[0])
        t = int(np.flatnonzero(got[s] != want_pool[entry[s]])[0])
        raise AssertionError("%s: %d of %d streams differ, first (stream, sample) = (%d, %d)" % (what, bad.size, len(entry), s, t))


def group_synth_device(group, f, spf):
    """group.synthesize_device on buffers that start FOFF floats / POFF samples into their allocations, on the group's own
    stream; the guard samples around the PCM must stay untouched"""
    import torch
    n, nf, stride = f.shape
    d_f = torch.full((FOFF + f.size,), float("nan"), dtype=torch.float32, device="cuda")
    d_f[FOFF:] = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32).ravel()).cuda()
    d_p = torch.full((2 * POFF + n * nf * spf,), GUARD, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    group.synthesize_device(d_f.data_ptr() + 4 * FOFF, nf, stride, d_p.data_ptr() + 2 * POFF, spf)
    out = d_p.cpu().numpy()
    assert (out[:POFF] == GUARD).all() and (out[-POFF:] == GUARD).all(), "the group wrote outside its PCM buffer"
    return out[POFF:-POFF].reshape(n, nf * spf)


def group_decode_device(group, pk):
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
        assert self.group.n == self.n

    def split(self, a):
        return [a[self.rows[k]:self.rows[k + 1]] for k in range(len(self.members))]

    def synth(self, f, spf=160, device=False):
        got = group_synth_device(self.group, f, spf) if device else self.group.synthesize(f, spf)
        want = np.concatenate([b.synthesize(x, spf) for b, x in zip(self.r, self.split(f))])
        check(got, want, "group synthesize%s (spf %d)" % ("_device" if device else "", spf))
        return got

    def decode(self, p, device=False):
        got = group_decode_device(self.group, p) if device else self.group.decode(p)
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
            streams = range(m.n) if m.n <= STATE_ALL else sorted(set([0, 1, m.n - 2, m.n - 1] + list(range(0, m.n, m.n // 24))))
            for s in streams:
                a, b = self.g[k].export_state(s), self.r[k].export_state(s)
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "member %d (%r) stream %d: state differs" % (k, m, s)

    def check_tails(self, samples=90):
        for k in range(len(self.members)):
            check(self.g[k].synthesize_tail(samples), self.r[k].synthesize_tail(samples), "member %d tail" % k)

    def close(self):
        self.group.close()
        for b in self.g + self.r:
            b.close()


def run_pool(P, K, oracle=None):
    """group rows from the pool in calls of T1 + T2 frames against member calls; each member (or those listed in `oracle`)
    against the pool oracle of its model; then state and tails"""
    entry = np.arange(P.n) % K
    f = pool_features(K)[entry]
    got = np.concatenate([P.synth(f[:, :T1]), P.synth(f[:, T1:])], axis=1)
    for k, (m, g, e) in enumerate(zip(P.members, P.split(got), P.split(entry))):
        if oracle is None or k in oracle:
            check_pool(g, pool_pcm(K, m.na, m.name), e, "member %d (%r) vs the oracle" % (k, m))
    P.check_state()
    P.check_tails()
    return got


def schedule(spc):
    return "onehalf" if spc <= HALF else "twohalves"


def kernel_of(members, spc):
    """the group kernel instance a launch of these members at `spc` runs: (GRU_A units, rounding, schedule)"""
    return (members[0].na, "cvtfree" if all(m.fast_cvt() for m in members) else "cvtunit", schedule(spc))


# ---- 1 + 2. every pinned spc at every size, and every kernel instance ----
def ragged(spc):
    return max(1, 2 * spc // 3)


def pinned_members(na, spc, variant=""):
    """A single stream; two full CTAs and a last one of spc - 1 streams (three full ones at spc 1); with two halves, one member
    whose last CTA leaves half B empty (ceil(spc / 2) streams) and one whose half B ends early; with one half, a member of one
    full CTA and a ragged one.  The members alternate between the default blob and a seeded one.  variant "exact": the second
    member is created with LPCNET_B200_EXACT_CVT=1; "hot": one more member of the "hot" stress model; either puts the whole
    group on the conversion unit."""
    sizes = [1, 2 * spc + max(1, spc - 1)]
    sizes += [spc + (spc + 1) // 2, spc + ragged(spc)] if spc > HALF else [spc + ragged(spc)]
    names = ["default", "seed%d" % SEED[na]]
    ms = [Member(na, names[i % 2], n, exact=(variant == "exact" and i == 1)) for i, n in enumerate(sizes)]
    if variant == "hot":
        ms.append(Member(na, "hot", spc + ragged(spc)))
    return ms


CVT_SPC = (1, 9, 17, 25, 32)
PINNED = [(na, spc, "") for na in TAGS for spc in range(1, SPC_MAX + 1)]
PINNED += [(na, spc, v) for v in ("exact", "hot") for na in TAGS for spc in CVT_SPC]


def _pinned_id(na, spc, v):
    rounding = "cvtunit-" + v if v else "cvtfree"
    return "na%d-spc%02d-%s-%s" % (na, spc, rounding, schedule(spc))


@gpu
@pytest.mark.parametrize("na,spc,variant", [pytest.param(*c, id=_pinned_id(*c)) for c in PINNED])
def test_pinned_spc(eng, clean_env, K, na, spc, variant):
    ms = pinned_members(na, spc, variant)
    assert kernel_of(ms, spc) == (na, "cvtunit" if variant else "cvtfree", schedule(spc))
    P = Pair(eng, clean_env, ms, spc=spc)
    run_pool(P, K)
    P.close()


def test_every_group_kernel_instance_is_reached():
    """(no GPU) the pinned cases reach all 12 group kernel instances; the rounding is derived from the members: the loader's
    verdict on each blob (layout[21] of lpcnet_b200_debug_image) and LPCNET_B200_EXACT_CVT at create"""
    reached = {kernel_of(pinned_members(na, spc, v), spc) for na, spc, v in PINNED}
    want = {(na, r, s) for na in TAGS for r in ("cvtfree", "cvtunit") for s in ("onehalf", "twohalves")}
    assert reached == want, sorted(want - reached)
    for na in TAGS:     # the premises: the two blobs of each size allow the conversion-free rounding, "hot" and "beyond" do not
        assert image_layout(na, "default")[21] == 1 and image_layout(na, "seed%d" % SEED[na])[21] == 1
        assert image_layout(na, "hot")[21] == 0
        assert image_layout(na, "beyond")[21] == 0


# ---- 3. the automatic plan at its switch points ----
SWITCH = [(m, p) for m in (1, 16, 32) for p in (0, 1)]      # S = SM count: m x S (+ 1) streams over the members
SPLITS = [(5, 3), (4, 1, 2), (7, 2, 3, 1), (1, 6, 2, 2, 4), (3, 1, 1), (2, 9)]


def plan_rule(sizes, sms):
    """the documented plan: the smallest spc for which the members, each on ceil(n_k / spc) CTAs of its own, fit on `sms` CTAs;
    32 when none does"""
    for spc in range(1, SPC_MAX + 1):
        ctas = sum(-(-n // spc) for n in sizes)
        if ctas <= sms:
            return spc, ctas
    return SPC_MAX, sum(-(-n // SPC_MAX) for n in sizes)


def switch_sizes(m, p, split, sms):
    """m x sms + p streams split unevenly: member k gets m x q_k streams (sum q_k = sms, q_k in proportion to split[k]), the
    first one p more.  At spc m they fill sms CTAs exactly, so the plan is spc m (p = 0) or m + 1 (p = 1, at most 32) on every
    SM count."""
    q = [sms * w // sum(split) for w in split[:-1]]
    q.append(sms - sum(q))
    assert min(q) >= 1
    sizes = [m * v for v in q]
    sizes[0] += p
    return sizes


def _switch_id(na, m, p):
    spc = min(SPC_MAX, m + p)
    return "na%d-n%dS%s-spc%02d-%s%s" % (na, m, "+1" if p else "", spc, schedule(spc), "-2waves" if m == SPC_MAX and p else "")


def test_group_plan_rule():
    """(no GPU) lpcnet_b200_debug_group_plan gives the documented plan at the switch points, on 132 and 114 SMs"""
    from lpcnet_b200 import api
    for sms in (132, 114):
        for i, (m, p) in enumerate(SWITCH):
            sizes = switch_sizes(m, p, SPLITS[i], sms)
            assert api.group_plan(sizes, sms) == plan_rule(sizes, sms), (sms, sizes)
            assert plan_rule(sizes, sms)[0] == min(SPC_MAX, m + p), (sms, sizes)
        assert api.group_plan([5, 100, 1], sms, 7) == (7, 1 + 15 + 1)


@gpu
@pytest.mark.parametrize("na,m,p", [pytest.param(na, m, p, id=_switch_id(na, m, p)) for na in TAGS for m, p in SWITCH])
def test_automatic_plan_switch_points(eng, clean_env, sms, K, na, m, p):
    from lpcnet_b200 import api
    sizes = switch_sizes(m, p, SPLITS[SWITCH.index((m, p))], sms)
    spc, ctas = api.group_plan(sizes, sms)
    assert (spc, ctas) == plan_rule(sizes, sms) and spc == min(SPC_MAX, m + p)
    assert (ctas > sms) == (m == SPC_MAX and p == 1)
    names = ["default", "seed%d" % SEED[na]]
    P = Pair(eng, clean_env, [Member(na, names[i % 2], n) for i, n in enumerate(sizes)])
    run_pool(P, K)
    P.close()


# ---- 4. past one wave ----
@gpu
@pytest.mark.parametrize("na", list(TAGS))
def test_past_one_wave(eng, clean_env, sms, K, na):
    """384 units: 16 members x 2048 = 32768 streams (spc 32, 1024 CTAs: 8 waves on 132 SMs); 256 and 128: 2 x 32 x SMs + 17
    streams over 3 members"""
    from lpcnet_b200 import api
    sizes = [2048] * GROUP_MAX if na == 384 else [SPC_MAX * sms + 5, 40, SPC_MAX * sms - 28]
    names = ["default", "seed%d" % SEED[na]]
    ms = [Member(na, names[i % 2], n) for i, n in enumerate(sizes)]
    spc, ctas = api.group_plan(sizes, sms)
    assert spc == SPC_MAX and ctas > 2 * sms
    P = Pair(eng, clean_env, ms)
    run_pool(P, K, oracle=[k for k, m in enumerate(ms) if m.name == "default"])
    P.close()


# ---- 5. sixteen members, members compacted out of the launch ----
MAX_SIZES = [1, 40, 7, 23, 2, 31, 16, 17, 33, 5, 12, 39, 3, 28, 9, 20]


@gpu
@pytest.mark.parametrize("na", list(TAGS))
def test_sixteen_members(eng, clean_env, na):
    """GROUP_MAX members of distinct seeds.  A 2-frame call right after creation is silent for every member (FEATURES_DELAY 2):
    zeros and no per-sample launch at all.  Then 1 + 18 frames (against the oracle).  Then the first eight members reset right
    before a 1-frame call: they are silent and compacted out, so members 8..15 sit at lower indices of the launch; then only
    the last member live (the others reset); then a call across a chunk with every member's silence ending at another frame."""
    ms = [Member(na, "seed%d" % (3200 + 16 * list(TAGS).index(na) + k), n) for k, n in enumerate(MAX_SIZES)]
    P = Pair(eng, clean_env, ms)
    assert len(P.g) == GROUP_MAX
    f = make_feature_batch(range(7500, 7500 + P.n), 2 + 1 + 18 + 1 + 1 + 18)
    silent = P.synth(f[:, :2])
    assert not silent.any()
    ms_, _ = P.group.last_sample_kernel_ms()
    assert ms_ == 0.0, "an all-silent group call ran a per-sample launch (%.3f ms)" % ms_
    got = np.concatenate([silent, P.synth(f[:, 2:3]), P.synth(f[:, 3:21])], axis=1)
    for k, (m, g, x) in enumerate(zip(ms, P.split(got), P.split(f[:, :21]))):
        check(g, H.oracle_synth(x, "int8", tag=m.tag, model_blob=m.blob), "member %d (%r) vs the oracle" % (k, m))
    P.check_state()
    P.both(lambda k, b: b.reset() if k < 8 else None)
    P.synth(f[:, 21:22])
    P.check_state()
    P.check_tails()
    P.both(lambda k, b: b.reset() if k < GROUP_MAX - 1 else None)
    P.synth(f[:, 22:23])
    P.check_state()
    P.both(lambda k, b: b.reset_streams([0]) if k % 3 == 0 else None)
    P.synth(f[:, 23:])
    P.check_state()
    P.check_tails()
    P.close()


@gpu
@pytest.mark.parametrize("na", list(TAGS))
@pytest.mark.parametrize("spc", [5, 21])
def test_silent_member_between_live_ones(eng, clean_env, K, na, spc):
    """member 1 of 4 is reset right before a 2-frame call: silent for the whole call, it is left out of the launch while the
    members after it run at lower launch indices; then it comes back in a 1-frame and an 18-frame call"""
    names = ["default", "seed%d" % SEED[na]]
    ms = [Member(na, names[i % 2], n) for i, n in enumerate([spc + 2, 2 * spc + 1, 3, spc + ragged(spc)])]
    P = Pair(eng, clean_env, ms, spc=spc)
    entry = np.arange(P.n) % K
    f = pool_features(K)[entry]
    first = P.synth(f[:, :T1])
    P.both(lambda k, b: b.reset() if k == 1 else None)
    got = np.concatenate([first, P.synth(f[:, T1:T1 + 2]), P.synth(f[:, T1 + 2:T1 + 3])], axis=1)
    for k, (m, g, e) in enumerate(zip(ms, P.split(got), P.split(entry))):
        if k == 1:
            check(g[:, T1 * 160:], H.oracle_synth(pool_features(K)[e, T1:T1 + 3], "int8", tag=m.tag, model_blob=m.blob),
                  "the reset member vs the oracle")
        else:
            check_pool(g, pool_pcm(K, na, m.name)[:, :(T1 + 3) * 160], e, "member %d (%r) vs the oracle" % (k, m))
    P.check_state()
    P.synth(f[:, T1 + 3:])
    P.check_state()
    P.check_tails()
    P.close()


# ---- 6. stress models in groups at 256 and 128 units ----
STRESS = [(na, spc, hot) for na in (256, 128) for spc in (9, 25) for hot in (False, True)]


@gpu
@pytest.mark.parametrize("na,spc,hot", [pytest.param(*c, id="na%d-spc%02d-%s" % (c[0], c[1], "hot-cvtunit" if c[2] else "cvtfree"))
                                        for c in STRESS])
def test_stress_models(eng, clean_env, K, na, spc, hot):
    """"full" (256 only: fewer dual_fc rows in shared memory, a footprint unlike its neighbours'; the group launches with the
    largest), "skew", "limits", "warm" and, in the hot cases, "hot" (the whole group on the conversion unit) next to the
    default and a seeded member"""
    names = ["default", "seed%d" % SEED[na]] + (["full"] if na == 256 else []) + ["skew", "limits", "warm"] + (["hot"] if hot else [])
    sizes = [1, spc + ragged(spc), 2 * spc - 1, spc, 3, spc + 1, spc // 2 + 1, 2 * spc + 3]
    ms = [Member(na, name, sizes[i]) for i, name in enumerate(names)]
    if na == 256:
        foot = [int(image_layout(na, m.name)[5]) for m in ms]
        assert foot[2] == max(foot) and len(set(foot)) > 2, foot
    assert kernel_of(ms, spc)[1] == ("cvtunit" if hot else "cvtfree")
    P = Pair(eng, clean_env, ms, spc=spc)
    run_pool(P, K)
    P.close()


@gpu
@pytest.mark.parametrize("na", list(TAGS))
@pytest.mark.parametrize("spc", [9, 25])
def test_accumulators_beyond_the_conversion_free_range(eng, clean_env, K, na, spc):
    """a member whose accumulators leave the conversion-free rounding's range (beyond_blob) next to members that allow it: the
    whole group must run on the conversion unit, or that member's PCM and state differ from its own calls and the oracle"""
    assert image_layout(na, "beyond")[21] == 0 and image_layout(na, "default")[21] == 1
    ms = [Member(na, "default", spc + 1), Member(na, "beyond", 2 * spc + ragged(spc)), Member(na, "seed%d" % SEED[na], 3)]
    assert kernel_of(ms, spc)[1] == "cvtunit"
    P = Pair(eng, clean_env, ms, spc=spc)
    run_pool(P, K)
    P.close()


# ---- 7. call shapes ----
def shape_members(na=384):
    return [Member(na, "default", 5), Member(na, "seed%d" % SEED[na], 9), Member(na, "default", 2)]


@gpu
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("spf", [80, 320, 1])
def test_samples_per_frame(eng, clean_env, K, spf, path):
    """group synthesis at `spf` samples per feature vector (3 then 18 frames), host buffers or `_device` ones at non-zero
    offsets; the oracle synthesizes `spf` samples per vector too"""
    P = Pair(eng, clean_env, shape_members())
    f = pool_features(K)[np.arange(P.n) % K]
    got = np.concatenate([P.synth(f[:, :T1], spf, path == "device"), P.synth(f[:, T1:], spf, path == "device")], axis=1)
    for k, (m, g, x) in enumerate(zip(P.members, P.split(got), P.split(f))):
        check(g, oracle_spf(x, m.na, m.name, spf), "member %d (%r) vs the oracle, spf %d" % (k, m, spf))
    P.check_state()
    P.check_tails()
    P.close()


@gpu
@pytest.mark.parametrize("path", ["host", "device"])
def test_feature_stride_36(eng, clean_env, K, path):
    """features of 36 floats per frame whose last 16 are NaN (host, or `_device` at non-zero offsets); the members' own calls
    take the same 36-float rows"""
    P = Pair(eng, clean_env, shape_members())
    f = pool_features(K)[np.arange(P.n) % K]
    f36 = np.full(f.shape[:2] + (36,), np.nan, np.float32)
    f36[:, :, :20] = f
    got = np.concatenate([P.synth(f36[:, :T1], device=path == "device"), P.synth(f36[:, T1:], device=path == "device")], axis=1)
    for k, (m, g, e) in enumerate(zip(P.members, P.split(got), P.split(np.arange(P.n) % K))):
        check_pool(g, pool_pcm(K, m.na, m.name), e, "member %d (%r) vs the oracle" % (k, m))
    P.check_state()
    P.check_tails()
    P.close()


@gpu
@pytest.mark.parametrize("path", ["host", "device"])
@pytest.mark.parametrize("na", [384, 128])
def test_decode_across_a_chunk(eng, clean_env, na, path):
    """group decode of 5 packets (20 frames: across the 16-frame chunk) with per-member codebooks, then synthesis, then 5 more
    packets; host buffers or `_device` ones at non-zero offsets"""
    import gen_model
    other = np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=78)]).astype(np.float32)
    ms = [Member(na, "default", 5), Member(na, "seed%d" % SEED[na], 6, codebooks=other), Member(na, "default", 3)]
    P = Pair(eng, clean_env, ms)
    pk = np.stack([make_packets(7700 + s, 10) for s in range(P.n)])
    got = P.decode(pk[:, :5], path == "device")
    for k in (0, 2):      # default codebooks: the oracle decodes them
        check(P.split(got)[k], H.oracle_decode(P.split(pk)[k][:, :5], "int8", tag=TAGS[na]), "member %d decode vs the oracle" % k)
    P.synth(make_feature_batch(range(7800, 7800 + P.n), 3), device=path == "device")
    P.check_tails()
    P.decode(pk[:, 5:], path == "device")
    P.check_state()
    P.check_tails()
    P.close()
