"""GPU tests (-m gpu) of launch geometry: the per-sample kernels at every streams-per-CTA value (spc), at the batch sizes where the
automatic schedule switches kernel or schedule, past one wave of CTAs, and the one-device multi API at the width of a 32768-stream
job.  The launcher (batch_api.cu group_plan / launch_sample) turns n streams into spc = ceil(n / SMs), clamped to 1..32,
and picks from it:
  * int8: one half (spc <= 16) or two halves (17..32; half A takes ceil(spc / 2) slots);
  * float: the neuron-per-lane kernel (spc <= 4: its 1-, 2- or 4-slot instance) or the lane==stream kernel (5..32);
and a batch of more than 32 x SMs streams runs in several waves.  Every geometry must give the same PCM, bit for bit, as the CPU
restatement.

Input pool: a stream's output depends only on its own inputs (every stream starts from the same fresh state and RNG seed), so
stream s of any batch takes entry s mod K of a pool of K feature (and packet) sequences, and the oracle runs on the pool only.
K is a prime chosen so that two streams whose indices differ by at most 64 (a neighbouring slot, the other half, the next CTA)
or by a whole number of waves get different inputs: a stream that reads another one's slot cannot pass by luck."""
import functools
import os
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

T1, T2, T3 = 3, 18, 6           # calls of 3 + 18 frames (state carried across calls, the second crosses the 16-frame chunk), then 6 more
T = T1 + T2
SPC_MAX, HALF, FN_S = 32, 16, 4  # engine.h STREAMS_PER_CTA, HALF, FN_S
N_BIG = 32768                    # INTEGRATION.md §3: a 32768-stream job on one device
KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "FLOAT_LANE_STREAM", "EXACT_CVT", "FCW_NODES")
TAGS = {"": 384, "na256": 256, "na128": 128}


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


@pytest.fixture
def auto(monkeypatch):
    """no create-time knob: the schedule is the one the launcher picks"""
    for k in KNOBS:
        monkeypatch.delenv("LPCNET_B200_" + k, raising=False)
    return monkeypatch


# ---- the input pool ----
def _is_prime(k):
    return k > 1 and all(k % d for d in range(2, int(k ** 0.5) + 1))


def pool_size(sms, n_max):
    """the smallest prime K >= 67 for which stream s -> pool entry s mod K gives different inputs to any two streams < n_max
    whose indices differ by 1..2*32 or by a whole number of waves (32 x sms streams)"""
    k = 67
    while not (_is_prime(k) and pool_distinct(k, sms, n_max)):
        k += 1
    return k


def pool_distinct(k, sms, n_max):
    wave = SPC_MAX * sms
    return all(d % k for d in list(range(1, 2 * SPC_MAX + 1)) + list(range(wave, n_max, wave)))


@pytest.fixture(scope="module")
def K(sms):
    k = pool_size(sms, N_BIG)
    assert pool_distinct(k, sms, N_BIG) and k >= 2 * SPC_MAX + 1
    return k


@functools.lru_cache(None)
def pool_features(k):
    """[k][T + T3][20]: frames 0..T-1 of the geometry runs, then T3 frames of the lifecycle test"""
    return make_feature_batch(range(6000, 6000 + k), T + T3)


@functools.lru_cache(None)
def pool_packets(k):
    return np.stack([make_packets(6000 + s, 3) for s in range(k)])


@functools.lru_cache(None)
def pool_pcm(k, kind, tag=""):
    """the oracle's PCM of every pool entry over all T + T3 frames from a fresh state"""
    return H.oracle_synth(pool_features(k), kind, tag=tag)


@functools.lru_cache(None)
def pool_pcm_restarted(k):
    """int8: the oracle's PCM of the last T3 frames of every pool entry from a fresh state (a stream reset after frame T)"""
    return H.oracle_synth(pool_features(k)[:, T:], "int8")


@functools.lru_cache(None)
def pool_pcm_spf(k, spf):
    """int8: the oracle's PCM of frames 0..T-1 of every pool entry, one feature vector per `spf` samples"""
    L = H.oracle_lib()
    f = pool_features(k)
    out = np.zeros((k, T * spf), np.int16)

    def one(s):
        st = L.oracle_state_create(H.oracle_model())
        for t in range(T):
            L.oracle_synthesize(st, f[s, t].ctypes.data, out[s, t * spf:].ctypes.data, spf)
        L.oracle_state_destroy(st)
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:        # (ctypes releases the GIL)
        list(ex.map(one, range(k)))
    return out


@functools.lru_cache(None)
def pool_decoded(k):
    return H.oracle_decode(pool_packets(k), "int8")


def check_streams(got, want_pool, entry, what):
    """stream s of `got` must equal row entry[s] of `want_pool` (compared by per-stream digests); names the first (stream, sample)"""
    assert got.shape == (len(entry), want_pool.shape[1]), "%s: shape %s" % (what, got.shape)
    bad = np.flatnonzero(H.stream_digests(got) != H.stream_digests(want_pool)[entry])
    if bad.size:
        s = int(bad[0])
        t = int(np.flatnonzero(got[s] != want_pool[entry[s]])[0])
        raise AssertionError("%s: %d of %d streams differ, first (stream, sample) = (%d, %d)" % (what, bad.size, len(entry), s, t))


def synth_pool(b, k, kind, tag, what):
    """n streams of the pool in calls of T1 + T2 frames, checked against the oracle"""
    entry = np.arange(b.n) % k
    f = pool_features(k)[entry]
    got = np.concatenate([b.synthesize(f[:, :T1]), b.synthesize(f[:, T1:T])], axis=1)
    check_streams(got, pool_pcm(k, kind, tag)[:, :T * 160], entry, what)
    return got


def kernel_of(kind, spc):
    """the kernel and schedule launch_sample picks for `spc` streams per CTA without knobs"""
    if kind == "int8":
        return "onehalf" if spc <= HALF else "twohalves"
    return "neuron%d" % (1 if spc <= 1 else 2 if spc == 2 else FN_S) if spc <= FN_S else "lanestream"


# ---- 1. every spc, pinned ----
def ragged(spc):
    """streams past two full CTAs: a ragged last CTA wherever spc > 1; for the two-half schedule r > ceil(spc / 2), so that half B
    of the last CTA is live but ends early, with both odd and even r across 17..32"""
    return max(1, 2 * spc // 3)


PINNED = [pytest.param(kind, tag, spc, id="%s-na%d-spc%02d-%s-n%d" % (kind, na, spc, kernel_of(kind, spc), 2 * spc + ragged(spc)))
          for kind in ("int8", "float") for tag, na in TAGS.items() for spc in range(1, SPC_MAX + 1)]


@pytest.mark.parametrize("kind,tag,spc", PINNED)
def test_every_streams_per_cta(eng, auto, K, kind, tag, spc):
    """n = 2 spc + r streams at spc streams per CTA (LPCNET_B200_STREAMS_PER_CTA, no other knob): two full CTAs and a ragged one"""
    auto.setenv("LPCNET_B200_STREAMS_PER_CTA", str(spc))
    b = eng.Batch(2 * spc + ragged(spc), H.blob(kind, tag), config=H.model_config(tag))
    synth_pool(b, K, kind, tag, "%s %s spc=%d" % (kind, tag or "na384", spc))
    b.close()


# pinned spc with more CTAs than SMs: the CTAs of the second wave start after some of the first have finished
PINNED_WAVES = [("int8", 5), ("int8", 17), ("int8", 31), ("float", 3), ("float", 5), ("float", 31)]


@pytest.mark.parametrize("kind,spc", PINNED_WAVES, ids=["%s-spc%02d-%s" % (k, s, kernel_of(k, s)) for k, s in PINNED_WAVES])
def test_pinned_streams_per_cta_past_one_wave(eng, auto, sms, K, kind, spc):
    """spc x (SMs + 3) + r streams at a pinned spc: three CTAs more than the device has SMs, the last one ragged"""
    auto.setenv("LPCNET_B200_STREAMS_PER_CTA", str(spc))
    n = spc * (sms + 3) + ragged(spc)
    b = eng.Batch(n, H.blob(kind), lpc_gamma=H.LPC_GAMMA)
    synth_pool(b, K, kind, "", "%s spc=%d n=%d" % (kind, spc, n))
    b.close()


# ---- 2. the automatic schedule's switch points ----
SWITCH = [(m, p) for m in (1, 2, 4, 16, 32) for p in (0, 1)]    # n = m x SMs + p


def _switch_id(kind, m, p):
    spc = min(SPC_MAX, m + (p > 0))
    waves = "-2waves" if m == SPC_MAX and p else ""
    return "%s-n%dS%s-spc%02d-%s%s" % (kind, m, "+1" if p else "", spc, kernel_of(kind, spc), waves)


@pytest.mark.parametrize("kind,m,p", [pytest.param(k, m, p, id=_switch_id(k, m, p)) for k in ("int8", "float") for m, p in SWITCH])
def test_automatic_schedule_switch_points(eng, auto, sms, K, kind, m, p):
    """n = m x SMs (+ 1) streams without knobs: 1 -> 2 slots per CTA, the neuron-per-lane -> lane==stream switch at 4 x SMs, one half ->
    two halves at 16 x SMs, and 32 x SMs + 1, whose last stream runs in a second wave"""
    n = m * sms + p
    b = eng.Batch(n, H.blob(kind), lpc_gamma=H.LPC_GAMMA)
    synth_pool(b, K, kind, "", "%s n=%d" % (kind, n))
    b.close()


# ---- 3. past one wave ----
@pytest.mark.parametrize("kind", ["int8", "float"])
@pytest.mark.parametrize("size", ["2waves+17", "32768"])
def test_synthesis_past_one_wave(eng, auto, sms, K, kind, size):
    """2 x 32 x SMs + 17 streams (three waves, the last one a single ragged CTA) and 32768 (8 waves on 132 SMs)"""
    n = 2 * SPC_MAX * sms + 17 if size == "2waves+17" else N_BIG
    b = eng.Batch(n, H.blob(kind), lpc_gamma=H.LPC_GAMMA)
    synth_pool(b, K, kind, "", "%s n=%d" % (kind, n))
    b.close()


def test_decode_past_one_wave(eng, auto, K):
    """lpcnet_decode of 3 packets (12 frames) on 32768 streams"""
    entry = np.arange(N_BIG) % K
    b = eng.Batch(N_BIG, H.blob("int8"), lpc_gamma=H.LPC_GAMMA, codebooks=H.codebooks())
    got = b.decode(pool_packets(K)[entry])
    b.close()
    check_streams(got, pool_decoded(K), entry, "decode n=%d" % N_BIG)


def test_lifecycle_across_waves(eng, auto, sms, K):
    """32768 int8 streams after T1 + T2 frames: reset_streams on streams of the first CTA, on both sides of a wave boundary and in
    the last CTA, then T3 frames (the mixed-silence path over all streams: a reset stream is silent for FEATURES_DELAY frames while
    the others go on); the exported state of a stream in the last CTA continues identically in a small fresh batch; a snapshot
    taken after the resets and restored after the call repeats it."""
    n, wave = N_BIG, SPC_MAX * sms
    entry = np.arange(n) % K
    f = pool_features(K)[entry]
    cont, fresh = pool_pcm(K, "int8")[:, T * 160:], pool_pcm_restarted(K)
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    synth_pool(b, K, "int8", "", "int8 n=%d" % n)
    reset = np.array([0, 7, wave - 1, wave, n - 1])
    moved = n - 3                                                   # in the last CTA, not reset
    state = b.export_state(moved)
    b.reset_streams(reset)
    snap = b.snapshot()
    third = b.synthesize(f[:, T:])
    want = cont[entry]
    want[reset] = fresh[entry[reset]]
    check_streams(third, want, np.arange(n), "after reset_streams")
    b.restore(snap)
    b.free_snapshot(snap)
    again = b.synthesize(f[:, T:])
    b.close()
    check_streams(again, third, np.arange(n), "repeat after snapshot restore")
    small = [1, moved, 2]
    c = eng.Batch(3, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    c.import_state(1, state)
    got = c.synthesize(f[small, T:])
    c.close()
    check_streams(got, np.stack([fresh[entry[1]], cont[entry[moved]], fresh[entry[2]]]), np.arange(3), "imported state")


# ---- 4. the multi API on one device at the width of the 32768-stream job ----
@pytest.mark.parametrize("spf", [80, 320])
def test_multi_one_device_full_width(eng, auto, K, spf):
    """Multi(32768, blob, [0]): a 36-float feature stride whose padding is NaN; the gather path at `spf` samples per feature vector
    over T frames (the second chunk lands at 16 x spf through the PCM sink); decode with and without the gather; reset() returns
    to the first call's output."""
    n = N_BIG
    entry = np.arange(n) % K
    f = pool_features(K)[entry, :T]
    f36 = np.full((n, T, 36), np.nan, np.float32)
    f36[:, :, :20] = f
    want = pool_pcm(K, "int8")[:, :T * 160]
    m = eng.Multi(n, H.blob("int8"), [0], config=(H.LPC_GAMMA, -1, -1), codebooks=H.codebooks())
    assert m.shard(0) == (0, 0, n)
    first = m.synthesize(f36)
    check_streams(first, want, entry, "multi synthesize, stride 36")
    m.reset()
    check_streams(m.synthesize(f, samples_per_frame=spf, gather=True), pool_pcm_spf(K, spf), entry, "multi gather, spf=%d" % spf)
    pk = pool_packets(K)[entry]
    m.reset()
    check_streams(m.decode(pk), pool_decoded(K), entry, "multi decode")
    m.reset()
    check_streams(m.decode(pk, gather=True), pool_decoded(K), entry, "multi decode, gather")
    m.reset()
    check_streams(m.synthesize(f36), first, np.arange(n), "multi synthesize after reset")
    m.close()


def test_pool_property(sms):
    """the pool really separates neighbours and waves on this device, and a pool that does not is detected"""
    k = pool_size(sms, N_BIG)
    entry = np.arange(N_BIG) % k
    for d in list(range(1, 2 * SPC_MAX + 1)) + list(range(SPC_MAX * sms, N_BIG, SPC_MAX * sms)):
        assert (entry[d:] != entry[:-d]).all(), d
    assert not pool_distinct(61, sms, N_BIG) and not pool_distinct(67, 67, N_BIG)
