"""Deterministic edge-case inputs (TEST INFRASTRUCTURE) for the analysis side and the conditioning network.

fixtures.make_pcm always adds noise and make_features stays in speech-like ranges; the inputs here are the ones that reach the
corners where an x86 build and a CUDA build can part ways (NaN and out-of-range float->int conversions, exact ties, signed
zeros, denormals, reciprocals that flush to zero).  Every case is a pure function of its name.  What each case is meant to
reach is checked from the reference's or the oracle's output by tests/test_edge_inputs.py (EDGE_CHECKS there).

  pcm_cases()        {name: int16 [NPK*640]}   lpcnet_encode / lpcnet_compute_features / single-frame analysis
  float_pcm_cases()  {name: float32 [NPK*640]} lpcnet_compute_single_frame_features_float only
  feature_cases()    {name: float32 [NFR][20]} the conditioning network (run_frame_network) and synthesis
"""
import numpy as np
from fixtures import make_pcm, make_features

NPK = 6                      # packets per PCM case (24 frames: two superframes of lead-in, the edge, room after it)
NS = NPK * 640
NFR = 24                     # frames per feature case
PITCH_MIN, PITCH_MAX = 32, 256
NAN_SLOPE_PACKET = 2         # the impulse pairs sit in the third superframe
FULL = 32767


def _speech(seed):
    return make_pcm(seed, NS // 160).astype(np.int64)


def _square(period):
    n = np.arange(NS)
    return np.where((n % period) < (period + 1) // 2, FULL, -FULL - 1)


def _train(period):
    x = np.zeros(NS, np.int64)
    x[::period] = FULL
    return x


def impulses(half, pair=True):
    """Silence with a 20000 impulse at the start of half-subframe `half` (2..9, the xc rows of process_superframe) of superframe
    NAN_SLOPE_PACKET, and with `pair` a second one 40 samples later.  The analysis delays the signal by TRAINING_OFFSET = 80
    samples, so only one half-subframe of the superframe holds excitation energy: the pitch slope is 0/0.  The pair is periodic
    enough to be voiced (the slope's NaN reaches the modulation field); the single impulse is its unvoiced twin."""
    x = np.zeros(NS, np.int64)
    s = NAN_SLOPE_PACKET * 640 + 80 * (half - 2)
    x[s] = 20000
    if pair:
        x[s + 40] = 20000
    return x


def pcm_cases():
    c = {}
    c["silence"] = np.zeros(NS, np.int64)
    g = _speech(4000)                         # digital silence between speech: from a frame boundary (frame 5), a superframe
    g[5 * 160:9 * 160] = 0                    # boundary (frame 12 = packet 3) and mid-frame (sample 37 of frame 19)
    g[12 * 160:17 * 160] = 0
    g[19 * 160 + 37:22 * 160] = 0
    c["silence_gaps"] = g
    for h in range(2, 10):
        c["pair_h%d" % h] = impulses(h)
    for h in (2, 9):
        c["single_h%d" % h] = impulses(h, pair=False)
    c["dc_max"] = np.full(NS, FULL)
    c["dc_min"] = np.full(NS, -FULL - 1)
    for p in (PITCH_MIN - 1, PITCH_MIN, PITCH_MAX, PITCH_MAX + 1):
        c["square_%d" % p] = _square(p)
        c["train_%d" % p] = _train(p)
    c["nyquist"] = np.where(np.arange(NS) % 2 == 0, FULL, -FULL - 1)
    c["clipped"] = np.clip(_speech(4001) * 8, -FULL - 1, FULL)
    rng = np.random.default_rng(4002)
    c["white_full"] = rng.integers(-FULL - 1, FULL + 1, NS)
    c["lsb"] = rng.integers(-1, 2, NS)
    c["periodic_80"] = np.tile(rng.integers(-8000, 8001, 80), NS // 80)      # 80 divides 160: every frame is the same frame
    return {k: v.astype(np.int16) for k, v in c.items()}


def float_pcm_cases():
    """Inputs only the float entry point can take: fractions, 4x full scale, amplitudes whose windowed values (x * w / 320) are
    denormal, and negative zeros."""
    sp = _speech(4010).astype(np.float64)
    rng = np.random.default_rng(4011)
    c = {}
    c["fractional"] = sp + rng.uniform(-0.5, 0.5, NS)
    c["x4_full"] = sp / np.abs(sp).max() * 4 * 32768
    tiny = sp / np.abs(sp).max()
    c["tiny"] = np.concatenate([tiny[:NS // 3] * 1e-30, tiny[NS // 3:2 * NS // 3] * 1e-36, tiny[2 * NS // 3:] * 1e-41])
    c["neg_zero"] = np.full(NS, -0.0)
    return {k: v.astype(np.float32) for k, v in c.items()}


def pitch_boundary(k):
    """(below, at, above): the float32 values around the smallest f with (int)floor(.1 + 50*f + 100) == k (50*f a float product,
    the sums in double, lpcnet.c:93)."""
    idx = lambda f: int(np.floor(.1 + float(np.float32(50) * np.float32(f)) + 100))
    f = np.float32((k - 100.1) / 50)
    while idx(f) >= k:
        f = np.nextafter(f, np.float32(-np.inf))
    while idx(f) < k:
        f = np.nextafter(f, np.float32(np.inf))
    return np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))


PITCH_FLOOR_K = (33, 34, 150, 254, 255)
PITCH_RANGE = (1e3, -1e3, 4.3e7, 1e9, np.inf, -np.inf)
RAMP = np.geomspace(1.0, 1e11, NFR)


def feature_cases():
    c = {}
    v = [x for k in PITCH_FLOOR_K for x in pitch_boundary(k)]
    f = make_features(5000, NFR)
    f[:, 18] = np.resize(np.array(v, np.float32), NFR)
    c["pitch_floor"] = f
    f = make_features(5001, NFR)                                        # the infinities last: as a feature input they make the
    f[:, 18] = np.resize(np.array(PITCH_RANGE[:4], np.float32), NFR)    # conditioning NaN from there on
    f[-4:, 18] = np.resize(np.array(PITCH_RANGE[4:], np.float32), 4)
    c["pitch_range"] = f
    f = make_features(5002, NFR)
    f[:, 0] = np.linspace(-40, 40, NFR)
    f[:, 1:18] *= 8
    c["ceps_wide"] = f
    f = make_features(5003, NFR)
    f[:, 19] = np.where(np.arange(NFR) % 2 == 0, 5.0, -5.0)
    c["corr_5"] = f
    f = make_features(5004, NFR)
    f[:, :18] = np.sign(f[:, :18] + 1e-3) * RAMP[:, None]                 # magnitudes 1 .. 1e11 over the frames
    c["ramp"] = f
    return {k: np.ascontiguousarray(v, np.float32) for k, v in c.items()}


def conv1_preactivations(features):
    """float64 estimate of the first conditioning layer's pre-activations [NFR][128] for one feature case on a fresh state (conv
    window = the two previous frames and this one, zeros before the first; lpcnet.c:93-98, nnet.c:452-470).  Only used to show
    where a case puts them, not to check the engine."""
    import gen_model
    common = {n: a for n, _, a in gen_model.make_model()[0]}
    w = np.asarray(common["feature_conv1_weights"], np.float64).reshape(3, -1, 128)
    b = np.asarray(common["feature_conv1_bias"], np.float64)
    emb = np.asarray(common["embed_pitch_weights"], np.float64).reshape(256, -1)
    f = np.asarray(features, np.float64)
    pitch = np.clip(np.floor(.1 + 50 * f[:, 18] + 100), 33, 255).astype(int)
    rows = np.concatenate([np.zeros((2, w.shape[1])), np.concatenate([f[:, :20], emb[pitch]], axis=1)])
    return np.stack([b + sum(rows[t + k] @ w[k] for k in range(3)) for t in range(len(f))])
