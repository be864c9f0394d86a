"""CPU tests (-m "not gpu") of the edge-case inputs of oracle/edge_inputs.py: each case reaches the edge it is named for (shown
from the reference's or the oracle's output), and the CPU restatement equals the compiled reference on every case: features
(int16 and float input), packets, unquantised superframe features, frame-network taps and synthesis (builds A and B).  Where
the reference is not compiled, the digests it gave (tests/golden/ref_digests.json, edge_* keys) stand in for it.

Taps and features are compared as bit patterns except at NaN, where only the positions must agree: x86's default NaN is
0xFFC00000 and CUDA's 0x7FFFFFFF, and the engine does not promise the payload."""
import numpy as np
import pytest
import edge_inputs as E
import helpers as H

PCM = E.pcm_cases()
FPCM = E.float_pcm_cases()
FEAT = E.feature_cases()
PCM_NAMES, FPCM_NAMES, FEAT_NAMES = list(PCM), list(FPCM), list(FEAT)
# feature cases whose reference conditioning and LPC stay finite: the ones synthesis is compared on (after a NaN in the
# conditioning every conversion of the sample loop would need x86 NaN semantics, which the engine does not promise)
FINITE_FEAT = ["pitch_floor", "ceps_wide", "corr_5"]


def pcm_batch():
    return np.stack([PCM[k] for k in PCM_NAMES])


def fpcm_batch():
    return np.stack([FPCM[k] for k in FPCM_NAMES])


def feat_batch(names=None):
    return np.stack([FEAT[k] for k in (names or FEAT_NAMES)])


def modulation_field(packet):
    """The 3-bit field after c0 (7 bits) and the pitch index (6 bits): modulation + 4 when voiced, 0 when unvoiced."""
    return (int.from_bytes(bytes(packet), "big") >> 48) & 7


def nan_bits(a):
    """Bit patterns with every NaN replaced by one canonical pattern (positions kept, payload dropped)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    return np.where(np.isnan(a), np.uint32(0x7FC00000), a.view(np.uint32))


def assert_same(got, want, what):
    d = np.argwhere(nan_bits(got) != nan_bits(want))
    assert d.size == 0, "%s: %d values differ, first at %s: got %r want %r" % (what, len(d), tuple(d[0]), got[tuple(d[0])], want[tuple(d[0])])


def digest_nan(a):
    """Digest that is the same for any NaN payload (the reference's taps are stored with NaNs canonicalised)."""
    return H.digest(nan_bits(a))


# ---- each case reaches its edge ----
def test_nan_slope_cases_are_voiced_with_modulation_field_1():
    """Impulse pairs in one half-subframe of a superframe: the reference's pitch regression divides 0 by 0 (the oracle, which
    matches the reference's packets byte for byte, reports the NaN slope), the superframe is still voiced, and x86's
    (int)floor(NaN) = INT_MIN clamps to -3: the packet's modulation field is 1 (a CUDA conversion would give 0, field 4)."""
    pk = H.ref_encode(pcm_batch()) if H.have_ref("A") else H.oracle_encode(pcm_batch())
    for h in range(2, 10):
        i = PCM_NAMES.index("pair_h%d" % h)
        p = E.NAN_SLOPE_PACKET + (h == 9)                  # the 80-sample analysis delay moves position 9 into the next superframe
        _, slopes = H.oracle_encode_slopes(PCM["pair_h%d" % h])
        assert np.isnan(slopes[p]), h
        assert [modulation_field(x) for x in pk[i]] == [1 if k == p else 0 for k in range(E.NPK)], h
    for h in (2, 9):                                       # the unvoiced twin: the same NaN slope, unvoiced, field 0
        i = PCM_NAMES.index("single_h%d" % h)
        p = E.NAN_SLOPE_PACKET + (h == 9)
        assert np.isnan(H.oracle_encode_slopes(PCM["single_h%d" % h])[1][p])
        assert all(modulation_field(x) == 0 for x in pk[i])


def test_pcm_cases_reach_their_edges():
    pcm = pcm_batch()
    f = H.ref_features(pcm) if H.have_ref("A") else H.oracle_features(pcm)
    f4 = H.ref_features4(pcm) if H.have_ref("A") else H.oracle_encode(pcm, features4=True)
    row = lambda k: PCM_NAMES.index(k)
    sil = f[row("silence")]
    assert (sil[1:] == sil[1]).all()                                         # digital silence: one steady frame
    g = f[row("silence_gaps")]
    for t in (7, 15):                                                         # inside the gaps: the cepstrum of silence
        np.testing.assert_array_equal(g[t, :18], sil[t, :18])
    for k in ("dc_max", "dc_min", "periodic_80"):                            # frames repeat exactly: later features are ties
        assert (f4[row(k), 12:, :] == f4[row(k), 12, :]).all(), k
    for k in ("square_31", "train_31", "square_32", "train_32"):             # below / at PITCH_MIN_PERIOD
        assert (f[row(k), 8:, 18] < -0.7).all(), k                           # pitch feature near its lowest value (.01*(66-200) = -1.34 .. -0.7)
    for k in ("square_256", "train_256", "square_257", "train_257"):         # at / past PITCH_MAX_PERIOD: the search's top lag
        assert (f[row(k), 8:, 18] == np.float32(.01 * (510 - 200))).all(), k
    assert pcm[row("nyquist")].min() == -32768 and (pcm[row("dc_min")] == -32768).all()
    assert (np.abs(pcm[row("clipped")].astype(int)) >= 32767).sum() > 100
    assert np.abs(pcm[row("lsb")]).max() == 1 and np.abs(pcm[row("white_full")].astype(int)).max() > 32000


def test_float_pcm_cases_reach_their_edges():
    x = fpcm_batch()
    f = H.ref_features(x) if H.have_ref("A") else H.oracle_features(x)
    sil = (H.ref_features if H.have_ref("A") else H.oracle_features)(np.zeros((1, E.NS), np.int16))[0]
    row = lambda k: FPCM_NAMES.index(k)
    assert (x[row("fractional")] != np.rint(x[row("fractional")])).mean() > .99
    assert np.abs(x[row("x4_full")]).max() > 4 * 32767
    w = np.abs(x[row("tiny")]) * np.float32(1 / 320.)                          # windowed, scaled values (w <= 1)
    assert ((w > 0) & (w < np.finfo(np.float32).tiny)).sum() > 1000             # denormal
    assert (np.signbit(x[row("neg_zero")]) & (x[row("neg_zero")] == 0)).all()
    for k in ("tiny", "neg_zero"):                                              # too small to register: exactly silence
        np.testing.assert_array_equal(f[row(k)].view(np.uint32), sil.view(np.uint32), err_msg=k)


def test_feature_cases_reach_their_edges():
    L = H.oracle_lib()
    pi = lambda v: L.oracle_pitch_index(float(v))
    for k in E.PITCH_FLOOR_K:                      # the float just below the boundary takes the previous row (or the clamp)
        below, at, above = E.pitch_boundary(k)
        assert (pi(below), pi(at), pi(above)) == (max(33, k - 1), k, k), k
    assert [pi(v) for v in E.PITCH_RANGE] == [255, 33, 33, 33, 33, 33]      # past int32 and at +inf: INT_MIN, clamped to 33
    f = feat_batch()
    ga, gb, lpc = H.ref_frame_taps(f) if H.have_ref("A") else H.oracle_frame_taps(f)
    nanf = lambda k: np.isnan(ga[FEAT_NAMES.index(k)]).any(-1)
    for k in FINITE_FEAT:
        i = FEAT_NAMES.index(k)
        assert np.isfinite(ga[i]).all() and np.isfinite(gb[i]).all() and np.isfinite(lpc[i]).all(), k
    assert not nanf("pitch_range")[:-4].any() and nanf("pitch_range")[-4:].all()
    pre = np.abs(E.conv1_preactivations(FEAT["ramp"])).max(1)
    first_nan = int(np.argmax(nanf("ramp")))
    assert nanf("ramp")[first_nan:].all() and pre[first_nan] > 1.6e9            # the reciprocal of the denominator flushes to 0
    assert ((pre > 5e7) & ~nanf("ramp")).any()                                   # the numerator is inf, the result still +-1


# ---- the oracle equals the compiled reference on every case ----
def test_oracle_matches_reference_on_edge_features():
    pcm = pcm_batch()
    got = H.oracle_features(pcm)
    assert H.digest(got) == H.ref_digest("edge_features_int16", lambda: H.ref_features(pcm))


def test_oracle_matches_reference_on_edge_float_features():
    x = fpcm_batch()
    got = H.oracle_features(x)
    assert H.digest(got) == H.ref_digest("edge_features_float", lambda: H.ref_features(x))


def test_oracle_matches_reference_on_edge_packets():
    pcm = pcm_batch()
    got = H.oracle_encode(pcm)
    assert H.digest(got) == H.ref_digest("edge_encode", lambda: H.ref_encode(pcm))


def test_oracle_matches_reference_on_edge_features4():
    pcm = pcm_batch()
    got = H.oracle_encode(pcm, features4=True)
    assert H.digest(got) == H.ref_digest("edge_features4", lambda: H.ref_features4(pcm))


@pytest.mark.parametrize("tap", [0, 1, 2])
def test_oracle_matches_reference_on_edge_frame_network(tap):
    """gru_a / gru_b conditioning and weighted LPC of every feature case, NaN positions included."""
    f = feat_batch()
    got = H.oracle_frame_taps(f)[tap]
    if H.have_ref("A"):
        assert_same(got, H.ref_frame_taps(f)[tap], "tap %d" % tap)
    assert digest_nan(got) == H.ref_digest("edge_frame_taps_%d" % tap, lambda: nan_bits(H.ref_frame_taps(f)[tap]))


@pytest.mark.parametrize("build,kind", [("A", "int8"), ("B", "float")])
def test_oracle_matches_reference_on_edge_synthesis(build, kind):
    f = feat_batch(FINITE_FEAT)
    got = H.oracle_synth(f, kind)
    assert np.abs(got[:, 320:]).max() > 100
    assert H.digest(got) == H.ref_digest("edge_synth_%s" % build, lambda: H.ref_synth(f, build))


def test_rcpps_edges_fixture_matches_this_cpu():
    """tests/golden/rcpps_edges.json holds _mm256_rcp_ps captured on an Intel CPU over the edges of the float range.  Where the
    compiled reference runs on an Intel CPU, it must give the same; the oracle's emulation must give it everywhere."""
    import json, os
    g = json.load(open(os.path.join(H.GOLDEN, "rcpps_edges.json")))
    x = np.array([int(v, 16) for v in g["x"]], np.uint32).view(np.float32)
    want = np.array([int(v, 16) for v in g["rcp"]], np.uint32)
    L = H.oracle_lib()
    m = H.oracle_model()
    got = np.array([np.float32(L.oracle_rcp(m, float(v))).view(np.uint32) for v in x], np.uint32)
    np.testing.assert_array_equal(got, want)
    cpu = [l.split(":")[1].strip() for l in open("/proc/cpuinfo") if l.startswith("vendor_id")][:1]
    if H.have_ref("A") and cpu == ["GenuineIntel"]:
        R = H.ref_lib()
        if hasattr(R, "ref_rcp8"):                                   # the packed instruction itself
            out = np.zeros_like(x)
            R.ref_rcp8(x.ctypes.data, out.ctypes.data, x.size)
        else:                                                        # an older shim: the scalar RCPSS of the same unit
            out = np.array([R.ref_rcp(float(v)) for v in x], np.float32)
        np.testing.assert_array_equal(out.view(np.uint32), want)

