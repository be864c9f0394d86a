"""GPU tests (-m gpu) of the edge-case inputs of oracle/edge_inputs.py: the encoder (all three modes, batched and in uneven
chunks, int16 and float input, the single-stream drop-in API), the conditioning network's taps, synthesis and decode, bit for
bit against the CPU restatement (pinned to the reference by tests/test_edge_inputs.py) and against the reference's digests.
NaN taps are compared by position only (x86 and CUDA NaN payloads differ)."""
import ctypes
import json
import os
import numpy as np
import pytest
import edge_inputs as E
import helpers as H
from fixtures import make_pcm_batch
from test_edge_inputs import (PCM, PCM_NAMES, FPCM_NAMES, FEAT_NAMES, FINITE_FEAT, pcm_batch, fpcm_batch, feat_batch,
                              modulation_field, nan_bits, assert_same, digest_nan)

pytestmark = pytest.mark.gpu
N_SPEECH = 37 - len(PCM_NAMES)          # make_pcm streams mixed in: a 37-stream ragged batch


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


def mixed():
    """[37][NS] int16: the edge streams interleaved with make_pcm streams; returns (pcm, rows of the edge streams in order)."""
    sp = make_pcm_batch(range(600, 600 + N_SPEECH), E.NS // 160)
    edge = pcm_batch()
    out, rows, i, j = [], [], 0, 0
    for k in range(37):
        if k % 4 == 3 and j < N_SPEECH:
            out.append(sp[j]); j += 1
        elif i < len(edge):
            rows.append(len(out)); out.append(edge[i]); i += 1
        else:
            out.append(sp[j]); j += 1
    return np.stack(out), rows


def name_of(rows, s):
    return PCM_NAMES[rows.index(s)] if s in rows else "make_pcm stream %d" % s


def assert_same_packets(got, want, rows):
    d = np.argwhere(got != want)
    if d.size:
        s, p, b = (int(v) for v in d[0])
        raise AssertionError("%d packet bytes differ, first: stream %d (%s) packet %d byte %d: got %d want %d; modulation field "
                             "got %d want %d" % (len(d), s, name_of(rows, s), p, b, got[s, p, b], want[s, p, b],
                                                 modulation_field(got[s, p]), modulation_field(want[s, p])))


def test_edge_streams_in_a_ragged_batch_all_modes(eng):
    pcm, rows = mixed()
    e = eng.EncBatch(37, codebooks=H.codebooks())
    f = e.compute_features(pcm)
    e.reset()
    pk = e.encode(pcm)
    e.reset()
    f4 = e.compute_features4(pcm)
    e.close()
    assert_same_packets(pk, H.oracle_encode(pcm), rows)
    assert_same(f, H.oracle_features(pcm), "features vs oracle")
    assert_same(f4, H.oracle_encode(pcm, features4=True), "features4 vs oracle")
    edge = pcm_batch()
    assert H.digest(pk[rows]) == H.ref_digest("edge_encode", lambda: H.ref_encode(edge))
    assert H.digest(f[rows]) == H.ref_digest("edge_features_int16", lambda: H.ref_features(edge))
    assert H.digest(f4[rows]) == H.ref_digest("edge_features4", lambda: H.ref_features4(edge))


def test_nan_slope_packets(eng):
    """The voiced superframes whose pitch slope is 0/0: modulation field 1 (x86's INT_MIN clamped to -3), as the reference."""
    edge = pcm_batch()
    e = eng.EncBatch(len(edge), codebooks=H.codebooks())
    pk = e.encode(edge)
    e.close()
    for h in range(2, 10):
        s = PCM_NAMES.index("pair_h%d" % h)
        p = E.NAN_SLOPE_PACKET + (h == 9)
        assert modulation_field(pk[s, p]) == 1, "stream %d (pair_h%d) packet %d: modulation field %d, want 1" % (s, h, p, modulation_field(pk[s, p]))
    assert_same_packets(pk, H.oracle_encode(edge), list(range(len(edge))))


def test_edge_streams_in_uneven_chunks(eng):
    pcm, rows = mixed()
    e = eng.EncBatch(37, codebooks=H.codebooks())
    parts, t = [], 0
    for k in (1, 3, 7, 13):
        parts.append(e.compute_features(pcm[:, t * 160:(t + k) * 160])); t += k
    assert t == E.NS // 160
    f = np.concatenate(parts, axis=1)
    e.reset()
    parts, p = [], 0
    for k in (1, 3, 2):
        parts.append(e.encode(pcm[:, p * 640:(p + k) * 640])); p += k
    assert p == E.NPK
    pk = np.concatenate(parts, axis=1)
    e.close()
    assert_same(f, H.oracle_features(pcm), "chunked features")
    assert_same_packets(pk, H.oracle_encode(pcm), rows)


def test_float_entry_point_on_edge_signals(eng):
    x = fpcm_batch()
    e = eng.EncBatch(len(x))
    f = e.compute_features(x)
    e.close()
    assert_same(f, H.oracle_features(x), "float features vs oracle")
    assert H.digest(f) == H.ref_digest("edge_features_float", lambda: H.ref_features(x))


def test_drop_in_encoder_on_the_nan_slope_case(eng):
    L = eng.lib()
    L.lpcnet_encoder_create.restype = ctypes.c_void_p
    L.lpcnet_encoder_destroy.argtypes = [ctypes.c_void_p]
    L.lpcnet_encode.argtypes = [ctypes.c_void_p] * 3
    cb = H.codebooks()
    assert L.lpcnet_b200_set_default_codebooks(cb.ctypes.data, cb.size) == 0
    pcm = np.ascontiguousarray(PCM["pair_h2"])
    want = H.oracle_encode(pcm[None])[0]
    st = L.lpcnet_encoder_create()
    assert st
    buf = np.zeros(8, np.uint8)
    for p in range(E.NPK):
        assert L.lpcnet_encode(st, pcm[p * 640:].ctypes.data, buf.ctypes.data) == 0
        np.testing.assert_array_equal(buf, want[p], err_msg="packet %d" % p)
    L.lpcnet_encoder_destroy(st)
    assert modulation_field(want[E.NAN_SLOPE_PACKET]) == 1


@pytest.mark.parametrize("stride", [20, 36])
def test_frame_network_taps_on_edge_features(eng, stride):
    """Pitch rows at the floor boundaries and past int32 (x86: INT_MIN, clamped to 33), cepstra far out of range, pre-activations
    through the inf numerator and the flushed reciprocal (NaN from there on, at the reference's positions)."""
    f20 = feat_batch()
    f = np.zeros(f20.shape[:2] + (stride,), np.float32)
    f[..., :20] = f20
    b = eng.Batch(len(f20), H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    half = E.NFR // 2                                  # two calls (the hook takes one chunk): the conv state carries across
    taps = [np.concatenate(p, axis=1) for p in zip(b.debug_frame_network(f[:, :half]), b.debug_frame_network(f[:, half:]))]
    b.close()
    want = H.oracle_frame_taps(f20)
    for t, (g, w) in enumerate(zip(taps, want)):
        for s, k in enumerate(FEAT_NAMES):
            assert_same(g[s], w[s], "%s tap %d" % (k, t))
        assert digest_nan(g) == H.ref_digest("edge_frame_taps_%d" % t, lambda: nan_bits(H.ref_frame_taps(f20)[t]))


@pytest.mark.parametrize("kind,build", [("int8", "A"), ("float", "B")])
def test_synthesis_on_edge_features(eng, kind, build):
    f = feat_batch(FINITE_FEAT)
    b = eng.Batch(len(f), H.blob(kind), lpc_gamma=H.LPC_GAMMA)
    got = b.synthesize(f)
    b.close()
    np.testing.assert_array_equal(got, H.oracle_synth(f, kind))
    assert H.digest(got) == H.ref_digest("edge_synth_%s" % build, lambda: H.ref_synth(f, build))


def test_decode_of_edge_packets(eng):
    pk = H.oracle_encode(pcm_batch())
    b = eng.Batch(len(pk), H.blob("int8"), lpc_gamma=H.LPC_GAMMA, codebooks=H.codebooks())
    got = b.decode(pk)
    b.close()
    np.testing.assert_array_equal(got, H.oracle_decode(pk, "int8"))


def test_full_range_rcpps_and_tanh_match_the_reference(eng):
    """The conditioning network's reciprocal (devmath.cuh rcp_emul_x86) against _mm256_rcp_ps captured on an Intel CPU
    (tests/golden/rcpps_edges.json): biased exponents 1, 2, 126, 127 and 250..254, zeros, denormals, infinities, NaNs, both signs.
    And its tanh against the oracle's over the whole range, through the inf numerator (|x| ~ 5e7) and the flushed reciprocal
    (|x| ~ 1.6e9), at the infinities and at NaN."""
    g = json.load(open(os.path.join(H.GOLDEN, "rcpps_edges.json")))
    x = np.array([int(v, 16) for v in g["x"]], np.uint32).view(np.float32)
    want = np.array([int(v, 16) for v in g["rcp"]], np.uint32)
    b = eng.Batch(1, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    rcp, _ = b.debug_tanh_x86(x)
    np.testing.assert_array_equal(rcp.view(np.uint32), want)
    mag = np.geomspace(1e-3, 3e38, 4000).astype(np.float32)
    xs = np.concatenate([mag, -mag, np.float32([0, -0.0, np.inf, -np.inf, np.nan, 5e7, 1.6e9, 1.7e9])]).astype(np.float32)
    _, th = b.debug_tanh_x86(xs)
    b.close()
    L = H.oracle_lib()
    m = H.oracle_model()
    wt = np.array([L.oracle_tanh(m, float(v)) for v in xs], np.float32)
    assert np.isnan(wt).any() and (np.abs(wt[np.isfinite(wt)]) == 1).any()
    assert_same(th, wt, "tanh8_approx")
