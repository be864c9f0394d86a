"""GPU parity tests (-m gpu): the CUDA engine, called through the C ABI (ctypes), against
  * the committed golden vectors produced by the untouched reference (tests/golden, make_golden.py), and
  * the CPU oracle restatement (oracle/lpcnet_oracle.c) on the same seeded inputs.
Bar: BIT-EXACT int16 PCM (integer GEMVs + op-for-op fp32 elementwise math), no tolerance anywhere.
"""
import hashlib
import json
import os
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


def _batch(eng, n):
    return eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA, codebooks=H.codebooks())


def _first_diff(a, b):
    d = np.argwhere(a != b)
    return None if d.size == 0 else tuple(d[0])


def test_frame_network_bit_exact(eng):
    """run_frame_network taps (gru_a/gru_b conditioning, weighted LPC) for 12 frames x 9 streams vs the oracle."""
    n, T = 9, 12
    f = make_feature_batch(range(20, 20 + n), T)
    b = _batch(eng, n)
    ga, gb, lpc = b.debug_frame_network(f)
    L = H.oracle_lib()
    for s in range(n):
        st = L.oracle_state_create(H.oracle_model())
        for t in range(T):
            a = np.zeros(1152, np.float32); c = np.zeros(48, np.float32); l = np.zeros(16, np.float32)
            L.oracle_frame_network(st, f[s, t].ctypes.data, a.ctypes.data, c.ctypes.data, l.ctypes.data)
            np.testing.assert_array_equal(ga[s, t].view(np.uint32), a.view(np.uint32), err_msg="gru_a_condition s=%d t=%d" % (s, t))
            np.testing.assert_array_equal(gb[s, t].view(np.uint32), c.view(np.uint32), err_msg="gru_b_condition s=%d t=%d" % (s, t))
            np.testing.assert_array_equal(lpc[s, t].view(np.uint32), l.view(np.uint32), err_msg="lpc s=%d t=%d" % (s, t))
        L.oracle_state_destroy(st)
    b.close()


def test_synthesis_matches_reference_golden(eng):
    gold = np.load(os.path.join(H.GOLDEN, "synth_A.npz"))["pcm"]
    b = _batch(eng, 4)
    got = b.synthesize(make_feature_batch(range(4), 40))
    assert (got[:, :320] == 0).all()
    assert _first_diff(got, gold) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, gold),)
    ms, launches = b.last_sample_kernel_ms()
    assert ms > 0 and launches >= 5
    b.close()


def test_conversion_unit_path_matches_golden_too(eng, monkeypatch):
    """The kernel rounds the GRU_A accumulators without F2I/I2F when the model's pre-activations are provably small
    (devmath.cuh acc_init_t); LPCNET_B200_EXACT_CVT forces the conversion-unit instantiation, which must agree."""
    gold = np.load(os.path.join(H.GOLDEN, "synth_A.npz"))["pcm"]
    monkeypatch.setenv("LPCNET_B200_EXACT_CVT", "1")
    b = _batch(eng, 4)
    got = b.synthesize(make_feature_batch(range(4), 40))
    b.close()
    assert _first_diff(got, gold) is None


@pytest.mark.parametrize("nodes", ["8", "32"])
def test_fewer_dual_fc_rows_in_shared_memory(eng, monkeypatch, nodes):
    """A model that needs the room keeps fewer dual_fc rows in shared memory (model.cu); the sampler then reads the other
    tree levels from global memory: same PCM."""
    gold = np.load(os.path.join(H.GOLDEN, "synth_A.npz"))["pcm"]
    monkeypatch.setenv("LPCNET_B200_FCW_NODES", nodes)
    b = _batch(eng, 4)
    got = b.synthesize(make_feature_batch(range(4), 40))
    b.close()
    assert _first_diff(got, gold) is None


def test_rcpps_table_matches_reference(eng):
    """The per-sample kernels' _mm256_rcp_ps emulation (devmath.cuh, rcp_emul: the 2048-entry table with the exponent negated
    separately) must equal the reference's RCPPS (tests/golden/rcpps_table.bin) for every one of the 2048 mantissa classes, at
    many exponents and for random low mantissa bits.  The exponents run up to 2^125: the loader keeps GRU_A pre-activations
    below 2^31 accumulator units (|x| < 2^17.1), so tanh/sigmoid denominators reach about 2^72, and up to 2^125 the reciprocal
    is still a normal number."""
    rng = np.random.default_rng(5)
    k = np.arange(2048, dtype=np.uint32)
    xs = []
    for e in list(range(100, 253)):                      # biased exponents 2^-27 .. 2^125
        for low in (0, 0xFFF, None, None):
            lo = rng.integers(0, 4096, 2048, dtype=np.uint32) if low is None else np.uint32(low)
            xs.append(((np.uint32(e) << 23) | (k << 12) | lo).astype(np.uint32))
    x = np.concatenate(xs).view(np.float32)
    b = _batch(eng, 1)
    tab = b.debug_rcp(x)
    b.close()
    ref = H.rcp_table().astype(np.uint32)                # T[k]: rcp(2^e * 1.m) bits = T[m >> 12] - (e << 23)
    u = x.view(np.uint32)
    want = (ref[(u >> 12) & 0x7FF] - ((u & np.uint32(0x7F800000)) - np.uint32(0x3F800000))).astype(np.uint32)
    np.testing.assert_array_equal(tab.view(np.uint32), want)


@pytest.mark.parametrize("spc,two", [("32", "0"), ("5", "1"), ("16", "0"), ("17", "0")])
def test_grid_shapes_do_not_change_results(eng, monkeypatch, spc, two):
    """The launcher spreads a batch over the SMs (live stream slots per CTA) and steps small batches with one half only;
    every shape must give the same PCM: full 32-slot CTAs + a ragged one, dead slots in both halves of the two-half
    schedule, the largest one-half CTA and the smallest two-half CTA."""
    n, T = 70, 7
    f = make_feature_batch(range(200, 200 + n), T)
    b = _batch(eng, n); want = b.synthesize(f); b.close()
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", spc)
    if two == "1":
        monkeypatch.setenv("LPCNET_B200_TWO_HALVES", "1")
    b = _batch(eng, n); got = b.synthesize(f); b.close()
    assert _first_diff(got, want) is None


def test_synthesis_matches_oracle_ragged_batch(eng):
    """70 streams (two full CTAs + a 6-lane tail), 36-float feature stride, distinct features per stream."""
    n, T = 70, 10
    f20 = make_feature_batch(range(300, 300 + n), T)
    f36 = np.zeros((n, T, 36), np.float32); f36[:, :, :20] = f20; f36[:, :, 20:] = 7.0    # padding must be ignored
    b = _batch(eng, n)
    got = b.synthesize(f36)
    want = H.oracle_synth(f20, "int8")
    assert _first_diff(got, want) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, want),)
    b.close()


def test_chunked_calls_equal_one_call_and_state_roundtrip(eng):
    """Streaming use: 3+1+20+17 frames in four calls (crossing the silent warm-up and the internal 16-frame chunk)
    must equal one 41-frame call; afterwards the device state equals the oracle's state."""
    n, T = 5, 41
    f = make_feature_batch(range(40, 40 + n), T)
    b1, b2 = _batch(eng, n), _batch(eng, n)
    one = b1.synthesize(f)
    parts, t0 = [], 0
    for k in (3, 1, 20, 17):
        parts.append(b2.synthesize(f[:, t0:t0 + k]))
        t0 += k
    np.testing.assert_array_equal(np.concatenate(parts, axis=1), one)
    np.testing.assert_array_equal(one, H.oracle_synth(f, "int8"))
    L = H.oracle_lib()
    st = L.oracle_state_create(H.oracle_model())
    pcm = np.zeros(160, np.int16)
    for t in range(T):
        L.oracle_synthesize(st, f[2, t].ctypes.data, pcm.ctypes.data, 160)
    ga = np.zeros(384, np.float32); gb = np.zeros(16, np.float32); ls = np.zeros(16, np.float32); misc = np.zeros(2, np.int32); rng = np.zeros(4, np.uint32)
    L.oracle_get_state(st, ga.ctypes.data, gb.ctypes.data, ls.ctypes.data, misc.ctypes.data, rng.ctypes.data)
    got = b2.get_state(2)
    np.testing.assert_array_equal(got["gru_a"].view(np.uint32), ga.view(np.uint32))
    np.testing.assert_array_equal(got["gru_b"].view(np.uint32), gb.view(np.uint32))
    np.testing.assert_array_equal(got["last_sig"].view(np.uint32), ls.view(np.uint32))
    assert got["last_exc"] == misc[0] and (got["rng"] == rng).all()
    # reset returns to the fresh-state trajectory
    b2.reset()
    np.testing.assert_array_equal(b2.synthesize(f[:, :6]), one[:, :6 * 160])
    b1.close(); b2.close(); L.oracle_state_destroy(st)


@pytest.mark.parametrize("N", [80, 1, 250])
def test_other_samples_per_call(eng, N):
    """N != 160 samples per call (the PLC uses 80; the reference loop takes any N): one feature vector per call."""
    n, T = 3, 9
    f = make_feature_batch(range(60, 60 + n), T)
    b = _batch(eng, n)
    got = b.synthesize(f, samples_per_frame=N)
    L = H.oracle_lib()
    for s in range(n):
        st = L.oracle_state_create(H.oracle_model())
        pcm = np.zeros(N, np.int16)
        for t in range(T):
            L.oracle_synthesize(st, f[s, t].ctypes.data, pcm.ctypes.data, N)
            np.testing.assert_array_equal(got[s, t * N:(t + 1) * N], pcm)
        L.oracle_state_destroy(st)
    b.close()


def test_decode_matches_reference_golden(eng):
    gold = np.load(os.path.join(H.GOLDEN, "decode_A.npz"))["pcm"]
    b = _batch(eng, 3)
    got = b.decode(np.stack([make_packets(s, 6) for s in range(3)]))
    assert _first_diff(got, gold) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, gold),)
    b.close()


def test_reference_digests(eng):
    """Longer runs pinned by sha256 of the reference's output (tests/golden/digests.json)."""
    dig = json.load(open(os.path.join(H.GOLDEN, "digests.json")))
    b = _batch(eng, 16)
    got = b.synthesize(make_feature_batch(range(16), 150))
    assert hashlib.sha256(got.tobytes()).hexdigest() == dig["synth_A_16x150"]
    b.close()
    b = _batch(eng, 8)
    got = b.decode(np.stack([make_packets(s, 25) for s in range(8)]))
    assert hashlib.sha256(got.tobytes()).hexdigest() == dig["decode_A_8x25"]
    b.close()


def test_drop_in_single_stream_api(eng):
    """include/lpcnet.h used exactly like src/lpcnet_demo.c:202-219 (-synthesis) and :176-188 (-decode)."""
    gold = np.load(os.path.join(H.GOLDEN, "synth_A.npz"))["pcm"]
    L = eng.lib()
    L.lpcnet_b200_set_default_model(H.blob("int8"), len(H.blob("int8")), H.LPC_GAMMA)
    cb = H.codebooks()
    L.lpcnet_b200_set_default_codebooks(cb.ctypes.data, cb.size)
    net = eng.LPCNet()
    f = make_feature_batch([1], 40)[0][:12]          # same generator call as the golden (features depend on the length)
    out = np.concatenate([net.synthesize(f[t]) for t in range(12)])
    np.testing.assert_array_equal(out, gold[1, :12 * 160])
    net.reset()
    out2 = np.concatenate([net.synthesize(f[t]) for t in range(4)])
    np.testing.assert_array_equal(out2, gold[1, :4 * 160])
    net.load_model(H.blob("int8"))                      # lpcnet_load_model on a live state (lpcnet.c:202)
    net.close()
    gdec = np.load(os.path.join(H.GOLDEN, "decode_A.npz"))["pcm"]
    dec = eng.LPCNetDecoder()
    pk = make_packets(2, 6)[:3]
    out = np.concatenate([dec.decode(pk[t]) for t in range(3)])
    np.testing.assert_array_equal(out, gdec[2, :3 * 640])
    dec.close()
    with pytest.raises(eng.LPCNetB200Error):
        eng.Batch(2, H.blob("int8")[:5000])              # malformed blob -> error, not a crash


@pytest.mark.parametrize("n", [1024, 4096])
def test_full_width_properties(eng, n):
    """BASELINE-sized batch (>=1024 streams): size-independent checks — (i) replicated inputs give replicated
    outputs in every CTA/lane position, (ii) a sample of streams equals the oracle, (iii) determinism across runs."""
    T = 6
    base = make_feature_batch(range(500, 508), T)
    f = base[np.arange(n) % 8]
    b = _batch(eng, n)
    got = b.synthesize(f)
    want = H.oracle_synth(base, "int8")
    for s in range(n):
        if not np.array_equal(got[s], want[s % 8]):
            raise AssertionError("stream %d differs from its replica source %d at sample %s" % (s, s % 8, np.argwhere(got[s] != want[s % 8])[0]))
    b.reset()
    np.testing.assert_array_equal(b.synthesize(f), got)
    b.close()


def test_untouched_reference_cli_links_and_runs(eng, tmp_path):
    """The reference's own src/lpcnet_demo.c, compiled against the reference's own include/lpcnet.h and linked with
    liblpcnet_b200.so (oracle/Makefile target `demo`, built where /root/reference exists), run exactly like the
    reference CLI: `lpcnet_demo -synthesis features.f32 out.pcm` and `-decode packets out.pcm`."""
    import subprocess
    exe = os.path.join(H.ORACLE, "_ref", "lpcnet_demo_b200")
    if not os.path.exists(exe):
        pytest.skip("drop-in CLI was not prebuilt (needs /root/reference at build time)")
    gold = np.load(os.path.join(H.GOLDEN, "synth_A.npz"))["pcm"]
    f36 = np.zeros((40, 36), np.float32)
    f36[:, :20] = make_feature_batch([0], 40)[0]
    (tmp_path / "feat.f32").write_bytes(f36.tobytes())
    os.symlink(os.path.join(H.gen_dir(), "model_int8.bin"), tmp_path / "weights_blob.bin")   # lpcnet_demo.c:160 loads this name
    env = dict(os.environ, LPCNET_B200_LPC_GAMMA=str(H.LPC_GAMMA), LPCNET_B200_MODEL=os.path.join(H.gen_dir(), "model_int8.bin"),
               LPCNET_B200_CODEBOOKS=os.path.join(H.gen_dir(), "codebooks.bin"))
    subprocess.run([exe, "-synthesis", "feat.f32", "out.pcm"], cwd=tmp_path, env=env, check=True, timeout=300)
    out = np.frombuffer((tmp_path / "out.pcm").read_bytes(), dtype=np.int16)
    np.testing.assert_array_equal(out, gold[0])
    gdec = np.load(os.path.join(H.GOLDEN, "decode_A.npz"))["pcm"]
    (tmp_path / "pk.bin").write_bytes(make_packets(1, 6).tobytes())
    subprocess.run([exe, "-decode", "pk.bin", "dec.pcm"], cwd=tmp_path, env=env, check=True, timeout=300)
    out = np.frombuffer((tmp_path / "dec.pcm").read_bytes(), dtype=np.int16)
    np.testing.assert_array_equal(out, gdec[1])


def test_decode_full_width_properties(eng):
    """BASELINE config 5 width (1024 streams, lpcnet_decode path): replicated packet streams must give replicated PCM
    in every CTA / lane position, equal to the oracle's decode of the 8 source streams."""
    n, P = 1024, 3
    base = np.stack([make_packets(700 + s, P) for s in range(8)])
    pk = base[np.arange(n) % 8]
    b = _batch(eng, n)
    got = b.decode(pk)
    want = H.oracle_decode(base, "int8")
    for s in range(n):
        if not np.array_equal(got[s], want[s % 8]):
            raise AssertionError("stream %d differs from its replica source %d at sample %s" % (s, s % 8, np.argwhere(got[s] != want[s % 8])[0]))
    b.close()


def test_device_pointer_api_matches_host_api(eng):
    """lpcnet_b200_batch_synthesize_device (inputs resident in HBM, the benchmark's `value` path) == host-pointer call."""
    import ctypes
    n, T = 40, 7
    f = make_feature_batch(range(900, 900 + n), T)
    L = eng.lib()
    b1, b2 = _batch(eng, n), _batch(eng, n)
    want = b1.synthesize(f)
    d_f = L.lpcnet_b200_device_alloc(f.nbytes); d_p = L.lpcnet_b200_device_alloc(want.nbytes)
    L.lpcnet_b200_memcpy_h2d(d_f, f.ctypes.data, f.nbytes)
    b2.synthesize_device(d_f, T, 20, d_p)
    got = np.zeros_like(want)
    L.lpcnet_b200_memcpy_d2h(got.ctypes.data, d_p, want.nbytes)
    np.testing.assert_array_equal(got, want)
    L.lpcnet_b200_device_free(d_f); L.lpcnet_b200_device_free(d_p)
    b1.close(); b2.close()


@pytest.mark.parametrize("spc", ["1", "2", "3", "32"])
def test_float_flavour_kernels_agree_with_oracle(eng, monkeypatch, spc):
    """Float flavour: the neuron-per-lane kernel (1, 2 or 4 stream slots per CTA, incl. a ragged last CTA) and the
    lane==stream kernel (32 slots) against the float oracle on 7 fresh streams."""
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", spc)
    n = 7
    f = make_feature_batch(range(300, 300 + n), 6)
    b = eng.Batch(n, H.blob("float"), lpc_gamma=H.LPC_GAMMA)
    got = b.synthesize(f[:, :4])
    got2 = b.synthesize(f[:, 4:])                       # second call: state carried through the kernel's save/restore
    b.close()
    want = H.oracle_synth(f, kind="float")
    assert _first_diff(np.concatenate([got, got2], axis=1), want) is None


def test_float_flavour_matches_reference_golden(eng):
    """BASELINE config 2 arithmetic: the DISABLE_DOT_PROD (float) model flavour with fp16-stored recurrent weights must
    reproduce the reference's float build (pinned oracle build B) bit for bit — order-sensitive FMA chains included."""
    gold = np.load(os.path.join(H.GOLDEN, "synth_B.npz"))["pcm"]
    b = eng.Batch(4, H.blob("float"), lpc_gamma=H.LPC_GAMMA)
    got = b.synthesize(make_feature_batch(range(4), 40))
    assert _first_diff(got, gold) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, gold),)
    b.close()
    n, T = 37, 9                                       # ragged batch vs the oracle's float path
    f = make_feature_batch(range(1200, 1200 + n), T)
    b = eng.Batch(n, H.blob("float"), lpc_gamma=H.LPC_GAMMA)
    got = b.synthesize(f)
    want = H.oracle_synth(f, "float")
    assert _first_diff(got, want) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, want),)
    dig = json.load(open(os.path.join(H.GOLDEN, "digests.json")))
    b.close()
    b = eng.Batch(16, H.blob("float"), lpc_gamma=H.LPC_GAMMA)
    assert hashlib.sha256(b.synthesize(make_feature_batch(range(16), 150)).tobytes()).hexdigest() == dig["synth_B_16x150"]
    b.close()
