"""GPU tests (-m gpu) of lpcnet_decode on the engine, checked as synthesis is: every model variant in both flavours against the
reference's stored digests and under every per-sample schedule against the CPU restatement; seeded random sequences that mix
decodes with synthesis and the lifecycle operations (scenarios.random_script(..., decode=True)); the decoder-memory contract
rule by rule; the device-pointer entry points on caller streams; and the benchmark's call pattern at BASELINE sizes against the
committed per-stream digests.

The decoder memory (vq_mem, the previous superframe's cepstrum) is per-stream state: a reset or reset_streams clears it as
lpcnet_decoder_init does, reset_signal keeps it, and the exported state and snapshots carry it."""
import ctypes
import json
import os
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
import helpers as H
import scenarios as S
from fixtures import make_feature_batch, make_packets, make_pcm, make_pcm_batch
from test_decode_sequences import CASES, SEEDS, TAGS, decode_inputs, decode_key, seq_inputs, seq_key
from test_gpu_lifecycle_sequences import SCHEDULES, _knob_id

pytestmark = pytest.mark.gpu
GPU_SEEDS = range(3)
KINDS = ["int8", "float"]
DIG = os.path.join(H.GOLDEN, "at_size_digests.npz")


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


@pytest.fixture(scope="module")
def pool():
    with ThreadPoolExecutor(os.cpu_count() or 4) as p:
        yield p


def _batch(eng, kind, tag, n):
    return eng.Batch(n, H.blob(kind, tag), config=H.model_config(tag), codebooks=H.codebooks())


def _assert_same(got, want, what):
    d = np.argwhere(got != want)
    assert d.size == 0, "%s: %d samples differ, first (stream, sample) = %s" % (what, len(d), tuple(d[0]))


def _packets(streams, P):
    """even stream ids: random packets; odd ones: packets the encoder made from speech"""
    return np.stack([make_packets(s, P) if s % 2 == 0 else H.oracle_encode(make_pcm(s, 4 * P)[None])[0] for s in streams])


def _vq_mem(b, blob):
    """vq_mem of an exported state: floats hA[na] hB[16] last_sig[16] deemph conv1[168] conv2[256] lpc_carry[32], then vq_mem[18]"""
    o = b.na + 16 + 16 + 1 + 168 + 256 + 32
    return blob[o:o + 18]


# ---- 1. every variant in both flavours ----
@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("kind,build", [("int8", "A"), ("float", "B")])
def test_variant_decode_matches_reference_digest(eng, tag, kind, build):
    """The packets of test_decode_sequences.decode_inputs in two calls (20 and 28 frames: both cross the 16-frame chunk)."""
    pk = decode_inputs()
    b = _batch(eng, kind, tag, len(pk))
    got = np.concatenate([b.decode(pk[:, :5]), b.decode(pk[:, 5:])], axis=1)
    b.close()
    assert H.digest(got) == json.load(open(H.REF_DIGESTS))[decode_key(tag, build)]


# (kind, streams, create-time knobs): pinned like test_gpu_variants.VARIANT_SPC, since a batch this small falls to one stream per
# CTA on its own
DECODE_SCHEDULES = [
    ("int8", 9, {}),                                                     # automatic: one half, one live slot per CTA
    ("int8", 70, {"STREAMS_PER_CTA": "32"}),                             # two halves, CTAs of 32, 32 and 6
    ("int8", 40, {"STREAMS_PER_CTA": "17"}),                             # the smallest two-half CTA
    ("int8", 12, {"STREAMS_PER_CTA": "5", "TWO_HALVES": "1"}),           # dead slots in both halves
    ("int8", 40, {"STREAMS_PER_CTA": "32", "EXACT_CVT": "1"}),           # the conversion unit
    ("float", 5, {}),                                                    # neuron-per-lane
    ("float", 8, {"STREAMS_PER_CTA": "3"}),                              # neuron-per-lane, ragged
    ("float", 6, {"FLOAT_LANE_STREAM": "1"}),                            # lane == stream
]


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("kind,n,knobs", DECODE_SCHEDULES, ids=[_knob_id((c[0], "", c[1], c[2])) for c in DECODE_SCHEDULES])
def test_variant_decode_batches_match_oracle(eng, monkeypatch, tag, kind, n, knobs):
    for k, v in knobs.items():
        monkeypatch.setenv("LPCNET_B200_" + k, v)
    streams = range(800, 800 + n)
    pk = _packets(streams, 7)
    b = _batch(eng, kind, tag, n)
    got = np.concatenate([b.decode(pk[:, :2]), b.decode(pk[:, 2:])], axis=1)
    b.close()
    _assert_same(got, H.oracle_decode(pk, kind, tag=tag), "%s %s" % (kind, tag))


# ---- 2. random sequences with decodes ----
def _engine(eng, kind, tag, f, streams, script):
    b = _batch(eng, kind, tag, len(streams))
    try:
        return S.run_engine_script(b, f, streams, script)
    finally:
        b.close()


def _oracle(kind, tag, f, streams, script, pool=None):
    return S.run_streams("oracle", H.oracle_lib(), S.OracleState(kind, tag), f, streams, script, pool)


@pytest.mark.parametrize("kind,tag,n,knobs", SCHEDULES, ids=[_knob_id(c) for c in SCHEDULES])
def test_random_decode_sequences_match_oracle(eng, pool, monkeypatch, kind, tag, n, knobs):
    for k, v in knobs.items():
        monkeypatch.setenv("LPCNET_B200_" + k, v)
    for seed in GPU_SEEDS:
        script = S.random_script(3000 + seed, n, decode=True)
        streams = list(range(900 + 100 * seed, 900 + 100 * seed + n))
        f = make_feature_batch(streams, max(script[1], 1))
        got = _engine(eng, kind, tag, f, streams, script)
        _assert_same(got, _oracle(kind, tag, f, streams, script, pool), "seed %d (%s packets) %s" % (seed, script[3], script[0]))


@pytest.mark.parametrize("build,tag", CASES)
def test_cpu_decode_seeds_match_reference_digests(eng, build, tag):
    stored = json.load(open(H.REF_DIGESTS))
    kind = "float" if build == "B" else "int8"
    for seed in SEEDS:
        script, f, streams = seq_inputs(seed)
        assert H.digest(_engine(eng, kind, tag, f, streams, script)) == stored[seq_key(build, tag, seed)], "seed %d" % seed


# ---- 3. the decoder-memory contract, one rule per test ----
@pytest.mark.parametrize("kind", KINDS)
def test_decode_split_over_calls_equals_one_call(eng, kind):
    n, P = 5, 9
    pk = _packets(range(20, 20 + n), P)
    b = _batch(eng, kind, "", n)
    whole = b.decode(pk)
    b.close()
    _assert_same(whole, H.oracle_decode(pk, kind), "one call")
    for split in ((1, 4, 4), (5, 4), (3, 3, 3), (2, 6, 1), (4, 5)):          # calls of 16 frames, and calls that cross the chunk
        b = _batch(eng, kind, "", n)
        starts = np.cumsum((0,) + split[:-1])
        got = np.concatenate([b.decode(pk[:, a:a + k]) for a, k in zip(starts, split)], axis=1)
        b.close()
        _assert_same(got, whole, "calls of %s packets" % (split,))


@pytest.mark.parametrize("kind", KINDS)
def test_exported_decoding_stream_continues_in_a_fresh_batch(eng, kind):
    n, P = 4, 7
    pk = _packets(range(30, 30 + n), P)
    a = _batch(eng, kind, "", n)
    a.decode(pk[:, :3])
    blob = a.export_state(2)
    cont = a.decode(pk[:, 3:])
    st = H.oracle_lib().oracle_state_create(H.oracle_model(kind))
    pcm = np.zeros(640, np.int16)
    for p in range(3):
        H.oracle_lib().oracle_decode(st, pk[2, p].ctypes.data, pcm.ctypes.data)
    want = np.zeros_like(blob)
    H.oracle_lib().oracle_export_state(st, want.ctypes.data)
    H.oracle_lib().oracle_state_destroy(st)
    np.testing.assert_array_equal(_vq_mem(a, blob).view(np.uint32), _vq_mem(a, want).view(np.uint32))
    assert np.abs(_vq_mem(a, blob)).max() > 0
    a.close()
    b = _batch(eng, kind, "", n)
    b.import_state(1, blob)
    q = pk[:, 3:].copy()
    q[1] = pk[2, 3:]
    got = b.decode(q)
    b.close()
    _assert_same(got[1], cont[2], "imported stream")


@pytest.mark.parametrize("kind", KINDS)
def test_restore_brings_back_the_decoder_memory(eng, kind):
    n = 4
    pk = _packets(range(40, 40 + n), 6)
    b = _batch(eng, kind, "", n)
    first = b.decode(pk[:, :2])
    snap = b.snapshot()
    x = b.decode(pk[:, 2:5])
    b.restore(snap)
    y = b.decode(pk[:, 2:5])
    b.free_snapshot(snap)
    b.close()
    _assert_same(y, x, "decode after restore")
    _assert_same(np.concatenate([first, x], axis=1), H.oracle_decode(pk[:, :5], kind), "decode vs oracle")


@pytest.mark.parametrize("kind", KINDS)
def test_reset_streams_starts_a_new_utterance_in_the_listed_streams(eng, kind):
    n, ids = 5, [0, 3]
    pk = _packets(range(50, 50 + n), 6)
    fresh = _batch(eng, kind, "", n).decode(pk[:, 3:])
    cont = _batch(eng, kind, "", n).decode(pk)[:, 3 * 640:]
    b = _batch(eng, kind, "", n)
    b.decode(pk[:, :3])
    b.reset_streams(ids)
    for s in range(n):
        assert (np.abs(_vq_mem(b, b.export_state(s))).max() == 0) == (s in ids), "stream %d" % s
    got = b.decode(pk[:, 3:])
    for s in range(n):
        _assert_same(got[s], (fresh if s in ids else cont)[s], "stream %d (%s)" % (s, "reset" if s in ids else "not reset"))
    b.reset()                                                  # the whole batch: every stream equals a fresh decoder
    _assert_same(b.decode(pk[:, 3:]), fresh, "after batch_reset")
    b.close()


@pytest.mark.parametrize("kind", KINDS)
def test_reset_signal_keeps_the_decoder_memory(eng, pool, kind):
    n = 4
    streams = list(range(60, 60 + n))
    script = ([("decode", 0, 2), ("reset_signal",), ("decode", 2, 2), ("reset_signal",), ("decode", 4, 5)], 1, "speech", "encoded")
    f = make_feature_batch(streams, 1)
    got = _engine(eng, kind, "", f, streams, script)
    _assert_same(got, _oracle(kind, "", f, streams, script, pool), "decode / reset_signal")
    b = _batch(eng, kind, "", n)
    b.decode(S.script_packets(script, streams)[:, :2])
    before = [_vq_mem(b, b.export_state(s)).copy() for s in range(n)]
    b.reset_signal()
    for s in range(n):
        np.testing.assert_array_equal(_vq_mem(b, b.export_state(s)), before[s])
        assert np.abs(before[s]).max() > 0
    b.close()


@pytest.mark.parametrize("kind", KINDS)
def test_tail_after_decode_reads_the_last_decoded_frame(eng, pool, kind):
    n = 4
    streams = list(range(70, 70 + n))
    script = ([("decode", 0, 3), ("tail", 160, 0), ("tail", 80, 40), ("decode", 3, 5), ("tail", 160, 0)], 1, "speech", "random")
    f = make_feature_batch(streams, 1)
    got = _engine(eng, kind, "", f, streams, script)
    _assert_same(got, _oracle(kind, "", f, streams, script, pool), "tails after decodes")
    assert np.abs(got[:, 3 * 640:3 * 640 + 160]).max() > 0


# ---- 4. the device-pointer entry points on caller streams ----
class Dev:
    """A device buffer `off` bytes into its allocation."""
    def __init__(self, L, nbytes, off=512):
        self.L, self.nbytes = L, nbytes
        self.base = L.lpcnet_b200_device_alloc(nbytes + off)
        assert self.base
        self.ptr = self.base + off

    def put(self, a):
        a = np.ascontiguousarray(a)
        assert a.nbytes == self.nbytes
        assert self.L.lpcnet_b200_memcpy_h2d(self.ptr, a.ctypes.data, a.nbytes) == 0
        one = np.zeros(1, np.uint8)                            # the copy has landed before work on other streams reads it
        assert self.L.lpcnet_b200_memcpy_d2h(one.ctypes.data, self.ptr, 1) == 0
        return self

    def get(self, shape, dtype):
        out = np.empty(shape, dtype)
        assert out.nbytes == self.nbytes
        assert self.L.lpcnet_b200_memcpy_d2h(out.ctypes.data, self.ptr, out.nbytes) == 0
        return out

    def free(self):
        self.L.lpcnet_b200_device_free(self.base)


@pytest.fixture
def streams2(eng):
    L = eng.lib()
    s = [L.lpcnet_b200_stream_create() for _ in range(2)]
    assert all(s)
    yield s
    for x in s:
        L.lpcnet_b200_stream_sync(x)
        L.lpcnet_b200_stream_destroy(x)


def _sync(L, streams):
    for s in streams:
        assert L.lpcnet_b200_stream_sync(s) == 0


def test_decode_device_on_two_streams_equals_host_decode(eng, streams2):
    L, n = eng.lib(), 6
    pk = _packets(range(80, 80 + n), 9)
    parts = [(0, 2), (2, 1), (3, 2)]                           # device calls on streams 0, 1, 0; then a host call of 4 packets
    h = _batch(eng, "int8", "", n)
    want = np.concatenate([h.decode(pk[:, a:a + k]) for a, k in parts + [(5, 4)]], axis=1)
    h.close()
    b = _batch(eng, "int8", "", n)
    bufs = []
    for i, (a, k) in enumerate(parts):
        dpk = Dev(L, n * k * 8, 512 * (i + 1)).put(pk[:, a:a + k])
        dpcm = Dev(L, n * k * 640 * 2, 512 * (i + 2))
        b.decode_device(dpk.ptr, k, dpcm.ptr, cuda_stream=streams2[i % 2])
        bufs.append((dpk, dpcm, k))
    last = b.decode(pk[:, 5:])                                 # grows the staging buffers right after a call on another stream
    _sync(L, streams2)
    got = np.concatenate([d.get((n, k * 640), np.int16) for _, d, k in bufs] + [last], axis=1)
    for x, y, _ in bufs:
        x.free(); y.free()
    b.close()
    _assert_same(got, want, "device calls vs host calls")
    _assert_same(got, H.oracle_decode(pk, "int8"), "vs oracle")


@pytest.mark.parametrize("kind", KINDS)
def test_synthesize_device_ex_preload_applies_to_the_first_chunk_only(eng, pool, streams2, kind):
    """20 frames with 40 forced samples (the second chunk of the call must not be forced), 10 frames with 17, then a host call."""
    L, n = eng.lib(), 6
    streams = list(range(90, 90 + n))
    script = ([("synth", 0, 20, 160, 40), ("synth", 20, 10, 160, 17), ("synth", 30, 20, 160, 0)], 50, "speech")
    f = make_feature_batch(streams, 50)
    want = _oracle(kind, "", f, streams, script, pool)
    h = eng.Batch(n, H.blob(kind), lpc_gamma=H.LPC_GAMMA)
    _assert_same(S.run_engine_script(h, f, streams, script), want, "host calls vs oracle")
    h.close()
    forced = np.stack([S.forced_pcm("speech", s, S.script_outputs(script)) for s in streams])
    b = eng.Batch(n, H.blob(kind), lpc_gamma=H.LPC_GAMMA)
    bufs, k0 = [], 0
    for i, (_, t, nf, N, pre) in enumerate(script[0][:2]):
        df = Dev(L, n * nf * 20 * 4, 512 * (i + 1)).put(f[:, t:t + nf])
        init = np.zeros((n, nf * N), np.int16)
        init[:, :pre] = forced[:, k0:k0 + pre]
        dp = Dev(L, init.nbytes, 512 * (i + 2)).put(init)
        b.synthesize_device(df.ptr, nf, 20, dp.ptr, samples_per_frame=N, cuda_stream=streams2[i], preload=pre)
        bufs.append((df, dp, nf * N)); k0 += nf * N
    last = b.synthesize(f[:, 30:50])
    _sync(L, streams2)
    got = np.concatenate([d.get((n, m), np.int16) for _, d, m in bufs] + [last], axis=1)
    for x, y, _ in bufs:
        x.free(); y.free()
    b.close()
    _assert_same(got, want, "device calls vs oracle")


def test_encoder_device_entry_points_on_two_streams_equal_host_calls(eng, streams2):
    L, n = eng.lib(), 5
    cb = H.codebooks()
    pcm = make_pcm_batch(range(100, 100 + n), 24)
    # features: frames [0, 3) on stream 0, [3, 8) on stream 1, then a host call of 16 frames
    h = eng.EncBatch(n, codebooks=cb)
    want = np.concatenate([h.compute_features(pcm[:, a * 160:b * 160]) for a, b in ((0, 3), (3, 8), (8, 24))], axis=1)
    h.close()
    e = eng.EncBatch(n, codebooks=cb)
    outs, bufs = [], []
    for i, (a, b) in enumerate(((0, 3), (3, 8))):
        dp = Dev(L, n * (b - a) * 160 * 2, 512 * (i + 1)).put(pcm[:, a * 160:b * 160])
        df = Dev(L, n * (b - a) * 36 * 4, 512 * (i + 2))
        e.compute_features_device(dp.ptr, b - a, df.ptr, cuda_stream=streams2[i])
        bufs.append((dp, df, b - a))
    last = e.compute_features(pcm[:, 8 * 160:])
    _sync(L, streams2)
    got = np.concatenate([d.get((n, k, 36), np.float32) for _, d, k in bufs] + [last], axis=1)
    for x, y, _ in bufs:
        x.free(); y.free()
    e.close()
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(got.view(np.uint32), H.oracle_features(pcm).view(np.uint32))
    # packets: [0, 1) on stream 0, [1, 3) on stream 1, then a host call of 3 packets
    h = eng.EncBatch(n, codebooks=cb)
    want = np.concatenate([h.encode(pcm[:, a * 640:b * 640]) for a, b in ((0, 1), (1, 3), (3, 6))], axis=1)
    h.close()
    e = eng.EncBatch(n, codebooks=cb)
    bufs = []
    for i, (a, b) in enumerate(((0, 1), (1, 3))):
        dp = Dev(L, n * (b - a) * 640 * 2, 512 * (i + 1)).put(pcm[:, a * 640:b * 640])
        dk = Dev(L, n * (b - a) * 8, 512 * (i + 2))
        e.encode_device(dp.ptr, b - a, dk.ptr, cuda_stream=streams2[i])
        bufs.append((dp, dk, b - a))
    last = e.encode(pcm[:, 3 * 640:])
    _sync(L, streams2)
    got = np.concatenate([d.get((n, k, 8), np.uint8) for _, d, k in bufs] + [last], axis=1)
    for x, y, _ in bufs:
        x.free(); y.free()
    e.close()
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got, H.oracle_encode(pcm))


# ---- 5. the benchmark's call pattern at BASELINE sizes ----
# bench.py times each step as flush_l2, timer_start, one `_device` call on the engine's stream, timer_stop, with the state carried
# from step to step, and then runs host-pointer calls on lpcnet_b200_host_alloc buffers.  It repeats the same 10 frames (or 2
# packets) every step; here each call takes the next slice of the at-size inputs instead, so that the committed per-stream digests
# of tests/golden/at_size_digests.npz (the reference over the whole duration) apply.
def _check(got, want, what):
    bad = np.nonzero(H.stream_digests(got) != want)[0]
    assert bad.size == 0, "%s: %d of %d streams differ from the reference, first: %s" % (what, bad.size, len(want), bad[:16].tolist())


def _timed(b, call):
    b.flush_l2()
    b.timer_start()
    call()
    assert b.timer_stop() > 0


def _device_steps(eng, b, inputs, per_call, step, out_per_unit):
    """inputs [n][U][...] in calls of `per_call` units through step(d_in, count, d_out); returns [n][U * out_per_unit] int16"""
    L = eng.lib()
    n, U = inputs.shape[:2]
    d_in = Dev(L, inputs[:, :per_call].nbytes)
    d_out = Dev(L, n * per_call * out_per_unit * 2)
    out = []
    for u in range(0, U, per_call):
        d_in.put(inputs[:, u:u + per_call])
        _timed(b, lambda: step(d_in.ptr, per_call, d_out.ptr))
        out.append(d_out.get((n, per_call * out_per_unit), np.int16))
    d_in.free(); d_out.free()
    return out


def test_config3_bench_call_pattern(eng):
    n, T = 4096, 100
    f = make_feature_batch(range(n), T)
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    out = _device_steps(eng, b, f[:, :80], 10, lambda d, k, p: b.synthesize_device(d, k, 20, p), 160)
    L = eng.lib()
    fb, pb = n * 10 * 20 * 4, n * 10 * 160 * 2
    h_feat, h_pcm = L.lpcnet_b200_host_alloc(fb), L.lpcnet_b200_host_alloc(pb)
    assert h_feat and h_pcm
    def step_e2e():                                            # bench.py step_e2e: the host-pointer call on pinned buffers
        assert L.lpcnet_b200_batch_synthesize(b._h, h_feat, 10, 20, 160, h_pcm) == 0, L.lpcnet_b200_last_error()
    for t in (80, 90):
        chunk = np.ascontiguousarray(f[:, t:t + 10])              # (a named array: it must outlive the copy)
        ctypes.memmove(h_feat, chunk.ctypes.data, fb)
        b.sync()
        _timed(b, step_e2e)
        out.append(np.ctypeslib.as_array(ctypes.cast(h_pcm, ctypes.POINTER(ctypes.c_int16)), shape=(n, 1600)).copy())
    L.lpcnet_b200_host_free(h_feat); L.lpcnet_b200_host_free(h_pcm)
    b.close()
    _check(np.concatenate(out, axis=1), np.load(DIG)["config3_int8"], "config3_int8 4096x100 in bench.py's calls")


def test_config2_bench_call_pattern(eng):
    n, T = 256, 1000
    b = eng.Batch(n, H.blob("float"), lpc_gamma=H.LPC_GAMMA)
    out = _device_steps(eng, b, make_feature_batch(range(n), T), 10, lambda d, k, p: b.synthesize_device(d, k, 20, p), 160)
    b.close()
    _check(np.concatenate(out, axis=1), np.load(DIG)["config2_float"], "config2_float 256x1000 in bench.py's calls")


def test_config5_bench_call_pattern(eng):
    n, P = 1024, 250
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA, codebooks=H.codebooks())
    pk = np.stack([make_packets(s, P) for s in range(n)])
    out = _device_steps(eng, b, pk, 2, lambda d, k, p: b.decode_device(d, k, p), 640)
    b.close()
    _check(np.concatenate(out, axis=1), np.load(DIG)["config5_decode"], "config5_decode 1024x250 in bench.py's calls")
