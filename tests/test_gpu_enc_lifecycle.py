"""GPU tests (-m gpu) of the per-stream state calls of an encoder batch: lpcnet_b200_enc_reset_streams, _export_state /
_import_state and _copy_streams.  Every comparison is bit for bit (floats as bit patterns, packets as bytes):
  * a reset row goes on exactly as the CPU restatement (oracle/lpcnet_enc_oracle.inc) run from a fresh state over the row's PCM
    since its reset, and every other row exactly as on an untouched control batch;
  * an exported, imported or copied row goes on exactly as its source row does in an uninterrupted run;
  * every refused call leaves both batches as they were (every row exported before and after);
  * the calls wait for `_device` work still queued on caller streams and give what the serial run gives."""
import random
import numpy as np
import pytest
import helpers as H
from fixtures import make_pcm_batch

pytestmark = pytest.mark.gpu

UNIT = {"features": 160, "featuresf": 160, "encode": 640, "features4": 640}
STATE_BYTES = 16044              # one LPCNetEncState row (enc_kernels.cu EncState)
PCOUNT_WORD, BEST_I_WORD = 161, 3848   # int32 words of the row: pcount after analysis_mem[160] and mem_preemph; best_i after pmp_all
BLOCK_CYCLES = 60_000_000        # the spin ahead of a queued call (as tests/test_gpu_ordering.py)


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


def pcm_rows(n, nframes, pool=97):
    """[n][nframes*160] int16 speech-like PCM.  Past `pool` rows, row i is a window of pool stream i % pool that starts
    37 * (i // pool) samples in, so that no two rows are alike (make_pcm is slow for thousands of rows)."""
    if n <= pool:
        return make_pcm_batch(range(500, 500 + n), nframes)
    shift = 37 * ((n - 1) // pool)
    base = make_pcm_batch(range(500, 500 + pool), nframes + shift // 160 + 1)
    i = np.arange(n)
    idx = (i // pool)[:, None] * 37 + np.arange(nframes * 160)[None, :]
    return np.ascontiguousarray(base[i % pool][i[:, None], idx])


def run_op(e, op, seg):
    if op == "features":
        return e.compute_features(seg)
    if op == "featuresf":
        return e.compute_features(seg.astype(np.float32))
    if op == "encode":
        return e.encode(seg)
    return e.compute_features4(seg)


def run_ops(e, pcm, ops, resets=None, start=0):
    """ops (op, first sample, units) on EncBatch e, row i reading pcm[i]; resets = {op index: rows} reset before that op"""
    outs = []
    for i, (op, a, k) in enumerate(ops):
        if resets and start + i in resets:
            e.reset_streams(resets[start + i])
        outs.append(run_op(e, op, pcm[:, a:a + k * UNIT[op]]))
    return outs


def run_oracle(pcm, ops, resets=None):
    """the same on the CPU restatement, one state per row; a reset row gets a fresh state"""
    L, cb = H.oracle_lib(), H.codebooks()
    n = pcm.shape[0]
    st = [L.oracle_enc_create(cb.ctypes.data) for _ in range(n)]
    outs = []
    for i, (op, a, k) in enumerate(ops):
        for r in set(int(v) for v in (resets or {}).get(i, [])):
            L.oracle_enc_destroy(st[r])
            st[r] = L.oracle_enc_create(cb.ctypes.data)
        seg = np.ascontiguousarray(pcm[:, a:a + k * UNIT[op]], dtype=np.float32 if op == "featuresf" else np.int16)
        if op in ("features", "featuresf"):
            out = np.zeros((n, k, 36), np.float32)
            fn = L.oracle_enc_single_frame_features_float if op == "featuresf" else L.oracle_enc_single_frame_features
            for s in range(n):
                for t in range(k):
                    fn(st[s], seg[s, t * 160:].ctypes.data, out[s, t].ctypes.data)
        elif op == "encode":
            out = np.zeros((n, k, 8), np.uint8)
            for s in range(n):
                for p in range(k):
                    L.oracle_enc_encode(st[s], seg[s, p * 640:].ctypes.data, out[s, p].ctypes.data)
        else:
            out = np.zeros((n, 4 * k, 36), np.float32)
            for s in range(n):
                for p in range(k):
                    L.oracle_enc_compute_features(st[s], seg[s, p * 640:].ctypes.data, out[s, 4 * p].ctypes.data)
        outs.append(out)
    for s in st:
        L.oracle_enc_destroy(s)
    return outs


def make_ops(spec, a=0):
    """[(op, units)] -> [(op, first sample, units)] from sample a on; returns (ops, next sample)"""
    ops = []
    for op, k in spec:
        ops.append((op, a, k))
        a += k * UNIT[op]
    return ops, a


def random_spec(seed, n_ops):
    rng = random.Random(seed)
    spec = []
    for _ in range(n_ops):
        op = rng.choice(["features", "features", "featuresf", "encode", "features4"])
        spec.append((op, rng.choice((1, 2, 3, 5)) if UNIT[op] == 160 else rng.choice((1, 2))))
    return spec


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = np.ascontiguousarray(g), np.ascontiguousarray(w)
        assert g.shape == w.shape and g.dtype == w.dtype, "%s, item %d: %s %s vs %s %s" % (what, i, g.dtype, g.shape, w.dtype, w.shape)
        if g.tobytes() != w.tobytes():
            rows = np.argwhere((g.view(np.uint8).reshape(g.shape[0], -1) != w.view(np.uint8).reshape(w.shape[0], -1)).any(axis=1)).ravel()
            raise AssertionError("%s, item %d: rows %s differ" % (what, i, rows[:10].tolist()))


def rows_of(outs, rows):
    return [o[rows] for o in outs]


def states(e, rows=None):
    return [e.export_state(r) for r in (range(e.n) if rows is None else rows)]


def word(blob, w):
    return int(blob.view(np.int32)[w])


# ---- 1: resets of some rows -------------------------------------------------------------------------------------------------
RESET_SCRIPTS = {
    # seeded mix of every entry point; row lists with row 0, the last row, a repeated id, an empty list, every row, a random set
    "random": (random_spec(7100, 16), {3: [0, 63, 17, 17], 6: [], 9: list(range(64)), 12: sorted(random.Random(1).sample(range(64), 20))}),
    # a reset on rows left mid-superframe by lpcnet_encode (pcount == 3), then single-frame calls
    "after_encode": ([("encode", 2), ("features", 3), ("features", 2), ("featuresf", 1), ("encode", 1), ("features", 2)], {2: [1, 3, 63]}),
}


@pytest.mark.parametrize("name", list(RESET_SCRIPTS))
def test_reset_streams_restarts_listed_rows_only(eng, name):
    spec, resets = RESET_SCRIPTS[name]
    n = 64
    ops, samples = make_ops(spec)
    pcm = pcm_rows(n, samples // 160)
    cb = H.codebooks()
    e, control = eng.EncBatch(n, codebooks=cb), eng.EncBatch(n, codebooks=cb)
    got, want_ctl = [], run_ops(control, pcm, ops)
    for i, (op, a, k) in enumerate(ops):
        if i in resets:
            if name == "after_encode":
                assert all(word(e.export_state(r), PCOUNT_WORD) == 3 for r in resets[i]), "premise: the reset rows are mid-superframe"
            e.reset_streams(resets[i])
        got.append(run_op(e, op, pcm[:, a:a + k * UNIT[op]]))
    assert_same(got, run_oracle(pcm, ops, resets), "%s: engine with resets vs CPU restatement" % name)
    reset_so_far, compared = set(), 0
    for i in range(len(ops)):
        reset_so_far |= set(resets.get(i, []))
        untouched = sorted(set(range(n)) - reset_so_far)
        assert_same([got[i][untouched]], [want_ctl[i][untouched]], "%s, op %d: rows not reset yet vs control batch" % (name, i))
        compared += len(untouched) > 0 and len(untouched) < n
    assert compared, "premise: some calls see reset and untouched rows side by side"
    e.close(); control.close()


def test_reset_of_every_row_equals_enc_reset(eng):
    n = 12
    ops, samples = make_ops([("features", 3), ("encode", 1), ("features", 1)])
    pcm = pcm_rows(n, samples // 160 + 8)
    cb = H.codebooks()
    a, b = eng.EncBatch(n, codebooks=cb), eng.EncBatch(n, codebooks=cb)
    for e in (a, b):
        run_ops(e, pcm, ops)
    assert any(blob.any() for blob in states(a)), "premise: the state is not zero before the reset"
    a.reset_streams(list(range(n)) + [4, 0])
    b.reset()
    assert_same(states(a), states(b), "reset_streams(every row) vs enc_reset")
    assert not any(blob.any() for blob in states(a)), "a reset row is lpcnet_encoder_init's zero state"
    more, _ = make_ops([("features", 2), ("encode", 1)], samples)
    assert_same(run_ops(a, pcm, more), run_ops(b, pcm, more), "after the resets")
    a.close(); b.close()


# ---- 2: export and import ---------------------------------------------------------------------------------------------------
PREFIXES = {"pcount0": ([("features", 3), ("featuresf", 2)], 0), "pcount3": ([("features", 3), ("encode", 1), ("features", 2)], 3)}


@pytest.mark.parametrize("prefix", list(PREFIXES))
def test_export_import_continues_exactly(eng, prefix):
    spec, pcount = PREFIXES[prefix]
    n = 16
    pre, a0 = make_ops(spec)
    post, samples = make_ops([("features", 3), ("encode", 2), ("features4", 1), ("featuresf", 2), ("features", 1)], a0)
    pcm = pcm_rows(n, samples // 160)
    cb = H.codebooks()
    ref = eng.EncBatch(n, codebooks=cb)
    run_ops(ref, pcm, pre)
    want = run_ops(ref, pcm, post)
    x, y = eng.EncBatch(n, codebooks=cb), eng.EncBatch(n, codebooks=cb)
    run_ops(x, pcm, pre)
    blobs = states(x)
    assert x.state_size() == STATE_BYTES and all(b.dtype == np.uint8 and b.size == x.state_size() for b in blobs)
    assert all(word(b, PCOUNT_WORD) == pcount for b in blobs), "premise: pcount after the prefix"
    assert all(0 <= word(b, BEST_I_WORD) < 256 for b in blobs)
    rng = np.random.default_rng(5)
    px, py = rng.permutation(n), rng.permutation(n)           # row d of x takes the row px[d] had; row d of y the row py[d] of x had
    for d in range(n):
        x.import_state(d, blobs[px[d]])
        y.import_state(d, blobs[py[d]])
    assert_same(states(x), [blobs[s] for s in px], "export, import, export")
    assert_same(states(y), [blobs[s] for s in py], "export, import into a fresh batch, export")
    # refused blobs change nothing: the row goes on as imported
    for w, v, msg in ((PCOUNT_WORD, 4, "pcount"), (PCOUNT_WORD, -1, "pcount"), (BEST_I_WORD, 256, "best_i")):
        bad = blobs[0].copy()
        bad.view(np.int32)[w] = v
        with pytest.raises(eng.LPCNetB200Error, match=msg):
            x.import_state(2, bad)
    assert_same(run_ops(x, pcm[px], post), rows_of(want, px), "%s: imported rows of the same batch vs uninterrupted run" % prefix)
    assert_same(run_ops(y, pcm[py], post), rows_of(want, py), "%s: rows imported into a fresh batch vs uninterrupted run" % prefix)
    for e in (ref, x, y):
        e.close()


# ---- 3: copies ----------------------------------------------------------------------------------------------------------------
def test_compaction_mid_script(eng):
    """100 scattered live rows of a 1024-row batch move into a 100-row batch between two calls (rows mid-superframe)."""
    n, live_n = 1024, 100
    pre, a0 = make_ops([("features", 3), ("encode", 1), ("featuresf", 2)])
    post, samples = make_ops([("features", 2), ("encode", 2), ("features4", 1), ("features", 3)], a0)
    pcm = pcm_rows(n, samples // 160)
    cb = H.codebooks()
    big = eng.EncBatch(n, codebooks=cb)
    run_ops(big, pcm, pre)
    live = np.sort(np.random.default_rng(11).choice(n, live_n, replace=False))
    small = eng.EncBatch(live_n, codebooks=cb)
    before = states(big, live)
    small.copy_streams(np.arange(live_n), big, live)
    assert_same(states(small), before, "copied rows vs their sources")
    assert_same(states(big, live), before, "the source rows are unchanged")
    assert_same(run_ops(small, pcm[live], post), rows_of(run_ops(big, pcm, post), live), "compacted rows vs their sources")
    big.close(); small.close()


def test_rotation_swap_and_clone_in_one_batch(eng):
    n = 16
    pre, a0 = make_ops([("features", 2), ("encode", 1), ("features", 1)])
    post, samples = make_ops([("features", 3), ("encode", 1)], a0)
    pcm = pcm_rows(n, samples // 160)
    cb = H.codebooks()
    e, control = eng.EncBatch(n, codebooks=cb), eng.EncBatch(n, codebooks=cb)
    run_ops(e, pcm, pre)
    run_ops(control, pcm, pre)
    before = states(e)
    assert len({b.tobytes() for b in before}) == n, "premise: every row differs"
    dst, src = [0, 1, 2, 3, 4, 5, 8, 9, 10], [1, 2, 3, 0, 5, 4, 11, 11, 11]
    e.copy_streams(dst, e, src)
    m = np.arange(n)
    m[dst] = src
    assert_same(states(e), [before[s] for s in m], "rotation, swap and clone")
    assert_same(run_ops(e, pcm[m], post), rows_of(run_ops(control, pcm, post), m), "after the copy")
    e.close(); control.close()


def test_permutation_of_4096_rows(eng):
    n = 4096
    pre, a0 = make_ops([("features", 2), ("encode", 1), ("features", 1)])
    post, samples = make_ops([("encode", 1), ("features", 2)], a0)
    pcm = pcm_rows(n, samples // 160)
    cb = H.codebooks()
    e, control = eng.EncBatch(n, codebooks=cb), eng.EncBatch(n, codebooks=cb)
    run_ops(e, pcm, pre)
    run_ops(control, pcm, pre)
    perm = np.random.default_rng(13).permutation(n)
    e.copy_streams(np.arange(n), e, perm)
    probe = [0, 1, 97, 2048, n - 1]
    assert_same(states(e, probe), states(control, perm[probe]), "permuted rows vs their sources")
    assert_same(run_ops(e, pcm[perm], post), rows_of(run_ops(control, pcm, post), perm), "after the permutation")
    e.close(); control.close()


def test_copy_into_batch_without_codebooks(eng):
    n = 8
    pre, a0 = make_ops([("features", 1), ("encode", 1), ("features", 2)])
    post, samples = make_ops([("features", 3), ("featuresf", 2)], a0)
    pcm = pcm_rows(n, samples // 160 + 4)
    src = eng.EncBatch(n, codebooks=H.codebooks())
    run_ops(src, pcm, pre)
    rows = np.array([6, 1, 3, 3])
    dst = eng.EncBatch(len(rows))
    dst.copy_streams(np.arange(len(rows)), src, rows)
    assert_same(run_ops(dst, pcm[rows], post), rows_of(run_ops(src, pcm, post), rows), "features under a batch without codebooks")
    with pytest.raises(eng.LPCNetB200Error, match="codebooks"):
        dst.encode(pcm[rows, samples:samples + 640])
    src.close(); dst.close()


def test_refusals_change_nothing(eng):
    L = eng.lib()
    cb = H.codebooks()
    ops, samples = make_ops([("features", 2), ("encode", 1), ("features", 1)])
    pcm = pcm_rows(8, samples // 160)
    a, b = eng.EncBatch(8, codebooks=cb), eng.EncBatch(6)
    run_ops(a, pcm, ops)
    run_ops(b, pcm[:6], [op for op in ops if op[0] != "encode"])
    before = states(a) + states(b)
    keep = []

    def ia(*v):
        keep.append(np.array(v, np.int32))
        return keep[-1].ctypes.data
    buf = np.zeros(STATE_BYTES, np.uint8)
    calls = {
        "copy: NULL dst": lambda: L.lpcnet_b200_enc_copy_streams(None, ia(0), a._h, ia(0), 1),
        "copy: NULL dst rows": lambda: L.lpcnet_b200_enc_copy_streams(b._h, None, a._h, ia(0), 1),
        "copy: NULL src": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0), None, ia(0), 1),
        "copy: NULL src rows": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0), a._h, None, 1),
        "copy: count < 0": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0), a._h, ia(0), -1),
        "copy: source row out of range": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0, 1, 2), a._h, ia(1, 2, 8), 3),
        "copy: negative source row": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0, 1), a._h, ia(1, -1), 2),
        "copy: destination row out of range": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0, 6), a._h, ia(1, 2), 2),
        "copy: destination row repeated": lambda: L.lpcnet_b200_enc_copy_streams(b._h, ia(0, 1, 2, 1), a._h, ia(1, 2, 3, 4), 4),
        "copy in one batch: destination row repeated": lambda: L.lpcnet_b200_enc_copy_streams(a._h, ia(3, 3), a._h, ia(1, 2), 2),
        "reset: NULL batch": lambda: L.lpcnet_b200_enc_reset_streams(None, ia(0), 1),
        "reset: NULL rows": lambda: L.lpcnet_b200_enc_reset_streams(a._h, None, 1),
        "reset: count < 0": lambda: L.lpcnet_b200_enc_reset_streams(a._h, ia(0), -1),
        "reset: row out of range": lambda: L.lpcnet_b200_enc_reset_streams(a._h, ia(0, 5, 8), 3),
        "export: row out of range": lambda: L.lpcnet_b200_enc_export_state(a._h, 8, buf.ctypes.data),
        "export: NULL buffer": lambda: L.lpcnet_b200_enc_export_state(a._h, 0, None),
        "import: row out of range": lambda: L.lpcnet_b200_enc_import_state(a._h, -1, buf.ctypes.data),
        "import: NULL buffer": lambda: L.lpcnet_b200_enc_import_state(a._h, 0, None),
    }
    for what, call in calls.items():
        assert call() == -1, what
        assert L.lpcnet_b200_last_error(), "%s: no error message" % what
    with pytest.raises(eng.LPCNetB200Error):
        b.copy_streams([0, 1], a, [1])
    assert L.lpcnet_b200_enc_state_size(None) == -1
    # count == 0 does nothing and succeeds
    assert L.lpcnet_b200_enc_copy_streams(b._h, ia(0), a._h, ia(0), 0) == 0
    assert L.lpcnet_b200_enc_reset_streams(a._h, ia(0), 0) == 0
    b.copy_streams([], a, [])
    a.reset_streams([])
    assert_same(states(a) + states(b), before, "both batches after the refused calls")
    a.close(); b.close()


def test_copy_across_devices(eng):
    if eng.device_count() < 2:
        pytest.skip("needs two CUDA devices (%d visible)" % eng.device_count())
    n = 8
    pre, a0 = make_ops([("features", 2), ("encode", 1), ("features", 1)])
    post, samples = make_ops([("features", 2), ("encode", 1)], a0)
    pcm = pcm_rows(n, samples // 160)
    cb = H.codebooks()
    a, b, control = eng.EncBatch(n, 0, cb), eng.EncBatch(n, 1, cb), eng.EncBatch(n, 0, cb)
    for e in (a, b, control):
        run_ops(e, pcm, pre)
    before = states(a)
    rows = np.array([7, 0, 0, 3])
    b.copy_streams([0, 1, 2, 5], a, rows)          # device 0 -> device 1
    a.copy_streams([6, 7], b, [0, 4])              # and back: row 6 of a gets a's old row 7, row 7 gets b's row 4 (= a's old 4)
    m = np.arange(n)
    mb = m.copy(); mb[[0, 1, 2, 5]] = rows
    ma = m.copy(); ma[[6, 7]] = [7, 4]
    assert_same(states(b), [before[s] for s in mb], "device 0 -> 1")
    assert_same(states(a), [before[s] for s in ma], "device 1 -> 0")
    want = run_ops(control, pcm, post)
    assert_same(run_ops(b, pcm[mb], post), rows_of(want, mb), "rows on device 1")
    assert_same(run_ops(a, pcm[ma], post), rows_of(want, ma), "rows back on device 0")
    for e in (a, b, control):
        e.close()


# ---- 4: calls while `_device` work is still queued on caller streams -----------------------------------------------------------
ENC_N = 8


def busy(s):
    """a spin kernel on caller stream s; the returned event completes when it ends (as tests/test_gpu_ordering.py)"""
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(s)):
        torch.cuda._sleep(BLOCK_CYCLES)
        ev = torch.cuda.Event()
        ev.record()
    return ev


class Dev:
    """device buffers of one run; outputs are read back into their host arrays by finish() once the streams have drained"""

    def __init__(self, L):
        self.L, self.ptrs, self.reads = L, [], []

    def put(self, a):
        a = np.ascontiguousarray(a)
        p = self.L.lpcnet_b200_device_alloc(a.nbytes)
        assert p and self.L.lpcnet_b200_memcpy_h2d(p, a.ctypes.data, a.nbytes) == 0
        self.ptrs.append(p)
        return p

    def out(self, host):
        p = self.put(host)
        self.reads.append((p, host))
        return p

    def finish(self, streams):
        for s in streams:
            assert self.L.lpcnet_b200_stream_sync(s) == 0
        for p, h in self.reads:
            assert self.L.lpcnet_b200_memcpy_d2h(h.ctypes.data, p, h.nbytes) == 0
        for p in self.ptrs:
            self.L.lpcnet_b200_device_free(p)


def _x_export_import(e, o):
    blob = e.export_state(5)
    e.import_state(0, blob)
    return [blob]


ORDER_X = {
    "reset_streams": lambda e, o: e.reset_streams([0, ENC_N - 1, 3, 3]) or [],
    "export_import": _x_export_import,
    "copy_streams": lambda e, o: e.copy_streams([0, 2, 5], o, [7, 1, 1]) or [],
    "copy_in_one_batch": lambda e, o: e.copy_streams([0, 1, 2, 6], e, [2, 0, 1, 2]) or [],
}


def order_run(eng, x, streams, concurrent):
    """both batches encode a packet, then queue an encode_device of two packets on their own caller stream (behind a spin
    kernel when concurrent), then `x` runs on e (o: the other batch of a copy), then both encode and export every row"""
    L = eng.lib()
    cb = H.codebooks()
    pcm = pcm_rows(2 * ENC_N, 20)
    pe, po = pcm[:ENC_N], pcm[ENC_N:]
    e, o = eng.EncBatch(ENC_N, codebooks=cb), eng.EncBatch(ENC_N, codebooks=cb)
    dev = Dev(L)
    outs = [e.encode(pe[:, :640]), o.encode(po[:, :640])]
    qe, qo = np.zeros((ENC_N, 2, 8), np.uint8), np.zeros((ENC_N, 2, 8), np.uint8)
    ins = [dev.put(pe[:, 640:1920]), dev.put(po[:, 640:1920])]
    evs = [busy(s) for s in streams] if concurrent else []
    e.encode_device(ins[0], 2, dev.out(qe), cuda_stream=streams[0])
    o.encode_device(ins[1], 2, dev.out(qo), cuda_stream=streams[1])
    if concurrent:
        assert not any(ev.query() for ev in evs), "premise not met: the spin kernels ended before %s was called (lengthen BLOCK_CYCLES)" % x
    else:
        for s in streams:
            assert L.lpcnet_b200_stream_sync(s) == 0
    outs += ORDER_X[x](e, o)
    outs += [e.encode(pe[:, 1920:2560]), o.encode(po[:, 1920:2560])] + states(e) + states(o)
    dev.finish(streams)
    outs += [qe, qo]
    e.close(); o.close()
    return outs


@pytest.mark.parametrize("x", list(ORDER_X))
def test_calls_while_device_work_is_queued(eng, x):
    L = eng.lib()
    streams = [L.lpcnet_b200_stream_create() for _ in range(2)]
    assert all(streams)
    try:
        serial = order_run(eng, x, streams, False)
        got = order_run(eng, x, streams, True)
    finally:
        for s in streams:
            L.lpcnet_b200_stream_sync(s)
            L.lpcnet_b200_stream_destroy(s)
    assert_same(got, serial, "%s while encode_device calls are queued on both batches" % x)
    pcm = pcm_rows(2 * ENC_N, 20)
    want = H.oracle_encode(pcm[:, :1920])
    np.testing.assert_array_equal(got[-2], want[:ENC_N, 1:3], err_msg="the queued encode of e")
    np.testing.assert_array_equal(got[-1], want[ENC_N:, 1:3], err_msg="the queued encode of o")
