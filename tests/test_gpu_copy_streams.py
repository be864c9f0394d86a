"""GPU tests (-m gpu) of lpcnet_b200_batch_copy_streams: whole streams copied by value, on the device, from rows of one batch to rows
of another or the same batch (compaction, shard rebalancing, cloning).  Every comparison is bit for bit: a copied row must go on
exactly as its source row would have, against the source batch itself and against the CPU restatement; rows that were not listed
must go on exactly as on an untouched control batch."""
import numpy as np
import pytest
import helpers as H
import scenarios as S
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

BLOCK_CYCLES = 60_000_000        # the spin ahead of a queued call (as tests/test_gpu_ordering.py)


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
    """the automatic launch plan: no create-time knob left over from the environment"""
    for k in ("STREAMS_PER_CTA", "TWO_HALVES", "FLOAT_LANE_STREAM", "EXACT_CVT"):
        monkeypatch.delenv("LPCNET_B200_" + k, raising=False)


def batch(eng, n, kind="int8", tag="", device=0, config=None):
    return eng.Batch(n, H.blob(kind, tag), config=config or H.model_config(tag), codebooks=H.codebooks(), device=device)


def states(b, rows):
    """every row's exported blob and get_state fields, as one list of arrays"""
    out = []
    for r in rows:
        g = b.get_state(int(r))
        out += [b.export_state(int(r)), g["gru_a"], g["gru_b"], g["last_sig"], np.array([g["last_exc"], g["frame_count"]]), g["rng"]]
    return out


def assert_same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = np.ascontiguousarray(g), np.ascontiguousarray(w)
        assert g.shape == w.shape and g.dtype == w.dtype, "%s, item %d: %s %s vs %s %s" % (what, i, g.dtype, g.shape, w.dtype, w.shape)
        assert g.tobytes() == w.tobytes(), "%s, item %d differs first at element %s" % (what, i, tuple(np.argwhere(g.view(np.uint8) != w.view(np.uint8))[0]))


# ---- 1: compaction in the middle of a random call sequence ----------------------------------------------------------------------
def run_ops(b, ops, feats, pk, forced, k):
    """ops of a scenarios script on Batch b; row i reads feats[i], pk[i], forced[i]; k = the script's output offset at ops[0].
    Returns the list of outputs."""
    out = []
    for op in ops:
        kind = op[0]
        if kind == "synth":
            _, t, nf, N, pre = op
            out.append(b.synthesize(feats[:, t:t + nf], samples_per_frame=N, preload=pre, pcm_in=forced[:, k:k + max(pre, 1)])); k += nf * N
        elif kind == "decode":
            _, p, npk = op
            out.append(b.decode(pk[:, p:p + npk])); k += npk * 640
        elif kind == "net":
            b.run_frame_network(feats[:, op[1]:op[1] + op[2]])
        elif kind == "tail":
            _, N, pre = op
            out.append(b.synthesize_tail(N, preload=pre, pcm_in=forced[:, k:k + max(pre, 1)])); k += N
        elif kind == "defer":
            b.frame_network_deferred(feats[:, op[1]])
        elif kind == "flush":
            b.frame_network_flush()
        elif kind == "reset_signal":
            b.reset_signal()
        elif kind == "reset":
            b.reset()
        elif kind == "reset_streams":
            b.reset_streams(op[1])
        elif kind == "save":
            if getattr(b, "_snap", None):
                b.free_snapshot(b._snap)
            b._snap = b.snapshot()
        elif kind == "restore":
            b.restore(b._snap)
        elif kind == "move":
            b.import_state(op[2], b.export_state(op[1]))
        else:
            raise AssertionError(op)
    return out


def second_half(ops):
    """The ops after the copy, run on A and on B alike: row-wise operations only.  Moves name rows of A and snapshots belong to one
    batch, so they are left out, and so is a tail the engine would refuse without them (after a move, before the next frame-network
    run)."""
    keep, refused = [], False
    for op in ops:
        if op[0] in ("move", "save", "restore"):
            refused = refused or op[0] == "move"
            continue
        if op[0] in ("synth", "net", "decode", "reset"):
            refused = False
        if op[0] == "tail" and refused:
            continue
        keep.append(op)
    return keep


NA = 37                     # rows of A
NB_ROWS = 13                # rows of B
COMPACT = [("int8", ""), ("float", ""), ("int8", "na256"), ("float", "na128")]


@pytest.mark.parametrize("kind,tag", COMPACT, ids=["%s-%s" % (k, t or "na384") for k, t in COMPACT])
def test_compaction_mid_sequence(eng, auto, kind, tag):
    seed = 7100 + COMPACT.index((kind, tag))
    ops, T, signal, source = S.random_script(seed, NA, decode=True)
    h = len(ops) // 2
    P = max([op[1] + op[2] for op in ops if op[0] == "decode"], default=0)
    # the situations the copied rows must carry: decoder memory (a decode), a teacher-forced call, queued frames, and rows that are
    # back in their silent frames (reset after the queue was filled, so their queue is empty)
    silent = [3, 20, 36]
    extra = [("decode", P, 1), ("synth", T, 1, 160, 40), ("defer", T + 1), ("defer", T + 2), ("reset_streams", silent)]
    ops2 = second_half(ops[h:])
    ops1 = ops[:h] + extra
    full = (ops1 + ops2, T + 3, signal, source)
    streams = list(range(600, 600 + NA))
    f = make_feature_batch(streams, T + 3)
    pk = S.script_packets(full, streams)
    total = S.script_outputs(full)
    forced = np.stack([S.forced_pcm(signal, s, total) for s in streams])
    k1 = S.script_outputs((ops1, 0, signal))

    a = batch(eng, NA, kind, tag)
    out_a1 = run_ops(a, ops1, f, pk, forced, 0)
    # B: its own unrelated calls, which leave it accepting tails and with a queued frame of its own
    b = batch(eng, NB_ROWS, kind, tag)
    fb = make_feature_batch(range(950, 950 + NB_ROWS), 4)
    b.synthesize(fb[:, :3])
    b.frame_network_deferred(fb[:, 3])
    rng = np.random.default_rng(seed)
    src = np.array(silent[:2] + [int(r) for r in rng.choice([r for r in range(NA) if r not in silent], NB_ROWS - 2, replace=False)])
    dst = rng.permutation(NB_ROWS)
    b.copy_streams(dst, a, src)
    amap = np.empty(NB_ROWS, int)
    amap[dst] = src                                        # B row d continues A row amap[d]
    # the B rows hold (by construction) silent rows, and rows with queued frames, decoder memory, after a teacher-forced call
    assert set(silent[:2]) <= set(amap) and any(r not in silent for r in amap)
    # ops2 row-wise on both; reset_streams lists are mapped to B's rows
    inv = {int(s): d for d, s in enumerate(amap)}
    ops2_b = []
    for op in ops2:
        if op[0] == "reset_streams":
            ids = sorted(inv[s] for s in op[1] if s in inv)
            if ids:
                ops2_b.append(("reset_streams", ids))
        else:
            ops2_b.append(op)
    out_a2 = run_ops(a, ops2, f, pk, forced, k1)
    out_b2 = run_ops(b, ops2_b, f[amap], pk[amap] if pk is not None else None, forced[amap], k1)
    assert len(out_a2) == len(out_b2)
    assert_same([o[amap] for o in out_a2], out_b2, "PCM after the copy (seed %d)" % seed)
    a.frame_network_flush(); b.frame_network_flush()
    assert_same(states(a, amap), states(b, range(NB_ROWS)), "state after the copy")
    # A against the CPU restatement on the whole script, and hence B's rows too
    got = np.concatenate(out_a1 + out_a2, axis=1)
    want = S.run_streams("oracle", H.oracle_lib(), S.OracleState(kind, tag), f, streams, full)
    assert_same([got], [want], "A against the oracle")
    assert_same([np.concatenate(out_b2, axis=1)], [want[amap, k1:]], "B against the oracle")
    for x in (a, b):
        if hasattr(x, "_snap"):
            x.free_snapshot(x._snap)
        x.close()


# ---- 2: tails ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["int8", "float"])
def test_copied_rows_take_their_tail_conditioning_along(eng, auto, kind):
    a = batch(eng, 6, kind)
    fa = make_feature_batch(range(10, 16), 4)
    a.synthesize(fa[:, :2])
    fb = make_feature_batch(range(20, 25), 4)
    b, c = batch(eng, 5, kind), batch(eng, 5, kind)          # c: control, the same calls without the copy
    for x in (b, c):
        x.synthesize(fb[:, :3])
    b.copy_streams([0, 3], a, [4, 1])
    ta, tb, tc = a.synthesize_tail(160), b.synthesize_tail(160), c.synthesize_tail(160)
    assert_same([tb[[0, 3]], tb[[1, 2, 4]]], [ta[[4, 1]], tc[[1, 2, 4]]], "first tail")
    assert np.abs(tb).max() > 0
    # a flush moves the tail frame out of the chunk slots (with the copied rows in it)
    fm = np.stack([fa[4, 2], fb[1, 3], fb[2, 3], fa[1, 2], fb[4, 3]])
    a.frame_network_deferred(fa[:, 2]); b.frame_network_deferred(fm); c.frame_network_deferred(fb[:, 3])
    for x in (a, b, c):
        x.frame_network_flush()
    ta, tb, tc = a.synthesize_tail(80, preload=20, pcm_in=np.full((6, 20), 300)), b.synthesize_tail(80, preload=20, pcm_in=np.full((5, 20), 300)), \
        c.synthesize_tail(80, preload=20, pcm_in=np.full((5, 20), 300))
    assert_same([tb[[0, 3]], tb[[1, 2, 4]]], [ta[[4, 1]], tc[[1, 2, 4]]], "tail after a flush")
    for x in (a, b, c):
        x.close()


def test_tails_refused_after_a_copy_from_a_batch_that_refuses_them(eng, auto):
    f = make_feature_batch(range(30, 34), 4)
    a, b = batch(eng, 4), batch(eng, 4)
    for x in (a, b):
        x.synthesize(f[:, :2])
    a.import_state(2, a.export_state(0))             # a refuses tails now
    b.synthesize_tail(80)
    b.copy_streams([1], a, [3])
    for x in (a, b):
        with pytest.raises(eng.LPCNetB200Error, match="imported"):
            x.synthesize_tail(80)
    b.frame_network_deferred(f[:, 2])
    b.frame_network_flush()                          # a flush is not a frame-network run that a tail reads
    with pytest.raises(eng.LPCNetB200Error, match="imported"):
        b.synthesize_tail(80)
    b.run_frame_network(f[:, 3:4])
    assert b.synthesize_tail(80).shape == (4, 80)
    # the other way round: a destination that refuses tails keeps refusing them
    c = batch(eng, 4)
    c.synthesize(f[:, :1])
    a.copy_streams([0], c, [1])
    with pytest.raises(eng.LPCNetB200Error, match="imported"):
        a.synthesize_tail(80)
    for x in (a, b, c):
        x.close()


# ---- 3: inside one batch ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["int8", "float"])
def test_rotation_inside_one_batch(eng, auto, kind):
    n = 5
    f = make_feature_batch(range(50, 50 + n), 6)
    a, c = batch(eng, n, kind), batch(eng, n, kind)
    for x in (a, c):
        x.synthesize(f[:, :3])
        x.frame_network_deferred(f[:, 3])
        x.reset_streams([2])                          # row 2: no queued frame, back in its silent frames
    a.copy_streams([1, 2, 0], a, [0, 1, 2])
    rot = [2, 0, 1, 3, 4]                             # a row r continues c row rot[r]
    for x in (a, c):
        x.frame_network_flush()
    assert_same(states(a, range(n)), states(c, rot), "state after the rotation")
    assert_same([a.synthesize_tail(160)], [c.synthesize_tail(160)[rot]], "tail after the rotation")
    assert_same([a.synthesize(f[rot, 4:6])], [c.synthesize(f[:, 4:6])[rot]], "synthesis after the rotation")
    a.close(); c.close()


@pytest.mark.parametrize("kind", ["int8", "float"])
def test_clone_one_row_into_three(eng, auto, kind):
    n = 6
    f = make_feature_batch(range(60, 60 + n), 8)
    a = batch(eng, n, kind)
    a.synthesize(f[:, :3])
    a.frame_network_deferred(f[:, 3])
    a.copy_streams([1, 4, 5], a, [2, 2, 2])
    same = [2, 1, 4, 5]
    g = f.copy()
    g[same] = f[2]
    a.frame_network_flush()
    pk = np.stack([make_packets(r, 2) for r in range(n)])
    pk[same] = pk[2]
    outs = [a.synthesize_tail(100), a.synthesize(g[:, 4:7]), a.decode(pk)]
    for o in outs:
        assert all((o[r] == o[2]).all() for r in same), "clones diverge"
    assert np.abs(outs[1][2]).max() > 0
    ref = states(a, [2])
    for r in same[1:]:
        assert_same(states(a, [r]), ref, "clone %d state" % r)
    a.close()


# ---- 4: launch geometry -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [0, 1], ids=["16xSMs", "16xSMs+1"])
def test_destination_at_the_schedule_switch(eng, auto, sms, extra):
    """16 x SMs rows: the last one-half schedule; one more: two halves.  Copied rows land in both halves and in many CTAs."""
    n, ns = 16 * sms + extra, 64
    fa = make_feature_batch(range(ns), 5)
    fd = make_feature_batch(range(1000, 1000 + n), 5)
    a = batch(eng, ns)
    a.synthesize(fa[:, :3])
    d, c = batch(eng, n), batch(eng, n)
    for x in (d, c):
        x.synthesize(fd[:, :3])
    rows = np.unique(np.r_[0, 1, 15, 16, 17, 31, 32, n // 2, n // 2 + 1, n - 17, n - 16, n - 2, n - 1,
                           np.random.default_rng(n).choice(n, 24, replace=False)])
    src = np.random.default_rng(n + 1).choice(ns, rows.size, replace=True)
    d.copy_streams(rows, a, src)
    g = fd.copy()
    g[rows] = fa[src]
    out_d, out_a, out_c = d.synthesize(g[:, 3:5]), a.synthesize(fa[:, 3:5]), c.synthesize(fd[:, 3:5])
    others = np.setdiff1d(np.arange(n), rows)
    assert_same([out_d[rows], out_d[others]], [out_a[src], out_c[others]], "after the copy")
    for x in (a, d, c):
        x.close()


def test_permutation_of_4096_rows_onto_themselves(eng, auto):
    n = 4096
    f = make_feature_batch(range(n), 4)
    a, c = batch(eng, n), batch(eng, n)
    for x in (a, c):
        x.synthesize(f[:, :2])
    perm = np.random.default_rng(4096).permutation(n)
    a.copy_streams(np.arange(n), a, perm)             # a row k continues c row perm[k]
    assert_same([a.synthesize(f[perm, 2:4])], [c.synthesize(f[:, 2:4])[perm]], "after the permutation")
    for r in (0, 1, 2047, 4095):
        assert_same(states(a, [r]), states(c, [perm[r]]), "row %d" % r)
    a.close(); c.close()


# ---- 5: ordering with `_device` work still queued ---------------------------------------------------------------------------------
def busy(s, cycles=BLOCK_CYCLES):
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(s)):
        torch.cuda._sleep(cycles)
        ev = torch.cuda.Event()
        ev.record()
    return ev


class Dev:
    def __init__(self, L):
        self.L, self.ptrs = L, []

    def put(self, a):
        a = np.ascontiguousarray(a)
        p = self.L.lpcnet_b200_device_alloc(a.nbytes)
        assert p and self.L.lpcnet_b200_memcpy_h2d(p, a.ctypes.data, a.nbytes) == 0
        self.ptrs.append(p)
        return p

    def get(self, p, like):
        out = np.empty_like(like)
        assert self.L.lpcnet_b200_memcpy_d2h(out.ctypes.data, p, out.nbytes) == 0
        return out

    def free(self):
        for p in self.ptrs:
            self.L.lpcnet_b200_device_free(p)


@pytest.mark.parametrize("kind", ["int8", "float"])
def test_copy_waits_for_device_calls_queued_on_both_batches(eng, auto, kind):
    L = eng.lib()
    n_a, n_b, T = 9, 7, 3
    fa, fb = make_feature_batch(range(70, 70 + n_a), 2 * T), make_feature_batch(range(80, 80 + n_b), 2 * T)
    src, dst = [8, 0, 4], [6, 0, 3]

    def run(queued):
        a, b = batch(eng, n_a, kind), batch(eng, n_b, kind)
        d = Dev(L)
        s1, s2 = L.lpcnet_b200_stream_create(), L.lpcnet_b200_stream_create()
        pa, pb = np.zeros((n_a, T * 160), np.int16), np.zeros((n_b, T * 160), np.int16)
        xa, xb = d.put(np.ascontiguousarray(fa[:, :T])), d.put(np.ascontiguousarray(fb[:, :T]))
        ya, yb = d.put(pa), d.put(pb)
        if queued:
            ev1, ev2 = busy(s1), busy(s2)
        a.synthesize_device(xa, T, fa.shape[2], ya, cuda_stream=s1)
        b.synthesize_device(xb, T, fb.shape[2], yb, cuda_stream=s2)
        if queued:
            assert not ev1.query() and not ev2.query(), "premise not met: the spins had ended before the copy (lengthen BLOCK_CYCLES)"
        else:
            L.lpcnet_b200_stream_sync(s1); L.lpcnet_b200_stream_sync(s2)
        b.copy_streams(dst, a, src)
        out = [d.get(ya, pa), d.get(yb, pb)]
        g = fb.copy()
        g[dst] = fa[src]
        out += [a.synthesize(fa[:, T:]), b.synthesize(g[:, T:])] + states(b, range(n_b))
        L.lpcnet_b200_stream_sync(s1); L.lpcnet_b200_stream_sync(s2)
        L.lpcnet_b200_stream_destroy(s1); L.lpcnet_b200_stream_destroy(s2)
        d.free(); a.close(); b.close()
        return out

    want = run(False)
    assert_same(run(True), want, "copy behind queued _device calls")
    assert_same([want[3][dst]], [want[2][src]], "copied rows continue their source rows")


# ---- 6: groups ----------------------------------------------------------------------------------------------------------------------
def test_copy_into_a_group_member_between_group_calls(eng, auto):
    n1, n2, ns = 11, 6, 5
    f = make_feature_batch(range(100, 100 + n1 + n2), 6)
    fs = make_feature_batch(range(200, 200 + ns), 6)
    s = batch(eng, ns)
    s.synthesize(fs[:, :2])
    m1, m2, t1, t2 = batch(eng, n1), batch(eng, n2), batch(eng, n1), batch(eng, n2)
    g = eng.Group([m1, m2])
    out_g = [g.synthesize(f[:, :2])]
    out_t = [np.concatenate([t1.synthesize(f[:n1, :2]), t2.synthesize(f[n1:, :2])])]
    for x in (m2, t2):
        x.copy_streams([0, 5], s, [3, 1])
    h = f.copy()
    h[n1 + np.array([0, 5])] = fs[[3, 1]]
    out_g.append(g.synthesize(h[:, 2:5]))
    out_t.append(np.concatenate([t1.synthesize(h[:n1, 2:5]), t2.synthesize(h[n1:, 2:5])]))
    assert_same(out_g + states(m2, range(n2)), out_t + states(t2, range(n2)), "group call after a copy into a member")
    assert_same([out_g[1][n1 + np.array([0, 5])]], [s.synthesize(fs[:, 2:5])[[3, 1]]], "copied rows continue their source rows")
    g.close()
    for x in (s, m1, m2, t1, t2):
        x.close()


# ---- 7: across devices ---------------------------------------------------------------------------------------------------------------
def _need2(eng):
    if eng.device_count() < 2:
        pytest.skip("needs two CUDA devices (%d visible)" % eng.device_count())


@pytest.mark.parametrize("kind", ["int8", "float"])
def test_copy_between_devices(eng, auto, kind):
    _need2(eng)
    f0, f1 = make_feature_batch(range(300, 308), 5), make_feature_batch(range(400, 406), 5)
    a, b, c = batch(eng, 8, kind, device=0), batch(eng, 6, kind, device=1), batch(eng, 6, kind, device=1)
    a.synthesize(f0[:, :2])
    for x in (b, c):
        x.synthesize(f1[:, :2])
        x.frame_network_deferred(f1[:, 2])
    a.frame_network_deferred(f0[:, 2])
    b.copy_streams([5, 2], a, [0, 7])
    g = f1.copy()
    g[[5, 2]] = f0[[0, 7]]
    for x in (a, b, c):
        x.frame_network_flush()
    ta, tb, tc = a.synthesize_tail(80), b.synthesize_tail(80), c.synthesize_tail(80)
    oa, ob, oc = a.synthesize(f0[:, 3:5]), b.synthesize(g[:, 3:5]), c.synthesize(f1[:, 3:5])
    assert_same([tb[[5, 2]], ob[[5, 2]], tb[[0, 1, 3, 4]], ob[[0, 1, 3, 4]]], [ta[[0, 7]], oa[[0, 7]], tc[[0, 1, 3, 4]], oc[[0, 1, 3, 4]]], "device 0 -> 1")
    a.copy_streams([1], b, [3])                       # and back
    assert_same(states(a, [1]), states(b, [3]), "device 1 -> 0")
    for x in (a, b, c):
        x.close()


class _Shard:
    """a Multi shard's batch, for Batch.copy_streams (the Multi owns it)"""
    def __init__(self, m, k):
        self._L = m._L
        self._h = m._L.lpcnet_b200_multi_batch(m._h, k)
        assert self._h


def test_rebalance_shards_of_a_multi(eng, auto):
    _need2(eng)
    n = 10
    f = make_feature_batch(range(500, 500 + n), 6)
    m = eng.Multi(n, H.blob("int8"), [0, 1], config=H.model_config(""))
    one = batch(eng, n)
    m.synthesize(f[:, :3]); one.synthesize(f[:, :3])
    (_, f0, c0), (_, f1, c1) = m.shard(0), m.shard(1)
    src, dst = [1, 4], [0, 2]                         # shard 0 local rows -> shard 1 local rows
    eng.Batch.copy_streams(_Shard(m, 1), dst, _Shard(m, 0), src)
    one.copy_streams([f1 + r for r in dst], one, [f0 + r for r in src])
    g = f.copy()
    g[[f1 + r for r in dst]] = f[[f0 + r for r in src]]
    assert_same([m.synthesize(g[:, 3:6])], [one.synthesize(g[:, 3:6])], "multi after the rebalance")
    m.close(); one.close()


# ---- 8: refusals -------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(eng, auto):
    L = eng.lib()
    f = make_feature_batch(range(700, 706), 3)
    base = H.model_config("")
    a, b = batch(eng, 6), batch(eng, 4)
    a.synthesize(f[:, :2]); b.synthesize(f[:4, 1:3])
    before = states(a, range(6)) + states(b, range(4))
    others = {
        "GRU_A size": batch(eng, 4, "int8", "na256"),
        "flavour": batch(eng, 4, "float"),
        "FEATURES_DELAY": batch(eng, 4, config=(base[0], 1, base[2])),
        "END2END": batch(eng, 4, config=(base[0], base[1], 1)),
        "LPC_GAMMA": batch(eng, 4, config=(1.0, base[1], base[2])),
    }
    for what, o in others.items():
        for d, s in ((a, o), (o, a)):
            with pytest.raises(eng.LPCNetB200Error):
                d.copy_streams([0], s, [0])
        o.close()
    bad = [([6], [0]), ([-1], [0]), ([0], [4]), ([0], [-1]), ([0, 0], [1, 2]), ([2, 3, 2], [0, 1, 2])]
    for dr, sr in bad:
        with pytest.raises(eng.LPCNetB200Error):
            a.copy_streams(dr, b, sr)
    with pytest.raises(eng.LPCNetB200Error):
        a.copy_streams([0, 0], a, [1, 2])
    rows = np.zeros(1, np.int32)
    for args in ((None, rows.ctypes.data, b._h, rows.ctypes.data, 1), (a._h, None, b._h, rows.ctypes.data, 1),
                 (a._h, rows.ctypes.data, None, rows.ctypes.data, 1), (a._h, rows.ctypes.data, b._h, None, 1),
                 (a._h, rows.ctypes.data, b._h, rows.ctypes.data, -1)):
        assert L.lpcnet_b200_batch_copy_streams(*args) == -1
        assert L.lpcnet_b200_last_error()
    a.copy_streams([], b, [])                         # count == 0: nothing to do
    assert_same(states(a, range(6)) + states(b, range(4)), before, "after the refusals")
    a.synthesize_tail(40); b.synthesize_tail(40)      # both still accept tails
    a.close(); b.close()
