"""GPU tests (-m gpu) of the call order of groups (INTEGRATION.md, "Groups"): group calls take part in each member's call order,
so a group `_device` call may use any CUDA stream and may be mixed with member calls, other group calls and the group's
lifecycle calls, and each call waits for the work the previous one enqueued on a member's state.

  * Work that is provably still queued: a caller stream is held busy by a spin kernel (torch.cuda._sleep through an
    ExternalStream), a group synthesize_device / decode_device is queued behind it, and then, while the stream is still busy
    (each case asserts that premise), one call is made: a member entry point on member 0, a group host call, a second group
    `_device` call on another stream, last_sample_kernel_ms, or group_destroy (after which the members carry on alone).  The
    queued call's PCM, what the call returns and everything after it (PCM, tails, every stream's exported state) must equal
    the serial run, the same calls with a synchronise between them.  At 384 units with automatic geometry, and for a subset
    of the calls at 256 units at a pinned two-half spc.
  * Two groups sharing a member: `_device` calls of {A, B} and {A, C} alternate on two caller streams with member calls in
    between; every member's PCM and state equal its own calls made in the same order."""
import types
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets

pytestmark = pytest.mark.gpu

BLOCK_CYCLES = 60_000_000        # the spin ahead of the queued call: 30-50 ms at H100 clocks, short on a shared GPU
TP, TQ, TX, TF = 3, 4, 2, 2      # synthesis frames: before the queued call, queued, used by the call under test, after it
PP, PQ, PX, PF = 2, 2, 1, 1      # packets, the same way
KNOBS = ("STREAMS_PER_CTA", "TWO_HALVES", "EXACT_CVT", "FCW_NODES")
TAGS = {384: "", 256: "na256", 128: "na128"}
SIZES = (3, 4)                   # member 0 (default blob), member 1 (a seeded blob)


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


@pytest.fixture
def streams(eng):
    """two caller streams"""
    L = eng.lib()
    ss = [L.lpcnet_b200_stream_create() for _ in range(2)]
    assert all(ss), L.lpcnet_b200_last_error()
    yield ss
    for s in ss:
        L.lpcnet_b200_stream_sync(s)
        L.lpcnet_b200_stream_destroy(s)


_SEEDED = {}


def seeded_blob(seed, na):
    import gen_model
    from lpcnet_b200 import api
    key = (seed, na)
    if key not in _SEEDED:
        common, only8, _ = gen_model.make_model(seed, na=None if na == 384 else na)
        _SEEDED[key] = api.write_blob([(n, t, a.tobytes()) for n, t, a in common + only8])
    return _SEEDED[key]


def codebooks_b():
    """a second set of VQ codebooks, flattened like H.codebooks()"""
    import gen_model
    return np.ascontiguousarray(np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=98)]), dtype=np.float32)


def busy(s, cycles=BLOCK_CYCLES):
    """enqueue a spin kernel on caller stream `s`; returns an event recorded right after it: while the event has not
    completed, nothing enqueued on `s` after busy() has started"""
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(s)):
        torch.cuda._sleep(cycles)
        ev = torch.cuda.Event()
        ev.record()
    return ev


def assert_still_queued(ev, what):
    assert not ev.query(), ("premise not met: the spin ahead of the queued call had already ended when %s was called, so this "
                            "run says nothing about ordering (lengthen BLOCK_CYCLES)" % what)


class Dev:
    """device buffers of one run: uploads, and outputs copied back into their host arrays by finish() once the caller streams
    have drained; all freed there"""

    def __init__(self, L):
        self.L, self.ptrs, self.reads = L, [], []

    def put(self, a):
        a = np.ascontiguousarray(a)
        p = self.L.lpcnet_b200_device_alloc(a.nbytes)
        assert p, self.L.lpcnet_b200_last_error()
        assert self.L.lpcnet_b200_memcpy_h2d(p, a.ctypes.data, a.nbytes) == 0
        self.ptrs.append(p)
        return p

    def out(self, host):
        p = self.put(host)
        self.reads.append((p, host))
        return p

    def finish(self, *ss):
        for s in ss:
            assert self.L.lpcnet_b200_stream_sync(s) == 0, self.L.lpcnet_b200_last_error()
        for p, h in self.reads:
            assert self.L.lpcnet_b200_memcpy_d2h(h.ctypes.data, p, h.nbytes) == 0
        for p in self.ptrs:
            self.L.lpcnet_b200_device_free(p)
        self.ptrs, self.reads = [], []


def assert_same(got, want, what):
    """bit-for-bit equality of two lists of arrays"""
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = np.ascontiguousarray(g), np.ascontiguousarray(w)
        assert g.shape == w.shape and g.dtype == w.dtype, "%s, output %d: %s %s vs %s %s" % (what, i, g.dtype, g.shape, w.dtype, w.shape)
        d = np.argwhere(g.view(np.uint8).reshape(g.shape[0], -1) != w.view(np.uint8).reshape(w.shape[0], -1)) if g.ndim else []
        assert len(d) == 0, "%s, output %d: differs first at row %d byte %d" % (what, i, d[0][0], d[0][1])


# ---- 1: one call while a group `_device` call is still queued on a caller stream ---------------------------------------------
def _x_set_codebooks(b, c):
    cb = codebooks_b()
    assert c.L.lpcnet_b200_batch_set_codebooks(b._h, cb.ctypes.data, cb.size) == 0, c.L.lpcnet_b200_last_error()
    return []


def _x_get_state(b, c):
    st = b.get_state(c.n - 1)
    return [st["gru_a"], st["gru_b"], st["last_sig"], np.array([st["last_exc"], st["frame_count"]]), st["rng"]]


def _x_export_import(b, c):
    blob = b.export_state(1)
    b.import_state(0, blob)
    return [blob]


def _x_deferred_flush(b, c):
    b.frame_network_deferred(c.f[:, c.x0])
    b.frame_network_deferred(c.f[:, c.x0 + 1])
    b.frame_network_flush()
    return []


def _x_snapshot_save(b, c):
    c.snap = b.snapshot()
    return []


def _x_set_pcm_sink(b, c):
    """a sink set, one member call forwarded to it, the sink taken away again (a group refuses members with a sink)"""
    b.set_pcm_sink(c.sink, TX * 160, 0)
    out = b.synthesize(c.f[:, c.x0:c.x0 + TX])
    b.set_pcm_sink(None, 0, 0)
    return [out]


def _x_destroy(b, c):
    """the group first (it must not outlive its members), then the member"""
    c.g.close()
    b.close()
    return []


def _x_group_host(b, c):
    return [c.g.synthesize(c.f_all[:, c.x0:c.x0 + TX]) if c.queued == "synth" else c.g.decode(c.pk_all[:, c.p0:c.p0 + PX])]


def _x_group_device_other_stream(b, c):
    if c.queued == "synth":
        pcm = np.zeros((c.g.n, TX * 160), np.int16)
        c.g.synthesize_device(c.dev.put(c.f_all[:, c.x0:c.x0 + TX]), TX, 20, c.dev.out(pcm), 160, c.s2)
    else:
        pcm = np.zeros((c.g.n, PX * 640), np.int16)
        c.g.decode_device(c.dev.put(c.pk_all[:, c.p0:c.p0 + PX]), PX, c.dev.out(pcm), c.s2)
    return [pcm]


def _x_group_ms(b, c):
    ms, launches = c.g.last_sample_kernel_ms()
    assert ms > 0, "the queued group call's per-sample launches took %r ms" % ms
    return [np.array([launches])]


def _x_group_destroy(b, c):
    c.g.close()
    return []


X = {
    "set_codebooks": _x_set_codebooks,
    "reset": lambda b, c: b.reset() or [],
    "reset_streams": lambda b, c: b.reset_streams([0, c.n - 1]) or [],
    "reset_signal": lambda b, c: b.reset_signal() or [],
    "synthesize": lambda b, c: [b.synthesize(c.f[:, c.x0:c.x0 + TX])],
    "decode": lambda b, c: [b.decode(c.pk[:, c.p0:c.p0 + PX])],
    "run_frame_network": lambda b, c: b.run_frame_network(c.f[:, c.x0:c.x0 + TX]) or [],
    "synthesize_tail": lambda b, c: [b.synthesize_tail(80)],
    "deferred_flush": _x_deferred_flush,
    "export_import": _x_export_import,
    "snapshot_save": _x_snapshot_save,
    "snapshot_restore": lambda b, c: b.restore(c.snap) or [],
    "get_state": _x_get_state,
    "set_pcm_sink": _x_set_pcm_sink,
    "destroy": _x_destroy,
    "group_host": _x_group_host,
    "group_device_other_stream": _x_group_device_other_stream,
    "group_last_sample_kernel_ms": _x_group_ms,
    "group_destroy": _x_group_destroy,
}
X_TWO_HALVES = ("set_codebooks", "reset_streams", "synthesize", "decode", "snapshot_restore", "destroy", "group_host",
                "group_device_other_stream", "group_destroy")


def group_inputs(n):
    ids = range(500, 500 + n)
    return make_feature_batch(ids, TP + TQ + TX + TF), np.stack([make_packets(s, PP + PQ + PX + PF) for s in ids])


def make_members(eng, na):
    tag = TAGS[na]
    blobs = [H.blob("int8", tag), seeded_blob(3301, na)]
    return [eng.Batch(n, b, config=H.model_config(tag), codebooks=H.codebooks()) for b, n in zip(blobs, SIZES)]


def group_run(eng, mp, na, spc, queued, x, ss, concurrent):
    """group call, `queued` (synth | decode) as a group `_device` call on caller stream ss[0], the call `x` (on member 0 for a
    member entry point), then a group call (or, once the group is gone, member calls), tails and every stream's state.
    concurrent: the queued call sits behind a spin kernel while x runs; else ss[0] is drained first.  Returns the outputs."""
    L = eng.lib()
    s, s2 = ss
    bs = make_members(eng, na)
    if spc:
        mp.setenv("LPCNET_B200_STREAMS_PER_CTA", str(spc))
    g = eng.Group(bs)
    mp.delenv("LPCNET_B200_STREAMS_PER_CTA", raising=False)
    f, pk = group_inputs(g.n)
    a = bs[0]
    dev = Dev(L)
    c = types.SimpleNamespace(L=L, n=a.n, f=f[:a.n], pk=pk[:a.n], f_all=f, pk_all=pk, x0=TP + TQ, p0=PP + PQ, snap=None, sink=None,
                              g=g, s2=s2, dev=dev, queued=queued)
    outs = []
    if x == "set_pcm_sink":
        c.sink = dev.out(np.zeros((a.n, TX * 160), np.int16))
        outs.append(dev.reads[-1][1])
    q_pcm = np.zeros((g.n, TQ * 160 if queued == "synth" else PQ * 640), np.int16)
    d_in = dev.put(f[:, TP:TP + TQ] if queued == "synth" else pk[:, PP:PP + PQ])
    d_q = dev.out(q_pcm)
    outs += [g.synthesize(f[:, :TP]) if queued == "synth" else g.decode(pk[:, :PP]), q_pcm]
    if x == "snapshot_restore":
        c.snap = a.snapshot()
    ev = busy(s) if concurrent else None
    if queued == "synth":
        g.synthesize_device(d_in, TQ, 20, d_q, 160, s)
    else:
        g.decode_device(d_in, PQ, d_q, s)
    if concurrent:
        assert_still_queued(ev, x)
    else:
        assert L.lpcnet_b200_stream_sync(s) == 0
    outs += X[x](a, c)
    live = bs[1:] if x == "destroy" else bs
    rest = (f[:, TP + TQ + TX:], pk[:, PP + PQ + PX:])
    rows = np.cumsum([0] + [b.n for b in bs])

    def after():
        if x in ("destroy", "group_destroy"):        # the members carry on alone
            k0 = 1 if x == "destroy" else 0
            return [b.synthesize(rest[0][rows[k]:rows[k + 1]]) if queued == "synth" else b.decode(rest[1][rows[k]:rows[k + 1]])
                    for k, b in enumerate(bs) if k >= k0]
        return [g.synthesize(rest[0]) if queued == "synth" else g.decode(rest[1])]
    outs += after()
    outs += [b.synthesize_tail(80) for b in live]
    if x == "snapshot_save":
        a.restore(c.snap)
        outs += after()
    outs += [b.export_state(t) for b in live for t in range(b.n)]
    dev.finish(s, s2)
    if c.snap:
        a.free_snapshot(c.snap)
    g.close()
    for b in live:
        b.close()
    return outs


CASES = [(384, None, q, x) for q in ("synth", "decode") for x in X]
CASES += [(256, 17, q, x) for q in ("synth", "decode") for x in X_TWO_HALVES]


@pytest.mark.parametrize("na,spc,queued,x", [pytest.param(*c, id="na%d-%s-%s-%s" % (c[0], "spc%d" % c[1] if c[1] else "auto", c[2], c[3]))
                                             for c in CASES])
def test_call_while_group_device_work_is_queued(eng, clean_env, streams, na, spc, queued, x):
    """entry point `x` called while a group synthesize_device / decode_device is still queued behind other work on a caller
    stream: the queued call's PCM and everything x returns or leaves in the members equal the serial run"""
    serial = group_run(eng, clean_env, na, spc, queued, x, streams, False)
    got = group_run(eng, clean_env, na, spc, queued, x, streams, True)
    assert_same(got, serial, "na%d, group %s queued, then %s" % (na, queued, x))
    if queued == "synth" and x == "synthesize":
        f, _ = group_inputs(sum(SIZES))
        n0 = SIZES[0]
        a = np.concatenate([got[0][:n0], got[1][:n0], got[2], got[3][:n0]], axis=1)
        b = np.concatenate([got[0][n0:], got[1][n0:], got[3][n0:]], axis=1)
        tag = TAGS[na]
        np.testing.assert_array_equal(a, H.oracle_synth(f[:n0], "int8", tag=tag))
        fb = np.concatenate([f[n0:, :TP + TQ], f[n0:, TP + TQ + TX:]], axis=1)
        np.testing.assert_array_equal(b, H.oracle_synth(fb, "int8", tag=tag, model_blob=seeded_blob(3301, na)))
    if queued == "decode" and x == "set_codebooks":
        _, pk = group_inputs(sum(SIZES))
        want = H.oracle_decode(pk[:SIZES[0]], "int8", tag=TAGS[na])
        np.testing.assert_array_equal(got[1][:SIZES[0]], want[:, PP * 640:(PP + PQ) * 640],
                                      err_msg="the queued group decode read the codebooks set after it")


# ---- 2: two groups sharing a member -------------------------------------------------------------------------------------------
def test_two_groups_sharing_a_member(eng, clean_env, streams):
    """groups {A, B} and {A, C}: `_device` calls alternate on two caller streams (the first behind a spin kernel), with member
    calls of A and a group host call in between; each member's PCM and state equal its own calls made in the same order"""
    L = eng.lib()
    s1, s2 = streams
    cfg = H.model_config("")
    blobs = [H.blob("int8"), seeded_blob(3302, 384), seeded_blob(3303, 384)]
    ns = (3, 5, 2)
    side = {w: [eng.Batch(n, b, config=cfg, codebooks=H.codebooks()) for b, n in zip(blobs, ns)] for w in ("g", "r")}
    A, B, C = side["g"]
    AB, AC = eng.Group([A, B]), eng.Group([A, C])
    fs = [make_feature_batch(range(600 + 20 * i, 600 + 20 * i + 8), 5) for i in range(5)]
    pk = np.stack([make_packets(650 + s, 2) for s in range(8)])
    dev = Dev(L)
    ab, ac = (lambda a: a[:8]), (lambda a: a[:5])          # group rows: A's 3, then B's 5 or C's 2
    out = {}

    def synth_dev(grp, rows, f, s, key):
        out[key] = np.zeros((grp.n, f.shape[1] * 160), np.int16)
        grp.synthesize_device(dev.put(rows(f)), f.shape[1], 20, dev.out(out[key]), 160, s)

    ev = busy(s1)
    synth_dev(AB, ab, fs[0], s1, "ab0")
    assert_still_queued(ev, "the second group's call")
    A.reset_streams([1])
    synth_dev(AC, ac, fs[1], s2, "ac1")
    out["a2"] = A.synthesize(fs[2][:3])
    out["ab3"] = np.zeros((AB.n, 2 * 640), np.int16)
    AB.decode_device(dev.put(ab(pk)), 2, dev.out(out["ab3"]), s2)
    synth_dev(AC, ac, fs[3], s1, "ac4")
    out["ac5"] = AC.synthesize(ac(fs[4]))
    dev.finish(s1, s2)
    AB.close()
    AC.close()

    Ar, Br, Cr = side["r"]
    want = {}
    want["ab0"] = np.concatenate([Ar.synthesize(fs[0][:3]), Br.synthesize(fs[0][3:8])])
    Ar.reset_streams([1])
    want["ac1"] = np.concatenate([Ar.synthesize(fs[1][:3]), Cr.synthesize(fs[1][3:5])])
    want["a2"] = Ar.synthesize(fs[2][:3])
    want["ab3"] = np.concatenate([Ar.decode(pk[:3]), Br.decode(pk[3:8])])
    want["ac4"] = np.concatenate([Ar.synthesize(fs[3][:3]), Cr.synthesize(fs[3][3:5])])
    want["ac5"] = np.concatenate([Ar.synthesize(fs[4][:3]), Cr.synthesize(fs[4][3:5])])
    for k in want:
        assert_same([out[k]], [want[k]], "call %s" % k)
    for g, r in zip(side["g"], side["r"]):
        assert_same([g.export_state(t) for t in range(g.n)], [r.export_state(t) for t in range(r.n)], "member state")
        assert_same([g.synthesize_tail(80)], [r.synthesize_tail(80)], "member tail")
    # the first calls start from fresh states: the oracle's
    np.testing.assert_array_equal(out["ab0"][:3], H.oracle_synth(fs[0][:3], "int8"))
    np.testing.assert_array_equal(out["ab0"][3:], H.oracle_synth(fs[0][3:8], "int8", model_blob=blobs[1]))
    for b in side["g"] + side["r"]:
        b.close()
