"""GPU tests (-m gpu) of the ordering promise of INTEGRATION.md ("Caller streams"): `_device` calls of a batch or an encoder batch
may use any CUDA stream and may be mixed with the host-pointer calls, and each call waits for the work the previous one enqueued
on the object's state.

  * Work that is provably still queued: a caller stream is held busy by a spin kernel (torch.cuda._sleep through an
    ExternalStream), a `_device` call is queued behind it, and every entry point that touches the state is called while the
    stream is still busy (each case asserts that premise).  The queued call's output and the entry point's own effect must equal
    the serial run, the same calls with a synchronise between them.  A few cases are checked against the CPU restatement too.
  * Several objects at once: batches of different models, encoder batches and drop-in states, each driven by its own host
    thread on its own caller stream (two threads share one), one thread making a call that fails.
  * The drop-in lifecycle on caller memory (lpcnet_init / lpcnet_decoder_init / lpcnet_encoder_init, init twice, deinit) and the
    LPCNET_B200_* defaults read once per process, in a child process."""
import ctypes
import os
import random
import subprocess
import sys
import threading
import types
import numpy as np
import pytest
import helpers as H
import scenarios as S
from fixtures import make_feature_batch, make_packets, make_pcm_batch

pytestmark = pytest.mark.gpu

BLOCK_CYCLES = 60_000_000        # the spin ahead of the queued call: 30-50 ms at H100 clocks, short on a shared GPU
TP, TQ, TX, TF = 3, 4, 2, 2      # synthesis frames: before the queued call, queued, used by the call under test, after it
PP, PQ, PX, PF = 2, 2, 1, 1      # packets, the same way (the host call before is as long as the queued one: no staging grows)
N_TWO_HALVES = 2200              # > 16 x 132 SMs: the automatic schedule steps each CTA's 32 slots as two halves
ENC_N = 8
E_PREP, E_Q, E_X, E_F = (0, 640), (640, 1920), (1920, 2560), (2560, 3200)     # encoder samples, the same way


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    L = lpcnet_b200.lib()
    L.lpcnet_encoder_create.restype = ctypes.c_void_p
    L.lpcnet_encoder_destroy.argtypes = [ctypes.c_void_p]
    for fn in ("lpcnet_encode", "lpcnet_compute_single_frame_features"):
        getattr(L, fn).argtypes = [ctypes.c_void_p] * 3
    return lpcnet_b200


@pytest.fixture
def stream(eng):
    L = eng.lib()
    s = L.lpcnet_b200_stream_create()
    assert s, L.lpcnet_b200_last_error()
    yield s
    L.lpcnet_b200_stream_sync(s)
    L.lpcnet_b200_stream_destroy(s)


def codebooks_b():
    """a second set of VQ codebooks, flattened like H.codebooks()"""
    import gen_model
    return np.ascontiguousarray(np.concatenate([a.ravel() for a in gen_model.make_codebooks(seed=97)]), dtype=np.float32)


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
    """device buffers of one run: uploads, and outputs copied back into their host arrays by finish() once the caller stream
    has drained; all freed there"""

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

    def finish(self, s):
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


# ---- 1 + 2: one state-touching call while a `_device` call is still queued on a caller stream -------------------------------
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
    b.set_pcm_sink(c.sink, 640, 0)
    return []


BATCH_X = {
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
    "destroy": lambda b, c: b.close() or [],
}
X_TWO_HALVES = ("set_codebooks", "reset_streams", "synthesize", "decode", "snapshot_restore", "destroy")


def batch_inputs(n):
    ids = range(400, 400 + n)
    return make_feature_batch(ids, TP + TQ + TX + TF), np.stack([make_packets(s, PP + PQ + PX + PF) for s in ids])


def batch_run(eng, kind, n, queued, x, s, concurrent):
    """prep call, `queued` (synth | decode) as a _device call on caller stream s, the call `x`, then calls that show the state x
    left.  concurrent: the queued call sits behind a spin kernel while x runs; else s is drained first.  Returns the outputs."""
    L = eng.lib()
    f, pk = batch_inputs(n)
    b = eng.Batch(n, H.blob(kind), config=H.model_config(), codebooks=H.codebooks())
    dev = Dev(L)
    c = types.SimpleNamespace(L=L, n=n, f=f, pk=pk, x0=TP + TQ, p0=PP + PQ, snap=None, sink=None)
    outs = []
    if x == "set_pcm_sink":
        c.sink = dev.out(np.zeros((n, 640), np.int16))
        outs.append(dev.reads[-1][1])
    q_pcm = np.zeros((n, TQ * 160 if queued == "synth" else PQ * 640), np.int16)
    d_in = dev.put(f[:, TP:TP + TQ] if queued == "synth" else pk[:, PP:PP + PQ])
    d_q = dev.out(q_pcm)
    outs += [b.synthesize(f[:, :TP]) if queued == "synth" else b.decode(pk[:, :PP]), q_pcm]
    if x == "snapshot_restore":
        c.snap = b.snapshot()
    ev = busy(s) if concurrent else None
    if queued == "synth":
        b.synthesize_device(d_in, TQ, 20, d_q, cuda_stream=s)
    else:
        b.decode_device(d_in, PQ, d_q, cuda_stream=s)
    if concurrent:
        assert_still_queued(ev, x)
    else:
        assert L.lpcnet_b200_stream_sync(s) == 0
    outs += BATCH_X[x](b, c)
    if x != "destroy":
        after = lambda: b.synthesize(f[:, TP + TQ + TX:]) if queued == "synth" else b.decode(pk[:, PP + PQ + PX:])
        outs += [after(), b.synthesize_tail(80)]
        if x == "snapshot_save":
            b.restore(c.snap)
            outs.append(after())
        if x == "set_pcm_sink":
            b.set_pcm_sink(None, 0, 0)
    dev.finish(s)               # (after a destroy: the caller's PCM buffer once its stream has drained)
    if c.snap:
        b.free_snapshot(c.snap)
    b.close()
    return outs


BATCH_CASES = [(kind, n, q, x) for kind, n in (("int8", 5), ("float", 6)) for q in ("synth", "decode") for x in BATCH_X]
BATCH_CASES += [("int8", N_TWO_HALVES, q, x) for q in ("synth", "decode") for x in X_TWO_HALVES]


@pytest.mark.parametrize("kind,n,queued,x", BATCH_CASES)
def test_batch_call_while_device_work_is_queued(eng, stream, kind, n, queued, x):
    """Batch entry point `x` called while a synthesize_device / decode_device is still queued behind other work on a caller
    stream: the queued call's PCM and everything x returns or leaves in the state equal the serial run."""
    serial = batch_run(eng, kind, n, queued, x, stream, False)
    got = batch_run(eng, kind, n, queued, x, stream, True)
    assert_same(got, serial, "%s %s, %s queued, then %s" % (kind, n, queued, x))
    if n > 16:
        return
    f, pk = batch_inputs(n)
    if queued == "synth" and x == "synthesize":
        np.testing.assert_array_equal(np.concatenate(got[:4], axis=1), H.oracle_synth(f, kind))
    if queued == "decode" and x == "decode":
        np.testing.assert_array_equal(np.concatenate(got[:4], axis=1), H.oracle_decode(pk, kind))
    if queued == "decode" and x == "set_codebooks":
        want = H.oracle_decode(pk, kind)
        np.testing.assert_array_equal(got[1], want[:, PP * 640:(PP + PQ) * 640], err_msg="the queued decode read the codebooks set after it")
        assert not np.array_equal(got[2], want[:, (PP + PQ + PX) * 640:]), "the second codebooks decode like the first: the case proves nothing"


def _enc_x_set_codebooks(e, c):
    cb = codebooks_b()
    assert c.L.lpcnet_b200_enc_set_codebooks(e._h, cb.ctypes.data, cb.size) == 0, c.L.lpcnet_b200_last_error()
    return []


ENC_X = {
    "set_codebooks": _enc_x_set_codebooks,
    "reset": lambda e, c: e.reset() or [],
    "compute_features": lambda e, c: [e.compute_features(c.pcm[:, E_X[0]:E_X[1]])],
    "encode": lambda e, c: [e.encode(c.pcm[:, E_X[0]:E_X[1]])],
    "compute_features4": lambda e, c: [e.compute_features4(c.pcm[:, E_X[0]:E_X[1]])],
    "destroy": lambda e, c: e.close() or [],
}


def enc_pcm():
    return make_pcm_batch(range(60, 60 + ENC_N), E_F[1] // 160)


def enc_run(eng, queued, x, s, concurrent):
    """as batch_run, on an encoder batch: `queued` is encode_device (encode) or compute_features_device (features)"""
    L = eng.lib()
    pcm = enc_pcm()
    e = eng.EncBatch(ENC_N, codebooks=H.codebooks())
    dev = Dev(L)
    c = types.SimpleNamespace(L=L, pcm=pcm)
    a, z = E_Q
    q_out = np.zeros((ENC_N, (z - a) // 640, 8), np.uint8) if queued == "encode" else np.zeros((ENC_N, (z - a) // 160, 36), np.float32)
    d_in, d_q = dev.put(pcm[:, a:z]), dev.out(q_out)
    prep = pcm[:, E_PREP[0]:E_PREP[1]]
    outs = [e.encode(prep) if queued == "encode" else e.compute_features(prep), q_out]
    ev = busy(s) if concurrent else None
    if queued == "encode":
        e.encode_device(d_in, q_out.shape[1], d_q, cuda_stream=s)
    else:
        e.compute_features_device(d_in, q_out.shape[1], d_q, cuda_stream=s)
    if concurrent:
        assert_still_queued(ev, x)
    else:
        assert L.lpcnet_b200_stream_sync(s) == 0
    outs += ENC_X[x](e, c)
    if x != "destroy":
        outs.append(e.encode(pcm[:, E_F[0]:E_F[1]]))
    dev.finish(s)
    e.close()
    return outs


@pytest.mark.parametrize("queued", ["encode", "features"])
@pytest.mark.parametrize("x", list(ENC_X))
def test_encoder_call_while_device_work_is_queued(eng, stream, queued, x):
    """EncBatch entry point `x` called while an encode_device / compute_features_device is still queued on a caller stream."""
    serial = enc_run(eng, queued, x, stream, False)
    got = enc_run(eng, queued, x, stream, True)
    assert_same(got, serial, "encoder, %s queued, then %s" % (queued, x))
    pcm = enc_pcm()
    if queued == "encode" and x == "encode":
        np.testing.assert_array_equal(np.concatenate(got, axis=1), H.oracle_encode(pcm))
    if queued == "encode" and x == "set_codebooks":
        want = H.oracle_encode(pcm)
        np.testing.assert_array_equal(got[1], want[:, 1:3], err_msg="the queued encode read the codebooks set after it")
        assert not np.array_equal(got[2], want[:, 4:5]), "the second codebooks encode like the first: the case proves nothing"
    if queued == "features" and x == "compute_features":
        np.testing.assert_array_equal(np.concatenate(got[:3], axis=1).view(np.uint32), H.oracle_features(pcm[:, :E_X[1]]).view(np.uint32))


# ---- 3: several objects at once, from several host threads and caller streams ---------------------------------------------
class OnStream:
    """A Batch for scenarios.run_engine_script whose synthesize / decode calls go, about half of them (seeded), through the
    `_device` entry points on caller stream `s`; their PCM arrives in the returned arrays at finish()."""

    def __init__(self, eng, b, s, seed):
        self.b, self.s, self.rng, self.dev = b, s, random.Random(seed), Dev(eng.lib())

    def __getattr__(self, name):
        return getattr(self.b, name)

    def synthesize(self, features, samples_per_frame=160, preload=0, pcm_in=None):
        if self.rng.random() < 0.5:
            return self.b.synthesize(features, samples_per_frame, preload, pcm_in)
        f = np.ascontiguousarray(features, dtype=np.float32)
        pcm = np.zeros((self.b.n, f.shape[1] * samples_per_frame), np.int16)
        if preload:
            pcm[:, :preload] = np.asarray(pcm_in)[:, :preload]
        self.b.synthesize_device(self.dev.put(f), f.shape[1], f.shape[2], self.dev.out(pcm), samples_per_frame=samples_per_frame,
                                 cuda_stream=self.s, preload=preload)
        return pcm

    def decode(self, packets):
        if self.rng.random() < 0.5:
            return self.b.decode(packets)
        p = np.ascontiguousarray(packets, dtype=np.uint8)
        pcm = np.zeros((self.b.n, p.shape[1] * 640), np.int16)
        self.b.decode_device(self.dev.put(p), p.shape[1], self.dev.out(pcm), cuda_stream=self.s)
        return pcm

    def finish(self):
        self.dev.finish(self.s)


CONCURRENT_MODELS = [("int8", "", 4), ("int8", "na256", 5), ("int8", "na128", 3), ("float", "", 6), ("int8", "na256e2e", 7)]


def enc_script(seed, samples):
    """seeded encoder calls (op, first sample, units) over `samples` samples of each stream"""
    rng = random.Random(seed)
    ops, a = [], 0
    while True:
        op = rng.choice(["encode", "encode", "features", "features", "features4", "reset"])
        k = rng.choice((1, 2, 3)) if op in ("encode", "features4") else rng.choice((1, 3, 4, 7))
        m = 0 if op == "reset" else k * (160 if op == "features" else 640)
        if a + m > samples:
            return ops
        ops.append((op, a, k)); a += m


def enc_script_run(eng, e, pcm, ops, s=None, seed=0):
    """the encoder script on `e`; with caller stream s about half of the encodes and frame analyses go through the `_device`
    entry points on s"""
    rng, dev, outs = random.Random(seed), Dev(eng.lib()), []
    for op, a, k in ops:
        if op == "reset":
            e.reset()
            continue
        seg = pcm[:, a:a + k * (160 if op == "features" else 640)]
        if s is not None and op != "features4" and rng.random() < 0.5:
            out = np.zeros((e.n, k, 8), np.uint8) if op == "encode" else np.zeros((e.n, k, 36), np.float32)
            (e.encode_device if op == "encode" else e.compute_features_device)(dev.put(seg), k, dev.out(out), cuda_stream=s)
            outs.append(out)
        else:
            outs.append({"encode": e.encode, "features": e.compute_features, "features4": e.compute_features4}[op](seg))
    if s is not None:
        dev.finish(s)
    return outs


def test_objects_run_concurrently_from_threads(eng):
    """Batches of five models, two encoder batches and a set of drop-in states, each driven by its own host thread on its own
    caller stream (the first two threads share one), run at the same time: every object's output equals its serial run bit for
    bit (the drop-in states equal the CPU restatement), and the one call that fails sets the error of its own thread only."""
    L = eng.lib()
    cb = H.codebooks()
    assert L.lpcnet_b200_set_default_codebooks(cb.ctypes.data, cb.size) == 0
    assert L.lpcnet_b200_set_default_model(H.blob("int8"), len(H.blob("int8")), H.LPC_GAMMA) == 0
    jobs, want = [], {}
    for i, (kind, tag, n) in enumerate(CONCURRENT_MODELS):
        ids = list(range(900 + 10 * i, 900 + 10 * i + n))
        script = S.random_script(8100 + i, n, n_ops=24, decode=True)
        f = make_feature_batch(ids, max(script[1], 1))
        make = lambda kind=kind, tag=tag, n=n: eng.Batch(n, H.blob(kind, tag), config=H.model_config(tag), codebooks=cb)
        b = make()
        want["batch%d" % i] = [S.run_engine_script(b, f, ids, script)]
        b.close()

        def job(s, make=make, f=f, ids=ids, script=script, i=i):
            b = make()
            if i == 2:                                       # the failing call
                with pytest.raises(eng.LPCNetB200Error):
                    b.synthesize_tail(0)
            o = OnStream(eng, b, s, 8200 + i)
            got = S.run_engine_script(o, f, ids, script, finish=o.finish)
            b.sync()
            b.close()
            return [got]
        jobs.append(("batch%d" % i, job))
    pcm = make_pcm_batch(range(80, 88), 40)
    for i, rows in enumerate((slice(0, 3), slice(3, 8))):
        ops = enc_script(8300 + i, pcm.shape[1])
        e = eng.EncBatch(rows.stop - rows.start, codebooks=cb)
        want["enc%d" % i] = enc_script_run(eng, e, pcm[rows], ops)
        e.close()

        def job(s, rows=rows, ops=ops, i=i):
            e = eng.EncBatch(rows.stop - rows.start, codebooks=cb)
            got = enc_script_run(eng, e, pcm[rows], ops, s, seed=8400 + i)
            e.close()
            return got
        jobs.append(("enc%d" % i, job))
    fa, ff = make_feature_batch([31], 8)[0], make_feature_batch([32], 8)[0]
    pk, epcm = make_packets(33, 2), make_pcm_batch([34], 8)[0]
    want["drop_in"] = [H.oracle_synth(fa[None], "int8")[0], H.oracle_synth(ff[None], "float")[0], H.oracle_decode(pk[None], "int8")[0],
                       H.oracle_features(epcm[None])[0]]

    def drop_in(s):
        """two synthesis states, a decoder and an encoder, interleaved frame by frame"""
        net_a, net_f, dec = eng.LPCNet(H.blob("int8")), eng.LPCNet(H.blob("float")), eng.LPCNetDecoder(H.blob("int8"))
        enc = L.lpcnet_encoder_create()
        assert enc
        a, fl, d, feat = [], [], [], np.zeros((8, 36), np.float32)
        for t in range(8):
            a.append(net_a.synthesize(fa[t]))
            if t % 4 == 0:
                d.append(dec.decode(pk[t // 4]))
            assert L.lpcnet_compute_single_frame_features(enc, epcm[t * 160:].ctypes.data, feat[t].ctypes.data) == 0
            fl.append(net_f.synthesize(ff[t]))
        for o in (net_a, net_f, dec):
            o.close()
        L.lpcnet_encoder_destroy(enc)
        return [np.concatenate(a), np.concatenate(fl), np.concatenate(d), feat]
    jobs.append(("drop_in", drop_in))

    streams = [L.lpcnet_b200_stream_create() for _ in range(len(jobs) - 1)]
    assert all(streams)
    lanes = [streams[0]] + streams                       # the first two jobs share a caller stream
    results, errors, last = {}, {}, {}
    start = threading.Barrier(len(jobs))

    def run(name, fn, s):
        try:
            start.wait()
            results[name] = fn(s)
        except BaseException as ex:                      # re-raised in the main thread below
            errors[name] = ex
        last[name] = (L.lpcnet_b200_last_error() or b"").decode()

    threads = [threading.Thread(target=run, args=(name, fn, s)) for (name, fn), s in zip(jobs, lanes)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for s in streams:
        L.lpcnet_b200_stream_destroy(s)
    for name, ex in errors.items():
        raise AssertionError("%s failed: %r" % (name, ex)) from ex
    for name, _ in jobs:
        assert_same(results[name], want[name], name)
        if name == "batch2":
            assert "synthesize_tail: bad arguments" in last[name], last[name]
        else:
            assert "synthesize_tail" not in last[name], "%s sees another thread's error: %s" % (name, last[name])


# ---- 4: drop-in lifecycle on caller memory, defaults from the environment ----------------------------------------------------
_CHILD = r"""
import ctypes, os, sys, numpy as np
sys.path[:0] = [%(root)r]
import lpcnet_b200
L = lpcnet_b200.lib()
c_p = ctypes.c_void_p
L.lpcnet_b200_deinit.argtypes = [c_p]
L.lpcnet_encoder_init.argtypes = [c_p]
L.lpcnet_encode.argtypes = [c_p] * 3
d = np.load(sys.argv[1])
f, pk, pcm = d["f"], d["pk"], d["pcm"]

def synth(mem):
    out = np.zeros((len(f), 160), np.int16)
    for t in range(len(f)):
        L.lpcnet_synthesize(ctypes.addressof(mem), f[t].ctypes.data, out[t].ctypes.data, 160)
    return out.ravel()

out = {}
mem = ctypes.create_string_buffer(L.lpcnet_get_size())
assert L.lpcnet_init(ctypes.addressof(mem)) == 0, L.lpcnet_b200_last_error()
out["first"] = synth(mem)
# read once per process: the values set now must change nothing
os.environ.update(LPCNET_B200_MODEL=sys.argv[3], LPCNET_B200_CODEBOOKS=sys.argv[4], LPCNET_B200_LPC_GAMMA="0.5")
assert L.lpcnet_init(ctypes.addressof(mem)) == 0       # init again on the same memory: the first batch is released
out["again"] = synth(mem)
L.lpcnet_b200_deinit(ctypes.addressof(mem))
out["after_deinit"] = synth(mem)
out["error"] = np.frombuffer(L.lpcnet_b200_last_error() or b"", np.uint8)
dmem = ctypes.create_string_buffer(L.lpcnet_decoder_get_size())
assert L.lpcnet_decoder_init(ctypes.addressof(dmem)) == 0
dec = np.zeros((len(pk), 640), np.int16)
for p in range(len(pk)):
    assert L.lpcnet_decode(ctypes.addressof(dmem), pk[p].ctypes.data, dec[p].ctypes.data) == 0, L.lpcnet_b200_last_error()
out["dec"] = dec.ravel()
L.lpcnet_b200_deinit(ctypes.addressof(dmem))
emem = ctypes.create_string_buffer(L.lpcnet_encoder_get_size())
assert L.lpcnet_encoder_init(ctypes.addressof(emem)) == 0
enc = np.zeros((len(pcm) // 640, 8), np.uint8)
for p in range(len(enc)):
    assert L.lpcnet_encode(ctypes.addressof(emem), pcm[p * 640:].ctypes.data, enc[p].ctypes.data) == 0, L.lpcnet_b200_last_error()
out["enc"] = enc
np.savez(sys.argv[2], **out)
print("child ok")
"""


def test_drop_in_init_on_caller_memory_and_defaults_read_once(eng, tmp_path):
    """lpcnet_get_size + lpcnet_init on caller memory, init again on the same memory, lpcnet_b200_deinit; lpcnet_decoder_init and
    lpcnet_encoder_init on caller memory; the model, codebooks and LPC gamma taken from LPCNET_B200_MODEL / _CODEBOOKS /
    _LPC_GAMMA, which are read once per process (a fresh one here).  Everything equals the CPU restatement."""
    f, pk, pcm = make_feature_batch([21], 6)[0], make_packets(22, 3), make_pcm_batch([23], 8)[0]
    np.savez(tmp_path / "in.npz", f=f, pk=pk, pcm=pcm)
    codebooks_b().tofile(tmp_path / "cb_b.bin")
    env = dict(os.environ, LPCNET_B200_MODEL=os.path.join(H.gen_dir(), "model_int8.bin"), LPCNET_B200_LPC_GAMMA=str(H.LPC_GAMMA),
               LPCNET_B200_CODEBOOKS=os.path.join(H.gen_dir(), "codebooks.bin"))
    r = subprocess.run([sys.executable, "-c", _CHILD % {"root": H.ROOT}, str(tmp_path / "in.npz"), str(tmp_path / "out.npz"),
                        os.path.join(H.gen_dir(), "model_float.bin"), str(tmp_path / "cb_b.bin")],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "child ok" in r.stdout, r.stdout + r.stderr
    got = np.load(tmp_path / "out.npz")
    want = H.oracle_synth(f[None], "int8")[0]
    np.testing.assert_array_equal(got["first"], want)
    np.testing.assert_array_equal(got["again"], want)
    assert not got["after_deinit"].any() and b"no model loaded" in got["error"].tobytes()
    np.testing.assert_array_equal(got["dec"], H.oracle_decode(pk[None], "int8")[0])
    np.testing.assert_array_equal(got["enc"], H.oracle_encode(pcm[None])[0])
