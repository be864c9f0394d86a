"""Call sequences over the reference's INTERNAL synthesis entry points (lpcnet_private.h:125-133: lpcnet_synthesize_impl with
`preload`, run_frame_network + lpcnet_synthesize_tail_impl, run_frame_network_deferred/_flush, lpcnet_reset_signal, state copies)
— what the reference's PLC does around the hot path (src/lpcnet_plc.c:188-503) — expressed once and run on three back ends:
the compiled reference (oracle/_ref, single stream), the CPU restatement (oracle port, single stream) and the CUDA engine
(a batch of streams).  TEST INFRASTRUCTURE."""
import ctypes
import functools
import numpy as np
import helpers as H


def plc_like_script(T):
    """(op, args) list over feature frames 0..T-1; every op consumes at most one frame index."""
    s = [("synth", t, 160, 0) for t in range(5)]                 # normal frames
    s += [("synth", 5, 160, 40)]                                 # lpcnet_synthesize_impl(..., preload=40): teacher-forced head
    s += [("net", 6), ("tail", 80, 0), ("tail", 80, 0)]           # run_frame_network + two half-frame tails (PLC uses N=80)
    s += [("net", 7), ("tail", 160, 160)]                         # a fully teacher-forced frame (state update only)
    s += [("defer", 8), ("defer", 9), ("flush",)]                 # queued conditioning frames, network run later
    s += [("net", 10), ("defer", 11), ("defer", 12), ("flush",), ("tail", 80, 0)]    # a flush keeps the conditioning a tail reads (lpcnet.c:134-144)
    s += [("synth", 13, 160, 0), ("reset_signal",), ("synth", 14, 160, 0)]
    s += [("save",), ("synth", 15, 160, 0), ("synth", 16, 160, 0), ("restore",), ("synth", 15, 160, 0), ("synth", 16, 160, 0)]
    s += [("synth", t, 160, 0) for t in range(17, T)]
    return s


def forced_signal(stream, n):
    """The 'known' signal a PLC would teacher-force with (deterministic, speech-like amplitude)."""
    rng = np.random.default_rng(5000 + int(stream))
    return (3000 * np.sin(np.arange(n) * 0.05 * (1 + stream % 3)) + rng.normal(0, 300, n)).astype(np.int16)


def run_single(backend, lib, st_new, feats, stream, script):
    """backend: 'ref' | 'oracle'.  feats [T][20].  Returns the concatenated PCM of all output-producing ops."""
    P = {"ref": dict(impl=lib.ref_synthesize_impl, net=lib.ref_run_frame_network, tail=lib.ref_synthesize_tail, defer=lib.ref_frame_network_deferred,
                     flush=lib.ref_frame_network_flush, rs=lib.ref_reset_signal) if backend == "ref" else None,
         "oracle": dict(impl=lib.oracle_synthesize_impl, net=lib.oracle_run_frame_network, tail=lib.oracle_synthesize_tail, defer=lib.oracle_frame_network_deferred,
                        flush=lib.oracle_frame_network_flush, rs=lib.oracle_reset_signal) if backend == "oracle" else None}[backend]
    st = st_new()
    saved = None
    out = []
    k = 0
    for op in script:
        if op[0] == "synth":
            _, t, N, pre = op
            buf = np.zeros(N, np.int16); buf[:pre] = forced_signal(stream, 4000)[k:k + pre]
            P["impl"](st, feats[t].ctypes.data, buf.ctypes.data, N, pre)
            out.append(buf); k += N
        elif op[0] == "net":
            P["net"](st, feats[op[1]].ctypes.data)
        elif op[0] == "tail":
            _, N, pre = op
            buf = np.zeros(N, np.int16); buf[:pre] = forced_signal(stream, 4000)[k:k + pre]
            P["tail"](st, buf.ctypes.data, N, pre)
            out.append(buf); k += N
        elif op[0] == "defer":
            P["defer"](st, feats[op[1]].ctypes.data)
        elif op[0] == "flush":
            P["flush"](st)
        elif op[0] == "reset_signal":
            P["rs"](st)
        elif op[0] == "save":
            saved = st_new.copy_of(st)
        elif op[0] == "restore":
            st_new.assign(st, saved)
    return np.concatenate(out)


class RefState:
    """state factory for run_single('ref', ...)"""
    def __init__(self, build="A", tag="", kind=None):
        self.L = H.ref_lib(build, tag); self.b = H.blob(kind or ("float" if build == "B" else "int8"), tag)
    def __call__(self):
        st = self.L.ref_state_create(self.b, len(self.b)); assert st; return st
    def copy_of(self, st):
        c = self(); self.L.ref_state_copy(c, st); return c
    def assign(self, dst, src):
        self.L.ref_state_copy(dst, src)
    def reset(self, st):
        self.L.ref_state_reset(st)
    def destroy(self, st):
        self.L.ref_state_destroy(st)


class RefDecState(RefState):
    """decoder-state factory for decode scripts on the reference: LPCNetDecState, whose reset is what lpcnet_decoder_init does to
    a loaded state (lpcnet_reset and vq_mem cleared) and whose copy includes vq_mem"""
    def __call__(self):
        st = self.L.ref_dec_state_create(self.b, len(self.b)); assert st; return st
    def copy_of(self, st):
        c = self(); self.assign(c, st); return c
    def assign(self, dst, src):
        self.L.ref_dec_state_copy(dst, src)
    def reset(self, st):
        self.L.ref_dec_reset(st)
    def destroy(self, st):
        self.L.ref_dec_state_destroy(st)


class OracleState:
    def __init__(self, kind="int8", tag=""):
        self.L = H.oracle_lib(); self.m = H.oracle_model(kind, tag)
        self.size = 1 << 16
    def __call__(self):
        return self.L.oracle_state_create(self.m)
    def copy_of(self, st):
        c = self(); ctypes.memmove(c, st, self.L.oracle_state_size()); return c
    def assign(self, dst, src):
        ctypes.memmove(dst, src, self.L.oracle_state_size())
    def reset(self, st):
        self.L.oracle_reset(st)
    def destroy(self, st):
        self.L.oracle_state_destroy(st)


def run_engine(batch, feats, streams, script):
    """feats [n][T][20]; the same script on all streams of a lpcnet_b200.Batch.  Returns PCM [n][total]."""
    n = batch.n
    forced = np.stack([forced_signal(s, 4000) for s in streams])
    out, k, snap = [], 0, None
    for op in script:
        if op[0] == "synth":
            _, t, N, pre = op
            out.append(batch.synthesize(feats[:, t:t + 1], samples_per_frame=N, preload=pre, pcm_in=forced[:, k:k + max(pre, 1)])); k += N
        elif op[0] == "net":
            batch.run_frame_network(feats[:, op[1]:op[1] + 1])
        elif op[0] == "tail":
            _, N, pre = op
            out.append(batch.synthesize_tail(N, preload=pre, pcm_in=forced[:, k:k + max(pre, 1)])); k += N
        elif op[0] == "defer":
            batch.frame_network_deferred(feats[:, op[1]])
        elif op[0] == "flush":
            batch.frame_network_flush()
        elif op[0] == "reset_signal":
            batch.reset_signal()
        elif op[0] == "save":
            snap = batch.snapshot()
        elif op[0] == "restore":
            batch.restore(snap)
    if snap is not None:
        batch.free_snapshot(snap)
    return np.concatenate(out, axis=1)


# ---- random call sequences over a batch of streams ------------------------------------------------------------------------------
# A script is (ops, T, signal): batch operations over feature frames 0..T-1 and the kind of signal the teacher-forced samples come from.
#   ("synth", t, k, N, pre)   frames t..t+k-1, N samples each, `pre` forced samples at the start of the first frame
#   ("net", t, k)             run_frame_network over frames t..t+k-1
#   ("tail", N, pre)          synthesize_tail
#   ("defer", t)              run_frame_network_deferred of frame t
#   ("flush",) ("reset_signal",) ("reset",) ("save",) ("restore",)
#   ("reset_streams", ids)    lpcnet_reset of the listed streams
#   ("move", a, b)            export stream a, import the blob into stream b
#   ("decode", p, k)          lpcnet_decode of packets p..p+k-1 of each stream's packet source (decode scripts only)
# Only what the batched ABI allows is generated: stream a of a move has no queued frames, and no tail follows a move before
# the next synth / net / decode (the exported state carries neither the queue nor the conditioning).
# A decode script, random_script(..., decode=True), is (ops, T, signal, source): `source` names where each stream's packets come
# from (PACKET_SOURCES, script_packets).  Synthesis and decode share one per-stream state, as lpcnet_decode shares LPCNetDecState's
# LPCNetState with the synthesis entry points: a decode advances the frame counter by 4 per packet and leaves the conditioning of
# the packet's last frame for a tail; resets, moves and snapshots carry or clear the previous superframe's cepstrum (vq_mem) too.
OUTPUT_OPS = ("synth", "tail", "decode")
SYNTH_FRAMES = (1, 2, 3, 17, 20)            # 17 and 20 cross the engine's 16-frame chunk
SAMPLES = (1, 80, 160, 250)
DECODE_PACKETS = (1, 2, 3, 4, 5, 6)         # 4 packets = one 16-frame chunk, 5 and 6 cross it
PACKET_SOURCES = ("random", "encoded", "edge")


def _preload(rng, N):
    r = rng.random()
    return 0 if r < 0.5 else (N if r < 0.75 else rng.randint(1, min(N, 40)))


def random_script(seed, n_streams, n_ops=22, decode=False):
    """A random script (ops, T, signal); with `decode` a decode script (ops, T, signal, source) that also decodes packets, often
    right after the ops that carry or clear the decoder's memory.  Without `decode` no extra random draw is made, so the scripts
    of a seed stay what they were before decode existed."""
    import random
    rng = random.Random(seed)
    ops, t = [], 0
    fill = [0] * n_streams               # queued frames per stream
    no_tail = False                       # a move since the last synth / net / decode
    saved = None                          # (fill, no_tail) at the last save
    signal = rng.choice(["speech", "square"])
    source = rng.choice(PACKET_SOURCES) if decode else None
    p = 0                                 # next packet of each stream's source

    def synth():
        nonlocal t, no_tail
        k = rng.choice(SYNTH_FRAMES) if rng.random() < 0.35 else rng.choice((1, 1, 2, 3))
        N = rng.choice(SAMPLES)
        ops.append(("synth", t, k, N, _preload(rng, N))); t += k; no_tail = False

    def dec():
        nonlocal p, no_tail
        k = rng.choice(DECODE_PACKETS)
        ops.append(("decode", p, k)); p += k; no_tail = False

    def maybe_dec(prob):
        if decode and rng.random() < prob:
            dec()

    def tail():
        if not no_tail:
            N = rng.choice(SAMPLES)
            ops.append(("tail", N, _preload(rng, N)))

    def flush():
        ops.append(("flush",))
        fill[:] = [0] * n_streams

    def reset_streams():
        ids = sorted(rng.sample(range(n_streams), rng.randint(1, max(1, n_streams // 2))))
        if rng.random() < 0.5:
            ids = sorted(set(ids) | {rng.choice((0, n_streams - 1))})
        ops.append(("reset_streams", ids))
        for s in ids:
            fill[s] = 0

    kinds = ["synth", "net", "tail", "defer", "flush", "reset_signal", "reset", "reset_streams", "save", "restore", "move"]
    weights = [5, 2, 2, 3, 2, 1, 1, 2, 1, 1, 1]
    if decode:
        kinds, weights = kinds + ["decode"], weights + [5]
    synth()
    while len(ops) < n_ops:
        op = rng.choices(kinds, weights)[0]
        if op == "synth":
            synth()
            maybe_dec(0.3)
        elif op == "decode":
            dec()
            r = rng.random()
            if r < 0.3:
                tail()
            elif r < 0.6:
                synth()
        elif op == "net":
            k = rng.choice((1, 2, 3))
            ops.append(("net", t, k)); t += k; no_tail = False
            if rng.random() < 0.5:
                tail()
        elif op == "tail":
            tail()
        elif op == "defer":
            for _ in range(rng.choice((1, 2, 3, 5, 6))):          # 5-6: the oldest queued frames drop out
                ops.append(("defer", t)); t += 1
                fill[:] = [min(4, v + 1) for v in fill]
            maybe_dec(0.5)                                        # a decode leaves the queue alone
            r = rng.random()
            if r < 0.3:
                reset_streams()                                   # with queued frames: only the other streams' queues stay
            if r < 0.7:
                flush()
                if rng.random() < 0.7:
                    tail()
        elif op == "flush":
            flush()
        elif op == "reset_signal":
            ops.append(("reset_signal",))
            maybe_dec(0.6)
        elif op == "reset":
            ops.append(("reset",)); fill[:] = [0] * n_streams; no_tail = False
            if rng.random() < 0.5:
                tail()
        elif op == "reset_streams":
            reset_streams()
            maybe_dec(0.5)
            r = rng.random()
            if r < 0.4:
                synth()                                           # within FEATURES_DELAY frames of the reset: a mixed silent segment
            elif r < 0.7 and any(fill):
                flush()
                tail()
        elif op == "save":
            ops.append(("save",)); saved = (list(fill), no_tail)
        elif op == "restore" and saved is not None:
            ops.append(("restore",)); fill[:] = saved[0]; no_tail = saved[1]
            maybe_dec(0.5)
            if rng.random() < 0.6:
                tail()
        elif op == "move":
            ok = [s for s in range(n_streams) if fill[s] == 0]
            if ok:
                a = rng.choice(ok)
                b = rng.choice([s for s in range(n_streams) if s != a] or [a])
                ops.append(("move", a, b)); fill[b] = 0; no_tail = True
                maybe_dec(0.6)
    return (ops, t, signal, source) if decode else (ops, t, signal)


def script_events(script, n_streams, delay=2):
    """The situations a script reaches, found by following each stream's queue and frame counter: a set of names."""
    ev = set()
    fill, fc = [0] * n_streams, [0] * n_streams
    prev, saved = None, None
    queued_decode = False                 # a decode ran while frames were queued, and no flush since
    for op in script[0]:
        kind = tag = op[0]
        ev.add(kind)
        if kind == "synth":
            k, N, pre = op[2:]
            if pre == N and k > 1:
                ev.add("preload_N_multi_frame")
            if k > 16:
                ev.add("synth_crosses_chunk")
            if min(k, max(0, delay - min(fc))) > min(k, max(0, delay - max(fc))):     # some streams silent, others not
                ev.add("mixed_silent_segment")
            if prev == "decode":
                ev.add("synth_after_decode")
            fc = [min(1000, v + k) for v in fc]
        elif kind == "decode":
            k = 4 * op[2]
            if k > 16:
                ev.add("decode_crosses_chunk")
            if min(k, max(0, delay - min(fc))) > min(k, max(0, delay - max(fc))):
                ev.add("decode_mixed_silent_segment")
            if any(fill):
                ev.add("decode_with_queue"); queued_decode = True
            after = {"synth": "decode_after_synth", "restore": "decode_after_restore", "move": "decode_after_move",
                     "reset_signal": "decode_after_reset_signal", "reset_streams": "decode_after_reset_streams",
                     "reset_streams+": "decode_after_reset_streams"}
            if prev in after:
                ev.add(after[prev])
            fc = [min(1000, v + k) for v in fc]
        elif kind == "net":
            fc = [min(1000, v + op[2]) for v in fc]
        elif kind == "defer":
            if 4 in fill:
                ev.add("queue_overflow")
            fill = [min(4, v + 1) for v in fill]
        elif kind == "flush":
            if any(fill):
                tag = "flush+"
                if prev == "reset_streams+":
                    ev.add("flush_after_reset_streams_with_queue")
                if len(set(fill)) > 1:
                    ev.add("flush_uneven_queues")
                if queued_decode:
                    ev.add("flush_after_decode_with_queue")
            queued_decode = False
            fc = [min(1000, v + f) for v, f in zip(fc, fill)]
            fill = [0] * n_streams
        elif kind == "tail":
            ev.add({"flush+": "tail_after_nonempty_flush", "reset": "tail_after_reset", "restore": "tail_after_restore",
                    "decode": "tail_after_decode"}.get(prev, "tail"))
        elif kind == "reset":
            fill, fc = [0] * n_streams, [0] * n_streams
        elif kind == "reset_streams":
            if any(fill[s] for s in op[1]):
                tag = "reset_streams+"
            if 0 in op[1] or n_streams - 1 in op[1]:
                ev.add("reset_streams_edge")
            for s in op[1]:
                fill[s] = fc[s] = 0
        elif kind == "save":
            saved = (list(fill), list(fc))
        elif kind == "restore":
            fill, fc = list(saved[0]), list(saved[1])
        elif kind == "move":
            fc[op[2]] = fc[op[1]]
            fill[op[2]] = 0
        prev = tag
    return ev


def script_outputs(script):
    """Samples per stream the script's synth, tail and decode ops produce."""
    return sum(op[2] * op[3] if op[0] == "synth" else op[2] * 640 if op[0] == "decode" else op[1] for op in script[0] if op[0] in OUTPUT_OPS)


def script_packets(script, streams):
    """Packets [n][P][8] of a decode script's source for the given stream ids (P: the packets its decode ops read), or None for a
    script without decodes.  random: fixtures.make_packets; encoded: the encoder (CPU restatement) on fixtures.make_pcm speech,
    so consecutive packets belong together; edge: the encoder on the edge signals of oracle/edge_inputs.py, one per stream,
    repeated to length."""
    P = max([op[1] + op[2] for op in script[0] if op[0] == "decode"], default=0)
    if len(script) < 4 or P == 0:
        return None
    return np.stack([_stream_packets(script[3], int(s), P) for s in streams])


@functools.lru_cache(None)
def _stream_packets(source, stream, P):
    from fixtures import make_packets, make_pcm
    if source == "random":
        return make_packets(stream, P)
    if source == "encoded":
        return H.oracle_encode(make_pcm(stream, 4 * P)[None])[0]
    assert source == "edge", source
    edge = _edge_packets()
    return np.resize(edge[stream % len(edge)], (P, 8))


_EDGE = []


def _edge_packets():
    if not _EDGE:
        import edge_inputs as E
        c = E.pcm_cases()
        _EDGE.append(H.oracle_encode(np.stack([c[k] for k in c])))
    return _EDGE[0]


def forced_pcm(signal, stream, n):
    """Teacher-forcing signal of one stream: the speech-like forced_signal, or a full-scale square wave (+32767 / -32768) that
    drives lin2ulaw of the forced excitation to its clamps."""
    if signal == "square":
        period = 24 + 2 * (int(stream) % 7)
        return np.where(np.arange(n) % period < period // 2, 32767, -32768).astype(np.int16)
    rng = np.random.default_rng(5000 + int(stream))
    return (3000 * np.sin(np.arange(n) * 0.05 * (1 + stream % 3)) + rng.normal(0, 300, n)).astype(np.int16)


def run_streams(backend, lib, factory, feats, streams, script, pool=None):
    """A script on one single-stream state per stream (backend 'ref' | 'oracle').  feats [n][T][20].  reset_streams resets the
    listed states, a move copies the whole source state, a snapshot copies every state (a decode script needs decoder states:
    RefDecState, or OracleState, whose state holds vq_mem).  Returns PCM [n][script_outputs]."""
    ops, signal = script[0], script[2]
    n = len(streams)
    P = (dict(impl=lib.ref_synthesize_impl, net=lib.ref_run_frame_network, tail=lib.ref_synthesize_tail, defer=lib.ref_frame_network_deferred,
              flush=lib.ref_frame_network_flush, rs=lib.ref_reset_signal) if backend == "ref" else
         dict(impl=lib.oracle_synthesize_impl, net=lib.oracle_run_frame_network, tail=lib.oracle_synthesize_tail, defer=lib.oracle_frame_network_deferred,
              flush=lib.oracle_frame_network_flush, rs=lib.oracle_reset_signal))
    pk = script_packets(script, streams)
    if pk is not None:
        P["decode"] = lib.ref_decode if backend == "ref" else lib.oracle_decode
    total = script_outputs(script)
    forced = [forced_pcm(signal, s, total) for s in streams]
    out = np.zeros((n, total), np.int16)
    st = [factory() for _ in range(n)]
    snap = None
    k = 0

    def each(fn):
        list(pool.map(fn, range(n))) if pool is not None else [fn(i) for i in range(n)]

    for op in ops:
        kind = op[0]
        if kind == "synth":
            _, t, nf, N, pre = op
            def run(i, t=t, nf=nf, N=N, pre=pre, k=k):
                for j in range(nf):
                    buf = out[i, k + j * N:k + (j + 1) * N]
                    if j == 0:
                        buf[:pre] = forced[i][k:k + pre]
                    P["impl"](st[i], feats[i, t + j].ctypes.data, buf.ctypes.data, N, pre if j == 0 else 0)
            each(run); k += nf * N
        elif kind == "decode":
            _, p, npk = op
            def run(i, p=p, npk=npk, k=k):
                for j in range(npk):
                    assert P["decode"](st[i], pk[i, p + j].ctypes.data, out[i, k + j * 640:k + (j + 1) * 640].ctypes.data) == 0
            each(run); k += npk * 640
        elif kind == "net":
            _, t, nf = op
            each(lambda i: [P["net"](st[i], feats[i, t + j].ctypes.data) for j in range(nf)])
        elif kind == "tail":
            _, N, pre = op
            def run(i, N=N, pre=pre, k=k):
                buf = out[i, k:k + N]
                buf[:pre] = forced[i][k:k + pre]
                P["tail"](st[i], buf.ctypes.data, N, pre)
            each(run); k += N
        elif kind == "defer":
            for i in range(n):
                P["defer"](st[i], feats[i, op[1]].ctypes.data)
        elif kind == "flush":
            each(lambda i: P["flush"](st[i]))
        elif kind == "reset_signal":
            for i in range(n):
                P["rs"](st[i])
        elif kind == "reset":
            for i in range(n):
                factory.reset(st[i])
        elif kind == "reset_streams":
            for i in op[1]:
                factory.reset(st[i])
        elif kind == "save":
            if snap is not None:
                for c in snap:
                    factory.destroy(c)
            snap = [factory.copy_of(x) for x in st]
        elif kind == "restore":
            for x, c in zip(st, snap):
                factory.assign(x, c)
        elif kind == "move":
            factory.assign(st[op[2]], st[op[1]])
    for x in st + (snap or []):
        factory.destroy(x)
    return out


def run_engine_script(batch, feats, streams, script):
    """The same script on a lpcnet_b200.Batch of len(streams) streams (with codebooks for a decode script).  Returns PCM
    [n][script_outputs]."""
    ops, signal = script[0], script[2]
    total = script_outputs(script)
    forced = np.stack([forced_pcm(signal, s, total) for s in streams])
    pk = script_packets(script, streams)
    out, k, snap = [], 0, None
    for op in ops:
        kind = op[0]
        if kind == "synth":
            _, t, nf, N, pre = op
            out.append(batch.synthesize(feats[:, t:t + nf], samples_per_frame=N, preload=pre, pcm_in=forced[:, k:k + max(pre, 1)])); k += nf * N
        elif kind == "decode":
            _, p, npk = op
            out.append(batch.decode(pk[:, p:p + npk])); k += npk * 640
        elif kind == "net":
            batch.run_frame_network(feats[:, op[1]:op[1] + op[2]])
        elif kind == "tail":
            _, N, pre = op
            out.append(batch.synthesize_tail(N, preload=pre, pcm_in=forced[:, k:k + max(pre, 1)])); k += N
        elif kind == "defer":
            batch.frame_network_deferred(feats[:, op[1]])
        elif kind == "flush":
            batch.frame_network_flush()
        elif kind == "reset_signal":
            batch.reset_signal()
        elif kind == "reset":
            batch.reset()
        elif kind == "reset_streams":
            batch.reset_streams(op[1])
        elif kind == "save":
            if snap is not None:
                batch.free_snapshot(snap)
            snap = batch.snapshot()
        elif kind == "restore":
            batch.restore(snap)
        elif kind == "move":
            batch.import_state(op[2], batch.export_state(op[1]))
    if snap is not None:
        batch.free_snapshot(snap)
    return np.concatenate(out, axis=1)
