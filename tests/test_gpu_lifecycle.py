"""GPU tests (-m gpu) of the entry semantics the reference's PLC needs from the hot path (SURVEY.md 8f N3) and of per-stream
lifecycle in the batched ABI: `preload` teacher forcing (lpcnet.c:256-259,269), run_frame_network + lpcnet_synthesize_tail_impl,
run_frame_network_deferred/_flush (lpcnet.c:122-144), lpcnet_reset_signal, state by value (export / import / device snapshot,
lpcnet_plc.c:216-230), per-stream reset with per-stream frame counters, and caller-owned CUDA streams."""
import numpy as np
import pytest
import helpers as H
import scenarios as S
from fixtures import make_feature_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


@pytest.mark.parametrize("kind,tag,n", [("int8", "", 40), ("int8", "", 5), ("float", "", 6), ("float", "", 40), ("int8", "na256e2e", 7), ("int8", "delay0", 3), ("int8", "delay1", 4)])
def test_plc_like_call_sequence_matches_oracle(eng, kind, tag, n):
    """The scripted sequence of scenarios.plc_like_script (preload, tails of 80, a fully forced frame, deferred + flush,
    reset_signal, snapshot / restore) on a batch == the same sequence per stream on the CPU restatement (which the CPU suite
    pins to the compiled reference, tests/test_oracle.py::test_oracle_port_plc_entry_points_match_reference)."""
    T = 18
    streams = list(range(100, 100 + n))
    f = make_feature_batch(streams, T)
    script = S.plc_like_script(T)
    b = eng.Batch(n, H.blob(kind, tag), config=H.model_config(tag))
    got = S.run_engine(b, f, streams, script)
    b.close()
    for i, s in enumerate(streams):
        want = S.run_single("oracle", H.oracle_lib(), S.OracleState(kind, tag), f[i], s, script)
        d = np.argwhere(got[i] != want)
        assert d.size == 0, "stream %d: first mismatch at sample %d" % (s, d[0][0])


def test_state_export_import_roundtrip_and_oracle_state(eng):
    """(i) export a stream, keep going, import into ANOTHER slot of another batch: identical continuation;
    (ii) a state produced by the CPU restatement imports into the engine and continues bit-exactly."""
    n, T = 6, 14
    f = make_feature_batch(range(50, 50 + n), T)
    a = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    head = a.synthesize(f[:, :7])
    st3 = a.export_state(3)
    rest = a.synthesize(f[:, 7:])
    c = eng.Batch(2, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    c.synthesize(make_feature_batch([900, 901], 3))                      # unrelated history in both slots
    c.import_state(1, st3)
    f2 = np.stack([f[0, 7:], f[3, 7:]])
    got = c.synthesize(f2)
    np.testing.assert_array_equal(got[1], rest[3])
    # oracle -> engine
    L = H.oracle_lib()
    st = L.oracle_state_create(H.oracle_model())
    pcm = np.zeros(160, np.int16)
    for t in range(7):
        L.oracle_synthesize(st, f[4, t].ctypes.data, pcm.ctypes.data, 160)
    buf = np.zeros(a.export_state(0).size, np.float32)
    assert L.oracle_export_state(st, buf.ctypes.data) == buf.size * 4
    np.testing.assert_array_equal(buf.view(np.uint32), _export_at(eng, f, 4, 7).view(np.uint32))
    c.import_state(0, buf)
    got = c.synthesize(np.stack([f[4, 7:], f[3, 7:]]))
    np.testing.assert_array_equal(got[0], rest[4])
    L.oracle_state_destroy(st)
    a.close(); c.close()
    assert np.abs(head).max() > 0


def _export_at(eng, f, s, frames):
    b = eng.Batch(f.shape[0], H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    b.synthesize(f[:, :frames])
    st = b.export_state(s)
    b.close()
    return st


def test_per_stream_reset_and_frame_counters(eng):
    """Streams 1 and 3 of a running batch start a new utterance (lpcnet_reset: two silent frames, fresh RNG) while the others
    carry on: every stream equals its own single-stream trajectory; includes the mixed frames in which only some streams are silent."""
    n, T1, T2 = 5, 6, 7
    f = make_feature_batch(range(70, 70 + n), T1 + T2)
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    first = b.synthesize(f[:, :T1])
    b.reset_streams([1, 3])
    second = np.concatenate([b.synthesize(f[:, T1:T1 + 1]), b.synthesize(f[:, T1 + 1:])], axis=1)   # 1-frame call, then the rest
    assert b.get_state(1)["frame_count"] == T2 and b.get_state(0)["frame_count"] == T1 + T2
    b.close()
    cont = H.oracle_synth(f, "int8")
    fresh = H.oracle_synth(f[:, T1:], "int8")
    np.testing.assert_array_equal(first, cont[:, :T1 * 160])
    for s in range(n):
        want = fresh[s] if s in (1, 3) else cont[s, T1 * 160:]
        np.testing.assert_array_equal(second[s], want, err_msg="stream %d" % s)
    assert (second[1, :320] == 0).all() and np.abs(second[0, :320]).max() > 0


def test_caller_streams_are_ordered_against_the_engine_state(eng):
    """`_device` calls on two different caller-owned CUDA streams, interleaved with host-pointer calls and a state read: the
    engine orders its state across streams (event hand-over), so the result equals the single-stream run."""
    n, T = 33, 12
    f = make_feature_batch(range(600, 600 + n), T)
    L = eng.lib()
    s1, s2 = L.lpcnet_b200_stream_create(), L.lpcnet_b200_stream_create()
    assert s1 and s2
    want = H.oracle_synth(f, "int8")
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    d_f = L.lpcnet_b200_device_alloc(f.nbytes)
    L.lpcnet_b200_memcpy_h2d(d_f, f.ctypes.data, f.nbytes)
    d_p = [L.lpcnet_b200_device_alloc(n * 3 * 160 * 2) for _ in range(3)]
    # frames 0-2 on stream 1, 3-5 on stream 2, 6-8 host-pointer call, 9-11 on stream 1 again
    def dev_call(t0, dp, st):
        fv = np.ascontiguousarray(f[:, t0:t0 + 3])
        ptr = L.lpcnet_b200_device_alloc(fv.nbytes); L.lpcnet_b200_memcpy_h2d(ptr, fv.ctypes.data, fv.nbytes)
        b.synthesize_device(ptr, 3, 20, dp, cuda_stream=st)
        return ptr
    tmp = [dev_call(0, d_p[0], s1), dev_call(3, d_p[1], s2)]
    mid = b.synthesize(f[:, 6:9])
    tmp.append(dev_call(9, d_p[2], s1))
    st = b.get_state(5)                                              # host-side read: waits for the work on stream 1
    got = [np.zeros((n, 480), np.int16) for _ in range(3)]
    for g, dp in zip(got, d_p):
        L.lpcnet_b200_memcpy_d2h(g.ctypes.data, dp, g.nbytes)
    full = np.concatenate([got[0], got[1], mid, got[2]], axis=1)
    np.testing.assert_array_equal(full, want)
    assert st["frame_count"] == T
    for p in tmp + d_p + [d_f]:
        L.lpcnet_b200_device_free(p)
    b.close()
    L.lpcnet_b200_stream_destroy(s1); L.lpcnet_b200_stream_destroy(s2)
