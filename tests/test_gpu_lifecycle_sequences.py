"""GPU tests (-m gpu): the seeded random call sequences of scenarios.random_script on the engine, bit for bit against the CPU
restatement run per stream, under every per-sample schedule (int8 one-half and two-half, ragged and dead slots, the conversion
unit; float neuron-per-lane and lane==stream), the seeds of tests/test_lifecycle_sequences.py against the compiled reference's
stored digests, and the contract rules of the tail, deferred and state-by-value entry points one by one."""
import os
from concurrent.futures import ThreadPoolExecutor
import json
import numpy as np
import pytest
import helpers as H
import scenarios as S
from fixtures import make_feature_batch, make_features
from test_lifecycle_sequences import CASES, SEEDS, seq_inputs, seq_key

pytestmark = pytest.mark.gpu

# (kind, tag, streams, create-time knobs LPCNET_B200_<name>): the schedule the launcher picks for that batch
SCHEDULES = [
    ("int8", "", 37, {}),                                                # automatic: one-half, one stream per CTA
    ("int8", "", 70, {"STREAMS_PER_CTA": "32"}),                         # two halves, two full CTAs + a ragged one
    ("int8", "", 40, {"STREAMS_PER_CTA": "17"}),                         # the smallest two-half CTA
    ("int8", "", 12, {"STREAMS_PER_CTA": "5", "TWO_HALVES": "1"}),       # dead slots in both halves
    ("int8", "", 40, {"STREAMS_PER_CTA": "32", "EXACT_CVT": "1"}),       # the conversion unit instead of the conversion-free rounding
] + [c for tag in ("na128", "na256e2e", "delay0", "delay1") for c in (("int8", tag, 5, {}), ("int8", tag, 40, {"STREAMS_PER_CTA": "32"}))] + [
    c for tag in ("", "delay1") for c in (("float", tag, 5, {}),                        # neuron-per-lane, one slot per CTA
                                           ("float", tag, 8, {"STREAMS_PER_CTA": "3"}),  # neuron-per-lane, ragged
                                           ("float", tag, 6, {"FLOAT_LANE_STREAM": "1"}))]   # lane == stream
GPU_SEEDS = range(3)


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


def _oracle(kind, tag, f, streams, script, pool):
    return S.run_streams("oracle", H.oracle_lib(), S.OracleState(kind, tag), f, streams, script, pool)


def _engine(eng, kind, tag, f, streams, script):
    b = eng.Batch(len(streams), H.blob(kind, tag), config=H.model_config(tag))
    try:
        return S.run_engine_script(b, f, streams, script)
    finally:
        b.close()


def _assert_same(got, want, what):
    d = np.argwhere(got != want)
    assert d.size == 0, "%s: first mismatch (stream, sample) = %s" % (what, tuple(d[0]))


def _knob_id(c):
    return "%s-%s-n%d-%s" % (c[0], c[1] or "base", c[2], "-".join("%s=%s" % kv for kv in sorted(c[3].items())) or "auto")


@pytest.mark.parametrize("kind,tag,n,knobs", SCHEDULES, ids=[_knob_id(c) for c in SCHEDULES])
def test_random_sequences_match_oracle(eng, pool, monkeypatch, kind, tag, n, knobs):
    for k, v in knobs.items():
        monkeypatch.setenv("LPCNET_B200_" + k, v)
    for seed in GPU_SEEDS:
        script = S.random_script(1000 + seed, n)
        streams = list(range(500 + 100 * seed, 500 + 100 * seed + n))
        f = make_feature_batch(streams, script[1])
        got = _engine(eng, kind, tag, f, streams, script)
        _assert_same(got, _oracle(kind, tag, f, streams, script, pool), "seed %d %s" % (seed, script[0]))


@pytest.mark.parametrize("build,tag", CASES)
def test_cpu_seeds_match_reference_digests(eng, build, tag):
    """The seeds of the CPU file, whose reference PCM is stored as digests: the engine equals the reference directly."""
    stored = json.load(open(H.REF_DIGESTS))
    kind = "float" if build == "B" else "int8"
    for seed in SEEDS:
        script, f, streams = seq_inputs(seed)
        assert H.digest(_engine(eng, kind, tag, f, streams, script)) == stored[seq_key(build, tag, seed)], "seed %d" % seed


# ---- the contract rules one by one, on the default int8 and float models ----
KINDS = ["int8", "float"]


def _check_script(eng, pool, kind, ops, n=4, signal="speech"):
    T = max([op[1] + (op[2] if op[0] in ("synth", "net") else 1) for op in ops if op[0] in ("synth", "net", "defer")])
    script = (ops, T, signal)
    streams = list(range(40, 40 + n))
    f = make_feature_batch(streams, T)
    got = _engine(eng, kind, "", f, streams, script)
    _assert_same(got, _oracle(kind, "", f, streams, script, pool), str(ops))
    return got


@pytest.mark.parametrize("kind", KINDS)
def test_tail_after_flush_uses_the_last_frame_network_run(eng, pool, kind):
    got = _check_script(eng, pool, kind, [("synth", 0, 5, 160, 0), ("net", 5, 1), ("defer", 6), ("defer", 7), ("flush",), ("tail", 160, 0),
                                          ("defer", 8), ("defer", 9), ("defer", 10), ("flush",), ("tail", 80, 40)])
    assert np.abs(got[:, 800:960]).max() > 0


@pytest.mark.parametrize("kind", KINDS)
def test_tail_after_reset_gives_zeros(eng, pool, kind):
    got = _check_script(eng, pool, kind, [("synth", 0, 3, 160, 0), ("reset",), ("tail", 80, 0), ("tail", 80, 80)])
    assert (got[:, 480:] == 0).all() and np.abs(got[:, 320:480]).max() > 0
    # after the reset, three flushed frames lift the counters past FEATURES_DELAY: the tail runs on zero conditioning and LPC
    got = _check_script(eng, pool, kind, [("synth", 0, 3, 160, 0), ("reset",), ("defer", 3), ("defer", 4), ("defer", 5), ("flush",), ("tail", 160, 0)])
    assert np.abs(got[:, 480:]).max() > 0


@pytest.mark.parametrize("kind", KINDS)
def test_restore_then_tail_matches_oracle(eng, pool, kind):
    _check_script(eng, pool, kind, [("synth", 0, 3, 160, 0), ("net", 3, 1), ("save",), ("synth", 4, 2, 160, 0), ("defer", 6), ("flush",),
                                    ("restore",), ("tail", 160, 0), ("tail", 80, 40), ("synth", 4, 1, 160, 0)])


@pytest.mark.parametrize("kind", KINDS)
def test_reset_streams_with_queued_frames_then_flush_matches_oracle(eng, pool, kind):
    _check_script(eng, pool, kind, [("synth", 0, 3, 160, 0), ("defer", 3), ("defer", 4), ("reset_streams", [0, 2]), ("defer", 5), ("flush",),
                                    ("tail", 80, 0), ("synth", 6, 2, 160, 0), ("net", 8, 1), ("defer", 9), ("reset_streams", [3]),
                                    ("flush",), ("tail", 160, 0), ("synth", 10, 3, 160, 0)])


def test_tail_after_import_is_refused(eng):
    n = 3
    f = make_feature_batch(range(n), 4)
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    b.synthesize(f[:, :2])
    b.import_state(1, b.export_state(0))
    with pytest.raises(eng.LPCNetB200Error, match="imported"):
        b.synthesize_tail(80)
    b.frame_network_deferred(f[:, 2])
    b.frame_network_flush()
    with pytest.raises(eng.LPCNetB200Error, match="imported"):
        b.synthesize_tail(80)
    b.run_frame_network(f[:, 3:4])
    assert b.synthesize_tail(80).shape == (n, 80)
    b.close()


def test_export_with_queued_frames_is_refused(eng):
    n = 3
    f = make_feature_batch(range(n), 3)
    b = eng.Batch(n, H.blob("int8"), lpc_gamma=H.LPC_GAMMA)
    b.synthesize(f[:, :1])
    b.frame_network_deferred(f[:, 1])
    with pytest.raises(eng.LPCNetB200Error, match="queued"):
        b.export_state(2)
    b.reset_streams([2])                      # its queue is gone with the reset
    b.export_state(2)
    b.frame_network_flush()
    b.export_state(0)
    b.close()
