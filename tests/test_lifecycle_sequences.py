"""CPU tests: seeded random call sequences over the reference's internal entry points (scenarios.random_script: synthesize with
`preload`, run_frame_network, tails, deferred frames and flushes, resets of all or some streams, snapshots, state export and
import), run on one state per stream by the CPU restatement and by the compiled reference.  The reference's PCM is pinned by
digests in tests/golden/ref_digests.json (keys seq_<build>_<tag>_<seed>), so the comparison also runs where no reference is
compiled.  tests/test_gpu_lifecycle_sequences.py runs the same seeds on the engine."""
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import pytest
import helpers as H
import scenarios as S
from fixtures import make_feature_batch, make_features

SEEDS = range(8)
N_STREAMS = 3
CASES = [("A", ""), ("A", "na256e2e"), ("A", "delay0"), ("A", "delay1"), ("B", ""), ("B", "delay1")]


def seq_streams(seed):
    return [300 + 10 * seed + i for i in range(N_STREAMS)]


def seq_inputs(seed):
    """(script, features [n][T][20], stream ids) of one seed of this file."""
    script = S.random_script(seed, N_STREAMS)
    streams = seq_streams(seed)
    return script, make_feature_batch(streams, script[1]), streams


def seq_key(build, tag, seed):
    return "seq_%s_%s_%d" % (build, tag, seed)


def test_seed_set_reaches_every_situation():
    """The fixed seeds reach each op kind and each situation the entry points' contract has a rule for."""
    seen = set()
    for seed in SEEDS:
        seen |= S.script_events(S.random_script(seed, N_STREAMS), N_STREAMS)
    want = {"synth", "net", "tail", "defer", "flush", "reset_signal", "reset", "reset_streams", "save", "restore", "move",
            "tail_after_nonempty_flush", "flush_after_reset_streams_with_queue", "flush_uneven_queues", "tail_after_reset",
            "tail_after_restore", "mixed_silent_segment", "preload_N_multi_frame", "synth_crosses_chunk", "queue_overflow",
            "reset_streams_edge"}
    assert want <= seen, "not reached: %s" % sorted(want - seen)
    signals = {S.random_script(seed, N_STREAMS)[2] for seed in SEEDS}
    assert signals == {"speech", "square"}


def test_scripts_follow_the_contract():
    """No stream with queued frames is exported, and no tail runs between an import and the next synth / net."""
    for seed in SEEDS:
        fill, no_tail = [0] * N_STREAMS, False
        saved = None
        for op in S.random_script(seed, N_STREAMS)[0]:
            if op[0] == "defer":
                fill = [min(4, v + 1) for v in fill]
            elif op[0] == "flush":
                fill = [0] * N_STREAMS
            elif op[0] == "reset":
                fill, no_tail = [0] * N_STREAMS, False
            elif op[0] == "reset_streams":
                for s in op[1]:
                    fill[s] = 0
            elif op[0] == "move":
                assert fill[op[1]] == 0
                fill[op[2]] = 0
                no_tail = True
            elif op[0] in ("synth", "net"):
                no_tail = False
            elif op[0] == "tail":
                assert not no_tail, "seed %d: tail after an import" % seed
            elif op[0] == "save":
                saved = (list(fill), no_tail)
            elif op[0] == "restore":
                fill, no_tail = list(saved[0]), saved[1]


@pytest.fixture(scope="module")
def pool():
    with ThreadPoolExecutor(N_STREAMS) as p:
        yield p


@pytest.mark.parametrize("build,tag", CASES)
def test_random_sequences_match_reference(build, tag, pool):
    kind = "float" if build == "B" else "int8"
    for seed in SEEDS:
        script, f, streams = seq_inputs(seed)
        got = S.run_streams("oracle", H.oracle_lib(), S.OracleState(kind, tag), f, streams, script, pool)
        want = H.ref_digest(seq_key(build, tag, seed),
                            lambda: S.run_streams("ref", H.ref_lib(build, tag), S.RefState(build, tag), f, streams, script, pool))
        assert H.digest(got) == want, "seed %d: %s" % (seed, script[0])
        assert np.abs(got).max() > 0


@pytest.mark.parametrize("build,tag", [("A", ""), ("A", "delay1"), ("B", "")])
def test_tail_after_flush_keeps_the_last_conditioning(build, tag):
    """synth x5, run_frame_network, two deferred frames, flush, tail: the reference's flush evaluates the queue into local
    arrays (lpcnet.c:134-144), so the tail still uses the conditioning and LPC of run_frame_network."""
    kind = "float" if build == "B" else "int8"
    f = make_features(7, 8)[None]
    script = ([("synth", 0, 5, 160, 0), ("net", 5, 1), ("defer", 6), ("defer", 7), ("flush",), ("tail", 160, 0)], 8, "speech")
    got = S.run_streams("oracle", H.oracle_lib(), S.OracleState(kind, tag), f, [7], script)
    want = H.ref_digest("seq_%s_%s_flush_tail" % (build, tag),
                        lambda: S.run_streams("ref", H.ref_lib(build, tag), S.RefState(build, tag), f, [7], script))
    assert H.digest(got) == want
    assert np.abs(got[0, 800:]).max() > 0
