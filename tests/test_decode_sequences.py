"""CPU tests: lpcnet_decode the way synthesis is checked.  Seeded random call sequences that mix decodes with the synthesis entry
points and the lifecycle operations (scenarios.random_script(..., decode=True)), run per stream by the CPU restatement and by the
compiled reference on its decoder state (LPCNetDecState), and whole-stream decode of every model variant in both flavours.  The
reference's PCM is pinned by digests in tests/golden/ref_digests.json (keys seqdec_<build>_<tag>_<seed> and decode_<tag>_<build>),
so the comparison also runs where no reference is compiled.  tests/test_gpu_decode.py runs the same inputs on the engine.

A reset clears the decoder's memory of the previous superframe (vq_mem), as lpcnet_decoder_init does: a reset stream starts a new
utterance.  reset_signal keeps it, and state copies carry it."""
from concurrent.futures import ThreadPoolExecutor
import os
import numpy as np
import pytest
import gen_model
import helpers as H
import scenarios as S
from fixtures import make_feature_batch, make_packets, make_pcm

SEEDS = range(2032, 2038)
N_STREAMS = 3
CASES = [("A", ""), ("A", "na128"), ("A", "na256e2e"), ("A", "delay0"), ("A", "delay1"), ("B", ""), ("B", "delay1")]
TAGS = [""] + list(gen_model.VARIANTS)
DEC_SHIM = ("ref_dec_state_create", "ref_dec_state_destroy", "ref_decode", "ref_dec_reset", "ref_dec_state_copy")


def seq_streams(seed):
    return [700 + 10 * (seed % 100) + i for i in range(N_STREAMS)]


def seq_inputs(seed):
    """(script, features [n][T][20], stream ids) of one decode seed of this file."""
    script = S.random_script(seed, N_STREAMS, decode=True)
    streams = seq_streams(seed)
    return script, make_feature_batch(streams, max(script[1], 1)), streams


def seq_key(build, tag, seed):
    return "seqdec_%s_%s_%d" % (build, tag, seed)


def decode_inputs():
    """Packets [5][12][8] of the whole-stream decode test: three streams of random packets, two of packets the encoder made from
    speech (consecutive packets belong together, so the interpolations against vq_mem see real trajectories)."""
    rnd = [make_packets(60 + s, 12) for s in range(3)]
    enc = [H.oracle_encode(make_pcm(70 + s, 48)[None])[0] for s in range(2)]
    return np.stack(rnd + enc)


def decode_key(tag, build):
    return "decode_%s_%s" % (tag, build)


def test_decode_seed_set_reaches_every_situation():
    seen, sources, signals = set(), set(), set()
    for seed in SEEDS:
        script = S.random_script(seed, N_STREAMS, decode=True)
        seen |= S.script_events(script, N_STREAMS)
        sources.add(script[3]); signals.add(script[2])
    want = {"decode", "decode_after_synth", "synth_after_decode", "tail_after_decode", "decode_with_queue", "flush_after_decode_with_queue",
            "decode_after_reset_streams", "decode_after_restore", "decode_after_move", "decode_crosses_chunk", "decode_after_reset_signal",
            "reset", "save", "restore", "move", "reset_streams", "reset_signal", "defer", "flush", "tail", "synth", "net"}
    assert want <= seen, "not reached: %s" % sorted(want - seen)
    assert sources == set(S.PACKET_SOURCES) and signals == {"speech", "square"}


def test_decode_scripts_follow_the_contract():
    """No stream with queued frames is exported, no tail runs between an import and the next synth / net / decode, and every
    decode reads packets the script's source has, in order."""
    for seed in SEEDS:
        script = S.random_script(seed, N_STREAMS, decode=True)
        fill, no_tail, nxt = [0] * N_STREAMS, False, 0
        for op in script[0]:
            if op[0] == "defer":
                fill = [min(4, v + 1) for v in fill]
            elif op[0] == "flush":
                fill = [0] * N_STREAMS
            elif op[0] in ("reset", "reset_streams"):
                for s in (op[1] if op[0] == "reset_streams" else range(N_STREAMS)):
                    fill[s] = 0
                no_tail = no_tail and op[0] == "reset_streams"
            elif op[0] == "move":
                assert fill[op[1]] == 0
                fill[op[2]] = 0
                no_tail = True
            elif op[0] in ("synth", "net", "decode"):
                no_tail = False
                if op[0] == "decode":
                    assert op[1] == nxt and 1 <= op[2] <= 6
                    nxt += op[2]
            elif op[0] == "tail":
                assert not no_tail, "seed %d: tail after an import" % seed
            elif op[0] == "save":
                saved = (list(fill), no_tail)
            elif op[0] == "restore":
                fill, no_tail = list(saved[0]), saved[1]
        assert S.script_packets(script, seq_streams(seed)).shape == (N_STREAMS, nxt, 8)


def test_every_variant_has_the_same_codebooks():
    """The restatement of every variant and the engine's tests load the default model's codebooks.bin, while each variant's
    reference build compiles its own generated ceps_codebooks.c: they must be the same codebooks."""
    want = open(os.path.join(H.gen_dir(), "codebooks.bin"), "rb").read()
    assert len(want) == 4 * (3 * 1024 * 17 + 4096 * 18)
    for tag in gen_model.VARIANTS:
        assert open(os.path.join(H.gen_dir(tag), "codebooks.bin"), "rb").read() == want, tag


@pytest.fixture(scope="module")
def pool():
    with ThreadPoolExecutor(N_STREAMS) as p:
        yield p


@pytest.mark.parametrize("build,tag", CASES)
def test_decode_sequences_match_reference(build, tag, pool):
    kind = "float" if build == "B" else "int8"
    for seed in SEEDS:
        script, f, streams = seq_inputs(seed)
        got = S.run_streams("oracle", H.oracle_lib(), S.OracleState(kind, tag), f, streams, script, pool)
        want = H.ref_digest(seq_key(build, tag, seed),
                            lambda: S.run_streams("ref", H.ref_lib(build, tag), S.RefDecState(build, tag), f, streams, script, pool),
                            runnable=H.ref_has(build, tag, *DEC_SHIM))
        assert H.digest(got) == want, "seed %d: %s" % (seed, script[0])
        assert np.abs(got).max() > 0


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("build", ["A", "B"])
def test_whole_stream_decode_matches_reference(build, tag):
    kind = "float" if build == "B" else "int8"
    pk = decode_inputs()
    got = H.oracle_decode(pk, kind, tag=tag)
    assert H.digest(got) == H.ref_digest(decode_key(tag, build), lambda: H.ref_decode(pk, build, tag))
    assert (np.abs(got[:, 640:]).max(axis=1) > 0).all()
