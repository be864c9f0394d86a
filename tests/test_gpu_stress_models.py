"""GPU tests (-m gpu) of the per-sample kernels on the stress models (oracle/gen_model.py STRESS, checked on the CPU by
test_stress_models.py): bit for bit against the CPU restatement, and against the digests of the compiled reference.  The models
reach kernel paths the default model does not: the sparse and the non-uniform GRU_B chains of the neuron-per-lane float kernel,
empty and partial int8 GRU_B K parts, skewed GRU_A lists with forced repeats of a bank-group class, a full image with fewer
dual_fc rows in shared memory, int8 weights at the loader's limit and the largest accumulators the conversion-free rounding
allows (and the conversion-unit path chosen by the loader just past that)."""
import json
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets
from test_stress_models import LOADED, STRESS_FEATURES, ref_key

pytestmark = pytest.mark.gpu

IDS = range(300, 307)          # STRESS_FEATURES' streams and one more (a ragged last CTA); first 6 streams = the reference digest
T = 12


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


def _first_diff(a, b):
    d = np.argwhere(a != b)
    return None if d.size == 0 else tuple(d[0])


def _check(got, want, what):
    assert got.shape == want.shape
    assert _first_diff(got, want) is None, "%s: first mismatch (stream, sample) = %s" % (what, _first_diff(got, want))


def _ref_digest(name, build):
    return json.load(open(H.REF_DIGESTS))[ref_key(name, build)]


@pytest.mark.parametrize("exact", ["0", "1"])
@pytest.mark.parametrize("name", LOADED)
def test_int8_stress_small_batch_in_chunks(eng, monkeypatch, name, exact):
    """7 streams (one half only), 12 frames in calls of 4+5+3 (state carried), with the loader's choice of rounding and with the
    conversion unit forced (LPCNET_B200_EXACT_CVT): equal to the oracle and to the compiled reference."""
    assert list(IDS[:6]) == list(STRESS_FEATURES[0]) and T == STRESS_FEATURES[1]
    if exact == "1":
        monkeypatch.setenv("LPCNET_B200_EXACT_CVT", "1")
    blob = H.stress_blob(name, "int8")
    f = make_feature_batch(IDS, T)
    b = eng.Batch(len(IDS), blob, lpc_gamma=H.LPC_GAMMA)
    got = np.concatenate([b.synthesize(f[:, 0:4]), b.synthesize(f[:, 4:9]), b.synthesize(f[:, 9:12])], axis=1)
    b.close()
    _check(got, H.oracle_synth(f, "int8", model_blob=blob), name)
    assert H.digest(got[:6]) == _ref_digest(name, "A")


@pytest.mark.parametrize("name", LOADED)
def test_int8_stress_two_halves_ragged(eng, monkeypatch, name):
    """70 streams in 32-slot CTAs (two full, one of 6): the two-half schedule with dead slots, state carried over two calls."""
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", "32")
    blob = H.stress_blob(name, "int8")
    n, TT = 70, 6
    f = make_feature_batch(range(500, 500 + n), TT)
    b = eng.Batch(n, blob, lpc_gamma=H.LPC_GAMMA)
    got = np.concatenate([b.synthesize(f[:, :4]), b.synthesize(f[:, 4:])], axis=1)
    b.close()
    _check(got, H.oracle_synth(f, "int8", model_blob=blob), name)


@pytest.mark.parametrize("name", LOADED)
def test_int8_stress_batch_decode(eng, name):
    """lpcnet_b200_batch_decode (packets -> features -> PCM) of 3 streams x 3 packets against the oracle's decode."""
    blob = H.stress_blob(name, "int8")
    pk = np.stack([make_packets(s, 3) for s in range(60, 63)])
    b = eng.Batch(3, blob, lpc_gamma=H.LPC_GAMMA, codebooks=H.codebooks())
    got = b.decode(pk)
    b.close()
    _check(got, H.oracle_decode(pk, "int8", model_blob=blob), name)


@pytest.mark.parametrize("spc", ["1", "2", "3", "32"])
@pytest.mark.parametrize("name", LOADED)
def test_float_stress_kernels(eng, monkeypatch, name, spc):
    """Float flavour: the neuron-per-lane kernel with 1, 2 and 3 streams per CTA (ragged last CTA) and the lane==stream kernel
    (32), 7 streams, 12 frames in calls of 8+4: equal to the float oracle and to the compiled reference build B."""
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", spc)
    blob = H.stress_blob(name, "float")
    f = make_feature_batch(IDS, T)
    b = eng.Batch(len(IDS), blob, lpc_gamma=H.LPC_GAMMA)
    got = np.concatenate([b.synthesize(f[:, :8]), b.synthesize(f[:, 8:])], axis=1)
    b.close()
    _check(got, H.oracle_synth(f, "float", model_blob=blob), name)
    assert H.digest(got[:6]) == _ref_digest(name, "B")
