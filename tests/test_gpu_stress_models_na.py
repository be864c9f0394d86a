"""GPU tests (-m gpu) of the 128- and 256-unit per-sample kernels on the stress models (checked on the CPU by
test_stress_models_na.py): bit for bit against the CPU restatement, and against the digests of the compiled reference where the
inputs are its.  Each GRU_A size is a kernel of its own (one neuron group per compute warp at 128, two at 256), and every
schedule is pinned here instead of being left to the batch size and the SM count:
  int8   automatic (one half, one live slot per CTA), 32 streams per CTA (two halves, full and ragged CTAs), 17 (the smallest
         two-half CTA: 9 + 8 rows), 16 (the largest one-half CTA, tile rows 0-15 live, those the sampler's GRU_B state shares),
         5 with both halves forced (3 + 2 rows: dead slots in both halves); the loader's rounding and the conversion unit
  float  the neuron-per-lane kernel with 1, 2 and 3 streams per CTA, the lane==stream kernel"""
import json
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch, make_packets
from test_stress_models import STRESS_FEATURES
from test_stress_models_na import LOADED_NA, FLOAT_NA, ref_key_na

pytestmark = pytest.mark.gpu

IDS = range(300, 307)          # STRESS_FEATURES' streams and one more; first 6 streams = the reference digest
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


def _ref_digest(na, name, build):
    return json.load(open(H.REF_DIGESTS))[ref_key_na(na, name, build)]


def _run(eng, blob, f, calls, na):
    b = eng.Batch(f.shape[0], blob, lpc_gamma=H.LPC_GAMMA)
    assert b.na == na
    t, out = 0, []
    for k in calls:
        out.append(b.synthesize(f[:, t:t + k])); t += k
    b.close()
    assert t == f.shape[1]
    return np.concatenate(out, axis=1)


@pytest.mark.parametrize("exact", ["0", "1"])
@pytest.mark.parametrize("na,name", LOADED_NA)
def test_int8_stress_na_small_batch_in_chunks(eng, monkeypatch, na, name, exact):
    """7 streams on the automatic schedule (one half, one live slot per CTA), 12 frames in calls of 4+5+3, with the loader's
    choice of rounding and with the conversion unit forced: equal to the oracle and to the compiled reference."""
    assert list(IDS[:6]) == list(STRESS_FEATURES[0]) and T == STRESS_FEATURES[1]
    if exact == "1":
        monkeypatch.setenv("LPCNET_B200_EXACT_CVT", "1")
    blob = H.stress_blob(name, "int8", na)
    f = make_feature_batch(IDS, T)
    got = _run(eng, blob, f, (4, 5, 3), na)
    _check(got, H.oracle_synth(f, "int8", model_blob=blob), (na, name))
    assert H.digest(got[:6]) == _ref_digest(na, name, "A")


# (streams per CTA, LPCNET_B200_TWO_HALVES, streams, frames per call)
SCHEDULES = [
    ("32", None, 70, (4, 2)),        # two halves; CTAs of 32, 32 and 6 streams
    ("17", None, 40, (18, 2)),       # smallest two-half CTA (CTAs of 17, 17, 6); an 18-frame call crosses the 16-frame chunk
    ("16", None, 40, (18, 2)),       # largest one-half CTA (16, 16, 8)
    ("5", "1", 12, (4, 2)),          # both halves forced at 5 streams per CTA: 3 + 2 live rows (5, 5, 2)
]


@pytest.mark.parametrize("spc,two,n,calls", SCHEDULES, ids=["spc32", "spc17", "spc16", "spc5-two-halves"])
@pytest.mark.parametrize("na,name", LOADED_NA)
def test_int8_stress_na_schedules(eng, monkeypatch, na, name, spc, two, n, calls):
    """The int8 kernel under each pinned schedule, ragged last CTA, state carried across calls: equal to the oracle."""
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", spc)
    if two:
        monkeypatch.setenv("LPCNET_B200_TWO_HALVES", two)
    blob = H.stress_blob(name, "int8", na)
    f = make_feature_batch(range(500, 500 + n), sum(calls))
    _check(_run(eng, blob, f, calls, na), H.oracle_synth(f, "int8", model_blob=blob), (na, name, spc))


@pytest.mark.parametrize("na,name", LOADED_NA)
def test_int8_stress_na_batch_decode(eng, na, name):
    """lpcnet_b200_batch_decode (packets -> features -> PCM) of 3 streams x 3 packets against the oracle's decode."""
    blob = H.stress_blob(name, "int8", na)
    pk = np.stack([make_packets(s, 3) for s in range(60, 63)])
    b = eng.Batch(3, blob, lpc_gamma=H.LPC_GAMMA, codebooks=H.codebooks())
    got = b.decode(pk)
    b.close()
    _check(got, H.oracle_decode(pk, "int8", model_blob=blob), (na, name))


@pytest.mark.parametrize("spc,lane", [("1", None), ("2", None), ("3", None), ("3", "1"), ("32", None)],
                         ids=["spc1", "spc2", "spc3", "spc3-lane-stream", "spc32"])
@pytest.mark.parametrize("na,name", FLOAT_NA)
def test_float_stress_na_kernels(eng, monkeypatch, na, name, spc, lane):
    """Float flavour: the neuron-per-lane kernel with 1, 2 and 3 streams per CTA (ragged last CTA) and the lane==stream kernel
    (32 streams per CTA, and 3 with LPCNET_B200_FLOAT_LANE_STREAM), 7 streams, 12 frames in calls of 8+4: equal to the float
    oracle and to the compiled reference build B."""
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", spc)
    if lane:
        monkeypatch.setenv("LPCNET_B200_FLOAT_LANE_STREAM", lane)
    blob = H.stress_blob(name, "float", na)
    f = make_feature_batch(IDS, T)
    got = _run(eng, blob, f, (8, 4), na)
    _check(got, H.oracle_synth(f, "float", model_blob=blob), (na, name, spc))
    assert H.digest(got[:6]) == _ref_digest(na, name, "B")


@pytest.mark.parametrize("fcw", ["8", "32"])
def test_int8_reduced_dual_fc_rows_na256(eng, monkeypatch, fcw):
    """The sampler with 8 and 32 dual_fc rows in shared memory at 256 units (the loader's choice for "full" is 32), 7 streams
    on the automatic schedule and 40 at 32 streams per CTA: equal to the oracle."""
    monkeypatch.setenv("LPCNET_B200_FCW_NODES", fcw)
    blob = H.stress_blob("skew", "int8", 256)
    f = make_feature_batch(IDS, T)
    _check(_run(eng, blob, f, (4, 5, 3), 256), H.oracle_synth(f, "int8", model_blob=blob), fcw)
    monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", "32")
    f = make_feature_batch(range(500, 540), 6)
    _check(_run(eng, blob, f, (4, 2), 256), H.oracle_synth(f, "int8", model_blob=blob), fcw)
