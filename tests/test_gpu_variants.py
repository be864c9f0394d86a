"""GPU parity for other model shapes and switches (-m gpu; SURVEY.md 8f N1): GRU_A with 256 / 128 units, END2END (LPC from the
network's reflection coefficients, lpcnet.c:57-78,107-108), FEATURES_DELAY 0 (lpcnet.c:113-115), int8 and float flavours.
Goldens: the reference compiled with each variant's generated nnet_data.h (tests/golden/variants.npz, make_golden.py);
wider / ragged batches against the CPU restatement, which the CPU suite pins to the same goldens."""
import os
import numpy as np
import pytest
import helpers as H
from fixtures import make_feature_batch

pytestmark = pytest.mark.gpu
TAGS = ["na256", "na128", "e2e", "delay0", "na256e2e", "delay1"]


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


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("kind,build", [("int8", "A"), ("float", "B")])
def test_variant_matches_reference_golden(eng, tag, kind, build):
    gold = np.load(os.path.join(H.GOLDEN, "variants.npz"))["%s_%s" % (tag, build)]
    b = eng.Batch(2, H.blob(kind, tag), config=H.model_config(tag))
    assert b.na == {"na256": 256, "na128": 128, "na256e2e": 256}.get(tag, 384) and b.config[1:] == tuple(int(x) for x in H.model_config(tag)[1:])
    got = b.synthesize(make_feature_batch(range(2), 20))
    b.close()
    assert _first_diff(got, gold) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, gold),)


# streams per CTA of each case, pinned: on its own a batch this small is spread over the SMs one stream per CTA
VARIANT_SPC = {("int8", 70): "32", ("float", 37): "32"}


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("kind,n", [("int8", 70), ("int8", 9), ("float", 37), ("float", 3)])
def test_variant_batches_match_oracle(eng, monkeypatch, tag, kind, n):
    """int8: 70 streams at 32 per CTA (two halves; CTAs of 32, 32 and 6) and 9 on the automatic schedule (one half, one live
    slot per CTA); float: 37 streams at 32 per CTA (the lane==stream kernel, a ragged CTA of 5) and 3 on the automatic schedule
    (the neuron-per-lane kernel)"""
    if (kind, n) in VARIANT_SPC:
        monkeypatch.setenv("LPCNET_B200_STREAMS_PER_CTA", VARIANT_SPC[(kind, n)])
    T = 9
    f = make_feature_batch(range(400, 400 + n), T)
    b = eng.Batch(n, H.blob(kind, tag), config=H.model_config(tag))
    got = np.concatenate([b.synthesize(f[:, :4]), b.synthesize(f[:, 4:])], axis=1)     # state carried across calls
    b.close()
    want = H.oracle_synth(f, kind, tag=tag)
    assert _first_diff(got, want) is None, "first mismatch (stream, sample) = %s" % (_first_diff(got, want),)


def test_variant_frame_network_taps(eng):
    """conditioning + LPC of an END2END / FEATURES_DELAY 0 / 256-unit model, bit-compared with the oracle per frame"""
    tag, n, T = "na256e2e", 5, 6
    f = make_feature_batch(range(30, 30 + n), T)
    b = eng.Batch(n, H.blob("int8", tag), config=H.model_config(tag))
    ga, gb, lpc = b.debug_frame_network(f)
    b.close()
    L = H.oracle_lib()
    for s in range(n):
        st = L.oracle_state_create(H.oracle_model("int8", tag))
        for t in range(T):
            a = np.zeros(3 * 256, np.float32); c = np.zeros(48, np.float32); l = np.zeros(16, np.float32)
            L.oracle_frame_network(st, f[s, t].ctypes.data, a.ctypes.data, c.ctypes.data, l.ctypes.data)
            np.testing.assert_array_equal(ga[s, t].view(np.uint32), a.view(np.uint32))
            np.testing.assert_array_equal(gb[s, t].view(np.uint32), c.view(np.uint32))
            np.testing.assert_array_equal(lpc[s, t].view(np.uint32), l.view(np.uint32))
        L.oracle_state_destroy(st)


def test_blob_metadata_record_selects_the_switches(eng):
    """A blob that carries the `lpcnet_b200_config` record needs no out-of-band LPC_GAMMA / FEATURES_DELAY / END2END."""
    import struct
    tag = "na256e2e"
    gamma, delay, e2e = H.model_config(tag)
    payload = struct.pack("<4f", gamma, delay, float(e2e), 1.0)
    rec = struct.pack("<4siiii44s", b"DNNw", 0, 0, len(payload), 64, b"lpcnet_b200_config") + payload + b"\0" * (64 - len(payload))
    f = make_feature_batch(range(2), 20)
    b = eng.Batch(2, H.blob("int8", tag) + rec, lpc_gamma=-1.0)       # <= 0: not given
    assert b.config == (np.float32(gamma), delay, int(e2e))
    got = b.synthesize(f)
    b.close()
    np.testing.assert_array_equal(got, np.load(os.path.join(H.GOLDEN, "variants.npz"))["%s_A" % tag])


def test_unsupported_size_is_refused_with_a_message(eng):
    import gen_model, tempfile
    d = tempfile.mkdtemp()
    gen_model.generate(d, c_sources=False, na=192)
    blob = open(os.path.join(d, "model_int8.bin"), "rb").read()
    with pytest.raises(eng.LPCNetB200Error, match="192 units"):
        eng.Batch(1, blob)
