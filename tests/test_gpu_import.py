"""GPU side of real-model entry (-m gpu): blobs that tools/import_nnet_data.py made from models in the nnet_data.c / nnet_data.h
form (oracle/dump_nnet_data.py) run bit-exact against the reference built from the same nnet_data.c with the arrays compiled
in (its digests, tests/test_import_nnet_data.py) and against the CPU restatement.  No switch is passed: the blob's config
record must supply LPC_GAMMA, FEATURES_DELAY and END2END.  Batches stay small; the kernels' geometries are covered elsewhere."""
import numpy as np
import pytest

import helpers as H
from test_import_nnet_data import BUILD, KINDS, MODELS, features, packets

pytestmark = pytest.mark.gpu

DROP_IN = ["default", "gamma085", "na256", "na128", "na256e2e", "delay1"]


@pytest.fixture(scope="module")
def eng():
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    assert lpcnet_b200.device_count() > 0, "GPU test selected but no CUDA device is visible"
    return lpcnet_b200


def _refused(model, kind):
    """Blobs the loader refuses, imported or generated: the int8 `overflow` stress model (its accumulator bound leaves int32)
    and the float `full` one (its fp16 image does not fit in one SM's shared memory)."""
    return (kind == "int8" and model.startswith("stress_overflow")) or (kind == "float" and model.startswith("stress_full"))


def _first_diff(a, b):
    d = np.argwhere(a != b)
    return None if d.size == 0 else tuple(d[0])


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("model", MODELS)
def test_imported_blob_synthesizes_like_the_reference(eng, model, kind):
    """3 streams, 8 frames in two calls of 3 and 5 (state carried across calls)."""
    blob, _, _ = H.imported(model, kind)
    if _refused(model, kind):
        with pytest.raises(eng.LPCNetB200Error, match="int32|more than one SM offers"):
            eng.Batch(3, blob)
        return
    b = eng.Batch(3, blob)
    assert b.config == eng.blob_config(blob)
    f = features()
    got = np.concatenate([b.synthesize(f[:, :3]), b.synthesize(f[:, 3:])], axis=1)
    b.close()
    want = H.oracle_with_config(blob, eng.blob_config(blob), features=f)
    assert _first_diff(got, want) is None, "first mismatch with the oracle (stream, sample) = %s" % (_first_diff(got, want),)
    assert H.digest(got) == H.ref_digest("dump_%s_%s_synth" % (model, BUILD[kind]), lambda: H.dump_ref_synth(model, BUILD[kind], f),
                                         runnable=H.have_dump_ref(model))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("model", MODELS)
def test_imported_blob_decodes_like_the_reference(eng, model, kind):
    """2 streams, 3 packets each."""
    if _refused(model, kind):
        pytest.skip("the int8 blob is refused (see the synthesis test)")
    blob, _, _ = H.imported(model, kind)
    b = eng.Batch(2, blob, codebooks=H.codebooks())
    p = packets()
    got = b.decode(p)
    b.close()
    want = H.oracle_with_config(blob, eng.blob_config(blob), packets=p)
    assert _first_diff(got, want) is None, "first mismatch with the oracle (stream, sample) = %s" % (_first_diff(got, want),)
    assert H.digest(got) == H.ref_digest("dump_%s_%s_decode" % (model, BUILD[kind]), lambda: H.dump_ref_decode(model, BUILD[kind], p),
                                         runnable=H.have_dump_ref(model))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("model", DROP_IN)
def test_drop_in_api_loads_the_imported_blob(eng, model, kind):
    """lpcnet_load_model with the imported blob, then lpcnet_synthesize frame by frame: the batch's (= the reference's) PCM."""
    blob, _, _ = H.imported(model, kind)
    f = features()[:1]
    st = eng.LPCNet(blob)
    got = np.concatenate([st.synthesize(f[0, t]) for t in range(f.shape[1])])
    st.close()
    want = H.oracle_with_config(blob, eng.blob_config(blob), features=f)[0]
    assert _first_diff(got, want) is None, "first mismatch at sample %s" % (_first_diff(got, want),)
