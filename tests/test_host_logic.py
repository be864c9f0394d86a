"""CPU tests (-m "not gpu") of the product's HOST logic: library loading, C-ABI surface, blob validation and the
shared-memory image the per-sample kernel consumes (checked by replaying the kernel's block walk in numpy against
a dense reconstruction of the model).  No compute entry point is called: without a GPU the engine must refuse."""
import os
import re
import pytest
import helpers as H
import image_replay as R
import lpcnet_b200
from lpcnet_b200 import api

ROOT = H.ROOT


@pytest.fixture(scope="module")
def L():
    from lpcnet_b200 import build
    build.build()
    return api.lib()


def _declared_symbols():
    syms = []
    for hdr in ("lpcnet.h", "lpcnet_b200.h"):
        txt = open(os.path.join(ROOT, "include", hdr)).read()
        txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
        syms += re.findall(r"LPCNET_EXPORT[^;(#]*?\b(lpcnet\w*)\s*\(", txt)
    return sorted(set(syms))


def test_library_exports_every_declared_symbol(L):
    syms = _declared_symbols()
    assert "lpcnet_synthesize" in syms and "lpcnet_decode" in syms and "lpcnet_b200_batch_synthesize" in syms
    assert len(syms) >= 25
    for s in syms:
        assert hasattr(L, s), "missing export " + s


def test_no_cpu_fallback_without_gpu(L):
    if L.lpcnet_b200_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(api.LPCNetB200Error, match="no CUDA device"):
        lpcnet_b200.Batch(4, H.blob("int8"))
    assert not L.lpcnet_create()
    assert not L.lpcnet_decoder_create()


_image = R.int8_image


def test_blob_validation(L):
    b = H.blob("int8")
    r, _, _ = _image(L, b)
    assert r > 0
    assert _image(L, b[:-100])[0] < 0                       # truncated record (parse_lpcnet_weights.c:40)
    bad = bytearray(b); bad[12:16] = (10 ** 9).to_bytes(4, "little")   # size > block_size
    assert _image(L, bytes(bad))[0] < 0
    assert _image(L, b"")[0] < 0
    assert _image(L, b[: 64 * 1000])[0] < 0                 # cut mid-way: arrays missing
    assert _image(L, H.blob("float"))[0] > 0                # float flavour (fp16-exact weights) is accepted


def test_smem_image_replays_to_the_dense_model(L):
    """Walk the image exactly like the kernel (warp -> slot -> gate -> list of quads = MMA operands; (row group, K half)
    for GRU_B) and check the integer GEMV it encodes equals the dense int8 matrices of the model for random u8 inputs."""
    import gen_model
    common, only8, _ = gen_model.make_model()
    s = R.replay_int8_image(L, H.blob("int8"), {n: a for n, _, a in common + only8})
    loads, nA = s["loads"], s["nA"]
    # LPT balancing of the compute warps: the warps that also walk the GRU_B GEMV (first 12) and / or finish GRU_B (last 8) get lighter
    # GRU_A lists (model.cu), so the quad counts differ by class but stay within +-35 % of the mean
    assert max(loads) <= 1.35 * (nA / s["nwc"]) and min(loads) >= 0.65 * (nA / s["nwc"])
    assert s["clashes"] <= 0.15 * 4 * nA                                  # slots of a quad mostly in different bank groups
    assert s["clashesB"] == 0                                             # dense rows: always conflict-free
    assert s["fcw_nodes"] == 64 and s["fast_cvt"] == 1


def test_denser_model_trades_dual_fc_rows_for_weight_room(L, tmp_path, monkeypatch):
    """The int8 image is sized for the default 5/5/20 % block densities with 64 dual_fc rows in shared memory; a model
    with more blocks must still load (fewer dual_fc rows kept, the sampler reads the others from L2) until the weights
    themselves no longer fit, which is refused with a message."""
    import gen_model
    def image_for(density):
        monkeypatch.setattr(gen_model, "DENSITY", density)
        common, only8, _ = gen_model.make_model()
        path = str(tmp_path / "m.bin")
        gen_model.write_blob(path, common + only8)
        return _image(L, open(path, "rb").read())
    r, img, lay = image_for((0.05, 0.05, 0.20))
    assert r > 0 and int(lay[18]) == 64 and int(lay[5]) <= 227 * 1024
    r, img, lay = image_for((0.06, 0.06, 0.22))
    assert r > 0 and int(lay[18]) in (8, 16, 32) and int(lay[5]) <= 227 * 1024
    r, img, lay = image_for((0.15, 0.15, 0.40))
    assert r < 0 and b"shared memory" in L.lpcnet_b200_last_error()


def test_float_neuron_image_replays_to_the_dense_model(L):
    """Image of the neuron-per-lane float kernel: every compute lane owns one neuron, the fp16 blocks are transposed to
    [8 rows][4 cols]; walking it like the kernel must reproduce the dense float matrices (the weights are fp16-exact)."""
    import gen_model
    common, _, onlyf = gen_model.make_model()
    s = R.replay_float_image(L, H.blob("float"), {n: a for n, _, a in common + onlyf})
    assert s["dense"] == 1 and s["chains"] == ["dense", "dense"]         # dense GRU_B input rows, in order


def test_python_mirror_matches_reference_operator_names():
    for name in ("LPCNet", "LPCNetDecoder", "Batch"):
        assert hasattr(lpcnet_b200, name)
    for m in ("load_model", "synthesize", "reset"):
        assert hasattr(lpcnet_b200.LPCNet, m)
    assert hasattr(lpcnet_b200.LPCNetDecoder, "decode")


@pytest.mark.parametrize("tag,na", [("na128", 128), ("na256", 256), ("na256e2e", 256), ("", 384)])
def test_images_of_all_gru_a_sizes_respect_the_kernel_budgets(L, tag, na):
    """Every supported GRU_A size builds a shared-memory image that fits one SM and replays to the dense model; every neuron group
    is owned by exactly one compute warp; and the quad arrays are followed by the readable slack that the pipelined GEMVs of
    sample_kernel.cu read past the end of a stream (4 quads of weights, 6 meta entries)."""
    import gen_model
    common, only8, _ = gen_model.make_model(na=na)
    R.replay_int8_image(L, H.blob("int8", tag), {n: a for n, _, a in common + only8}, na=na)
