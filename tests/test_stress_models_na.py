"""CPU tests (-m "not gpu") of the stress models (oracle/gen_model.py STRESS) at 128 and 256 GRU_A units.  The per-sample kernels
are compiled once per GRU_A size, and the smaller sizes have their own geometry: one neuron group per compute warp at 128 (so
the LPT assignment cannot pair an empty group with a full one, and a group empty in all three gates leaves a warp with no GRU_A
quad to walk), 32 / 64 column blocks, an 8- / 16-block K part for a dense GRU_B row.  Checked here, as test_stress_models.py
does at 384: each fixture's structure at the smaller width, the images the kernels consume, the loader's verdicts, and the
CPU restatement against the compiled reference builds of the na128 / na256 headers."""
import hashlib
import json
import os
import numpy as np
import pytest
import gen_model as G
import helpers as H
import image_replay as R
from fixtures import make_feature_batch
from test_stress_models import STRESS_FEATURES, _lists, _pairs

WIDTHS = [128, 256]
MODELS = [(na, n) for na in WIDTHS for n in G.stress_names(na)]       # (width, stress model): every STRESS model, and "full" at 256
LOADED_NA = [(na, n) for na, n in MODELS if n != "overflow"]           # the int8 blob of "overflow" is refused by the loader
FLOAT_NA = [(na, n) for na, n in LOADED_NA if n != "full"]             # the fp16 image of "full" does not fit in shared memory
STRESS_NA_GOLDEN = os.path.join(H.GOLDEN, "stress_models_na.json")


@pytest.fixture(scope="module")
def L():
    from lpcnet_b200 import build, api
    build.build()
    return api.lib()


def _countsA(L, blob):
    """Quads per (compute warp, slot, gate) of the int8 image: the dirA counts the kernel's GRU_A walkers take."""
    r, img, lay = R.int8_image(L, blob)
    assert r > 0
    DIRA, NWC, GPW = int(lay[10]), int(lay[16]), int(lay[17])
    return img[DIRA:DIRA + NWC * GPW * 3 * 2 * 4].view(np.uint32).reshape(NWC, GPW, 3, 2)[..., 1]


def test_stress_na_blobs_are_deterministic():
    want = json.load(open(STRESS_NA_GOLDEN))
    assert sorted(want) == sorted("na%d_%s_%s_sha256" % (na, n, k) for na, n in MODELS for k in ("int8", "float"))
    for na, name in MODELS:
        for kind in ("int8", "float"):
            assert hashlib.sha256(H.stress_blob(name, kind, na)).hexdigest() == want["na%d_%s_%s_sha256" % (na, name, kind)], (na, name, kind)


@pytest.mark.parametrize("na,name", MODELS)
def test_stress_na_model_has_its_structure(na, name):
    """Each fixture keeps, at the smaller width, the property it exists for."""
    a8, af = G.stress_arrays(name, "int8", na), G.stress_arrays(name, "float", na)
    np.testing.assert_array_equal(np.asarray(af["sparse_gru_a_recurrent_weights"], np.float64) * 128,
                                  np.asarray(a8["sparse_gru_a_recurrent_weights"], np.int8).reshape(-1, 8, 4).transpose(0, 2, 1).reshape(-1))
    np.testing.assert_array_equal(np.asarray(af["gru_b_weights"], np.float64) * 128,
                                  np.asarray(a8["gru_b_weights"], np.int8).reshape(-1, 8, 4).transpose(0, 2, 1).reshape(-1))
    la = _lists(a8, "sparse_gru_a_recurrent_weights_idx", 3 * na)
    lb = _lists(a8, "gru_b_weights_idx", 48)
    nb = [len(x) for x in lb]
    ngrp = na // 8
    same_sign = lambda p: (np.sign(p[:, 0]) * np.sign(p[:, 1]) >= 0)
    for arr in ("sparse_gru_a_recurrent_weights", "gru_b_weights", "gru_b_recurrent_weights"):   # what the loader accepts
        p = _pairs(a8[arr])
        assert (np.abs(p).sum(axis=1)[same_sign(p)]).max() <= 128
    bound = G.cvt_bound(a8, na)
    if name == "grub_split":
        assert nb[4:] == [na // 4] * 2                                   # candidate rows dense
        assert max(nb[:4]) < na // 4 and len(set(nb[:4])) == 4            # update / reset rows sparse, unequal counts
        assert 1 in nb and 3 in nb                                       # int8 K parts: one empty, one a partial quad
    elif name == "grub_even":
        n = G.GRUB_EVEN_BLOCKS[na]
        assert nb == [n] * 6 and n < na // 4                              # all alike, not dense
        assert (n // 2) % 4 != 0 and ((n + 1) // 2) % 4 != 0              # both int8 K parts end in a partial quad
        assert all(x != list(range(0, na, 4))[:n] for x in lb)            # scattered, not the first blocks in order
    elif name == "skew":
        for gate in range(3):
            lists = la[gate * ngrp:(gate + 1) * ngrp]
            n = [len(x) for x in lists]
            assert [n[g] for g in (0, 6, 7)] == [0, 0, 0] and n[1:4] == [1, 2, 3]
            if ngrp > 16:                                                 # (at 128 units all 16 row groups are forced ones)
                assert max(n) >= 4 * np.mean(n)                           # skewed, not uniform
            assert len(lists[4]) == 8 and len({(p // 4) & 3 for p in lists[4]}) == 1 and max(lists[4]) < na
            assert all(na - 4 in lists[g] for g in [5] + list(range(8, 16)))
    elif name == "limits":
        for arr in ("sparse_gru_a_recurrent_weights", "gru_b_weights", "gru_b_recurrent_weights"):
            p = _pairs(a8[arr])
            assert (np.abs(p).sum(axis=1)[same_sign(p) & (p[:, 0] != 0) & (p[:, 1] != 0)] == 128).any(), arr
            assert (p == -128).any(), arr
            assert (((p[:, 0] == 127) & (p[:, 1] == -128)) | ((p[:, 0] == -128) & (p[:, 1] == 127))).any(), arr
    elif name == "warm":
        assert G.FAST_CVT_LIMIT * 0.995 < bound < G.FAST_CVT_LIMIT
    elif name == "hot":
        assert G.FAST_CVT_LIMIT < bound < G.FAST_CVT_LIMIT * 1.005
    elif name == "overflow":
        assert bound >= 2.0 ** 31
    elif name == "full":
        assert all(0.45 < len(sum(la[g * ngrp:(g + 1) * ngrp], [])) / (ngrp * na // 4) < 0.52 for g in range(3))
    if name not in ("warm", "hot", "overflow"):
        assert bound < G.FAST_CVT_LIMIT


def test_skew_at_128_leaves_a_warp_without_gru_a_work(L):
    """At 128 units each compute warp owns one neuron group, so a group empty in all three gates leaves its warp an empty quad
    stream for every GRU_A GEMV (the walker starts and ends on the image's slack); the default model never does."""
    cA = _countsA(L, H.stress_blob("skew", "int8", 128))
    assert cA.shape[1] == 1
    assert (cA.sum(axis=(1, 2)) == 0).sum() == 3                         # row groups 0, 6 and 7
    assert (_countsA(L, H.blob("int8", "na128")).sum(axis=(1, 2)) > 0).all()


@pytest.mark.parametrize("na,name", LOADED_NA)
def test_stress_na_int8_image_replays_to_the_dense_model(L, na, name):
    a8 = G.stress_arrays(name, "int8", na)
    s = R.replay_int8_image(L, H.stress_blob(name, "int8", na), a8, na=na)
    nb = [len(x) for x in _lists(a8, "gru_b_weights_idx", 48)]
    assert s["kparts"] == 2
    np.testing.assert_array_equal(s["partsB"], [[-(-((n + 1) // 2) // 4), -(-(n - (n + 1) // 2) // 4)] for n in nb])
    assert s["fast_cvt"] == (0 if name == "hot" else 1)
    assert s["fcw_nodes"] == (32 if name == "full" else 64)               # only "full" makes the loader give up dual_fc rows
    if name == "grub_split":
        assert (s["partsB"] == 0).any() and s["padB"] > 0                  # an empty K part; partial quads
    if name == "grub_even":
        assert s["padB"] == 6 * 2 * (4 - (G.GRUB_EVEN_BLOCKS[na] // 2) % 4)   # every K part ends in a partial quad
    if name == "skew":
        assert s["padA"] > 0 and s["clashes"] > 0                          # partial quads; a class repeated inside a quad


@pytest.mark.parametrize("na,name", FLOAT_NA)
def test_stress_na_float_image_replays_to_the_dense_model(L, na, name):
    s = R.replay_float_image(L, H.stress_blob(name, "float", na), G.stress_arrays(name, "float", na), na=na)
    want = {"grub_split": (0, ["general", "general"]), "grub_even": (0, ["uniform", "uniform"])}.get(name, (1, ["dense", "dense"]))
    assert (s["dense"], s["chains"]) == want


@pytest.mark.parametrize("na", WIDTHS)
def test_loader_verdicts_on_the_accumulator_bound_na(L, na):
    """The range proof at the smaller widths: default and warm keep the conversion-free rounding, hot falls back to the
    conversion unit, overflow's int8 blob is refused with a message and its float blob loads.  At 256 units the float blob of
    "full" (fp16 blocks, twice the int8 bytes) is refused for its size."""
    verdict = lambda b: int(R.int8_image(L, b)[2][21])
    assert verdict(H.blob("int8", "na%d" % na)) == 1
    assert verdict(H.stress_blob("warm", "int8", na)) == 1
    assert verdict(H.stress_blob("hot", "int8", na)) == 0
    r, _, _ = R.int8_image(L, H.stress_blob("overflow", "int8", na))
    assert r < 0 and b"beyond int32" in L.lpcnet_b200_last_error()
    assert R.float_image(L, H.stress_blob("overflow", "float", na))[0] > 0
    if na == 256:
        assert R.float_image(L, H.stress_blob("full", "float", na))[0] < 0 and b"more than one SM offers" in L.lpcnet_b200_last_error()


def ref_key_na(na, name, build):
    ids, T = STRESS_FEATURES
    return "stress_na%d_%s_%d_%dx%d_%s" % (na, name, ids[0], ids[-1] + 1, T, build)


@pytest.mark.parametrize("na,name,build,kind", [c + ("A", "int8") for c in LOADED_NA] + [c + ("B", "float") for c in FLOAT_NA])
def test_oracle_matches_reference_on_stress_models_na(na, name, build, kind):
    """The CPU restatement against the compiled reference of the na<na> header (build A: int8, build B: float) on every stress
    model of that width; where the reference is not compiled, against the digests it gave."""
    f = make_feature_batch(*STRESS_FEATURES)
    b = H.stress_blob(name, kind, na)
    got = H.oracle_synth(f, kind, model_blob=b)
    assert np.abs(got[:, 320:]).max() > 100                               # not silent
    assert H.digest(got) == H.ref_digest(ref_key_na(na, name, build), lambda: H.ref_synth(f, build, tag="na%d" % na, model_blob=b))
