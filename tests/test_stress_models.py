"""CPU tests (-m "not gpu") of the stress models (oracle/gen_model.py STRESS): models whose block lists and int8 values are
unlike the default synthetic model's and reach the paths of the per-sample kernels that the default model never takes (sparse
GRU_B input rows, skewed GRU_A lists, int8 weights at the loader's limit, accumulator bounds on both sides of the range proof of
the conversion-free rounding).  Checked here: that each fixture has the structure it is meant to have, the images the kernels
consume, the loader's verdicts, and the CPU restatement against the compiled reference on every model."""
import hashlib
import json
import os
import numpy as np
import pytest
import gen_model as G
import helpers as H
import image_replay as R
from fixtures import make_feature_batch

NA = G.N_A
LOADED = [n for n in G.STRESS if n != "overflow"]           # the int8 blob of "overflow" is refused by the loader
STRESS_GOLDEN = os.path.join(H.GOLDEN, "stress_models.json")


@pytest.fixture(scope="module")
def L():
    from lpcnet_b200 import build, api
    build.build()
    return api.lib()


def _lists(arrs, name, nrows):
    """[(count, [pos, ...]) per 8-row group] of a block-sparse index array."""
    idx, p, out = arrs[name], 0, []
    for _ in range(nrows // 8):
        nb = int(idx[p]); out.append([int(v) for v in idx[p + 1:p + 1 + nb]]); p += nb + 1
    assert p == len(idx)
    return out


def _pairs(a):
    """int8 input pairs (w0, w1) of a blob array: consecutive bytes along the input axis (the operands of one maddubs lane)."""
    return np.asarray(a, np.int8).astype(np.int64).reshape(-1, 2)


def test_stress_blobs_are_deterministic():
    want = json.load(open(STRESS_GOLDEN))
    for name in G.STRESS:
        for kind in ("int8", "float"):
            assert hashlib.sha256(H.stress_blob(name, kind)).hexdigest() == want["%s_%s_sha256" % (name, kind)], (name, kind)
    assert sorted(want) == sorted("%s_%s_sha256" % (n, k) for n in G.STRESS for k in ("int8", "float"))


@pytest.mark.parametrize("name", list(G.STRESS))
def test_stress_model_has_its_structure(name):
    """Each fixture keeps the property it exists for (so that it cannot quietly degenerate into a default-like model)."""
    a8, af = G.stress_arrays(name, "int8"), G.stress_arrays(name, "float")
    for arr in ("sparse_gru_a_recurrent_weights", "gru_b_weights", "gru_b_recurrent_weights"):     # float blob = int8 values / 128
        np.testing.assert_array_equal(np.asarray(af[arr], np.float64) * 128, np.asarray(a8[arr], np.int8).reshape(-1, 8, 4).transpose(0, 2, 1).reshape(-1)
                                      if arr != "gru_b_recurrent_weights" else
                                      np.asarray(a8[arr], np.int8).reshape(6, 4, 8, 4).transpose(1, 3, 0, 2).reshape(-1))
    la = _lists(a8, "sparse_gru_a_recurrent_weights_idx", 3 * NA)
    lb = _lists(a8, "gru_b_weights_idx", 48)
    nb = [len(x) for x in lb]
    same_sign = lambda p: (np.sign(p[:, 0]) * np.sign(p[:, 1]) >= 0)
    for arr in ("sparse_gru_a_recurrent_weights", "gru_b_weights", "gru_b_recurrent_weights"):   # what the loader accepts
        p = _pairs(a8[arr])
        assert (np.abs(p).sum(axis=1)[same_sign(p)]).max() <= 128
    bound = G.cvt_bound(a8)
    if name == "grub_split":
        assert nb[4:] == [NA // 4] * 2                                   # candidate rows dense
        assert max(nb[:4]) < NA // 4 and len(set(nb[:4])) == 4            # update / reset rows sparse, unequal counts
        assert 1 in nb and 3 in nb                                       # int8 K parts: one empty, one a partial quad
    elif name == "grub_even":
        assert nb == [42] * 6 and (42 // 2) % 4 != 0                      # all alike, not dense; partial quad in each K part
        assert all(x != list(range(0, NA, 4))[:42] for x in lb)           # scattered, not the first blocks in order
    elif name == "skew":
        for gate in range(3):
            n = [len(x) for x in la[gate * NA // 8:(gate + 1) * NA // 8]]
            assert 0 in n and 1 in n and 2 in n and 3 in n
            assert max(n) >= 4 * np.mean(n)                               # skewed, not uniform
            assert any(len(x) >= 6 and len({(p // 4) & 3 for p in x}) == 1 for x in la[gate * NA // 8:(gate + 1) * NA // 8])
            assert any(NA - 4 in x for x in la[gate * NA // 8:(gate + 1) * NA // 8])
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
    if name not in ("warm", "hot", "overflow"):
        assert bound < G.FAST_CVT_LIMIT


@pytest.mark.parametrize("name", LOADED)
def test_stress_int8_image_replays_to_the_dense_model(L, name):
    a8 = G.stress_arrays(name, "int8")
    s = R.replay_int8_image(L, H.stress_blob(name, "int8"), a8)
    nb = [len(x) for x in _lists(a8, "gru_b_weights_idx", 48)]
    # each GRU_B input list is split into two K parts, the first one taking the odd block
    assert s["kparts"] == 2
    np.testing.assert_array_equal(s["partsB"], [[-(-((n + 1) // 2) // 4), -(-(n - (n + 1) // 2) // 4)] for n in nb])
    assert s["fast_cvt"] == (0 if name == "hot" else 1)
    if name == "grub_split":
        assert (s["partsB"] == 0).any() and s["padB"] > 0                  # an empty K part; partial quads
    if name == "grub_even":
        assert s["padB"] > 0
    if name == "skew":
        assert s["fcw_nodes"] < 64                                         # the image is full enough to give up dual_fc rows by itself
        assert s["padA"] > 0 and s["clashes"] > 0


@pytest.mark.parametrize("name", LOADED)
def test_stress_float_image_replays_to_the_dense_model(L, name):
    s = R.replay_float_image(L, H.stress_blob(name, "float"), G.stress_arrays(name, "float"))
    want = {"grub_split": (0, ["general", "general"]), "grub_even": (0, ["uniform", "uniform"])}.get(name, (1, ["dense", "dense"]))
    assert (s["dense"], s["chains"]) == want


def test_loader_verdicts_on_the_accumulator_bound(L):
    """warm: conversion-free rounding kept; hot: the loader falls back to the conversion unit by itself; overflow: the int8 blob
    is refused with a message (past int32 the reference's conversion and the kernel's would disagree).  The float blob of
    overflow has no integer accumulators and loads."""
    verdict = lambda b: int(R.int8_image(L, b)[2][21])
    assert R.int8_image(L, H.blob("int8"))[0] > 0 and verdict(H.blob("int8")) == 1
    assert verdict(H.stress_blob("warm", "int8")) == 1
    assert verdict(H.stress_blob("hot", "int8")) == 0
    r, _, _ = R.int8_image(L, H.stress_blob("overflow", "int8"))
    assert r < 0 and b"beyond int32" in L.lpcnet_b200_last_error()
    assert R.float_image(L, H.stress_blob("overflow", "float"))[0] > 0


STRESS_FEATURES = (range(300, 306), 12)


def stress_features():
    return make_feature_batch(*STRESS_FEATURES)


def ref_key(name, build):
    ids, T = STRESS_FEATURES
    return "stress_%s_%d_%dx%d_%s" % (name, ids[0], ids[-1] + 1, T, build)


@pytest.mark.parametrize("name", LOADED)
@pytest.mark.parametrize("build,kind", [("A", "int8"), ("B", "float")])
def test_oracle_matches_reference_on_stress_models(name, build, kind):
    """The CPU restatement against the compiled reference (build A: int8 with maddubs and cvtps2dq; build B: float) on every
    stress model; where the reference is not compiled, against the digests it gave."""
    f = stress_features()
    b = H.stress_blob(name, kind)
    got = H.oracle_synth(f, kind, model_blob=b)
    assert np.abs(got[:, 320:]).max() > 100                               # not silent
    assert H.digest(got) == H.ref_digest(ref_key(name, build), lambda: H.ref_synth(f, build, model_blob=b))
