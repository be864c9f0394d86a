#!/usr/bin/env python3
"""Dump-format writer (TEST INFRASTRUCTURE — not a product path).

A real LPCNet model reaches a user as the `nnet_data.c` / `nnet_data.h` pair that training_tf2/dump_lpcnet.py prints
(download_model.sh unpacks one), not as a DNNw blob.  This module prints any model of oracle/gen_model.py in that text
layout, so that tools/import_nnet_data.py can be checked against two independent ground truths built from the same file:
src/write_lpcnet_weights.c compiled against it (the blob it writes) and the reference compiled from it without
USE_WEIGHTS_FILE (the arrays compiled in, the C compiler doing the decimal -> float conversion).  oracle/Makefile `dumpref`
builds both for every model of MODELS.

The layout (dump_lpcnet.py printVector / printSparseVector / dump_grub and its main):
  * every array in `#ifndef USE_WEIGHTS_FILE` with `WEIGHTS_<name>_DEFINED` / `WEIGHTS_<name>_TYPE`, 8 values per line;
  * block-sparse weights (and GRU_B's recurrent weights) as an `#ifdef DOT_PROD / #else / #endif` pair: the int8 blocks
    in the first branch, the float layout in the second;
  * `idx` arrays as float-formatted ints (`16.0`); arrays the dumper holds as float64 (the GRU_A embeddings, a product
    np.dot(E, W), and the float branch of the sparse weights, concatenated onto a float64 array) at float64 precision;
  * the `lpcnet_arrays[]` table and `init_lpcnet_model` at the end; nnet_data.h with END2END (defined or commented out),
    LPC_GAMMA and FEATURES_DELAY.
Empty plc_data.c / dred_rdovae_{enc,dec}_data.c stubs let write_lpcnet_weights.c link.

  python3 oracle/dump_nnet_data.py --out oracle/_gen_dump [--model NAME]     (--list prints the model names)
"""
import argparse
import decimal
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_model as G  # noqa: E402

# dump_lpcnet.py's print order: the GRU_A input side, dense features, dump_grub, the generic layer loop, dump_sparse_gru.
# (name, C type of the DOT_PROD build, C type of the float build or None when both builds print one array)
LAYOUT = (
    ("gru_a_embed_sig_weights", "float", None), ("gru_a_embed_pred_weights", "float", None),
    ("gru_a_embed_exc_weights", "float", None),
    ("gru_a_dense_feature_weights", "float", None), ("gru_a_dense_feature_bias", "float", None),
    ("gru_b_dense_feature_weights", "float", None), ("gru_b_dense_feature_bias", "float", None),
    ("gru_b_weights", "qweight", "qweight"), ("gru_b_weights_idx", "int", None),
    ("gru_b_recurrent_weights", "qweight", "float"),
    ("gru_b_bias", "float", None), ("gru_b_subias", "float", None),
    ("embed_sig_weights", "float", None), ("embed_pitch_weights", "float", None),
    ("feature_conv1_weights", "float", None), ("feature_conv1_bias", "float", None),
    ("feature_conv2_weights", "float", None), ("feature_conv2_bias", "float", None),
    ("feature_dense1_weights", "float", None), ("feature_dense1_bias", "float", None),
    ("feature_dense2_weights", "float", None), ("feature_dense2_bias", "float", None),
    ("dual_fc_weights", "float", None), ("dual_fc_bias", "float", None), ("dual_fc_factor", "float", None),
    ("sparse_gru_a_recurrent_weights_diag", "float", None),
    ("sparse_gru_a_recurrent_weights", "qweight", "qweight"), ("sparse_gru_a_recurrent_weights_idx", "int", None),
    ("sparse_gru_a_bias", "float", None), ("sparse_gru_a_subias", "float", None),
)
EMBEDDINGS = ("gru_a_embed_sig_weights", "gru_a_embed_pred_weights", "gru_a_embed_exc_weights")
SPARSE = ("gru_b_weights", "sparse_gru_a_recurrent_weights")

# Hand-picked literals: the first TIE_COUNT elements of TIE_ARRAY with an even float32 mantissa are printed as a float32
# rounding midpoint moved by 1e-30 (relative) to the far side.  Decimal -> double lands exactly on the midpoint, and the
# tie then goes to the even value, the model's; decimal -> float rounded directly would give the odd neighbour.
TIE_ARRAY = "gru_a_embed_sig_weights"
TIE_COUNT = 16


def _midpoint_literal(x, up):
    """A decimal literal just beyond the midpoint between float32 x and its neighbour above (up) or below."""
    n = np.nextafter(x, np.float32(np.inf if up else -np.inf))
    ctx = decimal.Context(prec=80)
    m = ctx.divide(ctx.add(decimal.Decimal(float(x)), decimal.Decimal(float(n))), 2)         # exact: both are dyadic
    d = ctx.add(m, ctx.multiply(m.copy_abs(), decimal.Decimal("1e-30") * (1 if n > x else -1)))
    return format(d, "E")


def tie_literals(a):
    """{flat index: literal} of the hand-picked elements of the TIE_ARRAY array `a` (float32)."""
    v = np.ascontiguousarray(a, np.float32).reshape(-1)
    bits = v.view(np.uint32)
    out = {}
    for i in range(v.size):
        if len(out) == TIE_COUNT:
            break
        if v[i] != 0 and np.isfinite(v[i]) and not (bits[i] & 1):
            out[i] = _midpoint_literal(v[i], up=len(out) % 2 == 0)
    return out


def _float64_text(name, a):
    """The values of a float64 array of the dumper: float32 values moved by up to 1/8 float32 ulp, so that each literal
    is not itself a float32 and the conversion has to round (to the model's value)."""
    v = np.ascontiguousarray(a, np.float32).reshape(-1)
    rng = np.random.default_rng(sum(name.encode()))
    w = v.astype(np.float64) + rng.uniform(-0.125, 0.125, v.size) * np.spacing(np.abs(v)).astype(np.float64)
    w[v == 0] = 0.0
    return [repr(x) for x in w.tolist()]


def _values(name, ctype, a, float64):
    if ctype == "int":
        return [repr(float(x)) for x in np.asarray(a).reshape(-1).tolist()]          # np.append's idx: 16.0
    if ctype == "qweight" and np.asarray(a).dtype == np.int8:
        return [str(x) for x in np.asarray(a).reshape(-1).tolist()]
    if not float64:
        return [str(x) for x in np.ascontiguousarray(a, np.float32).reshape(-1)]
    if name in EMBEDDINGS:
        t = _float64_text(name, a)
        if name == TIE_ARRAY:
            for i, lit in tie_literals(a).items():
                t[i] = lit
        return t
    return [repr(x) for x in np.ascontiguousarray(a, np.float32).astype(np.float64).reshape(-1).tolist()]


def print_vector(name, ctype, vals):
    """printVector's text for one array."""
    out = ["#ifndef USE_WEIGHTS_FILE\n#define WEIGHTS_%s_DEFINED\n#define WEIGHTS_%s_TYPE WEIGHT_TYPE_%s\n" % (name, name, ctype),
           "static const %s %s[%d] = {\n   " % (ctype, name, len(vals))]
    lines = [", ".join(vals[i:i + 8]) for i in range(0, len(vals), 8)]
    out.append(",\n   ".join(lines))
    out.append("\n};\n#endif\n\n")
    return "".join(out)


def nnet_data_c(common, only8, onlyf, na):
    arrs8 = {n: a for n, _, a in common + only8}
    arrsf = {n: a for n, _, a in common + onlyf}
    assert set(arrs8) == set(arrsf) == {n for n, _, _ in LAYOUT}, "model arrays differ from the dump layout"
    out = ["/*This file is automatically generated from a Keras model*/\n/*based on model oracle/gen_model.py*/\n\n",
           "#ifdef HAVE_CONFIG_H\n#include \"config.h\"\n#endif\n\n#include \"nnet.h\"\n#include \"nnet_data.h\"\n\n"]
    for name, t8, tf in LAYOUT:
        f64 = name in EMBEDDINGS
        if tf is None:
            out.append(print_vector(name, t8, _values(name, t8, arrs8[name], f64)))
        else:
            out.append("#ifdef DOT_PROD\n")
            out.append(print_vector(name, t8, _values(name, t8, arrs8[name], False)))
            out.append("#else /*DOT_PROD*/\n")
            out.append(print_vector(name, tf, _values(name, tf, arrsf[name], name in SPARSE)))
            out.append("#endif /*DOT_PROD*/\n")
    out.append("#ifndef USE_WEIGHTS_FILE\nconst WeightArray lpcnet_arrays[] = {\n")
    for name, _, _ in LAYOUT:
        out.append("#ifdef WEIGHTS_%s_DEFINED\n  {\"%s\", WEIGHTS_%s_TYPE, sizeof(%s), %s},\n#endif\n" % (name, name, name, name, name))
    out.append("  {NULL, 0, 0, NULL}\n};\n#endif\n")
    init = G.NNET_DATA_C.format(n3a=3 * na, n3b=3 * G.N_B, embed=G.EMBED, pembed=G.PITCH_EMBED, cond=G.COND,
                                fin=G.FRAME_IN, na=na, nb=G.N_B)
    out.append(init[init.index("#ifndef DUMP_BINARY_WEIGHTS"):])
    return "".join(out)


STUBS = {
    "plc_data.c": "lpcnet_plc_arrays",
    "dred_rdovae_enc_data.c": "rdovae_enc_arrays",
    "dred_rdovae_dec_data.c": "rdovae_dec_arrays",
}


def _model_fn(kind, arg):
    if kind == "stress":
        name, na = arg
        return lambda: G.make_stress_model(name, na)
    return lambda: G.make_model(1234, na=arg.get("na"))


def _models():
    """name -> (arrays() -> (common, only8, onlyf), GRU_A units, header settings {e2e, delay, gamma})."""
    m = {"default": (_model_fn("gen", {}), G.N_A, {})}
    for tag, v in G.VARIANTS.items():
        m[tag] = (_model_fn("gen", v), v.get("na", G.N_A), {k: v[k] for k in ("e2e", "delay", "gamma") if k in v})
    m["gamma085"] = (_model_fn("gen", {}), G.N_A, {"gamma": 0.85})      # a non-default LPC_GAMMA: `#define LPC_GAMMA 0.85f`
    for na in G.STRESS_NA:
        for name in G.stress_names(na):
            m["stress_%s_na%d" % (name, na)] = (_model_fn("stress", (name, na)), na, {})
    return m


MODELS = _models()


def header_config(model):
    """(lpc_gamma, features_delay, end2end) that MODELS[model]'s nnet_data.h defines."""
    h = MODELS[model][2]
    return (G.LPC_GAMMA if h.get("gamma") is None else h["gamma"], G.FEATURES_DELAY if h.get("delay") is None else h["delay"],
            bool(h.get("e2e", False)))


def write_model(out, model):
    """nnet_data.c / nnet_data.h (+ the headers and stubs the reference sources include or link) of MODELS[model] into
    out/<model>; returns that directory.  Each file is written under a temporary name and renamed."""
    arrays, na, hdr = MODELS[model]
    d = os.path.join(out, model)
    os.makedirs(d, exist_ok=True)
    G.write_c_sources(d, na=na, **hdr)                       # nnet_data.h, plc_data.h, dred_rdovae_constants.h
    files = {"nnet_data.c": nnet_data_c(*arrays(), na=na)}
    for fn, sym in STUBS.items():
        files[fn] = "/* stub: only the LPCNet model is dumped */\n#include \"nnet.h\"\nconst WeightArray %s[] = {\n  {NULL, 0, 0, NULL}\n};\n" % sym
    for fn, text in files.items():
        tmp = os.path.join(d, "%s.tmp%d" % (fn, os.getpid()))
        with open(tmp, "w") as f:
            f.write(text)
        os.replace(tmp, os.path.join(d, fn))
    return d


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "_gen_dump"))
    ap.add_argument("--model", action="append", help="one of MODELS (default: all)")
    ap.add_argument("--list", action="store_true", help="print the model names")
    a = ap.parse_args()
    if a.list:
        print(" ".join(MODELS))
    else:
        for m in a.model or MODELS:
            write_model(a.out, m)
