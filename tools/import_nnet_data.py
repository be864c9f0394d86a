#!/usr/bin/env python3
"""import_nnet_data.py — real-model importer (SURVEY 8f N4): a model dumped by the reference's training_tf2/dump_lpcnet.py
(`nnet_data.c` + `nnet_data.h`, what download_model.sh:4-12 unpacks from lpcnet_data-*.tar.gz) -> a "DNNw" weight blob that
lpcnet_b200_batch_create / lpcnet_load_model read, with LPC_GAMMA / FEATURES_DELAY / END2END (nnet_data.h, dump_lpcnet.py:306-329)
embedded as the `lpcnet_b200_config` record, so nothing travels out-of-band.

It does what compiling src/write_lpcnet_weights.c:47-78 against that nnet_data.c would do, without a C compiler: the array
initialisers printed by dump_lpcnet.py:54-81 (`static const <type> <name>[<n>] = { ... };`) are parsed as text.  The
`#ifdef DOT_PROD ... #else ... #endif` pairs of dump_lpcnet.py:110-114 select the int8 blocks (default) or, with --float, the
float blocks of the DISABLE_DOT_PROD build.

  python tools/import_nnet_data.py path/to/nnet_data.c [--header nnet_data.h] [--float] -o weights_blob.bin
The blob is written through the library's own writer (lpcnet_b200_write_blob, csrc/blob_io.cu).
"""
import argparse
import ctypes
import os
import re
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

TYPE_ID = {"float": 0, "int": 1, "qweight": 2, "opus_int8": 2}
_ARRAY = re.compile(r"static\s+const\s+(float|int|qweight|opus_int8)\s+(\w+)\s*\[\s*(\d+)\s*\]\s*=\s*\{([^}]*)\}\s*;", re.S)


def select_branches(text, dot_prod):
    """Resolve the `#ifdef DOT_PROD / #else / #endif` pairs; every other preprocessor line is dropped (USE_WEIGHTS_FILE and
    DUMP_BINARY_WEIGHTS guards are taken as 'arrays present')."""
    out, stack = [], []            # stack entries: None (guard we ignore) or [is_dot_prod_block, currently_in_true_branch]
    for line in text.splitlines():
        s = line.strip()
        if s.startswith("#"):
            d = s[1:].strip()
            if re.match(r"ifdef\s+DOT_PROD\b", d):
                stack.append([True, True])
            elif re.match(r"ifndef\s+DOT_PROD\b", d):
                stack.append([True, False])
            elif d.startswith("if"):
                stack.append(None)
            elif d.startswith("else"):
                if stack and stack[-1] is not None:
                    stack[-1][1] = not stack[-1][1]
            elif d.startswith("endif"):
                if stack:
                    stack.pop()
            continue
        keep = all(e is None or e[1] == dot_prod for e in stack)
        if keep:
            out.append(line)
    return "\n".join(out)


def parse_arrays(text, dot_prod=True):
    """[(name, type id, numpy array)] in file order (= the order of lpcnet_arrays[], dump_lpcnet.py:359-366)."""
    arrays, seen = [], set()
    for m in _ARRAY.finditer(select_branches(text, dot_prod)):
        ctype, name, count, body = m.group(1), m.group(2), int(m.group(3)), m.group(4)
        if name in seen:
            continue
        seen.add(name)
        vals = body.replace("\n", " ").split(",")
        vals = [v.strip().rstrip("fF") for v in vals if v.strip()]
        if len(vals) != count:
            raise ValueError("array %s: %d initialisers for %d elements" % (name, len(vals), count))
        if ctype == "float" or (ctype == "qweight" and not dot_prod):
            a = np.array([float(v) for v in vals], dtype=np.float32)       # qweight is float in the DISABLE_DOT_PROD build (nnet.h)
        elif ctype == "int":
            a = np.array([int(float(v)) for v in vals], dtype=np.int32)
        else:
            a = np.array([int(float(v)) for v in vals], dtype=np.int8)
        arrays.append((name, TYPE_ID[ctype], a))
    if not arrays:
        raise ValueError("no `static const <type> name[n] = {...};` arrays found (was the model dumped with USE_WEIGHTS_FILE only?)")
    return arrays


def parse_header(text):
    """LPC_GAMMA, FEATURES_DELAY, END2END from nnet_data.h (dump_lpcnet.py:306-329).  Only live `#define` lines count: a
    non-end-to-end model's header carries `/* #define END2END */`, and a hand-edited one may keep old values in comments."""
    cfg = {"lpc_gamma": 1.0, "features_delay": 2, "end2end": 0}
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    text = re.sub(r"//[^\n]*", "", text)
    m = re.search(r"^\s*#\s*define\s+LPC_GAMMA\s+([0-9.eE+-]+)f?", text, flags=re.M)
    if m:
        cfg["lpc_gamma"] = float(m.group(1))
    m = re.search(r"^\s*#\s*define\s+FEATURES_DELAY\s+(\d+)", text, flags=re.M)
    if m:
        cfg["features_delay"] = int(m.group(1))
    if re.search(r"^\s*#\s*define\s+END2END\b", text, flags=re.M):
        cfg["end2end"] = 1
    return cfg


def write_blob(arrays, cfg, lib=None):
    """bytes of the DNNw blob, produced by the library's writer (lpcnet_b200_write_blob)."""
    import lpcnet_b200
    from lpcnet_b200 import api
    L = lib or lpcnet_b200.lib()
    n = len(arrays)
    recs = (api.Array * n)()
    keep = []
    for i, (name, typ, a) in enumerate(arrays):
        a = np.ascontiguousarray(a)
        nm = name.encode()
        keep += [a, nm]
        recs[i].name = nm; recs[i].type = typ; recs[i].size = a.nbytes; recs[i].data = a.ctypes.data
    c = api.Config(cfg["lpc_gamma"], cfg["features_delay"], cfg["end2end"]) if cfg is not None else None
    cp = ctypes.byref(c) if c is not None else None
    need = L.lpcnet_b200_write_blob(recs, n, cp, None, 0)
    if need < 0:
        raise RuntimeError(L.lpcnet_b200_last_error().decode())
    buf = (ctypes.c_ubyte * need)()
    if L.lpcnet_b200_write_blob(recs, n, cp, buf, need) != need:
        raise RuntimeError(L.lpcnet_b200_last_error().decode())
    return bytes(buf)


def import_model(c_path, h_path=None, is_float=False):
    arrays = parse_arrays(open(c_path).read(), dot_prod=not is_float)
    if h_path is None:
        h_path = os.path.join(os.path.dirname(os.path.abspath(c_path)), "nnet_data.h")
    cfg = parse_header(open(h_path).read()) if os.path.exists(h_path) else None
    return write_blob(arrays, cfg), arrays, cfg


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("nnet_data_c")
    ap.add_argument("--header", default=None, help="nnet_data.h (default: next to nnet_data.c)")
    ap.add_argument("--float", action="store_true", help="take the float (DISABLE_DOT_PROD) blocks instead of the int8 ones")
    ap.add_argument("-o", "--out", default="weights_blob.bin")
    a = ap.parse_args()
    blob, arrays, cfg = import_model(a.nnet_data_c, a.header, a.float)
    open(a.out, "wb").write(blob)
    print("%s: %d arrays, %d bytes, config %s" % (a.out, len(arrays), len(blob), cfg))


if __name__ == "__main__":
    main()
