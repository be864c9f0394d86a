"""Shared test plumbing: builds/loads the checkers (oracle port, compiled reference) through ctypes.

The oracle and the compiled reference are CHECKERS: they are only ever used from tests/, smoke() and the
bench's cpu_baseline leg — never by the product library.
"""
import ctypes
import functools
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
GEN = os.path.join(ORACLE, "_gen")
GOLDEN = os.path.join(ROOT, "tests", "golden")
LPC_GAMMA = 0.9

c_p = ctypes.c_void_p


@functools.lru_cache(None)
def gen_dir(tag=""):
    """Deterministically (re)generate the synthetic model files.  tag: "" (the default 384/16 model) or one of
    gen_model.VARIANTS (other GRU_A sizes, END2END, FEATURES_DELAY) -> oracle/_gen_<tag>."""
    import gen_model
    d = GEN + ("_" + tag if tag else "")
    need = ["model_int8.bin", "model_float.bin", "codebooks.bin"] + ([] if tag else ["model_int8_clamp.bin"])
    if not all(os.path.exists(os.path.join(d, n)) for n in need):
        gen_model.generate(d, c_sources=os.path.isdir("/root/reference/src"), **(gen_model.VARIANTS[tag] if tag else {}))
    return d


@functools.lru_cache(None)
def blob(kind="int8", tag=""):
    """kind: int8 | float | int8_clamp (default model only)."""
    return open(os.path.join(gen_dir(tag), "model_%s.bin" % kind), "rb").read()


STRESS_DIR = GEN + "_stress"


@functools.lru_cache(None)
def stress_blob(name, kind="int8", na=384):
    """Blob of one of gen_model.STRESS (kind int8 | float) with `na` GRU_A units (gen_model.STRESS_NA), generated into
    oracle/_gen_stress on first use."""
    import gen_model
    path = os.path.join(STRESS_DIR, gen_model.stress_blob_name(name, kind, na))
    if not os.path.exists(path):
        gen_model.generate_stress(STRESS_DIR)
    return open(path, "rb").read()


def model_config(tag=""):
    """(lpc_gamma, features_delay, end2end) the reference bakes into nnet_data.h for this variant."""
    import gen_model
    v = gen_model.VARIANTS[tag] if tag else {}
    g = v.get("gamma")
    d = v.get("delay")
    return (LPC_GAMMA if g is None else g, gen_model.FEATURES_DELAY if d is None else d, bool(v.get("e2e", False)))


@functools.lru_cache(None)
def codebooks():
    return np.fromfile(os.path.join(gen_dir(), "codebooks.bin"), dtype=np.float32)


@functools.lru_cache(None)
def rcp_table():
    return np.fromfile(os.path.join(GOLDEN, "rcpps_table.bin"), dtype="<u4")


@functools.lru_cache(None)
def oracle_lib():
    so = os.path.join(ORACLE, "_build", "liblpcnet_oracle.so")
    src = os.path.join(ORACLE, "lpcnet_oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(src), os.path.getmtime(os.path.join(ORACLE, "lpcnet_enc_oracle.inc"))):
        subprocess.check_call(["make", "-C", ORACLE, "port"], stdout=subprocess.DEVNULL)
    L = ctypes.CDLL(so)
    L.oracle_model_create.restype = c_p
    L.oracle_model_create.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_float, c_p]
    L.oracle_model_create_ex.restype = c_p
    L.oracle_model_create_ex.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_float, ctypes.c_int, ctypes.c_int, c_p]
    L.oracle_synthesize_impl.argtypes = [c_p, c_p, c_p, ctypes.c_int, ctypes.c_int]
    L.oracle_run_frame_network.argtypes = [c_p, c_p]
    L.oracle_synthesize_tail.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int]
    L.oracle_frame_network_deferred.argtypes = [c_p, c_p]
    L.oracle_frame_network_flush.argtypes = [c_p]
    L.oracle_reset_signal.argtypes = [c_p]
    L.oracle_export_state.argtypes = [c_p, c_p]
    L.oracle_model_na.argtypes = [c_p]
    L.oracle_state_size.argtypes = []
    L.oracle_state_create.restype = c_p
    L.oracle_state_create.argtypes = [c_p]
    L.oracle_state_destroy.argtypes = [c_p]
    L.oracle_reset.argtypes = [c_p]
    L.oracle_synthesize.argtypes = [c_p, c_p, c_p, ctypes.c_int]
    L.oracle_synthesize_trace.argtypes = [c_p, c_p, c_p, ctypes.c_int, c_p]
    L.oracle_decode.argtypes = [c_p, c_p, c_p]
    L.oracle_decode_packet.argtypes = [c_p, c_p, c_p]
    L.oracle_frame_network.argtypes = [c_p, c_p, c_p, c_p, c_p]
    L.oracle_get_tables.argtypes = [c_p] * 6
    L.oracle_get_state.argtypes = [c_p] * 6
    L.oracle_tanh.restype = ctypes.c_float
    L.oracle_tanh.argtypes = [c_p, ctypes.c_float]
    L.oracle_sigmoid.restype = ctypes.c_float
    L.oracle_sigmoid.argtypes = [c_p, ctypes.c_float]
    L.oracle_lin2ulaw.argtypes = [ctypes.c_float]
    L.oracle_synthesize_batch.restype = ctypes.c_double
    L.oracle_synthesize_batch.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.oracle_decode_batch.restype = ctypes.c_double
    L.oracle_decode_batch.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.oracle_enc_create.restype = c_p
    L.oracle_enc_create.argtypes = [c_p]
    L.oracle_enc_destroy.argtypes = [c_p]
    L.oracle_enc_single_frame_features.argtypes = [c_p, c_p, c_p]
    L.oracle_enc_encode.argtypes = [c_p, c_p, c_p]
    L.oracle_enc_compute_features.argtypes = [c_p, c_p, c_p]
    L.oracle_enc_single_frame_features_float.argtypes = [c_p, c_p, c_p]
    L.oracle_enc_last_best_a.restype = ctypes.c_float
    L.oracle_enc_last_best_a.argtypes = [c_p]
    L.oracle_pitch_index.argtypes = [ctypes.c_float]
    L.oracle_rcp.restype = ctypes.c_float
    L.oracle_rcp.argtypes = [c_p, ctypes.c_float]
    return L


@functools.lru_cache(None)
def oracle_model(kind="int8", tag="", model_blob=None):
    """CPU-restatement model for a blob flavour (int8 / float / int8_clamp) of a model variant (tag, gen_model.VARIANTS), or for
    the explicit blob `model_blob` (with the variant's header settings)."""
    L = oracle_lib()
    b = blob(kind, tag) if model_blob is None else model_blob
    gamma, delay, e2e = model_config(tag)
    m = L.oracle_model_create_ex(b, len(b), rcp_table().ctypes.data, gamma, delay, int(e2e), codebooks().ctypes.data)
    assert m, "oracle failed to parse the blob"
    return m


def oracle_synth(features, kind="int8", nthreads=8, tag="", model_blob=None):
    """features [n][T][20] float32 -> pcm [n][T*160] int16 via the CPU restatement (of `model_blob` when given)."""
    L = oracle_lib()
    f = np.ascontiguousarray(features, dtype=np.float32)
    n, T, stride = f.shape
    pcm = np.zeros((n, T * 160), dtype=np.int16)
    L.oracle_synthesize_batch(oracle_model(kind, tag, model_blob), f.ctypes.data, stride, n, T, nthreads, pcm.ctypes.data)
    return pcm


def oracle_decode(packets, kind="int8", nthreads=8, model_blob=None, tag=""):
    """packets [n][P][8] uint8 -> pcm [n][P*640] int16 (of the variant `tag`, or of `model_blob` when given)."""
    L = oracle_lib()
    p = np.ascontiguousarray(packets, dtype=np.uint8)
    n, P, _ = p.shape
    pcm = np.zeros((n, P * 640), dtype=np.int16)
    L.oracle_decode_batch(oracle_model(kind, tag, model_blob), p.ctypes.data, n, P, nthreads, pcm.ctypes.data)
    return pcm


def have_ref(build="A", tag=""):
    return os.path.exists(os.path.join(ORACLE, "_ref", "liblpcnet_ref_%s%s.so" % (build, "_" + tag if tag else "")))


@functools.lru_cache(None)
def ref_lib(build="A", tag=""):
    """The UNTOUCHED reference compiled by oracle/Makefile (`make ref`); tag selects a model variant's build."""
    L = ctypes.CDLL(os.path.join(ORACLE, "_ref", "liblpcnet_ref_%s%s.so" % (build, "_" + tag if tag else "")))
    L.ref_synth_batch.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.ref_decode_batch.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.ref_time_streams.restype = ctypes.c_double
    L.ref_time_streams.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, c_p]
    L.ref_synth_stream.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, c_p]
    L.ref_decode_stream.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, c_p]
    L.ref_decode_packet.argtypes = [c_p, c_p, c_p]
    L.ref_frame_network.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, c_p, c_p, c_p]
    L.ref_rcp.restype = ctypes.c_float
    L.ref_rcp.argtypes = [ctypes.c_float]
    if hasattr(L, "ref_rcp8"):                  # a reference compiled before the shim had it lacks the symbol
        L.ref_rcp8.argtypes = [c_p, c_p, ctypes.c_int]
    L.ref_ulaw2lin.restype = ctypes.c_float
    L.ref_ulaw2lin.argtypes = [ctypes.c_float]
    L.ref_lin2ulaw.argtypes = [ctypes.c_float]
    L.ref_activation.argtypes = [c_p, c_p, ctypes.c_int, ctypes.c_int]
    L.ref_state_create.restype = c_p
    L.ref_state_create.argtypes = [ctypes.c_char_p, ctypes.c_int]
    for fn in ("ref_features_stream", "ref_features_stream_float", "ref_encode_stream", "ref_features4_stream"):
        if hasattr(L, fn):
            getattr(L, fn).argtypes = [c_p, ctypes.c_int, c_p]
    if hasattr(L, "ref_encode_then_features"):
        L.ref_encode_then_features.argtypes = [c_p, ctypes.c_int, c_p, ctypes.c_int, c_p]
        L.ref_enc_tables.argtypes = [c_p, c_p]
    for fn, at in (("ref_state_destroy", [c_p]), ("ref_state_reset", [c_p]), ("ref_state_copy", [c_p, c_p]),
                   ("ref_synthesize_impl", [c_p, c_p, c_p, ctypes.c_int, ctypes.c_int]), ("ref_run_frame_network", [c_p, c_p]),
                   ("ref_synthesize_tail", [c_p, c_p, ctypes.c_int, ctypes.c_int]), ("ref_frame_network_deferred", [c_p, c_p]),
                   ("ref_frame_network_flush", [c_p]), ("ref_reset_signal", [c_p])):
        getattr(L, fn).argtypes = at
        getattr(L, fn).restype = None
    if hasattr(L, "ref_dec_state_create"):      # decoder-state entry points (ref_shim.c)
        L.ref_dec_state_create.restype = c_p
        L.ref_dec_state_create.argtypes = [ctypes.c_char_p, ctypes.c_int]
        L.ref_decode.argtypes = [c_p, c_p, c_p]
        for fn, at in (("ref_dec_state_destroy", [c_p]), ("ref_dec_reset", [c_p]), ("ref_dec_state_copy", [c_p, c_p])):
            getattr(L, fn).argtypes = at
            getattr(L, fn).restype = None
    return L


def ref_synth(features, build="A", tag="", kind=None, nthreads=None, model_blob=None):
    """features [n][T][stride] -> pcm [n][T*160] through the compiled reference (fresh lpcnet_create() per stream), loading
    `model_blob` when given."""
    L = ref_lib(build, tag)
    b = blob(kind or ("float" if build in ("B", "TB") else "int8"), tag) if model_blob is None else model_blob
    f = np.ascontiguousarray(features, dtype=np.float32)
    n, T, stride = f.shape
    pcm = np.zeros((n, T * 160), dtype=np.int16)
    assert L.ref_synth_batch(b, len(b), f.ctypes.data, stride, T, n, nthreads or min(n, os.cpu_count() or 1), pcm.ctypes.data) == 0
    return pcm


def ref_decode(packets, build="A", tag="", nthreads=None):
    L = ref_lib(build, tag)
    b = blob("float" if build in ("B", "TB") else "int8", tag)
    p = np.ascontiguousarray(packets, dtype=np.uint8)
    n, P, _ = p.shape
    pcm = np.zeros((n, P * 640), dtype=np.int16)
    assert L.ref_decode_batch(b, len(b), p.ctypes.data, P, n, nthreads or min(n, os.cpu_count() or 1), pcm.ctypes.data) == 0
    return pcm


REF_DIGESTS = os.path.join(GOLDEN, "ref_digests.json")


def digest(a):
    """dtype, shape and sha256 of an array's bytes: equal digests = bit-identical arrays."""
    import hashlib
    a = np.ascontiguousarray(a)
    return "%s%s:%s" % (a.dtype.str, list(a.shape), hashlib.sha256(a.tobytes()).hexdigest())


def ref_has(build, tag, *symbols):
    """The reference of (build, tag) is compiled and exports the shim entry points `symbols` (a reference compiled before
    oracle/ref_shim.c had them lacks them)."""
    return have_ref(build, tag) and all(hasattr(ref_lib(build, tag), s) for s in symbols)


def ref_digest(key, compute, runnable=True):
    """Digest of what the compiled reference returns for the input named `key` (compute() runs it).  Where the reference is
    compiled (and `runnable`: it has what compute() calls, see ref_has) it is run and must reproduce the digest stored in
    tests/golden/ref_digests.json (LPCNET_WRITE_REF_DIGESTS=1 stores it instead); elsewhere the stored digest stands in for
    the run."""
    import json
    stored = json.load(open(REF_DIGESTS)) if os.path.exists(REF_DIGESTS) else {}
    if not have_ref("A") or not runnable:
        assert key in stored, "no stored reference digest for %s" % key
        return stored[key]
    d = digest(compute())
    if os.environ.get("LPCNET_WRITE_REF_DIGESTS"):
        stored[key] = d
        with open(REF_DIGESTS, "w") as f:
            json.dump(stored, f, indent=1, sort_keys=True)
            f.write("\n")
    else:
        assert stored.get(key) == d, "the compiled reference no longer gives the stored digest for %s" % key
    return d


# ---- models printed in the reference's nnet_data.c / nnet_data.h form (oracle/dump_nnet_data.py) and imported ----
DUMP_GEN = GEN + "_dump"
DUMP_REF = os.path.join(ORACLE, "_ref", "dump")


@functools.lru_cache(None)
def dump_dir(model):
    """oracle/_gen_dump/<model>: nnet_data.c / nnet_data.h of dump_nnet_data.MODELS[model], written on first use."""
    import dump_nnet_data
    d = os.path.join(DUMP_GEN, model)
    if not all(os.path.exists(os.path.join(d, n)) for n in ("nnet_data.c", "nnet_data.h")):
        dump_nnet_data.write_model(DUMP_GEN, model)
    return d


def _importer():
    import sys
    tools = os.path.join(ROOT, "tools")
    if tools not in sys.path:
        sys.path.insert(0, tools)
    import import_nnet_data
    return import_nnet_data


@functools.lru_cache(None)
def imported(model, kind="int8"):
    """(blob, arrays, config) of tools/import_nnet_data.py run on the dumped model (kind int8, or float: --float)."""
    return _importer().import_model(os.path.join(dump_dir(model), "nnet_data.c"), is_float=kind == "float")


def have_dump_ref(model, blobs=False):
    """oracle/Makefile `dumpref` built the reference from this model's nnet_data.c (builds A and B; with blobs: the blobs
    write_lpcnet_weights wrote)."""
    files = ("weights_int8.bin", "weights_float.bin") if blobs else ("liblpcnet_ref_A.so", "liblpcnet_ref_B.so")
    return all(os.path.exists(os.path.join(DUMP_REF, model, f)) for f in files)


def dump_ref_blob(model, kind):
    """The blob write_lpcnet_weights wrote, compiled against the model's nnet_data.c (kind int8: DOT_PROD, float: not)."""
    return open(os.path.join(DUMP_REF, model, "weights_%s.bin" % kind), "rb").read()


@functools.lru_cache(None)
def _dump_ref_lib(model, build):
    L = ctypes.CDLL(os.path.join(DUMP_REF, model, "liblpcnet_ref_%s.so" % build))
    L.ref_synth_batch.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    L.ref_decode_batch.argtypes = [ctypes.c_char_p, ctypes.c_int, c_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_p]
    return L


def dump_ref_synth(model, build, features):
    """features [n][T][stride] -> pcm [n][T*160] of the reference built from the model's nnet_data.c (build A: int8, B: float)
    on its compiled-in arrays: no blob is loaded."""
    f = np.ascontiguousarray(features, dtype=np.float32)
    n, T, stride = f.shape
    pcm = np.zeros((n, T * 160), dtype=np.int16)
    assert _dump_ref_lib(model, build).ref_synth_batch(None, 0, f.ctypes.data, stride, T, n, n, pcm.ctypes.data) == 0
    return pcm


def dump_ref_decode(model, build, packets):
    """packets [n][P][8] -> pcm [n][P*640], as dump_ref_synth."""
    p = np.ascontiguousarray(packets, dtype=np.uint8)
    n, P, _ = p.shape
    pcm = np.zeros((n, P * 640), dtype=np.int16)
    assert _dump_ref_lib(model, build).ref_decode_batch(None, 0, p.ctypes.data, P, n, n, pcm.ctypes.data) == 0
    return pcm


def oracle_with_config(model_blob, cfg, features=None, packets=None, nthreads=8):
    """pcm of the CPU restatement on `model_blob` with the switches cfg = (lpc_gamma, features_delay, end2end): synthesis of
    features [n][T][stride] or decode of packets [n][P][8]."""
    L = oracle_lib()
    m = L.oracle_model_create_ex(model_blob, len(model_blob), rcp_table().ctypes.data, cfg[0], int(cfg[1]), int(cfg[2]),
                                 codebooks().ctypes.data)
    assert m, "oracle failed to parse the blob"
    L.oracle_model_destroy.argtypes = [c_p]
    try:
        if features is not None:
            f = np.ascontiguousarray(features, dtype=np.float32)
            n, T, stride = f.shape
            pcm = np.zeros((n, T * 160), dtype=np.int16)
            L.oracle_synthesize_batch(m, f.ctypes.data, stride, n, T, nthreads, pcm.ctypes.data)
        else:
            p = np.ascontiguousarray(packets, dtype=np.uint8)
            n, P, _ = p.shape
            pcm = np.zeros((n, P * 640), dtype=np.int16)
            L.oracle_decode_batch(m, p.ctypes.data, n, P, nthreads, pcm.ctypes.data)
    finally:
        L.oracle_model_destroy(m)
    return pcm


def stream_digests(pcm):
    """First 8 bytes of sha256 of every stream's PCM as uint64 [n] (a failing comparison names the stream)."""
    import hashlib
    return np.array([int.from_bytes(hashlib.sha256(np.ascontiguousarray(r).tobytes()).digest()[:8], "little") for r in pcm], dtype=np.uint64)


# ---- the analysis side (SURVEY 8f N2): the compiled reference's encoder entry points, one fresh state per stream ----
def ref_features(pcm, build="A"):
    """pcm [n][T*160] int16 (or float32) -> features [n][T][36] via lpcnet_compute_single_frame_features(_float)."""
    L = ref_lib(build)
    p = np.ascontiguousarray(pcm)
    n, T = p.shape[0], p.shape[1] // 160
    out = np.zeros((n, T, 36), np.float32)
    for s in range(n):
        row = np.ascontiguousarray(p[s])
        (L.ref_features_stream_float if p.dtype == np.float32 else L.ref_features_stream)(row.ctypes.data, T, out[s].ctypes.data)
    return out


def ref_encode(pcm, build="A"):
    """pcm [n][P*640] int16 -> packets [n][P][8] via lpcnet_encode."""
    L = ref_lib(build)
    p = np.ascontiguousarray(pcm, dtype=np.int16)
    n, P = p.shape[0], p.shape[1] // 640
    out = np.zeros((n, P, 8), np.uint8)
    for s in range(n):
        L.ref_encode_stream(p[s].ctypes.data, P, out[s].ctypes.data)
    return out


def ref_features4(pcm, build="A"):
    """pcm [n][P*640] int16 -> features [n][P*4][36] via lpcnet_compute_features."""
    L = ref_lib(build)
    p = np.ascontiguousarray(pcm, dtype=np.int16)
    n, P = p.shape[0], p.shape[1] // 640
    out = np.zeros((n, P * 4, 36), np.float32)
    for s in range(n):
        L.ref_features4_stream(p[s].ctypes.data, P, out[s].ctypes.data)
    return out


# ---- CPU restatement of the analysis side (oracle/lpcnet_enc_oracle.inc), one fresh state per stream ----
def oracle_features(pcm):
    """pcm [n][T*160] int16 (or float32: the _float entry point) -> features [n][T][36]."""
    L = oracle_lib()
    is_float = np.asarray(pcm).dtype == np.float32
    p = np.ascontiguousarray(pcm, dtype=np.float32 if is_float else np.int16)
    fn = L.oracle_enc_single_frame_features_float if is_float else L.oracle_enc_single_frame_features
    n, T = p.shape[0], p.shape[1] // 160
    out = np.zeros((n, T, 36), np.float32)
    for s in range(n):
        e = L.oracle_enc_create(None)
        for t in range(T):
            fn(e, p[s, t * 160:].ctypes.data, out[s, t].ctypes.data)
        L.oracle_enc_destroy(e)
    return out


def oracle_encode_slopes(pcm):
    """pcm [P*640] int16 of one stream -> (packets [P][8], pitch slope best_a of each superframe before the voicing decision)."""
    L = oracle_lib()
    p = np.ascontiguousarray(pcm, dtype=np.int16)
    P = p.shape[0] // 640
    cb = codebooks()
    out, slopes = np.zeros((P, 8), np.uint8), np.zeros(P, np.float32)
    e = L.oracle_enc_create(cb.ctypes.data)
    for k in range(P):
        L.oracle_enc_encode(e, p[k * 640:].ctypes.data, out[k].ctypes.data)
        slopes[k] = L.oracle_enc_last_best_a(e)
    L.oracle_enc_destroy(e)
    return out, slopes


def oracle_frame_taps(features, kind="int8"):
    """features [n][T][stride] -> (gru_a cond [n][T][3*na], gru_b cond [n][T][48], weighted lpc [n][T][16]) of the CPU
    restatement's run_frame_network on a fresh state per stream."""
    L = oracle_lib()
    f = np.ascontiguousarray(features, dtype=np.float32)
    n, T, _ = f.shape
    m = oracle_model(kind)
    na = L.oracle_model_na(m)
    ga, gb, lpc = np.zeros((n, T, 3 * na), np.float32), np.zeros((n, T, 48), np.float32), np.zeros((n, T, 16), np.float32)
    for s in range(n):
        st = L.oracle_state_create(m)
        for t in range(T):
            L.oracle_frame_network(st, f[s, t].ctypes.data, ga[s, t].ctypes.data, gb[s, t].ctypes.data, lpc[s, t].ctypes.data)
        L.oracle_state_destroy(st)
    return ga, gb, lpc


def ref_frame_taps(features, build="A"):
    """The same taps from the compiled reference's run_frame_network (ref_shim.c ref_frame_network)."""
    L = ref_lib(build)
    b = blob("float" if build in ("B", "TB") else "int8")
    f = np.ascontiguousarray(features, dtype=np.float32)
    n, T, stride = f.shape
    na = 384
    ga, gb, lpc = np.zeros((n, T, 3 * na), np.float32), np.zeros((n, T, 48), np.float32), np.zeros((n, T, 16), np.float32)
    for s in range(n):
        assert L.ref_frame_network(b, len(b), f[s].ctypes.data, stride, T, ga[s].ctypes.data, gb[s].ctypes.data, lpc[s].ctypes.data) == 0
    return ga, gb, lpc


def oracle_encode(pcm, features4=False):
    """pcm [n][P*640] -> packets [n][P][8] (lpcnet_encode), or with features4 the unquantised features [n][P*4][36] (lpcnet_compute_features)."""
    L = oracle_lib()
    p = np.ascontiguousarray(pcm, dtype=np.int16)
    n, P = p.shape[0], p.shape[1] // 640
    cb = codebooks()
    out = np.zeros((n, P * 4, 36), np.float32) if features4 else np.zeros((n, P, 8), np.uint8)
    for s in range(n):
        e = L.oracle_enc_create(cb.ctypes.data)
        for k in range(P):
            if features4:
                L.oracle_enc_compute_features(e, p[s, k * 640:].ctypes.data, out[s, 4 * k].ctypes.data)
            else:
                L.oracle_enc_encode(e, p[s, k * 640:].ctypes.data, out[s, k].ctypes.data)
        L.oracle_enc_destroy(e)
    return out
