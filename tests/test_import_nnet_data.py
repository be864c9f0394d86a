"""Real-model entry: a model in the nnet_data.c / nnet_data.h form training_tf2/dump_lpcnet.py prints (oracle/dump_nnet_data.py
writes every generated model that way) through tools/import_nnet_data.py, checked against two ground truths built by the
reference from the same file (oracle/Makefile `dumpref`): the blob src/write_lpcnet_weights.c writes, and the reference's
PCM on its compiled-in arrays (no USE_WEIGHTS_FILE, the C compiler converting the decimals).  Where the reference is not
built, the digests in tests/golden/ref_digests.json stand in for it."""
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import dump_nnet_data as D
import gen_model
import helpers as H
import lpcnet_b200
from fixtures import make_feature_batch, make_packets

MODELS = list(D.MODELS)
KINDS = ("int8", "float")
BUILD = {"int8": "A", "float": "B"}
CONFIG = "lpcnet_b200_config"


def features():
    return make_feature_batch(range(3), 8)


def packets():
    return np.stack([make_packets(s, 3) for s in range(2)])


def _lpcnet_records(blob):
    """[(name, type, bytes)] of a blob without the importer's config record."""
    return [r for r in lpcnet_b200.parse_blob(blob) if r[0] != CONFIG]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("model", MODELS)
def test_import_equals_write_lpcnet_weights(model, kind):
    """The importer's blob is what write_lpcnet_weights compiled against the same nnet_data.c writes: names, order, type ids
    and bytes of every lpcnet_arrays[] record (the config record is the importer's own addition)."""
    blob, _, _ = H.imported(model, kind)
    got = _lpcnet_records(blob)
    if H.have_dump_ref(model, blobs=True):
        want = lpcnet_b200.parse_blob(H.dump_ref_blob(model, kind))
        assert [r[0] for r in got] == [r[0] for r in want]
        for (name, t, d), (_, t_ref, d_ref) in zip(got, want):
            assert t == t_ref, "%s: type id %d, write_lpcnet_weights %d" % (name, t, t_ref)
            assert d == d_ref, "%s: bytes differ from write_lpcnet_weights" % name
    stored = H.ref_digest("dump_%s_wlw_%s" % (model, kind), lambda: np.frombuffer(H.dump_ref_blob(model, kind), np.uint8),
                          runnable=H.have_dump_ref(model, blobs=True))
    assert H.digest(np.frombuffer(lpcnet_b200.write_blob(got), np.uint8)) == stored


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("model", MODELS)
def test_import_equals_generated_arrays(model, kind):
    """...and every array is the generator's own, bit for bit, with the generator's type id."""
    common, only8, onlyf = D.MODELS[model][0]()
    want = {n: (t, np.ascontiguousarray(a).tobytes()) for n, t, a in common + (only8 if kind == "int8" else onlyf)}
    got = {n: (t, d) for n, t, d in _lpcnet_records(H.imported(model, kind)[0])}
    assert sorted(got) == sorted(want)
    for n in want:
        assert got[n][0] == want[n][0], "%s: type id %d, generator %d" % (n, got[n][0], want[n][0])
        assert got[n][1] == want[n][1], "%s: values differ from the generator's" % n


@pytest.mark.parametrize("model", MODELS)
def test_config_record_matches_header(model):
    """LPC_GAMMA, FEATURES_DELAY and END2END (defined, or commented out) of nnet_data.h land in the blob's config record."""
    gamma, delay, e2e = D.header_config(model)
    for kind in KINDS:
        blob, _, cfg = H.imported(model, kind)
        assert cfg == {"lpc_gamma": gamma, "features_delay": delay, "end2end": int(e2e)}
        assert lpcnet_b200.blob_config(blob) == (float(np.float32(gamma)), delay, int(e2e))
    header = open(os.path.join(H.dump_dir(model), "nnet_data.h")).read()
    assert ("/* #define END2END */" in header) == (not e2e)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("model", MODELS)
def test_oracle_on_imported_blob_matches_compiled_in_reference(model, kind):
    """The CPU restatement loaded from the imported blob, with the switches of its config record, gives the PCM of the
    reference built from nnet_data.c with the arrays compiled in: synthesis and decode."""
    blob, _, _ = H.imported(model, kind)
    cfg = lpcnet_b200.blob_config(blob)
    build, run = BUILD[kind], H.have_dump_ref(model)
    f, p = features(), packets()
    want = H.ref_digest("dump_%s_%s_synth" % (model, build), lambda: H.dump_ref_synth(model, build, f), runnable=run)
    assert H.digest(H.oracle_with_config(blob, cfg, features=f)) == want
    want = H.ref_digest("dump_%s_%s_decode" % (model, build), lambda: H.dump_ref_decode(model, build, p), runnable=run)
    assert H.digest(H.oracle_with_config(blob, cfg, packets=p)) == want


def _round_to_float32(lit):
    """The float32 nearest to the decimal literal (ties to even), computed exactly."""
    x = Fraction(lit)
    a = np.float32(float(x))
    cands = [a, np.nextafter(a, np.float32(-np.inf)), np.nextafter(a, np.float32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c).view(np.uint32)) & 1))


def test_hand_picked_literals_round_through_double():
    """The literals of dump_nnet_data.TIE_ARRAY that sit just beyond a float32 rounding midpoint: gcc converts them
    decimal -> double -> float (write_lpcnet_weights' blob and the compiled-in reference agree with the import above), and so
    must the importer; rounding each decimal to float32 directly would give the neighbour."""
    common, _, _ = D.MODELS["default"][0]()
    a = dict((n, x) for n, _, x in common)[D.TIE_ARRAY].reshape(-1)
    lits = D.tie_literals(a)
    assert len(lits) == D.TIE_COUNT
    text = open(os.path.join(H.dump_dir("default"), "nnet_data.c")).read()
    got = dict((n, x) for n, _, x in H.imported("default")[1])[D.TIE_ARRAY]
    for i, lit in lits.items():
        assert lit in text
        assert got[i].view(np.uint32) == a[i].view(np.uint32), (i, lit)
        assert _round_to_float32(lit) != a[i], "literal %s is not a double-rounding case" % lit


def test_header_defaults_and_comments():
    """A header without the defines gives gamma 1, delay 2, not end-to-end; commented-out defines do not count."""
    imp = H._importer()
    assert imp.parse_header("#ifndef RNN_DATA_H\n#define RNN_DATA_H\n#include \"nnet.h\"\n#endif\n") == \
        {"lpc_gamma": 1.0, "features_delay": 2, "end2end": 0}
    hand_edited = ("/* This is *not* an end-to-end model\n#define END2END\n*/\n"
                   "/* #define LPC_GAMMA 0.5f */\n// #define FEATURES_DELAY 0\n"
                   "#define LPC_GAMMA 0.85f\n#define FEATURES_DELAY 1\n")
    assert imp.parse_header(hand_edited) == {"lpc_gamma": 0.85, "features_delay": 1, "end2end": 0}
    assert imp.parse_header("  #  define END2END\n#define LPC_GAMMA 1e0f\n") == {"lpc_gamma": 1.0, "features_delay": 2, "end2end": 1}


def test_no_header_no_config_record(tmp_path):
    """Without nnet_data.h next to nnet_data.c the blob has no config record (the caller then passes the switches)."""
    os.symlink(os.path.join(H.dump_dir("na128"), "nnet_data.c"), str(tmp_path / "nnet_data.c"))
    blob, _, cfg = H._importer().import_model(str(tmp_path / "nnet_data.c"))
    assert cfg is None and lpcnet_b200.blob_config(blob) is None
    assert lpcnet_b200.parse_blob(blob) == _lpcnet_records(H.imported("na128")[0])


def test_refusals():
    """A count that disagrees with the initialisers, and a file without arrays (a USE_WEIGHTS_FILE-only nnet_data.c), are
    refused rather than imported short."""
    imp = H._importer()
    with pytest.raises(ValueError, match="2 initialisers for 3"):
        imp.parse_arrays("static const float a[3] = {\n   1.0, 2.0\n};\n")
    with pytest.raises(ValueError, match="2 initialisers for 3"):
        imp.parse_arrays("#ifdef DOT_PROD\nstatic const qweight w[2] = {1, 2};\n#else\nstatic const qweight w[3] = {1.0, 2.0};\n#endif\n",
                         dot_prod=False)
    only_init = gen_model.NNET_DATA_C.format(n3a=1152, n3b=48, embed=128, pembed=64, cond=128, fin=84, na=384, nb=16)
    with pytest.raises(ValueError, match="no `static const"):
        imp.parse_arrays(only_init)
    with pytest.raises(ValueError, match="no `static const"):
        imp.parse_arrays("#ifdef DOT_PROD\nstatic const qweight w[2] = {1, 2};\n#endif\n", dot_prod=False)


@pytest.mark.parametrize("kind", KINDS)
def test_script_writes_the_same_bytes(tmp_path, kind):
    """`python tools/import_nnet_data.py nnet_data.c -o blob` writes the bytes import_model returns."""
    out = tmp_path / "w.bin"
    cmd = [sys.executable, os.path.join(H.ROOT, "tools", "import_nnet_data.py"), os.path.join(H.dump_dir("na128"), "nnet_data.c"),
           "-o", str(out)] + (["--float"] if kind == "float" else [])
    subprocess.check_call(cmd, stdout=subprocess.DEVNULL)
    assert out.read_bytes() == H.imported("na128", kind)[0]
