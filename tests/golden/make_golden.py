#!/usr/bin/env python3
"""Regenerates the committed golden vectors by running the UNTOUCHED reference (oracle/_ref, built from
/root/reference by `make -C oracle ref`) on the deterministic synthetic model + fixtures.

Run in the build container only (needs /root/reference).  The reference holds no golden vectors of its own
(SURVEY.md 4: no test-suite, no known-answer data), so these files are the pin for the oracle and the engine.

  synth_A.npz   int8  build A : pcm[4][40*160]   for streams 0..3            (lpcnet_synthesize)
  synth_B.npz   float build B : same streams
  decode_A.npz  int8  build A : pcm[3][6*640]    for packet streams 0..2    (lpcnet_decode)
  digests.json  sha256 of larger runs (16 streams x 150 frames A and B; 8 streams x 25 packets) + CPU model
"""
import hashlib, json, os, sys
import numpy as np
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle"))
import helpers as H
from fixtures import make_feature_batch, make_packets

f = make_feature_batch(range(4), 40)
np.savez_compressed(os.path.join(HERE, "synth_A.npz"), pcm=H.ref_synth(f, "A"))
np.savez_compressed(os.path.join(HERE, "synth_B.npz"), pcm=H.ref_synth(f, "B"))
p = np.stack([make_packets(s, 6) for s in range(3)])
np.savez_compressed(os.path.join(HERE, "decode_A.npz"), pcm=H.ref_decode(p, "A"))

big = make_feature_batch(range(16), 150)
pk = np.stack([make_packets(s, 25) for s in range(8)])
cpu = [l.split(":")[1].strip() for l in open("/proc/cpuinfo") if l.startswith("model name")][0]
dig = {
    "cpu": cpu,
    "model_int8_sha256": hashlib.sha256(H.blob("int8")).hexdigest(),
    "model_float_sha256": hashlib.sha256(H.blob("float")).hexdigest(),
    "codebooks_sha256": hashlib.sha256(H.codebooks().tobytes()).hexdigest(),
    "synth_A_16x150": hashlib.sha256(H.ref_synth(big, "A").tobytes()).hexdigest(),
    "synth_B_16x150": hashlib.sha256(H.ref_synth(big, "B").tobytes()).hexdigest(),
    "decode_A_8x25": hashlib.sha256(H.ref_decode(pk, "A").tobytes()).hexdigest(),
}
json.dump(dig, open(os.path.join(HERE, "digests.json"), "w"), indent=1)
print(json.dumps(dig, indent=1))

# ---- model variants (SURVEY 8f N1): the reference compiled with each variant's generated nnet_data.h (oracle/Makefile VARIANTS)
var = {}
fv = make_feature_batch(range(2), 20)
for tag in ("na256", "na128", "e2e", "delay0", "na256e2e", "delay1"):
    for build in ("A", "B"):
        var["%s_%s" % (tag, build)] = H.ref_synth(fv, build, tag=tag)
np.savez_compressed(os.path.join(HERE, "variants.npz"), **var)
