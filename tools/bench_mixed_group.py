"""Mixed groups against one group call per shape: models of several shapes (GRU_A size, int8 or float) on one device, K models per
shape of n streams each (gen_model.make_model(seed), a different seed per model), served by
  (a) one lpcnet_b200_mixed_group_synthesize_device call;
  (b) one ordinary group call per shape, back to back on one CUDA stream (each group planned over the whole chip);
  (c) the same group calls, each on a CUDA stream of its own: the concurrency a caller could try without a mixed group.

Every call synthesizes 10 frames (160 samples each) per stream from device features into device PCM.  Wall time per call is a host
clock around calls that end in a device synchronise, averaged over --steps calls after --warmup.  For every variant it also reports
each shape's per-sample kernel time in the last call (lpcnet_b200_group_last_sample_kernel_ms), and for (a) the device time from
fork to join (lpcnet_b200_mixed_group_last_call_ms).  Prints one JSON line per case, and the card's name and power limit before
and after.

    python tools/bench_mixed_group.py [--mixes i384+i128,i384+i256+i128,i384+f384] [--ks 1,2,4] [--streams 64,256,1024]
                                      [--steps 5] [--warmup 2]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

FRAMES, SPF = 10, 160


def cards():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        out = "unavailable (%s)" % e
    return out.splitlines()


def blob_for(kind, na, seed):
    import gen_model
    import lpcnet_b200
    common, only8, onlyf = gen_model.make_model(seed, na=na)
    return lpcnet_b200.write_blob([(n, t, a.tobytes()) for n, t, a in common + (onlyf if kind == "f" else only8)])


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def run_case(lpcnet_b200, shapes, K, per_model, steps, warmup):
    import torch
    import helpers as H
    from fixtures import make_feature_batch
    batches = []                          # shape by shape, so that each shape's rows are one block
    for i, (kind, na) in enumerate(shapes):
        for k in range(K):
            blob = blob_for(kind, na, 1234 + 17 * k + 101 * i)
            batches.append(lpcnet_b200.Batch(per_model, blob, device=0, config=H.model_config("" if na == 384 else "na%d" % na)))
    mg = lpcnet_b200.MixedGroup(batches)
    assert mg.classes == len(shapes)
    groups = [lpcnet_b200.Group(batches[i * K:(i + 1) * K]) for i in range(len(shapes))]
    n = len(batches) * per_model
    pool = make_feature_batch(range(97), FRAMES)
    d_f = torch.from_numpy(np.ascontiguousarray(pool[np.arange(n) % 97])).cuda()
    d_p = torch.zeros((n, FRAMES * SPF), dtype=torch.int16, device="cuda")
    rows = K * per_model
    fstep, pstep = rows * FRAMES * 20 * 4, rows * FRAMES * SPF * 2
    main_st = torch.cuda.current_stream()
    side = [torch.cuda.Stream() for _ in shapes]

    def mixed():
        mg.synthesize_device(d_f.data_ptr(), FRAMES, 20, d_p.data_ptr(), SPF, main_st.cuda_stream)

    def per_shape(streams):
        for i, g in enumerate(groups):
            g.synthesize_device(d_f.data_ptr() + i * fstep, FRAMES, 20, d_p.data_ptr() + i * pstep, SPF, streams[i].cuda_stream)

    samples = n * FRAMES * SPF
    out = dict(shapes=["%s%d" % s for s in shapes], models_per_shape=K, streams_per_model=per_model, streams=n)
    res = {}
    for name, fn, kern in (("a_mixed_call", mixed, [mg.group(c) for c in range(mg.classes)]),
                           ("b_sequential_groups", lambda: per_shape([main_st] * len(shapes)), groups),
                           ("c_groups_on_own_streams", lambda: per_shape(side), groups)):
        ms = timed(fn, steps, warmup)
        res[name] = dict(ms=round(ms, 3), samples_per_s=samples / ms * 1e3,
                         sample_kernel_ms_per_shape=[round(g.last_sample_kernel_ms()[0], 3) for g in kern])
        if name == "a_mixed_call":
            res[name]["fork_to_join_ms"] = round(mg.last_call_ms(), 3)
    out.update(res)
    out["b_over_a"] = round(res["b_sequential_groups"]["ms"] / res["a_mixed_call"]["ms"], 3)
    out["c_over_a"] = round(res["c_groups_on_own_streams"]["ms"] / res["a_mixed_call"]["ms"], 3)
    for g in groups:
        g.close()
    mg.close()
    for b in batches:
        b.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mixes", default="i384+i128,i384+i256+i128,i384+f384", help="shapes per mix: i (int8) or f (float) + GRU_A size")
    ap.add_argument("--ks", default="1,2,4", help="models per shape")
    ap.add_argument("--streams", default="64,256,1024", help="streams per model")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    if lpcnet_b200.device_count() < 1:
        raise SystemExit("no CUDA device is visible")
    print(json.dumps(dict(cards=cards())), flush=True)
    for mix in a.mixes.split(","):
        shapes = [(s[0], int(s[1:])) for s in mix.split("+")]
        for per_model in [int(s) for s in a.streams.split(",")]:
            for K in [int(k) for k in a.ks.split(",")]:
                print(json.dumps(run_case(lpcnet_b200, shapes, K, per_model, a.steps, a.warmup)), flush=True)
    print(json.dumps(dict(cards=cards())), flush=True)


if __name__ == "__main__":
    main()
