"""Groups against separate member calls on one GPU: K int8 models of 384 units served (a) by K member `_device` calls back to
back, (b) by one group `_device` call, and, as the bound, (c) by one single-model batch of the same total.

Members are gen_model.make_model(seed) models with different seeds ("seeds") or K batches loading the same blob ("same"), which
separates the launch plan from the L2 footprint of K models' embedding tables.  Sizes: 4096 streams in total (4096 / K per
member) and 1024 streams per member.  Every step synthesizes 10 frames (160 samples each) per stream; timed with CUDA events
on one caller stream after warm-up.  Prints one JSON line per case plus the card's name and power limit.

--flavour float measures float models instead (gen_model.make_model(seed) float blobs, seeded members only) at 32, 64, 128 and
1024 streams per member: these sizes reach both float kernels (neuron-per-lane at up to 4 streams per CTA, lane == stream above)
and the batches that leave SMs idle on their own.

    python tools/bench_group.py [--steps 10] [--warmup 3] [--ks 1,2,4,8] [--flavour int8|float]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

FRAMES, SPF = 10, 160


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        out = "unavailable (%s)" % e
    return out


def blob_for(seed, flavour="int8"):
    import gen_model
    import lpcnet_b200
    common, only8, onlyf = gen_model.make_model(seed)
    return lpcnet_b200.write_blob([(n, t, a.tobytes()) for n, t, a in common + (onlyf if flavour == "float" else only8)])


def features(n, torch):
    from fixtures import make_feature_batch
    pool = make_feature_batch(range(97), FRAMES)
    f = pool[np.arange(n) % 97]
    return torch.from_numpy(np.ascontiguousarray(f)).cuda()


def timed(fn, steps, warmup, torch, stream):
    for _ in range(warmup):
        fn()
    stream.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def run_case(lpcnet_b200, torch, blobs, per_member, steps, warmup):
    import helpers as H
    K = len(blobs)
    n = K * per_member
    batches = [lpcnet_b200.Batch(per_member, b, device=0, config=H.model_config("")) for b in blobs]
    group = lpcnet_b200.Group(batches)
    d_f = features(n, torch)
    d_p = torch.zeros((n, FRAMES * SPF), dtype=torch.int16, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    fstep, pstep = per_member * FRAMES * 20, per_member * FRAMES * SPF

    def members():
        for k, b in enumerate(batches):
            b.synthesize_device(d_f.data_ptr() + 4 * k * fstep, FRAMES, 20, d_p.data_ptr() + 2 * k * pstep, SPF, s.cuda_stream)

    def grouped():
        group.synthesize_device(d_f.data_ptr(), FRAMES, 20, d_p.data_ptr(), SPF, s.cuda_stream)

    ms_a = timed(members, steps, warmup, torch, s)
    ker_a = sum(b.last_sample_kernel_ms()[0] for b in batches)
    ms_b = timed(grouped, steps, warmup, torch, s)
    ker_b, _ = group.last_sample_kernel_ms()
    group.close()
    for b in batches:
        b.close()
    single = lpcnet_b200.Batch(n, blobs[0], device=0, config=H.model_config(""))
    ms_c = timed(lambda: single.synthesize_device(d_f.data_ptr(), FRAMES, 20, d_p.data_ptr(), SPF, s.cuda_stream), steps, warmup, torch, s)
    ker_c, _ = single.last_sample_kernel_ms()
    single.close()
    samples = n * FRAMES * SPF
    return dict(members=K, streams_per_member=per_member, streams=n,
                a_member_calls=dict(ms=round(ms_a, 3), samples_per_s=samples / ms_a * 1e3, sample_kernel_ms=round(ker_a, 3)),
                b_group_call=dict(ms=round(ms_b, 3), samples_per_s=samples / ms_b * 1e3, sample_kernel_ms=round(ker_b, 3)),
                c_single_batch=dict(ms=round(ms_c, 3), samples_per_s=samples / ms_c * 1e3, sample_kernel_ms=round(ker_c, 3)),
                b_over_a=round(ms_a / ms_b, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ks", default="1,2,4,8")
    ap.add_argument("--flavour", choices=["int8", "float"], default="int8")
    a = ap.parse_args()
    import torch
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    print(json.dumps(dict(card=card())), flush=True)
    ks = [int(k) for k in a.ks.split(",")]
    seeded = [blob_for(1234 + 17 * i, a.flavour) for i in range(max(ks))]
    if a.flavour == "float":
        for per_member in (32, 64, 128, 1024):
            for K in ks:
                r = run_case(lpcnet_b200, torch, seeded[:K], per_member, a.steps, a.warmup)
                r.update(models="seeds", flavour="float")
                print(json.dumps(r), flush=True)
        print(json.dumps(dict(card=card())), flush=True)
        return
    for models in ("seeds", "same"):
        for K in ks:
            if models == "same" and K == 1:
                continue
            blobs = seeded[:K] if models == "seeds" else [seeded[0]] * K
            for per_member in sorted({4096 // K, 1024}):
                r = run_case(lpcnet_b200, torch, blobs, per_member, a.steps, a.warmup)
                r["models"] = models
                print(json.dumps(r), flush=True)
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
