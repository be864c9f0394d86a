"""Multi-GPU groups against one Multi call per model: K int8 models (gen_model.make_model(seed), different seeds) of n streams each,
every model sharded over --devices, served (a) by K lpcnet_b200_multi_synthesize calls back to back and (b) by one
lpcnet_b200_multi_group_synthesize call, each with the PCM to the host and gathered on devices[0] (`_gather`).

Every call synthesizes 10 frames (160 samples each) per stream from host features.  Wall time per call is a host clock around
calls that end in a device synchronise, averaged over --steps calls after --warmup.  For (b) it also reports each device's
per-sample kernel time in the last call (lpcnet_b200_group_last_sample_kernel_ms of multi_group_group(k)).  Prints one JSON line
per case, and the name and power limit of every card used, before and after.

    python tools/bench_multi_group.py [--devices 0,1] [--ks 2,4,8] [--streams 512,2048] [--steps 5] [--warmup 2]"""
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


def cards(devices):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", ",".join(str(d) for d in devices)], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:      # noqa: BLE001
        out = "unavailable (%s)" % e
    return out.splitlines()


def blob_for(seed):
    import gen_model
    import lpcnet_b200
    common, only8, _ = gen_model.make_model(seed)
    return lpcnet_b200.write_blob([(n, t, a.tobytes()) for n, t, a in common + only8])


def features(n):
    from fixtures import make_feature_batch
    pool = make_feature_batch(range(97), FRAMES)
    return np.ascontiguousarray(pool[np.arange(n) % 97])


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    return (time.perf_counter() - t0) / steps * 1e3


def run_case(lpcnet_b200, blobs, per_model, devices, steps, warmup):
    import helpers as H
    L = lpcnet_b200.lib()
    K = len(blobs)
    n = K * per_model
    multis = [lpcnet_b200.Multi(per_model, b, devices, config=H.model_config("")) for b in blobs]
    mg = lpcnet_b200.MultiGroup(multis)
    f = features(n)
    pcm = np.zeros((n, FRAMES * SPF), np.int16)
    d_gather = L.lpcnet_b200_device_alloc_on(devices[0], pcm.nbytes)
    fstep, pstep = per_model * FRAMES * 20 * 4, per_model * FRAMES * SPF * 2

    def ok(r):
        if r != 0:
            raise lpcnet_b200.LPCNetB200Error(lpcnet_b200.api._err())

    def per_model_calls(gather):
        for k, m in enumerate(multis):
            if gather:
                ok(L.lpcnet_b200_multi_synthesize_gather(m._h, f.ctypes.data + k * fstep, FRAMES, 20, SPF, d_gather + k * pstep))
            else:
                ok(L.lpcnet_b200_multi_synthesize(m._h, f.ctypes.data + k * fstep, FRAMES, 20, SPF, pcm.ctypes.data + k * pstep))

    def one_call(gather):
        if gather:
            ok(L.lpcnet_b200_multi_group_synthesize_gather(mg._h, f.ctypes.data, FRAMES, 20, SPF, d_gather))
        else:
            ok(L.lpcnet_b200_multi_group_synthesize(mg._h, f.ctypes.data, FRAMES, 20, SPF, pcm.ctypes.data))

    samples = n * FRAMES * SPF
    out = dict(models=K, streams_per_model=per_model, streams=n, devices=devices, peer_access=multis[0].peer_access())
    for gather in (False, True):
        ms_a = timed(lambda: per_model_calls(gather), steps, warmup)
        ms_b = timed(lambda: one_call(gather), steps, warmup)
        ker = [round(mg.group(k).last_sample_kernel_ms()[0], 3) for k in range(len(devices))]
        out["gather" if gather else "host"] = dict(
            a_multi_calls=dict(ms=round(ms_a, 3), samples_per_s=samples / ms_a * 1e3),
            b_multi_group_call=dict(ms=round(ms_b, 3), samples_per_s=samples / ms_b * 1e3, sample_kernel_ms_per_device=ker),
            b_over_a=round(ms_a / ms_b, 3))
    L.lpcnet_b200_device_free(d_gather)
    mg.close()
    for m in multis:
        m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0")
    ap.add_argument("--ks", default="2,4,8")
    ap.add_argument("--streams", default="512,2048", help="streams per model")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import lpcnet_b200
    from lpcnet_b200 import build
    build.build()
    devices = [int(d) for d in a.devices.split(",")]
    if lpcnet_b200.device_count() < len(devices):
        raise SystemExit("%d devices requested, %d visible" % (len(devices), lpcnet_b200.device_count()))
    print(json.dumps(dict(cards=cards(devices))), flush=True)
    ks = [int(k) for k in a.ks.split(",")]
    blobs = [blob_for(1234 + 17 * i) for i in range(max(ks))]
    for per_model in [int(s) for s in a.streams.split(",")]:
        for K in ks:
            print(json.dumps(run_case(lpcnet_b200, blobs[:K], per_model, devices, a.steps, a.warmup)), flush=True)
    print(json.dumps(dict(cards=cards(devices))), flush=True)


if __name__ == "__main__":
    main()
