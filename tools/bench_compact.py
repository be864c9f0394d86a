"""Compaction on one GPU: what a step costs a 4096-row batch that carries only L live sessions, what it costs after those L
streams were copied into an L-row batch (lpcnet_b200_batch_copy_streams), and what the copy itself costs.

A 4096-row int8 batch of the default 384-unit test model runs warm-up steps on all rows; L rows spread over the batch are the
live ones.  Per L in --live: the per-sample kernel time of a 10-frame step (CUDA events, lpcnet_b200_batch_last_sample_kernel_ms)
on the 4096-row batch, the wall time of copy_streams into an L-row batch (a host clock around the call, which returns after a
synchronise), and the per-sample kernel time of the same 10-frame step on the L-row batch.  Prints the card's name and power
limit, then one JSON line per L.

    python tools/bench_compact.py [--steps 5] [--copies 5] [--live 256,1024,2048]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

N, FRAMES = 4096, 10


def kernel_ms(b, f, steps):
    """median per-sample kernel ms of `steps` 10-frame steps"""
    ms = []
    for _ in range(steps):
        b.synthesize(f)
        ms.append(b.last_sample_kernel_ms()[0])
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--copies", type=int, default=5)
    ap.add_argument("--live", default="256,1024,2048")
    a = ap.parse_args()
    import lpcnet_b200
    from lpcnet_b200 import build
    from bench_group import card
    from fixtures import make_feature_batch
    import helpers as H
    build.build()
    print(json.dumps(dict(card=card())), flush=True)
    blob = H.blob("int8")
    f = make_feature_batch(range(97), FRAMES)[np.arange(N) % 97]
    big = lpcnet_b200.Batch(N, blob, device=0, config=H.model_config(""))
    for _ in range(2):
        big.synthesize(f)                         # past the silent frames of a fresh batch
    full_ms = kernel_ms(big, f, a.steps)
    for L in [int(v) for v in a.live.split(",")]:
        live = np.sort(np.random.default_rng(L).choice(N, L, replace=False))
        small = lpcnet_b200.Batch(L, blob, device=0, config=H.model_config(""))
        rows = np.arange(L)
        small.copy_streams(rows, big, live)       # warm-up: grows both staging buffers
        copy_ms = []
        for _ in range(a.copies):
            t0 = time.perf_counter()
            small.copy_streams(rows, big, live)
            copy_ms.append((time.perf_counter() - t0) * 1e3)
        compact_ms = kernel_ms(small, f[live], a.steps)
        small.close()
        print(json.dumps(dict(live=L, rows_before=N, step_frames=FRAMES, kernel_ms_before=round(full_ms, 3),
                              copy_ms_median=round(float(np.median(copy_ms)), 3), copy_ms_min=round(min(copy_ms), 3),
                              kernel_ms_after=round(compact_ms, 3))), flush=True)
    big.close()
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
