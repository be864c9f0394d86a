"""Compaction of an encoder batch on one GPU: what one second of audio costs a 4096-row encoder batch that carries only L live
sessions, what it costs after those L rows were copied into an L-row batch (lpcnet_b200_enc_copy_streams), and what the copy
itself costs.

A 4096-row encoder batch encodes four warm-up packets of int16 speech-like PCM (oracle/fixtures.make_pcm_batch) on every row.
Timed: one encode_device call of 25 packets (1 s of audio per row) on the 4096-row batch, CUDA events on a caller stream around
the call.  Per L in --live, L rows spread over the batch are the live ones: the wall time of copy_streams into an L-row batch
(a host clock around the call, which returns after a synchronise), and the same encode_device call on the L-row batch.  Each
time is the median of --reps calls.  Prints the card's name and power limit, then one JSON line per L.

    python tools/bench_enc_compact.py [--reps 5] [--live 256,1024,2048]"""
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

N, PACKETS, WARM, POOL = 4096, 25, 4, 97


def pcm_rows(n, nframes):
    """[n][nframes*160] int16: row i is a window of fixture stream i % POOL that starts 37 * (i // POOL) samples in"""
    from fixtures import make_pcm_batch
    shift = 37 * ((n - 1) // POOL)
    base = make_pcm_batch(range(POOL), nframes + shift // 160 + 1)
    i = np.arange(n)
    idx = (i // POOL)[:, None] * 37 + np.arange(nframes * 160)[None, :]
    return np.ascontiguousarray(base[i % POOL][i[:, None], idx])


def encode_ms(e, pcm, reps, torch):
    """median device ms of an encode_device call of PACKETS packets on every row of e"""
    d_pcm = torch.from_numpy(pcm).cuda()
    d_pk = torch.empty((e.n, PACKETS, 8), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    ms = []
    for _ in range(reps + 1):                      # the first call is a warm-up
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        e.encode_device(d_pcm.data_ptr(), PACKETS, d_pk.data_ptr(), cuda_stream=s.cuda_stream)
        b.record(s)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms[1:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--live", default="256,1024,2048")
    a = ap.parse_args()
    import torch
    import lpcnet_b200
    from lpcnet_b200 import build
    from bench_group import card
    import helpers as H
    build.build()
    print(json.dumps(dict(card=card())), flush=True)
    cb = H.codebooks()
    pcm = pcm_rows(N, 4 * (WARM + PACKETS))
    warm, timed = pcm[:, :640 * WARM], np.ascontiguousarray(pcm[:, 640 * WARM:])
    big = lpcnet_b200.EncBatch(N, codebooks=cb)
    big.encode(warm)
    full_ms = encode_ms(big, timed, a.reps, torch)
    for L in [int(v) for v in a.live.split(",")]:
        live = np.sort(np.random.default_rng(L).choice(N, L, replace=False))
        small = lpcnet_b200.EncBatch(L, codebooks=cb)
        rows = np.arange(L)
        small.copy_streams(rows, big, live)        # warm-up: grows the row-list staging
        copy_ms = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            small.copy_streams(rows, big, live)
            copy_ms.append((time.perf_counter() - t0) * 1e3)
        small_ms = encode_ms(small, timed[live], a.reps, torch)
        small.close()
        print(json.dumps(dict(live=L, rows_before=N, packets=PACKETS, encode_ms_before=round(full_ms, 3),
                              copy_ms_median=round(float(np.median(copy_ms)), 3), copy_ms_min=round(min(copy_ms), 3),
                              encode_ms_after=round(small_ms, 3))), flush=True)
    big.close()
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
