#!/usr/bin/env python
"""Where does the scan spend its time?  Runs the profiling build of the scan kernel (option "profile": per-CTA cycle
counters for each warp role) and the production build (CUDA-event time) on the BASELINE shapes and prints, per shape,

    prod   : scan ms (mean of --iters back-to-back searches after a preheat), achieved GB/s and TFLOP/s
    roles  : cycles per tile -- TMA producer blocked on a free smem slot, MMA issuer blocked on data / on the epilogue,
             epilogue blocked on the MMA / busy, share of 32-column chunks that took the insertion path.  The MMAs of
             both halves of a tile retire together, so "blocked on the MMA" is one wait per tile; staging and epilogue
             are summed over the tile's two halves.

A role that is never blocked is the bottleneck.  Usage (GPU box):  python tools/gpu_prof.py [--shapes cfg5,b128,...]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from qsa_b200.engine import VectorIndex  # noqa: E402

SHAPES = {
    "cfg5": (6_250_000, 768, 128, 5),      # config 5, one of 8 shards
    "b128": (10_000_000, 1536, 128, 10),   # config 3', HBM-bound capture
    "b1024": (10_000_000, 1536, 1024, 10), # config 3, headline
    "cfg2": (1_000_000, 1536, 256, 10),    # config 2
    "cfg4": (1_250_000, 1536, 4096, 10),   # config 4, one of 8 shards
    "n8shard": (1_250_000, 1536, 1024, 10),  # the headline batch on one of 8 shards
    "b256": (10_000_000, 1536, 256, 10),
    "b512": (10_000_000, 1536, 512, 10),
}


def fill(ix, n, dim, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    step = 1 << 18
    for lo in range(0, n, step):
        m = min(step, n - lo)
        x = torch.randn((m, dim), generator=g, device="cuda", dtype=torch.float32)
        x *= torch.exp(torch.empty((m, 1), device="cuda").uniform_(-0.7, 0.7, generator=g))
        ix.rows[lo:lo + m].copy_(x)
    ix.commit(0, n)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="cfg5,b128,b1024,cfg2")
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--preheat", type=float, default=1.0)
    ap.add_argument("--opts", default="", help="engine options, e.g. share_thresholds=0,pace_gain=0")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    res = []
    cache = {}
    for name in a.shapes.split(","):
        n, dim, B, k = SHAPES[name]
        key = (n, dim)
        if key not in cache:
            cache.clear()
            torch.cuda.empty_cache()
            ix = VectorIndex(dim=dim, capacity=n, max_batch=4096, max_k=10)
            fill(ix, n, dim, 1234)
            cache[key] = ix
        ix = cache[key]
        for kv in filter(None, a.opts.split(",")):
            o, v = kv.split("=")
            ix.set_option(o, int(v))
        g = torch.Generator(device="cuda").manual_seed(4321)
        q = torch.randn((B, dim), generator=g, device="cuda").to(torch.bfloat16)
        t0 = time.perf_counter()
        while time.perf_counter() - t0 < a.preheat:
            for _ in range(4):
                ix.search(q, k)
            torch.cuda.synchronize()
        for _ in range(a.iters):
            ix.search(q, k)
        torch.cuda.synchronize()
        scan_ms, total_ms, m = ix.timing_mean(min(a.iters, 16))
        t = ix.last_timing()
        gbs = (n * dim * 2 + n * 4) * t.launches / (scan_ms * 1e-3) / 1e9
        tfs = t.flops / (scan_ms * 1e-3) / 1e12
        ix.set_option("profile", 1)
        for _ in range(3):
            ix.search(q, k)
        torch.cuda.synchronize()
        p = ix.scan_profile()
        ix.set_option("profile", 0)
        tiles = np.maximum(p["tiles"], 1)
        lead = p["tiles"] > 0

        issuer = lead & ((p["mma_wait_full"] + p["mma_wait_tempty"]) > 0)   # with CTA pairs only the leader issues MMAs

        def per_tile(x, mask=None):
            mask = lead if mask is None else mask
            return float((x[mask] / tiles[mask]).mean()) if mask.any() else 0.0
        row = {
            "shape": name, "rows": n, "dim": dim, "batch": B, "k": k, "grid": ix.info("last_grid"), "launches": t.launches,
            "scan_ms": scan_ms, "total_ms": total_ms, "tail_ms": total_ms - scan_ms, "gbs": gbs, "tflops": tfs,
            "cycles_per_tile": per_tile(p["total"]),
            "cta_cycles_min_max": [int(p["total"][lead].min()), int(p["total"][lead].max())] if lead.any() else None,
            "prod_wait_empty": per_tile(p["prod_wait_empty"]),
            "mma_wait_full": per_tile(p["mma_wait_full"], issuer), "mma_wait_tempty": per_tile(p["mma_wait_tempty"], issuer),
            "epi_wait_tfull": per_tile(p["epi_wait_tfull"]), "epi_busy": per_tile(p["epi_busy"]),
            "epi_slow_chunk_share": float(p["epi_slow_chunks"][lead].sum() / (8.0 * p["tiles"][lead].sum())) if lead.any() else 0.0,
        }
        res.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
