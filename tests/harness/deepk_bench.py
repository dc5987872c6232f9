#!/usr/bin/env python3
"""Search throughput and exactness of deep searches (28 < k <= 64) beside the k <= 28 searches they extend.

For each shape (rows x dim, batch B) the corpus is generated once with bench.py's recipe (as tests/harness/
similarity_bench.py does: HostData + upload, mirrored to the host for the oracle) and searched with k in {10, 28, 29, 64}
under cosine and euclidean, plus one filtered cosine case at k = 64 whose filter admits 1 % of the rows.  Each case runs
W untimed batches, then K timed batches between CUDA events.  One JSON line per case:

    qps, ms_per_batch, scan_ms and total_ms_engine (means of the engine's CUDA events over the timed batches: the scan
    kernels, and the whole search including the merge and the fallback), merge_fix_ms = total - scan, recall and
    strict_order against the float64 definition for a sample of the batch's queries, last_fix_entries from a separate
    untimed search with count_fix = 1, and the GPU's name and power limit.

    python tests/harness/deepk_bench.py                       # 10M x 1536 (B 1024) and 1M x 1536 (B 256)
    python tests/harness/deepk_bench.py --shapes 1000000x1536x256 --steps 20 --warmup 3
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402
from harness.similarity_bench import exact_topk, gpu_identity  # noqa: E402
from harness.similarity_oracle import topk_f64  # noqa: E402

KS = (10, 28, 29, 64)
SIMS = ("cosine", "euclidean")
FILTER_K, FILTER_P = 64, 0.01


def log(msg):
    print(f"[deepk_bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def timed(ix, qd, k, a, filters=None):
    import torch
    for _ in range(a.warmup):
        ix.search(qd, k, filters=filters)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(a.steps):
        ix.search(qd, k, filters=filters)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / a.steps
    scan_ms, total_ms, _ = ix.timing_mean(min(a.steps, 16))
    ix.set_option("count_fix", 1)
    s, i = ix.search(qd, k, filters=filters)                    # untimed: exactness and fallback work
    torch.cuda.synchronize()
    fix = ix.info("last_fix_entries")
    ix.set_option("count_fix", 0)
    return ms, scan_ms, total_ms, fix, i.cpu().numpy()


def emit(n, dim, B, k, sim, filt, ms, scan_ms, total_ms, fix, got, want, a, name, power, sample):
    k_ok = want.shape[1]
    recall = float(np.mean([len(np.intersect1d(got[r], want[r][want[r] >= 0])) / max(1, (want[r] >= 0).sum())
                            for r in range(sample)]))
    print(json.dumps({
        "workload": f"{n}x{dim}_b{B}_k{k}", "similarity": sim, "filter": filt, "deep": k > 28,
        "qps": round(B / (ms * 1e-3), 1), "ms_per_batch": round(ms, 3), "scan_ms": round(scan_ms, 3),
        "total_ms_engine": round(total_ms, 3), "merge_fix_ms": round(total_ms - scan_ms, 3), "recall": recall,
        "strict_order": float((got[:, :k_ok] == want).all(axis=1).mean()), "recall_queries": sample,
        "last_fix_entries": int(fix), "steps": a.steps, "warmup": a.warmup, "data": a.data,
        "gpu": name, "power_limit_w": power}), flush=True)


def run_shape(host, n, dim, B, a, name, power):
    import torch
    from oracle import bruteforce as bf
    from qsa_b200.engine import VectorIndex
    sample = min(a.sample, B)
    kmax = max(KS)
    prev = None
    ref = None
    for sim in SIMS:
        ix = VectorIndex(dim=dim, capacity=n, max_batch=B, max_k=kmax, similarity=sim)
        log(f"{n}x{dim} b{B}: {sim}")
        if prev is None:
            bench.upload(host, ix, torch, a.seed, dim, 0, n, n, a.data)
            q_bits = bf.synth_queries(a.seed + 1, B, dim, host.view(min(n, bench.CHUNK), dim))
            qd = torch.from_numpy(q_bits.view(np.int16)).view(torch.bfloat16).cuda()
            log("uploaded; exact answers for the query sample")
            ref = exact_topk(host, q_bits[:sample], n, dim, kmax)    # top-64: its first k columns are the top-k
        else:
            ix.rows[:n].copy_(prev.rows[:n])
            prev.close()
            del prev
            ix.commit(0, n)
        torch.cuda.synchronize()
        for k in KS:
            ms, scan_ms, total_ms, fix, got = timed(ix, qd, k, a)
            emit(n, dim, B, k, sim, None, ms, scan_ms, total_ms, fix, got[:sample].astype(np.int64), ref[sim][:, :k], a,
                 name, power, sample)
        if sim == "cosine":
            g = np.random.default_rng(a.seed + 7)
            tags = (g.random(n) < FILTER_P).astype(np.uint64)
            ix.set_tags(np.arange(n), tags)
            f = np.zeros((B, 4), np.uint64)
            f[:, 0] = 1
            ms, scan_ms, total_ms, fix, got = timed(ix, qd, FILTER_K, a, filters=f)
            rows = np.flatnonzero(tags)
            _, wi = topk_f64(q_bits[:sample], np.ascontiguousarray(host.view(n, dim)[rows]), FILTER_K, sim)
            want = np.where(wi >= 0, rows[np.maximum(wi, 0)], -1)
            emit(n, dim, B, FILTER_K, sim, f"1 tag bit on {FILTER_P:.0%} of rows", ms, scan_ms, total_ms, fix,
                 got[:sample].astype(np.int64), want, a, name, power, sample)
        prev = ix
    prev.close()


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="10000000x1536x1024,1000000x1536x256", help="ROWSxDIMxBATCH,...")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=16, help="queries of the batch checked against the exact definition")
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--data", default="philox", choices=["philox", "numpy"], help="as bench.py's data modes")
    ap.add_argument("--workers", type=int, default=0)
    a = ap.parse_args(argv)
    shapes = [tuple(int(x) for x in s.split("x")) for s in a.shapes.split(",") if s]
    need = max(n * d * 2 for n, d, _ in shapes)
    host = bench.HostData(need, a.workers or bench.auto_workers(1, need, bench.host_memory_available()))
    try:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("deepk_bench needs a CUDA device (H100); there is no CPU fallback")
        name, power = gpu_identity()
        for n, d, B in shapes:
            run_shape(host, n, d, B, a, name, power)
    finally:
        host.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
