#!/usr/bin/env python3
"""Search throughput and exactness under each similarity of the index (cosine, dotProduct, euclidean).

For each shape (rows x dim, batch B, top-k) the corpus is generated once with bench.py's recipe (HostData + upload: the
canonical numpy chunk 0, the rest from the device generator, mirrored to the host for the oracle) and searched under
all three similarities with the same warmup / steps discipline as bench.py: W untimed batches, then K timed batches
between CUDA events.  One JSON line per (shape, similarity):

    qps, ms_per_batch, scan_ms (mean of the scan kernels per batch), recall and strict_order against the float64
    definition (tests/harness/similarity_oracle semantics, over ALL rows: fp32 prefilter + float64 rescoring, see
    exact_topk) for a sample of the batch's queries,
    last_fix_entries from a separate untimed search with count_fix = 1, and the GPU's name and power limit.

    python tests/harness/similarity_bench.py                                 # 1M x 1536 (B 256) and 10M x 1536 (B 1024), k 10
    python tests/harness/similarity_bench.py --shapes 1000000x1536x256 --steps 20 --warmup 3
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402
from harness.similarity_oracle import SIMILARITIES, RunningTopk, internal_scores  # noqa: E402

PIECE = 65_536


def _w_prefilter(task):
    """fp32 prefilter of one piece of the shared corpus: per similarity, the piece's `keep` best rows per query."""
    from oracle import bruteforce as bf
    q_bits, first, off, rows, dim, keep = task
    q = bf.bf16_bits_to_f32(q_bits)
    c = bf.bf16_bits_to_f32(bench._shared_view(off, rows, dim))
    dots = (q @ c.T).astype(np.float64)
    qq = (q.astype(np.float64) ** 2).sum(axis=1)
    cc = np.einsum("ij,ij->i", c, c, dtype=np.float64)
    out = {}
    for sim in SIMILARITIES:
        s = internal_scores(sim, dots, qq, cc)
        kk = min(keep, s.shape[1])
        part = np.argpartition(s, s.shape[1] - kk, axis=1)[:, s.shape[1] - kk:]
        out[sim] = part.astype(np.int64) + first
    return out


def exact_topk(host, q_bits, n_rows, dim, k, margin=64):
    """{similarity: row int64 [nq, k]} over all n_rows rows of the host copy: an fp32 prefilter keeps k + margin rows
    per query and piece (spread over the pool), then those candidates are re-scored in float64 (the definition) and
    selected by (value desc, row asc).  Equal to the definition unless more than `margin` rows of one piece sit within
    fp32 rounding (~1e-6 relative) of a query's k-th value."""
    from oracle import bruteforce as bf
    tasks = [(q_bits, lo, lo * dim * 2, min(PIECE, n_rows - lo), dim, k + margin) for lo in range(0, n_rows, PIECE)]
    cand = {sim: [] for sim in SIMILARITIES}
    for part in host.pool.imap_unordered(_w_prefilter, tasks, chunksize=1):
        for sim, rows in part.items():
            cand[sim].append(rows)
    shard = host.view(n_rows, dim)
    q = bf.bf16_bits_to_f32(q_bits).astype(np.float64)
    out = {}
    for sim in SIMILARITIES:
        rows_all = np.concatenate(cand[sim], axis=1)
        res = np.full((len(q), k), -1, dtype=np.int64)
        for r in range(len(q)):
            rows = np.unique(rows_all[r])
            c = bf.bf16_bits_to_f32(shard[rows]).astype(np.float64)
            acc = RunningTopk(1, k)
            s = internal_scores(sim, (c @ q[r])[None, :], np.array([q[r] @ q[r]]), (c * c).sum(axis=1))
            acc.add(s, 0)
            res[r] = np.where(acc.i[0] >= 0, rows[np.maximum(acc.i[0], 0)], -1)
        out[sim] = res
    return out


def log(msg):
    print(f"[similarity_bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def gpu_identity():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def run_shape(host, n, dim, B, k, a, name, power):
    import torch
    from oracle import bruteforce as bf
    from qsa_b200.engine import VectorIndex
    sample = min(a.sample, B)
    oracle_s = None
    prev = None
    for sim in SIMILARITIES:
        ix = VectorIndex(dim=dim, capacity=n, max_batch=B, max_k=k, similarity=sim)
        log(f"{n}x{dim} b{B}: {sim}")
        if prev is None:
            bench.upload(host, ix, torch, a.seed, dim, 0, n, n, a.data)
            # bench.py's query recipe: odd queries are planted near rows of the corpus' first chunk (now in the host copy)
            q_bits = bf.synth_queries(a.seed + 1, B, dim, host.view(min(n, bench.CHUNK), dim))
            qd = torch.from_numpy(q_bits.view(np.int16)).view(torch.bfloat16).cuda()
            log("uploaded; exact answers for the query sample")
            t0 = time.perf_counter()
            ref = exact_topk(host, q_bits[:sample], n, dim, k)
            oracle_s = time.perf_counter() - t0
            log(f"oracle {oracle_s:.0f} s")
        else:
            ix.rows[:n].copy_(prev.rows[:n])                   # the same bits, device to device
            prev.close()
            del prev
            ix.commit(0, n)
        torch.cuda.synchronize()
        for _ in range(a.warmup):
            ix.search(qd, k)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(a.steps):
            ix.search(qd, k)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / a.steps
        scan_ms, total_ms, used = ix.timing_mean(min(a.steps, 16))
        ix.set_option("count_fix", 1)
        s, i = ix.search(qd, k)                                # untimed: exactness and fallback work
        torch.cuda.synchronize()
        fix = ix.info("last_fix_entries")
        ix.set_option("count_fix", 0)
        got = i.cpu().numpy()[:sample].astype(np.int64)
        want = ref[sim]
        recall = float(np.mean([len(np.intersect1d(got[r], want[r])) / k for r in range(sample)]))
        print(json.dumps({
            "workload": f"{n}x{dim}_b{B}_k{k}", "similarity": sim, "qps": round(B / (ms * 1e-3), 1),
            "ms_per_batch": round(ms, 3), "scan_ms": round(scan_ms, 3), "total_ms_engine": round(total_ms, 3),
            "recall": recall, "strict_order": float((got == want).all(axis=1).mean()), "recall_queries": sample,
            "last_fix_entries": int(fix), "steps": a.steps, "warmup": a.warmup, "data": a.data,
            "gpu": name, "power_limit_w": power, "oracle_s": round(oracle_s, 1)}), flush=True)
        prev = ix
    prev.close()


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="1000000x1536x256,10000000x1536x1024", help="ROWSxDIMxBATCH,...")
    ap.add_argument("--k", type=int, default=10)
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
            raise SystemExit("similarity_bench needs a CUDA device (H100); there is no CPU fallback")
        name, power = gpu_identity()
        for n, d, B in shapes:
            run_shape(host, n, d, B, a.k, a, name, power)
    finally:
        host.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
