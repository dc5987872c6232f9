#!/usr/bin/env python3
"""Throughput and exactness of the pre-filtered search at several filter selectivities.

Same data recipe and step discipline as similarity_bench.py (bench.py's HostData + upload; W untimed batches, then K
timed batches between CUDA events).  Each row gets a random tag: bit 0 with probability 10 %, bit 1 with 1 %, bit 2 with
0.1 % (seeded).  Cases, one JSON line each:

    unfiltered   sa_search, for reference
    all          a match-all filter through the filtered kernel (100 % of the rows eligible)
    10pct, 1pct, 0.1pct   all_of = bit 0, 1, 2
    mixed        per-query filters cycling through all_of / none_of / any_of forms of the above

Each line: qps, ms_per_batch, scan_ms (mean of the scan kernels per batch), last_fix_entries (separate untimed search
with count_fix = 1), recall and strict_order against the filtered float64 definition for a sample of the batch's
queries (fp32 prefilter over the eligible rows, float64 rescoring, as similarity_bench.exact_topk), the GPU's name and
power limit.

    python tests/harness/filter_bench.py                                   # 1M x 1536 (B 256) and 10M x 1536 (B 1024), k 10
    python tests/harness/filter_bench.py --shapes 1000000x1536x256 --similarities cosine,euclidean
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
from harness.filter_oracle import eligibility  # noqa: E402
from harness.similarity_bench import PIECE, gpu_identity  # noqa: E402
from harness.similarity_oracle import RunningTopk, internal_scores  # noqa: E402

U64 = np.uint64
B0, B1, B2 = U64(1), U64(2), U64(4)


def make_tags(seed: int, n: int) -> np.ndarray:
    u = np.random.default_rng(seed).random(n)
    return (u < 0.1).astype(U64) * B0 | (u < 0.01).astype(U64) * B1 | (u < 0.001).astype(U64) * B2


def case_filters(name: str, B: int):
    """uint64 [B, 4] filters of a case (None: the unfiltered search)."""
    f = np.zeros((B, 4), U64)
    if name == "unfiltered":
        return None
    if name == "10pct":
        f[:, 0] = B0
    elif name == "1pct":
        f[:, 0] = B1
    elif name == "0.1pct":
        f[:, 0] = B2
    elif name == "mixed":
        forms = [(0, B0), (0, B1), (1, B0), (2, B1 | B2), (0, 0)]
        for i in range(B):
            col, word = forms[i % len(forms)]
            f[i, col] = word
    return f


CASES = ("unfiltered", "all", "10pct", "1pct", "0.1pct", "mixed")


def _w_prefilter(task):
    """fp32 prefilter of one piece for every (similarity, case): the piece's `keep` best eligible rows per query."""
    from oracle import bruteforce as bf
    q_bits, first, off, rows, dim, keep, sims, tags, filters = task
    q = bf.bf16_bits_to_f32(q_bits)
    c = bf.bf16_bits_to_f32(bench._shared_view(off, rows, dim))
    dots = (q @ c.T).astype(np.float64)
    qq = (q.astype(np.float64) ** 2).sum(axis=1)
    cc = np.einsum("ij,ij->i", c, c, dtype=np.float64)
    out = {}
    for sim in sims:
        s0 = internal_scores(sim, dots, qq, cc)
        for case, f in filters.items():
            s = s0.copy()
            if f is not None:
                s[~eligibility(tags, f)] = -np.inf
            kk = min(keep, s.shape[1])
            part = np.argpartition(s, s.shape[1] - kk, axis=1)[:, s.shape[1] - kk:]
            out[(sim, case)] = (part.astype(np.int64) + first, np.take_along_axis(s, part, axis=1))
    return out


def exact_topk(host, q_bits, n_rows, dim, k, sims, tags, filters, margin=64):
    """{(similarity, case): row int64 [nq, k]} of the filtered definition over all rows (-1 = empty slot)."""
    from oracle import bruteforce as bf
    tasks = [(q_bits, lo, lo * dim * 2, min(PIECE, n_rows - lo), dim, k + margin, sims, tags[lo:lo + PIECE], filters)
             for lo in range(0, n_rows, PIECE)]
    cand = {}
    for part in host.pool.imap_unordered(_w_prefilter, tasks, chunksize=1):
        for key, (rows, vals) in part.items():
            cand.setdefault(key, []).append(np.where(np.isfinite(vals), rows, -1))
    shard = host.view(n_rows, dim)
    q = bf.bf16_bits_to_f32(q_bits).astype(np.float64)
    out = {}
    for key, parts in cand.items():
        sim = key[0]
        rows_all = np.concatenate(parts, axis=1)
        res = np.full((len(q), k), -1, dtype=np.int64)
        for r in range(len(q)):
            rows = np.unique(rows_all[r][rows_all[r] >= 0])
            if len(rows) == 0:
                continue
            c = bf.bf16_bits_to_f32(shard[rows]).astype(np.float64)
            acc = RunningTopk(1, k)
            s = internal_scores(sim, (c @ q[r])[None, :], np.array([q[r] @ q[r]]), (c * c).sum(axis=1))
            acc.add(s, 0)
            res[r] = np.where(acc.i[0] >= 0, rows[np.maximum(acc.i[0], 0)], -1)
        out[key] = res
    return out


def log(msg):
    print(f"[filter_bench {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def run_shape(host, n, dim, B, k, a, sims, name, power):
    import torch
    from oracle import bruteforce as bf
    from qsa_b200.engine import VectorIndex
    sample = min(a.sample, B)
    tags = make_tags(a.seed + 7, n)
    filters = {c: case_filters(c, B) for c in CASES}
    prev, ref = None, None
    for sim in sims:
        ix = VectorIndex(dim=dim, capacity=n, max_batch=B, max_k=k, similarity=sim)
        log(f"{n}x{dim} b{B}: {sim}")
        if prev is None:
            bench.upload(host, ix, torch, a.seed, dim, 0, n, n, a.data)
            q_bits = bf.synth_queries(a.seed + 1, B, dim, host.view(min(n, bench.CHUNK), dim))
            qd = torch.from_numpy(q_bits.view(np.int16)).view(torch.bfloat16).cuda()
            log("uploaded; exact answers for the query sample")
            t0 = time.perf_counter()
            ref = exact_topk(host, q_bits[:sample], n, dim, k, sims, tags,
                             {c: (None if f is None else f[:sample]) for c, f in filters.items()})
            log(f"oracle {time.perf_counter() - t0:.0f} s")
        else:
            ix.rows[:n].copy_(prev.rows[:n])
            prev.close()
            del prev
            ix.commit(0, n)
        ix.tags[:n].copy_(torch.from_numpy(tags.view(np.int64)))
        torch.cuda.synchronize()
        for case in CASES:
            f = filters[case]
            fd = None if f is None else torch.from_numpy(f.view(np.int64)).cuda()

            def run():
                if fd is None:
                    return ix.search(qd, k)
                return _filtered(ix, qd, fd, k)
            for _ in range(a.warmup):
                run()
            torch.cuda.synchronize()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(a.steps):
                run()
            ev1.record()
            torch.cuda.synchronize()
            ms = ev0.elapsed_time(ev1) / a.steps
            scan_ms, total_ms, _ = ix.timing_mean(min(a.steps, 16))
            ix.set_option("count_fix", 1)
            s, i = run()
            torch.cuda.synchronize()
            fix = ix.info("last_fix_entries")
            ix.set_option("count_fix", 0)
            got = i.cpu().numpy()[:sample].astype(np.int64)
            want = ref[(sim, case)]
            recall = float(np.mean([
                len(np.intersect1d(got[r][got[r] >= 0], want[r][want[r] >= 0])) / max(1, int((want[r] >= 0).sum()))
                for r in range(sample)]))
            print(json.dumps({
                "workload": f"{n}x{dim}_b{B}_k{k}", "similarity": sim, "case": case, "qps": round(B / (ms * 1e-3), 1),
                "ms_per_batch": round(ms, 3), "scan_ms": round(scan_ms, 3), "total_ms_engine": round(total_ms, 3),
                "recall": recall, "strict_order": float((got == want).all(axis=1).mean()), "recall_queries": sample,
                "last_fix_entries": int(fix), "steps": a.steps, "warmup": a.warmup, "data": a.data,
                "gpu": name, "power_limit_w": power}), flush=True)
        prev = ix
    prev.close()


def _filtered(ix, qd, fd, k):
    """sa_search_filtered with a device filter tensor already in place (no per-step upload)."""
    import torch
    from qsa_b200 import capi
    nq = qd.shape[0]
    score = torch.empty((nq, k), dtype=torch.float32, device=qd.device)
    idx = torch.empty((nq, k), dtype=torch.int32, device=qd.device)
    capi.check(ix.lib.sa_search_filtered(ix._h, qd.data_ptr(), fd.data_ptr(), nq, k, score.data_ptr(), idx.data_ptr(),
                                         None, ix._stream()), "sa_search_filtered")
    return score, idx


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="1000000x1536x256,10000000x1536x1024", help="ROWSxDIMxBATCH,...")
    ap.add_argument("--similarities", default="cosine", help="comma-separated: cosine,dotProduct,euclidean")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=16, help="queries of the batch checked against the exact definition")
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--data", default="philox", choices=["philox", "numpy"], help="as bench.py's data modes")
    ap.add_argument("--workers", type=int, default=0)
    a = ap.parse_args(argv)
    shapes = [tuple(int(x) for x in s.split("x")) for s in a.shapes.split(",") if s]
    sims = [s for s in a.similarities.split(",") if s]
    need = max(n * d * 2 for n, d, _ in shapes)
    host = bench.HostData(need, a.workers or bench.auto_workers(1, need, bench.host_memory_available()))
    try:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit("filter_bench needs a CUDA device (H100); there is no CPU fallback")
        name, power = gpu_identity()
        for n, d, B in shapes:
            run_shape(host, n, d, B, a.k, a, sims, name, power)
    finally:
        host.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
