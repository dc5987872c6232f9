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

import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from harness.similarity_bench import exact_topk, indexes, log, main, report, timed_case  # noqa: E402

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


def run_shape(host, n, dim, B, a, gpu):
    import torch
    sample = min(a.sample, B)
    sims = [s for s in a.similarities.split(",") if s]
    tags = make_tags(a.seed + 7, n)
    filters = {c: case_filters(c, B) for c in CASES}
    ref = None
    for sim, ix, q_bits, qd in indexes(host, n, dim, B, a.k, sims, a):
        if ref is None:
            log("uploaded; exact answers for the query sample")
            t0 = time.perf_counter()
            ref = exact_topk(host, q_bits[:sample], n, dim, a.k, sims,
                             (tags, {c: (None if f is None else f[:sample]) for c, f in filters.items()}))
            log(f"oracle {time.perf_counter() - t0:.0f} s")
        ix.tags[:n].copy_(torch.from_numpy(tags.view(np.int64)))
        for case in CASES:
            timing, fix, got = timed_case(ix, qd, a.k, a, filters[case])
            report({"workload": f"{n}x{dim}_b{B}_k{a.k}", "similarity": sim, "case": case}, timing, fix, got,
                   ref[(sim, case)], a, gpu)


def add_args(ap):
    ap.add_argument("--similarities", default="cosine", help="comma-separated: cosine,dotProduct,euclidean")
    ap.add_argument("--k", type=int, default=10)


if __name__ == "__main__":
    sys.exit(main(doc=__doc__, run_shape=run_shape, add_args=add_args))
