#!/usr/bin/env python3
"""Search throughput and exactness of deep searches (28 < k <= 64) beside the k <= 28 searches they extend.

For each shape (rows x dim, batch B) the corpus is generated once with bench.py's recipe (as tests/harness/
similarity_bench.py does: HostData + upload, mirrored to the host for the oracle) and searched with k in {10, 28, 29, 64}
under cosine and euclidean, plus one filtered cosine case at k = 64 whose filter admits 1 % of the rows (staged on the
device once, outside the timed batches).  Each case runs W untimed batches, then K timed batches between CUDA events.
One JSON line per case:

    qps, ms_per_batch, scan_ms and total_ms_engine (means of the engine's CUDA events over the timed batches: the scan
    kernels, and the whole search including the merge and the fallback), merge_fix_ms = total - scan, recall and
    strict_order against the float64 definition for a sample of the batch's queries, last_fix_entries from a separate
    untimed search with count_fix = 1, and the GPU's name and power limit.

    python tests/harness/deepk_bench.py                       # 10M x 1536 (B 1024) and 1M x 1536 (B 256)
    python tests/harness/deepk_bench.py --shapes 1000000x1536x256 --steps 20 --warmup 3
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from harness.similarity_bench import exact_topk, indexes, log, main, report, timed_case  # noqa: E402
from harness.similarity_oracle import topk_f64  # noqa: E402

KS = (10, 28, 29, 64)
SIMS = ("cosine", "euclidean")
FILTER_K, FILTER_P = 64, 0.01


def run_shape(host, n, dim, B, a, gpu):
    sample = min(a.sample, B)
    ref = None
    for sim, ix, q_bits, qd in indexes(host, n, dim, B, max(KS), SIMS, a):
        if ref is None:
            log("uploaded; exact answers for the query sample")
            ref = exact_topk(host, q_bits[:sample], n, dim, max(KS), SIMS)    # top-64: its first k columns are the top-k
        cases = [(k, None, None, ref[sim][:, :k]) for k in KS]
        if sim == "cosine":
            tags = (np.random.default_rng(a.seed + 7).random(n) < FILTER_P).astype(np.uint64)
            ix.set_tags(np.arange(n), tags)
            f = np.zeros((B, 4), np.uint64)
            f[:, 0] = 1
            rows = np.flatnonzero(tags)                                   # float64 brute force over the eligible rows
            _, wi = topk_f64(q_bits[:sample], np.ascontiguousarray(host.view(n, dim)[rows]), FILTER_K, sim)
            want = np.where(wi >= 0, rows[np.maximum(wi, 0)], -1)
            cases.append((FILTER_K, f"1 tag bit on {FILTER_P:.0%} of rows", f, want))
        for k, filt, f, want in cases:
            timing, fix, got = timed_case(ix, qd, k, a, f)
            report({"workload": f"{n}x{dim}_b{B}_k{k}", "similarity": sim, "filter": filt, "deep": k > 28}, timing, fix,
                   got, want, a, gpu, merge_fix_ms=round(timing["total_ms_engine"] - timing["scan_ms"], 3))


if __name__ == "__main__":
    sys.exit(main(doc=__doc__, run_shape=run_shape, shapes="10000000x1536x1024,1000000x1536x256",
                  add_args=lambda ap: None))
