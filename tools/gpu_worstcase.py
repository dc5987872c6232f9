#!/usr/bin/env python
"""Data-dependent worst cases of the scan's epilogue (VERDICT r01 weak #11): the register-list top-k is cheap because,
on exchangeable data, a value beats the running threshold with probability ~ kKL / n.  Two orders break that premise:

  sorted    the corpus sorted by ASCENDING similarity to the batch centroid, with the queries clustered around that
            centroid (paraphrases of one question): every tile brings rows better than everything before it
  clustered embeddings drawn from a mixture of 1000 centres, stored cluster by cluster (documents ingested source by
            source), queries near some of the centres

For each, the production scan kernel is timed against the same rows in random order, with and without the sampled
threshold pre-pass (option "presample"), or with any other engine option swept (--option window_bound --presample 0,1).  Answers are compared with the shuffled run (same set of rows => same scores).

    python tools/gpu_worstcase.py [--rows 4000000] [--batches 128,1024] [--out worstcase.json]
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


def timed(ix, q, k, iters=12):
    for _ in range(3):
        s, i = ix.search(q, k)
    torch.cuda.synchronize()
    for _ in range(iters):
        s, i, s64 = ix.search(q, k, want_score64=True)
    torch.cuda.synchronize()
    scan, total, _ = ix.timing_mean(min(iters, 16))
    return scan, total, s64, i


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--batches", default="128,1024")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--presample", default="0,64", help="values of the engine option to compare")
    ap.add_argument("--option", default="presample", help="the engine option those values are for (e.g. window_bound)")
    ap.add_argument("--noise", type=float, default=0.6, help="spread of the queries around their centroid (0.1 = near-duplicates)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    n, dim, k = a.rows, a.dim, a.k
    dev = torch.device("cuda")
    g = torch.Generator(device="cuda").manual_seed(11)
    ix = VectorIndex(dim=dim, capacity=n, max_batch=1024, max_k=k)
    res = []

    def fill(order_fn, kind):
        """Generate the rows chunk-wise, then lay them out in the order given by order_fn(rows) (a permutation)."""
        step = 1 << 18
        if kind == "iid":
            for lo in range(0, n, step):
                m = min(step, n - lo)
                ix.rows[lo:lo + m].copy_(torch.randn((m, dim), generator=g, device=dev))
        else:
            centres = torch.randn((1000, dim), generator=g, device=dev)
            for lo in range(0, n, step):
                m = min(step, n - lo)
                cid = torch.randint(0, 1000, (m,), generator=g, device=dev)
                ix.rows[lo:lo + m].copy_(centres[cid] + 0.7 * torch.randn((m, dim), generator=g, device=dev))
        perm = order_fn()
        if perm is not None:
            tmp = torch.empty_like(ix.rows)
            for lo in range(0, n, step):
                tmp[lo:lo + step] = ix.rows[perm[lo:lo + step]]
            ix.rows.copy_(tmp)
            del tmp
        ix.lib.sa_corpus_reset(ix._h)
        ix.commit(0, n)
        torch.cuda.synchronize()

    def sim_to(vec):
        out = torch.empty(n, device=dev)
        step = 1 << 20
        v = vec.to(torch.bfloat16)
        for lo in range(0, n, step):
            r = ix.rows[lo:lo + step]
            out[lo:lo + step] = (r @ v).float() / r.float().norm(dim=1)
        return out

    for B in [int(x) for x in a.batches.split(",")]:
        centre = torch.randn(dim, generator=g, device=dev)
        q_near = (centre[None, :] + a.noise * torch.randn((B, dim), generator=g, device=dev)).to(torch.bfloat16)
        cases = []
        # ---- iid rows, queries clustered around `centre`: random order, then ascending similarity to the centroid
        fill(lambda: None, "iid")
        cases.append(("iid rows, clustered queries, random order", q_near, None))
        for name, q, _ in list(cases):
            pass
        base = {}
        for ps in [int(x) for x in a.presample.split(",")]:
            ix.set_option(a.option, ps)
            scan, total, s64, i = timed(ix, q_near, k)
            base[ps] = (scan, total)
            ref_scores = s64.clone()
            res.append({"batch": B, "case": "random order", a.option: ps, "scan_ms": scan, "search_ms": total})
            print(json.dumps(res[-1]), flush=True)
        order = torch.argsort(sim_to(q_near.float().mean(0)))
        tmp = torch.empty_like(ix.rows)
        step = 1 << 18
        for lo in range(0, n, step):
            tmp[lo:lo + step] = ix.rows[order[lo:lo + step]]
        ix.rows.copy_(tmp)
        del tmp
        ix.lib.sa_corpus_reset(ix._h)
        ix.commit(0, n)
        for ps in [int(x) for x in a.presample.split(",")]:
            ix.set_option(a.option, ps)
            scan, total, s64, i = timed(ix, q_near, k)
            same = bool(torch.equal(s64, ref_scores))          # same set of rows => identical sorted cosine lists
            res.append({"batch": B, "case": "ascending similarity to the batch centroid", a.option: ps, "scan_ms": scan,
                        "search_ms": total, "slowdown_vs_random": total / base[ps][1], "same_scores_as_random_order": same})
            print(json.dumps(res[-1]), flush=True)
        # ---- clustered embeddings stored cluster by cluster
        fill(lambda: None, "clustered")
        q_c = (ix.rows[torch.randint(0, n, (B,), generator=g, device=dev)].float() +
               a.noise * torch.randn((B, dim), generator=g, device=dev)).to(torch.bfloat16)
        base = {}
        for ps in [int(x) for x in a.presample.split(",")]:
            ix.set_option(a.option, ps)
            scan, total, s64, i = timed(ix, q_c, k)
            base[ps] = (scan, total)
            ref_scores = s64.clone()
            res.append({"batch": B, "case": "clustered, random order", a.option: ps, "scan_ms": scan, "search_ms": total})
            print(json.dumps(res[-1]), flush=True)
        # cluster by cluster: sort rows by their nearest-centre id (approximated by the sign pattern of a projection)
        key = sim_to(torch.randn(dim, generator=g, device=dev))
        order = torch.argsort(key)
        tmp = torch.empty_like(ix.rows)
        for lo in range(0, n, step):
            tmp[lo:lo + step] = ix.rows[order[lo:lo + step]]
        ix.rows.copy_(tmp)
        del tmp
        ix.lib.sa_corpus_reset(ix._h)
        ix.commit(0, n)
        for ps in [int(x) for x in a.presample.split(",")]:
            ix.set_option(a.option, ps)
            scan, total, s64, i = timed(ix, q_c, k)
            res.append({"batch": B, "case": "clustered, sorted along a random direction", a.option: ps, "scan_ms": scan,
                        "search_ms": total, "slowdown_vs_random": total / base[ps][1],
                        "same_scores_as_random_order": bool(torch.equal(s64, ref_scores))})
            print(json.dumps(res[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
