"""Regenerates tests/golden/cosine_topk_independent_*.npz WITHOUT importing oracle/: an independent statement of the same
published semantics (cosine similarity, k best, descending; index definition assets/pre-setup/MongoDB-Setup.md:72-83,
operator terraform/lab2-vector-search/main.tf:292), built from other people's code only:

  * data        numpy Philox generator (not the oracle's PCG64 recipe), plus duplicates / a zero row / a scaled copy /
                a one-ulp crowd in consecutive rows
  * bf16        torch's float32 -> bfloat16 conversion (round-to-nearest-even) and back, not the oracle's bit arithmetic
  * cosine      scipy.spatial.distance.cdist(..., metric="cosine") in float64, cross-checked against
                sklearn.metrics.pairwise.cosine_similarity
  * selection   numpy lexsort by (score descending, row ascending); all-zero rows excluded

The oracle (tests/test_golden.py::test_oracle_reproduces_golden) and the CUDA path (test_engine_reproduces_golden) are
both held to these files.  Run from the repo root:  python tests/golden/make_independent_golden.py
"""
import os

import numpy as np
import torch
from scipy.spatial.distance import cdist
from sklearn.metrics.pairwise import cosine_similarity

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = {
    # name: (n, dim, nq, k, seed)
    "d256_n2000_q40_k10": (2000, 256, 40, 10, 7001),       # sizes keep every file under 1 MB
    "d1536_n360_q12_k5": (360, 1536, 12, 5, 7002),
}


def to_bf16_bits(x):
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16)
    return t.view(torch.int16).numpy().view(np.uint16).copy()


def from_bf16_bits(b):
    return torch.from_numpy(b.view(np.int16)).view(torch.bfloat16).to(torch.float64).numpy()


def build(name):
    n, dim, nq, k, seed = CASES[name]
    g = np.random.Generator(np.random.Philox(seed))
    cf = g.standard_normal((n, dim)) * np.exp(g.uniform(-1.0, 1.0, (n, 1)))
    c = to_bf16_bits(cf)
    c[n // 2] = c[5]                                   # exact duplicate: the lower row must come first
    c[n // 3] = 0                                      # an all-zero row is never returned
    c[n - 1] = to_bf16_bits(from_bf16_bits(c[17:18]) * 4)[0]      # scaled copy: same cosine as row 17
    for j in range(20):                                # a crowd of one-ulp variants of row 40 in consecutive rows
        row = c[40].copy()
        row[3 + 7 * j] = np.uint16(int(row[3 + 7 * j]) ^ 1)
        c[100 + j] = row
    qf = g.standard_normal((nq, dim))
    q = to_bf16_bits(qf)
    q[0] = c[5]
    q[1] = c[17]
    q[2] = to_bf16_bits(from_bf16_bits(c[40:41]) + 0.05 * g.standard_normal((1, dim)))[0]   # next to the crowd
    C, Q = from_bf16_bits(c), from_bf16_bits(q)
    live = np.flatnonzero(np.abs(C).sum(axis=1) > 0)
    sim = 1.0 - cdist(Q, C[live], metric="cosine")     # scipy, float64
    sim2 = cosine_similarity(Q, C[live])               # scikit-learn, float64
    assert np.abs(sim - sim2).max() < 1e-12
    index = np.empty((nq, k), np.int64)
    score = np.empty((nq, k), np.float64)
    for r in range(nq):
        order = np.lexsort((live, -sim[r]))[:k]
        index[r], score[r] = live[order], sim[r][order]
        gaps = np.abs(np.diff(np.sort(sim[r])[::-1][:k + 8]))
        # the expected ORDER is only meaningful where the cosines are distinguishable in float64 or exactly tied
        assert ((gaps > 1e-12) | (gaps == 0)).all(), (name, r, gaps.min())
    return dict(corpus=c, queries=q, k=np.int64(k), score=score, index=index)


if __name__ == "__main__":
    for name in CASES:
        np.savez_compressed(os.path.join(HERE, f"cosine_topk_independent_{name}.npz"), **build(name))
        print("wrote", name)
