"""Independent fixture for the pre-filtered search (filter_topk_independent_*.npz).

Built without the repository's oracle or test harness: bf16 rounding in numpy, cosine and Euclidean values from scipy's
cdist, dot products from a float64 matmul, eligibility from explicit Python sets of tag bits per row, and the ranking
from numpy.lexsort.  One query's filter excludes every row of its unfiltered top-k.

    python tests/golden/make_filter_golden.py      # rewrites the .npz next to this script
"""
import os

import numpy as np
from scipy.spatial.distance import cdist

HERE = os.path.dirname(os.path.abspath(__file__))


def bf16_round(x: np.ndarray) -> np.ndarray:
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return r


def bits_to_f64(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def rank(values: np.ndarray, ok: np.ndarray, k: int, ascending: bool):
    """Per query: the k best eligible rows by (value, row asc); empty slots -1 / worst value."""
    nq, n = values.shape
    idx = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), np.inf if ascending else -np.inf)
    rows = np.arange(n)
    for i in range(nq):
        cand = rows[ok[i]]
        v = values[i, cand]
        order = np.lexsort((cand, v if ascending else -v))[:k]
        idx[i, :len(order)] = cand[order]
        sc[i, :len(order)] = v[order]
    return sc, idx


def main():
    g = np.random.default_rng(20261017)
    n, dim, nq, k = 900, 128, 12, 8
    c_bits = bf16_round(g.standard_normal((n, dim)) * np.exp(g.uniform(-1, 1, (n, 1))))
    q_bits = bf16_round(g.standard_normal((nq, dim)))
    c, q = bits_to_f64(c_bits), bits_to_f64(q_bits)
    # tag bits per row as explicit sets: 6 "fields" worth of bits 0..11
    row_bits = [set(int(b) for b in np.flatnonzero(g.random(12) < 0.3)) for _ in range(n)]
    tags = np.array([sum(1 << b for b in s) for s in row_bits], dtype=np.uint64)
    filters = np.zeros((nq, 4), np.uint64)
    rules = []
    for i in range(nq):
        kind = i % 4
        a, b = int(g.integers(12)), int(g.integers(12))
        if kind == 0:
            rules.append(lambda s, a=a: a in s); filters[i, 0] = 1 << a
        elif kind == 1:
            rules.append(lambda s, a=a: a not in s); filters[i, 1] = 1 << a
        elif kind == 2:
            rules.append(lambda s, a=a, b=b: a in s or b in s); filters[i, 2] = (1 << a) | (1 << b)
        else:
            rules.append(lambda s, a=a, b=b: (a in s) and (b not in s or a == b) if a != b else a in s)
            filters[i, 0] = 1 << a
            if a != b:
                filters[i, 1] = 1 << b
    cos = 1.0 - cdist(q, c, "cosine")
    dot = q @ c.T
    euc = cdist(q, c, "euclidean")
    # query 0: exclude every row of its unfiltered cosine top-k by a bit only those rows carry (bit 12)
    top0 = np.lexsort((np.arange(n), -cos[0]))[:k]
    for r in top0:
        row_bits[r].add(12)
        tags[r] |= np.uint64(1 << 12)
    filters[0] = 0
    filters[0, 1] = 1 << 12
    rules[0] = lambda s: 12 not in s
    ok = np.array([[rules[i](row_bits[r]) for r in range(n)] for i in range(nq)])
    out = dict(corpus_bits=c_bits, query_bits=q_bits, tags=tags, filters=filters, k=np.int64(k), eligible=ok,
               excluded_top_query0=top0)
    for name, vals, asc in (("cosine", cos, False), ("dot", dot, False), ("euclidean", euc, True)):
        s, i = rank(vals, ok, k, asc)
        out[f"{name}_score"], out[f"{name}_idx"] = s, i
    path = os.path.join(HERE, f"filter_topk_independent_d{dim}_n{n}_q{nq}_k{k}.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
