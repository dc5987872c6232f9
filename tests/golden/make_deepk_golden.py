"""Independent fixture for the deep search, k = 64 (deepk_topk_independent_*.npz).

Built without the repository's oracle or test harness: bf16 rounding in numpy, dot products from a float64 matmul,
cosines from that matmul over numpy norms (cross-checked against 1 - scipy's cosine cdist), Euclidean distances from
scipy's cdist (cross-checked against sqrt of its sqeuclidean), and the ranking from numpy.lexsort.  The corpus has:
  * one 256-row tile holding a 100-row crowd, one row and 99 one-ulp variants of it; query 0 sits next to it, so its
    whole top-64 lies in the crowd;
  * 40 exact duplicates of another row;
  * an all-zero row, never returned under cosine and a live row under dotProduct and euclidean.

    python tests/golden/make_deepk_golden.py      # rewrites the .npz next to this script
"""
import os

import numpy as np
from scipy.spatial.distance import cdist

HERE = os.path.dirname(os.path.abspath(__file__))


def bf16_round(x: np.ndarray) -> np.ndarray:
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bits_to_f64(b: np.ndarray) -> np.ndarray:
    return (b.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def rank(values: np.ndarray, ok: np.ndarray, k: int, ascending: bool):
    """Per query: the k best rows with ok[row] by (value, row asc); empty slots -1 / worst value."""
    nq, n = values.shape
    idx = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), np.inf if ascending else -np.inf)
    cand = np.arange(n)[ok]
    for i in range(nq):
        v = values[i, cand]
        order = np.lexsort((cand, v if ascending else -v))[:k]
        idx[i, :len(order)] = cand[order]
        sc[i, :len(order)] = v[order]
    return sc, idx


def main():
    g = np.random.default_rng(20261018)
    n, dim, nq, k = 1400, 128, 10, 64
    c_bits = bf16_round(g.standard_normal((n, dim)) * np.exp(g.uniform(-0.5, 0.5, (n, 1))))
    crowd = np.arange(512 + 60, 512 + 160)                      # 100 rows inside tile 2 (rows 512 .. 767):
    base = int(crowd[0])                                        # row 572 and 99 one-ulp variants of it, each in its own
    for j, r in enumerate(crowd[1:]):                           # column
        c_bits[r] = c_bits[base]
        c_bits[r, j] ^= np.uint16(1)
    dups = np.sort(g.choice(np.setdiff1d(np.arange(n), np.r_[crowd, base, 1000]), 40, replace=False))
    c_bits[dups] = c_bits[7]
    c_bits[1000] = 0                                            # the all-zero row
    q = g.standard_normal((nq, dim))
    q[0] = bits_to_f64(c_bits[base]) + 0.002 * q[0]             # next to the crowd
    q[1] = bits_to_f64(c_bits[7]) + 0.05 * q[1]                 # next to the duplicates
    q[2] *= 1e-3                                                # short query: the zero row ranks high under euclidean
    q_bits = bf16_round(q)
    c, qf = bits_to_f64(c_bits), bits_to_f64(q_bits)

    dot = qf @ c.T
    qn, cn = np.sqrt(np.einsum("ij,ij->i", qf, qf)), np.sqrt(np.einsum("ij,ij->i", c, c))
    live_cos = cn > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        cos = dot / (qn[:, None] * cn[None, :])
    ref = 1.0 - cdist(qf, c[live_cos], "cosine")
    assert np.allclose(cos[:, live_cos], ref, rtol=0, atol=1e-12), "matmul cosine and scipy cosine disagree"
    euc = cdist(qf, c, "euclidean")
    assert np.array_equal(euc, np.sqrt(cdist(qf, c, "sqeuclidean"))), "cdist euclidean != sqrt(sqeuclidean)"

    out = dict(corpus_bits=c_bits, query_bits=q_bits, k=np.int64(k), crowd_rows=crowd, dup_rows=dups,
               zero_row=np.int64(1000))
    everything = np.ones(n, bool)
    for name, vals, ok, asc in (("cosine", cos, live_cos, False), ("dot", dot, everything, False),
                                ("euclidean", euc, everything, True)):
        s, i = rank(vals, ok, k, asc)
        out[f"{name}_score"], out[f"{name}_idx"] = s, i
    assert np.isin(out["cosine_idx"][0], crowd).all()
    path = os.path.join(HERE, f"deepk_topk_independent_d{dim}_n{n}_q{nq}_k{k}.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
