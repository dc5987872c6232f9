"""Independent fixtures for the dotProduct and euclidean searches: tests/golden/similarity_topk_independent_*.npz.

Generated WITHOUT importing oracle/ or the package, from independent implementations:
  * data: numpy Philox, rounded to bf16 by torch (``tensor.to(torch.bfloat16)``);
  * dotProduct: numpy float64 matmul, cross-checked against torch float64;
  * euclidean: ``scipy.spatial.distance.cdist(metric="euclidean")`` (sqrt of the sum of squared differences), cross-checked
    against ``cdist(metric="sqeuclidean")`` and torch's ``cdist`` in float64;
  * selection: ``numpy.lexsort`` by (score desc, row asc), distances by (distance asc, row asc).
The corpus holds exact duplicates, all-zero rows (live rows for both similarities), scaled copies (which rank differently
under dotProduct and euclidean than under cosine) and a 20-row crowd of one-ulp variants in consecutive rows.

    python tests/golden/make_similarity_golden.py
"""
from __future__ import annotations

import os

import numpy as np
import torch
from scipy.spatial.distance import cdist

HERE = os.path.dirname(os.path.abspath(__file__))


def bf16_bits(x: np.ndarray) -> np.ndarray:
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).view(torch.int16).numpy() \
        .view(np.uint16)


def bits_f64(b: np.ndarray) -> np.ndarray:
    return torch.from_numpy(b.view(np.int16)).view(torch.bfloat16).to(torch.float64).numpy()


def select(score: np.ndarray, k: int, ascending: bool):
    rows = np.arange(score.shape[1])
    idx = np.stack([np.lexsort((rows, s if ascending else -s))[:k] for s in score])
    return np.take_along_axis(score, idx, axis=1), idx.astype(np.int64)


def make(seed: int, n: int, dim: int, nq: int, k: int) -> str:
    g = np.random.Generator(np.random.Philox(seed))
    c = g.standard_normal((n, dim)).astype(np.float32) * np.exp(g.uniform(-1.5, 1.5, (n, 1))).astype(np.float32)
    c[n // 2] = c[5]; c[n // 2 + 1] = c[5]                        # exact duplicates: ties resolve to the lowest row
    c[7] = 0.0; c[n - 1] = 0.0                                   # all-zero rows: live under both similarities
    c[n // 3] = c[11] * 4.0; c[n // 3 + 1] = c[11] * 0.25         # scaled copies: same cosine, other dot and distance
    cb = bf16_bits(c)
    crowd = 3 * n // 4                                           # 20 one-ulp variants of row 13, consecutive rows
    for j in range(20):
        cb[crowd + j] = cb[13]
        cb[crowd + j, (3 + 7 * j) % dim] ^= np.uint16(1)
    q = g.standard_normal((nq, dim)).astype(np.float32)
    cf = bits_f64(cb)
    q[0] = cf[5]                                                 # on the duplicates
    q[1] = cf[11]                                                # on the scaled family
    q[2] = cf[13] + 0.01 * g.standard_normal(dim)                # next to the crowd
    q[3] = 0.0                                                   # all-zero query
    q[4] = -np.abs(cf).max(axis=0) * np.sign(cf.sum(axis=0) + 1e-9)   # mostly negative dots
    qb = bf16_bits(q)
    qf = bits_f64(qb)

    dots = qf @ cf.T
    dots_t = (torch.from_numpy(qf) @ torch.from_numpy(cf).T).numpy()
    assert np.array_equal(dots, dots_t), "numpy and torch float64 dot products disagree"
    dist = cdist(qf, cf, metric="euclidean")
    sq = cdist(qf, cf, metric="sqeuclidean")
    dist_t = torch.cdist(torch.from_numpy(qf), torch.from_numpy(cf), compute_mode="donot_use_mm_for_euclid_dist").numpy()
    assert np.array_equal(dist, np.sqrt(sq)), "cdist euclidean != sqrt(sqeuclidean)"
    assert np.allclose(dist, dist_t, rtol=1e-12, atol=0), "scipy and torch distances disagree"

    dot_s, dot_i = select(dots, k, ascending=False)
    euc_s, euc_i = select(dist, k, ascending=True)
    name = f"similarity_topk_independent_d{dim}_n{n}_q{nq}_k{k}.npz"
    path = os.path.join(HERE, name)
    np.savez_compressed(path, corpus_bits=cb, query_bits=qb, k=np.int64(k), dot_score=dot_s, dot_idx=dot_i,
                        euclidean_score=euc_s, euclidean_idx=euc_i)
    return path


if __name__ == "__main__":
    for args in ((20261017, 1500, 128, 24, 10), (77, 800, 256, 16, 7)):
        p = make(*args)
        print(p, os.path.getsize(p), "bytes")
