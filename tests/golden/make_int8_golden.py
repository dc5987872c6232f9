"""Independent fixture for int8 indexes (int8_topk_independent_*.npz), k = 64.

Built with numpy and scipy only, without the repository's oracle, harness or package.  Every sum is an exact integer:
  * dot products and squared norms: numpy int64 matmuls;
  * cosine: dot / sqrt(|q|^2 |c|^2) in float64 (the product of the two squared norms is an exact integer below 2^53),
    cross-checked against 1 - scipy's cosine cdist;
  * Euclidean distance: scipy's cdist, which is one correctly rounded sqrt of the exact integer sum of squared
    differences -- checked bit for bit against sqrt of that sum computed in int64;
  * ranking: numpy.lexsort by (value, row asc), distances ascending; all-zero rows are never returned under cosine.
The corpus (dim 1536) has:
  * random int8 rows over the full range, and rows of small values;
  * a row of all -128 and a row of all 127 (their dot is 25 165 824 > 2^24, so fp32 alone could not hold it);
  * an all-zero row;
  * 200 consecutive rows that are permutations of one sparse vector: exact ties under every similarity against the
    all-ones query;
  * 10 exact duplicates of row 3.
Each row carries a 64-bit filter tag and each query one sa_filter (all_of, none_of, any_of[0], any_of[1]); the filtered
answers use the predicate of include/sa_api.h.  One filter admits fewer than k rows.

    python tests/golden/make_int8_golden.py      # rewrites the .npz next to this script
"""
import os

import numpy as np
from scipy.spatial.distance import cdist

HERE = os.path.dirname(os.path.abspath(__file__))
SIMS = ("cosine", "dotProduct", "euclidean")


def rank(values: np.ndarray, ok: np.ndarray, k: int, ascending: bool):
    """Per query: the k best rows r with ok[i, r], by (value, row asc); empty slots -1 / the worst value."""
    nq, n = values.shape
    idx = np.full((nq, k), -1, np.int64)
    sc = np.full((nq, k), np.inf if ascending else -np.inf)
    for i in range(nq):
        cand = np.flatnonzero(ok[i])
        v = values[i, cand]
        order = np.lexsort((cand, v if ascending else -v))[:k]
        idx[i, :len(order)] = cand[order]
        sc[i, :len(order)] = v[order]
    return sc, idx


def passes(tags: np.ndarray, filters: np.ndarray) -> np.ndarray:
    """bool [nq, n]: (t & all_of) == all_of, (t & none_of) == 0, each nonzero any_of word meets t."""
    t = tags[None, :]
    f = filters
    ok = ((t & f[:, 0:1]) == f[:, 0:1]) & ((t & f[:, 1:2]) == 0)
    for j in (2, 3):
        ok &= (f[:, j:j + 1] == 0) | ((t & f[:, j:j + 1]) != 0)
    return ok


def make(seed: int = 20261018, dim: int = 1536, k: int = 64) -> str:
    g = np.random.Generator(np.random.Philox(seed))
    parts = [
        g.integers(-128, 128, (40, dim)),                        # 0 .. 39: full range
        g.integers(-6, 7, (64, dim)),                            # 40 .. 103: small values
        np.full((1, dim), -128), np.full((1, dim), 127),         # 104, 105: the extremes
        np.zeros((1, dim)),                                      # 106: all zero
    ]
    v = np.zeros(dim, np.int64)
    nz = g.choice(dim, 48, replace=False)
    v[nz] = g.integers(-127, 128, 48)
    parts.append(np.stack([g.permutation(v) for _ in range(200)]))   # 107 .. 306: permutations of v
    c = np.concatenate(parts).astype(np.int8)
    c = np.concatenate([c, np.repeat(c[3:4], 10, axis=0)])          # 307 .. 316: duplicates of row 3
    n = c.shape[0]

    q = np.stack([
        np.ones(dim), np.zeros(dim), np.full(dim, -128), np.full(dim, 127),
        g.integers(-128, 128, dim), g.integers(-128, 128, dim), g.integers(-3, 4, dim),
        c[3], v, -c[105].astype(np.int64),
    ]).astype(np.int8)
    nq = q.shape[0]

    tags = g.integers(0, 1 << 8, n).astype(np.uint64) | (np.uint64(1) << np.uint64(40))
    tags[g.choice(n, 20, replace=False)] |= np.uint64(1) << np.uint64(50)   # a rare bit: 20 rows carry it
    filters = np.zeros((nq, 4), np.uint64)
    filters[1] = [1, 0, 0, 0]                                    # bit 0 set
    filters[2] = [0, 2, 0, 0]                                    # bit 1 clear
    filters[3] = [0, 0, 12, 0]                                   # bit 2 or 3
    filters[4] = [1 << 50, 0, 0, 0]                              # the rare bit: 20 rows, fewer than k
    filters[5] = [1 << 40, 1, 48, 0x81]
    filters[7] = [0, 0, 1 << 62, 0]                              # no row passes
    filters[8] = [0, 4, 0, 0]

    qi, ci = q.astype(np.int64), c.astype(np.int64)
    dots = qi @ ci.T
    qq, cc = (qi * qi).sum(axis=1), (ci * ci).sum(axis=1)
    assert np.abs(dots).max() < 2 ** 31 and np.abs(dots).max() > 2 ** 24
    den = np.sqrt((qq[:, None] * cc[None, :]).astype(np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        cos = np.where(den > 0, dots.astype(np.float64) / den, 0.0)
    live_q, live_c = qq > 0, cc > 0
    ref = 1.0 - cdist(qi[live_q].astype(np.float64), ci[live_c].astype(np.float64), metric="cosine")
    assert np.allclose(cos[np.ix_(live_q, live_c)], ref, rtol=0, atol=1e-12), "cosine disagrees with scipy"
    dist = cdist(qi.astype(np.float64), ci.astype(np.float64), metric="euclidean")
    d2 = ((qi[:, None, :] - ci[None, :, :]) ** 2).sum(axis=2)
    assert np.array_equal(dist, np.sqrt(d2.astype(np.float64))), "scipy's distance is not sqrt of the exact sum"
    values = {"cosine": (cos, False), "dotProduct": (dots.astype(np.float64), False), "euclidean": (dist, True)}

    everyone = np.ones((nq, n), bool)
    eligible = passes(tags, filters)
    assert eligible[4].sum() < k and not eligible[7].any()
    out = dict(corpus=c, queries=q, k=np.int64(k), tags=tags, filters=filters)
    for sim in SIMS:
        val, asc = values[sim]
        never = np.broadcast_to(~live_c, (nq, n)) if sim == "cosine" else np.zeros((nq, n), bool)
        out[f"{sim}_score"], out[f"{sim}_idx"] = rank(val, everyone & ~never, k, asc)
        out[f"{sim}_filtered_score"], out[f"{sim}_filtered_idx"] = rank(val, eligible & ~never, k, asc)
    # the all-ones query: the permutation rows tie exactly under every similarity
    assert len(np.unique(dots[0, 107:307])) == 1 and len(np.unique(dist[0, 107:307])) == 1
    path = os.path.join(HERE, f"int8_topk_independent_d{dim}_n{n}_q{nq}_k{k}.npz")
    np.savez_compressed(path, **out)
    return path


if __name__ == "__main__":
    p = make()
    print(p, os.path.getsize(p), "bytes")
