"""CPU definition of the search under every similarity of the index -- TEST INFRASTRUCTURE ONLY.

The counterpart of ``oracle.bruteforce.cosine_topk_f64`` for the three similarities an Atlas vector index accepts
("cosine", "dotProduct", "euclidean"; include/sa_api.h, SA_SIM_*).  ``oracle.bruteforce`` is left as it is: cosine
keeps its own definition there, and this module reuses its bf16 helpers.

    value(q, c)   cosine      <q,c> / (|q| |c|)                        (all-zero rows are never returned)
                  dotProduct  <q,c>
                  euclidean   d = sqrt(max(0, (|q|^2 - 2 <q,c>) + |c|^2))   -- the engine's formula, term for term
    result        the k best rows: (value desc, row asc), for euclidean (d asc, row asc);
                  rows with live[r] False (tombstones) are never returned, nor is a row whose value is not finite (a
                  row holding a NaN or inf element, under every similarity); empty slots hold (-inf, -1), (+inf, -1)
                  for d

All arithmetic runs over the bf16-rounded values with float64 sums.  bf16 x bf16 products have at most 16 significant
bits, so the sums are exact for any data whose magnitudes span less than ~2^30 within a row, and the summation order
does not matter; the euclidean formula then rounds identically here and on the device, so ties resolve identically.
"""
from __future__ import annotations

import numpy as np

from oracle import bruteforce as bf

SIMILARITIES = ("cosine", "dotProduct", "euclidean")


def internal_scores(similarity: str, dots: np.ndarray, qq: np.ndarray, cc: np.ndarray) -> np.ndarray:
    """[nq, m] float64 values where larger is better (euclidean: -d), from <q,c> [nq, m], |q|^2 [nq], |c|^2 [m]."""
    if similarity == "cosine":
        den = np.sqrt(qq)[:, None] * np.sqrt(cc)[None, :]
        with np.errstate(divide="ignore", invalid="ignore"):
            s = np.where(den > 0, dots / den, 0.0)
        s[:, cc == 0] = -np.inf                       # all-zero rows are never returned under cosine
        return s
    if similarity == "dotProduct":
        return dots.copy()
    if similarity == "euclidean":
        d2 = (qq[:, None] - 2.0 * dots) + cc[None, :]
        return -np.sqrt(np.maximum(d2, 0.0))
    raise ValueError(f"unknown similarity {similarity!r}")


def public_scores(similarity: str, s: np.ndarray) -> np.ndarray:
    """Internal (larger is better) values -> the returned scores (euclidean: the distance; empty slots +inf)."""
    return -s if similarity == "euclidean" else s


class RunningTopk:
    """Running top-k of internal values over row chunks, by (value desc, row asc)."""

    def __init__(self, nq: int, k: int):
        self.k = k
        self.s = np.full((nq, k), -np.inf)
        self.i = np.full((nq, k), -1, dtype=np.int64)

    def add(self, s: np.ndarray, first_row: int) -> None:
        m = s.shape[1]
        if m == 0:
            return
        s = np.where(np.isfinite(s), s, -np.inf)     # a NaN would sort last in the partition below and hide a row
        kk = min(self.k, m)
        kth = np.partition(s, m - kk, axis=1)[:, m - kk]
        for r in range(s.shape[0]):
            cand = np.flatnonzero(s[r] >= kth[r])
            cs = np.concatenate([self.s[r], s[r, cand]])
            ci = np.concatenate([self.i[r], cand.astype(np.int64) + first_row])
            keep = np.isfinite(cs)
            order = np.lexsort((ci[keep], -cs[keep]))[: self.k]
            self.s[r] = -np.inf
            self.i[r] = -1
            self.s[r, : len(order)] = cs[keep][order]
            self.i[r, : len(order)] = ci[keep][order]


def topk_f64(q_bits: np.ndarray, c_bits: np.ndarray, k: int, similarity: str = "cosine", live=None,
             chunk: int = 32768):
    """Exact top-k under ``similarity``.  Returns (score float64 [nq,k], row int64 [nq,k])."""
    if similarity not in SIMILARITIES:
        raise ValueError(f"unknown similarity {similarity!r}")
    q = bf.bf16_bits_to_f32(q_bits).astype(np.float64)
    qq = (q * q).sum(axis=1)
    live = None if live is None else np.asarray(live, dtype=bool)
    acc = RunningTopk(q.shape[0], k)
    for lo in range(0, c_bits.shape[0], chunk):
        c = bf.bf16_bits_to_f32(c_bits[lo: lo + chunk]).astype(np.float64)
        s = internal_scores(similarity, q @ c.T, qq, (c * c).sum(axis=1))
        if live is not None:
            s[:, ~live[lo: lo + chunk]] = -np.inf
        acc.add(s, lo)
    return public_scores(similarity, acc.s), acc.i


def merge_shard_topk(shard_scores, shard_rows, offsets, k: int, descending: bool = True):
    """``oracle.bruteforce.merge_shard_topk`` with a direction: descending=False merges distances (value asc, row asc);
    empty slots are then (+inf, -1)."""
    if descending:
        return bf.merge_shard_topk(shard_scores, shard_rows, offsets, k)
    s, i = bf.merge_shard_topk([-np.asarray(x) for x in shard_scores], shard_rows, offsets, k)
    return -s, i
