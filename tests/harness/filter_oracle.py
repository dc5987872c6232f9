"""CPU definition of the pre-filtered search -- TEST INFRASTRUCTURE ONLY.

The answer for query i is ``similarity_oracle.topk_f64`` restricted to the rows eligible for it: live (not a tombstone)
and passing its filter.  ``eligible`` is a boolean mask [nq, n]; ``eligibility`` builds it from the rows' tags and the
queries' sa_filter words with the predicate of include/sa_api.h.  ``oracle/`` and ``similarity_oracle`` are reused as
they are.
"""
from __future__ import annotations

import numpy as np

from harness.similarity_oracle import SIMILARITIES, RunningTopk, internal_scores, public_scores
from oracle import bruteforce as bf


def eligibility(tags: np.ndarray, filters: np.ndarray, live=None) -> np.ndarray:
    """bool [nq, n]: live[r] and pass(tags[r], filters[i]); filters uint64 [nq, 4] (all_of, none_of, any_of[2])."""
    t = np.asarray(tags, dtype=np.uint64)[None, :]
    f = np.asarray(filters, dtype=np.uint64)
    z = np.uint64(0)
    ok = ((t & f[:, 0:1]) == f[:, 0:1]) & ((t & f[:, 1:2]) == z)
    for j in (2, 3):
        a = f[:, j:j + 1]
        ok &= (a == z) | ((t & a) != z)
    if live is not None:
        ok &= np.asarray(live, dtype=bool)[None, :]
    return ok


def topk_f64(q_bits: np.ndarray, c_bits: np.ndarray, k: int, similarity: str, eligible: np.ndarray,
             chunk: int = 32768):
    """Exact filtered top-k.  Returns (score float64 [nq,k], row int64 [nq,k]); empty slots (-inf / +inf, -1)."""
    if similarity not in SIMILARITIES:
        raise ValueError(f"unknown similarity {similarity!r}")
    q = bf.bf16_bits_to_f32(q_bits).astype(np.float64)
    qq = (q * q).sum(axis=1)
    acc = RunningTopk(q.shape[0], k)
    for lo in range(0, c_bits.shape[0], chunk):
        c = bf.bf16_bits_to_f32(c_bits[lo: lo + chunk]).astype(np.float64)
        s = internal_scores(similarity, q @ c.T, qq, (c * c).sum(axis=1))
        s[~eligible[:, lo: lo + chunk]] = -np.inf
        acc.add(s, lo)
    return public_scores(similarity, acc.s), acc.i
