"""Regenerates tests/golden/cosine_topk_*.npz: small seeded inputs and the float64 oracle's answers.

The reference holds no golden vector for this arithmetic (SURVEY.md section 8c: parity unpinned), so these
fixtures pin the ORACLE's behaviour over time (and keep the tests independent of a reference checkout).
Run from the repo root:  python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import bruteforce as bf  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

CASES = {
    # name: (n, dim, nq, k, corpus seed, query seed)
    "d64_n2500_q37_k10": (2500, 64, 37, 10, 101, 202),
    "d128_n1000_q130_k5": (1000, 128, 130, 5, 303, 404),
    "d192_n777_q9_k3": (777, 192, 9, 3, 505, 606),
}


def build(name):
    n, dim, nq, k, cs, qs = CASES[name]
    c = bf.synth_rows(cs, 0, n, dim)
    # edge material: duplicates (ties), an all-zero row, a scaled copy (same cosine as the original)
    c[n // 2] = c[5]
    c[n // 3] = 0
    c[n - 1] = bf.f32_to_bf16_bits(bf.bf16_bits_to_f32(c[17]) * 4)
    q = bf.synth_queries(qs, nq, dim, c)
    q[0] = c[5]
    q[min(2, nq - 1)] = c[17]
    s, i = bf.cosine_topk_f64(q, c, k)
    return dict(corpus=c, queries=q, k=np.int64(k), score=s, index=i)


if __name__ == "__main__":
    for name in CASES:
        np.savez_compressed(os.path.join(HERE, f"cosine_topk_{name}.npz"), **build(name))
        print("wrote", name)
