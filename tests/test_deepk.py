"""Deep search (28 < k <= 64) on a CPU box: the C ABI's limits, the deep window bound compiled for the host from the very
source lines of csrc/sa_scan.cuh (`sa_debug_window_bound_deep`), a CPU model of the three stages with the deep bounds
(32-entry lane lists under the kernel's own list rule, merge certificate, exact fallback), exact against
`harness.similarity_oracle.topk_f64`, and the independent k = 64 fixture.  The GPU side is tests/test_gpu_deepk.py."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from harness.similarity_oracle import internal_scores, topk_f64
from oracle import bruteforce as bf
from qsa_b200 import capi

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "deepk_topk_independent_*.npz")))
KL = 32            # entries per lane list of a deep search
SEL_MAX = 128      # candidates the merge kernel re-scores
WIN_POS, WIN_RANK = 5, 14   # the deep window: each lane's 5th best, 14th largest of 16 lanes


def ptr(a):
    return a.ctypes.data_as(C.c_void_p)


# ------------------------------------------------------------------------------------------------ C ABI limits
def test_max_k_is_64():
    assert capi.SA_MAX_K == 64


@pytest.mark.parametrize("max_k", [65, 99])
def test_max_k_past_64_is_refused_before_the_device(lib, max_k):
    h = C.c_void_p()
    assert lib.sa_engine_create(C.byref(h), 0, 128, 1000, 128, max_k) == capi.SA_ERR_ARG
    assert b"max_k" in lib.sa_last_error()
    assert lib.sa_engine_create_sim(C.byref(h), 0, 128, 1000, 128, max_k, capi.SA_SIM_EUCLIDEAN) == capi.SA_ERR_ARG
    assert b"max_k" in lib.sa_last_error()
    assert not h.value


def test_max_k_64_passes_the_argument_stage(lib):
    h = C.c_void_p()
    rc = lib.sa_engine_create(C.byref(h), 0, 128, 1000, 128, 64)
    if rc == capi.SA_OK:                           # a GPU is present: the engine exists
        lib.sa_engine_destroy(h)
        return
    assert b"max_k" not in lib.sa_last_error()     # a GPU-less box fails at the device, not at max_k
    assert rc in (capi.SA_ERR_CUDA, capi.SA_ERR_ARG, capi.SA_ERR_DEVICE)


@pytest.mark.gpu
def test_forced_16_entry_lists_still_refuse_k_past_16():
    from qsa_b200.engine import VectorIndex
    ix = VectorIndex(dim=128, capacity=1024, max_batch=128, max_k=64)
    try:
        ix.append(np.random.default_rng(0).standard_normal((600, 128)).astype(np.float32))
        ix.set_option("list_len", 16)
        with pytest.raises(capi.SaError, match="list_len 16"):
            ix.search_host(np.ones((2, 128), np.float32), 20)
        ix.set_option("list_len", 32)                # forced 32 serves every k up to 64
        s, i = ix.search_host(np.ones((2, 128), np.float32), 64)
        assert (i >= 0).all()
    finally:
        ix.close()


# ------------------------------------------------------------------------------------------------ the deep window
def window_deep(lib, keys):
    keys = np.ascontiguousarray(keys, np.uint32).reshape(-1, 16)
    out = np.empty(len(keys), np.uint32)
    assert lib.sa_debug_window_bound_deep(ptr(keys), len(keys), ptr(out)) == 0
    return out


def f32_keys(lib, x):
    x = np.ascontiguousarray(x, np.float32)
    key, back, below = (np.empty(len(x), t) for t in (np.uint32, np.float32, np.float32))
    assert lib.sa_debug_float_keys(ptr(x), len(x), ptr(key), ptr(back), ptr(below)) == 0
    return key


def test_deep_window_is_the_14th_largest_of_16(lib):
    g = np.random.default_rng(3)
    w = g.integers(1, 2**32, (4000, 16), dtype=np.uint64).astype(np.uint32)
    w[g.random(w.shape) < 0.3] = 0                  # lanes that have published nothing yet
    w[:50] = 0
    w[50:100, :3] = 0                               # exactly 13 published: still a bound (14th largest is the first zero)
    w[100:150] = w[100:150, :1]                     # ties
    out = window_deep(lib, w)
    assert (out == -np.sort(-w.astype(np.int64), axis=1)[:, WIN_RANK - 1]).all()
    assert (out[:50] == 0).all()
    assert (out[50:100] <= np.sort(w[50:100], axis=1)[:, 16 - WIN_RANK]).all()


@pytest.mark.parametrize("seed", range(6))
def test_deep_window_never_exceeds_the_70th_best_of_the_lanes(lib, seed):
    """16 simulated lanes with random rows (some with fewer than 5): the bound from their 5th bests is never above the
    70th largest row of the 16 lanes together, hence never above the k-th best for any k <= 64."""
    g = np.random.default_rng(seed)
    lanes = [g.standard_normal(int(g.choice([2, 4, 5, 9, 40, 300]))).astype(np.float32) * 0.03 for _ in range(16)]
    keys = np.zeros(16, np.uint32)
    for i, rows in enumerate(lanes):
        if len(rows) >= WIN_POS:
            keys[i] = f32_keys(lib, np.sort(rows)[::-1][WIN_POS - 1: WIN_POS])[0]
    bound = window_deep(lib, keys)[0]
    allrows = np.sort(np.concatenate(lanes))[::-1]
    if bound == 0:
        assert (keys != 0).sum() < WIN_RANK
        return
    assert len(allrows) >= WIN_POS * WIN_RANK
    kb = f32_keys(lib, allrows[WIN_POS * WIN_RANK - 1: WIN_POS * WIN_RANK])[0]
    assert bound <= kb
    assert bound <= f32_keys(lib, allrows[63:64])[0]


# ------------------------------------------------------------------------------------------------ the three stages
def lane_list(lib, approx, rows, floor=None):
    approx = np.ascontiguousarray(approx, np.float32)
    rows = np.ascontiguousarray(rows, np.int32)
    out_s, out_r, drop = np.empty(KL, np.float32), np.empty(KL, np.int32), np.empty(1, np.float32)
    f = None if floor is None else ptr(np.ascontiguousarray(floor, np.float32))
    assert lib.sa_debug_list_insert(ptr(approx), ptr(rows), len(approx), KL, f, ptr(out_s), ptr(out_r), ptr(drop)) == 0
    return out_s, out_r, float(drop[0])


def kth_of_union(lists, k):
    cs = np.concatenate([s for s, _ in lists])
    cr = np.concatenate([r for _, r in lists])
    ok = cr >= 0
    cs, cr = cs[ok], cr[ok]
    order = np.lexsort((cr, -cs))
    return cs, cr, (cs[order[k - 1]] if len(order) >= k else None)


def deep_model(lib, exact, approx, eps, n_lanes, k, presample=0):
    """The deep search on one query: exact (float64) / approx (float32, |approx - exact| <= eps) per row.  Tiles of 256
    rows go to lane t % n_lanes.  Stage 0 (presample = S > 1): the lanes scan every S-th tile, and the k-th best of
    their union seeds the shared bound.  Stage 1: every lane scans its tiles under that bound and, with >= 16 lanes, the
    deep window (lock-step: a lane's bound for its tile t is the 14th largest of 16 lanes' 5th bests after tile t-1);
    lanes publish nothing else.  Stage 2: certificate; stage 3: exact rescan of the ambiguous lanes.
    Returns (answer rows, lanes sent to the fallback, whether the union held the approximate top-k)."""
    n = len(exact)
    tiles = np.arange(n) // 256
    lane_rows = [np.flatnonzero(tiles % n_lanes == L).astype(np.int32) for L in range(n_lanes)]
    seed = -np.inf
    if presample > 1:
        lists = []
        for L in range(n_lanes):
            rows = lane_rows[L][(tiles[lane_rows[L]] % presample) == 0]
            s, r, _ = lane_list(lib, approx[rows], rows)
            lists.append((s, r))
        _, _, a = kth_of_union(lists, k)
        if a is not None:
            seed = float(a)
    floors = []
    n_t = max((len(r) + 255) // 256 for r in lane_rows)
    wb = np.full((n_lanes, n_t), -np.inf, np.float32)            # each lane's 5th best after its tile t
    if n_lanes >= 16:
        for L, rows in enumerate(lane_rows):
            for t in range(n_t):
                pre = approx[rows[: (t + 1) * 256]]
                if len(pre) >= WIN_POS:
                    wb[L, t] = np.sort(pre)[::-1][WIN_POS - 1]
    for L, rows in enumerate(lane_rows):
        f = np.full(len(rows), -np.inf, np.float32)
        if len(rows) and np.isfinite(seed):
            f[0] = seed
        if n_lanes >= 16:
            for t in range(1, (len(rows) + 255) // 256):
                win = wb[[(L + i) % n_lanes for i in range(16)], t - 1]
                keys = np.zeros(16, np.uint32)
                fin = np.isfinite(win)
                if fin.any():
                    keys[fin] = f32_keys(lib, win[fin])
                b = window_deep(lib, keys)[0]
                if b != 0:
                    f[t * 256] = win[fin][keys[fin] == b][0]
        floors.append(f)
    lists, drops = [], []
    for rows, f in zip(lane_rows, floors):
        s, r, d = lane_list(lib, approx[rows], rows, f)
        lists.append((s, r))
        drops.append(d)
    cs, cr, a_k = kth_of_union(lists, k)
    union_ok = np.array_equal(np.sort(cs)[::-1][:k], np.sort(approx)[::-1][:k])
    band = -np.inf if a_k is None else np.float32(a_k) - np.float32(2 * eps)
    amb = [d > -np.inf and d >= band for d in drops]
    sel = cr[cs >= band]
    if len(sel) > SEL_MAX:
        amb, sel = [True] * n_lanes, sel[:SEL_MAX]
    best = set(sel.tolist())
    for L in np.flatnonzero(amb):
        rows = lane_rows[L]
        best.update(rows[exact[rows] >= band].tolist())
    cand = np.fromiter(best, dtype=np.int64)
    return cand[np.lexsort((cand, -exact[cand]))[:k]], int(np.sum(amb)), union_ok


def query_and_corpus(g, n, dim, near=None):
    c = bf.f32_to_bf16_bits(g.standard_normal((n, dim)).astype(np.float32))
    q = g.standard_normal((1, dim)).astype(np.float32)
    if near is not None:
        q = bf.bf16_bits_to_f32(c[near])[None] + np.float32(0.05) * q
    return bf.f32_to_bf16_bits(q), c


def exact_values(q, c, sim):
    qf, cf = bf.bf16_bits_to_f32(q).astype(np.float64), bf.bf16_bits_to_f32(c).astype(np.float64)
    return internal_scores(sim, qf @ cf.T, (qf * qf).sum(1), (cf * cf).sum(1))[0]


def check_model(lib, q, c, approx, exact, eps, k, sim, n_lanes, presample=0):
    got, fixed, union_ok = deep_model(lib, exact, approx, eps, n_lanes, k, presample)
    _, want = topk_f64(q, c, k, sim)
    assert (got == want[0]).all(), (k, n_lanes, presample)
    return fixed, union_ok


@pytest.mark.parametrize("sim", ["cosine", "euclidean"])
def test_deep_model_is_exact_on_iid_data_without_fallback(lib, sim):
    g = np.random.default_rng(11)
    q, c = query_and_corpus(g, 24000, 64)
    exact = exact_values(q, c, sim)
    eps = 2e-5 * np.abs(exact).max()
    fixed_total = 0
    for k in (29, 33, 48, 64):
        for n_lanes, presample in ((1, 0), (5, 0), (18, 0), (33, 0), (18, 4)):
            approx = (exact + g.uniform(-1, 1, len(exact)) * eps * 0.01).astype(np.float32)
            fixed, union_ok = check_model(lib, q, c, approx, exact, eps, k, sim, n_lanes, presample)
            if n_lanes == 1:
                # one lane: U holds 32 rows; k > 32 finds fewer than k candidates and must end in the fallback
                assert fixed == (1 if k > KL else 0), k
                continue
            assert union_ok, (k, n_lanes, presample)     # the deep bounds never cut the approximate top-k
            fixed_total += fixed
    assert fixed_total == 0     # the margin of the deep bounds leaves the certificate its room on iid data


@pytest.mark.parametrize("err", [0.01, 0.999])
def test_deep_model_is_exact_for_any_error_up_to_eps(lib, err):
    g = np.random.default_rng(12)
    q, c = query_and_corpus(g, 16000, 64)
    exact = exact_values(q, c, "dotProduct")
    eps = 1e-3
    for k, n_lanes in ((30, 4), (64, 18), (64, 40), (50, 16)):
        approx = (exact + err * g.choice([-eps, eps], len(exact))).astype(np.float32)
        check_model(lib, q, c, approx, exact, eps, k, "dotProduct", n_lanes, presample=3 if n_lanes == 18 else 0)


def test_deep_model_crowd_of_40_near_ties_in_one_lane(lib):
    """40 one-ulp variants of one row in one tile (one lane), the query next to them, the approximate order reversed:
    that lane holds only 32 of the true top-k, its drop falls in the band, and the fallback rescans it."""
    g = np.random.default_rng(13)
    q, c = query_and_corpus(g, 20000, 64, near=123)
    crowd = np.arange(5000, 5040)
    for j, r in enumerate(crowd):
        c[r] = c[123]
        c[r, j % 64] ^= np.uint16(1 + j // 64)
    exact = exact_values(q, c, "cosine")
    eps = 2e-5
    rank = np.argsort(np.argsort(-exact[crowd]))
    approx = exact.astype(np.float32)
    approx[crowd] = np.float32(exact[crowd].max()) + rank.astype(np.float32) * np.float32(1e-7)   # reversed order
    for k in (33, 64):
        for n_lanes in (1, 18, 33):
            fixed, _ = check_model(lib, q, c, approx, exact, eps, k, "cosine", n_lanes, presample=4 if n_lanes == 18 else 0)
            assert fixed >= 1


def test_deep_model_600_exact_duplicates(lib):
    g = np.random.default_rng(14)
    q, c = query_and_corpus(g, 20000, 64, near=77)
    dup = np.sort(g.choice(np.arange(100, 20000), 600, replace=False))
    c[dup] = c[77]
    exact = exact_values(q, c, "dotProduct")
    approx = exact.astype(np.float32)
    for k, n_lanes in ((64, 18), (40, 33), (64, 1)):
        fixed, _ = check_model(lib, q, c, approx, exact, 1e-4, k, "dotProduct", n_lanes)
        assert fixed == n_lanes        # more band candidates than the merge kernel re-scores: every lane is rescanned


def test_deep_model_ascending_similarity_order(lib):
    """Rows sorted by ascending similarity: every row beats its lane's list while it fills; the deep pre-pass bound and
    the window must still leave the answer exact."""
    g = np.random.default_rng(15)
    q, c = query_and_corpus(g, 12000, 64)
    exact = exact_values(q, c, "euclidean")
    order = np.argsort(exact, kind="stable")
    c = c[order]
    exact = exact[order]
    eps = 1e-4 * np.abs(exact).max()
    approx = (exact + g.uniform(-1, 1, len(exact)) * eps * 0.5).astype(np.float32)
    for k, n_lanes, presample in ((64, 16, 0), (64, 16, 2), (29, 40, 0), (48, 5, 3)):
        check_model(lib, q, c, approx, exact, eps, k, "euclidean", n_lanes, presample)


# ------------------------------------------------------------------------------------------------ independent fixture
def test_deepk_fixture_exists():
    assert len(GOLDEN) == 1 and os.path.getsize(GOLDEN[0]) < 1 << 20


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_oracle_reproduces_the_independent_deep_fixture(path):
    z = np.load(path)
    k = int(z["k"])
    assert k == 64
    for sim, key in (("cosine", "cosine"), ("dotProduct", "dot"), ("euclidean", "euclidean")):
        s, i = topk_f64(z["query_bits"], z["corpus_bits"], k, sim)
        assert (i == z[f"{key}_idx"]).all(), sim
        assert np.array_equal(s, z[f"{key}_score"]), sim
    crowd = z["crowd_rows"]
    assert len(crowd) == 100 and len(np.unique(crowd // 256)) == 1          # one tile
    assert np.isin(z["cosine_idx"][0], crowd).sum() == k                    # query 0's top-64 lies in the crowd


def test_serve_cli_accepts_k_up_to_64():
    from scripts.sa_serve import build_parser
    assert build_parser().parse_args(["--k", "64"]).k == 64
    with pytest.raises(SystemExit):
        build_parser().parse_args(["--k", "65"])
    with pytest.raises(SystemExit):
        build_parser().parse_args(["--k", "0"])
