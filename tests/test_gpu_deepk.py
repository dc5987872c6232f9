"""Deep search (28 < k <= 64) on the H100 against the float64 definition (tests/harness/similarity_oracle.py and, for
filters, tests/harness/filter_oracle.py): index lists equal element for element, scores within 1e-6 * max(1, |ref|),
through the deep scan variant (no own-tail publication, the deep window, the deep pre-pass), the merge's certificate
with k > 32 and the exact fallback scan with 64-entry lists.

Run on an H100 with:  python -m pytest tests -m gpu
"""
import glob
import os

import numpy as np
import pytest

from harness.filter_oracle import eligibility
from harness.filter_oracle import topk_f64 as topk_filtered
from harness.similarity_oracle import topk_f64

pytestmark = pytest.mark.gpu

SIMS = ["cosine", "dotProduct", "euclidean"]
KS = [29, 32, 33, 48, 64]
U64 = np.uint64
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "deepk_topk_independent_*.npz")))


@pytest.fixture(scope="module")
def bf():
    from oracle import bruteforce
    return bruteforce


def dev(bits):
    import torch
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(torch.bfloat16).cuda()


def index(sim, dim, capacity, max_batch=512, max_k=64):
    from qsa_b200.engine import VectorIndex
    return VectorIndex(dim=dim, capacity=capacity, max_batch=max_batch, max_k=max_k, similarity=sim)


def compare(got_s, got_i, rs, ri):
    bad = (got_i != ri).any(axis=1)
    assert not bad.any(), (np.flatnonzero(bad)[:8], got_i[bad][:1], ri[bad][:1])
    got_s = got_s.astype(np.float64)
    fin = np.isfinite(rs)
    assert (got_s[~fin] == rs[~fin]).all()
    if fin.any():
        assert (np.abs(got_s - rs) / np.maximum(1.0, np.abs(rs)))[fin].max() < 1e-6


def check(ix, q, c, k, cg=None, live=None, rows=None):
    """Search all of q; compare the queries `rows` (default all) with the definition."""
    import torch
    if cg is not None:
        ix.set_option("cta_group", cg)
    s, i = ix.search(dev(q), k)
    torch.cuda.synchronize()
    s, i = s.cpu().numpy(), i.cpu().numpy()
    sel = slice(None) if rows is None else rows
    compare(s[sel], i[sel], *topk_f64(q[sel], c, k, ix.similarity, live))
    return s, i


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("n,dim,nq", [
    (20000, 1536, 200),
    (60000, 768, 300),
    (3000, 128, 40),
    (300, 128, 9),       # two tiles, two lanes: U holds 64 rows at most, k > 32 lives on the fallback
    (40, 128, 5),        # fewer rows than k: the remaining slots are empty
])
def test_deep_search_matches_oracle(bf, sim, cg, n, dim, nq):
    c = bf.synth_rows(1000 + n, 0, n, dim)
    q = bf.synth_queries(2000 + n, nq, dim, c)
    ix = index(sim, dim, n)
    ix.append_bf16_bits(c)
    for k in KS:
        s, i = check(ix, q, c, k, cg)
        if n < k:
            assert (i[:, n:] == -1).all()
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_deep_search_over_several_launches(bf, sim):
    n, dim, nq = 40000, 256, 1000
    c = bf.synth_rows(31, 0, n, dim)
    q = bf.synth_queries(32, nq, dim, c)
    ix = index(sim, dim, n, max_batch=1024)
    ix.append_bf16_bits(c)
    ix.set_option("max_launch_qblocks", 2)
    for k in (33, 64):
        check(ix, q, c, k)
        assert ix.last_timing().launches > 1
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_crowd_duplicates_tombstones_and_force_fix(bf, sim, cg):
    """A 100-row crowd of one-ulp variants in one tile with a query next to it (its whole top-64 in one tile lane),
    600 exact duplicates, tombstones among the best rows, then every lane through the fallback."""
    n, dim, nq = 6000, 768, 70
    c = bf.synth_rows(41, 0, n, dim)
    for j in range(99):
        c[1025 + j] = c[1024]
        c[1025 + j, 5 + 7 * j] ^= np.uint16(1)
    c[3000:3600] = c[77]
    q = bf.synth_queries(42, nq, dim, c)
    base = bf.bf16_bits_to_f32(c[1024])
    q[0] = bf.f32_to_bf16_bits(base + np.float32(0.02 * np.abs(base).mean()) *
                               np.random.default_rng(9).standard_normal(dim).astype(np.float32))
    q[1] = c[77]
    ix = index(sim, dim, 8192, max_batch=128)
    ix.append_bf16_bits(c)
    ix.set_option("count_fix", 1)
    ix.set_option("cta_group", cg)
    s, i = check(ix, q, c, 64)
    assert np.isin(i[0], np.arange(1024, 1124)).all()               # query 0's answer is the crowd
    assert ix.info("last_fix_entries") > 0
    dead = [1030, 1031, 3001, 3500, int(i[0, 0])]
    ix.delete_rows(dead)
    live = np.ones(n, bool)
    live[dead] = False
    for k in (33, 64):
        check(ix, q, c, k, live=live)
    ix.set_option("force_fix", 1)
    check(ix, q, c, 64, live=live)
    assert ix.info("last_fix_entries") > 0
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("presample", [0, 4])
def test_window_bound_and_pre_pass_in_force(bf, sim, presample):
    """120 000 rows x 1024 queries: 16 and more tile lanes, so the deep window runs, with and without the pre-pass."""
    n, dim, nq = 120000, 128, 1024
    c = bf.synth_rows(51, 0, n, dim)
    q = bf.synth_queries(52, nq, dim, c)
    ix = index(sim, dim, n, max_batch=1024)
    ix.append_bf16_bits(c)
    ix.set_option("presample", presample)
    ix.set_option("window_bound", 1)
    ix.set_option("count_fix", 1)
    for cg in (1, 2):
        for k in (29, 64):
            check(ix, q, c, k, cg)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_ascending_similarity_order(bf, sim):
    """Rows sorted by ascending similarity to the queries' common direction: without a good early bound every row is an
    insertion; the pre-pass and the window must keep the answer exact either way."""
    n, dim, nq = 100000, 128, 512     # 33 tile lanes: the window runs, and a pre-pass with stride 2 is taken
    g = np.random.default_rng(61)
    v = g.standard_normal(dim).astype(np.float32)
    c = bf.synth_rows(62, 0, n, dim)
    cf = bf.bf16_bits_to_f32(c).astype(np.float64)
    key = cf @ v if sim == "dotProduct" else (cf @ v / np.linalg.norm(cf, axis=1) if sim == "cosine"
                                             else -np.linalg.norm(cf - v, axis=1))
    c = c[np.argsort(key, kind="stable")]
    q = bf.f32_to_bf16_bits(v[None] + np.float32(0.3) * g.standard_normal((nq, dim)).astype(np.float32))
    ix = index(sim, dim, n)
    ix.append_bf16_bits(c)
    for presample in (0, 2):
        ix.set_option("presample", presample)
        for k in (33, 64):
            check(ix, q, c, k)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_filtered_deep_search_selectivities(bf, sim, cg):
    import torch
    n, dim, nq, k = 30000, 256, 160, 64
    g = np.random.default_rng(71)
    c = bf.synth_rows(72, 0, n, dim)
    q = bf.synth_queries(73, nq, dim, c)
    u = g.random(n)
    tags = ((u < 0.10).astype(U64) | ((u < 0.01).astype(U64) << U64(1)) | ((u < 0.001).astype(U64) << U64(2)))
    exact = g.choice(n, k, replace=False)
    fewer = g.choice(n, 40, replace=False)
    tags[exact] |= U64(1 << 3)
    tags[fewer] |= U64(1 << 4)
    ix = index(sim, dim, n)
    ix.append_bf16_bits(c, tags=tags)
    ix.set_option("cta_group", cg)
    for bit in (None, 0, 1, 2, 3, 4):                      # 100 %, 10 %, 1 %, 0.1 %, exactly k, fewer than k
        f = np.tile(np.array([0 if bit is None else 1 << bit, 0, 0, 0], U64), (nq, 1))
        s, i = ix.search(dev(q), k, filters=f)
        torch.cuda.synchronize()
        s, i = s.cpu().numpy(), i.cpu().numpy()
        compare(s, i, *topk_filtered(q, c, k, sim, eligibility(tags, f)))
        if bit == 3:
            assert (np.sort(i, axis=1) == np.sort(exact)).all()
        if bit == 4:
            assert (i[:, 40:] == -1).all()
    s0, i0 = ix.search(dev(q), k)
    s1, i1 = ix.search(dev(q), k, filters=np.zeros(4, U64))
    torch.cuda.synchronize()
    assert torch.equal(i0, i1) and torch.equal(s0.view(torch.int32), s1.view(torch.int32))
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_host_slots_and_shard_exchange(bf, sim):
    import torch
    dim, n, nq = 768, 8000, 150
    c = bf.synth_rows(81, 0, n, dim)
    q = bf.synth_queries(82, nq, dim, c)
    qf = bf.bf16_bits_to_f32(q)
    ix = index(sim, dim, n, max_batch=256)
    ix.append_bf16_bits(c)
    ix.search_host_submit(qf[:70], 64, 0)                  # two searches with different k in flight
    ix.search_host_submit(qf[70:], 33, 1)
    s0, i0 = ix.search_host_wait(0)
    s1, i1 = ix.search_host_wait(1)
    compare(s0, i0, *topk_f64(q[:70], c, 64, sim))
    compare(s1, i1, *topk_f64(q[70:], c, 33, sim))
    cut = 3100
    a, b = index(sim, dim, cut, max_batch=256), index(sim, dim, n - cut, max_batch=256)
    a.append_bf16_bits(c[:cut])
    b.append_bf16_bits(c[cut:])
    hits = torch.stack([a.search_hits(dev(q), 64, 0), b.search_hits(dev(q), 64, cut)])   # k > 32: the serial merge
    ms, mi = a.merge_hits(hits)
    torch.cuda.synchronize()
    compare(ms.cpu().numpy(), mi.cpu().numpy(), *topk_f64(q, c, 64, sim))
    for x in (ix, a, b):
        x.close()


def test_two_gpu_deep_merge(bf):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from qsa_b200.sharded import MultiGpuIndex
    dim, n, nq, k = 256, 8000, 100, 64
    c = bf.synth_rows(91, 0, n, dim)
    q = bf.synth_queries(92, nq, dim, c)
    mi = MultiGpuIndex(dim=dim, capacity_per_gpu=n, max_batch=128, max_k=k, n_gpus=2)
    for lo in range(0, n, 1000):
        mi.append(bf.bf16_bits_to_f32(c[lo:lo + 1000]))
    s, rows = mi.search_host(bf.bf16_bits_to_f32(q), k)
    assert (rows == topk_f64(q, c, k, "cosine")[1]).all()
    mi.close()


def test_vector_table_search_agg_k50(bf):
    from qsa_b200.engine import VectorIndex
    from qsa_b200.operator import VectorTable, vector_search_agg
    dim, n, k = 256, 3000, 50
    c = bf.synth_rows(95, 0, n, dim)
    ix = VectorIndex(dim=dim, capacity=4096, max_batch=64, max_k=64)
    t = VectorTable(ix, name="documents_vectordb_lab2")
    t.upsert_many([f"doc{i}" for i in range(n)], [f"chunk {i}" for i in range(n)], bf.bf16_bits_to_f32(c),
                  [{} for _ in range(n)])
    q = bf.synth_queries(96, 8, dim, c)
    hits = vector_search_agg(t, "embedding", bf.bf16_bits_to_f32(q), k)
    rs, ri = topk_f64(q, c, k, "cosine")
    assert [[h.row for h in hs] for hs in hits] == ri.tolist()
    assert all(len(hs) == k for hs in hits)
    ix.close()


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
@pytest.mark.parametrize("cg", [1, 2])
def test_engine_reproduces_the_independent_deep_fixture(path, cg):
    import torch
    z = np.load(path)
    k = int(z["k"])
    c, q = z["corpus_bits"], z["query_bits"]
    for sim, key in (("cosine", "cosine"), ("dotProduct", "dot"), ("euclidean", "euclidean")):
        ix = index(sim, c.shape[1], len(c), max_batch=128)
        ix.append_bf16_bits(c)
        ix.set_option("cta_group", cg)
        s, i = ix.search(dev(q), k)
        torch.cuda.synchronize()
        compare(s.cpu().numpy(), i.cpu().numpy(), z[f"{key}_score"], z[f"{key}_idx"])
        ix.close()


def test_iid_1m_x_768_k64_needs_no_fallback(bf):
    """The deep bounds must leave the certificate its margin: on iid data nothing goes through the fallback."""
    import torch
    n, dim, nq, k = 1_000_000, 768, 1024, 64
    c = np.concatenate([bf.synth_rows(7, j, 125_000, dim) for j in range(8)])
    q = bf.synth_queries(8, nq, dim, c[:125_000])
    ix = index("cosine", dim, n, max_batch=1024)
    ix.append_bf16_bits(c)
    ix.set_option("count_fix", 1)
    s, i = ix.search(dev(q), k)
    torch.cuda.synchronize()
    assert ix.info("last_fix_entries") == 0
    sample = np.arange(0, nq, 16)
    compare(s.cpu().numpy()[sample], i.cpu().numpy()[sample], *topk_f64(q[sample], c, k, "cosine"))
    ix.close()
