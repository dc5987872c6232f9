"""Pre-filtered search on the H100 against the filtered definition (tests/harness/filter_oracle.py): index lists equal
element for element, scores within 1e-6 * max(1, |ref|), for both CTA groupings and every similarity, through the
filtered scan, the merge's certificate over the eligible rows, and the exact fallback scan.

Run on an H100 with:  python -m pytest tests -m gpu
"""
import glob
import os

import numpy as np
import pytest

from harness.filter_oracle import eligibility, topk_f64

pytestmark = pytest.mark.gpu

SIMS = ["cosine", "dotProduct", "euclidean"]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "filter_topk_independent_*.npz")))
U64 = np.uint64


@pytest.fixture(scope="module")
def bf():
    from oracle import bruteforce
    return bruteforce


def dev(bits):
    import torch
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(torch.bfloat16).cuda()


def index(sim, dim, capacity, max_batch=512, max_k=28):
    from qsa_b200.engine import VectorIndex
    return VectorIndex(dim=dim, capacity=capacity, max_batch=max_batch, max_k=max_k, similarity=sim)


def random_tags(g, n, p=0.5, bits=8):
    return (g.random((n, bits)) < p).astype(np.uint64) @ (U64(1) << np.arange(bits, dtype=np.uint64))


def compare(got_s, got_i, rs, ri):
    assert (got_i == ri).all(), (np.flatnonzero((got_i != ri).any(axis=1))[:8], got_i[(got_i != ri).any(axis=1)][:2],
                                 ri[(got_i != ri).any(axis=1)][:2])
    got_s = got_s.astype(np.float64)
    fin = np.isfinite(rs)
    assert (got_s[~fin] == rs[~fin]).all()
    if fin.any():
        assert (np.abs(got_s - rs) / np.maximum(1.0, np.abs(rs)))[fin].max() < 1e-6


def check(ix, q, c, k, tags, filters, cg=None, live=None):
    import torch
    if cg is not None:
        ix.set_option("cta_group", cg)
    f = np.broadcast_to(np.asarray(filters, U64), (len(q), 4))
    s, i = ix.search(dev(q), k, filters=f)
    torch.cuda.synchronize()
    rs, ri = topk_f64(q, c, k, ix.similarity, eligibility(tags, f, live))
    compare(s.cpu().numpy(), i.cpu().numpy(), rs, ri)
    return s.cpu().numpy(), i.cpu().numpy()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("n,dim,nq,k", [
    (20000, 1536, 200, 10),
    (5000, 768, 37, 5),
    (256, 64, 1, 1),
    (257, 128, 129, 3),
    (70000, 256, 300, 12),
    (70000, 256, 300, 16),
    (2000, 256, 40, 16),
    (9000, 192, 64, 28),
])
def test_filtered_search_matches_oracle(bf, sim, cg, n, dim, nq, k):
    """Per-query filters drawn from every clause kind, several selectivities in one batch."""
    g = np.random.default_rng(n + nq)
    c = bf.synth_rows(1234, 0, n, dim)
    q = bf.synth_queries(4321, nq, dim, c)
    tags = random_tags(g, n)
    f = np.zeros((nq, 4), U64)
    for i in range(nq):
        a, b = U64(1) << U64(g.integers(8)), U64(1) << U64(g.integers(8))
        f[i, i % 4] = a | (b if i % 3 == 0 else U64(0))
    ix = index(sim, dim, n + 513)
    ix.append_bf16_bits(c, tags=tags)
    check(ix, q, c, k, tags, f, cg)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_selectivities_down_to_none(bf, sim, cg):
    n, dim, nq, k = 30000, 256, 160, 10
    g = np.random.default_rng(7)
    c = bf.synth_rows(21, 0, n, dim)
    q = bf.synth_queries(22, nq, dim, c)
    u = g.random(n)
    tags = ((u < 0.10).astype(U64) | ((u < 0.01).astype(U64) << U64(1)) | ((u < 0.001).astype(U64) << U64(2)))
    exact = g.choice(n, k, replace=False)
    fewer = g.choice(n, 3, replace=False)
    tags[exact] |= U64(1 << 3)
    tags[fewer] |= U64(1 << 4)
    ix = index(sim, dim, n)
    ix.append_bf16_bits(c, tags=tags)
    ix.set_option("count_fix", 1)
    for bit in (None, 0, 1, 2, 3, 4, 5):                      # 100 %, 10 %, 1 %, 0.1 %, exactly k, fewer than k, none
        f = [0, 0, 0, 0] if bit is None else [1 << bit, 0, 0, 0]
        s, i = check(ix, q, c, k, tags, f, cg)
        if bit == 3:
            assert (np.sort(i, axis=1) == np.sort(exact)).all()
        if bit == 4:
            assert (i[:, 3:] == -1).all()
        if bit == 5:
            assert (i == -1).all() and (s == (np.inf if sim == "euclidean" else -np.inf)).all()
            assert ix.info("last_fix_entries") == 0
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("presample", [0, 4])
def test_adversarial_exclusion_of_the_best_rows(bf, sim, presample):
    """The 1 000 best rows of every query carry a tag the filter excludes: any leak of an ineligible row into a list,
    a dropped bound, a shared threshold, the window bound or the sampling pre-pass would show."""
    import torch
    n, dim, nq, k = 120000, 128, 1024, 10         # 1024 queries: 16 tile lanes, so the window bound and the pre-pass run
    c = bf.synth_rows(51, 0, n, dim)
    q = bf.synth_queries(52, nq, dim, c)
    tags = np.zeros(n, U64)
    ix = index(sim, dim, n, max_batch=1024)
    ix.append_bf16_bits(c)
    # the best 1 000 of each query under this similarity, from the definition
    from harness.similarity_oracle import topk_f64 as plain
    _, best = plain(q, c, 1000, sim)
    tags[np.unique(best)] = U64(1)
    ix.set_tags(np.arange(n), tags)
    ix.set_option("presample", presample)
    ix.set_option("window_bound", 1)
    ix.set_option("count_fix", 1)
    for cg in (1, 2):
        check(ix, q, c, k, tags, [0, 1, 0, 0], cg)
    torch.cuda.synchronize()
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_per_query_filters_across_launches_and_match_all_equals_unfiltered(bf, sim):
    import torch
    n, dim, nq, k = 40000, 256, 1000, 10
    g = np.random.default_rng(8)
    c = bf.synth_rows(61, 0, n, dim)
    q = bf.synth_queries(62, nq, dim, c)
    tags = random_tags(g, n, 0.3)
    f = np.zeros((nq, 4), U64)
    f[:, 0] = U64(1) << g.integers(8, size=nq).astype(U64)
    f[::5, 0] = 0
    f[1::5, 1] = U64(1) << U64(2)
    ix = index(sim, dim, n, max_batch=1024)
    ix.append_bf16_bits(c, tags=tags)
    ix.set_option("max_launch_qblocks", 2)                      # several scan launches in one search
    check(ix, q, c, k, tags, f)
    assert ix.last_timing().launches > 1
    s0, i0 = ix.search(dev(q), k)
    s1, i1 = ix.search(dev(q), k, filters=np.zeros(4, U64))
    torch.cuda.synchronize()
    assert torch.equal(i0, i1) and torch.equal(s0.view(torch.int32), s1.view(torch.int32))
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_crowds_fallback_and_force_fix(bf, sim, cg):
    n, dim, nq = 3000, 1536, 70
    c = bf.synth_rows(1234, 0, n, dim)
    for j in range(24):
        c[1000 + j] = c[123]
        c[1000 + j, 7 + 61 * j] ^= np.uint16(1)
    c[2000:2600] = c[77]
    q = bf.synth_queries(4321, nq, dim, c)
    base = bf.bf16_bits_to_f32(c[123])
    q[0] = bf.f32_to_bf16_bits(base + np.float32(0.1 * np.abs(base).mean()) *
                               np.random.default_rng(99).standard_normal(dim).astype(np.float32))
    q[1] = c[77]
    tags = np.zeros(n, U64)
    tags[::2] = U64(1)                                           # half of each crowd is eligible
    ix = index(sim, dim, 4096, max_batch=128)
    ix.append_bf16_bits(c, tags=tags)
    ix.delete_rows([1002, 2004])
    live = np.ones(n, bool)
    live[[1002, 2004]] = False
    for k in (10, 12):
        check(ix, q, c, k, tags, [1, 0, 0, 0], cg, live=live)
    ix.set_option("force_fix", 1)
    ix.set_option("count_fix", 1)
    check(ix, q, c, 10, tags, [0, 1, 0, 0], cg, live=live)
    assert ix.info("last_fix_entries") > 0
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_streaming_tags_set_tags_and_reset(bf, sim):
    n, dim, nq, k = 6000, 256, 100, 10
    g = np.random.default_rng(12)
    c = bf.synth_rows(71, 0, n, dim)
    q = bf.synth_queries(72, nq, dim, c)
    tags = random_tags(g, n, 0.4, 4)
    ix = index(sim, dim, 8192, max_batch=128)
    assert ix.info("has_tags") == 1
    ix.append_bf16_bits(c[:2000], tags=tags[:2000])
    cf = bf.bf16_bits_to_f32(c)
    ix.append(cf[2000:4000], tags=tags[2000:4000])            # host fp32 ingest
    import torch
    ix.append(torch.from_numpy(cf[4000:]).cuda(), tags=tags[4000:])   # device fp32 ingest
    check(ix, q, c, k, tags, [1, 0, 0, 0])
    flip = g.choice(n, 500, replace=False)
    tags[flip] ^= U64(1)
    ix.set_tags(flip, tags[flip])
    check(ix, q, c, k, tags, [1, 0, 0, 0])
    ix.delete_rows([5, 6])
    live = np.ones(n, bool)
    live[[5, 6]] = False
    check(ix, q, c, k, tags, [0, 2, 0, 0], live=live)
    ix.reset()
    ix.append_bf16_bits(c[:3000])                               # tags=None: zeros, not the old rows' tags
    check(ix, q, c[:3000], k, np.zeros(3000, U64), [0, 0, 1, 0])  # requires bit 0: nothing matches
    check(ix, q, c[:3000], k, np.zeros(3000, U64), [0, 1, 0, 0])  # excludes bit 0: everything matches
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_host_slots_hits_and_snapshot(bf, sim, tmp_path):
    import torch
    dim, n, nq, k = 768, 8000, 150, 10
    g = np.random.default_rng(3)
    c = bf.synth_rows(81, 0, n, dim)
    q = bf.synth_queries(82, nq, dim, c)
    qf = bf.bf16_bits_to_f32(q)
    tags = random_tags(g, n, 0.5, 4)
    ix = index(sim, dim, n, max_batch=256, max_k=k)
    ix.append_bf16_bits(c, tags=tags)
    fa, fb = np.array([1, 0, 0, 0], U64), np.array([0, 0, 6, 0], U64)
    ix.search_host_submit(qf[:70], k, 0, filters=fa)
    f1 = np.tile(fb, (80, 1))
    ix.search_host_submit(qf[70:], k, 1, filters=f1)
    f1[:] = 0                                                   # the staged copy is what the search reads
    s0, i0 = ix.search_host_wait(0)
    s1, i1 = ix.search_host_wait(1)
    r0 = topk_f64(q[:70], c, k, sim, eligibility(tags, np.tile(fa, (70, 1))))
    r1 = topk_f64(q[70:], c, k, sim, eligibility(tags, np.tile(fb, (80, 1))))
    compare(s0, i0, *r0)
    compare(s1, i1, *r1)
    hs, hi = ix.search_host(qf[:70], k, filters=fa)
    compare(hs, hi, *r0)
    # fp32 device queries, unfiltered and filtered; filters staged on the device give the numpy form's bits
    fd = torch.from_numpy(np.tile(fb, (nq, 1)).view(np.int64)).cuda()
    rb = topk_f64(q, c, k, sim, eligibility(tags, np.tile(fb, (nq, 1))))
    for filters, want in ((None, topk_f64(q, c, k, sim, np.ones((nq, n), bool))), (fb, rb), (fd, rb)):
        s, i = ix.search(torch.from_numpy(qf).cuda(), k, filters=filters)
        torch.cuda.synchronize()
        compare(s.cpu().numpy(), i.cpu().numpy(), *want)
    (sn, i_n), (sd, i_d) = ix.search(dev(q), k, filters=fb), ix.search(dev(q), k, filters=fd)
    assert torch.equal(sn, sd) and torch.equal(i_n, i_d)
    for bad, err in ((fd[:10], ValueError), (fd.int(), TypeError), (fd.t().contiguous().t(), ValueError)):
        with pytest.raises(err):
            ix.search(dev(q), k, filters=bad)
    with pytest.raises(ValueError, match="host"):
        ix.search_host(qf, k, filters=fd)                       # device filters cannot serve a host-buffer search
    # a one-GPU ShardedIndex (torch transport): search_hits + merge_hits
    from qsa_b200.sharded import ShardedIndex
    sh = ShardedIndex(ix, row_offset=0)
    assert sh.transport == "torch"
    s, i = sh.search(dev(q), k, filters=fb)
    torch.cuda.synchronize()
    compare(s.cpu().numpy(), i.cpu().numpy(), *rb)
    compare(*sh.search_host(qf, k, filters=fb), *rb)
    # two shards on one GPU through the packed exchange
    cut = 3100
    a, b = index(sim, dim, cut, max_batch=256, max_k=k), index(sim, dim, n - cut, max_batch=256, max_k=k)
    a.append_bf16_bits(c[:cut], tags=tags[:cut])
    b.append_bf16_bits(c[cut:], tags=tags[cut:])
    hits = torch.stack([a.search_hits(dev(q), k, 0, filters=fb), b.search_hits(dev(q), k, cut, filters=fb)])
    ms, mi = a.merge_hits(hits)
    torch.cuda.synchronize()
    compare(ms.cpu().numpy(), mi.cpu().numpy(), *topk_f64(q, c, k, sim, eligibility(tags, np.tile(fb, (nq, 1)))))
    # snapshot / restore carries the tags
    ix.snapshot(str(tmp_path / "s"))
    ix2 = index(sim, dim, n, max_batch=256, max_k=k)
    assert ix2.restore(str(tmp_path / "s")) == n
    check(ix2, q, c, k, tags, fb)
    for x in (ix, ix2, a, b):
        x.close()


def test_filtered_search_without_tags_or_filters_is_refused(bf):
    import torch
    from qsa_b200 import capi
    ix = index("cosine", 128, 1024, max_batch=64, max_k=10)
    c = bf.synth_rows(1, 0, 600, 128)
    ix.append_bf16_bits(c)
    qd = dev(bf.synth_queries(2, 4, 128, c))
    out_s = torch.empty((4, 10), dtype=torch.float32, device="cuda")
    out_i = torch.empty((4, 10), dtype=torch.int32, device="cuda")
    f = torch.zeros((4, 4), dtype=torch.int64, device="cuda")
    lib = ix.lib
    assert lib.sa_search_filtered(ix._h, qd.data_ptr(), None, 4, 10, out_s.data_ptr(), out_i.data_ptr(), None, 0) == \
        capi.SA_ERR_ARG
    assert lib.sa_corpus_bind_tags(ix._h, None) == 0 and ix.info("has_tags") == 0
    rc = lib.sa_search_filtered(ix._h, qd.data_ptr(), f.data_ptr(), 4, 10, out_s.data_ptr(), out_i.data_ptr(), None, 0)
    assert rc == capi.SA_ERR_ARG and b"sa_corpus_bind_tags" in lib.sa_last_error()
    hf = np.zeros((4, 4), U64)
    qf = bf.bf16_bits_to_f32(bf.synth_queries(2, 4, 128, c))
    rc = lib.sa_search_host_filtered(ix._h, qf.ctypes.data, hf.ctypes.data, 4, 10, np.zeros((4, 10), np.float32).ctypes.data,
                                     np.zeros((4, 10), np.int32).ctypes.data)
    assert rc == capi.SA_ERR_ARG
    s, i = ix.search(qd, 10)                                     # the unfiltered search is unaffected
    torch.cuda.synchronize()
    assert (i.cpu().numpy() >= 0).all()
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_engine_reproduces_the_independent_fixture(path, sim, cg):
    import torch
    z = np.load(path)
    k = int(z["k"])
    cb, qb = z["corpus_bits"], z["query_bits"]
    ix = index(sim, cb.shape[1], len(cb) + 256, max_batch=64, max_k=k)
    ix.append_bf16_bits(cb, tags=z["tags"])
    ix.set_option("cta_group", cg)
    s, i = ix.search(dev(qb), k, filters=z["filters"])
    torch.cuda.synchronize()
    key = {"cosine": "cosine", "dotProduct": "dot", "euclidean": "euclidean"}[sim]
    assert (i.cpu().numpy() == z[f"{key}_idx"]).all()
    ref = z[f"{key}_score"]
    fin = np.isfinite(ref)
    assert (np.abs(s.cpu().numpy() - ref) / np.maximum(1.0, np.abs(ref)))[fin].max() < 1e-6
    ix.close()


def test_two_gpu_filtered_merge(bf):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from qsa_b200.sharded import MultiGpuIndex
    dim, n, nq, k = 256, 8000, 100, 10
    g = np.random.default_rng(4)
    c = bf.synth_rows(41, 0, n, dim)
    q = bf.synth_queries(42, nq, dim, c)
    tags = random_tags(g, n, 0.3, 4)
    mi = MultiGpuIndex(dim=dim, capacity_per_gpu=n, max_batch=128, max_k=k, n_gpus=2)
    for lo in range(0, n, 1000):
        mi.append(bf.bf16_bits_to_f32(c[lo:lo + 1000]), tags=tags[lo:lo + 1000])
    f = np.array([1, 0, 0, 0], U64)
    s, rows = mi.search_host(bf.bf16_bits_to_f32(q), k, filters=f)
    rs, ri = topk_f64(q, c, k, "cosine", eligibility(tags, np.tile(f, (nq, 1))))
    assert (rows == ri).all()
    mi.close()


def test_lab4_table_filtered_vector_search_agg(bf):
    from qsa_b200.engine import VectorIndex
    from qsa_b200.operator import VectorTable, vector_search_agg
    dim, n, k = 256, 3000, 5
    g = np.random.default_rng(6)
    c = bf.synth_rows(91, 0, n, dim)
    cats = ["duplicate_benefits", "identity_theft", "contractor_fraud", "false_claims"]
    titles = ["Stafford Act", "44 CFR 206", "Disaster Fraud Guide"]
    meta = [{"fraud_categories": [x for x in cats if g.random() < 0.3], "title": titles[int(g.integers(3))],
             "section_reference": f"s{i % 7}"} for i in range(n)]
    ix = VectorIndex(dim=dim, capacity=4096, max_batch=64, max_k=k)
    t = VectorTable(ix, name="fema_policies_vectordb", filter_fields=("fraud_categories", "title"))
    cf = bf.bf16_bits_to_f32(c)
    t.upsert_many([f"doc{i}" for i in range(n)], [f"chunk {i}" for i in range(n)], cf, meta)
    q = bf.synth_queries(92, 8, dim, c)
    mql = {"fraud_categories": {"$in": ["identity_theft", "false_claims"]}, "title": {"$ne": "Stafford Act"}}
    hits = vector_search_agg(t, "embedding", bf.bf16_bits_to_f32(q), k, filter=mql)
    ok = np.array([any(x in m["fraud_categories"] for x in ("identity_theft", "false_claims")) and
                   m["title"] != "Stafford Act" for m in meta])
    rs, ri = topk_f64(q, c, k, "cosine", np.tile(ok, (len(q), 1)))
    assert [[h.row for h in hs] for hs in hits] == ri.tolist()
    for hs in hits:
        for h in hs:
            assert h.metadata["title"] != "Stafford Act" and h.document_id == f"doc{h.row}"
    per_query = vector_search_agg(t, "embedding", bf.bf16_bits_to_f32(q[:2]), k,
                                  filter=[{"title": "44 CFR 206"}, {"fraud_categories": "contractor_fraud"}])
    assert all(h.metadata["title"] == "44 CFR 206" for h in per_query[0])
    assert all("contractor_fraud" in h.metadata["fraud_categories"] for h in per_query[1])
    ix.close()
