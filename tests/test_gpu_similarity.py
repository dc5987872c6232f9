"""dotProduct and euclidean search on the H100 against the CPU definition (tests/harness/similarity_oracle.py): index lists
equal element for element, scores within 1e-6 * max(1, |ref|), for both CTA groupings, through the scan's two epilogues
(multiply for dotProduct, subtract for euclidean), the certificate with its norm-dependent bound, the exact rescoring and
the fallback scan.

Run on an H100 with:  python -m pytest tests -m gpu
"""
import glob
import json
import os
import struct

import numpy as np
import pytest

from harness.similarity_oracle import topk_f64

pytestmark = pytest.mark.gpu

SIMS = ["dotProduct", "euclidean"]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "similarity_topk_independent_*.npz")))


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


def check(ix, q_bits, c_bits, k, cg=None, live=None):
    import torch
    if cg is not None:
        ix.set_option("cta_group", cg)
    s, i = ix.search(dev(q_bits), k)
    torch.cuda.synchronize()
    rs, ri = topk_f64(q_bits, c_bits, k, ix.similarity, live=live)
    got_i, got_s = i.cpu().numpy(), s.cpu().numpy().astype(np.float64)
    assert (got_i == ri).all(), (np.flatnonzero((got_i != ri).any(axis=1))[:8], got_i[(got_i != ri).any(axis=1)][:2],
                                 ri[(got_i != ri).any(axis=1)][:2])
    fin = np.isfinite(rs)
    assert (got_s[~fin] == rs[~fin]).all()                       # empty slots: -inf, or +inf for distances
    if fin.any():
        assert (np.abs(got_s - rs) / np.maximum(1.0, np.abs(rs)))[fin].max() < 1e-6
    return got_s, got_i


def cmax(ix):
    return struct.unpack("<f", struct.pack("<I", ix.info("cmax_bits")))[0]


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
def test_search_matches_oracle(bf, sim, cg, n, dim, nq, k):
    c = bf.synth_rows(1234, 0, n, dim)
    q = bf.synth_queries(4321, nq, dim, c)
    ix = index(sim, dim, n + 513)
    ix.append_bf16_bits(c)
    assert ix.info("similarity") == {"dotProduct": 1, "euclidean": 2}[sim]
    check(ix, q, c, k, cg)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_zero_rows_tombstones_ties_and_zero_query(bf, sim, cg):
    dim, n = 128, 1000
    c = bf.bf16_bits_to_f32(bf.synth_rows(5, 0, n, dim))
    c = bf.f32_to_bf16_bits(np.abs(c))                          # every entry >= 0 ...
    c[11] = 0; c[999] = 0; c[500] = 0                          # ... but three all-zero rows (live rows)
    c[700] = c[3]; c[701] = c[3]; c[2] = c[3]                  # exact duplicates
    q = bf.synth_queries(6, 20, dim, c)
    q[0] = c[3]
    q[1] = 0                                                   # all-zero query
    q[2] = bf.f32_to_bf16_bits(-np.abs(bf.bf16_bits_to_f32(q[2])) - 0.01)   # <q,c> < 0 for every nonzero row
    ix = index(sim, dim, 2048, max_batch=128)
    ix.append_bf16_bits(c)
    ix.delete_rows([40, 41, 999])                              # tombstones, one of them a zero row
    live = np.ones(n, bool)
    live[[40, 41, 999]] = False
    s, i = check(ix, q, c, 10, cg, live=live)
    assert not np.isin(i, [40, 41, 999]).any()
    if sim == "dotProduct":
        assert i[2, :2].tolist() == [11, 500] and (s[2, :2] == 0).all()    # zero rows first, lowest row first
        assert i[1].tolist() == [r for r in range(12) if r not in (40, 41)][:10] and (s[1] == 0).all()
    else:
        assert i[0, :3].tolist() == [2, 3, 700] and (s[0, :3] == 0).all()
        assert set(i[1, :2].tolist()) == {11, 500}                       # zero query: zero rows at distance 0
    # corpus shorter than k: the empty slots hold the worst value
    ix2 = index(sim, dim, 256, max_batch=128)
    ix2.append_bf16_bits(c[:12])
    s2, i2 = check(ix2, q[:5], c[:12], 20, cg)
    assert (i2[:, 12:] == -1).all()
    assert (s2[:, 12:] == (np.inf if sim == "euclidean" else -np.inf)).all()
    ix.close(); ix2.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_one_tile_crowd_of_near_duplicates_is_exact(bf, sim, cg):
    n, dim, nq = 3000, 1536, 70
    c = bf.synth_rows(1234, 0, n, dim)
    for j in range(24):
        c[1000 + j] = c[123]
        c[1000 + j, 7 + 61 * j] ^= np.uint16(1)
    c[2000:2600] = c[77]                                       # 600 exact duplicates
    q = bf.synth_queries(4321, nq, dim, c)
    base = bf.bf16_bits_to_f32(c[123])
    q[0] = bf.f32_to_bf16_bits(base + np.float32(0.1 * np.abs(base).mean()) *
                               np.random.default_rng(99).standard_normal(dim).astype(np.float32))
    q[1] = c[77]
    ix = index(sim, dim, 4096, max_batch=128)
    ix.append_bf16_bits(c)
    for k in (10, 12):
        check(ix, q, c, k, cg)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_exact_fallback_scan_alone_reproduces_the_oracle(bf, sim):
    n, dim, nq, k = 9000, 256, 150, 10
    c = bf.synth_rows(8, 0, n, dim)
    c[5] = 0
    q = bf.synth_queries(9, nq, dim, c)
    ix = index(sim, dim, n)
    ix.append_bf16_bits(c)
    ix.delete_rows([17, 18])
    live = np.ones(n, bool)
    live[[17, 18]] = False
    ix.set_option("force_fix", 1)
    ix.set_option("count_fix", 1)
    for cg in (1, 2):
        check(ix, q, c, k, cg, live=live)
        assert ix.info("last_fix_entries") > 0
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_scan_error_is_inside_the_bound(bf, sim, cg):
    """The certificate's bound for the new similarities depends on the rows' norms (DESIGN.md section 4.2).  Rows span
    2^-8 .. 2^8 in norm with heavy cancellation; the scan's value is rebuilt from the raw accumulators exactly as the
    epilogue forms it (one fp32 op with the row term) and compared with the exact value in the same units."""
    dim, n, nq = 1536, 512, 128 * cg
    g = np.random.default_rng(17)
    cf = g.standard_normal((n, dim)).astype(np.float32)
    cf /= np.linalg.norm(cf, axis=1, keepdims=True)
    cf *= np.exp2(g.uniform(-8, 8, (n, 1))).astype(np.float32)
    cf[: n // 4] = np.abs(cf[: n // 4])                                          # all-positive products
    qf = g.standard_normal((nq, dim)).astype(np.float32) * np.exp2(g.uniform(-4, 4, (nq, 1))).astype(np.float32)
    qf[: nq // 4] = np.abs(qf[: nq // 4]) * np.exp(g.uniform(-4, 4, (nq // 4, dim))).astype(np.float32)
    c, q = bf.f32_to_bf16_bits(cf), bf.f32_to_bf16_bits(qf)
    ix = index(sim, dim, n, max_batch=nq, max_k=10)
    ix.append_bf16_bits(c)
    eps_rel = ix.info("eps_rel_e12") * 1e-12
    cd, qd = bf.bf16_bits_to_f32(c).astype(np.float64), bf.bf16_bits_to_f32(q).astype(np.float64)
    norms = np.linalg.norm(cd, axis=1)
    cm = cmax(ix)
    assert cm >= norms.max() and cm <= norms.max() * (1 + 1e-6)
    qq = (qd * qd).sum(axis=1)
    qn = np.sqrt(qq)
    if sim == "dotProduct":
        eps = eps_rel * qn * cm
    else:
        u = 2.0 ** -23
        eps = (eps_rel + u) * qn * cm + u * cm * cm + 2.0 ** -50 * qq
    w = ix.inv_norm[:n].cpu().numpy().astype(np.float32)
    worst = 0.0
    for tile in (0, 1):
        acc = ix.debug_tile_dots(dev(q), tile, cg).cpu().numpy()[:nq]
        rows = slice(tile * 256, tile * 256 + 256)
        dots = qd @ cd[rows].T
        if sim == "dotProduct":
            assert (w[rows] == 1.0).all()
            a = acc * w[rows][None, :]
            e = dots
        else:
            assert (w[rows] == ((cd[rows] ** 2).sum(axis=1) / 2).astype(np.float32)).all()
            a = acc - w[rows][None, :]                                           # one fp32 subtraction, as the epilogue
            e = dots - (cd[rows] ** 2).sum(axis=1)[None, :] / 2
        assert a.dtype == np.float32
        worst = max(worst, float((np.abs(a.astype(np.float64) - e) / eps[:, None]).max()))
    print(f"{sim} cg={cg}: worst |a - e| / eps = {worst:.3e} (margin {1 / worst:.0f}x)")
    assert worst < 1.0
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_streaming_a_much_longer_row_raises_the_bound(bf, sim):
    dim = 256
    c = bf.synth_rows(77, 0, 4000, dim)
    q = bf.synth_queries(78, 60, dim, c)
    ix = index(sim, dim, 8192, max_batch=128)
    ix.append_bf16_bits(c[:3000])
    check(ix, q, c[:3000], 10)
    before = cmax(ix)
    big = bf.bf16_bits_to_f32(c[3000:3001]) * np.float32(100 * before / np.linalg.norm(bf.bf16_bits_to_f32(c[3000])))
    c[3000] = bf.f32_to_bf16_bits(big)[0]
    q[5] = bf.f32_to_bf16_bits(big * np.float32(0.01))[0]
    ix.append_bf16_bits(c[3000:3001])                          # Cmax grows mid-stream
    assert cmax(ix) > 50 * before
    check(ix, q, c[:3001], 10)
    ix.append_bf16_bits(c[3001:])
    check(ix, q, c, 10)
    ix.reset()
    assert cmax(ix) == 0.0
    ix.append_bf16_bits(c[:500])
    check(ix, q, c[:500], 10)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_snapshot_restore_keeps_the_similarity_and_the_bound(bf, sim, tmp_path):
    dim, n = 128, 3000
    c = bf.synth_rows(3, 0, n, dim)
    q = bf.synth_queries(4, 40, dim, c)
    ix = index(sim, dim, 4096, max_batch=128)
    ix.append_bf16_bits(c)
    ix.delete_rows([7, 8])
    live = np.ones(n, bool)
    live[[7, 8]] = False
    ix.snapshot(str(tmp_path / "s"))
    z = np.load(str(tmp_path / "s.npz"))
    assert str(z["similarity"]) == sim
    ix2 = index(sim, dim, 4096, max_batch=128)
    assert ix2.restore(str(tmp_path / "s")) == n
    norms = np.linalg.norm(bf.bf16_bits_to_f32(c[live]).astype(np.float64), axis=1)
    assert norms.max() <= cmax(ix2) <= cmax(ix)
    check(ix2, q, c, 10, live=live)
    other = index("euclidean" if sim == "dotProduct" else "dotProduct", dim, 4096, max_batch=128)
    with pytest.raises(ValueError, match="similarity"):
        other.restore(str(tmp_path / "s"))
    for x in (ix, ix2, other):
        x.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_engine_reproduces_independent_fixtures(path, sim, cg):
    import torch
    z = np.load(path)
    k = int(z["k"])
    cb, qb = z["corpus_bits"], z["query_bits"]
    ix = index(sim, cb.shape[1], len(cb) + 256, max_batch=64, max_k=k)
    ix.append_bf16_bits(cb)
    ix.set_option("cta_group", cg)
    s, i = ix.search(dev(qb), k)
    torch.cuda.synchronize()
    key = "dot" if sim == "dotProduct" else "euclidean"
    assert (i.cpu().numpy() == z[f"{key}_idx"]).all()
    ref = z[f"{key}_score"]
    assert (np.abs(s.cpu().numpy() - ref) / np.maximum(1.0, np.abs(ref))).max() < 1e-6
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_host_submit_wait_and_fp32_ingest(bf, sim):
    import torch
    dim, n, nq, k = 768, 6000, 150, 10
    g = np.random.default_rng(3)
    cf = g.standard_normal((n, dim), dtype=np.float32) * np.exp(g.uniform(-1, 1, (n, 1))).astype(np.float32)
    qf = g.standard_normal((nq, dim), dtype=np.float32)
    c, q = bf.f32_to_bf16_bits(cf), bf.f32_to_bf16_bits(qf)
    ix = index(sim, dim, 8192, max_batch=256, max_k=k)
    ix.append(cf[:2500])                                       # host fp32
    ix.append(torch.from_numpy(cf[2500:]).cuda())              # device fp32
    assert (ix.rows[:n].view(torch.int16).cpu().numpy().view(np.uint16) == c).all()
    rs, ri = topk_f64(q, c, k, sim)
    ix.search_host_submit(qf[:70], k, 0)
    ix.search_host_submit(qf[70:], k, 1)
    s0, i0 = ix.search_host_wait(0)
    s1, i1 = ix.search_host_wait(1)
    assert (np.concatenate([i0, i1]) == ri).all()
    assert (np.abs(np.concatenate([s0, s1]) - rs) / np.maximum(1, np.abs(rs))).max() < 1e-6
    hs, hi = ix.search_host(qf, k)
    assert (hi == ri).all()
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_shard_merges_follow_the_similarity(bf, sim):
    """Row shards on one GPU: the packed exchange (sa_search_hits / sa_merge_hits) and the split merge order distances
    ascending, and equal the unsharded answer; a tie across shards goes to the lower global row."""
    import torch
    dim, n, nq, k = 256, 12000, 140, 10
    c = bf.synth_rows(31, 0, n, dim)
    c[9000] = c[10]
    q = bf.synth_queries(32, nq, dim, c)
    q[0] = c[10]
    cuts = [0, 2500, 6000, 9500, n]
    keep, ss, ii = [], [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        ix = index(sim, dim, b - a, max_batch=256, max_k=k)
        ix.append_bf16_bits(c[a:b])
        s, i, s64 = ix.search(dev(q), k, want_score64=True)
        ss.append(s64)
        ii.append(torch.where(i >= 0, i.to(torch.int64) + a, torch.full_like(i, -1, dtype=torch.int64)))
        keep.append(ix)
    rs, ri = topk_f64(q, c, k, sim)
    fs, fi = keep[0].merge_shards(torch.stack(ss), torch.stack(ii))
    hits = torch.stack([ix.search_hits(dev(q), k, a) for ix, a in zip(keep, cuts[:-1])])
    hs, hi = keep[0].merge_hits(hits)
    torch.cuda.synchronize()
    assert (fi.cpu().numpy() == ri).all() and torch.equal(hi, fi) and torch.equal(hs, fs)
    top = fi[0].tolist()
    assert 10 in top and top[top.index(10) + 1] == 9000        # duplicates on two shards: the lower global row first
    assert (np.abs(fs.cpu().numpy() - rs) / np.maximum(1, np.abs(rs))).max() < 1e-6
    for ix in keep:
        ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_two_gpu_merge_equals_the_unsharded_answer(bf, sim):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from qsa_b200.sharded import MultiGpuIndex
    dim, n, nq, k = 256, 8000, 100, 10
    c = bf.synth_rows(41, 0, n, dim)
    q = bf.synth_queries(42, nq, dim, c)
    mi = MultiGpuIndex(dim=dim, capacity_per_gpu=n, max_batch=128, max_k=k, n_gpus=2, similarity=sim)
    for lo in range(0, n, 1000):
        mi.append(bf.bf16_bits_to_f32(c[lo:lo + 1000]))
    s, rows = mi.search_host(bf.bf16_bits_to_f32(q), k)
    rs, ri = topk_f64(q, c, k, sim)
    assert (rows == ri).all()
    mi.close()


def test_sa_serve_euclidean_atlas_end_to_end(tmp_path, capsys):
    from qsa_b200.pipeline.serve import Codec
    from qsa_b200.transport.filelog import Consumer
    from scripts import lab2_publish_queries, publish_docs, sa_serve
    from test_cli_and_pipeline import write_docs
    docs, logd = tmp_path / "docs", str(tmp_path / "topics")
    write_docs(docs, 40)
    assert publish_docs.main(["--docs-dir", str(docs), "--log-dir", logd]) == 0
    assert lab2_publish_queries.main(["How do tumble windows work?", "--log-dir", logd]) == 0
    capsys.readouterr()
    assert sa_serve.main(["--log-dir", logd, "--once", "--capacity", "1024", "--max-batch", "64", "--k", "3",
                          "--similarity", "euclidean", "--score-mode", "atlas", "--snapshot-dir", str(tmp_path / "ck")]) == 0
    stats = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert stats["documents"] == 41 and stats["searches"] == 1 and stats["quarantined"] == 0
    c = Consumer({"log.dir": logd, "group.id": "t"})
    c.subscribe(["search_results"])
    row = Codec(logd).decode(c.consume(1, 0.0)[0].value())
    sc = [row[f"score_{j}"] for j in (1, 2, 3)]
    assert all(0 < s <= 1 for s in sc) and sc[0] >= sc[1] >= sc[2]          # 1 / (1 + d), best first
    assert json.load(open(tmp_path / "ck" / "manifest.json"))["similarity"] == "euclidean"
    with pytest.raises(ValueError, match="similarity"):                         # a cosine restart refuses the checkpoint
        sa_serve.main(["--log-dir", logd, "--once", "--capacity", "1024", "--max-batch", "64", "--k", "3",
                       "--snapshot-dir", str(tmp_path / "ck")])
