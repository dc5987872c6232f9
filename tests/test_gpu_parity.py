"""Parity tests proper: the CUDA path, called through the C ABI (ctypes), against the CPU oracle on the same
seeded inputs.  Index lists must be equal element for element (integer work: bit-exact); scores are float32
roundings of float64 cosines and must agree within 1e-6 (north_star allows 1e-3).

Run on an H100 with:  python -m pytest tests -m gpu
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SCORE_TOL = 1e-6


def dev(bits):
    import torch
    return torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(torch.bfloat16).cuda()


def check(ix, q_bits, c_bits, k, cg=None):
    import torch
    from oracle import bruteforce as bf
    if cg is not None:
        ix.set_option("cta_group", cg)
    s, i = ix.search(dev(q_bits), k)
    torch.cuda.synchronize()
    rs, ri = bf.cosine_topk_f64(q_bits, c_bits, k)
    got_i, got_s = i.cpu().numpy(), s.cpu().numpy()
    assert (got_i == ri).all(), bf.compare_topk(got_i, got_s, ri, rs)
    fin = np.isfinite(rs)
    assert (np.isneginf(got_s) == ~fin).all()
    if fin.any():
        assert np.abs(got_s.astype(np.float64) - rs)[fin].max() < SCORE_TOL
    return got_s, got_i


@pytest.fixture(scope="module")
def bf():
    from oracle import bruteforce
    return bruteforce


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("n,dim,nq,k", [
    (20000, 1536, 200, 10),    # Lab2 shape: ragged last query block, 79 tiles (last one partial)
    (5000, 768, 37, 5),        # config-5 shape (768-d, top-5)
    (256, 64, 1, 1),           # one tile, one query
    (257, 128, 129, 3),        # one row into the second tile; one query into the second block
    (70000, 256, 300, 12),     # more tiles than tile lanes
    (70000, 256, 300, 16),     # k == the 16-entry list length: every spare entry gone, still exact (certificate)
    (2000, 256, 40, 16),       # ... with very few rows per lane (the fallback scan does the work)
    (9000, 192, 64, 28),       # 32-entry candidate lists, SA_MAX_K
])
def test_search_matches_oracle(bf, cg, n, dim, nq, k):
    from qsa_b200.engine import VectorIndex
    c = bf.synth_rows(1234, 0, n, dim)
    q = bf.synth_queries(4321, nq, dim, c)
    ix = VectorIndex(dim=dim, capacity=n + 513, max_batch=512, max_k=28)
    ix.append_bf16_bits(c)
    check(ix, q, c, k, cg)
    ix.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_ties_zero_rows_zero_queries_and_short_corpus(bf, cg):
    from qsa_b200.engine import VectorIndex
    dim, n = 128, 1000
    c = bf.synth_rows(5, 0, n, dim)
    c[700] = c[3]; c[701] = c[3]; c[2] = c[3]      # exact duplicates -> ties broken by ascending row
    c[11] = 0; c[999] = 0                          # all-zero rows are never returned
    c[500] = bf.f32_to_bf16_bits(bf.bf16_bits_to_f32(c[40]) * 2)   # scaled copy: same cosine as row 40
    q = bf.synth_queries(6, 20, dim, c)
    q[0] = c[3]
    q[1] = c[40]
    q[2] = 0                                       # all-zero query: score 0 everywhere, lowest rows win
    ix = VectorIndex(dim=dim, capacity=2048, max_batch=128, max_k=28)
    ix.append_bf16_bits(c)
    s, i = check(ix, q, c, 10, cg)
    assert i[0, :4].tolist() == [2, 3, 700, 701]
    assert set(i[1, :2].tolist()) == {40, 500} and i[1, 0] == 40
    assert i[2].tolist() == [0, 1, 2, 3, 4, 5, 6, 7, 8, 9] and (s[2] == 0).all()
    # corpus shorter than k: unused slots are (-inf, -1)
    ix2 = VectorIndex(dim=dim, capacity=256, max_batch=128, max_k=28)
    ix2.append_bf16_bits(c[:12])                   # 11 eligible rows (row 11 is zero)
    s2, i2 = check(ix2, q[:5], c[:12], 20, cg)
    assert (i2[:, 11:] == -1).all()
    ix.close(); ix2.close()


def test_empty_corpus_returns_no_rows(bf):
    import torch
    from qsa_b200.engine import VectorIndex
    ix = VectorIndex(dim=64, capacity=512, max_batch=128, max_k=10)
    q = bf.synth_rows(1, 0, 3, 64)
    s, i = ix.search(dev(q), 4)
    torch.cuda.synchronize()
    assert (i.cpu().numpy() == -1).all() and np.isneginf(s.cpu().numpy()).all()
    ix.close()


def test_streaming_epochs_search_sees_committed_prefix(bf):
    """Append-while-serving (LAB2-Walkthrough.md:41-51 ingest half): every search sees exactly the committed
    prefix; rows written but not yet committed are invisible; reset() empties the index."""
    from qsa_b200.engine import VectorIndex
    dim = 256
    c = bf.synth_rows(77, 0, 3000, dim)
    q = bf.synth_queries(78, 50, dim, c)
    ix = VectorIndex(dim=dim, capacity=4096, max_batch=128, max_k=10)
    import torch
    ix.rows[:3000].copy_(dev(c))                   # all bytes are already in HBM ...
    done = 0
    for step in (300, 212, 1, 999, 1488):          # ... but only committed rows may be returned
        ix.commit(done, step)
        done += step
        assert len(ix) == done
        check(ix, q, c[:done], 10)
    ix.reset()
    assert len(ix) == 0
    ix.append_bf16_bits(c[:100])
    check(ix, q[:7], c[:100], 10)
    ix.close()


def test_fp32_ingest_and_host_path_round_like_the_oracle(bf):
    """fp32 embeddings (ARRAY<FLOAT>, main.tf:141,215) are rounded to bf16 (RNE) on the device exactly as the
    oracle rounds them; sa_search_host (host buffers) equals the device path."""
    import torch
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 1536, 6000, 150, 10
    g = np.random.default_rng(3)
    cf = g.standard_normal((n, dim), dtype=np.float32) * np.exp(g.uniform(-1, 1, (n, 1))).astype(np.float32)
    qf = g.standard_normal((nq, dim), dtype=np.float32)
    qf[1::2] = cf[(np.arange(1, nq, 2) * 37) % n] + 0.3 * g.standard_normal((nq // 2, dim), dtype=np.float32)
    c, q = bf.f32_to_bf16_bits(cf), bf.f32_to_bf16_bits(qf)
    ix = VectorIndex(dim=dim, capacity=8192, max_batch=256, max_k=10)
    ix.append(cf[:2500])                           # host fp32 -> pinned staging -> device convert
    ix.append(torch.from_numpy(cf[2500:]).cuda())  # device fp32
    assert (ix.rows[:n].view(torch.int16).cpu().numpy().view(np.uint16) == c).all()
    rs, ri = bf.cosine_topk_f64(q, c, k)
    s, i = ix.search(torch.from_numpy(qf).cuda(), k)     # fp32 device queries
    torch.cuda.synchronize()
    assert (i.cpu().numpy() == ri).all()
    hs, hi = ix.search_host(qf, k)                       # host fp32 queries, host results
    assert (hi == ri).all() and np.abs(hs.astype(np.float64) - rs).max() < SCORE_TOL
    t = ix.last_timing()
    assert t.launches >= 1 and t.kernels >= 3 and t.scan_ms > 0 and t.flops == 2.0 * nq * n * dim
    ix.close()


def test_batch_larger_than_one_launch_and_launch_split(bf):
    """Batches beyond one wave of query blocks are split into several scan launches; forcing small launches
    must not change the answer."""
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 128, 30000, 1100, 10
    c = bf.synth_rows(21, 0, n, dim)
    q = bf.synth_queries(22, nq, dim, c)
    ix = VectorIndex(dim=dim, capacity=n, max_batch=2048, max_k=10)
    ix.append_bf16_bits(c)
    for cg in (1, 2):
        check(ix, q, c, k, cg)
    ix.set_option("max_launch_qblocks", 2)
    for cg in (1, 2):
        check(ix, q, c, k, cg)
    assert ix.last_timing().launches == 3          # 1100 queries / (2 pair blocks x 256)
    ix.close()


def test_merge_shards_equals_global(bf):
    """Row-sharded search on one GPU (4 engines), device merge kernel vs the unsharded oracle."""
    import torch
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 256, 12000, 140, 10
    c = bf.synth_rows(31, 0, n, dim)
    c[9000] = c[10]                                # a tie across shards: the lower global row must win
    q = bf.synth_queries(32, nq, dim, c)
    q[0] = c[10]
    cuts = [0, 2500, 6000, 9500, n]
    ss, ii = [], []
    keep = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        ix = VectorIndex(dim=dim, capacity=b - a, max_batch=256, max_k=10)
        ix.append_bf16_bits(c[a:b])
        s, i, s64 = ix.search(dev(q), k, want_score64=True)
        ss.append(s64)
        ii.append(torch.where(i >= 0, i.to(torch.int64) + a, torch.full_like(i, -1, dtype=torch.int64)))
        keep.append(ix)
    fs, fi = keep[0].merge_shards(torch.stack(ss), torch.stack(ii))
    torch.cuda.synchronize()
    rs, ri = bf.cosine_topk_f64(q, c, k)
    assert (fi.cpu().numpy() == ri).all()
    assert fi[0, 0].item() == 10 and fi[0, 1].item() == 9000
    # the exchange format of the sharded path (sa_search_hits / sa_merge_hits): one packed buffer per shard
    hits = torch.stack([ix.search_hits(dev(q), k, a) for ix, a in zip(keep, cuts[:-1])])
    hs, hi = keep[0].merge_hits(hits)
    torch.cuda.synchronize()
    assert torch.equal(hi, fi) and torch.equal(hs, fs)
    assert np.abs(fs.cpu().numpy().astype(np.float64) - rs).max() < SCORE_TOL
    for ix in keep:
        ix.close()


def test_full_size_properties_1M(bf):
    """Config 2 scale (1M x 1536, batch 256, top-10) through size-independent properties:
    planted queries return their planted row first; results are sorted; a sample of queries is checked against
    the oracle over all rows; searching the two halves and merging equals searching the whole."""
    import torch
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 1536, 1_000_000, 256, 10
    ix = VectorIndex(dim=dim, capacity=n, max_batch=256, max_k=10)
    chunks = []
    for ci in range((n + bf.CHUNK_ROWS - 1) // bf.CHUNK_ROWS):
        m = min(bf.CHUNK_ROWS, n - ci * bf.CHUNK_ROWS)
        bits = bf.synth_rows(1234, ci, m, dim)
        ix.append_bf16_bits(bits)
        chunks.append((ci * bf.CHUNK_ROWS, bits))
    q = bf.synth_queries(4321, nq, dim, chunks[0][1])
    s, i, s64 = ix.search(dev(q), k, want_score64=True)
    torch.cuda.synchronize()
    gi, gs = i.cpu().numpy(), s.cpu().numpy()
    for r in range(1, nq, 2):
        assert gi[r, 0] == bf.planted_row(r, len(chunks[0][1]))
    assert (np.diff(s64.cpu().numpy(), axis=1) <= 0).all()
    assert (gi >= 0).all() and all(len(set(row)) == k for row in gi.tolist())
    sample = np.arange(0, nq, 16)
    rs, ri = bf.cosine_topk_fast(q[sample], chunks, k)
    assert (gi[sample] == ri).all()
    assert np.abs(gs[sample].astype(np.float64) - rs).max() < SCORE_TOL
    ix.close()


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("n,dim,nq,k", [
    (30000, 128, 1100, 10),     # several launches / odd number of query blocks
    (70000, 256, 512, 12),      # exactly two pair blocks
    (5000, 1536, 300, 3),       # ragged batch, few tiles
    (9000, 192, 64, 28),        # 32-entry lists
])
def test_exact_fallback_scan_alone_reproduces_the_oracle(bf, cg, n, dim, nq, k):
    """force_fix = 1 routes EVERY (query, tile lane) through the fallback scan (sa_fixup_kernel): CUDA-core prefilter,
    float64 re-scoring, locked insertion into the result lists.  Its answer must equal the oracle's on its own, with
    duplicates (rows the merge kernel already re-scored) skipped, and the normal path must agree with it."""
    from qsa_b200.engine import VectorIndex
    c = bf.synth_rows(71, 0, n, dim)
    c[n // 2] = c[9]
    c[17] = 0
    q = bf.synth_queries(72, nq, dim, c)
    q[0] = c[9]
    ix = VectorIndex(dim=dim, capacity=n, max_batch=2048, max_k=28)
    ix.append_bf16_bits(c)
    ix.set_option("count_fix", 1)
    check(ix, q, c, k, cg)
    assert ix.info("last_fix_entries") == 0          # iid data: the certificate holds for every query
    ix.set_option("force_fix", 1)
    check(ix, q, c, k, cg)
    assert ix.info("last_fix_entries") > 0
    ix.set_option("unit_map", 1)
    check(ix, q, c, k, cg)
    ix.set_option("force_fix", 0)
    check(ix, q, c, k, cg)                            # scratch was left clean by the fallback run
    assert ix.info("last_fix_entries") == 0
    ix.close()


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("k", [10, 12])
def test_one_tile_crowd_of_near_duplicates_is_exact(bf, cg, k):
    """The case round 1 lost (VERDICT r01, weak #1b): 24 one-ulp variants of one row stored in CONSECUTIVE rows -- one
    256-row tile, hence one tile lane -- as consecutively ingested near-duplicate chunks are.  Their cosines differ by
    ~1e-8..1e-6, below the scan's fp32 resolution, and a 16-entry lane list cannot hold them all: the lane's dropped
    bound lands inside the certificate's band, the query goes to the exact fallback scan of that lane, and the answer
    is the brute-force one."""
    from qsa_b200.engine import VectorIndex
    dim, n = 1536, 40000
    c = bf.synth_rows(61, 0, n, dim)
    g = np.random.default_rng(62)
    base = c[123].copy()
    first = 5000 + 7                                           # rows 5007 .. 5030: inside tile 19
    assert first // 256 == (first + 23) // 256
    for j in range(24):
        row = base.copy()
        col = 7 + 61 * j
        row[col] = np.uint16(int(row[col]) + (1 if j % 2 else -1))   # one ulp up or down in one coordinate
        c[first + j] = row
    q = bf.synth_queries(63, 8, dim, c)
    bf32 = bf.bf16_bits_to_f32(base)
    for r in (0, 1):     # queries NEAR the crowd (not on it: at the exact maximum the differences are second order)
        q[r] = bf.f32_to_bf16_bits(bf32 + np.float32(0.1 * np.abs(bf32).mean()) * g.standard_normal(dim).astype(np.float32))
    rs, ri = bf.cosine_topk_f64(q[:2], c, 25)
    gaps = np.abs(np.diff(rs, axis=1))
    assert gaps.min() > 1e-13 and np.median(gaps) < 1e-7     # resolvable in float64, far below fp32 resolution
    s3, i3 = bf.cosine_topk_sgemm(q[:2], [(0, c)], k)
    assert (i3 != ri[:, :k]).any()                             # an fp32-only ranking really does get this wrong
    ix = VectorIndex(dim=dim, capacity=n, max_batch=128, max_k=28)
    ix.append_bf16_bits(c)
    ix.set_option("count_fix", 1)
    s, i = check(ix, q, c, k, cg)
    assert ix.info("last_fix_entries") >= 2                    # the two crowd queries were certified ambiguous ...
    assert set(i[0]).issubset(set(range(first, first + 24)) | {123})
    ix.set_option("share_thresholds", 0)
    check(ix, q, c, k, cg)
    ix.set_option("share_thresholds", 1)
    check(ix, q, c, 20, cg)                                    # 32-entry lists hold the whole crowd
    # 600 exact copies of one row spread over three tiles: more near-ties than any list or re-scoring set holds;
    # ties must resolve to the lowest rows
    c2 = c.copy()
    c2[20000:20600] = base
    ix2 = VectorIndex(dim=dim, capacity=n, max_batch=128, max_k=28)
    ix2.append_bf16_bits(c2)
    s2, i2 = check(ix2, q, c2, k, cg)
    qq = q.copy(); qq[0] = base
    s2, i2 = check(ix2, qq, c2, k, cg)
    assert i2[0, 0] == 123 and i2[0, 1:].tolist() == list(range(20000, 20000 + k - 1))
    ix.close(); ix2.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_scan_error_is_inside_eps(bf, cg):
    """The certificate rests on |a - e| <= eps_rel * |q| for the scan's approximate score.  Measure it on inputs built to
    maximise fp32 accumulation error (all-positive products, wide dynamic range, large magnitudes first) through the
    raw-accumulator test hook, and require a 10x margin."""
    import torch
    from qsa_b200.engine import VectorIndex
    dim, n, nq = 1536, 512, 128 * cg
    g = np.random.default_rng(7)
    cf = np.abs(g.standard_normal((n, dim)).astype(np.float32)) * np.exp(g.uniform(-6, 6, (n, dim))).astype(np.float32)
    qf = np.abs(g.standard_normal((nq, dim)).astype(np.float32)) * np.exp(g.uniform(-6, 6, (nq, dim))).astype(np.float32)
    cf[: n // 2] = -np.sort(-cf[: n // 2], axis=1)             # descending magnitudes: late small terms get absorbed
    cf[n // 2:] *= g.choice([-1.0, 1.0], (n - n // 2, dim)).astype(np.float32)   # and heavy cancellation
    c, q = bf.f32_to_bf16_bits(cf), bf.f32_to_bf16_bits(qf)
    ix = VectorIndex(dim=dim, capacity=n, max_batch=nq, max_k=10)
    ix.append_bf16_bits(c)
    eps_rel = ix.info("eps_rel_e12") * 1e-12
    assert 1.5e-4 < eps_rel < 2.5e-4
    worst = 0.0
    cd, qd = bf.bf16_bits_to_f32(c).astype(np.float64), bf.bf16_bits_to_f32(q).astype(np.float64)
    inv = ix.inv_norm[:n].cpu().numpy().astype(np.float32)
    for tile in (0, 1):
        dots = ix.debug_tile_dots(dev(q), tile, cg).cpu().numpy()[:nq]
        rows = slice(tile * 256, tile * 256 + 256)
        a = dots * inv[rows][None, :]                                              # the scan's approximate score
        e = (qd @ cd[rows].T) / np.linalg.norm(cd[rows], axis=1)[None, :]          # exact, same units
        worst = max(worst, float((np.abs(a - e) / np.linalg.norm(qd, axis=1)[:, None]).max()))
    assert worst < eps_rel / 10, (worst, eps_rel)
    ix.close()


def test_scan_profile_counters(bf):
    """The profiling build of the scan reports where each role spent its cycles (tools/gpu_prof.py prints them)."""
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 768, 50000, 128, 5
    c = bf.synth_rows(5678, 0, n, dim)
    q = bf.synth_queries(8765, nq, dim, c)
    ix = VectorIndex(dim=dim, capacity=n, max_batch=nq, max_k=k)
    ix.append_bf16_bits(c)
    ix.set_option("profile", 1)
    check(ix, q, c, k)
    p = ix.scan_profile()
    grid = ix.info("last_grid")
    assert len(p["total"]) == grid and (p["total"] > 0).all()
    assert p["tiles"].sum() == (n + 255) // 256
    assert ((p["epi_busy"] > 0) | (p["tiles"] == 0)).all() and (p["epi_busy"] <= p["total"]).all()
    ix.set_option("profile", 0)
    check(ix, q, c, k)
    ix.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_sampling_prepass_keeps_answers_and_tames_an_ascending_corpus(bf, cg):
    """Option "presample": a pre-pass over every S-th tile seeds the shared thresholds.  It may only move work around; and
    on a corpus stored in ASCENDING order of similarity to the queries -- where without it every tile brings rows that
    beat everything seen before -- it keeps the scan's time near the random-order time."""
    import torch
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 64, 520_000, 300, 10          # 2032 tiles: enough for a stride-8 sample on 49 (37) tile lanes
    g = np.random.default_rng(5)
    centre = g.standard_normal(dim).astype(np.float32)
    cf = g.standard_normal((n, dim)).astype(np.float32)
    order = np.argsort(cf @ centre / np.linalg.norm(cf, axis=1))
    qf = centre[None, :] + 0.3 * g.standard_normal((nq, dim)).astype(np.float32)
    q = bf.f32_to_bf16_bits(qf)
    times = {}
    for name, rows in (("random", cf), ("ascending", cf[order])):
        c = bf.f32_to_bf16_bits(rows)
        ix = VectorIndex(dim=dim, capacity=n, max_batch=512, max_k=k)
        ix.append_bf16_bits(c)
        ix.set_option("cta_group", cg)
        rs, ri = bf.cosine_topk_fast(q[:40], [(0, c)], k)
        # the pre-pass is measured against the plain shared threshold (the window bound, which also softens this
        # case, switched off); "wb" = the default configuration, no pre-pass
        for ps in (0, 2, 8, "wb"):
            ix.set_option("presample", 0 if ps == "wb" else ps)
            ix.set_option("window_bound", 1 if ps == "wb" else 0)
            s, i = ix.search(dev(q), k)
            torch.cuda.synchronize()
            assert (i.cpu().numpy()[:40] == ri).all(), (name, ps)
            for _ in range(5):
                ix.search(dev(q), k)
            torch.cuda.synchronize()
            times[(name, ps)] = ix.timing_mean(5)[1]
        ix.close()
    assert times[("ascending", 8)] < 0.7 * times[("ascending", 0)], times      # the pre-pass removes the blow-up ...
    assert times[("ascending", 8)] < 2.5 * times[("random", 0)], times         # ... to ~1.7x the random order (measured; slack for clocks)
    assert times[("ascending", "wb")] < 1.1 * times[("ascending", 0)], times   # the window bound never makes it worse


def test_drift_control_and_mapping_options_do_not_change_answers(bf):
    """Pacing, unit mapping and CTA grouping only move work around in time and space."""
    from qsa_b200.engine import VectorIndex
    dim, n, nq, k = 128, 60000, 700, 10
    c = bf.synth_rows(51, 0, n, dim)
    q = bf.synth_queries(52, nq, dim, c)
    ix = VectorIndex(dim=dim, capacity=n, max_batch=1024, max_k=10)
    ix.append_bf16_bits(c)
    for cg in (1, 2):
        for gain, drift, umap in ((0, 1, 0), (16, 1, 0), (64, 0, 1), (4096, 0, 0)):
            ix.set_option("pace_gain", gain); ix.set_option("max_drift", drift); ix.set_option("unit_map", umap)
            ix.set_option("window_bound", 0 if gain == 16 else 1)
            check(ix, q, c, k, cg)
    scan, total, m = ix.timing_mean(16)
    assert m == 8 and 0 < scan <= total
    ix.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_window_bound_with_ties_scattered_over_every_lane(bf, cg):
    """The window bound (kKL/2 lanes holding two rows >= x each) at its sharpest: exact copies of one row scattered over
    the whole corpus, so that most lanes' second best EQUALS the best score and the bound equals the score to keep.  Ties
    must still resolve to the lowest rows, for k up to the list length, on short scans (two tiles per lane) and long."""
    from qsa_b200.engine import VectorIndex
    dim = 256
    for n, every in ((132 * 256 * 2 + 77, 211), (200_000, 97)):   # two tiles per lane on 132 lanes, and long
        c = bf.synth_rows(71, 0, n, dim)
        base = c[5].copy()
        c[every::every] = base                                          # hundreds of copies, a few per lane
        q = bf.synth_queries(72, 100, dim, c)
        q[0] = base
        b32 = bf.bf16_bits_to_f32(base)
        g = np.random.default_rng(73)
        for r in range(1, 6):                                           # near the crowd: every copy ties exactly
            q[r] = bf.f32_to_bf16_bits(b32 + np.float32(0.2 * np.abs(b32).mean()) * g.standard_normal(dim).astype(np.float32))
        ix = VectorIndex(dim=dim, capacity=n, max_batch=128, max_k=28)
        ix.append_bf16_bits(c)
        for wb in (1, 0):
            ix.set_option("window_bound", wb)
            for k in (10, 16, 20):
                s, i = check(ix, q, c, k, cg)
                assert i[0, 0] == 5 and i[0, 1:].tolist() == [every * (j + 1) for j in range(k - 1)]
        ix.close()


def test_full_size_properties_10M(bf):
    """BASELINE.json's full size (10M x 1536 bf16, batch 1024, top-10) through size-independent properties:
    planted queries return their planted row first; scores are sorted and equal an independent float64 cosine of the
    returned rows; searching two row shards and merging equals searching the whole; batch position does not matter."""
    import torch
    from qsa_b200.engine import VectorIndex
    free, _ = torch.cuda.mem_get_info()
    if free < 70e9:
        pytest.skip("needs ~65 GB of free HBM")
    dim, n, nq, k = 1536, 10_000_000, 1024, 10
    ix = VectorIndex(dim=dim, capacity=n, max_batch=nq, max_k=k)
    g = torch.Generator(device="cuda").manual_seed(99)
    step = 1 << 18
    for lo in range(0, n, step):
        m = min(step, n - lo)
        x = torch.randn((m, dim), generator=g, device="cuda")
        x *= torch.exp(torch.empty((m, 1), device="cuda").uniform_(-0.7, 0.7, generator=g))
        ix.rows[lo:lo + m].copy_(x)
    ix.commit(0, n)
    planted = (torch.arange(nq, device="cuda", dtype=torch.int64) * 2654435761) % n
    q = torch.randn((nq, dim), generator=g, device="cuda")
    base = ix.rows[planted[1::2]].float()
    q[1::2] = base + 0.5 * base.norm(dim=1, keepdim=True) / dim ** 0.5 * torch.randn(base.shape, generator=g, device="cuda")
    q = q.to(torch.bfloat16)
    s, i, s64 = ix.search(q, k, want_score64=True)
    torch.cuda.synchronize()
    gi = i.cpu().numpy().astype(np.int64)
    assert (gi[1::2, 0] == planted[1::2].cpu().numpy()).all()                        # known neighbours come first
    s64c = s64.cpu().numpy()
    assert (np.diff(s64c, axis=1) <= 0).all() and (gi >= 0).all()
    assert all(len(set(r)) == k for r in gi.tolist())
    # returned scores == independent float64 cosine of the returned rows (a sample of queries, CPU arithmetic)
    for r in range(0, nq, 37):
        rows = bf.bf16_bits_to_f32(ix.rows[i[r].long()].view(torch.int16).cpu().numpy().view(np.uint16)).astype(np.float64)
        qq = bf.bf16_bits_to_f32(q[r:r + 1].view(torch.int16).cpu().numpy().view(np.uint16)).astype(np.float64)[0]
        cos = rows @ qq / np.sqrt((rows * rows).sum(1) * (qq * qq).sum())
        assert np.abs(cos - s64c[r]).max() < 1e-12 and np.abs(cos - s.cpu().numpy()[r]).max() < SCORE_TOL
    # a permutation of the batch permutes the answers (no cross-query leakage, launch split independent)
    perm = torch.randperm(nq, generator=torch.Generator().manual_seed(5))
    s2, i2 = ix.search(q[perm.cuda()], k)
    assert torch.equal(i2.cpu(), i.cpu()[perm])
    # shard-and-merge == whole (two row shards re-indexed on the same GPU)
    cut = 4_500_000
    parts = []
    for lo, hi in ((0, cut), (cut, n)):
        sub = VectorIndex(dim=dim, capacity=hi - lo, max_batch=256, max_k=k)
        sub.rows.copy_(ix.rows[lo:hi])
        sub.commit(0, hi - lo)
        ss, si, ss64 = sub.search(q[:256], k, want_score64=True)
        parts.append((ss64, torch.where(si >= 0, si.to(torch.int64) + lo, torch.full_like(si, -1, dtype=torch.int64)), sub))
    fs, fi = ix.merge_shards(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]))
    torch.cuda.synchronize()
    assert torch.equal(fi.cpu(), i[:256].cpu().to(torch.int64))
    for p in parts:
        p[2].close()
    ix.close()


def test_c_abi_error_behaviour_on_device(bf):
    """Error paths through the C ABI on a real device: codes and messages, no silent fallback, engine stays usable."""
    import ctypes as C
    import torch
    from qsa_b200 import capi
    from qsa_b200.engine import VectorIndex
    ix = VectorIndex(dim=128, capacity=1000, max_batch=64, max_k=10)
    c = bf.synth_rows(1, 0, 600, 128)
    ix.append_bf16_bits(c)
    lib = ix.lib
    q = dev(bf.synth_rows(2, 0, 64, 128))
    s = torch.empty((64, 10), dtype=torch.float32, device="cuda")
    i = torch.empty((64, 10), dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert lib.sa_search(ix._h, q.data_ptr(), 65, 10, s.data_ptr(), i.data_ptr(), None, st) == capi.SA_ERR_CAPACITY
    assert lib.sa_search(ix._h, q.data_ptr(), 64, 11, s.data_ptr(), i.data_ptr(), None, st) == capi.SA_ERR_ARG
    assert b"max_k" in lib.sa_last_error()
    assert lib.sa_search(ix._h, q.data_ptr() + 2, 8, 5, s.data_ptr(), i.data_ptr(), None, st) == capi.SA_ERR_ARG   # alignment
    assert lib.sa_search(ix._h, q.data_ptr(), 8, 5, None, i.data_ptr(), None, st) == capi.SA_ERR_ARG
    with pytest.raises(capi.SaError, match="capacity"):
        ix.append(np.zeros((500, 128), np.float32))                      # 600 + 500 > 1000
    assert lib.sa_corpus_commit(ix._h, 10, 5, st) == capi.SA_ERR_ARG     # commits must start at the row count
    with pytest.raises(capi.SaError):
        ix.set_option("cta_group", 3)
    with pytest.raises(capi.SaError):
        ix.set_option("no_such_option", 1)
    h = C.c_void_p()
    assert lib.sa_engine_create(C.byref(h), 99, 128, 1000, 64, 10) == capi.SA_ERR_ARG      # no such device
    unbound = C.c_void_p()
    assert lib.sa_engine_create(C.byref(unbound), 0, 128, 1000, 64, 10) == 0
    assert lib.sa_search(unbound, q.data_ptr(), 8, 5, s.data_ptr(), i.data_ptr(), None, st) == capi.SA_ERR_ARG
    assert b"sa_corpus_bind" in lib.sa_last_error()
    # every option takes both ends of its range and refuses one past each; a flag takes any value
    for name, lo, hi in (("cta_group", 0, 2), ("unit_map", 0, 1), ("wait_hint_ns", -1, 1_000_000),
                         ("presample", -1, 4096), ("pace_gain", -1, 4096), ("pace_max", -1, 65536),
                         ("max_drift", -1, 1024), ("max_launch_qblocks", 0, 2**31 - 1)):
        for v, rc in ((lo - 1, capi.SA_ERR_ARG), (lo, 0), (hi, 0), (hi + 1, capi.SA_ERR_ARG)):
            assert lib.sa_set_option(unbound, name.encode(), v) == rc, (name, v)
    assert lib.sa_set_option(unbound, b"max_launch_qblocks", 2**32) == capi.SA_ERR_ARG   # not wrapped to 0 ("no cap")
    for v, rc in ((0, 0), (16, 0), (32, 0), (-1, capi.SA_ERR_ARG), (15, capi.SA_ERR_ARG), (33, capi.SA_ERR_ARG)):
        assert lib.sa_set_option(unbound, b"list_len", v) == rc, ("list_len", v)
    for name in ("force_fix", "count_fix", "profile", "share_thresholds", "window_bound", "record_times"):
        for v in (0, 1, 7):
            assert lib.sa_set_option(unbound, name.encode(), v) == 0, (name, v)
    lib.sa_engine_destroy(unbound)
    check(ix, bf.synth_rows(2, 0, 64, 128), c, 10)                        # still healthy after all of that
    ix.close()
    # the profiling build of the scan has 16-entry lists only and no filtered or deep form: such searches are refused,
    # and the engine answers exactly once the option is off again
    deep = VectorIndex(dim=128, capacity=1000, max_batch=64, max_k=capi.SA_MAX_K)
    deep.append_bf16_bits(c)
    deep.set_option("profile", 1)
    for k, filters in ((20, None), (10, np.zeros(4, np.uint64)), (29, None)):
        with pytest.raises(capi.SaError) as err:
            deep.search(q, k, filters=filters)
        assert err.value.rc == capi.SA_ERR_ARG, (k, filters)
    deep.set_option("profile", 0)
    check(deep, bf.synth_rows(2, 0, 64, 128), c, 10)
    deep.close()


@pytest.mark.parametrize("cg", [1, 2])
def test_near_duplicate_cluster_does_not_break_exactness(bf, cg):
    """A crowd of rows that differ from the best match by one bf16 ulp in one coordinate, scattered over the corpus: their
    cosines are ~1e-6 apart -- the scale of the tensor-core scan's fp32 rounding -- so the scan alone cannot order them;
    the float64 re-scoring of the certificate's band candidates must."""
    from qsa_b200.engine import VectorIndex
    dim, n, k = 1536, 40000, 10
    c = bf.synth_rows(61, 0, n, dim)
    g = np.random.default_rng(62)
    base = c[123].copy()
    crowd = g.choice(np.arange(1000, n), size=24, replace=False)
    for j, r in enumerate(crowd):
        row = base.copy()
        col = 7 + 61 * j
        row[col] = np.uint16(int(row[col]) + (1 if j % 2 else -1))   # one ulp up or down in one coordinate
        c[r] = row
    q = bf.synth_queries(63, 8, dim, c)
    bf32 = bf.bf16_bits_to_f32(base)
    for r in (0, 1):     # queries NEAR the crowd (not on it: at the exact maximum the differences are second order)
        q[r] = bf.f32_to_bf16_bits(bf32 + np.float32(0.1 * np.abs(bf32).mean()) * g.standard_normal(dim).astype(np.float32))
    rs, ri = bf.cosine_topk_f64(q[:2], c, 25)
    gaps = np.abs(np.diff(rs, axis=1))
    assert gaps.min() > 1e-13 and np.median(gaps) < 1e-7     # resolvable in float64, far below fp32 resolution
    s3, i3 = bf.cosine_topk_sgemm(q[:2], [(0, c)], k)
    assert (i3 != ri[:, :k]).any()                             # an fp32-only ranking really does get this wrong
    ix = VectorIndex(dim=dim, capacity=n, max_batch=128, max_k=28)
    ix.append_bf16_bits(c)
    s, i = check(ix, q, c, k, cg)
    assert set(i[0]).issubset(set(crowd.tolist()) | {123})
    check(ix, q, c, 20, cg)                                  # 32-entry lists
    ix.close()


def test_host_slots_submit_wait(bf):
    """sa_search_host_submit / _wait: two batches in flight, results come back per slot in submission order, misuse
    is an error, and the blocking call still works in between."""
    from qsa_b200 import capi
    from qsa_b200.engine import VectorIndex
    dim, n, k = 256, 20000, 10
    c = bf.synth_rows(81, 0, n, dim)
    ix = VectorIndex(dim=dim, capacity=n, max_batch=300, max_k=10)
    ix.append_bf16_bits(c)
    batches = [bf.synth_queries(90 + j, nq, dim, c) for j, nq in enumerate((300, 17, 128, 256, 1))]
    refs = [bf.cosine_topk_f64(q, c, k) for q in batches]
    f32 = [bf.bf16_bits_to_f32(q) for q in batches]
    pinned = ix.pinned_array((300, dim), np.float32)
    got = {}
    ix.search_host_submit(f32[0], k, 0)
    for j in range(1, len(batches)):
        src = f32[j]
        if j == 2:                                   # a page-locked source is DMA'd in place
            pinned[:len(src)] = src
            src = pinned[:len(src)]
        ix.search_host_submit(src, k, j & 1)
        got[j - 1] = ix.search_host_wait((j - 1) & 1)
    got[len(batches) - 1] = ix.search_host_wait((len(batches) - 1) & 1)
    for j, (rs, ri) in enumerate(refs):
        assert (got[j][1] == ri).all() and np.abs(got[j][0].astype(np.float64) - rs).max() < SCORE_TOL
    ix.search_host_submit(f32[1], k, 0)
    with pytest.raises(capi.SaError, match="unwaited"):
        ix.lib and capi.check(ix.lib.sa_search_host_submit(ix._h, 0, f32[1].ctypes.data, 17, k), "submit")
    hs, hi = ix.search_host(f32[2], k)               # the blocking call has its own slot
    assert (hi == refs[2][1]).all()
    s0, i0 = ix.search_host_wait(0)
    assert (i0 == refs[1][1]).all()
    with pytest.raises(capi.SaError, match="no search in flight"):
        capi.check(ix.lib.sa_search_host_wait(ix._h, 1, hs.ctypes.data, hi.ctypes.data), "wait")
    with pytest.raises(capi.SaError):
        capi.check(ix.lib.sa_search_host_submit(ix._h, 2, f32[1].ctypes.data, 17, k), "submit")
    ix.close()


def test_index_snapshot_restore(bf, tmp_path):
    """Checkpoint / resume of the HBM half: a restored index answers exactly like the original, and keeps growing."""
    from qsa_b200.engine import VectorIndex
    dim, n = 192, 7000
    c = bf.synth_rows(95, 0, n, dim)
    q = bf.synth_queries(96, 50, dim, c)
    ix = VectorIndex(dim=dim, capacity=8000, max_batch=64, max_k=10)
    ix.append_bf16_bits(c[:6000])
    ix.delete_rows([5, 17])
    assert ix.snapshot(str(tmp_path / "index.npz")) == 6000
    ix2 = VectorIndex(dim=dim, capacity=8000, max_batch=64, max_k=10)
    assert ix2.restore(str(tmp_path / "index.npz")) == 6000 and len(ix2) == 6000
    ref = c[:6000].copy(); ref[[5, 17]] = 0
    check(ix2, q, ref, 10)
    ix2.append_bf16_bits(c[6000:])
    check(ix2, q, np.concatenate([ref, c[6000:]]), 10)
    with pytest.raises(ValueError):
        VectorIndex(dim=128, capacity=8000, max_batch=64, max_k=10).restore(str(tmp_path / "index.npz"))
    ix.close(); ix2.close()
