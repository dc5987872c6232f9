"""int8 indexes on the H100: the s8 wgmma scan, the int8 ingest, merge and fallback paths against the definition on the
integers (exact float64 sums of int8 products), and against a bf16 index holding the same integers, which must return
byte-identical results.

Run on an H100 with:  python -m pytest tests -m gpu
"""
import ctypes as C
import glob
import os
import struct

import numpy as np
import pytest

from harness.similarity_oracle import RunningTopk

pytestmark = pytest.mark.gpu

SIMS = ["cosine", "dotProduct", "euclidean"]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "int8_topk_independent_*.npz")))


def ref_topk(q, c, k, sim, ok=None):
    """The definition on int8 rows and queries: sums of int8 products in float64 are exact, then the engine's formulas
    (cosine dot / sqrt(|q|^2 |c|^2), dotProduct dot, euclidean sqrt((|q|^2 - 2 dot) + |c|^2)); all-zero rows are never
    returned under cosine; ok [nq, n] masks rows out (tombstones, filters).  (score f64 [nq, k], row i64 [nq, k])."""
    qf, cf = np.asarray(q, np.float64), np.asarray(c, np.float64)
    dots = qf @ cf.T
    qq, cc = (qf * qf).sum(axis=1), (cf * cf).sum(axis=1)
    if sim == "cosine":
        den = np.sqrt(qq[:, None] * cc[None, :])
        with np.errstate(divide="ignore", invalid="ignore"):
            s = np.where(den > 0, dots / den, 0.0)
        s[:, cc == 0] = -np.inf
    elif sim == "dotProduct":
        s = dots
    else:
        s = -np.sqrt(np.maximum((qq[:, None] - 2.0 * dots) + cc[None, :], 0.0))
    if ok is not None:
        s = np.where(ok, s, -np.inf)
    acc = RunningTopk(len(qf), k)
    acc.add(s, 0)
    return (-acc.s if sim == "euclidean" else acc.s), acc.i


def dev8(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.int8)).cuda()


def dev_bf16(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda().to(torch.bfloat16)


def index(sim, dim, capacity, max_batch=512, max_k=64, dtype="int8"):
    from qsa_b200.engine import VectorIndex
    return VectorIndex(dim=dim, capacity=capacity, max_batch=max_batch, max_k=max_k, similarity=sim, dtype=dtype)


def rows(seed, n, dim, lo=-128, hi=128):
    return np.random.default_rng(seed).integers(lo, hi, (n, dim)).astype(np.int8)


def queries(seed, nq, dim, c):
    """Random int8 queries, every other one planted next to a corpus row (top-k lists with real structure)."""
    g = np.random.default_rng(seed)
    q = g.integers(-128, 128, (nq, dim))
    pick = g.integers(0, len(c), nq)
    near = np.clip(c[pick].astype(np.int64) + g.integers(-20, 21, (nq, dim)), -128, 127)
    q[1::2] = near[1::2]
    return q.astype(np.int8)


def check(ix, q, c, k, cg=None, ok=None, filters=None):
    import torch
    if cg is not None:
        ix.set_option("cta_group", cg)
    s, i = ix.search(dev8(q), k, filters=filters)
    torch.cuda.synchronize()
    rs, ri = ref_topk(q, c, k, ix.similarity, ok)
    got_i, got_s = i.cpu().numpy(), s.cpu().numpy().astype(np.float64)
    bad = (got_i != ri).any(axis=1)
    assert not bad.any(), (np.flatnonzero(bad)[:8], got_i[bad][:2], ri[bad][:2])
    fin = np.isfinite(rs)
    assert (got_s[~fin] == rs[~fin]).all()                       # empty slots: -inf, or +inf for distances
    if fin.any():
        assert (np.abs(got_s[fin] - rs[fin]) / np.maximum(1.0, np.abs(rs[fin]))).max() < 1e-6
    return got_s, got_i


def cmax(ix):
    return struct.unpack("<f", struct.pack("<I", ix.info("cmax_bits")))[0]


# ------------------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("n,dim,nq,k", [
    (20000, 1536, 200, 10),
    (5000, 768, 37, 16),
    (257, 128, 129, 1),
    (40, 384, 20, 64),            # fewer rows than k
    (9000, 384, 64, 28),
    (3001, 768, 100, 29),         # a partial last tile
    (70000, 128, 300, 64),
    (2000, 1536, 130, 16),
])
def test_search_matches_the_definition(sim, cg, n, dim, nq, k):
    c = rows(1234 + dim, n, dim)
    q = queries(4321 + n, nq, dim, c)
    ix = index(sim, dim, n + 513)
    ix.append(c)
    assert ix.info("elem") == 1 and ix.dtype == "int8"
    s, i = check(ix, q, c, k, cg)
    if n < k:
        assert (i[:, n:] == -1).all() and (s[:, n:] == (np.inf if sim == "euclidean" else -np.inf)).all()
    ix.close()


# ---------------------------------------------------------------------------------- int8 index == bf16 index
def pair(sim, c, max_batch=256, max_k=64):
    """An int8 index and a bf16 index holding the same integer rows, with the same tags."""
    n, dim = c.shape
    tags = np.random.default_rng(n).integers(0, 1 << 16, n).astype(np.uint64)
    a = index(sim, dim, n, max_batch, max_k)
    b = index(sim, dim, n, max_batch, max_k, dtype="bfloat16")
    a.append(c, tags=tags)
    b.append(c.astype(np.float32), tags=tags)
    return a, b


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("k", [10, 64])
@pytest.mark.parametrize("filtered", [False, True])
def test_int8_index_equals_bf16_index_byte_for_byte(sim, k, filtered):
    import torch
    n, dim, nq = 12000, 768, 150
    c = rows(5, n, dim)
    c[100:140] = c[7]                                          # duplicates: ties
    q = queries(6, nq, dim, c)
    a, b = pair(sim, c)
    f = None
    if filtered:
        g = np.random.default_rng(1)
        f = np.zeros((nq, 4), np.uint64)
        f[:, 0] = np.uint64(1) << g.integers(0, 16, nq).astype(np.uint64)
    for cg in (1, 2):
        a.set_option("cta_group", cg)
        b.set_option("cta_group", cg)
        sa, ia, s64a = a.search(dev8(q), k, want_score64=True, filters=f)
        sb, ib, s64b = b.search(dev_bf16(q), k, want_score64=True, filters=f)
        torch.cuda.synchronize()
        assert torch.equal(ia, ib)
        assert sa.cpu().numpy().tobytes() == sb.cpu().numpy().tobytes()
        assert s64a.cpu().numpy().tobytes() == s64b.cpu().numpy().tobytes()
    qf = q.astype(np.float32)                                  # host forms: fp32 queries, converted by each index
    ha, hia = a.search_host(qf, k, filters=f)
    hb, hib = b.search_host(qf, k, filters=f)
    assert np.array_equal(hia, hib) and ha.tobytes() == hb.tobytes()
    assert np.array_equal(hia, ia.cpu().numpy())
    a.close(); b.close()


# ------------------------------------------------------------------------------------------------------ accumulators
@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_accumulators_are_exact_and_the_scan_error_is_inside_the_bound(sim, cg):
    """The debug dump of the s8 wgmma accumulators equals float32(exact integer dot) bit for bit, the extreme rows
    (dots beyond 2^24) included; the scan's value, rebuilt from them as the epilogue forms it, stays inside eps."""
    dim, n, nq = 1536, 512, 128 * cg
    g = np.random.default_rng(17)
    c = rows(18, n, dim)
    c[0], c[1], c[2], c[300] = -128, 127, 0, -128
    c[3:40] = g.integers(-3, 4, (37, dim))                     # short rows next to long ones
    c[40] = 127
    c[40, 0] = 126                                             # <q0, c40> is odd and above 2^24: fp32 rounds it
    q = rows(19, nq, dim)
    q[0], q[1], q[2] = 127, -128, 1
    ix = index(sim, dim, n, max_batch=nq, max_k=10)
    ix.append(c)
    eps_rel = ix.info("eps_rel_e12") * 1e-12
    assert eps_rel == pytest.approx(4 * 2.0 ** -23, rel=1e-6)
    cd, qd = c.astype(np.float64), q.astype(np.float64)
    cc = (cd * cd).sum(axis=1)
    cm = cmax(ix)
    assert cm >= np.sqrt(cc.max()) and cm <= np.sqrt(cc.max()) * (1 + 1e-6)
    qq = (qd * qd).sum(axis=1)
    qn = np.sqrt(qq)
    u = 2.0 ** -23
    eps = {"cosine": eps_rel * qn, "dotProduct": eps_rel * qn * cm,
           "euclidean": (eps_rel + u) * qn * cm + u * cm * cm + 2.0 ** -50 * qq}[sim]
    w = ix.inv_norm[:n].cpu().numpy().astype(np.float32)
    worst = 0.0
    for tile in (0, 1):
        acc = ix.debug_tile_dots(dev8(q), tile, cg).cpu().numpy()[:nq]
        r = slice(tile * 256, tile * 256 + 256)
        dots = q.astype(np.int64) @ c[r].astype(np.int64).T
        assert acc.view(np.uint32).tobytes() == dots.astype(np.float32).view(np.uint32).tobytes()
        if tile == 0:
            assert dots[0, 1] == 1536 * 127 * 127 and dots[1, 0] == 1536 * 128 * 128 > 2 ** 24
        live = cc[r] > 0
        if sim == "euclidean":
            assert (w[r] == (cc[r] / 2).astype(np.float32)).all()
            a, e = acc - w[r][None, :], dots - cc[r][None, :] / 2
        else:
            want_w = np.where(live, (1.0 / np.sqrt(np.where(live, cc[r], 1.0))), 0.0).astype(np.float32) \
                if sim == "cosine" else np.ones(256, np.float32)
            assert (w[r] == want_w).all()
            a = acc * w[r][None, :]
            e = dots * (np.where(live, 1.0 / np.sqrt(np.where(live, cc[r], 1.0)), 0.0) if sim == "cosine" else 1.0)
        assert a.dtype == np.float32
        err = np.abs(a.astype(np.float64) - e)[:, live] / np.maximum(eps[:, None], 1e-300)
        err[np.broadcast_to(eps[:, None] == 0, err.shape)] = 0.0           # a zero query: a = e = 0
        worst = max(worst, float(err.max()))
    print(f"{sim} cg={cg}: worst |a - e| / eps = {worst:.3e} (margin {1 / max(worst, 1e-30):.0f}x)")
    assert worst < 1.0
    ix.close()


# ---------------------------------------------------------------------------------------------- ties and fallback
@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("k", [10, 64])
def test_permutation_crowd_over_many_lanes_returns_the_lowest_rows(sim, k):
    """200 permutations of one vector spread over many tiles: a constant query ties them exactly under every
    similarity, and they are its best rows, so the answer is the k lowest of them."""
    n, dim = 60000, 768
    g = np.random.default_rng(23)
    c = g.integers(-20, 21, (n, dim)).astype(np.int8)
    v = g.integers(60, 128, dim)
    at = np.sort(g.choice(n, 200, replace=False))
    c[at] = np.stack([g.permutation(v) for _ in range(200)]).astype(np.int8)
    q = np.full((2, dim), 127, np.int8)
    q[1] = 1 if sim != "euclidean" else 100
    ix = index(sim, dim, n)
    ix.append(c)
    for cg in (1, 2):
        _, i = check(ix, q, c, k, cg)
        assert i[0].tolist() == at[:k].tolist()
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
def test_duplicates_zero_rows_tombstones_and_zero_query(sim, cg):
    n, dim = 4000, 256
    c = rows(31, n, dim)
    c[2000:2600] = c[77]                                       # 600 exact duplicates
    c[11] = 0; c[3999] = 0; c[500] = 0                         # all-zero rows
    q = queries(32, 40, dim, c)
    q[0] = c[77]
    q[1] = 0                                                   # all-zero query
    ix = index(sim, dim, 4096, max_batch=128)
    ix.append(c)
    ix.delete_rows([40, 41, 3999, 2100])                       # tombstones, one a zero row, one a duplicate
    ok = np.ones((len(q), n), bool)
    ok[:, [40, 41, 3999, 2100]] = False
    for k in (10, 64):
        s, i = check(ix, q, c, k, cg, ok=ok)
        assert not np.isin(i, [40, 41, 3999, 2100]).any()
    if sim != "dotProduct":
        assert i[0, :3].tolist() == [77, 2000, 2001]           # cosine 1 / distance 0, lowest rows first
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_exact_fallback_scan_alone_reproduces_the_definition(sim):
    n, dim, nq = 9000, 384, 150
    c = rows(8, n, dim)
    c[5] = 0
    q = queries(9, nq, dim, c)
    ix = index(sim, dim, n)
    ix.append(c)
    ix.delete_rows([17, 18])
    ok = np.ones((nq, n), bool)
    ok[:, [17, 18]] = False
    ix.set_option("force_fix", 1)
    ix.set_option("count_fix", 1)
    for cg in (1, 2):
        for k in (10, 64):
            check(ix, q, c, k, cg, ok=ok)
            assert ix.info("last_fix_entries") > 0
    ix.close()


# ------------------------------------------------------------------------------------------------ filters, deep k
@pytest.mark.parametrize("sim", SIMS)
def test_filters_from_everything_to_almost_nothing(sim):
    """Selectivities 100 %, 10 %, 1 %, 0.1 %, exactly k eligible rows and fewer than k, shallow and deep k."""
    n, dim, nq = 40000, 256, 64
    g = np.random.default_rng(41)
    c = rows(42, n, dim)
    q = queries(43, nq, dim, c)
    u = g.random(n)
    tags = np.ones(n, np.uint64)                               # bit 0: every row
    tags |= (u < 0.1).astype(np.uint64) << np.uint64(1)
    tags |= (u < 0.01).astype(np.uint64) << np.uint64(2)
    tags |= (u < 0.001).astype(np.uint64) << np.uint64(3)
    ix = index(sim, dim, n, max_batch=nq)
    for k in (10, 64):
        t = tags.copy()
        t[g.choice(n, k, replace=False)] |= np.uint64(1) << np.uint64(4)        # exactly k rows
        t[g.choice(n, k - 3, replace=False)] |= np.uint64(1) << np.uint64(5)    # fewer than k rows
        ix.reset()
        ix.append(c, tags=t)
        f = np.zeros((nq, 4), np.uint64)
        f[:, 0] = np.uint64(1) << (np.arange(nq) % 6).astype(np.uint64)
        ok = (t[None, :] & f[:, 0:1]) == f[:, 0:1]
        for cg in (1, 2):
            s, i = check(ix, q, c, k, cg, ok=ok, filters=f)
            assert (i[4::6] >= 0).all() and (i[5::6, k - 3:] == -1).all()
    ix.close()


# ---------------------------------------------------------------------------------------------- ingest, snapshots
@pytest.mark.parametrize("sim", SIMS)
def test_fp32_ingest_and_queries_follow_the_int8_rule(sim):
    import torch
    n, dim, nq, k = 5000, 384, 100, 10
    g = np.random.default_rng(51)
    c = rows(52, n, dim)
    q = queries(53, nq, dim, c)
    ix = index(sim, dim, 2 * n, max_batch=nq)
    ix.append(c[:2000].astype(np.float32))                     # integer-valued floats: the int8 answer exactly
    ix.append(torch.from_numpy(c[2000:].astype(np.float32)).cuda())
    assert np.array_equal(ix.rows[:n].cpu().numpy(), c)
    s8, i8 = check(ix, q, c, k)
    sf, i_f = ix.search(torch.from_numpy(q.astype(np.float32)).cuda(), k)
    assert torch.equal(i_f.cpu(), torch.from_numpy(i8.astype(np.int32)))
    # non-integral and out-of-range floats: the answer for clip(rint(x))
    xf = (g.standard_normal((n, dim)) * 90).astype(np.float32)
    xf[:5, :3] = [[0.5, 1.5, -2.5]] * 5
    xf[7, 0], xf[8, 1] = 1e9, -np.inf
    qx = (g.standard_normal((nq, dim)) * 90).astype(np.float32)
    cx, qr = np.clip(np.rint(xf), -128, 127).astype(np.int8), np.clip(np.rint(qx), -128, 127).astype(np.int8)
    ix.reset()
    ix.append(torch.from_numpy(xf).cuda())
    assert np.array_equal(ix.rows[:n].cpu().numpy(), cx)
    ix.reset()
    ix.append(xf)
    assert np.array_equal(ix.rows[:n].cpu().numpy(), cx)
    sq, iq = ix.search(torch.from_numpy(qx).cuda(), k)
    torch.cuda.synchronize()
    rs, ri = ref_topk(qr, cx, k, sim)
    assert np.array_equal(iq.cpu().numpy(), ri)
    hs, hi = ix.search_host(qx, k)
    assert np.array_equal(hi, ri)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_streaming_commit_and_append_mid_stream(sim):
    n, dim, nq, k = 9000, 512, 60, 16
    c = rows(61, n, dim)
    q = queries(62, nq, dim, c)
    ix = index(sim, dim, n, max_batch=nq)
    cuts = [0, 1, 300, 2600, 2601, 7000, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        if a % 2:
            ix.rows[a:b].copy_(dev8(c[a:b]))                   # written in place, then committed
            ix.commit(a, b - a)
        else:
            assert ix.append(c[a:b]) == a
        check(ix, q, c[:b], k)
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_snapshot_restore_keeps_the_dtype_and_refuses_the_other(sim, tmp_path):
    dim, n = 256, 3000
    c = rows(71, n, dim)
    q = queries(72, 40, dim, c)
    ix = index(sim, dim, 4096, max_batch=128)
    ix.append(c)
    ix.delete_rows([7, 8])
    ok = np.ones((len(q), n), bool)
    ok[:, [7, 8]] = False
    ix.snapshot(str(tmp_path / "s8"))
    z = np.load(str(tmp_path / "s8.npz"))
    assert str(z["dtype"]) == "int8" and z["rows"].dtype == np.int8
    ix2 = index(sim, dim, 4096, max_batch=128)
    assert ix2.restore(str(tmp_path / "s8")) == n
    assert cmax(ix2) <= cmax(ix)
    check(ix2, q, c, 10, ok=ok)
    b = index(sim, dim, 4096, max_batch=128, dtype="bfloat16")
    with pytest.raises(ValueError, match="dtype"):
        b.restore(str(tmp_path / "s8"))
    b.append(c.astype(np.float32))
    b.snapshot(str(tmp_path / "sb"))
    with pytest.raises(ValueError, match="dtype"):
        ix2.restore(str(tmp_path / "sb"))
    with pytest.raises(TypeError):
        ix2.append_bf16_bits(np.zeros((1, dim), np.uint16))
    import torch
    with pytest.raises(TypeError):
        ix2.search(dev_bf16(q), 10)                            # bf16 queries on an int8 index
    with pytest.raises(TypeError):
        b.search(dev8(q), 10)                                  # int8 queries on a bf16 index
    for x in (ix, ix2, b):
        x.close()
    torch.cuda.synchronize()


def test_vector_table_checkpoint_round_trip(tmp_path):
    from qsa_b200.operator import VectorTable, vector_search_agg
    dim, n, k = 384, 2000, 50
    c = rows(81, n, dim)
    q = queries(82, 12, dim, c)
    t = VectorTable(index("cosine", dim, 4096, max_batch=64))
    t.upsert_many([f"d{j}" for j in range(n)], [f"chunk {j}" for j in range(n)], c.astype(np.float32))
    before = vector_search_agg(t, "embedding", q.astype(np.float32), k)
    t.save(str(tmp_path / "ck"))
    t2 = VectorTable(index("cosine", dim, 4096, max_batch=64))
    assert t2.load(str(tmp_path / "ck")) == n
    after = vector_search_agg(t2, "embedding", q.astype(np.float32), k)
    assert [[(h.document_id, h.score, h.row) for h in r] for r in before] == \
           [[(h.document_id, h.score, h.row) for h in r] for r in after]
    _, ri = ref_topk(q, c, k, "cosine")
    assert [[h.row for h in r] for r in after] == ri.tolist()
    t3 = VectorTable(index("cosine", dim, 4096, max_batch=64, dtype="bfloat16"))
    with pytest.raises(ValueError, match="dtype"):
        t3.load(str(tmp_path / "ck"))
    for x in (t, t2, t3):
        x.index.close()


# ---------------------------------------------------------------------------------- host slots, shards, fixture
@pytest.mark.parametrize("sim", SIMS)
def test_host_submit_wait_with_both_slots_in_flight(sim):
    n, dim, nq, k = 6000, 768, 150, 10
    c = rows(91, n, dim)
    q = queries(92, nq, dim, c)
    ix = index(sim, dim, n, max_batch=256)
    ix.append(c)
    rs, ri = ref_topk(q, c, k, sim)
    qf = q.astype(np.float32)
    ix.search_host_submit(qf[:70], k, 0)
    ix.search_host_submit(qf[70:], k, 1)
    s0, i0 = ix.search_host_wait(0)
    s1, i1 = ix.search_host_wait(1)
    assert np.array_equal(np.concatenate([i0, i1]), ri)
    assert (np.abs(np.concatenate([s0, s1]) - rs) / np.maximum(1, np.abs(rs))).max() < 1e-6
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
def test_search_hits_and_merge_hits_over_two_shards(sim):
    import torch
    n, dim, nq, k = 10000, 256, 100, 64
    c = rows(101, n, dim)
    c[8000] = c[10]
    q = queries(102, nq, dim, c)
    q[0] = c[10]
    cut = 4000
    a, b = index(sim, dim, cut), index(sim, dim, n - cut)
    a.append(c[:cut]); b.append(c[cut:])
    hits = torch.stack([a.search_hits(dev8(q), k, 0), b.search_hits(dev8(q), k, cut)])
    s, gi = a.merge_hits(hits)
    torch.cuda.synchronize()
    rs, ri = ref_topk(q, c, k, sim)
    assert np.array_equal(gi.cpu().numpy(), ri)
    assert (np.abs(s.cpu().numpy() - rs) / np.maximum(1, np.abs(rs))).max() < 1e-6
    top = gi[0].tolist()
    assert top[top.index(10) + 1] == 8000 if sim != "dotProduct" else 8000 in top
    with pytest.raises(AssertionError):
        a.search_hits(dev_bf16(q), k, 0)
    a.close(); b.close()


@pytest.mark.parametrize("sim", SIMS)
def test_one_gpu_multi_gpu_index(sim):
    from qsa_b200.sharded import MultiGpuIndex
    n, dim, nq, k = 5000, 384, 64, 29
    c = rows(111, n, dim)
    q = queries(112, nq, dim, c)
    mi = MultiGpuIndex(dim=dim, capacity_per_gpu=n, max_batch=nq, max_k=k, n_gpus=1, similarity=sim, dtype="int8")
    assert mi.shards[0].dtype == "int8"
    mi.append(c[:2000])                                        # int8 rows
    mi.append(c[2000:].astype(np.float32))                     # fp32 rows, converted
    s, r = mi.search_host(q.astype(np.float32), k)
    rs, ri = ref_topk(q, c, k, sim)
    assert np.array_equal(r, ri)
    mi.close()


def test_mixed_element_types_are_refused_across_gpus():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from qsa_b200 import capi
    from qsa_b200.engine import VectorIndex
    dim = 256
    a = VectorIndex(dim=dim, capacity=1024, max_batch=64, max_k=10, device=0, dtype="int8")
    b = VectorIndex(dim=dim, capacity=1024, max_batch=64, max_k=10, device=1, dtype="bfloat16")
    c = rows(121, 600, dim)
    a.append(c); b.append(c.astype(np.float32))
    lib = a.lib
    h = C.c_void_p()
    capi.check(lib.sa_comm_create(C.byref(h), 2, (C.c_int * 2)(0, 1)), "sa_comm_create")
    engines = (C.c_void_p * 2)(a._h, b._h)
    offs = (C.c_int64 * 2)(0, 1024)
    q = np.ascontiguousarray(c[:8].astype(np.float32))
    score, row = np.empty((8, 10), np.float32), np.empty((8, 10), np.int64)
    rc = lib.sa_gather_merge(h, engines, q.ctypes.data, 8, 10, offs, score.ctypes.data, row.ctypes.data)
    assert rc == capi.SA_ERR_ARG and b"element type" in lib.sa_last_error()
    lib.sa_comm_destroy(h)
    a.close(); b.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_engine_reproduces_the_independent_fixture(path, sim, cg):
    import torch
    from qsa_b200.engine import stage_filters
    z = np.load(path)
    k = int(z["k"])
    c, q = z["corpus"], z["queries"]
    ix = index(sim, c.shape[1], len(c) + 256, max_batch=64, max_k=k)
    ix.append(c, tags=z["tags"])
    ix.set_option("cta_group", cg)
    for key, f in (("", None), ("_filtered", z["filters"])):
        s, i = ix.search(dev8(q), k, filters=None if f is None else stage_filters(f, len(q), torch.device("cuda")))
        torch.cuda.synchronize()
        assert np.array_equal(i.cpu().numpy(), z[f"{sim}{key}_idx"])
        ref = z[f"{sim}{key}_score"]
        got = s.cpu().numpy().astype(np.float64)
        fin = np.isfinite(ref)
        assert (got[~fin] == ref[~fin]).all()
        assert (np.abs(got[fin] - ref[fin]) / np.maximum(1.0, np.abs(ref[fin]))).max() < 1e-6
    ix.close()


# ----------------------------------------------------------------------------------------------- no fallback at size
@pytest.mark.parametrize("sim", SIMS)
def test_no_fallback_work_at_one_million_rows(sim):
    """1M x 768 iid int8: the certificate settles every query of a full batch without the fallback, at k 10 and 64, and
    a sample of the answers equals the definition (computed on the GPU in float64, exact for int8)."""
    import torch
    n, dim, nq = 1_000_000, 768, 512
    gen = torch.Generator(device="cuda").manual_seed(131)
    ix = index(sim, dim, n, max_batch=nq)
    for lo in range(0, n, 250_000):
        ix.append(torch.randint(-128, 128, (250_000, dim), generator=gen, device="cuda", dtype=torch.int8))
    q = torch.randint(-128, 128, (nq, dim), generator=gen, device="cuda", dtype=torch.int8)
    ix.set_option("count_fix", 1)
    c64 = ix.rows[:n].to(torch.float64)
    q64 = q[:16].to(torch.float64)
    dots = q64 @ c64.T
    cc = (c64 * c64).sum(axis=1)
    qq = (q64 * q64).sum(axis=1)
    if sim == "cosine":
        val = dots / torch.sqrt(qq[:, None] * cc[None, :])
    elif sim == "dotProduct":
        val = dots
    else:
        val = -torch.sqrt(torch.clamp((qq[:, None] - 2 * dots) + cc[None, :], min=0))
    cand_v, cand_i = torch.topk(val, 80, dim=1)
    cand_v, cand_i = cand_v.cpu().numpy(), cand_i.cpu().numpy()
    del c64, dots, val
    for k in (10, 64):
        s, i = ix.search(q, k)
        torch.cuda.synchronize()
        assert ix.info("last_fix_entries") == 0
        got = i[:16].cpu().numpy()
        for r in range(16):
            order = np.lexsort((cand_i[r], -cand_v[r]))[:k]
            assert got[r].tolist() == cand_i[r][order].tolist()
    ix.close()
