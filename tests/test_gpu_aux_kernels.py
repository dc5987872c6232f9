"""The kernels either side of the scan (csrc/sa_aux.cuh) on the H100, each against a float64 or integer reference
written here: fp32 -> bf16 and fp32 -> int8 conversion on the device, the row terms of every ingest path, the norm bound
Cmax, rows holding NaN or inf, the finalisation of the scores, the two shard merges on both sides of the switch from the
warp merge to the serial one, and dimensions up to SA_MAX_DIM.

The search tests elsewhere see these kernels only through the returned index lists, and the certificate keeps those
right even when a row term is one rounding off or Cmax is slightly too small.  The exactness argument (DESIGN.md
section 4.2) still rests on what these kernels claim, so the claims are checked here bit for bit where they are exact.

The data are integers times powers of two, so every float64 sum of products below is exact; ``assert_exact_sums``
checks that before a test relies on it.

Run on an H100 with:  python -m pytest tests/test_gpu_aux_kernels.py -m gpu
"""
import os
import tempfile

import numpy as np
import pytest

from harness import similarity_oracle as so
from oracle import bruteforce as bf

pytestmark = pytest.mark.gpu

SIMS = so.SIMILARITIES
ELEMS = ("bfloat16", "int8")
U23 = 2.0 ** -23


# ---------------------------------------------------------------------------------------------------------- helpers
def make_index(sim, dim, capacity, dtype="bfloat16", max_k=64, max_batch=256):
    from qsa_b200.engine import VectorIndex
    return VectorIndex(dim=dim, capacity=capacity, max_batch=max_batch, max_k=max_k, similarity=sim, dtype=dtype)


def f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def dev(x, dtype):
    """Rows or queries (bf16 bit patterns or int8) as a CUDA tensor of the index's dtype."""
    import torch
    if dtype == "int8":
        return torch.from_numpy(np.ascontiguousarray(x, np.int8)).cuda()
    return torch.from_numpy(np.ascontiguousarray(x, np.uint16).view(np.int16)).cuda().view(torch.bfloat16)


def stored(ix, lo=0, hi=None):
    """The rows the index holds: bf16 bit patterns (uint16) or int8."""
    import torch
    torch.cuda.synchronize()
    r = ix.rows[lo:len(ix) if hi is None else hi]
    return r.cpu().numpy() if ix.dtype == "int8" else r.view(torch.int16).cpu().numpy().view(np.uint16)


def terms(ix):
    import torch
    torch.cuda.synchronize()
    return ix.inv_norm[:len(ix)].cpu().numpy()


def cmax(ix) -> np.float32:
    return np.array(ix.info("cmax_bits"), np.uint32).view(np.float32)[()]


def values(x, dtype):
    """float64 values of bf16 bit patterns or int8 elements."""
    return x.astype(np.float64) if dtype == "int8" else bf.bf16_bits_to_f32(x).astype(np.float64)


def as_f32(x, dtype):
    """The rows as fp32 input that converts to exactly these elements."""
    return values(x, dtype).astype(np.float32)


def lsb(x):
    """Per row of float64 values: the weight of the lowest set bit over its nonzero elements (inf for a zero row)."""
    m, e = np.frexp(np.abs(x))
    mi = (m * 2.0 ** 53).astype(np.int64)
    low = (mi & -mi).astype(np.float64) * np.exp2(e.astype(np.float64) - 53)
    return np.where(mi > 0, low, np.inf).min(axis=1)


def assert_exact_sums(a, b):
    """Every <a_i, b_j> is exact in float64: each product is a multiple of lsb(a_i) lsb(b_j), and the sum of their
    magnitudes stays below 2^52 of that unit, so no partial sum in any order rounds."""
    unit = lsb(a)[:, None] * lsb(b)[None, :]
    mag = np.abs(a) @ np.abs(b).T
    ok = (mag == 0) | (mag < 2.0 ** 52 * unit)
    assert ok.all(), "test data too wide for exact float64 sums"


def bf16_rows(g, n, dim, lo=-7, hi=-7, row_scale=0):
    """bf16 rows of elements m 2^e: m an integer in [-127, 127] (8 significant bits, exact in bf16), e per element in
    [lo, hi], and a per-row factor 2^s with s in [-row_scale, row_scale].  Returned as bit patterns."""
    m = g.integers(-127, 128, (n, dim)).astype(np.float64)
    e = g.integers(lo, hi + 1, (n, dim)) + g.integers(-row_scale, row_scale + 1, (n, 1))
    return bf.f32_to_bf16_bits((m * np.exp2(e)).astype(np.float32))


def mixed_rows(g, n, dim, dtype):
    """Rows for the row-term tests: iid rows, rows whose magnitudes spread over 2^10 with per-row scales over 2^24,
    rows with a few large elements over many tiny ones (an fp32 sum absorbs the tiny squares), and all-zero rows."""
    if dtype == "int8":
        x = g.integers(-128, 128, (n, dim)).astype(np.int8)
        x[1::4] = np.where(g.random((len(x[1::4]), dim)) < 0.05, 127, g.integers(-1, 2, (len(x[1::4]), dim)))
        x[2::4] = g.integers(-3, 4, (len(x[2::4]), dim))
        x[3::9] = -128
    else:
        x = bf16_rows(g, n, dim)
        x[1::4] = bf16_rows(g, len(x[1::4]), dim, -8, 2, row_scale=12)
        big = bf16_rows(g, len(x[2::4]), dim, 4, 4)
        tiny = bf16_rows(g, len(x[2::4]), dim, -10, -10)
        x[2::4] = np.where(g.random(big.shape) < 0.01, big, tiny)
    x[0] = 0
    x[n // 2] = 0
    return x


def ingest(ix, x, path, pieces):
    """Rows x into ix by one ingest path, in pieces of the given sizes (odd first rows and partial warps and blocks)."""
    import torch
    lo = 0
    for n in pieces:
        part = x[lo:lo + n]
        if path == "host":
            ix.append(as_f32(part, ix.dtype))
        elif path == "device":
            ix.append(torch.from_numpy(as_f32(part, ix.dtype)).cuda())
        elif path == "elements":                         # append_bf16_bits / int8 rows: written in place + commit
            add_rows(ix, part)
        elif path == "commit":                           # the caller writes the rows in place, then commits them
            first = len(ix)
            ix.rows[first:first + n].copy_(dev(part, ix.dtype))
            ix.commit(first, n)
        else:
            raise ValueError(path)
        lo += n
    assert lo == len(x) == len(ix)


def restored(ix, sim, capacity):
    """A fresh index of ix's kind holding ix's snapshot (sa_corpus_bind recomputes Cmax over the restored rows); ix is
    closed."""
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "snap.npz")
        ix.snapshot(p)
        ix.close()
        out = make_index(sim, ix.dim, capacity, ix.dtype)
        out.restore(p)
    return out


def add_rows(ix, x):
    """Rows of the index's element type, written in place and committed (append_bf16_bits, or int8 rows)."""
    return ix.append(x) if ix.dtype == "int8" else ix.append_bf16_bits(x)


def near(g, x, pick, frac=0.1):
    """Rows x[pick] with a fraction of their elements replaced by those of fresh rows of the same kind."""
    fresh = g.integers(-128, 128, (len(pick), x.shape[1])).astype(np.int8) if x.dtype == np.int8 else \
        bf16_rows(g, len(pick), x.shape[1])
    return np.where(g.random(fresh.shape) < frac, fresh, x[pick])


def ref_row_terms(x, sim, dtype):
    """dotProduct 1, euclidean fp32(|c|^2 / 2), int8 cosine fp32(1 / |c|) from the exact sum; 0 for a zero row under
    cosine.  bf16 cosine is None: it keeps its fp32 sum and is checked against a bound."""
    ss = (values(x, dtype) ** 2).sum(axis=1)
    if sim == "dotProduct":
        return np.ones(len(x), np.float32)
    if sim == "euclidean":
        return (0.5 * ss).astype(np.float32)
    if dtype == "int8":
        with np.errstate(divide="ignore"):
            return np.where(ss > 0, 1.0 / np.sqrt(ss), 0.0).astype(np.float32)
    return None


def assert_cmax_bounds(ix, x, dtype, live=None):
    """max |c| <= Cmax <= max |c| (1 + 2^-20) over the live rows."""
    norms = np.sqrt((values(x, dtype) ** 2).sum(axis=1))
    top = norms.max() if live is None else norms[live].max()
    c = float(cmax(ix))
    assert top <= c <= top * (1 + 2.0 ** -20), (top, c)


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


# ------------------------------------------------------------------------------------------- 1. conversion on the device
def bf16_edge_inputs(g, dim):
    """fp32 inputs at the edges of fp32 -> bf16 rounding, padded with random fp32 bit patterns."""
    edges = [
        0x3f808000, 0x3f818000, 0xbf808000, 0xbf818000,   # ties: even upper half stays, odd rounds up (both signs)
        0x3f80c000, 0x3f804000, 0x40490fdb,               # above / below a tie, pi
        0x3fffffff, 0x3fff8000, 0xbfffffff, 0x3f7fffff,   # round up into the next binade
        0x7f7fffff, 0xff7fffff, 0x7f7f8000, 0x7f7f7fff,   # FLT_MAX and its neighbours: to +-inf or not
        0x7f800000, 0xff800000, 0x00000000, 0x80000000,   # +-inf, +-0
        0x00000001, 0x00008000, 0x00018000, 0x007fffff, 0x80000001, 0x807fffff, 0x00400000,  # subnormals
        0x7fc00000, 0x7f800001, 0xffffffff, 0x7fbfffff, 0xff800001, 0x7fc12345, 0x7f80ffff, 0xffc00001,  # NaN payloads
    ]
    n = 4
    u = g.integers(0, 2 ** 32, (n, dim), dtype=np.uint64).astype(np.uint32)
    u.reshape(-1)[: len(edges)] = np.asarray(edges, np.uint32)
    u[2, 1::3] = np.asarray(edges, np.uint32)[np.arange(len(u[2, 1::3])) % len(edges)]
    return u.view(np.float32)


@pytest.mark.parametrize("source", ["host", "device"])
@pytest.mark.parametrize("sim", SIMS)
def test_fp32_to_bf16_conversion_is_rne_bit_for_bit(sim, source):
    """sa_convert_rows_kernel (cosine) and sa_convert_rows_term_kernel (the others) store f32_to_bf16_bits of each
    input: ties to even, overflow to inf, subnormals, and NaN kept NaN with its payload's top bits and the quiet bit."""
    import torch
    dim = 64
    x = bf16_edge_inputs(np.random.default_rng(11), dim)
    ix = make_index(sim, dim, 64)
    ix.append(x if source == "host" else torch.from_numpy(x).cuda())
    want = bf.f32_to_bf16_bits(x)
    got = stored(ix)
    assert np.array_equal(got, want), np.argwhere(got != want)[:8]
    ix.close()


def int8_want(x):
    with np.errstate(invalid="ignore"):
        r = np.clip(np.rint(x.astype(np.float64)), -128, 127)
    return np.where(np.isnan(r), 0, r).astype(np.int8)


INT8_EDGES = np.array([127.5, -127.5, 128.5, -128.5, 126.5, -126.5, 0.5, -0.5, 1.5, -1.5, 2.5, 127.49998, -128.49998,
                       127.0, -128.0, 1e30, -1e30, np.inf, -np.inf, -0.0, 0.0, np.nan, -np.nan, 1e-45],
                      np.float32)


@pytest.mark.parametrize("source", ["host", "device"])
def test_fp32_to_int8_conversion_of_rows_on_the_device(source):
    """sa_convert_rows_i8_kernel on rows: clip(rint(x), -128, 127), NaN -> 0, at the rounding and saturation edges."""
    import torch
    dim = 128
    g = np.random.default_rng(12)
    x = (g.standard_normal((3, dim)) * 90).astype(np.float32)
    x[0, :len(INT8_EDGES)] = INT8_EDGES
    x[1, ::5] = INT8_EDGES[np.arange(len(x[1, ::5])) % len(INT8_EDGES)]
    ix = make_index("dotProduct", dim, 16, "int8")
    ix.append(x if source == "host" else torch.from_numpy(x).cuda())
    assert np.array_equal(stored(ix), int8_want(x))
    ix.close()


def test_fp32_to_int8_conversion_of_queries_on_the_device():
    """sa_convert_rows_i8_kernel on queries (device and host fp32 searches), read back through a dotProduct index of
    unit rows e_j: the exact score of row j is the converted query's element j."""
    import torch
    dim, m = 128, 64
    c = np.zeros((m, dim), np.int8)
    c[np.arange(m), np.arange(m)] = 1
    g = np.random.default_rng(13)
    q = (g.standard_normal((5, dim)) * 90).astype(np.float32)
    q[0, :len(INT8_EDGES)] = INT8_EDGES
    q[1, :len(INT8_EDGES)] = -INT8_EDGES
    q[2, :m] = INT8_EDGES[np.arange(m) % len(INT8_EDGES)][::-1]
    want = int8_want(q[:, :m]).astype(np.float64)
    ix = make_index("dotProduct", dim, m, "int8")
    ix.append(c)
    _, i, s64 = ix.search(torch.from_numpy(q).cuda(), m, want_score64=True)
    i, s64 = i.cpu().numpy(), s64.cpu().numpy()
    got = np.zeros_like(want)
    np.put_along_axis(got, i.astype(np.int64), s64, axis=1)
    assert np.array_equal(np.sort(i, axis=1), np.tile(np.arange(m), (len(q), 1)))
    assert np.array_equal(got, want)
    _, hi = ix.search_host(q, m)
    assert np.array_equal(hi, i)
    ix.close()


# ---------------------------------------------------------------------------------------------------- 2. row terms
PIECES = [3, 1, 7, 33, 257, 1000]          # odd first rows, partial warps and blocks
PATHS = ["host", "device", "elements", "commit", "restore"]
DIMS = {"bfloat16": 1600, "int8": 1664}    # 16-byte vectors per row not a multiple of 32 lanes


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("dtype", ELEMS)
@pytest.mark.parametrize("sim", SIMS)
def test_row_terms_and_cmax_of_every_ingest_path(sim, dtype, path):
    """Row terms bit for bit against the exact sum of squares rounded once (dotProduct 1, euclidean fp32(|c|^2 / 2),
    int8 cosine fp32(1 / |c|)); bf16 cosine keeps its fp32 sum and must stay within its share of eps_rel,
    |w |c| - 1| <= (D/4 + 2) 2^-23.  Zero rows: cosine 0, dotProduct 1, euclidean 0.  Cmax bounds the norms tightly."""
    dim = DIMS[dtype]
    n = sum(PIECES)
    x = mixed_rows(np.random.default_rng(21), n, dim, dtype)
    v = values(x, dtype)
    assert_exact_sums(v, v)
    ix = make_index(sim, dim, n, dtype)
    ingest(ix, x, "elements" if path == "restore" else path, PIECES)
    if path == "restore":
        ix = restored(ix, sim, n)
    assert np.array_equal(stored(ix), x)
    w = terms(ix)
    want = ref_row_terms(x, sim, dtype)
    if want is not None:
        bad = np.flatnonzero(w.view(np.uint32) != want.view(np.uint32))
        assert bad.size == 0, (bad[:8], w[bad[:8]], want[bad[:8]])
    else:
        norm = np.sqrt((v ** 2).sum(axis=1))
        live = norm > 0
        err = np.abs(w[live].astype(np.float64) * norm[live] - 1.0)
        assert err.max() <= (dim / 4 + 2) * U23, err.max()
        assert (w[~live] == 0).all()
    zero = ~v.any(axis=1)
    assert zero.sum() == 2
    assert (w[zero] == {"cosine": 0.0, "dotProduct": 1.0, "euclidean": 0.0}[sim]).all()
    if sim != "cosine":
        assert_cmax_bounds(ix, x, dtype)
    ix.close()


# ------------------------------------------------------------------------------------------------------ 3. Cmax
@pytest.mark.parametrize("dtype", ELEMS)
@pytest.mark.parametrize("sim", ["dotProduct", "euclidean"])
def test_cmax_through_append_delete_restore_and_reset(sim, dtype):
    """Cmax: tight after each append; raised by a longer row, unchanged by a shorter one; not lowered by delete_rows
    (a tombstone only writes the row's term, and a bound that stays too large only widens the certificate's band);
    recomputed over the restored rows by restore; 0 after reset, and then the bound of the new rows alone."""
    dim = 256
    g = np.random.default_rng(31)
    if dtype == "int8":
        x = g.integers(-40, 41, (300, dim)).astype(np.int8)
        longer = np.full((1, dim), 100, np.int8)
        shorter = np.full((1, dim), 3, np.int8)
    else:
        x = bf16_rows(g, 300, dim)
        longer = bf16_rows(g, 1, dim, -4, -4)
        shorter = bf16_rows(g, 1, dim, -12, -12)
    norms = np.sqrt((values(x, dtype) ** 2).sum(axis=1))
    top = norms.max()
    assert np.float64(np.float32(top)) != top, "the largest norm must not be a float (a bound rounded down would fail)"
    ix = make_index(sim, dim, 400, dtype)
    add_rows(ix, x)
    assert_cmax_bounds(ix, x, dtype)
    before = cmax(ix)
    add_rows(ix, shorter)
    assert same_bits(cmax(ix), before)
    add_rows(ix, longer)
    allx = np.concatenate([x, shorter, longer])
    assert float(cmax(ix)) > float(before)
    assert_cmax_bounds(ix, allx, dtype)
    raised = cmax(ix)
    ix.delete_rows([len(ix) - 1])
    assert same_bits(cmax(ix), raised)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "snap.npz")
        ix.snapshot(p)                                # the deleted row is stored zeroed
        ix.restore(p)
    assert_cmax_bounds(ix, np.concatenate([x, shorter]), dtype)
    ix.reset()
    assert cmax(ix) == 0
    add_rows(ix, x[:5])
    assert_cmax_bounds(ix, x[:5], dtype)
    ix.close()


# ------------------------------------------------------------------------------------------------ 4. non-finite rows
BAD_ROWS = [5, 300, 1299]


@pytest.mark.parametrize("path", ["bits", "fp32", "restore"])
@pytest.mark.parametrize("sim", SIMS)
def test_rows_with_nan_or_inf_are_not_live(sim, path):
    """A bf16 row holding one NaN, +inf or -inf element is never returned, as in the definition (which drops
    non-finite values): its row term is the tombstone's and it does not enter Cmax, so Cmax equals that of the same
    corpus without those rows and the searches of every other row stay exact, without the fallback on iid data."""
    import torch
    dim, n, nq, k = 256, 1300, 48, 10
    g = np.random.default_rng(41)
    c = bf16_rows(g, n, dim)
    clean = c.copy()
    clean[BAD_ROWS] = 0
    if path == "fp32":
        # fp32 inputs that round past FLT_MAX to +-inf, and a NaN with a payload
        x = as_f32(c, "bfloat16")
        for r, u in zip(BAD_ROWS, [0x7f7fffff, 0xff7fffff, 0x7fa00001]):
            x[r, 17 + r % 50] = f32(u)
        half = n // 2
        ix = make_index(sim, dim, n)
        ix.append(x[:half])
        ix.append(torch.from_numpy(x[half:]).cuda())
        c = bf.f32_to_bf16_bits(x)
    else:
        for r, b in zip(BAD_ROWS, [0x7fc1, 0x7f80, 0xff80]):
            c[r, 17 + r % 50] = b
        ix = make_index(sim, dim, n)
        ix.append_bf16_bits(c)
        if path == "restore":
            ix = restored(ix, sim, n)
    assert np.array_equal(stored(ix), c)
    nonfinite = ~np.isfinite(bf.bf16_bits_to_f32(c)).all(axis=1)
    assert np.flatnonzero(nonfinite).tolist() == BAD_ROWS
    q = bf16_rows(g, nq, dim)
    q[::2] = near(g, c, g.choice(np.flatnonzero(~nonfinite), nq // 2))
    q[1] = c[BAD_ROWS[0]]
    q[1, 17 + BAD_ROWS[0] % 50] = 0x3f80                                        # next to a NaN row
    v = values(q, "bfloat16"), values(clean, "bfloat16")
    assert_exact_sums(*v)
    with np.errstate(all="ignore"):
        rs, ri = so.topk_f64(q, c, k, sim)
    ix.set_option("count_fix", 1)
    s, i = (t.cpu().numpy() for t in ix.search(dev(q, "bfloat16"), k))
    fixed = ix.info("last_fix_entries")
    assert np.array_equal(i, ri), f"empty slots {np.mean(i < 0):.2f}, non-finite scores {np.mean(~np.isfinite(s)):.2f}, " \
                                  f"fallback entries {fixed}"
    assert np.isfinite(s).all()
    assert fixed == 0
    assert (terms(ix)[BAD_ROWS] == (-1.0 if sim == "euclidean" else 0.0)).all()
    if sim != "cosine":
        twin = make_index(sim, dim, n)
        twin.append_bf16_bits(clean)
        assert np.isfinite(cmax(ix)) and same_bits(cmax(ix), cmax(twin)), (cmax(ix), cmax(twin))
        twin.close()
    ix.close()


# ------------------------------------------------------------------------------------------------- 5. finalisation
def exact_score64(q, c, idx, sim, dtype):
    """The engine's documented formula in numpy on exact sums, evaluated op for op as the device does:
    dot <q,c>; cosine <q,c> / sqrt(|q|^2 |c|^2); euclidean sqrt(max(0, (|q|^2 - 2 <q,c>) + |c|^2)).
    (The cosine of harness/similarity_oracle.py divides by |q| |c| instead, which can differ by one ulp; the
    index lists do not depend on it and it stays as it is.)"""
    qv, cv = values(q, dtype), values(c, dtype)
    out = np.full(idx.shape, np.nan)
    for a in range(len(q)):
        ok = idx[a] >= 0
        rows = cv[idx[a][ok]]
        dot = rows @ qv[a]
        qq, cc = qv[a] @ qv[a], (rows * rows).sum(axis=1)
        if sim == "dotProduct":
            s = dot
        elif sim == "cosine":
            s = dot / np.sqrt(qq * cc)
        else:
            s = np.sqrt(np.maximum(0.0, (qq - 2.0 * dot) + cc))
        out[a, ok] = s
    return out


def finalise_data(dtype, n, dim, nq):
    g = np.random.default_rng(51)
    if dtype == "int8":
        c = g.integers(-128, 128, (n, dim)).astype(np.int8)
        q = g.integers(-127, 128, (nq, dim)).astype(np.int8)
    else:
        c = bf16_rows(g, n, dim)
        q = bf16_rows(g, nq, dim)
    # heavy cancellation: rows 10..39 repeat their first half, and every third query is [q_lo, -q_lo], so their dot
    # products cancel to exactly 0 (a plain fp32 sum of the halves would not)
    h = dim // 2
    c[10:40, h:] = c[10:40, :h]
    q[::3, h:] = (-values(q[::3, :h], dtype)).astype(np.int8) if dtype == "int8" else q[::3, :h] ^ np.uint16(0x8000)
    q[1::3] = near(g, c, g.integers(0, n, len(q[1::3])))
    q[2] = c[12]                            # a distance of exactly 0
    c[3] = 0
    return c, q


@pytest.mark.parametrize("force_fix", [0, 1])
@pytest.mark.parametrize("dtype", ELEMS)
@pytest.mark.parametrize("sim", SIMS)
def test_finalised_scores_are_the_documented_formula_rounded_once(sim, dtype, force_fix):
    """score == fp32(score64) bit for bit (one RNE rounding), score64 == the documented formula on exact sums bit for
    bit, search_hits records carry (score64, idx + row_offset), and empty slots are -1 with -inf (+inf for distances)
    in score, score64 and the hit records -- through the merge kernel alone and through the fallback scan."""
    import torch
    dim = 256 if dtype == "bfloat16" else 384
    n, nq, k = 700, 40, 16
    c, q = finalise_data(dtype, n, dim, nq)
    assert_exact_sums(values(q, dtype), values(c, dtype))
    ix = make_index(sim, dim, n, dtype)
    add_rows(ix, c)
    ix.set_option("force_fix", force_fix)
    s, i, s64 = (t.cpu().numpy() for t in ix.search(dev(q, dtype), k, want_score64=True))
    assert (i >= 0).all()
    assert same_bits(s, s64.astype(np.float32))
    want = exact_score64(q, c, i, sim, dtype)
    assert same_bits(s64, want), np.argwhere(s64.view(np.uint64) != want.view(np.uint64))[:8]
    off = (1 << 33) + 7
    hits = ix.search_hits(dev(q, dtype), k, row_offset=off)
    torch.cuda.synchronize()
    h = hits.cpu().numpy().reshape(nq, k, 16)
    assert same_bits(h[..., :8].copy().view(np.float64)[..., 0], s64)
    assert np.array_equal(h[..., 8:].copy().view(np.int64)[..., 0], i.astype(np.int64) + off)
    ix.close()

    # fewer rows than k: the last slots are empty in every output (cosine never returns the zero row)
    small = make_index(sim, dim, 8, dtype)
    add_rows(small, c[:6])
    small.set_option("force_fix", force_fix)
    s, i, s64 = (t.cpu().numpy() for t in small.search(dev(q[:3], dtype), k, want_score64=True))
    h = small.search_hits(dev(q[:3], dtype), k, row_offset=off).cpu().numpy().reshape(3, k, 16)
    full = 5 if sim == "cosine" else 6
    empty = np.inf if sim == "euclidean" else -np.inf
    assert (i[:, :full] >= 0).all() and (i[:, full:] == -1).all()
    assert (s[:, full:] == empty).all() and (s64[:, full:] == empty).all()
    assert (h[:, full:, :8].copy().view(np.float64) == empty).all()
    assert (h[:, full:, 8:].copy().view(np.int64) == -1).all()
    assert same_bits(s64[:, :full], exact_score64(q[:3], c, i, sim, dtype)[:, :full])
    small.close()


# ---------------------------------------------------------------------------------------------- 6. shard merges
# n_shards x k on both sides of the warp merge's limits (32 shards, k 32, 256 hits per query); 257 hits cannot be
# written as n_shards x k with both at most 32, so 260 (10 x 26, 13 x 20) are the nearest past the limit.
MERGE_CASES = [(g, k) for g in (1, 2, 7, 8, 31, 32, 33, 64) for k in (1, 10, 31, 32, 33, 64)]
MERGE_CASES += [(16, 16), (32, 8), (10, 26), (13, 20), (9, 29)]      # 256 hits, and just past it
SCORE_POOL = np.array([-0.0, 0.0, 0.1, -0.1, 1.0 / 3.0, 2.5, -7.75, 1e-30, 3e38, -3e38])   # exact ties across shards


def shard_lists(g, n_shards, nq, k, asc):
    """Per-shard hit lists [n_shards, nq, k], each sorted by (score desc, row asc) -- asc: (score asc, row asc) --
    with unique global rows per query, exact ties (+-0.0 among them) across shards, shards with fewer than k hits, one
    shard with none, and a query (0) whose every shard is empty.  Empty slots: row -1, score -inf (+inf when asc)."""
    score = SCORE_POOL[g.integers(0, len(SCORE_POOL), (n_shards, nq, k))]
    score[..., ::3] = g.standard_normal(score[..., ::3].shape)
    rows = np.argsort(g.random((nq, n_shards * k * 2)), axis=1)[:, :n_shards * k]
    rows = rows.reshape(nq, n_shards, k).transpose(1, 0, 2).astype(np.int64) * 3 + 1000
    fill = g.integers(0, k + 1, (n_shards, nq))
    fill[g.random((n_shards, nq)) < 0.5] = k
    if n_shards > 1:
        fill[(n_shards - 1) // 2] = 0                # not the last shard, whose hits must still be read
    fill[:, 0] = 0
    empty = np.arange(k)[None, None, :] >= fill[..., None]
    score[empty] = np.inf if asc else -np.inf
    rows[empty] = -1
    key = score if asc else -score
    order = np.lexsort((rows, key, empty), axis=-1)
    return np.take_along_axis(score, order, -1), np.take_along_axis(rows, order, -1)


def numpy_merge(score, rows, k, asc):
    """np.lexsort over the union of the shards' hits: (score desc, global row asc), or ascending scores when asc."""
    n_shards, nq, _ = score.shape
    s = score.transpose(1, 0, 2).reshape(nq, -1)
    r = rows.transpose(1, 0, 2).reshape(nq, -1)
    empty = r < 0
    order = np.lexsort((r, s if asc else -s, empty), axis=-1)[:, :k]
    ms, mr = np.take_along_axis(s, order, -1), np.take_along_axis(r, order, -1)
    return ms.astype(np.float32), mr


@pytest.fixture(scope="module")
def merge_engines():
    ixs = {asc: make_index("euclidean" if asc else "cosine", 64, 64) for asc in (False, True)}
    yield ixs
    for ix in ixs.values():
        ix.close()


@pytest.mark.parametrize("fn", ["merge_hits", "merge_shards"])
@pytest.mark.parametrize("n_shards,k", MERGE_CASES)
def test_shard_merges_against_a_numpy_merge(merge_engines, n_shards, k, fn):
    """sa_merge_hits (the warp merge up to 32 shards, k 32 and 256 hits per query, the serial merge past any of them)
    and sa_merge_shards (always serial) return the numpy merge: indices exactly, scores as fp32 of the winning hit."""
    import torch
    from qsa_b200.engine import HIT_DTYPE
    g = np.random.default_rng(1000 * n_shards + k)
    for asc in (False, True):
        ix = merge_engines[asc]
        for nq in (1, 3, 5, 129):
            score, rows = shard_lists(g, n_shards, nq, k, asc)
            if fn == "merge_hits":
                rec = np.empty(score.shape, HIT_DTYPE)
                rec["score"], rec["row"] = score, rows
                hits = torch.from_numpy(rec.view(np.uint8).reshape(n_shards, nq, k, 16).copy()).cuda()
                s, r = ix.merge_hits(hits)
            else:
                s, r = ix.merge_shards(torch.from_numpy(score).cuda(), torch.from_numpy(rows).cuda())
            ws, wr = numpy_merge(score, rows, k, asc)
            s, r = s.cpu().numpy(), r.cpu().numpy()
            assert np.array_equal(r, wr), (asc, nq, np.argwhere(r != wr)[:4])
            assert same_bits(s, ws), (asc, nq)
            assert (r[0] == -1).all()


@pytest.mark.parametrize("n_shards", [0, 65])
def test_shard_merges_refuse_0_and_65_shards(merge_engines, n_shards):
    import torch
    from qsa_b200 import capi
    ix = merge_engines[False]
    nq, k = 2, 4
    buf = torch.zeros((65, nq, k, 16), dtype=torch.uint8, device="cuda")     # valid memory for either count
    score = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    row = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    rc = ix.lib.sa_merge_hits(ix._h, buf.data_ptr(), n_shards, nq, k, score.data_ptr(), row.data_ptr(), 0)
    assert rc == capi.SA_ERR_ARG and b"n_shards" in ix.lib.sa_last_error()
    rc = ix.lib.sa_merge_shards(ix._h, buf.data_ptr(), buf.data_ptr(), n_shards, nq, k, score.data_ptr(),
                                row.data_ptr(), 0)
    assert rc == capi.SA_ERR_ARG and b"n_shards" in ix.lib.sa_last_error()


# ---------------------------------------------------------------------------------------------------- 7. dimensions
def dims_data(dtype, n, dim, nq, seed):
    g = np.random.default_rng(seed)
    if dtype == "int8":
        c = g.integers(-128, 128, (n, dim)).astype(np.int8)
        q = np.clip(c[g.integers(0, n, nq)].astype(np.int64) + g.integers(-30, 31, (nq, dim)), -128, 127)
        return c, q.astype(np.int8)
    c = bf16_rows(g, n, dim)
    q = near(g, c, g.integers(0, n, nq))
    q[::2] = bf16_rows(g, len(q[::2]), dim)
    return c, q


def check_search(ix, c, q, k, sim, dtype):
    v = values(q, dtype), values(c, dtype)
    assert_exact_sums(*v)
    s, i = ix.search(dev(q, dtype), k)
    if dtype == "int8":      # the same integers as bf16 are exact in the definition too
        qb, cb = bf.f32_to_bf16_bits(v[0].astype(np.float32)), bf.f32_to_bf16_bits(v[1].astype(np.float32))
    else:
        qb, cb = q, c
    rs, ri = so.topk_f64(qb, cb, k, sim)
    assert np.array_equal(i.cpu().numpy(), ri)
    assert np.abs(s.cpu().numpy() - rs).max() <= 1e-6 * max(1.0, np.abs(rs).max())


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("dim", [2048, 3072, 4096])
def test_common_embedding_sizes_match_the_definition(dim, sim, cg):
    c, q = dims_data("bfloat16", 700, dim, 24, dim)
    ix = make_index(sim, dim, 700)
    ix.append_bf16_bits(c)
    ix.set_option("cta_group", cg)
    check_search(ix, c, q, 10, sim, "bfloat16")
    ix.close()


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("dtype,dim", [("bfloat16", 12288), ("bfloat16", 12352), ("bfloat16", 16384),
                                       ("bfloat16", 65536), ("int8", 49152), ("int8", 49280), ("int8", 65536)])
def test_large_dims_up_to_the_limit_match_the_definition(dtype, dim, sim):
    """Both sides of the fallback scan's 48 KB shared-memory step (bf16 query rows of 2 D bytes, int8 of D bytes) up to
    SA_MAX_DIM: the search, and the same search through the fallback scan alone (force_fix)."""
    c, q = dims_data(dtype, 300, dim, 8, dim + len(sim))
    ix = make_index(sim, dim, 300, dtype, max_k=10, max_batch=8)
    add_rows(ix, c)
    check_search(ix, c, q, 10, sim, dtype)
    ix.set_option("force_fix", 1)
    check_search(ix, c, q, 10, sim, dtype)
    ix.close()
