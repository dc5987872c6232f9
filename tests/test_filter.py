"""Pre-filtered search, CPU side: the kernels' predicate (host-compiled through sa_debug_filter_pass), the MQL compiler
and its schema, the table checkpoint's filter fields, and the filtered definition against an independent fixture."""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest

from harness.filter_oracle import eligibility, topk_f64
from qsa_b200.filters import NEVER, FilterSchema, compile_filter, filter_pass

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "filter_topk_independent_*.npz")))


def lib():
    from qsa_b200 import capi
    try:
        return capi.load()
    except capi.SaLibraryMissing:
        pytest.skip("libsa_b200.so not built")


def numpy_pass(tags, f):
    t = [int(x) for x in tags]
    a, n, o0, o1 = (int(x) for x in f)
    return np.array([(x & a) == a and (x & n) == 0 and (o0 == 0 or x & o0) and (o1 == 0 or x & o1) for x in t], bool)


def test_debug_filter_pass_matches_the_normal_form():
    L = lib()
    g = np.random.default_rng(5)
    for trial in range(300):
        # sparse random words so that every clause both passes and fails on some rows
        def word(p):
            return np.uint64(sum(1 << int(b) for b in np.flatnonzero(g.random(64) < p)))
        tags = np.array([word(0.4) for _ in range(97)], dtype=np.uint64)
        f = np.array([word(0.03), word(0.03), word(0.05) if trial % 3 else 0, word(0.05) if trial % 2 else 0],
                     dtype=np.uint64)
        out = np.zeros(len(tags), np.uint8)
        assert L.sa_debug_filter_pass(tags.ctypes.data, len(tags), f.ctypes.data, out.ctypes.data) == 0
        ref = numpy_pass(tags, f)
        assert (out.astype(bool) == ref).all()
        assert (filter_pass(tags, f) == ref).all()
    out = np.zeros(3, np.uint8)
    tags = np.array([0, 1, 2**64 - 1], dtype=np.uint64)
    zero = np.zeros(4, np.uint64)
    assert L.sa_debug_filter_pass(tags.ctypes.data, 3, zero.ctypes.data, out.ctypes.data) == 0 and out.all()
    never = np.array([NEVER, 0, 0, 0], np.uint64)
    assert L.sa_debug_filter_pass(tags[:2].ctypes.data, 2, never.ctypes.data, out.ctypes.data) == 0 and not out[:2].any()


# ---------------------------------------------------------------------------------------------------- MQL reference
def _has(row, field, v):
    x = row.get(field)
    if x is None:
        return False
    items = x if isinstance(x, list) else [x]
    return any(type(i) is type(v) and i == v for i in items)


def mql_eval(doc, row) -> bool:
    """Direct evaluation of the supported MQL subset over one metadata dict (array fields: "contains")."""
    ok = True
    for key, val in doc.items():
        if key == "$and":
            ok &= all(mql_eval(d, row) for d in val)
        elif key == "$or":
            ok &= any(mql_eval(d, row) for d in val)
        elif key == "$nor":
            ok &= not any(mql_eval(d, row) for d in val)
        else:
            ops = val if isinstance(val, dict) else {"$eq": val}
            for op, v in ops.items():
                if op == "$eq":
                    ok &= _has(row, key, v)
                elif op == "$ne":
                    ok &= not _has(row, key, v)
                elif op == "$in":
                    ok &= any(_has(row, key, x) for x in v)
                elif op == "$nin":
                    ok &= not any(_has(row, key, x) for x in v)
                elif op == "$not":
                    ok &= not mql_eval({key: v}, row)
    return ok


CATS = ["fraud", "waste", "abuse", "eligibility", "duplicate"]
TITLES = ["Hazard Mitigation", "Public Assistance", "Individual Assistance", "Debris"]


def random_rows(g, n):
    rows = []
    for _ in range(n):
        r = {}
        if g.random() < 0.9:
            r["fraud_categories"] = [c for c in CATS if g.random() < 0.35]
        if g.random() < 0.85:
            r["title"] = TITLES[int(g.integers(len(TITLES)))]
        if g.random() < 0.8:
            r["flag"] = bool(g.random() < 0.5)
        if g.random() < 0.8:
            r["section"] = int(g.integers(4))
        r["other"] = "ignored"
        rows.append(r)
    return rows


FILTERS = [
    {},
    {"title": "Debris"},
    {"title": {"$eq": "Debris"}},
    {"fraud_categories": "fraud"},
    {"fraud_categories": {"$ne": "fraud"}},
    {"title": {"$ne": "Debris"}, "flag": True},
    {"fraud_categories": {"$in": ["waste", "abuse"]}},
    {"fraud_categories": {"$nin": ["waste", "abuse"]}},
    {"title": {"$not": {"$eq": "Public Assistance"}}},
    {"title": {"$not": {"$in": ["Public Assistance", "Debris"]}}},
    {"$nor": [{"title": "Debris"}, {"fraud_categories": "fraud"}, {"section": {"$in": [0, 1]}}]},
    {"$or": [{"title": "Debris"}, {"fraud_categories": "duplicate"}, {"flag": False}]},
    {"$and": [{"fraud_categories": "fraud"}, {"fraud_categories": "waste"}, {"section": {"$ne": 2}}]},
    {"$or": [{"title": "Debris"}, {"flag": True}], "fraud_categories": {"$in": ["fraud", "waste"]}, "section": 3},
    {"section": 1, "flag": False},
    {"section": True},                                    # bool is not int: no row has section == True
    {"flag": 1},
    {"title": "Unseen Title"},                            # unseen value under $eq: NEVER
    {"title": {"$in": []}},                               # empty $in: NEVER
    {"title": {"$in": ["Unseen", "Debris"]}},
    {"title": {"$ne": "Unseen"}},                         # $ne of an unseen value: no constraint
    {"fraud_categories": {"$nin": ["unseen"]}},
    {"$or": [{"title": "Unseen"}, {"section": 99}]},      # every branch unseen: NEVER
]


@pytest.mark.parametrize("i", range(len(FILTERS)))
def test_compiled_filter_equals_direct_mql_evaluation(i):
    g = np.random.default_rng(11 + i)
    rows = random_rows(g, 400)
    schema = FilterSchema(("fraud_categories", "title", "flag", "section"))
    tags = schema.tags(rows)
    f = compile_filter(schema, FILTERS[i])
    got = filter_pass(tags, f)
    ref = np.array([mql_eval(FILTERS[i], r) for r in rows])
    assert (got == ref).all(), (FILTERS[i], np.flatnonzero(got != ref)[:5])
    if FILTERS[i] in ({"title": "Unseen Title"}, {"title": {"$in": []}}, {"$or": [{"title": "Unseen"}, {"section": 99}]}):
        assert not got.any() and (f & NEVER).any()


def test_compiled_forms():
    s = FilterSchema(("a", "b"))
    s.tags([{"a": ["x", "y"], "b": True}, {"a": "z", "b": 3}])
    bx, by, bz = (1 << s.bit("a", v) for v in ("x", "y", "z"))
    bt, b3 = 1 << s.bit("b", True), 1 << s.bit("b", 3)
    assert [s.bit("a", "x"), s.bit("a", "y"), s.bit("b", True), s.bit("a", "z"), s.bit("b", 3)] == [0, 1, 2, 3, 4]
    assert compile_filter(s, {"a": "x"}).tolist() == [bx, 0, 0, 0]
    assert compile_filter(s, {"a": {"$nin": ["x", "z"]}}).tolist() == [0, bx | bz, 0, 0]
    assert compile_filter(s, {"a": {"$in": ["x", "z"]}}).tolist() == [0, 0, bx | bz, 0]
    assert compile_filter(s, {"$or": [{"a": "y"}, {"b": 3}], "a": {"$in": ["x"]}}).tolist() == [0, 0, by | b3, bx]
    assert compile_filter(s, {"$nor": [{"a": "y"}, {"b": {"$in": [True]}}]}).tolist() == [0, by | bt, 0, 0]
    assert compile_filter(s, None).tolist() == [0, 0, 0, 0]


@pytest.mark.parametrize("doc,msg", [
    ({"a": {"$gt": "x"}}, "range"),
    ({"a": {"$lte": 3}}, "range"),
    ({"a": {"$eq": None}}, "null"),
    ({"a": None}, "null"),
    ({"c": "x"}, "not a filter field"),
    ({"a": {"$in": ["x"]}, "b": {"$in": [3]}, "$or": [{"a": "y"}]}, "at most 2"),
    ({"$or": [{"a": "x", "b": 3}, {"a": "y"}]}, "single-field"),
    ({"$or": [{"$and": [{"a": "x"}]}]}, "single-field"),
    ({"a": {"$regex": "x"}}, "not supported"),
    ({"a": ["x", "y"]}, "array"),
    ({"a": {"$not": {"$ne": "x"}}}, "\\$not"),
])
def test_refusals(doc, msg):
    s = FilterSchema(("a", "b"))
    s.tags([{"a": ["x", "y"], "b": 3}])
    with pytest.raises(ValueError, match=msg):
        compile_filter(s, doc)


def test_schema_is_deterministic_and_refuses_overflow_before_mutating():
    rows = random_rows(np.random.default_rng(3), 200)
    a, b = FilterSchema(("title", "fraud_categories")), FilterSchema(("title", "fraud_categories"))
    ta, tb = a.tags(rows), b.tags(rows)
    assert (ta == tb).all() and a.to_json() == b.to_json()
    assert FilterSchema.from_json(json.loads(json.dumps(a.to_json()))).bits == a.bits
    assert a.to_json()["bits"][0][0] == "title" or rows[0].get("title") is None
    s = FilterSchema(("tag", "kind"))
    s.tags([{"tag": f"v{i}"} for i in range(60)])
    before = dict(s.bits)
    with pytest.raises(ValueError, match="'kind'"):
        s.tags([{"tag": "v0", "kind": [f"k{i}" for i in range(4)]}])     # 60 + 4 > 63
    assert s.bits == before
    t = s.tags([{"kind": ["k0", "k1", "k2"], "tag": None}, {}])            # exactly 63; null and missing get no bit
    assert len(s) == 63 and int(t[1]) == 0 and int(t[0]) >> 63 == 0
    with pytest.raises(ValueError, match="not a string, bool or int"):
        FilterSchema(("x",)).tags([{"x": 1.5}])


class FakeIndex:
    """The VectorTable interface with tags, on the CPU: records what the table writes."""

    def __init__(self, similarity="cosine"):
        self.similarity = similarity
        self.n = 0
        self.tags = np.zeros(0, np.uint64)

    def __len__(self):
        return self.n

    def append(self, rows, tags=None):
        first = self.n
        self.n += len(rows)
        self.tags = np.concatenate([self.tags, np.zeros(len(rows), np.uint64) if tags is None else tags])
        return first

    def set_tags(self, rows, tags):
        self.tags[np.asarray(rows)] = tags

    def delete_rows(self, rows):
        pass

    def reset(self):
        self.n = 0
        self.tags = np.zeros(0, np.uint64)


def test_table_checkpoint_round_trip_and_mismatch(tmp_path):
    from qsa_b200.operator import VectorTable
    rows = random_rows(np.random.default_rng(9), 50)
    t = VectorTable(FakeIndex(), filter_fields=("fraud_categories", "title"))
    t.upsert_many([f"d{i}" for i in range(50)], ["c"] * 50, np.zeros((50, 8), np.float32), rows)
    want = t.index.tags.copy()
    assert (want == t.filter_schema.tags(rows)).all()
    t.save(str(tmp_path))
    man = json.load(open(tmp_path / "manifest.json"))
    assert man["filter_fields"] == ["fraud_categories", "title"] and len(man["filter_bits"]) == len(t.filter_schema)
    ix2 = FakeIndex()
    ix2.append(np.zeros((50, 8), np.float32))                  # the vectors are already in the index (bulk load)
    t2 = VectorTable(ix2, filter_fields=("fraud_categories", "title"))
    assert t2.load(str(tmp_path)) == 50
    assert (ix2.tags == want).all() and t2.filter_schema.bits == t.filter_schema.bits
    with pytest.raises(ValueError, match="filter fields"):
        VectorTable(FakeIndex(), filter_fields=("title",)).load(str(tmp_path))
    # an older checkpoint without filter fields: tags are rebuilt from its metadata column
    del man["filter_fields"], man["filter_bits"]
    json.dump(man, open(tmp_path / "manifest.json", "w"))
    ix3 = FakeIndex()
    ix3.append(np.zeros((50, 8), np.float32))
    t3 = VectorTable(ix3, filter_fields=("fraud_categories", "title"))
    t3.load(str(tmp_path))
    assert (ix3.tags == want).all()


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_the_independent_fixture(path):
    z = np.load(path)
    k = int(z["k"])
    ok = eligibility(z["tags"], z["filters"])
    assert (ok == z["eligible"]).all()
    assert not np.isin(z["cosine_idx"][0], z["excluded_top_query0"]).any()
    for sim, key in (("cosine", "cosine"), ("dotProduct", "dot"), ("euclidean", "euclidean")):
        s, i = topk_f64(z["query_bits"], z["corpus_bits"], k, sim, ok)
        assert (i == z[f"{key}_idx"]).all(), sim
        fin = np.isfinite(z[f"{key}_score"])
        assert (np.abs(s - z[f"{key}_score"])[fin] < 1e-9).all()


def test_bench_harness_exact_topk_equals_the_definitions():
    """The bench harnesses' exact_topk (fp32 prefilter per piece + float64 rescoring) over bench.HostData at three
    pieces equals similarity_oracle.topk_f64 per similarity and, with filters, filter_oracle.topk_f64 -- including a
    filter no row passes."""
    import bench
    from harness import similarity_oracle
    from harness.similarity_bench import PIECE, exact_topk
    from oracle import bruteforce as bf
    n, dim, nq, k, seed = 2 * PIECE + 1000, 64, 6, 12, 5
    tags = np.random.default_rng(seed).integers(0, 4, n).astype(np.uint64)
    filters = {"bit0": np.tile(np.array([1, 0, 0, 0], np.uint64), (nq, 1)),
               "none": np.tile(np.array([8, 0, 0, 0], np.uint64), (nq, 1))}
    host = bench.HostData(n * dim * 2, 2)
    try:
        host.generate(seed, dim, 0, n, n)
        c_bits = host.view(n, dim)
        q_bits = bf.synth_queries(seed + 1, nq, dim, c_bits[:1000])
        plain = exact_topk(host, q_bits, n, dim, k)
        filtered = exact_topk(host, q_bits, n, dim, k, similarity_oracle.SIMILARITIES, (tags, filters))
        for sim in similarity_oracle.SIMILARITIES:
            assert (plain[sim] == similarity_oracle.topk_f64(q_bits, c_bits, k, sim)[1]).all(), sim
            for case, f in filters.items():
                want = topk_f64(q_bits, c_bits, k, sim, eligibility(tags, f))[1]
                assert (filtered[(sim, case)] == want).all(), (sim, case)
        assert (filtered[("cosine", "none")] == -1).all()
    finally:
        host.close()
