"""dotProduct and euclidean similarity of the vector index, on a CPU box: the oracle against independent implementations
and fixtures, the C ABI's argument check, the Atlas score conversions, the native encoder, checkpoints and snapshots,
the sharded merge direction and the serve CLI.  The GPU side is tests/test_gpu_similarity.py."""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest
import torch
from scipy.spatial.distance import cdist

from harness.similarity_oracle import merge_shard_topk, topk_f64
from oracle import bruteforce as bf
from qsa_b200 import capi
from qsa_b200.operator import VectorTable, atlas_score, vector_search_agg, wire_score_mode
from qsa_b200.pipeline.serve import Codec, Lab2Pipeline
from qsa_b200.transport.filelog import Consumer, Producer

from doubles import PipelinedOracleIndex

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "similarity_topk_independent_*.npz")))


class SimOracleIndex(PipelinedOracleIndex):
    """Oracle-backed double of engine.VectorIndex for any similarity, with tombstones and engine-style snapshots."""

    def __init__(self, dim, capacity=1 << 20, similarity="cosine"):
        super().__init__(dim, capacity)
        self.similarity = similarity
        self.live = np.zeros(0, dtype=bool)

    def append(self, rows_f32):
        first = super().append(rows_f32)
        self.live = np.concatenate([self.live, np.ones(len(self.bits) - first, dtype=bool)])
        return first

    def reset(self):
        super().reset()
        self.live = np.zeros(0, dtype=bool)

    def delete_rows(self, rows):
        super().delete_rows(rows)
        self.live[list(rows)] = False

    def search_host(self, q_f32, k):
        s, i = topk_f64(bf.f32_to_bf16_bits(np.asarray(q_f32, dtype=np.float32)), self.bits, k, self.similarity,
                        live=self.live)
        return s.astype(np.float32), i.astype(np.int32)

    def snapshot(self, path):
        np.savez(path, rows=self.bits, live=self.live, similarity=np.str_(self.similarity))
        return len(self.bits)

    def restore(self, path):
        z = np.load(path)
        sim = str(z["similarity"]) if "similarity" in z.files else "cosine"
        if sim != self.similarity:
            raise ValueError(f"snapshot has similarity {sim!r}, index has {self.similarity!r}")
        self.bits, self.live = z["rows"], z["live"]
        return len(self.bits)


def _data(seed, n, dim, nq):
    c = bf.synth_rows(seed, 0, n, dim)
    c[3] = 0                                                 # an all-zero row: live for dotProduct and euclidean
    c[10] = c[20]                                            # duplicates
    c[30] = bf.f32_to_bf16_bits(bf.bf16_bits_to_f32(c[40]) * 8)   # a scaled copy
    q = bf.synth_queries(seed + 1, nq, dim, c)
    q[0] = 0
    q[1] = c[20]
    return q, c


# ---------------------------------------------------------------------------------------------------------- oracle
def test_topk_f64_agrees_with_scipy_numpy_and_torch():
    q, c = _data(5, 900, 128, 17)
    k = 12
    qf, cf = bf.bf16_bits_to_f32(q).astype(np.float64), bf.bf16_bits_to_f32(c).astype(np.float64)
    live = np.ones(len(c), bool)
    live[[50, 51, 20]] = False                               # tombstones, one of them a duplicate
    rows = np.arange(len(c))

    s, i = topk_f64(q, c, k, "euclidean", live=live)
    d = cdist(qf, cf, "euclidean")
    sq = cdist(qf, cf, "sqeuclidean")
    dt = torch.cdist(torch.from_numpy(qf), torch.from_numpy(cf), compute_mode="donot_use_mm_for_euclid_dist").numpy()
    assert np.array_equal(np.sqrt(sq), d) and np.allclose(d, dt, rtol=1e-12, atol=0)
    d[:, ~live] = np.inf
    ref_i = np.stack([np.lexsort((rows, x))[:k] for x in d])
    assert (i == ref_i).all()
    assert np.array_equal(s, np.take_along_axis(d, ref_i, axis=1))          # bit-exact: the sums are exact here
    assert not np.isin(i, [50, 51, 20]).any() and (i[1, 0] == 10) and s[1, 0] == 0.0
    assert (i[0, :1] == 3).all() and s[0, 0] == 0.0                         # zero query: the zero row is at distance 0

    s, i = topk_f64(q, c, k, "dotProduct", live=live)
    dots = qf @ cf.T
    assert np.array_equal(dots, (torch.from_numpy(qf) @ torch.from_numpy(cf).T).numpy())
    dots[:, ~live] = -np.inf
    ref_i = np.stack([np.lexsort((rows, -x))[:k] for x in dots])
    assert (i == ref_i).all() and np.array_equal(s, np.take_along_axis(dots, ref_i, axis=1))
    assert i[0].tolist() == [j for j in range(k + 3) if live[j]][:k] and (s[0] == 0).all()   # zero query: lowest rows
    assert 30 in i[1] or 30 in topk_f64(q[1:2], c, 40, "dotProduct")[1]    # the scaled copy outranks its original

    # cosine through the same entry point is the cosine oracle
    s, i = topk_f64(q, c, k, "cosine")
    rs, ri = bf.cosine_topk_f64(q, c, k)
    assert (i == ri).all() and np.array_equal(s, rs)
    with pytest.raises(ValueError):
        topk_f64(q, c, k, "manhattan")


def test_scaled_copies_rank_differently_than_under_cosine():
    q, c = _data(9, 300, 64, 4)
    c[100] = bf.f32_to_bf16_bits(bf.bf16_bits_to_f32(c[200]) * 4)
    q[2] = c[200]
    _, ic = topk_f64(q[2:3], c, 2, "cosine")
    _, idot = topk_f64(q[2:3], c, 1, "dotProduct")
    _, ieu = topk_f64(q[2:3], c, 1, "euclidean")
    assert set(ic[0]) == {100, 200} and ic[0, 0] == 100               # equal cosines: the lower row first
    assert idot[0, 0] == 100 and ieu[0, 0] == 200                     # 4x longer wins the dot, the copy itself is at 0


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_reproduces_independent_similarity_fixtures(path):
    z = np.load(path)
    k = int(z["k"])
    assert os.path.getsize(path) < 1 << 20
    for sim, key in (("dotProduct", "dot"), ("euclidean", "euclidean")):
        s, i = topk_f64(z["query_bits"], z["corpus_bits"], k, sim)
        assert (i == z[f"{key}_idx"]).all(), sim
        assert np.array_equal(s, z[f"{key}_score"]), sim


def test_golden_fixtures_exist():
    assert len(GOLDEN) == 2


def test_merge_shard_topk_orders_distances_ascending():
    s = [np.array([[0.5, 2.0, np.inf]]), np.array([[0.5, 1.0, 3.0]])]
    r = [np.array([[4, 1, -1]]), np.array([[0, 2, 5]])]
    ms, mi = merge_shard_topk(s, r, [0, 100], 4, descending=False)
    assert mi.tolist() == [[4, 100, 102, 1]] and ms.tolist() == [[0.5, 0.5, 1.0, 2.0]]
    ms, mi = merge_shard_topk(s, r, [0, 100], 6, descending=False)
    assert mi[0, -1] == -1 and ms[0, -1] == np.inf
    ds, di = merge_shard_topk(s, r, [0, 100], 2)                     # default: today's direction
    assert di.tolist() == [[105, 1]]


# --------------------------------------------------------------------------------------------------------- C ABI
def test_bad_similarity_is_rejected_before_touching_a_device(lib):
    h = C.c_void_p()
    for bad in (-1, 3, 99):
        assert lib.sa_engine_create_sim(C.byref(h), 0, 128, 1000, 128, 10, bad) == capi.SA_ERR_ARG
        assert b"similarity" in lib.sa_last_error()
        assert not h.value
    assert capi.similarity_code("dotProduct") == capi.SA_SIM_DOT == 1
    assert capi.similarity_code("euclidean") == capi.SA_SIM_EUCLIDEAN == 2
    assert capi.similarity_code("cosine") == capi.SA_SIM_COSINE == 0
    with pytest.raises(ValueError):
        capi.similarity_code("dot")
    from qsa_b200.engine import VectorIndex
    with pytest.raises(ValueError):
        VectorIndex(dim=64, capacity=256, similarity="l2")            # refused before any device work


def test_header_declares_the_similarity_constants():
    text = open(os.path.join(HERE, "..", "include", "sa_api.h")).read()
    for name, v in (("SA_SIM_COSINE", 0), ("SA_SIM_DOT", 1), ("SA_SIM_EUCLIDEAN", 2)):
        assert f"#define {name} {v}" in text


# ---------------------------------------------------------------------------------------------------------- Atlas
def test_atlas_conversions():
    assert atlas_score(0.5) == 0.75 and atlas_score(-1.0, "cosine") == 0.0
    assert atlas_score(3.0, "dotProduct") == 2.0 and atlas_score(-3.0, "dotProduct") == -1.0
    assert atlas_score(0.0, "euclidean") == 1.0 and atlas_score(3.0, "euclidean") == 0.25
    with pytest.raises(ValueError):
        atlas_score(1.0, "hamming")
    assert wire_score_mode("cosine", "euclidean") == 0
    assert wire_score_mode("atlas", "cosine") == 1 and wire_score_mode("atlas", "dotProduct") == 1
    assert wire_score_mode("atlas", "euclidean") == 2


def test_vector_search_agg_scores_per_similarity():
    g = np.random.default_rng(3)
    for sim in ("dotProduct", "euclidean"):
        table = VectorTable(SimOracleIndex(64, similarity=sim))
        emb = g.standard_normal((30, 64)).astype(np.float32)
        table.upsert_many([f"d{i}" for i in range(30)], [f"c{i}" for i in range(30)], emb)
        raw = vector_search_agg(table, "embedding", emb[:3], 4)
        atl = vector_search_agg(table, "embedding", emb[:3], 4, score_mode="atlas")
        for hr, ha in zip(raw, atl):
            assert [h.row for h in hr] == [h.row for h in ha]
            for a, b in zip(hr, ha):
                assert b.score == pytest.approx(atlas_score(a.score, sim))
        if sim == "euclidean":
            assert raw[0][0].row == 0 and raw[0][0].score == 0.0 and atl[0][0].score == 1.0
            assert all(x.score <= y.score for x, y in zip(raw[1], raw[1][1:]))     # distances ascend
    with pytest.raises(ValueError):
        vector_search_agg(table, "embedding", emb[:1], 2, score_mode="dot")


def test_native_encoder_score_mode_2_equals_the_generic_codec(tmp_path):
    from test_cli_and_pipeline import _odd_queries_embed_records
    dim = 64
    outs = {}
    for name in ("generic", "native"):
        logd = str(tmp_path / name)
        table = VectorTable(SimOracleIndex(dim, similarity="euclidean"))
        gg = np.random.default_rng(12)
        table.upsert_many([f"d{i}" if i % 7 else None for i in range(50)], [f"chunk {i}" if i % 5 else None for i in range(50)],
                          gg.standard_normal((50, dim)).astype(np.float32))
        table.upsert_many(["d3"], ["replaced"], gg.standard_normal((1, dim)).astype(np.float32))   # a tombstone
        pipe = Lab2Pipeline(logd, table, k=5, max_batch=7, native=(name == "native"), score_mode="atlas")
        assert (pipe._wire is not None) == (name == "native")
        p = Producer({"log.dir": logd})
        for raw in _odd_queries_embed_records(pipe.codec, dim, np.random.default_rng(13)):
            p.produce("queries_embed", value=raw)
        p.produce("queries_embed", value=None)
        p.flush()
        assert pipe.stage_search() == 13
        pipe.producer.flush()
        c = Consumer({"log.dir": logd, "group.id": "t"})
        c.subscribe(["search_results"])
        outs[name] = [m.value() for m in c.consume(100, 0.0)]
    assert outs["native"] == outs["generic"] and len(outs["native"]) == 7
    recs = [Codec(str(tmp_path / "native")).decode(v) for v in outs["native"]]
    scores = [r[f"score_{j}"] for r in recs for j in (1, 2, 3) if r[f"score_{j}"] is not None]
    assert scores and all(0 < s <= 1 for s in scores)                # 1 / (1 + d)
    assert all(r["document_id_1"] != "d3" or r["chunk_1"] == "replaced" for r in recs)


# ------------------------------------------------------------------------------------------ checkpoint / snapshot
def test_checkpoint_records_the_similarity_and_refuses_a_mismatch(tmp_path):
    g = np.random.default_rng(1)
    emb = g.standard_normal((12, 32)).astype(np.float32)
    t = VectorTable(SimOracleIndex(32, similarity="euclidean"))
    t.upsert_many([f"d{i}" for i in range(12)], [f"c{i}" for i in range(12)], emb)
    t.upsert_many(["d4"], ["new"], emb[:1])                          # tombstones row 4
    t.save(str(tmp_path / "ck"))
    man = json.load(open(tmp_path / "ck" / "manifest.json"))
    assert man["similarity"] == "euclidean"
    t2 = VectorTable(SimOracleIndex(32, similarity="euclidean"))
    assert t2.load(str(tmp_path / "ck")) == 13
    a = vector_search_agg(t, "embedding", emb[:4], 5)
    b = vector_search_agg(t2, "embedding", emb[:4], 5)
    assert [[h.row for h in x] for x in a] == [[h.row for h in x] for x in b]
    assert all(h.row != 4 for x in b for h in x)
    for other in ("cosine", "dotProduct"):
        with pytest.raises(ValueError, match="similarity"):
            VectorTable(SimOracleIndex(32, similarity=other)).load(str(tmp_path / "ck"))
    # a manifest from before similarities were recorded is a cosine checkpoint
    man.pop("similarity")
    json.dump(man, open(tmp_path / "ck" / "manifest.json", "w"))
    with pytest.raises(ValueError, match="similarity"):
        VectorTable(SimOracleIndex(32, similarity="euclidean")).load(str(tmp_path / "ck"))
    with pytest.raises(ValueError, match="similarity"):                # the index snapshot itself says euclidean
        VectorTable(SimOracleIndex(32, similarity="cosine")).load(str(tmp_path / "ck"))


def test_index_snapshot_refuses_another_similarity(tmp_path):
    ix = SimOracleIndex(16, similarity="dotProduct")
    ix.append(np.ones((3, 16), np.float32))
    ix.snapshot(str(tmp_path / "s.npz"))
    assert SimOracleIndex(16, similarity="dotProduct").restore(str(tmp_path / "s.npz")) == 3
    with pytest.raises(ValueError):
        SimOracleIndex(16, similarity="euclidean").restore(str(tmp_path / "s.npz"))


def test_sharded_index_passes_the_similarity_through():
    from qsa_b200.sharded import ShardedIndex
    assert ShardedIndex(SimOracleIndex(8, similarity="euclidean"), 0).similarity == "euclidean"
    assert ShardedIndex(PipelinedOracleIndex(8), 0).similarity == "cosine"


# -------------------------------------------------------------------------------------------------------------- CLI
def test_sa_serve_similarity_flag(tmp_path, capsys, monkeypatch):
    import qsa_b200.engine as engine_mod
    from scripts import sa_serve
    p = sa_serve.build_parser()
    assert p.parse_args([]).similarity == "cosine"
    assert p.parse_args(["--similarity", "dotProduct"]).similarity == "dotProduct"
    assert p.parse_args(["--similarity", "euclidean", "--score-mode", "atlas"]).score_mode == "atlas"
    with pytest.raises(SystemExit):
        p.parse_args(["--similarity", "dot"])
    capsys.readouterr()
    made = []

    class Index(SimOracleIndex):
        def __init__(self, dim=1536, capacity=0, max_batch=0, max_k=0, device=None, similarity="cosine"):
            super().__init__(dim, capacity, similarity)
            made.append(similarity)

    monkeypatch.setattr(engine_mod, "VectorIndex", Index)
    logd = str(tmp_path / "topics")
    assert sa_serve.main(["--log-dir", logd, "--once", "--dim", "64", "--similarity", "euclidean"]) == 0
    assert made == ["euclidean"]
