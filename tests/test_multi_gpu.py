"""The multi-GPU exchange inside the C ABI (include/sa_api.h "multi-GPU": sa_comm_*, sa_gather_merge*, sa_sharded_search*),
against the unsharded oracle.  One-GPU boxes run the single-rank forms (a communicator of one still goes through NCCL);
the 2-rank tests need two GPUs and skip otherwise."""
import json
import os
import socket
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def n_gpus():
    import torch
    return torch.cuda.device_count()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("n", [1, 2, 4])
def test_single_process_gather_merge_equals_oracle(n):
    """sa_comm_create (ncclCommInitAll) + sa_gather_merge[_submit/_wait]: shards on n devices, host queries in, merged
    host results out, two batches in flight."""
    if n_gpus() < n:
        pytest.skip(f"needs {n} GPUs")
    from oracle import bruteforce as bf
    from qsa_b200.sharded import MultiGpuIndex
    dim, k = 256, 10
    g = np.random.default_rng(7)
    mi = MultiGpuIndex(dim=dim, capacity_per_gpu=6000, max_batch=300, max_k=k, n_gpus=n)
    parts = [g.standard_normal((m, dim)).astype(np.float32) for m in (1500, 700, 1, 2200, 900)]
    firsts = [mi.append(p) for p in parts]
    assert firsts == [0, 1500, 2200, 2201, 4401] and len(mi) == 5301
    c = bf.f32_to_bf16_bits(np.concatenate(parts))
    batches = [bf.synth_queries(20 + j, nq, dim, c) for j, nq in enumerate((300, 37, 128))]
    refs = [bf.cosine_topk_f64(q, c, k) for q in batches]
    f32 = [bf.bf16_bits_to_f32(q) for q in batches]
    s, i = mi.search_host(f32[0], k)
    assert (i == refs[0][1]).all() and np.abs(s.astype(np.float64) - refs[0][0]).max() < 1e-6
    mi.search_host_submit(f32[1], k, 0)
    mi.search_host_submit(f32[2], k, 1)
    for slot, j in ((0, 1), (1, 2)):
        s, i = mi.search_host_wait(slot)
        assert (i == refs[j][1]).all() and np.abs(s.astype(np.float64) - refs[j][0]).max() < 1e-6
    # filtered, host call and submit / wait: each shard filters its own rows by their tags
    from harness.filter_oracle import eligibility, topk_f64
    tags = g.integers(0, 4, len(mi)).astype(np.uint64)
    mi.set_tags(np.arange(len(mi)), tags)
    f = np.zeros((37, 4), np.uint64)
    f[:, 0], f[::2, 1] = 1, 2
    want = topk_f64(batches[1], c, k, "cosine", eligibility(tags, f))[1]
    assert (mi.search_host(f32[1], k, filters=f)[1] == want).all()
    mi.search_host_submit(f32[1], k, 1, filters=f)
    out = (np.empty((37, k), np.float32), np.empty((37, k), np.int64))
    assert mi.search_host_wait(1, out=out)[1] is out[1] and (out[1] == want).all()
    mi.delete_rows([int(refs[0][1][0, 0])])                       # tombstone the best hit of query 0: the runner-up moves up
    s, i = mi.search_host(f32[0][:1], k)
    assert i[0, 0] == refs[0][1][0, 1]
    mi.reset()
    assert len(mi) == 0 and (mi.search_host(f32[1], k)[1] == -1).all()
    mi.close()


@pytest.mark.parametrize("gpus", [1, 2])
def test_sa_serve_cli_multi_gpu(tmp_path, capsys, gpus):
    """`sa_serve --gpus N --once`: the Lab2 topic graph with the table row-sharded over N GPUs of one process."""
    if n_gpus() < gpus:
        pytest.skip(f"needs {gpus} GPUs")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_cli_and_pipeline import write_docs
    from qsa_b200.pipeline.serve import Codec
    from qsa_b200.transport.filelog import Consumer
    from scripts import lab2_publish_queries, publish_docs, sa_serve
    docs, logd = tmp_path / "docs", str(tmp_path / "topics")
    write_docs(docs, 60)
    assert publish_docs.main(["--docs-dir", str(docs), "--log-dir", logd]) == 0
    for q in ("How do tumble windows work?", "What about watermarks?"):
        assert lab2_publish_queries.main([q, "--log-dir", logd]) == 0
    capsys.readouterr()
    args = ["--log-dir", logd, "--once", "--capacity", "1024", "--max-batch", "64", "--k", "3", "--score-mode", "atlas",
            "--metrics-file", str(tmp_path / "m.jsonl")]
    if gpus > 1:
        args += ["--gpus", str(gpus)]
    assert sa_serve.main(args) == 0
    stats = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert stats["documents"] == 61 and stats["searches"] == 2 and stats["responses"] == 2 and stats["quarantined"] == 0
    c = Consumer({"log.dir": logd, "group.id": "t"}); c.subscribe(["search_results"])
    rows = [Codec(logd).decode(m.value()) for m in c.consume(10, 0.0)]
    assert [r["query"] for r in rows] == ["How do tumble windows work?", "What about watermarks?"]
    assert "window functions" in rows[0]["chunk_1"].lower() and all(0.5 <= r["score_1"] <= 1.0 for r in rows)
    assert json.loads(open(tmp_path / "m.jsonl").readline())["queries"] >= 1


def _rank_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    from oracle import bruteforce as bf
    from qsa_b200.engine import VectorIndex
    from qsa_b200.sharded import ShardedIndex, shard_bounds
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    n, dim, k = 40000, 1536, 10
    c = bf.synth_rows(41, 0, n, dim)
    c[n - 5] = c[3]                                   # a tie that straddles the shard boundary
    lo, hi = shard_bounds(n, world, rank)
    ix = VectorIndex(dim=dim, capacity=hi - lo, max_batch=300, max_k=k, device=rank)
    ix.append_bf16_bits(c[lo:hi])
    sh = ShardedIndex(ix, row_offset=lo)
    assert sh.transport == "nccl" and sh._comm is not None
    out = {}
    for j, nq in enumerate((300, 9)):
        q = bf.synth_queries(42 + j, nq, dim, c)
        q[0] = c[3]
        qd = torch.from_numpy(q.view(np.int16)).view(torch.bfloat16).cuda()
        s, gi = sh.search(qd, k)                     # device form: sa_sharded_search
        torch.cuda.synchronize()
        out[f"s{j}"], out[f"i{j}"] = s.cpu().numpy(), gi.cpu().numpy()
        sh.search_host_submit(bf.bf16_bits_to_f32(q), k, j & 1)      # host form, both slots in flight
    for j in range(2):
        hs, hi_ = sh.search_host_wait(j & 1)
        out[f"hs{j}"], out[f"hi{j}"] = hs, hi_
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **out)
    dist.barrier()
    sh.close()
    ix.close()
    dist.destroy_process_group()


def test_two_rank_sharded_search_through_the_c_abi(tmp_path):
    """One process per GPU (the bench's launch form): communicator from sa_comm_create_rank, one packed all-gather."""
    if n_gpus() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from oracle import bruteforce as bf
    world = 2
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    n, dim, k = 40000, 1536, 10
    c = bf.synth_rows(41, 0, n, dim)
    c[n - 5] = c[3]
    r = [np.load(tmp_path / f"rank{i}.npz") for i in range(world)]
    for j, nq in enumerate((300, 9)):
        q = bf.synth_queries(42 + j, nq, dim, c)
        q[0] = c[3]
        rs, ri = bf.cosine_topk_f64(q, c, k)
        for rk in r:
            assert (rk[f"i{j}"] == ri).all() and (rk[f"hi{j}"] == ri).all()       # every rank ends with the global answer
            assert np.abs(rk[f"s{j}"].astype(np.float64) - rs).max() < 1e-6
            assert np.abs(rk[f"hs{j}"].astype(np.float64) - rs).max() < 1e-6
        assert ri[0, 0] == 3 and ri[0, 1] == n - 5                                # lower global row wins the cross-shard tie
