#!/usr/bin/env python3
"""Search throughput and exactness under each similarity of the index (cosine, dotProduct, euclidean).

For each shape (rows x dim, batch B, top-k) the corpus is generated once with bench.py's recipe (HostData + upload: the
canonical numpy chunk 0, the rest from the device generator, mirrored to the host for the oracle) and searched under
all three similarities with the same warmup / steps discipline as bench.py: W untimed batches, then K timed batches
between CUDA events.  One JSON line per (shape, similarity):

    qps, ms_per_batch, scan_ms (mean of the scan kernels per batch), recall and strict_order against the float64
    definition (tests/harness/similarity_oracle semantics, over ALL rows: fp32 prefilter + float64 rescoring, see
    exact_topk) for a sample of the batch's queries,
    last_fix_entries from a separate untimed search with count_fix = 1, and the GPU's name and power limit.

    python tests/harness/similarity_bench.py                                 # 1M x 1536 (B 256) and 10M x 1536 (B 1024), k 10
    python tests/harness/similarity_bench.py --shapes 1000000x1536x256 --steps 20 --warmup 3
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bench  # noqa: E402
from harness.filter_oracle import eligibility  # noqa: E402
from harness.similarity_oracle import SIMILARITIES, RunningTopk, internal_scores  # noqa: E402

PIECE = 65_536
PROG = os.path.splitext(os.path.basename(sys.argv[0]))[0]


def _w_prefilter(task):
    """fp32 prefilter of one piece of the shared corpus: per (similarity, case), the piece's `keep` best eligible rows
    per query, with their fp32 values (-inf: not eligible)."""
    from oracle import bruteforce as bf
    q_bits, first, off, rows, dim, keep, sims, tags, filters = task
    q = bf.bf16_bits_to_f32(q_bits)
    c = bf.bf16_bits_to_f32(bench._shared_view(off, rows, dim))
    dots = (q @ c.T).astype(np.float64)
    qq = (q.astype(np.float64) ** 2).sum(axis=1)
    cc = np.einsum("ij,ij->i", c, c, dtype=np.float64)
    out = {}
    for sim in sims:
        s0 = internal_scores(sim, dots, qq, cc)
        for case, f in filters.items():
            s = s0
            if f is not None:
                s = s0.copy()
                s[~eligibility(tags, f)] = -np.inf
            kk = min(keep, s.shape[1])
            part = np.argpartition(s, s.shape[1] - kk, axis=1)[:, s.shape[1] - kk:]
            out[(sim, case)] = (part.astype(np.int64) + first, np.take_along_axis(s, part, axis=1))
    return out


def exact_topk(host, q_bits, n_rows, dim, k, sims=SIMILARITIES, filtered=None, margin=64):
    """Row int64 [nq, k] (-1 = empty slot) of the float64 definition over all n_rows rows of the host copy, per
    similarity: {similarity: rows}; with ``filtered`` = (tags uint64 [n_rows], {case: filters uint64 [nq, 4] or None}),
    per similarity and case over each query's eligible rows: {(similarity, case): rows}.  An fp32 prefilter keeps
    k + margin rows per query and piece (spread over the pool), then those candidates are re-scored in float64 (the
    definition) and selected by (value desc, row asc).  Equal to the definition unless more than `margin` rows of one
    piece sit within fp32 rounding (~1e-6 relative) of a query's k-th value."""
    from oracle import bruteforce as bf
    tags, filters = filtered if filtered is not None else (None, {None: None})
    tasks = [(q_bits, lo, lo * dim * 2, min(PIECE, n_rows - lo), dim, k + margin, sims,
              None if tags is None else tags[lo:lo + PIECE], filters) for lo in range(0, n_rows, PIECE)]
    cand = {}
    for part in host.pool.imap_unordered(_w_prefilter, tasks, chunksize=1):
        for key, (rows, vals) in part.items():
            cand.setdefault(key, []).append(np.where(np.isfinite(vals), rows, -1))
    shard = host.view(n_rows, dim)
    q = bf.bf16_bits_to_f32(q_bits).astype(np.float64)
    out = {}
    for (sim, case), parts in cand.items():
        rows_all = np.concatenate(parts, axis=1)
        res = np.full((len(q), k), -1, dtype=np.int64)
        for r in range(len(q)):
            rows = np.unique(rows_all[r][rows_all[r] >= 0])
            if len(rows) == 0:
                continue
            c = bf.bf16_bits_to_f32(shard[rows]).astype(np.float64)
            acc = RunningTopk(1, k)
            s = internal_scores(sim, (c @ q[r])[None, :], np.array([q[r] @ q[r]]), (c * c).sum(axis=1))
            acc.add(s, 0)
            res[r] = np.where(acc.i[0] >= 0, rows[np.maximum(acc.i[0], 0)], -1)
        out[sim if filtered is None else (sim, case)] = res
    return out


def log(msg):
    print(f"[{PROG} {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def gpu_identity():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def indexes(host, n, dim, B, max_k, sims, a):
    """(similarity, index, q_bits, qd) per similarity over one corpus: bench.py's recipe uploaded into the first index
    (HostData + upload, mirrored to the host copy) and copied device to device into each next one, which closes the
    one before; bench.py's queries (odd ones planted near rows of the first chunk), as bf16 bits and on the device."""
    import torch
    from oracle import bruteforce as bf
    from qsa_b200.engine import VectorIndex
    prev = q_bits = qd = None
    for sim in sims:
        ix = VectorIndex(dim=dim, capacity=n, max_batch=B, max_k=max_k, similarity=sim)
        log(f"{n}x{dim} b{B}: {sim}")
        if prev is None:
            bench.upload(host, ix, torch, a.seed, dim, 0, n, n, a.data)
            q_bits = bf.synth_queries(a.seed + 1, B, dim, host.view(min(n, bench.CHUNK), dim))
            qd = torch.from_numpy(q_bits.view(np.int16)).view(torch.bfloat16).cuda()
        else:
            ix.rows[:n].copy_(prev.rows[:n])                   # the same bits, device to device
            prev.close()
            ix.commit(0, n)
        torch.cuda.synchronize()
        yield sim, ix, q_bits, qd
        prev = ix
    prev.close()


def timed_case(ix, qd, k, a, filters=None):
    """One case with bench.py's step discipline: the filters staged on the device once, W untimed searches, then K
    searches between CUDA events; the engine's mean scan and total ms over them; one more untimed search with
    count_fix = 1 for exactness and fallback work.  Returns (timing fields, last_fix_entries, its rows int64 [nq, k])."""
    import torch
    from qsa_b200.engine import stage_filters
    f = stage_filters(filters, qd.shape[0], qd.device)
    for _ in range(a.warmup):
        ix.search(qd, k, filters=f)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(a.steps):
        ix.search(qd, k, filters=f)
    ev1.record()
    torch.cuda.synchronize()
    ms = ev0.elapsed_time(ev1) / a.steps
    scan_ms, total_ms, _ = ix.timing_mean(min(a.steps, 16))
    ix.set_option("count_fix", 1)
    _, i = ix.search(qd, k, filters=f)
    torch.cuda.synchronize()
    fix = ix.info("last_fix_entries")
    ix.set_option("count_fix", 0)
    timing = {"qps": round(qd.shape[0] / (ms * 1e-3), 1), "ms_per_batch": round(ms, 3), "scan_ms": round(scan_ms, 3),
              "total_ms_engine": round(total_ms, 3)}
    return timing, int(fix), i.cpu().numpy().astype(np.int64)


def report(head, timing, fix, got, want, a, gpu, **tail):
    """Print a case's JSON line: ``head``, ``timing``, recall and strict order of the first len(want) result rows
    against ``want`` (-1 = empty slot), the run's settings and the GPU's (name, power limit), then ``tail``."""
    got = got[:len(want)]
    recall = float(np.mean([
        len(np.intersect1d(got[r][got[r] >= 0], want[r][want[r] >= 0])) / max(1, int((want[r] >= 0).sum()))
        for r in range(len(want))]))
    print(json.dumps({
        **head, **timing, "recall": recall, "strict_order": float((got == want).all(axis=1).mean()),
        "recall_queries": len(want), "last_fix_entries": fix, "steps": a.steps, "warmup": a.warmup, "data": a.data,
        "gpu": gpu[0], "power_limit_w": gpu[1], **tail}), flush=True)


def run_shape(host, n, dim, B, a, gpu):
    sample = min(a.sample, B)
    ref = None
    for sim, ix, q_bits, qd in indexes(host, n, dim, B, a.k, SIMILARITIES, a):
        if ref is None:
            log("uploaded; exact answers for the query sample")
            t0 = time.perf_counter()
            ref = exact_topk(host, q_bits[:sample], n, dim, a.k)
            oracle_s = time.perf_counter() - t0
            log(f"oracle {oracle_s:.0f} s")
        timing, fix, got = timed_case(ix, qd, a.k, a)
        report({"workload": f"{n}x{dim}_b{B}_k{a.k}", "similarity": sim}, timing, fix, got, ref[sim], a, gpu,
               oracle_s=round(oracle_s, 1))


def main(argv=None, doc=__doc__, run_shape=run_shape, shapes="1000000x1536x256,10000000x1536x1024",
         add_args=lambda ap: ap.add_argument("--k", type=int, default=10)) -> int:
    """The bench harnesses' command line: ``add_args`` adds a harness's own options, then ``run_shape(host, n, dim, B,
    args, (gpu name, power limit))`` runs for each ROWSxDIMxBATCH of --shapes over one shared host copy."""
    ap = argparse.ArgumentParser(description=doc, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default=shapes, help="ROWSxDIMxBATCH,...")
    add_args(ap)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sample", type=int, default=16, help="queries of the batch checked against the exact definition")
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--data", default="philox", choices=["philox", "numpy"], help="as bench.py's data modes")
    ap.add_argument("--workers", type=int, default=0)
    a = ap.parse_args(argv)
    shapes = [tuple(int(x) for x in s.split("x")) for s in a.shapes.split(",") if s]
    need = max(n * d * 2 for n, d, _ in shapes)
    host = bench.HostData(need, a.workers or bench.auto_workers(1, need, bench.host_memory_available()))
    try:
        import torch
        if not torch.cuda.is_available():
            raise SystemExit(f"{PROG} needs a CUDA device (H100); there is no CPU fallback")
        gpu = gpu_identity()
        for n, d, B in shapes:
            run_shape(host, n, d, B, a, gpu)
    finally:
        host.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
