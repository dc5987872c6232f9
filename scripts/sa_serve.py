#!/usr/bin/env python3
"""sa_serve -- run the Lab2 topic graph locally on the GPUs of this box.

Consumes ``documents`` / ``queries`` (and pre-embedded ``documents_embed`` / ``queries_embed``) from the topic log,
keeps the vector table in HBM, writes ``search_results`` and ``search_results_response``
(replaces the Flink statements of terraform/lab2-vector-search/main.tf:233-331).  Needs a CUDA device.

    python -m scripts.sa_serve --log-dir .sa_topics --once          # drain what is there, then exit
    python -m scripts.sa_serve --capacity 2000000 --k 3             # run until interrupted
    python -m scripts.sa_serve --gpus 8 --capacity 1250000          # corpus row-sharded over 8 GPUs, one process

The vector table is volatile (HBM).  Without ``--snapshot-dir`` every start rebuilds it by re-reading the durable
``documents_embed`` topic from its beginning; with it, the table is checkpointed (atomically, every
``--snapshot-every`` seconds while it changes, and on exit / SIGTERM) together with the ``documents_embed`` offsets it
covers, and a restart resumes exactly there.
"""
from __future__ import annotations

import argparse
import json
import signal
import sys

try:
    from ._local import resolve_log_dir, setup_logging
except ImportError:
    from _local import resolve_log_dir, setup_logging


def _k_arg(v: str) -> int:
    """VECTOR_SEARCH_AGG k: 1 .. SA_MAX_K (64; searches with k > 28 run the deep scan variant)."""
    from qsa_b200 import capi    # constants only: loads no library
    k = int(v)
    if not 1 <= k <= capi.SA_MAX_K:
        raise argparse.ArgumentTypeError(f"k must be in [1, {capi.SA_MAX_K}], not {k}")
    return k


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--log-dir", default=None)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--capacity", type=int, default=1 << 20, help="rows of HBM to reserve for the vector table (per GPU)")
    ap.add_argument("--max-batch", type=int, default=1024)
    ap.add_argument("--k", type=_k_arg, default=3,
                    help="VECTOR_SEARCH_AGG k, 1 .. 64 (the reference uses 3; search_results carries the first 3)")
    ap.add_argument("--gpus", type=int, default=1,
                    help="row-shard the table over this many GPUs of the box (one process, NCCL all-gather of the per-shard "
                         "candidates inside libsa_b200.so: sa_comm_create / sa_gather_merge)")
    ap.add_argument("--similarity", default="cosine", choices=["cosine", "dotProduct", "euclidean"],
                    help="the vector index's similarity, as in an Atlas index definition (the reference declares cosine, "
                         "assets/pre-setup/MongoDB-Setup.md:72-83); fixed for the table and recorded in its checkpoints")
    ap.add_argument("--score-mode", default="cosine", choices=["cosine", "atlas"],
                    help="score_i on search_results: the raw score of the similarity (cosine, dot product, Euclidean "
                         "distance), or the value MongoDB Atlas reports: (1 + s) / 2, or 1 / (1 + d) for euclidean; "
                         "the ranking is the same")
    ap.add_argument("--lateral", action="append", default=[], choices=["lab3", "lab4"],
                    help="also run the operator joined onto an upstream stream, over the same table: lab3 = "
                         "anomalies_per_zone -> anomalies_enriched (LAB3-Walkthrough.md:225-375), lab4 = claims_to_investigate "
                         "-> claims_to_investigate_with_policies (LAB4-Walkthrough.md:251-309); repeatable")
    ap.add_argument("--once", action="store_true", help="process everything pending, print stats, exit")
    ap.add_argument("--snapshot-dir", default=None,
                    help="checkpoint directory: loaded at start if it holds a checkpoint, written periodically and on exit")
    ap.add_argument("--snapshot-every", type=float, default=30.0, help="seconds between checkpoints while the table changes")
    ap.add_argument("--metrics-file", default=None, help="append one JSON line of batch-latency p50/p99 and QPS every few seconds")
    ap.add_argument("--verbose", action="store_true")
    return ap


def main(argv=None) -> int:
    a = build_parser().parse_args(argv)
    setup_logging(a.verbose)

    from qsa_b200 import engine as engine_mod  # CUDA only; raises without a device (no CPU fallback)
    from qsa_b200.operator import VectorTable
    from qsa_b200.pipeline.serve import Lab2Pipeline

    sim = {} if a.similarity == "cosine" else {"similarity": a.similarity}   # cosine is every index's default
    if a.gpus > 1:
        from qsa_b200.sharded import MultiGpuIndex
        index = MultiGpuIndex(dim=a.dim, capacity_per_gpu=a.capacity, max_batch=a.max_batch, max_k=max(a.k, 3), n_gpus=a.gpus,
                              **sim)
    else:
        index = engine_mod.VectorIndex(dim=a.dim, capacity=a.capacity, max_batch=a.max_batch, max_k=max(a.k, 3), **sim)
    table = VectorTable(index)
    if a.snapshot_dir and VectorTable.has_checkpoint(a.snapshot_dir):
        print(f"resumed {table.load(a.snapshot_dir)} rows from {a.snapshot_dir} at {table.source_offsets}", file=sys.stderr)
    pipe = Lab2Pipeline(resolve_log_dir(a.log_dir), table, k=a.k, max_batch=a.max_batch, score_mode=a.score_mode,
                        metrics_file=a.metrics_file)
    if a.lateral:
        from qsa_b200.pipeline import lateral
        make = {"lab3": lateral.lab3_anomalies_enriched, "lab4": lateral.lab4_claims_with_policies}
        for name in a.lateral:
            pipe.extra_stages.append(make[name](pipe.log_dir, table, score_mode=a.score_mode, max_batch=a.max_batch))

    def on_term(signum, frame):      # SIGTERM takes the same exit path as Ctrl-C: stats, final checkpoint
        raise KeyboardInterrupt
    try:
        signal.signal(signal.SIGTERM, on_term)
    except ValueError:               # not the main thread (tests)
        pass
    try:
        if a.once:
            pipe.run_until_idle()
            print(json.dumps(pipe.stats))
        else:
            pipe.run_forever(snapshot_dir=a.snapshot_dir, snapshot_every_s=a.snapshot_every)
    except KeyboardInterrupt:
        print(json.dumps(pipe.stats))
    finally:
        if a.snapshot_dir:
            pipe.snapshot(a.snapshot_dir)
        if a.metrics_file:
            pipe.write_metrics()
    return 0


if __name__ == "__main__":
    sys.exit(main())
