#!/usr/bin/env python
"""bench.py -- the headline metric of BASELINE.json on this repo's engine.

    metric : RAG queries/sec, 10M x 1536 bf16 corpus, top-10 (cosine), recall@10 vs numpy
    step   : one batch of `--batch` queries searched against the whole corpus (VECTOR_SEARCH_AGG, reference call
             site terraform/lab2-vector-search/main.tf:292); the timed region is exactly `--steps` steps, after an
             untimed preheat that brings the GPU to its sustained clocks
    value  : whole-job queries/sec with the queries already resident in HBM (CUDA events, max over ranks)
    e2e    : same metric through the host-buffer C-ABI calls (H2D of the fp32 queries and D2H of the results inside
             the timed region, two batches in flight): sa_search_host_submit/_wait at N = 1,
             sa_sharded_search_host_submit/_wait (shard scan + NCCL all-gather + merge inside the library) at N > 1

N > 1 (torchrun, one rank per GPU): the corpus is row-sharded, every rank searches its shard, ONE NCCL all-gather of the
packed per-shard (cosine, global row) lists issued from inside libsa_b200.so, merge kernel on every rank ("strong"
scaling: the corpus and the batch are fixed as N grows).

Data (SURVEY.md section 8d): the corpus and the queries are the canonical numpy PCG64 recipe of oracle.synth_rows /
synth_queries (seeds 1234 / 4321; half of the queries planted next to rows of chunk 0), generated in 262 144-row chunks by
a pool of worker processes forked before CUDA is initialised, into one anonymous shared mapping that is both the H2D
source and what the CPU oracle reads: builder, judge and oracle see identical bits.

After the headline measurement the same process measures the other BASELINE.json configs (`extra_configs`: config 2,
config 4's batch and config 5's shard shape with streaming epochs), each with its own recall check and roofline.

`--dump-outputs DIR` writes what the last timed step returned (DIR/scores.npy float32, DIR/indices.npy float64, one
row per query) so that two builds can be compared output for output: the inputs are seeded and identical run to run.

`--impl reference` times the CPU arm instead: the numpy brute-force oracle (BASELINE.md section 4) with all host
threads on a bounded sample of the same workload.  It never touches the GPU engine.

Use of `oracle/` here: (i) the canonical DATA recipe (`synth_rows` / `synth_queries`, SURVEY.md section 8d) in the worker
pool, (ii) the recall / parity CHECKS after the timed regions, (iii) the CPU legs (`cpu_baseline`, `--impl reference`).
Nothing under `oracle/` is on any timed GPU path, and the engine never imports it.
"""
from __future__ import annotations

import argparse
import json
import math
import mmap
import os
import subprocess
import sys
import threading
import time

# torchrun exports OMP_NUM_THREADS=1 to its children; the CPU legs must be allowed every host thread, and OpenBLAS
# sizes its pool from the environment when numpy is first imported -- so fix the environment before that import.
if os.environ.get("RANK", "0") == "0":
    for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
        os.environ[_v] = str(os.cpu_count() or 1)
    os.environ.setdefault("OMP_PROC_BIND", "false")   # let the kernel spread BLAS threads over both sockets

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "rag_queries_per_sec_10Mx1536_top10"
UNIT = "queries/s"
CHUNK = 262_144           # rows per generation chunk (oracle.CHUNK_ROWS)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=1536)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--seed", type=int, default=1234, help="corpus seed (queries use --qseed)")
    ap.add_argument("--qseed", type=int, default=4321)
    ap.add_argument("--cta-group", type=int, default=0, help="0 auto, 1, 2")
    ap.add_argument("--no-share", action="store_true", help="disable cross-lane threshold sharing")
    ap.add_argument("--list-len", type=int, default=0, help="candidate list length (0 auto, 16, 32)")
    ap.add_argument("--pace-gain", type=int, default=-1, help="drift-control gain (-1 = engine default, 0 = off)")
    ap.add_argument("--recall-queries", type=int, default=256, help="queries checked against numpy over ALL rows")
    ap.add_argument("--cpu-sample-queries", type=int, default=256)
    ap.add_argument("--cpu-sample-rows", type=int, default=524_288)
    ap.add_argument("--min-timed-s", type=float, default=2.0, help="minimum length of the Avro pipeline's timed region")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps, write the last step's results (scores.npy float32, indices.npy float64)")
    ap.add_argument("--preheat-max", type=float, default=6.0,
                    help="untimed back-to-back searches until the SM clock has been stable for 1 s (at most this long), so "
                         "the timed steps run at the sustained (power-capped) clocks the sustained peak was measured at")
    ap.add_argument("--workers", type=int, default=0, help="data-generation / oracle worker processes (0 = auto)")
    ap.add_argument("--no-cpu", action="store_true", help="skip cpu_baseline / recall (profiling runs)")
    ap.add_argument("--no-extra", action="store_true", help="skip the extra BASELINE configs")
    ap.add_argument("--no-pipeline", action="store_true", help="skip the Avro-in / Avro-out serve-stage measurement")
    ap.add_argument("--extra", default="cfg2,cfg4,cfg5", help="which extra configs to run")
    ap.add_argument("--data", default="numpy", choices=["numpy", "philox"],
                    help="philox: device generator for chunks >= 1 (quick profiling runs only; chunk 0 stays canonical)")
    return ap.parse_args()


def bits_to_f32(bits):
    """bf16 bit patterns (uint16) -> the float32 values they denote."""
    return (np.ascontiguousarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def workload_name(rows, dim, batch, k):
    return f"{rows}x{dim} bf16 corpus, batch {batch}, top-{k}, cosine"


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return {"hbm_gbs": d["hbm_gbs"], "tflops_burst": d["bf16_tflops"],
                "tflops_sustained": d.get("bf16_tflops_sustained", d["bf16_tflops"]), "source": "measured"}
    # H100 SXM data sheet (700 W part): HBM3 bandwidth and dense BF16 tensor rate -- ceilings, not measurements
    return {"hbm_gbs": 3350.0, "tflops_burst": 989.0, "tflops_sustained": 989.0, "source": "H100 SXM data sheet"}


# ----------------------------------------------------------------------------------------------------
# worker pool: canonical data generation and the oracle's per-chunk work (numpy only; never touches CUDA)
# ----------------------------------------------------------------------------------------------------
_SHARED = None      # (mmap, nbytes) inherited by the forked workers


def _w_init():
    for v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
        os.environ[v] = "1"
    try:
        from threadpoolctl import threadpool_limits
        threadpool_limits(1)
    except Exception:
        pass


def _shared_view(offset_bytes, rows, dim):
    return np.frombuffer(_SHARED[0], dtype=np.uint16, count=rows * dim, offset=offset_bytes).reshape(rows, dim)


def _w_gen(task):
    """Generate rows [lo, hi) of corpus (seed, dim) -- part of canonical chunk c -- into the shared mapping."""
    from oracle import bruteforce as bf
    seed, c, dim, chunk_rows, lo_in_chunk, hi_in_chunk, dst_off = task
    rows = bf.synth_rows(seed, c, chunk_rows, dim)     # the canonical chunk (its row count is part of the recipe)
    _shared_view(dst_off, hi_in_chunk - lo_in_chunk, dim)[:] = rows[lo_in_chunk:hi_in_chunk]
    return c


def _w_oracle(task):
    """Oracle prefilter of one chunk: k + margin candidates per query (fp32 sgemm), as oracle.cosine_topk_fast does."""
    from oracle import bruteforce as bf
    q_bits, first_row, off, rows, dim, keep = task
    bits = _shared_view(off, rows, dim)
    q = bf.bf16_bits_to_f32(q_bits)
    qn = np.sqrt((q.astype(np.float64) ** 2).sum(axis=1)).astype(np.float32)
    qh = q / np.where(qn > 0, qn, 1)[:, None]
    c = bf.bf16_bits_to_f32(bits)
    cn = np.sqrt(np.einsum("ij,ij->i", c, c, dtype=np.float32))
    inv = np.where(cn > 0, 1.0 / np.where(cn > 0, cn, 1), 0).astype(np.float32)
    s = (qh @ c.T) * inv[None, :]
    s[:, cn == 0] = -np.inf
    kk = min(keep, s.shape[1])
    part = np.argpartition(s, s.shape[1] - kk, axis=1)[:, s.shape[1] - kk:]
    return first_row, np.take_along_axis(s, part, axis=1), part.astype(np.int64)


class HostData:
    """The shared host copy of this rank's corpus shard + the worker pool.  Must be created before CUDA is initialised
    (the workers are forked)."""

    def __init__(self, nbytes, workers):
        global _SHARED
        import multiprocessing as mp
        self.nbytes = int(nbytes)
        self.mm = mmap.mmap(-1, max(self.nbytes, 4096))      # MAP_SHARED | MAP_ANONYMOUS
        _SHARED = (self.mm, self.nbytes)
        self.workers = workers
        self.pool = mp.get_context("fork").Pool(workers, initializer=_w_init)

    def view(self, rows, dim, offset_bytes=0):
        return _shared_view(offset_bytes, rows, dim)

    def generate(self, seed, dim, lo_row, hi_row, n_total, on_piece=None):
        """Fill the mapping with canonical rows [lo_row, hi_row) of the n_total-row corpus `seed` (chunk c of it is
        oracle.synth_rows(seed, c, min(CHUNK, n_total - c*CHUNK), dim)); calls on_piece(first_local_row, n) as pieces
        complete (out of order)."""
        tasks, pieces = [], {}
        for c in range(lo_row // CHUNK, (hi_row + CHUNK - 1) // CHUNK):
            a, b = max(lo_row, c * CHUNK), min(hi_row, (c + 1) * CHUNK)
            tasks.append((seed, c, dim, min(CHUNK, n_total - c * CHUNK), a - c * CHUNK, b - c * CHUNK, (a - lo_row) * dim * 2))
            pieces[c] = (a - lo_row, b - a)
        for c in self.pool.imap_unordered(_w_gen, tasks):
            if on_piece:
                on_piece(*pieces[c])

    def oracle_topk(self, q_bits, n_rows, dim, k, margin=32):
        """oracle.cosine_topk_fast over the shard in the mapping, the per-chunk prefilter spread over the pool."""
        from oracle import bruteforce as bf
        keep = k + margin
        piece = 65_536
        tasks = [(q_bits, lo, lo * dim * 2, min(piece, n_rows - lo), dim, keep) for lo in range(0, n_rows, piece)]
        nq = len(q_bits)
        cand_s = np.full((nq, keep), -np.inf, dtype=np.float32)
        cand_i = np.full((nq, keep), -1, dtype=np.int64)
        for first, ps, pi in self.pool.imap_unordered(_w_oracle, tasks, chunksize=1):
            cs = np.concatenate([cand_s, ps], axis=1)
            ci = np.concatenate([cand_i, pi + first], axis=1)
            order = np.lexsort((ci, -cs), axis=1)[:, :keep]
            cand_s = np.take_along_axis(cs, order, axis=1)
            cand_i = np.take_along_axis(ci, order, axis=1)
        shard = self.view(n_rows, dim)
        out_s = np.full((nq, k), -np.inf)
        out_i = np.full((nq, k), -1, dtype=np.int64)
        for r in range(nq):
            ok = cand_i[r] >= 0
            if not ok.any():
                continue
            rows = cand_i[r][ok]
            s64 = bf._rescore_f64(q_bits[r], shard[rows])
            fin = np.isfinite(s64)
            ts, ti = bf._select_topk(s64[fin], rows[fin], k)
            out_s[r, :len(ts)] = ts
            out_i[r, :len(ti)] = ti
        return out_s, out_i

    def close(self):
        self.pool.terminate()
        self.pool.join()


def host_memory_available():
    """Bytes this process may still use: MemAvailable, capped by the cgroup limit when there is one."""
    avail = None
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    avail = int(line.split()[1]) * 1024
    except OSError:
        pass
    for lim_p, cur_p in (("/sys/fs/cgroup/memory.max", "/sys/fs/cgroup/memory.current"),
                         ("/sys/fs/cgroup/memory/memory.limit_in_bytes", "/sys/fs/cgroup/memory/memory.usage_in_bytes")):
        try:
            lim = open(lim_p).read().strip()
            if lim != "max" and int(lim) < (1 << 60):
                room = int(lim) - int(open(cur_p).read().strip())
                avail = room if avail is None else min(avail, room)
        except (OSError, ValueError):
            pass
    return avail if avail is not None else 64 << 30


WORKER_PEAK_BYTES = 3 << 30      # one canonical chunk in fp32 (1.6 GB) + its bf16 copy + slack


def auto_workers(world, shared_bytes=0, mem_avail=None):
    """Worker processes per rank: bounded by the cores AND by memory -- every worker holds a whole 262144 x dim fp32
    chunk while it generates it, and the shared host copy of the shard has to fit beside them (a first version of this
    pool took a GPU box down by running 48 workers x 10 GB)."""
    n = os.cpu_count() or 8
    by_cpu = max(2, min(32, (n - 2 * world) // max(world, 1)))
    mem = (host_memory_available() if mem_avail is None else mem_avail) // max(world, 1)
    by_mem = int((0.6 * mem - shared_bytes) // WORKER_PEAK_BYTES)
    return max(1, min(by_cpu, by_mem))


# ----------------------------------------------------------------------------------------------------
# CPU arm (oracle; the only place besides tests/ and smoke() that touches oracle/)
# ----------------------------------------------------------------------------------------------------
def cpu_info():
    info = {"cores_logical": os.cpu_count()}
    try:
        out = subprocess.run(["lscpu"], capture_output=True, text=True, timeout=5).stdout
        for line in out.splitlines():
            for key, name in (("Model name", "model"), ("Socket(s)", "sockets"), ("NUMA node(s)", "numa_nodes"),
                              ("Core(s) per socket", "cores_per_socket")):
                if line.startswith(key + ":"):
                    info[name] = line.split(":", 1)[1].strip()
    except Exception:
        pass
    try:
        from threadpoolctl import threadpool_info
        info["blas"] = [{k: p.get(k) for k in ("internal_api", "version", "threading_layer", "num_threads")}
                        for p in threadpool_info() if p.get("user_api") == "blas"]
    except Exception:
        pass
    return info


def blas_all_threads():
    """Context manager: let numpy's BLAS use every host thread (torchrun exports OMP_NUM_THREADS=1 to its children,
    which would otherwise cripple the CPU arm).  Yields the thread count actually in effect."""
    import contextlib

    @contextlib.contextmanager
    def cm():
        n = os.cpu_count() or 1
        try:
            from threadpoolctl import threadpool_info, threadpool_limits
            with threadpool_limits(limits=n):
                got = [p.get("num_threads", 1) for p in threadpool_info() if p.get("user_api") == "blas"]
                yield max(got) if got else n
        except ImportError:
            yield int(os.environ.get("OMP_NUM_THREADS", n))
    return cm()


def cpu_sample_run(q_bits, prepared, k, full_rows):
    """Time numpy brute force on (queries x sample rows) over a corpus already resident in RAM as unit-norm fp32
    rows (ingest-time work, like the GPU engine's inverse norms, is not timed).  Returns (qps scaled to
    `full_rows`, seconds)."""
    from oracle import bruteforce as bf
    t0 = time.perf_counter()
    bf.cosine_topk_sgemm_prepared(q_bits, prepared, k)
    dt = time.perf_counter() - t0
    rows = sum(len(c) for _, c, _ in prepared)
    qps_full = (len(q_bits) * rows / dt) / full_rows
    return qps_full, dt


def cpu_baseline_block(q_bits, sample_chunks, k, full_rows, steps=1, warm=True):
    """The CPU leg: prepare (untimed), warm the BLAS pool, time `steps` passes; median QPS scaled to `full_rows`."""
    from oracle import bruteforce as bf
    prepared = bf.prepare_chunks_f32(sample_chunks)
    vals, dts = [], []
    with blas_all_threads() as cores:
        if warm:
            cpu_sample_run(q_bits[:max(8, len(q_bits) // 8)], prepared[:1], k, full_rows)
        for _ in range(steps):
            v, dt = cpu_sample_run(q_bits, prepared, k, full_rows)
            vals.append(v)
            dts.append(dt)
    rows = sum(len(c) for _, c, _ in prepared)
    sample = (f"{len(q_bits)} queries x {rows} rows per pass, {steps} pass(es), {np.mean(dts):.2f} s each (numpy fp32 sgemm "
              f"brute force over unit-norm fp32 rows in RAM; top-k selection "
              f"{'oracle/topk.c on all cores' if bf._topk_lib() is not None else 'numpy argpartition'}; QPS scaled by rows to "
              f"{full_rows})")
    return {"value": float(np.median(vals)), "unit": UNIT, "cores": cores, "kind": "port", "sample": sample,
            "spread": [float(min(vals)), float(max(vals))], "host": cpu_info()}, float(np.sum(dts))


def run_reference(a):
    """--impl reference: the reference's own (CPU) way of answering the query, per BASELINE.md section 4."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from oracle import bruteforce as bf
    nq, rows = a.cpu_sample_queries, a.cpu_sample_rows
    host = HostData(rows * a.dim * 2, min(auto_workers(1, rows * a.dim * 2), max(2, (rows + CHUNK - 1) // CHUNK)))
    host.generate(a.seed, a.dim, 0, rows, rows)
    host.close()
    shard = host.view(rows, a.dim)
    chunks = [(lo, shard[lo:lo + CHUNK]) for lo in range(0, rows, CHUNK)]
    q = bf.synth_queries(a.qseed, nq, a.dim, chunks[0][1])
    t0 = time.perf_counter()
    block, cpu_s = cpu_baseline_block(q, chunks, a.k, a.rows, steps=max(1, a.steps), warm=a.warmup > 0)
    v = block["value"]
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": a.gpus, "steps": a.steps,
        "warmup": a.warmup, "ms_per_step": cpu_s / max(1, a.steps) * 1e3, "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": "bf16",
        "data": f"synthetic (numpy PCG64, oracle.synth_rows seed {a.seed} / synth_queries seed {a.qseed}, half planted)",
        "config": {"workload": workload_name(a.rows, a.dim, a.batch, a.k), "k": a.k,
                   "cpu": "numpy fp32 sgemm brute force over unit-norm fp32 rows in RAM, all BLAS threads"},
        "cpu_baseline": block,
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "wall_s": time.perf_counter() - t0,
    }))


# ----------------------------------------------------------------------------------------------------
# clocks
# ----------------------------------------------------------------------------------------------------
class ClockSampler:
    """Samples SM clock, power and throttle reasons of one GPU every ~20 ms on a thread (NVML)."""

    def __init__(self, device_index):
        self.idx = device_index
        self.rows = []
        self._stop = threading.Event()
        self._t = None
        self._max = None

    def start(self):
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = int(vis.split(",")[self.idx]) if vis and vis.split(",")[self.idx].isdigit() else self.idx
            h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self._max = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
        except Exception:
            return
        R = pynvml

        def loop():
            while not self._stop.is_set():
                try:
                    sm = R.nvmlDeviceGetClockInfo(h, R.NVML_CLOCK_SM)
                    pw = R.nvmlDeviceGetPowerUsage(h) / 1000.0
                    rs = R.nvmlDeviceGetCurrentClocksEventReasons(h)
                    self.rows.append((time.perf_counter(), sm, pw, rs))
                except Exception:
                    pass
                time.sleep(0.02)

        self._t = threading.Thread(target=loop, daemon=True)
        self._t.start()

    def stop(self):
        self._stop.set()
        if self._t:
            self._t.join(timeout=1)

    def stable(self, window_s=1.0, tol_mhz=45):
        """Has the SM clock stayed within tol_mhz for the last window_s seconds?  (True without NVML.)"""
        if self._t is None:
            return True
        now = time.perf_counter()
        rows = [r[1] for r in self.rows if r[0] >= now - window_s]
        old = [r for r in self.rows if r[0] < now - window_s]
        return bool(old) and len(rows) >= 10 and (max(rows) - min(rows)) <= tol_mhz

    def summary(self, t0, t1):
        rows = [r for r in self.rows if t0 <= r[0] <= t1]
        if not rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        import pynvml as R
        names = {"hw_slowdown": R.nvmlClocksEventReasonHwSlowdown,
                 "hw_thermal_slowdown": R.nvmlClocksEventReasonHwThermalSlowdown,
                 "sw_thermal_slowdown": R.nvmlClocksEventReasonSwThermalSlowdown,
                 "sw_power_cap": R.nvmlClocksEventReasonSwPowerCap}
        reasons = sorted(n for n, bit in names.items() if any(r[3] & bit for r in rows))
        return {"sm_mhz": float(np.median([r[1] for r in rows])), "sm_max_mhz": float(self._max),
                "sm_mhz_min": float(min(r[1] for r in rows)), "sm_mhz_p90": float(np.percentile([r[1] for r in rows], 90)),
                "power_w_max": float(max(r[2] for r in rows)), "power_w_median": float(np.median([r[2] for r in rows])),
                "reasons": reasons, "samples": len(rows)}


# ----------------------------------------------------------------------------------------------------
# GPU arm
# ----------------------------------------------------------------------------------------------------
def collective_preheat(step, sync, stop_flags, world, all_reduce_max=None, chunk=4, max_chunks=100000):
    """Run `step` back to back, untimed, until `stop_flags()` -> (stable, time_up) says so.  With several ranks every
    step contains collectives, so all ranks MUST run the same number of steps: the loop proceeds in chunks of `chunk`
    steps and the decision to stop is itself a collective (every rank stable, or any rank out of time), never a per-rank
    clock.  Returns (steps run, seconds)."""
    n = 0
    t0 = time.perf_counter()
    for _ in range(max_chunks):
        for _ in range(chunk):
            step()
        n += chunk
        sync()
        stable, time_up = stop_flags()
        flags = [0 if stable else 1, 1 if time_up else 0]
        if world > 1:
            flags = all_reduce_max(flags)
        if flags[0] == 0 or flags[1] == 1:
            break
    return n, time.perf_counter() - t0


def _all_reduce_max_list(vals, dist, torch):
    t = torch.tensor(vals, device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.tolist()


def settle_and_estimate(step, sync, barrier, sampler, world, allmax, preheat_max, settle_s=1.5):
    """Bring the GPU to its sustained state and time a batch.  Returns (preheat seconds, preheat batches, seconds per
    batch).
      1. one-time costs first (NCCL connection set-up, first-use allocations): they must not reach any estimate -- a first
         version let them in, took 0.3 s for a batch, and timed a 0.06 s region at boost clocks;
      2. preheat (untimed) until the SM clock is stable UNDER LOAD: a 1 kW part boosts for the first second and then
         settles at its power cap; the roofline denominator (cuBLAS, 4 s back to back) is a settled number;
      3. seconds per batch from a short settled burst."""
    for _ in range(3):
        step()
    barrier()
    t_ph0 = time.perf_counter()

    def stop_flags():
        el = time.perf_counter() - t_ph0
        return (el >= settle_s and sampler.stable()), el >= preheat_max
    n_ph, ph_s = collective_preheat(step, sync, stop_flags, world, allmax)
    barrier()
    t_e0 = time.perf_counter()
    for _ in range(8):
        step()
    sync()
    est = (time.perf_counter() - t_e0) / 8
    if world > 1:
        est = allmax([est])[0]
    return ph_s, n_ph, est


class Workload:
    """One (corpus shard, batch, k) measurement on this rank's engine: device-resident loop, host-buffer e2e loops,
    scan-kernel event times, recall against the oracle."""

    def __init__(self, a, env, ix, sh, host, n_total, n_local, lo_row, dim, B, k, q_bits, name):
        self.a, self.env, self.ix, self.sh, self.host = a, env, ix, sh, host
        self.n_total, self.n_local, self.lo_row, self.dim, self.B, self.k = n_total, n_local, lo_row, dim, B, k
        self.q_bits, self.name = q_bits, name
        torch = env["torch"]
        self.q_bf16 = torch.from_numpy(q_bits.view(np.int16)).view(torch.bfloat16).cuda()
        from qsa_b200.engine import pinned_array
        qf = bits_to_f32(q_bits)
        self.q_host = [pinned_array((B, dim), np.float32) for _ in range(2)]
        for h in self.q_host:
            h[:] = qf
        idt = np.int32 if env["world"] == 1 else np.int64
        self.out_host = [(pinned_array((B, k), np.float32), pinned_array((B, k), idt)) for _ in range(2)]

    # -- one batch
    def step_device(self):
        if self.env["world"] == 1:
            return self.ix.search(self.q_bf16, self.k)
        return self.sh.search(self.q_bf16, self.k)     # shard scan -> one all-gather of packed hits -> merge (C ABI)

    def submit(self, i):
        if self.env["world"] == 1:
            self.ix.search_host_submit(self.q_host[i & 1], self.k, i & 1)
        else:
            self.sh.search_host_submit(self.q_host[i & 1], self.k, i & 1)

    def wait(self, i):
        if self.env["world"] == 1:
            return self.ix.search_host_wait(i & 1, out=self.out_host[i & 1])
        return self.sh.search_host_wait(i & 1, out=self.out_host[i & 1])

    def e2e_loop(self, n_batches, blocking=False):
        """n_batches through the host-buffer API; returns (seconds, last result).  Pipelined form: as a serving loop
        drives it, two slots keep one batch on the device while the next is submitted; every batch still moves its own
        queries host->device and its own results device->host inside the timed region."""
        env = self.env
        env["barrier"]()
        t0 = time.perf_counter()
        if blocking:
            for i in range(n_batches):
                self.submit(0)
                res = self.wait(0)
        else:
            self.submit(0)
            for i in range(1, n_batches):
                self.submit(i)
                self.wait(i - 1)
            res = self.wait(n_batches - 1)
        env["torch"].cuda.synchronize()
        env["barrier"]()
        return time.perf_counter() - t0, res

    def measure(self, steps, warmup, preheat_max, sampler):
        a, env = self.a, self.env
        torch = env["torch"]
        world = env["world"]
        ph_s, n_ph, est = settle_and_estimate(self.step_device, torch.cuda.synchronize, env["barrier"], sampler, world,
                                              env["allmax"], preheat_max)
        inner = 1   # batches per step
        # ---- warm-up steps
        for _ in range(warmup):
            out = self.step_device()
        env["barrier"]()

        t_region0 = time.perf_counter()
        for _ in range(2):
            self.submit(0)
            self.wait(0)
        n_a = inner * steps
        e2e_a, res_host = self.e2e_loop(n_a)
        for _ in range(warmup):   # back to back again: the timed device loop must not start from the e2e loop's tail
            out = self.step_device()

        # ---- timed: device-resident queries, exactly `steps` steps
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        env["barrier"]()
        t_w0 = time.perf_counter()
        ev0.record()
        for _ in range(steps * inner):
            out = self.step_device()
        ev1.record()
        env["barrier"]()
        t_w1 = time.perf_counter()
        ms_total = ev0.elapsed_time(ev1)
        t = self.ix.last_timing()
        # scan-kernel time: CUDA events recorded inside the C ABI on the launching stream around every scan launch of
        # the timed loop above (ring of the last 16 searches) -- back to back, no host synchronisation in between
        scan_ms_avg, total_ms_avg, n_timed = self.ix.timing_mean(min(steps * inner, 16))

        n_b = inner * steps
        e2e_b, res_host = self.e2e_loop(n_b)
        e2e_s = e2e_a + e2e_b            # the GPU drifts under its power cap: pool a loop before and one after
        nb = max(4, min(inner * steps, int(math.ceil(0.5 / max(est, 1e-9)))))
        e2e_blocking_s, res_host = self.e2e_loop(nb, blocking=True)   # diagnostic: a caller without pipelining
        t_region1 = time.perf_counter()
        clocks = sampler.summary(t_w0, t_w1)
        clocks_all = sampler.summary(t_region0, t_region1)

        if world > 1:
            ms_total, e2e_s, scan_ms_avg, total_ms_avg = env["allmax"]([ms_total, e2e_s, scan_ms_avg, total_ms_avg])
        nb_total = steps * inner
        nb_e2e = n_a + n_b
        B, k, dim, n_local = self.B, self.k, self.dim, self.n_local
        launches = t.launches
        kernels_per_batch = t.kernels
        peaks = measured_peaks()
        flops_launch = 2.0 * B * n_local * dim / launches
        bytes_launch = n_local * dim * 2.0 + n_local * 4.0 + (B * dim * 2.0 + B * k * 8.0) / launches
        t_launch = scan_ms_avg / launches * 1e-3
        ach_tf = flops_launch / t_launch / 1e12
        ach_gbs = bytes_launch / t_launch / 1e9
        ridge = peaks["tflops_sustained"] * 1e3 / peaks["hbm_gbs"]
        tensor_bound = (B / launches) >= ridge  # arithmetic intensity of a launch = its batch, flop/byte
        if tensor_bound:
            roof = {"bound": "tensor", "achieved": ach_tf, "peak": peaks["tflops_sustained"], "unit": "TFLOP/s",
                    "frac": ach_tf / peaks["tflops_sustained"],
                    "peak_kind": f"{peaks['source']} cuBLAS bf16 sustained (kernel timed inside a long step)"}
        else:
            roof = {"bound": "hbm", "achieved": ach_gbs, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                    "frac": ach_gbs / peaks["hbm_gbs"], "peak_kind": f"{peaks['source']} copy bandwidth"}
        roof.update({"algorithmic_bytes": bytes_launch, "algorithmic_flops": flops_launch,
                     "kernel": "sa_scan_kernel", "launch_ms": t_launch * 1e3, "launches_per_batch": launches,
                     "launches_timed": n_timed * launches, "achieved_gbs": ach_gbs, "achieved_tflops": ach_tf,
                     "hbm_frac": ach_gbs / peaks["hbm_gbs"], "tensor_frac_sustained": ach_tf / peaks["tflops_sustained"],
                     "tensor_frac_burst": ach_tf / peaks["tflops_burst"],
                     "scan_share_of_step": scan_ms_avg / (ms_total / nb_total),
                     "search_ms_events": total_ms_avg})
        idb = 4 if world == 1 else 8
        return {
            "workload": self.name, "value": B * nb_total / (ms_total * 1e-3), "unit": UNIT,
            "ms_per_batch": ms_total / nb_total, "batches_per_step": inner, "timed_region_s": ms_total * 1e-3,
            "preheat_s": ph_s, "preheat_batches": n_ph,
            "e2e": {"value": B * nb_e2e / e2e_s, "unit": UNIT, "h2d_bytes_per_step": B * dim * 4 * inner,
                    "d2h_bytes_per_step": B * k * (4 + idb) * inner, "timed_region_s": e2e_s, "batches": nb_e2e,
                    "blocking_value": B * nb / e2e_blocking_s,
                    "api": ("sa_search_host_submit/_wait" if world == 1 else "sa_sharded_search_host_submit/_wait") +
                           " (C ABI: host fp32 queries in, host results out, page-locked buffers, 2 batches in flight)"
                           "; blocking_value = one batch at a time"},
            "gpu_launches_per_batch": kernels_per_batch, "clocks": clocks, "clocks_whole_region": clocks_all,
            "roofline": roof,
        }, out, res_host, ms_total, nb_total

    def recall(self, out, res_host, nrq):
        """Engine answer vs the oracle over ALL rows for the first nrq queries (half of them planted).  N > 1: every
        rank runs the oracle over ITS shard, the per-shard oracle lists are gathered and merged on the CPU, and rank 0
        compares; also checks that every rank ended with the same answer and the e2e path agrees."""
        from oracle import bruteforce as bf
        env = self.env
        torch, dist, world, rank = env["torch"], env["dist"], env["world"], env["rank"]
        nrq = min(nrq, self.B)
        got_s, got_i = [x.cpu().numpy() for x in out]
        t0 = time.perf_counter()
        rs, ri = self.host.oracle_topk(self.q_bits[:nrq], self.n_local, self.dim, self.k)
        if world > 1:
            ts = torch.from_numpy(rs).cuda()
            ti = torch.from_numpy(np.where(ri >= 0, ri + self.lo_row, -1)).cuda()
            all_s = [torch.empty_like(ts) for _ in range(world)]
            all_i = [torch.empty_like(ti) for _ in range(world)]
            dist.all_gather(all_s, ts)
            dist.all_gather(all_i, ti)
            mine = torch.from_numpy(got_i.astype(np.int64)).cuda()
            ref0 = mine.clone()
            dist.broadcast(ref0, src=0)
            same = torch.tensor([int(torch.equal(mine, ref0))], device="cuda")
            dist.all_reduce(same, op=dist.ReduceOp.MIN)
            if rank != 0:
                return None
            rs, ri = bf.merge_shard_topk([x.cpu().numpy() for x in all_s], [x.cpu().numpy() for x in all_i],
                                         [0] * world, self.k)
        rep = bf.compare_topk(got_i[:nrq], got_s[:nrq], ri, rs)
        rep_host = bf.compare_topk(res_host[1][:nrq], res_host[0][:nrq], ri, rs)
        planted_ok = None
        if self.lo_row == 0 and self.n_local >= min(CHUNK, self.n_total):
            n0 = min(CHUNK, self.n_total)
            odd = np.arange(1, self.B, 2)
            planted_ok = float(np.mean(got_i[odd, 0] == [(i * 2654435761) % n0 for i in odd]))
        r = {"queries_checked": nrq, "rows": self.n_total, "recall_at_k": rep["recall"], "strict_order": rep["strict_order"],
             "max_abs_dscore": rep["max_abs_dscore"], "e2e_strict_order": rep_host["strict_order"],
             "planted_top1_all_queries": planted_ok, "oracle_s": time.perf_counter() - t0}
        if world > 1:
            r["all_ranks_same_answer"] = bool(same.item())
        return r


def dump_outputs(path, out):
    """What the timed path returned to its caller in its last step: the top-k cosines (float32) and rows (float64,
    exact), one row per query of the batch."""
    os.makedirs(path, exist_ok=True)
    scores, rows = (t.cpu().numpy() for t in out)
    np.save(os.path.join(path, "scores.npy"), scores.astype(np.float32))
    np.save(os.path.join(path, "indices.npy"), rows.astype(np.float64))


def pipeline_e2e(env, index_like, n_total, dim, B, k, q_bits, est_batch_s, min_timed_s, check_rows=None):
    """QPS_e2e as SURVEY.md section 8d defines it: Confluent-framed Avro `queries_embed` records on the file-log transport
    in, `search_results` records out -- read, decode, H2D, search, D2H, encode, append, commit -- through the product's own
    serve stage (pipeline/serve.py::Lab2Pipeline.stage_search, native batch codecs of include/sa_wire.h).  Every rank
    reads its own copy of the same topic, so the sharded search's collectives pair up; all ranks end with the same output.
    The table's non-vector columns are synthetic fixed-width strings ("doc-<row>" / a 96-byte chunk naming the row)."""
    import ctypes as C
    import shutil
    import tempfile
    from qsa_b200 import capi
    from qsa_b200.operator import VectorTable
    from qsa_b200.pipeline.serve import Codec, Lab2Pipeline
    from qsa_b200.transport.filelog import Consumer
    torch, rank, world = env["torch"], env["rank"], env["world"]
    lib = capi.load()
    logd = tempfile.mkdtemp(prefix=f"sa_bench_topics_r{rank}_")
    try:
        # ---- side table: rows -> pre-serialised Avro ["null","string"] values, built without a Python loop
        table = VectorTable(index_like)
        digits = ((np.arange(n_total, dtype=np.int64)[:, None] // 10 ** np.arange(8, -1, -1)) % 10 + 48).astype(np.uint8)

        def fixed(prefix: bytes, pad: bytes):
            body_len = len(prefix) + 9 + len(pad)
            assert body_len < 64                     # one-byte Avro length
            m = np.empty((n_total, 2 + body_len), np.uint8)
            m[:, 0], m[:, 1] = 2, body_len << 1
            m[:, 2:2 + len(prefix)] = np.frombuffer(prefix, np.uint8)
            m[:, 2 + len(prefix):2 + len(prefix) + 9] = digits
            if pad:
                m[:, 2 + len(prefix) + 9:] = np.frombuffer(pad, np.uint8)
            return m.reshape(-1), np.arange(n_total + 1, dtype=np.uint64) * np.uint64(2 + body_len)
        for arena, (data, off) in ((table.arena_document_id, fixed(b"doc-", b"")),
                                   (table.arena_chunk, fixed(b"chunk of row ", b" lorem ipsum dolor sit amet, consectetur."))):
            arena.data, arena.off, arena.n, arena.used = data, off, n_total, len(data)
        table.document_id = range(n_total)           # len(table) == n_total; the native stage reads the arenas only
        pipe = Lab2Pipeline(logd, table, k=k, max_batch=B, native=True, group=f"bench-r{rank}")
        # ---- the input topic: n_batches x B records, encoded and framed natively, one append per batch
        n_batches = max(4, int(math.ceil(min_timed_s / max(est_batch_s, 1e-6))))
        n_batches = min(n_batches, 256)
        vec = np.ascontiguousarray(bits_to_f32(q_bits))
        texts = [f"question {i}".encode() for i in range(B)]
        tbuf = b"".join(texts)
        tlen = np.array([len(t) for t in texts], np.uint32)
        toff = np.concatenate([[0], np.cumsum(tlen[:-1], dtype=np.uint64)]).astype(np.uint64)
        rec_off = np.empty(B + 1, np.uint64)
        need = C.c_uint64()
        sid = pipe.codec.schema_id("queries_embed")
        lib.sa_wire_encode_queries_embed(B, dim, sid, tbuf, toff.ctypes.data, tlen.ctypes.data, vec.ctypes.data, 0, None, 0,
                                         rec_off.ctypes.data, C.byref(need))
        out = np.empty(int(need.value), np.uint8)
        capi.check(lib.sa_wire_encode_queries_embed(B, dim, sid, tbuf, toff.ctypes.data, tlen.ctypes.data, vec.ctypes.data,
                                                    int(time.time() * 1000), out.ctypes.data, out.size, rec_off.ctypes.data,
                                                    C.byref(need)), "sa_wire_encode_queries_embed")
        for _ in range(n_batches + 2):
            pipe.producer.produce_framed("queries_embed", out.data, rec_off[:B])
        # ---- warm-up on two batches (also page-locks the staging buffers), then the timed drain
        pipe.max_batch = B
        c = pipe.consumers["queries_embed"]
        real_consume = c.consume_raw
        budget = [2]

        def limited(nmax, out=None):
            if budget[0] <= 0:
                return None
            budget[0] -= 1
            return real_consume(nmax, out)
        c.consume_raw = limited
        assert pipe.stage_search() == 2 * B
        c.consume_raw = real_consume
        env["barrier"]()
        t0 = time.perf_counter()
        moved = pipe.stage_search()
        torch.cuda.synchronize()
        env["barrier"]()
        dt = time.perf_counter() - t0
        if world > 1:
            dt = env["allmax"]([dt])[0]
        assert moved == n_batches * B, (moved, n_batches, B)
        res = {"value": moved / dt, "unit": UNIT, "records": moved, "batches": n_batches, "timed_region_s": dt,
               "bytes_in_per_record": int(rec_off[1]), "api": "Lab2Pipeline.stage_search over the file-log transport: "
               "consume_raw -> sa_wire_split_log / sa_wire_decode_queries_embed -> " +
               ("sa_search_host_submit/_wait" if world == 1 else "sa_sharded_search_host_submit/_wait") +
               " -> sa_wire_encode_search_results -> produce_framed -> commit",
               "batch_latency_ms": pipe.write_metrics()["batch_latency_ms"]}
        if rank == 0:
            cs = Consumer({"log.dir": logd, "group.id": "check"})
            cs.subscribe(["search_results"])
            msgs = cs.consume(B, 0.0)
            recs = [Codec(logd).decode(m.value()) for m in msgs[:64]]
            res["bytes_out_per_record"] = len(msgs[0].value())
            ok = all(r["query"] == f"question {i}" for i, r in enumerate(recs))
            if check_rows is not None:     # the same queries went through the device-resident loop: same rows expected
                ok = ok and all(r[f"document_id_{j + 1}"] == "doc-%09d" % check_rows[i][j] for i, r in enumerate(recs) for j in range(3))
            res["output_matches_device_path"] = bool(ok)
        return res
    finally:
        shutil.rmtree(logd, ignore_errors=True)


def upload(host, ix, torch, seed, dim, lo_row, hi_row, n_total, data_mode):
    """Generate rows [lo_row, hi_row) of corpus `seed` on the host pool and copy each piece to the device as it
    completes; commit.  data_mode == 'philox': only chunk 0 is canonical, the rest comes from the device generator."""
    n_local = hi_row - lo_row
    shard = host.view(n_local, dim)

    def on_piece(first, n):
        src = torch.from_numpy(shard[first:first + n].view(np.int16)).view(torch.bfloat16)
        ix.rows[first:first + n].copy_(src, non_blocking=False)

    if data_mode == "numpy":
        host.generate(seed, dim, lo_row, hi_row, n_total, on_piece)
    else:
        canon_hi = min(hi_row, max(lo_row, CHUNK))
        if canon_hi > lo_row:
            host.generate(seed, dim, lo_row, canon_hi, n_total, on_piece)
        g = torch.Generator(device="cuda").manual_seed(seed + 7919 * (lo_row // CHUNK + 1))
        for lo in range(canon_hi - lo_row, n_local, CHUNK):
            m = min(CHUNK, n_local - lo)
            x = torch.randn((m, dim), generator=g, device="cuda", dtype=torch.float32)
            x *= torch.exp(torch.empty((m, 1), device="cuda").uniform_(-0.7, 0.7, generator=g))
            ix.rows[lo:lo + m].copy_(x)
            shard[lo:lo + m] = ix.rows[lo:lo + m].view(torch.int16).cpu().numpy().view(np.uint16)   # the oracle's copy
    ix.commit(0, n_local)
    torch.cuda.synchronize()


def cublas_same_box(torch, seconds=1.5):
    """cuBLAS bf16 8192^3 back to back on this GPU, in the thermal state the bench left it in."""
    a = torch.randn((8192, 8192), device="cuda", dtype=torch.bfloat16)
    b = torch.randn((8192, 8192), device="cuda", dtype=torch.bfloat16)
    for _ in range(5):
        torch.matmul(a, b)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n, t0 = 0, time.perf_counter()
    ev0.record()
    while time.perf_counter() - t0 < seconds:
        for _ in range(20):
            torch.matmul(a, b)
        n += 20
        torch.cuda.synchronize()
    ev1.record()
    torch.cuda.synchronize()
    return 2.0 * 8192 ** 3 * n / (ev0.elapsed_time(ev1) * 1e-3) / 1e12


def run_b200(a):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world != a.gpus and world == 1 and a.gpus > 1:
        raise SystemExit("--gpus N>1 must be launched with torch.distributed.run (one rank per GPU)")
    t_start = time.perf_counter()
    extras = [] if a.no_extra else [x for x in a.extra.split(",") if x]
    n_total, dim, B, k = a.rows, a.dim, a.batch, a.k
    lo_row, hi_row = rank * n_total // world, (rank + 1) * n_total // world
    n_local = hi_row - lo_row
    # config 5: 50M x 768 over all GPUs (76.8 GB); a single 80 GB H100 holds half of it
    n5_total, dim5 = (50_000_000 if world > 1 else 25_000_000), 768
    lo5, hi5 = rank * n5_total // world, (rank + 1) * n5_total // world
    shared_bytes = n_local * dim * 2
    mem_avail = host_memory_available()
    notes = []
    if "cfg5" in extras and 0.6 * mem_avail / world < (hi5 - lo5) * dim5 * 2 + 2 * WORKER_PEAK_BYTES:
        extras.remove("cfg5")        # every rank decides alike: same box, same arithmetic
        notes.append(f"cfg5 skipped: its host copy ({(hi5 - lo5) * dim5 * 2 / 2**30:.0f} GiB per rank) does not fit in the "
                     f"{mem_avail / 2**30:.0f} GiB of host memory available")
    if "cfg5" in extras:
        shared_bytes = max(shared_bytes, (hi5 - lo5) * dim5 * 2)
    if 0.6 * mem_avail / world < shared_bytes + WORKER_PEAK_BYTES:
        raise SystemExit(f"bench.py needs {shared_bytes / 2**30:.0f} GiB of host memory per rank for the canonical corpus copy; "
                         f"{mem_avail / 2**30:.0f} GiB available for {world} rank(s)")
    # ---- host side first: the worker pool is forked before CUDA exists in this process
    n_workers = a.workers or auto_workers(world, shared_bytes, mem_avail)
    host = HostData(shared_bytes, n_workers)

    import torch
    import torch.distributed as dist
    from qsa_b200.engine import VectorIndex
    from qsa_b200.sharded import ShardedIndex
    from oracle import bruteforce as bf

    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    env = {"torch": torch, "dist": dist, "world": world, "rank": rank, "barrier": barrier,
           "allmax": (lambda v: _all_reduce_max_list(v, dist, torch)) if world > 1 else None}

    def bcast_queries(seed, nq, d, chunk0_bits):
        """Rank 0 (which holds chunk 0) builds the canonical query block; the others receive it."""
        if rank == 0:
            q = bf.synth_queries(seed, nq, d, chunk0_bits)
        if world == 1:
            return q
        # NCCL has no 16-bit integer type: ship the bit patterns as bytes
        t = (torch.from_numpy(q.view(np.uint8)).cuda() if rank == 0
             else torch.empty((nq, 2 * d), dtype=torch.uint8, device="cuda"))
        dist.broadcast(t, src=0)
        return np.ascontiguousarray(t.cpu().numpy()).view(np.uint16)

    maxB = max([B] + ([4096] if "cfg4" in extras else []))
    ix = VectorIndex(dim=dim, capacity=n_local, max_batch=maxB, max_k=k, device=local)
    if a.cta_group:
        ix.set_option("cta_group", a.cta_group)
    if a.pace_gain >= 0:
        ix.set_option("pace_gain", a.pace_gain)
    if a.list_len:
        ix.set_option("list_len", a.list_len)
    if a.no_share:
        ix.set_option("share_thresholds", 0)
    t_gen0 = time.perf_counter()
    upload(host, ix, torch, a.seed, dim, lo_row, hi_row, n_total, a.data)
    gen_s = time.perf_counter() - t_gen0
    chunk0 = host.view(n_local, dim)[:min(CHUNK, n_local)] if rank == 0 else None
    q_bits = bcast_queries(a.qseed, B, dim, chunk0)        # each batch size has its own canonical query block
    q_bits2 = bcast_queries(a.qseed, 256, dim, chunk0) if "cfg2" in extras and world == 1 else None
    q_bits4 = bcast_queries(a.qseed, 4096, dim, chunk0) if "cfg4" in extras else None
    sh = ShardedIndex(ix, row_offset=lo_row)

    sampler = ClockSampler(local)
    sampler.start()
    time.sleep(0.1)

    # ================================================================ headline
    wl = Workload(a, env, ix, sh, host, n_total, n_local, lo_row, dim, B, k, q_bits,
                  workload_name(n_total, dim, B, k))
    m, out, res_host, ms_total, nb_total = wl.measure(a.steps, a.warmup, a.preheat_max, sampler)
    result = None
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, out)
    if rank == 0:
        data_note = (f"synthetic, canonical numpy PCG64 (oracle.synth_rows seed {a.seed} per 262144-row chunk, rows not "
                     f"pre-normalised; oracle.synth_queries seed {a.qseed}, odd queries planted next to rows of chunk 0)")
        if a.data != "numpy":
            data_note += "; chunks >= 1 from the device Philox generator (--data philox, profiling only)"
        result = {
            "metric": METRIC, "value": m["value"], "unit": UNIT, "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": ms_total / a.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "bf16", "data": data_note,
            "config": {"workload": wl.name, "rows_per_gpu": n_local, "batch": B, "k": k, "dim": dim,
                       "parallelism": f"row-shard x{world}, one NCCL all-gather of packed hits inside the C ABI" if world > 1 else "single GPU",
                       "batches_per_step": m["batches_per_step"], "timed_region_s": m["timed_region_s"],
                       "l2": "inputs larger than L2 (corpus shard %.1f GB per batch)" % (n_local * dim * 2 / 1e9),
                       "cta_group": a.cta_group or "auto", "preheat": "until the SM clock is stable for 1 s "
                       f"(<= {a.preheat_max} s): {m['preheat_s']:.1f} s, {m['preheat_batches']} batches",
                       "data_generation_s": gen_s, "host": {"workers": n_workers, "mem_available_gib": mem_avail / 2**30,
                                                            "notes": notes}},
            "e2e": m["e2e"], "gpu_launches": int(m["gpu_launches_per_batch"] * nb_total),
            "clocks": m["clocks"], "clocks_whole_region": m["clocks_whole_region"], "roofline": m["roofline"],
        }

    # ---- QPS_e2e through the serve stage (Avro in, Avro out, file-log transport), same queries, same engine
    if not a.no_pipeline:
        try:
            rows_dev = out[1].cpu().numpy()
            pe = pipeline_e2e(env, ix if world == 1 else sh, n_total, dim, B, k, q_bits, m["ms_per_batch"] * 1e-3,
                              a.min_timed_s, check_rows=rows_dev)
            if rank == 0:
                result["e2e_pipeline"] = pe
        except Exception as exc:
            if world > 1:
                raise
            result["e2e_pipeline"] = {"error": f"{type(exc).__name__}: {exc}"}
    # ---- outside the timed region: recall vs numpy, cuBLAS on the same box, CPU baseline
    if not a.no_cpu:
        try:
            nrq = a.recall_queries if world == 1 else max(32, a.recall_queries // 4)
            rec = wl.recall(out, res_host, nrq)
            if rank == 0:
                result["recall"] = rec
        except Exception as exc:   # the measured line must still be printed; say what could not be checked
            if rank == 0:
                result["recall"] = None
                result["post_check_error"] = f"recall: {type(exc).__name__}: {exc}"
    if rank == 0:
        try:
            cb = cublas_same_box(torch)
            result["roofline"]["same_box"] = {
                "cublas_bf16_8192_tflops": cb, "scan_over_cublas": m["roofline"]["achieved_tflops"] / cb,
                "note": "torch.matmul bf16 8192^3 back to back for 1.5 s on this GPU right after the timed loops"}
        except Exception as exc:
            result["roofline"]["same_box"] = f"{type(exc).__name__}: {exc}"
    if world > 1:
        barrier()
    if rank == 0 and world == 1 and not a.no_cpu:
        try:
            nsq = min(a.cpu_sample_queries, B)
            srows = min(a.cpu_sample_rows, n_local)
            shard = host.view(n_local, dim)
            block, _ = cpu_baseline_block(q_bits[:nsq], [(lo, shard[lo:min(lo + CHUNK, srows)]) for lo in range(0, srows, CHUNK)],
                                          k, n_total, steps=2)
            result["cpu_baseline"] = block
        except Exception as exc:
            result["cpu_baseline"] = None
            result["post_check_error"] = result.get("post_check_error", "") + f" cpu: {type(exc).__name__}: {exc}"
    elif rank == 0:
        result.setdefault("cpu_baseline", None)

    # ================================================================ extra BASELINE configs
    extra_out = {}

    def run_extra(tag, fn):
        try:
            r = fn()
            if rank == 0:
                extra_out[tag] = r
        except Exception as exc:
            if rank == 0:
                extra_out[tag] = {"error": f"{type(exc).__name__}: {exc}"}
            if world > 1:
                raise   # ranks must not diverge inside collectives

    ex_steps, ex_ph = max(4, min(a.steps, 10)), min(a.preheat_max, 2.0)

    def finish(w, mm, o, rh, nrq):
        rec = None if a.no_cpu else w.recall(o, rh, nrq)
        if rank != 0:
            return None
        keep = {kk: mm[kk] for kk in ("workload", "value", "unit", "ms_per_batch", "batches_per_step", "timed_region_s", "e2e",
                                      "roofline", "clocks")}
        keep["recall"] = rec
        return keep

    if "cfg2" in extras and world == 1:
        def cfg2():
            n2 = min(1_000_000, n_local)
            ix.lib.sa_corpus_reset(ix._h)
            ix.commit(0, n2)                                   # config 2 = the first 1M rows of the same canonical corpus
            w = Workload(a, env, ix, sh, host, n2, n2, 0, dim, 256, k, q_bits2, workload_name(n2, dim, 256, k))
            mm, o, rh, _, _ = w.measure(ex_steps, a.warmup, ex_ph, sampler)
            r = finish(w, mm, o, rh, 64)
            ix.lib.sa_corpus_reset(ix._h)
            ix.commit(0, n_local)
            return r
        run_extra("cfg2_1Mx1536_b256", cfg2)
    if "cfg4" in extras:
        def cfg4():
            w = Workload(a, env, ix, sh, host, n_total, n_local, lo_row, dim, 4096, k, q_bits4,
                         workload_name(n_total, dim, 4096, k))
            mm, o, rh, _, _ = w.measure(ex_steps, a.warmup, ex_ph, sampler)
            return finish(w, mm, o, rh, 64 if world == 1 else 32)
        run_extra("cfg4_10Mx1536_b4096", cfg4)
    if "cfg5" in extras:
        def cfg5():
            nonlocal ix, sh
            sh.close()
            ix.close()
            wl.ix = wl.sh = ix = sh = None                      # drop the 10M-row shard before the config-5 one is built
            torch.cuda.empty_cache()
            n5 = hi5 - lo5
            ix5 = VectorIndex(dim=dim5, capacity=n5, max_batch=128, max_k=5, device=local)
            upload(host, ix5, torch, 5678, dim5, lo5, hi5, n5_total, a.data)
            c0 = host.view(n5, dim5)[:min(CHUNK, n5)] if rank == 0 else None
            q5 = bcast_queries(8765, 128, dim5, c0)
            sh5 = ShardedIndex(ix5, row_offset=lo5)
            w = Workload(a, env, ix5, sh5, host, n5_total, n5, lo5, dim5, 128, 5, q5, workload_name(n5_total, dim5, 128, 5))
            mm, o, rh, _, _ = w.measure(ex_steps, a.warmup, ex_ph, sampler)
            r = finish(w, mm, o, rh, 32)
            # streaming form (BASELINE config 5: "appended in 1M-row epochs"): start with the last 8 epochs uncommitted,
            # publish one epoch (1M rows over all GPUs) every 4 batches while searching; final state == the full corpus
            epoch = max(1, 1_000_000 // world)
            n_ep = min(8, n5 // epoch - 1)
            ix5.lib.sa_corpus_reset(ix5._h)
            ix5.commit(0, n5 - n_ep * epoch)
            barrier()
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            done, nb = n5 - n_ep * epoch, 0
            while done < n5 or nb < 64:
                if nb % 4 == 3 and done < n5:
                    ix5.commit(done, epoch if done + epoch <= n5 else n5 - done)
                    done = min(n5, done + epoch)
                o = w.step_device()
                nb += 1
            ev1.record()
            barrier()
            ms = ev0.elapsed_time(ev1)
            if world > 1:
                ms = env["allmax"]([ms])[0]
            o = w.step_device()
            barrier()
            srec = None if a.no_cpu else w.recall(o, (o[0].cpu().numpy(), o[1].cpu().numpy()), 32)
            if rank == 0:
                r["streaming"] = {"value": 128 * nb / (ms * 1e-3), "unit": UNIT, "batches": nb, "epochs_appended": n_ep,
                                  "epoch_rows_total": epoch * world, "rows_per_s_ingested": n_ep * epoch * world / (ms * 1e-3),
                                  "final_state_recall": srec}
            sh5.close()
            ix5.close()
            return r
        run_extra(f"cfg5_{n5_total // 1_000_000}Mx768_b128_k5", cfg5)

    sampler.stop()
    host.close()
    if rank == 0:
        if extra_out:
            result["extra_configs"] = extra_out
        result["wall_s"] = time.perf_counter() - t_start
        print(json.dumps(result))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    a = parse_args()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_b200(a)


if __name__ == "__main__":
    main()
