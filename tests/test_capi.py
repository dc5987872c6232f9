"""CPU tests of the boundary: libsa_b200.so builds for sm_90a without a GPU, loads, exports every symbol
include/sa_api.h declares, and fails loudly (no fallback) when there is no CUDA device."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from qsa_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def header_functions():
    names = set()
    for h in ("sa_api.h", "sa_wire.h"):
        src = open(os.path.join(ROOT, "include", h)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names |= set(re.findall(r"\b(sa_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_header_and_binding_agree():
    assert header_functions() == sorted(capi.EXPORTS)


def test_library_exports_every_symbol(lib):
    for name in header_functions():
        assert hasattr(lib, name), name
    assert lib.sa_version() >= 100
    assert lib.sa_strerror(capi.SA_ERR_DEVICE).decode().startswith("unsupported device")


def test_library_contains_only_sm90a_native_code(lib):
    out = subprocess.run([CUOBJDUMP, "-lelf", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert not re.search(r"sm_(?!90a)\d+", out), out
    sass = subprocess.run([CUOBJDUMP, "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA.64x128x16.F32.BF16", "UTMALDG.2D", "UTMALDG.2D.MULTICAST"):   # wgmma, TMA, TMA multicast
        assert mnemonic in sass, mnemonic
    assert "HMMA." not in sass                                  # no legacy mma.sync path


def test_argument_validation_without_touching_the_gpu(lib):
    h = C.c_void_p()
    assert lib.sa_engine_create(C.byref(h), 0, 100, 1000, 128, 10) == capi.SA_ERR_ARG       # dim % 64
    assert b"multiple of 64" in lib.sa_last_error()
    assert lib.sa_engine_create(C.byref(h), 0, 128, 0, 128, 10) == capi.SA_ERR_ARG          # capacity
    assert lib.sa_engine_create(C.byref(h), 0, 128, 1000, 128, 99) == capi.SA_ERR_ARG       # max_k
    assert lib.sa_corpus_rows(None) == -1
    assert lib.sa_search(None, None, 1, 1, None, None, None, None) == capi.SA_ERR_ARG


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_gpu_means_loud_failure_not_fallback(lib):
    h = C.c_void_p()
    rc = lib.sa_engine_create(C.byref(h), 0, 1536, 1000, 128, 10)
    assert rc in (capi.SA_ERR_CUDA, capi.SA_ERR_ARG) and not h.value
    from qsa_b200.engine import VectorIndex
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        VectorIndex(dim=1536, capacity=1000)


def test_missing_library_raises(monkeypatch, tmp_path):
    monkeypatch.setattr(capi, "_lib", None)
    monkeypatch.setattr(capi, "LIB_PATH", str(tmp_path / "libsa_b200.so"))
    with pytest.raises(capi.SaLibraryMissing, match="no CPU fallback"):
        capi.load()


def plan(lib, num_sms, nq, cg, num_tiles, cap=0):
    out = (C.c_int * (4 * 16))()
    n = C.c_int()
    rc = lib.sa_debug_plan(num_sms, nq, cg, num_tiles, cap, out, 16, C.byref(n))
    assert rc == 0, lib.sa_last_error()
    return [tuple(out[4 * i + j] for j in range(4)) for i in range(n.value)]


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("nq", [1, 37, 128, 129, 256, 700, 1024, 1100, 4096, 5000])
@pytest.mark.parametrize("num_tiles", [0, 1, 5, 79, 39063])
@pytest.mark.parametrize("sms", [148, 160])
def test_launch_planner_invariants(lib, cg, nq, num_tiles, sms):
    """Host logic of the scan: every query is covered exactly once, a launch never needs more CTAs than SMs,
    tile lanes never outnumber tiles nor the merge kernel's 132-lane table, and the machine is used when the batch
    allows it."""
    launches = plan(lib, sms, nq, cg, num_tiles)
    rows = 128 * cg
    nxt = 0
    for q0, n, nqb, tl in launches:
        assert q0 == nxt and n > 0 and q0 % rows == 0
        assert nqb == (n + rows - 1) // rows and tl >= 1
        assert nqb * tl * cg <= sms and tl <= max(num_tiles, 1) and tl <= 132
        nxt += n
    assert nxt == nq
    if num_tiles >= 148 and nq >= rows:
        used = max(nqb * tl * cg for _, _, nqb, tl in launches)
        assert used >= 0.85 * 148, launches


def test_launch_planner_headline_shapes(lib):
    assert plan(lib, 132, 1024, 2, 39063) == [(0, 512, 2, 33), (512, 512, 2, 33)]   # 2 launches of 2 pair blocks x 33 lanes
    assert plan(lib, 132, 128, 1, 39063) == [(0, 128, 1, 132)]              # HBM-bound: every SM its own lane
    assert plan(lib, 148, 128, 1, 39063) == [(0, 128, 1, 132)]              # ... capped at the merge kernel's 132 lanes
    assert plan(lib, 132, 512, 2, 39063) == [(0, 512, 2, 33)]               # already fills the machine
    p = plan(lib, 132, 4096, 2, 4883)                                       # config 4 per GPU: 6 launches
    assert [x[2:] for x in p] == [(3, 22)] * 4 + [(2, 33)] * 2
    assert len(plan(lib, 132, 1100, 2, 118, cap=2)) == 3                    # forced small launches


def test_filtered_twins_take_the_filter_right_after_the_query(lib):
    """Every X_filtered is X with one sa_filter* inserted right after the query pointer -- the rule capi.search relies
    on -- in the binding's signatures and in the header's parameter names."""
    twins = sorted(n[:-len("_filtered")] for n in capi.EXPORTS if n.endswith("_filtered"))
    assert twins == sorted(capi.QUERY_ARG)
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sa_api.h")).read(), flags=re.S)
    params = {m[0]: [p.split()[-1].lstrip("*") for p in m[1].split(",")]
              for m in re.findall(r"\b(sa_[a-z0-9_]+)\s*\(([^)]*)\)", src)}
    for name in twins:
        at = capi.QUERY_ARG[name] + 1
        base, twin = list(getattr(lib, name).argtypes), list(getattr(lib, name + "_filtered").argtypes)
        assert twin == base[:at] + [C.c_void_p] + base[at:], name
        assert params[name][at - 1].startswith("q_"), (name, params[name])
        f = params[name + "_filtered"][at]
        assert f.startswith("filters_") and params[name + "_filtered"] == params[name][:at] + [f] + params[name][at:], name
