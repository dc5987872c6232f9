"""int8 vector indexes on a CPU box: the C ABI's argument checks, the fp32 -> int8 conversion rule, the binding, and the
independent fixture against the existing definition fed the same integers as bf16.  The GPU side is
tests/test_gpu_int8.py."""
import ctypes as C
import glob
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from harness import filter_oracle
from harness.similarity_oracle import topk_f64
from oracle import bruteforce as bf
from qsa_b200 import capi

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = sorted(glob.glob(os.path.join(HERE, "golden", "int8_topk_independent_*.npz")))
SIMS = ("cosine", "dotProduct", "euclidean")
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")


def create(lib, dim, elem, sim=capi.SA_SIM_COSINE):
    h = C.c_void_p()
    rc = lib.sa_engine_create_elem(C.byref(h), 0, dim, 1000, 128, 10, sim, elem)
    return rc, h


@pytest.mark.parametrize("dim,elem,what", [
    (256, 2, b"elem 2"), (256, -1, b"elem -1"),                                  # unknown element types
    (64, capi.SA_ELEM_INT8, b"multiple of 128"), (192, capi.SA_ELEM_INT8, b"multiple of 128"),
    (65664, capi.SA_ELEM_INT8, b"at most 65536"),                               # |<q,c>| would leave int32
    (65600, capi.SA_ELEM_BF16, b"at most 65536"),         # the fallback scan's query row would not fit shared memory
])
def test_create_elem_refuses_before_touching_a_device(lib, dim, elem, what):
    rc, h = create(lib, dim, elem)
    assert rc == capi.SA_ERR_ARG and not h.value
    assert what in lib.sa_last_error()


def test_create_elem_checks_the_similarity_first(lib):
    rc, _ = create(lib, 256, capi.SA_ELEM_INT8, sim=7)
    assert rc == capi.SA_ERR_ARG and b"similarity 7" in lib.sa_last_error()


def int8_round(lib, x):
    x = np.ascontiguousarray(x, dtype=np.float32)
    out = np.empty(x.shape, np.int8)
    assert lib.sa_debug_int8_round(x.ctypes.data, x.size, out.ctypes.data) == 0
    return out


def test_int8_round_is_rne_saturated_and_nan_is_zero(lib):
    g = np.random.default_rng(3)
    x = np.concatenate([g.standard_normal(20000) * 60, g.uniform(-300, 300, 20000), np.arange(-140, 141) + 0.5,
                        [0.5, -0.5, 1.5, -1.5, 2.5, 127.5, -127.5, 128.5, -128.5, 126.5, -128.0, 127.0, 1e30, -1e30,
                         np.inf, -np.inf, -0.0, 0.0, 1e-45]]).astype(np.float32)
    want = np.clip(np.rint(x.astype(np.float64)), -128, 127).astype(np.int8)      # np.rint rounds half to even
    assert np.array_equal(int8_round(lib, x), want)
    assert int8_round(lib, np.array([np.nan, -np.nan], np.float32)).tolist() == [0, 0]
    ints = np.arange(-128, 128, dtype=np.float32)
    assert np.array_equal(int8_round(lib, ints), ints.astype(np.int8))        # integer-valued floats pass unchanged


def test_engine_int8_round_helper_uses_the_library(lib):
    from qsa_b200.engine import int8_round as helper
    x = np.array([[0.5, 1.5, -2.5, 200.0, np.nan, -129.0]], np.float32)
    assert helper(x).tolist() == [[0, 2, -2, 127, 0, -128]]


def test_elem_names():
    assert capi.ELEMS == {"bfloat16": capi.SA_ELEM_BF16, "int8": capi.SA_ELEM_INT8}
    assert (capi.SA_ELEM_BF16, capi.SA_ELEM_INT8) == (0, 1)
    assert capi.elem_code("int8") == 1 and capi.elem_code("bfloat16") == 0
    for bad in ("float16", "bf16", "uint8", ""):
        with pytest.raises(ValueError, match="dtype must be one of"):
            capi.elem_code(bad)


def header_prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "sa_api.h")).read(), flags=re.S)
    m = re.search(r"\b" + name + r"\s*\(([^)]*)\)", src)
    return [a.strip() for a in m.group(1).split(",")]


def test_binding_signatures_match_the_header(lib):
    i32, i64, vp = C.c_int, C.c_int64, C.c_void_p
    assert header_prototype("sa_engine_create_elem") == [
        "sa_engine** out", "int device", "int dim", "int64_t capacity_rows", "int max_batch", "int max_k",
        "int similarity", "int elem"]
    assert lib.sa_engine_create_elem.argtypes == [C.POINTER(vp), i32, i32, i64, i32, i32, i32, i32]
    assert lib.sa_engine_create_elem.restype is i32
    assert header_prototype("sa_debug_int8_round") == ["const float* x", "int n", "int8_t* out"]
    assert lib.sa_debug_int8_round.argtypes == [vp, i32, vp]
    src = open(os.path.join(ROOT, "include", "sa_api.h")).read()
    assert re.search(r"#define SA_ELEM_BF16 0\b", src) and re.search(r"#define SA_ELEM_INT8 1\b", src)
    for name in ("sa_engine_create_elem", "sa_debug_int8_round"):
        assert name in capi.EXPORTS


def test_library_has_the_s8_wgmma_scan(lib):
    sass = subprocess.run([CUOBJDUMP, "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "IGMMA.64x128x32.S8.S8" in sass
    names = set(re.findall(r"Function : (_ZN2sa14sa_scan_kernel\S+)", sass))
    epis = [int(m.group(1)) for m in (re.search(r"ILi\d+ELi\d+ELi\d+ELi(\d+)EE", n) for n in names)]
    assert len(names) == 58 and sum(e & 8 != 0 for e in epis) == 28


def as_bf16_bits(x):
    """int8 values as bf16 bit patterns: every int8 is exactly representable in bf16."""
    b = bf.f32_to_bf16_bits(np.asarray(x, dtype=np.float32))
    assert np.array_equal(bf.bf16_bits_to_f32(b), np.asarray(x, dtype=np.float32))
    return b


def test_golden_fixture_exists():
    assert len(GOLDEN) == 1


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
@pytest.mark.parametrize("sim", SIMS)
def test_definition_on_the_integers_reproduces_the_fixture(path, sim):
    z = np.load(path)
    c, q, k = as_bf16_bits(z["corpus"]), as_bf16_bits(z["queries"]), int(z["k"])
    s, i = topk_f64(q, c, k, sim)
    assert np.array_equal(i, z[f"{sim}_idx"])
    fin = np.isfinite(z[f"{sim}_score"])
    assert np.array_equal(np.isfinite(s), fin)
    assert np.allclose(s[fin], z[f"{sim}_score"][fin], rtol=1e-12, atol=0)
    ok = filter_oracle.eligibility(z["tags"], z["filters"])
    s, i = filter_oracle.topk_f64(q, c, k, sim, ok)
    assert np.array_equal(i, z[f"{sim}_filtered_idx"])
    fin = np.isfinite(z[f"{sim}_filtered_score"])
    assert np.array_equal(np.isfinite(s), fin)
    assert np.allclose(s[fin], z[f"{sim}_filtered_score"][fin], rtol=1e-12, atol=0)
    assert (i[4] >= 0).sum() < k and (i[7] == -1).all()                     # fewer than k eligible rows; none
    # the all-ones query: the 200 permutation rows tie, so they appear in ascending row order
    perm = i[0][(i[0] >= 107) & (i[0] < 307)]
    assert (np.diff(perm) > 0).all()
