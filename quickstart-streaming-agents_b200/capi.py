"""ctypes binding of libsa_b200.so -- one Python function per entry point of include/sa_api.h.

No compute happens in this file and there is no fallback: if the shared library is missing or a call
fails, an exception is raised (``SaLibraryMissing`` / ``SaError``).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SA_LIB_PATH") or os.path.join(_HERE, "libsa_b200.so")   # SA_LIB_PATH: A/B experiment builds

SA_OK = 0
SA_ERR_CUDA = -1
SA_ERR_ARG = -2
SA_ERR_COMM = -3
SA_ERR_CAPACITY = -4
SA_ERR_DEVICE = -5
SA_MAX_K = 64   # deep searches (28 < k <= 64) keep 32-entry lists with bounds valid for their k
SA_MAX_DIM = 65536   # largest dim of either element type
SA_HOST_SLOTS = 2
SA_COMM_ID_BYTES = 128
SA_SIM_COSINE = 0
SA_SIM_DOT = 1
SA_SIM_EUCLIDEAN = 2
# Atlas's names for the index's "similarity" setting -> the engine's constants
SIMILARITIES = {"cosine": SA_SIM_COSINE, "dotProduct": SA_SIM_DOT, "euclidean": SA_SIM_EUCLIDEAN}


SA_ELEM_BF16 = 0
SA_ELEM_INT8 = 1
# an index's element type (the dtype of its rows and device queries) -> the engine's constants
ELEMS = {"bfloat16": SA_ELEM_BF16, "int8": SA_ELEM_INT8}


def similarity_code(name: str) -> int:
    if name not in SIMILARITIES:
        raise ValueError(f"similarity must be one of {sorted(SIMILARITIES)}, not {name!r}")
    return SIMILARITIES[name]


def elem_code(name: str) -> int:
    if name not in ELEMS:
        raise ValueError(f"dtype must be one of {sorted(ELEMS)}, not {name!r}")
    return ELEMS[name]


# every symbol include/sa_api.h declares (tests check the .so exports each of them)
EXPORTS = (
    "sa_version", "sa_strerror", "sa_last_error", "sa_engine_create", "sa_engine_create_sim", "sa_engine_destroy", "sa_corpus_bind",
    "sa_corpus_commit", "sa_corpus_append_f32", "sa_corpus_append_host_f32", "sa_corpus_reset", "sa_corpus_rows",
    "sa_search", "sa_search_f32", "sa_search_host", "sa_search_host_submit", "sa_search_host_wait",
    "sa_search_hits", "sa_merge_hits", "sa_merge_shards",
    "sa_comm_set_library", "sa_comm_nccl_version", "sa_comm_create", "sa_comm_unique_id", "sa_comm_create_rank",
    "sa_comm_destroy", "sa_comm_ranks", "sa_sharded_search", "sa_sharded_search_host_submit",
    "sa_sharded_search_host_wait", "sa_gather_merge", "sa_gather_merge_submit", "sa_gather_merge_wait",
    "sa_last_timing", "sa_timing_mean", "sa_set_option",
    "sa_get_info", "sa_scan_profile", "sa_debug_tile_dots", "sa_debug_plan", "sa_debug_float_keys", "sa_debug_bf16_round",
    "sa_debug_merge_keys", "sa_debug_list_insert", "sa_debug_window_bound", "sa_host_alloc", "sa_host_free",
    # deep search (28 < k <= 64)
    "sa_debug_window_bound_deep",
    # pre-filtered search
    "sa_corpus_bind_tags", "sa_search_filtered", "sa_search_f32_filtered", "sa_search_host_filtered",
    "sa_search_host_submit_filtered", "sa_search_hits_filtered", "sa_sharded_search_filtered",
    "sa_sharded_search_host_submit_filtered", "sa_gather_merge_filtered", "sa_gather_merge_submit_filtered",
    "sa_debug_filter_pass",
    # int8 indexes
    "sa_engine_create_elem", "sa_debug_int8_round",
    # include/sa_wire.h
    "sa_wire_split_log", "sa_wire_decode_queries_embed", "sa_wire_decode_documents_embed", "sa_wire_encode_search_results", "sa_wire_encode_queries_embed",
)


class SaLibraryMissing(RuntimeError):
    pass


class SaError(RuntimeError):
    def __init__(self, rc: int, what: str, detail: str):
        super().__init__(f"{what}: {detail} (rc={rc})")
        self.rc = rc


_lib = None


def load() -> C.CDLL:
    """Load libsa_b200.so (built in-tree by ``__graft_entry__.build()`` / ``make -C csrc``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SaLibraryMissing(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, u64, f32p = C.c_void_p, C.c_int, C.c_int64, C.c_uint64, C.POINTER(C.c_float)
    sig = {
        "sa_version": (i32, []),
        "sa_strerror": (C.c_char_p, [i32]),
        "sa_last_error": (C.c_char_p, []),
        "sa_engine_create": (i32, [C.POINTER(vp), i32, i32, i64, i32, i32]),
        "sa_engine_create_sim": (i32, [C.POINTER(vp), i32, i32, i64, i32, i32, i32]),
        "sa_engine_destroy": (None, [vp]),
        "sa_corpus_bind": (i32, [vp, vp, vp, i64]),
        "sa_corpus_commit": (i32, [vp, i64, i64, vp]),
        "sa_corpus_append_f32": (i32, [vp, vp, i64, vp]),
        "sa_corpus_append_host_f32": (i32, [vp, vp, i64]),
        "sa_corpus_reset": (i32, [vp]),
        "sa_corpus_rows": (i64, [vp]),
        "sa_search": (i32, [vp, vp, i32, i32, vp, vp, vp, vp]),
        "sa_search_f32": (i32, [vp, vp, i32, i32, vp, vp, vp, vp]),
        "sa_search_host": (i32, [vp, vp, i32, i32, vp, vp]),
        "sa_search_host_submit": (i32, [vp, i32, vp, i32, i32]),
        "sa_search_host_wait": (i32, [vp, i32, vp, vp]),
        "sa_merge_shards": (i32, [vp, vp, vp, i32, i32, i32, vp, vp, vp]),
        "sa_search_hits": (i32, [vp, vp, i32, i32, i64, vp, vp]),
        "sa_merge_hits": (i32, [vp, vp, i32, i32, i32, vp, vp, vp]),
        "sa_comm_set_library": (i32, [C.c_char_p]),
        "sa_comm_nccl_version": (i32, [C.POINTER(i32), C.c_char_p, i32]),
        "sa_comm_create": (i32, [C.POINTER(vp), i32, C.POINTER(i32)]),
        "sa_comm_unique_id": (i32, [vp]),
        "sa_comm_create_rank": (i32, [C.POINTER(vp), i32, i32, vp, i32]),
        "sa_comm_destroy": (None, [vp]),
        "sa_comm_ranks": (i32, [vp]),
        "sa_sharded_search": (i32, [vp, vp, vp, i32, i32, i64, vp, vp, vp]),
        "sa_sharded_search_host_submit": (i32, [vp, vp, i32, vp, i32, i32, i64]),
        "sa_sharded_search_host_wait": (i32, [vp, vp, i32, vp, vp]),
        "sa_gather_merge": (i32, [vp, C.POINTER(vp), vp, i32, i32, C.POINTER(i64), vp, vp]),
        "sa_gather_merge_submit": (i32, [vp, C.POINTER(vp), i32, vp, i32, i32, C.POINTER(i64)]),
        "sa_gather_merge_wait": (i32, [vp, C.POINTER(vp), i32, vp, vp]),
        "sa_last_timing": (i32, [vp, f32p, f32p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i32),
                                 C.POINTER(i32)]),
        "sa_timing_mean": (i32, [vp, i32, f32p, f32p, C.POINTER(i32)]),
        "sa_set_option": (i32, [vp, C.c_char_p, i64]),
        "sa_get_info": (i32, [vp, C.c_char_p, C.POINTER(i64)]),
        "sa_scan_profile": (i32, [vp, vp, i32, C.POINTER(i32)]),
        "sa_debug_tile_dots": (i32, [vp, vp, i32, i32, i32, vp, vp]),
        "sa_debug_plan": (i32, [i32, i32, i32, i32, i32, C.POINTER(i32), i32, C.POINTER(i32)]),
        "sa_debug_float_keys": (i32, [vp, i32, vp, vp, vp]),
        "sa_debug_bf16_round": (i32, [vp, i32, vp, vp]),
        "sa_debug_merge_keys": (i32, [vp, vp, i32, vp, vp]),
        "sa_debug_list_insert": (i32, [vp, vp, i32, i32, vp, vp, vp, vp]),
        "sa_debug_window_bound": (i32, [vp, i32, i32, vp, vp]),
        "sa_debug_window_bound_deep": (i32, [vp, i32, vp]),
        "sa_wire_split_log": (i32, [vp, u64, i32, vp, vp, vp, vp, vp]),
        "sa_wire_decode_queries_embed": (i32, [vp, vp, vp, i32, i32, C.c_uint32, vp, vp, vp, vp, C.POINTER(i32)]),
        "sa_wire_decode_documents_embed": (i32, [vp, vp, vp, i32, i32, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp, C.POINTER(i32)]),
        "sa_wire_encode_search_results": (i32, [i32, i32, i32, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i32, i64,
                                                vp, u64, vp, C.POINTER(u64)]),
        "sa_wire_encode_queries_embed": (i32, [i32, i32, C.c_uint32, vp, vp, vp, vp, i64, vp, u64, vp, C.POINTER(u64)]),
        "sa_corpus_bind_tags": (i32, [vp, vp]),
        "sa_search_filtered": (i32, [vp, vp, vp, i32, i32, vp, vp, vp, vp]),
        "sa_search_f32_filtered": (i32, [vp, vp, vp, i32, i32, vp, vp, vp, vp]),
        "sa_search_host_filtered": (i32, [vp, vp, vp, i32, i32, vp, vp]),
        "sa_search_host_submit_filtered": (i32, [vp, i32, vp, vp, i32, i32]),
        "sa_search_hits_filtered": (i32, [vp, vp, vp, i32, i32, i64, vp, vp]),
        "sa_sharded_search_filtered": (i32, [vp, vp, vp, vp, i32, i32, i64, vp, vp, vp]),
        "sa_sharded_search_host_submit_filtered": (i32, [vp, vp, i32, vp, vp, i32, i32, i64]),
        "sa_gather_merge_filtered": (i32, [vp, C.POINTER(vp), vp, vp, i32, i32, C.POINTER(i64), vp, vp]),
        "sa_gather_merge_submit_filtered": (i32, [vp, C.POINTER(vp), i32, vp, vp, i32, i32, C.POINTER(i64)]),
        "sa_debug_filter_pass": (i32, [vp, i32, vp, vp]),
        "sa_engine_create_elem": (i32, [C.POINTER(vp), i32, i32, i64, i32, i32, i32, i32]),
        "sa_debug_int8_round": (i32, [vp, i32, vp]),
        "sa_host_alloc": (i32, [C.POINTER(vp), u64]),
        "sa_host_free": (i32, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def bundled_nccl_path() -> str | None:
    """Path of the NCCL that ships with torch's wheels (nvidia-nccl-cu12), if present -- handed to sa_comm_set_library so
    a process that has not imported torch.distributed still loads the same NCCL torch would."""
    import importlib.util
    spec = importlib.util.find_spec("nvidia")
    for root in (list(spec.submodule_search_locations) if spec and spec.submodule_search_locations else []):
        pth = os.path.join(root, "nccl", "lib", "libnccl.so.2")
        if os.path.exists(pth):
            return pth
    return None


def check(rc: int, what: str) -> None:
    if rc != SA_OK:
        lib = load()
        detail = lib.sa_last_error().decode() or lib.sa_strerror(rc).decode()
        raise SaError(rc, what, detail)


# the search entry points with a "_filtered" twin -> the position of their query pointer; the twin takes the same
# arguments with the filter pointer (sa_filter*) inserted right after it
QUERY_ARG = {
    "sa_search": 1, "sa_search_f32": 1, "sa_search_host": 1, "sa_search_host_submit": 2, "sa_search_hits": 1,
    "sa_sharded_search": 2, "sa_sharded_search_host_submit": 3, "sa_gather_merge": 2, "sa_gather_merge_submit": 3,
}


def search(lib: C.CDLL, name: str, *args, filters=None) -> None:
    """Call the search entry point ``name``, or with ``filters`` (staged per-query sa_filter words: a numpy array for a
    host call, a CUDA tensor for a device call) its twin ``name + "_filtered"``.  Raises ``SaError`` naming the symbol
    called."""
    if filters is not None:
        at = QUERY_ARG[name] + 1
        ptr = filters.data_ptr() if hasattr(filters, "data_ptr") else filters.ctypes.data
        name, args = name + "_filtered", args[:at] + (ptr,) + args[at:]
    check(getattr(lib, name)(*args), name)
