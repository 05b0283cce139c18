"""ctypes binding of libcfgpu.so (include/cfgpu.h).  There is no CPU fallback: if the library is
missing or no H100 is visible, everything here raises."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_int, c_uint32, c_uint64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "libcfgpu.so")

CF_OK = 0
CF_E_CUDA, CF_E_BADARG, CF_E_UNSUPPORTED, CF_E_TOO_LARGE, CF_E_CAPACITY, CF_E_NOGPU, CF_E_NOMEM = -1, -2, -3, -4, -5, -6, -7
CF_PAT_SEARCH, CF_PAT_ORDERED = 0, 1
CF_STAGE_SCAN, CF_STAGE_SUB, CF_STAGE_MASK, CF_STAGE_TOON = 1, 2, 4, 8
CF_RUN_OUTPUTS_RESIDENT = 32
CF_TOON_REPORT_ERRORS, CF_TOON_PARSE_ONLY, CF_TOON_SEQUENTIAL, CF_TOON_NO_HANDOVER = 1, 4, 8, 16
CF_V_REWRITTEN, CF_V_TOON, CF_V_MASKED, CF_V_RESUBMIT = 1, 2, 4, 8
ERR_NAMES = {-1: "CF_E_CUDA", -2: "CF_E_BADARG", -3: "CF_E_UNSUPPORTED", -4: "CF_E_TOO_LARGE", -5: "CF_E_CAPACITY", -6: "CF_E_NOGPU", -7: "CF_E_NOMEM"}


class CfError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{ERR_NAMES.get(code, code)}: {msg}")
        self.code = code


class CompileStats(ctypes.Structure):
    _fields_ = [(n, c_uint32) for n in ("n_patterns", "words_per_bitmap", "n_classes", "n_states", "n_accsets", "n_ordered", "trans_bytes", "prefilter")]


_SIGS = {
    "cf_builder_new": (c_int, [POINTER(c_void_p)]),
    "cf_builder_free": (None, [c_void_p]),
    "cf_builder_last_error": (c_char_p, [c_void_p]),
    "cf_builder_set_word_set": (c_int, [c_void_p, c_void_p, c_uint32]),
    "cf_builder_add_pattern": (c_int, [c_void_p, c_void_p, c_uint32, c_uint32, POINTER(c_uint32)]),
    "cf_builder_set_replacement": (c_int, [c_void_p, c_uint32, c_char_p, c_uint32]),
    "cf_builder_set_template": (c_int, [c_void_p, c_uint32, c_char_p, c_uint32, c_void_p, c_uint32]),
    "cf_builder_compile_host": (c_int, [c_void_p, POINTER(CompileStats)]),
    "cf_init": (c_int, [c_int, POINTER(c_void_p)]),
    "cf_shutdown": (None, [c_void_p]),
    "cf_last_error": (c_char_p, [c_void_p]),
    "cf_compile": (c_int, [c_void_p, c_void_p, POINTER(c_void_p)]),
    "cf_free_prog": (None, [c_void_p]),
    "cf_prog_words": (c_uint32, [c_void_p]),
    "cf_prog_patterns": (c_uint32, [c_void_p]),
    "cf_batch_create": (c_int, [c_void_p, c_uint64, c_uint32, POINTER(c_void_p)]),
    "cf_batch_free": (None, [c_void_p]),
    "cf_run_batch_device_output": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_uint64)]),
    "cf_copy_to_host": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64]),
    "cf_host_alloc": (c_int, [c_void_p, c_uint64, POINTER(c_void_p)]),
    "cf_host_free": (None, [c_void_p, c_void_p]),
    "cf_batch_upload": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p]),
    "cf_batch_pack_device": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_uint64, c_void_p]),
    "cf_batch_units": (c_uint32, [c_void_p]),
    "cf_batch_bytes": (c_uint64, [c_void_p]),
    "cf_scan": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cf_scan_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p]),
    "cf_sub_host": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_uint64, c_void_p, POINTER(c_uint64)]),
    "cf_mask_host": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_int, c_void_p, c_uint64, c_void_p, c_void_p, POINTER(c_uint64)]),
    "cf_classify_keys_host": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p]),
    "cf_toon": (c_int, [c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cf_toon_host": (c_int, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p]),
    "cf_json_index": (c_int, [c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p]),
    "cf_json_index_host": (c_int, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p]),
    "cf_run_batch": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_uint32, c_void_p, c_uint32, c_int, c_void_p, c_void_p,
                             c_void_p, c_uint64, c_void_p, POINTER(c_uint64)]),
    "cf_run_create": (c_int, [c_void_p, c_uint32, c_uint64, c_uint64, POINTER(c_void_p)]),
    "cf_run_free": (None, [c_void_p]),
    "cf_run_enqueue": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64,
                               c_void_p]),
    "cf_run_finish": (c_int, [c_void_p, c_void_p, POINTER(c_uint64)]),
    "cf_run_set_mask": (c_int, [c_void_p, c_void_p, c_int]),
    "cf_kernel_launches": (c_uint64, [c_void_p]),
    "cf_scan_counters": (c_int, [c_void_p, c_void_p]),
    "cf_profile_begin": (c_int, [c_void_p, c_uint32]),
    "cf_profile_collect": (c_int, [c_void_p, POINTER(ctypes.c_double), POINTER(c_uint32)]),
    "cf_profile_collect_each": (c_int, [c_void_p, c_void_p, c_uint32, POINTER(c_uint32)]),
}

_lib = None


def exported_symbols():
    return sorted(_SIGS)


def load() -> ctypes.CDLL:
    """Load libcfgpu.so (building is the job of __graft_entry__.build / build.py)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(f"{SO_PATH} is missing — run `python -m mcp_context_forge_b200.build` (nvcc, sm_90a). There is no CPU fallback.")
    lib = ctypes.CDLL(SO_PATH)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
