"""ctypes binding of libonesweep_b200.so (the C-ABI declared in include/onesweep_b200.h).

There is no CPU or PyTorch fallback: if the shared library has not been built (``python -c "import
__graft_entry__ as g; g.build()"`` or ``make -C gpusorting_b200/csrc``) importing this module raises.
"""
from __future__ import annotations

import ctypes
import os

# torch must be imported BEFORE the shared library is loaded: libonesweep_b200.so needs libnccl.so.2 (sharded sort) and the
# dynamic loader binds one library per soname per process -- torch ships a newer NCCL than the system one, and
# libtorch_cuda.so fails to load ("undefined symbol ncclDevCommCreate") if the older system copy got in first.
import torch  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OSB200_LIB") or os.path.join(_HERE, "lib", "libonesweep_b200.so")  # override: build sweeps only

c_u64, c_u32, c_i64, c_int, c_vp = ctypes.c_uint64, ctypes.c_uint32, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p

# name -> (restype, argtypes); mirrors include/onesweep_b200.h one to one
SIGNATURES = {
    "osb200_version": (c_int, []),
    "osb200_status_string": (ctypes.c_char_p, [c_int]),
    "osb200_create": (c_int, [ctypes.POINTER(c_vp), c_u64, c_int, c_int]),
    "osb200_create_pairs64": (c_int, [ctypes.POINTER(c_vp), c_u64]),
    "osb200_destroy": (c_int, [c_vp]),
    "osb200_workspace_bytes": (c_u64, [c_u64, c_int, c_int]),
    "osb200_sort_keys_u32": (c_int, [c_vp, c_vp, c_u64, c_vp]),
    "osb200_sort_pairs_u32": (c_int, [c_vp, c_vp, c_vp, c_u64, c_vp]),
    "osb200_sort_keys_u64": (c_int, [c_vp, c_vp, c_u64, c_vp]),
    "osb200_sort_keys_typed": (c_int, [c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_sort_pairs_typed": (c_int, [c_vp, c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_argsort": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_sort_keys16": (c_int, [c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_sort_pairs16": (c_int, [c_vp, c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_argsort16": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_sort_rows": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, ctypes.c_uint32, c_int, c_int, c_int, c_vp]),
    "osb200_sort_long_rows": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, ctypes.c_uint32, c_int, c_int, c_int, c_vp]),
    "osb200_sort_segments": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, c_vp, c_u64, ctypes.c_uint32, c_int, c_int, c_int, c_vp]),
    "osb200_sort_long_segments": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, c_vp, c_u64, ctypes.c_uint32, c_int, c_int, c_int, c_vp]),
    "osb200_topk_rows": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, ctypes.c_uint32, ctypes.c_uint32, c_int, c_int, c_int, c_int,
                                 c_vp]),
    "osb200_topk_long_rows": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, ctypes.c_uint32, ctypes.c_uint32, c_int, c_int, c_int, c_int,
                                 c_vp]),
    "osb200_select_rows": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, ctypes.c_uint32, ctypes.POINTER(c_u32), ctypes.c_uint32, c_int, c_int,
                                   c_vp]),
    "osb200_select_segments": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, c_vp, c_u64, ctypes.c_uint32, c_vp, ctypes.c_uint32, c_int,
                                       c_int, c_vp]),
    "osb200_select_segments_workspace_words": (c_u64, [c_u64, c_u64, ctypes.c_uint32, c_int, c_int]),
    "osb200_topk_segments": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, c_vp, c_u64, ctypes.c_uint32, c_int, c_int, c_int, c_int,
                                     c_vp]),
    "osb200_sort_bits": (c_int, [c_vp, c_vp, c_vp, c_u64, c_int, c_int, c_vp]),
    "osb200_segmented_sort_u32": (c_int, [c_vp, c_vp, c_vp, c_vp, c_u64, ctypes.c_uint32, c_vp]),
    "osb200_sort_host_keys_u32": (c_int, [c_vp, c_vp, c_u64]),
    "osb200_sort_host_pairs_u32": (c_int, [c_vp, c_vp, c_vp, c_u64]),
    "osb200_sort_host_keys_u64": (c_int, [c_vp, c_vp, c_u64]),
    "osb200_global_histogram": (c_int, [c_vp, c_vp, c_u64, c_vp, c_vp]),
    "osb200_digit_binning_pass": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_u64, c_u32, c_vp]),
    "osb200_validate": (c_int, [c_vp, c_vp, c_u64, ctypes.POINTER(c_u64), c_vp]),
    "osb200_init_random_u32": (c_int, [c_vp, c_vp, c_u64, c_u32, c_u32, c_int, c_vp]),
    "osb200_set_option": (c_int, [c_vp, ctypes.c_char_p, c_i64]),
    "osb200_get_info": (c_i64, [c_vp, ctypes.c_char_p]),
    "osb200_get_profile": (c_int, [c_vp, ctypes.POINTER(ctypes.c_float), c_int]),
    "osb200_sharded_unique_id": (c_int, [c_vp]),
    "osb200_sharded_create": (c_int, [ctypes.POINTER(c_vp), c_vp, c_int, c_int, c_u64, c_int]),
    "osb200_sharded_destroy": (c_int, [c_vp]),
    "osb200_sharded_sort_keys_u32": (c_int, [c_vp, c_vp, c_u64, ctypes.POINTER(c_vp), ctypes.POINTER(c_u64), c_vp]),
    "osb200_sharded_plan": (c_int, [c_vp, c_int, c_int, c_vp, c_vp, c_vp]),
    "osb200_sharded_set_fused": (c_int, [c_vp, c_int]),
    "osb200_sharded_force_fine": (c_int, [c_vp, c_int]),
    "osb200_sharded_capacity": (c_u64, [c_u64, c_int]),
    "osb200_sharded_exchange_layout": (c_int, [c_vp, c_int, c_int, c_u64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                               c_vp, c_vp, c_vp]),
    "osb200_debug_digit_histogram": (c_int, [c_vp, c_vp, c_u64, c_u32, c_vp, c_vp]),
    "osb200_debug_exchange_pass": (c_int, [c_vp, c_vp, c_vp, c_u64, c_u32, c_vp, c_vp, c_vp]),
    "osb200_sharded_local_handle": (c_int, [c_vp, ctypes.POINTER(c_vp), ctypes.POINTER(c_vp)]),
    "osb200_sharded_last_timing": (c_int, [c_vp, ctypes.POINTER(ctypes.c_float)]),
}


class OneSweepError(RuntimeError):
    def __init__(self, status: int, what: str):
        self.status = status
        super().__init__(f"{what}: osb200 status {status} ({status_string(status)})")


def _load() -> ctypes.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the sm_90a CUDA library has not been built and this package has no "
            "fallback path. Build it with `make -C gpusorting_b200/csrc` (or __graft_entry__.build())."
        )
    lib = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == header and library out of sync: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def status_string(status: int) -> str:
    return lib.osb200_status_string(int(status)).decode()


def check(status: int, what: str) -> None:
    if status != 0:
        raise OneSweepError(int(status), what)
