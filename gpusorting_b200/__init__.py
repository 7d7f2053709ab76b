"""gpusorting_b200 -- an H100-native (sm_90a) OneSweep radix sort behind the reference's interface.

Only the hot path named by BASELINE.json is here: csrc/ (CUDA kernels + C-ABI, built into
lib/libonesweep_b200.so) and the host-side mirror of the reference's OneSweep interface (onesweep.py,
sharded.py).  Importing the package loads the shared library and fails loudly if it is missing.
"""
from ._lib import LIB_PATH, OneSweepError, lib, status_string  # noqa: F401  (import == load the .so)
from .onesweep import (  # noqa: F401
    ENTROPY_PRESET_1,
    ENTROPY_PRESET_2,
    ENTROPY_PRESET_3,
    ENTROPY_PRESET_4,
    ENTROPY_PRESET_5,
    OneSweepDispatcher,
    OneSweepSorter,
    Sort,
    argsort,
    argsort16,
    init_random,
    kthvalue,
    median,
    median_segments,
    quantile,
    quantile_segments,
    release_cached_sorters,
    select_rows,
    select_segments,
    select_segments_workspace,
    select_workspace_words,
    sort_long_rows,
    sort_long_segments,
    sort_rows,
    sort_segments,
    topk,
    topk_long_rows,
    topk_segments,
)

__version__ = "0.1.0"
