"""Host-side mirror of the reference's OneSweep interface, on top of the C-ABI.

Reference (paths relative to /root/reference):
  * class OneSweepDispatcher(bool keysOnly, uint32_t maxSize), GPUSortingCUDA/Sort/OneSweepDispatcher.cuh:17-392
    -- TestAllKeysOnly / TestAllPairs / BatchTimingKeysOnly / BatchTimingPairs keep their names and argument
    meaning here so the parity tests read like the reference's own.
  * OneSweep.Sort(...), GPUSortingUnity/Runtime/OneSweep.cs:297-306,358-370 -- the only public `Sort` in the
    reference; `Sort(keys[, values], n)` below is BASELINE.json's north-star shape of it.

PyTorch is used for device memory and streams only; every byte of sorting work happens in
libonesweep_b200.so.
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional

import numpy as np
import torch

from . import _lib
from ._lib import check, lib

ENTROPY_PRESET_1, ENTROPY_PRESET_2, ENTROPY_PRESET_3, ENTROPY_PRESET_4, ENTROPY_PRESET_5 = range(5)

# sort_keys / sort_pairs order keys by their UNSIGNED bit pattern: only integer containers are accepted there (a float
# tensor would silently sort negatives wrongly).  Float tensors go through sort_*_typed, which states the key type.
_KEY_DTYPES_4 = (torch.int32, torch.uint32)
_KEY_DTYPES_8 = (torch.int64, torch.uint64)
_TYPED_DTYPES_4 = (torch.int32, torch.uint32, torch.float32)
_TYPED_DTYPES_8 = (torch.int64, torch.uint64, torch.float64)
KEY_TYPES = {"u32": 0, "i32": 1, "f32": 2, "u64": 3, "i64": 4, "f64": 5}
# 16-bit keys (sort_keys16 / sort_pairs16 / argsort16, on a 4-byte sorter): key_type states the order, the dtype the width
_TYPED_DTYPES_2 = (torch.int16, torch.uint16, torch.float16, torch.bfloat16)
KEY16_TYPES = {"u16": 0, "i16": 1, "f16": 2, "bf16": 3}
# row sort (sort_rows): the key type of every dtype it takes
_ROW_KEY_TYPES = {torch.int16: "i16", torch.uint16: "u16", torch.float16: "f16", torch.bfloat16: "bf16",
                  torch.int32: "i32", torch.uint32: "u32", torch.float32: "f32",
                  torch.int64: "i64", torch.uint64: "u64", torch.float64: "f64"}


def _stream_ptr(stream: Optional[torch.cuda.Stream]) -> int:
    s = stream if stream is not None else torch.cuda.current_stream()
    return int(s.cuda_stream)


def _check_dev_tensor(t: torch.Tensor, dtypes, name: str, n: Optional[int] = None, device: Optional[int] = None) -> None:
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.is_contiguous() and t.dtype in dtypes and t.dim() == 1):
        raise TypeError(f"{name} must be a contiguous 1-D CUDA tensor with dtype in {dtypes}")
    if device is not None and t.device.index != device:
        raise ValueError(f"{name} lives on cuda:{t.device.index}, the sorter on cuda:{device}")
    if n is not None and not (0 <= n <= t.numel()):
        raise ValueError(f"n={n} is outside 0..{name}.numel()={t.numel()}")


def _new_outputs(stream, x: torch.Tensor, shape, indices: bool = True, out: Optional[torch.Tensor] = None):
    """(keys, int32 indices) of `shape` on x's device, the keys in x's dtype, allocated with torch.empty on the stream
    (None: the current stream): the outputs belong to the stream that writes them.  out: the keys to write instead of new
    ones; indices=False: no indices (None)."""
    with torch.cuda.stream(stream):
        if out is None:
            out = torch.empty(shape, dtype=x.dtype, device=x.device)
        idx = torch.empty(shape, dtype=torch.int32, device=x.device) if indices else None
    return out, idx


class OneSweepSorter:
    """Owns one C-ABI sorter handle (alt buffers, tile descriptors) for up to ``max_n`` elements.

    Keys are ordered by their UNSIGNED bit pattern, as in the reference CUDA path (uint32 keys,
    OneSweep.cuh:24-52); int32/int64 tensors are accepted as raw 32/64-bit containers.
    (8, 4) -- 64-bit keys with 32-bit payloads -- is created by osb200_create_pairs64.
    """

    def __init__(self, max_n: int, key_bytes: int = 4, value_bytes: int = 0, device: Optional[int] = None):
        if not torch.cuda.is_available():
            raise RuntimeError("gpusorting_b200 needs a CUDA device (sm_90); there is no CPU fallback")
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.max_n, self.key_bytes, self.value_bytes = int(max_n), int(key_bytes), int(value_bytes)
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            if (self.key_bytes, self.value_bytes) == (8, 4):
                check(lib.osb200_create_pairs64(ctypes.byref(h), self.max_n), "osb200_create_pairs64")
            else:
                check(lib.osb200_create(ctypes.byref(h), self.max_n, self.key_bytes, self.value_bytes), "osb200_create")
        self._h = h

    # -- lifetime ---------------------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            lib.osb200_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- options ----------------------------------------------------------------------------------
    def set_option(self, key: str, value: int) -> None:
        check(lib.osb200_set_option(self._h, key.encode(), int(value)), f"osb200_set_option({key})")

    def info(self, key: str) -> int:
        v = lib.osb200_get_info(self._h, key.encode())
        if v < 0:
            raise KeyError(key)
        return int(v)

    def last_profile(self):
        """Per-kernel milliseconds of the last sort when option 'profile' is on: [hist, scan, pass0, pass1, ...]."""
        buf = (ctypes.c_float * 16)()
        k = lib.osb200_get_profile(self._h, buf, 16)
        if k < 0:
            check(k, "osb200_get_profile")
        return [float(buf[i]) for i in range(k)]

    # -- device sorts -------------------------------------------------------------------------------
    # Every entry point validates dtype / device / contiguity / n against the tensors it is handed and makes the
    # sorter's device current for the launch (the C side launches on the current device).
    def _raw(self):
        return _KEY_DTYPES_4 if self.key_bytes == 4 else _KEY_DTYPES_8

    def _typed(self):
        return _TYPED_DTYPES_4 if self.key_bytes == 4 else _TYPED_DTYPES_8

    def _call(self, fn, *args, stream=None) -> None:
        """fn(handle, *args, stream pointer) on the sorter's device; a failing status raises OneSweepError naming fn."""
        with torch.cuda.device(self.device):
            check(fn(self._h, *args, _stream_ptr(stream)), fn.__name__)

    def _ragged_keys(self, x: torch.Tensor, key_type: str, offsets: Optional[torch.Tensor] = None):
        """The checks of the row calls (x of rank >= 1) and, given offsets, of the segment calls (1-D x and its offsets);
        returns x's key width and the C key type."""
        if offsets is None:
            if not (isinstance(x, torch.Tensor) and x.is_cuda and x.is_contiguous() and x.dim() >= 1 and x.dtype in _ROW_KEY_TYPES):
                raise TypeError(f"x must be a contiguous CUDA tensor of rank >= 1 with dtype in {tuple(_ROW_KEY_TYPES)}")
        elif not (isinstance(x, torch.Tensor) and x.is_cuda and x.is_contiguous() and x.dim() == 1 and x.dtype in _ROW_KEY_TYPES):
            raise TypeError(f"x must be a contiguous 1-D CUDA tensor with dtype in {tuple(_ROW_KEY_TYPES)}")
        if x.device.index != self.device:
            raise ValueError(f"x lives on cuda:{x.device.index}, the sorter on cuda:{self.device}")
        if offsets is not None and not (isinstance(offsets, torch.Tensor) and offsets.dtype == torch.int64
                                        and offsets.is_contiguous() and offsets.dim() == 1 and offsets.device == x.device):
            raise TypeError("offsets must be a contiguous 1-D int64 tensor on the device of x")
        kb = x.element_size()
        return kb, (KEY16_TYPES if kb == 2 else KEY_TYPES)[key_type]

    def sort_keys(self, keys: torch.Tensor, n: Optional[int] = None, stream=None) -> torch.Tensor:
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._raw(), "keys", n, self.device)
        fn = lib.osb200_sort_keys_u32 if self.key_bytes == 4 else lib.osb200_sort_keys_u64
        self._call(fn, keys.data_ptr(), n, stream=stream)
        return keys

    def sort_keys_typed(self, keys: torch.Tensor, key_type: str, descending: bool = False, n: Optional[int] = None,
                        stream=None) -> torch.Tensor:
        """Signed / float keys and descending order (reference HLSL: SortCommon.hlsl:134-154,594-656).  key_type in
        KEY_TYPES; it states how the bits are ordered, whatever the tensor dtype (which only has to have the width)."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._typed(), "keys", n, self.device)
        self._call(lib.osb200_sort_keys_typed, keys.data_ptr(), n, KEY_TYPES[key_type], 1 if descending else 0, stream=stream)
        return keys

    def sort_pairs_typed(self, keys: torch.Tensor, values: torch.Tensor, key_type: str, descending: bool = False,
                         n: Optional[int] = None, stream=None):
        """sort_keys_typed with 32-bit payloads that move with their keys (stable).  Keys must start on a 16-byte boundary
        (OneSweepError status -1 otherwise); values need only their natural 4-byte alignment, so any contiguous view will do.
        Keys are 32-bit on a (4, 4) sorter and int64 / uint64 / float64 on a (8, 4) sorter."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._typed(), "keys", n, self.device)
        _check_dev_tensor(values, _TYPED_DTYPES_4, "values", n, self.device)
        self._call(lib.osb200_sort_pairs_typed, keys.data_ptr(), values.data_ptr(), n, KEY_TYPES[key_type],
                   1 if descending else 0, stream=stream)
        return keys, values

    def argsort(self, keys: torch.Tensor, key_type: str, descending: bool = False, n: Optional[int] = None, stream=None):
        """Stable sort of keys[:n] that leaves `keys` untouched (osb200_argsort; the shape of torch.sort(stable=True)).

        Returns (sorted_keys, indices): new tensors of n elements on the keys' device, allocated with torch.empty (so the call
        can be captured in a CUDA graph).  sorted_keys has the dtype of `keys`; indices[i] is the input position of
        sorted_keys[i], stored as torch.int32, the container of the library's 32-bit payloads.  Positions >= 2^31 (n > 2^31)
        read as negative in it: ``indices.long() & 0xFFFFFFFF`` recovers them.  key_type is "u32", "i32" or "f32" on a (4, 4)
        sorter, "u64", "i64" or "f64" (int64 / uint64 / float64 keys) on a (8, 4) sorter; equal keys keep their input order in
        both directions."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._typed(), "keys", n, self.device)
        out, idx = _new_outputs(stream, keys, n)
        self._call(lib.osb200_argsort, keys.data_ptr(), out.data_ptr(), idx.data_ptr(), n, KEY_TYPES[key_type],
                   1 if descending else 0, stream=stream)
        return out, idx

    # -- 16-bit keys: two digit passes over 2-byte keys, on this (4-byte) sorter's workspace --------------------------
    def sort_keys16(self, keys: torch.Tensor, key_type: str, descending: bool = False, n: Optional[int] = None,
                    stream=None) -> torch.Tensor:
        """Stable in-place sort of int16 / uint16 / float16 / bfloat16 keys (osb200_sort_keys16).  key_type in KEY16_TYPES
        ("u16", "i16", "f16", "bf16") states how the bits are ordered; floats follow the total order of their bit patterns.
        Keys must start on a 16-byte boundary (OneSweepError status -1 otherwise).  Needs a sorter with key_bytes == 4."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, _TYPED_DTYPES_2, "keys", n, self.device)
        self._call(lib.osb200_sort_keys16, keys.data_ptr(), n, KEY16_TYPES[key_type], 1 if descending else 0, stream=stream)
        return keys

    def sort_pairs16(self, keys: torch.Tensor, values: torch.Tensor, key_type: str, descending: bool = False,
                     n: Optional[int] = None, stream=None):
        """sort_keys16 with 32-bit payloads that move with their keys (osb200_sort_pairs16).  Values need only their natural
        4-byte alignment.  Needs a (4, 4) sorter."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, _TYPED_DTYPES_2, "keys", n, self.device)
        _check_dev_tensor(values, _TYPED_DTYPES_4, "values", n, self.device)
        self._call(lib.osb200_sort_pairs16, keys.data_ptr(), values.data_ptr(), n, KEY16_TYPES[key_type],
                   1 if descending else 0, stream=stream)
        return keys, values

    def argsort16(self, keys: torch.Tensor, key_type: str, descending: bool = False, n: Optional[int] = None, stream=None):
        """argsort of 16-bit keys (osb200_argsort16): returns (sorted_keys, indices), new tensors of n elements, sorted_keys in
        the dtype of `keys` and indices as torch.int32 (positions >= 2^31 read as negative: ``indices.long() & 0xFFFFFFFF``).
        `keys` is left untouched.  Needs a (4, 4) sorter."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, _TYPED_DTYPES_2, "keys", n, self.device)
        out, idx = _new_outputs(stream, keys, n)
        self._call(lib.osb200_argsort16, keys.data_ptr(), out.data_ptr(), idx.data_ptr(), n, KEY16_TYPES[key_type],
                   1 if descending else 0, stream=stream)
        return out, idx

    # -- row sort: every row of a batch along its last dimension, no workspace (any sorter will do) -------------------
    def sort_rows(self, x: torch.Tensor, key_type: str, descending: bool = False, return_indices: bool = True,
                  inplace: bool = False, stream=None):
        """Stable sort of every row of `x` along its last dimension (osb200_sort_rows), the shape of
        ``torch.sort(x, dim=-1, stable=True)``.  `x` is a contiguous CUDA tensor of rank >= 1 of any of the ten key dtypes;
        key_type states how its bits are ordered: one of KEY16_TYPES for 2-byte dtypes, of KEY_TYPES of the dtype's width
        otherwise.  Floats follow the total order of their bit patterns; equal keys keep their order in both directions.

        Returns (values, indices) shaped like `x`, indices as torch.int32 positions within the row, or `values` alone with
        return_indices=False.  The outputs are new tensors allocated with torch.empty on the stream; inplace=True sorts `x`
        itself and returns it as `values`.  The last dimension may hold at most 16,384 keys (8,192 for 8-byte dtypes)."""
        kb, kt = self._ragged_keys(x, key_type)
        row_len = x.shape[-1]
        num_rows = x.numel() // row_len if row_len else 0
        out, idx = _new_outputs(stream, x, x.shape, return_indices, x if inplace else None)
        self._call(lib.osb200_sort_rows, x.data_ptr(), out.data_ptr(), idx.data_ptr() if idx is not None else None, num_rows,
                   row_len, kb, kt, 1 if descending else 0, stream=stream)
        return (out, idx) if return_indices else out

    def sort_long_rows(self, x: torch.Tensor, key_type: str, descending: bool = False, return_indices: bool = True,
                       inplace: bool = False, stream=None):
        """sort_rows for rows of any length (osb200_sort_long_rows): the same arguments, shapes and results.  Rows of at most
        16,384 keys (8,192 for 8-byte dtypes) are sorted by sort_rows' own kernels on any sorter.  Longer rows use this
        sorter's workspace: x.numel() may be at most max_n, the sorter's key_bytes must be at least x's element size, and
        return_indices=True needs value_bytes == 4 -- a (4, 4) sorter for 2- and 4-byte dtypes, a (8, 4) one for any."""
        kb, kt = self._ragged_keys(x, key_type)
        row_len = x.shape[-1]
        num_rows = x.numel() // row_len if row_len else 0
        out, idx = _new_outputs(stream, x, x.shape, return_indices, x if inplace else None)
        self._call(lib.osb200_sort_long_rows, x.data_ptr(), out.data_ptr(), idx.data_ptr() if idx is not None else None,
                   num_rows, row_len, kb, kt, 1 if descending else 0, stream=stream)
        return (out, idx) if return_indices else out

    # -- row top-k: the first k keys of every row's stable sort, no workspace (any sorter will do) ------------------------
    def topk_rows(self, x: torch.Tensor, k: int, key_type: str, largest: bool = True, sorted: bool = True, stream=None):
        """The k largest (or smallest) keys of every row of `x` along its last dimension and their positions
        (osb200_topk_rows), the shape of ``torch.topk(x, k, dim=-1, largest, sorted)``.  `x` and key_type as in sort_rows.
        The selected set is exactly the first k columns of the stable row sort (descending for largest): of equal keys at
        the boundary the lowest positions are taken.  sorted=True returns them in that order, bit-identical to
        ``sort_rows(x, descending=largest)`` cut to k; sorted=False returns the same pairs in an unspecified order.

        Returns (values, indices) shaped ``x.shape[:-1] + (k,)``, indices as torch.int32 positions within the row, allocated
        with torch.empty on the stream.  The rows may be of any length; k may be at most 16,384 (8,192 for 8-byte dtypes)
        and at most the row length."""
        kb, kt = self._ragged_keys(x, key_type)
        k = int(k)
        row_len = x.shape[-1]
        num_rows = x.numel() // row_len if row_len else 0
        shape = tuple(x.shape[:-1]) + (k,)
        out, idx = _new_outputs(stream, x, shape)
        self._call(lib.osb200_topk_rows, x.data_ptr(), out.data_ptr(), idx.data_ptr(), num_rows, row_len, k, kb, kt,
                   1 if largest else 0, 1 if sorted else 0, stream=stream)
        return out, idx

    def topk_long_rows(self, x: torch.Tensor, k: int, key_type: str, largest: bool = True, sorted: bool = True, stream=None):
        """topk_rows for any k up to the row length and rows of any length (osb200_topk_long_rows): the same arguments, shapes
        and results.  k above 16,384 (8,192 for 8-byte dtypes), and fewer rows than the GPU has SMs of more than 65,536 keys,
        split their rows across thread blocks on this sorter's workspace; every other call is topk_rows' own launch on any
        sorter.  The split path needs: x.numel() may be at most max_n, the sorter's key_bytes must be at least x's element size and its
        value_bytes 4 -- a (4, 4) sorter for 2- and 4-byte dtypes, a (8, 4) one for any."""
        kb, kt = self._ragged_keys(x, key_type)
        k = int(k)
        row_len = x.shape[-1]
        num_rows = x.numel() // row_len if row_len else 0
        shape = tuple(x.shape[:-1]) + (k,)
        out, idx = _new_outputs(stream, x, shape)
        self._call(lib.osb200_topk_long_rows, x.data_ptr(), out.data_ptr(), idx.data_ptr(), num_rows, row_len, k, kb, kt,
                   1 if largest else 0, 1 if sorted else 0, stream=stream)
        return out, idx

    # -- row select: given columns of every row's ascending stable sort ---------------------------------------------------
    def select_rows(self, x: torch.Tensor, ranks, key_type: str, return_indices: bool = True, stream=None):
        """Columns `ranks` of every row's ascending stable sort along the last dimension of `x`, and their positions within
        the row (osb200_select_rows).  `x` and key_type as in sort_rows; `ranks` a sequence of 1 to 16 strictly increasing
        ints below the row length, shared by every row.  Among equal keys a rank picks by position: the values are bit for
        bit those of ``sort_rows(x)[..., ranks]``.

        Returns (values, indices) shaped ``x.shape[:-1] + (len(ranks),)``, indices as torch.int32, or values alone with
        return_indices=False, allocated with torch.empty on the stream.  Rows of at most 16,384 keys (8,192 for 8-byte dtypes)
        need no workspace; longer rows use this sorter's alternate keys, for a bound that depends on the number of rows, the
        row length and len(ranks) only (see select_workspace_words)."""
        kb, kt = self._ragged_keys(x, key_type)
        ranks = [int(r) for r in ranks]
        if any(not 0 <= r <= 0xFFFFFFFF for r in ranks):
            raise ValueError(f"ranks must lie in [0, 2^32), got {ranks}")
        row_len = x.shape[-1]
        num_rows = math.prod(x.shape[:-1])
        arr = (ctypes.c_uint32 * max(len(ranks), 1))(*ranks)
        out, idx = _new_outputs(stream, x, tuple(x.shape[:-1]) + (len(ranks),), return_indices)
        self._call(lib.osb200_select_rows, x.data_ptr(), out.data_ptr(), idx.data_ptr() if idx is not None else None, num_rows,
                   row_len, arr, len(ranks), kb, kt, stream=stream)
        return (out, idx) if return_indices else out

    # -- segment select: given columns of every segment's ascending stable sort ---------------------------------------------
    def select_segments(self, x: torch.Tensor, offsets: torch.Tensor, ranks, key_type: str, return_indices: bool = True,
                        max_segment_len: Optional[int] = None, stream=None):
        """Columns `ranks` of every segment [offsets[s], offsets[s+1])'s ascending stable sort, and their positions within the
        segment (osb200_select_segments).  `x`, `offsets` and key_type as in sort_segments.  `ranks` is either a CUDA integer
        tensor [num_segments, R] of each segment's own ranks, non-decreasing per row (values outside [0, 2^32) become ranks
        that take no part), or a sequence of R ints shared by every segment; 1 <= R <= 16.  The values are bit for bit those
        of ``sort_long_segments(x)`` at ``offsets[s] + rank``.  A column whose rank is at or past the segment's length, every
        column of a row whose ranks decrease, and every column of a segment whose offsets decrease, pass x.numel() or exceed
        max_segment_len is padding: index -1 and the maximum of an integer dtype or the NaN 0x7F..F.

        Returns (values, indices) of shape [num_segments, R], indices as torch.int32, or values alone with
        return_indices=False, allocated with torch.empty on the stream.  max_segment_len None reads the longest segment with
        one device->host read; pass it when capturing a CUDA graph.  Up to 16,384 (8,192 for 8-byte dtypes) the call needs one
        uint32 per segment of workspace; above that it also uses this sorter's alternate payloads (value_bytes == 4), for a
        bound that depends on x.numel(), num_segments and R only (see select_segments_workspace)."""
        kb, kt = self._ragged_keys(x, key_type, offsets)
        segs = max(offsets.numel() - 1, 0)
        rk = _segment_ranks(ranks, segs, x.device, stream)
        if max_segment_len is None:
            max_segment_len = max(int((offsets[1:] - offsets[:-1]).max().item()), 0) if segs else 0
        out, idx = _new_outputs(stream, x, (segs, rk.shape[1]), return_indices)
        self._call(lib.osb200_select_segments, x.data_ptr() if x.numel() else None, out.data_ptr(),
                   idx.data_ptr() if idx is not None else None, x.numel(), offsets.data_ptr(), segs,
                   min(int(max_segment_len), 0xFFFFFFFF), rk.data_ptr(), rk.shape[1], kb, kt, stream=stream)
        return (out, idx) if return_indices else out

    # -- segment sort: ragged rows given by offsets -------------------------------------------------------------------------
    def sort_segments(self, x: torch.Tensor, offsets: torch.Tensor, key_type: str, descending: bool = False,
                      return_indices: bool = True, inplace: bool = False, max_segment_len: Optional[int] = None, stream=None):
        """Stable sort of every segment [offsets[s], offsets[s+1]) of `x` into the same positions (osb200_sort_segments):
        sort_rows for ragged rows.  `x` is a contiguous 1-D CUDA tensor of any of the ten key dtypes, key_type as in
        sort_rows; `offsets` a contiguous int64 tensor of num_segments + 1 offsets on the same device.  Floats follow the
        total order of their bit patterns; equal keys keep their order in both directions.

        Returns (values, indices), indices as torch.int32 positions within the segment (``indices + offsets[:-1]
        .repeat_interleave(lengths)`` makes them global), or `values` alone with return_indices=False.  The outputs are new
        tensors allocated with torch.empty on the stream, so positions outside every segment are uninitialised;
        inplace=True sorts `x` itself and returns it as `values`.  Segments longer than max_segment_len are not written, nor
        are segments whose offsets decrease or pass x.numel().  max_segment_len may be at most 16,384 (8,192 for 8-byte
        dtypes); None computes the longest segment here, with one device->host read -- pass it when capturing a CUDA graph.
        num_segments may be at most the sorter's max_n."""
        kb, kt = self._ragged_keys(x, key_type, offsets)
        segs = max(offsets.numel() - 1, 0)
        if max_segment_len is None:
            max_segment_len = max(int((offsets[1:] - offsets[:-1]).max().item()), 0) if segs else 0
        out, idx = _new_outputs(stream, x, x.shape, return_indices, x if inplace else None)
        self._call(lib.osb200_sort_segments, x.data_ptr(), out.data_ptr(), idx.data_ptr() if idx is not None else None,
                   x.numel(), offsets.data_ptr(), segs, int(max_segment_len), kb, kt, 1 if descending else 0, stream=stream)
        return (out, idx) if return_indices else out

    def sort_long_segments(self, x: torch.Tensor, offsets: torch.Tensor, key_type: str, descending: bool = False,
                           return_indices: bool = True, inplace: bool = False, max_segment_len: Optional[int] = None,
                           stream=None):
        """sort_segments for segments of any length (osb200_sort_long_segments): the same arguments, shapes and results, with
        max_segment_len any uint32 (None: the longest segment, read with one device->host read).  Up to 16,384 (8,192 for
        8-byte dtypes) it is sort_segments' own launch on any sorter.  Above that the longer segments use this sorter's
        workspace: x.numel() may be at most max_n, the sorter's key_bytes must be at least x's element size, and
        return_indices=True needs value_bytes == 4 -- a (4, 4) sorter for 2- and 4-byte dtypes, a (8, 4) one for any."""
        kb, kt = self._ragged_keys(x, key_type, offsets)
        segs = max(offsets.numel() - 1, 0)
        if max_segment_len is None:
            max_segment_len = max(int((offsets[1:] - offsets[:-1]).max().item()), 0) if segs else 0
        out, idx = _new_outputs(stream, x, x.shape, return_indices, x if inplace else None)
        self._call(lib.osb200_sort_long_segments, x.data_ptr(), out.data_ptr(), idx.data_ptr() if idx is not None else None,
                   x.numel(), offsets.data_ptr(), segs, int(max_segment_len), kb, kt, 1 if descending else 0, stream=stream)
        return (out, idx) if return_indices else out

    # -- segment top-k: row top-k for ragged rows given by offsets -----------------------------------------------------------
    def topk_segments(self, x: torch.Tensor, offsets: torch.Tensor, k: int, key_type: str, largest: bool = True,
                      sorted: bool = True, stream=None):
        """The k largest (or smallest) keys of every segment [offsets[s], offsets[s+1]) of `x` and their positions within
        the segment (osb200_topk_segments): topk_rows for ragged rows.  `x`, `offsets` and key_type as in sort_segments.
        Segment s's result is row s of a [num_segments, k] output.  Its first m = min(length, k) columns hold the first m keys
        of the segment's stable sort (descending for largest); of equal keys at the boundary the lowest positions are taken.
        sorted=True returns them in that order, sorted=False the same pairs in an unspecified order.  Columns m .. k-1 are
        padding: index -1 and the key that sorts last -- for largest=True 0, the minimum of a signed dtype or the float of
        all-ones bits (a NaN), for largest=False the maximum of an integer dtype or the NaN 0x7F..F.  Segments whose offsets
        decrease or pass x.numel() are all padding.

        Returns (values, indices) of shape [num_segments, k], indices as torch.int32, allocated with torch.empty on the
        stream.  k may be at most 16,384 (8,192 for 8-byte dtypes) and may exceed a segment's length; num_segments may be
        at most the sorter's max_n."""
        kb, kt = self._ragged_keys(x, key_type, offsets)
        k = int(k)
        if k < 0:
            raise ValueError(f"k must be >= 0, got {k}")
        segs = max(offsets.numel() - 1, 0)
        out, idx = _new_outputs(stream, x, (segs, k))
        self._call(lib.osb200_topk_segments, x.data_ptr() if x.numel() else None, out.data_ptr(), idx.data_ptr(), x.numel(),
                   offsets.data_ptr(), segs, k, kb, kt, 1 if largest else 0, 1 if sorted else 0, stream=stream)
        return out, idx

    def sort_bits(self, keys: torch.Tensor, begin_bit: int, end_bit: int, values: Optional[torch.Tensor] = None,
                  n: Optional[int] = None, stream=None):
        """Stable sort on the key bits [begin_bit, end_bit) only (osb200_sort_bits).  Keys must start on a 16-byte boundary
        (OneSweepError status -1 otherwise); values need only their natural 4-byte alignment, so any contiguous view will do."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._raw(), "keys", n, self.device)
        if values is not None:
            _check_dev_tensor(values, _TYPED_DTYPES_4, "values", n, self.device)
        self._call(lib.osb200_sort_bits, keys.data_ptr(), values.data_ptr() if values is not None else None, n, int(begin_bit),
                   int(end_bit), stream=stream)
        return keys if values is None else (keys, values)

    def segmented_sort(self, keys: torch.Tensor, segment_offsets: torch.Tensor, values: Optional[torch.Tensor] = None,
                       max_segment_len: Optional[int] = None, stream=None):
        """Sort every segment [offsets[i], offsets[i+1]) of `keys` (and `values`) ascending and stable, in place, one thread
        block per segment (osb200_segmented_sort_u32; reference: SplitSort, SegSort/SplitSort/SplitSort.cuh:702-938).
        `segment_offsets`: int64 device tensor of num_segments + 1 offsets.  `max_segment_len` (default: computed here, which
        costs a device->host read) must not exceed 16,384; segments longer than `max_segment_len` are left as they are."""
        _check_dev_tensor(keys, _KEY_DTYPES_4, "keys", keys.numel(), self.device)
        if values is not None:
            _check_dev_tensor(values, _TYPED_DTYPES_4, "values", keys.numel(), self.device)
        if segment_offsets.dtype != torch.int64 or not segment_offsets.is_cuda or not segment_offsets.is_contiguous():
            raise TypeError("segment_offsets must be a contiguous int64 CUDA tensor")
        segs = segment_offsets.numel() - 1
        if segs <= 0:
            return keys if values is None else (keys, values)
        if max_segment_len is None:
            max_segment_len = int((segment_offsets[1:] - segment_offsets[:-1]).max().item())
        self._call(lib.osb200_segmented_sort_u32, keys.data_ptr(), values.data_ptr() if values is not None else None,
                   segment_offsets.data_ptr(), segs, int(max_segment_len), stream=stream)
        return keys if values is None else (keys, values)

    def sort_pairs(self, keys: torch.Tensor, values: torch.Tensor, n: Optional[int] = None, stream=None):
        """Stable sort of keys[:n] with 32-bit payloads values[:n], in place.  Keys must start on a 16-byte boundary
        (OneSweepError status -1 otherwise); values need only their natural 4-byte alignment, so any contiguous view will do.
        On a (8, 4) sorter the keys are int64 / uint64 containers ordered by their unsigned bits (key type "u64")."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._raw(), "keys", n, self.device)
        _check_dev_tensor(values, _TYPED_DTYPES_4, "values", n, self.device)  # payloads are opaque 32-bit words
        if self.key_bytes == 8:
            return self.sort_pairs_typed(keys, values, "u64", False, n, stream)
        self._call(lib.osb200_sort_pairs_u32, keys.data_ptr(), values.data_ptr(), n, stream=stream)
        return keys, values

    def sort_host(self, keys, values=None, n: Optional[int] = None):
        """keys/values: numpy arrays or CPU torch tensors (pinned or pageable), sorted in place."""
        kp, kn, kb = _host_ptr(keys)
        n = kn if n is None else int(n)
        if kb != self.key_bytes:
            raise TypeError("key width does not match the sorter")
        if values is None:
            fn = lib.osb200_sort_host_keys_u32 if kb == 4 else lib.osb200_sort_host_keys_u64
            check(fn(self._h, kp, n), "osb200_sort_host_keys")
        else:
            vp, vn, vb = _host_ptr(values)
            if vb != 4 or vn < n:
                raise TypeError("values must be 4-byte elements, at least n long")
            check(lib.osb200_sort_host_pairs_u32(self._h, kp, vp, n), "osb200_sort_host_pairs_u32")
        return keys if values is None else (keys, values)

    # -- kernel-level entry points (parity tests) ---------------------------------------------------
    def global_histogram(self, keys: torch.Tensor, n: Optional[int] = None, stream=None) -> torch.Tensor:
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._typed(), "keys", n, self.device)
        hist = torch.empty(self.key_bytes * 256, dtype=torch.int64, device=keys.device)
        self._call(lib.osb200_global_histogram, keys.data_ptr(), n, hist.data_ptr(), stream=stream)
        return hist.view(self.key_bytes, 256)

    def digit_binning_pass(self, src: torch.Tensor, dst: torch.Tensor, radix_shift: int, src_values=None,
                           dst_values=None, n: Optional[int] = None, stream=None) -> None:
        n = src.numel() if n is None else int(n)
        _check_dev_tensor(src, self._typed(), "src", n, self.device)
        _check_dev_tensor(dst, self._typed(), "dst", n, self.device)
        if (src_values is None) != (dst_values is None):
            raise ValueError("src_values and dst_values go together")
        if src_values is not None:
            _check_dev_tensor(src_values, _TYPED_DTYPES_4, "src_values", n, self.device)
            _check_dev_tensor(dst_values, _TYPED_DTYPES_4, "dst_values", n, self.device)
        sv = src_values.data_ptr() if src_values is not None else None
        dv = dst_values.data_ptr() if dst_values is not None else None
        self._call(lib.osb200_digit_binning_pass, src.data_ptr(), dst.data_ptr(), sv, dv, n, int(radix_shift), stream=stream)

    def validate(self, keys: torch.Tensor, n: Optional[int] = None, stream=None) -> int:
        """Number of adjacent inversions (reference Validate, UtilityKernels.cuh:403-429); 0 == sorted."""
        n = keys.numel() if n is None else int(n)
        _check_dev_tensor(keys, self._typed(), "keys", n, self.device)
        err = ctypes.c_uint64(0)
        self._call(lib.osb200_validate, keys.data_ptr(), n, ctypes.byref(err), stream=stream)
        return int(err.value)


def _host_ptr(a):
    if isinstance(a, np.ndarray):
        if not a.flags["C_CONTIGUOUS"]:
            raise TypeError("host array must be contiguous")
        return a.ctypes.data, a.size, a.dtype.itemsize
    if isinstance(a, torch.Tensor) and not a.is_cuda:
        if not a.is_contiguous():
            raise TypeError("host tensor must be contiguous")
        return a.data_ptr(), a.numel(), a.element_size()
    raise TypeError("expected a numpy array or a CPU torch tensor")


def init_random(keys: torch.Tensor, and_count: int, seed: int, n: Optional[int] = None,
                payload: Optional[torch.Tensor] = None, payload_is_index: bool = False, stream=None) -> None:
    """The reference's input generator InitRandom<<<256,256>>> (UtilityKernels.cuh:53-117), on the device."""
    n = keys.numel() if n is None else int(n)
    _check_dev_tensor(keys, _TYPED_DTYPES_4, "keys", n)
    if payload is not None:
        _check_dev_tensor(payload, _TYPED_DTYPES_4, "payload", n, keys.device.index)
    pp = payload.data_ptr() if payload is not None else None
    check(lib.osb200_init_random_u32(keys.data_ptr(), pp, n, int(and_count), int(seed) & 0xFFFFFFFF,
                                     1 if payload_is_index else 0, _stream_ptr(stream)), "osb200_init_random_u32")


# --------------------------------------------------------------------------------------------------
# module-level Sort(keys[, values], n): the north-star call shape.  Sorters are cached per
# (device, key width, pairs) and grown on demand, so repeated calls do not re-allocate.
# --------------------------------------------------------------------------------------------------
_CACHE: dict = {}
# Sorters the cache has replaced with larger ones.  They stay open: a CUDA graph that captured a module call holds their
# buffers, and closing them would leave its replays reading and writing freed device memory.
_RETIRED: list = []


def _cached_sorter(device: int, key_bytes: int, value_bytes: int, n: int, stream_ptr: int) -> OneSweepSorter:
    # one handle per stream: the ABI allows one sort in flight per handle, and sorts on one stream are ordered
    k = (device, key_bytes, value_bytes, stream_ptr)
    s = _CACHE.get(k)
    if s is None or s.max_n < n:
        if s is not None:
            _RETIRED.append(s)
        s = OneSweepSorter(max(n, 1), key_bytes, value_bytes, device)
        _CACHE[k] = s
    return s


def release_cached_sorters() -> None:
    """Frees the sorters the module calls' cache has replaced with larger ones, after synchronizing every device they live
    on.  Safe only when no live CUDA graph uses them: a graph that captured a module call before its cached sorter grew
    keeps that sorter's buffers, so destroy such graphs first.  The sorters in use stay cached."""
    for d in sorted({s.device for s in _RETIRED}):
        torch.cuda.synchronize(d)
    while _RETIRED:
        _RETIRED.pop().close()


def _module_sorter(t, name: str, key_bytes: int, n: int, stream, dtypes=None, value_bytes: int = 4) -> OneSweepSorter:
    """The cached sorter of t's device and the stream for a module call on t, which must be a CUDA tensor (with a dtype of
    `dtypes`, if given).  The stream is read with t's device current."""
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise TypeError(f"{name} must be a CUDA tensor")
    if dtypes is not None and t.dtype not in dtypes:
        raise TypeError(f"{name}.dtype must be one of {tuple(dtypes)}")
    with torch.cuda.device(t.device.index):
        sp = _stream_ptr(stream)
    return _cached_sorter(t.device.index, key_bytes, value_bytes, n, sp)


def Sort(keys: torch.Tensor, values: Optional[torch.Tensor] = None, n: Optional[int] = None, stream=None):
    """OneSweep::Sort(keys[, values], n): ascending, stable, in place; returns its arguments."""
    n = keys.numel() if n is None else int(n)
    s = _module_sorter(keys, "keys", keys.element_size(), n, stream, value_bytes=0 if values is None else 4)
    if values is None:
        return s.sort_keys(keys, n, stream)
    return s.sort_pairs(keys, values, n, stream)


def argsort(keys: torch.Tensor, key_type: str, descending: bool = False, n: Optional[int] = None, stream=None):
    """Stable (sorted_keys, indices) of 32- or 64-bit keys, input untouched: OneSweepSorter.argsort on the stream's cached
    (4, 4) sorter, or its (8, 4) sorter for int64 / uint64 / float64 keys (one handle per stream, as for Sort)."""
    n = keys.numel() if n is None else int(n)
    wide = isinstance(keys, torch.Tensor) and keys.element_size() == 8
    s = _module_sorter(keys, "keys", 8 if wide else 4, n, stream)
    return s.argsort(keys, key_type, descending, n, stream)


def argsort16(keys: torch.Tensor, key_type: str, descending: bool = False, n: Optional[int] = None, stream=None):
    """Stable (sorted_keys, indices) of 16-bit keys (int16, uint16, float16, bfloat16; key_type "u16", "i16", "f16" or
    "bf16"), input untouched: OneSweepSorter.argsort16 on the stream's cached (4, 4) sorter, the one argsort uses."""
    n = keys.numel() if n is None else int(n)
    return _module_sorter(keys, "keys", 4, n, stream).argsort16(keys, key_type, descending, n, stream)


def sort_rows(x: torch.Tensor, descending: bool = False, return_indices: bool = True, stream=None):
    """``torch.sort(x, dim=-1, stable=True)`` for a contiguous CUDA tensor of int16, uint16, float16, bfloat16, int32, uint32,
    float32, int64, uint64 or float64: (values, int32 indices), or values alone.  The key type follows the dtype.
    OneSweepSorter.sort_rows on the stream's cached (4, 4) sorter, the one argsort uses (the row sort needs no workspace)."""
    s = _module_sorter(x, "x", 4, 1, stream, _ROW_KEY_TYPES)
    return s.sort_rows(x, _ROW_KEY_TYPES[x.dtype], descending, return_indices, False, stream)


# the longest row sort_rows takes, by element size: sort_long_rows needs a sorter's workspace only above it
_ROW_CAPACITY = {2: 16384, 4: 16384, 8: 8192}
# the long paths' tile: topk_long_rows splits only longer rows across thread blocks
_LONG_ROW_TILE = 8192


def sort_long_rows(x: torch.Tensor, descending: bool = False, return_indices: bool = True, stream=None):
    """sort_rows for rows of any length: ``torch.sort(x, dim=-1, stable=True)`` for a contiguous CUDA tensor of one of
    sort_rows' ten dtypes, returning (values, int32 positions within the row) or values alone.  Rows above sort_rows' limit
    run on the stream's cached (4, 4) sorter, the one argsort uses, or its (8, 4) sorter for 8-byte dtypes, grown to
    x.numel(); shorter rows on the (4, 4) one as in sort_rows."""
    kb = x.element_size() if isinstance(x, torch.Tensor) else 4
    row_len = x.shape[-1] if isinstance(x, torch.Tensor) and x.dim() else 0
    if row_len > _ROW_CAPACITY.get(kb, 16384):
        s = _module_sorter(x, "x", 8 if kb == 8 else 4, x.numel(), stream, _ROW_KEY_TYPES)
    else:
        s = _module_sorter(x, "x", 4, 1, stream, _ROW_KEY_TYPES)
    return s.sort_long_rows(x, _ROW_KEY_TYPES[x.dtype], descending, return_indices, False, stream)


def topk(x: torch.Tensor, k: int, largest: bool = True, sorted: bool = True, stream=None):
    """``torch.topk(x, k, dim=-1, largest, sorted)`` for a contiguous CUDA tensor of one of sort_rows' ten dtypes: (values,
    int32 positions within the row), with ties taken in input order -- exactly the first k columns of the stable row sort.
    The key type follows the dtype.  OneSweepSorter.topk_rows on the stream's cached (4, 4) sorter, the one argsort uses
    (the top-k needs no workspace)."""
    s = _module_sorter(x, "x", 4, 1, stream, _ROW_KEY_TYPES)
    return s.topk_rows(x, k, _ROW_KEY_TYPES[x.dtype], largest, sorted, stream)


def topk_long_rows(x: torch.Tensor, k: int, largest: bool = True, sorted: bool = True, stream=None):
    """topk for any k up to the row length and rows of any length: ``torch.topk(x, k, dim=-1, largest, sorted)`` for a
    contiguous CUDA tensor of one of sort_rows' ten dtypes, returning (values, int32 positions within the row), ties taken in
    input order.  Rows longer than 8,192 keys run on the stream's cached (4, 4) sorter, the one argsort uses, or its (8, 4)
    sorter for 8-byte dtypes, grown to x.numel(); shorter rows (which never take the split path) on the (4, 4) one as in
    topk."""
    kb = x.element_size() if isinstance(x, torch.Tensor) else 4
    row_len = x.shape[-1] if isinstance(x, torch.Tensor) and x.dim() else 0
    if row_len > _LONG_ROW_TILE:
        s = _module_sorter(x, "x", 8 if kb == 8 else 4, x.numel(), stream, _ROW_KEY_TYPES)
    else:
        s = _module_sorter(x, "x", 4, 1, stream, _ROW_KEY_TYPES)
    return s.topk_long_rows(x, k, _ROW_KEY_TYPES[x.dtype], largest, sorted, stream)


def select_workspace_words(num_rows: int, row_len: int, num_ranks: int, indices: bool = True) -> int:
    """The 32-bit words of a sorter's alternate keys that select_rows' split path (rows above sort_rows' limit) needs -- the
    bound of osb200_select_rows in include/onesweep_b200.h: per rank a 4-word state and 256 totals, and with indices one count
    per rank and tile of 8,192 keys plus the scan's chunk sums.  A (4, 4) sorter with max_n >= this many has the room."""
    def round4(w):
        return (w + 3) // 4 * 4
    tiles = (row_len + _LONG_ROW_TILE - 1) // _LONG_ROW_TILE
    words = round4(16 + num_rows * num_ranks * (4 + 256))
    if indices:
        words += round4(num_rows * num_ranks * tiles)
        chunks = (num_ranks * tiles + 4095) // 4096
        if chunks > 1:
            words += round4(num_rows * chunks)
    return words


def _select_sorter(x: torch.Tensor, rows: torch.Tensor, num_ranks: int, stream) -> OneSweepSorter:
    """The stream's cached (4, 4) sorter for select_rows on `rows` (a view of x), grown only when the split path's bound does
    not fit it -- never to x.numel()."""
    row_len = rows.shape[-1]
    if row_len > _ROW_CAPACITY.get(rows.element_size(), 16384):
        need = select_workspace_words(math.prod(rows.shape[:-1]), row_len, num_ranks)
        return _module_sorter(x, "x", 4, need, stream, _ROW_KEY_TYPES)
    return _module_sorter(x, "x", 4, 1, stream, _ROW_KEY_TYPES)


def _select_view(x: torch.Tensor, dim):
    """x as rows: dim None flattens it into one row of at most 2^32 - 1 keys, dim -1 (or x.dim() - 1) keeps its rows; any
    other dim raises ValueError."""
    if not isinstance(x, torch.Tensor):
        raise TypeError("x must be a CUDA tensor")
    if dim is None:
        if x.numel() > 0xFFFFFFFF:
            raise ValueError(f"dim=None takes at most 2^32 - 1 elements, got {x.numel()}")
        return x.reshape(1, x.numel())
    if dim not in (-1, max(x.dim(), 1) - 1):
        raise ValueError(f"only the last dimension (dim=-1) or dim=None can be reduced, got dim={dim}")
    return x if x.dim() else x.reshape(1)


def _reduced_shape(x: torch.Tensor, dim, keepdim: bool):
    if dim is None:
        return (1,) * x.dim() if keepdim else ()
    shape = tuple(x.shape[:-1])
    return shape + (1,) if keepdim and x.dim() else shape


def select_rows(x: torch.Tensor, ranks, dim=-1, return_indices: bool = True, stream=None):
    """Columns `ranks` (1 to 16 strictly increasing ints) of the ascending stable sort of every row of a contiguous CUDA tensor
    of one of sort_rows' ten dtypes: (values, int32 positions within the row) shaped ``rows.shape[:-1] + (len(ranks),)``, or
    values alone.  dim=-1 selects along the last dimension, dim=None in the flattened tensor (one row).  The key type follows
    the dtype.  OneSweepSorter.select_rows on the stream's cached (4, 4) sorter, grown only when rows above sort_rows' limit
    need more room than it has (select_workspace_words)."""
    rows = _select_view(x, dim)
    ranks = list(ranks)
    s = _select_sorter(x, rows, len(ranks), stream)
    return s.select_rows(rows, ranks, _ROW_KEY_TYPES[x.dtype], return_indices, stream)


def kthvalue(x: torch.Tensor, k: int, dim=-1, keepdim: bool = False, stream=None):
    """``torch.kthvalue(x, k, dim, keepdim)`` for a contiguous CUDA tensor of one of sort_rows' ten dtypes: the k-th smallest
    key (k 1-based) of every row and its int32 position, column k - 1 of the row's ascending stable sort -- of equal keys the
    one at the (k - taken)-th position among them.  dim is -1 (or the last dimension) or None (the flattened tensor).  Keys
    follow this library's total order: floats by their bits (-0.0 before +0.0, NaNs of either sign at the matching end)."""
    rows = _select_view(x, dim)
    k = int(k)
    if not 1 <= k <= rows.shape[-1]:
        raise ValueError(f"k={k} is outside 1 .. {rows.shape[-1]}")
    v, i = select_rows(rows, [k - 1], -1, True, stream)
    shape = _reduced_shape(x, dim, keepdim)
    return v.view(shape), i.view(shape)


def median(x: torch.Tensor, dim=None, keepdim: bool = False, stream=None):
    """``torch.median``: the lower median, rank (L - 1) // 2 of the ascending stable sort of rows of L keys.  dim=None returns
    the median of the flattened tensor as a 0-dim tensor; dim=-1 returns (values, int32 indices) of every row, as kthvalue."""
    rows = _select_view(x, dim)
    L = rows.shape[-1]
    if L == 0:
        raise ValueError("median of an empty row")
    if dim is None:
        return select_rows(rows, [(L - 1) // 2], -1, False, stream).view(())
    return kthvalue(x, (L - 1) // 2 + 1, dim, keepdim, stream)


_INTERPOLATIONS = ("linear", "lower", "higher", "midpoint", "nearest")


def quantile(x: torch.Tensor, q, dim=None, keepdim: bool = False, interpolation: str = "linear", stream=None):
    """``torch.quantile(x, q, dim, keepdim, interpolation)`` for a contiguous float32 or float64 CUDA tensor, bit for bit on
    inputs without -0.0 (torch's sort does not order the two zeros): rows with a NaN give NaN, as in torch.  q is a float, a
    sequence or a CPU tensor of values in [0, 1] (a CUDA q is refused: the ranks are needed on the host).  The ranks are ATen's,
    q * (L - 1) in x's dtype, then floor / ceil / round per mode; the distinct ranks, plus 0 and L - 1 (in this library's order
    a NaN sorts to one end, so they find NaN rows without another read), are selected 16 per call, and torch.lerp finishes the
    [rows, q] result.  Unlike torch.quantile it takes rows above 2^24 keys.  dim is None (the flattened tensor) or -1."""
    if not (isinstance(x, torch.Tensor) and x.dtype in (torch.float32, torch.float64)):
        raise TypeError("quantile() takes float32 or float64 tensors")
    if interpolation not in _INTERPOLATIONS:
        raise ValueError(f"interpolation must be one of {_INTERPOLATIONS}, got {interpolation!r}")
    if isinstance(q, torch.Tensor) and q.is_cuda:
        raise ValueError("q must be a float, a sequence or a CPU tensor: the ranks are computed on the host")
    qt = torch.as_tensor(q, dtype=x.dtype, device="cpu")
    if qt.dim() > 1:
        raise ValueError("q must be a scalar or a 1-D tensor")
    if not bool(((qt >= 0) & (qt <= 1)).all()):
        raise ValueError("q values must lie in [0, 1]")
    rows = _select_view(x, dim)
    L = rows.shape[-1]
    if L == 0:
        raise ValueError("quantile() input rows must be non-empty")
    num_rows = math.prod(rows.shape[:-1])
    qv = qt.reshape(-1)
    pos = qv * (L - 1)  # ATen's ranks, in x's dtype
    if interpolation == "lower":
        pos = pos.floor()
    elif interpolation == "higher":
        pos = pos.ceil()
    elif interpolation == "nearest":
        pos = pos.round()
    below = pos.to(torch.int64).clamp_(0, L - 1)
    above = pos.ceil().to(torch.int64).clamp_(0, L - 1)
    lerp = interpolation in ("linear", "midpoint")
    wanted = sorted(set(below.tolist()) | (set(above.tolist()) if lerp else set()) | {0, L - 1})
    flat = rows.reshape(num_rows, L)
    parts = [select_rows(flat, wanted[c:c + 16], -1, False, stream) for c in range(0, len(wanted), 16)]
    with torch.cuda.stream(stream):
        vals = parts[0] if len(parts) == 1 else torch.cat(parts, dim=-1)
        col = {r: j for j, r in enumerate(wanted)}
        dev = x.device
        res = vals[:, torch.tensor([col[r] for r in below.tolist()], device=dev)]
        if lerp:
            w = torch.full_like(qv, 0.5) if interpolation == "midpoint" else pos - below.to(x.dtype)
            hi = vals[:, torch.tensor([col[r] for r in above.tolist()], device=dev)]
            res = torch.lerp(res, hi, w.to(dev).expand_as(res))
        nan_row = vals[:, col[0]].isnan() | vals[:, col[L - 1]].isnan()
        res = torch.where(nan_row[:, None], torch.full_like(res, float("nan")), res)
        shape = _reduced_shape(x, dim, keepdim)
        if qt.dim() == 0:
            return res.reshape(shape)
        return res.t().reshape((qv.numel(),) + shape)


def _segment_ranks(ranks, segs: int, device, stream) -> torch.Tensor:
    """select_segments' ranks as a contiguous int32 [segs, R] tensor on `device` whose bits are the uint32 ranks: a CUDA
    integer tensor [segs, R] (values outside [0, 2^32) become 0xFFFFFFFF, a rank that takes no part), or a sequence of R
    ints shared by every segment."""
    if isinstance(ranks, torch.Tensor):
        if not ranks.is_cuda:
            raise TypeError("ranks must be a CUDA tensor [num_segments, R] or a sequence of ints; a CPU tensor is refused")
        if ranks.dtype.is_floating_point or ranks.dtype == torch.bool or ranks.dim() != 2 or ranks.shape[0] != segs:
            raise TypeError(f"ranks must be an integer CUDA tensor of shape [{segs}, R]")
        if ranks.device != device:
            raise ValueError(f"ranks live on {ranks.device}, x on {device}")
        if not 1 <= ranks.shape[1] <= 16:
            raise ValueError(f"1 to 16 ranks per segment, got {ranks.shape[1]}")
        if ranks.dtype in (torch.int32, torch.uint32) and ranks.is_contiguous():
            return ranks
        with torch.cuda.stream(stream):
            r = ranks.to(torch.int64)
            r = torch.where((r >= 0) & (r <= 0xFFFFFFFF), r, 0xFFFFFFFF)
            return (r - ((r >> 31) << 32)).to(torch.int32).contiguous()  # the uint32 bits as int32
    ranks = [int(r) for r in ranks]
    if not 1 <= len(ranks) <= 16:
        raise ValueError(f"1 to 16 ranks, got {len(ranks)}")
    if any(not 0 <= r <= 0xFFFFFFFF for r in ranks):
        raise ValueError(f"ranks must lie in [0, 2^32), got {ranks}")
    row = np.array(ranks, dtype=np.uint32).view(np.int32)
    with torch.cuda.stream(stream):
        return torch.from_numpy(row).to(device).expand(max(segs, 1), len(ranks))[:segs].contiguous()


def select_segments_workspace(n: int, num_segments: int, num_ranks: int, key_bytes: int = 4, indices: bool = True) -> int:
    """The 32-bit words of a sorter's alternate payloads that select_segments needs when max_segment_len exceeds sort_segments'
    limit -- the bound of osb200_select_segments in include/onesweep_b200.h: per long segment and rank a 4-word state and 256
    totals, the long list and its tile map, and with indices one count per rank and tile of 8,192 keys plus the scan's chunk
    sums; 0 where the long path cannot run (n at most 16,384, or 8,192 for 8-byte keys).  This is the library's
    osb200_select_segments_workspace_words.  A (4, 4) sorter with max_n >= max(this, num_segments) has the room."""
    def round4(w):
        return (w + 3) // 4 * 4
    long_min = _ROW_CAPACITY.get(key_bytes, 16384) + 1
    if n < long_min or num_segments == 0:
        return 0  # max_segment_len is clamped to n: no segment can take the long path
    listed = min(n // long_min, num_segments)
    tiles = (n + _LONG_ROW_TILE - 1) // _LONG_ROW_TILE + listed
    words = round4(16 + listed * num_ranks * (4 + 256)) + round4(listed) + 2 * round4(listed + 1)
    if indices:
        words += round4(tiles * num_ranks) + round4((tiles + 15) // 16 + listed)
    return words


def _segment_args(x, offsets, max_segment_len):
    """(number of segments, max_segment_len) of a module segment call; None reads the longest segment (one device->host read)"""
    if not (isinstance(offsets, torch.Tensor) and offsets.is_cuda):
        raise TypeError("offsets must be a CUDA tensor")
    segs = max(offsets.numel() - 1, 0)
    if max_segment_len is None:
        max_segment_len = max(int((offsets[1:] - offsets[:-1]).max().item()), 0) if segs else 0
    return segs, int(max_segment_len)


def select_segments(x: torch.Tensor, offsets: torch.Tensor, ranks, return_indices: bool = True, max_segment_len: Optional[int] = None,
                    stream=None):
    """Columns `ranks` of the ascending stable sort of every segment [offsets[s], offsets[s+1]) of a contiguous 1-D CUDA tensor
    of one of sort_rows' ten dtypes: (values, int32 positions within the segment) of shape [num_segments, R], or values alone;
    see OneSweepSorter.select_segments for `ranks` and the padding.  The key type follows the dtype.  Runs on the stream's
    cached (4, 4) sorter, grown to the number of segments, and with max_segment_len above sort_segments' limit only to
    select_segments_workspace's bound -- never to x.numel()."""
    segs, max_len = _segment_args(x, offsets, max_segment_len)
    if isinstance(ranks, torch.Tensor):
        if not ranks.is_cuda:
            raise TypeError("ranks must be a CUDA tensor [num_segments, R] or a sequence of ints; a CPU tensor is refused")
    else:
        ranks = [int(r) for r in ranks]  # (read once: a generator would be consumed here)
    num_ranks = ranks.shape[-1] if isinstance(ranks, torch.Tensor) else len(ranks)
    kb = x.element_size() if isinstance(x, torch.Tensor) else 4
    need = max(segs, 1)
    if max_len > _ROW_CAPACITY.get(kb, 16384):
        need = max(need, select_segments_workspace(x.numel(), segs, num_ranks, kb, return_indices))
    s = _module_sorter(x, "x", 4, need, stream, _ROW_KEY_TYPES)
    return s.select_segments(x, offsets, ranks, _ROW_KEY_TYPES[x.dtype], return_indices, max_len, stream)


def median_segments(x: torch.Tensor, offsets: torch.Tensor, max_segment_len: Optional[int] = None, stream=None):
    """The lower median of every segment, rank (L - 1) // 2 of its ascending stable sort: (values, int32 positions within the
    segment) of shape [num_segments]; an empty segment is padding (see OneSweepSorter.select_segments).  The ranks are
    computed on the device from the offsets."""
    segs, max_len = _segment_args(x, offsets, max_segment_len)
    with torch.cuda.stream(stream):
        lengths = offsets[1:] - offsets[:-1]
        ranks = torch.where(lengths > 0, (lengths - 1) // 2, -1)[:, None]
    v, i = select_segments(x, offsets, ranks, True, max_len, stream)
    return v.view(segs), i.view(segs)


def quantile_segments(x: torch.Tensor, offsets: torch.Tensor, q, interpolation: str = "linear", max_segment_len: Optional[int] = None,
                      stream=None):
    """``torch.quantile(x[offsets[s]:offsets[s+1]], q, interpolation=...)`` of every segment of a contiguous 1-D float32 or
    float64 CUDA tensor: [Q, num_segments], or [num_segments] for a scalar q, bit for bit on inputs without -0.0 or NaN.
    Segments with a NaN give NaN, as in torch, but the canonical NaN rather than the NaN bits torch returns; empty segments
    give NaN.  Past 2^24 keys (float32), which torch.quantile refuses, q * (L - 1) may round past L - 1: the rank is clamped
    to L - 1.  q is a float, a sequence or a CPU tensor of values in [0, 1].
    ATen's ranks are computed on the device from the lengths -- q * (L - 1) in x's dtype, then floor / ceil / round per
    mode -- with ranks 0 and L - 1 added (a NaN sorts to one end, so they find NaN segments without another read); each
    segment's ranks are sorted on the device and selected 16 per call, and torch.lerp finishes.  With max_segment_len given
    nothing waits for the device."""
    if not (isinstance(x, torch.Tensor) and x.dtype in (torch.float32, torch.float64)):
        raise TypeError("quantile_segments() takes float32 or float64 tensors")
    if interpolation not in _INTERPOLATIONS:
        raise ValueError(f"interpolation must be one of {_INTERPOLATIONS}, got {interpolation!r}")
    if isinstance(q, torch.Tensor) and q.is_cuda:
        raise ValueError("q must be a float, a sequence or a CPU tensor")
    qt = torch.as_tensor(q, dtype=x.dtype, device="cpu")
    if qt.dim() > 1:
        raise ValueError("q must be a scalar or a 1-D tensor")
    if not bool(((qt >= 0) & (qt <= 1)).all()):
        raise ValueError("q values must lie in [0, 1]")
    segs, max_len = _segment_args(x, offsets, max_segment_len)
    nq = qt.numel()
    lerp = interpolation in ("linear", "midpoint")
    with torch.cuda.stream(stream):
        qv = qt.reshape(-1).to(x.device)
        lengths = offsets[1:] - offsets[:-1]
        last = (lengths - 1).clamp_(min=0)
        lastf = last.to(x.dtype)[:, None]
        pos = torch.minimum(qv[None, :] * lastf, lastf)  # ATen's ranks, in x's dtype (clamped: they can round past L - 1)
        if interpolation == "lower":
            pos = pos.floor()
        elif interpolation == "higher":
            pos = pos.ceil()
        elif interpolation == "nearest":
            pos = pos.round()
        below = pos.to(torch.int64)
        above = pos.ceil().to(torch.int64)
        cols = [below, above] if lerp else [below]
        wanted = torch.cat(cols + [torch.zeros_like(last)[:, None], last[:, None]], dim=1)  # [S, M]
        ranks, perm = torch.sort(wanted, dim=1)
    parts = [select_segments(x, offsets, ranks[:, c:c + 16], False, max_len, stream) for c in range(0, ranks.shape[1], 16)]
    with torch.cuda.stream(stream):
        vals = parts[0] if len(parts) == 1 else torch.cat(parts, dim=1)
        vals = torch.empty_like(vals).scatter_(1, perm, vals)  # back to the order of `wanted`
        res = vals[:, :nq]
        if lerp:
            w = torch.full_like(pos, 0.5) if interpolation == "midpoint" else pos - below.to(x.dtype)
            res = torch.lerp(res, vals[:, nq:2 * nq], w)
        m = vals.shape[1]
        bad = vals[:, m - 2].isnan() | vals[:, m - 1].isnan() | (lengths <= 0)
        res = torch.where(bad[:, None], torch.full_like(res, float("nan")), res)
        return res[:, 0] if qt.dim() == 0 else res.t().contiguous()


def sort_segments(x: torch.Tensor, offsets: torch.Tensor, descending: bool = False, return_indices: bool = True,
                  max_segment_len: Optional[int] = None, stream=None):
    """Stable sort of every segment [offsets[s], offsets[s+1]) of a contiguous 1-D CUDA tensor of one of sort_rows' ten
    dtypes: (values, int32 positions within the segment), or values alone.  The key type follows the dtype.
    OneSweepSorter.sort_segments on the stream's cached (4, 4) sorter, the one argsort uses, grown to the number of segments
    (the call keeps one uint32 per segment in the sorter's workspace); see there for max_segment_len and what is written."""
    s = _module_sorter(x, "x", 4, max(offsets.numel() - 1, 1), stream, _ROW_KEY_TYPES)
    return s.sort_segments(x, offsets, _ROW_KEY_TYPES[x.dtype], descending, return_indices, False, max_segment_len, stream)


def sort_long_segments(x: torch.Tensor, offsets: torch.Tensor, descending: bool = False, return_indices: bool = True,
                       max_segment_len: Optional[int] = None, stream=None):
    """sort_segments for segments of any length: (values, int32 positions within the segment), or values alone, for a
    contiguous 1-D CUDA tensor of one of sort_rows' ten dtypes.  With max_segment_len above sort_segments' limit (None: the
    longest segment, one device->host read) it runs on the stream's cached (4, 4) sorter, or its (8, 4) sorter for 8-byte
    dtypes, grown to max(x.numel(), number of segments); otherwise on the (4, 4) one grown to the number of segments, as in
    sort_segments."""
    segs = max(offsets.numel() - 1, 0) if isinstance(offsets, torch.Tensor) else 0
    if max_segment_len is None and segs:
        max_segment_len = max(int((offsets[1:] - offsets[:-1]).max().item()), 0)
    kb = x.element_size() if isinstance(x, torch.Tensor) else 4
    if (max_segment_len or 0) > _ROW_CAPACITY.get(kb, 16384):
        s = _module_sorter(x, "x", 8 if kb == 8 else 4, max(x.numel(), segs), stream, _ROW_KEY_TYPES)
    else:
        s = _module_sorter(x, "x", 4, max(segs, 1), stream, _ROW_KEY_TYPES)
    return s.sort_long_segments(x, offsets, _ROW_KEY_TYPES[x.dtype], descending, return_indices, False, max_segment_len, stream)


def topk_segments(x: torch.Tensor, offsets: torch.Tensor, k: int, largest: bool = True, sorted: bool = True, stream=None):
    """The k largest (or smallest) keys of every segment [offsets[s], offsets[s+1]) of a contiguous 1-D CUDA tensor of one of
    sort_rows' ten dtypes, and their int32 positions within the segment: (values, indices) of shape [num_segments, k],
    padded past each segment's length with index -1 and the key that sorts last.  The key type follows the dtype.
    OneSweepSorter.topk_segments on the stream's cached (4, 4) sorter, the one argsort uses, grown to the number of segments
    (the call keeps one uint32 per segment in the sorter's workspace)."""
    s = _module_sorter(x, "x", 4, max(offsets.numel() - 1, 1), stream, _ROW_KEY_TYPES)
    return s.topk_segments(x, offsets, k, _ROW_KEY_TYPES[x.dtype], largest, sorted, stream)


class OneSweepDispatcher:
    """Mirror of the reference's class OneSweepDispatcher (Sort/OneSweepDispatcher.cuh:17-392).

    Same constructor arguments (keysOnly, maxSize) and the same public methods; like the reference it owns
    m_sort / m_sortPayload and sorts them in place.  Tests print nothing unless ``verbose``.
    """

    k_partitionSize = 7680  # the reference's sweep bounds (OneSweepDispatcher.cuh:23,98) are kept for TestAll*

    def __init__(self, keysOnly: bool, maxSize: int, verbose: bool = False):
        self.k_keysOnly, self.k_maxSize, self.verbose = bool(keysOnly), int(maxSize), verbose
        self.m_sort = torch.empty(self.k_maxSize, dtype=torch.int32, device="cuda")
        self.m_sortPayload = None if keysOnly else torch.empty(self.k_maxSize, dtype=torch.int32, device="cuda")
        self._sorter = OneSweepSorter(self.k_maxSize, 4, 0 if keysOnly else 4)

    # reference: DispatchKernelsKeysOnly / DispatchKernelsPairs (private there; :311-363)
    def DispatchKernelsKeysOnly(self, size: int) -> None:
        self._sorter.sort_keys(self.m_sort, size)

    def DispatchKernelsPairs(self, size: int) -> None:
        self._sorter.sort_pairs(self.m_sort, self.m_sortPayload, size)

    # reference: DispatchValidateKeys / DispatchValidatePairs (:365-391)
    def DispatchValidateKeys(self, size: int) -> bool:
        return self._sorter.validate(self.m_sort, size) == 0

    def DispatchValidatePairs(self, size: int) -> bool:
        # the reference relies on payload == key (UtilityKernels.cuh:432-479)
        return self._sorter.validate(self.m_sort, size) == 0 and self._sorter.validate(self.m_sortPayload, size) == 0

    def _sizes(self, small_step: int, large_exps):
        for i in range(self.k_partitionSize, self.k_partitionSize * 2 + 1, small_step):
            yield i, i
        for e in large_exps:
            if (1 << e) <= self.k_maxSize:
                yield 1 << e, e

    def TestAllKeysOnly(self, small_step: int = 1, large_exps=(26, 27, 28)) -> tuple[int, int]:
        """reference :87-134 -- every n in [7680, 15360] then 2^26..2^28; returns (passed, total)."""
        passed = total = 0
        for n, seed in self._sizes(small_step, large_exps):
            init_random(self.m_sort, ENTROPY_PRESET_1, seed, n)
            self.DispatchKernelsKeysOnly(n)
            ok = self.DispatchValidateKeys(n)
            passed += ok
            total += 1
            if not ok and self.verbose:
                print(f"Test failed at size {n}")
        return passed, total

    def TestAllPairs(self, small_step: int = 1, large_exps=(26, 27, 28)) -> tuple[int, int]:
        """reference :136-191"""
        passed = total = 0
        for n, seed in self._sizes(small_step, large_exps):
            init_random(self.m_sort, ENTROPY_PRESET_1, seed, n, payload=self.m_sortPayload)
            self.DispatchKernelsPairs(n)
            ok = self.DispatchValidatePairs(n)
            passed += ok
            total += 1
            if not ok and self.verbose:
                print(f"Test failed at size {n}")
        return passed, total

    def _batch(self, size: int, batchCount: int, seed: int, entropyPreset: int, pairs: bool) -> float:
        if size > self.k_maxSize:
            raise ValueError("Error, requested test size exceeds max initialized size.")
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        total_ms = 0.0
        for i in range(batchCount + 1):  # i == 0 is the discarded warm-up (reference :228)
            init_random(self.m_sort, entropyPreset, i + seed, size, payload=self.m_sortPayload if pairs else None)
            torch.cuda.synchronize()
            start.record()
            (self.DispatchKernelsPairs if pairs else self.DispatchKernelsKeysOnly)(size)
            stop.record()
            stop.synchronize()
            if i:
                total_ms += start.elapsed_time(stop)
        keys_per_sec = size / (total_ms / 1000.0) * batchCount
        if self.verbose:
            print(f"Total time elapsed: {total_ms / 1000.0}\nEstimated speed at {size} 32-bit elements: {keys_per_sec:E} keys/sec")
        return keys_per_sec

    def BatchTimingKeysOnly(self, size: int, batchCount: int, seed: int, entropyPreset: int = ENTROPY_PRESET_1) -> float:
        """reference :193-239; returns keys/sec."""
        return self._batch(size, batchCount, seed, entropyPreset, False)

    def BatchTimingPairs(self, size: int, batchCount: int, seed: int, entropyPreset: int = ENTROPY_PRESET_1) -> float:
        """reference :241-293; returns pairs/sec."""
        if self.k_keysOnly:
            raise ValueError("Error, object was initialized for keys only.")
        return self._batch(size, batchCount, seed, entropyPreset, True)
