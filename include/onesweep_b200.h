/*
 * onesweep_b200.h -- C-ABI of the H100-native OneSweep radix sort (libonesweep_b200.so).
 *
 * This is the drop-in boundary for the ONE hot path of b0nes164/GPUSorting that this repository
 * rebuilds: the CUDA OneSweep 8-bit LSD radix sort.  Plain C types only (no torch / C++ types).
 * Each entry point cites the reference interface it replaces; paths are relative to
 * /root/reference/GPUSortingCUDA/ unless stated otherwise.
 *
 * Conventions
 *   - All `d_*` pointers are device pointers on the handle's device.  Keys must be 16-byte aligned on every entry point
 *     that checks them -- the sorts, osb200_global_histogram and osb200_digit_binning_pass return OSB200_ERR_INVALID_ARG
 *     for keys at any other offset (the reference assumes this too: Sort/OneSweep.cu:77 reinterpret_cast<uint4*>).
 *     Values need only their natural 4-byte alignment: a view that starts at any element of a larger buffer may be
 *     passed as d_values.  osb200_argsort needs all three of its pointers 16-byte aligned.
 *   - The sorted result is returned IN the caller's key/value buffers (even number of passes, like
 *     Sort/OneSweepDispatcher.cuh:325-335 which ends in m_sort).
 *   - Calls are asynchronous on `stream` (a cudaStream_t passed as void*; NULL = default stream) and
 *     never synchronise the host, unlike the reference (cudaDeviceSynchronize inside the dispatch,
 *     OneSweepDispatcher.cuh:318).  One sort in flight per handle; distinct handles are independent.
 *   - The single-GPU calls may be captured into a CUDA graph (cudaStreamBeginCapture, torch.cuda.graph) and the graph
 *     replayed with new data in the same buffers.  The chained-scan descriptors carry a per-pass epoch that the host
 *     passes at launch, so a replay reuses the epochs of the capture: a sort enqueued on a capturing stream therefore
 *     also clears the descriptors of its tiles (2 KiB per tile) before its first pass and after its last.  Eager calls
 *     do not.  The sharded sort (osb200_sharded_*) is not supported under capture.
 *   - Return value: 0 on success, a negative osb200_status otherwise.  Nothing aborts or prints (the
 *     reference ignores every CUDA error and printf()s on misuse, OneSweepDispatcher.cuh:195-199).
 *   - n == 0 or 1 is a successful no-op; n > max_n (from create) is OSB200_ERR_SIZE.
 *   - There is NO CPU fallback: if no sm_90 device / driver is usable, create fails.
 */
#ifndef ONESWEEP_B200_H_
#define ONESWEEP_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(OSB200_BUILDING) && defined(__GNUC__)
#define OSB200_API __attribute__((visibility("default")))
#else
#define OSB200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct osb200_sorter* osb200_handle;          /* opaque single-GPU sorter  */
typedef struct osb200_sharded_sorter* osb200_sharded_handle; /* opaque multi-GPU sorter */

typedef enum osb200_status {
    OSB200_OK = 0,
    OSB200_ERR_INVALID_ARG = -1, /* null handle/pointer, bad key/value width, misaligned keys    */
    OSB200_ERR_SIZE = -2,        /* n > max_n of the handle                                        */
    OSB200_ERR_UNSUPPORTED = -3, /* combination not built (e.g. u64 keys with values)              */
    OSB200_ERR_NO_DEVICE = -4,   /* no CUDA device of compute capability 10.x                      */
    OSB200_ERR_ALLOC = -5,       /* device allocation failed                                       */
    OSB200_ERR_NCCL = -6,        /* NCCL failure in the sharded path                               */
    OSB200_ERR_CUDA = -1000      /* -(1000 + cudaError_t) for any other CUDA runtime error         */
} osb200_status;

/* ABI version of this header (major*1000 + minor). */
OSB200_API int osb200_version(void);
/* Static string for a status code returned by any function below. */
OSB200_API const char* osb200_status_string(int status);

/* ------------------------------------------------------------------------------------------------
 * Sorter object.  Replaces  OneSweepDispatcher::OneSweepDispatcher(bool keysOnly, uint32_t maxSize)
 * / ~OneSweepDispatcher()  (Sort/OneSweepDispatcher.cuh:42-83): owns the alternate (ping-pong)
 * buffers, the global histogram, the tile tickets and the chained-scan tile descriptors.  Unlike the
 * reference the caller owns the keys/values being sorted (as in the Unity API,
 * /root/reference/GPUSortingUnity/Runtime/OneSweep.cs:297-306).
 *   key_bytes   4 (uint32 keys, the reference's only CUDA type) or 8 (uint64 keys, 8 digit passes)
 *   value_bytes 0 (keys only == keysOnly=true) or 4 (uint32 payload == keysOnly=false)
 *   max_n       largest n a sort call may pass (reference: maxSize), up to 2^34
 * The device is the calling thread's current CUDA device.
 * key_bytes 8 with value_bytes 4 returns OSB200_ERR_UNSUPPORTED here: that shape comes from osb200_create_pairs64.
 * ---------------------------------------------------------------------------------------------- */
OSB200_API int osb200_create(osb200_handle* out, uint64_t max_n, int key_bytes, int value_bytes);
/* A handle for 64-bit keys with uint32 payloads (key_bytes 8, value_bytes 4): osb200_sort_pairs_typed and osb200_argsort with
 * OSB200_KEY_U64, _I64 or _F64 keys.  Its workspace is alternate keys (8 * max_n bytes) and payloads (4 * max_n), the tile
 * descriptors and reductions, and the control block; osb200_workspace_bytes(max_n, 8, 4) is what it allocates.  The keys-only
 * calls (osb200_sort_keys_u64, osb200_sort_keys_typed, osb200_sort_host_keys_u64) work on it as on a (8, 0) handle.
 * osb200_sort_pairs_u32, the host-buffer pairs call, the segmented sort and osb200_sort_bits with values do not take 64-bit
 * keys: they return OSB200_ERR_INVALID_ARG on it, as on any 8-byte handle.  Argument errors and OSB200_ERR_NO_DEVICE as for
 * osb200_create (a null `out`, max_n == 0 or max_n > 2^34: OSB200_ERR_INVALID_ARG). */
OSB200_API int osb200_create_pairs64(osb200_handle* out, uint64_t max_n);
OSB200_API int osb200_destroy(osb200_handle h);
/* Device bytes a handle with these parameters allocates (alt buffers + control state). */
OSB200_API uint64_t osb200_workspace_bytes(uint64_t max_n, int key_bytes, int value_bytes);

/* ------------------------------------------------------------------------------------------------
 * Sort entry points.
 *   osb200_sort_keys_u32      replaces OneSweepDispatcher::DispatchKernelsKeysOnly(uint32_t size)
 *                             (Sort/OneSweepDispatcher.cuh:311-336)
 *   osb200_sort_pairs_u32     replaces OneSweepDispatcher::DispatchKernelsPairs(uint32_t size)
 *                             (Sort/OneSweepDispatcher.cuh:338-363); stable: equal keys keep their
 *                             input order (in-order ranking, Sort/OneSweep.cu:207-253)
 *   osb200_sort_keys_u64      no CUDA reference (SURVEY D3); same plan with 8 digit places, shape of
 *                             GPUSortingUnity/Runtime/OneSweep.cs:297-306 Sort(...)
 * ---------------------------------------------------------------------------------------------- */
OSB200_API int osb200_sort_keys_u32(osb200_handle h, uint32_t* d_keys, uint64_t n, void* stream);
OSB200_API int osb200_sort_pairs_u32(osb200_handle h, uint32_t* d_keys, uint32_t* d_values, uint64_t n, void* stream);
OSB200_API int osb200_sort_keys_u64(osb200_handle h, uint64_t* d_keys, uint64_t n, void* stream);

/* Typed keys and descending order (the reference has them only in its HLSL path: IntToUint / FloatToUint and inverses,
 * GPUSortingD3D12/Shaders/SortCommon.hlsl:134-154; descending :594-656).  The order-preserving bit transform is fused
 * into the first pass (and the histogram) and undone in the last pass's stores: no extra traffic.  Floats follow the
 * IEEE total order of their bit patterns (-0.0 < +0.0, NaNs at the ends), as the reference's transform does.
 * Descending is the complement of the transformed key, so equal keys KEEP their input order (stable) -- unlike the
 * reference's index reversal, which reverses ties.  key_type must match the handle's key width.
 * osb200_sort_pairs_typed needs value_bytes == 4: a (4, 4) handle with 32-bit key types, or a (8, 4) handle
 * (osb200_create_pairs64) with 64-bit ones.  Keys must be 16-byte aligned, values 4-byte aligned. */
typedef enum osb200_key_type {
    OSB200_KEY_U32 = 0, OSB200_KEY_I32 = 1, OSB200_KEY_F32 = 2, OSB200_KEY_U64 = 3, OSB200_KEY_I64 = 4, OSB200_KEY_F64 = 5
} osb200_key_type;
OSB200_API int osb200_sort_keys_typed(osb200_handle h, void* d_keys, uint64_t n, int key_type, int descending, void* stream);
OSB200_API int osb200_sort_pairs_typed(osb200_handle h, void* d_keys, uint32_t* d_values, uint64_t n, int key_type,
                                       int descending, void* stream);

/* Argsort: the stable sort of d_keys_in[0..n) and its permutation, leaving the input as it is (the shape of torch.sort).
 * d_keys_in is read and never written; d_keys_out receives the keys sorted, and d_indices[i] the input position of
 * d_keys_out[i].  Equal keys keep their input order in both directions (the stable descending order of
 * osb200_sort_pairs_typed).  key_type is ordered as in osb200_sort_keys_typed: OSB200_KEY_U32, _I32 or _F32 on a handle
 * with key_bytes == 4 and value_bytes == 4, OSB200_KEY_U64, _I64 or _F64 on a (8, 4) handle (osb200_create_pairs64).  The
 * handle's alternate buffers are the ping-pong partners of d_keys_out and d_indices, so no other workspace is used.  The
 * indices are made on the device rather than loaded: the histogram and the first executed digit pass read the keys from
 * d_keys_in, and that pass writes each key's own position as its payload (every later pass is the pairs pass; a sort of at
 * most 16,384 keys, 8,192 64-bit keys, is one launch of the single-block sort).  Against copying the keys, writing 0..n-1
 * and calling osb200_sort_pairs_typed this saves the copy, the iota and a payload read.
 * All three pointers must be 16-byte aligned, and none of the three arrays (keys key_bytes * n bytes, indices 4n) may
 * overlap another.
 * Returns OSB200_ERR_INVALID_ARG for a null, misaligned or overlapping pointer, a handle without payloads or a key_type of
 * the other width; OSB200_ERR_UNSUPPORTED unless option "variant" is 2 (the default); OSB200_ERR_SIZE when n > max_n or
 * n > 2^32 (the indices are uint32).  n == 0 is a no-op; n == 1 writes d_keys_out[0] = d_keys_in[0] and d_indices[0] = 0.
 * Asynchronous and graph-capturable like the other single-GPU calls. */
OSB200_API int osb200_argsort(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                              int key_type, int descending, void* stream);

/* 16-bit keys: uint16, int16, IEEE half (float16) and bfloat16, sorted in TWO digit passes over 2-byte keys (instead of
 * converting them to float32 and running four passes over 4-byte keys).  They run on a handle with key_bytes == 4, which
 * owns all the workspace they need; a caller sorting both float32 and bfloat16 keys uses one handle.
 *   osb200_sort_keys16   as osb200_sort_keys_typed: d_keys sorted in place; any 4-byte handle
 *   osb200_sort_pairs16  as osb200_sort_pairs_typed: uint32 payloads move with their keys; needs value_bytes == 4
 *   osb200_argsort16     as osb200_argsort: d_keys_in untouched, d_keys_out sorted, d_indices[i] = input position of
 *                        d_keys_out[i] (uint32, so n <= 2^32); needs value_bytes == 4
 * Stable in both directions (descending is the complement of the transformed key).  F16 and BF16 are ordered by the total
 * order of their bit patterns (-NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN) and share one transform.
 * Keys must be 16-byte aligned (argsort16: all three pointers); values need 4-byte alignment; the argsort16 arrays (keys 2n
 * bytes, indices 4n bytes) must not overlap.  Returns OSB200_ERR_INVALID_ARG for a handle with key_bytes != 4 (or without
 * payloads, for pairs16 / argsort16), a key_type outside osb200_key16_type, a null, misaligned or overlapping pointer;
 * OSB200_ERR_SIZE for n > max_n (argsort16 also for n > 2^32); OSB200_ERR_UNSUPPORTED unless option "variant" is 2.  n <= 1
 * is a no-op, except that argsort16 with n == 1 writes both outputs.  Options and info keys apply as to the 32-bit sorts
 * (profile intervals: [hist, scan, pass0, pass1]); a sort of at most 16,384 keys is one launch of the single-block sort.
 * Asynchronous, no host synchronisation, graph-capturable. */
typedef enum osb200_key16_type {
    OSB200_KEY16_U16 = 0, OSB200_KEY16_I16 = 1, OSB200_KEY16_F16 = 2, OSB200_KEY16_BF16 = 3
} osb200_key16_type;
OSB200_API int osb200_sort_keys16(osb200_handle h, void* d_keys, uint64_t n, int key_type, int descending, void* stream);
OSB200_API int osb200_sort_pairs16(osb200_handle h, void* d_keys, uint32_t* d_values, uint64_t n, int key_type,
                                   int descending, void* stream);
OSB200_API int osb200_argsort16(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                                int key_type, int descending, void* stream);

/* Row sort: every row of a batch sorted along its last dimension, the shape of torch.sort(x, dim=-1, stable=True).
 * Row r of d_keys_in is elements [r*row_len, (r+1)*row_len); it is sorted stable into the same row of d_keys_out, ascending
 * or descending (the complement of the encoded key, as in osb200_sort_keys_typed: equal keys keep their input order in both
 * directions).  d_indices may be NULL (keys only); otherwise d_indices[r*row_len + j] is the position within row r of
 * output key j (uint32).
 *   key_bytes 2: key_type is an osb200_key16_type;  4 or 8: an osb200_key_type of that width.  Floats follow the total order
 *                of their bit patterns, as everywhere else in this library.
 * Any handle will do, whatever its key or value width: the call uses only the handle's device, rank mode and SM count, and
 * allocates nothing.  d_keys_out == d_keys_in sorts in place; any other overlap among the three arrays is
 * OSB200_ERR_INVALID_ARG.  Only natural alignment is required (the kernels load element by element).
 * Returns OSB200_ERR_INVALID_ARG for a null handle or key pointer, a misaligned pointer, a key_bytes / key_type that do not
 * match, or array sizes that overflow 64 bits; OSB200_ERR_SIZE for row_len above 16,384 (2- and 4-byte keys) or 8,192 (8-byte
 * keys).  num_rows == 0 or row_len == 0 is a no-op; row_len == 1 copies the keys and writes zero indices.
 * Rows of at most 256 keys are sorted one per warp, longer rows one per thread block in shared memory (option
 * "debug_rows_block" = 1 sends the short rows to the block path too; a test hook).  One launch: asynchronous, no host
 * synchronisation, graph-capturable (there is nothing to clear under capture). */
OSB200_API int osb200_sort_rows(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t num_rows,
                                uint32_t row_len, int key_bytes, int key_type, int descending, void* stream);

/* Long-row sort: osb200_sort_rows for every row_len from 1 to 2^32 - 1, with the same semantics -- key_bytes / key_type and
 * codec, stable in both directions, d_indices NULL or uint32 positions within the row, d_keys_out == d_keys_in in place (any
 * other overlap OSB200_ERR_INVALID_ARG), natural alignment only, num_rows == 0 or row_len == 0 a no-op and row_len == 1 a copy
 * with zero indices.  The argument errors of osb200_sort_rows come first.
 * Rows of at most 16,384 keys (8,192 for 8-byte keys) are sorted by osb200_sort_rows' own launch, on any handle and with no
 * workspace.  Longer rows take the long path, which uses the handle's workspace and allocates nothing.  It needs:
 *   - num_rows * row_len <= max_n, else OSB200_ERR_SIZE;
 *   - a handle key width of at least key_bytes -- a (4, 0) or (4, 4) handle for 2- and 4-byte keys, a (8, 0) or (8, 4) handle
 *     for any width -- else OSB200_ERR_INVALID_ARG;
 *   - value_bytes == 4 when d_indices is given (a (4, 4) handle, or osb200_create_pairs64's (8, 4)), else
 *     OSB200_ERR_INVALID_ARG;
 *   - room in the handle's reductions for 1 KiB per tile of 8,192 keys (a ragged last tile per row included) and the chunk
 *     sums: a handle of max_n >= num_rows * row_len always has it for rows above the limit; else OSB200_ERR_SIZE.
 * The long path writes the handle's alternate key buffer (key_bytes * n bytes), its alternate payloads (4n, with indices),
 * its control block (histogram and plan: info "last_executed_passes" / "last_skip_mask" read this call's plan) and its
 * compact reductions.  It never writes the chained-scan descriptors.
 * It is an LSD radix sort per row over tiles that never straddle rows: a GlobalHistogram over all keys decides, as for
 * osb200_sort_keys_typed, which digit places every key shares (skipped; option "short_circuit"); per executed place a count
 * of each tile's digits, a scan of each row's tile counts and a stable scatter, and a copy home when an odd number of places
 * ran.  No tile waits on another.  One memset and a fixed sequence of launches: asynchronous, no host synchronisation,
 * graph-capturable; one call in flight per handle.  Option "debug_long_rows" = 1 (a test hook) sends rows of 2 .. 16,384
 * (8,192) keys to the long path too, with its workspace rules. */
OSB200_API int osb200_sort_long_rows(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices,
                                     uint64_t num_rows, uint32_t row_len, int key_bytes, int key_type, int descending, void* stream);

/* Segment sort: osb200_sort_rows for ragged rows given by offsets.  Segment s is [off[s], off[s+1]) of arrays of n elements
 * (off = d_segment_offsets, num_segments + 1 of them, 8-byte aligned); it is sorted stable into the same positions of
 * d_keys_out, ascending or descending (the complement of the encoded key: equal keys keep their order).  d_indices may be
 * NULL; otherwise it receives every output key's position within its segment (uint32).  key_bytes / key_type, the in-place
 * rule (d_keys_out == d_keys_in; any other overlap, and offsets overlapping an output, are OSB200_ERR_INVALID_ARG) and the
 * alignment are those of osb200_sort_rows.
 *   max_segment_len: the caller's bound on the segment lengths; it decides which kernels are launched.  Above 16,384 (8,192
 *                    for 8-byte keys): OSB200_ERR_SIZE.  Segments longer than the bound are not written; 0 is a no-op.
 * Only positions inside segments are written.  A segment whose offsets decrease (off[s+1] < off[s]) or pass n (off[s+1] > n)
 * is not written, and nothing outside [0, n) is touched: the offsets need not be trusted.  Positions outside every segment,
 * such as those before off[0], keep what they held.
 * A binning kernel reads the offsets once and writes one-key segments itself; segments of 2-256 keys are sorted one per
 * warp, 257-2,048 keys one per 256-thread block and longer ones one per 512-thread block, each class by one kernel that
 * returns at once when it has no segment.  At most four launches and one memset: asynchronous, no host synchronisation,
 * graph-capturable.  Workspace: one uint32 per segment of the handle's alternate key buffer, so num_segments above
 * min(max_n, 2^32) is OSB200_ERR_SIZE (any key or value width of handle will do); one call in flight per handle.
 * n == 0 or num_segments == 0 is a no-op. */
OSB200_API int osb200_sort_segments(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                                    const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t max_segment_len,
                                    int key_bytes, int key_type, int descending, void* stream);

/* Segments of any length: osb200_sort_segments with max_segment_len any uint32, the same arguments and the same semantics for
 * every segment -- stable in both directions, uint32 positions within the segment, in place when d_keys_out == d_keys_in,
 * natural alignment only.  Nothing outside segments is written; segments whose offsets decrease or pass n, and segments
 * longer than max_segment_len, are not written.  Segments that overlap (offsets that go back) have no defined result, as in
 * osb200_sort_segments; if overlapping long segments hold more tiles than the workspace bound below, the call leaves every
 * long segment untouched and still returns OSB200_OK.  The argument errors of osb200_sort_segments come first, in the same
 * order.
 * max_segment_len <= 16,384 (8,192 for 8-byte keys): osb200_sort_segments' own launch, on any handle, with its workspace rule.
 * Above that, segments longer than the limit take the long path, which uses the handle's workspace and allocates nothing.
 * It needs:
 *   - n <= max_n and num_segments <= min(max_n, 2^32), else OSB200_ERR_SIZE;
 *   - a handle key width of at least key_bytes, else OSB200_ERR_INVALID_ARG;
 *   - value_bytes == 4 when d_indices is given, else OSB200_ERR_INVALID_ARG;
 *   - room in the handle's reductions for the tile counts of the worst case, segments of limit + 1 keys: 1 KiB per tile of
 *     8,192 keys, ceil(n / 8,192) + floor(n / (limit + 1)) tiles, and the tile map.  The bound depends on n and key_bytes
 *     only, never on the offsets, and a handle of the right shape with max_n >= max(n, num_segments) always has the room;
 *     else OSB200_ERR_SIZE.
 * The binning kernel of osb200_sort_segments lists the long segments apart; the shorter ones are sorted by its class kernels.
 * A one-CTA kernel maps the long list to tiles of 8,192 keys that never straddle segments, and the long rows' passes
 * (osb200_sort_long_rows) sort them, each tile finding its segment by a search over the map: a GlobalHistogram over all n
 * keys decides which digit places are skipped (info "last_executed_passes" reads this call's plan), then per executed place a
 * count, a scan of each segment's tile counts and a stable scatter, and a copy home within the long segments only.  The long
 * path writes the handle's alternate key buffer and payloads, control block and compact reductions.  Asynchronous, no host
 * synchronisation, graph-capturable; one call in flight per handle.  Option "debug_long_rows" = 1 (a test hook) sends
 * segments of 2 .. 16,384 (8,192) keys to the long path too, with its workspace rules (bounded then by n / 2 segments). */
OSB200_API int osb200_sort_long_segments(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                                         const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t max_segment_len,
                                         int key_bytes, int key_type, int descending, void* stream);

/* Row top-k: the k smallest (largest = 0) or largest (largest = 1) keys of every row and their positions, the shape of
 * torch.topk(x, k, dim=-1, largest, sorted).  Row r of d_keys_in is elements [r*row_len, (r+1)*row_len); its result is
 * [r*k, (r+1)*k) of d_values_out and d_indices (uint32 positions within the row, required).
 *   key_bytes / key_type: those of osb200_sort_rows.  largest = 1 selects through the descending codec, as descending does there.
 *   The selected set is exactly the first k keys of the row's stable sort (ascending, or descending for largest = 1): of equal
 *   keys at the boundary the lowest positions are taken.  sorted = 1 writes them in that order, bit-identical to the first k
 *   columns of osb200_sort_rows with descending = largest; sorted = 0 writes the same k (key, position) pairs in an
 *   unspecified order.
 * row_len may be any uint32; k may be at most 16,384 (2- and 4-byte keys) or 8,192 (8-byte keys): OSB200_ERR_SIZE above.
 * k > row_len is OSB200_ERR_INVALID_ARG; num_rows == 0, row_len == 0 or k == 0 is a no-op.  Natural alignment of the keys and
 * 4-byte alignment of the indices are required; array sizes that overflow 64 bits, a null pointer and any overlap between the
 * input and either output or between the two outputs are OSB200_ERR_INVALID_ARG (there is no in-place form).
 * Any handle will do: the call uses only the handle's device, rank mode, SM count and the test hooks "debug_rows_block" and
 * "debug_topk_capacity", and allocates nothing.  Rows of at most 256 keys are sorted one per warp and cut to k; longer rows
 * are radix-selected one per thread block, from the most significant digit, with the candidates in shared memory once at
 * most 16,384 (8,192) of them are left.  sorted = 1 then sorts the [num_rows, k] result in place.  At most two launches:
 * asynchronous, no host synchronisation, graph-capturable. */
OSB200_API int osb200_topk_rows(osb200_handle h, const void* d_keys_in, void* d_values_out, uint32_t* d_indices,
                                uint64_t num_rows, uint32_t row_len, uint32_t k, int key_bytes, int key_type,
                                int largest, int sorted, void* stream);

/* Segment top-k: osb200_topk_rows for ragged segments given by offsets.  Segment s is [off[s], off[s+1]) of n keys (off =
 * d_segment_offsets, num_segments + 1 of them, 8-byte aligned, as for osb200_sort_segments).  With L its length and
 * m = min(L, k), its result is row s of a [num_segments, k] output, elements [s*k, s*k + k) of d_values_out and d_indices:
 *   columns 0 .. m-1: the first m keys of the segment's stable sort (ascending, or descending for largest = 1; the codec of
 *   osb200_topk_rows) and their uint32 positions within the segment.  Of equal keys at the boundary the lowest positions are
 *   taken.  sorted = 1 writes them in sort order, bit-identical to the first m keys and indices osb200_sort_segments writes
 *   for the segment (descending = largest) wherever that call accepts it; sorted = 0 writes the same m pairs in an
 *   unspecified order.
 *   columns m .. k-1: padding, position 0xFFFFFFFF (-1 as int32) and the key that sorts last in the selection order, the
 *   decode of the all-ones radix image: UINT_MAX, INT_MAX or the NaN 0x7F..F for largest = 0; 0, INT_MIN or the NaN 0xF..F
 *   for largest = 1.
 * A segment whose offsets decrease, whose end passes n, or that is longer than 2^32 - 1 keys is empty: its row is all padding.
 * Nothing outside [0, n) is read and nothing outside [0, num_segments*k) of either output is written: the offsets need not
 * be trusted.
 * k may be at most 16,384 (2- and 4-byte keys) or 8,192 (8-byte keys): OSB200_ERR_SIZE above; k larger than a segment is
 * fine.  k == 0 or num_segments == 0 is a no-op; n == 0 is not (every row is padding), and d_keys_in may be NULL only then.
 * key_bytes / key_type are those of osb200_sort_rows.  d_indices is required.  Natural alignment of the keys, 4-byte alignment
 * of the indices, a null handle, output or offsets pointer, array sizes that overflow 64 bits and any overlap between the
 * input, the offsets and the two outputs are OSB200_ERR_INVALID_ARG (there is no in-place form).
 * Workspace: one uint32 per segment of the handle's alternate key buffer and the class counts in its control block, so
 * num_segments above min(max_n, 2^32) is OSB200_ERR_SIZE (any key or value width of handle will do); one call in flight per
 * handle.  A binning kernel reads the offsets once; segments of at most 256 keys, and the empty and invalid ones, are sorted
 * and padded one per warp, longer ones radix-selected one per thread block as in osb200_topk_rows, a segment of at most k
 * keys in one pass.  sorted = 1 then sorts the block-selected rows in place.  The test hooks "debug_rows_block" (every
 * non-empty segment to the radix select) and "debug_topk_capacity" apply.  At most one memset and four launches:
 * asynchronous, no host synchronisation, graph-capturable. */
OSB200_API int osb200_topk_segments(osb200_handle h, const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t n,
                                    const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t k, int key_bytes,
                                    int key_type, int largest, int sorted, void* stream);

/* Sort on a bit range [begin_bit, end_bit) of the (unsigned) key only, CUB-style: keys that agree on those bits keep their
 * input order (stable).  ceil((end_bit-begin_bit)/8) digit passes instead of key_bytes; the last digit may be narrower
 * than 8 bits; an odd pass count is handled inside (the result is always returned in the caller's buffers).  d_values may
 * be NULL (keys only).  begin_bit == end_bit is a no-op.  Reference: none in CUDA (its passes are fixed at radixShift
 * 0/8/16/24, Sort/OneSweepDispatcher.cuh:325-335); SURVEY 8f rank 2. */
OSB200_API int osb200_sort_bits(osb200_handle h, void* d_keys, uint32_t* d_values, uint64_t n, int begin_bit, int end_bit,
                                void* stream);

/* Segmented sort: every segment [offsets[i], offsets[i+1]) of d_keys (and d_values, may be NULL) is sorted ascending and
 * stable, in place, by ONE thread block in shared memory (all four digit passes in one launch; no histogram, descriptor or
 * lookback traffic).  d_segment_offsets: num_segments + 1 non-decreasing element offsets in device memory.
 * max_segment_len: an upper bound of the segment lengths known to the caller; it picks the block geometry (<= 256 or 2,048 keys:
 * 256 threads, up to 8 blocks per SM; <= 16,384: 512 threads) -- segments longer than 16,384 keys return OSB200_ERR_SIZE
 * (sort those with osb200_sort_*), segments longer than max_segment_len are left untouched.  Empty segments are fine.
 * Reference: SplitSort, the reference's segmented sort (GPUSortingCUDA/SegSort/SplitSort/SplitSort.cuh:702-938 bins
 * segments by length and dispatches one kernel per bin); SURVEY 8f rank 4.  The same kernel is the small-n path of every
 * osb200_sort_* call: n <= 16,384 (8,192 for 64-bit keys) is one segment, one launch (option "small_path", default 1). */
OSB200_API int osb200_segmented_sort_u32(osb200_handle h, uint32_t* d_keys, uint32_t* d_values, const uint64_t* d_segment_offsets,
                                         uint64_t num_segments, uint32_t max_segment_len, void* stream);

/* Host-buffer entry points: copy in, sort, copy back, synchronise.  `h_*` may be pageable or pinned
 * host memory.  This is the end-to-end call a host-side caller of the reference would make (the
 * reference itself has no host-data API; its buffers are generated on the device,
 * OneSweepDispatcher.cuh:215-219). */
OSB200_API int osb200_sort_host_keys_u32(osb200_handle h, uint32_t* h_keys, uint64_t n);
OSB200_API int osb200_sort_host_pairs_u32(osb200_handle h, uint32_t* h_keys, uint32_t* h_values, uint64_t n);
OSB200_API int osb200_sort_host_keys_u64(osb200_handle h, uint64_t* h_keys, uint64_t n);

/* ------------------------------------------------------------------------------------------------
 * Kernel-level entry points (for parity tests against the reference's individual kernels).
 *   osb200_global_histogram   replaces OneSweep::GlobalHistogram<<<...>>> (Sort/OneSweep.cu:44-123):
 *                             d_hist[place*256 + digit], uint64 counts, key_bytes places, overwritten.
 *   osb200_digit_binning_pass replaces OneSweep::Scan + one OneSweep::DigitBinningPassKeysOnly/Pairs
 *                             launch (Sort/OneSweep.cu:125-162,164-344,346-600): a stable counting
 *                             sort of d_in (and d_in_values, may be NULL) on the 8-bit digit at
 *                             `radix_shift` into d_out (d_out_values).  Out-of-place.  radix_shift is 0/8/16/24
 *                             in the reference; any shift below the key width is accepted (a shift within 8
 *                             bits of the top yields fewer than 256 bins -- the sharded exchange uses that).
 *   osb200_validate           replaces Validate<<<...>>> (UtilityKernels.cuh:403-429,432-479):
 *                             *h_err_count = number of adjacent inversions in d_keys (synchronises).
 * ---------------------------------------------------------------------------------------------- */
OSB200_API int osb200_global_histogram(osb200_handle h, const void* d_keys, uint64_t n, uint64_t* d_hist, void* stream);
OSB200_API int osb200_digit_binning_pass(osb200_handle h, const void* d_in, void* d_out, const uint32_t* d_in_values,
                              uint32_t* d_out_values, uint64_t n, uint32_t radix_shift, void* stream);
OSB200_API int osb200_validate(osb200_handle h, const void* d_keys, uint64_t n, uint64_t* h_err_count, void* stream);

/* Test-input generator.  Replaces InitRandom<<<256,256>>> (UtilityKernels.cuh:53-83 keys, :85-117 pairs):
 * the reference's deterministic hybrid Tausworthe/LCG generator with Thearling-Smith entropy reduction
 * (and_count = ENTROPY_PRESET value 0..4).  d_payload may be NULL; if not, it receives a copy of the key
 * (reference behaviour, UtilityKernels.cuh:115) or the element index when payload_is_index != 0 (stricter
 * stability test, SURVEY 8c).  The whole 64-bit n is honoured (the reference takes uint32 size). */
OSB200_API int osb200_init_random_u32(uint32_t* d_keys, uint32_t* d_payload, uint64_t n, uint32_t and_count, uint32_t seed,
                           int payload_is_index, void* stream);

/* Tuning / introspection (no reference equivalent; the reference's constants are #defines,
 * Sort/OneSweep.cu:17-42).  Returns OSB200_ERR_INVALID_ARG for unknown keys/values.  Options:
 *   "rank_mode"      0 = atomic-ranked (default), 1 = ballot-ranked.  The default ranks keys with ONE shared-memory
 *                    atomicAdd per key and relies on the GPU handing the return values of one warp-wide ATOMS.ADD to
 *                    same-address lanes in ascending lane order -- an UNDOCUMENTED hardware property on which the
 *                    stability of every pass rests.  osb200_create verifies it on the device (a self-test kernel in the
 *                    production geometry) and falls back to 1 if it ever fails; 1 is the supported escape hatch: it uses
 *                    the reference's documented 8-ballot warp multisplit (Sort/OneSweep.cu:208-253) at a longer pass time.
 *                    The assumption failed once, in ONE development build of the pairs kernel (rank phase of some
 *                    warps concurrent with the chained-scan loads of others, n >= 2^28; DESIGN.md 4.1); the shipped
 *                    kernels never overlap the two and the GPU suite
 *                    compares full-size sorts element by element.
 *   "variant"        kernel variant id (2 = default wide-tile kernel; 0/1 development baselines)
 *   "short_circuit"  1 (default) = digit passes on which ALL keys agree are skipped, decided on the device from the
 *                    global histogram without any host synchronisation; 0 = always run every pass like the reference
 *   "spin_cap"       lookback polls of one predecessor tile before a digit thread stops waiting and re-reduces that
 *                    tile itself (forward-progress fallback, reference: Sort/EmulatedDeadlocking.cu:159-267)
 *   "debug_stall_every"  test hook for that fallback: N > 0 makes every N-th tile withhold its reduction
 *   "debug_max_ctas" test hook of the persistent DigitBinningPass (uint32 keys, HOT passes): N > 0 runs it on at most N CTAs (the tiles after
 *                    each CTA's first are handed out by an atomic ticket); 0 (default) = as many as can be resident
 *   "debug_rows_block"  test hook of osb200_sort_rows: 1 = rows of at most 256 keys go through the block path (2,048-key
 *                    geometry) instead of one warp per row, to compare the two paths; 0 (default) = the warp path.
 *                    osb200_topk_rows honours it too: its rows of at most 256 keys are then radix-selected one per block
 *   "debug_long_rows"  test hook of osb200_sort_long_rows: 1 = rows of 2 .. 16,384 keys (8,192 for 8-byte keys) take the long
 *                    path too, with its workspace rules (short rows have a tile each, so many of them may need more room
 *                    than max_n gives: OSB200_ERR_SIZE), to compare it with osb200_sort_rows; 0 (default) = osb200_sort_rows' launch.
 *                    osb200_sort_long_segments honours it too: its segments of 2 .. 16,384 (8,192) keys then take the long path
 *   "debug_topk_capacity"  test hook of osb200_topk_rows: N > 0 keeps at most N candidates of a row in shared memory (instead
 *                    of 16,384, or 8,192 for 8-byte keys), so that short rows exercise the passes that read global memory
 *                    and the switch to shared memory; 0 (default) = the full capacity
 *   "debug_epoch"    test hook of the descriptor epochs: sets the handle's epoch counter (0 .. 2^24 - 1; info "epoch"), so
 *                    that the next passes cross the wrap-around (which clears every descriptor) or reuse the epochs of a
 *                    captured sort
 *   "profile"        1 = record CUDA events between the kernels of a sort (osb200_get_profile)
 *   "small_path"     1 (default) = a sort of at most one tile (info "small_path_max_n": 16,384 keys, 8,192 for 64-bit keys)
 *                    is ONE launch of the single-block shared-memory sort (see osb200_segmented_sort_u32); 0 = always the
 *                    multi-kernel path
 *   "hot_passes"     1 (default) = a digit place in which one bin holds >= n/8 keys (low-entropy inputs; reference presets
 *                    UtilityKernels.cuh:42-52) is executed by the HOT instantiation of the DigitBinningPass, which ranks
 *                    a tile's most frequent digit with one ballot per round instead of serialised same-address atomics;
 *                    decided on the device, both instantiations are enqueued for every pass; 0 = plain kernel only
 *   "fused_histogram" 1 (default) = whole-key u32 keys-only sorts of at least 64 tiles and below 2^32 keys run no
 *                    GlobalHistogram in front: the first digit pass counts it and scatters into fixed regions, and the
 *                    classic histogram, scan and first pass run only when a region overflows; 0 = the classic path
 * Info keys: "tile_keys","launches_per_sort","memsets_per_sort","sm_count","rank_mode","variant","atomic_order_ok",
 * "max_n","epoch","short_circuit","spin_cap","small_path","small_path_max_n","hot_passes","fused_histogram","last_skip_mask",
 * "last_hot_mask","last_executed_passes","last_fused_kept" (the last four read the device plan of the previous sort and
 * synchronise; "last_fused_kept" = 1 when its fused first pass stood). */
OSB200_API int osb200_set_option(osb200_handle h, const char* key, int64_t value);
OSB200_API int64_t osb200_get_info(osb200_handle h, const char* key);
/* With option "profile"=1 every sort records CUDA events on its stream between its kernels.  Returns the number of
 * intervals written (waits for the last sort): out_ms[0]=GlobalHistogram, [1]=Scan, [2+p]=DigitBinningPass p.
 * (The reference times only the whole dispatch, OneSweepDispatcher.cuh:221-224.) */
OSB200_API int osb200_get_profile(osb200_handle h, float* out_ms, int capacity); /* "tile_keys","launches_per_sort","sm_count",... ; <0 if unknown */

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU sharded sort (one process per GPU).  No reference equivalent (the reference is single
 * device, SURVEY 2.1); this is BASELINE.json's "MSD bucket-exchange then local OneSweep".
 *
 *   osb200_sharded_unique_id  rank 0 fills a 128-byte NCCL unique id; the host application broadcasts
 *                             it to all ranks (torch.distributed / MPI / files).
 *   osb200_sharded_create     every rank: joins the communicator (world ranks on ONE node), allocates
 *                             receive + local-sort workspace for up to max_n_local keys per rank plus
 *                             `slack_percent` head-room for bucket imbalance.  max_n_local and slack_percent MUST
 *                             be the same on every rank: if any rank's share exceeds that capacity, every rank
 *                             returns OSB200_ERR_SIZE from the sort call together (no rank is left in a collective).
 *   osb200_sharded_sort_keys_u32
 *                             every rank passes its n_local unsorted keys.  After the call rank r owns
 *                             the r-th contiguous slice of the global ascending order: *d_out points
 *                             into handle-owned memory valid until the next call, *n_out is its length.
 *                             Steps: local top-digit histogram -> all-gather of the 256-bin histograms
 *                             -> bucket->rank assignment -> exchange pass (keys move over NVLink) ->
 *                             local OneSweep.
 * ---------------------------------------------------------------------------------------------- */
OSB200_API int osb200_sharded_unique_id(void* out_128_bytes);
OSB200_API int osb200_sharded_create(osb200_sharded_handle* out, const void* unique_id_128_bytes, int rank, int world,
                          uint64_t max_n_local, int slack_percent);
OSB200_API int osb200_sharded_destroy(osb200_sharded_handle h);
OSB200_API int osb200_sharded_sort_keys_u32(osb200_sharded_handle h, const uint32_t* d_keys_local, uint64_t n_local,
                                 uint32_t** d_out, uint64_t* n_out, void* stream);
/* The host-side exchange plan, a pure function of the all-gathered histograms (exported so the N>1 logic can be
 * tested on CPU): dest[256] = owner rank of every most-significant-digit bucket (contiguous, non-decreasing,
 * balanced on the global counts); recv_count[world] = keys every rank ends up with; recv_off[256] = for source
 * `rank`, the element offset inside dest[d]'s receive buffer where its bucket-d keys go (bucket-major,
 * source-rank-minor: the globally stable order of the MSD partition). */
OSB200_API int osb200_sharded_plan(const uint64_t* hist_all /*[world][256]*/, int world, int rank, int32_t* dest,
                                   uint64_t* recv_count, uint64_t* recv_off);
/* Keys every rank's receive buffer holds: max_n_local + max_n_local / 100 * slack_percent + 4096 (integer division), the
 * capacity osb200_sharded_create allocates.  0 for a slack_percent outside 0..400. */
OSB200_API uint64_t osb200_sharded_capacity(uint64_t max_n_local, int slack_percent);
/* The whole host-side layout of one exchange, a pure function of the all-gathered histograms that
 * osb200_sharded_sort_keys_u32 calls on every rank (exported so the layout and, with the two debug hooks below, the
 * exchange pass itself can be tested without NCCL or a second GPU).  Inputs: hist_all[world][256] (the counts of every
 * rank's top bytes), this `rank`, the receive `capacity` in keys, force_fine (see osb200_sharded_force_fine), and
 * recv_addrs[world], the byte addresses of the receive buffers (4-byte aligned; NULL when no fused bases are wanted).
 * Outputs:
 *   *xshift, *bins   the exchange pass's digit: 32 - log2(world) and world bins when world is a power of two > 1, force_fine
 *                    is 0 and every rank's share of the equal-width split fits `capacity` (coarse); else 24 and 256 (fine)
 *   dest[256]        destination rank of every bin (coarse: bin b < world goes to rank b; fine: osb200_sharded_plan's)
 *   recv_count[world] keys every rank receives
 *   recv_off[256]    for this rank as a source, the element offset of its keys of bin b in dest[b]'s receive buffer:
 *                    bucket-major, source-rank-minor, the stable order of the MSD partition
 *   pass_hist[256]   the histogram the exchange pass scans: this rank's counts of its digit (coarse: bins 0..world-1)
 *   out_base[256]    only if recv_addrs: the fused pass's base of every bin as a virtual element index,
 *                    recv_addrs[dest[b]] / 4 + recv_off[b] (recv_addrs and out_base go together)
 *   send_off[world+1]      staged: destination p's keys are [send_off[p], send_off[p+1]) of the pass's bin-major output
 *   recv_from_off[world+1] staged: this rank receives source s's keys at [recv_from_off[s], recv_from_off[s+1])
 * Returns OSB200_ERR_SIZE when neither split fits `capacity` -- the same on every rank, so all ranks stop together; then
 * only xshift, bins, dest and recv_count are meaningful (the fine plan that does not fit). */
OSB200_API int osb200_sharded_exchange_layout(const uint64_t* hist_all, int world, int rank, uint64_t capacity, int force_fine,
                                              const uint64_t* recv_addrs, uint32_t* xshift, int32_t* bins, int32_t* dest,
                                              uint64_t* recv_count, uint64_t* recv_off, uint64_t* pass_hist,
                                              uint64_t* out_base, uint64_t* send_off, uint64_t* recv_from_off);
/* 1 (default when CUDA IPC peer mapping works) = the exchange is the DigitBinningPass kernel scattering straight into
 * the peers' receive buffers over NVLink; 0 = staged: local pass + ncclSend/ncclRecv.  Same value on every rank. */
OSB200_API int osb200_sharded_set_fused(osb200_sharded_handle h, int fused);
/* Exchange granularity: by default, when world is a power of two and the equal-width split of the key space fits the
 * receive buffers, the exchange bins on the top log2(world) bits only (long runs, full NVLink sectors); otherwise on
 * the top 8 bits with the greedy plan.  on=1 forces the 256-bucket plan (tests / skewed data).  Same on every rank. */
OSB200_API int osb200_sharded_force_fine(osb200_sharded_handle h, int on);
/* Testing hooks on an ordinary single-GPU handle (key_bytes 4), for running every rank's exchange pass in one process:
 *   osb200_debug_digit_histogram  d_hist256[256] = counts of the digit (d_in[i] >> shift) & 0xFF over d_in[0..n), the
 *                                 sharded sort's first step (shift 24)
 *   osb200_debug_exchange_pass    the sharded sort's exchange pass over d_in[0..n), binning on the digit at `shift` (8 bits,
 *                                 or 32 - shift bits above 24), stable.  With d_out_base (device [256]: the out_base of
 *                                 osb200_sharded_exchange_layout) the keys of bin b go to the 4-byte words at virtual
 *                                 element indices d_out_base[b], d_out_base[b] + 1, ... -- plain device addresses divided by
 *                                 4 -- and d_out must be NULL (fused mode); without it the pass scans d_hist256, which must
 *                                 hold the counts of that digit, into d_out (staged mode: the stable bin-major partition).
 * d_in must be 16-byte aligned, n <= max_n, shift < 32.  Asynchronous on `stream`; not supported under graph capture. */
OSB200_API int osb200_debug_digit_histogram(osb200_handle h, const uint32_t* d_in, uint64_t n, uint32_t shift,
                                            uint64_t* d_hist256, void* stream);
OSB200_API int osb200_debug_exchange_pass(osb200_handle h, const uint32_t* d_in, uint32_t* d_out, uint64_t n, uint32_t shift,
                                          const uint64_t* d_hist256, const uint64_t* d_out_base, void* stream);
/* The two single-GPU sorters inside a sharded sorter (exchange pass / local sort), e.g. to set options. */
OSB200_API int osb200_sharded_local_handle(osb200_sharded_handle h, osb200_handle* exch, osb200_handle* local);
/* Milliseconds of the phases of the last sharded sort on this rank: [0]=histogram+allgather,
 * [1]=exchange, [2]=local sort, [3]=total (device time, CUDA events). */
OSB200_API int osb200_sharded_last_timing(osb200_sharded_handle h, float* out_ms4);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* ONESWEEP_B200_H_ */
