// OneSweepB200.hpp -- header-only C++ mirror of the reference's interface on top of the C-ABI.
//
//   namespace OneSweep { Sort(keys[, values], n[, stream]) }   the north-star call shape: the only public `Sort` of the
//       reference is GPUSortingUnity/Runtime/OneSweep.cs:297-306,358-370; in CUDA, OneSweep is a namespace of kernels
//       (GPUSortingCUDA/Sort/OneSweep.cuh:22-53) driven by private dispatcher methods (SURVEY D1).
//   class OneSweepSorterB200                                    RAII owner of one osb200 handle
//       (reference: OneSweepDispatcher ctor/dtor, Sort/OneSweepDispatcher.cuh:42-83).
// Errors: std::runtime_error carrying osb200_status_string() -- the reference ignores CUDA errors entirely.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>

#include "onesweep_b200.h"

class OneSweepSorterB200 {
  public:
    // (8, 4) -- 64-bit keys with uint32 payloads -- is made by osb200_create_pairs64
    OneSweepSorterB200(uint64_t max_n, int key_bytes, int value_bytes) : max_n_(max_n)
    {
        if (key_bytes == 8 && value_bytes == 4) check(osb200_create_pairs64(&h_, max_n), "osb200_create_pairs64");
        else check(osb200_create(&h_, max_n, key_bytes, value_bytes), "osb200_create");
    }
    ~OneSweepSorterB200() { if (h_) osb200_destroy(h_); }
    OneSweepSorterB200(const OneSweepSorterB200&) = delete;
    OneSweepSorterB200& operator=(const OneSweepSorterB200&) = delete;

    void SortKeys(uint32_t* d_keys, uint64_t n, void* stream = nullptr) { check(osb200_sort_keys_u32(h_, d_keys, n, stream), "osb200_sort_keys_u32"); }
    void SortKeys(uint64_t* d_keys, uint64_t n, void* stream = nullptr) { check(osb200_sort_keys_u64(h_, d_keys, n, stream), "osb200_sort_keys_u64"); }
    void SortPairs(uint32_t* d_keys, uint32_t* d_values, uint64_t n, void* stream = nullptr)
    {
        check(osb200_sort_pairs_u32(h_, d_keys, d_values, n, stream), "osb200_sort_pairs_u32");
    }
    // uint64 keys with uint32 payloads, on a (8, 4) sorter
    void SortPairs(uint64_t* d_keys, uint32_t* d_values, uint64_t n, void* stream = nullptr)
    {
        check(osb200_sort_pairs_typed(h_, d_keys, d_values, n, OSB200_KEY_U64, 0, stream), "osb200_sort_pairs_typed");
    }
    // stable sort on the key bits [begin_bit, end_bit) only; d_values may be null
    void SortBits(void* d_keys, uint32_t* d_values, uint64_t n, int begin_bit, int end_bit, void* stream = nullptr)
    {
        check(osb200_sort_bits(h_, d_keys, d_values, n, begin_bit, end_bit, stream), "osb200_sort_bits");
    }
    // signed / float keys and descending order (osb200_key_type)
    void SortKeysTyped(void* d_keys, uint64_t n, int key_type, bool descending, void* stream = nullptr)
    {
        check(osb200_sort_keys_typed(h_, d_keys, n, key_type, descending ? 1 : 0, stream), "osb200_sort_keys_typed");
    }
    // stable sort of d_keys_in (left untouched) into d_keys_out, with d_indices[i] = input position of d_keys_out[i]; 32-bit
    // key types on a (4, 4) sorter, 64-bit key types on a (8, 4) sorter; n <= 2^32
    void ArgSort(const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n, int key_type, bool descending,
                 void* stream = nullptr)
    {
        check(osb200_argsort(h_, d_keys_in, d_keys_out, d_indices, n, key_type, descending ? 1 : 0, stream), "osb200_argsort");
    }
    // 16-bit keys (osb200_key16_type: uint16, int16, float16, bfloat16) in two digit passes, on a 4-byte sorter; pairs and
    // argsort need a (4, 4) sorter
    void SortKeys16(void* d_keys, uint64_t n, int key_type, bool descending, void* stream = nullptr)
    {
        check(osb200_sort_keys16(h_, d_keys, n, key_type, descending ? 1 : 0, stream), "osb200_sort_keys16");
    }
    void SortPairs16(void* d_keys, uint32_t* d_values, uint64_t n, int key_type, bool descending, void* stream = nullptr)
    {
        check(osb200_sort_pairs16(h_, d_keys, d_values, n, key_type, descending ? 1 : 0, stream), "osb200_sort_pairs16");
    }
    void ArgSort16(const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n, int key_type, bool descending,
                   void* stream = nullptr)
    {
        check(osb200_argsort16(h_, d_keys_in, d_keys_out, d_indices, n, key_type, descending ? 1 : 0, stream), "osb200_argsort16");
    }
    // every row [r*row_len, (r+1)*row_len) of d_keys_in sorted stable into d_keys_out (== d_keys_in: in place), with
    // d_indices (may be null) = positions within the row; key_bytes 2 (osb200_key16_type) or 4 / 8 (osb200_key_type);
    // row_len <= 16,384 (8,192 for 8-byte keys); any sorter
    void SortRows(const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t num_rows, uint32_t row_len,
                  int key_bytes, int key_type, bool descending, void* stream = nullptr)
    {
        check(osb200_sort_rows(h_, d_keys_in, d_keys_out, d_indices, num_rows, row_len, key_bytes, key_type, descending ? 1 : 0,
                               stream),
              "osb200_sort_rows");
    }
    // SortRows for rows of any length: rows above SortRows' limit use this handle's workspace (num_rows * row_len <= max_n, a
    // key width of at least key_bytes, and value_bytes 4 with indices)
    void SortLongRows(const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t num_rows, uint32_t row_len, int key_bytes,
                      int key_type, bool descending, void* stream = nullptr)
    {
        check(osb200_sort_long_rows(h_, d_keys_in, d_keys_out, d_indices, num_rows, row_len, key_bytes, key_type, descending ? 1 : 0,
                                    stream),
              "osb200_sort_long_rows");
    }
    // the first k keys of every row [r*row_len, (r+1)*row_len) in its stable sort (ascending, or descending for largest) and
    // their positions within the row, into [r*k, (r+1)*k) of d_values_out and d_indices; sorted = false leaves each row's k
    // pairs in an unspecified order; any row_len, k <= 16,384 (8,192 for 8-byte keys); any sorter
    void TopkRows(const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t num_rows, uint32_t row_len, uint32_t k,
                  int key_bytes, int key_type, bool largest, bool sorted, void* stream = nullptr)
    {
        check(osb200_topk_rows(h_, d_keys_in, d_values_out, d_indices, num_rows, row_len, k, key_bytes, key_type, largest ? 1 : 0,
                               sorted ? 1 : 0, stream),
              "osb200_topk_rows");
    }
    // TopkRows for any k <= row_len and rows of any length: k above TopkRows' limit, or fewer rows than SMs of more than 65,536
    // keys, are split across thread blocks on this handle's workspace (num_rows * row_len <= max_n, a key width of at least
    // key_bytes, value_bytes 4)
    void TopkLongRows(const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t num_rows, uint32_t row_len, uint32_t k,
                      int key_bytes, int key_type, bool largest, bool sorted, void* stream = nullptr)
    {
        check(osb200_topk_long_rows(h_, d_keys_in, d_values_out, d_indices, num_rows, row_len, k, key_bytes, key_type,
                                    largest ? 1 : 0, sorted ? 1 : 0, stream),
              "osb200_topk_long_rows");
    }
    // columns h_ranks[0 .. num_ranks) (host array, 1 to 16 strictly increasing ranks below row_len) of every row's ascending
    // stable sort into [r*num_ranks, (r+1)*num_ranks) of d_values_out, and their positions within the row into d_indices (may be
    // null); rows above 16,384 keys (8,192 for 8-byte keys) use this handle's alternate keys for a bound that depends on
    // num_rows, row_len and num_ranks only
    void SelectRows(const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t num_rows, uint32_t row_len,
                    const uint32_t* h_ranks, uint32_t num_ranks, int key_bytes, int key_type, void* stream = nullptr)
    {
        check(osb200_select_rows(h_, d_keys_in, d_values_out, d_indices, num_rows, row_len, h_ranks, num_ranks, key_bytes, key_type,
                                 stream),
              "osb200_select_rows");
    }
    // columns d_ranks[s*num_ranks .. (s+1)*num_ranks) (device array, 1 to 16 non-decreasing ranks per segment) of every segment
    // [offsets[s], offsets[s+1])'s ascending stable sort into row s of [num_segments, num_ranks] outputs, and their positions
    // within the segment into d_indices (may be null); ranks at or past the length, rows whose ranks decrease and invalid
    // segments are padding (position 0xFFFFFFFF); max_segment_len above 16,384 (8,192 for 8-byte keys) uses this handle's
    // alternate payloads for a bound that depends on n, num_segments and num_ranks only
    void SelectSegments(const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t n, const uint64_t* d_segment_offsets,
                        uint64_t num_segments, uint32_t max_segment_len, const uint32_t* d_ranks, uint32_t num_ranks, int key_bytes,
                        int key_type, void* stream = nullptr)
    {
        check(osb200_select_segments(h_, d_keys_in, d_values_out, d_indices, n, d_segment_offsets, num_segments, max_segment_len, d_ranks,
                                     num_ranks, key_bytes, key_type, stream),
              "osb200_select_segments");
    }
    // the first m = min(length, k) keys of every segment [offsets[s], offsets[s+1]) in its stable sort (ascending, or descending
    // for largest) and their positions within the segment, into row s of [num_segments, k] outputs; columns m .. k-1 are
    // padding (position 0xFFFFFFFF, the key that sorts last); segments whose offsets decrease or pass n are all padding;
    // k <= 16,384 (8,192 for 8-byte keys); num_segments <= the handle's max_n
    void TopkSegments(const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t n, const uint64_t* d_segment_offsets,
                      uint64_t num_segments, uint32_t k, int key_bytes, int key_type, bool largest, bool sorted, void* stream = nullptr)
    {
        check(osb200_topk_segments(h_, d_keys_in, d_values_out, d_indices, n, d_segment_offsets, num_segments, k, key_bytes, key_type,
                                   largest ? 1 : 0, sorted ? 1 : 0, stream),
              "osb200_topk_segments");
    }
    // every segment [offsets[s], offsets[s+1]) of n keys sorted stable into the same positions of d_keys_out (ragged rows);
    // d_indices may be null; max_segment_len <= 16,384 (8,192 for 8-byte keys); num_segments <= the handle's max_n
    void SortSegments(const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n, const uint64_t* d_segment_offsets,
                      uint64_t num_segments, uint32_t max_segment_len, int key_bytes, int key_type, bool descending,
                      void* stream = nullptr)
    {
        check(osb200_sort_segments(h_, d_keys_in, d_keys_out, d_indices, n, d_segment_offsets, num_segments, max_segment_len,
                                   key_bytes, key_type, descending ? 1 : 0, stream),
              "osb200_sort_segments");
    }
    // SortSegments for any max_segment_len: segments above SortSegments' limit use this handle's workspace (n <= max_n, a key
    // width of at least key_bytes, and value_bytes 4 with indices)
    void SortLongSegments(const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n, const uint64_t* d_segment_offsets,
                          uint64_t num_segments, uint32_t max_segment_len, int key_bytes, int key_type, bool descending,
                          void* stream = nullptr)
    {
        check(osb200_sort_long_segments(h_, d_keys_in, d_keys_out, d_indices, n, d_segment_offsets, num_segments, max_segment_len,
                                        key_bytes, key_type, descending ? 1 : 0, stream),
              "osb200_sort_long_segments");
    }
    // every segment [offsets[i], offsets[i+1]) sorted ascending and stable in place, one thread block per segment
    // (reference: SplitSort, SegSort/SplitSort/SplitSort.cuh:702-938); d_values may be null; max_segment_len <= 16,384
    void SegmentedSort(uint32_t* d_keys, uint32_t* d_values, const uint64_t* d_segment_offsets, uint64_t num_segments,
                       uint32_t max_segment_len, void* stream = nullptr)
    {
        check(osb200_segmented_sort_u32(h_, d_keys, d_values, d_segment_offsets, num_segments, max_segment_len, stream),
              "osb200_segmented_sort_u32");
    }
    void SetOption(const char* key, int64_t value) { check(osb200_set_option(h_, key, value), "osb200_set_option"); }
    uint64_t Validate(const void* d_keys, uint64_t n, void* stream = nullptr)
    {
        uint64_t e = 0;
        check(osb200_validate(h_, d_keys, n, &e, stream), "osb200_validate");
        return e;
    }
    uint64_t max_n() const { return max_n_; }
    osb200_handle handle() const { return h_; }

    static void check(int status, const char* what)
    {
        if (status != OSB200_OK) throw std::runtime_error(std::string(what) + ": " + osb200_status_string(status));
    }

  private:
    osb200_handle h_ = nullptr;
    uint64_t max_n_;
};

namespace OneSweep {
namespace detail {
// one cached sorter per (key width, pairs); grown on demand.  Not thread-safe across concurrent sorts of the same kind
// (neither is the reference's dispatcher: shared tickets/descriptors).
inline OneSweepSorterB200& sorter(int key_bytes, int value_bytes, uint64_t n)
{
    static std::mutex mu;
    static std::map<std::tuple<int, int>, std::unique_ptr<OneSweepSorterB200>> cache;
    std::lock_guard<std::mutex> lock(mu);
    auto& slot = cache[{key_bytes, value_bytes}];
    if (!slot || slot->max_n() < n) slot.reset(new OneSweepSorterB200(n ? n : 1, key_bytes, value_bytes));
    return *slot;
}
}  // namespace detail

inline void Sort(uint32_t* d_keys, uint64_t n, void* stream = nullptr) { detail::sorter(4, 0, n).SortKeys(d_keys, n, stream); }
inline void Sort(uint64_t* d_keys, uint64_t n, void* stream = nullptr) { detail::sorter(8, 0, n).SortKeys(d_keys, n, stream); }
inline void Sort(uint32_t* d_keys, uint32_t* d_values, uint64_t n, void* stream = nullptr)
{
    detail::sorter(4, 4, n).SortPairs(d_keys, d_values, n, stream);
}
inline void Sort(uint64_t* d_keys, uint32_t* d_values, uint64_t n, void* stream = nullptr)
{
    detail::sorter(8, 4, n).SortPairs(d_keys, d_values, n, stream);
}
}  // namespace OneSweep
