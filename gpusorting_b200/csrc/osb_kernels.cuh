// osb_kernels.cuh -- launch interface of the sm_90a OneSweep kernels (implemented in osb_kernels.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "osb_common.cuh"

namespace osb {

// Kernel variants of the digit-binning pass (osb200_set_option "variant").
enum BinningVariant : int {
    kVariantTilePerCta = 0,  // one CTA per partition tile, keys loaded straight into registers
    kVariantPersistent = 1,  // persistent CTAs, TMA (cp.async.bulk) double-buffered tile staging
    kVariantWide = 2,        // 16,384-key tiles, two-phase atomic ranking, compact reductions + one-shot lookback
};
constexpr int kNumVariants = 3;
enum RankMode : int {
    kRankAtomic = 0,  // one shared-memory atomicAdd per key (lane order verified on the device at create)
    kRankBallot = 1,  // 8 ballots per key (the reference's warp-level multisplit, OneSweep.cu:208-253)
};

struct BinningConfig {
    int variant = kVariantTilePerCta;
    int rank_mode = kRankAtomic;
    int sm_count = 132;
    KeyCodec codec;  // typed keys: encode-on-load / decode-on-store for THIS launch (flags 0 = plain unsigned keys)
    // --- per-launch pass parameters (kVariantWide honours all of them; the other variants need the defaults) ---
    uint32_t digit_bits = 8;          // width of this pass's digit, 1..8 (narrower: last place of a begin/end-bit sort)
    const SortPlan* plan = nullptr;   // device plan: skip flag, ping-pong parity, dynamic codec flags; null = as launched
    uint32_t place = 0;               // index of this pass in the plan
    uint32_t spin_cap = 2048;         // lookback polls of one predecessor before the digit thread re-reduces that tile itself
    uint32_t debug_stall_every = 0;   // test hook: tiles with tile % N == N-1 never publish their reduction (0 = off)
    uint32_t debug_max_ctas = 0;      // test hook: at most this many persistent CTAs per pass (0 = as many as can be resident)
    bool hot_passes = false;          // also enqueue the HOT instantiation (the plan decides which of the two runs the pass)
    const void* argsort_in = nullptr; // argsort (u32/u16/u64 pairs, needs the plan): the first executed pass reads its keys from here
                                      // and makes every payload from the key's input position (in/in_val: output keys/indices)
    // fused sorts (u32 keys, DESIGN §4.12): the region capacity and place 0's dense digit bases, with which the first executed
    // pass after place 0 reads the gapped layout the fused first pass leaves when the plan keeps it (0 / null: not a fused sort)
    uint64_t fused_region = 0;
    const unsigned long long* fused_dense_base0 = nullptr;
};

// keys per partition tile for a key width / pairs flag / variant (host needs it to size descriptors)
uint32_t binning_tile_keys(int key_bytes, bool pairs, const BinningConfig& cfg);
// whether the pass that runs these keys in cfg.variant has a HOT instantiation (BinningConfig::hot_passes)
bool binning_has_hot_twin(int key_bytes, bool pairs, bool indices, const BinningConfig& cfg);

// One-time per-process kernel attribute setup (dynamic shared memory opt-in). Returns cudaError_t.
cudaError_t configure_kernels();

// GlobalHistogram (reference: OneSweep::GlobalHistogram, Sort/OneSweep.cu:44-123).
// ghist[place*256 + digit] += counts; caller zeroes ghist first.  gate != null: the fallback of a fused sort, which returns
// at once when the plan keeps the fused first pass.
cudaError_t launch_global_histogram(const void* keys, uint64_t n, int key_bytes, unsigned long long* ghist,
                                    int sm_count, cudaStream_t stream, const KeyCodec* codec = nullptr, const SortPlan* gate = nullptr);

// ---- fused sorts: whole-key u32 keys-only sorts without a GlobalHistogram in front (DESIGN §4.12) -------------------------
// The fused first pass: reads keys (codec: encode on load), writes digit d's keys to alt[d * region, (d + 1) * region), adds
// the histogram of places 0-3 to ghist[0..1023] (zeroed by the caller), and sets *abort_word (zeroed by the caller) instead
// of overflowing a region.  No plan; its own ticket, place 0's epoch and reductions.  *ctas: the CTAs it launched.
cudaError_t launch_fused_first_pass(const uint32_t* keys, uint32_t* alt, uint64_t n, uint64_t region, unsigned long long* ghist,
                                    uint32_t* abort_word, uint64_t* desc, uint16_t* agg16, uint32_t* ticket, uint32_t epoch,
                                    const BinningConfig& cfg, cudaStream_t stream, uint32_t* ctas);
// The scan after the fused first pass (fallback = false): the plan of launch_scan plus kPlanFusedKept when the fused pass
// stands.  The fallback's scan (fallback = true) returns at once when it does, else writes the classic plan.
cudaError_t launch_scan_fused(const unsigned long long* ghist, unsigned long long* gbase, int places, cudaStream_t stream,
                              SortPlan* plan, uint64_t n, bool allow_skip, bool allow_hot, bool fallback, const uint32_t* fused_abort,
                              uint64_t region);
// The fallback's clear of place 0's reductions and the descriptors of the tiles the fused pass reached (its ctas and the
// tiles drawn from its ticket, at most tiles); returns at once when the plan keeps the fused pass.
cudaError_t launch_fused_fallback_zero(const SortPlan* plan, const uint32_t* ticket, uint32_t ctas, uint64_t tiles, uint16_t* agg16,
                                       uint64_t* desc, int sm_count, cudaStream_t stream);

// Single-place histogram (used by the sharded path for the most significant digit): hist256[digit] += counts.
cudaError_t launch_digit_histogram(const void* keys, uint64_t n, int key_bytes, uint32_t shift,
                                   unsigned long long* hist256, int sm_count, cudaStream_t stream);

// Scan (reference: OneSweep::Scan, Sort/OneSweep.cu:125-162): per place exclusive prefix of ghist -> gbase.
// With plan != null the kernel also writes the device launch plan: a place is skipped when one of its bins holds all n
// keys (allow_skip), and the first/last executed places are recorded for the typed-key codec.
cudaError_t launch_scan(const unsigned long long* ghist, unsigned long long* gbase, int places, cudaStream_t stream,
                        SortPlan* plan = nullptr, uint64_t n = 0, bool allow_skip = false, bool allow_hot = false);

// GlobalHistogram of a begin_bit/end_bit sort: place p counts the digit (key >> (begin_bit + 8p)) & mask_p, mask_p = 255
// except for the last place, which keeps last_bits bits.  (The byte-aligned full-width case uses launch_global_histogram.)
cudaError_t launch_global_histogram_bits(const void* keys, uint64_t n, int key_bytes, unsigned long long* ghist, int sm_count,
                                         cudaStream_t stream, const KeyCodec* codec, uint32_t begin_bit, int places,
                                         uint32_t last_bits);

// If the plan says an odd number of passes ran, the sorted data sits in the alt buffers: move it to the caller's.
cudaError_t launch_copy_back(const SortPlan* plan, const void* alt_keys, void* keys, const uint32_t* alt_vals, uint32_t* vals,
                             uint64_t n, int key_bytes, int sm_count, cudaStream_t stream);
// The same for an argsort (16-, 32- or 64-bit keys, u32 indices): an odd number of executed passes -> move keys and indices from
// the alt buffers; none (every digit place constant) -> the keys are copied from the untouched input and the indices are 0..n-1.
cudaError_t launch_argsort_copy_back(const SortPlan* plan, const void* keys_in, const void* alt_keys, void* keys,
                                     const uint32_t* alt_idx, uint32_t* idx, uint64_t n, int key_bytes, int sm_count,
                                     cudaStream_t stream);

// DigitBinningPass (reference: OneSweep::DigitBinningPassKeysOnly / Pairs, Sort/OneSweep.cu:164-600).
//   gbase_place: [256] exclusive global digit bases for this digit place
//   desc:        [tiles][256] 64-bit tile descriptors (not cleared between eager launches; `epoch` distinguishes them)
//   agg16:       [tiles][256] 16-bit tile reductions (flag:1|count:15) used by kVariantWide; zeroed per sort
//   ticket:      one zeroed u32 (dynamic tile id counter, reference `index[]`)
cudaError_t launch_digit_binning(const void* in, void* out, const uint32_t* in_val, uint32_t* out_val, uint64_t n,
                                 int key_bytes, uint32_t shift, const unsigned long long* gbase_place, uint64_t* desc,
                                 uint16_t* agg16, uint32_t* ticket, uint32_t epoch, const BinningConfig& cfg,
                                 cudaStream_t stream);

// Segment sort / small-n path: one CTA sorts one segment (<= segment_sort_capacity keys) in shared memory, all digit passes
// in one launch.  seg_off == nullptr: the single segment [0, single_n).  max_len (an upper bound of the segment lengths)
// picks the geometry; segments longer than the capacity are skipped by the kernel (the caller must not pass them).
// keys_in != null (argsort of the single segment; u16, u32 or u64 keys, vals = indices): the keys are read from keys_in, the
// payloads are the keys' input positions, and the sorted keys and indices are stored to keys / vals.
// key_bytes 2 (16-bit keys), and key_bytes 8 with vals: only the single segment of a sort (seg_off null), up to 16,384 keys
// (8,192 for 64-bit keys).
uint32_t segment_sort_capacity(int key_bytes);
cudaError_t launch_segment_sort(void* keys, uint32_t* vals, int key_bytes, const unsigned long long* seg_off, uint64_t num_segments,
                                uint64_t single_n, uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits,
                                const KeyCodec* codec, int rank_mode, int sm_count, cudaStream_t stream,
                                const void* keys_in = nullptr);

// Row sort: row r = elements [r * row_len, (r + 1) * row_len) of keys_in, sorted stable into the same row of keys_out
// (keys_out == keys_in: in place); indices (may be null) receives every output key's position within its row.  Rows of at
// most kRowWarpMaxLen keys are sorted one per warp (row_sort_warp_kernel) unless block_only; longer rows, up to
// row_sort_capacity(key_bytes), one per CTA by segment_sort_kernel (2,048- or 16,384-key geometry).  key_bytes 2, 4 or 8; the
// codec (both flags set, or null for plain unsigned ascending keys) is applied on load and undone on store.  The caller
// handles row_len == 1, which the block path leaves untouched.
constexpr uint32_t kRowWarpMaxLen = 256;
uint32_t row_sort_capacity(int key_bytes);
cudaError_t launch_row_sort(const void* keys_in, void* keys_out, uint32_t* indices, uint64_t num_rows, uint32_t row_len,
                            int key_bytes, const KeyCodec* codec, int rank_mode, bool block_only, int sm_count,
                            cudaStream_t stream);

// Long rows (osb200_sort_long_rows): rows of any length >= 2, LSD radix sort over tiles of kLongRowTile keys that never straddle
// rows, reduce-then-scan within each row (no tile waits on another).  Enqueues the GlobalHistogram over all n = num_rows *
// row_len keys into ghist (zeroed by the caller), the scan that writes `plan` (gbase is written too, and not used), per digit
// place a count, a scan of each row's tile counts and a scatter, then the copy home.  alt_keys: n keys of key_bytes;
// alt_idx: n u32 when indices is not null; scratch: long_rows_scratch_bytes(num_rows, row_len) bytes, 16-byte aligned, which
// the call overwrites before it reads them.  The codec as for launch_row_sort.
constexpr uint32_t kLongRowTile = 8192;
uint64_t long_rows_scratch_bytes(uint64_t num_rows, uint32_t row_len);
cudaError_t launch_long_rows(const void* keys_in, void* keys_out, uint32_t* indices, void* alt_keys, uint32_t* alt_idx,
                             uint64_t num_rows, uint32_t row_len, int key_bytes, const KeyCodec* codec, int rank_mode,
                             bool allow_skip, unsigned long long* ghist, unsigned long long* gbase, SortPlan* plan,
                             uint32_t* scratch, int sm_count, cudaStream_t stream);

// Long segments (osb200_sort_long_segments): launch_sort_segments for segments of 2 to long_min - 1 keys, and the long
// rows' passes for segments of long_min to max_len keys (long_min >= 2), whose tiles of kLongRowTile keys never straddle
// segments; nothing outside [0, n)'s valid segments of at most max_len keys is written.  Enqueues the binning (the class
// lists in `list`, num_segments u32), the class kernels, a one-CTA tile map of the long list, the GlobalHistogram over all
// n keys into ghist (zeroed by the caller) and the scan that writes `plan`, per digit place a count, a scan of each long
// segment's tile counts and a scatter, then the copy home of the long segments.  counts: 7 u64, cleared here.  alt_keys:
// n keys of key_bytes (it may hold `list`: the class kernels run before the passes); alt_idx: n u32 when indices is not
// null; scratch: long_segments_layout(n, long_min).words u32, 16-byte aligned.  The codec as for launch_row_sort.
// The layout bounds every listed set of disjoint segments of long_min or more keys among n: at most list_cap = n / long_min
// of them, with at most tile_cap tiles and chunk_cap scan chunks.
struct LongSegLayout { uint64_t list_cap, tile_cap, chunk_cap, csum, list, tfirst, cfirst, words; };  // offsets in u32 words
LongSegLayout long_segments_layout(uint64_t n, uint32_t long_min);
cudaError_t launch_long_segments(const void* keys_in, void* keys_out, uint32_t* indices, void* alt_keys, uint32_t* alt_idx, uint64_t n,
                                 const unsigned long long* off, uint64_t num_segments, uint32_t max_len, uint32_t long_min,
                                 int key_bytes, const KeyCodec* codec, int rank_mode, bool allow_skip, unsigned long long* ghist,
                                 unsigned long long* gbase, SortPlan* plan, uint32_t* list, unsigned long long* counts,
                                 uint32_t* scratch, int sm_count, cudaStream_t stream);

// Segment sort by offsets (osb200_sort_segments): segment s = [off[s], off[s + 1]) of keys_in, sorted stable into the same
// positions of keys_out (== keys_in: in place); indices (may be null) receives every output key's position within its segment.
// A binning kernel puts every segment of 2 to max_len keys that lies inside [0, n) into a class by its length -- one warp
// (at most kRowWarpMaxLen keys), the 2,048-key block geometry (at most kSegBlock1Max) or the largest one -- and writes the
// one-key segments itself; then one kernel per class that max_len reaches sorts its segments.  max_len in 1 ..
// row_sort_capacity(key_bytes).  list: num_segments u32 of workspace; counts: 4 u64 of workspace, cleared here.  The codec
// as for launch_row_sort.
constexpr uint32_t kSegBlock1Max = 2048;
cudaError_t launch_sort_segments(const void* keys_in, void* keys_out, uint32_t* indices, uint64_t n,
                                 const unsigned long long* off, uint64_t num_segments, uint32_t max_len, int key_bytes,
                                 const KeyCodec* codec, int rank_mode, int sm_count, uint32_t* list,
                                 unsigned long long* counts, cudaStream_t stream);

// Row top-k (osb200_topk_rows): the first k keys of row r = [r * row_len, (r + 1) * row_len) of keys_in in its stable sort, and
// their positions within the row, into [r * k, (r + 1) * k) of values_out and indices.  Rows of at most kRowWarpMaxLen keys are
// sorted one per warp unless block_only; longer rows are radix-selected one per CTA (topk_select_kernel), the candidates held
// in shared memory once at most `capacity` of them are left (0: row_sort_capacity(key_bytes)).  sorted: the block path's
// result is then sorted in place (a second launch); without it the k pairs of a row are in an unspecified order.
// k in 1 .. min(row_len, row_sort_capacity(key_bytes)); the codec as for launch_row_sort.
cudaError_t launch_topk_rows(const void* keys_in, void* values_out, uint32_t* indices, uint64_t num_rows, uint32_t row_len,
                             uint32_t k, int key_bytes, const KeyCodec* codec, bool sorted, uint32_t capacity, int rank_mode,
                             bool block_only, int sm_count, cudaStream_t stream);

// Segment top-k (osb200_topk_segments): segment s = [off[s], off[s + 1]) of keys_in; its first m = min(length, k) keys in the
// stable sort and their positions within the segment go to [s * k, s * k + m) of values_out and indices, and columns m .. k - 1
// are padding (the decoded all-ones key, position 0xFFFFFFFF).  Segments whose offsets decrease, pass n or span 2^32 keys or
// more are all padding.  A binning kernel lists segments of at most kRowWarpMaxLen keys (0 with block_only), and the empty and
// invalid ones, for one warp each and the longer ones for the radix select, one CTA each, the candidates held in shared
// memory once at most `capacity` are left (0: row_sort_capacity(key_bytes)); sorted then sorts the select's rows in place.
// k in 0 .. row_sort_capacity(key_bytes); list: num_segments u32 of workspace; counts: 4 u64 of workspace, cleared here.  The
// codec as for launch_row_sort.
cudaError_t launch_topk_segments(const void* keys_in, void* values_out, uint32_t* indices, uint64_t n, const unsigned long long* off,
                                 uint64_t num_segments, uint32_t k, int key_bytes, const KeyCodec* codec, bool sorted,
                                 uint32_t capacity, int rank_mode, bool block_only, int sm_count, uint32_t* list,
                                 unsigned long long* counts, cudaStream_t stream);

// Validate (reference: Validate, UtilityKernels.cuh:403-429): err_count += #(keys[i] > keys[i+1]).
cudaError_t launch_validate(const void* keys, uint64_t n, int key_bytes, unsigned long long* err_count, int sm_count,
                            cudaStream_t stream);

// InitRandom (reference: InitRandom, UtilityKernels.cuh:53-117, launched <<<256,256>>> by
// OneSweepDispatcher.cuh:100-104): the reference's deterministic test-input generator.  65,536 hybrid
// Tausworthe/LCG streams; stream g writes elements g, g+65536, ...; each element ANDs and_count+1 draws.
// payload (may be null) receives a copy of the key (reference pairs overload) or, if payload_is_index, i.
cudaError_t launch_init_random(uint32_t* keys, uint32_t* payload, uint64_t n, uint32_t and_count, uint32_t seed,
                               bool payload_is_index, cudaStream_t stream);

// Device self-test: does a shared-memory atomicAdd hand out its return values in ascending lane order among
// the lanes of one warp instruction that hit the same address?  (kRankAtomic depends on it.)
// mismatches (device u64) receives the number of violations found.
cudaError_t launch_atomic_order_selftest(unsigned long long* mismatches, int sm_count, cudaStream_t stream);

}  // namespace osb
