// osb_host.cu -- host driver + C-ABI (include/onesweep_b200.h) of the H100 OneSweep sort.
//
// The sorter object plays the role of the reference's OneSweepDispatcher (Sort/OneSweepDispatcher.cuh:17-83):
// it owns the ping-pong buffers and the control state and issues the launch plan of
// OneSweepDispatcher.cuh:311-363 -- GlobalHistogram, Scan, then one DigitBinningPass per digit place,
// ping-ponging keys -> alt -> keys.  Differences, all deliberate (DESIGN.md):
//   * no per-sort memset of the 64-bit inclusive descriptors (epoch-stamped); per sort there are two memsets: the 8.3 KB
//     control block (global histogram + tile tickets) and the compact 16-bit reductions (512 B per tile and place:
//     128 MiB at n = 2^30 u32, ~20 us) -- against the reference's 6 memsets over ~573 MB at n = 2^30.  A sort enqueued
//     under stream capture also clears its descriptors before and after its passes (is_capturing);
//   * passes whose digit is the same for every key are skipped, and passes with one dominant bin run in the HOT
//     instantiation of the pass, both decided on the device (osb::SortPlan);
//   * a sort of at most one tile is ONE launch of the single-CTA shared-memory sort (also the segmented sort);
//   * no host synchronisation inside the sort; everything is enqueued on the caller's stream;
//   * the caller owns keys/values.
#include <cstdio>
#include <cstring>
#include <new>

#include "../../include/onesweep_b200.h"
#include "osb_kernels.cuh"
#include "osb_common.cuh"
#include "osb_internal.h"

namespace {

constexpr int kVersion = 1011;  // 1002: device plan, bit ranges, forward-progress fallback, hot passes, segmented sort; 1003: argsort;
                                // 1004: 16-bit keys (osb200_sort_keys16, osb200_sort_pairs16, osb200_argsort16);
                                // 1005: row sort (osb200_sort_rows);
                                // 1006: 64-bit keys with uint32 payloads and their argsort (osb200_create_pairs64);
                                // 1007: segment sort by offsets (osb200_sort_segments);
                                // 1008: row top-k (osb200_topk_rows);
                                // 1009: segment top-k (osb200_topk_segments);
                                // 1010: rows of any length (osb200_sort_long_rows);
                                // 1011: segments of any length (osb200_sort_long_segments)
constexpr int kMaxPlaces = 8;

inline int cuda_status(cudaError_t e) { return e == cudaSuccess ? OSB200_OK : OSB200_ERR_CUDA - static_cast<int>(e); }

#define OSB_TRY(expr)                                      \
    do {                                                   \
        cudaError_t e__ = (expr);                          \
        if (e__ != cudaSuccess) return cuda_status(e__);   \
    } while (0)

// Control block, zeroed by ONE memset per sort: [ghist: 8*256 u64][tickets: 8 u32 (padded)]
struct ControlLayout {
    static constexpr size_t ghist_bytes = kMaxPlaces * osb::kRadix * sizeof(unsigned long long);
    static constexpr size_t ticket_bytes = 64;  // 8 u32 tickets, padded
    static constexpr size_t zeroed_bytes = ghist_bytes + ticket_bytes;
    static constexpr size_t gbase_bytes = kMaxPlaces * osb::kRadix * sizeof(unsigned long long);
    static constexpr size_t err_bytes = 64;   // scratch of the calls that clear it first: validate, the segment calls' counts
    static constexpr size_t plan_bytes = 64;  // osb::SortPlan, written by the scan kernel of every sort
    static constexpr size_t total = zeroed_bytes + gbase_bytes + err_bytes + plan_bytes;
};

}  // namespace

struct osb200_sorter {
    int device = 0;
    int sm_count = 132;
    uint64_t max_n = 0;
    int key_bytes = 4;
    int value_bytes = 0;
    osb::BinningConfig cfg;
    bool atomic_order_ok = false;
    bool short_circuit = true;   // skip passes whose digit is the same for all keys (decided on the device, no host sync)
    bool small_path = true;      // n <= one tile: the single-CTA shared-memory sort (one launch)
    bool hot_passes = true;      // low-entropy digit places run in the HOT instantiation of the pass (decided on the device)
    bool debug_rows_block = false;  // test hook: osb200_sort_rows sorts rows of <= 256 keys on the block path, not the warp path
    uint32_t debug_topk_capacity = 0;  // test hook: N > 0 holds at most N candidates of osb200_topk_rows in shared memory
    bool debug_long_rows = false;   // test hook: osb200_sort_long_rows and osb200_sort_long_segments sort rows and segments of
                                    // 2 .. row_sort_capacity keys on the long path
    bool fused_histogram = true;    // whole-key u32 keys-only sorts of >= kFusedMinTiles tiles: the fused first pass (§4.12)

    void* alt_keys = nullptr;
    uint64_t alt_key_slots = 0;        // keys (of key_bytes) the alt key buffer holds: max_n, or the fused regions' 256 c(max_n)
    uint32_t* alt_vals = nullptr;
    unsigned char* control = nullptr;  // ControlLayout
    uint64_t* desc = nullptr;          // [tiles][256] 64-bit descriptors (epoch-stamped, cleared only by captured sorts)
    uint16_t* agg16 = nullptr;         // [places][tiles][256] compact reductions (zeroed once per sort)
    uint64_t agg16_bytes = 0;
    uint64_t desc_tiles = 0;
    uint32_t epoch = 0;

    // optional per-kernel timing of the last sort (osb200_set_option "profile"): events on the launching stream, and the
    // spans between them that make up each reported entry ([histogram, scan, pass 0, pass 1, ...])
    bool profile = false;
    static constexpr int kMaxEvents = kMaxPlaces + 6;
    cudaEvent_t ev[kMaxEvents] = {};
    int ev_count = 0;
    struct Span { int entry, from, to; };
    Span spans[kMaxEvents] = {};
    int span_count = 0;

    // lazily created staging for the host-buffer entry points
    void* stage_keys = nullptr;
    uint32_t* stage_vals = nullptr;
    cudaStream_t own_stream = nullptr;

    unsigned long long* ghist() const { return reinterpret_cast<unsigned long long*>(control); }
    uint32_t* tickets() const { return reinterpret_cast<uint32_t*>(control + ControlLayout::ghist_bytes); }
    unsigned long long* gbase() const { return reinterpret_cast<unsigned long long*>(control + ControlLayout::zeroed_bytes); }
    unsigned long long* err() const
    {
        return reinterpret_cast<unsigned long long*>(control + ControlLayout::zeroed_bytes + ControlLayout::gbase_bytes);
    }
    osb::SortPlan* plan() const
    {
        return reinterpret_cast<osb::SortPlan*>(control + ControlLayout::zeroed_bytes + ControlLayout::gbase_bytes + ControlLayout::err_bytes);
    }

};

namespace {

uint64_t tiles_for(uint64_t n, uint32_t tile_keys) { return (n + tile_keys - 1) / tile_keys; }

// Fused sorts (DESIGN §4.12): whole-key u32 keys-only sorts on the default pass of at least this many tiles, and below 2^32
// keys (the fused pass counts in 32-bit words).  Smaller sorts keep the classic launch plan: there the saved read is a few
// microseconds, and a region's slack is a large share of its keys.
constexpr uint64_t kFusedMinTiles = 64;
constexpr int kFusedTicket = 4, kFusedAbort = 5;  // control-block slots of the fused pass (a u32 sort uses tickets 0-3)

bool fused_size(uint64_t n)
{
    osb::BinningConfig wide;
    wide.variant = osb::kVariantWide;
    return n < (1ull << 32) && tiles_for(n, osb::binning_tile_keys(4, false, wide)) >= kFusedMinTiles;
}

// keys the alt key buffer of a handle holds: max_n, or the fused pass's 256 regions when a u32 sort of max_n keys is fused
uint64_t alt_key_slots_for(uint64_t max_n, int key_bytes)
{
    const uint64_t regions = key_bytes == 4 && fused_size(max_n) ? osb::kRadix * osb::fused_region_keys(max_n) : 0;
    return regions > max_n ? regions : max_n;
}
// the compact reductions are stored in blocks of 8 tiles ([tile/8][digit][tile%8], see osb_kernels.cu agg_index)
uint64_t agg_tiles_for(uint64_t n, uint32_t tile_keys) { return (tiles_for(n, tile_keys) + 7) / 8 * 8; }

uint32_t smallest_tile(int key_bytes, bool pairs)
{
    // descriptors are sized for the smallest tile any variant may use
    osb::BinningConfig c;
    uint32_t t = osb::binning_tile_keys(key_bytes, pairs, c);
    for (int v = 1; v < osb::kNumVariants; ++v) {
        c.variant = v;
        const uint32_t t2 = osb::binning_tile_keys(key_bytes, pairs, c);
        if (t2 < t) t = t2;
    }
    return t;
}

// advance the epoch; on wrap-around clear the descriptors once (every ~16M passes)
int next_epoch(osb200_sorter* s, cudaStream_t stream, uint32_t* out)
{
    if (s->epoch >= osb::kEpochMax) {
        OSB_TRY(cudaMemsetAsync(s->desc, 0, s->desc_tiles * osb::kRadix * sizeof(uint64_t), stream));
        s->epoch = 0;
    }
    *out = ++s->epoch;
    return OSB200_OK;
}

// Under stream capture the epochs become launch arguments frozen into the graph: every replay runs with the epochs of the
// capture.  Where the previous replay's last executed pass is the digit place of this replay's first (always for a single
// pass; else when the plan skips passes), a tile would take the previous replay's inclusive prefixes for its own where no
// other sort has overwritten them since.  So a captured sort clears the words of
// its tiles before its first pass and after its last: the first clear hides words an eager sort left with the same epochs
// (after a wrap-around), the second hides the replay's words from a later eager sort that reuses them.  Eager sorts never
// clear.
int is_capturing(cudaStream_t stream, bool* out)
{
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    OSB_TRY(cudaStreamGetCaptureInfo(stream, &st));
    *out = st == cudaStreamCaptureStatusActive;
    return OSB200_OK;
}

int check_handle(const osb200_sorter* s) { return s ? OSB200_OK : OSB200_ERR_INVALID_ARG; }

bool overlaps(uintptr_t a, uint64_t alen, uintptr_t b, uint64_t blen) { return a < b + blen && b < a + alen; }

// An array argument of the row and segment sorts and top-k: its address, size in bytes and natural alignment, whether null
// is an error (else a null array is absent), and whether the call writes it.
struct ArrayArg { const void* p; uint64_t bytes; int align; bool required, written; };

// The argument checks of osb200_sort_rows, osb200_sort_segments, osb200_topk_rows and osb200_topk_segments, in order:
// every required array is given; every array is naturally aligned (the kernels load and store element by element); the
// byte sizes fit in 64 bits (sizes_fit); no array the call writes overlaps another one -- except a[1] == a[0] (out == in)
// where the call sorts in place, since a row or segment is read whole before it is written.
template <size_t N>
int check_arrays(const ArrayArg (&a)[N], bool sizes_fit, bool in_place)
{
    for (const ArrayArg& x : a)
        if ((x.required && !x.p) || (reinterpret_cast<uintptr_t>(x.p) & static_cast<uintptr_t>(x.align - 1)))
            return OSB200_ERR_INVALID_ARG;
    if (!sizes_fit) return OSB200_ERR_INVALID_ARG;
    for (size_t i = 0; i < N; ++i)
        for (size_t j = i + 1; j < N; ++j) {
            const ArrayArg &x = a[i], &y = a[j];
            if (!x.p || !y.p || !(x.written || y.written) || (in_place && i == 0 && j == 1 && x.p == y.p)) continue;
            if (overlaps(reinterpret_cast<uintptr_t>(x.p), x.bytes, reinterpret_cast<uintptr_t>(y.p), y.bytes))
                return OSB200_ERR_INVALID_ARG;
        }
    return OSB200_OK;
}

// The workspace of the segment calls: one u32 per segment of the alt key buffer for the class lists (at least 4 max_n bytes
// for every handle shape; segment ids are u32) and the 4 u64 class counts in the control block's scratch words (err()).
int check_segment_workspace(const osb200_sorter* h, uint64_t num_segments)
{
    static_assert(ControlLayout::err_bytes >= 4 * sizeof(unsigned long long), "the class counts live in the scratch words");
    return num_segments > h->max_n || num_segments > (1ull << 32) ? OSB200_ERR_SIZE : OSB200_OK;
}

// The launch plan (reference: OneSweepDispatcher.cuh:311-363): GlobalHistogram, Scan, one DigitBinningPass per digit
// place of [begin_bit, end_bit), then the (normally empty) copy-back.  Everything is enqueued on `stream`; which passes
// actually move data is decided on the device (osb::SortPlan): the host never waits for the histogram.
// keys_in != null is an argsort (osb200_argsort): d_keys / d_vals are its outputs, the keys and indices, and are not read.
// The histogram reads keys_in, the first executed pass reads keys_in and makes the indices, and the copy-back also covers
// a sort in which no pass executes.
// key_bytes is the width of the keys being sorted: the handle's own, or 2 for the 16-bit calls (osb200_sort_keys16 & co.),
// which run on a 4-byte handle -- its alternate buffers (4 B per key), descriptors (sized for its smallest tile, which the
// 16-bit tiles are not below) and reductions (four digit places) cover a 16-bit sort of up to max_n keys.
int sort_impl(osb200_sorter* s, int key_bytes, void* d_keys, uint32_t* d_vals, uint64_t n, cudaStream_t stream,
              const osb::KeyCodec* codec = nullptr, int begin_bit = 0, int end_bit = -1, const void* keys_in = nullptr)
{
    const int key_bits = key_bytes * 8;
    if (end_bit < 0) end_bit = key_bits;
    if (begin_bit < 0 || end_bit > key_bits || begin_bit > end_bit) return OSB200_ERR_INVALID_ARG;
    if (n <= 1 || begin_bit == end_bit) return OSB200_OK;
    if (n > s->max_n) return OSB200_ERR_SIZE;
    if (!d_keys || (reinterpret_cast<uintptr_t>(d_keys) & 15u)) return OSB200_ERR_INVALID_ARG;
    // d_vals == nullptr is a keys-only sort (also on a pairs-capable handle); the handle is never modified to say so
    if (d_vals && !s->value_bytes) return OSB200_ERR_INVALID_ARG;
    const int places = (end_bit - begin_bit + 7) / 8;
    const uint32_t last_bits = static_cast<uint32_t>(end_bit - begin_bit - 8 * (places - 1));
    const bool whole_key = begin_bit == 0 && end_bit == key_bits;
    const bool wide = s->cfg.variant == osb::kVariantWide;
    // the device plan (pass skipping, odd pass counts, bit ranges) is a feature of the default kernel
    if (!wide && !whole_key) return OSB200_ERR_UNSUPPORTED;
    const bool use_plan = wide;

    // small-n path (SURVEY 8f rank 4): up to one tile of keys is sorted by ONE CTA in shared memory, one launch
    if (wide && s->small_path && n <= osb::segment_sort_capacity(key_bytes)) {
        osb::KeyCodec c;
        if (codec) { c = *codec; c.flags = osb::kCodecEncodeOnLoad | osb::kCodecDecodeOnStore; }
        s->ev_count = 0;
        OSB_TRY(osb::launch_segment_sort(d_keys, d_vals, key_bytes, nullptr, 1, n, static_cast<uint32_t>(n),
                                         static_cast<uint32_t>(begin_bit), static_cast<uint32_t>(places), last_bits,
                                         codec ? &c : nullptr, s->cfg.rank_mode, s->sm_count, stream, keys_in));
        return OSB200_OK;
    }

    bool capturing = false;
    int st = is_capturing(stream, &capturing);
    if (st != OSB200_OK) return st;
    const uint32_t tile_keys = osb::binning_tile_keys(key_bytes, d_vals != nullptr, s->cfg);
    const size_t desc_bytes = tiles_for(n, tile_keys) * osb::kRadix * sizeof(uint64_t);
    if (capturing) OSB_TRY(cudaMemsetAsync(s->desc, 0, desc_bytes, stream));
    OSB_TRY(cudaMemsetAsync(s->control, 0, ControlLayout::zeroed_bytes, stream));
    const bool compact = s->cfg.variant != osb::kVariantTilePerCta;  // every other variant uses the compact reductions
    const uint64_t agg_stride = agg_tiles_for(n, tile_keys) * osb::kRadix;
    // reductions carry no epoch (16-bit words): they are cleared per sort, 512 B per tile and place (128 MiB at n = 2^30)
    if (compact) OSB_TRY(cudaMemsetAsync(s->agg16, 0, agg_stride * places * sizeof(uint16_t), stream));
    // profile: events in stream order, and the spans between them that make up each entry of osb200_get_profile
    int ne = 0;
    s->span_count = 0;
    auto mark = [&]() -> cudaError_t {
        if (!s->profile) return cudaSuccess;
        if (!s->ev[ne]) { cudaError_t e = cudaEventCreate(&s->ev[ne]); if (e != cudaSuccess) return e; }
        return cudaEventRecord(s->ev[ne++], stream);
    };
    auto span = [&](int entry) -> cudaError_t {  // entry: the launches since the previous mark
        if (s->profile) s->spans[s->span_count++] = {entry, ne - 1, ne};
        return mark();
    };
    s->ev_count = 0;
    OSB_TRY(mark());
    osb::KeyCodec enc;  // typed keys: the histogram and the first executed pass see encoded keys, the last one stores them decoded
    if (codec) { enc = *codec; enc.flags = osb::kCodecEncodeOnLoad; }
    // hot passes (low-entropy inputs): the default kernel has a second instantiation for them; both are enqueued per pass
    const bool hot_passes = use_plan && s->hot_passes && osb::binning_has_hot_twin(key_bytes, d_vals != nullptr, keys_in != nullptr, s->cfg);
    // Fused sort (DESIGN §4.12): the first pass counts the global histogram and scatters into fixed regions of the alt
    // buffer; the scan after it keeps that result or calls the fallback -- the classic histogram, scan and first pass,
    // enqueued always and returning at once when the fused pass stands.
    const uint64_t region = osb::fused_region_keys(n);
    const bool fused = s->fused_histogram && use_plan && whole_key && key_bytes == 4 && !d_vals && !keys_in && fused_size(n) &&
                       osb::kRadix * region <= s->alt_key_slots;
    // (the fused pass runs on place 0's epoch: one epoch per digit place, as in the classic plan)
    uint32_t fused_epoch = 0;
    if (fused) {
        st = next_epoch(s, stream, &fused_epoch);
        if (st != OSB200_OK) return st;
        const uint32_t epoch = fused_epoch;
        osb::BinningConfig cfg = s->cfg;
        if (codec) cfg.codec = enc;
        unsigned long long* fallback_hist = s->ghist() + 4 * osb::kRadix;  // a 4-place sort's unused places 4-7
        uint32_t* abort_word = s->tickets() + kFusedAbort;
        uint32_t ctas = 0;
        OSB_TRY(osb::launch_fused_first_pass(static_cast<const uint32_t*>(d_keys), static_cast<uint32_t*>(s->alt_keys), n, region,
                                             s->ghist(), abort_word, s->desc, s->agg16, s->tickets() + kFusedTicket, epoch, cfg, stream,
                                             &ctas));
        OSB_TRY(span(2));
        OSB_TRY(osb::launch_scan_fused(s->ghist(), s->gbase(), places, stream, s->plan(), n, s->short_circuit, hot_passes, false,
                                       abort_word, region));
        OSB_TRY(span(1));
        OSB_TRY(osb::launch_fused_fallback_zero(s->plan(), s->tickets() + kFusedTicket, ctas, tiles_for(n, tile_keys), s->agg16, s->desc,
                                                s->sm_count, stream));
        OSB_TRY(osb::launch_global_histogram(d_keys, n, key_bytes, fallback_hist, s->sm_count, stream, codec ? &enc : nullptr, s->plan()));
        OSB_TRY(span(0));
        OSB_TRY(osb::launch_scan_fused(fallback_hist, s->gbase(), places, stream, s->plan(), n, s->short_circuit, hot_passes, true,
                                       nullptr, 0));
        OSB_TRY(span(1));
    } else {
        if (whole_key)
            OSB_TRY(osb::launch_global_histogram(keys_in ? keys_in : d_keys, n, key_bytes, s->ghist(), s->sm_count, stream,
                                                 codec ? &enc : nullptr));
        else
            OSB_TRY(osb::launch_global_histogram_bits(d_keys, n, key_bytes, s->ghist(), s->sm_count, stream, codec ? &enc : nullptr,
                                                      static_cast<uint32_t>(begin_bit), places, last_bits));
        OSB_TRY(span(0));
        OSB_TRY(osb::launch_scan(s->ghist(), s->gbase(), places, stream, use_plan ? s->plan() : nullptr, n, s->short_circuit, hot_passes));
        OSB_TRY(span(1));
    }

    void* src = d_keys;
    void* dst = s->alt_keys;
    uint32_t* sv = d_vals;
    uint32_t* dv = d_vals ? s->alt_vals : nullptr;
    for (int p = 0; p < places; ++p) {
        uint32_t epoch = fused_epoch;
        if (!fused || p > 0) {
            st = next_epoch(s, stream, &epoch);
            if (st != OSB200_OK) return st;
        }
        osb::BinningConfig cfg = s->cfg;
        cfg.digit_bits = p == places - 1 ? last_bits : 8u;
        cfg.place = static_cast<uint32_t>(p);
        if (use_plan) cfg.plan = s->plan();
        cfg.hot_passes = hot_passes;
        cfg.argsort_in = keys_in;
        if (fused) { cfg.fused_region = region; cfg.fused_dense_base0 = s->gbase(); }
        if (codec) {
            cfg.codec = *codec;
            cfg.codec.flags = use_plan ? osb::kCodecFromPlan
                                       : (p == 0 ? osb::kCodecEncodeOnLoad : 0u) | (p == places - 1 ? osb::kCodecDecodeOnStore : 0u);
        }
        // with a plan every launch gets (caller buffers, alt buffers) and picks its direction on the device
        OSB_TRY(osb::launch_digit_binning(use_plan ? d_keys : src, use_plan ? s->alt_keys : dst, use_plan ? d_vals : sv,
                                          use_plan ? (d_vals ? s->alt_vals : nullptr) : dv, n, key_bytes,
                                          static_cast<uint32_t>(begin_bit + 8 * p), s->gbase() + p * osb::kRadix, s->desc,
                                          s->agg16 + p * agg_stride, s->tickets() + p, epoch, cfg, stream));
        OSB_TRY(span(2 + p));
        void* t = src; src = dst; dst = t;
        uint32_t* tv = sv; sv = dv; dv = tv;
    }
    // an odd number of EXECUTED passes leaves the result in the alt buffers.  Without skipping the count is known here
    // (even for whole keys: no launch); with skipping only the device knows, and the kernel exits at once if it is even.
    if (use_plan && (s->short_circuit || (places & 1))) {
        if (keys_in)
            OSB_TRY(osb::launch_argsort_copy_back(s->plan(), keys_in, s->alt_keys, d_keys, s->alt_vals, d_vals, n, key_bytes, s->sm_count,
                                                      stream));
        else
            OSB_TRY(osb::launch_copy_back(s->plan(), s->alt_keys, d_keys, d_vals ? s->alt_vals : nullptr, d_vals, n, key_bytes,
                                          s->sm_count, stream));
    }
    if (capturing) OSB_TRY(cudaMemsetAsync(s->desc, 0, desc_bytes, stream));
    s->ev_count = ne;
    return OSB200_OK;
}

int ensure_staging(osb200_sorter* s)
{
    if (!s->own_stream) OSB_TRY(cudaStreamCreateWithFlags(&s->own_stream, cudaStreamNonBlocking));
    if (!s->stage_keys) {
        if (cudaMalloc(&s->stage_keys, s->max_n * s->key_bytes) != cudaSuccess) return OSB200_ERR_ALLOC;
    }
    if (s->value_bytes && !s->stage_vals) {
        if (cudaMalloc(&s->stage_vals, s->max_n * sizeof(uint32_t)) != cudaSuccess) return OSB200_ERR_ALLOC;
    }
    return OSB200_OK;
}

int sort_host_impl(osb200_sorter* s, void* h_keys, uint32_t* h_vals, uint64_t n)
{
    if (n <= 1) return OSB200_OK;
    if (n > s->max_n) return OSB200_ERR_SIZE;
    if (!h_keys || (h_vals && !s->value_bytes)) return OSB200_ERR_INVALID_ARG;
    int st = ensure_staging(s);
    if (st != OSB200_OK) return st;
    cudaStream_t q = s->own_stream;
    OSB_TRY(cudaMemcpyAsync(s->stage_keys, h_keys, n * s->key_bytes, cudaMemcpyHostToDevice, q));
    if (h_vals) OSB_TRY(cudaMemcpyAsync(s->stage_vals, h_vals, n * sizeof(uint32_t), cudaMemcpyHostToDevice, q));
    st = sort_impl(s, s->key_bytes, s->stage_keys, h_vals ? s->stage_vals : nullptr, n, q);
    if (st != OSB200_OK) return st;
    OSB_TRY(cudaMemcpyAsync(h_keys, s->stage_keys, n * s->key_bytes, cudaMemcpyDeviceToHost, q));
    if (h_vals) OSB_TRY(cudaMemcpyAsync(h_vals, s->stage_vals, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, q));
    OSB_TRY(cudaStreamSynchronize(q));
    return OSB200_OK;
}

}  // namespace

// ---- internal interfaces used by the sharded path (osb_internal.h) -----------------------------------------
int osb_internal_digit_histogram(osb200_handle h, const void* d_in, uint64_t n, uint32_t shift,
                                 unsigned long long* d_hist256, cudaStream_t stream)
{
    OSB_TRY(cudaMemsetAsync(d_hist256, 0, osb::kRadix * sizeof(unsigned long long), stream));
    if (n) OSB_TRY(osb::launch_digit_histogram(d_in, n, h->key_bytes, shift, d_hist256, h->sm_count, stream));
    return OSB200_OK;
}

int osb_internal_binning_pass(osb200_handle h, const void* d_in, void* d_out, uint64_t n, uint32_t shift,
                              const unsigned long long* d_hist256, const unsigned long long* out_base,
                              cudaStream_t stream)
{
    if (n == 0) return OSB200_OK;
    if (n > h->max_n) return OSB200_ERR_SIZE;
    const unsigned long long* base = out_base;
    OSB_TRY(cudaMemsetAsync(h->tickets(), 0, ControlLayout::ticket_bytes, stream));
    if (!base) {
        OSB_TRY(osb::launch_scan(d_hist256, h->gbase(), 1, stream));
        base = h->gbase();
    }
    if (h->cfg.variant != osb::kVariantTilePerCta) {
        const uint64_t tiles = agg_tiles_for(n, osb::binning_tile_keys(h->key_bytes, false, h->cfg));
        OSB_TRY(cudaMemsetAsync(h->agg16, 0, tiles * osb::kRadix * sizeof(uint16_t), stream));
    }
    uint32_t epoch = 0;
    int st = next_epoch(h, stream, &epoch);
    if (st != OSB200_OK) return st;
    osb::BinningConfig cfg = h->cfg;
    const uint32_t key_bits = static_cast<uint32_t>(h->key_bytes) * 8u;
    cfg.digit_bits = key_bits - shift < 8u ? key_bits - shift : 8u;  // a shift within 8 bits of the top: fewer than 256 bins
    OSB_TRY(osb::launch_digit_binning(d_in, d_out, nullptr, nullptr, n, h->key_bytes, shift, base, h->desc, h->agg16,
                                      h->tickets(), epoch, cfg, stream));
    return OSB200_OK;
}

extern "C" {

int osb200_version(void) { return kVersion; }

const char* osb200_status_string(int status)
{
    switch (status) {
        case OSB200_OK: return "ok";
        case OSB200_ERR_INVALID_ARG: return "invalid argument";
        case OSB200_ERR_SIZE: return "n exceeds the sorter's max_n";
        case OSB200_ERR_UNSUPPORTED: return "unsupported key/value combination";
        case OSB200_ERR_NO_DEVICE: return "no usable sm_90 CUDA device";
        case OSB200_ERR_ALLOC: return "device allocation failed";
        case OSB200_ERR_NCCL: return "NCCL error";
        default: break;
    }
    if (status <= OSB200_ERR_CUDA) return cudaGetErrorString(static_cast<cudaError_t>(OSB200_ERR_CUDA - status));
    return "unknown status";
}

uint64_t osb200_workspace_bytes(uint64_t max_n, int key_bytes, int value_bytes)
{
    if ((key_bytes != 4 && key_bytes != 8) || (value_bytes != 0 && value_bytes != 4)) return 0;
    const uint64_t tiles = tiles_for(max_n ? max_n : 1, smallest_tile(key_bytes, value_bytes != 0));
    return alt_key_slots_for(max_n, key_bytes) * key_bytes + max_n * value_bytes + tiles * osb::kRadix * sizeof(uint64_t) +
           (tiles + 8) * osb::kRadix * sizeof(uint16_t) * key_bytes + ControlLayout::total;
}

}  // extern "C"

namespace {

// What osb200_create and osb200_create_pairs64 share once the shape is accepted: the size check, the device check, the
// workspace, and the rank-mode self-test.
int create_impl(osb200_handle* out, uint64_t max_n, int key_bytes, int value_bytes)
{
    if (max_n == 0 || max_n > (1ull << 34)) return OSB200_ERR_INVALID_ARG;

    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return OSB200_ERR_NO_DEVICE; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { cudaGetLastError(); return OSB200_ERR_NO_DEVICE; }
    if (prop.major != 9 || prop.minor != 0) return OSB200_ERR_NO_DEVICE;  // sm_90a binary only: no fallback of any kind

    osb200_sorter* s = new (std::nothrow) osb200_sorter();
    if (!s) return OSB200_ERR_ALLOC;
    s->device = dev;
    s->sm_count = prop.multiProcessorCount;
    s->cfg.sm_count = s->sm_count;
    s->cfg.variant = osb::kVariantWide;
    s->max_n = max_n;
    s->key_bytes = key_bytes;
    s->value_bytes = value_bytes;

    cudaError_t e = osb::configure_kernels();
    if (e != cudaSuccess) { delete s; return cuda_status(e); }

    s->desc_tiles = tiles_for(max_n, smallest_tile(key_bytes, value_bytes != 0));
    s->alt_key_slots = alt_key_slots_for(max_n, key_bytes);
    bool ok = cudaMalloc(&s->alt_keys, s->alt_key_slots * key_bytes) == cudaSuccess;
    if (ok && value_bytes) ok = cudaMalloc(&s->alt_vals, max_n * sizeof(uint32_t)) == cudaSuccess;
    ok = ok && cudaMalloc(&s->control, ControlLayout::total) == cudaSuccess;
    ok = ok && cudaMalloc(&s->desc, s->desc_tiles * osb::kRadix * sizeof(uint64_t)) == cudaSuccess;
    s->agg16_bytes = (s->desc_tiles + 8) * osb::kRadix * sizeof(uint16_t) * key_bytes;
    ok = ok && cudaMalloc(&s->agg16, s->agg16_bytes) == cudaSuccess;
    if (!ok) { cudaGetLastError(); osb200_destroy(s); return OSB200_ERR_ALLOC; }
    e = cudaMemset(s->desc, 0, s->desc_tiles * osb::kRadix * sizeof(uint64_t));  // epoch 0 == never valid
    if (e == cudaSuccess) e = cudaMemset(s->control, 0, ControlLayout::total);

    // Verify on THIS device the hardware property the atomic ranking depends on; otherwise use ballots.
    if (e == cudaSuccess) e = osb::launch_atomic_order_selftest(s->err(), s->sm_count, nullptr);
    unsigned long long mism = 1;
    if (e == cudaSuccess) e = cudaMemcpy(&mism, s->err(), sizeof(mism), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) { osb200_destroy(s); return cuda_status(e); }
    s->atomic_order_ok = (mism == 0);
    s->cfg.rank_mode = s->atomic_order_ok ? osb::kRankAtomic : osb::kRankBallot;
    *out = s;
    return OSB200_OK;
}

}  // namespace

extern "C" {

int osb200_create(osb200_handle* out, uint64_t max_n, int key_bytes, int value_bytes)
{
    if (!out) return OSB200_ERR_INVALID_ARG;
    *out = nullptr;
    if ((key_bytes != 4 && key_bytes != 8) || (value_bytes != 0 && value_bytes != 4)) return OSB200_ERR_INVALID_ARG;
    if (key_bytes == 8 && value_bytes != 0) return OSB200_ERR_UNSUPPORTED;  // osb200_create_pairs64 makes that shape
    return create_impl(out, max_n, key_bytes, value_bytes);
}

int osb200_create_pairs64(osb200_handle* out, uint64_t max_n)
{
    if (!out) return OSB200_ERR_INVALID_ARG;
    *out = nullptr;
    return create_impl(out, max_n, 8, 4);
}

int osb200_destroy(osb200_handle h)
{
    if (!h) return OSB200_ERR_INVALID_ARG;
    cudaFree(h->alt_keys);
    cudaFree(h->alt_vals);
    cudaFree(h->control);
    cudaFree(h->desc);
    cudaFree(h->agg16);
    cudaFree(h->stage_keys);
    cudaFree(h->stage_vals);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    for (cudaEvent_t e : h->ev) if (e) cudaEventDestroy(e);
    delete h;
    return OSB200_OK;
}

int osb200_sort_keys_u32(osb200_handle h, uint32_t* d_keys, uint64_t n, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4) return OSB200_ERR_INVALID_ARG;
    return sort_impl(h, h->key_bytes, d_keys, nullptr, n, static_cast<cudaStream_t>(stream));  // a pairs-capable sorter may sort keys only
}

int osb200_sort_pairs_u32(osb200_handle h, uint32_t* d_keys, uint32_t* d_values, uint64_t n, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4 || h->value_bytes != 4) return OSB200_ERR_INVALID_ARG;
    if (n > 1 && !d_values) return OSB200_ERR_INVALID_ARG;
    return sort_impl(h, h->key_bytes, d_keys, d_values, n, static_cast<cudaStream_t>(stream));
}

int osb200_sort_keys_u64(osb200_handle h, uint64_t* d_keys, uint64_t n, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 8) return OSB200_ERR_INVALID_ARG;
    return sort_impl(h, h->key_bytes, d_keys, nullptr, n, static_cast<cudaStream_t>(stream));
}

// Typed keys (SURVEY 8f rank 1).  The codec of key_type for keys of key_bytes: 2 (osb200_key16_type, on a 4-byte handle
// the same driver with a key width of 2 -- two digit passes; F16 and BF16 share the float codec, sign bit 15, and differ
// only in the dtype the caller keeps them in), 4 or 8 (osb200_key_type of that width).  A type of another width, or
// another key_bytes: INVALID_ARG.  *codec is c with `flags`, or null for plain unsigned ascending keys, which the kernels
// sort as they are.
static int codec_for(int key_bytes, int key_type, int descending, uint32_t flags, osb::KeyCodec* c, const osb::KeyCodec** codec)
{
    const bool wide64 = key_bytes == 8;
    const unsigned long long all = wide64 ? ~0ull : key_bytes == 4 ? 0xffffffffull : 0xffffull, sign = all ^ (all >> 1);
    if (key_bytes == 2) {
        switch (key_type) {
            case OSB200_KEY16_U16: c->a = 0; c->b = 0; break;
            case OSB200_KEY16_I16: c->a = 0; c->b = sign; break;
            case OSB200_KEY16_F16:
            case OSB200_KEY16_BF16: c->a = all; c->b = sign; break;
            default: return OSB200_ERR_INVALID_ARG;
        }
    } else if (key_bytes == 4 || key_bytes == 8) {
        switch (key_type) {
            case OSB200_KEY_U32: case OSB200_KEY_U64: c->a = 0; c->b = 0; break;
            case OSB200_KEY_I32: case OSB200_KEY_I64: c->a = 0; c->b = sign; break;
            case OSB200_KEY_F32: case OSB200_KEY_F64: c->a = all; c->b = sign; break;
            default: return OSB200_ERR_INVALID_ARG;
        }
        if ((key_type >= OSB200_KEY_U64) != wide64) return OSB200_ERR_INVALID_ARG;  // a type of the other width
    } else {
        return OSB200_ERR_INVALID_ARG;
    }
    c->d = descending ? all : 0;
    c->flags = flags;
    *codec = c->a == 0 && c->b == 0 && c->d == 0 ? nullptr : c;
    return OSB200_OK;
}

// What every typed sort and argsort checks once the handle's shape is accepted: the key type (a type of another width:
// INVALID_ARG), then the variant (typed keys and the indices mode live in the default pass's device plan).
static int typed_codec(const osb200_sorter* h, int key_bytes, int key_type, int descending, osb::KeyCodec* c, const osb::KeyCodec** codec)
{
    const int st = codec_for(key_bytes, key_type, descending, 0u, c, codec);
    if (st != OSB200_OK) return st;
    return h->cfg.variant == osb::kVariantWide ? OSB200_OK : OSB200_ERR_UNSUPPORTED;
}

// The typed keys and pairs sorts once the handle's shape is accepted; pairs: d_vals may be null only when n <= 1.
static int typed_sort(osb200_sorter* h, int key_bytes, void* d_keys, uint32_t* d_vals, bool pairs, uint64_t n, int key_type,
                      int descending, void* stream)
{
    osb::KeyCodec c;
    const osb::KeyCodec* codec = nullptr;
    const int st = typed_codec(h, key_bytes, key_type, descending, &c, &codec);
    if (st != OSB200_OK) return st;
    if (pairs && n > 1 && !d_vals) return OSB200_ERR_INVALID_ARG;
    return sort_impl(h, key_bytes, d_keys, d_vals, n, static_cast<cudaStream_t>(stream), codec);
}

// The argsorts once the handle's shape is accepted: keys of key_bytes (the handle's, or 2), 32-bit indices.
static int argsort_impl(osb200_sorter* h, int key_bytes, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                        int key_type, int descending, void* stream)
{
    osb::KeyCodec c;
    const osb::KeyCodec* codec = nullptr;
    const int st = typed_codec(h, key_bytes, key_type, descending, &c, &codec);
    if (st != OSB200_OK) return st;
    if (n == 0) return OSB200_OK;
    const uintptr_t in = reinterpret_cast<uintptr_t>(d_keys_in), out = reinterpret_cast<uintptr_t>(d_keys_out),
                    idx = reinterpret_cast<uintptr_t>(d_indices);
    if (!in || !out || !idx || ((in | out | idx) & 15u)) return OSB200_ERR_INVALID_ARG;
    if (n > h->max_n || n > (1ull << 32)) return OSB200_ERR_SIZE;  // the indices are 32-bit
    // the input is read until the last pass; outputs that overlap it (or each other) would overwrite keys still to be read
    // (the key arrays are key_bytes * n bytes, the index array 4n)
    const uint64_t kb = n * static_cast<uint64_t>(key_bytes), ib = n * sizeof(uint32_t);
    if (overlaps(in, kb, out, kb) || overlaps(in, kb, idx, ib) || overlaps(out, kb, idx, ib)) return OSB200_ERR_INVALID_ARG;
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    if (n == 1) {  // already sorted, but the outputs still have to be written
        OSB_TRY(cudaMemcpyAsync(d_keys_out, d_keys_in, key_bytes, cudaMemcpyDeviceToDevice, q));
        OSB_TRY(cudaMemsetAsync(d_indices, 0, sizeof(uint32_t), q));
        return OSB200_OK;
    }
    return sort_impl(h, key_bytes, d_keys_out, d_indices, n, q, codec, 0, -1, d_keys_in);
}

int osb200_sort_keys_typed(osb200_handle h, void* d_keys, uint64_t n, int key_type, int descending, void* stream)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    return typed_sort(h, h->key_bytes, d_keys, nullptr, false, n, key_type, descending, stream);
}

int osb200_segmented_sort_u32(osb200_handle h, uint32_t* d_keys, uint32_t* d_values, const uint64_t* d_segment_offsets,
                              uint64_t num_segments, uint32_t max_segment_len, void* stream)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    if (h->key_bytes != 4 || (d_values && h->value_bytes != 4)) return OSB200_ERR_INVALID_ARG;
    if (num_segments == 0 || max_segment_len <= 1) return OSB200_OK;
    if (!d_keys || !d_segment_offsets) return OSB200_ERR_INVALID_ARG;
    if (max_segment_len > osb::segment_sort_capacity(4)) return OSB200_ERR_SIZE;  // sort longer segments with osb200_sort_*
    OSB_TRY(osb::launch_segment_sort(d_keys, d_values, 4, reinterpret_cast<const unsigned long long*>(d_segment_offsets), num_segments,
                                     0, max_segment_len, 0, 4, 8, nullptr, h->cfg.rank_mode, h->sm_count,
                                     static_cast<cudaStream_t>(stream)));
    return OSB200_OK;
}

int osb200_sort_bits(osb200_handle h, void* d_keys, uint32_t* d_values, uint64_t n, int begin_bit, int end_bit, void* stream)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    if (d_values && (h->key_bytes != 4 || h->value_bytes != 4)) return OSB200_ERR_INVALID_ARG;
    return sort_impl(h, h->key_bytes, d_keys, d_values, n, static_cast<cudaStream_t>(stream), nullptr, begin_bit, end_bit);
}

// Pairs and argsort take a (4, 4) handle with 32-bit key types or a (8, 4) handle (osb200_create_pairs64) with 64-bit ones.
int osb200_sort_pairs_typed(osb200_handle h, void* d_keys, uint32_t* d_values, uint64_t n, int key_type, int descending,
                            void* stream)
{
    if (check_handle(h) != OSB200_OK || h->value_bytes != 4) return OSB200_ERR_INVALID_ARG;
    if (n > 1 && !d_values) return OSB200_ERR_INVALID_ARG;  // before the key type, unlike osb200_sort_pairs16
    return typed_sort(h, h->key_bytes, d_keys, d_values, true, n, key_type, descending, stream);
}

int osb200_argsort(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n, int key_type,
                   int descending, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->value_bytes != 4) return OSB200_ERR_INVALID_ARG;
    return argsort_impl(h, h->key_bytes, d_keys_in, d_keys_out, d_indices, n, key_type, descending, stream);
}

int osb200_sort_keys16(osb200_handle h, void* d_keys, uint64_t n, int key_type, int descending, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4) return OSB200_ERR_INVALID_ARG;
    return typed_sort(h, 2, d_keys, nullptr, false, n, key_type, descending, stream);
}

int osb200_sort_pairs16(osb200_handle h, void* d_keys, uint32_t* d_values, uint64_t n, int key_type, int descending, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4 || h->value_bytes != 4) return OSB200_ERR_INVALID_ARG;
    return typed_sort(h, 2, d_keys, d_values, true, n, key_type, descending, stream);
}

int osb200_argsort16(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n, int key_type,
                     int descending, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4 || h->value_bytes != 4) return OSB200_ERR_INVALID_ARG;
    return argsort_impl(h, 2, d_keys_in, d_keys_out, d_indices, n, key_type, descending, stream);
}

// The row and segment sorts and top-k take 2-, 4- or 8-byte keys of any handle; their kernels encode every key they load and
// decode every key they store.
static constexpr uint32_t kRaggedCodecFlags = osb::kCodecEncodeOnLoad | osb::kCodecDecodeOnStore;

// The row sorts.  Rows of at most row_sort_capacity keys: one launch of osb::launch_row_sort, no workspace -- only the handle's
// device, rank mode and SM count are used, so any handle will do.  long_rows (osb200_sort_long_rows): longer rows, and with the
// test hook debug_long_rows every row of two or more keys, take the long path on the handle's alternate buffers, control
// block and reductions (agg16: the tile counts and chunk sums, which every other call clears or overwrites before reading).
static int sort_rows_impl(osb200_sorter* h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t num_rows,
                          uint32_t row_len, int key_bytes, int key_type, int descending, void* stream, bool long_rows)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    osb::KeyCodec c;
    const osb::KeyCodec* codec = nullptr;
    int st = codec_for(key_bytes, key_type, descending, kRaggedCodecFlags, &c, &codec);
    if (st != OSB200_OK) return st;
    if (num_rows == 0 || row_len == 0) return OSB200_OK;
    const uint64_t n = num_rows * row_len, kb = n * static_cast<uint64_t>(key_bytes), ib = n * sizeof(uint32_t);
    const ArrayArg arrays[] = {{d_keys_in, kb, key_bytes, true, false}, {d_keys_out, kb, key_bytes, true, true},
                               {d_indices, ib, 4, false, true}};
    st = check_arrays(arrays, num_rows <= UINT64_MAX / row_len && n <= UINT64_MAX / 8, true);
    if (st != OSB200_OK) return st;
    const bool fits = row_len <= osb::row_sort_capacity(key_bytes);
    if (!long_rows && !fits) return OSB200_ERR_SIZE;
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    if (row_len == 1) {  // every row is sorted already
        if (d_keys_in != d_keys_out) OSB_TRY(cudaMemcpyAsync(d_keys_out, d_keys_in, kb, cudaMemcpyDeviceToDevice, q));
        if (d_indices) OSB_TRY(cudaMemsetAsync(d_indices, 0, ib, q));
        return OSB200_OK;
    }
    if (!long_rows || (fits && !h->debug_long_rows)) {
        OSB_TRY(osb::launch_row_sort(d_keys_in, d_keys_out, d_indices, num_rows, row_len, key_bytes, codec,
                                     h->cfg.rank_mode, h->debug_rows_block, h->sm_count, q));
        return OSB200_OK;
    }
    // the long path's workspace: alternate keys at least as wide as the row's, payloads for the indices, n <= max_n, and the
    // tile counts and chunk sums inside the reductions
    if (h->key_bytes < key_bytes || (d_indices && h->value_bytes != 4)) return OSB200_ERR_INVALID_ARG;
    if (n > h->max_n || osb::long_rows_scratch_bytes(num_rows, row_len) > h->agg16_bytes) return OSB200_ERR_SIZE;
    OSB_TRY(cudaMemsetAsync(h->control, 0, ControlLayout::zeroed_bytes, q));
    OSB_TRY(osb::launch_long_rows(d_keys_in, d_keys_out, d_indices, h->alt_keys, d_indices ? h->alt_vals : nullptr, num_rows, row_len,
                                  key_bytes, codec, h->cfg.rank_mode, h->short_circuit, h->ghist(), h->gbase(), h->plan(),
                                  reinterpret_cast<uint32_t*>(h->agg16), h->sm_count, q));
    return OSB200_OK;
}

int osb200_sort_rows(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t num_rows,
                     uint32_t row_len, int key_bytes, int key_type, int descending, void* stream)
{
    return sort_rows_impl(h, d_keys_in, d_keys_out, d_indices, num_rows, row_len, key_bytes, key_type, descending, stream, false);
}

int osb200_sort_long_rows(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t num_rows,
                          uint32_t row_len, int key_bytes, int key_type, int descending, void* stream)
{
    return sort_rows_impl(h, d_keys_in, d_keys_out, d_indices, num_rows, row_len, key_bytes, key_type, descending, stream, true);
}

// The segment sorts.  Segments of at most row_sort_capacity keys: the row sort's kernels for ragged rows, with the workspace
// of check_segment_workspace.  long_segments (osb200_sort_long_segments) with a larger max_segment_len, or with the test hook
// debug_long_rows: segments longer than row_sort_capacity (with the hook, every segment of two or more keys) take the long
// path, with the long rows' handle rules: the alternate buffers, the control block's scratch words and the reductions
// (agg16: the tile counts, chunk sums and tile map, which every other call clears or overwrites before reading).  The room
// the long path needs is bounded by n and the shortest long segment only (long_segments_layout), never by the offsets.
static int sort_segments_impl(osb200_sorter* h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                              const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t max_segment_len, int key_bytes,
                              int key_type, int descending, void* stream, bool long_segments)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    osb::KeyCodec c;
    const osb::KeyCodec* codec = nullptr;
    int st = codec_for(key_bytes, key_type, descending, kRaggedCodecFlags, &c, &codec);
    if (st != OSB200_OK) return st;
    if (n == 0 || num_segments == 0 || max_segment_len == 0) return OSB200_OK;
    const uint64_t kb = n * static_cast<uint64_t>(key_bytes), ib = n * sizeof(uint32_t), ob = (num_segments + 1) * sizeof(uint64_t);
    // the offsets are read by every kernel of the call
    const ArrayArg arrays[] = {{d_keys_in, kb, key_bytes, true, false}, {d_keys_out, kb, key_bytes, true, true},
                               {d_indices, ib, 4, false, true}, {d_segment_offsets, ob, 8, true, false}};
    st = check_arrays(arrays, n <= UINT64_MAX / 8 && num_segments <= UINT64_MAX / 8 - 1, true);
    if (st != OSB200_OK) return st;
    const uint32_t cap = osb::row_sort_capacity(key_bytes);
    if (!long_segments && max_segment_len > cap) return OSB200_ERR_SIZE;
    if ((st = check_segment_workspace(h, num_segments)) != OSB200_OK) return st;
    const auto* off = reinterpret_cast<const unsigned long long*>(d_segment_offsets);
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    const uint32_t long_min = h->debug_long_rows ? 2u : cap + 1;
    if (!long_segments || max_segment_len < long_min) {
        OSB_TRY(osb::launch_sort_segments(d_keys_in, d_keys_out, d_indices, n, off, num_segments, max_segment_len, key_bytes, codec,
                                          h->cfg.rank_mode, h->sm_count, static_cast<uint32_t*>(h->alt_keys), h->err(), q));
        return OSB200_OK;
    }
    static_assert(ControlLayout::err_bytes >= 7 * sizeof(unsigned long long), "the long path's counts live in the scratch words");
    if (h->key_bytes < key_bytes || (d_indices && h->value_bytes != 4)) return OSB200_ERR_INVALID_ARG;
    const osb::LongSegLayout l = osb::long_segments_layout(n, long_min);
    if (n > h->max_n || l.words * sizeof(uint32_t) > h->agg16_bytes || l.tile_cap > UINT32_MAX || l.chunk_cap > UINT32_MAX)
        return OSB200_ERR_SIZE;
    OSB_TRY(cudaMemsetAsync(h->control, 0, ControlLayout::zeroed_bytes, q));
    OSB_TRY(osb::launch_long_segments(d_keys_in, d_keys_out, d_indices, h->alt_keys, d_indices ? h->alt_vals : nullptr, n, off,
                                      num_segments, max_segment_len, long_min, key_bytes, codec, h->cfg.rank_mode, h->short_circuit,
                                      h->ghist(), h->gbase(), h->plan(), static_cast<uint32_t*>(h->alt_keys), h->err(),
                                      reinterpret_cast<uint32_t*>(h->agg16), h->sm_count, q));
    return OSB200_OK;
}

int osb200_sort_segments(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                         const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t max_segment_len, int key_bytes,
                         int key_type, int descending, void* stream)
{
    return sort_segments_impl(h, d_keys_in, d_keys_out, d_indices, n, d_segment_offsets, num_segments, max_segment_len, key_bytes,
                              key_type, descending, stream, false);
}

int osb200_sort_long_segments(osb200_handle h, const void* d_keys_in, void* d_keys_out, uint32_t* d_indices, uint64_t n,
                              const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t max_segment_len, int key_bytes,
                              int key_type, int descending, void* stream)
{
    return sort_segments_impl(h, d_keys_in, d_keys_out, d_indices, n, d_segment_offsets, num_segments, max_segment_len, key_bytes,
                              key_type, descending, stream, true);
}

// Row top-k: at most two launches, no workspace -- like the row sort, any handle will do.
int osb200_topk_rows(osb200_handle h, const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t num_rows,
                     uint32_t row_len, uint32_t k, int key_bytes, int key_type, int largest, int sorted, void* stream)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    osb::KeyCodec c;
    const osb::KeyCodec* codec = nullptr;
    int st = codec_for(key_bytes, key_type, largest, kRaggedCodecFlags, &c, &codec);
    if (st != OSB200_OK) return st;
    if (num_rows == 0 || row_len == 0 || k == 0) return OSB200_OK;
    if (k > row_len) return OSB200_ERR_INVALID_ARG;
    // (the outputs are smaller than the input: k <= row_len)
    const uint64_t n = num_rows * row_len, m = num_rows * k;
    const uint64_t kb = n * static_cast<uint64_t>(key_bytes), ob = m * static_cast<uint64_t>(key_bytes), ib = m * sizeof(uint32_t);
    // the outputs have another shape than the input: no in-place form
    const ArrayArg arrays[] = {{d_keys_in, kb, key_bytes, true, false}, {d_values_out, ob, key_bytes, true, true},
                               {d_indices, ib, 4, true, true}};
    st = check_arrays(arrays, num_rows <= UINT64_MAX / row_len && n <= UINT64_MAX / 8, false);
    if (st != OSB200_OK) return st;
    if (k > osb::row_sort_capacity(key_bytes)) return OSB200_ERR_SIZE;
    OSB_TRY(osb::launch_topk_rows(d_keys_in, d_values_out, d_indices, num_rows, row_len, k, key_bytes, codec, sorted != 0,
                                  h->debug_topk_capacity, h->cfg.rank_mode, h->debug_rows_block, h->sm_count,
                                  static_cast<cudaStream_t>(stream)));
    return OSB200_OK;
}

// Segment top-k: row top-k for ragged segments, with the workspace of check_segment_workspace.
int osb200_topk_segments(osb200_handle h, const void* d_keys_in, void* d_values_out, uint32_t* d_indices, uint64_t n,
                         const uint64_t* d_segment_offsets, uint64_t num_segments, uint32_t k, int key_bytes, int key_type,
                         int largest, int sorted, void* stream)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    osb::KeyCodec c;
    const osb::KeyCodec* codec = nullptr;
    int st = codec_for(key_bytes, key_type, largest, kRaggedCodecFlags, &c, &codec);
    if (st != OSB200_OK) return st;
    // (n == 0 is not a no-op: every row is then padding)
    if (num_segments == 0 || k == 0) return OSB200_OK;
    const uint64_t m = num_segments * k;
    const uint64_t kb = n * static_cast<uint64_t>(key_bytes), ob = m * static_cast<uint64_t>(key_bytes), ib = m * sizeof(uint32_t),
                   fb = (num_segments + 1) * sizeof(uint64_t);
    // the outputs have another shape than the input: no in-place form
    const ArrayArg arrays[] = {{d_keys_in, kb, key_bytes, n != 0, false}, {d_values_out, ob, key_bytes, true, true},
                               {d_indices, ib, 4, true, true}, {d_segment_offsets, fb, 8, true, false}};
    st = check_arrays(arrays, n <= UINT64_MAX / 8 && num_segments <= UINT64_MAX / 8 - 1 && num_segments <= UINT64_MAX / 8 / k, false);
    if (st != OSB200_OK) return st;
    // unlike osb200_sort_segments, input keys that overlap the offsets are refused too, though the call only reads both
    if (overlaps(reinterpret_cast<uintptr_t>(d_keys_in), kb, reinterpret_cast<uintptr_t>(d_segment_offsets), fb))
        return OSB200_ERR_INVALID_ARG;
    if (k > osb::row_sort_capacity(key_bytes)) return OSB200_ERR_SIZE;
    if ((st = check_segment_workspace(h, num_segments)) != OSB200_OK) return st;
    OSB_TRY(osb::launch_topk_segments(d_keys_in, d_values_out, d_indices, n, reinterpret_cast<const unsigned long long*>(d_segment_offsets),
                                      num_segments, k, key_bytes, codec, sorted != 0, h->debug_topk_capacity, h->cfg.rank_mode,
                                      h->debug_rows_block, h->sm_count, static_cast<uint32_t*>(h->alt_keys), h->err(),
                                      static_cast<cudaStream_t>(stream)));
    return OSB200_OK;
}

int osb200_sort_host_keys_u32(osb200_handle h, uint32_t* h_keys, uint64_t n)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4) return OSB200_ERR_INVALID_ARG;
    return sort_host_impl(h, h_keys, nullptr, n);
}

int osb200_sort_host_pairs_u32(osb200_handle h, uint32_t* h_keys, uint32_t* h_values, uint64_t n)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4 || h->value_bytes != 4) return OSB200_ERR_INVALID_ARG;
    if (n > 1 && !h_values) return OSB200_ERR_INVALID_ARG;
    return sort_host_impl(h, h_keys, h_values, n);
}

int osb200_sort_host_keys_u64(osb200_handle h, uint64_t* h_keys, uint64_t n)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 8) return OSB200_ERR_INVALID_ARG;
    return sort_host_impl(h, h_keys, nullptr, n);
}

int osb200_global_histogram(osb200_handle h, const void* d_keys, uint64_t n, uint64_t* d_hist, void* stream)
{
    if (check_handle(h) != OSB200_OK || !d_hist || (n && !d_keys)) return OSB200_ERR_INVALID_ARG;
    if (reinterpret_cast<uintptr_t>(d_keys) & 15u) return OSB200_ERR_INVALID_ARG;
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    OSB_TRY(cudaMemsetAsync(d_hist, 0, static_cast<size_t>(h->key_bytes) * osb::kRadix * sizeof(uint64_t), q));
    if (n == 0) return OSB200_OK;
    OSB_TRY(osb::launch_global_histogram(d_keys, n, h->key_bytes, reinterpret_cast<unsigned long long*>(d_hist),
                                         h->sm_count, q));
    return OSB200_OK;
}

int osb200_digit_binning_pass(osb200_handle h, const void* d_in, void* d_out, const uint32_t* d_in_values,
                              uint32_t* d_out_values, uint64_t n, uint32_t radix_shift, void* stream)
{
    if (check_handle(h) != OSB200_OK) return OSB200_ERR_INVALID_ARG;
    if (n == 0) return OSB200_OK;
    if (!d_in || !d_out || d_in == d_out) return OSB200_ERR_INVALID_ARG;
    if ((reinterpret_cast<uintptr_t>(d_in) & 15u) || (reinterpret_cast<uintptr_t>(d_out) & 15u)) return OSB200_ERR_INVALID_ARG;
    if (n > h->max_n) return OSB200_ERR_SIZE;
    if (radix_shift >= static_cast<uint32_t>(h->key_bytes) * 8u) return OSB200_ERR_INVALID_ARG;
    if ((d_in_values != nullptr) != (d_out_values != nullptr)) return OSB200_ERR_INVALID_ARG;
    if (d_in_values && (h->key_bytes != 4 || h->value_bytes != 4)) return OSB200_ERR_UNSUPPORTED;
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    bool capturing = false;
    int st = is_capturing(q, &capturing);
    if (st != OSB200_OK) return st;
    const size_t desc_bytes = tiles_for(n, osb::binning_tile_keys(h->key_bytes, d_in_values != nullptr, h->cfg)) * osb::kRadix *
                              sizeof(uint64_t);
    if (capturing) OSB_TRY(cudaMemsetAsync(h->desc, 0, desc_bytes, q));
    // histogram of this digit only, then the pass (the reference's multiples of 8 and any other shift alike)
    st = osb_internal_digit_histogram(h, d_in, n, radix_shift, h->ghist(), q);
    if (st != OSB200_OK) return st;
    OSB_TRY(cudaMemsetAsync(h->tickets(), 0, ControlLayout::ticket_bytes, q));
    OSB_TRY(osb::launch_scan(h->ghist(), h->gbase(), 1, q));
    if (h->cfg.variant != osb::kVariantTilePerCta)
        OSB_TRY(cudaMemsetAsync(h->agg16, 0, (h->desc_tiles + 8) * osb::kRadix * sizeof(uint16_t), q));
    uint32_t epoch = 0;
    st = next_epoch(h, q, &epoch);
    if (st != OSB200_OK) return st;
    osb::BinningConfig cfg = h->cfg;
    const uint32_t key_bits = static_cast<uint32_t>(h->key_bytes) * 8u;
    cfg.digit_bits = key_bits - radix_shift < 8u ? key_bits - radix_shift : 8u;
    OSB_TRY(osb::launch_digit_binning(d_in, d_out, d_in_values, d_out_values, n, h->key_bytes, radix_shift, h->gbase(), h->desc,
                                      h->agg16, h->tickets(), epoch, cfg, q));
    if (capturing) OSB_TRY(cudaMemsetAsync(h->desc, 0, desc_bytes, q));
    return OSB200_OK;
}

// Testing hooks: the two kernels of the sharded sort's exchange, on an ordinary handle (the sharded sort calls the internal
// functions directly; nothing here is on a sort path).
int osb200_debug_digit_histogram(osb200_handle h, const uint32_t* d_in, uint64_t n, uint32_t shift, uint64_t* d_hist256,
                                 void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4 || !d_hist256 || shift >= 32) return OSB200_ERR_INVALID_ARG;
    if (n && (!d_in || (reinterpret_cast<uintptr_t>(d_in) & 15u))) return OSB200_ERR_INVALID_ARG;
    if (n > h->max_n) return OSB200_ERR_SIZE;
    return osb_internal_digit_histogram(h, d_in, n, shift, reinterpret_cast<unsigned long long*>(d_hist256),
                                        static_cast<cudaStream_t>(stream));
}

int osb200_debug_exchange_pass(osb200_handle h, const uint32_t* d_in, uint32_t* d_out, uint64_t n, uint32_t shift,
                               const uint64_t* d_hist256, const uint64_t* d_out_base, void* stream)
{
    if (check_handle(h) != OSB200_OK || h->key_bytes != 4 || shift >= 32) return OSB200_ERR_INVALID_ARG;
    // fused: the bases are absolute (virtual element indices), so there is no output pointer
    if (d_out_base && d_out) return OSB200_ERR_INVALID_ARG;
    if (n == 0) return OSB200_OK;
    if (!d_in || (reinterpret_cast<uintptr_t>(d_in) & 15u) || d_in == d_out) return OSB200_ERR_INVALID_ARG;
    // staged: an output and the histogram the pass scans
    if (!d_out_base && (!d_out || !d_hist256 || (reinterpret_cast<uintptr_t>(d_out) & 3u))) return OSB200_ERR_INVALID_ARG;
    if (n > h->max_n) return OSB200_ERR_SIZE;
    return osb_internal_binning_pass(h, d_in, d_out, n, shift, reinterpret_cast<const unsigned long long*>(d_hist256),
                                     reinterpret_cast<const unsigned long long*>(d_out_base), static_cast<cudaStream_t>(stream));
}

int osb200_validate(osb200_handle h, const void* d_keys, uint64_t n, uint64_t* h_err_count, void* stream)
{
    if (check_handle(h) != OSB200_OK || !h_err_count) return OSB200_ERR_INVALID_ARG;
    *h_err_count = 0;
    if (n < 2) return OSB200_OK;
    if (!d_keys) return OSB200_ERR_INVALID_ARG;
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    OSB_TRY(cudaMemsetAsync(h->err(), 0, sizeof(unsigned long long), q));
    OSB_TRY(osb::launch_validate(d_keys, n, h->key_bytes, h->err(), h->sm_count, q));
    unsigned long long v = 0;
    OSB_TRY(cudaMemcpyAsync(&v, h->err(), sizeof(v), cudaMemcpyDeviceToHost, q));
    OSB_TRY(cudaStreamSynchronize(q));
    *h_err_count = v;
    return OSB200_OK;
}

int osb200_init_random_u32(uint32_t* d_keys, uint32_t* d_payload, uint64_t n, uint32_t and_count, uint32_t seed,
                           int payload_is_index, void* stream)
{
    if (n == 0) return OSB200_OK;
    if (!d_keys) return OSB200_ERR_INVALID_ARG;
    OSB_TRY(osb::launch_init_random(d_keys, d_payload, n, and_count, seed, payload_is_index != 0,
                                    static_cast<cudaStream_t>(stream)));
    return OSB200_OK;
}

int osb200_set_option(osb200_handle h, const char* key, int64_t value)
{
    if (check_handle(h) != OSB200_OK || !key) return OSB200_ERR_INVALID_ARG;
    if (!std::strcmp(key, "rank_mode")) {
        if (value != osb::kRankAtomic && value != osb::kRankBallot) return OSB200_ERR_INVALID_ARG;
        if (value == osb::kRankAtomic && !h->atomic_order_ok) return OSB200_ERR_UNSUPPORTED;
        h->cfg.rank_mode = static_cast<int>(value);
        return OSB200_OK;
    }
    if (!std::strcmp(key, "profile")) { h->profile = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "short_circuit")) { h->short_circuit = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "small_path")) { h->small_path = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "hot_passes")) { h->hot_passes = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "fused_histogram")) { h->fused_histogram = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "spin_cap")) {
        if (value < 1 || value > (1ll << 30)) return OSB200_ERR_INVALID_ARG;
        h->cfg.spin_cap = static_cast<uint32_t>(value);
        return OSB200_OK;
    }
    if (!std::strcmp(key, "debug_stall_every")) {  // test hook of the forward-progress fallback (0 = off)
        if (value < 0 || value > (1ll << 30)) return OSB200_ERR_INVALID_ARG;
        h->cfg.debug_stall_every = static_cast<uint32_t>(value);
        return OSB200_OK;
    }
    if (!std::strcmp(key, "debug_max_ctas")) {  // test hook of the persistent pass's tile schedule (0 = off)
        if (value < 0 || value > (1ll << 30)) return OSB200_ERR_INVALID_ARG;
        h->cfg.debug_max_ctas = static_cast<uint32_t>(value);
        return OSB200_OK;
    }
    if (!std::strcmp(key, "debug_rows_block")) { h->debug_rows_block = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "debug_long_rows")) { h->debug_long_rows = value != 0; return OSB200_OK; }
    if (!std::strcmp(key, "debug_topk_capacity")) {  // test hook of osb200_topk_rows' shared-memory candidates (0 = off)
        if (value < 0 || value > (1ll << 30)) return OSB200_ERR_INVALID_ARG;
        h->debug_topk_capacity = static_cast<uint32_t>(value);
        return OSB200_OK;
    }
    if (!std::strcmp(key, "debug_epoch")) {  // test hook: the epoch counter, to reach the wrap-around or reuse epochs
        if (value < 0 || value > osb::kEpochMax) return OSB200_ERR_INVALID_ARG;
        h->epoch = static_cast<uint32_t>(value);
        return OSB200_OK;
    }
    if (!std::strcmp(key, "variant")) {
        if (value < 0 || value >= osb::kNumVariants) return OSB200_ERR_INVALID_ARG;
        h->cfg.variant = static_cast<int>(value);
        return OSB200_OK;
    }
    return OSB200_ERR_INVALID_ARG;
}

int osb200_get_profile(osb200_handle h, float* out_ms, int capacity)
{
    if (check_handle(h) != OSB200_OK || !out_ms) return OSB200_ERR_INVALID_ARG;
    if (h->ev_count < 2) return 0;
    OSB_TRY(cudaEventSynchronize(h->ev[h->ev_count - 1]));
    int k = 0;
    for (int i = 0; i < h->span_count; ++i) {
        const osb200_sorter::Span& sp = h->spans[i];
        if (sp.entry >= capacity) continue;
        for (; k <= sp.entry; ++k) out_ms[k] = 0.0f;
        float ms = 0.0f;
        OSB_TRY(cudaEventElapsedTime(&ms, h->ev[sp.from], h->ev[sp.to]));
        out_ms[sp.entry] += ms;
    }
    return k;
}

int64_t osb200_get_info(osb200_handle h, const char* key)
{
    if (check_handle(h) != OSB200_OK || !key) return OSB200_ERR_INVALID_ARG;
    if (!std::strcmp(key, "tile_keys")) return osb::binning_tile_keys(h->key_bytes, h->value_bytes != 0, h->cfg);
    if (!std::strcmp(key, "launches_per_sort")) {  // histogram + scan + one pass per place (+ copy-back: keys [+ values])
        const bool wide = h->cfg.variant == osb::kVariantWide;
        const bool cb = wide && h->short_circuit;
        return 2 + h->key_bytes * ((wide && h->hot_passes) ? 2 : 1) + (cb ? (h->value_bytes ? 2 : 1) : 0);
    }
    if (!std::strcmp(key, "memsets_per_sort")) return h->cfg.variant != osb::kVariantTilePerCta ? 2 : 1;
    if (!std::strcmp(key, "short_circuit")) return h->short_circuit ? 1 : 0;
    if (!std::strcmp(key, "small_path")) return h->small_path ? 1 : 0;
    if (!std::strcmp(key, "hot_passes")) return h->hot_passes ? 1 : 0;
    if (!std::strcmp(key, "fused_histogram")) return h->fused_histogram ? 1 : 0;
    if (!std::strcmp(key, "last_fused_kept")) {  // 1: the last sort's fused first pass stood (0 also for a sort that was not fused)
        osb::SortPlan pl;
        if (cudaMemcpy(&pl, h->plan(), sizeof(pl), cudaMemcpyDeviceToHost) != cudaSuccess) return OSB200_ERR_CUDA;
        return (pl.skip_mask & osb::kPlanFusedKept) ? 1 : 0;
    }
    if (!std::strcmp(key, "last_hot_mask")) {
        osb::SortPlan pl;
        if (cudaMemcpy(&pl, h->plan(), sizeof(pl), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
        return static_cast<int>((pl.skip_mask >> osb::kPlanHotShift) & 0xffu);
    }
    if (!std::strcmp(key, "small_path_max_n")) return osb::segment_sort_capacity(h->key_bytes);
    if (!std::strcmp(key, "spin_cap")) return h->cfg.spin_cap;
    if (!std::strcmp(key, "last_skip_mask") || !std::strcmp(key, "last_executed_passes")) {
        // the plan of the last sort on this handle (synchronises the device: introspection / tests only)
        osb::SortPlan pl;
        if (cudaMemcpy(&pl, h->plan(), sizeof(pl), cudaMemcpyDeviceToHost) != cudaSuccess) return OSB200_ERR_CUDA;
        return key[5] == 's' ? static_cast<int64_t>(pl.skip_mask & 0xffffu) : static_cast<int64_t>(pl.executed);
    }
    if (!std::strcmp(key, "sm_count")) return h->sm_count;
    if (!std::strcmp(key, "rank_mode")) return h->cfg.rank_mode;
    if (!std::strcmp(key, "variant")) return h->cfg.variant;
    if (!std::strcmp(key, "atomic_order_ok")) return h->atomic_order_ok ? 1 : 0;
    if (!std::strcmp(key, "max_n")) return static_cast<int64_t>(h->max_n);
    if (!std::strcmp(key, "epoch")) return h->epoch;
    return OSB200_ERR_INVALID_ARG;
}

}  // extern "C"
