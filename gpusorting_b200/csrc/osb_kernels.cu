// osb_kernels.cu -- hand-written sm_90a kernels of the OneSweep path.
//
// Three kernels per sort, as in the reference (GPUSortingCUDA/Sort/OneSweep.cu), each re-designed for a bandwidth-bound GPU:
//   global_histogram_kernel  <-> OneSweep::GlobalHistogram        (OneSweep.cu:44-123)
//   scan_kernel              <-> OneSweep::Scan                   (OneSweep.cu:125-162)
//   digit_binning_kernel     <-> OneSweep::DigitBinningPassKeysOnly / Pairs (OneSweep.cu:164-344, 346-600)
//
// The design point (see DESIGN.md): at HBM speed a binning pass must retire well over one key per SM clock
// (H100 SXM: 3.35 TB/s over 132 SMs at ~1.7 GHz is ~15 B/clk/SM, ~1.9 keys/clk/SM at 8 B per key and pass), and the
// reference's 8-ballots-per-key warp multisplit spends 8 ballots and their masking on every key.  Ranking is therefore
// done with ONE shared-memory atomicAdd per key on a warp-private histogram: if the returning shared-memory atomic hands
// its values to same-address lanes of a warp instruction in ascending lane order -- checked by a device self-test when a
// sorter is created -- it is a single-instruction stable multisplit.  The ballot formulation is kept as
// RankMode::kRankBallot and is used when the self-test fails.
#include "osb_kernels.cuh"
#include "osb_common.cuh"

namespace osb {

// =====================================================================================================
// GlobalHistogram
//
// One streaming read of the keys, counting all digit places at once (reference: OneSweep.cu:44-123).  At HBM
// bandwidth this kernel needs ~15 shared-memory atomic lanes per SM clock on H100 (~3.8 u32 keys/clk/SM x 4 places), so
// bank conflicts between the lanes of one ATOMS instruction are unaffordable.  The per-CTA histogram is therefore
// laid out [place][digit][column] with column = lane (32 columns for u32 keys, 16 for u64): every lane of a warp
// instruction hits its own bank, whatever the data.  128 KB of shared memory, one 1024-thread CTA per SM.
// =====================================================================================================
constexpr int kHistThreads = 1024;

template <typename KeyT> struct HistGeom;
template <> struct HistGeom<uint32_t> { static constexpr int COLS = 32; };
template <> struct HistGeom<uint64_t> { static constexpr int COLS = 16; };

// MASKED: a sort on the key bits [0, end_bit) -- only the first `places` byte places count and the last of them keeps
// `last_mask` (the sharded path's local sort after an exchange on the top log2(R) bits: bits [0, 32 - log2 R))
template <typename KeyT, bool MASKED = false>
__device__ __forceinline__ void hist_count_word(uint32_t* s_col, uint32_t w, int word_in_vec, int places = 0, uint32_t last_mask = 255u)
{
    constexpr int PLACES = sizeof(KeyT);
    constexpr int COLS = HistGeom<KeyT>::COLS;
    // byte q of 32-bit word `word_in_vec` of a 16-byte vector is digit place ((word*4+q) % PLACES) of some key
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int place = (word_in_vec * 4 + q) % PLACES;
        if constexpr (MASKED) {
            if (place < places)
                atomicAdd(&s_col[(place * kRadix + ((w >> (8 * q)) & (place == places - 1 ? last_mask : 255u))) * COLS], 1u);
        } else {
            atomicAdd(&s_col[(place * kRadix + ((w >> (8 * q)) & 255u)) * COLS], 1u);
        }
    }
}

// typed keys: histogram the ENCODED keys (the passes see them encoded)
template <typename KeyT>
__device__ __forceinline__ uint4 hist_encode_vec(uint4 v, const KeyCodec& c)
{
    if constexpr (sizeof(KeyT) == 4) {
        const uint32_t a = static_cast<uint32_t>(c.a), b = static_cast<uint32_t>(c.b), d = static_cast<uint32_t>(c.d);
        v.x = codec_encode<uint32_t>(v.x, a, b, d); v.y = codec_encode<uint32_t>(v.y, a, b, d);
        v.z = codec_encode<uint32_t>(v.z, a, b, d); v.w = codec_encode<uint32_t>(v.w, a, b, d);
    } else {
        unsigned long long k0 = (static_cast<unsigned long long>(v.y) << 32) | v.x, k1 = (static_cast<unsigned long long>(v.w) << 32) | v.z;
        k0 = codec_encode<unsigned long long>(k0, c.a, c.b, c.d); k1 = codec_encode<unsigned long long>(k1, c.a, c.b, c.d);
        v.x = static_cast<uint32_t>(k0); v.y = static_cast<uint32_t>(k0 >> 32); v.z = static_cast<uint32_t>(k1); v.w = static_cast<uint32_t>(k1 >> 32);
    }
    return v;
}

template <typename KeyT, bool MASKED = false>
__device__ __forceinline__ void hist_count_vec(uint32_t* s_col, const uint4& v, int places = 0, uint32_t last_mask = 255u)
{
    hist_count_word<KeyT, MASKED>(s_col, v.x, 0, places, last_mask);
    hist_count_word<KeyT, MASKED>(s_col, v.y, 1, places, last_mask);
    hist_count_word<KeyT, MASKED>(s_col, v.z, 2, places, last_mask);
    hist_count_word<KeyT, MASKED>(s_col, v.w, 3, places, last_mask);
}

template <typename KeyT, bool MASKED = false>
__global__ void __launch_bounds__(kHistThreads, 1)
global_histogram_kernel(const KeyT* __restrict__ keys, uint64_t n, unsigned long long* __restrict__ ghist, KeyCodec codec,
                        int places = 0, uint32_t last_mask = 255u)
{
    constexpr int PLACES = sizeof(KeyT);
    constexpr int VEC = 16 / sizeof(KeyT);
    constexpr int COLS = HistGeom<KeyT>::COLS;
    constexpr int BINS = PLACES * kRadix;
    extern __shared__ __align__(16) uint32_t s_hist[];  // [BINS][COLS]
    for (int i = threadIdx.x; i < BINS * COLS; i += kHistThreads) s_hist[i] = 0;
    __syncthreads();
    uint32_t* s_col = s_hist + (threadIdx.x & (COLS - 1));  // this lane's private column (bank)

    const uint64_t nvec = n / VEC;
    const uint4* __restrict__ vp = reinterpret_cast<const uint4*>(keys);
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kHistThreads;
    uint64_t i = static_cast<uint64_t>(blockIdx.x) * kHistThreads + threadIdx.x;
    const bool enc = codec.flags & kCodecEncodeOnLoad;
    for (; i + 3 * stride < nvec; i += 4 * stride) {
        uint4 a = __ldcs(vp + i);
        uint4 b = __ldcs(vp + i + stride);
        uint4 c = __ldcs(vp + i + 2 * stride);
        uint4 d = __ldcs(vp + i + 3 * stride);
        if (enc) { a = hist_encode_vec<KeyT>(a, codec); b = hist_encode_vec<KeyT>(b, codec); c = hist_encode_vec<KeyT>(c, codec); d = hist_encode_vec<KeyT>(d, codec); }
        hist_count_vec<KeyT, MASKED>(s_col, a, places, last_mask);
        hist_count_vec<KeyT, MASKED>(s_col, b, places, last_mask);
        hist_count_vec<KeyT, MASKED>(s_col, c, places, last_mask);
        hist_count_vec<KeyT, MASKED>(s_col, d, places, last_mask);
    }
    for (; i < nvec; i += stride) {
        uint4 a = __ldcs(vp + i);
        if (enc) a = hist_encode_vec<KeyT>(a, codec);
        hist_count_vec<KeyT, MASKED>(s_col, a, places, last_mask);
    }
    // ragged tail (n not a multiple of the vector width)
    if (blockIdx.x == 0) {
        const uint64_t t = nvec * VEC + threadIdx.x;
        if (t < n) {
            KeyT k = keys[t];
            if (enc) k = codec_encode<KeyT>(k, static_cast<KeyT>(codec.a), static_cast<KeyT>(codec.b), static_cast<KeyT>(codec.d));
#pragma unroll
            for (int p = 0; p < PLACES; ++p) {
                if (MASKED && p >= places) break;
                const uint32_t m = (MASKED && p == places - 1) ? last_mask : 255u;
                atomicAdd(&s_col[(p * kRadix + (static_cast<uint32_t>(k >> (8 * p)) & m)) * COLS], 1u);
            }
        }
    }
    __syncthreads();
    // fold the columns (rotated start so the 32 lanes of a warp read 32 different banks)
    for (int bin = threadIdx.x; bin < BINS; bin += kHistThreads) {
        uint32_t sum = 0;
#pragma unroll 8
        for (int c = 0; c < COLS; ++c) sum += s_hist[bin * COLS + ((c + threadIdx.x) & (COLS - 1))];
        if (sum) atomicAdd(&ghist[bin], static_cast<unsigned long long>(sum));
    }
}

template <typename KeyT> constexpr size_t hist_smem_bytes() { return sizeof(KeyT) * kRadix * HistGeom<KeyT>::COLS * sizeof(uint32_t); }

cudaError_t launch_global_histogram(const void* keys, uint64_t n, int key_bytes, unsigned long long* ghist,
                                    int sm_count, cudaStream_t stream, const KeyCodec* codec_in)
{
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    const uint64_t vecs = n / (16 / key_bytes);
    uint64_t want = (vecs + kHistThreads - 1) / kHistThreads;
    if (want < 1) want = 1;
    const unsigned grid = static_cast<unsigned>(want < static_cast<uint64_t>(sm_count) ? want : sm_count);
    if (key_bytes == 4)
        global_histogram_kernel<uint32_t><<<grid, kHistThreads, hist_smem_bytes<uint32_t>(), stream>>>(
            static_cast<const uint32_t*>(keys), n, ghist, codec);
    else
        global_histogram_kernel<uint64_t><<<grid, kHistThreads, hist_smem_bytes<uint64_t>(), stream>>>(
            static_cast<const uint64_t*>(keys), n, ghist, codec);
    return cudaGetLastError();
}

// Single digit place (the sharded path's most-significant-digit histogram): one atomic per key, same
// bank-private column layout, 32 KB of shared memory.
template <typename KeyT>
__global__ void __launch_bounds__(kHistThreads, 1)
digit_histogram_kernel(const KeyT* __restrict__ keys, uint64_t n, uint32_t shift, unsigned long long* __restrict__ hist256)
{
    __shared__ uint32_t s_hist[kRadix * 32];
    for (int i = threadIdx.x; i < kRadix * 32; i += kHistThreads) s_hist[i] = 0;
    __syncthreads();
    uint32_t* s_col = s_hist + (threadIdx.x & 31);
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kHistThreads;
    uint64_t i = static_cast<uint64_t>(blockIdx.x) * kHistThreads + threadIdx.x;
    for (; i + 3 * stride < n; i += 4 * stride) {
        const KeyT a = __ldcs(keys + i), b = __ldcs(keys + i + stride), c = __ldcs(keys + i + 2 * stride),
                   d = __ldcs(keys + i + 3 * stride);
        atomicAdd(&s_col[digit_of(a, shift) * 32], 1u);
        atomicAdd(&s_col[digit_of(b, shift) * 32], 1u);
        atomicAdd(&s_col[digit_of(c, shift) * 32], 1u);
        atomicAdd(&s_col[digit_of(d, shift) * 32], 1u);
    }
    for (; i < n; i += stride) atomicAdd(&s_col[digit_of(__ldcs(keys + i), shift) * 32], 1u);
    __syncthreads();
    for (int bin = threadIdx.x; bin < kRadix; bin += kHistThreads) {
        uint32_t sum = 0;
#pragma unroll 8
        for (int c = 0; c < 32; ++c) sum += s_hist[bin * 32 + ((c + threadIdx.x) & 31)];
        if (sum) atomicAdd(&hist256[bin], static_cast<unsigned long long>(sum));
    }
}

cudaError_t launch_digit_histogram(const void* keys, uint64_t n, int key_bytes, uint32_t shift,
                                   unsigned long long* hist256, int sm_count, cudaStream_t stream)
{
    uint64_t want = (n + kHistThreads * 4 - 1) / (kHistThreads * 4);
    if (want < 1) want = 1;
    const unsigned grid = static_cast<unsigned>(want < static_cast<uint64_t>(sm_count) * 2 ? want : sm_count * 2);
    if (key_bytes == 4)
        digit_histogram_kernel<uint32_t><<<grid, kHistThreads, 0, stream>>>(static_cast<const uint32_t*>(keys), n, shift, hist256);
    else
        digit_histogram_kernel<uint64_t><<<grid, kHistThreads, 0, stream>>>(static_cast<const uint64_t*>(keys), n, shift, hist256);
    return cudaGetLastError();
}

// =====================================================================================================
// Scan: exclusive prefix over the 256 bins of each digit place (reference: OneSweep::Scan, OneSweep.cu:125-162), and --
// new here -- the device-side launch plan: a place whose histogram has ONE non-empty bin (all n keys share that digit)
// is marked skipped, so its DigitBinningPass exits at once; the passes derive their source/destination from the
// number of executed passes before them, and a final copy moves the result home if that number is odd.
// One CTA walks the (at most 8) places: the plan needs all of them.
// =====================================================================================================
__global__ void __launch_bounds__(kRadix)
scan_kernel(const unsigned long long* __restrict__ ghist, unsigned long long* __restrict__ gbase, int places,
            SortPlan* plan, unsigned long long n, int allow_skip, int allow_hot)
{
    __shared__ unsigned long long s_warp[kRadix / 32];
    const int d = threadIdx.x, lane = d & 31, warp = d >> 5;
    uint32_t skip_mask = 0;
    for (int p = 0; p < places; ++p) {
        const unsigned long long c = ghist[p * kRadix + d];
        unsigned long long incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[warp] = incl;
        const int single_bin = __syncthreads_or(plan != nullptr && allow_skip && c == n);
        // hot pass: one bin holds at least an eighth of the keys (and the input is large enough for resident CTAs to pay)
        const int hot_bin = __syncthreads_or(plan != nullptr && allow_hot && n >= (1ull << 22) && c * 8ull >= n);
        unsigned long long pre = 0;
        for (int w = 0; w < warp; ++w) pre += s_warp[w];
        gbase[p * kRadix + d] = pre + incl - c;
        if (single_bin) skip_mask |= 1u << p;
        else if (hot_bin) skip_mask |= 1u << (kPlanHotShift + p);
        __syncthreads();  // s_warp is reused by the next place
    }
    if (plan != nullptr && d == 0) {
        SortPlan pl;
        pl.skip_mask = skip_mask;
        const uint32_t run = ~skip_mask & ((places >= 32 ? 0u : (1u << places)) - 1u);
        pl.executed = __popc(run);
        pl.first_exec = run ? static_cast<uint32_t>(__ffs(run) - 1) : 0xffffffffu;
        pl.last_exec = run ? static_cast<uint32_t>(31 - __clz(run)) : 0xffffffffu;
        *plan = pl;
    }
}

cudaError_t launch_scan(const unsigned long long* ghist, unsigned long long* gbase, int places, cudaStream_t stream,
                        SortPlan* plan, uint64_t n, bool allow_skip, bool allow_hot)
{
    scan_kernel<<<1, kRadix, 0, stream>>>(ghist, gbase, places, plan, n, allow_skip ? 1 : 0, allow_hot ? 1 : 0);
    return cudaGetLastError();
}

// =====================================================================================================
// GlobalHistogram for begin_bit/end_bit sorts: digit places start at an arbitrary bit and the last one may be narrower
// than 8 bits, so the digits are extracted key by key (the byte-aligned kernel above slices the loaded words directly).
// Same bank-private column layout.
// =====================================================================================================
template <typename KeyT>
__global__ void __launch_bounds__(kHistThreads, 1)
global_histogram_bits_kernel(const KeyT* __restrict__ keys, uint64_t n, unsigned long long* __restrict__ ghist, KeyCodec codec,
                             uint32_t begin_bit, int places, uint32_t last_mask)
{
    constexpr int COLS = HistGeom<KeyT>::COLS;
    extern __shared__ __align__(16) uint32_t s_hist[];  // [places * 256][COLS]
    const int bins = places * kRadix;
    for (int i = threadIdx.x; i < bins * COLS; i += kHistThreads) s_hist[i] = 0;
    __syncthreads();
    uint32_t* s_col = s_hist + (threadIdx.x & (COLS - 1));
    const bool enc = codec.flags & kCodecEncodeOnLoad;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * kHistThreads;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kHistThreads + threadIdx.x; i < n; i += stride) {
        KeyT k = __ldcs(keys + i);
        if (enc) k = codec_encode<KeyT>(k, ca, cb, cd);
        for (int p = 0; p < places; ++p) {
            const uint32_t dg = digit_of(k, begin_bit + 8u * p, p == places - 1 ? last_mask : 255u);
            atomicAdd(&s_col[(p * kRadix + dg) * COLS], 1u);
        }
    }
    __syncthreads();
    for (int bin = threadIdx.x; bin < bins; bin += kHistThreads) {
        uint32_t sum = 0;
#pragma unroll 8
        for (int c = 0; c < COLS; ++c) sum += s_hist[bin * COLS + ((c + threadIdx.x) & (COLS - 1))];
        if (sum) atomicAdd(&ghist[bin], static_cast<unsigned long long>(sum));
    }
}

cudaError_t launch_global_histogram_bits(const void* keys, uint64_t n, int key_bytes, unsigned long long* ghist, int sm_count,
                                         cudaStream_t stream, const KeyCodec* codec_in, uint32_t begin_bit, int places,
                                         uint32_t last_bits)
{
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    const uint32_t last_mask = (1u << last_bits) - 1u;
    if (begin_bit == 0) {  // byte-aligned places: the fast kernel slices the loaded words, the last place keeps last_bits
        const uint64_t vecs = n / (16 / key_bytes);
        uint64_t w2 = (vecs + kHistThreads - 1) / kHistThreads;
        if (w2 < 1) w2 = 1;
        const unsigned g2 = static_cast<unsigned>(w2 < static_cast<uint64_t>(sm_count) ? w2 : sm_count);
        if (key_bytes == 4)
            global_histogram_kernel<uint32_t, true><<<g2, kHistThreads, hist_smem_bytes<uint32_t>(), stream>>>(
                static_cast<const uint32_t*>(keys), n, ghist, codec, places, last_mask);
        else
            global_histogram_kernel<uint64_t, true><<<g2, kHistThreads, hist_smem_bytes<uint64_t>(), stream>>>(
                static_cast<const uint64_t*>(keys), n, ghist, codec, places, last_mask);
        return cudaGetLastError();
    }
    uint64_t want = (n + kHistThreads * 4 - 1) / (kHistThreads * 4);
    if (want < 1) want = 1;
    const unsigned grid = static_cast<unsigned>(want < static_cast<uint64_t>(sm_count) ? want : sm_count);
    if (key_bytes == 4)
        global_histogram_bits_kernel<uint32_t><<<grid, kHistThreads, hist_smem_bytes<uint32_t>(), stream>>>(
            static_cast<const uint32_t*>(keys), n, ghist, codec, begin_bit, places, last_mask);
    else
        global_histogram_bits_kernel<uint64_t><<<grid, kHistThreads, hist_smem_bytes<uint64_t>(), stream>>>(
            static_cast<const uint64_t*>(keys), n, ghist, codec, begin_bit, places, last_mask);
    return cudaGetLastError();
}

// =====================================================================================================
// copy_back: an odd number of executed passes leaves the result in the alt buffers
// =====================================================================================================
// W is the word each thread moves: uint4 when both buffers are 16-byte aligned, else uint32_t.  The caller's keys are
// always 16-byte aligned (sort_impl checks them), but values need only their natural 4-byte alignment, and a 16-byte
// access to a value buffer that starts at another offset is a misaligned-address fault.
template <typename W>
__global__ void __launch_bounds__(512)
copy_back_kernel(const SortPlan* __restrict__ plan, const W* __restrict__ src, W* __restrict__ dst, uint64_t words,
                 const unsigned char* __restrict__ src_tail, unsigned char* __restrict__ dst_tail, uint32_t tail_bytes)
{
    if (!(plan->executed & 1u)) return;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < words; i += stride) __stcs(dst + i, __ldcs(src + i));
    if (blockIdx.x == 0 && threadIdx.x < tail_bytes) dst_tail[threadIdx.x] = src_tail[threadIdx.x];
}

cudaError_t launch_copy_back(const SortPlan* plan, const void* alt_keys, void* keys, const uint32_t* alt_vals, uint32_t* vals,
                             uint64_t n, int key_bytes, int sm_count, cudaStream_t stream)
{
    auto launch = [&](auto word, const void* s, void* d, uint64_t bytes) {
        using W = decltype(word);
        const uint64_t words = bytes / sizeof(W);
        uint64_t want = (words + 511) / 512;
        if (want < 1) want = 1;
        const unsigned grid = static_cast<unsigned>(want < static_cast<uint64_t>(sm_count) * 4 ? want : sm_count * 4);
        copy_back_kernel<W><<<grid, 512, 0, stream>>>(plan, static_cast<const W*>(s), static_cast<W*>(d), words,
                                                      static_cast<const unsigned char*>(s) + words * sizeof(W),
                                                      static_cast<unsigned char*>(d) + words * sizeof(W),
                                                      static_cast<uint32_t>(bytes - words * sizeof(W)));
    };
    auto one = [&](const void* s, void* d, uint64_t bytes) {
        if (((reinterpret_cast<uintptr_t>(s) | reinterpret_cast<uintptr_t>(d)) & 15u) == 0) launch(uint4{}, s, d, bytes);
        else launch(uint32_t{}, s, d, bytes);
    };
    one(alt_keys, keys, n * key_bytes);
    if (vals) one(alt_vals, vals, n * sizeof(uint32_t));
    return cudaGetLastError();
}

// argsort: keys and indices in one launch.  Odd executed passes: both from the alt buffers.  No executed pass (all keys
// equal): the input is its own stable sort -- keys from the untouched input, indices 0..n-1.  (All pointers 16-byte aligned.)
__global__ void __launch_bounds__(512)
argsort_copy_back_kernel(const SortPlan* __restrict__ plan, const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ alt_keys,
                         uint32_t* __restrict__ keys, const uint32_t* __restrict__ alt_idx, uint32_t* __restrict__ idx, uint64_t n)
{
    const uint32_t ex = plan->executed;
    if (ex != 0 && !(ex & 1u)) return;
    const uint32_t* src = ex ? alt_keys : keys_in;
    const uint64_t vecs = n / 4, stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < vecs; i += stride) {
        __stcs(reinterpret_cast<uint4*>(keys) + i, __ldcs(reinterpret_cast<const uint4*>(src) + i));
        const uint32_t b = static_cast<uint32_t>(i * 4);
        __stcs(reinterpret_cast<uint4*>(idx) + i, ex ? __ldcs(reinterpret_cast<const uint4*>(alt_idx) + i) : make_uint4(b, b + 1, b + 2, b + 3));
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3u)) {
        const uint64_t j = vecs * 4 + threadIdx.x;
        keys[j] = src[j];
        idx[j] = ex ? alt_idx[j] : static_cast<uint32_t>(j);
    }
}

cudaError_t launch_argsort_copy_back(const SortPlan* plan, const void* keys_in, const void* alt_keys, void* keys,
                                     const uint32_t* alt_idx, uint32_t* idx, uint64_t n, int sm_count, cudaStream_t stream)
{
    uint64_t want = (n / 4 + 511) / 512;
    if (want < 1) want = 1;
    const unsigned grid = static_cast<unsigned>(want < static_cast<uint64_t>(sm_count) * 4 ? want : sm_count * 4);
    argsort_copy_back_kernel<<<grid, 512, 0, stream>>>(plan, static_cast<const uint32_t*>(keys_in), static_cast<const uint32_t*>(alt_keys),
                                                       static_cast<uint32_t*>(keys), alt_idx, idx, n);
    return cudaGetLastError();
}

// =====================================================================================================
// Shared pieces of the digit-binning kernels
// =====================================================================================================

// 8-ballot warp match (RankMode::kRankBallot): mask of lanes holding the same digit.
__device__ __forceinline__ uint32_t warp_match_digit(uint32_t d)
{
    uint32_t m = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < kRadixLog; ++b) {
        const bool p = (d >> b) & 1u;
        const uint32_t bal = __ballot_sync(0xffffffffu, p);
        m &= p ? bal : ~bal;
    }
    return m;
}

// Rank of one key per lane inside its warp's running histogram (returns #earlier keys of this warp with the
// same digit, in tile order) and bumps the histogram.  `wh` = this warp's 256-bin histogram in shared memory.
template <int RANK_MODE>
__device__ __forceinline__ uint32_t warp_rank_and_count(uint32_t* wh, uint32_t d, uint32_t lt_mask)
{
    if constexpr (RANK_MODE == kRankAtomic) {
        (void)lt_mask;
        return atomicAdd(&wh[d], 1u);  // lane-ordered among same-digit lanes of this instruction (see header)
    } else {
        const uint32_t m = warp_match_digit(d);
        const uint32_t below = __popc(m & lt_mask);
        uint32_t pre = 0;
        if (below == 0) { pre = wh[d]; wh[d] = pre + __popc(m); }
        __syncwarp();
        pre = __shfl_sync(0xffffffffu, pre, __ffs(m) - 1);
        return pre + below;
    }
}

// Exclusive scan of one value per digit thread (threads 0..255 contribute, all THREADS threads call).
template <int THREADS>
__device__ __forceinline__ uint32_t block_excl_scan_256(uint32_t c, uint32_t* s_wtot /*[8]*/)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (tid < kRadix && lane == 31) s_wtot[warp] = incl;
    __syncthreads();
    uint32_t pre = 0;
    if (tid < kRadix) {
#pragma unroll
        for (int w = 0; w < kRadix / 32; ++w) pre += (w < warp) ? s_wtot[w] : 0u;
    }
    return pre + incl - c;
}

// Decoupled lookback for (tile, digit d): sum of the digit counts of all predecessor tiles plus the global
// digit base.  Reference: OneSweep.cu:306-327.  `tile_count` is this tile's count of digit d.
__device__ __forceinline__ unsigned long long
lookback_and_publish(uint64_t* desc, uint32_t tile, uint32_t d, uint32_t tile_count, uint32_t epoch,
                     const unsigned long long* __restrict__ gbase)
{
    uint64_t* mine = desc + static_cast<uint64_t>(tile) * kRadix + d;
    unsigned long long excl = 0;
    int64_t k = static_cast<int64_t>(tile) - 1;
    while (true) {
        if (k < 0) break;
        const uint64_t v = ld_relaxed_gpu_u64(desc + static_cast<uint64_t>(k) * kRadix + d);
        const uint64_t flag = v & kFlagMask;
        if (desc_epoch(v) != epoch || flag == kFlagNotReady) { __nanosleep(20); continue; }
        excl += desc_value(v);
        if (flag == kFlagInclusive) break;
        --k;
    }
    // descriptors carry counts relative to the start of the array (< n <= 2^38); the global digit base -- which in the
    // sharded exchange pass is a peer ADDRESS, far larger than the value field -- is added only to the result
    st_relaxed_gpu_u64(mine, desc_pack(epoch, kFlagInclusive, excl + tile_count));
    return excl + gbase[d];
}

// =====================================================================================================
// DigitBinningPass, variant 0: one CTA per partition tile (dynamic tile id), keys held in registers.
// =====================================================================================================
template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE>
__global__ void __launch_bounds__(WARPS * 32, (RANK_MODE == kRankAtomic && !PAIRS) ? 2 : 1)
digit_binning_tile_kernel(const KeyT* __restrict__ in, KeyT* __restrict__ out, const uint32_t* __restrict__ in_val,
                          uint32_t* __restrict__ out_val, uint64_t n, uint32_t shift,
                          const unsigned long long* __restrict__ gbase, uint64_t* desc, uint32_t* ticket, uint32_t epoch)
{
    constexpr int THREADS = WARPS * 32;
    constexpr int T = THREADS * K;  // keys per partition tile
    static_assert(WARPS >= 8, "need one thread per digit");
    extern __shared__ __align__(128) unsigned char s_raw[];  // max(WARPS*256*4, T*sizeof(KeyT)) bytes
    uint32_t* s_hist = reinterpret_cast<uint32_t*>(s_raw);  // [WARPS][256] during ranking
    KeyT* s_keys = reinterpret_cast<KeyT*>(s_raw);          // [T] digit-sorted tile afterwards
    uint32_t* s_vals = reinterpret_cast<uint32_t*>(s_raw);  // [T] payloads in the same order (pairs)
    __shared__ unsigned long long s_keyptr[kRadix];  // per digit: byte address of out[global_base - tile_base]
    __shared__ unsigned long long s_valptr[PAIRS ? kRadix : 1];
    __shared__ uint32_t s_wtot[kRadix / 32];
    __shared__ uint32_t s_tile;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int i = tid; i < WARPS * kRadix; i += THREADS) s_hist[i] = 0;
    if (tid == 0) s_tile = atomicAdd(ticket, 1u);  // dynamic tile id: predecessors are already scheduled
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint64_t tile_base = static_cast<uint64_t>(tile) * T;
    const uint32_t valid = static_cast<uint32_t>(n - tile_base < static_cast<uint64_t>(T) ? n - tile_base : T);

    // ---- load: warp-striped, one coalesced 128 B (256 B for u64) row per warp instruction --------------
    KeyT key[K];
    const uint32_t warp_off = warp * (32 * K) + lane;
    if (valid == T) {
#pragma unroll
        for (int i = 0; i < K; ++i) key[i] = ld_stream(in + tile_base + warp_off + i * 32);
    } else {
        // the last tile is padded with all-ones keys: they rank after every real key of digit 255 and
        // therefore land at tile positions >= valid, which are never written (reference: OneSweep.cu:195-205)
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t idx = warp_off + i * 32;
            key[i] = idx < valid ? in[tile_base + idx] : static_cast<KeyT>(~static_cast<KeyT>(0));
        }
    }

    // ---- rank inside the warp (tile order = warp-major, then round, then lane) ------------------------
    uint32_t off[K];
    uint32_t* wh = s_hist + warp * kRadix;
    const uint32_t lt = lanemask_lt();
#pragma unroll
    for (int i = 0; i < K; ++i) off[i] = warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], shift), lt);
    __syncthreads();

    // ---- per digit: exclusive prefix over the warps, tile reduction, publish, scan over digits --------
    uint32_t tile_count = 0, tile_excl = 0;
    {
        if (tid < kRadix) {
#pragma unroll
            for (int w = 0; w < WARPS; ++w) tile_count += s_hist[w * kRadix + tid];
            st_relaxed_gpu_u64(desc + static_cast<uint64_t>(tile) * kRadix + tid,
                               desc_pack(epoch, kFlagReduction, tile_count));
        }
        tile_excl = block_excl_scan_256<THREADS>(tile_count, s_wtot);
        if (tid < kRadix) {
            uint32_t run = tile_excl;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) { const uint32_t c = s_hist[w * kRadix + tid]; s_hist[w * kRadix + tid] = run; run += c; }
        }
    }
    __syncthreads();

    // ---- position of every key inside the digit-sorted tile -------------------------------------------
#pragma unroll
    for (int i = 0; i < K; ++i) off[i] += wh[digit_of(key[i], shift)];
    __syncthreads();  // histograms are dead; the same shared memory now receives the sorted tile

#pragma unroll
    for (int i = 0; i < K; ++i) s_keys[off[i]] = key[i];

    // payload loads are issued here so that their latency overlaps the lookback
    uint32_t val[PAIRS ? K : 1];
    if constexpr (PAIRS) {
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t idx = warp_off + i * 32;
            val[i] = idx < valid ? ld_stream(in_val + tile_base + idx) : 0u;
        }
    }

    // ---- chained scan with decoupled lookback, one thread per digit -----------------------------------
    if (tid < kRadix) {
        const unsigned long long excl = lookback_and_publish(desc, tile, tid, tile_count, epoch, gbase);
        const unsigned long long first = excl - tile_excl;  // out index of tile position 0 "as if" of this digit
        s_keyptr[tid] = reinterpret_cast<unsigned long long>(out) + first * sizeof(KeyT);
        if constexpr (PAIRS) s_valptr[tid] = reinterpret_cast<unsigned long long>(out_val) + first * sizeof(uint32_t);
    }
    __syncthreads();

    // ---- scatter: consecutive threads write consecutive addresses inside each digit run ---------------
    uint32_t dg[PAIRS ? K : 1];
#pragma unroll
    for (int j = 0; j < K; ++j) {
        const uint32_t idx = j * THREADS + tid;
        if (idx < valid) {
            const KeyT k = s_keys[idx];
            const uint32_t d = digit_of(k, shift);
            if constexpr (PAIRS) dg[j] = d;
            KeyT* dst = reinterpret_cast<KeyT*>(s_keyptr[d]) + idx;
            st_stream(dst, k);
        }
    }
    if constexpr (PAIRS) {
        __syncthreads();
#pragma unroll
        for (int i = 0; i < K; ++i) s_vals[off[i]] = val[i];
        __syncthreads();
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const uint32_t idx = j * THREADS + tid;
            if (idx < valid) {
                uint32_t* dst = reinterpret_cast<uint32_t*>(s_valptr[dg[j]]) + idx;
                st_stream(dst, s_vals[idx]);
            }
        }
    }
}

// =====================================================================================================
// TMA / mbarrier helpers used by DigitBinningPass variant 1 (the persistent, TMA-staged ring kernel further down).
// =====================================================================================================
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy completing on an mbarrier (bytes and both addresses multiples of 16)
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_addr(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// =====================================================================================================
// DigitBinningPass, variant 2 ("wide tile"): 16,384-key partition tiles, two CTAs per SM.
//
// Why the tile is this large.  In a chained scan the number of predecessor tiles that have published only their
// reduction when a tile starts looking back is (tiles entering per second) x (latency from publishing a reduction
// to publishing the inclusive prefix).  With variant 0's 8,192-key tiles at HBM rate that window is tens of tiles,
// one L2 round trip per lookback step, and the lookback becomes the critical path.  Doubling the tile
// halves the window and halves the per-key cost of each step; the remaining window (~16) is covered in ONE round
// trip by issuing all of its loads at once.  To keep that affordable the reductions live in a compact array of
// 16-bit words (flag:1 | count:15 -- a tile holds at most 16,384 keys), 512 B per tile instead of 2 KB; only the
// inclusive prefixes use the 64-bit epoch-stamped descriptors.
//
// Ranking is two shared-memory atomics per key on warp-private histograms: a non-returning count, then -- after
// the per-digit bases of the tile have been scanned into the same counters -- a returning atomicAdd whose result
// IS the key's slot in the digit-sorted tile (lane-ordered, see top of file).  No per-key offsets are kept in
// registers, so 32 keys per thread fit in a 64-register budget (2 x 512 threads per SM).
// =====================================================================================================
// OSB_PHASE_PROBE=1 (development builds only; 0 in the product build): the wide kernel's per-phase clock probe, read by
// tools/phase_probe.py through the exported osb200_debug_phases.
#ifndef OSB_PHASE_PROBE
#define OSB_PHASE_PROBE 0
#endif

#if OSB_PHASE_PROBE
// per-phase wall clocks of the wide kernel, summed over tiles by thread 0: [0]=tile start (the first tile of a CTA: plan,
// histogram clear), [1]=wait for the tile's keys, [2]=count, [3]=reduce/scan/bases, [4]=rank + next tile's loads issued,
// [5]=lookback, [6]=scatter, [7]=tiles, [8]=barrier after lookback, [9]=lookback windows (digit 0), [10]=stalled polls
__device__ unsigned long long g_phase[11];
#define OSB_PHASE(i) do { if (tid == 0) { const long long t_now = clock64(); atomicAdd(&g_phase[i], static_cast<unsigned long long>(t_now - t_prev)); t_prev = t_now; } } while (0)
}  // namespace osb
extern "C" __attribute__((visibility("default"))) int osb200_debug_phases(unsigned long long* out11 /*[11]*/, int reset)
{
    if (out11) cudaMemcpyFromSymbol(out11, osb::g_phase, sizeof(osb::g_phase));
    if (reset) { unsigned long long z[11] = {0}; cudaMemcpyToSymbol(osb::g_phase, z, sizeof(z)); }
    return 0;
}
namespace osb {
#else
#define OSB_PHASE(i) do {} while (0)
#endif

constexpr uint32_t kAggReady = 0x8000u;   // agg16 word: bit 15 = reduction published, bits 0..14 = count

__device__ __forceinline__ void st_relaxed_gpu_u16(uint16_t* p, uint32_t v)
{
    asm volatile("st.relaxed.gpu.global.u16 [%0], %1;" ::"l"(p), "h"(static_cast<uint16_t>(v)) : "memory");
}

// What a digit thread needs to re-reduce a predecessor tile by itself (forward-progress fallback).
template <typename KeyT>
struct TileRereduce {
    const KeyT* in;      // this pass's input keys
    uint32_t tile_keys;  // T
    uint32_t shift, mask;
    bool encode;         // typed keys, first executed pass: the digits are those of the ENCODED keys
    KeyT ca, cb, cd;
};

// Forward-progress fallback (reference: EmulatedDeadlocking.cu:159-267, SweepCommon.hlsl:317-425 -- a thread block that
// has spun too long on a predecessor's flag stops waiting and computes that tile's reduction itself).  Here every digit
// thread that gives up on tile x counts ITS digit over the tile's keys (the whole warp reads the same key: one
// broadcast transaction per load; predecessor tiles are never the ragged last tile) and publishes the reduction on the
// owner's behalf -- the value is the one the owner would write, so concurrent publishers agree.  Cold path, kept out of
// line (scalar arguments: nothing of the caller's goes through the stack).
template <typename KeyT>
__device__ __noinline__ uint32_t rereduce_tile(const KeyT* p, uint32_t tile_keys, uint32_t shift, uint32_t mask, uint32_t encode,
                                               KeyT ca, KeyT cb, KeyT cd, uint16_t* dst, uint32_t d)
{
    uint32_t c = 0;
#pragma unroll 8
    for (uint32_t i = 0; i < tile_keys; ++i) {
        KeyT k = p[i];
        if (encode) k = codec_encode<KeyT>(k, ca, cb, cd);
        c += digit_of(k, shift, mask) == d;
    }
    st_relaxed_gpu_u16(dst, kAggReady | c);
    return c;
}

// Layout of the compact reductions: blocks of 8 consecutive tiles, [tile / 8][digit][tile % 8] 16-bit words, so that ONE
// 16-byte load returns a digit's reductions of 8 consecutive tiles (a [tile][digit] layout needs eight 2-byte loads per
// window, and the lookback windows then take a large share of a CTA's lifetime).
__device__ __forceinline__ uint64_t agg_index(uint64_t tile, uint32_t d) { return ((tile >> 3) * kRadix + d) * 8 + (tile & 7); }

__device__ __forceinline__ uint4 ld_relaxed_gpu_v4(const void* p)
{
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
// 16-bit element t (0..7) of a block vector
__device__ __forceinline__ uint32_t agg_elem(const uint4& v, int t)
{
    const uint32_t w = t < 2 ? v.x : t < 4 ? v.y : t < 6 ? v.z : v.w;
    return (t & 1) ? (w >> 16) : (w & 0xffffu);
}

// Decoupled lookback over the compact reductions.  One round trip fetches NBLK blocks of 8 tiles (the nearest one partial:
// the predecessors inside this tile's own block) plus, per block, the inclusive prefix of the tile just before it.  Returns
// the number of keys with digit d in all predecessor tiles (relative to the start of the array: the global digit base is
// added by the caller, so descriptor values stay below n even when the bases are peer addresses in the sharded exchange
// pass).  A predecessor whose reduction is still missing after spin_cap polls is re-reduced by this thread
// (rereduce_tile): the spin is bounded.
template <int NBLK, typename KeyT>
__device__ __forceinline__ unsigned long long
lookback_wide(uint16_t* agg16, const uint64_t* incl64, uint32_t tile, uint32_t d, uint32_t epoch, uint32_t spin_cap,
              const TileRereduce<KeyT>& rr)
{
    unsigned long long sum = 0;                       // reductions of tiles (cur, tile-1] already added
    int64_t cur = static_cast<int64_t>(tile) - 1;     // nearest predecessor not yet accounted for
    uint32_t polls = 0;                               // consecutive unsuccessful polls of tile `cur`
    while (true) {
        if (cur < 0) return sum;
#if OSB_PHASE_PROBE
        if (d == 0) atomicAdd(&g_phase[9], 1ull);
#endif
        const int64_t b0 = cur >> 3;
        uint4 v[NBLK];
        uint64_t c[NBLK];
#pragma unroll
        for (int k = 0; k < NBLK; ++k) {
            const int64_t b = b0 - k;
            v[k] = b >= 0 ? ld_relaxed_gpu_v4(agg16 + (static_cast<uint64_t>(b) * kRadix + d) * 8)
                          : make_uint4(0x80008000u, 0x80008000u, 0x80008000u, 0x80008000u);
            c[k] = b > 0 ? ld_relaxed_gpu_u64(incl64 + (static_cast<uint64_t>(b) * 8 - 1) * kRadix + d) : 0ull;
        }
        unsigned long long run = sum;
        int64_t next = (b0 - NBLK + 1) * 8 - 1;  // where to continue if the whole window was reductions only
        bool stalled = false;
        const int hi0 = static_cast<int>(cur & 7);
#pragma unroll
        for (int k = 0; k < NBLK; ++k) {
            const int64_t b = b0 - k;
            if (b < 0) return run;
#pragma unroll
            for (int t = 7; t >= 0; --t) {
                if (k == 0 && t > hi0) continue;
                const uint32_t a = agg_elem(v[k], t);
                if (!(a & kAggReady)) { next = b * 8 + t; stalled = true; break; }
                run += a & 0x7fffu;
            }
            if (stalled) break;
            if (b == 0) return run;  // tile 0 has no predecessors
            if (desc_epoch(c[k]) == epoch && (c[k] & kFlagMask) == kFlagInclusive) return run + desc_value(c[k]);
        }
        sum = run;
        if (stalled) {
            polls = next == cur ? polls + 1 : 1;
            if (polls > spin_cap) {
                // maybe the stalled tile has finished altogether meanwhile: its inclusive prefix settles everything
                const uint64_t w = ld_relaxed_gpu_u64(incl64 + next * kRadix + d);
                if (desc_epoch(w) == epoch && (w & kFlagMask) == kFlagInclusive) return sum + desc_value(w);
                sum += rereduce_tile<KeyT>(rr.in + static_cast<uint64_t>(next) * rr.tile_keys, rr.tile_keys, rr.shift, rr.mask,
                                           rr.encode ? 1u : 0u, rr.ca, rr.cb, rr.cd, agg16 + agg_index(next, d), d);
                --next;
                polls = 0;
            } else {
#if OSB_PHASE_PROBE
                if (d == 0) atomicAdd(&g_phase[10], 1ull);
#endif
                __nanosleep(40);
            }
        } else {
            polls = 0;
        }
        cur = next;
    }
}


// ---- hot digit -------------------------------------------------------------------------------------------------------
// Low-entropy inputs (the reference's entropy presets 2-5, UtilityKernels.cuh:42-52: AND of several random words) put a
// large share of every tile into ONE bin.  Same-address returning atomics serialise lane by lane, so such passes run far
// below the uniform rate.  Remedy: the Scan kernel flags a digit place whose
// global histogram has a bin with >= n/8 keys ("hot pass", SortPlan); such a pass is executed by the HOT instantiation of
// digit_binning_wide_kernel -- resident CTAs striding over the tiles -- in which the keys of a tile's most frequent digit
// are ranked with one ballot per round (rank = popc of the lower lanes + a running count in a register) and only the other
// lanes issue the atomic; the hot keys' slots are consecutive, so their transposing stores are conflict-free as well.
// It is a second instantiation rather than a branch because the extra state costs registers the plain loop does not have
// (keeping both in one kernel spills in the uniform path); the host enqueues both kernels
// for every pass and the plan decides which one returns at once -- the resident form makes the idle one a ~5 us launch.
constexpr uint32_t kNoHotDigit = 0xffffffffu;
#ifndef OSB_HOT_MINB  // resident CTAs per SM of the HOT instantiation: 1 = up to 128 registers, no spills
#define OSB_HOT_MINB 1
#endif

__device__ __forceinline__ void hot_digit_publish(uint32_t tile_count, uint32_t* s_wmax)
{
    const int tid = threadIdx.x;
    if (tid < kRadix) {
        const uint32_t m = __reduce_max_sync(0xffffffffu, (tile_count << 8) | static_cast<uint32_t>(tid));
        if ((tid & 31) == 0) s_wmax[tid >> 5] = m;
    }
}
__device__ __forceinline__ uint32_t hot_digit_of_tile(const uint32_t* s_wmax, uint32_t tile_keys)
{
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < kRadix / 32; ++w) m = max(m, s_wmax[w]);
    m = __shfl_sync(0xffffffffu, m, 0);
    return (m >> 8) >= tile_keys / 8 ? (m & 255u) : kNoHotDigit;
}

// Per-launch parameters of one DigitBinningPass.
struct PassParams {
    uint32_t shift;        // bit position of this pass's digit
    uint32_t dbits;        // digit width, 1..8
    uint32_t epoch;        // descriptor epoch of this launch
    uint32_t place;        // index of this pass in the plan
    uint32_t spin_cap;     // lookback polls before the fallback re-reduction
    uint32_t stall_every;  // test hook (0 = off): tiles with tile % N == N-1 never publish their reduction
    const SortPlan* plan;  // device plan or null
    const void* keys_in = nullptr;  // argsort (INDICES): the caller's untouched keys, read by the first executed pass
};

// plan_bits of an argsort pass (INDICES): this is the first executed pass -- its keys come from PassParams::keys_in and its
// payloads are the keys' own input positions
constexpr uint32_t kPlanBitsFirstIndices = 8u;

// Reads a copy of a value the caller also holds in a register, kept in shared memory for this purpose: the compiler cannot
// prove the two equal, so whatever is computed from the copy is computed again rather than taken from earlier expressions
// that are still live.  (An empty inline-asm copy does not survive ptxas once the kernel loops over tiles.)
__device__ __forceinline__ uint32_t opaque_copy(const uint32_t* smem_copy)
{
    return *reinterpret_cast<const volatile uint32_t*>(smem_copy);
}

template <typename KeyT, bool PAIRS, int K, int WARPS>
struct WideSmem {
    static constexpr int THREADS = WARPS * 32;
    static constexpr int T = THREADS * K;
    alignas(16) KeyT sorted[T];                      // digit-sorted tile
    alignas(16) uint32_t sorted_val[PAIRS ? T : 4];  // payloads in the same order
    alignas(16) uint32_t hist[WARPS * kRadix];       // warp-private digit counters (counts, then running slots)
    unsigned long long keyptr[kRadix];               // per digit: byte address of out[first key of the digit - tile slot]
    unsigned long long valptr[PAIRS ? kRadix : 1];
    uint32_t run[32];                                // few-bins passes: first slot (low 16 bits) | live length (high 16)
    uint32_t wtot[kRadix / 32];
    uint32_t wmax[kRadix / 32];                      // (HOT) per digit warp: max of (tile count << 8 | digit)
    uint32_t next_tile;                              // the tile this CTA works on after the current one (drawn ticket)
    uint32_t plan_bits;                              // bit 0: source is the alt buffer; bits 1-2: codec flags of this pass;
                                                     // bit 3: first pass of an argsort (kPlanBitsFirstIndices)
    uint32_t digit_shift, digit_mask;                // copies of the pass's digit, re-read by the rank phase (opaque_copy)
};

// INDICES (argsort, pairs only): buf0/val0 are the caller's output keys and indices, buf1/val1 the alt buffers.  The first
// executed pass, which by the plan's parity would read the caller's side, reads its keys from pp.keys_in instead and makes
// every payload from the key's position in the input; every other pass is the pairs pass as it is.
template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE, int LOOK, int MINB, bool HOT = false, bool INDICES = false>
__global__ void __launch_bounds__(WARPS * 32, HOT ? OSB_HOT_MINB : MINB)
digit_binning_wide_kernel(KeyT* buf0, KeyT* buf1, uint32_t* val0, uint32_t* val1, uint64_t n,
                          const unsigned long long* __restrict__ gbase, uint16_t* agg16, uint64_t* incl64,
                          uint32_t* ticket, PassParams pp, KeyCodec codec)
{
    static_assert(!INDICES || (PAIRS && sizeof(KeyT) == 4), "the indices are the 32-bit payloads of a pairs pass");
    using S = WideSmem<KeyT, PAIRS, K, WARPS>;
    constexpr int THREADS = S::THREADS;
    constexpr int T = S::T;
    static_assert(T < 32768, "agg16 holds 15-bit counts");
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);
    // pairs: key and payload of a tile slot are ONE 64-bit word of shared memory ({key, payload}; `sorted` and `sorted_val`
    // are adjacent and together hold T such words) -- one transposing STS.64 and one LDS.64 per pair instead of two of each,
    // and the payload's destination is the key's plus a constant (reference: OneSweep.cu:522-599 moves them separately)
    static_assert(!PAIRS || (sizeof(KeyT) == 4 && offsetof(S, sorted_val) == offsetof(S, sorted) + sizeof(KeyT) * T), "kv layout");
    uint2* const kv = reinterpret_cast<uint2*>(sm.sorted);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    uint32_t* wh = sm.hist + warp * kRadix;
    const uint32_t shift = pp.shift, epoch = pp.epoch;
    const uint32_t dmask = (1u << pp.dbits) - 1u;
#if OSB_PHASE_PROBE
    long long t_prev = clock64();
#endif

    // The device plan (if any) decides whether this pass runs at all, which buffer it reads, and -- typed keys -- whether it
    // is the pass that encodes / decodes; without a plan the launch arguments are taken as they are.  Every thread reads the
    // 16-byte plan itself (L1 hit for all but the first CTA of an SM).
    uint32_t my_bits = (codec.flags & (kCodecEncodeOnLoad | kCodecDecodeOnStore)) << 1;
    bool my_skip = false, my_hot = false;
    if (pp.plan != nullptr) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(pp.plan));
        SortPlan pl; pl.skip_mask = raw.x; pl.executed = raw.y; pl.first_exec = raw.z; pl.last_exec = raw.w;
        my_skip = (pl.skip_mask >> pp.place) & 1u;
        my_hot = (pl.skip_mask >> (kPlanHotShift + pp.place)) & 1u;
        my_bits = plan_src_is_alt(pl, pp.place) ? 1u : 0u;
        if (codec.flags & kCodecFromPlan)
            my_bits |= (pp.place == pl.first_exec ? kCodecEncodeOnLoad << 1 : 0u) | (pp.place == pl.last_exec ? kCodecDecodeOnStore << 1 : 0u);
        if constexpr (INDICES) my_bits |= pp.place == pl.first_exec ? kPlanBitsFirstIndices : 0u;
    }
    if (my_skip) return;  // all keys share this digit: nothing to move (the plan accounts for the parity)
    if (HOT != my_hot) return;  // a pass is executed by exactly one of the two instantiations the host enqueues
    const uint32_t num_tiles = static_cast<uint32_t>((n + T - 1) / T);

    // ---- tile loads (warp-striped: every warp instruction reads one contiguous 128 B / 256 B row) ----------------
    // The ragged last tile is padded with all-ones keys (they rank last); a tile at or past num_tiles loads nothing.
    KeyT key[K];
    uint32_t val[PAIRS ? K : 1];
    const uint32_t warp_off = warp * (32 * K) + lane;
    auto load_tile = [&](uint32_t t) {
        const bool swap = my_bits & 1u;
        const bool iota = INDICES && (my_bits & kPlanBitsFirstIndices);  // argsort, first pass: payload = input position
        const KeyT* __restrict__ in = iota ? static_cast<const KeyT*>(pp.keys_in) : swap ? buf1 : buf0;
        const uint32_t* __restrict__ in_val = swap ? val1 : val0;
        const uint64_t base = static_cast<uint64_t>(t) * T;
        // (an argsort has n <= 2^32: every input position fits the 32-bit payload)
        const uint32_t pos0 = static_cast<uint32_t>(base) + warp_off;
        if (base + T <= n) {
#pragma unroll
            for (int i = 0; i < K; ++i) key[i] = ld_stream(in + base + warp_off + i * 32);
            if constexpr (PAIRS) {
                if (iota) {
#pragma unroll
                    for (int i = 0; i < K; ++i) val[i] = pos0 + i * 32;
                } else {
#pragma unroll
                    for (int i = 0; i < K; ++i) val[i] = ld_stream(in_val + base + warp_off + i * 32);
                }
            }
        } else {
            const uint32_t live = base < n ? static_cast<uint32_t>(n - base) : 0u;
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const uint32_t idx = warp_off + i * 32;
                key[i] = idx < live ? in[base + idx] : static_cast<KeyT>(~static_cast<KeyT>(0));  // pad: ranks last
                if constexpr (PAIRS) val[i] = iota ? pos0 + i * 32 : idx < live ? in_val[base + idx] : 0u;
            }
        }
    };

    // Persistent CTAs (min(tiles, SMs x resident CTAs per SM)).  A CTA's first tile is blockIdx.x; every later one is drawn
    // from the pass's ticket during the tile before it (after its count phase), and its keys are loaded into the registers the rank phase
    // has just freed, so that they are in flight during the lookback and the scatter.  Tickets are handed out in time order:
    // a drawn tile belongs to a running CTA and its predecessors were drawn before it.  Forward progress does not rest on
    // the dispatch order of the first tiles: a predecessor that is not running is re-reduced by its successors after
    // spin_cap polls (rereduce_tile), so the chained scan cannot hang.
    uint32_t tile = blockIdx.x;
    load_tile(tile);
    {
        uint4* h4 = reinterpret_cast<uint4*>(sm.hist);
        for (int i = tid; i < WARPS * kRadix / 4; i += THREADS) h4[i] = make_uint4(0, 0, 0, 0);
    }
    if (tid == 0) { sm.plan_bits = my_bits; sm.digit_shift = shift; sm.digit_mask = dmask; }
    __syncthreads();  // histograms cleared, plan_bits visible (the loads above are already in flight)
    // plan_bits (direction, codec flags) is re-read from shared memory where it is needed instead of being carried in
    // registers across the phases: the 64-register budget of this kernel is spent on the 32 keys (the rank phase recomputes
    // their counter addresses, see opaque_copy below)
    // The plain u64 keys and pairs passes keep one tile per CTA (their launch has one CTA per tile; the loop body runs once).
    // u64: with its window of 32 tiles the lookback holds four 16-byte blocks per round trip, and 16 prefetched keys held
    // across it spill (180 B per thread); issued after the lookback instead they made the pass 4 % slower on the H100.
    // Pairs: persistent, the pass was up to 0.9 % slower on the H100 (26.01 -> 25.79 Gpairs/s at 400 W).
    constexpr bool kPersistent = (sizeof(KeyT) == 4 && !PAIRS) || HOT;
    while (true) {
    const uint64_t tile_base = static_cast<uint64_t>(tile) * T;
    const bool full = tile_base + T <= n;
    const uint32_t valid = full ? T : static_cast<uint32_t>(n - tile_base);
    OSB_PHASE(0);

    // typed keys: the first executed pass of a sort turns the caller's keys into order-equivalent unsigned keys.  The
    // padding of the ragged last tile is encoded too and stays the largest key only if it was loaded as the pre-image of
    // all-ones, so it is simply re-set after encoding.
    if ((sm.plan_bits >> 1) & kCodecEncodeOnLoad) {
        const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
#pragma unroll
        for (int i = 0; i < K; ++i) {
            key[i] = codec_encode<KeyT>(key[i], ca, cb, cd);
            if (!full && warp_off + i * 32 >= valid) key[i] = static_cast<KeyT>(~static_cast<KeyT>(0));
        }
    }

#if OSB_PHASE_PROBE
#pragma unroll
    for (int i = 0; i < K; ++i) asm volatile("" ::"l"(static_cast<unsigned long long>(key[i])));  // all loads have landed
    OSB_PHASE(1);
#endif
    // ---- phase 1: count digits per warp (order-free, non-returning atomics) ---------------------------
#pragma unroll
    for (int i = 0; i < K; ++i) atomicAdd(&wh[digit_of(key[i], shift, dmask)], 1u);
    __syncthreads();
    OSB_PHASE(2);
    // The next tile is drawn now, as late as its round trip still hides behind the reduce phase: a tile drawn earlier (at the
    // start of the tile before it) starts after that tile's whole, variable lifetime, so tiles begin further out of ticket
    // order and the lookback meets more predecessors that have not published yet.
    uint32_t drawn = 0;
    if (kPersistent && tid == 0) drawn = atomicAdd(ticket, 1u);

    // ---- per digit: tile reduction -> publish; scan over digits; per-warp slot bases --------------------
    uint32_t tile_count = 0, tile_excl = 0;
    if (tid < kRadix) {
#pragma unroll
        for (int w = 0; w < WARPS; ++w) tile_count += sm.hist[w * kRadix + tid];
        // (test hook: a "stalled" tile never publishes its reduction; its successors must re-reduce it themselves)
        if (pp.stall_every == 0 || (tile % pp.stall_every) != pp.stall_every - 1)
            st_relaxed_gpu_u16(agg16 + agg_index(tile, tid), kAggReady | tile_count);
    }
    if constexpr (HOT) hot_digit_publish(tile_count, sm.wmax);
    tile_excl = block_excl_scan_256<THREADS>(tile_count, sm.wtot);
    if (tid < kRadix) {
        uint32_t run = tile_excl;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) { const uint32_t c = sm.hist[w * kRadix + tid]; sm.hist[w * kRadix + tid] = run; run += c; }
    }
    if (tid == 0) sm.next_tile = kPersistent ? gridDim.x + drawn : num_tiles;  // every thread reads it before the barrier after the lookback
    __syncthreads();
    OSB_PHASE(3);

    // ---- chained scan with decoupled lookback (one thread per digit) -------------------------------------
    // Called once, after the rank phase and the next tile's loads: no warp of this CTA ranks while another looks back
    // (DESIGN §4.1).  It stays a lambda because the same statements written out at the call compile to another schedule.
    auto chained_scan = [&]() {
        if (tid < kRadix) {
            TileRereduce<KeyT> rr;
            // (an argsort's first pass re-reduces the tile it would have loaded: the caller's input)
            rr.in = (INDICES && (sm.plan_bits & kPlanBitsFirstIndices)) ? static_cast<const KeyT*>(pp.keys_in)
                    : (sm.plan_bits & 1u) ? buf1 : buf0;
            rr.tile_keys = T; rr.shift = shift; rr.mask = dmask;
            rr.encode = (sm.plan_bits >> 1) & kCodecEncodeOnLoad;
            rr.ca = static_cast<KeyT>(codec.a); rr.cb = static_cast<KeyT>(codec.b); rr.cd = static_cast<KeyT>(codec.d);
            const unsigned long long prior = lookback_wide<LOOK / 8, KeyT>(agg16, incl64, tile, tid, epoch, pp.spin_cap, rr);
            const bool swap = sm.plan_bits & 1u;
            KeyT* out = swap ? buf0 : buf1;
            uint32_t* out_val = swap ? val0 : val1;
            st_relaxed_gpu_u64(incl64 + static_cast<uint64_t>(tile) * kRadix + tid,
                               desc_pack(epoch, kFlagInclusive, prior + tile_count));
            const unsigned long long first = gbase[tid] + prior - tile_excl;  // element index (relative to out) of tile slot 0
            sm.keyptr[tid] = reinterpret_cast<unsigned long long>(out) + first * sizeof(KeyT);
            if constexpr (PAIRS) sm.valptr[tid] = reinterpret_cast<unsigned long long>(out_val) + first * sizeof(uint32_t);
            if (tid < 32) {
                // the all-ones padding of the ragged last tile sits at the end of the run of its digit: not live
                const uint32_t pad_digit = digit_of(static_cast<KeyT>(~static_cast<KeyT>(0)), shift, dmask);
                const uint32_t live = tile_count - ((tid == pad_digit && !full) ? (T - valid) : 0u);
                sm.run[tid] = tile_excl | (live << 16);
            }
        }
    };

    // ---- phase 2: the returning atomic hands every key its slot in the digit-sorted tile -----------------
    // (typed keys: the last pass stores the keys decoded; the digit was taken from the encoded key, and the scatter
    // below re-derives it from the tile, so the decoded form is produced only at the very end, in the store)
    // The rank phase recomputes each key's digit and counter address from the key (two ALU ops) instead of reusing the count
    // phase's: the compiler would otherwise keep the 32 addresses live across the barrier next to the 32 keys, which exceeds
    // 64 registers and spills to local memory on sm_90a.  Opaque copies of shift and mask make the reuse impossible.  (Not of
    // the histogram pointer: an opaque copy of it loses its shared-memory space, and the atomics become generic ones.  The
    // ballot mode spills either way, and more with the copies; the HOT instantiation has 128 registers and does not spill.)
    constexpr bool kRecompute = RANK_MODE == kRankAtomic && !HOT;
    const uint32_t rshift = kRecompute ? opaque_copy(&sm.digit_shift) : shift;
    const uint32_t rmask = kRecompute ? opaque_copy(&sm.digit_mask) : dmask;
    uint32_t hot = kNoHotDigit;
    if constexpr (HOT && RANK_MODE == kRankAtomic) hot = hot_digit_of_tile(sm.wmax, T);
    if (HOT && hot != kNoHotDigit) {
        uint32_t hot_run = __shfl_sync(0xffffffffu, wh[hot], 0);  // this warp's next slot of the hot digit (warp-uniform)
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t d = digit_of(key[i], rshift, rmask);
            const bool is_hot = d == hot;
            const uint32_t b = __ballot_sync(0xffffffffu, is_hot);
            uint32_t slot = hot_run + __popc(b & lt);
            if (!is_hot) slot = warp_rank_and_count<RANK_MODE>(wh, d, lt);
            hot_run += __popc(b);
            if constexpr (PAIRS) kv[slot] = make_uint2(static_cast<uint32_t>(key[i]), val[i]);
            else sm.sorted[slot] = key[i];
        }
    } else {
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t slot = warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], rshift, rmask), lt);
            if constexpr (PAIRS) kv[slot] = make_uint2(static_cast<uint32_t>(key[i]), val[i]);
            else sm.sorted[slot] = key[i];
        }
    }
    // this warp's histogram row is dead now (rows are warp-private from the count phase to here): clear it for the next tile
    __syncwarp();
    {
        uint4* r4 = reinterpret_cast<uint4*>(wh);
#pragma unroll
        for (int i = lane; i < kRadix / 4; i += 32) r4[i] = make_uint4(0, 0, 0, 0);
    }

    // ---- the next tile's loads, into the registers the rank phase has just freed ---------------------------
    // They are issued in front of the lookback, so that they fly during it and the scatter.
    // HOT: only the warps that do not look back (8-15) issue them here, the digit warps after the lookback -- faster for the
    // HOT instantiation on the H100 (entropy preset 5: 64.5 against 58 Gkeys/s); in the plain one the split spills.
    const uint32_t next = sm.next_tile;
    if constexpr (kPersistent) { if (!HOT || warp >= kRadix / 32) load_tile(next); }
    OSB_PHASE(4);
    chained_scan();
    OSB_PHASE(5);
    __syncthreads();
    OSB_PHASE(8);
    if constexpr (HOT) { if (warp < kRadix / 32) load_tile(next); }

    // ---- scatter -----------------------------------------------------------------------------------------
    // Few bins (a digit of <= 5 bits: the sharded exchange on log2(R) bits): runs are thousands of keys long, so
    // the stores are issued run by run in chunks that start on 128-byte boundaries of the DESTINATION -- every warp
    // store is then one full line (4 full sectors), which is what keeps NVLink peer stores at their aligned rate
    // (partial-sector peer stores run well below it; tools/microbench/p2p_store_ub.cu measures both).
    const bool dec = (sm.plan_bits >> 1) & kCodecDecodeOnStore;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    // pairs: a payload goes where its key goes, in the other output array (same element size: a constant byte distance)
    long long val_delta = 0;
    if constexpr (PAIRS) {
        const bool swap = sm.plan_bits & 1u;
        val_delta = reinterpret_cast<const char*>(swap ? val0 : val1) - reinterpret_cast<const char*>(swap ? buf0 : buf1);
    }
    auto slot_key = [&](uint32_t x) -> KeyT { if constexpr (PAIRS) return static_cast<KeyT>(kv[x].x); else return sm.sorted[x]; };
    (void)slot_key;
    if (pp.dbits <= 5) {
        const uint32_t nbins = 1u << pp.dbits;
        for (uint32_t b = 0; b < nbins; ++b) {
            const uint32_t rd = sm.run[b];
            const uint32_t lo = rd & 0xffffu, len = rd >> 16;
            if (len == 0) continue;
            const unsigned long long kp = sm.keyptr[b];
            constexpr uint32_t kLine = 128 / sizeof(KeyT);  // keys per 128-byte line
            const uint32_t ga = static_cast<uint32_t>((kp / sizeof(KeyT) + lo) & (kLine - 1));  // run start inside its line
            const uint32_t total = len + ga;
            for (uint32_t p = tid; p < total; p += THREADS) {
                if (p >= ga) {
                    const uint32_t x = lo + p - ga;
                    if constexpr (PAIRS) {
                        const uint2 e = kv[x];
                        KeyT k = static_cast<KeyT>(e.x);
                        if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
                        KeyT* dst = reinterpret_cast<KeyT*>(kp) + x;
                        st_scatter(dst, k);
                        st_scatter(reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(dst) + val_delta), e.y);
                    } else {
                        KeyT k = sm.sorted[x];
                        if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
                        st_scatter(reinterpret_cast<KeyT*>(kp) + x, k);
                    }
                }
            }
        }
    } else if (full && !dec) {  // branch-free: all shared loads of the unrolled body in flight together
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const uint32_t idx = j * THREADS + tid;
            if constexpr (PAIRS) {
                const uint2 e = kv[idx];
                KeyT* dst = reinterpret_cast<KeyT*>(sm.keyptr[digit_of(static_cast<KeyT>(e.x), shift, dmask)]) + idx;
                st_scatter(dst, static_cast<KeyT>(e.x));
                st_scatter(reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(dst) + val_delta), e.y);
            } else {
                const KeyT k = sm.sorted[idx];
                const uint32_t d = digit_of(k, shift, dmask);
                st_scatter(reinterpret_cast<KeyT*>(sm.keyptr[d]) + idx, k);
            }
        }
    } else {  // ragged last tile, or the last pass of a typed sort (keys leave decoded)
#pragma unroll 4
        for (int j = 0; j < K; ++j) {
            const uint32_t idx = j * THREADS + tid;
            if (idx < valid) {
                if constexpr (PAIRS) {
                    const uint2 e = kv[idx];
                    const KeyT k = static_cast<KeyT>(e.x);
                    KeyT* dst = reinterpret_cast<KeyT*>(sm.keyptr[digit_of(k, shift, dmask)]) + idx;
                    st_scatter(dst, dec ? codec_decode<KeyT>(k, ca, cb, cd) : k);
                    st_scatter(reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(dst) + val_delta), e.y);
                } else {
                    const KeyT k = sm.sorted[idx];
                    const uint32_t d = digit_of(k, shift, dmask);
                    st_scatter(reinterpret_cast<KeyT*>(sm.keyptr[d]) + idx, dec ? codec_decode<KeyT>(k, ca, cb, cd) : k);
                }
            }
        }
    }
    OSB_PHASE(6);
#if OSB_PHASE_PROBE
    if (tid == 0) atomicAdd(&g_phase[7], 1ull);
#endif
    if (!kPersistent || next >= num_tiles) break;
    tile = next;
    // No barrier here: the next tile's first shared-memory writes are this warp's own histogram row (cleared after its
    // rank) and next_tile (read by every thread before the barrier above); the sorted tile, the digit pointers and the run
    // table this scatter reads are rewritten only after the next tile's count barrier.
    }  // tile loop
}

// =====================================================================================================
// DigitBinningPass for (uint32 key, uint32 payload) pairs: 16,384-PAIR tiles (reference: OneSweep::DigitBinningPassPairs,
// OneSweep.cu:346-600, which like this kernel moves the payloads after the keys, through the same shared memory).
//
// The pairs instantiation of the kernel above holds keys AND payloads in registers and therefore stops at 8,192-pair
// tiles: twice the tiles, twice the per-tile work (ticket, histogram clear/reduce, chained scan, barriers) per pair.
// Here a tile is as large as for keys: the keys are ranked and scattered first; each thread remembers the tile slots
// of its 32 keys (14 bits each, two per register); the payloads are loaded into the registers the keys have left (the
// loads fly during the chained scan and the key scatter), go through the SAME 64 KB buffer at the remembered slots, and
// are scattered with the digit the key scatter has noted per slot (one byte).  100 KB of shared memory, two CTAs per SM.
// =====================================================================================================
// The PAIRS instantiation of digit_binning_wide_kernel (8,192-pair tiles, key and payload staged as one 64-bit word) is
// the default; -DOSB_PAIRS16K=1 selects this kernel.
#ifndef OSB_PAIRS16K
#define OSB_PAIRS16K 0
#endif
template <int WARPS, int K>
struct PairsSmem {
    static constexpr int THREADS = WARPS * 32;
    static constexpr int T = THREADS * K;
    alignas(16) uint32_t sorted[T];            // digit-sorted keys, later the payloads in the same order
    alignas(16) uint32_t hist[WARPS * kRadix];
    unsigned long long keyptr[kRadix];
    unsigned long long valptr[kRadix];
    alignas(16) unsigned char dig[T];          // digit of every tile slot (written by the key scatter)
    uint32_t wtot[kRadix / 32];
    uint32_t tile;
    uint32_t plan_bits;
};

template <int K, int WARPS, int RANK_MODE, int LOOK>
__global__ void __launch_bounds__(WARPS * 32, 2)
digit_binning_pairs_kernel(uint32_t* buf0, uint32_t* buf1, uint32_t* val0, uint32_t* val1, uint64_t n,
                           const unsigned long long* __restrict__ gbase, uint16_t* agg16, uint64_t* incl64,
                           uint32_t* ticket, PassParams pp, KeyCodec codec)
{
    using KeyT = uint32_t;
    using S = PairsSmem<WARPS, K>;
    constexpr int THREADS = S::THREADS;
    constexpr int T = S::T;
    static_assert(T <= 16384 && (K % 2) == 0, "slots are kept as 14-bit halves of a register");
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    uint32_t* wh = sm.hist + warp * kRadix;
    const uint32_t shift = pp.shift, epoch = pp.epoch;
    const uint32_t dmask = (1u << pp.dbits) - 1u;

    {
        uint4* h4 = reinterpret_cast<uint4*>(sm.hist);
        for (int i = tid; i < WARPS * kRadix / 4; i += THREADS) h4[i] = make_uint4(0, 0, 0, 0);
    }
    // tile id = blockIdx.x, every thread reads the plan itself (see digit_binning_wide_kernel)
    uint32_t my_bits = (codec.flags & (kCodecEncodeOnLoad | kCodecDecodeOnStore)) << 1;
    if (pp.plan != nullptr) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(pp.plan));
        SortPlan pl; pl.skip_mask = raw.x; pl.executed = raw.y; pl.first_exec = raw.z; pl.last_exec = raw.w;
        if ((pl.skip_mask >> pp.place) & 1u) return;
        my_bits = plan_src_is_alt(pl, pp.place) ? 1u : 0u;
        if (codec.flags & kCodecFromPlan)
            my_bits |= (pp.place == pl.first_exec ? kCodecEncodeOnLoad << 1 : 0u) | (pp.place == pl.last_exec ? kCodecDecodeOnStore << 1 : 0u);
    }
    if (tid == 0) { sm.plan_bits = my_bits; sm.tile = blockIdx.x; }
    const uint32_t tile = blockIdx.x;
    const uint64_t tile_base = static_cast<uint64_t>(tile) * T;
    const bool full = tile_base + T <= n;
    const uint32_t valid = full ? T : static_cast<uint32_t>(n - tile_base);
    const uint32_t warp_off = warp * (32 * K) + lane;

    // ---- keys ---------------------------------------------------------------------------------------------
    uint32_t key[K];  // later: the payloads
    {
        const KeyT* __restrict__ in = (my_bits & 1u) ? buf1 : buf0;
        if (full) {
#pragma unroll
            for (int i = 0; i < K; ++i) key[i] = ld_stream(in + tile_base + warp_off + i * 32);
        } else {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const uint32_t idx = warp_off + i * 32;
                key[i] = idx < valid ? in[tile_base + idx] : 0xffffffffu;  // pad: ranks last
            }
        }
    }
    __syncthreads();  // histograms cleared, plan_bits visible (the loads above are already in flight)
    if ((sm.plan_bits >> 1) & kCodecEncodeOnLoad) {
        const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
#pragma unroll
        for (int i = 0; i < K; ++i) {
            key[i] = codec_encode<KeyT>(key[i], ca, cb, cd);
            if (!full && warp_off + i * 32 >= valid) key[i] = 0xffffffffu;
        }
    }
#pragma unroll
    for (int i = 0; i < K; ++i) atomicAdd(&wh[digit_of(key[i], shift, dmask)], 1u);
    __syncthreads();

    uint32_t tile_count = 0, tile_excl = 0;
    if (tid < kRadix) {
#pragma unroll
        for (int w = 0; w < WARPS; ++w) tile_count += sm.hist[w * kRadix + tid];
        if (pp.stall_every == 0 || (tile % pp.stall_every) != pp.stall_every - 1)
            st_relaxed_gpu_u16(agg16 + agg_index(tile, tid), kAggReady | tile_count);
    }
    tile_excl = block_excl_scan_256<THREADS>(tile_count, sm.wtot);
    if (tid < kRadix) {
        uint32_t run = tile_excl;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) { const uint32_t c = sm.hist[w * kRadix + tid]; sm.hist[w * kRadix + tid] = run; run += c; }
    }
    __syncthreads();

    // ---- rank: keys to their slots; the slots are kept for the payloads --------------------------------------
    uint32_t slots[K / 2];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const uint32_t slot = warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], shift, dmask), lt);
        sm.sorted[slot] = key[i];
        if (i & 1) slots[i / 2] |= slot << 16; else slots[i / 2] = slot;
    }
    // ---- chained scan, AFTER the rank phase (as in digit_binning_wide_kernel): the keys are dead by now, so nothing of
    // theirs is spilled around the lookback, and no warp of this CTA ranks while the lookback's loads are in flight.  (With
    // the lookback ahead of the rank phase a build of this kernel produced rare order violations inside single warps at
    // n >= 2^28; the cause was not pinned down, this order has never shown one.)
    if (tid < kRadix) {
        TileRereduce<KeyT> rr;
        rr.in = (sm.plan_bits & 1u) ? buf1 : buf0; rr.tile_keys = T; rr.shift = shift; rr.mask = dmask;
        rr.encode = (sm.plan_bits >> 1) & kCodecEncodeOnLoad;
        rr.ca = static_cast<KeyT>(codec.a); rr.cb = static_cast<KeyT>(codec.b); rr.cd = static_cast<KeyT>(codec.d);
        const unsigned long long prior = lookback_wide<LOOK / 8, KeyT>(agg16, incl64, tile, tid, epoch, pp.spin_cap, rr);
        st_relaxed_gpu_u64(incl64 + static_cast<uint64_t>(tile) * kRadix + tid, desc_pack(epoch, kFlagInclusive, prior + tile_count));
        const bool swap = sm.plan_bits & 1u;
        const unsigned long long first = gbase[tid] + prior - tile_excl;
        sm.keyptr[tid] = reinterpret_cast<unsigned long long>(swap ? buf0 : buf1) + first * sizeof(KeyT);
        sm.valptr[tid] = reinterpret_cast<unsigned long long>(swap ? val0 : val1) + first * sizeof(uint32_t);
    }
    __syncthreads();

    // ---- payloads: loaded into the registers the keys have left; in flight during the key scatter (issued after the
    // chained scan, whose lookback needs the registers)
    asm volatile("" ::: "memory");
    {
        const uint32_t* __restrict__ in_val = (sm.plan_bits & 1u) ? val1 : val0;
        if (full) {
#pragma unroll
            for (int i = 0; i < K; ++i) key[i] = ld_stream(in_val + tile_base + warp_off + i * 32);
        } else {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const uint32_t idx = warp_off + i * 32;
                key[i] = idx < valid ? in_val[tile_base + idx] : 0u;
            }
        }
    }

    // ---- key scatter (notes the digit of every slot for the payload scatter) ---------------------------------
    {
        const bool dec = (sm.plan_bits >> 1) & kCodecDecodeOnStore;
        const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
        if (full && !dec) {
#pragma unroll
            for (int j = 0; j < K; ++j) {
                const uint32_t idx = j * THREADS + tid;
                const KeyT k = sm.sorted[idx];
                const uint32_t d = digit_of(k, shift, dmask);
                sm.dig[idx] = static_cast<unsigned char>(d);
                st_stream(reinterpret_cast<KeyT*>(sm.keyptr[d]) + idx, k);
            }
        } else {
#pragma unroll 4
            for (int j = 0; j < K; ++j) {
                const uint32_t idx = j * THREADS + tid;
                const KeyT k = sm.sorted[idx];
                const uint32_t d = digit_of(k, shift, dmask);
                sm.dig[idx] = static_cast<unsigned char>(d);
                if (idx < valid) st_stream(reinterpret_cast<KeyT*>(sm.keyptr[d]) + idx, dec ? codec_decode<KeyT>(k, ca, cb, cd) : k);
            }
        }
    }
    __syncthreads();  // every key has left the buffer

    // ---- payloads through the same buffer ---------------------------------------------------------------------
#pragma unroll
    for (int i = 0; i < K; ++i) sm.sorted[(slots[i / 2] >> (16 * (i & 1))) & 0xffffu] = key[i];
    __syncthreads();
    if (full) {
#pragma unroll
        for (int j = 0; j < K; ++j) {
            const uint32_t idx = j * THREADS + tid;
            st_stream(reinterpret_cast<uint32_t*>(sm.valptr[sm.dig[idx]]) + idx, sm.sorted[idx]);
        }
    } else {
#pragma unroll 4
        for (int j = 0; j < K; ++j) {
            const uint32_t idx = j * THREADS + tid;
            if (idx < valid) st_stream(reinterpret_cast<uint32_t*>(sm.valptr[sm.dig[idx]]) + idx, sm.sorted[idx]);
        }
    }
}

// =====================================================================================================
// DigitBinningPass, variant 1 ("ring"): persistent CTAs, partition tiles staged by TMA bulk copies (cp.async.bulk,
// SASS UBLKCP) into a two-deep shared-memory ring, with the wide kernel's ranking (two atomics per key), compact
// reductions and windowed lookback.  While a CTA ranks and scatters tile p, the keys of its next tile are already
// in flight (a full tile per CTA, all the time), so neither the ticket round trip nor the HBM load latency is on the
// per-tile critical path and the memory system sees a steady stream instead of one burst per CTA lifetime.  The ring
// costs shared memory: 8,192-key tiles (2 x 32 KB stages + 16 KB histograms, two CTAs per SM).
// Every CTA draws a ticket when a stage becomes free and consumes its tickets in order, so the lowest unfinished tile
// is always being processed by a resident CTA: the chained scan cannot deadlock (OneSweep.cu:181-184 argument).
// =====================================================================================================
template <typename KeyT, int K, int WARPS>
struct RingSmem {
    static constexpr int THREADS = WARPS * 32;
    static constexpr int T = THREADS * K;
    alignas(128) KeyT stage[2][T];              // TMA destination; after ranking, the digit-sorted tile of the same slot
    alignas(16) uint32_t hist[WARPS * kRadix];  // warp-private digit counters
    unsigned long long keyptr[kRadix];
    alignas(8) uint64_t bar[2];                 // "stage filled" mbarriers
    uint32_t tile[2];                           // ticket held in each stage
    uint32_t wtot[kRadix / 32];
};

// Lookback window in tiles (a multiple of 8: whole blocks of reductions, one inclusive probe per block); overridable for
// parameter sweeps (tools/sweep.sh).
#ifndef OSB_LOOK
#define OSB_LOOK 16
#endif
#ifndef OSB_PAIRS_LOOK  // (key, payload) pairs, either kernel; 8 beat 16 and 32 on the H100 with the default kernel's 8,192-pair tiles (DESIGN §4.2)
#define OSB_PAIRS_LOOK 8
#endif
#ifndef OSB_U64_LOOK    // 64-bit keys: 8,192-key tiles, twice the tiles per byte
#define OSB_U64_LOOK 32
#endif
#ifndef OSB_RING_K  // u32 geometry of the ring kernel, overridable for sweeps: keys per thread, resident CTAs per SM
#define OSB_RING_K 16
#define OSB_RING_MINB 2
#endif
template <typename KeyT, int K, int WARPS, int RANK_MODE, int LOOK>
__global__ void __launch_bounds__(WARPS * 32, (sizeof(KeyT) == 4 ? OSB_RING_MINB : 2))
digit_binning_ring_kernel(const KeyT* __restrict__ in, KeyT* __restrict__ out, uint64_t n, uint32_t shift,
                          const unsigned long long* __restrict__ gbase, uint16_t* agg16, uint64_t* incl64,
                          uint32_t* ticket, uint32_t epoch, uint32_t num_tiles)
{
    using S = RingSmem<KeyT, K, WARPS>;
    constexpr int THREADS = S::THREADS;
    constexpr int T = S::T;
    constexpr uint32_t TILE_BYTES = T * sizeof(KeyT);
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    uint32_t* wh = sm.hist + warp * kRadix;
    const uint32_t warp_off = warp * (32 * K) + lane;

    // a stage is filled by TMA only for full tiles; the (single) ragged last tile is read with guarded loads
    auto fetch = [&](int slot) {  // thread 0 only
        const uint32_t t = atomicAdd(ticket, 1u);
        sm.tile[slot] = t;
        if (t < num_tiles && static_cast<uint64_t>(t + 1) * T <= n) {
            mbar_expect_tx(&sm.bar[slot], TILE_BYTES);
            tma_load_1d(sm.stage[slot], in + static_cast<uint64_t>(t) * T, TILE_BYTES, &sm.bar[slot]);
        }
    };
    auto zero_hist = [&]() {
        uint4* h4 = reinterpret_cast<uint4*>(sm.hist);
        for (int i = tid; i < WARPS * kRadix / 4; i += THREADS) h4[i] = make_uint4(0, 0, 0, 0);
    };

    zero_hist();
    if (tid == 0) {
        mbar_init(&sm.bar[0], 1);
        mbar_init(&sm.bar[1], 1);
        fence_mbar_init();
        fetch(0);
        fetch(1);
    }
    __syncthreads();

    for (uint32_t it = 0;; ++it) {
        const int slot = it & 1;
        const uint32_t tile = sm.tile[slot];
        if (tile >= num_tiles) break;  // tickets only grow: nothing left for this CTA
        const uint64_t tile_base = static_cast<uint64_t>(tile) * T;
        const bool full = tile_base + T <= n;
        const uint32_t valid = full ? T : static_cast<uint32_t>(n - tile_base);
        KeyT* s_keys = sm.stage[slot];

        // ---- keys: shared (TMA-filled) -> registers, warp-striped so every LDS row is conflict-free ------
        KeyT key[K];
        if (full) {
            mbar_wait(&sm.bar[slot], (it >> 1) & 1u);
#pragma unroll
            for (int i = 0; i < K; ++i) key[i] = s_keys[warp_off + i * 32];
        } else {
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const uint32_t idx = warp_off + i * 32;
                key[i] = idx < valid ? in[tile_base + idx] : static_cast<KeyT>(~static_cast<KeyT>(0));
            }
        }

        // ---- phase 1: count ----------------------------------------------------------------------------
#pragma unroll
        for (int i = 0; i < K; ++i) atomicAdd(&wh[digit_of(key[i], shift)], 1u);
        __syncthreads();  // counts complete; every key of the stage is in registers

        uint32_t tile_count = 0, tile_excl = 0;
        if (tid < kRadix) {
#pragma unroll
            for (int w = 0; w < WARPS; ++w) tile_count += sm.hist[w * kRadix + tid];
            st_relaxed_gpu_u16(agg16 + agg_index(tile, tid), kAggReady | tile_count);
        }
        tile_excl = block_excl_scan_256<THREADS>(tile_count, sm.wtot);
        if (tid < kRadix) {
            uint32_t run = tile_excl;
#pragma unroll
            for (int w = 0; w < WARPS; ++w) { const uint32_t c = sm.hist[w * kRadix + tid]; sm.hist[w * kRadix + tid] = run; run += c; }
        }
        __syncthreads();

        // ---- phase 2: rank; the stage now receives the digit-sorted tile --------------------------------
#pragma unroll
        for (int i = 0; i < K; ++i) s_keys[warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], shift), lt)] = key[i];

        if (tid < kRadix) {
            TileRereduce<KeyT> rr;
            rr.in = in; rr.tile_keys = T; rr.shift = shift; rr.mask = kRadix - 1; rr.encode = false;
            rr.ca = rr.cb = rr.cd = 0;
            const unsigned long long prior = lookback_wide<LOOK / 8, KeyT>(agg16, incl64, tile, tid, epoch, 1u << 20, rr);
            st_relaxed_gpu_u64(incl64 + static_cast<uint64_t>(tile) * kRadix + tid,
                               desc_pack(epoch, kFlagInclusive, prior + tile_count));
            sm.keyptr[tid] = reinterpret_cast<unsigned long long>(out) + (gbase[tid] + prior - tile_excl) * sizeof(KeyT);
        }
        __syncthreads();

        // ---- scatter -----------------------------------------------------------------------------------
        if (full) {
#pragma unroll
            for (int j = 0; j < K; ++j) {
                const uint32_t idx = j * THREADS + tid;
                const KeyT k = s_keys[idx];
                st_stream(reinterpret_cast<KeyT*>(sm.keyptr[digit_of(k, shift)]) + idx, k);
            }
        } else {
#pragma unroll 4
            for (int j = 0; j < K; ++j) {
                const uint32_t idx = j * THREADS + tid;
                if (idx < valid) {
                    const KeyT k = s_keys[idx];
                    st_stream(reinterpret_cast<KeyT*>(sm.keyptr[digit_of(k, shift)]) + idx, k);
                }
            }
        }
        zero_hist();
        __syncthreads();  // stage drained, histograms cleared
        if (tid == 0) {
            fence_proxy_async_smem();  // generic-proxy accesses of the stage happen-before the next TMA write
            fetch(slot);
        }
        // the other stage's ticket was written at least one iteration (and one barrier) ago
    }
}

template <typename KeyT> struct RingGeom;
template <> struct RingGeom<uint32_t> { static constexpr int K = OSB_RING_K, WARPS = 16, LOOK = OSB_LOOK; };
template <> struct RingGeom<uint64_t> { static constexpr int K = 8,  WARPS = 16, LOOK = OSB_LOOK; };

template <typename KeyT, int RANK_MODE>
static cudaError_t launch_ring_variant(const void* in, void* out, uint64_t n, uint32_t shift, const unsigned long long* gbase,
                                       uint16_t* agg16, uint64_t* incl64, uint32_t* ticket, uint32_t epoch, int sm_count,
                                       cudaStream_t stream)
{
    using G = RingGeom<KeyT>;
    using S = RingSmem<KeyT, G::K, G::WARPS>;
    const uint64_t tiles = (n + S::T - 1) / S::T;
    const uint64_t cap = static_cast<uint64_t>(sm_count) * (sizeof(KeyT) == 4 ? OSB_RING_MINB : 2);
    const unsigned grid = static_cast<unsigned>(tiles < cap ? tiles : cap);
    auto kern = digit_binning_ring_kernel<KeyT, G::K, G::WARPS, RANK_MODE, G::LOOK>;
    kern<<<grid, S::THREADS, sizeof(S), stream>>>(static_cast<const KeyT*>(in), static_cast<KeyT*>(out), n, shift, gbase, agg16,
                                                   incl64, ticket, epoch, static_cast<uint32_t>(tiles));
    return cudaGetLastError();
}

template <typename KeyT, int RANK_MODE>
static cudaError_t set_ring_attr()
{
    using G = RingGeom<KeyT>;
    using S = RingSmem<KeyT, G::K, G::WARPS>;
    return cudaFuncSetAttribute(digit_binning_ring_kernel<KeyT, G::K, G::WARPS, RANK_MODE, G::LOOK>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(S)));
}

// Geometry and lookback window: 16,384-key tiles on 2 x 512 threads per SM (~82 KB of shared memory per CTA, inside
// H100's 227 KB per block and 228 KB per SM).  Re-swept on the H100 with tools/sweep.sh (DESIGN §4.2): 8,192-key tiles on
// 256 threads at 3 or 4 CTAs per SM are 11-18 % slower per sort -- twice the tiles double the chained scan's length, and the
// lookback grows to half of a CTA's life -- and the u32 window of 32 tiles is within run-to-run noise of 16.
template <typename KeyT, bool PAIRS> struct WideGeom;
#ifndef OSB_WIDE_WARPS  // geometry of the u32 keys-only kernel, overridable for sweeps
#define OSB_WIDE_WARPS 16
#define OSB_WIDE_K 32
#define OSB_WIDE_MINB 2
#endif
#ifndef OSB_PAIRS_WIDE_WARPS  // geometry of the u32 pairs kernel, overridable for sweeps
#define OSB_PAIRS_WIDE_WARPS 16
#define OSB_PAIRS_WIDE_K 16
#define OSB_PAIRS_WIDE_MINB 2
#endif
#ifndef OSB_U64_WARPS  // geometry of the u64 keys kernel, overridable for sweeps
#define OSB_U64_WARPS 16
#define OSB_U64_MINB 2
#endif
#ifndef OSB_U64_K
#define OSB_U64_K 16
#endif
template <> struct WideGeom<uint32_t, false> { static constexpr int K = OSB_WIDE_K, WARPS = OSB_WIDE_WARPS, MINB = OSB_WIDE_MINB, LOOK = OSB_LOOK; };
template <> struct WideGeom<uint32_t, true>  { static constexpr int K = OSB_PAIRS_WIDE_K, WARPS = OSB_PAIRS_WIDE_WARPS, MINB = OSB_PAIRS_WIDE_MINB, LOOK = OSB_PAIRS_LOOK; };
template <> struct WideGeom<uint64_t, false> { static constexpr int K = OSB_U64_K, WARPS = OSB_U64_WARPS, MINB = OSB_U64_MINB, LOOK = OSB_U64_LOOK; };

template <typename KeyT, bool PAIRS, int RANK_MODE, bool INDICES = false>
static cudaError_t launch_wide_variant(const void* in, void* out, const uint32_t* in_val, uint32_t* out_val, uint64_t n,
                                       uint32_t shift, const unsigned long long* gbase, uint16_t* agg16, uint64_t* incl64,
                                       uint32_t* ticket, uint32_t epoch, const BinningConfig& cfg, cudaStream_t stream)
{
    using G = WideGeom<KeyT, PAIRS>;
    using S = WideSmem<KeyT, PAIRS, G::K, G::WARPS>;
    const uint64_t tiles = (n + S::T - 1) / S::T;
    PassParams pp;
    pp.shift = shift;
    pp.dbits = cfg.digit_bits;
    pp.epoch = epoch;
    pp.place = cfg.place;
    pp.spin_cap = cfg.spin_cap;
    pp.stall_every = cfg.debug_stall_every;
    pp.plan = cfg.plan;
    pp.keys_in = cfg.argsort_in;
    // Persistent instantiations (all but the plain u64 keys and pairs passes, which run one CTA per tile): as many CTAs as can be resident
    // at once (capped by debug_max_ctas), at most one per tile; the tiles after the first of each CTA are handed out by
    // `ticket`, which the host zeroes before the pass.
    auto grid_for = [&](auto kernel, int& per_sm, bool persistent) -> unsigned {
        if (!persistent) return static_cast<unsigned>(tiles);
        if (per_sm == 0) {
            int b = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, kernel, S::THREADS, sizeof(S)) != cudaSuccess || b < 1) b = 1;
            per_sm = b;
        }
        uint64_t cap = static_cast<uint64_t>(cfg.sm_count) * per_sm;
        if (cfg.debug_max_ctas && cfg.debug_max_ctas < cap) cap = cfg.debug_max_ctas;
        return static_cast<unsigned>(tiles < cap ? tiles : cap);
    };
    auto kern = digit_binning_wide_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, G::LOOK, G::MINB, false, INDICES>;
    static int plain_per_sm = 0;  // (one value per instantiation of this function template)
    // with a device plan `in`/`out` are the caller's and the alt buffers (the kernel picks the direction); both are written
    kern<<<grid_for(kern, plain_per_sm, sizeof(KeyT) == 4 && !PAIRS), S::THREADS, sizeof(S), stream>>>(
        static_cast<KeyT*>(const_cast<void*>(in)), static_cast<KeyT*>(out), const_cast<uint32_t*>(in_val), out_val, n, gbase,
        agg16, incl64, ticket, pp, cfg.codec);
    if (cfg.plan != nullptr && cfg.hot_passes) {
        // the HOT instantiation of the same pass; returns at once unless the plan calls the pass hot, before drawing a ticket
        // (same geometry, one resident CTA per SM with up to 128 registers: no spills.  Two CTAs per SM at 64 registers
        // spill; 1,024 threads x 16 keys at 64 registers is slower than this)
        auto hot = digit_binning_wide_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, G::LOOK, G::MINB, true, INDICES>;
        static int hot_per_sm = 0;
        hot<<<grid_for(hot, hot_per_sm, true), S::THREADS, sizeof(S), stream>>>(
            static_cast<KeyT*>(const_cast<void*>(in)), static_cast<KeyT*>(out), const_cast<uint32_t*>(in_val), out_val, n, gbase,
            agg16, incl64, ticket, pp, cfg.codec);
    }
    return cudaGetLastError();
}

constexpr int kPairsK = 32, kPairsWarps = 16;

template <int RANK_MODE>
static cudaError_t launch_pairs_variant(const void* in, void* out, const uint32_t* in_val, uint32_t* out_val, uint64_t n,
                                        uint32_t shift, const unsigned long long* gbase, uint16_t* agg16, uint64_t* incl64,
                                        uint32_t* ticket, uint32_t epoch, const BinningConfig& cfg, cudaStream_t stream)
{
    using S = PairsSmem<kPairsWarps, kPairsK>;
    const uint64_t tiles = (n + S::T - 1) / S::T;
    PassParams pp;
    pp.shift = shift;
    pp.dbits = cfg.digit_bits;
    pp.epoch = epoch;
    pp.place = cfg.place;
    pp.spin_cap = cfg.spin_cap;
    pp.stall_every = cfg.debug_stall_every;
    pp.plan = cfg.plan;
    auto kern = digit_binning_pairs_kernel<kPairsK, kPairsWarps, RANK_MODE, OSB_PAIRS_LOOK>;
    kern<<<static_cast<unsigned>(tiles), S::THREADS, sizeof(S), stream>>>(
        static_cast<uint32_t*>(const_cast<void*>(in)), static_cast<uint32_t*>(out), const_cast<uint32_t*>(in_val), out_val, n,
        gbase, agg16, incl64, ticket, pp, cfg.codec);
    return cudaGetLastError();
}

template <int RANK_MODE>
static cudaError_t set_pairs_attr()
{
    using S = PairsSmem<kPairsWarps, kPairsK>;
    return cudaFuncSetAttribute(digit_binning_pairs_kernel<kPairsK, kPairsWarps, RANK_MODE, OSB_PAIRS_LOOK>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(S)));
}

template <typename KeyT, bool PAIRS, int RANK_MODE, bool INDICES = false>
static cudaError_t set_wide_attr()
{
    using G = WideGeom<KeyT, PAIRS>;
    using S = WideSmem<KeyT, PAIRS, G::K, G::WARPS>;
    cudaError_t e = cudaFuncSetAttribute(digit_binning_wide_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, G::LOOK, G::MINB, false, INDICES>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(S)));
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(digit_binning_wide_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, G::LOOK, G::MINB, true, INDICES>,
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(sizeof(S)));
    return e;
}

// ---- variant-0 geometry ------------------------------------------------------------------------------
template <typename KeyT, bool PAIRS> struct TileGeom;
template <> struct TileGeom<uint32_t, false> { static constexpr int K = 16, WARPS = 16; };
template <> struct TileGeom<uint32_t, true>  { static constexpr int K = 16, WARPS = 16; };
template <> struct TileGeom<uint64_t, false> { static constexpr int K = 8,  WARPS = 16; };

template <typename KeyT, bool PAIRS>
constexpr size_t tile_smem_bytes()
{
    using G = TileGeom<KeyT, PAIRS>;
    const size_t hist = static_cast<size_t>(G::WARPS) * kRadix * 4;
    const size_t keys = static_cast<size_t>(G::WARPS) * 32 * G::K * sizeof(KeyT);
    return hist > keys ? hist : keys;
}

template <typename KeyT, bool PAIRS, int RANK_MODE>
static cudaError_t launch_tile_variant(const void* in, void* out, const uint32_t* in_val, uint32_t* out_val, uint64_t n,
                                       uint32_t shift, const unsigned long long* gbase, uint64_t* desc, uint32_t* ticket,
                                       uint32_t epoch, cudaStream_t stream)
{
    using G = TileGeom<KeyT, PAIRS>;
    constexpr int T = G::WARPS * 32 * G::K;
    const uint64_t tiles = (n + T - 1) / T;
    auto kern = digit_binning_tile_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE>;
    kern<<<static_cast<unsigned>(tiles), G::WARPS * 32, tile_smem_bytes<KeyT, PAIRS>(), stream>>>(
        static_cast<const KeyT*>(in), static_cast<KeyT*>(out), in_val, out_val, n, shift, gbase, desc, ticket, epoch);
    return cudaGetLastError();
}

uint32_t binning_tile_keys(int key_bytes, bool pairs, const BinningConfig& cfg)
{
    if (cfg.variant == kVariantPersistent && !pairs)
        return key_bytes == 8 ? RingGeom<uint64_t>::K * RingGeom<uint64_t>::WARPS * 32 : RingGeom<uint32_t>::K * RingGeom<uint32_t>::WARPS * 32;
    if (cfg.variant == kVariantWide) {
        if (key_bytes == 8) return WideGeom<uint64_t, false>::K * WideGeom<uint64_t, false>::WARPS * 32;
        return pairs ? (OSB_PAIRS16K ? kPairsK * kPairsWarps * 32 : WideGeom<uint32_t, true>::K * WideGeom<uint32_t, true>::WARPS * 32)
                     : WideGeom<uint32_t, false>::K * WideGeom<uint32_t, false>::WARPS * 32;
    }
    if (key_bytes == 8) return TileGeom<uint64_t, false>::WARPS * 32 * TileGeom<uint64_t, false>::K;
    if (pairs) return TileGeom<uint32_t, true>::WARPS * 32 * TileGeom<uint32_t, true>::K;
    return TileGeom<uint32_t, false>::WARPS * 32 * TileGeom<uint32_t, false>::K;
}

template <typename KeyT, bool PAIRS, int RANK_MODE>
static cudaError_t set_tile_attr()
{
    using G = TileGeom<KeyT, PAIRS>;
    return cudaFuncSetAttribute(digit_binning_tile_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(tile_smem_bytes<KeyT, PAIRS>()));
}

static cudaError_t configure_segment_kernels();

cudaError_t configure_kernels()
{
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(global_histogram_kernel<uint32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(hist_smem_bytes<uint32_t>()))) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(global_histogram_kernel<uint64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(hist_smem_bytes<uint64_t>()))) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(global_histogram_kernel<uint32_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(hist_smem_bytes<uint32_t>()))) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(global_histogram_kernel<uint64_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(hist_smem_bytes<uint64_t>()))) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(global_histogram_bits_kernel<uint32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(hist_smem_bytes<uint32_t>()))) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(global_histogram_bits_kernel<uint64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(hist_smem_bytes<uint64_t>()))) != cudaSuccess) return e;
    if ((e = set_tile_attr<uint32_t, false, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_tile_attr<uint32_t, false, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_tile_attr<uint32_t, true, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_tile_attr<uint32_t, true, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_tile_attr<uint64_t, false, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_tile_attr<uint64_t, false, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_ring_attr<uint32_t, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_ring_attr<uint32_t, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_ring_attr<uint64_t, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_ring_attr<uint64_t, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint32_t, false, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint32_t, false, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint32_t, true, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint32_t, true, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint64_t, false, kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint64_t, false, kRankBallot>()) != cudaSuccess) return e;
    if ((e = set_wide_attr<uint32_t, true, kRankAtomic, true>()) != cudaSuccess) return e;  // argsort
    if ((e = set_wide_attr<uint32_t, true, kRankBallot, true>()) != cudaSuccess) return e;
    if ((e = set_pairs_attr<kRankAtomic>()) != cudaSuccess) return e;
    if ((e = set_pairs_attr<kRankBallot>()) != cudaSuccess) return e;
    return configure_segment_kernels();
}

cudaError_t launch_digit_binning(const void* in, void* out, const uint32_t* in_val, uint32_t* out_val, uint64_t n,
                                 int key_bytes, uint32_t shift, const unsigned long long* gbase_place, uint64_t* desc,
                                 uint16_t* agg16, uint32_t* ticket, uint32_t epoch, const BinningConfig& cfg,
                                 cudaStream_t stream)
{
    const bool pairs = in_val != nullptr;
    const bool ballot = cfg.rank_mode == kRankBallot;
    if (cfg.variant != kVariantWide && (cfg.codec.flags || cfg.plan != nullptr || cfg.debug_stall_every || cfg.argsort_in))
        return cudaErrorNotSupported;
    if (cfg.digit_bits < 1 || cfg.digit_bits > 8) return cudaErrorInvalidValue;
    // variants 0 and 1 always take 8-bit digits: a narrower digit is only correct for them when the bits above it do not exist
    if (cfg.variant != kVariantWide && cfg.digit_bits != 8 && shift + cfg.digit_bits != static_cast<uint32_t>(key_bytes) * 8u)
        return cudaErrorNotSupported;
    if (cfg.variant == kVariantWide) {
#define OSB_WIDE(KEYT, PAIRS)                                                                                          \
    (ballot ? launch_wide_variant<KEYT, PAIRS, kRankBallot>(in, out, in_val, out_val, n, shift, gbase_place, agg16, desc, \
                                                           ticket, epoch, cfg, stream)                                 \
            : launch_wide_variant<KEYT, PAIRS, kRankAtomic>(in, out, in_val, out_val, n, shift, gbase_place, agg16, desc, \
                                                           ticket, epoch, cfg, stream))
        if (cfg.argsort_in != nullptr) {  // argsort: the first executed pass reads argsort_in and makes the indices
            if (key_bytes != 4 || !pairs || cfg.plan == nullptr) return cudaErrorInvalidValue;
            return ballot ? launch_wide_variant<uint32_t, true, kRankBallot, true>(in, out, in_val, out_val, n, shift, gbase_place, agg16,
                                                                                  desc, ticket, epoch, cfg, stream)
                          : launch_wide_variant<uint32_t, true, kRankAtomic, true>(in, out, in_val, out_val, n, shift, gbase_place, agg16,
                                                                                  desc, ticket, epoch, cfg, stream);
        }
        if (key_bytes == 4 && pairs && OSB_PAIRS16K)
            return ballot ? launch_pairs_variant<kRankBallot>(in, out, in_val, out_val, n, shift, gbase_place, agg16, desc, ticket, epoch, cfg, stream)
                          : launch_pairs_variant<kRankAtomic>(in, out, in_val, out_val, n, shift, gbase_place, agg16, desc, ticket, epoch, cfg, stream);
        if (key_bytes == 4) return pairs ? OSB_WIDE(uint32_t, true) : OSB_WIDE(uint32_t, false);
        if (key_bytes == 8 && !pairs) return OSB_WIDE(uint64_t, false);
#undef OSB_WIDE
        return cudaErrorInvalidValue;
    }
    if (cfg.variant == kVariantPersistent && !pairs) {
        if (key_bytes == 4)
            return ballot ? launch_ring_variant<uint32_t, kRankBallot>(in, out, n, shift, gbase_place, agg16, desc, ticket, epoch, cfg.sm_count, stream)
                          : launch_ring_variant<uint32_t, kRankAtomic>(in, out, n, shift, gbase_place, agg16, desc, ticket, epoch, cfg.sm_count, stream);
        if (key_bytes == 8)
            return ballot ? launch_ring_variant<uint64_t, kRankBallot>(in, out, n, shift, gbase_place, agg16, desc, ticket, epoch, cfg.sm_count, stream)
                          : launch_ring_variant<uint64_t, kRankAtomic>(in, out, n, shift, gbase_place, agg16, desc, ticket, epoch, cfg.sm_count, stream);
    }
#define OSB_DISPATCH(KEYT, PAIRS)                                                                                   \
    (ballot ? launch_tile_variant<KEYT, PAIRS, kRankBallot>(in, out, in_val, out_val, n, shift, gbase_place, desc,  \
                                                           ticket, epoch, stream)                                   \
            : launch_tile_variant<KEYT, PAIRS, kRankAtomic>(in, out, in_val, out_val, n, shift, gbase_place, desc,  \
                                                           ticket, epoch, stream))
    if (key_bytes == 4) return pairs ? OSB_DISPATCH(uint32_t, true) : OSB_DISPATCH(uint32_t, false);
    if (key_bytes == 8 && !pairs) return OSB_DISPATCH(uint64_t, false);
#undef OSB_DISPATCH
    return cudaErrorInvalidValue;
}

// =====================================================================================================
// Segment sort / small-n path: ONE CTA sorts ONE segment of at most T keys entirely in shared memory (all digit passes:
// count, scan, rank, read back), one launch, no global histogram, no descriptors, no lookback.
//
// Reference: the reference's other contribution, SplitSort (SegSort/SplitSort/SplitSort.cuh:702-938), sorts many short
// segments by binning them by length; and a OneSweep::Sort of n < ~2^16 keys is launch-bound (6 launches + memsets,
// SURVEY 8f rank 4).  Here both are the same kernel: osb200_segmented_sort_u32 runs it over an array of segment offsets
// (grid-stride over the segments), and every osb200_sort_* call with n <= T takes it as its single segment [0, n).
// The ranking is the DigitBinningPass's (warp-private histograms, returning atomic = slot), so the sort is stable and typed
// keys / bit ranges cost nothing extra.  Segments longer than T are not this kernel's business (the caller sorts them with
// the ordinary path).
// =====================================================================================================
template <typename KeyT, bool PAIRS, int K, int WARPS>
struct SegSmem {
    static constexpr int THREADS = WARPS * 32;
    static constexpr int T = THREADS * K;
    alignas(16) KeyT sorted[T];
    alignas(16) uint32_t sorted_val[PAIRS ? T : 4];
    alignas(16) uint32_t hist[WARPS * kRadix];
    uint32_t wtot[kRadix / 32];
};

// INDICES (argsort of the single segment): the keys come from keys_in, every payload is the key's position in the segment.
// max_len: the caller's max_segment_len (<= T); longer segments are left as they are.
template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE, bool INDICES = false>
__global__ void __launch_bounds__(WARPS * 32)
segment_sort_kernel(KeyT* keys, uint32_t* vals, const unsigned long long* __restrict__ seg_off, uint64_t num_segments,
                    uint64_t single_n, uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits, KeyCodec codec,
                    const KeyT* __restrict__ keys_in)
{
    static_assert(!INDICES || PAIRS, "the indices are the payloads");
    using S = SegSmem<KeyT, PAIRS, K, WARPS>;
    constexpr int THREADS = S::THREADS;
    constexpr int T = S::T;
    static_assert(WARPS >= 8, "one thread per digit");
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    uint32_t* wh = sm.hist + warp * kRadix;
    const uint32_t warp_off = warp * (32 * K) + lane;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = codec.flags & kCodecEncodeOnLoad, dec = codec.flags & kCodecDecodeOnStore;

    for (uint64_t seg = blockIdx.x; seg < num_segments; seg += gridDim.x) {
        const uint64_t lo = seg_off ? seg_off[seg] : 0ull;
        const uint64_t hi = seg_off ? seg_off[seg + 1] : single_n;
        // empty / one key / longer than max_segment_len or the geometry (both the caller's contract: left untouched)
        if (hi <= lo + 1 || hi - lo > static_cast<uint64_t>(max_len) || hi - lo > static_cast<uint64_t>(T)) continue;
        const uint32_t len = static_cast<uint32_t>(hi - lo);

        KeyT key[K];
        uint32_t val[PAIRS ? K : 1];
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t idx = warp_off + i * 32;
            KeyT k = idx < len ? (INDICES ? keys_in : keys)[lo + idx] : static_cast<KeyT>(0);
            if (enc) k = codec_encode<KeyT>(k, ca, cb, cd);
            key[i] = idx < len ? k : static_cast<KeyT>(~static_cast<KeyT>(0));  // padding ranks last in every pass
            if constexpr (PAIRS) val[i] = INDICES ? idx : idx < len ? vals[lo + idx] : 0u;
        }

        for (uint32_t p = 0; p < places; ++p) {
            const uint32_t shift = begin_bit + 8u * p;
            const uint32_t dmask = p == places - 1 ? (1u << last_bits) - 1u : 255u;
            __syncthreads();  // the previous pass (or segment) has read the tile back
            {
                uint4* h4 = reinterpret_cast<uint4*>(sm.hist);
                for (int i = tid; i < WARPS * kRadix / 4; i += THREADS) h4[i] = make_uint4(0, 0, 0, 0);
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < K; ++i) atomicAdd(&wh[digit_of(key[i], shift, dmask)], 1u);
            __syncthreads();
            uint32_t tile_count = 0;
            if (tid < kRadix) {
#pragma unroll
                for (int w = 0; w < WARPS; ++w) tile_count += sm.hist[w * kRadix + tid];
            }
            const uint32_t tile_excl = block_excl_scan_256<THREADS>(tile_count, sm.wtot);
            if (tid < kRadix) {
                uint32_t run = tile_excl;
#pragma unroll
                for (int w = 0; w < WARPS; ++w) { const uint32_t c = sm.hist[w * kRadix + tid]; sm.hist[w * kRadix + tid] = run; run += c; }
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < K; ++i) {
                const uint32_t slot = warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], shift, dmask), lt);
                sm.sorted[slot] = key[i];
                if constexpr (PAIRS) sm.sorted_val[slot] = val[i];
            }
            __syncthreads();
            if (p + 1 < places) {  // back into registers in tile order for the next digit
#pragma unroll
                for (int i = 0; i < K; ++i) {
                    key[i] = sm.sorted[warp_off + i * 32];
                    if constexpr (PAIRS) val[i] = sm.sorted_val[warp_off + i * 32];
                }
            }
        }
        // the padding sits behind the `len` real keys
        for (uint32_t idx = tid; idx < len; idx += THREADS) {
            KeyT k = sm.sorted[idx];
            if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
            keys[lo + idx] = k;
            if constexpr (PAIRS) vals[lo + idx] = sm.sorted_val[idx];
        }
    }
}

// three geometries per key type (SIZE 0 / 1 / 2): tiny and short segments (many resident CTAs; the work per segment is
// proportional to the geometry's capacity, padding included) and up to a DigitBinningPass tile
template <typename KeyT, int SIZE> struct SegGeomN;
template <> struct SegGeomN<uint32_t, 0> { static constexpr int K = 1,  WARPS = 8; };   //    256 keys, 256 threads
template <> struct SegGeomN<uint32_t, 1> { static constexpr int K = 8,  WARPS = 8; };   //  2,048 keys, 256 threads
template <> struct SegGeomN<uint32_t, 2> { static constexpr int K = 32, WARPS = 16; };  // 16,384 keys, 512 threads
template <> struct SegGeomN<uint64_t, 0> { static constexpr int K = 1,  WARPS = 8; };   //    256 keys
template <> struct SegGeomN<uint64_t, 1> { static constexpr int K = 8,  WARPS = 8; };   //  2,048 keys
template <> struct SegGeomN<uint64_t, 2> { static constexpr int K = 16, WARPS = 16; };  //  8,192 keys
template <typename KeyT, int SIZE> constexpr uint32_t seg_cap() { return SegGeomN<KeyT, SIZE>::K * SegGeomN<KeyT, SIZE>::WARPS * 32; }

uint32_t segment_sort_capacity(int key_bytes, bool small)
{
    if (key_bytes == 8) return small ? seg_cap<uint64_t, 1>() : seg_cap<uint64_t, 2>();
    return small ? seg_cap<uint32_t, 1>() : seg_cap<uint32_t, 2>();
}

template <typename KeyT, bool PAIRS, int SIZE, int RANK_MODE, bool INDICES = false>
static cudaError_t seg_attr()
{
    using G = SegGeomN<KeyT, SIZE>;
    return cudaFuncSetAttribute(segment_sort_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, INDICES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(sizeof(SegSmem<KeyT, PAIRS, G::K, G::WARPS>)));
}
static cudaError_t configure_segment_kernels()
{
    cudaError_t e;
#define OSB_SEG_ATTR(KEYT, PAIRS)                                                                          \
    if ((e = seg_attr<KEYT, PAIRS, 0, kRankAtomic>()) != cudaSuccess) return e;                             \
    if ((e = seg_attr<KEYT, PAIRS, 0, kRankBallot>()) != cudaSuccess) return e;                             \
    if ((e = seg_attr<KEYT, PAIRS, 1, kRankAtomic>()) != cudaSuccess) return e;                             \
    if ((e = seg_attr<KEYT, PAIRS, 1, kRankBallot>()) != cudaSuccess) return e;                             \
    if ((e = seg_attr<KEYT, PAIRS, 2, kRankAtomic>()) != cudaSuccess) return e;                             \
    if ((e = seg_attr<KEYT, PAIRS, 2, kRankBallot>()) != cudaSuccess) return e;
    OSB_SEG_ATTR(uint32_t, false)
    OSB_SEG_ATTR(uint32_t, true)
    OSB_SEG_ATTR(uint64_t, false)
#undef OSB_SEG_ATTR
    // argsort: the single segment of a sort of at most one tile
    if ((e = seg_attr<uint32_t, true, 2, kRankAtomic, true>()) != cudaSuccess) return e;
    if ((e = seg_attr<uint32_t, true, 2, kRankBallot, true>()) != cudaSuccess) return e;
    return cudaSuccess;
}

template <typename KeyT, bool PAIRS, int SIZE, bool INDICES = false>
static cudaError_t launch_seg(void* keys, uint32_t* vals, const unsigned long long* seg_off, uint64_t num_segments, uint64_t single_n,
                              uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits, const KeyCodec& codec,
                              int rank_mode, int sm_count, cudaStream_t stream, const void* keys_in = nullptr)
{
    using G = SegGeomN<KeyT, SIZE>;
    using S = SegSmem<KeyT, PAIRS, G::K, G::WARPS>;
    const uint64_t cap = static_cast<uint64_t>(sm_count) * (SIZE == 2 ? 2 : 8);
    const unsigned grid = static_cast<unsigned>(num_segments < cap ? num_segments : cap);
    const KeyT* in = static_cast<const KeyT*>(keys_in);
    if (rank_mode == kRankBallot)
        segment_sort_kernel<KeyT, PAIRS, G::K, G::WARPS, kRankBallot, INDICES><<<grid, S::THREADS, sizeof(S), stream>>>(
            static_cast<KeyT*>(keys), vals, seg_off, num_segments, single_n, max_len, begin_bit, places, last_bits, codec, in);
    else
        segment_sort_kernel<KeyT, PAIRS, G::K, G::WARPS, kRankAtomic, INDICES><<<grid, S::THREADS, sizeof(S), stream>>>(
            static_cast<KeyT*>(keys), vals, seg_off, num_segments, single_n, max_len, begin_bit, places, last_bits, codec, in);
    return cudaGetLastError();
}

cudaError_t launch_segment_sort(void* keys, uint32_t* vals, int key_bytes, const unsigned long long* seg_off, uint64_t num_segments,
                                uint64_t single_n, uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits,
                                const KeyCodec* codec_in, int rank_mode, int sm_count, cudaStream_t stream, const void* keys_in)
{
    if (num_segments == 0) return cudaSuccess;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    if (keys_in != nullptr) {  // argsort: one segment of up to a tile, in the largest geometry (the only one instantiated for it)
        if (key_bytes != 4 || !vals || seg_off || num_segments != 1 || max_len > seg_cap<uint32_t, 2>()) return cudaErrorInvalidValue;
        return launch_seg<uint32_t, true, 2, true>(keys, vals, nullptr, 1, single_n, max_len, begin_bit, places, last_bits, codec,
                                                   rank_mode, sm_count, stream, keys_in);
    }
    const int size = max_len <= (key_bytes == 8 ? seg_cap<uint64_t, 0>() : seg_cap<uint32_t, 0>()) ? 0
                     : max_len <= segment_sort_capacity(key_bytes, true) ? 1 : 2;
    if (max_len > segment_sort_capacity(key_bytes, false)) return cudaErrorInvalidValue;
#define OSB_SEG_ARGS keys, vals, seg_off, num_segments, single_n, max_len, begin_bit, places, last_bits, codec, rank_mode, sm_count, stream
#define OSB_SEG(KEYT, PAIRS) \
    (size == 0 ? launch_seg<KEYT, PAIRS, 0>(OSB_SEG_ARGS) : size == 1 ? launch_seg<KEYT, PAIRS, 1>(OSB_SEG_ARGS) : launch_seg<KEYT, PAIRS, 2>(OSB_SEG_ARGS))
    if (key_bytes == 4) return vals ? OSB_SEG(uint32_t, true) : OSB_SEG(uint32_t, false);
    if (key_bytes == 8 && !vals) return OSB_SEG(uint64_t, false);
#undef OSB_SEG_ARGS
#undef OSB_SEG
    return cudaErrorInvalidValue;
}

// =====================================================================================================
// Validate: adjacent-inversion count (reference: UtilityKernels.cuh:403-429)
// =====================================================================================================
template <typename KeyT>
__global__ void __launch_bounds__(256)
validate_kernel(const KeyT* __restrict__ keys, uint64_t n, unsigned long long* err_count)
{
    unsigned long long bad = 0;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i + 1 < n; i += stride)
        bad += keys[i] > keys[i + 1];
    for (int o = 16; o > 0; o >>= 1) bad += __shfl_down_sync(0xffffffffu, bad, o);
    if ((threadIdx.x & 31) == 0 && bad) atomicAdd(err_count, bad);
}

cudaError_t launch_validate(const void* keys, uint64_t n, int key_bytes, unsigned long long* err_count, int sm_count,
                            cudaStream_t stream)
{
    const unsigned grid = static_cast<unsigned>(sm_count) * 8;
    if (key_bytes == 4) validate_kernel<uint32_t><<<grid, 256, 0, stream>>>(static_cast<const uint32_t*>(keys), n, err_count);
    else validate_kernel<uint64_t><<<grid, 256, 0, stream>>>(static_cast<const uint64_t*>(keys), n, err_count);
    return cudaGetLastError();
}

// =====================================================================================================
// InitRandom: the reference's input generator (UtilityKernels.cuh:26-33,53-117), restated from its
// published recurrences (hybrid Tausworthe + LCG, GPU Gems 3 ch. 37).  Test/bench utility, not on the hot path.
// =====================================================================================================
constexpr uint32_t kGenStreams = 65536;

struct HybridTaus {
    uint32_t a, b, c, l;
    __device__ __forceinline__ uint32_t next()
    {
        a = ((a & 0xfffffffeu) << 12) ^ (((a << 13) ^ a) >> 19);
        b = ((b & 0xfffffff8u) << 4) ^ (((b << 2) ^ b) >> 25);
        c = ((c & 0xfffffff0u) << 17) ^ (((c << 3) ^ c) >> 11);
        l = l * 1664525u + 1013904223u;
        return a ^ b ^ c ^ l;
    }
};

__global__ void __launch_bounds__(256)
init_random_kernel(uint32_t* __restrict__ keys, uint32_t* __restrict__ payload, uint64_t n, uint32_t and_count,
                   uint32_t seed, bool payload_is_index)
{
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;  // stream id, 0..65535
    HybridTaus s{(g * 4u) * seed, (g * 4u + 1u) * seed, (g * 4u + 2u) * seed, (g * 4u + 3u) * seed};
    (void)s.next();  // one warm-up step
    for (uint64_t i = g; i < n; i += kGenStreams) {
        uint32_t t = 0xffffffffu;
        for (uint32_t k = 0; k <= and_count; ++k) t &= s.next();
        keys[i] = t;
        if (payload) payload[i] = payload_is_index ? static_cast<uint32_t>(i) : t;
    }
}

cudaError_t launch_init_random(uint32_t* keys, uint32_t* payload, uint64_t n, uint32_t and_count, uint32_t seed,
                               bool payload_is_index, cudaStream_t stream)
{
    init_random_kernel<<<kGenStreams / 256, 256, 0, stream>>>(keys, payload, n, and_count, seed, payload_is_index);
    return cudaGetLastError();
}

// =====================================================================================================
// Self-test of the hardware property RankMode::kRankAtomic relies on
// =====================================================================================================
// Production geometry on purpose: 512 threads = 16 warps with a 256-bin histogram each, two CTAs per SM, batches of 16
// back-to-back returning atomics per thread interleaved with data-dependent shared-memory stores (the rank phase of
// digit_binning_wide_kernel), digits from uniform down to "every lane the same".  The ballot formulation on a second
// histogram is the reference answer.
constexpr int kSelfTestWarps = 16;
__global__ void __launch_bounds__(kSelfTestWarps * 32, 2)
atomic_order_selftest_kernel(unsigned long long* mismatches)
{
    __shared__ uint32_t s_hist[kSelfTestWarps * kRadix];
    __shared__ uint32_t s_ref[kSelfTestWarps * kRadix];
    __shared__ volatile uint32_t s_scratch[kSelfTestWarps * 32 * 4];  // stands in for the sorted tile: random-bank STS traffic
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* wh = s_hist + warp * kRadix;
    uint32_t* wr = s_ref + warp * kRadix;
    uint32_t s = (blockIdx.x * blockDim.x + threadIdx.x) * 2654435761u + 12345u;
    const uint32_t lt = lanemask_lt();
    unsigned long long bad = 0;
    constexpr int B = 16;
    for (int it = 0; it < 24; ++it) {
        for (int i = lane; i < kRadix; i += 32) { wh[i] = 0; wr[i] = 0; }
        __syncwarp();
        for (int batch = 0; batch < 2; ++batch) {
            uint32_t d[B], got[B];
#pragma unroll
            for (int i = 0; i < B; ++i) {
                uint32_t x = 255u;
                const int draws = 1 + (it % 6);  // entropy sweep: uniform digits down to heavy collisions
                for (int k = 0; k < draws; ++k) { s = s * 1664525u + 1013904223u; x &= (s >> 13); }
                if (it % 6 == 5) x = (it + i) & 255u;  // every lane the same digit
                d[i] = x;
            }
#pragma unroll
            for (int i = 0; i < B; ++i) {
                got[i] = warp_rank_and_count<kRankAtomic>(wh, d[i], lt);
                s_scratch[(got[i] * 37u + d[i] * 5u + threadIdx.x) & (kSelfTestWarps * 32 * 4 - 1)] = d[i];
            }
#pragma unroll
            for (int i = 0; i < B; ++i) {
                const uint32_t want = warp_rank_and_count<kRankBallot>(wr, d[i], lt);
                bad += (got[i] != want);
                __syncwarp();
            }
        }
    }
    if (bad) atomicAdd(mismatches, bad);
}

cudaError_t launch_atomic_order_selftest(unsigned long long* mismatches, int sm_count, cudaStream_t stream)
{
    atomic_order_selftest_kernel<<<sm_count * 2, kSelfTestWarps * 32, 0, stream>>>(mismatches);
    return cudaGetLastError();
}

}  // namespace osb
