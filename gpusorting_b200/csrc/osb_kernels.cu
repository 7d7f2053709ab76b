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
#include <type_traits>

#include "osb_kernels.cuh"
#include "osb_common.cuh"

namespace osb {

// =====================================================================================================
// Host-side dispatch.  Each kernel family lists the instantiations it is compiled for once, as a TypeList of shapes;
// configure_kernels() walks the lists and the launchers find the shape that matches their run-time arguments in the same
// list, so every launched instantiation is a configured one.
// =====================================================================================================
template <typename... Ts> struct TypeList {};

// f(T{}) for every type of the list, in order, until one returns an error
template <typename... Ts, typename F>
static cudaError_t for_each_type(TypeList<Ts...>, F&& f)
{
    cudaError_t e = cudaSuccess;
    (void)(((e = f(Ts{})) == cudaSuccess) && ...);
    return e;
}

// f(T{}) for the first type of the list that `match` accepts; cudaErrorInvalidValue if there is none
template <typename... Ts, typename M, typename F>
static cudaError_t find_type(TypeList<Ts...>, M&& match, F&& f)
{
    cudaError_t e = cudaErrorInvalidValue;
    (void)((match(Ts{}) && ((e = f(Ts{})), true)) || ...);
    return e;
}

// The key type of the list that is key_bytes wide: f(KeyT{}); cudaErrorInvalidValue if the launcher has none that wide.
template <typename... Keys, typename F>
static cudaError_t with_key_type(TypeList<Keys...> keys, int key_bytes, F&& f)
{
    return find_type(keys, [&](auto k) { return key_bytes == static_cast<int>(sizeof(k)); }, f);
}

// The rank mode as a compile-time constant: f(std::integral_constant<int, RANK_MODE>{}).
template <typename F>
static cudaError_t with_rank_mode(int rank_mode, F&& f)
{
    return rank_mode == kRankBallot ? f(std::integral_constant<int, kRankBallot>{}) : f(std::integral_constant<int, kRankAtomic>{});
}

// ceil(work / per_cta) CTAs, at least one and at most cap
static unsigned capped_grid(uint64_t work, uint64_t per_cta, uint64_t cap)
{
    uint64_t want = (work + per_cta - 1) / per_cta;
    if (want < 1) want = 1;
    return static_cast<unsigned>(want < cap ? want : cap);
}

// Kern<<<grid, THREADS, SMEM, stream>>>(args...) on the CTAs that are resident on the device at once, at most max_ctas of
// them: kernels that grid-stride over their work (or over lists whose length only the device knows) want every CTA
// resident from the start.  The occupancy is queried once per process and kernel: the static belongs to this
// instantiation, and kernels with the same signature are still different template arguments.
constexpr uint64_t kAllResident = ~0ull;
template <auto Kern, int THREADS, size_t SMEM, typename... Args>
static cudaError_t launch_resident(uint64_t max_ctas, int sm_count, cudaStream_t stream, Args... args)
{
    static const int per_sm = [] {
        int b = 0;
        return cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, Kern, THREADS, SMEM) == cudaSuccess ? b : 0;
    }();
    if (per_sm <= 0) return cudaErrorLaunchOutOfResources;
    const uint64_t ctas = static_cast<uint64_t>(per_sm) * sm_count;
    Kern<<<static_cast<unsigned>(max_ctas < ctas ? max_ctas : ctas), THREADS, SMEM, stream>>>(args...);
    return cudaGetLastError();
}

template <typename K>
static cudaError_t set_smem(K* kernel, size_t bytes)
{
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
}

// Opts both rank modes of a shape's kernel (and of its HOT twin, if it has one) into the shape's dynamic shared memory.
template <typename Shape>
static cudaError_t configure_shape(Shape)
{
    cudaError_t e = set_smem(Shape::template kernel<kRankAtomic>(), Shape::smem);
    if (e == cudaSuccess) e = set_smem(Shape::template kernel<kRankBallot>(), Shape::smem);
    if constexpr (Shape::has_hot) {
        if (e == cudaSuccess) e = set_smem(Shape::template kernel<kRankAtomic, true>(), Shape::smem);
        if (e == cudaSuccess) e = set_smem(Shape::template kernel<kRankBallot, true>(), Shape::smem);
    }
    return e;
}

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
template <> struct HistGeom<uint16_t> { static constexpr int COLS = 32; };  // 2 places x 256 digits x 32 columns: 64 KB

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
    } else if constexpr (sizeof(KeyT) == 2) {
        const uint16_t a = static_cast<uint16_t>(c.a), b = static_cast<uint16_t>(c.b), d = static_cast<uint16_t>(c.d);
        auto enc2 = [&](uint32_t w) {  // the two keys of a 32-bit word
            return static_cast<uint32_t>(codec_encode<uint16_t>(static_cast<uint16_t>(w), a, b, d)) |
                   (static_cast<uint32_t>(codec_encode<uint16_t>(static_cast<uint16_t>(w >> 16), a, b, d)) << 16);
        };
        v.x = enc2(v.x); v.y = enc2(v.y); v.z = enc2(v.z); v.w = enc2(v.w);
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
                        int places = 0, uint32_t last_mask = 255u, const SortPlan* gate = nullptr)
{
    if (gate != nullptr && (gate->skip_mask & kPlanFusedKept)) return;  // fallback of a fused sort whose first pass stood
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

using HistKeys = TypeList<uint16_t, uint32_t, uint64_t>;  // global_histogram_kernel of whole keys
using HistBitsKeys = TypeList<uint32_t, uint64_t>;        // its MASKED form and global_histogram_bits_kernel (bit-range sorts)

template <typename KeyT, bool MASKED>
static cudaError_t launch_histogram_vec(const void* keys, uint64_t n, unsigned long long* ghist, int sm_count, cudaStream_t stream,
                                        const KeyCodec& codec, int places = 0, uint32_t last_mask = 255u,
                                        const SortPlan* gate = nullptr)
{
    const unsigned grid = capped_grid(n / (16 / sizeof(KeyT)), kHistThreads, sm_count);
    global_histogram_kernel<KeyT, MASKED><<<grid, kHistThreads, hist_smem_bytes<KeyT>(), stream>>>(
        static_cast<const KeyT*>(keys), n, ghist, codec, places, last_mask, gate);
    return cudaGetLastError();
}

cudaError_t launch_global_histogram(const void* keys, uint64_t n, int key_bytes, unsigned long long* ghist,
                                    int sm_count, cudaStream_t stream, const KeyCodec* codec_in, const SortPlan* gate)
{
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    return with_key_type(HistKeys{}, key_bytes, [&](auto k) {
        return launch_histogram_vec<decltype(k), false>(keys, n, ghist, sm_count, stream, codec, 0, 255u, gate);
    });
}

// The fallback of a fused sort clears what the fused pass left for place 0's classic pass, which runs on the same
// reductions and the same epoch: place 0's reductions and the descriptors of the tiles it reached -- at most its first
// CTAs' tiles and those drawn from its ticket (few when it stopped early).  Returns at once when the fused pass stood.
__global__ void __launch_bounds__(512)
fused_fallback_zero_kernel(const SortPlan* __restrict__ plan, const uint32_t* __restrict__ ticket, uint32_t ctas, uint64_t tiles,
                           uint4* __restrict__ agg16, uint4* __restrict__ desc)
{
    if (plan->skip_mask & kPlanFusedKept) return;
    uint64_t reached = static_cast<uint64_t>(ctas) + *ticket;
    if (reached > tiles) reached = tiles;
    const uint64_t agg_vecs = (reached + 7) / 8 * 8 * kRadix * sizeof(uint16_t) / 16;  // whole blocks of 8 tiles
    const uint64_t desc_vecs = reached * kRadix * sizeof(uint64_t) / 16;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < agg_vecs + desc_vecs; i += stride)
        (i < agg_vecs ? agg16[i] : desc[i - agg_vecs]) = make_uint4(0, 0, 0, 0);
}

cudaError_t launch_fused_fallback_zero(const SortPlan* plan, const uint32_t* ticket, uint32_t ctas, uint64_t tiles, uint16_t* agg16,
                                       uint64_t* desc, int sm_count, cudaStream_t stream)
{
    fused_fallback_zero_kernel<<<static_cast<unsigned>(sm_count) * 4, 512, 0, stream>>>(plan, ticket, ctas, tiles,
                                                                                         reinterpret_cast<uint4*>(agg16),
                                                                                         reinterpret_cast<uint4*>(desc));
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
    const unsigned grid = capped_grid(n, kHistThreads * 4, static_cast<uint64_t>(sm_count) * 2);
    return with_key_type(TypeList<uint32_t, uint64_t>{}, key_bytes, [&](auto k) {
        using KeyT = decltype(k);
        digit_histogram_kernel<KeyT><<<grid, kHistThreads, 0, stream>>>(static_cast<const KeyT*>(keys), n, shift, hist256);
        return cudaGetLastError();
    });
}

// =====================================================================================================
// Scan: exclusive prefix over the 256 bins of each digit place (reference: OneSweep::Scan, OneSweep.cu:125-162), and --
// new here -- the device-side launch plan: a place whose histogram has ONE non-empty bin (all n keys share that digit)
// is marked skipped, so its DigitBinningPass exits at once; the passes derive their source/destination from the
// number of executed passes before them, and a final copy moves the result home if that number is odd.
// One CTA walks the (at most 8) places: the plan needs all of them.
// =====================================================================================================
// Fused sorts (DESIGN §4.12): kScanFused follows the fused first pass and adds kPlanFusedKept to the plan when that pass's
// result stands; kScanFallback is the fallback's scan and returns at once when it does.
enum ScanMode : int { kScanClassic = 0, kScanFused = 1, kScanFallback = 2 };

__global__ void __launch_bounds__(kRadix)
scan_kernel(const unsigned long long* __restrict__ ghist, unsigned long long* __restrict__ gbase, int places,
            SortPlan* plan, unsigned long long n, int allow_skip, int allow_hot, int mode, const uint32_t* fused_abort,
            unsigned long long region)
{
    __shared__ unsigned long long s_warp[kRadix / 32];
    if (mode == kScanFallback && (plan->skip_mask & kPlanFusedKept)) return;  // (read by all threads before any writes it)
    const int d = threadIdx.x, lane = d & 31, warp = d >> 5;
    uint32_t skip_mask = 0;
    // fused: the first pass stood if no tile of it found a digit's region too small (it then scattered nothing) and no
    // place-0 bin exceeds its region
    const int overfull = mode == kScanFused ? __syncthreads_or(ghist[d] > region || *fused_abort != 0) : 0;
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
        // kept: place 0 ran in the plain pass (it cannot be skipped or hot and fit its regions, but say so) and a later
        // place executes -- that pass reads the gapped layout and leaves it dense
        if (mode == kScanFused && !overfull && (run & 1u) && !((skip_mask >> kPlanHotShift) & 1u) && (run & ~1u))
            pl.skip_mask |= kPlanFusedKept;
        *plan = pl;
    }
}

cudaError_t launch_scan(const unsigned long long* ghist, unsigned long long* gbase, int places, cudaStream_t stream,
                        SortPlan* plan, uint64_t n, bool allow_skip, bool allow_hot)
{
    scan_kernel<<<1, kRadix, 0, stream>>>(ghist, gbase, places, plan, n, allow_skip ? 1 : 0, allow_hot ? 1 : 0, kScanClassic,
                                          nullptr, 0ull);
    return cudaGetLastError();
}

cudaError_t launch_scan_fused(const unsigned long long* ghist, unsigned long long* gbase, int places, cudaStream_t stream,
                              SortPlan* plan, uint64_t n, bool allow_skip, bool allow_hot, bool fallback, const uint32_t* fused_abort,
                              uint64_t region)
{
    scan_kernel<<<1, kRadix, 0, stream>>>(ghist, gbase, places, plan, n, allow_skip ? 1 : 0, allow_hot ? 1 : 0,
                                          fallback ? kScanFallback : kScanFused, fused_abort, region);
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
    return with_key_type(HistBitsKeys{}, key_bytes, [&](auto k) {
        using KeyT = decltype(k);
        // byte-aligned places: the fast kernel slices the loaded words, the last place keeps last_bits
        if (begin_bit == 0) return launch_histogram_vec<KeyT, true>(keys, n, ghist, sm_count, stream, codec, places, last_mask);
        global_histogram_bits_kernel<KeyT><<<capped_grid(n, kHistThreads * 4, sm_count), kHistThreads, hist_smem_bytes<KeyT>(), stream>>>(
            static_cast<const KeyT*>(keys), n, ghist, codec, begin_bit, places, last_mask);
        return cudaGetLastError();
    });
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
        copy_back_kernel<W><<<capped_grid(words, 512, static_cast<uint64_t>(sm_count) * 4), 512, 0, stream>>>(plan, static_cast<const W*>(s), static_cast<W*>(d), words,
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
// Four keys per step: one uint4 of 32-bit keys, one uint2 of 16-bit keys, two uint4 of 64-bit keys.
template <typename KeyT>
__global__ void __launch_bounds__(512)
argsort_copy_back_kernel(const SortPlan* __restrict__ plan, const KeyT* __restrict__ keys_in, const KeyT* __restrict__ alt_keys,
                         KeyT* __restrict__ keys, const uint32_t* __restrict__ alt_idx, uint32_t* __restrict__ idx, uint64_t n)
{
    using KV = typename std::conditional<sizeof(KeyT) == 2, uint2, uint4>::type;
    constexpr int KV_PER_STEP = 4 * sizeof(KeyT) / sizeof(KV);
    static_assert(KV_PER_STEP * sizeof(KV) == 4 * sizeof(KeyT), "four keys per step");
    const uint32_t ex = plan->executed;
    if (ex != 0 && !(ex & 1u)) return;
    const KeyT* src = ex ? alt_keys : keys_in;
    const uint64_t vecs = n / 4, stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < vecs; i += stride) {
#pragma unroll
        for (int v = 0; v < KV_PER_STEP; ++v)
            __stcs(reinterpret_cast<KV*>(keys) + i * KV_PER_STEP + v, __ldcs(reinterpret_cast<const KV*>(src) + i * KV_PER_STEP + v));
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
                                     const uint32_t* alt_idx, uint32_t* idx, uint64_t n, int key_bytes, int sm_count,
                                     cudaStream_t stream)
{
    const unsigned grid = capped_grid(n / 4, 512, static_cast<uint64_t>(sm_count) * 4);
    return with_key_type(TypeList<uint16_t, uint32_t, uint64_t>{}, key_bytes, [&](auto k) {
        using KeyT = decltype(k);
        argsort_copy_back_kernel<KeyT><<<grid, 512, 0, stream>>>(plan, static_cast<const KeyT*>(keys_in), static_cast<const KeyT*>(alt_keys),
                                                                 static_cast<KeyT*>(keys), alt_idx, idx, n);
        return cudaGetLastError();
    });
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

// The stalled path's hook of lookback_wide (fused sorts, DESIGN §4.12): hook(-1) on every stalled poll -- kHookAbort stops
// the lookback (a fused first pass that has aborted keeps nothing, and the stalled tile may never run); hook(t) when giving
// up on tile t -- a count is the hook's own re-reduction of t (the gapped source), kHookDefault leaves it to rereduce_tile.
// It reads what it needs where it is called, so that nothing of it is held in registers across the lookback.
constexpr long long kHookAbort = -1, kHookDefault = -2;
struct NoStallHook {
    __device__ __forceinline__ long long operator()(long long) const { return kHookDefault; }
};

// rereduce_tile for the gapped source a fused sort's first pass leaves (DESIGN §4.12): logical position p of the input is
// at p + (r * region - gap[r]) for the region r whose dense range holds p.  Cold path, like rereduce_tile.
template <typename KeyT>
__device__ __noinline__ uint32_t rereduce_tile_gapped(const KeyT* in, uint64_t base, uint32_t tile_keys, uint32_t shift, uint32_t mask,
                                                      const unsigned long long* gap, unsigned long long region, uint16_t* dst,
                                                      uint32_t d)
{
    uint32_t c = 0, r = 0;
    for (uint32_t step = kRadix / 2; step; step >>= 1) if (gap[r + step] <= base) r += step;
    for (uint32_t i = 0; i < tile_keys; ++i) {
        const uint64_t p = base + i;
        while (r + 1 < kRadix && gap[r + 1] <= p) ++r;
        c += digit_of(in[p + r * region - gap[r]], shift, mask) == d;
    }
    st_relaxed_gpu_u16(dst, kAggReady | c);
    return c;
}

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
template <int NBLK, typename KeyT, typename Hook = NoStallHook>
__device__ __forceinline__ unsigned long long
lookback_wide(uint16_t* agg16, const uint64_t* incl64, uint32_t tile, uint32_t d, uint32_t epoch, uint32_t spin_cap,
              const TileRereduce<KeyT>& rr, Hook hook = Hook())
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
            if (hook(-1) == kHookAbort) return sum;
            polls = next == cur ? polls + 1 : 1;
            if (polls > spin_cap) {
                // maybe the stalled tile has finished altogether meanwhile: its inclusive prefix settles everything
                const uint64_t w = ld_relaxed_gpu_u64(incl64 + next * kRadix + d);
                if (desc_epoch(w) == epoch && (w & kFlagMask) == kFlagInclusive) return sum + desc_value(w);
                const long long h = hook(next);
                if (h >= 0)
                    sum += static_cast<unsigned long long>(h);
                else
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
    // fused sorts (u32 keys only, DESIGN §4.12): the region capacity c (0: not a fused sort); the fused first pass's abort
    // word and the global histogram it fills; place 0's dense digit bases, which map the gapped source to positions
    unsigned long long region = 0;
    uint32_t* fused_abort = nullptr;
    unsigned long long* fused_hist = nullptr;
    const unsigned long long* dense_base0 = nullptr;
};

// plan_bits of an argsort pass (INDICES): this is the first executed pass -- its keys come from PassParams::keys_in and its
// payloads are the keys' own input positions
constexpr uint32_t kPlanBitsFirstIndices = 8u;
// plan_bits of the first executed pass after the fused first pass: its source is gapped (plan_reads_gapped)
constexpr uint32_t kPlanBitsGapped = 16u;

__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

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
    // 16-bit pairs: `sorted` itself holds the tile's T {key, payload} uint2 words (8 B per slot; see the kernel)
    // (64-bit pairs: the keys in `sorted`, the payloads in `sorted_val` -- no {key, payload} word)
    static constexpr bool KV_IN_SORTED = PAIRS && sizeof(KeyT) == 2;
    alignas(16) KeyT sorted[KV_IN_SORTED ? T * 8 / sizeof(KeyT) : T];  // digit-sorted tile
    alignas(16) uint32_t sorted_val[PAIRS && !KV_IN_SORTED ? T : 4];   // payloads in the same order
    alignas(16) uint32_t hist[WARPS * kRadix];       // warp-private digit counters (counts, then running slots)
    unsigned long long keyptr[kRadix];               // per digit: byte address of out[first key of the digit - tile slot]
    unsigned long long valptr[PAIRS ? kRadix : 1];
    uint32_t run[32];                                // few-bins passes: first slot (low 16 bits) | live length (high 16)
    uint32_t wtot[kRadix / 32];
    uint32_t wmax[kRadix / 32];                      // (HOT) per digit warp: max of (tile count << 8 | digit)
    uint32_t next_tile;                              // the tile this CTA works on after the current one (drawn ticket)
    uint32_t plan_bits;                              // bit 0: source is the alt buffer; bits 1-2: codec flags of this pass;
                                                     // bit 3: first pass of an argsort (kPlanBitsFirstIndices); bit 4: the
                                                     // source is gapped (kPlanBitsGapped)
    uint32_t digit_shift, digit_mask;                // copies of the pass's digit, re-read by the rank phase (opaque_copy)
    // u32 keys only (fused sorts): place 0's dense digit bases (gapped source); the fused first pass's counts of places
    // 1-3 over the CTA's tiles, and whether it stops
    static constexpr bool kFusable = sizeof(KeyT) == 4 && !PAIRS;
    unsigned long long gap_base[kFusable ? kRadix : 1];
    uint32_t fhist[kFusable ? 3 * kRadix : 1];
    uint32_t fused_stop;
};

// INDICES (argsort, pairs only): buf0/val0 are the caller's output keys and indices, buf1/val1 the alt buffers.  The first
// executed pass, which by the plan's parity would read the caller's side, reads its keys from pp.keys_in instead and makes
// every payload from the key's position in the input; every other pass is the pairs pass as it is.
// FUSED (u32 keys, the fused first pass of a whole-key sort, DESIGN §4.12): runs without a plan, reads buf0 and writes
// buf1 with digit d's keys in the region [d * c, (d + 1) * c), c = pp.region; counts places 0-3 into pp.fused_hist; a tile
// that would overflow a region scatters nothing, sets *pp.fused_abort, and every tile after it stops as well.
template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE, int LOOK, int MINB, bool HOT = false, bool INDICES = false,
          bool FUSED = false>
__global__ void __launch_bounds__(WARPS * 32, HOT ? OSB_HOT_MINB : MINB)
digit_binning_wide_kernel(KeyT* buf0, KeyT* buf1, uint32_t* val0, uint32_t* val1, uint64_t n,
                          const unsigned long long* __restrict__ gbase, uint16_t* agg16, uint64_t* incl64,
                          uint32_t* ticket, PassParams pp, KeyCodec codec)
{
    static_assert(!INDICES || PAIRS, "the indices are the 32-bit payloads of a pairs pass");
    static_assert(!FUSED || (sizeof(KeyT) == 4 && !PAIRS && !HOT && WARPS * 32 > kRadix), "the fused first pass: u32 keys, plain");
    using S = WideSmem<KeyT, PAIRS, K, WARPS>;
    constexpr int THREADS = S::THREADS;
    constexpr int T = S::T;
    static_assert(T < 32768, "agg16 holds 15-bit counts");
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);
    // pairs: key and payload of a tile slot are ONE 64-bit word of shared memory ({key, payload}; `sorted` and `sorted_val`
    // are adjacent and together hold T such words) -- one transposing STS.64 and one LDS.64 per pair instead of two of each,
    // and the payload's destination is the key's plus a constant (reference: OneSweep.cu:522-599 moves them separately)
    // (16-bit keys: the word is {key zero-extended, payload}, and `sorted` is sized for T of them)
    // (64-bit keys: a 12-byte slot has no such word; keys and payloads are staged in their own arrays, and every payload is
    // stored through its digit's own pointer, as for 16-bit keys)
    constexpr bool KV_WORD = PAIRS && sizeof(KeyT) <= 4;
    static_assert(!PAIRS || (sizeof(KeyT) == 4 && offsetof(S, sorted_val) == offsetof(S, sorted) + sizeof(KeyT) * T) ||
                  (S::KV_IN_SORTED && sizeof(S::sorted) == sizeof(uint2) * T) ||
                  (sizeof(KeyT) == 8 && sizeof(S::sorted) == sizeof(KeyT) * T && sizeof(S::sorted_val) == sizeof(uint32_t) * T),
                  "kv layout");
    uint2* const kv = reinterpret_cast<uint2*>(sm.sorted);
    // a tile slot's key and payload: stored by the rank phase, read by the scatter
    auto put_slot = [&](uint32_t slot, KeyT k, uint32_t v) {
        if constexpr (KV_WORD) kv[slot] = make_uint2(static_cast<uint32_t>(k), v);
        else { sm.sorted[slot] = k; sm.sorted_val[slot] = v; }
    };
    auto get_slot = [&](uint32_t x, KeyT& k, uint32_t& v) {
        if constexpr (KV_WORD) { const uint2 e = kv[x]; k = static_cast<KeyT>(e.x); v = e.y; }
        else { k = sm.sorted[x]; v = sm.sorted_val[x]; }
    };

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
        if constexpr (S::kFusable) my_bits |= plan_reads_gapped(pl, pp.place) ? kPlanBitsGapped : 0u;
        // a fused sort whose fused first pass stood: the classic pass of place 0 (its fallback) has nothing to do
        if (pp.place == 0 && (pl.skip_mask & kPlanFusedKept)) my_skip = true;
    }
    if (my_skip) return;  // all keys share this digit: nothing to move (the plan accounts for the parity)
    if (HOT != my_hot) return;  // a pass is executed by exactly one of the two instantiations the host enqueues
    const uint32_t num_tiles = static_cast<uint32_t>((n + T - 1) / T);

    // ---- tile loads (warp-striped: every warp instruction reads one contiguous 128 B / 256 B row) ----------------
    // The ragged last tile is padded with all-ones keys (they rank last); a tile at or past num_tiles loads nothing.
    // (16-bit keys-only passes hold their keys zero-extended in 32-bit registers: as 16-bit values they spill in atomic mode;
    // the pairs pass spills the other way round.)
    using KeyReg = typename std::conditional<sizeof(KeyT) == 2 && !PAIRS, uint32_t, KeyT>::type;
    KeyReg key[K];
    uint32_t val[PAIRS ? K : 1];
    const uint32_t warp_off = warp * (32 * K) + lane;
    // The gapped source (the first executed pass after a fused first pass; u32 keys): logical position p is at
    // p + (r * c - B0[r]) of the alt buffer, r the region whose dense range [B0[r], B0[r + 1]) holds p.  A full tile inside
    // one region takes one offset; a tile across a region boundary, and the ragged last tile, look the region up per key.
    auto region_of = [&](uint64_t p) {
        uint32_t r = 0;
#pragma unroll 1
        for (uint32_t step = kRadix / 2; step; step >>= 1) if (sm.gap_base[r + step] <= p) r += step;
        return r;
    };
    auto load_gapped = [&](uint32_t t) {
        const KeyT* __restrict__ in = buf1;
        const unsigned long long c = pp.region;
        const uint64_t base = static_cast<uint64_t>(t) * T;
        if (base + T <= n) {
            const uint32_t r0 = region_of(base);
            if (r0 == region_of(base + T - 1)) {
                const KeyT* __restrict__ src = in + (base + r0 * c - sm.gap_base[r0]) + warp_off;
#pragma unroll
                for (int i = 0; i < K; ++i) key[i] = ld_stream(src + i * 32);
                return;
            }
        }
        const uint64_t live = base < n ? n - base : 0u;
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t idx = warp_off + i * 32;
            if (idx < live) {
                const uint64_t p = base + idx;
                const uint32_t r = region_of(p);
                key[i] = in[p + r * c - sm.gap_base[r]];
            } else {
                key[i] = static_cast<KeyT>(~static_cast<KeyT>(0));
            }
        }
    };
    auto load_tile = [&](uint32_t t) {
        if constexpr (S::kFusable) {
            if (my_bits & kPlanBitsGapped) { load_gapped(t); return; }
        }
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
    if constexpr (S::kFusable) {
        if (my_bits & kPlanBitsGapped) {  // (my_bits is the same in every thread)
            for (int i = tid; i < kRadix; i += THREADS) sm.gap_base[i] = pp.dense_base0[i];
            __syncthreads();
        }
    }
    load_tile(tile);
    {
        uint4* h4 = reinterpret_cast<uint4*>(sm.hist);
        for (int i = tid; i < WARPS * kRadix / 4; i += THREADS) h4[i] = make_uint4(0, 0, 0, 0);
    }
    if constexpr (FUSED) {
        for (int i = tid; i < 3 * kRadix; i += THREADS) sm.fhist[i] = 0;
        if (tid == 0) sm.fused_stop = 0;
    }
    uint32_t fused_count = 0;  // FUSED, digit threads: this CTA's keys with digit tid in place 0
    if (tid == 0) { sm.plan_bits = my_bits; sm.digit_shift = shift; sm.digit_mask = dmask; }
    __syncthreads();  // histograms cleared, plan_bits visible (the loads above are already in flight)
    // plan_bits (direction, codec flags) is re-read from shared memory where it is needed instead of being carried in
    // registers across the phases: the 64-register budget of this kernel is spent on the 32 keys (the rank phase recomputes
    // their counter addresses, see opaque_copy below)
    // The plain u64 keys and pairs passes keep one tile per CTA (their launch has one CTA per tile; the loop body runs once).
    // u64: with its window of 32 tiles the lookback holds four 16-byte blocks per round trip, and 16 prefetched keys held
    // across it spill (180 B per thread); issued after the lookback instead they made the pass 4 % slower on the H100.
    // Pairs: persistent, the pass was up to 0.9 % slower on the H100 (26.01 -> 25.79 Gpairs/s at 400 W).
    // 16-bit keys follow the u32 choices (same registers per key: a 16-bit key occupies a 32-bit register).
    constexpr bool kPersistent = (sizeof(KeyT) <= 4 && !PAIRS) || HOT;
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
            key[i] = codec_encode<KeyT>(static_cast<KeyT>(key[i]), ca, cb, cd);
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
            auto hook = [&](long long t) -> long long {
                if (t < 0) {
                    if constexpr (FUSED) return *reinterpret_cast<const volatile uint32_t*>(pp.fused_abort) ? kHookAbort : kHookDefault;
                    return kHookDefault;
                }
                if (S::kFusable && (sm.plan_bits & kPlanBitsGapped))
                    return rereduce_tile_gapped<KeyT>(buf1, static_cast<uint64_t>(t) * T, T, shift, dmask, pp.dense_base0, pp.region,
                                                      agg16 + agg_index(t, tid), tid);
                return kHookDefault;
            };
            const unsigned long long prior = lookback_wide<LOOK / 8, KeyT>(agg16, incl64, tile, tid, epoch, pp.spin_cap, rr, hook);
            const bool swap = sm.plan_bits & 1u;
            KeyT* out = swap ? buf0 : buf1;
            uint32_t* out_val = swap ? val0 : val1;
            st_relaxed_gpu_u64(incl64 + static_cast<uint64_t>(tile) * kRadix + tid,
                               desc_pack(epoch, kFlagInclusive, prior + tile_count));
            // FUSED: digit tid's region starts at tid * c; a digit whose keys would run past it stops the pass, as does
            // an abort seen here (this tile's lookback may have given up on a predecessor that never ran).  So does a digit
            // holding more than a sixteenth of the tile (uniform keys: 64 +- 8 of 16,384): such low-entropy inputs mostly
            // overflow a region anyway, only thousands of tiles later, and stopping at once saves that part of the pass.
            if constexpr (FUSED) {
                const uint32_t live_d = tile_count - ((tid == kRadix - 1 && !full) ? (T - valid) : 0u);  // (padding: digit 255)
                fused_count += live_d;
                if (prior + live_d > pp.region || live_d > T / 16) {
                    *reinterpret_cast<volatile uint32_t*>(pp.fused_abort) = 1u;
                    sm.fused_stop = 1u;
                } else if (*reinterpret_cast<const volatile uint32_t*>(pp.fused_abort)) {
                    sm.fused_stop = 1u;
                }
            }
            // element index (relative to out) of tile slot 0
            const unsigned long long first = (FUSED ? tid * pp.region : gbase[tid]) + prior - tile_excl;
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
            if constexpr (PAIRS) put_slot(slot, key[i], val[i]);
            else sm.sorted[slot] = key[i];
        }
    } else {
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t slot = warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], rshift, rmask), lt);
            if constexpr (PAIRS) put_slot(slot, key[i], val[i]);
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
    // FUSED: the warps that do not look back count places 1-3 of the digit-sorted tile meanwhile (the ragged tile's padding
    // holds its last slots), into the CTA's histogram; the digit warps only signal that their rank stores are done.
    if constexpr (FUSED) {
        if (warp < kRadix / 32) {
            named_bar_arrive(1, THREADS);
        } else {
            named_bar_sync(1, THREADS);
            const uint4* s4 = reinterpret_cast<const uint4*>(sm.sorted);
#pragma unroll 1
            for (uint32_t j = tid - kRadix; j < T / 4; j += THREADS - kRadix) {
                const uint4 v = s4[j];
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (full || 4 * j + q < valid) {
                        atomicAdd(&sm.fhist[(w[q] >> 8) & 255u], 1u);
                        atomicAdd(&sm.fhist[kRadix + ((w[q] >> 16) & 255u)], 1u);
                        atomicAdd(&sm.fhist[2 * kRadix + (w[q] >> 24)], 1u);
                    }
                }
            }
        }
    }
    chained_scan();
    OSB_PHASE(5);
    __syncthreads();
    OSB_PHASE(8);
    if constexpr (FUSED) { if (sm.fused_stop) break; }  // nothing of this pass is kept: leave the rest to the fallback
    if constexpr (HOT) { if (warp < kRadix / 32) load_tile(next); }

    // ---- scatter -----------------------------------------------------------------------------------------
    // Few bins (a digit of <= 5 bits: the sharded exchange on log2(R) bits): runs are thousands of keys long, so
    // the stores are issued run by run in chunks that start on 128-byte boundaries of the DESTINATION -- every warp
    // store is then one full line (4 full sectors), which is what keeps NVLink peer stores at their aligned rate
    // (partial-sector peer stores run well below it; tools/microbench/p2p_store_ub.cu measures both).
    const bool dec = (sm.plan_bits >> 1) & kCodecDecodeOnStore;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    // pairs: a payload goes where its key goes, in the other output array (same element size: a constant byte distance;
    // 16- and 64-bit keys: the payload's own digit pointer)
    long long val_delta = 0;
    if constexpr (PAIRS && sizeof(KeyT) == 4) {
        const bool swap = sm.plan_bits & 1u;
        val_delta = reinterpret_cast<const char*>(swap ? val0 : val1) - reinterpret_cast<const char*>(swap ? buf0 : buf1);
    }
    auto val_dst = [&](KeyT* dst, uint32_t d, uint32_t x) -> uint32_t* {
        if constexpr (sizeof(KeyT) == 4) return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(dst) + val_delta);
        else return reinterpret_cast<uint32_t*>(sm.valptr[d]) + x;
    };
    (void)val_dst;
    auto slot_key = [&](uint32_t x) -> KeyT { if constexpr (KV_WORD) return static_cast<KeyT>(kv[x].x); else return sm.sorted[x]; };
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
                        KeyT k;
                        uint32_t v;
                        get_slot(x, k, v);
                        if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
                        KeyT* dst = reinterpret_cast<KeyT*>(kp) + x;
                        st_scatter(dst, k);
                        st_scatter(val_dst(dst, b, x), v);
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
                KeyT k;
                uint32_t v;
                get_slot(idx, k, v);
                const uint32_t d = digit_of(k, shift, dmask);
                KeyT* dst = reinterpret_cast<KeyT*>(sm.keyptr[d]) + idx;
                st_scatter(dst, k);
                st_scatter(val_dst(dst, d, idx), v);
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
                    KeyT k;
                    uint32_t v;
                    get_slot(idx, k, v);
                    const uint32_t d = digit_of(k, shift, dmask);
                    KeyT* dst = reinterpret_cast<KeyT*>(sm.keyptr[d]) + idx;
                    st_scatter(dst, dec ? codec_decode<KeyT>(k, ca, cb, cd) : k);
                    st_scatter(val_dst(dst, d, idx), v);
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
    // FUSED: the CTA's counts go to the global histogram once (its last tile's were complete at the barrier after the lookback)
    if constexpr (FUSED) {
        if (!sm.fused_stop) {
            if (tid < kRadix && fused_count) atomicAdd(&pp.fused_hist[tid], static_cast<unsigned long long>(fused_count));
            for (int i = tid; i < 3 * kRadix; i += THREADS)
                if (sm.fhist[i]) atomicAdd(&pp.fused_hist[kRadix + i], static_cast<unsigned long long>(sm.fhist[i]));
        }
    }
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

// ---- what every DigitBinningPass shape has ------------------------------------------------------------
// The arguments of one pass, whichever kernel runs it.
struct PassArgs {
    const void* in; void* out; const uint32_t* in_val; uint32_t* out_val; uint64_t n; uint32_t shift;
    const unsigned long long* gbase; uint64_t* desc; uint16_t* agg16; uint32_t* ticket; uint32_t epoch;
    const BinningConfig& cfg; cudaStream_t stream;

    PassParams params() const
    {
        PassParams pp;
        pp.shift = shift;
        pp.dbits = cfg.digit_bits;
        pp.epoch = epoch;
        pp.place = cfg.place;
        pp.spin_cap = cfg.spin_cap;
        pp.stall_every = cfg.debug_stall_every;
        pp.plan = cfg.plan;
        pp.keys_in = cfg.argsort_in;
        pp.region = cfg.fused_region;
        pp.dense_base0 = cfg.fused_dense_base0;
        return pp;
    }
};

// A pass shape: the keys, pairs and indices it sorts.  Each family adds its tile T, its dynamic shared memory `smem`,
// kernel<RANK_MODE, HOT>() and launch<RANK_MODE>(const PassArgs&).
template <typename KeyT, bool PAIRS, bool INDICES = false>
struct PassShape {
    using Key = KeyT;
    static constexpr bool pairs = PAIRS, indices = INDICES;
    static constexpr bool enabled = true;   // whether launch_digit_binning runs it (the shape is configured either way)
    static constexpr bool has_hot = false;  // whether it has a HOT twin for low-entropy passes
};

template <typename KeyT>
struct RingShape : PassShape<KeyT, false> {
    using G = RingGeom<KeyT>;
    using S = RingSmem<KeyT, G::K, G::WARPS>;
    static constexpr uint32_t T = S::T;
    static constexpr size_t smem = sizeof(S);
    template <int RANK_MODE, bool HOT = false>
    static auto kernel() { return digit_binning_ring_kernel<KeyT, G::K, G::WARPS, RANK_MODE, G::LOOK>; }
    template <int RANK_MODE>
    static cudaError_t launch(const PassArgs& a)
    {
        const uint64_t tiles = (a.n + T - 1) / T;
        const uint64_t cap = static_cast<uint64_t>(a.cfg.sm_count) * (sizeof(KeyT) == 4 ? OSB_RING_MINB : 2);
        const auto kern = kernel<RANK_MODE>();
        kern<<<static_cast<unsigned>(tiles < cap ? tiles : cap), S::THREADS, smem, a.stream>>>(
            static_cast<const KeyT*>(a.in), static_cast<KeyT*>(a.out), a.n, a.shift, a.gbase, a.agg16, a.desc, a.ticket, a.epoch,
            static_cast<uint32_t>(tiles));
        return cudaGetLastError();
    }
};

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
// 16-bit keys (osb200_sort_keys16 & co., run on a 4-byte handle).  A 16-bit key takes a 32-bit register like a u32 key;
// each tile load is one warp-striped 16-bit load per key (64 B per warp instruction, tile order = input order, so the
// stability argument of the u32 pass is unchanged).  Keys: 24 keys per thread (12,288-key tiles) -- with the u32 kernel's 32
// the atomic-mode pass spills on sm_90a (12 B; 28 and 30 keys spill too, 24 does not).  Pairs: the u32 pairs geometry.
// DESIGN §4.4.
#ifndef OSB_K16_K  // geometry of the 16-bit keys-only kernel, overridable for sweeps
#define OSB_K16_K 24
#define OSB_K16_WARPS 16
#endif
#ifndef OSB_P16_K  // geometry of the 16-bit pairs / argsort kernel
#define OSB_P16_K 16
#define OSB_P16_WARPS 16
#endif
template <> struct WideGeom<uint16_t, false> { static constexpr int K = OSB_K16_K, WARPS = OSB_K16_WARPS, MINB = 2, LOOK = OSB_LOOK; };
template <> struct WideGeom<uint16_t, true>  { static constexpr int K = OSB_P16_K, WARPS = OSB_P16_WARPS, MINB = 2, LOOK = OSB_PAIRS_LOOK; };
// 64-bit keys with 32-bit payloads (osb200_create_pairs64: osb200_sort_pairs_typed, osb200_argsort).  A pair takes three
// registers, so the u32 pairs shape (16 pairs per thread at 64 registers) does not fit.  16 pairs per thread with ONE CTA
// per SM (8,192-pair tiles, 116 KiB of shared memory, up to 128 registers: no spills) beat 8 and 12 pairs per thread at two
// CTAs per SM by 23 % and 15 % on the H100 (2^30 keys, argsort: 91 against 118 and 107 ms).  DESIGN §4.11.
#ifndef OSB_P64_K  // geometry of the 64-bit pairs / argsort kernel, overridable for sweeps
#define OSB_P64_K 16
#define OSB_P64_WARPS 16
#define OSB_P64_MINB 1
#endif
#ifndef OSB_P64_LOOK
#define OSB_P64_LOOK 32
#endif
template <> struct WideGeom<uint64_t, true>  { static constexpr int K = OSB_P64_K, WARPS = OSB_P64_WARPS, MINB = OSB_P64_MINB, LOOK = OSB_P64_LOOK; };
template <typename KeyT, bool PAIRS, bool INDICES = false>
struct WideShape : PassShape<KeyT, PAIRS, INDICES> {
    using G = WideGeom<KeyT, PAIRS>;
    using S = WideSmem<KeyT, PAIRS, G::K, G::WARPS>;
    static constexpr uint32_t T = S::T;
    static constexpr size_t smem = sizeof(S);
    static constexpr bool has_hot = true;
    template <int RANK_MODE, bool HOT = false>
    static auto kernel() { return digit_binning_wide_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, G::LOOK, G::MINB, HOT, INDICES>; }
    template <int RANK_MODE>
    static cudaError_t launch(const PassArgs& a)
    {
        const uint64_t tiles = (a.n + T - 1) / T;
        const PassParams pp = a.params();
        // Persistent instantiations (all but the plain u64 keys and pairs passes, which run one CTA per tile): as many CTAs as can be resident
        // at once (capped by debug_max_ctas), at most one per tile; the tiles after the first of each CTA are handed out by
        // `ticket`, which the host zeroes before the pass.
        auto grid_for = [&](auto kernel, int& per_sm, bool persistent) -> unsigned {
            if (!persistent) return static_cast<unsigned>(tiles);
            if (per_sm == 0) {
                int b = 0;
                if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, kernel, S::THREADS, smem) != cudaSuccess || b < 1) b = 1;
                per_sm = b;
            }
            uint64_t cap = static_cast<uint64_t>(a.cfg.sm_count) * per_sm;
            if (a.cfg.debug_max_ctas && a.cfg.debug_max_ctas < cap) cap = a.cfg.debug_max_ctas;
            return static_cast<unsigned>(tiles < cap ? tiles : cap);
        };
        KeyT* buf0 = static_cast<KeyT*>(const_cast<void*>(a.in));
        uint32_t* val0 = const_cast<uint32_t*>(a.in_val);
        const auto kern = kernel<RANK_MODE>();
        static int plain_per_sm = 0;  // (one value per instantiation)
        // with a device plan `in`/`out` are the caller's and the alt buffers (the kernel picks the direction); both are written
        kern<<<grid_for(kern, plain_per_sm, sizeof(KeyT) <= 4 && !PAIRS), S::THREADS, smem, a.stream>>>(
            buf0, static_cast<KeyT*>(a.out), val0, a.out_val, a.n, a.gbase, a.agg16, a.desc, a.ticket, pp, a.cfg.codec);
        if (a.cfg.plan != nullptr && a.cfg.hot_passes) {
            // the HOT instantiation of the same pass; returns at once unless the plan calls the pass hot, before drawing a ticket
            // (same geometry, one resident CTA per SM with up to 128 registers: no spills.  Two CTAs per SM at 64 registers
            // spill; 1,024 threads x 16 keys at 64 registers is slower than this)
            const auto hot = kernel<RANK_MODE, true>();
            static int hot_per_sm = 0;
            hot<<<grid_for(hot, hot_per_sm, true), S::THREADS, smem, a.stream>>>(
                buf0, static_cast<KeyT*>(a.out), val0, a.out_val, a.n, a.gbase, a.agg16, a.desc, a.ticket, pp, a.cfg.codec);
        }
        return cudaGetLastError();
    }
};

constexpr int kPairsK = 32, kPairsWarps = 16;

// u32 pairs in 16,384-pair tiles: the default pass's shape only in a -DOSB_PAIRS16K=1 build
struct Pairs16KShape : PassShape<uint32_t, true> {
    static constexpr bool enabled = OSB_PAIRS16K != 0;
    using S = PairsSmem<kPairsWarps, kPairsK>;
    static constexpr uint32_t T = S::T;
    static constexpr size_t smem = sizeof(S);
    template <int RANK_MODE, bool HOT = false>
    static auto kernel() { return digit_binning_pairs_kernel<kPairsK, kPairsWarps, RANK_MODE, OSB_PAIRS_LOOK>; }
    template <int RANK_MODE>
    static cudaError_t launch(const PassArgs& a)
    {
        const auto kern = kernel<RANK_MODE>();
        kern<<<static_cast<unsigned>((a.n + T - 1) / T), S::THREADS, smem, a.stream>>>(
            static_cast<uint32_t*>(const_cast<void*>(a.in)), static_cast<uint32_t*>(a.out), const_cast<uint32_t*>(a.in_val), a.out_val,
            a.n, a.gbase, a.agg16, a.desc, a.ticket, a.params(), a.cfg.codec);
        return cudaGetLastError();
    }
};

// ---- variant-0 geometry ------------------------------------------------------------------------------
template <typename KeyT, bool PAIRS> struct TileGeom;
template <> struct TileGeom<uint32_t, false> { static constexpr int K = 16, WARPS = 16; };
template <> struct TileGeom<uint32_t, true>  { static constexpr int K = 16, WARPS = 16; };
template <> struct TileGeom<uint64_t, false> { static constexpr int K = 8,  WARPS = 16; };

template <typename KeyT, bool PAIRS>
struct TileShape : PassShape<KeyT, PAIRS> {
    using G = TileGeom<KeyT, PAIRS>;
    static constexpr uint32_t T = G::WARPS * 32 * G::K;
    static constexpr size_t hist_bytes = static_cast<size_t>(G::WARPS) * kRadix * 4, keys_bytes = T * sizeof(KeyT);
    static constexpr size_t smem = hist_bytes > keys_bytes ? hist_bytes : keys_bytes;  // the histograms, then the sorted tile
    template <int RANK_MODE, bool HOT = false>
    static auto kernel() { return digit_binning_tile_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE>; }
    template <int RANK_MODE>
    static cudaError_t launch(const PassArgs& a)
    {
        const auto kern = kernel<RANK_MODE>();
        kern<<<static_cast<unsigned>((a.n + T - 1) / T), G::WARPS * 32, smem, a.stream>>>(
            static_cast<const KeyT*>(a.in), static_cast<KeyT*>(a.out), a.in_val, a.out_val, a.n, a.shift, a.gbase, a.desc, a.ticket,
            a.epoch);
        return cudaGetLastError();
    }
};

// The instantiations of each variant.  Variant 2, the default pass: 16-, 32- and 64-bit keys, pairs and argsort, each with a
// HOT twin (and the 16K-pair kernel, which takes the u32 pairs when enabled).
using DefaultPassShapes = TypeList<Pairs16KShape,
                                   WideShape<uint16_t, false>, WideShape<uint16_t, true>, WideShape<uint16_t, true, true>,
                                   WideShape<uint32_t, false>, WideShape<uint32_t, true>, WideShape<uint32_t, true, true>,
                                   WideShape<uint64_t, false>, WideShape<uint64_t, true>, WideShape<uint64_t, true, true>>;
using RingShapes = TypeList<RingShape<uint32_t>, RingShape<uint64_t>>;  // variant 1: keys only
using TileShapes = TypeList<TileShape<uint32_t, false>, TileShape<uint32_t, true>, TileShape<uint64_t, false>>;  // variant 0

// f(Shape{}) for the pass launch_digit_binning runs on these keys in this variant: variant 1 has no pairs kernel, and
// runs pairs in variant 0's.  cudaErrorInvalidValue if the variant has no such pass.
template <typename F>
static cudaError_t with_pass_shape(int key_bytes, bool pairs, bool indices, int variant, F&& f)
{
    auto match = [&](auto s) {
        using S = decltype(s);
        return S::enabled && key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::pairs == pairs && S::indices == indices;
    };
    if (variant == kVariantWide) return find_type(DefaultPassShapes{}, match, f);
    if (variant == kVariantPersistent && !pairs) return find_type(RingShapes{}, match, f);
    return find_type(TileShapes{}, match, f);
}

// 16-bit keys run on a 4-byte handle, whose descriptors and reductions are sized for its smallest tile (smallest_tile in
// osb_host.cu: the minimum over the variants of the 4-byte tiles): their tiles must not be smaller.
constexpr uint32_t cmin(uint32_t a, uint32_t b) { return a < b ? a : b; }
constexpr uint32_t kSmallestTileU32Keys = cmin(cmin(TileShape<uint32_t, false>::T, RingShape<uint32_t>::T), WideShape<uint32_t, false>::T);
constexpr uint32_t kSmallestTileU32Pairs = cmin(TileShape<uint32_t, true>::T, WideShape<uint32_t, true>::T);
static_assert(WideShape<uint16_t, false>::T >= kSmallestTileU32Keys && WideShape<uint16_t, false>::T >= kSmallestTileU32Pairs,
              "16-bit keys (either 4-byte handle): a smaller tile would need more descriptors than the handle has");
static_assert(WideShape<uint16_t, true>::T >= kSmallestTileU32Pairs,
              "16-bit pairs (a (4, 4) handle): a smaller tile would need more descriptors than the handle has");
static_assert(WideShape<uint16_t, false>::T < 32768 && WideShape<uint16_t, true>::T < 32768, "agg16 holds 15-bit counts");
// A (8, 4) handle sizes its descriptors and reductions for smallest_tile(8, true): the variant-0 u64 tile (osb200_workspace_bytes
// relies on it as well).
static_assert(WideShape<uint64_t, true>::T >= TileShape<uint64_t, false>::T,
              "64-bit pairs: a smaller tile would need more descriptors than the handle has");
static_assert(WideShape<uint64_t, true>::T < 32768, "agg16 holds 15-bit counts");

uint32_t binning_tile_keys(int key_bytes, bool pairs, const BinningConfig& cfg)
{
    uint32_t t = 0;
    auto tile = [&](auto s) { t = decltype(s)::T; return cudaSuccess; };
    // pairs in a variant without a pairs pass for these keys (variant 0, 64-bit keys): the tile of its keys pass
    if (with_pass_shape(key_bytes, pairs, false, cfg.variant, tile) != cudaSuccess) with_pass_shape(key_bytes, false, false, cfg.variant, tile);
    return t;
}

bool binning_has_hot_twin(int key_bytes, bool pairs, bool indices, const BinningConfig& cfg)
{
    bool hot = false;
    with_pass_shape(key_bytes, pairs, indices, cfg.variant, [&](auto s) { hot = decltype(s)::has_hot; return cudaSuccess; });
    return hot;
}

// The fused first pass of the u32 keys pass (DESIGN §4.12), both rank modes.
using FusedShape = WideShape<uint32_t, false>;
template <int RANK_MODE>
static auto fused_kernel()
{
    using G = FusedShape::G;
    return digit_binning_wide_kernel<uint32_t, false, G::K, G::WARPS, RANK_MODE, G::LOOK, G::MINB, false, false, true>;
}

cudaError_t launch_fused_first_pass(const uint32_t* keys, uint32_t* alt, uint64_t n, uint64_t region, unsigned long long* ghist,
                                    uint32_t* abort_word, uint64_t* desc, uint16_t* agg16, uint32_t* ticket, uint32_t epoch,
                                    const BinningConfig& cfg, cudaStream_t stream, uint32_t* ctas)
{
    return with_rank_mode(cfg.rank_mode, [&](auto r) {
        constexpr int RANK_MODE = decltype(r)::value;
        const auto kern = fused_kernel<RANK_MODE>();
        static int per_sm = 0;  // (one value per rank mode)
        if (per_sm == 0) {
            int b = 0;
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, kern, FusedShape::S::THREADS, FusedShape::smem) != cudaSuccess || b < 1) b = 1;
            per_sm = b;
        }
        const uint64_t tiles = (n + FusedShape::T - 1) / FusedShape::T;
        uint64_t cap = static_cast<uint64_t>(cfg.sm_count) * per_sm;
        if (cfg.debug_max_ctas && cfg.debug_max_ctas < cap) cap = cfg.debug_max_ctas;
        PassParams pp;
        pp.shift = 0;
        pp.dbits = 8;
        pp.epoch = epoch;
        pp.place = 0;
        pp.spin_cap = cfg.spin_cap;
        pp.stall_every = cfg.debug_stall_every;
        pp.plan = nullptr;
        pp.region = region;
        pp.fused_abort = abort_word;
        pp.fused_hist = ghist;
        KeyCodec codec = cfg.codec;
        codec.flags &= kCodecEncodeOnLoad;
        *ctas = static_cast<uint32_t>(tiles < cap ? tiles : cap);
        kern<<<*ctas, FusedShape::S::THREADS, FusedShape::smem, stream>>>(
            const_cast<uint32_t*>(keys), alt, nullptr, nullptr, n, nullptr, agg16, desc, ticket, pp, codec);
        return cudaGetLastError();
    });
}

cudaError_t launch_digit_binning(const void* in, void* out, const uint32_t* in_val, uint32_t* out_val, uint64_t n,
                                 int key_bytes, uint32_t shift, const unsigned long long* gbase_place, uint64_t* desc,
                                 uint16_t* agg16, uint32_t* ticket, uint32_t epoch, const BinningConfig& cfg,
                                 cudaStream_t stream)
{
    const bool pairs = in_val != nullptr;
    if (cfg.variant != kVariantWide && (cfg.codec.flags || cfg.plan != nullptr || cfg.debug_stall_every || cfg.argsort_in))
        return cudaErrorNotSupported;
    if (cfg.digit_bits < 1 || cfg.digit_bits > 8) return cudaErrorInvalidValue;
    // variants 0 and 1 always take 8-bit digits: a narrower digit is only correct for them when the bits above it do not exist
    if (cfg.variant != kVariantWide && cfg.digit_bits != 8 && shift + cfg.digit_bits != static_cast<uint32_t>(key_bytes) * 8u)
        return cudaErrorNotSupported;
    // argsort: the first executed pass reads argsort_in and makes the indices
    const bool indices = cfg.argsort_in != nullptr;
    if (indices && (!pairs || cfg.plan == nullptr)) return cudaErrorInvalidValue;
    const PassArgs a{in, out, in_val, out_val, n, shift, gbase_place, desc, agg16, ticket, epoch, cfg, stream};
    return with_rank_mode(cfg.rank_mode, [&](auto r) {
        return with_pass_shape(key_bytes, pairs, indices, cfg.variant,
                               [&](auto s) { return decltype(s)::template launch<decltype(r)::value>(a); });
    });
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

// ranks.r[i] (0 for i >= kMaxSelectRanks), read with constant indices only, so the ranks stay in the launch parameters
__device__ __forceinline__ uint32_t select_rank_of(const SelectRanks& ranks, uint32_t i)
{
    uint32_t r = 0;
#pragma unroll
    for (uint32_t j = 0; j < kMaxSelectRanks; ++j) r = i == j ? ranks.r[j] : r;
    return r;
}

// osb200_select_segments' ranks of one segment, by one whole warp, lane i < nr holding rank i in r: how many of them take part
// -- the ranks below the segment's length len, a prefix since they do not decrease -- or 0 when they decrease anywhere (the
// whole row is then padding).
__device__ __forceinline__ uint32_t select_ranks_active(uint32_t r, uint32_t nr, unsigned long long len)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t prev = __shfl_up_sync(0xffffffffu, r, 1);
    if (__any_sync(0xffffffffu, lane > 0 && lane < nr && r < prev)) return 0;
    return static_cast<uint32_t>(__popc(__ballot_sync(0xffffffffu, lane < nr && r < len)));
}

// The RCOLS store (osb200_select_segments' warp and block classes), by one whole warp over a sorted run of len keys in shared
// memory (encoded, positions in sorted_idx): lane i < nr stores column ranks[i] to obase + i of out and idx_out, or padding --
// the decoded all-ones key and the position 0xFFFFFFFF -- for a rank that takes no part (select_ranks_active).
template <typename KeyT, bool INDICES>
__device__ __forceinline__ void select_store_ranks(const KeyT* sorted, const uint32_t* sorted_idx, uint32_t len,
                                                   const uint32_t* __restrict__ ranks, uint32_t nr, KeyT* out, uint32_t* idx_out,
                                                   uint64_t obase, bool dec, KeyT ca, KeyT cb, KeyT cd)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t r = lane < nr ? ranks[lane] : 0xffffffffu;
    const uint32_t na = select_ranks_active(r, nr, len);
    if (lane < nr) {
        KeyT k = lane < na ? sorted[r] : static_cast<KeyT>(~static_cast<KeyT>(0));
        if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
        out[obase + lane] = k;
        if constexpr (INDICES) idx_out[obase + lane] = lane < na ? sorted_idx[r] : 0xFFFFFFFFu;
    }
}

// osb200_sort_segments' class counts (see segment_bin_kernel)
enum SegCount : int { kSegCountWarp = 0, kSegCountBlock1 = 1, kSegCountBlock2 = 2, kSegCountBlockList = 3, kSegCounts = 4 };
// osb200_sort_long_segments' counts after them: the long list's length, then its tiles and scan chunks (see launch_long_segments)
enum LongSegCount : int { kSegCountLong = 4, kSegCountLongTiles = 5, kSegCountLongChunks = 6, kLongSegCounts = 7 };

// INDICES (argsort): the keys come from keys_in, every payload is the key's position in its segment.
// ROWS (row sort, osb200_sort_rows): segment s is row s, [s * single_n, (s + 1) * single_n) (seg_off is not read), and the
// keys are always read from keys_in (== keys in place).  A compile-time flag rather than a runtime one, so that the
// segmented sort's and small path's instantiations compile as before (a runtime select cost the 8,192-key u64 kernel spills).
// LIST (osb200_sort_segments, segment_list_sort_kernel): the CTAs sort the segments whose ids the binning kernel put at the
// back of seg_list (entry i at seg_list[num_segments - 1 - i], seg_counts[kSegCountBlockList] of them), segment s =
// [seg_off[s], seg_off[s + 1]), reading the keys from keys_in and writing them to keys (== keys_in in place).  Both block
// classes share that list: the 2,048-key geometry takes its segments of up to kSegBlock1Max keys and the larger geometry the
// rest; a kernel whose own class count is 0 returns at once.  (A kernel of its own, sharing this body, so that the other
// modes' kernels keep their names.)
// ROW_SEL (with ROWS; osb200_topk_segments' sorted pass, topk_segment_sort_kernel): row s is sorted only if segment s =
// [seg_off[s], seg_off[s + 1]) is one the radix select wrote: inside [0, sel_n), longer than sel_min and shorter than 2^32
// keys (the binning kernel's test).  (Not its block list: with the list and its device-side count the 16,384-key
// instantiations spill; the row count is a kernel parameter, as for ROWS.)
// COLS (with ROWS; osb200_select_rows, select_rows_block_kernel): only the sorted row's columns ranks->r[0 .. count - 1] are
// stored, to [s * count, (s + 1) * count) of keys and vals.
// RCOLS (with LIST; osb200_select_segments, select_segment_block_kernel): only the sorted segment's columns
// seg_ranks[s * nr .. s * nr + nr) are stored, to [s * nr, (s + 1) * nr) of keys and vals (select_store_ranks, by warp 0).
// max_len: the caller's max_segment_len (<= T); longer segments are left as they are.
template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE, bool INDICES, bool ROWS, bool LIST, bool ROW_SEL = false,
          bool COLS = false, bool RCOLS = false>
__device__ __forceinline__ void segment_sort_body(KeyT* keys, uint32_t* vals, const unsigned long long* __restrict__ seg_off,
                                                  uint64_t num_segments, uint64_t single_n, uint32_t max_len, uint32_t begin_bit,
                                                  uint32_t places, uint32_t last_bits, const KeyCodec& codec,
                                                  const KeyT* __restrict__ keys_in, const uint32_t* __restrict__ seg_list,
                                                  const unsigned long long* __restrict__ seg_counts, uint64_t sel_n = 0,
                                                  uint32_t sel_min = 0, const SelectRanks* ranks = nullptr,
                                                  const uint32_t* __restrict__ seg_ranks = nullptr, uint32_t nr = 0)
{
    static_assert(!(ROWS && LIST), "one addressing mode");
    static_assert(!RCOLS || LIST, "the columns of listed segments");
    static_assert(!ROW_SEL || ROWS, "a selection of rows");
    static_assert(!COLS || (ROWS && !ROW_SEL), "the columns of rows");
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

    const uint64_t work = !LIST ? num_segments
                          : seg_counts[T <= kSegBlock1Max ? kSegCountBlock1 : kSegCountBlock2] ? seg_counts[kSegCountBlockList] : 0ull;
    for (uint64_t it = blockIdx.x; it < work; it += gridDim.x) {
        if constexpr (ROW_SEL) {
            const unsigned long long slo = seg_off[it], shi = seg_off[it + 1];
            if (!(slo <= shi && shi <= sel_n && shi - slo > sel_min && shi - slo <= 0xFFFFFFFFull)) continue;
        }
        const uint64_t seg = LIST ? seg_list[num_segments - 1 - it] : it;
        const uint64_t lo = ROWS ? seg * single_n : seg_off ? seg_off[seg] : 0ull;
        const uint64_t hi = ROWS ? lo + single_n : seg_off ? seg_off[seg + 1] : single_n;
        // empty / one key / longer than max_segment_len or the geometry (both the caller's contract: left untouched)
        if (hi <= lo + 1 || hi - lo > static_cast<uint64_t>(max_len) || hi - lo > static_cast<uint64_t>(T)) continue;
        const uint32_t len = static_cast<uint32_t>(hi - lo);
        if (LIST && (len <= kSegBlock1Max) != (T <= kSegBlock1Max)) continue;  // the other block class's segment

        KeyT key[K];
        uint32_t val[PAIRS ? K : 1];
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t idx = warp_off + i * 32;
            KeyT k = idx < len ? (INDICES || ROWS || LIST ? keys_in : keys)[lo + idx] : static_cast<KeyT>(0);
            if (enc) k = codec_encode<KeyT>(k, ca, cb, cd);
            key[i] = idx < len ? k : static_cast<KeyT>(~static_cast<KeyT>(0));  // padding ranks last in every pass
            if constexpr (PAIRS) val[i] = INDICES ? idx : idx < len ? vals[lo + idx] : 0u;
        }

        // ROWS, LIST: a warp's 32 keys of step i that all lie behind the row are padding, and every padding key has digit 255 in
        // every pass: ranking them costs one serialised same-address atomic per key.  Such chunks are neither counted nor
        // ranked (what they read back from slots nobody wrote is never used).  The padding of the one chunk that straddles
        // `len` is ranked; it follows every real key in tile order, so it takes the slots from `len` on, which are its own
        // positions.  (The condition is warp-uniform, so the ballot ranking sees full warps.)
        const uint32_t warp_lo = warp * (32 * K);  // this warp's chunks: [warp_lo + 32 i, warp_lo + 32 i + 32)
        const uint32_t live_chunks = ROWS || LIST ? (len > warp_lo ? (len - warp_lo + 31) / 32 : 0u) : static_cast<uint32_t>(K);
        auto live = [&](int i) { return !(ROWS || LIST) || static_cast<uint32_t>(i) < live_chunks; };
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
            for (int i = 0; i < K; ++i)
                if (live(i)) atomicAdd(&wh[digit_of(key[i], shift, dmask)], 1u);
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
                if (!live(i)) continue;
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
        if constexpr (COLS) {  // the last pass ended with a block barrier: the sorted row is in sm.sorted
            const uint32_t rk = select_rank_of(*ranks, static_cast<uint32_t>(tid));
            if (static_cast<uint32_t>(tid) < ranks->count) {
                KeyT k = sm.sorted[rk];
                if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
                keys[seg * ranks->count + tid] = k;
                if constexpr (PAIRS) vals[seg * ranks->count + tid] = sm.sorted_val[rk];
            }
            continue;
        }
        if constexpr (RCOLS) {  // (as COLS)
            if (warp == 0)
                select_store_ranks<KeyT, PAIRS>(sm.sorted, sm.sorted_val, len, seg_ranks + seg * nr, nr, keys, vals, seg * nr, dec, ca,
                                                cb, cd);
            continue;
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

// (ROWS, LIST: one resident CTA per SM is stated, or ptxas caps some 512-thread instantiations at 64 registers and spills.)
template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE, bool INDICES = false, bool ROWS = false>
__global__ void __launch_bounds__(WARPS * 32, ROWS ? 1 : 0)
segment_sort_kernel(KeyT* keys, uint32_t* vals, const unsigned long long* __restrict__ seg_off, uint64_t num_segments,
                    uint64_t single_n, uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits, KeyCodec codec,
                    const KeyT* __restrict__ keys_in)
{
    segment_sort_body<KeyT, PAIRS, K, WARPS, RANK_MODE, INDICES, ROWS, false>(keys, vals, seg_off, num_segments, single_n, max_len,
                                                                             begin_bit, places, last_bits, codec, keys_in, nullptr,
                                                                             nullptr);
}

template <typename KeyT, bool PAIRS, int K, int WARPS, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(WARPS * 32, 1)
segment_list_sort_kernel(KeyT* keys, uint32_t* vals, const unsigned long long* __restrict__ seg_off, uint64_t num_segments,
                         uint32_t max_len, uint32_t places, KeyCodec codec, const KeyT* __restrict__ keys_in,
                         const uint32_t* __restrict__ seg_list, const unsigned long long* __restrict__ seg_counts)
{
    segment_sort_body<KeyT, PAIRS, K, WARPS, RANK_MODE, INDICES, false, true>(keys, vals, seg_off, num_segments, 0, max_len, 0u,
                                                                             places, 8u, codec, keys_in, seg_list, seg_counts);
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
// 16-bit keys: the small-n path of their sorts (one segment of up to 16,384 keys) and the row sort; no segmented sort
template <> struct SegGeomN<uint16_t, 1> { static constexpr int K = 8,  WARPS = 8; };   //  2,048 keys (row sort only)
template <> struct SegGeomN<uint16_t, 2> { static constexpr int K = 32, WARPS = 16; };  // 16,384 keys, 512 threads
template <typename KeyT, bool PAIRS, int SIZE, bool INDICES = false, bool ROWS = false, bool LIST = false>
struct SegShape {
    using Key = KeyT;
    static constexpr bool pairs = PAIRS, indices = INDICES, has_hot = false;
    using G = SegGeomN<KeyT, SIZE>;
    using S = SegSmem<KeyT, PAIRS, G::K, G::WARPS>;
    static constexpr uint32_t T = S::T;  // the longest segment it sorts
    static constexpr size_t smem = sizeof(S);
    static constexpr int ctas_per_sm = SIZE == 2 ? 2 : 8;
    template <int RANK_MODE, bool HOT = false>
    static constexpr auto kernel()
    {
        if constexpr (LIST) return segment_list_sort_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, INDICES>;
        else return segment_sort_kernel<KeyT, PAIRS, G::K, G::WARPS, RANK_MODE, INDICES, ROWS>;
    }
};
template <typename KeyT, int SIZE, bool INDICES> using RowShape = SegShape<KeyT, INDICES, SIZE, INDICES, true>;
template <typename KeyT, int SIZE, bool INDICES> using ListShape = SegShape<KeyT, INDICES, SIZE, INDICES, false, true>;
static_assert(SegShape<uint16_t, false, 1>::T == kSegBlock1Max && SegShape<uint32_t, false, 1>::T == kSegBlock1Max &&
                  SegShape<uint64_t, false, 1>::T == kSegBlock1Max,
              "the first block class of osb200_sort_segments is the 2,048-key geometry of every key width");

// Each kind of sort lists its geometries smallest first: the launchers take the first one that holds the longest segment.
// Segmented sort and small path (launch_segment_sort).
using SegShapes = TypeList<
    // segmented sort and small path: 32-bit keys and pairs, 64-bit keys
    SegShape<uint32_t, false, 0>, SegShape<uint32_t, false, 1>, SegShape<uint32_t, false, 2>,
    SegShape<uint32_t, true, 0>, SegShape<uint32_t, true, 1>, SegShape<uint32_t, true, 2>,
    SegShape<uint64_t, false, 0>, SegShape<uint64_t, false, 1>, SegShape<uint64_t, false, 2>,
    // small path only (the single segment of a sort of at most one tile): 16-bit keys and pairs, 64-bit pairs, every argsort
    SegShape<uint16_t, false, 2>, SegShape<uint16_t, true, 2>, SegShape<uint64_t, true, 2>,
    SegShape<uint16_t, true, 2, true>, SegShape<uint32_t, true, 2, true>, SegShape<uint64_t, true, 2, true>>;
// Row sort, block path (launch_row_sort): keys only and with indices.
using RowShapes = TypeList<
    RowShape<uint16_t, 1, false>, RowShape<uint16_t, 2, false>, RowShape<uint16_t, 1, true>, RowShape<uint16_t, 2, true>,
    RowShape<uint32_t, 1, false>, RowShape<uint32_t, 2, false>, RowShape<uint32_t, 1, true>, RowShape<uint32_t, 2, true>,
    RowShape<uint64_t, 1, false>, RowShape<uint64_t, 2, false>, RowShape<uint64_t, 1, true>, RowShape<uint64_t, 2, true>>;
// Segment sort by offsets (launch_sort_segments), block classes: keys only and with indices.
using ListShapes = TypeList<
    ListShape<uint16_t, 1, false>, ListShape<uint16_t, 2, false>, ListShape<uint16_t, 1, true>, ListShape<uint16_t, 2, true>,
    ListShape<uint32_t, 1, false>, ListShape<uint32_t, 2, false>, ListShape<uint32_t, 1, true>, ListShape<uint32_t, 2, true>,
    ListShape<uint64_t, 1, false>, ListShape<uint64_t, 2, false>, ListShape<uint64_t, 1, true>, ListShape<uint64_t, 2, true>>;

// the longest segment of key_bytes-wide keys that a shape of the list sorts; 0 if there is none
template <typename... Shapes>
static uint32_t capacity_of(TypeList<Shapes...> shapes, int key_bytes)
{
    uint32_t cap = 0;
    for_each_type(shapes, [&](auto s) {
        using S = decltype(s);
        if (key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::T > cap) cap = S::T;
        return cudaSuccess;
    });
    return cap;
}

uint32_t segment_sort_capacity(int key_bytes) { return capacity_of(SegShapes{}, key_bytes); }
uint32_t row_sort_capacity(int key_bytes) { return capacity_of(RowShapes{}, key_bytes); }

template <typename Shape>
static cudaError_t launch_seg(Shape, void* keys, uint32_t* vals, const unsigned long long* seg_off, uint64_t num_segments,
                              uint64_t single_n, uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits,
                              const KeyCodec& codec, int rank_mode, int sm_count, cudaStream_t stream, const void* keys_in)
{
    using KeyT = typename Shape::Key;
    const uint64_t cap = static_cast<uint64_t>(sm_count) * Shape::ctas_per_sm;
    const unsigned grid = static_cast<unsigned>(num_segments < cap ? num_segments : cap);
    return with_rank_mode(rank_mode, [&](auto r) {
        const auto kern = Shape::template kernel<decltype(r)::value>();
        kern<<<grid, Shape::S::THREADS, Shape::smem, stream>>>(static_cast<KeyT*>(keys), vals, seg_off, num_segments, single_n,
                                                              max_len, begin_bit, places, last_bits, codec,
                                                              static_cast<const KeyT*>(keys_in));
        return cudaGetLastError();
    });
}

cudaError_t launch_segment_sort(void* keys, uint32_t* vals, int key_bytes, const unsigned long long* seg_off, uint64_t num_segments,
                                uint64_t single_n, uint32_t max_len, uint32_t begin_bit, uint32_t places, uint32_t last_bits,
                                const KeyCodec* codec_in, int rank_mode, int sm_count, cudaStream_t stream, const void* keys_in)
{
    if (num_segments == 0) return cudaSuccess;
    const bool pairs = vals != nullptr, indices = keys_in != nullptr;
    // argsort, 16-bit keys and 64-bit pairs: only the single segment of a small sort
    if ((indices || key_bytes == 2 || (key_bytes == 8 && pairs)) && (seg_off || num_segments != 1)) return cudaErrorInvalidValue;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    return find_type(
        SegShapes{},
        [&](auto s) {
            using S = decltype(s);
            return key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::pairs == pairs && S::indices == indices &&
                   max_len <= S::T;
        },
        [&](auto s) {
            return launch_seg(s, keys, vals, seg_off, num_segments, single_n, max_len, begin_bit, places, last_bits, codec, rank_mode,
                              sm_count, stream, keys_in);
        });
}

// =====================================================================================================
// Row sort, warp path: rows of at most 256 keys, ONE WARP sorts one row at a time (grid-stride over the rows).  The block
// path would pad such a row to a block's tile and pay six block barriers and an 8 x 256-bin histogram clear and scan per
// pass; a warp needs no block barrier at all.  Reference: SplitSort packs short segments at warp level
// (SegSort/SplitSort/SplitSort.cuh:31-130); the ranking here is the DigitBinningPass's (warp_rank_and_count), so the order is
// stable by the same lane-order property (or the ballot mode).
//
// Per pass: count the row's digits in the warp's own 256 bins (real keys only), one lane scans 8 bins and the warp scans
// the lane totals with shuffles, every key is ranked in tile order (key i*32 + lane) and stored at its slot in the warp's
// staging area, and read back in tile order.  The padding keys (all ones) rank after every real key, at slots >= row_len.
// A pass in which one bin holds the whole row would leave the order as it is, so the warp skips it: 64-bit rows of small
// values execute only the passes of their low digits.
// =====================================================================================================
constexpr int kRowWarps = 8;  // warps per CTA (independent: no block barrier)

template <typename KeyT, int K, bool INDICES>
struct RowWarpSmem {  // one per warp: 1 KB of bins + the staging area (at most 4 KB: 64-bit keys with indices, K = 8)
    alignas(16) uint32_t hist[kRadix];
    alignas(16) KeyT keys[32 * K];
    uint32_t idx[INDICES ? 32 * K : 1];
};
template <typename KeyT, int K, bool INDICES>
constexpr size_t kRowWarpSmemBytes = kRowWarps * sizeof(RowWarpSmem<KeyT, K, INDICES>);  // a CTA's dynamic shared memory

// The keys per lane of a warp that sorts a run of len <= kRowWarpMaxLen keys: f(std::integral_constant<int, K>{}), K = 1, 2,
// 4 or 8.
template <typename F>
static cudaError_t with_warp_k(uint32_t len, F&& f)
{
    if (len <= 32) return f(std::integral_constant<int, 1>{});
    if (len <= 64) return f(std::integral_constant<int, 2>{});
    if (len <= 128) return f(std::integral_constant<int, 4>{});
    return f(std::integral_constant<int, 8>{});
}

// What a warp keeps across the runs it sorts: its lane, lane mask, the hist of its staging area as uint4 (lane l owns bins
// 8l .. 8l+7: h4[2l], h4[2l+1]) and the codec as key-wide words.
template <typename KeyT>
struct WarpSortCtx {
    int lane;
    uint32_t lt;
    uint4* h4;
    KeyT ca, cb, cd;
    bool enc, dec;
};

template <typename KeyT>
__device__ __forceinline__ WarpSortCtx<KeyT> warp_sort_ctx(uint32_t* hist, const KeyCodec& codec)
{
    return {static_cast<int>(threadIdx.x & 31), lanemask_lt(), reinterpret_cast<uint4*>(hist), static_cast<KeyT>(codec.a),
            static_cast<KeyT>(codec.b), static_cast<KeyT>(codec.d), (codec.flags & kCodecEncodeOnLoad) != 0,
            (codec.flags & kCodecDecodeOnStore) != 0};
}

// One warp sorts the len <= 32 K keys [base, base + len) of `in` into the same positions of `out` (and their positions within
// the run into idx_out), in the warp's own staging area sm.  The row kernel calls it per row, the segment kernel per segment.
// TOPK (top-k, topk_warp_kernel; with INDICES): only the first `keep` sorted keys and payloads are stored, at
// [obase, obase + keep) of out and idx_out; the payloads are loaded from idx_in[base ..] when idx_in is not null, else
// they are the positions in the run.  (A compile-time flag, so that the other kernels' instantiations compile as before.)
// PAD (with TOPK; osb200_topk_segments, whose keep may pass len): the stored columns at or past len are padding, the decoded
// all-ones key that the padding carries through the sort and the position 0xFFFFFFFF.
// COLS (osb200_select_rows, select_rows_warp_kernel; not with TOPK): only the sorted run's columns ranks->r[0 .. count - 1] are
// stored, at [obase, obase + count) of out and (with INDICES) idx_out.
// RCOLS (osb200_select_segments, select_segment_warp_kernel; not with TOPK or COLS): only the sorted run's columns
// seg_ranks[0 .. nr) are stored, at [obase, obase + nr), by select_store_ranks.
template <typename KeyT, int K, int RANK_MODE, bool INDICES, bool TOPK = false, bool PAD = false, bool COLS = false,
          bool RCOLS = false>
__device__ __forceinline__ void warp_sort_run(RowWarpSmem<KeyT, K, INDICES>& sm, const WarpSortCtx<KeyT>& x, const KeyT* in, KeyT* out,
                                              uint32_t* idx_out, uint64_t base, uint32_t len, const uint32_t* idx_in = nullptr,
                                              uint64_t obase = 0, uint32_t keep = 0, const SelectRanks* ranks = nullptr,
                                              const uint32_t* seg_ranks = nullptr, uint32_t nr = 0)
{
    static_assert(!TOPK || INDICES, "top-k stores positions");
    static_assert(!PAD || TOPK, "padding is a top-k store");
    static_assert(!(COLS && TOPK), "one store");
    static_assert(!(RCOLS && (TOPK || COLS)), "one store");
    const int lane = x.lane;
    uint4* h4 = x.h4;
    const uint32_t lt = x.lt;
    const KeyT ca = x.ca, cb = x.cb, cd = x.cd;
    const bool enc = x.enc, dec = x.dec;

    KeyT key[K];
    uint32_t val[INDICES ? K : 1];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const uint32_t idx = i * 32 + lane;
        KeyT k = idx < len ? in[base + idx] : static_cast<KeyT>(0);
        if (enc) k = codec_encode<KeyT>(k, ca, cb, cd);
        key[i] = idx < len ? k : static_cast<KeyT>(~static_cast<KeyT>(0));
        if constexpr (TOPK) val[i] = idx_in && idx < len ? idx_in[base + idx] : idx;
        else if constexpr (INDICES) val[i] = idx;
    }
#pragma unroll 1
    for (uint32_t shift = 0; shift < sizeof(KeyT) * 8; shift += 8) {
        h4[2 * lane] = make_uint4(0, 0, 0, 0);
        h4[2 * lane + 1] = make_uint4(0, 0, 0, 0);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < K; ++i)
            if (i * 32 + lane < len) atomicAdd(&sm.hist[digit_of(key[i], shift)], 1u);
        __syncwarp();
        const uint4 lo4 = h4[2 * lane], hi4 = h4[2 * lane + 1];
        const uint32_t c[8] = {lo4.x, lo4.y, lo4.z, lo4.w, hi4.x, hi4.y, hi4.z, hi4.w};
        uint32_t sum = 0;
        bool whole = false;
#pragma unroll
        for (int j = 0; j < 8; ++j) { sum += c[j]; whole |= c[j] == len; }
        if (__any_sync(0xffffffffu, whole)) continue;  // one digit for the whole run: this pass keeps the order
        uint32_t incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        uint32_t run = incl - sum, e[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) { e[j] = run; run += c[j]; }
        h4[2 * lane] = make_uint4(e[0], e[1], e[2], e[3]);
        h4[2 * lane + 1] = make_uint4(e[4], e[5], e[6], e[7]);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < K; ++i) {
            const uint32_t slot = warp_rank_and_count<RANK_MODE>(sm.hist, digit_of(key[i], shift), lt);
            sm.keys[slot] = key[i];
            if constexpr (INDICES) sm.idx[slot] = val[i];
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < K; ++i) {
            key[i] = sm.keys[i * 32 + lane];
            if constexpr (INDICES) val[i] = sm.idx[i * 32 + lane];
        }
        __syncwarp();
    }
    if constexpr (COLS) {
        // the registers hold the sorted run in tile order (the staging area does not when no pass moved a key): through
        // the staging area to the lanes that store a column
#pragma unroll
        for (int i = 0; i < K; ++i) {
            sm.keys[i * 32 + lane] = key[i];
            if constexpr (INDICES) sm.idx[i * 32 + lane] = val[i];
        }
        __syncwarp();
        const uint32_t rk = select_rank_of(*ranks, static_cast<uint32_t>(lane));
        if (static_cast<uint32_t>(lane) < ranks->count) {
            KeyT k = sm.keys[rk];
            if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
            out[obase + lane] = k;
            if constexpr (INDICES) idx_out[obase + lane] = sm.idx[rk];
        }
        __syncwarp();  // the next run's passes overwrite the staging area
        return;
    }
    if constexpr (RCOLS) {  // (as COLS)
#pragma unroll
        for (int i = 0; i < K; ++i) {
            sm.keys[i * 32 + lane] = key[i];
            if constexpr (INDICES) sm.idx[i * 32 + lane] = val[i];
        }
        __syncwarp();
        select_store_ranks<KeyT, INDICES>(sm.keys, sm.idx, len, seg_ranks, nr, out, idx_out, obase, dec, ca, cb, cd);
        __syncwarp();
        return;
    }
#pragma unroll
    for (int i = 0; i < K; ++i) {
        const uint32_t idx = i * 32 + lane;
        if constexpr (TOPK) {
            if (idx < keep) {
                KeyT k = key[i];
                if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
                out[obase + idx] = k;
                idx_out[obase + idx] = PAD && idx >= len ? 0xFFFFFFFFu : val[i];
            }
        } else if (idx < len) {
            KeyT k = key[i];
            if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
            out[base + idx] = k;
            if constexpr (INDICES) idx_out[base + idx] = val[i];
        }
    }
}

template <typename KeyT, int K, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(kRowWarps * 32)
row_sort_warp_kernel(const KeyT* in, KeyT* out, uint32_t* __restrict__ idx_out, uint64_t num_rows, uint32_t row_len,
                     KeyCodec codec)
{
    using W = RowWarpSmem<KeyT, K, INDICES>;
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    W& sm = reinterpret_cast<W*>(s_raw)[warp];
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(sm.hist, codec);
    for (uint64_t row = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; row < num_rows;
         row += static_cast<uint64_t>(gridDim.x) * kRowWarps)
        warp_sort_run<KeyT, K, RANK_MODE, INDICES>(sm, x, in, out, idx_out, row * row_len, row_len);
}

cudaError_t launch_row_sort(const void* keys_in, void* keys_out, uint32_t* indices, uint64_t num_rows, uint32_t row_len,
                            int key_bytes, const KeyCodec* codec_in, int rank_mode, bool block_only, int sm_count,
                            cudaStream_t stream)
{
    if (num_rows == 0 || row_len == 0) return cudaSuccess;
    if (row_len > row_sort_capacity(key_bytes)) return cudaErrorInvalidValue;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    if (row_len <= kRowWarpMaxLen && !block_only) {
        return with_key_type(TypeList<uint16_t, uint32_t, uint64_t>{}, key_bytes, [&](auto k) {
            return with_rank_mode(rank_mode, [&](auto r) {
                return with_warp_k(row_len, [&](auto kk) {
                    using KeyT = decltype(k);
                    constexpr int R = decltype(r)::value, K = decltype(kk)::value;
                    auto go = [&](auto ind) {
                        constexpr bool I = decltype(ind)::value;
                        return launch_resident<row_sort_warp_kernel<KeyT, K, R, I>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, K, I>>(
                            (num_rows + kRowWarps - 1) / kRowWarps, sm_count, stream, static_cast<const KeyT*>(keys_in),
                            static_cast<KeyT*>(keys_out), indices, num_rows, row_len, codec);
                    };
                    return indices ? go(std::true_type{}) : go(std::false_type{});
                });
            });
        });
    }
    // block path: segment s of segment_sort_kernel is row s
    return find_type(
        RowShapes{},
        [&](auto s) {
            using S = decltype(s);
            return key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::indices == (indices != nullptr) && row_len <= S::T;
        },
        [&](auto s) {
            return launch_seg(s, keys_out, indices, nullptr, num_rows, row_len, row_len, 0u, static_cast<uint32_t>(key_bytes), 8u, codec,
                              rank_mode, sm_count, stream, keys_in);
        });
}

// =====================================================================================================
// Segment sort by offsets (osb200_sort_segments).  The host does not know the segment lengths, so a binning kernel reads
// the offsets once and sorts each segment into a class by its length (reference: SplitSort's BinSimple,
// SegSort/SplitSort/SplitSort.cuh:618-668, here without its host round trip):
//   0 keys: nothing; 1 key: written here; 2-256: the warp list; 257 - kSegBlock1Max and beyond: the block list;
//   offsets that decrease or pass n, and segments longer than max_len: skipped (never written).
// The lists share one array of num_segments ids: the warp list grows from its front, the block list from its back, so
// neither can overflow.  counts = [warp list, 2,048-key class, larger class, block list]; the class kernels read their
// count on the device, so the host enqueues them without waiting, and each segment of two or more keys is in exactly one
// list and sorted by exactly one kernel.
// TOPK (osb200_topk_segments, topk_segment_bin_kernel): every segment is listed, for every one has k output columns to
// fill.  Segments of warp_max + 1 to 2^32 - 1 keys inside [0, n) go to the block list (counted as the 2,048-key class);
// all others -- up to warp_max keys, empty, and invalid ones, which the warp class treats as empty -- to the warp list.
// Nothing is written here but the lists and counts (keys_in, keys_out, idx_out and max_len are not used).
// LONG (osb200_sort_long_segments, long_segment_bin_kernel): segments of long_min to max_len keys go to the long list
// instead (ids in arrival order, at most long_cap of them; counts[kSegCountLong] counts them all), the shorter ones to the
// classes as above.
// SEL (osb200_select_segments, select_segment_bin_kernel): every segment is listed, as with TOPK.  Segments of 2 to max_len
// keys inside [0, n) go to the block classes by length (with LONG those of long_min or more to the long list) unless they
// have at most warp_max keys; all others -- fewer than two keys, empty, and invalid ones -- to the warp list.
// =====================================================================================================
template <typename KeyT, bool TOPK, bool LONG = false, bool SEL = false>
__device__ __forceinline__ void segment_bin_body(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n,
                                                 uint32_t max_len, uint32_t* __restrict__ list,
                                                 unsigned long long* __restrict__ counts, const KeyT* keys_in, KeyT* keys_out,
                                                 uint32_t* idx_out, uint32_t warp_max, uint32_t long_min = 0,
                                                 uint32_t* __restrict__ long_list = nullptr, uint64_t long_cap = 0)
{
    const uint32_t lane = threadIdx.x & 31, lt = lanemask_lt();
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    // whole warps step together, so the ballots below always see 32 lanes
    for (uint64_t base = static_cast<uint64_t>(blockIdx.x) * blockDim.x + (threadIdx.x & ~31u); base < num_segments; base += stride) {
        const uint64_t s = base + lane;
        int cls = -1;  // 0: warp list, 1 / 2: block classes
        if (TOPK && s < num_segments) {
            const unsigned long long lo = off[s], hi = off[s + 1];
            cls = lo <= hi && hi <= n && hi - lo > warp_max && hi - lo <= 0xFFFFFFFFull ? 1 : 0;
        } else if (SEL && s < num_segments) {
            const unsigned long long lo = off[s], hi = off[s + 1], len = hi - lo;
            cls = !(lo <= hi && hi <= n && len <= max_len) || len < 2 ? 0
                  : LONG && len >= long_min                          ? 3
                  : len <= warp_max                                  ? 0
                  : len <= kSegBlock1Max                             ? 1
                                                                     : 2;
        } else if (s < num_segments) {
            const unsigned long long lo = off[s], hi = off[s + 1];
            if (lo <= hi && hi <= n && hi - lo <= max_len) {
                const uint32_t len = static_cast<uint32_t>(hi - lo);
                if (len == 1) {
                    if (keys_out != keys_in) keys_out[lo] = keys_in[lo];
                    if (idx_out) idx_out[lo] = 0u;
                } else if (LONG && len >= long_min) {
                    cls = 3;
                } else if (len > 1) {
                    cls = len <= kRowWarpMaxLen ? 0 : len <= kSegBlock1Max ? 1 : 2;
                }
            }
        }
        if constexpr (LONG) {
            const uint32_t l = __ballot_sync(0xffffffffu, cls == 3);
            unsigned long long lpos = 0;
            if (lane == 0 && l) lpos = atomicAdd(&counts[kSegCountLong], static_cast<unsigned long long>(__popc(l)));
            lpos = __shfl_sync(0xffffffffu, lpos, 0) + __popc(l & lt);
            if (cls == 3 && lpos < long_cap) long_list[lpos] = static_cast<uint32_t>(s);
        }
        const uint32_t w = __ballot_sync(0xffffffffu, cls == 0), b = __ballot_sync(0xffffffffu, cls > 0 && (!LONG || cls < 3));
        const uint32_t b1 = __ballot_sync(0xffffffffu, cls == 1), b2 = b & ~b1;
        unsigned long long wpos = 0, bpos = 0;
        if (lane == 0) {
            if (w) wpos = atomicAdd(&counts[kSegCountWarp], static_cast<unsigned long long>(__popc(w)));
            if (b) bpos = atomicAdd(&counts[kSegCountBlockList], static_cast<unsigned long long>(__popc(b)));
            if (b1) atomicAdd(&counts[kSegCountBlock1], static_cast<unsigned long long>(__popc(b1)));
            if (b2) atomicAdd(&counts[kSegCountBlock2], static_cast<unsigned long long>(__popc(b2)));
        }
        wpos = __shfl_sync(0xffffffffu, wpos, 0);
        bpos = __shfl_sync(0xffffffffu, bpos, 0);
        if (cls == 0) list[wpos + __popc(w & lt)] = static_cast<uint32_t>(s);
        if (cls > 0 && (!LONG || cls < 3)) list[num_segments - 1 - (bpos + __popc(b & lt))] = static_cast<uint32_t>(s);
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(256)
segment_bin_kernel(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n, uint32_t max_len,
                   uint32_t* __restrict__ list, unsigned long long* __restrict__ counts, const KeyT* keys_in, KeyT* keys_out,
                   uint32_t* idx_out)
{
    segment_bin_body<KeyT, false>(off, num_segments, n, max_len, list, counts, keys_in, keys_out, idx_out, kRowWarpMaxLen);
}

// The warp class: one warp per segment of the warp list (grid-stride), 1, 2, 4 or 8 keys per lane by the segment's length.
// Each warp's staging area is sized for 8.
template <typename KeyT, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(kRowWarps * 32)
segment_sort_warp_kernel(const KeyT* in, KeyT* out, uint32_t* __restrict__ idx_out, const unsigned long long* __restrict__ off,
                         const uint32_t* __restrict__ list, const unsigned long long* __restrict__ counts, KeyCodec codec)
{
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    unsigned char* wsm = s_raw + warp * sizeof(RowWarpSmem<KeyT, 8, INDICES>);  // every K's layout starts with the same hist
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(reinterpret_cast<uint32_t*>(wsm), codec);
    const uint64_t count = counts[kSegCountWarp];
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; i < count; i += static_cast<uint64_t>(gridDim.x) * kRowWarps) {
        const uint32_t s = list[i];
        const uint64_t lo = off[s];
        const uint32_t len = static_cast<uint32_t>(off[s + 1] - lo);
        if (len <= 32)
            warp_sort_run<KeyT, 1, RANK_MODE, INDICES>(*reinterpret_cast<RowWarpSmem<KeyT, 1, INDICES>*>(wsm), x, in, out, idx_out, lo, len);
        else if (len <= 64)
            warp_sort_run<KeyT, 2, RANK_MODE, INDICES>(*reinterpret_cast<RowWarpSmem<KeyT, 2, INDICES>*>(wsm), x, in, out, idx_out, lo, len);
        else if (len <= 128)
            warp_sort_run<KeyT, 4, RANK_MODE, INDICES>(*reinterpret_cast<RowWarpSmem<KeyT, 4, INDICES>*>(wsm), x, in, out, idx_out, lo, len);
        else
            warp_sort_run<KeyT, 8, RANK_MODE, INDICES>(*reinterpret_cast<RowWarpSmem<KeyT, 8, INDICES>*>(wsm), x, in, out, idx_out, lo, len);
    }
}

static cudaError_t launch_segment_classes(const void* keys_in, void* keys_out, uint32_t* indices, const unsigned long long* off,
                                          uint64_t num_segments, uint32_t max_len, int key_bytes, const KeyCodec& codec,
                                          int rank_mode, int sm_count, uint32_t* list, unsigned long long* counts,
                                          cudaStream_t stream);

cudaError_t launch_sort_segments(const void* keys_in, void* keys_out, uint32_t* indices, uint64_t n,
                                 const unsigned long long* off, uint64_t num_segments, uint32_t max_len, int key_bytes,
                                 const KeyCodec* codec_in, int rank_mode, int sm_count, uint32_t* list,
                                 unsigned long long* counts, cudaStream_t stream)
{
    if (num_segments == 0 || max_len == 0) return cudaSuccess;
    if (max_len > row_sort_capacity(key_bytes)) return cudaErrorInvalidValue;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    cudaError_t e = cudaMemsetAsync(counts, 0, kSegCounts * sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    e = with_key_type(TypeList<uint16_t, uint32_t, uint64_t>{}, key_bytes, [&](auto k) {
        using KeyT = decltype(k);
        segment_bin_kernel<KeyT><<<capped_grid(num_segments, 256, static_cast<uint64_t>(sm_count) * 8), 256, 0, stream>>>(
            off, num_segments, n, max_len, list, counts, static_cast<const KeyT*>(keys_in), static_cast<KeyT*>(keys_out), indices);
        return cudaGetLastError();
    });
    if (e != cudaSuccess || max_len < 2) return e;
    return launch_segment_classes(keys_in, keys_out, indices, off, num_segments, max_len, key_bytes, codec, rank_mode, sm_count,
                                  list, counts, stream);
}

// The class kernels of the binned segments of 2 to max_len <= row_sort_capacity keys: the warp list, then the block classes
// that max_len reaches.
static cudaError_t launch_segment_classes(const void* keys_in, void* keys_out, uint32_t* indices, const unsigned long long* off,
                                          uint64_t num_segments, uint32_t max_len, int key_bytes, const KeyCodec& codec,
                                          int rank_mode, int sm_count, uint32_t* list, unsigned long long* counts,
                                          cudaStream_t stream)
{
    cudaError_t e = with_key_type(TypeList<uint16_t, uint32_t, uint64_t>{}, key_bytes, [&](auto k) {
        return with_rank_mode(rank_mode, [&](auto r) {
            using KeyT = decltype(k);
            constexpr int R = decltype(r)::value;
            auto go = [&](auto ind) {  // each warp's staging area is sized for 8 keys per lane
                constexpr bool I = decltype(ind)::value;
                return launch_resident<segment_sort_warp_kernel<KeyT, R, I>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, 8, I>>(
                    kAllResident, sm_count, stream, static_cast<const KeyT*>(keys_in), static_cast<KeyT*>(keys_out), indices, off,
                    list, counts, codec);
            };
            return indices ? go(std::true_type{}) : go(std::false_type{});
        });
    });
    // the block classes that max_len reaches: both share the block list, each takes its own lengths
    for (int cls = 1; e == cudaSuccess && cls <= 2; ++cls) {
        if (max_len <= (cls == 1 ? kRowWarpMaxLen : kSegBlock1Max)) break;
        e = find_type(
            ListShapes{},
            [&](auto s) {
                using S = decltype(s);
                return key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::indices == (indices != nullptr) &&
                       (S::T == kSegBlock1Max) == (cls == 1);
            },
            [&](auto s) {
                using S = decltype(s);
                using KeyT = typename S::Key;
                return with_rank_mode(rank_mode, [&](auto r) {
                    return launch_resident<S::template kernel<decltype(r)::value>(), S::S::THREADS, S::smem>(
                        kAllResident, sm_count, stream, static_cast<KeyT*>(keys_out), indices, off, num_segments, max_len,
                        static_cast<uint32_t>(key_bytes), codec, static_cast<const KeyT*>(keys_in), list, counts);
                });
            });
    }
    return e;
}

// =====================================================================================================
// Long rows (osb200_sort_long_rows): an LSD radix sort of every row, reduce-then-scan within the row, so no tile ever
// waits on another one (DESIGN §4.16).
//
// Row r is cut into tpr = ceil(row_len / kLongRowTile) tiles that never straddle rows; the last one is ragged.  The plan is
// the DigitBinningPass's (GlobalHistogram over all n keys, the scan's SortPlan: a place on which every key of the call agrees
// is skipped, and the parity / first_exec / last_exec of the executed places give every pass its source, destination and
// codec).  Per executed place p:
//   count    each tile counts digit p of its keys into cnt[row][digit][tile] (digit-major within the row);
//   scan     a segmented exclusive scan of each row's 256 * tpr counts, in place: chunk sums, a scan of the chunk sums within
//            the row, then the chunks with their prefixes (one level when a row's counts fit one chunk).  A long row is
//            spread over as many CTAs as it has chunks;
//   scatter  each tile ranks its keys stably in shared memory (the DigitBinningPass's warp ranking, both rank modes), stages
//            them in digit order and writes key j of digit d to row base + cnt[row][d][tile] + (j - the tile's first slot of
//            d): a warp's stores are consecutive within a digit run.  Indices move with their keys; the first executed pass
//            reads keys_in and makes each index from the key's position within the row.
// Every kernel returns at once when the plan skips its place.  copy home: an odd number of executed passes leaves the rows
// in the alternate buffers; none leaves keys_in sorted as it is (indices 0 .. row_len - 1 per row).
// =====================================================================================================
constexpr int kLongWarps = 16, kLongThreads = kLongWarps * 32, kLongK = static_cast<int>(kLongRowTile) / kLongThreads;
static_assert(kLongK * kLongThreads == static_cast<int>(kLongRowTile), "a tile is kLongK keys per thread");
constexpr int kLongScanPer = 8;                                         // counts per thread of a scan chunk
constexpr uint32_t kLongChunk = kLongThreads * kLongScanPer;            // counts per scan chunk
static_assert(kRadix % kLongScanPer == 0, "a row's counts are whole threads' worth");

uint64_t long_rows_scratch_bytes(uint64_t num_rows, uint32_t row_len)
{
    const uint64_t tpr = (static_cast<uint64_t>(row_len) + kLongRowTile - 1) / kLongRowTile;
    const uint64_t cpr = (tpr * kRadix + kLongChunk - 1) / kLongChunk;
    // the tile counts, then (when a row has more than one chunk) the chunk sums, 16-byte aligned
    return (num_rows * tpr * kRadix + (cpr > 1 ? num_rows * cpr + 3 : 0)) / 4 * 4 * sizeof(uint32_t);
}

// What an executed pass of the plan reads and writes: keys_in on the first executed place, else the buffer an even
// number of earlier executed passes left the keys in (keys_out, or alt when odd).
struct LongPass { bool skip, first, last, from_alt; };
__device__ __forceinline__ LongPass long_pass(const SortPlan* plan, uint32_t place)
{
    const SortPlan pl = *plan;
    return {((pl.skip_mask >> place) & 1u) != 0, place == pl.first_exec, place == pl.last_exec, plan_src_is_alt(pl, place)};
}

// The GlobalHistogram reads 16-byte vectors; the keys before the first 16-byte boundary of a naturally aligned input are
// counted here (at most 7 of them).
template <typename KeyT>
__global__ void __launch_bounds__(32)
long_rows_head_hist_kernel(const KeyT* __restrict__ keys, uint32_t head, unsigned long long* __restrict__ ghist, KeyCodec codec)
{
    if (threadIdx.x >= head) return;
    KeyT k = keys[threadIdx.x];
    if (codec.flags & kCodecEncodeOnLoad)
        k = codec_encode<KeyT>(k, static_cast<KeyT>(codec.a), static_cast<KeyT>(codec.b), static_cast<KeyT>(codec.d));
#pragma unroll
    for (int p = 0; p < static_cast<int>(sizeof(KeyT)); ++p) atomicAdd(&ghist[p * kRadix + digit_of(k, 8u * p)], 1ull);
}

// Where the long path's tiles are.  LongRowGeo: row r is tiles r * tpr .. (r + 1) * tpr - 1, its counts start at
// r * 256 * tpr, its scan chunks at r * cpr.  LongSegGeo (osb200_sort_long_segments) finds a tile's segment on the device.
// Both give: tiles() and tile(g) (the start lo of g's row or segment, g's tile t in it, its first key t0 and length len),
// cnt_index(tile, d) (where the tile's count of digit d is), chunks() and chunk(g) (the counts of the row or segment that
// chunk g covers, and its first count c0), groups() and group(i) (the chunk sums of row or segment i).
struct LongRowGeo {
    uint64_t num_rows;
    uint32_t row_len, tpr;
    uint64_t row_counts;
    uint32_t cpr;
    struct Tile { uint64_t r, lo; uint32_t t, t0, len; };
    struct Chunk { uint64_t base, c0, row_counts; };
    struct Group { uint64_t first; uint32_t count; };
    __device__ __forceinline__ uint64_t tiles() const { return num_rows * tpr; }
    __device__ __forceinline__ Tile tile(uint64_t g) const
    {
        const uint64_t r = g / tpr;
        const uint32_t t = static_cast<uint32_t>(g - r * tpr), t0 = t * kLongRowTile;
        const uint32_t len = row_len - t0 < kLongRowTile ? row_len - t0 : kLongRowTile;
        return {r, r * row_len, t, t0, len};
    }
    template <typename D>  // the digit as the caller holds it (a thread index): the row kernels' arithmetic as it was
    __device__ __forceinline__ uint64_t cnt_index(const Tile& x, D d) const { return (x.r * kRadix + d) * tpr + x.t; }
    __device__ __forceinline__ uint64_t chunks() const { return num_rows * cpr; }
    __device__ __forceinline__ Chunk chunk(uint64_t g) const
    {
        const uint64_t r = g / cpr, c0 = (g - r * cpr) * kLongChunk;
        return {r * row_counts, c0, row_counts};
    }
    __device__ __forceinline__ uint64_t groups() const { return num_rows; }
    __device__ __forceinline__ Group group(uint64_t r) const { return {r * cpr, cpr}; }
};

// The largest j < m with pre[j] <= g, for pre increasing from pre[0] = 0.  All threads of the CTA call it; each round reads
// kLongThreads entries at once and narrows the range as many times, so a list of up to 2^18 entries takes two rounds.
__device__ __forceinline__ uint32_t cta_find(const uint32_t* __restrict__ pre, uint32_t m, uint64_t g)
{
    uint32_t lo = 0, hi = m;
    while (hi - lo > 1) {
        const uint32_t step = (hi - lo + kLongThreads - 1) / kLongThreads, i = lo + threadIdx.x * step;
        lo += step * static_cast<uint32_t>(__syncthreads_count(threadIdx.x > 0 && i < hi && pre[i] <= g));
        hi = lo + step < hi ? lo + step : hi;
    }
    return lo;
}

// The long segments: the tile map of long_segments_map_kernel.  list[j] is the j-th listed segment, tfirst[j] and cfirst[j]
// its first tile and first scan chunk (tfirst[m], cfirst[m]: the totals), counts[kSegCountLong...] the list's length and
// totals.  A tile's counts are digit-major within its segment, as within a row.
struct LongSegGeo {
    const unsigned long long* off;
    const uint32_t* list;
    const uint32_t* tfirst;
    const uint32_t* cfirst;
    const unsigned long long* counts;
    struct Tile { uint64_t cb, lo; uint32_t t, t0, len, tpr; uint64_t r; };  // r: the list entry (osb200_select_segments)
    struct Chunk { uint64_t base, c0, row_counts; };
    struct Group { uint64_t first; uint32_t count; };
    __device__ __forceinline__ uint32_t listed() const { return static_cast<uint32_t>(counts[kSegCountLong]); }
    __device__ __forceinline__ uint64_t tiles() const { return counts[kSegCountLongTiles]; }
    __device__ __forceinline__ Tile tile(uint64_t g) const
    {
        const uint32_t j = cta_find(tfirst, listed(), g), f = tfirst[j], s = list[j];
        const uint64_t lo = off[s];
        const uint32_t seg_len = static_cast<uint32_t>(off[s + 1] - lo);
        const uint32_t t = static_cast<uint32_t>(g - f), t0 = t * kLongRowTile;
        const uint32_t len = seg_len - t0 < kLongRowTile ? seg_len - t0 : kLongRowTile;
        return {static_cast<uint64_t>(f) * kRadix, lo, t, t0, len, tfirst[j + 1] - f, j};
    }
    template <typename D>
    __device__ __forceinline__ uint64_t cnt_index(const Tile& x, D d) const { return x.cb + static_cast<uint64_t>(d) * x.tpr + x.t; }
    __device__ __forceinline__ uint64_t chunks() const { return counts[kSegCountLongChunks]; }
    __device__ __forceinline__ Chunk chunk(uint64_t g) const
    {
        const uint32_t j = cta_find(cfirst, listed(), g), f = tfirst[j];
        return {static_cast<uint64_t>(f) * kRadix, (g - cfirst[j]) * kLongChunk, static_cast<uint64_t>(tfirst[j + 1] - f) * kRadix};
    }
    __device__ __forceinline__ uint64_t groups() const { return listed(); }
    __device__ __forceinline__ Group group(uint64_t j) const { return {cfirst[j], cfirst[j + 1] - cfirst[j]}; }
};

template <typename KeyT, typename Geo>
__device__ __forceinline__ void long_count_body(const Geo& geo, const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in,
                                                const KeyT* keys_out, const KeyT* alt, uint32_t* __restrict__ cnt, KeyCodec codec)
{
    const LongPass ps = long_pass(plan, place);
    if (ps.skip) return;
    const KeyT* src = ps.first ? keys_in : ps.from_alt ? alt : keys_out;
    const bool enc = ps.first && (codec.flags & kCodecEncodeOnLoad);
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const uint32_t shift = 8u * place;
    // bank-private columns, as in the GlobalHistogram: every lane of a warp instruction hits its own bank
    __shared__ uint32_t s_hist[kRadix * 32];
    uint32_t* s_col = s_hist + (threadIdx.x & 31);
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        const uint32_t len = x.len;
        const KeyT* tile = src + x.lo + x.t0;
        for (int i = threadIdx.x; i < kRadix * 32; i += kLongThreads) s_hist[i] = 0;
        __syncthreads();
        KeyT key[kLongK];
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            const uint32_t j = threadIdx.x + i * kLongThreads;
            key[i] = j < len ? tile[j] : static_cast<KeyT>(0);
        }
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            if (threadIdx.x + i * kLongThreads >= len) break;
            const KeyT k = enc ? codec_encode<KeyT>(key[i], ca, cb, cd) : key[i];
            atomicAdd(&s_col[digit_of(k, shift) * 32], 1u);
        }
        __syncthreads();
        if (threadIdx.x < kRadix) {
            uint32_t sum = 0;
#pragma unroll 8
            for (int c = 0; c < 32; ++c) sum += s_hist[threadIdx.x * 32 + ((c + threadIdx.x) & 31)];
            cnt[geo.cnt_index(x, threadIdx.x)] = sum;
        }
        __syncthreads();  // the fold has read s_hist
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
long_rows_count_kernel(const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in, const KeyT* keys_out, const KeyT* alt,
                       uint64_t num_rows, uint32_t row_len, uint32_t tpr, uint32_t* __restrict__ cnt, KeyCodec codec)
{
    long_count_body<KeyT>(LongRowGeo{num_rows, row_len, tpr, 0, 0}, plan, place, keys_in, keys_out, alt, cnt, codec);
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
long_segments_count_kernel(const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in, const KeyT* keys_out, const KeyT* alt,
                           LongSegGeo geo, uint32_t* __restrict__ cnt, KeyCodec codec)
{
    long_count_body<KeyT>(geo, plan, place, keys_in, keys_out, alt, cnt, codec);
}

// The m <= kLongChunk counts at p, thread i holding counts 8i .. 8i+7: their sum (to every thread), and with SCAN their
// exclusive prefix plus carry written back in place.  All kLongThreads threads call it.
template <bool SCAN>
__device__ __forceinline__ uint32_t long_chunk(uint32_t* p, uint32_t m, uint32_t carry, uint32_t* s_w /*[kLongWarps]*/)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t b = static_cast<uint32_t>(tid) * kLongScanPer;
    uint32_t v[kLongScanPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kLongScanPer; ++j) { v[j] = b + j < m ? p[b + j] : 0u; sum += v[j]; }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t pre = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kLongWarps; ++w) { const uint32_t x = s_w[w]; pre += w < warp ? x : 0u; total += x; }
    __syncthreads();  // s_w is reused by the next chunk
    if constexpr (SCAN) {
        uint32_t run = carry + pre + incl - sum;
#pragma unroll
        for (int j = 0; j < kLongScanPer; ++j) {
            if (b + j < m) p[b + j] = run;
            run += v[j];
        }
    }
    return total;
}

// Chunk g covers counts [c0, min(c0 + kLongChunk, row_counts)) of its row's or segment's row_counts = 256 * tiles:
// csum[g] = their sum.
template <typename Geo>
__device__ __forceinline__ void long_chunk_sum_body(const Geo& geo, const SortPlan* __restrict__ plan, uint32_t place, uint32_t* cnt,
                                                    uint32_t* __restrict__ csum)
{
    if (long_pass(plan, place).skip) return;
    __shared__ uint32_t s_w[kLongWarps];
    for (uint64_t g = blockIdx.x; g < geo.chunks(); g += gridDim.x) {
        const auto x = geo.chunk(g);
        const uint32_t m = static_cast<uint32_t>(x.row_counts - x.c0 < kLongChunk ? x.row_counts - x.c0 : kLongChunk);
        const uint32_t s = long_chunk<false>(cnt + x.base + x.c0, m, 0u, s_w);
        if (threadIdx.x == 0) csum[g] = s;
    }
}

__global__ void __launch_bounds__(kLongThreads)
long_rows_chunk_sum_kernel(const SortPlan* __restrict__ plan, uint32_t place, uint32_t* cnt, uint32_t* __restrict__ csum,
                           uint64_t num_rows, uint64_t row_counts, uint32_t cpr)
{
    long_chunk_sum_body(LongRowGeo{num_rows, 0, 0, row_counts, cpr}, plan, place, cnt, csum);
}

__global__ void __launch_bounds__(kLongThreads)
long_segments_chunk_sum_kernel(const SortPlan* __restrict__ plan, uint32_t place, uint32_t* cnt, uint32_t* __restrict__ csum, LongSegGeo geo)
{
    long_chunk_sum_body(geo, plan, place, cnt, csum);
}

// The exclusive scan of each row's or segment's chunk sums, in place; one CTA per row or segment at a time.
template <typename Geo>
__device__ __forceinline__ void long_chunk_scan_body(const Geo& geo, const SortPlan* __restrict__ plan, uint32_t place, uint32_t* csum)
{
    if (long_pass(plan, place).skip) return;
    __shared__ uint32_t s_w[kLongWarps];
    for (uint64_t r = blockIdx.x; r < geo.groups(); r += gridDim.x) {
        const auto x = geo.group(r);
        uint32_t carry = 0;
        for (uint32_t c0 = 0; c0 < x.count; c0 += kLongChunk)
            carry += long_chunk<true>(csum + x.first + c0, x.count - c0 < kLongChunk ? x.count - c0 : kLongChunk, carry, s_w);
    }
}

__global__ void __launch_bounds__(kLongThreads)
long_rows_chunk_scan_kernel(const SortPlan* __restrict__ plan, uint32_t place, uint32_t* csum, uint64_t num_rows, uint32_t cpr)
{
    long_chunk_scan_body(LongRowGeo{num_rows, 0, 0, 0, cpr}, plan, place, csum);
}

__global__ void __launch_bounds__(kLongThreads)
long_segments_chunk_scan_kernel(const SortPlan* __restrict__ plan, uint32_t place, uint32_t* csum, LongSegGeo geo)
{
    long_chunk_scan_body(geo, plan, place, csum);
}

// Every chunk's counts become their exclusive prefix within the row or segment: the chunk's own scan plus its chunk prefix
// (csum null: every row or segment is one chunk).
template <typename Geo>
__device__ __forceinline__ void long_scan_body(const Geo& geo, const SortPlan* __restrict__ plan, uint32_t place, uint32_t* cnt,
                                               const uint32_t* __restrict__ csum)
{
    if (long_pass(plan, place).skip) return;
    __shared__ uint32_t s_w[kLongWarps];
    for (uint64_t g = blockIdx.x; g < geo.chunks(); g += gridDim.x) {
        const auto x = geo.chunk(g);
        const uint32_t m = static_cast<uint32_t>(x.row_counts - x.c0 < kLongChunk ? x.row_counts - x.c0 : kLongChunk);
        long_chunk<true>(cnt + x.base + x.c0, m, csum ? csum[g] : 0u, s_w);
    }
}

__global__ void __launch_bounds__(kLongThreads)
long_rows_scan_kernel(const SortPlan* __restrict__ plan, uint32_t place, uint32_t* cnt, const uint32_t* __restrict__ csum,
                      uint64_t num_rows, uint64_t row_counts, uint32_t cpr)
{
    long_scan_body(LongRowGeo{num_rows, 0, 0, row_counts, cpr}, plan, place, cnt, csum);
}

__global__ void __launch_bounds__(kLongThreads)
long_segments_scan_kernel(const SortPlan* __restrict__ plan, uint32_t place, uint32_t* cnt, const uint32_t* __restrict__ csum,
                          LongSegGeo geo)
{
    long_scan_body(geo, plan, place, cnt, csum);
}

template <typename KeyT, bool INDICES>
struct LongRowsSmem {
    alignas(16) KeyT sorted[kLongRowTile];
    alignas(16) uint32_t sorted_idx[INDICES ? kLongRowTile : 4];
    alignas(16) uint32_t hist[kLongWarps * kRadix];
    uint32_t first[kRadix];  // the tile's first slot of every digit
    uint32_t base[kRadix];   // the row-relative output position of the tile's first key of every digit
    uint32_t wtot[kRadix / 32];
};

// GIVEN (topk_long_sort_scatter_kernel): the first executed pass loads the indices given in idx_out instead of making them.
template <typename KeyT, int RANK_MODE, bool INDICES, typename Geo, bool GIVEN = false>
__device__ __forceinline__ void long_scatter_body(const Geo& geo, const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in,
                                                  KeyT* keys_out, KeyT* alt, uint32_t* idx_out, uint32_t* alt_idx,
                                                  const uint32_t* __restrict__ base, KeyCodec codec)
{
    const LongPass ps = long_pass(plan, place);
    if (ps.skip) return;
    const KeyT* src = ps.first ? keys_in : ps.from_alt ? alt : keys_out;
    KeyT* dst = ps.from_alt ? keys_out : alt;
    const uint32_t* src_idx = ps.from_alt ? alt_idx : idx_out;
    uint32_t* dst_idx = ps.from_alt ? idx_out : alt_idx;
    const bool enc = ps.first && (codec.flags & kCodecEncodeOnLoad), dec = ps.last && (codec.flags & kCodecDecodeOnStore);
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const uint32_t shift = 8u * place;

    using S = LongRowsSmem<KeyT, INDICES>;
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    uint32_t* wh = sm.hist + warp * kRadix;
    const uint32_t warp_lo = warp * (32 * kLongK), warp_off = warp_lo + lane;
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        const uint64_t row_lo = x.lo;
        const uint32_t t0 = x.t0, len = x.len;
        __syncthreads();  // the previous tile has been stored from shared memory
        {
            uint4* h4 = reinterpret_cast<uint4*>(sm.hist);
            for (int i = tid; i < kLongWarps * kRadix / 4; i += kLongThreads) h4[i] = make_uint4(0, 0, 0, 0);
        }
        // tile order: key i of a lane is warp_lo + 32 i + lane; the padding (all ones) ranks after every real key
        KeyT key[kLongK];
        uint32_t val[INDICES ? kLongK : 1];
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            const uint32_t j = warp_off + i * 32;
            KeyT k = j < len ? src[row_lo + t0 + j] : static_cast<KeyT>(0);
            if (enc) k = codec_encode<KeyT>(k, ca, cb, cd);
            key[i] = j < len ? k : static_cast<KeyT>(~static_cast<KeyT>(0));
            if constexpr (INDICES) val[i] = ps.first && !GIVEN ? t0 + j : j < len ? src_idx[row_lo + t0 + j] : 0u;
        }
        // a warp's chunks of 32 keys that lie wholly behind the tile are neither counted nor ranked (as in segment_sort_body)
        const uint32_t live_chunks = len > warp_lo ? (len - warp_lo + 31) / 32 : 0u;
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kLongK; ++i)
            if (static_cast<uint32_t>(i) < live_chunks) atomicAdd(&wh[digit_of(key[i], shift)], 1u);
        __syncthreads();
        uint32_t tile_count = 0;
        if (tid < kRadix) {
#pragma unroll
            for (int w = 0; w < kLongWarps; ++w) tile_count += sm.hist[w * kRadix + tid];
        }
        const uint32_t tile_excl = block_excl_scan_256<kLongThreads>(tile_count, sm.wtot);
        if (tid < kRadix) {
            uint32_t run = tile_excl;
#pragma unroll
            for (int w = 0; w < kLongWarps; ++w) { const uint32_t c = sm.hist[w * kRadix + tid]; sm.hist[w * kRadix + tid] = run; run += c; }
            sm.first[tid] = tile_excl;
            sm.base[tid] = base[geo.cnt_index(x, tid)];
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            if (static_cast<uint32_t>(i) >= live_chunks) continue;
            const uint32_t slot = warp_rank_and_count<RANK_MODE>(wh, digit_of(key[i], shift), lt);
            sm.sorted[slot] = key[i];
            if constexpr (INDICES) sm.sorted_idx[slot] = val[i];
        }
        __syncthreads();
        for (uint32_t j = tid; j < len; j += kLongThreads) {
            KeyT k = sm.sorted[j];
            const uint32_t d = digit_of(k, shift);
            const uint64_t o = row_lo + (sm.base[d] + (j - sm.first[d]));
            if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
            st_scatter(dst + o, k);
            if constexpr (INDICES) st_scatter(dst_idx + o, sm.sorted_idx[j]);
        }
    }
}

// (Two resident CTAs per SM are stated for 16- and 32-bit keys only: with indices they spill at 64 registers.)
template <typename KeyT, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(kLongThreads, sizeof(KeyT) == 8 || INDICES ? 1 : 2)
long_rows_scatter_kernel(const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in, KeyT* keys_out, KeyT* alt,
                         uint32_t* idx_out, uint32_t* alt_idx, uint64_t num_rows, uint32_t row_len, uint32_t tpr,
                         const uint32_t* __restrict__ base, KeyCodec codec)
{
    long_scatter_body<KeyT, RANK_MODE, INDICES>(LongRowGeo{num_rows, row_len, tpr, 0, 0}, plan, place, keys_in, keys_out, alt, idx_out,
                                                alt_idx, base, codec);
}

template <typename KeyT, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(kLongThreads, sizeof(KeyT) == 8 || INDICES ? 1 : 2)
long_segments_scatter_kernel(const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in, KeyT* keys_out, KeyT* alt,
                             uint32_t* idx_out, uint32_t* alt_idx, LongSegGeo geo, const uint32_t* __restrict__ base, KeyCodec codec)
{
    long_scatter_body<KeyT, RANK_MODE, INDICES>(geo, plan, place, keys_in, keys_out, alt, idx_out, alt_idx, base, codec);
}

// Odd executed passes: keys and indices from the alternate buffers.  None: keys_in is its own stable sort -- its keys (not
// copied in place) and the positions 0 .. row_len - 1 of every row.
template <typename KeyT>
__global__ void __launch_bounds__(512)
long_rows_copy_home_kernel(const SortPlan* __restrict__ plan, const KeyT* keys_in, const KeyT* __restrict__ alt, KeyT* keys_out,
                           const uint32_t* __restrict__ alt_idx, uint32_t* __restrict__ idx_out, uint64_t n, uint32_t row_len)
{
    const uint32_t ex = plan->executed;
    if (ex != 0 && !(ex & 1u)) return;
    const KeyT* src = ex ? alt : keys_in;
    const bool keys = src != keys_out;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (keys) __stcs(keys_out + i, __ldcs(src + i));
        if (idx_out) __stcs(idx_out + i, ex ? __ldcs(alt_idx + i) : static_cast<uint32_t>(i % row_len));
    }
}


// osb200_topk_long_rows' sort of k > C selected keys per row, in place: the long rows' passes with the positions as payloads
template <typename KeyT, int RANK_MODE>
__global__ void __launch_bounds__(kLongThreads, 1)
topk_long_sort_scatter_kernel(const SortPlan* __restrict__ plan, uint32_t place, const KeyT* keys_in, KeyT* keys_out, KeyT* alt,
                              uint32_t* idx_out, uint32_t* alt_idx, uint64_t num_rows, uint32_t row_len, uint32_t tpr,
                              const uint32_t* __restrict__ base, KeyCodec codec)
{
    long_scatter_body<KeyT, RANK_MODE, true, LongRowGeo, true>(LongRowGeo{num_rows, row_len, tpr, 0, 0}, plan, place, keys_in, keys_out, alt,
                                                               idx_out, alt_idx, base, codec);
}

// Its copy home: an odd number of executed passes moves keys and indices from the alternate buffers; after none the sort was
// in place already, and the given indices stay.
template <typename KeyT>
__global__ void __launch_bounds__(512)
topk_long_sort_copy_home_kernel(const SortPlan* __restrict__ plan, const KeyT* __restrict__ alt, KeyT* __restrict__ keys,
                                const uint32_t* __restrict__ alt_idx, uint32_t* __restrict__ idx, uint64_t n)
{
    if (!(plan->executed & 1u)) return;
    const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        __stcs(keys + i, __ldcs(alt + i));
        __stcs(idx + i, __ldcs(alt_idx + i));
    }
}

// The long segments' copy home, tile by tile so that nothing outside them is written: as long_rows_copy_home_kernel, with
// positions 0 .. L - 1 within each segment when no pass executes.
template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
long_segments_copy_home_kernel(const SortPlan* __restrict__ plan, const KeyT* keys_in, const KeyT* __restrict__ alt, KeyT* keys_out,
                               const uint32_t* __restrict__ alt_idx, uint32_t* __restrict__ idx_out, LongSegGeo geo)
{
    const uint32_t ex = plan->executed;
    if (ex != 0 && !(ex & 1u)) return;
    const KeyT* src = ex ? alt : keys_in;
    const bool keys = src != keys_out;
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        for (uint32_t j = threadIdx.x; j < x.len; j += kLongThreads) {
            const uint64_t i = x.lo + x.t0 + j;
            if (keys) __stcs(keys_out + i, __ldcs(src + i));
            if (idx_out) __stcs(idx_out + i, ex ? __ldcs(alt_idx + i) : x.t0 + j);
        }
    }
}

// The tile map of the long list, one CTA: the tiles ceil(L / kLongRowTile) and scan chunks ceil(256 tiles / kLongChunk) of
// every listed segment become exclusive prefixes in list order (tfirst, cfirst), with the totals at [m] and in counts.
// Listed segments are disjoint unless the offsets make valid segments overlap; only then can the list or its totals pass
// the workspace's bounds, and the long path is left empty.
__global__ void __launch_bounds__(kLongThreads)
long_segments_map_kernel(const unsigned long long* __restrict__ off, const uint32_t* __restrict__ list, uint32_t* tfirst,
                         uint32_t* cfirst, unsigned long long* counts, uint64_t list_cap, uint64_t tile_cap, uint64_t chunk_cap)
{
    __shared__ uint32_t s_w[kLongWarps];
    __shared__ unsigned long long s_tiles, s_chunks;
    const unsigned long long listed = counts[kSegCountLong];
    const uint32_t m = static_cast<uint32_t>(listed < list_cap ? listed : list_cap);
    if (threadIdx.x == 0) s_tiles = s_chunks = 0;
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < m; j += kLongThreads) {
        const uint32_t s = list[j];
        const unsigned long long tiles = (off[s + 1] - off[s] + kLongRowTile - 1) / kLongRowTile;
        const unsigned long long chunks = (tiles * kRadix + kLongChunk - 1) / kLongChunk;
        tfirst[j] = static_cast<uint32_t>(tiles);
        cfirst[j] = static_cast<uint32_t>(chunks);
        atomicAdd(&s_tiles, tiles);
        atomicAdd(&s_chunks, chunks);
    }
    __syncthreads();
    const bool fits = listed <= list_cap && s_tiles <= tile_cap && s_chunks <= chunk_cap;
    uint32_t tc = 0, cc = 0;
    for (uint32_t c0 = 0; fits && c0 < m; c0 += kLongChunk) {
        const uint32_t k = m - c0 < kLongChunk ? m - c0 : kLongChunk;
        tc += long_chunk<true>(tfirst + c0, k, tc, s_w);
        cc += long_chunk<true>(cfirst + c0, k, cc, s_w);
    }
    if (threadIdx.x == 0) {
        if (fits) { tfirst[m] = tc; cfirst[m] = cc; }
        counts[kSegCountLong] = fits ? m : 0u;
        counts[kSegCountLongTiles] = tc;
        counts[kSegCountLongChunks] = cc;
    }
}

using LongRowKeys = TypeList<uint16_t, uint32_t, uint64_t>;

// The long paths' plan over keys[0, n): the keys before the first 16-byte boundary of a naturally aligned input (at most
// 7, and never more than n) by the one-warp head kernel, the rest by the GlobalHistogram, which reads 16-byte vectors;
// then the scan that writes `plan`.  enc: the codec's encode only (null: plain unsigned keys).
template <typename KeyT>
static cudaError_t launch_long_plan(const KeyT* in, uint64_t n, int key_bytes, const KeyCodec* enc, bool allow_skip,
                                   unsigned long long* ghist, unsigned long long* gbase, SortPlan* plan, int sm_count,
                                   cudaStream_t stream)
{
    uint64_t head = ((16u - (reinterpret_cast<uintptr_t>(in) & 15u)) & 15u) / sizeof(KeyT);
    if (head > n) head = n;
    if (head) long_rows_head_hist_kernel<KeyT><<<1, 32, 0, stream>>>(in, static_cast<uint32_t>(head), ghist, enc ? *enc : KeyCodec());
    cudaError_t e = launch_global_histogram(in + head, n - head, key_bytes, ghist, sm_count, stream, enc);
    return e == cudaSuccess ? launch_scan(ghist, gbase, key_bytes, stream, plan, n, allow_skip, false) : e;
}


cudaError_t launch_long_rows(const void* keys_in, void* keys_out, uint32_t* indices, void* alt_keys, uint32_t* alt_idx,
                             uint64_t num_rows, uint32_t row_len, int key_bytes, const KeyCodec* codec_in, int rank_mode,
                             bool allow_skip, unsigned long long* ghist, unsigned long long* gbase, SortPlan* plan,
                             uint32_t* scratch, int sm_count, cudaStream_t stream, bool given_indices)
{
    if (num_rows == 0 || row_len < 2 || (given_indices && !indices)) return cudaErrorInvalidValue;
    const uint64_t n = num_rows * row_len;
    const uint32_t tpr = (row_len + kLongRowTile - 1) / kLongRowTile;
    const uint64_t row_counts = static_cast<uint64_t>(tpr) * kRadix;
    const uint32_t cpr = static_cast<uint32_t>((row_counts + kLongChunk - 1) / kLongChunk);
    uint32_t* cnt = scratch;
    uint32_t* csum = cpr > 1 ? scratch + (num_rows * row_counts + 3) / 4 * 4 : nullptr;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    KeyCodec enc = codec;
    enc.flags &= kCodecEncodeOnLoad;
    return with_key_type(LongRowKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        KeyT* out = static_cast<KeyT*>(keys_out);
        KeyT* alt = static_cast<KeyT*>(alt_keys);
        cudaError_t e = launch_long_plan(in, n, key_bytes, codec_in ? &enc : nullptr, allow_skip, ghist, gbase, plan, sm_count, stream);
        const unsigned scan_grid = capped_grid(num_rows * cpr, 1, static_cast<uint64_t>(sm_count) * 4);
        for (uint32_t p = 0; e == cudaSuccess && p < sizeof(KeyT); ++p) {
            e = launch_resident<long_rows_count_kernel<KeyT>, kLongThreads, 0>(num_rows * tpr, sm_count, stream, plan, p, in, out, alt,
                                                                               num_rows, row_len, tpr, cnt, codec);
            if (e == cudaSuccess && csum) {
                long_rows_chunk_sum_kernel<<<scan_grid, kLongThreads, 0, stream>>>(plan, p, cnt, csum, num_rows, row_counts, cpr);
                long_rows_chunk_scan_kernel<<<capped_grid(num_rows, 1, static_cast<uint64_t>(sm_count) * 4), kLongThreads, 0, stream>>>(
                    plan, p, csum, num_rows, cpr);
            }
            if (e == cudaSuccess) {
                long_rows_scan_kernel<<<scan_grid, kLongThreads, 0, stream>>>(plan, p, cnt, csum, num_rows, row_counts, cpr);
                e = cudaGetLastError();
            }
            if (e == cudaSuccess) e = with_rank_mode(rank_mode, [&](auto rm) {
                auto go = [&](auto ind) {
                    constexpr bool I = decltype(ind)::value;
                    return launch_resident<long_rows_scatter_kernel<KeyT, decltype(rm)::value, I>, kLongThreads, sizeof(LongRowsSmem<KeyT, I>)>(
                        num_rows * tpr, sm_count, stream, plan, p, in, out, alt, indices, alt_idx, num_rows, row_len, tpr,
                        static_cast<const uint32_t*>(cnt), codec);
                };
                if (given_indices)
                    return launch_resident<topk_long_sort_scatter_kernel<KeyT, decltype(rm)::value>, kLongThreads, sizeof(LongRowsSmem<KeyT, true>)>(
                        num_rows * tpr, sm_count, stream, plan, p, in, out, alt, indices, alt_idx, num_rows, row_len, tpr,
                        static_cast<const uint32_t*>(cnt), codec);
                return indices ? go(std::true_type{}) : go(std::false_type{});
            });
        }
        if (e != cudaSuccess) return e;
        const unsigned home_grid = capped_grid(n, 512, static_cast<uint64_t>(sm_count) * 4);
        if (given_indices)
            topk_long_sort_copy_home_kernel<KeyT><<<home_grid, 512, 0, stream>>>(plan, alt, out, alt_idx, indices, n);
        else
            long_rows_copy_home_kernel<KeyT><<<home_grid, 512, 0, stream>>>(plan, in, alt, out, alt_idx, indices, n, row_len);
        return cudaGetLastError();
    });
}

// =====================================================================================================
// Long segments (osb200_sort_long_segments): the segment sort's binning and classes for segments of up to long_min - 1 keys,
// and the long-row passes over the tiles of the longer ones (DESIGN §4.17).  The tiles of segment j of the long list are
// tfirst[j] .. tfirst[j + 1] - 1 and its counts start at 256 * tfirst[j]; each kernel finds a tile's or chunk's segment
// by a search over the prefixes (LongSegGeo).  The list's order comes from atomics; it moves where a segment's counts are,
// never where its keys go.
// =====================================================================================================
template <typename KeyT>
__global__ void __launch_bounds__(256)
long_segment_bin_kernel(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n, uint32_t max_len,
                        uint32_t* __restrict__ list, unsigned long long* __restrict__ counts, const KeyT* keys_in, KeyT* keys_out,
                        uint32_t* idx_out, uint32_t long_min, uint32_t* __restrict__ long_list, uint64_t long_cap)
{
    segment_bin_body<KeyT, false, true>(off, num_segments, n, max_len, list, counts, keys_in, keys_out, idx_out, kRowWarpMaxLen,
                                        long_min, long_list, long_cap);
}

LongSegLayout long_segments_layout(uint64_t n, uint32_t long_min)
{
    auto whole = [](uint64_t words) { return (words + 3) / 4 * 4; };  // every array 16-byte aligned
    LongSegLayout l;
    l.list_cap = n / long_min;
    l.tile_cap = (n + kLongRowTile - 1) / kLongRowTile + l.list_cap;
    l.chunk_cap = (l.tile_cap * kRadix + kLongChunk - 1) / kLongChunk + l.list_cap;
    l.csum = whole(l.tile_cap * kRadix);
    l.list = l.csum + whole(l.chunk_cap);
    l.tfirst = l.list + whole(l.list_cap);
    l.cfirst = l.tfirst + whole(l.list_cap + 1);
    l.words = l.cfirst + whole(l.list_cap + 1);
    return l;
}

cudaError_t launch_long_segments(const void* keys_in, void* keys_out, uint32_t* indices, void* alt_keys, uint32_t* alt_idx, uint64_t n,
                                 const unsigned long long* off, uint64_t num_segments, uint32_t max_len, uint32_t long_min,
                                 int key_bytes, const KeyCodec* codec_in, int rank_mode, bool allow_skip, unsigned long long* ghist,
                                 unsigned long long* gbase, SortPlan* plan, uint32_t* list, unsigned long long* counts,
                                 uint32_t* scratch, int sm_count, cudaStream_t stream)
{
    if (num_segments == 0 || max_len < long_min || long_min < 2) return cudaErrorInvalidValue;
    const LongSegLayout l = long_segments_layout(n, long_min);
    uint32_t* cnt = scratch;
    uint32_t* csum = max_len > kLongChunk / kRadix * kLongRowTile ? scratch + l.csum : nullptr;  // some segment has 2+ chunks
    uint32_t* llist = scratch + l.list;
    const LongSegGeo geo{off, llist, scratch + l.tfirst, scratch + l.cfirst, counts};
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    KeyCodec enc = codec;
    enc.flags &= kCodecEncodeOnLoad;
    cudaError_t e = cudaMemsetAsync(counts, 0, kLongSegCounts * sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    return with_key_type(LongRowKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        KeyT* out = static_cast<KeyT*>(keys_out);
        KeyT* alt = static_cast<KeyT*>(alt_keys);
        long_segment_bin_kernel<KeyT><<<capped_grid(num_segments, 256, static_cast<uint64_t>(sm_count) * 8), 256, 0, stream>>>(
            off, num_segments, n, max_len, list, counts, in, out, indices, long_min, llist, l.list_cap);
        cudaError_t e = cudaGetLastError();
        // the classes first: their lists live in the alternate keys, which the long passes overwrite
        if (e == cudaSuccess && long_min > 2)
            e = launch_segment_classes(keys_in, keys_out, indices, off, num_segments, long_min - 1, key_bytes, codec, rank_mode, sm_count,
                                       list, counts, stream);
        if (e == cudaSuccess) {
            long_segments_map_kernel<<<1, kLongThreads, 0, stream>>>(off, llist, scratch + l.tfirst, scratch + l.cfirst, counts, l.list_cap,
                                                                     l.tile_cap, l.chunk_cap);
            e = cudaGetLastError();
        }
        // the plan over all n keys, as for the long rows
        if (e == cudaSuccess)
            e = launch_long_plan(in, n, key_bytes, codec_in ? &enc : nullptr, allow_skip, ghist, gbase, plan, sm_count, stream);
        const unsigned scan_grid = capped_grid(l.chunk_cap, 1, static_cast<uint64_t>(sm_count) * 4);
        for (uint32_t p = 0; e == cudaSuccess && p < sizeof(KeyT); ++p) {
            e = launch_resident<long_segments_count_kernel<KeyT>, kLongThreads, 0>(l.tile_cap, sm_count, stream, plan, p, in,
                                                                                   static_cast<const KeyT*>(out), static_cast<const KeyT*>(alt),
                                                                                   geo, cnt, codec);
            if (e == cudaSuccess && csum) {
                long_segments_chunk_sum_kernel<<<scan_grid, kLongThreads, 0, stream>>>(plan, p, cnt, csum, geo);
                long_segments_chunk_scan_kernel<<<capped_grid(l.list_cap, 1, static_cast<uint64_t>(sm_count) * 4), kLongThreads, 0, stream>>>(
                    plan, p, csum, geo);
            }
            if (e == cudaSuccess) {
                long_segments_scan_kernel<<<scan_grid, kLongThreads, 0, stream>>>(plan, p, cnt, csum, geo);
                e = cudaGetLastError();
            }
            if (e == cudaSuccess) e = with_rank_mode(rank_mode, [&](auto rm) {
                auto go = [&](auto ind) {
                    constexpr bool I = decltype(ind)::value;
                    return launch_resident<long_segments_scatter_kernel<KeyT, decltype(rm)::value, I>, kLongThreads, sizeof(LongRowsSmem<KeyT, I>)>(
                        l.tile_cap, sm_count, stream, plan, p, in, out, alt, indices, alt_idx, geo, static_cast<const uint32_t*>(cnt), codec);
                };
                return indices ? go(std::true_type{}) : go(std::false_type{});
            });
        }
        if (e != cudaSuccess) return e;
        return launch_resident<long_segments_copy_home_kernel<KeyT>, kLongThreads, 0>(l.tile_cap, sm_count, stream, plan, in,
                                                                                      static_cast<const KeyT*>(alt), out,
                                                                                      static_cast<const uint32_t*>(alt_idx), indices, geo);
    });
}

// =====================================================================================================
// Row top-k (osb200_topk_rows): the first k keys of every row in the stable row sort, with their positions.
//
// Rows of at most kRowWarpMaxLen keys: one warp sorts the row (warp_sort_run, TOPK) and stores its first k keys.
// Longer rows: one CTA per row (grid-stride over the rows on the resident CTAs) runs a radix select from the most significant
// digit over the encoded keys.  Pass t (t = 0 .. D, D digit places) reads the candidates S_t -- the keys whose t top digits
// are the prefix V_t chosen so far -- and
//   * selects the keys of S_{t-1} whose t top digits are below V_t (the buckets below the one chosen at level t - 1);
//   * counts digit t of S_t in per-warp bins; the scan picks the bucket b holding the k'-th candidate (k' = the keys still
//     needed), k' drops by the keys below b and b is appended to V.
// When b holds exactly k' keys, or after the last digit, the next pass is the final one: it also selects the keys equal to
// the prefix, the first k' of them in position order.  Every selection is an ordered compaction (per-warp ballots, a scan
// of the chunk's warp counts) in row order, so equal keys -- always selected in the same pass -- reach the output in position
// order, and the ties at the boundary are the lowest positions.
// The candidates are read from the row in global memory until their count fits `cap` (row_sort_capacity keys, or less as a
// test hook): the pass that reads S_t then also compacts it, in row order, into shared memory, and later passes read only
// that.  So a row of at most cap keys is read once, and a row is never read more than D + 1 times.
// The selected keys leave in pass order, not key order; `sorted` sorts the [num_rows, k] output in place afterwards
// (topk_warp_kernel for k <= 256, else topk_sort_kernel: the row sort's block body with the payloads loaded).
// =====================================================================================================
constexpr int kTopkWarps = 16, kTopkThreads = kTopkWarps * 32;
constexpr int kTopkE = 8;  // keys per thread and chunk: a chunk is 4,096 keys, one block barrier

// osb200_topk_long_rows' state of one row on the split path: the digits chosen so far, v under the mask m (encoded keys); the
// keys selected so far, taken (those with (x & m) < v); the candidates, cand ((x & m) == v); the last chosen digit b.  All
// zero is a row at level 0.
constexpr uint32_t kTopkLongActive = 0, kTopkLongResolved = 1, kTopkLongStopped = 2;
struct TopkLongRow { unsigned long long v, m; uint32_t taken, cand, b, status; };

template <typename KeyT>
struct TopkSmem {
    static constexpr uint32_t C = SegGeomN<KeyT, 2>::K * SegGeomN<KeyT, 2>::WARPS * 32;  // row_sort_capacity
    alignas(16) KeyT keys[C];
    alignas(16) uint32_t pos[C];
    alignas(16) uint32_t hist[kTopkWarps * kRadix];
    uint32_t cnt[2][kTopkE * kTopkWarps];  // per chunk (double-buffered): selected | candidates << 16 of each (e, warp)
    uint32_t wtot[kRadix / 32];
    uint32_t pick[3];  // the chosen bucket, the candidates below it, the candidates in it
};

// LIST (osb200_topk_segments, topk_segment_select_kernel): the rows are the segments whose ids the binning kernel put at the
// back of `list` (entry i at list[num_rows - 1 - i], counts[kSegCountBlockList] of them), row s = [off[s], off[s + 1]) of
// `in`, with k' = m = min(length, k) and its result at row s * k; columns m .. k - 1 are padding (the decoded all-ones key,
// position 0xFFFFFFFF).  A segment of at most k keys starts with `last` set: one ordered pass selects all of it.
// FIN (osb200_topk_long_rows' finisher, topk_long_finish_kernel): only the rows the split path stopped (TopkLongRow) are
// selected.  Row r's candidates are `in` + r * row_len (encoded keys, row order) and pos + r * row_len (their positions);
// they are the row's first cand keys, of which the row still needs k - taken, written from column taken.
template <typename KeyT, bool LIST, bool FIN = false>
__device__ __forceinline__ void topk_select_body(const KeyT* __restrict__ in, KeyT* __restrict__ out, uint32_t* __restrict__ idx_out,
                                                 uint64_t num_rows, uint32_t row_len, uint32_t k, uint32_t cap, const KeyCodec& codec,
                                                 const unsigned long long* __restrict__ off, const uint32_t* __restrict__ list,
                                                 const unsigned long long* __restrict__ counts,
                                                 const TopkLongRow* __restrict__ rows = nullptr, const uint32_t* __restrict__ pos = nullptr)
{
    using S = TopkSmem<KeyT>;
    using U = std::conditional_t<sizeof(KeyT) == 8, uint64_t, uint32_t>;
    constexpr uint32_t BITS = sizeof(KeyT) * 8, D = sizeof(KeyT);
    constexpr uint32_t CHUNK = kTopkE * kTopkThreads;
    extern __shared__ __align__(128) unsigned char s_raw[];
    S& sm = *reinterpret_cast<S*>(s_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    uint32_t* wh = sm.hist + warp * kRadix;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = !FIN && (codec.flags & kCodecEncodeOnLoad), dec = codec.flags & kCodecDecodeOnStore;

    const uint64_t work = LIST ? counts[kSegCountBlockList] : num_rows;
    if (LIST && work == 0) return;
    for (int i = tid; i < kTopkWarps * kRadix; i += kTopkThreads) sm.hist[i] = 0;
    __syncthreads();
    for (uint64_t it = blockIdx.x; it < work; it += gridDim.x) {
        const uint64_t row = LIST ? list[num_rows - 1 - it] : it;
        TopkLongRow fin{};
        if constexpr (FIN) {
            fin = rows[row];
            if (fin.status != kTopkLongStopped) continue;
        }
        const uint64_t lo = LIST ? off[row] : row * row_len;
        const uint32_t len = LIST ? static_cast<uint32_t>(off[row + 1] - lo) : FIN ? fin.cand : row_len;  // (LIST: binned as 257 .. 2^32 - 1)
        const KeyT* src = in + lo;
        KeyT* dst = out + row * k + (FIN ? fin.taken : 0u);
        uint32_t* dst_idx = idx_out + row * k + (FIN ? fin.taken : 0u);
        const uint32_t m = LIST ? min(len, k) : FIN ? k - fin.taken : k;
        // S_{t-1} = {x : (x & mprev) == vprev}; selected this pass: x in S_{t-1} with (x & mcur) < vcur; S_t: (x & mcur) == vcur
        U mprev = 0, vprev = 0, mcur = 0, vcur = 0;
        uint32_t need = m, cand = len, written = 0, in_smem = 0;  // in_smem: 0, or the number of candidates held there
        bool last = LIST && len <= k;
        for (uint32_t t = 0;; ++t) {
            const bool compact = !last && !in_smem && cand <= cap;
            const bool order = t > 0 || compact || (LIST && last);  // anything to place in row order this pass
            const uint32_t shift = last ? 0u : BITS - 8u * (t + 1);
            const uint64_t n_src = in_smem ? in_smem : len;
            uint32_t sel_run = 0, eq_run = 0, chunk = 0;
            for (uint64_t c0 = 0; c0 < n_src; c0 += CHUNK, ++chunk) {
                U x[kTopkE];
                uint32_t p[kTopkE];
                bool sel[kTopkE], eq[kTopkE];
#pragma unroll
                for (int e = 0; e < kTopkE; ++e) {
                    const uint64_t i = c0 + static_cast<uint32_t>(e * kTopkThreads + tid);
                    const bool valid = i < n_src;
                    KeyT v = 0;
                    if (valid) v = in_smem ? sm.keys[i] : src[i];
                    if (valid && !in_smem && enc) v = codec_encode<KeyT>(v, ca, cb, cd);
                    x[e] = static_cast<U>(v);
                    if constexpr (FIN) p[e] = valid ? (in_smem ? sm.pos[i] : pos[lo + i]) : 0u;
                    else p[e] = in_smem && valid ? sm.pos[i] : static_cast<uint32_t>(i);
                    sel[e] = valid && (x[e] & mprev) == vprev && (x[e] & mcur) < vcur;
                    eq[e] = valid && (x[e] & mcur) == vcur;
                    if (!last && eq[e]) atomicAdd(&wh[static_cast<uint32_t>(x[e] >> shift) & 0xffu], 1u);
                }
                if (!order) continue;
                uint32_t bsel[kTopkE], beq[kTopkE];
                uint32_t* cnt = sm.cnt[chunk & 1];
#pragma unroll
                for (int e = 0; e < kTopkE; ++e) {
                    bsel[e] = __ballot_sync(0xffffffffu, sel[e]);
                    beq[e] = __ballot_sync(0xffffffffu, eq[e]);
                    if (lane == 0) cnt[e * kTopkWarps + warp] = __popc(bsel[e]) | (__popc(beq[e]) << 16);
                }
                __syncthreads();
                // exclusive prefix of the (e, warp) counts in row order: lane l scans entries 4l .. 4l + 3
                const uint4 c4 = reinterpret_cast<const uint4*>(cnt)[lane];
                const uint32_t s4 = c4.x + c4.y + c4.z + c4.w;
                uint32_t incl = s4;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
                const uint32_t sub = warp & 3;
                const uint32_t mine = incl - s4 + (sub > 0 ? c4.x : 0u) + (sub > 1 ? c4.y : 0u) + (sub > 2 ? c4.z : 0u);
#pragma unroll
                for (int e = 0; e < kTopkE; ++e) {
                    const uint32_t pre = __shfl_sync(0xffffffffu, mine, 4 * e + (warp >> 2));
                    const uint32_t s_before = sel_run + (pre & 0xffffu) + __popc(bsel[e] & lt);
                    const uint32_t e_before = eq_run + (pre >> 16) + __popc(beq[e] & lt);
                    if (sel[e] || (last && eq[e] && e_before < need)) {
                        const uint32_t o = written + s_before + (last ? min(e_before, need) : 0u);
                        KeyT v = static_cast<KeyT>(x[e]);
                        if (dec) v = codec_decode<KeyT>(v, ca, cb, cd);
                        dst[o] = v;
                        dst_idx[o] = p[e];
                    }
                    if (compact && eq[e]) {
                        sm.keys[e_before] = static_cast<KeyT>(x[e]);
                        sm.pos[e_before] = p[e];
                    }
                }
                sel_run += total & 0xffffu;
                eq_run += total >> 16;
            }
            if (last) break;
            written += sel_run;
            if (compact) in_smem = cand;
            // the bucket of digit t that holds the need-th candidate
            __syncthreads();
            uint32_t c = 0;
            if (tid < kRadix) {
#pragma unroll
                for (int w = 0; w < kTopkWarps; ++w) { c += sm.hist[w * kRadix + tid]; sm.hist[w * kRadix + tid] = 0; }
            }
            const uint32_t excl = block_excl_scan_256<kTopkThreads>(c, sm.wtot);
            if (tid < kRadix && c && excl < need && need <= excl + c) {
                sm.pick[0] = tid;
                sm.pick[1] = excl;
                sm.pick[2] = c;
            }
            __syncthreads();
            const uint32_t b = sm.pick[0];
            need -= sm.pick[1];
            cand = sm.pick[2];
            mprev = mcur;
            vprev = vcur;
            mcur |= static_cast<U>(0xffu) << shift;
            vcur |= static_cast<U>(b) << shift;
            last = cand == need || t + 1 == D;
        }
        if constexpr (LIST) {
            const KeyT pad = dec ? codec_decode<KeyT>(static_cast<KeyT>(~static_cast<KeyT>(0)), ca, cb, cd) : static_cast<KeyT>(~static_cast<KeyT>(0));
            for (uint32_t c = m + tid; c < k; c += kTopkThreads) {
                dst[c] = pad;
                dst_idx[c] = 0xFFFFFFFFu;
            }
        }
        __syncthreads();  // the next row's pass 0 may compact into the buffer this row's last pass read
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kTopkThreads, 1)
topk_select_kernel(const KeyT* __restrict__ in, KeyT* __restrict__ out, uint32_t* __restrict__ idx_out, uint64_t num_rows,
                   uint32_t row_len, uint32_t k, uint32_t cap, KeyCodec codec)
{
    topk_select_body<KeyT, false>(in, out, idx_out, num_rows, row_len, k, cap, codec, nullptr, nullptr, nullptr);
}

// topk_warp_kernel: rows of row_len <= 32 K keys of `in`; the first k of each sorted row go to row r * k of out / idx_out.
// With idx_in (the in-place sort of a block-path result: in == out, idx_in == idx_out, row_len == k) the payloads are loaded.
template <typename KeyT, int K, int RANK_MODE>
__global__ void __launch_bounds__(kRowWarps * 32)
topk_warp_kernel(const KeyT* in, KeyT* out, const uint32_t* idx_in, uint32_t* idx_out, uint64_t num_rows, uint32_t row_len,
                 uint32_t k, KeyCodec codec)
{
    using W = RowWarpSmem<KeyT, K, true>;
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    W& sm = reinterpret_cast<W*>(s_raw)[warp];
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(sm.hist, codec);
    for (uint64_t row = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; row < num_rows;
         row += static_cast<uint64_t>(gridDim.x) * kRowWarps)
        warp_sort_run<KeyT, K, RANK_MODE, true, true>(sm, x, in, out, idx_out, row * row_len, row_len, idx_in, row * k, k);
}

// topk_sort_kernel: the row sort's block body (ROWS) on the [num_rows, k] block-path result, in place, with the gathered
// positions as payloads.  A kernel of its own, so that segment_sort_kernel keeps its instantiations.
template <typename KeyT, int K, int WARPS, int RANK_MODE>
__global__ void __launch_bounds__(WARPS * 32, 1)
topk_sort_kernel(KeyT* keys, uint32_t* vals, uint64_t num_rows, uint32_t k, KeyCodec codec)
{
    segment_sort_body<KeyT, true, K, WARPS, RANK_MODE, false, true, false>(keys, vals, nullptr, num_rows, k, k, 0u, sizeof(KeyT),
                                                                          8u, codec, keys, nullptr, nullptr);
}

// =====================================================================================================
// Segment top-k (osb200_topk_segments): row top-k for ragged segments given by offsets.  Segment s's result is row s of a
// [num_segments, k] output: its first m = min(length, k) keys in the stable sort and their positions, then k - m columns of
// padding -- the key whose radix image is all ones (it sorts last) and the position 0xFFFFFFFF.
//   * topk_segment_bin_kernel (segment_bin_body, TOPK) lists every segment: up to 256 keys, and the empty and invalid ones,
//     on the warp list, longer ones on the block list.
//   * topk_segment_warp_kernel: one warp per segment of the warp list (warp_sort_run, TOPK and PAD), then the padding past
//     the warp's 32 K columns, coalesced.
//   * topk_segment_select_kernel: topk_select_body in list mode, one CTA per segment of the block list.
//   * sorted: only the radix select's rows are sorted in place, whole k-wide rows -- the padding's image is all ones and the
//     sort is stable, so it stays at the tail: topk_segment_sort_warp_kernel (over the block list) for k <= 256, else
//     topk_segment_sort_kernel (over all rows, skipping the warp class's by their offsets).
// Every class kernel runs on the resident CTAs and reads its count on the device, so nothing waits on the host.
// =====================================================================================================
__global__ void __launch_bounds__(256)
topk_segment_bin_kernel(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n, uint32_t warp_max,
                        uint32_t* __restrict__ list, unsigned long long* __restrict__ counts)
{
    segment_bin_body<uint32_t, true>(off, num_segments, n, 0u, list, counts, nullptr, nullptr, nullptr, warp_max);
}

template <typename KeyT, int RANK_MODE>
__global__ void __launch_bounds__(kRowWarps * 32)
topk_segment_warp_kernel(const KeyT* in, KeyT* out, uint32_t* __restrict__ idx_out, uint64_t n,
                         const unsigned long long* __restrict__ off, const uint32_t* __restrict__ list,
                         const unsigned long long* __restrict__ counts, uint32_t k, KeyCodec codec)
{
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    unsigned char* wsm = s_raw + warp * sizeof(RowWarpSmem<KeyT, 8, true>);  // every K's layout starts with the same hist
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(reinterpret_cast<uint32_t*>(wsm), codec);
    const KeyT ones = static_cast<KeyT>(~static_cast<KeyT>(0));
    const KeyT pad = x.dec ? codec_decode<KeyT>(ones, x.ca, x.cb, x.cd) : ones;
    const uint64_t count = counts[kSegCountWarp];
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; i < count; i += static_cast<uint64_t>(gridDim.x) * kRowWarps) {
        const uint32_t s = list[i];
        const unsigned long long lo = off[s], hi = off[s + 1];
        // offsets that decrease, pass n or span 2^32 keys or more: the binning kernel listed it here as empty
        const uint32_t len = lo <= hi && hi <= n && hi - lo <= kRowWarpMaxLen ? static_cast<uint32_t>(hi - lo) : 0u;
        const uint64_t obase = static_cast<uint64_t>(s) * k;
        uint32_t stored;  // the columns warp_sort_run stores: min(k, 32 K)
        if (len <= 32) {
            stored = min(k, 32u);
            warp_sort_run<KeyT, 1, RANK_MODE, true, true, true>(*reinterpret_cast<RowWarpSmem<KeyT, 1, true>*>(wsm), x, in, out, idx_out,
                                                                lo, len, nullptr, obase, stored);
        } else if (len <= 64) {
            stored = min(k, 64u);
            warp_sort_run<KeyT, 2, RANK_MODE, true, true, true>(*reinterpret_cast<RowWarpSmem<KeyT, 2, true>*>(wsm), x, in, out, idx_out,
                                                                lo, len, nullptr, obase, stored);
        } else if (len <= 128) {
            stored = min(k, 128u);
            warp_sort_run<KeyT, 4, RANK_MODE, true, true, true>(*reinterpret_cast<RowWarpSmem<KeyT, 4, true>*>(wsm), x, in, out, idx_out,
                                                                lo, len, nullptr, obase, stored);
        } else {
            stored = min(k, 256u);
            warp_sort_run<KeyT, 8, RANK_MODE, true, true, true>(*reinterpret_cast<RowWarpSmem<KeyT, 8, true>*>(wsm), x, in, out, idx_out,
                                                                lo, len, nullptr, obase, stored);
        }
        for (uint32_t c = stored + x.lane; c < k; c += 32) {
            out[obase + c] = pad;
            idx_out[obase + c] = 0xFFFFFFFFu;
        }
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kTopkThreads, 1)
topk_segment_select_kernel(const KeyT* __restrict__ in, KeyT* __restrict__ out, uint32_t* __restrict__ idx_out, uint64_t num_segments,
                           uint32_t k, uint32_t cap, KeyCodec codec, const unsigned long long* __restrict__ off,
                           const uint32_t* __restrict__ list, const unsigned long long* __restrict__ counts)
{
    topk_select_body<KeyT, true>(in, out, idx_out, num_segments, 0u, k, cap, codec, off, list, counts);
}

// the sorted pass of the block list's rows (k <= 32 K), in place, the positions loaded as payloads
template <typename KeyT, int K, int RANK_MODE>
__global__ void __launch_bounds__(kRowWarps * 32)
topk_segment_sort_warp_kernel(KeyT* keys, uint32_t* idx, uint64_t num_segments, uint32_t k, const uint32_t* __restrict__ list,
                              const unsigned long long* __restrict__ counts, KeyCodec codec)
{
    using W = RowWarpSmem<KeyT, K, true>;
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    W& sm = reinterpret_cast<W*>(s_raw)[warp];
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(sm.hist, codec);
    const uint64_t count = counts[kSegCountBlockList];
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; i < count; i += static_cast<uint64_t>(gridDim.x) * kRowWarps) {
        const uint64_t row = static_cast<uint64_t>(list[num_segments - 1 - i]) * k;
        warp_sort_run<KeyT, K, RANK_MODE, true, true>(sm, x, keys, keys, idx, row, k, idx, row, k);
    }
}

// the sorted pass of the radix select's rows for k > 256: the row sort's block body (ROWS, ROW_SEL), in place
template <typename KeyT, int K, int WARPS, int RANK_MODE>
__global__ void __launch_bounds__(WARPS * 32, 1)
topk_segment_sort_kernel(KeyT* keys, uint32_t* vals, uint64_t num_segments, uint32_t k, KeyCodec codec,
                         const unsigned long long* __restrict__ off, uint64_t n, uint32_t warp_max)
{
    segment_sort_body<KeyT, true, K, WARPS, RANK_MODE, false, true, false, true>(keys, vals, off, num_segments, k, k, 0u, sizeof(KeyT),
                                                                                8u, codec, keys, nullptr, nullptr, n, warp_max);
}

template <typename KeyT, int SIZE>
struct TopkSortShape {
    using Key = KeyT;
    static constexpr bool has_hot = false;
    using G = SegGeomN<KeyT, SIZE>;
    using S = SegSmem<KeyT, true, G::K, G::WARPS>;
    static constexpr uint32_t T = S::T;
    static constexpr size_t smem = sizeof(S);
    template <int RANK_MODE, bool HOT = false>
    static constexpr auto kernel() { return topk_sort_kernel<KeyT, G::K, G::WARPS, RANK_MODE>; }
    template <int RANK_MODE>
    static constexpr auto list_kernel() { return topk_segment_sort_kernel<KeyT, G::K, G::WARPS, RANK_MODE>; }
};
using TopkSortShapes = TypeList<TopkSortShape<uint16_t, 1>, TopkSortShape<uint16_t, 2>, TopkSortShape<uint32_t, 1>,
                                TopkSortShape<uint32_t, 2>, TopkSortShape<uint64_t, 1>, TopkSortShape<uint64_t, 2>>;
using TopkKeys = TypeList<uint16_t, uint32_t, uint64_t>;

// `sorted` for a [num_rows, k] result of at most C columns, in place with its positions as payloads: one warp per row for
// k <= 32 K, else the row sort's block body.
template <typename KeyT, int R>
static cudaError_t sort_topk_result(KeyT* out, uint32_t* indices, uint64_t num_rows, uint32_t k, const KeyCodec& codec, int sm_count,
                                    cudaStream_t stream)
{
    if (k <= kRowWarpMaxLen)
        return with_warp_k(k, [&](auto kk) {
            constexpr int K = decltype(kk)::value;
            return launch_resident<topk_warp_kernel<KeyT, K, R>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, K, true>>(
                (num_rows + kRowWarps - 1) / kRowWarps, sm_count, stream, out, out, indices, indices, num_rows, k, k, codec);
        });
    return find_type(
        TopkSortShapes{},
        [&](auto s) { using Sh = decltype(s); return std::is_same_v<typename Sh::Key, KeyT> && k <= Sh::T; },
        [&](auto s) {
            using Sh = decltype(s);
            return launch_resident<Sh::template kernel<R>(), Sh::S::THREADS, Sh::smem>(
                num_rows, sm_count, stream, reinterpret_cast<typename Sh::Key*>(out), indices, num_rows, k, codec);
        });
}

cudaError_t launch_topk_rows(const void* keys_in, void* values_out, uint32_t* indices, uint64_t num_rows, uint32_t row_len,
                             uint32_t k, int key_bytes, const KeyCodec* codec_in, bool sorted, uint32_t capacity, int rank_mode,
                             bool block_only, int sm_count, cudaStream_t stream)
{
    if (num_rows == 0 || row_len == 0 || k == 0) return cudaSuccess;
    if (k > row_len || k > row_sort_capacity(key_bytes)) return cudaErrorInvalidValue;
    const uint32_t cap = capacity && capacity < row_sort_capacity(key_bytes) ? capacity : row_sort_capacity(key_bytes);
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    return with_key_type(TopkKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        KeyT* out = static_cast<KeyT*>(values_out);
        return with_rank_mode(rank_mode, [&](auto r) {
            constexpr int R = decltype(r)::value;
            // one warp per row of `src`: its first k sorted keys go to row r * k of out
            auto warp_rows = [&](const KeyT* src, const uint32_t* idx_in, uint32_t len) {
                return with_warp_k(len, [&](auto kk) {
                    constexpr int K = decltype(kk)::value;
                    return launch_resident<topk_warp_kernel<KeyT, K, R>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, K, true>>(
                        (num_rows + kRowWarps - 1) / kRowWarps, sm_count, stream, src, out, idx_in, indices, num_rows, len, k, codec);
                });
            };
            if (row_len <= kRowWarpMaxLen && !block_only) return warp_rows(in, nullptr, row_len);  // sorted already
            const cudaError_t e = launch_resident<topk_select_kernel<KeyT>, kTopkThreads, sizeof(TopkSmem<KeyT>)>(
                num_rows, sm_count, stream, in, out, indices, num_rows, row_len, k, cap, codec);
            if (e != cudaSuccess || !sorted || k == 1) return e;
            return sort_topk_result<KeyT, R>(out, indices, num_rows, k, codec, sm_count, stream);
        });
    });
}

cudaError_t launch_topk_segments(const void* keys_in, void* values_out, uint32_t* indices, uint64_t n, const unsigned long long* off,
                                 uint64_t num_segments, uint32_t k, int key_bytes, const KeyCodec* codec_in, bool sorted,
                                 uint32_t capacity, int rank_mode, bool block_only, int sm_count, uint32_t* list,
                                 unsigned long long* counts, cudaStream_t stream)
{
    if (num_segments == 0 || k == 0) return cudaSuccess;
    if (k > row_sort_capacity(key_bytes)) return cudaErrorInvalidValue;
    const uint32_t cap = capacity && capacity < row_sort_capacity(key_bytes) ? capacity : row_sort_capacity(key_bytes);
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    cudaError_t e = cudaMemsetAsync(counts, 0, kSegCounts * sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const uint32_t warp_max = block_only ? 0u : kRowWarpMaxLen;
    topk_segment_bin_kernel<<<capped_grid(num_segments, 256, static_cast<uint64_t>(sm_count) * 8), 256, 0, stream>>>(
        off, num_segments, n, warp_max, list, counts);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return with_key_type(TopkKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        KeyT* out = static_cast<KeyT*>(values_out);
        return with_rank_mode(rank_mode, [&](auto r) {
            constexpr int R = decltype(r)::value;
            cudaError_t le = launch_resident<topk_segment_warp_kernel<KeyT, R>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, 8, true>>(
                kAllResident, sm_count, stream, in, out, indices, n, off, list, counts, k, codec);
            if (le == cudaSuccess)
                le = launch_resident<topk_segment_select_kernel<KeyT>, kTopkThreads, sizeof(TopkSmem<KeyT>)>(
                    kAllResident, sm_count, stream, in, out, indices, num_segments, k, cap, codec, off, list, counts);
            if (le != cudaSuccess || !sorted || k == 1) return le;
            // sorted: the block list's rows, in place (the warp list's are sorted already)
            if (k <= kRowWarpMaxLen)
                return with_warp_k(k, [&](auto kk) {
                    constexpr int K = decltype(kk)::value;
                    return launch_resident<topk_segment_sort_warp_kernel<KeyT, K, R>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, K, true>>(
                        kAllResident, sm_count, stream, out, indices, num_segments, k, list, counts, codec);
                });
            return find_type(
                TopkSortShapes{},
                [&](auto s) { using Sh = decltype(s); return std::is_same_v<typename Sh::Key, KeyT> && k <= Sh::T; },
                [&](auto s) {
                    using Sh = decltype(s);
                    return launch_resident<Sh::template list_kernel<R>(), Sh::S::THREADS, Sh::smem>(
                        num_segments, sm_count, stream, static_cast<typename Sh::Key*>(values_out), indices, num_segments, k, codec,
                        off, n, warp_max);
                });
        });
    });
}

// =====================================================================================================
// Row top-k of long rows (osb200_topk_long_rows, DESIGN §4.18): the split path.  An MSD radix select per row over the long
// rows' tiles (LongRowGeo: 8,192 keys, none straddling rows), every kernel grid-striding over all rows' tiles (or rows) on
// the resident CTAs; no tile waits on another, and each kernel returns at once when it has no work.
//   * level t = 0 .. D - 1: topk_long_count_kernel counts digit t of every tile's candidates of an active row into the
//     tile's 256 counts (cnt) and adds them to the row's totals (tot); first it adds the tile's keys below the previous
//     level's chosen digit to its selected count.  topk_long_pick_kernel picks per row the digit holding the need-th
//     candidate, as topk_select_body does; the row is resolved when its candidates are exactly the keys it needs or after
//     the last digit, stopped when they are at most cap.
//   * topk_long_tiles_kernel: the last level's fold, and each tile's candidate count.
//   * bases: the exclusive scan of each row's [selected of its tiles, candidates of its tiles] with the long rows' scan
//     kernels (a zeroed SortPlan: no place skipped), so the candidates' bases come out offset by the row's selected total.
//   * topk_long_compact_kernel: the ordered compaction of every tile, in row order -- selected keys to their columns, the
//     first `need` candidates of a resolved row after them, every candidate of a stopped row (at most cap) with its
//     position to the row's own range of the alternate buffers.
//   * topk_long_finish_kernel: topk_select_body (FIN) over the stopped rows' candidates, one CTA per row.
// =====================================================================================================
template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
topk_long_count_kernel(const KeyT* __restrict__ in, uint64_t num_rows, uint32_t row_len, uint32_t tpr, uint32_t k, uint32_t level,
                       const TopkLongRow* __restrict__ rows, uint32_t* __restrict__ tot, uint32_t* cnt, uint32_t* __restrict__ sc,
                       KeyCodec codec)
{
    if (k == row_len) return;  // every row is resolved before level 0
    using U = std::conditional_t<sizeof(KeyT) == 8, uint64_t, uint32_t>;
    const uint32_t shift = 8u * (static_cast<uint32_t>(sizeof(KeyT)) - 1u - level);
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = codec.flags & kCodecEncodeOnLoad;
    // bank-private columns, as in long_count_body
    __shared__ uint32_t s_hist[kRadix * 32];
    __shared__ uint32_t s_sel;
    uint32_t* s_col = s_hist + (threadIdx.x & 31);
    const LongRowGeo geo{num_rows, row_len, tpr, 0, 0};
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        const TopkLongRow st = rows[x.r];
        if (st.status != kTopkLongActive) continue;
        for (int i = threadIdx.x; i < kRadix * 32; i += kLongThreads) s_hist[i] = 0;
        if (threadIdx.x == 0) s_sel = 0;
        __syncthreads();
        // the previous level's counts below its chosen digit are selected keys
        if (level > 0 && threadIdx.x < st.b) atomicAdd(&s_sel, cnt[g * kRadix + threadIdx.x]);
        const U m = static_cast<U>(st.m), v = static_cast<U>(st.v);
        const KeyT* tile = in + x.lo + x.t0;
        KeyT key[kLongK];
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            const uint32_t j = threadIdx.x + i * kLongThreads;
            key[i] = j < x.len ? tile[j] : static_cast<KeyT>(0);
        }
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            if (threadIdx.x + i * kLongThreads >= x.len) break;
            const U e = static_cast<U>(enc ? codec_encode<KeyT>(key[i], ca, cb, cd) : key[i]);
            if ((e & m) == v) atomicAdd(&s_col[digit_of(e, shift) * 32], 1u);
        }
        __syncthreads();
        if (threadIdx.x < kRadix) {
            uint32_t sum = 0;
#pragma unroll 8
            for (int c = 0; c < 32; ++c) sum += s_hist[threadIdx.x * 32 + ((c + threadIdx.x) & 31)];
            cnt[g * kRadix + threadIdx.x] = sum;
            if (sum) atomicAdd(&tot[x.r * kRadix + threadIdx.x], sum);
        }
        if (threadIdx.x == 0 && level > 0) sc[x.r * 2 * tpr + x.t] += s_sel;
        __syncthreads();  // the fold has read s_hist
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kRadix)
topk_long_pick_kernel(uint64_t num_rows, uint32_t row_len, uint32_t k, uint32_t level, uint32_t cap, TopkLongRow* __restrict__ rows,
                      uint32_t* __restrict__ tot)
{
    if (k == row_len) return;
    constexpr uint32_t D = sizeof(KeyT);
    const uint32_t shift = 8u * (D - 1u - level);
    __shared__ uint32_t s_wtot[kRadix / 32];
    for (uint64_t r = blockIdx.x; r < num_rows; r += gridDim.x) {
        const TopkLongRow st = rows[r];
        if (st.status != kTopkLongActive) continue;
        const uint32_t c = tot[r * kRadix + threadIdx.x];
        tot[r * kRadix + threadIdx.x] = 0;  // for the next level
        const uint32_t excl = block_excl_scan_256<kRadix>(c, s_wtot);
        const uint32_t need = k - st.taken;
        if (c && excl < need && need <= excl + c) {
            TopkLongRow nx = st;
            nx.v |= static_cast<unsigned long long>(threadIdx.x) << shift;
            nx.m |= 0xffull << shift;
            nx.taken += excl;
            nx.cand = c;
            nx.b = threadIdx.x;
            nx.status = c == need - excl || level + 1 == D ? kTopkLongResolved : c <= cap ? kTopkLongStopped : kTopkLongActive;
            rows[r] = nx;
        }
        __syncthreads();  // s_wtot is reused by the next row
    }
}

// The last level's fold: each tile's selected count gains its keys below the row's last chosen digit, and its candidate
// count is its count of that digit (k == row_len: no level ran, every key is a candidate).
__global__ void __launch_bounds__(kRadix)
topk_long_tiles_kernel(uint64_t num_rows, uint32_t row_len, uint32_t tpr, uint32_t k, const TopkLongRow* __restrict__ rows,
                       const uint32_t* __restrict__ cnt, uint32_t* __restrict__ sc)
{
    __shared__ uint32_t s_sel;
    const LongRowGeo geo{num_rows, row_len, tpr, 0, 0};
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        uint32_t* s = sc + x.r * 2 * tpr;
        if (k == row_len) {
            if (threadIdx.x == 0) { s[x.t] = 0; s[tpr + x.t] = x.len; }
            continue;
        }
        const uint32_t b = rows[x.r].b;
        if (threadIdx.x == 0) s_sel = 0;
        __syncthreads();
        const uint32_t c = cnt[g * kRadix + threadIdx.x];
        if (threadIdx.x < b && c) atomicAdd(&s_sel, c);
        if (threadIdx.x == b) s[tpr + x.t] = c;
        __syncthreads();
        if (threadIdx.x == 0) s[x.t] += s_sel;
        __syncthreads();  // s_sel is reused by the next tile
    }
}

// The ordered compaction of every tile (two chunks of 4,096 keys, each ranked by per-warp ballots and a scan of the
// chunk's packed (e, warp) counts in row order, as in topk_select_body), from the tile's bases in sc.
template <typename KeyT>
__global__ void __launch_bounds__(kTopkThreads)
topk_long_compact_kernel(const KeyT* __restrict__ in, KeyT* __restrict__ out, uint32_t* __restrict__ idx_out, uint64_t num_rows,
                         uint32_t row_len, uint32_t tpr, uint32_t k, const TopkLongRow* __restrict__ rows,
                         const uint32_t* __restrict__ sc, KeyT* __restrict__ buf, uint32_t* __restrict__ buf_pos, KeyCodec codec)
{
    using U = std::conditional_t<sizeof(KeyT) == 8, uint64_t, uint32_t>;
    constexpr uint32_t CHUNK = kTopkE * kTopkThreads;
    __shared__ uint32_t s_cnt[2][kTopkE * kTopkWarps];  // per chunk (double-buffered): selected | candidates << 16
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t lt = lanemask_lt();
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = codec.flags & kCodecEncodeOnLoad, dec = codec.flags & kCodecDecodeOnStore;
    const LongRowGeo geo{num_rows, row_len, tpr, 0, 0};
    const uint64_t tiles = geo.tiles();
    uint32_t parity = 0;
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        TopkLongRow st{};
        st.status = kTopkLongResolved;
        if (k != row_len) st = rows[x.r];
        const uint32_t* s = sc + x.r * 2 * tpr;
        const uint32_t need = k - st.taken;
        const bool stopped = st.status == kTopkLongStopped;
        uint32_t sel_run = s[x.t], eq_run = s[tpr + x.t] - st.taken;
        const U m = static_cast<U>(st.m), v = static_cast<U>(st.v);
        const KeyT* src = in + x.lo + x.t0;
        KeyT* dst = out + x.r * k;
        uint32_t* dst_idx = idx_out + x.r * k;
        for (uint32_t c0 = 0; c0 < x.len; c0 += CHUNK, parity ^= 1u) {
            U xv[kTopkE];
            bool sel[kTopkE], eq[kTopkE];
#pragma unroll
            for (int e = 0; e < kTopkE; ++e) {
                const uint32_t i = c0 + static_cast<uint32_t>(e * kTopkThreads + tid);
                const bool valid = i < x.len;
                KeyT kv = valid ? src[i] : static_cast<KeyT>(0);
                xv[e] = static_cast<U>(enc ? codec_encode<KeyT>(kv, ca, cb, cd) : kv);
                sel[e] = valid && (xv[e] & m) < v;
                eq[e] = valid && (xv[e] & m) == v;
            }
            uint32_t bsel[kTopkE], beq[kTopkE];
            uint32_t* cnt = s_cnt[parity];
#pragma unroll
            for (int e = 0; e < kTopkE; ++e) {
                bsel[e] = __ballot_sync(0xffffffffu, sel[e]);
                beq[e] = __ballot_sync(0xffffffffu, eq[e]);
                if (lane == 0) cnt[e * kTopkWarps + warp] = __popc(bsel[e]) | (__popc(beq[e]) << 16);
            }
            __syncthreads();
            const uint4 c4 = reinterpret_cast<const uint4*>(cnt)[lane];
            const uint32_t s4 = c4.x + c4.y + c4.z + c4.w;
            uint32_t incl = s4;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
            const uint32_t sub = warp & 3;
            const uint32_t mine = incl - s4 + (sub > 0 ? c4.x : 0u) + (sub > 1 ? c4.y : 0u) + (sub > 2 ? c4.z : 0u);
#pragma unroll
            for (int e = 0; e < kTopkE; ++e) {
                const uint32_t pre = __shfl_sync(0xffffffffu, mine, 4 * e + (warp >> 2));
                const uint32_t p = x.t0 + c0 + static_cast<uint32_t>(e * kTopkThreads + tid);
                if (sel[e] || (eq[e] && !stopped)) {
                    const uint32_t s_before = sel_run + (pre & 0xffffu) + __popc(bsel[e] & lt);
                    const uint32_t e_before = eq_run + (pre >> 16) + __popc(beq[e] & lt);
                    if (sel[e] || e_before < need) {
                        const uint32_t o = sel[e] ? s_before : st.taken + e_before;
                        KeyT kv = static_cast<KeyT>(xv[e]);
                        if (dec) kv = codec_decode<KeyT>(kv, ca, cb, cd);
                        dst[o] = kv;
                        dst_idx[o] = p;
                    }
                } else if (eq[e]) {
                    const uint32_t e_before = eq_run + (pre >> 16) + __popc(beq[e] & lt);
                    buf[x.lo + e_before] = static_cast<KeyT>(xv[e]);
                    buf_pos[x.lo + e_before] = p;
                }
            }
            sel_run += total & 0xffffu;
            eq_run += total >> 16;
        }
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kTopkThreads, 1)
topk_long_finish_kernel(const KeyT* __restrict__ buf, KeyT* __restrict__ out, uint32_t* __restrict__ idx_out, uint64_t num_rows,
                        uint32_t row_len, uint32_t k, uint32_t cap, KeyCodec codec, const TopkLongRow* __restrict__ rows,
                        const uint32_t* __restrict__ buf_pos)
{
    topk_select_body<KeyT, false, true>(buf, out, idx_out, num_rows, row_len, k, cap, codec, nullptr, nullptr, nullptr, rows, buf_pos);
}

TopkLongLayout topk_long_layout(uint64_t num_rows, uint32_t row_len)
{
    static_assert(sizeof(SortPlan) <= 16 * sizeof(uint32_t) && sizeof(TopkLongRow) == 8 * sizeof(uint32_t), "the layout's words");
    auto whole = [](uint64_t words) { return (words + 3) / 4 * 4; };
    TopkLongLayout l;
    l.tpr = static_cast<uint32_t>((static_cast<uint64_t>(row_len) + kLongRowTile - 1) / kLongRowTile);
    l.cpr = static_cast<uint32_t>((2ull * l.tpr + kLongChunk - 1) / kLongChunk);
    l.rows = 16;
    l.tot = l.rows + num_rows * 8;
    l.sc = l.tot + num_rows * kRadix;
    l.zeroed = whole(l.sc + num_rows * 2 * l.tpr);
    l.words = l.zeroed + (l.cpr > 1 ? whole(num_rows * l.cpr) : 0);
    l.cnt_words = num_rows * l.tpr * kRadix;
    return l;
}

cudaError_t launch_topk_long_rows(const void* keys_in, void* values_out, uint32_t* indices, void* alt_keys, uint32_t* alt_idx,
                                  uint64_t num_rows, uint32_t row_len, uint32_t k, int key_bytes, const KeyCodec* codec_in, bool sorted,
                                  uint32_t capacity, int rank_mode, bool allow_skip, unsigned long long* ghist, unsigned long long* gbase,
                                  SortPlan* plan, uint32_t* scratch, int sm_count, cudaStream_t stream)
{
    if (num_rows == 0 || row_len < 2 || k == 0 || k > row_len) return cudaErrorInvalidValue;
    const TopkLongLayout l = topk_long_layout(num_rows, row_len);
    const uint32_t C = row_sort_capacity(key_bytes);
    const uint32_t cap = capacity && capacity < C ? capacity : C;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    cudaError_t e = cudaMemsetAsync(scratch, 0, l.zeroed * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    const SortPlan* none_skipped = reinterpret_cast<const SortPlan*>(scratch);
    TopkLongRow* rows = reinterpret_cast<TopkLongRow*>(scratch + l.rows);
    uint32_t* tot = scratch + l.tot;
    uint32_t* sc = scratch + l.sc;
    uint32_t* csum = l.cpr > 1 ? scratch + l.zeroed : nullptr;
    uint32_t* cnt = alt_idx;  // free until the compaction writes the candidates' positions there
    const uint64_t tiles = num_rows * l.tpr;
    return with_key_type(TopkKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        KeyT* out = static_cast<KeyT*>(values_out);
        KeyT* buf = static_cast<KeyT*>(alt_keys);
        cudaError_t le = cudaSuccess;
        for (uint32_t t = 0; le == cudaSuccess && t < sizeof(KeyT); ++t) {
            le = launch_resident<topk_long_count_kernel<KeyT>, kLongThreads, 0>(tiles, sm_count, stream, in, num_rows, row_len, l.tpr, k, t,
                                                                                static_cast<const TopkLongRow*>(rows), tot, cnt, sc, codec);
            if (le == cudaSuccess)
                le = launch_resident<topk_long_pick_kernel<KeyT>, kRadix, 0>(num_rows, sm_count, stream, num_rows, row_len, k, t, cap, rows, tot);
        }
        if (le == cudaSuccess)
            le = launch_resident<topk_long_tiles_kernel, kRadix, 0>(tiles, sm_count, stream, num_rows, row_len, l.tpr, k,
                                                                    static_cast<const TopkLongRow*>(rows), static_cast<const uint32_t*>(cnt), sc);
        if (le != cudaSuccess) return le;
        // the bases: per row, the exclusive scan of its 2 tpr counts [selected of each tile, candidates of each tile]
        const uint64_t row_counts = 2ull * l.tpr;
        const unsigned scan_grid = capped_grid(num_rows * l.cpr, 1, static_cast<uint64_t>(sm_count) * 4);
        if (csum) {
            long_rows_chunk_sum_kernel<<<scan_grid, kLongThreads, 0, stream>>>(none_skipped, 0, sc, csum, num_rows, row_counts, l.cpr);
            long_rows_chunk_scan_kernel<<<capped_grid(num_rows, 1, static_cast<uint64_t>(sm_count) * 4), kLongThreads, 0, stream>>>(
                none_skipped, 0, csum, num_rows, l.cpr);
        }
        long_rows_scan_kernel<<<scan_grid, kLongThreads, 0, stream>>>(none_skipped, 0, sc, csum, num_rows, row_counts, l.cpr);
        if ((le = cudaGetLastError()) != cudaSuccess) return le;
        le = launch_resident<topk_long_compact_kernel<KeyT>, kTopkThreads, 0>(tiles, sm_count, stream, in, out, indices, num_rows, row_len,
                                                                             l.tpr, k, static_cast<const TopkLongRow*>(rows),
                                                                             static_cast<const uint32_t*>(sc), buf, alt_idx, codec);
        if (le == cudaSuccess)
            le = launch_resident<topk_long_finish_kernel<KeyT>, kTopkThreads, sizeof(TopkSmem<KeyT>)>(
                num_rows, sm_count, stream, static_cast<const KeyT*>(buf), out, indices, num_rows, row_len, k, cap, codec,
                static_cast<const TopkLongRow*>(rows), static_cast<const uint32_t*>(alt_idx));
        if (le != cudaSuccess || !sorted || k == 1) return le;
        if (k <= C)
            return with_rank_mode(rank_mode, [&](auto r) { return sort_topk_result<KeyT, decltype(r)::value>(out, indices, num_rows, k, codec, sm_count, stream); });
        // k > C: the long rows' passes over the [num_rows, k] result, in place, loading the positions as payloads (the
        // control block's histogram was cleared by the caller)
        return launch_long_rows(out, out, indices, alt_keys, alt_idx, num_rows, k, key_bytes, codec_in, rank_mode, allow_skip, ghist, gbase,
                                plan, scratch, sm_count, stream, true);
    });
}

// =====================================================================================================
// Row select (osb200_select_rows, DESIGN §4.19): columns r_0 < .. < r_{R-1} (R <= 16) of every row's ascending stable sort,
// and their positions within the row.
//
// Rows of at most row_sort_capacity keys: the row sort's kernels (warp_sort_run, segment_sort_body's ROWS mode) with the
// COLS store, which writes only the R columns.
//
// Longer rows (and, with the test hook, every row of two or more keys), the split path: a multi-rank MSD radix select over the
// long rows' tiles (LongRowGeo), no tile waiting on another.  Every (row, rank) has a state (SelectState): the prefix v of
// its key's top t digits (encoded) and `taken`, the keys of the row below v's range.  Level t = 0 .. D - 1:
//   * select_count_kernel: the ranks of a row whose prefixes are equal form a group (contiguous, the ranks increasing; one
//     group at level 0).  Each key of a tile matches at most one group's prefix and is counted once, by digit t, into that
//     group's 256 bins; the tile adds them to the row's totals of the group's first rank.
//   * select_pick_kernel: per group, each rank takes the bucket holding its (r - taken)-th candidate, extends its prefix and
//     adds the candidates below the bucket to taken; the totals are cleared for the next level.  After the last level v is
//     the key itself, and the pick writes the values.
// Positions: select_eq_count_kernel counts per tile the keys equal to each rank's key, the long rows' scan kernels scan each
// row's [rank][tile] counts, and select_locate_kernel finds occurrence r - taken in the one tile whose range holds it.
// =====================================================================================================
template <typename KeyT, int K, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(kRowWarps * 32)
select_rows_warp_kernel(const KeyT* in, KeyT* out, uint32_t* __restrict__ idx_out, uint64_t num_rows, uint32_t row_len, KeyCodec codec,
                        SelectRanks ranks)
{
    using W = RowWarpSmem<KeyT, K, INDICES>;
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    W& sm = reinterpret_cast<W*>(s_raw)[warp];
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(sm.hist, codec);
    for (uint64_t row = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; row < num_rows;
         row += static_cast<uint64_t>(gridDim.x) * kRowWarps)
        warp_sort_run<KeyT, K, RANK_MODE, INDICES, false, false, true>(sm, x, in, out, idx_out, row * row_len, row_len, nullptr,
                                                                      row * ranks.count, 0u, &ranks);
}

template <typename KeyT, int K, int WARPS, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(WARPS * 32, 1)
select_rows_block_kernel(const KeyT* __restrict__ in, KeyT* out, uint32_t* idx_out, uint64_t num_rows, uint32_t row_len, KeyCodec codec,
                         SelectRanks ranks)
{
    segment_sort_body<KeyT, INDICES, K, WARPS, RANK_MODE, INDICES, true, false, false, true>(
        out, idx_out, nullptr, num_rows, row_len, row_len, 0u, sizeof(KeyT), 8u, codec, in, nullptr, nullptr, 0, 0u, &ranks);
}

// the block path's geometries: 2,048 keys, and the row sort's capacity
template <typename KeyT, int SIZE, bool INDICES>
struct SelectShape {
    using Key = KeyT;
    static constexpr bool indices = INDICES, has_hot = false;
    using G = SegGeomN<KeyT, SIZE>;
    using S = SegSmem<KeyT, INDICES, G::K, G::WARPS>;
    static constexpr uint32_t T = S::T;
    static constexpr size_t smem = sizeof(S);
    template <int RANK_MODE, bool HOT = false>
    static constexpr auto kernel() { return select_rows_block_kernel<KeyT, G::K, G::WARPS, RANK_MODE, INDICES>; }
};
using SelectShapes = TypeList<
    SelectShape<uint16_t, 1, false>, SelectShape<uint16_t, 2, false>, SelectShape<uint16_t, 1, true>, SelectShape<uint16_t, 2, true>,
    SelectShape<uint32_t, 1, false>, SelectShape<uint32_t, 2, false>, SelectShape<uint32_t, 1, true>, SelectShape<uint32_t, 2, true>,
    SelectShape<uint64_t, 1, false>, SelectShape<uint64_t, 2, false>, SelectShape<uint64_t, 1, true>, SelectShape<uint64_t, 2, true>>;

cudaError_t launch_select_rows(const void* keys_in, void* values_out, uint32_t* indices, uint64_t num_rows, uint32_t row_len,
                               const SelectRanks& ranks, int key_bytes, const KeyCodec* codec_in, int rank_mode, bool block_only,
                               int sm_count, cudaStream_t stream)
{
    if (num_rows == 0 || row_len < 2 || row_len > row_sort_capacity(key_bytes) || ranks.count == 0 || ranks.count > kMaxSelectRanks)
        return cudaErrorInvalidValue;
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    return with_rank_mode(rank_mode, [&](auto r) {
        constexpr int R = decltype(r)::value;
        if (row_len <= kRowWarpMaxLen && !block_only)
            return with_key_type(TopkKeys{}, key_bytes, [&](auto k) {
                using KeyT = decltype(k);
                return with_warp_k(row_len, [&](auto kk) {
                    constexpr int K = decltype(kk)::value;
                    auto go = [&](auto ind) {
                        constexpr bool I = decltype(ind)::value;
                        return launch_resident<select_rows_warp_kernel<KeyT, K, R, I>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, K, I>>(
                            (num_rows + kRowWarps - 1) / kRowWarps, sm_count, stream, static_cast<const KeyT*>(keys_in),
                            static_cast<KeyT*>(values_out), indices, num_rows, row_len, codec, ranks);
                    };
                    return indices ? go(std::true_type{}) : go(std::false_type{});
                });
            });
        return find_type(
            SelectShapes{},
            [&](auto s) {
                using S = decltype(s);
                return key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::indices == (indices != nullptr) && row_len <= S::T;
            },
            [&](auto s) {
                using S = decltype(s);
                using KeyT = typename S::Key;
                return launch_resident<S::template kernel<R>(), S::S::THREADS, S::smem>(
                    num_rows, sm_count, stream, static_cast<const KeyT*>(keys_in), static_cast<KeyT*>(values_out), indices, num_rows,
                    row_len, codec, ranks);
            });
    });
}

// One (row, rank) of the split path: the prefix v (encoded; the top t digits at level t, the key after the last level) and
// the row's keys below v's range.  All zero is level 0.
struct SelectState { unsigned long long v; uint32_t taken, pad; };

// The groups of row r's ranks, by one warp (the caller's warp 0): s_v[g] the prefix of group g (ascending), s_first[g] its
// first rank, s_gi[i] rank i's group, *s_ng the number of groups.
template <typename U>
__device__ __forceinline__ void select_groups(const SelectState* __restrict__ rs, uint32_t nr, U* s_v, uint32_t* s_first,
                                              uint32_t* s_gi, uint32_t* s_ng)
{
    const uint32_t i = threadIdx.x;
    const U v = i < nr ? static_cast<U>(rs[i].v) : static_cast<U>(0);
    const U prev = __shfl_up_sync(0xffffffffu, v, 1);
    const bool first = i < nr && (i == 0 || v != prev);
    const uint32_t b = __ballot_sync(0xffffffffu, first);
    const uint32_t gi = __popc(b & lanemask_lt()) + (first ? 0u : 0xffffffffu);  // the last group starting at or before i
    if (first) { s_v[gi] = v; s_first[gi] = i; }
    if (i < nr) s_gi[i] = gi;
    if (i == 0) *s_ng = __popc(b);
}

// The group whose prefix p is, among the ng ascending prefixes s_v; ng when there is none.
template <typename U>
__device__ __forceinline__ uint32_t select_group_of(U p, const U* s_v, uint32_t ng)
{
    uint32_t g = 0;
#pragma unroll
    for (uint32_t step = kMaxSelectRanks / 2; step; step >>= 1)
        if (g + step < ng && s_v[g + step] <= p) g += step;
    return s_v[g] == p ? g : ng;
}

// The split path's bodies are templated on where the rows are (Geo): LongRowGeo, osb200_select_rows' rows with the ranks
// of the launch parameters, or LongSegGeo, osb200_select_segments' long list (DESIGN §4.20), whose entry j is segment list[j]
// with the ranks seg_ranks[list[j] * nr ..] in device memory.  A state, its totals and its tile counts are indexed by row or
// list entry.  A segment's ranks at or past its length, or all of them when they decrease, take no part: only the first
// `active` ranks are grouped, counted, picked and located, and the pick's last level pads the others.
__device__ __forceinline__ uint32_t select_active(const LongRowGeo&, uint64_t, uint32_t nr, const uint32_t*, uint32_t* = nullptr)
{
    return nr;
}
// (one whole warp; lane i < nr gets rank i in *rk)
__device__ __forceinline__ uint32_t select_active(const LongSegGeo& geo, uint64_t j, uint32_t nr, const uint32_t* __restrict__ seg_ranks,
                                                  uint32_t* rk = nullptr)
{
    const uint32_t lane = threadIdx.x & 31, s = geo.list[j];
    const uint32_t r = lane < nr ? seg_ranks[static_cast<uint64_t>(s) * nr + lane] : 0xffffffffu;
    if (rk) *rk = r;
    return select_ranks_active(r, nr, geo.off[s + 1] - geo.off[s]);
}
// the rows of the pick: num_rows, or the listed segments
__device__ __forceinline__ uint64_t select_rows_of(const LongRowGeo&, uint64_t num_rows) { return num_rows; }
__device__ __forceinline__ uint64_t select_rows_of(const LongSegGeo& geo, uint64_t) { return geo.listed(); }
// where row r's columns go in the [rows or segments, nr] outputs
__device__ __forceinline__ uint64_t select_obase(const LongRowGeo&, uint64_t r, uint32_t nr) { return r * nr; }
__device__ __forceinline__ uint64_t select_obase(const LongSegGeo& geo, uint64_t j, uint32_t nr)
{
    return static_cast<uint64_t>(geo.list[j]) * nr;
}
// where the equal-key counts of rank i of a tile's row start (tile t's is t further): [row][rank][tile], or per list entry
// [rank][tile] from nr * its first tile
__device__ __forceinline__ uint64_t select_cnt_base(const LongRowGeo& geo, const LongRowGeo::Tile& x, uint32_t nr, uint32_t i)
{
    return (x.r * nr + i) * geo.tpr;
}
__device__ __forceinline__ uint64_t select_cnt_base(const LongSegGeo&, const LongSegGeo::Tile& x, uint32_t nr, uint32_t i)
{
    return x.cb / kRadix * nr + static_cast<uint64_t>(i) * x.tpr;
}
__device__ __forceinline__ uint32_t select_tpr(const LongRowGeo& geo, const LongRowGeo::Tile&) { return geo.tpr; }
__device__ __forceinline__ uint32_t select_tpr(const LongSegGeo&, const LongSegGeo::Tile& x) { return x.tpr; }

template <typename KeyT, typename Geo>
__device__ __forceinline__ void select_count_body(const Geo& geo, const KeyT* __restrict__ in, uint32_t nr, uint32_t level,
                                                  const SelectState* __restrict__ st, uint32_t* __restrict__ tot, const KeyCodec& codec,
                                                  const uint32_t* __restrict__ seg_ranks)
{
    using U = std::conditional_t<sizeof(KeyT) == 8, uint64_t, uint32_t>;
    constexpr uint32_t D = sizeof(KeyT);
    const uint32_t shift = 8u * (D - 1u - level);
    const U m = level ? static_cast<U>(~static_cast<U>(0) << (8u * (D - level))) : static_cast<U>(0);
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = codec.flags & kCodecEncodeOnLoad;
    // a bin's counts in 2^lc bank-private columns, as in long_count_body (32 columns for one group, the skewed rows' case);
    // G groups take 32 / G columns or more, at most 8,192 counters
    __shared__ uint32_t s_hist[kRadix * 32];
    __shared__ U s_v[kMaxSelectRanks];
    __shared__ uint32_t s_first[kMaxSelectRanks], s_gi[kMaxSelectRanks], s_ng;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        if (threadIdx.x < 32) select_groups<U>(st + x.r * nr, select_active(geo, x.r, nr, seg_ranks), s_v, s_first, s_gi, &s_ng);
        __syncthreads();
        const uint32_t ng = s_ng;
        const uint32_t lc = ng <= 1 ? 5u : ng <= 2 ? 4u : ng <= 4 ? 3u : ng <= 8 ? 2u : 1u, cm = (1u << lc) - 1u;
        for (uint32_t i = threadIdx.x; i < (ng * kRadix << lc); i += kLongThreads) s_hist[i] = 0;
        __syncthreads();
        const KeyT* tile = in + x.lo + x.t0;
        KeyT key[kLongK];
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            const uint32_t j = threadIdx.x + i * kLongThreads;
            key[i] = j < x.len ? tile[j] : static_cast<KeyT>(0);
        }
        const U v0 = s_v[0];
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            if (threadIdx.x + i * kLongThreads >= x.len) break;
            const U e = static_cast<U>(enc ? codec_encode<KeyT>(key[i], ca, cb, cd) : key[i]);
            const U p = e & m;
            const uint32_t gi = ng == 1 ? (p == v0 ? 0u : 1u) : select_group_of<U>(p, s_v, ng);
            if (gi < ng) atomicAdd(&s_hist[((gi * kRadix + digit_of(e, shift)) << lc) + (lane & cm)], 1u);
        }
        __syncthreads();
        for (uint32_t b = threadIdx.x; b < ng * kRadix; b += kLongThreads) {
            uint32_t sum = 0;
            for (uint32_t c = 0; c <= cm; ++c) sum += s_hist[(b << lc) + ((c + b) & cm)];
            if (sum) atomicAdd(&tot[(x.r * nr + s_first[b / kRadix]) * kRadix + (b % kRadix)], sum);
        }
        __syncthreads();  // the fold has read s_hist and the groups
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
select_count_kernel(const KeyT* __restrict__ in, uint64_t num_rows, uint32_t row_len, uint32_t tpr, uint32_t nr, uint32_t level,
                    const SelectState* __restrict__ st, uint32_t* __restrict__ tot, KeyCodec codec)
{
    select_count_body<KeyT>(LongRowGeo{num_rows, row_len, tpr, 0, 0}, in, nr, level, st, tot, codec, nullptr);
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
select_segments_count_kernel(const KeyT* __restrict__ in, LongSegGeo geo, const uint32_t* __restrict__ seg_ranks, uint32_t nr,
                             uint32_t level, const SelectState* __restrict__ st, uint32_t* __restrict__ tot, KeyCodec codec)
{
    select_count_body<KeyT>(geo, in, nr, level, st, tot, codec, seg_ranks);
}

// rows: num_rows, with the ranks of `ranks`; long segments: the listed ones, with their own ranks (seg_ranks), and after the
// last level the columns that take no part are padded (idx_out: their positions, may be null)
template <typename KeyT, typename Geo>
__device__ __forceinline__ void select_pick_body(const Geo& geo, uint64_t num_rows, uint32_t nr, uint32_t level, SelectState* __restrict__ st,
                                                 uint32_t* __restrict__ tot, KeyT* __restrict__ out, const SelectRanks* ranks,
                                                 const KeyCodec& codec, const uint32_t* __restrict__ seg_ranks, uint32_t* idx_out)
{
    constexpr bool SEG = std::is_same_v<Geo, LongSegGeo>;
    constexpr uint32_t D = sizeof(KeyT);
    const uint32_t shift = 8u * (D - 1u - level);
    const bool last = level + 1 == D, dec = codec.flags & kCodecDecodeOnStore;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    __shared__ unsigned long long s_v[kMaxSelectRanks];
    __shared__ uint32_t s_taken[kMaxSelectRanks], s_need[kMaxSelectRanks], s_wtot[kRadix / 32], s_na;
    uint32_t rk = SEG ? 0u : select_rank_of(*ranks, threadIdx.x);
    const uint64_t rows = select_rows_of(geo, num_rows);
    for (uint64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        SelectState* rs = st + r * nr;
        uint32_t na = nr;
        if constexpr (SEG) {
            if (threadIdx.x < 32) {
                const uint32_t a = select_active(geo, r, nr, seg_ranks, &rk);
                if (threadIdx.x == 0) s_na = a;
            }
        }
        if (threadIdx.x < nr) {
            const SelectState s = rs[threadIdx.x];
            s_v[threadIdx.x] = s.v;
            s_taken[threadIdx.x] = s.taken;
            s_need[threadIdx.x] = rk - s.taken;
        }
        __syncthreads();
        if constexpr (SEG) na = s_na;
        const uint64_t ob = select_obase(geo, r, nr);
        for (uint32_t i = 0; i < na;) {  // group [i, j)
            uint32_t j = i + 1;
            while (j < na && s_v[j] == s_v[i]) ++j;
            uint32_t* t = tot + (r * nr + i) * kRadix;
            const uint32_t c = t[threadIdx.x];
            t[threadIdx.x] = 0;  // for the next level
            const uint32_t excl = block_excl_scan_256<kRadix>(c, s_wtot);
            for (uint32_t q = i; q < j; ++q) {
                const uint32_t need = s_need[q];
                if (excl <= need && need < excl + c) {  // (c > 0)
                    SelectState ns;
                    ns.v = s_v[q] | static_cast<unsigned long long>(threadIdx.x) << shift;
                    ns.taken = s_taken[q] + excl;
                    ns.pad = 0;
                    rs[q] = ns;
                    if (last) {
                        KeyT k = static_cast<KeyT>(ns.v);
                        if (dec) k = codec_decode<KeyT>(k, ca, cb, cd);
                        out[ob + q] = k;
                    }
                }
            }
            __syncthreads();  // s_wtot is reused by the next group, s_v etc. by the next row
            i = j;
        }
        if constexpr (SEG) {
            if (last && threadIdx.x >= na && threadIdx.x < nr) {
                const KeyT ones = static_cast<KeyT>(~static_cast<KeyT>(0));
                out[ob + threadIdx.x] = dec ? codec_decode<KeyT>(ones, ca, cb, cd) : ones;
                if (idx_out) idx_out[ob + threadIdx.x] = 0xFFFFFFFFu;
            }
            __syncthreads();  // s_na and s_v are rewritten for the next entry even when it had no group
        }
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kRadix)
select_pick_kernel(uint64_t num_rows, uint32_t level, SelectState* __restrict__ st, uint32_t* __restrict__ tot, KeyT* __restrict__ out,
                   SelectRanks ranks, KeyCodec codec)
{
    select_pick_body<KeyT>(LongRowGeo{num_rows, 0, 0, 0, 0}, num_rows, ranks.count, level, st, tot, out, &ranks, codec, nullptr, nullptr);
}

template <typename KeyT>
__global__ void __launch_bounds__(kRadix)
select_segments_pick_kernel(LongSegGeo geo, const uint32_t* __restrict__ seg_ranks, uint32_t nr, uint32_t level,
                            SelectState* __restrict__ st, uint32_t* __restrict__ tot, KeyT* __restrict__ out, uint32_t* idx_out,
                            KeyCodec codec)
{
    select_pick_body<KeyT>(geo, 0, nr, level, st, tot, out, nullptr, codec, seg_ranks, idx_out);
}

// Per tile, the keys equal to each rank's key (its group's), into the tile's count of the rank (select_cnt_index); a warp adds
// the lanes of one group at once.
template <typename KeyT, typename Geo>
__device__ __forceinline__ void select_eq_count_body(const Geo& geo, const KeyT* __restrict__ in, uint32_t nr,
                                                     const SelectState* __restrict__ st, uint32_t* __restrict__ cnt, const KeyCodec& codec,
                                                     const uint32_t* __restrict__ seg_ranks)
{
    using U = std::conditional_t<sizeof(KeyT) == 8, uint64_t, uint32_t>;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = codec.flags & kCodecEncodeOnLoad;
    __shared__ U s_v[kMaxSelectRanks];
    __shared__ uint32_t s_first[kMaxSelectRanks], s_gi[kMaxSelectRanks], s_ng, s_c[kMaxSelectRanks];
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        uint32_t na = nr;  // (warp 0's, which writes the counts)
        if (threadIdx.x < 32) {
            na = select_active(geo, x.r, nr, seg_ranks);
            select_groups<U>(st + x.r * nr, na, s_v, s_first, s_gi, &s_ng);
        }
        if (threadIdx.x < kMaxSelectRanks) s_c[threadIdx.x] = 0;
        __syncthreads();
        const uint32_t ng = s_ng;
        const KeyT* tile = in + x.lo + x.t0;
        KeyT key[kLongK];
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            const uint32_t j = threadIdx.x + i * kLongThreads;
            key[i] = j < x.len ? tile[j] : static_cast<KeyT>(0);
        }
#pragma unroll
        for (int i = 0; i < kLongK; ++i) {
            const bool valid = threadIdx.x + i * kLongThreads < x.len;
            const U e = static_cast<U>(enc ? codec_encode<KeyT>(key[i], ca, cb, cd) : key[i]);
            const uint32_t gi = valid ? select_group_of<U>(e, s_v, ng) : ng;
            const uint32_t peers = __match_any_sync(0xffffffffu, gi);
            if (gi < ng && lane == static_cast<uint32_t>(__ffs(peers) - 1)) atomicAdd(&s_c[gi], static_cast<uint32_t>(__popc(peers)));
        }
        __syncthreads();
        if (threadIdx.x < na) cnt[select_cnt_base(geo, x, nr, threadIdx.x) + x.t] = s_c[s_gi[threadIdx.x]];
        __syncthreads();  // s_c and the groups are reused by the next tile
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
select_eq_count_kernel(const KeyT* __restrict__ in, uint64_t num_rows, uint32_t row_len, uint32_t tpr, uint32_t nr,
                       const SelectState* __restrict__ st, uint32_t* __restrict__ cnt, KeyCodec codec)
{
    select_eq_count_body<KeyT>(LongRowGeo{num_rows, row_len, tpr, 0, 0}, in, nr, st, cnt, codec, nullptr);
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
select_segments_eq_count_kernel(const KeyT* __restrict__ in, LongSegGeo geo, const uint32_t* __restrict__ seg_ranks, uint32_t nr,
                                const SelectState* __restrict__ st, uint32_t* __restrict__ cnt, KeyCodec codec)
{
    select_eq_count_body<KeyT>(geo, in, nr, st, cnt, codec, seg_ranks);
}

// For every (row, rank) whose occurrence o = r - taken of its key lies in this tile by the scanned counts: the position of the
// tile's (o - tile prefix)-th key equal to it, in tile order (per-warp ballots and a scan of the warp counts, chunk by chunk).
template <typename KeyT, typename Geo>
__device__ __forceinline__ void select_locate_body(const Geo& geo, const KeyT* __restrict__ in, uint32_t* __restrict__ idx_out, uint32_t nr,
                                                   const SelectState* __restrict__ st, const uint32_t* __restrict__ cnt,
                                                   const SelectRanks* ranks, const KeyCodec& codec, const uint32_t* __restrict__ seg_ranks)
{
    constexpr bool SEG = std::is_same_v<Geo, LongSegGeo>;
    using U = std::conditional_t<sizeof(KeyT) == 8, uint64_t, uint32_t>;
    const KeyT ca = static_cast<KeyT>(codec.a), cb = static_cast<KeyT>(codec.b), cd = static_cast<KeyT>(codec.d);
    const bool enc = codec.flags & kCodecEncodeOnLoad;
    __shared__ uint32_t s_w[kLongWarps], s_na;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lt = lanemask_lt();
    const uint64_t tiles = geo.tiles();
    for (uint64_t g = blockIdx.x; g < tiles; g += gridDim.x) {
        const auto x = geo.tile(g);
        const KeyT* tile = in + x.lo + x.t0;
        const uint32_t tpr = select_tpr(geo, x);
        uint32_t na = nr;
        if constexpr (SEG) {
            if (threadIdx.x < 32) {
                const uint32_t a = select_active(geo, x.r, nr, seg_ranks);
                if (threadIdx.x == 0) s_na = a;
            }
            __syncthreads();
            na = s_na;
        }
        for (uint32_t i = 0; i < na; ++i) {
            const uint32_t* s = cnt + select_cnt_base(geo, x, nr, i);  // the scan ran over the row's ranks one after another
            const uint32_t b0 = s[0], lo = s[x.t] - b0, hi = x.t + 1 < tpr ? s[x.t + 1] - b0 : 0xffffffffu;
            const SelectState ss = st[x.r * nr + i];
            uint32_t o;
            if constexpr (SEG) o = seg_ranks[select_obase(geo, x.r, nr) + i] - ss.taken;
            else o = select_rank_of(*ranks, i) - ss.taken;
            if (o < lo || o >= hi) continue;
            const U v = static_cast<U>(ss.v);
            const uint32_t want = o - lo;
            uint32_t run = 0;
            for (uint32_t c0 = 0; c0 < x.len; c0 += kLongThreads) {
                const uint32_t j = c0 + threadIdx.x;
                KeyT k = j < x.len ? tile[j] : static_cast<KeyT>(0);
                const bool eq = j < x.len && static_cast<U>(enc ? codec_encode<KeyT>(k, ca, cb, cd) : k) == v;
                const uint32_t b = __ballot_sync(0xffffffffu, eq);
                if (lane == 0) s_w[warp] = __popc(b);
                __syncthreads();
                uint32_t pre = 0, total = 0;
#pragma unroll
                for (int w = 0; w < kLongWarps; ++w) { const uint32_t y = s_w[w]; pre += static_cast<uint32_t>(w) < warp ? y : 0u; total += y; }
                __syncthreads();  // s_w is reused by the next chunk
                if (eq && run + pre + __popc(b & lt) == want) idx_out[select_obase(geo, x.r, nr) + i] = x.t0 + j;
                run += total;
                if (run > want) break;
            }
        }
        if constexpr (SEG) __syncthreads();  // s_na is rewritten for the next tile
    }
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
select_locate_kernel(const KeyT* __restrict__ in, uint32_t* __restrict__ idx_out, uint64_t num_rows, uint32_t row_len, uint32_t tpr,
                     const SelectState* __restrict__ st, const uint32_t* __restrict__ cnt, SelectRanks ranks, KeyCodec codec)
{
    select_locate_body<KeyT>(LongRowGeo{num_rows, row_len, tpr, 0, 0}, in, idx_out, ranks.count, st, cnt, &ranks, codec, nullptr);
}

template <typename KeyT>
__global__ void __launch_bounds__(kLongThreads)
select_segments_locate_kernel(const KeyT* __restrict__ in, uint32_t* __restrict__ idx_out, LongSegGeo geo,
                              const uint32_t* __restrict__ seg_ranks, uint32_t nr, const SelectState* __restrict__ st,
                              const uint32_t* __restrict__ cnt, KeyCodec codec)
{
    select_locate_body<KeyT>(geo, in, idx_out, nr, st, cnt, nullptr, codec, seg_ranks);
}

SelectLayout select_layout(uint64_t num_rows, uint32_t row_len, uint32_t num_ranks, bool positions)
{
    static_assert(sizeof(SortPlan) <= 16 * sizeof(uint32_t) && sizeof(SelectState) == 4 * sizeof(uint32_t), "the layout's words");
    auto whole = [](uint64_t words) { return (words + 3) / 4 * 4; };
    SelectLayout l;
    l.tpr = static_cast<uint32_t>((static_cast<uint64_t>(row_len) + kLongRowTile - 1) / kLongRowTile);
    l.cpr = static_cast<uint32_t>((static_cast<uint64_t>(num_ranks) * l.tpr + kLongChunk - 1) / kLongChunk);
    l.st = 16;  // words 0 .. 15: a zeroed SortPlan, with which the long rows' scan kernels skip nothing
    l.tot = l.st + num_rows * num_ranks * 4;
    l.zeroed = whole(l.tot + num_rows * num_ranks * kRadix);
    l.cnt = l.zeroed;
    l.csum = positions ? whole(l.cnt + num_rows * num_ranks * l.tpr) : l.cnt;
    l.words = positions && l.cpr > 1 ? whole(l.csum + num_rows * l.cpr) : l.csum;
    return l;
}

cudaError_t launch_select_long_rows(const void* keys_in, void* values_out, uint32_t* indices, uint64_t num_rows, uint32_t row_len,
                                    const SelectRanks& ranks, int key_bytes, const KeyCodec* codec_in, uint32_t* scratch, int sm_count,
                                    cudaStream_t stream)
{
    if (num_rows == 0 || row_len < 2 || ranks.count == 0 || ranks.count > kMaxSelectRanks) return cudaErrorInvalidValue;
    const uint32_t nr = ranks.count;
    const SelectLayout l = select_layout(num_rows, row_len, nr, indices != nullptr);
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    cudaError_t e = cudaMemsetAsync(scratch, 0, l.zeroed * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    const SortPlan* none_skipped = reinterpret_cast<const SortPlan*>(scratch);
    SelectState* st = reinterpret_cast<SelectState*>(scratch + l.st);
    uint32_t* tot = scratch + l.tot;
    uint32_t* cnt = scratch + l.cnt;
    uint32_t* csum = l.cpr > 1 ? scratch + l.csum : nullptr;
    const uint64_t tiles = num_rows * l.tpr;
    return with_key_type(TopkKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        cudaError_t le = cudaSuccess;
        for (uint32_t t = 0; le == cudaSuccess && t < sizeof(KeyT); ++t) {
            le = launch_resident<select_count_kernel<KeyT>, kLongThreads, 0>(tiles, sm_count, stream, in, num_rows, row_len, l.tpr, nr, t,
                                                                             static_cast<const SelectState*>(st), tot, codec);
            if (le == cudaSuccess)
                le = launch_resident<select_pick_kernel<KeyT>, kRadix, 0>(num_rows, sm_count, stream, num_rows, t, st, tot,
                                                                          static_cast<KeyT*>(values_out), ranks, codec);
        }
        if (le != cudaSuccess || !indices) return le;
        le = launch_resident<select_eq_count_kernel<KeyT>, kLongThreads, 0>(tiles, sm_count, stream, in, num_rows, row_len, l.tpr, nr,
                                                                            static_cast<const SelectState*>(st), cnt, codec);
        if (le != cudaSuccess) return le;
        // per row, the exclusive scan of its nr * tpr counts [rank][tile]
        const uint64_t row_counts = static_cast<uint64_t>(nr) * l.tpr;
        const unsigned scan_grid = capped_grid(num_rows * l.cpr, 1, static_cast<uint64_t>(sm_count) * 4);
        if (csum) {
            long_rows_chunk_sum_kernel<<<scan_grid, kLongThreads, 0, stream>>>(none_skipped, 0, cnt, csum, num_rows, row_counts, l.cpr);
            long_rows_chunk_scan_kernel<<<capped_grid(num_rows, 1, static_cast<uint64_t>(sm_count) * 4), kLongThreads, 0, stream>>>(
                none_skipped, 0, csum, num_rows, l.cpr);
        }
        long_rows_scan_kernel<<<scan_grid, kLongThreads, 0, stream>>>(none_skipped, 0, cnt, csum, num_rows, row_counts, l.cpr);
        if ((le = cudaGetLastError()) != cudaSuccess) return le;
        return launch_resident<select_locate_kernel<KeyT>, kLongThreads, 0>(tiles, sm_count, stream, in, indices, num_rows, row_len, l.tpr,
                                                                            static_cast<const SelectState*>(st),
                                                                            static_cast<const uint32_t*>(cnt), ranks, codec);
    });
}

// =====================================================================================================
// Segment select (osb200_select_segments, DESIGN §4.20): the row select for ragged segments given by offsets, each with its
// own ranks seg_ranks[s * nr .. s * nr + nr) (device memory, non-decreasing).  Segment s's result is row s of [num_segments,
// nr] outputs; a column whose rank takes no part (select_ranks_active: at or past the length, or the row's ranks decrease),
// and every column of an empty or invalid segment, is padding.
//   * select_segment_bin_kernel (segment_bin_body, SEL) lists every segment: up to warp_max keys (or fewer than two), and the
//     empty and invalid ones, on the warp list; with LONG segments of long_min or more keys on the long list; the others on
//     the block list, by the segment sort's two block classes.
//   * select_segment_warp_kernel (warp_sort_run, RCOLS) and select_segment_block_kernel (segment_sort_body, LIST and RCOLS)
//     sort each segment in shared memory and store only its columns.
//   * the long list: long_segments_map_kernel's tile map, then the split path's bodies over it (LongSegGeo), and with
//     positions the long segments' scan bodies over each entry's [rank][tile] counts (SelectSegScanGeo).  Should the map
//     not fit its bounds (only offsets that make valid segments overlap can do that), select_segment_unmapped_kernel pads
//     every long segment instead.
// =====================================================================================================
__global__ void __launch_bounds__(256)
select_segment_bin_kernel(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n, uint32_t max_len,
                          uint32_t warp_max, uint32_t* __restrict__ list, unsigned long long* __restrict__ counts)
{
    segment_bin_body<uint32_t, false, false, true>(off, num_segments, n, max_len, list, counts, nullptr, nullptr, nullptr, warp_max);
}

__global__ void __launch_bounds__(256)
select_long_segment_bin_kernel(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n, uint32_t max_len,
                               uint32_t warp_max, uint32_t* __restrict__ list, unsigned long long* __restrict__ counts,
                               uint32_t long_min, uint32_t* __restrict__ long_list, uint64_t long_cap)
{
    segment_bin_body<uint32_t, false, true, true>(off, num_segments, n, max_len, list, counts, nullptr, nullptr, nullptr, warp_max,
                                                  long_min, long_list, long_cap);
}

template <typename KeyT, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(kRowWarps * 32)
select_segment_warp_kernel(const KeyT* in, KeyT* out, uint32_t* __restrict__ idx_out, uint64_t n, uint32_t max_len,
                           const unsigned long long* __restrict__ off, const uint32_t* __restrict__ list,
                           const unsigned long long* __restrict__ counts, const uint32_t* __restrict__ seg_ranks, uint32_t nr,
                           KeyCodec codec)
{
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int warp = threadIdx.x >> 5;
    unsigned char* wsm = s_raw + warp * sizeof(RowWarpSmem<KeyT, 8, INDICES>);  // every K's layout starts with the same hist
    const WarpSortCtx<KeyT> x = warp_sort_ctx<KeyT>(reinterpret_cast<uint32_t*>(wsm), codec);
    const uint64_t count = counts[kSegCountWarp];
    for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * kRowWarps + warp; i < count; i += static_cast<uint64_t>(gridDim.x) * kRowWarps) {
        const uint32_t s = list[i];
        const unsigned long long lo = off[s], hi = off[s + 1];
        // offsets that decrease, pass n or exceed max_len: the binning kernel listed it here as empty
        const uint32_t len = lo <= hi && hi <= n && hi - lo <= max_len && hi - lo <= kRowWarpMaxLen ? static_cast<uint32_t>(hi - lo) : 0u;
        const uint64_t obase = static_cast<uint64_t>(s) * nr;
        const uint32_t* rk = seg_ranks + obase;
        if (len <= 32)
            warp_sort_run<KeyT, 1, RANK_MODE, INDICES, false, false, false, true>(*reinterpret_cast<RowWarpSmem<KeyT, 1, INDICES>*>(wsm), x,
                                                                                  in, out, idx_out, lo, len, nullptr, obase, 0u, nullptr, rk, nr);
        else if (len <= 64)
            warp_sort_run<KeyT, 2, RANK_MODE, INDICES, false, false, false, true>(*reinterpret_cast<RowWarpSmem<KeyT, 2, INDICES>*>(wsm), x,
                                                                                  in, out, idx_out, lo, len, nullptr, obase, 0u, nullptr, rk, nr);
        else if (len <= 128)
            warp_sort_run<KeyT, 4, RANK_MODE, INDICES, false, false, false, true>(*reinterpret_cast<RowWarpSmem<KeyT, 4, INDICES>*>(wsm), x,
                                                                                  in, out, idx_out, lo, len, nullptr, obase, 0u, nullptr, rk, nr);
        else
            warp_sort_run<KeyT, 8, RANK_MODE, INDICES, false, false, false, true>(*reinterpret_cast<RowWarpSmem<KeyT, 8, INDICES>*>(wsm), x,
                                                                                  in, out, idx_out, lo, len, nullptr, obase, 0u, nullptr, rk, nr);
    }
}

template <typename KeyT, int K, int WARPS, int RANK_MODE, bool INDICES>
__global__ void __launch_bounds__(WARPS * 32, 1)
select_segment_block_kernel(const KeyT* __restrict__ in, KeyT* out, uint32_t* idx_out, const unsigned long long* __restrict__ off,
                            uint64_t num_segments, uint32_t max_len, KeyCodec codec, const uint32_t* __restrict__ list,
                            const unsigned long long* __restrict__ counts, const uint32_t* __restrict__ seg_ranks, uint32_t nr)
{
    segment_sort_body<KeyT, INDICES, K, WARPS, RANK_MODE, INDICES, false, true, false, false, true>(
        out, idx_out, off, num_segments, 0, max_len, 0u, sizeof(KeyT), 8u, codec, in, list, counts, 0, 0u, nullptr, seg_ranks, nr);
}

// the block classes' geometries: 2,048 keys, and the row sort's capacity
template <typename KeyT, int SIZE, bool INDICES>
struct SelectSegShape {
    using Key = KeyT;
    static constexpr bool indices = INDICES, has_hot = false;
    using G = SegGeomN<KeyT, SIZE>;
    using S = SegSmem<KeyT, INDICES, G::K, G::WARPS>;
    static constexpr uint32_t T = S::T;
    static constexpr size_t smem = sizeof(S);
    template <int RANK_MODE, bool HOT = false>
    static constexpr auto kernel() { return select_segment_block_kernel<KeyT, G::K, G::WARPS, RANK_MODE, INDICES>; }
};
using SelectSegShapes = TypeList<
    SelectSegShape<uint16_t, 1, false>, SelectSegShape<uint16_t, 2, false>, SelectSegShape<uint16_t, 1, true>, SelectSegShape<uint16_t, 2, true>,
    SelectSegShape<uint32_t, 1, false>, SelectSegShape<uint32_t, 2, false>, SelectSegShape<uint32_t, 1, true>, SelectSegShape<uint32_t, 2, true>,
    SelectSegShape<uint64_t, 1, false>, SelectSegShape<uint64_t, 2, false>, SelectSegShape<uint64_t, 1, true>, SelectSegShape<uint64_t, 2, true>>;

// The long segments' equal-key counts for the scan bodies: entry j's nr * tiles counts [rank][tile] from nr * tfirst[j], cut
// into chunks of 16 tiles' counts per rank -- as many as long_segments_map_kernel gives the entry (ceil(tiles / 16), from
// cfirst[j]), so its chunk map serves here too.
struct SelectSegScanGeo {
    LongSegGeo seg;
    uint32_t nr;
    using Chunk = LongSegGeo::Chunk;
    using Group = LongSegGeo::Group;
    __device__ __forceinline__ uint64_t chunks() const { return seg.chunks(); }
    __device__ __forceinline__ Chunk chunk(uint64_t g) const
    {
        const uint32_t j = cta_find(seg.cfirst, seg.listed(), g), f = seg.tfirst[j];
        const uint64_t w = static_cast<uint64_t>(kLongChunk / kRadix) * nr, c0 = (g - seg.cfirst[j]) * w;
        const uint64_t rc = static_cast<uint64_t>(seg.tfirst[j + 1] - f) * nr;
        return {static_cast<uint64_t>(f) * nr + c0, 0, rc - c0 < w ? rc - c0 : w};
    }
    __device__ __forceinline__ uint64_t groups() const { return seg.groups(); }
    __device__ __forceinline__ Group group(uint64_t j) const { return seg.group(j); }
};
static_assert(kLongChunk % kRadix == 0, "a chunk of the tile map is whole tiles");

__global__ void __launch_bounds__(kLongThreads)
select_segments_chunk_sum_kernel(const SortPlan* __restrict__ plan, uint32_t* cnt, uint32_t* __restrict__ csum, SelectSegScanGeo geo)
{
    long_chunk_sum_body(geo, plan, 0u, cnt, csum);
}

__global__ void __launch_bounds__(kLongThreads)
select_segments_chunk_scan_kernel(const SortPlan* __restrict__ plan, uint32_t* csum, SelectSegScanGeo geo)
{
    long_chunk_scan_body(geo, plan, 0u, csum);
}

__global__ void __launch_bounds__(kLongThreads)
select_segments_scan_kernel(const SortPlan* __restrict__ plan, uint32_t* cnt, const uint32_t* __restrict__ csum, SelectSegScanGeo geo)
{
    long_scan_body(geo, plan, 0u, cnt, csum);
}

// When the tile map did not fit (counts[kSegCountLong] == 0), every segment the binning kernel sent to the long list is padding.
template <typename KeyT>
__global__ void __launch_bounds__(256)
select_segment_unmapped_kernel(const unsigned long long* __restrict__ off, uint64_t num_segments, uint64_t n, uint32_t max_len,
                               uint32_t long_min, const unsigned long long* __restrict__ counts, KeyT* out, uint32_t* idx_out,
                               uint32_t nr, KeyCodec codec)
{
    if (counts[kSegCountLong] != 0) return;
    const KeyT ones = static_cast<KeyT>(~static_cast<KeyT>(0));
    const KeyT pad = codec.flags & kCodecDecodeOnStore
                         ? codec_decode<KeyT>(ones, static_cast<KeyT>(codec.a), static_cast<KeyT>(codec.b), static_cast<KeyT>(codec.d))
                         : ones;
    for (uint64_t s = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x; s < num_segments;
         s += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
        const unsigned long long lo = off[s], hi = off[s + 1];
        if (!(lo <= hi && hi <= n && hi - lo <= max_len && hi - lo >= long_min)) continue;
        for (uint32_t i = 0; i < nr; ++i) {
            out[s * nr + i] = pad;
            if (idx_out) idx_out[s * nr + i] = 0xFFFFFFFFu;
        }
    }
}

SelectSegLayout select_segments_layout(uint64_t n, uint64_t num_segments, uint32_t long_min, uint32_t num_ranks, bool positions)
{
    auto whole = [](uint64_t words) { return (words + 3) / 4 * 4; };  // every array 16-byte aligned
    SelectSegLayout l;
    l.list_cap = n / long_min < num_segments ? n / long_min : num_segments;
    l.tile_cap = (n + kLongRowTile - 1) / kLongRowTile + l.list_cap;
    l.chunk_cap = (l.tile_cap * kRadix + kLongChunk - 1) / kLongChunk + l.list_cap;
    l.st = 16;  // words 0 .. 15: a zeroed SortPlan, with which the scan bodies skip nothing
    l.tot = l.st + l.list_cap * num_ranks * 4;
    l.zeroed = whole(l.tot + l.list_cap * num_ranks * kRadix);
    l.list = l.zeroed;
    l.tfirst = l.list + whole(l.list_cap);
    l.cfirst = l.tfirst + whole(l.list_cap + 1);
    l.cnt = l.cfirst + whole(l.list_cap + 1);
    l.csum = positions ? l.cnt + whole(l.tile_cap * num_ranks) : l.cnt;
    l.words = positions ? l.csum + whole(l.chunk_cap) : l.csum;
    return l;
}

cudaError_t launch_select_segments(const void* keys_in, void* values_out, uint32_t* indices, uint64_t n, const unsigned long long* off,
                                   uint64_t num_segments, uint32_t max_len, const uint32_t* seg_ranks, uint32_t nr, int key_bytes,
                                   const KeyCodec* codec_in, int rank_mode, bool block_only, uint32_t long_min, int sm_count,
                                   uint32_t* list, unsigned long long* counts, uint32_t* scratch, cudaStream_t stream)
{
    if (num_segments == 0 || nr == 0 || nr > kMaxSelectRanks || (long_min && (long_min < 2 || !scratch))) return cudaErrorInvalidValue;
    if (!long_min && max_len > row_sort_capacity(key_bytes)) return cudaErrorInvalidValue;
    const bool lng = long_min && max_len >= long_min && n >= long_min;  // (then the long list has room for one segment or more)
    const KeyCodec codec = codec_in ? *codec_in : KeyCodec();
    const SelectSegLayout l = select_segments_layout(n, num_segments, lng ? long_min : 1u, nr, indices != nullptr);
    cudaError_t e = cudaMemsetAsync(counts, 0, (lng ? kLongSegCounts : kSegCounts) * sizeof(unsigned long long), stream);
    if (e == cudaSuccess && lng) e = cudaMemsetAsync(scratch, 0, l.zeroed * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    const uint32_t warp_max = block_only ? 0u : kRowWarpMaxLen;
    const unsigned bin_grid = capped_grid(num_segments, 256, static_cast<uint64_t>(sm_count) * 8);
    if (lng)
        select_long_segment_bin_kernel<<<bin_grid, 256, 0, stream>>>(off, num_segments, n, max_len, warp_max, list, counts, long_min,
                                                                     scratch + l.list, l.list_cap);
    else
        select_segment_bin_kernel<<<bin_grid, 256, 0, stream>>>(off, num_segments, n, max_len, warp_max, list, counts);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // the classes: every segment the long list does not take
    const uint32_t class_max = lng ? long_min - 1 : max_len;
    e = with_key_type(TopkKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        return with_rank_mode(rank_mode, [&](auto r) {
            constexpr int R = decltype(r)::value;
            auto go = [&](auto ind) {  // each warp's staging area is sized for 8 keys per lane
                constexpr bool I = decltype(ind)::value;
                return launch_resident<select_segment_warp_kernel<KeyT, R, I>, kRowWarps * 32, kRowWarpSmemBytes<KeyT, 8, I>>(
                    kAllResident, sm_count, stream, static_cast<const KeyT*>(keys_in), static_cast<KeyT*>(values_out), indices, n,
                    max_len, off, list, counts, seg_ranks, nr, codec);
            };
            return indices ? go(std::true_type{}) : go(std::false_type{});
        });
    });
    for (int cls = 1; e == cudaSuccess && cls <= 2; ++cls) {
        if (class_max < 2 || class_max <= (cls == 1 ? warp_max : kSegBlock1Max)) break;
        e = find_type(
            SelectSegShapes{},
            [&](auto s) {
                using S = decltype(s);
                return key_bytes == static_cast<int>(sizeof(typename S::Key)) && S::indices == (indices != nullptr) &&
                       (S::T == kSegBlock1Max) == (cls == 1);
            },
            [&](auto s) {
                using S = decltype(s);
                using KeyT = typename S::Key;
                return with_rank_mode(rank_mode, [&](auto r) {
                    return launch_resident<S::template kernel<decltype(r)::value>(), S::S::THREADS, S::smem>(
                        kAllResident, sm_count, stream, static_cast<const KeyT*>(keys_in), static_cast<KeyT*>(values_out), indices,
                        off, num_segments, class_max, codec, list, counts, seg_ranks, nr);
                });
            });
    }
    if (e != cudaSuccess || !lng) return e;
    // the long list: its tile map, then the split path over its tiles
    const SortPlan* none_skipped = reinterpret_cast<const SortPlan*>(scratch);
    SelectState* st = reinterpret_cast<SelectState*>(scratch + l.st);
    uint32_t* tot = scratch + l.tot;
    uint32_t* cnt = scratch + l.cnt;
    uint32_t* csum = max_len > kLongChunk / kRadix * kLongRowTile ? scratch + l.csum : nullptr;  // some segment has 2+ chunks
    const LongSegGeo geo{off, scratch + l.list, scratch + l.tfirst, scratch + l.cfirst, counts};
    long_segments_map_kernel<<<1, kLongThreads, 0, stream>>>(off, scratch + l.list, scratch + l.tfirst, scratch + l.cfirst, counts,
                                                             l.list_cap, l.tile_cap, l.chunk_cap);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return with_key_type(TopkKeys{}, key_bytes, [&](auto kt) {
        using KeyT = decltype(kt);
        const KeyT* in = static_cast<const KeyT*>(keys_in);
        KeyT* out = static_cast<KeyT*>(values_out);
        select_segment_unmapped_kernel<KeyT><<<bin_grid, 256, 0, stream>>>(off, num_segments, n, max_len, long_min, counts, out, indices, nr,
                                                                          codec);
        cudaError_t le = cudaGetLastError();
        for (uint32_t t = 0; le == cudaSuccess && t < sizeof(KeyT); ++t) {
            le = launch_resident<select_segments_count_kernel<KeyT>, kLongThreads, 0>(l.tile_cap, sm_count, stream, in, geo, seg_ranks, nr,
                                                                                      t, static_cast<const SelectState*>(st), tot, codec);
            if (le == cudaSuccess)
                le = launch_resident<select_segments_pick_kernel<KeyT>, kRadix, 0>(l.list_cap, sm_count, stream, geo, seg_ranks, nr, t, st,
                                                                                   tot, out, indices, codec);
        }
        if (le != cudaSuccess || !indices) return le;
        le = launch_resident<select_segments_eq_count_kernel<KeyT>, kLongThreads, 0>(l.tile_cap, sm_count, stream, in, geo, seg_ranks, nr,
                                                                                     static_cast<const SelectState*>(st), cnt, codec);
        if (le != cudaSuccess) return le;
        // per list entry, the exclusive scan of its nr * tiles counts [rank][tile]
        const SelectSegScanGeo sg{geo, nr};
        const unsigned scan_grid = capped_grid(l.chunk_cap, 1, static_cast<uint64_t>(sm_count) * 4);
        if (csum) {
            select_segments_chunk_sum_kernel<<<scan_grid, kLongThreads, 0, stream>>>(none_skipped, cnt, csum, sg);
            select_segments_chunk_scan_kernel<<<capped_grid(l.list_cap, 1, static_cast<uint64_t>(sm_count) * 4), kLongThreads, 0, stream>>>(
                none_skipped, csum, sg);
        }
        select_segments_scan_kernel<<<scan_grid, kLongThreads, 0, stream>>>(none_skipped, cnt, csum, sg);
        if ((le = cudaGetLastError()) != cudaSuccess) return le;
        return launch_resident<select_segments_locate_kernel<KeyT>, kLongThreads, 0>(l.tile_cap, sm_count, stream, in, indices, geo,
                                                                                     seg_ranks, nr, static_cast<const SelectState*>(st),
                                                                                     static_cast<const uint32_t*>(cnt), codec);
    });
}

cudaError_t configure_kernels()
{
    cudaError_t e = for_each_type(HistKeys{}, [](auto k) {
        using KeyT = decltype(k);
        return set_smem(global_histogram_kernel<KeyT>, hist_smem_bytes<KeyT>());
    });
    if (e == cudaSuccess) e = for_each_type(HistBitsKeys{}, [](auto k) {
        using KeyT = decltype(k);
        const cudaError_t m = set_smem(global_histogram_kernel<KeyT, true>, hist_smem_bytes<KeyT>());
        return m != cudaSuccess ? m : set_smem(global_histogram_bits_kernel<KeyT>, hist_smem_bytes<KeyT>());
    });
    auto shape = [](auto s) { return configure_shape(s); };
    if (e == cudaSuccess) e = for_each_type(DefaultPassShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(RingShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(TileShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(SegShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(RowShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(ListShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(TopkSortShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(TopkKeys{}, [](auto k) {
        using KeyT = decltype(k);
        const cudaError_t m = set_smem(topk_select_kernel<KeyT>, sizeof(TopkSmem<KeyT>));
        return m != cudaSuccess ? m : set_smem(topk_segment_select_kernel<KeyT>, sizeof(TopkSmem<KeyT>));
    });
    if (e == cudaSuccess) e = for_each_type(TopkSortShapes{}, [](auto s) {
        using Sh = decltype(s);
        const cudaError_t m = set_smem(Sh::template list_kernel<kRankAtomic>(), Sh::smem);
        return m != cudaSuccess ? m : set_smem(Sh::template list_kernel<kRankBallot>(), Sh::smem);
    });
    if (e == cudaSuccess) e = set_smem(fused_kernel<kRankAtomic>(), FusedShape::smem);
    if (e == cudaSuccess) e = set_smem(fused_kernel<kRankBallot>(), FusedShape::smem);
    if (e == cudaSuccess) e = for_each_type(LongRowKeys{}, [](auto k) {
        using KeyT = decltype(k);
        cudaError_t m = set_smem(long_rows_scatter_kernel<KeyT, kRankAtomic, false>, sizeof(LongRowsSmem<KeyT, false>));
        if (m == cudaSuccess) m = set_smem(long_rows_scatter_kernel<KeyT, kRankBallot, false>, sizeof(LongRowsSmem<KeyT, false>));
        if (m == cudaSuccess) m = set_smem(long_rows_scatter_kernel<KeyT, kRankAtomic, true>, sizeof(LongRowsSmem<KeyT, true>));
        return m != cudaSuccess ? m : set_smem(long_rows_scatter_kernel<KeyT, kRankBallot, true>, sizeof(LongRowsSmem<KeyT, true>));
    });
    if (e == cudaSuccess) e = for_each_type(LongRowKeys{}, [](auto k) {
        using KeyT = decltype(k);
        cudaError_t m = set_smem(long_segments_scatter_kernel<KeyT, kRankAtomic, false>, sizeof(LongRowsSmem<KeyT, false>));
        if (m == cudaSuccess) m = set_smem(long_segments_scatter_kernel<KeyT, kRankBallot, false>, sizeof(LongRowsSmem<KeyT, false>));
        if (m == cudaSuccess) m = set_smem(long_segments_scatter_kernel<KeyT, kRankAtomic, true>, sizeof(LongRowsSmem<KeyT, true>));
        return m != cudaSuccess ? m : set_smem(long_segments_scatter_kernel<KeyT, kRankBallot, true>, sizeof(LongRowsSmem<KeyT, true>));
    });
    if (e == cudaSuccess) e = for_each_type(TopkKeys{}, [](auto k) {
        using KeyT = decltype(k);
        cudaError_t m = set_smem(topk_long_finish_kernel<KeyT>, sizeof(TopkSmem<KeyT>));
        if (m == cudaSuccess) m = set_smem(topk_long_sort_scatter_kernel<KeyT, kRankAtomic>, sizeof(LongRowsSmem<KeyT, true>));
        return m != cudaSuccess ? m : set_smem(topk_long_sort_scatter_kernel<KeyT, kRankBallot>, sizeof(LongRowsSmem<KeyT, true>));
    });
    if (e == cudaSuccess) e = for_each_type(SelectShapes{}, shape);
    if (e == cudaSuccess) e = for_each_type(SelectSegShapes{}, shape);
    return e;
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
    return with_key_type(TypeList<uint32_t, uint64_t>{}, key_bytes, [&](auto k) {
        using KeyT = decltype(k);
        validate_kernel<KeyT><<<static_cast<unsigned>(sm_count) * 8, 256, 0, stream>>>(static_cast<const KeyT*>(keys), n, err_count);
        return cudaGetLastError();
    });
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
