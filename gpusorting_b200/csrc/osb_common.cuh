// osb_common.cuh -- constants, tile-descriptor format and PTX helpers shared by the sm_90a kernels.
//
// Domain vocabulary follows the reference (b0nes164/GPUSorting, GPUSortingCUDA/Sort/OneSweep.cu):
// digit place, partition tile, tile reduction / inclusive prefix, chained scan with decoupled lookback.
#pragma once
#include <cstdint>
#include <type_traits>
#include <cuda_runtime.h>

namespace osb {

constexpr int kRadix = 256;      // bins per digit place          (reference: RADIX, OneSweep.cu:17)
constexpr int kRadixLog = 8;     // bits per digit                (reference: RADIX_LOG, OneSweep.cu:19)

// ---- chained-scan tile descriptor -------------------------------------------------------------------
// One 64-bit word per (tile, digit):  [63:40] epoch | [39:2] value | [1:0] flag.
// The reference packs {value:30, flag:2} into 32 bits (OneSweep.cu:39-42), which caps n at 2^30 and
// forces a memset of every descriptor before every sort (OneSweepDispatcher.cuh:301-309).  Here the value
// field is 38 bits (n <= 2^38 per GPU) and the epoch field makes stale words from earlier passes / sorts
// read as NOT_READY, so descriptors are not cleared between eager sorts.  (A graph replays the epochs of its capture, so
// a captured sort clears its descriptors before and after its passes: osb_host.cu, is_capturing.)
constexpr uint64_t kFlagNotReady = 0;   // reference: FLAG_NOT_READY
constexpr uint64_t kFlagReduction = 1;  // reference: FLAG_REDUCTION (tile-local digit count published)
constexpr uint64_t kFlagInclusive = 2;  // reference: FLAG_INCLUSIVE (prefix over tiles 0..p published)
constexpr uint64_t kFlagMask = 3;
constexpr int kValueBits = 38;
constexpr int kEpochShift = 40;
constexpr uint32_t kEpochMax = (1u << 24) - 1;

__host__ __device__ __forceinline__ uint64_t desc_pack(uint32_t epoch, uint64_t flag, uint64_t value)
{
    return (static_cast<uint64_t>(epoch) << kEpochShift) | ((value & ((1ull << kValueBits) - 1)) << 2) | flag;
}
__host__ __device__ __forceinline__ uint64_t desc_value(uint64_t d) { return (d >> 2) & ((1ull << kValueBits) - 1); }
__host__ __device__ __forceinline__ uint32_t desc_epoch(uint64_t d) { return static_cast<uint32_t>(d >> kEpochShift); }

// ---- PTX helpers ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lane_id() { uint32_t v; asm("mov.u32 %0, %%laneid;" : "=r"(v)); return v; }
__device__ __forceinline__ uint32_t lanemask_lt() { uint32_t v; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(v)); return v; }

// Descriptors carry flag and value in one naturally-atomic 64-bit word, so relaxed GPU-scope accesses are
// sufficient (no separate payload to order against); .gpu scope keeps them out of the non-coherent L1.
__device__ __forceinline__ uint64_t ld_relaxed_gpu_u64(const uint64_t* p)
{
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u64(uint64_t* p, uint64_t v)
{
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Streaming loads/stores: every key is read once and written once per pass; do not let them displace the
// descriptor words (which are re-read by successor tiles) from L1/L2 earlier than necessary.
// ld_stream (the DigitBinningPass's tile loads) caches in L2 only (ld.global.cg) rather than evict-first (ld.global.cs):
// the 2^30 uint32 keys sort went from 61.0-61.3 to 62.2-62.6 Gkeys/s on an H100 80GB HBM3 at a 400 W power limit
// (max SM clock 1,980 MHz; three alternating bench.py runs each).  Why it helps (L1 bypass or L2 eviction priority) was
// not isolated.
template <typename T> __device__ __forceinline__ T ld_stream(const T* p) { return __ldcg(p); }
template <typename T> __device__ __forceinline__ void st_stream(T* p, T v) { __stcs(p, v); }
// Scatter stores of the DigitBinningPass (`digit_binning_wide_kernel`): plain write-back stores, NOT evict-first.  A
// tile writes each digit as a run of ~64 keys whose ends share 32-byte sectors with the runs of the tiles next to it,
// written by other CTAs at about the same time.  Write-back lets L2 hold such a sector until both halves have arrived;
// with evict-first stores it leaves L2 partly written.  On an H100 at a 400 W power limit this made the pass 11 % faster
// (DESIGN §4.2).
// (A plain C++ store, the form that was measured; `__stwb` compiles to a volatile asm store instead.)
template <typename T> __device__ __forceinline__ void st_scatter(T* p, T v) { *p = v; }

// ---- typed keys: order-preserving bijection onto unsigned keys -----------------------------------------
// The reference's CUDA path sorts uint32 only; its HLSL path sorts int/float keys by transforming their bits on the way
// in and out (GPUSortingD3D12/Shaders/SortCommon.hlsl:134-154: FloatToUint / IntToUint and inverses) and reverses the
// index on the last pass for descending order (:594-656, which reverses ties).  Here: encode(k) = k ^ m(k) ^ D with
// m(k) = (sar(k) & A) | B; (A,B) = (0,0) unsigned, (0,SIGN) signed, (ALL,SIGN) IEEE float; D = ALL for descending
// (complement: equal keys keep their input order, i.e. descending sorts are STABLE, unlike the reference's).
struct KeyCodec {
    unsigned long long a = 0, b = 0, d = 0;
    uint32_t flags = 0;  // bit 0: encode keys right after loading; bit 1: decode keys right before storing
};
constexpr uint32_t kCodecEncodeOnLoad = 1u, kCodecDecodeOnStore = 2u;
constexpr uint32_t kCodecFromPlan = 4u;  // encode/decode flags of a pass are taken from the device plan (first/last executed pass)

template <typename KeyT> __device__ __forceinline__ KeyT codec_encode(KeyT k, KeyT a, KeyT b, KeyT d)
{
    using S = typename std::make_signed<KeyT>::type;
    const KeyT sar = static_cast<KeyT>(static_cast<S>(k) >> (sizeof(KeyT) * 8 - 1));
    return k ^ (((sar & a) | b) ^ d);
}
template <typename KeyT> __device__ __forceinline__ KeyT codec_decode(KeyT e, KeyT a, KeyT b, KeyT d)
{
    using S = typename std::make_signed<KeyT>::type;
    e ^= d;
    const KeyT sar = static_cast<KeyT>(static_cast<S>(e) >> (sizeof(KeyT) * 8 - 1));
    return e ^ ((~sar & a) | b);
}

template <typename KeyT> __device__ __forceinline__ uint32_t digit_of(KeyT k, uint32_t shift)
{
    return static_cast<uint32_t>(k >> shift) & (kRadix - 1);
}
// digit narrower than 8 bits (the last place of a begin_bit/end_bit sort): mask = 2^bits - 1
template <typename KeyT> __device__ __forceinline__ uint32_t digit_of(KeyT k, uint32_t shift, uint32_t mask)
{
    return static_cast<uint32_t>(k >> shift) & mask;
}

// ---- device-side launch plan -----------------------------------------------------------------------------
// Written by the scan kernel, read by every DigitBinningPass of the same sort: the host enqueues a fixed sequence of
// launches and never synchronises, yet passes whose digit is the same for ALL keys (one non-empty bin in the global
// histogram) move nothing.  Reference idea: the entropy benchmark of GPUSortingD3D12/Tests.h:383-393 shows what low-entropy
// inputs cost; skipping is this repository's answer (the reference itself always runs its 4 passes).
constexpr uint32_t kPlanHotShift = 16;  // SortPlan::skip_mask bit 16+p: pass p is "hot" (a bin holds >= n/8 keys: HOT instantiation)
struct SortPlan {
    uint32_t skip_mask;   // bit p: pass p is skipped (its CTAs exit at once); bits 16+p: hot passes
    uint32_t executed;    // number of passes that run; odd -> the result is in the alt buffers -> copy_back_kernel moves it
    uint32_t first_exec;  // first / last executed pass (typed keys: encode in the first one, decode in the last one)
    uint32_t last_exec;
};
// pass `place` reads the caller's buffers iff an even number of passes ran before it
__device__ __forceinline__ bool plan_src_is_alt(const SortPlan& pl, uint32_t place)
{
    return __popc(~pl.skip_mask & ((1u << place) - 1u)) & 1u;
}

// ---- fused first pass (whole-key u32 keys-only sorts, DESIGN §4.12) ----------------------------------------------------
// The first digit pass counts the global histogram itself and scatters digit d into a region of fixed capacity c(n) at
// d * c(n) of the alt buffer, so it needs no digit bases and no GlobalHistogram in front of it.  SortPlan::skip_mask bit
// kPlanFusedKept says its result stands; otherwise the classic GlobalHistogram, Scan and first pass run after it.
constexpr uint32_t kPlanFusedKept = 1u << 24;
// Region capacity: n/256 plus 1/32 of it plus 1,024 keys, in whole 128-byte lines (uniform keys: ~64 standard deviations of
// slack at n = 2^30, ~18 at 2^20).
__host__ __device__ constexpr uint64_t fused_region_keys(uint64_t n)
{
    const uint64_t q = (n + 255) / 256;
    return (q + q / 32 + 1024 + 31) / 32 * 32;
}
// the first executed pass after place 0 of a fused sort reads the gapped layout the fused pass left
__device__ __forceinline__ bool plan_reads_gapped(const SortPlan& pl, uint32_t place)
{
    const uint32_t later = ~pl.skip_mask & 0xfeu;
    return (pl.skip_mask & kPlanFusedKept) && later && place == static_cast<uint32_t>(__ffs(later) - 1);
}

}  // namespace osb
