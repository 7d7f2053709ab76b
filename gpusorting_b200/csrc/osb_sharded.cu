// osb_sharded.cu -- multi-GPU sharded sort: one MSD bucket-exchange pass over NVLink, then a local OneSweep.
//
// No reference equivalent (the reference is single-device, SURVEY 2.1); this is BASELINE.json's fifth config.
// One process per GPU.  Every rank holds n_local unsorted keys; after the call rank r holds the r-th contiguous
// slice of the global ascending order.
//
//   1. 256-bin histogram of the most significant digit of the local keys            (digit_histogram_kernel)
//   2. all-gather of the R histograms                                                (ncclAllGather, 2 KB per rank)
//   3. layout: top log2(R) bits split evenly, or contiguous ranges of 256 buckets      (osb200_sharded_exchange_layout,
//      balanced on the global counts; bases and offsets of both exchange modes          host)
//   4. exchange pass, two implementations:
//        fused  (default): the ordinary DigitBinningPass kernel scatters straight into the peers' receive buffers
//                through CUDA-IPC-mapped NVLink addresses -- its per-digit output bases are "virtual element indices"
//                that encode peer addresses, so ranking, chained scan and the NVLink stores are ONE kernel and the
//                keys cross HBM once (read) + NVLink once (write);
//        staged: DigitBinningPass into a local send buffer, then ncclSend/ncclRecv per peer (baseline).
//   5. local OneSweep (osb200_sort_keys_u32) on the received keys.
#include <cstring>
#include <new>
#include <vector>

#include <nccl.h>

#include "../../include/onesweep_b200.h"
#include "osb_internal.h"

namespace {

constexpr int kRadix = 256;
constexpr int kMaxWorld = 64;

inline int cuda_status(cudaError_t e) { return e == cudaSuccess ? OSB200_OK : OSB200_ERR_CUDA - static_cast<int>(e); }
#define OSB_TRY(expr)                                    \
    do {                                                 \
        cudaError_t e__ = (expr);                        \
        if (e__ != cudaSuccess) return cuda_status(e__); \
    } while (0)

// busy poll (see osb200_sharded_sort_keys_u32): returns as soon as the event has completed
inline cudaError_t spin_until(cudaEvent_t e)
{
    cudaError_t r;
    while ((r = cudaEventQuery(e)) == cudaErrorNotReady)
        for (int i = 0; i < 32; ++i) __builtin_ia32_pause();
    return r;
}
#define OSB_NCCL(expr)                                   \
    do {                                                 \
        ncclResult_t r__ = (expr);                       \
        if (r__ != ncclSuccess) return OSB200_ERR_NCCL;  \
    } while (0)

}  // namespace

struct osb200_sharded_sorter {
    int rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    uint64_t max_n_local = 0, capacity = 0;  // capacity = receive-side keys (max_n_local + slack)
    osb200_handle exch = nullptr;            // kernels/state for the exchange pass over the local input
    osb200_handle local = nullptr;           // local OneSweep over the received keys
    uint32_t* send_buf = nullptr;            // staged mode only
    uint32_t* recv_buf = nullptr;
    unsigned long long* d_hist = nullptr;      // [256] local MSD histogram
    unsigned long long* d_hist_all = nullptr;  // [world][256]
    unsigned long long* d_out_base = nullptr;  // [256] virtual element indices (fused mode)
    unsigned long long* h_hist_all = nullptr;  // pinned
    unsigned long long* h_out_base = nullptr;  // pinned
    unsigned long long* h_pass_hist = nullptr;  // pinned: the coarse histogram the exchange pass scans
    uint32_t* d_flag = nullptr;                // 1-element all-reduce used as a stream-ordered cross-GPU barrier
    void* peer_recv[kMaxWorld] = {};           // IPC-mapped receive buffers of all ranks (own = recv_buf)
    bool fused = true;
    bool force_fine = false;  // always use the 256-bucket plan (tests)
    cudaEvent_t ev[4] = {};
    cudaEvent_t sync_ev = nullptr;  // host wait for the all-gathered histograms (busy-polled)
    float last_ms[4] = {0, 0, 0, 0};
};

extern "C" {

// Host-side plan shared by every rank (pure function of the all-gathered histograms; exported for CPU tests).
//   hist_all   [world][256]  digit counts per source rank
//   dest       [256]         owner rank of every bucket: contiguous, non-decreasing, balanced on global counts
//   recv_count [world]       keys each rank ends up with
//   recv_off   [world][256]  for THIS rank as a source (`rank`): element offset inside dest[d]'s receive buffer where
//                            its keys of bucket d go.  Layout at a destination: bucket-major, source-rank-minor,
//                            i.e. exactly the globally stable order of the MSD partition.
OSB200_API int osb200_sharded_plan(const uint64_t* hist_all, int world, int rank, int32_t* dest, uint64_t* recv_count,
                                   uint64_t* recv_off)
{
    if (!hist_all || !dest || !recv_count || !recv_off || world < 1 || world > kMaxWorld || rank < 0 || rank >= world)
        return OSB200_ERR_INVALID_ARG;
    uint64_t bucket[kRadix], total = 0;
    for (int d = 0; d < kRadix; ++d) {
        bucket[d] = 0;
        for (int r = 0; r < world; ++r) bucket[d] += hist_all[r * kRadix + d];
        total += bucket[d];
    }
    // greedy contiguous split: bucket d goes to the rank whose ideal range contains the bucket's midpoint
    uint64_t before = 0;
    int prev = 0;
    for (int d = 0; d < kRadix; ++d) {
        int q = prev;
        if (total) {
            const long double mid = static_cast<long double>(before) + static_cast<long double>(bucket[d]) / 2;
            q = static_cast<int>(mid * world / static_cast<long double>(total));
            if (q >= world) q = world - 1;
            if (q < prev) q = prev;
        }
        dest[d] = q;
        prev = q;
        before += bucket[d];
    }
    for (int r = 0; r < world; ++r) recv_count[r] = 0;
    uint64_t fill[kMaxWorld] = {};  // running fill of every destination, bucket-major
    for (int d = 0; d < kRadix; ++d) {
        const int q = dest[d];
        uint64_t off = fill[q];
        for (int r = 0; r < world; ++r) {
            if (r == rank) recv_off[d] = off;
            off += hist_all[r * kRadix + d];
        }
        fill[q] = off;
    }
    for (int r = 0; r < world; ++r) recv_count[r] = fill[r];
    return OSB200_OK;
}

OSB200_API uint64_t osb200_sharded_capacity(uint64_t max_n_local, int slack_percent)
{
    if (slack_percent < 0 || slack_percent > 400) return 0;
    return max_n_local + max_n_local / 100 * static_cast<uint64_t>(slack_percent) + 4096;
}

// The whole host-side layout of one exchange (see the header), as osb200_sharded_sort_keys_u32 uses it.
//   Preferred: R = 2^k ranks and the equal-width split of the key space fits the receive buffers -> exchange on the top k
//   bits only (R bins instead of 256): runs of ~n/(tiles*R) keys (8 KB at R = 8) keep the NVLink stores full-sector (short
//   misaligned runs reach a fraction of the 128-B-aligned peer store rate, tools/microbench/p2p_store_ub.cu) and the ranking
//   atomics nearly conflict-free.  Otherwise: 256 buckets, greedy (osb200_sharded_plan).
OSB200_API int osb200_sharded_exchange_layout(const uint64_t* hist_all, int world, int rank, uint64_t capacity, int force_fine,
                                              const uint64_t* recv_addrs, uint32_t* xshift, int32_t* bins, int32_t* dest,
                                              uint64_t* recv_count, uint64_t* recv_off, uint64_t* pass_hist,
                                              uint64_t* out_base, uint64_t* send_off, uint64_t* recv_from_off)
{
    if (!hist_all || !xshift || !bins || !dest || !recv_count || !recv_off || !pass_hist || !send_off || !recv_from_off ||
        world < 1 || world > kMaxWorld || rank < 0 || rank >= world || (recv_addrs == nullptr) != (out_base == nullptr))
        return OSB200_ERR_INVALID_ARG;
    if (recv_addrs)
        for (int q = 0; q < world; ++q)
            if (recv_addrs[q] % sizeof(uint32_t)) return OSB200_ERR_INVALID_ARG;
    const int R = world;
    const uint64_t* mine = hist_all + static_cast<size_t>(rank) * kRadix;
    int k = 0;
    while ((1 << k) < R) ++k;
    const int per = kRadix >> k;  // fine buckets per coarse bin
    bool coarse = R > 1 && (1 << k) == R && !force_fine;
    if (coarse) {
        for (int q = 0; q < R; ++q) recv_count[q] = 0;
        for (int src = 0; src < R; ++src)
            for (int d = 0; d < kRadix; ++d) recv_count[d / per] += hist_all[static_cast<size_t>(src) * kRadix + d];
        for (int q = 0; q < R; ++q) coarse = coarse && recv_count[q] <= capacity;
    }
    if (coarse) {
        *xshift = 32 - k;
        *bins = R;
        for (int b = 0; b < kRadix; ++b) { dest[b] = b < R ? b : R - 1; recv_off[b] = 0; pass_hist[b] = 0; }
        // bucket-major, source-minor: this rank's keys of bin b follow those of every lower source rank
        for (int src = 0; src < rank; ++src)
            for (int d = 0; d < kRadix; ++d) recv_off[d / per] += hist_all[static_cast<size_t>(src) * kRadix + d];
        // the coarse histogram of THIS rank's keys, in the layout the pass expects (bins beyond R are empty)
        for (int d = 0; d < kRadix; ++d) pass_hist[d / per] += mine[d];
    } else {
        *xshift = 24;
        *bins = kRadix;
        const int st = osb200_sharded_plan(hist_all, R, rank, dest, recv_count, recv_off);
        if (st != OSB200_OK) return st;
        for (int d = 0; d < kRadix; ++d) pass_hist[d] = mine[d];
    }
    // Bucket imbalance beyond the capacity.  Every rank computes the whole recv_count[] from the same histograms, so with the
    // same capacity every rank takes this exit together.
    for (int q = 0; q < R; ++q)
        if (recv_count[q] > capacity) return OSB200_ERR_SIZE;
    if (recv_addrs)
        for (int d = 0; d < kRadix; ++d) out_base[d] = recv_addrs[dest[d]] / sizeof(uint32_t) + recv_off[d];
    // staged: the pass output is bin-major and dest[] is non-decreasing, so the bins of one destination are contiguous in
    // it; a destination receives source-major
    for (int p = 0; p <= R; ++p) send_off[p] = 0;
    for (int b = 0; b < kRadix; ++b) send_off[dest[b] + 1] += pass_hist[b];
    for (int p = 0; p < R; ++p) send_off[p + 1] += send_off[p];
    recv_from_off[0] = 0;
    for (int src = 0; src < R; ++src) {
        uint64_t c = 0;
        for (int d = 0; d < kRadix; ++d)
            if (dest[coarse ? d / per : d] == rank) c += hist_all[static_cast<size_t>(src) * kRadix + d];
        recv_from_off[src + 1] = recv_from_off[src] + c;
    }
    return OSB200_OK;
}

int osb200_sharded_unique_id(void* out_128_bytes)
{
    if (!out_128_bytes) return OSB200_ERR_INVALID_ARG;
    static_assert(sizeof(ncclUniqueId) == 128, "unique id size");
    ncclUniqueId id;
    OSB_NCCL(ncclGetUniqueId(&id));
    std::memcpy(out_128_bytes, &id, sizeof(id));
    return OSB200_OK;
}

int osb200_sharded_destroy(osb200_sharded_handle h)
{
    if (!h) return OSB200_ERR_INVALID_ARG;
    for (int r = 0; r < h->world; ++r)
        if (r != h->rank && h->peer_recv[r]) cudaIpcCloseMemHandle(h->peer_recv[r]);
    if (h->exch) osb200_destroy(h->exch);
    if (h->local) osb200_destroy(h->local);
    cudaFree(h->send_buf);
    cudaFree(h->recv_buf);
    cudaFree(h->d_hist);
    cudaFree(h->d_hist_all);
    cudaFree(h->d_out_base);
    cudaFree(h->d_flag);
    cudaFreeHost(h->h_hist_all);
    cudaFreeHost(h->h_out_base);
    cudaFreeHost(h->h_pass_hist);
    for (cudaEvent_t e : h->ev) if (e) cudaEventDestroy(e);
    if (h->sync_ev) cudaEventDestroy(h->sync_ev);
    if (h->comm) ncclCommDestroy(h->comm);
    delete h;
    return OSB200_OK;
}

int osb200_sharded_create(osb200_sharded_handle* out, const void* unique_id_128_bytes, int rank, int world,
                          uint64_t max_n_local, int slack_percent)
{
    if (!out) return OSB200_ERR_INVALID_ARG;
    *out = nullptr;
    if (!unique_id_128_bytes || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || max_n_local == 0 ||
        slack_percent < 0 || slack_percent > 400)
        return OSB200_ERR_INVALID_ARG;
    osb200_sharded_sorter* s = new (std::nothrow) osb200_sharded_sorter();
    if (!s) return OSB200_ERR_ALLOC;
    s->rank = rank;
    s->world = world;
    s->max_n_local = max_n_local;
    s->capacity = osb200_sharded_capacity(max_n_local, slack_percent);

    ncclUniqueId id;
    std::memcpy(&id, unique_id_128_bytes, sizeof(id));
    if (ncclCommInitRank(&s->comm, world, id, rank) != ncclSuccess) { osb200_sharded_destroy(s); return OSB200_ERR_NCCL; }

    int st = osb200_create(&s->exch, max_n_local, 4, 0);
    if (st == OSB200_OK) st = osb200_create(&s->local, s->capacity, 4, 0);
    if (st != OSB200_OK) { osb200_sharded_destroy(s); return st; }
    bool ok = cudaMalloc(&s->recv_buf, s->capacity * sizeof(uint32_t)) == cudaSuccess;
    ok = ok && cudaMalloc(&s->d_hist, kRadix * sizeof(unsigned long long)) == cudaSuccess;
    ok = ok && cudaMalloc(&s->d_hist_all, static_cast<size_t>(world) * kRadix * sizeof(unsigned long long)) == cudaSuccess;
    ok = ok && cudaMalloc(&s->d_out_base, kRadix * sizeof(unsigned long long)) == cudaSuccess;
    ok = ok && cudaMalloc(&s->d_flag, 64) == cudaSuccess;
    ok = ok && cudaMallocHost(&s->h_hist_all, static_cast<size_t>(world) * kRadix * sizeof(unsigned long long)) == cudaSuccess;
    ok = ok && cudaMallocHost(&s->h_out_base, kRadix * sizeof(unsigned long long)) == cudaSuccess;
    ok = ok && cudaMallocHost(&s->h_pass_hist, kRadix * sizeof(unsigned long long)) == cudaSuccess;
    for (auto& e : s->ev) ok = ok && cudaEventCreate(&e) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&s->sync_ev, cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { cudaGetLastError(); osb200_sharded_destroy(s); return OSB200_ERR_ALLOC; }
    cudaMemset(s->d_flag, 0, 64);

    // Map every peer's receive buffer (CUDA IPC over NVLink/NVSwitch; all ranks are processes on one node).
    s->peer_recv[rank] = s->recv_buf;
    s->fused = world > 1;
    if (world > 1) {
        cudaIpcMemHandle_t mine;
        std::vector<cudaIpcMemHandle_t> all(world);
        cudaIpcMemHandle_t* d_handles = nullptr;
        bool ipc_ok = cudaIpcGetMemHandle(&mine, s->recv_buf) == cudaSuccess;
        ipc_ok = ipc_ok && cudaMalloc(&d_handles, sizeof(cudaIpcMemHandle_t) * world) == cudaSuccess;
        if (ipc_ok) {
            cudaMemcpy(d_handles + rank, &mine, sizeof(mine), cudaMemcpyHostToDevice);
            ncclResult_t r = ncclAllGather(d_handles + rank, d_handles, sizeof(mine), ncclChar, s->comm, nullptr);
            ipc_ok = r == ncclSuccess && cudaStreamSynchronize(nullptr) == cudaSuccess;
            if (ipc_ok) cudaMemcpy(all.data(), d_handles, sizeof(mine) * world, cudaMemcpyDeviceToHost);
        }
        // every rank must take the same decision: agree on success with an all-reduce(min)
        int* d_ok = reinterpret_cast<int*>(s->d_flag) + 8;
        int flag = ipc_ok ? 1 : 0;
        if (ipc_ok) {
            for (int r = 0; r < world && flag; ++r) {
                if (r == rank) continue;
                if (cudaIpcOpenMemHandle(&s->peer_recv[r], all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                    cudaGetLastError();
                    s->peer_recv[r] = nullptr;
                    flag = 0;
                }
            }
        }
        cudaMemcpy(d_ok, &flag, sizeof(int), cudaMemcpyHostToDevice);
        if (ncclAllReduce(d_ok, d_ok, 1, ncclInt, ncclMin, s->comm, nullptr) != ncclSuccess ||
            cudaStreamSynchronize(nullptr) != cudaSuccess) {
            cudaFree(d_handles);
            osb200_sharded_destroy(s);
            return OSB200_ERR_NCCL;
        }
        cudaMemcpy(&flag, d_ok, sizeof(int), cudaMemcpyDeviceToHost);
        s->fused = flag == 1;
        cudaFree(d_handles);
        cudaGetLastError();
    }
    if (!s->fused && world > 1) {
        if (cudaMalloc(&s->send_buf, max_n_local * sizeof(uint32_t)) != cudaSuccess) { osb200_sharded_destroy(s); return OSB200_ERR_ALLOC; }
    }
    *out = s;
    return OSB200_OK;
}

// 0 = staged (NCCL send/recv), 1 = fused NVLink scatter.  Must be called identically on every rank.
OSB200_API int osb200_sharded_set_fused(osb200_sharded_handle h, int fused)
{
    if (!h) return OSB200_ERR_INVALID_ARG;
    if (fused) {
        for (int r = 0; r < h->world; ++r) if (!h->peer_recv[r]) return OSB200_ERR_UNSUPPORTED;
        h->fused = true;
        return OSB200_OK;
    }
    if (!h->send_buf && cudaMalloc(&h->send_buf, h->max_n_local * sizeof(uint32_t)) != cudaSuccess) return OSB200_ERR_ALLOC;
    h->fused = false;
    return OSB200_OK;
}

// Testing hook: 1 = always use the 256-bucket greedy plan even when the 2^k equal-width split would fit.
OSB200_API int osb200_sharded_force_fine(osb200_sharded_handle h, int on)
{
    if (!h) return OSB200_ERR_INVALID_ARG;
    h->force_fine = on != 0;
    return OSB200_OK;
}

OSB200_API int osb200_sharded_local_handle(osb200_sharded_handle h, osb200_handle* exch, osb200_handle* local)
{
    if (!h) return OSB200_ERR_INVALID_ARG;
    if (exch) *exch = h->exch;
    if (local) *local = h->local;
    return OSB200_OK;
}

int osb200_sharded_sort_keys_u32(osb200_sharded_handle h, const uint32_t* d_keys_local, uint64_t n_local,
                                 uint32_t** d_out, uint64_t* n_out, void* stream)
{
    if (!h || !d_out || !n_out || (n_local && !d_keys_local)) return OSB200_ERR_INVALID_ARG;
    if (n_local > h->max_n_local) return OSB200_ERR_SIZE;
    cudaStream_t q = static_cast<cudaStream_t>(stream);
    const int R = h->world;

    OSB_TRY(cudaEventRecord(h->ev[0], q));
    // 1-2. most-significant-digit histogram, all-gather
    int st = osb_internal_digit_histogram(h->exch, d_keys_local, n_local, 24, h->d_hist, q);
    if (st != OSB200_OK) return st;
    OSB_NCCL(ncclAllGather(h->d_hist, h->d_hist_all, kRadix, ncclUint64, h->comm, q));
    OSB_TRY(cudaMemcpyAsync(h->h_hist_all, h->d_hist_all, static_cast<size_t>(R) * kRadix * sizeof(unsigned long long),
                            cudaMemcpyDeviceToHost, q));
    // The plan (and the receive size) is needed on the host: the one host wait of a step, busy-polled.
    OSB_TRY(cudaEventRecord(h->sync_ev, q));
    OSB_TRY(spin_until(h->sync_ev));

    // 3. layout (osb200_sharded_exchange_layout): which bits the exchange pass bins on, where every bucket goes, the
    //    histogram the pass scans, the fused pass's per-bucket bases and the staged send/receive offsets.  OSB200_ERR_SIZE
    //    when the buckets do not fit the slack chosen at create: every rank holds the whole recv_count[] and the same
    //    capacity (max_n_local and slack_percent must be identical on all ranks), so ALL ranks take this exit together,
    //    before any collective or peer store of the exchange: nobody is left waiting in a barrier for a rank that bailed out.
    int32_t dest[kRadix];
    uint64_t recv_count[kMaxWorld], recv_off[kRadix], send_off[kMaxWorld + 1], roff[kMaxWorld + 1], recv_addrs[kMaxWorld];
    uint32_t xshift = 24;  // digit position of the exchange pass
    int32_t bins = kRadix;
    const bool fused = R > 1 && h->fused;
    if (fused)
        for (int r = 0; r < R; ++r) recv_addrs[r] = reinterpret_cast<uint64_t>(h->peer_recv[r]);
    // (h_out_base and h_pass_hist are free: the wait above ordered the previous call's copies from them)
    st = osb200_sharded_exchange_layout(reinterpret_cast<const uint64_t*>(h->h_hist_all), R, h->rank, h->capacity,
                                        h->force_fine ? 1 : 0, fused ? recv_addrs : nullptr, &xshift, &bins, dest, recv_count,
                                        recv_off, reinterpret_cast<uint64_t*>(h->h_pass_hist),
                                        fused ? reinterpret_cast<uint64_t*>(h->h_out_base) : nullptr, send_off, roff);
    if (st != OSB200_OK) return st;
    const uint64_t mine = recv_count[h->rank];
    // d_hist holds this rank's 256-bucket histogram already; a coarse pass scans the coarse one
    if (bins != kRadix)
        OSB_TRY(cudaMemcpyAsync(h->d_hist, h->h_pass_hist, kRadix * sizeof(unsigned long long), cudaMemcpyHostToDevice, q));
    OSB_TRY(cudaEventRecord(h->ev[1], q));

    // 4. exchange
    if (R == 1) {
        OSB_TRY(cudaMemcpyAsync(h->recv_buf, d_keys_local, n_local * sizeof(uint32_t), cudaMemcpyDeviceToDevice, q));
    } else if (fused) {
        // all ranks have finished reading their receive buffers from the previous call before anyone writes
        OSB_NCCL(ncclAllReduce(h->d_flag, h->d_flag, 1, ncclUint32, ncclSum, h->comm, q));
        OSB_TRY(cudaMemcpyAsync(h->d_out_base, h->h_out_base, kRadix * sizeof(unsigned long long), cudaMemcpyHostToDevice, q));
        st = osb_internal_binning_pass(h->exch, d_keys_local, nullptr, n_local, xshift, h->d_hist, h->d_out_base, q);
        if (st != OSB200_OK) return st;
        // every rank's scatter kernel has completed (and its NVLink stores are performed) before any local sort starts
        OSB_NCCL(ncclAllReduce(h->d_flag, h->d_flag, 1, ncclUint32, ncclSum, h->comm, q));
    } else {
        st = osb_internal_binning_pass(h->exch, d_keys_local, h->send_buf, n_local, xshift, h->d_hist, nullptr, q);
        if (st != OSB200_OK) return st;
        // send_buf is bin-major; the bins of destination p are contiguous.  Receive source-major.
        OSB_NCCL(ncclGroupStart());
        for (int p = 0; p < R; ++p) {
            if (send_off[p + 1] - send_off[p])
                OSB_NCCL(ncclSend(h->send_buf + send_off[p], send_off[p + 1] - send_off[p], ncclUint32, p, h->comm, q));
            if (roff[p + 1] - roff[p]) OSB_NCCL(ncclRecv(h->recv_buf + roff[p], roff[p + 1] - roff[p], ncclUint32, p, h->comm, q));
        }
        OSB_NCCL(ncclGroupEnd());
    }
    OSB_TRY(cudaEventRecord(h->ev[2], q));

    // 5. local OneSweep over the whole key.  (After a coarse exchange the keys of a rank share their top log2(R) bits, and a
    //    sort on the bits below them alone -- osb200_sort_bits(0, 32 - log2 R) -- is correct too, but was slower at 2^30
    //    keys: its masked histogram costs more and its 5-bit last digit takes the few-bins scatter.)
    st = osb200_sort_keys_u32(h->local, h->recv_buf, mine, q);
    if (st != OSB200_OK) return st;
    OSB_TRY(cudaEventRecord(h->ev[3], q));
    *d_out = h->recv_buf;
    *n_out = mine;
    return OSB200_OK;
}

int osb200_sharded_last_timing(osb200_sharded_handle h, float* out_ms4)
{
    if (!h || !out_ms4) return OSB200_ERR_INVALID_ARG;
    OSB_TRY(spin_until(h->ev[3]));
    OSB_TRY(cudaEventElapsedTime(&out_ms4[0], h->ev[0], h->ev[1]));
    OSB_TRY(cudaEventElapsedTime(&out_ms4[1], h->ev[1], h->ev[2]));
    OSB_TRY(cudaEventElapsedTime(&out_ms4[2], h->ev[2], h->ev[3]));
    OSB_TRY(cudaEventElapsedTime(&out_ms4[3], h->ev[0], h->ev[3]));
    return OSB200_OK;
}

}  // extern "C"
