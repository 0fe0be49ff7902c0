// m2s_sort.cu — the viewer's depth sort (SURVEY 8 f-5): RadixSortPass::execute (src/renderer/renderPasses/RadixSortPass.cpp
// :8-90) = radixSortPrepass.glsl (key = the bits of the view depth, value = the index) + glu::RadixSort
// (thirdParty/RadixSort.hpp:1393-1562: 8 stable LSD passes of 4 bits) + radixSortGather.glsl (the quads in sorted order and
// the DrawElementsIndirectCommand).
//
// Shape: a stable LSD radix sort with 8-bit digits (4 passes give the permutation 8 passes of 4 bits give), onesweep:
//   sort_hist_kernel    reads the keys once and builds all four 256-bin digit histograms (shared-memory atomics, one
//                       global add per bin per CTA)
//   sort_scan_kernel    one CTA: the four histograms -> exclusive digit offsets, in place
//   sort_pass_kernel    one launch per pass.  A CTA claims its tile of kSortTile keys from the pass's atomic counter (so
//                       every tile it looks back on is already running), ranks the keys stably (warp multisplit with
//                       __match_any_sync, warp offsets in warp order), publishes its per-digit counts, looks back over
//                       the earlier tiles for their inclusive prefix (decoupled look-back), stages the tile by digit in
//                       shared memory and stores it in runs.  Pass 0 reads the depths as keys and makes the values
//                       (iota); the last pass stores only the values: the permutation.
//   sort_gather_kernel  sorted[i] = quads[order[i]], six threads per 96-byte quad with 16-byte loads and stores; the draw
//                       command.
// A separate gather rather than one fused into the last pass: the random 96-byte reads are latency-bound and want the
// occupancy of a small kernel, which the last pass (41 KB of shared memory per CTA) does not have; the order round trip it
// costs is 8 of the ~260 bytes per quad.
#include <algorithm>
#include <cuda/atomic>

#include "m2s_sort.cuh"

namespace m2s {

constexpr int kSortWarps = kSortThreads / 32;
constexpr uint32_t kStatusAggregate = 1u << 30;   // the tile's own count is published
constexpr uint32_t kStatusPrefix = 1u << 31;      // the inclusive prefix over tiles 0..t is published
constexpr uint32_t kStatusCount = (1u << 30) - 1u;

__device__ __forceinline__ uint32_t sort_count(unsigned long long count, const uint32_t* d_count) {
    unsigned long long n = count;
    if (d_count) n = min(n, (unsigned long long)*d_count);
    return (uint32_t)n;   // count < 2^30
}
__device__ __forceinline__ void store_release(uint32_t* p, uint32_t v) {
    cuda::atomic_ref<uint32_t, cuda::thread_scope_device>(*p).store(v, cuda::memory_order_release);
}
__device__ __forceinline__ uint32_t load_acquire(uint32_t* p) {
    return cuda::atomic_ref<uint32_t, cuda::thread_scope_device>(*p).load(cuda::memory_order_acquire);
}

// exclusive prefix of one value per thread over the CTA (thread order); s_warp: kSortWarps words
__device__ __forceinline__ uint32_t cta_exclusive_scan(uint32_t v, uint32_t* s_warp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t x = warp_inclusive_scan(v, lane);
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) before += w < warp ? s_warp[w] : 0u;
    __syncthreads();   // s_warp is free again
    return before + x - v;
}

__global__ void __launch_bounds__(kSortThreads) sort_hist_kernel(const uint32_t* __restrict__ keys, unsigned long long count,
                                                                 const uint32_t* d_count, uint32_t* hist) {
    __shared__ uint32_t s_hist[kSortPasses * 256];
    for (int i = threadIdx.x; i < kSortPasses * 256; i += kSortThreads) s_hist[i] = 0;
    __syncthreads();
    const uint32_t n = sort_count(count, d_count);
    const unsigned lane = threadIdx.x & 31;
    // warp-uniform loop bound (the top digit is counted with __match_any_sync): sign and exponent take few values in any
    // depth distribution, and a warp's same-address shared atomics serialise
    for (unsigned long long base = (unsigned long long)blockIdx.x * kSortThreads + (threadIdx.x & ~31u); base < n;
         base += (unsigned long long)gridDim.x * kSortThreads) {
        const unsigned long long i = base + lane;
        const bool ok = i < n;
        const uint32_t k = ok ? __ldg(keys + i) : 0u;
        if (ok) {
            atomicAdd(&s_hist[0 * 256 + (k & 255u)], 1u);
            atomicAdd(&s_hist[1 * 256 + ((k >> 8) & 255u)], 1u);
            atomicAdd(&s_hist[2 * 256 + ((k >> 16) & 255u)], 1u);
        }
        const uint32_t top = ok ? k >> 24 : 256u;
        const unsigned peers = __match_any_sync(0xffffffffu, top);
        if (ok && (peers & ((1u << lane) - 1u)) == 0) atomicAdd(&s_hist[3 * 256 + top], (uint32_t)__popc(peers));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kSortPasses * 256; i += kSortThreads)
        if (s_hist[i]) atomicAdd(hist + i, s_hist[i]);
}

__global__ void __launch_bounds__(kSortThreads) sort_scan_kernel(uint32_t* hist) {
    __shared__ uint32_t s_warp[kSortWarps];
    for (int p = 0; p < kSortPasses; ++p) {
        const uint32_t v = hist[p * 256 + threadIdx.x];
        hist[p * 256 + threadIdx.x] = cta_exclusive_scan(v, s_warp);
    }
}

// kFirst: keys_in are the depth bits, the values are the indices; kLast: only the values (the permutation) are stored
template <bool kFirst, bool kLast>
__global__ void __launch_bounds__(kSortThreads) sort_pass_kernel(const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                                                                 uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out,
                                                                 unsigned long long count, const uint32_t* d_count,
                                                                 const uint32_t* __restrict__ digit_off, uint32_t* tile_counter,
                                                                 uint32_t* status, unsigned shift) {
    __shared__ uint32_t s_keys[kSortTile], s_vals[kSortTile];   // the tile, staged by digit
    __shared__ uint32_t s_whist[kSortWarps][256];                // per warp and digit: count, then offset within the tile
    __shared__ uint32_t s_tile_off[256];                         // per digit: offset of its run within the tile
    __shared__ uint32_t s_base[256];                             // per digit: global position of staged slot 0
    __shared__ uint32_t s_warp[kSortWarps];
    __shared__ uint32_t s_tile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(tile_counter, 1u);
    for (int i = tid; i < kSortWarps * 256; i += kSortThreads) (&s_whist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t n = sort_count(count, d_count);
    const uint32_t t0 = tile * (uint32_t)kSortTile;
    if ((unsigned long long)tile * kSortTile >= n) return;   // at or beyond n: publishes nothing, and no tile below n waits on it
    const uint32_t tn = min(n - t0, (uint32_t)kSortTile);
    // ---- load: warp w takes keys [w * 512, (w + 1) * 512) of the tile, lane l key j * 32 + l of those (coalesced) ----
    const uint32_t wbase = (uint32_t)warp * 32u * kSortKeysPerThread;
    uint32_t k[kSortKeysPerThread], v[kSortKeysPerThread], r[kSortKeysPerThread];
#pragma unroll
    for (int j = 0; j < kSortKeysPerThread; ++j) {
        const uint32_t idx = wbase + j * 32u + lane;
        const bool ok = idx < tn;
        k[j] = ok ? __ldg(keys_in + t0 + idx) : 0u;
        v[j] = kFirst ? t0 + idx : (ok ? __ldg(vals_in + t0 + idx) : 0u);
    }
    // ---- rank within the warp, in input order (j-major, lane-minor): a key's rank = earlier keys of its digit ----
    const unsigned lt = (1u << lane) - 1u;
#pragma unroll
    for (int j = 0; j < kSortKeysPerThread; ++j) {
        const bool ok = wbase + j * 32u + lane < tn;
        const uint32_t d = ok ? (k[j] >> shift) & 255u : 256u;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const uint32_t before = ok ? s_whist[warp][d] : 0u;
        r[j] = before + __popc(peers & lt);
        __syncwarp();
        if (ok && (peers & lt) == 0) s_whist[warp][d] = before + __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    // ---- thread = digit: warp offsets in warp order, the tile's count; publish it ----
    const uint32_t dig = tid;
    uint32_t cnt = 0;
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) {
        const uint32_t c = s_whist[w][dig];
        s_whist[w][dig] = cnt;
        cnt += c;
    }
    uint32_t* my_status = status + (size_t)tile * 256 + dig;
    store_release(my_status, (tile == 0 ? kStatusPrefix : kStatusAggregate) | cnt);
    s_tile_off[dig] = cta_exclusive_scan(cnt, s_warp);
    __syncthreads();
    // ---- stage the tile by digit: stable positions within the tile ----
#pragma unroll
    for (int j = 0; j < kSortKeysPerThread; ++j) {
        if (wbase + j * 32u + lane < tn) {
            const uint32_t d = (k[j] >> shift) & 255u;
            const uint32_t pos = s_tile_off[d] + s_whist[warp][d] + r[j];
            s_keys[pos] = k[j];
            s_vals[pos] = v[j];
        }
    }
    // ---- decoupled look-back: the counts of this digit in the tiles before this one ----
    uint32_t excl = 0;
    if (tile > 0) {
        for (uint32_t t = tile - 1;; --t) {
            uint32_t s;
            do { s = load_acquire(status + (size_t)t * 256 + dig); } while ((s & (kStatusAggregate | kStatusPrefix)) == 0);
            excl += s & kStatusCount;
            if (s & kStatusPrefix) break;
        }
        store_release(my_status, kStatusPrefix | (excl + cnt));
    }
    s_base[dig] = digit_off[dig] + excl - s_tile_off[dig];
    __syncthreads();
    // ---- store: consecutive staged slots of a digit go to consecutive global positions ----
    for (uint32_t i = tid; i < tn; i += kSortThreads) {
        const uint32_t key = s_keys[i];
        const uint32_t dst = s_base[(key >> shift) & 255u] + i;
        if (!kLast) keys_out[dst] = key;
        vals_out[dst] = s_vals[i];
    }
}

constexpr int kGatherThreads = 256;

__global__ void __launch_bounds__(kGatherThreads) sort_gather_kernel(const float4* __restrict__ quads, const uint32_t* __restrict__ order,
                                                                     float4* __restrict__ sorted, unsigned long long count,
                                                                     const uint32_t* d_count, uint32_t* draw) {
    const uint32_t n = sort_count(count, d_count);
    if (draw && blockIdx.x == 0 && threadIdx.x == 0) {   // radixSortGather.glsl: {6, u_count, 0, 0}; the fifth word is 0
        draw[0] = 6u; draw[1] = n; draw[2] = 0u; draw[3] = 0u; draw[4] = 0u;
    }
    const unsigned long long total = (unsigned long long)n * 6ull;
    for (unsigned long long i = (unsigned long long)blockIdx.x * kGatherThreads + threadIdx.x; i < total;
         i += (unsigned long long)gridDim.x * kGatherThreads) {
        const unsigned long long q = i / 6ull;
        const unsigned j = (unsigned)(i - q * 6ull);
        sorted[i] = __ldg(quads + (unsigned long long)__ldg(order + q) * 6ull + j);
    }
}

cudaError_t sort_order_launch(const uint32_t* keys, unsigned long long count, const uint32_t* d_count, uint32_t* order, uint32_t* scratch,
                              int sm_count, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    const SortLayout l = sort_layout(count);
    uint32_t* hist = scratch;
    uint32_t* counters = scratch + kSortPasses * 256;
    uint32_t* status = counters + 32;
    uint32_t* kb[2] = {scratch + l.ctrl_words, scratch + l.ctrl_words + 2 * l.buf_words};
    uint32_t* vb[2] = {scratch + l.ctrl_words + l.buf_words, scratch + l.ctrl_words + 3 * l.buf_words};
    cudaError_t e = cudaMemsetAsync(scratch, 0, l.ctrl_words * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    const unsigned hist_grid = (unsigned)std::min<uint64_t>(l.tiles, 2ull * sm_count);
    sort_hist_kernel<<<hist_grid, kSortThreads, 0, stream>>>(keys, count, d_count, hist);
    sort_scan_kernel<<<1, kSortThreads, 0, stream>>>(hist);
    const unsigned grid = (unsigned)l.tiles;
    const size_t sw = l.tiles * 256;
    sort_pass_kernel<true, false><<<grid, kSortThreads, 0, stream>>>(keys, nullptr, kb[0], vb[0], count, d_count, hist + 0 * 256,
                                                                      counters + 0, status + 0 * sw, 0u);
    sort_pass_kernel<false, false><<<grid, kSortThreads, 0, stream>>>(kb[0], vb[0], kb[1], vb[1], count, d_count, hist + 1 * 256,
                                                                       counters + 1, status + 1 * sw, 8u);
    sort_pass_kernel<false, false><<<grid, kSortThreads, 0, stream>>>(kb[1], vb[1], kb[0], vb[0], count, d_count, hist + 2 * 256,
                                                                       counters + 2, status + 2 * sw, 16u);
    sort_pass_kernel<false, true><<<grid, kSortThreads, 0, stream>>>(kb[0], vb[0], nullptr, order, count, d_count, hist + 3 * 256,
                                                                      counters + 3, status + 3 * sw, 24u);
    return cudaGetLastError();
}

cudaError_t sort_launch(const SortArgs& a, int sm_count, cudaStream_t stream) {
    const cudaError_t e = sort_order_launch(a.depth_bits, a.count, a.d_count, a.order, a.scratch, sm_count, stream);
    if (e != cudaSuccess) return e;
    if (a.count > 0 || a.draw) {
        const uint64_t want = (a.count * 6ull + kGatherThreads - 1) / kGatherThreads;
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, 16ull * sm_count));
        sort_gather_kernel<<<grid, kGatherThreads, 0, stream>>>(a.quads, a.order, a.sorted, a.count, a.d_count, a.draw);
    }
    return cudaGetLastError();
}

cudaError_t sort_pairs16_launch(uint32_t* scratch, uint64_t capacity, const uint32_t* d_n, int sm_count, cudaStream_t stream) {
    if (capacity == 0) return cudaSuccess;
    const SortLayout l = sort_layout(capacity);
    uint32_t* hist = scratch;
    uint32_t* counters = scratch + kSortPasses * 256;
    uint32_t* status = counters + 32;
    uint32_t* kb[2] = {scratch + l.ctrl_words, sort_pairs16_keys(scratch, capacity)};
    uint32_t* vb[2] = {scratch + l.ctrl_words + l.buf_words, sort_pairs16_vals(scratch, capacity)};
    cudaError_t e = cudaMemsetAsync(scratch, 0, l.ctrl_words * sizeof(uint32_t), stream);
    if (e != cudaSuccess) return e;
    const unsigned hist_grid = (unsigned)std::min<uint64_t>(l.tiles, 2ull * sm_count);
    sort_hist_kernel<<<hist_grid, kSortThreads, 0, stream>>>(kb[1], capacity, d_n, hist);
    sort_scan_kernel<<<1, kSortThreads, 0, stream>>>(hist);
    const unsigned grid = (unsigned)l.tiles;
    const size_t sw = l.tiles * 256;
    sort_pass_kernel<false, false><<<grid, kSortThreads, 0, stream>>>(kb[1], vb[1], kb[0], vb[0], capacity, d_n,
                                                                       hist + 0 * 256, counters + 0, status + 0 * sw, 0u);
    sort_pass_kernel<false, false><<<grid, kSortThreads, 0, stream>>>(kb[0], vb[0], kb[1], vb[1], capacity, d_n,
                                                                       hist + 1 * 256, counters + 1, status + 1 * sw, 8u);
    return cudaGetLastError();
}

}  // namespace m2s
