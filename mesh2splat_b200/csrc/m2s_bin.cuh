// m2s_bin.cuh — the tile binning of the viewer's tiled rasterisers: the splat draw (m2s_splat.cu), the shadow pass's
// cube raster (m2s_light.cu) and the mesh depth pre-pass (m2s_depth.cu).  Each pass bins its items (quads, light
// records, source triangles) into 16 x 16 tiles and then runs its own tile kernel over each tile's run of pairs:
//   bin_count_kernel     per item: the number of its (tile, value) pairs, scanned within the block of kBinBlock items
//   bin_scan_kernel      one CTA: exclusive prefix over the block sums; the total number of pairs
//   bin_emit_kernel      per item of the longest prefix whose pairs fit the budget: its pairs at its scan offset, so the
//                        pairs come out in item order; the prefix length and its pair count
//   sort_pairs16_launch  stable onesweep sort of the pairs by tile id (the depth sort's kernels, m2s_sort.cu)
//   bin_ranges_kernel    each tile's run in the sorted pairs
// The kernels are templates over a small per-pass binner B, named after its pass so that the kernel names say which
// pass they belong to (bin_emit_kernel<m2s::ShadowBins>):
//   B::a                                  the pass's arguments, with a.scratch (bin_layout(items(), tiles())),
//                                         a.pairs (SortLayout(a.max_pairs) words, m2s_sort.cuh) and a.max_pairs (< 2^30)
//   B::items(), B::tiles()                capacity (the grids and the scratch are sized for it) and tile count
//   __device__ uint32_t B::n()            the items binned by this call, <= items()
//   __device__ uint32_t B::visit(i, f)    calls f(tile, value) for every pair of item i, in tile-id order; returns
//                                         their number
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_sort.cuh"

namespace m2s {

constexpr int kBinBlock = 512;          // items per CTA of the count and emit kernels (and per scan block)
constexpr int kBinScanThreads = 1024;   // the one-CTA scan of the block sums

// Per-call scratch (bytes), one allocation:
//   ctrl    uint64 total pairs | uint32 drawn | uint32 pairs emitted (= pairs of the drawn prefix)
//   excl    uint32 per item: exclusive prefix of the pair counts within its block of kBinBlock items
//   blocks  uint64 per block: its pair count, then (in place) the exclusive prefix over the blocks
//   ranges  uint32 [2][tiles]: start and end of each tile's run in the sorted pairs (zeroed per call)
struct BinLayout {
    uint64_t blocks, tiles;
    size_t excl_off, blocks_off, ranges_off, total_bytes;
};
__host__ __device__ inline BinLayout bin_layout(uint64_t items, uint64_t tiles) {
    BinLayout l;
    l.blocks = (items + kBinBlock - 1) / kBinBlock;
    l.tiles = tiles;
    l.excl_off = 256;
    l.blocks_off = (l.excl_off + items * 4 + 255) & ~size_t(255);
    l.ranges_off = (l.blocks_off + l.blocks * 8 + 255) & ~size_t(255);
    l.total_bytes = l.ranges_off + l.tiles * 8;
    return l;
}

// ---- count and scan ------------------------------------------------------------------------------------------------
template <typename B>
__global__ void __launch_bounds__(kBinBlock) bin_count_kernel(B b) {
    __shared__ uint32_t s_warp[kBinBlock / 32];
    const BinLayout l = bin_layout(b.items(), b.tiles());
    uint32_t* excl = reinterpret_cast<uint32_t*>(b.a.scratch + l.excl_off);
    unsigned long long* blocks = reinterpret_cast<unsigned long long*>(b.a.scratch + l.blocks_off);
    const uint32_t n = b.n();
    const uint64_t i = (uint64_t)blockIdx.x * kBinBlock + threadIdx.x;
    if ((uint64_t)blockIdx.x * kBinBlock >= n) return;   // blocks at or past n are never read
    const uint32_t cnt = i < n ? b.visit((uint32_t)i, [](uint32_t, uint32_t) {}) : 0u;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kBinBlock / 32; ++w) {
        before += w < warp ? s_warp[w] : 0u;
        total += s_warp[w];
    }
    if (i < n) excl[i] = before + x - cnt;
    if (threadIdx.x == 0) blocks[blockIdx.x] = total;
}

template <typename B>
__global__ void __launch_bounds__(kBinScanThreads) bin_scan_kernel(B b) {
    __shared__ unsigned long long s_warp[kBinScanThreads / 32];
    __shared__ unsigned long long s_carry;
    const BinLayout l = bin_layout(b.items(), b.tiles());
    unsigned long long* blocks = reinterpret_cast<unsigned long long*>(b.a.scratch + l.blocks_off);
    const uint32_t nb = (b.n() + kBinBlock - 1) / kBinBlock;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nb; base += kBinScanThreads) {
        const uint32_t k = base + threadIdx.x;
        const unsigned long long v = k < nb ? blocks[k] : 0ull;
        unsigned long long x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        unsigned long long before = s_carry, chunk = 0;
        for (int w = 0; w < kBinScanThreads / 32; ++w) {
            before += w < warp ? s_warp[w] : 0ull;
            chunk += s_warp[w];
        }
        if (k < nb) blocks[k] = before + x - v;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) *reinterpret_cast<unsigned long long*>(b.a.scratch) = s_carry;
}

// ---- pair emission and tile ranges ---------------------------------------------------------------------------------
template <typename B>
__global__ void __launch_bounds__(kBinBlock) bin_emit_kernel(B b, uint32_t* keys, uint32_t* vals) {
    const BinLayout l = bin_layout(b.items(), b.tiles());
    const uint32_t* excl = reinterpret_cast<const uint32_t*>(b.a.scratch + l.excl_off);
    const unsigned long long* blocks = reinterpret_cast<const unsigned long long*>(b.a.scratch + l.blocks_off);
    uint32_t* ctrl = reinterpret_cast<uint32_t*>(b.a.scratch);
    const unsigned long long total = *reinterpret_cast<const unsigned long long*>(b.a.scratch);
    const uint32_t n = b.n();
    const uint64_t i64 = (uint64_t)blockIdx.x * kBinBlock + threadIdx.x;
    if (i64 >= n) return;
    const uint32_t i = (uint32_t)i64;
    auto offset = [&](uint32_t k) { return k < n ? blocks[k / kBinBlock] + excl[k] : total; };
    const unsigned long long start = offset(i), end = offset(i + 1);
    if (end > b.a.max_pairs) return;   // not in the prefix whose pairs fit
    if (i + 1 == n || offset(i + 2) > b.a.max_pairs) {   // the prefix's last item
        ctrl[2] = i + 1;
        ctrl[3] = (uint32_t)end;
    }
    if (end == start) return;
    uint32_t c = 0;
    b.visit(i, [&](uint32_t tile, uint32_t value) {
        keys[start + c] = tile;
        vals[start + c] = value;
        ++c;
    });
}

template <typename B>
__global__ void bin_ranges_kernel(B b, const uint32_t* keys) {
    const BinLayout l = bin_layout(b.items(), b.tiles());
    uint32_t* start = reinterpret_cast<uint32_t*>(b.a.scratch + l.ranges_off);
    uint32_t* end = start + l.tiles;
    const uint32_t np = reinterpret_cast<const uint32_t*>(b.a.scratch)[3];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
        const uint32_t k = keys[i];
        if (i == 0 || keys[i - 1] != k) start[k] = i;
        if (i + 1 == np || keys[i + 1] != k) end[k] = i + 1;
    }
}

// ---- launches ------------------------------------------------------------------------------------------------------
// the pair values in tile order once bin_pairs_launch has run (the tile kernel's input); NULL without a budget
template <typename B>
uint32_t* bin_vals(const B& b) {
    return b.a.max_pairs ? sort_pairs16_vals(b.a.pairs, b.a.max_pairs) : nullptr;
}

// counts the pairs of the n items and scans them; the total lands in the scratch's ctrl words
template <typename B>
cudaError_t bin_count_launch(const B& b, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(b.a.scratch, 0, 16, stream);   // total pairs, drawn, pairs emitted
    if (e != cudaSuccess) return e;
    const BinLayout l = bin_layout(b.items(), b.tiles());
    if (l.blocks) bin_count_kernel<B><<<(unsigned)l.blocks, kBinBlock, 0, stream>>>(b);
    bin_scan_kernel<B><<<1, kBinScanThreads, 0, stream>>>(b);
    return cudaGetLastError();
}

// emits and sorts the pairs of the longest prefix that fits max_pairs and finds each tile's run; with no budget the
// emission still finds the prefix (the leading items with no pair) and writes no pair
template <typename B>
cudaError_t bin_pairs_launch(const B& b, int sm_count, cudaStream_t stream) {
    const BinLayout l = bin_layout(b.items(), b.tiles());
    cudaError_t e = cudaMemsetAsync(b.a.scratch + l.ranges_off, 0, l.tiles * 8, stream);
    if (e != cudaSuccess) return e;
    const unsigned long long max_pairs = b.a.max_pairs;
    uint32_t* keys = max_pairs ? sort_pairs16_keys(b.a.pairs, max_pairs) : nullptr;
    if (l.blocks) bin_emit_kernel<B><<<(unsigned)l.blocks, kBinBlock, 0, stream>>>(b, keys, bin_vals(b));
    if (max_pairs > 0) {
        e = sort_pairs16_launch(b.a.pairs, max_pairs, reinterpret_cast<const uint32_t*>(b.a.scratch) + 3, sm_count, stream);
        if (e != cudaSuccess) return e;
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((max_pairs + 255) / 256, 8ull * sm_count));
        bin_ranges_kernel<B><<<grid, 256, 0, stream>>>(b, keys);
    }
    return cudaGetLastError();
}

}  // namespace m2s
