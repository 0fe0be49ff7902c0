// m2s_splat.cuh — arguments and scratch layout of the viewer's splat draw (m2s_splat.cu), shared with the C-ABI host code
// (m2s_api.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

constexpr int kSplatTile = 16;                           // screen tiles of 16 x 16 pixels, one CTA per tile
constexpr int kSplatThreads = kSplatTile * kSplatTile;   // tile kernel: one thread per pixel
constexpr int kSplatBlock = 512;                         // quads per CTA of the per-quad kernels (and per scan block)
constexpr uint32_t kSplatMaxSide = 4096;                 // 256 x 256 tiles: a tile id fits in 16 bits
constexpr uint64_t kSplatMaxCount = 1ull << 30;
constexpr uint64_t kSplatMaxPairs = 1ull << 30;          // the pair sort's count limit (kSortMaxCount)

// Per-call scratch (bytes), one allocation:
//   ctrl    uint64 total pairs | uint32 drawn | uint32 pairs emitted (= pairs of the drawn prefix)
//   excl    uint32 per quad: exclusive prefix of the pair counts within its block of kSplatBlock quads
//   blocks  uint64 per block: its pair count, then (in place) the exclusive prefix over the blocks
//   ranges  uint32 [2][tiles]: start and end of each tile's run in the sorted pairs (zeroed per call)
struct SplatLayout {
    uint64_t blocks, tiles;
    size_t excl_off, blocks_off, ranges_off, total_bytes;
};
__host__ __device__ inline SplatLayout splat_layout(uint64_t count, uint32_t width, uint32_t height) {
    SplatLayout l;
    l.blocks = (count + kSplatBlock - 1) / kSplatBlock;
    l.tiles = (uint64_t)((width + kSplatTile - 1) / kSplatTile) * ((height + kSplatTile - 1) / kSplatTile);
    l.excl_off = 256;
    l.blocks_off = (l.excl_off + count * 4 + 255) & ~size_t(255);
    l.ranges_off = (l.blocks_off + l.blocks * 8 + 255) & ~size_t(255);
    l.total_bytes = l.ranges_off + l.tiles * 8;
    return l;
}

struct SplatArgs {
    const float4* quads;            // count x 96 B, sorted front to back
    unsigned long long count;       // capacity: the grids are sized for it
    const uint32_t* d_draw;         // optional DrawElementsIndirectCommand: n = min(count, d_draw[1])
    uint32_t width, height, mode;
    uint16_t* position;             // W x H x 4 fp16 bits, or NULL
    uint16_t* normal;
    uint8_t* albedo;                // W x H x 4 uint8, or NULL
    uint16_t* depth;
    uint8_t* metallic_roughness;
    unsigned long long max_pairs;   // pair budget (< kSplatMaxPairs)
    unsigned char* scratch;         // SplatLayout of (count, width, height)
    uint32_t* pairs;                // SortLayout(max_pairs) words (m2s_sort.cuh): the pair keys and values and their sort
};

// counts the (tile, quad) pairs of the n quads and scans them; the total lands in the scratch's ctrl words
cudaError_t splat_count_launch(const SplatArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest prefix that fits max_pairs, then draws every tile
cudaError_t splat_draw_launch(const SplatArgs& a, int sm_count, cudaStream_t stream);

}  // namespace m2s
