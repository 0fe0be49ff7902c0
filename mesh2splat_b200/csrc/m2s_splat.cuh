// m2s_splat.cuh — arguments and scratch layout of the viewer's splat draw (m2s_splat.cu), shared with the C-ABI host code
// (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_tile.cuh"

namespace m2s {

constexpr uint64_t kSplatMaxCount = 1ull << 30;

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
    unsigned long long max_pairs;   // pair budget (< kTileMaxPairs)
    unsigned char* scratch;         // bin_layout(count, tile_count(width, height)) (m2s_bin.cuh)
    uint32_t* pairs;                // SortLayout(max_pairs) words (m2s_sort.cuh): the pair keys and values and their sort
};

// counts the (tile, quad) pairs of the n quads and scans them (bin_count_launch); the total lands in the ctrl words
cudaError_t splat_count_launch(const SplatArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest prefix that fits max_pairs (bin_pairs_launch), then draws every tile
cudaError_t splat_draw_launch(const SplatArgs& a, int sm_count, cudaStream_t stream);

}  // namespace m2s
