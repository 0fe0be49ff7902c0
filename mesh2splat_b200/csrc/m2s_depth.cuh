// m2s_depth.cuh — arguments and scratch layout of the viewer's mesh depth pre-pass (m2s_depth.cu), shared with the C-ABI
// host code (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_device.cuh"
#include "m2s_tile.cuh"

namespace m2s {

constexpr uint64_t kDepthMaxTris = 1ull << 29;     // pair value = source triangle << 3 | fan triangle

// Scratch: bin_layout (m2s_bin.cuh) with one pair count per SOURCE triangle, W x H pixels.
struct DepthArgs {
    const float4* tris;             // the scene's triangle soup, 9 float4 per triangle (m2s_device.cuh)
    unsigned long long ntri;        // < kDepthMaxTris
    const DRange* ranges;           // triangle -> primitive
    uint32_t nranges;
    const DPrim* prims;             // a triangle is drawn iff its primitive's factor.a == 1.0f
    float pvm[16];                  // (P V) M, column-major, GLM's mat4 * mat4 in fp32
    uint32_t width, height;
    float* depth;                   // W x H floats: (float)code / 16777215, row 0 = window y 0
    unsigned long long max_pairs;   // (tile, fan triangle) pair budget (< kTileMaxPairs)
    unsigned char* scratch;         // bin_layout(ntri, tile_count(width, height))
    uint32_t* pairs;                // SortLayout(max_pairs) words (m2s_sort.cuh)
};

// counts and scans the (tile, fan triangle) pairs of every source triangle; the total lands in the scratch's ctrl words
cudaError_t depth_count_launch(const DepthArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest prefix of source triangles that fits max_pairs, then writes every texel
cudaError_t depth_draw_launch(const DepthArgs& a, int sm_count, cudaStream_t stream);

}  // namespace m2s
