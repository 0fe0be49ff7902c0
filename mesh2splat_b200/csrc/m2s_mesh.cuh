// m2s_mesh.cuh — arguments of the viewer's mesh G-buffer pass (m2s_mesh.cu), shared with the C-ABI host code
// (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_depth.cuh"
#include "m2s_device.cuh"
#include "m2s_tile.cuh"

namespace m2s {

// Scratch: bin_layout (m2s_bin.cuh) with one pair count per SOURCE triangle, W x H pixels (as the depth pass).
struct MeshArgs {
    const float4* tris;             // the scene's triangle soup, 9 float4 per triangle (m2s_device.cuh)
    unsigned long long ntri;        // < kDepthMaxTris
    const DRange* ranges;           // triangle -> primitive; a triangle of no primitive is not drawn
    uint32_t nranges;
    const DPrim* prims;             // base colour factor and maps
    const DTexture* texs;           // the mip chains (m2s_scene_upload)
    const uint32_t* arena;
    float M[16], V[16], P[16];      // u_modelToWorld, u_worldToView, u_viewToClip, column-major
    float N[9];                     // mat3(transpose(inverse(M))), column-major, GLM's fp32 inverse (host)
    float near_far[2];              // u_nearFar
    uint32_t width, height, mode;
    uint16_t* position;             // W x H x 4 fp16 bits, or NULL
    uint16_t* normal;
    uint8_t* albedo;                // W x H x 4 uint8, or NULL
    uint16_t* depth;
    uint8_t* metallic_roughness;
    unsigned long long max_pairs;   // (tile, fan triangle) pair budget (< kTileMaxPairs)
    unsigned char* scratch;         // bin_layout(ntri, tile_count(width, height))
    uint32_t* pairs;                // SortLayout(max_pairs) words (m2s_sort.cuh)
};

// counts and scans the (tile, fan triangle) pairs of every source triangle; the total lands in the scratch's ctrl words
cudaError_t mesh_count_launch(const MeshArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest prefix of source triangles that fits max_pairs, then writes every pixel of
// every non-NULL target
cudaError_t mesh_draw_launch(const MeshArgs& a, int sm_count, cudaStream_t stream);

}  // namespace m2s
