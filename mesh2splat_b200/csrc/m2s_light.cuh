// m2s_light.cuh — arguments and scratch layout of the viewer's shadow pass and deferred lighting (m2s_light.cu), shared
// with the C-ABI host code (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_splat.cuh"

namespace m2s {

constexpr uint32_t kShadowMaxSize = 1024;                 // 6 faces x 64 x 64 tiles of 16 x 16: a tile id fits in 16 bits
constexpr uint64_t kShadowMaxCount = 1ull << 30;
constexpr uint32_t kShadowClearCode = 0xFFFFFFu;          // D24 clear value 1.0 = 2^24 - 1
constexpr uint32_t kShadowCulled = 0xFFFFFFFFu;           // face word of a culled light record
constexpr int kLightPrepassThreads = 256;
constexpr int kLightThreads = 256;                        // deferred lighting: one thread per pixel

// One light-space record per source gaussian, in source order (32 B = two float4):
//   float4 0: mean NDC x, y | quadScaleNdc x, y (major axis)      float4 1: quadScaleNdc z, w (minor axis) | gl_FragDepth | face
// face is 0..5 (+X -X +Y -Y +Z -Z), or kShadowCulled with every other word 0.
constexpr size_t kLightRecordBytes = 32;

// the cube raster's tiles: 6 faces of S x S pixels, each ceil(S/16)^2 tiles of 16 x 16
__host__ __device__ inline uint64_t shadow_tiles(uint32_t size) { return splat_tiles(size, size) * 6; }

struct ShadowArgs {
    // light prepass (gaussianPointShadowMappingCS.glsl)
    const unsigned char* records;   // count x 96 B (REF96) or 56 B (PACKED56)
    unsigned long long count;
    const unsigned long long* d_count;   // optional: n = min(count, *d_count)
    uint32_t layout;                // record layout: 0 REF96, 1 PACKED56
    uint32_t fmt;                   // the reference's u_format: 0 conversion, 1 PACKED56 or a loaded .ply
    float M[16];                    // u_modelToWorld
    float V[6][16];                 // u_worldToViews: glm::lookAt per face
    float P[16];                    // u_viewToClip: glm::perspective(90 deg, 1, near, far)
    float Rinv[9];                  // inverse(mat3(u_modelToWorld)), GLM's fp32 formula
    float mscale2[3];               // modelScale * modelScale, modelScale = |M[0]|, |M[0]|, |M[1]| (GLM's fp32 length)
    float light[3];
    float res[2];                   // the renderer's resolution (sic)
    float near_far[2];
    float std_dev;
    float4* light_quads;            // count x 32 B
    // cube raster (gaussianPointLightCubeMapShadowVS/PS.glsl into 6 x size^2 D24 texels)
    uint32_t size;
    float* cube;                    // 6 x size x size floats: (float)code / 16777215
    unsigned long long max_pairs;   // (tile, record) pair budget (< kSplatMaxPairs)
    unsigned char* scratch;         // bin_layout(count, shadow_tiles(size)) (m2s_bin.cuh)
    uint32_t* pairs;                // SortLayout(max_pairs) words (m2s_sort.cuh)
};

// the light prepass: one 32-byte record per source gaussian
cudaError_t light_prepass_launch(const ShadowArgs& a, cudaStream_t stream);
// counts and scans the (tile, record) pairs of the n light records (bin_count_launch); the total lands in the ctrl words
cudaError_t shadow_count_launch(const ShadowArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest prefix that fits max_pairs (bin_pairs_launch), then writes every texel of the
// cube
cudaError_t shadow_draw_launch(const ShadowArgs& a, int sm_count, cudaStream_t stream);

struct LightArgs {
    const uint16_t* position;       // G-buffer, as m2s_gbuffer (RGBA16F bits / RGBA8)
    const uint16_t* normal;
    const uint8_t* albedo;
    const uint8_t* metallic_roughness;
    const float* cube;              // 6 x shadow_size^2 (mode 6 only)
    uint32_t width, height, mode, shadow_size;
    float light[3], light_color[3], light_intensity, cam[3], far_plane;
    uint8_t* image;                 // width x height x 4, row 0 = the bottom row
};

cudaError_t deferred_light_launch(const LightArgs& a, cudaStream_t stream);

}  // namespace m2s
