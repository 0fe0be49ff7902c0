// m2s_3dgs.cuh — arguments and scratch layout of the standard 3DGS render (m2s_3dgs.cu), shared with the C-ABI host code
// (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_sort.cuh"
#include "m2s_tile.cuh"

namespace m2s {

constexpr uint64_t kGs3dMaxCount = 1ull << 30;   // the depth sort's count limit (kSortMaxCount)
constexpr uint32_t kGs3dCulled = 0xFFFFFFFFu;   // the depth key of a culled record: past every survivor's (d > 0)

// the per-gaussian splat record of the preprocess kernel, 48 B (zero for a culled record):
//   a = (u, v, conic.x, conic.y)   mean in pixels, the inverse 2-D covariance
//   b = (conic.z, opacity, r, g)
//   c = (b, x0 | x1 << 16, y0 | y1 << 16, radius)   the tile rectangle [x0, x1) x [y0, y1) as uint32 bits, radius in pixels
struct Gs3dSplat {
    float4 a, b, c;
};
constexpr int kGs3dVaryings = 9;   // what the tile kernels stage per gaussian: u, v, conic.xyz, opacity, r, g, b

// Context scratch of one render (bytes), one allocation:
//   ctrl    uint32 n (the records considered) | uint32 survivors
//   splats  Gs3dSplat per record
//   keys    uint32 per record: the depth key
//   order   uint32 per record: the record indices in (depth key, index) order
struct Gs3dLayout {
    size_t splats_off, keys_off, order_off, total_bytes;
};
inline Gs3dLayout gs3d_layout(uint64_t count) {
    Gs3dLayout l;
    l.splats_off = 256;
    l.keys_off = (l.splats_off + count * sizeof(Gs3dSplat) + 255) & ~size_t(255);
    l.order_off = (l.keys_off + count * 4 + 255) & ~size_t(255);
    l.total_bytes = l.order_off + count * 4;
    return l;
}

struct Gs3dArgs {
    float MV[16], P[16];            // world_to_view * model_to_world (fp64, rounded once), view_to_clip; column-major
    float cam[3];                   // the camera in model space (SH direction)
    float near, mult, scale_modifier, bg[3];
    uint32_t width, height;
    uint32_t layout;                // record layout: 0 REF96 (96 B), 1 PACKED56 (56 B)
    uint32_t sh_vec4, sh_degree;    // the SH buffer's float4 per gaussian, the degree evaluated (0: none)
    const float4* sh;
    unsigned long long count;       // capacity: the grids are sized for it
    const unsigned long long* d_count;   // optional: n = min(count, *d_count)
    const unsigned char* records;
    uint32_t* ctrl;                 // gs3d_layout: n, survivors
    Gs3dSplat* splats;
    uint32_t* keys;
    uint32_t* order;
    uint32_t* sort_scratch;         // SortLayout(count) words (m2s_sort.cuh)
    float4* rgba32f;                // W x H float4, or NULL
    uint32_t* rgba8;                // W x H RGBA8 words, or NULL
    int sm_count;
    unsigned long long max_pairs;   // pair budget (< kTileMaxPairs)
    unsigned char* scratch;         // bin_layout(count, tile_count(width, height)) (m2s_bin.cuh)
    uint32_t* pairs;                // SortLayout(max_pairs) words: the pair keys and values and their sort
};

// the forward pass that keeps its state for the backward pass (m2s_3dgs_render_grad): Gs3dSaveLayout
struct Gs3dSaveArgs : Gs3dArgs {
    uint32_t* rank;                 // per record: its position in order (the inverse of order)
    float* final_T;                 // per pixel: the transmittance after the last blended gaussian
    uint32_t* n_contrib;            // per pixel: 1 + the run position of its last blended gaussian (0: none)
};

// What the forward pass keeps for the backward pass besides the render's own scratch (bytes), one allocation:
//   rank       uint32 per record
//   final_T    float per pixel (row-major, row 0 = the bottom row)
//   n_contrib  uint32 per pixel
struct Gs3dSaveLayout {
    size_t rank_off, final_T_off, contrib_off, total_bytes;
};
inline Gs3dSaveLayout gs3d_save_layout(uint64_t count, uint32_t width, uint32_t height) {
    Gs3dSaveLayout l;
    const size_t pix = (size_t)width * height;
    l.rank_off = 0;
    l.final_T_off = (count * 4 + 255) & ~size_t(255);
    l.contrib_off = (l.final_T_off + pix * 4 + 255) & ~size_t(255);
    l.total_bytes = l.contrib_off + pix * 4;
    return l;
}

// The backward pass (m2s_3dgs_grad.cu) of the state's last forward pass, PACKED56 records.  a: that forward's arguments
// (the state's scratch, with the budget it drew); grad_rgba: dL/d(RGBA32F image); grad: count x 14 floats, written whole.
// Context scratch: kGs3dPartials floats per pair slot of the budget, then one uint32 per tile (Gs3dGradLayout).
constexpr int kGs3dPartials = 9;   // dL/du, dL/dv, dL/dconic (3), dL/dopacity, dL/dcolour (3)
constexpr int kPacked56Floats = 14;
struct Gs3dGradLayout {
    size_t tile_last_off, total_bytes;
};
inline Gs3dGradLayout gs3d_grad_layout(uint64_t max_pairs, uint64_t tiles) {
    Gs3dGradLayout l;
    l.tile_last_off = (max_pairs * kGs3dPartials * 4 + 255) & ~size_t(255);
    l.total_bytes = l.tile_last_off + tiles * 4;
    return l;
}
struct Gs3dGradArgs {
    Gs3dSaveArgs a;
    const float4* grad_rgba;
    float* grad;
    float* part;             // kGs3dPartials per pair slot
    uint32_t* tile_last;     // per tile: the run positions the backward walked (max n_contrib over the tile's pixels)
    const uint32_t* vals;    // the sorted pair values (bin_vals), NULL without a budget
};

// the preprocess kernel alone: one splat record and depth key per record, n and the survivors in ctrl
cudaError_t gs3d_preprocess_launch(const Gs3dArgs& a, cudaStream_t stream);
// preprocess, depth order, and the count and scan of the (tile, gaussian) pairs of the survivors (bin_count_launch)
cudaError_t gs3d_count_launch(const Gs3dArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest depth-ordered prefix that fits max_pairs (bin_pairs_launch), then every tile
cudaError_t gs3d_draw_launch(const Gs3dArgs& a, int sm_count, cudaStream_t stream);
// the same two steps keeping the state: the ranks of the depth order, then the tile kernel that also writes the per-pixel
// state; the image is the render's bit for bit
cudaError_t gs3d_count_save_launch(const Gs3dSaveArgs& a, cudaStream_t stream);
cudaError_t gs3d_draw_save_launch(const Gs3dSaveArgs& a, int sm_count, cudaStream_t stream);
// the tile backward, then the per-record gather and chain rule (m2s_3dgs_grad.cu)
cudaError_t gs3d_backward_launch(const Gs3dGradArgs& g, cudaStream_t stream);

}  // namespace m2s
