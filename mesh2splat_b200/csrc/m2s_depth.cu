// m2s_depth.cu — the viewer's mesh depth pre-pass (SURVEY 8 f-9): DepthPrepass::execute
// (src/renderer/renderPasses/DepthPrepass.cpp:8-49) + depthPrepassVS.glsl / depthPrepassPS.glsl.  Every triangle of an
// opaque primitive (baseColorFactor.a == 1.0f) drawn into a W x H D24 map cleared to 1, depth test LESS, no culling.
//
// Shape (the shadow pass's cube raster over one W x H viewport, DESIGN §2 "The mesh depth pre-pass"):
//   binning (m2s_bin.cuh) per source triangle: transform, clip (six planes, guard factor 2 in x and y), fan, snap,
//                        and the 16 x 16 tiles each fan triangle touches; (tile, source triangle << 3 | fan triangle)
//                        pairs of the longest prefix of source triangles that fits the budget, stably sorted by tile;
//                        each tile's run
//   depth_tile_kernel    one CTA per tile, one thread per pixel: fan triangles staged in shared memory, depth from the
//                        exact edge values in fp64, the minimum D24 code in a register, one store per texel
// The unit of a pair is the fan triangle, so the tile kernel stages one triangle per pair; it re-clips the source
// triangle to find it (a triangle that needs no clipping is its own fan of one).  Every operation that decides a bit of
// the map is round-to-nearest fp32 / fp64 with no contraction (__f*_rn, __d*_rn), integer, or a conversion of DESIGN
// §2, so the map equals the oracle's (oracle/m2s_depth_oracle.c) bit for bit.
#include "m2s_bin.cuh"
#include "m2s_clip.cuh"
#include "m2s_depth.cuh"

namespace m2s {

namespace {
// a triangle of no primitive or of a non-opaque one is not drawn
__device__ __forceinline__ bool depth_opaque(const DepthArgs& a, uint32_t tri) {
    DRange r;
    return prim_range(a.ranges, a.nranges, tri, r) && __ldg(&a.prims[r.prim].factor[3]) == 1.0f;   // DepthPrepass.cpp:33, an exact compare
}

// the vertex transform: (P V) M p
struct DepthXf {
    const DepthArgs& a;
    __device__ __forceinline__ float4 operator()(float x, float y, float z) const {
        return make_float4(clip_row(a.pvm, 0, x, y, z, 1.0f), clip_row(a.pvm, 1, x, y, z, 1.0f), clip_row(a.pvm, 2, x, y, z, 1.0f),
                           clip_row(a.pvm, 3, x, y, z, 1.0f));
    }
};

}  // namespace

// the binning (m2s_bin.cuh): source triangles, n = ntri, one pair per tile each fan triangle of an opaque triangle
// touches, pair value = source triangle << 3 | fan triangle
struct DepthBins {
    DepthArgs a;
    __host__ __device__ unsigned long long items() const { return a.ntri; }
    __host__ __device__ uint64_t tiles() const { return tile_count(a.width, a.height); }
    __device__ __forceinline__ uint32_t n() const { return (uint32_t)a.ntri; }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        return clip_visit<false>(a.tris, i, a.width, a.height, [&](uint32_t t) { return depth_opaque(a, t); }, DepthXf{a}, f);
    }
};

// stages fan triangle v & 7 of source triangle v >> 3 (which has pairs, so is opaque) in slot `slot`, edge values
// relative to pixel (ox, oy).  Not inlined: the tile kernel's pixel loop then keeps its registers, where the division
// slow paths of the set-up would otherwise make it spill them.
__device__ __noinline__ void depth_stage(const DepthArgs& a, uint32_t v, int ox, int oy, FanEdges& s, int slot) {
    float4 poly[kClipMaxPoly];
    clip_tri_poly(a.tris, v >> 3, DepthXf{a}, poly);
    clip_stage<false>(poly, (int)(v & 7u), a.width, a.height, ox, oy, s, slot);
}

__global__ void __launch_bounds__(kTileThreads) depth_tile_kernel(const __grid_constant__ DepthArgs a, const uint32_t* __restrict__ vals) {
    __shared__ FanEdges s;
    const TileFrame f = tile_frame(a.scratch, bin_layout(a.ntri, tile_count(a.width, a.height)), tiles_x(a.width), blockIdx.x);
    uint32_t best = kD24Clear;
    tile_batches(f, vals, [&](int tid, uint32_t val) { depth_stage(a, val, f.ox, f.oy, s, tid); }, [&](uint32_t j) {
        uint32_t code;
        if (clip_depth(s, j, f.lx, f.ly, code)) best = min(best, code);   // LESS on codes
    });
    if (f.x >= (int)a.width || f.y >= (int)a.height) return;
    a.depth[(size_t)f.y * a.width + f.x] = d24_decode(best);
}

// ---- launches -------------------------------------------------------------------------------------------------------
cudaError_t depth_count_launch(const DepthArgs& a, cudaStream_t stream) { return bin_count_launch(DepthBins{a}, stream); }

cudaError_t depth_draw_launch(const DepthArgs& a, int sm_count, cudaStream_t stream) {
    return bin_draw_launch(DepthBins{a}, depth_tile_kernel, sm_count, stream);
}

}  // namespace m2s
