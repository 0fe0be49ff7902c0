// m2s_splat.cu — the viewer's splat draw (SURVEY 8 f-6): GaussianSplattingPass::execute (src/renderer/renderPasses/
// GaussianSplattingPass.cpp:37-97) = one instanced glDrawElementsIndirect of the sorted quads (two triangles each) through
// gaussianSplattingVS.glsl and gaussianSplattingPS.glsl into the five G-buffer targets, blended front to back
// (GL_ONE_MINUS_DST_ALPHA, GL_ONE; GL_ONE, GL_ONE in render mode 4).  The fixed-function parts follow DESIGN §2.
//
// Shape: a tiled rasteriser that keeps GL's per-pixel order (instance, then triangle):
//   binning (m2s_bin.cuh) per quad: snap the four corners, set up both triangles, the 16 x 16 tiles they touch (edge
//                         functions against the tile's pixel-centre box); (tile, quad) pairs of the longest prefix of
//                         quads that fits the budget, in quad order, stably sorted by tile; each tile's run
//   splat_tile_kernel     one CTA per tile, one thread per pixel: the tile's quads staged in shared memory in batches,
//                         coverage, fragment shader and blends in registers (each target rounded to its format after
//                         every blend), one coalesced store per live target
// All arithmetic that decides a bit of the image is round-to-nearest fp32 with no contraction (__f*_rn), integer, or
// the conversions to the target formats, so the image equals the oracle's (oracle/m2s_splat_oracle.c) bit for bit.
#include "m2s_bin.cuh"
#include "m2s_splat.cuh"

namespace m2s {

// ---- binning (m2s_bin.cuh): quads, n = min(count, d_draw[1]), pair value = quad index -------------------------------
struct SplatBins {
    SplatArgs a;
    __host__ __device__ unsigned long long items() const { return a.count; }
    __host__ __device__ uint64_t tiles() const { return tile_count(a.width, a.height); }
    __device__ __forceinline__ uint32_t n() const {
        unsigned long long n = a.count;
        if (a.d_draw) n = min(n, (unsigned long long)a.d_draw[1]);
        return (uint32_t)n;   // count < 2^30
    }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        TileTri t[2];
        tile_quad_setup(a.quads + (uint64_t)i * 6, (int)a.width, (int)a.height, t);
        return tile_walk_quad(t, tiles_x(a.width), [&](uint32_t, uint32_t tile) { f(tile, i); });
    }
};

// ---- fragment shader, blend, formats -------------------------------------------------------------------------------

// RGBA16F: dst = src * f + dst in fp32, then one conversion to half.  dst holds the channel's half value as a float.
__device__ __forceinline__ void splat_blend_f16(float (&dst)[4], const float (&src)[4], bool additive) {
    const float f = additive ? 1.0f : sb(1.0f, dst[3]);
    uint16_t b;
#pragma unroll
    for (int c = 0; c < 4; ++c) dst[c] = to_half(ad(ml(src[c], f), dst[c]), b);
}

// RGBA8: dst = d / 255; src, f and the result clamped to [0, 1]; stored as round-half-even(result * 255)
__device__ __forceinline__ void splat_blend_u8(uint32_t (&dst)[4], const float (&src)[4], bool additive) {
    const float f = additive ? 1.0f : sat(sb(1.0f, dv((float)dst[3], 255.0f)));
#pragma unroll
    for (int c = 0; c < 4; ++c) dst[c] = unorm8(ad(ml(sat(src[c]), f), dv((float)dst[c], 255.0f)));
}

// per staged quad: both triangles' edges (quad_stage) and the varyings of gaussianSplattingVS.glsl
constexpr int kSplatVaryings = 18;
struct SplatStage {
    QuadEdges e;
    float v[kSplatVaryings][kTileThreads];
};

__global__ void __launch_bounds__(kTileThreads) splat_tile_kernel(SplatArgs a, const uint32_t* __restrict__ vals) {
    __shared__ SplatStage s;
    const TileFrame f = tile_frame(a.scratch, bin_layout(a.count, tile_count(a.width, a.height)), tiles_x(a.width), blockIdx.x);
    const bool additive = a.mode == 4;
    const float fx = (float)f.x + 0.5f, fy = (float)f.y + 0.5f;   // gl_FragCoord.xy
    float pos[4] = {0, 0, 0, 0}, nrm[4] = {0, 0, 0, 0}, dep[4] = {0, 0, 0, 0};
    uint32_t alb[4] = {0, 0, 0, 0}, mr[4] = {0, 0, 0, 0};
    const float fw = (float)a.width, fh = (float)a.height;
    auto stage = [&](int tid, uint32_t val) {
        const float4* q = a.quads + (uint64_t)val * 6;
        TileTri t[2];
        tile_quad_setup(q, (int)a.width, (int)a.height, t);
        quad_stage(t, f.ox, f.oy, s.e, tid);
        const float4 m = q[0], col = q[2], con = q[3], n = q[4], ws = q[5];
        // gaussianSplattingVS.glsl:33-40
        s.v[0][tid] = ml(ml(ad(m.x, 1.0f), 0.5f), fw);   // out_screen
        s.v[1][tid] = ml(ml(ad(m.y, 1.0f), 0.5f), fh);
        s.v[2][tid] = ml(-0.5f, con.x);                   // out_conic
        s.v[3][tid] = -con.y;
        s.v[4][tid] = ml(-0.5f, con.z);
        s.v[5][tid] = ml(col.x, col.w);                   // out_color
        s.v[6][tid] = ml(col.y, col.w);
        s.v[7][tid] = ml(col.z, col.w);
        s.v[8][tid] = col.w;                              // out_opacity
        s.v[9][tid] = n.x; s.v[10][tid] = n.y; s.v[11][tid] = n.z;       // out_normal
        s.v[12][tid] = ws.x; s.v[13][tid] = ws.y; s.v[14][tid] = ws.z;   // out_wsPos
        s.v[15][tid] = con.w;                                            // out_depth
        s.v[16][tid] = n.w; s.v[17][tid] = ws.w;                         // metallicRoughness
    };
    tile_batches(f, vals, stage, [&](uint32_t j) {
        const int cover = quad_cover(s.e, j, f.lx, f.ly);
        if (!cover) return;
        // gaussianSplattingPS.glsl:29-46
        const float dx = sb(s.v[0][j], fx), dy = sb(s.v[1][j], fy);
        const float alpha = ad(ad(ml(s.v[2][j], ml(dx, dx)), ml(s.v[4][j], ml(dy, dy))), ml(s.v[3][j], ml(dx, dy)));
        const float g = rn_exp(alpha);
        const float op = ml(s.v[8][j], g);
        const float src_pos[4] = {ml(s.v[12][j], g), ml(s.v[13][j], g), ml(s.v[14][j], g), g};
        const float src_nrm[4] = {ml(s.v[9][j], g), ml(s.v[10][j], g), ml(s.v[11][j], g), op};
        const float dp = ml(s.v[15][j], g);
        const float src_dep[4] = {dp, dp, dp, op};
        float src_alb[4] = {0.01f, 0.005f, 0.0f, 0.01f};
        if (!additive) { src_alb[0] = ml(s.v[5][j], g); src_alb[1] = ml(s.v[6][j], g); src_alb[2] = ml(s.v[7][j], g); src_alb[3] = op; }
        const float src_mr[4] = {ml(s.v[16][j], g), ml(s.v[17][j], g), ml(0.0f, g), g};
        for (int c = 0; c < cover; ++c) {   // a pixel both snapped triangles cover is blended twice
            if (a.position) splat_blend_f16(pos, src_pos, additive);
            if (a.normal) splat_blend_f16(nrm, src_nrm, additive);
            if (a.albedo) splat_blend_u8(alb, src_alb, additive);
            if (a.depth) splat_blend_f16(dep, src_dep, additive);
            if (a.metallic_roughness) splat_blend_u8(mr, src_mr, additive);
        }
    });
    if (f.x >= (int)a.width || f.y >= (int)a.height) return;
    const GTexel o = {half4(pos[0], pos[1], pos[2], pos[3]), half4(nrm[0], nrm[1], nrm[2], nrm[3]), half4(dep[0], dep[1], dep[2], dep[3]),
                      alb[0] | alb[1] << 8 | alb[2] << 16 | alb[3] << 24, mr[0] | mr[1] << 8 | mr[2] << 16 | mr[3] << 24};
    gbuffer_store(a, (size_t)f.y * a.width + f.x, o);
}

// ---- launches ------------------------------------------------------------------------------------------------------
cudaError_t splat_count_launch(const SplatArgs& a, cudaStream_t stream) { return bin_count_launch(SplatBins{a}, stream); }

cudaError_t splat_draw_launch(const SplatArgs& a, int sm_count, cudaStream_t stream) {
    return bin_draw_launch(SplatBins{a}, splat_tile_kernel, sm_count, stream);
}

}  // namespace m2s
