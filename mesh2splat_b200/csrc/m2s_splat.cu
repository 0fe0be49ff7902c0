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
#include <cuda_fp16.h>

#include "m2s_bin.cuh"
#include "m2s_splat.cuh"

namespace m2s {

__device__ __forceinline__ int splat_tiles_x(const SplatArgs& a) { return (int)((a.width + kSplatTile - 1) / kSplatTile); }

// ---- binning (m2s_bin.cuh): quads, n = min(count, d_draw[1]), pair value = quad index -------------------------------
struct SplatBins {
    SplatArgs a;
    __host__ __device__ unsigned long long items() const { return a.count; }
    __host__ __device__ uint64_t tiles() const { return splat_tiles(a.width, a.height); }
    __device__ __forceinline__ uint32_t n() const {
        unsigned long long n = a.count;
        if (a.d_draw) n = min(n, (unsigned long long)a.d_draw[1]);
        return (uint32_t)n;   // count < 2^30
    }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        SplatTri t[2];
        splat_quad_setup(a.quads + (uint64_t)i * 6, (int)a.width, (int)a.height, t);
        return splat_for_each_tile(t, splat_tiles_x(a), [&](uint32_t, uint32_t tile) { f(tile, i); });
    }
};

// ---- fragment shader, blend, formats -------------------------------------------------------------------------------

// fp32 -> fp16 bits, round to nearest even; overflow gives +-inf, NaN gives 0x7FFF, subnormals are kept
__device__ __forceinline__ float splat_to_half(float v, uint16_t& bits) {
    if (v != v) { bits = 0x7FFFu; return v; }
    const __half h = __float2half_rn(v);
    bits = __half_as_ushort(h);
    return __half2float(h);
}

// RGBA16F: dst = src * f + dst in fp32, then one conversion to half.  dst holds the channel's half value as a float.
__device__ __forceinline__ void splat_blend_f16(float (&dst)[4], const float (&src)[4], bool additive) {
    const float f = additive ? 1.0f : __fsub_rn(1.0f, dst[3]);
    uint16_t b;
#pragma unroll
    for (int c = 0; c < 4; ++c) dst[c] = splat_to_half(__fadd_rn(__fmul_rn(src[c], f), dst[c]), b);
}

__device__ __forceinline__ float splat_sat(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

// RGBA8: dst = d / 255; src, f and the result clamped to [0, 1]; stored as round-half-even(result * 255)
__device__ __forceinline__ void splat_blend_u8(uint32_t (&dst)[4], const float (&src)[4], bool additive) {
    const float f = additive ? 1.0f : splat_sat(__fsub_rn(1.0f, __fdiv_rn((float)dst[3], 255.0f)));
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float d = __fdiv_rn((float)dst[c], 255.0f);
        const float r = splat_sat(__fadd_rn(__fmul_rn(splat_sat(src[c]), f), d));
        dst[c] = __float2uint_rn(__fmul_rn(r, 255.0f));
    }
}

// per staged quad: both triangles' edge functions relative to the tile origin, with the top-left rule folded in
// (E >= 0 inside), and the varyings of gaussianSplattingVS.glsl
constexpr int kSplatVaryings = 18;
struct SplatStage {
    int32_t A[6][kSplatThreads], B[6][kSplatThreads];
    long long C[6][kSplatThreads];
    float v[kSplatVaryings][kSplatThreads];
};

__global__ void __launch_bounds__(kSplatThreads) splat_tile_kernel(SplatArgs a, const uint32_t* __restrict__ vals) {
    __shared__ SplatStage s;
    const BinLayout l = bin_layout(a.count, splat_tiles(a.width, a.height));
    const uint32_t* start = reinterpret_cast<const uint32_t*>(a.scratch + l.ranges_off);
    const uint32_t tiles_x = (uint32_t)splat_tiles_x(a);
    const uint32_t tile = blockIdx.x;
    const int ox = (int)(tile % tiles_x) * kSplatTile, oy = (int)(tile / tiles_x) * kSplatTile;
    const int tid = threadIdx.x, lx = tid % kSplatTile, ly = tid / kSplatTile;
    const int x = ox + lx, y = oy + ly;
    const uint32_t r0 = start[tile], r1 = start[l.tiles + tile];
    const bool additive = a.mode == 4;
    const float fx = (float)x + 0.5f, fy = (float)y + 0.5f;   // gl_FragCoord.xy
    float pos[4] = {0, 0, 0, 0}, nrm[4] = {0, 0, 0, 0}, dep[4] = {0, 0, 0, 0};
    uint32_t alb[4] = {0, 0, 0, 0}, mr[4] = {0, 0, 0, 0};
    const float fw = (float)a.width, fh = (float)a.height;
    for (uint32_t base = r0; base < r1; base += kSplatThreads) {
        const uint32_t nb = min(r1 - base, (uint32_t)kSplatThreads);
        __syncthreads();
        if ((uint32_t)tid < nb) {
            const float4* q = a.quads + (uint64_t)vals[base + tid] * 6;
            SplatTri t[2];
            splat_quad_setup(q, (int)a.width, (int)a.height, t);
#pragma unroll
            for (int e = 0; e < 6; ++e) {
                const SplatTri& tt = t[e / 3];
                const int k = e % 3;
                s.A[e][tid] = tt.A[k];
                s.B[e][tid] = tt.B[k];
                s.C[e][tid] = tt.C[k] + (long long)tt.A[k] * ox + (long long)tt.B[k] * oy - (tt.incl[k] ? 0 : 1);
            }
            const float4 m = q[0], col = q[2], con = q[3], n = q[4], ws = q[5];
            // gaussianSplattingVS.glsl:33-40
            s.v[0][tid] = __fmul_rn(__fmul_rn(__fadd_rn(m.x, 1.0f), 0.5f), fw);   // out_screen
            s.v[1][tid] = __fmul_rn(__fmul_rn(__fadd_rn(m.y, 1.0f), 0.5f), fh);
            s.v[2][tid] = __fmul_rn(-0.5f, con.x);                                // out_conic
            s.v[3][tid] = -con.y;
            s.v[4][tid] = __fmul_rn(-0.5f, con.z);
            s.v[5][tid] = __fmul_rn(col.x, col.w);                                // out_color
            s.v[6][tid] = __fmul_rn(col.y, col.w);
            s.v[7][tid] = __fmul_rn(col.z, col.w);
            s.v[8][tid] = col.w;                                                  // out_opacity
            s.v[9][tid] = n.x; s.v[10][tid] = n.y; s.v[11][tid] = n.z;            // out_normal
            s.v[12][tid] = ws.x; s.v[13][tid] = ws.y; s.v[14][tid] = ws.z;        // out_wsPos
            s.v[15][tid] = con.w;                                                 // out_depth
            s.v[16][tid] = n.w; s.v[17][tid] = ws.w;                              // metallicRoughness
        }
        __syncthreads();
        for (uint32_t j = 0; j < nb; ++j) {
            int cover = 0;
#pragma unroll
            for (int tri = 0; tri < 2; ++tri) {
                bool in = true;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const int e = tri * 3 + k;
                    in &= s.C[e][j] + (long long)s.A[e][j] * lx + (long long)s.B[e][j] * ly >= 0;
                }
                cover += in ? 1 : 0;
            }
            if (!cover) continue;
            // gaussianSplattingPS.glsl:29-46
            const float dx = __fsub_rn(s.v[0][j], fx), dy = __fsub_rn(s.v[1][j], fy);
            const float alpha = __fadd_rn(__fadd_rn(__fmul_rn(s.v[2][j], __fmul_rn(dx, dx)), __fmul_rn(s.v[4][j], __fmul_rn(dy, dy))),
                                          __fmul_rn(s.v[3][j], __fmul_rn(dx, dy)));
            const float g = splat_exp(alpha);
            const float op = __fmul_rn(s.v[8][j], g);
            const float src_pos[4] = {__fmul_rn(s.v[12][j], g), __fmul_rn(s.v[13][j], g), __fmul_rn(s.v[14][j], g), g};
            const float src_nrm[4] = {__fmul_rn(s.v[9][j], g), __fmul_rn(s.v[10][j], g), __fmul_rn(s.v[11][j], g), op};
            const float dp = __fmul_rn(s.v[15][j], g);
            const float src_dep[4] = {dp, dp, dp, op};
            float src_alb[4] = {0.01f, 0.005f, 0.0f, 0.01f};
            if (!additive) { src_alb[0] = __fmul_rn(s.v[5][j], g); src_alb[1] = __fmul_rn(s.v[6][j], g); src_alb[2] = __fmul_rn(s.v[7][j], g); src_alb[3] = op; }
            const float src_mr[4] = {__fmul_rn(s.v[16][j], g), __fmul_rn(s.v[17][j], g), __fmul_rn(0.0f, g), g};
            for (int c = 0; c < cover; ++c) {   // a pixel both snapped triangles cover is blended twice
                if (a.position) splat_blend_f16(pos, src_pos, additive);
                if (a.normal) splat_blend_f16(nrm, src_nrm, additive);
                if (a.albedo) splat_blend_u8(alb, src_alb, additive);
                if (a.depth) splat_blend_f16(dep, src_dep, additive);
                if (a.metallic_roughness) splat_blend_u8(mr, src_mr, additive);
            }
        }
    }
    if (x >= (int)a.width || y >= (int)a.height) return;
    const size_t px = (size_t)y * a.width + x;
    uint16_t h[4];
    if (a.position) {
        for (int c = 0; c < 4; ++c) splat_to_half(pos[c], h[c]);
        reinterpret_cast<uint2*>(a.position)[px] = make_uint2(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16);
    }
    if (a.normal) {
        for (int c = 0; c < 4; ++c) splat_to_half(nrm[c], h[c]);
        reinterpret_cast<uint2*>(a.normal)[px] = make_uint2(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16);
    }
    if (a.depth) {
        for (int c = 0; c < 4; ++c) splat_to_half(dep[c], h[c]);
        reinterpret_cast<uint2*>(a.depth)[px] = make_uint2(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16);
    }
    if (a.albedo) reinterpret_cast<uint32_t*>(a.albedo)[px] = alb[0] | alb[1] << 8 | alb[2] << 16 | alb[3] << 24;
    if (a.metallic_roughness) reinterpret_cast<uint32_t*>(a.metallic_roughness)[px] = mr[0] | mr[1] << 8 | mr[2] << 16 | mr[3] << 24;
}

// ---- launches ------------------------------------------------------------------------------------------------------
cudaError_t splat_count_launch(const SplatArgs& a, cudaStream_t stream) { return bin_count_launch(SplatBins{a}, stream); }

cudaError_t splat_draw_launch(const SplatArgs& a, int sm_count, cudaStream_t stream) {
    const SplatBins b{a};
    const cudaError_t e = bin_pairs_launch(b, sm_count, stream);
    if (e != cudaSuccess) return e;
    splat_tile_kernel<<<(unsigned)b.tiles(), kSplatThreads, 0, stream>>>(a, bin_vals(b));
    return cudaGetLastError();
}

}  // namespace m2s
