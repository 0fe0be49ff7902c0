// m2s_splat.cu — the viewer's splat draw (SURVEY 8 f-6): GaussianSplattingPass::execute (src/renderer/renderPasses/
// GaussianSplattingPass.cpp:37-97) = one instanced glDrawElementsIndirect of the sorted quads (two triangles each) through
// gaussianSplattingVS.glsl and gaussianSplattingPS.glsl into the five G-buffer targets, blended front to back
// (GL_ONE_MINUS_DST_ALPHA, GL_ONE; GL_ONE, GL_ONE in render mode 4).  The fixed-function parts follow DESIGN §2.
//
// Shape: a tiled rasteriser that keeps GL's per-pixel order (instance, then triangle):
//   splat_count_kernel    per quad: snap the four corners, set up both triangles, count the 16 x 16 tiles they touch
//                         (edge functions against the tile's pixel-centre box), scan the counts within the block
//   splat_scan_kernel     one CTA: exclusive prefix over the block sums; the total number of pairs
//   splat_emit_kernel     per quad of the prefix whose pairs fit the budget: its (tile, quad) pairs at its scan offset, so
//                         the pairs come out in quad order; the prefix length and its pair count
//   sort_pairs16_launch   stable onesweep sort of the pairs by tile id (the depth sort's kernels, m2s_sort.cu)
//   splat_ranges_kernel   each tile's run in the sorted pairs
//   splat_tile_kernel     one CTA per tile, one thread per pixel: the tile's quads staged in shared memory in batches,
//                         coverage, fragment shader and blends in registers (each target rounded to its format after
//                         every blend), one coalesced store per live target
// All arithmetic that decides a bit of the image is round-to-nearest fp32 with no contraction (__f*_rn), integer, or
// the conversions to the target formats, so the image equals the oracle's (oracle/m2s_splat_oracle.c) bit for bit.
#include <algorithm>
#include <cuda_fp16.h>

#include "m2s_sort.cuh"
#include "m2s_splat.cuh"

namespace m2s {

__device__ __forceinline__ uint32_t splat_n(const SplatArgs& a) {
    unsigned long long n = a.count;
    if (a.d_draw) n = min(n, (unsigned long long)a.d_draw[1]);
    return (uint32_t)n;   // count < 2^30
}

__device__ __forceinline__ int splat_tiles_x(const SplatArgs& a) { return (int)((a.width + kSplatTile - 1) / kSplatTile); }

// ---- count and scan ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kSplatBlock) splat_count_kernel(SplatArgs a) {
    __shared__ uint32_t s_warp[kSplatBlock / 32];
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
    uint32_t* excl = reinterpret_cast<uint32_t*>(a.scratch + l.excl_off);
    unsigned long long* blocks = reinterpret_cast<unsigned long long*>(a.scratch + l.blocks_off);
    const uint32_t n = splat_n(a);
    const uint64_t i = (uint64_t)blockIdx.x * kSplatBlock + threadIdx.x;
    if ((uint64_t)blockIdx.x * kSplatBlock >= n) return;   // blocks at or past n are never read
    uint32_t cnt = 0;
    if (i < n) {
        SplatTri t[2];
        splat_quad_setup(a.quads + i * 6, (int)a.width, (int)a.height, t);
        cnt = splat_for_each_tile(t, splat_tiles_x(a), [](uint32_t, uint32_t) {});
    }
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
    for (int w = 0; w < kSplatBlock / 32; ++w) {
        before += w < warp ? s_warp[w] : 0u;
        total += s_warp[w];
    }
    if (i < n) excl[i] = before + x - cnt;
    if (threadIdx.x == 0) blocks[blockIdx.x] = total;
}

constexpr int kSplatScanThreads = 1024;

__global__ void __launch_bounds__(kSplatScanThreads) splat_scan_kernel(SplatArgs a) {
    __shared__ unsigned long long s_warp[kSplatScanThreads / 32];
    __shared__ unsigned long long s_carry;
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
    unsigned long long* blocks = reinterpret_cast<unsigned long long*>(a.scratch + l.blocks_off);
    const uint32_t n = splat_n(a);
    const uint32_t nb = (n + kSplatBlock - 1) / kSplatBlock;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nb; base += kSplatScanThreads) {
        const uint32_t b = base + threadIdx.x;
        const unsigned long long v = b < nb ? blocks[b] : 0ull;
        unsigned long long x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        unsigned long long before = s_carry, chunk = 0;
        for (int w = 0; w < kSplatScanThreads / 32; ++w) {
            before += w < warp ? s_warp[w] : 0ull;
            chunk += s_warp[w];
        }
        if (b < nb) blocks[b] = before + x - v;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) *reinterpret_cast<unsigned long long*>(a.scratch) = s_carry;
}

// ---- pair emission -------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long splat_offset(const uint32_t* excl, const unsigned long long* blocks, uint32_t i,
                                                           uint32_t n, unsigned long long total) {
    return i < n ? blocks[i / kSplatBlock] + excl[i] : total;
}

__global__ void __launch_bounds__(kSplatBlock) splat_emit_kernel(SplatArgs a, uint32_t* keys, uint32_t* vals) {
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
    const uint32_t* excl = reinterpret_cast<const uint32_t*>(a.scratch + l.excl_off);
    const unsigned long long* blocks = reinterpret_cast<const unsigned long long*>(a.scratch + l.blocks_off);
    uint32_t* ctrl = reinterpret_cast<uint32_t*>(a.scratch);
    const unsigned long long total = *reinterpret_cast<const unsigned long long*>(a.scratch);
    const uint32_t n = splat_n(a);
    const uint64_t i64 = (uint64_t)blockIdx.x * kSplatBlock + threadIdx.x;
    if (i64 >= n) return;
    const uint32_t i = (uint32_t)i64;
    const unsigned long long start = splat_offset(excl, blocks, i, n, total);
    const unsigned long long end = splat_offset(excl, blocks, i + 1, n, total);
    if (end > a.max_pairs) return;   // not in the prefix whose pairs fit
    if (i + 1 == n || splat_offset(excl, blocks, i + 2, n, total) > a.max_pairs) {   // the prefix's last quad
        ctrl[2] = i + 1;
        ctrl[3] = (uint32_t)end;
    }
    if (end == start) return;
    SplatTri t[2];
    splat_quad_setup(a.quads + (uint64_t)i * 6, (int)a.width, (int)a.height, t);
    splat_for_each_tile(t, splat_tiles_x(a), [&](uint32_t c, uint32_t tile) {
        keys[start + c] = tile;
        vals[start + c] = i;
    });
}

__global__ void splat_ranges_kernel(SplatArgs a, const uint32_t* keys) {
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
    uint32_t* start = reinterpret_cast<uint32_t*>(a.scratch + l.ranges_off);
    uint32_t* end = start + l.tiles;
    const uint32_t np = reinterpret_cast<const uint32_t*>(a.scratch)[3];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
        const uint32_t k = keys[i];
        if (i == 0 || keys[i - 1] != k) start[k] = i;
        if (i + 1 == np || keys[i + 1] != k) end[k] = i + 1;
    }
}

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
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
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
cudaError_t splat_count_launch(const SplatArgs& a, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(a.scratch, 0, 16, stream);   // total pairs, drawn, pairs emitted
    if (e != cudaSuccess) return e;
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
    if (l.blocks) splat_count_kernel<<<(unsigned)l.blocks, kSplatBlock, 0, stream>>>(a);
    splat_scan_kernel<<<1, kSplatScanThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t splat_draw_launch(const SplatArgs& a, int sm_count, cudaStream_t stream) {
    const SplatLayout l = splat_layout(a.count, a.width, a.height);
    cudaError_t e = cudaMemsetAsync(a.scratch + l.ranges_off, 0, l.tiles * 8, stream);
    if (e != cudaSuccess) return e;
    // with no budget the emission still finds the prefix (the leading quads that touch no tile) and writes no pair
    uint32_t* keys = a.max_pairs ? sort_pairs16_keys(a.pairs, a.max_pairs) : nullptr;
    uint32_t* vals = a.max_pairs ? sort_pairs16_vals(a.pairs, a.max_pairs) : nullptr;
    if (l.blocks) splat_emit_kernel<<<(unsigned)l.blocks, kSplatBlock, 0, stream>>>(a, keys, vals);
    if (a.max_pairs > 0) {
        const uint32_t* d_np = reinterpret_cast<const uint32_t*>(a.scratch) + 3;
        e = sort_pairs16_launch(a.pairs, a.max_pairs, d_np, sm_count, stream);
        if (e != cudaSuccess) return e;
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((a.max_pairs + 255) / 256, 8ull * sm_count));
        splat_ranges_kernel<<<grid, 256, 0, stream>>>(a, keys);
        splat_tile_kernel<<<(unsigned)l.tiles, kSplatThreads, 0, stream>>>(a, vals);
    } else {
        splat_tile_kernel<<<(unsigned)l.tiles, kSplatThreads, 0, stream>>>(a, nullptr);
    }
    return cudaGetLastError();
}

}  // namespace m2s
