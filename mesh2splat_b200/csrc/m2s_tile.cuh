// m2s_tile.cuh — what the viewer's four tiled rasterisers share: the splat draw (m2s_splat.cu), the shadow pass's cube
// raster (m2s_light.cu), the mesh depth pre-pass (m2s_depth.cu) and the mesh G-buffer pass (m2s_mesh.cu).  The 16 x 16
// tiles, the rasteriser's set-up (DESIGN §2: viewport transform, 1/256 snap, sign-normalised edge functions), the tile
// tests and walks, the quad staging of the splat and shadow tile kernels, and the formats of the depth and G-buffer
// targets.  Every operation is round-to-nearest fp32 / fp64 with no contraction, so the oracles restate it bit for bit.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace m2s {

constexpr int kTile = 16;                            // screen tiles of 16 x 16 pixels, one CTA per tile
constexpr int kTileThreads = kTile * kTile;          // tile kernels: one thread per pixel
constexpr uint32_t kTileMaxSide = 4096;              // 256 x 256 tiles: a tile id fits in 16 bits
constexpr uint64_t kTileMaxPairs = 1ull << 30;       // the pair sort's count limit (kSortMaxCount)

// the tiles of one row of a viewport `width` pixels wide, and the tiles of a W x H viewport
__host__ __device__ inline uint32_t tiles_x(uint32_t width) { return (width + kTile - 1) / kTile; }
__host__ __device__ inline uint64_t tile_count(uint32_t width, uint32_t height) { return (uint64_t)tiles_x(width) * tiles_x(height); }

// round-to-nearest fp32 operations, never contracted
__device__ __forceinline__ float ad(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sb(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ml(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dv(float a, float b) { return __fdiv_rn(a, b); }

// ---- the rasteriser's set-up ---------------------------------------------------------------------------------------
// E_k(i, j) = A_k i + B_k j + C_k at the centre of pixel (i, j); inside iff E_k >= 0 where the edge owns its samples
// (top-left rule), E_k > 0 elsewhere.  |X|, |Y| <= 2^21, so |A|, |B| <= 2^30 fit 32 bits.
struct TileTri {
    int32_t A[3], B[3];
    long long C[3];
    bool incl[3];
    int x0, x1, y0, y1;   // candidate pixel box, empty if x1 < x0 (also for a dropped or degenerate triangle)
};

// the viewport transform xw = ndc * (W/2) + W/2 and the 1/256 snap; ok is false outside the +-8192 guard band
__device__ __forceinline__ void tile_snap(float nx, float ny, float hw, float hh, bool& ok, int& X, int& Y) {
    const float xw = ad(ml(nx, hw), hw), yw = ad(ml(ny, hh), hh);
    ok = isfinite(xw) && isfinite(yw) && fabsf(xw) <= 8192.0f && fabsf(yw) <= 8192.0f;
    X = ok ? __float2int_rn(ml(xw, 256.0f)) : 0;
    Y = ok ? __float2int_rn(ml(yw, 256.0f)) : 0;
}

__device__ inline void tile_tri_setup(const int X[3], const int Y[3], bool ok, int W, int H, TileTri& t) {
    t.x0 = 0; t.x1 = -1; t.y0 = 0; t.y1 = -1;
    for (int k = 0; k < 3; ++k) { t.A[k] = 0; t.B[k] = 0; t.C[k] = -1; t.incl[k] = false; }
    if (!ok) return;
    const long long area2 = (long long)(X[1] - X[0]) * (Y[2] - Y[0]) - (long long)(X[2] - X[0]) * (Y[1] - Y[0]);
    if (area2 == 0) return;
    const long long sg = area2 < 0 ? -1 : 1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        const long long dx = X[b] - X[a], dy = Y[b] - Y[a];
        t.A[k] = (int32_t)(sg * (-dy * 256));
        t.B[k] = (int32_t)(sg * (dx * 256));
        t.C[k] = sg * (dx * (128 - (long long)Y[a]) - dy * (128 - (long long)X[a]));
        t.incl[k] = t.A[k] > 0 || (t.A[k] == 0 && t.B[k] > 0);
    }
    const int xmin = min(X[0], min(X[1], X[2])), xmax = max(X[0], max(X[1], X[2]));
    const int ymin = min(Y[0], min(Y[1], Y[2])), ymax = max(Y[0], max(Y[1], Y[2]));
    t.x0 = max((xmin + 127) >> 8, 0); t.x1 = min((xmax - 128) >> 8, W - 1);
    t.y0 = max((ymin + 127) >> 8, 0); t.y1 = min((ymax - 128) >> 8, H - 1);
}

// a quad (q[0] = mean, q[1] = the two axes, NDC) as two triangles, (V0, V1, V2) and (V0, V2, V3) with V0..V3 = (-1,-1),
// (-1,1), (1,1), (1,-1); corner = mean.xy + (vx * scale.xy + vy * scale.zw) (gaussianSplattingVS.glsl:32)
__device__ inline void tile_quad_setup(const float4* q, int W, int H, TileTri t[2]) {
    const float4 m = q[0], s = q[1];
    const float hw = ml((float)W, 0.5f), hh = ml((float)H, 0.5f);
    const float vx[4] = {-1.0f, -1.0f, 1.0f, 1.0f}, vy[4] = {-1.0f, 1.0f, 1.0f, -1.0f};
    int X[4], Y[4];
    bool ok[4];
#pragma unroll
    for (int v = 0; v < 4; ++v) {
        const float nx = ad(m.x, ad(ml(vx[v], s.x), ml(vy[v], s.z)));
        const float ny = ad(m.y, ad(ml(vx[v], s.y), ml(vy[v], s.w)));
        tile_snap(nx, ny, hw, hh, ok[v], X[v], Y[v]);
    }
    const int X0[3] = {X[0], X[1], X[2]}, Y0[3] = {Y[0], Y[1], Y[2]};
    const int X1[3] = {X[0], X[2], X[3]}, Y1[3] = {Y[0], Y[2], Y[3]};
    tile_tri_setup(X0, Y0, ok[0] && ok[1] && ok[2], W, H, t[0]);
    tile_tri_setup(X1, Y1, ok[0] && ok[2] && ok[3], W, H, t[1]);
}

// ---- tile tests and walks ------------------------------------------------------------------------------------------
// can the triangle cover a pixel centre of tile (tx, ty)?  Each edge function's largest value over the pixel box where
// the tile meets the triangle's candidate box (conservative: a tile that passes may still be empty)
__device__ __forceinline__ bool tile_touches(const TileTri& t, int tx, int ty) {
    const int a0 = max(t.x0, tx * kTile), a1 = min(t.x1, tx * kTile + kTile - 1);
    const int b0 = max(t.y0, ty * kTile), b1 = min(t.y1, ty * kTile + kTile - 1);
    if (a1 < a0 || b1 < b0) return false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const long long e = (long long)t.A[k] * (t.A[k] > 0 ? a1 : a0) + (long long)t.B[k] * (t.B[k] > 0 ? b1 : b0) + t.C[k];
        if (e < 0 || (e == 0 && !t.incl[k])) return false;
    }
    return true;
}

// visits the tiles the quad touches in tile-id order, f(index, tile); returns their number
template <typename F>
__device__ __forceinline__ uint32_t tile_walk_quad(const TileTri t[2], int tiles_x, F&& f) {
    const bool e0 = t[0].x1 < t[0].x0 || t[0].y1 < t[0].y0, e1 = t[1].x1 < t[1].x0 || t[1].y1 < t[1].y0;
    if (e0 && e1) return 0;
    const int x0 = e0 ? t[1].x0 : (e1 ? t[0].x0 : min(t[0].x0, t[1].x0));
    const int x1 = e0 ? t[1].x1 : (e1 ? t[0].x1 : max(t[0].x1, t[1].x1));
    const int y0 = e0 ? t[1].y0 : (e1 ? t[0].y0 : min(t[0].y0, t[1].y0));
    const int y1 = e0 ? t[1].y1 : (e1 ? t[0].y1 : max(t[0].y1, t[1].y1));
    uint32_t c = 0;
    for (int ty = y0 / kTile; ty <= y1 / kTile; ++ty)
        for (int tx = x0 / kTile; tx <= x1 / kTile; ++tx)
            if (tile_touches(t[0], tx, ty) || tile_touches(t[1], tx, ty)) f(c++, (uint32_t)(ty * tiles_x + tx));
    return c;
}

// visits the tiles the triangle touches in tile-id order, f(index, tile); returns their number
template <typename F>
__device__ __forceinline__ uint32_t tile_walk_tri(const TileTri& t, int tiles_x, F&& f) {
    if (t.x1 < t.x0 || t.y1 < t.y0) return 0;
    uint32_t c = 0;
    for (int ty = t.y0 / kTile; ty <= t.y1 / kTile; ++ty)
        for (int tx = t.x0 / kTile; tx <= t.x1 / kTile; ++tx)
            if (tile_touches(t, tx, ty)) f(c++, (uint32_t)(ty * tiles_x + tx));
    return c;
}

// ---- quad staging (the splat and shadow tile kernels) ---------------------------------------------------------------
// per staged quad: both triangles' edge functions relative to the tile origin, with the top-left rule folded into C
// (E >= 0 inside)
struct QuadEdges {
    int32_t A[6][kTileThreads], B[6][kTileThreads];
    long long C[6][kTileThreads];
};

__device__ __forceinline__ void quad_stage(const TileTri t[2], int ox, int oy, QuadEdges& s, int slot) {
#pragma unroll
    for (int e = 0; e < 6; ++e) {
        const TileTri& tt = t[e / 3];
        const int k = e % 3;
        s.A[e][slot] = tt.A[k];
        s.B[e][slot] = tt.B[k];
        s.C[e][slot] = tt.C[k] + (long long)tt.A[k] * ox + (long long)tt.B[k] * oy - (tt.incl[k] ? 0 : 1);
    }
}

// does triangle tri (0 or 1) of staged quad j cover pixel (lx, ly) of the tile?
__device__ __forceinline__ bool quad_tri_in(const QuadEdges& s, uint32_t j, int tri, int lx, int ly) {
    bool in = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int e = tri * 3 + k;
        in &= s.C[e][j] + (long long)s.A[e][j] * lx + (long long)s.B[e][j] * ly >= 0;
    }
    return in;
}

// how many of staged quad j's two triangles cover pixel (lx, ly) of the tile: 0, 1 or 2
__device__ __forceinline__ int quad_cover(const QuadEdges& s, uint32_t j, int lx, int ly) {
    return (int)quad_tri_in(s, j, 0, lx, ly) + (int)quad_tri_in(s, j, 1, lx, ly);
}

// ---- exp and the target formats (DESIGN §2) --------------------------------------------------------------------------
// exp(x) from round-to-nearest fp32 operations only (the same steps as the oracle's orc_splat_exp): x = k ln2 + r with a
// two-part ln2 (Cody-Waite), a degree-7 polynomial for e^r, then 2^k applied in two exact-or-once-rounded multiplies.
__device__ __forceinline__ float rn_exp(float x) {
    if (x != x) return x;
    if (x > 88.72283905206835f) return __int_as_float(0x7f800000);
    if (x < -103.97208f) return 0.0f;
    const float fk = rintf(ml(x, 1.44269504088896341f));
    float r = sb(x, ml(fk, 0.693359375f));
    r = sb(r, ml(fk, -2.12194440e-4f));
    const float z = ml(r, r);
    float p = 1.9875691500e-4f;
    p = ad(ml(p, r), 1.3981999507e-3f);
    p = ad(ml(p, r), 8.3334519073e-3f);
    p = ad(ml(p, r), 4.1665795894e-2f);
    p = ad(ml(p, r), 1.6666665459e-1f);
    p = ad(ml(p, r), 5.0000001201e-1f);
    p = ad(ad(ml(p, z), r), 1.0f);
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return ml(ml(p, __int_as_float((k1 + 127) << 23)), __int_as_float((k2 + 127) << 23));
}

// D24: round-half-even(clamp(z, 0, 1) * (2^24 - 1)), the product exact in fp64; false for NaN (no write).  The depth
// targets store code / (2^24 - 1) as a float and are cleared to the code kD24Clear (1.0).
constexpr uint32_t kD24Clear = 0xFFFFFFu;
__device__ __forceinline__ bool d24_encode(double z, uint32_t& code) {
    if (z != z) return false;
    const double zc = z < 0.0 ? 0.0 : (z > 1.0 ? 1.0 : z);
    code = __double2uint_rn(__dmul_rn(zc, 16777215.0));
    return true;
}
__device__ __forceinline__ float d24_decode(uint32_t code) { return dv(__uint2float_rn(code), 16777215.0f); }

// fp32 -> fp16 bits, round to nearest even; overflow gives +-inf, NaN gives 0x7FFF, subnormals are kept
__device__ __forceinline__ float to_half(float v, uint16_t& bits) {
    if (v != v) { bits = 0x7FFFu; return v; }
    const __half h = __float2half_rn(v);
    bits = __half_as_ushort(h);
    return __half2float(h);
}

// an RGBA16F texel: four fp16 bits in two words
__device__ __forceinline__ uint2 half4(float x, float y, float z, float w) {
    uint16_t h[4];
    to_half(x, h[0]); to_half(y, h[1]); to_half(z, h[2]); to_half(w, h[3]);
    return make_uint2(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16);
}

// RGBA8 channels are clamped to [0, 1] and stored as round-half-even(v * 255); NaN clamps to 0
__device__ __forceinline__ float sat(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }
__device__ __forceinline__ uint32_t unorm8(float v) { return __float2uint_rn(ml(sat(v), 255.0f)); }

// the five G-buffer targets of one pixel: RGBA16F as two words of fp16 bits, RGBA8 as one word
struct GTexel {
    uint2 pos, nrm, dep;
    uint32_t alb, mr;
};

// stores texel o at pixel px of every non-NULL target of a (the position, normal, albedo, depth and
// metallic_roughness pointers of SplatArgs and MeshArgs)
template <typename A>
__device__ __forceinline__ void gbuffer_store(const A& a, size_t px, const GTexel& o) {
    if (a.position) reinterpret_cast<uint2*>(a.position)[px] = o.pos;
    if (a.normal) reinterpret_cast<uint2*>(a.normal)[px] = o.nrm;
    if (a.albedo) reinterpret_cast<uint32_t*>(a.albedo)[px] = o.alb;
    if (a.depth) reinterpret_cast<uint2*>(a.depth)[px] = o.dep;
    if (a.metallic_roughness) reinterpret_cast<uint32_t*>(a.metallic_roughness)[px] = o.mr;
}

}  // namespace m2s
