// m2s_splat.cuh — arguments and scratch layout of the viewer's splat draw (m2s_splat.cu), shared with the C-ABI host code
// (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

constexpr int kSplatTile = 16;                           // screen tiles of 16 x 16 pixels, one CTA per tile
constexpr int kSplatThreads = kSplatTile * kSplatTile;   // tile kernel: one thread per pixel
constexpr uint32_t kSplatMaxSide = 4096;                 // 256 x 256 tiles: a tile id fits in 16 bits
constexpr uint64_t kSplatMaxCount = 1ull << 30;
constexpr uint64_t kSplatMaxPairs = 1ull << 30;          // the pair sort's count limit (kSortMaxCount)

// the 16 x 16 tiles of a W x H viewport
__host__ __device__ inline uint64_t splat_tiles(uint32_t width, uint32_t height) {
    return (uint64_t)((width + kSplatTile - 1) / kSplatTile) * ((height + kSplatTile - 1) / kSplatTile);
}

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
    unsigned long long max_pairs;   // pair budget (< kSplatMaxPairs)
    unsigned char* scratch;         // bin_layout(count, splat_tiles(width, height)) (m2s_bin.cuh)
    uint32_t* pairs;                // SortLayout(max_pairs) words (m2s_sort.cuh): the pair keys and values and their sort
};

// ---- shared with the cube raster of the shadow pass (m2s_light.cu) and the mesh depth pre-pass (m2s_depth.cu) ---
// ---- the rasteriser's set-up (DESIGN §2): viewport transform, 1/256 snap, sign-normalised edge functions ----------
// E_k(i, j) = A_k i + B_k j + C_k at the centre of pixel (i, j); inside iff E_k >= 0 where the edge owns its samples
// (top-left rule), E_k > 0 elsewhere.  |X|, |Y| <= 2^21, so |A|, |B| <= 2^30 fit 32 bits.
struct SplatTri {
    int32_t A[3], B[3];
    long long C[3];
    bool incl[3];
    int x0, x1, y0, y1;   // candidate pixel box, empty if x1 < x0 (also for a dropped or degenerate triangle)
};

// the viewport transform xw = ndc * (W/2) + W/2 and the 1/256 snap; ok is false outside the +-8192 guard band
__device__ __forceinline__ void splat_snap(float nx, float ny, float hw, float hh, bool& ok, int& X, int& Y) {
    const float xw = __fadd_rn(__fmul_rn(nx, hw), hw), yw = __fadd_rn(__fmul_rn(ny, hh), hh);
    ok = isfinite(xw) && isfinite(yw) && fabsf(xw) <= 8192.0f && fabsf(yw) <= 8192.0f;
    X = ok ? __float2int_rn(__fmul_rn(xw, 256.0f)) : 0;
    Y = ok ? __float2int_rn(__fmul_rn(yw, 256.0f)) : 0;
}

__device__ __forceinline__ void splat_corner(const float4& m, const float4& s, float vx, float vy, float hw, float hh,
                                             bool& ok, int& X, int& Y) {
    // gaussianSplattingVS.glsl:32: mean.xy + (vx * scale.xy + vy * scale.zw)
    const float nx = __fadd_rn(m.x, __fadd_rn(__fmul_rn(vx, s.x), __fmul_rn(vy, s.z)));
    const float ny = __fadd_rn(m.y, __fadd_rn(__fmul_rn(vx, s.y), __fmul_rn(vy, s.w)));
    splat_snap(nx, ny, hw, hh, ok, X, Y);
}

__device__ inline void splat_tri_setup(const int X[3], const int Y[3], bool ok, int W, int H, SplatTri& t) {
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

// the quad's two triangles, (V0, V1, V2) and (V0, V2, V3) with V0..V3 = (-1,-1), (-1,1), (1,1), (1,-1)
__device__ inline void splat_quad_setup(const float4* q, int W, int H, SplatTri t[2]) {
    const float4 m = q[0], s = q[1];
    const float hw = __fmul_rn((float)W, 0.5f), hh = __fmul_rn((float)H, 0.5f);
    const float vx[4] = {-1.0f, -1.0f, 1.0f, 1.0f}, vy[4] = {-1.0f, 1.0f, 1.0f, -1.0f};
    int X[4], Y[4];
    bool ok[4];
#pragma unroll
    for (int v = 0; v < 4; ++v) splat_corner(m, s, vx[v], vy[v], hw, hh, ok[v], X[v], Y[v]);
    const int X0[3] = {X[0], X[1], X[2]}, Y0[3] = {Y[0], Y[1], Y[2]};
    const int X1[3] = {X[0], X[2], X[3]}, Y1[3] = {Y[0], Y[2], Y[3]};
    splat_tri_setup(X0, Y0, ok[0] && ok[1] && ok[2], W, H, t[0]);
    splat_tri_setup(X1, Y1, ok[0] && ok[2] && ok[3], W, H, t[1]);
}

// can the triangle cover a pixel centre of tile (tx, ty)?  Each edge function's largest value over the pixel box where
// the tile meets the triangle's candidate box (conservative: a tile that passes may still be empty)
__device__ __forceinline__ bool splat_tri_touches(const SplatTri& t, int tx, int ty) {
    const int a0 = max(t.x0, tx * kSplatTile), a1 = min(t.x1, tx * kSplatTile + kSplatTile - 1);
    const int b0 = max(t.y0, ty * kSplatTile), b1 = min(t.y1, ty * kSplatTile + kSplatTile - 1);
    if (a1 < a0 || b1 < b0) return false;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const long long e = (long long)t.A[k] * (t.A[k] > 0 ? a1 : a0) + (long long)t.B[k] * (t.B[k] > 0 ? b1 : b0) + t.C[k];
        if (e < 0 || (e == 0 && !t.incl[k])) return false;
    }
    return true;
}

// visits the tiles the quad touches in tile-id order; returns their number
template <typename F>
__device__ __forceinline__ uint32_t splat_for_each_tile(const SplatTri t[2], int tiles_x, F&& f) {
    const bool e0 = t[0].x1 < t[0].x0 || t[0].y1 < t[0].y0, e1 = t[1].x1 < t[1].x0 || t[1].y1 < t[1].y0;
    if (e0 && e1) return 0;
    const int x0 = e0 ? t[1].x0 : (e1 ? t[0].x0 : min(t[0].x0, t[1].x0));
    const int x1 = e0 ? t[1].x1 : (e1 ? t[0].x1 : max(t[0].x1, t[1].x1));
    const int y0 = e0 ? t[1].y0 : (e1 ? t[0].y0 : min(t[0].y0, t[1].y0));
    const int y1 = e0 ? t[1].y1 : (e1 ? t[0].y1 : max(t[0].y1, t[1].y1));
    uint32_t c = 0;
    for (int ty = y0 / kSplatTile; ty <= y1 / kSplatTile; ++ty)
        for (int tx = x0 / kSplatTile; tx <= x1 / kSplatTile; ++tx)
            if (splat_tri_touches(t[0], tx, ty) || splat_tri_touches(t[1], tx, ty)) f(c++, (uint32_t)(ty * tiles_x + tx));
    return c;
}

// exp(x) from round-to-nearest fp32 operations only (the same steps as the oracle's orc_splat_exp): x = k ln2 + r with a
// two-part ln2 (Cody-Waite), a degree-7 polynomial for e^r, then 2^k applied in two exact-or-once-rounded multiplies.
__device__ __forceinline__ float splat_exp(float x) {
    if (x != x) return x;
    if (x > 88.72283905206835f) return __int_as_float(0x7f800000);
    if (x < -103.97208f) return 0.0f;
    const float fk = rintf(__fmul_rn(x, 1.44269504088896341f));
    float r = __fsub_rn(x, __fmul_rn(fk, 0.693359375f));
    r = __fsub_rn(r, __fmul_rn(fk, -2.12194440e-4f));
    const float z = __fmul_rn(r, r);
    float p = 1.9875691500e-4f;
    p = __fadd_rn(__fmul_rn(p, r), 1.3981999507e-3f);
    p = __fadd_rn(__fmul_rn(p, r), 8.3334519073e-3f);
    p = __fadd_rn(__fmul_rn(p, r), 4.1665795894e-2f);
    p = __fadd_rn(__fmul_rn(p, r), 1.6666665459e-1f);
    p = __fadd_rn(__fmul_rn(p, r), 5.0000001201e-1f);
    p = __fadd_rn(__fadd_rn(__fmul_rn(p, z), r), 1.0f);
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return __fmul_rn(__fmul_rn(p, __int_as_float((k1 + 127) << 23)), __int_as_float((k2 + 127) << 23));
}

// counts the (tile, quad) pairs of the n quads and scans them (bin_count_launch); the total lands in the ctrl words
cudaError_t splat_count_launch(const SplatArgs& a, cudaStream_t stream);
// emits and sorts the pairs of the longest prefix that fits max_pairs (bin_pairs_launch), then draws every tile
cudaError_t splat_draw_launch(const SplatArgs& a, int sm_count, cudaStream_t stream);

}  // namespace m2s
