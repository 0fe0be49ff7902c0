// m2s_3dgs.cu — the standard 3DGS render (beyond the reference): graphdeco's forward pass (Kerbl et al. 2023,
// diff-gaussian-rasterization preprocessCUDA + renderCUDA) for the project's GL camera, as DESIGN §2 fixes it.  The
// picture a downstream 3DGS renderer makes of exported or loaded gaussians.
//
// Shape, on one stream with no host synchronisation:
//   gs3d_preprocess_kernel  one thread per record: decode, view, cull, 2-D covariance, conic, radius, tile rectangle,
//                           colour (SH when given); one 48-byte splat record and the depth key (culled: kGs3dCulled,
//                           past every survivor, so the order never depends on atomic arrival)
//   sort_order_launch       the depth sort's onesweep kernels (m2s_sort.cu): the records in (depth key, index) order
//   binning (m2s_bin.cuh)   per survivor in depth order: its rectangle's tiles in tile-id order; the pairs of the longest
//                           prefix that fits the budget, stably sorted by tile, so each tile's run is depth-ordered
//   gs3d_tile_kernel        one CTA per tile, one thread per pixel: front-to-back compositing in registers, the tile
//                           stops once every pixel has terminated; one coalesced store per target
// All arithmetic that decides a bit of the image is round-to-nearest fp32 with no contraction (__f*_rn) and rn_exp, so
// the images equal the checker's (oracle/m2s_3dgs_oracle.c) bit for bit.
#include "m2s_3dgs.cuh"
#include "m2s_bin.cuh"
#include "m2s_gauss.cuh"

namespace m2s {

constexpr int kGs3dThreads = 256;

// row r of the column-major 4 x 4 m applied to (x, y, z, 1): ((m_r0 x + m_r1 y) + m_r2 z) + m_r3
__device__ __forceinline__ float gs3d_row(const float* m, int r, float x, float y, float z) {
    return ad(ad(ad(ml(m[r], x), ml(m[4 + r], y)), ml(m[8 + r], z)), m[12 + r]);
}

// one record -> its splat record and depth key (DESIGN §2, the 3DGS render: per record); false if culled
__device__ __forceinline__ bool gs3d_splat(const Gs3dArgs& a, unsigned long long gid, Gs3dSplat& out, uint32_t& key) {
    GaussFields g;
    if (a.layout == 0) {
        const float4* r = reinterpret_cast<const float4*>(a.records) + gid * 6;
        ref96_fields(__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3), __ldg(r + 4), __ldg(r + 5), g);
    } else {
        const float2* r = reinterpret_cast<const float2*>(a.records + gid * 56ull);
        packed56_fields<true>(__ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3), __ldg(r + 4), __ldg(r + 5), __ldg(r + 6), g);
    }
    // ---- view and cull ----
    const float tx = gs3d_row(a.MV, 0, g.px, g.py, g.pz), ty = gs3d_row(a.MV, 1, g.px, g.py, g.pz), tz = gs3d_row(a.MV, 2, g.px, g.py, g.pz);
    const float d = -tz;
    if (!(d > a.near)) return false;
    // ---- mean in pixels (ndc2Pix) ----
    const float c0 = gs3d_row(a.P, 0, tx, ty, tz), c1 = gs3d_row(a.P, 1, tx, ty, tz), c3 = gs3d_row(a.P, 3, tx, ty, tz);
    const float pw = dv(1.0f, ad(c3, 1e-7f));
    const float W = (float)a.width, H = (float)a.height;
    const float u = ml(sb(ml(ad(ml(c0, pw), 1.0f), W), 1.0f), 0.5f), v = ml(sb(ml(ad(ml(c1, pw), 1.0f), H), 1.0f), 0.5f);
    // ---- 3-D covariance (computeCov3D): scale, normalised rotation, Sigma = (S R^T)^T (S R^T) ----
    const float s[3] = {ml(ml(g.sx, a.mult), a.scale_modifier), ml(ml(g.sy, a.mult), a.scale_modifier), ml(ml(g.sz, a.mult), a.scale_modifier)};
    const float qn = fmaxf(__fsqrt_rn(ad(ad(ad(ml(g.qx, g.qx), ml(g.qy, g.qy)), ml(g.qz, g.qz)), ml(g.qw, g.qw))), 1e-12f);
    const float qr = dv(g.qx, qn), qi = dv(g.qy, qn), qj = dv(g.qz, qn), qk = dv(g.qw, qn);   // (w, x, y, z)
    const float R[3][3] = {{sb(1.0f, ml(2.0f, ad(ml(qj, qj), ml(qk, qk)))), ml(2.0f, sb(ml(qi, qj), ml(qr, qk))), ml(2.0f, ad(ml(qi, qk), ml(qr, qj)))},
                           {ml(2.0f, ad(ml(qi, qj), ml(qr, qk))), sb(1.0f, ml(2.0f, ad(ml(qi, qi), ml(qk, qk)))), ml(2.0f, sb(ml(qj, qk), ml(qr, qi)))},
                           {ml(2.0f, sb(ml(qi, qk), ml(qr, qj))), ml(2.0f, ad(ml(qj, qk), ml(qr, qi))), sb(1.0f, ml(2.0f, ad(ml(qi, qi), ml(qj, qj))))}};
    float Mk[3][3];   // Mk[k][j] = s_k R[j][k]
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j) Mk[k][j] = ml(s[k], R[j][k]);
    float S[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) S[i][j] = ad(ad(ml(Mk[0][i], Mk[0][j]), ml(Mk[1][i], Mk[1][j])), ml(Mk[2][i], Mk[2][j]));
    // ---- 2-D covariance (computeCov2D in GL axes): cov = J W Sigma W^T J^T + 0.3 I ----
    const float fx = ml(ml(a.P[0], W), 0.5f), fy = ml(ml(a.P[5], H), 0.5f);
    const float limx = dv(1.3f, a.P[0]), limy = dv(1.3f, a.P[5]);
    const float txc = ml(fminf(limx, fmaxf(-limx, dv(tx, d))), d), tyc = ml(fminf(limy, fmaxf(-limy, dv(ty, d))), d);
    const float dd = ml(d, d);
    const float J00 = dv(fx, d), J02 = dv(ml(fx, txc), dd), J11 = dv(fy, d), J12 = dv(ml(fy, tyc), dd);
    float T[2][3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        T[0][j] = ad(ml(J00, a.MV[4 * j + 0]), ml(J02, a.MV[4 * j + 2]));
        T[1][j] = ad(ml(J11, a.MV[4 * j + 1]), ml(J12, a.MV[4 * j + 2]));
    }
    float A[2][3];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) A[i][j] = ad(ad(ml(T[i][0], S[0][j]), ml(T[i][1], S[1][j])), ml(T[i][2], S[2][j]));
    auto cov = [&](int i, int j) { return ad(ad(ml(A[i][0], T[j][0]), ml(A[i][1], T[j][1])), ml(A[i][2], T[j][2])); };
    const float ca = ad(cov(0, 0), 0.3f), cb = cov(0, 1), cc = ad(cov(1, 1), 0.3f);
    // ---- conic, radius, tile rectangle (getRect) ----
    const float det = sb(ml(ca, cc), ml(cb, cb));
    if (det == 0.0f) return false;
    const float inv = dv(1.0f, det);
    const float mid = ml(0.5f, ad(ca, cc));
    const float sq = __fsqrt_rn(fmaxf(0.1f, sb(ml(mid, mid), det)));
    const float radius = ceilf(ml(3.0f, __fsqrt_rn(fmaxf(ad(mid, sq), sb(mid, sq)))));
    const int gx = (int)tiles_x(a.width), gy = (int)tiles_x(a.height);
    const int x0 = min(gx, max(0, __float2int_rz(ml(sb(u, radius), 0.0625f))));
    const int y0 = min(gy, max(0, __float2int_rz(ml(sb(v, radius), 0.0625f))));
    const int x1 = min(gx, max(0, __float2int_rz(ml(ad(ad(u, radius), 15.0f), 0.0625f))));
    const int y1 = min(gy, max(0, __float2int_rz(ml(ad(ad(v, radius), 15.0f), 0.0625f))));
    if ((x1 - x0) * (y1 - y0) == 0) return false;
    // ---- colour ----
    float r = g.cr, gg = g.cg, b = g.cb;
    if (a.sh_degree) sh_colour(a.sh, a.sh_vec4, a.sh_degree, a.cam, gid, g.px, g.py, g.pz, r, gg, b);
    else { r = r < 0.0f ? 0.0f : r; gg = gg < 0.0f ? 0.0f : gg; b = b < 0.0f ? 0.0f : b; }
    out.a = make_float4(u, v, ml(cc, inv), ml(-cb, inv));
    out.b = make_float4(ml(ca, inv), g.ca, r, gg);
    out.c = make_float4(b, __uint_as_float((uint32_t)x0 | (uint32_t)x1 << 16), __uint_as_float((uint32_t)y0 | (uint32_t)y1 << 16), radius);
    key = __float_as_uint(d);
    return true;
}

__global__ void __launch_bounds__(kGs3dThreads) gs3d_preprocess_kernel(const __grid_constant__ Gs3dArgs a) {
    unsigned long long n = a.count;
    if (a.d_count) n = min(n, *a.d_count);
    const unsigned long long gid = (unsigned long long)blockIdx.x * kGs3dThreads + threadIdx.x;
    if (gid == 0) a.ctrl[0] = (uint32_t)n;
    if ((unsigned long long)blockIdx.x * kGs3dThreads >= n) return;   // whole warps leave together: the ballot below is full
    Gs3dSplat sp = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
    uint32_t key = kGs3dCulled;
    const bool alive = gid < n && gs3d_splat(a, gid, sp, key);
    if (gid < n) {
        a.splats[gid] = sp;
        a.keys[gid] = key;
    }
    const unsigned mask = __ballot_sync(0xffffffffu, alive);
    if ((threadIdx.x & 31) == 0 && mask) atomicAdd(a.ctrl + 1, (uint32_t)__popc(mask));
}

// ---- binning (m2s_bin.cuh): the survivors in depth order, pair value = record index ---------------------------------------
struct Gs3dBins {
    Gs3dArgs a;
    __host__ __device__ unsigned long long items() const { return a.count; }
    __host__ __device__ uint64_t tiles() const { return tile_count(a.width, a.height); }
    __device__ __forceinline__ uint32_t n() const { return a.ctrl[1]; }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        const uint32_t id = a.order[i];
        const float4 c = a.splats[id].c;
        const uint32_t rx = __float_as_uint(c.y), ry = __float_as_uint(c.z);
        const uint32_t x0 = rx & 0xFFFFu, x1 = rx >> 16, y0 = ry & 0xFFFFu, y1 = ry >> 16, tx = tiles_x(a.width);
        for (uint32_t ty = y0; ty < y1; ++ty)
            for (uint32_t t = x0; t < x1; ++t) f(ty * tx + t, id);
        return (x1 - x0) * (y1 - y0);
    }
};

// ---- tile kernel: front-to-back compositing (renderCUDA) ------------------------------------------------------------------
constexpr int kGs3dVaryings = 9;   // u, v, conic.xyz, opacity, r, g, b
struct Gs3dStage {
    float v[kGs3dVaryings][kTileThreads];
};

__global__ void __launch_bounds__(kTileThreads) gs3d_tile_kernel(Gs3dArgs a, const uint32_t* __restrict__ vals) {
    __shared__ Gs3dStage s;
    const TileFrame f = tile_frame(a.scratch, bin_layout(a.count, tile_count(a.width, a.height)), tiles_x(a.width), blockIdx.x);
    const bool inside = f.x < (int)a.width && f.y < (int)a.height;
    const float px = (float)f.x, py = (float)f.y;
    float T = 1.0f, C0 = 0.0f, C1 = 0.0f, C2 = 0.0f;
    bool done = !inside;
    auto stage = [&](int tid, uint32_t val) {
        const Gs3dSplat sp = a.splats[val];
        s.v[0][tid] = sp.a.x; s.v[1][tid] = sp.a.y; s.v[2][tid] = sp.a.z; s.v[3][tid] = sp.a.w;
        s.v[4][tid] = sp.b.x; s.v[5][tid] = sp.b.y; s.v[6][tid] = sp.b.z; s.v[7][tid] = sp.b.w; s.v[8][tid] = sp.c.x;
    };
    tile_batches(
        f, vals, stage,
        [&](uint32_t j) {
            if (done) return;
            const float dx = sb(s.v[0][j], px), dy = sb(s.v[1][j], py);
            const float power = sb(ml(-0.5f, ad(ml(ml(s.v[2][j], dx), dx), ml(ml(s.v[4][j], dy), dy))), ml(ml(s.v[3][j], dx), dy));
            if (power > 0.0f) return;
            const float alpha = fminf(0.99f, ml(s.v[5][j], rn_exp(power)));
            if (alpha < 1.0f / 255.0f) return;
            const float tt = ml(T, sb(1.0f, alpha));
            if (tt < 0.0001f) { done = true; return; }
            C0 = ad(C0, ml(ml(s.v[6][j], alpha), T));
            C1 = ad(C1, ml(ml(s.v[7][j], alpha), T));
            C2 = ad(C2, ml(ml(s.v[8][j], alpha), T));
            T = tt;
        },
        [&] { return done; });
    if (!inside) return;
    const float4 o = make_float4(ad(C0, ml(T, a.bg[0])), ad(C1, ml(T, a.bg[1])), ad(C2, ml(T, a.bg[2])), sb(1.0f, T));
    const size_t pix = (size_t)f.y * a.width + f.x;
    if (a.rgba32f) a.rgba32f[pix] = o;
    if (a.rgba8) a.rgba8[pix] = unorm8(o.x) | unorm8(o.y) << 8 | unorm8(o.z) << 16 | unorm8(o.w) << 24;
}

// ---- launches ------------------------------------------------------------------------------------------------------------
cudaError_t gs3d_preprocess_launch(const Gs3dArgs& a, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(a.ctrl, 0, 8, stream);   // n, survivors
    if (e != cudaSuccess || a.count == 0) return e;
    gs3d_preprocess_kernel<<<(unsigned)((a.count + kGs3dThreads - 1) / kGs3dThreads), kGs3dThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t gs3d_count_launch(const Gs3dArgs& a, cudaStream_t stream) {
    cudaError_t e = gs3d_preprocess_launch(a, stream);
    if (e != cudaSuccess) return e;
    e = sort_order_launch(a.keys, a.count, a.ctrl, a.order, a.sort_scratch, a.sm_count, stream);
    if (e != cudaSuccess) return e;
    return bin_count_launch(Gs3dBins{a}, stream);
}

cudaError_t gs3d_draw_launch(const Gs3dArgs& a, int sm_count, cudaStream_t stream) {
    return bin_draw_launch(Gs3dBins{a}, gs3d_tile_kernel, sm_count, stream);
}

}  // namespace m2s
