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
// The forward pass that keeps its state for the backward pass (m2s_3dgs_grad.cu) runs the same steps with
// gs3d_rank_kernel (the inverse of the depth order) after the sort and gs3d_tile_kernel<true>, which also stores each
// pixel's final T and last contributor; gs3d_tile_kernel<false> is the render's kernel unchanged.
// All arithmetic that decides a bit of the image is round-to-nearest fp32 with no contraction (__f*_rn) and rn_exp, so
// the images equal the checker's (oracle/m2s_3dgs_oracle.c) bit for bit.
#include "m2s_3dgs.cuh"
#include "m2s_3dgs_proj.cuh"
#include "m2s_bin.cuh"

namespace m2s {

constexpr int kGs3dThreads = 256;

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
    Gs3dProj pr;
    if (!gs3d_project(a, g, pr)) return false;
    const float u = pr.u, v = pr.v, ca = pr.ca, cb = pr.cb, cc = pr.cc, d = pr.d;
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
template <typename A>
struct Gs3dBinner {
    A a;
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
struct Gs3dBins : Gs3dBinner<Gs3dArgs> {};
struct Gs3dSaveBins : Gs3dBinner<Gs3dSaveArgs> {};   // the same pairs; the arguments carry the forward state

// ---- tile kernel: front-to-back compositing (renderCUDA) ------------------------------------------------------------------
struct Gs3dStage {
    float v[kGs3dVaryings][kTileThreads];
};

// kSave: also the per-pixel state of the backward pass (a.final_T, a.n_contrib); kSave = false is the render's kernel
template <bool kSave>
__global__ void __launch_bounds__(kTileThreads) gs3d_tile_kernel(std::conditional_t<kSave, Gs3dSaveArgs, Gs3dArgs> a,
                                                                  const uint32_t* __restrict__ vals) {
    __shared__ Gs3dStage s;
    const TileFrame f = tile_frame(a.scratch, bin_layout(a.count, tile_count(a.width, a.height)), tiles_x(a.width), blockIdx.x);
    const bool inside = f.x < (int)a.width && f.y < (int)a.height;
    const float px = (float)f.x, py = (float)f.y;
    float T = 1.0f, C0 = 0.0f, C1 = 0.0f, C2 = 0.0f;
    bool done = !inside;
    uint32_t seen = 0, last = 0;   // kSave: the run positions this pixel has visited, 1 + its last blended one
    auto stage = [&](int tid, uint32_t val) {
        const Gs3dSplat sp = a.splats[val];
        s.v[0][tid] = sp.a.x; s.v[1][tid] = sp.a.y; s.v[2][tid] = sp.a.z; s.v[3][tid] = sp.a.w;
        s.v[4][tid] = sp.b.x; s.v[5][tid] = sp.b.y; s.v[6][tid] = sp.b.z; s.v[7][tid] = sp.b.w; s.v[8][tid] = sp.c.x;
    };
    tile_batches(
        f, vals, stage,
        [&](uint32_t j) {
            if (done) return;
            if constexpr (kSave) ++seen;
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
            if constexpr (kSave) last = seen;
        },
        [&] { return done; });
    if (!inside) return;
    const float4 o = make_float4(ad(C0, ml(T, a.bg[0])), ad(C1, ml(T, a.bg[1])), ad(C2, ml(T, a.bg[2])), sb(1.0f, T));
    const size_t pix = (size_t)f.y * a.width + f.x;
    if (a.rgba32f) a.rgba32f[pix] = o;
    if (a.rgba8) a.rgba8[pix] = unorm8(o.x) | unorm8(o.y) << 8 | unorm8(o.z) << 16 | unorm8(o.w) << 24;
    if constexpr (kSave) {
        a.final_T[pix] = T;
        a.n_contrib[pix] = last;
    }
}

// the inverse of the depth order: rank[order[k]] = k
__global__ void __launch_bounds__(kGs3dThreads) gs3d_rank_kernel(const uint32_t* __restrict__ order, uint32_t* __restrict__ rank,
                                                                  unsigned long long count) {
    const unsigned long long k = (unsigned long long)blockIdx.x * kGs3dThreads + threadIdx.x;
    if (k < count) rank[order[k]] = (uint32_t)k;
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
    return bin_count_launch(Gs3dBins{{a}}, stream);
}

cudaError_t gs3d_draw_launch(const Gs3dArgs& a, int sm_count, cudaStream_t stream) {
    return bin_draw_launch(Gs3dBins{{a}}, gs3d_tile_kernel<false>, sm_count, stream);
}

cudaError_t gs3d_count_save_launch(const Gs3dSaveArgs& a, cudaStream_t stream) {
    cudaError_t e = gs3d_preprocess_launch(a, stream);
    if (e != cudaSuccess) return e;
    e = sort_order_launch(a.keys, a.count, a.ctrl, a.order, a.sort_scratch, a.sm_count, stream);
    if (e != cudaSuccess) return e;
    e = bin_count_launch(Gs3dSaveBins{{a}}, stream);
    if (e != cudaSuccess || a.count == 0) return e;
    gs3d_rank_kernel<<<(unsigned)((a.count + kGs3dThreads - 1) / kGs3dThreads), kGs3dThreads, 0, stream>>>(a.order, a.rank, a.count);
    return cudaGetLastError();
}

cudaError_t gs3d_draw_save_launch(const Gs3dSaveArgs& a, int sm_count, cudaStream_t stream) {
    return bin_draw_launch(Gs3dSaveBins{{a}}, gs3d_tile_kernel<true>, sm_count, stream);
}

}  // namespace m2s
