// m2s_compare.cu — how closely two RGBA8 images agree: SSIM, squared error and coverage (beyond the reference, whose
// split screen, GaussianRelightingPass.cpp:90-135, is judged by eye).  The definition (Wang et al. 2004 with an 11 x 11
// Gaussian window, sigma 1.5, valid windows only) and its operation order are DESIGN §2; oracle/m2s_compare_oracle.c
// restates them, and the map equals its map bit for bit.
//
// Shape:
//   compare_tile_kernel    one CTA per tile of 32 x 32 windows: the tile's 42 x 42 pixels of A and B staged in shared
//                          memory; the squared error and coverage of the pixels the tile owns (its window centres, plus
//                          the 5-pixel border of an edge tile); then per channel a horizontal pass (one thread per staged
//                          row and window column) into five moment planes and a vertical pass (each thread four
//                          windows of one column); the tile's totals reduced in a fixed order into one column of the
//                          context's partials
//   compare_total_kernel   one CTA: the partials summed in a fixed order into the m2s_compare_result
// Every fp32 operation that decides a map value is one round-to-nearest operation with no contraction (__f*_rn), so
// two calls, and the kernel and the oracle, agree bit for bit; the fp64 sums depend only on the image size.
#include "m2s_ctx.cuh"

namespace m2s {

constexpr int kCmpTW = 32, kCmpTH = 32;                    // windows per tile
constexpr int kCmpIW = kCmpTW + 10, kCmpIH = kCmpTH + 10;  // staged pixels per tile
constexpr int kCmpThreads = 256;                           // 8 warps: lane = window column, warp = 4 window rows
constexpr int kCmpRows = kCmpTH / (kCmpThreads / 32);      // window rows per thread
constexpr int kCmpTotalThreads = 1024;
constexpr uint32_t kCmpMinSide = 11, kCmpMaxSide = 4096;
// the partial totals of a tile, in this order: sq_err[3], sq_err_covered[3], pixels_both, pixels_a_only, pixels_b_only,
// covered_windows (uint64), then ssim[3], ssim_covered[3] (fp64 bits)
constexpr int kCmpInts = 10, kCmpFields = 16;

// w_i = g_i / sum(g), g_i = exp(-i^2 / 4.5), i = -5..5, in fp64, rounded once to fp32
static __constant__ float kTap[11] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f, 0x1.b43c40p-3f, 0x1.106560p-2f,
                               0x1.b43c40p-3f, 0x1.bff0fep-4f, 0x1.26eb18p-5f, 0x1.f1fe02p-8f, 0x1.0d956cp-10f};
constexpr float kC1 = 0x1.a028f6p+2f;   // (0.01 * 255)^2 rounded once
constexpr float kC2 = 0x1.d42e14p+5f;   // (0.03 * 255)^2 rounded once

struct CompareArgs {
    const uint32_t *a, *b, *cover_a, *cover_b;   // RGBA8 as words; covers may be NULL
    uint32_t width, height, cover_min, tiles_x, tiles;
    unsigned long long windows;
    float* map;                                  // optional
    unsigned long long* part;                    // kCmpFields x tiles, field-major
    m2s_compare_result* result;
};

__device__ __forceinline__ float chan(uint32_t px, int c) { return (float)((px >> (8 * c)) & 255u); }

// a fixed-order sum over the CTA: shuffle tree within each warp, then the warps' sums in warp order by thread f
template <typename T>
__device__ __forceinline__ T warp_tree(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = v + __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

template <int NW>
__device__ void cta_reduce(unsigned long long (&u)[kCmpInts], double (&d)[kCmpFields - kCmpInts], unsigned long long (*red)[kCmpFields],
                           unsigned long long* out, size_t stride) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int f = 0; f < kCmpInts; ++f) u[f] = warp_tree(u[f]);
#pragma unroll
    for (int f = 0; f < kCmpFields - kCmpInts; ++f) d[f] = warp_tree(d[f]);
    if (lane == 0) {
#pragma unroll
        for (int f = 0; f < kCmpInts; ++f) red[warp][f] = u[f];
#pragma unroll
        for (int f = 0; f < kCmpFields - kCmpInts; ++f) red[warp][kCmpInts + f] = __double_as_longlong(d[f]);
    }
    __syncthreads();
    const int f = threadIdx.x;
    if (f < kCmpInts) {
        unsigned long long s = red[0][f];
        for (int w = 1; w < NW; ++w) s += red[w][f];
        out[f * stride] = s;
    } else if (f < kCmpFields) {
        double s = __longlong_as_double(red[0][f]);
        for (int w = 1; w < NW; ++w) s = s + __longlong_as_double(red[w][f]);
        out[f * stride] = __double_as_longlong(s);
    }
}

__global__ void __launch_bounds__(kCmpThreads) compare_tile_kernel(const __grid_constant__ CompareArgs a) {
    __shared__ uint32_t pa[kCmpIH][kCmpIW], pb[kCmpIH][kCmpIW];
    __shared__ float mom[5][kCmpIH][kCmpTW];   // x, y, x x, y y, x y blurred along rows
    __shared__ uint8_t cov[kCmpTH][kCmpTW];    // the window's centre is covered in A or B
    __shared__ unsigned long long red[kCmpThreads / 32][kCmpFields];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int W = (int)a.width, H = (int)a.height, nwx = W - 10, nwy = H - 10;
    const int tx = (int)(blockIdx.x % a.tiles_x), ty = (int)(blockIdx.x / a.tiles_x);
    const int tiles_y = (int)(a.tiles / a.tiles_x);
    const int x0 = tx * kCmpTW, y0 = ty * kCmpTH;   // the staged block's origin: the first window centre minus 5
    const int sw = min(kCmpIW, W - x0), sh = min(kCmpIH, H - y0);
    for (int i = threadIdx.x; i < kCmpIH * kCmpIW; i += kCmpThreads) {
        const int r = i / kCmpIW, c = i - r * kCmpIW;
        uint32_t va = 0u, vb = 0u;
        if (r < sh && c < sw) {
            const size_t o = (size_t)(y0 + r) * W + (x0 + c);
            va = __ldg(a.a + o);
            vb = __ldg(a.b + o);
        }
        pa[r][c] = va;
        pb[r][c] = vb;
    }
    __syncthreads();

    // ---- the pixels the tile owns: its window centres, and the image border beside them on an edge tile ----
    unsigned long long u[kCmpInts] = {};
    double d[kCmpFields - kCmpInts] = {};
    const int ox0 = tx == 0 ? 0 : x0 + 5, ox1 = tx == (int)a.tiles_x - 1 ? W : x0 + 5 + kCmpTW;
    const int oy0 = ty == 0 ? 0 : y0 + 5, oy1 = ty == tiles_y - 1 ? H : y0 + 5 + kCmpTH;
    const int ow = ox1 - ox0, npix = ow * (oy1 - oy0);
    for (int i = threadIdx.x; i < npix; i += kCmpThreads) {
        const int r = i / ow, c = i - r * ow;
        const int sr = oy0 - y0 + r, sc = ox0 - x0 + c;   // staged coordinates
        const uint32_t va = pa[sr][sc], vb = pb[sr][sc];
        uint32_t e[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int dd = (int)((va >> (8 * k)) & 255u) - (int)((vb >> (8 * k)) & 255u);
            e[k] = (uint32_t)(dd * dd);
            u[k] += e[k];
        }
        const size_t o = (size_t)(oy0 + r) * W + (ox0 + c);
        const bool ia = a.cover_a && (__ldg(a.cover_a + o) >> 24) >= a.cover_min;
        const bool ib = a.cover_b && (__ldg(a.cover_b + o) >> 24) >= a.cover_min;
        if (ia || ib) {
#pragma unroll
            for (int k = 0; k < 3; ++k) u[3 + k] += e[k];
        }
        u[6] += ia && ib;
        u[7] += ia && !ib;
        u[8] += ib && !ia;
        const int wc = sc - 5, wr = sr - 5;
        if (wc >= 0 && wc < kCmpTW && wr >= 0 && wr < kCmpTH) cov[wr][wc] = ia || ib;
    }

    // ---- SSIM: per channel, rows then columns ----
    const int wr0 = warp * kCmpRows;
    const bool col_ok = x0 + lane < nwx;
    float m[kCmpRows];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        __syncthreads();   // the previous channel's vertical pass (and the coverage flags) are done
        for (int r = warp; r < kCmpIH; r += kCmpThreads / 32) {
            float s[5];
#pragma unroll
            for (int i = 0; i < 11; ++i) {
                const float x = chan(pa[r][lane + i], ch), y = chan(pb[r][lane + i], ch);
                const float q[5] = {x, y, __fmul_rn(x, x), __fmul_rn(y, y), __fmul_rn(x, y)};
#pragma unroll
                for (int k = 0; k < 5; ++k) s[k] = i == 0 ? __fmul_rn(kTap[0], q[k]) : __fadd_rn(s[k], __fmul_rn(kTap[i], q[k]));
            }
#pragma unroll
            for (int k = 0; k < 5; ++k) mom[k][r][lane] = s[k];
        }
        __syncthreads();
        float v[kCmpRows][5];
#pragma unroll
        for (int j = 0; j < kCmpRows + 10; ++j) {
            float t[5];
#pragma unroll
            for (int k = 0; k < 5; ++k) t[k] = mom[k][wr0 + j][lane];
#pragma unroll
            for (int w = 0; w < kCmpRows; ++w) {
                const int tap = j - w;
                if (tap < 0 || tap > 10) continue;
#pragma unroll
                for (int k = 0; k < 5; ++k) v[w][k] = tap == 0 ? __fmul_rn(kTap[0], t[k]) : __fadd_rn(v[w][k], __fmul_rn(kTap[tap], t[k]));
            }
        }
#pragma unroll
        for (int w = 0; w < kCmpRows; ++w) {
            if (!col_ok || y0 + wr0 + w >= nwy) continue;
            const float mx = v[w][0], my = v[w][1];
            const float mx2 = __fmul_rn(mx, mx), my2 = __fmul_rn(my, my), mxy = __fmul_rn(mx, my);
            const float vx = __fsub_rn(v[w][2], mx2), vy = __fsub_rn(v[w][3], my2), cxy = __fsub_rn(v[w][4], mxy);
            const float num = __fmul_rn(__fadd_rn(__fmul_rn(2.0f, mxy), kC1), __fadd_rn(__fmul_rn(2.0f, cxy), kC2));
            const float den = __fmul_rn(__fadd_rn(__fadd_rn(mx2, my2), kC1), __fadd_rn(__fadd_rn(vx, vy), kC2));
            const float s = __fdiv_rn(num, den);
            m[w] = ch == 0 ? s : __fadd_rn(m[w], s);
            d[ch] += (double)s;
            if (cov[wr0 + w][lane]) {
                d[3 + ch] += (double)s;
                if (ch == 0) ++u[9];
            }
        }
    }
    if (a.map) {
#pragma unroll
        for (int w = 0; w < kCmpRows; ++w)
            if (col_ok && y0 + wr0 + w < nwy) a.map[(size_t)(y0 + wr0 + w) * nwx + (x0 + lane)] = __fdiv_rn(m[w], 3.0f);
    }
    cta_reduce<kCmpThreads / 32>(u, d, red, a.part + blockIdx.x, a.tiles);
}

__global__ void __launch_bounds__(kCmpTotalThreads) compare_total_kernel(const __grid_constant__ CompareArgs a) {
    __shared__ unsigned long long red[kCmpTotalThreads / 32][kCmpFields];
    __shared__ unsigned long long tot[kCmpFields];
    unsigned long long u[kCmpInts] = {};
    double d[kCmpFields - kCmpInts] = {};
    for (uint32_t t = threadIdx.x; t < a.tiles; t += kCmpTotalThreads) {
#pragma unroll
        for (int f = 0; f < kCmpInts; ++f) u[f] += a.part[(size_t)f * a.tiles + t];
#pragma unroll
        for (int f = 0; f < kCmpFields - kCmpInts; ++f) d[f] = d[f] + __longlong_as_double(a.part[(size_t)(kCmpInts + f) * a.tiles + t]);
    }
    cta_reduce<kCmpTotalThreads / 32>(u, d, red, tot, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        m2s_compare_result* r = a.result;
        r->windows = a.windows;
        r->covered_windows = tot[9];
        r->pixels_both = tot[6];
        r->pixels_a_only = tot[7];
        r->pixels_b_only = tot[8];
        for (int k = 0; k < 3; ++k) {
            r->sq_err[k] = tot[k];
            r->sq_err_covered[k] = tot[3 + k];
            r->ssim[k] = __longlong_as_double(tot[kCmpInts + k]);
            r->ssim_covered[k] = __longlong_as_double(tot[kCmpInts + 3 + k]);
        }
    }
}

static size_t compare_scratch_bytes(uint32_t tiles) { return (size_t)kCmpFields * sizeof(unsigned long long) * tiles; }

static m2s_status compare_check(const m2s_ctx* ctx, const uint8_t* d_a, const uint8_t* d_b, const uint8_t* d_cover_a,
                                const uint8_t* d_cover_b, const m2s_compare_params* p, bool has_result, const float* d_map) {
    const char* fn = "m2s_image_compare";
    if (!ctx || !d_a || !d_b || !p || !has_result) return invalid(fn, "NULL argument");
    if (p->width < kCmpMinSide || p->width > kCmpMaxSide || p->height < kCmpMinSide || p->height > kCmpMaxSide)
        return invalid(fn, "width and height must be 11..4096");
    if (p->cover_min < 1 || p->cover_min > 255) return invalid(fn, "cover_min must be 1..255");
    return aligned_ok(fn, "the images, covers and map must be 4-byte aligned",
                      {{d_a, 4}, {d_b, 4}, {d_cover_a, 4}, {d_cover_b, 4}, {d_map, 4}})
               ? M2S_OK
               : M2S_E_INVALID;
}

// after compare_check: the two kernels on `stream`, the partials in the context's scratch
static m2s_status compare_launch(m2s_ctx* ctx, const uint8_t* d_a, const uint8_t* d_b, const uint8_t* d_cover_a, const uint8_t* d_cover_b,
                                 const m2s_compare_params* p, m2s_compare_result* d_result, float* d_map, cudaStream_t stream) {
    CompareArgs a;
    a.a = reinterpret_cast<const uint32_t*>(d_a);
    a.b = reinterpret_cast<const uint32_t*>(d_b);
    a.cover_a = reinterpret_cast<const uint32_t*>(d_cover_a);
    a.cover_b = reinterpret_cast<const uint32_t*>(d_cover_b);
    a.width = p->width;
    a.height = p->height;
    a.cover_min = p->cover_min;
    a.tiles_x = (p->width - 10 + kCmpTW - 1) / kCmpTW;
    a.tiles = a.tiles_x * ((p->height - 10 + kCmpTH - 1) / kCmpTH);
    a.windows = (unsigned long long)(p->width - 10) * (p->height - 10);
    a.map = d_map;
    a.result = d_result;
    const m2s_status st = grow(ctx, ctx->compare, compare_scratch_bytes(a.tiles), stream);
    if (st != M2S_OK) return st;
    a.part = static_cast<unsigned long long*>(ctx->compare.p);
    compare_tile_kernel<<<a.tiles, kCmpThreads, 0, stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    compare_total_kernel<<<1, kCmpTotalThreads, 0, stream>>>(a);
    CUDA_TRY(cudaGetLastError());
    return M2S_OK;
}

}  // namespace m2s

using namespace m2s;

M2S_EXPORT m2s_status m2s_image_compare_enqueue(m2s_ctx* ctx, const uint8_t* d_a, const uint8_t* d_b, const uint8_t* d_cover_a,
                                                const uint8_t* d_cover_b, const m2s_compare_params* p, m2s_compare_result* d_result,
                                                float* d_ssim_map, void* stream) {
    m2s_status st = compare_check(ctx, d_a, d_b, d_cover_a, d_cover_b, p, d_result != nullptr, d_ssim_map);
    if (st != M2S_OK) return st;
    if (!aligned_ok("m2s_image_compare", "the result must be 8-byte aligned", {{d_result, 8}})) return M2S_E_INVALID;
    CUDA_TRY(cudaSetDevice(ctx->device));
    return compare_launch(ctx, d_a, d_b, d_cover_a, d_cover_b, p, d_result, d_ssim_map, pick_stream(ctx, stream));
}

M2S_EXPORT m2s_status m2s_image_compare(m2s_ctx* ctx, const uint8_t* d_a, const uint8_t* d_b, const uint8_t* d_cover_a,
                                        const uint8_t* d_cover_b, const m2s_compare_params* p, m2s_compare_result* h_result,
                                        float* d_ssim_map) {
    m2s_status st = compare_check(ctx, d_a, d_b, d_cover_a, d_cover_b, p, h_result != nullptr, d_ssim_map);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaSetDevice(ctx->device));
    // the result goes through the context's own device word, behind the partials
    const uint32_t tiles = ((p->width - 10 + kCmpTW - 1) / kCmpTW) * ((p->height - 10 + kCmpTH - 1) / kCmpTH);
    st = grow(ctx, ctx->compare, compare_scratch_bytes(tiles) + sizeof(m2s_compare_result), ctx->stream);
    if (st != M2S_OK) return st;
    m2s_compare_result* d_result =
        reinterpret_cast<m2s_compare_result*>(static_cast<unsigned char*>(ctx->compare.p) + compare_scratch_bytes(tiles));
    st = compare_launch(ctx, d_a, d_b, d_cover_a, d_cover_b, p, d_result, d_ssim_map, ctx->stream);
    if (st != M2S_OK) return st;
    m2s_compare_result r;
    CUDA_TRY(cudaMemcpyAsync(&r, d_result, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *h_result = r;
    return M2S_OK;
}
