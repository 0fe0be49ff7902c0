// m2s_span.cuh — exact coverage of one pixel row of a triangle's candidate box as an interval.
//
// The rasteriser's rule (GL 4.6 14.6.1, restated in oracle/m2s_oracle.c): pixel (x, y) of the box is covered iff
// E'_k(x, y) = E_k(x, y) - (edge k owns its zero set ? 0 : 1) >= 0 for the three sign-normalised integer edge
// functions E_k = A_k x + B_k y + C_k.  For a fixed row the covered set is the intersection of three half-lines,
// i.e. ONE interval [xl, xl + n): it is computed here with three estimated divisions, each corrected by exact
// int64 evaluations, so the result is bit-identical to testing every pixel centre — at O(1) per row instead
// of O(width).  Used by raster_kernel (to count) and fragment_kernel (to enumerate); also compiled for the host
// by tests/test_span_host.py (g++), which checks it against the brute-force per-pixel test.
// box_mask: the same rule over the whole candidate box of a small triangle, as the raster kernel's 64-bit coverage mask
// (host check: tests/test_box_mask_host.py).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define M2S_HD __host__ __device__ __forceinline__
#else
#define M2S_HD inline
#endif

namespace m2s {

struct RowState {   // one triangle, relative to the origin (x0, y0) of its candidate box
    long long E[3]; // E'_k at the box origin (ownership bias folded in: covered <=> all E' >= 0)
    int A[3];       // dE_k/dx per pixel
    int B[3];       // dE_k/dy per pixel
    int w;          // box width in pixels (1..4096)
};

M2S_HD float span_quot(long long num, int den) {  // estimate of num / den, num >= 0, den > 0
#if defined(__CUDA_ARCH__)
    return __fdividef(__ll2float_rn(num), __int2float_rn(den));
#else
    return (float)num / (float)den;
#endif
}

// Row `yrel` (0-based inside the box): returns the number of covered pixels, xl = first covered column.
M2S_HD uint32_t span_row(const RowState& s, int yrel, int& xl) {
    int lo = 0, hi = s.w - 1;
    const float wlim = (float)s.w + 2.0f;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int k = 0; k < 3; ++k) {
        const long long D = s.E[k] + (long long)s.B[k] * yrel;  // E'_k at column 0 of this row
        const int A = s.A[k];
        if (A == 0) {
            if (D < 0) hi = -1;
        } else if (A > 0) {             // covered for x >= ceil(-D / A)
            if (D < 0) {
                const float qf = span_quot(-D, A);
                if (!(qf < wlim)) hi = -1;      // the boundary lies right of the box (also catches inf/NaN)
                else {
                    int x = (int)qf;
                    long long e = D + (long long)A * x;
                    while (e < 0) { ++x; e += A; }                     // exact fix-up of the estimate
                    while (x > 0 && e - A >= 0) { --x; e -= A; }
                    lo = lo > x ? lo : x;
                }
            }
        } else {                        // covered for x <= floor(D / -A)
            if (D < 0) hi = -1;
            else {
                const float qf = span_quot(D, -A);
                if (qf < wlim) {                // else: no constraint inside the box
                    int x = (int)qf + 1;
                    long long e = D + (long long)A * x;
                    while (e < 0) { --x; e -= A; }                     // A < 0: stepping left raises e
                    while (e + A >= 0) { ++x; e += A; }
                    hi = hi < x ? hi : x;
                }
            }
        }
    }
    xl = lo;
    return hi >= lo ? (uint32_t)(hi - lo + 1) : 0u;
}

// ---- small triangles: the whole candidate box as one 64-bit mask ----
M2S_HD uint32_t push_outside(uint32_t acc, uint32_t f) {   // acc << 1 | the sign bit of f
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(f, acc, 1);
#else
    return (acc << 1) | (f >> 31);
#endif
}
M2S_HD uint32_t bit_reverse(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __brev(v);
#else
    v = ((v >> 1) & 0x55555555u) | ((v & 0x55555555u) << 1);
    v = ((v >> 2) & 0x33333333u) | ((v & 0x33333333u) << 2);
    v = ((v >> 4) & 0x0f0f0f0fu) | ((v & 0x0f0f0f0fu) << 4);
    v = ((v >> 8) & 0x00ff00ffu) | ((v & 0x00ff00ffu) << 8);
    return (v >> 16) | (v << 16);
#endif
}

// The coverage of a candidate box of at most 64 pixels whose E' values all fit in int32 (the raster kernel's small
// triangles, one per lane): bit row * w + column is set iff that pixel is covered, by the rule of span_row.  e: E' at the
// box origin; a, b: the steps of E' per column and per row; w: the box width; n: its pixels (w * h; 0: none).  The lanes
// of a warp walk in lock step, maxc >= n candidates (the largest n among them), row-major with incremental edge functions,
// 4 per loop step.  A candidate's outside bit enters a 32-bit word by a funnel shift (no variable 64-bit shift per
// candidate); only the step to the next row depends on the box.  Unsigned arithmetic: the walk past n may wrap, its bits
// are dropped.
M2S_HD unsigned long long box_mask(int e0, int e1, int e2, int a0, int a1, int a2, int b0, int b1, int b2, int w, uint32_t n,
                                   uint32_t maxc) {
    const uint32_t s0 = (uint32_t)a0, s1 = (uint32_t)a1, s2 = (uint32_t)a2;
    const uint32_t r0 = (uint32_t)b0 - (uint32_t)(w - 1) * s0, r1 = (uint32_t)b1 - (uint32_t)(w - 1) * s1,
                   r2 = (uint32_t)b2 - (uint32_t)(w - 1) * s2;   // last pixel of a row -> first pixel of the next
    uint32_t f0 = (uint32_t)e0, f1 = (uint32_t)e1, f2 = (uint32_t)e2;
    uint32_t end = (uint32_t)w - 1u;   // the candidate that ends the current row
    const uint32_t last = (maxc + 3u) & ~3u;   // the walk ends on a multiple of 4 candidates
    unsigned long long in = 0;
    for (uint32_t c0 = 0; c0 < last; c0 += 32u) {   // 32-candidate words
        const uint32_t stop = last < c0 + 32u ? last : c0 + 32u;
        uint32_t out = 0;   // outside bits of the word's candidates, the latest one in bit 0
        for (uint32_t c = c0; c < stop; c += 4u) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
            for (uint32_t j = 0; j < 4u; ++j) {
                out = push_outside(out, f0 | f1 | f2);
                const bool wrap = c + j == end;
                end += wrap ? (uint32_t)w : 0u;
                f0 += wrap ? r0 : s0; f1 += wrap ? r1 : s1; f2 += wrap ? r2 : s2;
            }
        }
        in |= (unsigned long long)~(bit_reverse(out) >> (32u - (stop - c0))) << c0;
    }
    const unsigned long long all = n >= 64u ? ~0ull : (1ull << n) - 1ull;
    return in & all;
}

}  // namespace m2s
