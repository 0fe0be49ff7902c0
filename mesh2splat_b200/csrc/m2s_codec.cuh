// m2s_codec.cuh — the per-value encodings of the .ply and PACKED56 outputs and the decodings of the .ply loader, in one
// place: the conversion's shading (raster and fragment kernels), ply_rows_kernel (m2s_ply_encode) and the .ply decode
// kernel include this header and nothing else computes these values.  m2s_debug_codec_eval evaluates each function
// elementwise, so the tests compare them with glibc on every input bit pattern.
//
// Every function returns what the reference computes on x86-64 with glibc (2.28 or later, the FMA variant of expf /
// logf that glibc selects on a CPU with FMA and AVX2), bit for bit, NaN as NaN:
//   sh0_encode     (c - 0.5f) / SH_COEFF0                             utils.cpp:47 (getShFromColor)
//   opacity_logit  -std::log(1.0f / (clamp(a, 0, 1) + 1e-8f) - 1.0f)  utils.hpp:270 (invSigmoid)
//   log_scale      std::log(s * mult)                                 parsers.cpp:497-499
//   sh0_decode     f * SH_COEFF0 + 0.5f                               utils.cpp:53 (getColorFromSh)
//   ref_expf       std::exp(x)                                        parsers.cpp:590-592 (glm::exp of the scales)
//   opacity_sigmoid 1.0 / (1.0 + std::exp(-o)), the exp in fp32       utils.hpp:269
// CUDA's own logf / expf are up to 1 / 2 ulp away from glibc's, __logf and __fdividef further, and a multiply by the
// fp32 reciprocal of SH_COEFF0 differs from the division in about one value of six.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

constexpr float kShC0 = 0.28209479177387814f;  // SH_COEFF0 (params.hpp:17)

// ---- glibc's logf and expf (the table-driven fp64 algorithms of ARM's optimized-routines, glibc >= 2.28) ----
// logf: x = 2^k z, z in [0x3f330000, 2 * that) split into 16 subintervals with c near each centre; log(x) =
// log1p(z / c - 1) + log(c) + k ln2, log1p by a degree-3 polynomial in fp64, one rounding to fp32 at the end.
// kLogfTab: (1 / c, log(c)) of each subinterval, as the bits of glibc's __logf_data.tab.
static __device__ const double kLogfTab[32] = {
    0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2, 0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2,
    0x1.49539f0f010bp+0,  -0x1.01eae7f513a67p-2, 0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3,
    0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3, 0x1.25e227b0b8eap+0,  -0x1.1aa2bc79c81p-3,
    0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4, 0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4,
    0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5, 0x1p+0,               0x0p+0,
    0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5,  0x1.ca4b31f026aap-1,  0x1.c5e53aa362eb4p-4,
    0x1.b2036576afce6p-1, 0x1.526e57720db08p-3,  0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3,
    0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2,  0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2};
__device__ __forceinline__ float ref_logf(float x) {
    uint32_t ix = __float_as_uint(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {   // subnormal, zero, negative, inf or NaN
        if (ix * 2u == 0u) return __int_as_float(0xff800000);             // +-0 -> -inf
        if (ix == 0x7f800000u) return x;                                  // +inf
        if ((ix & 0x80000000u) || ix * 2u >= 0xff000000u) return __int_as_float(0x7fc00000);   // NaN
        ix = __float_as_uint(__fmul_rn(x, 0x1p23f)) - (23u << 23);       // subnormal: normalise
    }
    const uint32_t tmp = ix - 0x3f330000u;
    const int i = (int)((tmp >> 19) & 15u), k = (int32_t)tmp >> 23;
    const double z = (double)__uint_as_float(ix - (tmp & 0xff800000u));
    const double invc = __ldg(kLogfTab + 2 * i), logc = __ldg(kLogfTab + 2 * i + 1);
    const double kLn2 = 0x1.62e42fefa39efp-1, kA0 = -0x1.00ea348b88334p-2, kA1 = 0x1.5575b0be00b6ap-2, kA2 = -0x1.ffffef20a4123p-2;
    const double r = __fma_rn(z, invc, -1.0);
    const double y0 = __dadd_rn(logc, __dmul_rn((double)k, kLn2));
    const double r2 = __dmul_rn(r, r);
    double y = __fma_rn(kA1, r, kA2);
    y = __fma_rn(kA0, r2, y);
    y = __fma_rn(y, r2, __dadd_rn(y0, r));
    return __double2float_rn(y);
}

// expf: x N / ln2 = k + r, exp(x) = 2^(k/N) (C0 r^3 + C1 r^2 + C2 r + 1), N = 32, the reduction and the polynomial fused,
// one rounding to fp32 at the end (denormal results kept).  tab: kExp2Tab or a copy of it (the .ply decoder keeps one in
// shared memory).
static __device__ const unsigned long long kExp2Tab[32] = {   // the bits of 2^(i/32) rounded to fp64, minus i << 47
    0x3ff0000000000000ULL, 0x3fefd9b0d3158574ULL, 0x3fefb5586cf9890fULL, 0x3fef9301d0125b51ULL,
    0x3fef72b83c7d517bULL, 0x3fef54873168b9aaULL, 0x3fef387a6e756238ULL, 0x3fef1e9df51fdee1ULL,
    0x3fef06fe0a31b715ULL, 0x3feef1a7373aa9cbULL, 0x3feedea64c123422ULL, 0x3feece086061892dULL,
    0x3feebfdad5362a27ULL, 0x3feeb42b569d4f82ULL, 0x3feeab07dd485429ULL, 0x3feea47eb03a5585ULL,
    0x3feea09e667f3bcdULL, 0x3fee9f75e8ec5f74ULL, 0x3feea11473eb0187ULL, 0x3feea589994cce13ULL,
    0x3feeace5422aa0dbULL, 0x3feeb737b0cdc5e5ULL, 0x3feec49182a3f090ULL, 0x3feed503b23e255dULL,
    0x3feee89f995ad3adULL, 0x3feeff76f2fb5e47ULL, 0x3fef199bdd85529cULL, 0x3fef3720dcef9069ULL,
    0x3fef5818dcfba487ULL, 0x3fef7c97337b9b5fULL, 0x3fefa4afa2a490daULL, 0x3fefd0765b6e4540ULL};
__device__ __forceinline__ float ref_expf(float x, const unsigned long long* tab) {
    const uint32_t ux = __float_as_uint(x), abstop = (ux >> 20) & 0x7ffu;
    if (abstop >= 0x42bu) {                            // |x| >= 88 or NaN
        if (ux == 0xff800000u) return 0.0f;            // -inf
        if (abstop >= 0x7f8u) return x + x;            // +inf, NaN
        if (x > 0x1.62e42ep6f) return __int_as_float(0x7f800000);   // overflow
        if (x < -0x1.9fe368p6f) return 0.0f;           // underflow
    }
    const double kInvLn2N = 0x1.71547652b82fep+0 * 32, kShift = 0x1.8p+52;
    const double kC0 = 0x1.c6af84b912394p-5 / (32.0 * 32.0 * 32.0), kC1 = 0x1.ebfce50fac4f3p-3 / (32.0 * 32.0), kC2 = 0x1.62e42ff0c52d6p-1 / 32.0;
    const double xd = (double)x;
    double kd = __dadd_rn(__dmul_rn(kInvLn2N, xd), kShift);
    const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
    kd = __dsub_rn(kd, kShift);
    const double r = __fma_rn(kInvLn2N, xd, -kd);
    const double s = __longlong_as_double((long long)(tab[ki & 31u] + (ki << 47)));
    const double z = __fma_rn(kC0, r, kC1), r2 = __dmul_rn(r, r);
    const double y = __fma_rn(z, r2, __fma_rn(kC2, r, 1.0));
    return __double2float_rn(__dmul_rn(y, s));
}

// ---- the writer's encodings ----
// The IEEE quotient d / SH_COEFF0 without a division: the product with the rounded reciprocal, corrected once by its
// fused residual, is the correctly rounded quotient for every finite one (checked on all 2^32 inputs, test_gpu_codec.py);
// an infinite or NaN product is the quotient already.
__device__ __forceinline__ float sh0_encode(float c) {
    const float kInvShC0 = __uint_as_float(0x4062dfc4u);   // 1.0f / SH_COEFF0, rounded to nearest
    const float d = __fsub_rn(c, 0.5f), q = __fmul_rn(d, kInvShC0);
    return isfinite(q) ? __fmaf_rn(__fmaf_rn(-q, kShC0, d), kInvShC0, q) : q;
}
// std::clamp keeps a NaN alpha (NaN < 0 and 1 < NaN are false), so NaN encodes to NaN; alpha 1 encodes to +inf.
// __frcp_rn is the IEEE 1.0f / x.
__device__ __forceinline__ float opacity_logit(float a) {
    a = a < 0.0f ? 0.0f : (1.0f < a ? 1.0f : a);
    return -ref_logf(__fsub_rn(__frcp_rn(__fadd_rn(a, 1e-8f)), 1.0f));
}
__device__ __forceinline__ float log_scale(float s, float mult) { return ref_logf(__fmul_rn(s, mult)); }

// ---- the loader's decodings ----
__device__ __forceinline__ float sh0_decode(float f) { return __fadd_rn(__fmul_rn(f, kShC0), 0.5f); }
__device__ __forceinline__ float opacity_sigmoid(float o, const unsigned long long* tab) {
    return __double2float_rn(__ddiv_rn(1.0, __dadd_rn(1.0, (double)ref_expf(-o, tab))));
}

}  // namespace m2s
