// m2s_light.cu — the viewer's lighting (SURVEY 8 f-7, f-8): the two passes after the splat draw.
//
// f-7 GaussianShadowPass::execute (src/renderer/renderPasses/GaussianShadowPass.cpp:83-236): the light prepass
// (gaussianPointShadowMappingCS.glsl:58-207 + common.glsl) and six face draws (gaussianPointLightCubeMapShadowVS.glsl /
// ...PS.glsl) into a D24 cube map cleared to 1, depth test LESS.
// f-8 GaussianRelightingPass::execute (GaussianRelightingPass.cpp:42-150): a full-screen pass over the G-buffer
// (gaussianSplattingDeferredPS.glsl:32-165) into RGBA8.
//
// Shape:
//   light_prepass_kernel   one thread per source record: one 32-byte light record in source order (no per-face append)
//   binning (m2s_bin.cuh)  per record: the 16 x 16 tiles of its face its two triangles touch (the splat draw's test
//                          over 6 faces); (tile, record) pairs of the longest prefix that fits the budget, stably sorted
//                          by tile; each tile's run
//   shadow_tile_kernel     one CTA per tile, one thread per texel: the minimum depth code in registers (depth is constant
//                          per quad and the test is LESS, so the result does not depend on draw order), one store
//   deferred_light_kernel  one thread per pixel: fetch, shade, RGBA8
// Every operation that decides a bit of the output is round-to-nearest fp32 with no contraction (__f*_rn), integer, or
// one of the conversions of DESIGN §2, so the records, the cube and the image equal the oracle's
// (oracle/m2s_light_oracle.c) bit for bit.
#include <cuda_fp16.h>

#include "m2s_bin.cuh"
#include "m2s_light.cuh"

namespace m2s {

__device__ __forceinline__ float ad(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sb(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ml(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float dot3(float x, float y, float z) { return ad(ad(ml(x, x), ml(y, y)), ml(z, z)); }   // GLM dot(v, v)

// GLM mat3 * mat3, column-major: r[c][row] = (a[0][row] b[c][0] + a[1][row] b[c][1]) + a[2][row] b[c][2]
__device__ __forceinline__ void light_m3mul(const float* a, const float* b, float* r) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int row = 0; row < 3; ++row)
            r[c * 3 + row] = ad(ad(ml(a[row], b[c * 3]), ml(a[3 + row], b[c * 3 + 1])), ml(a[6 + row], b[c * 3 + 2]));
}

// GLM mat4 * vec4(x, y, z, 1): (m0 x + m1 y) + (m2 z + m3 1)
__device__ __forceinline__ float light_m4row(const float* m, int row, float x, float y, float z, float w) {
    return ad(ad(ml(m[row], x), ml(m[4 + row], y)), ad(ml(m[8 + row], z), ml(m[12 + row], w)));
}

// determineFaceIndex (gaussianPointShadowMappingCS.glsl:58-69) and the cube sampler's major axis (DESIGN §2): x wins
// ties over y and z, y over z; a NaN component fails every comparison and falls through to z, sign "> 0" else negative
__device__ __forceinline__ int light_face(float x, float y, float z) {
    const float ax = fabsf(x), ay = fabsf(y), az = fabsf(z);
    if (ax >= ay && ax >= az) return x > 0.0f ? 0 : 1;
    if (ay >= ax && ay >= az) return y > 0.0f ? 2 : 3;
    return z > 0.0f ? 4 : 5;
}

// ---- light prepass --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLightPrepassThreads) light_prepass_kernel(const __grid_constant__ ShadowArgs a) {
    unsigned long long n = a.count;
    if (a.d_count) n = min(n, *a.d_count);
    const unsigned long long gid = (unsigned long long)blockIdx.x * kLightPrepassThreads + threadIdx.x;
    if (gid >= n) return;
    float px, py, pz, sx, sy, sz, qx, qy, qz, qw;
    if (a.layout == 0) {   // REF96: position color scale normal rotation pbr
        const float4* g = reinterpret_cast<const float4*>(a.records) + gid * 6;
        const float4 p = __ldg(g), s = __ldg(g + 2), q = __ldg(g + 4);
        px = p.x; py = p.y; pz = p.z; sx = s.x; sy = s.y; sz = s.z; qx = q.x; qy = q.y; qz = q.z; qw = q.w;
    } else {               // PACKED56: xyz | quat wxyz | log-scale | SH0 | opacity logit; scale = exp (DESIGN §2's exp)
        const float2* g = reinterpret_cast<const float2*>(a.records + gid * 56ull);
        const float2 f0 = __ldg(g), f1 = __ldg(g + 1), f2 = __ldg(g + 2), f3 = __ldg(g + 3), f4 = __ldg(g + 4);
        px = f0.x; py = f0.y; pz = f1.x; qx = f1.y; qy = f2.x; qz = f2.y; qw = f3.x;
        sx = splat_exp(f3.y); sy = splat_exp(f4.x); sz = splat_exp(f4.y);
    }
    float4 o0 = make_float4(0.f, 0.f, 0.f, 0.f), o1 = make_float4(0.f, 0.f, 0.f, __uint_as_float(kShadowCulled));
    // :80-82 world position, face from normalize(ws - light)
    const float w0 = light_m4row(a.M, 0, px, py, pz, 1.0f), w1 = light_m4row(a.M, 1, px, py, pz, 1.0f), w2 = light_m4row(a.M, 2, px, py, pz, 1.0f);
    const float dx = sb(w0, a.light[0]), dy = sb(w1, a.light[1]), dz = sb(w2, a.light[2]);
    const float dd = dot3(dx, dy, dz), inv = dv(1.0f, __fsqrt_rn(dd));
    const int face = light_face(ml(dx, inv), ml(dy, inv), ml(dz, inv));
    const float* V = a.V[face];
    const float v0 = light_m4row(V, 0, w0, w1, w2, 1.0f), v1 = light_m4row(V, 1, w0, w1, w2, 1.0f), v2 = light_m4row(V, 2, w0, w1, w2, 1.0f),
                v3 = light_m4row(V, 3, w0, w1, w2, 1.0f);
    const float c0 = light_m4row(a.P, 0, v0, v1, v2, v3), c1 = light_m4row(a.P, 1, v0, v1, v2, v3), c2 = light_m4row(a.P, 2, v0, v1, v2, v3),
                c3 = light_m4row(a.P, 3, v0, v1, v2, v3);
    const float clip = ml(1.05f, c3);   // :89-94
    bool alive = !(c2 < -clip || c0 < -clip || c0 > clip || c1 < -clip || c1 > clip);
    if (alive) {
        const float mult = a.fmt == 0 ? a.std_dev : 1.0f;      // :96-98
        const float s[3] = {ml(ml(sx, mult), a.mscale2[0]), ml(ml(sy, mult), a.mscale2[1]), ml(ml(sz, mult), a.mscale2[2])};
        // castQuatToMat3 (common.glsl:22-48): the three "rows" are the columns; quat = (w, x, y, z) in (x, y, z, w)
        const float rot0[9] = {sb(1.f, ml(2.f, ad(ml(qz, qz), ml(qw, qw)))), ml(2.f, sb(ml(qy, qz), ml(qx, qw))), ml(2.f, ad(ml(qy, qw), ml(qx, qz))),
                               ml(2.f, ad(ml(qy, qz), ml(qx, qw))), sb(1.f, ml(2.f, ad(ml(qy, qy), ml(qw, qw)))), ml(2.f, sb(ml(qz, qw), ml(qx, qy))),
                               ml(2.f, sb(ml(qy, qw), ml(qx, qz))), ml(2.f, ad(ml(qz, qw), ml(qx, qy))), sb(1.f, ml(2.f, ad(ml(qy, qy), ml(qz, qz))))};
        float rot[9], S[9] = {s[0], 0.f, 0.f, 0.f, s[1], 0.f, 0.f, 0.f, s[2]}, mm[9], mmT[9], cov[9];
        light_m3mul(rot0, a.Rinv, rot);   // :110
        light_m3mul(S, rot, mm);          // computeCov3D (common.glsl:50-61)
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int k = 0; k < 3; ++k) mmT[c * 3 + k] = mm[k * 3 + c];
        light_m3mul(mmT, mm, cov);
        // :160-176 EWA projection with the renderer's resolution (sic)
        const float tzSq = ml(v2, v2), two_z = ml(2.0f, v2), two_tz = ml(2.0f, tzSq);
        const float jsx = dv(-ml(a.P[0], a.res[0]), two_z), jsy = dv(-ml(a.P[5], a.res[1]), two_z);
        const float jtx = dv(ml(ml(a.P[0], v0), a.res[0]), two_tz), jty = dv(ml(ml(a.P[5], v1), a.res[1]), two_tz);
        const float jtz = dv(ml(sb(a.near_far[1], a.near_far[0]), a.P[14]), two_tz);
        const float J[9] = {jsx, 0.f, 0.f, 0.f, jsy, 0.f, jtx, jty, jtz};
        const float W[9] = {V[0], V[1], V[2], V[4], V[5], V[6], V[8], V[9], V[10]};
        float JW[9], JWT[9], t9[9], Vp[9];
        light_m3mul(J, W, JW);
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int k = 0; k < 3; ++k) JWT[c * 3 + k] = JW[k * 3 + c];
        light_m3mul(JW, cov, t9);
        light_m3mul(t9, JWT, Vp);
        const float c00 = ad(Vp[0], 0.3f), c01 = Vp[1], c11 = ad(Vp[4], 0.3f);
        const float mid = ad(c00, c11), ex = sb(c00, c11), ey = ml(2.0f, c01);   // :182-187
        const float delta = __fsqrt_rn(ad(ml(ex, ex), ml(ey, ey)));
        const float l1 = ml(0.5f, ad(mid, delta)), l2 = ml(0.5f, sb(mid, delta));
        if (l2 < 0.0f) alive = false;
        else {
            const float dgy = dv(ad(ad(-c00, c01), l1), ad(sb(c01, c11), l1));   // :191
            const float di = dv(1.0f, __fsqrt_rn(ad(ml(1.0f, 1.0f), ml(dgy, dgy))));
            const float dvx = ml(1.0f, di), dvy = ml(dgy, di);
            const float t1 = ml(3.0f, __fsqrt_rn(l1)), t2 = ml(3.0f, __fsqrt_rn(l2));
            const float r1 = 1024.0f < t1 ? 1024.0f : t1, r2 = 1024.0f < t2 ? 1024.0f : t2;   // GLM min(x, y) = y < x ? y : x
            const float hx = ml(a.res[0], 0.5f), hy = ml(a.res[1], 0.5f);
            o0 = make_float4(dv(c0, c3), dv(c1, c3), dv(ml(r1, dvx), hx), dv(ml(r1, dvy), hy));
            // gaussianPointLightCubeMapShadowPS.glsl:17: length(wsPos - light) / far, constant per quad
            o1 = make_float4(dv(ml(r2, dvy), hx), dv(ml(r2, -dvx), hy), dv(__fsqrt_rn(dd), a.near_far[1]), __uint_as_float((uint32_t)face));
        }
    }
    float4* out = a.light_quads + gid * 2;
    out[0] = o0;
    out[1] = o1;
}

// ---- cube raster ----------------------------------------------------------------------------------------------------
// D24 (DESIGN §2): round-half-even(clamp(d, 0, 1) * (2^24 - 1)), the product exact in fp64; false for NaN (no write)
__device__ __forceinline__ bool shadow_code(float d, uint32_t& code) {
    if (d != d) return false;
    code = __double2uint_rn((double)fminf(fmaxf(d, 0.0f), 1.0f) * 16777215.0);
    return true;
}

// the record's two triangles in its face's S x S viewport (the splat draw's rule); false if it draws nothing
__device__ __forceinline__ bool shadow_setup(const float4* r, uint32_t S, SplatTri t[2], uint32_t& face, uint32_t& code) {
    const float4 a = r[0], b = r[1];
    face = __float_as_uint(b.w);
    if (face > 5u || !shadow_code(b.z, code)) return false;
    const float4 q[2] = {make_float4(a.x, a.y, 0.f, 0.f), make_float4(a.z, a.w, b.x, b.y)};   // mean, quadScaleNdc
    splat_quad_setup(q, (int)S, (int)S, t);
    return true;
}

__device__ __forceinline__ int shadow_tiles_x(uint32_t S) { return (int)((S + kSplatTile - 1) / kSplatTile); }

// the binning (m2s_bin.cuh): light records, n = min(count, *d_count), tile = face * (S/16)^2 + tile of the face, pair
// value = record index
struct ShadowBins {
    ShadowArgs a;
    __host__ __device__ unsigned long long items() const { return a.count; }
    __host__ __device__ uint64_t tiles() const { return shadow_tiles(a.size); }
    __device__ __forceinline__ uint32_t n() const {
        unsigned long long n = a.count;
        if (a.d_count) n = min(n, *a.d_count);
        return (uint32_t)n;   // count < 2^30
    }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        SplatTri t[2];
        uint32_t face, code;
        if (!shadow_setup(a.light_quads + (uint64_t)i * 2, a.size, t, face, code)) return 0;
        const int tx = shadow_tiles_x(a.size);
        const uint32_t base = face * (uint32_t)(tx * tx);
        return splat_for_each_tile(t, tx, [&](uint32_t, uint32_t tile) { f(base + tile, i); });
    }
};

struct ShadowStage {
    int32_t A[6][kSplatThreads], B[6][kSplatThreads];
    long long C[6][kSplatThreads];
    uint32_t code[kSplatThreads];
};

__global__ void __launch_bounds__(kSplatThreads) shadow_tile_kernel(ShadowArgs a, const uint32_t* __restrict__ vals) {
    __shared__ ShadowStage s;
    const BinLayout l = bin_layout(a.count, shadow_tiles(a.size));
    const uint32_t* start = reinterpret_cast<const uint32_t*>(a.scratch + l.ranges_off);
    const uint32_t S = a.size, tx = (uint32_t)shadow_tiles_x(S), tpf = tx * tx;
    const uint32_t tile = blockIdx.x, face = tile / tpf, lt = tile % tpf;
    const int ox = (int)(lt % tx) * kSplatTile, oy = (int)(lt / tx) * kSplatTile;
    const int tid = threadIdx.x, lx = tid % kSplatTile, ly = tid / kSplatTile;
    const int x = ox + lx, y = oy + ly;
    const uint32_t r0 = vals ? start[tile] : 0u, r1 = vals ? start[l.tiles + tile] : 0u;
    uint32_t best = kShadowClearCode;
    for (uint32_t base = r0; base < r1; base += kSplatThreads) {
        const uint32_t nb = min(r1 - base, (uint32_t)kSplatThreads);
        __syncthreads();
        if ((uint32_t)tid < nb) {
            SplatTri t[2];
            uint32_t f, code;
            shadow_setup(a.light_quads + (uint64_t)vals[base + tid] * 2, S, t, f, code);   // a record with pairs draws
#pragma unroll
            for (int e = 0; e < 6; ++e) {
                const SplatTri& tt = t[e / 3];
                const int k = e % 3;
                s.A[e][tid] = tt.A[k];
                s.B[e][tid] = tt.B[k];
                s.C[e][tid] = tt.C[k] + (long long)tt.A[k] * ox + (long long)tt.B[k] * oy - (tt.incl[k] ? 0 : 1);
            }
            s.code[tid] = code;
        }
        __syncthreads();
        for (uint32_t j = 0; j < nb; ++j) {
            const uint32_t code = s.code[j];
            if (code >= best) continue;   // LESS against the best so far
            bool cover = false;
#pragma unroll
            for (int tri = 0; tri < 2; ++tri) {
                bool in = true;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const int e = tri * 3 + k;
                    in &= s.C[e][j] + (long long)s.A[e][j] * lx + (long long)s.B[e][j] * ly >= 0;
                }
                cover |= in;
            }
            if (cover) best = code;
        }
    }
    if (x >= (int)S || y >= (int)S) return;
    a.cube[((size_t)face * S + y) * S + x] = __fdiv_rn(__uint2float_rn(best), 16777215.0f);
}

// ---- deferred lighting ----------------------------------------------------------------------------------------------
// log2, exp2 and pow = exp2(y log2 x) from round-to-nearest fp32 operations only (DESIGN §2; the same steps as the
// oracle's orc_light_log2 / orc_light_exp2)
__device__ __forceinline__ float light_log2(float x) {
    if (x != x) return x;
    if (x < 0.0f) return __int_as_float(0x7fc00000);
    if (x == 0.0f) return __int_as_float(0xff800000);
    if (x == __int_as_float(0x7f800000)) return x;
    uint32_t u = __float_as_uint(x);
    int e = 0;
    if (u < 0x00800000u) { u = __float_as_uint(ml(x, 8388608.0f)); e = -23; }   // subnormal: exact scaling by 2^23
    e += (int)(u >> 23) - 127;
    float m = __uint_as_float((u & 0x007fffffu) | 0x3f800000u);   // [1, 2)
    if (m > 1.41421356f) { m = ml(m, 0.5f); e += 1; }               // [sqrt(1/2), sqrt(2)], exact
    const float f = dv(sb(m, 1.0f), ad(m, 1.0f));                    // log2 m = 2/ln2 artanh f
    const float z = ml(f, f);
    float p = 0.26230818925f;
    p = ad(ml(p, z), 0.32059889798f);
    p = ad(ml(p, z), 0.41219858311f);
    p = ad(ml(p, z), 0.57707801636f);
    p = ad(ml(p, z), 0.96179669393f);
    p = ad(ml(p, z), 2.88539008178f);
    return ad((float)e, ml(f, p));
}

__device__ __forceinline__ float light_exp2(float t) {
    if (t != t) return t;
    if (t >= 128.0f) return __int_as_float(0x7f800000);
    if (t < -150.0f) return 0.0f;
    const float fk = rintf(t);
    const float r = sb(t, fk);   // exact, |r| <= 1/2
    float p = 1.5252733804e-5f;
    p = ad(ml(p, r), 1.5403530393e-4f);
    p = ad(ml(p, r), 1.3333558146e-3f);
    p = ad(ml(p, r), 9.6181291076e-3f);
    p = ad(ml(p, r), 5.5504108665e-2f);
    p = ad(ml(p, r), 2.4022650696e-1f);
    p = ad(ml(p, r), 6.9314718056e-1f);
    p = ad(ml(p, r), 1.0f);
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return ml(ml(p, __int_as_float((k1 + 127) << 23)), __int_as_float((k2 + 127) << 23));
}

__device__ __forceinline__ float light_pow(float x, float y) { return light_exp2(ml(y, light_log2(x))); }

// GL 4.6 §8.13 table 8.19 with DESIGN §2's tie and non-finite rules; NEAREST, CLAMP_TO_EDGE
__device__ __forceinline__ float light_cube_fetch(const float* cube, uint32_t S, float rx, float ry, float rz) {
    const int face = light_face(rx, ry, rz);
    float sc, tc, ma;
    switch (face) {
        case 0: sc = -rz; tc = -ry; ma = rx; break;
        case 1: sc = rz; tc = -ry; ma = rx; break;
        case 2: sc = rx; tc = rz; ma = ry; break;
        case 3: sc = rx; tc = -rz; ma = ry; break;
        case 4: sc = rx; tc = -ry; ma = rz; break;
        default: sc = -rx; tc = -ry; ma = rz; break;
    }
    ma = fabsf(ma);
    const float s = ml(ad(dv(sc, ma), 1.0f), 0.5f), t = ml(ad(dv(tc, ma), 1.0f), 0.5f);
    const float fS = (float)S, top = (float)(S - 1);
    const uint32_t i = (uint32_t)fminf(fmaxf(floorf(ml(s, fS)), 0.0f), top), j = (uint32_t)fminf(fmaxf(floorf(ml(t, fS)), 0.0f), top);
    return __ldg(cube + ((size_t)face * S + j) * S + i);
}

__device__ __forceinline__ uint32_t light_u8(float v) { return __float2uint_rn(ml(fminf(fmaxf(v, 0.0f), 1.0f), 255.0f)); }
__device__ __forceinline__ float light_unorm(uint32_t c) { return dv((float)c, 255.0f); }

__global__ void __launch_bounds__(kLightThreads) deferred_light_kernel(const __grid_constant__ LightArgs a) {
    const uint64_t px = (uint64_t)blockIdx.x * kLightThreads + threadIdx.x;
    if (px >= (uint64_t)a.width * a.height) return;
    const uint32_t ab = __ldg(reinterpret_cast<const uint32_t*>(a.albedo) + px);
    float out[3];
    if (a.mode == 5) {   // gaussianSplattingDeferredPS.glsl:105-109
        const uint32_t mb = __ldg(reinterpret_cast<const uint32_t*>(a.metallic_roughness) + px);
        out[0] = light_unorm(mb & 255u); out[1] = light_unorm((mb >> 8) & 255u); out[2] = 0.0f;
    } else if (a.mode != 6) {   // :113-117
        out[0] = light_unorm(ab & 255u); out[1] = light_unorm((ab >> 8) & 255u); out[2] = light_unorm((ab >> 16) & 255u);
    } else {
        const uint32_t mb = __ldg(reinterpret_cast<const uint32_t*>(a.metallic_roughness) + px);
        const uint2 pb = __ldg(reinterpret_cast<const uint2*>(a.position) + px), nb = __ldg(reinterpret_cast<const uint2*>(a.normal) + px);
        float alb[3] = {light_unorm(ab & 255u), light_unorm((ab >> 8) & 255u), light_unorm((ab >> 16) & 255u)};
        const float metallic = light_unorm((mb >> 16) & 255u), roughness = light_unorm((mb >> 8) & 255u);   // :119-122
        const float pos[3] = {__half2float(__ushort_as_half((unsigned short)(pb.x & 0xffffu))), __half2float(__ushort_as_half((unsigned short)(pb.x >> 16))),
                              __half2float(__ushort_as_half((unsigned short)(pb.y & 0xffffu)))};
        float nv[3] = {__half2float(__ushort_as_half((unsigned short)(nb.x & 0xffffu))), __half2float(__ushort_as_half((unsigned short)(nb.x >> 16))),
                       __half2float(__ushort_as_half((unsigned short)(nb.y & 0xffffu)))};
#pragma unroll
        for (int c = 0; c < 3; ++c) nv[c] = sb(ml(nv[c], 2.0f), 1.0f);   // :126
        const float ni = dv(1.0f, __fsqrt_rn(dot3(nv[0], nv[1], nv[2])));
        const float N[3] = {ml(nv[0], ni), ml(nv[1], ni), ml(nv[2], ni)};
        // computeShadowFactor (:70-99): 20 taps, offsets not normalised
        const float ld[3] = {sb(pos[0], a.light[0]), sb(pos[1], a.light[1]), sb(pos[2], a.light[2])};
        const float ldd = dot3(ld[0], ld[1], ld[2]);
        const float current = __fsqrt_rn(ldd), si = dv(1.0f, __fsqrt_rn(ldd));
        const float sd[3] = {ml(ld[0], si), ml(ld[1], si), ml(ld[2], si)};
        const float thr = sb(current, 0.05f);
        float shadow = 0.0f;
        // sampleOffsetDirections[20]: per tap three 2-bit fields (component + 1), ten taps per word
        constexpr unsigned long long kOff0 = 0x049a20008aa208aaull, kOff1 = 0x0241869106926610ull;
#pragma unroll 1
        for (int i = 0; i < 20; ++i) {
            const uint32_t b = (uint32_t)((i < 10 ? kOff0 : kOff1) >> (6 * (i % 10))) & 63u;
            const float ox = (float)((int)(b & 3u) - 1), oy = (float)((int)((b >> 2) & 3u) - 1), oz = (float)((int)(b >> 4) - 1);
            const float closest = ml(light_cube_fetch(a.cube, a.shadow_size, ad(sd[0], ml(ox, 0.025f)), ad(sd[1], ml(oy, 0.025f)),
                                                      ad(sd[2], ml(oz, 0.025f))), a.far_plane);
            shadow = ad(shadow, thr > closest ? 1.0f : 0.0f);
        }
        shadow = dv(shadow, 20.0f);
#pragma unroll
        for (int c = 0; c < 3; ++c) alb[c] = light_pow(alb[c], 2.2f);   // :130
        float L[3] = {sb(a.light[0], pos[0]), sb(a.light[1], pos[1]), sb(a.light[2], pos[2])};
        const float lpd = dot3(L[0], L[1], L[2]), li = dv(1.0f, __fsqrt_rn(lpd));
        const float d = __fsqrt_rn(lpd);   // :138 length(u_LightPosition - pos)
#pragma unroll
        for (int c = 0; c < 3; ++c) L[c] = ml(L[c], li);
        float V[3] = {sb(a.cam[0], pos[0]), sb(a.cam[1], pos[1]), sb(a.cam[2], pos[2])};
        const float vi = dv(1.0f, __fsqrt_rn(dot3(V[0], V[1], V[2])));
#pragma unroll
        for (int c = 0; c < 3; ++c) V[c] = ml(V[c], vi);
        float H[3] = {ad(V[0], L[0]), ad(V[1], L[1]), ad(V[2], L[2])};
        const float hi = dv(1.0f, __fsqrt_rn(dot3(H[0], H[1], H[2])));
#pragma unroll
        for (int c = 0; c < 3; ++c) H[c] = ml(H[c], hi);
        const float atten = dv(1.0f, ml(d, d));
        auto dotv = [](const float* p, const float* q) { return ad(ad(ml(p[0], q[0]), ml(p[1], q[1])), ml(p[2], q[2])); };
        auto mx0 = [](float v) { return v < 0.0f ? 0.0f : v; };   // GLM max(x, y) = x < y ? y : x
        const float HdotV = mx0(dotv(H, V));
        const float c01 = mx0(sb(1.0f, HdotV)), fr = light_pow(1.0f < c01 ? 1.0f : c01, 5.0f);   // fresnelSchlick, GLM clamp
        // DistributionGGX: PI * denom * denom = ((22/7) denom) denom
        const float ra = ml(roughness, roughness), a2 = ml(ra, ra);
        const float NdotH = mx0(dotv(N, H));
        float den = ad(ml(ml(NdotH, NdotH), sb(a2, 1.0f)), 1.0f);
        den = ml(ml(22.0f / 7.0f, den), den);
        const float NDF = dv(a2, den);
        // GeometrySmith
        const float NdotV = mx0(dotv(N, V)), NdotL = mx0(dotv(N, L));
        const float rr = ad(roughness, 1.0f), k = dv(ml(rr, rr), 8.0f);
        const float ggx2 = dv(NdotV, ad(ml(NdotV, sb(1.0f, k)), k)), ggx1 = dv(NdotL, ad(ml(NdotL, sb(1.0f, k)), k));
        const float G = ml(ggx1, ggx2);
        const float denominator = ad(ml(ml(4.0f, NdotV), NdotL), 0.0001f);
        const float NG = ml(NDF, G), unshadowed = sb(1.0f, shadow), om = sb(1.0f, metallic);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float F0 = ad(ml(0.04f, sb(1.0f, metallic)), ml(alb[c], metallic));   // GLM mix(x, y, a) = x (1 - a) + y a
            const float F = ad(F0, ml(sb(1.0f, F0), fr));
            const float spec = dv(ml(NG, F), denominator);
            const float kD = ml(sb(1.0f, F), om);
            const float radiance = ml(ml(a.light_color[c], a.light_intensity), atten);
            // (kD * albedo / PI + specular) * radiance * NdotL * (1 - shadow), PI = 22.0f/7.0f without parentheses
            const float Lo = ml(ml(ml(ad(dv(dv(ml(kD, alb[c]), 22.0f), 7.0f), spec), radiance), NdotL), unshadowed);
            float col = ad(ml(0.3f, alb[c]), Lo);
            col = dv(col, ad(col, 1.0f));
            out[c] = light_pow(col, 1.0f / 2.2f);
        }
    }
    reinterpret_cast<uint32_t*>(a.image)[px] = light_u8(out[0]) | light_u8(out[1]) << 8 | light_u8(out[2]) << 16 | 255u << 24;
}

// ---- launches -------------------------------------------------------------------------------------------------------
cudaError_t light_prepass_launch(const ShadowArgs& a, cudaStream_t stream) {
    if (a.count == 0) return cudaSuccess;
    light_prepass_kernel<<<(unsigned)((a.count + kLightPrepassThreads - 1) / kLightPrepassThreads), kLightPrepassThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t shadow_count_launch(const ShadowArgs& a, cudaStream_t stream) { return bin_count_launch(ShadowBins{a}, stream); }

cudaError_t shadow_draw_launch(const ShadowArgs& a, int sm_count, cudaStream_t stream) {
    const ShadowBins b{a};
    const cudaError_t e = bin_pairs_launch(b, sm_count, stream);
    if (e != cudaSuccess) return e;
    shadow_tile_kernel<<<(unsigned)b.tiles(), kSplatThreads, 0, stream>>>(a, bin_vals(b));
    return cudaGetLastError();
}

cudaError_t deferred_light_launch(const LightArgs& a, cudaStream_t stream) {
    const uint64_t n = (uint64_t)a.width * a.height;
    deferred_light_kernel<<<(unsigned)((n + kLightThreads - 1) / kLightThreads), kLightThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace m2s
