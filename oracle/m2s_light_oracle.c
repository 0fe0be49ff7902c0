/* m2s_light_oracle.c — CPU restatement of the viewer's shadow pass and deferred lighting (rows f-7, f-8).
 *
 * TEST INFRASTRUCTURE ONLY, like m2s_oracle.c: nothing under mesh2splat_b200/ includes, links or calls it.
 *
 * Restated (paths relative to the reference tree):
 *   light prepass     src/shaders/rendering/gaussianPointShadowMappingCS.glsl:58-207 + common.glsl:22-61
 *   uniforms          src/renderer/renderPasses/GaussianShadowPass.cpp:85-130 (glm::perspective, glm::lookAt per face)
 *   cube face draws   gaussianPointLightCubeMapShadowVS.glsl, gaussianPointLightCubeMapShadowPS.glsl,
 *                     GaussianShadowPass.cpp:156-236 (1024^2 GL_DEPTH_COMPONENT faces cleared to 1, LESS, no blend)
 *   lighting          gaussianSplattingDeferredPS.glsl:32-165, GaussianRelightingPass.cpp:42-150
 * The fixed-function parts are the contract of DESIGN §2: the splat draw's rasteriser in an S x S viewport, D24 depth
 * codes (round-half-even of clamp(d, 0, 1) (2^24 - 1), the product in fp64), GL 4.6 table 8.19 cube sampling with the
 * tie rule of determineFaceIndex, NEAREST + CLAMP_TO_EDGE, the texel-exact full-screen fetch, RGBA8 stores (clamp,
 * NaN -> 0, ties to even) and pow = exp2(y log2 x) built from round-to-nearest fp32 operations.
 *
 * The cube is drawn record by record, both triangles, pixel by pixel, with the depth test on codes: GL's order.
 *
 * Arithmetic: fp32, one rounding per operation (built with -ffp-contract=off), GLSL / GLM operation order.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

static inline float bits_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t f_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* include/m2s.h m2s_shadow_params / m2s_light_params, field for field */
typedef struct {
    float model_to_world[16], light_position[3], near_far[2], resolution[2], std_dev;
    uint32_t layout, size;
} shadow_params;
typedef struct {
    uint32_t width, height, render_mode;
    float light_position[3], light_color[3], light_intensity, cam_pos[3], far_plane;
    uint32_t shadow_size;
} light_params;

/* ---- exp2, log2, pow (DESIGN §2) ---------------------------------------------------------------------------------- */
/* log2: x = 2^e m with m in [sqrt(1/2), sqrt(2)], log2 m = (2/ln2) artanh f, f = (m - 1)/(m + 1), odd series to f^11 */
ORC_API float orc_light_log2(float x) {
    if (x != x) return x;
    if (x < 0.0f) return bits_f(0x7fc00000u);
    if (x == 0.0f) return bits_f(0xff800000u);
    if (x == bits_f(0x7f800000u)) return x;
    uint32_t u = f_bits(x);
    int e = 0;
    if (u < 0x00800000u) { u = f_bits(x * 8388608.0f); e = -23; }
    e += (int)(u >> 23) - 127;
    float m = bits_f((u & 0x007fffffu) | 0x3f800000u);
    if (m > 1.41421356f) { m = m * 0.5f; e += 1; }
    const float f = (m - 1.0f) / (m + 1.0f);
    const float z = f * f;
    float p = 0.26230818925f;
    p = p * z + 0.32059889798f;
    p = p * z + 0.41219858311f;
    p = p * z + 0.57707801636f;
    p = p * z + 0.96179669393f;
    p = p * z + 2.88539008178f;
    return (float)e + f * p;
}

/* exp2: t = k + r, |r| <= 1/2 (r exact), degree-7 Taylor polynomial of 2^r, 2^k in two exact-or-once-rounded multiplies */
ORC_API float orc_light_exp2(float t) {
    if (t != t) return t;
    if (t >= 128.0f) return bits_f(0x7f800000u);
    if (t < -150.0f) return 0.0f;
    const float fk = rintf(t);
    const float r = t - fk;
    float p = 1.5252733804e-5f;
    p = p * r + 1.5403530393e-4f;
    p = p * r + 1.3333558146e-3f;
    p = p * r + 9.6181291076e-3f;
    p = p * r + 5.5504108665e-2f;
    p = p * r + 2.4022650696e-1f;
    p = p * r + 6.9314718056e-1f;
    p = p * r + 1.0f;
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return p * bits_f((uint32_t)(k1 + 127) << 23) * bits_f((uint32_t)(k2 + 127) << 23);
}

ORC_API float orc_light_pow(float x, float y) { return orc_light_exp2(y * orc_light_log2(x)); }

/* the splat draw's exp (DESIGN §2), for the PACKED56 scales */
static float exp_rn(float x) {
    if (x != x) return x;
    if (x > 88.72283905206835f) return bits_f(0x7f800000u);
    if (x < -103.97208f) return 0.0f;
    const float fk = rintf(x * 1.44269504088896341f);
    float r = x - fk * 0.693359375f;
    r = r - fk * -2.12194440e-4f;
    const float z = r * r;
    float p = 1.9875691500e-4f;
    p = p * r + 1.3981999507e-3f;
    p = p * r + 8.3334519073e-3f;
    p = p * r + 4.1665795894e-2f;
    p = p * r + 1.6666665459e-1f;
    p = p * r + 5.0000001201e-1f;
    p = p * z + r + 1.0f;
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return p * bits_f((uint32_t)(k1 + 127) << 23) * bits_f((uint32_t)(k2 + 127) << 23);
}

/* ---- cube faces ----------------------------------------------------------------------------------------------------- */
/* determineFaceIndex (gaussianPointShadowMappingCS.glsl:58-69), also the sampler's major axis: x wins ties, then y */
ORC_API int orc_light_face(float x, float y, float z) {
    const float ax = fabsf(x), ay = fabsf(y), az = fabsf(z);
    if (ax >= ay && ax >= az) return x > 0.0f ? 0 : 1;
    if (ay >= ax && ay >= az) return y > 0.0f ? 2 : 3;
    return z > 0.0f ? 4 : 5;
}

/* GL 4.6 §8.13 table 8.19, NEAREST, CLAMP_TO_EDGE: face and texel (i, j) of direction r in an S x S cube */
ORC_API void orc_cube_texel(float rx, float ry, float rz, uint32_t S, int* face, int* ti, int* tj) {
    const int f = orc_light_face(rx, ry, rz);
    float sc, tc, ma;
    switch (f) {
        case 0: sc = -rz; tc = -ry; ma = rx; break;
        case 1: sc = rz; tc = -ry; ma = rx; break;
        case 2: sc = rx; tc = rz; ma = ry; break;
        case 3: sc = rx; tc = -rz; ma = ry; break;
        case 4: sc = rx; tc = -ry; ma = rz; break;
        default: sc = -rx; tc = -ry; ma = rz; break;
    }
    ma = fabsf(ma);
    const float s = (sc / ma + 1.0f) * 0.5f, t = (tc / ma + 1.0f) * 0.5f;
    const float top = (float)(S - 1);
    *face = f;
    *ti = (int)fminf(fmaxf(floorf(s * (float)S), 0.0f), top);
    *tj = (int)fminf(fmaxf(floorf(t * (float)S), 0.0f), top);
}

static float cube_sample(const float* cube, uint32_t S, float rx, float ry, float rz) {
    int f, i, j;
    orc_cube_texel(rx, ry, rz, S, &f, &i, &j);
    return cube[((size_t)f * S + (size_t)j) * S + (size_t)i];
}

/* D24: code of a depth; 0 for NaN (no write) */
ORC_API int orc_d24(float d, uint32_t* code) {
    if (d != d) return 0;
    *code = (uint32_t)llrint((double)fminf(fmaxf(d, 0.0f), 1.0f) * 16777215.0);
    return 1;
}

/* ---- uniforms (GaussianShadowPass::execute) ------------------------------------------------------------------------- */
static void normalize3(float v[3]) {
    const float inv = 1.0f / sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    v[0] = v[0] * inv; v[1] = v[1] * inv; v[2] = v[2] * inv;
}
static void cross3(const float a[3], const float b[3], float r[3]) {
    r[0] = a[1] * b[2] - b[1] * a[2]; r[1] = a[2] * b[0] - b[2] * a[0]; r[2] = a[0] * b[1] - b[0] * a[1];
}

/* out: V[6][16] (glm::lookAt per face), P[16] (glm::perspective), Rinv[9] (inverse(mat3(M))), mscale2[3] */
ORC_API void orc_light_uniforms(const shadow_params* p, float* V, float* P, float* Rinv, float* mscale2) {
    static const float D[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
    static const float U[6][3] = {{0, -1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}, {0, -1, 0}, {0, -1, 0}};
    const float* e = p->light_position;
    for (int f = 0; f < 6; ++f) {
        float fw[3] = {(e[0] + D[f][0]) - e[0], (e[1] + D[f][1]) - e[1], (e[2] + D[f][2]) - e[2]}, s[3], u[3];
        normalize3(fw);
        cross3(fw, U[f], s);
        normalize3(s);
        cross3(s, fw, u);
        float* v = V + 16 * f;
        memset(v, 0, 64);
        v[0] = s[0]; v[4] = s[1]; v[8] = s[2];
        v[1] = u[0]; v[5] = u[1]; v[9] = u[2];
        v[2] = -fw[0]; v[6] = -fw[1]; v[10] = -fw[2];
        v[12] = -(s[0] * e[0] + s[1] * e[1] + s[2] * e[2]);
        v[13] = -(u[0] * e[0] + u[1] * e[1] + u[2] * e[2]);
        v[14] = fw[0] * e[0] + fw[1] * e[1] + fw[2] * e[2];
        v[15] = 1.0f;
    }
    const float n = p->near_far[0], fa = p->near_far[1];
    const float th = tanf((90.0f * 0.01745329251994329576923690768489f) / 2.0f);
    memset(P, 0, 64);
    P[0] = 1.0f / (1.0f * th); P[5] = 1.0f / th;
    P[10] = -(fa + n) / (fa - n); P[11] = -1.0f; P[14] = -(2.0f * fa * n) / (fa - n);
    const float* M = p->model_to_world;
#define m(c, r) M[4 * (c) + (r)]
    const float ood = 1.0f / (m(0, 0) * (m(1, 1) * m(2, 2) - m(2, 1) * m(1, 2)) - m(1, 0) * (m(0, 1) * m(2, 2) - m(2, 1) * m(0, 2)) +
                              m(2, 0) * (m(0, 1) * m(1, 2) - m(1, 1) * m(0, 2)));
    Rinv[0] = (m(1, 1) * m(2, 2) - m(2, 1) * m(1, 2)) * ood;
    Rinv[3] = -(m(1, 0) * m(2, 2) - m(2, 0) * m(1, 2)) * ood;
    Rinv[6] = (m(1, 0) * m(2, 1) - m(2, 0) * m(1, 1)) * ood;
    Rinv[1] = -(m(0, 1) * m(2, 2) - m(2, 1) * m(0, 2)) * ood;
    Rinv[4] = (m(0, 0) * m(2, 2) - m(2, 0) * m(0, 2)) * ood;
    Rinv[7] = -(m(0, 0) * m(2, 1) - m(2, 0) * m(0, 1)) * ood;
    Rinv[2] = (m(0, 1) * m(1, 2) - m(1, 1) * m(0, 2)) * ood;
    Rinv[5] = -(m(0, 0) * m(1, 2) - m(1, 0) * m(0, 2)) * ood;
    Rinv[8] = (m(0, 0) * m(1, 1) - m(1, 0) * m(0, 1)) * ood;
#undef m
    const float l0 = sqrtf((M[0] * M[0] + M[1] * M[1]) + (M[2] * M[2] + M[3] * M[3]));
    const float l1 = sqrtf((M[4] * M[4] + M[5] * M[5]) + (M[6] * M[6] + M[7] * M[7]));
    mscale2[0] = l0 * l0; mscale2[1] = l0 * l0; mscale2[2] = l1 * l1;
}

/* ---- light prepass -------------------------------------------------------------------------------------------------- */
static void m3mul(const float* a, const float* b, float* r) {   /* GLM mat3 * mat3, column-major */
    for (int c = 0; c < 3; ++c)
        for (int row = 0; row < 3; ++row) r[c * 3 + row] = a[row] * b[c * 3] + a[3 + row] * b[c * 3 + 1] + a[6 + row] * b[c * 3 + 2];
}
static float m4row(const float* m, int row, float x, float y, float z, float w) {   /* GLM mat4 * vec4 */
    return (m[row] * x + m[4 + row] * y) + (m[8 + row] * z + m[12 + row] * w);
}

/* records 0..n-1 -> n light records of 8 words: mean NDC xy, quadScaleNdc xyzw, gl_FragDepth, face (uint32; 0xFFFFFFFF
 * and zeros when culled) */
ORC_API void orc_light_prepass(const void* records, uint64_t n, const shadow_params* p, float* out) {
    float V[96], P[16], Rinv[9], ms2[3];
    orc_light_uniforms(p, V, P, Rinv, ms2);
    const float* M = p->model_to_world;
    const float* L = p->light_position;
    const float res0 = p->resolution[0], res1 = p->resolution[1], nr = p->near_far[0], fr = p->near_far[1];
    for (uint64_t g = 0; g < n; ++g) {
        float px, py, pz, sx, sy, sz, qx, qy, qz, qw;
        if (p->layout == 0) {
            const float* r = (const float*)records + g * 24;
            px = r[0]; py = r[1]; pz = r[2]; sx = r[8]; sy = r[9]; sz = r[10]; qx = r[16]; qy = r[17]; qz = r[18]; qw = r[19];
        } else {
            const float* r = (const float*)((const unsigned char*)records + g * 56);
            px = r[0]; py = r[1]; pz = r[2]; qx = r[3]; qy = r[4]; qz = r[5]; qw = r[6];
            sx = exp_rn(r[7]); sy = exp_rn(r[8]); sz = exp_rn(r[9]);
        }
        float* o = out + g * 8;
        memset(o, 0, 32);
        const uint32_t culled = 0xFFFFFFFFu;
        memcpy(o + 7, &culled, 4);
        const float w0 = m4row(M, 0, px, py, pz, 1.0f), w1 = m4row(M, 1, px, py, pz, 1.0f), w2 = m4row(M, 2, px, py, pz, 1.0f);
        const float dx = w0 - L[0], dy = w1 - L[1], dz = w2 - L[2];
        const float dd = dx * dx + dy * dy + dz * dz, inv = 1.0f / sqrtf(dd);
        const int face = orc_light_face(dx * inv, dy * inv, dz * inv);
        const float* Vf = V + 16 * face;
        const float v0 = m4row(Vf, 0, w0, w1, w2, 1.0f), v1 = m4row(Vf, 1, w0, w1, w2, 1.0f), v2 = m4row(Vf, 2, w0, w1, w2, 1.0f),
                    v3 = m4row(Vf, 3, w0, w1, w2, 1.0f);
        const float c0 = m4row(P, 0, v0, v1, v2, v3), c1 = m4row(P, 1, v0, v1, v2, v3), c2 = m4row(P, 2, v0, v1, v2, v3),
                    c3 = m4row(P, 3, v0, v1, v2, v3);
        const float clip = 1.05f * c3;
        if (c2 < -clip || c0 < -clip || c0 > clip || c1 < -clip || c1 > clip) continue;
        const float mult = p->layout == 0 ? p->std_dev : 1.0f;
        const float s0 = sx * mult * ms2[0], s1 = sy * mult * ms2[1], s2 = sz * mult * ms2[2];
        const float rot0[9] = {1.f - 2.f * (qz * qz + qw * qw), 2.f * (qy * qz - qx * qw), 2.f * (qy * qw + qx * qz),
                               2.f * (qy * qz + qx * qw), 1.f - 2.f * (qy * qy + qw * qw), 2.f * (qz * qw - qx * qy),
                               2.f * (qy * qw - qx * qz), 2.f * (qz * qw + qx * qy), 1.f - 2.f * (qy * qy + qz * qz)};
        float rot[9], S[9] = {s0, 0.f, 0.f, 0.f, s1, 0.f, 0.f, 0.f, s2}, mm[9], mmT[9], cov[9];
        m3mul(rot0, Rinv, rot);
        m3mul(S, rot, mm);
        for (int c = 0; c < 3; ++c)
            for (int k = 0; k < 3; ++k) mmT[c * 3 + k] = mm[k * 3 + c];
        m3mul(mmT, mm, cov);
        const float tzSq = v2 * v2;
        const float jsx = -(P[0] * res0) / (2.0f * v2), jsy = -(P[5] * res1) / (2.0f * v2);
        const float jtx = (P[0] * v0 * res0) / (2.0f * tzSq), jty = (P[5] * v1 * res1) / (2.0f * tzSq);
        const float jtz = ((fr - nr) * P[14]) / (2.0f * tzSq);
        const float J[9] = {jsx, 0.f, 0.f, 0.f, jsy, 0.f, jtx, jty, jtz};
        const float W[9] = {Vf[0], Vf[1], Vf[2], Vf[4], Vf[5], Vf[6], Vf[8], Vf[9], Vf[10]};
        float JW[9], JWT[9], t9[9], Vp[9];
        m3mul(J, W, JW);
        for (int c = 0; c < 3; ++c)
            for (int k = 0; k < 3; ++k) JWT[c * 3 + k] = JW[k * 3 + c];
        m3mul(JW, cov, t9);
        m3mul(t9, JWT, Vp);
        const float c00 = Vp[0] + 0.3f, c01 = Vp[1], c11 = Vp[4] + 0.3f;
        const float mid = c00 + c11, ex = c00 - c11, ey = 2.0f * c01;
        const float delta = sqrtf(ex * ex + ey * ey);
        const float l1 = 0.5f * (mid + delta), l2 = 0.5f * (mid - delta);
        if (l2 < 0.0f) continue;
        const float dgy = (-c00 + c01 + l1) / (c01 - c11 + l1);
        const float di = 1.0f / sqrtf(1.0f * 1.0f + dgy * dgy);
        const float dvx = 1.0f * di, dvy = dgy * di;
        const float t1 = 3.0f * sqrtf(l1), t2 = 3.0f * sqrtf(l2);
        const float r1 = 1024.0f < t1 ? 1024.0f : t1, r2 = 1024.0f < t2 ? 1024.0f : t2;
        const float hx = res0 * 0.5f, hy = res1 * 0.5f;
        o[0] = c0 / c3; o[1] = c1 / c3;
        o[2] = r1 * dvx / hx; o[3] = r1 * dvy / hy; o[4] = r2 * dvy / hx; o[5] = r2 * -dvx / hy;
        o[6] = sqrtf(dd) / fr;
        const uint32_t fu = (uint32_t)face;
        memcpy(o + 7, &fu, 4);
    }
}

/* ---- cube raster: the splat draw's rasteriser (m2s_splat_oracle.c) in the face's S x S viewport --------------------- */
typedef struct { int64_t A[3], B[3], C[3]; int incl[3]; int x0, x1, y0, y1; } stri;

static void snap(float nx, float ny, float W, float H, int* ok, int32_t* X, int32_t* Y) {
    const float hw = W * 0.5f, hh = H * 0.5f;
    const float xw = nx * hw + hw, yw = ny * hh + hh;
    *ok = isfinite(xw) && isfinite(yw) && fabsf(xw) <= 8192.0f && fabsf(yw) <= 8192.0f;
    *X = *ok ? (int32_t)lrintf(xw * 256.0f) : 0;
    *Y = *ok ? (int32_t)lrintf(yw * 256.0f) : 0;
}

static void tri_setup(const int32_t X[3], const int32_t Y[3], int ok, int W, int H, stri* s) {
    memset(s, 0, sizeof(*s));
    s->x1 = -1; s->y1 = -1;
    if (!ok) return;
    const int64_t area2 = (int64_t)(X[1] - X[0]) * (Y[2] - Y[0]) - (int64_t)(X[2] - X[0]) * (Y[1] - Y[0]);
    if (area2 == 0) return;
    const int64_t sg = area2 < 0 ? -1 : 1;
    for (int k = 0; k < 3; ++k) {
        const int a = (k + 1) % 3, b = (k + 2) % 3;
        const int64_t dx = X[b] - X[a], dy = Y[b] - Y[a];
        s->A[k] = sg * (-dy * 256);
        s->B[k] = sg * (dx * 256);
        s->C[k] = sg * (dx * (128 - (int64_t)Y[a]) - dy * (128 - (int64_t)X[a]));
        s->incl[k] = (s->A[k] > 0) || (s->A[k] == 0 && s->B[k] > 0);
    }
    int32_t xmin = X[0], xmax = X[0], ymin = Y[0], ymax = Y[0];
    for (int k = 1; k < 3; ++k) {
        if (X[k] < xmin) xmin = X[k];
        if (X[k] > xmax) xmax = X[k];
        if (Y[k] < ymin) ymin = Y[k];
        if (Y[k] > ymax) ymax = Y[k];
    }
    int64_t x0 = ((int64_t)xmin + 127) >> 8, x1 = ((int64_t)xmax - 128) >> 8;
    int64_t y0 = ((int64_t)ymin + 127) >> 8, y1 = ((int64_t)ymax - 128) >> 8;
    if (x0 < 0) x0 = 0;
    if (y0 < 0) y0 = 0;
    if (x1 > W - 1) x1 = W - 1;
    if (y1 > H - 1) y1 = H - 1;
    s->x0 = (int)x0; s->x1 = (int)x1; s->y0 = (int)y0; s->y1 = (int)y1;
}

static int tri_inside(const stri* s, int i, int j) {
    for (int k = 0; k < 3; ++k) {
        const int64_t e = s->A[k] * i + s->B[k] * j + s->C[k];
        if (e < 0 || (e == 0 && !s->incl[k])) return 0;
    }
    return 1;
}

/* gaussianPointLightCubeMapShadowVS.glsl:21 for the quad corners, both triangles; 0 if the record draws nothing */
static int record_setup(const float* r, uint32_t S, stri t[2], uint32_t* face, uint32_t* code) {
    memcpy(face, r + 7, 4);
    if (*face > 5u || !orc_d24(r[6], code)) return 0;
    static const float VX[4] = {-1.0f, -1.0f, 1.0f, 1.0f}, VY[4] = {-1.0f, 1.0f, 1.0f, -1.0f};
    int ok[4];
    int32_t X[4], Y[4];
    for (int v = 0; v < 4; ++v) {
        const float nx = r[0] + (VX[v] * r[2] + VY[v] * r[4]), ny = r[1] + (VX[v] * r[3] + VY[v] * r[5]);
        snap(nx, ny, (float)S, (float)S, &ok[v], &X[v], &Y[v]);
    }
    const int32_t X0[3] = {X[0], X[1], X[2]}, Y0[3] = {Y[0], Y[1], Y[2]};
    const int32_t X1[3] = {X[0], X[2], X[3]}, Y1[3] = {Y[0], Y[2], Y[3]};
    tri_setup(X0, Y0, ok[0] && ok[1] && ok[2], (int)S, (int)S, &t[0]);
    tri_setup(X1, Y1, ok[0] && ok[2] && ok[3], (int)S, (int)S, &t[1]);
    return 1;
}

static int tri_touches(const stri* s, int tx, int ty) {
    int a0 = tx * 16, a1 = tx * 16 + 15, b0 = ty * 16, b1 = ty * 16 + 15;
    if (s->x0 > a0) a0 = s->x0;
    if (s->x1 < a1) a1 = s->x1;
    if (s->y0 > b0) b0 = s->y0;
    if (s->y1 < b1) b1 = s->y1;
    if (a1 < a0 || b1 < b0) return 0;
    for (int k = 0; k < 3; ++k) {
        const int64_t e = s->A[k] * (s->A[k] > 0 ? a1 : a0) + s->B[k] * (s->B[k] > 0 ? b1 : b0) + s->C[k];
        if (e < 0 || (e == 0 && !s->incl[k])) return 0;
    }
    return 1;
}

/* (16 x 16 face tile, record) pairs per record as the cube raster's binning makes them; returns the total */
ORC_API uint64_t orc_cube_pairs(const float* recs, uint32_t n, uint32_t S, uint32_t* counts) {
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        stri t[2];
        uint32_t face, code, c = 0;
        if (record_setup(recs + (size_t)i * 8, S, t, &face, &code)) {
            int x0 = (int)S, x1 = -1, y0 = (int)S, y1 = -1;
            for (int k = 0; k < 2; ++k)
                if (t[k].x1 >= t[k].x0 && t[k].y1 >= t[k].y0) {
                    if (t[k].x0 < x0) x0 = t[k].x0;
                    if (t[k].x1 > x1) x1 = t[k].x1;
                    if (t[k].y0 < y0) y0 = t[k].y0;
                    if (t[k].y1 > y1) y1 = t[k].y1;
                }
            for (int ty = y0 / 16; x1 >= 0 && ty <= y1 / 16; ++ty)
                for (int tx = x0 / 16; tx <= x1 / 16; ++tx)
                    if (tri_touches(&t[0], tx, ty) || tri_touches(&t[1], tx, ty)) ++c;
        }
        if (counts) counts[i] = c;
        total += c;
    }
    return total;
}

/* glClear(GL_DEPTH_BUFFER_BIT) to 1 on all six faces, then records 0..n-1 in order, depth test LESS on D24 codes.
 * cube: 6 x S x S floats, (float)code / 16777215. */
ORC_API void orc_cube_raster(const float* recs, uint32_t n, uint32_t S, float* cube) {
    const size_t per = (size_t)S * S;
    uint32_t* codes = (uint32_t*)cube;   /* codes in place, converted at the end */
    for (size_t k = 0; k < 6 * per; ++k) codes[k] = 0xFFFFFFu;
    for (uint32_t i = 0; i < n; ++i) {
        stri t[2];
        uint32_t face, code;
        if (!record_setup(recs + (size_t)i * 8, S, t, &face, &code)) continue;
        uint32_t* fc = codes + face * per;
        for (int tri = 0; tri < 2; ++tri) {
            const stri* s = &t[tri];
            for (int j = s->y0; j <= s->y1; ++j)
                for (int x = s->x0; x <= s->x1; ++x)
                    if (tri_inside(s, x, j) && code < fc[(size_t)j * S + x]) fc[(size_t)j * S + x] = code;
        }
    }
    for (size_t k = 0; k < 6 * per; ++k) cube[k] = (float)codes[k] / 16777215.0f;
}

/* ---- deferred lighting ---------------------------------------------------------------------------------------------- */
static float h2f(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 0x3ffu;
    if (e == 31u) return bits_f(sign | 0x7f800000u | (m << 13));
    if (e) return bits_f(sign | ((e + 112u) << 23) | (m << 13));
    return m ? (sign ? -1.0f : 1.0f) * (float)m * bits_f(0x33800000u) : bits_f(sign);
}
static uint8_t u8(float v) { return (uint8_t)lrintf(fminf(fmaxf(v, 0.0f), 1.0f) * 255.0f); }
static float mx0(float v) { return v < 0.0f ? 0.0f : v; }   /* GLM max(v, 0) */
static float dotv(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

/* gaussianSplattingDeferredPS.glsl main() for one pixel: texels as fetched (position / normal fp16 bits, albedo / mr
 * bytes); out: FragColor (4 floats) */
ORC_API void orc_deferred_fs(const uint16_t* pos16, const uint16_t* nrm16, const uint8_t* alb8, const uint8_t* mr8, const float* cube,
                             const light_params* p, float* frag) {
    float col[3];
    if (p->render_mode == 5) {
        col[0] = (float)mr8[0] / 255.0f; col[1] = (float)mr8[1] / 255.0f; col[2] = 0.0f;
    } else if (p->render_mode != 6) {
        for (int c = 0; c < 3; ++c) col[c] = (float)alb8[c] / 255.0f;
    } else {
        float alb[3];
        for (int c = 0; c < 3; ++c) alb[c] = (float)alb8[c] / 255.0f;
        const float metallic = (float)mr8[2] / 255.0f, roughness = (float)mr8[1] / 255.0f;
        const float pos[3] = {h2f(pos16[0]), h2f(pos16[1]), h2f(pos16[2])};
        float nv[3];
        for (int c = 0; c < 3; ++c) nv[c] = h2f(nrm16[c]) * 2.0f - 1.0f;
        const float ni = 1.0f / sqrtf(dotv(nv, nv));
        const float N[3] = {nv[0] * ni, nv[1] * ni, nv[2] * ni};
        /* computeShadowFactor */
        static const float OFF[20][3] = {{1, 1, 1}, {1, -1, 1}, {-1, -1, 1}, {-1, 1, 1}, {1, 1, -1}, {1, -1, -1}, {-1, -1, -1}, {-1, 1, -1},
                                         {1, 1, 0}, {1, -1, 0}, {-1, -1, 0}, {-1, 1, 0}, {1, 0, 1}, {-1, 0, 1}, {1, 0, -1}, {-1, 0, -1},
                                         {0, 1, 1}, {0, -1, 1}, {0, -1, -1}, {0, 1, -1}};
        const float* LP = p->light_position;
        const float ld[3] = {pos[0] - LP[0], pos[1] - LP[1], pos[2] - LP[2]};
        const float current = sqrtf(dotv(ld, ld)), si = 1.0f / sqrtf(dotv(ld, ld));
        const float sd[3] = {ld[0] * si, ld[1] * si, ld[2] * si};
        float shadow = 0.0f;
        for (int i = 0; i < 20; ++i) {
            const float closest = cube_sample(cube, p->shadow_size, sd[0] + OFF[i][0] * 0.025f, sd[1] + OFF[i][1] * 0.025f,
                                              sd[2] + OFF[i][2] * 0.025f) * p->far_plane;
            shadow += current - 0.05f > closest ? 1.0f : 0.0f;
        }
        shadow = shadow / 20.0f;
        for (int c = 0; c < 3; ++c) alb[c] = orc_light_pow(alb[c], 2.2f);
        float L[3] = {LP[0] - pos[0], LP[1] - pos[1], LP[2] - pos[2]};
        const float lpd = dotv(L, L), li = 1.0f / sqrtf(lpd), d = sqrtf(lpd);
        for (int c = 0; c < 3; ++c) L[c] = L[c] * li;
        float V[3] = {p->cam_pos[0] - pos[0], p->cam_pos[1] - pos[1], p->cam_pos[2] - pos[2]};
        const float vi = 1.0f / sqrtf(dotv(V, V));
        for (int c = 0; c < 3; ++c) V[c] = V[c] * vi;
        float H[3] = {V[0] + L[0], V[1] + L[1], V[2] + L[2]};
        const float hi = 1.0f / sqrtf(dotv(H, H));
        for (int c = 0; c < 3; ++c) H[c] = H[c] * hi;
        const float atten = 1.0f / (d * d);
        const float HdotV = mx0(dotv(H, V));
        const float cl = mx0(1.0f - HdotV), fr = orc_light_pow(1.0f < cl ? 1.0f : cl, 5.0f);
        const float ra = roughness * roughness, a2 = ra * ra;
        const float NdotH = mx0(dotv(N, H));
        float den = NdotH * NdotH * (a2 - 1.0f) + 1.0f;
        den = 22.0f / 7.0f * den * den;   /* PI * denom * denom with PI = 22.0f/7.0f */
        const float NDF = a2 / den;
        const float NdotV = mx0(dotv(N, V)), NdotL = mx0(dotv(N, L));
        const float rr = roughness + 1.0f, k = (rr * rr) / 8.0f;
        const float ggx2 = NdotV / (NdotV * (1.0f - k) + k), ggx1 = NdotL / (NdotL * (1.0f - k) + k);
        const float G = ggx1 * ggx2;
        const float denominator = 4.0f * NdotV * NdotL + 0.0001f;
        for (int c = 0; c < 3; ++c) {
            const float F0 = 0.04f * (1.0f - metallic) + alb[c] * metallic;   /* GLM mix */
            const float F = F0 + (1.0f - F0) * fr;
            const float spec = NDF * G * F / denominator;
            const float kD = (1.0f - F) * (1.0f - metallic);
            const float radiance = p->light_color[c] * p->light_intensity * atten;
            const float Lo = (kD * alb[c] / 22.0f / 7.0f + spec) * radiance * NdotL * (1.0f - shadow);   /* / PI, unparenthesised */
            float v = 0.3f * alb[c] + Lo;
            v = v / (v + 1.0f);
            col[c] = orc_light_pow(v, 1.0f / 2.2f);
        }
    }
    frag[0] = col[0]; frag[1] = col[1]; frag[2] = col[2]; frag[3] = 1.0f;
}

/* the same pixel stored into the RGBA8 framebuffer */
ORC_API void orc_deferred_ps(const uint16_t* pos16, const uint16_t* nrm16, const uint8_t* alb8, const uint8_t* mr8, const float* cube,
                             const light_params* p, uint8_t* out) {
    float f[4];
    orc_deferred_fs(pos16, nrm16, alb8, mr8, cube, p, f);
    for (int c = 0; c < 4; ++c) out[c] = u8(f[c]);
}

/* the full-screen pass: pixel (x, y) fetches texel (x, y) of every target; NULL targets read as zeros */
ORC_API void orc_deferred_light(const uint16_t* pos, const uint16_t* nrm, const uint8_t* alb, const uint8_t* mr, const float* cube,
                                const light_params* p, uint8_t* image) {
    static const uint16_t z16[4] = {0, 0, 0, 0};
    static const uint8_t z8[4] = {0, 0, 0, 0};
    const size_t n = (size_t)p->width * p->height;
    for (size_t i = 0; i < n; ++i)
        orc_deferred_ps(pos ? pos + 4 * i : z16, nrm ? nrm + 4 * i : z16, alb ? alb + 4 * i : z8, mr ? mr + 4 * i : z8, cube, p, image + 4 * i);
}
