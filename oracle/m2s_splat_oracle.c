/* m2s_splat_oracle.c — CPU restatement of the viewer's splat draw (row f-6).
 *
 * TEST INFRASTRUCTURE ONLY, like m2s_oracle.c: nothing under mesh2splat_b200/ includes, links or calls it.
 *
 * Restated (paths relative to the reference tree):
 *   vertex shader     src/shaders/rendering/gaussianSplattingVS.glsl:31-41
 *   fragment shader   src/shaders/rendering/gaussianSplattingPS.glsl:29-46
 *   pass state        src/renderer/renderPasses/GaussianSplattingPass.cpp:10-20 (the quad), :37-97 (viewport, clear,
 *                     blend functions, one instanced indirect draw), renderer.cpp:325-379 (target formats)
 * The fixed-function parts are the contract of DESIGN §2, restated from the OpenGL 4.6 core spec: the conversion's
 * rasteriser rule (viewport transform in two fp32 steps, 1/256-pixel snap, non-finite or |.| > 8192 vertices drop the
 * triangle, sign-normalised int64 edge functions with the top-left rule, both windings, pixel centres), the blend of
 * 17.3.6 at destination precision (RGBA16F: fp32 blend, one round-to-nearest-even conversion to half; RGBA8: clamped,
 * stored as round-half-even of x 255) and one exp made of round-to-nearest fp32 operations.
 *
 * The draw goes instance by instance, triangle (V0,V1,V2) before (V0,V2,V3), pixel by pixel: GL's order.  A pixel both
 * snapped triangles of a quad cover is blended twice.
 *
 * Arithmetic: fp32, one rounding per operation (built with -ffp-contract=off), GLSL / GLM operation order.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

static inline float bits_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t f_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* exp from round-to-nearest fp32 operations only: x = k ln2 + r with ln2 in two parts (Cody-Waite), a degree-7
 * polynomial for e^r, then 2^k applied in two multiplies (the first exact, the second rounding once). */
ORC_API float orc_splat_exp(float x) {
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

/* fp32 -> fp16 bits, round to nearest even; overflow -> +-inf, NaN -> 0x7FFF, subnormals kept */
ORC_API uint16_t orc_f2h(float f) {
    const uint32_t x = f_bits(f), sign = (x >> 16) & 0x8000u, ax = x & 0x7fffffffu;
    if (ax > 0x7f800000u) return 0x7fffu;
    if (ax >= 0x477ff000u) return (uint16_t)(sign | 0x7c00u);
    if (ax >= 0x38800000u) {   /* normal half */
        const uint32_t m = ax - 0x38000000u;
        uint32_t h = m >> 13;
        const uint32_t rem = m & 0x1fffu;
        if (rem > 0x1000u || (rem == 0x1000u && (h & 1u))) ++h;
        return (uint16_t)(sign | h);
    }
    if (ax < 0x33000000u) return (uint16_t)sign;
    const uint32_t mant = (ax & 0x7fffffu) | 0x800000u, s = 126u - (ax >> 23);
    uint32_t h = mant >> s;
    const uint32_t rem = mant & ((1u << s) - 1u), halfway = 1u << (s - 1u);
    if (rem > halfway || (rem == halfway && (h & 1u))) ++h;
    return (uint16_t)(sign | h);
}

ORC_API float orc_h2f(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 0x3ffu;
    if (e == 31u) return bits_f(sign | 0x7f800000u | (m << 13));
    if (e) return bits_f(sign | ((e + 112u) << 23) | (m << 13));
    return m ? (sign ? -1.0f : 1.0f) * (float)m * bits_f(0x33800000u) : bits_f(sign);   /* m * 2^-24, exact */
}

/* gaussianSplattingVS.glsl for one vertex of one quad (24 floats: mean, scale, color, conic, normal, wsPos).
 * out: gl_Position.xy, then the 18 varyings: out_screen.xy, out_conic.xyz, out_color.rgb, out_opacity, out_normal.xyz,
 * out_wsPos.xyz, out_depth, metallicRoughness.xy */
ORC_API void orc_splat_vs(const float* q, int vertex, float width, float height, float* out) {
    static const float VX[4] = {-1.0f, -1.0f, 1.0f, 1.0f}, VY[4] = {-1.0f, 1.0f, 1.0f, -1.0f};
    const float vx = VX[vertex & 3], vy = VY[vertex & 3];
    out[0] = q[0] + (vx * q[4] + vy * q[6]);
    out[1] = q[1] + (vx * q[5] + vy * q[7]);
    float* v = out + 2;
    v[0] = (q[0] + 1.0f) * 0.5f * width;
    v[1] = (q[1] + 1.0f) * 0.5f * height;
    v[2] = -0.5f * q[12]; v[3] = -q[13]; v[4] = -0.5f * q[14];
    v[5] = q[8] * q[11]; v[6] = q[9] * q[11]; v[7] = q[10] * q[11];
    v[8] = q[11];
    v[9] = q[16]; v[10] = q[17]; v[11] = q[18];
    v[12] = q[20]; v[13] = q[21]; v[14] = q[22];
    v[15] = q[15];
    v[16] = q[19]; v[17] = q[23];
}

/* gaussianSplattingPS.glsl:29-46 at gl_FragCoord.xy = (fx, fy).  out: gPosition, gNormal, gAlbedo, gDepth,
 * gMetallicRoughness (4 floats each) */
ORC_API void orc_splat_fs(const float* v, float fx, float fy, int mode, float* out) {
    const float dx = v[0] - fx, dy = v[1] - fy;
    const float t0 = v[2] * (dx * dx), t1 = v[4] * (dy * dy), t2 = v[3] * (dx * dy);   /* dot(out_conic.xzy, ...) */
    const float g = orc_splat_exp(t0 + t1 + t2);
    const float op = v[8] * g;
    out[0] = v[12] * g; out[1] = v[13] * g; out[2] = v[14] * g; out[3] = 1.0f * g;
    out[4] = v[9] * g; out[5] = v[10] * g; out[6] = v[11] * g; out[7] = op;
    if (mode == 4) { out[8] = .01f; out[9] = .005f; out[10] = 0.0f; out[11] = .01f; }
    else { out[8] = v[5] * g; out[9] = v[6] * g; out[10] = v[7] * g; out[11] = op; }
    const float dp = v[15] * g;
    out[12] = dp; out[13] = dp; out[14] = dp; out[15] = op;
    out[16] = v[16] * g; out[17] = v[17] * g; out[18] = 0.0f * g; out[19] = 1.0f * g;
}

/* ---- rasteriser: the conversion's rule (m2s_oracle.c orc_triangle_setup) in a W x H viewport ---------------------- */
typedef struct { int64_t A[3], B[3], C[3]; int incl[3]; int x0, x1, y0, y1; } stri;

static void snap(const float* gp, float W, float H, int* ok, int32_t* X, int32_t* Y) {
    const float hw = W * 0.5f, hh = H * 0.5f;
    const float xw = gp[0] * hw + hw, yw = gp[1] * hh + hh;
    *ok = isfinite(xw) && isfinite(yw) && fabsf(xw) <= 8192.0f && fabsf(yw) <= 8192.0f;
    *X = *ok ? (int32_t)lrintf(xw * 256.0f) : 0;
    *Y = *ok ? (int32_t)lrintf(yw * 256.0f) : 0;
}

static int tri_setup(const int32_t X[3], const int32_t Y[3], int ok, int W, int H, stri* s) {
    memset(s, 0, sizeof(*s));
    s->x1 = -1; s->y1 = -1;
    if (!ok) return 0;
    const int64_t area2 = (int64_t)(X[1] - X[0]) * (Y[2] - Y[0]) - (int64_t)(X[2] - X[0]) * (Y[1] - Y[0]);
    if (area2 == 0) return 0;
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
    return x1 >= x0 && y1 >= y0;
}

static inline int tri_inside(const stri* s, int i, int j) {
    for (int k = 0; k < 3; ++k) {
        const int64_t e = s->A[k] * i + s->B[k] * j + s->C[k];
        if (e < 0 || (e == 0 && !s->incl[k])) return 0;
    }
    return 1;
}

static void quad_setup(const float* q, uint32_t W, uint32_t H, stri t[2]) {
    int ok[4];
    int32_t X[4], Y[4];
    float out[20];
    for (int v = 0; v < 4; ++v) {
        orc_splat_vs(q, v, (float)W, (float)H, out);
        snap(out, (float)W, (float)H, &ok[v], &X[v], &Y[v]);
    }
    const int32_t X0[3] = {X[0], X[1], X[2]}, Y0[3] = {Y[0], Y[1], Y[2]};
    const int32_t X1[3] = {X[0], X[2], X[3]}, Y1[3] = {Y[0], Y[2], Y[3]};
    tri_setup(X0, Y0, ok[0] && ok[1] && ok[2], (int)W, (int)H, &t[0]);
    tri_setup(X1, Y1, ok[0] && ok[2] && ok[3], (int)W, (int)H, &t[1]);
}

/* which pixels triangle `tri` of quad q covers: mask[y * W + x] = 1 (for the coverage tests) */
ORC_API void orc_splat_coverage(const float* q, int tri, uint32_t W, uint32_t H, uint8_t* mask) {
    stri t[2];
    quad_setup(q, W, H, t);
    memset(mask, 0, (size_t)W * H);
    const stri* s = &t[tri & 1];
    for (int j = s->y0; j <= s->y1; ++j)
        for (int i = s->x0; i <= s->x1; ++i)
            if (tri_inside(s, i, j)) mask[(size_t)j * W + i] = 1;
}

/* the tile pass's pair count per quad: 16 x 16 tiles where an edge-function box test of either triangle passes */
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

ORC_API uint64_t orc_splat_pairs(const float* quads, uint32_t n, uint32_t W, uint32_t H, uint32_t* counts) {
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; ++i) {
        stri t[2];
        quad_setup(quads + (size_t)i * 24, W, H, t);
        uint32_t c = 0;
        int x0 = (int)W, x1 = -1, y0 = (int)H, y1 = -1;   /* the tiles of the union of the triangles' boxes */
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
        if (counts) counts[i] = c;
        total += c;
    }
    return total;
}

/* ---- blend (GL 4.6 17.3.6) ----------------------------------------------------------------------------------------- */
static inline float sat(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

static void blend_f16(uint16_t* px, const float* src, int additive) {
    const float f = additive ? 1.0f : 1.0f - orc_h2f(px[3]);
    for (int c = 0; c < 4; ++c) px[c] = orc_f2h(src[c] * f + orc_h2f(px[c]));
}

static void blend_u8(uint8_t* px, const float* src, int additive) {
    const float f = additive ? 1.0f : sat(1.0f - (float)px[3] / 255.0f);
    for (int c = 0; c < 4; ++c) {
        const float r = sat(sat(src[c]) * f + (float)px[c] / 255.0f);
        px[c] = (uint8_t)lrintf(r * 255.0f);
    }
}

/* glClear to 0, then the first n quads (24 floats each) in order.  Targets: W x H x 4, row 0 = window y 0; NULL = not
 * drawn. */
ORC_API void orc_splat_draw(const float* quads, uint32_t n, uint32_t W, uint32_t H, uint32_t mode, uint16_t* pos, uint16_t* nrm,
                            uint8_t* alb, uint16_t* dep, uint8_t* mr) {
    const size_t np = (size_t)W * H * 4;
    if (pos) memset(pos, 0, np * 2);
    if (nrm) memset(nrm, 0, np * 2);
    if (alb) memset(alb, 0, np);
    if (dep) memset(dep, 0, np * 2);
    if (mr) memset(mr, 0, np);
    const int additive = mode == 4;
    for (uint32_t i = 0; i < n; ++i) {
        const float* q = quads + (size_t)i * 24;
        stri t[2];
        quad_setup(q, W, H, t);
        float vs[20];
        orc_splat_vs(q, 0, (float)W, (float)H, vs);   /* the varyings are the same at all four vertices */
        for (int tri = 0; tri < 2; ++tri) {
            const stri* s = &t[tri];
            for (int j = s->y0; j <= s->y1; ++j)
                for (int x = s->x0; x <= s->x1; ++x) {
                    if (!tri_inside(s, x, j)) continue;
                    float o[20];
                    orc_splat_fs(vs + 2, (float)x + 0.5f, (float)j + 0.5f, (int)mode, o);
                    const size_t p = ((size_t)j * W + x) * 4;
                    if (pos) blend_f16(pos + p, o + 0, additive);
                    if (nrm) blend_f16(nrm + p, o + 4, additive);
                    if (alb) blend_u8(alb + p, o + 8, additive);
                    if (dep) blend_f16(dep + p, o + 12, additive);
                    if (mr) blend_u8(mr + p, o + 16, additive);
                }
        }
    }
}
