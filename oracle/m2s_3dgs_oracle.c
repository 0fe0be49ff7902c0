/* m2s_3dgs_oracle.c — plain-C restatement of the standard 3DGS render (m2s_3dgs_render; beyond the reference: graphdeco's
 * preprocessCUDA + renderCUDA for the project's GL camera, DESIGN §2) (TEST INFRASTRUCTURE: the checker of m2s_3dgs.cu).
 * Built with gcc -ffp-contract=off: every operation is one IEEE fp32 rounding, in the order DESIGN §2 states; the exp is
 * orc_splat_exp (libm2s_splat_oracle.so, the project's rn_exp), the SH colour orc_sh_colours (libm2s_sh_oracle.so).
 *
 * Records: n records of the layout (0 REF96 / M2S_VIEW_PLY*: 24 floats, 1 PACKED56: 14 floats).  Splat records: 12 floats
 * each, as the kernel writes them (zero for a culled record); keys: the bits of the view depth, 0xFFFFFFFF when culled. */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

float orc_splat_exp(float x);
int orc_sh_camera(const float* V, const float* M, float cam[3]);
void orc_sh_colours(const float* gaussians, uint32_t n, const float* sh, uint32_t buffer_degree, uint32_t sh_degree, const float cam[3],
                    float* rgb);

enum { LAYOUT_REF96 = 0, LAYOUT_PACKED56 = 1, VIEW_PLY = 16, VIEW_PLY_PBR = 17 };

/* (int)x as the GPU's cvt.rzi.s32.f32 gives it: toward zero, saturated, NaN -> 0 */
static int trunc_sat(float x) {
    if (x != x) return 0;
    if (x >= 2147483648.0f) return INT_MAX;
    if (x <= -2147483648.0f) return INT_MIN;
    return (int)x;
}
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }

/* row r of the column-major m applied to (x, y, z, 1) */
static float row4(const float* m, int r, float x, float y, float z) { return ((m[r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r]; }

/* V M in fp64 from the fp32 matrices, rounded once to fp32 (the host code's sh_camera) */
static void view_model(const float* V, const float* M, float mv[16]) {
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r)
            mv[c * 4 + r] = (float)((((double)V[r] * M[c * 4] + (double)V[4 + r] * M[c * 4 + 1]) + (double)V[8 + r] * M[c * 4 + 2]) +
                                    (double)V[12 + r] * M[c * 4 + 3]);
}

/* the fields of record i: position, colour, opacity, scale, rotation (w, x, y, z) */
static void fields(const float* records, uint32_t layout, uint32_t i, float p[3], float col[3], float* op, float s[3], float q[4]) {
    if (layout == LAYOUT_PACKED56) {
        const float* f = records + (size_t)i * 14;
        const float kC0 = 0.28209479177387814f;
        p[0] = f[0]; p[1] = f[1]; p[2] = f[2];
        q[0] = f[3]; q[1] = f[4]; q[2] = f[5]; q[3] = f[6];
        s[0] = orc_splat_exp(f[7]); s[1] = orc_splat_exp(f[8]); s[2] = orc_splat_exp(f[9]);
        col[0] = f[10] * kC0 + 0.5f; col[1] = f[11] * kC0 + 0.5f; col[2] = f[12] * kC0 + 0.5f;
        *op = 1.0f / (1.0f + orc_splat_exp(-f[13]));
    } else {
        const float* g = records + (size_t)i * 24;
        p[0] = g[0]; p[1] = g[1]; p[2] = g[2];
        col[0] = g[4]; col[1] = g[5]; col[2] = g[6]; *op = g[7];
        s[0] = g[8]; s[1] = g[9]; s[2] = g[10];
        q[0] = g[16]; q[1] = g[17]; q[2] = g[18]; q[3] = g[19];
    }
}

/* one record -> splat record (12 floats) and key; 0 if culled.  rgb: the record's colour after SH (or NULL: max(c, 0)) */
static int splat(const float* records, uint32_t layout, uint32_t i, const float* MV, const float* P, uint32_t width, uint32_t height,
                 float near, float mult, float scale_modifier, const float* rgb, float out[12], uint32_t* key) {
    float p[3], col[3], op, sc[3], q[4];
    fields(records, layout, i, p, col, &op, sc, q);
    const float tx = row4(MV, 0, p[0], p[1], p[2]), ty = row4(MV, 1, p[0], p[1], p[2]), tz = row4(MV, 2, p[0], p[1], p[2]);
    const float d = -tz;
    if (!(d > near)) return 0;
    const float c0 = row4(P, 0, tx, ty, tz), c1 = row4(P, 1, tx, ty, tz), c3 = row4(P, 3, tx, ty, tz);
    const float pw = 1.0f / (c3 + 1e-7f);
    const float W = (float)width, H = (float)height;
    const float u = (((c0 * pw) + 1.0f) * W - 1.0f) * 0.5f, v = (((c1 * pw) + 1.0f) * H - 1.0f) * 0.5f;
    const float s[3] = {(sc[0] * mult) * scale_modifier, (sc[1] * mult) * scale_modifier, (sc[2] * mult) * scale_modifier};
    const float qn = fmaxf(sqrtf(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]), 1e-12f);
    const float qr = q[0] / qn, qi = q[1] / qn, qj = q[2] / qn, qk = q[3] / qn;
    const float R[3][3] = {{1.0f - 2.0f * (qj * qj + qk * qk), 2.0f * (qi * qj - qr * qk), 2.0f * (qi * qk + qr * qj)},
                           {2.0f * (qi * qj + qr * qk), 1.0f - 2.0f * (qi * qi + qk * qk), 2.0f * (qj * qk - qr * qi)},
                           {2.0f * (qi * qk - qr * qj), 2.0f * (qj * qk + qr * qi), 1.0f - 2.0f * (qi * qi + qj * qj)}};
    float Mk[3][3], S[3][3];
    for (int k = 0; k < 3; ++k)
        for (int j = 0; j < 3; ++j) Mk[k][j] = s[k] * R[j][k];
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) S[a][b] = (Mk[0][a] * Mk[0][b] + Mk[1][a] * Mk[1][b]) + Mk[2][a] * Mk[2][b];
    const float fx = (P[0] * W) * 0.5f, fy = (P[5] * H) * 0.5f;
    const float limx = 1.3f / P[0], limy = 1.3f / P[5];
    const float txc = fminf(limx, fmaxf(-limx, tx / d)) * d, tyc = fminf(limy, fmaxf(-limy, ty / d)) * d;
    const float dd = d * d;
    const float J00 = fx / d, J02 = (fx * txc) / dd, J11 = fy / d, J12 = (fy * tyc) / dd;
    float T[2][3], A[2][3];
    for (int j = 0; j < 3; ++j) {
        T[0][j] = J00 * MV[4 * j + 0] + J02 * MV[4 * j + 2];
        T[1][j] = J11 * MV[4 * j + 1] + J12 * MV[4 * j + 2];
    }
    for (int a = 0; a < 2; ++a)
        for (int j = 0; j < 3; ++j) A[a][j] = (T[a][0] * S[0][j] + T[a][1] * S[1][j]) + T[a][2] * S[2][j];
    const float ca = ((A[0][0] * T[0][0] + A[0][1] * T[0][1]) + A[0][2] * T[0][2]) + 0.3f;
    const float cb = (A[0][0] * T[1][0] + A[0][1] * T[1][1]) + A[0][2] * T[1][2];
    const float cc = ((A[1][0] * T[1][0] + A[1][1] * T[1][1]) + A[1][2] * T[1][2]) + 0.3f;
    const float det = ca * cc - cb * cb;
    if (det == 0.0f) return 0;
    const float inv = 1.0f / det;
    const float mid = 0.5f * (ca + cc);
    const float sq = sqrtf(fmaxf(0.1f, mid * mid - det));
    const float radius = ceilf(3.0f * sqrtf(fmaxf(mid + sq, mid - sq)));
    const int gx = (int)((width + 15) / 16), gy = (int)((height + 15) / 16);
    const int x0 = imin(gx, imax(0, trunc_sat((u - radius) * 0.0625f))), y0 = imin(gy, imax(0, trunc_sat((v - radius) * 0.0625f)));
    const int x1 = imin(gx, imax(0, trunc_sat(((u + radius) + 15.0f) * 0.0625f))), y1 = imin(gy, imax(0, trunc_sat(((v + radius) + 15.0f) * 0.0625f)));
    if ((x1 - x0) * (y1 - y0) == 0) return 0;
    float r[3];
    for (int c = 0; c < 3; ++c) {
        const float x = rgb ? rgb[(size_t)i * 3 + c] : col[c];
        r[c] = x < 0.0f ? 0.0f : x;
    }
    const uint32_t rx = (uint32_t)x0 | (uint32_t)x1 << 16, ry = (uint32_t)y0 | (uint32_t)y1 << 16;
    out[0] = u; out[1] = v; out[2] = cc * inv; out[3] = -cb * inv;
    out[4] = ca * inv; out[5] = op; out[6] = r[0]; out[7] = r[1];
    out[8] = r[2]; memcpy(out + 9, &rx, 4); memcpy(out + 10, &ry, 4); out[11] = radius;
    memcpy(key, &d, 4);
    return 1;
}

/* the preprocess of every record; the survivors, UINT32_MAX for arguments m2s_3dgs_render rejects as singular */
ORC_API uint32_t orc_3dgs_preprocess(const float* records, uint32_t n, uint32_t layout, const float* V, const float* P, const float* M,
                                     uint32_t width, uint32_t height, float near, float std_dev, float scale_modifier, const float* sh,
                                     uint32_t buffer_degree, uint32_t sh_degree, float* splats, uint32_t* keys) {
    float cam[3], MV[16];
    if (!orc_sh_camera(V, M, cam)) return UINT32_MAX;
    view_model(V, M, MV);
    float* rgb = NULL;
    if (sh_degree > 0 && n > 0) {
        rgb = (float*)malloc((size_t)n * 3 * sizeof(float));
        if (!rgb) return UINT32_MAX;
        orc_sh_colours(records, n, sh, buffer_degree, sh_degree, cam, rgb);
    }
    const float mult = layout == LAYOUT_REF96 ? std_dev : 1.0f;
    const uint32_t rec_layout = layout == LAYOUT_PACKED56 ? LAYOUT_PACKED56 : LAYOUT_REF96;
    uint32_t alive = 0;
    for (uint32_t i = 0; i < n; ++i) {
        memset(splats + (size_t)i * 12, 0, 12 * sizeof(float));
        keys[i] = 0xFFFFFFFFu;
        alive += (uint32_t)splat(records, rec_layout, i, MV, P, width, height, near, mult, scale_modifier, rgb, splats + (size_t)i * 12, keys + i);
    }
    free(rgb);
    return alive;
}

static const uint32_t* g_keys;
static int by_key(const void* a, const void* b) {
    const uint32_t i = *(const uint32_t*)a, j = *(const uint32_t*)b;
    if (g_keys[i] != g_keys[j]) return g_keys[i] < g_keys[j] ? -1 : 1;
    return i < j ? -1 : (i > j);
}

static float sat(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }
static uint8_t unorm8(float v) { return (uint8_t)nearbyintf(sat(v) * 255.0f); }

/* the render: rgba32f (W x H x 4 floats) and rgba8 (W x H x 4 bytes), either may be NULL; *drawn the depth-ordered prefix
 * whose pairs fit max_pairs, *pairs the pairs every survivor needs.  0, or 1 for singular arguments / no memory. */
ORC_API int orc_3dgs_render(const float* records, uint32_t n, uint32_t layout, const float* V, const float* P, const float* M, uint32_t width,
                            uint32_t height, float near, float std_dev, float scale_modifier, const float background[3], const float* sh,
                            uint32_t buffer_degree, uint32_t sh_degree, uint64_t max_pairs, float* rgba32f, uint8_t* rgba8, uint32_t* drawn,
                            uint64_t* pairs) {
    float* sp = (float*)malloc(((size_t)n + 1) * 12 * sizeof(float));
    uint32_t* keys = (uint32_t*)malloc(((size_t)n + 1) * sizeof(uint32_t));
    uint32_t* order = (uint32_t*)malloc(((size_t)n + 1) * sizeof(uint32_t));
    const uint32_t gx = (width + 15) / 16, gy = (height + 15) / 16, ntiles = gx * gy;
    uint32_t* tcount = (uint32_t*)calloc((size_t)ntiles + 1, sizeof(uint32_t));
    int rc = 1;
    uint32_t* toff = NULL;
    uint32_t* lists = NULL;
    if (!sp || !keys || !order || !tcount) goto out;
    const uint32_t alive = orc_3dgs_preprocess(records, n, layout, V, P, M, width, height, near, std_dev, scale_modifier, sh, buffer_degree,
                                               sh_degree, sp, keys);
    if (alive == UINT32_MAX) goto out;
    for (uint32_t i = 0; i < n; ++i) order[i] = i;
    g_keys = keys;
    qsort(order, n, sizeof(uint32_t), by_key);
    /* the survivors come first; the prefix whose pairs fit */
    uint64_t total = 0, fit = 0;
    uint32_t nd = 0;
    for (uint32_t k = 0; k < alive; ++k) {
        const float* s = sp + (size_t)order[k] * 12;
        uint32_t rx, ry;
        memcpy(&rx, s + 9, 4); memcpy(&ry, s + 10, 4);
        const uint64_t np = (uint64_t)((rx >> 16) - (rx & 0xFFFFu)) * ((ry >> 16) - (ry & 0xFFFFu));
        total += np;
        if (total <= max_pairs) { nd = k + 1; fit = total; }
    }
    *drawn = nd;
    *pairs = total;
    /* each tile's gaussians in depth order */
    for (uint32_t k = 0; k < nd; ++k) {
        const float* s = sp + (size_t)order[k] * 12;
        uint32_t rx, ry;
        memcpy(&rx, s + 9, 4); memcpy(&ry, s + 10, 4);
        for (uint32_t ty = ry & 0xFFFFu; ty < (ry >> 16); ++ty)
            for (uint32_t tx = rx & 0xFFFFu; tx < (rx >> 16); ++tx) tcount[ty * gx + tx]++;
    }
    toff = (uint32_t*)calloc((size_t)ntiles + 1, sizeof(uint32_t));
    lists = (uint32_t*)malloc((size_t)(fit + 1) * sizeof(uint32_t));
    if (!toff || !lists) goto out;
    for (uint32_t t = 0; t < ntiles; ++t) toff[t + 1] = toff[t] + tcount[t];
    memset(tcount, 0, (size_t)ntiles * sizeof(uint32_t));
    for (uint32_t k = 0; k < nd; ++k) {
        const float* s = sp + (size_t)order[k] * 12;
        uint32_t rx, ry;
        memcpy(&rx, s + 9, 4); memcpy(&ry, s + 10, 4);
        for (uint32_t ty = ry & 0xFFFFu; ty < (ry >> 16); ++ty)
            for (uint32_t tx = rx & 0xFFFFu; tx < (rx >> 16); ++tx) {
                const uint32_t t = ty * gx + tx;
                lists[toff[t] + tcount[t]++] = order[k];
            }
    }
    /* per pixel: front to back */
    for (uint32_t y = 0; y < height; ++y)
        for (uint32_t x = 0; x < width; ++x) {
            const uint32_t t = (y / 16) * gx + x / 16;
            const float px = (float)x, py = (float)y;
            float T = 1.0f, C[3] = {0.0f, 0.0f, 0.0f};
            for (uint32_t k = toff[t]; k < toff[t + 1]; ++k) {
                const float* s = sp + (size_t)lists[k] * 12;
                const float dx = s[0] - px, dy = s[1] - py;
                const float power = -0.5f * ((s[2] * dx) * dx + (s[4] * dy) * dy) - (s[3] * dx) * dy;
                if (power > 0.0f) continue;
                const float alpha = fminf(0.99f, s[5] * orc_splat_exp(power));
                if (alpha < 1.0f / 255.0f) continue;
                const float tt = T * (1.0f - alpha);
                if (tt < 0.0001f) break;
                for (int c = 0; c < 3; ++c) C[c] = C[c] + (s[6 + c] * alpha) * T;
                T = tt;
            }
            const float o[4] = {C[0] + T * background[0], C[1] + T * background[1], C[2] + T * background[2], 1.0f - T};
            const size_t pix = (size_t)y * width + x;
            for (int c = 0; c < 4; ++c) {
                if (rgba32f) rgba32f[pix * 4 + c] = o[c];
                if (rgba8) rgba8[pix * 4 + c] = unorm8(o[c]);
            }
        }
    rc = 0;
out:
    free(sp); free(keys); free(order); free(tcount); free(toff); free(lists);
    return rc;
}
