/* m2s_mesh_oracle.c — CPU restatement of the viewer's mesh G-buffer pass and of the split-screen composite of the
 * deferred lighting (SURVEY 8 row 14).
 *
 * TEST INFRASTRUCTURE ONLY, like m2s_oracle.c: nothing under mesh2splat_b200/ includes, links or calls it.  Linked with
 * m2s_splat_oracle.c (orc_f2h, orc_splat_exp) and m2s_depth_oracle.c (orc_depth_code).
 *
 * Restated (paths relative to the reference tree):
 *   mesh pass      src/renderer/renderPasses/MeshRenderPass.cpp:8-73, meshRenderVS.glsl, meshRenderPS.glsl, common.glsl
 *   split screen   src/renderer/renderPasses/GaussianRelightingPass.cpp:90-135
 * The fixed-function parts are DESIGN §2 "The mesh G-buffer pass": gl_Position = P (V (M p)) with GLM's mat4 * vec4, the
 * normal matrix from GLM's fp32 inverse, the depth pass's clipping (here carrying source barycentrics), fan, snap and
 * rasteriser, back faces (negative snapped area) culled, D24 LESS in draw order (primitive table order, then triangle
 * order), perspective-correct interpolation in fp64 from the exact edge values, the LOD from the coarse derivatives of
 * the winner's uv over the 2 x 2 quad, the conversion kernels' sampler (bilinear weights with fused multiply-adds), and
 * the splat draw's target formats.
 *
 * The triangles are drawn in order, fan triangle by fan triangle, pixel by pixel (GL's order); each pixel's last winner
 * is then shaded once.
 *
 * Arithmetic: fp32 / fp64, one rounding per operation (built with -ffp-contract=off); fmaf where the sampler fuses.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))
#define MAX_POLY 9
#define GUARD 2.0f
#define CLEAR_CODE 0xFFFFFFu

uint16_t orc_f2h(float f);
float orc_splat_exp(float x);
int orc_depth_code(double z, uint32_t* code);

/* ---- host uniforms: GLM 1.0.1's fp32 compute_inverse<4, 4>, transposed, upper 3 x 3; 0 for a singular matrix ------- */
ORC_API int orc_mesh_normal_matrix(const float* M, float* N) {
#define m(c, r) M[4 * (c) + (r)]
    const float c00 = m(2, 2) * m(3, 3) - m(3, 2) * m(2, 3), c02 = m(1, 2) * m(3, 3) - m(3, 2) * m(1, 3), c03 = m(1, 2) * m(2, 3) - m(2, 2) * m(1, 3);
    const float c04 = m(2, 1) * m(3, 3) - m(3, 1) * m(2, 3), c06 = m(1, 1) * m(3, 3) - m(3, 1) * m(1, 3), c07 = m(1, 1) * m(2, 3) - m(2, 1) * m(1, 3);
    const float c08 = m(2, 1) * m(3, 2) - m(3, 1) * m(2, 2), c10 = m(1, 1) * m(3, 2) - m(3, 1) * m(1, 2), c11 = m(1, 1) * m(2, 2) - m(2, 1) * m(1, 2);
    const float c12 = m(2, 0) * m(3, 3) - m(3, 0) * m(2, 3), c14 = m(1, 0) * m(3, 3) - m(3, 0) * m(1, 3), c15 = m(1, 0) * m(2, 3) - m(2, 0) * m(1, 3);
    const float c16 = m(2, 0) * m(3, 2) - m(3, 0) * m(2, 2), c18 = m(1, 0) * m(3, 2) - m(3, 0) * m(1, 2), c19 = m(1, 0) * m(2, 2) - m(2, 0) * m(1, 2);
    const float c20 = m(2, 0) * m(3, 1) - m(3, 0) * m(2, 1), c22 = m(1, 0) * m(3, 1) - m(3, 0) * m(1, 1), c23 = m(1, 0) * m(2, 1) - m(2, 0) * m(1, 1);
    const float f0[4] = {c00, c00, c02, c03}, f1[4] = {c04, c04, c06, c07}, f2[4] = {c08, c08, c10, c11};
    const float f3[4] = {c12, c12, c14, c15}, f4[4] = {c16, c16, c18, c19}, f5[4] = {c20, c20, c22, c23};
    const float sa[4] = {1, -1, 1, -1}, sb[4] = {-1, 1, -1, 1};
    float v0[4], v1[4], v2[4], v3[4], inv[4][4];
    for (int i = 0; i < 4; ++i) {
        const int c = i == 0 ? 1 : 0;
        v0[i] = m(c, 0); v1[i] = m(c, 1); v2[i] = m(c, 2); v3[i] = m(c, 3);
    }
    for (int i = 0; i < 4; ++i) {
        inv[0][i] = (v1[i] * f0[i] - v2[i] * f1[i] + v3[i] * f2[i]) * sa[i];
        inv[1][i] = (v0[i] * f0[i] - v2[i] * f3[i] + v3[i] * f4[i]) * sb[i];
        inv[2][i] = (v0[i] * f1[i] - v1[i] * f3[i] + v3[i] * f5[i]) * sa[i];
        inv[3][i] = (v0[i] * f2[i] - v1[i] * f4[i] + v2[i] * f5[i]) * sb[i];
    }
    const float det = (m(0, 0) * inv[0][0] + m(0, 1) * inv[1][0]) + (m(0, 2) * inv[2][0] + m(0, 3) * inv[3][0]);
#undef m
    if (det == 0.0f || !isfinite(det)) return 0;
    const float ood = 1.0f / det;
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) N[c * 3 + r] = inv[r][c] * ood;
    return 1;
}

/* ---- the fixed sequences shared with the kernel ------------------------------------------------------------------- */
ORC_API double orc_mesh_log2(double x) {
    if (x != x) return x;
    if (x == 0.0) return -INFINITY;
    if (isinf(x)) return x;
    int e;
    double m = frexp(x, &e);
    if (m < 0.70710678118654752440) { m = m * 2.0; e -= 1; }
    const double f = (m + -1.0) / (m + 1.0), f2 = f * f;
    double p = 1.0 / 19.0;
    p = p * f2 + 1.0 / 17.0;
    p = p * f2 + 1.0 / 15.0;
    p = p * f2 + 1.0 / 13.0;
    p = p * f2 + 1.0 / 11.0;
    p = p * f2 + 1.0 / 9.0;
    p = p * f2 + 1.0 / 7.0;
    p = p * f2 + 1.0 / 5.0;
    p = p * f2 + 1.0 / 3.0;
    p = p * f2 + 1.0;
    return (double)e + ((2.0 * f) * p) * 1.4426950408889634074;
}

ORC_API double orc_mesh_sin(double x) {
    if (!isfinite(x)) return x - x;
    const double k = rint(x * 6.36619772367581382433e-01);
    double r = x + -(k * 1.570796012878418);
    r = r + -(k * 3.139164164167596e-07);
    r = r + -(k * 6.22337468017542e-14);
    r = r + -(k * -2.508278806334166e-20);
    const double z = r * r;
    double s = 1.58969099521155010221e-10;
    s = s * z + -2.50507602534068634195e-08;
    s = s * z + 2.75573137070700676789e-06;
    s = s * z + -1.98412698298579493134e-04;
    s = s * z + 8.33333333332248946124e-03;
    s = s * z + -1.66666666666666324348e-01;
    s = r + (r * z) * s;
    double c = -1.13596475577881948265e-11;
    c = c * z + 2.08757232129817482790e-09;
    c = c * z + -2.75573143513906633035e-07;
    c = c * z + 2.48015872894767294178e-05;
    c = c * z + -1.38888888888741095749e-03;
    c = c * z + 4.16666666666666019037e-02;
    c = (1.0 + -(0.5 * z)) + (z * z) * c;
    switch ((int)((long long)k & 3)) {
        case 0: return s;
        case 1: return c;
        case 2: return -s;
        default: return -c;
    }
}

/* fract(sin(arg) * 43758.5453) of render mode 3 */
ORC_API float orc_mesh_hash(float arg) {
    const float v = (float)orc_mesh_sin((double)arg) * 43758.5453f;
    return v - floorf(v);
}

/* ---- vertex stage ----------------------------------------------------------------------------------------------------- */
static float m4row(const float* m, int row, float x, float y, float z, float w) {
    return (m[row] * x + m[4 + row] * y) + (m[8 + row] * z + m[12 + row] * w);
}
static void normalize3(float* v) {
    const float i = 1.0f / sqrtf((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    v[0] = v[0] * i; v[1] = v[1] * i; v[2] = v[2] * i;
}
static void mat3mul(const float* n, float x, float y, float z, float* r) {
    for (int k = 0; k < 3; ++k) r[k] = (n[k] * x + n[3 + k] * y) + n[6 + k] * z;
}

typedef struct { const float *M, *V, *P; float N[9]; } uni;

/* meshRenderVS.glsl for vertex k of a triangle (36 floats): clip position, and the 13 varyings worldPos, v_normal,
 * v_tangent, v_uv, v_viewDepth */
ORC_API void orc_mesh_vs_one(const float* vtx12, const float* M, const float* V, const float* P, const float* N, float* clip4, float* vary13) {
    const float* p = vtx12;
    float w[4], v[4];
    for (int r = 0; r < 4; ++r) w[r] = m4row(M, r, p[0], p[1], p[2], 1.0f);
    for (int r = 0; r < 4; ++r) v[r] = m4row(V, r, w[0], w[1], w[2], w[3]);
    for (int r = 0; r < 4; ++r) clip4[r] = m4row(P, r, v[0], v[1], v[2], v[3]);
    if (!vary13) return;
    float n[3], t[3];
    mat3mul(N, p[3], p[4], p[5], n);
    normalize3(n);
    mat3mul(N, p[6], p[7], p[8], t);
    normalize3(t);
    vary13[0] = w[0]; vary13[1] = w[1]; vary13[2] = w[2];
    vary13[3] = n[0]; vary13[4] = n[1]; vary13[5] = n[2];
    vary13[6] = t[0]; vary13[7] = t[1]; vary13[8] = t[2]; vary13[9] = p[9];
    vary13[10] = p[10]; vary13[11] = p[11];
    vary13[12] = -v[2];
}

/* ---- clip with barycentrics ------------------------------------------------------------------------------------------ */
typedef struct { float x, y, z, w, b[3]; } cv;

static float plane(const cv* v, int p) {
    const float gw = GUARD * v->w;
    switch (p) {
        case 0: return v->z + v->w;
        case 1: return v->w - v->z;
        case 2: return v->x + gw;
        case 3: return gw - v->x;
        case 4: return v->y + gw;
        default: return gw - v->y;
    }
}
static float lerp1(float a, float b, float t) { return a + t * (b - a); }
static cv cut(const cv* a, const cv* b, float da, float db) {
    const float t = da / (da - db);
    cv r = {lerp1(a->x, b->x, t), lerp1(a->y, b->y, t), lerp1(a->z, b->z, t), lerp1(a->w, b->w, t),
            {lerp1(a->b[0], b->b[0], t), lerp1(a->b[1], b->b[1], t), lerp1(a->b[2], b->b[2], t)}};
    return r;
}

static int mesh_poly(const float* tri36, const uni* u, cv* v) {
    for (int k = 0; k < 3; ++k) {
        float c[4];
        orc_mesh_vs_one(tri36 + 12 * k, u->M, u->V, u->P, u->N, c, NULL);
        v[k].x = c[0]; v[k].y = c[1]; v[k].z = c[2]; v[k].w = c[3];
        for (int j = 0; j < 3; ++j) v[k].b[j] = j == k ? 1.0f : 0.0f;
        if (!isfinite(c[0]) || !isfinite(c[1]) || !isfinite(c[2]) || !isfinite(c[3])) return 0;
    }
    int n = 3;
    for (int p = 0; p < 6 && n > 0; ++p) {
        cv o[MAX_POLY];
        int m = 0;
        for (int i = 0; i < n; ++i) {
            const int prev = i == 0 ? n - 1 : i - 1;
            const float dc = plane(&v[i], p), dp = plane(&v[prev], p);
            if (dc >= 0.0f) {
                if (dp < 0.0f && m < MAX_POLY) o[m++] = cut(&v[i], &v[prev], dc, dp);
                if (m < MAX_POLY) o[m++] = v[i];
            } else if (dp >= 0.0f && m < MAX_POLY) {
                o[m++] = cut(&v[prev], &v[i], dp, dc);
            }
        }
        memcpy(v, o, sizeof(cv) * (size_t)m);
        n = m;
    }
    return n;
}

/* ---- fan triangle: snap, cull, edge functions (the splat draw's rasteriser) -------------------------------------------- */
typedef struct { int64_t A[3], B[3], C[3]; int incl[3]; int x0, x1, y0, y1; float z[3]; double w[3], b[3][3]; } ftri;

static void snap(float nx, float ny, float W, float H, int* ok, int32_t* X, int32_t* Y) {
    const float hw = W * 0.5f, hh = H * 0.5f;
    const float xw = nx * hw + hw, yw = ny * hh + hh;
    *ok = isfinite(xw) && isfinite(yw) && fabsf(xw) <= 8192.0f && fabsf(yw) <= 8192.0f;
    *X = *ok ? (int32_t)lrintf(xw * 256.0f) : 0;
    *Y = *ok ? (int32_t)lrintf(yw * 256.0f) : 0;
}

static void fan_setup(const cv* v, int k, uint32_t W, uint32_t H, ftri* s) {
    memset(s, 0, sizeof(*s));
    s->x1 = -1; s->y1 = -1;
    int32_t X[3], Y[3];
    int ok = 1;
    for (int c = 0; c < 3; ++c) {
        const cv* p = &v[c == 0 ? 0 : k + c];
        int okc;
        snap(p->x / p->w, p->y / p->w, (float)W, (float)H, &okc, &X[c], &Y[c]);
        ok = ok && okc;
        s->z[c] = (p->z / p->w) * 0.5f + 0.5f;
        s->w[c] = (double)p->w;
        for (int j = 0; j < 3; ++j) s->b[c][j] = (double)p->b[j];
    }
    if (!ok) return;
    const int64_t area2 = (int64_t)(X[1] - X[0]) * (Y[2] - Y[0]) - (int64_t)(X[2] - X[0]) * (Y[1] - Y[0]);
    if (area2 <= 0) return;   /* zero area: nothing; negative (clockwise, y up): a back face, culled */
    for (int e = 0; e < 3; ++e) {
        const int a = (e + 1) % 3, b = (e + 2) % 3;
        const int64_t dx = X[b] - X[a], dy = Y[b] - Y[a];
        s->A[e] = -dy * 256;
        s->B[e] = dx * 256;
        s->C[e] = dx * (128 - (int64_t)Y[a]) - dy * (128 - (int64_t)X[a]);
        s->incl[e] = (s->A[e] > 0) || (s->A[e] == 0 && s->B[e] > 0);
    }
    int32_t xmin = X[0], xmax = X[0], ymin = Y[0], ymax = Y[0];
    for (int c = 1; c < 3; ++c) {
        if (X[c] < xmin) xmin = X[c];
        if (X[c] > xmax) xmax = X[c];
        if (Y[c] < ymin) ymin = Y[c];
        if (Y[c] > ymax) ymax = Y[c];
    }
    int64_t x0 = ((int64_t)xmin + 127) >> 8, x1 = ((int64_t)xmax - 128) >> 8;
    int64_t y0 = ((int64_t)ymin + 127) >> 8, y1 = ((int64_t)ymax - 128) >> 8;
    if (x0 < 0) x0 = 0;
    if (y0 < 0) y0 = 0;
    if (x1 > (int64_t)W - 1) x1 = (int64_t)W - 1;
    if (y1 > (int64_t)H - 1) y1 = (int64_t)H - 1;
    s->x0 = (int)x0; s->x1 = (int)x1; s->y0 = (int)y0; s->y1 = (int)y1;
}

static int covers(const ftri* s, int i, int j, int64_t* e) {
    for (int k = 0; k < 3; ++k) {
        e[k] = s->A[k] * i + s->B[k] * j + s->C[k];
        if (e[k] < 0 || (e[k] == 0 && !s->incl[k])) return 0;
    }
    return 1;
}

static int tri_touches(const ftri* s, int tx, int ty) {
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

/* GL 4.6 §14.6.1: source weights beta at pixel (i, j), extrapolated outside the triangle */
static void weights(const ftri* s, int i, int j, double* beta) {
    double q[3];
    for (int c = 0; c < 3; ++c) q[c] = (double)(s->A[c] * i + s->B[c] * j + s->C[c]) / s->w[c];
    const double sum = (q[0] + q[1]) + q[2];
    for (int k = 0; k < 3; ++k) beta[k] = ((q[0] * s->b[0][k] + q[1] * s->b[1][k]) + q[2] * s->b[2][k]) / sum;
}
static float interp(const double* beta, const float (*vary)[13], int i) {
    return (float)((beta[0] * (double)vary[0][i] + beta[1] * (double)vary[1][i]) + beta[2] * (double)vary[2][i]);
}

/* ---- the conversion kernels' sampler (m2s_shade.cuh): REPEAT, bilinear weights with fused multiply-adds ---------------- */
typedef struct { uint32_t off[5], w[5], h[5], nlevels; } mtex;

static float fast_floor(float x, int* i) {
    const float t = (x - 0.5f) + 12582912.0f;
    uint32_t b;
    memcpy(&b, &t, 4);
    *i = (int)b - 0x4B400000;
    return t - 12582912.0f;
}
static float wrap01(float u) {
    int d;
    u = fminf(fmaxf(u, -1048576.0f), 1048576.0f);
    return u - fast_floor(u, &d);
}
static void footprint(int ix, int iy, int W, int H, uint32_t* idx) {
    const int x0 = ix + ((ix >> 31) & W), y0 = iy + ((iy >> 31) & H);
    const int x1 = x0 + 1 == W ? 0 : x0 + 1, y1 = y0 + 1 == H ? 0 : y0 + 1;
    idx[0] = (uint32_t)(y0 * W + x0); idx[1] = (uint32_t)(y0 * W + x1);
    idx[2] = (uint32_t)(y1 * W + x0); idx[3] = (uint32_t)(y1 * W + x1);
}

/* the level pair of a map (level-0 size W0 x H0, nlevels levels) for the quad's uv steps: the first level and the blend
 * fraction toward the next.  A NaN rho samples level 0, +inf the last level. */
ORC_API void orc_mesh_level(uint32_t W0, uint32_t H0, uint32_t nlevels, float dudx, float dvdx, float dudy, float dvdy, int* l0_, float* frac_) {
    const float W = (float)W0, H = (float)H0;
    const float ax = dudx * W, bx = dvdx * H, ay = dudy * W, by = dvdy * H;
    const float sx = ax * ax + bx * bx, sy = ay * ay + by * by;
    const float s2 = (sx != sx || sy != sy) ? NAN : fmaxf(sx, sy);
    const float lam = (float)(0.5 * orc_mesh_log2((double)s2));
    const int q = (int)nlevels - 1;
    int l0 = 0;
    float frac = 0.0f;
    if (!(lam > 0.0f)) l0 = 0;
    else if (lam >= (float)q) l0 = q;
    else { const float d = floorf(lam); l0 = (int)d; frac = lam - d; }
    *l0_ = l0;
    *frac_ = frac;
}

/* texture() of one map at uv with the quad's uv steps: RGBA in [0, 1] */
static void sample(const mtex* t, const uint32_t* arena, float u, float v, float dudx, float dvdx, float dudy, float dvdy, float* out) {
    int l0;
    float frac;
    orc_mesh_level(t->w[0], t->h[0], t->nlevels, dudx, dvdx, dudy, dvdy, &l0, &frac);
    const int q = (int)t->nlevels - 1;
    const int l1 = l0 + 1 < q ? l0 + 1 : q;
    u = wrap01(u); v = wrap01(v);
    const int lv[2] = {l0, l1};
    const float lw[2] = {1.0f - frac, frac};
    float acc[2][4];
    for (int h = 0; h < 2; ++h) {
        const uint32_t Wl = t->w[lv[h]], Hl = t->h[lv[h]];
        const float x = fmaf(u, (float)Wl, -0.5f), y = fmaf(v, (float)Hl, -0.5f);
        int ix, iy;
        const float fx = fast_floor(x, &ix), fy = fast_floor(y, &iy);
        const float axx = fmaf(fx, -1.0f, x), ayy = fmaf(fy, -1.0f, y);
        uint32_t idx[4], tx[4];
        footprint(ix, iy, (int)Wl, (int)Hl, idx);
        const int load = h == 0 || frac > 0.0f;
        for (int c = 0; c < 4; ++c) tx[c] = load ? arena[t->off[lv[h]] + idx[c]] : 0u;
        const float k = lw[h] * (1.0f / 255.0f);
        const float bxx = fmaf(axx, -1.0f, 1.0f);
        const float cy = ayy * k, byy = fmaf(ayy, -k, k);
        const float w00 = bxx * byy, w10 = axx * byy, w01 = bxx * cy, w11 = axx * cy;
        for (int ch = 0; ch < 4; ++ch) {
            float a = w00 * (float)((tx[0] >> (8 * ch)) & 255u);
            a = fmaf(w10, (float)((tx[1] >> (8 * ch)) & 255u), a);
            a = fmaf(w01, (float)((tx[2] >> (8 * ch)) & 255u), a);
            a = fmaf(w11, (float)((tx[3] >> (8 * ch)) & 255u), a);
            acc[h][ch] = a;
        }
    }
    for (int ch = 0; ch < 4; ++ch) out[ch] = acc[0][ch] + acc[1][ch];
}

/* ---- the pass ----------------------------------------------------------------------------------------------------- */
static float clamp01(float x) { const float t = x < 0.0f ? 0.0f : x; return 1.0f < t ? 1.0f : t; }   /* GLM clamp */
static uint8_t u8(float v) { return (uint8_t)lrintf(fminf(fmaxf(v, 0.0f), 1.0f) * 255.0f); }

typedef struct {
    const float* tris;
    const uint32_t *prim_first, *prim_count;
    const float* prim_factor;
    const int32_t* prim_tex;
    const mtex* texs;
    const uint32_t* arena;
    uni u;
    float near_far[2];
    uint32_t W, H, mode;
} pass;

/* meshRenderPS.glsl for one fragment: v13 the interpolated varyings (worldPos, v_normal, v_tangent, v_uv, v_viewDepth),
 * tex12 what texture() returns for the albedo, normal and metallic-roughness maps (RGBA each), has bit m: map m is bound,
 * prim_id gl_PrimitiveID.  out20: gPosition, gNormal, gAlbedo, gDepth, gMetallicRoughness as fp32 values, before the
 * targets' formats. */
ORC_API void orc_mesh_fs(const float* v, const float* tex12, uint32_t has, const float* fac, const float* near_far, uint32_t mode,
                         uint32_t prim_id, float* out) {
    float alb[3] = {fac[0], fac[1], fac[2]};
    if (has & 1u)
        for (int c = 0; c < 3; ++c) alb[c] = alb[c] * tex12[c];
    float N[3] = {v[3], v[4], v[5]};
    normalize3(N);
    if (has & 2u) {
        const float* tx = tex12 + 4;
        float m[3] = {tx[0] * 2.0f - 1.0f, tx[1] * 2.0f - 1.0f, tx[2] * 2.0f - 1.0f};
        normalize3(m);
        float T[3] = {v[6], v[7], v[8]};
        normalize3(T);
        float B[3] = {N[1] * T[2] - T[1] * N[2], N[2] * T[0] - T[2] * N[0], N[0] * T[1] - T[0] * N[1]};
        normalize3(B);
        for (int c = 0; c < 3; ++c) B[c] = B[c] * v[9];
        float n2[3];
        for (int c = 0; c < 3; ++c) n2[c] = (T[c] * m[0] + B[c] * m[1]) + N[c] * m[2];
        normalize3(n2);
        memcpy(N, n2, sizeof(N));
    }
    const float en[3] = {N[0] * 0.5f + 0.5f, N[1] * 0.5f + 0.5f, N[2] * 0.5f + 0.5f};
    float metal = 0.1f, rough = 0.5f;
    if (has & 4u) {
        metal = tex12[8 + 2];
        rough = tex12[8 + 1];
    }
    const float nd = clamp01((v[12] - near_far[0]) / (near_far[1] - near_far[0]));
    const float dep = clamp01(orc_splat_exp(-20.0f * nd));
    float col[3] = {alb[0], alb[1], alb[2]};
    if (mode == 1) { col[0] = col[1] = col[2] = dep; }
    else if (mode == 2) { memcpy(col, en, sizeof(col)); }
    else if (mode == 3) {
        const float id = (float)prim_id;
        col[0] = orc_mesh_hash(id * 311.7f);
        col[1] = orc_mesh_hash(id * 269.5f + 1.3f);
        col[2] = orc_mesh_hash(id * 183.3f + 2.7f);
    } else if (mode == 4) { col[0] = 0.01f; col[1] = 0.005f; col[2] = 0.0f; }
    const float o[20] = {v[0], v[1], v[2], 1.0f, en[0], en[1], en[2], 1.0f, col[0], col[1], col[2], 1.0f,
                         dep, dep, dep, 1.0f, metal, rough, 0.0f, 1.0f};
    memcpy(out, o, sizeof(o));
}

/* meshRenderVS/PS.glsl for pixel (x, y) whose winner is fan triangle k of triangle tri of primitive p; 20 output words:
 * position, normal, depth as fp16 bits (4 each), albedo and metallic-roughness as bytes (4 each) */
static void shade(const pass* a, uint32_t tri, int k, uint32_t p, int x, int y, uint16_t* h16, uint8_t* b8) {
    const float* t36 = a->tris + (size_t)tri * 36;
    cv poly[MAX_POLY];
    mesh_poly(t36, &a->u, poly);
    ftri s;
    fan_setup(poly, k, a->W, a->H, &s);
    float vary[3][13], clip[4];
    for (int j = 0; j < 3; ++j) orc_mesh_vs_one(t36 + 12 * j, a->u.M, a->u.V, a->u.P, a->u.N, clip, vary[j]);
    double beta[3];
    float v[13];
    weights(&s, x, y, beta);
    for (int i = 0; i < 13; ++i) v[i] = interp(beta, (const float(*)[13])vary, i);
    const int qx = x & ~1, qy = y & ~1;
    weights(&s, qx, qy, beta);
    const float u00 = interp(beta, (const float(*)[13])vary, 10), v00 = interp(beta, (const float(*)[13])vary, 11);
    weights(&s, qx + 1, qy, beta);
    const float dudx = interp(beta, (const float(*)[13])vary, 10) - u00, dvdx = interp(beta, (const float(*)[13])vary, 11) - v00;
    weights(&s, qx, qy + 1, beta);
    const float dudy = interp(beta, (const float(*)[13])vary, 10) - u00, dvdy = interp(beta, (const float(*)[13])vary, 11) - v00;

    const float* fac = a->prim_factor + 4 * p;
    const int32_t* tex = a->prim_tex + 3 * p;
    float tx[12] = {0};
    uint32_t has = 0;
    for (int m = 0; m < 3; ++m)
        if (tex[m] >= 0) {
            sample(&a->texs[tex[m]], a->arena, v[10], v[11], dudx, dvdx, dudy, dvdy, tx + 4 * m);
            has |= 1u << m;
        }
    float o[20];
    orc_mesh_fs(v, tx, has, fac, a->near_far, a->mode, tri - a->prim_first[p], o);
    for (int c = 0; c < 4; ++c) { h16[c] = orc_f2h(o[c]); h16[4 + c] = orc_f2h(o[4 + c]); h16[8 + c] = orc_f2h(o[12 + c]); }
    for (int c = 0; c < 4; ++c) { b8[c] = u8(o[8 + c]); b8[4 + c] = u8(o[16 + c]); }
}

/* The G-buffer after drawing the triangles < n_drawn (a prefix of the source triangles) of every primitive, in primitive
 * table order.  Textures: per texture nlevels and per level the texel offset in `arena` (RGBA8 words) and its size.
 * Outputs (each W x H x 4, or NULL): position, normal, depth as fp16 bits; albedo, metallic_roughness as bytes. */
ORC_API int orc_mesh_render(const float* tris, uint64_t n_drawn, uint32_t nprims, const uint32_t* prim_first, const uint32_t* prim_count,
                            const float* prim_factor, const int32_t* prim_tex, const uint32_t* tex_nlevels, const uint32_t* tex_off,
                            const uint32_t* tex_w, const uint32_t* tex_h, uint32_t ntex, const uint32_t* arena, const float* V,
                            const float* P, const float* M, const float* near_far, uint32_t W, uint32_t H, uint32_t mode,
                            uint16_t* position, uint16_t* normal, uint8_t* albedo, uint16_t* depth, uint8_t* mr) {
    pass a;
    memset(&a, 0, sizeof(a));
    if (!orc_mesh_normal_matrix(M, a.u.N)) return 0;
    a.u.M = M; a.u.V = V; a.u.P = P;
    a.tris = tris; a.prim_first = prim_first; a.prim_count = prim_count; a.prim_factor = prim_factor; a.prim_tex = prim_tex;
    mtex* texs = (mtex*)calloc(ntex ? ntex : 1, sizeof(mtex));
    for (uint32_t t = 0; t < ntex; ++t) {
        texs[t].nlevels = tex_nlevels[t];
        for (int l = 0; l < 5; ++l) { texs[t].off[l] = tex_off[5 * t + l]; texs[t].w[l] = tex_w[5 * t + l]; texs[t].h[l] = tex_h[5 * t + l]; }
    }
    a.texs = texs; a.arena = arena;
    a.near_far[0] = near_far[0]; a.near_far[1] = near_far[1];
    a.W = W; a.H = H; a.mode = mode;
    const size_t np = (size_t)W * H;
    uint32_t* code = (uint32_t*)malloc(np * 4);
    uint64_t* win = (uint64_t*)malloc(np * 8);   /* primitive << 32 | triangle << 3 | fan triangle */
    for (size_t i = 0; i < np; ++i) code[i] = CLEAR_CODE;
    for (uint32_t p = 0; p < nprims; ++p)
        for (uint64_t t = prim_first[p]; t < (uint64_t)prim_first[p] + prim_count[p] && t < n_drawn; ++t) {
            cv poly[MAX_POLY];
            const int nv = mesh_poly(tris + t * 36, &a.u, poly);
            for (int k = 0; k + 2 < nv; ++k) {
                ftri s;
                fan_setup(poly, k, W, H, &s);
                for (int j = s.y0; j <= s.y1; ++j)
                    for (int i = s.x0; i <= s.x1; ++i) {
                        int64_t e[3];
                        uint32_t c;
                        if (!covers(&s, i, j, e)) continue;
                        const double z = ((double)e[0] * (double)s.z[0] + (double)e[1] * (double)s.z[1] + (double)e[2] * (double)s.z[2]) /
                                         (double)(e[0] + e[1] + e[2]);
                        const size_t px = (size_t)j * W + i;
                        if (orc_depth_code(z, &c) && c < code[px]) {
                            code[px] = c;
                            win[px] = (uint64_t)p << 32 | (uint64_t)t << 3 | (uint64_t)k;
                        }
                    }
            }
        }
    for (uint32_t y = 0; y < H; ++y)
        for (uint32_t x = 0; x < W; ++x) {
            const size_t px = (size_t)y * W + x;
            uint16_t h16[12] = {0};
            uint8_t b8[8] = {0};
            if (code[px] < CLEAR_CODE)
                shade(&a, (uint32_t)(win[px] >> 3) & 0x1fffffffu, (int)(win[px] & 7u), (uint32_t)(win[px] >> 32), (int)x, (int)y, h16, b8);
            if (position) memcpy(position + 4 * px, h16, 8);
            if (normal) memcpy(normal + 4 * px, h16 + 4, 8);
            if (depth) memcpy(depth + 4 * px, h16 + 8, 8);
            if (albedo) memcpy(albedo + 4 * px, b8, 4);
            if (mr) memcpy(mr + 4 * px, b8 + 4, 4);
        }
    free(code); free(win); free(texs);
    return 1;
}

/* (16 x 16 tile, fan triangle) pairs of each source triangle of a primitive as the pass bins them; returns the total */
ORC_API uint64_t orc_mesh_pairs(const float* tris, uint64_t ntri, const uint8_t* drawn, const float* V, const float* P, const float* M,
                                uint32_t W, uint32_t H, uint32_t* counts) {
    uni u;
    if (!orc_mesh_normal_matrix(M, u.N)) return 0;
    u.M = M; u.V = V; u.P = P;
    uint64_t total = 0;
    for (uint64_t t = 0; t < ntri; ++t) {
        uint32_t c = 0;
        cv v[MAX_POLY];
        const int n = drawn[t] ? mesh_poly(tris + t * 36, &u, v) : 0;
        for (int k = 0; k + 2 < n; ++k) {
            ftri s;
            fan_setup(v, k, W, H, &s);
            if (s.x1 < s.x0 || s.y1 < s.y0) continue;
            for (int ty = s.y0 / 16; ty <= s.y1 / 16; ++ty)
                for (int tx = s.x0 / 16; tx <= s.x1 / 16; ++tx) c += (uint32_t)tri_touches(&s, tx, ty);
        }
        if (counts) counts[t] = c;
        total += c;
    }
    return total;
}

/* the split composite: columns x < (int)(position * W) from `left` (the mesh side), the rest from `right`, then the
 * columns [max(0, split - 1), +2) clipped to the image set to 255; RGBA8 images of W x H */
ORC_API void orc_mesh_split(const uint8_t* left, const uint8_t* right, uint32_t W, uint32_t H, float position, uint8_t* out) {
    const uint32_t split = (uint32_t)(int)(position * (float)(int)W);
    const uint32_t d0 = split > 0 ? split - 1 : 0, d1 = d0 + 2 < W ? d0 + 2 : W;
    for (uint32_t y = 0; y < H; ++y)
        for (uint32_t x = 0; x < W; ++x) {
            const size_t px = ((size_t)y * W + x) * 4;
            if (x >= d0 && x < d1) memset(out + px, 255, 4);
            else memcpy(out + px, (x < split ? left : right) + px, 4);
        }
}
