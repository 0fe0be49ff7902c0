/* m2s_depth_oracle.c — CPU restatement of the viewer's mesh depth pre-pass and of the prepass's mesh depth test (row f-9).
 *
 * TEST INFRASTRUCTURE ONLY, like m2s_oracle.c: nothing under mesh2splat_b200/ includes, links or calls it.
 *
 * Restated (paths relative to the reference tree):
 *   depth pre-pass    src/renderer/renderPasses/DepthPrepass.cpp:8-49, depthPrepassVS.glsl, depthPrepassPS.glsl
 *   depth test        src/shaders/rendering/gaussianSplattingPrepassCS.glsl:78-91 (u_depthTestMesh 1)
 * The fixed-function parts are the contract of DESIGN §2 "The mesh depth pre-pass": PVM = (P V) M with GLM's mat4 * mat4,
 * clipping (Sutherland-Hodgman, z >= -w, z <= w, then x and y against +-2 w, intersections from the inside vertex), fan
 * triangulation, the splat draw's rasteriser, depth interpolated in fp64 from the exact edge values, D24 codes (LESS,
 * clear 2^24 - 1, NaN writes nothing) and NEAREST + CLAMP_TO_EDGE sampling.
 *
 * The map is drawn triangle by triangle, fan triangle by fan triangle, pixel by pixel: GL's order.
 *
 * Arithmetic: fp32 (fp64 for the depth interpolation), one rounding per operation (built with -ffp-contract=off).
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))
#define MAX_POLY 9
#define GUARD 2.0f

/* GLM mat4 * mat4, column-major: r[c][row] = ((a0 b[c][0] + a1 b[c][1]) + a2 b[c][2]) + a3 b[c][3] */
static void m4mul(const float* a, const float* b, float* r) {
    for (int c = 0; c < 4; ++c)
        for (int row = 0; row < 4; ++row)
            r[c * 4 + row] = ((a[row] * b[c * 4] + a[4 + row] * b[c * 4 + 1]) + a[8 + row] * b[c * 4 + 2]) + a[12 + row] * b[c * 4 + 3];
}

/* u_viewToClip * u_worldToView * u_modelToWorld, left to right */
ORC_API void orc_depth_pvm(const float* V, const float* P, const float* M, float* out) {
    float pv[16];
    m4mul(P, V, pv);
    m4mul(pv, M, out);
}

/* GLM mat4 * vec4: (m0 x + m1 y) + (m2 z + m3 w) */
static float m4row(const float* m, int row, float x, float y, float z, float w) {
    return (m[row] * x + m[4 + row] * y) + (m[8 + row] * z + m[12 + row] * w);
}

/* D24 of an fp64 depth: round-half-even(clamp(z, 0, 1) (2^24 - 1)), the product rounded once in fp64; 0 for NaN */
ORC_API int orc_depth_code(double z, uint32_t* code) {
    if (z != z) return 0;
    const double zc = z < 0.0 ? 0.0 : (z > 1.0 ? 1.0 : z);
    *code = (uint32_t)llrint(zc * 16777215.0);
    return 1;
}

/* depthPrepassVS.glsl's gl_Position for n positions (n x 3) under pvm: PVM (p, 1); out n x 4 */
ORC_API void orc_depth_vs(const float* pos, uint64_t n, const float* pvm, float* out) {
    for (uint64_t k = 0; k < n; ++k)
        for (int row = 0; row < 4; ++row) out[4 * k + row] = m4row(pvm, row, pos[3 * k], pos[3 * k + 1], pos[3 * k + 2], 1.0f);
}

/* ---- transform and clip ---------------------------------------------------------------------------------------------- */
typedef struct { float x, y, z, w; } v4;

static float plane(v4 v, int p) {
    const float gw = GUARD * v.w;
    switch (p) {
        case 0: return v.z + v.w;
        case 1: return v.w - v.z;
        case 2: return v.x + gw;
        case 3: return gw - v.x;
        case 4: return v.y + gw;
        default: return gw - v.y;
    }
}

static v4 cut(v4 a, v4 b, float da, float db) {   /* a inside, b outside */
    const float t = da / (da - db);
    v4 r = {a.x + t * (b.x - a.x), a.y + t * (b.y - a.y), a.z + t * (b.z - a.z), a.w + t * (b.w - a.w)};
    return r;
}

/* clip-space polygon of one triangle (36 floats: 3 x {pos3 nrm3 tan4 uv2}); returns its vertex count, 0 if nothing is left
 * or a clip coordinate is not finite.  out: MAX_POLY x 4 floats. */
ORC_API int orc_depth_poly(const float* tri36, const float* pvm, float* out) {
    v4 v[MAX_POLY];
    for (int k = 0; k < 3; ++k) {
        const float* p = tri36 + 12 * k;
        v[k].x = m4row(pvm, 0, p[0], p[1], p[2], 1.0f);
        v[k].y = m4row(pvm, 1, p[0], p[1], p[2], 1.0f);
        v[k].z = m4row(pvm, 2, p[0], p[1], p[2], 1.0f);
        v[k].w = m4row(pvm, 3, p[0], p[1], p[2], 1.0f);
        if (!isfinite(v[k].x) || !isfinite(v[k].y) || !isfinite(v[k].z) || !isfinite(v[k].w)) return 0;
    }
    int n = 3;
    for (int p = 0; p < 6 && n > 0; ++p) {
        v4 o[MAX_POLY];
        int m = 0;
        for (int i = 0; i < n; ++i) {
            const int prev = i == 0 ? n - 1 : i - 1;
            const float dc = plane(v[i], p), dp = plane(v[prev], p);
            if (dc >= 0.0f) {
                if (dp < 0.0f && m < MAX_POLY) o[m++] = cut(v[i], v[prev], dc, dp);
                if (m < MAX_POLY) o[m++] = v[i];
            } else if (dp >= 0.0f && m < MAX_POLY) {
                o[m++] = cut(v[prev], v[i], dp, dc);
            }
        }
        memcpy(v, o, sizeof(v4) * (size_t)m);
        n = m;
    }
    memcpy(out, v, sizeof(v4) * (size_t)n);
    return n;
}

/* ---- the splat draw's rasteriser (m2s_splat_oracle.c) in the W x H viewport ------------------------------------------ */
typedef struct { int64_t A[3], B[3], C[3]; int incl[3]; int x0, x1, y0, y1; float z[3]; } dtri;

static void snap(float nx, float ny, float W, float H, int* ok, int32_t* X, int32_t* Y) {
    const float hw = W * 0.5f, hh = H * 0.5f;
    const float xw = nx * hw + hw, yw = ny * hh + hh;
    *ok = isfinite(xw) && isfinite(yw) && fabsf(xw) <= 8192.0f && fabsf(yw) <= 8192.0f;
    *X = *ok ? (int32_t)lrintf(xw * 256.0f) : 0;
    *Y = *ok ? (int32_t)lrintf(yw * 256.0f) : 0;
}

/* fan triangle (v0, vk+1, vk+2) of a clipped polygon: perspective divide, window depth, snap, edge functions */
static void fan_setup(const v4* v, int k, uint32_t W, uint32_t H, dtri* s) {
    memset(s, 0, sizeof(*s));
    s->x1 = -1; s->y1 = -1;
    int32_t X[3], Y[3];
    int ok = 1;
    for (int c = 0; c < 3; ++c) {
        const v4 p = v[c == 0 ? 0 : k + c];
        int okc;
        snap(p.x / p.w, p.y / p.w, (float)W, (float)H, &okc, &X[c], &Y[c]);
        ok = ok && okc;
        s->z[c] = (p.z / p.w) * 0.5f + 0.5f;
    }
    if (!ok) return;
    const int64_t area2 = (int64_t)(X[1] - X[0]) * (Y[2] - Y[0]) - (int64_t)(X[2] - X[0]) * (Y[1] - Y[0]);
    if (area2 == 0) return;
    const int64_t sg = area2 < 0 ? -1 : 1;
    for (int e = 0; e < 3; ++e) {
        const int a = (e + 1) % 3, b = (e + 2) % 3;
        const int64_t dx = X[b] - X[a], dy = Y[b] - Y[a];
        s->A[e] = sg * (-dy * 256);
        s->B[e] = sg * (dx * 256);
        s->C[e] = sg * (dx * (128 - (int64_t)Y[a]) - dy * (128 - (int64_t)X[a]));
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

static int tri_touches(const dtri* s, int tx, int ty) {
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

/* the depth at pixel (i, j) if the fan triangle covers its centre: ((E0 z0 + E1 z1) + E2 z2) / (E0 + E1 + E2) in fp64 */
static int tri_depth(const dtri* s, int i, int j, double* z) {
    int64_t e[3];
    for (int k = 0; k < 3; ++k) {
        e[k] = s->A[k] * i + s->B[k] * j + s->C[k];
        if (e[k] < 0 || (e[k] == 0 && !s->incl[k])) return 0;
    }
    *z = ((double)e[0] * (double)s->z[0] + (double)e[1] * (double)s->z[1] + (double)e[2] * (double)s->z[2]) / (double)(e[0] + e[1] + e[2]);
    return 1;
}

/* (16 x 16 tile, fan triangle) pairs per source triangle as the pass bins them; returns the total.  opaque[t] != 0 draws
 * triangle t. */
ORC_API uint64_t orc_depth_pairs(const float* tris, uint64_t ntri, const uint8_t* opaque, const float* pvm, uint32_t W, uint32_t H,
                                 uint32_t* counts) {
    uint64_t total = 0;
    for (uint64_t t = 0; t < ntri; ++t) {
        uint32_t c = 0;
        v4 v[MAX_POLY];
        const int n = opaque[t] ? orc_depth_poly(tris + t * 36, pvm, (float*)v) : 0;
        for (int k = 0; k + 2 < n; ++k) {
            dtri s;
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

/* glClear(GL_DEPTH_BUFFER_BIT) to 1, then the opaque triangles among 0..n-1 in order, depth test LESS on D24 codes.
 * out: W x H floats, (float)code / 16777215, row 0 = window y 0. */
ORC_API void orc_mesh_depth(const float* tris, uint64_t n, const uint8_t* opaque, const float* pvm, uint32_t W, uint32_t H, float* out) {
    const size_t np = (size_t)W * H;
    uint32_t* codes = (uint32_t*)out;   /* codes in place, converted at the end */
    for (size_t k = 0; k < np; ++k) codes[k] = 0xFFFFFFu;
    for (uint64_t t = 0; t < n; ++t) {
        if (!opaque[t]) continue;
        v4 v[MAX_POLY];
        const int nv = orc_depth_poly(tris + t * 36, pvm, (float*)v);
        for (int k = 0; k + 2 < nv; ++k) {
            dtri s;
            fan_setup(v, k, W, H, &s);
            for (int j = s.y0; j <= s.y1; ++j)
                for (int i = s.x0; i <= s.x1; ++i) {
                    double z;
                    uint32_t code;
                    if (tri_depth(&s, i, j, &z) && orc_depth_code(z, &code) && code < codes[(size_t)j * W + i]) codes[(size_t)j * W + i] = code;
                }
        }
    }
    for (size_t k = 0; k < np; ++k) out[k] = (float)codes[k] / 16777215.0f;
}

/* ---- the prepass's depth test ----------------------------------------------------------------------------------------- */
/* per REF96 gaussian (24 floats): 1 if the depth test keeps it (u_format 0, color.a > .95f, myDepth > depth + eps drops
 * it), evaluated in GLSL / GLM order without contraction.  The frustum cull is not part of the mask: the prepass applies
 * it before the test, and a gaussian it drops is dropped either way.  fmt != 0 keeps everything. */
ORC_API void orc_depth_test_mask(const float* g24, uint64_t n, const float* V, const float* P, const float* M, const float* map,
                                 uint32_t W, uint32_t H, uint32_t fmt, uint8_t* keep) {
    for (uint64_t k = 0; k < n; ++k) {
        const float* g = g24 + k * 24;
        keep[k] = 1;
        if (fmt != 0 || !(g[7] > 0.95f)) continue;
        const float w0 = m4row(M, 0, g[0], g[1], g[2], 1.0f), w1 = m4row(M, 1, g[0], g[1], g[2], 1.0f), w2 = m4row(M, 2, g[0], g[1], g[2], 1.0f);
        const float v0 = m4row(V, 0, w0, w1, w2, 1.0f), v1 = m4row(V, 1, w0, w1, w2, 1.0f), v2 = m4row(V, 2, w0, w1, w2, 1.0f),
                    v3 = m4row(V, 3, w0, w1, w2, 1.0f);
        const float c0 = m4row(P, 0, v0, v1, v2, v3), c1 = m4row(P, 1, v0, v1, v2, v3), c2 = m4row(P, 2, v0, v1, v2, v3),
                    c3 = m4row(P, 3, v0, v1, v2, v3);
        const float u = (c0 / c3) * 0.5f + 0.5f, v = (c1 / c3) * 0.5f + 0.5f;
        const uint32_t i = (uint32_t)fminf(fmaxf(floorf(u * (float)W), 0.0f), (float)(W - 1));
        const uint32_t j = (uint32_t)fminf(fmaxf(floorf(v * (float)H), 0.0f), (float)(H - 1));
        const float depth = map[(size_t)j * W + i];
        const float my = (c2 / c3) * 0.5f + 0.5f;
        if (my > depth + 0.00002f) keep[k] = 0;
    }
}
