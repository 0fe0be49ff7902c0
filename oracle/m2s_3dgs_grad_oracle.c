/* m2s_3dgs_grad_oracle.c — plain-C restatement of the standard 3DGS render's backward pass (m2s_3dgs_backward_enqueue;
 * beyond the reference: graphdeco's renderCUDA / preprocessCUDA backward for the project's GL camera and PACKED56 records,
 * DESIGN §2) (TEST INFRASTRUCTURE: the checker of m2s_3dgs_grad.cu).  Built with gcc -ffp-contract=off: every operation
 * is one IEEE fp32 rounding in DESIGN §2's order: the per-pixel terms, the tile tree (a shuffle-down tree within each warp
 * of 32 pixels, then the 8 warps in order), the gather over the record's tiles in tile-id order, the chain rule.  The
 * forward values come from the forward checker (orc_3dgs_preprocess) and a restatement of its per-pixel loop; the exp
 * is orc_splat_exp (the project's rn_exp). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

float orc_splat_exp(float x);
uint32_t orc_3dgs_preprocess(const float* records, uint32_t n, uint32_t layout, const float* V, const float* P, const float* M, uint32_t width,
                             uint32_t height, float near, float std_dev, float scale_modifier, const float* sh, uint32_t buffer_degree,
                             uint32_t sh_degree, float* splats, uint32_t* keys);

enum { LAYOUT_PACKED56 = 1, NPART = 9 };

static float ad(float a, float b) { return a + b; }
static float sb(float a, float b) { return a - b; }
static float ml(float a, float b) { return a * b; }
static float dv(float a, float b) { return a / b; }

static float row4(const float* m, int r, float x, float y, float z) { return ad(ad(ad(ml(m[r], x), ml(m[4 + r], y)), ml(m[8 + r], z)), m[12 + r]); }

static void view_model(const float* V, const float* M, float mv[16]) {   /* the host code's sh_camera: fp64, rounded once */
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r)
            mv[c * 4 + r] = (float)((((double)V[r] * M[c * 4] + (double)V[4 + r] * M[c * 4 + 1]) + (double)V[8 + r] * M[c * 4 + 2]) +
                                    (double)V[12 + r] * M[c * 4 + 3]);
}

static const uint32_t* g_keys;
static int by_key(const void* a, const void* b) {
    const uint32_t i = *(const uint32_t*)a, j = *(const uint32_t*)b;
    if (g_keys[i] != g_keys[j]) return g_keys[i] < g_keys[j] ? -1 : 1;
    return i < j ? -1 : (i > j);
}

static void rect_of(const float* s, uint32_t* x0, uint32_t* x1, uint32_t* y0, uint32_t* y1) {
    uint32_t rx, ry;
    memcpy(&rx, s + 9, 4); memcpy(&ry, s + 10, 4);
    *x0 = rx & 0xFFFFu; *x1 = rx >> 16; *y0 = ry & 0xFFFFu; *y1 = ry >> 16;
}

/* the chain rule of record f (14 floats) from its summed partials P (DESIGN §2, backward: per record) into out */
static void chain(const float* f, const float* MV, const float* Pm, uint32_t width, uint32_t height, float scale_modifier, const float P[NPART],
                  float out[14]) {
    const float kC0 = 0.28209479177387814f;
    const float sx = orc_splat_exp(f[7]), sy = orc_splat_exp(f[8]), sz = orc_splat_exp(f[9]);
    const float cr = ad(ml(f[10], kC0), 0.5f), cg = ad(ml(f[11], kC0), 0.5f), cb_ = ad(ml(f[12], kC0), 0.5f);
    const float op = dv(1.0f, ad(1.0f, orc_splat_exp(-f[13])));
    /* forward values (gs3d_project) */
    const float tx = row4(MV, 0, f[0], f[1], f[2]), ty = row4(MV, 1, f[0], f[1], f[2]), tz = row4(MV, 2, f[0], f[1], f[2]);
    const float d = -tz;
    const float c0 = row4(Pm, 0, tx, ty, tz), c1 = row4(Pm, 1, tx, ty, tz), c3 = row4(Pm, 3, tx, ty, tz);
    const float pw = dv(1.0f, ad(c3, 1e-7f));
    const float W = (float)width, H = (float)height;
    const float s[3] = {ml(ml(sx, 1.0f), scale_modifier), ml(ml(sy, 1.0f), scale_modifier), ml(ml(sz, 1.0f), scale_modifier)};
    const float qn = fmaxf(sqrtf(ad(ad(ad(ml(f[3], f[3]), ml(f[4], f[4])), ml(f[5], f[5])), ml(f[6], f[6]))), 1e-12f);
    const float qr = dv(f[3], qn), qi = dv(f[4], qn), qj = dv(f[5], qn), qk = dv(f[6], qn);
    const float R[3][3] = {{sb(1.0f, ml(2.0f, ad(ml(qj, qj), ml(qk, qk)))), ml(2.0f, sb(ml(qi, qj), ml(qr, qk))), ml(2.0f, ad(ml(qi, qk), ml(qr, qj)))},
                           {ml(2.0f, ad(ml(qi, qj), ml(qr, qk))), sb(1.0f, ml(2.0f, ad(ml(qi, qi), ml(qk, qk)))), ml(2.0f, sb(ml(qj, qk), ml(qr, qi)))},
                           {ml(2.0f, sb(ml(qi, qk), ml(qr, qj))), ml(2.0f, ad(ml(qj, qk), ml(qr, qi))), sb(1.0f, ml(2.0f, ad(ml(qi, qi), ml(qj, qj))))}};
    float Mk[3][3], S[3][3], T[2][3], A[2][3];
    for (int k = 0; k < 3; ++k)
        for (int j = 0; j < 3; ++j) Mk[k][j] = ml(s[k], R[j][k]);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) S[i][j] = ad(ad(ml(Mk[0][i], Mk[0][j]), ml(Mk[1][i], Mk[1][j])), ml(Mk[2][i], Mk[2][j]));
    const float fx = ml(ml(Pm[0], W), 0.5f), fy = ml(ml(Pm[5], H), 0.5f);
    const float limx = dv(1.3f, Pm[0]), limy = dv(1.3f, Pm[5]);
    const float txd = dv(tx, d), tyd = dv(ty, d);
    const int clamp_x = txd < -limx || txd > limx, clamp_y = tyd < -limy || tyd > limy;
    const float txc = ml(fminf(limx, fmaxf(-limx, txd)), d), tyc = ml(fminf(limy, fmaxf(-limy, tyd)), d);
    const float dd = ml(d, d);
    const float J00 = dv(fx, d), J02 = dv(ml(fx, txc), dd), J11 = dv(fy, d), J12 = dv(ml(fy, tyc), dd);
    for (int j = 0; j < 3; ++j) {
        T[0][j] = ad(ml(J00, MV[4 * j + 0]), ml(J02, MV[4 * j + 2]));
        T[1][j] = ad(ml(J11, MV[4 * j + 1]), ml(J12, MV[4 * j + 2]));
    }
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 3; ++j) A[i][j] = ad(ad(ml(T[i][0], S[0][j]), ml(T[i][1], S[1][j])), ml(T[i][2], S[2][j]));
    const float ca = ad(ad(ad(ml(A[0][0], T[0][0]), ml(A[0][1], T[0][1])), ml(A[0][2], T[0][2])), 0.3f);
    const float cb = ad(ad(ml(A[0][0], T[1][0]), ml(A[0][1], T[1][1])), ml(A[0][2], T[1][2]));
    const float cc = ad(ad(ad(ml(A[1][0], T[1][0]), ml(A[1][1], T[1][1])), ml(A[1][2], T[1][2])), 0.3f);
    const float det = sb(ml(ca, cc), ml(cb, cb));
    /* colour and opacity */
    out[10] = cr < 0.0f ? 0.0f : ml(P[6], kC0);
    out[11] = cg < 0.0f ? 0.0f : ml(P[7], kC0);
    out[12] = cb_ < 0.0f ? 0.0f : ml(P[8], kC0);
    out[13] = isfinite(f[13]) ? ml(P[5], ml(op, sb(1.0f, op))) : 0.0f;
    /* conic -> covariance */
    const float i2 = dv(1.0f, ml(det, det));
    const float dA = P[2], dB = P[3], dC = P[4];
    const float dca = ml(ad(ad(ml(dA, -ml(cc, cc)), ml(dB, ml(cb, cc))), ml(dC, -ml(cb, cb))), i2);
    const float dcb = ml(ad(ad(ml(dA, ml(2.0f, ml(cb, cc))), ml(dB, -ad(ml(ca, cc), ml(cb, cb)))), ml(dC, ml(2.0f, ml(cb, ca)))), i2);
    const float dcc = ml(ad(ad(ml(dA, -ml(cb, cb)), ml(dB, ml(cb, ca))), ml(dC, -ml(ca, ca))), i2);
    const float hb = ml(0.5f, dcb);
    const float Gc[2][2] = {{dca, hb}, {hb, dcc}};
    float dS[3][3], dT[2][3];
    for (int p = 0; p < 3; ++p)
        for (int q = 0; q < 3; ++q)
            dS[p][q] = ad(ad(ad(ml(ml(T[0][p], Gc[0][0]), T[0][q]), ml(ml(T[0][p], Gc[0][1]), T[1][q])), ml(ml(T[1][p], Gc[1][0]), T[0][q])),
                          ml(ml(T[1][p], Gc[1][1]), T[1][q]));
    for (int m = 0; m < 2; ++m)
        for (int j = 0; j < 3; ++j) dT[m][j] = ml(2.0f, ad(ml(Gc[m][0], A[0][j]), ml(Gc[m][1], A[1][j])));
    float dJ00 = 0.0f, dJ02 = 0.0f, dJ11 = 0.0f, dJ12 = 0.0f;
    for (int j = 0; j < 3; ++j) {
        dJ00 = ad(dJ00, ml(dT[0][j], MV[4 * j + 0]));
        dJ02 = ad(dJ02, ml(dT[0][j], MV[4 * j + 2]));
        dJ11 = ad(dJ11, ml(dT[1][j], MV[4 * j + 1]));
        dJ12 = ad(dJ12, ml(dT[1][j], MV[4 * j + 2]));
    }
    const float d3 = ml(dd, d);
    const float dd_J = sb(sb(sb(-ml(dJ00, dv(fx, dd)), ml(dJ11, dv(fy, dd))), ml(dJ02, dv(ml(2.0f, ml(fx, txc)), d3))), ml(dJ12, dv(ml(2.0f, ml(fy, tyc)), d3)));
    float dt[3];
    dt[0] = clamp_x ? 0.0f : ml(dJ02, dv(fx, dd));
    dt[1] = clamp_y ? 0.0f : ml(dJ12, dv(fy, dd));
    dt[2] = -dd_J;
    const float du = ml(ml(P[0], W), 0.5f), dvv = ml(ml(P[1], H), 0.5f);
    const float dc0 = ml(du, pw), dc1 = ml(dvv, pw);
    const float dc3 = -ml(ad(ml(du, c0), ml(dvv, c1)), ml(pw, pw));
    for (int k = 0; k < 3; ++k) dt[k] = ad(dt[k], ad(ad(ml(dc0, Pm[4 * k + 0]), ml(dc1, Pm[4 * k + 1])), ml(dc3, Pm[4 * k + 3])));
    for (int j = 0; j < 3; ++j) out[j] = ad(ad(ml(dt[0], MV[4 * j + 0]), ml(dt[1], MV[4 * j + 1])), ml(dt[2], MV[4 * j + 2]));
    float dR[3][3], ds[3];
    for (int k = 0; k < 3; ++k) {
        ds[k] = 0.0f;
        for (int j = 0; j < 3; ++j) {
            const float dM = ml(2.0f, ad(ad(ml(Mk[k][0], dS[0][j]), ml(Mk[k][1], dS[1][j])), ml(Mk[k][2], dS[2][j])));
            ds[k] = ad(ds[k], ml(dM, R[j][k]));
            dR[j][k] = ml(dM, s[k]);
        }
        out[7 + k] = ml(ds[k], s[k]);
    }
    const float gr = ml(2.0f, ad(ad(ml(qk, sb(dR[1][0], dR[0][1])), ml(qj, sb(dR[0][2], dR[2][0]))), ml(qi, sb(dR[2][1], dR[1][2]))));
    const float gi = sb(ml(2.0f, ad(ad(ml(qj, ad(dR[0][1], dR[1][0])), ml(qk, ad(dR[0][2], dR[2][0]))), ml(qr, sb(dR[2][1], dR[1][2])))),
                        ml(ml(4.0f, qi), ad(dR[1][1], dR[2][2])));
    const float gj = sb(ml(2.0f, ad(ad(ml(qi, ad(dR[0][1], dR[1][0])), ml(qr, sb(dR[0][2], dR[2][0]))), ml(qk, ad(dR[1][2], dR[2][1])))),
                        ml(ml(4.0f, qj), ad(dR[0][0], dR[2][2])));
    const float gk = sb(ml(2.0f, ad(ad(ml(qr, sb(dR[1][0], dR[0][1])), ml(qi, ad(dR[0][2], dR[2][0]))), ml(qj, ad(dR[1][2], dR[2][1])))),
                        ml(ml(4.0f, qk), ad(dR[0][0], dR[1][1])));
    const float dot = ad(ad(ad(ml(qr, gr), ml(qi, gi)), ml(qj, gj)), ml(qk, gk));
    out[3] = dv(sb(gr, ml(qr, dot)), qn);
    out[4] = dv(sb(gi, ml(qi, dot)), qn);
    out[5] = dv(sb(gj, ml(qj, dot)), qn);
    out[6] = dv(sb(gk, ml(qk, dot)), qn);
}

/* the backward pass of the forward pass m2s_3dgs_render_grad(_enqueue) makes of n PACKED56 records with pair budget
 * max_pairs (UINT64_MAX: every survivor): grad_rgba W x H x 4 floats of dL/d(image), grad n x 14 floats written whole.
 * *drawn the drawn prefix.  0, or 1 for singular arguments / no memory. */
ORC_API int orc_3dgs_backward(const float* records, uint32_t n, const float* V, const float* Pm, const float* M, uint32_t width, uint32_t height,
                              float near, float scale_modifier, const float background[3], uint64_t max_pairs, const float* grad_rgba,
                              float* grad, uint32_t* drawn) {
    const uint32_t gx = (width + 15) / 16, gy = (height + 15) / 16, ntiles = gx * gy;
    float* sp = (float*)malloc(((size_t)n + 1) * 12 * sizeof(float));
    uint32_t* keys = (uint32_t*)malloc(((size_t)n + 1) * sizeof(uint32_t));
    uint32_t* order = (uint32_t*)malloc(((size_t)n + 1) * sizeof(uint32_t));
    uint32_t* rank = (uint32_t*)malloc(((size_t)n + 1) * sizeof(uint32_t));
    uint32_t* toff = (uint32_t*)calloc((size_t)ntiles + 1, sizeof(uint32_t));
    uint32_t* tcount = (uint32_t*)calloc((size_t)ntiles + 1, sizeof(uint32_t));
    uint32_t* tlast = (uint32_t*)calloc((size_t)ntiles + 1, sizeof(uint32_t));
    uint32_t* contrib = (uint32_t*)calloc((size_t)width * height, sizeof(uint32_t));
    float* finalT = (float*)calloc((size_t)width * height, sizeof(float));
    uint32_t* lists = NULL;
    float* part = NULL;
    int rc = 1;
    float MV[16];
    if (!sp || !keys || !order || !rank || !toff || !tcount || !tlast || !contrib || !finalT) goto out;
    const uint32_t alive = orc_3dgs_preprocess(records, n, LAYOUT_PACKED56, V, Pm, M, width, height, near, 1.0f, scale_modifier, NULL, 0, 0, sp, keys);
    if (alive == UINT32_MAX) goto out;
    view_model(V, M, MV);
    for (uint32_t i = 0; i < n; ++i) order[i] = i;
    g_keys = keys;
    qsort(order, n, sizeof(uint32_t), by_key);
    for (uint32_t k = 0; k < n; ++k) rank[order[k]] = k;
    /* the drawn prefix and each tile's run in depth order */
    uint64_t total = 0, fit = 0;
    uint32_t nd = 0;
    for (uint32_t k = 0; k < alive; ++k) {
        uint32_t x0, x1, y0, y1;
        rect_of(sp + (size_t)order[k] * 12, &x0, &x1, &y0, &y1);
        total += (uint64_t)(x1 - x0) * (y1 - y0);
        if (total <= max_pairs) { nd = k + 1; fit = total; }
    }
    *drawn = nd;
    for (uint32_t k = 0; k < nd; ++k) {
        uint32_t x0, x1, y0, y1;
        rect_of(sp + (size_t)order[k] * 12, &x0, &x1, &y0, &y1);
        for (uint32_t ty = y0; ty < y1; ++ty)
            for (uint32_t tx = x0; tx < x1; ++tx) tcount[ty * gx + tx]++;
    }
    lists = (uint32_t*)malloc((size_t)(fit + 1) * sizeof(uint32_t));
    part = (float*)calloc((size_t)(fit + 1) * NPART, sizeof(float));
    if (!lists || !part) goto out;
    for (uint32_t t = 0; t < ntiles; ++t) toff[t + 1] = toff[t] + tcount[t];
    memset(tcount, 0, (size_t)ntiles * sizeof(uint32_t));
    for (uint32_t k = 0; k < nd; ++k) {
        uint32_t x0, x1, y0, y1;
        rect_of(sp + (size_t)order[k] * 12, &x0, &x1, &y0, &y1);
        for (uint32_t ty = y0; ty < y1; ++ty)
            for (uint32_t tx = x0; tx < x1; ++tx) {
                const uint32_t t = ty * gx + tx;
                lists[toff[t] + tcount[t]++] = order[k];
            }
    }
    /* the forward pass per pixel: final T and 1 + the run position of the last blended gaussian */
    for (uint32_t y = 0; y < height; ++y)
        for (uint32_t x = 0; x < width; ++x) {
            const uint32_t t = (y / 16) * gx + x / 16;
            const float px = (float)x, py = (float)y;
            float T = 1.0f;
            uint32_t last = 0;
            for (uint32_t k = toff[t]; k < toff[t + 1]; ++k) {
                const float* s = sp + (size_t)lists[k] * 12;
                const float dx = sb(s[0], px), dy = sb(s[1], py);
                const float power = sb(ml(-0.5f, ad(ml(ml(s[2], dx), dx), ml(ml(s[4], dy), dy))), ml(ml(s[3], dx), dy));
                if (power > 0.0f) continue;
                const float alpha = fminf(0.99f, ml(s[5], orc_splat_exp(power)));
                if (alpha < 1.0f / 255.0f) continue;
                const float tt = ml(T, sb(1.0f, alpha));
                if (tt < 0.0001f) break;
                T = tt;
                last = k - toff[t] + 1;
            }
            finalT[(size_t)y * width + x] = T;
            contrib[(size_t)y * width + x] = last;
        }
    /* the tile backward: per pixel back to front, the 9 partials of each run position summed over the tile's pixels */
    const float* bg = background;
    for (uint32_t t = 0; t < ntiles; ++t) {
        const uint32_t ox = (t % gx) * 16, oy = (t / gx) * 16;
        float pT[256], acc[256][3], la[256], lc[256][3], gp[256][4], bgd[256], Tf[256];
        uint32_t last[256], run = 0;
        int in[256];
        for (int p = 0; p < 256; ++p) {
            const uint32_t x = ox + (uint32_t)(p % 16), y = oy + (uint32_t)(p / 16);
            in[p] = x < width && y < height;
            const size_t pix = (size_t)y * width + x;
            last[p] = in[p] ? contrib[pix] : 0;
            Tf[p] = in[p] ? finalT[pix] : 0.0f;
            for (int c = 0; c < 4; ++c) gp[p][c] = in[p] ? grad_rgba[pix * 4 + c] : 0.0f;
            bgd[p] = sb(ad(ad(ml(bg[0], gp[p][0]), ml(bg[1], gp[p][1])), ml(bg[2], gp[p][2])), gp[p][3]);
            pT[p] = Tf[p]; la[p] = 0.0f;
            for (int c = 0; c < 3; ++c) acc[p][c] = lc[p][c] = 0.0f;
            if (last[p] > run) run = last[p];
        }
        tlast[t] = run;
        for (uint32_t pos1 = run; pos1 > 0; --pos1) {
            const uint32_t pos = pos1 - 1;
            const float* s = sp + (size_t)lists[toff[t] + pos] * 12;
            float pp[256][NPART];
            for (int p = 0; p < 256; ++p) {
                for (int k = 0; k < NPART; ++k) pp[p][k] = 0.0f;
                if (!(pos < last[p])) continue;
                const float px = (float)(ox + (uint32_t)(p % 16)), py = (float)(oy + (uint32_t)(p / 16));
                const float dx = sb(s[0], px), dy = sb(s[1], py);
                const float power = sb(ml(-0.5f, ad(ml(ml(s[2], dx), dx), ml(ml(s[4], dy), dy))), ml(ml(s[3], dx), dy));
                if (power > 0.0f) continue;
                const float G = orc_splat_exp(power);
                const float alpha = fminf(0.99f, ml(s[5], G));
                if (alpha < 1.0f / 255.0f) continue;
                const float om = sb(1.0f, alpha);
                pT[p] = dv(pT[p], om);
                const float w = ml(alpha, pT[p]);
                float dL_dalpha = 0.0f;
                for (int c = 0; c < 3; ++c) {
                    const float col = s[6 + c];
                    acc[p][c] = ad(ml(la[p], lc[p][c]), ml(sb(1.0f, la[p]), acc[p][c]));
                    lc[p][c] = col;
                    dL_dalpha = ad(dL_dalpha, ml(sb(col, acc[p][c]), gp[p][c]));
                    pp[p][6 + c] = ml(w, gp[p][c]);
                }
                dL_dalpha = ml(dL_dalpha, pT[p]);
                la[p] = alpha;
                dL_dalpha = ad(dL_dalpha, ml(dv(-Tf[p], om), bgd[p]));
                const float dL_dG = ml(s[5], dL_dalpha);
                const float gdx = ml(G, dx), gdy = ml(G, dy);
                pp[p][0] = ml(dL_dG, sb(ml(-gdx, s[2]), ml(gdy, s[3])));
                pp[p][1] = ml(dL_dG, sb(ml(-gdy, s[4]), ml(gdx, s[3])));
                pp[p][2] = ml(ml(ml(-0.5f, gdx), dx), dL_dG);
                pp[p][3] = ml(ml(-gdx, dy), dL_dG);
                pp[p][4] = ml(ml(ml(-0.5f, gdy), dy), dL_dG);
                pp[p][5] = ml(G, dL_dalpha);
            }
            for (int k = 0; k < NPART; ++k) {
                float wsum[8];
                for (int w = 0; w < 8; ++w) {
                    float v[32];
                    for (int l = 0; l < 32; ++l) v[l] = pp[w * 32 + l][k];
                    for (int off = 16; off > 0; off >>= 1)
                        for (int l = 0; l < off; ++l) v[l] = ad(v[l], v[l + off]);
                    wsum[w] = v[0];
                }
                float sum = wsum[0];
                for (int w = 1; w < 8; ++w) sum = ad(sum, wsum[w]);
                part[(size_t)(toff[t] + pos) * NPART + k] = sum;
            }
        }
    }
    /* the gather in tile-id order and the chain rule */
    for (uint32_t i = 0; i < n; ++i) {
        float* o = grad + (size_t)i * 14;
        memset(o, 0, 14 * sizeof(float));
        if (keys[i] == 0xFFFFFFFFu || rank[i] >= nd || records[(size_t)i * 14 + 13] != records[(size_t)i * 14 + 13]) continue;   /* NaN logit: zero row */
        uint32_t x0, x1, y0, y1;
        rect_of(sp + (size_t)i * 12, &x0, &x1, &y0, &y1);
        float P[NPART] = {0};
        for (uint32_t ty = y0; ty < y1; ++ty)
            for (uint32_t tx = x0; tx < x1; ++tx) {
                const uint32_t t = ty * gx + tx;
                uint32_t k = toff[t];
                while (lists[k] != i) ++k;
                if (k - toff[t] >= tlast[t]) continue;
                for (int q = 0; q < NPART; ++q) P[q] = ad(P[q], part[(size_t)k * NPART + q]);
            }
        chain(records + (size_t)i * 14, MV, Pm, width, height, scale_modifier, P, o);
    }
    rc = 0;
out:
    free(sp); free(keys); free(order); free(rank); free(toff); free(tcount); free(tlast); free(contrib); free(finalT); free(lists); free(part);
    return rc;
}
