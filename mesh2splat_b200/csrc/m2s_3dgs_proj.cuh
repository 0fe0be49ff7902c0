// m2s_3dgs_proj.cuh — the per-record projection of the standard 3DGS render (DESIGN §2, the 3DGS render: per record), shared
// by its preprocess kernel (m2s_3dgs.cu) and the backward pass's chain rule (m2s_3dgs_grad.cu), which needs the same
// intermediate values bit for bit.  Every operation is round-to-nearest fp32 without contraction.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_3dgs.cuh"
#include "m2s_gauss.cuh"

namespace m2s {

// row r of the column-major 4 x 4 m applied to (x, y, z, 1): ((m_r0 x + m_r1 y) + m_r2 z) + m_r3
__device__ __forceinline__ float gs3d_row(const float* m, int r, float x, float y, float z) {
    return ad(ad(ad(ml(m[r], x), ml(m[4 + r], y)), ml(m[8 + r], z)), m[12 + r]);
}

// the view-space mean, the pixel mean, and the covariance chain of one record up to the dilated 2-D covariance
struct Gs3dProj {
    float tx, ty, tz, d;              // view-space mean (GL), view depth d = -tz
    float c0, c1, pw;                 // clip x, y and 1 / (w + 1e-7)
    float u, v;                       // mean in pixels
    float s[3];                       // scales (times mult and scale_modifier)
    float qn, qr, qi, qj, qk;         // |q| (at least 1e-12), the normalised rotation (w, x, y, z)
    float R[3][3], Mk[3][3], S[3][3]; // rotation, Mk[k][j] = s_k R[j][k], Sigma = Mk^T Mk
    float fx, fy, txc, tyc, dd;       // focal lengths, the clamped view x and y, d^2
    bool clamp_x, clamp_y;            // t.x / d or t.y / d outside +-1.3 tan(fov / 2)
    float J00, J02, J11, J12;         // the Jacobian of the pixel mean in view space
    float T[2][3], A[2][3];           // T = J W, A = T Sigma
    float ca, cb, cc;                 // dilated 2-D covariance
};

// false if the record is culled at the near plane (the rest is not written then)
__device__ __forceinline__ bool gs3d_project(const Gs3dArgs& a, const GaussFields& g, Gs3dProj& o) {
    // ---- view and cull ----
    o.tx = gs3d_row(a.MV, 0, g.px, g.py, g.pz); o.ty = gs3d_row(a.MV, 1, g.px, g.py, g.pz); o.tz = gs3d_row(a.MV, 2, g.px, g.py, g.pz);
    o.d = -o.tz;
    const float d = o.d;
    if (!(d > a.near)) return false;
    // ---- mean in pixels (ndc2Pix) ----
    o.c0 = gs3d_row(a.P, 0, o.tx, o.ty, o.tz); o.c1 = gs3d_row(a.P, 1, o.tx, o.ty, o.tz);
    const float c3 = gs3d_row(a.P, 3, o.tx, o.ty, o.tz);
    o.pw = dv(1.0f, ad(c3, 1e-7f));
    const float W = (float)a.width, H = (float)a.height;
    o.u = ml(sb(ml(ad(ml(o.c0, o.pw), 1.0f), W), 1.0f), 0.5f); o.v = ml(sb(ml(ad(ml(o.c1, o.pw), 1.0f), H), 1.0f), 0.5f);
    // ---- 3-D covariance (computeCov3D): scale, normalised rotation, Sigma = (S R^T)^T (S R^T) ----
    o.s[0] = ml(ml(g.sx, a.mult), a.scale_modifier); o.s[1] = ml(ml(g.sy, a.mult), a.scale_modifier); o.s[2] = ml(ml(g.sz, a.mult), a.scale_modifier);
    o.qn = fmaxf(__fsqrt_rn(ad(ad(ad(ml(g.qx, g.qx), ml(g.qy, g.qy)), ml(g.qz, g.qz)), ml(g.qw, g.qw))), 1e-12f);
    const float qr = dv(g.qx, o.qn), qi = dv(g.qy, o.qn), qj = dv(g.qz, o.qn), qk = dv(g.qw, o.qn);   // (w, x, y, z)
    o.qr = qr; o.qi = qi; o.qj = qj; o.qk = qk;
    o.R[0][0] = sb(1.0f, ml(2.0f, ad(ml(qj, qj), ml(qk, qk)))); o.R[0][1] = ml(2.0f, sb(ml(qi, qj), ml(qr, qk))); o.R[0][2] = ml(2.0f, ad(ml(qi, qk), ml(qr, qj)));
    o.R[1][0] = ml(2.0f, ad(ml(qi, qj), ml(qr, qk))); o.R[1][1] = sb(1.0f, ml(2.0f, ad(ml(qi, qi), ml(qk, qk)))); o.R[1][2] = ml(2.0f, sb(ml(qj, qk), ml(qr, qi)));
    o.R[2][0] = ml(2.0f, sb(ml(qi, qk), ml(qr, qj))); o.R[2][1] = ml(2.0f, ad(ml(qj, qk), ml(qr, qi))); o.R[2][2] = sb(1.0f, ml(2.0f, ad(ml(qi, qi), ml(qj, qj))));
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j) o.Mk[k][j] = ml(o.s[k], o.R[j][k]);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) o.S[i][j] = ad(ad(ml(o.Mk[0][i], o.Mk[0][j]), ml(o.Mk[1][i], o.Mk[1][j])), ml(o.Mk[2][i], o.Mk[2][j]));
    // ---- 2-D covariance (computeCov2D in GL axes): cov = J W Sigma W^T J^T + 0.3 I ----
    o.fx = ml(ml(a.P[0], W), 0.5f); o.fy = ml(ml(a.P[5], H), 0.5f);
    const float limx = dv(1.3f, a.P[0]), limy = dv(1.3f, a.P[5]);
    const float txd = dv(o.tx, d), tyd = dv(o.ty, d);
    o.clamp_x = txd < -limx || txd > limx; o.clamp_y = tyd < -limy || tyd > limy;
    o.txc = ml(fminf(limx, fmaxf(-limx, txd)), d); o.tyc = ml(fminf(limy, fmaxf(-limy, tyd)), d);
    o.dd = ml(d, d);
    o.J00 = dv(o.fx, d); o.J02 = dv(ml(o.fx, o.txc), o.dd); o.J11 = dv(o.fy, d); o.J12 = dv(ml(o.fy, o.tyc), o.dd);
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        o.T[0][j] = ad(ml(o.J00, a.MV[4 * j + 0]), ml(o.J02, a.MV[4 * j + 2]));
        o.T[1][j] = ad(ml(o.J11, a.MV[4 * j + 1]), ml(o.J12, a.MV[4 * j + 2]));
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) o.A[i][j] = ad(ad(ml(o.T[i][0], o.S[0][j]), ml(o.T[i][1], o.S[1][j])), ml(o.T[i][2], o.S[2][j]));
    auto cov = [&](int i, int j) { return ad(ad(ml(o.A[i][0], o.T[j][0]), ml(o.A[i][1], o.T[j][1])), ml(o.A[i][2], o.T[j][2])); };
    o.ca = ad(cov(0, 0), 0.3f); o.cb = cov(0, 1); o.cc = ad(cov(1, 1), 0.3f);
    return true;
}

}  // namespace m2s
