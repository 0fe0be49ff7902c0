// m2s_3dgs_grad.cu — the backward pass of the standard 3DGS render (beyond the reference): graphdeco's renderCUDA and
// preprocessCUDA backward (Kerbl et al. 2023, diff-gaussian-rasterization) for PACKED56 records, as DESIGN §2 fixes it.
//
// Shape, on one stream, after a forward pass that kept its state (gs3d_draw_save_launch):
//   gs3d_tile_backward_kernel  one CTA per tile, one thread per pixel: the tile's run back to front from the CTA's last
//                              contributor; per pixel and gaussian the 9 partials; summed over the tile's 256 pixels by a
//                              warp-shuffle tree, then the warps in order; one 9-float partial per pair slot
//   gs3d_gather_kernel         one thread per record: its pairs' partials over its tile rectangle in tile-id order (its
//                              slot in each run by binary search on depth rank), then the chain rule to the 14 fields
// No floating-point atomic decides a bit, and every operation is round-to-nearest fp32 without contraction, so the
// result equals the checker's (oracle/m2s_3dgs_grad_oracle.c) bit for bit and two calls give identical bits.
#include "m2s_3dgs.cuh"
#include "m2s_3dgs_proj.cuh"
#include "m2s_bin.cuh"

namespace m2s {

constexpr int kGs3dGatherThreads = 256;
constexpr int kGs3dRedRows = 32;   // gaussians whose warp sums wait in shared memory before the cross-warp sum

// ---- tile backward ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTileThreads) gs3d_tile_backward_kernel(const __grid_constant__ Gs3dGradArgs g) {
    __shared__ float s_v[kGs3dVaryings][kTileThreads];
    __shared__ float s_red[kGs3dRedRows][kTileThreads / 32][kGs3dPartials];
    __shared__ uint32_t s_last;
    const Gs3dSaveArgs& a = g.a;
    const TileFrame f = tile_frame(a.scratch, bin_layout(a.count, tile_count(a.width, a.height)), tiles_x(a.width), blockIdx.x);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool inside = f.x < (int)a.width && f.y < (int)a.height;
    const size_t pix = (size_t)f.y * a.width + f.x;
    const float px = (float)f.x, py = (float)f.y;
    const uint32_t last = inside ? a.n_contrib[pix] : 0u;
    const float T_final = inside ? a.final_T[pix] : 0.0f;
    const float4 gp = inside ? g.grad_rgba[pix] : make_float4(0.f, 0.f, 0.f, 0.f);
    // dL/dT_final: the colour's T bg and the alpha output 1 - T
    const float bg_dot = sb(ad(ad(ml(a.bg[0], gp.x), ml(a.bg[1], gp.y)), ml(a.bg[2], gp.z)), gp.w);
    if (tid == 0) s_last = 0;
    __syncthreads();
    if (last) atomicMax(&s_last, last);
    __syncthreads();
    const uint32_t run = s_last;
    if (tid == 0) g.tile_last[blockIdx.x] = run;
    float T = T_final, acc[3] = {0.0f, 0.0f, 0.0f}, last_alpha = 0.0f, last_col[3] = {0.0f, 0.0f, 0.0f};
    for (uint32_t top = run; top > 0;) {   // positions [top - nb, top), staged back to front
        const uint32_t nb = min(top, (uint32_t)kTileThreads);
        __syncthreads();
        if ((uint32_t)tid < nb) {
            const Gs3dSplat sp = a.splats[g.vals[f.r0 + top - 1 - tid]];
            s_v[0][tid] = sp.a.x; s_v[1][tid] = sp.a.y; s_v[2][tid] = sp.a.z; s_v[3][tid] = sp.a.w;
            s_v[4][tid] = sp.b.x; s_v[5][tid] = sp.b.y; s_v[6][tid] = sp.b.z; s_v[7][tid] = sp.b.w; s_v[8][tid] = sp.c.x;
        }
        __syncthreads();
        for (uint32_t j0 = 0; j0 < nb; j0 += kGs3dRedRows) {
            const uint32_t jn = min(nb - j0, (uint32_t)kGs3dRedRows);
            for (uint32_t jj = 0; jj < jn; ++jj) {
                const uint32_t j = j0 + jj, pos = top - 1 - j;   // pos: the run position, 0-based
                float p[kGs3dPartials] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
                bool use = pos < last;
                float G = 0.0f, alpha = 0.0f, dx = 0.0f, dy = 0.0f;
                if (use) {
                    dx = sb(s_v[0][j], px); dy = sb(s_v[1][j], py);
                    const float power = sb(ml(-0.5f, ad(ml(ml(s_v[2][j], dx), dx), ml(ml(s_v[4][j], dy), dy))), ml(ml(s_v[3][j], dx), dy));
                    use = !(power > 0.0f);
                    if (use) {
                        G = rn_exp(power);
                        alpha = fminf(0.99f, ml(s_v[5][j], G));
                        use = !(alpha < 1.0f / 255.0f);
                    }
                }
                if (use) {
                    const float om = sb(1.0f, alpha);
                    T = dv(T, om);
                    const float w = ml(alpha, T);
                    const float gc[3] = {gp.x, gp.y, gp.z};
                    float dL_dalpha = 0.0f;
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const float col = s_v[6 + c][j];
                        acc[c] = ad(ml(last_alpha, last_col[c]), ml(sb(1.0f, last_alpha), acc[c]));
                        last_col[c] = col;
                        dL_dalpha = ad(dL_dalpha, ml(sb(col, acc[c]), gc[c]));
                        p[6 + c] = ml(w, gc[c]);
                    }
                    dL_dalpha = ml(dL_dalpha, T);
                    last_alpha = alpha;
                    dL_dalpha = ad(dL_dalpha, ml(dv(-T_final, om), bg_dot));
                    const float dL_dG = ml(s_v[5][j], dL_dalpha);
                    const float gdx = ml(G, dx), gdy = ml(G, dy);
                    const float cA = s_v[2][j], cB = s_v[3][j], cC = s_v[4][j];
                    p[0] = ml(dL_dG, sb(ml(-gdx, cA), ml(gdy, cB)));   // dL/du
                    p[1] = ml(dL_dG, sb(ml(-gdy, cC), ml(gdx, cB)));   // dL/dv
                    p[2] = ml(ml(ml(-0.5f, gdx), dx), dL_dG);          // dL/dconic.x
                    p[3] = ml(ml(-gdx, dy), dL_dG);                    // dL/dconic.y (the off-diagonal, once)
                    p[4] = ml(ml(ml(-0.5f, gdy), dy), dL_dG);          // dL/dconic.z
                    p[5] = ml(G, dL_dalpha);                           // dL/dopacity
                }
                // the tile's sum of the 9 partials: a shuffle tree per warp (lane 0), then the warps in order
                if (__any_sync(0xffffffffu, use)) {
#pragma unroll
                    for (int k = 0; k < kGs3dPartials; ++k)
#pragma unroll
                        for (int off = 16; off > 0; off >>= 1) p[k] = ad(p[k], __shfl_down_sync(0xffffffffu, p[k], off));
                }
                if (lane == 0)
#pragma unroll
                    for (int k = 0; k < kGs3dPartials; ++k) s_red[jj][warp][k] = p[k];
            }
            __syncthreads();
            for (uint32_t o = tid; o < jn * kGs3dPartials; o += kTileThreads) {
                const uint32_t jj = o / kGs3dPartials, k = o % kGs3dPartials;
                float s = s_red[jj][0][k];
#pragma unroll
                for (int w = 1; w < kTileThreads / 32; ++w) s = ad(s, s_red[jj][w][k]);
                g.part[(size_t)(f.r0 + top - 1 - (j0 + jj)) * kGs3dPartials + k] = s;
            }
            __syncthreads();
        }
        top -= nb;
    }
}

// ---- gather and chain rule -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kGs3dGatherThreads) gs3d_gather_kernel(const __grid_constant__ Gs3dGradArgs g) {
    const Gs3dSaveArgs& a = g.a;
    const unsigned long long i = (unsigned long long)blockIdx.x * kGs3dGatherThreads + threadIdx.x;
    if (i >= a.count) return;
    float* out = g.grad + i * kPacked56Floats;
    const uint32_t drawn = reinterpret_cast<const uint32_t*>(a.scratch)[2];
    const uint32_t rk = a.rank[i];
    const float2* r = reinterpret_cast<const float2*>(a.records + i * 56ull);
    const float* rec = reinterpret_cast<const float*>(r);
    // a NaN logit: opacity NaN, alpha min(0.99, NaN) = 0.99, and NaN in every partial of the record; its row is zero
    if (a.keys[i] == kGs3dCulled || rk >= drawn || rec[13] != rec[13]) {
#pragma unroll
        for (int k = 0; k < kPacked56Floats; ++k) out[k] = 0.0f;
        return;
    }
    // ---- the partials of the record's pairs, tile by tile in tile-id order ----
    const BinLayout l = bin_layout(a.count, tile_count(a.width, a.height));
    const uint32_t* start = reinterpret_cast<const uint32_t*>(a.scratch + l.ranges_off);
    const uint32_t* end = start + l.tiles;
    const Gs3dSplat sp = a.splats[i];
    const uint32_t rx = __float_as_uint(sp.c.y), ry = __float_as_uint(sp.c.z), gx = tiles_x(a.width);
    float P[kGs3dPartials] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    for (uint32_t ty = ry & 0xFFFFu; ty < (ry >> 16); ++ty)
        for (uint32_t tx = rx & 0xFFFFu; tx < (rx >> 16); ++tx) {
            const uint32_t t = ty * gx + tx, r0 = start[t];
            uint32_t lo = r0, hi = end[t];   // the run is in depth-rank order: the first slot whose rank is >= rk
            while (lo < hi) {
                const uint32_t mid = lo + (hi - lo) / 2;
                if (a.rank[g.vals[mid]] < rk) lo = mid + 1;
                else hi = mid;
            }
            if (lo - r0 >= g.tile_last[t]) continue;   // past the tile's last contributor: no partial was written
            const float* q = g.part + (size_t)lo * kGs3dPartials;
#pragma unroll
            for (int k = 0; k < kGs3dPartials; ++k) P[k] = ad(P[k], q[k]);
        }
    // ---- the record's forward values ----
    GaussFields gf;
    packed56_fields<true>(r[0], r[1], r[2], r[3], r[4], r[5], r[6], gf);
    Gs3dProj o;
    gs3d_project(a, gf, o);   // not culled: true
    const float det = sb(ml(o.ca, o.cc), ml(o.cb, o.cb));
    // ---- colour -> SH0 (C0; a channel clamped at 0 gets nothing) and opacity -> logit (an infinite logit gets 0) ----
    const float kC0 = 0.28209479177387814f;
    out[10] = gf.cr < 0.0f ? 0.0f : ml(P[6], kC0);
    out[11] = gf.cg < 0.0f ? 0.0f : ml(P[7], kC0);
    out[12] = gf.cb < 0.0f ? 0.0f : ml(P[8], kC0);
    out[13] = isfinite(rec[13]) ? ml(P[5], ml(gf.ca, sb(1.0f, gf.ca))) : 0.0f;
    // ---- conic -> dilated 2-D covariance: conic = (c, -b, a) / det ----
    const float i2 = dv(1.0f, ml(det, det));
    const float dA = P[2], dB = P[3], dC = P[4];
    const float dca = ml(ad(ad(ml(dA, -ml(o.cc, o.cc)), ml(dB, ml(o.cb, o.cc))), ml(dC, -ml(o.cb, o.cb))), i2);
    const float dcb = ml(ad(ad(ml(dA, ml(2.0f, ml(o.cb, o.cc))), ml(dB, -ad(ml(o.ca, o.cc), ml(o.cb, o.cb)))), ml(dC, ml(2.0f, ml(o.cb, o.ca)))), i2);
    const float dcc = ml(ad(ad(ml(dA, -ml(o.cb, o.cb)), ml(dB, ml(o.cb, o.ca))), ml(dC, -ml(o.ca, o.ca))), i2);
    // ---- cov = T Sigma T^T: dL/dSigma = T^T Gc T, dL/dT = 2 Gc T Sigma = 2 Gc A, Gc = [[dca, dcb/2], [dcb/2, dcc]] ----
    const float hb = ml(0.5f, dcb);
    const float Gc[2][2] = {{dca, hb}, {hb, dcc}};
    float dS[3][3], dT[2][3];
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
        for (int q = 0; q < 3; ++q)
            dS[p][q] = ad(ad(ad(ml(ml(o.T[0][p], Gc[0][0]), o.T[0][q]), ml(ml(o.T[0][p], Gc[0][1]), o.T[1][q])),
                             ml(ml(o.T[1][p], Gc[1][0]), o.T[0][q])), ml(ml(o.T[1][p], Gc[1][1]), o.T[1][q]));
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < 3; ++j) dT[m][j] = ml(2.0f, ad(ml(Gc[m][0], o.A[0][j]), ml(Gc[m][1], o.A[1][j])));
    // ---- T = J W -> J -> view position (graphdeco: a clamped t.x / d or t.y / d passes nothing to t.x or t.y) ----
    float dJ00 = 0.0f, dJ02 = 0.0f, dJ11 = 0.0f, dJ12 = 0.0f;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        dJ00 = ad(dJ00, ml(dT[0][j], a.MV[4 * j + 0]));
        dJ02 = ad(dJ02, ml(dT[0][j], a.MV[4 * j + 2]));
        dJ11 = ad(dJ11, ml(dT[1][j], a.MV[4 * j + 1]));
        dJ12 = ad(dJ12, ml(dT[1][j], a.MV[4 * j + 2]));
    }
    const float W = (float)a.width, H = (float)a.height, d3 = ml(o.dd, o.d);
    // dL/dd of J00 = fx / d, J11 = fy / d, J02 = fx txc / d^2, J12 = fy tyc / d^2 (txc, tyc held)
    const float dd_J = sb(sb(sb(-ml(dJ00, dv(o.fx, o.dd)), ml(dJ11, dv(o.fy, o.dd))), ml(dJ02, dv(ml(2.0f, ml(o.fx, o.txc)), d3))),
                          ml(dJ12, dv(ml(2.0f, ml(o.fy, o.tyc)), d3)));
    float dt[3];
    dt[0] = o.clamp_x ? 0.0f : ml(dJ02, dv(o.fx, o.dd));
    dt[1] = o.clamp_y ? 0.0f : ml(dJ12, dv(o.fy, o.dd));
    dt[2] = -dd_J;   // d = -t.z
    // ---- the pixel mean: u = ((c0 pw + 1) W - 1) / 2, v likewise, pw = 1 / (c3 + 1e-7) ----
    const float du = ml(ml(P[0], W), 0.5f), dvv = ml(ml(P[1], H), 0.5f);
    const float dc0 = ml(du, o.pw), dc1 = ml(dvv, o.pw);
    const float dc3 = -ml(ad(ml(du, o.c0), ml(dvv, o.c1)), ml(o.pw, o.pw));
#pragma unroll
    for (int k = 0; k < 3; ++k) dt[k] = ad(dt[k], ad(ad(ml(dc0, a.P[4 * k + 0]), ml(dc1, a.P[4 * k + 1])), ml(dc3, a.P[4 * k + 3])));
#pragma unroll
    for (int j = 0; j < 3; ++j) out[j] = ad(ad(ml(dt[0], a.MV[4 * j + 0]), ml(dt[1], a.MV[4 * j + 1])), ml(dt[2], a.MV[4 * j + 2]));
    // ---- Sigma = Mk^T Mk, Mk[k][j] = s_k R[j][k]: dL/dMk = 2 Mk dSigma ----
    float dR[3][3], ds[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        ds[k] = 0.0f;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float dM = ml(2.0f, ad(ad(ml(o.Mk[k][0], dS[0][j]), ml(o.Mk[k][1], dS[1][j])), ml(o.Mk[k][2], dS[2][j])));
            ds[k] = ad(ds[k], ml(dM, o.R[j][k]));
            dR[j][k] = ml(dM, o.s[k]);
        }
        out[7 + k] = ml(ds[k], o.s[k]);   // s = exp(log-scale) scale_modifier
    }
    // ---- R(q / |q|) -> q ----
    const float qr = o.qr, qi = o.qi, qj = o.qj, qk = o.qk;
    const float gr = ml(2.0f, ad(ad(ml(qk, sb(dR[1][0], dR[0][1])), ml(qj, sb(dR[0][2], dR[2][0]))), ml(qi, sb(dR[2][1], dR[1][2]))));
    const float gi = sb(ml(2.0f, ad(ad(ml(qj, ad(dR[0][1], dR[1][0])), ml(qk, ad(dR[0][2], dR[2][0]))), ml(qr, sb(dR[2][1], dR[1][2])))),
                        ml(ml(4.0f, qi), ad(dR[1][1], dR[2][2])));
    const float gj = sb(ml(2.0f, ad(ad(ml(qi, ad(dR[0][1], dR[1][0])), ml(qr, sb(dR[0][2], dR[2][0]))), ml(qk, ad(dR[1][2], dR[2][1])))),
                        ml(ml(4.0f, qj), ad(dR[0][0], dR[2][2])));
    const float gk = sb(ml(2.0f, ad(ad(ml(qr, sb(dR[1][0], dR[0][1])), ml(qi, ad(dR[0][2], dR[2][0]))), ml(qj, ad(dR[1][2], dR[2][1])))),
                        ml(ml(4.0f, qk), ad(dR[0][0], dR[1][1])));
    const float dot = ad(ad(ad(ml(qr, gr), ml(qi, gi)), ml(qj, gj)), ml(qk, gk));
    out[3] = dv(sb(gr, ml(qr, dot)), o.qn);
    out[4] = dv(sb(gi, ml(qi, dot)), o.qn);
    out[5] = dv(sb(gj, ml(qj, dot)), o.qn);
    out[6] = dv(sb(gk, ml(qk, dot)), o.qn);
}

cudaError_t gs3d_backward_launch(const Gs3dGradArgs& g, cudaStream_t stream) {
    if (g.a.count == 0) return cudaSuccess;
    gs3d_tile_backward_kernel<<<(unsigned)tile_count(g.a.width, g.a.height), kTileThreads, 0, stream>>>(g);
    gs3d_gather_kernel<<<(unsigned)((g.a.count + kGs3dGatherThreads - 1) / kGs3dGatherThreads), kGs3dGatherThreads, 0, stream>>>(g);
    return cudaGetLastError();
}

}  // namespace m2s
