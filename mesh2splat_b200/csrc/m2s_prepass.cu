// m2s_prepass.cu — the step after the conversion in the reference's frame graph (SURVEY 8 f-4): the viewer prepass,
// GaussiansPrepass::execute (src/renderer/renderPasses/GaussiansPrepass.cpp:8-55) + gaussianSplattingPrepassCS.glsl:58-204
// + common.glsl.  Per gaussian: model/view/clip transform, frustum cull, 3-D covariance, EWA projection, screen axes,
// append of one 96-byte QuadNdcTransformation and of the view depth the radix sort keys on.
//
// Shape: a streaming kernel, HBM-bound (96 or 56 B in, 100 B out per survivor, ~250 flops).  One thread per gaussian; the
// survivors of a warp are appended with ONE atomicAdd (the reference: one atomicCounterIncrement per gaussian), staged in
// shared memory and written as one contiguous span with 16-byte stores.  Consumes the conversion's REF96 records
// (u_format 0), its PACKED56 records (a standard 3DGS gaussian: u_format 1 without PBR values), or the REF96 records
// m2s_ply_read loads from a .ply (u_format 1, u_plyHasPbr 0 or 1): the record layout and u_format are separate arguments.
#include "m2s_prepass.cuh"

namespace m2s {

__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
__device__ __forceinline__ void m3mul(const float* a, const float* b, float* r) {   // column-major: r = a * b
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int row = 0; row < 3; ++row)
            r[c * 3 + row] = a[0 * 3 + row] * b[c * 3 + 0] + a[1 * 3 + row] * b[c * 3 + 1] + a[2 * 3 + row] * b[c * 3 + 2];
}

constexpr int kPrepassThreads = 256;

// kStage: fetch the warp's records as one contiguous span through shared memory (large inputs: fewer, wider memory
// transactions) or with six strided 16-byte loads per lane straight into registers (small inputs: one dependent stage less)
// GLM mat4 * vec4: (m0 x + m1 y) + (m2 z + m3 w), round-to-nearest fp32, no contraction
__device__ __forceinline__ float m4row_rn(const float* m, int row, float x, float y, float z, float w) {
    return __fadd_rn(__fadd_rn(__fmul_rn(m[row], x), __fmul_rn(m[4 + row], y)), __fadd_rn(__fmul_rn(m[8 + row], z), __fmul_rn(m[12 + row], w)));
}

// the mesh depth test (gaussianSplattingPrepassCS.glsl:78-91, u_depthTestMesh 1, DESIGN §2): pos2d again in GLSL / GLM
// order without contraction, uv and myDepth as the shader writes them, the map read NEAREST + CLAMP_TO_EDGE (a NaN
// coordinate reads texel 0); true if the gaussian is behind the mesh
__device__ __forceinline__ bool prepass_behind_mesh(const PrepassArgs& a, const float* map, uint32_t dw, uint32_t dh,
                                                    float px, float py, float pz) {
    const float w0 = m4row_rn(a.M, 0, px, py, pz, 1.0f), w1 = m4row_rn(a.M, 1, px, py, pz, 1.0f), w2 = m4row_rn(a.M, 2, px, py, pz, 1.0f);
    const float v0 = m4row_rn(a.V, 0, w0, w1, w2, 1.0f), v1 = m4row_rn(a.V, 1, w0, w1, w2, 1.0f), v2 = m4row_rn(a.V, 2, w0, w1, w2, 1.0f),
                v3 = m4row_rn(a.V, 3, w0, w1, w2, 1.0f);
    const float c0 = m4row_rn(a.P, 0, v0, v1, v2, v3), c1 = m4row_rn(a.P, 1, v0, v1, v2, v3), c2 = m4row_rn(a.P, 2, v0, v1, v2, v3),
                c3 = m4row_rn(a.P, 3, v0, v1, v2, v3);
    const float u = __fadd_rn(__fmul_rn(__fdiv_rn(c0, c3), 0.5f), 0.5f), v = __fadd_rn(__fmul_rn(__fdiv_rn(c1, c3), 0.5f), 0.5f);
    const uint32_t i = (uint32_t)fminf(fmaxf(floorf(__fmul_rn(u, (float)dw)), 0.0f), (float)(dw - 1));
    const uint32_t j = (uint32_t)fminf(fmaxf(floorf(__fmul_rn(v, (float)dh)), 0.0f), (float)(dh - 1));
    const float depth = __ldg(map + (size_t)j * dw + i);
    const float my = __fadd_rn(__fmul_rn(__fdiv_rn(c2, c3), 0.5f), 0.5f);
    return my > __fadd_rn(depth, 0.00002f);
}

// kDepth: the prepass with the mesh depth test (map: dw x dh floats as m2s_mesh_depth writes them)
template <bool kStage, bool kDepth>
__device__ __forceinline__ void prepass_body(const PrepassArgs& a, const float* map, uint32_t dw, uint32_t dh) {
    __shared__ float4 stage[kPrepassThreads / 32][32 * 6];   // 3 KB per warp: the warp's surviving quads
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long n = a.count;
    if (a.d_count) n = min(n, *a.d_count);
    const unsigned long long gid = (unsigned long long)blockIdx.x * kPrepassThreads + threadIdx.x;
    bool alive = gid < n;
    // ---- the warp's 32 records: one contiguous span of the input, fetched with 16-byte loads (lane i takes float4 i, i + 32,
    // ...) into the warp's stage; then every lane reads its own record from shared memory ----
    const unsigned stride = a.layout == 0 ? 96u : 56u;
    if (kStage) {
        const unsigned long long w0 = gid - lane;                     // first gaussian of the warp
        const unsigned long long nb = w0 < n ? min((unsigned long long)32, n - w0) * stride : 0ull;   // bytes of the span
        const float4* src = reinterpret_cast<const float4*>(a.records + w0 * stride);   // 16-byte aligned: 32 * stride is a multiple of 16
        for (unsigned i = lane; i * 16ull < nb; i += 32) {
            if (i * 16ull + 16ull <= nb) stage[warp][i] = __ldg(src + i);
            else {   // the last 8 bytes of a PACKED56 span that ends on an odd record
                const float2 t = __ldg(reinterpret_cast<const float2*>(src + i));
                stage[warp][i] = make_float4(t.x, t.y, 0.f, 0.f);
            }
        }
    }
    if (kStage) __syncwarp();
    // ---- the gaussian as the shader sees it (GaussianVertex) ----
    float px = 0, py = 0, pz = 0, cr = 0, cg = 0, cb = 0, ca = 0, sx = 0, sy = 0, sz = 0, nx = 0, ny = 0, nz = 0, qx = 1, qy = 0, qz = 0, qw = 0, pb0 = 0, pb1 = 0;
    if (alive) {
        if (a.layout == 0) {   // REF96: position color scale normal rotation pbr
            const float4* gs = stage[warp] + lane * 6;
            const float4* gg = reinterpret_cast<const float4*>(a.records) + gid * 6;
            const float4 p = kStage ? gs[0] : __ldg(gg), c = kStage ? gs[1] : __ldg(gg + 1), s = kStage ? gs[2] : __ldg(gg + 2),
                         nn = kStage ? gs[3] : __ldg(gg + 3), q = kStage ? gs[4] : __ldg(gg + 4), pb = kStage ? gs[5] : __ldg(gg + 5);
            px = p.x; py = p.y; pz = p.z; cr = c.x; cg = c.y; cb = c.z; ca = c.w; sx = s.x; sy = s.y; sz = s.z;
            nx = nn.x; ny = nn.y; nz = nn.z; qx = q.x; qy = q.y; qz = q.z; qw = q.w; pb0 = pb.x; pb1 = pb.y;
        } else {               // PACKED56: xyz | quat wxyz | log-scale | SH0 | opacity logit  (parsers.cpp:560-622 on load)
            const float2* gs = reinterpret_cast<const float2*>(reinterpret_cast<const unsigned char*>(stage[warp]) + lane * 56u);
            const float2* gg = reinterpret_cast<const float2*>(a.records + gid * 56ull);
            const float2 f0 = kStage ? gs[0] : __ldg(gg), f1 = kStage ? gs[1] : __ldg(gg + 1), f2 = kStage ? gs[2] : __ldg(gg + 2),
                         f3 = kStage ? gs[3] : __ldg(gg + 3), f4 = kStage ? gs[4] : __ldg(gg + 4), f5 = kStage ? gs[5] : __ldg(gg + 5),
                         f6 = kStage ? gs[6] : __ldg(gg + 6);
            px = f0.x; py = f0.y; pz = f1.x; qx = f1.y; qy = f2.x; qz = f2.y; qw = f3.x;
            sx = expf(f3.y); sy = expf(f4.x); sz = expf(f4.y);
            const float kC0 = 0.28209479177387814f;
            cr = f5.x * kC0 + 0.5f; cg = f5.y * kC0 + 0.5f; cb = f6.x * kC0 + 0.5f;
            ca = 1.0f / (1.0f + expf(-f6.y));
        }
    }
    if (kStage) __syncwarp();   // every lane has its record: the stage is free for the warp's output
    float ws0 = 0, ws1 = 0, ws2 = 0, vs0 = 0, vs1 = 0, vs2 = -1, c0 = 0, c1 = 0, c2 = 0, c3 = 1;
    if (alive) {
        ws0 = a.M[0] * px + a.M[4] * py + a.M[8] * pz + a.M[12];      // :66
        ws1 = a.M[1] * px + a.M[5] * py + a.M[9] * pz + a.M[13];
        ws2 = a.M[2] * px + a.M[6] * py + a.M[10] * pz + a.M[14];
        vs0 = a.V[0] * ws0 + a.V[4] * ws1 + a.V[8] * ws2 + a.V[12];   // :68
        vs1 = a.V[1] * ws0 + a.V[5] * ws1 + a.V[9] * ws2 + a.V[13];
        vs2 = a.V[2] * ws0 + a.V[6] * ws1 + a.V[10] * ws2 + a.V[14];
        const float vs3 = a.V[3] * ws0 + a.V[7] * ws1 + a.V[11] * ws2 + a.V[15];
        c0 = a.P[0] * vs0 + a.P[4] * vs1 + a.P[8] * vs2 + a.P[12] * vs3;   // :70
        c1 = a.P[1] * vs0 + a.P[5] * vs1 + a.P[9] * vs2 + a.P[13] * vs3;
        c2 = a.P[2] * vs0 + a.P[6] * vs1 + a.P[10] * vs2 + a.P[14] * vs3;
        c3 = a.P[3] * vs0 + a.P[7] * vs1 + a.P[11] * vs2 + a.P[15] * vs3;
        const float clip = 1.05f * c3;                                   // :72-76
        if (c2 < -clip || c0 < -clip || c0 > clip || c1 < -clip || c1 > clip) alive = false;
        if (kDepth && alive && a.fmt == 0 && ca > 0.95f && prepass_behind_mesh(a, map, dw, dh, px, py, pz)) alive = false;
    }
    float4 q0, q1, q2, q3, q4, q5;
    q0 = q1 = q2 = q3 = q4 = q5 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (alive) {
        const bool fmt0 = a.fmt == 0;
        const float mult = fmt0 ? a.std_dev : 1.0f;                     // :95-97
        const float s0 = sx * mult * a.mscale2[0], s1 = sy * mult * a.mscale2[1], s2 = sz * mult * a.mscale2[2];
        // castQuatToMat3 (common.glsl:22-48): the three "rows" are the COLUMNS of the matrix; quat = (w, x, y, z)
        const float rot0[9] = {1.f - 2.f * (qz * qz + qw * qw), 2.f * (qy * qz - qx * qw), 2.f * (qy * qw + qx * qz),
                               2.f * (qy * qz + qx * qw), 1.f - 2.f * (qy * qy + qw * qw), 2.f * (qz * qw - qx * qy),
                               2.f * (qy * qw - qx * qz), 2.f * (qz * qw + qx * qy), 1.f - 2.f * (qy * qy + qz * qz)};
        float rot[9];
        m3mul(rot0, a.Ninv, rot);                                       // :109
        float mm[9], mmT[9], cov3d[9];                                  // computeCov3D (common.glsl:50-61)
#pragma unroll
        for (int c = 0; c < 3; ++c) { mm[c * 3 + 0] = s0 * rot[c * 3 + 0]; mm[c * 3 + 1] = s1 * rot[c * 3 + 1]; mm[c * 3 + 2] = s2 * rot[c * 3 + 2]; }
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int k = 0; k < 3; ++k) mmT[c * 3 + k] = mm[k * 3 + c];
        m3mul(mmT, mm, cov3d);
        float n0 = 1.f, n1 = 0.f, n2 = 0.f, n3 = 0.f;
        if (fmt0 || a.ply_has_pbr) {                                     // :117-121 normal through the normal matrix
            n0 = (a.Nmat[0] * nx + a.Nmat[4] * ny + a.Nmat[8] * nz + a.Nmat[12]) * 0.5f + 0.5f;
            n1 = (a.Nmat[1] * nx + a.Nmat[5] * ny + a.Nmat[9] * nz + a.Nmat[13]) * 0.5f + 0.5f;
            n2 = (a.Nmat[2] * nx + a.Nmat[6] * ny + a.Nmat[10] * nz + a.Nmat[14]) * 0.5f + 0.5f;
            n3 = ca;
        } else {                                                         // :123-130 shortest axis (raw scales)
            const unsigned idx = (unsigned)((sy < sz) && (sy < sx)) + (unsigned)((sz < sy) && (sz < sx)) * 2u;
            const float r0 = idx == 0 ? rot[0] : (idx == 1 ? rot[3] : rot[6]), r1 = idx == 0 ? rot[1] : (idx == 1 ? rot[4] : rot[7]),
                        r2 = idx == 0 ? rot[2] : (idx == 1 ? rot[5] : rot[8]);
            n0 = r0 * 0.5f + 0.5f; n1 = r1 * 0.5f + 0.5f; n2 = r2 * 0.5f + 0.5f; n3 = ca;
        }
        float o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f;                    // :132-148
        if (a.render_mode == 0 || a.render_mode == 6) { o0 = cr; o1 = cg; o2 = cb; o3 = ca; }
        else if (a.render_mode == 1) {
            const float d = clamp01(expf(-20.0f * clamp01((-vs2 - a.near_far[0]) / (a.near_far[1] - a.near_far[0]))));   // common.glsl:80-84
            o0 = o1 = o2 = d; o3 = ca;
        } else if (a.render_mode == 2) { o0 = n0; o1 = n1; o2 = n2; o3 = n3; }
        // :153-170 EWA projection
        const float tzSq = vs2 * vs2;
        const float jsx = -(a.P[0] * a.res[0]) / (2 * vs2), jsy = -(a.P[5] * a.res[1]) / (2 * vs2);
        const float jtx = (a.P[0] * vs0 * a.res[0]) / (2 * tzSq), jty = (a.P[5] * vs1 * a.res[1]) / (2 * tzSq);
        const float jtz = ((a.near_far[1] - a.near_far[0]) * a.P[14]) / (2 * tzSq);
        const float J[9] = {jsx, 0.f, 0.f, 0.f, jsy, 0.f, jtx, jty, jtz};
        const float W[9] = {a.V[0], a.V[1], a.V[2], a.V[4], a.V[5], a.V[6], a.V[8], a.V[9], a.V[10]};
        float JW[9], JWT[9], t9[9], Vp[9];
        m3mul(J, W, JW);
#pragma unroll
        for (int c = 0; c < 3; ++c)
#pragma unroll
            for (int k = 0; k < 3; ++k) JWT[c * 3 + k] = JW[k * 3 + c];
        m3mul(JW, cov3d, t9);
        m3mul(t9, JWT, Vp);
        const float c00 = Vp[0] + 0.3f, c01 = Vp[1], c10 = Vp[3], c11 = Vp[4] + 0.3f;   // :172-176
        const float mid = c00 + c11, dx = c00 - c11, dy = 2 * c01;
        const float delta = sqrtf(dx * dx + dy * dy);
        const float lambda1 = 0.5f * (mid + delta), lambda2 = 0.5f * (mid - delta);
        if (lambda2 < 0.0f) alive = false;                                               // :185
        else {
            float dvx = 1.0f, dvy = (-c00 + c01 + lambda1) / (c01 - c11 + lambda1);        // :187 (0/0 for a round splat, as in the reference)
            const float dinv = 1.0f / sqrtf(dvx * dvx + dvy * dvy);
            dvx *= dinv; dvy *= dinv;
            const float r1 = fminf(3 * sqrtf(lambda1), 1024.0f), r2 = fminf(3 * sqrtf(lambda2), 1024.0f);
            const float hx = a.res[0] * 0.5f, hy = a.res[1] * 0.5f;
            q0 = make_float4(c0 / c3, c1 / c3, c2 / c3, c3);                               // :150, :196
            q1 = make_float4(r1 * dvx / hx, r1 * dvy / hy, r2 * dvy / hx, r2 * -dvx / hy);
            q2 = make_float4(o0, o1, o2, o3);
            const float det = c00 * c11 - c01 * c10;                                       // inverseMat2 (common.glsl:63-78)
            float i00 = 0.f, i01 = 0.f, i11 = 0.f;
            if (det != 0.0f) { i00 = c11 / det; i01 = -c01 / det; i11 = c00 / det; }
            q3 = make_float4(i00, i01, i11, -vs2);
            q4 = make_float4(n0, n1, n2, pb0);
            q5 = make_float4(ws0, ws1, ws2, pb1);
        }
    }
    // ---- append: one atomicAdd per warp, the warp's quads leave as one contiguous span ----
    const unsigned mask = __ballot_sync(0xffffffffu, alive);
    const unsigned cnt = __popc(mask), rank = __popc(mask & ((1u << lane) - 1u));
    unsigned base = 0;
    if (lane == 0 && cnt) base = atomicAdd(a.valid, cnt);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (alive) {
        float4* s = stage[warp] + rank * 6;
        s[0] = q0; s[1] = q1; s[2] = q2; s[3] = q3; s[4] = q4; s[5] = q5;
        a.depths[base + rank] = vs2;                                                       // :204
    }
    __syncwarp();
    float4* dst = a.quads + (size_t)base * 6;
    for (unsigned i = lane; i < cnt * 6; i += 32) dst[i] = stage[warp][i];
}

template <bool kStage>
__global__ void __launch_bounds__(kPrepassThreads) prepass_kernel(const __grid_constant__ PrepassArgs a) {
    prepass_body<kStage, false>(a, nullptr, 0, 0);
}

template <bool kStage>
__global__ void __launch_bounds__(kPrepassThreads) prepass_depth_kernel(const __grid_constant__ PrepassDepthArgs a) {
    prepass_body<kStage, true>(a.p, a.map, a.width, a.height);
}

cudaError_t prepass_launch(const PrepassArgs& args, cudaStream_t stream) {
    if (args.count == 0) return cudaSuccess;
    const unsigned long long blocks = (args.count + kPrepassThreads - 1) / kPrepassThreads;
    if (args.count >= (2ull << 20)) prepass_kernel<true><<<(unsigned)blocks, kPrepassThreads, 0, stream>>>(args);
    else prepass_kernel<false><<<(unsigned)blocks, kPrepassThreads, 0, stream>>>(args);
    return cudaGetLastError();
}

cudaError_t prepass_depth_launch(const PrepassDepthArgs& args, cudaStream_t stream) {
    if (args.p.count == 0) return cudaSuccess;
    const unsigned long long blocks = (args.p.count + kPrepassThreads - 1) / kPrepassThreads;
    if (args.p.count >= (2ull << 20)) prepass_depth_kernel<true><<<(unsigned)blocks, kPrepassThreads, 0, stream>>>(args);
    else prepass_depth_kernel<false><<<(unsigned)blocks, kPrepassThreads, 0, stream>>>(args);
    return cudaGetLastError();
}

}  // namespace m2s
