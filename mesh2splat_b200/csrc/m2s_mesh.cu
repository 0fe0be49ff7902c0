// m2s_mesh.cu — the viewer's mesh G-buffer pass (SURVEY 8 row 14, f-11): MeshRenderPass::execute
// (src/renderer/renderPasses/MeshRenderPass.cpp:8-73) + meshRenderVS.glsl / meshRenderPS.glsl (+ common.glsl).  Every
// triangle of every primitive drawn into its own five-target G-buffer cleared to 0, back faces culled, depth test LESS
// on a D24 buffer cleared to 1, no blending.
//
// Shape (the depth pre-pass's, m2s_depth.cu, with the clip stage of m2s_clip.cuh):
//   binning (m2s_bin.cuh) per source triangle: P (V (M p)), clip, fan, snap, cull, and the 16 x 16 tiles each fan
//                        triangle touches; (tile, source triangle << 3 | fan triangle) pairs of the longest prefix of
//                        source triangles that fits the budget, stably sorted by tile; each tile's run
//   mesh_tile_kernel     one CTA per tile, one thread per pixel.  Pass 1: the fan triangles staged in shared memory, the
//                        depth from the exact edge values in fp64, the minimum D24 code and the first fragment (in draw
//                        order) that reached it.  Pass 2: the winner shaded once — the fragment shader has no side
//                        effects and no discard, so this is GL's result — and one store per live target.
// The vertex stage of the winner's source triangle is recomputed by each pixel that shades it (mesh_shade): no
// per-triangle record, and the same arithmetic wherever it runs.  The fixed-function choices (perspective-correct
// interpolation, 2 x 2 quad derivatives, the LOD's log2, the sin of render mode 3) are DESIGN §2; every operation that
// decides a bit is round-to-nearest fp32 / fp64 with no contraction, so the G-buffer equals the oracle's
// (oracle/m2s_mesh_oracle.c) bit for bit.
#include "m2s_bin.cuh"
#include "m2s_clip.cuh"
#include "m2s_mesh.cuh"
#include "m2s_shade.cuh"

namespace m2s {

namespace {
__device__ __forceinline__ double dad(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dml(double a, double b) { return __dmul_rn(a, b); }

// meshRenderVS.glsl:26-37: worldPos = M (p, 1), viewPos = V worldPos, gl_Position = P viewPos (GLM's mat4 * vec4 each)
__device__ __forceinline__ void mesh_positions(const MeshArgs& a, float x, float y, float z, float (&w)[4], float (&v)[4], float4& c) {
#pragma unroll
    for (int r = 0; r < 4; ++r) w[r] = clip_row(a.M, r, x, y, z, 1.0f);
#pragma unroll
    for (int r = 0; r < 4; ++r) v[r] = clip_row(a.V, r, w[0], w[1], w[2], w[3]);
    c = make_float4(clip_row(a.P, 0, v[0], v[1], v[2], v[3]), clip_row(a.P, 1, v[0], v[1], v[2], v[3]),
                    clip_row(a.P, 2, v[0], v[1], v[2], v[3]), clip_row(a.P, 3, v[0], v[1], v[2], v[3]));
}

// the vertex transform of the clip stage: gl_Position
struct MeshXf {
    const MeshArgs& a;
    __device__ __forceinline__ float4 operator()(float x, float y, float z) const {
        float w[4], v[4];
        float4 c;
        mesh_positions(a, x, y, z, w, v, c);
        return c;
    }
};

// GLM: dot(v, v) = (x x + y y) + z z; normalize(v) = v * (1 / sqrt(dot(v, v)))
__device__ __forceinline__ void mesh_normalize(float (&v)[3]) {
    const float i = dv(1.0f, __fsqrt_rn(ad(ad(ml(v[0], v[0]), ml(v[1], v[1])), ml(v[2], v[2]))));
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = ml(v[c], i);
}
// GLM mat3 * vec3, column-major n: (n0 x + n1 y) + n2 z
__device__ __forceinline__ void mesh_mat3(const float* n, float x, float y, float z, float (&r)[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) r[k] = ad(ad(ml(n[k], x), ml(n[3 + k], y)), ml(n[6 + k], z));
}

// log2 of x >= 0 from round-to-nearest fp64 operations only (the oracle's orc_mesh_log2 is the same sequence):
// x = m 2^e with m in [sqrt(1/2), sqrt(2)), ln m = 2 atanh((m - 1) / (m + 1)) by its series to the 19th power
__device__ __forceinline__ double mesh_log2(double x) {
    if (x != x) return x;
    if (x == 0.0) return __longlong_as_double(0xfff0000000000000ll);   // -inf
    if (isinf(x)) return x;
    int e;
    double m = frexp(x, &e);
    if (m < 0.70710678118654752440) { m = dml(m, 2.0); e -= 1; }
    const double f = __ddiv_rn(dad(m, -1.0), dad(m, 1.0)), f2 = dml(f, f);
    double p = 1.0 / 19.0;
    p = dad(dml(p, f2), 1.0 / 17.0);
    p = dad(dml(p, f2), 1.0 / 15.0);
    p = dad(dml(p, f2), 1.0 / 13.0);
    p = dad(dml(p, f2), 1.0 / 11.0);
    p = dad(dml(p, f2), 1.0 / 9.0);
    p = dad(dml(p, f2), 1.0 / 7.0);
    p = dad(dml(p, f2), 1.0 / 5.0);
    p = dad(dml(p, f2), 1.0 / 3.0);
    p = dad(dml(p, f2), 1.0);
    return dad((double)e, dml(dml(dml(2.0, f), p), 1.4426950408889634074));
}

// sin from round-to-nearest fp64 operations only (the oracle's orc_mesh_sin is the same sequence): Cody-Waite reduction
// by pi/2 in four parts (three of 21 bits: exact products for |k| < 2^32, every fp32 argument of render mode 3), then
// the quadrant's sine or cosine polynomial
__device__ __forceinline__ double mesh_sin(double x) {
    if (!isfinite(x)) return x - x;
    const double k = rint(dml(x, 6.36619772367581382433e-01));
    double r = dad(x, -dml(k, 1.570796012878418));
    r = dad(r, -dml(k, 3.139164164167596e-07));
    r = dad(r, -dml(k, 6.22337468017542e-14));
    r = dad(r, -dml(k, -2.508278806334166e-20));
    const double z = dml(r, r);
    double s = 1.58969099521155010221e-10;
    s = dad(dml(s, z), -2.50507602534068634195e-08);
    s = dad(dml(s, z), 2.75573137070700676789e-06);
    s = dad(dml(s, z), -1.98412698298579493134e-04);
    s = dad(dml(s, z), 8.33333333332248946124e-03);
    s = dad(dml(s, z), -1.66666666666666324348e-01);
    s = dad(r, dml(dml(r, z), s));
    double c = -1.13596475577881948265e-11;
    c = dad(dml(c, z), 2.08757232129817482790e-09);
    c = dad(dml(c, z), -2.75573143513906633035e-07);
    c = dad(dml(c, z), 2.48015872894767294178e-05);
    c = dad(dml(c, z), -1.38888888888741095749e-03);
    c = dad(dml(c, z), 4.16666666666666019037e-02);
    c = dad(dad(1.0, -dml(0.5, z)), dml(dml(z, z), c));
    switch ((int)((long long)k & 3)) {
        case 0: return s;
        case 1: return c;
        case 2: return -s;
        default: return -c;
    }
}
// meshRenderPS.glsl:68-70: fract(sin(arg) * 43758.5453), fract(x) = x - floor(x)
__device__ __forceinline__ float mesh_hash(float arg) {
    const float v = ml(__double2float_rn(mesh_sin((double)arg)), 43758.5453f);
    return sb(v, floorf(v));
}

// sampler state of one map for a pixel (GL 4.6 §8.14, the conversion's level rule): rho^2 = the larger squared length
// of the quad's uv steps in texels, lambda = 0.5 log2(rho^2); NaN samples level 0 (lambda > 0 fails), +inf the last
__device__ __forceinline__ void mesh_ref(const DTexture& t, float dudx, float dvdx, float dudy, float dvdy, TexRef& ref, float& frac) {
    const float W = (float)t.w[0], H = (float)t.h[0];
    const float ax = ml(dudx, W), bx = ml(dvdx, H), ay = ml(dudy, W), by = ml(dvdy, H);
    const float sx = ad(ml(ax, ax), ml(bx, bx)), sy = ad(ml(ay, ay), ml(by, by));
    const float s2 = (sx != sx || sy != sy) ? __int_as_float(0x7fffffff) : fmaxf(sx, sy);
    const float lam = __double2float_rn(dml(0.5, mesh_log2((double)s2)));
    const int q = (int)t.nlevels - 1;
    int l0 = 0;
    frac = 0.0f;
    if (!(lam > 0.0f)) l0 = 0;                      // magnification (or NaN): LINEAR on level 0
    else if (lam >= (float)q) l0 = q;              // clamped to the last level
    else { const float d = floorf(lam); l0 = (int)d; frac = sb(lam, d); }
    const int l1 = min(l0 + 1, q);
    ref.off0 = t.off[l0]; ref.off1 = t.off[l1];
    ref.w0 = t.w[l0]; ref.h0 = t.h[l0]; ref.w1 = t.w[l1]; ref.h1 = t.h[l1];
}

// texture(map, uv) with the map's sampler state: RGBA in [0, 1] (the conversion's trilinear REPEAT sampler)
__device__ __forceinline__ void mesh_sample(const MeshArgs& a, const TexRef& ref, float frac, float u, float v, float (&out)[4]) {
    const Bilin2 bl = bilin_setup2(ref, wrap01(u), wrap01(v), f2(sb(1.0f, frac), frac));
    uint32_t tx[8];
    fetch_footprint(a.arena, ref, frac, bl, tx);
    const uint32_t k4b = opaque_4b();
    out[0] = filt2<0>(bl.w, tx, k4b); out[1] = filt2<1>(bl.w, tx, k4b);
    out[2] = filt2<2>(bl.w, tx, k4b); out[3] = filt2<3>(bl.w, tx, k4b);
}

}  // namespace

// the binning (m2s_bin.cuh): source triangles, n = ntri, one pair per tile each front-facing fan triangle touches, pair
// value = source triangle << 3 | fan triangle
struct MeshBins {
    MeshArgs a;
    __host__ __device__ unsigned long long items() const { return a.ntri; }
    __host__ __device__ uint64_t tiles() const { return tile_count(a.width, a.height); }
    __device__ __forceinline__ uint32_t n() const { return (uint32_t)a.ntri; }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        auto drawn = [&](uint32_t t) {
            DRange r;
            return prim_range(a.ranges, a.nranges, t, r);
        };
        return clip_visit<true>(a.tris, i, a.width, a.height, drawn, MeshXf{a}, f);
    }
};

struct MeshStage {
    FanEdges e;
    uint32_t prim[kTileThreads];   // the draw order is (primitive, pair value)
    uint32_t val[kTileThreads];
};

// stages fan triangle v & 7 of source triangle v >> 3 in slot `slot`, edge values relative to pixel (ox, oy).  Not
// inlined, as depth_stage.
__device__ __noinline__ void mesh_stage(const MeshArgs& a, uint32_t v, int ox, int oy, MeshStage& s, int slot) {
    DRange r;
    prim_range(a.ranges, a.nranges, v >> 3, r);   // a triangle with pairs has a primitive
    float4 poly[kClipMaxPoly];
    clip_tri_poly(a.tris, v >> 3, MeshXf{a}, poly);
    clip_stage<true>(poly, (int)(v & 7u), a.width, a.height, ox, oy, s.e, slot);
    s.prim[slot] = r.prim;
    s.val[slot] = v;
}

// meshRenderVS.glsl + meshRenderPS.glsl for pixel (x, y) whose winner is pair value `val`: the fan triangle's set-up, the
// vertex stage of its source triangle, the varyings at the pixel and at the three quad pixels the derivatives need, the
// maps, the shading and the target formats.  Not inlined: the tile kernel's pass 1 keeps its registers.
__device__ __noinline__ void mesh_shade(const MeshArgs& a, uint32_t val, int x, int y, GTexel& o) {
    const uint32_t tri = val >> 3;
    const int k = (int)(val & 7u);
    DRange r;
    prim_range(a.ranges, a.nranges, tri, r);
    ClipVert poly[kClipMaxPoly];
    clip_tri_poly(a.tris, tri, MeshXf{a}, poly);
    FanTri d;
    clip_fan<true>(poly, k, a.width, a.height, d);
    double w[3], bc[3][3];   // the fan vertices' clip w and source barycentrics
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const ClipVert& pv = poly[c == 0 ? 0 : k + c];
        w[c] = (double)pv.p.w;
#pragma unroll
        for (int j = 0; j < 3; ++j) bc[c][j] = (double)pv.b[j];
    }
    // vertex stage (meshRenderVS.glsl:26-37) of the three source vertices: worldPos, normal, tangent, uv, viewDepth
    constexpr int kVary = 13;
    float vary[3][kVary];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float4 p0 = __ldg(a.tris + (size_t)tri * 9 + j * 3), p1 = __ldg(a.tris + (size_t)tri * 9 + j * 3 + 1),
                     p2 = __ldg(a.tris + (size_t)tri * 9 + j * 3 + 2);
        float wp[4], vp[4], n[3], t[3];
        float4 c;
        mesh_positions(a, p0.x, p0.y, p0.z, wp, vp, c);
        mesh_mat3(a.N, p0.w, p1.x, p1.y, n);
        mesh_normalize(n);
        mesh_mat3(a.N, p1.z, p1.w, p2.x, t);
        mesh_normalize(t);
        float* o_ = vary[j];
        o_[0] = wp[0]; o_[1] = wp[1]; o_[2] = wp[2];
        o_[3] = n[0]; o_[4] = n[1]; o_[5] = n[2];
        o_[6] = t[0]; o_[7] = t[1]; o_[8] = t[2]; o_[9] = p2.y;
        o_[10] = p2.z; o_[11] = p2.w;
        o_[12] = -vp[2];
    }
    // GL 4.6 §14.6.1 with the exact edge values of the snapped fan triangle: source weights
    // beta = sum (e_k / w_k) beta_k / sum (e_k / w_k), fp64; a pixel outside the triangle extrapolates (helpers)
    auto weights = [&](int px, int py, double (&beta)[3]) {
        double q[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) q[c] = __ddiv_rn((double)((long long)d.t.A[c] * px + (long long)d.t.B[c] * py + d.t.C[c]), w[c]);
        const double s = dad(dad(q[0], q[1]), q[2]);
#pragma unroll
        for (int j = 0; j < 3; ++j) beta[j] = __ddiv_rn(dad(dad(dml(q[0], bc[0][j]), dml(q[1], bc[1][j])), dml(q[2], bc[2][j])), s);
    };
    auto interp = [&](const double (&beta)[3], int i) {
        return __double2float_rn(dad(dad(dml(beta[0], (double)vary[0][i]), dml(beta[1], (double)vary[1][i])), dml(beta[2], (double)vary[2][i])));
    };
    double beta[3];
    weights(x, y, beta);
    float v[kVary];
#pragma unroll
    for (int i = 0; i < kVary; ++i) v[i] = interp(beta, i);
    // coarse derivatives of the 2 x 2 quad (window coordinates, y up): f(2i+1, 2j) - f(2i, 2j), f(2i, 2j+1) - f(2i, 2j)
    const int qx = x & ~1, qy = y & ~1;
    weights(qx, qy, beta);
    const float u00 = interp(beta, 10), v00 = interp(beta, 11);
    weights(qx + 1, qy, beta);
    const float dudx = sb(interp(beta, 10), u00), dvdx = sb(interp(beta, 11), v00);
    weights(qx, qy + 1, beta);
    const float dudy = sb(interp(beta, 10), u00), dvdy = sb(interp(beta, 11), v00);

    // meshRenderPS.glsl:34-93
    const DPrim& pr = a.prims[r.prim];
    float tex[4];
    TexRef ref;
    float frac;
    float alb[3] = {pr.factor[0], pr.factor[1], pr.factor[2]};
    if (pr.tex[0] >= 0) {
        mesh_ref(a.texs[pr.tex[0]], dudx, dvdx, dudy, dvdy, ref, frac);
        mesh_sample(a, ref, frac, v[10], v[11], tex);
#pragma unroll
        for (int c = 0; c < 3; ++c) alb[c] = ml(alb[c], tex[c]);
    }
    float N[3] = {v[3], v[4], v[5]};
    mesh_normalize(N);
    if (pr.tex[1] >= 0) {
        mesh_ref(a.texs[pr.tex[1]], dudx, dvdx, dudy, dvdy, ref, frac);
        mesh_sample(a, ref, frac, v[10], v[11], tex);
        float m[3] = {sb(ml(tex[0], 2.0f), 1.0f), sb(ml(tex[1], 2.0f), 1.0f), sb(ml(tex[2], 2.0f), 1.0f)};
        mesh_normalize(m);
        float T[3] = {v[6], v[7], v[8]};
        mesh_normalize(T);
        float B[3] = {sb(ml(N[1], T[2]), ml(T[1], N[2])), sb(ml(N[2], T[0]), ml(T[2], N[0])), sb(ml(N[0], T[1]), ml(T[0], N[1]))};
        mesh_normalize(B);
#pragma unroll
        for (int c = 0; c < 3; ++c) B[c] = ml(B[c], v[9]);
        float n2[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) n2[c] = ad(ad(ml(T[c], m[0]), ml(B[c], m[1])), ml(N[c], m[2]));
        mesh_normalize(n2);
#pragma unroll
        for (int c = 0; c < 3; ++c) N[c] = n2[c];
    }
    const float en[3] = {ad(ml(N[0], 0.5f), 0.5f), ad(ml(N[1], 0.5f), 0.5f), ad(ml(N[2], 0.5f), 0.5f)};
    float metal = 0.1f, rough = 0.5f;
    if (pr.tex[2] >= 0) {
        mesh_ref(a.texs[pr.tex[2]], dudx, dvdx, dudy, dvdy, ref, frac);
        mesh_sample(a, ref, frac, v[10], v[11], tex);
        metal = tex[2];
        rough = tex[1];
    }
    // computeExponentialDepth (common.glsl:80-84) with GLM's clamp = min(max(x, lo), hi) and rn_exp
    auto glm_clamp01 = [](float x) { const float t = x < 0.0f ? 0.0f : x; return 1.0f < t ? 1.0f : t; };
    const float nd = glm_clamp01(dv(sb(v[12], a.near_far[0]), sb(a.near_far[1], a.near_far[0])));
    const float dep = glm_clamp01(rn_exp(ml(-20.0f, nd)));
    float col[3] = {alb[0], alb[1], alb[2]};   // modes 0, 5, 6
    if (a.mode == 1) { col[0] = col[1] = col[2] = dep; }
    else if (a.mode == 2) { col[0] = en[0]; col[1] = en[1]; col[2] = en[2]; }
    else if (a.mode == 3) {   // gl_PrimitiveID restarts at 0 for each primitive's draw
        const float id = (float)(tri - r.first);
        col[0] = mesh_hash(ml(id, 311.7f));
        col[1] = mesh_hash(ad(ml(id, 269.5f), 1.3f));
        col[2] = mesh_hash(ad(ml(id, 183.3f), 2.7f));
    } else if (a.mode == 4) { col[0] = 0.01f; col[1] = 0.005f; col[2] = 0.0f; }
    o.pos = half4(v[0], v[1], v[2], 1.0f);
    o.nrm = half4(en[0], en[1], en[2], 1.0f);
    o.dep = half4(dep, dep, dep, 1.0f);
    o.alb = unorm8(col[0]) | unorm8(col[1]) << 8 | unorm8(col[2]) << 16 | 255u << 24;
    o.mr = unorm8(metal) | unorm8(rough) << 8 | 255u << 24;
}

__global__ void __launch_bounds__(kTileThreads) mesh_tile_kernel(const __grid_constant__ MeshArgs a, const uint32_t* __restrict__ vals) {
    __shared__ MeshStage s;
    const TileFrame f = tile_frame(a.scratch, bin_layout(a.ntri, tile_count(a.width, a.height)), tiles_x(a.width), blockIdx.x);
    // pass 1: LESS on D24 codes in draw order (primitive table order, then triangle order): the minimum code, and among
    // the fragments that reach it the first one drawn; a code equal to the clear value never passes
    uint32_t best = kD24Clear;
    unsigned long long key = ~0ull;
    tile_batches(f, vals, [&](int tid, uint32_t val) { mesh_stage(a, val, f.ox, f.oy, s, tid); }, [&](uint32_t j) {
        uint32_t code;
        if (!clip_depth(s.e, j, f.lx, f.ly, code)) return;
        const unsigned long long kj = (unsigned long long)s.prim[j] << 32 | s.val[j];
        if (code < best || (code == best && kj < key)) { best = code; key = kj; }
    });
    if (f.x >= (int)a.width || f.y >= (int)a.height) return;
    // pass 2: the winner's fragment shader; the clear colour 0 elsewhere
    GTexel o = {make_uint2(0, 0), make_uint2(0, 0), make_uint2(0, 0), 0u, 0u};
    if (best < kD24Clear) mesh_shade(a, (uint32_t)key, f.x, f.y, o);
    gbuffer_store(a, (size_t)f.y * a.width + f.x, o);
}

// ---- launches -------------------------------------------------------------------------------------------------------
cudaError_t mesh_count_launch(const MeshArgs& a, cudaStream_t stream) { return bin_count_launch(MeshBins{a}, stream); }

cudaError_t mesh_draw_launch(const MeshArgs& a, int sm_count, cudaStream_t stream) {
    return bin_draw_launch(MeshBins{a}, mesh_tile_kernel, sm_count, stream);
}

}  // namespace m2s
