// m2s_depth.cu — the viewer's mesh depth pre-pass (SURVEY 8 f-9): DepthPrepass::execute
// (src/renderer/renderPasses/DepthPrepass.cpp:8-49) + depthPrepassVS.glsl / depthPrepassPS.glsl.  Every triangle of an
// opaque primitive (baseColorFactor.a == 1.0f) drawn into a W x H D24 map cleared to 1, depth test LESS, no culling.
//
// Shape (the shadow pass's cube raster over one W x H viewport, DESIGN §2 "The mesh depth pre-pass"):
//   binning (m2s_bin.cuh) per source triangle: transform, clip (six planes, guard factor 2 in x and y), fan, snap,
//                        and the 16 x 16 tiles each fan triangle touches; (tile, source triangle << 3 | fan triangle)
//                        pairs of the longest prefix of source triangles that fits the budget, stably sorted by tile;
//                        each tile's run
//   depth_tile_kernel    one CTA per tile, one thread per pixel: fan triangles staged in shared memory, depth from the
//                        exact edge values in fp64, the minimum D24 code in a register, one store per texel
// The unit of a pair is the fan triangle, so the tile kernel stages one triangle per pair; it re-clips the source
// triangle to find it (a triangle that needs no clipping is its own fan of one).  Every operation that decides a bit of
// the map is round-to-nearest fp32 / fp64 with no contraction (__f*_rn, __d*_rn), integer, or a conversion of DESIGN
// §2, so the map equals the oracle's (oracle/m2s_depth_oracle.c) bit for bit.
#include "m2s_bin.cuh"
#include "m2s_depth.cuh"

namespace m2s {

namespace {
__device__ __forceinline__ float ad(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sb(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ml(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dv(float a, float b) { return __fdiv_rn(a, b); }

// GLM mat4 * vec4(x, y, z, 1): (m0 x + m1 y) + (m2 z + m3)
__device__ __forceinline__ float depth_row(const float* m, int row, float x, float y, float z) {
    return ad(ad(ml(m[row], x), ml(m[4 + row], y)), ad(ml(m[8 + row], z), ml(m[12 + row], 1.0f)));
}

// signed distance to clip plane p (inside iff >= 0): z >= -w, z <= w, x >= -G w, x <= G w, y >= -G w, y <= G w
__device__ __forceinline__ float depth_plane(const float4& v, int p) {
    const float gw = ml(kDepthGuard, v.w);
    switch (p) {
        case 0: return ad(v.z, v.w);
        case 1: return sb(v.w, v.z);
        case 2: return ad(v.x, gw);
        case 3: return sb(gw, v.x);
        case 4: return ad(v.y, gw);
        default: return sb(gw, v.y);
    }
}

// the point where edge (a inside, b outside) meets the plane, always computed from the inside vertex
__device__ __forceinline__ float4 depth_cut(const float4& a, const float4& b, float da, float db) {
    const float t = dv(da, sb(da, db));
    return make_float4(ad(a.x, ml(t, sb(b.x, a.x))), ad(a.y, ml(t, sb(b.y, a.y))), ad(a.z, ml(t, sb(b.z, a.z))),
                       ad(a.w, ml(t, sb(b.w, a.w))));
}

// triangle -> primitive (sorted, disjoint ranges); a triangle of no primitive or of a non-opaque one is not drawn
__device__ __forceinline__ bool depth_opaque(const DepthArgs& a, uint32_t tri) {
    int lo = 0, hi = (int)a.nranges - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const DRange r = a.ranges[mid];
        if (tri < r.first) hi = mid - 1;
        else if (tri >= r.end) lo = mid + 1;
        else return __ldg(&a.prims[r.prim].factor[3]) == 1.0f;   // DepthPrepass.cpp:33, an exact compare
    }
    return false;
}

// clip-space polygon of source triangle `tri` after Sutherland-Hodgman against the six planes in order; returns its
// vertex count (0: not drawn).  A polygon that would grow past kDepthMaxPoly vertices (only through rounding) keeps
// its first kDepthMaxPoly.
__device__ int depth_poly(const DepthArgs& a, uint32_t tri, float4 (&v)[kDepthMaxPoly]) {
    if (!depth_opaque(a, tri)) return 0;
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 p = __ldg(a.tris + (size_t)tri * 9 + k * 3);
        v[k] = make_float4(depth_row(a.pvm, 0, p.x, p.y, p.z), depth_row(a.pvm, 1, p.x, p.y, p.z),
                           depth_row(a.pvm, 2, p.x, p.y, p.z), depth_row(a.pvm, 3, p.x, p.y, p.z));
        finite &= isfinite(v[k].x) && isfinite(v[k].y) && isfinite(v[k].z) && isfinite(v[k].w);
    }
    if (!finite) return 0;
    bool inside = true;
#pragma unroll
    for (int p = 0; p < 6; ++p)
#pragma unroll
        for (int k = 0; k < 3; ++k) inside &= depth_plane(v[k], p) >= 0.0f;
    if (inside) return 3;
    int n = 3;
    for (int p = 0; p < 6 && n > 0; ++p) {
        float4 o[kDepthMaxPoly];
        int m = 0;
        float dp = depth_plane(v[n - 1], p);
        for (int i = 0; i < n; ++i) {
            const float dc = depth_plane(v[i], p);
            const int prev = i == 0 ? n - 1 : i - 1;
            if (dc >= 0.0f) {
                if (dp < 0.0f && m < kDepthMaxPoly) o[m++] = depth_cut(v[i], v[prev], dc, dp);
                if (m < kDepthMaxPoly) o[m++] = v[i];
            } else if (dp >= 0.0f && m < kDepthMaxPoly) {
                o[m++] = depth_cut(v[prev], v[i], dp, dc);
            }
            dp = dc;
        }
        for (int i = 0; i < m; ++i) v[i] = o[i];
        n = m;
    }
    return n;
}

struct DepthTri {
    SplatTri t;
    float z[3];   // window depth (z / w) 0.5 + 0.5 of the three vertices
};

// fan triangle (v0, vk+1, vk+2): perspective divide, the splat draw's viewport transform, snap and edge set-up
__device__ __forceinline__ void depth_fan(const DepthArgs& a, const float4 (&v)[kDepthMaxPoly], int k, DepthTri& d) {
    const float hw = ml((float)a.width, 0.5f), hh = ml((float)a.height, 0.5f);
    int X[3], Y[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float4 p = v[c == 0 ? 0 : k + c];
        bool okc;
        splat_snap(dv(p.x, p.w), dv(p.y, p.w), hw, hh, okc, X[c], Y[c]);
        ok &= okc;
        d.z[c] = ad(ml(dv(p.z, p.w), 0.5f), 0.5f);
    }
    splat_tri_setup(X, Y, ok, (int)a.width, (int)a.height, d.t);
}

__device__ __forceinline__ int depth_tiles_x(const DepthArgs& a) { return (int)((a.width + kSplatTile - 1) / kSplatTile); }

// visits the tiles the fan triangle touches in tile-id order; returns their number
template <typename F>
__device__ __forceinline__ uint32_t depth_for_each_tile(const SplatTri& t, int tiles_x, F&& f) {
    if (t.x1 < t.x0 || t.y1 < t.y0) return 0;
    uint32_t c = 0;
    for (int ty = t.y0 / kSplatTile; ty <= t.y1 / kSplatTile; ++ty)
        for (int tx = t.x0 / kSplatTile; tx <= t.x1 / kSplatTile; ++tx)
            if (splat_tri_touches(t, tx, ty)) f(c++, (uint32_t)(ty * tiles_x + tx));
    return c;
}

}  // namespace

// the binning (m2s_bin.cuh): source triangles, n = ntri, one pair per tile each fan triangle touches, pair value =
// source triangle << 3 | fan triangle
struct DepthBins {
    DepthArgs a;
    __host__ __device__ unsigned long long items() const { return a.ntri; }
    __host__ __device__ uint64_t tiles() const { return splat_tiles(a.width, a.height); }
    __device__ __forceinline__ uint32_t n() const { return (uint32_t)a.ntri; }
    template <typename F>
    __device__ __forceinline__ uint32_t visit(uint32_t i, F&& f) const {
        float4 v[kDepthMaxPoly];
        const int np = depth_poly(a, i, v);
        const int tx = depth_tiles_x(a);
        uint32_t cnt = 0;
        for (int k = 0; k + 2 < np; ++k) {
            DepthTri d;
            depth_fan(a, v, k, d);
            cnt += depth_for_each_tile(d.t, tx, [&](uint32_t, uint32_t tile) { f(tile, i << 3 | (uint32_t)k); });
        }
        return cnt;
    }
};

struct DepthStage {
    int32_t A[3][kSplatThreads], B[3][kSplatThreads];
    long long C[3][kSplatThreads];   // exact edge values at the tile's pixel (0, 0)
    float z[3][kSplatThreads];
    uint32_t incl[kSplatThreads];    // bit k: edge k owns the samples on it (top-left rule)
};

// stages fan triangle v & 7 of source triangle v >> 3 in slot `slot`, edge values relative to pixel (ox, oy).  Not
// inlined: the tile kernel's pixel loop then keeps its registers, where the division slow paths of the set-up would
// otherwise make it spill them.
__device__ __noinline__ void depth_stage(const DepthArgs& a, uint32_t v, int ox, int oy, DepthStage& s, int slot) {
    float4 poly[kDepthMaxPoly];
    depth_poly(a, v >> 3, poly);   // a triangle with pairs has fan triangle v & 7
    DepthTri d;
    depth_fan(a, poly, (int)(v & 7u), d);
    uint32_t incl = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        s.A[k][slot] = d.t.A[k];
        s.B[k][slot] = d.t.B[k];
        s.C[k][slot] = d.t.C[k] + (long long)d.t.A[k] * ox + (long long)d.t.B[k] * oy;
        s.z[k][slot] = d.z[k];
        incl |= d.t.incl[k] ? 1u << k : 0u;
    }
    s.incl[slot] = incl;
}

__global__ void __launch_bounds__(kSplatThreads) depth_tile_kernel(const __grid_constant__ DepthArgs a, const uint32_t* __restrict__ vals) {
    __shared__ DepthStage s;
    const BinLayout l = bin_layout(a.ntri, splat_tiles(a.width, a.height));
    const uint32_t* start = reinterpret_cast<const uint32_t*>(a.scratch + l.ranges_off);
    const uint32_t tile = blockIdx.x, tx = (uint32_t)depth_tiles_x(a);
    const int ox = (int)(tile % tx) * kSplatTile, oy = (int)(tile / tx) * kSplatTile;
    const int tid = threadIdx.x, lx = tid % kSplatTile, ly = tid / kSplatTile;
    const int x = ox + lx, y = oy + ly;
    const uint32_t r0 = vals ? start[tile] : 0u, r1 = vals ? start[l.tiles + tile] : 0u;
    uint32_t best = kDepthClearCode;
    for (uint32_t base = r0; base < r1; base += kSplatThreads) {
        const uint32_t nb = min(r1 - base, (uint32_t)kSplatThreads);
        __syncthreads();
        if ((uint32_t)tid < nb) depth_stage(a, vals[base + tid], ox, oy, s, tid);
        __syncthreads();
        for (uint32_t j = 0; j < nb; ++j) {
            const uint32_t incl = s.incl[j];
            long long e[3];
            bool in = true;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                e[k] = s.C[k][j] + (long long)s.A[k][j] * lx + (long long)s.B[k][j] * ly;
                in &= e[k] >= ((incl >> k & 1u) ? 0ll : 1ll);
            }
            if (!in) continue;
            // GL 4.6 §14.6.1: z = ((E0 z0 + E1 z1) + E2 z2) / (E0 + E1 + E2), fp64 (the E are exact below 2^46)
            const double num = __dadd_rn(__dadd_rn(__dmul_rn((double)e[0], (double)s.z[0][j]), __dmul_rn((double)e[1], (double)s.z[1][j])),
                                         __dmul_rn((double)e[2], (double)s.z[2][j]));
            const double z = __ddiv_rn(num, (double)(e[0] + e[1] + e[2]));
            if (z != z) continue;   // NaN writes nothing
            const double zc = z < 0.0 ? 0.0 : (z > 1.0 ? 1.0 : z);
            const uint32_t code = __double2uint_rn(__dmul_rn(zc, 16777215.0));   // D24, LESS on codes
            best = min(best, code);
        }
    }
    if (x >= (int)a.width || y >= (int)a.height) return;
    a.depth[(size_t)y * a.width + x] = __fdiv_rn(__uint2float_rn(best), 16777215.0f);
}

// ---- launches -------------------------------------------------------------------------------------------------------
cudaError_t depth_count_launch(const DepthArgs& a, cudaStream_t stream) { return bin_count_launch(DepthBins{a}, stream); }

cudaError_t depth_draw_launch(const DepthArgs& a, int sm_count, cudaStream_t stream) {
    const DepthBins b{a};
    const cudaError_t e = bin_pairs_launch(b, sm_count, stream);
    if (e != cudaSuccess) return e;
    depth_tile_kernel<<<(unsigned)b.tiles(), kSplatThreads, 0, stream>>>(a, bin_vals(b));
    return cudaGetLastError();
}

}  // namespace m2s
