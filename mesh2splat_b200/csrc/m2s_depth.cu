// m2s_depth.cu — the viewer's mesh depth pre-pass (SURVEY 8 f-9): DepthPrepass::execute
// (src/renderer/renderPasses/DepthPrepass.cpp:8-49) + depthPrepassVS.glsl / depthPrepassPS.glsl.  Every triangle of an
// opaque primitive (baseColorFactor.a == 1.0f) drawn into a W x H D24 map cleared to 1, depth test LESS, no culling.
//
// Shape (the shadow pass's cube raster over one W x H viewport, DESIGN §2 "The mesh depth pre-pass"):
//   depth_count_kernel   per source triangle: transform, clip (six planes, guard factor 2 in x and y), fan, snap, and
//                        the 16 x 16 tiles each fan triangle touches; scanned within the block
//   depth_scan_kernel    one CTA: exclusive prefix over the block sums; the total number of pairs
//   depth_emit_kernel    (tile, source triangle << 3 | fan triangle) pairs of the longest prefix of source triangles
//                        that fits the budget
//   sort_pairs16_launch  the depth sort's stable onesweep sort of the pairs by tile id (m2s_sort.cu)
//   depth_ranges_kernel  each tile's run in the sorted pairs
//   depth_tile_kernel    one CTA per tile, one thread per pixel: fan triangles staged in shared memory, depth from the
//                        exact edge values in fp64, the minimum D24 code in a register, one store per texel
// The unit of a pair is the fan triangle, so the tile kernel stages one triangle per pair; it re-clips the source
// triangle to find it (a triangle that needs no clipping is its own fan of one).  Every operation that decides a bit of
// the map is round-to-nearest fp32 / fp64 with no contraction (__f*_rn, __d*_rn), integer, or a conversion of DESIGN
// §2, so the map equals the oracle's (oracle/m2s_depth_oracle.c) bit for bit.
#include <algorithm>

#include "m2s_depth.cuh"
#include "m2s_sort.cuh"

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

constexpr int kDepthScanThreads = 1024;
}  // namespace

__global__ void __launch_bounds__(kSplatBlock) depth_count_kernel(DepthArgs a) {
    __shared__ uint32_t s_warp[kSplatBlock / 32];
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
    uint32_t* excl = reinterpret_cast<uint32_t*>(a.scratch + l.excl_off);
    unsigned long long* blocks = reinterpret_cast<unsigned long long*>(a.scratch + l.blocks_off);
    const uint64_t i = (uint64_t)blockIdx.x * kSplatBlock + threadIdx.x;
    uint32_t cnt = 0;
    if (i < a.ntri) {
        float4 v[kDepthMaxPoly];
        const int n = depth_poly(a, (uint32_t)i, v);
        const int tx = depth_tiles_x(a);
        for (int k = 0; k + 2 < n; ++k) {
            DepthTri d;
            depth_fan(a, v, k, d);
            cnt += depth_for_each_tile(d.t, tx, [](uint32_t, uint32_t) {});
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    uint32_t before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kSplatBlock / 32; ++w) {
        before += w < warp ? s_warp[w] : 0u;
        total += s_warp[w];
    }
    if (i < a.ntri) excl[i] = before + x - cnt;
    if (threadIdx.x == 0) blocks[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kDepthScanThreads) depth_scan_kernel(DepthArgs a) {
    __shared__ unsigned long long s_warp[kDepthScanThreads / 32];
    __shared__ unsigned long long s_carry;
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
    unsigned long long* blocks = reinterpret_cast<unsigned long long*>(a.scratch + l.blocks_off);
    const uint32_t nb = (uint32_t)l.blocks;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nb; base += kDepthScanThreads) {
        const uint32_t b = base + threadIdx.x;
        const unsigned long long v = b < nb ? blocks[b] : 0ull;
        unsigned long long x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) s_warp[warp] = x;
        __syncthreads();
        unsigned long long before = s_carry, chunk = 0;
        for (int w = 0; w < kDepthScanThreads / 32; ++w) {
            before += w < warp ? s_warp[w] : 0ull;
            chunk += s_warp[w];
        }
        if (b < nb) blocks[b] = before + x - v;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) *reinterpret_cast<unsigned long long*>(a.scratch) = s_carry;
}

__global__ void __launch_bounds__(kSplatBlock) depth_emit_kernel(DepthArgs a, uint32_t* keys, uint32_t* vals) {
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
    const uint32_t* excl = reinterpret_cast<const uint32_t*>(a.scratch + l.excl_off);
    const unsigned long long* blocks = reinterpret_cast<const unsigned long long*>(a.scratch + l.blocks_off);
    uint32_t* ctrl = reinterpret_cast<uint32_t*>(a.scratch);
    const unsigned long long total = *reinterpret_cast<const unsigned long long*>(a.scratch);
    const uint32_t n = (uint32_t)a.ntri;
    const uint64_t i64 = (uint64_t)blockIdx.x * kSplatBlock + threadIdx.x;
    if (i64 >= n) return;
    const uint32_t i = (uint32_t)i64;
    auto offset = [&](uint32_t k) { return k < n ? blocks[k / kSplatBlock] + excl[k] : total; };
    const unsigned long long start = offset(i), end = offset(i + 1);
    if (end > a.max_pairs) return;   // not in the prefix whose pairs fit
    if (i + 1 == n || offset(i + 2) > a.max_pairs) {   // the prefix's last triangle
        ctrl[2] = i + 1;
        ctrl[3] = (uint32_t)end;
    }
    if (end == start) return;
    float4 v[kDepthMaxPoly];
    const int np = depth_poly(a, i, v);
    const int tx = depth_tiles_x(a);
    unsigned long long at = start;
    for (int k = 0; k + 2 < np; ++k) {
        DepthTri d;
        depth_fan(a, v, k, d);
        at += depth_for_each_tile(d.t, tx, [&](uint32_t c, uint32_t tile) {
            keys[at + c] = tile;
            vals[at + c] = i << 3 | (uint32_t)k;
        });
    }
}

__global__ void depth_ranges_kernel(DepthArgs a, const uint32_t* keys) {
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
    uint32_t* start = reinterpret_cast<uint32_t*>(a.scratch + l.ranges_off);
    uint32_t* end = start + l.tiles;
    const uint32_t np = reinterpret_cast<const uint32_t*>(a.scratch)[3];
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
        const uint32_t k = keys[i];
        if (i == 0 || keys[i - 1] != k) start[k] = i;
        if (i + 1 == np || keys[i + 1] != k) end[k] = i + 1;
    }
}

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
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
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
cudaError_t depth_count_launch(const DepthArgs& a, cudaStream_t stream) {
    cudaError_t e = cudaMemsetAsync(a.scratch, 0, 16, stream);   // total pairs, drawn, pairs emitted
    if (e != cudaSuccess) return e;
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
    if (l.blocks) depth_count_kernel<<<(unsigned)l.blocks, kSplatBlock, 0, stream>>>(a);
    depth_scan_kernel<<<1, kDepthScanThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t depth_draw_launch(const DepthArgs& a, int sm_count, cudaStream_t stream) {
    const SplatLayout l = splat_layout(a.ntri, a.width, a.height);
    cudaError_t e = cudaMemsetAsync(a.scratch + l.ranges_off, 0, l.tiles * 8, stream);
    if (e != cudaSuccess) return e;
    uint32_t* keys = a.max_pairs ? sort_pairs16_keys(a.pairs, a.max_pairs) : nullptr;
    uint32_t* vals = a.max_pairs ? sort_pairs16_vals(a.pairs, a.max_pairs) : nullptr;
    if (l.blocks) depth_emit_kernel<<<(unsigned)l.blocks, kSplatBlock, 0, stream>>>(a, keys, vals);
    if (a.max_pairs > 0) {
        e = sort_pairs16_launch(a.pairs, a.max_pairs, reinterpret_cast<const uint32_t*>(a.scratch) + 3, sm_count, stream);
        if (e != cudaSuccess) return e;
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((a.max_pairs + 255) / 256, 8ull * sm_count));
        depth_ranges_kernel<<<grid, 256, 0, stream>>>(a, keys);
    }
    depth_tile_kernel<<<(unsigned)l.tiles, kSplatThreads, 0, stream>>>(a, vals);
    return cudaGetLastError();
}

}  // namespace m2s
