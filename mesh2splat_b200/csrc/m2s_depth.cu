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
#include "m2s_clip.cuh"
#include "m2s_depth.cuh"

namespace m2s {

namespace {
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

// clip-space polygon of source triangle `tri` (m2s_clip.cuh); returns its vertex count (0: not drawn)
__device__ int depth_poly(const DepthArgs& a, uint32_t tri, float4 (&v)[kDepthMaxPoly]) {
    if (!depth_opaque(a, tri)) return 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 p = __ldg(a.tris + (size_t)tri * 9 + k * 3);
        v[k] = make_float4(clip_row(a.pvm, 0, p.x, p.y, p.z, 1.0f), clip_row(a.pvm, 1, p.x, p.y, p.z, 1.0f),
                           clip_row(a.pvm, 2, p.x, p.y, p.z, 1.0f), clip_row(a.pvm, 3, p.x, p.y, p.z, 1.0f));
    }
    return clip_poly(v);
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
        const int tx = clip_tiles_x(a.width);
        uint32_t cnt = 0;
        for (int k = 0; k + 2 < np; ++k) {
            DepthTri d;
            clip_fan<false>(v, k, a.width, a.height, d);
            cnt += clip_for_each_tile(d.t, tx, [&](uint32_t, uint32_t tile) { f(tile, i << 3 | (uint32_t)k); });
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
    clip_fan<false>(poly, (int)(v & 7u), a.width, a.height, d);
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
    const uint32_t tile = blockIdx.x, tx = (uint32_t)clip_tiles_x(a.width);
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
