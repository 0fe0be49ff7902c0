// m2s_device.cuh — device-side data layout shared by the kernels and the C-ABI host code.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

constexpr int kMaxPeers = 8;             // GPUs of one NVSwitch domain
constexpr int kMaxLevels = 5;            // levels 0..4 (GL_TEXTURE_MAX_LEVEL 4, glUtils.cpp:313)
constexpr int kUnitTris = 32;            // max triangles per work unit (one lane per triangle)
constexpr int kTriBytes = 144;           // 36 floats
constexpr uint32_t kSmallCand = 64;      // <= this many candidate pixels (and <= 32 rows): coverage as a 64-bit mask
constexpr int kItemBlocks = 32;          // row blocks (<= 32 pixel rows of one triangle) per fragment work item
constexpr int kStashItems = 8;           // work items a raster warp publishes with one atomic
constexpr uint32_t kItemMaxFrags = 2048; // upper bound of ConvertArgs::item_max_frags
constexpr uint32_t kDeferUnitBlocks = 24; // a work unit whose larger triangles have more row blocks than this posts the tall ones to its CTA's help queue
constexpr uint32_t kDeferBlocks = 4;      // row blocks per help-queue entry
constexpr uint32_t kMaxSplit = 64;       // queue slots one oversized row block can take (item_max_frags >= R / 2)
constexpr unsigned long long kFragMask = (1ull << 40) - 1;  // ConvertArgs::counter: fragments | queue slots << 40
constexpr float kGuard = 8192.0f;        // window-coordinate guard band (|xw| beyond -> triangle dropped)
#ifndef M2S_DIRECT_MAX
#define M2S_DIRECT_MAX 512   // a unit whose small triangles emit at most this many fragments is shaded by the raster kernel itself (<= 1024)
#endif

// ---- raster_kernel -> fragment_kernel interface (context-owned scratch, L2-resident at the sizes of interest) ----
// The raster kernel only COUNTS: per triangle it leaves a record (TriRec, m2s_kernels.cu) holding the exact edge
// functions, the shading constants and — for small triangles — the 64-bit coverage mask of the candidate box; the
// fragment kernel enumerates the covered pixels itself (mask rows / exact row spans, m2s_span.cuh).
// Work of the fragment kernel = the queued FragItems: the small triangles of one work unit, or up to 32 row blocks of
// its larger triangles, or a fragment sub-range of one oversized row block.
struct BlockRef {               // <= 32 consecutive pixel rows of one triangle
    uint32_t prefix;            // fragments of the item before this block
    uint32_t ref;               // slot in the unit (5 bits) | first row relative to the box (12) << 5 | rows (6) << 17
};
struct FragItem {               // 288 B
    unsigned long long first;   // output index (this launch) of fragment 0 of the item
    uint32_t unit;              // work unit the blocks' triangles belong to
    uint32_t nblocks;           // bit 31: the blocks are implicit — block t = small triangle t of the unit (TriRec::first/hits)
    uint32_t frag_begin, frag_end;  // fragments [frag_begin, frag_end) of the item are this item's work
    uint32_t pad[2];
    BlockRef blocks[kItemBlocks];
};
static_assert(sizeof(FragItem) == 288, "FragItem layout");

// RGBA8 mip chain of one texture inside the texture arena (one allocation for all textures).
// Levels are pitch-linear, tightly packed, row 0 first; off[] are TEXEL offsets from the arena base.
struct DTexture {
    uint32_t off[kMaxLevels];
    uint16_t w[kMaxLevels];
    uint16_t h[kMaxLevels];
    uint32_t nlevels;  // q + 1, q = min(4, floor(log2(max(w,h))))
    uint32_t pad;
};
static_assert(sizeof(DTexture) == 48, "DTexture layout");

// One glTF primitive: the uniforms ConversionPass::conversion uploads per draw call
// (ConversionPass.cpp:77-112).
struct DPrim {
    float bmin[3];
    float bmax[3];
    float factor[4];
    int tex[3];  // albedo, normal, metallic-roughness; -1 = has*Map == 0
    int pad;
};

static_assert(sizeof(DPrim) == 56, "DPrim layout");

// sorted, disjoint triangle ranges -> primitive
struct DRange {
    uint32_t first, end, prim, pad;
};

struct ConvertArgs {
    const float4* tris;   // 9 float4 per triangle (3 x {pos3 nrm3 tan4 uv2})
    uint32_t tri_first;   // shard
    uint32_t tri_count;
    const DRange* ranges;
    uint32_t nranges;
    const DPrim* prims;
    uint32_t nprims;
    const DTexture* texs;
    const uint32_t* tex_base;  // texture arena
    uint32_t ntex;
    uint32_t R;
    uint32_t row_begin, row_end;  // pixel-row band [row_begin, row_end) of the R x R grid (whole grid: 0, R)
    float half_R;
    float mult;  // sigma / R (SceneManager.cpp:668)
    float log_sz;  // ln(1e-7 * mult): the constant third log-scale of the packed layout
    // intermediates between the two kernels (context-owned scratch, L2-resident at the sizes of interest);
    // the fragment kernel reads the vertices themselves from `tris`
    unsigned char* tri_frag;           // one TriRec per triangle of the shard
    FragItem* items;                   // [queue_cap]
    uint32_t queue_cap;
    uint32_t item_max_frags;           // a row block with more fragments is cut into items of this size (multiple of 32)
    uint32_t flush_frags;              // pending row blocks become one item once they hold this many fragments
    uint32_t* n_items_out;             // items queued by this launch (published by the raster kernel's last CTA)
    uint8_t* out;
    unsigned long long cap;
    unsigned long long* keys;          // optional
    unsigned long long* counter;       // low 40 bits: fragments generated (the reference's atomic counter), high 24 bits:
                                       // work items queued; context-owned, zero at launch, re-zeroed by the last CTA
    unsigned long long* total_out;     // receives the final count (last CTA out)
    const unsigned long long* prev_totals;  // appended launches: counts of the earlier chunks (records start after them)
    uint32_t nprev;
    unsigned long long* host_total;    // optional, mapped pinned host memory: {count, tag} written by the raster kernel's
    unsigned long long host_tag;       // last CTA so the host can size the download while the fragment kernel still runs
    // scheduling state (zero at launch, re-armed by the last CTA)
    uint32_t* sched;                   // words 128 B apart: 0 unit counter, 4 raster CTAs finished, 6 fragment CTAs finished
                                       // (fused gather)
    uint32_t unit_tris;                // triangles per work unit (<= 32), chosen by the host for balance
    uint32_t n_units;
    uint32_t direct_ok;                // the raster kernel may shade light units itself (ConvertPlan::direct_ok)
    uint32_t claim_late;               // ... and claims its next unit once the current one is done (ConvertPlan::claim_late)
    unsigned long long* trace;         // M2S_TRACE builds only: 16 per-phase sums per raster warp (TraceSlot)
    // multi-GPU fused gather (world <= 1: off).  peer_out[p] / peer_xch[p] are rank p's final buffer and
    // exchange block mapped into this process (NVLink peer memory); every rank's fragment kernel stores its
    // records into ALL final buffers at its global offset.  xch block: [kMaxPeers][4] u64 =
    // {count, count_epoch, done_epoch, pad} per source rank.
    uint32_t world, rank;
    uint8_t* peer_out[kMaxPeers];
    unsigned long long* peer_xch[kMaxPeers];
    unsigned long long epoch;
    unsigned long long gcap;           // capacity of the final buffers (records)
    uint32_t* status;                  // context status word (mapped pinned host memory): bit 0/1 = a gather wait timed out
};

// ---- launchers (m2s_kernels.cu) ----
int convert_warps_per_cta(int layout);
size_t tri_frag_bytes(int layout);
cudaError_t convert_configure(int layout, int* raster_blocks_per_sm, int* fragment_blocks_per_sm);
cudaError_t convert_launch(int layout, const ConvertArgs& args, int raster_grid, int fragment_grid, cudaStream_t stream, cudaEvent_t mid);
cudaError_t gather_wait_launch(const unsigned long long* xch, uint32_t world, unsigned long long epoch, unsigned long long gcap,
                               unsigned long long* total_global, uint32_t* status, cudaStream_t stream);
cudaError_t mip_groups_launch(uint32_t* arena, const DTexture& t, uint32_t g0, uint32_t g1, cudaStream_t stream);
cudaError_t vrange_launch(const float4* tris, uint32_t first, uint32_t count, const DRange* ranges, uint32_t nranges, const DPrim* prims,
                          uint32_t ntex, int* minmax, cudaStream_t stream);
cudaError_t vrange_publish_launch(int* minmax, uint32_t ntex, int* host, unsigned long long* host_tag, unsigned long long tag, cudaStream_t stream);
cudaError_t ply_rows_launch(const void* ref96, unsigned long long count, const unsigned long long* d_count,
                            uint32_t format, float mult, void* rows, cudaStream_t stream);

}  // namespace m2s
