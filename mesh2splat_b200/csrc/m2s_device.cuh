// m2s_device.cuh — device-side data layout shared by the kernels and the C-ABI host code.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

constexpr int kMaxPeers = 8;             // GPUs of one NVSwitch domain
constexpr int kMaxLevels = 5;            // levels 0..4 (GL_TEXTURE_MAX_LEVEL 4, glUtils.cpp:313)
constexpr int kUnitTris = 32;            // max triangles per work unit (one lane per triangle)
constexpr int kTriBytes = 144;           // 36 floats
constexpr int kSlimTriBytes = 64;        // the position/uv stream of PACKED56's raster pass: 4 float4 per triangle
constexpr uint32_t kSmallCand = 64;      // <= this many candidate pixels (and <= 32 rows): coverage as a 64-bit mask
constexpr int kItemBlocks = 32;          // row blocks (<= 32 pixel rows of one triangle) per fragment work item
constexpr int kStashItems = 8;           // work items a raster warp publishes with one atomic
constexpr uint32_t kItemMaxFrags = 2048; // upper bound of ConvertArgs::item_max_frags
constexpr uint32_t kDeferUnitBlocks = 24; // a work unit whose larger triangles have more row blocks than this posts the tall ones to its CTA's help queue
constexpr uint32_t kDeferBlocks = 4;      // row blocks per help-queue entry
constexpr uint32_t kMaxSplit = 64;       // queue slots one oversized row block can take (item_max_frags >= R / 2)
constexpr unsigned long long kFragMask = (1ull << 40) - 1;  // ConvertArgs::counter: fragments | queue slots << 40
constexpr int kSchedStride = 32;        // scheduler words live on separate 128-byte lines (m2s_ctx::d_sched)
constexpr float kGuard = 8192.0f;        // window-coordinate guard band (|xw| beyond -> triangle dropped)
// M2S_TRACE builds (scripts/trace_raster.py): the trace buffer starts with a header, then the raster warps' slots
constexpr int kTraceHeader = 32;
constexpr int kTraceWarpSlots = 32;
constexpr int kTrFragEndNs = 0;          // header word: globaltimer when the fragment kernel's last CTA ended
constexpr int kTrFragStartNs = 1;        // ... when its first CTA started, before griddepcontrol.wait (atomicMin: the reader sets it to ~0)
constexpr int kTrFragWaitNs = 2;         // ... when its first CTA left griddepcontrol.wait (atomicMin: the reader sets it to ~0)
#ifndef M2S_DIRECT_MAX
#define M2S_DIRECT_MAX 512   // a unit whose small triangles emit at most this many fragments is shaded by the raster kernel itself (<= 1024)
#endif

// ---- raster_kernel -> fragment_kernel interface (context-owned scratch, L2-resident at the sizes of interest) ----
// The raster kernel only COUNTS: per triangle it leaves a record (TriRec, m2s_shade.cuh) holding the exact edge
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
// FragItem::nblocks flags (the raster kernel's stash carries the same bits)
constexpr uint32_t kItUnit = 0x80000000u;   // item = the unit's small triangles (one implicit block per triangle)
constexpr uint32_t kItSplit = 0x40000000u;  // item = one oversized row block, cut into several queue slots
constexpr uint32_t kItMicro = 0x20000000u;  // unit item of <= 32 fragments: the block area holds the fragments themselves
                                            // (slot | x << 5 | y << 11, box-relative), one warp shades it with direct loads

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
    const float4* tris_slim;  // PACKED56 when the scene has it, else null: 4 float4 per triangle, {P0 u0} {P1 u1} {P2 u2}
                              // {v0 v1 v2 0} (m2s_dscene::d_tris_slim), what the raster kernel stages instead of `tris`
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
    uint8_t* out;
    unsigned long long cap;
    unsigned long long* keys;          // optional
    unsigned long long* counter;       // low 40 bits: fragments generated (the reference's atomic counter), high 24 bits:
                                       // work items queued; this launch's scheduler set (below), final when the fragment
                                       // kernel starts: every CTA reads its item count there
    unsigned long long* total_out;     // receives the final count (the fragment kernel's CTA 0; on single launches the
                                       // raster kernel's last CTA)
    const unsigned long long* prev_totals;  // appended launches: counts of the earlier chunks (records start after them)
    uint32_t nprev;
    unsigned long long* host_total;    // optional, mapped pinned host memory: {count, tag} written by the fragment kernel's
    unsigned long long host_tag;       // CTA 0 as it starts, so the host can size the download while the kernel still runs
    // scheduling state: two sets {unit counter, packed counter} in the context, alternated by launch (m2s_ctx::sched_parity).
    // This launch's set is zero at launch; its raster kernel zeroes the other set for the next launch as it starts: the
    // launch before, which used that set, has ended by then (stream order: the raster kernel is launched without PDL)
    uint32_t* claim;                   // this launch's unit counter (the set of `counter`)
    uint32_t* next_claim;              // the next launch's set, zeroed by this launch's raster kernel
    unsigned long long* next_counter;
    uint32_t* sched;                   // words 128 B apart (SCHED): 6 fragment CTAs finished (fused gather); SCHED 0-3 are
                                       // the two sets (m2s_ctx::d_sched)
    uint32_t unit_tris;                // triangles per work unit (<= 32), chosen by the host for balance
    uint32_t n_units;
    uint32_t direct_ok;                // the raster kernel may shade light units itself (ConvertPlan::direct_ok)
    uint32_t claim_late;               // ... and claims its next unit once the current one is done (ConvertPlan::claim_late)
    uint32_t pair_first;               // a warp's first pass sets up units 2g and 2g + 1 on its two half warps (ConvertPlan::pair_first)
    uint32_t single_launch;            // no fragment kernel follows: the raster kernel shades every unit and publishes the
                                       // count itself (ConvertPlan::single_launch)
    unsigned long long* trace;         // M2S_TRACE builds only: kTraceHeader words (kTrFrag*Ns), then kTraceWarpSlots
                                       // per raster warp (TraceSlot, m2s_raster.cu)
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

// ---- launchers ----
// m2s_raster.cu
int convert_warps_per_cta(int layout);
size_t tri_frag_bytes(int layout);
cudaError_t raster_configure(int layout, int* blocks_per_sm);
cudaError_t raster_launch(int layout, const ConvertArgs& args, int grid, cudaStream_t stream);
// m2s_fragment.cu; pdl: launched with programmatic dependent launch, overlapping the raster kernel's tail
cudaError_t fragment_configure(int layout, int* blocks_per_sm);
cudaError_t fragment_launch(int layout, const ConvertArgs& args, int grid, bool pdl, cudaStream_t stream);
cudaError_t gather_wait_launch(const unsigned long long* xch, uint32_t world, unsigned long long epoch, unsigned long long gcap,
                               unsigned long long* total_global, uint32_t* status, cudaStream_t stream);
// m2s_scene.cu
cudaError_t mip_groups_launch(uint32_t* arena, const DTexture& t, uint32_t g0, uint32_t g1, cudaStream_t stream);
// m2s_codec.cu
cudaError_t ply_rows_launch(const void* ref96, unsigned long long count, uint32_t format, float mult, void* rows, cudaStream_t stream);

}  // namespace m2s
