// m2s_sort.cuh — arguments and scratch layout of the viewer's depth sort (m2s_sort.cu), shared with the C-ABI host code
// (m2s_viewer.cu).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

constexpr int kSortThreads = 256;                              // one thread per digit in the per-digit steps
constexpr int kSortKeysPerThread = 16;
constexpr int kSortTile = kSortThreads * kSortKeysPerThread;   // 4096 keys per tile of a pass
constexpr int kSortPasses = 4;                                 // 8-bit digits
constexpr uint64_t kSortMaxCount = 1ull << 30;                 // a 30-bit count fits beside the two flag bits of a status word

// Context scratch of one sort, in 32-bit words:
//   ctrl  = digit histograms [4][256] (then, in place, the exclusive digit offsets) | tile counters [4] (one 128-byte
//           line) | status words [4][tiles][256];  zeroed by one memset per call
//   keys and values, two buffers each (the passes alternate between them), 64-byte aligned
struct SortLayout {
    uint64_t tiles;
    size_t ctrl_words;     // words the memset clears
    size_t buf_words;      // words of each key / value buffer
    size_t total_bytes;
};
inline SortLayout sort_layout(uint64_t count) {
    SortLayout l;
    l.tiles = (count + kSortTile - 1) / kSortTile;
    l.ctrl_words = kSortPasses * 256 + 32 + (size_t)kSortPasses * l.tiles * 256;
    l.ctrl_words = (l.ctrl_words + 15) & ~size_t(15);
    l.buf_words = ((size_t)count + 15) & ~size_t(15);
    l.total_bytes = (l.ctrl_words + 4 * l.buf_words) * sizeof(uint32_t);
    return l;
}

struct SortArgs {
    unsigned long long count;      // capacity: the grids are sized for it
    const uint32_t* d_count;       // optional: n = min(count, *d_count)
    const uint32_t* depth_bits;    // count floats, read as uint32 keys
    const float4* quads;           // count x 96 B
    float4* sorted;                // count x 96 B, n written
    uint32_t* order;               // n source indices (caller's buffer or scratch)
    uint32_t* draw;                // optional: DrawElementsIndirectCommand {6, n, 0, 0, 0}
    uint32_t* scratch;             // SortLayout of `count`
};

cudaError_t sort_launch(const SortArgs& args, int sm_count, cudaStream_t stream);

// The splat draw's (tile, quad) pairs: a stable sort of n = *d_n <= capacity (key < 2^16, value) pairs with the same
// histogram, scan and onesweep pass kernels, two passes (digits 0 and 1).  The pairs go in, and come out, in key and
// value buffer 1 of SortLayout(capacity) at `scratch`.
inline uint32_t* sort_pairs16_keys(uint32_t* scratch, uint64_t capacity) {
    const SortLayout l = sort_layout(capacity);
    return scratch + l.ctrl_words + 2 * l.buf_words;
}
inline uint32_t* sort_pairs16_vals(uint32_t* scratch, uint64_t capacity) {
    const SortLayout l = sort_layout(capacity);
    return scratch + l.ctrl_words + 3 * l.buf_words;
}
cudaError_t sort_pairs16_launch(uint32_t* scratch, uint64_t capacity, const uint32_t* d_n, int sm_count, cudaStream_t stream);

}  // namespace m2s
