// Host check of box_mask() (mesh2splat_b200/csrc/m2s_span.cuh), the raster kernel's coverage walk of small triangles,
// against the per-pixel rule: bit row * w + column set <=> all three E'_k >= 0 at that pixel.  Two sources of boxes:
// triangles set up exactly as raster_kernel does (24.8 fixed point, sign-normalised edge functions, top-left ownership,
// candidate box) whose boxes pass the kernel's small test, and every box shape w x h <= 64 pixels (h <= 32) with random
// edge coefficients.  Each box is walked with maxc = n and with a larger lock-step count, as a warp's other lanes make it.
// Built and run by tests/test_box_mask_host.py (g++).
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <algorithm>
#include "../mesh2splat_b200/csrc/m2s_span.cuh"

static uint64_t rng_state = 0x2545F4914F6CDD1Dull;
static uint64_t rnd() { rng_state ^= rng_state << 13; rng_state ^= rng_state >> 7; rng_state ^= rng_state << 17; return rng_state; }
static long long rnd_range(long long lo, long long hi) { return lo + (long long)(rnd() % (uint64_t)(hi - lo + 1)); }

static unsigned long long brute(const long long E[3], const int A[3], const int B[3], int w, int h) {
    unsigned long long m = 0;
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            bool in = true;
            for (int k = 0; k < 3; ++k) in = in && E[k] + (long long)A[k] * x + (long long)B[k] * y >= 0;
            if (in) m |= 1ull << (y * w + x);
        }
    return m;
}

// the kernel's small test: box <= 64 pixels, <= 32 rows, every |E'| over the box below 2^31
static bool small_box(const long long E[3], const int A[3], const int B[3], int w, int h) {
    if (w * h > 64 || h > 32) return false;
    for (int k = 0; k < 3; ++k)
        if (std::llabs(E[k]) + (long long)(w - 1) * std::abs(A[k]) + (long long)(h - 1) * std::abs(B[k]) >= 0x7fffffffll) return false;
    return true;
}

static long checked = 0;
static bool check(const long long E[3], const int A[3], const int B[3], int w, int h, const char* what, long c) {
    const unsigned long long want = brute(E, A, B, w, h);
    const uint32_t n = (uint32_t)(w * h);
    const uint32_t extra[3] = {n, n + (uint32_t)rnd_range(0, 64 - n), 64u};
    for (uint32_t maxc : extra) {
        const unsigned long long got = m2s::box_mask((int)E[0], (int)E[1], (int)E[2], A[0], A[1], A[2], B[0], B[1], B[2], w, n, maxc);
        if (got != want) {
            printf("MISMATCH %s case %ld w %d h %d maxc %u: mask %016llx want %016llx\n", what, c, w, h, maxc, got, want);
            return false;
        }
        ++checked;
    }
    // a lane without a small triangle walks with n = 0 and must leave no bit
    if (m2s::box_mask((int)E[0], (int)E[1], (int)E[2], A[0], A[1], A[2], B[0], B[1], B[2], w, 0u, 64u) != 0ull) {
        printf("MISMATCH %s case %ld: n = 0 left bits\n", what, c);
        return false;
    }
    return true;
}

int main(int argc, char** argv) {
    const long cases = argc > 1 ? atol(argv[1]) : 200000;
    long tris = 0, shapes = 0;
    // 1. triangles as raster_kernel sets them up (the generators of span_harness.cpp, scaled to small boxes)
    for (long c = 0; c < cases; ++c) {
        const int R = (c % 3 == 0) ? 4096 : (c % 3 == 1 ? 512 : 97);
        int X[3], Y[3];
        const int mode = (int)(rnd() % 5);
        const int cx = (int)rnd_range(0, R * 256), cy = (int)rnd_range(0, R * 256);
        for (int k = 0; k < 3; ++k) {
            if (mode == 0) { X[k] = cx + (int)rnd_range(-600, 600); Y[k] = cy + (int)rnd_range(-600, 600); }                     // small
            else if (mode == 1) { X[k] = cx + (int)rnd_range(-2400, 2400); Y[k] = cy + (int)rnd_range(-1200, 1200); }          // up to the box limit
            else if (mode == 2) { X[k] = cx + (int)rnd_range(-16000, 16000); Y[k] = cy + (int)rnd_range(-60, 60); }            // flat sliver
            else if (mode == 3) { X[k] = ((cx + (int)rnd_range(-1200, 1200)) & ~255) | 128; Y[k] = ((cy + (int)rnd_range(-1200, 1200)) & ~255) | 128; }  // ties
            else { X[k] = cx + (int)rnd_range(-60, 60); Y[k] = cy + (int)rnd_range(-8000, 8000); }                             // tall sliver
        }
        const long long area2 = (long long)(X[1] - X[0]) * (Y[2] - Y[0]) - (long long)(X[2] - X[0]) * (Y[1] - Y[0]);
        if (area2 == 0) continue;
        const int sg = area2 < 0 ? -1 : 1;
        long long C[3]; int A[3], B[3]; unsigned incl = 0;
        for (int k = 0; k < 3; ++k) {
            const int va = (k + 1) % 3, vb = (k + 2) % 3;
            const int dx = X[vb] - X[va], dy = Y[vb] - Y[va];
            A[k] = sg * (-dy * 256); B[k] = sg * (dx * 256);
            C[k] = (long long)sg * ((long long)dx * (128 - Y[va]) - (long long)dy * (128 - X[va]));
            if (A[k] > 0 || (A[k] == 0 && B[k] > 0)) incl |= 1u << k;
        }
        const int xmin = std::min(X[0], std::min(X[1], X[2])), xmax = std::max(X[0], std::max(X[1], X[2]));
        const int ymin = std::min(Y[0], std::min(Y[1], Y[2])), ymax = std::max(Y[0], std::max(Y[1], Y[2]));
        const int x0 = std::max(0, (xmin + 127) >> 8), x1 = std::min(R - 1, (xmax - 128) >> 8);
        const int y0 = std::max(0, (ymin + 127) >> 8), y1 = std::min(R - 1, (ymax - 128) >> 8);
        if (x1 < x0 || y1 < y0) continue;
        const int w = x1 - x0 + 1, h = y1 - y0 + 1;
        long long E[3];
        for (int k = 0; k < 3; ++k) E[k] = C[k] + (long long)A[k] * x0 + (long long)B[k] * y0 - ((incl >> k) & 1 ? 0 : 1);
        if (!small_box(E, A, B, w, h)) continue;
        ++tris;
        if (!check(E, A, B, w, h, "triangle", c)) return 1;
    }
    // 2. every box shape up to the small-triangle limits, random edge coefficients (half-planes in any direction)
    for (int w = 1; w <= 64; ++w)
        for (int h = 1; h <= 32 && w * h <= 64; ++h)
            for (int rep = 0; rep < 400; ++rep) {
                long long E[3]; int A[3], B[3];
                const int mag = rep % 4 == 0 ? 300 : 1 << 20;
                for (int k = 0; k < 3; ++k) {
                    A[k] = (int)rnd_range(-mag, mag); B[k] = (int)rnd_range(-mag, mag);
                    E[k] = rnd_range(-(long long)mag * 40, (long long)mag * 40);
                    if (rep % 8 == 1) A[k] = 0;   // axis-aligned edges and exact zeros
                    if (rep % 8 == 2) B[k] = 0;
                }
                if (!small_box(E, A, B, w, h)) continue;
                ++shapes;
                if (!check(E, A, B, w, h, "shape", rep)) return 1;
            }
    printf("ok %ld triangles %ld boxes %ld walks\n", tris, shapes, checked);
    return 0;
}
