/* m2s_compare_oracle.c — plain-C restatement of the image comparison (m2s_image_compare; beyond the reference: SSIM,
 * squared error and coverage of two RGBA8 images) (TEST INFRASTRUCTURE: the checker of m2s_image_compare).  Built with
 * gcc -ffp-contract=off: every fp32 operation is one IEEE rounding, in the order DESIGN §2 fixes, so the map equals the
 * kernel's bit for bit.  The fp64 sums are of the same per-window values in another fixed order than the kernel's. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/m2s.h"

#define ORC_API __attribute__((visibility("default")))

/* w_i = g_i / sum(g), g_i = exp(-i^2 / 4.5), i = -5..5, in fp64, rounded once to fp32 */
static const float kTap[11] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f, 0x1.b43c40p-3f, 0x1.106560p-2f,
                               0x1.b43c40p-3f, 0x1.bff0fep-4f, 0x1.26eb18p-5f, 0x1.f1fe02p-8f, 0x1.0d956cp-10f};
static const float kC1 = 0x1.a028f6p+2f, kC2 = 0x1.d42e14p+5f;

ORC_API void orc_compare_taps(float out[11]) { memcpy(out, kTap, sizeof(kTap)); }
ORC_API void orc_compare_constants(float out[2]) { out[0] = kC1; out[1] = kC2; }

/* The SSIM of one channel from its five blurred moments, in the kernel's order */
ORC_API float orc_ssim_value(float mx, float my, float exx, float eyy, float exy) {
    const float mx2 = mx * mx, my2 = my * my, mxy = mx * my;
    const float vx = exx - mx2, vy = eyy - my2, cxy = exy - mxy;
    const float num = (2.0f * mxy + kC1) * (2.0f * cxy + kC2);
    const float den = ((mx2 + my2) + kC1) * ((vx + vy) + kC2);
    return num / den;
}

/* the five quantities x, y, x x, y y, x y of channel c of pixel p */
static void quantities(const uint8_t* a, const uint8_t* b, size_t p, int c, float q[5]) {
    const float x = (float)a[4 * p + c], y = (float)b[4 * p + c];
    q[0] = x; q[1] = y; q[2] = x * x; q[3] = y * y; q[4] = x * y;
}

/* window rows [wy0, wy1): the horizontal sums of the rows they need kept in a ring of 11 rows; per window row the sums of
 * its windows in raster order (rows[wy][0..5]: ssim[3], ssim_covered[3]) */
static void window_rows(const uint8_t* a, const uint8_t* b, const uint8_t* cover_a, const uint8_t* cover_b, uint32_t w, uint32_t cover_min,
                        uint32_t wy0, uint32_t wy1, float* ring, float* map, float* planes, uint32_t nwy, double (*rows)[6], uint64_t* covered) {
    const uint32_t nwx = w - 10;
    float* hrow[11];
    for (uint32_t wy = wy0; wy < wy1; ++wy) {
        for (uint32_t y = (wy == wy0 ? wy : wy + 10); y <= wy + 10; ++y) {   /* the image rows not yet in the ring */
            float* r = ring + (size_t)(y % 11) * 15 * nwx;   /* [c][k][wx] */
            for (uint32_t wx = 0; wx < nwx; ++wx)
                for (int c = 0; c < 3; ++c) {
                    float s[5], q[5];
                    for (int i = 0; i < 11; ++i) {   /* left to right */
                        quantities(a, b, (size_t)y * w + wx + i, c, q);
                        for (int k = 0; k < 5; ++k) s[k] = i == 0 ? kTap[0] * q[k] : s[k] + kTap[i] * q[k];
                    }
                    for (int k = 0; k < 5; ++k) r[(size_t)(c * 5 + k) * nwx + wx] = s[k];
                }
        }
        for (int j = 0; j < 11; ++j) hrow[j] = ring + (size_t)((wy + j) % 11) * 15 * nwx;
        double* acc = rows[wy];
        for (int t = 0; t < 6; ++t) acc[t] = 0.0;
        for (uint32_t wx = 0; wx < nwx; ++wx) {
            const size_t centre = (size_t)(wy + 5) * w + (wx + 5);
            const int cov = (cover_a && cover_a[4 * centre + 3] >= cover_min) || (cover_b && cover_b[4 * centre + 3] >= cover_min);
            covered[wy] += cov;
            float m = 0.0f;
            for (int c = 0; c < 3; ++c) {
                float v[5];
                for (int k = 0; k < 5; ++k)
                    for (int j = 0; j < 11; ++j) {   /* bottom to top */
                        const float t = kTap[j] * hrow[j][(size_t)(c * 5 + k) * nwx + wx];
                        v[k] = j == 0 ? t : v[k] + t;
                    }
                const float s = orc_ssim_value(v[0], v[1], v[2], v[3], v[4]);
                if (planes) planes[(size_t)c * nwx * nwy + (size_t)wy * nwx + wx] = s;
                m = c == 0 ? s : m + s;
                acc[c] += (double)s;
                if (cov) acc[3 + c] += (double)s;
            }
            if (map) map[(size_t)wy * nwx + wx] = m / 3.0f;
        }
    }
}

/* a, b, cover_a, cover_b: w x h RGBA8 (covers may be NULL).  map (optional): (w - 10) (h - 10) floats; planes (optional):
 * 3 x (w - 10) (h - 10) floats, the per-channel values.  The fp64 sums: each window row in raster order, then the rows
 * bottom to top.  Returns 0, or -1 for a size or cover_min out of range (or no memory). */
ORC_API int orc_image_compare(const uint8_t* a, const uint8_t* b, const uint8_t* cover_a, const uint8_t* cover_b, uint32_t w, uint32_t h,
                              uint32_t cover_min, float* map, float* planes, m2s_compare_result* out) {
    if (w < 11 || w > 4096 || h < 11 || h > 4096 || cover_min < 1 || cover_min > 255) return -1;
    memset(out, 0, sizeof(*out));
    const uint32_t nwx = w - 10, nwy = h - 10;
    out->windows = (uint64_t)nwx * nwy;
    for (size_t p = 0; p < (size_t)w * h; ++p) {
        const int ia = cover_a && cover_a[4 * p + 3] >= cover_min, ib = cover_b && cover_b[4 * p + 3] >= cover_min;
        for (int c = 0; c < 3; ++c) {
            const int d = (int)a[4 * p + c] - (int)b[4 * p + c];
            out->sq_err[c] += (uint64_t)(d * d);
            if (ia || ib) out->sq_err_covered[c] += (uint64_t)(d * d);
        }
        out->pixels_both += ia && ib;
        out->pixels_a_only += ia && !ib;
        out->pixels_b_only += ib && !ia;
    }
    double (*rows)[6] = malloc(sizeof(double[6]) * nwy);
    uint64_t* covered = calloc(nwy, sizeof(uint64_t));
    const uint32_t band = 32, nband = (nwy + band - 1) / band;
    int fail = !rows || !covered;
    #pragma omp parallel for schedule(dynamic) reduction(|: fail)
    for (uint32_t k = 0; k < nband; ++k) {
        if (fail) continue;
        float* ring = malloc(sizeof(float) * 11 * 15 * nwx);
        if (!ring) { fail = 1; continue; }
        const uint32_t wy1 = (k + 1) * band < nwy ? (k + 1) * band : nwy;
        window_rows(a, b, cover_a, cover_b, w, cover_min, k * band, wy1, ring, map, planes, nwy, rows, covered);
        free(ring);
    }
    if (!fail)
        for (uint32_t wy = 0; wy < nwy; ++wy) {
            out->covered_windows += covered[wy];
            for (int c = 0; c < 3; ++c) {
                out->ssim[c] += rows[wy][c];
                out->ssim_covered[c] += rows[wy][3 + c];
            }
        }
    free(rows);
    free(covered);
    return fail ? -1 : 0;
}
