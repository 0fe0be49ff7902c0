/* m2s_ply_oracle.c — plain-C restatement of parsers::loadPlyFile's per-vertex arithmetic (src/parsers/parsers.cpp:577-622)
 * on raw .ply vertex rows (TEST INFRASTRUCTURE: the checker of m2s_ply_decode_enqueue / m2s_ply_read at sizes no golden
 * fixture holds).  Built with gcc -ffp-contract=off: every operation is one IEEE fp32 (or fp64) rounding, as in the
 * reference compiled without contraction, and expf is glibc's, as the reference calls it.
 *
 * rows: count rows of info->row_stride bytes (no alignment); out: count x 24 floats (GaussianDataSSBO). */
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../include/m2s.h"

#define ORC_API __attribute__((visibility("default")))

static float field(const unsigned char* row, const m2s_ply_info* info, int k) {
    float v = 0.0f;
    if (info->offset[k] >= 0) memcpy(&v, row + info->offset[k], 4);
    return v;
}

ORC_API void orc_ply_load(const unsigned char* rows, const m2s_ply_info* info, uint64_t count, float* out) {
    const float kC0 = 0.28209479177387814f; /* SH_COEFF0 */
    for (uint64_t i = 0; i < count; ++i) {
        const unsigned char* r = rows + i * info->row_stride;
        float* g = out + i * 24;
        /* position (x, y, z, 1) */
        g[0] = field(r, info, M2S_PLY_X); g[1] = field(r, info, M2S_PLY_Y); g[2] = field(r, info, M2S_PLY_Z); g[3] = 1.0f;
        /* utils::getColorFromSh: sh * SH_COEFF0 + 0.5f; utils::sigmoid: 1.0 / (1.0 + std::exp(-opacity)) in double */
        for (int c = 0; c < 3; ++c) {
            const float p = field(r, info, M2S_PLY_F_DC_0 + c) * kC0;
            g[4 + c] = p + 0.5f;
        }
        g[7] = (float)(1.0 / (1.0 + (double)expf(-field(r, info, M2S_PLY_OPACITY))));
        /* glm::exp of the log scales */
        for (int c = 0; c < 3; ++c) g[8 + c] = expf(field(r, info, M2S_PLY_SCALE_0 + c));
        g[11] = 1.0f;
        if (info->has_pbr) {
            g[12] = field(r, info, M2S_PLY_NX); g[13] = field(r, info, M2S_PLY_NY); g[14] = field(r, info, M2S_PLY_NZ); g[15] = 0.0f;
            g[20] = field(r, info, M2S_PLY_METALLIC); g[21] = field(r, info, M2S_PLY_ROUGHNESS); g[22] = 0.0f; g[23] = 0.0f;
        } else {
            memset(g + 12, 0, 4 * sizeof(float));
            memset(g + 20, 0, 4 * sizeof(float));
        }
        /* glm::normalize(glm::quat(w, x, y, z)) (quaternion_geometric.inl): len = sqrt((w w + x x) + (y y + z z)),
         * identity for len <= 0, else each component times 1 / len; stored w, x, y, z */
        const float w = field(r, info, M2S_PLY_ROT_0), x = field(r, info, M2S_PLY_ROT_1), y = field(r, info, M2S_PLY_ROT_2),
                    z = field(r, info, M2S_PLY_ROT_3);
        const float ww = w * w, xx = x * x, yy = y * y, zz = z * z;
        const float a = ww + xx, b = yy + zz;
        const float len = sqrtf(a + b);
        if (len <= 0.0f) { g[16] = 1.0f; g[17] = 0.0f; g[18] = 0.0f; g[19] = 0.0f; }
        else {
            const float inv = 1.0f / len;
            g[16] = w * inv; g[17] = x * inv; g[18] = y * inv; g[19] = z * inv;
        }
    }
}
