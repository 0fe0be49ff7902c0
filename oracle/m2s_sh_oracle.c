/* m2s_sh_oracle.c — plain-C restatement of the prepass's view-dependent colour (m2s_prepass_sh; beyond the reference:
 * graphdeco's computeColorFromSH on the SH rest coefficients of a loaded .ply) (TEST INFRASTRUCTURE: the checker of
 * m2s_prepass_sh).  Built with gcc -ffp-contract=off: every operation is one IEEE fp32 rounding, in the order m2s.h states.
 *
 * orc_prepass_sh is orc_prepass (m2s_oracle.c, linked from libm2s_oracle.so) on records whose colour is the SH colour:
 * the prepass writes the record colour into the quad in render modes 0 and 6 and reads it nowhere else, so that is the
 * whole of the variant.  Records: n x 24 floats (GaussianDataSSBO); sh: n x M2S_SH_FLOATS(buffer_degree) floats,
 * coefficient-major (the r, g, b of coefficient k at 3 (k - 1) .. 3 (k - 1) + 2). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

uint32_t orc_prepass(const float* gaussians, uint32_t n, const float* world_to_view, const float* view_to_clip, const float* model_to_world,
                     const float resolution[2], const float near_far[2], float std_dev, int render_mode, uint32_t format, uint32_t ply_has_pbr,
                     float* quads, float* depths);

static uint32_t sh_floats(uint32_t d) { return d == 1 ? 12u : d == 2 ? 24u : d == 3 ? 48u : 0u; }

/* general 4x4 inverse by cofactors in fp64, column-major; 0 for a zero determinant */
static int invert4(const double m[16], double inv[16]) {
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    if (det == 0.0) return 0;
    for (int k = 0; k < 16; ++k) inv[k] /= det;
    return 1;
}

/* the camera in model space: the translation column of inverse(V M), V M and the inverse in fp64 from the fp32 matrices,
 * rounded once to fp32; 0 for a singular V M */
ORC_API int orc_sh_camera(const float* V, const float* M, float cam[3]) {
    double VM[16], inv[16];
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r)
            VM[c * 4 + r] = (((double)V[r] * M[c * 4] + (double)V[4 + r] * M[c * 4 + 1]) + (double)V[8 + r] * M[c * 4 + 2]) +
                            (double)V[12 + r] * M[c * 4 + 3];
    if (!invert4(VM, inv) || !isfinite(inv[12]) || !isfinite(inv[13]) || !isfinite(inv[14])) return 0;
    for (int k = 0; k < 3; ++k) cam[k] = (float)inv[12 + k];
    return 1;
}

/* rgb[i] = max(record colour + rest, 0) per channel (glm::max: NaN kept) for gaussian i seen from cam */
ORC_API void orc_sh_colours(const float* gaussians, uint32_t n, const float* sh, uint32_t buffer_degree, uint32_t sh_degree, const float cam[3],
                            float* rgb) {
    const float C1 = 0.4886025119029199f;
    const float C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f, 0.5462742152960396f};
    const float C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f, -0.4570457994644658f,
                         1.445305721320277f, -0.5900435899266435f};
    const uint32_t K = (sh_degree + 1) * (sh_degree + 1) - 1, stride = sh_floats(buffer_degree);
    for (uint32_t i = 0; i < n; ++i) {
        const float* g = gaussians + (size_t)i * 24;
        const float* c = sh + (size_t)i * stride;
        float rest[3] = {0.0f, 0.0f, 0.0f};
        const float dx = g[0] - cam[0], dy = g[1] - cam[1], dz = g[2] - cam[2];
        const float len = sqrtf((dx * dx + dy * dy) + dz * dz);
        if (K > 0 && len != 0.0f) {
            const float inv = 1.0f / len;
            const float x = dx * inv, y = dy * inv, z = dz * inv;
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            const float B[15] = {-C1 * y, C1 * z, -C1 * x,
                                 C2[0] * xy, C2[1] * yz, C2[2] * (2.0f * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy),
                                 C3[0] * y * (3.0f * xx - yy), C3[1] * xy * z, C3[2] * y * (4.0f * zz - xx - yy),
                                 C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy), C3[4] * x * (4.0f * zz - xx - yy), C3[5] * z * (xx - yy),
                                 C3[6] * x * (xx - 3.0f * yy)};
            for (uint32_t k = 0; k < K; ++k)
                for (int ch = 0; ch < 3; ++ch) rest[ch] = rest[ch] + B[k] * c[3 * k + ch];
        }
        for (int ch = 0; ch < 3; ++ch) {
            const float v = g[4 + ch] + rest[ch];
            rgb[(size_t)i * 3 + ch] = v < 0.0f ? 0.0f : v;
        }
    }
}

/* orc_prepass with the SH colour; the arguments of orc_prepass plus the SH buffer, its degree and the degree evaluated.
 * UINT32_MAX for a singular V M (m2s_prepass_sh: M2S_E_INVALID). */
ORC_API uint32_t orc_prepass_sh(const float* gaussians, uint32_t n, const float* world_to_view, const float* view_to_clip,
                                const float* model_to_world, const float resolution[2], const float near_far[2], float std_dev, int render_mode,
                                uint32_t format, uint32_t ply_has_pbr, const float* sh, uint32_t buffer_degree, uint32_t sh_degree, float* quads,
                                float* depths) {
    float cam[3];
    if (!orc_sh_camera(world_to_view, model_to_world, cam)) return UINT32_MAX;
    if (sh_degree == 0 || n == 0)
        return orc_prepass(gaussians, n, world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev, render_mode, format,
                           ply_has_pbr, quads, depths);
    float* g = (float*)malloc((size_t)n * 24 * sizeof(float));
    float* rgb = (float*)malloc((size_t)n * 3 * sizeof(float));
    if (!g || !rgb) { free(g); free(rgb); return UINT32_MAX; }
    memcpy(g, gaussians, (size_t)n * 24 * sizeof(float));
    orc_sh_colours(gaussians, n, sh, buffer_degree, sh_degree, cam, rgb);
    for (uint32_t i = 0; i < n; ++i) memcpy(g + (size_t)i * 24 + 4, rgb + (size_t)i * 3, 3 * sizeof(float));
    const uint32_t valid = orc_prepass(g, n, world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev, render_mode, format,
                                       ply_has_pbr, quads, depths);
    free(g);
    free(rgb);
    return valid;
}
