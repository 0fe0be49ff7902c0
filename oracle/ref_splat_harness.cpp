// ref_splat_harness.cpp — hosts the REFERENCE's splat vertex and fragment shaders on the CPU (TEST INFRASTRUCTURE).
//
// oracle/build_splat.py rewrites gaussianSplattingVS.glsl and gaussianSplattingPS.glsl (qualifier / literal / swizzle
// token rewrites only) into oracle/_ref/splat{VS,PS}.inc.  This file is the GL environment they run in, as DESIGN §2
// fixes it: the instanced draw of GaussianSplattingPass::execute (two triangles per instance, in order), the viewport
// transform and 1/256-pixel snap, edge functions with the top-left rule, one fragment per covered pixel centre, the
// blend functions, the RGBA16F / RGBA8 targets and the exp built-in.  No shader arithmetic is restated here.
#define GLM_FORCE_SWIZZLE
#include <cmath>
#include <cstdint>
#include <cstring>
#include <glm/glm.hpp>

#define REF_API extern "C" __attribute__((visibility("default")))

static float bitsf(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

// the exp built-in (DESIGN §2): round-to-nearest fp32 operations only
static float glsl_exp(float x) {
    if (x != x) return x;
    if (x > 88.72283905206835f) return bitsf(0x7f800000u);
    if (x < -103.97208f) return 0.0f;
    const float fk = std::rint(x * 1.44269504088896341f);
    float r = x - fk * 0.693359375f;
    r = r - fk * -2.12194440e-4f;
    const float z = r * r;
    float p = 1.9875691500e-4f;
    p = p * r + 1.3981999507e-3f;
    p = p * r + 8.3334519073e-3f;
    p = p * r + 4.1665795894e-2f;
    p = p * r + 1.6666665459e-1f;
    p = p * r + 5.0000001201e-1f;
    p = p * z + r + 1.0f;
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return p * bitsf((uint32_t)(k1 + 127) << 23) * bitsf((uint32_t)(k2 + 127) << 23);
}

namespace refvs {
using namespace glm;
static vec4 gl_Position;
#include "splatVS.inc"
}  // namespace refvs
namespace refps {
using namespace glm;
static vec4 gl_FragCoord;
#include "splatPS.inc"
}  // namespace refps

// one vertex (GaussianSplattingPass.cpp:10-20: V0..V3 = (-1,-1), (-1,1), (1,1), (1,-1)); out: gl_Position.xy + 18 varyings
REF_API void ref_splat_vs(const float* q, int vertex, float width, float height, float* out) {
    using namespace refvs;
    static const float V[4][2] = {{-1, -1}, {-1, 1}, {1, 1}, {1, -1}};
    vertexPos = glm::vec4(V[vertex & 3][0], V[vertex & 3][1], 0.0f, 1.0f);
    std::memcpy(&gaussianMean2Ndc, q + 0, 16); std::memcpy(&quadScaleNdc, q + 4, 16); std::memcpy(&color, q + 8, 16);
    std::memcpy(&conic, q + 12, 16); std::memcpy(&normal, q + 16, 16); std::memcpy(&gaussianWsPos, q + 20, 16);
    u_resolution = glm::vec2(width, height);
    shader_main();
    const float v[20] = {gl_Position.x, gl_Position.y, out_screen.x, out_screen.y, out_conic.x, out_conic.y, out_conic.z,
                         out_color.x, out_color.y, out_color.z, out_opacity, out_normal.x, out_normal.y, out_normal.z,
                         out_wsPos.x, out_wsPos.y, out_wsPos.z, out_depth, metallicRoughness.x, metallicRoughness.y};
    std::memcpy(out, v, sizeof(v));
}

// one fragment; var: the 18 varyings in ref_splat_vs order; out: the five outputs, 4 floats each
REF_API void ref_splat_fs(const float* v, float fx, float fy, int mode, float* out) {
    using namespace refps;
    out_screen = glm::vec2(v[0], v[1]); out_conic = glm::vec3(v[2], v[3], v[4]); out_color = glm::vec3(v[5], v[6], v[7]);
    out_opacity = v[8]; out_normal = glm::vec3(v[9], v[10], v[11]); out_wsPos = glm::vec3(v[12], v[13], v[14]);
    out_depth = v[15]; metallicRoughness = glm::vec2(v[16], v[17]);
    gl_FragCoord = glm::vec4(fx, fy, 0.0f, 1.0f);
    u_renderMode = mode;
    shader_main();
    const glm::vec4* o[5] = {&gPosition, &gNormal, &gAlbedo, &gDepth, &gMetallicRoughness};
    for (int t = 0; t < 5; ++t) std::memcpy(out + 4 * t, o[t], 16);
}

// ---- the fixed-function environment --------------------------------------------------------------------------------
static uint16_t to_half(float f) {   // RGBA16F store: round to nearest even (the compiler's _Float16), NaN -> 0x7FFF
    if (f != f) return 0x7fffu;
    _Float16 h = (_Float16)f;
    uint16_t b; std::memcpy(&b, &h, 2); return b;
}
static float from_half(uint16_t b) { _Float16 h; std::memcpy(&h, &b, 2); return (float)h; }
static float clamp01(float v) { return std::fmin(std::fmax(v, 0.0f), 1.0f); }

REF_API void ref_splat_draw(const float* quads, uint32_t n, uint32_t W, uint32_t H, int mode, uint16_t* pos, uint16_t* nrm,
                            uint8_t* alb, uint16_t* dep, uint8_t* mr) {
    uint16_t* f16[5] = {pos, nrm, nullptr, dep, nullptr};
    uint8_t* u8[5] = {nullptr, nullptr, alb, nullptr, mr};
    for (int t = 0; t < 5; ++t) {   // glClearColor(0, 0, 0, 0) + glClear
        if (f16[t]) std::memset(f16[t], 0, (size_t)W * H * 8);
        if (u8[t]) std::memset(u8[t], 0, (size_t)W * H * 4);
    }
    static const int tris[2][3] = {{0, 1, 2}, {0, 2, 3}};   // quadIndices
    for (uint32_t i = 0; i < n; ++i) {                      // instances in buffer order
        float vo[4][20];
        int64_t X[4], Y[4];
        bool ok[4];
        for (int v = 0; v < 4; ++v) {
            ref_splat_vs(quads + (size_t)i * 24, v, (float)W, (float)H, vo[v]);
            const float xw = vo[v][0] * ((float)W * 0.5f) + (float)W * 0.5f, yw = vo[v][1] * ((float)H * 0.5f) + (float)H * 0.5f;
            ok[v] = std::isfinite(xw) && std::isfinite(yw) && std::fabs(xw) <= 8192.0f && std::fabs(yw) <= 8192.0f;
            X[v] = ok[v] ? (int64_t)std::lrint(xw * 256.0f) : 0;
            Y[v] = ok[v] ? (int64_t)std::lrint(yw * 256.0f) : 0;
        }
        for (const auto& t : tris) {
            if (!ok[t[0]] || !ok[t[1]] || !ok[t[2]]) continue;
            const int64_t x0 = X[t[0]], y0 = Y[t[0]], x1 = X[t[1]], y1 = Y[t[1]], x2 = X[t[2]], y2 = Y[t[2]];
            const int64_t area = (x1 - x0) * (y2 - y0) - (x2 - x0) * (y1 - y0);
            if (area == 0) continue;
            const int64_t ex[3][2] = {{x1, y1}, {x2, y2}, {x0, y0}}, ey[3][2] = {{x2, y2}, {x0, y0}, {x1, y1}};
            for (int64_t py = 0; py < H; ++py)
                for (int64_t px = 0; px < W; ++px) {
                    const int64_t cx = px * 256 + 128, cy = py * 256 + 128;   // pixel centre, 1/256 units
                    bool in = true;
                    for (int k = 0; k < 3 && in; ++k) {
                        // edge from a to b, oriented so that the interior is positive; top-left ownership on zero
                        const int64_t ax = ex[k][0], ay = ex[k][1], bx = ey[k][0], by = ey[k][1];
                        const int64_t s = area > 0 ? 1 : -1;
                        const int64_t e = s * ((bx - ax) * (cy - ay) - (by - ay) * (cx - ax));
                        const int64_t a = s * (ay - by), b = s * (bx - ax);
                        in = e > 0 || (e == 0 && (a > 0 || (a == 0 && b > 0)));
                    }
                    if (!in) continue;
                    float o[20];
                    ref_splat_fs(vo[t[0]] + 2, (float)px + 0.5f, (float)py + 0.5f, mode, o);
                    const size_t p = ((size_t)py * W + px) * 4;
                    for (int tg = 0; tg < 5; ++tg) {
                        const float* src = o + 4 * tg;
                        if (f16[tg]) {   // GL_ONE_MINUS_DST_ALPHA, GL_ONE (GL_ONE, GL_ONE in mode 4), fp32, one rounding to half
                            uint16_t* d = f16[tg] + p;
                            const float f = mode == 4 ? 1.0f : 1.0f - from_half(d[3]);
                            for (int c = 0; c < 4; ++c) d[c] = to_half(src[c] * f + from_half(d[c]));
                        } else if (u8[tg]) {   // normalised fixed point: clamped, stored as round-half-even(x * 255)
                            uint8_t* d = u8[tg] + p;
                            const float f = mode == 4 ? 1.0f : clamp01(1.0f - (float)d[3] / 255.0f);
                            for (int c = 0; c < 4; ++c)
                                d[c] = (uint8_t)std::nearbyint(clamp01(clamp01(src[c]) * f + (float)d[c] / 255.0f) * 255.0f);
                        }
                    }
                }
        }
    }
}
