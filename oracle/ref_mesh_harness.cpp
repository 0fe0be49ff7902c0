// ref_mesh_harness.cpp — hosts the REFERENCE's mesh render shaders on the CPU (TEST INFRASTRUCTURE).
//
// oracle/build_mesh.py rewrites meshRenderVS.glsl and meshRenderPS.glsl (+ common.glsl, spliced where the fragment shader
// includes it) into oracle/_ref/mesh{VS,PS}.inc (qualifier / literal / swizzle token rewrites only).  This file is the GL
// environment they run in: the vertex attributes, gl_Position and gl_PrimitiveID, the uniforms, and texture(), which
// returns the texel supplied for the invocation, so that the shader arithmetic is pinned apart from the sampler.  The
// exp built-in is the splat draw's (DESIGN §2); sin is the C library's sinf, as GLM calls it.  No shader arithmetic is
// restated here.
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

namespace refmvs {
using namespace glm;
static vec4 gl_Position;
#include "meshVS.inc"
}  // namespace refmvs

namespace refmps {
using namespace glm;
struct sampler2D { int unit; };
static vec4 g_texel[3];
static vec4 texture(const sampler2D& s, const vec2&) { return g_texel[s.unit]; }
static int gl_PrimitiveID;
#include "meshPS.inc"
}  // namespace refmps

// meshRenderVS.glsl for n vertices (n x 12 floats: position, normal, tangent, uv); out: gl_Position (n x 4) and the
// varyings (n x 13: v_worldPos, v_normal, v_tangent, v_uv, v_viewDepth).  Matrices column-major (glm::mat4).
REF_API void ref_mesh_vs(const float* vtx, uint32_t n, const float* world_to_view, const float* view_to_clip, const float* model_to_world,
                         float* clip, float* vary) {
    using namespace refmvs;
    std::memcpy(&u_worldToView, world_to_view, 64);
    std::memcpy(&u_viewToClip, view_to_clip, 64);
    std::memcpy(&u_modelToWorld, model_to_world, 64);
    for (uint32_t k = 0; k < n; ++k) {
        const float* p = vtx + 12 * k;
        position = glm::vec3(p[0], p[1], p[2]);
        normal = glm::vec3(p[3], p[4], p[5]);
        tangent = glm::vec4(p[6], p[7], p[8], p[9]);
        uv = glm::vec2(p[10], p[11]);
        shader_main();
        std::memcpy(clip + 4 * k, &gl_Position, 16);
        float* o = vary + 13 * k;
        std::memcpy(o, &v_worldPos, 12);
        std::memcpy(o + 3, &v_normal, 12);
        std::memcpy(o + 6, &v_tangent, 16);
        std::memcpy(o + 10, &v_uv, 8);
        o[12] = v_viewDepth;
    }
}

// meshRenderPS.glsl for one fragment: v13 the varyings, tex12 the texels texture() returns for the albedo, normal and
// metallic-roughness maps, has bit m: has*Map == 1 for map m.  out20: gPosition, gNormal, gAlbedo, gDepth,
// gMetallicRoughness.
REF_API void ref_mesh_ps(const float* v, const float* tex12, uint32_t has, const float* factor, const float* near_far, int mode,
                         int prim_id, float* out) {
    using namespace refmps;
    v_worldPos = glm::vec3(v[0], v[1], v[2]);
    v_normal = glm::vec3(v[3], v[4], v[5]);
    v_tangent = glm::vec4(v[6], v[7], v[8], v[9]);
    v_uv = glm::vec2(v[10], v[11]);
    v_viewDepth = v[12];
    for (int m = 0; m < 3; ++m) g_texel[m] = glm::vec4(tex12[4 * m], tex12[4 * m + 1], tex12[4 * m + 2], tex12[4 * m + 3]);
    albedoTexture = sampler2D{0}; normalTexture = sampler2D{1}; metallicRoughnessTexture = sampler2D{2};
    hasAlbedoMap = (int)(has & 1u); hasNormalMap = (int)((has >> 1) & 1u); hasMetallicRoughnessMap = (int)((has >> 2) & 1u);
    u_baseColorFactor = glm::vec4(factor[0], factor[1], factor[2], factor[3]);
    u_nearFar = glm::vec2(near_far[0], near_far[1]);
    u_renderMode = mode;
    gl_PrimitiveID = prim_id;
    shader_main();
    std::memcpy(out, &gPosition, 16);
    std::memcpy(out + 4, &gNormal, 16);
    std::memcpy(out + 8, &gAlbedo, 16);
    std::memcpy(out + 12, &gDepth, 16);
    std::memcpy(out + 16, &gMetallicRoughness, 16);
}
