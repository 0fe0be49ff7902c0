// ref_depth_harness.cpp — hosts the REFERENCE's mesh depth pre-pass shaders and its viewer prepass with the mesh depth
// test on the CPU (TEST INFRASTRUCTURE).
//
// oracle/build_depth.py rewrites depthPrepassVS.glsl, depthPrepassPS.glsl and gaussianSplattingPrepassCS.glsl
// (+ common.glsl) into oracle/_ref/depth{VS,PS,PrepassCS}.inc (qualifier / literal / swizzle token rewrites only).  This
// file is the GL environment they run in: the vertex attribute and gl_Position, gl_FragCoord, the SSBOs, the atomic
// counter, the invocation id, and the depth texture bound to u_depthTexture — an unsized GL_DEPTH_COMPONENT texture
// sampled NEAREST with CLAMP_TO_EDGE as DESIGN §2 fixes it (texel i = clamp(floor(u W), 0, W - 1) with u W in fp32, a
// NaN coordinate reading texel 0).  u_depthTestMesh is 1.  No shader arithmetic is restated here.
#define GLM_FORCE_SWIZZLE
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <glm/glm.hpp>

#define REF_API extern "C" __attribute__((visibility("default")))

namespace refdvs {
using namespace glm;
static vec4 gl_Position;
#include "depthVS.inc"
}  // namespace refdvs
namespace refdps {
using namespace glm;
static vec4 gl_FragCoord;
#include "depthPS.inc"
}  // namespace refdps

namespace refdcs {
using namespace glm;
typedef unsigned int atomic_uint;
typedef unsigned int uint;
struct sampler2D { int unit; };
static const float* g_map = nullptr;
static uint32_t g_w = 1, g_h = 1;
static vec4 texture(const sampler2D&, const vec2& uv) {
    const float fi = std::fmin(std::fmax(std::floor(uv.x * (float)g_w), 0.0f), (float)(g_w - 1));
    const float fj = std::fmin(std::fmax(std::floor(uv.y * (float)g_h), 0.0f), (float)(g_h - 1));
    return vec4(g_map[(size_t)fj * g_w + (size_t)fi]);   // the depth texture's .r (and the rest, unused)
}
static uint atomicCounterIncrement(atomic_uint& c) { return c++; }
static uvec3 gl_NumWorkGroups, gl_WorkGroupSize(16, 16, 1), gl_GlobalInvocationID;
#include "depthPrepassCS.inc"
}  // namespace refdcs

// depthPrepassVS.glsl for n vertices (positions n x 3); out: gl_Position, n x 4.  Matrices column-major (glm::mat4).
REF_API void ref_depth_vs(const float* pos, uint32_t n, const float* world_to_view, const float* view_to_clip, const float* model_to_world,
                          float* out) {
    using namespace refdvs;
    std::memcpy(&u_worldToView, world_to_view, 64);
    std::memcpy(&u_viewToClip, view_to_clip, 64);
    std::memcpy(&u_modelToWorld, model_to_world, 64);
    for (uint32_t k = 0; k < n; ++k) {
        position = glm::vec3(pos[3 * k], pos[3 * k + 1], pos[3 * k + 2]);
        shader_main();
        std::memcpy(out + 4 * k, &gl_Position, 16);
    }
}

// depthPrepassPS.glsl: the colour it writes for a fragment of window depth z (the depth buffer itself takes z)
REF_API float ref_depth_ps(float z) {
    using namespace refdps;
    gl_FragCoord = glm::vec4(0.5f, 0.5f, z, 1.0f);
    shader_main();
    return fragmentdepth;
}

// the prepass with the mesh depth test, as ref_prepass (ref_prepass_harness.cpp) with u_depthTestMesh = 1 and the map
// (width x height floats, row 0 = window y 0) bound as u_depthTexture.  depth_test = 0 runs it with u_depthTestMesh = 0.
REF_API uint32_t ref_depth_prepass(const float* gaussians, uint32_t n, const float* world_to_view, const float* view_to_clip,
                                   const float* model_to_world, const float* resolution, const float* near_far, float std_dev,
                                   int render_mode, uint32_t format, const float* map, uint32_t width, uint32_t height,
                                   uint32_t depth_test, float* quads, float* depths) {
    using namespace refdcs;
    std::memcpy(&u_worldToView, world_to_view, 64);
    std::memcpy(&u_viewToClip, view_to_clip, 64);
    std::memcpy(&u_modelToWorld, model_to_world, 64);
    u_resolution = glm::vec2(resolution[0], resolution[1]);
    u_nearFar = glm::vec2(near_far[0], near_far[1]);
    u_stdDev = std_dev; u_renderMode = render_mode; u_format = format; u_plyHasPbr = 0; u_depthTestMesh = depth_test ? 1u : 0u;
    u_gaussianCount = (int)n;
    g_map = map; g_w = width; g_h = height;
    gaussianBuffer.gaussians = reinterpret_cast<GaussianVertex*>(const_cast<float*>(gaussians));
    perQuadTransformations.ndcTransformations = reinterpret_cast<QuadNdcTransformation*>(quads);
    gaussianDepthPostFiltering.depths_vs = depths;
    g_validCounter = 0;
    const unsigned groups_needed = (n + 255u) / 256u;
    const unsigned gx = (unsigned)std::ceil(std::sqrt((float)groups_needed));
    const unsigned gy = gx ? (unsigned)((groups_needed + gx - 1) / std::max(float(gx), 1.0f)) : 0u;
    gl_NumWorkGroups = glm::uvec3(gx, gy, 1);
    const unsigned w = gx * 16u;
    for (unsigned y = 0; y < gy * 16u; ++y)
        for (unsigned x = 0; x < w; ++x) {
            gl_GlobalInvocationID = glm::uvec3(x, y, 0);
            prepass_main();
        }
    return g_validCounter;
}

// per gaussian: 1 if the prepass with the test keeps it, run one gaussian at a time (what survives the frustum cull and
// the test); survived_cull[k]: 1 if it survives with the test off
REF_API void ref_depth_keep(const float* gaussians, uint32_t n, const float* world_to_view, const float* view_to_clip,
                            const float* model_to_world, const float* resolution, const float* near_far, float std_dev, uint32_t format,
                            const float* map, uint32_t width, uint32_t height, uint8_t* kept, uint8_t* survived_cull) {
    float q[24], d;
    for (uint32_t k = 0; k < n; ++k) {
        kept[k] = (uint8_t)ref_depth_prepass(gaussians + 24 * (size_t)k, 1, world_to_view, view_to_clip, model_to_world, resolution, near_far,
                                             std_dev, 0, format, map, width, height, 1, q, &d);
        survived_cull[k] = (uint8_t)ref_depth_prepass(gaussians + 24 * (size_t)k, 1, world_to_view, view_to_clip, model_to_world, resolution,
                                                      near_far, std_dev, 0, format, map, width, height, 0, q, &d);
    }
}
