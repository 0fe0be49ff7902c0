// ref_light_harness.cpp — hosts the REFERENCE's shadow-pass and deferred-lighting shaders on the CPU (TEST INFRASTRUCTURE).
//
// oracle/build_light.py rewrites gaussianPointShadowMappingCS.glsl (+ common.glsl), gaussianPointLightCubeMapShadowVS.glsl,
// gaussianPointLightCubeMapShadowPS.glsl, gaussianSplattingDeferredVS.glsl and gaussianSplattingDeferredPS.glsl (qualifier,
// literal, swizzle, array-constructor and built-in-name token rewrites only) into oracle/_ref/light*.inc.  This file is the
// GL environment they run in, as DESIGN §2 fixes it: the compute dispatch of GaussianShadowPass::execute with its six
// per-face atomic counters and the face matrices from glm::lookAt / glm::perspective (as the pass builds them), the six
// instanced face draws (two triangles per instance, viewport transform, 1/256 snap, top-left rule, D24 codes, LESS), the
// full-screen pass's texel fetch, the cube sampler, the pow / exp2 / log2 built-ins and the RGBA8 store.  No shader
// arithmetic is restated here.
#define GLM_FORCE_SWIZZLE
#include <cmath>
#include <cstdint>
#include <cstring>
#include <sys/mman.h>
#include <glm/glm.hpp>
#include <glm/gtc/matrix_transform.hpp>

#define REF_API extern "C" __attribute__((visibility("default")))

static float bitsf(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static uint32_t fbits(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }

// ---- built-ins (DESIGN §2): pow = exp2(y log2 x), both from round-to-nearest fp32 operations ---------------------------
static float glsl_log2(float x) {
    if (x != x) return x;
    if (x < 0.0f) return bitsf(0x7fc00000u);
    if (x == 0.0f) return bitsf(0xff800000u);
    if (x == bitsf(0x7f800000u)) return x;
    uint32_t u = fbits(x);
    int e = 0;
    if (u < 0x00800000u) { u = fbits(x * 8388608.0f); e = -23; }
    e += (int)(u >> 23) - 127;
    float m = bitsf((u & 0x007fffffu) | 0x3f800000u);
    if (m > 1.41421356f) { m = m * 0.5f; e += 1; }
    const float f = (m - 1.0f) / (m + 1.0f), z = f * f;
    float p = 0.26230818925f;
    p = p * z + 0.32059889798f;
    p = p * z + 0.41219858311f;
    p = p * z + 0.57707801636f;
    p = p * z + 0.96179669393f;
    p = p * z + 2.88539008178f;
    return (float)e + f * p;
}
static float glsl_exp2(float t) {
    if (t != t) return t;
    if (t >= 128.0f) return bitsf(0x7f800000u);
    if (t < -150.0f) return 0.0f;
    const float fk = std::rint(t), r = t - fk;
    float p = 1.5252733804e-5f;
    p = p * r + 1.5403530393e-4f;
    p = p * r + 1.3333558146e-3f;
    p = p * r + 9.6181291076e-3f;
    p = p * r + 5.5504108665e-2f;
    p = p * r + 2.4022650696e-1f;
    p = p * r + 6.9314718056e-1f;
    p = p * r + 1.0f;
    const int k = (int)fk, k1 = k / 2, k2 = k - k1;
    return p * bitsf((uint32_t)(k1 + 127) << 23) * bitsf((uint32_t)(k2 + 127) << 23);
}
static float glsl_pow(float x, float y) { return glsl_exp2(y * glsl_log2(x)); }
static glm::vec3 glsl_pow(const glm::vec3& x, const glm::vec3& y) { return glm::vec3(glsl_pow(x.x, y.x), glsl_pow(x.y, y.y), glsl_pow(x.z, y.z)); }

// ---- samplers -----------------------------------------------------------------------------------------------------------
struct sampler2D { const void* data; int rgba8; int w, h; };   // NULL data reads as 0
struct samplerCube { const float* data; int size; };
static float half_to_float(uint16_t b) { _Float16 h; std::memcpy(&h, &b, 2); return (float)h; }
// the full-screen fetch: fragUV is the texel centre, so LINEAR filtering returns that texel
static glm::vec4 glsl_texture(const sampler2D& s, const glm::vec2& uv) {
    if (!s.data) return glm::vec4(0.0f);
    const int x = std::min(std::max((int)std::floor(uv.x * (float)s.w), 0), s.w - 1);
    const int y = std::min(std::max((int)std::floor(uv.y * (float)s.h), 0), s.h - 1);
    const size_t i = ((size_t)y * s.w + x) * 4;
    float c[4];
    for (int k = 0; k < 4; ++k)
        c[k] = s.rgba8 ? (float)static_cast<const uint8_t*>(s.data)[i + k] / 255.0f : half_to_float(static_cast<const uint16_t*>(s.data)[i + k]);
    return glm::vec4(c[0], c[1], c[2], c[3]);
}
// GL 4.6 §8.13 table 8.19; the major axis as DESIGN §2 fixes it (x before y before z on ties, NaN falls through to z,
// sign from "> 0"); NEAREST, CLAMP_TO_EDGE; faces +X -X +Y -Y +Z -Z; row 0 = window y 0 of the face's draw
static glm::vec4 glsl_texture(const samplerCube& c, const glm::vec3& r) {
    const float ax = std::fabs(r.x), ay = std::fabs(r.y), az = std::fabs(r.z);
    int face;
    float sc, tc, ma;
    if (ax >= ay && ax >= az) {
        ma = r.x;
        if (r.x > 0.0f) { face = 0; sc = -r.z; tc = -r.y; } else { face = 1; sc = r.z; tc = -r.y; }
    } else if (ay >= ax && ay >= az) {
        ma = r.y;
        if (r.y > 0.0f) { face = 2; sc = r.x; tc = r.z; } else { face = 3; sc = r.x; tc = -r.z; }
    } else {
        ma = r.z;
        if (r.z > 0.0f) { face = 4; sc = r.x; tc = -r.y; } else { face = 5; sc = -r.x; tc = -r.y; }
    }
    const float s = (sc / std::fabs(ma) + 1.0f) * 0.5f, t = (tc / std::fabs(ma) + 1.0f) * 0.5f;
    auto texel = [&](float v) {
        const float f = std::floor(v * (float)c.size);
        if (f != f || f < 0.0f) return 0;
        return f > (float)(c.size - 1) ? c.size - 1 : (int)f;
    };
    return glm::vec4(c.data[((size_t)face * c.size + texel(t)) * c.size + texel(s)]);
}

// ---- the shaders --------------------------------------------------------------------------------------------------------
namespace lightcs {
using namespace glm;
typedef unsigned int uint;
static uint atomicAdd(uint& c, uint v) { const uint o = c; c += v; return o; }
static uvec3 gl_NumWorkGroups, gl_WorkGroupSize(16, 16, 1), gl_GlobalInvocationID;
#include "lightCS.inc"
}  // namespace lightcs
namespace cubevs {
using namespace glm;
static vec4 gl_Position;
#include "lightCubeVS.inc"
}  // namespace cubevs
namespace cubeps {
using namespace glm;
static float gl_FragDepth;
#include "lightCubePS.inc"
}  // namespace cubeps
namespace defvs {
using namespace glm;
static vec4 gl_Position;
#include "lightDeferredVS.inc"
}  // namespace defvs
namespace defps {
using namespace glm;
using ::glsl_pow;
using ::glsl_texture;
using ::sampler2D;
using ::samplerCube;
#include "lightDeferredPS.inc"
}  // namespace defps

// include/m2s.h m2s_shadow_params / m2s_light_params, field for field
struct ShadowParams {
    float model_to_world[16], light_position[3], near_far[2], resolution[2], std_dev;
    uint32_t layout, size;
};
struct LightParams {
    uint32_t width, height, render_mode;
    float light_position[3], light_color[3], light_intensity, cam_pos[3], far_plane;
    uint32_t shadow_size;
};

static constexpr size_t kPerFace = 7000000;   // MAX_GAUSSIANS_PER_FACE, the stride of the unified buffer
static lightcs::QuadNdcTransformation* g_buckets = nullptr;

// GaussianShadowPass::execute (:85-146): uniforms, then the dispatch; per invocation, the face whose counter moved
static void dispatch(const float* gaussians, uint32_t n, const ShadowParams& p, uint32_t format, int32_t* face_of, uint32_t* index_of) {
    using namespace lightcs;
    if (!g_buckets)
        g_buckets = static_cast<QuadNdcTransformation*>(mmap(nullptr, 6 * kPerFace * sizeof(QuadNdcTransformation), PROT_READ | PROT_WRITE,
                                                             MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0));
    const glm::vec3 L(p.light_position[0], p.light_position[1], p.light_position[2]);
    u_worldToViews[0] = glm::lookAt(L, L + glm::vec3(1.0, 0.0, 0.0), glm::vec3(0.0, -1.0, 0.0));
    u_worldToViews[1] = glm::lookAt(L, L + glm::vec3(-1.0, 0.0, 0.0), glm::vec3(0.0, -1.0, 0.0));
    u_worldToViews[2] = glm::lookAt(L, L + glm::vec3(0.0, 1.0, 0.0), glm::vec3(0.0, 0.0, 1.0));
    u_worldToViews[3] = glm::lookAt(L, L + glm::vec3(0.0, -1.0, 0.0), glm::vec3(0.0, 0.0, -1.0));
    u_worldToViews[4] = glm::lookAt(L, L + glm::vec3(0.0, 0.0, 1.0), glm::vec3(0.0, -1.0, 0.0));
    u_worldToViews[5] = glm::lookAt(L, L + glm::vec3(0.0, 0.0, -1.0), glm::vec3(0.0, -1.0, 0.0));
    u_viewToClip = glm::perspective(glm::radians(90.0f), 1.0f, p.near_far[0], p.near_far[1]);
    u_stdDev = p.std_dev;
    u_resolution = glm::vec2(p.resolution[0], p.resolution[1]);
    u_renderMode = 6;
    u_format = format;
    std::memcpy(&u_modelToWorld, p.model_to_world, 64);
    u_gaussianCount = (int)n;
    u_lightPos = L;
    u_nearFar = glm::vec2(p.near_far[0], p.near_far[1]);
    for (auto& c : cmds) c = DrawElementsIndirectCommand{6, 0, 0, 0, 0};
    gaussianBuffer.gaussians = reinterpret_cast<GaussianVertex*>(const_cast<float*>(gaussians));
    perQuadTransformations.ndcTransformations = g_buckets;
    const unsigned groups = (n + 255u) / 256u;
    const unsigned gx = (unsigned)std::ceil(std::sqrt((float)groups)), gy = gx ? (groups + gx - 1) / gx : 0u;
    gl_NumWorkGroups = glm::uvec3(gx, gy, 1);
    for (unsigned y = 0; y < gy * 16u; ++y)
        for (unsigned x = 0; x < gx * 16u; ++x) {
            uint before[6];
            for (int f = 0; f < 6; ++f) before[f] = cmds[f].instanceCount;
            gl_GlobalInvocationID = glm::uvec3(x, y, 0);
            main_cs();
            const uint32_t gid = y * gx * 16u + x;
            if (gid >= n) continue;
            face_of[gid] = -1;
            for (int f = 0; f < 6; ++f)
                if (cmds[f].instanceCount != before[f]) { face_of[gid] = f; index_of[gid] = before[f]; }
        }
}

static float cube_ps(const glm::vec3& pos, const glm::vec3& light, float far_plane) {
    cubeps::out_pos = pos;
    cubeps::u_lightPos = light;
    cubeps::u_farPlane = far_plane;
    cubeps::shader_main();
    return cubeps::gl_FragDepth;
}

// records 0..n-1 as the oracle writes them (8 words): the appended QuadNdcTransformation's mean.xy and quadScaleNdc, the
// cube pixel shader's gl_FragDepth for its wsPos, and the face (0xFFFFFFFF and zeros when nothing was appended)
REF_API void ref_light_prepass(const float* gaussians, uint32_t n, const ShadowParams* p, uint32_t format, float* out) {
    int32_t* face = new int32_t[n ? n : 1];
    uint32_t* idx = new uint32_t[n ? n : 1];
    dispatch(gaussians, n, *p, format, face, idx);
    const glm::vec3 L(p->light_position[0], p->light_position[1], p->light_position[2]);
    for (uint32_t g = 0; g < n; ++g) {
        float* o = out + (size_t)g * 8;
        std::memset(o, 0, 32);
        uint32_t fw = 0xFFFFFFFFu;
        if (face[g] >= 0) {
            const auto& q = g_buckets[(size_t)face[g] * kPerFace + idx[g]];
            o[0] = q.gaussianMean2dNdc.x; o[1] = q.gaussianMean2dNdc.y;
            o[2] = q.quadScaleNdc.x; o[3] = q.quadScaleNdc.y; o[4] = q.quadScaleNdc.z; o[5] = q.quadScaleNdc.w;
            o[6] = cube_ps(glm::vec3(q.wsPos), L, p->near_far[1]);
            fw = (uint32_t)face[g];
        }
        std::memcpy(o + 7, &fw, 4);
    }
    delete[] face;
    delete[] idx;
}

// drawToCubeMapFaces (:156-236): per face an S x S viewport, glClear(depth) to 1, the face's instances in append order,
// triangles (0,1,2), (0,2,3), depth test LESS on D24 codes.  cube: 6 x S x S floats, (float)code / 16777215.
REF_API void ref_shadow_map(const float* gaussians, uint32_t n, const ShadowParams* p, uint32_t format, uint32_t S, float* cube) {
    int32_t* face = new int32_t[n ? n : 1];
    uint32_t* idx = new uint32_t[n ? n : 1];
    dispatch(gaussians, n, *p, format, face, idx);
    delete[] face;
    delete[] idx;
    static const float V[4][3] = {{-1, -1, 0}, {-1, 1, 0}, {1, 1, 0}, {1, -1, 0}};   // quadVertices
    static const int tris[2][3] = {{0, 1, 2}, {0, 2, 3}};                           // quadIndices
    const glm::vec3 L(p->light_position[0], p->light_position[1], p->light_position[2]);
    uint32_t* codes = new uint32_t[(size_t)S * S];
    for (int f = 0; f < 6; ++f) {
        for (size_t k = 0; k < (size_t)S * S; ++k) codes[k] = 0xFFFFFFu;
        for (uint32_t i = 0; i < lightcs::cmds[f].instanceCount; ++i) {
            const auto& q = g_buckets[(size_t)f * kPerFace + i];
            float vx[4], vy[4];
            glm::vec3 vpos[4];
            for (int v = 0; v < 4; ++v) {
                cubevs::vertexPos = glm::vec4(V[v][0], V[v][1], V[v][2], 1.0f);
                cubevs::gaussianMean2LightNdc = q.gaussianMean2dNdc;
                cubevs::quadScaleLightNdc = q.quadScaleNdc;
                cubevs::position = q.wsPos;
                cubevs::shader_main();
                vx[v] = cubevs::gl_Position.x; vy[v] = cubevs::gl_Position.y;
                vpos[v] = cubevs::out_pos;
            }
            int64_t X[4], Y[4];
            bool ok[4];
            for (int v = 0; v < 4; ++v) {
                const float xw = vx[v] * ((float)S * 0.5f) + (float)S * 0.5f, yw = vy[v] * ((float)S * 0.5f) + (float)S * 0.5f;
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
                for (int64_t py = 0; py < S; ++py)
                    for (int64_t px = 0; px < S; ++px) {
                        const int64_t cx = px * 256 + 128, cy = py * 256 + 128;
                        bool in = true;
                        for (int k = 0; k < 3 && in; ++k) {
                            const int64_t ax = ex[k][0], ay = ex[k][1], bx = ey[k][0], by = ey[k][1];
                            const int64_t s = area > 0 ? 1 : -1;
                            const int64_t e = s * ((bx - ax) * (cy - ay) - (by - ay) * (cx - ax));
                            const int64_t a = s * (ay - by), b = s * (bx - ax);
                            in = e > 0 || (e == 0 && (a > 0 || (a == 0 && b > 0)));
                        }
                        if (!in) continue;
                        const float d = cube_ps(vpos[t[0]], L, p->near_far[1]);   // out_pos is the same at every vertex
                        if (d != d) continue;                                     // a NaN depth writes nothing
                        const uint32_t code = (uint32_t)std::llrint((double)std::fmin(std::fmax(d, 0.0f), 1.0f) * 16777215.0);
                        uint32_t& dst = codes[(size_t)py * S + px];
                        if (code < dst) dst = code;
                    }
            }
        }
        for (size_t k = 0; k < (size_t)S * S; ++k) cube[(size_t)f * S * S + k] = (float)codes[k] / 16777215.0f;
    }
    delete[] codes;
}

static void set_uniforms(const LightParams& p, const float* cube) {
    using namespace defps;
    u_LightPosition = glm::vec3(p.light_position[0], p.light_position[1], p.light_position[2]);
    u_camPos = glm::vec3(p.cam_pos[0], p.cam_pos[1], p.cam_pos[2]);
    u_lightColor = glm::vec3(p.light_color[0], p.light_color[1], p.light_color[2]);
    u_farPlane = p.far_plane;
    u_lightIntensity = p.light_intensity;
    u_renderMode = (int)p.render_mode;
    u_resolution = glm::vec2((float)p.width, (float)p.height);
    u_isLightingEnalbed = true;
    u_shadowCubemap = samplerCube{cube, (int)p.shadow_size};
}

static uint8_t store_u8(float v) {   // RGBA8: clamp, NaN -> 0, round half to even
    return (uint8_t)std::nearbyint(std::fmin(std::fmax(v, 0.0f), 1.0f) * 255.0f);
}

// one pixel-shader invocation on 1 x 1 textures holding the given texels; out: FragColor
REF_API void ref_deferred_fs(const uint16_t* pos16, const uint16_t* nrm16, const uint8_t* alb8, const uint8_t* mr8, const float* cube,
                             const LightParams* p, float* out) {
    using namespace defps;
    set_uniforms(*p, cube);
    static const uint16_t zero16[4] = {0, 0, 0, 0};
    gPosition = sampler2D{pos16, 0, 1, 1}; gNormal = sampler2D{nrm16, 0, 1, 1}; gAlbedo = sampler2D{alb8, 1, 1, 1};
    gDepth = sampler2D{zero16, 0, 1, 1}; gMetallicRoughness = sampler2D{mr8, 1, 1, 1};
    fragUV = glm::vec2(0.5f, 0.5f);
    shader_main();
    std::memcpy(out, &FragColor, 16);
}

// GaussianRelightingPass::execute without split screen: the full-screen quad over W x H, RGBA8, row 0 = window y 0
REF_API void ref_deferred_light(const uint16_t* pos, const uint16_t* nrm, const uint8_t* alb, const uint8_t* mr, const float* cube,
                                const LightParams* p, uint8_t* image) {
    using namespace defps;
    set_uniforms(*p, cube);
    const int W = (int)p->width, H = (int)p->height;
    gPosition = sampler2D{pos, 0, W, H}; gNormal = sampler2D{nrm, 0, W, H}; gAlbedo = sampler2D{alb, 1, W, H};
    gDepth = sampler2D{nullptr, 0, W, H}; gMetallicRoughness = sampler2D{mr, 1, W, H};
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            fragUV = glm::vec2(((float)x + 0.5f) / (float)W, ((float)y + 0.5f) / (float)H);
            shader_main();
            uint8_t* o = image + ((size_t)y * W + x) * 4;
            for (int c = 0; c < 4; ++c) o[c] = store_u8(FragColor[c]);
        }
}
