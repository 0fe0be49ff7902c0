/* m2s.h — C ABI of the H100-native mesh -> 3D-gaussian-splat conversion path.
 *
 * This is the drop-in boundary for ONE path of electronicarts/mesh2splat: the
 * conversion pass.  Every entry point names the reference interface it stands
 * in for (paths relative to the reference tree):
 *
 *   reference                                                  here
 *   ---------------------------------------------------------  ----------------------------
 *   SceneManager::setupMeshBuffers + glUtils::generateTextures  m2s_scene_upload
 *     (src/utils/SceneManager.cpp:468-576,
 *      src/utils/glUtils.cpp:252-317)
 *   ConversionPass::execute / ::conversion                      m2s_convert, m2s_convert_enqueue,
 *     (src/renderer/renderPasses/ConversionPass.cpp:9-117)      m2s_convert_host
 *     + converter{VS,GS,FS}.glsl + SSBO atomic append
 *   SceneManager::exportPly + parsers::savePlyVector            m2s_ply_encode, m2s_ply_write
 *   DepthPrepass::execute + depthPrepassVS/PS.glsl              m2s_mesh_depth, m2s_mesh_depth_enqueue
 *     (src/renderer/renderPasses/DepthPrepass.cpp:8-49)
 *   GaussiansPrepass::execute + gaussianSplattingPrepassCS.glsl  m2s_prepass, m2s_prepass_enqueue,
 *     (src/utils/SceneManager.cpp:651-678,                       m2s_prepass_mesh_depth (u_depthTestMesh 1),
 *      src/parsers/parsers.cpp:232-316,339-428,431-514,631-651)  m2s_prepass_mesh_depth_enqueue
 *   RadixSortPass::execute + radixSortPrepass.glsl               m2s_depth_sort, m2s_depth_sort_enqueue
 *     + glu::RadixSort + radixSortGather.glsl
 *     (src/renderer/renderPasses/RadixSortPass.cpp:8-90,
 *      thirdParty/RadixSort.hpp:1393-1562)
 *   GaussianSplattingPass::execute + gaussianSplattingVS.glsl     m2s_splat_draw, m2s_splat_draw_enqueue
 *     + gaussianSplattingPS.glsl
 *     (src/renderer/renderPasses/GaussianSplattingPass.cpp:37-97)
 *   GaussianShadowPass::execute                                 m2s_shadow_map, m2s_shadow_map_enqueue
 *     + gaussianPointShadowMappingCS.glsl
 *     + gaussianPointLightCubeMapShadowVS/PS.glsl
 *     (src/renderer/renderPasses/GaussianShadowPass.cpp:83-236)
 *   GaussianRelightingPass::execute                             m2s_deferred_light, m2s_deferred_light_enqueue
 *     + gaussianSplattingDeferredVS/PS.glsl
 *     (src/renderer/renderPasses/GaussianRelightingPass.cpp:42-150)
 *   SceneManager::loadModel -> execute -> exportPly             m2s_convert_file
 *     (src/utils/SceneManager.hpp:18-20)
 *   SceneManager::loadPly + parsers::loadPlyFile                 m2s_ply_parse_header, m2s_ply_decode_enqueue,
 *     (src/utils/SceneManager.cpp:37-47,                         m2s_ply_read; M2S_VIEW_PLY / M2S_VIEW_PLY_PBR
 *      src/parsers/parsers.cpp:516-629)                          as the viewer passes' input
 *
 * Plain pointers and sizes only; no C++/torch types.  All functions return an
 * m2s_status; m2s_last_error() gives the thread-local message of the last
 * failure.  The library has NO CPU fallback: without a usable CUDA device every
 * compute entry point fails with M2S_E_NOGPU.
 */
#ifndef M2S_H
#define M2S_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define M2S_VERSION 100 /* 0.1.0 */

typedef enum m2s_status {
    M2S_OK = 0,
    M2S_E_INVALID = 1,  /* bad argument */
    M2S_E_NOGPU = 2,    /* no CUDA device / driver */
    M2S_E_CUDA = 3,     /* CUDA runtime error (message in m2s_last_error) */
    M2S_E_CAPACITY = 4, /* more gaussians generated than the output holds; result.total has the
                           true count (the reference silently discards: converterFS.glsl:48-51) */
    M2S_E_IO = 5,
    M2S_E_FORMAT = 6    /* malformed .glb / unsupported feature */
} m2s_status;

/* Output record layouts (stride in bytes = m2s_record_stride(layout)). */
typedef enum m2s_layout {
    /* 6 x float4, bit-compatible with GaussianDataSSBO (src/utils/utils.hpp:145-152) /
     * GaussianVertex (converterFS.glsl:21-28): position.xyz1 | color.rgba | scale.xyz0 (raw) |
     * normal.xyz0 | rotation (w,x,y,z) | pbr (metallic, roughness, 0, 1). */
    M2S_LAYOUT_REF96 = 0,
    /* 14 floats: xyz | rot (w,x,y,z) | log(scale*sigma/R) xyz | SH0 rgb | opacity logit — the values
     * parsers.cpp:469-511 derives from the SSBO record, minus normal and f_rest. */
    M2S_LAYOUT_PACKED56 = 1,
    /* one row of the three .ply bodies the reference writes (format 0/1/2 of savePlyVector) */
    M2S_LAYOUT_PLY_STANDARD = 2,   /* 62 floats = 248 B, parsers.cpp:431-514 */
    M2S_LAYOUT_PLY_PBR = 3,        /* 19 floats =  76 B, parsers.cpp:232-316 */
    M2S_LAYOUT_PLY_COMPRESSED = 4  /* 48 B,               parsers.cpp:339-428 */
} m2s_layout;

enum {
    M2S_FLAG_NONE = 0,
    /* cap = min(6*R*R*primitive_count, 7 000 000) exactly as ConversionPass.cpp:21-24 when
     * max_gaussians == 0 (default).  With this flag and max_gaussians == 0 the cap is only the
     * capacity of the output buffer handed in. */
    M2S_FLAG_UNCAPPED = 1u << 0
};

#define M2S_FLOATS_PER_VERTEX 12u   /* pos3 normal3 tangent4 uv2: the live part of the reference's
                                       17-float vertex (SceneManager.cpp:484-512) */
#define M2S_FLOATS_PER_TRIANGLE 36u /* 144 B */
#define M2S_MAX_MIP_LEVEL 4u        /* GL_TEXTURE_MAX_LEVEL 4, glUtils.cpp:313 */
#define M2S_REFERENCE_MAX_GAUSSIANS 7000000u /* MAX_GAUSSIANS_TO_SORT, RenderPass.hpp:8 */

/* RGBA8 image, row 0 first, exactly the bytes tinygltf hands to glTexImage2D
 * (glUtils.cpp:292-303); wrap REPEAT, trilinear, levels 0..4 generated on upload. */
typedef struct m2s_texture {
    const uint8_t* rgba;
    uint32_t width, height;
} m2s_texture;

/* One glTF primitive = one utils::Mesh = one glDrawArrays of the reference
 * (ConversionPass.cpp:70-117). */
typedef struct m2s_primitive {
    uint64_t first_triangle;
    uint64_t triangle_count;
    float bbox_min[3];           /* u_bboxMin (ConversionPass.cpp:111) */
    float bbox_max[3];           /* u_bboxMax */
    float base_color_factor[4];  /* u_materialFactor (ConversionPass.cpp:110) */
    int32_t albedo_texture;      /* index into m2s_scene.textures, -1 = hasAlbedoMap 0 */
    int32_t normal_texture;
    int32_t metallic_roughness_texture;
    int32_t reserved;
} m2s_primitive;

typedef struct m2s_scene {
    /* triangle soup, world space, M2S_FLOATS_PER_TRIANGLE floats per triangle:
     * 3 x { position xyz, normal xyz, tangent xyzw, uv } */
    const float* triangles;
    uint64_t triangle_count;
    const m2s_primitive* primitives;
    uint32_t primitive_count;
    const m2s_texture* textures;
    uint32_t texture_count;
} m2s_scene;

typedef struct m2s_params {
    uint32_t resolution;    /* R = resolutionTarget (ConversionPass.cpp:45): 1..4096 */
    float gaussian_std;     /* sigma (main.cpp:26 default 0.65); used by every layout but REF96 */
    uint64_t max_gaussians; /* 0 = reference rule (see M2S_FLAG_UNCAPPED) */
    uint32_t layout;        /* m2s_layout */
    uint32_t flags;
    /* shard of the flattened triangle list this call converts (multi-GPU: one contiguous range
     * per rank); triangle_count == 0 means "to the end" */
    uint64_t first_triangle;
    uint64_t triangle_count;
    /* pixel-row band of the R x R grid this call rasterises: rows [row_begin, row_end); row_end == 0 means
     * "to R".  Lets a multi-GPU plan split meshes made of a few huge triangles (SURVEY 8e: "split very large
     * triangles by pixel-row bands"): every rank takes all triangles but only its rows. */
    uint32_t row_begin;
    uint32_t row_end;
} m2s_params;

typedef struct m2s_result {
    uint64_t total;    /* fragments generated = the reference's numberOfGaussians
                          (may exceed capacity, ConversionPass.cpp:56-59) */
    uint64_t written;  /* records actually stored = min(total, cap) */
    uint64_t cap;      /* effective cap applied */
    float device_ms;   /* device time of the conversion kernel(s), CUDA events */
} m2s_result;

typedef struct m2s_ctx m2s_ctx;       /* one per GPU; externally synchronised */
typedef struct m2s_dscene m2s_dscene; /* device-resident scene (triangles, primitive table, mip chains) */

/* ---- housekeeping ------------------------------------------------------------------------- */
int m2s_version(void);
const char* m2s_last_error(void);
const char* m2s_status_string(m2s_status s);
uint32_t m2s_record_stride(uint32_t layout);
/* min(6*R*R*max(1,primitive_count), 7 000 000): ConversionPass.cpp:21-24 */
uint64_t m2s_reference_capacity(uint32_t resolution, uint32_t primitive_count);
void m2s_params_default(m2s_params* p);

m2s_status m2s_ctx_create(int device, m2s_ctx** out);
void m2s_ctx_destroy(m2s_ctx* ctx);
int m2s_ctx_device(const m2s_ctx* ctx);
/* Conditions raised on the device that an enqueue-only call cannot return (a fused-gather wait that timed out after
 * 2 s because a peer never published): M2S_OK or M2S_E_CUDA; clears the condition.  Call after synchronising. */
m2s_status m2s_ctx_status(m2s_ctx* ctx);
int m2s_ctx_sm_count(const m2s_ctx* ctx);

/* ---- inputs: replaces setupMeshBuffers + generateTextures ---------------------------------- */
/* Fills primitives[i].bbox_{min,max} from the triangle positions.  cumulative != 0 reproduces
 * the reference, where primitive k gets the union bbox of primitives 0..k
 * (SceneManager.cpp:476-477,514-520,527); 0 gives each primitive its own box. Host-only. */
m2s_status m2s_compute_bboxes(const float* triangles, m2s_primitive* primitives,
                              uint32_t primitive_count, int cumulative);

/* Copies triangles + primitive table + textures to the device and builds mip levels 1..4
 * (2x2 box, round-to-nearest) on the GPU.  Host pointers may be pageable. */
m2s_status m2s_scene_upload(m2s_ctx* ctx, const m2s_scene* scene, m2s_dscene** out);
/* One shard of a scene (multi-GPU: one contiguous triangle range per rank): copies the triangles
 * [first_triangle, first_triangle + triangle_count) to their global positions and, of the maps `layout` consumes, only
 * the texture rows those triangles can sample (16-row groups incl. their mip rows, REPEAT wrap and all five levels'
 * footprints considered).  Converting any triangle outside the range with the returned scene is undefined. */
m2s_status m2s_scene_upload_range(m2s_ctx* ctx, const m2s_scene* scene, uint32_t layout, uint64_t first_triangle,
                                  uint64_t triangle_count, m2s_dscene** out);
/* Payload bytes copied host -> device for this scene so far (triangles + texture rows); accounting for benchmarks. */
uint64_t m2s_scene_h2d_bytes(const m2s_dscene* scene);
/* The enqueue stream of the last conversion that used the scene must be idle (scratch and scene memory are
 * stream-ordered allocations of the context stream). */
void m2s_scene_free(m2s_ctx* ctx, m2s_dscene* scene);
/* Copies one generated mip level (RGBA8, tightly packed) back to the host; for parity tests. */
m2s_status m2s_scene_read_mip(m2s_ctx* ctx, const m2s_dscene* scene, uint32_t texture,
                              uint32_t level, uint8_t* dst, uint32_t* width, uint32_t* height);

/* ---- the hot path: replaces ConversionPass::execute ---------------------------------------- */
/* Enqueue-only form.  d_out: device buffer of out_capacity records; d_keys: optional device
 * array of out_capacity uint64 (fragment identity: triangle << 24 | y << 12 | x), may be NULL;
 * d_total: device uint64 receiving the fragment count; stream: cudaStream_t (NULL = context
 * stream).  Nothing is synchronised. */
m2s_status m2s_convert_enqueue(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_params* params,
                               void* d_out, uint64_t out_capacity, uint64_t* d_keys,
                               uint64_t* d_total, void* stream);
/* enqueue + wait + read the counter back (the glFinish + counter readback of
 * ConversionPass.cpp:54-59).  Returns M2S_E_CAPACITY if total > cap (records up to cap are valid). */
m2s_status m2s_convert(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_params* params,
                       void* d_out, uint64_t out_capacity, uint64_t* d_keys, m2s_result* result);
/* Measurement aid (not part of the reference's surface): one conversion on the context stream with an event between
 * the two kernels (which then do not overlap) — the per-kernel times of the step, for bench.py's roofline. */
m2s_status m2s_convert_timed(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_params* params,
                             void* d_out, uint64_t out_capacity, float* raster_ms, float* fragment_ms);
/* Host-buffer form: upload scene, convert, download records (and keys if h_keys != NULL).
 * Everything a caller holding CPU data pays for.  Only the maps the layout consumes are uploaded, and of those only
 * the texture rows the converted triangle range can sample.  With >= 16384 triangles the call is pipelined: the
 * triangle range is converted in chunks (each bringing its triangles and texture rows with it) whose records are
 * appended on the device, and each chunk's download overlaps the next chunk's upload and kernels (pass pinned host
 * memory to benefit; M2S_HOST_CHUNKS=n overrides the chunk count, 1 = unpipelined).  The cap and the returned total
 * behave as in one launch. */
m2s_status m2s_convert_host(m2s_ctx* ctx, const m2s_scene* scene, const m2s_params* params,
                            void* h_out, uint64_t out_capacity, uint64_t* h_keys,
                            m2s_result* result);

/* ---- multi-GPU: conversion fused with the gather ------------------------------------------------
 * One process per GPU; rank r converts its own triangle range (params->first_triangle/triangle_count)
 * and its fragment kernel stores the records straight into the final buffer of EVERY rank (peer
 * memory over NVLink) at the rank-major global offset — the "single all-gather" of the conversion
 * result without a separate collective pass or a host round trip.  Buffers come from any allocator
 * that maps peer memory into each process (torch symmetric memory, cudaIpc*, cuMem*).
 * xch[p]: rank p's exchange block, M2S_MAX_PEERS*4 uint64, zeroed once before first use.
 * Every rank must make the same sequence of calls (an epoch counter pairs them up).  Layouts REF96 and
 * PACKED56.  d_total_global (device, optional) receives the number of records in the final buffer
 * once all ranks' records have landed; work enqueued after this call on `stream` sees the full buffer. */
#define M2S_MAX_PEERS 8
typedef struct m2s_peers {
    uint32_t world, rank;
    void* out[M2S_MAX_PEERS];
    uint64_t* xch[M2S_MAX_PEERS];
} m2s_peers;
m2s_status m2s_convert_gather_enqueue(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_params* params,
                                      const m2s_peers* peers, uint64_t out_capacity, uint64_t* d_total_global,
                                      void* stream);

/* ---- outputs: replaces exportPly / savePlyVector -------------------------------------------- */
/* ASCII header of format 0/1/2 for `count` vertices; returns bytes written (excl. NUL) or the
 * needed size if dst is too small. */
size_t m2s_ply_header(uint32_t format, uint64_t count, char* dst, size_t dst_size);
/* GPU encoder: REF96 device records -> .ply body rows on the device (format 0/1/2). */
m2s_status m2s_ply_encode(m2s_ctx* ctx, const void* d_ref96, uint64_t count, uint32_t format,
                          float scale_multiplier, void* d_rows, void* stream);
/* Host writer: REF96 host records -> file, byte-identical to parsers::savePlyVector. */
m2s_status m2s_ply_write(const char* path, const void* h_ref96, uint64_t count, uint32_t format,
                         float scale_multiplier);

/* ---- inputs of the viewer: replaces SceneManager::loadPly / parsers::loadPlyFile (SURVEY 8 f-10) --------------------
 * A .ply file -> REF96 records exactly as loadPlyFile fills GaussianDataSSBO (parsers.cpp:577-622):
 *   position  (x, y, z, 1)
 *   color     (f_dc * SH_COEFF0 + 0.5f per channel: two fp32 roundings, no FMA,  1 / (1 + (double)expf(-opacity)) in fp64)
 *   scale     (expf(scale_0), expf(scale_1), expf(scale_2), 1)
 *   normal    (nx, ny, nz, 0) with has_pbr, else 0
 *   rotation  glm::normalize(glm::quat(rot_0, rot_1, rot_2, rot_3)) stored (w, x, y, z): each component times
 *             1 / sqrt((r0 r0 + r1 r1) + (r2 r2 + r3 r3)); (1, 0, 0, 0) when that length is <= 0; NaN propagates
 *   pbr       (metallicFactor, roughnessFactor, 0, 0) with has_pbr, else 0
 * expf is evaluated on the device with glibc's own algorithm (the table-driven fp64 expf glibc selects on x86-64 with FMA),
 * bit-identical to it on all 2^32 inputs (tests/test_gpu_codec.py); against a glibc that uses its non-FMA variant
 * scale.xyz and color.a may differ by 1 ulp, every other field is bit-exact.  The writers' encodings are exact the same
 * way: SH0 = (c - 0.5f) / SH_COEFF0 (the IEEE quotient), the opacity logit and the log-scale with glibc's logf, in the
 * conversion's .ply and PACKED56 layouts, m2s_ply_encode and m2s_convert_file.  Denormals are kept.  SH rest coefficients are skipped, as in the reference.
 * Property rules (happly): the properties are found by name in the first element "vertex" (order and extra properties do
 * not matter); x y z f_dc_0..2 opacity scale_0..2 rot_0..3 are required; every property read must be float / float32
 * (happly does not narrow a double); has_pbr = nx ny nz metallicFactor roughnessFactor all present, and 1 for a file of 0
 * vertices whatever its properties (the reference compares vector sizes: 0 == 0).
 * Deviations from the reference, each M2S_E_FORMAT with a message naming the cause (the reference prints the error, keeps
 * the previous gaussians and loadPly still returns true):
 *   - ascii and binary_big_endian bodies (happly reads them; 3DGS files are binary_little_endian);
 *   - an element with a list property before "vertex" (fixed-size elements before it are skipped by arithmetic; elements
 *     after it are ignored);
 *   - a header without end_header, or a body shorter than body_offset + vertex_count * row_stride (checked with
 *     overflow-safe arithmetic before anything is allocated; happly reads past the end of the file and keeps garbage);
 *   - vertex rows longer than M2S_PLY_MAX_STRIDE bytes, or a list property in "vertex";
 *   - the compressed format (2) of m2s_ply_write is rejected because f_dc_0 is missing, as the reference rejects it. */
#define M2S_PLY_PROPS 19
enum {   /* index into m2s_ply_info.offset */
    M2S_PLY_X = 0, M2S_PLY_Y, M2S_PLY_Z, M2S_PLY_NX, M2S_PLY_NY, M2S_PLY_NZ, M2S_PLY_F_DC_0, M2S_PLY_F_DC_1, M2S_PLY_F_DC_2,
    M2S_PLY_METALLIC, M2S_PLY_ROUGHNESS, M2S_PLY_OPACITY, M2S_PLY_SCALE_0, M2S_PLY_SCALE_1, M2S_PLY_SCALE_2,
    M2S_PLY_ROT_0, M2S_PLY_ROT_1, M2S_PLY_ROT_2, M2S_PLY_ROT_3
};
#define M2S_PLY_MAX_STRIDE 4096u   /* bytes per vertex row the decoder takes */
typedef struct m2s_ply_info {
    uint64_t vertex_count;
    uint64_t body_offset;            /* file offset of vertex row 0 */
    uint32_t row_stride;             /* bytes per vertex row: 1..M2S_PLY_MAX_STRIDE */
    uint32_t has_pbr;                /* loadPlyFile's hasPbr */
    int32_t offset[M2S_PLY_PROPS];   /* byte offset in the row of x y z nx ny nz f_dc_0..2 metallicFactor roughnessFactor
                                        opacity scale_0..2 rot_0..3; -1 = absent */
} m2s_ply_info;
/* Host only.  bytes/size: the first `size` bytes of the file (the whole file, or any prefix that holds the header);
 * file_size: the size of the whole file.  Never reads outside [bytes, bytes + size). */
m2s_status m2s_ply_parse_header(const void* bytes, size_t size, uint64_t file_size, m2s_ply_info* info);
/* Enqueue-only.  d_rows: `count` rows of info->row_stride bytes (row 0 = the file's vertex row 0 of this block; no
 * alignment required); d_ref96: count x 96 B, 16-byte aligned.  stream NULL = the context stream. */
m2s_status m2s_ply_decode_enqueue(m2s_ctx* ctx, const m2s_ply_info* info, const void* d_rows, uint64_t count,
                                  void* d_ref96, void* stream);
/* The whole load, synchronous on the context stream: header parsed on the host, the body read in row-aligned blocks
 * into two pinned buffers, each block copied to a two-slot device staging area and decoded into d_ref96 + first_row * 96
 * while the next block is read from the file.  d_ref96 == NULL: only fills *info (the probe that sizes the buffer).
 * capacity < vertex_count: M2S_E_CAPACITY, *info filled, nothing written. */
m2s_status m2s_ply_read(m2s_ctx* ctx, const char* path, void* d_ref96, uint64_t capacity, m2s_ply_info* info);
/* Payload bytes m2s_ply_read copied host -> device on this context so far (accounting for benchmarks). */
uint64_t m2s_ply_h2d_bytes(const m2s_ctx* ctx);
/* `layout` values of m2s_prepass* and m2s_shadow_map* for REF96 records as loadPlyFile fills them (not conversion
 * layouts: m2s_record_stride and m2s_convert* do not take them).  The reference's u_format 1: scale multiplier 1, no mesh
 * depth test (m2s_prepass_mesh_depth gives m2s_prepass's output); the normal through the normal matrix with u_plyHasPbr 1,
 * the shortest axis with 0 (gaussianSplattingPrepassCS.glsl:93-130, gaussianPointShadowMappingCS.glsl:96). */
#define M2S_VIEW_PLY     16u   /* u_format 1, u_plyHasPbr 0 */
#define M2S_VIEW_PLY_PBR 17u   /* u_format 1, u_plyHasPbr 1 */

/* ---- file-level surface: loadModel -> execute -> exportPly --------------------------------- */
/* .glb -> host scene: SceneManager::parseGltfFile + setupMeshBuffers (bbox rule) + loadTextures
 * (src/utils/SceneManager.cpp:195-459,468-649): scene-graph world transforms, de-indexing, flat
 * normal / per-face tangent fallbacks, one primitive per glTF primitive, RGBA8 images.
 * cumulative_bbox != 0 keeps the reference's running-union bbox. */
typedef struct m2s_hscene m2s_hscene;
m2s_status m2s_glb_load(const char* glb_path, int cumulative_bbox, m2s_hscene** out);
const m2s_scene* m2s_hscene_view(const m2s_hscene* scene);
/* "<mesh name or 'mesh'>_<counter>" exactly as utils::Mesh::name (SceneManager.cpp:305-307) */
const char* m2s_hscene_primitive_name(const m2s_hscene* scene, uint32_t primitive);
void m2s_hscene_free(m2s_hscene* scene);

/* loadModel -> ConversionPass::execute -> exportPly in one call (the batch loop of
 * guiRendererConcreteMediator.cpp:146-193): capacity = the reference rule, .ply rows encoded on the GPU and
 * streamed to disk through two pinned buffers.  ply_format as exportPly's exportFormat (0 standard,
 * 1 PBR, 2 compressed; anything else = 0).  M2S_E_CAPACITY: the file holds the `cap` valid records. */
m2s_status m2s_convert_file(m2s_ctx* ctx, const char* glb_path, uint32_t resolution,
                            float gaussian_std, uint32_t ply_format, const char* ply_path,
                            m2s_result* result);

/* ---- the step after the path in the reference's frame graph: the viewer prepass (SURVEY 8 f-4) ----------------
 * GaussiansPrepass::execute (src/renderer/renderPasses/GaussiansPrepass.cpp:8-55) + gaussianSplattingPrepassCS.glsl
 * :58-204: per gaussian — model/view/clip transform, frustum cull (1.05 w), 3-D covariance from scale and rotation,
 * EWA projection to a 2-D conic (+0.3 low-pass), screen-space axes, atomic append of one QuadNdcTransformation (96 B:
 * gaussianMean2dNdc, quadScaleNdc, color, conic (.w = view depth), normal (.w = pbr.x), wsPos (.w = pbr.y)) and of the
 * view-space depth the radix sort keys on.  Matrices are column-major (glm::mat4).  Input records:
 *   M2S_LAYOUT_REF96     the reference's GaussianVertex, u_format 0 (scale * std_dev, normal through the normal matrix)
 *   M2S_LAYOUT_PACKED56  a standard 3DGS gaussian as the reference loads it from a .ply without PBR values, u_format 1
 *                        (scale = exp(log_scale), colour = SH0 * C0 + 0.5, alpha = sigmoid(opacity), normal = the
 *                        shortest axis, pbr = 0)
 *   M2S_VIEW_PLY(_PBR)   REF96 records as m2s_ply_read loads them, u_format 1 (u_plyHasPbr 0 / 1; see above)
 * The mesh depth test (u_depthTestMesh 1) is m2s_prepass_mesh_depth below.  Not reproduced: render mode 3 (debug colours
 * from the invocation id).  Output order is unspecified, as in the reference (atomic arrival order). */
typedef struct m2s_prepass_params {
    float world_to_view[16];   /* renderContext.viewMat */
    float view_to_clip[16];    /* renderContext.projMat */
    float model_to_world[16];  /* renderContext.modelMat */
    float resolution[2];       /* renderContext.rendererResolution */
    float near_far[2];
    float std_dev;             /* gaussianStd / resolutionTarget (GaussiansPrepass.cpp:18) */
    uint32_t render_mode;      /* 0 (or 6) colour, 1 depth, 2 normal */
    uint32_t layout;           /* M2S_LAYOUT_REF96, M2S_LAYOUT_PACKED56, M2S_VIEW_PLY or M2S_VIEW_PLY_PBR */
    uint32_t reserved;
} m2s_prepass_params;
#define M2S_QUAD_BYTES 96u
/* Enqueue-only: d_quads holds `count` x 96 B, d_depths `count` floats, d_valid one uint32 (zeroed by the call, then the
 * number of surviving gaussians).  d_count (optional): device-side count that overrides `count` downwards (the
 * counter of a conversion that was only enqueued). */
m2s_status m2s_prepass_enqueue(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count,
                               const m2s_prepass_params* params, void* d_quads, float* d_depths, uint32_t* d_valid,
                               void* stream);
/* Synchronous variant on the context stream; *valid receives the counter. */
m2s_status m2s_prepass(m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_prepass_params* params,
                       void* d_quads, float* d_depths, uint32_t* valid);

/* ---- the mesh depth pre-pass (SURVEY 8 f-9) and the prepass's mesh depth test -----------------------------------------
 * DepthPrepass::execute (src/renderer/renderPasses/DepthPrepass.cpp:8-49) + depthPrepassVS/PS.glsl: every triangle of
 * the scene whose primitive has base_color_factor[3] == 1.0f (an exact compare; texture alpha plays no part) drawn into
 * a width x height depth map cleared to 1, depth test LESS, both windings.  gl_Position = ((P V) M) (p, 1), the product
 * built on the host with GLM's fp32 mat4 * mat4.  GL's fixed-function parts are fixed in DESIGN §2: clipping against
 * the near and far planes and a guard band of twice the viewport in x and y (a deviation: GL clips to the viewport's
 * guard band of its own choosing), the splat draw's rasteriser, depth interpolated in fp64 from the exact edge values,
 * and D24 codes.  d_depth: width x height floats, row 0 = window y 0, each texel (float)code / 16777215 as
 * texture(...).r returns it; every texel is written exactly once, clear included (a scene without an opaque triangle
 * gives the cleared map).  The scene must come from m2s_scene_upload (all triangles resident). */
typedef struct m2s_mesh_depth_params {
    float world_to_view[16];   /* renderContext.viewMat, column-major */
    float view_to_clip[16];    /* renderContext.projMat */
    float model_to_world[16];  /* renderContext.modelMat */
    uint32_t width, height;    /* renderContext.rendererResolution: 1..4096 each */
} m2s_mesh_depth_params;
/* Enqueue-only.  max_pairs (< 2^30) is the budget of (16 x 16 tile, clipped triangle) pairs: when the triangles need more,
 * the longest prefix of source triangles (scene order) whose pairs fit is drawn.  d_drawn (optional, device uint32)
 * receives the prefix length, d_pairs (optional, device uint64) the pairs all triangles need.  The scene has fewer than
 * 2^29 triangles.  Scratch is stream-ordered context memory grown on `stream` (NULL = context stream); nothing is
 * synchronised. */
m2s_status m2s_mesh_depth_enqueue(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_mesh_depth_params* params, float* d_depth,
                                  uint64_t max_pairs, uint64_t* d_pairs, uint32_t* d_drawn, void* stream);
/* Synchronous form on the context stream: counts the pairs, reads the count back once, grows the scratch and draws every
 * triangle.  *pairs (optional, host) receives the pair count. */
m2s_status m2s_mesh_depth(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_mesh_depth_params* params, float* d_depth,
                          uint64_t* pairs);
/* The prepass with the mesh depth test (gaussianSplattingPrepassCS.glsl:78-91, u_depthTestMesh 1): a REF96 gaussian that
 * passes the frustum cull and has color.a > 0.95f is dropped when (pos2d.z / pos2d.w) 0.5 + 0.5 > depth + 0.00002f,
 * depth = the map's texel at uv = (pos2d.xy / pos2d.w) 0.5 + 0.5, sampled NEAREST with CLAMP_TO_EDGE.  PACKED56 and
 * M2S_VIEW_PLY* input (u_format 1) never reads the map: the output equals m2s_prepass's.  d_mesh_depth: depth_width x depth_height floats
 * as m2s_mesh_depth writes them (1..4096 each).  Everything else as m2s_prepass_enqueue / m2s_prepass. */
m2s_status m2s_prepass_mesh_depth_enqueue(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count,
                                          const m2s_prepass_params* params, const float* d_mesh_depth, uint32_t depth_width,
                                          uint32_t depth_height, void* d_quads, float* d_depths, uint32_t* d_valid, void* stream);
m2s_status m2s_prepass_mesh_depth(m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_prepass_params* params,
                                  const float* d_mesh_depth, uint32_t depth_width, uint32_t depth_height, void* d_quads,
                                  float* d_depths, uint32_t* valid);

/* ---- the step after the prepass: the viewer's depth sort (SURVEY 8 f-5) ----------------------------------------------
 * RadixSortPass::execute (src/renderer/renderPasses/RadixSortPass.cpp:8-90): radixSortPrepass.glsl + glu::RadixSort
 * + radixSortGather.glsl.  Stable ascending sort of the quads by the uint32 bits of their view depth (front to back).
 * n = count, or min(count, *d_count) with d_count (the prepass's d_valid).  d_quads: count x 96 B, d_depths: count
 * floats (both unchanged); d_sorted_quads: count x 96 B, n written; d_order (optional): n uint32 source indices;
 * d_draw (optional): 5 uint32 = DrawElementsIndirectCommand {6, n, 0, 0, 0}.  count < 2^30.
 * Deviation: with n = 0 the draw command is written too (instanceCount 0), where the reference dispatches nothing and
 * leaves the previous frame's command in place.  Scratch is a stream-ordered allocation of the context, grown on `stream`
 * (NULL = context stream); nothing is synchronised. */
m2s_status m2s_depth_sort_enqueue(m2s_ctx* ctx, const void* d_quads, const float* d_depths, uint64_t count,
                                  const uint32_t* d_count, void* d_sorted_quads, uint32_t* d_order,
                                  uint32_t* d_draw, void* stream);
m2s_status m2s_depth_sort(m2s_ctx* ctx, const void* d_quads, const float* d_depths, uint64_t count,
                          void* d_sorted_quads, uint32_t* d_order, uint32_t* d_draw);   /* context stream, synchronised */

/* ---- the step after the depth sort: the viewer's splat draw (SURVEY 8 f-6) ------------------------------------------
 * GaussianSplattingPass::execute (src/renderer/renderPasses/GaussianSplattingPass.cpp:37-97) + gaussianSplattingVS.glsl
 * + gaussianSplattingPS.glsl:29-46: every sorted quad, as the two triangles (V0,V1,V2), (V0,V2,V3), drawn into the
 * G-buffer cleared to 0, blended front to back (dst = src * (1 - dst.a) + dst per target, with the target's own alpha;
 * dst = src + dst in render mode 4).  The rasterisation, exp, blend and format rules the GL driver would supply are
 * fixed in DESIGN §2.  Row 0 of every target is the bottom row (window y = 0), as glReadPixels returns it. */
typedef struct m2s_gbuffer {
    uint16_t* position;            /* attachment 0, RGBA16F: width x height x 4 fp16 bits, 8-byte aligned, or NULL */
    uint16_t* normal;              /* attachment 1, RGBA16F */
    uint8_t* albedo;               /* attachment 2, RGBA8: width x height x 4 bytes, 4-byte aligned, or NULL */
    uint16_t* depth;               /* attachment 3, RGBA16F */
    uint8_t* metallic_roughness;   /* attachment 4, RGBA8 */
} m2s_gbuffer;
typedef struct m2s_splat_params {
    uint32_t width, height;        /* renderContext.rendererResolution: 1..4096 each */
    uint32_t render_mode;          /* 0..6; only mode 4 (overdraw) draws differently */
} m2s_splat_params;
/* Enqueue-only.  n = count, or min(count, d_draw[1]) with d_draw the sort's DrawElementsIndirectCommand.  Every pixel of
 * every non-NULL target is written exactly once (no memset needed); a NULL target is not drawn and changes nothing in
 * the others.  max_pairs (< 2^30) is the budget of (16 x 16 tile, quad) pairs: when the n quads need more, the longest
 * prefix of quads whose pairs fit is drawn, and the image is the reference's with that many instances.  d_drawn
 * (optional, device uint32) receives the prefix length, d_pairs (optional, device uint64) the pairs all n quads need.
 * count < 2^30; d_sorted_quads 16-byte aligned.  Scratch is stream-ordered context memory grown on `stream` (NULL =
 * context stream), kept between calls; nothing is synchronised. */
m2s_status m2s_splat_draw_enqueue(m2s_ctx* ctx, const void* d_sorted_quads, uint64_t count, const uint32_t* d_draw,
                                  const m2s_splat_params* params, const m2s_gbuffer* gbuffer, uint64_t max_pairs,
                                  uint64_t* d_pairs, uint32_t* d_drawn, void* stream);
/* Synchronous form on the context stream: counts the pairs, reads the count back once, grows the scratch and draws all
 * `count` quads.  *pairs (optional, host) receives the pair count. */
m2s_status m2s_splat_draw(m2s_ctx* ctx, const void* d_sorted_quads, uint64_t count, const m2s_splat_params* params,
                          const m2s_gbuffer* gbuffer, uint64_t* pairs);

/* ---- the shadow pass (SURVEY 8 f-7) ------------------------------------------------------------------------------------
 * GaussianShadowPass::execute (src/renderer/renderPasses/GaussianShadowPass.cpp:83-236): the light prepass
 * (gaussianPointShadowMappingCS.glsl:58-207) and six face draws (gaussianPointLightCubeMapShadowVS/PS.glsl) into a
 * point-light depth cube map.  Per gaussian: world position, cube face of normalize(ws - light) (x wins ties over y and
 * z, y over z; a NaN direction gives face 5), that face's glm::lookAt view and glm::perspective(90 deg, 1, near, far),
 * the main prepass's 1.05 w cull, covariance, EWA projection and axes (with the renderer's resolution, sic), then one
 * quad drawn into its face with gl_FragDepth = length(ws - light) / far, depth test LESS on a D24 face cleared to 1.
 * The D24 code, rasteriser and sampling rules are DESIGN §2.  Deviation: one light record per source gaussian instead
 * of the reference's per-face buckets of 7 000 000 (an overflowing bucket writes past its region there). */
typedef struct m2s_shadow_params {
    float model_to_world[16];  /* renderContext.modelMat, column-major */
    float light_position[3];   /* pointLightModel[3].xyz */
    float near_far[2];
    float resolution[2];       /* renderContext.rendererResolution (not the face size: sic, the reference's u_resolution) */
    float std_dev;             /* gaussianStd / resolutionTarget */
    uint32_t layout;           /* M2S_LAYOUT_REF96, M2S_LAYOUT_PACKED56, M2S_VIEW_PLY or M2S_VIEW_PLY_PBR */
    uint32_t size;             /* face size S: 1..1024 (the reference uses 1024) */
} m2s_shadow_params;
#define M2S_LIGHT_RECORD_BYTES 32u
/* Enqueue-only.  n = count, or min(count, *d_count) with d_count the conversion's device counter (uint64).  d_cube:
 * 6 x S x S floats, face-major in the order +X -X +Y -Y +Z -Z, row 0 = window y 0 of the face's draw; each texel is
 * the D24 value as a sampler returns it, (float)code / 16777215.  Every texel is written exactly once, clear
 * included; n = 0 gives the cleared map.  d_light_quads (optional, 16-byte aligned, count x 32 B; NULL = context
 * scratch) receives the light records 0..n-1 in source order: mean NDC x, y, the four quadScaleNdc values, the
 * gl_FragDepth, and the face as a uint32 (0xFFFFFFFF and zeros for a culled gaussian).  max_pairs (< 2^30) is the budget
 * of (16 x 16 face tile, record) pairs: when the n records need more, the longest prefix of records whose pairs fit is
 * drawn.  d_drawn (optional, device uint32) receives the prefix length, d_pairs (optional, device uint64) the pairs all
 * n records need.  count < 2^30; d_records 16-byte aligned.  Scratch is stream-ordered context memory grown on
 * `stream` (NULL = context stream); nothing is synchronised. */
m2s_status m2s_shadow_map_enqueue(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count,
                                  const m2s_shadow_params* params, float* d_cube, void* d_light_quads, uint64_t max_pairs,
                                  uint64_t* d_pairs, uint32_t* d_drawn, void* stream);
/* Synchronous form on the context stream: counts the pairs, reads the count back once, grows the scratch and draws all
 * `count` records.  *pairs (optional, host) receives the pair count. */
m2s_status m2s_shadow_map(m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_shadow_params* params,
                          float* d_cube, void* d_light_quads, uint64_t* pairs);

/* ---- the deferred lighting (SURVEY 8 f-8) ------------------------------------------------------------------------------
 * GaussianRelightingPass::execute (src/renderer/renderPasses/GaussianRelightingPass.cpp:42-150) +
 * gaussianSplattingDeferredPS.glsl:32-165: pixel (x, y) reads G-buffer texel (x, y) and writes RGBA8 (no sRGB).
 *   render mode 5       (metallic_roughness.rg, 0, 1)
 *   modes 0-4           (albedo.rgb, 1)
 *   mode 6 (FINAL)      GGX with one point light (1/d^2), 20-tap PCF of the cube map (bias 0.05), ambient 0.3 albedo,
 *                       Reinhard, pow 1/2.2 — with the shader's quirks kept (DESIGN §6)
 * Required: albedo (every mode), metallic_roughness (modes 5, 6), position, normal and d_cube (mode 6); the rest may
 * be NULL.  d_cube as m2s_shadow_map writes it, with shadow_size = S.  The pow, sampling and format rules are DESIGN §2.
 * Not built: split screen and the mesh G-buffer (GaussianRelightingPass.cpp:90-135). */
typedef struct m2s_light_params {
    uint32_t width, height;    /* renderContext.rendererResolution: 1..4096 each */
    uint32_t render_mode;      /* 0..6 */
    float light_position[3];
    float light_color[3];
    float light_intensity;
    float cam_pos[3];
    float far_plane;
    uint32_t shadow_size;      /* S of d_cube: 1..1024 (mode 6) */
} m2s_light_params;
/* Enqueue-only.  d_image: width x height x 4 bytes, 4-byte aligned, row 0 = the bottom row.  Every pixel is written
 * once.  Nothing is synchronised. */
m2s_status m2s_deferred_light_enqueue(m2s_ctx* ctx, const m2s_gbuffer* gbuffer, const float* d_cube,
                                      const m2s_light_params* params, uint8_t* d_image, void* stream);
/* Synchronous form on the context stream. */
m2s_status m2s_deferred_light(m2s_ctx* ctx, const m2s_gbuffer* gbuffer, const float* d_cube,
                              const m2s_light_params* params, uint8_t* d_image);

#ifdef __cplusplus
}
#endif
#endif /* M2S_H */
