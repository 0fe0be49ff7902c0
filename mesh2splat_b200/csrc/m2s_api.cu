// m2s_api.cu — C-ABI implementation (include/m2s.h): housekeeping and the context.  The rest of the C ABI lives in
// m2s_scene.cu (device scene), m2s_convert.cu (conversion, .ply output) and m2s_viewer.cu (viewer passes); the loader and
// the .ply writer in m2s_glb.cpp and m2s_host.cpp.
// There is deliberately NO CPU compute path: without a CUDA device every entry point fails.
#include "m2s_ctx.cuh"

using namespace m2s;

M2S_EXPORT int m2s_version(void) { return M2S_VERSION; }

M2S_EXPORT const char* m2s_status_string(m2s_status s) {
    switch (s) {
        case M2S_OK: return "ok";
        case M2S_E_INVALID: return "invalid argument";
        case M2S_E_NOGPU: return "no CUDA device";
        case M2S_E_CUDA: return "CUDA error";
        case M2S_E_CAPACITY: return "output capacity exceeded";
        case M2S_E_IO: return "I/O error";
        case M2S_E_FORMAT: return "unsupported or malformed input";
    }
    return "unknown";
}

M2S_EXPORT uint32_t m2s_record_stride(uint32_t layout) {
    switch (layout) {
        case M2S_LAYOUT_REF96: return 96;
        case M2S_LAYOUT_PACKED56: return 56;
        case M2S_LAYOUT_PLY_STANDARD: return 248;
        case M2S_LAYOUT_PLY_PBR: return 76;
        case M2S_LAYOUT_PLY_COMPRESSED: return 48;
    }
    return 0;
}

M2S_EXPORT uint64_t m2s_reference_capacity(uint32_t R, uint32_t primitive_count) {
    const uint64_t mc = primitive_count ? primitive_count : 1;
    return std::min<uint64_t>((uint64_t)R * R * 6ull * mc, M2S_REFERENCE_MAX_GAUSSIANS);
}

M2S_EXPORT void m2s_params_default(m2s_params* p) {
    if (!p) return;
    std::memset(p, 0, sizeof(*p));
    p->resolution = 520;  // int(16 + 0.5 * (1024 - 16)): ImGuiUI.cpp:512 with the default quality
    p->gaussian_std = 0.65f;
    p->layout = M2S_LAYOUT_REF96;
}

// everything a context owns beyond its device and SM count; on failure m2s_ctx_destroy releases what was made so far
static m2s_status ctx_init(m2s_ctx* c) {
    CUDA_TRY(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    cudaMemPool_t pool;
    CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, c->device));
    uint64_t thresh = UINT64_MAX;  // keep freed blocks cached: uploads in steady state never hit cudaMalloc
    CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
    CUDA_TRY(cudaMalloc(&c->d_sched, 8 * 128));
    CUDA_TRY(cudaMalloc(&c->d_total, sizeof(unsigned long long)));
    CUDA_TRY(cudaMallocHost(&c->h_total, sizeof(unsigned long long)));
    CUDA_TRY(cudaHostAlloc(&c->h_status, sizeof(uint32_t), cudaHostAllocMapped));
    *c->h_status = 0;
    CUDA_TRY(cudaHostGetDevicePointer((void**)&c->d_status, c->h_status, 0));
    for (cudaEvent_t* ev : {&c->ev0, &c->ev1}) CUDA_TRY(cudaEventCreate(ev));
    for (cudaEvent_t* ev : {&c->ev_stage[0], &c->ev_stage[1]}) CUDA_TRY(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
    const m2s_status st = c->pipeline.create();
    if (st != M2S_OK) return st;
    for (int l = 0; l < m2s_ctx::kLayouts; ++l) {
        CUDA_TRY(raster_configure(l, &c->blocks_per_sm[l]));
        CUDA_TRY(fragment_configure(l, &c->frag_blocks_per_sm[l]));
        if (c->blocks_per_sm[l] < 1 || c->frag_blocks_per_sm[l] < 1) { set_error("conversion kernel does not fit on this device"); return M2S_E_CUDA; }
    }
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_ctx_create(int device, m2s_ctx** out) {
    if (!out) { set_error("m2s_ctx_create: out is NULL"); return M2S_E_INVALID; }
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        set_error(std::string("no CUDA device available: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0"));
        return M2S_E_NOGPU;
    }
    if (device < 0 || device >= n) { set_error("m2s_ctx_create: bad device index"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) { set_error("mesh2splat_b200 kernels are built for sm_90a (H100) only"); return M2S_E_NOGPU; }
    m2s_ctx* c = new m2s_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    const m2s_status st = ctx_init(c);
    if (st != M2S_OK) { m2s_ctx_destroy(c); return st; }
    *out = c;
    return M2S_OK;
}

// Also releases a context that ctx_init left half built: every handle is checked before it is released.
M2S_EXPORT void m2s_ctx_destroy(m2s_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (Scratch* s : c->all_scratch()) if (s->p) cudaFreeAsync(s->p, c->stream);
    cudaStreamSynchronize(c->stream);
    if (c->d_prepass_valid) cudaFree(c->d_prepass_valid);
    cudaFree(c->d_sched); cudaFree(c->d_total);
    if (c->h_total) cudaFreeHost(c->h_total);
    if (c->h_status) cudaFreeHost(c->h_status);
    for (int i = 0; i < 2; ++i) if (c->h_stage[i]) cudaFreeHost(c->h_stage[i]);
    c->pipeline.release();
    for (cudaEvent_t ev : {c->ev0, c->ev1, c->ev_mid, c->ev_stage[0], c->ev_stage[1]}) if (ev) cudaEventDestroy(ev);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

M2S_EXPORT int m2s_ctx_device(const m2s_ctx* c) { return c ? c->device : -1; }
// Device-side conditions the enqueue-only entry points cannot return: call after synchronising the stream.
M2S_EXPORT m2s_status m2s_ctx_status(m2s_ctx* c) {
    if (!c) { set_error("m2s_ctx_status: ctx is NULL"); return M2S_E_INVALID; }
    const uint32_t v = __atomic_exchange_n(c->h_status, 0u, __ATOMIC_ACQ_REL);
    if (v == 0) return M2S_OK;
    c->dirty = true;
    set_error(std::string("fused gather: a peer rank did not publish its ") + ((v & 1u) ? "count" : "completion flag") +
              " within 2 s (did every rank call m2s_convert_gather_enqueue the same number of times?)");
    return M2S_E_CUDA;
}
M2S_EXPORT int m2s_ctx_sm_count(const m2s_ctx* c) { return c ? c->sm_count : 0; }
