// m2s_codec.cu — m2s_debug_codec_eval: each function of m2s_codec.cuh applied elementwise on the device, so that tests
// compare the encodings the kernels use with glibc on every input.  Exported, not declared in m2s.h (like
// m2s_debug_convert_plan); the function ids are mirrored in _abi.py (CODEC_*).
#include "m2s_codec.cuh"
#include "m2s_ctx.cuh"

namespace m2s {
namespace {

enum CodecFn : uint32_t { kSh0Encode = 0, kOpacityLogit = 1, kLogScale = 2, kExpf = 3, kOpacitySigmoid = 4, kCodecFns };

__global__ void codec_eval_kernel(uint32_t fn, float arg, const float* __restrict__ in, unsigned long long n, float* __restrict__ out) {
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const float x = in[i];
        float y;
        switch (fn) {
            case kSh0Encode: y = sh0_encode(x); break;
            case kOpacityLogit: y = opacity_logit(x); break;
            case kLogScale: y = log_scale(x, arg); break;
            case kExpf: y = ref_expf(x, kExp2Tab); break;
            default: y = opacity_sigmoid(x, kExp2Tab); break;
        }
        out[i] = y;
    }
}

}  // namespace
}  // namespace m2s

using namespace m2s;

// fn: 0 sh0_encode, 1 opacity_logit, 2 log_scale with mult = arg, 3 ref_expf, 4 opacity_sigmoid; arg is unused by the others
M2S_EXPORT m2s_status m2s_debug_codec_eval(m2s_ctx* ctx, uint32_t fn, float arg, const void* d_in, uint64_t n, void* d_out, void* stream) {
    const char* name = "m2s_debug_codec_eval";
    if (!ctx || (n && (!d_in || !d_out))) return invalid(name, "NULL argument");
    if (fn >= kCodecFns) return invalid(name, "unknown function id");
    if (!aligned_ok(name, "the buffers must be 4-byte aligned", {{d_in, 4}, {d_out, 4}})) return M2S_E_INVALID;
    if (n == 0) return M2S_OK;
    CUDA_TRY(cudaSetDevice(ctx->device));
    const unsigned blocks = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)ctx->sm_count * 16);
    codec_eval_kernel<<<blocks, 256, 0, pick_stream(ctx, stream)>>>(fn, arg, static_cast<const float*>(d_in), n, static_cast<float*>(d_out));
    CUDA_TRY(cudaGetLastError());
    return M2S_OK;
}
