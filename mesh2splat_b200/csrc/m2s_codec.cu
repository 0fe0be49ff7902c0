// m2s_codec.cu — the .ply rows of REF96 records (ply_rows_kernel, behind m2s_ply_encode), and m2s_debug_codec_eval: each
// function of m2s_codec.cuh applied elementwise on the device, so that tests compare the encodings the kernels use with
// glibc on every input.  m2s_debug_codec_eval is exported, not declared in m2s.h (like m2s_debug_convert_plan); the
// function ids are mirrored in _abi.py (CODEC_*).
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

// .ply body rows from REF96 records (parsers.cpp:232-316,339-428,431-514); format 0 rows 8-byte aligned
__global__ void ply_rows_kernel(const float4* __restrict__ rec, unsigned long long count, uint32_t format, float mult,
                                unsigned char* __restrict__ rows) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const float4 pos = rec[i * 6 + 0], col = rec[i * 6 + 1], sc = rec[i * 6 + 2], nrm = rec[i * 6 + 3], rot = rec[i * 6 + 4],
                 pbr = rec[i * 6 + 5];
    const float3 p = make_float3(pos.x, pos.y, pos.z), n = make_float3(nrm.x, nrm.y, nrm.z);
    const float ls[2] = {log_scale(sc.x, mult), log_scale(sc.y, mult)};
    if (format == 1) {
        ply_row<1>(rows + i * 76ull, p, n, col, &rot.x, ls, log_scale(sc.z, mult), pbr.x, pbr.y);
    } else if (format == 2) {
        const float mn = (sc.y < sc.x) ? sc.y : sc.x;
        ply_row<2>(rows + i * 48ull, p, n, col, &rot.x, ls, log_scale(mn, mult), pbr.x, pbr.y);
    } else {
        ply_row<0>(rows + i * 248ull, p, n, col, &rot.x, ls, log_scale(sc.z, mult), pbr.x, pbr.y);
    }
}

}  // namespace

cudaError_t ply_rows_launch(const void* ref96, unsigned long long count, uint32_t format, float mult, void* rows, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((count + 255) / 256);
    ply_rows_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const float4*>(ref96), count, format, mult,
                                                reinterpret_cast<unsigned char*>(rows));
    return cudaGetLastError();
}

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
