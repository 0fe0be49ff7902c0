// m2s_prepass.cuh — arguments of the viewer prepass kernel (m2s_prepass.cu), filled by the C-ABI host code (m2s_viewer.cu).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace m2s {

struct PrepassArgs {
    float V[16], P[16], M[16];     // world -> view, view -> clip, model -> world (column-major)
    float Ninv[9];                 // inverse(mat3(M)), column-major                      (:103-109)
    float Nmat[16];                // transpose(inverse(M))                                (:119)
    float mscale2[3];              // (|M[0]|^2, |M[0]|^2, |M[1]|^2)  (sic, :96)
    float res[2], near_far[2];
    float std_dev;
    uint32_t render_mode;
    uint32_t layout;               // record layout: 0 REF96 (96 B), 1 PACKED56 (56 B)
    uint32_t fmt, ply_has_pbr;     // the reference's u_format (0 conversion, 1 loaded .ply) and u_plyHasPbr
    unsigned long long count;
    const unsigned long long* d_count;
    const unsigned char* records;
    float4* quads;
    float* depths;
    uint32_t* valid;
};

// the prepass with the mesh depth test: map is width x height floats, row 0 = window y 0 (m2s_depth.cu's output)
struct PrepassDepthArgs {
    PrepassArgs p;
    const float* map;
    uint32_t width, height;
};

cudaError_t prepass_launch(const PrepassArgs& args, cudaStream_t stream);
cudaError_t prepass_depth_launch(const PrepassDepthArgs& args, cudaStream_t stream);

}  // namespace m2s
