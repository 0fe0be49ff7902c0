// m2s_host.h — declarations shared by the C-ABI host code: the export macro, the error string and the .ply file path.
// CUDA-free: the loader (m2s_glb.cpp, m2s_image.cpp, m2s_host.cpp) also builds with plain g++
// (scripts/fuzz_loader_asan.py).
#pragma once
#include <stdexcept>
#include <string>

#include "../../include/m2s.h"

#define M2S_EXPORT extern "C" __attribute__((visibility("default")))

namespace m2s {
// a malformed input file: the loader reports it as M2S_E_FORMAT
struct FormatError : std::runtime_error { using std::runtime_error::runtime_error; };
// the text m2s_last_error returns (per thread), m2s_host.cpp
void set_error(const std::string& msg);
// scene -> .ply file: rows encoded on the GPU, streamed to disk (m2s_convert.cu)
m2s_status convert_scene_to_ply(m2s_ctx* ctx, const m2s_scene* sc, const m2s_params* p, const char* path, m2s_result* res);
}  // namespace m2s
