// m2s_image.h — the .glb loader's texture decoders (m2s_image.cpp).  CUDA-free, like m2s_host.h.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace m2s {
struct Image { uint32_t w = 0, h = 0; std::vector<uint8_t> rgba; };
// a PNG or JPEG file (told apart by its signature) -> RGBA8; throws FormatError on anything it cannot decode
Image decode_image(const uint8_t* d, size_t n);
}  // namespace m2s
