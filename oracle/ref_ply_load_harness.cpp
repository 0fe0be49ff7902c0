// TEST INFRASTRUCTURE.  C entry point around the REFERENCE's own .ply loader: parsers::loadPlyFile
// (src/parsers/parsers.cpp:516-629, happly from thirdParty/happly.h).  oracle/build_ply_load.py compiles the reference's
// parsers.cpp and utils.cpp where they lie (with the stand-in headers oracle/build.py generates) and links them with this
// file into oracle/_ref/libm2s_refplyload.so.
//
// loadPlyFile catches its own exceptions (it prints the message and returns), so a rejected file is recognised by what
// it leaves untouched: the vector is pre-filled with one sentinel record and hasPbr with the byte 2; a load that failed
// changes neither.
#define STB_IMAGE_IMPLEMENTATION
#define STB_IMAGE_RESIZE_IMPLEMENTATION
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "parsers/parsers.hpp"

static const uint32_t kSentinel = 0x7FC0BEEFu;   // a NaN pattern no loaded value reproduces in all 24 words

// Returns -1 when the reference rejected the file, else the vertex count; the first min(count, capacity) records are
// copied to out (24 floats each) and *has_pbr receives hasPbr.
extern "C" __attribute__((visibility("default"))) int64_t ref_load_ply(const char* path, float* out, uint64_t capacity,
                                                                        int* has_pbr) {
    static_assert(sizeof(utils::GaussianDataSSBO) == 96, "GaussianDataSSBO is the 96-byte SSBO record");
    std::vector<utils::GaussianDataSSBO> v(1);
    uint32_t words[24];
    for (uint32_t& w : words) w = kSentinel;
    std::memcpy(&v[0], words, 96);
    bool pbr;
    const unsigned char two = 2;
    std::memcpy(&pbr, &two, 1);
    parsers::loadPlyFile(std::string(path), v, pbr);
    unsigned char pb;
    std::memcpy(&pb, &pbr, 1);
    if (pb == 2 && v.size() == 1 && std::memcmp(&v[0], words, 96) == 0) return -1;
    *has_pbr = pb;
    const uint64_t n = v.size();
    if (n && out) std::memcpy(out, v.data(), (size_t)std::min<uint64_t>(n, capacity) * 96);
    return (int64_t)n;
}
