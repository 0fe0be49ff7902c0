// m2s_host.cpp — host-only parts of the C ABI: error string, .ply header + writer.
// Byte-compatible with parsers::savePlyVector (src/parsers/parsers.cpp:232-316,339-428,431-514,
// 631-651) but written as one buffered block write per 64 Ki records instead of one 4-byte
// ofstream::write per property.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "m2s_host.h"

namespace m2s {
static thread_local std::string g_error;
void set_error(const std::string& msg) { g_error = msg; }
}  // namespace m2s

M2S_EXPORT const char* m2s_last_error(void) { return m2s::g_error.c_str(); }

M2S_EXPORT size_t m2s_ply_header(uint32_t format, uint64_t count, char* dst, size_t dst_size) {
    std::string h = "ply\nformat binary_little_endian 1.0\nelement vertex " + std::to_string(count) + "\n";
    auto prop = [&](const char* type, const std::string& name) { h += std::string("property ") + type + " " + name + "\n"; };
    if (format == 1) {  // writePbrPLY, parsers.cpp:240-266
        for (const char* n : {"x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "metallicFactor", "roughnessFactor",
                              "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"})
            prop("float", n);
    } else if (format == 2) {  // writeCompressedPbrPLY, parsers.cpp:346-368
        for (const char* n : {"x", "y", "z"}) prop("float", n);
        for (const char* n : {"red", "green", "blue", "opacity"}) prop("uint8", n);
        for (const char* n : {"rot_0", "rot_1", "rot_2", "rot_3", "scale_0", "scale_1", "scale_2"}) prop("float", n);
        for (const char* n : {"octa_nx", "octa_ny", "roughness", "metallic"}) prop("uint8", n);
    } else {  // writeBinaryPlyStandardFormat, parsers.cpp:439-466 (also the default branch, :646-648)
        for (const char* n : {"x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"}) prop("float", n);
        for (int i = 0; i <= 44; ++i) prop("float", "f_rest_" + std::to_string(i));
        for (const char* n : {"opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"}) prop("float", n);
    }
    h += "end_header\n";
    if (dst && dst_size > h.size()) std::memcpy(dst, h.c_str(), h.size() + 1);
    return h.size();
}

namespace {
inline float inv_sigmoid(float a) {  // utils.hpp:270
    a = std::min(std::max(a, 0.0f), 1.0f);
    return -std::log((1.0f / (a + 1e-8f)) - 1.0f);
}
inline uint8_t to_byte(float v) {  // parsers.cpp:370-375
    v = std::min(std::max(v, 0.0f), 1.0f);
    return (uint8_t)std::round(v * 255.0f);
}
constexpr float kC0 = 0.28209479177387814f;  // params.hpp:17

size_t row_bytes(uint32_t format) { return format == 1 ? 76 : (format == 2 ? 48 : 248); }

void encode_row(uint32_t format, const float* r, float mult, uint8_t* dst) {
    const float sh[3] = {(r[4] - 0.5f) / kC0, (r[5] - 0.5f) / kC0, (r[6] - 0.5f) / kC0};
    const float op = inv_sigmoid(r[7]);
    const float ls[3] = {std::log(r[8] * mult), std::log(r[9] * mult), std::log(r[10] * mult)};
    if (format == 1) {
        const float f[19] = {r[0], r[1], r[2], r[12], r[13], r[14], sh[0], sh[1], sh[2], r[20], r[21], op,
                             ls[0], ls[1], ls[2], r[16], r[17], r[18], r[19]};
        std::memcpy(dst, f, sizeof(f));
    } else if (format == 2) {
        std::memcpy(dst, r, 12);
        dst[12] = to_byte(r[4]); dst[13] = to_byte(r[5]); dst[14] = to_byte(r[6]); dst[15] = to_byte(r[7]);
        std::memcpy(dst + 16, r + 16, 16);
        const float mn = std::min(r[8], r[9]);  // parsers.cpp:402-406: z takes min(x,y)
        const float cs[3] = {ls[0], ls[1], std::log(mn * mult)};
        std::memcpy(dst + 32, cs, 12);
        const float s = std::fabs(r[12]) + std::fabs(r[13]) + std::fabs(r[14]) + 1e-8f;  // EncodeOcta :324-337
        const float nx = r[12] / s, ny = r[13] / s, nz = r[14] / s;
        float rx, ry;
        if (nz >= 0.0f) { rx = nx; ry = ny; }
        else { const float m = (nx >= 0.0f && ny >= 0.0f) ? 1.0f : -1.0f; rx = (1.0f - std::fabs(ny)) * m; ry = (1.0f - std::fabs(nx)) * m; }
        const float ox = rx * 0.5f + 0.5f, oy = ry * 0.5f + 0.5f;
        dst[44] = (uint8_t)std::min(std::max(std::round(ox * 255.0f), 0.0f), 255.0f);
        dst[45] = (uint8_t)std::min(std::max(std::round(oy * 255.0f), 0.0f), 255.0f);
        dst[46] = to_byte(r[21]); dst[47] = to_byte(r[20]);
    } else {
        float f[62];
        std::memset(f, 0, sizeof(f));
        f[0] = r[0]; f[1] = r[1]; f[2] = r[2]; f[3] = r[12]; f[4] = r[13]; f[5] = r[14];
        f[6] = sh[0]; f[7] = sh[1]; f[8] = sh[2];
        f[54] = op; f[55] = ls[0]; f[56] = ls[1]; f[57] = ls[2];
        f[58] = r[16]; f[59] = r[17]; f[60] = r[18]; f[61] = r[19];
        std::memcpy(dst, f, sizeof(f));
    }
}
}  // namespace

M2S_EXPORT m2s_status m2s_ply_write(const char* path, const void* h_ref96, uint64_t count, uint32_t format, float mult) {
    if (!path || (count && !h_ref96)) { m2s::set_error("m2s_ply_write: NULL argument"); return M2S_E_INVALID; }
    if (format > 2) format = 0;
    FILE* f = std::fopen(path, "wb");
    if (!f) { m2s::set_error(std::string("cannot open ") + path); return M2S_E_IO; }
    char hdr[4096];
    const size_t n = m2s_ply_header(format, count, hdr, sizeof(hdr));
    bool ok = std::fwrite(hdr, 1, n, f) == n;
    const size_t rb = row_bytes(format);
    const uint64_t kBlock = 65536;
    std::vector<uint8_t> buf((size_t)std::min<uint64_t>(count, kBlock) * rb);
    const float* rec = static_cast<const float*>(h_ref96);
    for (uint64_t i0 = 0; ok && i0 < count; i0 += kBlock) {
        const uint64_t m = std::min(kBlock, count - i0);
        for (uint64_t i = 0; i < m; ++i) encode_row(format, rec + (i0 + i) * 24, mult, buf.data() + i * rb);
        ok = std::fwrite(buf.data(), 1, (size_t)m * rb, f) == (size_t)m * rb;
    }
    ok = (std::fclose(f) == 0) && ok;
    if (!ok) { m2s::set_error(std::string("short write to ") + path); return M2S_E_IO; }
    return M2S_OK;
}
