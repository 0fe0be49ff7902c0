// m2s_ply_read.cu — the viewer's other input (SURVEY 8 f-10): SceneManager::loadPly + parsers::loadPlyFile
// (src/utils/SceneManager.cpp:37-47, src/parsers/parsers.cpp:516-629).  A .ply file -> REF96 records (GaussianDataSSBO)
// exactly as loadPlyFile fills them; the rules and the deviations are in m2s.h.
//
// Shape: the header is parsed on the host (happly's line rules); the body goes from the file through the two pinned
// staging buffers of the context to a two-slot device staging area, and a streaming kernel decodes the raw rows into
// 96-byte records (row_stride bytes in, 96 out, bandwidth-bound).  The file read of block b+1 overlaps the copy and the
// decode of block b.
#include <sys/stat.h>

#include <cstdio>
#include <string>
#include <vector>

#include "m2s_codec.cuh"
#include "m2s_ctx.cuh"

namespace m2s {

// ---- header (host) -----------------------------------------------------------------------------------------------------
namespace {

const char* const kPlyNames[M2S_PLY_PROPS] = {"x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "metallicFactor",
                                              "roughnessFactor", "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1",
                                              "rot_2", "rot_3"};
const bool kPlyRequired[M2S_PLY_PROPS] = {true, true, true, false, false, false, true, true, true, false, false, true,
                                          true, true, true, true, true, true, true};
constexpr int kPbrProps[5] = {M2S_PLY_NX, M2S_PLY_NY, M2S_PLY_NZ, M2S_PLY_METALLIC, M2S_PLY_ROUGHNESS};

// happly's trimSpaces: ' ' off the front, ' ', '\n', '\r' off the back
std::string trim(const std::string& s) {
    size_t a = 0, b = s.size();
    while (a < b && s[a] == ' ') ++a;
    while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\n' || s[b - 1] == '\r')) --b;
    return s.substr(a, b - a);
}
// happly's tokenSplit: split on ' ', trim every token, drop empty ones
std::vector<std::string> tokens(const std::string& line) {
    std::vector<std::string> r;
    size_t cur = 0, f;
    while ((f = line.find(' ', cur)) != std::string::npos) {
        std::string t = trim(line.substr(cur, f - cur));
        if (!t.empty()) r.push_back(t);
        cur = f + 1;
    }
    std::string t = trim(line.substr(cur));
    if (!t.empty()) r.push_back(t);
    return r;
}
bool starts(const std::string& s, const char* q) { return s.compare(0, std::strlen(q), q) == 0; }
// bytes of a property type happly knows (createPropertyWithType), 0 for an unknown name
uint32_t type_bytes(const std::string& t) {
    if (t == "uchar" || t == "uint8" || t == "char" || t == "int8") return 1;
    if (t == "ushort" || t == "uint16" || t == "short" || t == "int16") return 2;
    if (t == "uint" || t == "uint32" || t == "int" || t == "int32" || t == "float" || t == "float32") return 4;
    if (t == "double" || t == "float64") return 8;
    return 0;
}
// `istringstream >> size_t` as happly reads an element count: optional sign, decimal digits up to the first other
// character; no digit gives 0, an overflow the maximum, a '-' the unsigned negation
uint64_t parse_count(const std::string& s) {
    size_t i = 0;
    bool neg = false;
    if (i < s.size() && (s[i] == '+' || s[i] == '-')) neg = s[i++] == '-';
    uint64_t v = 0;
    for (; i < s.size() && s[i] >= '0' && s[i] <= '9'; ++i) {
        const uint64_t d = (uint64_t)(s[i] - '0');
        if (v > (UINT64_MAX - d) / 10) return UINT64_MAX;
        v = v * 10 + d;
    }
    return neg ? (uint64_t)0 - v : v;
}
// a + b and a * b, false on uint64 overflow
bool add_ok(uint64_t a, uint64_t b, uint64_t& r) { r = a + b; return r >= a; }
bool mul_ok(uint64_t a, uint64_t b, uint64_t& r) { if (a && b > UINT64_MAX / a) return false; r = a * b; return true; }

struct PlyProp { std::string name; uint32_t bytes; bool is_float; };
struct PlyElement { std::string name; uint64_t count; std::vector<PlyProp> props; bool has_list = false; };

m2s_status format_error(const std::string& msg) { set_error("m2s_ply: " + msg); return M2S_E_FORMAT; }

}  // namespace

m2s_status ply_parse_header(const unsigned char* bytes, size_t size, uint64_t file_size, m2s_ply_info* info) {
    size_t pos = 0;
    bool eof = false;
    auto getline = [&](std::string& line) {   // std::getline on the bytes given: up to '\n' (consumed) or the end
        if (pos >= size) { eof = true; line.clear(); return; }
        const void* nl = std::memchr(bytes + pos, '\n', size - pos);
        const size_t end = nl ? (size_t)(static_cast<const unsigned char*>(nl) - bytes) : size;
        line.assign(reinterpret_cast<const char*>(bytes) + pos, end - pos);
        pos = nl ? end + 1 : size;
        if (!nl) eof = true;
    };
    std::string line;
    getline(line);
    if (trim(line) != "ply") return format_error("not a .ply file (the first line is not 'ply')");
    getline(line);
    {
        const std::vector<std::string> t = tokens(line);
        if (t.size() != 3 || t[0] != "format") return format_error("bad format line");
        if (t[1] == "ascii") return format_error("ascii bodies are not supported (binary_little_endian only)");
        if (t[1] == "binary_big_endian") return format_error("binary_big_endian bodies are not supported (binary_little_endian only)");
        if (t[1] != "binary_little_endian") return format_error("bad format line");
        if (t[2] != "1.0") return format_error("version other than 1.0");
    }
    std::vector<PlyElement> elems;
    bool ended = false;
    while (!eof) {
        getline(line);
        if (eof && line.empty()) break;
        if (starts(line, "comment") || starts(line, "obj_info")) continue;
        if (starts(line, "element")) {
            const std::vector<std::string> t = tokens(line);
            if (t.size() != 3) return format_error("invalid element line");
            elems.push_back({t[1], parse_count(t[2]), {}});
        } else if (starts(line, "property list")) {
            const std::vector<std::string> t = tokens(line);
            if (t.size() != 5) return format_error("invalid property list line");
            if (elems.empty()) return format_error("property list before any element");
            const uint32_t cb = type_bytes(t[2]);
            if (cb == 0 || cb == 8 || t[2] == "float" || t[2] == "float32") return format_error("unrecognized list count type " + t[2]);
            if (type_bytes(t[3]) == 0) return format_error("unknown property type " + t[3]);
            elems.back().has_list = true;
            elems.back().props.push_back({t[4], 0, false});
        } else if (starts(line, "property")) {
            const std::vector<std::string> t = tokens(line);
            if (t.size() != 3) return format_error("invalid property line");
            if (elems.empty()) return format_error("property before any element");
            const uint32_t b = type_bytes(t[1]);
            if (b == 0) return format_error("unknown property type " + t[1]);
            elems.back().props.push_back({t[2], b, t[1] == "float" || t[1] == "float32"});
        } else if (starts(line, "end_header")) {
            ended = true;
            break;
        } else {
            return format_error("unrecognized header line '" + line.substr(0, 64) + "'");
        }
    }
    if (!ended) return format_error("no end_header line in the header bytes given");
    // the first element "vertex"; the fixed-size elements before it are skipped
    uint64_t skip = 0;
    const PlyElement* v = nullptr;
    for (const PlyElement& e : elems) {
        if (e.name == "vertex") { v = &e; break; }
        if (e.has_list) return format_error("element '" + e.name + "' before 'vertex' has a list property (its size is not in the header)");
        uint64_t row = 0, bytes_e = 0;
        for (const PlyProp& p : e.props) row += p.bytes;
        if (!mul_ok(row, e.count, bytes_e) || !add_ok(skip, bytes_e, skip)) return format_error("element '" + e.name + "' is larger than 2^64 bytes");
    }
    if (!v) return format_error("no element 'vertex'");
    if (v->has_list) return format_error("element 'vertex' has a list property");
    uint64_t stride = 0;
    for (const PlyProp& p : v->props) stride += p.bytes;
    for (int k = 0; k < M2S_PLY_PROPS; ++k) {   // getProperty<float>: the first property of that name, float only
        uint64_t off = 0;
        const PlyProp* hit = nullptr;
        for (const PlyProp& p : v->props) {
            if (p.name == kPlyNames[k]) { hit = &p; break; }
            off += p.bytes;
        }
        if (!hit) {
            if (kPlyRequired[k]) return format_error(std::string("element 'vertex' has no property '") + kPlyNames[k] + "'");
            continue;
        }
        if (!hit->is_float) return format_error(std::string("property '") + kPlyNames[k] + "' is not float (happly does not narrow it)");
        info->offset[k] = (int32_t)std::min<uint64_t>(off, INT32_MAX);
    }
    if (stride > M2S_PLY_MAX_STRIDE) return format_error("vertex rows of " + std::to_string(stride) + " bytes (at most 4096 supported)");
    bool pbr = true;
    for (int k : kPbrProps) pbr = pbr && info->offset[k] >= 0;
    info->vertex_count = v->count;
    info->row_stride = (uint32_t)stride;
    info->has_pbr = (v->count == 0 || pbr) ? 1u : 0u;   // loadPlyFile compares vector sizes: 0 == 0 for an empty file
    uint64_t body = 0, end = 0;
    if (!add_ok(pos, skip, body) || !mul_ok(v->count, stride, end) || !add_ok(body, end, end))
        return format_error("vertex count " + std::to_string(v->count) + " overflows the file size");
    info->body_offset = body;
    if (end > file_size)
        return format_error("body truncated: the header needs " + std::to_string(end) + " bytes, the file has " + std::to_string(file_size));
    return M2S_OK;
}

// ---- the decode kernel -------------------------------------------------------------------------------------------------
constexpr int kDecodeThreads = 128;
constexpr uint32_t kWarpStage = 8192;   // bytes of rows one warp fetches per pass (32 rows of the standard 248-byte layout)

struct PlyDecodeArgs {
    const unsigned char* rows;
    unsigned long long count;
    uint32_t stride, rows_per_warp, has_pbr;
    int32_t off[M2S_PLY_PROPS];
    float4* out;
};

// the float at byte p of the shared stage (any alignment: odd strides and offsets)
__device__ __forceinline__ float ld_f32(const unsigned char* p) {
    if ((reinterpret_cast<uintptr_t>(p) & 3u) == 0) return *reinterpret_cast<const float*>(p);
    return __uint_as_float((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
}
__global__ void __launch_bounds__(kDecodeThreads) ply_decode_kernel(const __grid_constant__ PlyDecodeArgs a) {
    __shared__ uint4 stage[kDecodeThreads / 32][kWarpStage / 16 + 2];   // + 32 B: the span's 16-byte-aligned cover
    __shared__ unsigned long long tab[32];
    if (threadIdx.x < 32) tab[threadIdx.x] = kExp2Tab[threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned long long r0 = ((unsigned long long)blockIdx.x * (kDecodeThreads / 32) + warp) * a.rows_per_warp;
    if (r0 >= a.count) return;
    const uint32_t nrows = (uint32_t)min((unsigned long long)a.rows_per_warp, a.count - r0);
    // ---- the warp's rows: one contiguous span, fetched as the 16-byte chunks that cover it (the partial first and last
    // chunks byte by byte: nothing outside the span is read) ----
    const uintptr_t s = reinterpret_cast<uintptr_t>(a.rows + r0 * a.stride), e = s + (uintptr_t)nrows * a.stride;
    const uintptr_t lo = s & ~(uintptr_t)15;
    const uint32_t nchunks = (uint32_t)((e - lo + 15) >> 4);
    for (uint32_t i = lane; i < nchunks; i += 32) {
        const uintptr_t c = lo + (uintptr_t)i * 16;
        if (c >= s && c + 16 <= e) stage[warp][i] = __ldcs(reinterpret_cast<const uint4*>(c));
        else {
            unsigned char* d = reinterpret_cast<unsigned char*>(&stage[warp][i]);
            for (int k = 0; k < 16; ++k)
                if (c + k >= s && c + k < e) d[k] = __ldcs(reinterpret_cast<const unsigned char*>(c + k));
        }
    }
    __syncwarp();
    // ---- one row per lane: the record as parsers.cpp:577-622 fills it ----
    float4 q0, q1, q2, q3, q4, q5;
    if ((uint32_t)lane < nrows) {
        const unsigned char* row = reinterpret_cast<const unsigned char*>(stage[warp]) + (s - lo) + (size_t)lane * a.stride;
        auto f = [&](int k) { return ld_f32(row + a.off[k]); };
        q0 = make_float4(f(M2S_PLY_X), f(M2S_PLY_Y), f(M2S_PLY_Z), 1.0f);
        q1 = make_float4(sh0_decode(f(M2S_PLY_F_DC_0)), sh0_decode(f(M2S_PLY_F_DC_1)), sh0_decode(f(M2S_PLY_F_DC_2)),
                         opacity_sigmoid(f(M2S_PLY_OPACITY), tab));
        q2 = make_float4(ref_expf(f(M2S_PLY_SCALE_0), tab), ref_expf(f(M2S_PLY_SCALE_1), tab), ref_expf(f(M2S_PLY_SCALE_2), tab), 1.0f);
        q3 = a.has_pbr ? make_float4(f(M2S_PLY_NX), f(M2S_PLY_NY), f(M2S_PLY_NZ), 0.0f) : make_float4(0.f, 0.f, 0.f, 0.f);
        // glm::normalize(glm::quat(w = rot_0, x = rot_1, y = rot_2, z = rot_3)), stored (w, x, y, z)
        const float w = f(M2S_PLY_ROT_0), x = f(M2S_PLY_ROT_1), y = f(M2S_PLY_ROT_2), z = f(M2S_PLY_ROT_3);
        const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(w, w), __fmul_rn(x, x)), __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z))));
        if (len <= 0.0f) q4 = make_float4(1.f, 0.f, 0.f, 0.f);
        else {
            const float inv = __fdiv_rn(1.0f, len);
            q4 = make_float4(__fmul_rn(w, inv), __fmul_rn(x, inv), __fmul_rn(y, inv), __fmul_rn(z, inv));
        }
        q5 = a.has_pbr ? make_float4(f(M2S_PLY_METALLIC), f(M2S_PLY_ROUGHNESS), 0.0f, 0.0f) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();   // every lane has read its row: the stage takes the warp's records
    if ((uint32_t)lane < nrows) {
        float4* r = reinterpret_cast<float4*>(stage[warp]) + lane * 6;
        r[0] = q0; r[1] = q1; r[2] = q2; r[3] = q3; r[4] = q4; r[5] = q5;
    }
    __syncwarp();
    float4* dst = a.out + r0 * 6;
    const float4* src = reinterpret_cast<const float4*>(stage[warp]);
    for (uint32_t i = lane; i < nrows * 6; i += 32) __stcs(dst + i, src[i]);
}

cudaError_t ply_decode_launch(const m2s_ply_info* info, const void* d_rows, uint64_t count, void* d_ref96, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    PlyDecodeArgs a;
    std::memset(&a, 0, sizeof(a));
    a.rows = static_cast<const unsigned char*>(d_rows);
    a.count = count;
    a.stride = info->row_stride;
    a.rows_per_warp = std::min<uint32_t>(32u, kWarpStage / info->row_stride);
    a.has_pbr = info->has_pbr;
    for (int k = 0; k < M2S_PLY_PROPS; ++k) a.off[k] = info->offset[k] < 0 ? 0 : info->offset[k];   // absent: never read (has_pbr 0)
    a.out = static_cast<float4*>(d_ref96);
    const unsigned long long warps = (count + a.rows_per_warp - 1) / a.rows_per_warp;
    const unsigned long long blocks = (warps + kDecodeThreads / 32 - 1) / (kDecodeThreads / 32);
    ply_decode_kernel<<<(unsigned)blocks, kDecodeThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace m2s

using namespace m2s;

static void ply_info_clear(m2s_ply_info* info) {
    std::memset(info, 0, sizeof(*info));
    for (int k = 0; k < M2S_PLY_PROPS; ++k) info->offset[k] = -1;
}

M2S_EXPORT m2s_status m2s_ply_parse_header(const void* bytes, size_t size, uint64_t file_size, m2s_ply_info* info) {
    if (!info || (!bytes && size)) { set_error("m2s_ply_parse_header: NULL argument"); return M2S_E_INVALID; }
    ply_info_clear(info);
    m2s_ply_info tmp = *info;
    const m2s_status st = ply_parse_header(static_cast<const unsigned char*>(bytes), size, file_size, &tmp);
    if (st == M2S_OK) *info = tmp;
    return st;
}

M2S_EXPORT m2s_status m2s_ply_decode_enqueue(m2s_ctx* ctx, const m2s_ply_info* info, const void* d_rows, uint64_t count, void* d_ref96,
                                             void* stream) {
    const char* fn = "m2s_ply_decode";
    if (!ctx || !info || (count && (!d_rows || !d_ref96))) return invalid(fn, "NULL argument");
    if (info->row_stride < 1 || info->row_stride > M2S_PLY_MAX_STRIDE) return invalid(fn, "row_stride must be 1..4096");
    for (int k = 0; k < M2S_PLY_PROPS; ++k) {
        const int32_t o = info->offset[k];
        const bool needed = kPlyRequired[k] || (info->has_pbr && (k == M2S_PLY_NX || k == M2S_PLY_NY || k == M2S_PLY_NZ ||
                                                                   k == M2S_PLY_METALLIC || k == M2S_PLY_ROUGHNESS));
        if ((needed && o < 0) || (o >= 0 && (uint32_t)o + 4u > info->row_stride))
            return invalid(fn, std::string("offset of '") + kPlyNames[k] + "' outside the row");
    }
    if (count >= (1ull << 32)) return invalid(fn, "too many rows (< 2^32 supported)");
    if (!aligned_ok(fn, "the record buffer must be 16-byte aligned", {{d_ref96, 16}})) return M2S_E_INVALID;
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(ply_decode_launch(info, d_rows, count, d_ref96, pick_stream(ctx, stream)));
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_ply_read(m2s_ctx* ctx, const char* path, void* d_ref96, uint64_t capacity, m2s_ply_info* info) {
    const char* fn = "m2s_ply_read";
    if (!ctx || !path || !info) return invalid(fn, "NULL argument");
    ply_info_clear(info);
    FILE* f = std::fopen(path, "rb");
    if (!f) { set_error(std::string("m2s_ply_read: cannot open ") + path); return M2S_E_IO; }
    struct Closer { FILE* f; ~Closer() { std::fclose(f); } } closer{f};
    struct stat sb;
    if (fstat(fileno(f), &sb) != 0) { set_error(std::string("m2s_ply_read: cannot stat ") + path); return M2S_E_IO; }
    const uint64_t file_size = (uint64_t)sb.st_size;
    // the header: the first 1 MB at most (a 3DGS header is a few hundred bytes)
    std::vector<unsigned char> head((size_t)std::min<uint64_t>(file_size, 1u << 20));
    if (std::fread(head.data(), 1, head.size(), f) != head.size()) { set_error(std::string("m2s_ply_read: short read of ") + path); return M2S_E_IO; }
    m2s_status st = m2s_ply_parse_header(head.data(), head.size(), file_size, info);
    if (st != M2S_OK) return st;
    if (!d_ref96) return M2S_OK;
    const uint64_t n = info->vertex_count;
    if (capacity < n) {
        set_error("m2s_ply_read: " + std::to_string(n) + " vertices, capacity " + std::to_string(capacity));
        return M2S_E_CAPACITY;
    }
    if (!aligned_ok(fn, "the record buffer must be 16-byte aligned", {{d_ref96, 16}})) return M2S_E_INVALID;
    if (n == 0) return M2S_OK;
    CUDA_TRY(cudaSetDevice(ctx->device));
    for (int i = 0; i < 2; ++i)
        if (!ctx->h_stage[i]) CUDA_TRY(cudaMallocHost(&ctx->h_stage[i], m2s_ctx::kStageBytes));
    const uint32_t stride = info->row_stride;
    const uint64_t rows_per_block = m2s_ctx::kStageBytes / stride;
    const size_t slot_bytes = (size_t)rows_per_block * stride;
    st = grow(ctx, ctx->ply_rows, 2 * slot_bytes);
    if (st != M2S_OK) return st;
    if (fseeko(f, (off_t)info->body_offset, SEEK_SET) != 0) { set_error(std::string("m2s_ply_read: cannot seek in ") + path); return M2S_E_IO; }
    // block b: read into pinned slot b & 1 (once block b-2, which used the slot, is copied and decoded), copy to device
    // slot b & 1, decode; the read of block b+1 runs while the copy engine and the decode kernel work on block b
    const uint64_t nblocks = (n + rows_per_block - 1) / rows_per_block;
    unsigned char* d_slots = static_cast<unsigned char*>(ctx->ply_rows.p);
    cudaError_t e = cudaSuccess;
    st = M2S_OK;
    for (uint64_t b = 0; b < nblocks && e == cudaSuccess && st == M2S_OK; ++b) {
        const int slot = (int)(b & 1);
        const uint64_t first = b * rows_per_block, rows = std::min(rows_per_block, n - first);
        const size_t bytes = (size_t)rows * stride;
        if (b >= 2) e = cudaEventSynchronize(ctx->ev_chunk[slot]);
        if (e != cudaSuccess) break;
        if (std::fread(ctx->h_stage[slot], 1, bytes, f) != bytes) {
            set_error(std::string("m2s_ply_read: short read of ") + path);
            st = M2S_E_IO;
            break;
        }
        unsigned char* d = d_slots + slot * slot_bytes;
        e = cudaMemcpyAsync(d, ctx->h_stage[slot], bytes, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = ply_decode_launch(info, d, rows, static_cast<unsigned char*>(d_ref96) + first * 96, ctx->stream);
        if (e == cudaSuccess) e = cudaEventRecord(ctx->ev_chunk[slot], ctx->stream);
        if (e == cudaSuccess) ctx->ply_h2d += bytes;
    }
    const cudaError_t es = cudaStreamSynchronize(ctx->stream);   // the pinned buffers are idle before the call returns
    if (e == cudaSuccess) e = es;
    if (e != cudaSuccess) { set_error(std::string("m2s_ply_read: ") + cudaGetErrorString(e)); return M2S_E_CUDA; }
    return st;
}

M2S_EXPORT uint64_t m2s_ply_h2d_bytes(const m2s_ctx* ctx) { return ctx ? ctx->ply_h2d : 0; }
