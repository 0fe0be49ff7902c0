// m2s_glb.cpp — .glb -> host scene, and the file-level convert(glb, density) -> .ply surface.
//
// Re-implements the INPUT side of the path with the semantics of the reference's loader
// (src/utils/SceneManager.cpp):
//   parseGltfFile     :195-459  scene-graph traversal with world transforms (matrix or T*R*S),
//                               one output primitive per glTF primitive (name "<mesh>_<counter>"),
//                               de-indexing (u8/u16/u32 indices or sequential), positions * world,
//                               normals * normalMatrix then normalised or flat face normal,
//                               tangents * mat3(world) normalised (w kept) or per-face uv-derived
//                               tangent with handedness, TEXCOORD_0 only
//   getBufferData     :50-61    accessors are read as TIGHTLY PACKED (bufferView.byteStride is
//                               ignored) — reproduced, see DESIGN.md "quirks"
//   parseGltfMaterial :99-193   baseColorFactor, baseColor / normal / metallicRoughness textures
//   setupMeshBuffers  :468-576  per-primitive bbox = running union over primitives 0..k
//   loadTextures + glUtils::generateTextures: RGBA8 images (tinygltf forces 4 channels,
//                               thirdParty/tiny_gltf.h:2609)
// No third-party code: own GLB/JSON reader here, own PNG and JPEG decoders in m2s_image.cpp.
#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <map>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "m2s_host.h"
#include "m2s_image.h"

// ---- the host scene object -------------------------------------------------------------------------
struct m2s_hscene {
    std::vector<float> triangles;
    std::vector<m2s_primitive> primitives;
    std::vector<std::string> names;
    std::vector<m2s::Image> images;
    std::vector<m2s_texture> textures;
    m2s_scene view;
};

namespace {

using m2s::FormatError;
using m2s::Image;

// ---- minimal JSON DOM ---------------------------------------------------------------------------
struct JValue {
    enum Type { Null, Bool, Number, String, Array, Object } type = Null;
    bool b = false;
    double num = 0.0;
    std::string str;
    std::vector<JValue> arr;
    std::vector<std::pair<std::string, JValue>> obj;

    const JValue* get(const char* key) const {
        if (type != Object) return nullptr;
        for (auto& kv : obj)
            if (kv.first == key) return &kv.second;
        return nullptr;
    }
    int as_int(int dflt) const { return type == Number ? (int)num : dflt; }
    double as_num(double dflt) const { return type == Number ? num : dflt; }
    int get_int(const char* key, int dflt) const { const JValue* v = get(key); return v ? v->as_int(dflt) : dflt; }
    // byte offsets / lengths / element counts: non-negative integers below 2^53, anything else is malformed
    // (a negative double cast to size_t wraps and defeats every later range check)
    uint64_t get_size(const char* key, uint64_t dflt) const {
        const JValue* v = get(key);
        if (!v) return dflt;
        if (v->type != Number || !(v->num >= 0.0) || v->num > 9007199254740992.0 || v->num != std::floor(v->num))
            throw FormatError(std::string("'") + key + "' is not a non-negative integer");
        return (uint64_t)v->num;
    }
    std::string get_str(const char* key) const { const JValue* v = get(key); return (v && v->type == String) ? v->str : std::string(); }
    size_t size() const { return type == Array ? arr.size() : 0; }
};

struct JParser {
    const char* p;
    const char* end;
    void ws() { while (p < end && (*p == ' ' || *p == '\n' || *p == '\r' || *p == '\t')) ++p; }
    [[noreturn]] void fail(const char* what) { throw FormatError(std::string("JSON: ") + what); }
    JValue parse() { ws(); JValue v = value(0); ws(); return v; }
    JValue value(int depth) {
        if (depth > 256) fail("nesting too deep");
        ws();
        if (p >= end) fail("unexpected end");
        JValue v;
        const char c = *p;
        if (c == '{') {
            v.type = JValue::Object; ++p; ws();
            if (p < end && *p == '}') { ++p; return v; }
            while (true) {
                ws();
                if (p >= end || *p != '"') fail("expected key");
                std::string k = string();
                ws();
                if (p >= end || *p != ':') fail("expected ':'");
                ++p;
                v.obj.emplace_back(std::move(k), value(depth + 1));
                ws();
                if (p < end && *p == ',') { ++p; continue; }
                if (p < end && *p == '}') { ++p; break; }
                fail("expected ',' or '}'");
            }
        } else if (c == '[') {
            v.type = JValue::Array; ++p; ws();
            if (p < end && *p == ']') { ++p; return v; }
            while (true) {
                v.arr.push_back(value(depth + 1));
                ws();
                if (p < end && *p == ',') { ++p; continue; }
                if (p < end && *p == ']') { ++p; break; }
                fail("expected ',' or ']'");
            }
        } else if (c == '"') {
            v.type = JValue::String; v.str = string();
        } else if (c == 't' && end - p >= 4 && !std::strncmp(p, "true", 4)) { v.type = JValue::Bool; v.b = true; p += 4; }
        else if (c == 'f' && end - p >= 5 && !std::strncmp(p, "false", 5)) { v.type = JValue::Bool; v.b = false; p += 5; }
        else if (c == 'n' && end - p >= 4 && !std::strncmp(p, "null", 4)) { v.type = JValue::Null; p += 4; }
        else {
            const char* s = p;
            while (p < end && (std::strchr("+-0123456789.eE", *p) != nullptr)) ++p;
            if (s == p) fail("unexpected character");
            v.type = JValue::Number;
            v.num = std::strtod(std::string(s, p).c_str(), nullptr);
        }
        return v;
    }
    std::string string() {
        ++p;  // opening quote
        std::string out;
        while (p < end && *p != '"') {
            if (*p == '\\') {
                ++p;
                if (p >= end) fail("bad escape");
                switch (*p) {
                    case 'n': out += '\n'; break; case 't': out += '\t'; break; case 'r': out += '\r'; break;
                    case 'b': out += '\b'; break; case 'f': out += '\f'; break;
                    case 'u': {
                        if (end - p < 5) fail("bad \\u");
                        unsigned cp = (unsigned)std::strtoul(std::string(p + 1, p + 5).c_str(), nullptr, 16);
                        p += 4;
                        if (cp < 0x80) out += (char)cp;
                        else if (cp < 0x800) { out += (char)(0xC0 | (cp >> 6)); out += (char)(0x80 | (cp & 0x3F)); }
                        else { out += (char)(0xE0 | (cp >> 12)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
                        break;
                    }
                    default: out += *p;
                }
                ++p;
            } else out += *p++;
        }
        if (p >= end) fail("unterminated string");
        ++p;
        return out;
    }
};

// ---- small linear algebra (column-major, GLM conventions) ----------------------------------------
struct M4 { float m[4][4]; };  // m[col][row]
M4 identity() { M4 r; std::memset(&r, 0, sizeof(r)); for (int i = 0; i < 4; ++i) r.m[i][i] = 1.0f; return r; }
M4 mul(const M4& a, const M4& b) {
    M4 r;
    for (int c = 0; c < 4; ++c)
        for (int row = 0; row < 4; ++row) {
            float s = 0.0f;
            for (int k = 0; k < 4; ++k) s += a.m[k][row] * b.m[c][k];
            r.m[c][row] = s;
        }
    return r;
}
struct V3 { float x, y, z; };
V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
V3 operator*(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
V3 cross(V3 a, V3 b) { return {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; }
float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
V3 normalize(V3 a) { const float inv = 1.0f / std::sqrt(dot(a, a)); return a * inv; }
// glm::vec3(worldTransform * glm::vec4(p, 1)) in GLM 1.0.1's operation order (type_mat4x4.inl operator*(mat4, vec4)):
// (m0*x + m1*y) + (m2*z + m3*w) — pairwise, not left to right; checked bit for bit against the reference's own
// parser (oracle/_ref/libm2s_refloader.so, tests/test_oracle.py)
V3 xform_point(const M4& M, V3 p) {
    auto row = [&](int r) { return (M.m[0][r] * p.x + M.m[1][r] * p.y) + (M.m[2][r] * p.z + M.m[3][r] * 1.0f); };
    return {row(0), row(1), row(2)};
}
struct M3 { float m[3][3]; };
V3 mul3(const M3& M, V3 p) {
    return {M.m[0][0] * p.x + M.m[1][0] * p.y + M.m[2][0] * p.z, M.m[0][1] * p.x + M.m[1][1] * p.y + M.m[2][1] * p.z,
            M.m[0][2] * p.x + M.m[1][2] * p.y + M.m[2][2] * p.z};
}
M3 upper3(const M4& M) { M3 r; for (int c = 0; c < 3; ++c) for (int row = 0; row < 3; ++row) r.m[c][row] = M.m[c][row]; return r; }
// glm::transpose(glm::inverse(mat3)) with GLM 1.0.1's cofactors and determinant expansion (func_matrix.inl,
// compute_inverse<3,3>), so that normals match the reference bit for bit
M3 inverse_transpose(const M3& a) {
    const float (*m)[3] = a.m;  // m[column][row]
    const float det = +m[0][0] * (m[1][1] * m[2][2] - m[2][1] * m[1][2]) - m[1][0] * (m[0][1] * m[2][2] - m[2][1] * m[0][2]) +
                      m[2][0] * (m[0][1] * m[1][2] - m[1][1] * m[0][2]);
    const float id = 1.0f / det;
    float inv[3][3];  // inv[column][row]
    inv[0][0] = +(m[1][1] * m[2][2] - m[2][1] * m[1][2]) * id;
    inv[1][0] = -(m[1][0] * m[2][2] - m[2][0] * m[1][2]) * id;
    inv[2][0] = +(m[1][0] * m[2][1] - m[2][0] * m[1][1]) * id;
    inv[0][1] = -(m[0][1] * m[2][2] - m[2][1] * m[0][2]) * id;
    inv[1][1] = +(m[0][0] * m[2][2] - m[2][0] * m[0][2]) * id;
    inv[2][1] = -(m[0][0] * m[2][1] - m[2][0] * m[0][1]) * id;
    inv[0][2] = +(m[0][1] * m[1][2] - m[1][1] * m[0][2]) * id;
    inv[1][2] = -(m[0][0] * m[1][2] - m[1][0] * m[0][2]) * id;
    inv[2][2] = +(m[0][0] * m[1][1] - m[1][0] * m[0][1]) * id;
    M3 r;
    for (int c = 0; c < 3; ++c) for (int row = 0; row < 3; ++row) r.m[c][row] = inv[row][c];
    return r;
}
M4 trs(const JValue& node) {
    M4 T = identity(), R = identity(), S = identity();
    const JValue* t = node.get("translation");
    if (t && t->size() == 3) for (int i = 0; i < 3; ++i) T.m[3][i] = (float)t->arr[i].as_num(0);
    const JValue* q = node.get("rotation");
    if (q && q->size() == 4) {  // glm::mat4_cast(quat(w,x,y,z))
        const float x = (float)q->arr[0].as_num(0), y = (float)q->arr[1].as_num(0), z = (float)q->arr[2].as_num(0), w = (float)q->arr[3].as_num(1);
        const float qxx = x * x, qyy = y * y, qzz = z * z, qxz = x * z, qxy = x * y, qyz = y * z, qwx = w * x, qwy = w * y, qwz = w * z;
        R.m[0][0] = 1 - 2 * (qyy + qzz); R.m[0][1] = 2 * (qxy + qwz); R.m[0][2] = 2 * (qxz - qwy);
        R.m[1][0] = 2 * (qxy - qwz); R.m[1][1] = 1 - 2 * (qxx + qzz); R.m[1][2] = 2 * (qyz + qwx);
        R.m[2][0] = 2 * (qxz + qwy); R.m[2][1] = 2 * (qyz - qwx); R.m[2][2] = 1 - 2 * (qxx + qyy);
    }
    const JValue* s = node.get("scale");
    if (s && s->size() == 3) for (int i = 0; i < 3; ++i) S.m[i][i] = (float)s->arr[i].as_num(1);
    return mul(mul(T, R), S);
}

struct Glb {
    JValue json;
    const uint8_t* bin = nullptr;
    size_t bin_size = 0;
};

struct AccessorView { const uint8_t* data; size_t count; int componentType; size_t avail; };

AccessorView accessor(const Glb& g, int index) {
    const JValue* accs = g.json.get("accessors");
    if (!accs || index < 0 || (size_t)index >= accs->size()) throw FormatError("accessor index out of range");
    const JValue& a = accs->arr[index];
    const int bv = a.get_int("bufferView", -1);
    const JValue* bvs = g.json.get("bufferViews");
    if (!bvs || bv < 0 || (size_t)bv >= bvs->size()) throw FormatError("accessor without bufferView (sparse accessors unsupported)");
    const JValue& v = bvs->arr[bv];
    if (v.get_int("buffer", 0) != 0) throw FormatError("only the GLB-embedded buffer 0 is supported");
    const uint64_t off_v = v.get_size("byteOffset", 0), off_a = a.get_size("byteOffset", 0);
    if (off_v > g.bin_size || off_a > g.bin_size - off_v) throw FormatError("accessor offset beyond the BIN chunk");
    const size_t off = (size_t)(off_v + off_a);
    AccessorView r;
    r.data = g.bin + off; r.avail = g.bin_size - off;
    r.count = (size_t)a.get_size("count", 0);
    r.componentType = a.get_int("componentType", 0);
    return r;
}

// getBufferData<T> (SceneManager.cpp:50-61): tightly packed float arrays, stride ignored
// `holder` receives an aligned copy when the data does not start on a 4-byte boundary (invalid glTF, but the bytes
// are still read the way the reference's reinterpret_cast would read them on x86)
const float* float_array(const Glb& g, int acc, int comps, size_t* count, std::vector<float>& holder) {
    const AccessorView v = accessor(g, acc);
    if (v.componentType != 5126) throw FormatError("vertex attribute is not FLOAT (normalised integer attributes unsupported, as in the reference)");
    if (v.count > v.avail / (comps * sizeof(float))) throw FormatError("vertex attribute exceeds the BIN chunk");
    *count = v.count;
    if (reinterpret_cast<uintptr_t>(v.data) & 3u) {
        holder.resize(v.count * comps);
        std::memcpy(holder.data(), v.data, holder.size() * sizeof(float));
        return holder.data();
    }
    return reinterpret_cast<const float*>(v.data);
}

int texture_image(const Glb& g, const JValue* texinfo) {
    if (!texinfo) return -1;
    const int ti = texinfo->get_int("index", -1);
    const JValue* texs = g.json.get("textures");
    if (!texs || ti < 0 || (size_t)ti >= texs->size()) return -1;
    const int src = texs->arr[ti].get_int("source", -1);
    const JValue* imgs = g.json.get("images");
    if (!imgs || src < 0 || (size_t)src >= imgs->size()) return -1;
    return src;
}

// the primitive's material, nullptr when it has none or its index is out of range
const JValue* material(const Glb& g, const JValue& prim) {
    const JValue* mats = g.json.get("materials");
    const int mi = prim.get_int("material", -1);
    return (mats && mi >= 0 && (size_t)mi < mats->size()) ? &mats->arr[mi] : nullptr;
}

// the images of a material's baseColor, metallicRoughness and normal textures, -1 where it has none
std::array<int, 3> material_images(const Glb& g, const JValue& m) {
    const JValue* pbr = m.get("pbrMetallicRoughness");
    return {texture_image(g, pbr ? pbr->get("baseColorTexture") : nullptr),
            texture_image(g, pbr ? pbr->get("metallicRoughnessTexture") : nullptr), texture_image(g, m.get("normalTexture"))};
}

// the whole file; M2S_E_IO, with the error text set, when it cannot be opened or read
m2s_status read_file(const char* path, std::vector<uint8_t>& file) {
    FILE* f = std::fopen(path, "rb");
    if (!f) { m2s::set_error(std::string("Failed to load glTF: cannot open ") + path); return M2S_E_IO; }
    std::fseek(f, 0, SEEK_END);
    const long sz = std::ftell(f);
    std::fseek(f, 0, SEEK_SET);
    file.resize(sz > 0 ? (size_t)sz : 0);
    const size_t rd = file.empty() ? 0 : std::fread(file.data(), 1, file.size(), f);
    std::fclose(f);
    if (rd != file.size()) { m2s::set_error(std::string("short read from ") + path); return M2S_E_IO; }
    return M2S_OK;
}

// the GLB container: its first JSON chunk, parsed, and its first BIN chunk, which stays in `file`
Glb parse_container(const std::vector<uint8_t>& file) {
    if (file.size() < 20 || std::memcmp(file.data(), "glTF", 4)) throw FormatError("not a binary glTF (.glb) file");
    auto le32 = [&](size_t o) { return (uint32_t)file[o] | (uint32_t)file[o + 1] << 8 | (uint32_t)file[o + 2] << 16 | (uint32_t)file[o + 3] << 24; };
    if (le32(4) != 2) throw FormatError("unsupported glTF container version");
    const size_t total = std::min<size_t>(le32(8), file.size());
    Glb g;
    size_t pos = 12;
    bool have_json = false;
    while (pos + 8 <= total) {
        const uint32_t clen = le32(pos), ctype = le32(pos + 4);
        if (pos + 8 + (size_t)clen > total) throw FormatError("truncated chunk");
        if (ctype == 0x4E4F534A && !have_json) {
            JParser jp{reinterpret_cast<const char*>(file.data() + pos + 8), reinterpret_cast<const char*>(file.data() + pos + 8 + clen)};
            g.json = jp.parse();
            have_json = true;
        } else if (ctype == 0x004E4942 && !g.bin) { g.bin = file.data() + pos + 8; g.bin_size = clen; }
        pos += 8 + (size_t)clen;
        pos = (pos + 3) & ~(size_t)3;
    }
    if (!have_json) throw FormatError("no JSON chunk");
    return g;
}

// ---- scene graph -> mesh instances (SceneManager.cpp:213-283) ----
// the meshes the default scene's node trees draw, in pre-order, each with its world transform; every mesh once,
// untransformed, when they draw none
struct Inst { int mesh; M4 world; };
std::vector<Inst> mesh_instances(const Glb& g) {
    std::vector<Inst> insts;
    const JValue* nodes = g.json.get("nodes");
    const JValue* meshes = g.json.get("meshes");
    const size_t nmesh = meshes ? meshes->size() : 0;
    const JValue* scenes = g.json.get("scenes");
    int si = g.json.get_int("scene", -1);
    if (si < 0 || (size_t)si >= (scenes ? scenes->size() : 0)) si = 0;
    const JValue* roots = (scenes && scenes->size()) ? scenes->arr[si].get("nodes") : nullptr;
    struct Frame { int node; M4 parent; };
    if (roots) for (const JValue& root : roots->arr) {
        std::vector<Frame> stack{{root.as_int(-1), identity()}};
        size_t visited = 0;
        while (!stack.empty()) {
            Frame fr = stack.back(); stack.pop_back();
            if (!nodes || fr.node < 0 || (size_t)fr.node >= nodes->size()) continue;
            if (++visited > 4 * nodes->size() + 16) throw FormatError("node graph has a cycle");
            const JValue& nd = nodes->arr[fr.node];
            M4 local = identity();
            const JValue* mat = nd.get("matrix");
            if (mat && mat->size() == 16) { for (int c = 0; c < 4; ++c) for (int r = 0; r < 4; ++r) local.m[c][r] = (float)mat->arr[c * 4 + r].as_num(0); }
            else local = trs(nd);
            const M4 world = mul(fr.parent, local);
            const int mi = nd.get_int("mesh", -1);
            if (mi >= 0 && (size_t)mi < nmesh) insts.push_back({mi, world});
            const JValue* ch = nd.get("children");
            if (ch) for (size_t i = ch->size(); i-- > 0;) stack.push_back({ch->arr[i].as_int(-1), world});  // reversed: pre-order like the recursion
        }
    }
    if (insts.empty()) for (size_t i = 0; i < nmesh; ++i) insts.push_back({(int)i, identity()});
    return insts;
}

// ---- images are decoded once and shared ----
// The images any material of a drawn primitive uses are decoded up front and IN PARALLEL (one thread per image,
// bounded by the core count): PNG inflate / JPEG entropy decoding are the bulk of a load.  (tinygltf decodes every
// image of the file serially inside LoadBinaryFromFile.)  Only get() adds an image to the scene, so texture indices
// follow first use in primitive order, and a prefetched image's decode error surfaces only when a primitive that is
// assembled asks for that image.
struct TextureTable {
    struct Slot { bool ready = false; Image img; std::exception_ptr err; };
    const Glb& g;
    std::vector<Image>& images;  // the scene's, in texture order
    std::vector<Slot> slots;     // per glTF image
    std::map<int, int> image_to_tex;

    Image decode(int image) const {
        const JValue& im = g.json.get("images")->arr[image];
        const int bv = im.get_int("bufferView", -1);
        const JValue* bvs = g.json.get("bufferViews");
        if (bv < 0 || !bvs || (size_t)bv >= bvs->size()) throw FormatError("image without bufferView (external uri images unsupported in .glb)");
        const JValue& v = bvs->arr[bv];
        const uint64_t off = v.get_size("byteOffset", 0), len = v.get_size("byteLength", 0);
        if (off > g.bin_size || len > g.bin_size - off) throw FormatError("image exceeds the BIN chunk");
        return m2s::decode_image(g.bin + off, len);
    }
    // prefetches the images of every triangle-mode primitive with a material, including primitives that assembly
    // skips later; the calling thread is one of the min(wanted, cores) decoders, and with one decoder get() does the work
    TextureTable(const Glb& g_, const std::vector<Inst>& insts, std::vector<Image>& images_) : g(g_), images(images_) {
        const JValue* jimages = g.json.get("images");
        slots.resize(jimages ? jimages->size() : 0);
        std::vector<int> wanted;
        const JValue* meshes = g.json.get("meshes");
        for (const Inst& in : insts) {
            const JValue* prims = meshes->arr[in.mesh].get("primitives");
            if (!prims) continue;
            for (const JValue& pr : prims->arr) {
                const JValue* m = pr.get_int("mode", 4) == 4 ? material(g, pr) : nullptr;
                if (!m) continue;
                std::array<int, 3> want{-1, -1, -1};
                try { want = material_images(g, *m); } catch (const FormatError&) {}  // reported later, in order
                for (int image : want)
                    if (image >= 0 && (size_t)image < slots.size() && std::find(wanted.begin(), wanted.end(), image) == wanted.end()) wanted.push_back(image);
            }
        }
        const size_t nthreads = std::min<size_t>(wanted.size(), std::max(1u, std::thread::hardware_concurrency()));
        if (nthreads <= 1) return;
        std::atomic<size_t> next{0};
        auto work = [&]() {
            for (size_t k = next.fetch_add(1); k < wanted.size(); k = next.fetch_add(1)) {
                Slot& sl = slots[wanted[k]];
                try { sl.img = decode(wanted[k]); } catch (...) { sl.err = std::current_exception(); }
                sl.ready = true;
            }
        };
        std::vector<std::thread> pool;
        for (size_t t = 0; t + 1 < nthreads; ++t) pool.emplace_back(work);
        work();
        for (auto& th : pool) th.join();
    }
    // the texture index of glTF image `image` (-1: none), decoding the image now unless the constructor did
    int get(int image) {
        if (image < 0) return -1;
        auto it = image_to_tex.find(image);
        if (it != image_to_tex.end()) return it->second;
        if ((size_t)image >= slots.size()) throw FormatError("image index out of range");
        Slot& sl = slots[image];
        if (sl.err) std::rethrow_exception(sl.err);
        images.push_back(sl.ready ? std::move(sl.img) : decode(image));
        const int idx = (int)images.size() - 1;
        image_to_tex[image] = idx;
        return idx;
    }
};

// ---- primitives (SceneManager.cpp:286-457) ----
// the primitive's vertex indices, or false for a primitive the reference skips
bool primitive_indices(const Glb& g, const JValue& pr, size_t nverts, std::vector<uint32_t>& indices) {
    const int ia = pr.get_int("indices", -1);
    if (ia >= 0) {
        const AccessorView iv = accessor(g, ia);
        const size_t es = iv.componentType == 5123 ? 2 : (iv.componentType == 5125 ? 4 : (iv.componentType == 5121 ? 1 : 0));
        if (!es) return false;  // unsupported index type: primitive skipped (:336-339)
        if (iv.count > iv.avail / es) throw FormatError("index accessor exceeds the BIN chunk");
        indices.resize(iv.count);  // only after the count is known to fit the BIN chunk
        for (size_t i = 0; i < iv.count; ++i) {
            if (es == 2) { uint16_t v; std::memcpy(&v, iv.data + 2 * i, 2); indices[i] = v; }
            else if (es == 4) { uint32_t v; std::memcpy(&v, iv.data + 4 * i, 4); indices[i] = v; }
            else indices[i] = iv.data[i];
        }
    } else { indices.resize(nverts); for (size_t i = 0; i < nverts; ++i) indices[i] = (uint32_t)i; }
    return indices.size() >= 3 && indices.size() % 3 == 0;  // (:350-353)
}

// an optional vertex attribute, nullptr when the primitive has none
const float* optional_attribute(const Glb& g, const JValue& attrs, const char* name, int comps, size_t nverts, std::vector<float>& holder) {
    const JValue* a = attrs.get(name);
    if (!a) return nullptr;
    size_t cnt = 0;
    const float* data = float_array(g, a->as_int(-1), comps, &cnt, holder);
    if (data && cnt < nverts) throw FormatError(std::string(name) + " accessor shorter than POSITION");
    return data;
}

// one glTF primitive of a mesh instance -> one m2s_primitive and its de-indexed triangles.  The checks run in the
// reference's order (indices, index range, attribute lengths, then the material's textures): with several faults in
// a file, that order decides which one is reported.
void append_primitive(const Glb& g, const JValue& mesh, const JValue& pr, const M4& world, const M3& world3,
                      const M3& normalMatrix, TextureTable& textures, int& meshCounter, m2s_hscene& hs) {
    if (pr.get_int("mode", 4) != 4) return;  // non-triangle primitive skipped (:291-294)
    const JValue* attrs = pr.get("attributes");
    if (!attrs || !attrs->get("POSITION")) return;  // (:297-300)
    std::string base = mesh.get_str("name");
    if (base.empty()) base = "mesh";
    // the counter also advances for a primitive skipped below, as the reference's does: quad_0, quad_2 but no quad_1
    const std::string name = base + "_" + std::to_string(meshCounter++);

    size_t nverts = 0;
    std::vector<float> hold_pos, hold_nrm, hold_uv, hold_tan;
    const float* pos = float_array(g, attrs->get("POSITION")->as_int(-1), 3, &nverts, hold_pos);
    std::vector<uint32_t> indices;
    if (!primitive_indices(g, pr, nverts, indices)) return;
    for (uint32_t ix : indices) if (ix >= nverts) throw FormatError("vertex index out of range");
    const float* nrm = optional_attribute(g, *attrs, "NORMAL", 3, nverts, hold_nrm);
    const float* uvs = optional_attribute(g, *attrs, "TEXCOORD_0", 2, nverts, hold_uv);
    const float* tan = optional_attribute(g, *attrs, "TANGENT", 4, nverts, hold_tan);

    m2s_primitive P;
    std::memset(&P, 0, sizeof(P));
    P.base_color_factor[0] = P.base_color_factor[1] = P.base_color_factor[2] = P.base_color_factor[3] = 1.0f;
    P.albedo_texture = P.normal_texture = P.metallic_roughness_texture = -1;
    if (const JValue* m = material(g, pr)) {  // parseGltfMaterial (:99-193)
        const JValue* pbr = m->get("pbrMetallicRoughness");
        const JValue* bf = pbr ? pbr->get("baseColorFactor") : nullptr;
        if (bf && bf->size() == 4) for (int i = 0; i < 4; ++i) P.base_color_factor[i] = (float)bf->arr[i].as_num(1);
        const std::array<int, 3> images = material_images(g, *m);
        P.albedo_texture = textures.get(images[0]);
        P.metallic_roughness_texture = textures.get(images[1]);
        P.normal_texture = textures.get(images[2]);
    }

    P.first_triangle = hs.triangles.size() / M2S_FLOATS_PER_TRIANGLE;
    P.triangle_count = indices.size() / 3;
    hs.triangles.resize(hs.triangles.size() + P.triangle_count * M2S_FLOATS_PER_TRIANGLE);
    float* dst = hs.triangles.data() + P.first_triangle * M2S_FLOATS_PER_TRIANGLE;
    for (size_t i = 0; i < indices.size(); i += 3, dst += M2S_FLOATS_PER_TRIANGLE) {
        V3 p[3], n[3]; float t4[3][4], uv[3][2];
        for (int e = 0; e < 3; ++e) {
            const uint32_t ix = indices[i + e];
            p[e] = xform_point(world, {pos[3 * ix], pos[3 * ix + 1], pos[3 * ix + 2]});
            uv[e][0] = uvs ? uvs[2 * ix] : 0.0f; uv[e][1] = uvs ? uvs[2 * ix + 1] : 0.0f;
            if (nrm) n[e] = normalize(mul3(normalMatrix, {nrm[3 * ix], nrm[3 * ix + 1], nrm[3 * ix + 2]}));
        }
        if (!nrm) { const V3 fn = normalize(cross(p[1] - p[0], p[2] - p[0])); n[0] = n[1] = n[2] = fn; }  // (:406-413)
        if (tan) {
            for (int e = 0; e < 3; ++e) {
                const uint32_t ix = indices[i + e];
                const V3 tv = normalize(mul3(world3, {tan[4 * ix], tan[4 * ix + 1], tan[4 * ix + 2]}));
                t4[e][0] = tv.x; t4[e][1] = tv.y; t4[e][2] = tv.z; t4[e][3] = tan[4 * ix + 3];
            }
        } else {  // (:421-451)
            const V3 dp1 = p[1] - p[0], dp2 = p[2] - p[0];
            const float du1 = uv[1][0] - uv[0][0], dv1 = uv[1][1] - uv[0][1], du2 = uv[2][0] - uv[0][0], dv2 = uv[2][1] - uv[0][1];
            float det = du1 * dv2 - dv1 * du2;
            if (std::fabs(det) < 1e-8f) det = 1.0f;
            const float inv = 1.0f / det;
            V3 tg = (dp1 * dv2 - dp2 * dv1) * inv, bt = (dp2 * du1 - dp1 * du2) * inv;
            tg = normalize(tg); bt = normalize(bt);
            const V3 nn = normalize(cross(dp1, dp2));
            const float hd = dot(cross(nn, tg), bt) < 0.0f ? -1.0f : 1.0f;
            for (int e = 0; e < 3; ++e) { t4[e][0] = tg.x; t4[e][1] = tg.y; t4[e][2] = tg.z; t4[e][3] = hd; }
        }
        for (int e = 0; e < 3; ++e) {
            float* v = dst + 12 * e;
            v[0] = p[e].x; v[1] = p[e].y; v[2] = p[e].z; v[3] = n[e].x; v[4] = n[e].y; v[5] = n[e].z;
            v[6] = t4[e][0]; v[7] = t4[e][1]; v[8] = t4[e][2]; v[9] = t4[e][3]; v[10] = uv[e][0]; v[11] = uv[e][1];
        }
    }
    hs.primitives.push_back(P);
    hs.names.push_back(name);
}

}  // namespace

M2S_EXPORT void m2s_hscene_free(m2s_hscene* s) { delete s; }
M2S_EXPORT const m2s_scene* m2s_hscene_view(const m2s_hscene* s) { return s ? &s->view : nullptr; }
M2S_EXPORT const char* m2s_hscene_primitive_name(const m2s_hscene* s, uint32_t i) {
    return (s && i < s->names.size()) ? s->names[i].c_str() : "";
}

M2S_EXPORT m2s_status m2s_glb_load(const char* path, int cumulative_bbox, m2s_hscene** out) {
    if (!path || !out) { m2s::set_error("m2s_glb_load: NULL argument"); return M2S_E_INVALID; }
    *out = nullptr;
    std::vector<uint8_t> file;
    const m2s_status st = read_file(path, file);
    if (st != M2S_OK) return st;
    std::unique_ptr<m2s_hscene> hs(new m2s_hscene());
    try {
        const Glb g = parse_container(file);
        const std::vector<Inst> insts = mesh_instances(g);
        TextureTable textures(g, insts, hs->images);
        int meshCounter = 0;
        const JValue* meshes = g.json.get("meshes");
        for (const Inst& in : insts) {
            const JValue& mesh = meshes->arr[in.mesh];
            const M3 world3 = upper3(in.world);
            const M3 normalMatrix = inverse_transpose(world3);
            const JValue* prims = mesh.get("primitives");
            if (prims) for (const JValue& pr : prims->arr) append_primitive(g, mesh, pr, in.world, world3, normalMatrix, textures, meshCounter, *hs);
        }
        m2s_compute_bboxes(hs->triangles.data(), hs->primitives.data(), (uint32_t)hs->primitives.size(), cumulative_bbox);
        for (const Image& im : hs->images) hs->textures.push_back({im.rgba.data(), im.w, im.h});
    } catch (const FormatError& e) {
        m2s::set_error(std::string("Failed to load glTF: ") + e.what());
        return M2S_E_FORMAT;
    } catch (const std::bad_alloc&) {
        m2s::set_error("Failed to load glTF: out of memory");
        return M2S_E_IO;
    } catch (const std::exception& e) {  // nothing may cross the extern "C" boundary
        m2s::set_error(std::string("Failed to load glTF: ") + e.what());
        return M2S_E_FORMAT;
    }
    hs->view.triangles = hs->triangles.data();
    hs->view.triangle_count = hs->triangles.size() / M2S_FLOATS_PER_TRIANGLE;
    hs->view.primitives = hs->primitives.data();
    hs->view.primitive_count = (uint32_t)hs->primitives.size();
    hs->view.textures = hs->textures.data();
    hs->view.texture_count = (uint32_t)hs->textures.size();
    *out = hs.release();
    return M2S_OK;
}

// loadModel -> ConversionPass::execute -> exportPly in one call
M2S_EXPORT m2s_status m2s_convert_file(m2s_ctx* ctx, const char* glb_path, uint32_t resolution, float gaussian_std, uint32_t ply_format,
                                       const char* ply_path, m2s_result* result) {
    if (!ctx || !glb_path || !ply_path) { m2s::set_error("m2s_convert_file: NULL argument"); return M2S_E_INVALID; }
    if (ply_format > 2) ply_format = 0;
    m2s_hscene* hs = nullptr;
    m2s_status st = m2s_glb_load(glb_path, 1, &hs);
    if (st != M2S_OK) return st;
    m2s_params p;
    m2s_params_default(&p);
    p.resolution = resolution;
    p.gaussian_std = gaussian_std;
    p.layout = M2S_LAYOUT_PLY_STANDARD + ply_format;  // rows are encoded on the GPU and streamed to disk
    m2s_result r;
    std::memset(&r, 0, sizeof(r));
    try {
        st = m2s::convert_scene_to_ply(ctx, &hs->view, &p, ply_path, &r);
    } catch (const std::exception& e) {  // nothing may cross the extern "C" boundary
        m2s::set_error(std::string("m2s_convert_file: ") + e.what());
        st = M2S_E_IO;
    }
    m2s_hscene_free(hs);
    if (result) *result = r;
    return st;
}
