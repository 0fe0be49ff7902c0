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
// No third-party code: own GLB/JSON reader, own inflate + PNG decoder (every colour type / depth, Adam7), own
// JPEG decoder (baseline + progressive Huffman; arithmetic / lossless / 12-bit are rejected with M2S_E_FORMAT).
#include <algorithm>
#include <chrono>
#include <exception>
#include <thread>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "m2s_host.h"

namespace {

struct FormatError : std::runtime_error {
    using std::runtime_error::runtime_error;
};

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

// ---- inflate (RFC 1951) + zlib wrapper ------------------------------------------------------------
struct BitReader {  // LSB-first bit stream (RFC 1951), 64-bit window
    const uint8_t* p; const uint8_t* end; uint64_t buf = 0; int cnt = 0;
    void refill() { while (cnt <= 56 && p < end) { buf |= (uint64_t)(*p++) << cnt; cnt += 8; } }
    uint32_t bits(int n) {
        if (cnt < n) { refill(); if (cnt < n) throw FormatError("inflate: out of input"); }
        const uint32_t v = (uint32_t)(buf & ((n == 32) ? 0xffffffffull : ((1ull << n) - 1ull)));
        buf >>= n; cnt -= n;
        return v;
    }
    void align_to_byte() { const int r = cnt & 7; buf >>= r; cnt -= r; }
};
// canonical Huffman code (lengths <= 15): a 10-bit table resolves the common codes in one look-up (index = the next
// bits of the LSB-first stream, i.e. the bit-reversed code), longer codes fall back to the canonical walk
struct Huff {
    static constexpr int kFast = 10;
    uint16_t count[16]; uint16_t symbol[288];
    uint16_t fast[1 << kFast];  // (length << 9) | symbol, 0 = not in the table
    void build(const uint8_t* len, int n) {
        std::memset(count, 0, sizeof(count));
        for (int i = 0; i < n; ++i) count[len[i]]++;
        count[0] = 0;
        uint16_t offs[16]; offs[1] = 0;
        for (int i = 1; i < 15; ++i) offs[i + 1] = offs[i] + count[i];
        for (int i = 0; i < n; ++i) if (len[i]) symbol[offs[len[i]]++] = (uint16_t)i;
        std::memset(fast, 0, sizeof(fast));
        int code = 0, index = 0;
        for (int l = 1; l <= kFast; ++l) {
            for (int k = 0; k < count[l]; ++k, ++code, ++index) {
                int rev = 0;
                for (int b = 0; b < l; ++b) rev |= ((code >> b) & 1) << (l - 1 - b);
                const uint16_t e = (uint16_t)((l << 9) | symbol[index]);
                for (int hi = rev; hi < (1 << kFast); hi += 1 << l) fast[hi] = e;
            }
            code <<= 1;
        }
    }
    int decode(BitReader& br) const {
        if (br.cnt < 15) br.refill();
        const uint16_t e = fast[br.buf & ((1u << kFast) - 1u)];
        if (e) {
            const int l = e >> 9;
            if (l > br.cnt) throw FormatError("inflate: out of input");
            br.buf >>= l; br.cnt -= l;
            return e & 511;
        }
        int code = 0, first = 0, index = 0;
        for (int len = 1; len <= 15; ++len) {
            code |= (int)br.bits(1);
            const int c = count[len];
            if (code - c < first) return symbol[index + (code - first)];
            index += c; first += c; first <<= 1; code <<= 1;
        }
        throw FormatError("inflate: bad code");
    }
};
std::vector<uint8_t> inflate_zlib(const uint8_t* src, size_t n, size_t expected) {
    if (n < 6) throw FormatError("zlib: too short");
    if ((src[0] & 0x0f) != 8 || ((src[0] << 8 | src[1]) % 31) != 0 || (src[1] & 0x20)) throw FormatError("zlib: bad header");
    BitReader br{src + 2, src + n};
    std::vector<uint8_t> out;
    out.reserve(expected);
    static const uint16_t lbase[29] = {3,4,5,6,7,8,9,10,11,13,15,17,19,23,27,31,35,43,51,59,67,83,99,115,131,163,195,227,258};
    static const uint16_t lext[29] = {0,0,0,0,0,0,0,0,1,1,1,1,2,2,2,2,3,3,3,3,4,4,4,4,5,5,5,5,0};
    static const uint16_t dbase[30] = {1,2,3,4,5,7,9,13,17,25,33,49,65,97,129,193,257,385,513,769,1025,1537,2049,3073,4097,6145,8193,12289,16385,24577};
    static const uint16_t dext[30] = {0,0,0,0,1,1,2,2,3,3,4,4,5,5,6,6,7,7,8,8,9,9,10,10,11,11,12,12,13,13};
    int last;
    do {
        last = (int)br.bits(1);
        const int type = (int)br.bits(2);
        if (type == 0) {
            br.align_to_byte();
            br.p -= br.cnt / 8;  // give whole bytes of the look-ahead window back
            br.buf = 0; br.cnt = 0;
            if (br.end - br.p < 4) throw FormatError("inflate: stored block");
            const unsigned len = br.p[0] | (br.p[1] << 8);
            br.p += 4;
            if ((size_t)(br.end - br.p) < len) throw FormatError("inflate: stored block");
            out.insert(out.end(), br.p, br.p + len);
            br.p += len;
        } else if (type == 1 || type == 2) {
            Huff hl, hd;
            uint8_t lens[320];
            if (type == 1) {
                int i = 0;
                for (; i < 144; ++i) lens[i] = 8;
                for (; i < 256; ++i) lens[i] = 9;
                for (; i < 280; ++i) lens[i] = 7;
                for (; i < 288; ++i) lens[i] = 8;
                hl.build(lens, 288);
                for (i = 0; i < 30; ++i) lens[i] = 5;
                hd.build(lens, 30);
            } else {
                const int nlen = (int)br.bits(5) + 257, ndist = (int)br.bits(5) + 1, ncode = (int)br.bits(4) + 4;
                static const uint8_t order[19] = {16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15};
                uint8_t cl[19] = {0};
                for (int i = 0; i < ncode; ++i) cl[order[i]] = (uint8_t)br.bits(3);
                Huff hc; hc.build(cl, 19);
                int idx = 0;
                while (idx < nlen + ndist) {
                    int sym = hc.decode(br);
                    if (sym < 16) lens[idx++] = (uint8_t)sym;
                    else {
                        int rep, val = 0;
                        if (sym == 16) { if (!idx) throw FormatError("inflate: repeat"); val = lens[idx - 1]; rep = 3 + (int)br.bits(2); }
                        else if (sym == 17) rep = 3 + (int)br.bits(3);
                        else rep = 11 + (int)br.bits(7);
                        if (idx + rep > nlen + ndist) throw FormatError("inflate: too many lengths");
                        while (rep--) lens[idx++] = (uint8_t)val;
                    }
                }
                hl.build(lens, nlen);
                hd.build(lens + nlen, ndist);
            }
            while (true) {
                int sym = hl.decode(br);
                if (sym < 256) { out.push_back((uint8_t)sym); }
                else if (sym == 256) break;
                else {
                    sym -= 257;
                    if (sym >= 29) throw FormatError("inflate: bad length");
                    const int len = lbase[sym] + (int)br.bits(lext[sym]);
                    const int ds = hd.decode(br);
                    if (ds >= 30) throw FormatError("inflate: bad distance");
                    const size_t dist = dbase[ds] + br.bits(dext[ds]);
                    if (dist > out.size()) throw FormatError("inflate: distance too far");
                    const size_t from = out.size() - dist, at = out.size();
                    out.resize(at + (size_t)len);
                    uint8_t* o = out.data();
                    if (dist >= (size_t)len) std::memcpy(o + at, o + from, (size_t)len);
                    else for (int i = 0; i < len; ++i) o[at + i] = o[from + i];  // overlapping run
                }
            }
        } else throw FormatError("inflate: bad block type");
    } while (!last);
    return out;
}

// ---- PNG (every colour type and bit depth, Adam7 interlace, tRNS) -> RGBA8.  16-bit samples keep their high
// byte; sub-byte gray is scaled to 0..255 (as stb_image, tinygltf's decoder, does) --------------------------
struct Image { uint32_t w = 0, h = 0; std::vector<uint8_t> rgba; };
uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

Image decode_png(const uint8_t* d, size_t n) {
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    if (n < 8 || std::memcmp(d, sig, 8)) throw FormatError("png: bad signature");
    size_t pos = 8;
    uint32_t w = 0, h = 0; int depth = 0, ctype = 0, interlace = 0;
    std::vector<uint8_t> idat, plte, trns;
    bool have_trns = false;
    while (pos + 12 <= n) {
        const uint32_t len = be32(d + pos);
        const uint8_t* type = d + pos + 4;
        const uint8_t* data = d + pos + 8;
        if (pos + 12 + (size_t)len > n) throw FormatError("png: truncated chunk");
        if (!std::memcmp(type, "IHDR", 4)) {
            if (len < 13) throw FormatError("png: bad IHDR");
            w = be32(data); h = be32(data + 4); depth = data[8]; ctype = data[9]; interlace = data[12];
        } else if (!std::memcmp(type, "PLTE", 4)) plte.assign(data, data + len);
        else if (!std::memcmp(type, "tRNS", 4)) { trns.assign(data, data + len); have_trns = true; }
        else if (!std::memcmp(type, "IDAT", 4)) idat.insert(idat.end(), data, data + len);
        else if (!std::memcmp(type, "IEND", 4)) break;
        pos += 12 + (size_t)len;
    }
    if (!w || !h || w > 32768 || h > 32768) throw FormatError("png: bad dimensions");
    int ch;
    switch (ctype) { case 0: ch = 1; break; case 2: ch = 3; break; case 3: ch = 1; break; case 4: ch = 2; break; case 6: ch = 4; break;
                     default: throw FormatError("png: bad colour type"); }
    const bool depth_ok = (ctype == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
                          (ctype == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                          ((ctype == 2 || ctype == 4 || ctype == 6) && (depth == 8 || depth == 16));
    if (!depth_ok) throw FormatError("png: bad bit depth for the colour type");
    if (interlace > 1) throw FormatError("png: bad interlace method");
    const int bpp = ch * depth;                       // bits per pixel
    const size_t fb = bpp >= 8 ? (size_t)bpp / 8 : 1;  // filter distance in bytes
    auto row_bytes = [&](uint32_t pw) { return ((size_t)pw * bpp + 7) / 8; };
    // the passes: one for a plain image, seven for Adam7 (x0, y0, dx, dy)
    static const int adam7[7][4] = {{0, 0, 8, 8}, {4, 0, 8, 8}, {0, 4, 4, 8}, {2, 0, 4, 4}, {0, 2, 2, 4}, {1, 0, 2, 2}, {0, 1, 1, 2}};
    static const int plain[1][4] = {{0, 0, 1, 1}};
    const int (*passes)[4] = interlace ? adam7 : plain;
    const int npass = interlace ? 7 : 1;
    size_t expect = 0;
    for (int k = 0; k < npass; ++k) {
        const uint32_t x0 = passes[k][0], y0 = passes[k][1], dx = passes[k][2], dy = passes[k][3];
        if (x0 >= w || y0 >= h) continue;
        const uint32_t pw = (w - x0 + dx - 1) / dx, ph = (h - y0 + dy - 1) / dy;
        expect += (row_bytes(pw) + 1) * ph;
    }
    std::vector<uint8_t> raw = inflate_zlib(idat.data(), idat.size(), expect);
    if (raw.size() < expect) throw FormatError("png: not enough pixel data");
    Image out; out.w = w; out.h = h; out.rgba.resize((size_t)w * h * 4);
    // sample k of an unfiltered row -> 8 bits: 16-bit samples keep their high byte, sub-byte GRAY samples are
    // scaled to 0..255 (x255, x85, x17) as stb_image does; palette indices stay indices
    const int gray_scale = (ctype == 0 && depth < 8) ? 255 / ((1 << depth) - 1) : 1;
    auto sample = [&](const uint8_t* row, size_t k) -> uint32_t {
        if (depth == 8) return row[k];
        if (depth == 16) return row[2 * k];
        const size_t bit = k * depth;
        return (uint32_t)(row[bit >> 3] >> (8 - depth - (bit & 7))) & ((1u << depth) - 1u);
    };
    // colour key (tRNS of gray / rgb images): compared on the stored sample (16-bit: both bytes)
    auto sample16 = [&](const uint8_t* row, size_t k) -> uint32_t {
        return depth == 16 ? ((uint32_t)row[2 * k] << 8 | row[2 * k + 1]) : sample(row, k);
    };
    auto key16 = [&](size_t i) -> uint32_t { return (uint32_t)trns[2 * i] << 8 | trns[2 * i + 1]; };
    size_t rp = 0;
    std::vector<uint8_t> cur, prev;
    for (int k = 0; k < npass; ++k) {
        const uint32_t x0 = passes[k][0], y0 = passes[k][1], dx = passes[k][2], dy = passes[k][3];
        if (x0 >= w || y0 >= h) continue;
        const uint32_t pw = (w - x0 + dx - 1) / dx, ph = (h - y0 + dy - 1) / dy;
        const size_t rb = row_bytes(pw);
        cur.assign(rb, 0); prev.assign(rb, 0);
        for (uint32_t y = 0; y < ph; ++y) {
            const uint8_t ft = raw[rp];
            const uint8_t* in = raw.data() + rp + 1;
            rp += rb + 1;
            {   // unfilter: one loop per filter type (the per-byte type test was a third of the PNG decode time)
                uint8_t* c8 = cur.data(); const uint8_t* p8 = prev.data();
                const size_t head = std::min(fb, rb);
                switch (ft) {
                    case 0: std::memcpy(c8, in, rb); break;
                    case 1: for (size_t i = 0; i < head; ++i) c8[i] = in[i];
                            for (size_t i = head; i < rb; ++i) c8[i] = (uint8_t)(in[i] + c8[i - fb]); break;
                    case 2: for (size_t i = 0; i < rb; ++i) c8[i] = (uint8_t)(in[i] + p8[i]); break;
                    case 3: for (size_t i = 0; i < head; ++i) c8[i] = (uint8_t)(in[i] + (p8[i] >> 1));
                            for (size_t i = head; i < rb; ++i) c8[i] = (uint8_t)(in[i] + ((c8[i - fb] + p8[i]) >> 1)); break;
                    case 4: for (size_t i = 0; i < head; ++i) c8[i] = (uint8_t)(in[i] + p8[i]);  // a = c = 0: the predictor is b
                            for (size_t i = head; i < rb; ++i) {
                                const int a = c8[i - fb], b = p8[i], c = p8[i - fb];
                                const int pp = a + b - c, pa = std::abs(pp - a), pb = std::abs(pp - b), pc = std::abs(pp - c);
                                c8[i] = (uint8_t)(in[i] + ((pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c)));
                            }
                            break;
                    default: throw FormatError("png: bad filter");
                }
            }
            uint8_t* orow = &out.rgba[((size_t)(y0 + y * dy) * w) * 4];
            if (depth == 8 && dx == 1 && ctype == 6) { std::memcpy(orow + (size_t)x0 * 4, cur.data(), (size_t)pw * 4); std::swap(cur, prev); continue; }
            if (depth == 8 && dx == 1 && ctype == 2 && !have_trns) {
                const uint8_t* sp = cur.data(); uint8_t* o = orow + (size_t)x0 * 4;
                for (uint32_t x = 0; x < pw; ++x, sp += 3, o += 4) { o[0] = sp[0]; o[1] = sp[1]; o[2] = sp[2]; o[3] = 255; }
                std::swap(cur, prev); continue;
            }
            for (uint32_t x = 0; x < pw; ++x) {
                uint8_t* o = orow + (size_t)(x0 + x * dx) * 4;
                const size_t s0 = (size_t)x * ch;
                switch (ctype) {
                    case 0: { const uint32_t v = sample(cur.data(), s0);
                              o[0] = o[1] = o[2] = (uint8_t)(v * gray_scale);
                              o[3] = (have_trns && trns.size() >= 2 && key16(0) == sample16(cur.data(), s0)) ? 0 : 255; break; }
                    case 2: o[0] = (uint8_t)sample(cur.data(), s0); o[1] = (uint8_t)sample(cur.data(), s0 + 1); o[2] = (uint8_t)sample(cur.data(), s0 + 2);
                            o[3] = (have_trns && trns.size() >= 6 && key16(0) == sample16(cur.data(), s0) && key16(1) == sample16(cur.data(), s0 + 1) &&
                                    key16(2) == sample16(cur.data(), s0 + 2)) ? 0 : 255; break;
                    case 3: { const size_t idx = sample(cur.data(), s0); if (idx * 3 + 2 >= plte.size()) throw FormatError("png: palette index");
                              o[0] = plte[idx * 3]; o[1] = plte[idx * 3 + 1]; o[2] = plte[idx * 3 + 2]; o[3] = idx < trns.size() ? trns[idx] : 255; break; }
                    case 4: o[0] = o[1] = o[2] = (uint8_t)sample(cur.data(), s0); o[3] = (uint8_t)sample(cur.data(), s0 + 1); break;
                    case 6: o[0] = (uint8_t)sample(cur.data(), s0); o[1] = (uint8_t)sample(cur.data(), s0 + 1); o[2] = (uint8_t)sample(cur.data(), s0 + 2);
                            o[3] = (uint8_t)sample(cur.data(), s0 + 3); break;
                }
            }
            std::swap(cur, prev);
        }
    }
    return out;
}


// ---- JPEG (baseline, extended-sequential and PROGRESSIVE DCT, 8-bit, Huffman; 1 or 3 components, any sampling
// up to 2x2, restart intervals, interleaved and per-component scans) -> RGBA8.  Arithmetic / lossless / 12-bit
// files are rejected (M2S_E_FORMAT).  IDCT: separable
// float reference form (exact to the DCT definition, rounded once); chroma upsampling: the 3:1 triangle
// filter stb_image (tinygltf's decoder) and libjpeg use.  Decoders differ by +-1..2 code values in rounding,
// inside the 2/255 colour tolerance the path states.
struct JpegDecoder {
    const uint8_t* p; const uint8_t* end;
    struct Comp { int id = 0, h = 1, v = 1, tq = 0, td = 0, ta = 0, dcpred = 0; std::vector<uint8_t> plane; int pw = 0, ph = 0;
                  int bw = 0, bh = 0, vbw = 0, vbh = 0; std::vector<short> coef; };  // coefficients in NATURAL order
    uint16_t qt[4][64]; bool have_qt[4] = {false, false, false, false};
    static constexpr int kFast = 9;
    struct HT { uint8_t bits[17]; uint8_t vals[256]; int mincode[17], maxcode[18], valptr[17]; uint16_t fast[1 << 9]; bool ok = false; } dc[4], ac[4];
    std::vector<Comp> comps; int W = 0, H = 0, restart = 0;
    uint64_t bitbuf = 0; int bitcnt = 0; bool hit_marker = false;

    static constexpr uint8_t zz[64] = {0,1,8,16,9,2,3,10,17,24,32,25,18,11,4,5,12,19,26,33,40,48,41,34,27,20,13,6,7,14,21,28,35,42,49,56,57,50,43,36,29,22,15,23,30,37,44,51,58,59,52,45,38,31,39,46,53,60,61,54,47,55,62,63};

    int u8() { if (p >= end) throw FormatError("jpeg: truncated"); return *p++; }
    int u16() { const int a = u8(); return (a << 8) | u8(); }
    void build(HT& t) {
        int code = 0, k = 0;
        std::memset(t.fast, 0xff, sizeof(t.fast));
        for (int l = 1; l <= 16; ++l) {
            t.valptr[l] = k; t.mincode[l] = code;
            if (l <= kFast)  // every 9-bit window that starts with this code resolves in one look-up
                for (int j = 0; j < t.bits[l]; ++j) {
                    const int first = (code + j) << (kFast - l);
                    if (first + (1 << (kFast - l)) > (1 << kFast)) break;  // over-subscribed table: left to the slow path's check
                    for (int f = 0; f < (1 << (kFast - l)); ++f) t.fast[first + f] = (uint16_t)((l << 8) | t.vals[k + j]);
                }
            code += t.bits[l]; k += t.bits[l];
            t.maxcode[l] = t.bits[l] ? code - 1 : -1;
            code <<= 1;
        }
        t.maxcode[17] = 0x7fffffff; t.ok = true;
    }
    // MSB-first bit window; 0xFF00 is a stuffed 0xFF, any other 0xFFxx is a marker: the stream then yields zeros and
    // p stays on the marker (the look-ahead never crosses one)
    void fill() {
        while (bitcnt <= 56) {
            unsigned b = 0;
            if (!hit_marker) {
                if (p >= end) hit_marker = true;
                else {
                    b = *p++;
                    if (b == 0xff) {
                        const int b2 = p < end ? *p : 0xd9;
                        if (b2 == 0) ++p;
                        else { hit_marker = true; --p; b = 0; }
                    }
                }
            }
            bitbuf = (bitbuf << 8) | b; bitcnt += 8;
        }
    }
    int getbit() {
        if (!bitcnt) fill();
        --bitcnt;
        return (int)((bitbuf >> bitcnt) & 1u);
    }
    int getbits(int n) {
        if (n <= 0) return 0;
        if (bitcnt < n) fill();
        bitcnt -= n;
        return (int)((bitbuf >> bitcnt) & ((1ull << n) - 1ull));
    }
    int decode(const HT& t) {
        if (bitcnt < 16) fill();
        const uint16_t e = t.fast[(bitbuf >> (bitcnt - kFast)) & ((1u << kFast) - 1u)];
        if (e != 0xffffu) { bitcnt -= e >> 8; return e & 255; }
        int code = 0;
        for (int l = 1; l <= 16; ++l) {
            code = (int)(((uint32_t)code << 1) | (uint32_t)getbit());
            if (t.maxcode[l] >= 0 && code <= t.maxcode[l] && code >= t.mincode[l]) return t.vals[t.valptr[l] + code - t.mincode[l]];
        }
        throw FormatError("jpeg: bad huffman code");
    }
    static int extend(int v, int n) { return (n && v < (1 << (n - 1))) ? v - (1 << n) + 1 : v; }
    // Inverse DCT in the fixed-point form stb_image v2.29 (tinygltf's decoder in the reference) uses, so that decoded
    // texels match the reference bit for bit: the Loeffler-Ligtenberg-Moschytz factorisation with 12-bit constants;
    // columns first (result kept with 2 extra bits: +512 >> 10), then rows (+65536 + (128 << 17)) >> 17, clamped.
    static int fx(double v) { return (int)(v * 4096.0 + 0.5); }
    struct Lane { int s[8]; };
    static void lane_idct(const int* in, int stride, int out[8]) {  // one 8-point pass; outputs are sums/differences x_k +- t_k
        // two's-complement wrap-around arithmetic (unsigned): identical to int for every valid stream, defined for garbage
        typedef uint32_t U;
        const U s0 = (U)in[0], s1 = (U)in[stride], s2 = (U)in[2 * stride], s3 = (U)in[3 * stride], s4 = (U)in[4 * stride],
                s5 = (U)in[5 * stride], s6 = (U)in[6 * stride], s7 = (U)in[7 * stride];
        auto k = [](double v) { return (U)fx(v); };
        // even part
        const U pe = (s2 + s6) * k(0.5411961);
        const U e2 = pe + s6 * k(-1.847759065), e3 = pe + s2 * k(0.765366865);
        const U e0 = (s0 + s4) * 4096u, e1 = (s0 - s4) * 4096u;
        const U x0 = e0 + e3, x3 = e0 - e3, x1 = e1 + e2, x2 = e1 - e2;
        // odd part
        const U q3 = s7 + s3, q4 = s5 + s1, q1 = s7 + s1, q2 = s5 + s3;
        const U q5 = (q3 + q4) * k(1.175875602);
        const U r1 = q5 + q1 * k(-0.899976223), r2 = q5 + q2 * k(-2.562915447);
        const U r3 = q3 * k(-1.961570560), r4 = q4 * k(-0.390180644);
        const U t3 = s1 * k(1.501321110) + r1 + r4, t2 = s3 * k(3.072711026) + r2 + r3;
        const U t1 = s5 * k(2.053119869) + r2 + r4, t0 = s7 * k(0.298631336) + r1 + r3;
        out[0] = (int)x0; out[1] = (int)x1; out[2] = (int)x2; out[3] = (int)x3; out[4] = (int)t0; out[5] = (int)t1; out[6] = (int)t2; out[7] = (int)t3;
    }
    void idct_store(const short* blk, const uint16_t* q, uint8_t* dst, int stride) {
        int d[64], v[64];
        for (int i = 0; i < 64; ++i) d[zz[i]] = (int)(short)((int)blk[zz[i]] * (int)q[i]);  // DQT is stored in zig-zag order; 16-bit product
        for (int c = 0; c < 8; ++c) {  // columns
            const int* col = d + c;
            if (!(col[8] | col[16] | col[24] | col[32] | col[40] | col[48] | col[56])) {
                const int dc = (int)((uint32_t)col[0] * 4u);
                for (int r = 0; r < 8; ++r) v[r * 8 + c] = dc;
                continue;
            }
            int o[8];
            lane_idct(col, 8, o);
            auto add = [](int a, int b2) { return (int)((uint32_t)a + (uint32_t)b2); };
            auto sub = [](int a, int b2) { return (int)((uint32_t)a - (uint32_t)b2); };
            const int x0 = add(o[0], 512), x1 = add(o[1], 512), x2 = add(o[2], 512), x3 = add(o[3], 512);
            v[0 * 8 + c] = add(x0, o[7]) >> 10; v[7 * 8 + c] = sub(x0, o[7]) >> 10;
            v[1 * 8 + c] = add(x1, o[6]) >> 10; v[6 * 8 + c] = sub(x1, o[6]) >> 10;
            v[2 * 8 + c] = add(x2, o[5]) >> 10; v[5 * 8 + c] = sub(x2, o[5]) >> 10;
            v[3 * 8 + c] = add(x3, o[4]) >> 10; v[4 * 8 + c] = sub(x3, o[4]) >> 10;
        }
        auto clamp8 = [](int x) { return (uint8_t)(x < 0 ? 0 : (x > 255 ? 255 : x)); };
        for (int r = 0; r < 8; ++r) {  // rows
            int o[8];
            lane_idct(v + r * 8, 1, o);
            auto add = [](int a, int b2) { return (int)((uint32_t)a + (uint32_t)b2); };
            auto sub = [](int a, int b2) { return (int)((uint32_t)a - (uint32_t)b2); };
            const int bias = 65536 + (128 << 17);
            const int x0 = add(o[0], bias), x1 = add(o[1], bias), x2 = add(o[2], bias), x3 = add(o[3], bias);
            uint8_t* row = dst + r * stride;
            row[0] = clamp8(add(x0, o[7]) >> 17); row[7] = clamp8(sub(x0, o[7]) >> 17);
            row[1] = clamp8(add(x1, o[6]) >> 17); row[6] = clamp8(sub(x1, o[6]) >> 17);
            row[2] = clamp8(add(x2, o[5]) >> 17); row[5] = clamp8(sub(x2, o[5]) >> 17);
            row[3] = clamp8(add(x3, o[4]) >> 17); row[4] = clamp8(sub(x3, o[4]) >> 17);
        }
    }
    // ---- entropy decoding into coefficient arrays (all scans), then dequantise + IDCT ----------------
    bool progressive = false;
    int hmax = 1, vmax = 1, mx = 0, my = 0;
    int eobrun = 0;
    void frame_setup() {
        hmax = vmax = 1;
        for (auto& c : comps) { hmax = std::max(hmax, c.h); vmax = std::max(vmax, c.v); }
        const int mcuw = 8 * hmax, mcuh = 8 * vmax;
        mx = (W + mcuw - 1) / mcuw; my = (H + mcuh - 1) / mcuh;
        for (auto& c : comps) {
            c.bw = mx * c.h; c.bh = my * c.v;                      // blocks incl. MCU padding
            c.vbw = ((W * c.h + hmax - 1) / hmax + 7) / 8;          // blocks a non-interleaved scan visits
            c.vbh = ((H * c.v + vmax - 1) / vmax + 7) / 8;
            c.pw = c.bw * 8; c.ph = c.bh * 8;
            c.coef.assign((size_t)c.bw * c.bh * 64, 0);
        }
    }
    void restart_point() {  // RSTn: byte-align, skip the marker, reset predictors and the EOB run
        bitcnt = 0; hit_marker = false;
        while (p + 1 < end && !(p[0] == 0xff && p[1] >= 0xd0 && p[1] <= 0xd7)) {
            if (p[0] == 0xff && p[1] != 0 && p[1] != 0xff) { hit_marker = true; return; }  // some other marker: scan is over
            ++p;
        }
        if (p + 1 < end) p += 2;
        for (auto& c : comps) c.dcpred = 0;
        eobrun = 0;
    }
    // one 8x8 block of one scan (T.81 F.2.2 sequential, G.1.2 progressive); coefficients in natural order
    void decode_block(Comp& c, short* blk, int Ss, int Se, int Ah, int Al) {
        if (!progressive) {
            const int t = decode(dc[c.td]);
            if (t > 15) throw FormatError("jpeg: bad DC size");
            c.dcpred += extend(getbits(t), t);
            blk[0] = (short)c.dcpred;
            for (int k = 1; k < 64;) {
                const int rs = decode(ac[c.ta]); const int r = rs >> 4, sz = rs & 15;
                if (!sz) { if (r == 15) { k += 16; continue; } break; }
                k += r; if (k > 63) throw FormatError("jpeg: bad AC run");
                blk[zz[k++]] = (short)extend(getbits(sz), sz);
            }
            return;
        }
        if (Ss == 0) {  // DC scan
            if (Ah == 0) {
                const int t = decode(dc[c.td]);
                if (t > 15) throw FormatError("jpeg: bad DC size");
                c.dcpred += extend(getbits(t), t);
                blk[0] = (short)((uint32_t)c.dcpred * (1u << Al));
            }
            else if (getbit()) blk[0] = (short)(blk[0] | (1 << Al));
            return;
        }
        const int p1 = 1 << Al, m1 = -(1 << Al);
        if (Ah == 0) {  // AC, first pass of this band
            if (eobrun > 0) { --eobrun; return; }
            for (int k = Ss; k <= Se;) {
                const int rs = decode(ac[c.ta]); const int r = rs >> 4, sz = rs & 15;
                if (sz == 0) {
                    if (r < 15) { eobrun = (1 << r) - 1; if (r) eobrun += getbits(r); break; }
                    k += 16;
                } else {
                    k += r; if (k > Se) throw FormatError("jpeg: bad AC run");
                    blk[zz[k++]] = (short)(extend(getbits(sz), sz) * p1);
                }
            }
            return;
        }
        // AC refinement: one more bit for the coefficients already non-zero, new +-1 coefficients in between
        auto refine = [&](short& v) { if (getbit() && (v & p1) == 0) v = (short)(v + (v >= 0 ? p1 : m1)); };
        int k = Ss;
        if (eobrun == 0) {
            for (; k <= Se; ++k) {
                const int rs = decode(ac[c.ta]); int r = rs >> 4; const int sz = rs & 15;
                int val = 0;
                if (sz) { if (sz != 1) throw FormatError("jpeg: bad refinement code"); val = getbit() ? p1 : m1; }
                else if (r != 15) { eobrun = 1 << r; if (r) eobrun += getbits(r); break; }
                // skip r still-zero coefficients, refining the non-zero ones passed on the way
                for (; k <= Se; ++k) {
                    short& v = blk[zz[k]];
                    if (v != 0) refine(v);
                    else if (--r < 0) break;
                }
                if (val && k <= Se) blk[zz[k]] = (short)val;
            }
        }
        if (eobrun > 0) {
            for (; k <= Se; ++k) { short& v = blk[zz[k]]; if (v != 0) refine(v); }
            --eobrun;
        }
    }
    void decode_scan(const std::vector<int>& sc, int Ss, int Se, int Ah, int Al) {
        bitcnt = 0; hit_marker = false; eobrun = 0;
        for (auto& c : comps) c.dcpred = 0;
        int rst_left = restart;
        auto tick = [&]() { if (restart && --rst_left == 0) { restart_point(); rst_left = restart; } };
        if (sc.size() == 1) {  // non-interleaved: the component's own block grid
            Comp& c = comps[sc[0]];
            const int nb = c.vbw * c.vbh;
            for (int i = 0; i < nb; ++i) {
                const int bx = i % c.vbw, by = i / c.vbw;
                decode_block(c, &c.coef[((size_t)by * c.bw + bx) * 64], Ss, Se, Ah, Al);
                if (i + 1 < nb) tick();
            }
        } else {
            for (int y = 0; y < my; ++y) for (int x = 0; x < mx; ++x) {
                for (int ci : sc) { Comp& c = comps[ci];
                    for (int by = 0; by < c.v; ++by) for (int bx = 0; bx < c.h; ++bx)
                        decode_block(c, &c.coef[((size_t)(y * c.v + by) * c.bw + (x * c.h + bx)) * 64], Ss, Se, Ah, Al);
                }
                if (!(y == my - 1 && x == mx - 1)) tick();
            }
        }
        // the scan's entropy-coded segment ends at the next marker that is not RSTn / stuffed 0xFF00
        while (p + 1 < end && !(p[0] == 0xff && p[1] != 0 && p[1] != 0xff && !(p[1] >= 0xd0 && p[1] <= 0xd7))) ++p;
    }
    Image run() {
        if (u16() != 0xffd8) throw FormatError("jpeg: no SOI");
        bool eoi = false, have_scan = false;
        while (!eoi && p < end) {
            int m = u8();
            if (m != 0xff) continue;
            while ((m = u8()) == 0xff) {}
            if (m == 0xd8 || m == 0x01 || m == 0x00 || (m >= 0xd0 && m <= 0xd7)) continue;
            if (m == 0xd9) { eoi = true; break; }
            const int len = u16();
            const uint8_t* seg_end = p + len - 2;
            if (len < 2 || seg_end > end) throw FormatError("jpeg: bad segment length");
            if (m == 0xdb) {
                while (p < seg_end) { const int pq = u8(); const int tq = pq & 15; if (tq > 3) throw FormatError("jpeg: bad DQT"); for (int i = 0; i < 64; ++i) qt[tq][i] = (uint16_t)((pq >> 4) ? u16() : u8()); have_qt[tq] = true; }
            } else if (m == 0xc4) {
                while (p < seg_end) {
                    const int tc = u8(); const int th = tc & 15; if (th > 3) throw FormatError("jpeg: bad DHT");
                    HT& t = (tc >> 4) ? ac[th] : dc[th];
                    int n = 0; t.bits[0] = 0;
                    for (int l = 1; l <= 16; ++l) { t.bits[l] = (uint8_t)u8(); n += t.bits[l]; }
                    if (n > 256) throw FormatError("jpeg: bad DHT");
                    for (int i = 0; i < n; ++i) t.vals[i] = (uint8_t)u8();
                    build(t);
                }
            } else if (m == 0xc0 || m == 0xc1 || m == 0xc2) {
                if (!comps.empty()) throw FormatError("jpeg: more than one frame");
                progressive = m == 0xc2;
                if (u8() != 8) throw FormatError("jpeg: only 8-bit samples are supported");
                H = u16(); W = u16();
                const int nc = u8();
                if (!W || !H || W > 32768 || H > 32768 || (nc != 1 && nc != 3)) throw FormatError("jpeg: unsupported frame");
                comps.resize(nc);
                for (auto& c : comps) { c.id = u8(); const int hv = u8(); c.h = hv >> 4; c.v = hv & 15; c.tq = u8(); if (c.h < 1 || c.h > 2 || c.v < 1 || c.v > 2 || c.tq > 3) throw FormatError("jpeg: unsupported sampling"); }
                if (nc == 1) { comps[0].h = comps[0].v = 1; }  // a single component is never sub-sampled (T.81 A.2.2)
                frame_setup();
            } else if (m >= 0xc3 && m <= 0xcf && m != 0xc4 && m != 0xc8 && m != 0xcc) {
                throw FormatError("jpeg: lossless / hierarchical / arithmetic JPEG is not supported");
            } else if (m == 0xdd) { restart = u16(); }
            else if (m == 0xda) {
                const int ns = u8();
                if (comps.empty() || ns < 1 || ns > (int)comps.size()) throw FormatError("jpeg: unsupported scan");
                std::vector<int> sc;
                for (int i = 0; i < ns; ++i) {
                    const int id = u8(); const int t = u8(); int found = -1;
                    for (size_t ci = 0; ci < comps.size(); ++ci) if (comps[ci].id == id) found = (int)ci;
                    if (found < 0) throw FormatError("jpeg: bad scan component");
                    if ((t >> 4) > 3 || (t & 15) > 3) throw FormatError("jpeg: bad table selector");
                    for (int prev : sc) if (prev == found) throw FormatError("jpeg: component listed twice in a scan");
                    comps[found].td = t >> 4; comps[found].ta = t & 15; sc.push_back(found);
                }
                const int Ss = u8(), Se = u8(), AhAl = u8();
                const int Ah = AhAl >> 4, Al = AhAl & 15;
                if (progressive) {
                    if (Ss > Se || Se > 63 || (Ss == 0 && Se != 0) || (Ss != 0 && ns != 1) || Al > 13) throw FormatError("jpeg: bad progressive scan");
                } else if (ns != (int)comps.size() && comps.size() != 1 && ns != 1) throw FormatError("jpeg: unsupported scan");
                for (int ci : sc) {
                    const Comp& c = comps[ci];
                    if ((!progressive || Ss == 0) && !(progressive && Ah) && !dc[c.td].ok) throw FormatError("jpeg: missing DC table");
                    if ((!progressive || Ss != 0) && !ac[c.ta].ok) throw FormatError("jpeg: missing AC table");
                }
                p = seg_end;
                decode_scan(sc, progressive ? Ss : 0, progressive ? Se : 63, progressive ? Ah : 0, progressive ? Al : 0);
                have_scan = true;
                continue;
            }
            p = seg_end;
        }
        if (comps.empty() || !have_scan) throw FormatError("jpeg: no image data");
        for (auto& c : comps) {
            if (!have_qt[c.tq]) throw FormatError("jpeg: missing quantisation table");
            c.plane.assign((size_t)c.pw * c.ph, 0);
            for (int by = 0; by < c.bh; ++by) for (int bx = 0; bx < c.bw; ++bx)
                idct_store(&c.coef[((size_t)by * c.bw + bx) * 64], qt[c.tq], c.plane.data() + ((size_t)by * 8) * c.pw + (size_t)bx * 8, c.pw);
        }
        // Chroma upsampling and colour conversion, again in stb_image's integer form (bit-identical texels):
        //   2x horizontally: out[2i] = (3 c[i] + c[i-1] + 2) >> 2, out[2i+1] = (3 c[i] + c[i+1] + 2) >> 2, ends copied
        //   2x vertically:   (3 near + far + 2) >> 2 with near = row y>>1, far = the row above (even y) / below (odd y)
        //   2x both:         t[i] = 3 near[i] + far[i];  out[2i-1] = (3 t[i-1] + t[i] + 8) >> 4, out[2i] = (3 t[i] + t[i-1] + 8) >> 4
        //   anything else:   nearest sample
        // rows/columns outside the component's valid extent (not the MCU padding) are clamped.
        std::vector<std::vector<uint8_t>> line(comps.size(), std::vector<uint8_t>((size_t)W + 8));
        Image out; out.w = (uint32_t)W; out.h = (uint32_t)H; out.rgba.resize((size_t)W * H * 4);
        for (int y = 0; y < H; ++y) {
            for (size_t ci = 0; ci < comps.size(); ++ci) {
                const Comp& c = comps[ci];
                const int sx = hmax / c.h, sy = vmax / c.v;
                const int cw = (W * c.h + hmax - 1) / hmax, chh = (H * c.v + vmax - 1) / vmax;  // valid extent of the plane
                uint8_t* o = line[ci].data();
                auto rowp = [&](int r) { r = r < 0 ? 0 : (r >= chh ? chh - 1 : r); return c.plane.data() + (size_t)r * c.pw; };
                if (sx == 1 && sy == 1) { std::memcpy(o, rowp(y), (size_t)W); continue; }
                const int ny = sy == 2 ? (y >> 1) : (sy == 1 ? y : y / sy);
                const uint8_t* near = rowp(ny);
                const uint8_t* far = sy == 2 ? rowp((y & 1) ? ny + 1 : ny - 1) : near;
                if (sx == 1 && sy == 2) {
                    for (int i = 0; i < cw && i < W; ++i) o[i] = (uint8_t)((3 * near[i] + far[i] + 2) >> 2);
                } else if (sx == 2 && sy == 1) {
                    if (cw == 1) { o[0] = o[1] = near[0]; }
                    else {
                        o[0] = near[0]; o[1] = (uint8_t)((near[0] * 3 + near[1] + 2) >> 2);
                        int i = 1;
                        for (; i < cw - 1; ++i) { const int n = 3 * near[i] + 2; o[2 * i] = (uint8_t)((n + near[i - 1]) >> 2); o[2 * i + 1] = (uint8_t)((n + near[i + 1]) >> 2); }
                        o[2 * i] = (uint8_t)((near[cw - 2] * 3 + near[cw - 1] + 2) >> 2); o[2 * i + 1] = near[cw - 1];
                    }
                } else if (sx == 2 && sy == 2) {
                    if (cw == 1) { o[0] = o[1] = (uint8_t)((3 * near[0] + far[0] + 2) >> 2); }
                    else {
                        int t1 = 3 * near[0] + far[0];
                        o[0] = (uint8_t)((t1 + 2) >> 2);
                        for (int i = 1; i < cw; ++i) {
                            const int t0 = t1;
                            t1 = 3 * near[i] + far[i];
                            o[2 * i - 1] = (uint8_t)((3 * t0 + t1 + 8) >> 4);
                            o[2 * i] = (uint8_t)((3 * t1 + t0 + 8) >> 4);
                        }
                        o[2 * cw - 1] = (uint8_t)((t1 + 2) >> 2);
                    }
                } else {
                    for (int x = 0; x < W; ++x) o[x] = near[std::min(x / sx, cw - 1)];
                }
            }
            uint8_t* orow = &out.rgba[(size_t)y * W * 4];
            if (comps.size() == 1) {
                for (int x = 0; x < W; ++x) { orow[4 * x] = orow[4 * x + 1] = orow[4 * x + 2] = line[0][x]; orow[4 * x + 3] = 255; }
            } else {
                // YCbCr -> RGB with 20 fractional bits; constants are 12-bit values shifted by 8
                auto f2f = [](float v) { return ((int)(v * 4096.0f + 0.5f)) << 8; };
                auto clamp8 = [](int v) { return (uint8_t)((unsigned)v > 255 ? (v < 0 ? 0 : 255) : v); };
                for (int x = 0; x < W; ++x) {
                    const int yf = (line[0][x] << 20) + (1 << 19);
                    const int cb = line[1][x] - 128, cr = line[2][x] - 128;
                    const int r = yf + cr * f2f(1.40200f);
                    const int g = yf + cr * -f2f(0.71414f) + (int)((unsigned)(cb * -f2f(0.34414f)) & 0xffff0000u);
                    const int b = yf + cb * f2f(1.77200f);
                    orow[4 * x] = clamp8(r >> 20); orow[4 * x + 1] = clamp8(g >> 20); orow[4 * x + 2] = clamp8(b >> 20); orow[4 * x + 3] = 255;
                }
            }
        }
        return out;
    }
};
constexpr uint8_t JpegDecoder::zz[64];

Image decode_jpeg(const uint8_t* d, size_t n) {
    JpegDecoder dec;
    dec.p = d; dec.end = d + n;
    return dec.run();
}

Image decode_image(const uint8_t* d, size_t n) {
    if (n >= 8 && d[0] == 0x89 && d[1] == 'P') return decode_png(d, n);
    if (n >= 3 && d[0] == 0xff && d[1] == 0xd8) return decode_jpeg(d, n);
    throw FormatError("unknown image format");
}

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

}  // namespace

// ---- the host scene object -------------------------------------------------------------------------
struct m2s_hscene {
    std::vector<float> triangles;
    std::vector<m2s_primitive> primitives;
    std::vector<std::string> names;
    std::vector<Image> images;
    std::vector<m2s_texture> textures;
    m2s_scene view;
};

namespace {

struct Glb {
    JValue json;
    const uint8_t* bin = nullptr;
    size_t bin_size = 0;
};

struct AccessorView { const uint8_t* data; size_t count; int componentType; std::string type; size_t avail; };

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
    r.type = a.get_str("type");
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
    {
        FILE* f = std::fopen(path, "rb");
        if (!f) { m2s::set_error(std::string("Failed to load glTF: cannot open ") + path); return M2S_E_IO; }
        std::fseek(f, 0, SEEK_END);
        const long sz = std::ftell(f);
        std::fseek(f, 0, SEEK_SET);
        file.resize(sz > 0 ? (size_t)sz : 0);
        const size_t rd = file.empty() ? 0 : std::fread(file.data(), 1, file.size(), f);
        std::fclose(f);
        if (rd != file.size()) { m2s::set_error(std::string("short read from ") + path); return M2S_E_IO; }
    }
    std::unique_ptr<m2s_hscene> hs(new m2s_hscene());
    try {
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

        // ---- scene graph -> mesh instances (SceneManager.cpp:213-283) ----
        struct Inst { int mesh; M4 world; };
        std::vector<Inst> insts;
        const JValue* nodes = g.json.get("nodes");
        const JValue* meshes = g.json.get("meshes");
        const size_t nmesh = meshes ? meshes->size() : 0;
        struct Frame { int node; M4 parent; };
        auto traverse = [&](int root) {
            std::vector<Frame> stack{{root, identity()}};
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
        };
        const JValue* scenes = g.json.get("scenes");
        if (scenes && scenes->size()) {
            int si = g.json.get_int("scene", -1);
            if (si < 0 || (size_t)si >= scenes->size()) si = 0;
            const JValue* roots = scenes->arr[si].get("nodes");
            if (roots) for (auto& r : roots->arr) traverse(r.as_int(-1));
        }
        if (insts.empty()) for (size_t i = 0; i < nmesh; ++i) insts.push_back({(int)i, identity()});

        // ---- images are decoded once and shared ----
        std::map<int, int> image_to_tex;
        // Images are decoded once each, the ones any material of a drawn primitive uses up front and IN PARALLEL (one
        // thread per image, bounded by the core count): PNG inflate / JPEG entropy decoding are the bulk of a load.
        // (tinygltf decodes every image of the file serially inside LoadBinaryFromFile.)
        struct Slot { bool ready = false; Image img; std::exception_ptr err; const uint8_t* data = nullptr; size_t len = 0; };
        const JValue* jimages = g.json.get("images");
        std::vector<Slot> slots(jimages ? jimages->size() : 0);
        auto locate = [&](int image, Slot& sl) {
            const JValue& im = jimages->arr[image];
            const int bv = im.get_int("bufferView", -1);
            const JValue* bvs = g.json.get("bufferViews");
            if (bv < 0 || !bvs || (size_t)bv >= bvs->size()) throw FormatError("image without bufferView (external uri images unsupported in .glb)");
            const JValue& v = bvs->arr[bv];
            const uint64_t off = v.get_size("byteOffset", 0), len = v.get_size("byteLength", 0);
            if (off > g.bin_size || len > g.bin_size - off) throw FormatError("image exceeds the BIN chunk");
            sl.data = g.bin + off; sl.len = len;
        };
        {
            std::vector<int> wanted;
            const JValue* mats = g.json.get("materials");
            for (const Inst& in : insts) {
                const JValue* prims = meshes->arr[in.mesh].get("primitives");
                if (!prims) continue;
                for (const JValue& pr : prims->arr) {
                    const int mi = pr.get_int("material", -1);
                    if (pr.get_int("mode", 4) != 4 || !mats || mi < 0 || (size_t)mi >= mats->size()) continue;
                    const JValue& m = mats->arr[mi];
                    const JValue* pbr = m.get("pbrMetallicRoughness");
                    const JValue* infos[3] = {pbr ? pbr->get("baseColorTexture") : nullptr, pbr ? pbr->get("metallicRoughnessTexture") : nullptr, m.get("normalTexture")};
                    for (const JValue* ti : infos) {
                        int image = -1;
                        try { image = texture_image(g, ti); } catch (const FormatError&) { image = -1; }  // reported later, in order
                        if (image >= 0 && (size_t)image < slots.size() && std::find(wanted.begin(), wanted.end(), image) == wanted.end()) wanted.push_back(image);
                    }
                }
            }
            const size_t nthreads = std::min<size_t>(wanted.size(), std::max(1u, std::thread::hardware_concurrency()));
            if (nthreads > 1) {
                std::atomic<size_t> next{0};
                auto work = [&]() {
                    for (size_t k = next.fetch_add(1); k < wanted.size(); k = next.fetch_add(1)) {
                        Slot& sl = slots[wanted[k]];
                        try { locate(wanted[k], sl);
#ifdef M2S_GLB_TIMING
                              auto t0 = std::chrono::steady_clock::now();
#endif
                              sl.img = decode_image(sl.data, sl.len);
#ifdef M2S_GLB_TIMING
                              std::fprintf(stderr, "[glb] image %d (%zu bytes) decoded in %.1f ms\n", wanted[k], sl.len, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
#endif
                        }
                        catch (...) { sl.err = std::current_exception(); }
                        sl.ready = true;
                    }
                };
                std::vector<std::thread> pool;
                for (size_t t = 0; t + 1 < nthreads; ++t) pool.emplace_back(work);
                work();
                for (auto& th : pool) th.join();
            }
        }
        auto get_texture = [&](int image) -> int {
            if (image < 0) return -1;
            auto it = image_to_tex.find(image);
            if (it != image_to_tex.end()) return it->second;
            if ((size_t)image >= slots.size()) throw FormatError("image index out of range");
            Slot& sl = slots[image];
            if (sl.ready) {
                if (sl.err) std::rethrow_exception(sl.err);
                hs->images.push_back(std::move(sl.img));
            } else {
                locate(image, sl);
                hs->images.push_back(decode_image(sl.data, sl.len));
            }
            const int idx = (int)hs->images.size() - 1;
            image_to_tex[image] = idx;
            return idx;
        };

        // ---- primitives (SceneManager.cpp:286-457) ----
        int meshCounter = 0;
        const JValue* materials = g.json.get("materials");
        for (const Inst& in : insts) {
            const JValue& mesh = meshes->arr[in.mesh];
            const M3 world3 = upper3(in.world);
            const M3 normalMatrix = inverse_transpose(world3);
            const JValue* prims = mesh.get("primitives");
            if (!prims) continue;
            for (const JValue& pr : prims->arr) {
                const int mode = pr.get_int("mode", 4);
                if (mode != 4) continue;  // non-triangle primitive skipped (:291-294)
                const JValue* attrs = pr.get("attributes");
                if (!attrs || !attrs->get("POSITION")) continue;  // (:297-300)
                std::string base = mesh.get_str("name");
                if (base.empty()) base = "mesh";
                const std::string name = base + "_" + std::to_string(meshCounter++);

                size_t nverts = 0;
                std::vector<float> hold_pos, hold_nrm, hold_uv, hold_tan;
                const float* pos = float_array(g, attrs->get("POSITION")->as_int(-1), 3, &nverts, hold_pos);
                std::vector<uint32_t> indices;
                const int ia = pr.get_int("indices", -1);
                if (ia >= 0) {
                    const AccessorView iv = accessor(g, ia);
                    const size_t es = iv.componentType == 5123 ? 2 : (iv.componentType == 5125 ? 4 : (iv.componentType == 5121 ? 1 : 0));
                    if (!es) continue;  // unsupported index type: primitive skipped (:336-339)
                    if (iv.count > iv.avail / es) throw FormatError("index accessor exceeds the BIN chunk");
                    indices.resize(iv.count);  // only after the count is known to fit the BIN chunk
                    for (size_t i = 0; i < iv.count; ++i) {
                        if (es == 2) { uint16_t v; std::memcpy(&v, iv.data + 2 * i, 2); indices[i] = v; }
                        else if (es == 4) { uint32_t v; std::memcpy(&v, iv.data + 4 * i, 4); indices[i] = v; }
                        else indices[i] = iv.data[i];
                    }
                } else { indices.resize(nverts); for (size_t i = 0; i < nverts; ++i) indices[i] = (uint32_t)i; }
                if (indices.size() < 3 || indices.size() % 3 != 0) continue;  // (:350-353)
                for (uint32_t ix : indices) if (ix >= nverts) throw FormatError("vertex index out of range");

                size_t cnt = 0;
                const float* nrm = attrs->get("NORMAL") ? float_array(g, attrs->get("NORMAL")->as_int(-1), 3, &cnt, hold_nrm) : nullptr;
                if (nrm && cnt < nverts) throw FormatError("NORMAL accessor shorter than POSITION");
                const float* uvs = attrs->get("TEXCOORD_0") ? float_array(g, attrs->get("TEXCOORD_0")->as_int(-1), 2, &cnt, hold_uv) : nullptr;
                if (uvs && cnt < nverts) throw FormatError("TEXCOORD_0 accessor shorter than POSITION");
                const float* tan = attrs->get("TANGENT") ? float_array(g, attrs->get("TANGENT")->as_int(-1), 4, &cnt, hold_tan) : nullptr;
                if (tan && cnt < nverts) throw FormatError("TANGENT accessor shorter than POSITION");

                m2s_primitive P;
                std::memset(&P, 0, sizeof(P));
                P.base_color_factor[0] = P.base_color_factor[1] = P.base_color_factor[2] = P.base_color_factor[3] = 1.0f;
                P.albedo_texture = P.normal_texture = P.metallic_roughness_texture = -1;
                const int mi = pr.get_int("material", -1);
                if (materials && mi >= 0 && (size_t)mi < materials->size()) {  // parseGltfMaterial (:99-193)
                    const JValue& m = materials->arr[mi];
                    const JValue* pbr = m.get("pbrMetallicRoughness");
                    if (pbr) {
                        const JValue* bf = pbr->get("baseColorFactor");
                        if (bf && bf->size() == 4) for (int i = 0; i < 4; ++i) P.base_color_factor[i] = (float)bf->arr[i].as_num(1);
                        P.albedo_texture = get_texture(texture_image(g, pbr->get("baseColorTexture")));
                        P.metallic_roughness_texture = get_texture(texture_image(g, pbr->get("metallicRoughnessTexture")));
                    }
                    P.normal_texture = get_texture(texture_image(g, m.get("normalTexture")));
                }

                P.first_triangle = hs->triangles.size() / M2S_FLOATS_PER_TRIANGLE;
                P.triangle_count = indices.size() / 3;
                hs->triangles.resize(hs->triangles.size() + P.triangle_count * M2S_FLOATS_PER_TRIANGLE);
                float* dst = hs->triangles.data() + P.first_triangle * M2S_FLOATS_PER_TRIANGLE;
                for (size_t i = 0; i < indices.size(); i += 3, dst += M2S_FLOATS_PER_TRIANGLE) {
                    V3 p[3], n[3]; float t4[3][4], uv[3][2];
                    for (int e = 0; e < 3; ++e) {
                        const uint32_t ix = indices[i + e];
                        p[e] = xform_point(in.world, {pos[3 * ix], pos[3 * ix + 1], pos[3 * ix + 2]});
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
                hs->primitives.push_back(P);
                hs->names.push_back(name);
            }
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
