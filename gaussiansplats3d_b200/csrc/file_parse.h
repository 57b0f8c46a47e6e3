// file_parse.h -- host-only: header parsing and validation of `.ply` (INRIA v1, PlayCanvas compressed), `.splat` and `.spz` files for
// gs_probe_file / gs_upload_file.  Plain C++ (no CUDA) so that gs_probe_file runs without a device.  The rules restate the reference's loaders:
//   .ply    PlyParserUtils.readHeaderFromBuffer / convertHeaderTextToLines / determineHeaderFormatFromHeaderText (:222-271),
//           decodeSectionHeader (:31-130: first element only, offsets = running sum of property sizes),
//           decodeSphericalHarmonicsFromSectionHeader (:132-165), INRIAV1PlyParser.decodeHeaderLines (:18-48);
//           PlayCanvasCompressedPlyParser.decodeHeader / decodeHeaderText / readPly (:74-313) where the header selects that flavour
//   .splat  SplatParser (32-byte rows), SplatLoader (count = bytes / 32)
//   .spz    SpzLoader.deserializePackedGaussians (:255-342) on the gunzipped stream
// Every input the reference would turn into garbage (NaN centres, misplaced fields, reads past the body) is rejected here, before
// anything touches the device.
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace gs {

// logical fields of a splat record: PLY property names (BaseFieldNamesToRead + f_rest_1..44, INRIAV1PlyParser.js:7-8)
enum PlyFieldId {
    PF_X, PF_Y, PF_Z, PF_SCALE0, PF_SCALE1, PF_SCALE2, PF_ROT0, PF_ROT1, PF_ROT2, PF_ROT3, PF_DC0, PF_DC1, PF_DC2, PF_OPACITY,
    PF_RED, PF_GREEN, PF_BLUE, PF_REST0, PF_COUNT = PF_REST0 + 45
};
// PLY scalar types (PlyParserUtils.js:3-25; `char` only in PlayCanvasCompressedPlyParser's DataTypeMap); 0 = property absent
enum PlyType : uint8_t { PT_NONE = 0, PT_DOUBLE, PT_INT, PT_UINT, PT_FLOAT, PT_SHORT, PT_USHORT, PT_UCHAR, PT_CHAR };

// PlayCanvas-compressed .ply: the 18 per-chunk extremes in the order of the f64 chunk table the kernel reads
enum PcExtreme {
    PC_MIN_X, PC_MIN_Y, PC_MIN_Z, PC_MAX_X, PC_MAX_Y, PC_MAX_Z, PC_MIN_SX, PC_MIN_SY, PC_MIN_SZ, PC_MAX_SX, PC_MAX_SY, PC_MAX_SZ,
    PC_MIN_R, PC_MIN_G, PC_MIN_B, PC_MAX_R, PC_MAX_G, PC_MAX_B, PC_EXTREMES
};
static constexpr uint32_t kPcChunkSplats = 256;   // splats per PLY chunk row (decompressBaseSplat: floor(i / 256))

struct FileLayout {
    int format = 0;                       // GS_FILE_PLY / GS_FILE_SPLAT / GS_FILE_SPZ
    uint32_t count = 0;                   // splats
    uint32_t stride = 0;                  // bytes per file record (PlayCanvas: per vertex row)
    uint64_t data_offset = 0;             // first record (PlayCanvas: first vertex row)
    int sh_degree = 0;                    // the file's SH degree as loaded (0..2)
    uint32_t sh_per_channel = 0;          // f_rest count / 3 (channel stride of the f_rest_* fields)
    uint16_t offset[PF_COUNT] = {};       // byte offset of each field in the record
    uint8_t type[PF_COUNT] = {};          // PlyType, PT_NONE = absent
    // PlayCanvas-compressed .ply (pc = true): element blocks chunk, vertex, sh in that order
    bool pc = false;
    uint32_t pc_chunks = 0, pc_chunk_stride = 0;  // chunk rows, bytes per chunk row
    uint64_t pc_chunk_offset = 0, pc_sh_offset = 0;
    uint16_t pc_ext_offset[PC_EXTREMES] = {};     // byte offset of each extreme in a chunk row
    uint8_t pc_ext_type[PC_EXTREMES] = {};        // PlyType, PT_NONE = absent (colour extremes only)
    uint16_t pc_packed[4] = {};                   // offsets of packed_position, packed_rotation, packed_scale, packed_color
    uint32_t pc_sh_stride = 0;                    // uchar f_rest_* per sh row (0 without an sh element)
    int pc_sh_file_degree = 0;                    // 0..3
    uint32_t pc_color_mask = 0;                   // bit c: the chunk has both min_<c> and max_<c>
    // .spz (format 4): the decompressed packed stream, one plane per attribute for all splats
    uint32_t spz_version = 0;                     // 1: float16 positions, 2: 24-bit fixed point
    uint32_t spz_sh_coeff = 0;                    // the file's SH coefficients per channel: 0, 3, 8, 15
    double spz_pos_scale = 0.0;                   // 1.0 / (1 << fractionalBits) as JavaScript computes it
    uint64_t spz_plane[6] = {};                   // offsets of the position, alpha, colour, scale, rotation and SH planes
};
enum SpzPlane { SPZ_POS, SPZ_ALPHA, SPZ_COLOR, SPZ_SCALE, SPZ_ROT, SPZ_SH, SPZ_PLANES };
static constexpr uint32_t kSpzMagic = 0x5053474e;            // "NGSP"
static constexpr uint32_t kSpzMaxPoints = 10000000;          // SpzLoader's MAX_POINTS_TO_READ

namespace file_detail {
inline int type_of(const std::string &s, bool with_char = false) {
    static const char *names[] = {"double", "int", "uint", "float", "short", "ushort", "uchar", "char"};
    for (int i = 0; i < (with_char ? 8 : 7); ++i) if (s == names[i]) return i + 1;
    return 0;
}
inline uint32_t size_of(int t) { static const uint32_t sz[] = {0, 8, 4, 4, 4, 2, 2, 1, 1}; return sz[t]; }
inline int field_of(const std::string &name) {
    static const char *base[] = {"x", "y", "z", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3",
                                 "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "red", "green", "blue"};
    for (int i = 0; i < PF_REST0; ++i) if (name == base[i]) return i;
    if (name.compare(0, 7, "f_rest_") == 0 && name.size() > 7 && name.size() <= 9) {
        int k = 0;
        for (size_t i = 7; i < name.size(); ++i) { if (name[i] < '0' || name[i] > '9') return -1; k = 10 * k + (name[i] - '0'); }
        if (std::to_string(k) != name.substr(7)) return -1;      // no leading zeros: f_rest_01 is not f_rest_1
        if (k < 45) return PF_REST0 + k;
    }
    return -1;
}
inline std::vector<std::string> words(const std::string &line) {
    std::vector<std::string> w;
    size_t i = 0;
    while (i < line.size()) {
        while (i < line.size() && (line[i] == ' ' || line[i] == '\t')) ++i;
        size_t j = i;
        while (j < line.size() && line[j] != ' ' && line[j] != '\t') ++j;
        if (j > i) w.push_back(line.substr(i, j - i));
        i = j;
    }
    return w;
}
inline int fail_msg(char *err, size_t n, const char *fmt, ...) __attribute__((format(printf, 3, 4)));
inline int fail_msg(char *err, size_t n, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(err, n, fmt, ap);
    va_end(ap);
    return 1;
}
inline std::string trim(const std::string &s) {
    size_t a = 0, b = s.size();
    while (a < b && (s[a] == ' ' || s[a] == '\t' || s[a] == '\r' || s[a] == '\f' || s[a] == '\v')) ++a;
    while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\t' || s[b - 1] == '\r' || s[b - 1] == '\f' || s[b - 1] == '\v')) --b;
    return s.substr(a, b - a);
}
// A PLY scalar as the reference's typed-array storage holds it, as a JavaScript number (little-endian)
inline double scalar_value(const unsigned char *p, int type) {
    switch (type) {
        case PT_DOUBLE: { double v; memcpy(&v, p, 8); return v; }
        case PT_FLOAT: { float v; memcpy(&v, p, 4); return (double)v; }
        case PT_INT: { int32_t v; memcpy(&v, p, 4); return (double)v; }
        case PT_UINT: { uint32_t v; memcpy(&v, p, 4); return (double)v; }
        case PT_SHORT: { int16_t v; memcpy(&v, p, 2); return (double)v; }
        case PT_USHORT: { uint16_t v; memcpy(&v, p, 2); return (double)v; }
        case PT_UCHAR: return (double)p[0];
        case PT_CHAR: return (double)(int8_t)p[0];
        default: return 0.0;
    }
}

// PlayCanvas-compressed .ply (PlayCanvasCompressedPlyParser.decodeHeaderText :74-157, readPly :297-313).  `lines` are the trimmed
// header lines, the last one "end_header"; `data` is the first byte after it.  Every message starts with kPcPrefix.
#define kPcPrefix ".ply: PlayCanvas compressed .ply: "
inline int parse_pcply_header(const unsigned char *f, size_t bytes, const std::vector<std::string> &lines, uint64_t data, FileLayout &L,
                              char *err, size_t err_len) {
#define bad(fmt, ...) fail_msg(err, err_len, kPcPrefix fmt, ##__VA_ARGS__)
    struct Prop { std::string name; int type; uint32_t offset; };
    struct Element { std::string name; uint64_t count; uint32_t stride; std::vector<Prop> props; };
    static const char *kOrder[] = {"chunk", "vertex", "sh"};   // readPly reads these blocks in this order, whatever the header says
    static const uint32_t kMaxRow = 0xffff;                     // row offsets are 16-bit; 256 rows of both kinds stay far below 64 MiB
    if (bytes < 4 || memcmp(f, "ply\n", 4) != 0) return bad("the file does not start with 'ply\\n'");
    bool have_format = false;
    std::vector<Element> el;
    for (size_t i = 1; i + 1 < lines.size(); ++i) {
        const std::string &l = lines[i];
        const auto w = words(l);
        if (!w.empty() && w[0] == "comment") continue;   // a bare `comment` too, which the reference throws on (DESIGN §2)
        if (w.empty()) return bad("empty header line %zu", i);
        if (w[0] == "format") {
            if (w.size() != 3 || w[1] != "binary_little_endian" || w[2] != "1.0")
                return bad("format '%s' (only binary_little_endian 1.0 is supported)", l.c_str());
            have_format = true;
        } else if (w[0] == "element") {
            if (w.size() != 3 || w[2].empty() || w[2].size() > 10 || w[2].find_first_not_of("0123456789") != std::string::npos)
                return bad("malformed element line '%s'", l.c_str());
            if (el.size() == 3 || w[1] != kOrder[el.size()])
                return bad("element '%s' where '%s' is expected (elements chunk, vertex, then optionally sh)", w[1].c_str(),
                           el.size() < 3 ? kOrder[el.size()] : "end_header");
            const unsigned long long count = std::stoull(w[2]);
            if (count > 0xffffffffull) return bad("element count %s too large", w[2].c_str());
            el.push_back(Element{w[1], count, 0, {}});
        } else if (w[0] == "property") {
            if (el.empty()) return bad("property before the first element: '%s'", l.c_str());
            if (w.size() >= 2 && w[1] == "list") return bad("'property list' is not supported: '%s'", l.c_str());
            if (w.size() != 3) return bad("malformed property line '%s'", l.c_str());
            const int t = type_of(w[1], true);
            if (!t) return bad("property type '%s' unknown (char uchar short ushort int uint float double)", w[1].c_str());
            Element &e = el.back();
            for (auto &p : e.props) if (p.name == w[2]) return bad("property '%s' declared twice in element %s", w[2].c_str(), e.name.c_str());
            e.props.push_back(Prop{w[2], t, e.stride});
            e.stride += size_of(t);
            if (e.stride > kMaxRow) return bad("element %s has rows larger than %u bytes", e.name.c_str(), kMaxRow);
        } else return bad("header keyword '%s' (ply format element property comment end_header)", w[0].c_str());
    }
    if (!have_format) return bad("no 'format binary_little_endian 1.0' line");
    if (el.size() < 2) return bad("needs a chunk and a vertex element");
    auto find = [](const Element &e, const char *name) -> const Prop * {
        for (auto &p : e.props) if (p.name == name) return &p;
        return nullptr;
    };
    const Element &ch = el[0], &vx = el[1];
    static const char *kExt[PC_EXTREMES] = {"min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
                                            "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b", "max_r", "max_g", "max_b"};
    for (int k = 0; k < PC_EXTREMES; ++k) {
        const Prop *p = find(ch, kExt[k]);
        if (!p && k < PC_MIN_R) return bad("chunk property '%s' missing", kExt[k]);
        if (p) { L.pc_ext_offset[k] = (uint16_t)p->offset; L.pc_ext_type[k] = (uint8_t)p->type; }
    }
    for (int c = 0; c < 3; ++c)
        if (L.pc_ext_type[PC_MIN_R + c] && L.pc_ext_type[PC_MAX_R + c]) L.pc_color_mask |= 1u << c;
    static const char *kPacked[4] = {"packed_position", "packed_rotation", "packed_scale", "packed_color"};
    for (int k = 0; k < 4; ++k) {
        const Prop *p = find(vx, kPacked[k]);
        if (!p) return bad("vertex property '%s' missing", kPacked[k]);
        if (p->type != PT_UINT) return bad("vertex property '%s' must be a uint", kPacked[k]);
        L.pc_packed[k] = (uint16_t)p->offset;
    }
    const uint64_t n = vx.count;
    if (ch.count < (n + kPcChunkSplats - 1) / kPcChunkSplats)
        return bad("%llu chunk rows for %llu splats (need ceil(n / 256) = %llu)", (unsigned long long)ch.count, (unsigned long long)n,
                   (unsigned long long)((n + kPcChunkSplats - 1) / kPcChunkSplats));
    uint32_t nsh = 0;
    if (el.size() == 3) {
        const Element &sh = el[2];
        nsh = (uint32_t)sh.props.size();
        if (sh.count != n) return bad("sh element has %llu rows for %llu splats", (unsigned long long)sh.count, (unsigned long long)n);
        if (nsh != 9 && nsh != 24 && nsh != 45) return bad("sh element has %u properties (expected 9, 24 or 45)", nsh);
        for (uint32_t k = 0; k < nsh; ++k) {
            if (sh.props[k].name != "f_rest_" + std::to_string(k)) return bad("sh properties must be f_rest_0 .. f_rest_%u in order", nsh - 1);
            if (sh.props[k].type != PT_UCHAR) return bad("sh property '%s' must be a uchar", sh.props[k].name.c_str());
        }
    }
    // strides < 64 KiB and counts < 2^32: every product below fits in 64 bits
    const uint64_t need = ch.count * ch.stride + n * vx.stride + n * nsh;
    if (need > bytes - data)
        return bad("body holds %llu bytes, shorter than its chunk, vertex and sh blocks (%llu bytes)", (unsigned long long)(bytes - data),
                   (unsigned long long)need);
    L.format = 1;
    L.pc = true;
    L.count = (uint32_t)n;
    L.stride = vx.stride;
    L.pc_chunks = (uint32_t)ch.count;
    L.pc_chunk_stride = ch.stride;
    L.pc_chunk_offset = data;
    L.data_offset = data + ch.count * ch.stride;
    L.pc_sh_offset = L.data_offset + n * vx.stride;
    L.pc_sh_stride = nsh;
    L.pc_sh_file_degree = nsh >= 45 ? 3 : (nsh >= 24 ? 2 : (nsh >= 9 ? 1 : 0));
    L.sh_degree = std::min(L.pc_sh_file_degree, 2);
    return 0;
#undef bad
}
#undef kPcPrefix

// The f64 chunk table [ceil(count / 256)][PC_EXTREMES] of a parsed PlayCanvas file; absent colour extremes are 0 (never read).
inline std::vector<double> pc_chunk_table(const unsigned char *f, const FileLayout &L) {
    const size_t rows = ((size_t)L.count + kPcChunkSplats - 1) / kPcChunkSplats;
    std::vector<double> t(rows * PC_EXTREMES, 0.0);
    for (size_t r = 0; r < rows; ++r) {
        const unsigned char *row = f + L.pc_chunk_offset + r * L.pc_chunk_stride;
        for (int k = 0; k < PC_EXTREMES; ++k)
            if (L.pc_ext_type[k]) t[r * PC_EXTREMES + k] = scalar_value(row + L.pc_ext_offset[k], L.pc_ext_type[k]);
    }
    return t;
}
} // namespace file_detail

// Returns 0 (GS_OK) or 1 (GS_ERR_BAD_ARG) with a message in err.
inline int parse_ply_header(const unsigned char *f, size_t bytes, FileLayout &L, char *err, size_t err_len) {
    using namespace file_detail;
#define bad(...) file_detail::fail_msg(err, err_len, __VA_ARGS__)
    static const char kEnd[] = "end_header";
    const size_t kEndLen = sizeof(kEnd) - 1;
    // the data starts right after the first "end_header" and one '\n' (INRIAV1PlyParser.decodeHeaderText :55)
    size_t end = (size_t)-1;
    for (size_t i = 0; i + kEndLen <= bytes; ++i)
        if (f[i] == 'e' && memcmp(f + i, kEnd, kEndLen) == 0) { end = i; break; }
    if (end == (size_t)-1) return bad(".ply: no end_header line");
    for (size_t i = 0; i < end + kEndLen; ++i)
        if (f[i] >= 0x80) return bad(".ply: header byte %zu is not ASCII", i);
    if (end + kEndLen >= bytes || f[end + kEndLen] != '\n') return bad(".ply: end_header must be followed by a single '\\n'");
    const std::string text((const char *)f, end + kEndLen);
    std::vector<std::string> lines;
    for (size_t a = 0; a <= text.size();) {
        size_t b = text.find('\n', a);
        if (b == std::string::npos) b = text.size();
        lines.push_back(trim(text.substr(a, b - a)));
        a = b + 1;
    }
    if (lines.back() != kEnd) return bad(".ply: end_header is not on a line of its own");
    // other PLY flavours the reference dispatches to other parsers (determineHeaderFormatFromHeaderText :257-271)
    int other = 0;
    for (auto &l : lines) {
        if (l.compare(0, 13, "element chunk") == 0 || l.find("packed_") != std::string::npos) other = 1;
        else if (l.compare(0, 24, "element codebook_centers") == 0) other = 2;
    }
    if (other == 1) return parse_pcply_header(f, bytes, lines, end + kEndLen + 1, L, err, err_len);
    if (other == 2) return bad(".ply: INRIA v2 (codebook) .ply is not supported");
    bool have_format = false;
    int element = 0;                              // 0 before the first element, 1 inside it, 2 after it
    long long count = -1;
    uint32_t stride = 0;
    std::vector<std::string> names;
    uint32_t rest = 0, rest_lines = 0;
    for (size_t i = 0; i + 1 < lines.size(); ++i) {
        const std::string &l = lines[i];
        if (l.find("f_rest_") != std::string::npos) ++rest_lines;
        const auto w = words(l);
        if (w.empty()) continue;
        if (w[0] == "format") {
            if (w.size() != 3 || w[1] != "binary_little_endian" || w[2] != "1.0")
                return bad(".ply: format '%s' (only binary_little_endian 1.0 is supported)", l.c_str());
            have_format = true;
        } else if (w[0] == "element") {
            if (element == 0) {
                if (w.size() != 3 || w[2].empty() || w[2].size() > 10 || w[2].find_first_not_of("0123456789") != std::string::npos)
                    return bad(".ply: malformed element line '%s'", l.c_str());
                count = std::stoll(w[2]);
                if (count > 0xffffffffll) return bad(".ply: element count %s too large", w[2].c_str());
                element = 1;
            } else element = 2;
        } else if (w[0] == "property") {
            if (element == 0) return bad(".ply: property before the first element: '%s'", l.c_str());
            if (element == 2) continue;           // properties of later elements: ignored like the reference ignores them
            if (w.size() >= 2 && w[1] == "list") return bad(".ply: 'property list' is not supported: '%s'", l.c_str());
            if (w.size() != 3) return bad(".ply: malformed property line '%s'", l.c_str());
            const int t = type_of(w[1]);
            if (!t) return bad(".ply: property type '%s' unknown (double int uint float short ushort uchar)", w[1].c_str());
            for (auto &n : names) if (n == w[2]) return bad(".ply: property '%s' declared twice", w[2].c_str());
            names.push_back(w[2]);
            const int fid = field_of(w[2]);
            if (w[2].compare(0, 6, "f_rest") == 0) ++rest;
            if (fid >= 0) {
                if (t == PT_DOUBLE) return bad(".ply: property '%s' is a double (not read by the loader)", w[2].c_str());
                if (stride > 0xffff) return bad(".ply: property '%s' lies beyond 64 KiB into the record", w[2].c_str());
                L.offset[fid] = (uint16_t)stride;
                L.type[fid] = (uint8_t)t;
            }
            stride += size_of(t);
            if (stride > (1u << 20)) return bad(".ply: records larger than 1 MiB");
        }
    }
    if (!have_format) return bad(".ply: no 'format binary_little_endian 1.0' line");
    if (element == 0) return bad(".ply: no element");
    if (stride == 0) return bad(".ply: the first element has no properties");
    for (int k : {PF_X, PF_Y, PF_Z}) if (!L.type[k]) return bad(".ply: missing property x, y or z");
    for (int k : {PF_ROT0, PF_ROT1, PF_ROT2, PF_ROT3}) if (!L.type[k]) return bad(".ply: missing property rot_0..rot_3");
    auto group = [&](int a, int n, const char *what) {
        int have = 0;
        for (int k = a; k < a + n; ++k) have += L.type[k] != PT_NONE;
        return have == 0 || have == n ? 0 : bad(".ply: incomplete property group %s", what);
    };
    if (group(PF_SCALE0, 3, "scale_0..scale_2") || group(PF_DC0, 3, "f_dc_0..f_dc_2") || group(PF_RED, 3, "red/green/blue")) return 1;
    if (rest != 0 && rest != 9 && rest != 24 && rest != 45) return bad(".ply: %u f_rest properties (expected 0, 9, 24 or 45)", rest);
    for (uint32_t k = 0; k < rest; ++k)
        if (!L.type[PF_REST0 + k]) return bad(".ply: f_rest properties must be f_rest_0 .. f_rest_%u", rest - 1);
    if (rest_lines != rest) return bad(".ply: 'f_rest_' appears on header lines other than the first element's properties");
    L.format = 1;
    L.count = (uint32_t)count;
    L.stride = stride;
    L.data_offset = end + kEndLen + 1;
    L.sh_per_channel = rest / 3;
    L.sh_degree = L.sh_per_channel >= 8 ? 2 : (L.sh_per_channel >= 3 ? 1 : 0);
    if ((unsigned long long)L.stride * L.count > bytes - L.data_offset)
        return bad(".ply: body holds %llu bytes, shorter than %u splats x %u-byte records", (unsigned long long)(bytes - L.data_offset), L.count, L.stride);
    return 0;
#undef bad
}

// .spz: the packed stream SpzLoader.deserializePackedGaussians reads once it has gunzipped the file (the caller inflates it).  A 16-byte
// header (magic, version, numPoints u32; shDegree, fractionalBits, flags, reserved u8), then the planes, each for all splats: positions
// (v2: 3 x 24-bit fixed point, v1: 3 x float16), alphas (1 B), colours (3 B), scales (3 B), rotations (3 B), SH (3 x {0, 3, 8, 15} B).
// Every input the reference returns null for is rejected, the length included: it must be exactly the header plus the planes.  Bit 0
// of flags (antialiased) is read and then ignored by the reference; it is ignored here too.
inline int parse_spz_header(const unsigned char *f, size_t bytes, FileLayout &L, char *err, size_t err_len) {
    using namespace file_detail;
#define bad(...) file_detail::fail_msg(err, err_len, __VA_ARGS__)
    if (bytes >= 2 && f[0] == 0x1f && f[1] == 0x8b)
        return bad(".spz: the data is gzip-compressed (starts 1f 8b): decompress it first and pass the packed stream");
    if (bytes < 16) return bad(".spz: %zu bytes, shorter than the 16-byte header", bytes);
    uint32_t magic, version, n;
    memcpy(&magic, f, 4); memcpy(&version, f + 4, 4); memcpy(&n, f + 8, 4);
    const uint32_t degree = f[12], fractional_bits = f[13];
    if (magic != kSpzMagic) return bad(".spz: magic 0x%08x is not 0x%08x ('NGSP')", magic, kSpzMagic);
    if (version < 1 || version > 2)
        return bad(".spz: version %u not supported (1 and 2; version 3 stores smallest-three rotations, which the reference does not read)", version);
    if (n > kSpzMaxPoints) return bad(".spz: %u points, more than %u", n, kSpzMaxPoints);
    if (degree > 3) return bad(".spz: SH degree %u (0..3)", degree);
    static const uint32_t kDim[4] = {0, 3, 8, 15};
    const uint32_t pos = version == 1 ? 6 : 9;
    const uint64_t plane[SPZ_PLANES] = {pos, 1, 3, 3, 3, 3ull * kDim[degree]};
    uint64_t at = 16;
    for (int p = 0; p < SPZ_PLANES; ++p) { L.spz_plane[p] = at; at += (uint64_t)n * plane[p]; }
    if (at != bytes)
        return bad(".spz: %zu bytes where the header and planes of %u splats at SH degree %u take exactly %llu", bytes, n, degree,
                   (unsigned long long)at);
    L.format = 4;
    L.count = n;
    L.stride = pos + 10;                               // bytes per splat outside the SH plane
    L.sh_degree = std::min<int>((int)degree, 2);
    L.spz_version = version;
    L.spz_sh_coeff = kDim[degree];
    // JavaScript's `1 << fractionalBits` shifts an int32 by the count mod 32: 31 gives -2^31 (every coordinate flips sign), 32 gives 1
    L.spz_pos_scale = 1.0 / (double)(int32_t)(1u << (fractional_bits & 31));
    return 0;
#undef bad
}

inline int parse_file(int format, const void *data, size_t bytes, FileLayout &L, char *err, size_t err_len) {
    L = FileLayout{};
    if (!data && bytes) { snprintf(err, err_len, "gs_probe_file / gs_upload_file: null data"); return 1; }
    if (format == 1) return parse_ply_header((const unsigned char *)data, bytes, L, err, err_len);
    if (format == 4) return parse_spz_header((const unsigned char *)data, bytes, L, err, err_len);
    if (format == 2) {
        if (bytes % 32) { snprintf(err, err_len, ".splat: %zu bytes is not a whole number of 32-byte rows", bytes); return 1; }
        if (bytes / 32 > 0xffffffffull) { snprintf(err, err_len, ".splat: too many rows"); return 1; }
        L.format = 2; L.count = (uint32_t)(bytes / 32); L.stride = 32; L.data_offset = 0; L.sh_degree = 0;
        return 0;
    }
    snprintf(err, err_len, "file format %d unknown (GS_FILE_PLY = 1, GS_FILE_SPLAT = 2, GS_FILE_SPZ = 4)", format);
    return 1;
}

} // namespace gs
