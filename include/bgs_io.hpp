// bgs_io.hpp -- C++ host mirror of the reference's cloud loader for the splat path's input row (SURVEY.md §8 f1),
// header-only, no dependency on the C ABI: it produces the four planes `bgs::PlanarGaussian3d` (bgs.hpp) uploads.
//
//   parse_ply_3d     src/io/ply.rs:23-132   INRIA 3DGS `.ply` -> PlanarGaussian3d, with the reference's quirks:
//     * only `float` properties of the `vertex` element are consumed (ply.rs:33-90: `Property::Float`)
//     * opacity = sigmoid(raw)                                          ply.rs:40-42
//     * f_rest_i -> channel i / 16 (not / 15), coefficient (i % 15) + 1, interleaved index coefficient * 3 + channel,
//       dropped when >= 48; later properties overwrite earlier ones       ply.rs:49-69
//       (at SH degree d, the reference's sh_d build: K = (d + 1)^2, channel i / K, coefficient 1 if K == 1 else
//       (i % (K - 1)) + 1, dropped when coefficient * 3 + channel >= S_d)
//     * scale_i = exp(clamp(raw_i, mean(raw) -+ 4))                      ply.rs:103-116
//     * rotation normalised                                              ply.rs:118-124
//     * padded with default gaussians by 32 - (n % 32) entries           ply.rs:127-129
//   decode_gcloud / encode_gcloud   src/io/gcloud/flexbuffers.rs:9-22, src/io/codec.rs:4-18   the reference's DEFAULT asset
//     path (src/io/loader.rs:22-66: `Some("gcloud") => PlanarGaussian3d::decode(bytes)`): the serde serialisation of
//     PlanarGaussian3d into a FlexBuffer (map of four vectors of per-gaussian maps).  The reader below is a generic
//     FlexBuffers reader (google/flatbuffers flexbuffers.h wire format: root at the end, backward offsets, typed /
//     fixed-typed / untyped vectors, maps with a sorted key vector, every scalar width), the writer emits the same
//     shapes as the Python host mirror (bevy_gaussian_splatting_b200/gcloud.py): each reads what the other writes.  As there, parity with
//     bytes written by the Rust `flexbuffers` crate is UNPINNED (no reference-written file exists in this image); the bar
//     is the reference's own: a round trip (tests/io.rs:7-17).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <istream>
#include <iterator>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "bgs.hpp"

namespace bgs {
namespace io {

namespace detail {
struct PlyProp { std::string name; int size; bool is_f32; bool is_f64; int list_count_size = 0; };   // list: size = item size
struct PlyElement { std::string name; size_t count = 0; std::vector<PlyProp> props; };

inline int ply_type_size(const std::string& t, bool& f32, bool& f64) {
    f32 = (t == "float" || t == "float32"); f64 = (t == "double" || t == "float64");
    if (f32) return 4;
    if (f64) return 8;
    if (t == "uchar" || t == "uint8" || t == "char" || t == "int8") return 1;
    if (t == "short" || t == "int16" || t == "ushort" || t == "uint16") return 2;
    if (t == "int" || t == "int32" || t == "uint" || t == "uint32") return 4;
    throw std::runtime_error("ply: unknown property type " + t);
}
inline float load_f32(const unsigned char* p, bool big_endian) {
    unsigned char b[4];
    if (big_endian) { b[0] = p[3]; b[1] = p[2]; b[2] = p[1]; b[3] = p[0]; } else std::memcpy(b, p, 4);
    float v; std::memcpy(&v, b, 4); return v;
}
}  // namespace detail

inline PlanarGaussian3d parse_ply_3d(std::istream& in, uint32_t sh_degree = 3) {
    using namespace detail;
    if (sh_degree > 3) throw std::runtime_error("ply: sh_degree must be 0..3");
    const size_t S = sh_width(sh_degree), K = (size_t)(sh_degree + 1) * (sh_degree + 1);
    std::string line;
    if (!std::getline(in, line) || line.substr(0, 3) != "ply") throw std::runtime_error("not a PLY file");
    std::string format;
    std::vector<PlyElement> elements;
    bool ended = false;
    while (std::getline(in, line)) {
        std::istringstream ls(line);
        std::string tok; ls >> tok;
        if (tok == "format") ls >> format;
        else if (tok == "element") { PlyElement e; ls >> e.name >> e.count; elements.push_back(e); }
        else if (tok == "property") {
            std::string ty, name; ls >> ty;
            if (elements.empty()) throw std::runtime_error("ply: property before element");
            PlyProp p;
            if (ty == "list") {   // fine in other elements (faces), which are skipped; not in the vertex element
                if (elements.back().name == "vertex") throw std::runtime_error("ply: list properties are not supported in the vertex element");
                std::string cty, ity; ls >> cty >> ity >> name;
                bool a, b;
                p.list_count_size = ply_type_size(cty, a, b);
                p.size = ply_type_size(ity, a, b); p.is_f32 = p.is_f64 = false;
            } else {
                ls >> name;
                p.size = ply_type_size(ty, p.is_f32, p.is_f64);
            }
            p.name = name;
            elements.back().props.push_back(p);
        } else if (tok == "end_header") { ended = true; break; }
    }
    if (!ended) throw std::runtime_error("unterminated PLY header");
    const bool ascii = format == "ascii", big = format == "binary_big_endian";
    if (!ascii && !big && format != "binary_little_endian") throw std::runtime_error("ply: unknown format " + format);

    // column index of every consumed property inside the vertex rows (header order = the order set_property is called in)
    size_t n = 0;
    std::vector<std::vector<float>> cols;       // one vector per float property of the vertex element
    std::vector<std::string> names;
    bool have_vertex = false;
    for (const PlyElement& el : elements) {
        size_t stride = 0;
        for (const PlyProp& p : el.props) stride += (size_t)p.size;
        if (el.name != "vertex") {   // skip
            bool lists = false;
            for (const PlyProp& p : el.props) lists = lists || p.list_count_size != 0;
            if (ascii) {
                in >> std::ws;
                for (size_t i = 0; i < el.count; ++i) std::getline(in, line);
            } else if (!lists) {
                in.ignore((std::streamsize)(stride * el.count));
            } else {
                for (size_t i = 0; i < el.count; ++i)
                    for (const PlyProp& p : el.props) {
                        if (p.list_count_size == 0) { in.ignore(p.size); continue; }
                        unsigned char cb[8] = {0};
                        in.read((char*)cb, p.list_count_size);
                        uint64_t cnt = 0;
                        for (int k = 0; k < p.list_count_size; ++k)
                            cnt |= (uint64_t)cb[big ? p.list_count_size - 1 - k : k] << (8 * k);
                        in.ignore((std::streamsize)(cnt * (uint64_t)p.size));
                    }
            }
            continue;
        }
        static const char* required[] = {"x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "scale_0", "scale_1", "opacity",
                                         "rot_0", "rot_1", "rot_2", "rot_3"};
        for (const char* r : required) {
            bool found = false;
            for (const PlyProp& p : el.props) found = found || p.name == r;
            if (!found) throw std::runtime_error("missing required properties");   // ply.rs:92-97
        }
        have_vertex = true; n = el.count;
        for (const PlyProp& p : el.props)
            if (ascii || p.is_f32) { names.push_back(p.name); cols.emplace_back(n); }
        if (ascii) {
            for (size_t i = 0; i < n; ++i) {
                size_t c = 0;
                for (size_t k = 0; k < el.props.size(); ++k) { double v; in >> v; cols[c++][i] = (float)v; }
            }
        } else {
            std::vector<unsigned char> row(stride);
            for (size_t i = 0; i < n; ++i) {
                in.read((char*)row.data(), (std::streamsize)stride);
                if (!in) throw std::runtime_error("ply: truncated vertex data");
                size_t off = 0, c = 0;
                for (const PlyProp& p : el.props) {
                    if (p.is_f32) cols[c++][i] = load_f32(row.data() + off, big);
                    off += (size_t)p.size;
                }
            }
        }
    }
    PlanarGaussian3d out;
    out.sh_degree = sh_degree;
    if (!have_vertex) return out;
    const size_t pad = 32 - (n % 32), total = n + pad;
    out.position_visibility.assign(total * 4, 0.0f);
    out.spherical_harmonic.assign(total * S, 0.0f);
    out.rotation.assign(total * 4, 0.0f);
    out.scale_opacity.assign(total * 4, 0.0f);
    for (size_t i = 0; i < total; ++i) out.position_visibility[4 * i + 3] = 1.0f;   // PositionVisibility::default
    for (size_t c = 0; c < names.size(); ++c) {
        const std::string& key = names[c];
        const std::vector<float>& v = cols[c];
        auto put = [&](std::vector<float>& plane, size_t stride, size_t at) { for (size_t i = 0; i < n; ++i) plane[stride * i + at] = v[i]; };
        if (key == "x") put(out.position_visibility, 4, 0);
        else if (key == "y") put(out.position_visibility, 4, 1);
        else if (key == "z") put(out.position_visibility, 4, 2);
        else if (key == "visibility") put(out.position_visibility, 4, 3);
        else if (key == "f_dc_0") put(out.spherical_harmonic, S, 0);
        else if (key == "f_dc_1") put(out.spherical_harmonic, S, 1);
        else if (key == "f_dc_2") put(out.spherical_harmonic, S, 2);
        else if (key == "scale_0") put(out.scale_opacity, 4, 0);
        else if (key == "scale_1") put(out.scale_opacity, 4, 1);
        else if (key == "scale_2") put(out.scale_opacity, 4, 2);
        else if (key == "opacity") { for (size_t i = 0; i < n; ++i) out.scale_opacity[4 * i + 3] = 1.0f / (1.0f + std::exp(-v[i])); }
        else if (key == "rot_0") put(out.rotation, 4, 0);
        else if (key == "rot_1") put(out.rotation, 4, 1);
        else if (key == "rot_2") put(out.rotation, 4, 2);
        else if (key == "rot_3") put(out.rotation, 4, 3);
        else if (key.compare(0, 7, "f_rest_") == 0) {
            // the reference does `parse::<usize>().unwrap()` (io/ply.rs): anything but decimal digits is a hard error
            const char* dig = key.c_str() + 7;
            if (*dig == 0 || std::strlen(dig) > 6) throw std::runtime_error("ply: bad property name " + key);
            for (const char* q = dig; *q; ++q)
                if (*q < '0' || *q > '9') throw std::runtime_error("ply: bad property name " + key);
            const unsigned long i = std::strtoul(dig, nullptr, 10);
            const unsigned long channel = i / K, coefficient = K == 1 ? 1 : (i % (K - 1)) + 1, idx = coefficient * 3 + channel;
            if (idx < S) put(out.spherical_harmonic, S, (size_t)idx);
        }
    }
    for (size_t i = 0; i < n; ++i) {
        float* so = &out.scale_opacity[4 * i];
        const float mean = ((so[0] + so[1]) + so[2]) / 3.0f;
        for (int k = 0; k < 3; ++k) so[k] = std::exp(std::fmin(std::fmax(so[k], mean - 4.0f), mean + 4.0f));
        float* q = &out.rotation[4 * i];
        const float norm = std::sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3]);
        for (int k = 0; k < 4; ++k) q[k] = q[k] / norm;
    }
    return out;
}

// ---------------------------------------------------------------------------------------------------- .gcloud
namespace flex {
enum Type { T_NULL = 0, T_INT = 1, T_UINT = 2, T_FLOAT = 3, T_KEY = 4, T_STRING = 5, T_IND_INT = 6, T_IND_UINT = 7, T_IND_FLOAT = 8,
            T_MAP = 9, T_VECTOR = 10, T_VECTOR_INT = 11, T_VECTOR_UINT = 12, T_VECTOR_FLOAT = 13, T_VECTOR_KEY = 14,
            T_VECTOR_STRING_DEPRECATED = 15, T_VECTOR_INT2 = 16, T_VECTOR_FLOAT4 = 24, T_BLOB = 25, T_BOOL = 26, T_VECTOR_BOOL = 36 };

struct Ref {
    const unsigned char* buf; size_t len; size_t pos; unsigned parent_width; unsigned type; unsigned byte_width;
    Ref(const unsigned char* b, size_t l, size_t p, unsigned pw, unsigned packed)
        : buf(b), len(l), pos(p), parent_width(pw), type(packed >> 2), byte_width(1u << (packed & 3u)) {
        if (p + pw > l) throw std::runtime_error("gcloud: value outside the buffer");
    }
    uint64_t u(size_t p, unsigned w) const {
        if (p + w > len) throw std::runtime_error("gcloud: read outside the buffer");
        uint64_t v = 0;
        std::memcpy(&v, buf + p, w);                 // little-endian host (x86-64 / aarch64), as the reference's targets
        return v;
    }
    size_t target() const {
        const uint64_t off = u(pos, parent_width);
        if (off > pos) throw std::runtime_error("gcloud: offset outside the buffer");
        return pos - (size_t)off;
    }
    static double f_at(const unsigned char* p, unsigned w) {
        if (w == 4) { float v; std::memcpy(&v, p, 4); return v; }
        if (w == 8) { double v; std::memcpy(&v, p, 8); return v; }
        throw std::runtime_error("gcloud: float of unsupported width");
    }
    int64_t as_int() const {
        size_t p = pos; unsigned w = parent_width;
        if (type == T_IND_INT || type == T_IND_UINT) { p = target(); w = byte_width; }
        else if (type == T_FLOAT || type == T_IND_FLOAT) return (int64_t)as_float();
        else if (type == T_NULL) return 0;
        else if (type != T_INT && type != T_UINT && type != T_BOOL) throw std::runtime_error("gcloud: not a number");
        const uint64_t v = u(p, w);
        if (type == T_INT || type == T_IND_INT) {      // sign-extend
            const unsigned sh = 64 - 8 * w;
            return (int64_t)(v << sh) >> sh;
        }
        return (int64_t)v;
    }
    double as_float() const {
        if (type == T_FLOAT) { if (pos + parent_width > len) throw std::runtime_error("gcloud: read outside the buffer"); return f_at(buf + pos, parent_width); }
        if (type == T_IND_FLOAT) { const size_t t = target(); if (t + byte_width > len) throw std::runtime_error("gcloud: read outside the buffer"); return f_at(buf + t, byte_width); }
        if (type == T_NULL) return 0.0;
        return (double)as_int();
    }
    bool is_vector() const { return type == T_MAP || type == T_VECTOR || type == T_VECTOR_BOOL || (type >= T_VECTOR_INT && type <= T_VECTOR_FLOAT4); }
    // (position of element 0, length, element type or -1 when untyped)
    void vector_info(size_t& t, size_t& n, int& ety) const {
        t = target();
        if (type >= T_VECTOR_INT2 && type <= T_VECTOR_FLOAT4) { n = (type - T_VECTOR_INT2) / 3 + 2; ety = (int)((type - T_VECTOR_INT2) % 3 + T_INT); return; }
        if (t < byte_width) throw std::runtime_error("gcloud: vector without a length");
        n = (size_t)u(t - byte_width, byte_width);
        if (type == T_VECTOR || type == T_MAP) { ety = -1; return; }
        if (type == T_VECTOR_BOOL) { ety = T_BOOL; return; }
        if (type >= T_VECTOR_INT && type <= T_VECTOR_STRING_DEPRECATED) { ety = (int)(type - T_VECTOR_INT + T_INT); return; }
        throw std::runtime_error("gcloud: not a vector");
    }
    size_t size() const { size_t t, n; int e; vector_info(t, n, e); return n; }
    Ref at(size_t i) const {
        size_t t, n; int ety; vector_info(t, n, ety);
        if (i >= n) throw std::runtime_error("gcloud: index past the end of a vector");
        const unsigned w = byte_width;
        unsigned packed;
        if (ety < 0) packed = (unsigned)u(t + n * w + i, 1);
        else packed = ((unsigned)ety << 2) | (w == 1 ? 0u : w == 2 ? 1u : w == 4 ? 2u : 3u);
        return Ref(buf, len, t + i * w, w, packed);
    }
    // numbers of any vector, appended to `out` (typed f32 vectors are copied in one piece)
    void floats(std::vector<float>& out, size_t expect) const {
        size_t t, n; int ety; vector_info(t, n, ety);
        if (n != expect) throw std::runtime_error("gcloud: array of unexpected length");
        if (ety == T_FLOAT && byte_width == 4) {
            if (t + 4 * n > len) throw std::runtime_error("gcloud: vector outside the buffer");
            const size_t at0 = out.size(); out.resize(at0 + n); std::memcpy(out.data() + at0, buf + t, 4 * n);
            return;
        }
        for (size_t i = 0; i < n; ++i) out.push_back((float)at(i).as_float());
    }
    std::string key_at(size_t kvec, unsigned kw, size_t i) const {
        const size_t slot = kvec + i * kw;
        const uint64_t off = u(slot, kw);
        if (off > slot) throw std::runtime_error("gcloud: key offset outside the buffer");
        const size_t t = slot - (size_t)off;
        size_t e = t; while (e < len && buf[e] != 0) ++e;
        if (e >= len) throw std::runtime_error("gcloud: unterminated key");
        return std::string((const char*)buf + t, e - t);
    }
    // value of `key` in a map (keys are sorted: binary search like the reference crate; linear is fine for <= 4 keys)
    Ref get(const char* key) const {
        if (type != T_MAP) throw std::runtime_error("gcloud: not a map");
        const size_t t = target(); const unsigned w = byte_width;
        if (t < 3 * (size_t)w) throw std::runtime_error("gcloud: truncated map");
        const size_t kpos = t - 3 * w;
        const uint64_t koff = u(kpos, w);
        if (koff > kpos) throw std::runtime_error("gcloud: key vector outside the buffer");
        const size_t kvec = kpos - (size_t)koff;
        const unsigned kw = (unsigned)u(t - 2 * w, w);
        if (kw != 1 && kw != 2 && kw != 4 && kw != 8) throw std::runtime_error("gcloud: bad key width");
        if (kvec < kw) throw std::runtime_error("gcloud: truncated key vector");
        const size_t n = (size_t)u(kvec - kw, kw);
        for (size_t i = 0; i < n; ++i) if (key_at(kvec, kw, i) == key) return at(i);
        throw std::runtime_error(std::string("gcloud: missing field ") + key);
    }
};
inline Ref root(const unsigned char* buf, size_t len) {
    if (len < 3) throw std::runtime_error("gcloud: buffer too small");
    const unsigned width = buf[len - 1];
    if ((width != 1 && width != 2 && width != 4 && width != 8) || len < 2 + (size_t)width) throw std::runtime_error("gcloud: bad root width");
    return Ref(buf, len, len - 2 - width, width, buf[len - 2]);
}

// writer: 4-byte slots throughout, children first -- the layout of gcloud.py's Builder
struct Builder {
    std::vector<unsigned char> out;
    void align() { while (out.size() % 4) out.push_back(0); }
    void u32(uint64_t v) { if (v >> 32) throw std::runtime_error("gcloud: offset does not fit 32 bits"); const uint32_t x = (uint32_t)v; const size_t a = out.size(); out.resize(a + 4); std::memcpy(out.data() + a, &x, 4); }
    void f32(float v) { const size_t a = out.size(); out.resize(a + 4); std::memcpy(out.data() + a, &v, 4); }
    size_t key(const char* k) { const size_t p = out.size(); out.insert(out.end(), k, k + std::strlen(k) + 1); return p; }
};
}  // namespace flex

// CloudCodec::decode for PlanarGaussian3d (src/io/gcloud/flexbuffers.rs:18-22).
inline PlanarGaussian3d decode_gcloud(const unsigned char* data, size_t len) {
    const flex::Ref r = flex::root(data, len);
    PlanarGaussian3d out;
    // the SH degree the file was written at, from the first coefficient tuple's length (4, 12, 28 or 48)
    const flex::Ref shv = r.get("spherical_harmonic");
    if (shv.is_vector() && shv.size() > 0) {
        const size_t w = shv.at(0).get("coefficients").size();
        out.sh_degree = w == 4 ? 0 : w == 12 ? 1 : w == 28 ? 2 : w == 48 ? 3 : 4;
        if (out.sh_degree > 3) throw std::runtime_error("gcloud: coefficients hold 4, 12, 28 or 48 floats (SH degree 0..3)");
    }
    struct Plane { const char* name; std::vector<float>* dst; const char* f0; size_t w0; const char* f1; };
    const Plane planes[4] = {{"position_visibility", &out.position_visibility, "position", 3, "visibility"},
                             {"spherical_harmonic", &out.spherical_harmonic, "coefficients", sh_width(out.sh_degree), nullptr},
                             {"rotation", &out.rotation, "rotation", 4, nullptr},
                             {"scale_opacity", &out.scale_opacity, "scale", 3, "opacity"}};
    size_t n = 0;
    for (int p = 0; p < 4; ++p) {
        const flex::Ref vec = r.get(planes[p].name);
        if (!vec.is_vector()) throw std::runtime_error(std::string("gcloud: ") + planes[p].name + " is not a vector");
        const size_t cnt = vec.size();
        if (p == 0) n = cnt; else if (cnt != n) throw std::runtime_error("gcloud: planes disagree on the gaussian count");
        if (cnt > len) throw std::runtime_error("gcloud: element count exceeds the buffer");   // every element occupies >= 1 byte: a corrupted length must not size an allocation
        planes[p].dst->reserve(cnt * (planes[p].w0 + (planes[p].f1 ? 1 : 0)));
        for (size_t i = 0; i < cnt; ++i) {
            const flex::Ref e = vec.at(i);
            e.get(planes[p].f0).floats(*planes[p].dst, planes[p].w0);
            if (planes[p].f1) planes[p].dst->push_back((float)e.get(planes[p].f1).as_float());
        }
    }
    return out;
}
inline PlanarGaussian3d decode_gcloud(const std::vector<unsigned char>& bytes) { return decode_gcloud(bytes.data(), bytes.size()); }

// CloudCodec::encode (src/io/gcloud/flexbuffers.rs:9-16): struct -> map keyed by field name (keys sorted), Vec / array ->
// vector; 2..4 floats use the fixed-length typed vector, more a length-prefixed VECTOR_FLOAT.  The SH tuple is the
// cloud's S_d.
inline std::vector<unsigned char> encode_gcloud(const PlanarGaussian3d& c) {
    using namespace flex;
    Builder b;
    const size_t n = c.len(), S = sh_width(c.sh_degree);
    struct Field { const char* name; size_t col, w; };
    struct Plane { const char* name; const std::vector<float>* src; size_t stride; std::vector<Field> fields; };   // fields sorted by name
    const Plane planes[4] = {{"position_visibility", &c.position_visibility, 4, {{"position", 0, 3}, {"visibility", 3, 1}}},
                             {"rotation", &c.rotation, 4, {{"rotation", 0, 4}}},
                             {"scale_opacity", &c.scale_opacity, 4, {{"opacity", 3, 1}, {"scale", 0, 3}}},
                             {"spherical_harmonic", &c.spherical_harmonic, S, {{"coefficients", 0, S}}}};     // (sorted by name)
    size_t plane_pos[4]; unsigned plane_type[4];
    // gcloud.py encodes the planes in struct order (position_visibility, spherical_harmonic, rotation, scale_opacity)
    const int order[4] = {0, 3, 1, 2};
    for (int oi = 0; oi < 4; ++oi) {
        const Plane& pl = planes[order[oi]];
        std::vector<size_t> kpos;
        for (const Field& f : pl.fields) kpos.push_back(b.key(f.name));
        b.align(); b.u32(pl.fields.size());
        const size_t kv = b.out.size();
        for (size_t k : kpos) b.u32(b.out.size() - k);
        b.align();
        std::vector<size_t> elem_pos(n);
        for (size_t i = 0; i < n; ++i) {
            const float* row = pl.src->data() + i * pl.stride;
            std::vector<size_t> vec_at(pl.fields.size(), 0);
            for (size_t fi = 0; fi < pl.fields.size(); ++fi) {
                const Field& f = pl.fields[fi];
                if (f.w == 1) continue;
                if (f.w > 4) b.u32(f.w);
                vec_at[fi] = b.out.size();
                for (size_t k = 0; k < f.w; ++k) b.f32(row[f.col + k]);
            }
            b.u32(b.out.size() - kv); b.u32(4); b.u32(pl.fields.size());
            elem_pos[i] = b.out.size();
            std::vector<unsigned char> types;
            for (size_t fi = 0; fi < pl.fields.size(); ++fi) {
                const Field& f = pl.fields[fi];
                if (f.w == 1) { b.f32(row[f.col]); types.push_back((unsigned char)((T_FLOAT << 2) | 2)); }
                else {
                    b.u32(b.out.size() - vec_at[fi]);
                    const unsigned ty = f.w <= 4 ? (unsigned)(T_VECTOR_INT2 + (f.w - 2) * 3 + (T_FLOAT - T_INT)) : (unsigned)T_VECTOR_FLOAT;
                    types.push_back((unsigned char)((ty << 2) | 2));
                }
            }
            b.out.insert(b.out.end(), types.begin(), types.end());
            b.align();
        }
        // the plane: an untyped vector of the n element maps
        b.align(); b.u32(n);
        plane_pos[order[oi]] = b.out.size();
        for (size_t i = 0; i < n; ++i) b.u32(b.out.size() - elem_pos[i]);
        for (size_t i = 0; i < n; ++i) b.out.push_back((unsigned char)((T_MAP << 2) | 2));
        plane_type[order[oi]] = (T_VECTOR << 2) | 2;
    }
    // root map, keys sorted
    std::vector<size_t> kpos;
    for (int p = 0; p < 4; ++p) kpos.push_back(b.key(planes[p].name));
    b.align(); b.u32(4);
    const size_t kv = b.out.size();
    for (size_t k : kpos) b.u32(b.out.size() - k);
    b.align();
    b.u32(b.out.size() - kv); b.u32(4); b.u32(4);
    const size_t root_pos = b.out.size();
    for (int p = 0; p < 4; ++p) b.u32(b.out.size() - plane_pos[p]);
    for (int p = 0; p < 4; ++p) b.out.push_back((unsigned char)plane_type[p]);
    b.align();
    b.u32(b.out.size() - root_pos);
    b.out.push_back((unsigned char)((T_MAP << 2) | 2)); b.out.push_back(4);
    return b.out;
}

// src/io/loader.rs:38-66: dispatch on the file extension
inline PlanarGaussian3d load_cloud(const std::string& path) {
    std::ifstream in(path, std::ios::binary);
    if (!in) throw std::runtime_error("cannot open " + path);
    const size_t dot = path.rfind('.');
    const std::string ext = dot == std::string::npos ? "" : path.substr(dot + 1);
    if (ext == "ply") return parse_ply_3d(in);
    if (ext == "gcloud") {
        std::vector<unsigned char> bytes((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
        return decode_gcloud(bytes);
    }
    throw std::runtime_error("unsupported cloud file extension: ." + ext);     // loader.rs: "only .ply and .gcloud supported"
}

}  // namespace io

// src/query/select.rs:156-176: cloud.subset(selected), then write_to_file (declared in bgs.hpp)
inline uint32_t GaussianSplattingPlugin::save_selection(const PlanarGaussian3dHandle& cloud, const std::string& path) {
    const PlanarGaussian3dHandle sub = subset(cloud);
    if (!sub.get()) throw Error(BGS_EINVAL, "save_selection: nothing is selected");
    const std::vector<unsigned char> bytes = io::encode_gcloud(download(sub));
    std::ofstream f(path, std::ios::binary);
    if (!f.write(reinterpret_cast<const char*>(bytes.data()), (std::streamsize)bytes.size()))
        throw std::runtime_error("save_selection: cannot write " + path);
    return sub.len();
}
}  // namespace bgs
