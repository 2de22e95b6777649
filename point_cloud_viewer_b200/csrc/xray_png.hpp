// xray_png.hpp — host side of the X-ray quadtree's on-disk form (SURVEY 8 f3 "PNG encode", which stays on the host):
// `<node id>.png` per tile (xray/src/utils.rs:33-37 get_image_path, IMAGE_FILE_EXTENSION = "png"; RGBA, 8 bit) and the
// quadtree's meta file (xray/src/lib.rs:88-139 Meta::to_disk / to_proto, xray_proto_rust/src/proto.proto:22-56; file name =
// the root node's id with the "r" prefix replaced by "meta", + ".pb": utils.rs:7-11).  The PNG stream is a plain
// non-interlaced RGBA image with filter type 0 on every scanline, deflated by zlib: the pixels are what the reference's
// `image.save` stores, the bytes of the file are not (another encoder).
// The merge of partial quadtrees (xray_merge.inl) reads both back: decode_png_rgba takes the PNGs this project and the
// reference's `image` crate write (8-bit RGBA, non-interlaced, any filter types, any IDAT split), decode_xray_meta the meta
// files of versions 2 and 3 (Meta::from_proto, lib.rs:59-116).
#pragma once
#include <zlib.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "disk_io.hpp"

namespace pcv {

inline void png_put32(std::string& s, uint32_t v) {
    const char b[4] = {(char)(v >> 24), (char)(v >> 16), (char)(v >> 8), (char)v};
    s.append(b, 4);
}
inline void png_chunk(std::string& out, const char type[4], const std::string& data) {
    png_put32(out, (uint32_t)data.size());
    std::string body(type, 4);
    body += data;
    out += body;
    png_put32(out, (uint32_t)crc32(0L, (const Bytef*)body.data(), (uInt)body.size()));
}
inline bool encode_png_rgba(const uint8_t* rgba, uint32_t w, uint32_t h, std::string& out, int level = 3) {
    if (w == 0 || h == 0 || (uint64_t)w * h * 4 + h >= 0xFFFFFFFFull) return false;
    std::vector<uint8_t> raw((size_t)h * ((size_t)w * 4 + 1));
    for (uint32_t y = 0; y < h; ++y) {
        uint8_t* row = &raw[(size_t)y * ((size_t)w * 4 + 1)];
        row[0] = 0;  // filter type None
        memcpy(row + 1, rgba + (size_t)y * w * 4, (size_t)w * 4);
    }
    uLongf cap = compressBound((uLong)raw.size());
    std::string z(cap, '\0');
    if (compress2((Bytef*)&z[0], &cap, raw.data(), (uLong)raw.size(), level) != Z_OK) return false;
    z.resize(cap);
    out.assign("\x89PNG\r\n\x1a\n", 8);
    std::string ihdr;
    png_put32(ihdr, w);
    png_put32(ihdr, h);
    ihdr += std::string("\x08\x06\x00\x00\x00", 5);  // 8 bit, colour type 6 (RGBA), deflate, adaptive filtering, no interlace
    png_chunk(out, "IHDR", ihdr);
    png_chunk(out, "IDAT", z);
    png_chunk(out, "IEND", std::string());
    return true;
}

// quadtree NodeId Display (quadtree/src/lib.rs:216-233): "r" + one base-4 digit per level, most significant first
inline std::string quad_node_name(uint8_t level, uint64_t index) {
    std::string s = "r";
    for (int l = (int)level - 1; l >= 0; --l) s.push_back((char)('0' + ((index >> (2 * l)) & 3)));
    return s;
}

struct XrayMetaData {
    double min_x = 0, min_y = 0, edge = 0;
    uint32_t deepest_level = 0, tile_size = 0;
    std::vector<std::pair<uint32_t, uint64_t>> nodes;  // (level, index)
};
// xray Meta::to_proto (lib.rs:117-139): version = CURRENT_VERSION = 3
inline std::string encode_xray_meta(const XrayMetaData& m) {
    std::string v2;  // Vector2d { 1: x, 2: y }
    pb::put_double(v2, 1, m.min_x);
    pb::put_double(v2, 2, m.min_y);
    std::string rect;  // Rect { 3: min, 4: edge_length }
    pb::put_bytes(rect, 3, v2);
    pb::put_double(rect, 4, m.edge);
    std::string meta;  // Meta { 1: version, 2: bounding_rect, 3: deepest_level, 4: tile_size, 5: repeated NodeId { 1: level, 2: index } }
    pb::put_uint(meta, 1, 3);
    pb::put_bytes(meta, 2, rect);
    pb::put_uint(meta, 3, m.deepest_level);
    pb::put_uint(meta, 4, m.tile_size);
    for (const auto& n : m.nodes) {
        std::string id;
        pb::put_uint(id, 1, n.first);
        pb::put_uint(id, 2, n.second);
        pb::put_bytes(meta, 5, id);
    }
    return meta;
}

inline uint32_t png_get32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | (uint32_t)p[3]; }
inline uint8_t png_paeth(int a, int b, int c) {  // PNG spec 9.4
    const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c);
    return (uint8_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}
// A PNG file's bytes -> w x h RGBA pixels.  Accepts 8-bit RGBA (colour type 6), non-interlaced, scanlines of any of the five
// filter types, the image data in any number of IDAT chunks; ancillary chunks are skipped.  The CRC of every chunk used and
// the zlib stream (its Adler-32 included) are checked.  Returns PCV_OK; PCV_ERR_UNSUPPORTED for other bit depths, colour types,
// interlacing or unknown critical chunks; PCV_ERR_INVALID for anything corrupt or truncated.  *why says what was wrong.
inline int decode_png_rgba(const std::string& file, uint32_t& w, uint32_t& h, std::vector<uint8_t>& rgba, std::string* why) {
    auto bad = [&](int code, const char* msg) {
        if (why) *why = msg;
        return code;
    };
    const uint8_t* p = (const uint8_t*)file.data();
    const size_t n = file.size();
    if (n < 8 || memcmp(p, "\x89PNG\r\n\x1a\n", 8) != 0) return bad(PCV_ERR_INVALID, "not a PNG signature");
    size_t at = 8;
    bool have_ihdr = false, have_iend = false;
    std::string z;
    w = h = 0;
    while (!have_iend) {
        if (n - at < 12) return bad(PCV_ERR_INVALID, "truncated chunk");
        const uint32_t len = png_get32(p + at);
        if (len > n - at - 12) return bad(PCV_ERR_INVALID, "truncated chunk");
        const uint8_t* type = p + at + 4;
        const uint8_t* data = type + 4;
        const bool ancillary = (type[0] & 0x20) != 0;
        if (!ancillary && png_get32(data + len) != (uint32_t)crc32(0L, type, (uInt)len + 4)) return bad(PCV_ERR_INVALID, "chunk CRC mismatch");
        if (!have_ihdr && memcmp(type, "IHDR", 4) != 0) return bad(PCV_ERR_INVALID, "first chunk is not IHDR");
        if (memcmp(type, "IHDR", 4) == 0) {
            if (have_ihdr || len != 13) return bad(PCV_ERR_INVALID, "bad IHDR");
            have_ihdr = true;
            w = png_get32(data);
            h = png_get32(data + 4);
            if (w == 0 || h == 0 || w > 0x7FFFFFFFu || h > 0x7FFFFFFFu) return bad(PCV_ERR_INVALID, "bad image size");
            if (data[10] != 0 || data[11] != 0) return bad(PCV_ERR_INVALID, "unknown compression or filter method");
            if (data[8] != 8 || data[9] != 6) return bad(PCV_ERR_UNSUPPORTED, "not 8-bit RGBA");
            if (data[12] != 0) return bad(PCV_ERR_UNSUPPORTED, "interlaced");
            if ((uint64_t)w * h * 4 > (1ull << 34)) return bad(PCV_ERR_UNSUPPORTED, "image too large");
        } else if (memcmp(type, "IDAT", 4) == 0) {
            z.append((const char*)data, len);
        } else if (memcmp(type, "IEND", 4) == 0) {
            have_iend = true;
        } else if (!ancillary) {
            return bad(PCV_ERR_UNSUPPORTED, "unknown critical chunk");
        }
        at += (size_t)len + 12;
    }
    const size_t stride = (size_t)w * 4, raw_n = (size_t)h * (stride + 1);
    std::vector<uint8_t> raw(raw_n);
    z_stream zs{};
    if (inflateInit(&zs) != Z_OK) return bad(PCV_ERR_INVALID, "zlib init");
    zs.next_in = (Bytef*)z.data();
    zs.next_out = raw.data();
    int zr = Z_OK;
    for (size_t in_left = z.size(), out_left = raw_n; zr == Z_OK;) {  // avail_* are 32-bit: feed at most 1 GiB per call
        const uInt ci = (uInt)std::min<size_t>(in_left, 1u << 30), co = (uInt)std::min<size_t>(out_left, 1u << 30);
        zs.avail_in = ci;
        zs.avail_out = co;
        zr = inflate(&zs, Z_NO_FLUSH);
        in_left -= ci - zs.avail_in;
        out_left -= co - zs.avail_out;
        if (zr == Z_BUF_ERROR && out_left == 0 && in_left) zr = Z_DATA_ERROR;  // more data than the image holds
        if (zr == Z_BUF_ERROR && (in_left == 0 || out_left == 0)) break;
    }
    const size_t got = (size_t)(zs.next_out - raw.data());
    inflateEnd(&zs);
    if (zr != Z_STREAM_END || got != raw_n) return bad(PCV_ERR_INVALID, "corrupt or truncated image data");
    rgba.resize((size_t)h * stride);
    for (uint32_t y = 0; y < h; ++y) {
        const uint8_t f = raw[(size_t)y * (stride + 1)];
        const uint8_t* in = &raw[(size_t)y * (stride + 1) + 1];
        uint8_t* out = &rgba[(size_t)y * stride];
        const uint8_t* up = y ? out - stride : nullptr;
        for (size_t i = 0; i < stride; ++i) {
            const int a = i >= 4 ? out[i - 4] : 0, b = up ? up[i] : 0, c = i >= 4 && up ? up[i - 4] : 0;
            switch (f) {
                case 0: out[i] = in[i]; break;
                case 1: out[i] = (uint8_t)(in[i] + a); break;
                case 2: out[i] = (uint8_t)(in[i] + b); break;
                case 3: out[i] = (uint8_t)(in[i] + ((a + b) >> 1)); break;
                case 4: out[i] = (uint8_t)(in[i] + png_paeth(a, b, c)); break;
                default: return bad(PCV_ERR_INVALID, "unknown scanline filter type");
            }
        }
    }
    return PCV_OK;
}

// A meta file's bytes -> its contents, as Meta::from_proto reads them (lib.rs:59-116): versions 2 and 3; the rect's `min`
// (Vector2d) and `edge_length`, or, when `min` is unset, `deprecated_min` (Vector2f) and `deprecated_edge_length` widened to
// f64; levels and deepest_level cast to u8.  Nodes keep their order and repeats (the reference collects them into a set).
// False for any other version and for a malformed message.
inline bool decode_xray_meta(const std::string& buf, XrayMetaData& m, int& version) {
    m = XrayMetaData{};
    version = 0;
    pb::Cursor c{(const uint8_t*)buf.data(), (const uint8_t*)buf.data() + buf.size()};
    bool have_min = false;
    double dmin[2] = {0, 0}, dedge = 0;
    while (c.more()) {
        const uint64_t k = c.varint();
        const uint32_t f = (uint32_t)(k >> 3), wt = (uint32_t)(k & 7);
        if (f == 1 && wt == 0) {
            version = (int)(int32_t)c.varint();
        } else if (f == 2 && wt == 2) {  // Rect { 1: deprecated_min, 2: deprecated_edge_length, 3: min, 4: edge_length }
            pb::Cursor r = c.sub();
            while (r.more()) {
                const uint64_t k2 = r.varint();
                const uint32_t f2 = (uint32_t)(k2 >> 3), w2 = (uint32_t)(k2 & 7);
                if ((f2 == 1 || f2 == 3) && w2 == 2) {
                    pb::Cursor v = r.sub();
                    double xy[2] = {0, 0};
                    while (v.more()) {
                        const uint64_t k3 = v.varint();
                        const uint32_t f3 = (uint32_t)(k3 >> 3), w3 = (uint32_t)(k3 & 7);
                        if (f3 >= 1 && f3 <= 2 && w3 == (f2 == 3 ? 1u : 5u))
                            xy[f3 - 1] = f2 == 3 ? v.fixed64() : (double)v.fixed32();
                        else if (f3 >= 1 && f3 <= 2)
                            return false;
                        else
                            v.skip(w3);
                    }
                    if (v.bad) return false;
                    if (f2 == 3) {
                        have_min = true;
                        m.min_x = xy[0], m.min_y = xy[1];
                    } else {
                        dmin[0] = xy[0], dmin[1] = xy[1];
                    }
                } else if (f2 == 2 && w2 == 5) {
                    dedge = (double)r.fixed32();
                } else if (f2 == 4 && w2 == 1) {
                    m.edge = r.fixed64();
                } else if (f2 >= 1 && f2 <= 4) {
                    return false;
                } else {
                    r.skip(w2);
                }
            }
            if (r.bad) return false;
        } else if ((f == 3 || f == 4) && wt == 0) {
            const uint32_t v = (uint32_t)c.varint();
            if (f == 3)
                m.deepest_level = v & 0xFF;
            else
                m.tile_size = v;
        } else if (f == 5 && wt == 2) {  // NodeId { 1: level, 2: index }
            pb::Cursor n = c.sub();
            uint32_t level = 0;
            uint64_t index = 0;
            while (n.more()) {
                const uint64_t k2 = n.varint();
                const uint32_t f2 = (uint32_t)(k2 >> 3), w2 = (uint32_t)(k2 & 7);
                if (f2 == 1 && w2 == 0)
                    level = (uint32_t)n.varint() & 0xFF;
                else if (f2 == 2 && w2 == 0)
                    index = n.varint();
                else if (f2 == 1 || f2 == 2)
                    return false;
                else
                    n.skip(w2);
            }
            if (n.bad) return false;
            m.nodes.emplace_back(level, index);
        } else if (f >= 1 && f <= 5) {
            return false;
        } else {
            c.skip(wt);
        }
    }
    if (c.bad || (version != 2 && version != 3)) return false;
    if (!have_min) m.min_x = dmin[0], m.min_y = dmin[1], m.edge = dedge;
    return true;
}

}  // namespace pcv
