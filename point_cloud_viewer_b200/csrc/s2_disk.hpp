// s2_disk.hpp — the on-disk form of an S2-cell point cloud: what S2Splitter<RawNodeWriter> leaves in a directory
// (src/read_write/s2.rs:127-145: one file set per cell, stem = CellID::to_token(); raw.rs / node_writer.rs: `<stem>.xyz` =
// f64 LE x, y, z per point for Encoding::Plain, `<stem>.rgb` = u8 x 3, `<stem>.intensity` = f32 LE; lib.rs:74-80 extensions)
// and its meta.pb: Meta { version = 13, bounding_box, s2 = S2Meta { cells { id, num_points }, attributes { name, data_type } } }
// (src/s2_cells/mod.rs:77-104 to_proto, :106-147 from_proto; point_viewer_proto_rust/src/proto.proto:92-149).
#pragma once
#include <string>
#include <vector>

#include "disk_io.hpp"
#include "s2.h"

namespace pcv {

struct S2MetaData {
    double bbox_min[3] = {0, 0, 0}, bbox_max[3] = {0, 0, 0};
    std::vector<uint64_t> ids, counts;
    bool has_color = false, has_intensity = false;
};
constexpr int kAttrF32 = 11, kAttrU8Vec3 = 27;  // AttributeDataType (proto.proto:92-111)

inline std::string encode_s2_meta(const S2MetaData& m) {
    auto vec3 = [](const double v[3]) {
        std::string s;
        pb::put_double(s, 1, v[0]);
        pb::put_double(s, 2, v[1]);
        pb::put_double(s, 3, v[2]);
        return s;
    };
    std::string cuboid;  // AxisAlignedCuboid { 3: min, 4: max }
    pb::put_bytes(cuboid, 3, vec3(m.bbox_min));
    pb::put_bytes(cuboid, 4, vec3(m.bbox_max));
    std::string s2;  // S2Meta { 1: repeated S2Cell { 1: id, 2: num_points }, 2: repeated Attribute { 1: name, 2: data_type } }
    for (size_t k = 0; k < m.ids.size(); ++k) {
        std::string cell;
        pb::put_uint(cell, 1, m.ids[k]);
        pb::put_uint(cell, 2, m.counts[k]);
        pb::put_bytes(s2, 1, cell);
    }
    auto attr = [&](const char* name, int type) {
        std::string a;
        pb::put_bytes(a, 1, name);
        pb::put_uint(a, 2, (uint64_t)type);
        pb::put_bytes(s2, 2, a);
    };
    if (m.has_color) attr("color", kAttrU8Vec3);
    if (m.has_intensity) attr("intensity", kAttrF32);
    std::string meta;  // Meta { 1: version, 4: bounding_box, 7: s2 }
    pb::put_uint(meta, 1, 13);
    pb::put_bytes(meta, 4, cuboid);
    pb::put_bytes(meta, 7, s2);
    return meta;
}

// S2Meta::from_proto (mod.rs:106-147).  Returns an empty string on success, else the reference's error text.
inline std::string decode_s2_meta(const std::string& buf, S2MetaData& m, int& version) {
    pb::Cursor c{(const uint8_t*)buf.data(), (const uint8_t*)buf.data() + buf.size()};
    bool has_s2 = false;
    version = 0;
    m = S2MetaData{};
    auto vec3 = [](pb::Cursor v, double out[3]) {
        while (v.more()) {
            const uint64_t key = v.varint();
            const uint32_t f = (uint32_t)(key >> 3), w = (uint32_t)(key & 7);
            if (w == 1 && f >= 1 && f <= 3)
                out[f - 1] = v.fixed64();
            else
                v.skip(w);
        }
        return !v.bad;
    };
    std::string bad_attr;
    while (c.more()) {
        const uint64_t key = c.varint();
        const uint32_t f = (uint32_t)(key >> 3), w = (uint32_t)(key & 7);
        if (f == 1 && w == 0) {
            version = (int)c.varint();
        } else if (f == 4 && w == 2) {
            pb::Cursor b = c.sub();
            while (b.more()) {
                const uint64_t k2 = b.varint();
                const uint32_t f2 = (uint32_t)(k2 >> 3), w2 = (uint32_t)(k2 & 7);
                if (w2 == 2 && (f2 == 3 || f2 == 4)) {
                    if (!vec3(b.sub(), f2 == 3 ? m.bbox_min : m.bbox_max)) return "Could not parse meta.pb";
                } else {
                    b.skip(w2);
                }
            }
            if (b.bad) return "Could not parse meta.pb";
        } else if (f == 7 && w == 2) {
            has_s2 = true;
            pb::Cursor s = c.sub();
            while (s.more()) {
                const uint64_t k2 = s.varint();
                const uint32_t f2 = (uint32_t)(k2 >> 3), w2 = (uint32_t)(k2 & 7);
                if (f2 == 1 && w2 == 2) {
                    pb::Cursor cell = s.sub();
                    uint64_t id = 0, np = 0;
                    while (cell.more()) {
                        const uint64_t k3 = cell.varint();
                        const uint32_t f3 = (uint32_t)(k3 >> 3), w3 = (uint32_t)(k3 & 7);
                        if (w3 == 0 && f3 == 1)
                            id = cell.varint();
                        else if (w3 == 0 && f3 == 2)
                            np = cell.varint();
                        else
                            cell.skip(w3);
                    }
                    if (cell.bad) return "Could not parse meta.pb";
                    m.ids.push_back(id);
                    m.counts.push_back(np);
                } else if (f2 == 2 && w2 == 2) {
                    pb::Cursor a = s.sub();
                    std::string name;
                    uint64_t type = 0;
                    while (a.more()) {
                        const uint64_t k3 = a.varint();
                        const uint32_t f3 = (uint32_t)(k3 >> 3), w3 = (uint32_t)(k3 & 7);
                        if (w3 == 2 && f3 == 1) {
                            pb::Cursor n = a.sub();
                            name.assign((const char*)n.p, (size_t)(n.end - n.p));
                        } else if (w3 == 0 && f3 == 2) {
                            type = a.varint();
                        } else {
                            a.skip(w3);
                        }
                    }
                    if (a.bad) return "Could not parse meta.pb";
                    if (name == "color" && type == (uint64_t)kAttrU8Vec3)
                        m.has_color = true;
                    else if (name == "intensity" && type == (uint64_t)kAttrF32)
                        m.has_intensity = true;
                    else
                        bad_attr = name;  // this implementation carries the two attributes the octree side carries
                } else {
                    s.skip(w2);
                }
            }
            if (s.bad) return "Could not parse meta.pb";
        } else {
            c.skip(w);
        }
    }
    if (c.bad) return "Could not parse meta.pb";
    if (version < 12) return "No S2 point cloud supported with version " + std::to_string(version);
    if (!has_s2) return "This meta does not describe S2 point clouds";
    if (!bad_attr.empty()) return "unsupported attribute '" + bad_attr + "' (color: U8Vec3 and intensity: F32 are carried)";
    return "";
}

// The cells of an S2 directory as pcv_s2_load_dir lays them out, from its meta.pb alone: cells in id order, the first slot
// of each, the total and the deepest cell level (the split level).
struct S2DirCells {
    S2MetaData m;                // the box and attributes; m.ids / m.counts in the proto's order
    std::vector<uint64_t> ids, counts, starts;
    uint64_t n = 0;
    int level = -1;
};
// meta.pb of `dir` -> its cells.  PCV_OK, or PCV_ERR_IO (meta.pb unreadable) / PCV_ERR_INVALID (not an S2 meta of version
// 12 or 13, an invalid or duplicated cell id) with the message in `err`.  No cell file is touched.
inline int open_s2_dir_cells(const std::string& dir, S2DirCells& out, std::string& err) {
    const std::string base = dir + "/";
    std::string raw;
    out = S2DirCells{};
    if (!read_whole_file(base + "meta.pb", raw)) return err = "cannot read " + base + "meta.pb", PCV_ERR_IO;
    int version = 0;
    err = decode_s2_meta(raw, out.m, version);
    if (!err.empty()) return PCV_ERR_INVALID;
    // cells in id order (the proto carries them in hash-map order)
    const S2MetaData& m = out.m;
    std::vector<size_t> order(m.ids.size());
    for (size_t k = 0; k < order.size(); ++k) order[k] = k;
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return m.ids[a] < m.ids[b]; });
    for (size_t k : order) {
        char buf[96];
        if (!s2_is_valid(m.ids[k])) {
            snprintf(buf, sizeof buf, "invalid S2 cell id %llx in meta.pb", (unsigned long long)m.ids[k]);
            return err = buf, PCV_ERR_INVALID;
        }
        if (!out.ids.empty() && out.ids.back() == m.ids[k]) return err = "cell " + s2_to_token(m.ids[k]) + " is listed twice", PCV_ERR_INVALID;
        out.ids.push_back(m.ids[k]);
        out.counts.push_back(m.counts[k]);
        out.starts.push_back(out.n);
        out.n += m.counts[k];
        out.level = std::max(out.level, s2_level(m.ids[k]));
    }
    return PCV_OK;
}

}  // namespace pcv
