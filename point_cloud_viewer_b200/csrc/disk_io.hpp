// disk_io.hpp — the reference's on-disk octree layout, host side.
//   <dir>/<NodeId Display>.xyz / .rgb / .intensity      src/data_provider/on_disk.rs:17-33, src/lib.rs:74-80
//   <dir>/meta.pb  (proto3, version 13)                 point_viewer_proto_rust/src/proto.proto:58-149
// Files of nodes with zero points are not created (node_writer.rs:78-89); such nodes still appear in
// meta.pb (generation.rs:241-243).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/pcv.h"

namespace pcv {

// Index of NodeId (hi, lo) in `nodes` (sorted by NodeId), -1 if absent.
inline int find_node(const std::vector<pcv_node_meta>& nodes, uint64_t hi, uint64_t lo) {
    auto it = std::lower_bound(nodes.begin(), nodes.end(), std::make_pair(hi, lo),
                               [](const pcv_node_meta& m, const std::pair<uint64_t, uint64_t>& k) { return m.id_high != k.first ? m.id_high < k.first : m.id_low < k.second; });
    return it != nodes.end() && it->id_high == hi && it->id_low == lo ? (int)(it - nodes.begin()) : -1;
}

// NodeId Display (node.rs:73-86): 'r' followed by the octal path, one digit per level.
inline std::string node_name(uint64_t hi, uint64_t lo) {
    unsigned __int128 v = ((unsigned __int128)hi << 64) | lo;
    int level = (int)(v >> 120);
    std::string s(1, 'r');
    for (int i = level - 1; i >= 0; --i) s.push_back((char)('0' + (int)((v >> (3 * i)) & 7)));
    return s;
}

namespace pb {
inline void put_varint(std::string& s, uint64_t v) {
    do {
        uint8_t b = v & 0x7f;
        v >>= 7;
        if (v) b |= 0x80;
        s.push_back((char)b);
    } while (v);
}
inline void put_key(std::string& s, uint32_t field, uint32_t wire) { put_varint(s, (uint64_t)field << 3 | wire); }
inline void put_double(std::string& s, uint32_t field, double d) {
    uint64_t bits;
    memcpy(&bits, &d, 8);
    if (!bits) return;  // proto3 omits default scalars
    put_key(s, field, 1);
    char b[8];
    memcpy(b, &bits, 8);  // little-endian host
    s.append(b, 8);
}
inline void put_uint(std::string& s, uint32_t field, uint64_t v) {
    if (!v) return;
    put_key(s, field, 0);
    put_varint(s, v);
}
inline void put_bytes(std::string& s, uint32_t field, const std::string& m) {
    put_key(s, field, 2);
    put_varint(s, m.size());
    s += m;
}
struct Cursor {
    const uint8_t* p;
    const uint8_t* end;
    bool bad = false;
    bool more() const { return !bad && p < end; }
    uint64_t varint() {
        uint64_t v = 0;
        for (int sh = 0; p < end && sh < 64; sh += 7) {
            uint8_t b = *p++;
            v |= (uint64_t)(b & 0x7f) << sh;
            if (!(b & 0x80)) return v;
        }
        bad = true;
        return 0;
    }
    double fixed64() {
        if (end - p < 8) {
            bad = true;
            return 0;
        }
        double d;
        memcpy(&d, p, 8);
        p += 8;
        return d;
    }
    float fixed32() {
        if (end - p < 4) {
            bad = true;
            return 0;
        }
        float f;
        memcpy(&f, p, 4);
        p += 4;
        return f;
    }
    Cursor sub() {
        uint64_t n = varint();
        if ((uint64_t)(end - p) < n) {
            bad = true;
            n = 0;
        }
        Cursor c{p, p + n};
        p += n;
        return c;
    }
    void skip(uint32_t wire) {
        switch (wire) {
            case 0: varint(); break;
            case 1: p += 8; break;
            case 2: sub(); break;
            case 5: p += 4; break;
            default: bad = true;
        }
        if (p > end) bad = true;
    }
};
}  // namespace pb

struct MetaHeader {
    double resolution = 0;
    double bbox_min[3] = {0, 0, 0}, bbox_max[3] = {0, 0, 0};
};

inline std::string encode_meta(const MetaHeader& h, const std::vector<pcv_node_meta>& nodes) {
    auto vec3 = [](const double v[3]) {
        std::string s;
        pb::put_double(s, 1, v[0]);
        pb::put_double(s, 2, v[1]);
        pb::put_double(s, 3, v[2]);
        return s;
    };
    std::string cuboid;  // AxisAlignedCuboid { 3: min, 4: max }
    pb::put_bytes(cuboid, 3, vec3(h.bbox_min));
    pb::put_bytes(cuboid, 4, vec3(h.bbox_max));
    std::string octree;  // OctreeMeta { 2: resolution, 3: repeated OctreeNode }
    pb::put_double(octree, 2, h.resolution);
    for (const auto& n : nodes) {
        std::string id;  // NodeId { 3: high, 4: low }
        pb::put_uint(id, 3, n.id_high);
        pb::put_uint(id, 4, n.id_low);
        std::string node;  // OctreeNode { 2: position_encoding, 3: num_points, 4: id }
        pb::put_uint(node, 2, (uint64_t)n.position_encoding);
        pb::put_uint(node, 3, (uint64_t)n.num_points);
        pb::put_bytes(node, 4, id);
        pb::put_bytes(octree, 3, node);
    }
    std::string meta;  // Meta { 1: version, 4: bounding_box, 6: octree }
    pb::put_uint(meta, 1, 13);
    pb::put_bytes(meta, 4, cuboid);
    pb::put_bytes(meta, 6, octree);
    return meta;
}

struct ParsedNode {
    uint64_t hi = 0, lo = 0;
    int64_t num_points = 0;
    int enc = 0;
};

// Version 13 only (the reference also reads 9-12 through deprecated fields; octree/mod.rs:165-194).
inline bool decode_meta(const std::string& buf, MetaHeader& h, std::vector<ParsedNode>& nodes, int& version) {
    pb::Cursor c{(const uint8_t*)buf.data(), (const uint8_t*)buf.data() + buf.size()};
    auto vec3 = [](pb::Cursor v, double out[3]) {
        while (v.more()) {
            uint64_t k = v.varint();
            uint32_t f = (uint32_t)(k >> 3), w = (uint32_t)(k & 7);
            if (w == 1 && f >= 1 && f <= 3)
                out[f - 1] = v.fixed64();
            else
                v.skip(w);
        }
        return !v.bad;
    };
    version = 0;
    while (c.more()) {
        uint64_t k = c.varint();
        uint32_t f = (uint32_t)(k >> 3), w = (uint32_t)(k & 7);
        if (f == 1 && w == 0) {
            version = (int)c.varint();
        } else if (f == 4 && w == 2) {
            pb::Cursor b = c.sub();
            while (b.more()) {
                uint64_t k2 = b.varint();
                uint32_t f2 = (uint32_t)(k2 >> 3), w2 = (uint32_t)(k2 & 7);
                if (f2 == 3 && w2 == 2) {
                    if (!vec3(b.sub(), h.bbox_min)) return false;
                } else if (f2 == 4 && w2 == 2) {
                    if (!vec3(b.sub(), h.bbox_max)) return false;
                } else
                    b.skip(w2);
            }
            if (b.bad) return false;
        } else if (f == 6 && w == 2) {
            pb::Cursor o = c.sub();
            while (o.more()) {
                uint64_t k2 = o.varint();
                uint32_t f2 = (uint32_t)(k2 >> 3), w2 = (uint32_t)(k2 & 7);
                if (f2 == 2 && w2 == 1) {
                    h.resolution = o.fixed64();
                } else if (f2 == 3 && w2 == 2) {
                    pb::Cursor n = o.sub();
                    ParsedNode pn;
                    while (n.more()) {
                        uint64_t k3 = n.varint();
                        uint32_t f3 = (uint32_t)(k3 >> 3), w3 = (uint32_t)(k3 & 7);
                        if (f3 == 2 && w3 == 0)
                            pn.enc = (int)n.varint();
                        else if (f3 == 3 && w3 == 0)
                            pn.num_points = (int64_t)n.varint();
                        else if (f3 == 4 && w3 == 2) {
                            pb::Cursor i = n.sub();
                            while (i.more()) {
                                uint64_t k4 = i.varint();
                                uint32_t f4 = (uint32_t)(k4 >> 3), w4 = (uint32_t)(k4 & 7);
                                if (f4 == 3 && w4 == 0)
                                    pn.hi = i.varint();
                                else if (f4 == 4 && w4 == 0)
                                    pn.lo = i.varint();
                                else
                                    i.skip(w4);
                            }
                            if (i.bad) return false;
                        } else
                            n.skip(w3);
                    }
                    if (n.bad) return false;
                    nodes.push_back(pn);
                } else
                    o.skip(w2);
            }
            if (o.bad) return false;
        } else
            c.skip(w);
    }
    return !c.bad && version == 13;
}

inline bool write_whole_file(const std::string& path, const void* data, size_t n) {
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    bool ok = n == 0 || fwrite(data, 1, n, f) == n;
    ok = fclose(f) == 0 && ok;
    return ok;
}
inline bool read_whole_file(const std::string& path, std::string& out) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    out.resize(n > 0 ? (size_t)n : 0);
    bool ok = n <= 0 || fread(&out[0], 1, (size_t)n, f) == (size_t)n;
    fclose(f);
    return ok;
}

}  // namespace pcv
