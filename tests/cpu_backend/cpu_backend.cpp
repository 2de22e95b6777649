// TEST-ONLY backend for csrc/build_host.hpp: runs the host orchestration (pass planning, bucket
// tables, closed-form subsample plan, output layout) with the kernels replaced by sequential loops
// that follow the CUDA kernels' index arithmetic line by line.  It lets `-m "not gpu"` tests compare
// the product's *algorithm* with the oracle on a machine without a GPU.  It is NOT part of the
// shipped library (libpcv_b200.so contains only the CUDA backend and has no CPU fallback).
#include <cstdlib>
#include <map>

#include "../../include/pcv.h"
#include "../../point_cloud_viewer_b200/csrc/build_host.hpp"
#include "../../point_cloud_viewer_b200/csrc/disk_io.hpp"

using namespace pcv;

namespace {

struct CpuBackend : Backend {
    void* dmalloc(size_t b) override { return std::malloc(b ? b : 16); }
    void dfree(void* p) override { std::free(p); }
    void h2d(void* d, const void* h, size_t b) override { std::memcpy(d, h, b); }
    void d2h(void* h, const void* d, size_t b) override { std::memcpy(h, d, b); }
    // "device" memory is host memory here: the read-back is the buffer itself, kept alive by a private copy
    std::vector<std::vector<uint8_t>> back;
    const void* d2h_begin(const void* d, size_t b) override {
        back.emplace_back((const uint8_t*)d, (const uint8_t*)d + b);
        return back.back().data();
    }
    void d2h_wait() override {
        if (back.size() > 16) back.erase(back.begin(), back.end() - 8);
    }
    void finish_plan(const FinishArgs& f, int last_level) override { finish_plan_seq(f, last_level); }

    static void load_rec(const void* base, uint64_t i, bool wide, uint64_t c[3], uint32_t& idx) {
        if (wide) {
            const RecW& r = ((const RecW*)base)[i];
            c[0] = r.c[0], c[1] = r.c[1], c[2] = r.c[2], idx = r.idx;
        } else {
            const RecN& r = ((const RecN*)base)[i];
            c[0] = r.c[0], c[1] = r.c[1], c[2] = r.c[2], idx = r.idx;
        }
    }
    static void store_rec(void* base, uint64_t i, bool wide, const uint64_t c[3], uint32_t idx) {
        if (wide) {
            RecW& r = ((RecW*)base)[i];
            r.c[0] = c[0], r.c[1] = c[1], r.c[2] = c[2], r.idx = idx, r.pad = 0;
        } else {
            RecN& r = ((RecN*)base)[i];
            r.c[0] = (uint32_t)c[0], r.c[1] = (uint32_t)c[1], r.c[2] = (uint32_t)c[2], r.idx = idx;
        }
    }
    void zero(void* d, size_t b) override { std::memset(d, 0, b); }

    // k_ingest: first step of the chain from the raw position, digits of the first pass
    void ingest(const IngestArgs& a) override {
        for (uint64_t g = 0; g < a.pts.n; ++g) {
            double q[3] = {a.pts.x[g * a.pts.stride], a.pts.y[g * a.pts.stride], a.pts.z[g * a.pts.stride]};
            double m[3] = {a.root_min[0], a.root_min[1], a.root_min[2]};
            Step s = a.lv.fast ? descend_fast(q, m, a.lv.edge[0], a.lv.edge[1], a.lv.ry[1], a.lv.enc[1]) : descend(q, m, a.lv.edge[0], a.lv.edge[1], a.lv.enc[1]);
            unsigned dig = s.digit;
            if (a.G0 == 2) {
                double q2[3] = {q[0], q[1], q[2]}, m2[3] = {m[0], m[1], m[2]};
                Step s2 = a.lv.fast ? descend_fast(q2, m2, a.lv.edge[1], a.lv.edge[2], a.lv.ry[2], a.lv.enc[2]) : descend(q2, m2, a.lv.edge[1], a.lv.edge[2], a.lv.enc[2]);
                dig = (dig << 3) | s2.digit;
            }
            store_rec(a.rec_out, g, a.wide, s.code, (uint32_t)g);
            a.col_out[g] = (uint32_t)a.pts.rgb[3 * g] | ((uint32_t)a.pts.rgb[3 * g + 1] << 8) | ((uint32_t)a.pts.rgb[3 * g + 2] << 16);
            a.dig_out[g] = (uint8_t)dig;
        }
    }

    // k_dighist + k_scan_* + k_plan + k_pass of one pass, sequentially, over the same device-resident state
    void pass(const PassArgs& a) override {
        BuildState* st = a.st;
        const PassState ps = st->pass[a.pass];
        const int nb = a.nbins;
        // digit histogram per tile
        for (uint32_t b = 0; b < ps.ntiles; ++b) {
            const TileDesc t = tile_of(a.active, ps.nactive, b);
            uint32_t* out = a.tile_counts + (size_t)b * nb;
            for (int k = 0; k < nb; ++k) out[k] = 0;
            for (uint32_t i = 0; i < t.count; ++i) out[a.dig_in[t.start + i] & 63]++;
        }
        // scan
        for (uint32_t ch = 0; ch < ps.nchunks; ++ch) {
            const ChunkDesc c = a.chunks[ch];
            for (int b = 0; b < nb; ++b) {
                uint32_t s = 0;
                for (uint32_t t = 0; t < c.ntiles; ++t) s += a.tile_counts[(size_t)(c.tile_begin + t) * nb + b];
                a.chunk_sums[(size_t)ch * nb + b] = s;
            }
        }
        for (uint32_t n = 0; n < ps.nactive; ++n) {
            const ActiveDesc act = a.active[n];
            for (int b = 0; b < nb; ++b) {
                uint64_t run = 0;
                for (uint32_t c = 0; c < act.nchunks; ++c) {
                    uint32_t& v = a.chunk_sums[(size_t)(act.chunk_begin + c) * nb + b];
                    uint32_t old = v;
                    v = (uint32_t)run;
                    run += old;
                }
                a.node_bins[(size_t)n * nb + b] = run;
            }
        }
        for (uint32_t ch = 0; ch < ps.nchunks; ++ch) {
            const ChunkDesc c = a.chunks[ch];
            for (int b = 0; b < nb; ++b) {
                uint32_t run = a.chunk_sums[(size_t)ch * nb + b];
                for (uint32_t t = 0; t < c.ntiles; ++t) {
                    uint32_t& v = a.tile_counts[(size_t)(c.tile_begin + t) * nb + b];
                    uint32_t old = v;
                    v = run;
                    run += old;
                }
            }
        }
        // plan (the product's planner function, one active node after the other)
        PlanRun run{};
        run.nodes = st->nnodes;
        run.arena_pts = st->arena_used;
        int32_t err = 0;
        uint32_t deepest = st->deepest_level;
        for (uint32_t ai = 0; ai < ps.nactive; ++ai) {
            PlanRun cnt{};
            plan_active<false>(a, ai, cnt, err, deepest);
            if ((uint64_t)run.nodes + cnt.nodes > a.cap_nodes || (uint64_t)run.actives + cnt.actives > a.cap_active || (uint64_t)run.tiles + cnt.tiles > a.cap_tiles ||
                (uint64_t)run.chunks + cnt.chunks > a.cap_chunks)
                err = kErrCapacity;
            int32_t e2 = 0;
            uint32_t d2 = 0;
            plan_active<true>(a, ai, run, e2, d2);  // emit advances the running bases by exactly the node's demand
        }
        if (err && !st->error) st->error = err;
        PassState nx{};
        if (!st->error) {
            nx.nactive = run.actives;
            nx.ntiles = run.tiles;
            nx.nchunks = run.chunks;
            nx.npoints = run.next_pts;
        }
        st->pass[a.pass + 1] = nx;
        st->nnodes = run.nodes;
        st->arena_used = run.arena_pts;
        st->deepest_level = deepest;
        if (st->error) return;
        // partition + the next pass's descent (k_pass), tile by tile in tile order == stable order
        std::vector<uint32_t> incl(nb), base(nb), lut(nb);
        std::vector<BucketDesc> bds(nb);
        for (uint32_t blk = 0; blk < ps.ntiles; ++blk) {
            const TileDesc t = tile_of(a.active, ps.nactive, blk);
            const ActiveDesc act = a.active[t.active];
            const uint32_t* pfx = a.tile_counts + (size_t)blk * nb;
            uint32_t r = 0;
            for (int b = 0; b < nb; ++b) {
                r += pfx[b];
                incl[b] = r;
                lut[b] = 0xFFFF;
            }
            for (int lb = 0; lb < nb; ++lb) {
                const BucketDesc bd = a.buckets[(size_t)t.active * nb + lb];
                bds[lb] = bd;
                base[lb] = 0;
                if (bd.b1 != 0) {
                    const uint32_t hi = incl[bd.b1 - 1], lo = bd.b0 ? incl[bd.b0 - 1] : 0u;
                    base[lb] = (uint32_t)bd.dest + (hi - lo);
                    for (uint32_t d = bd.b0; d < bd.b1; ++d) lut[d] = (uint32_t)lb;
                }
            }
            for (uint32_t i = 0; i < t.count; ++i) {
                const uint64_t g = t.start + i;
                uint64_t c[3];
                uint32_t idx;
                load_rec(a.rec_in, g, a.wide, c, idx);
                const unsigned dig = a.dig_in[g];
                const uint32_t lb = lut[dig];
                const BucketDesc& bd = bds[lb];
                const bool next = bd.kind == 0;
                const uint32_t dst = base[lb]++;
                unsigned dig_out = 0;
                if (next || bd.keep == 2) {
                    const int L1 = a.level + 1;
                    const unsigned d1 = a.G == 2 ? (dig >> 3) : dig, d2 = dig & 7u;
                    const double e1 = a.lv.edge[L1];
                    double m[3] = {(d1 & 4u) ? act.m[0] + e1 : act.m[0], (d1 & 2u) ? act.m[1] + e1 : act.m[1], (d1 & 1u) ? act.m[2] + e1 : act.m[2]};
                    double q[3];
                    for (int k = 0; k < 3; ++k) q[k] = a.lv.fast ? decode1_fast(c[k], m[k], e1, a.lv.enc[L1]) : decode1(c[k], m[k], e1, a.lv.enc[L1]);
                    int Lb = L1;
                    if (bd.keep == 2) {
                        const int L2 = L1 + 1;
                        const double e2 = a.lv.edge[L2];
                        if (d2 & 4u) m[0] = m[0] + e2;
                        if (d2 & 2u) m[1] = m[1] + e2;
                        if (d2 & 1u) m[2] = m[2] + e2;
                        for (int k = 0; k < 3; ++k) {
                            c[k] = a.lv.fast ? encode1_fast(q[k], m[k], e2, a.lv.ry[L2], a.lv.enc[L2]) : encode1(q[k], m[k], e2, a.lv.enc[L2]);
                            q[k] = a.lv.fast ? decode1_fast(c[k], m[k], e2, a.lv.enc[L2]) : decode1(c[k], m[k], e2, a.lv.enc[L2]);
                        }
                        Lb = L2;
                    }
                    if (next) {
                        Step s = a.lv.fast ? descend_fast(q, m, a.lv.edge[Lb], a.lv.edge[Lb + 1], a.lv.ry[Lb + 1], a.lv.enc[Lb + 1])
                                           : descend(q, m, a.lv.edge[Lb], a.lv.edge[Lb + 1], a.lv.enc[Lb + 1]);
                        dig_out = s.digit;
                        for (int k = 0; k < 3; ++k) c[k] = s.code[k];
                        if (a.Gn == 2) {
                            Step s2 = a.lv.fast ? descend_fast(q, m, a.lv.edge[Lb + 1], a.lv.edge[Lb + 2], a.lv.ry[Lb + 2], a.lv.enc[Lb + 2])
                                                : descend(q, m, a.lv.edge[Lb + 1], a.lv.edge[Lb + 2], a.lv.enc[Lb + 2]);
                            dig_out = (dig_out << 3) | s2.digit;
                        }
                    }
                }
                store_rec(next ? a.rec_next : a.arena, dst, a.wide, c, idx);
                (next ? a.col_next : a.col_arena)[dst] = a.col_in[g];
                if (next) a.dig_next[dst] = (uint8_t)dig_out;
            }
        }
    }
    void place(const PlaceArgs& a) override {
        for (uint32_t b = 0; b < a.ntiles; ++b) {
            const LeafTile lt = leaf_tile_of(a, b);
            const DNode leaf = a.d_nodes[lt.node];
            for (uint32_t i = 0; i < lt.count; ++i) {
                uint64_t c[3];
                uint32_t idx;
                load_rec(a.arena, lt.arena_start + i, a.wide, c, idx);
                uint64_t j = lt.j0 + i;
                DNode nd = leaf;
                while (nd.parent >= 0 && (j & 7) == 0) {
                    const DNode P = a.d_nodes[nd.parent];
                    for (int k = 0; k < 3; ++k)
                        c[k] = a.fast ? encode1_fast(decode1_fast(c[k], nd.m[k], nd.e, nd.enc), P.m[k], P.e, P.ry, P.enc)
                                      : encode1(decode1(c[k], nd.m[k], nd.e, nd.enc), P.m[k], P.e, P.enc);
                    j = nd.off_in_parent + (j >> 3);
                    nd = P;
                }
                uint64_t slot = j;
                if (nd.parent >= 0) {
                    for (int k = 0; k < 3; ++k)
                        c[k] = a.fast ? encode1_fast(decode1_fast(c[k], nd.m[k], nd.e, nd.enc), nd.m[k], nd.e, nd.ry, nd.enc)
                                      : encode1(decode1(c[k], nd.m[k], nd.e, nd.enc), nd.m[k], nd.e, nd.enc);
                    slot = j - (j >> 3) - 1;
                }
                const uint64_t dp = nd.out_point_off + slot;
                const int bpc = enc_bytes(nd.enc);
                uint8_t* px = a.out_xyz + nd.out_xyz_off + slot * 3 * (uint64_t)bpc;
                for (int k = 0; k < 3; ++k) std::memcpy(px + k * bpc, &c[k], (size_t)bpc);  // little-endian host
                const uint32_t col = a.col_arena[lt.arena_start + i];
                a.out_rgb[3 * dp] = (uint8_t)col;
                a.out_rgb[3 * dp + 1] = (uint8_t)(col >> 8);
                a.out_rgb[3 * dp + 2] = (uint8_t)(col >> 16);
                a.out_src[dp] = idx;
                if (a.out_intensity) a.out_intensity[dp] = a.pts.intensity[idx];
            }
        }
    }
};

struct TbTree {
    BuildResult R;
    std::vector<pcv_node_meta> nodes;
};

}  // namespace

extern "C" {

void* tb_build(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, const uint8_t* rgb, const float* intensity,
               double resolution, const double* bmin, const double* bmax, uint64_t max_points, int levels_per_pass, char* err, int errcap) {
    CpuBackend be;
    PointsView v{x, y, z, stride, rgb, intensity, n};
    try {
        BuildPlan plan(be, max_points, levels_per_pass);
        TbTree* t = new TbTree();
        t->R = plan.run(v, resolution, bmin, bmax);
        for (int i : t->R.sorted) {
            const HNode& h = t->R.nodes[i];
            pcv_node_meta m{};
            u128 id = ((u128)h.level << 120) | h.index;
            m.id_high = (uint64_t)(id >> 64);
            m.id_low = (uint64_t)id;
            m.num_points = (int64_t)h.final_count;
            m.position_encoding = h.enc;
            m.level = h.level;
            for (int a = 0; a < 3; ++a) m.cube_min[a] = h.m[a];
            m.cube_edge = h.e;
            m.point_offset = h.out_point_off;
            m.xyz_byte_offset = h.out_xyz_off;
            t->nodes.push_back(m);
        }
        return t;
    } catch (const std::exception& e) {
        if (err) snprintf(err, (size_t)errcap, "%s", e.what());
        return nullptr;
    }
}
uint64_t tb_num_nodes(void* h) { return ((TbTree*)h)->nodes.size(); }
void tb_nodes(void* h, pcv_node_meta* out) { std::memcpy(out, ((TbTree*)h)->nodes.data(), ((TbTree*)h)->nodes.size() * sizeof(pcv_node_meta)); }
uint64_t tb_xyz_bytes(void* h) { return ((TbTree*)h)->R.xyz_bytes; }
uint32_t tb_passes(void* h) { return ((TbTree*)h)->R.passes; }
void tb_download(void* h, uint8_t* xyz, uint8_t* rgb, float* intensity, uint32_t* src) {
    BuildResult& R = ((TbTree*)h)->R;
    if (R.n == 0) return;
    std::memcpy(xyz, R.d_xyz, R.xyz_bytes);
    std::memcpy(rgb, R.d_rgb, R.n * 3);
    if (intensity && R.d_intensity) std::memcpy(intensity, R.d_intensity, R.n * 4);
    std::memcpy(src, R.d_src, R.n * 4);
}
void tb_free(void* h) {
    TbTree* t = (TbTree*)h;
    std::free(t->R.d_xyz);
    std::free(t->R.d_rgb);
    std::free(t->R.d_intensity);
    std::free(t->R.d_src);
    delete t;
}
}

// ---- exactness checks of the fast paths in chain.h (host execution) -----------------------------------------
extern "C" {
// exhaustive: unit_frac<8>/<16>(v) == (double)v / 255.0 | 65535.0 for every v; returns the number of mismatches
uint64_t tb_check_unit_frac() {
    uint64_t bad = 0;
    for (uint32_t v = 0; v <= 255; ++v) {
        bad += pcv::f64_to_bits(pcv::unit_frac<8>(v)) != pcv::f64_to_bits((double)v / 255.0);
        bad += pcv::f64_to_bits(pcv::unit_frac_int<8>(v)) != pcv::f64_to_bits((double)v / 255.0);
    }
    for (uint32_t v = 0; v <= 65535; ++v) {
        bad += pcv::f64_to_bits(pcv::unit_frac<16>(v)) != pcv::f64_to_bits((double)v / 65535.0);
        bad += pcv::f64_to_bits(pcv::unit_frac_int<16>(v)) != pcv::f64_to_bits((double)v / 65535.0);
    }
    return bad;
}
// random + adversarial: div_known(a, b, 1/b) == a / b.  Divisors are edge-like (E * 2^-L), numerators are the
// differences the descent produces (multiples of an ulp near the cube) plus near-tie constructions a = RN((k+0.5ulp) * b).
uint64_t tb_check_div(uint64_t n, uint64_t seed) {
    uint64_t bad = 0, s = seed;
    auto next = [&]() {
        s += 0x9E3779B97F4A7C15ull;
        uint64_t x = s;
        x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
        x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
        return x ^ (x >> 31);
    };
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t r0 = next(), r1 = next(), r2 = next();
        double b = 1.0 + (double)(r0 >> 11) * 0x1.0p-53;          // significand
        b = std::ldexp(b, (int)(r1 % 60) - 40);                     // edges from 2^-40 to 2^19
        if (!pcv::div_known_ok(b)) continue;
        const double y = 1.0 / b;
        double a;
        switch (r2 & 3) {
            case 0: a = b * ((double)(r1 >> 11) * 0x1.0p-53); break;                       // t uniform in [0,1)
            case 1: a = b * ((double)(r2 >> 40) / 65535.0); break;                          // near code lattice
            case 2: {                                                                       // near-tie quotients
                double q = 1.0 + (double)(r1 >> 12) * 0x1.0p-52;
                a = q * b;
                a = std::nextafter(a, (r2 & 4) ? 0.0 : 4.0 * a);
                break;
            }
            default: a = std::ldexp(1.0 + (double)(r2 >> 11) * 0x1.0p-53, (int)(r1 % 200) - 100) * ((r2 & 8) ? -1.0 : 1.0);  // wide range
        }
        bad += pcv::f64_to_bits(pcv::div_known(a, b, y)) != pcv::f64_to_bits(a / b);
    }
    // guard paths: zero, tiny, huge, inf, nan numerators
    const double specials[] = {0.0, -0.0, 1e-320, 1e-200, 1e200, INFINITY, -INFINITY, NAN};
    for (double a : specials) {
        const double b = 3.7, y = 1.0 / b, r = pcv::div_known(a, b, y), w = a / b;
        bad += !((r != r && w != w) || pcv::f64_to_bits(r) == pcv::f64_to_bits(w));
    }
    return bad;
}
// The level table the build derives from a root cube (make_level_table, so PCV_CHECKED_FAST / PCV_NO_POW2 apply as in the
// library): the division mode, the deepest level and the encoding of every level.  root_min may be NULL.
void tb_level_table(double root_edge, double resolution, const double* root_min, int* fast, int* last_level, int8_t* enc) {
    const LevelTable t = make_level_table(root_edge, resolution, root_min);
    *fast = t.fast;
    *last_level = t.last_level;
    for (int L = 0; L < kMaxLevels; ++L) enc[L] = t.enc[L];
}
// div_known's Markstein sequence WITHOUT its range guard: what a kernel stores for a flagged numerator if the block did not
// repeat the work with the IEEE operator
double tb_div_unguarded(double a, double b, double y) {
    const double q0 = a * y;
    const double q1 = std::fma(std::fma(-q0, b, a), y, q0);
    return std::fma(std::fma(-q1, b, a), y, q1);
}
// encode/decode fast == plain for random cubes at ECEF-like offsets, all encodings
uint64_t tb_check_codec(uint64_t n, uint64_t seed) {
    uint64_t bad = 0, s = seed;
    auto next = [&]() {
        s += 0x9E3779B97F4A7C15ull;
        uint64_t x = s;
        x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
        x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
        return x ^ (x >> 31);
    };
    for (uint64_t i = 0; i < n; ++i) {
        const uint64_t r0 = next(), r1 = next(), r2 = next();
        const double edge = std::ldexp(1.0 + (double)(r0 >> 11) * 0x1.0p-53, (int)(r1 % 30) - 12);
        if (!pcv::div_known_ok(edge)) continue;
        const double mn = ((double)(int64_t)(r1 >> 20) - 8.0e12) * 1e-6;  // up to +-8e6 (ECEF scale)
        const double v = mn + edge * (((double)(r2 >> 11) * 0x1.0p-53) * 1.002 - 0.001);  // slightly outside too
        for (int enc = 1; enc <= 4; ++enc) {
            const uint64_t c0 = pcv::encode1(v, mn, edge, enc), c1 = pcv::encode1_fast(v, mn, edge, 1.0 / edge, enc);
            bad += c0 != c1;
            bad += pcv::f64_to_bits(pcv::decode1(c0, mn, edge, enc)) != pcv::f64_to_bits(pcv::decode1_fast(c0, mn, edge, enc));
        }
    }
    return bad;
}
}

// ---- sharded build with the sequential stand-ins (host logic of the multi-GPU path) ---------------------------
extern "C" {
void tb_prefix_cells(uint64_t n, const double* x, const double* y, const double* z, uint64_t stride, double resolution, const double* bmin,
                     const double* bmax, int k, uint32_t* cells_out) {
    const double E = std::fmax(std::fmax(bmax[0] - bmin[0], bmax[1] - bmin[1]), bmax[2] - bmin[2]);
    const LevelTable lv = make_level_table(E, resolution);
    for (uint64_t i = 0; i < n; ++i) {
        double q[3] = {x[i * stride], y[i * stride], z[i * stride]}, m[3] = {bmin[0], bmin[1], bmin[2]}, e = lv.edge[0];
        uint32_t cell = 0;
        for (int j = 1; j <= k; ++j) {
            Step s = lv.fast ? descend_fast(q, m, e, lv.edge[j], lv.ry[j], lv.enc[j]) : descend(q, m, e, lv.edge[j], lv.enc[j]);
            cell = (cell << 3) | s.digit;
            e = lv.edge[j];
        }
        cells_out[i] = cell;
    }
}

static void* tb_wrap(BuildResult&& R) {
    TbTree* t = new TbTree();
    t->R = std::move(R);
    for (int i : t->R.sorted) {
        const HNode& h = t->R.nodes[i];
        pcv_node_meta m{};
        u128 id = ((u128)h.level << 120) | h.index;
        m.id_high = (uint64_t)(id >> 64);
        m.id_low = (uint64_t)id;
        m.num_points = (int64_t)h.final_count;
        m.position_encoding = h.enc;
        m.level = h.level;
        for (int a = 0; a < 3; ++a) m.cube_min[a] = h.m[a];
        m.cube_edge = h.e;
        m.point_offset = h.out_point_off;
        m.xyz_byte_offset = h.out_xyz_off;
        t->nodes.push_back(m);
    }
    return t;
}

void* tb_build_sharded(uint64_t n, const double* xyz_aos, const uint8_t* rgb, const float* intensity, double resolution, const double* bmin,
                       const double* bmax, uint64_t max_points, int levels_per_pass, int k, const uint64_t* prefix_counts, char* err, int errcap) {
    CpuBackend be;
    PointsView v{xyz_aos, xyz_aos + 1, xyz_aos + 2, 3, rgb, intensity, n};
    try {
        BuildPlan plan(be, max_points, levels_per_pass);
        plan.shard.k = k;
        plan.shard.counts = prefix_counts;
        return tb_wrap(plan.run(v, resolution, bmin, bmax));
    } catch (const std::exception& e) {
        if (err) snprintf(err, (size_t)errcap, "%s", e.what());
        return nullptr;
    }
}

void* tb_assemble_top(double resolution, const double* bmin, const double* bmax, int k, const uint64_t* prefix_counts, const uint64_t* unit_nsub,
                      const uint8_t* xyz, const uint8_t* rgb, const float* intensity, uint64_t npoints, char* err, int errcap) {
    CpuBackend be;
    try {
        return tb_wrap(assemble_top(be, resolution, bmin, bmax, k, prefix_counts, unit_nsub, xyz, rgb, intensity, npoints));
    } catch (const std::exception& e) {
        if (err) snprintf(err, (size_t)errcap, "%s", e.what());
        return nullptr;
    }
}

// n(X) of every node, in the order of tb_nodes
void tb_nsub(void* h, uint64_t* out) {
    TbTree* t = (TbTree*)h;
    size_t k = 0;
    for (int i : t->R.sorted) out[k++] = t->R.nodes[i].n_sub;
}
}

// ---- the product's meta.pb writer / reader (csrc/disk_io.hpp), host code: pinned against python-protobuf on the CPU ----
extern "C" {
// nodes: n x (high, low, num_points, enc).  Returns the byte count (or -needed if cap is too small).
int64_t tb_encode_meta(double resolution, const double* bmin, const double* bmax, const uint64_t* nodes4, uint64_t n, uint8_t* out, uint64_t cap) {
    MetaHeader h;
    h.resolution = resolution;
    for (int a = 0; a < 3; ++a) h.bbox_min[a] = bmin[a], h.bbox_max[a] = bmax[a];
    std::vector<pcv_node_meta> v(n);
    for (uint64_t i = 0; i < n; ++i) {
        v[i] = pcv_node_meta{};
        v[i].id_high = nodes4[4 * i];
        v[i].id_low = nodes4[4 * i + 1];
        v[i].num_points = (int64_t)nodes4[4 * i + 2];
        v[i].position_encoding = (int32_t)nodes4[4 * i + 3];
    }
    const std::string s = encode_meta(h, v);
    if (s.size() > cap) return -(int64_t)s.size();
    std::memcpy(out, s.data(), s.size());
    return (int64_t)s.size();
}
// Returns the node count (or -1 if rejected); nodes4 receives up to cap entries.
int64_t tb_decode_meta(const uint8_t* buf, uint64_t len, double* resolution, double* bmin, double* bmax, int* version, uint64_t* nodes4, uint64_t cap) {
    MetaHeader h;
    std::vector<ParsedNode> pn;
    int ver = 0;
    const bool ok = decode_meta(std::string((const char*)buf, len), h, pn, ver);
    *version = ver;
    if (!ok) return -1;
    *resolution = h.resolution;
    for (int a = 0; a < 3; ++a) bmin[a] = h.bbox_min[a], bmax[a] = h.bbox_max[a];
    for (uint64_t i = 0; i < pn.size() && i < cap; ++i) {
        nodes4[4 * i] = pn[i].hi, nodes4[4 * i + 1] = pn[i].lo, nodes4[4 * i + 2] = (uint64_t)pn[i].num_points, nodes4[4 * i + 3] = (uint64_t)pn[i].enc;
    }
    return (int64_t)pn.size();
}
}
