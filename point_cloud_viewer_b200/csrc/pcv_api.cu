// pcv_api.cu — the C ABI (include/pcv.h) over the CUDA kernels.  One translation unit; built with
//   nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo ... (see __graft_entry__.build()).
// There is no CPU fallback in this library: every compute entry point needs a CUDA device.
#include <cuda_runtime.h>
#include <sys/stat.h>

#include <cstdarg>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <functional>
#include <string>
#include <memory>
#include <thread>

#include "../../include/pcv.h"
#include "dir_query_plan.h"
#include "disk_io.hpp"
#include "octree_obj.hpp"
#include "ooc_plan.h"
#include "ply.cuh"
#include "ply_host.hpp"
#include "kernels_shard.cuh"
#include "query.cuh"
#include "xray_pyramid.cuh"
#include "xray_dir_plan.h"
#include "s2.cuh"
#include "s2_dir_writer.hpp"
#include "s2_stream_plan.h"
#include "synth.cuh"

using namespace pcv;

static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define API_TRY try {
#define API_CATCH                                            \
    }                                                        \
    catch (const BuildError& e) { return fail(e.code, "%s", e.what()); } \
    catch (const std::bad_alloc&) { return fail(PCV_ERR_INVALID, "host out of memory"); } \
    catch (const std::exception& e) { return fail(PCV_ERR_INVALID, "%s", e.what()); }

static void sharded_forget(pcv_ctx* c);  // sharded_build.inl: drops the slab a context still caches (no collective)

extern "C" {

const char* pcv_last_error(void) { return g_err.c_str(); }

int pcv_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int pcv_create(int device, const pcv_config* cfg, pcv_ctx** out) {
    if (!out) return fail(PCV_ERR_INVALID, "out is null");
    *out = nullptr;
    API_TRY
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(PCV_ERR_CUDA, "no CUDA device: this library has no CPU fallback");
    }
    if (device < 0 || device >= n) return fail(PCV_ERR_INVALID, "device %d out of range (have %d)", device, n);
    CU(cudaSetDevice(device));
    pcv_ctx* c = new pcv_ctx();
    c->device = device;
    if (cfg) c->cfg = *cfg;
    if (c->cfg.max_points_per_node == 0) c->cfg.max_points_per_node = 100000;
    if (c->cfg.levels_per_pass == 0 || c->cfg.levels_per_pass > 3) c->cfg.levels_per_pass = 3;
    CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CU(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device));
    // keep freed blocks in the stream-ordered pool so repeated builds do not pay cudaMalloc again
    cudaMemPool_t pool;
    CU(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thr = UINT64_MAX;
    CU(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    c->be = new CudaBackend(c->stream);
    // per-device attribute (a second context on another GPU of the same process needs its own opt-in)
    CU(cudaFuncSetAttribute(k_ply_unpack, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CU(cudaFuncSetAttribute(k_xray_subtile, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kXraySub * kXraySub * 128)));
    *out = c;
    return PCV_OK;
    API_CATCH
}

void pcv_destroy(pcv_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    sharded_forget(c);
    c->be->dfree(c->shard_cells);
    cudaStreamSynchronize(c->stream);
    delete c->be;
    cudaStreamDestroy(c->stream);
    delete c;
}

static PointsView view_of(const pcv_points* p) {
    PointsView v;
    v.x = p->x;
    v.y = p->y;
    v.z = p->z;
    v.stride = p->stride ? p->stride : 1;
    v.rgb = p->rgb;
    v.intensity = p->intensity;
    v.n = p->n;
    return v;
}

// Host points -> freshly allocated device copies, held by `owned`.
static PointsView stage_points(pcv_ctx* c, const pcv_points* hp, Scratch& owned) {
    PointsView v{};
    v.n = hp->n;
    const uint64_t n = hp->n;
    const uint64_t stride = hp->stride ? hp->stride : 1;
    if (n == 0) return v;
    if (stride == 3 && hp->y == hp->x + 1 && hp->z == hp->x + 2) {
        double* d = owned.alloc<double>(n * 3);
        CU(cudaMemcpyAsync(d, hp->x, n * 24, cudaMemcpyHostToDevice, c->stream));
        v.x = d;
        v.y = d + 1;
        v.z = d + 2;
        v.stride = 3;
    } else if (stride == 1) {
        // three separate blocks: after earlier builds the stream-ordered pool holds free blocks of the working-set sizes
        // (N x 16 / 4 bytes), which an N x 8 request can reuse; one N x 24 block would make the pool map fresh memory on
        // every call (measured: +0.5 s per 1e9-point call)
        const double* src[3] = {hp->x, hp->y, hp->z};
        const double* dst[3];
        for (int k = 0; k < 3; ++k) {
            double* d = owned.alloc<double>(n);
            CU(cudaMemcpyAsync(d, src[k], n * 8, cudaMemcpyHostToDevice, c->stream));
            dst[k] = d;
        }
        v.x = dst[0];
        v.y = dst[1];
        v.z = dst[2];
        v.stride = 1;
    } else {
        throw BuildError(PCV_ERR_INVALID, "positions must be SoA (stride 1) or interleaved xyz (stride 3, y=x+1, z=x+2)");
    }
    if (hp->rgb) {
        uint8_t* r = owned.alloc<uint8_t>(n * 3);
        CU(cudaMemcpyAsync(r, hp->rgb, n * 3, cudaMemcpyHostToDevice, c->stream));
        v.rgb = r;
    }
    if (hp->intensity) {
        float* f = owned.alloc<float>(n);
        CU(cudaMemcpyAsync(f, hp->intensity, n * 4, cudaMemcpyHostToDevice, c->stream));
        v.intensity = f;
    }
    return v;
}

int pcv_bbox_device(pcv_ctx* c, const pcv_points* dp, double out_min[3], double out_max[3]) {
    if (!c || !dp || !out_min || !out_max) return fail(PCV_ERR_INVALID, "null argument");
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    c->be->bbox(view_of(dp), out_min, out_max);
    return PCV_OK;
    API_CATCH
}

int pcv_bbox(pcv_ctx* c, const pcv_points* hp, double out_min[3], double out_max[3]) {
    if (!c || !hp || !out_min || !out_max) return fail(PCV_ERR_INVALID, "null argument");
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    Scratch owned(c);
    pcv_points tmp = *hp;
    tmp.rgb = nullptr;
    tmp.intensity = nullptr;
    PointsView v = stage_points(c, &tmp, owned);
    c->be->bbox(v, out_min, out_max);
    return PCV_OK;
    API_CATCH
}

static pcv_octree* octree_from_result(pcv_ctx* c, BuildResult& R, double resolution, const double bmin[3], const double bmax[3],
                                      bool has_intensity) {
    pcv_octree* o = new pcv_octree();
    o->ctx = c;
    o->resolution = resolution;
    // Aabb::new takes inf/sup of the two corners (aabb.rs:19-24)
    for (int a = 0; a < 3; ++a) {
        o->bbox_min[a] = std::fmin(bmin[a], bmax[a]);
        o->bbox_max[a] = std::fmax(bmin[a], bmax[a]);
    }
    o->has_intensity = has_intensity;
    o->n = R.n;
    o->xyz_bytes = R.xyz_bytes;
    o->d_xyz = R.d_xyz;
    o->d_rgb = R.d_rgb;
    o->d_intensity = R.d_intensity;
    o->d_src = R.d_src;
    o->nodes.reserve(R.sorted.size());
    for (int i : R.sorted) {
        const HNode& x = R.nodes[i];
        pcv_node_meta m{};
        const u128 id = ((u128)x.level << 120) | x.index;  // node.rs:108-111
        m.id_high = (uint64_t)(id >> 64);
        m.id_low = (uint64_t)id;
        m.num_points = (int64_t)x.final_count;
        m.position_encoding = x.enc;
        m.level = x.level;
        for (int a = 0; a < 3; ++a) m.cube_min[a] = x.m[a];
        m.cube_edge = x.e;
        m.point_offset = x.out_point_off;
        m.xyz_byte_offset = x.out_xyz_off;
        o->nodes.push_back(m);
        o->nsub.push_back(x.n_sub);
    }
    return o;
}

static int build_impl(pcv_ctx* c, const PointsView& v, double resolution, const double bmin_in[3], const double bmax_in[3],
                      pcv_octree** out, const ShardSpec* shard = nullptr, const ExternalRecords* ext = nullptr) {
    double bmin[3], bmax[3];
    for (int a = 0; a < 3; ++a) {
        bmin[a] = std::fmin(bmin_in[a], bmax_in[a]);
        bmax[a] = std::fmax(bmin_in[a], bmax_in[a]);
    }
    if (v.n && !v.rgb) throw BuildError(PCV_ERR_INVALID, "color is mandatory (point counts come from .rgb, on_disk.rs:23-33)");
    CudaBackend& be = *c->be;
    const uint64_t l0 = be.launches;
    Events<2> ev;
    CU(cudaEventRecord(ev.e[0], c->stream));
    BuildPlan plan(be, c->cfg.max_points_per_node, (int)c->cfg.levels_per_pass);
    if (shard) plan.shard = *shard;
    if (ext) plan.ext = *ext;
    BuildResult R = plan.run(v, resolution, bmin, bmax);
    CU(cudaEventRecord(ev.e[1], c->stream));
    CU(cudaStreamSynchronize(c->stream));
    pcv_build_stats& s = c->stats;
    s = pcv_build_stats{};
    s.kernel_launches = be.launches - l0;
    s.passes = R.passes;
    s.deepest_level = R.deepest_level;
    s.num_nodes = R.nodes.size();
    s.algorithmic_bytes = R.algorithmic_bytes;
    s.ms_host_plan = (float)R.host_ms_plan;
    s.ms_host_wait = (float)R.host_ms_wait;
    cudaEventElapsedTime(&s.ms_total, ev.e[0], ev.e[1]);
    if (v.n) {
        cudaEventElapsedTime(&s.ms_partition, be.ev[0], be.ev[1]);
        cudaEventElapsedTime(&s.ms_place, be.ev[1], be.ev[2]);
    }
    *out = octree_from_result(c, R, resolution, bmin, bmax, v.intensity != nullptr);
    return PCV_OK;
}

int pcv_build_octree_device(pcv_ctx* c, const pcv_points* dp, double resolution, const double bbox_min[3], const double bbox_max[3],
                            pcv_octree** out) {
    if (!c || !dp || !bbox_min || !bbox_max || !out) return fail(PCV_ERR_INVALID, "null argument");
    *out = nullptr;
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    return build_impl(c, view_of(dp), resolution, bbox_min, bbox_max, out);
    API_CATCH
}

int pcv_build_octree(pcv_ctx* c, const pcv_points* hp, double resolution, const double bbox_min[3], const double bbox_max[3],
                     pcv_octree** out) {
    if (!c || !hp || !bbox_min || !bbox_max || !out) return fail(PCV_ERR_INVALID, "null argument");
    *out = nullptr;
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    Scratch owned(c);
    const bool timing = std::getenv("PCV_TIMING") != nullptr;
    const auto t0 = std::chrono::steady_clock::now();
    PointsView v = stage_points(c, hp, owned);
    if (timing) {  // diagnostic only: the extra synchronisation separates the copies from the build
        CU(cudaStreamSynchronize(c->stream));
        const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
        fprintf(stderr, "[pcv_build_octree] staged %.2f GB host->device in %.1f ms (%.1f GB/s)\n", hp->n * 27e-9, ms, hp->n * 27e-6 / ms);
    }
    return build_impl(c, v, resolution, bbox_min, bbox_max, out);
    API_CATCH
}

void pcv_octree_free(pcv_octree* o) {
    if (!o) return;
    pcv_ctx* c = o->ctx;
    cudaSetDevice(c->device);
    delete o;
    cudaStreamSynchronize(c->stream);
}

int pcv_device_alloc(pcv_ctx* c, uint64_t bytes, void** out) {
    if (!c || !out) return fail(PCV_ERR_INVALID, "null argument");
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    *out = c->be->dmalloc(bytes);
    CU(cudaStreamSynchronize(c->stream));
    return PCV_OK;
    API_CATCH
}
int pcv_device_free(pcv_ctx* c, void* ptr) {
    if (!c) return fail(PCV_ERR_INVALID, "null context");
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    c->be->dfree(ptr);
    return PCV_OK;
}

int pcv_release_cached_memory(pcv_ctx* c) {
    if (!c) return fail(PCV_ERR_INVALID, "null context");
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    c->be->cache_release();
    cudaMemPool_t pool;
    CU(cudaDeviceGetDefaultMemPool(&pool, c->device));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaMemPoolTrimTo(pool, 0));
    return PCV_OK;
    API_CATCH
}

int pcv_last_build_stats(pcv_ctx* c, pcv_build_stats* out) {
    if (!c || !out) return fail(PCV_ERR_INVALID, "null argument");
    *out = c->stats;
    return PCV_OK;
}
uint64_t pcv_kernel_launch_count(pcv_ctx* c) { return c ? c->be->launches : 0; }

int pcv_set_profiling(pcv_ctx* c, int on) {
    if (!c) return fail(PCV_ERR_INVALID, "null context");
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->be->prof_collect();
    c->be->prof_reset();
    c->be->profile = on != 0;
    return PCV_OK;
}

int pcv_kernel_stats(pcv_ctx* c, pcv_kernel_stat* out, uint32_t cap, uint32_t* n_out) {
    if (!c || !n_out) return fail(PCV_ERR_INVALID, "null argument");
    std::lock_guard<std::mutex> g(c->mu);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->be->prof_collect();
    static const char* names[CudaBackend::K_COUNT] = {"k_bbox", "k_ingest", "k_dighist", "k_scan", "k_plan", "k_pass", "k_place", "k_ply_unpack"};
    uint32_t n = 0;
    for (int k = 0; k < CudaBackend::K_COUNT; ++k) {
        if (n < cap && out) {
            pcv_kernel_stat& s = out[n];
            memset(&s, 0, sizeof s);
            snprintf(s.name, sizeof s.name, "%s", names[k]);
            s.launches = c->be->kstat[k].launches;
            s.algorithmic_bytes = c->be->kstat[k].bytes;
            s.ms = c->be->kstat[k].ms;
        }
        ++n;
    }
    *n_out = n;
    return PCV_OK;
}

int pcv_octree_info(const pcv_octree* o, uint64_t* num_nodes, uint64_t* num_points, uint64_t* xyz_bytes, double* resolution,
                    double bbox_min[3], double bbox_max[3], int* has_intensity) {
    if (!o) return fail(PCV_ERR_INVALID, "null octree");
    if (num_nodes) *num_nodes = o->nodes.size();
    if (num_points) *num_points = o->n;
    if (xyz_bytes) *xyz_bytes = o->xyz_bytes;
    if (resolution) *resolution = o->resolution;
    for (int a = 0; a < 3; ++a) {
        if (bbox_min) bbox_min[a] = o->bbox_min[a];
        if (bbox_max) bbox_max[a] = o->bbox_max[a];
    }
    if (has_intensity) *has_intensity = o->has_intensity ? 1 : 0;
    return PCV_OK;
}

int pcv_octree_nodes(const pcv_octree* o, pcv_node_meta* out, uint64_t cap) {
    if (!o || (!out && cap)) return fail(PCV_ERR_INVALID, "null argument");
    if (cap < o->nodes.size()) return fail(PCV_ERR_INVALID, "capacity %llu < %zu nodes", (unsigned long long)cap, o->nodes.size());
    memcpy(out, o->nodes.data(), o->nodes.size() * sizeof(pcv_node_meta));
    return PCV_OK;
}

static void widen_src(const std::vector<uint32_t>& in, uint64_t* out) {
    for (size_t i = 0; i < in.size(); ++i) out[i] = in[i];
}

int pcv_octree_node_data(const pcv_octree* o, uint64_t hi, uint64_t lo, void* xyz_out, uint8_t* rgb_out, float* intensity_out,
                         uint64_t* src_out) {
    if (!o) return fail(PCV_ERR_INVALID, "null octree");
    API_TRY
    int i = o->find(hi, lo);
    if (i < 0) return fail(PCV_ERR_NOT_FOUND, "node %s not found", node_name(hi, lo).c_str());
    const pcv_node_meta& m = o->nodes[i];
    pcv_ctx* c = o->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    const uint64_t n = (uint64_t)m.num_points;
    if (n == 0) return PCV_OK;
    const uint64_t bpc = (uint64_t)enc_bytes(m.position_encoding);
    if (xyz_out) CU(cudaMemcpyAsync(xyz_out, o->d_xyz + m.xyz_byte_offset, n * 3 * bpc, cudaMemcpyDeviceToHost, c->stream));
    if (rgb_out) CU(cudaMemcpyAsync(rgb_out, o->d_rgb + 3 * m.point_offset, n * 3, cudaMemcpyDeviceToHost, c->stream));
    if (intensity_out && o->d_intensity)
        CU(cudaMemcpyAsync(intensity_out, o->d_intensity + m.point_offset, n * 4, cudaMemcpyDeviceToHost, c->stream));
    std::vector<uint32_t> tmp;
    if (src_out) {
        tmp.resize(n);
        CU(cudaMemcpyAsync(tmp.data(), o->d_src + m.point_offset, n * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaStreamSynchronize(c->stream));
    if (src_out) widen_src(tmp, src_out);
    return PCV_OK;
    API_CATCH
}

int pcv_octree_download(const pcv_octree* o, void* xyz_out, uint8_t* rgb_out, float* intensity_out, uint64_t* src_out) {
    if (!o) return fail(PCV_ERR_INVALID, "null octree");
    API_TRY
    pcv_ctx* c = o->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    if (o->n == 0) return PCV_OK;
    if (xyz_out) CU(cudaMemcpyAsync(xyz_out, o->d_xyz, o->xyz_bytes, cudaMemcpyDeviceToHost, c->stream));
    if (rgb_out) CU(cudaMemcpyAsync(rgb_out, o->d_rgb, o->n * 3, cudaMemcpyDeviceToHost, c->stream));
    if (intensity_out && o->d_intensity) CU(cudaMemcpyAsync(intensity_out, o->d_intensity, o->n * 4, cudaMemcpyDeviceToHost, c->stream));
    std::vector<uint32_t> tmp;
    if (src_out) {
        tmp.resize(o->n);
        CU(cudaMemcpyAsync(tmp.data(), o->d_src, o->n * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaStreamSynchronize(c->stream));
    if (src_out) widen_src(tmp, src_out);
    return PCV_OK;
    API_CATCH
}

int pcv_octree_device_arrays(const pcv_octree* o, const void** xyz, const uint8_t** rgb, const float** intensity, const uint32_t** src) {
    if (!o) return fail(PCV_ERR_INVALID, "null octree");
    if (xyz) *xyz = o->d_xyz;
    if (rgb) *rgb = o->d_rgb;
    if (intensity) *intensity = o->d_intensity;
    if (src) *src = o->d_src;
    return PCV_OK;
}

}  // extern "C"

// Host copies of an octree's node-contiguous arrays (the caller holds the context's lock).
struct HostArrays {
    std::vector<uint8_t> xyz, rgb;
    std::vector<float> inten;
};
static void download_arrays(const pcv_octree* o, HostArrays& h) {
    pcv_ctx* c = o->ctx;
    h.xyz.resize(o->xyz_bytes);
    h.rgb.resize(o->n * 3);
    h.inten.resize(o->has_intensity ? o->n : 0);
    CU(cudaSetDevice(c->device));
    if (!o->n) return;
    CU(cudaMemcpyAsync(h.xyz.data(), o->d_xyz, o->xyz_bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaMemcpyAsync(h.rgb.data(), o->d_rgb, o->n * 3, cudaMemcpyDeviceToHost, c->stream));
    if (o->has_intensity) CU(cudaMemcpyAsync(h.inten.data(), o->d_intensity, o->n * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
}

// <dir>/<NodeId>.xyz|.rgb|.intensity of the nodes of `o` whose level is in [level_lo, level_hi), from the host copies.
static void write_node_files(const std::string& d, const pcv_octree* o, const HostArrays& h, int level_lo, int level_hi) {
    for (const auto& m : o->nodes) {
        if (m.num_points == 0 || m.level < level_lo || m.level >= level_hi) continue;  // node_writer.rs:78-89: empty files do not exist
        const std::string stem = d + "/" + node_name(m.id_high, m.id_low);
        const uint64_t n = (uint64_t)m.num_points, bpc = (uint64_t)enc_bytes(m.position_encoding);
        if (!write_whole_file(stem + ".xyz", h.xyz.data() + m.xyz_byte_offset, n * 3 * bpc) ||
            !write_whole_file(stem + ".rgb", h.rgb.data() + 3 * m.point_offset, n * 3) ||
            (o->has_intensity && !write_whole_file(stem + ".intensity", h.inten.data() + m.point_offset, n * 4)))
            throw BuildError(PCV_ERR_IO, "cannot write node files " + stem + ".*");
    }
}

// <dir>/meta.pb over `nodes` (sorted by NodeId)
static void write_meta(const std::string& d, double resolution, const double bmin[3], const double bmax[3], const std::vector<pcv_node_meta>& nodes) {
    MetaHeader h;
    h.resolution = resolution;
    for (int a = 0; a < 3; ++a) {
        h.bbox_min[a] = bmin[a];
        h.bbox_max[a] = bmax[a];
    }
    const std::string meta = encode_meta(h, nodes);
    if (!write_whole_file(d + "/meta.pb", meta.data(), meta.size())) throw BuildError(PCV_ERR_IO, "cannot write " + d + "/meta.pb");
}

extern "C" {

int pcv_octree_write_dir(const pcv_octree* o, const char* dir) {
    if (!o || !dir) return fail(PCV_ERR_INVALID, "null argument");
    API_TRY
    pcv_ctx* c = o->ctx;
    mkdir(dir, 0777);  // "Ignore errors, maybe directory is already there." generation.rs:306-307
    HostArrays h;
    {
        std::lock_guard<std::mutex> g(c->mu);
        download_arrays(o, h);
    }
    const std::string d(dir);
    write_node_files(d, o, h, 0, INT32_MAX);
    write_meta(d, o->resolution, o->bbox_min, o->bbox_max, o->nodes);
    return PCV_OK;
    API_CATCH
}

// pcv_octree_load_dir: dir_octree.inl

// ---- synthetic inputs ---------------------------------------------------------------------------
int pcv_synth_points_device(pcv_ctx* c, int kind, uint64_t seed, uint64_t first, uint64_t n, double* x, double* y, double* z, uint8_t* rgb) {
    if (!c || !x || !y || !z || !rgb) return fail(PCV_ERR_INVALID, "null argument");
    if (kind != PCV_SYNTH_SLAB_ECEF && kind != PCV_SYNTH_GAUSS_CLUSTERS) return fail(PCV_ERR_INVALID, "unknown synthetic kind %d", kind);
    API_TRY
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    if (n) {
        k_synth<<<c->sm_count * 8, 256, 0, c->stream>>>(kind, seed, first, n, x, y, z, rgb);
        c->be->launches++;
        CU(cudaGetLastError());
        CU(cudaStreamSynchronize(c->stream));
    }
    return PCV_OK;
    API_CATCH
}

int pcv_synth_points_host(int kind, uint64_t seed, uint64_t first, uint64_t n, double* x, double* y, double* z, uint8_t* rgb) {
    if (!x || !y || !z || !rgb) return fail(PCV_ERR_INVALID, "null argument");
    if (kind != PCV_SYNTH_SLAB_ECEF && kind != PCV_SYNTH_GAUSS_CLUSTERS) return fail(PCV_ERR_INVALID, "unknown synthetic kind %d", kind);
    for (uint64_t i = 0; i < n; ++i) {
        double p[3];
        uint8_t c[3];
        synth_point(kind, seed, first + i, p, c);
        x[i] = p[0];
        y[i] = p[1];
        z[i] = p[2];
        rgb[3 * i] = c[0];
        rgb[3 * i + 1] = c[1];
        rgb[3 * i + 2] = c[2];
    }
    return PCV_OK;
}

int pcv_synth_bbox(int kind, double bbox_min[3], double bbox_max[3], double* resolution) {
    if (!bbox_min || !bbox_max) return fail(PCV_ERR_INVALID, "null argument");
    if (kind != PCV_SYNTH_SLAB_ECEF && kind != PCV_SYNTH_GAUSS_CLUSTERS) return fail(PCV_ERR_INVALID, "unknown synthetic kind %d", kind);
    synth_bbox(kind, bbox_min, bbox_max, resolution);
    return PCV_OK;
}

}  // extern "C"

#include "query_api.inl"
#include "xray_api.inl"
#include "xray_merge.inl"
#include "xray_inpaint.inl"
#include "dir_octree.inl"
#include "xray_dir.inl"
#include "dir_query.inl"
#include "s2_api.inl"
#include "query_batch_points.inl"
#include "s2_xray.inl"
#include "s2_dir_xray.inl"
#include "s2_dir_query.inl"
#include "dir_query_batch_points.inl"
#include "ply_api.inl"
#include "shard_api.inl"
#include "sharded_build.inl"
#include "ooc_build.inl"
#include "s2_stream.inl"
