// TEST-ONLY: the host side of the streamed S2 split (csrc/s2_dir_writer.hpp, csrc/s2_stream_plan.h) behind a C interface, so
// that the CPU tests drive them with ctypes.  NOT part of the shipped library.
#include <cstring>
#include <string>

#include "../../point_cloud_viewer_b200/csrc/s2_dir_writer.hpp"
#include "../../point_cloud_viewer_b200/csrc/s2_stream_plan.h"

using namespace pcv;

extern "C" {
void* sdw_new(const char* dir, int threads, int rgb, int intensity) { return new S2DirWriter(dir, threads, rgb != 0, intensity != 0); }
void sdw_free(void* w) { delete (S2DirWriter*)w; }
int sdw_begin(void* w) { return ((S2DirWriter*)w)->begin() ? 0 : 1; }
int sdw_submit(void* w, uint64_t seq, const uint8_t* xyz, const uint8_t* rgb, const uint8_t* intensity, const uint64_t* ids, const uint64_t* counts,
               uint64_t ncells) {
    const uint8_t* data[3] = {xyz, rgb, intensity};
    return ((S2DirWriter*)w)->submit(seq, data, ids, counts, (size_t)ncells) ? 0 : 1;
}
void sdw_wait(void* w, uint64_t seq) { ((S2DirWriter*)w)->wait(seq); }
int sdw_finish(void* w, const double* bmin, const double* bmax) { return ((S2DirWriter*)w)->finish(bmin, bmax) ? 0 : 1; }
void sdw_error(void* w, char* out, int cap) { snprintf(out, (size_t)cap, "%s", ((S2DirWriter*)w)->error().c_str()); }
void sdw_stats(void* w, uint64_t* out) {
    S2DirWriter* s = (S2DirWriter*)w;
    out[0] = s->bytes_written;
    out[1] = s->file_writes;
    out[2] = s->num_cells();
}

// plan_s2_stream: in = {budget, free, n, attr_bytes, sort_per_point, sort_fixed, chunk, granule, src_chunk_bytes};
// out = {budget, batch, chunk, per_point, fixed, planned}; returns 1 and the message on the budget error
int sdw_plan(const uint64_t* in, uint64_t* out, char* err, int cap) {
    S2StreamPlanIn i;
    i.budget = in[0], i.free_bytes = in[1], i.n = in[2], i.attr_bytes = in[3], i.sort_per_point = in[4], i.sort_fixed = in[5];
    i.chunk = in[6], i.granule = in[7], i.src_chunk_bytes = in[8];
    const S2StreamPlan p = plan_s2_stream(i);
    out[0] = p.budget, out[1] = p.batch, out[2] = p.chunk, out[3] = p.per_point, out[4] = p.fixed, out[5] = p.planned;
    snprintf(err, (size_t)cap, "%s", p.error.c_str());
    return p.error.empty() ? 0 : 1;
}
}
