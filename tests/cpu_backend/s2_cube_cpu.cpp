// TEST-ONLY: sequential drivers of the cell-union node test of csrc/s2.h (s2_to_face_ij_level, s2_cube_relation), the PCV_HD
// functions the query kernels call.  NOT part of the shipped library.
#include <vector>

#include "../../point_cloud_viewer_b200/csrc/s2.h"

using namespace pcv;

extern "C" {
void tbc_to_face_ij_level(uint64_t id, int32_t* face_out, uint32_t* i0_out, uint32_t* j0_out, uint32_t* size_out) {
    const S2Square q = s2_to_face_ij_level(id);
    *face_out = q.face, *i0_out = q.i0, *j0_out = q.j0, *size_out = q.size;
}
// s2_cube_relation of every cube (m[3k .. 3k+2], e[k]) against the normalised union `cu`
void tbc_cube_relation(const uint64_t* cu, uint32_t ncu, const double* m3, const double* e, uint64_t ncubes, int32_t* rel_out) {
    std::vector<S2Square> sq(ncu);
    for (uint32_t k = 0; k < ncu; ++k) sq[k] = s2_to_face_ij_level(cu[k]);
    for (uint64_t k = 0; k < ncubes; ++k) rel_out[k] = s2_cube_relation(m3 + 3 * k, e[k], sq.data(), ncu);
}
}
