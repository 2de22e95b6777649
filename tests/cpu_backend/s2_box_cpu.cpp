// TEST-ONLY: sequential driver of the cell test of the S2 cloud's location queries (csrc/geometry_host.hpp: project_location_axis,
// sat_box), the PCV_HD functions k_s2_select_cells calls.  NOT part of the shipped library.
#include "../../point_cloud_viewer_b200/csrc/geometry_host.hpp"

using namespace pcv;

extern "C" {
// sat_box of the location against every box [mn[3k .. 3k+2], mx[3k .. 3k+2]]: 0 In, 1 Cross, 2 Out
void tbb_sat_box(const pcv_location* loc, const double* mn, const double* mx, uint64_t nboxes, int32_t* rel_out) {
    const QueryGeom g = make_query_geom(*loc);
    double aproj[26][2];
    for (int k = 0; k < g.naxes; ++k) project_location_axis(g, k, aproj[k][0], aproj[k][1]);
    for (uint64_t k = 0; k < nboxes; ++k) rel_out[k] = sat_box(g, aproj, mn + 3 * k, mx + 3 * k);
}
}
