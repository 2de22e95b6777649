/*
 * pcv.h — C ABI of the H100-native octree builder / LOD + frustum point-query engine.
 *
 * This is the drop-in boundary for point_cloud_viewer's hot path: each entry point replaces a Rust
 * function or trait method of crate `point_viewer` (citations = reference file:line).  The reference
 * has no FFI of its own; INTEGRATION.md shows the Rust `extern "C"` block + shim a maintainer adds.
 *
 * Conventions
 *  - plain pointers and sizes only; every function returns 0 (PCV_OK) or a negative pcv_status and
 *    never unwinds across the boundary; pcv_last_error() returns the text for the calling thread.
 *  - "host" entry points take host memory (pinned or pageable) and copy inside the call; "_device"
 *    entry points take device pointers already resident in HBM on the context's GPU.
 *  - positions are f64; element i of a coordinate array is at ptr[i * stride] so both the SoA layout
 *    (stride 1, three arrays) and the crate's AoS `Vec<Point3<f64>>` (stride 3, y = x+1, z = x+2) are
 *    accepted without a host-side transpose.
 *  - matrices are column-major like nalgebra::Matrix4<f64>; isometries are tx,ty,tz,qi,qj,qk,qw.
 *  - NodeId is the crate's u128 (level << 120 | octal path index, src/octree/node.rs:52-111) passed
 *    as (high, low) u64 halves exactly like proto::NodeId (node.rs:101-106).
 *  - there is no CPU fallback: without a CUDA device every compute entry point fails with
 *    PCV_ERR_CUDA.
 */
#ifndef PCV_H
#define PCV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pcv_ctx pcv_ctx;       /* one per device; internally stream ordered              */
typedef struct pcv_octree pcv_octree; /* a built / loaded octree, node data resident in HBM     */

typedef enum pcv_status {
    PCV_OK = 0,
    PCV_ERR_INVALID = -1,     /* bad argument                                                    */
    PCV_ERR_CUDA = -2,        /* CUDA runtime error or no device                                 */
    PCV_ERR_IO = -3,          /* file system error (the reference unwrap()s these)               */
    PCV_ERR_NOT_FOUND = -4,   /* ErrorKind::NodeNotFound (src/errors.rs)                         */
    PCV_ERR_CANCELLED = -5,   /* callback returned non-zero == ErrorKind::Channel                */
    PCV_ERR_UNSUPPORTED = -6, /* e.g. more than 2^32-1 points per context, depth > 40            */
    PCV_ERR_SINGULAR = -7     /* get_visible_nodes: "Invalid projection matrix." (mod.rs:230)    */
} pcv_status;

/* PositionEncoding (src/read_write/codec.rs:22-28, proto.proto:78-84) */
enum { PCV_ENC_UINT8 = 1, PCV_ENC_UINT16 = 2, PCV_ENC_FLOAT32 = 3, PCV_ENC_FLOAT64 = 4 };

typedef struct pcv_config {
    uint64_t max_points_per_node; /* MAX_POINTS_PER_NODE, generation.rs:37; 0 -> 100000          */
    uint32_t levels_per_pass;     /* kept for ABI stability: the split phase resolves 2 levels/pass */
    uint32_t reserved;
} pcv_config;

typedef struct pcv_points {
    const double* x; /* element i at x[i*stride]                                                 */
    const double* y;
    const double* z;
    uint64_t stride;        /* 1 = SoA, 3 = AoS xyz                                              */
    const uint8_t* rgb;     /* n * 3, "color" U8Vec3 (mandatory: on_disk.rs:23-33)               */
    const float* intensity; /* n or NULL ("intensity" F32, octree/mod.rs:62-74)                  */
    uint64_t n;
} pcv_points;

typedef struct pcv_node_meta {
    uint64_t id_high, id_low; /* NodeId u128 halves                                              */
    int64_t num_points;       /* may be 0: such nodes stay in meta.pb (generation.rs:241-243)    */
    int32_t position_encoding;
    int32_t level;
    double cube_min[3]; /* NodeId::find_bounding_cube (node.rs:157-172)                          */
    double cube_edge;
    uint64_t point_offset;    /* first point of the node in the node-contiguous arrays           */
    uint64_t xyz_byte_offset; /* first byte of the node's .xyz content                           */
} pcv_node_meta;

/* PointLocation (src/iterator.rs:13-20).  Same field layout as the oracle's orc_location.
 * PCV_LOC_WEB_MERCATOR_RECT (web_mercator_rect.rs) keeps north_west in aabb_min[0..1] and south_east in aabb_max[0..1], both
 * normalised to [0, 1) as pcv_web_mercator_rect leaves them; every other field is zero.  A kind-4 location the constructor
 * could not have made (non-finite or outside [0, 1), north_west.y > south_east.y, or more than one zoom-0 pixel across) is
 * PCV_ERR_INVALID for every query. */
enum { PCV_LOC_ALL = 0, PCV_LOC_AABB = 1, PCV_LOC_FRUSTUM = 2, PCV_LOC_OBB = 3, PCV_LOC_WEB_MERCATOR_RECT = 4 };
typedef struct pcv_location {
    int32_t kind;
    int32_t pad;
    double aabb_min[3], aabb_max[3];                 /* Aabb{mins,maxs}        aabb.rs:12-16     */
    double clip_from_query[16], query_from_clip[16]; /* Frustum fields         frustum.rs:95-98  */
    double query_from_obb[7], obb_from_query[7];     /* Obb fields             obb.rs:13-17      */
    double half_extent[3];
} pcv_location;

typedef struct pcv_interval { /* ClosedInterval<f64> on "intensity" (math/mod.rs:65-89)          */
    double lo, hi;
} pcv_interval;

/* A PointsBatch (src/lib.rs:102-107) delivered to the consumer: AoS positions + SoA attributes.  */
typedef struct pcv_batch {
    uint64_t n;
    const double* xyz;         /* n * 3                                                          */
    const uint8_t* rgb;        /* n * 3                                                          */
    const float* intensity;    /* n or NULL                                                      */
    const uint64_t* src_index; /* provenance: index of the point in the build input              */
} pcv_batch;
typedef int (*pcv_batch_cb)(void* user, const pcv_batch* batch); /* non-zero return cancels      */

/* ---- context ------------------------------------------------------------------------------- */
int pcv_create(int device, const pcv_config* cfg, pcv_ctx** out);
void pcv_destroy(pcv_ctx* ctx);
const char* pcv_last_error(void);
int pcv_device_count(void);

/* ---- a1: find_bounding_box (generation.rs:256-270, aabb.rs:41-44) -------------------------- */
int pcv_bbox(pcv_ctx* ctx, const pcv_points* host_points, double out_min[3], double out_max[3]);
int pcv_bbox_device(pcv_ctx* ctx, const pcv_points* dev_points, double out_min[3], double out_max[3]);

/* ---- a2-a8: build_octree (generation.rs:289-403) -------------------------------------------- */
int pcv_build_octree(pcv_ctx* ctx, const pcv_points* host_points, double resolution, const double bbox_min[3],
                     const double bbox_max[3], pcv_octree** out);
int pcv_build_octree_device(pcv_ctx* ctx, const pcv_points* dev_points, double resolution, const double bbox_min[3],
                            const double bbox_max[3], pcv_octree** out);
void pcv_octree_free(pcv_octree* o);

/* ---- a8-a10: node table, node bytes, on-disk layout ----------------------------------------- */
int pcv_octree_info(const pcv_octree* o, uint64_t* num_nodes, uint64_t* num_points, uint64_t* xyz_bytes, double* resolution,
                    double bbox_min[3], double bbox_max[3], int* has_intensity);
int pcv_octree_nodes(const pcv_octree* o, pcv_node_meta* out, uint64_t cap); /* sorted by NodeId   */
/* Octree::get_node_data (octree/mod.rs:285-307): raw .xyz / .rgb bytes (+ intensity, provenance). */
int pcv_octree_node_data(const pcv_octree* o, uint64_t id_high, uint64_t id_low, void* xyz_out, uint8_t* rgb_out,
                         float* intensity_out, uint64_t* src_index_out);
/* The web viewer's `/nodes_data` reply (octree_web_viewer/src/backend.rs:66-75, 92-165): for every requested node, in
 * request order: cube min (3 f64 LE), edge (f64), num_points (u32), bytes per coordinate (u8), zero padding to 8 bytes,
 * position bytes, padding, colour bytes, padding.  ids_hi_lo = num_nodes x (high, low).  out == NULL: size query.
 * An unknown id or a node without points is PCV_ERR_NOT_FOUND (get_node_data -> NodeNotFound: no files). */
int pcv_nodes_data_blob(const pcv_octree* o, const uint64_t* ids_hi_lo, uint32_t num_nodes, void* out, uint64_t cap, uint64_t* size_out);
/* LOD draw order (sdl_viewer/src/node_drawer.rs:34-43,185-205: the viewer shuffles every node it loads so that "the first N"
 * points are a uniform subsample; octree/mod.rs:286-287 asks for that order to be applied when the node is written).
 * pcv_octree_shuffle_nodes permutes positions, colours, intensity and provenance of every node in place (on the GPU) with the
 * keyed permutation pcv_lod_order(seed, node id, n) returns on the host: shuffled[i] = original[new_order[i]] (`reshuffle`). */
int pcv_octree_shuffle_nodes(pcv_octree* o, uint64_t seed);
int pcv_lod_order(uint64_t seed, uint64_t id_high, uint64_t id_low, uint64_t n, uint64_t* new_order_out);
/* All nodes at once into caller (ideally pinned) buffers: node n occupies points [point_offset, +num_points) and
 * bytes [xyz_byte_offset, +num_points*3*bpc) of these arrays (offsets from pcv_octree_nodes; no particular order). */
int pcv_octree_download(const pcv_octree* o, void* xyz_out, uint8_t* rgb_out, float* intensity_out, uint64_t* src_index_out);
/* Device views of the same arrays (valid until pcv_octree_free). */
int pcv_octree_device_arrays(const pcv_octree* o, const void** xyz, const uint8_t** rgb, const float** intensity,
                             const uint32_t** src_index);
/* <dir>/<NodeId>.xyz|.rgb|.intensity + meta.pb (on_disk.rs:17-33, lib.rs:49,74-80, proto.proto:68-149). */
int pcv_octree_write_dir(const pcv_octree* o, const char* dir);
int pcv_octree_load_dir(pcv_ctx* ctx, const char* dir, pcv_octree** out); /* Octree::from_data_provider, mod.rs:156-215 */

/* ---- a11-a14: nodes_in_location (octree/mod.rs:309-323, octree_iterator.rs:30-43) ---------- */
int pcv_nodes_in_location(const pcv_octree* o, const pcv_location* loc, uint64_t* ids_hi_lo, uint64_t cap, uint64_t* n_out);

/* ---- PointLocation::WebMercatorRect (src/geometry/web_mercator_rect.rs), host only ------------------------------------------
 * pcv_web_mercator_rect: WebMercatorRect::from_zoomed_coordinates(min, max, z) as a kind-4 location.  PCV_ERR_INVALID where the
 * reference returns None (z > 23, a corner component < 0 or >= 256 * 2^z, (max - min) / 2^z with x rem_euclid 256 > 1, y > 1
 * or y < 0) and for non-finite input.  x may wrap around the antimeridian (min.x > max.x); such a rect selects nodes but
 * contains no point.
 * pcv_web_mercator_coord: the map position of an ECEF point at zoom z, in [0, 256 * 2^z)^2 (x east, y south):
 * WebMercatorCoord::from_lat_lng(ECEF -> WGS84).to_zoomed_coordinate(z), with the arithmetic of the cull kernels' point test.
 * PCV_ERR_INVALID for z > 23. */
int pcv_web_mercator_rect(const double min[2], const double max[2], uint32_t z, pcv_location* out);
int pcv_web_mercator_coord(const double ecef[3], uint32_t z, double out[2]);

/* ---- a17: Octree::get_visible_nodes (octree/mod.rs:228-283) --------------------------------- */
int pcv_visible_nodes(const pcv_octree* o, const double clip_from_world[16], uint64_t* ids_hi_lo, uint64_t cap, uint64_t* n_out);

/* ---- a15-a16: PointQuery streaming (iterator.rs:66-119,255-333) ----------------------------- */
/* Streams every point of every node in `loc` that passes the culling + interval filters, re-chunked
 * into batches of exactly batch_size points (last one short), on the caller's thread.
 * The argument contract holds for all three sources (octree, octree directory, S2 cloud) and their nodes / cells, stream and
 * batch calls: a location kind outside PCV_LOC_ALL..PCV_LOC_WEB_MERCATOR_RECT, an invalid kind-4 rect, nfilt > 0 with
 * filters == NULL, or filters over points without intensity is PCV_ERR_INVALID; a callback that returns non-zero ends the
 * stream with PCV_ERR_CANCELLED. */
int pcv_query_points(const pcv_octree* o, const pcv_location* loc, const pcv_interval* filters, uint32_t nfilt,
                     uint64_t batch_size, pcv_batch_cb cb, void* user);
/* Throughput form: nloc locations in one call; survivors stay compacted in HBM.  counts_out[i] =
 * survivors of location i, tested_out[i] = points decoded + tested for location i. */
int pcv_query_batch_device(const pcv_octree* o, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters,
                           uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);

/* ---- PointLocation::S2Cells: queries by S2 cell union (src/geometry/s2_cell_union.rs) ------ */
/* A point passes iff the union contains the leaf cell of its decoded position (CellUnion::contains(CellID::from_point(p))).
 * The ids are validated and normalised (CellUnion::normalize); an invalid id, or n > 0 with ids == NULL, is PCV_ERR_INVALID.
 * An empty union selects no node and returns no point.  The points equal every point of the octree that passes the test, in
 * the order the AllPoints stream delivers them.  The node list holds every node with a passing point, in BFS order; it is not
 * the reference's list (which pre-selects with latitude / longitude rectangles): it may hold nodes without one. */
typedef struct pcv_cell_union {
    const uint64_t* ids;
    uint32_t n;
    uint32_t pad;
} pcv_cell_union;
int pcv_nodes_in_cell_union(const pcv_octree* o, const pcv_cell_union* cu, uint64_t* ids_hi_lo, uint64_t cap, uint64_t* n_out);
int pcv_query_cell_union(const pcv_octree* o, const pcv_cell_union* cu, const pcv_interval* filters, uint32_t nfilt,
                         uint64_t batch_size, pcv_batch_cb cb, void* user);
/* pcv_query_batch_device over nunion cell unions; fills pcv_last_query_stats the same way. */
int pcv_query_cell_unions_batch_device(const pcv_octree* o, const pcv_cell_union* unions, uint32_t nunion, const pcv_interval* filters,
                                       uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);

/* Batched queries that return their points.  For locations L0..Ln-1 the call fills the host offsets offsets_out[0..n] and writes,
 * for every i, the points pcv_query_points(Li) (pcv_query_cell_union for a union) streams, in the same order and bit for bit in
 * every field, to [offsets_out[i], offsets_out[i+1]) of the device arrays d_xyz (3 f64 per point), d_rgb (3 u8), d_intensity
 * (f32) and d_src (u64, the build input index).  offsets_out[i+1] - offsets_out[i] is pcv_query_batch_device's counts_out[i]; a
 * location's segment does not depend on the other locations of the call.
 * d_xyz == NULL is a size query: offsets_out is filled and nothing is written.  d_rgb, d_intensity and d_src may each be NULL to
 * skip the field; a non-null d_intensity on points without intensity (or a non-null d_rgb on an S2 cloud without colour) is
 * PCV_ERR_INVALID.  cap < offsets_out[n] is PCV_ERR_INVALID with offsets_out complete (the device arrays are then unspecified).
 * The argument contract of pcv_query_points holds; a selection too large for one call is PCV_ERR_UNSUPPORTED ("split the
 * batch").  pcv_last_query_stats: returned_points = offsets_out[n], stored_points = the points written, tested_points as
 * pcv_query_batch_device; ms_select covers selection and ordering, ms_cull the count, scan and place passes. */
int pcv_query_batch_points_device(const pcv_octree* o, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters, uint32_t nfilt,
                                  uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb, float* d_intensity, uint64_t* d_src, uint64_t cap);
int pcv_query_cell_unions_batch_points_device(const pcv_octree* o, const pcv_cell_union* unions, uint32_t nunion, const pcv_interval* filters,
                                              uint32_t nfilt, uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb, float* d_intensity,
                                              uint64_t* d_src, uint64_t cap);

/* Timing / traffic of the last pcv_query_batch_device call on the context (CUDA events on the context's stream). */
typedef struct pcv_query_stats {
    float ms_device;            /* first kernel to last kernel of the call                                   */
    float ms_select;            /* node selection: per-level frontier kernels + work-list build              */
    float ms_cull;              /* the culling kernel                                                        */
    uint32_t kernel_launches;
    uint64_t algorithmic_bytes; /* SURVEY 8(d) B_query: sum over visited (location, node) of n (3 bpc + 3) + 27 per survivor */
    uint64_t tested_points, returned_points, stored_points; /* stored <= returned: survivors beyond the output capacity are only counted */
    uint64_t visited_pairs;     /* (location, node) pairs with points that were culled                       */
} pcv_query_stats;
int pcv_last_query_stats(pcv_ctx* ctx, pcv_query_stats* out);

/* ---- a19: X-ray leaf tile (xray/src/generation.rs:108-127,159-198,464-513) ------------------ */
/* query_from_global: 7 doubles or NULL.  rgba_out: w*h*4.  Returns any_points_out=0 for an empty tile
 * (the reference returns None). zbits_out (optional): w*h*32 u32 z-bucket bitsets. */
int pcv_xray_tile(const pcv_octree* o, const double tile_min[3], const double tile_max[3], uint32_t w, uint32_t h,
                  const double* query_from_global, uint8_t* rgba_out, uint32_t* zbits_out, int* any_points_out);
/* Timing / traffic of the last pcv_xray_tile[_attr] call on the context. */
typedef struct pcv_xray_stats {
    float ms_device;            /* CUDA events around the call's kernels                                    */
    uint32_t kernel_launches;
    uint64_t points;            /* points of the nodes the tile intersects (decoded + tested)               */
    uint64_t algorithmic_bytes; /* SURVEY 8(d) B_xray: sum over nodes of n (3 bpc + 3) + 4 W H               */
} pcv_xray_stats;
int pcv_last_xray_stats(pcv_ctx* ctx, pcv_xray_stats* out);
/* The other ColoringStrategyKinds (xray/src/generation.rs:76-97): point colour mean (:294-363), intensity mean brightened
 * by ln(mean - min) / ln(max - min) (:210-290; p0 = min, p1 = max), height standard deviation through the Jet (0) or
 * Purplish (1) colormap (:365-405, xray/src/colormap.rs; p0 = max_stddev).  Binning = None.  The reference accumulates in
 * arrival order from several threads, so results are defined up to rounding: expect +-1 per channel. */
enum { PCV_XRAY_COLORED = 1, PCV_XRAY_INTENSITY = 2, PCV_XRAY_HEIGHT_STDDEV = 3 };
int pcv_xray_tile_attr(const pcv_octree* o, const double tile_min[3], const double tile_max[3], uint32_t w, uint32_t h,
                       const double* query_from_global /* 7 or NULL */, int strategy, float p0, float p1, int colormap, uint8_t* rgba_out,
                       int* any_out);

/* Pixels no point falls into are TRANSPARENT.to_u8() = (255, 255, 255, 0) in every tile (src/color.rs:154-159,
 * xray/src/generation.rs:506-511). */

/* ---- f3: the rest of the X-ray pipeline (xray/src/generation.rs:129-157, 410-451, 515-759) ---- */
/* Colored / ColoredWithIntensity with Binning = Some(("intensity", bin_size)) (:66-67, :129-157): per pixel and bin
 * (bin = (intensity as f64 / bin_size) as i64) the mean colour / intensity, per pixel the mean of its bins' means
 * (:276-290, :339-346).  Needs an octree with intensities ("Binning attribute needs to be available").  The reference sums
 * in arrival / hash-map order: results are defined up to f32 rounding (+-1 per channel). */
int pcv_xray_tile_attr_binned(const pcv_octree* o, const double tile_min[3], const double tile_max[3], uint32_t w, uint32_t h,
                              const double* query_from_global /* 7 or NULL */, int strategy /* PCV_XRAY_COLORED | PCV_XRAY_INTENSITY */,
                              float p0, float p1, double bin_size, uint8_t* rgba_out, int* any_out);
/* assign_background (:695-720): every pixel with alpha < 128 becomes `background` (RGBA), in place (host buffer). */
int pcv_xray_assign_background(pcv_ctx* ctx, uint8_t* rgba, uint64_t num_pixels, const uint8_t background[4]);
/* build_node (:722-759) for one parent: build_parent's 2 x 2 mosaic of the four child images (:410-451; children[i] =
 * child_px x child_px RGBA of quadtree child i or NULL -> background; child 1 top left, 0 bottom left, 3 top right, 2 bottom
 * right) reduced to tile_px x tile_px with image 0.23's `imageops::resize(.., FilterType::Lanczos3)` (vertical pass into
 * u8, then horizontal pass; f32 weights; round-to-nearest conversion - restated, the crate is not vendored).  Host buffers. */
int pcv_xray_build_parent(pcv_ctx* ctx, const uint8_t* const children[4], uint32_t child_px, const uint8_t background[4],
                          uint32_t tile_px, uint8_t* rgba_out /* tile_px * tile_px * 4 */);
/* build_xray_quadtree (:560-622) as one call: bounding rect and levels (:515-533), every leaf tile at the deepest level
 * (:535-551, :624-667) with the chosen strategy, assign_background on the created leaves, and the parents (:669-693).  A leaf
 * exists iff at least one point passes its location test (:489-504).  Each finished tile is handed to `on_tile` (host
 * pointer, valid during the call; return non-zero to cancel -> PCV_ERR_CANCELLED; must not call into the same context) in
 * post-order: every tile after all of its children, siblings in index order, the root last.  What the reference writes as
 * <id>.png and meta.pb is what on_tile receives plus `info`; PNG encoding stays on the host.  pcv_xray_quadtree is
 * pcv_xray_quadtree_bounded with max_device_bytes = 0. */
typedef struct pcv_xray_quadtree_params {
    int32_t strategy;             /* 0 = XRay, or PCV_XRAY_COLORED / _INTENSITY / _HEIGHT_STDDEV                 */
    float p0, p1;                 /* as in pcv_xray_tile_attr                                                     */
    int32_t colormap;
    double bin_size;              /* 0: Binning = None                                                            */
    int32_t has_query_from_global;
    double query_from_global[7];  /* tx,ty,tz, qi,qj,qk,qw                                                        */
    uint8_t background[4];        /* tile_background_color: WHITE (255,255,255,255) or TRANSPARENT (255,255,255,0) */
    uint32_t tile_size_px;
    double pixel_size_m;
    uint8_t root_level;           /* root_node_id (quadtree/src/lib.rs:143-150); NodeId::root() = (0, 0)          */
    uint64_t root_index;
} pcv_xray_quadtree_params;
typedef struct pcv_xray_quadtree_info {
    double rect_min_x, rect_min_y, rect_edge; /* Meta::bounding_rect = the (sub-)root node's rect                 */
    uint8_t deepest_level;                    /* Meta::deepest_level                                              */
    uint32_t tile_size_px;                    /* Meta::tile_size                                                  */
    uint32_t num_nodes, num_leaves;           /* Meta::nodes = the ids on_tile received                           */
    float ms_leaves, ms_parents;              /* CUDA events: leaf tiles + background; parent kernels             */
    uint32_t kernel_launches;
    uint64_t leaf_points;                     /* XRay strategy: points decoded for the leaf tiles                 */
} pcv_xray_quadtree_info;
typedef int (*pcv_xray_tile_fn)(void* user, uint8_t level, uint64_t index, const uint8_t* rgba, uint32_t tile_size_px);
int pcv_xray_quadtree(const pcv_octree* o, const pcv_xray_quadtree_params* params, pcv_xray_tile_fn on_tile, void* user,
                      pcv_xray_quadtree_info* info_out);

/* ... with the reference's outputs: <directory>/<node id>.png for every tile ("r", "r0", "r123323": quadtree/src/lib.rs:216-233;
 * 8-bit RGBA, deflated on the host with zlib) and the quadtree's meta file (xray Meta, version 3: bounding_rect, deepest_level,
 * tile_size, nodes; "meta.pb" for the root, "meta<digits>.pb" for a sub-root: xray/src/utils.rs:7-11, lib.rs:88-139). */
int pcv_xray_quadtree_write_dir(const pcv_octree* o, const pcv_xray_quadtree_params* params, const char* directory,
                                pcv_xray_quadtree_info* info_out);

/* The same quadtree of any size in bounded device memory.  Leaves are made in blocks: the subtree of one quadtree node `block
 * level` levels down from the root, all its leaves located with one batched node selection and binned by one kernel per key
 * batch.  Above the block level at most four finished children per level wait for their parent.  Only quadtree nodes that a
 * point of the octree falls into (with a margin) are enumerated, level by level from the root.  max_device_bytes bounds what
 * the driver allocates besides the resident octree (0: most of the free device memory); a budget that cannot hold one leaf,
 * or a leaf whose possible keys or working memory do not fit what the budget leaves, returns PCV_ERR_UNSUPPORTED.  A block
 * holds at most 1 GiB of images, staged in as much page-locked host memory for delivery; the context's allocator cache is
 * emptied after every block.  bounded_info_out may be NULL. */
typedef struct pcv_xray_bounded_info {
    uint64_t max_device_bytes;    /* the budget used                                                              */
    uint64_t peak_device_bytes;   /* the most the driver held at once (the resident octree not counted)           */
    uint64_t blocks_processed;    /* blocks at the block level whose subtree was visited                          */
    uint64_t blocks_pruned;       /* block positions below the root never visited                                 */
    uint64_t positions_evaluated; /* leaf positions tested with their exact location                              */
    uint64_t key_batches;         /* XRay strategy: binning passes over a batch of leaves                         */
    uint32_t block_level;         /* quadtree level of the block roots                                            */
} pcv_xray_bounded_info;
int pcv_xray_quadtree_bounded(const pcv_octree* o, const pcv_xray_quadtree_params* params, uint64_t max_device_bytes, pcv_xray_tile_fn on_tile,
                              void* user, pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out);
/* ... written as pcv_xray_quadtree_write_dir writes it; the PNGs are encoded and written by a small pool of host threads
 * behind a bounded queue while the device builds the next block. */
int pcv_xray_quadtree_bounded_write_dir(const pcv_octree* o, const pcv_xray_quadtree_params* params, uint64_t max_device_bytes, const char* directory,
                                        pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out);

/* The same quadtree straight from an octree directory (meta.pb + node files, as pcv_octree_write_dir and
 * pcv_build_octree_to_dir leave it), which is never resident as a whole: the same tiles, post-order, cancellation and outputs as
 * pcv_xray_quadtree_bounded over pcv_octree_load_dir of the directory.  One streaming pass over every node's positions marks
 * the leaves a point falls into (with the driver's margin); then each block of leaves runs on its window, the nodes the block's
 * location (widened by the margin) can meet, read from disk.  Nodes the previous window holds are copied on the device when the
 * budget has room for both.  Here max_device_bytes bounds everything the call allocates, the windows included (0: most of the
 * free device memory).  Host memory holds the largest window, the occupied leaves and the driver's staging.  Errors: a meta.pb
 * other than version 13 -> PCV_ERR_INVALID; a missing or wrongly sized .xyz / .rgb file -> PCV_ERR_NOT_FOUND; a leaf whose window
 * alone does not fit the budget or holds 2^32 points or more -> PCV_ERR_UNSUPPORTED.  bounded_info_out and dir_info_out may be NULL. */
typedef struct pcv_xray_dir_info {
    uint64_t windows_loaded;        /* blocks whose window was loaded                                               */
    uint64_t node_files_read;       /* .xyz / .rgb / .intensity files read, the occupancy pass included             */
    uint64_t bytes_read;            /* bytes read from those files                                                  */
    uint64_t nodes_reread;          /* window nodes read again from disk after an earlier window had loaded them    */
    uint64_t nodes_reused;          /* window nodes copied on the device from the previous window                   */
    uint64_t bytes_reused;          /* bytes of those copies                                                        */
    uint64_t bytes_uploaded;        /* host -> device bytes of node data (occupancy pass and windows)               */
    uint64_t largest_window_bytes;  /* device bytes of the largest window (arrays and query tables)                 */
    uint64_t largest_window_points;
    uint64_t occupied_leaves;       /* leaves the occupancy pass marked                                             */
    double ms_occupancy;            /* wall time of the occupancy pass                                              */
    double ms_windows;              /* wall time of window planning and loading (reads, uploads, query tables)      */
} pcv_xray_dir_info;
int pcv_xray_quadtree_from_dir(pcv_ctx* ctx, const char* octree_dir, const pcv_xray_quadtree_params* params, uint64_t max_device_bytes,
                               pcv_xray_tile_fn on_tile, void* user, pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out,
                               pcv_xray_dir_info* dir_info_out);
/* ... written as pcv_xray_quadtree_bounded_write_dir writes it. */
int pcv_xray_quadtree_from_dir_write_dir(pcv_ctx* ctx, const char* octree_dir, const pcv_xray_quadtree_params* params, uint64_t max_device_bytes,
                                         const char* out_dir, pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out,
                                         pcv_xray_dir_info* dir_info_out);

/* ... with filter intervals on the intensity (closed, the attribute as f64): a leaf is made only of the points of its location
 * that pass every interval, and a leaf whose location holds only points that fail does not exist.  The occupancy pass ignores
 * the filters.  Filters on a directory without intensities -> PCV_ERR_INVALID; with a binned strategy -> PCV_ERR_UNSUPPORTED.
 * nfilt = 0 is pcv_xray_quadtree_from_dir. */
int pcv_xray_quadtree_from_dir_filtered(pcv_ctx* ctx, const char* octree_dir, const pcv_xray_quadtree_params* params, const pcv_interval* filters,
                                        uint32_t nfilt, uint64_t max_device_bytes, pcv_xray_tile_fn on_tile, void* user, pcv_xray_quadtree_info* info_out,
                                        pcv_xray_bounded_info* bounded_info_out, pcv_xray_dir_info* dir_info_out);
int pcv_xray_quadtree_from_dir_filtered_write_dir(pcv_ctx* ctx, const char* octree_dir, const pcv_xray_quadtree_params* params, const pcv_interval* filters,
                                                  uint32_t nfilt, uint64_t max_device_bytes, const char* out_dir, pcv_xray_quadtree_info* info_out,
                                                  pcv_xray_bounded_info* bounded_info_out, pcv_xray_dir_info* dir_info_out);

/* The X-ray quadtree straight from one or more octree directories (build_xray_quadtree over a list of octree locations), none of
 * them ever resident as a whole: the same tiles, node set, rect, levels, cancellation and <id>.png + meta<...>.pb outputs as
 * pcv_xray_quadtree_clouds over pcv_octree_load_dir of every directory, in the same order.  The quadtree lies over the union of
 * the directories' meta.pb boxes.  XRay tiles are byte for byte the same at every budget and in any order of the directories;
 * the attribute strategies accumulate as the resident path does.  ndirs = 1 is pcv_xray_quadtree_from_dir_filtered in every
 * tile, delivery and counter.  One streaming pass over every node's positions of every directory marks the leaves a point falls
 * into; then each block of leaves runs on one window per directory (each as pcv_xray_quadtree_from_dir selects it), all of a
 * block's windows on the device together.  The block depth is chosen so that the largest block's windows together fit; nodes the
 * previous block's window of the same directory holds are copied on the device when the budget holds both blocks' windows.
 * There is no limit on the total, which may exceed device memory and 2^32 points.  max_device_bytes bounds everything the call
 * allocates, the windows included (0: most of the free device memory).  pcv_xray_dir_info's counters are summed over the
 * directories; its largest window is the largest block's windows together.  Errors: ndirs == 0 or a null path ->
 * PCV_ERR_INVALID; an unreadable meta.pb -> PCV_ERR_IO; a meta.pb other than version 13 -> PCV_ERR_INVALID; a missing or wrongly
 * sized .xyz / .rgb file -> PCV_ERR_NOT_FOUND, found by stat for every directory before the first read (no tile is delivered);
 * then the checks of pcv_xray_quadtree_clouds in its order: filters, or an intensity strategy, and a directory without
 * intensities -> PCV_ERR_INVALID; a binned strategy over more than one directory, or with filters -> PCV_ERR_UNSUPPORTED; a
 * budget too small for the occupancy pass, a leaf whose windows together do not fit besides one leaf tile (named), a leaf whose
 * window in one directory holds 2^32 points or more (leaf and directory named) -> PCV_ERR_UNSUPPORTED.  bounded_info_out and
 * dir_info_out may be NULL. */
int pcv_xray_quadtree_from_dirs(pcv_ctx* ctx, const char* const* dirs, uint32_t ndirs, const pcv_xray_quadtree_params* params, const pcv_interval* filters,
                                uint32_t nfilt, uint64_t max_device_bytes, pcv_xray_tile_fn on_tile, void* user, pcv_xray_quadtree_info* info_out,
                                pcv_xray_bounded_info* bounded_info_out, pcv_xray_dir_info* dir_info_out);
int pcv_xray_quadtree_from_dirs_write_dir(pcv_ctx* ctx, const char* const* dirs, uint32_t ndirs, const pcv_xray_quadtree_params* params,
                                          const pcv_interval* filters, uint32_t nfilt, uint64_t max_device_bytes, const char* out_dir,
                                          pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out, pcv_xray_dir_info* dir_info_out);

/* merge_xray_quadtrees (xray/src/bin/merge_xray_quadtrees.rs): partial X-ray quadtrees, each written by a *_write_dir entry with
 * params.root_level / root_index set (<id>.png + meta<digits>.pb), joined into one quadtree in `output_dir`, in the
 * reference's order:
 *   1. every input directory must exist (else PCV_ERR_NOT_FOUND) and be a directory (else PCV_ERR_INVALID) (:101-117); the
 *      output directory is created with its parents if missing (:201-203);
 *   2. every meta*.pb directly inside each input directory is read (:55-72; subdirectories are not searched), as
 *      Meta::from_proto reads it (xray/src/lib.rs:59-116): version 3, or version 2 through deprecated_min / _edge_length when
 *      `min` is unset.  Another version or a malformed file -> PCV_ERR_INVALID naming the file;
 *   3. validate_and_merge_metadata (:125-176), in its order: no meta file -> PCV_ERR_NOT_FOUND ("No subquadtrees meta files
 *      found."); every meta empty -> PCV_ERR_INVALID; roots (a meta's node of least level) not unique, roots on different
 *      levels, deepest_level or tile_size not the same in every meta (empty ones included) -> PCV_ERR_INVALID.  Empty metas are
 *      skipped and counted.  The merged rect is Node::parent (quadtree/src/lib.rs:100-120) walked to level 0 from the root of
 *      the first non-empty meta, taking directories in argument order and their meta files by name;
 *   4. a budget below the walk's device bytes (below) -> PCV_ERR_UNSUPPORTED naming them, before any file is written;
 *   5. copy_images (:28-46): every *.png directly inside each input directory is copied byte for byte into the output
 *      directory, except from an input directory that resolves to the output directory;
 *   6. create_non_leaf_nodes(roots, root level, 0) (generation.rs:656-682, :726-759): every parent from the roots' level - 1 up
 *      to level 0, build_parent's mosaic of its children (background where one is missing) reduced with Lanczos3 to tile_size,
 *      as pcv_xray_build_parent makes it, written as <id>.png.  The sub-roots' images are read back from the output
 *      directory: a missing one -> PCV_ERR_NOT_FOUND; one that is not 8-bit non-interlaced RGBA -> PCV_ERR_UNSUPPORTED; a
 *      corrupt one or one that is not tile_size px square -> PCV_ERR_INVALID;
 *   7. meta.pb (version 3): the merged rect, deepest_level, tile_size and every meta's nodes together with the parents.
 * A call that fails writes no meta.pb, so its output directory does not load as a quadtree.  With root level 0 (one non-empty
 * meta) nothing is built: the images are copied and meta.pb written.
 * Device memory: the sub-roots are walked depth-first in index order, each decoded on host threads ahead of the walk and
 * uploaded once; at most four finished children per level wait for their parent.  The walk holds at most
 * (4 L + 1) tile_size^2 * 4 bytes of tiles, the vertically reduced mosaic (8 tile_size^2 bytes) and the Lanczos3 taps
 * (device_bytes_needed); max_device_bytes bounds it (0: most of the free device memory).  Parent tiles are encoded and written
 * by the PNG writer threads of pcv_xray_quadtree_bounded_write_dir.  Null pointers -> PCV_ERR_INVALID; a file that cannot be
 * read, listed, copied or written -> PCV_ERR_IO. */
typedef struct pcv_xray_merge_info {
    uint32_t metas_read;          /* meta*.pb files read                                                          */
    uint32_t metas_empty;         /* of those, the ones without nodes (skipped)                                   */
    uint8_t root_level;           /* level of the sub-roots                                                       */
    uint8_t deepest_level;        /* Meta::deepest_level                                                          */
    uint32_t tile_size_px;        /* Meta::tile_size                                                              */
    uint64_t roots_decoded;       /* sub-root PNGs decoded and uploaded                                           */
    uint64_t parents_built;       /* parent tiles built and written                                               */
    uint64_t files_copied;        /* *.png files copied into the output directory                                 */
    uint64_t bytes_copied;
    float ms_parents;             /* CUDA events: the parents' Lanczos3 kernels                                   */
    double ms_copy;               /* wall time of the copy                                                        */
    double ms_decode;             /* wall time of reading and decoding the sub-root PNGs, summed over them        */
    double ms_write;              /* wall time of encoding and writing the parent PNGs, summed over them          */
    double ms_total;              /* wall time of the whole call                                                  */
    uint64_t max_device_bytes;    /* the budget used                                                              */
    uint64_t device_bytes_needed; /* what the walk may hold at most                                               */
    uint64_t peak_device_bytes;   /* the most the walk held at once                                               */
} pcv_xray_merge_info;
int pcv_xray_merge_quadtrees(pcv_ctx* ctx, const char* const* input_dirs, uint32_t n, const char* output_dir, const uint8_t background[4],
                             uint64_t max_device_bytes, pcv_xray_merge_info* info_out);

/* inpaint_xray_quadtree (xray/src/bin/inpaint_xray_quadtree.rs, xray/src/inpaint.rs): the leaves of the (possibly partial)
 * quadtree with root R = (root_level, root_index) in `input_dir` - meta<R>.pb and <id>.png files as the *_write_dir entries
 * and pcv_xray_merge_quadtrees leave them, built with a transparent background - get their small holes filled, into
 * `output_dir` (created if missing; it may be `input_dir`):
 *   1. meta<R>.pb is read (missing -> PCV_ERR_NOT_FOUND, as is a missing input directory); the leaves are its nodes at
 *      deepest_level.  A leaf outside R, or R outside its level -> PCV_ERR_INVALID; an odd tile size -> PCV_ERR_UNSUPPORTED;
 *   2. the adjacent leaves (:41-71): the deepest nodes of the metas of R's Left, Top, Right and Bottom neighbour pieces in
 *      `input_dir` whose neighbour in the opposite direction is a leaf (a warning on stderr when there is none and R is not
 *      the root);
 *   3. with inpaint_distance_px = k > 0, every leaf gets a 2T x 2T image stitched from the visible tiles of its 3 x 3
 *      neighbourhood (transparent (255, 255, 255, 0) elsewhere).  Visible: in place (the same realpath) every <id>.png of
 *      deepest_level in the directory; otherwise the leaves and the adjacent leaves.  The alpha channel is closed (dilate,
 *      then erode, LInf square of radius k, clipped to the image); a closed pixel of alpha 0 takes the RGBA of the nearest
 *      pixel of alpha != 0 in Euclidean distance, the smaller column, then the smaller row on a tie (texture synthesis in the
 *      reference: see DESIGN.md section 3).  Each image is blended with its Right, then its Bottom neighbour's where that
 *      neighbour is a leaf (weights i / (T - 1), rounded per channel, in f32), and the centre T x T is kept;
 *   4. every leaf's pixels of alpha < 128 become `background` (assign_background_color); k = 0 does only this;
 *   5. the parents from deepest_level - 1 up to root_level, as pcv_xray_merge_quadtrees builds them, from the leaves;
 *   6. the adjacent leaves are not left in `output_dir`, and (copying) meta<R>.pb is copied last, so that a failed call
 *      leaves no meta there.
 * A listed leaf (copying: or adjacent leaf) that is missing or cannot be read -> PCV_ERR_IO; one that is not T x T px ->
 * PCV_ERR_INVALID; k > 255 -> PCV_ERR_INVALID.  Device memory: the leaves go in aligned 2^j x 2^j blocks in index order, j the
 * largest (at most 5) whose block and the parents' walk fit max_device_bytes (0: most of the free device memory); a budget
 * below device_bytes_needed (j = 0) -> PCV_ERR_UNSUPPORTED naming it, before any file is written.  The output does not depend
 * on the budget.  Null pointers -> PCV_ERR_INVALID. */
typedef struct pcv_xray_inpaint_info {
    uint8_t root_level;
    uint8_t deepest_level;
    uint32_t tile_size_px;
    uint32_t inpaint_distance_px;
    uint32_t block_depth;         /* j: blocks of 2^j x 2^j leaves                                               */
    uint64_t leaves;              /* the meta's nodes at deepest_level                                           */
    uint64_t adjacent_leaves;     /* leaves of the neighbour pieces next to them                                 */
    uint64_t tiles_decoded;       /* PNGs decoded (halo tiles count once per block that reads them)              */
    uint64_t hole_pixels_filled;  /* over the leaves' inpaint images, each counted once                          */
    uint64_t blocks;
    uint64_t parents_built;
    uint64_t files_copied;        /* meta<R>.pb when copying                                                     */
    uint64_t bytes_copied;
    uint64_t max_device_bytes;    /* the budget used                                                             */
    uint64_t device_bytes_needed; /* what blocks of one leaf and the parents' walk hold at most                  */
    uint64_t peak_device_bytes;   /* the most held at once                                                       */
    double ms_decode;             /* wall time of reading and decoding the tiles, summed over them               */
    double ms_kernels;            /* CUDA events: stitch, close, fill, blends, crop and background               */
    double ms_parents;            /* CUDA events: the parents' Lanczos3 kernels                                  */
    double ms_encode;             /* wall time of encoding and writing the PNGs, summed over them                */
    double ms_total;              /* wall time of the whole call                                                 */
} pcv_xray_inpaint_info;
int pcv_xray_inpaint_quadtree(pcv_ctx* ctx, const char* input_dir, const char* output_dir, uint8_t root_level, uint64_t root_index,
                              uint32_t inpaint_distance_px, const uint8_t background[4], uint64_t max_device_bytes, pcv_xray_inpaint_info* info_out);

/* The X-ray quadtree straight from one or more S2 directories (meta.pb + cell files, as pcv_s2_write_dir and pcv_s2_build_to_dir
 * leave them), none of them ever resident as a whole: the same tiles, delivery (every tile after its children; the order across
 * blocks follows the block level, as in every bounded entry), cancellation, <id>.png + meta<...>.pb outputs and
 * pcv_xray_bounded_info as pcv_s2_xray_quadtree_clouds over pcv_s2_load_dir of every directory, in the same order.  The
 * quadtree lies over the union of the directories' meta.pb boxes; XRay tiles are byte for byte the same at every budget; the
 * attribute strategies (Binning = None) accumulate as the resident path does, so they are equal up to float atomic ordering.
 * There is no limit on the total, which may exceed device memory and 2^32 points: only one window must fit the budget and hold
 * fewer than 2^32 points.  One streaming pass over every cell's positions marks the leaves a point falls into and takes every
 * cell's exact point box; then each block of leaves runs on its window, the cells of any directory whose point box the block's
 * location (widened by the driver's margin) is not Out of, read from disk (XRay without filters reads .xyz only).  Cells the
 * previous window holds are copied on the device when the budget has room for both.  max_device_bytes bounds everything the
 * call allocates, the windows included (0: most of the free device memory).  Host memory holds the cell tables (id, count,
 * directory, point box: about 64 B per cell), the occupied leaves and the staging of the largest window.  In dir_info_out the
 * "node" counters count cells.  Errors: ndirs == 0 or a null path -> PCV_ERR_INVALID; an unreadable meta.pb -> PCV_ERR_IO; a
 * meta.pb that is not a version 12/13 S2 meta, an invalid or duplicated cell id -> PCV_ERR_INVALID; any cell file a meta
 * declares missing or wrongly sized -> PCV_ERR_NOT_FOUND, found by stat for every directory before the first read (no tile is
 * delivered); filters and a directory without intensity, or PCV_XRAY_COLORED and a directory without colour -> PCV_ERR_INVALID;
 * a binned strategy -> PCV_ERR_UNSUPPORTED; a budget too small for the scan pass, a leaf whose window alone does not fit or holds
 * 2^32 points or more (named), a cell of 2^32 points or more (named by its token) -> PCV_ERR_UNSUPPORTED.  bounded_info_out and
 * dir_info_out may be NULL. */
int pcv_s2_xray_quadtree_from_dirs(pcv_ctx* ctx, const char* const* dirs, uint32_t ndirs, const pcv_xray_quadtree_params* params,
                                   const pcv_interval* filters, uint32_t nfilt, uint64_t max_device_bytes, pcv_xray_tile_fn on_tile, void* user,
                                   pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out, pcv_xray_dir_info* dir_info_out);
int pcv_s2_xray_quadtree_from_dirs_write_dir(pcv_ctx* ctx, const char* const* dirs, uint32_t ndirs, const pcv_xray_quadtree_params* params,
                                             const pcv_interval* filters, uint32_t nfilt, uint64_t max_device_bytes, const char* out_dir,
                                             pcv_xray_quadtree_info* info_out, pcv_xray_bounded_info* bounded_info_out, pcv_xray_dir_info* dir_info_out);

/* The X-ray quadtree of several resident octrees at once (build_xray_quadtree over a list of point_cloud_locations,
 * point_cloud_client/src/lib.rs:118-141), with filter intervals on the intensity.  The quadtree lies over the union of the
 * clouds' boxes (component-wise min and max, empty clouds included).  A leaf is made of every point of every cloud that its
 * location contains and that passes every interval (closed, the attribute as f64); it exists iff one such point does.  XRay
 * tiles do not depend on the clouds' order.  Delivery order, cancellation, the budget (the clouds' own arrays not counted) and
 * the counters are those of pcv_xray_quadtree_bounded, which equals this call with n = 1 and no filters.  Errors: n = 0, a null
 * cloud, clouds on different contexts, filters or the intensity strategy when a cloud has no intensities -> PCV_ERR_INVALID;
 * a binned strategy with n > 1 or with filters -> PCV_ERR_UNSUPPORTED. */
int pcv_xray_quadtree_clouds(const pcv_octree* const* octrees, uint32_t n, const pcv_xray_quadtree_params* params, const pcv_interval* filters, uint32_t nfilt,
                             uint64_t max_device_bytes, pcv_xray_tile_fn on_tile, void* user, pcv_xray_quadtree_info* info_out,
                             pcv_xray_bounded_info* bounded_info_out);
int pcv_xray_quadtree_clouds_write_dir(const pcv_octree* const* octrees, uint32_t n, const pcv_xray_quadtree_params* params, const pcv_interval* filters,
                                       uint32_t nfilt, uint64_t max_device_bytes, const char* directory, pcv_xray_quadtree_info* info_out,
                                       pcv_xray_bounded_info* bounded_info_out);

/* ---- point queries straight from an octree directory (Octree over OnDiskDataProvider, octree/mod.rs:156-215, 337-352) ---- */
/* A directory-backed octree: open reads meta.pb into the node table pcv_octree_load_dir builds and puts its query tables on the
 * device; node files are only stat'ed.  Every call reads, uploads and culls only the nodes it selects, in chunks cut at 2048-point
 * tile boundaries (a node larger than a chunk is read in byte ranges across several chunks), with two pinned host buffers: host
 * threads read chunk i+1 while the device culls chunk i.  Results equal the same calls over pcv_octree_load_dir of the directory,
 * except that src_index is the point's slot (point_offset + j of its node in pcv_octree_dir_nodes; load_dir reports 0).
 * max_device_bytes bounds everything the handle and its calls allocate, the tables included (0: most of the free device memory);
 * a budget that cannot hold the tables, the selection scratch and one chunk of one tile at the widest encoding fails at open with
 * PCV_ERR_UNSUPPORTED.  Errors: a meta.pb other than version 13 -> PCV_ERR_INVALID; a missing or wrongly sized .xyz / .rgb file
 * -> PCV_ERR_NOT_FOUND at open, and from the call that reads a file that has shrunk since.  A handle serialises on its context. */
typedef struct pcv_octree_dir pcv_octree_dir;
int pcv_octree_dir_open(pcv_ctx* ctx, const char* dir, uint64_t max_device_bytes, pcv_octree_dir** out);
void pcv_octree_dir_close(pcv_octree_dir* d);
int pcv_octree_dir_info(const pcv_octree_dir* d, uint64_t* num_nodes, uint64_t* num_points, uint64_t* xyz_bytes, double* resolution,
                        double bbox_min[3], double bbox_max[3], int* has_intensity);
int pcv_octree_dir_nodes(const pcv_octree_dir* d, pcv_node_meta* out, uint64_t cap); /* == pcv_octree_nodes of load_dir */
/* Selection only: no node file is read. */
int pcv_octree_dir_nodes_in_location(const pcv_octree_dir* d, const pcv_location* loc, uint64_t* ids_hi_lo, uint64_t cap, uint64_t* n_out);
int pcv_octree_dir_visible_nodes(const pcv_octree_dir* d, const double clip_from_world[16], uint64_t* ids_hi_lo, uint64_t cap, uint64_t* n_out);
int pcv_octree_dir_query_points(const pcv_octree_dir* d, const pcv_location* loc, const pcv_interval* filters, uint32_t nfilt,
                                uint64_t batch_size, pcv_batch_cb cb, void* user);
/* counts_out / tested_out as pcv_query_batch_device; every node some location visits is read once per call.  A frontier that
 * does not fit what the budget leaves -> PCV_ERR_UNSUPPORTED ("split the batch"). */
int pcv_octree_dir_query_batch(const pcv_octree_dir* d, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters,
                               uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);
/* The cell-union calls over the directory (src_index = slot, max_device_bytes bounds the unions' tables too). */
int pcv_octree_dir_nodes_in_cell_union(const pcv_octree_dir* d, const pcv_cell_union* cu, uint64_t* ids_hi_lo, uint64_t cap, uint64_t* n_out);
int pcv_octree_dir_query_cell_union(const pcv_octree_dir* d, const pcv_cell_union* cu, const pcv_interval* filters, uint32_t nfilt,
                                    uint64_t batch_size, pcv_batch_cb cb, void* user);
int pcv_octree_dir_query_cell_unions_batch(const pcv_octree_dir* d, const pcv_cell_union* unions, uint32_t nunion, const pcv_interval* filters,
                                           uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);
/* pcv_nodes_data_blob's reply, read from the node files straight into `out` on the host. */
int pcv_octree_dir_nodes_data_blob(const pcv_octree_dir* d, const uint64_t* ids_hi_lo, uint32_t num_nodes, void* out, uint64_t cap,
                                   uint64_t* size_out);
typedef struct pcv_dir_query_stats {  /* the last call on the handle                                                     */
    uint64_t max_device_bytes, peak_device_bytes;   /* peak: everything the handle held during the call, tables included */
    uint64_t chunks, node_files_read, bytes_read, bytes_uploaded;
    uint64_t visited_pairs, tested_points, returned_points;
    double ms_select, ms_read_wait, ms_total;       /* wall; ms_read_wait: time the device sat idle waiting for reads    */
    float ms_cull;                                  /* CUDA events, summed over chunks                                   */
    uint32_t kernel_launches;
} pcv_dir_query_stats;
int pcv_octree_dir_last_stats(const pcv_octree_dir* d, pcv_dir_query_stats* out);
/* pcv_query_batch_points_device over the directory: [offsets_out[i], offsets_out[i+1]) of the device arrays holds what
 * pcv_octree_dir_query_points (pcv_octree_dir_query_cell_union for a union) streams for Li, in the same order and bit for bit
 * (d_src: the slot), and offsets_out[i+1] - offsets_out[i] is pcv_octree_dir_query_batch's counts_out[i].  The size query, NULL
 * fields and the argument checks are the resident entry's.  Two passes over one chunk list: a count pass reads every visited
 * node once (.xyz, and .intensity with filters); unless this is a size query, a place pass reads the nodes again (.xyz, and
 * .rgb / .intensity for the fields written or the filters) and writes every survivor at its position; the chunk the count
 * pass ended on is placed without a second read, so a batch whose visited nodes fit one chunk reads every file once.
 * cap < offsets_out[n] is PCV_ERR_INVALID naming both numbers, with offsets_out complete, decided before the place pass: the
 * device arrays are untouched.  max_device_bytes bounds everything but the caller's arrays; a batch whose frontier or per-tile
 * state (4 bytes per (location, node tile)) does not fit -> PCV_ERR_UNSUPPORTED ("split the batch"), the handle still usable.
 * A node file rewritten between the passes -> PCV_ERR_IO (no write ever goes past a tile's counted survivors or past cap).
 * pcv_octree_dir_last_stats: returned_points = offsets_out[n]; tested_points and visited_pairs as query_batch; chunks,
 * node_files_read, bytes_read, bytes_uploaded and ms_cull over both passes (bytes_uploaded counts every chunk image whole,
 * including the colour / intensity regions a count-pass chunk carries for the place pass without reading them). */
int pcv_octree_dir_query_batch_points_device(const pcv_octree_dir* d, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters,
                                             uint32_t nfilt, uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb, float* d_intensity,
                                             uint64_t* d_src, uint64_t cap);
int pcv_octree_dir_query_cell_unions_batch_points_device(const pcv_octree_dir* d, const pcv_cell_union* unions, uint32_t nunion,
                                                         const pcv_interval* filters, uint32_t nfilt, uint64_t* offsets_out, double* d_xyz,
                                                         uint8_t* d_rgb, float* d_intensity, uint64_t* d_src, uint64_t cap);

/* ---- f4: the S2-cell point cloud (src/read_write/s2.rs, src/s2_cells/mod.rs, src/geometry/s2_cell_union.rs) ---- */
/* Cell ids are the S2 library's 64-bit CellID values (face, Hilbert position, level marker bit); the arithmetic is the `s2`
 * crate's, restated (csrc/s2.h): integer and IEEE +, *, /, sqrt only, identical on host and device. */
/* CellID::from_point(p).parent(level) for every point (src/math/mod.rs:119-131). */
int pcv_s2_cell_ids(pcv_ctx* ctx, const pcv_points* host_points, uint32_t level, uint64_t* ids_out);
/* S2Splitter::write over the cloud + get_meta (read_write/s2.rs:52-125,165-173; DEFAULT_S2_SPLIT_LEVEL = 20): every point must
 * be a valid ECEF point (|p| in [6 352 800, 6 384 400] m, else PCV_ERR_INVALID with the reference's message); points are grouped
 * by cell - cells in id order, inside a cell in input order - as Plain-encoded f64 positions plus colour / intensity. */
typedef struct pcv_s2cloud pcv_s2cloud;
int pcv_s2_build(pcv_ctx* ctx, const pcv_points* host_points, uint32_t split_level, pcv_s2cloud** out);
int pcv_s2_build_device(pcv_ctx* ctx, const pcv_points* dev_points, uint32_t split_level, pcv_s2cloud** out);
void pcv_s2_free(pcv_s2cloud* cloud);
/* S2Meta: cells + num_points (mod.rs:23-41), bounding box, attributes. */
int pcv_s2_info(const pcv_s2cloud* cloud, uint64_t* num_cells, uint64_t* num_points, uint32_t* split_level, double bbox_min[3],
                double bbox_max[3], int* has_color, int* has_intensity);
int pcv_s2_cells(const pcv_s2cloud* cloud, uint64_t* ids_out, uint64_t* num_points_out);
/* Device time of the build (CUDA events: keys, sort, run starts, gather; the bounding-box pass and the host reads between them
 * included), kernel launches, and the compulsory bytes: every point read once and written once into its cell. */
int pcv_s2_build_stats(const pcv_s2cloud* cloud, float* ms_device, uint32_t* kernel_launches, uint64_t* algorithmic_bytes);
/* points_in_node (mod.rs:174-190): one cell's arrays; PCV_ERR_NOT_FOUND for an id the cloud does not hold. */
int pcv_s2_cell_data(const pcv_s2cloud* cloud, uint64_t cell_id, double* xyz_out /* n*3 */, uint8_t* rgb_out, float* intensity_out,
                     uint64_t* src_index_out);
/* nodes_in_location for PointLocation::AllPoints (union_ids == NULL) and PointLocation::S2Cells (mod.rs:157-168, 233-241:
 * the cells whose id range intersects the union's; the union is normalised first).  ids_out may be NULL to count. */
int pcv_s2_cells_in_union(const pcv_s2cloud* cloud, const uint64_t* union_ids, uint32_t n_union, uint64_t* ids_out, uint64_t cap,
                          uint64_t* n_out);
/* The FilteredIterator over those cells with the CellUnion as PointCulling (s2_cell_union.rs:27-31): survivors in cell order,
 * input order inside a cell.  n_out = number of survivors (may exceed cap: only cap are written). */
int pcv_s2_query_union(const pcv_s2cloud* cloud, const uint64_t* union_ids, uint32_t n_union, double* xyz_out, uint8_t* rgb_out,
                       float* intensity_out, uint64_t* src_index_out, uint64_t cap, uint64_t* n_out, uint64_t* tested_out);
/* Every PointLocation, with interval filters, streamed or batched on the GPU.  A cell's point box is the exact component-wise
 * min and max of its stored positions.  AllPoints selects every cell; Aabb, Obb, Frustum and WebMercatorRect select the
 * cells whose point box the location's separating-axis test (cache_separating_axes_for_aabb, sat.rs) does not call Out (a cell
 * without points has no box and is never selected); a cell union selects the cells whose id range intersects it.  This cell
 * list is not the reference's (which selects through latitude / longitude rectangles); the points are a superset of the
 * reference's: every point of a selected cell that passes PointCulling::contains and every filter interval (intensity as f64,
 * closed).  Points come in cell (id) order, input order inside a cell; positions are the stored doubles, rgb is NULL for a
 * cloud without colour, src_index is the build input index (the slot for a loaded directory).
 * pcv_s2_cells_in_location: the selected cells in id order (AllPoints: every cell); ids_out may be NULL to count, n_out may
 * exceed cap (only cap are written).  The stream and batch calls behave like pcv_query_points / pcv_query_batch_device
 * (batches of exactly batch_size points but the last, PCV_ERR_CANCELLED when the callback stops, filters on a cloud without
 * intensity are PCV_ERR_INVALID) and fill pcv_last_query_stats the same way; their algorithmic_bytes are 24 B per tested
 * position (+ 4 B of intensity with filters) plus every survivor's position, colour and intensity. */
int pcv_s2_cells_in_location(const pcv_s2cloud* cloud, const pcv_location* loc, uint64_t* ids_out, uint64_t cap, uint64_t* n_out);
int pcv_s2_query_points(const pcv_s2cloud* cloud, const pcv_location* loc, const pcv_interval* filters, uint32_t nfilt,
                        uint64_t batch_size, pcv_batch_cb cb, void* user);
int pcv_s2_query_cell_union(const pcv_s2cloud* cloud, const pcv_cell_union* cu, const pcv_interval* filters, uint32_t nfilt,
                            uint64_t batch_size, pcv_batch_cb cb, void* user);
int pcv_s2_query_batch_device(const pcv_s2cloud* cloud, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters,
                              uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);
int pcv_s2_query_cell_unions_batch_device(const pcv_s2cloud* cloud, const pcv_cell_union* unions, uint32_t nunion,
                                          const pcv_interval* filters, uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);
/* pcv_query_batch_points_device over the cloud: each segment is what pcv_s2_query_points / pcv_s2_query_cell_union streams. */
int pcv_s2_query_batch_points_device(const pcv_s2cloud* cloud, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters,
                                     uint32_t nfilt, uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb, float* d_intensity, uint64_t* d_src,
                                     uint64_t cap);
int pcv_s2_query_cell_unions_batch_points_device(const pcv_s2cloud* cloud, const pcv_cell_union* unions, uint32_t nunion,
                                                 const pcv_interval* filters, uint32_t nfilt, uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb,
                                                 float* d_intensity, uint64_t* d_src, uint64_t cap);
/* The directory an S2Splitter<RawNodeWriter> leaves behind (read_write/s2.rs:127-145, raw.rs): per cell `<to_token()>.xyz`
 * (f64 LE x, y, z), `.rgb`, `.intensity`, and meta.pb = Meta { version 13, bounding_box, s2 { cells, attributes } }
 * (s2_cells/mod.rs:77-104); load = S2Cells::from_data_provider over such a directory (:106-147, :203-216; versions < 12 and
 * octree metas are rejected with the reference's messages). */
int pcv_s2_write_dir(const pcv_s2cloud* cloud, const char* directory);
int pcv_s2_load_dir(pcv_ctx* ctx, const char* directory, pcv_s2cloud** out);
/* S2Splitter::write batch by batch + get_meta (read_write/s2.rs:52-175) for a cloud of any size, straight to a directory in
 * bounded device memory: the directory is byte for byte what pcv_s2_build + pcv_s2_write_dir write for the same points (for a
 * PLY file: pcv_s2_build_device over the points pcv_ply_load_device gives), at every budget and split level.
 *  - Host points (pageable or pinned, SoA or AoS like pcv_s2_build) carry colour / intensity when those pointers are set; a PLY
 *    file carries the attributes it has.  The total may exceed 2^32 points.
 *  - max_device_bytes bounds everything the call allocates on the device (0: most of the free memory); a budget that cannot
 *    hold one minimal batch is PCV_ERR_UNSUPPORTED.  Host memory: two pinned output slots of one batch and 16 B per cell.
 *  - An existing directory: a cell's files are truncated the first time the call writes them, files of other cells are left
 *    alone (OpenMode::Truncate).  Its meta.pb is removed before the first cell file is written; the new one is written last,
 *    through a temporary name, and only on success.  So a failed call (an invalid point in a late batch, an I/O error) leaves
 *    no loadable directory, where the reference would leave the old meta.pb beside half-rewritten cells.
 *  - Errors: an invalid ECEF point is pcv_s2_build's PCV_ERR_INVALID for the first one in input order; no points is
 *    pcv_s2_write_dir's error and writes nothing; a file that cannot be written is PCV_ERR_IO naming it; a truncated PLY body
 *    is PCV_ERR_IO. */
typedef struct pcv_s2_dir_build_info {
    uint64_t num_points, num_cells;
    uint64_t batches, largest_batch;              /* points per batch                                                  */
    uint64_t max_device_bytes, peak_device_bytes; /* the budget used; the most the call held at once                   */
    uint64_t h2d_bytes, d2h_bytes;                /* input read once; cell-ordered output read back once               */
    uint64_t bytes_written, file_writes;          /* node-file bytes; (cell, batch, attribute) writes                  */
    double ms_split;                              /* CUDA events around each batch's split, summed over batches        */
    double ms_input_wait, ms_write_wait, ms_total;/* device time between splits (input); wall time blocked on the
                                                     writers; wall time of the call                                    */
} pcv_s2_dir_build_info;
int pcv_s2_build_to_dir(pcv_ctx* ctx, const pcv_points* host_points, uint32_t split_level, uint64_t max_device_bytes,
                        const char* dir, pcv_s2_dir_build_info* info /* may be NULL */);
int pcv_s2_build_from_file_to_dir(pcv_ctx* ctx, const char* ply_path, uint32_t split_level, uint64_t max_device_bytes,
                                  const char* dir, pcv_s2_dir_build_info* info);
/* build_xray_quadtree over an S2 cloud (xray/src/build_quadtree.rs with S2 locations), in bounded device memory like
 * pcv_xray_quadtree_bounded[_write_dir]: the same post-order delivery, cancellation, <id>.png + meta[<digits>].pb output and
 * pcv_xray_bounded_info.  The quadtree's frame, rect and levels come from the cloud's box (pcv_s2_info: the exact min and max
 * of the stored positions, S2Splitter::get_meta's box), a leaf's location is the Aabb (or, with query_from_global, the Obb) the
 * octree driver builds for it, and a leaf's points are every stored point p (the stored doubles) with loc.contains(p) and
 * lo <= (double)intensity <= hi for every filter interval: xray_from_points over FilteredIterator without the reference's
 * rectangle pre-selection, so a superset of the reference's points as for the S2 location queries.  A leaf exists iff that set
 * is not empty.  XRay tiles are exact; Colored, ColoredWithIntensity and ColoredWithHeightStddev (Binning = None) accumulate
 * like pcv_xray_tile_attr.  Binned strategies (bin_size != 0) are PCV_ERR_UNSUPPORTED; filters on a cloud without intensity
 * and Colored on a cloud without colour are PCV_ERR_INVALID.  max_device_bytes (0: most of the free memory) bounds what the
 * call allocates besides the cloud's arrays and its location tables; info.leaf_points counts the points every binning pass
 * reads.  A block's points are read once to count every leaf's keys and once per key batch to place them (the attribute
 * strategies: once per batch of leaves whose per-pixel sums fit the budget). */
int pcv_s2_xray_quadtree(const pcv_s2cloud* cloud, const pcv_xray_quadtree_params* params, const pcv_interval* filters, uint32_t nfilt,
                         uint64_t max_device_bytes, pcv_xray_tile_fn on_tile, void* user, pcv_xray_quadtree_info* info_out,
                         pcv_xray_bounded_info* bounded_info_out);
int pcv_s2_xray_quadtree_write_dir(const pcv_s2cloud* cloud, const pcv_xray_quadtree_params* params, const pcv_interval* filters, uint32_t nfilt,
                                   uint64_t max_device_bytes, const char* directory, pcv_xray_quadtree_info* info_out,
                                   pcv_xray_bounded_info* bounded_info_out);
/* The X-ray quadtree of several resident S2 clouds at once, with the contract of pcv_xray_quadtree_clouds; also
 * PCV_ERR_INVALID for XRAY_COLORED when a cloud has no colours, and PCV_ERR_UNSUPPORTED for every binned strategy.  n = 1 is
 * pcv_s2_xray_quadtree. */
int pcv_s2_xray_quadtree_clouds(const pcv_s2cloud* const* clouds, uint32_t n, const pcv_xray_quadtree_params* params, const pcv_interval* filters,
                                uint32_t nfilt, uint64_t max_device_bytes, pcv_xray_tile_fn on_tile, void* user, pcv_xray_quadtree_info* info_out,
                                pcv_xray_bounded_info* bounded_info_out);
int pcv_s2_xray_quadtree_clouds_write_dir(const pcv_s2cloud* const* clouds, uint32_t n, const pcv_xray_quadtree_params* params, const pcv_interval* filters,
                                          uint32_t nfilt, uint64_t max_device_bytes, const char* directory, pcv_xray_quadtree_info* info_out,
                                          pcv_xray_bounded_info* bounded_info_out);
/* ---- point queries straight from an S2 directory (S2Cells over OnDiskDataProvider, s2_cells/mod.rs:203-216) ---- */
/* A directory-backed S2 cloud.  Every call returns what the same call returns over pcv_s2_load_dir of the directory: the same cell
 * lists in id order; the same batches (sizes, and element for element xyz, rgb - NULL for a directory without colour -,
 * intensity and src_index, the slot: the cell's start + j, as load_dir reports it); for the batch calls the same counts and
 * tested.  Unlike load_dir the total has no limit: it may exceed device memory and 2^32 points (src_index keeps counting in u64).
 *  - open reads meta.pb and stats every cell file the meta declares; it reads no cell data.  Its errors are those of
 *    pcv_s2_load_dir and pcv_s2_xray_quadtree_from_dirs: meta.pb unreadable -> PCV_ERR_IO; not an S2 meta of version 12 / 13, an
 *    invalid or repeated cell id -> PCV_ERR_INVALID; a declared file missing or of the wrong size -> PCV_ERR_NOT_FOUND; a cell
 *    of 2^32 points or more -> PCV_ERR_UNSUPPORTED naming its token; a budget that cannot hold the handle's tables, the
 *    selection of one location and one chunk -> PCV_ERR_UNSUPPORTED.  A file that shrinks after open is PCV_ERR_NOT_FOUND from
 *    the call that reads it.
 *  - max_device_bytes (0: most of the free memory) bounds everything the handle and its calls allocate: the cell table reserved
 *    at open (a Float64 query node, the id and the 48 B point box per cell), the selection scratch, the locations' tables and
 *    the chunks.  pcv_s2_dir_last_stats: peak_device_bytes <= max_device_bytes after every call.
 *  - Selection: cell unions and AllPoints select by id range and read no file.  Aabb, Obb, Frustum and WebMercatorRect select by
 *    each cell's exact point box (as pcv_s2_cells_in_location); the boxes need every position, so the first call that needs them
 *    streams every .xyz file once and keeps the boxes on the handle (that call's bytes_read, node_files_read and ms_select
 *    include the scan; no later call repeats it).  The boxes equal the loaded cloud's bit for bit.
 *  - Reading: a query reads only the selected cells that hold points, in chunks cut at 2048-point tile boundaries (a cell
 *    larger than a chunk is read in byte ranges across consecutive chunks); host threads read chunk i+1 while the device culls
 *    chunk i.  pcv_s2_dir_query_points / _query_cell_union read .xyz, .rgb when the directory has colour and .intensity when it
 *    has intensity; the batch calls read .xyz, and .intensity only with filters.  A batch call reads every cell some location
 *    selects once, each (location, cell) pair getting its own work tiles; a batch whose tables, selection and one chunk do not
 *    fit the budget -> PCV_ERR_UNSUPPORTED ("split the batch").
 *  - Filters on a directory without intensity -> PCV_ERR_INVALID; a callback that stops -> PCV_ERR_CANCELLED.  The stats'
 *    "node" counters count cells.  A handle serialises on its context. */
typedef struct pcv_s2_dir pcv_s2_dir;
int pcv_s2_dir_open(pcv_ctx* ctx, const char* dir, uint64_t max_device_bytes, pcv_s2_dir** out);
void pcv_s2_dir_close(pcv_s2_dir* d);
int pcv_s2_dir_info(const pcv_s2_dir* d, uint64_t* num_cells, uint64_t* num_points, uint32_t* split_level, double bbox_min[3], double bbox_max[3],
                    int* has_color, int* has_intensity);                                            /* == pcv_s2_info of load_dir */
int pcv_s2_dir_cells(const pcv_s2_dir* d, uint64_t* ids_out, uint64_t* num_points_out);            /* == pcv_s2_cells            */
int pcv_s2_dir_cell_data(const pcv_s2_dir* d, uint64_t cell_id, double* xyz_out, uint8_t* rgb_out, float* intensity_out,
                         uint64_t* src_index_out);                                                   /* points_in_node, from the files */
int pcv_s2_dir_cells_in_union(const pcv_s2_dir* d, const uint64_t* union_ids, uint32_t n_union, uint64_t* ids_out, uint64_t cap, uint64_t* n_out);
int pcv_s2_dir_cells_in_location(const pcv_s2_dir* d, const pcv_location* loc, uint64_t* ids_out, uint64_t cap, uint64_t* n_out);
int pcv_s2_dir_query_points(const pcv_s2_dir* d, const pcv_location* loc, const pcv_interval* filters, uint32_t nfilt, uint64_t batch_size,
                            pcv_batch_cb cb, void* user);
int pcv_s2_dir_query_cell_union(const pcv_s2_dir* d, const pcv_cell_union* cu, const pcv_interval* filters, uint32_t nfilt, uint64_t batch_size,
                                pcv_batch_cb cb, void* user);
int pcv_s2_dir_query_batch(const pcv_s2_dir* d, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters, uint32_t nfilt,
                           uint64_t* counts_out, uint64_t* tested_out);
int pcv_s2_dir_query_cell_unions_batch(const pcv_s2_dir* d, const pcv_cell_union* unions, uint32_t nunion, const pcv_interval* filters,
                                       uint32_t nfilt, uint64_t* counts_out, uint64_t* tested_out);
int pcv_s2_dir_last_stats(const pcv_s2_dir* d, pcv_dir_query_stats* out);
/* pcv_octree_dir_query_batch_points_device over the cells: each segment is what pcv_s2_dir_query_points /
 * pcv_s2_dir_query_cell_union streams (d_src: the slot); a non-null d_rgb on a directory without colour is PCV_ERR_INVALID. */
int pcv_s2_dir_query_batch_points_device(const pcv_s2_dir* d, const pcv_location* locs, uint32_t nloc, const pcv_interval* filters, uint32_t nfilt,
                                         uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb, float* d_intensity, uint64_t* d_src, uint64_t cap);
int pcv_s2_dir_query_cell_unions_batch_points_device(const pcv_s2_dir* d, const pcv_cell_union* unions, uint32_t nunion, const pcv_interval* filters,
                                                     uint32_t nfilt, uint64_t* offsets_out, double* d_xyz, uint8_t* d_rgb, float* d_intensity,
                                                     uint64_t* d_src, uint64_t cap);
/* CellUnion::contains for arbitrary points: mask_out[i] = union.contains_cellid(CellID::from_point(p_i)). */
int pcv_s2_union_contains(pcv_ctx* ctx, const pcv_points* host_points, const uint64_t* union_ids, uint32_t n_union, uint8_t* mask_out);

/* ---- multi-GPU helpers (points shard by level-k path prefix; SURVEY.md 8e) ------------------ */
/* Per-point level-k cell (first k steps of the re-quantising descent on the raw positions) ->
 * 8^k histogram; then a stable pack of the points of each destination rank into contiguous send
 * buffers.  The exchange itself is one NCCL all-to-all issued by the host layer. */
int pcv_prefix_histogram_device(pcv_ctx* ctx, const pcv_points* dev_points, double resolution, const double bbox_min[3],
                                const double bbox_max[3], uint32_t k, uint64_t* counts_out /* 8^k, host */);
/* The same histogram with find_bounding_box (generation.rs:256-270) of the local points folded into the one read of the
 * positions.  Both histogram calls keep the per-point cells on the context for exactly ONE following pack call over the same
 * device arrays, box and resolution, which reuses them instead of repeating the descent and then drops them (the caller must not
 * modify the points between the histogram and that pack; a pack without a fresh histogram recomputes the cells). */
int pcv_prefix_histogram_bbox_device(pcv_ctx* ctx, const pcv_points* dev_points, double resolution, const double bbox_min[3],
                                     const double bbox_max[3], uint32_t k, uint64_t* counts_out, double data_min[3], double data_max[3]);
int pcv_prefix_pack_device(pcv_ctx* ctx, const pcv_points* dev_points, const uint64_t* dev_global_index /* or NULL */,
                           uint64_t global_index_base /* used when dev_global_index == NULL: index = base + i */, double resolution,
                           const double bbox_min[3], const double bbox_max[3], uint32_t k,
                           const int32_t* cell_to_rank /* 8^k, host */, uint32_t nranks, double* dev_xyz_out /* n*3 AoS */,
                           uint8_t* dev_rgb_out, float* dev_intensity_out, uint64_t* dev_index_out,
                           uint64_t* rank_counts_out /* nranks, host */);
/* Fused pack + exchange: the same stable pack, but every record is stored straight into the destination rank's receive
 * arrays (SoA: x, y, z f64; global index u64; intensity f32; colour packed r | g << 8 | b << 16 as u32) - local memory
 * for the own rank, peer memory mapped through CUDA IPC (below) for the others, so the transfer over NVLink / NVSwitch
 * overlaps the ranking; there is no send buffer and no collective call.  dst_*[r]: base pointers of rank r's arrays as
 * mapped in THIS process; dst_first[r]: first slot of this rank's block inside them (sum of the counts of lower ranks).
 * The call returns after the kernel has completed; the caller then runs one inter-process barrier. */
int pcv_prefix_pack_exchange_device(pcv_ctx* ctx, const pcv_points* dev_points, const uint64_t* dev_global_index /* or NULL */,
                                    uint64_t global_index_base, double resolution, const double bbox_min[3], const double bbox_max[3],
                                    uint32_t k, const int32_t* cell_to_rank /* 8^k, host */, uint32_t nranks,
                                    const uint64_t* dst_first /* nranks, host */, void* const* dst_x, void* const* dst_y, void* const* dst_z,
                                    void* const* dst_index, void* const* dst_intensity /* or NULL */, void* const* dst_colour,
                                    uint64_t* rank_counts_out /* nranks, host */);
int pcv_unpack_colours_device(pcv_ctx* ctx, const uint32_t* dev_colour, uint64_t n, uint8_t* dev_rgb /* n * 3 */);
/* Exportable device memory (plain cudaMalloc + cudaIpcGetMemHandle) and its mapping in a peer process. */
int pcv_ipc_alloc(pcv_ctx* ctx, uint64_t bytes, void** dev_ptr, uint8_t handle_out[64]);
int pcv_ipc_free(pcv_ctx* ctx, void* dev_ptr);
int pcv_ipc_open(pcv_ctx* ctx, const uint8_t handle[64], void** dev_ptr);
int pcv_ipc_close(pcv_ctx* ctx, void* dev_ptr);
/* ---- exchange of ingested records (SURVEY.md 8e, round 2): every rank runs the first step of the chain on its own points, the
 * records (three level-1 codes 12 B + packed colour 4 B as one 16-byte record, digits 1 B [+ intensity 4 B]; Float64 trees: 32-byte
 * records + a separate colour array) move once into the owners' receive slabs, and every owner's build starts at its first
 * partition pass - nothing is computed twice and 17 instead of 40 bytes per point cross NVLink.
 *   pcv_shard_ingest_device   ingest kernel + per-tile digit histogram of the local points; counts_out = their 8^k level-k cells
 *   pcv_shard_exchange_device one kernel: rank every record by destination and store it straight into the destination slab
 *                             (dst_*[r] = rank r's slab arrays as mapped in THIS process, capacity + 64 bytes of slack each;
 *                             dst_first[r] = first slot of this rank's block in them).  idx of a stored record = its slot.
 *                             Returns after the kernel has completed; the caller then runs one inter-process barrier.
 *   pcv_shard_send_dest       per local point the rank it went to (device, n bytes; valid until pcv_shard_send_free)
 *   pcv_build_octree_from_records_device  the owner's build over its slab (dev_col == NULL: narrow records carrying their colour,
 *                             as pcv_shard_exchange_device stores them; the slab is reused as scratch by the build). */
typedef struct pcv_shard_send pcv_shard_send;
int pcv_shard_ingest_device(pcv_ctx* ctx, const pcv_points* dev_points, double resolution, const double bbox_min[3], const double bbox_max[3],
                            uint32_t k, uint64_t* counts_out /* 8^k, host */, pcv_shard_send** out);
int pcv_shard_exchange_device(pcv_shard_send* s, uint32_t k, const int32_t* cell_to_rank /* 8^k, host */, uint32_t nranks,
                              const uint64_t* dst_first /* nranks, host */, void* const* dst_rec, void* const* dst_col, void* const* dst_dig,
                              void* const* dst_intensity /* or NULL */, uint64_t* rank_counts_out /* nranks, host */);
int pcv_shard_send_info(const pcv_shard_send* s, int* wide_records /* 1: 32-byte records (a Float64 level exists) */, int* digit_levels);
int pcv_shard_send_dest(const pcv_shard_send* s, const uint8_t** dev_dest, uint64_t* n);
void pcv_shard_send_free(pcv_shard_send* s);
int pcv_build_octree_from_records_device(pcv_ctx* ctx, void* dev_rec, uint32_t* dev_col, uint8_t* dev_dig, const float* dev_intensity, uint64_t n,
                                         double resolution, const double bbox_min[3], const double bbox_max[3], uint32_t k,
                                         const uint64_t* prefix_counts, pcv_octree** out);
/* ---- fused exchange pass: the sender's first partition pass (root -> level-2 cells, two levels of the chain finished, the next
 * pass's first step done) stores every bucket straight into the buffers of the cell's owner - peer memory over NVLink - so the
 * transfer overlaps the partition tile by tile and the owner's build starts at its SECOND pass.  Narrow records that continue travel
 * as {codes, colour} + 1 digit byte (17 B per point), their index implied by their position (= slot); records of level-2 leaves go
 * to the owner's arena with an explicit slot.  Needs prefix depth 2; everything follows from the gathered histograms:
 *   hist_all[s * 64 + c]  points of sender s in level-2 cell c (all-gather of pcv_shard_ingest_device's counts at k = 2)
 *   dst[r]                rank r's buffers as mapped in THIS process (capacity >= slots_out[r] entries + 64 bytes of slack each)
 *   slots_out[r]          slots rank r owns; first_bins_out: this rank's own per-cell counts (input of the owner's build)
 * Returns PCV_ERR_UNSUPPORTED when the layout does not allow it (the caller then uses pcv_shard_exchange_device). */
typedef struct pcv_shard_bufs {
    void* rec_next;   /* slots x 16 B (32 B for wide records) */
    void* col_next;   /* wide records only: slots x 4 B, else NULL */
    void* dig_next;   /* slots x 1 B */
    void* arena;      /* slots x 16 / 32 B: leaf records (the whole build's leaf arena) */
    void* col_arena;  /* slots x 4 B */
    void* intensity;  /* slots x 4 B or NULL */
} pcv_shard_bufs;
int pcv_shard_pass_device(pcv_shard_send* s, uint32_t nranks, uint32_t rank, const int32_t* cell_to_rank /* 64 */, const uint64_t* hist_all,
                          const pcv_shard_bufs* dst /* nranks */, uint64_t* slots_out /* nranks or NULL */, uint64_t* first_bins_out /* 64 or NULL */);
/* after pcv_shard_pass_device: per local point its level-2 cell (device, n bytes; valid until pcv_shard_send_free) */
int pcv_shard_send_cells(const pcv_shard_send* s, const uint8_t** dev_cells, uint64_t* n);
/* the owner's build after every sender's pcv_shard_pass_device has completed (one inter-process barrier in between) */
int pcv_build_octree_after_pass_device(pcv_ctx* ctx, const pcv_shard_bufs* own, uint64_t nslots, const uint64_t* first_bins /* 64 */, double resolution,
                                       const double bbox_min[3], const double bbox_max[3], const uint64_t* prefix_counts /* levels 1..2 */, pcv_octree** out);
/* Local part of a sharded build: like pcv_build_octree_device, but nodes of levels <= k take their split decision from
 * the GLOBAL counts (`prefix_counts`: levels 1..k concatenated, 8 + 64 + .. entries, host), and the nodes of level k-1
 * collect the every-8th points of their local children for pcv_assemble_top. */
int pcv_build_octree_sharded_device(pcv_ctx* ctx, const pcv_points* dev_points, double resolution, const double bbox_min[3],
                                    const double bbox_max[3], uint32_t k, const uint64_t* prefix_counts, pcv_octree** out);
/* n(X): size of node X at the moment it is subsampled into its parent (needed from every level-k node by the assembly). */
int pcv_octree_node_nsub(const pcv_octree* o, uint64_t id_high, uint64_t id_low, uint64_t* nsub_out);
int pcv_octree_nsub_all(const pcv_octree* o, uint64_t* out, uint64_t cap); /* same order as pcv_octree_nodes */
/* Nodes of levels 0..k-1 from the gathered collector content (host buffers; level k-1 nodes in index order, inside a
 * node child order, positions as node-file bytes in the collector's encoding).  src_index of the result = position in
 * the gathered arrays. */
int pcv_assemble_top(pcv_ctx* ctx, double resolution, const double bbox_min[3], const double bbox_max[3], uint32_t k,
                     const uint64_t* prefix_counts, const uint64_t* unit_nsub /* 8^k */, const void* xyz_codes, const uint8_t* rgb,
                     const float* intensity, uint64_t npoints, pcv_octree** out);

/* ---- the whole sharded build as ONE call per rank (SURVEY.md 8e).  The three collectives come from the caller (NCCL, MPI,
 * torch.distributed ...: anything that offers them over host buffers), everything else - ingest, global histogram, cells -> ranks,
 * the slab set-up over CUDA IPC (cached per context), the fused record exchange over NVLink, the owner's build, the assembly of the
 * nodes above level k on rank 0 - happens behind this boundary.  Every callback returns 0 on success.  All ranks must call with the
 * same resolution / bbox / prefix_levels (1 or 2); one process per GPU on one node.
 *   local_out: this rank's nodes of levels >= k (and the collectors it contributed to); top_out: rank 0 only, levels < k
 *   k_out: the prefix depth actually used (<= prefix_levels, distributed.py usable_prefix_levels)
 *   cell_to_rank_out / unit_nsub_out: optional, 8^prefix_levels entries each (the first 8^k are written)
 *   recv_points_out: optional, the points this rank owns
 *   send_out: optional; when given, the caller owns the handle and frees it with pcv_shard_send_free.  It keeps one byte per
 *   local point - its level-2 cell (pcv_shard_send_cells) after the fused exchange pass, else the rank it went to
 *   (pcv_shard_send_dest) - which together with the gathered histograms reconstructs the provenance of every slot.
 * PCV_NO_FUSED_PASS=1 (environment) forces the exchange of ingested records + the owner's full build. */
typedef struct pcv_comm {
    void* user;
    int rank, world;
    int (*allreduce_sum_u64)(void* user, uint64_t* inout, uint64_t count);
    int (*allgather)(void* user, const void* send, uint64_t bytes, void* recv /* world * bytes, rank order */);
    int (*barrier)(void* user);
} pcv_comm;
int pcv_build_octree_sharded(pcv_ctx* ctx, const pcv_comm* comm, const pcv_points* dev_points, double resolution, const double bbox_min[3],
                             const double bbox_max[3], uint32_t prefix_levels, pcv_octree** local_out, pcv_octree** top_out, uint32_t* k_out,
                             int32_t* cell_to_rank_out, uint64_t* unit_nsub_out, uint64_t* recv_points_out, pcv_shard_send** send_out);
/* Wall-clock milliseconds of the last pcv_build_octree_sharded on this context, per phase (each ends in a stream synchronisation or
 * a barrier): ingest + histogram, all-reduce + plan (+ slab set-up on the first call), exchange, local build, top assembly;
 * out[5] = 1 when the exchange was the fused exchange pass. */
int pcv_sharded_phases(pcv_ctx* ctx, double out[6]);
/* Releases the receive slab pcv_build_octree_sharded caches on the context (collective: every rank calls it). */
int pcv_sharded_release(pcv_ctx* ctx, const pcv_comm* comm);

/* ---- PLY input (SURVEY.md 8f rank 1): src/read_write/ply.rs:126-229 (parse_header), :327-450
 * (PlyIterator::from_file), :453-556 (batches), src/octree/generation.rs:256-287 (find_bounding_box,
 * build_octree_from_file).  The file body goes to the GPU as raw vertex records through a pinned,
 * double-buffered staging ring; one kernel turns the records into the SoA arrays pcv_build_octree_device
 * takes (position = (x, y, z) as f64 + header offset, colour r,g,b, intensity) and reduces the bounding box
 * in the same pass (the reference reads the whole file twice). ------------------------------------- */
enum {  /* property types, ply.rs:43-73 */
    PCV_PLY_I8 = 0, PCV_PLY_U8, PCV_PLY_I16, PCV_PLY_U16, PCV_PLY_I32, PCV_PLY_U32, PCV_PLY_I64, PCV_PLY_U64, PCV_PLY_F32, PCV_PLY_F64
};
typedef struct pcv_ply_info {
    uint64_t num_points;   /* `element vertex N`                                                   */
    uint64_t header_bytes; /* the body starts here (the vertex element must come first)            */
    uint32_t record_bytes; /* bytes per vertex, skipped properties included                        */
    int32_t has_color;     /* uchar red/green/blue (or r/g/b) present                              */
    int32_t has_intensity; /* float `intensity` present                                            */
    int32_t type_xyz[3];   /* PCV_PLY_* of x, y, z (cast to f64 like `as f64`; int8 reads unsigned) */
    uint32_t off_xyz[3];   /* byte offsets inside the record                                       */
    uint32_t off_rgb[3];
    uint32_t off_intensity;
    double offset[3];      /* `comment offset: x y z`, added to every position                     */
} pcv_ply_info;
/* Parses the header with the reference's rules and error conditions (where the reference panics — no vertex element,
 * not binary_little_endian, missing x/y/z — this returns PCV_ERR_INVALID; unreadable file: PCV_ERR_IO). */
int pcv_ply_read_header(const char* path, pcv_ply_info* out);
/* Kernel-level entry: `n` raw records already in device memory (16-byte aligned) -> SoA arrays (device).  rgb /
 * intensity may be NULL.  bbox_min/max (host, may be NULL) receive the component-wise min/max of the positions
 * (Aabb::grow, aabb.rs:41-44); for n == 0 they are Aabb::zero (generation.rs:269). */
int pcv_ply_unpack_device(pcv_ctx* ctx, const pcv_ply_info* info, const void* dev_records, uint64_t n, double* dev_x,
                          double* dev_y, double* dev_z, uint8_t* dev_rgb, float* dev_intensity, double bbox_min[3],
                          double bbox_max[3]);
/* File -> device SoA arrays (capacity info->num_points each) + bounding box; a truncated body is PCV_ERR_IO. */
int pcv_ply_load_device(pcv_ctx* ctx, const char* path, const pcv_ply_info* info, double* dev_x, double* dev_y,
                        double* dev_z, uint8_t* dev_rgb, float* dev_intensity, double bbox_min[3], double bbox_max[3]);
/* build_octree_from_file (generation.rs:272-287): bounding box of the file's points, then build_octree.  Colour is
 * mandatory; `with_intensity` mirrors "intensity" in the reference's `attributes` argument. */
int pcv_build_octree_from_file(pcv_ctx* ctx, const char* path, double resolution, int with_intensity, pcv_octree** out);

/* ---- out-of-core build_octree: clouds larger than one GPU's memory, straight into the on-disk octree ------------------
 * The input streams through the GPU once to count the level-3 cells, then once per group: a group is a run of consecutive
 * non-empty cells of the prefix level k actually used, filled up to the budget, and is built like one rank of
 * pcv_build_octree_sharded; the nodes above level k come from pcv_assemble_top at the end.  The directory is byte for byte what
 * pcv_build_octree[_from_file] + pcv_octree_write_dir write for the same input.  Device memory stays within one in-core build
 * of the budget; the total point count may exceed 2^32 (each group and the nodes above level k stay below 2^32 - 1).
 * A single level-k cell above the budget is PCV_ERR_UNSUPPORTED (the message names the cell, its count and the budget); that
 * includes a cloud whose usable prefix level dropped because a node above it is a leaf. */
/* Points one in-core build (pcv_build_octree[_device]) can take on this context now: free device memory over the build's
 * per-point working set, capped at 2^32-2.  Also the default group budget below. */
int pcv_in_core_capacity(pcv_ctx* ctx, int with_intensity, uint64_t* max_points);
typedef struct pcv_ooc_info {
    uint32_t prefix_levels; /* k actually used (1..3; 0 for an empty cloud)                              */
    uint32_t groups;        /* in-core builds run                                                       */
    uint64_t num_points, num_nodes, largest_group;
    uint64_t h2d_bytes;     /* input bytes copied host -> device over all passes                         */
    double ms_histogram, ms_select, ms_build, ms_write, ms_top, ms_total; /* wall clock, each phase ends in a stream sync;
                                                                            ms_histogram includes a PLY file's bounding-box pass */
} pcv_ooc_info;
/* build_octree (generation.rs:289-295) for a cloud in host memory of any size (pageable or pinned, SoA or AoS like
 * pcv_build_octree): writes <dir>/<NodeId>.xyz|.rgb|.intensity + meta.pb.  max_points_in_core = 0: pcv_in_core_capacity.
 * info may be NULL. */
int pcv_build_octree_to_dir(pcv_ctx* ctx, const pcv_points* host_points, double resolution, const double bbox_min[3],
                            const double bbox_max[3], uint64_t max_points_in_core, const char* dir, pcv_ooc_info* info);
/* build_octree_from_file (generation.rs:272-287) for a PLY file of any size: the body streams from disk on every pass (one
 * bounding-box pass, one histogram pass, one pass per group). */
int pcv_build_octree_from_file_to_dir(pcv_ctx* ctx, const char* ply_path, double resolution, int with_intensity,
                                      uint64_t max_points_in_core, const char* dir, pcv_ooc_info* info);

/* ---- synthetic inputs for benchmarks / parity tests (integer-only, counter based) ----------- */
enum { PCV_SYNTH_SLAB_ECEF = 1, PCV_SYNTH_GAUSS_CLUSTERS = 2 };
int pcv_synth_points_device(pcv_ctx* ctx, int kind, uint64_t seed, uint64_t first_index, uint64_t n, double* dev_x,
                            double* dev_y, double* dev_z, uint8_t* dev_rgb);
int pcv_synth_points_host(int kind, uint64_t seed, uint64_t first_index, uint64_t n, double* x, double* y, double* z, uint8_t* rgb);
int pcv_synth_bbox(int kind, double bbox_min[3], double bbox_max[3], double* resolution);

/* ---- device memory from the context's stream-ordered pool (so that callers' staging buffers, e.g. the all-to-all
 * send/receive buffers of the sharded build, share one allocator with the build's working set) --------------------- */
int pcv_device_alloc(pcv_ctx* ctx, uint64_t bytes, void** out); /* usable on any stream after the call returns */
int pcv_device_free(pcv_ctx* ctx, void* ptr);                   /* caller guarantees its own streams are done with it */

/* ---- instrumentation ------------------------------------------------------------------------ */
typedef struct pcv_build_stats {
    uint64_t kernel_launches; /* CUDA kernels launched by the last build on this context           */
    uint32_t passes;
    uint32_t deepest_level;
    uint64_t num_nodes;
    uint64_t algorithmic_bytes; /* 27*N + sum_nodes n*(3*bpc+3) (+8*N with intensity)             */
    float ms_host_plan, ms_partition, ms_place, ms_total; /* ms_partition/place/total: CUDA events on the context's stream;
                                                             ms_host_plan: host time spent planning passes (inside ms_total) */
    float ms_host_wait;                                   /* host time blocked on the per-pass histogram read-back       */
} pcv_build_stats;
/* Work buffers are recycled inside the context (by exact size, at most half of the device memory) and in the device's stream-ordered
 * pool, so that repeated builds make no allocator calls.  This returns all of it to the driver (e.g. before another library needs
 * the memory). */
int pcv_release_cached_memory(pcv_ctx* ctx);
int pcv_last_build_stats(pcv_ctx* ctx, pcv_build_stats* out);
/* Optional per-kernel timing: CUDA events on the context's stream around every launch of the build kernels.
 * Off by default (the events serialise nothing but cost host time); turn on for a measurement build. */
typedef struct pcv_kernel_stat {
    char name[24];
    uint64_t launches;
    uint64_t algorithmic_bytes; /* bytes the launches had to move (reads of inputs/records + writes of records/outputs) */
    double ms;
} pcv_kernel_stat;
int pcv_set_profiling(pcv_ctx* ctx, int on); /* also resets the accumulated statistics */
int pcv_kernel_stats(pcv_ctx* ctx, pcv_kernel_stat* out, uint32_t cap, uint32_t* n_out);
uint64_t pcv_kernel_launch_count(pcv_ctx* ctx); /* cumulative, all entry points                    */

#ifdef __cplusplus
}
#endif
#endif /* PCV_H */
