/* oracle/tsdf_oracle.h — C API of the CPU oracle.  TEST INFRASTRUCTURE ONLY.
 *
 * The oracle is a CPU restatement of the reference's volumetric path
 * (sdmiller/cpu_tsdf @ 9b973cb): octree storage, integrateCloud/updateVoxel, point
 * queries, renderView, marching cubes and the .vol writer.  It exists to CHECK the CUDA
 * engine; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load it.  The product library never links or calls it.
 *
 * Parity status: the reference ships no tests, golden vectors or fixtures for this path
 * (SURVEY.md §4, §8c), and its third-party arithmetic (PCL/Eigen) is not in this
 * container.  The restatement is pinned against the reference's own sources compiled
 * verbatim (oracle/_ref, built by oracle/Makefile when /root/reference is present) and
 * against analytic known-answer tests; where that pin is unavailable the parity is
 * "unpinned" in the sense of the task statement.  See DESIGN.md §Oracle.
 */
#ifndef TSDF_ORACLE_H
#define TSDF_ORACLE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_config
{
  int32_t xres, yres, zres;            /* setResolution   (tsdf_volume_octree.cpp:93)  */
  float xsize, ysize, zsize;           /* setGridSize     (:111)                        */
  float max_dist_pos, max_dist_neg;    /* setDepthTruncationLimits (:145)               */
  float max_weight;                    /* setWeightTruncationLimit (:162)               */
  float min_sensor_dist, max_sensor_dist; /* setSensorDistanceBounds (h:174)            */
  float max_cell_x, max_cell_y, max_cell_z; /* setMaxVoxelSize (h:154)                  */
  double fx, fy, cx, cy;               /* setCameraIntrinsics (:176)                    */
  int32_t image_width, image_height;   /* setImageSize (:129)                           */
  int32_t integrate_color;             /* setIntegrateColor (h:162); colour mode "RGB"  */
  int32_t num_threads;                 /* OpenMP threads for update/render; 0 = default */
  double global_transform[16];         /* setGlobalTransform (h:119), row-major 4x4     */
  int32_t color_mode;                  /* setColorMode (h:290): 0 "RGB", 1 "RGBNormalized" (octree.cpp:378-433) */
  int32_t reserved_;
} orc_config;

typedef struct orc_volume orc_volume;

void orc_default_config (orc_config* cfg);          /* ctor defaults, cpp:54-85 */
orc_volume* orc_create (const orc_config* cfg);
void orc_destroy (orc_volume* v);
int  orc_reset (orc_volume* v);                     /* cpp:201-219 */

/* integrateCloud (hpp:48-103).  points: organized W x H, row-major, `stride` bytes per
 * point, xyz floats at xyz_off, PCL-order colour bytes (b,g,r,a) at rgba_off (or -1).
 * pose = camera->world 4x4 row-major double. */
int  orc_integrate (orc_volume* v, const void* points, size_t stride, int xyz_off, int rgba_off,
                    int width, int height, const double* pose);

/* per-frame statistics of the last integrate call */
typedef struct orc_stats
{
  int64_t n_add_observation;   /* addObservation calls                 */
  int64_t n_node_visits;       /* updateVoxel calls                    */
  int64_t n_presplit;          /* split() calls in the pre-split loop  */
  int64_t n_culled_cells;      /* coarse cells kept by the frustum cull */
  int64_t n_nodes;             /* live nodes in the tree               */
  double t_presplit, t_cull, t_update;  /* seconds */
  int64_t n_prune_existing;    /* nodes whose children, present before this frame, were all pruned (hpp:136-141) */
  int64_t n_prune_resplit;     /* of those, nodes that split again in the same updateVoxel call (hpp:161-165) */
} orc_stats;
void orc_get_stats (const orc_volume* v, orc_stats* s);

/* what: bit0 = value, bit1 = gradient, bit2 = hessian.  mode 0 = separate getFxn /
 * getGradient / getHessian (cpp:655-725); mode 1 = combined getFxnAndGradient /
 * getFxnGradientAndHessian (cpp:728-794).  ok[i] = return value. */
int  orc_query (const orc_volume* v, const float* xyz, int n, int what, int mode,
                float* val, float* grad, float* hess, uint8_t* ok);

/* renderView (cpp:278-424): out = (W/ds)*(H/ds) points of `stride` bytes, xyz floats at
 * xyz_off, normal at normal_off (PointNormal: 0 / 16 / stride 48).  rgb_out (optional,
 * 3 bytes r,g,b per pixel) follows renderColoredView (cpp:427-450). */
/* interpolateTrilinearly / getTSDFValue (tsdf_volume_octree.cpp:454-541; protected in the reference, reached through a derived
 * accessor in the verbatim build): valid_in_out[i] is the caller's `*valid` on entry (the reference only ever clears it) */
int  orc_interpolate (const orc_volume* v, const float* xyz, int n, float* val, uint8_t* valid_in_out);
int  orc_render (const orc_volume* v, const double* pose, int downsample, void* out, size_t stride,
                 int xyz_off, int normal_off, uint8_t* rgb_out);

/* MarchingCubesTSDFOctree::performReconstruction (marching_cubes_tsdf_octree.cpp:108).
 * color_mode: 0 none, 1 rgb, 2 confidence.  Returns number of vertices (3 per triangle);
 * buffers are owned by the volume until the next call. */
int64_t orc_mesh (orc_volume* v, float w_min, int color_mode, const float** verts, const uint8_t** rgb);

int  orc_save (const orc_volume* v, const char* path);   /* cpp:222-245 */

/* dump every node at depth >= coarse level, sorted by (level, x, y, z).
 * keys: 4 int32 per node (level, ix, iy, iz); dw: 2 floats; flags: bit0 = has children;
 * rgb: 3 bytes; M: float; ns: int32.  Any pointer may be NULL.  Returns node count. */
int64_t orc_dump_nodes (const orc_volume* v, int32_t* keys, float* dw, uint8_t* flags,
                        uint8_t* rgb, float* M, int32_t* ns);
int  orc_levels (const orc_volume* v, int* coarse_level, int* finest_level);
/* RGBNormalized payload (r_n_, g_n_, b_n_, i_: 4 floats per node) in the node order of orc_dump_nodes; returns the node
 * count, or 0 when the volume does not use that node type */
int64_t orc_dump_color_payload (const orc_volume* v, float* out4);

/* helpers exposed for known-answer tests */
void orc_voxel_center (const orc_volume* v, int64_t x, int64_t y, int64_t z, float* out3);      /* cpp:553 */
int  orc_voxel_index (const orc_volume* v, float x, float y, float z, int* out3);               /* cpp:562 */
int  orc_frustum_cull (const orc_volume* v, const double* pose, uint8_t* mask /* 8^coarse */);  /* cpp:619 */

#ifdef __cplusplus
}
#endif
#endif
