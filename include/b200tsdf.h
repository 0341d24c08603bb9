/* b200tsdf.h — C ABI of the H100-native TSDF fusion engine (libb200tsdf.so).
 *
 * Drop-in boundary for the volumetric path of sdmiller/cpu_tsdf.  The reference has no FFI
 * layer: its boundary is the C++ class surface cpu_tsdf::TSDFVolumeOctree /
 * cpu_tsdf::MarchingCubesTSDFOctree.  Each entry point below names the reference method it
 * replaces (paths relative to the reference tree); the C++ shim in
 * include/cpu_tsdf_b200/tsdf_volume_octree.h and the Python mirror in cpu_tsdf_b200/ marshal
 * PCL/Eigen-shaped arguments into these calls.  See INTEGRATION.md.
 *
 * Conventions: plain pointers and sizes only; every function returns 0 on success or a
 * negative B200TSDF_E* code (the library never throws across the ABI);
 * b200tsdf_last_error() gives a message.  A handle owns one CUDA device + one stream and is
 * not thread-safe for concurrent mutation (same contract as the reference, SURVEY.md §8b).
 * There is NO CPU fallback: without a CUDA device b200tsdf_create fails with
 * B200TSDF_ENODEVICE.
 */
#ifndef B200TSDF_H
#define B200TSDF_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200TSDF_OK          0
#define B200TSDF_EINVAL     -1   /* bad argument / unsupported configuration          */
#define B200TSDF_ENODEVICE  -2   /* no CUDA device (there is no CPU path)             */
#define B200TSDF_ECUDA      -3   /* CUDA runtime error                                */
#define B200TSDF_ENOMEM     -4   /* brick pool / device memory exhausted              */
#define B200TSDF_ESTATE     -5   /* call order (e.g. integrate before reset)          */
#define B200TSDF_EIO        -6   /* file I/O                                          */

#define B200TSDF_COLOR_RGB             0
#define B200TSDF_COLOR_RGB_NORMALIZED  1
#define B200TSDF_COLOR_LAB             2   /* not supported: b200tsdf_reset returns B200TSDF_EINVAL */

typedef struct b200tsdf b200tsdf_t;

/* Mirrors the TSDFVolumeOctree setters; defaults = its constructor
 * (src/lib/tsdf_volume_octree.cpp:54-85).  As in the reference, changes take effect at the
 * next b200tsdf_reset() (cpp:201-211). */
typedef struct b200tsdf_config
{
  int32_t xres, yres, zres;                 /* setResolution            cpp:93   */
  float   xsize, ysize, zsize;              /* setGridSize              cpp:111  */
  float   max_dist_pos, max_dist_neg;       /* setDepthTruncationLimits cpp:145  */
  float   max_weight;                       /* setWeightTruncationLimit cpp:162  */
  float   min_sensor_dist, max_sensor_dist; /* setSensorDistanceBounds  tsdf_volume_octree.h:174 */
  float   max_cell_x, max_cell_y, max_cell_z; /* setMaxVoxelSize        tsdf_volume_octree.h:154 */
  double  fx, fy, cx, cy;                   /* setCameraIntrinsics      cpp:176  */
  int32_t image_width, image_height;        /* setImageSize             cpp:129  */
  int32_t integrate_color;                  /* setIntegrateColor        tsdf_volume_octree.h:162 (colour mode "RGB") */
  int32_t track_variance;                   /* keep OctreeNode::M_/nsample_ (octree.cpp:160-161) for .vol fidelity */
  int32_t device;                           /* CUDA device ordinal                                */
  int32_t pool_log2;                        /* brick pool capacity = 2^pool_log2 (0 = default 20) */
  int32_t shard_rank, shard_count;          /* this handle owns coarse cells with hash(cell) % shard_count == shard_rank */
  int32_t debug_flags;                      /* bit0: general depth-first update kernel only; bit1: per-level upper sweeps instead of the fused per-cell ones;
                                               bit2: .vol save and load through the host writer and loader; other bits are ignored */
  int32_t color_mode;                       /* setColorMode (tsdf_volume_octree.h:290) — B200TSDF_COLOR_RGB (default) or B200TSDF_COLOR_RGB_NORMALIZED
                                               (octree.cpp:379-434; fused by the general kernel).  "LAB" (octree.cpp:436-581) is refused: RGB2LAB needs libm pow */
  int32_t reserved[2];
  double  global_transform[16];             /* setGlobalTransform tsdf_volume_octree.h:119; row-major 4x4 */
} b200tsdf_config;

void b200tsdf_default_config (b200tsdf_config* cfg);

/* TSDFVolumeOctree ctor / dtor (cpp:54, :86) */
int  b200tsdf_create (const b200tsdf_config* cfg, b200tsdf_t** out);
void b200tsdf_destroy (b200tsdf_t* h);
const char* b200tsdf_last_error (const b200tsdf_t* h);

/* the setters: stores the configuration used by the next reset() */
int  b200tsdf_set_config (b200tsdf_t* h, const b200tsdf_config* cfg);
int  b200tsdf_get_config (const b200tsdf_t* h, b200tsdf_config* cfg);

/* TSDFVolumeOctree::reset (cpp:201-219).  B200TSDF_EINVAL for a configuration the engine refuses leaves the handle as it
 * was, its volume included.  Any other failure (B200TSDF_ENOMEM when the device memory of the new volume cannot be had)
 * leaves the handle without a volume: every call that needs one returns B200TSDF_ESTATE until a reset succeeds.
 * b200tsdf_load resets the handle to the file's configuration and leaves it the same way when that reset fails. */
int  b200tsdf_reset (b200tsdf_t* h);

/* (no counterpart in the reference) Moves the live volume into a brick pool of 2^pool_log2 bricks (0: the default, 2^20),
 * on the device, so that a volume can start with a small pool and grow, or give back memory it does not use.  The call waits
 * behind all work queued on the handle and returns once the new pool is installed.  The old and the new pool exist side by
 * side while the bricks move: the peak device memory is the sum of both.
 *   B200TSDF_OK: every claimed brick is in the new pool with its key, {d, w} nodes, split words, colour, RGBNormalized and
 *     variance payload and work byte; every other slot of the new pool is fresh.  The root arrays, isEmpty, the frame
 *     numbering and the configuration are unchanged, except that pool_log2 (b200tsdf_get_config) and pool_capacity
 *     (b200tsdf_get_stats) report the new size.  Integration continues bit for bit as on a handle reset with that pool.
 *     The same size as now is allowed and rehashes too.
 *   B200TSDF_EINVAL, nothing changed: pool_log2 outside what reset() accepts ([8, 26], or 0); the claimed bricks
 *     (b200tsdf_stats::n_bricks) above 7/8 of the new capacity, the load limit of a resize; or a brick that finds no slot
 *     within the probe limit of the new pool.
 *   B200TSDF_ENOMEM, nothing changed: the new pool cannot be allocated.
 *   B200TSDF_ESTATE, nothing changed: before reset(), or when an earlier call left an error latched (a pool that overflowed
 *     in an earlier frame, a frame left half launched): resizing does not make an incomplete volume whole; reset() it.
 *   B200TSDF_ECUDA: a CUDA error; one while the new pool is installed leaves the handle without a volume, as reset() does.
 * Not collective: each shard resizes its own handle, and b200tsdf_gather_volume takes shards of any pool sizes. */
int  b200tsdf_resize_pool (b200tsdf_t* h, int pool_log2);

/* TSDFVolumeOctree::integrateCloud<PointT,NormalT> (include/cpu_tsdf/impl/
 * tsdf_volume_octree.hpp:48-103).  points: organized W x H cloud in the sensor frame,
 * row-major (cloud(u,v) = points[v*W+u]), `stride` bytes per point, xyz as 3 floats at
 * xyz_off, PCL colour bytes (b,g,r,a) at rgba_off or -1.  NaN z = invalid.  pose_c2w =
 * camera->world Affine3d as a row-major 4x4.  The normals argument of the reference is unused
 * there (hpp:51) and has no counterpart.  The host buffer is not retained after return.
 * Points wider than 16 bytes are packed to 16-byte pixels {x, y, z, bgra} on the host (a small pool of worker threads,
 * csrc/host_pack.h; bit-preserving) so that only the bytes the fusion reads cross PCIe — pageable clouds included; environment
 * switches in INTEGRATION.md §5. */
int  b200tsdf_integrate (b200tsdf_t* h, const void* points, size_t stride, int xyz_off, int rgba_off,
                         int width, int height, const double* pose_c2w);
/* same, with the cloud already resident in device memory of h's device (no copy, async on the
 * handle's stream; call b200tsdf_sync before reading results on the host) */
int  b200tsdf_integrate_device (b200tsdf_t* h, const void* d_points, size_t stride, int xyz_off, int rgba_off,
                                int width, int height, const double* pose_c2w);
/* n consecutive integrateCloud calls (hpp:48-103) on clouds resident in device memory, fused in order: the frame
 * parameters go to the device in one copy and the launches of the whole batch are one CUDA-graph launch (captured once
 * per batch size, replayed afterwards), so the host issues ~3 driver calls per batch instead of ~6 per frame.
 * d_points: n device pointers (same layout for all); poses_c2w: n row-major 4x4 matrices back to back.  Asynchronous
 * like b200tsdf_integrate_device.  Every configuration takes this path, those fused by the general depth-first kernel
 * (track_variance, RGBNormalized payload) included.  Every argument of every frame is checked before the first frame is
 * fused: a refused call (B200TSDF_EINVAL, e.g. a NULL pointer anywhere in d_points) enqueues nothing and leaves the handle
 * as it was. */
int  b200tsdf_integrate_batch_device (b200tsdf_t* h, int n, const void* const* d_points, size_t stride, int xyz_off, int rgba_off,
                                      int width, int height, const double* poses_c2w);
/* streaming variant of b200tsdf_integrate for producers that keep their (pinned) frame buffers alive:
 * returns as soon as the copy and the kernels are enqueued.  `points` must stay valid and unmodified
 * until b200tsdf_sync() or until two further frames have been submitted on this handle by b200tsdf_integrate or
 * b200tsdf_integrate_async (the call that submits frame i+2 of these two waits for the upload of frame i before it returns;
 * frames of the other entry points do not count); when the upload is packed on the host (see
 * b200tsdf_integrate) the buffer is already free on return.
 * Error reporting of the asynchronous entry points (integrate_device / _batch_device / _async, and integrate itself, which
 * waits for its upload only): a device-side failure of frame i (brick pool exhausted, work queue overflow) is reported by
 * the next call on the handle (integrate*, query*, interpolate*, render*) and at the latest by sync / get_stats / mesh / save. */
int  b200tsdf_integrate_async (b200tsdf_t* h, const void* points, size_t stride, int xyz_off, int rgba_off,
                               int width, int height, const double* pose_c2w);
int  b200tsdf_sync (b200tsdf_t* h);

/* ---- unorganised clouds: the z-buffer re-organisation of the reference's `integrate` program ----
 * (src/prog/integrate.cpp:548-635).  Per input point, in this order: scale by cloud_units (:550-559),
 * turn (0,0,0) into NaN when zero_nans (:561-568), map world -> camera with world_to_camera when it is
 * not NULL (pcl::transformPointCloud with poses[i].inverse(), :570-571; row-major 4x4, rows 0..2 used),
 * project with the handle's intrinsics in float (reprojectPoint, :216-222), keep per pixel the point
 * with the smallest z, the earliest such point on ties (:603-606).  Unfilled pixels are x=y=0, z=NaN,
 * rgba=(0,0,0,255) (a default pcl::PointXYZRGBA with z overwritten, :597-598).  */
typedef struct b200tsdf_organize_opts
{
  float   cloud_units;          /* 1 = metres                                   */
  int32_t zero_nans;            /* --zero-nans                                  */
  const double* world_to_camera;/* NULL unless --world (clouds in world frame)  */
} b200tsdf_organize_opts;
/* z-buffer `n` host points (stride / xyz_off / rgba_off as for b200tsdf_integrate) into an organized
 * image_width x image_height cloud written to `out` (host; out_stride >= 16 bytes per pixel: xyz at 0,
 * 1.0f at 12 when out_stride >= 32, colour bytes b,g,r,a at out_rgba_off or not written when -1).
 * n_filled (may be NULL) receives the number of pixels that got a point. */
int  b200tsdf_organize (b200tsdf_t* h, const void* points, size_t n, size_t stride, int xyz_off, int rgba_off,
                        const b200tsdf_organize_opts* opts, void* out, size_t out_stride, int out_rgba_off,
                        int64_t* n_filled);
/* organise + integrateCloud without the organized cloud ever leaving HBM (integrate.cpp:582-635 + :673) */
int  b200tsdf_integrate_unorganized (b200tsdf_t* h, const void* points, size_t n, size_t stride, int xyz_off,
                                     int rgba_off, const b200tsdf_organize_opts* opts, const double* pose_c2w);
/* n consecutive b200tsdf_integrate_unorganized calls (cloud i, pose i, world_to_camera matrix i) on clouds resident in device
 * memory of h's device, with the same result bit for bit.  d_points: n device pointers; counts: n point counts in host memory
 * (0 is allowed and gives an all-NaN organised image; that cloud's pointer may then be NULL; each count < 2^32); one point
 * layout for all (stride, xyz_off and rgba_off multiples of 4, xyz_off + 12 <= stride, rgba_off + 4 <= stride).
 * opts->world_to_camera: NULL or n row-major 4x4 matrices back to back; cloud_units and zero_nans apply to every cloud.
 * poses_c2w: n row-major 4x4 matrices back to back.  Every 32 frames are organised and fused by one CUDA-graph launch
 * (captured once per batch size, replayed afterwards).  Asynchronous on the handle's stream; errors as for
 * b200tsdf_integrate_device.  B200TSDF_EINVAL for a bad argument of any frame (a refused call enqueues nothing and leaves the
 * handle as it was), B200TSDF_ESTATE before reset(), B200TSDF_ENOMEM when the
 * organised images (32 * image_width * image_height * 24 bytes, allocated at the first unorganised integrate and freed by
 * reset()) do not fit. */
int  b200tsdf_integrate_unorganized_batch_device (b200tsdf_t* h, int n, const void* const* d_points, const size_t* counts,
                                                  size_t stride, int xyz_off, int rgba_off,
                                                  const b200tsdf_organize_opts* opts, const double* poses_c2w);

/* ---- depth images ----
 * A depth frame is exactly one integrateCloud of the organised cloud it unprojects to.  For pixel (u, v) of a row-major
 * width x height depth map D, with the handle's intrinsics rounded to float, each operation a float32 operation rounded to
 * nearest:  z = (float) D[v*width + u] * depth_scale;  x = ((float) u - cx) * z / fx;  y = ((float) v - cy) * z / fy.
 * A pixel with D == 0 or z not finite (NaN / inf input, overflow) is invalid: x = y = z = NaN.  Negative z passes through.
 * rgb (optional): a registered image of 3 bytes per pixel, R, G, B, same size; it becomes the PCL colour bytes b, g, r, 255
 * (0, 0, 0, 255 without one) and is ignored by a volume without colour.  width x height must be the configured image size;
 * images are contiguous.  Refused with B200TSDF_EINVAL, nothing enqueued and the handle unchanged: a bad format, a scale that
 * is not finite or <= 0, another size, a NULL depth pointer (in a batch: any of them, or a NULL entry of d_rgb), a depth
 * pointer not aligned to its element size.  B200TSDF_ESTATE before reset() and on a sharded handle; B200TSDF_ENOMEM when the
 * images of one batch (32 * image_width * image_height * 24 bytes, shared with the unorganised batches) do not fit. */
#define B200TSDF_DEPTH_U16  1   /* uint16_t in sensor units (depth_scale metres per unit, e.g. 1e-3) */
#define B200TSDF_DEPTH_F32  2   /* float                                                          */
/* one depth frame from host memory.  The caller's buffers are free when the call returns; the call waits only for the
 * handle's own staging (a small ring of pinned slots), never for the fusion of earlier frames, so the upload of frame i+1
 * overlaps the fusion of frame i.  Errors of the fusion are reported as for b200tsdf_integrate_device. */
int  b200tsdf_integrate_depth (b200tsdf_t* h, const void* depth, int depth_format, float depth_scale, const uint8_t* rgb,
                               int width, int height, const double* pose_c2w);
/* n consecutive b200tsdf_integrate_depth calls on images resident in device memory of h's device (d_depth: n device
 * pointers; d_rgb: NULL or n device pointers; poses_c2w: n row-major 4x4 matrices back to back).  Every 32 frames are
 * unprojected and fused by one CUDA-graph launch.  Asynchronous like b200tsdf_integrate_batch_device. */
int  b200tsdf_integrate_depth_batch_device (b200tsdf_t* h, int n, const void* const* d_depth, int depth_format, float depth_scale,
                                            const void* const* d_rgb, int width, int height, const double* poses_c2w);
/* the organised cloud of one depth frame (device memory) written to d_out as 16-byte pixels {x, y, z, bgra} (device memory,
 * 16-byte aligned, width * height * 16 bytes); the colour word is written whether or not the volume has colour.  Returns when
 * the image is written. */
int  b200tsdf_depth_to_cloud_device (b200tsdf_t* h, const void* d_depth, int depth_format, float depth_scale, const uint8_t* d_rgb,
                                     int width, int height, void* d_out);

/* ---- tracking (no counterpart in the reference; DESIGN.md §3i) ----
 * Refines the camera->world pose of a live frame against the volume by point-to-SDF Gauss-Newton: each sample's residual r and
 * gradient g are b200tsdf_query mode 1's value and gradient at the transformed point.  For every iteration at level l, with
 * estimate T:
 *   samples: pixels (u, v) with u % stride[l] == 0 and v % stride[l] == 0 whose xyz is finite (a depth map is unprojected as
 *     b200tsdf_integrate_depth unprojects it);
 *   q = (float) rows 0..2 of T applied to the point as integrate maps a cloud point into the volume;
 *   inlier: the query at q succeeds, each of its eight neighbour leaves has weight > w_min, and |r| < d_max;
 *   J = [q x g ; g] (left perturbation T <- Exp (xi) T, xi = (omega, v)), Huber weight rho = 1 if |r| <= huber_delta, else
 *     huber_delta / |r|; A = sum rho J J^T, b = sum rho J r, summed in double in a fixed order (identical run to run);
 *   (A + damping diag (A)) xi = -b by LDL^T in double; T <- Exp (xi) T (Rodrigues), rotation re-orthonormalised.
 * A level ends when |omega| < eps_rot and |v| < eps_trans, or after iters[l] iterations.  The call stops early, T kept at the
 * last accepted estimate, with fewer than min_inliers inliers (B200TSDF_TRACK_TOO_FEW_INLIERS) or a pivot that is not > 0 or
 * a non-finite step (B200TSDF_TRACK_SINGULAR).  Each of these is a successful call.
 * The whole schedule is one CUDA-graph launch (captured once per schedule shape and input kind), ordered after all work
 * queued on the handle; the call returns once the result is on the host.  The volume is only read: no node, statistic, frame
 * number or change epoch changes.
 * Refused with B200TSDF_EINVAL, nothing enqueued: a NULL pose, params or result; a pose that is not finite; levels outside
 * 1..4, a stride < 1, iters outside 0..64, huber_delta or d_max not > 0, w_min, damping, eps_rot or eps_trans not finite or
 * (damping, eps_*) < 0, min_inliers < 0; and the input checks of the integrate entry point of the same input.
 * B200TSDF_ESTATE before reset() and on a sharded handle; a latched device error is reported as by b200tsdf_query. */
#define B200TSDF_TRACK_CONVERGED        0   /* the last level ended by the convergence test          */
#define B200TSDF_TRACK_MAX_ITERS        1   /* the last level ran out of iterations                  */
#define B200TSDF_TRACK_TOO_FEW_INLIERS  2
#define B200TSDF_TRACK_SINGULAR         3
typedef struct b200tsdf_track_params
{
  int32_t levels;                           /* 1..4, coarse to fine                                                  */
  int32_t stride[4];                        /* pixel stride of each level, >= 1                                      */
  int32_t iters[4];                         /* iteration cap of each level, 0..64                                    */
  float   huber_delta;                      /* metres                                                                */
  float   d_max;                            /* inlier bound on |r|, metres                                           */
  float   w_min;                            /* inlier bound on the neighbour weights (w > w_min)                     */
  int32_t min_inliers;
  double  damping;                          /* lambda                                                                */
  double  eps_rot, eps_trans;               /* radians, metres                                                       */
} b200tsdf_track_params;
void b200tsdf_default_track_params (b200tsdf_track_params* prm);
typedef struct b200tsdf_track_result
{
  double  pose_c2w[16];                     /* refined pose, row-major                                               */
  int32_t status;                           /* B200TSDF_TRACK_*                                                      */
  int32_t iters[4];                         /* iterations run per level                                              */
  int32_t inliers;                          /* of the last iteration                                                 */
  int32_t n_log;                            /* entries written to the log (the sum of iters)                         */
  int32_t reserved;
  double  rms;                              /* sqrt (sum r^2 / inliers) of the last iteration, 0 without inliers     */
  double  A[36];                            /* sum rho J J^T of the last iteration (undamped), row-major             */
  double  b[6];                             /* sum rho J r of the last iteration                                     */
} b200tsdf_track_result;
/* one iteration of the optional log: its level, inliers, sum rho r^2 and the step xi (zero when the call stopped there) */
typedef struct b200tsdf_track_iter
{
  int32_t level, inliers;
  double  cost;
  double  step[6];
} b200tsdf_track_iter;
/* log: NULL, or room for sum (iters[0 .. levels-1]) entries.  Host depth map (format and size as b200tsdf_integrate_depth;
 * staged through the same pinned slots; the buffer is free when the call returns). */
int  b200tsdf_track_depth (b200tsdf_t* h, const void* depth, int depth_format, float depth_scale, int width, int height,
                           const double* pose0_c2w, const b200tsdf_track_params* prm, b200tsdf_track_result* res,
                           b200tsdf_track_iter* log);
/* the same with the depth map in device memory of h's device */
int  b200tsdf_track_depth_device (b200tsdf_t* h, const void* d_depth, int depth_format, float depth_scale, int width, int height,
                                  const double* pose0_c2w, const b200tsdf_track_params* prm, b200tsdf_track_result* res,
                                  b200tsdf_track_iter* log);
/* an organised cloud in device memory, in the layout of b200tsdf_integrate_device (the colour is not read) */
int  b200tsdf_track_cloud_device (b200tsdf_t* h, const void* d_points, size_t stride, int xyz_off, int width, int height,
                                  const double* pose0_c2w, const b200tsdf_track_params* prm, b200tsdf_track_result* res,
                                  b200tsdf_track_iter* log);

/* getFxn / getGradient / getHessian (cpp:655-725) with mode 0, or the combined
 * getFxnAndGradient / getFxnGradientAndHessian (cpp:728-794) with mode 1.  what: bit0 value,
 * bit1 gradient (3 floats), bit2 hessian (9 floats, row-major).  ok[i] = the reference's bool; where it is 0 the outputs of
 * point i keep the caller's values, as the reference leaves its reference arguments.  xyz/val/grad/hess/ok are host pointers. */
int  b200tsdf_query (b200tsdf_t* h, const float* xyz, int n, int what, int mode,
                     float* val, float* grad, float* hess, uint8_t* ok);

/* getTSDFValue (cpp:454-478) = interpolateTrilinearly (cpp:486-541; use_trilinear_interpolation_ is always true, cpp:80):
 * the trilinear blend of the eight voxels around each point.  val[i] is NaN when the point's voxel is outside the volume or on
 * its border layer; valid_in_out[i] is the caller's `*valid` on entry and is only ever cleared (border, or a neighbour with
 * weight 0), exactly like the reference's pointer argument.  Host pointers. */
int  b200tsdf_interpolate (b200tsdf_t* h, const float* xyz, int n, float* val, uint8_t* valid_in_out);
/* b200tsdf_query / b200tsdf_interpolate on arrays resident in device memory of h's device (every pointer is a device
 * pointer; the same argument checks).  Asynchronous on the handle's stream, ordered after earlier integrates: call
 * b200tsdf_sync (or order the caller's stream behind it) before reading the results.  Errors as for b200tsdf_integrate_device. */
int  b200tsdf_query_device (b200tsdf_t* h, const float* d_xyz, int n, int what, int mode,
                            float* d_val, float* d_grad, float* d_hess, uint8_t* d_ok);
int  b200tsdf_interpolate_device (b200tsdf_t* h, const float* d_xyz, int n, float* d_val, uint8_t* d_valid_in_out);

/* renderView (cpp:278-424) and, with rgb_out != NULL, renderColoredView (cpp:427-450).
 * out: (W/ds)*(H/ds) points of `stride` bytes; xyz at xyz_off, normal at normal_off
 * (pcl::PointNormal: 0 / 16 / 48).  Camera frame, NaN xyz = miss. */
int  b200tsdf_render (b200tsdf_t* h, const double* pose_c2w, int downsample, void* out, size_t stride,
                      int xyz_off, int normal_off, uint8_t* rgb_out);
/* renderView (and renderColoredView with d_rgb != NULL) for n >= 1 poses into device memory of h's device, the same pixels
 * as n calls of b200tsdf_render.  poses_c2w: n row-major 4x4 matrices in host memory (read before the call returns).  Pose
 * i's image starts at d_out + i*(W/ds)*(H/ds)*stride, pixels row-major; 12 bytes of xyz are written at xyz_off and 12 of
 * normal at normal_off, no other byte (d_out, stride and both offsets 4-byte aligned).  d_rgb: 3 bytes per pixel, images
 * back to back.  Asynchronous on the handle's stream and ordered after earlier integrates; errors as for
 * b200tsdf_integrate_device. */
int  b200tsdf_render_batch_device (b200tsdf_t* h, int n, const double* poses_c2w, int downsample, void* d_out, size_t stride,
                                   int xyz_off, int normal_off, uint8_t* d_rgb);

/* MarchingCubesTSDFOctree::performReconstruction (src/lib/marching_cubes_tsdf_octree.cpp:
 * 108-143): triangle soup, 3 vertices per triangle, global transform applied.
 * color_mode 0 none / 1 setColorByRGB / 2 setColorByConfidence.  *verts (3 floats per vertex)
 * and *rgb (3 bytes per vertex, or NULL) are library-owned until the next mesh call or
 * b200tsdf_free.  B200TSDF_ENOMEM when the triangle or sort buffers do not fit. */
int  b200tsdf_mesh (b200tsdf_t* h, float w_min, int color_mode, float** verts, uint8_t** rgb, size_t* nverts);
void b200tsdf_free (void* p);
/* b200tsdf_mesh into device memory of h's device: the same vertices and colours, in the same order.  d_verts: 3 floats per
 * vertex (4-byte aligned); d_rgb: 3 bytes per vertex, or NULL.  capacity: vertices d_verts can hold.  *nverts receives the
 * vertex count (3 per triangle) once the volume has been walked.  d_verts == NULL: count only, nothing is written.
 * capacity < count: B200TSDF_EINVAL, nothing is written.  Exactly 12 * count bytes of d_verts and, when color_mode != 0 and
 * d_rgb != NULL, 3 * count bytes of d_rgb are written.  Ordered after every integrate queued on the handle; returns once the
 * mesh is written (the handle's stream is synchronised, since the count has to reach the host).  Buffers the caller used on
 * its own stream must be idle before the call.  B200TSDF_ESTATE before reset(), B200TSDF_ENOMEM when the triangle or sort
 * buffers do not fit. */
int  b200tsdf_mesh_device (b200tsdf_t* h, float w_min, int color_mode, float* d_verts, uint8_t* d_rgb, size_t capacity,
                           size_t* nverts);

/* ---- incremental meshing: change epochs per coarse cell (DESIGN.md §3g) ------------------------------------
 * A handle keeps a 64-bit epoch, 0 at create.  Every integrated frame (every route), every node-writing
 * b200tsdf_set_containing_voxels[_device] call and every whole-volume change (reset, load, load_device, import_shard, the full
 * handle of gather_volume, a set_config that changes a field) advances it by one.  resize_pool, saves, reads and refused calls
 * do not.  The mesh triangles of coarse cell c depend only on the nodes of cells c + {0,1}^3, and the full mesh is the runs of
 * the cells one after the other in Morton order, so the triangles of the cells a change may have touched can be re-meshed and
 * spliced into an earlier mesh.
 *
 * *now = the handle's epoch.  mask (optional, 8^C bytes, host, layout of b200tsdf_frustum_cull): mask[c] = 1 iff a mesh of
 * cell c taken at epoch `since` may differ from one taken now, i.e. some cell c + {0,1}^3 was stamped after `since`
 * (since = 0: every cell).  Ordered after all queued work (waits for the handle's stream).  B200TSDF_ESTATE before reset()
 * and on a sharded handle; a latched device error is reported as by the other reads. */
int  b200tsdf_changed_cells (b200tsdf_t* h, uint64_t since, uint64_t* now, uint8_t* mask);
/* b200tsdf_mesh_device restricted to the leaves whose coarse cell has mask[c] != 0 (mask == NULL: every cell): exactly the
 * triangles of the full mesh that lie in those cells, in the same relative order, so a cell's triangles are contiguous and
 * cells follow in Morton order.  cell_nverts (optional, host, 8^C int64): the vertex count of each cell, 0 where not selected.
 * d_verts == NULL counts only (cell_nverts is filled); capacity, alignment, colour and error rules as b200tsdf_mesh_device.
 * With a mask or cell_nverts, B200TSDF_ESTATE on a sharded handle. */
int  b200tsdf_mesh_cells_device (b200tsdf_t* h, float w_min, int color_mode, const uint8_t* mask,
                                 float* d_verts, uint8_t* d_rgb, size_t capacity, size_t* nverts, int64_t* cell_nverts);

/* ---- mesh post-processing of the reference's `integrate` program (no volume handle needed) ----------
 * Meshes are indexed: nverts xyz triples + ntris index triples (a marching-cubes soup is tris = 0,1,2,...).
 * Outputs are malloc'ed by the library; release each with b200tsdf_mesh_free.  Vertex colours are not
 * carried: the reference converts the mesh cloud to pcl::PointXYZ in both functions (integrate.cpp:106, 186).
 * flattenVertices (src/prog/integrate.cpp:103-150): vertices closer than min_dist are welded (in index
 * order, as the reference's sweep does), faces that become degenerate are dropped. */
int  b200tsdf_mesh_flatten (int device, const float* verts, size_t nverts, const int32_t* tris, size_t ntris, float min_dist,
                            float** out_verts, size_t* out_nverts, int32_t** out_tris, size_t* out_ntris);
/* cleanupMesh (src/prog/integrate.cpp:152-214): faces whose centroids form clusters (cluster tolerance
 * face_dist) of at most min_neighbors faces are removed, then the vertices no face uses.
 * Both check the triangle indices on the device (the routine of b200tsdf_mesh_flatten_device / _cleanup_device below), so
 * the mesh is uploaded before a bad index is refused with B200TSDF_EINVAL, and without a CUDA device that call fails with
 * B200TSDF_ENODEVICE first. */
int  b200tsdf_mesh_cleanup (int device, const float* verts, size_t nverts, const int32_t* tris, size_t ntris,
                            float face_dist, int min_neighbors,
                            float** out_verts, size_t* out_nverts, int32_t** out_tris, size_t* out_ntris);
void b200tsdf_mesh_free (void* p);
const char* b200tsdf_meshpost_last_error (void);   /* thread-local message of the last failed call above */
/* b200tsdf_mesh_flatten / _cleanup on arrays in device memory of h's device, on h's stream, with the same result bit for bit.
 * d_tris == NULL: a triangle soup, triangle t = {3t, 3t+1, 3t+2}, and nverts must equal 3 * ntris (no index array is
 * built).  The outputs are the caller's and sized like the inputs: d_out_verts 3 * nverts floats, d_out_tris 3 * ntris int32
 * (all four arrays 4-byte aligned); a result never exceeds its input and no byte past *out_nverts / *out_ntris entries is
 * written.  The outputs must not overlap the inputs or each other; the inputs are only read.  The indices are checked on
 * the device: one out of range gives B200TSDF_EINVAL before any output byte is written.  Limits as for the host entry
 * points (nverts < 2^31, min_neighbors in 1..16); B200TSDF_ESTATE before reset(), B200TSDF_ENOMEM when the scratch does not
 * fit; a pending device error of an earlier frame is reported as by the other reads.  Returns once the outputs are written.
 * Errors come through b200tsdf_last_error (h). */
int  b200tsdf_mesh_flatten_device (b200tsdf_t* h, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                                   float min_dist, float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris);
int  b200tsdf_mesh_cleanup_device (b200tsdf_t* h, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                                   float face_dist, int min_neighbors,
                                   float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris);

/* Diagnostics: per-phase timing of the bottom-up per-cell kernel (k_celltop_up).  The first call arms the counters,
 * every call returns and clears them: out16[0..5] = max SM cycles << 32 | tag (total, level-3, level-2, level-1, cell,
 * wait before the first cell), out16[6..10] = slow level-2 nodes, slow level-1 nodes, cell leaf visits, cell
 * fall-throughs, cells folded.  Used by tools/dbg_celltop.py; not needed for normal operation. */
int  b200tsdf_debug_timing (b200tsdf_t* h, unsigned long long* out16);

/* TSDFVolumeOctree::save (cpp:222-245): reference-compatible .vol */
int  b200tsdf_save (b200tsdf_t* h, const char* path);

/* TSDFVolumeOctree::load (cpp:248-275) / TSDFInterface::instantiateFromFile (src/lib/tsdf_interface.cpp:44-51):
 * reads a reference-format .vol (written by the reference or by b200tsdf_save), adopts its configuration
 * (resolution, size, truncation, intrinsics, ..., colour node type) and rebuilds the volume on the device.
 * OctreeNode::M_/nsample_ are kept only if track_variance was set on the handle. */
int  b200tsdf_load (b200tsdf_t* h, const char* path);

/* .vol images in device memory (DESIGN.md §3e).  b200tsdf_save_device writes the whole file image that b200tsdf_save would
 * write (header and body, byte for byte) into d_buf, device memory of the handle's device, and sets *nbytes to its size.
 * d_buf == NULL only sets *nbytes; capacity < *nbytes returns B200TSDF_EINVAL with nothing written.  Ordered after every
 * integrate queued on the handle; returns once the image is written.  B200TSDF_ESTATE before reset(), B200TSDF_ENOMEM when
 * the node records or their sort do not fit.
 * b200tsdf_load_device (h, d_buf, nbytes) is b200tsdf_load of a file holding those nbytes bytes: the same configuration,
 * volume, result codes and messages (the messages name the "device image" instead of a path).
 * Both loaders parse the body on the device when every record of it is where the reference's writer would put it, and
 * otherwise, or when the parser's work space cannot be allocated, run the host loader on the same bytes; bytes after the
 * tree are ignored.  A file holding a {d, w} that fusion does
 * not produce (|d| > 2^38, w < 0, w = -0, 0 < w < 1e-20 or w > 2^38) moves later integrates to the general kernel until the
 * next b200tsdf_reset or load, as b200tsdf_set_containing_voxels does. */
int  b200tsdf_save_device (b200tsdf_t* h, void* d_buf, size_t capacity, size_t* nbytes);
int  b200tsdf_load_device (b200tsdf_t* h, const void* d_buf, size_t nbytes);
/* *on_device = 1 when the last b200tsdf_load / b200tsdf_load_device placed the file's body with the device parser, 0 when the
 * host loader did (debug_flags bit 2, a file no writer produces, or parser work space that could not be allocated) or when
 * the volume comes from b200tsdf_reset.  B200TSDF_ESTATE before reset(). */
int  b200tsdf_load_path (b200tsdf_t* h, int32_t* on_device);

/* Shard gather (multi-GPU, DESIGN.md §5): a handle created with shard_count > 1 owns the coarse cells with
 * hash(cell) % shard_count == shard_rank.  b200tsdf_export_shard serialises everything this handle owns (the
 * coarse-cell entries and every brick below them) into a host buffer (*nbytes needed; pass buf == NULL to query);
 * b200tsdf_import_shard merges such a buffer into a handle with the same grid configuration.  Importing all
 * shards into one volume reproduces the unsharded volume bit for bit; rendering, queries and meshing then run on
 * that volume.  Only grids whose coarse cells are the top-tier roots are supported (e.g. 2048^3/10 m, 512^3/3 m). */
int  b200tsdf_export_shard (b200tsdf_t* h, void* buf, size_t capacity, size_t* nbytes);
int  b200tsdf_import_shard (b200tsdf_t* h, const void* buf, size_t nbytes);

/* ---- multi-GPU data paths (one process per GPU; DESIGN.md §5).  NCCL is loaded at run time; without it these return
 * B200TSDF_ESTATE.  b200tsdf_comm_unique_id: 128 bytes, created on one rank and handed to the others by any means;
 * b200tsdf_comm_init: collective, binds the handle to a communicator of `nranks` ranks (normally shard_rank / shard_count). */
int  b200tsdf_comm_unique_id (void* id128);
int  b200tsdf_comm_init (b200tsdf_t* h, const void* id128, int rank, int nranks);
/* rows [*row0, *row1) of a `height`-row frame are this rank's slice (ceil(height / nranks) rows per rank) */
int  b200tsdf_row_slice (const b200tsdf_t* h, int height, int* row0, int* row1);
/* n <= 32 consecutive integrateCloud calls where this rank's HOST memory holds only its row slice of every frame
 * (rows[i] -> points (v * width + u), v in the slice; layout as for b200tsdf_integrate).  The slice is uploaded over this
 * GPU's PCIe link, packed to 16-byte pixels and all-gathered over NVLink into the full frame on every rank (collective: all
 * ranks call with the same n), then the batch is fused like b200tsdf_integrate_batch_device.  Without a communicator the
 * slice is the whole frame and nothing is exchanged.  With a single rank the slice is packed on the host first (see
 * b200tsdf_integrate) and rows[i] are free on return; otherwise they must stay valid until b200tsdf_sync or two further calls
 * of this entry point.
 * B200TSDF_EINVAL for n > 32, a NULL row slice or a bad layout: a refused call enqueues nothing and leaves the handle as it
 * was.  n == 0 returns B200TSDF_OK and does nothing. */
int  b200tsdf_integrate_batch_rows (b200tsdf_t* h, int n, const void* const* rows, size_t stride, int xyz_off, int rgba_off,
                                    int width, int height, const double* poses_c2w);
/* Collective: every rank's shard goes device to device (NCCL send/recv over NVLink, no host staging) to rank `root`, which
 * merges them into `full` — a handle on the root's device with shard_count 1 and the same grid, already reset (NULL on the
 * other ranks).  renderView / queries / marching cubes then run on `full` (reads across shards are replicas only). */
int  b200tsdf_gather_volume (b200tsdf_t* h, b200tsdf_t* full, int root);

/* getVoxelCenter / getVoxelIndex (cpp:553-574) */
int  b200tsdf_voxel_center (const b200tsdf_t* h, int64_t x, int64_t y, int64_t z, float* out3);
int  b200tsdf_voxel_index (const b200tsdf_t* h, float x, float y, float z, int32_t* out3, int32_t* inside);

/* ---- leaf enumeration (Octree::getLeaves, octree.cpp:99-109, 608-617), in the reference's depth-first order ----
 * Results are library-owned: valid until the next call of the same entry point or b200tsdf_destroy.  Both return
 * B200TSDF_ESTATE before reset() and on a sharded handle (shard_count > 1: a shard keeps the coarse cells it does not
 * own as unsplit leaves; enumerate on the replica of b200tsdf_gather_volume), B200TSDF_ENOMEM when the output or the
 * sort buffers do not fit.
 * TSDFVolumeOctree::getVoxelCenters (tsdf_volume_octree.cpp:576-588): the centres (OctreeNode::getCenter) of the nodes
 * of getLeaves (nlevels) — nlevels == 0: the root; < 0: every leaf; else every leaf above depth nlevels and every node
 * at depth nlevels.  *xyz = 3 floats per node. */
int  b200tsdf_voxel_centers (b200tsdf_t* h, int nlevels, float** xyz, size_t* n);
/* TSDFVolumeOctree::getOccupiedVoxelIndices (cpp:590-609): getVoxelIndex (cpp:562-574) of the centre of every leaf with
 * w > 0 && |d| < 1.  *ijk = 3 int32 per leaf. */
int  b200tsdf_occupied_voxel_indices (b200tsdf_t* h, int32_t** ijk, size_t* n);
/* TSDFVolumeOctree::isEmpty (tsdf_volume_octree.h:283-287): 1 after reset(), 0 after any integrateCloud, the file's
 * value after b200tsdf_load.  B200TSDF_ESTATE before reset(). */
int  b200tsdf_is_empty (b200tsdf_t* h, int32_t* out);

/* ---- raw node reads: tsdf->octree_->getContainingVoxel (x, y, z, min_size) and the node's accessors ----
 * Octree::getContainingVoxel (octree.cpp:628-634): NaN z, or |coordinate| > size/2 on any axis, gives NULL (level -1, every
 * other field 0).  NaN x or y with a finite z descends with every comparison false, as in the reference.
 * OctreeNode::getContainingVoxel (octree.cpp:112-121): the child is chosen with the strict (x - ctr) > 0 per axis (a point on
 * a splitting plane goes to the lower child); the descent stops at a leaf or at the first node with
 * min_size > 0 && size <= min_size, which may have children.  Nodes with no state of their own (above the root arrays, and
 * the levels above the coarse depth, which Octree::init splits and nothing updates) report the constructor's state. */
typedef struct b200tsdf_voxel
{
  int32_t level;              /* depth of the node, 0 = root; -1 when getContainingVoxel returns NULL (other fields then 0) */
  int32_t x, y, z;            /* node index at its level                                                           */
  float   cx, cy, cz, size;   /* OctreeNode::getCenter / getSize (octree.cpp:52-66)                                */
  float   d, w;               /* OctreeNode::getData (octree.cpp:124-130)                                          */
  uint8_t r, g, b;            /* getRGB: the stored bytes (RGBNode), the RGBNormalized conversion (octree.cpp:396-402),
                                 127,127,127 without colour (OctreeNode::getRGB, octree.cpp:173-178)                */
  uint8_t has_children;       /* OctreeNode::hasChildren (octree.cpp:41-45)                                        */
} b200tsdf_voxel;             /* 44 bytes */

/* n point lookups.  xyz: 3 floats per point, out: n records; host pointers (copied in, b200tsdf_containing_voxels_device,
 * copied out).  B200TSDF_ESTATE before reset() and on a sharded handle (shard_count > 1: read the replica of
 * b200tsdf_gather_volume); n == 0 is a no-op. */
int  b200tsdf_containing_voxels (b200tsdf_t* h, const float* xyz, size_t n, float min_size, b200tsdf_voxel* out);
/* the same on device memory of h's device (d_xyz and d_out 4-byte aligned).  Asynchronous on the handle's stream and ordered
 * after every integrate queued on the handle; errors as for b200tsdf_query_device. */
int  b200tsdf_containing_voxels_device (b200tsdf_t* h, const float* d_xyz, size_t n, float min_size, b200tsdf_voxel* d_out);
/* Dense crop of the finest-voxel box [i0,i1) x [j0,j1) x [k0,k1) (box = {i0, j0, k0, i1, j1, k1}, host memory): entry (i,j,k)
 * is the lookup with min_size = -1 at getVoxelCenter (i, j, k) (tsdf_volume_octree.cpp:553-560), written at offset
 * ((i-i0)*(j1-j0) + (j-j0))*(k1-k0) + (k-k0) (64-bit: a whole 2048^3 box is 8.6 G entries).  d_d, d_w: getData (4-byte
 * aligned floats); d_rgb: getRGB, 3 bytes per entry; d_level: the node's depth.  Any output may be NULL and is then not
 * written; all four NULL is B200TSDF_EINVAL, as is a box without 0 <= lo < hi <= resolution on every axis.  No byte outside
 * the box's extent is written.  Asynchronous, ordered and reported like b200tsdf_containing_voxels_device;
 * B200TSDF_ESTATE before reset() and on a sharded handle. */
int  b200tsdf_dense_device (b200tsdf_t* h, const int32_t box[6], float* d_d, float* d_w, uint8_t* d_rgb, int8_t* d_level);

/* ---- raw node writes: tsdf->octree_->getContainingVoxel (x, y, z, min_size)->setData (d, w) ----
 * For every point i in order, the node is found as by b200tsdf_containing_voxels (Octree::getContainingVoxel,
 * octree.cpp:628-634; OctreeNode::getContainingVoxel, :112-121) and OctreeNode::setData (d[i], w[i]) (:144-150) sets its
 * distance and weight; colour, variance and the RGBNormalized payload are left as they are, as setData leaves them.  setData
 * changes no structure, so when several points reach one node the last of them in batch order wins, as in the sequential
 * loop.  status[i] (optional, one byte per point):
 *   0  written (also when a later point of the batch wrote the same node),
 *   1  no node: getContainingVoxel returns NULL (NaN z, or |coordinate| > size/2),
 *   2  refused: the node lies above the coarse depth (a node of Octree::init that nothing updates; min_size at or above the
 *      coarse cell size reaches these),
 *   3  refused: d[i] or w[i] is not finite.
 * Refused points change nothing: the volume equals the reference's after the loop over the points with status 0.  The call
 * is queued behind every integrate already submitted to the handle and returns once the writes are done; later integrates
 * and reads see them.  A write with |d| > 2^38, w < 0, w = -0, 0 < w < 1e-20 or w > 2^38 moves later integrates to the
 * general kernel (IEEE division) until the next b200tsdf_reset or b200tsdf_load.  On a colour volume a negative weight
 * lets a later colour average (w c + c') / (w + 1) (octree.cpp:328-337) leave [0, 255], or divide by zero at w = -1; the
 * reference's float-to-uint8 cast of such a value is undefined, and the byte the engine stores is the one case outside
 * parity (the parity tests write negative weights on volumes without colour only).  B200TSDF_ESTATE before reset() and on a
 * sharded handle (write the replica of b200tsdf_gather_volume); B200TSDF_EINVAL for NULL xyz, d or w with n > 0, or
 * n > 2^31 - 1; n == 0 does nothing.  Host arrays: copied in, written as by the device entry point, status copied out. */
int  b200tsdf_set_containing_voxels (b200tsdf_t* h, const float* xyz, size_t n, float min_size, const float* d, const float* w,
                                     uint8_t* status);
/* the same on device memory of h's device (d_xyz, d_d and d_w 4-byte aligned, else B200TSDF_EINVAL; d_status may be NULL) */
int  b200tsdf_set_containing_voxels_device (b200tsdf_t* h, const float* d_xyz, size_t n, float min_size, const float* d_d,
                                            const float* d_w, uint8_t* d_status);

/* ---- introspection (tests, bench accounting) ------------------------------------------- */
typedef struct b200tsdf_stats
{
  int64_t n_updates;        /* voxels whose stored {sdf,weight} changed in the last frame (= addObservation calls) */
  int64_t n_node_visits;    /* updateVoxel visits in the last frame */
  int64_t n_culled_cells;   /* coarse cells kept by the frustum cull in the last frame */
  int64_t n_bricks;         /* allocated bricks */
  int64_t n_block_visits;   /* finest-tier bricks processed in the last frame */
  int64_t pool_capacity;
  int32_t coarse_level, finest_level, tiers, reserved;   /* reserved: always 0 */
  double  ms_last_integrate;   /* device time of the last integrate (CUDA events on the handle's stream) */
  double  ms_last_kernel;      /* device time of the dominant (brick update) kernel in the last integrate */
  int64_t n_bail;              /* always 0 (kept for the layout) */
  int64_t n_slow_visits;       /* always 0 (kept for the layout) */
} b200tsdf_stats;
int  b200tsdf_get_stats (b200tsdf_t* h, b200tsdf_stats* s);

/* Measurement hooks for bench.py: CUDA events on the handle's own stream (torch.cuda.Event only
 * sees torch's stream).  profile_begin records the start event and clears the accumulators;
 * profile_end records the end event, synchronizes and reports. */
typedef struct b200tsdf_profile
{
  double  ms_elapsed;        /* start event -> end event on the handle's stream                     */
  double  ms_kernel;         /* sum of the dominant (brick update) kernel's launch durations          */
  int64_t kernel_launches;   /* launches of the dominant kernel                                       */
  int64_t total_launches;    /* all kernel launches of this library in the region                     */
  int64_t n_frames;          /* integrate calls in the region                                         */
  int64_t n_updates;         /* sum over frames of voxels whose {sdf,weight} changed                  */
  int64_t n_node_visits;
  int64_t h2d_bytes, d2h_bytes; /* bytes this library copied across PCIe in the region                */
  double  ms_kernel_device;  /* the same kernel timed on the device (%globaltimer, first block start -> last block end):  */
  int64_t kernel_launches_device; /* also available for frames replayed from a CUDA graph, where no event can be placed   */
  int64_t graph_launches;    /* cudaGraphLaunch calls in the region (b200tsdf_integrate_batch_device)                      */
  int64_t nvlink_bytes;      /* bytes this rank received / sent over NCCL in the region (row all-gather, shard gather)     */
} b200tsdf_profile;
int  b200tsdf_profile_begin (b200tsdf_t* h);
int  b200tsdf_profile_end (b200tsdf_t* h, b200tsdf_profile* out);

/* Every existing octree node at depth >= coarse level, sorted by (level,x,y,z) — the same
 * record the oracle dumps.  Pass all-NULL to get the count.  keys: 4 int32; dw: 2 floats;
 * flags bit0 = has children; rgb 3 bytes; M float; ns int32. */
int64_t b200tsdf_download_nodes (b200tsdf_t* h, int32_t* keys, float* dw, uint8_t* flags,
                                 uint8_t* rgb, float* M, int32_t* ns);
/* RGBNormalized volumes: the four floats {r_n_, g_n_, b_n_, i_} of every node, in the order of b200tsdf_download_nodes
 * (returns the node count, or 0 when the volume does not carry that payload) */
int64_t b200tsdf_download_color_payload (b200tsdf_t* h, float* out4);
/* frustum-culled coarse-cell mask of getFrustumCulledVoxels (cpp:619-652): 8^coarse bytes */
int  b200tsdf_frustum_cull (b200tsdf_t* h, const double* pose_c2w, uint8_t* mask, int32_t* kept);

#ifdef __cplusplus
}
#endif
#endif
