/*
 * dfusion.h -- C ABI of the H100-native DynamicFusion hot path (libdfusion.so).
 *
 * The reference (mihaibujanca/dynamicfusion) has no FFI layer; its seam is the internal launcher layer
 * `kfusion::device::*` declared in kfusion/src/internal.hpp:105-147, called by the host classes
 * cuda::TsdfVolume / cuda::ProjectiveICP / imgproc free functions / WarpField / KinFu.  Every entry point
 * below replaces one of those launchers (cited per function) and is what the C++ mirror classes in
 * include/kfusion/ (and the ctypes binding in dynamicfusion_b200/capi.py) bind.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - 2-D images are (ptr, pitch in BYTES, cols, rows), as kfusion::cuda::PtrStepSz (kernel_containers.hpp:37-63);
 *   - float4 maps hold (x, y, z, w) per pixel: kfusion::Point / Normal (types.hpp:31-42);
 *   - `stream` is a cudaStream_t passed as void* (0 = default stream); calls are asynchronous unless stated;
 *   - return value: 0 on success, otherwise a cudaError_t value (df_error_string() describes it).  The C++
 *     mirror turns a non-zero status into the reference's behaviour (print "KinFu2 error: ..." and exit,
 *     device_memory.cpp:7-11).
 * No torch / C++ types cross this boundary.
 */
#ifndef DFUSION_H
#define DFUSION_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* device::TsdfVolume POD (internal.hpp:29-49).  data: one u32 per voxel, low 16 bits = fp16 TSDF, high 16 bits =
 * u16 weight (ushort2{x,y}); linear index x + y*dims[0] + z*dims[0]*dims[1] (device.hpp:17-27). */
typedef struct df_volume {
    uint32_t *data;
    int dims[3];
    float voxel_size[3];
    float trunc_dist;
    int max_weight;
} df_volume;

/* device::Aff3f (internal.hpp:26-27): R row-major, then t */
typedef struct df_aff3f { float R[9]; float t[3]; } df_aff3f;
/* kfusion::Intr (types.hpp:20-27) */
typedef struct df_intr { float fx, fy, cx, cy; } df_intr;

const char *df_error_string(int status);
int df_version(void);

/* ------------------------------------------------------------------ TSDF volume ---------------------------------------------------------- */
/* device::clear_volume (internal.hpp:105, tsdf_volume.cu:15-41) */
int df_clear_volume(df_volume vol, void *stream);

/* device::compute_dists (internal.hpp:121, imgproc.cu:259-294): u16 mm depth -> fp16 metric ray length */
int df_compute_dists(const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_intr intr,
                     uint16_t *dists, size_t dists_pitch, void *stream);

/* device::integrate (internal.hpp:106, tsdf_volume.cu:51-112,141-161).  vol2cam = camera_pose^-1 * volume_pose
 * (tsdf_volume.cpp:112).  If n_updated (device, u64) is non-NULL the number of voxels written is ADDED to it. */
int df_integrate(df_volume vol, const uint16_t *dists, size_t dists_pitch, int cols, int rows,
                 df_aff3f vol2cam, df_intr intr, unsigned long long *n_updated, void *stream);

/* Activity map (optional accelerator for df_extract_cloud_tracked): one byte per DF_ACTIVITY_VOXELS consecutive voxels of the
 * volume array, non-zero iff an integration stored a voxel with W != 0 && F != 1 there since the map was last zeroed.  Only such
 * voxels can emit a zero crossing (tsdf_volume.cu:548-633), so extraction may skip every other stretch of the volume and still
 * return exactly the full scan's points.  The caller zeroes the map whenever it clears the volume and must route EVERY
 * integration of that volume through df_integrate_tracked. */
#define DF_ACTIVITY_VOXELS 1024
/* Second part of the same allocation (behind the per-stretch bytes, see df_volume_activity_bytes): a BRICK table, one byte per
 * DF_BRICK x DF_BRICK x DF_BRICK block of voxels (brick (bx, by, bz) at ((bz * nby) + by) * nbx + bx, n* = ceil(dims / DF_BRICK)), non-zero iff an
 * integration stored a voxel with F < 0 there since the map was last zeroed.  The ray-cast's march only ever acts on a sample pair that
 * contains a negative value (tsdf_volume.cu:311-336: (-,+) stops the ray, (+,-) is the surface), so df_raycast_points_tracked replays the
 * march's float chain without fetching from bricks that hold no negative voxel and returns exactly the dense march's maps.  The volume
 * itself stays the reference's dense array (TsdfVolume::data()/swap() are part of its API): sparse traversal, not sparse storage. */
#define DF_BRICK 8
size_t df_volume_activity_bytes(df_volume vol);
/* workspace (optional, device memory, df_integrate_workspace_bytes(cols, rows) bytes): per-tile maximum ray length of the frame,
 * used to skip the parts of the volume that lie behind the observed surface; NULL = allocated stream-ordered per call. */
size_t df_integrate_workspace_bytes(int cols, int rows);
int df_integrate_launch_count(df_volume vol);   /* kernels one integrate call launches for this volume (bookkeeping for gpu_launches) */
int df_integrate_last_kernel(void);             /* diagnostic: which integrate kernel the last call of this process launched (5 = packed-arithmetic kernel, 3 / 4 = scalar culling kernels, 0 = plain) */
int df_integrate_selftest(unsigned long long *mismatch_dev4, void *stream);   /* test hook: the packed integrate kernel's division / square-root sequences against the '/' operator and sqrtf() on this device; 4 mismatch counters (all 0 on a conforming device) */
int df_integrate_tracked(df_volume vol, const uint16_t *dists, size_t dists_pitch, int cols, int rows,
                         df_aff3f vol2cam, df_intr intr, unsigned long long *n_updated, unsigned char *activity, void *workspace,
                         void *stream);

/* device::raycast, points variant (internal.hpp:113-114, tsdf_volume.cu:341-405,459-474).
 * cam2vol = volume_pose^-1 * camera_pose, Rinv = cam2vol.R^-1 (tsdf_volume.cpp:157-174). */
int df_raycast_points(df_volume vol, df_aff3f cam2vol, const float *Rinv_host9, df_intr intr, int cols, int rows,
                      float step_factor, float delta_factor,
                      float *points, size_t points_pitch, float *normals, size_t normals_pitch, void *stream);

/* same maps, bit for bit; the march skips the bricks that hold no negative voxel (activity: the volume's activity map, maintained by
 * df_integrate_tracked / df_integrate_warped -- NULL falls back to df_raycast_points) */
int df_raycast_points_tracked(df_volume vol, df_aff3f cam2vol, const float *Rinv_host9, df_intr intr, int cols, int rows,
                              float step_factor, float delta_factor, float *points, size_t points_pitch, float *normals, size_t normals_pitch,
                              const unsigned char *activity, void *stream);

/* Measurement variant of df_raycast_points (bench.py's ray-cast roofline; never on the frame path): the same kernel instantiated with
 * counters.  touched: df_raycast_touched_bytes(vol) bytes, zeroed by the caller, one bit per voxel the launch reads (its popcount is U of
 * SURVEY.md 8d: algorithmic bytes = 4*U + 32*cols*rows); stats (device, 2 x u64, zeroed by the caller): [0] rays that produced a vertex,
 * [1] march samples fetched after the entry sample. */
size_t df_raycast_touched_bytes(df_volume vol);
int df_raycast_points_stats(df_volume vol, df_aff3f cam2vol, const float *Rinv_host9, df_intr intr, int cols, int rows,
                            float step_factor, float delta_factor, float *points, size_t points_pitch,
                            float *normals, size_t normals_pitch, unsigned int *touched, unsigned long long *stats, void *stream);

/* the counting instantiation of df_raycast_points_tracked (activity != NULL: [1] counts the march samples EXAMINED; only those in
 * negative bricks are fetched and appear in `touched`) */
int df_raycast_points_stats_tracked(df_volume vol, df_aff3f cam2vol, const float *Rinv_host9, df_intr intr, int cols, int rows,
                                    float step_factor, float delta_factor, float *points, size_t points_pitch,
                                    float *normals, size_t normals_pitch, unsigned int *touched, unsigned long long *stats,
                                    const unsigned char *activity, void *stream);

/* device::project_and_remove (internal.hpp:108-109, tsdf_volume.cu:114-137,164-177): `dists` is sampled as fp16 and
 * the pixels the vertices land on are zeroed; vertices become (u*Dp, v*Dp, Dp, 0) or NaN when off-image.
 * Deterministic (the reference races the scatter with the sampling): samples always see the original image.
 * workspace: df_project_workspace_bytes(cols, rows) bytes, zero on entry, returned zeroed. */
size_t df_project_workspace_bytes(int cols, int rows);
int df_project_and_remove(uint16_t *dists, size_t dists_pitch, int cols, int rows, df_intr intr,
                          float *points, size_t points_pitch, int pcols, int prows, void *workspace, void *stream);

/* device::extractCloud (internal.hpp:138, tsdf_volume.cu:486-710,799-815).  Deterministic: points are emitted in
 * ascending (z, y, x) voxel order, +x,+y,+z edge within a voxel.  `workspace` needs df_extract_workspace_bytes();
 * the point count (clamped to capacity) is written to *count (device, int32) -- no host sync. */
size_t df_extract_workspace_bytes(df_volume vol);
int df_extract_cloud(df_volume vol, df_aff3f pose, float *out_points, int capacity, int *count,
                     void *workspace, void *stream);
/* same, skipping the stretches of the volume whose activity byte is zero (activity == NULL: full scan) */
int df_extract_cloud_tracked(df_volume vol, df_aff3f pose, float *out_points, int capacity, int *count, void *workspace,
                             const unsigned char *activity, void *stream);

/* device::extractNormals (internal.hpp:139, tsdf_volume.cu:714-795,817-831).  n_points may be given on the host
 * (count_dev == NULL) or read from device memory (count_dev != NULL, upper bound n_points). */
int df_extract_normals(df_volume vol, const float *points, int n_points, const int *count_dev, df_aff3f pose,
                       const float *Rinv_host9, float delta_factor, float *out_normals, void *stream);

/* Brick packing of a volume (snapshots; csrc/snapshot.cu).  The volume is cut into the DF_BRICK^3 bricks of the brick table (brick (bx, by, bz)
 * at ((bz * nby) + by) * nbx + bx; edge bricks hold only their in-volume voxels).  Each brick is one class byte:
 *   0 empty    every voxel is 0 (what df_clear_volume writes): no payload;
 *   1 uniform  every voxel holds the same non-zero word (free space): that word;
 *   2 mixed    anything else: its 512 words in (z, y, x) order inside the brick, slots outside the volume written as 0 and ignored on load.
 * The payload is the bricks' words in brick order.  It holds no offsets or indices, so nothing in it can point outside the volume; its
 * length is 4 * (n_uniform + 512 * n_mixed) bytes -- at most about 4 * V (every brick mixed), the only staging a pack or an unpack needs
 * besides the class bytes and the workspace.  The bytes are deterministic for a given volume.  Requirements: dims[0] % 32 == 0, fewer than
 * 2^31 voxels, data 16-byte aligned.
 *   df_volume_brick_count        class bytes of the volume (device buffer `classes`);
 *   df_volume_pack_workspace_bytes  device workspace of all three calls (block counts and their scan: about V / 1024 bytes);
 *   df_volume_pack_count         reads the volume once, writes the class bytes and *payload_bytes (device u64);
 *   df_volume_pack_emit          after _count with the same workspace and an unchanged volume: writes the payload, never at or past
 *                                `capacity` bytes;
 *   df_volume_unpack             checks on the device that every class byte is in {0, 1, 2} and that payload_bytes equals the length the
 *                                classes imply, writes *status (device int: 0, DF_UNPACK_BAD_CLASS or DF_UNPACK_BAD_LENGTH) and, only
 *                                when it is 0, writes EVERY voxel of the volume (no clear needed; the result does not depend on what the
 *                                volume held).  A failed check leaves the volume untouched.  payload must be 4-byte aligned. */
#define DF_UNPACK_BAD_CLASS 1
#define DF_UNPACK_BAD_LENGTH 2
size_t df_volume_brick_count(df_volume vol);
size_t df_volume_pack_workspace_bytes(df_volume vol);
int df_volume_pack_count(df_volume vol, void *workspace, unsigned char *classes, unsigned long long *payload_bytes, void *stream);
int df_volume_pack_emit(df_volume vol, const void *workspace, const unsigned char *classes, uint32_t *payload, size_t capacity, void *stream);
int df_volume_unpack(df_volume vol, const unsigned char *classes, const uint32_t *payload, size_t payload_bytes, void *workspace, int *status,
                     void *stream);

/* Triangle mesh over the extracted cloud (csrc/mesh.cu).  The mesh's vertex buffer IS the cloud of df_extract_cloud(_tracked) for the same
 * volume; the triangles are int32 index triples into it.  The pose does not enter: indices do not depend on it.
 *   Rule.  The cube at voxel (x, y, z) is the 8 voxels (x..x+1, y..y+1, z..z+1).  It is polygonised iff
 *     x <= Dx-2, y <= Dy-2 and z <= Dz-3 (the cloud has no crossing owned by a voxel of the last z slice, so a cube at z = Dz-2 would
 *     need points that do not exist on its top face), every corner is active (W != 0 and F != +1) and every corner has F < 0 or F > 0
 *     (the cloud's sign test is strict: an edge that touches an exact zero, or a NaN, has no point).
 *   Inside means F < 0.  Then every edge of the cube that changes sign owns exactly one cloud point (the one its lower voxel emits on that
 *   axis) and the triangles of the cube's case (include/df_mc_table.h, the marching-cubes table with corner/edge numbering and case bits
 *   as described there) use exactly those points.  Triangles come out in ascending cube order (z, y, x), within a cube in table order, and
 *   wind counter-clockwise seen from the free-space (F > 0) side: the right-hand face normal points the way df_extract_normals' do.
 *   Two cubes that share a face draw the same segments on it, so the mesh has no cracks between polygonised cubes.
 * workspace: df_mesh_workspace_bytes(vol) bytes of device memory for THIS volume (dims and data alignment pick the 4-voxel or the 1-voxel
 * path, as the extraction does): one int per 4 voxels (1 per voxel on the 1-voxel path) plus the block scans.
 *   df_mesh_count  counts the triangles into *tri_count_dev (device int) and recounts the cloud's points.  *status_dev (device int) is 0, or
 *                  DF_MESH_CLOUD_MISMATCH when that recount differs from *cloud_count_dev: the cloud was truncated at its capacity or was
 *                  not extracted from the volume as it is now.  activity: the volume's activity map (df_integrate_tracked), or NULL.
 *   df_mesh_emit   after df_mesh_count with the same workspace and an unchanged volume: writes the triangles (int32 x 3 each), never at or
 *                  past `capacity` triangles.  Its result is meaningful only when the status was 0. */
#define DF_MESH_CLOUD_MISMATCH 1
size_t df_mesh_workspace_bytes(df_volume vol);
int df_mesh_count(df_volume vol, const unsigned char *activity, const int *cloud_count_dev, void *workspace, int *tri_count_dev,
                  int *status_dev, void *stream);
int df_mesh_emit(df_volume vol, const unsigned char *activity, const void *workspace, int32_t *tris, int capacity, void *stream);

/* Z-buffer rasteriser of a triangle mesh into the ray-cast's maps (csrc/raster.cu): camera-frame points and normals (float4, four NaNs where
 * nothing is drawn, so df_render_image / df_render_tangent_colors shade them unchanged) and, optionally, the index of the triangle each
 * pixel shows (-1 where nothing is drawn).  The result is a function of the inputs alone, independent of launch and thread order.
 *   Rule (tests/raster_oracle.c implements it operation for operation and agrees bit for bit; float operations are IEEE round-to-nearest
 *   without contraction, fma only where written):
 *   Camera frame  c = world2cam * v, each component r.x*x + r.y*y + r.z*z + t evaluated left to right.
 *   Skipped       (stats[1]) a triangle with an index outside [0, n_verts), or a vertex whose c is not finite, has c.z < DF_RASTER_NEAR,
 *                 or whose snapped position lies outside the guard band.  Triangles are not clipped.
 *   Projection    u = fma(fx, c.x / c.z, cx), v = fma(fy, c.y / c.z, cy) (the Projector); U = u * 256, V = v * 256 (8 sub-pixel bits)
 *                 must satisfy |U|, |V| <= 2^24 (the guard band, +-2^16 pixels) and are rounded to the nearest integer, ties to even.
 *   Facing        A = (U1-U0)(V2-V0) - (V1-V0)(U2-U0) in int64.  The mesh winds counter-clockwise seen from free space and v points down,
 *                 so a triangle facing the camera has A < 0; A >= 0 (back-facing or zero area) draws nothing (stats[0]).
 *   Coverage      pixel (i, j) samples at exactly (i, j), fixed point (256 i, 256 j).  With the vertices taken as (0, 2, 1) (positive area),
 *                 edge k runs from vertex k to k+1 with (dx, dy) = end - start, E_k = dx * (256 j - start.V) - dy * (256 i - start.U)
 *                 in int64; the sample is covered iff every E_k > 0, or E_k == 0 on a top or left edge (dy < 0, or dy == 0 and dx > 0).
 *                 Two triangles sharing an edge traverse it in opposite directions, so a closed surface covers every sample exactly once.
 *   Depth         d = ((i - cx) * (1/fx), (j - cy) * (1/fy), 1) (the ray-cast's Reprojector), n = cross(c1 - c0, c2 - c0) in the mesh's
 *                 order, t = dot(n, c0) / dot(n, d); only 0 < t < inf is drawn.
 *   Z-test        key = (bits of t) << 32 | triangle index, the minimum over all drawn triangles per pixel: the nearest surface, and on a
 *                 tie the smaller index.
 *   Output        points = (d.x * t, d.y * t, t, 0), normals = (n / sqrt(dot(n, n)), 0) (pointing to free space, as the ray-cast's do),
 *                 tri_ids = the index.
 *   stats_dev (optional, device, 5 x u64, overwritten): [0] back-facing or zero area, [1] skipped, [2] drawn by the small-triangle path
 *   (clipped bounding box of at most 8 x 8 samples), [3] drawn by the large-triangle path, [4] pixels written.
 * verts: device, n_verts points of vstride (3 or 4) floats; tris: device, n_tris x 3 int32.  cols, rows <= DF_RASTER_MAX_DIM.  Pitches in
 * bytes: points and normals at least cols * 16 and a multiple of 16, tri_ids at least cols * 4 and a multiple of 4 (else
 * cudaErrorInvalidValue, nothing written).  workspace:
 * df_raster_workspace_bytes(n_verts, n_tris, cols, rows) bytes of device memory (a 64-bit key per pixel, 24 bytes per vertex, 4 per triangle). */
#define DF_RASTER_NEAR 0.01f
#define DF_RASTER_MAX_DIM 32768
size_t df_raster_workspace_bytes(int n_verts, int n_tris, int cols, int rows);
int df_raster_mesh(const float *verts, int n_verts, int vstride, const int32_t *tris, int n_tris, df_aff3f world2cam, df_intr intr, int cols,
                   int rows, int32_t *tri_ids, size_t tri_pitch, float *points, size_t points_pitch, float *normals, size_t normals_pitch,
                   unsigned long long *stats_dev, void *workspace, void *stream);

/* Per-pixel correspondences on a second vertex set with the same faces (csrc/raster.cu): for a df_raster_mesh view of a mesh (tri_ids and
 * the drawn points of that call, and its verts / vstride / tris / world2cam), the point of the SOURCE mesh (src_verts: same count, stride and
 * triangles as verts) at the same barycentric position on the drawn triangle, and that source triangle's face normal.  The frame loop uses
 * it to pair each pixel of the rendered live model with the canonical surface drawn there (DF_KINFU_LIVE_MODEL).
 *   Rule (tests/correspond_oracle.c implements it operation for operation; IEEE round-to-nearest, no contraction, evaluated as written):
 *   c0, c1, c2    the drawn triangle's corners in the camera frame, computed as df_raster_mesh's Camera frame rule; s0, s1, s2 its source
 *                 corners (xyz of src_verts).
 *   P             the drawn point (xyz).  e0 = c1 - c0, e1 = c2 - c0, q = P - c0; d00 = dot(e0, e0), d01 = dot(e0, e1), d11 = dot(e1, e1),
 *                 d20 = dot(q, e0), d21 = dot(q, e1) (dot = x*x' + y*y' + z*z' left to right); den = d00 * d11 - d01 * d01;
 *                 b1 = (d11 * d20 - d01 * d21) / den, b2 = (d00 * d21 - d01 * d20) / den, b0 = (1 - b1) - b2.
 *   Output        src_points = ((b0 * s0 + b1 * s1) + b2 * s2, 0) per component; src_normals = (n / sqrt(dot(n, n)), 0) with
 *                 n = cross(s1 - s0, s2 - s0) in the mesh's order (pointing to free space, like df_raster_mesh's normals).
 *   No correspondence (four NaNs in both maps): tri id < 0 (or not below n_tris, or a corner index outside [0, n_verts)); den not finite or
 *                 zero; a target map is given (float4 vertex map, e.g. the frame's) and its vertex at the pixel has a NaN component, or
 *                 (T - P) has dx*dx + dy*dy + dz*dz > max_dist * max_dist.
 * target may be NULL (no gate).  cols, rows <= DF_RASTER_MAX_DIM.  Pitches in bytes: points, target, src_points and src_normals at least
 * cols * 16 and a multiple of 16, tri_ids at least cols * 4 and a multiple of 4 (else cudaErrorInvalidValue, nothing written).  One thread per
 * pixel, one launch. */
int df_mesh_correspond(const int32_t *tri_ids, size_t tri_pitch, const float *points, size_t points_pitch, const float *verts,
                       const float *src_verts, int n_verts, int vstride, const int32_t *tris, int n_tris, df_aff3f world2cam, int cols, int rows,
                       const float *target, size_t target_pitch, float max_dist, float *src_points, size_t src_points_pitch, float *src_normals,
                       size_t src_normals_pitch, void *stream);

/* Colours of a df_raster_mesh view (csrc/raster.cu): every drawn pixel gets the barycentric mix of its triangle's three vertex colours.
 *   Rule (tests/color_oracle.c implements it operation for operation; IEEE round-to-nearest, no contraction, evaluated as written):
 *   b0, b1, b2    df_mesh_correspond's weights for the pixel (its c0..c2, P, den rule, computed by the same device function).
 *   Vertex k      colour word vert_rgba[index k]: bytes R, G, B, A in memory order; it takes part iff A != 0.
 *   Mix           sw = 0, s_c = 0; for k = 0, 1, 2 in order, if vertex k takes part: sw = sw + b_k, s_c = s_c + b_k * (float)channel_c.
 *                 Drawn iff sw > 0; channel = min(max(rint(s_c / sw), 0), 255) (round to nearest, ties to even).
 *   Output        image pixel bytes B, G, R, 0 (df_render_image's layout); four zero bytes when the tri id is < 0 or not below n_tris, a
 *                 corner index lies outside [0, n_verts), den is not finite or zero, or no vertex takes part (sw > 0 fails).
 * vert_rgba: device, n_verts words (df_sample_colors' output).  Pitches in bytes: points at least cols * 16 and a multiple of 16, tri_ids and
 * image at least cols * 4 and a multiple of 4 (else cudaErrorInvalidValue, nothing written).  One thread per pixel, one launch. */
int df_mesh_colors(const int32_t *tri_ids, size_t tri_pitch, const float *points, size_t points_pitch, const float *verts, int n_verts,
                   int vstride, const int32_t *tris, int n_tris, df_aff3f world2cam, const uint32_t *vert_rgba, int cols, int rows,
                   void *image_bgra, size_t image_pitch, void *stream);

/* ------------------------------------------------------------------ colour volume --------------------------------------------------------- */
/* An optional second volume next to a df_volume (csrc/color.cu): one u32 per voxel, indexed like df_volume.data, bytes R, G, B, W in memory
 * order (the word is R | G << 8 | B << 16 | W << 24); W = samples averaged so far, 0 = never coloured.  All zero means "no colour", so
 * df_clear_volume and df_volume_pack_* / df_volume_unpack work on it through a df_volume whose data points at it.  The TSDF volume itself is
 * never read by these calls: the df_volume argument supplies dims, voxel_size, trunc_dist and max_weight.
 *
 * df_integrate_color: fuse one registered colour image into the colour volume, next to the surface the frame's depth shows.
 *   Rule (tests/color_oracle.c implements it operation for operation and agrees bit for bit; IEEE round-to-nearest, fma only where written):
 *   Visited       voxel index i = x + Dx * (y + Dy * z), every voxel whose stretch i / DF_ACTIVITY_VOXELS has a non-zero activity byte
 *                 (activity == NULL: every voxel).  Pass the activity map the frame's df_integrate_tracked has just updated: a voxel near
 *                 the surface the frame shows lies in a marked stretch, because that integrate stored an active voxel there.
 *   Position      p = ((float)x * vs_x, (float)y * vs_y, (float)z * vs_z); vc_c = fma(r_c.x, p.x, fma(r_c.y, p.y, r_c.z * p.z)) + t_c for
 *                 the rows r_c and translation t of vol2cam (closed form per voxel: df_integrate's serial z-chain is NOT replayed, so
 *                 vc may differ from that kernel's in the last bit).
 *   Projection    u = fma(fx, vc.x / vc.z, cx), v = fma(fy, vc.y / vc.z, cy) (the Projector); the pixel is ((int)u, (int)v).
 *   Skipped, in this order: u < 0 or v < 0 or u >= cols or v >= rows; vc.z <= 0; u or v NaN; Dp == 0, Dp = dists(pixel) as fp16;
 *                 then with sdf = Dp - sqrt(fma(vc.x, vc.x, fma(vc.y, vc.y, vc.z * vc.z))): not (|sdf| <= DF_COLOR_BAND * trunc_dist)
 *                 (one float product).  The band is narrower than the TSDF's, so that colour is only taken next to the surface.
 *   Update        per channel c with sample s (image pixel bytes B, G, R, x -> s_R = byte 2, s_G = byte 1, s_B = byte 0), in integers:
 *                 c' = (c * W + s + ((W + 1) >> 1)) / (W + 1) (truncating division), W' = min(W + 1, min(max_weight, 255)).
 *   One thread owns a voxel (no atomics), so the result does not depend on launch or thread order.
 * dists: the fp16 ray lengths the frame's integrate read (df_compute_dists), pitch in bytes; bgra: device, 4 bytes per pixel, pitch at
 * least cols * 4 and a multiple of 4.  One launch. */
#define DF_COLOR_BAND 0.5f
int df_integrate_color(df_volume vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, const void *bgra, size_t bgra_pitch,
                       int cols, int rows, df_aff3f vol2cam, df_intr intr, const unsigned char *activity, void *stream);

/* Lens distortion of a calibrated camera (OpenCV's coefficient order): the 5-coefficient Brown-Conrady model (k1, k2, p1, p2, k3; k4..k6 =
 * 0) or the 8-coefficient rational model; unused coefficients are 0.  r2_max is the squared normalised radius over which the calibration
 * holds: polynomial models fold back beyond some radius, and without a bound a point far off-axis (a voxel beside the camera) could land
 * inside the image.  36 bytes, no padding.
 *   Rule (csrc/lens.cuh holds the one device statement; tests/lens_oracle.c restates it; IEEE round-to-nearest, no contraction, evaluated
 *   left to right as written).  The forward distortion of the normalised point (x, y):
 *                 r2 = x*x + y*y; invalid unless r2 <= r2_max (a NaN is invalid);
 *                 radial = (1 + r2*(k1 + r2*(k2 + r2*k3))) / (1 + r2*(k4 + r2*(k5 + r2*k6)));
 *                 xd = x*radial + (2*p1*x*y + p2*(r2 + 2*x*x));  yd = y*radial + (p1*(r2 + 2*y*y) + 2*p2*x*y).
 *   Only the forward direction is used: every use goes from an ideal ray to a raw pixel, so nothing is inverted on the device.
 * df_lens_check (host only): 0, or cudaErrorInvalidValue when a value is not finite, r2_max is not > 0, the denominator is not > 0 on
 *   [0, r2_max], or r -> r * radial(r*r) is not strictly increasing on [0, sqrt(r2_max)] (both checked in double at 4097 radii
 *   sqrt(r2_max) * i / 4096).  All eight coefficients 0 (with any valid r2_max) is the "no lens" value. */
typedef struct df_lens { float k1, k2, p1, p2, k3, k4, k5, k6, r2_max; } df_lens;
int df_lens_check(df_lens lens);

/* df_undistort: a raw depth frame (and optionally its registered BGRA image) of a camera with `lens` -> the ideal pinhole images of the same
 * intrinsics and size, which is what every other entry point here takes.  One thread per output pixel, one launch for both images.
 *   Rule (tests/lens_oracle.c; the distortion above):  output pixel (i, j): x = ((float)i - cx) * finv_x, y = ((float)j - cy) * finv_y with
 *                 finv = 1.f / f (df_points_normals' reprojection); distort (x, y); u = fma(fx, xd, cx), v = fma(fy, yd, cy);
 *                 su = floorf(u + 0.5f), sv = floorf(v + 0.5f).  The output is the input at (su, sv) (nearest neighbour: interpolating
 *                 depth across an edge invents flying points, and the bilateral filter does the smoothing), or 0 -- four zero bytes in
 *                 bgra_out -- when the point is invalid or not (0 <= su < cols and 0 <= sv < rows) (a NaN fails).  The BGRA image takes
 *                 the same source pixel, so colour stays registered to depth.  A lens whose eight coefficients are all 0 is the identity
 *                 whatever its r2_max: the output is a copy of the input, bit for bit.
 * depth / depth_out: device u16, pitch in bytes; bgra / bgra_out: device, 4 bytes per pixel, both NULL or both set.  Every pitch holds a
 * whole row and is a multiple of the element size, the inputs and outputs do not overlap, and df_lens_check passes; otherwise
 * cudaErrorInvalidValue and nothing is written. */
int df_undistort(const uint16_t *depth, size_t depth_pitch, uint16_t *depth_out, size_t out_pitch, const void *bgra, size_t bgra_pitch,
                 void *bgra_out, size_t bgra_out_pitch, int cols, int rows, df_intr intr, df_lens lens, void *stream);

/* A colour camera with its own calibration: RGB-D sensors put the colour camera a few centimetres beside the depth camera, with its own
 * intrinsics and image size (Kinect v1: two 640 x 480 cameras 2.5 cm apart; Kinect v2 class: 512 x 424 depth, 1920 x 1080 colour, 5 cm).
 * Its lens distortion is a separate df_lens (the _lens entries below); no time offset between the two sensors is modelled.  72 bytes, no
 * padding. */
typedef struct df_color_camera {
    int cols, rows;              /* colour image size, 1..16384 each */
    df_intr intr;                /* colour intrinsics: fx, fy > 0; all four finite */
    df_aff3f depth_to_color;     /* a point in the depth camera's frame -> the same point in the colour camera's frame (finite) */
} df_color_camera;

/* df_color_depth_map: the occlusion map of a depth frame as the colour camera sees it -- a z-buffer of the frame's depth pixels, coarsened
 * to cells of cell x cell colour pixels so that adjacent depth pixels at equal depth land in the same or adjacent cells.
 *   Cells         cell = max(1, (int)ceilf(fmaxf(cam.fx / fx, cam.fy / fy))) (fx, fy: the depth intrinsics); the map is
 *                 ceil(cam.cols / cell) x ceil(cam.rows / cell) u32 words.  df_color_map_dims computes the three numbers (host only;
 *                 cudaErrorInvalidValue for an invalid camera or depth intrinsics: non-finite values, fx or fy not > 0, a size outside 1..16384).
 *   Rule (tests/color_camera_oracle.c implements it operation for operation; IEEE round-to-nearest, fma only where written):
 *                 every word is first set to 0xffffffff (empty).  Then for each depth pixel (i, j) with d = depth(i, j) != 0:
 *                 z = (float)d * 0.001f; p = (z * ((float)i - cx) * finv_x, z * ((float)j - cy) * finv_y, z) with finv = 1.f / f (left
 *                 to right, as df_points_normals reprojects); pc_c = fma(r_c.x, p.x, fma(r_c.y, p.y, r_c.z * p.z)) + t_c for the rows r_c
 *                 and translation t of depth_to_color; uc = fma(cam.fx, pc.x / pc.z, cam.cx), vc = fma(cam.fy, pc.y / pc.z, cam.cy).
 *                 Skipped unless pc.z > 0 and 0 <= uc < cam.cols and 0 <= vc < cam.rows (a NaN is skipped); else
 *                 map[(int)vc / cell][(int)uc / cell] = min(word, bits of pc.z) (atomicMin: positive floats order as their bit patterns,
 *                 so the map does not depend on thread order).
 * depth: device u16 mm, pitch in bytes; map: device, pitch in bytes (at least map_cols * 4, a multiple of 4).  One memset, one kernel. */
int df_color_map_dims(df_intr intr, df_color_camera cam, int *map_cols, int *map_rows, int *cell);
int df_color_depth_map(const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_intr intr, df_color_camera cam, uint32_t *map,
                       size_t map_pitch, void *stream);

/* df_integrate_color_camera: df_integrate_color for a colour image taken by `cam`.
 *   Rule (tests/color_camera_oracle.c): the voxels visited, their position vc, the depth projection and the depth-side skips (in the same
 *                 order, against the depth frame's dists and DF_COLOR_BAND) are df_integrate_color's.  Then:
 *   Colour pixel  pc = depth_to_color * vc (fma chain as above), uc = fma(cam.fx, pc.x / pc.z, cam.cx), vc' = fma(cam.fy, pc.y / pc.z, cam.cy);
 *                 skipped unless pc.z > 0 and 0 <= uc < cam.cols and 0 <= vc' < cam.rows (a NaN is skipped).
 *   Occlusion     zmin = the word of map cell ((int)vc' / cell, (int)uc / cell) (df_color_depth_map of the same frame); skipped if the cell is
 *                 empty (0xffffffff) or pc.z > zmin + DF_COLOR_OCCLUSION * trunc_dist (the product is one float, then one float sum): the
 *                 colour camera sees a nearer surface there, so its pixel does not show this voxel.
 *   Update        with the sample bgra[(int)vc'][(int)uc], df_integrate_color's integer running average.
 *   One thread owns a voxel (no atomics).  bgra: device, cam.cols x cam.rows pixels, pitch at least cam.cols * 4 and a multiple of 4; map as
 * df_color_depth_map writes it.  One launch. */
#define DF_COLOR_OCCLUSION 1.0f
int df_integrate_color_camera(df_volume vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, int cols, int rows, df_aff3f vol2cam,
                              df_intr intr, df_color_camera cam, const void *bgra, size_t bgra_pitch, const uint32_t *map, size_t map_pitch,
                              const unsigned char *activity, void *stream);

/* df_sample_colors: the colour of the volume at arbitrary points, as R, G, B, A words (A = 255 where coloured, else the word is 0).
 *   Rule (tests/color_oracle.c; IEEE round-to-nearest, no contraction, evaluated as written):
 *   Grid coordinate  q = vol_pose^-1 * p with the inverse formed by df_hostmath.h's dfh_aff_inv and each component
 *                 r.x*x + r.y*y + r.z*z + t left to right; g_c = q_c / vs_c - offset.  offset = 0 for points in the convention of
 *                 df_integrate and the ray-cast (voxel i at i * vs); offset = 0.5 for points of df_extract_cloud, which puts voxel i at
 *                 (i + 1/2) * vs.  Forgetting it shifts every texture by half a voxel.
 *   Outside       a NaN component of p, or not (0 <= g_c < D_c - 1) on some axis: the word 0.
 *   Corners       i_c = floor(g_c), f_c = g_c - i_c; corner k = 0..7 is voxel (i_x + (k & 1), i_y + ((k >> 1) & 1), i_z + (k >> 2)) with
 *                 weight w_k = (wx * wy) * wz, w = 1 - f for a clear bit and f for a set bit.
 *   Mix           sw = 0, s_c = 0; for k = 0..7 in order, if corner k has W != 0: sw = sw + w_k, s_c = s_c + w_k * (float)channel_c.
 *                 Coloured iff sw > 0: channel = min(rint(s_c / sw), 255) (ties to even), A = 255.  Corners never coloured are left out and
 *                 the rest renormalised; no coloured corner with a positive weight gives the word 0.
 * points: device, a rows x cols image of points; point (i, j) is the 3 floats at byte j * points_pitch + i * stride * 4 (stride 3 or 4).  A
 * list of n points is cols = n, rows = 1; then count_dev (optional, device int) bounds the points read and written (min(*count_dev, cols)).
 * rgba: device, word (i, j) at byte j * rgba_pitch + i * 4.  rows <= 65535; pitches are multiples of 4 (else cudaErrorInvalidValue, nothing
 * written).  One kernel, one launch, for the cloud, a ray-cast vertex map or any point set. */
int df_sample_colors(df_volume vol, const uint32_t *colors, df_aff3f vol_pose, float offset, const float *points, size_t points_pitch,
                     int stride, int cols, int rows, const int *count_dev, uint32_t *rgba, size_t rgba_pitch, void *stream);

/* ---- colour tracking (DF_KINFU_COLOR_TRACKING): intensity maps of the frame and of the model, and the photometric ICP rows -------------
 * Rules (tests/color_track_oracle.c implements them operation for operation and agrees bit for bit; IEEE round-to-nearest, no contraction,
 * evaluated as written):
 *   Intensity     of bytes R, G, B: Y = (77 * R + 150 * G + 29 * B + 128) >> 8 in integers, I = (float)Y / 255.f.  A BGRA pixel has
 *                 B = byte 0, G = byte 1, R = byte 2; a colour-volume word has R = bits 0..7, G = 8..15, B = 16..23.
 *
 * df_frame_intensity: the frame's intensity pyramid, one float per pixel, NaN = no value.  Level l has the size of the depth pyramid's
 * level l (cols[l] x rows[l], each level half the one before, rounded down).
 *   Level 0, registered image (cam == NULL): the intensity of bgra pixel (x, y); bgra is cols[0] x rows[0].
 *   Level 0, colour camera (cam != NULL): p = xyz of the level-0 vertex map at (x, y) (df_points_normals of the frame); NaN in p.x: NaN.
 *                 pc = depth_to_color * p, uc, vc' and their test as df_color_depth_map computes them (outside the colour image: NaN); then
 *                 the occlusion test of df_integrate_color_camera against map (df_color_depth_map of the same frame): an empty cell, or
 *                 pc.z > zmin + DF_COLOR_OCCLUSION * trunc_dist, gives NaN.  Else the intensity of bgra pixel ((int)uc, (int)vc').  The
 *                 device code is that of the colour-camera fusion (the same functions), so a pixel passes exactly where a voxel at p would.
 *   Level l > 0:  the mean of the non-NaN values among level l-1's (2x + dx, 2y + dy), taken in the order (0,0), (1,0), (0,1), (1,1):
 *                 s = 0; n = 0; s = s + value; n = n + 1 for each; s / (float)n, or NaN when n = 0.
 *   One launch per level.  intensity[l]: device, pitch[l] bytes per row (at least cols[l] * 4, a multiple of 4).  bgra pitch at least
 *   its width * 4 and a multiple of 4; points pitch a multiple of 16; map as df_color_depth_map writes it (ignored without a camera).
 *
 * df_model_intensity: the model's intensity and its image gradient at every pixel of a camera-frame vertex map pyramid.  One launch for
 * all levels.
 *   Sample        I(x, y): p = xyz of points[l] at (x, y); the word c = df_sample_colors' rule at p with the volume transform q = cam2vol * p
 *                 (each component r.x*x + r.y*y + r.z*z + t left to right) and offset 0 -- the ray-cast's convention, voxel i at i * vs,
 *                 which is what the frame loop's vertex maps are in.  I = the intensity of c, or NaN where c = 0 (no colour, outside the
 *                 volume, or a NaN point).
 *   Gradient      gu = (I(x+1, y) - I(x-1, y)) * 0.5f, gv = (I(x, y+1) - I(x, y-1)) * 0.5f; NaN on the border of the level or where any of
 *                 the five values is NaN.
 *   Output        maps[l] at (x, y) = (I, gu, gv, 0) as float4, or four NaNs where any of I, gu, gv is NaN.  cam2vol = volume_pose^-1 *
 *                 camera_pose (the ray-cast's).  maps[l] pitch: at least cols[l] * 16, a multiple of 16; points[l] likewise.
 *
 * Photometric ICP row (df_icp_accumulate_color): at a pixel (x, y) whose geometric row exists (every test of df_icp_accumulate passed, with
 * s = T * v_curr and its projection (u, v) into the previous frame as that rule forms them):
 *   Current       I_c = icurr(x, y); none when NaN.
 *   Model         i0 = (int)floorf(u), j0 = (int)floorf(v), a = u - floorf(u), b = v - floorf(v); the four samples m00 = model(i0, j0),
 *                 m10 = (i0 + 1, j0), m01 = (i0, j0 + 1), m11 = (i0 + 1, j0 + 1) (sample i sits at coordinate i, as the projection puts
 *                 pixel centres); none when i0 + 1 >= cols or j0 + 1 >= rows or a sample is NaN.  Per component
 *                 val = (m00 * (1.f - a) + m10 * a) * (1.f - b) + (m01 * (1.f - a) + m11 * a) * b, giving I_m, gu, gv.
 *   Residual      r = I_c - I_m; none when |r| > max_residual.
 *   Jacobian      g = (gu * fx / s.z, gv * fy / s.z, -(gu * fx * s.x + gv * fy * s.y) / (s.z * s.z)) with the level's fx, fy (products
 *                 and sums left to right).
 *   Row           weight * (s x g, g, r) (cross3 as the geometric row's), component by component: the geometric row's convention
 *                 A (omega, t) = b for s' = s + omega x s + t.  The pixel's geometric products go into the 27 float accumulators first,
 *                 then the photometric row's.  With weight = 0 every photometric product is an exact zero and the sums are
 *                 df_icp_accumulate's bit for bit.
 *
 * DF_COLOR_TRACK_WEIGHT: geometric rows have entries of order 1 (normals, metre-scale moments); a photometric row's Jacobian is the
 * intensity gradient per pixel times f / z, some 15 to 50 per metre at level 0 on a 5 to 7 cm texture 1 m away.  A weight of 0.03 to 0.1
 * brings it to the same order, so that neither term drowns the other.  Chosen once with the float64 estimate (tests/color_track_reference.py)
 * on a frame pair of the textured wall and of C2 with colour: on the wall every weight from 0.02 to 0.1 gives the same pose to 0.01 mm
 * (geometry alone fails the determinant gate), on C2 the rotation error of the pair is 0.58 degrees with geometry alone, 0.15 at 0.05 and
 * 0.03 at 0.1.
 * DF_COLOR_TRACK_MAX_RESIDUAL: a pixel whose intensities differ by more than 0.2 (a fifth of the range) does not see the same surface
 * point (occlusion edges, a wrong match a texture period away) and is left out rather than pulling the pose; 0.1 to 0.3 change the
 * pair's poses by less than 0.2 mm. */
#define DF_COLOR_TRACK_WEIGHT 0.1f
#define DF_COLOR_TRACK_MAX_RESIDUAL 0.2f
int df_frame_intensity(const void *bgra, size_t bgra_pitch, const df_color_camera *cam, df_intr intr, const float *points, size_t points_pitch,
                       const uint32_t *map, size_t map_pitch, float trunc_dist, int levels, const int *cols, const int *rows, float *const *intensity,
                       const size_t *pitch, void *stream);
int df_model_intensity(df_volume vol, const uint32_t *colors, df_aff3f cam2vol, int levels, const int *cols, const int *rows,
                       const float *const *points, const size_t *points_pitch, float *const *maps, const size_t *maps_pitch, void *stream);

/* The three entries that project into the colour camera, through the colour camera's lens.  Each rule is its entry's above with the
 * colour pixel formed as: pc = depth_to_color * p (the same fma chain), x = pc.x / pc.z, y = pc.y / pc.z, then the lens distortion (an
 * invalid point is skipped, as one outside the image is), uc = fma(cam.fx, xd, cam.cx), vc' = fma(cam.fy, yd, cam.cy); the image bounds,
 * the cell, the occlusion test and the sample are unchanged.  lens == NULL, or all eight coefficients 0: the entry without _lens, bit for
 * bit (the same kernel instance).  An invalid lens (df_lens_check): cudaErrorInvalidValue, nothing written. */
int df_color_depth_map_lens(const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_intr intr, df_color_camera cam, const df_lens *lens,
                            uint32_t *map, size_t map_pitch, void *stream);
int df_integrate_color_camera_lens(df_volume vol, uint32_t *colors, const uint16_t *dists, size_t dists_pitch, int cols, int rows,
                                   df_aff3f vol2cam, df_intr intr, df_color_camera cam, const df_lens *lens, const void *bgra, size_t bgra_pitch,
                                   const uint32_t *map, size_t map_pitch, const unsigned char *activity, void *stream);
int df_frame_intensity_lens(const void *bgra, size_t bgra_pitch, const df_color_camera *cam, const df_lens *lens, df_intr intr, const float *points,
                            size_t points_pitch, const uint32_t *map, size_t map_pitch, float trunc_dist, int levels, const int *cols,
                            const int *rows, float *const *intensity, const size_t *pitch, void *stream);

/* ------------------------------------------------------------------ image processing ----------------------------------------------------- */
/* device::bilateralFilter (internal.hpp:125, imgproc.cu:11-57) */
int df_bilateral(const uint16_t *src, size_t src_pitch, int cols, int rows, uint16_t *dst, size_t dst_pitch,
                 int kernel_size, float sigma_spatial, float sigma_depth, void *stream);
/* device::truncateDepth (internal.hpp:124, imgproc.cu:66-85) */
int df_truncate_depth(uint16_t *depth, size_t pitch, int cols, int rows, float max_dist, void *stream);
/* device::depthPyr (internal.hpp:126, imgproc.cu:94-136): dst is (src_cols/2, src_rows/2) */
int df_pyr_down(const uint16_t *src, size_t src_pitch, int src_cols, int src_rows, uint16_t *dst, size_t dst_pitch,
                float sigma_depth, void *stream);
/* device::computePointNormals (internal.hpp:132, imgproc.cu:210-250) */
int df_points_normals(df_intr intr, const uint16_t *depth, size_t depth_pitch, int cols, int rows,
                      float *points, size_t points_pitch, float *normals, size_t normals_pitch, void *stream);
/* device::resizePointsNormals (internal.hpp:129, imgproc.cu:368-414): dst is (src_cols/2, src_rows/2) */
int df_resize_points_normals(const float *vsrc, size_t vsrc_pitch, const float *nsrc, size_t nsrc_pitch,
                             int src_cols, int src_rows, float *vdst, size_t vdst_pitch, float *ndst, size_t ndst_pitch,
                             void *stream);

/* device::renderImage points variant / renderTangentColors (internal.hpp:134-136, imgproc.cu:484-583): display only, BGRA out */
int df_render_image(const float *points, size_t points_pitch, const float *normals, size_t normals_pitch, int cols, int rows,
                    const float *light_pose_host3, void *image_bgra, size_t image_pitch, void *stream);
int df_render_tangent_colors(const float *normals, size_t normals_pitch, int cols, int rows, void *image_bgra, size_t image_pitch,
                             void *stream);

/* The reference's USE_DEPTH-path image operations (cuda/imgproc.hpp:15,21,23,31; imgproc.cu:145-200,277-303,307-366,420-537).  The
 * default build of the reference does not take this path; they exist so that every function of its public header is served. */
int df_render_image_depth(const uint16_t *depth, size_t depth_pitch, const float *normals, size_t normals_pitch, int cols, int rows,
                          df_intr intr, const float *light_pose_host3, void *image_bgra, size_t image_pitch, void *stream);
int df_normals_mask_depth(df_intr intr, uint16_t *depth, size_t depth_pitch, int cols, int rows, float *normals, size_t normals_pitch, void *stream);
int df_cloud_to_depth(const float *cloud, size_t cloud_pitch, int cols, int rows, uint16_t *depth, size_t depth_pitch, void *stream);
int df_resize_depth_normals(const uint16_t *dsrc, size_t dsrc_pitch, const float *nsrc, size_t nsrc_pitch, int src_cols, int src_rows,
                            uint16_t *ddst, size_t ddst_pitch, float *ndst, size_t ndst_pitch, void *stream);

/* ------------------------------------------------------------------ projective ICP -------------------------------------------------------- */
/* ComputeIcpHelper::operator() points variant (internal.hpp:67-102, proj_icp.cu:80-108,350-394,448-467): one
 * data-association + 27-term reduction pass at one pyramid level.  scratch: 16-byte aligned device buffer of
 * DF_ICP_SCRATCH_DOUBLES doubles; on completion scratch[0..26] hold the 27 sums, order (i, j>=i) for i = 0..5, j = 0..6 (the rest holds the
 * per-block partials, summed in a fixed order: results are run-to-run deterministic).  intr_level are the level's
 * intrinsics (setLevelIntr, projective_icp.cpp:17-23). */
#define DF_ICP_SCRATCH_DOUBLES (32 + 27 * 1024)
int df_icp_accumulate(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch,
                      const float *vprev, size_t vprev_pitch, const float *nprev, size_t nprev_pitch,
                      int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres, float min_cosine,
                      double *scratch, void *stream);

/* ProjectiveICP::estimateTransform, points variant (projective_icp.hpp:39, projective_icp.cpp:169-213) executed
 * entirely on the device: per iteration the association/reduction kernel, then the 6x6 solve + Rodrigues update in a
 * one-thread tail (replaces StreamHelper::get + cv::solve + 19 host round trips).  Arrays of `levels` entries, index 0 =
 * finest.  T_dev (device, 12 floats: R row-major + t) receives curr->prev; ok_dev (device int) is 0 when the
 * reference would have returned false (|det| < 1e-15 or NaN). */
int df_icp_estimate(const float *const *vcurr, const float *const *ncurr, const float *const *vprev, const float *const *nprev,
                    const int *cols, const int *rows, const size_t *pitch, int levels, const int *iters,
                    df_intr intr, float dist_thres, float angle_thres, float *T_dev, int *ok_dev, double *scratch,
                    void *stream);

/* The reference's compile-time USE_DEPTH alternative (internal.hpp:6; ComputeIcpHelper::find_coresp proj_icp.cu:47-78,
 * ComputeIcpHelper::operator()(const Depth&, ...) proj_icp.cu:396-418): the current depth map (u16 millimetres) is
 * re-projected per pixel, the previous depth map is point-sampled at the projection and re-projected at the fractional
 * coordinates; normal maps as above.  Same scratch / sums layout as df_icp_accumulate. */
int df_icp_accumulate_depth(const unsigned short *dcurr, size_t dcurr_pitch, const float *ncurr, size_t ncurr_pitch,
                            const unsigned short *dprev, size_t dprev_pitch, const float *nprev, size_t nprev_pitch,
                            int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres, float min_cosine,
                            double *scratch, void *stream);

/* ProjectiveICP::estimateTransform, depth-pyramid overload (projective_icp.hpp:38, projective_icp.cpp:126-167), device
 * resident like df_icp_estimate. */
int df_icp_estimate_depth(const unsigned short *const *dcurr, const float *const *ncurr, const unsigned short *const *dprev,
                          const float *const *nprev, const int *cols, const int *rows, const size_t *depth_pitch,
                          const size_t *normals_pitch, int levels, const int *iters, df_intr intr, float dist_thres,
                          float angle_thres, float *T_dev, int *ok_dev, double *scratch, void *stream);

/* Test hook: one solve step of df_icp_estimate on a caller's table of per-block partial sums, as the iteration loop runs it after each
 * accumulate pass.  partials: nblocks rows of 27 doubles in device memory, 16-byte aligned; when 27 * nblocks is odd the table is
 * followed by one more (slack) double that is read and ignored.  The rows are summed in the loop's fixed order, rounded to float,
 * solved (Cholesky, else the |det| < 1e-15 gate and the eigen pseudo-inverse) and T (device, 12 floats) <- Tinc * T in place.
 * *ok (device int) must be non-zero on entry, else the step is skipped as after a failed iteration; it is set to 0 when the step
 * fails, and T is then left unchanged. */
int df_icp_solve_step(const double *partials, int nblocks, float *T, int *ok, void *stream);

/* Colour tracking: df_icp_accumulate plus the photometric row of each pixel (the rule above df_frame_intensity).  icurr: the current
 * frame's intensity at the level (df_frame_intensity, float, pitch in bytes); model: the model's (I, gu, gv, 0) map at the level
 * (df_model_intensity, float4, pitch in bytes), both cols x rows.  weight: DF_COLOR_TRACK_WEIGHT in the frame loop, max_residual:
 * DF_COLOR_TRACK_MAX_RESIDUAL.  Same launch rule, scratch and sums layout as df_icp_accumulate. */
int df_icp_accumulate_color(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch, const float *vprev,
                            size_t vprev_pitch, const float *nprev, size_t nprev_pitch, const float *icurr, size_t icurr_pitch,
                            const float *model, size_t model_pitch, int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres,
                            float min_cosine, float weight, float max_residual, double *scratch, void *stream);
/* df_icp_estimate with the photometric rows: per iteration df_icp_accumulate_color's kernel and the same solve kernel, so the launch count
 * is df_icp_estimate's.  icurr / model: per-level arrays as above, with their own pitches. */
int df_icp_estimate_color(const float *const *vcurr, const float *const *ncurr, const float *const *vprev, const float *const *nprev,
                          const float *const *icurr, const size_t *icurr_pitch, const float *const *model, const size_t *model_pitch,
                          const int *cols, const int *rows, const size_t *pitch, int levels, const int *iters, df_intr intr, float dist_thres,
                          float angle_thres, float weight, float max_residual, float *T_dev, int *ok_dev, double *scratch, void *stream);

/* ---- relocaliser (DF_KINFU_RELOCALISE): fern codes of the frame's depth, a keyframe database, and the gate on an ICP result ----------------
 * Rules (tests/reloc_oracle.c states them again, independently; everything but the gate's residual sum is integer, so the kernels and the
 * oracle agree bit for bit):
 *   Table     DF_RELOC_FERNS ferns x 4 binary tests (u, v, theta_mm), drawn for a cols x rows image from the splitmix64 sequence of `seed`:
 *             s = seed; next() = { s += 0x9e3779b97f4a7c15; z = s; z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9;
 *             z = (z ^ (z >> 27)) * 0x94d049bb133111eb; return z ^ (z >> 31) } (u64 arithmetic).  For fern f = 0.., test j = 0..3 in
 *             order: u = next() % cols, v = next() % rows, theta = DF_RELOC_NEAR_MM + next() % (DF_RELOC_FAR_MM - DF_RELOC_NEAR_MM).
 *             df_reloc_fern_table writes them as int32 (u, v, theta) triples, fern-major: 12 * DF_RELOC_FERNS values.
 *   Image     the frame loop codes the ICP pyramid's level 2 of the current depth (bilateral-filtered, truncated when
 *             icp_truncate_depth_dist is set, halved twice by df_pyr_down: 160 x 120 for 640 x 480), with the table drawn for its size
 *             and seed DF_RELOC_SEED.
 *   Code      bit j of fern f is d(u, v) != 0 && d(u, v) < theta (u16 millimetres); the fern's byte is sum of bit_j << j.  A frame's code
 *             is DF_RELOC_FERNS bytes.
 *   Dissimilarity   of two codes: the number of ferns whose bytes differ.
 *   Lookup    the DF_RELOC_CANDIDATES keyframes with the smallest dissimilarity to the frame, ranked by (dissimilarity, index).
 *   Harvest   a frame whose pose the loop accepted (the first frame after create or reset, or a frame that passed the gate) is appended
 *             with that pose when the database is empty, or when its smallest dissimilarity to the database is greater than
 *             DF_RELOC_HARVEST_FERNS and the database holds fewer than DF_RELOC_KEYFRAMES entries.  A full database stops growing; nothing
 *             is evicted.
 *   Gate      for a pose increment T (the ICP's curr -> prev): at level 0, n_valid = current pixels whose vertex is not NaN, n_in = those the
 *             ICP's association accepts (its projection, distance and angle tests, df_icp_accumulate's rule with dist_thres and
 *             angle_thres), sum_sq = the sum over them of r * r in double, r = the row's float residual n_prev . (d - T v_curr).  The pose
 *             is accepted when the ICP's ok holds, n_valid >= DF_RELOC_MIN_VALID, n_in >= DF_RELOC_MIN_INLIER_FRAC * n_valid (in float)
 *             and sqrt(sum_sq / n_in) <= DF_RELOC_MAX_RMS.
 *   Loss      a frame the gate rejects is lost: it fuses and extracts nothing, appends no pose, leaves the frame counter, the previous-frame
 *             maps, the nodes, the cloud and both volumes as they were, and returns 0.  The object stays lost until a frame is accepted
 *             or it is reset.
 *   Relocalise  a frame that arrives while lost tries, in order: the ordinary ICP (with colour rows where the loop uses them) against the
 *             kept previous-frame maps from the last good pose; then each lookup candidate: the canonical volume ray-cast from the
 *             keyframe's pose into maps of the object's own (the kept maps stay as they were) and the geometric ICP against them, pose =
 *             keyframe pose * T.  The first that passes the gate is the frame's pose and the frame continues as a tracked one.  A keyframe
 *             win sets every node's transform to the identity (positions and weights kept); the ordinary ICP's win keeps the field.
 *
 * DF_RELOC_NEAR_MM / DF_RELOC_FAR_MM: the depth range the thresholds are drawn from, the working range of a structured-light or
 * time-of-flight sensor at arm's length; a threshold outside the scene's depths makes a test that never changes.
 * DF_RELOC_HARVEST_FERNS: a view becomes a keyframe when more than this many of its ferns differ from every stored one (Glocker et al. use
 * a fifth of the ferns as the novelty bar; here a smaller share, so that a slow sweep of one scene still leaves several keyframes).
 * DF_RELOC_MIN_VALID, DF_RELOC_MIN_INLIER_FRAC and DF_RELOC_MAX_RMS: a frame with almost no depth, or whose points mostly find no model
 * surface, or whose associated points lie centimetres off it, is not tracked.  The inlier share is of every valid pixel, and a volume
 * smaller than the view leaves the pixels beyond it unassociated: with the 1 m cube of the synthetic sequences some 45 % of a 640 x 480
 * frame sees no model, and the warped loop with a growing field was measured at 20 % on a tracked frame of C2 (frame 53), hence 0.1;
 * blank frames and views of another scene associate next to nothing.  The RMS bar allows the breathing surfaces of the non-rigid loop, whose ray-cast reference is the
 * undeformed canonical model. */
#define DF_RELOC_FERNS 500
#define DF_RELOC_CANDIDATES 3
#define DF_RELOC_KEYFRAMES 512
#define DF_RELOC_NEAR_MM 400
#define DF_RELOC_FAR_MM 3000
#define DF_RELOC_SEED 0x5eedf00dull
#define DF_RELOC_HARVEST_FERNS 40
#define DF_RELOC_MIN_VALID 5000
#define DF_RELOC_MIN_INLIER_FRAC 0.1f
#define DF_RELOC_MAX_RMS 0.03f

/* the gate's result as df_icp_inliers writes it (72 bytes): the ICP's T and ok copied alongside the counts, so that one copy brings all of
 * it to the host */
typedef struct df_reloc_gate {
    float T[12];
    int ok, n_valid, n_in, pad;
    double sum_sq;
} df_reloc_gate;

/* df_fern_match's output (device): the lookup's candidates (index -1 and dissimilarity DF_RELOC_FERNS + 1 past the database's count), whether
 * the frame was appended, the database's count after the call, and the candidates' poses (12 floats each, zero past the count) */
typedef struct df_reloc_match {
    int index[DF_RELOC_CANDIDATES];
    int dissimilarity[DF_RELOC_CANDIDATES];
    int appended, count;
    float pose[DF_RELOC_CANDIDATES][12];
} df_reloc_match;

/* the Table rule for a cols x rows image into out_host (12 * n_ferns int32); host only.  cols, rows or n_ferns < 1: cudaErrorInvalidValue */
int df_reloc_fern_table(unsigned long long seed, int cols, int rows, int n_ferns, int32_t *out_host);
/* the Code rule: one thread per fern, one launch.  depth: device u16, pitch in bytes (even, at least cols * 2); table: device, as
 * df_reloc_fern_table writes it for this size (a test outside the image reads as 0 bit); codes: device, n_ferns bytes. */
int df_fern_encode(const uint16_t *depth, size_t pitch, int cols, int rows, const int32_t *table, int n_ferns, uint8_t *codes, void *stream);
/* Dissimilarity, Lookup and (append != 0) the Harvest rule in one single-block launch.  db_codes: device, capacity x n_ferns bytes;
 * db_poses: device, capacity x 12 floats; count: device int, the entries held (updated on an append); code: device, the frame's n_ferns bytes;
 * pose: the frame's pose, stored on an append.  capacity <= DF_RELOC_KEYFRAMES, n_ferns <= DF_RELOC_FERNS, else cudaErrorInvalidValue. */
int df_fern_match(uint8_t *db_codes, float *db_poses, int *count, int capacity, const uint8_t *code, int n_ferns, int append, df_aff3f pose,
                  df_reloc_match *out, void *stream);
/* the Gate rule's counts at one level: vertex and normal maps as df_icp_accumulate's (float4, pitches in bytes, multiples of 16), T_dev
 * (device, 12 floats; NULL: the identity) and ok_dev (device int; NULL: 1) copied into out.  One launch; the residual sum is reduced in a
 * fixed order (run-to-run deterministic).  ws: device, DF_RELOC_GATE_WS_BYTES, zeroed before its first use (every call leaves it zeroed). */
#define DF_RELOC_GATE_WS_BYTES 4096
int df_icp_inliers(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch, const float *vprev, size_t vprev_pitch,
                   const float *nprev, size_t nprev_pitch, int cols, int rows, df_intr intr, const float *T_dev, const int *ok_dev,
                   float dist_thres, float angle_thres, df_reloc_gate *out, void *ws, void *stream);
/* the Gate rule's decision on a result of df_icp_inliers; host only */
int df_reloc_gate_accepts(const df_reloc_gate *g);

/* ------------------------------------------------------------------ warp field ------------------------------------------------------------ */
/* deformation_node (warp_field.hpp:35-40) as 12 floats: vertex[3], rotation quat (w,x,y,z), dual/translation quat
 * (w,x,y,z) = 0.5*t*r (dual_quaternion.hpp:59-63), weight. */
#define DF_NODE_STRIDE 12
#define DF_KNN 8                          /* KNN_NEIGHBOURS, warp_field.hpp:10 */

/* WarpField::KNN (warp_field.hpp:66, warp_field.cpp:247-251) for N queries: exact 8-NN, ascending squared distance,
 * ties -> lower node index; idx = -1 / d2 = FLT_MAX for NaN queries or when M < 8.  qstride in floats. */
int df_knn8(const float *nodes, int M, const void *node_grid, const float *queries, int N, int qstride, int32_t *idx, float *d2,
            void *stream);

/* WarpField::buildKDTree (warp_field.hpp:84, warp_field.cpp:275-282): uniform grid over the node vertices that replaces the
 * nanoflann index.  Optional everywhere (`node_grid` = NULL -> exhaustive shared-memory scan); results are identical either
 * way (candidates ranked by (distance, index)).  Build once per node set: vertices do not move after WarpField::init. */
size_t df_node_grid_bytes(int M);
int df_build_node_grid(const float *nodes, int M, void *node_grid, void *stream);

/* Extending the warp field (SURVEY.md 8f(3); Report.md "4. Extending the warp field - stubbed out functionality"): nodes are appended for
 * the points of the extracted canonical cloud that the field does not support.  A point is unsupported when its nearest node (of the M
 * nodes present on entry) is farther than `radius`; every step-th unsupported point, in cloud order (the subsampling rule of
 * WarpField::init, warp_field.cpp:49-60), becomes a node as init makes them (identity DualQuaternion(), weight 3, :68-80), appended to
 * `nodes` (capacity max_nodes) until it is full.  cloud: float[capacity][stride], count_dev (optional, device) = valid points;
 * M_out_dev (device int) receives the new node count -- rebuild the node grid (df_build_node_grid) when it differs from M.
 * workspace: df_extend_field_workspace_bytes(capacity) bytes. */
size_t df_extend_field_workspace_bytes(int capacity);
int df_extend_field(float *nodes, int M, int max_nodes, const void *node_grid, const float *cloud, int capacity, const int *count_dev,
                    int stride, float radius, int step, int *M_out_dev, void *workspace, void *stream);

/* WarpField::warp (warp_field.hpp:62, warp_field.cpp:180-195): k-NN + weights + DQB + transform of points and
 * normals in place (stride in floats, 3 or 4).  flags: bit0 = reference normal cursor (advance only on valid points),
 * bit1 = rotate normals only (extension).  idx_out / w_out (optional, N*8) receive the neighbours and weights. */
#define DF_WARP_REF_NORMAL_INDEX 1
#define DF_WARP_NORMAL_ROTATE_ONLY 2
#define DF_WARP_REUSE_KNN 4        /* idx_out / w_out are INPUTS: neighbours + weights of these points from an earlier pass */
/* flags bits 8..23: the points are an image of that many columns (N = cols * rows, cols % 32 == 0, rows % 8 == 0): a warp then takes an
 * 8 x 4 pixel patch, whose queries share one short candidate list in the 8-NN search.  Results do not depend on it. */
#define DF_WARP_IMAGE_COLS(c) (((c) & 0xffff) << 8)
int df_warp(const float *nodes, int M, const void *node_grid, float *points, float *normals, int N, int stride, df_aff3f warp_to_live,
            int flags, int32_t *idx_out, float *w_out, void *stream);

/* Per-voxel warped integration (SURVEY.md 8f(1)): the update TsdfVolume::surface_fusion (tsdf_volume.hpp:76-79,
 * tsdf_volume.cpp:228-254) was written towards and left commented out (:248-251) -- DynamicFusion eq. 4-5.  For every voxel:
 *   x_c = vol2world * (x*vs, y*vs, z*vs);  x_t = world2cam * DQB(8-NN of x_c).transform(x_c)   (WarpField::warp, warp_field.cpp:180-251)
 *   rho = depth_mm(floor v, floor u) * 0.001 - x_t.z                                            (TsdfVolume::psdf, tsdf_volume.cpp:266-292)
 *   if rho > -trunc:  tsdf = min(1, rho/trunc);  w = clamp(rint(weight_scale * mean node distance), 1, max_weight)  (TsdfVolume::weighting,
 *   :300-306; weight_scale <= 0 -> w = 1);  F' = (F*W + tsdf*w)/(W + w);  W' = min(W + w, max_weight).
 * depth: the frame's u16 millimetre image (not the ray lengths df_integrate takes); nodes / node_grid: the warp field (node_grid is
 * required).  counters (optional, device, 2 x u64): [0] += voxels written, [1] += voxels warped (k-NN + blend evaluated).
 * activity: as df_integrate_tracked.  workspace (optional, device): df_integrate_warped_workspace_bytes(cols, rows, M) bytes
 * (M = the largest node count it will be used with). */
size_t df_integrate_warped_workspace_bytes(int cols, int rows, int M);
int df_integrate_warped_launch_count(void);
int df_integrate_warped(df_volume vol, const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_aff3f vol2world,
                        df_aff3f world2cam, df_intr intr, const float *nodes, int M, const void *node_grid, float weight_scale,
                        unsigned long long *counters, unsigned char *activity, void *workspace, void *stream);

/* df_integrate_warped_color: df_integrate_warped, and in the same voxel walk the frame's colour image fused into the colour volume `colors`
 * (laid out as vol.data, df_integrate_color's words).  The TSDF volume, the activity map and counters[0..1] are df_integrate_warped's on the
 * same inputs, bit for bit, with the same launches (df_integrate_warped_launch_count).
 *   Rule (tests/warped_color_oracle.c, over the per-voxel records of oracle/orc_fusion.c's warped fusion; IEEE round-to-nearest, fma only
 *                 where written): for every voxel that df_integrate_warped's rule writes, with the values that rule formed -- the warped
 *                 camera-frame point x_t = (tx, ty, tz), its depth pixel ((int)u, (int)v) and rho = depth_mm * 0.001f - tz -- and after its
 *                 TSDF update:
 *   Band          skipped unless |rho| <= DF_COLOR_BAND * trunc_dist (the product is one float).  The band is on warped fusion's z-difference
 *                 rho, not on the ray length from dists that df_integrate_color's band uses: the voxel reaches its pixel through the field,
 *                 and rho is what its TSDF sample is made of.  It lies inside the TSDF gate rho > -trunc_dist.
 *   Sample        cam == NULL: bgra pixel ((int)u, (int)v) of an image registered to the depth (cols x rows).  cam != NULL: x_t through
 *                 the colour camera as df_integrate_color_camera_lens takes vc: pc = depth_to_color * x_t (its fma chain), the colour pixel
 *                 (through `lens` when it is neither NULL nor the zero lens), the image bounds, the occlusion test against `map`
 *                 (df_color_depth_map of the same frame) with DF_COLOR_OCCLUSION * trunc_dist, then the pixel of bgra; a voxel the colour
 *                 camera does not see is skipped.
 *   Update        df_integrate_color's integer running average, W' = min(W + 1, min(max_weight, 255)).
 * counters (optional, device, 3 x u64): [0], [1] as df_integrate_warped's, [2] += voxels that took a colour sample.  bgra: device, pitch a
 * multiple of 4 and at least its width * 4 (cols, or cam->cols); depth_pitch at least cols * 2, even; map as df_color_depth_map writes it.
 * A NULL pointer, a bad pitch, an invalid camera (df_color_map_dims) or lens (df_lens_check): cudaErrorInvalidValue, nothing written. */
int df_integrate_warped_color(df_volume vol, const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_aff3f vol2world,
                              df_aff3f world2cam, df_intr intr, const float *nodes, int M, const void *node_grid, float weight_scale,
                              unsigned long long *counters, unsigned char *activity, void *workspace, uint32_t *colors, const void *bgra,
                              size_t bgra_pitch, const df_color_camera *cam, const df_lens *lens, const uint32_t *map, size_t map_pitch,
                              void *stream);

/* WarpFieldOptimiser::optimiseWarpData (warp_field_optimiser.hpp:14-17) -> CombinedSolver (CombinedSolver.h:25-110)
 * -> Opt LM/PCG on kfusion/solvers/dynamicfusion.t: translation-only data term solved on the device; node
 * translations are updated in place (encodeTranslation, CombinedSolver.h:189-197).
 * params: nonlinear (LM) iterations, linear (PCG) iterations; stats_dev (device, 8 doubles): initial cost, final cost,
 * LM iterations run, valid rows, PCG iterations run, row-overflow flag, [6] non-zeros of the normal matrix, [7] which LM kernel solved it
 * (>= 0: the one-exchange cluster kernel, value = halo columns exchanged per PCG step; -1: the two-exchange cluster kernel, its fallback;
 * -2: the one-block kernel, for systems no cluster holds; fraction .5 (0.5, -0.5, -1.5): matrix assembled from tile records).  If a node's row of the normal matrix couples to more columns
 * than the kernels store (512), the flag is raised and the solve leaves the node translations UNCHANGED (0 LM iterations) rather than
 * solving a truncated, asymmetric system; callers must look at stats[5] (the frame loop reports it through df_kinfu_get_info[11] and on
 * stderr, the C++ mirror prints an error).  workspace from df_solve_workspace_bytes(M, N).
 * Rows with a NaN in canon or live are skipped (the reference zero-fills them with stale k-NN scratch). */
size_t df_solve_workspace_bytes(int M, int N);
/* after df_solve_data_term: the per-vertex neighbour indices (N*8, -1 for skipped rows) and weights (N*8) it computed for
 * `canon`, inside `workspace` -- valid until the workspace is reused; lets the following warp of the same vertices skip its
 * k-NN pass (DF_WARP_REUSE_KNN) */
int df_solve_knn_buffers(void *workspace, int M, int N, int32_t **idx, float **w);
/* after df_solve_data_term: the normal system A x = gb the LM iteration was given, as device pointers into `workspace` (A = W^T W,
 * gb = W^T b of the data term).  A is stored ELL, column-major with stride M: row i has rownnz[i] entries, entry e at col[e * M + i] /
 * val[e * M + i] (e < 512), columns ascending; gb is axis-major [3 * M] (gb[a * M + i]); diag [M] = A_ii (0 for a row without support).
 * Only the assembly kernels write these arrays (the LM kernels read them), so they stay valid until the workspace is reused.  Not
 * meaningful when stats[5] reported a row overflow. */
int df_solve_normal_system(void *workspace, int M, int N, int32_t **rownnz, int32_t **col, double **val, double **gb, double **diag);
#define DF_SOLVE_REF_GRAPH_QUIRK 1
/* flags bits 8..23: the vertices are an image of that many columns (N = cols * rows, row-major, cols % 16 == 0, rows % 8 == 0): lets the
 * assembly of the normal matrix work tile by tile (16 x 8 pixels share a dozen nodes) instead of entry by entry.  Same result up to the
 * order of the double sums; 0 (a flat vertex list) always takes the per-entry path. */
#define DF_SOLVE_IMAGE_COLS(c) (((c) & 0xffff) << 8)
int df_solve_data_term(float *nodes, int M, const void *node_grid, const float *canon, const float *live, int N, int stride,
                       int nonlinear_iters, int linear_iters, int flags, double *stats_dev, void *workspace, void *stream);

/* SURVEY.md 8f(2), OPT-IN beside df_solve_data_term: the robust data term over 6-DoF node increments plus the regularisation term -- the
 * energy the reference defines piecewise and never assembles (6-wide parameter blocks optimisation.hpp:108-110,141-143; tukeyPenalty :84-88,
 * dynamicfusion.t:43-51; huberPenalty optimisation.hpp:134-138, dynamicfusion.t:34-40; empty DynamicFusionRegEnergy :125-132 /
 * WarpField::energy_reg warp_field.cpp:168-172; KinFu::edges_ kinfu.hpp:95).  PARITY UNPINNED (no reference code evaluates it); restated in
 * oracle/orc_reg.c, solved in csrc/regsolve.cu:
 *   E = sum_v sum_c rho_T(live_v - warp(canon_v))_c  +  reg_lambda sum_(i,j) max(weight_i, weight_j) sum_c rho_H(T_i(g_j) - T_j(g_j))_c
 * warp = WarpField::DQB + transform over the 8 nearest nodes; T_k(p) = rotate(q_k, p) + t_k; j runs over the reg_k (<= 7) nearest other nodes
 * of node i; rho_T' = tukeyPenalty(., tukey_c) (DF_F2_TUKEY, else squared loss); rho_H = huberPenalty(., huber_delta) (DF_F2_HUBER, else
 * squared loss).  Unknowns per node: (omega, tau), q <- exp(omega) q, t <- t + tau (DF_F2_TWIST; without it omega = 0: translation-only).
 * Gauss-Newton / IRLS, gn_iters steps, each solved by block-Jacobi PCG (at most lin_iters steps) with Levenberg damping lm_mu * diag(H).
 * Nodes are updated in place (rotation + dual part).  stats_dev (device, 16 doubles): [0] energy before, [1] energy after, [2] GN steps,
 * [3] valid vertices, [4] data energy after, [5] regularisation energy after, [6] edge slots, [7] PCG steps in total, [8 + i] energy before
 * GN step i (i < 8).  workspace: df_solve_f2_workspace_bytes(M, N, reg_k). */
typedef struct df_f2_params {
    double reg_lambda, tukey_c, huber_delta, lm_mu;   /* 0 = no regulariser, 0.01, 1e-4 (the reference's defaults for c and delta), 1e-4 */
    int gn_iters, reg_k, flags, lin_iters;
} df_f2_params;
#define DF_F2_TWIST 1
#define DF_F2_TUKEY 2
#define DF_F2_HUBER 4
size_t df_solve_f2_workspace_bytes(int M, int N, int reg_k);
int df_solve_f2(float *nodes, int M, const void *node_grid, const float *canon, const float *live, int N, int stride,
                const df_f2_params *params, double *stats_dev, void *workspace, void *stream);

/* ------------------------------------------------------------------ per-frame pipeline ----------------------------------------------------- */
/* kfusion::KinFuParams (kinfu.hpp:15-47) as a POD, plus the solver settings KinFu::KinFu hard-codes (kinfu.cpp:114-120)
 * and the knobs of the GPU-resident warp field. */
typedef struct df_kinfu_params {
    int cols, rows;
    df_intr intr;
    int volume_dims[3];
    float volume_size[3];
    df_aff3f volume_pose;
    float bilateral_sigma_depth, bilateral_sigma_spatial;
    int bilateral_kernel_size;
    float icp_truncate_depth_dist, icp_dist_thres, icp_angle_thres;
    int icp_iter_num[4];
    float tsdf_min_camera_movement, tsdf_trunc_dist;
    int tsdf_max_weight;
    float raycast_step_factor, gradient_delta_factor;
    float light_pose[3];
    int solver_nonlinear_iters, solver_linear_iters;   /* 5, 100 (kinfu.cpp:116-117) */
    int max_nodes;        /* cap on warp nodes; node_step grows to respect it */
    int node_step;        /* every node_step-th extracted point becomes a node: 50 (warp_field.cpp:49) */
    int cloud_capacity;   /* extracted-cloud buffer, points: 256^3 in the reference (tsdf_volume.cpp:184) */
    int flags;            /* DF_KINFU_* */
    float fusion_weight_scale;   /* DF_KINFU_WARPED_INTEGRATE: weight_scale of df_integrate_warped (0 = every sample weighs 1) */
    float extend_radius;         /* DF_KINFU_EXTEND_FIELD: support radius of df_extend_field in metres (<= 0: 0.03) */
} df_kinfu_params;

#define DF_KINFU_RIGID_ONLY 1      /* skip warp + solve (plain KinFu loop: config 1) */
#define DF_KINFU_STAGE_TIMING 2    /* record CUDA events per stage (df_kinfu_get_stage_ms) */
#define DF_KINFU_REF_GRAPH_QUIRK 4 /* forward DF_SOLVE_REF_GRAPH_QUIRK to the solve */
#define DF_KINFU_WARPED_INTEGRATE 8 /* SURVEY 8f(1): the fusion step of KinFu::dynamicfusion integrates the frame through the warp field, voxel by
                                      voxel (df_integrate_warped), instead of project_and_remove + the rigid integrate the reference falls back to
                                      (tsdf_volume.cpp:234-238).  Also switched on by the environment variable DF_KINFU_WARPED_INTEGRATE=1, so that an
                                      unchanged apps/demo.cpp can run it; DF_FUSION_WEIGHT_SCALE sets fusion_weight_scale the same way. */

#define DF_KINFU_F2_SOLVE 32       /* SURVEY 8f(2): the frame's warp solve is df_solve_f2 (robust 6-DoF data term + regulariser) instead of the reference's
                                      translation-only data term; parameters from df_kinfu_set_f2_params (defaults: lambda 5, reg_k 4, twist + Tukey(0.05) + Huber(1e-4),
                                      2 GN x 30 PCG steps).  Environment: DF_KINFU_F2_SOLVE=1. */
#define DF_KINFU_USE_DEPTH 64       /* the reference's compile-time USE_DEPTH frame loop (internal.hpp:6; kinfu.cpp:237-238,253-255,271,293-295): normals from the depth
                                      pyramid with masking (df_normals_mask_depth), ICP on depth pyramids (df_icp_estimate_depth), the model ray-cast stored as a depth map
                                      (df_cloud_to_depth) and halved by df_resize_depth_normals.  Environment: DF_KINFU_USE_DEPTH=1. */
#define DF_KINFU_EXTEND_FIELD 16    /* SURVEY 8f(3): after every extraction the warp field is extended (df_extend_field, radius = extend_radius, step = node_step,
                                      up to max_nodes) and the node grid rebuilt; costs one 4-byte read-back per frame.  Environment: DF_KINFU_EXTEND_FIELD=1,
                                      DF_EXTEND_RADIUS. */
#define DF_KINFU_LIVE_MODEL 128     /* track and solve against the rendered live model (DynamicFusion's model-to-frame association) instead of ray-casts of the
                                      undeformed canonical volume.  At the end of every frame fused with a warp field, the frame's mesh (df_mesh_count / _emit
                                      over the cloud, the cloud moved by -R_vol * (vs/2) to the ray-cast's voxel convention, carried through the field by
                                      df_warp) is rasterised at the identity camera into the previous-frame maps that the next ICP tracks against.  The next
                                      frame renders that mesh from the ICP increment poses[-2]^-1 * poses[-1] and takes its canonical points from
                                      df_mesh_correspond (source = the moved, unwarped cloud; target = the frame's vertex map, max_dist = icp_dist_thres): they
                                      are model coordinates, not pose^-1 * p_camera.  Rigid frames keep the ray-casts; a mesh that cannot be built (cloud
                                      truncated at cloud_capacity) falls back to them for the frame (df_kinfu_get_info[12], reported once on stderr).  The
                                      extraction then runs on the main stream, and the triangle count costs one host read-back per frame.  Environment:
                                      DF_KINFU_LIVE_MODEL=1. */

#define DF_KINFU_COLOR 256          /* fuse RGB-D frames: the object also owns a colour volume (df_integrate_color; 4 bytes per voxel, 512 MiB at 512^3), one
                                      RGBA word per cloud slot and a device colour frame.  df_kinfu_process_host_color / _device_color fuse the frame's
                                      BGRA image right after its rigid integrate (same dists, vol2cam and activity map; in the dynamic loop the dists have
                                      been through df_project_and_remove), and every extraction is followed by df_sample_colors over the cloud (offset
                                      0.5).  Colour never feeds back: poses, volume, nodes and cloud equal those of the same run without the flag bit for
                                      bit; a colour frame launches two kernels more (three with a colour camera, df_kinfu_set_color_camera), a
                                      depth-only frame on a colour object one (the cloud's colours).
                                      Without the flag nothing is allocated or launched.  Refused at create (reason on stderr) together with
                                      DF_KINFU_WARPED_INTEGRATE unless DF_KINFU_WARPED_COLOR is set too: there a voxel meets its pixel through the warp
                                      field, which the rigid colour rule does not follow; every other flag combines with it.
                                      Environment: DF_KINFU_COLOR=1. */
#define DF_KINFU_COLOR_TRACKING 512 /* track colour frames with colour as well as geometry: a frame that carries a colour image builds its intensity pyramid
                                      at the end of pre-processing (df_frame_intensity: `levels` launches, through the colour camera when one is set), and
                                      its ICP starts from the model's intensity maps -- df_model_intensity of the colour volume at the previous vertex maps,
                                      seen from poses.back() (one launch) -- and runs df_icp_estimate_color (weight DF_COLOR_TRACK_WEIGHT, gate
                                      DF_COLOR_TRACK_MAX_RESIDUAL) instead of df_icp_estimate.  The maps are a function of the state at the start of the
                                      frame, so snapshots are unchanged and a resumed run equals the uninterrupted one.  A depth-only frame runs the
                                      geometric ICP and launches nothing more.  Buffers: DF_KINFU_BUF_INTENSITY and DF_KINFU_BUF_MODEL_INTENSITY, by
                                      level.  Refused at create (reason on stderr) without DF_KINFU_COLOR, and with DF_KINFU_USE_DEPTH or
                                      DF_KINFU_LIVE_MODEL (their previous maps are not the ray-cast's vertex maps of the canonical volume).  Without the
                                      flag nothing is computed, allocated or launched.  Environment: DF_KINFU_COLOR_TRACKING=1 switches it on for every colour object
                                      (DF_KINFU_COLOR by flag or by its variable); colourless objects are left as they are. */
#define DF_KINFU_WARPED_COLOR 1024  /* colour under per-voxel warped fusion: with DF_KINFU_COLOR and DF_KINFU_WARPED_INTEGRATE (refused at create without
                                      either, reason on stderr), a colour frame fused through a warp field calls df_integrate_warped_color instead of
                                      df_integrate_warped -- the frame's colour image (through the colour camera, its lens and the frame's occlusion
                                      map when one is set) goes into the colour volume in the same voxel walk, each voxel sampled where the field
                                      carries it, so surface that moves keeps taking the colour it shows now.  The launches are df_integrate_warped's.
                                      Rigid frames (the first one, fewer than 8 nodes) keep the rigid colour rule of DF_KINFU_COLOR; depth-only frames
                                      call df_integrate_warped and leave the colour volume as it was.  Colour never feeds back unless
                                      DF_KINFU_COLOR_TRACKING is set (which combines with it): poses, volume, nodes and cloud equal those of the same
                                      run with DF_KINFU_WARPED_INTEGRATE alone, bit for bit.  Snapshots carry the flag in their parameters.
                                      Environment: DF_KINFU_WARPED_COLOR=1 adds it to every object that has both other flags; others are left as they
                                      are. */
#define DF_KINFU_RELOCALISE 2048    /* keep the model through tracking loss and relocalise the camera from fern-coded keyframes (rules below, "relocaliser")
                                      instead of resetting when the ICP fails.  Every frame's level-2 depth is fern-coded (df_fern_encode) and every
                                      ICP result goes through the gate (df_icp_inliers); a frame that fails it is lost: it returns 0 and changes no
                                      state.  Frames that arrive while lost try the ordinary ICP from the last good pose first, then the
                                      DF_RELOC_CANDIDATES most similar keyframes.  A tracked frame launches three kernels more (encode, gate, match);
                                      its {T, ok} and the gate's counts come home in one copy, at the ICP's existing synchronisation.  Combines with
                                      every flag but DF_KINFU_USE_DEPTH and DF_KINFU_LIVE_MODEL (refused at create, reason on stderr: their ICP
                                      references are depth pyramids and a raster of the live mesh, not ray-casts of the canonical volume); needs at
                                      least 3 used ICP levels.  The pose of df_kinfu_set_overrides bypasses the gate.  df_kinfu_get_info[13..16]
                                      report it; df_kinfu_reset empties the keyframe database and ends a loss; snapshots carry both (version 5).
                                      The C++ mirror takes it in dfusion_flags (KinFu::isLost()).  Without the flag nothing is computed,
                                      allocated or launched, and ICP failure resets the object as before.  Environment: DF_KINFU_RELOCALISE=1. */

/* which = 0: KinFuParams::default_params_dynamicfusion (kinfu.cpp:14-49); 1: default_params (kinfu.cpp:55-89) */
void df_kinfu_default_params(df_kinfu_params *p, int which);
/* KinFu::KinFu (kinfu.cpp:95-125): allocates volume, pyramids, ICP and warp/solver state on the current device */
void *df_kinfu_create(const df_kinfu_params *p);
void df_kinfu_destroy(void *kinfu);
int df_kinfu_set_stream(void *kinfu, void *stream);
/* KinFu::reset (kinfu.cpp:196-207) */
int df_kinfu_reset(void *kinfu);
/* KinFu::operator()(depth) (kinfu.cpp:221-305).  Returns 1 = frame fused and ray-cast image available, 0 = first frame or
 * tracking reset (the reference's `false`; under DF_KINFU_RELOCALISE a lost frame instead), < 0 = -(cudaError).  _host: depth is a HOST u16 image (any pitch), copied to
 * the device inside the call (the path apps/demo.cpp takes: imread -> upload -> operator()); _device: depth already in HBM. */
int df_kinfu_process_host(void *kinfu, const uint16_t *depth_host, size_t pitch);
int df_kinfu_process_device(void *kinfu, const uint16_t *depth_dev, size_t pitch);
/* The same with the frame's colour image (DF_KINFU_COLOR): BGRA, 4 bytes per pixel, registered to the depth image (or taken by the colour
 * camera df_kinfu_set_color_camera set, at its size), pitch in bytes (at least its cols * 4, a multiple of 4).  On an object without the flag they return -cudaErrorInvalidValue and do nothing.  The depth-only entries
 * above on a colour object fuse geometry only: the colour volume stays as it was, and the cloud's colours are sampled from it again. */
int df_kinfu_process_host_color(void *kinfu, const uint16_t *depth_host, size_t pitch, const void *bgra_host, size_t bgra_pitch);
int df_kinfu_process_device_color(void *kinfu, const uint16_t *depth_dev, size_t pitch, const void *bgra_dev, size_t bgra_pitch);
/* DF_KINFU_COLOR with a colour camera of its own calibration (df_color_camera): from the next frame on, the _color entries take an image of
 * cam->cols x cam->rows pixels (pitch at least cam->cols * 4, a multiple of 4) taken by that camera.  Each colour frame builds the occlusion
 * map df_color_depth_map from the frame's input depth (the full frame, before the bilateral filter and before df_project_and_remove) and
 * fuses with df_integrate_color_camera instead of df_integrate_color, with the same dists, vol2cam and activity map; a colour frame then
 * launches three kernels more than a colourless one.  Colour still never feeds back.  Accepted only on a colour object whose frame counter
 * is 0 (after create or a reset); cam == NULL goes back to the registered image.  Invalid values (df_color_map_dims' rule), a colourless
 * object or a running sequence: cudaErrorInvalidValue and nothing changes.  Reallocates the device colour frame at the image's size and
 * allocates the map (DF_KINFU_BUF_COLOR_MAP).  Reset keeps the camera: it is calibration, not state.  Synchronises the object's stream. */
int df_kinfu_set_color_camera(void *kinfu, const df_color_camera *cam);
/* Lenses (df_lens).  df_kinfu_set_depth_lens: the depth camera's lens, on any object.  From the next frame on, the first thing a frame
 * does is df_undistort of the caller's depth (and of its registered colour image; a registered colour image shares the depth lens) into
 * buffers the object owns, allocated only while a lens is set; every later stage reads those, and the caller's buffers are never
 * written.  One launch more per frame.  The lens acts before every stage, so it combines with every flag.
 * df_kinfu_set_color_lens: the lens of the colour camera df_kinfu_set_color_camera set (a colour object with a camera only): the colour
 * camera's launches become the _lens entries; no launch more.  df_kinfu_set_color_camera drops the colour lens (it belongs to the camera
 * it was calibrated with).
 * Both follow df_kinfu_set_color_camera's rules: accepted while the frame counter is 0 (after create or a reset); NULL, or all eight
 * coefficients 0, removes the lens; an invalid lens (df_lens_check), or a call the object refuses: cudaErrorInvalidValue and nothing
 * changes.  Reset keeps the lenses.  Synchronise the object's stream.  df_kinfu_dynamicfusion, df_kinfu_render*, the meshes and the
 * exports take and produce ideal pinhole images and points: no lens applies to them. */
int df_kinfu_set_depth_lens(void *kinfu, const df_lens *lens);
int df_kinfu_set_color_lens(void *kinfu, const df_lens *lens);
/* Multi-device host entry (config 5: independent sequences batched across the GPUs of one box).  A KinFu object belongs to the CUDA device
 * that was current when it was created (cudaSetDevice(i) before df_kinfu_create) and every df_kinfu_* call switches to it.  This call
 * advances n objects by one frame each CONCURRENTLY -- one host thread per object, because a frame contains one host synchronisation --
 * and returns 0 or the most negative status; results[i] = what df_kinfu_process_host returns for object i. */
int df_kinfu_batch_process_host(void *const *kinfus, const uint16_t *const *depth_host, const size_t *pitch, int n, int *results);
/* KinFu::dynamicfusion(depth, live_frame, current_normals) (kinfu.hpp:87, kinfu.cpp:344-400) on caller-provided device buffers,
 * at the latest pose: raycast -> warp -> solve -> warp -> project/remove -> integrate -> extract.  depth is modified in place. */
int df_kinfu_dynamicfusion(void *kinfu, uint16_t *depth_dev, size_t depth_pitch, const float *live_points_dev, size_t live_pitch);
/* The surface extraction of a frame (compute_points / compute_normals, kinfu.cpp:398-399) runs on an auxiliary stream of the object and
 * overlaps the frame's last ray-cast and the next frame's pre-processing + ICP: nothing later in the loop reads the cloud, and the volume it
 * reads is not written before the next integrate (which waits for it).  Every accessor of the cloud (df_kinfu_get_info, _read_buffer,
 * _get_buffer(DF_KINFU_BUF_CLOUD*), _state_digest) waits for it; df_kinfu_join makes the object's MAIN stream wait for it without a host synchronisation
 * (what a caller timing frames with events on that stream wants).  DF_KINFU_OVERLAP_EXTRACT=0 (environment) keeps everything on one stream. */
int df_kinfu_join(void *kinfu);
/* KinFu::getCameraPose(time) (kinfu.cpp:213-218): 12 floats, R row-major then t; time < 0 = latest */
int df_kinfu_get_pose(void *kinfu, int time, float *pose12_host);
/* info[0] frame counter, [1] warp nodes M, [2] extracted cloud points, [3] poses stored, [4] last ICP ok,
 * [5] kernels launched in the last frame (memsets are not counted; DF_KINFU_COLOR adds df_integrate_color, or df_color_depth_map and
 * df_integrate_color_camera with a colour camera, on a colour frame, and df_sample_colors after every extraction; with DF_KINFU_WARPED_COLOR a
 * colour frame fused through the warp field adds only df_color_depth_map with a colour camera (df_integrate_warped_color launches what
 * df_integrate_warped would); DF_KINFU_COLOR_TRACKING adds
 * df_frame_intensity's launches (one per ICP level) on a colour frame and df_model_intensity on a tracked one; a depth lens adds df_undistort
 * on every frame), [6] resets so far, [7] solver LM iterations (last frame),
 * [8] voxels written by the last integrate (DF_KINFU_STAGE_TIMING only), [9] solver PCG iterations (last frame),
 * [10] voxels carried through the warp field by the last df_integrate_warped (DF_KINFU_WARPED_INTEGRATE + STAGE_TIMING),
 * [11] frames whose warp solve was skipped because a normal-matrix row overflowed (df_solve_data_term: stats[5]); also reported on stderr,
 * [12] DF_KINFU_LIVE_MODEL: frames that fell back to the ray-casts because the live mesh could not be built (the first one reported on stderr),
 * DF_KINFU_RELOCALISE (0 without it): [13] 1 while tracking is lost, [14] lost frames so far, [15] relocalisations so far (a loss that
 * ended), [16] keyframes held.  A tracked frame's launch count [5] includes df_fern_encode, df_icp_inliers and df_fern_match.  Counters [14]
 * and [15] count over the object's life, as [6] does. */
int df_kinfu_get_info(void *kinfu, long long *info_host, int n);
/* DF_KINFU_RELOCALISE: the keyframe database -- *n = the entries held; the first min(*n, capacity) poses (12 floats each, as
 * df_kinfu_get_pose) into poses_host and codes (DF_RELOC_FERNS bytes each) into codes_host (either may be NULL).  An object without the
 * flag: cudaErrorInvalidValue.  Synchronous. */
int df_kinfu_get_keyframes(void *kinfu, float *poses_host, uint8_t *codes_host, int capacity, int *n);
/* device buffers of the current state, the `which` of df_kinfu_get_buffer / _read_buffer */
#define DF_KINFU_BUF_VOLUME 0              /* the TSDF volume (u32) */
#define DF_KINFU_BUF_DISTS 1
#define DF_KINFU_BUF_CURR_DEPTH 2          /* the current frame's depth, points and normals (ICP level 0) */
#define DF_KINFU_BUF_CURR_POINTS 3
#define DF_KINFU_BUF_CURR_NORMALS 4
#define DF_KINFU_BUF_PREV_POINTS 5         /* the previous frame's points and normals (ICP level 0) */
#define DF_KINFU_BUF_PREV_NORMALS 6
#define DF_KINFU_BUF_CANONICAL 7           /* after the 2nd warp */
#define DF_KINFU_BUF_CANONICAL_NORMALS 8
#define DF_KINFU_BUF_CLOUD 9               /* the extracted cloud and its normals */
#define DF_KINFU_BUF_CLOUD_NORMALS 10
#define DF_KINFU_BUF_NODES 11
#define DF_KINFU_BUF_CANONICAL_VISIBLE 12
#define DF_KINFU_BUF_SOLVE_STATS 13        /* solver stats (8 doubles) */
#define DF_KINFU_BUF_ACTIVITY 14           /* activity map (bytes) */
#define DF_KINFU_BUF_F2_STATS 15           /* df_solve_f2 stats (16 doubles, DF_KINFU_F2_SOLVE) */
#define DF_KINFU_BUF_COLOR_VOLUME 16       /* colour volume (u32 R, G, B, W); DF_KINFU_COLOR only */
#define DF_KINFU_BUF_CLOUD_COLORS 17       /* the cloud's colours (u32 R, G, B, A per cloud slot); DF_KINFU_COLOR only */
#define DF_KINFU_BUF_COLOR_MAP 18          /* the occlusion map of the last colour frame (u32 words, df_color_depth_map), only while a colour
                                              camera is set */
#define DF_KINFU_BUF_INTENSITY 19          /* the frame's intensity (float, df_frame_intensity); DF_KINFU_COLOR_TRACKING only */
#define DF_KINFU_BUF_MODEL_INTENSITY 20    /* the model's intensity maps (float4 (I, gu, gv, 0), df_model_intensity); DF_KINFU_COLOR_TRACKING only */
/* a DF_KINFU_BUF_* buffer; one the object does not have: cudaErrorInvalidValue.  The ICP's pyramid levels: which + 256 * level (level < the
 * used ICP levels) for DF_KINFU_BUF_CURR_DEPTH .. DF_KINFU_BUF_PREV_NORMALS, DF_KINFU_BUF_INTENSITY and DF_KINFU_BUF_MODEL_INTENSITY gives
 * level `level` of that buffer (level 0 is the buffer itself), at its own size */
int df_kinfu_get_buffer(void *kinfu, int which, void **ptr, size_t *pitch, int *cols, int *rows);
/* synchronous device-to-host copy of one of those buffers (diagnostics / tests), at most `bytes` bytes */
int df_kinfu_read_buffer(void *kinfu, int which, void *dst_host, size_t bytes);
/* Lock-step parity hook (tests; never used by the frame loop's callers): one-shot replacements for the NEXT df_kinfu_process_* call.
 * Each non-NULL argument replaces the corresponding intermediate result of that frame, so that everything downstream can be compared
 * with a CPU run of the same frame BIT FOR BIT instead of statistically:
 *   bilateral_depth_host  cols x rows u16: used instead of this frame's bilateral filter output (CUDA expf vs glibc expf: +-1 LSB);
 *   pose12_host           absolute camera pose of the frame (R row-major, t): used instead of poses.back() * ICP(affine); ICP is skipped;
 *   nodes_host            M x DF_NODE_STRIDE floats: the node table after the data-term solve (ignored unless M equals the loop's node count).
 * NULL = compute as usual. */
int df_kinfu_set_overrides(void *kinfu, const uint16_t *bilateral_depth_host, size_t pitch, const float *pose12_host, const float *nodes_host, int M);
/* parameters of the DF_KINFU_F2_SOLVE variant of the frame loop */
int df_kinfu_set_f2_params(void *kinfu, const df_f2_params *params);
/* digest of the current state (multi-GPU correctness record, SURVEY 8e: ranks exchange it and rank 0 compares every rank's with a
 * single-GPU run of the same sequence): out4_host[0] order-independent 64-bit checksum of the packed volume, [1] the same over the node
 * table, [2] extracted cloud points, [3] FNV-style hash of every camera pose so far (bit patterns).  Synchronous. */
int df_kinfu_state_digest(void *kinfu, unsigned long long *out4_host);
/* per-stage milliseconds of the last frame (DF_KINFU_STAGE_TIMING): preprocess, icp, raycast_canonical, warp1, solve,
 * warp2, project_remove, integrate, extract, raycast_prev; returns the number written */
int df_kinfu_get_stage_ms(void *kinfu, float *ms_host, int n);

/* Snapshots: save the whole state of the frame loop to host memory and resume it later, in another process or on another device.  Run
 * frames 0..k, save, load into an object created with the same parameters, run frames k+1..n: after every frame the state equals that
 * of an uninterrupted run bit for bit (DF_KINFU_F2_SOLVE: to the last bits of its double atomics, DESIGN 4).
 *
 * Format (version 1), one little-endian byte string:
 *   header      32 bytes: magic "DFUSNAP\0", u32 version = 1, u32 header length = 32, u64 total length, u64 checksum of every byte after the
 *               header (c = n + sum over the zero-padded u64 words w_i of splitmix64(w_i ^ i * 0x9e3779b97f4a7c15), mod 2^64)
 *   params      df_kinfu_params (byte copy, environment-set flags included), then df_f2_params
 *   counters    i32 frame_counter, resets, last_ok, M, cloud_count, n_poses; i64 solve_overflows; u64 payload_bytes
 *   poses       n_poses x 12 floats (the pose chain since the last reset)
 *   nodes       M x DF_NODE_STRIDE floats
 *   activity    df_volume_activity_bytes(volume) bytes, verbatim
 *   pyramids    for each used ICP level l (dense rows, (cols >> l) x (rows >> l)): the previous frame's points (float4) -- depth (u16) under
 *               DF_KINFU_USE_DEPTH -- then its normals (float4)
 *   cloud       cloud_count float4 points, then cloud_count float4 normals (stored: under DF_KINFU_RIGID_ONLY it is frame 0's cloud)
 *   volume      df_volume_brick_count(volume) class bytes, then payload_bytes of payload (df_volume_pack_count / _emit)
 * Version 2 is what an object with DF_KINFU_COLOR writes (without the flag a snapshot is version 1, byte for byte as above): version 1 with
 * u32 version = 2, followed by
 *   colour      u64 colour payload length, df_volume_brick_count(volume) class bytes, then that many payload bytes: the colour volume through
 *               df_volume_pack_count / _emit
 *   colours     cloud_count u32 R, G, B, A words: the cloud's colours
 * Version 3 is what a colour object with a colour camera writes (df_kinfu_set_color_camera; without one it writes version 2, byte for byte as
 * above): version 2 with u32 version = 3, followed by
 *   camera      the 72-byte df_color_camera record (byte copy)
 * The version must match the colour flag of the stored params.  The colour bricks' class bytes and payload length are checked on the host
 * (the rule of df_volume_unpack), by df_kinfu_snapshot_params as well, so that a load can refuse before it writes either volume; so is the
 * camera record (df_color_map_dims' rule).  A load also requires the object's colour camera to equal the record byte for byte (no record:
 * no camera set).
 * Version 4 is what an object with a lens writes (df_kinfu_set_depth_lens / _set_color_lens; without one it writes version 1, 2 or 3,
 * byte for byte as above): the content of the version its flags and camera give, with u32 version = 4, followed by
 *   lenses      u8 depth lens present, the 36-byte df_lens record; u8 colour lens present, its record (a record that is not present is
 *               36 zero bytes)
 * Whether a version-4 snapshot of a colour object holds the camera record follows from its length (72 bytes).  A present record passes
 * df_lens_check and is not the zero lens; at least one is present; a colour lens needs the camera record.  A load also requires the
 * object's lenses to equal the records byte for byte (no record: no lens set).
 * Version 5 is what an object with DF_KINFU_RELOCALISE writes (without the flag it writes version 1 to 4, byte for byte as above): the
 * content of the version its flags, camera and lenses give, with u32 version = 5, followed by
 *   relocaliser u32 base version (the 1 to 4 the content has), u8 lost, 3 zero bytes, i64 lost frames, i64 relocalisations, u64 fern seed
 *               (DF_RELOC_SEED), i32 keyframe count, i32 ferns (DF_RELOC_FERNS); count x DF_RELOC_FERNS code bytes; count x 12 pose floats;
 *               u64 the section's length, these 8 bytes included (so a reader finds the section from the end)
 * The last good pose is the pose chain's last entry.  Version 5 must match the flag of the stored params both ways; a section that is
 * truncated, has another seed or fern count, more keyframes than DF_RELOC_KEYFRAMES, or a length its count does not give is rejected.
 * The node grid is rebuilt on load.  Per-frame scratch is not stored: dists, the current-frame images and pyramids, the canonical maps,
 * the solver statistics and workspaces hold undefined contents after a load until the next frame writes them.
 *
 * df_kinfu_save: the snapshot into dst_host (capacity bytes); *bytes_out (optional) = its length.  dst_host == NULL: size query only.
 *   capacity too small: cudaErrorInvalidValue.  Completes the last frame's extraction first; device staging of the packed volume only.
 * df_kinfu_load: all-or-nothing.  Checks magic, version, lengths, checksum, byte equality of the params with the object's, the node and
 *   cloud counts against its capacities, then (on the device, df_volume_unpack) the brick classes and payload length, before it changes
 *   anything; any failure returns cudaErrorInvalidValue (reason on stderr) and leaves the object as it was.  Writes into the object's
 *   existing allocations (pointers from df_kinfu_get_buffer stay valid); no extraction is owed afterwards.
 * df_kinfu_snapshot_params: host only -- validates the header, checksum and section lengths and returns the params, so that a caller can
 *   create a matching object before loading.
 * df_kinfu_snapshot_color_camera: host only -- the same checks; *present = 1 and *cam (may be NULL) = the record of a version-3 snapshot,
 *   else *present = 0 and *cam zeroed, so that a caller can set the same camera on that object before loading.
 * df_kinfu_snapshot_lenses: host only -- the same checks; *depth_present / *color_present and the records (either pointer may be NULL) of
 *   a version-4 snapshot's lenses, else 0 and zeroed records, so that a caller can set the same lenses before loading.
 * All return 0 or a cudaError_t value; save and load work on the object's stream and synchronise before returning. */
int df_kinfu_save(void *kinfu, void *dst_host, size_t capacity, size_t *bytes_out);
int df_kinfu_load(void *kinfu, const void *src_host, size_t bytes);
int df_kinfu_snapshot_params(const void *src_host, size_t bytes, df_kinfu_params *params);
int df_kinfu_snapshot_color_camera(const void *src_host, size_t bytes, df_color_camera *cam, int *present);
int df_kinfu_snapshot_lenses(const void *src_host, size_t bytes, df_lens *depth, int *depth_present, df_lens *color, int *color_present);

/* Mesh of the reconstruction (df_mesh_count / _emit over the object's volume and its extracted cloud).  live = 0: the canonical model,
 * vertices = the cloud's xyz, normals = the cloud's normals (df_extract_normals; NaN where it gives none).  live = 1: the same points and
 * normals carried through the warp field by the frame loop's own call (df_warp, warp_to_live = identity, flags 0); fails
 * (cudaErrorInvalidValue) when the object has fewer than 8 nodes.  Every cloud point is a vertex, referenced or not, so face indices are cloud
 * indices and the canonical and live meshes share their faces.
 *   verts_host / normals_host: n_verts x 3 floats; tris_host: n_tris x 3 int32 (host memory).  verts_host == NULL: size query only
 *   (*n_verts, *n_tris).  normals_host may be NULL.  A capacity (vertices, triangles) below the size: cudaErrorInvalidValue.  The last
 *   frame's extraction is completed first; a cloud that does not match the volume (truncated at cloud_capacity, or not re-extracted since
 *   the volume changed, as under DF_KINFU_RIGID_ONLY after the first frame): cudaErrorInvalidValue (reason on stderr).  A failed call writes
 *   nothing.  The call reads the volume, the cloud and the nodes and changes no state; the device workspace is allocated on the first call.
 *   Runs on the object's stream and synchronises before returning. */
int df_kinfu_mesh(void *kinfu, int live, float *verts_host, float *normals_host, int32_t *tris_host, int vert_capacity, int tri_capacity,
                  int *n_verts, int *n_tris);

/* Render the mesh df_kinfu_mesh(live) returns, built on the device the same way, with df_raster_mesh into cols x rows device maps (the
 * object's params; pitches as df_raster_mesh requires): points_dev / normals_dev float4 in the virtual camera's frame, tri_ids_dev (may be
 * NULL) int32 cloud-mesh triangle indices.  pose12_host: the virtual camera's camera-to-model pose, 12 floats as df_kinfu_get_pose returns them; the renderer applies its
 * inverse.  NULL = the model's own camera: for the canonical model the latest camera pose (what the ray-cast of the frame loop shows); for
 * the live model the identity, because the live model's coordinates ARE the current camera's: the warp is solved so that
 * warp(pose^-1 * p_cam) matches the current depth's camera-frame points (the reference's KinFu::dynamicfusion, DESIGN 5.7).
 * Fails where df_kinfu_mesh fails (live with fewer than 8 nodes, a cloud that does not match the volume) and then writes nothing.  Changes
 * no state (state digest, launch count); the triangle buffer, the live copy and the raster workspace are allocated on first use and grown
 * when too small.  Runs on the object's stream and synchronises before returning; returns 0 or a cudaError_t value. */
int df_kinfu_render(void *kinfu, int live, const float *pose12_host, int32_t *tri_ids_dev, size_t tri_pitch, float *points_dev,
                    size_t points_pitch, float *normals_dev, size_t normals_pitch);

/* DF_KINFU_COLOR: the vertex colours of df_kinfu_mesh, one u32 (bytes R, G, B, A; A = 255 coloured, else the word is 0) per vertex, in
 * vertex order: the cloud's colours, so they serve the canonical and the live mesh alike.  rgba_host == NULL: size query (*n).  A capacity
 * below the size, or an object without the flag: cudaErrorInvalidValue.  Completes the last frame's extraction first; synchronous. */
int df_kinfu_mesh_colors(void *kinfu, uint32_t *rgba_host, int capacity, int *n);

/* DF_KINFU_COLOR: df_kinfu_render's device sequence into maps the object keeps, followed by df_mesh_colors with the cloud's colours: the
 * coloured picture of the canonical or the live (warped) model.  image_dev: device, rows x cols BGRA pixels in df_render_image's layout,
 * pitch in bytes (at least cols * 4, a multiple of 4); 0 where nothing is drawn or the surface has no colour.  live and pose12_host as
 * df_kinfu_render; fails where it fails, and on an object without the flag.  Changes no state; synchronises before returning. */
int df_kinfu_render_colors(void *kinfu, int live, const float *pose12_host, void *image_dev, size_t pitch);

#ifdef __cplusplus
}
#endif
#endif /* DFUSION_H */
