// pipeline.cu -- the per-frame DynamicFusion loop, device-resident, behind the C ABI (df_kinfu_*).
// Mirrors kfusion::KinFu (kfusion/include/kfusion/kinfu.hpp:49-97, kfusion/src/kinfu.cpp): same stage order, buffer swaps,
// first-frame special case and pose chaining.  What changes is where the data lives: the reference's
// KinFu::dynamicfusion (kinfu.cpp:344-400) downloads three 4.9 MB maps, runs ~1 M CPU k-NN queries, re-uploads, and
// syncs ~25 times a frame; here the frame touches the host exactly once (ICP status + 12-float pose, needed for the
// return value) and everything else is stream-ordered kernels on one stream.
#include "kinfu_object.cuh"
#include "lens.cuh"
#include "../../include/df_hostmath.h"
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <thread>

using namespace dfb;
using namespace dfb::kinfu;

namespace {

int node_capacity(const df_kinfu_params &p) { return p.max_nodes > 0 ? p.max_nodes : (p.cloud_capacity + 49) / 50; }
// a colour frame is tracked with its photometric rows as well (DF_KINFU_COLOR_TRACKING)
bool color_tracked(const KinFu &k) { return (k.p.flags & DF_KINFU_COLOR_TRACKING) && k.frame_bgra; }

// canonical[i] = inverse_pose * cloud[i]: cv::Affine3f * Vec3f, m0*x + m1*y + m2*z + m3 left to right (kinfu.cpp:356-362);
// NaN pixels stay NaN.  Also writes the `canonical_visible` copy (kinfu.cpp:383).
__global__ void __launch_bounds__(256) to_canonical_kernel(const float4 *src, Aff inv_pose, float4 *dst, float4 *dst_copy, int n)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = src[i];
    float4 o;
    o.x = inv_pose.r0.x * v.x + inv_pose.r0.y * v.y + inv_pose.r0.z * v.z + inv_pose.t.x;
    o.y = inv_pose.r1.x * v.x + inv_pose.r1.y * v.y + inv_pose.r1.z * v.z + inv_pose.t.y;
    o.z = inv_pose.r2.x * v.x + inv_pose.r2.y * v.y + inv_pose.r2.z * v.z + inv_pose.t.z;
    o.w = v.w;
    dst[i] = o;
    dst_copy[i] = o;
}

// WarpField::init (warp_field.cpp:41-62): every `step`-th extracted point becomes a node with the identity
// DualQuaternion() (rotation (1,0,0,0), dual part (1,0,0,0)) and weight 3 * voxel_size with voxel_size forced to 1.
__global__ void __launch_bounds__(256) init_nodes_kernel(const float4 *cloud, int step, int M, float *nodes)
{
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const float4 p = cloud[(size_t)m * step];
    float *n = nodes + (size_t)m * DF_NODE_STRIDE;
    n[0] = p.x; n[1] = p.y; n[2] = p.z;
    n[3] = 1.f; n[4] = 0.f; n[5] = 0.f; n[6] = 0.f;
    n[7] = 1.f; n[8] = 0.f; n[9] = 0.f; n[10] = 0.f;
    n[11] = 3.f;
}

// DF_KINFU_RELOCALISE, a keyframe's relocalisation: every node's transform back to init_nodes_kernel's identity; position and weight kept
__global__ void __launch_bounds__(256) identity_transforms_kernel(int M, float *nodes)
{
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    float *n = nodes + (size_t)m * DF_NODE_STRIDE;
    n[3] = 1.f; n[4] = 0.f; n[5] = 0.f; n[6] = 0.f;
    n[7] = 1.f; n[8] = 0.f; n[9] = 0.f; n[10] = 0.f;
}

// order-independent 64-bit checksum of a u32 array: sum over i of mix(i, a[i]) (splitmix64 finaliser); one u64 atomicAdd per block
__global__ void __launch_bounds__(256) digest_kernel(const uint32_t *__restrict__ a, size_t n, unsigned long long *out)
{
    unsigned long long acc = 0ull;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        unsigned long long z = ((unsigned long long)a[i] << 32) ^ (unsigned long long)i;
        z += 0x9e3779b97f4a7c15ull;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        acc += z ^ (z >> 31);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

// the extraction itself (compute_points + compute_normals, tsdf_volume.cpp:313-325) on stream `es`
int run_extract(KinFu &k, cudaStream_t es)
{
    const df_kinfu_params &p = k.p;
    const df_volume vol = vol_of(k);
    CK(df_extract_cloud_tracked(vol, p.volume_pose, k.cloud, p.cloud_capacity, k.cloud_count, k.extract_ws, k.activity, es));
    k.last_cloud = -1;
    CK(df_extract_normals(vol, k.cloud, p.cloud_capacity, k.cloud_count, p.volume_pose, k.Rinv_vol, p.gradient_delta_factor, k.cloud_nrm, es));
    if (!color_on(k)) return 0;
    // the cloud's colours: the extraction puts voxel i at (i + 1/2) * vs, hence the offset
    return df_sample_colors(vol, k.color_vol, p.volume_pose, 0.5f, k.cloud, 0, 4, p.cloud_capacity, 1, k.cloud_count, k.cloud_rgba, 0, es);
}

// start the deferred extraction on the auxiliary stream once `after` (an event of the main stream) has happened
int launch_deferred_extract(KinFu &k, cudaEvent_t after)
{
    if (!k.extract_deferred) return 0;
    k.extract_deferred = false;
    if (cudaStreamWaitEvent(k.aux, after, 0) != cudaSuccess) return (int)cudaGetLastError();
    if (int st = run_extract(k, k.aux)) return st;
    if (cudaEventRecord(k.ev_extract_done, k.aux) != cudaSuccess) return (int)cudaGetLastError();
    k.extract_pending = true;
    return 0;
}

// the main stream may not write the volume / activity map / cloud buffers while an extraction is still owed or in flight
int wait_extract_on_main(KinFu &k)
{
    if (k.extract_deferred) {
        if (cudaEventRecord(k.ev_volume_ready, k.stream) != cudaSuccess) return (int)cudaGetLastError();
        if (int st = launch_deferred_extract(k, k.ev_volume_ready)) return st;
    }
    if (!k.extract_pending) return 0;
    k.extract_pending = false;
    return (int)cudaStreamWaitEvent(k.stream, k.ev_extract_done, 0);
}

void mark(KinFu &k, int stage)
{
    if (k.p.flags & DF_KINFU_STAGE_TIMING) cudaEventRecord(k.ev[stage], k.stream);
    k.stage_mark[stage] = 1;
}

int do_reset(KinFu &k)
{
    if (k.frame_counter) { printf("Reset\n"); ++k.resets; }          // kinfu.cpp:198-199
    k.frame_counter = 0;
    k.M = 0;                                                         // warp_->clear(), kinfu.cpp:206: the next first frame re-initialises the field
    k.lm_valid = false;
    k.poses.clear();
    k.poses.resize(12);
    dfh_aff_identity(k.poses.data());
    if (int w = wait_extract_on_main(k)) return w;
    if (k.activity && cudaMemsetAsync(k.activity, 0, k.activity_bytes, k.stream) != cudaSuccess) return (int)cudaGetLastError();
    if (color_on(k)) CK(df_clear_volume(color_vol_of(k), k.stream));
    if (reloc_on(k)) {                                               // the keyframe database empties and a loss ends
        k.lost = false;
        CK(cudaMemsetAsync(k.kf_count, 0, sizeof(int), k.stream));
    }
    return df_clear_volume(vol_of(k), k.stream);
}

// per-frame bookkeeping at the start of df_kinfu_process_* and df_kinfu_dynamicfusion: launch count and stage marks start afresh
void begin_frame(KinFu &k)
{
    k.launches = 0;
    k.lm_fell_back = false;
    memset(k.stage_mark, 0, sizeof k.stage_mark);
    mark(k, 0);
}

static inline double now_us() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int integrate_rigid(KinFu &k, const float *cam_pose)
{
    const df_kinfu_params &p = k.p;
    const df_volume vol = vol_of(k);
    float inv[12], vol2cam[12];
    dfh_aff_inv(cam_pose, inv);
    dfh_aff_mul(inv, k.vol_pose, vol2cam);                             // camera_pose.inv() * pose_, tsdf_volume.cpp:112
    k.launches += df_integrate_launch_count(vol);
    unsigned long long *counter = (p.flags & DF_KINFU_STAGE_TIMING) ? k.n_upd.p : nullptr;
    if (counter) cudaMemsetAsync(counter, 0, 8, k.stream);
    if (int w = wait_extract_on_main(k)) return w;                     // write-after-read: the previous frame's extraction reads this volume
    CK(df_integrate_tracked(vol, (const uint16_t *)k.dists.ptr, k.dists.pitch, p.cols, p.rows, to_aff(vol2cam), p.intr, counter, k.activity,
                            k.integrate_ws, k.stream));
    if (!k.frame_bgra) return 0;
    ++k.launches;                                                      // the frame's colours, where the same dists show the surface
    if (k.has_cam)
        return df_integrate_color_camera_lens(vol, k.color_vol, (const uint16_t *)k.dists.ptr, k.dists.pitch, p.cols, p.rows, to_aff(vol2cam), p.intr,
                                              k.cam, color_lens_of(k), k.frame_bgra, k.frame_bgra_pitch, (const uint32_t *)k.color_map.ptr,
                                              k.color_map.pitch, k.activity, k.stream);
    return df_integrate_color(vol, k.color_vol, (const uint16_t *)k.dists.ptr, k.dists.pitch, k.frame_bgra, k.frame_bgra_pitch, p.cols, p.rows,
                              to_aff(vol2cam), p.intr, k.activity, k.stream);
}

// pose_.inv() * camera_pose, tsdf_volume.cpp:162: a point of the camera's frame in the volume's
void cam2vol_of(const KinFu &k, const float *cam_pose, float *cam2vol)
{
    float inv[12];
    dfh_aff_inv(k.vol_pose, inv);
    dfh_aff_mul(inv, cam_pose, cam2vol);
}

int raycast_model(KinFu &k, const float *cam_pose, Img &pts, Img &nrm)
{
    const df_kinfu_params &p = k.p;
    float cam2vol[12], Rinv[9];
    cam2vol_of(k, cam_pose, cam2vol);
    dfh_mat3_inv(cam2vol, Rinv);
    ++k.launches;
    // the loop's own volume is only ever integrated through the activity map, so the march may skip the bricks without negative voxels
    return df_raycast_points_tracked(vol_of(k), to_aff(cam2vol), Rinv, p.intr, p.cols, p.rows, p.raycast_step_factor, p.gradient_delta_factor,
                                     (float *)pts.ptr, pts.pitch, (float *)nrm.ptr, nrm.pitch, k.activity.p, k.stream);
}

// compute_points + compute_normals, tsdf_volume.cpp:313-325.  needed_now: the caller reads the cloud right after (first frame: node
// initialisation; field extension): stay on the main stream
int extract_cloud(KinFu &k, bool needed_now)
{
    k.launches += 5 + color_on(k);                                     // count, 2 scans, emit + the normals kernel (+ the cloud's colours)
    const bool overlap = k.overlap_extract && !needed_now && !(k.p.flags & DF_KINFU_STAGE_TIMING);
    if (int w = wait_extract_on_main(k)) return w;                     // an older extraction may still own the cloud buffers
    if (!overlap) return run_extract(k, k.stream);
    k.extract_deferred = true;                                         // launched when the next frame's LM/PCG kernel starts, or on demand
    k.last_cloud = -1;
    return 0;
}

int extend_field(KinFu &k)                                             // SURVEY 8f(3) / Report.md step 4, DF_KINFU_EXTEND_FIELD
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    if (!(p.flags & DF_KINFU_EXTEND_FIELD) || k.M <= 0 || k.M >= k.max_nodes_cap) return 0;
    CK(df_extend_field(k.nodes, k.M, k.max_nodes_cap, k.node_grid, k.cloud, p.cloud_capacity, k.cloud_count, 4,
                       p.extend_radius > 0 ? p.extend_radius : 0.03f, p.node_step > 0 ? p.node_step : 50, k.M_dev, k.extend_ws, s));
    k.launches += 3;
    int Mn = k.M;
    if (cudaMemcpyAsync(&Mn, k.M_dev, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess) return (int)cudaGetLastError();
    if (cudaStreamSynchronize(s) != cudaSuccess) return (int)cudaGetLastError();
    if (Mn == k.M) return 0;
    k.M = Mn;
    ++k.launches;
    return df_build_node_grid(k.nodes, k.M, k.node_grid, s);           // buildKDTree() after the node set changed
}

// a pyramid as the parallel per-level arrays of the ICP and intensity ABIs (df_icp_estimate*, df_frame_intensity, df_model_intensity)
template <class T> struct Levels {
    T *ptr[MAX_LEVELS]; size_t pitch[MAX_LEVELS]; int cols[MAX_LEVELS], rows[MAX_LEVELS];
    Levels(const Img (&im)[MAX_LEVELS], int n)
    {
        for (int i = 0; i < n; ++i) { ptr[i] = (T *)im[i].ptr; pitch[i] = im[i].pitch; cols[i] = im[i].cols; rows[i] = im[i].rows; }
    }
};

// ---- pre-processing, kinfu.cpp:226-242 ---------------------------------------------------------------------------
int preprocess(KinFu &k, const uint16_t *depth_dev, size_t depth_pitch)
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    CK(df_compute_dists(depth_dev, depth_pitch, p.cols, p.rows, p.intr, (uint16_t *)k.dists.ptr, k.dists.pitch, s));
    if (k.frame_bgra && k.has_cam) {                                   // the colour camera's view of the whole input frame
        CK(df_color_depth_map_lens(depth_dev, depth_pitch, p.cols, p.rows, p.intr, k.cam, color_lens_of(k), (uint32_t *)k.color_map.ptr,
                                   k.color_map.pitch, s));
        ++k.launches;
    }
    if (k.has_ov_depth) {              // lock-step parity hook: the caller's bilateral image instead of this frame's (expf differs by 1 LSB between CUDA and glibc)
        CK(cudaMemcpy2DAsync(k.cur_depth[0].ptr, k.cur_depth[0].pitch, k.ov_depth.data(), (size_t)p.cols * 2, (size_t)p.cols * 2, p.rows, cudaMemcpyHostToDevice, s));
        CK(cudaStreamSynchronize(s));  // the host vector may be replaced right after the call
        k.has_ov_depth = false;
        ++k.launches;
    } else {
        CK(df_bilateral(depth_dev, depth_pitch, p.cols, p.rows, (uint16_t *)k.cur_depth[0].ptr, k.cur_depth[0].pitch,
                        p.bilateral_kernel_size, p.bilateral_sigma_spatial, p.bilateral_sigma_depth, s));
        k.launches += 2;
    }
    if (p.icp_truncate_depth_dist > 0) {
        CK(df_truncate_depth((uint16_t *)k.cur_depth[0].ptr, k.cur_depth[0].pitch, p.cols, p.rows, p.icp_truncate_depth_dist, s));
        ++k.launches;
    }
    for (int i = 1; i < k.levels; ++i) {
        CK(df_pyr_down((const uint16_t *)k.cur_depth[i - 1].ptr, k.cur_depth[i - 1].pitch, k.cur_depth[i - 1].cols, k.cur_depth[i - 1].rows,
                       (uint16_t *)k.cur_depth[i].ptr, k.cur_depth[i].pitch, p.bilateral_sigma_depth, s));
        ++k.launches;
    }
    const bool use_depth = (p.flags & DF_KINFU_USE_DEPTH) != 0;
    for (int i = 0; i < k.levels; ++i) {
        const int div = 1 << i;                                       // Intr::operator()(level), precomp.cpp:10-14
        const df_intr li = {p.intr.fx / div, p.intr.fy / div, p.intr.cx / div, p.intr.cy / div};
        if (use_depth) {
            // the reference's compile-time USE_DEPTH loop (internal.hpp:6, kinfu.cpp:237-238): normals from the depth map, depth masked
            // where the normal is invalid; the vertex pyramid is not built.  KinFu::dynamicfusion is still handed curr_.points_pyr[0]
            // (kinfu.cpp:284-287), which that build never writes; here it receives what the variable is meant to hold: the vertex map of
            // the level-0 depth (computed before the masking, normals to a scratch map) -- documented divergence, DESIGN 5.
            if (i == 0) {
                CK(df_points_normals(li, (const uint16_t *)k.cur_depth[0].ptr, k.cur_depth[0].pitch, k.cur_depth[0].cols, k.cur_depth[0].rows,
                                     (float *)k.cur_pts[0].ptr, k.cur_pts[0].pitch, (float *)k.canon_nrm.ptr, k.canon_nrm.pitch, s));
                ++k.launches;
            }
            CK(df_normals_mask_depth(li, (uint16_t *)k.cur_depth[i].ptr, k.cur_depth[i].pitch, k.cur_depth[i].cols, k.cur_depth[i].rows,
                                     (float *)k.cur_nrm[i].ptr, k.cur_nrm[i].pitch, s));
        } else
        CK(df_points_normals(li, (const uint16_t *)k.cur_depth[i].ptr, k.cur_depth[i].pitch, k.cur_depth[i].cols, k.cur_depth[i].rows,
                             (float *)k.cur_pts[i].ptr, k.cur_pts[i].pitch, (float *)k.cur_nrm[i].ptr, k.cur_nrm[i].pitch, s));
        ++k.launches;
    }
    if (color_tracked(k)) {
        // the colour frame's intensity pyramid for the photometric ICP rows; through the colour camera its level 0 is looked up from the
        // vertex map above, with the occlusion map built at the top of this function
        const Levels<float> out(k.cur_int, k.levels);
        CK(df_frame_intensity_lens(k.frame_bgra, k.frame_bgra_pitch, k.has_cam ? &k.cam : nullptr, color_lens_of(k), p.intr, (const float *)k.cur_pts[0].ptr,
                                   k.cur_pts[0].pitch, (const uint32_t *)k.color_map.ptr, k.color_map.pitch, k.trunc_dist, k.levels, out.cols, out.rows,
                                   out.ptr, out.pitch, s));
        k.launches += k.levels;
    }
    if (reloc_on(k)) {                                                 // the frame's fern code, for the harvest and the lookup
        const Img &d2 = k.cur_depth[2];
        CK(df_fern_encode((const uint16_t *)d2.ptr, d2.pitch, d2.cols, d2.rows, k.fern_table, DF_RELOC_FERNS, k.frame_code, s));
        ++k.launches;
    }
    mark(k, 1);
    return 0;
}

// ---- first frame, kinfu.cpp:245-264 --------------------------------------------------------------------------------
int first_frame(KinFu &k)
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    CK(integrate_rigid(k, latest_pose(k)));
    CK(extract_cloud(k, true));
    if (!(p.flags & DF_KINFU_RIGID_ONLY)) {
        int count = 0;
        CK(cudaMemcpyAsync(&count, k.cloud_count, sizeof(int), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        k.last_cloud = count;
        int step = p.node_step > 0 ? p.node_step : 50;
        int M = (count + step - 1) / step;
        if (p.max_nodes > 0 && M > p.max_nodes) { step = (count + p.max_nodes - 1) / p.max_nodes; M = (count + step - 1) / step; }
        k.M = M;
        if (M > 0) {
            init_nodes_kernel<<<div_up(M, 256), 256, 0, s>>>((const float4 *)k.cloud.p, step, M, k.nodes);
            CK(df_build_node_grid(k.nodes, M, k.node_grid, s));        // buildKDTree(), warp_field.cpp:61
            k.launches += 2;
        }
    }
    for (int i = 0; i < MAX_LEVELS; ++i) {                              // kinfu.cpp:253-261
        if (p.flags & DF_KINFU_USE_DEPTH) std::swap(k.cur_depth[i], k.prev_depth[i]);
        else std::swap(k.cur_pts[i], k.prev_pts[i]);
        std::swap(k.cur_nrm[i], k.prev_nrm[i]);
    }
    ++k.frame_counter;
    return 0;
}

// ---- ICP, kinfu.cpp:268-280 (device-resident; one host read of {ok, T}), or the pose of df_kinfu_set_overrides --------
// the ICP of the current pyramid against the previous-frame maps, into icp_T / icp_ok (no host read)
int launch_icp(KinFu &k)
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    const Levels<float> vc(k.cur_pts, k.levels), nc(k.cur_nrm, k.levels), vp(k.prev_pts, k.levels), np(k.prev_nrm, k.levels);
    if (p.flags & DF_KINFU_USE_DEPTH) {                                // estimateTransform(depth pyramids), kinfu.cpp:271
        const Levels<unsigned short> dc(k.cur_depth, k.levels), dp(k.prev_depth, k.levels);
        CK(df_icp_estimate_depth(dc.ptr, nc.ptr, dp.ptr, np.ptr, vc.cols, vc.rows, dc.pitch, nc.pitch, k.levels, p.icp_iter_num, p.intr,
                                 p.icp_dist_thres, p.icp_angle_thres, k.icp_T, k.icp_ok, k.icp_scratch, s));
    } else if (color_tracked(k)) {
        // DF_KINFU_COLOR_TRACKING: the model's intensity maps at the previous vertex maps, seen from poses.back(), then the ICP with
        // the photometric rows
        float cam2vol[12];
        cam2vol_of(k, latest_pose(k), cam2vol);
        const Levels<float> ic(k.cur_int, k.levels), mo(k.model_int, k.levels);
        CK(df_model_intensity(vol_of(k), k.color_vol, to_aff(cam2vol), k.levels, vc.cols, vc.rows, vp.ptr, vp.pitch, mo.ptr, mo.pitch, s));
        ++k.launches;
        CK(df_icp_estimate_color(vc.ptr, nc.ptr, vp.ptr, np.ptr, ic.ptr, ic.pitch, mo.ptr, mo.pitch, vc.cols, vc.rows, vc.pitch, k.levels,
                                 p.icp_iter_num, p.intr, p.icp_dist_thres, p.icp_angle_thres, DF_COLOR_TRACK_WEIGHT,
                                 DF_COLOR_TRACK_MAX_RESIDUAL, k.icp_T, k.icp_ok, k.icp_scratch, s));
    } else
    CK(df_icp_estimate(vc.ptr, nc.ptr, vp.ptr, np.ptr, vc.cols, vc.rows, vc.pitch, k.levels, p.icp_iter_num, p.intr, p.icp_dist_thres, p.icp_angle_thres,
                       k.icp_T, k.icp_ok, k.icp_scratch, s));
    for (int i = 0; i < k.levels; ++i) k.launches += 2 * p.icp_iter_num[i];
    ++k.launches;
    return 0;
}

// ---- DF_KINFU_RELOCALISE (rules in include/dfusion.h) ---------------------------------------------------------------------------------
// the gate on the ICP result in icp_T / icp_ok against the level-0 maps (pts, nrm), and its copy home (T and ok ride in it)
int launch_gate(KinFu &k, const Img &pts, const Img &nrm)
{
    const df_kinfu_params &p = k.p;
    CK(df_icp_inliers((const float *)k.cur_pts[0].ptr, k.cur_pts[0].pitch, (const float *)k.cur_nrm[0].ptr, k.cur_nrm[0].pitch, (const float *)pts.ptr,
                      pts.pitch, (const float *)nrm.ptr, nrm.pitch, p.cols, p.rows, p.intr, k.icp_T, k.icp_ok, p.icp_dist_thres, p.icp_angle_thres,
                      k.gate, k.gate_ws, k.stream));
    ++k.launches;
    CK(cudaMemcpyAsync(k.gate_host, k.gate, sizeof(df_reloc_gate), cudaMemcpyDeviceToHost, k.stream));
    return 0;
}

// the match of the frame's code against the database; append: the harvest rule with the frame's accepted pose
int launch_match(KinFu &k, int append, const float *pose)
{
    ++k.launches;
    return df_fern_match(k.kf_codes, k.kf_poses, k.kf_count, DF_RELOC_KEYFRAMES, k.frame_code, DF_RELOC_FERNS, append, to_aff(pose), k.match,
                         k.stream);
}

// a lost frame's keyframe candidates, in lookup order: the canonical volume ray-cast from the keyframe's pose into rl_pts / rl_nrm, the
// geometric ICP against them, the gate.  accepted: one passed, and pose is its keyframe pose * T
int try_keyframes(KinFu &k, float *pose, bool &accepted)
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    CK(launch_match(k, 0, latest_pose(k)));
    CK(cudaMemcpyAsync(k.match_host, k.match, sizeof(df_reloc_match), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const df_reloc_match m = *k.match_host;
    for (int c = 0; c < DF_RELOC_CANDIDATES && m.index[c] >= 0; ++c) {
        const float *kf = m.pose[c];
        CK(raycast_model(k, kf, k.rl_pts[0], k.rl_nrm[0]));
        for (int i = 1; i < k.levels; ++i) {
            CK(df_resize_points_normals((const float *)k.rl_pts[i - 1].ptr, k.rl_pts[i - 1].pitch, (const float *)k.rl_nrm[i - 1].ptr,
                                        k.rl_nrm[i - 1].pitch, k.rl_pts[i - 1].cols, k.rl_pts[i - 1].rows, (float *)k.rl_pts[i].ptr,
                                        k.rl_pts[i].pitch, (float *)k.rl_nrm[i].ptr, k.rl_nrm[i].pitch, s));
            ++k.launches;
        }
        const Levels<float> vc(k.cur_pts, k.levels), nc(k.cur_nrm, k.levels), vp(k.rl_pts, k.levels), np(k.rl_nrm, k.levels);
        CK(df_icp_estimate(vc.ptr, nc.ptr, vp.ptr, np.ptr, vc.cols, vc.rows, vc.pitch, k.levels, p.icp_iter_num, p.intr, p.icp_dist_thres,
                           p.icp_angle_thres, k.icp_T, k.icp_ok, k.icp_scratch, s));
        for (int i = 0; i < k.levels; ++i) k.launches += 2 * p.icp_iter_num[i];
        ++k.launches;
        CK(launch_gate(k, k.rl_pts[0], k.rl_nrm[0]));
        CK(cudaStreamSynchronize(s));
        k.last_ok = k.gate_host->ok;
        if (!df_reloc_gate_accepts(k.gate_host)) continue;
        dfh_aff_mul(kf, k.gate_host->T, pose);
        accepted = true;
        if (k.M > 0) {                                                 // the field's motion belonged to the lost trajectory
            identity_transforms_kernel<<<div_up(k.M, 256), 256, 0, s>>>(k.M, k.nodes);
            CK(cudaGetLastError());
            ++k.launches;
        }
        k.lm_valid = false;
        return 0;
    }
    return 0;
}

// the ICP and the gate; while lost, the keyframe candidates after it.  accepted = false: the frame is lost (nothing else changes)
int track_reloc(KinFu &k, double &t_sync0, double &t_sync1, float *pose, bool &accepted)
{
    CK(launch_icp(k));                                                 // candidate 0: the ordinary ICP from the last good pose
    CK(launch_gate(k, k.prev_pts[0], k.prev_nrm[0]));
    t_sync0 = now_us();
    CK(cudaStreamSynchronize(k.stream));
    t_sync1 = now_us();
    k.last_ok = k.gate_host->ok;
    note_solve_overflow(k);
    accepted = df_reloc_gate_accepts(k.gate_host) != 0;
    if (accepted) dfh_aff_mul(latest_pose(k), k.gate_host->T, pose);
    else if (k.lost) CK(try_keyframes(k, pose, accepted));
    if (!accepted) {
        if (!k.lost) {
            const df_reloc_gate &g = *k.gate_host;
            fprintf(stderr, "df_kinfu: tracking lost at frame %d (ICP ok %d, %d of %d pixels associated, RMS %.4f m); the model is kept and the "
                            "camera relocalised from keyframes\n", k.frame_counter, g.ok, g.n_in, g.n_valid, g.n_in ? sqrt(g.sum_sq / g.n_in) : 0.0);
        }
        k.lost = true;
        ++k.lost_frames;
        return 0;
    }
    if (k.lost) { k.lost = false; ++k.relocalisations; }
    return 0;
}

// Appends the frame's pose.  ICP failure resets the object (kinfu.cpp:276-277), which leaves frame_counter at 0; under DF_KINFU_RELOCALISE
// it leaves accepted false instead and changes nothing.
int track(KinFu &k, double &t_sync0, double &t_sync1, bool &accepted)
{
    cudaStream_t s = k.stream;
    float pose[12];
    accepted = true;
    if (k.has_ov_pose) {               // lock-step parity hook: the caller's pose instead of this frame's ICP
        k.last_ok = 1;
        CK(cudaStreamSynchronize(s));
        note_solve_overflow(k);
        memcpy(pose, k.ov_pose, sizeof pose);
        k.has_ov_pose = false;
        if (k.lost) { k.lost = false; ++k.relocalisations; }           // the caller's pose ends a loss as an accepted one does
    } else if (reloc_on(k)) {
        CK(track_reloc(k, t_sync0, t_sync1, pose, accepted));
        if (!accepted) return 0;
    } else {
        CK(launch_icp(k));
        CK(cudaMemcpyAsync(k.pinned, k.icp_T, 12 * sizeof(float), cudaMemcpyDeviceToHost, s));
        CK(cudaMemcpyAsync(k.pinned + 12, k.icp_ok, sizeof(int), cudaMemcpyDeviceToHost, s));
        t_sync0 = now_us();
        CK(cudaStreamSynchronize(s));
        t_sync1 = now_us();
        int ok;
        memcpy(&ok, k.pinned + 12, sizeof(int));
        k.last_ok = ok;
        note_solve_overflow(k);                                       // the previous frame's solve flag arrived with this sync
        if (!ok) return do_reset(k);                                  // kinfu.cpp:276-277
        dfh_aff_mul(latest_pose(k), k.pinned, pose);                 // poses_.back() * affine, kinfu.cpp:280
    }
    if (reloc_on(k)) CK(launch_match(k, 1, pose));                     // the harvest
    mark(k, 2);
    k.poses.insert(k.poses.end(), pose, pose + 12);
    return 0;
}

// ---- the live model of DF_KINFU_LIVE_MODEL: the mesh of the current state (kinfu_mesh.cu), warped and rasterised ----------------

// DF_KINFU_LIVE_MODEL: p - shift for every cloud point (w kept), written twice: the association's source vertices and the copy df_warp carries
// into the live frame
__global__ void __launch_bounds__(256) shift_points_kernel(const float4 *cloud, int n, float sx, float sy, float sz, float4 *src, float4 *live)
{
    DF_PDL_ENTRY();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = cloud[i];
    const float4 o = make_float4(p.x - sx, p.y - sy, p.z - sz, p.w);
    src[i] = o;
    live[i] = o;
}

bool live_model_on(const KinFu &k) { return (k.p.flags & DF_KINFU_LIVE_MODEL) != 0; }

// a frame whose live mesh could not be built tracks and solves against the ray-casts; counted once per frame (get_info[12])
void note_live_model_fallback(KinFu &k, int cloud_points)
{
    if (k.lm_fell_back) return;
    k.lm_fell_back = true;
    if (k.lm_fallbacks++ == 0)
        fprintf(stderr, "df_kinfu: no live model: the extracted cloud (%d points) does not match the volume (truncated at cloud_capacity = %d); "
                        "frames like this one track and solve against the ray-casts (df_kinfu_get_info[12] counts them)\n",
                cloud_points, k.p.cloud_capacity);
}

// the live mesh of the current state into lm_src / lm_live / mesh_tris (k.lm_valid), or a fallback when the cloud does not match the volume
int build_live_mesh(KinFu &k)
{
    cudaStream_t s = k.stream;
    k.lm_valid = false;
    int N = 0, T = 0;
    bool match = false;
    CK(mesh_count_now(k, N, T, match));
    k.launches += 7;
    if (!match) {
        note_live_model_fallback(k, N);
        return 0;
    }
    const float *unused;
    CK(mesh_build(k, 0, N, T, unused, nullptr));                       // the faces, shared with df_kinfu_mesh: the same state emits the same faces
    ++k.launches;
    CK(grow(k.lm_src, k.lm_src_bytes, (size_t)N * 16));
    CK(grow(k.lm_live, k.lm_live_bytes, (size_t)N * 32));
    float *live_pts = k.lm_live, *live_nrm = live_pts + (size_t)N * 4;
    CK(cudaMemcpyAsync(live_nrm, k.cloud_nrm, (size_t)N * 16, cudaMemcpyDeviceToDevice, s));
    if (N > 0) {
        launch_pdl(shift_points_kernel, dim3(div_up(N, 256)), dim3(256), 0, s, (const float4 *)k.cloud.p, N, k.lm_shift[0], k.lm_shift[1],
                   k.lm_shift[2], (float4 *)k.lm_src.p, (float4 *)live_pts);
        CK(df_warp(k.nodes, k.M, k.node_grid, live_pts, live_nrm, N, 4, AFF_IDENTITY, 0, nullptr, nullptr, s));   // as mesh_build(live)
        k.launches += 2;
    }
    k.lm_N = N; k.lm_T = T; k.lm_valid = true;
    return 0;
}

// df_raster_mesh of the kept live mesh seen through world2cam
int raster_live_mesh(KinFu &k, const df_aff3f &world2cam, int32_t *ids, size_t ids_pitch, Img &pts, Img &nrm)
{
    const df_kinfu_params &p = k.p;
    CK(grow(k.raster_ws, k.raster_ws_bytes, df_raster_workspace_bytes(k.lm_N, k.lm_T, p.cols, p.rows)));
    CK(df_raster_mesh(k.lm_live, k.lm_N, 4, k.mesh_tris, k.lm_T, world2cam, p.intr, p.cols, p.rows, ids, ids_pitch, (float *)pts.ptr,
                      pts.pitch, (float *)nrm.ptr, nrm.pitch, nullptr, k.raster_ws, k.stream));
    k.launches += 2 + (k.lm_N > 0) + 2 * (k.lm_T > 0);                 // clear, vertex, triangle + large, resolve
    return 0;
}

// ---- KinFu::dynamicfusion, kinfu.cpp:344-400, at the latest pose ---------------------------------------------------
// depth: the frame's bilateral-filtered depth, modified in place by project-and-remove; live_pts: its level-0 vertex map; prev_pose: the
// pose of the frame the kept live mesh was built in (DF_KINFU_LIVE_MODEL).
// Without a warp field (DF_KINFU_RIGID_ONLY, or fewer than 8 nodes) the frame is integrated rigidly: the plain KinFu (Nerei) loop.
int dynamicfusion(KinFu &k, const Img &depth, const Img &live_pts, const float *prev_pose)
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    const float *cam_pose = latest_pose(k);
    k.field_frame = false;
    if ((p.flags & DF_KINFU_RIGID_ONLY) || k.M < 8) {
        k.lm_valid = false;
        mark(k, 3); mark(k, 4); mark(k, 5); mark(k, 6); mark(k, 7);
        CK(integrate_rigid(k, cam_pose));
        mark(k, 8); mark(k, 9);
        return 0;
    }
    k.field_frame = true;
    const int npix = p.cols * p.rows;
    float inv_pose[12];
    dfh_aff_inv(cam_pose, inv_pose);
    if (live_model_on(k) && !k.lm_valid) CK(build_live_mesh(k));      // first frame after create, reset or load: the same bits as kept
    if (live_model_on(k) && k.lm_valid) {
        // model-to-frame association: the kept live mesh (camera frame of prev_pose) seen from this frame's camera, each pixel paired with
        // the canonical surface point drawn there; canonical points are model coordinates
        float inv_prev[12], cam2model[12], world2cam[12];
        dfh_aff_inv(prev_pose, inv_prev);
        dfh_aff_mul(inv_prev, cam_pose, cam2model);
        dfh_aff_inv(cam2model, world2cam);
        CK(raster_live_mesh(k, to_aff(world2cam), (int32_t *)k.lm_ids.ptr, k.lm_ids.pitch, k.canon_visible, k.canon_nrm));
        CK(df_mesh_correspond((const int32_t *)k.lm_ids.ptr, k.lm_ids.pitch, (const float *)k.canon_visible.ptr, k.canon_visible.pitch, k.lm_live,
                              k.lm_src, k.lm_N, 4, k.mesh_tris, k.lm_T, to_aff(world2cam), p.cols, p.rows, (const float *)live_pts.ptr,
                              live_pts.pitch, p.icp_dist_thres, (float *)k.canon.ptr, k.canon.pitch, (float *)k.canon_nrm.ptr, k.canon_nrm.pitch, s));
        ++k.launches;
        CK(cudaMemcpy2DAsync(k.canon_visible.ptr, k.canon_visible.pitch, k.canon.ptr, k.canon.pitch, (size_t)p.cols * 16, p.rows,
                             cudaMemcpyDeviceToDevice, s));
    } else {
        CK(raycast_model(k, cam_pose, k.canon_visible, k.canon_nrm));     // tsdf().raycast(camera_pose, ...), :351 (camera frame)
        launch_pdl(to_canonical_kernel, dim3(div_up(npix, 256)), dim3(256), 0, s, (const float4 *)k.canon_visible.ptr, make_aff(to_aff(inv_pose)),
                                                               (float4 *)k.canon.ptr, (float4 *)k.canon_visible.ptr, npix);
        ++k.launches;
    }
    k.lm_valid = false;                                                // the frame changes the state the mesh was built from
    mark(k, 3);
    // the warps pass warp_to_live_, which stays the identity (never set)
    CK(df_warp(k.nodes, k.M, k.node_grid, (float *)k.canon.ptr, (float *)k.canon_nrm.ptr, npix, 4, AFF_IDENTITY, DF_WARP_IMAGE_COLS(p.cols), nullptr, nullptr, s));   // :385
    ++k.launches;
    mark(k, 4);
    const bool f2_solve = (p.flags & DF_KINFU_F2_SOLVE) != 0;
    if (f2_solve) {
        // SURVEY 8f(2): robust 6-DoF data term + regulariser instead of the reference's translation-only data term (opt-in)
        CK(df_solve_f2(k.nodes, k.M, k.node_grid, (const float *)k.canon.ptr, (const float *)live_pts.ptr, npix, 4, &k.f2, k.f2_stats, k.f2_ws, s));
        k.launches += 6 + (k.f2.gn_iters + 1) * 4 + k.f2.gn_iters * (3 + 3 * k.f2.lin_iters);
    } else {
        CK(solve_data_term_ev(k.nodes, k.M, k.node_grid, (const float *)k.canon.ptr, (const float *)live_pts.ptr, npix, 4,
                              p.solver_nonlinear_iters, p.solver_linear_iters,
                              ((p.flags & DF_KINFU_REF_GRAPH_QUIRK) ? DF_SOLVE_REF_GRAPH_QUIRK : 0) | DF_SOLVE_IMAGE_COLS(p.cols), k.solve_stats, k.solve_ws, s,
                              k.ev_before_lm));   // :387
        k.launches += 9;                                               // prepare, blockscan, scan, tiles, rows (tiles), fill + rows (fallback), lm v6, lm v5 (fallback)
        CK(launch_deferred_extract(k, k.ev_before_lm));                // the previous frame's extraction rides on the 132 SMs the solve leaves idle
    }
    // row-overflow flag of this solve (stats[5]): lands in pinned memory, looked at after the next stream synchronisation
    CK(cudaMemcpyAsync(k.pinned + 14, k.solve_stats.p + 5, sizeof(double), cudaMemcpyDeviceToHost, s));
    if (k.has_ov_nodes) {              // lock-step parity hook: the caller's solved node table (CPU and GPU PCG round differently in the last bits)
        if (k.ov_nodes.size() == (size_t)k.M * DF_NODE_STRIDE) {
            CK(cudaMemcpyAsync(k.nodes, k.ov_nodes.data(), k.ov_nodes.size() * 4, cudaMemcpyHostToDevice, s));
            CK(cudaStreamSynchronize(s));
        }
        k.has_ov_nodes = false;
    }
    mark(k, 5);
    if (f2_solve) {
        CK(df_warp(k.nodes, k.M, k.node_grid, (float *)k.canon.ptr, (float *)k.canon_nrm.ptr, npix, 4, AFF_IDENTITY, 0, nullptr, nullptr, s));
    } else {
        // second warp (:389) queries exactly the vertices the solve just built its graph for (CombinedSolver.h:66-84):
        // re-use those neighbours + weights instead of a third k-NN pass
        int32_t *knn_idx; float *knn_w;
        CK(df_solve_knn_buffers(k.solve_ws, k.M, npix, &knn_idx, &knn_w));
        CK(df_warp(k.nodes, k.M, k.node_grid, (float *)k.canon.ptr, (float *)k.canon_nrm.ptr, npix, 4, AFF_IDENTITY, DF_WARP_REUSE_KNN, knn_idx, knn_w, s));
    }
    ++k.launches;
    mark(k, 6);
    if (p.flags & DF_KINFU_WARPED_INTEGRATE) {
        // SURVEY 8f(1): the update surface_fusion was written towards (tsdf_volume.cpp:240-252) -- every voxel is carried through
        // the field solved above and fused against the (bilateral-filtered) frame; no pixel is removed, no rigid integrate.
        mark(k, 7);
        unsigned long long *counter = (p.flags & DF_KINFU_STAGE_TIMING) ? k.n_upd.p : nullptr;
        // write-after-read: the previous frame's extraction (deferred to the auxiliary stream) reads the volume, the activity map and the
        // colour volume this step writes
        if (int w = wait_extract_on_main(k)) return w;
        if ((p.flags & DF_KINFU_WARPED_COLOR) && k.frame_bgra) {
            // DF_KINFU_WARPED_COLOR: the frame's colours go in during the same voxel walk, each voxel sampled where the field carries it
            if (counter) cudaMemsetAsync(counter, 0, 24, s);
            CK(df_integrate_warped_color(vol_of(k), (const uint16_t *)depth.ptr, depth.pitch, p.cols, p.rows, p.volume_pose, to_aff(inv_pose),
                                         p.intr, k.nodes, k.M, k.node_grid, p.fusion_weight_scale, counter, k.activity, k.fusion_ws, k.color_vol,
                                         k.frame_bgra, k.frame_bgra_pitch, k.has_cam ? &k.cam : nullptr, color_lens_of(k),
                                         (const uint32_t *)k.color_map.ptr, k.color_map.pitch, s));
        } else {
            if (counter) cudaMemsetAsync(counter, 0, 16, s);
            CK(df_integrate_warped(vol_of(k), (const uint16_t *)depth.ptr, depth.pitch, p.cols, p.rows, p.volume_pose, to_aff(inv_pose),
                                   p.intr, k.nodes, k.M, k.node_grid, p.fusion_weight_scale, counter, k.activity, k.fusion_ws, s));
        }
        k.launches += df_integrate_warped_launch_count();
    } else {
        // surface_fusion (tsdf_volume.cpp:228-255): psdf projects the warped vertices into the (bilateral-filtered) depth,
        // zeroes the pixels they explain, then the ordinary rigid integrate runs on what is left.
        CK(df_project_and_remove((uint16_t *)depth.ptr, depth.pitch, p.cols, p.rows, p.intr, (float *)k.canon.ptr, k.canon.pitch, p.cols, p.rows,
                                 k.project_ws, s));
        k.launches += 2;
        CK(df_compute_dists((const uint16_t *)depth.ptr, depth.pitch, p.cols, p.rows, p.intr, (uint16_t *)k.dists.ptr, k.dists.pitch, s));
        ++k.launches;
        mark(k, 7);                                                    // stage "integrate" brackets the integrate kernel alone
        CK(integrate_rigid(k, cam_pose));
    }
    mark(k, 8);
    // compute_points / compute_normals, :398-399; the field extension and the live mesh (raycast_next) read the cloud right away
    CK(extract_cloud(k, (p.flags & DF_KINFU_EXTEND_FIELD) != 0 || live_model_on(k)));
    CK(extend_field(k));
    mark(k, 9);
    return 0;
}

// ---- ray-cast for the next frame's ICP, kinfu.cpp:297-301 ------------------------------------------------------------
int raycast_next(KinFu &k)
{
    const df_kinfu_params &p = k.p;
    cudaStream_t s = k.stream;
    if (live_model_on(k) && k.field_frame) CK(build_live_mesh(k));
    if (k.lm_valid) {
        // DF_KINFU_LIVE_MODEL: the live mesh is in this camera's frame; it is kept for the next frame's association
        CK(raster_live_mesh(k, AFF_IDENTITY, nullptr, 0, k.prev_pts[0], k.prev_nrm[0]));
    } else
    CK(raycast_model(k, latest_pose(k), k.prev_pts[0], k.prev_nrm[0]));
    if (p.flags & DF_KINFU_USE_DEPTH) {
        // TsdfVolume::raycast(pose, intr, Depth&, Normals&) (tsdf_volume.cu:273-339,441-456) = the same march storing ushort(vertex.z * 1000),
        // then resizeDepthNormals per level (kinfu.cpp:293-295)
        CK(df_cloud_to_depth((const float *)k.prev_pts[0].ptr, k.prev_pts[0].pitch, p.cols, p.rows, (uint16_t *)k.prev_depth[0].ptr, k.prev_depth[0].pitch, s));
        ++k.launches;
        for (int i = 1; i < k.levels; ++i) {
            CK(df_resize_depth_normals((const uint16_t *)k.prev_depth[i - 1].ptr, k.prev_depth[i - 1].pitch, (const float *)k.prev_nrm[i - 1].ptr,
                                       k.prev_nrm[i - 1].pitch, k.prev_depth[i - 1].cols, k.prev_depth[i - 1].rows,
                                       (uint16_t *)k.prev_depth[i].ptr, k.prev_depth[i].pitch, (float *)k.prev_nrm[i].ptr, k.prev_nrm[i].pitch, s));
            ++k.launches;
        }
    } else
    for (int i = 1; i < k.levels; ++i) {
        CK(df_resize_points_normals((const float *)k.prev_pts[i - 1].ptr, k.prev_pts[i - 1].pitch, (const float *)k.prev_nrm[i - 1].ptr,
                                    k.prev_nrm[i - 1].pitch, k.prev_pts[i - 1].cols, k.prev_pts[i - 1].rows,
                                    (float *)k.prev_pts[i].ptr, k.prev_pts[i].pitch, (float *)k.prev_nrm[i].ptr, k.prev_nrm[i].pitch, s));
        ++k.launches;
    }
    mark(k, 10);
    return 0;
}

// df_kinfu_set_depth_lens: the caller's raw frame -> the pinhole frame every later stage reads, in the object's own buffers (a registered
// colour image shares the depth lens; a colour camera's image is projected through its own lens instead)
int undistort_frame(KinFu &k, const uint16_t *&depth_dev, size_t &depth_pitch)
{
    const df_kinfu_params &p = k.p;
    const bool registered = k.frame_bgra && !k.has_cam;
    CK(df_undistort(depth_dev, depth_pitch, (uint16_t *)k.depth_ud.ptr, k.depth_ud.pitch, registered ? k.frame_bgra : nullptr, k.frame_bgra_pitch,
                    registered ? k.bgra_ud.ptr : nullptr, k.bgra_ud.pitch, p.cols, p.rows, p.intr, k.depth_lens, k.stream));
    ++k.launches;
    depth_dev = (const uint16_t *)k.depth_ud.ptr; depth_pitch = k.depth_ud.pitch;
    if (registered) { k.frame_bgra = k.bgra_ud.ptr; k.frame_bgra_pitch = k.bgra_ud.pitch; }
    return 0;
}

// KinFu::operator()(depth), kinfu.cpp:221-305: the stages in order.  fused = its return value (false: first frame, or tracking lost).
int process(KinFu &k, const uint16_t *depth_dev, size_t depth_pitch, bool &fused)
{
    const double t_begin = now_us();
    double t_sync0 = t_begin, t_sync1 = t_begin;
    fused = false;
    begin_frame(k);
    if (k.has_depth_lens) CK(undistort_frame(k, depth_dev, depth_pitch));
    CK(preprocess(k, depth_dev, depth_pitch));
    if (k.frame_counter == 0) {
        CK(first_frame(k));
        return reloc_on(k) ? launch_match(k, 1, latest_pose(k)) : 0;   // the first frame is keyframe 0
    }
    bool accepted;
    CK(track(k, t_sync0, t_sync1, accepted));
    if (!accepted) return 0;                                           // DF_KINFU_RELOCALISE: a lost frame
    if (k.frame_counter == 0) return 0;                                // tracking lost: the object was reset
    CK(dynamicfusion(k, k.cur_depth[0], k.cur_pts[0], &k.poses[k.poses.size() - 24]));
    CK(raycast_next(k));
    ++k.frame_counter;
    const double t_end = now_us();
    k.host_us[0] += t_sync0 - t_begin; k.host_us[1] += t_sync1 - t_sync0; k.host_us[2] += t_end - t_sync1; k.host_us[3] += t_end - t_begin;
    ++k.host_frames;
    fused = true;
    return 0;
}

}  // namespace

void dfb::kinfu::sync_extract(KinFu &k)
{
    if (!k.aux) return;
    if (k.extract_deferred) {
        cudaEventRecord(k.ev_volume_ready, k.stream);
        launch_deferred_extract(k, k.ev_volume_ready);
    }
    cudaStreamSynchronize(k.aux);
}

// A normal-matrix row that does not fit (solve.cu: more than ROWCAP coupled columns) makes the solve leave the warp field unchanged for
// that frame and raise stats[5]; the flag is copied to pinned memory after every solve and reported here, loudly, at the next sync.
void dfb::kinfu::note_solve_overflow(KinFu &k)
{
    double f;
    memcpy(&f, k.pinned + 14, sizeof f);
    if (f != 0.0) {
        ++k.solve_overflows;
        fprintf(stderr, "df_kinfu: warp solve skipped for one frame: a normal-matrix row exceeded the row capacity (df_kinfu_get_info[11] = %lld)\n", k.solve_overflows);
        f = 0.0;
        memcpy(k.pinned + 14, &f, sizeof f);
    }
}

extern "C" void df_kinfu_default_params(df_kinfu_params *p, int which)
{
    memset(p, 0, sizeof *p);
    p->cols = 640; p->rows = 480;
    const int iters[4] = {10, 5, 4, 0};
    memcpy(p->icp_iter_num, iters, sizeof iters);
    float pose[12];
    dfh_aff_identity(pose);
    if (which == 0) {          // default_params_dynamicfusion, kinfu.cpp:14-49
        p->intr = df_intr{570.342f, 570.342f, 320.f, 240.f};
        for (int i = 0; i < 3; ++i) { p->volume_dims[i] = 256; p->volume_size[i] = 1.f; }
    } else {                   // default_params, kinfu.cpp:55-89
        p->intr = df_intr{525.f, 525.f, 640 / 2 - 0.5f, 480 / 2 - 0.5f};
        for (int i = 0; i < 3; ++i) { p->volume_dims[i] = 512; p->volume_size[i] = 3.f; }
    }
    pose[9] = -p->volume_size[0] / 2; pose[10] = -p->volume_size[1] / 2; pose[11] = 0.5f;
    memcpy(p->volume_pose.R, pose, 36); memcpy(p->volume_pose.t, pose + 9, 12);
    p->bilateral_sigma_depth = 0.04f; p->bilateral_sigma_spatial = 4.5f; p->bilateral_kernel_size = 7;
    p->icp_truncate_depth_dist = 0.f; p->icp_dist_thres = 0.1f; p->icp_angle_thres = 30.f * 0.017453293f;
    p->tsdf_min_camera_movement = 0.f; p->tsdf_trunc_dist = 0.04f; p->tsdf_max_weight = 64;
    p->raycast_step_factor = 0.75f; p->gradient_delta_factor = 0.5f;
    p->solver_nonlinear_iters = 5; p->solver_linear_iters = 100;     // kinfu.cpp:116-117
    p->max_nodes = 4096; p->node_step = 50; p->cloud_capacity = 256 * 256 * 256 / 4;
    p->flags = 0;
}

extern "C" void *df_kinfu_create(const df_kinfu_params *pp)
{
    if (pp->volume_dims[0] % 32 != 0) {                               // CV_Assert, kinfu.cpp:97
        fprintf(stderr, "df_kinfu_create: volume_dims[0] %% 32 != 0\n");
        return nullptr;
    }
    KinFu *k = new KinFu();
    k->p = *pp;
    cudaGetDevice(&k->device);
    {
        // the flags the environment can switch on (dfusion.h): <name>=<non-zero integer>
        static const struct { const char *name; int flag; } env_flags[] = {
            {"DF_KINFU_WARPED_INTEGRATE", DF_KINFU_WARPED_INTEGRATE}, {"DF_KINFU_EXTEND_FIELD", DF_KINFU_EXTEND_FIELD},
            {"DF_KINFU_USE_DEPTH", DF_KINFU_USE_DEPTH}, {"DF_KINFU_F2_SOLVE", DF_KINFU_F2_SOLVE}, {"DF_KINFU_LIVE_MODEL", DF_KINFU_LIVE_MODEL},
            {"DF_KINFU_COLOR", DF_KINFU_COLOR}, {"DF_KINFU_RELOCALISE", DF_KINFU_RELOCALISE}};
        for (const auto &f : env_flags) {
            const char *e = getenv(f.name);
            if (e && atoi(e) != 0) k->p.flags |= f.flag;
        }
        const char *xr = getenv("DF_EXTEND_RADIUS");
        if (xr) k->p.extend_radius = (float)atof(xr);
        const char *wc = getenv("DF_KINFU_WARPED_COLOR");                  // for objects with both flags it needs only
        if (wc && atoi(wc) != 0 && (k->p.flags & DF_KINFU_COLOR) && (k->p.flags & DF_KINFU_WARPED_INTEGRATE)) k->p.flags |= DF_KINFU_WARPED_COLOR;
        const char *ct = getenv("DF_KINFU_COLOR_TRACKING");                // for colour objects only: a colourless one stays as it was
        if (ct && atoi(ct) != 0 && (k->p.flags & DF_KINFU_COLOR)) k->p.flags |= DF_KINFU_COLOR_TRACKING;
        const char *w = getenv("DF_FUSION_WEIGHT_SCALE");
        if (w) k->p.fusion_weight_scale = (float)atof(w);
    }
    const df_kinfu_params &p = k->p;
    if ((p.flags & DF_KINFU_WARPED_COLOR) && !((p.flags & DF_KINFU_COLOR) && (p.flags & DF_KINFU_WARPED_INTEGRATE))) {
        fprintf(stderr, "df_kinfu_create: DF_KINFU_WARPED_COLOR needs %s: it fuses the colour volume during the per-voxel warped fusion\n",
                !(p.flags & DF_KINFU_COLOR) ? "DF_KINFU_COLOR" : "DF_KINFU_WARPED_INTEGRATE");
        delete k;
        return nullptr;
    }
    if ((p.flags & DF_KINFU_COLOR) && (p.flags & DF_KINFU_WARPED_INTEGRATE) && !(p.flags & DF_KINFU_WARPED_COLOR)) {
        fprintf(stderr, "df_kinfu_create: DF_KINFU_COLOR cannot be combined with DF_KINFU_WARPED_INTEGRATE alone: under per-voxel warped fusion a "
                        "voxel meets its pixel through the warp field, and the rigid colour rule does not follow it; add DF_KINFU_WARPED_COLOR, "
                        "which carries each voxel's colour sample through the field\n");
        delete k;
        return nullptr;
    }
    if (p.flags & DF_KINFU_COLOR_TRACKING) {
        const char *why = !(p.flags & DF_KINFU_COLOR) ? "it needs DF_KINFU_COLOR: the model's intensity comes from the colour volume"
                          : (p.flags & DF_KINFU_USE_DEPTH) ? "cannot be combined with DF_KINFU_USE_DEPTH: its previous maps are depth maps, not the vertex maps the model's "
                                                              "intensity is sampled at"
                          : (p.flags & DF_KINFU_LIVE_MODEL) ? "cannot be combined with DF_KINFU_LIVE_MODEL: its previous maps are a raster of the live mesh in the camera's "
                                                               "frame, not points of the canonical volume the colour was fused into"
                          : nullptr;
        if (why) {
            fprintf(stderr, "df_kinfu_create: DF_KINFU_COLOR_TRACKING %s\n", why);
            delete k;
            return nullptr;
        }
    }
    k->levels = used_levels(p);
    if (p.flags & DF_KINFU_RELOCALISE) {
        const char *why = (p.flags & DF_KINFU_USE_DEPTH) ? "cannot be combined with DF_KINFU_USE_DEPTH: its ICP reference is the model's depth pyramid"
                          : (p.flags & DF_KINFU_LIVE_MODEL) ? "cannot be combined with DF_KINFU_LIVE_MODEL: its ICP reference is a raster of the live mesh, "
                                                               "not a ray-cast of the canonical volume a keyframe can be seen in"
                          : k->levels < 3 ? "needs at least 3 used ICP levels: the fern codes read the pyramid's level 2"
                          : nullptr;
        if (why) {
            fprintf(stderr, "df_kinfu_create: DF_KINFU_RELOCALISE %s\n", why);
            delete k;
            return nullptr;
        }
    }
    k->max_nodes_cap = node_capacity(p);
    memcpy(k->vol_pose, p.volume_pose.R, 36); memcpy(k->vol_pose + 9, p.volume_pose.t, 12);
    dfh_mat3_inv(k->vol_pose, k->Rinv_vol);
    float vmax = 0.f;
    for (int d = 0; d < 3; ++d) { k->voxel_size[d] = p.volume_size[d] / p.volume_dims[d]; vmax = vmax > k->voxel_size[d] ? vmax : k->voxel_size[d]; }
    k->trunc_dist = p.tsdf_trunc_dist > 2.1f * vmax ? p.tsdf_trunc_dist : 2.1f * vmax;   // setTruncDist, tsdf_volume.cpp:68-73
    {
        const float h[3] = {k->voxel_size[0] / 2.f, k->voxel_size[1] / 2.f, k->voxel_size[2] / 2.f};
        for (int r = 0; r < 3; ++r) k->lm_shift[r] = k->vol_pose[3 * r] * h[0] + k->vol_pose[3 * r + 1] * h[1] + k->vol_pose[3 * r + 2] * h[2];
    }
    const size_t nvox = (size_t)p.volume_dims[0] * p.volume_dims[1] * p.volume_dims[2];
    bool ok = k->volume.alloc(nvox * 4) == cudaSuccess;
    ok = ok && alloc_img(k->depth_in, p.rows, p.cols, 2) == 0 && alloc_img(k->dists, p.rows, p.cols, 2) == 0;
    int cols = p.cols, rows = p.rows;
    for (int l = 0; l < MAX_LEVELS && ok; ++l) {                      // allocate_buffers, kinfu.cpp:151-194
        ok = ok && alloc_img(k->cur_depth[l], rows, cols, 2) == 0 && alloc_img(k->cur_pts[l], rows, cols, 16) == 0 &&
             alloc_img(k->cur_nrm[l], rows, cols, 16) == 0 && alloc_img(k->prev_pts[l], rows, cols, 16) == 0 &&
             alloc_img(k->prev_nrm[l], rows, cols, 16) == 0 && alloc_img(k->prev_depth[l], rows, cols, 2) == 0;
        cols /= 2; rows /= 2;
    }
    if (p.flags & DF_KINFU_COLOR_TRACKING)
        for (int l = 0, c = p.cols, r = p.rows; l < k->levels && ok; ++l, c /= 2, r /= 2)
            ok = alloc_img(k->cur_int[l], r, c, 4) == 0 && alloc_img(k->model_int[l], r, c, 16) == 0;
    ok = ok && alloc_img(k->canon, p.rows, p.cols, 16) == 0 && alloc_img(k->canon_nrm, p.rows, p.cols, 16) == 0 &&
         alloc_img(k->canon_visible, p.rows, p.cols, 16) == 0;
    if (p.flags & DF_KINFU_LIVE_MODEL) ok = ok && alloc_img(k->lm_ids, p.rows, p.cols, 4) == 0;
    if (p.flags & DF_KINFU_COLOR)
        ok = ok && k->color_vol.alloc(nvox * 4) == cudaSuccess && k->cloud_rgba.alloc((size_t)p.cloud_capacity * 4) == cudaSuccess &&
             cudaMemset(k->cloud_rgba, 0, (size_t)p.cloud_capacity * 4) == cudaSuccess && alloc_img(k->color_in, p.rows, p.cols, 4) == 0;
    ok = ok && k->cloud.alloc((size_t)p.cloud_capacity * 16) == cudaSuccess && k->cloud_nrm.alloc((size_t)p.cloud_capacity * 16) == cudaSuccess;
    ok = ok && k->cloud_count.alloc(64) == cudaSuccess;
    const int maxM = k->max_nodes_cap;
    ok = ok && k->nodes.alloc((size_t)maxM * DF_NODE_STRIDE * 4) == cudaSuccess && k->node_grid.alloc(df_node_grid_bytes(maxM)) == cudaSuccess;
    ok = ok && k->icp_T.alloc(64) == cudaSuccess && k->icp_ok.alloc(64) == cudaSuccess &&
         k->icp_scratch.alloc((size_t)DF_ICP_SCRATCH_DOUBLES * 8) == cudaSuccess;
    ok = ok && k->solve_ws.alloc(df_solve_workspace_bytes(maxM, p.cols * p.rows)) == cudaSuccess && k->solve_stats.alloc(64) == cudaSuccess;
    k->f2 = df_f2_params{5.0, 0.05, 1e-4, 1e-4, 2, 4, DF_F2_TWIST | DF_F2_TUKEY | DF_F2_HUBER, 30};
    if (p.flags & DF_KINFU_F2_SOLVE)
        ok = ok && k->f2_ws.alloc(df_solve_f2_workspace_bytes(maxM, p.cols * p.rows, 7)) == cudaSuccess && k->f2_stats.alloc(16 * 8) == cudaSuccess;
    df_volume v = vol_of(*k);
    ok = ok && k->extract_ws.alloc(df_extract_workspace_bytes(v)) == cudaSuccess;
    ok = ok && k->integrate_ws.alloc(df_integrate_workspace_bytes(p.cols, p.rows)) == cudaSuccess;
    ok = ok && k->extend_ws.alloc(df_extend_field_workspace_bytes(p.cloud_capacity)) == cudaSuccess && k->M_dev.alloc(64) == cudaSuccess;
    ok = ok && k->fusion_ws.alloc(df_integrate_warped_workspace_bytes(p.cols, p.rows, maxM)) == cudaSuccess;
    k->activity_bytes = df_volume_activity_bytes(v);
    ok = ok && k->activity.alloc(k->activity_bytes) == cudaSuccess && cudaMemset(k->activity, 0, k->activity_bytes) == cudaSuccess;
    ok = ok && k->project_ws.alloc(df_project_workspace_bytes(p.cols, p.rows)) == cudaSuccess;
    if (p.flags & DF_KINFU_RELOCALISE) {
        std::vector<int32_t> table((size_t)DF_RELOC_FERNS * 12);
        ok = ok && df_reloc_fern_table(DF_RELOC_SEED, k->cur_depth[2].cols, k->cur_depth[2].rows, DF_RELOC_FERNS, table.data()) == 0;
        ok = ok && k->fern_table.alloc(table.size() * 4) == cudaSuccess &&
             cudaMemcpy(k->fern_table, table.data(), table.size() * 4, cudaMemcpyHostToDevice) == cudaSuccess;
        ok = ok && k->frame_code.alloc(DF_RELOC_FERNS) == cudaSuccess && k->kf_codes.alloc((size_t)DF_RELOC_KEYFRAMES * DF_RELOC_FERNS) == cudaSuccess &&
             k->kf_poses.alloc((size_t)DF_RELOC_KEYFRAMES * 48) == cudaSuccess && k->kf_count.alloc(64) == cudaSuccess;
        ok = ok && k->gate_ws.alloc(DF_RELOC_GATE_WS_BYTES) == cudaSuccess && cudaMemset(k->gate_ws, 0, DF_RELOC_GATE_WS_BYTES) == cudaSuccess;
        ok = ok && k->gate.alloc(sizeof(df_reloc_gate)) == cudaSuccess && k->match.alloc(sizeof(df_reloc_match)) == cudaSuccess;
        ok = ok && cudaMallocHost(&k->gate_host, sizeof(df_reloc_gate)) == cudaSuccess && cudaMallocHost(&k->match_host, sizeof(df_reloc_match)) == cudaSuccess;
        for (int l = 0, c = p.cols, r = p.rows; l < k->levels && ok; ++l, c /= 2, r /= 2)
            ok = alloc_img(k->rl_pts[l], r, c, 16) == 0 && alloc_img(k->rl_nrm[l], r, c, 16) == 0;
    }
    ok = ok && cudaMemset(k->project_ws, 0, df_project_workspace_bytes(p.cols, p.rows)) == cudaSuccess;
    ok = ok && cudaMemset(k->solve_stats, 0, 64) == cudaSuccess && cudaMemset(k->cloud_count, 0, 64) == cudaSuccess;
    ok = ok && cudaMallocHost(&k->pinned, 64) == cudaSuccess && (memset(k->pinned, 0, 64), true) && k->n_upd.alloc(64) == cudaSuccess && cudaMemset(k->n_upd, 0, 64) == cudaSuccess;
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);              // lo = numerically greatest = lowest priority
    ok = ok && cudaStreamCreateWithPriority(&k->aux, cudaStreamNonBlocking, prio_lo) == cudaSuccess &&
         cudaEventCreateWithFlags(&k->ev_before_lm, cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&k->ev_volume_ready, cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&k->ev_extract_done, cudaEventDisableTiming) == cudaSuccess;
    { const char *oe = getenv("DF_KINFU_OVERLAP_EXTRACT"); if (oe && atoi(oe) == 0) k->overlap_extract = false; }
    for (int e = 0; e <= NSTAGES && ok; ++e) ok = cudaEventCreate(&k->ev[e]) == cudaSuccess;
    if (!ok) {
        fprintf(stderr, "df_kinfu_create: CUDA allocation failed: %s\n", cudaGetErrorString(cudaGetLastError()));
        delete k;
        return nullptr;
    }
    int st = do_reset(*k);                                            // an object is only handed out with its volume cleared
    if (!st) st = (int)cudaStreamSynchronize(k->stream);
    if (st) {
        fprintf(stderr, "df_kinfu_create: clearing the volume failed: %s\n", cudaGetErrorString((cudaError_t)st));
        delete k;
        return nullptr;
    }
    return k;
}

extern "C" void df_kinfu_destroy(void *h)
{
    KinFu *k = (KinFu *)h;
    if (!k) return;
    if (getenv("DF_KINFU_HOSTPROF") && k->host_frames)
        fprintf(stderr, "[df_kinfu host profile] frames %lld: launch-A %.1f us, ICP wait %.1f us, launch-B %.1f us, total %.1f us per frame\n", k->host_frames,
                k->host_us[0] / k->host_frames, k->host_us[1] / k->host_frames, k->host_us[2] / k->host_frames, k->host_us[3] / k->host_frames);
    delete k;
}

extern "C" int df_kinfu_set_stream(void *h, void *stream) { ((KinFu *)h)->stream = (cudaStream_t)stream; return 0; }
extern "C" int df_kinfu_reset(void *h) { return -do_reset(*(KinFu *)h); }

static void finish_timing(KinFu &k)
{
    if (!(k.p.flags & DF_KINFU_STAGE_TIMING)) return;
    cudaStreamSynchronize(k.stream);
    int prev = 0;
    for (int s = 1; s <= NSTAGES; ++s) {
        k.stage_ms[s - 1] = 0.f;
        if (!k.stage_mark[s]) continue;
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, k.ev[prev], k.ev[s]) == cudaSuccess) k.stage_ms[s - 1] = ms;
        prev = s;
    }
}

// Multi-device host entry (SURVEY 8e: the path shards by SEQUENCE): n independent KinFu objects -- typically one per GPU, created after
// cudaSetDevice(i) -- advance by one frame each, concurrently: one host thread per object (a frame has one host synchronisation, the ICP
// status, so a sequential loop would serialise the devices).  results[i] receives what df_kinfu_process_host returns for object i.
extern "C" int df_kinfu_batch_process_host(void *const *kinfus, const uint16_t *const *depth_host, const size_t *pitch, int n, int *results)
{
    if (n <= 0) return 0;
    std::vector<std::thread> th;
    th.reserve((size_t)n);
    for (int i = 1; i < n; ++i)
        th.emplace_back([=] { results[i] = df_kinfu_process_host(kinfus[i], depth_host[i], pitch[i]); });
    results[0] = df_kinfu_process_host(kinfus[0], depth_host[0], pitch[0]);
    for (auto &t : th) t.join();
    int worst = 0;
    for (int i = 0; i < n; ++i) if (results[i] < worst) worst = results[i];
    return worst;                                                    // 0, or the first negative status (-cudaError) of any object
}

// one frame from device images; bgra (optional) is the frame's colour image for the length of the call
static int process_device(KinFu &k, const uint16_t *depth_dev, size_t pitch, const void *bgra_dev, size_t bgra_pitch)
{
    cudaSetDevice(k.device);
    bool fused;
    k.frame_bgra = bgra_dev; k.frame_bgra_pitch = bgra_pitch;
    const int st = process(k, depth_dev, pitch, fused);
    k.frame_bgra = nullptr;
    finish_timing(k);
    return st ? -st : fused;
}

// the _color entries need a colour object and an image with whole pixels per row: the depth frame's width, or the colour camera's
static bool color_frame_ok(const KinFu *k, const void *bgra, size_t bgra_pitch)
{
    return k && color_on(*k) && bgra && bgra_pitch >= (size_t)k->color_in.cols * 4 && bgra_pitch % 4 == 0;
}

extern "C" int df_kinfu_process_device(void *h, const uint16_t *depth_dev, size_t pitch)
{
    return process_device(*(KinFu *)h, depth_dev, pitch, nullptr, 0);
}

extern "C" int df_kinfu_process_device_color(void *h, const uint16_t *depth_dev, size_t pitch, const void *bgra_dev, size_t bgra_pitch)
{
    KinFu *k = (KinFu *)h;
    if (!color_frame_ok(k, bgra_dev, bgra_pitch)) return -(int)cudaErrorInvalidValue;
    return process_device(*k, depth_dev, pitch, bgra_dev, bgra_pitch);
}

// KinFu::dynamicfusion(depth, live_frame, current_normals) (kinfu.hpp:87, kinfu.cpp:344-400) as a stand-alone call on
// caller-provided device buffers (depth is modified in place by the project-and-remove step, like the reference)
extern "C" int df_kinfu_dynamicfusion(void *h, uint16_t *depth_dev, size_t depth_pitch, const float *live_points_dev, size_t live_pitch)
{
    KinFu *k = (KinFu *)h;
    if (k->poses.size() < 12) return 0;
    begin_frame(*k);
    mark(*k, 2);                                                      // no tracking: the latest pose is the frame's
    const Img depth{depth_dev, depth_pitch, k->p.cols, k->p.rows}, live{(void *)live_points_dev, live_pitch, k->p.cols, k->p.rows};
    const int st = dynamicfusion(*k, depth, live, latest_pose(*k));   // the latest pose is also the kept live mesh's
    return st ? -st : 1;
}

// one frame from host images, copied to the device inside the call; bgra_host is optional
static int process_host(KinFu *k, const uint16_t *depth_host, size_t pitch, const void *bgra_host, size_t bgra_pitch)
{
    cudaSetDevice(k->device);                                         // per host thread: lets one process drive one object per GPU
    // depth_device_.upload(depth.data, depth.step, rows, cols), apps/demo.cpp:89
    cudaError_t e = cudaMemcpy2DAsync(k->depth_in.ptr, k->depth_in.pitch, depth_host, pitch, (size_t)k->p.cols * 2, k->p.rows,
                                      cudaMemcpyHostToDevice, k->stream);
    if (e == cudaSuccess && bgra_host)
        e = cudaMemcpy2DAsync(k->color_in.ptr, k->color_in.pitch, bgra_host, bgra_pitch, (size_t)k->color_in.cols * 4, k->color_in.rows,
                              cudaMemcpyHostToDevice, k->stream);
    if (e != cudaSuccess) return -(int)e;
    bool fused;
    k->frame_bgra = bgra_host ? k->color_in.ptr : nullptr; k->frame_bgra_pitch = k->color_in.pitch;
    const int pst = process(*k, (const uint16_t *)k->depth_in.ptr, k->depth_in.pitch, fused);
    k->frame_bgra = nullptr;
    if (pst) return -pst;
    e = cudaStreamSynchronize(k->stream);        // the caller owns the result when the call returns (renderImage / getCameraPose next)
    if (e == cudaSuccess) note_solve_overflow(*k);
    finish_timing(*k);
    return e == cudaSuccess ? fused : -(int)e;
}

extern "C" int df_kinfu_process_host(void *h, const uint16_t *depth_host, size_t pitch)
{
    return process_host((KinFu *)h, depth_host, pitch, nullptr, 0);
}

extern "C" int df_kinfu_process_host_color(void *h, const uint16_t *depth_host, size_t pitch, const void *bgra_host, size_t bgra_pitch)
{
    KinFu *k = (KinFu *)h;
    if (!color_frame_ok(k, bgra_host, bgra_pitch)) return -(int)cudaErrorInvalidValue;
    return process_host(k, depth_host, pitch, bgra_host, bgra_pitch);
}

extern "C" int df_kinfu_set_color_camera(void *h, const df_color_camera *cam)
{
    KinFu *k = (KinFu *)h;
    if (!k || !color_on(*k) || k->frame_counter != 0) return (int)cudaErrorInvalidValue;
    int mcols = 0, mrows = 0, cell = 0;
    if (cam && df_color_map_dims(k->p.intr, *cam, &mcols, &mrows, &cell) != 0) return (int)cudaErrorInvalidValue;
    cudaSetDevice(k->device);
    CK(cudaStreamSynchronize(k->stream));                              // a host frame's upload may still read the old colour frame
    Img frame, map, bgra_ud;
    if (cam) {
        CK(alloc_img(frame, cam->rows, cam->cols, 4));
        CK(alloc_img(map, mrows, mcols, 4));
    } else {
        CK(alloc_img(frame, k->p.rows, k->p.cols, 4));
        if (k->has_depth_lens) CK(alloc_img(bgra_ud, k->p.rows, k->p.cols, 4));   // registered images share the depth lens
    }
    k->color_in = std::move(frame);                                    // the old buffers are freed with `frame`, `map` and `bgra_ud`
    k->color_map = std::move(map);
    k->bgra_ud = std::move(bgra_ud);
    k->has_cam = cam != nullptr;
    if (cam) memcpy(&k->cam, cam, sizeof k->cam);
    else memset(&k->cam, 0, sizeof k->cam);
    k->has_color_lens = false;                                          // a colour lens belongs to the camera it was calibrated with
    memset(&k->color_lens, 0, sizeof k->color_lens);
    return 0;
}

// the lens argument of the two setters: `on` is false for NULL and for the zero lens (no lens); an invalid lens is refused
static int lens_setting(const df_lens *lens, bool &on)
{
    on = lens && !lens_is_zero(*lens);
    return lens && df_lens_check(*lens) ? (int)cudaErrorInvalidValue : 0;
}

extern "C" int df_kinfu_set_depth_lens(void *h, const df_lens *lens)
{
    KinFu *k = (KinFu *)h;
    bool on = false;
    if (!k || k->frame_counter != 0 || lens_setting(lens, on)) return (int)cudaErrorInvalidValue;
    cudaSetDevice(k->device);
    CK(cudaStreamSynchronize(k->stream));                              // the last frame may still read the old buffers
    Img depth, bgra;
    if (on) {
        CK(alloc_img(depth, k->p.rows, k->p.cols, 2));
        if (color_on(*k) && !k->has_cam) CK(alloc_img(bgra, k->p.rows, k->p.cols, 4));   // only a registered image is undistorted
    }
    k->depth_ud = std::move(depth);                                    // the old buffers are freed with `depth` and `bgra`
    k->bgra_ud = std::move(bgra);
    k->has_depth_lens = on;
    k->depth_lens = on ? *lens : df_lens{};
    return 0;
}

extern "C" int df_kinfu_set_color_lens(void *h, const df_lens *lens)
{
    KinFu *k = (KinFu *)h;
    bool on = false;
    if (!k || !color_on(*k) || !k->has_cam || k->frame_counter != 0 || lens_setting(lens, on)) return (int)cudaErrorInvalidValue;
    cudaSetDevice(k->device);
    CK(cudaStreamSynchronize(k->stream));
    k->has_color_lens = on;
    k->color_lens = on ? *lens : df_lens{};
    return 0;
}

extern "C" int df_kinfu_get_pose(void *h, int time, float *pose12)
{
    KinFu *k = (KinFu *)h;
    const int n = (int)(k->poses.size() / 12);
    if (time > n || time < 0) time = n - 1;                            // kinfu.cpp:213-218
    if (time >= n) time = n - 1;
    memcpy(pose12, &k->poses[(size_t)time * 12], 48);
    return 0;
}

extern "C" int df_kinfu_get_info(void *h, long long *info, int n)
{
    KinFu *k = (KinFu *)h;
    sync_extract(*k);
    if (k->last_cloud < 0) {
        int c = 0;
        cudaMemcpyAsync(&c, k->cloud_count, sizeof(int), cudaMemcpyDeviceToHost, k->stream);
        cudaStreamSynchronize(k->stream);
        k->last_cloud = c;
    }
    double st[8] = {0};
    cudaMemcpyAsync(st, k->solve_stats, sizeof st, cudaMemcpyDeviceToHost, k->stream);
    cudaStreamSynchronize(k->stream);
    unsigned long long nu2[2] = {0, 0};
    cudaMemcpyAsync(nu2, k->n_upd, 16, cudaMemcpyDeviceToHost, k->stream);
    cudaStreamSynchronize(k->stream);
    const unsigned long long nu = nu2[0];
    note_solve_overflow(*k);
    int keyframes = 0;
    if (reloc_on(*k) && n > 16) {
        cudaMemcpyAsync(&keyframes, k->kf_count, sizeof(int), cudaMemcpyDeviceToHost, k->stream);
        cudaStreamSynchronize(k->stream);
    }
    const long long vals[17] = {k->frame_counter, k->M, k->last_cloud, (long long)(k->poses.size() / 12), k->last_ok, k->launches, k->resets,
                                (long long)st[2], (long long)nu, (long long)st[4], (long long)nu2[1], k->solve_overflows, k->lm_fallbacks,
                                k->lost, k->lost_frames, k->relocalisations, keyframes};
    for (int i = 0; i < n && i < 17; ++i) info[i] = vals[i];
    return 0;
}

extern "C" int df_kinfu_get_keyframes(void *h, float *poses_host, uint8_t *codes_host, int capacity, int *n)
{
    KinFu *k = (KinFu *)h;
    if (!k || !reloc_on(*k) || !n) return (int)cudaErrorInvalidValue;
    cudaSetDevice(k->device);
    int count = 0;
    CK(cudaMemcpyAsync(&count, k->kf_count, sizeof(int), cudaMemcpyDeviceToHost, k->stream));
    CK(cudaStreamSynchronize(k->stream));
    *n = count;
    const int m = count < capacity ? count : capacity;
    if (m <= 0) return 0;
    if (poses_host) CK(cudaMemcpy(poses_host, k->kf_poses, (size_t)m * 48, cudaMemcpyDeviceToHost));
    if (codes_host) CK(cudaMemcpy(codes_host, k->kf_codes, (size_t)m * DF_RELOC_FERNS, cudaMemcpyDeviceToHost));
    return 0;
}

// stream-ordered join: the object's main stream waits for the extraction in flight on its auxiliary stream (no host synchronisation)
extern "C" int df_kinfu_join(void *h)
{
    KinFu *k = (KinFu *)h;
    return wait_extract_on_main(*k);
}

extern "C" int df_kinfu_get_buffer(void *h, int which, void **ptr, size_t *pitch, int *cols, int *rows)
{
    KinFu *k = (KinFu *)h;
    if (which == DF_KINFU_BUF_CLOUD || which == DF_KINFU_BUF_CLOUD_NORMALS || which == DF_KINFU_BUF_CLOUD_COLORS)
        sync_extract(*k);                                              // the caller is about to use the cloud on a stream of its own
    Img im;
    const int level = which >> 8, base = which & 255;                 // the ICP's pyramid levels: which + 256 * level
    if (which >= 256) {
        if (level >= k->levels || !((base >= DF_KINFU_BUF_CURR_DEPTH && base <= DF_KINFU_BUF_PREV_NORMALS) || base == DF_KINFU_BUF_INTENSITY ||
                                    base == DF_KINFU_BUF_MODEL_INTENSITY))
            return (int)cudaErrorInvalidValue;
        which = base;
    }
    if ((which == DF_KINFU_BUF_INTENSITY || which == DF_KINFU_BUF_MODEL_INTENSITY) && !(k->p.flags & DF_KINFU_COLOR_TRACKING))
        return (int)cudaErrorInvalidValue;
    switch (which) {
        case DF_KINFU_BUF_VOLUME: im.ptr = k->volume; im.pitch = (size_t)k->p.volume_dims[0] * 4; im.cols = k->p.volume_dims[0]; im.rows = k->p.volume_dims[1] * k->p.volume_dims[2]; break;
        case DF_KINFU_BUF_DISTS: im = k->dists.view(); break;
        case DF_KINFU_BUF_CURR_DEPTH: im = k->cur_depth[level].view(); break;
        case DF_KINFU_BUF_CURR_POINTS: im = k->cur_pts[level].view(); break;
        case DF_KINFU_BUF_CURR_NORMALS: im = k->cur_nrm[level].view(); break;
        case DF_KINFU_BUF_PREV_POINTS: im = k->prev_pts[level].view(); break;
        case DF_KINFU_BUF_PREV_NORMALS: im = k->prev_nrm[level].view(); break;
        case DF_KINFU_BUF_INTENSITY: im = k->cur_int[level].view(); break;
        case DF_KINFU_BUF_MODEL_INTENSITY: im = k->model_int[level].view(); break;
        case DF_KINFU_BUF_CANONICAL: im = k->canon.view(); break;
        case DF_KINFU_BUF_CANONICAL_NORMALS: im = k->canon_nrm.view(); break;
        case DF_KINFU_BUF_CLOUD: im.ptr = k->cloud; im.pitch = 16; im.cols = 1; im.rows = k->p.cloud_capacity; break;
        case DF_KINFU_BUF_CLOUD_NORMALS: im.ptr = k->cloud_nrm; im.pitch = 16; im.cols = 1; im.rows = k->p.cloud_capacity; break;
        case DF_KINFU_BUF_NODES: im.ptr = k->nodes; im.pitch = DF_NODE_STRIDE * 4; im.cols = 1; im.rows = k->M; break;
        case DF_KINFU_BUF_CANONICAL_VISIBLE: im = k->canon_visible.view(); break;
        case DF_KINFU_BUF_SOLVE_STATS: im.ptr = k->solve_stats; im.pitch = 64; im.cols = 8; im.rows = 1; break;
        case DF_KINFU_BUF_F2_STATS: im.ptr = k->f2_stats; im.pitch = 128; im.cols = 16; im.rows = 1; break;
        case DF_KINFU_BUF_ACTIVITY: im.ptr = k->activity; im.pitch = k->activity_bytes; im.cols = (int)k->activity_bytes; im.rows = 1; break;
        case DF_KINFU_BUF_COLOR_VOLUME: if (!color_on(*k)) return (int)cudaErrorInvalidValue;
                 im.ptr = k->color_vol; im.pitch = (size_t)k->p.volume_dims[0] * 4; im.cols = k->p.volume_dims[0]; im.rows = k->p.volume_dims[1] * k->p.volume_dims[2]; break;
        case DF_KINFU_BUF_CLOUD_COLORS: if (!color_on(*k)) return (int)cudaErrorInvalidValue;
                 im.ptr = k->cloud_rgba; im.pitch = 4; im.cols = 1; im.rows = k->p.cloud_capacity; break;
        case DF_KINFU_BUF_COLOR_MAP: if (!k->has_cam) return (int)cudaErrorInvalidValue;
                 im = k->color_map.view(); break;
        default: return (int)cudaErrorInvalidValue;
    }
    *ptr = im.ptr; *pitch = im.pitch; *cols = im.cols; *rows = im.rows;
    return 0;
}

extern "C" int df_kinfu_read_buffer(void *h, int which, void *dst_host, size_t bytes)
{
    KinFu *k = (KinFu *)h;
    void *ptr; size_t pitch; int cols, rows;
    const int st = df_kinfu_get_buffer(h, which, &ptr, &pitch, &cols, &rows);
    if (st) return st;
    const size_t have = pitch * (size_t)rows;
    sync_extract(*k);
    cudaError_t e = cudaStreamSynchronize(k->stream);
    if (e != cudaSuccess) return (int)e;
    e = cudaMemcpy(dst_host, ptr, bytes < have ? bytes : have, cudaMemcpyDeviceToHost);
    return (int)e;
}

extern "C" int df_kinfu_set_overrides(void *h, const uint16_t *bilateral_depth_host, size_t pitch, const float *pose12_host, const float *nodes_host, int M)
{
    KinFu *k = (KinFu *)h;
    k->has_ov_depth = bilateral_depth_host != nullptr;
    if (bilateral_depth_host) {
        k->ov_depth.resize((size_t)k->p.cols * k->p.rows);
        for (int y = 0; y < k->p.rows; ++y) memcpy(&k->ov_depth[(size_t)y * k->p.cols], (const char *)bilateral_depth_host + (size_t)y * pitch, (size_t)k->p.cols * 2);
    }
    k->has_ov_pose = pose12_host != nullptr;
    if (pose12_host) memcpy(k->ov_pose, pose12_host, 48);
    k->has_ov_nodes = nodes_host != nullptr && M > 0;
    if (k->has_ov_nodes) k->ov_nodes.assign(nodes_host, nodes_host + (size_t)M * DF_NODE_STRIDE);
    return 0;
}

extern "C" int df_kinfu_set_f2_params(void *h, const df_f2_params *prm)
{
    KinFu *k = (KinFu *)h;
    if (!prm) return (int)cudaErrorInvalidValue;
    k->f2 = *prm;
    if (k->f2.reg_k > 7) k->f2.reg_k = 7;
    return 0;
}

extern "C" int df_kinfu_state_digest(void *h, unsigned long long *out4_host)
{
    KinFu *k = (KinFu *)h;
    sync_extract(*k);
    DevMem<unsigned long long> d;
    if (d.alloc(32) != cudaSuccess) return (int)cudaGetLastError();
    cudaMemsetAsync(d, 0, 32, k->stream);
    const size_t nvox = (size_t)k->p.volume_dims[0] * k->p.volume_dims[1] * k->p.volume_dims[2];
    digest_kernel<<<DF_NUM_SMS * 8, 256, 0, k->stream>>>(k->volume, nvox, d);
    if (k->M > 0) digest_kernel<<<8, 256, 0, k->stream>>>((const uint32_t *)k->nodes.p, (size_t)k->M * DF_NODE_STRIDE, d + 1);
    cudaMemcpyAsync(d + 2, k->cloud_count, sizeof(int), cudaMemcpyDeviceToDevice, k->stream);
    cudaError_t e = cudaMemcpyAsync(out4_host, d, 32, cudaMemcpyDeviceToHost, k->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(k->stream);
    if (e != cudaSuccess) return (int)e;
    unsigned long long ph = 0x243f6a8885a308d3ull;                      // camera poses so far, bit pattern by bit pattern
    for (float f : k->poses) { uint32_t u; memcpy(&u, &f, 4); ph = (ph ^ u) * 0x100000001b3ull; }
    out4_host[3] = ph;
    return 0;
}

extern "C" int df_kinfu_get_stage_ms(void *h, float *ms, int n)
{
    KinFu *k = (KinFu *)h;
    const int m = n < NSTAGES ? n : NSTAGES;
    for (int i = 0; i < m; ++i) ms[i] = k->stage_ms[i];
    return m;
}
