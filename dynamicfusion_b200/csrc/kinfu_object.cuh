// kinfu_object.cuh -- the frame loop's object (KinFu) and the helpers its translation units share: the loop (pipeline.cu), snapshots
// (kinfu_snapshot.cu) and the mesh entries (kinfu_mesh.cu).  Internal: the C ABI is include/dfusion.h.
#pragma once
#include "df_common.cuh"
#include <cstring>
#include <utility>
#include <vector>

namespace dfb::kinfu {

constexpr int MAX_LEVELS = 4;      // ProjectiveICP::MAX_PYRAMID_LEVELS, projective_icp.hpp:12
constexpr int NSTAGES = 10;

// internal helpers and stages return 0 or a positive status (a cudaError_t value, or what a df_* launcher returned); each extern "C"
// entry point turns it into its documented convention once, where it returns
#define CK(call)                                      \
    do {                                              \
        const int s__ = (int)(call);                  \
        if (s__ != 0) return s__;                     \
    } while (0)

// device memory owned by whoever holds it: freed on destruction, moved (and so swapped) but never copied
template <class T> struct DevMem {
    T *p = nullptr;
    DevMem() = default;
    DevMem(DevMem &&o) noexcept : p(o.p) { o.p = nullptr; }
    DevMem &operator=(DevMem &&o) noexcept { std::swap(p, o.p); return *this; }   // what this held is freed with `o`
    ~DevMem() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t bytes) { return cudaMalloc((void **)&p, bytes ? bytes : 16); }
    operator T *() const { return p; }
};

// a pitched image; `mem` holds `ptr` for the object's own images and is empty in a view of a caller's buffer
struct Img {
    void *ptr = nullptr; size_t pitch = 0; int cols = 0, rows = 0;
    DevMem<void> mem;
    Img view() const { return Img{ptr, pitch, cols, rows}; }
};

struct KinFu {
    df_kinfu_params p;
    int device = 0;                       // the CUDA device the object was created on; every entry point switches to it
    cudaStream_t stream = 0;
    int levels = 0;                       // used_levels(p)
    int max_nodes_cap = 0;                // node_capacity(p)
    float vol_pose[12], Rinv_vol[9];      // p.volume_pose as 12 floats, and the inverse of its rotation
    float trunc_dist = 0.f;
    float voxel_size[3];
    DevMem<uint32_t> volume;
    Img depth_in, dists;
    Img cur_depth[MAX_LEVELS], cur_pts[MAX_LEVELS], cur_nrm[MAX_LEVELS], prev_pts[MAX_LEVELS], prev_nrm[MAX_LEVELS];
    Img prev_depth[MAX_LEVELS];           // DF_KINFU_USE_DEPTH only: the model's depth pyramid (prev_.depth_pyr)
    Img canon, canon_nrm, canon_visible;
    DevMem<float> cloud, cloud_nrm; DevMem<int> cloud_count;
    DevMem<float> nodes; int M = 0; DevMem<void> node_grid;
    DevMem<float> icp_T; DevMem<int> icp_ok; DevMem<double> icp_scratch;
    DevMem<void> solve_ws; DevMem<double> solve_stats;
    DevMem<double> f2_stats;
    DevMem<void> extract_ws, project_ws;
    DevMem<void> integrate_ws;
    DevMem<void> extend_ws; DevMem<int> M_dev;   // df_extend_field workspace / new node count (DF_KINFU_EXTEND_FIELD)
    DevMem<void> fusion_ws;               // df_integrate_warped workspace (DF_KINFU_WARPED_INTEGRATE)
    DevMem<unsigned char> activity; size_t activity_bytes = 0;   // dfusion.h DF_ACTIVITY_VOXELS: which stretches of the volume hold surface
    // DF_KINFU_COLOR: the colour volume (dfusion.h), one RGBA word per cloud slot, and the device copy of a host frame's BGRA image.  frame_bgra
    // is the colour image of the frame being processed (null: a depth-only frame, which leaves the colour volume as it was)
    DevMem<uint32_t> color_vol, cloud_rgba; Img color_in;
    const void *frame_bgra = nullptr; size_t frame_bgra_pitch = 0;
    // df_kinfu_set_color_camera: the colour camera's calibration (has_cam; color_in then has the colour image's size) and the occlusion map
    // df_color_depth_map builds from each colour frame's input depth.  Calibration, not state: reset keeps it
    bool has_cam = false; df_color_camera cam = {}; Img color_map;
    // df_kinfu_set_depth_lens / _set_color_lens: the lenses (never the zero lens; has_* false = a pinhole) and, while a depth lens is set,
    // the frame's undistorted depth and registered colour image (df_undistort), which every stage reads instead of the caller's (bgra_ud
    // only on a colour object without a colour camera: a colour camera's image is projected through its own lens instead).
    // Calibration, not state: reset keeps them
    bool has_depth_lens = false, has_color_lens = false; df_lens depth_lens = {}, color_lens = {};
    Img depth_ud, bgra_ud;
    // DF_KINFU_COLOR_TRACKING: the colour frame's intensity pyramid (float) and the model's intensity maps (float4 (I, gu, gv, 0)) per ICP level
    Img cur_int[MAX_LEVELS], model_int[MAX_LEVELS];
    Img rc_ids, rc_pts, rc_nrm;           // df_kinfu_render_colors: the maps it renders into; allocated by the first call
    const float *rm_pts = nullptr; int rm_N = 0, rm_T = 0;   // the vertex buffer and sizes of the last render_mesh()
    DevMem<void> mesh_ws; DevMem<int> mesh_dev;   // df_kinfu_mesh: df_mesh_* workspace, {triangles, status}; allocated by the first call
    // df_kinfu_mesh / df_kinfu_render: the triangles, the live copy of the cloud (points, then normals) and df_raster_mesh's workspace;
    // allocated on first use, grown when too small (capacities in bytes)
    DevMem<int32_t> mesh_tris; size_t mesh_tris_bytes = 0;
    DevMem<float> mesh_moved; size_t mesh_moved_bytes = 0;
    DevMem<void> raster_ws; size_t raster_ws_bytes = 0;
    // DF_KINFU_LIVE_MODEL: the live mesh kept for the next frame (lm_valid): the cloud moved to the ray-cast's voxel convention (lm_src), the
    // same carried through the warp field (lm_live: points, then normals), lm_N points, lm_T faces in mesh_tris (read through the member at
    // every use: a re-grow by df_kinfu_mesh / _render re-emits the same faces); lm_ids is the association render's triangle map
    DevMem<float> lm_src, lm_live; size_t lm_src_bytes = 0, lm_live_bytes = 0;
    Img lm_ids;
    int lm_N = 0, lm_T = 0;
    bool lm_valid = false;
    bool field_frame = false;            // the last dynamicfusion() warped and solved (a warp field, not a rigid frame)
    float lm_shift[3] = {0.f, 0.f, 0.f}; // R_vol * (vs/2): extraction puts voxel i at (i + 1/2) vs, integrate and the ray-cast at i vs
    long long lm_fallbacks = 0; bool lm_fell_back = false;   // frames without a live model; info[12]
    // DF_KINFU_RELOCALISE (all allocated with the flag only): the fern table of the level-2 image, the frame's code, the keyframe database
    // (codes, poses, count on the device: the match kernel appends without a host round trip), the gate's workspace and result with its
    // pinned copy, the lookup's result, and the pyramid a keyframe candidate is ray-cast into (the kept previous-frame maps survive a
    // failed attempt).  lost: the last frame failed the gate; the last good pose is poses.back().  info[13..16]
    DevMem<int32_t> fern_table; DevMem<uint8_t> frame_code, kf_codes; DevMem<float> kf_poses; DevMem<int> kf_count;
    DevMem<void> gate_ws; DevMem<df_reloc_gate> gate; DevMem<df_reloc_match> match;
    df_reloc_gate *gate_host = nullptr; df_reloc_match *match_host = nullptr;
    Img rl_pts[MAX_LEVELS], rl_nrm[MAX_LEVELS];
    bool lost = false;
    long long lost_frames = 0, relocalisations = 0;
    float *pinned = nullptr;            // 16 floats: T(12) + ok
    std::vector<float> poses;            // 12 floats per pose
    int frame_counter = 0, resets = 0, last_ok = 1, launches = 0;
    // df_kinfu_set_overrides (lock-step parity hook): one-shot replacements for the NEXT frame
    std::vector<uint16_t> ov_depth; bool has_ov_depth = false;       // bilateral-filtered depth, dense cols x rows
    float ov_pose[12]; bool has_ov_pose = false;                     // absolute camera pose of the frame
    std::vector<float> ov_nodes; bool has_ov_nodes = false;          // node table after the solve
    df_f2_params f2; DevMem<void> f2_ws;  // DF_KINFU_F2_SOLVE (SURVEY 8f(2))
    long long solve_overflows = 0;       // frames whose solve was skipped because a normal-matrix row overflowed (solve.cu ROWCAP); info[11]
    long long last_cloud = -1;
    double host_us[4] = {0, 0, 0, 0}; long long host_frames = 0;   // DF_KINFU_HOSTPROF: launch A, ICP wait, launch B, total
    DevMem<unsigned long long> n_upd;    // voxels written by the last integrate (filled when DF_KINFU_STAGE_TIMING)
    // Extraction runs on a second stream: nothing later in the frame loop reads the extracted cloud (the reference recomputes it every
    // frame for its host copies, kinfu.cpp:398-399), it only READS the volume, and the volume is not written again before the next
    // frame's integrate -- so it overlaps the ray-cast and the next frame's pre-processing + ICP (mostly launch latency).
    cudaStream_t aux = nullptr;           // extraction stream (non-blocking, lowest priority: the main stream's kernels are placed first)
    cudaEvent_t ev_volume_ready = nullptr, ev_extract_done = nullptr, ev_before_lm = nullptr;
    bool extract_deferred = false;        // frame t's extraction has not been launched yet: it starts when frame t+1's LM/PCG kernel does
                                          // (one 16-SM cluster while the other SMs idle), or as soon as anybody needs the cloud or the volume
    bool extract_pending = false;         // an extraction is in flight on `aux`
    bool overlap_extract = true;          // DF_KINFU_OVERLAP_EXTRACT=0: everything on one stream
    cudaEvent_t ev[NSTAGES + 1] = {};
    float stage_ms[NSTAGES] = {};
    int stage_mark[NSTAGES + 1] = {};

    // the work queued on both streams finishes before the device memory above is released
    ~KinFu()
    {
        cudaSetDevice(device);
        cudaStreamSynchronize(stream);
        if (aux) { cudaStreamSynchronize(aux); cudaStreamDestroy(aux); }
        for (cudaEvent_t e : {ev_volume_ready, ev_before_lm, ev_extract_done}) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        cudaFreeHost(pinned);
        if (gate_host) cudaFreeHost(gate_host);
        if (match_host) cudaFreeHost(match_host);
    }
};

inline int alloc_img(Img &im, int rows, int cols, size_t elem)
{
    im.cols = cols; im.rows = rows; im.pitch = (size_t)cols * elem;     // dense rows (pitch is still carried everywhere)
    const cudaError_t e = im.mem.alloc(im.pitch * rows);
    im.ptr = im.mem;
    return (int)e;
}

// `m` holds at least `need` bytes (its contents are not kept when it grows)
template <class T> int grow(DevMem<T> &m, size_t &have, size_t need)
{
    if (m && have >= need) return 0;
    DevMem<T> fresh;
    CK(fresh.alloc(need));
    m = std::move(fresh);                                              // the old block is freed with `fresh`
    have = need;
    return 0;
}

// getUsedLevelsNum, projective_icp.cpp:110-115
inline int used_levels(const df_kinfu_params &p)
{
    int i = MAX_LEVELS - 1;
    for (; i >= 0 && !p.icp_iter_num[i]; --i) {}
    return i + 1;
}

inline df_volume vol_of(const KinFu &k)
{
    df_volume v;
    v.data = k.volume;
    for (int i = 0; i < 3; ++i) { v.dims[i] = k.p.volume_dims[i]; v.voxel_size[i] = k.voxel_size[i]; }
    v.trunc_dist = k.trunc_dist; v.max_weight = k.p.tsdf_max_weight;
    return v;
}

inline bool color_on(const KinFu &k) { return (k.p.flags & DF_KINFU_COLOR) != 0; }
inline bool reloc_on(const KinFu &k) { return (k.p.flags & DF_KINFU_RELOCALISE) != 0; }
// the colour volume as a df_volume, for the calls that treat it as one (clear, brick packing)
inline df_volume color_vol_of(const KinFu &k) { df_volume v = vol_of(k); v.data = k.color_vol; return v; }

// the colour camera's lens for the _lens entries (NULL: a pinhole)
inline const df_lens *color_lens_of(const KinFu &k) { return k.has_color_lens ? &k.color_lens : nullptr; }

inline df_aff3f to_aff(const float *a12) { df_aff3f a; memcpy(a.R, a12, 36); memcpy(a.t, a12 + 9, 12); return a; }
constexpr df_aff3f AFF_IDENTITY = {{1.f, 0.f, 0.f, 0.f, 1.f, 0.f, 0.f, 0.f, 1.f}, {0.f, 0.f, 0.f}};

// the latest camera pose (poses_.back()); there is always one
inline const float *latest_pose(const KinFu &k) { return &k.poses[k.poses.size() - 12]; }

// host-side readers of the cloud (count, buffers, digest) make sure the extraction has been launched and wait for it
void sync_extract(KinFu &k);
// reports, once per frame, a solve skipped because a normal-matrix row overflowed (pipeline.cu)
void note_solve_overflow(KinFu &k);

// the mesh of the current state (kinfu_mesh.cu), shared by df_kinfu_mesh / df_kinfu_render and the live model of DF_KINFU_LIVE_MODEL.
// mesh_count_now completes the last frame's extraction, counts the triangles (df_mesh_count: 7 launches) and reads back the triangle count,
// the status and the cloud's point count: one host synchronisation.  match: the cloud matches the volume.
int mesh_count_now(KinFu &k, int &N, int &T, bool &match);
// after mesh_count_now: the T triangles into k.mesh_tris and the vertex buffer (float4 points and, when `nrm` is not null, normals of the N
// cloud points): the cloud itself, or for `live` copies of it carried through the warp field by the frame loop's own df_warp call
// (kinfu.cpp:385)
int mesh_build(KinFu &k, int live, int N, int T, const float *&pts, const float **nrm);

}  // namespace dfb::kinfu
