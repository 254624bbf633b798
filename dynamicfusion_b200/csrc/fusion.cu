// fusion.cu -- per-voxel warped TSDF integration on sm_90a (SURVEY.md 8f(1)): k-NN + node weights + dual-quaternion blend +
// projective signed distance + weighted running average fused into one kernel over the voxels that can be updated.
//
// The reference stops short of this step: TsdfVolume::surface_fusion (kfusion/src/tsdf_volume.cpp:228-254) evaluates psdf() for the
// warped ray-cast points, runs the RIGID integrate and leaves the per-entry update commented out (:248-251).  The update built here
// is the one that code was written towards (DynamicFusion eq. 4-5), assembled only from operations the reference defines, in the
// reference's operation order (each cited below); the CPU restatement it is tested against is oracle/orc_fusion.c.
//
//   x_c = pose_vol * (x*vs, y*vs, z*vs)            TsdfIntegrator's voxel position (tsdf_volume.cu:62-64), Aff3f * float3 (device.hpp:71-74)
//   8-NN of x_c, weights, DQB, transform           WarpField::KNN / weighting / DQB / warp (warp_field.cpp:180-251)
//   x_t = world2cam * x_w                          cv::Affine3f * Vec3f (the last step of WarpField::warp)
//   rho = depth(floor v, floor u) * 0.001 - x_t.z  TsdfVolume::psdf (tsdf_volume.cpp:266-292) with Projector (device.hpp:32-38)
//   if rho > -trunc:  tsdf = min(1, rho / trunc);  w = mean node distance (TsdfVolume::weighting, :300-306) quantised to the u16 weight;
//                     F' = (F*W + tsdf*w) / (W + w), W' = min(W + w, max_weight)          (:248-251 in the arithmetic of tsdf_volume.cu:97-103)
//
// Cost model.  Unlike the rigid rule, a voxel's pixel is only known after its warp, i.e. after an exact 8-NN search and a blend with
// eight double-precision exponentials (~2 k instructions): the kernel is instruction-bound by three orders of magnitude over its
// 8 bytes of volume traffic per written voxel, so the design levers are (i) not searching for voxels that cannot be updated and
// (ii) making the search cheap:
//   (i)  a warp owns an 8 x 4 voxel footprint; before every run of FUS_SUB slices it tests the sub-brick GROWN BY THE LARGEST
//        DISPLACEMENT THE FIELD CAN PRODUCE against the frustum and against the per-tile depth maxima (three levels: 16-pixel tiles,
//        64-pixel tiles, whole image).  The bound: weights are exp(-d^2/2s^2) <= 1 and are not normalised (warp_field.cpp:203-217), so
//        |x_w - x_c| <= 8 max_i |t_i| when every node rotation is the identity (true for everything the translation-only solve
//        produces); one small kernel per call reduces it over the node table and reports +inf (no culling) if any node is rotated.
//   (ii) consecutive voxels of a z-column have almost the same neighbours: the previous voxel's eight neighbours, re-measured from the new
//        voxel, seed the branch-and-bound (knn8_bvh_seeded) so that it prunes with a near-final bound from the first box on and inserts only
//        the few nodes that actually changed.  Results are ranked by (distance, index) on every path: identical to the exhaustive scan.
#include "warp_common.cuh"
#include "color_sample.cuh"
#include <cmath>
#include <cstdlib>

using namespace dfb;

namespace {

constexpr int FUS_SUB = 8;          // slices per visibility test
constexpr int FUS_TILE = 16;        // fine depth tiles (pixels)
constexpr int FUS_COARSE = 4;       // coarse tile = FUS_COARSE x FUS_COARSE fine tiles
constexpr int FUS_LIST_CAP = 768;   // candidate nodes per warp run, as 16-bit positions in the block list (1.5 KB per warp)
constexpr int FUS_BLOCK_CAP = 2048; // candidate nodes of a block's 32 x 8 x zchunk region (float4 each, 32 KB): what the warp runs select from

struct FusionParams {
    uint32_t *data;
    int Dx, Dy, Dz;
    float vsx, vsy, vsz;
    float trunc, trunc_inv;
    int max_weight;
    const unsigned short *depth;
    size_t pitch;
    int cols, rows;
    float fcols, frows;
    Aff vol2world, world2cam, vol2cam;     // vol2cam = world2cam o vol2world: used by the visibility test only
    float fx, fy, cx, cy;
    const float *nodes; int M; const void *grid;
    const float4 *node_rec;                // three arrays of M records (fusion_prepare_kernel): [i] rotation quaternion, [M + i] translation quaternion, [2M + i] (vertex, weight)
    float weight_scale;
    int cull;                              // 0: the two poses are not rigid -> no visibility test
    const float *ws;                       // [0] displacement bound, [1] global depth maximum, [2] 1 = every node rotation is the identity, [16..] fine tile maxima, then coarse
    int tiles_x, tiles_y, ctiles_x, ctiles_y;
    int zchunk;
    unsigned long long *counters;          // [0] voxels written, [1] voxels warped
    unsigned char *activity;
    BrickTable bricks;
    int use_list;                          // candidate lists per warp run (round 2, see integrate_warped_body); 0: branch-and-bound per voxel only
    float half_diag;                       // upper bound on the distance (world space) from a run's centre to any of its voxel centres
    float half_diag_block;                 // the same for the block's 32 x 8 x zchunk region
};

// The colour side of df_integrate_warped_color: kColor selects what a warped voxel in the band samples (WC_NONE: no colour side at all --
// df_integrate_warped's instances); kLens (WC_CAMERA only) projects through the colour camera's lens, as color.cu's LENS instances do.
enum { WC_NONE = 0, WC_REGISTERED = 1, WC_CAMERA = 2 };

struct WarpedColorParams {
    uint32_t *colors;                      // the colour volume, laid out as the TSDF volume
    const uchar4 *bgra; size_t cpitch;     // the frame's colour image: registered to the depth (cols x rows) or the colour camera's
    float band;                            // DF_COLOR_BAND * trunc_dist
    int wcap;                              // min(max_weight, 255)
    OcclusionParams o;                     // WC_CAMERA: the colour camera, the frame's df_color_depth_map and DF_COLOR_OCCLUSION * trunc_dist
    unsigned long long *counter;           // optional (the entry's counters[2]): += voxels that took a colour sample
};

// metric depth maxima per FUS_TILE x FUS_TILE pixel tile
__global__ void __launch_bounds__(256) depth_tile_max_kernel(const unsigned short *__restrict__ depth, size_t pitch, int cols, int rows, float *tile_max, int tiles_x)
{
    DF_PDL_ENTRY();
    const int tx = blockIdx.x, ty = blockIdx.y;
    const int x = tx * FUS_TILE + (threadIdx.x & (FUS_TILE - 1)), y = ty * FUS_TILE + (threadIdx.x / FUS_TILE);
    float v = 0.f;
    if (x < cols && y < rows) v = (float)__ldg(row_ptr(depth, pitch, y) + x) * 0.001f;
    __shared__ float wm[8];
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = wm[0];
        for (int i = 1; i < 8; ++i) m = fmaxf(m, wm[i]);
        tile_max[ty * tiles_x + tx] = m;
    }
}

// block 0: coarse tile maxima + global maximum from the fine ones; block 1: displacement bound of the node table and the per-node
// (rotation, translation) records -- DualQuaternion::getTranslation (dual_quaternion.hpp:120-125) depends on the node alone
__global__ void __launch_bounds__(256) fusion_prepare_kernel(float *ws, int tiles_x, int tiles_y, int ctiles_x, int ctiles_y, const float *__restrict__ nodes, int M,
                                                             float4 *node_rec)
{
    DF_PDL_ENTRY();
    __shared__ float red[256];
    __shared__ int flag;
    const int t = threadIdx.x;
    float *fine = ws + 16, *coarse = fine + tiles_x * tiles_y;
    if (blockIdx.x == 0) {
        float g = 0.f;
        for (int c = t; c < ctiles_x * ctiles_y; c += 256) {
            const int cx = c % ctiles_x, cy = c / ctiles_x;
            float m = 0.f;
            for (int j = 0; j < FUS_COARSE; ++j)
                for (int i = 0; i < FUS_COARSE; ++i) {
                    const int fx = cx * FUS_COARSE + i, fy = cy * FUS_COARSE + j;
                    if (fx < tiles_x && fy < tiles_y) m = fmaxf(m, fine[fy * tiles_x + fx]);
                }
            coarse[c] = m;
            g = fmaxf(g, m);
        }
        red[t] = g;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) { if (t < o) red[t] = fmaxf(red[t], red[t + o]); __syncthreads(); }
        if (t == 0) ws[1] = red[0];
    } else {
        if (t == 0) flag = 0;
        __syncthreads();
        float tmax = 0.f;
        bool rotated = false;
        for (int i = t; i < M; i += 256) {
            const float4 *n4 = reinterpret_cast<const float4 *>(nodes + (size_t)i * DF_NODE_STRIDE);
            const float4 a = __ldg(n4), b = __ldg(n4 + 1), c = __ldg(n4 + 2);
            const Quat rot = {a.w, b.x, b.y, b.z};
            const Quat dual = {b.w, c.x, c.y, c.z};
            if (!(rot.w == 1.f && rot.x == 0.f && rot.y == 0.f && rot.z == 0.f)) rotated = true;
            const Quat tr = dq_translation(rot, dual);
            node_rec[i] = make_float4(rot.w, rot.x, rot.y, rot.z);          // the blend needs only these per neighbour: 8 normalisations
            node_rec[M + i] = make_float4(tr.w, tr.x, tr.y, tr.z);          // and quaternion products per voxel leave the inner loop.  Array by array:
            node_rec[2 * M + i] = make_float4(a.x, a.y, a.z, c.w);          // the identity path never touches the rotations, 64 KB at 2 k nodes stay in L1
            const float len = sqrtf(tr.x * tr.x + tr.y * tr.y + tr.z * tr.z);
            tmax = fmaxf(tmax, len);
            if (!(len == len)) rotated = true;              // NaN translation: no bound
        }
        if (rotated) atomicOr(&flag, 1);
        red[t] = tmax;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) { if (t < o) red[t] = fmaxf(red[t], red[t + o]); __syncthreads(); }
        if (t == 0) { ws[0] = flag ? __int_as_float(0x7f800000) : 8.f * red[0] * 1.0001f + 1e-6f; ws[2] = flag ? 0.f : 1.f; }
    }
}

// true when no voxel with x in [xa, xb], y in [ya, yb], z in [za, zb] can be updated whatever the field does to it within `delta`:
// the sub-brick, grown by one voxel and by delta along every volume axis (this contains its Minkowski sum with the delta-ball), is
// convex, so half-space tests on its eight corners decide the frustum; every point of it is at least zmin deep, so
// rho = Dp - z <= max depth of the tiles it can project to - zmin.
__device__ __forceinline__ bool fusion_run_invisible(const FusionParams &p, int lane, float delta, int xa, int xb, int ya, int yb, int za, int zb)
{
    const int k = lane & 7;
    const float3 c = make_float3((k & 1) ? (float)(xb + 1) * p.vsx + delta : (float)(xa - 1) * p.vsx - delta,
                                 (k & 2) ? (float)(yb + 1) * p.vsy + delta : (float)(ya - 1) * p.vsy - delta,
                                 (k & 4) ? (float)(zb + 1) * p.vsz + delta : (float)(za - 1) * p.vsz - delta);
    const float3 pc = aff_mul(p.vol2cam, c);
    const unsigned full = 0xffffffffu;
    if (__all_sync(full, pc.z < -1e-3f)) return true;             // x_t.z <= 0 for every voxel
    if (__any_sync(full, !(pc.z > 1e-2f))) return false;          // straddles the camera plane: no projective reasoning
    const float u = p.fx * (pc.x / pc.z) + p.cx, v = p.fy * (pc.y / pc.z) + p.cy;
    if (__all_sync(full, u < -1.f) || __all_sync(full, v < -1.f) || __all_sync(full, u > p.fcols + 1.f) || __all_sync(full, v > p.frows + 1.f)) return true;
    float umin = u, umax = u, vmin = v, vmax = v, zmin = pc.z;
    for (int o = 4; o > 0; o >>= 1) {
        umin = fminf(umin, __shfl_xor_sync(full, umin, o)); umax = fmaxf(umax, __shfl_xor_sync(full, umax, o));
        vmin = fminf(vmin, __shfl_xor_sync(full, vmin, o)); vmax = fmaxf(vmax, __shfl_xor_sync(full, vmax, o));
        zmin = fminf(zmin, __shfl_xor_sync(full, zmin, o));
    }
    const int px0 = max(0, (int)floorf(umin - 1.f)), px1 = min(p.cols - 1, (int)floorf(umax + 1.f));
    const int py0 = max(0, (int)floorf(vmin - 1.f)), py1 = min(p.rows - 1, (int)floorf(vmax + 1.f));
    if (px1 < px0 || py1 < py0) return true;                      // projects entirely off the image
    float m;
    {
        const float *fine = p.ws + 16;
        int tx0 = px0 / FUS_TILE, tx1 = px1 / FUS_TILE, ty0 = py0 / FUS_TILE, ty1 = py1 / FUS_TILE, stride = p.tiles_x;
        const float *tiles = fine;
        int nx = tx1 - tx0 + 1, nt = nx * (ty1 - ty0 + 1);
        if (nt > 32) {                                             // too many fine tiles: 64-pixel tiles
            tiles = fine + p.tiles_x * p.tiles_y; stride = p.ctiles_x;
            tx0 /= FUS_COARSE; tx1 /= FUS_COARSE; ty0 /= FUS_COARSE; ty1 /= FUS_COARSE;
            nx = tx1 - tx0 + 1; nt = nx * (ty1 - ty0 + 1);
        }
        if (nt > 32) m = __ldg(p.ws + 1);                          // whole image
        else {
            m = 0.f;
            if (lane < nt) m = __ldg(tiles + (ty0 + lane / nx) * stride + tx0 + lane % nx);
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(full, m, o));
        }
    }
    return zmin - 1e-3f > m + p.trunc;                             // rho < -trunc (or no depth at all) for every voxel of the run
}

// WarpField::DQB (warp_field.cpp:203-217) + DualQuaternion::transform (dual_quaternion.hpp:204-210) of the voxel position, as
// dqb_blend() / dq_transform() compute them, with every node's getTranslation() read from the records instead of being re-derived per
// voxel: same float values, same accumulation order, same result bit for bit.
//
// kIdentity (every node rotation is exactly (1,0,0,0): fusion_prepare_kernel checked it): the rotation sum is (W,0,0,0) with W > 0, and
// then every later step is the identity in IEEE arithmetic -- sqrtf(W*W) == W, (float)((1.0/W)*W) == 1.f, a quaternion product with
// (1,0,0,0) returns its other operand (x*1 == x, x +- 0 == x), halving and doubling are exact, and rotate() adds a cross product with the
// zero vector -- so DQB(x).transform(x) == x + (sum_i w_i t_i).xyz bit for bit, and the normalisations (three double divisions), the two
// quaternion products and the rotation are not executed.  (Only the sign of an exactly-zero component can differ, which no later
// operation distinguishes.)  The parity tests compare this path with the oracle's unabridged arithmetic voxel for voxel.
template <bool kIdentity>
__device__ __forceinline__ float3 fusion_warp_point(const FusionParams &p, const int (&bi)[8], const float (&bd)[8], const float3 xc)
{
    Quat tsum = {0.f, 0.f, 0.f, 0.f}, rsum = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        if (bi[i] >= 0) {
            const float4 t = __ldg(p.node_rec + p.M + bi[i]), pw = __ldg(p.node_rec + 2 * p.M + bi[i]);
            const float w = node_weighting(bd[i], pw.w);
            tsum.w = tsum.w + w * t.x; tsum.x = tsum.x + w * t.y; tsum.y = tsum.y + w * t.z; tsum.z = tsum.z + w * t.w;
            if (!kIdentity) {
                const float4 r = __ldg(p.node_rec + bi[i]);
                rsum.w = rsum.w + w * r.x; rsum.x = rsum.x + w * r.y; rsum.y = rsum.y + w * r.z; rsum.z = rsum.z + w * r.w;
            }
        }
    }
    if (kIdentity) return make_float3(xc.x + tsum.x, xc.y + tsum.y, xc.z + tsum.z);
    Dqb d;
    d.rot = qnormalize(rsum);
    d.dual = qmul(qhalf(tsum), d.rot);
    return dq_transform(d, xc);
}

// TsdfVolume::weighting (tsdf_volume.cpp:300-306) quantised to the volume's u16 weight
__device__ __forceinline__ int fusion_sample_weight(const FusionParams &p, const int (&bi)[8], const float (&bd)[8])
{
    if (!(p.weight_scale > 0)) return 1;
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) if (bi[k] >= 0) sum += sqrtf(bd[k]);
    const float w = sum / 8;
    const float s = rintf(w * p.weight_scale);
    return s < 1.f ? 1 : (s > (float)p.max_weight ? p.max_weight : (int)s);
}

// The per-voxel search of round 1 (branch-and-bound over the node BVH seeded with the z-predecessor's neighbours, or the grid walk when
// the field has no BVH): now the fallback for runs without a candidate list.  Out of line on purpose -- three inlined tree walks with
// unrolled leaf loops were most of the kernel's 200 KB of code, and the kernel is bound by instruction fetch.
__device__ __noinline__ void fusion_tree_search(const void *grid, const float4 *node_pos, const float3 xc, bool have_prev, const int *prev, int *bi_out, float *bd_out)
{
    const NodeGridHeader h = *reinterpret_cast<const NodeGridHeader *>(grid);
    const bool has_bvh = h.pad[2] != 0;
    const float4 *bvh_box = reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(grid) + h.pad[2]);
    const float4 *bvh_leaf = reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(grid) + h.pad[3]);
    int bi[8]; float bd[8];
    if (has_bvh) {
        bool seeded = false;
        if (have_prev) {                                           // the previous voxel's neighbours at this voxel's position
            seeded = true;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float4 v = __ldg(node_pos + prev[k]);
                const float d0 = xc.x - v.x, d1 = xc.y - v.y, d2 = xc.z - v.z;
                bi[k] = prev[k];
                bd[k] = d0 * d0 + d1 * d1 + d2 * d2;
                seeded = seeded && bd[k] == bd[k];
            }
        } else {
            seeded = knn8_bvh_greedy_seed(bvh_box, bvh_leaf, h.pad[4], xc.x, xc.y, xc.z, bi, bd);
        }
        if (seeded) knn8_bvh_seeded(bvh_box, bvh_leaf, h.pad[4], xc.x, xc.y, xc.z, bi, bd);
        else knn8_bvh_bounded(bvh_box, bvh_leaf, h.pad[4], xc.x, xc.y, xc.z, 3.402823466e+38f, bi, bd);
    } else {
        knn8_grid(grid, true, xc.x, xc.y, xc.z, bi, bd);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) { bi_out[k] = bi[k]; bd_out[k] = bd[k]; }
}

template <bool kIdentity, int kColor = WC_NONE, bool kLens = false>
__device__ __forceinline__ void integrate_warped_body(const FusionParams &p, const WarpedColorParams *wc = nullptr, const df_lens *lens = nullptr)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int xw = blockIdx.x * 32 + (warp & 3) * 8, yw = blockIdx.y * 8 + (warp >> 2) * 4;       // the warp's 8 x 4 voxel footprint
    const int x = xw + (lane & 7), y = yw + (lane >> 3);
    const bool inb = x < p.Dx && y < p.Dy;
    const int z0 = blockIdx.z * p.zchunk, z1 = min(p.Dz, z0 + p.zchunk);
    const float delta = p.cull ? __ldg(p.ws) : __int_as_float(0x7f800000);
    const bool can_cull = delta < 3.0e38f;

    const NodeGridHeader h = *reinterpret_cast<const NodeGridHeader *>(p.grid);
    const bool has_bvh = h.pad[2] != 0;
    const float4 *bvh_box = reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(p.grid) + h.pad[2]);
    const float4 *bvh_leaf = reinterpret_cast<const float4 *>(reinterpret_cast<const char *>(p.grid) + h.pad[3]);

    // Candidate lists (round 2).  The exact 8-NN search per voxel was ~5 k instructions, most of the kernel.  The 256 voxels of a warp run
    // (8 x 4 x FUS_SUB) share almost all of their neighbours, and a superset of them is cheap to bound: with c the run's centre, h the
    // largest distance from c to a voxel centre of the run and R >= d8(c) (distance from c to its 8th nearest node), every voxel x of the run has
    // d8(x) <= d8(c) + h (the 8 nodes nearest to c are that close to x), so each of its eight nearest nodes n has |n - c| <= |n - x| + h <= R + 2h.
    // The warp scans the node table twice (32 nodes per step, coalesced 16-byte records): pass 1 forms R as the 8th smallest of the 32 lane
    // minima (distances of 32 distinct nodes, so >= d8(c)), pass 2 compacts the nodes within (R + 2h)(1 + 2e-4) of c into shared memory.
    // Each voxel then ranks the list (a broadcast read per candidate) with the same float distance and the same (distance, index)
    // order as every other search path, seeded with its z-predecessor's result: identical neighbours, ~10 instructions per candidate
    // instead of a branch-and-bound.  The list also bounds the run's displacement by ITS nodes' translations (8 max |t|), which is what the
    // visibility test needs: the global bound is useless in the live loop (rim nodes drift by decimetres), the local one is tight
    // everywhere else.  A list that does not fit (first version: 256 float4 entries per run; far from the node cloud the shell holds more) falls
    // back to the tree, at ten times the cost per voxel: lists are therefore 16-bit positions in the block list and practically never overflow.
    // Two levels: the block first selects, once, the nodes its whole 32 x 8 x zchunk region can need (same argument with the region's
    // centre and half diagonal; 256 threads, 8 nodes each at M = 2 k), and the warp runs then select from those few hundred instead of from
    // the node table (the two passes over M nodes per run were a visible share of the kernel).  A block list that overflows is simply not used.
    __shared__ unsigned short s_list[8][FUS_LIST_CAP];
    __shared__ float4 s_block[FUS_BLOCK_CAP];
    __shared__ float s_wmin[8][8];
    __shared__ float s_rb2;
    __shared__ int s_block_n;
    unsigned short *list = s_list[warp];
    const bool use_list = p.use_list && has_bvh && p.M >= 8;
    const bool identity = __ldg(p.ws + 2) != 0.f;
    int n_src = 0;                                                 // entries of the block list the runs select from
    bool from_block = false;
    if (use_list) {
        const float3 cb = aff_mul(p.vol2world, make_float3(((float)(blockIdx.x * 32) + 15.5f) * p.vsx, ((float)(blockIdx.y * 8) + 3.5f) * p.vsy,
                                                           ((float)z0 + 0.5f * (float)(p.zchunk - 1)) * p.vsz));
        float mn = 3.402823466e+38f;
        for (int i = threadIdx.x; i < p.M; i += 256) {
            const float4 v = __ldg(p.node_rec + 2 * p.M + i);
            const float d0 = cb.x - v.x, d1 = cb.y - v.y, d2 = cb.z - v.z;
            mn = fminf(mn, d0 * d0 + d1 * d1 + d2 * d2);
        }
        if (threadIdx.x == 0) s_block_n = 0;
#pragma unroll 1
        for (int r = 0; r < 8; ++r) {                              // the warp's 8 smallest thread minima, ascending
            const unsigned b = __reduce_min_sync(0xffffffffu, __float_as_uint(mn));
            const unsigned who = __ballot_sync(0xffffffffu, __float_as_uint(mn) == b);
            if (lane == __ffs(who) - 1) { mn = __int_as_float(0x7f800000); s_wmin[warp][r] = __uint_as_float(b); }
        }
        __syncthreads();
        if (warp == 0) {                                           // 8th smallest of the 64: distances of distinct nodes, so >= d8(cb)
            float a = (&s_wmin[0][0])[lane], b2 = (&s_wmin[0][0])[lane + 32];
            unsigned r2 = 0u;
#pragma unroll 1
            for (int r = 0; r < 8; ++r) {
                const float m = fminf(a, b2);
                r2 = __reduce_min_sync(0xffffffffu, __float_as_uint(m));
                const unsigned who = __ballot_sync(0xffffffffu, __float_as_uint(m) == r2);
                if (lane == __ffs(who) - 1) { if (__float_as_uint(a) == r2) a = __int_as_float(0x7f800000); else b2 = __int_as_float(0x7f800000); }
            }
            if (lane == 0) s_rb2 = __uint_as_float(r2);
        }
        __syncthreads();
        const float rb2 = s_rb2;
        if (rb2 < 1e30f) {
            const float thr = (sqrtf(rb2) + 2.f * p.half_diag_block) * 1.0002f + 1e-6f, thr2 = thr * thr;
            for (int i0 = 0; i0 < p.M; i0 += 256) {
                const int i = i0 + threadIdx.x;
                bool in = false;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (i < p.M) {
                    v = __ldg(p.node_rec + 2 * p.M + i);
                    const float d0 = cb.x - v.x, d1 = cb.y - v.y, d2 = cb.z - v.z;
                    in = d0 * d0 + d1 * d1 + d2 * d2 <= thr2;
                }
                const unsigned m = __ballot_sync(0xffffffffu, in);
                int base = 0;
                if (lane == 0 && m) base = atomicAdd(&s_block_n, __popc(m));
                base = __shfl_sync(0xffffffffu, base, 0);
                if (in) {
                    const int pos = base + __popc(m & ((1u << lane) - 1u));
                    if (pos < FUS_BLOCK_CAP) s_block[pos] = make_float4(v.x, v.y, v.z, __int_as_float(i));
                }
            }
            __syncthreads();
            if (s_block_n >= 8 && s_block_n <= FUS_BLOCK_CAP) { from_block = true; n_src = s_block_n; }
        }
    }

    int prev[8];
    bool have_prev = false;
    unsigned int n_upd = 0, n_warp = 0, n_col = 0;
    const size_t slice = (size_t)p.Dx * p.Dy;
    for (int za = z0; za < z1; za += FUS_SUB) {
        const int zb = min(z1, za + FUS_SUB);
        int L = -1;                                                // candidates in the list; -1: no list for this run
        bool culled = false;
        // pass 0 tests the run against the field's global displacement bound before any work is spent on it; pass 1 builds the candidate
        // list and tests again with the list's own bound.  (A loop so that the visibility test exists once in the kernel's code.)
#pragma unroll 1
        for (int pass = 0; pass < 2 && !culled; ++pass) {
            float run_delta = delta;
            if (pass == 1) {
                if (!from_block) break;
                run_delta = 3.402823466e+38f;
                __syncwarp();                                      // the previous run's readers are done with the list
                const float3 c = aff_mul(p.vol2world, make_float3(((float)xw + 3.5f) * p.vsx, ((float)yw + 1.5f) * p.vsy, ((float)za + 0.5f * (float)(FUS_SUB - 1)) * p.vsz));
                float mn = 3.402823466e+38f;
                for (int i = lane; i < n_src; i += 32) {
                    const float4 v = s_block[i];
                    const float d0 = c.x - v.x, d1 = c.y - v.y, d2 = c.z - v.z;
                    mn = fminf(mn, d0 * d0 + d1 * d1 + d2 * d2);   // a NaN node never lowers the minimum, like it never enters a neighbour set
                }
                unsigned r2bits = 0u;
#pragma unroll 1
                for (int r = 0; r < 8; ++r) {                      // 8th smallest lane minimum (non-negative floats order like their bit patterns)
                    r2bits = __reduce_min_sync(0xffffffffu, __float_as_uint(mn));
                    const unsigned who = __ballot_sync(0xffffffffu, __float_as_uint(mn) == r2bits);
                    if (lane == __ffs(who) - 1) mn = __int_as_float(0x7f800000);
                }
                const float R2 = __uint_as_float(r2bits);
                if (R2 < 1e30f) {
                    const float thr = (sqrtf(R2) + 2.f * p.half_diag) * 1.0002f + 1e-6f, thr2 = thr * thr;
                    int base = 0;
                    float tmax = 0.f;
                    for (int i0 = 0; i0 < n_src; i0 += 32) {
                        const int i = i0 + lane;
                        bool in = false;
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (i < n_src) {
                            v = s_block[i];
                            const float d0 = c.x - v.x, d1 = c.y - v.y, d2 = c.z - v.z;
                            in = d0 * d0 + d1 * d1 + d2 * d2 <= thr2;
                        }
                        const unsigned m = __ballot_sync(0xffffffffu, in);
                        if (in) {
                            const int pos = base + __popc(m & ((1u << lane) - 1u));
                            if (pos < FUS_LIST_CAP) list[pos] = (unsigned short)i;
                            const float4 t = __ldg(p.node_rec + p.M + __float_as_int(v.w));
                            tmax = fmaxf(tmax, sqrtf(t.y * t.y + t.z * t.z + t.w * t.w));
                        }
                        base += __popc(m);
                    }
                    if (base <= FUS_LIST_CAP) {
                        L = base;
                        if (identity) {                            // this run moves by at most 8 max |t| over ITS candidate nodes
                            for (int o = 16; o > 0; o >>= 1) tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, o));
                            const float local = 8.f * tmax * 1.0001f + 1e-6f;
                            if (local < delta) run_delta = local;
                        }
                    }
                    __syncwarp();
                }
            }
            if (can_cull && run_delta < 3.0e38f)
                culled = fusion_run_invisible(p, lane, run_delta, xw, min(xw + 7, p.Dx - 1), yw, min(yw + 3, p.Dy - 1), za, zb - 1);
        }
        if (culled || !inb) continue;
        uint32_t *vptr = p.data + x + (size_t)p.Dx * y + slice * za;
        for (int z = za; z < zb; ++z, vptr += slice) {
            const float3 xc = aff_mul(p.vol2world, make_float3((float)x * p.vsx, (float)y * p.vsy, (float)z * p.vsz));
            int bi[8]; float bd[8];
            if (L >= 0) {
                bool seeded = have_prev;
                if (have_prev) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        const float4 v = __ldg(p.node_rec + 2 * p.M + prev[k]);
                        const float d0 = xc.x - v.x, d1 = xc.y - v.y, d2 = xc.z - v.z;
                        bi[k] = prev[k];
                        bd[k] = d0 * d0 + d1 * d1 + d2 * d2;
                        seeded = seeded && bd[k] == bd[k];
                    }
                }
                if (seeded) {
#define DF_CS(a, b) knn8_cswap_lex(bd[a], bi[a], bd[b], bi[b])
                    DF_CS(0, 1); DF_CS(2, 3); DF_CS(4, 5); DF_CS(6, 7);
                    DF_CS(0, 2); DF_CS(1, 3); DF_CS(4, 6); DF_CS(5, 7);
                    DF_CS(1, 2); DF_CS(5, 6);
                    DF_CS(0, 4); DF_CS(1, 5); DF_CS(2, 6); DF_CS(3, 7);
                    DF_CS(2, 4); DF_CS(3, 5);
                    DF_CS(1, 2); DF_CS(3, 4); DF_CS(5, 6);
#undef DF_CS
                } else {
#pragma unroll
                    for (int k = 0; k < 8; ++k) { bi[k] = 0x7fffffff; bd[k] = 3.402823466e+38f; }
                }
#pragma unroll 1
                for (int j = 0; j < L; ++j) {
                    const float4 nd = s_block[list[j]];
                    const float d0 = xc.x - nd.x, d1 = xc.y - nd.y, d2 = xc.z - nd.z;
                    const float dist = d0 * d0 + d1 * d1 + d2 * d2;
                    if (dist <= bd[7]) {                           // one compare on the common (reject) path; ties and seeds sorted out inside
                        const int idx = __float_as_int(nd.w);
                        if (dist < bd[7] || idx < bi[7]) {
                            const bool held = idx == bi[0] || idx == bi[1] || idx == bi[2] || idx == bi[3] || idx == bi[4] || idx == bi[5] || idx == bi[6];
                            if (!held) knn8_insert_lex(bi, bd, dist, idx);
                        }
                    }
                }
#pragma unroll
                for (int k = 0; k < 8; ++k) if (bi[k] == 0x7fffffff) bi[k] = -1;
            } else {                                               // cold path: copies keep bi / bd / prev themselves in registers
                int tp[8], tb[8]; float td[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) tp[k] = prev[k];
                fusion_tree_search(p.grid, p.node_rec + 2 * p.M, xc, have_prev, tp, tb, td);
#pragma unroll
                for (int k = 0; k < 8; ++k) { bi[k] = tb[k]; bd[k] = td[k]; }
            }
            have_prev = bi[7] >= 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) prev[k] = bi[k];
            ++n_warp;

            const float3 xwp = fusion_warp_point<kIdentity>(p, bi, bd, xc);
            const float tx = p.world2cam.r0.x * xwp.x + p.world2cam.r0.y * xwp.y + p.world2cam.r0.z * xwp.z + p.world2cam.t.x;
            const float ty = p.world2cam.r1.x * xwp.x + p.world2cam.r1.y * xwp.y + p.world2cam.r1.z * xwp.z + p.world2cam.t.y;
            const float tz = p.world2cam.r2.x * xwp.x + p.world2cam.r2.y * xwp.y + p.world2cam.r2.z * xwp.z + p.world2cam.t.z;
            if (!(tz > 0)) continue;
            const float u = __fmaf_rn(p.fx, tx / tz, p.cx), v = __fmaf_rn(p.fy, ty / tz, p.cy);
            if (!(u >= 0 && v >= 0 && u < p.fcols && v < p.frows)) continue;
            const unsigned short mm = __ldg(row_ptr(p.depth, p.pitch, (int)v) + (int)u);
            if (mm == 0) continue;
            const float rho = (float)mm * 0.001f - tz;
            if (!(rho > -p.trunc)) continue;
            const float tsdf = fminf(1.f, rho * p.trunc_inv);
            const int wq = fusion_sample_weight(p, bi, bd);
            const uint32_t packed = *vptr;
            const int weight_prev = (int)(packed >> 16);
            const float tsdf_prev = half_bits_to_float((unsigned short)(packed & 0xffffu));
            const float tsdf_new = __fmaf_rn(tsdf_prev, (float)weight_prev, tsdf * (float)wq) / (float)(weight_prev + wq);
            const int weight_new = min(weight_prev + wq, p.max_weight);
            const uint32_t val = (uint32_t)float_to_half_bits(tsdf_new) | ((uint32_t)weight_new << 16);
            *vptr = val;
            if (p.activity && vox_active(val)) {
                p.activity[(size_t)(vptr - p.data) / DF_ACTIVITY_VOXELS] = 1;
                if (vox_negative(val)) brick_mark(p.bricks, x, y, z);
            }
            ++n_upd;
            if constexpr (kColor != WC_NONE) {
                // df_integrate_warped_color's rule, on the values the TSDF side just formed: the warped point (tx, ty, tz), its depth pixel
                // ((int)u, (int)v) and rho.  The band |rho| <= DF_COLOR_BAND * trunc lies inside the TSDF gate rho > -trunc, so every voxel
                // that can take a colour sample has been written above; the culling (runs skipped when rho < -trunc for all of their voxels
                // whatever the field does) is conservative for the TSDF and therefore for the colour too.
                if (fabsf(rho) <= wc->band) {
                    uchar4 smp;
                    bool ok = true;
                    if constexpr (kColor == WC_REGISTERED) smp = __ldg(row_ptr(wc->bgra, wc->cpitch, (int)v) + (int)u);
                    else ok = camera_sample<kLens>(wc->o, *lens, wc->bgra, wc->cpitch, make_float3(tx, ty, tz), smp);
                    if (ok) {
                        uint32_t *cptr = wc->colors + (vptr - p.data);
                        *cptr = color_update(*cptr, smp, wc->wcap);
                        ++n_col;
                    }
                }
            }
        }
    }
    if (p.counters) {
        __syncwarp();
        for (int o = 16; o > 0; o >>= 1) { n_upd += __shfl_xor_sync(0xffffffffu, n_upd, o); n_warp += __shfl_xor_sync(0xffffffffu, n_warp, o); }
        if (lane == 0) {
            if (n_upd) atomicAdd(p.counters, (unsigned long long)n_upd);
            if (n_warp) atomicAdd(p.counters + 1, (unsigned long long)n_warp);
        }
    }
    if constexpr (kColor != WC_NONE) {
        if (wc->counter) {
            __syncwarp();
            for (int o = 16; o > 0; o >>= 1) n_col += __shfl_xor_sync(0xffffffffu, n_col, o);
            if (lane == 0 && n_col) atomicAdd(wc->counter, (unsigned long long)n_col);
        }
    }
}

// Two instantiations are launched back to back and the one whose kIdentity does not match the node table returns at once (the flag is a
// device-side result of fusion_prepare_kernel; reading it on the host would stall the frame loop): each path keeps its own register
// allocation.  4 blocks per SM: 64 registers, a few dozen bytes of spills; 3 blocks (80 registers) was slower at 512^3
// (integrate stage 12.55 vs 12.48 ms per frame, H100 80GB HBM3 at 700 W), 5 blocks (48 registers, 600 bytes of spills) much slower.
template <bool kIdentity>
__global__ void __launch_bounds__(256, 4) integrate_warped_kernel(const FusionParams p)
{
    DF_PDL_ENTRY();
    if ((__ldg(p.ws + 2) != 0.f) != kIdentity) return;
    integrate_warped_body<kIdentity>(p);
}

// df_integrate_warped_color: the same voxel walk with the colour side compiled in (kColor, kLens), one kernel per mode so that the
// colourless instances above keep their code.
template <bool kIdentity, int kColor, bool kLens>
__global__ void __launch_bounds__(256, 4) integrate_warped_color_kernel(const FusionParams p, const WarpedColorParams wc, const df_lens lens)
{
    DF_PDL_ENTRY();
    if ((__ldg(p.ws + 2) != 0.f) != kIdentity) return;
    integrate_warped_body<kIdentity, kColor, kLens>(p, &wc, &lens);
}

// |R^T R - I|_max: how far a pose's linear part is from a rotation
double orthonormal_defect(const df_aff3f &a)
{
    double worst = 0.0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += (double)a.R[3 * k + i] * (double)a.R[3 * k + j];
            worst = fmax(worst, fabs(s - (i == j ? 1.0 : 0.0)));
        }
    return worst;
}

}  // namespace

static size_t fusion_rec_offset_floats(int cols, int rows)
{
    const int tx = div_up(cols, FUS_TILE), ty = div_up(rows, FUS_TILE);
    return ((size_t)(16 + tx * ty + div_up(tx, FUS_COARSE) * div_up(ty, FUS_COARSE)) + 3) & ~(size_t)3;      // 16-byte aligned
}

extern "C" size_t df_integrate_warped_workspace_bytes(int cols, int rows, int M)
{
    return (fusion_rec_offset_floats(cols, rows) + (size_t)12 * (M > 0 ? M : 0)) * sizeof(float) + 64;
}

extern "C" int df_integrate_warped_launch_count(void) { return 4; }

// both entries: wc == NULL launches df_integrate_warped's kernels, else the colour instances of kColor (lens: WC_CAMERA only, NULL = pinhole)
static int integrate_warped(df_volume vol, const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_aff3f vol2world, df_aff3f world2cam,
                            df_intr intr, const float *nodes, int M, const void *node_grid, float weight_scale, unsigned long long *counters,
                            unsigned char *activity, void *workspace, const WarpedColorParams *wc, int kColor, const df_lens *lens, void *stream)
{
    if (!node_grid || !nodes || M <= 0 || !vol.data || !depth) return (int)cudaErrorInvalidValue;
    cudaStream_t s = (cudaStream_t)stream;
    FusionParams p;
    p.data = vol.data;
    p.Dx = vol.dims[0]; p.Dy = vol.dims[1]; p.Dz = vol.dims[2];
    p.vsx = vol.voxel_size[0]; p.vsy = vol.voxel_size[1]; p.vsz = vol.voxel_size[2];
    p.trunc = vol.trunc_dist; p.trunc_inv = 1.f / vol.trunc_dist;
    p.max_weight = vol.max_weight;
    p.depth = depth; p.pitch = depth_pitch; p.cols = cols; p.rows = rows; p.fcols = (float)cols; p.frows = (float)rows;
    p.vol2world = make_aff(vol2world); p.world2cam = make_aff(world2cam);
    df_aff3f v2c;                                   // composed in double: only the (conservative) visibility test uses it
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            double a = 0.0;
            for (int k = 0; k < 3; ++k) a += (double)world2cam.R[3 * i + k] * (double)vol2world.R[3 * k + j];
            v2c.R[3 * i + j] = (float)a;
        }
        double t = world2cam.t[i];
        for (int k = 0; k < 3; ++k) t += (double)world2cam.R[3 * i + k] * (double)vol2world.t[k];
        v2c.t[i] = (float)t;
    }
    p.vol2cam = make_aff(v2c);
    p.cull = orthonormal_defect(vol2world) < 1e-3 && orthonormal_defect(world2cam) < 1e-3;
    {
        const char *e = getenv("DF_FUSION_CULL");      // test knob, looked up per call (tests toggle it in-process; the kernel runs for milliseconds)
        if (e && atoi(e) == 0) p.cull = 0;
    }
    p.fx = intr.fx; p.fy = intr.fy; p.cx = intr.cx; p.cy = intr.cy;
    p.nodes = nodes; p.M = M; p.grid = node_grid;
    p.weight_scale = weight_scale;
    p.counters = counters; p.activity = activity;
    p.bricks = brick_table(activity, vol.dims[0], vol.dims[1], vol.dims[2]);
    p.tiles_x = div_up(cols, FUS_TILE); p.tiles_y = div_up(rows, FUS_TILE);
    p.ctiles_x = div_up(p.tiles_x, FUS_COARSE); p.ctiles_y = div_up(p.tiles_y, FUS_COARSE);
    {
        const char *e = getenv("DF_FUSION_LIST");      // test knob, per call: 0 = branch-and-bound per voxel only (round 1)
        p.use_list = !(e && atoi(e) == 0);
        double worst = 0.0;                             // half the longest diagonal of the box of voxel centres of a warp run, in world space
        for (int sgn = 0; sgn < 4; ++sgn) {
            const double ex = 7.0 * p.vsx, ey = ((sgn & 1) ? -3.0 : 3.0) * p.vsy, ez = ((sgn & 2) ? -(double)(FUS_SUB - 1) : (double)(FUS_SUB - 1)) * p.vsz;
            double d2 = 0.0;
            for (int i = 0; i < 3; ++i) { const double v = vol2world.R[3 * i] * ex + vol2world.R[3 * i + 1] * ey + vol2world.R[3 * i + 2] * ez; d2 += v * v; }
            worst = fmax(worst, sqrt(d2));
        }
        p.half_diag = (float)(0.5 * worst * 1.001 + 1e-7);
    }
    p.zchunk = vol.dims[2] >= 64 ? 32 : vol.dims[2];
    {
        const char *e = getenv("DF_FUSION_ZCHUNK");    // test knob, per call
        if (e && atoi(e) > 0) p.zchunk = atoi(e);
    }
    {
        double worst = 0.0;
        for (int sgn = 0; sgn < 4; ++sgn) {
            const double ex = 31.0 * p.vsx, ey = ((sgn & 1) ? -7.0 : 7.0) * p.vsy, ez = ((sgn & 2) ? -1.0 : 1.0) * (double)(p.zchunk - 1) * p.vsz;
            double d2 = 0.0;
            for (int i = 0; i < 3; ++i) { const double v = vol2world.R[3 * i] * ex + vol2world.R[3 * i + 1] * ey + vol2world.R[3 * i + 2] * ez; d2 += v * v; }
            worst = fmax(worst, sqrt(d2));
        }
        p.half_diag_block = (float)(0.5 * worst * 1.001 + 1e-7);
    }
    float *ws = (float *)workspace;
    const bool own = ws == nullptr;
    if (own) {
        const cudaError_t e = cudaMallocAsync((void **)&ws, df_integrate_warped_workspace_bytes(cols, rows, M), s);
        if (e != cudaSuccess) return (int)e;
    }
    p.ws = ws;
    float4 *rec = reinterpret_cast<float4 *>(ws + fusion_rec_offset_floats(cols, rows));
    p.node_rec = rec;
    launch_pdl(depth_tile_max_kernel, dim3(p.tiles_x, p.tiles_y), dim3(256), 0, s, depth, depth_pitch, cols, rows, ws + 16, p.tiles_x);
    launch_pdl(fusion_prepare_kernel, dim3(2), dim3(256), 0, s, ws, p.tiles_x, p.tiles_y, p.ctiles_x, p.ctiles_y, nodes, M, rec);
    dim3 grid(div_up(vol.dims[0], 32), div_up(vol.dims[1], 8), div_up(vol.dims[2], p.zchunk));
    if (wc) {
        const df_lens L = lens ? *lens : df_lens{};
        if (kColor == WC_REGISTERED) {
            launch_pdl(integrate_warped_color_kernel<true, WC_REGISTERED, false>, grid, dim3(256), 0, s, p, *wc, L);
            launch_pdl(integrate_warped_color_kernel<false, WC_REGISTERED, false>, grid, dim3(256), 0, s, p, *wc, L);
        } else if (!lens) {
            launch_pdl(integrate_warped_color_kernel<true, WC_CAMERA, false>, grid, dim3(256), 0, s, p, *wc, L);
            launch_pdl(integrate_warped_color_kernel<false, WC_CAMERA, false>, grid, dim3(256), 0, s, p, *wc, L);
        } else {
            launch_pdl(integrate_warped_color_kernel<true, WC_CAMERA, true>, grid, dim3(256), 0, s, p, *wc, L);
            launch_pdl(integrate_warped_color_kernel<false, WC_CAMERA, true>, grid, dim3(256), 0, s, p, *wc, L);
        }
    } else {
        launch_pdl(integrate_warped_kernel<true>, grid, dim3(256), 0, s, p);
        launch_pdl(integrate_warped_kernel<false>, grid, dim3(256), 0, s, p);
    }
    if (own) cudaFreeAsync(ws, s);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_integrate_warped(df_volume vol, const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_aff3f vol2world,
                                   df_aff3f world2cam, df_intr intr, const float *nodes, int M, const void *node_grid, float weight_scale,
                                   unsigned long long *counters, unsigned char *activity, void *workspace, void *stream)
{
    return integrate_warped(vol, depth, depth_pitch, cols, rows, vol2world, world2cam, intr, nodes, M, node_grid, weight_scale, counters, activity,
                            workspace, nullptr, WC_NONE, nullptr, stream);
}

extern "C" int df_integrate_warped_color(df_volume vol, const uint16_t *depth, size_t depth_pitch, int cols, int rows, df_aff3f vol2world,
                                         df_aff3f world2cam, df_intr intr, const float *nodes, int M, const void *node_grid, float weight_scale,
                                         unsigned long long *counters, unsigned char *activity, void *workspace, uint32_t *colors, const void *bgra,
                                         size_t bgra_pitch, const df_color_camera *cam, const df_lens *lens, const uint32_t *map, size_t map_pitch,
                                         void *stream)
{
    if (!node_grid || !nodes || M <= 0 || !vol.data || !depth || !colors || !bgra || cols <= 0 || rows <= 0 || vol.dims[0] <= 0 || vol.dims[1] <= 0 ||
        vol.dims[2] <= 0 || depth_pitch < (size_t)cols * 2 || depth_pitch % 2 || bgra_pitch % 4)
        return (int)cudaErrorInvalidValue;
    WarpedColorParams wc = {};
    wc.colors = colors;
    wc.bgra = (const uchar4 *)bgra; wc.cpitch = bgra_pitch;
    wc.band = DF_COLOR_BAND * vol.trunc_dist;
    wc.wcap = vol.max_weight < 255 ? vol.max_weight : 255;
    wc.counter = counters ? counters + 2 : nullptr;
    bool use_lens = false;
    if (cam) {
        int mcols = 0, mrows = 0, cell = 0;
        if (df_color_map_dims(intr, *cam, &mcols, &mrows, &cell) || !map || map_pitch < (size_t)mcols * 4 || map_pitch % 4 ||
            bgra_pitch < (size_t)cam->cols * 4 || (lens && df_lens_check(*lens)))
            return (int)cudaErrorInvalidValue;
        use_lens = lens && !lens_is_zero(*lens);
        wc.o.cam = camera_params(*cam, cell);
        wc.o.map = map; wc.o.mpitch = map_pitch;
        wc.o.tol = DF_COLOR_OCCLUSION * vol.trunc_dist;
    } else if (bgra_pitch < (size_t)cols * 4)
        return (int)cudaErrorInvalidValue;
    return integrate_warped(vol, depth, depth_pitch, cols, rows, vol2world, world2cam, intr, nodes, M, node_grid, weight_scale, counters, activity,
                            workspace, &wc, cam ? WC_CAMERA : WC_REGISTERED, use_lens ? lens : nullptr, stream);
}
