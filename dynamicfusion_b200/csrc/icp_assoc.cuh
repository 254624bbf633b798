// icp_assoc.cuh -- the projective ICP's data association (find_coresp + row build), shared by the ICP's accumulate kernels (icp.cu) and the
// relocaliser's gate (reloc.cu, df_icp_inliers), so that the gate counts exactly the pixels the ICP uses.  Internal.
#pragma once
#include "df_common.cuh"

namespace {

using namespace dfb;

struct IcpParams {
    const float4 *vcurr; size_t vcpitch;
    const float4 *ncurr; size_t ncpitch;
    const float4 *vprev; size_t vppitch;
    const float4 *nprev; size_t nppitch;
    const unsigned short *dcurr; size_t dcpitch;     // depth variant (USE_DEPTH, proj_icp.cu:47-78): u16 millimetres
    const unsigned short *dprev; size_t dppitch;
    float finvx, finvy;                              // 1/f of the level (setLevelIntr, projective_icp.cpp:22)
    int cols, rows;
    float fcols, frows;
    float fx, fy, cx, cy;
    float dist2_thres, min_cosine;
    Aff T_val;
    const float *T_ptr;       // when non-null: 12 floats (R row-major, t) in device memory
    const int *ok_ptr;        // when non-null and *ok_ptr == 0 the iteration is skipped
    double *partials;         // [gridDim.x][27]
};

// find_coresp proj_icp.cu:47-78 (DEPTH: the reference's compile-time USE_DEPTH alternative) / :80-108 (points) + row build :359-368
// an accepted pixel also hands back s = T * v_curr and its projection (u, v), for the photometric row of the colour variant
template <bool DEPTH>
__device__ __forceinline__ bool icp_row(const IcpParams &p, const Aff &T, int x, int y, float row[7], float3 &s_out, float &u_out, float &v_out)
{
    // the loads of one pixel go out in two batches (current maps at (x, y), previous maps at the projection) instead of one
    // dependent round trip per test: the order of the reference's tests is kept, only the fetches are hoisted
    const float4 nc = __ldg(row_ptr(p.ncurr, p.ncpitch, y) + x);
    float3 s;
    if (DEPTH) {
        const int src_z = __ldg(row_ptr(p.dcurr, p.dcpitch, y) + x);
        if (src_z == 0) return false;
        const float z = src_z * 0.001f;
        s = make_float3(z * ((float)x - p.cx) * p.finvx, z * ((float)y - p.cy) * p.finvy, z);    // reproj, proj_icp.cu:39-45
    } else {
        const float4 vc = __ldg(row_ptr(p.vcurr, p.vcpitch, y) + x);
        s = make_float3(vc.x, vc.y, vc.z);
        if (isnan(s.x)) return false;
    }
    s = aff_mul(T, s);
    const float u = __fmaf_rn(p.fx, s.x / s.z, p.cx);
    const float v = __fmaf_rn(p.fy, s.y / s.z, p.cy);
    if (s.z <= 0 || u < 0 || v < 0 || u >= p.fcols || v >= p.frows) return false;
    if (!(u == u) || !(v == v)) return false;
    const float4 np = __ldg(row_ptr(p.nprev, p.nppitch, (int)v) + (int)u);     // point sampling of the previous maps
    float3 d;
    if (DEPTH) {
        const int dst_z = __ldg(row_ptr(p.dprev, p.dppitch, (int)v) + (int)u);
        if (dst_z == 0) return false;
        const float z = dst_z * 0.001f;
        d = make_float3(z * (u - p.cx) * p.finvx, z * (v - p.cy) * p.finvy, z);  // re-projected at the fractional coordinates
    } else {
        const float4 dp = __ldg(row_ptr(p.vprev, p.vppitch, (int)v) + (int)u);
        d = make_float3(dp.x, dp.y, dp.z);
        if (isnan(d.x)) return false;
    }
    const float3 df = sub3(s, d);
    if (dot3(df, df) > p.dist2_thres) return false;
    const float3 ns = mat_mul(T.r0, T.r1, T.r2, make_float3(nc.x, nc.y, nc.z));
    const float3 nd = make_float3(np.x, np.y, np.z);
    if (fabsf(dot3(ns, nd)) < p.min_cosine) return false;
    const float3 c = cross3(s, nd);
    row[0] = c.x; row[1] = c.y; row[2] = c.z; row[3] = nd.x; row[4] = nd.y; row[5] = nd.z;
    row[6] = dot3(nd, sub3(d, s));
    s_out = s; u_out = u; v_out = v;
    return true;
}

}  // namespace
