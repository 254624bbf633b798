// icp.cu -- projective point-to-plane ICP on sm_90a, fully device-resident.
// Replaces kfusion/src/cuda/proj_icp.cu (icp_helper_kernel + 27 sequential 256-thread smem tree reductions +
// icp_final_reduce_kernel) and the host loop of kfusion/src/projective_icp.cpp:169-213 (per iteration: D2H of 27
// floats, stream sync, cv::determinant, cv::solve(DECOMP_SVD), Rodrigues, H2D of the pose = 19 round trips a frame).
//
// Per iteration two launches, no host involvement:
//   icp_accumulate_kernel  at most one block per SM; each thread forms its 7-vector rows and keeps the 27 products in registers
//                          across its pixels (float products as the reference, proj_icp.cu:137-345), then one
//                          double-precision warp-shuffle reduction and one partial row per block (deterministic order);
//   icp_solve_kernel       one block: fixed-order sum of the partials, 6x6 solve, Rodrigues, T <- Tinc * T in place.
#include "df_common.cuh"
#include <float.h>
#include <stdlib.h>

using namespace dfb;

int dfb::pdl_enabled()
{
    static const int v = [] { const char *e = getenv("DF_PDL"); return e ? (int)(atoi(e) != 0) : 1; }();   // thread-safe one-time read
    return v;
}

namespace {


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
template <bool DEPTH>
__device__ __forceinline__ bool icp_row(const IcpParams &p, const Aff &T, int x, int y, float row[7])
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
    return true;
}

// One row of partials per block and at most ICP_MAX_PARTIAL_BLOCKS (= one per SM) blocks: the solve tail's fixed-order sum over the
// rows is a chain of L2 round trips, so the row count is what its latency scales with (hence one row per SM of 768-thread blocks
// rather than four rows per SM of 256-thread blocks).  Pixels are dealt to threads linearly (coalesced
// along x, balanced to one pixel per warp whatever the image size).
template <bool DEPTH, int NT>
__global__ void __launch_bounds__(NT) icp_accumulate_kernel(const IcpParams p)
{
    constexpr int NW = NT / 32;
    __shared__ double smem[NW][27];
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    float acc[27];
#pragma unroll
    for (int i = 0; i < 27; ++i) acc[i] = 0.f;
    pdl_wait();
    pdl_trigger();

    // pose and gate written by the previous solve: both loads are issued before either is consumed
    Aff T = p.T_val;
    int active = 1;
    if (p.T_ptr) {
        float t[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) t[i] = p.T_ptr[i];
        active = *p.ok_ptr;
        T.r0 = make_float3(t[0], t[1], t[2]);
        T.r1 = make_float3(t[3], t[4], t[5]);
        T.r2 = make_float3(t[6], t[7], t[8]);
        T.t = make_float3(t[9], t[10], t[11]);
    }
    if (active) {
        const int npix = p.cols * p.rows;
        for (int i = blockIdx.x * NT + tid; i < npix; i += gridDim.x * NT) {
            const int y = i / p.cols, x = i - y * p.cols;
            float row[7];
            if (icp_row<DEPTH>(p, T, x, y, row)) {
                int k = 0;
#pragma unroll
                for (int a = 0; a < 6; ++a)
#pragma unroll
                    for (int j = a; j < 7; ++j) acc[k++] += row[a] * row[j];
            }
        }
    }
    // the warp stage stays in float (the reference's whole reduction is a float tree, proj_icp.cu:111-348): 135 shuffles per warp instead
    // of the 270 a double butterfly needs (they were a large share of the ICP kernels' instructions); warps are then summed in double
#pragma unroll
    for (int i = 0; i < 27; ++i) {
        float v = acc[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) smem[warp][i] = (double)v;
    }
    __syncthreads();
    if (tid < 27) {
        double v = 0.0;
#pragma unroll
        for (int w = 0; w < NW; ++w) v += smem[w][tid];
        p.partials[(size_t)blockIdx.x * 27 + tid] = v;
    }
}

// fixed-order reduction of the block partials into sums[27].  The rows are first staged in shared memory with cp.async (every
// thread's copies are in flight together: ONE L2 round trip for the whole table; a register-accumulating loop was serialised by
// the compiler into one round trip per load), then each warp sums its columns s = warp, warp + nwarps, ... lane-strided.
constexpr int RED_ROWS = 160;                               // rows staged per pass (>= ICP_MAX_PARTIAL_BLOCKS)
__device__ void reduce_partials(const double *partials, int nblocks, double *sums_smem, double *stage)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    for (int base = 0; base < nblocks; base += RED_ROWS) {
        const int rows = nblocks - base < RED_ROWS ? nblocks - base : RED_ROWS;
        const int chunks = (rows * 27 + 1) >> 1;            // 16-byte chunks (an odd tail reads one double of slack)
        const double *src = partials + (size_t)base * 27;
        for (int c = threadIdx.x; c < chunks; c += blockDim.x) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(stage + 2 * c);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src + 2 * c) : "memory");
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int s = warp + q * nwarps;
            if (s < 27)
                for (int b = lane; b < rows; b += 32) v[q] += stage[b * 27 + s];
        }
        __syncthreads();
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        double t = v[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        const int s = warp + q * nwarps;
        if (lane == 0 && s < 27) sums_smem[s] = t;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(256) icp_reduce_kernel(const double *partials, int nblocks, double *out27)
{
    __shared__ double sums[27];
    __shared__ __align__(16) double stage[RED_ROWS * 27];
    reduce_partials(partials, nblocks, sums, stage);
    if (threadIdx.x < 27) out27[threadIdx.x] = sums[threadIdx.x];
}

__device__ double det6_dev(const double *Ain)
{
    double A[36];
    for (int i = 0; i < 36; ++i) A[i] = Ain[i];
    double det = 1.0;
    for (int c = 0; c < 6; ++c) {
        int pv = c;
        for (int r = c + 1; r < 6; ++r) if (fabs(A[r * 6 + c]) > fabs(A[pv * 6 + c])) pv = r;
        if (A[pv * 6 + c] == 0.0) return 0.0;
        if (pv != c) { for (int j = 0; j < 6; ++j) { const double t = A[c * 6 + j]; A[c * 6 + j] = A[pv * 6 + j]; A[pv * 6 + j] = t; } det = -det; }
        det *= A[c * 6 + c];
        for (int r = c + 1; r < 6; ++r) {
            const double f = A[r * 6 + c] / A[c * 6 + c];
            for (int j = c; j < 6; ++j) A[r * 6 + j] -= f * A[c * 6 + j];
        }
    }
    return det;
}

// Cholesky solve, fully unrolled so that L, y, x live in registers (the tail is one thread: local-memory round trips
// would sit on the serial path of every ICP iteration).  Returns false when a pivot is not safely positive (caller falls back to LU + the eigen
// solve).  *det receives det(A) = (prod L_jj)^2.
// The tail is the serial part of every one of a frame's 19 ICP iterations, so its LATENCY is what counts: a double sqrt or division is
// a ~250-cycle dependent chain, and the textbook form needs 6 + 18 of them.  Here each pivot costs one rsqrt (L_jj = d * rsqrt(d),
// 1 / L_jj = rsqrt(d)) and the substitutions multiply by the stored inverses: ~1.5 k cycles instead of ~6.5 k.  The solution moves by
// a few double ulps (the pose is cast to float right after).  tests/test_icp_reference_gpu.py holds every step, on this path and the
// fallback's, to the float64 eigen-decomposition step of tests/icp_reference.py: a few float ulps plus 8 kappa_eff eps64 |r| (1 + |t|).
__device__ __forceinline__ bool chol6_solve(const double (&A)[36], const double (&b)[6], double (&x)[6], double *det)
{
    double L[36], inv[6];
    double dmax = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) dmax = fmax(dmax, fabs(A[i * 6 + i]));
    bool ok = true;
    double dprod = 1.0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        double d = A[j * 6 + j];
#pragma unroll
        for (int k = 0; k < j; ++k) d -= L[j * 6 + k] * L[j * 6 + k];
        if (!(d > dmax * 1e-13)) { ok = false; d = 1.0; }
        const double dinv = rsqrt(d);
        d = d * dinv;
        dprod *= d;
        L[j * 6 + j] = d;
        inv[j] = dinv;
#pragma unroll
        for (int i = j + 1; i < 6; ++i) {
            double s = A[i * 6 + j];
#pragma unroll
            for (int k = 0; k < j; ++k) s -= L[i * 6 + k] * L[j * 6 + k];
            L[i * 6 + j] = s * dinv;
        }
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double s = b[i];
#pragma unroll
        for (int k = 0; k < i; ++k) s -= L[i * 6 + k] * y[k];
        y[i] = s * inv[i];
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double s = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; ++k) s -= L[k * 6 + i] * x[k];
        x[i] = s * inv[i];
    }
    *det = dprod * dprod;
    return ok;
}

// symmetric-eigen pseudo-inverse (what cv::solve(DECOMP_SVD) computes for a symmetric matrix); slow path
__device__ void sym6_solve_dev(const double *Ain, const double *b, double *x)
{
    double A[36], V[36];
    for (int i = 0; i < 36; ++i) { A[i] = Ain[i]; V[i] = 0.0; }
    for (int i = 0; i < 6; ++i) V[i * 6 + i] = 1.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 6; ++p) for (int q = p + 1; q < 6; ++q) off += A[p * 6 + q] * A[p * 6 + q];
        if (off < 1e-300) break;
        for (int p = 0; p < 6; ++p)
            for (int q = p + 1; q < 6; ++q) {
                const double apq = A[p * 6 + q];
                if (apq == 0.0) continue;
                const double theta = (A[q * 6 + q] - A[p * 6 + p]) / (2.0 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 6; ++k) { const double akp = A[k * 6 + p], akq = A[k * 6 + q]; A[k * 6 + p] = c * akp - s * akq; A[k * 6 + q] = s * akp + c * akq; }
                for (int k = 0; k < 6; ++k) { const double apk = A[p * 6 + k], aqk = A[q * 6 + k]; A[p * 6 + k] = c * apk - s * aqk; A[q * 6 + k] = s * apk + c * aqk; }
                for (int k = 0; k < 6; ++k) { const double vkp = V[k * 6 + p], vkq = V[k * 6 + q]; V[k * 6 + p] = c * vkp - s * vkq; V[k * 6 + q] = s * vkp + c * vkq; }
            }
    }
    double wmax = 0.0;
    for (int i = 0; i < 6; ++i) wmax = fmax(wmax, fabs(A[i * 6 + i]));
    const double thr = wmax * 6 * DBL_EPSILON;
    for (int i = 0; i < 6; ++i) x[i] = 0.0;
    for (int e = 0; e < 6; ++e) {
        const double w = A[e * 6 + e];
        if (fabs(w) <= thr) continue;
        double proj = 0.0;
        for (int i = 0; i < 6; ++i) proj += V[i * 6 + e] * b[i];
        proj /= w;
        for (int i = 0; i < 6; ++i) x[i] += V[i * 6 + e] * proj;
    }
}

// host step projective_icp.cpp:195-209 on the device: sums -> A, b -> r = solve(A, b) -> T <- Affine3f(r) * T.  Tin/Tout: 12 floats
// (R row-major, t).  Returns false where the reference returns false (|det| < 1e-15 or NaN).  `r` solved by the caller's
// Cholesky (chol6_solve, in registers); this part is the general fallback + the pose composition.
__device__ bool icp_fallback_solve(const double (&A)[36], const double (&b)[6], double (&r)[6])
{
    const double det = det6_dev(A);
    if (fabs(det) < 1e-15 || det != det) return false;
    sym6_solve_dev(A, b, r);
    return true;
}

__device__ void icp_compose_pose(const double (&r)[6], const float *Tin, float *Tout)
{
    float rf[6];
    for (int i = 0; i < 6; ++i) rf[i] = (float)r[i];
    // cv::Affine3f(rvec, t): Rodrigues evaluated in double on float inputs (opencv2/core/affine.hpp)
    float Rinc[9];
    const double theta2 = (double)rf[0] * rf[0] + (double)rf[1] * rf[1] + (double)rf[2] * rf[2];
    if (theta2 < DBL_EPSILON * DBL_EPSILON) {                      // theta < DBL_EPSILON
        for (int i = 0; i < 9; ++i) Rinc[i] = (i % 4 == 0) ? 1.f : 0.f;
    } else {
        const double itheta = rsqrt(theta2), theta = theta2 * itheta;   // one dependent chain instead of sqrt, then 1 / theta
        double s, c;
        sincos(theta, &s, &c);                                     // one argument reduction for both (this tail is latency-bound)
        const double c1 = 1. - c;
        const float rx = (float)(rf[0] * itheta), ry = (float)(rf[1] * itheta), rz = (float)(rf[2] * itheta);
        const float rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
        const float r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
        for (int i = 0; i < 9; ++i) Rinc[i] = (float)(c * ((i % 4 == 0) ? 1.0 : 0.0) + c1 * rrt[i] + s * r_x[i]);
    }
    float Rn[9], tn[3];
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j)
            Rn[i * 3 + j] = Rinc[i * 3 + 0] * Tin[0 * 3 + j] + Rinc[i * 3 + 1] * Tin[1 * 3 + j] + Rinc[i * 3 + 2] * Tin[2 * 3 + j];
        tn[i] = Rinc[i * 3 + 0] * Tin[9] + Rinc[i * 3 + 1] * Tin[10] + Rinc[i * 3 + 2] * Tin[11] + rf[3 + i];
    }
    for (int i = 0; i < 9; ++i) Tout[i] = Rn[i];
    for (int i = 0; i < 3; ++i) Tout[9 + i] = tn[i];
}

// A (symmetric) and b from the 27 sums; the reference's buffer is float (projective_icp.cpp:51-60)
__device__ __forceinline__ void icp_unpack_sums(const double *sums, double (&A)[36], double (&b)[6])
{
    int shift = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 7; ++j) {
            const double value = (double)(float)sums[shift++];
            if (j == 6) b[i] = value; else A[j * 6 + i] = A[i * 6 + j] = value;
        }
}

// StreamHelper::get (projective_icp.cpp:43-62) + host step :195-209, on the device
__global__ void __launch_bounds__(256) icp_solve_kernel(const double *partials, int nblocks, float *T, int *ok, const float *T_src, const int *ok_src)
{
    __shared__ double sums[27];
    __shared__ __align__(16) double stage[RED_ROWS * 27];
    pdl_wait();
    pdl_trigger();
    float Tin[12];                                                       // loaded up front: in flight with the partials
#pragma unroll
    for (int i = 0; i < 12; ++i) Tin[i] = T_src[i];
    if (*ok_src == 0) { if (ok != ok_src && threadIdx.x == 0) *ok = 0; return; }
    if (ok != ok_src && threadIdx.x == 0) *ok = 1;
    reduce_partials(partials, nblocks, sums, stage);
    if (threadIdx.x != 0) return;
    double A[36], b[6];
    icp_unpack_sums(sums, A, b);
    double r[6];
    double det;
    if (!chol6_solve(A, b, r, &det)) {                                  // not safely SPD (or NaN): general path
        if (!icp_fallback_solve(A, b, r)) { *ok = 0; return; }
    } else if (fabs(det) < 1e-15 || det != det) { *ok = 0; return; }     // projective_icp.cpp:197-203
    icp_compose_pose(r, Tin, T);
}

__global__ void icp_init_kernel(float *T, int *ok)
{
    if (threadIdx.x < 12) T[threadIdx.x] = (threadIdx.x < 9 && threadIdx.x % 4 == 0) ? 1.f : 0.f;
    if (threadIdx.x == 0) *ok = 1;
}

constexpr int ICP_MAX_PARTIAL_BLOCKS = DF_NUM_SMS;

template <int NT>
void launch_accumulate_nt(const IcpParams &p, int blocks, cudaStream_t s)
{
    if (p.dcurr) launch_pdl(icp_accumulate_kernel<true, NT>, dim3(blocks), dim3(NT), 0, s, p);
    else launch_pdl(icp_accumulate_kernel<false, NT>, dim3(blocks), dim3(NT), 0, s, p);
}

int launch_accumulate(IcpParams &p, cudaStream_t s)
{
    const int npix = p.cols * p.rows;
    int blocks;
    if (npix >= ICP_MAX_PARTIAL_BLOCKS * 768) {         // 768 threads x 80 registers = one full-register-file block per SM
        blocks = ICP_MAX_PARTIAL_BLOCKS;
        launch_accumulate_nt<768>(p, blocks, s);
    } else {
        blocks = div_up(npix, 256) < ICP_MAX_PARTIAL_BLOCKS ? div_up(npix, 256) : ICP_MAX_PARTIAL_BLOCKS;
        if (blocks < 1) blocks = 1;
        launch_accumulate_nt<256>(p, blocks, s);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return -(int)e;
    return blocks;
}

}  // namespace

extern "C" int df_icp_accumulate(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch,
                                 const float *vprev, size_t vprev_pitch, const float *nprev, size_t nprev_pitch,
                                 int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres, float min_cosine,
                                 double *scratch, void *stream)
{
    if ((size_t)scratch & 15) return (int)cudaErrorMisalignedAddress;
    IcpParams p;
    p.vcurr = (const float4 *)vcurr; p.vcpitch = vcurr_pitch; p.ncurr = (const float4 *)ncurr; p.ncpitch = ncurr_pitch;
    p.vprev = (const float4 *)vprev; p.vppitch = vprev_pitch; p.nprev = (const float4 *)nprev; p.nppitch = nprev_pitch;
    p.dcurr = p.dprev = nullptr; p.dcpitch = p.dppitch = 0; p.finvx = p.finvy = 0.f;
    p.cols = cols; p.rows = rows; p.fcols = (float)cols; p.frows = (float)rows;
    p.fx = intr_level.fx; p.fy = intr_level.fy; p.cx = intr_level.cx; p.cy = intr_level.cy;
    p.dist2_thres = dist2_thres; p.min_cosine = min_cosine;
    p.T_val = make_aff(T); p.T_ptr = nullptr; p.ok_ptr = nullptr;
    p.partials = scratch + 32;
    const int blocks = launch_accumulate(p, (cudaStream_t)stream);
    if (blocks < 0) return -blocks;
    icp_reduce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(p.partials, blocks, scratch);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_icp_accumulate_depth(const unsigned short *dcurr, size_t dcurr_pitch, const float *ncurr, size_t ncurr_pitch,
                                       const unsigned short *dprev, size_t dprev_pitch, const float *nprev, size_t nprev_pitch,
                                       int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres, float min_cosine,
                                       double *scratch, void *stream)
{
    if (!dcurr || !dprev) return (int)cudaErrorInvalidValue;
    if ((size_t)scratch & 15) return (int)cudaErrorMisalignedAddress;
    IcpParams p;
    p.vcurr = p.vprev = nullptr; p.vcpitch = p.vppitch = 0;
    p.ncurr = (const float4 *)ncurr; p.ncpitch = ncurr_pitch; p.nprev = (const float4 *)nprev; p.nppitch = nprev_pitch;
    p.dcurr = dcurr; p.dcpitch = dcurr_pitch; p.dprev = dprev; p.dppitch = dprev_pitch;
    p.cols = cols; p.rows = rows; p.fcols = (float)cols; p.frows = (float)rows;
    p.fx = intr_level.fx; p.fy = intr_level.fy; p.cx = intr_level.cx; p.cy = intr_level.cy;
    p.finvx = 1.f / p.fx; p.finvy = 1.f / p.fy;
    p.dist2_thres = dist2_thres; p.min_cosine = min_cosine;
    p.T_val = make_aff(T); p.T_ptr = nullptr; p.ok_ptr = nullptr;
    p.partials = scratch + 32;
    const int blocks = launch_accumulate(p, (cudaStream_t)stream);
    if (blocks < 0) return -blocks;
    icp_reduce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(p.partials, blocks, scratch);
    DF_LAUNCH_CHECK();
    return 0;
}

namespace {
// the coarse-to-fine loop of both estimateTransform overloads (projective_icp.cpp:126-167 depth, :169-213 points)
int icp_estimate_impl(const float *const *vcurr, const unsigned short *const *dcurr, const float *const *ncurr, const float *const *vprev,
                      const unsigned short *const *dprev, const float *const *nprev, const int *cols, const int *rows, const size_t *pitch,
                      const size_t *dpitch, int levels, const int *iters, df_intr intr, float dist_thres, float angle_thres, float *T_dev,
                      int *ok_dev, double *scratch, cudaStream_t s)
{
    if ((size_t)scratch & 15) return (int)cudaErrorMisalignedAddress;
    icp_init_kernel<<<1, 32, 0, s>>>(T_dev, ok_dev);           // affine = Identity, projective_icp.cpp:175
    DF_LAUNCH_CHECK();
    for (int level = levels - 1; level >= 0; --level) {
        const int div = 1 << level;                          // setLevelIntr, projective_icp.cpp:17-23
        IcpParams p;
        p.vcurr = p.vprev = nullptr; p.dcurr = p.dprev = nullptr; p.dcpitch = p.dppitch = 0;
        if (dcurr) { p.dcurr = dcurr[level]; p.dprev = dprev[level]; p.dcpitch = p.dppitch = dpitch[level]; }
        else { p.vcurr = (const float4 *)vcurr[level]; p.vprev = (const float4 *)vprev[level]; }
        p.ncurr = (const float4 *)ncurr[level]; p.nprev = (const float4 *)nprev[level];
        p.vcpitch = p.ncpitch = p.vppitch = p.nppitch = pitch[level];
        p.cols = cols[level]; p.rows = rows[level]; p.fcols = (float)cols[level]; p.frows = (float)rows[level];
        p.fx = intr.fx / div; p.fy = intr.fy / div; p.cx = intr.cx / div; p.cy = intr.cy / div;
        p.finvx = 1.f / p.fx; p.finvy = 1.f / p.fy;
        p.dist2_thres = dist_thres * dist_thres;             // ComputeIcpHelper ctor, projective_icp.cpp:11-15
        p.min_cosine = cosf(angle_thres);
        p.T_val = Aff(); p.T_ptr = T_dev; p.ok_ptr = ok_dev;
        p.partials = scratch + 32;
        // (tried and dropped, round 1: running the solve as a last-block tail of the accumulate kernel -- the tail's 190 registers
        //  become the whole kernel's allocation, occupancy falls to one block per SM and the stage got slower; replacing the
        //  substitutions' divisions by reciprocal multiplies made the one-thread tail slower, not faster)
        for (int it = 0; it < iters[level]; ++it) {
            const int blocks = launch_accumulate(p, s);
            if (blocks < 0) return -blocks;
            launch_pdl(icp_solve_kernel, dim3(1), dim3(256), 0, s, (const double *)p.partials, blocks, T_dev, ok_dev, (const float *)T_dev, (const int *)ok_dev);
            DF_LAUNCH_CHECK();
        }
    }
    return 0;
}
}  // namespace

extern "C" int df_icp_estimate(const float *const *vcurr, const float *const *ncurr, const float *const *vprev, const float *const *nprev,
                               const int *cols, const int *rows, const size_t *pitch, int levels, const int *iters,
                               df_intr intr, float dist_thres, float angle_thres, float *T_dev, int *ok_dev, double *scratch,
                               void *stream)
{
    return icp_estimate_impl(vcurr, nullptr, ncurr, vprev, nullptr, nprev, cols, rows, pitch, nullptr, levels, iters, intr, dist_thres,
                             angle_thres, T_dev, ok_dev, scratch, (cudaStream_t)stream);
}

extern "C" int df_icp_estimate_depth(const unsigned short *const *dcurr, const float *const *ncurr, const unsigned short *const *dprev,
                                     const float *const *nprev, const int *cols, const int *rows, const size_t *depth_pitch,
                                     const size_t *normals_pitch, int levels, const int *iters, df_intr intr, float dist_thres,
                                     float angle_thres, float *T_dev, int *ok_dev, double *scratch, void *stream)
{
    if (!dcurr || !dprev) return (int)cudaErrorInvalidValue;
    return icp_estimate_impl(nullptr, dcurr, ncurr, nullptr, dprev, nprev, cols, rows, normals_pitch, depth_pitch, levels, iters, intr,
                             dist_thres, angle_thres, T_dev, ok_dev, scratch, (cudaStream_t)stream);
}

extern "C" int df_icp_solve_step(const double *partials, int nblocks, float *T, int *ok, void *stream)
{
    if ((size_t)partials & 15) return (int)cudaErrorMisalignedAddress;
    if (nblocks < 1) return (int)cudaErrorInvalidValue;
    launch_pdl(icp_solve_kernel, dim3(1), dim3(256), 0, (cudaStream_t)stream, partials, nblocks, T, ok, (const float *)T, (const int *)ok);
    DF_LAUNCH_CHECK();
    return 0;
}
