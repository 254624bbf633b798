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
// Colour tracking (df_icp_accumulate_color / df_icp_estimate_color) swaps the first kernel for icp_accumulate_color_kernel: the same body,
// plus a photometric row per accepted pixel into the same sums (rule in include/dfusion.h); the solve kernel and the launch count are unchanged.
#include "icp_assoc.cuh"
#include <float.h>
#include <stdlib.h>

using namespace dfb;

int dfb::pdl_enabled()
{
    static const int v = [] { const char *e = getenv("DF_PDL"); return e ? (int)(atoi(e) != 0) : 1; }();   // thread-safe one-time read
    return v;
}

namespace {

// the 27 float products of one 7-float row, in the sums' order (i, j >= i)
__device__ __forceinline__ void icp_add_row(float (&acc)[27], const float row[7])
{
    int k = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
        for (int j = a; j < 7; ++j) acc[k++] += row[a] * row[j];
}

// One row of partials per block and at most ICP_MAX_PARTIAL_BLOCKS (= one per SM) blocks: the solve tail's fixed-order sum over the
// rows is a chain of L2 round trips, so the row count is what its latency scales with (hence one row per SM of 768-thread blocks
// rather than four rows per SM of 256-thread blocks).  Pixels are dealt to threads linearly (coalesced
// along x, balanced to one pixel per warp whatever the image size).
// The body both accumulate kernels share: after an accepted pixel's geometric products, extra(x, y, s, u, v, acc) may add more rows (the
// colour kernel's photometric row; nothing in icp_accumulate_kernel).
template <bool DEPTH, int NT, class Extra>
__device__ __forceinline__ void icp_accumulate_body(const IcpParams &p, Extra extra)
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
            float3 s;
            float u, v;
            if (icp_row<DEPTH>(p, T, x, y, row, s, u, v)) {
                icp_add_row(acc, row);
                extra(x, y, s, u, v, acc);
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

template <bool DEPTH, int NT>
__global__ void __launch_bounds__(NT) icp_accumulate_kernel(const IcpParams p)
{
    icp_accumulate_body<DEPTH, NT>(p, [](int, int, float3, float, float, float (&)[27]) {});
}

// ---- colour tracking: the photometric row beside the geometric one (rule: include/dfusion.h, df_icp_accumulate_color) -------------------
struct IcpColorParams {
    IcpParams g;                     // the points variant's maps, level and gates
    const float *icurr; size_t icpitch;      // the current frame's intensity at the level
    const float4 *model; size_t mpitch;      // the model's (I, gu, gv, 0) at the level
    float weight, max_residual;
};

// the photometric row of pixel (x, y), whose geometric row gave s and (u, v): false where the rule has none
__device__ __forceinline__ bool photo_row(const IcpColorParams &p, int x, int y, const float3 s, float u, float v, float row[7])
{
    const float ic = __ldg(row_ptr(p.icurr, p.icpitch, y) + x);
    if (isnan(ic)) return false;
    const float fu = floorf(u), fv = floorf(v);
    const int i0 = (int)fu, j0 = (int)fv;
    if (i0 + 1 >= p.g.cols || j0 + 1 >= p.g.rows) return false;
    const float4 *r0 = row_ptr(p.model, p.mpitch, j0) + i0, *r1 = row_ptr(p.model, p.mpitch, j0 + 1) + i0;
    const float4 m00 = __ldg(r0), m10 = __ldg(r0 + 1), m01 = __ldg(r1), m11 = __ldg(r1 + 1);
    if (isnan(m00.x) || isnan(m10.x) || isnan(m01.x) || isnan(m11.x)) return false;
    const float a = u - fu, b = v - fv, a1 = 1.f - a, b1 = 1.f - b;
    const float im = (m00.x * a1 + m10.x * a) * b1 + (m01.x * a1 + m11.x * a) * b;
    const float r = ic - im;
    if (fabsf(r) > p.max_residual) return false;
    const float gu = (m00.y * a1 + m10.y * a) * b1 + (m01.y * a1 + m11.y * a) * b;
    const float gv = (m00.z * a1 + m10.z * a) * b1 + (m01.z * a1 + m11.z * a) * b;
    const float gfx = gu * p.g.fx, gfy = gv * p.g.fy;
    const float3 g = make_float3(gfx / s.z, gfy / s.z, -(gfx * s.x + gfy * s.y) / (s.z * s.z));
    const float3 c = cross3(s, g);
    const float w = p.weight;
    row[0] = w * c.x; row[1] = w * c.y; row[2] = w * c.z; row[3] = w * g.x; row[4] = w * g.y; row[5] = w * g.z;
    row[6] = w * r;
    return true;
}

// icp_accumulate_kernel<false, NT> with up to two rows per pixel: the geometric row, then the photometric one, into the same accumulators
template <int NT>
__global__ void __launch_bounds__(NT) icp_accumulate_color_kernel(const IcpColorParams p)
{
    icp_accumulate_body<false, NT>(p.g, [&](int x, int y, float3 s, float u, float v, float (&acc)[27]) {
        float row[7];
        if (photo_row(p, x, y, s, u, v, row)) icp_add_row(acc, row);
    });
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

// the launch rule of both accumulate kernels: 768 threads x 80 registers = one full-register-file block per SM from 132 x 768 pixels on,
// else 256-thread blocks, one per 256 pixels up to one per SM
int accumulate_blocks(int npix, int &nt)
{
    if (npix >= ICP_MAX_PARTIAL_BLOCKS * 768) {
        nt = 768;
        return ICP_MAX_PARTIAL_BLOCKS;
    }
    nt = 256;
    const int blocks = div_up(npix, 256) < ICP_MAX_PARTIAL_BLOCKS ? div_up(npix, 256) : ICP_MAX_PARTIAL_BLOCKS;
    return blocks < 1 ? 1 : blocks;
}

template <int NT>
void launch_accumulate_nt(const IcpParams &p, int blocks, cudaStream_t s)
{
    if (p.dcurr) launch_pdl(icp_accumulate_kernel<true, NT>, dim3(blocks), dim3(NT), 0, s, p);
    else launch_pdl(icp_accumulate_kernel<false, NT>, dim3(blocks), dim3(NT), 0, s, p);
}

// color == nullptr: the geometric kernel on p; else the colour kernel on *color (whose g is p)
int launch_accumulate(IcpParams &p, const IcpColorParams *color, cudaStream_t s)
{
    int nt;
    const int blocks = accumulate_blocks(p.cols * p.rows, nt);
    if (color) {
        if (nt == 768) launch_pdl(icp_accumulate_color_kernel<768>, dim3(blocks), dim3(768), 0, s, *color);
        else launch_pdl(icp_accumulate_color_kernel<256>, dim3(blocks), dim3(256), 0, s, *color);
    } else if (nt == 768) launch_accumulate_nt<768>(p, blocks, s);
    else launch_accumulate_nt<256>(p, blocks, s);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return -(int)e;
    return blocks;
}

// the points variant's parameters of one level (df_icp_accumulate, df_icp_accumulate_color)
IcpParams points_params(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch, const float *vprev, size_t vprev_pitch,
                        const float *nprev, size_t nprev_pitch, int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres,
                        float min_cosine, double *scratch)
{
    IcpParams p;
    p.vcurr = (const float4 *)vcurr; p.vcpitch = vcurr_pitch; p.ncurr = (const float4 *)ncurr; p.ncpitch = ncurr_pitch;
    p.vprev = (const float4 *)vprev; p.vppitch = vprev_pitch; p.nprev = (const float4 *)nprev; p.nppitch = nprev_pitch;
    p.dcurr = p.dprev = nullptr; p.dcpitch = p.dppitch = 0; p.finvx = p.finvy = 0.f;
    p.cols = cols; p.rows = rows; p.fcols = (float)cols; p.frows = (float)rows;
    p.fx = intr_level.fx; p.fy = intr_level.fy; p.cx = intr_level.cx; p.cy = intr_level.cy;
    p.dist2_thres = dist2_thres; p.min_cosine = min_cosine;
    p.T_val = make_aff(T); p.T_ptr = nullptr; p.ok_ptr = nullptr;
    p.partials = scratch + 32;
    return p;
}

}  // namespace

extern "C" int df_icp_accumulate(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch,
                                 const float *vprev, size_t vprev_pitch, const float *nprev, size_t nprev_pitch,
                                 int cols, int rows, df_intr intr_level, df_aff3f T, float dist2_thres, float min_cosine,
                                 double *scratch, void *stream)
{
    if ((size_t)scratch & 15) return (int)cudaErrorMisalignedAddress;
    IcpParams p = points_params(vcurr, vcurr_pitch, ncurr, ncurr_pitch, vprev, vprev_pitch, nprev, nprev_pitch, cols, rows, intr_level, T,
                                dist2_thres, min_cosine, scratch);
    const int blocks = launch_accumulate(p, nullptr, (cudaStream_t)stream);
    if (blocks < 0) return -blocks;
    icp_reduce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(p.partials, blocks, scratch);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_icp_accumulate_color(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch, const float *vprev,
                                       size_t vprev_pitch, const float *nprev, size_t nprev_pitch, const float *icurr, size_t icurr_pitch,
                                       const float *model, size_t model_pitch, int cols, int rows, df_intr intr_level, df_aff3f T,
                                       float dist2_thres, float min_cosine, float weight, float max_residual, double *scratch, void *stream)
{
    if ((size_t)scratch & 15) return (int)cudaErrorMisalignedAddress;
    if (!icurr || !model || icurr_pitch % 4 || model_pitch % 16) return (int)cudaErrorInvalidValue;
    IcpColorParams c;
    c.g = points_params(vcurr, vcurr_pitch, ncurr, ncurr_pitch, vprev, vprev_pitch, nprev, nprev_pitch, cols, rows, intr_level, T,
                        dist2_thres, min_cosine, scratch);
    c.icurr = icurr; c.icpitch = icurr_pitch; c.model = (const float4 *)model; c.mpitch = model_pitch;
    c.weight = weight; c.max_residual = max_residual;
    const int blocks = launch_accumulate(c.g, &c, (cudaStream_t)stream);
    if (blocks < 0) return -blocks;
    icp_reduce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(c.g.partials, blocks, scratch);
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
    const int blocks = launch_accumulate(p, nullptr, (cudaStream_t)stream);
    if (blocks < 0) return -blocks;
    icp_reduce_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(p.partials, blocks, scratch);
    DF_LAUNCH_CHECK();
    return 0;
}

namespace {
// the intensity maps of df_icp_estimate_color, per level
struct ColorLevels {
    const float *const *icurr; const size_t *ipitch;
    const float *const *model; const size_t *mpitch;
    float weight, max_residual;
};

// the coarse-to-fine loop of both estimateTransform overloads (projective_icp.cpp:126-167 depth, :169-213 points); color (points
// variant only): the photometric rows as well
int icp_estimate_impl(const float *const *vcurr, const unsigned short *const *dcurr, const float *const *ncurr, const float *const *vprev,
                      const unsigned short *const *dprev, const float *const *nprev, const int *cols, const int *rows, const size_t *pitch,
                      const size_t *dpitch, int levels, const int *iters, df_intr intr, float dist_thres, float angle_thres, float *T_dev,
                      int *ok_dev, double *scratch, cudaStream_t s, const ColorLevels *color = nullptr)
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
        IcpColorParams c;
        if (color) {
            c.g = p;
            c.icurr = color->icurr[level]; c.icpitch = color->ipitch[level];
            c.model = (const float4 *)color->model[level]; c.mpitch = color->mpitch[level];
            c.weight = color->weight; c.max_residual = color->max_residual;
        }
        // (tried and dropped, round 1: running the solve as a last-block tail of the accumulate kernel -- the tail's 190 registers
        //  become the whole kernel's allocation, occupancy falls to one block per SM and the stage got slower; replacing the
        //  substitutions' divisions by reciprocal multiplies made the one-thread tail slower, not faster)
        for (int it = 0; it < iters[level]; ++it) {
            const int blocks = launch_accumulate(p, color ? &c : nullptr, s);
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

extern "C" int df_icp_estimate_color(const float *const *vcurr, const float *const *ncurr, const float *const *vprev, const float *const *nprev,
                                     const float *const *icurr, const size_t *icurr_pitch, const float *const *model, const size_t *model_pitch,
                                     const int *cols, const int *rows, const size_t *pitch, int levels, const int *iters, df_intr intr,
                                     float dist_thres, float angle_thres, float weight, float max_residual, float *T_dev, int *ok_dev,
                                     double *scratch, void *stream)
{
    if (!icurr || !model || !icurr_pitch || !model_pitch) return (int)cudaErrorInvalidValue;
    for (int l = 0; l < levels; ++l)
        if (!icurr[l] || !model[l] || icurr_pitch[l] % 4 || model_pitch[l] % 16) return (int)cudaErrorInvalidValue;
    const ColorLevels c{icurr, icurr_pitch, model, model_pitch, weight, max_residual};
    return icp_estimate_impl(vcurr, nullptr, ncurr, vprev, nullptr, nprev, cols, rows, pitch, nullptr, levels, iters, intr, dist_thres,
                             angle_thres, T_dev, ok_dev, scratch, (cudaStream_t)stream, &c);
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
