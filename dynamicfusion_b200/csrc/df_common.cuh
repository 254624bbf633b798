// df_common.cuh -- shared device helpers for the sm_90a kernels.
//
// Numerics contract (DESIGN.md "Numerics"): every float operation is the IEEE round-to-nearest operation at the same
// position and in the same order as the reference kernel it replaces; translation units are compiled with
// -fmad=false so nvcc never contracts a*b+c, and fused multiply-adds appear ONLY where the reference wrote
// __fmaf_rn (dot(), Projector).  This is what makes the kernels bit-comparable with oracle/ (gcc -ffp-contract=off).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/dfusion.h"

namespace dfb {

// SMs of the H100 SXM: the fixed grids of the grid-stride kernels and the ICP partial-sum row count are sized for one wave on it
constexpr int DF_NUM_SMS = 132;

struct Aff { float3 r0, r1, r2, t; };

__host__ inline Aff make_aff(const df_aff3f &a)
{
    Aff o;
    o.r0 = make_float3(a.R[0], a.R[1], a.R[2]);
    o.r1 = make_float3(a.R[3], a.R[4], a.R[5]);
    o.r2 = make_float3(a.R[6], a.R[7], a.R[8]);
    o.t = make_float3(a.t[0], a.t[1], a.t[2]);
    return o;
}
struct Mat3 { float3 r0, r1, r2; };
__host__ inline Mat3 make_mat3(const float *R)
{
    Mat3 o;
    o.r0 = make_float3(R[0], R[1], R[2]); o.r1 = make_float3(R[3], R[4], R[5]); o.r2 = make_float3(R[6], R[7], R[8]);
    return o;
}

// reference temp_utils.hpp:27-30
__device__ __forceinline__ float dot3(const float3 a, const float3 b) { return __fmaf_rn(a.x, b.x, __fmaf_rn(a.y, b.y, a.z * b.z)); }
__device__ __forceinline__ float3 add3(const float3 a, const float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 sub3(const float3 a, const float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 mul3(const float3 a, const float3 b) { return make_float3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float3 scale3(const float3 a, const float s) { return make_float3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float3 cross3(const float3 a, const float3 b)
{ return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
// normalized(): v * rsqrt(dot) in the reference (temp_utils.hpp:95-98); IEEE restatement 1/sqrt
__device__ __forceinline__ float3 normalized3(const float3 v) { return scale3(v, 1.0f / sqrtf(dot3(v, v))); }
// device.hpp:71-74
__device__ __forceinline__ float3 mat_mul(const float3 r0, const float3 r1, const float3 r2, const float3 v)
{ return make_float3(dot3(r0, v), dot3(r1, v), dot3(r2, v)); }
__device__ __forceinline__ float3 aff_mul(const Aff &a, const float3 v) { return add3(mat_mul(a.r0, a.r1, a.r2, v), a.t); }
__device__ __forceinline__ float3 mat3_mul(const Mat3 &m, const float3 v) { return mat_mul(m.r0, m.r1, m.r2, v); }

__device__ __forceinline__ float half_bits_to_float(unsigned short h) { return __half2float(__ushort_as_half(h)); }
__device__ __forceinline__ unsigned short float_to_half_bits(float f) { return __half_as_ushort(__float2half_rn(f)); }
__device__ __forceinline__ float qnan() { return __int_as_float(0x7fffffff); }

template <typename T> __device__ __forceinline__ const T *row_ptr(const T *base, size_t pitch, int y)
{ return (const T *)((const char *)base + (size_t)y * pitch); }
template <typename T> __device__ __forceinline__ T *row_ptr(T *base, size_t pitch, int y)
{ return (T *)((char *)base + (size_t)y * pitch); }

static inline int div_up(int a, int b) { return (a + b - 1) / b; }

// a voxel takes part in surface extraction iff W != 0 && F != 1.f (tsdf_volume.cu:548-633); 0x3c00 = half(1.0)
__device__ __forceinline__ bool vox_active(uint32_t v) { return (v >> 16) != 0 && (v & 0xffffu) != 0x3c00u; }
// F < 0 as the ray-cast's float comparison sees it: sign bit set, not -0, not NaN (a stored tsdf is never NaN)
__device__ __forceinline__ bool vox_negative(uint32_t v) { return (v & 0x8000u) != 0 && (v & 0x7fffu) != 0 && (v & 0x7fffu) <= 0x7c00u; }

// Brick table of the activity map (dfusion.h DF_BRICK): one byte per 8 x 8 x 8 brick of voxels, behind the per-stretch bytes, set when
// an integration stores a voxel with F < 0 in the brick.  Host + device view of where it lives.
struct BrickTable {
    unsigned char *bytes;      // nullptr: not tracked
    int nbx, nby, nbz;
};
__host__ __device__ inline size_t activity_stretch_bytes(int Dx, int Dy, int Dz)
{
    const size_t nvox = (size_t)Dx * Dy * Dz;
    return (((nvox + DF_ACTIVITY_VOXELS - 1) / DF_ACTIVITY_VOXELS + 16) + 255) & ~(size_t)255;
}
__host__ __device__ inline BrickTable brick_table(unsigned char *activity, int Dx, int Dy, int Dz)
{
    BrickTable b;
    b.nbx = (Dx + DF_BRICK - 1) / DF_BRICK; b.nby = (Dy + DF_BRICK - 1) / DF_BRICK; b.nbz = (Dz + DF_BRICK - 1) / DF_BRICK;
    b.bytes = activity ? activity + activity_stretch_bytes(Dx, Dy, Dz) : nullptr;
    return b;
}
// mark the brick of voxel (x, y, z); a quad of 4 x-adjacent voxels starting at a multiple of 4 lies in one brick
__device__ __forceinline__ void brick_mark(const BrickTable &b, int x, int y, int z)
{
    b.bytes[((size_t)(z >> 3) * b.nby + (y >> 3)) * b.nbx + (x >> 3)] = 1;
}

// Programmatic dependent launch (sm_90+): a kernel launched through launch_pdl may be scheduled while its predecessor in the
// stream is still draining; it must execute pdl_wait() before it touches anything the predecessor wrote (or overwrites anything
// the predecessor reads).  Every kernel of a chain calls pdl_wait() first and pdl_trigger() right after, so the data flow stays
// fully serialised and only the launch latency of the successor is hidden.  Both are no-ops in a normal launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

int pdl_enabled();          // DF_PDL (default 1), read once (df_common.cu)

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// df_solve_data_term with one more argument: an event recorded on the stream right before the LM/PCG kernel is launched (the frame loop
// starts the previous frame's surface extraction there: the solve occupies one 16-SM cluster while the other SMs idle).  solve.cu
int solve_data_term_ev(float *nodes, int M, const void *node_grid, const float *canon, const float *live, int N, int stride, int nonlinear_iters,
                       int linear_iters, int flags, double *stats_dev, void *workspace, cudaStream_t stream, cudaEvent_t before_lm);

}  // namespace dfb

// first statement of every kernel launched through launch_pdl
#define DF_PDL_ENTRY() do { dfb::pdl_wait(); dfb::pdl_trigger(); } while (0)

#define DF_LAUNCH_CHECK()                                  \
    do {                                                   \
        cudaError_t e__ = cudaGetLastError();              \
        if (e__ != cudaSuccess) return (int)e__;           \
    } while (0)
