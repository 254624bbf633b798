// reloc.cu -- the relocaliser's kernels (DF_KINFU_RELOCALISE; rules in include/dfusion.h): fern codes of a depth image, the keyframe
// lookup with the harvest append in the same launch, and the gate's counts on an ICP result.  The ray-cast, the pyramid and the ICP a
// relocalisation attempt runs are the frame loop's own entries.
#include "icp_assoc.cuh"
#include <math.h>

using namespace dfb;

namespace {

constexpr int MATCH_THREADS = DF_RELOC_KEYFRAMES;    // one thread per keyframe slot
constexpr int GATE_THREADS = 512;
constexpr int GATE_MAX_BLOCKS = DF_NUM_SMS;
static_assert(DF_RELOC_FERNS % 4 == 0, "the match compares codes a word at a time");
static_assert(GATE_MAX_BLOCKS * 24 + 16 <= DF_RELOC_GATE_WS_BYTES, "the gate's partials and counter fit its workspace");

// one thread per fern: the fern's byte from its four tests
__global__ void __launch_bounds__(256) fern_encode_kernel(const uint16_t *depth, size_t pitch, int cols, int rows, const int32_t *table,
                                                          int n_ferns, uint8_t *codes)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_ferns) return;
    const int32_t *t = table + (size_t)f * 12;
    unsigned code = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int u = t[3 * j], v = t[3 * j + 1], theta = t[3 * j + 2];
        if (u < 0 || v < 0 || u >= cols || v >= rows) continue;
        const int d = __ldg(row_ptr(depth, pitch, v) + u);
        code |= (unsigned)(d != 0 && d < theta) << j;
    }
    codes[f] = (uint8_t)code;
}

// dissimilarity of every held keyframe, the (dissimilarity, index) top-K by K rounds of a block-wide minimum, then the harvest append
__global__ void __launch_bounds__(MATCH_THREADS) fern_match_kernel(uint8_t *db_codes, float *db_poses, int *count_ptr, int capacity,
                                                                   const uint8_t *code, int n_ferns, int append, df_aff3f pose,
                                                                   df_reloc_match *out)
{
    __shared__ uint32_t frame_words[DF_RELOC_FERNS / 4];
    __shared__ unsigned long long warp_min[MATCH_THREADS / 32];
    __shared__ unsigned long long winner;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int count = *count_ptr;
    const int nw = n_ferns / 4;                                        // df_fern_match admits multiples of 4 only
    for (int i = tid; i < nw; i += blockDim.x) frame_words[i] = ((const uint32_t *)code)[i];
    __syncthreads();
    // key = dissimilarity << 32 | index: the smallest key is the (dissimilarity, index) minimum; a slot past the count never wins
    unsigned long long key = ~0ull;
    if (tid < count) {
        const uint8_t *row = db_codes + (size_t)tid * n_ferns;
        const uint32_t *rw = (const uint32_t *)row;
        int dis = 0;
        for (int i = 0; i < nw; ++i) dis += __popc(__vcmpne4(rw[i], frame_words[i]) & 0x01010101u);
        key = ((unsigned long long)dis << 32) | (unsigned)tid;
    }
    for (int r = 0; r < DF_RELOC_CANDIDATES; ++r) {
        unsigned long long m = key;
        for (int o = 16; o > 0; o >>= 1) { const unsigned long long x = __shfl_xor_sync(0xffffffffu, m, o); m = x < m ? x : m; }
        if (lane == 0) warp_min[warp] = m;
        __syncthreads();
        if (tid == 0) {
            unsigned long long w = warp_min[0];
            for (int i = 1; i < MATCH_THREADS / 32; ++i) w = warp_min[i] < w ? warp_min[i] : w;
            winner = w;
            const bool some = w != ~0ull;
            const int idx = some ? (int)(w & 0xffffffffu) : -1;
            out->index[r] = idx;
            out->dissimilarity[r] = some ? (int)(w >> 32) : DF_RELOC_FERNS + 1;
            for (int i = 0; i < 12; ++i) out->pose[r][i] = some ? db_poses[(size_t)idx * 12 + i] : 0.f;
        }
        __syncthreads();
        if (key == winner) key = ~0ull;                               // taken: the next round finds the next one
        __syncthreads();
    }
    if (tid != 0) return;
    const int min_dis = out->dissimilarity[0];
    const bool add = append && count < capacity && (count == 0 || min_dis > DF_RELOC_HARVEST_FERNS);
    if (add) {
        for (int i = 0; i < n_ferns; ++i) db_codes[(size_t)count * n_ferns + i] = code[i];
        float *p = db_poses + (size_t)count * 12;
        for (int i = 0; i < 9; ++i) p[i] = pose.R[i];
        for (int i = 0; i < 3; ++i) p[9 + i] = pose.t[i];
        *count_ptr = count + 1;
    }
    out->appended = add;
    out->count = count + add;
}

// the gate's counts: per-block partials (n_valid, n_in, sum_sq), then the last block to finish sums them in block order
__global__ void __launch_bounds__(GATE_THREADS) icp_inliers_kernel(const IcpParams p, const int *ok_ptr, df_reloc_gate *out, unsigned char *ws)
{
    constexpr int NW = GATE_THREADS / 32;
    __shared__ double s_sum[NW];
    __shared__ int s_valid[NW], s_in[NW];
    __shared__ bool last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    Aff T = p.T_val;
    if (p.T_ptr) {
        float t[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) t[i] = p.T_ptr[i];
        T.r0 = make_float3(t[0], t[1], t[2]);
        T.r1 = make_float3(t[3], t[4], t[5]);
        T.r2 = make_float3(t[6], t[7], t[8]);
        T.t = make_float3(t[9], t[10], t[11]);
    }
    int n_valid = 0, n_in = 0;
    double sum = 0.0;
    const int npix = p.cols * p.rows;
    for (int i = blockIdx.x * GATE_THREADS + tid; i < npix; i += gridDim.x * GATE_THREADS) {
        const int y = i / p.cols, x = i - y * p.cols;
        n_valid += !isnan(__ldg(row_ptr(p.vcurr, p.vcpitch, y) + x).x);
        float row[7];
        float3 s;
        float u, v;
        if (icp_row<false>(p, T, x, y, row, s, u, v)) {
            ++n_in;
            sum += (double)row[6] * (double)row[6];
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        n_valid += __shfl_xor_sync(0xffffffffu, n_valid, o);
        n_in += __shfl_xor_sync(0xffffffffu, n_in, o);
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
    }
    if (lane == 0) { s_sum[warp] = sum; s_valid[warp] = n_valid; s_in[warp] = n_in; }
    __syncthreads();
    double *part_sum = (double *)ws;
    int *part_cnt = (int *)(ws + GATE_MAX_BLOCKS * 8);
    unsigned *done = (unsigned *)(ws + GATE_MAX_BLOCKS * 16);
    if (tid == 0) {
        double bs = 0.0; int bv = 0, bi = 0;
        for (int w = 0; w < NW; ++w) { bs += s_sum[w]; bv += s_valid[w]; bi += s_in[w]; }
        part_sum[blockIdx.x] = bs;
        part_cnt[2 * blockIdx.x] = bv;
        part_cnt[2 * blockIdx.x + 1] = bi;
        __threadfence();
        last = atomicAdd(done, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || tid != 0) return;
    __threadfence();
    double ts = 0.0; int tv = 0, ti = 0;
    for (int b = 0; b < (int)gridDim.x; ++b) {
        ts += ((volatile double *)part_sum)[b];
        tv += ((volatile int *)part_cnt)[2 * b];
        ti += ((volatile int *)part_cnt)[2 * b + 1];
    }
    *done = 0u;                                                        // the workspace is left zeroed for the next call
    out->T[0] = T.r0.x; out->T[1] = T.r0.y; out->T[2] = T.r0.z;
    out->T[3] = T.r1.x; out->T[4] = T.r1.y; out->T[5] = T.r1.z;
    out->T[6] = T.r2.x; out->T[7] = T.r2.y; out->T[8] = T.r2.z;
    out->T[9] = T.t.x; out->T[10] = T.t.y; out->T[11] = T.t.z;
    out->ok = ok_ptr ? *ok_ptr : 1;
    out->n_valid = tv;
    out->n_in = ti;
    out->pad = 0;
    out->sum_sq = ts;
}

uint64_t splitmix_next(uint64_t &s)
{
    s += 0x9e3779b97f4a7c15ull;
    uint64_t z = s;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

}  // namespace

extern "C" int df_reloc_fern_table(unsigned long long seed, int cols, int rows, int n_ferns, int32_t *out)
{
    if (cols < 1 || rows < 1 || n_ferns < 1 || !out) return (int)cudaErrorInvalidValue;
    uint64_t s = seed;
    for (int f = 0; f < n_ferns; ++f)
        for (int j = 0; j < 4; ++j) {
            int32_t *t = out + (size_t)f * 12 + 3 * j;
            t[0] = (int32_t)(splitmix_next(s) % (uint64_t)cols);
            t[1] = (int32_t)(splitmix_next(s) % (uint64_t)rows);
            t[2] = (int32_t)(DF_RELOC_NEAR_MM + splitmix_next(s) % (uint64_t)(DF_RELOC_FAR_MM - DF_RELOC_NEAR_MM));
        }
    return 0;
}

extern "C" int df_fern_encode(const uint16_t *depth, size_t pitch, int cols, int rows, const int32_t *table, int n_ferns, uint8_t *codes,
                              void *stream)
{
    if (!depth || !table || !codes || cols < 1 || rows < 1 || n_ferns < 1 || pitch % 2 || pitch < (size_t)cols * 2)
        return (int)cudaErrorInvalidValue;
    fern_encode_kernel<<<div_up(n_ferns, 256), 256, 0, (cudaStream_t)stream>>>(depth, pitch, cols, rows, table, n_ferns, codes);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_fern_match(uint8_t *db_codes, float *db_poses, int *count, int capacity, const uint8_t *code, int n_ferns, int append,
                             df_aff3f pose, df_reloc_match *out, void *stream)
{
    if (!db_codes || !db_poses || !count || !code || !out || capacity < 1 || capacity > DF_RELOC_KEYFRAMES || n_ferns < 1 ||
        n_ferns > DF_RELOC_FERNS || n_ferns % 4 || (size_t)db_codes % 4 || (size_t)code % 4)
        return (int)cudaErrorInvalidValue;
    fern_match_kernel<<<1, MATCH_THREADS, 0, (cudaStream_t)stream>>>(db_codes, db_poses, count, capacity, code, n_ferns, append, pose, out);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_icp_inliers(const float *vcurr, size_t vcurr_pitch, const float *ncurr, size_t ncurr_pitch, const float *vprev,
                              size_t vprev_pitch, const float *nprev, size_t nprev_pitch, int cols, int rows, df_intr intr, const float *T_dev,
                              const int *ok_dev, float dist_thres, float angle_thres, df_reloc_gate *out, void *ws, void *stream)
{
    if (!vcurr || !ncurr || !vprev || !nprev || !out || !ws || cols < 1 || rows < 1 || (vcurr_pitch | ncurr_pitch | vprev_pitch | nprev_pitch) % 16)
        return (int)cudaErrorInvalidValue;
    IcpParams p;
    p.vcurr = (const float4 *)vcurr; p.vcpitch = vcurr_pitch; p.ncurr = (const float4 *)ncurr; p.ncpitch = ncurr_pitch;
    p.vprev = (const float4 *)vprev; p.vppitch = vprev_pitch; p.nprev = (const float4 *)nprev; p.nppitch = nprev_pitch;
    p.dcurr = p.dprev = nullptr; p.dcpitch = p.dppitch = 0; p.finvx = p.finvy = 0.f;
    p.cols = cols; p.rows = rows; p.fcols = (float)cols; p.frows = (float)rows;
    p.fx = intr.fx; p.fy = intr.fy; p.cx = intr.cx; p.cy = intr.cy;
    p.dist2_thres = dist_thres * dist_thres;                           // as df_icp_estimate forms them
    p.min_cosine = cosf(angle_thres);
    p.T_val = Aff{make_float3(1.f, 0.f, 0.f), make_float3(0.f, 1.f, 0.f), make_float3(0.f, 0.f, 1.f), make_float3(0.f, 0.f, 0.f)};
    p.T_ptr = T_dev; p.ok_ptr = nullptr; p.partials = nullptr;
    const int blocks = div_up(cols * rows, GATE_THREADS) < GATE_MAX_BLOCKS ? div_up(cols * rows, GATE_THREADS) : GATE_MAX_BLOCKS;
    icp_inliers_kernel<<<blocks, GATE_THREADS, 0, (cudaStream_t)stream>>>(p, ok_dev, out, (unsigned char *)ws);
    DF_LAUNCH_CHECK();
    return 0;
}

extern "C" int df_reloc_gate_accepts(const df_reloc_gate *g)
{
    if (!g->ok || g->n_valid < DF_RELOC_MIN_VALID || g->n_in < 1) return 0;
    if ((float)g->n_in < DF_RELOC_MIN_INLIER_FRAC * (float)g->n_valid) return 0;
    const double rms = sqrt(g->sum_sq / g->n_in);
    return rms <= (double)DF_RELOC_MAX_RMS;
}
