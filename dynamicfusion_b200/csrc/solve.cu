// solve.cu -- warp-field data-term solve on sm_90a, fully device-resident.
//
// Replaces WarpFieldOptimiser::optimiseWarpData -> CombinedSolver -> Opt (Terra-JIT'd LM/PCG) of the reference
// (kfusion/src/warp_field_optimiser.cpp:7-16, kfusion/include/opt/CombinedSolver.h:25-197,
// kfusion/solvers/dynamicfusion.t:26-52, deps/Opt/API/src/solverGPUGaussNewton.t:1016-1177), which per frame
// re-allocates seven device images, runs N more CPU k-NN queries to build the graph, and then iterates a matrix-free
// PCG whose every product scatters through per-edge atomicAdd and whose every dot product is fetched to the host.
//
// The energy is LINEAR in the unknown node translations T (J block = -w_vk * I3, constant), so this design builds the
// small normal system once per frame and keeps the whole LM/PCG iteration on one SM:
//   1. solve_prepare   per vertex: 8-NN of the (warped) canonical vertex (shared-memory node tiles), weights
//                      exp(-d^2/2w^2), b_v = live_v - canon_v; per-node incidence counts (warp-aggregated atomics)
//   2. solve_scan/fill CSR incidence lists node -> (vertex, k)
//   3. solve_rows      one block per node i: A_i* = sum_v w_vi w_v* in a shared-memory hash (double), gb_i = sum_v w_vi b_v;
//                      rows are written sorted by column (deterministic) in column-major ELL
//   4. solve_lm        one 1024-thread block: Levenberg-Marquardt (Ceres-style trust region, radius 1e4) around a
//                      Jacobi-preconditioned CG on the sparse M x M system for 3 right-hand sides, all in double;
//                      writes the translations back into the nodes (encodeTranslation).  No host round trip.
// Sums over vertices are accumulated in double, so the atomics' ordering does not change the rounded result.
#include "warp_common.cuh"
#include <cooperative_groups.h>
#include <cstdlib>
#include <cstdio>

namespace cg = cooperative_groups;

using namespace dfb;

namespace {

constexpr int HCAP = 1024;      // hash slots per node row
constexpr int ROWCAP = 512;     // stored nonzeros per row (ELL stride); overflow is reported in stats[5]
constexpr int LM_THREADS = 1024;
constexpr int TILE_W = 16, TILE_H = 8, TILE_PIX = TILE_W * TILE_H;   // image tile of the tile-record assembly
constexpr int TILE_LCAP = 64;   // distinct nodes a tile's records hold; a tile with more hands the frame to the per-entry kernels

struct SolveWs {
    int *idx; float *w; float4 *b;                 // per vertex
    int *cnt, *off, *cursor, *inc;                 // incidence CSR
    int *rownnz; int *col; double *val;            // ELL (column-major): col[e * M + i]
    double *gb, *diag;                             // [3*M], [M]
    double *cd, *minv;                             // [M], [M]
    double *c0_partials;                           // per prepare-block 0.5*sum|b|^2 and valid count
    double *vec;                                   // 7 vectors of 3*M doubles
    int *flags;                                    // [0] overflow
    int *row_order;                                // [M] node index per solve_rows block: heaviest incidence lists first
    int *blockcnt;                                 // [M][prepare_blocks]: entries of node n contributed by vertex block b, then their exclusive prefix over b
    int prepare_blocks;
    // tile records of the image-shaped assembly (solve_tiles / solve_rows_tiles): NT = N / 128 tiles of 16 x 8 pixels, 0 = not available
    int ntiles;
    int *rec_L, *rec_nodes;                        // [NT], [NT][TILE_LCAP]: the tile's distinct nodes, ascending
    double *rec_T, *rec_g;                         // [NT][TILE_LCAP][TILE_LCAP], [NT][TILE_LCAP][4]: sum over the tile's vertices of w_a w_b, w_a b
    unsigned char *touch;                          // [M][NT]: 1 + local index of node n in tile t, 0 = the tile does not hold it
};

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

size_t layout(SolveWs &ws, char *base, int M, int N)
{
    size_t o = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + o : nullptr; o += align_up(bytes); return p; };
    ws.idx = (int *)take((size_t)N * 8 * 4);
    ws.w = (float *)take((size_t)N * 8 * 4);
    ws.b = (float4 *)take((size_t)N * 16);
    ws.cnt = (int *)take((size_t)(M + 1) * 4);
    ws.off = (int *)take((size_t)(M + 1) * 4);
    ws.cursor = (int *)take((size_t)(M + 1) * 4);
    ws.inc = (int *)take((size_t)N * 8 * 4);
    ws.rownnz = (int *)take((size_t)M * 4);
    ws.col = (int *)take((size_t)M * ROWCAP * 4);
    ws.val = (double *)take((size_t)M * ROWCAP * 8);
    ws.gb = (double *)take((size_t)M * 3 * 8);
    ws.diag = (double *)take((size_t)M * 8);
    ws.cd = (double *)take((size_t)M * 8);
    ws.minv = (double *)take((size_t)M * 8);
    ws.prepare_blocks = (N + 255) / 256;
    ws.c0_partials = (double *)take((size_t)ws.prepare_blocks * 8 * 2 * 8);   // one (0.5*|b|^2, count) pair per warp
    ws.vec = (double *)take((size_t)M * 3 * 8 * 7);
    ws.flags = (int *)take(64);
    ws.row_order = (int *)take((size_t)M * 4);
    ws.blockcnt = (int *)take((size_t)M * ws.prepare_blocks * 4);
    ws.ntiles = N % TILE_PIX == 0 ? N / TILE_PIX : 0;
    const size_t nrec = ws.ntiles ? (size_t)ws.ntiles + 256 * 8 : 0;   // one record per tile + TILE_OV_CAP * TILE_STRIPS strip records
    ws.rec_L = (int *)take(nrec * 4);
    ws.rec_nodes = (int *)take(nrec * TILE_LCAP * 4);
    ws.rec_T = (double *)take(nrec * TILE_LCAP * TILE_LCAP * 8);
    ws.rec_g = (double *)take(nrec * TILE_LCAP * 4 * 8);
    ws.touch = (unsigned char *)take((size_t)M * ws.ntiles);
    return o;
}

// ------------------------------------------------------------------------------------------------------------------
constexpr int PREPARE_THREADS = 256;

__global__ void __launch_bounds__(PREPARE_THREADS, 4) solve_prepare_kernel(const float *__restrict__ nodes, int M, const void *__restrict__ grid,
                                                            const float *__restrict__ canon, const float *__restrict__ live, int N, int stride,
                                                            SolveWs ws, int cols)
{
    DF_PDL_ENTRY();
    __shared__ KnnSmem sm;
    const int v = patch_vertex(blockIdx.x, threadIdx.x, cols);      // cols > 0: 8 x 4 pixel patches per warp (solve_fill maps the same way)
    float3 c = make_float3(0.f, 0.f, 0.f), l = c;
    bool valid = false, valid_c = false;       // valid_c: the vertex can be queried; valid: the row enters the solve
    if (v < N) {
        const float *cp = canon + (size_t)v * stride, *lp = live + (size_t)v * stride;
        c = make_float3(cp[0], cp[1], cp[2]); l = make_float3(lp[0], lp[1], lp[2]);
        valid_c = !(isnan(c.x) || isnan(c.y) || isnan(c.z));
        valid = valid_c && !(isnan(l.x) || isnan(l.y) || isnan(l.z));
    }
    int bi[8]; float bd[8];
    if (grid) knn8_grid(grid, valid_c, c.x, c.y, c.z, bi, bd);
    else knn8_scan(nodes, M, valid_c, c.x, c.y, c.z, sm, bi, bd);
    double half_b2 = 0.0;
    if (v < N) {
        float3 b = make_float3(0.f, 0.f, 0.f);
        if (valid) { b = sub3(l, c); half_b2 = 0.5 * ((double)b.x * b.x + (double)b.y * b.y + (double)b.z * b.z); }
        ws.b[v] = make_float4(b.x, b.y, b.z, valid ? 1.f : 0.f);
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        // idx / w describe the vertex itself (re-used by the following warp, DF_WARP_REUSE_KNN); only rows that are valid
        // for the solve are counted into the incidence lists
        const int nq = (v < N && valid_c) ? bi[k] : -1;
        float wk = 0.f;
        if (nq >= 0) wk = node_weighting(bd[k], __ldg(nodes + (size_t)nq * DF_NODE_STRIDE + 11));
        if (v < N) { ws.idx[(size_t)v * 8 + k] = nq; ws.w[(size_t)v * 8 + k] = wk; }
        const int n = valid ? nq : -1;
        // warp-aggregated incidence count: neighbouring pixels share nodes, one atomic per distinct node per warp
        const unsigned grp = __match_any_sync(0xffffffffu, n);
        if (n >= 0 && (int)(__ffs(grp) - 1) == (int)(threadIdx.x & 31)) atomicAdd(ws.blockcnt + (size_t)n * gridDim.x + blockIdx.x, __popc(grp));
    }
    // deterministic per-WARP partials of 0.5*|b|^2 and of the valid-row count (no block barrier: a warp whose queries are far
    // from the node cloud takes several times longer than its neighbours, and nobody should wait for it)
    double vcount = valid ? 1.0 : 0.0;
    for (int o = 16; o > 0; o >>= 1) { half_b2 += __shfl_xor_sync(0xffffffffu, half_b2, o); vcount += __shfl_xor_sync(0xffffffffu, vcount, o); }
    if ((threadIdx.x & 31) == 0) {
        const int wid = blockIdx.x * (PREPARE_THREADS / 32) + (threadIdx.x >> 5);
        ws.c0_partials[2 * wid] = half_b2; ws.c0_partials[2 * wid + 1] = vcount;
    }
}

__global__ void __launch_bounds__(1024) solve_scan_kernel(SolveWs ws, int M)
{
    DF_PDL_ENTRY();
    __shared__ int partial[1024];
    const int t = threadIdx.x;
    const int per = (M + 1023) / 1024;
    const int b = min(M, t * per), e = min(M, b + per);
    int s = 0;
    for (int i = b; i < e; ++i) s += ws.cnt[i];
    partial[t] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = t >= o ? partial[t - o] : 0;
        __syncthreads();
        partial[t] += v;
        __syncthreads();
    }
    int run = partial[t] - s;
    for (int i = b; i < e; ++i) { ws.off[i] = run; run += ws.cnt[i]; ws.cursor[i] = 0; }
    if (t == 1023) ws.off[M] = partial[1023];
    if (t == 0) { ws.flags[0] = 0; ws.flags[1] = 0; ws.flags[2] = 0; ws.flags[3] = 0; ws.flags[4] = 0; ws.flags[5] = 0; ws.flags[6] = 0; ws.flags[7] = 0; }   // [0] row overflow, [1] v6 handed the frame to v5, [2] the tile assembly handed it to fill + rows, [3] the tile assembly ran
    // Launch order of solve_rows: one block per node, and the rim nodes' lists are 100x the median -- scheduled last they are the
    // kernel's tail.  Longest-processing-time-first: nodes grouped by floor(log2(count)), heaviest group first (the order inside a
    // group is whatever the shared-memory atomics give: it affects only WHEN a row is assembled, never its value).
    __shared__ int hist[32], start[32];
    if (t < 32) hist[t] = 0;
    __syncthreads();
    for (int i = b; i < e; ++i) atomicAdd(&hist[31 - __clz(ws.cnt[i] | 1)], 1);
    __syncthreads();
    if (t == 0) { int acc = 0; for (int g = 31; g >= 0; --g) { start[g] = acc; acc += hist[g]; } }
    __syncthreads();
    for (int i = b; i < e; ++i) ws.row_order[atomicAdd(&start[31 - __clz(ws.cnt[i] | 1)], 1)] = i;
}

// per node: exclusive prefix of its per-block entry counts (in place) and the total -> cnt[n].  One warp per node, coalesced.
__global__ void __launch_bounds__(256) solve_blockscan_kernel(SolveWs ws, int M)
{
    DF_PDL_ENTRY();
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= M) return;
    int *row = ws.blockcnt + (size_t)n * ws.prepare_blocks;
    int run = 0;
    for (int b0 = 0; b0 < ws.prepare_blocks; b0 += 32) {
        const int b = b0 + lane;
        const int c = b < ws.prepare_blocks ? row[b] : 0;
        int inc = c;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (b < ws.prepare_blocks) row[b] = run + inc - c;
        run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) ws.cnt[n] = run;
}

// Incidence lists node -> (vertex, k) in a CANONICAL order: by vertex block, then warp, then neighbour slot k, then lane.  Round 1 handed
// out the positions with an atomic cursor per node, which made the order -- and through it the rounding of every double sum solve_rows
// forms over a list -- depend on kernel timing: a translation could differ in its last bit between two runs of the same frame (seen when
// several frame loops fed one stream).  Here a block owns, for every node its vertices touch, the range that solve_blockscan reserved for
// (node, block); the block's cursors live in a small shared-memory hash and its warps take their turns one after the other, so every
// entry's position is a pure function of the data.  (A first version sorted the block's 2,048 (node, entry) pairs with a bitonic
// network, which cost more than this.)
// >= distinct nodes a block of 256 vertices can touch: 256 x 8 = 2,048 entries (typically ~30 nodes for an image, but a flat list in no
// spatial order touches ~1,300 of 2,000 nodes).  A smaller table could overflow, and an overflowing block writes none of its entries.
constexpr int FILL_HASH = 2048;
__global__ void __launch_bounds__(256) solve_fill_kernel(SolveWs ws, int N, int only_if_flag, int cols)
{
    DF_PDL_ENTRY();
    if (only_if_flag && ws.flags[2] == 0) return;                  // launched behind the tile assembly as its fallback: nothing to do
    __shared__ int hkey[FILL_HASH], hcur[FILL_HASH];
    __shared__ int overflow;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int v = patch_vertex(blockIdx.x, tid, cols);             // the vertex -> block map of solve_prepare (its per-block counts are this block's bases)
    const bool valid = v < N && ws.b[v].w != 0.f;
    for (int s = tid; s < FILL_HASH; s += 256) hkey[s] = -1;
    if (tid == 0) overflow = 0;
    __syncthreads();
    int nk[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        nk[k] = valid ? ws.idx[(size_t)v * 8 + k] : -1;
        // one lane per distinct node of the warp claims the node's slot; whoever claims it first loads the block's base for that node
        const unsigned grp = __match_any_sync(0xffffffffu, nk[k]);
        if (nk[k] >= 0 && lane == __ffs(grp) - 1) {
            unsigned slot = ((unsigned)nk[k] * 2654435761u) & (FILL_HASH - 1);
            int probe = 0;
            for (; probe < FILL_HASH; ++probe) {
                const int prev = atomicCAS(&hkey[slot], -1, nk[k]);
                if (prev == -1) { hcur[slot] = ws.blockcnt[(size_t)nk[k] * gridDim.x + blockIdx.x]; break; }
                if (prev == nk[k]) break;
                slot = (slot + 1) & (FILL_HASH - 1);
            }
            if (probe == FILL_HASH) overflow = 1;
        }
    }
    __syncthreads();
    if (overflow) { if (tid == 0) ws.flags[0] = 1; return; }        // cannot happen for 256-vertex blocks (<= 2,048 entries < capacity): reported like a row overflow
    for (int w = 0; w < 8; ++w) {                                  // the warps take their turns: positions depend on the data only
        if (warp == w) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int n = nk[k];
                const unsigned grp = __match_any_sync(0xffffffffu, n);
                int base = 0;
                const int leader = __ffs(grp) - 1;
                if (n >= 0 && lane == leader) {
                    unsigned slot = ((unsigned)n * 2654435761u) & (FILL_HASH - 1);
                    while (hkey[slot] != n) slot = (slot + 1) & (FILL_HASH - 1);
                    base = hcur[slot];
                    hcur[slot] = base + __popc(grp);               // leaders of one match hold distinct nodes: no conflict
                }
                base = __shfl_sync(0xffffffffu, base, leader);
                if (n >= 0) ws.inc[ws.off[n] + base + __popc(grp & ((1u << lane) - 1u))] = v * 8 + k;
                __syncwarp();
            }
        }
        __syncthreads();
    }
}

// One block per node i: A_i* (sparse), gb_i, diag_i.
//
// A typical row has ~725 incident entries x 8 contributions that all land on the ~30 distinct columns of the row (a rim node late
// in a sequence: 10^5 entries).  History: v1 = hash insert + shared-memory double atomicAdd per contribution
// (contended compare-and-swap loops); v2 = equal keys combined inside the warp first (match.any + shuffles), faster on a
// late frame; a fixed-point integer-atomic variant was slower AND wrong (weights span 60 orders of magnitude).  This one:
//   pass 1  the column SET of the row: integer CAS inserts only (lanes holding the same key elect one leader with match.any);
//           the occupied slots are ranked by key -> the row's sorted column list, written straight to the ELL arrays;
//   pass 2  the values: every warp owns a private accumulator per column (ROWS_PRIV columns x 16 warps), a warp's lanes holding
//           the same column are summed with shuffles and the leader adds to the warp's own slot -- no atomics at all;
//           the per-warp slots are added in warp order at the end, so the row is bit-reproducible from run to run.
// Rows with more than ROWS_PRIV columns take the atomic path for the values.
constexpr int ROWS_THREADS = 512;
constexpr int ROWS_WARPS = ROWS_THREADS / 32;
constexpr int ROWS_PRIV = 128;

__device__ __forceinline__ int rows_find_slot(const int *keys, int j)
{
    unsigned slot = ((unsigned)j * 2654435761u) & (HCAP - 1);
    for (int probe = 0; probe < HCAP; ++probe) {
        if (keys[slot] == j) return (int)slot;
        slot = (slot + 1) & (HCAP - 1);
    }
    return 0;
}

__global__ void __launch_bounds__(ROWS_THREADS) solve_rows_kernel(SolveWs ws, int M, int N, int quirk, int only_if_flag)
{
    DF_PDL_ENTRY();
    if (only_if_flag && ws.flags[2] == 0) return;
    __shared__ int keys[HCAP];
    __shared__ int slot_rank[HCAP];
    __shared__ int list[HCAP];
    __shared__ double vals[HCAP];                       // only used by rows with more than ROWS_PRIV columns
    __shared__ double priv[ROWS_WARPS][ROWS_PRIV];
    __shared__ int nlist;
    __shared__ double red[3][ROWS_WARPS];
    const int i = ws.row_order[blockIdx.x];
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    for (int s = tid; s < HCAP; s += ROWS_THREADS) { keys[s] = -1; vals[s] = 0.0; }
    for (int s = tid; s < ROWS_WARPS * ROWS_PRIV; s += ROWS_THREADS) (&priv[0][0])[s] = 0.0;
    if (tid == 0) nlist = 0;
    __syncthreads();
    const int beg = ws.off[i], end = ws.off[i + 1];
    const bool quirk_row = quirk && i == 0 && N > 0 && ws.b[0].w != 0.f;

    // ---- pass 1: which columns does the row have?
    for (int base = beg; base < end; base += ROWS_THREADS) {
        const int e = base + tid;
        int js[8];
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) js[kk] = -1;
        if (e < end) {
            const int v = ws.inc[e] >> 3;
            const int4 ia = *reinterpret_cast<const int4 *>(ws.idx + (size_t)v * 8), ib = *reinterpret_cast<const int4 *>(ws.idx + (size_t)v * 8 + 4);
            js[0] = ia.x; js[1] = ia.y; js[2] = ia.z; js[3] = ia.w; js[4] = ib.x; js[5] = ib.y; js[6] = ib.z; js[7] = ib.w;
        }
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const int j = js[kk];
            const unsigned grp = __match_any_sync(0xffffffffu, j);
            if (j < 0 || lane != __ffs(grp) - 1) continue;
            unsigned slot = ((unsigned)j * 2654435761u) & (HCAP - 1);
            for (int probe = 0; probe < HCAP; ++probe) {
                const int prev = atomicCAS(&keys[slot], -1, j);
                if (prev == -1 || prev == j) break;
                slot = (slot + 1) & (HCAP - 1);
                if (probe == HCAP - 1) ws.flags[0] = 1;
            }
        }
    }
    if (quirk_row && tid == 0) {                          // CombinedSolver.h:70-79: N extra edges on (node 0, node 0)
        unsigned slot = 0u;
        for (int probe = 0; probe < HCAP; ++probe) {
            const int prev = atomicCAS(&keys[slot], -1, 0);
            if (prev == -1 || prev == 0) break;
            slot = (slot + 1) & (HCAP - 1);
        }
    }
    __syncthreads();
    for (int s = tid; s < HCAP; s += ROWS_THREADS)
        if (keys[s] >= 0) list[atomicAdd(&nlist, 1)] = s;
    __syncthreads();
    const int nn = nlist;
    if (nn > ROWCAP && tid == 0) ws.flags[0] = 1;
    for (int a = tid; a < nn; a += ROWS_THREADS) {        // rank by key = position in the sorted row
        const int sa = list[a], ka = keys[sa];
        int rank = 0;
        for (int bq = 0; bq < nn; ++bq) rank += keys[list[bq]] < ka;
        slot_rank[sa] = rank;
        if (rank < ROWCAP) ws.col[(size_t)rank * M + i] = ka;
    }
    __syncthreads();
    const bool use_priv = nn <= ROWS_PRIV;

    // ---- pass 2: the values
    double g0 = 0.0, g1 = 0.0, g2 = 0.0;
    for (int base = beg; base < end; base += ROWS_THREADS) {
        const int e = base + tid;
        double wi = 0.0;
        int js[8];
        float wj[8];
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) { js[kk] = -1; wj[kk] = 0.f; }
        if (e < end) {
            const int entry = ws.inc[e];
            const int v = entry >> 3;
            wi = (double)ws.w[entry];
            const float4 b = ws.b[v];
            g0 += wi * (double)b.x; g1 += wi * (double)b.y; g2 += wi * (double)b.z;
            const int4 ia = *reinterpret_cast<const int4 *>(ws.idx + (size_t)v * 8), ib = *reinterpret_cast<const int4 *>(ws.idx + (size_t)v * 8 + 4);
            const float4 wa = *reinterpret_cast<const float4 *>(ws.w + (size_t)v * 8), wb = *reinterpret_cast<const float4 *>(ws.w + (size_t)v * 8 + 4);
            js[0] = ia.x; js[1] = ia.y; js[2] = ia.z; js[3] = ia.w; js[4] = ib.x; js[5] = ib.y; js[6] = ib.z; js[7] = ib.w;
            wj[0] = wa.x; wj[1] = wa.y; wj[2] = wa.z; wj[3] = wa.w; wj[4] = wb.x; wj[5] = wb.y; wj[6] = wb.z; wj[7] = wb.w;
        }
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const int j = js[kk];
            const double contrib = wi * (double)wj[kk];
            const unsigned grp = __match_any_sync(0xffffffffu, j);
            if (j >= 0) {
                double sum = contrib;
                if (grp == 0xffffffffu) {
                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                } else if (grp & (grp - 1u)) {
                    sum = 0.0;
                    for (unsigned m = grp; m; m &= m - 1u) sum += __shfl_sync(grp, contrib, __ffs(m) - 1);
                }
                if (lane == __ffs(grp) - 1) {
                    const int slot = rows_find_slot(keys, j);
                    if (use_priv) priv[warp][slot_rank[slot]] += sum;     // leaders of one match hold distinct columns: no conflict
                    else atomicAdd(&vals[slot], sum);
                }
            }
            __syncwarp();                                  // the next neighbour slot may hit a column another lane just updated
        }
    }
    if (quirk_row && tid == 0) {
        double sw = 0.0;
        for (int k = 0; k < 8; ++k) sw += (double)ws.w[k];
        const float4 b = ws.b[0];
        g0 += (double)N * sw * (double)b.x; g1 += (double)N * sw * (double)b.y; g2 += (double)N * sw * (double)b.z;
        const int slot = rows_find_slot(keys, 0);
        if (use_priv) priv[0][slot_rank[slot]] += (double)N * sw * sw;
        else atomicAdd(&vals[slot], (double)N * sw * sw);
    }
    for (int o = 16; o > 0; o >>= 1) { g0 += __shfl_xor_sync(0xffffffffu, g0, o); g1 += __shfl_xor_sync(0xffffffffu, g1, o); g2 += __shfl_xor_sync(0xffffffffu, g2, o); }
    if (lane == 0) { red[0][warp] = g0; red[1][warp] = g1; red[2][warp] = g2; }
    __syncthreads();
    for (int a = tid; a < nn; a += ROWS_THREADS) {
        const int sa = list[a], ka = keys[sa], rank = slot_rank[sa];
        double total = 0.0;
        if (use_priv) {
#pragma unroll
            for (int w = 0; w < ROWS_WARPS; ++w) total += priv[w][rank];
        } else {
            total = vals[sa];
        }
        if (rank < ROWCAP) ws.val[(size_t)rank * M + i] = total;
        if (ka == i) ws.diag[i] = total;
    }
    if (tid == 0) {
        ws.rownnz[i] = min(nn, ROWCAP);
        double a = 0.0, b = 0.0, c = 0.0;
        for (int q = 0; q < ROWS_WARPS; ++q) { a += red[0][q]; b += red[1][q]; c += red[2][q]; }
        ws.gb[i] = a; ws.gb[M + i] = b; ws.gb[2 * M + i] = c;
        if (end == beg && !quirk_row) ws.diag[i] = 0.0;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Tile-record assembly (round 2, second session; default when the vertices are an image, DF_SOLVE_IMAGE_COLS in the flags).
//
// solve_fill + solve_rows above assemble A = W^T W entry by entry: every vertex is visited once per neighbour (8 x), each visit pushes 8
// products through match.any + shuffle groups into the node's hash -- 12 M contributions per frame, the largest kernels after the
// LM solve.  But the 128 pixels of a 16 x 8 image tile see the same dozen nodes (measured on the bench sequence: 16 distinct nodes on
// average, 42 at most), so the tile's contribution to A is a small DENSE block T = W_t^T W_t over its L local nodes.  One 128-thread
// block per tile builds the tile's node table (hash, ranked by node index: local indices are a function of the data), scatters its
// weights into a 128 x L shared-memory matrix and lets warp w form rows a = w, w+4, ... of T with lane = column: only the vertices that
// hold node a are visited (bit masks from ballots, in pixel order), products of two floats are exact in double, sums run in a fixed
// order.  The row of the normal matrix for node i is then the sum of row local(i) of the ~12 tiles that hold it (a byte map touch[i][tile]
// written by the tiles), accumulated by 8 warps in private shared-memory slots and combined in warp order: no atomics on values, bit-
// reproducible, and ~40 x fewer operations than the per-entry path.  Tiles with more than TILE_LCAP nodes or rows with more than
// RT_HCAP * 3/4 columns raise ws.flags[2] and the per-entry kernels (launched right behind, no-ops otherwise) redo the frame.
constexpr int TW_STRIDE = TILE_LCAP + 4;     // a vertex's row of the tile matrix (floats): 64 node columns, then (b.x, b.y, b.z, 0); 16-byte aligned quads
constexpr int TILE_HASH = 256;

constexpr int TILE_STRIPS = TILE_PIX / TILE_W;   // an overflowing tile is redone as its 8 pixel rows, one record each
constexpr int TILE_OV_CAP = 256;                 // overflowing tiles per frame that get strip records (beyond that: the per-entry kernels)
constexpr unsigned char TOUCH_STRIPS = 255;      // byte-map code: look the node up in the tile's strip records

__global__ void __launch_bounds__(TILE_PIX) solve_tiles_kernel(SolveWs ws, int cols, int rows)
{
    DF_PDL_ENTRY();
    __shared__ __align__(16) float wloc[TILE_PIX * TW_STRIDE];
    __shared__ int hkey[TILE_HASH], hval[TILE_HASH];
    __shared__ int list[TILE_HASH];
    __shared__ int sorted[TILE_LCAP];
    __shared__ int nl, ov_base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tiles_x = cols / TILE_W;
    const int tile = blockIdx.x, tx = tile % tiles_x, ty = tile / tiles_x;
    const int px = tx * TILE_W + (tid % TILE_W), py = ty * TILE_H + (tid / TILE_W);
    const int v = py * cols + px;
    const float4 b = ws.b[v];
    const bool valid = b.w != 0.f;
    if (blockIdx.x == 0 && tid == 0) ws.flags[3] = 1;
    if (!__syncthreads_or(valid)) { if (tid == 0) ws.rec_L[tile] = 0; return; }
    int nk[8]; float wk[8];
    {
        const int4 ia = *reinterpret_cast<const int4 *>(ws.idx + (size_t)v * 8), ib = *reinterpret_cast<const int4 *>(ws.idx + (size_t)v * 8 + 4);
        const float4 wa = *reinterpret_cast<const float4 *>(ws.w + (size_t)v * 8), wb = *reinterpret_cast<const float4 *>(ws.w + (size_t)v * 8 + 4);
        nk[0] = ia.x; nk[1] = ia.y; nk[2] = ia.z; nk[3] = ia.w; nk[4] = ib.x; nk[5] = ib.y; nk[6] = ib.z; nk[7] = ib.w;
        wk[0] = wa.x; wk[1] = wa.y; wk[2] = wa.z; wk[3] = wa.w; wk[4] = wb.x; wk[5] = wb.y; wk[6] = wb.z; wk[7] = wb.w;
    }

    // the node set of the member vertices -> nl distinct nodes in hkey / list (block-uniform result)
    auto build_table = [&](bool member) -> int {
        __syncthreads();                                           // the previous pass is done with the tables
        for (int s = tid; s < TILE_HASH; s += TILE_PIX) hkey[s] = -1;
        if (tid == 0) nl = 0;
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int j = member ? nk[k] : -1;
            const unsigned grp = __match_any_sync(0xffffffffu, j);
            if (j < 0 || lane != __ffs(grp) - 1) continue;
            unsigned slot = ((unsigned)j * 2654435761u) & (TILE_HASH - 1);
            for (int probe = 0; probe < TILE_HASH; ++probe) {
                const int prev = atomicCAS(&hkey[slot], -1, j);
                if (prev == -1 || prev == j) break;
                slot = (slot + 1) & (TILE_HASH - 1);
            }
        }
        __syncthreads();
        for (int s = tid; s < TILE_HASH; s += TILE_PIX)
            if (hkey[s] >= 0) list[atomicAdd(&nl, 1)] = s;
        __syncthreads();
        return nl;
    };
    // the record `rid` of the member vertices (L <= TILE_LCAP distinct nodes in the table)
    auto emit = [&](bool member, int L, int rid, bool write_touch) {
        if (tid < L) {                                             // local index = rank of the node index
            const int sa = list[tid], ka = hkey[sa];
            int rank = 0;
            for (int q = 0; q < L; ++q) rank += hkey[list[q]] < ka;
            hval[sa] = rank;
            sorted[rank] = ka;
        }
        for (int e = tid; e < TILE_PIX * TW_STRIDE / 4; e += TILE_PIX) reinterpret_cast<float4 *>(wloc)[e] = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        // scatter: the vertex's weights into its row (column = local node index), its right-hand side into columns 64..66
        if (member) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int j = nk[k];
                if (j < 0) continue;
                unsigned slot = ((unsigned)j * 2654435761u) & (TILE_HASH - 1);
                while (hkey[slot] != j) slot = (slot + 1) & (TILE_HASH - 1);
                wloc[tid * TW_STRIDE + hval[slot]] = wk[k];
            }
            wloc[tid * TW_STRIDE + TILE_LCAP] = b.x; wloc[tid * TW_STRIDE + TILE_LCAP + 1] = b.y; wloc[tid * TW_STRIDE + TILE_LCAP + 2] = b.z;
        }
        __syncthreads();
        // [T | g] = W^T [W | b] as a small dense product: a thread owns a 4 x 4 block of the result and one of KS interleaved slices of the
        // 128 vertices (quads of floats per load, products of two floats are exact in double, so the fused multiply-add rounds like mul + add);
        // the slices are lanes of one warp and are summed by a fixed butterfly.  (The first version walked, per row, the bit mask of the vertices
        // that hold the node: ~16 instructions per non-zero product, 25 k warp instructions per tile -- ncu r02_s2_c15; the zeros cost less.)
        const int nA = (L + 3) >> 2, nsb = nA * (nA + 1);        // blocks of four rows x (blocks of four node columns + the right-hand side)
        const int KS = nsb <= 16 ? 8 : (nsb <= 32 ? 4 : (nsb <= 64 ? 2 : 1));
        for (int sb0 = 0; sb0 < nsb; sb0 += TILE_PIX / KS) {
            const int sb = sb0 + tid / KS, ks = tid % KS;
            const bool act = sb < nsb;
            const int sa = act ? sb / (nA + 1) : 0, sq = act ? sb % (nA + 1) : 0;
            const int cb = sq == nA ? TILE_LCAP : 4 * sq;
            double acc[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
            if (act) {
                for (int u = ks; u < TILE_PIX; u += KS) {
                    const float4 A = *reinterpret_cast<const float4 *>(wloc + u * TW_STRIDE + 4 * sa);
                    const float4 B = *reinterpret_cast<const float4 *>(wloc + u * TW_STRIDE + cb);
                    const double av[4] = {(double)A.x, (double)A.y, (double)A.z, (double)A.w}, bv[4] = {(double)B.x, (double)B.y, (double)B.z, (double)B.w};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
                }
            }
            for (int o = 1; o < KS; o <<= 1) {
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] += __shfl_xor_sync(0xffffffffu, acc[i][j], o);
            }
            if (act && ks == 0) {
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int a = 4 * sa + i;
                    if (a >= L) continue;
                    if (sq == nA) {
#pragma unroll
                        for (int j = 0; j < 3; ++j) ws.rec_g[((size_t)rid * TILE_LCAP + a) * 4 + j] = acc[i][j];
                    } else {
                        double *T = ws.rec_T + ((size_t)rid * TILE_LCAP + a) * TILE_LCAP + cb;
#pragma unroll
                        for (int j = 0; j < 4; ++j) if (cb + j < L) T[j] = acc[i][j];
                        if (write_touch && sq == 0) ws.touch[(size_t)sorted[a] * ws.ntiles + tile] = (unsigned char)(a + 1);
                    }
                }
            }
        }
        if (tid < L) ws.rec_nodes[(size_t)rid * TILE_LCAP + tid] = sorted[tid];
        if (tid == 0) ws.rec_L[rid] = L;
    };

    const int L = build_table(valid);
    if (tid == 0) atomicMax(&ws.flags[4], L);                      // diagnostics (DF_SOLVE_TRACE): the frame's largest tile
    if (L <= TILE_LCAP) { emit(valid, L, tile, true); return; }
    // More nodes than a record holds (late in a sequence the warped rim scatters: 88 nodes seen in one tile).  The tile is redone as its
    // 8 pixel rows, each a record of its own in the overflow pool; the byte map sends the rows kernel there.  A full hash table (the
    // node set is then incomplete), a strip that still overflows or an exhausted pool hand the frame to the per-entry kernels.
    if (L >= TILE_HASH - 1) { if (tid == 0) { ws.flags[2] = 1; ws.rec_L[tile] = 0; } return; }
    if (tid == 0) ov_base = atomicAdd(&ws.flags[7], 1);
    __syncthreads();
    const int ov = ov_base;
    if (ov >= TILE_OV_CAP) { if (tid == 0) { ws.flags[2] = 1; ws.rec_L[tile] = 0; } return; }
    for (int q = tid; q < L; q += TILE_PIX) ws.touch[(size_t)hkey[list[q]] * ws.ntiles + tile] = TOUCH_STRIPS;
    if (tid == 0) ws.rec_L[tile] = -(ov + 1);                      // where the tile's strip records start: ntiles + ov * TILE_STRIPS
    for (int sidx = 0; sidx < TILE_STRIPS; ++sidx) {
        const bool member = valid && (tid / TILE_W) == sidx;
        const int Ls = build_table(member);
        const int rid = ws.ntiles + ov * TILE_STRIPS + sidx;
        if (Ls > TILE_LCAP) { if (tid == 0) { ws.flags[2] = 1; ws.rec_L[rid] = 0; } continue; }   // (16 vertices x 8 neighbours = 128 possible)
        emit(member, Ls, rid, false);
    }
}

constexpr int RT_THREADS = 256;
constexpr int RT_WARPS = RT_THREADS / 32;
constexpr int RT_HCAP = 256;                 // hash slots per row; rows with more than 3/4 of them in use go to the per-entry kernels
constexpr int RT_LIST = 4096;                // tiles per node kept in shared memory; longer lists are re-read from the byte map

__global__ void __launch_bounds__(RT_THREADS) solve_rows_tiles_kernel(SolveWs ws, int M, int N, int quirk)
{
    DF_PDL_ENTRY();
    __shared__ int keys[RT_HCAP];
    __shared__ int slot_rank[RT_HCAP];
    __shared__ int occ[RT_HCAP];
    __shared__ double priv[RT_WARPS][RT_HCAP];
    __shared__ double gpart[RT_WARPS][3];
    __shared__ int tlist[RT_LIST];                      // (tile << 8) | byte-map code
    __shared__ int wsum[RT_WARPS + 1];
    __shared__ int nocc, skip;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) skip = ws.flags[2];                    // a tile (or an earlier row) overflowed: fill + rows behind this kernel take the frame
    __syncthreads();                                     // (one reader: other blocks may raise the flag while this one starts)
    if (skip) return;
    const int i = ws.row_order[blockIdx.x];
    const int NT = ws.ntiles;
    for (int s = tid; s < RT_HCAP; s += RT_THREADS) keys[s] = -1;
    for (int s = tid; s < RT_WARPS * RT_HCAP; s += RT_THREADS) (&priv[0][0])[s] = 0.0;
    if (tid == 0) nocc = 0;
    // ---- the tiles that hold node i, in tile order (thread t owns a contiguous stretch of the byte map)
    const unsigned char *trow = ws.touch + (size_t)i * NT;
    const int per = (NT + RT_THREADS - 1) / RT_THREADS;
    const int t_beg = min(NT, tid * per), t_end = min(NT, t_beg + per);
    int mine = 0;
    for (int t = t_beg; t < t_end; ++t) mine += trow[t] != 0;
    int inc = mine;
    for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += x; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (tid == 0) { int acc = 0; for (int w = 0; w < RT_WARPS; ++w) { const int c = wsum[w]; wsum[w] = acc; acc += c; } wsum[RT_WARPS] = acc; }
    __syncthreads();
    const int ntl = wsum[RT_WARPS];
    if (tid == 0) atomicMax(&ws.flags[5], ntl);
    if (ntl > RT_LIST) { if (tid == 0) ws.flags[2] = 2; return; }
    {
        int at = wsum[warp] + inc - mine;
        for (int t = t_beg; t < t_end; ++t) { const int l = trow[t]; if (l) tlist[at++] = (t << 8) | l; }
    }
    __syncthreads();
    // ---- accumulate: warp w takes list entries w, w + 8, ... (tile order); lane = column of the tile's block
    double g = 0.0;
    bool over = false;
    auto add_row = [&](int rid, int a, int L) {             // row a of record rid into this warp's slots
        const double *T = ws.rec_T + ((size_t)rid * TILE_LCAP + a) * TILE_LCAP;
        const int *nd = ws.rec_nodes + (size_t)rid * TILE_LCAP;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int c = lane + 32 * h;
            if (c >= L) continue;
            const double val = T[c];
            if (val == 0.0) continue;                      // the two nodes share no vertex of this tile (or a weight underflowed: a zero entry)
            const int j = nd[c];
            unsigned slot = ((unsigned)j * 2654435761u) & (RT_HCAP - 1);
            int probe = 0;
            for (; probe < RT_HCAP; ++probe) {
                const int prev = atomicCAS(&keys[slot], -1, j);
                if (prev == -1 || prev == j) break;
                slot = (slot + 1) & (RT_HCAP - 1);
            }
            if (probe == RT_HCAP) { over = true; continue; }
            priv[warp][slot] += val;                       // the lanes of one step hold distinct columns: no conflict
        }
        if (lane < 3) g += ws.rec_g[((size_t)rid * TILE_LCAP + a) * 4 + lane];
        __syncwarp();
    };
    for (int e = warp; e < ntl; e += RT_WARPS) {
        const int tile = tlist[e] >> 8, code = tlist[e] & 255;
        if (code != TOUCH_STRIPS) { add_row(tile, code - 1, ws.rec_L[tile]); continue; }
        const int first = ws.ntiles + (-ws.rec_L[tile] - 1) * TILE_STRIPS;   // the tile overflowed: its pixel rows are records of their own
        for (int sidx = 0; sidx < TILE_STRIPS; ++sidx) {
            const int rid = first + sidx, L = ws.rec_L[rid];
            const int *nd = ws.rec_nodes + (size_t)rid * TILE_LCAP;
            const unsigned hit = __ballot_sync(0xffffffffu, (lane < L && nd[lane] == i) || (lane + 32 < L && nd[lane + 32] == i));
            if (!hit) continue;
            const int l0 = __ffs(hit) - 1;                  // the lane that saw node i: in column l0 or l0 + 32
            const int a = __shfl_sync(0xffffffffu, (lane < L && nd[lane] == i) ? lane : lane + 32, l0);
            add_row(rid, a, L);
        }
    }
    if (lane < 3) gpart[warp][lane] = g;
    const bool quirk_row = quirk && i == 0 && N > 0 && ws.b[0].w != 0.f;
    __syncthreads();
    if (quirk_row && tid == 0) {                          // CombinedSolver.h:70-79: N extra edges on (node 0, node 0)
        double sw = 0.0;
        for (int k = 0; k < 8; ++k) sw += (double)ws.w[k];
        unsigned slot = 0u;
        for (int probe = 0; probe < RT_HCAP; ++probe) {
            const int prev = atomicCAS(&keys[slot], -1, 0);
            if (prev == -1 || prev == 0) break;
            slot = (slot + 1) & (RT_HCAP - 1);
        }
        priv[0][slot] += (double)N * sw * sw;
        const float4 b = ws.b[0];
        gpart[0][0] += (double)N * sw * (double)b.x; gpart[0][1] += (double)N * sw * (double)b.y; gpart[0][2] += (double)N * sw * (double)b.z;
    }
    __syncthreads();
    for (int s = tid; s < RT_HCAP; s += RT_THREADS)
        if (keys[s] >= 0) occ[atomicAdd(&nocc, 1)] = s;
    __syncthreads();
    const int nn = nocc;
    if (tid == 0) atomicMax(&ws.flags[6], nn);
    if (over || nn > RT_HCAP * 3 / 4) ws.flags[2] = 3;    // too many columns for this kernel: the per-entry kernels redo the frame
    if (tid == 0) ws.diag[i] = 0.0;                       // a row whose own weights all underflowed has no diagonal entry
    __syncthreads();
    for (int q = tid; q < nn; q += RT_THREADS) {          // rank by key = position in the sorted row
        const int sa = occ[q], ka = keys[sa];
        int rank = 0;
        for (int r = 0; r < nn; ++r) rank += keys[occ[r]] < ka;
        double total = 0.0;
#pragma unroll
        for (int w = 0; w < RT_WARPS; ++w) total += priv[w][sa];
        ws.col[(size_t)rank * M + i] = ka;
        ws.val[(size_t)rank * M + i] = total;
        if (ka == i) ws.diag[i] = total;
    }
    if (tid == 0) {
        ws.rownnz[i] = nn;
        double a = 0.0, b = 0.0, c = 0.0;
        for (int w = 0; w < RT_WARPS; ++w) { a += gpart[w][0]; b += gpart[w][1]; c += gpart[w][2]; }
        ws.gb[i] = a; ws.gb[M + i] = b; ws.gb[2 * M + i] = c;
        if (ntl == 0 && !quirk_row) ws.diag[i] = 0.0;
    }
}

// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum(double v, double *smem)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < 32) {
        t = threadIdx.x < (blockDim.x >> 5) ? smem[threadIdx.x] : 0.0;
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) smem[32] = t;
    }
    __syncthreads();
    return smem[32];
}

__device__ __forceinline__ void spmv(const SolveWs &ws, int M, const double *in, double *out)
{
    for (int n = threadIdx.x; n < M; n += blockDim.x) {
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        const int nnz = ws.rownnz[n];
        for (int e = 0; e < nnz; ++e) {
            const int j = ws.col[(size_t)e * M + n];
            const double a = ws.val[(size_t)e * M + n];
            a0 += a * in[j]; a1 += a * in[M + j]; a2 += a * in[2 * M + j];
        }
        out[n] = a0; out[M + n] = a1; out[2 * M + n] = a2;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(LM_THREADS) solve_lm_kernel(float *nodes, int M, SolveWs ws, int nl_iters, int lin_iters, double *stats)
{
    __shared__ double red[40];
    const int tid = threadIdx.x;
    const int M3 = 3 * M;
    double *x = ws.vec, *g = x + M3, *dl = g + M3, *r = dl + M3, *z = r + M3, *p = z + M3, *Ap = p + M3;

    // x0 = current node translations (CombinedSolver.h:165-172)
    for (int n = tid; n < M; n += LM_THREADS) {
        const float4 *n4 = reinterpret_cast<const float4 *>(nodes + (size_t)n * DF_NODE_STRIDE);
        const float4 a = n4[0], b = n4[1], c = n4[2];
        const Quat t = dq_translation(Quat{a.w, b.x, b.y, b.z}, Quat{b.w, c.x, c.y, c.z});
        x[n] = t.x; x[M + n] = t.y; x[2 * M + n] = t.z;
    }
    __syncthreads();
    // cost0 = 0.5|b|^2 - x.gb + 0.5 x^T A x
    double c0 = 0.0, nvalid = 0.0, nnz = 0.0;
    for (int i = tid; i < ws.prepare_blocks * (PREPARE_THREADS / 32); i += LM_THREADS) { c0 += ws.c0_partials[2 * i]; nvalid += ws.c0_partials[2 * i + 1]; }
    for (int n = tid; n < M; n += LM_THREADS) nnz += (double)ws.rownnz[n];
    c0 = block_sum(c0, red);
    nvalid = block_sum(nvalid, red);
    nnz = block_sum(nnz, red);
    spmv(ws, M, x, Ap);
    double t0 = 0.0;
    for (int i = tid; i < M3; i += LM_THREADS) t0 += x[i] * (0.5 * Ap[i] - ws.gb[i]);
    double cost = c0 + block_sum(t0, red);
    const double cost0 = cost;

    double radius = 1e4, decrease = 2.0;          // solverGPUGaussNewton.t:26-39
    int it = 0, pcg_total = 0;
    const bool overflow = ws.flags[0] != 0;       // a row overflowed: leave the field unchanged (see solve_lm_v5_kernel)
    if (overflow) nl_iters = 0;
    for (; it < nl_iters; ++it) {
        // g = gb - A x
        spmv(ws, M, x, Ap);
        for (int i = tid; i < M3; i += LM_THREADS) g[i] = ws.gb[i] - Ap[i];
        __syncthreads();
        // PCG on (A + C) dl = g, C = clamp(diag, 1e-6, 1e32) / radius, Jacobi preconditioner
        double rz_part = 0.0;
        for (int i = tid; i < M3; i += LM_THREADS) {
            const double d = ws.diag[i % M];
            const double cdamp = fmin(fmax(d, 1e-6), 1e32) / radius;
            dl[i] = 0.0; r[i] = g[i];
            const double zi = g[i] / (d + cdamp);
            z[i] = zi; p[i] = zi;
            rz_part += g[i] * zi;
        }
        double rz = block_sum(rz_part, red);
        double Q0 = 0.0;
        for (int l = 0; l < lin_iters && rz > 0.0; ++l) {
            spmv(ws, M, p, Ap);
            double pAp_part = 0.0;
            for (int i = tid; i < M3; i += LM_THREADS) {
                const double d = ws.diag[i % M];
                const double ap = Ap[i] + fmin(fmax(d, 1e-6), 1e32) / radius * p[i];
                Ap[i] = ap;
                pAp_part += p[i] * ap;
            }
            const double pAp = block_sum(pAp_part, red);
            if (!(pAp > 0.0)) break;
            const double alpha = rz / pAp;
            double rz_new_part = 0.0, q_part = 0.0;
            for (int i = tid; i < M3; i += LM_THREADS) {
                const double d = ws.diag[i % M];
                const double dli = dl[i] + alpha * p[i];
                const double ri = r[i] - alpha * Ap[i];
                const double zi = ri / (d + fmin(fmax(d, 1e-6), 1e32) / radius);
                dl[i] = dli; r[i] = ri; z[i] = zi;
                rz_new_part += ri * zi;
                q_part += dli * (ri + g[i]);
            }
            const double rz_new = block_sum(rz_new_part, red);
            const double Q1 = -0.5 * block_sum(q_part, red);
            const double beta = rz_new / rz;
            for (int i = tid; i < M3; i += LM_THREADS) p[i] = z[i] + beta * p[i];
            __syncthreads();
            rz = rz_new;
            ++pcg_total;
            // Ceres/Opt q-tolerance (solverGPUGaussNewton.t:1093-1101)
            const double zeta = (double)(l + 1) * (Q1 - Q0) / Q1;
            Q0 = Q1;
            if (zeta < 1e-4) break;
        }
        // model change = 0.5 dl.(g + r + C dl);  A dl = g - r - C dl  => new cost = cost - dl.g + 0.5 dl.(A dl)
        double m_part = 0.0, a_part = 0.0, dg_part = 0.0;
        for (int i = tid; i < M3; i += LM_THREADS) {
            const double d = ws.diag[i % M];
            const double cd = fmin(fmax(d, 1e-6), 1e32) / radius * dl[i];
            m_part += dl[i] * (g[i] + r[i] + cd);
            a_part += dl[i] * (g[i] - r[i] - cd);
            dg_part += dl[i] * g[i];
        }
        const double model = 0.5 * block_sum(m_part, red);
        const double dAd = block_sum(a_part, red);
        const double dg = block_sum(dg_part, red);
        const double new_cost = cost - dg + 0.5 * dAd;
        const double change = cost - new_cost;
        const double rho = model > 0.0 ? change / model : 0.0;
        if (change >= 0.0 && rho > 1e-3) {
            for (int i = tid; i < M3; i += LM_THREADS) x[i] += dl[i];
            __syncthreads();
            const bool stop = change <= cost * 1e-6;        // function_tolerance, CombinedSolver.h:88
            cost = new_cost;
            const double f = 1.0 - (2.0 * rho - 1.0) * (2.0 * rho - 1.0) * (2.0 * rho - 1.0);
            radius /= fmax(f, 1.0 / 3.0);
            radius = fmin(radius, 1e16);
            decrease = 2.0;
            if (stop) { ++it; break; }
        } else {
            radius /= decrease; decrease *= 2.0;
            if (radius <= 1e-32) break;
        }
    }
    // write back: encodeTranslation (CombinedSolver.h:189-197, dual_quaternion.hpp:82-85)
    for (int n = tid; n < M && !overflow; n += LM_THREADS) {
        float *nd = nodes + (size_t)n * DF_NODE_STRIDE;
        const Quat rot = {nd[3], nd[4], nd[5], nd[6]};
        const Quat h = qhalf(Quat{0.f, (float)x[n], (float)x[M + n], (float)x[2 * M + n]});
        const Quat d = qmul(h, rot);
        nd[7] = d.w; nd[8] = d.x; nd[9] = d.y; nd[10] = d.z;
    }
    if (tid == 0 && stats) {
        stats[0] = cost0; stats[1] = cost; stats[2] = (double)it; stats[3] = nvalid; stats[4] = (double)pcg_total; stats[5] = (double)ws.flags[0];
        stats[6] = nnz; stats[7] = (ws.flags[3] && !ws.flags[2]) ? -1.5 : -2.0;   // -2: solved by this kernel; -1.5: matrix from the tile records
    }
}

// ------------------------------------------------------------------------------------------------------------------
// LM / PCG on ONE THREAD-BLOCK CLUSTER.  The linear system is tiny (M x M sparse, ~1e5 non-zeros) and every PCG iteration needs
// global dot products, so the iteration is bound by exchange latency, not by bandwidth.  History: v1 = the
// one-block kernel above (kept as the fallback for systems that do not fit a cluster's shared memory); v2 = 8-CTA cluster, vectors
// through L2; v3 = matrix + vectors in shared memory, DSMEM pushes; v4 = CG vectors in registers, Morton row order + need-mask, one
// cluster barrier per sum; v5 (below, the only cluster version left in the tree) = v4 with transaction barriers.
constexpr int LMC_CTAS = 8;

constexpr int LM4_THREADS = 512;

struct Lm4Layout {
    int rpc, tpr, ent_cap;
    size_t off_svec, off_val, off_col, total;
};

__host__ __device__ inline Lm4Layout lm4_layout(int M, int ent_cap, int ncta = LMC_CTAS)
{
    Lm4Layout L;
    L.rpc = (M + ncta - 1) / ncta;
    L.tpr = 1;
    while (L.tpr < 32 && L.tpr * 2 * L.rpc <= LM4_THREADS) L.tpr *= 2;
    L.ent_cap = ent_cap;
    size_t o = 0;
    L.off_svec = o; o += (size_t)3 * M * 8;
    L.off_val = o; o += (size_t)ent_cap * LM4_THREADS * 8;
    L.off_col = o; o += (((size_t)ent_cap * LM4_THREADS * 2) + 15) & ~(size_t)15;
    L.total = o;
    return L;
}

// ------------------------------------------------------------------------------------------------------------------
// v5: v4 with every cluster barrier inside the iteration replaced by transaction barriers.  A profile of v4 (source
// view): a large share of the stall samples sit on the barrier's MEMBAR.ALL.GPU / ERRBAR /
// UCGABAR_WAIT and many on the generic remote stores that the barrier's release fence has to drain (lg_throttle).
// Here a remote write is a `st.async` that carries its own completion: it lands in the destination CTA's shared memory and
// decrements the transaction count of an mbarrier there.  A CTA that has received all the bytes it expects simply goes on:
//   * cluster-wide sum: warp 0 sends the CTA's partial to all eight CTAs (8 x NV x 8 B expected per CTA), two mbarriers used
//     alternately (a fast CTA can be one reduction ahead, never two: it needs my next partial first);
//   * vector exchange: the owner lane sends its row's three values to the CTAs in its need-mask; the byte count every CTA will
//     receive is fixed by the sparsity pattern and is established once with an ordinary all-reduce;
//   * write-after-read safety comes for free: a partial is computed FROM the shared-memory reads of the mat-vec, so whoever has
//     received everybody's partial knows that everybody has finished reading the vector it is about to overwrite.
// No fence, no cluster barrier, no L1 flush inside the LM/PCG iteration; the arithmetic and its order are v4's.
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t mapa_u32(uint32_t addr, uint32_t rank)
{
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect(uint32_t bar, uint32_t bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile("{\n\t.reg .pred P1;\n\tLAB_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1, %2;\n\t@P1 bra DONE;\n\tbra LAB_WAIT;\n\tDONE:\n\t}"
                 ::"r"(bar), "r"(parity), "r"(0x989680) : "memory");
}
__device__ __forceinline__ void st_async_f64(uint32_t remote_addr, double v, uint32_t remote_bar)
{
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b64 [%0], %1, [%2];" ::"r"(remote_addr), "l"(__double_as_longlong(v)), "r"(remote_bar) : "memory");
}

// Row -> lane mapping of the cluster LM kernels (shared by v5 and v6).
struct LmRowMap {
    unsigned short t_rl[LM4_THREADS];
    unsigned char t_sub[LM4_THREADS], t_tr[LM4_THREADS], row_cls[LM4_THREADS];
    int cls_cnt[8], cls_start[8], bal_sum[2];
};

__device__ __forceinline__ void lm_map_rows(LmRowMap &mp, const SolveWs &ws, const int *order, int cta, int rpc, int tpr_fixed, int M, int balanced)
{
    const int tid = threadIdx.x;
    // Lanes per row in proportion to the row's length (round 2).  With a fixed 4 lanes per row the mat-vec of a step took as long as the
    // CTA's longest row (rim rows: 60-100 entries against a median of 20) while most lanes had 5 entries; a row now gets
    // 1, 2, 4, ... 32 consecutive lanes ~ nnz / target, target = the smallest entries-per-lane for which the CTA's rows fit its 512
    // lanes.  Groups are laid out longest first, so every group is aligned to its size and never straddles a warp; the position of a
    // row depends on its rank among the rows of its class only (deterministic: the order in which rows enter the sums is fixed).
    if (!balanced) {                                           // DF_SOLVE_BALANCED=0: the fixed power-of-two lanes per row of round 1
        const int r = tid / tpr_fixed;
        mp.t_rl[tid] = (unsigned short)r; mp.t_sub[tid] = (unsigned char)(tid % tpr_fixed); mp.t_tr[tid] = (unsigned char)(r < rpc ? tpr_fixed : 0);
        __syncthreads();
    } else {
        int my_nnz = 0;
        const bool row_here = tid < rpc && cta * rpc + tid < M;
        if (row_here) my_nnz = ws.rownnz[order ? order[cta * rpc + tid] : cta * rpc + tid];
        if (tid < 2) mp.bal_sum[tid] = 0;
        if (tid < 8) mp.cls_cnt[tid] = 0;
        mp.t_tr[tid] = 0; mp.t_rl[tid] = 0; mp.t_sub[tid] = 0;
        __syncthreads();
        if (row_here) atomicAdd(&mp.bal_sum[0], my_nnz);
        __syncthreads();
        int target = max(1, (mp.bal_sum[0] + LM4_THREADS - 1) / LM4_THREADS);
        int my_t = 0;
        for (int round = 0; round < 40; ++round) {              // block-uniform loop: every thread sees the same sums
            my_t = 0;
            if (row_here) {
                const int want = (my_nnz + target - 1) / target;
                my_t = 1;
                while (my_t < want && my_t < 32) my_t <<= 1;
            }
            __syncthreads();
            if (tid == 0) mp.bal_sum[1] = 0;
            __syncthreads();
            if (my_t) atomicAdd(&mp.bal_sum[1], my_t);
            __syncthreads();
            if (mp.bal_sum[1] <= LM4_THREADS) break;
            target = target + (target >> 2) + 1;
        }
        const int cls = my_t ? 31 - __clz(my_t) : 7;            // 0..5; 7 = no row
        mp.row_cls[tid] = (unsigned char)cls;
        if (my_t) atomicAdd(&mp.cls_cnt[cls], 1);
        __syncthreads();
        if (tid == 0) { int acc = 0; for (int c = 5; c >= 0; --c) { mp.cls_start[c] = acc; acc += mp.cls_cnt[c] << c; } }
        __syncthreads();
        if (my_t) {
            int rank = 0;                                       // rows of my class with a smaller slot index
            for (int j = 0; j < tid; ++j) rank += mp.row_cls[j] == cls;
            const int first = mp.cls_start[cls] + (rank << cls);
            for (int l = 0; l < my_t; ++l) { mp.t_rl[first + l] = (unsigned short)tid; mp.t_sub[first + l] = (unsigned char)l; mp.t_tr[first + l] = (unsigned char)my_t; }
        }
        __syncthreads();
    }
}

template <int NCTA>
struct Lm5Smem {
    double wpart[LM4_THREADS / 32][NCTA];
    double red_in[2][NCTA][NCTA];
    unsigned long long bar_red[2];
    unsigned long long bar_pub;
};

// -DDF_LM_PROFILE (build.py: DF_NVCC_EXTRA): thread-local clock64 accounting of the LM kernel's phases, printed per CTA at exit.
// 0 mat-vec, 1 per-row arithmetic, 2 sum: shuffles + block barrier + sends, 3 sum: wait, 4 sum: final tree, 5 publish: sends, 6 publish: wait
#ifdef DF_LM_PROFILE
#define LMP_MARK(sy, i) do { const long long t_ = clock64(); (sy).t[i] += t_ - (sy).last; (sy).last = t_; } while (0)
struct Lm5Sync { int parity; uint32_t phase_red[2]; uint32_t phase_pub; long long t[8]; long long last; };
#else
#define LMP_MARK(sy, i) do { } while (0)
struct Lm5Sync { int parity; uint32_t phase_red[2]; uint32_t phase_pub; };
#endif

// kOwnerOnly: only the lanes that own a row (lane % tpr == 0) hold a non-zero contribution, so the warp butterfly can stop at
// offset tpr (3 of 5 steps at the usual 4 threads per row).  Profiled: the shuffles of this function were
// a large share of the kernel's instructions and the final 16 x NV serial sum in every thread another; the final sum is now a 16-lane
// butterfly per warp (every warp forms the same tree on the same data: all threads of all CTAs still hold bit-identical totals).
template <int NCTA, int NV, bool kOwnerOnly = false>
__device__ __forceinline__ void cluster_sum5(Lm5Smem<NCTA> &sm, Lm5Sync &sy, int cta, double (&v)[NV], int tpr = 1)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int par = sy.parity;
    const int stop = kOwnerOnly ? tpr : 1;
    LMP_MARK(sy, 1);
#pragma unroll
    for (int k = 0; k < NV; ++k)
        for (int o = 16; o >= stop; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k) sm.wpart[warp][k] = v[k];
    }
    __syncthreads();
    const uint32_t bar = smem_u32(&sm.bar_red[par]);
    if (warp == 0) {
        const uint32_t rbar = mapa_u32(bar, (uint32_t)(lane & (NCTA - 1)));
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            double t = lane < LM4_THREADS / 32 ? sm.wpart[lane][k] : 0.0;
            for (int o = 8; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            if (lane < NCTA) st_async_f64(mapa_u32(smem_u32(&sm.red_in[par][cta][k]), (uint32_t)lane), t, rbar);   // lane = destination CTA
        }
        if (lane == 0) mbar_arrive_expect(bar, (uint32_t)(NCTA * NV * 8));
    }
    LMP_MARK(sy, 2);
    mbar_wait(bar, sy.phase_red[par]);
    LMP_MARK(sy, 3);
    sy.phase_red[par] ^= 1u;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        double t = sm.red_in[par][lane & (NCTA - 1)][k];
#pragma unroll
        for (int o = NCTA / 2; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        v[k] = t;
    }
    sy.parity = par ^ 1;
    LMP_MARK(sy, 4);
}

// NCTA = CTAs per cluster (8, or 16 = the non-portable maximum: half the rows, hence half the shared-memory gather traffic of the
// mat-vec, per SM); the cluster shape is a launch attribute.
template <int NCTA, bool merged>
__global__ void __launch_bounds__(LM4_THREADS, 1)
solve_lm_v5_kernel(float *nodes, int M, const void *grid, SolveWs ws, int nl_iters, int lin_iters, double *stats, int ent_cap, int balanced, int only_if_flag)
{
    DF_PDL_ENTRY();
    if (only_if_flag && ws.flags[1] == 0) return;               // launched behind v6 as its fallback: v6 solved the frame (cluster-uniform)
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ Lm5Smem<NCTA> sm;
    extern __shared__ __align__(16) unsigned char dyn[];
    const Lm4Layout L = lm4_layout(M, ent_cap, NCTA);
    double *svec = reinterpret_cast<double *>(dyn + L.off_svec);          // full-length copy of the multiplied vector, [3 * node + axis]
    double *mval = reinterpret_cast<double *>(dyn + L.off_val);           // [entry][thread]
    unsigned short *mcol = reinterpret_cast<unsigned short *>(dyn + L.off_col);   // 3 * column
    const int rpc = L.rpc;

    Lm5Sync sy; sy.parity = 0; sy.phase_red[0] = sy.phase_red[1] = 0u; sy.phase_pub = 0u;
    const int cta = (int)cluster.block_rank();
    const int tid = threadIdx.x;
    // Rows are dealt to the CTAs in the node grid's Morton order (nodegrid.cu step 5): a CTA's rows are neighbours in space, so
    // most of the columns they touch are the CTA's own rows and a row's search-direction entry is needed by few other CTAs.
    const int *order = grid ? nodegrid_order(grid) : nullptr;
    const int *slot = grid ? nodegrid_slot(grid) : nullptr;
    __shared__ LmRowMap mp;
    lm_map_rows(mp, ws, order, cta, rpc, L.tpr, M, balanced);
    const int tpr = mp.t_tr[tid];                              // lanes serving this thread's row (0: idle lane)
    const int rl = tpr ? (int)mp.t_rl[tid] : rpc, sub = mp.t_sub[tid];
    const int wtpr = __reduce_min_sync(0xffffffffu, tpr ? tpr : 32);   // the warp's smallest group: owner lanes sit at multiples of it
    const int wmax = __reduce_max_sync(0xffffffffu, tpr);             // ... and its largest: the row sums need log2(wmax) shuffle steps
    const int s_row = cta * rpc + rl;                          // slot of this thread's row
    const bool has_row = rl < rpc && s_row < M;
    const int n = has_row ? (order ? order[s_row] : s_row) : 0;   // node index = row/column index of the normal matrix
    const bool owner = has_row && sub == 0;

    const int nnz = has_row ? ws.rownnz[n] : 0;
    int my_ent = 0;
    unsigned need = 0u;                                        // CTAs that own a row coupled to this one (A is structurally symmetric)
    for (int e = sub; e < nnz; e += max(tpr, 1)) {
        const int j = ws.col[(size_t)e * M + n];
        need |= 1u << ((slot ? slot[j] : j) / rpc);
        if (my_ent < ent_cap) {
            mcol[my_ent * LM4_THREADS + tid] = (unsigned short)(3 * j);
            mval[my_ent * LM4_THREADS + tid] = ws.val[(size_t)e * M + n];
            ++my_ent;
        }
    }
    for (int o = wmax >> 1; o > 0; o >>= 1) { const unsigned t = __shfl_xor_sync(0xffffffffu, need, o); if (o < tpr) need |= t; }
    need |= 1u << cta;
    const int e_rest = sub + my_ent * tpr;                     // entries that did not fit are streamed from L2 (rare)
    const double diag_n = has_row ? ws.diag[n] : 0.0;
    double gb0 = 0.0, gb1 = 0.0, gb2 = 0.0;
    if (owner) { gb0 = ws.gb[n]; gb1 = ws.gb[M + n]; gb2 = ws.gb[2 * M + n]; }

    const uint32_t svec_addr = smem_u32(svec), pub_bar = smem_u32(&sm.bar_pub);
    uint32_t pub_bytes = 0;                                    // bytes this CTA receives per exchange (set once below)
    // this row's three values -> the svec of every CTA that multiplies by them; then wait until this CTA's own svec is complete
    auto publish = [&](double a0, double a1, double a2) {
        LMP_MARK(sy, 1);
        if (owner) {
#pragma unroll
            for (int c = 0; c < NCTA; ++c) {
                if (!((need >> c) & 1u)) continue;
                const uint32_t dst = mapa_u32(svec_addr + 24u * (uint32_t)n, (uint32_t)c), rb = mapa_u32(pub_bar, (uint32_t)c);
                st_async_f64(dst, a0, rb); st_async_f64(dst + 8u, a1, rb); st_async_f64(dst + 16u, a2, rb);
            }
        }
        if (tid == 0) mbar_arrive_expect(pub_bar, pub_bytes);
        LMP_MARK(sy, 5);
        mbar_wait(pub_bar, sy.phase_pub);
        LMP_MARK(sy, 6);
        sy.phase_pub ^= 1u;
    };
    auto spmv = [&](double &o0, double &o1, double &o2) {      // (A * svec)[row], valid in the owner lane
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        LMP_MARK(sy, 1);
#pragma unroll 4
        for (int k = 0; k < my_ent; ++k) {
            const double *sv = svec + mcol[k * LM4_THREADS + tid];
            const double a = mval[k * LM4_THREADS + tid];
            a0 += a * sv[0]; a1 += a * sv[1]; a2 += a * sv[2];
        }
        for (int e = e_rest; e < nnz; e += max(tpr, 1)) {
            const double *sv = svec + 3 * __ldg(ws.col + (size_t)e * M + n);
            const double a = __ldg(ws.val + (size_t)e * M + n);
            a0 += a * sv[0]; a1 += a * sv[1]; a2 += a * sv[2];
        }
        for (int o = wmax >> 1; o > 0; o >>= 1) {              // group sizes differ inside a warp: everybody shuffles, a lane adds what is in its group
            const double b0 = __shfl_xor_sync(0xffffffffu, a0, o), b1 = __shfl_xor_sync(0xffffffffu, a1, o), b2 = __shfl_xor_sync(0xffffffffu, a2, o);
            if (o < tpr) { a0 += b0; a1 += b1; a2 += b2; }
        }
        o0 = a0; o1 = a1; o2 = a2;
        LMP_MARK(sy, 0);
    };

    // x0 = current node translations (CombinedSolver.h:165-172)
    double x0 = 0.0, x1 = 0.0, x2 = 0.0;
    if (owner) {
        const float4 *n4 = reinterpret_cast<const float4 *>(nodes + (size_t)n * DF_NODE_STRIDE);
        const float4 a = n4[0], b = n4[1], c = n4[2];
        const Quat t = dq_translation(Quat{a.w, b.x, b.y, b.z}, Quat{b.w, c.x, c.y, c.z});
        x0 = t.x; x1 = t.y; x2 = t.z;
    }
    const int T = NCTA * LM4_THREADS, gt = cta * LM4_THREADS + tid;
    double c0n[3] = {0.0, 0.0, 0.0};
    for (int i = gt; i < ws.prepare_blocks * (PREPARE_THREADS / 32); i += T) { c0n[0] += ws.c0_partials[2 * i]; c0n[1] += ws.c0_partials[2 * i + 1]; }
    c0n[2] = (owner ? (double)nnz : 0.0);
    if (tid == 0) {
        mbar_init(smem_u32(&sm.bar_red[0]), 1u); mbar_init(smem_u32(&sm.bar_red[1]), 1u); mbar_init(pub_bar, 1u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    cluster.sync();                                            // every CTA is running, its barriers are initialised
    {   // how many rows will send to me: all-reduce of the per-destination row counts
        double cnt[NCTA];
#pragma unroll
        for (int c = 0; c < NCTA; ++c) cnt[c] = (owner && ((need >> c) & 1u)) ? 1.0 : 0.0;
        cluster_sum5<NCTA>(sm, sy, cta, cnt);
        double mine = 0.0;
#pragma unroll
        for (int c = 0; c < NCTA; ++c) if (c == cta) mine = cnt[c];
        pub_bytes = 24u * (uint32_t)mine;
    }
    publish(x0, x1, x2);
    cluster_sum5<NCTA>(sm, sy, cta, c0n);
    const double nvalid = c0n[1], nnz_total = c0n[2];
    double Ap0, Ap1, Ap2;
    spmv(Ap0, Ap1, Ap2);
    double t0[1] = {0.0};
    if (owner) {
        t0[0] += x0 * (0.5 * Ap0 - gb0);
        t0[0] += x1 * (0.5 * Ap1 - gb1);
        t0[0] += x2 * (0.5 * Ap2 - gb2);
    }
    cluster_sum5<NCTA, sizeof(t0) / sizeof(double), true>(sm, sy, cta, t0, wtpr);
    double cost = c0n[0] + t0[0];
    const double cost0 = cost;

    double radius = 1e4, decrease = 2.0;                       // solverGPUGaussNewton.t:26-39
    int it = 0, pcg_total = 0;
#ifdef DF_LM_PROFILE
    for (int i = 0; i < 8; ++i) sy.t[i] = 0;
    sy.last = clock64();
    const long long lmp_begin = sy.last;
#endif
    const bool overflow = ws.flags[0] != 0;                    // a row overflowed (solve_rows): the stored system is truncated -> leave the field
    if (overflow) nl_iters = 0;                                // unchanged (not even re-encoded), stats[5] says so
    for (; it < nl_iters; ++it) {
        spmv(Ap0, Ap1, Ap2);                                   // svec holds x here
        double rzv[1] = {0.0};
        double cdn = 0.0, mi = 0.0;
        double g0 = 0.0, g1 = 0.0, g2 = 0.0, dl0 = 0.0, dl1 = 0.0, dl2 = 0.0, r0 = 0.0, r1 = 0.0, r2 = 0.0, p0 = 0.0, p1 = 0.0, p2 = 0.0;
        if (owner) {
            cdn = fmin(fmax(diag_n, 1e-6), 1e32) / radius;
            mi = 1.0 / (diag_n + cdn);
            g0 = gb0 - Ap0; g1 = gb1 - Ap1; g2 = gb2 - Ap2;
            r0 = g0; r1 = g1; r2 = g2;
            p0 = g0 * mi; p1 = g1 * mi; p2 = g2 * mi;
            rzv[0] += g0 * p0; rzv[0] += g1 * p1; rzv[0] += g2 * p2;
        }
        cluster_sum5<NCTA, sizeof(rzv) / sizeof(double), true>(sm, sy, cta, rzv, wtpr);                        // completes only when every CTA has finished reading svec (x) ...
        publish(p0, p1, p2);                                   // ... so p may overwrite it
        double rz = rzv[0];
        double Q0 = 0.0;
        // One cluster-wide reduction per PCG step instead of two (DF_SOLVE_MERGED, default on).  The second reduction of the textbook
        // step only exists because r.z and the model value Q are formed AFTER alpha is known.  Both follow from sums that do not need
        // alpha:   r' = r - alpha Ap,  z' = M r'   =>   r'.z' = r.Mr - 2 alpha (r.M Ap) + alpha^2 (Ap.M Ap)
        //          Q(d + alpha p) = Q(d) - alpha p.r + alpha^2/2 p.Ap = Q(d) - alpha/2 (r.Mr)      (p.r = r.z, alpha = r.z / p.Ap)
        // so p.Ap, r.Mr, r.MAp and Ap.MAp are summed in ONE exchange, after which every CTA knows alpha, beta and Q and updates its
        // rows: the iterates are the textbook ones up to rounding (r.Mr is re-measured every step: nothing drifts), with two DSMEM
        // round trips per step (sum, publish) instead of three.
        for (int l = 0; merged && l < lin_iters && rz > 0.0; ++l) {
            spmv(Ap0, Ap1, Ap2);
            double v[4] = {0.0, 0.0, 0.0, 0.0};
            if (owner) {
                double m, n;
                Ap0 = Ap0 + cdn * p0; m = mi * r0; n = mi * Ap0; v[0] += p0 * Ap0; v[1] += m * r0; v[2] += m * Ap0; v[3] += n * Ap0;
                Ap1 = Ap1 + cdn * p1; m = mi * r1; n = mi * Ap1; v[0] += p1 * Ap1; v[1] += m * r1; v[2] += m * Ap1; v[3] += n * Ap1;
                Ap2 = Ap2 + cdn * p2; m = mi * r2; n = mi * Ap2; v[0] += p2 * Ap2; v[1] += m * r2; v[2] += m * Ap2; v[3] += n * Ap2;
            }
            cluster_sum5<NCTA, sizeof(v) / sizeof(double), true>(sm, sy, cta, v, wtpr);                      // every CTA finished reading svec (p)
            if (!(v[0] > 0.0) || !(v[1] > 0.0)) break;
            const double rz_now = v[1];
            const double alpha = rz_now / v[0];
            const double rz_new = rz_now - 2.0 * alpha * v[2] + alpha * alpha * v[3];
            const double Q1 = Q0 - 0.5 * alpha * rz_now;
            const double beta = rz_new / rz_now;
            if (owner) {
                dl0 = dl0 + alpha * p0; r0 = r0 - alpha * Ap0; p0 = r0 * mi + beta * p0;
                dl1 = dl1 + alpha * p1; r1 = r1 - alpha * Ap1; p1 = r1 * mi + beta * p1;
                dl2 = dl2 + alpha * p2; r2 = r2 - alpha * Ap2; p2 = r2 * mi + beta * p2;
            }
            rz = rz_new;
            ++pcg_total;
            const double zeta = (double)(l + 1) * (Q1 - Q0) / Q1;   // Ceres/Opt q-tolerance, solverGPUGaussNewton.t:1093-1101
            Q0 = Q1;
            publish(p0, p1, p2);
            if (zeta < 1e-4) break;
        }
        for (int l = 0; !merged && l < lin_iters && rz > 0.0; ++l) {
            spmv(Ap0, Ap1, Ap2);
            double pap[1] = {0.0};
            if (owner) {
                Ap0 = Ap0 + cdn * p0; Ap1 = Ap1 + cdn * p1; Ap2 = Ap2 + cdn * p2;
                pap[0] += p0 * Ap0; pap[0] += p1 * Ap1; pap[0] += p2 * Ap2;
            }
            cluster_sum5<NCTA, sizeof(pap) / sizeof(double), true>(sm, sy, cta, pap, wtpr);                    // every CTA finished reading svec (p)
            if (!(pap[0] > 0.0)) break;
            const double alpha = rz / pap[0];
            double rq[2] = {0.0, 0.0};
            double z0 = 0.0, z1 = 0.0, z2 = 0.0;
            if (owner) {
                dl0 = dl0 + alpha * p0; r0 = r0 - alpha * Ap0; z0 = r0 * mi; rq[0] += r0 * z0; rq[1] += dl0 * (r0 + g0);
                dl1 = dl1 + alpha * p1; r1 = r1 - alpha * Ap1; z1 = r1 * mi; rq[0] += r1 * z1; rq[1] += dl1 * (r1 + g1);
                dl2 = dl2 + alpha * p2; r2 = r2 - alpha * Ap2; z2 = r2 * mi; rq[0] += r2 * z2; rq[1] += dl2 * (r2 + g2);
            }
            cluster_sum5<NCTA, sizeof(rq) / sizeof(double), true>(sm, sy, cta, rq, wtpr);
            const double rz_new = rq[0], Q1 = -0.5 * rq[1];
            const double beta = rz_new / rz;
            if (owner) { p0 = z0 + beta * p0; p1 = z1 + beta * p1; p2 = z2 + beta * p2; }
            rz = rz_new;
            ++pcg_total;
            const double zeta = (double)(l + 1) * (Q1 - Q0) / Q1;   // Ceres/Opt q-tolerance, solverGPUGaussNewton.t:1093-1101
            Q0 = Q1;
            publish(p0, p1, p2);
            if (zeta < 1e-4) break;
        }
        // model change = 0.5 dl.(g + r + C dl);  A dl = g - r - C dl  => new cost = cost - dl.g + 0.5 dl.(A dl)
        double mad[3] = {0.0, 0.0, 0.0};
        if (owner) {
            double c;
            c = cdn * dl0; mad[0] += dl0 * (g0 + r0 + c); mad[1] += dl0 * (g0 - r0 - c); mad[2] += dl0 * g0;
            c = cdn * dl1; mad[0] += dl1 * (g1 + r1 + c); mad[1] += dl1 * (g1 - r1 - c); mad[2] += dl1 * g1;
            c = cdn * dl2; mad[0] += dl2 * (g2 + r2 + c); mad[1] += dl2 * (g2 - r2 - c); mad[2] += dl2 * g2;
        }
        cluster_sum5<NCTA, sizeof(mad) / sizeof(double), true>(sm, sy, cta, mad, wtpr);
        const double model = 0.5 * mad[0];
        const double new_cost = cost - mad[2] + 0.5 * mad[1];
        const double change = cost - new_cost;
        const double rho = model > 0.0 ? change / model : 0.0;
        bool stop = false;
        if (change >= 0.0 && rho > 1e-3) {
            if (owner) { x0 += dl0; x1 += dl1; x2 += dl2; }
            stop = change <= cost * 1e-6;                       // function_tolerance, CombinedSolver.h:88
            cost = new_cost;
            const double f = 1.0 - (2.0 * rho - 1.0) * (2.0 * rho - 1.0) * (2.0 * rho - 1.0);
            radius /= fmax(f, 1.0 / 3.0);
            radius = fmin(radius, 1e16);
            decrease = 2.0;
        } else {
            radius /= decrease; decrease *= 2.0;
            if (radius <= 1e-32) stop = true;
        }
        if (stop) { ++it; break; }
        publish(x0, x1, x2);                                   // svec <- x for the next linearisation (the mad reduction proves nobody reads p any more)
    }
#ifdef DF_LM_PROFILE
    LMP_MARK(sy, 1);
    if ((tid == 0 || tid == LM4_THREADS - 1) && (cta == 0 || cta == NCTA - 1 || cta == NCTA / 2))
        printf("LMP cta %d tid %d my_ent %d tpr %d steps %d total %lld | spmv %lld arith %lld sum_send %lld sum_wait %lld sum_tree %lld pub_send %lld pub_wait %lld\n",
               cta, tid, my_ent, tpr, pcg_total, clock64() - lmp_begin, sy.t[0], sy.t[1], sy.t[2], sy.t[3], sy.t[4], sy.t[5], sy.t[6]);
#endif
    cluster.sync();                                            // no CTA may exit while others can still write into its shared memory
    // write back: encodeTranslation (CombinedSolver.h:189-197, dual_quaternion.hpp:82-85)
    if (owner && !overflow) {
        float *nd = nodes + (size_t)n * DF_NODE_STRIDE;
        const Quat rot = {nd[3], nd[4], nd[5], nd[6]};
        const Quat h = qhalf(Quat{0.f, (float)x0, (float)x1, (float)x2});
        const Quat d = qmul(h, rot);
        nd[7] = d.w; nd[8] = d.x; nd[9] = d.y; nd[10] = d.z;
    }
    if (gt == 0 && stats) {
        stats[0] = cost0; stats[1] = cost; stats[2] = (double)it; stats[3] = nvalid; stats[4] = (double)pcg_total; stats[5] = (double)ws.flags[0];
        stats[6] = nnz_total; stats[7] = (ws.flags[3] && !ws.flags[2]) ? -0.5 : -1.0;   // < 0: solved by v5; -0.5: matrix from the tile records
    }
}

// ------------------------------------------------------------------------------------------------------------------
// v6 (round 2, default): ONE DSMEM exchange per PCG step.
//
// clock64 accounting of v5 (tools/build_variant.py lmprof): the two mbarrier waits are a small part of a step; the rest is
// issue/latency inside the CTA -- the gather of the mat-vec (random 24-byte reads of shared memory, bank conflicts), four
// cluster-wide sums with three shuffle trees each and the per-row st.async loop of the vector exchange.  A CTA's step is a serial chain on 4 warps per scheduler; what shortens it is
// fewer links, not faster links:
//   * Chronopoulos-Gear form of the preconditioned CG step: with u = M r and w = (A + C) u the step needs only gamma = r.u and
//     delta = w.u (beta = gamma/gamma', alpha = gamma / (delta - beta gamma / alpha'), p = u + beta p, s = w + beta s, x += alpha p,
//     r -= alpha s): TWO sums per step instead of four, formed in one exchange, and the same iterates as the textbook step in exact
//     arithmetic (the model value Q for the q-tolerance follows from Q' = Q - alpha gamma / 2 as before);
//   * the exchange of the multiplied vector rides on the same exchange: a row's owner sends w_j to the CTAs that multiply by column j
//     TOGETHER with its CTA's partial sums; every CTA keeps (r_j, s_j, 1/M_jj) of its halo columns and, once alpha and beta are
//     known, advances them with the very operations the owner applies -- bit-identical replicas, no second round trip;
//   * the sends come from a flat (row, destination) list walked by all 512 threads (no predicated loop over 16 CTAs per owner lane).
// A step is: mat-vec -> partial sums + halo sends -> ONE wait -> scalars -> update of own + halo rows -> block barrier.
// Set-up finds a CTA's halo (bitmap of the columns its rows touch), ranks it, and lets every owner look up its rows' positions in the
// destination CTAs' halos through DSMEM loads; both sides verify the other's view (A is structurally symmetric), and a system whose
// halo or send list does not fit -- or any mismatch -- raises ws.flags[1] and leaves the solve to v5 (launched right behind, a no-op
// otherwise).
constexpr int LM6_HALO = 512;      // halo columns per CTA (one per thread)
constexpr int LM6_SEND = 1536;     // (row, destination) pairs per CTA
constexpr int LM6_BITW = 128;      // bitmap words: M <= 4096

struct Lm6Layout {
    int rpc, tpr, ent_cap;
    size_t off_svec, off_win, off_hr, off_hs, off_hdiag, off_hmi, off_hj, off_wown, off_need, off_srl, off_sdst, off_sbar, off_val, off_col, total;
};

__host__ __device__ inline Lm6Layout lm6_layout(int M, int ent_cap, int ncta)
{
    Lm6Layout L;
    L.rpc = (M + ncta - 1) / ncta;
    L.tpr = 1;
    while (L.tpr < 32 && L.tpr * 2 * L.rpc <= LM4_THREADS) L.tpr *= 2;
    L.ent_cap = ent_cap;
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 15) & ~(size_t)15; return at; };
    L.off_svec = take((size_t)3 * M * 8);
    L.off_win = take((size_t)2 * LM6_HALO * 3 * 8);
    L.off_hr = take((size_t)LM6_HALO * 3 * 8);
    L.off_hs = take((size_t)LM6_HALO * 3 * 8);
    L.off_hdiag = take((size_t)LM6_HALO * 8);
    L.off_hmi = take((size_t)LM6_HALO * 8);
    L.off_hj = take((size_t)LM6_HALO * 4);
    L.off_wown = take((size_t)L.rpc * 3 * 8);
    L.off_need = take((size_t)L.rpc * 4);
    L.off_srl = take((size_t)LM6_SEND * 2);
    L.off_sdst = take((size_t)LM6_SEND * 4);
    L.off_sbar = take((size_t)LM6_SEND * 4);
    L.off_val = take((size_t)ent_cap * LM4_THREADS * 8);
    L.off_col = take((size_t)ent_cap * LM4_THREADS * 2);
    L.total = o;
    return L;
}

template <int NCTA>
struct Lm6Smem {
    double wpart[LM4_THREADS / 32][4];
    double red_in[2][NCTA][4];
    unsigned long long bar[2];
    unsigned refbits[LM6_BITW];      // columns this CTA's rows touch, then: its halo (columns owned by other CTAs)
    int haloprefix[LM6_BITW];        // halo columns below word w
    int scan[LM4_THREADS / 32 + 1];
    int H, nsend, bad;
};

struct Lm6Sync { int parity; uint32_t phase[2]; };

struct Lm6Ctx {
    int cta, H, nsend;
    const double *wown;
    const unsigned short *send_rl;
    const uint32_t *send_dst, *send_bar;
};

__device__ __forceinline__ uint32_t ld_cluster_u32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}

// One exchange: cluster-wide sums of v[0..NV) (every thread of every CTA ends up with bit-identical totals: fixed trees) and, with
// kHalo, the three doubles the owner lanes put into wown[] go to the halos that hold their rows (w_in[parity] over there).
// Returns the parity (= which w_in / red_in buffer the data of this exchange sits in).  Buffers and barriers alternate: a CTA can be
// one exchange ahead of another, never two (its next wait needs everybody's partial sums of this one).
template <int NCTA, int NV, bool kHalo>
__device__ __forceinline__ int lm6_exchange(Lm6Smem<NCTA> &sm, Lm6Sync &sy, const Lm6Ctx &cx, double (&v)[NV], int wtpr)
{
    static_assert(NV >= 1 && NV <= 4, "partial-sum slots");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int par = sy.parity;
#pragma unroll
    for (int k = 0; k < NV; ++k)
        for (int o = 16; o >= wtpr; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k) sm.wpart[warp][k] = v[k];
    }
    __syncthreads();                                           // wpart and wown are complete
    const uint32_t bar = smem_u32(&sm.bar[par]);
    if (warp == 0) {
        const uint32_t rbar = mapa_u32(bar, (uint32_t)(lane & (NCTA - 1)));
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            double t = lane < LM4_THREADS / 32 ? sm.wpart[lane][k] : 0.0;
            for (int o = 8; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            if (lane < NCTA) st_async_f64(mapa_u32(smem_u32(&sm.red_in[par][cx.cta][k]), (uint32_t)lane), t, rbar);   // lane = destination CTA
        }
    }
    if (kHalo) {
        const uint32_t dpar = par ? (uint32_t)(LM6_HALO * 24) : 0u, bpar = par ? 8u : 0u;
        for (int i = tid; i < cx.nsend; i += LM4_THREADS) {
            const double *src = cx.wown + 3 * (int)cx.send_rl[i];
            const uint32_t dst = cx.send_dst[i] + dpar, rb = cx.send_bar[i] + bpar;
            st_async_f64(dst, src[0], rb); st_async_f64(dst + 8u, src[1], rb); st_async_f64(dst + 16u, src[2], rb);
        }
    }
    if (tid == 0) mbar_arrive_expect(bar, (uint32_t)(NCTA * NV * 8 + (kHalo ? 24 * cx.H : 0)));
    mbar_wait(bar, sy.phase[par]);
    sy.phase[par] ^= 1u;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        double t = sm.red_in[par][lane & (NCTA - 1)][k];
#pragma unroll
        for (int o = NCTA / 2; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        v[k] = t;
    }
    sy.parity = par ^ 1;
    return par;
}

template <int NCTA>
__global__ void __launch_bounds__(LM4_THREADS, 1)
solve_lm_v6_kernel(float *nodes, int M, const void *grid, SolveWs ws, int nl_iters, int lin_iters, double *stats, int ent_cap, int balanced)
{
    DF_PDL_ENTRY();
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ Lm6Smem<NCTA> sm;
    __shared__ LmRowMap mp;
    extern __shared__ __align__(16) unsigned char dyn[];
    const Lm6Layout L = lm6_layout(M, ent_cap, NCTA);
    double *svec = reinterpret_cast<double *>(dyn + L.off_svec);          // the multiplied vector, [3 * node + axis]: own rows + halo columns
    double *w_in = reinterpret_cast<double *>(dyn + L.off_win);           // [parity][halo slot][3]: what the owners sent
    double *hr = reinterpret_cast<double *>(dyn + L.off_hr);              // replicas of the halo columns' residual ...
    double *hs = reinterpret_cast<double *>(dyn + L.off_hs);              // ... and A-conjugate direction
    double *hdiag = reinterpret_cast<double *>(dyn + L.off_hdiag);
    double *hmi = reinterpret_cast<double *>(dyn + L.off_hmi);
    int *hj = reinterpret_cast<int *>(dyn + L.off_hj);                    // halo slot -> node index
    double *wown = reinterpret_cast<double *>(dyn + L.off_wown);          // [local row][3]: what this CTA's rows send
    unsigned *needmask = reinterpret_cast<unsigned *>(dyn + L.off_need);  // [local row]: CTAs whose rows couple to it
    unsigned short *send_rl = reinterpret_cast<unsigned short *>(dyn + L.off_srl);
    uint32_t *send_dst = reinterpret_cast<uint32_t *>(dyn + L.off_sdst);
    uint32_t *send_bar = reinterpret_cast<uint32_t *>(dyn + L.off_sbar);
    double *mval = reinterpret_cast<double *>(dyn + L.off_val);           // [entry][thread]
    unsigned short *mcol = reinterpret_cast<unsigned short *>(dyn + L.off_col);   // 3 * column
    const int rpc = L.rpc;

    Lm6Sync sy; sy.parity = 0; sy.phase[0] = sy.phase[1] = 0u;
    const int cta = (int)cluster.block_rank();
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int *order = grid ? nodegrid_order(grid) : nullptr;
    const int *slot = grid ? nodegrid_slot(grid) : nullptr;
    if (tid == 0) {
        mbar_init(smem_u32(&sm.bar[0]), 1u); mbar_init(smem_u32(&sm.bar[1]), 1u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        sm.bad = 0;
    }
    for (int w = tid; w < LM6_BITW; w += LM4_THREADS) sm.refbits[w] = 0u;
    for (int r = tid; r < rpc; r += LM4_THREADS) needmask[r] = 0u;
    const bool force_fallback = (balanced & 2) != 0;            // DF_SOLVE_V6_FORCE_FALLBACK (tests): behave as if the set-up had not fitted
    lm_map_rows(mp, ws, order, cta, rpc, L.tpr, M, balanced & 1);   // (ends with a block barrier)
    const int tpr = mp.t_tr[tid];
    const int rl = tpr ? (int)mp.t_rl[tid] : rpc, sub = mp.t_sub[tid];
    const int wtpr = __reduce_min_sync(0xffffffffu, tpr ? tpr : 32);
    const int wmax = __reduce_max_sync(0xffffffffu, tpr);
    const int s_row = cta * rpc + rl;
    const bool has_row = rl < rpc && s_row < M;
    const int n = has_row ? (order ? order[s_row] : s_row) : 0;
    const bool owner = has_row && sub == 0;

    const int nnz = has_row ? ws.rownnz[n] : 0;
    int my_ent = 0;
    unsigned need = 0u;
    for (int e = sub; e < nnz; e += max(tpr, 1)) {
        const int j = ws.col[(size_t)e * M + n];
        need |= 1u << ((slot ? slot[j] : j) / rpc);
        atomicOr(&sm.refbits[j >> 5], 1u << (j & 31));
        if (my_ent < ent_cap) {
            mcol[my_ent * LM4_THREADS + tid] = (unsigned short)(3 * j);
            mval[my_ent * LM4_THREADS + tid] = ws.val[(size_t)e * M + n];
            ++my_ent;
        }
    }
    for (int o = wmax >> 1; o > 0; o >>= 1) { const unsigned t = __shfl_xor_sync(0xffffffffu, need, o); if (o < tpr) need |= t; }
    need &= ~(1u << cta);                                      // remote CTAs only
    if (owner) needmask[rl] = need;
    const int e_rest = sub + my_ent * tpr;
    const double diag_n = has_row ? ws.diag[n] : 0.0;
    double gb0 = 0.0, gb1 = 0.0, gb2 = 0.0;
    if (owner) { gb0 = ws.gb[n]; gb1 = ws.gb[M + n]; gb2 = ws.gb[2 * M + n]; }
    __syncthreads();

    // ---- the halo: touched columns that belong to other CTAs, ranked by node index
    const int words = (M + 31) >> 5;
    int hcount = 0;
    if (tid < words) {
        unsigned bits = sm.refbits[tid];
        for (unsigned m = bits; m; m &= m - 1u) {
            const int j = 32 * tid + (__ffs(m) - 1);
            if (((slot ? slot[j] : j) / rpc) == cta) bits &= ~(1u << (j & 31));
        }
        sm.refbits[tid] = bits;
        hcount = __popc(bits);
    }
    {   // exclusive prefix of hcount over the first `words` threads (words <= 128: four warps)
        int inc = hcount;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) sm.scan[warp] = inc;
        __syncthreads();
        if (tid == 0) { int acc = 0; for (int w = 0; w < LM4_THREADS / 32; ++w) { const int c = sm.scan[w]; sm.scan[w] = acc; acc += c; } sm.scan[LM4_THREADS / 32] = acc; }
        __syncthreads();
        const int excl = sm.scan[warp] + inc - hcount;
        if (tid < words) sm.haloprefix[tid] = excl;
        if (tid == 0) { sm.H = sm.scan[LM4_THREADS / 32]; if (sm.H > LM6_HALO) sm.bad = 1; }
        if (tid < words) {
            int h = excl;
            for (unsigned m = sm.refbits[tid]; m; m &= m - 1u, ++h) {
                const int j = 32 * tid + (__ffs(m) - 1);
                if (h < LM6_HALO) { hj[h] = j; hdiag[h] = ws.diag[j]; }
            }
        }
    }
    cluster.sync();                                            // barriers initialised, halo tables and need masks readable by the peers
    const int H = min(sm.H, LM6_HALO);

    // ---- the send list: for every row and every remote CTA that multiplies by it, where its values go over there
    const int ndst = owner ? __popc(need) : 0;
    int send_at = 0, nsend = 0;
    {
        int inc = ndst;
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) sm.scan[warp] = inc;
        __syncthreads();
        if (tid == 0) { int acc = 0; for (int w = 0; w < LM4_THREADS / 32; ++w) { const int c = sm.scan[w]; sm.scan[w] = acc; acc += c; } sm.scan[LM4_THREADS / 32] = acc; }
        __syncthreads();
        send_at = sm.scan[warp] + inc - ndst;
        nsend = sm.scan[LM4_THREADS / 32];
    }
    bool bad = nsend > LM6_SEND || force_fallback;
    if (owner && !bad) {
        int at = send_at;
        for (unsigned m = need; m; m &= m - 1u, ++at) {
            const uint32_t c = (uint32_t)(__ffs(m) - 1);
            const uint32_t bits = ld_cluster_u32(mapa_u32(smem_u32(&sm.refbits[n >> 5]), c));
            const uint32_t pre = ld_cluster_u32(mapa_u32(smem_u32(&sm.haloprefix[n >> 5]), c));
            if (!((bits >> (n & 31)) & 1u)) bad = true;         // the peer does not list this row: structure not symmetric
            const uint32_t h = pre + (uint32_t)__popc(bits & ((1u << (n & 31)) - 1u));
            send_rl[at] = (unsigned short)rl;
            send_dst[at] = mapa_u32(smem_u32(w_in + 3 * min(h, (uint32_t)(LM6_HALO - 1))), c);
            send_bar[at] = mapa_u32(smem_u32(&sm.bar[0]), c);
        }
    }
    // ... and the other direction: every halo column's owner must list this CTA
    for (int h = tid; h < H; h += LM4_THREADS) {
        const int sl = slot ? slot[hj[h]] : hj[h];
        const uint32_t o = (uint32_t)(sl / rpc);
        const uint32_t nm = ld_cluster_u32(mapa_u32(smem_u32(&needmask[sl - (int)o * rpc]), o));
        if (!((nm >> cta) & 1u)) bad = true;
    }
    if (bad) sm.bad = 1;                                       // benign race: everybody writes 1
    __syncthreads();
    Lm6Ctx cx; cx.cta = cta; cx.H = H; cx.nsend = min(nsend, LM6_SEND); cx.wown = wown; cx.send_rl = send_rl; cx.send_dst = send_dst; cx.send_bar = send_bar;

    // first exchange: does the set-up hold everywhere?  (+ the constant part of the cost, the row count, the non-zero count)
    const int T = NCTA * LM4_THREADS, gt = cta * LM4_THREADS + tid;
    double c0n[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = gt; i < ws.prepare_blocks * (PREPARE_THREADS / 32); i += T) { c0n[0] += ws.c0_partials[2 * i]; c0n[1] += ws.c0_partials[2 * i + 1]; }
    c0n[2] = (owner ? (double)nnz : 0.0);
    c0n[3] = (tid == 0 && sm.bad) ? 1.0 : 0.0;
    lm6_exchange<NCTA, 4, false>(sm, sy, cx, c0n, 1);
    const double nvalid = c0n[1], nnz_total = c0n[2];
    const bool overflow = ws.flags[0] != 0;                    // a row overflowed (solve_rows): the stored system is truncated -> leave the field
    if (c0n[3] > 0.0) {                                        // cluster-uniform: hand the frame to v5
        if (gt == 0) ws.flags[1] = 1;
        cluster.sync();
        return;
    }
    int hmax_i = 0;
    {
        double hm[1] = {0.0};
        // max over the CTAs through a sum of one-hot-free values is not available: report this CTA's halo from CTA 0 and the total
        hm[0] = tid == 0 ? (double)H : 0.0;
        lm6_exchange<NCTA, 1, false>(sm, sy, cx, hm, 1);
        hmax_i = (int)hm[0];                                   // total halo columns of the cluster
    }

    auto spmv = [&](double &o0, double &o1, double &o2) {      // (A * svec)[row], valid in the owner lane
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll 4
        for (int k = 0; k < my_ent; ++k) {
            const double *sv = svec + mcol[k * LM4_THREADS + tid];
            const double a = mval[k * LM4_THREADS + tid];
            a0 += a * sv[0]; a1 += a * sv[1]; a2 += a * sv[2];   // (contracted multiply-adds measured: no gain)
        }
        for (int e = e_rest; e < nnz; e += max(tpr, 1)) {
            const double *sv = svec + 3 * __ldg(ws.col + (size_t)e * M + n);
            const double a = __ldg(ws.val + (size_t)e * M + n);
            a0 += a * sv[0]; a1 += a * sv[1]; a2 += a * sv[2];
        }
        for (int o = wmax >> 1; o > 0; o >>= 1) {
            const double b0 = __shfl_xor_sync(0xffffffffu, a0, o), b1 = __shfl_xor_sync(0xffffffffu, a1, o), b2 = __shfl_xor_sync(0xffffffffu, a2, o);
            if (o < tpr) { a0 += b0; a1 += b1; a2 += b2; }
        }
        o0 = a0; o1 = a1; o2 = a2;
    };

    // x0 = current node translations (CombinedSolver.h:165-172)
    double x0 = 0.0, x1 = 0.0, x2 = 0.0;
    if (owner) {
        const float4 *n4 = reinterpret_cast<const float4 *>(nodes + (size_t)n * DF_NODE_STRIDE);
        const float4 a = n4[0], b = n4[1], c = n4[2];
        const Quat t = dq_translation(Quat{a.w, b.x, b.y, b.z}, Quat{b.w, c.x, c.y, c.z});
        x0 = t.x; x1 = t.y; x2 = t.z;
    }
    double cost = 0.0, cost0 = 0.0;
    double radius = 1e4, decrease = 2.0;                       // solverGPUGaussNewton.t:26-39
    int it = 0, pcg_total = 0;
    if (overflow) nl_iters = 0;                                // unchanged (not even re-encoded), stats[5] says so
    for (; it < nl_iters; ++it) {
        // svec <- x (own rows directly, halo columns from their owners)
        if (owner) { wown[3 * rl] = x0; wown[3 * rl + 1] = x1; wown[3 * rl + 2] = x2; svec[3 * n] = x0; svec[3 * n + 1] = x1; svec[3 * n + 2] = x2; }
        {
            double z[1] = {0.0};
            const int par = lm6_exchange<NCTA, 1, true>(sm, sy, cx, z, 1);
            for (int h = tid; h < H; h += LM4_THREADS) {
                const double *wi = w_in + (par * LM6_HALO + h) * 3;
                double *sv = svec + 3 * hj[h];
                sv[0] = wi[0]; sv[1] = wi[1]; sv[2] = wi[2];
            }
        }
        __syncthreads();
        double Ap0, Ap1, Ap2;
        spmv(Ap0, Ap1, Ap2);
        double cdn = 0.0, mi = 0.0;
        double g0 = 0.0, g1 = 0.0, g2 = 0.0, dl0 = 0.0, dl1 = 0.0, dl2 = 0.0, r0 = 0.0, r1 = 0.0, r2 = 0.0, p0 = 0.0, p1 = 0.0, p2 = 0.0;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, u0 = 0.0, u1 = 0.0, u2 = 0.0;
        double t0[1] = {0.0};
        if (owner) {
            cdn = fmin(fmax(diag_n, 1e-6), 1e32) / radius;
            mi = 1.0 / (diag_n + cdn);
            g0 = gb0 - Ap0; g1 = gb1 - Ap1; g2 = gb2 - Ap2;
            r0 = g0; r1 = g1; r2 = g2;
            u0 = g0 * mi; u1 = g1 * mi; u2 = g2 * mi;
            t0[0] += x0 * (0.5 * Ap0 - gb0);
            t0[0] += x1 * (0.5 * Ap1 - gb1);
            t0[0] += x2 * (0.5 * Ap2 - gb2);
            wown[3 * rl] = g0; wown[3 * rl + 1] = g1; wown[3 * rl + 2] = g2;
        }
        {   // gradient -> the halos (replicas start as r = g, s = 0, u = M g); everybody finished reading svec (x) when this completes
            const int par = lm6_exchange<NCTA, 1, true>(sm, sy, cx, t0, wtpr);
            if (it == 0) { cost = c0n[0] + t0[0]; cost0 = cost; }
            if (owner) { svec[3 * n] = u0; svec[3 * n + 1] = u1; svec[3 * n + 2] = u2; }
            for (int h = tid; h < H; h += LM4_THREADS) {
                const double *wi = w_in + (par * LM6_HALO + h) * 3;
                const double d = hdiag[h];
                const double m = 1.0 / (d + fmin(fmax(d, 1e-6), 1e32) / radius);
                hmi[h] = m;
                double *sv = svec + 3 * hj[h];
#pragma unroll
                for (int c = 0; c < 3; ++c) { const double gj = wi[c]; hr[3 * h + c] = gj; hs[3 * h + c] = 0.0; sv[c] = gj * m; }
            }
        }
        __syncthreads();
        double Q0 = 0.0, inv_gamma_prev = 0.0, inv_alpha_prev = 0.0;
        for (int l = 0; l < lin_iters; ++l) {
            spmv(Ap0, Ap1, Ap2);                               // svec holds u = M r
            double v[2] = {0.0, 0.0};
            double w0 = 0.0, w1 = 0.0, w2 = 0.0;
            if (owner) {
                w0 = Ap0 + cdn * u0; w1 = Ap1 + cdn * u1; w2 = Ap2 + cdn * u2;
                v[0] += r0 * u0; v[0] += r1 * u1; v[0] += r2 * u2;
                v[1] += w0 * u0; v[1] += w1 * u1; v[1] += w2 * u2;
                wown[3 * rl] = w0; wown[3 * rl + 1] = w1; wown[3 * rl + 2] = w2;
            }
            const int par = lm6_exchange<NCTA, 2, true>(sm, sy, cx, v, wtpr);
            const double gamma = v[0], delta = v[1];
            if (!(gamma > 0.0)) break;
            // every thread of the cluster waits for these scalars: ONE double division (a ~150-cycle dependent chain) on the path from the
            // sums to alpha instead of three -- 1 / gamma and 1 / alpha of the previous step were formed next to its own division
            const double beta = l == 0 ? 0.0 : gamma * inv_gamma_prev;
            const double pap = l == 0 ? delta : delta - beta * gamma * inv_alpha_prev;   // p.(A + C)p of the textbook step
            if (!(pap > 0.0)) break;
            const double inv_gamma = 1.0 / gamma;              // independent of alpha: the two divisions overlap
            const double alpha = gamma / pap;
            if (owner) {
                p0 = u0 + beta * p0; s0 = w0 + beta * s0; dl0 = dl0 + alpha * p0; r0 = r0 - alpha * s0; u0 = r0 * mi;
                p1 = u1 + beta * p1; s1 = w1 + beta * s1; dl1 = dl1 + alpha * p1; r1 = r1 - alpha * s1; u1 = r1 * mi;
                p2 = u2 + beta * p2; s2 = w2 + beta * s2; dl2 = dl2 + alpha * p2; r2 = r2 - alpha * s2; u2 = r2 * mi;
                svec[3 * n] = u0; svec[3 * n + 1] = u1; svec[3 * n + 2] = u2;
            }
            for (int h = tid; h < H; h += LM4_THREADS) {       // the same operations on the replicas of the halo columns
                const double *wi = w_in + (par * LM6_HALO + h) * 3;
                const double m = hmi[h];
                double *sv = svec + 3 * hj[h];
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    const double sj = wi[c] + beta * hs[3 * h + c];
                    const double rj = hr[3 * h + c] - alpha * sj;
                    hs[3 * h + c] = sj; hr[3 * h + c] = rj; sv[c] = rj * m;
                }
            }
            const double Q1 = Q0 - 0.5 * alpha * gamma;
            inv_gamma_prev = inv_gamma; inv_alpha_prev = pap * inv_gamma;
            ++pcg_total;
            // Ceres/Opt q-tolerance, solverGPUGaussNewton.t:1093-1101: zeta = (l + 1) (Q1 - Q0) / Q1 < 1e-4, without the division
            // (Q decreases from 0, so Q1 < 0 in every regular step; a zero or NaN Q1 never stops the loop, as with the quotient)
            const double znum = (double)(l + 1) * (Q1 - Q0), zthr = 1e-4 * Q1;
            const bool q_stop = Q1 < 0.0 ? znum > zthr : (Q1 > 0.0 ? znum < zthr : false);
            Q0 = Q1;
            __syncthreads();                                   // svec (own + halo) is complete
            if (q_stop) break;
        }
        // model change = 0.5 dl.(g + r + C dl);  A dl = g - r - C dl  => new cost = cost - dl.g + 0.5 dl.(A dl)
        double mad[3] = {0.0, 0.0, 0.0};
        if (owner) {
            double c;
            c = cdn * dl0; mad[0] += dl0 * (g0 + r0 + c); mad[1] += dl0 * (g0 - r0 - c); mad[2] += dl0 * g0;
            c = cdn * dl1; mad[0] += dl1 * (g1 + r1 + c); mad[1] += dl1 * (g1 - r1 - c); mad[2] += dl1 * g1;
            c = cdn * dl2; mad[0] += dl2 * (g2 + r2 + c); mad[1] += dl2 * (g2 - r2 - c); mad[2] += dl2 * g2;
        }
        lm6_exchange<NCTA, 3, false>(sm, sy, cx, mad, wtpr);
        const double model = 0.5 * mad[0];
        const double new_cost = cost - mad[2] + 0.5 * mad[1];
        const double change = cost - new_cost;
        const double rho = model > 0.0 ? change / model : 0.0;
        bool stop = false;
        if (change >= 0.0 && rho > 1e-3) {
            if (owner) { x0 += dl0; x1 += dl1; x2 += dl2; }
            stop = change <= cost * 1e-6;                       // function_tolerance, CombinedSolver.h:88
            cost = new_cost;
            const double f = 1.0 - (2.0 * rho - 1.0) * (2.0 * rho - 1.0) * (2.0 * rho - 1.0);
            radius /= fmax(f, 1.0 / 3.0);
            radius = fmin(radius, 1e16);
            decrease = 2.0;
        } else {
            radius /= decrease; decrease *= 2.0;
            if (radius <= 1e-32) stop = true;
        }
        if (stop) { ++it; break; }
    }
    if (nl_iters == 0 || overflow) {                           // the cost of the unchanged field, as v5 reports it
        if (owner) { wown[3 * rl] = x0; wown[3 * rl + 1] = x1; wown[3 * rl + 2] = x2; svec[3 * n] = x0; svec[3 * n + 1] = x1; svec[3 * n + 2] = x2; }
        double z[1] = {0.0};
        const int par = lm6_exchange<NCTA, 1, true>(sm, sy, cx, z, 1);
        for (int h = tid; h < H; h += LM4_THREADS) {
            const double *wi = w_in + (par * LM6_HALO + h) * 3;
            double *sv = svec + 3 * hj[h];
            sv[0] = wi[0]; sv[1] = wi[1]; sv[2] = wi[2];
        }
        __syncthreads();
        double Ap0, Ap1, Ap2;
        spmv(Ap0, Ap1, Ap2);
        double t0[1] = {0.0};
        if (owner) { t0[0] += x0 * (0.5 * Ap0 - gb0); t0[0] += x1 * (0.5 * Ap1 - gb1); t0[0] += x2 * (0.5 * Ap2 - gb2); }
        lm6_exchange<NCTA, 1, false>(sm, sy, cx, t0, wtpr);
        cost = c0n[0] + t0[0]; cost0 = cost;
    }
    cluster.sync();                                            // no CTA may exit while others can still write into its shared memory
    // write back: encodeTranslation (CombinedSolver.h:189-197, dual_quaternion.hpp:82-85)
    if (owner && !overflow) {
        float *nd = nodes + (size_t)n * DF_NODE_STRIDE;
        const Quat rot = {nd[3], nd[4], nd[5], nd[6]};
        const Quat h = qhalf(Quat{0.f, (float)x0, (float)x1, (float)x2});
        const Quat d = qmul(h, rot);
        nd[7] = d.w; nd[8] = d.x; nd[9] = d.y; nd[10] = d.z;
    }
    if (gt == 0 && (balanced & 4))                             // DF_SOLVE_TRACE=1
        printf("solve: tiles ran %d fallback reason %d (1 tile nodes, 2 tile list, 3 row columns) max tile nodes %d overflowing tiles %d max tiles/node %d max row columns %d | halo total %d pcg %d\n",
               ws.flags[3], ws.flags[2], ws.flags[4], ws.flags[7], ws.flags[5], ws.flags[6], hmax_i, pcg_total);
    if (gt == 0 && stats) {
        stats[0] = cost0; stats[1] = cost; stats[2] = (double)it; stats[3] = nvalid; stats[4] = (double)pcg_total; stats[5] = (double)ws.flags[0];
        stats[6] = nnz_total; stats[7] = (double)hmax_i + ((ws.flags[3] && !ws.flags[2]) ? 0.5 : 0.0);   // halo columns of the cluster; + 0.5: matrix from the tile records
    }
}

int solve_lm_impl()           // DF_SOLVE_LM_IMPL=1 forces the one-block fallback kernel (tests)
{
    static const int impl = [] { const char *e = getenv("DF_SOLVE_LM_IMPL"); return e ? atoi(e) : 6; }();
    return impl;
}

}  // namespace

extern "C" size_t df_solve_workspace_bytes(int M, int N)
{
    SolveWs ws;
    return layout(ws, nullptr, M, N) + 256;
}

extern "C" int df_solve_knn_buffers(void *workspace, int M, int N, int32_t **idx, float **w)
{
    SolveWs ws;
    char *base = (char *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    layout(ws, base, M, N);
    *idx = ws.idx; *w = ws.w;
    return 0;
}

// The assembly kernels (solve_rows / solve_rows_tiles) write these arrays; the LM kernels (one-block, v5, v6) only read them, so after a
// solve they hold the system the LM iteration was given.
extern "C" int df_solve_normal_system(void *workspace, int M, int N, int32_t **rownnz, int32_t **col, double **val, double **gb, double **diag)
{
    SolveWs ws;
    char *base = (char *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    layout(ws, base, M, N);
    *rownnz = ws.rownnz; *col = ws.col; *val = ws.val; *gb = ws.gb; *diag = ws.diag;
    return 0;
}

extern "C" int df_solve_data_term(float *nodes, int M, const void *node_grid, const float *canon, const float *live, int N, int stride,
                                  int nonlinear_iters, int linear_iters, int flags, double *stats_dev, void *workspace, void *stream)
{
    return dfb::solve_data_term_ev(nodes, M, node_grid, canon, live, N, stride, nonlinear_iters, linear_iters, flags, stats_dev, workspace,
                                   (cudaStream_t)stream, nullptr);
}

int dfb::solve_data_term_ev(float *nodes, int M, const void *node_grid, const float *canon, const float *live, int N, int stride, int nonlinear_iters,
                            int linear_iters, int flags, double *stats_dev, void *workspace, cudaStream_t s, cudaEvent_t before_lm)
{
    if (M <= 0 || N <= 0) { if (before_lm) cudaEventRecord(before_lm, s); return 0; }
    SolveWs ws;
    char *base = (char *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
    layout(ws, base, M, N);
    cudaError_t e = cudaMemsetAsync(ws.blockcnt, 0, (size_t)M * ws.prepare_blocks * 4, s);
    if (e != cudaSuccess) return (int)e;
    if (ws.ntiles > 0 && ((flags >> 8) & 0xffff) > 0) {
        e = cudaMemsetAsync(ws.touch, 0, (size_t)M * ws.ntiles, s);
        if (e != cudaSuccess) return (int)e;
    }
    const int img_cols = (flags >> 8) & 0xffff;
    const int patch_cols = (img_cols > 0 && N % img_cols == 0 && img_cols % 32 == 0 && (N / img_cols) % 8 == 0) ? img_cols : 0;
    launch_pdl(solve_prepare_kernel, dim3(ws.prepare_blocks), dim3(256), 0, s, nodes, M, node_grid, canon, live, N, stride, ws, patch_cols);
    DF_LAUNCH_CHECK();
    launch_pdl(solve_blockscan_kernel, dim3(div_up(M, 8)), dim3(256), 0, s, ws, M);
    DF_LAUNCH_CHECK();
    launch_pdl(solve_scan_kernel, dim3(1), dim3(1024), 0, s, ws, M);
    DF_LAUNCH_CHECK();
    // image-shaped vertices: tile records (DF_SOLVE_TILES=0 disables), with the per-entry kernels behind them as the fallback
    static const int want_tiles = [] { const char *e = getenv("DF_SOLVE_TILES"); return e ? atoi(e) : 1; }();
    const int cols = (flags >> 8) & 0xffff;
    const bool tiles = want_tiles && cols > 0 && ws.ntiles > 0 && N % cols == 0 && cols % TILE_W == 0 && (N / cols) % TILE_H == 0 && M * (size_t)ws.ntiles > 0;
    if (tiles) {
        launch_pdl(solve_tiles_kernel, dim3(ws.ntiles), dim3(TILE_PIX), 0, s, ws, cols, N / cols);
        DF_LAUNCH_CHECK();
        launch_pdl(solve_rows_tiles_kernel, dim3(M), dim3(RT_THREADS), 0, s, ws, M, N, flags & DF_SOLVE_REF_GRAPH_QUIRK);
        DF_LAUNCH_CHECK();
    }
    launch_pdl(solve_fill_kernel, dim3(ws.prepare_blocks), dim3(256), 0, s, ws, N, tiles ? 1 : 0, patch_cols);
    DF_LAUNCH_CHECK();
    launch_pdl(solve_rows_kernel, dim3(M), dim3(ROWS_THREADS), 0, s, ws, M, N, flags & DF_SOLVE_REF_GRAPH_QUIRK, tiles ? 1 : 0);
    DF_LAUNCH_CHECK();
    if (before_lm && cudaEventRecord(before_lm, s) != cudaSuccess) return (int)cudaGetLastError();
    // One cluster when the system fits its shared memory (16 CTAs = the non-portable maximum: half the rows, hence half the mat-vec
    // gather traffic, per SM; DF_SOLVE_LM_CTAS=8 selects the portable size); otherwise the one-block kernel (matrix in L2).
    // DF_SOLVE_LM_IMPL: 6 (default) = v6 with v5 launched behind it as its fallback, 5 = v5 alone, 1 = the one-block kernel.
    static const int want = [] { const char *e = getenv("DF_SOLVE_LM_CTAS"); return e ? atoi(e) : 16; }();
    // a 16-CTA cluster of ~216 KB CTAs needs 16 free SMs in one GPC; how many SMs a GPC keeps differs between H100 parts, so the
    // occupancy calculator is asked once (for the largest shared-memory size used below) and the portable 8 taken when it says no
    static const bool cluster16 = [] {
        const auto kern = solve_lm_v5_kernel<16, true>;
        const int smem = 216 * 1024;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
            cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) { (void)cudaGetLastError(); return false; }
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(16); cfg.blockDim = dim3(LM4_THREADS); cfg.dynamicSmemBytes = smem;
        cudaLaunchAttribute at;
        at.id = cudaLaunchAttributeClusterDimension;
        at.val.clusterDim.x = 16; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
        cfg.attrs = &at; cfg.numAttrs = 1;
        int clusters = 0;
        if (cudaOccupancyMaxActiveClusters(&clusters, kern, &cfg) != cudaSuccess) { (void)cudaGetLastError(); return false; }
        return clusters >= 1;
    }();
    const int ncta = (want == 16 && cluster16 && M >= 256) ? 16 : 8;
    static const int balanced = [] { const char *e = getenv("DF_SOLVE_BALANCED"); return e ? atoi(e) : 1; }();
    auto launch_cluster = [&](auto kern, size_t smem_budget, size_t smem, auto... args) -> cudaError_t {
        // function attributes are per device: set them on every launch (cheap) rather than once per process.  The limit set is the
        // kernel's fixed budget, never this launch's size: objects advanced from several host threads (df_kinfu_batch_process_host)
        // share the attribute, and a smaller size set by one thread between another's set and launch would fail that launch
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_budget);
        if (ncta == 16) cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(ncta); cfg.blockDim = dim3(LM4_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = s;
        cudaLaunchAttribute at[2];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = ncta; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[1].val.programmaticStreamSerializationAllowed = pdl_enabled();
        cfg.attrs = at; cfg.numAttrs = 2;
        return cudaLaunchKernelEx(&cfg, kern, args...);
    };
    const Lm4Layout Lb = lm4_layout(M, 0, ncta);
    const size_t budget = ncta == 16 ? (size_t)216 * 1024 : (size_t)220 * 1024;      // 227 KB minus the static shared memory (8.6 KB with 16 CTAs, 4.6 KB with 8)
    if (solve_lm_impl() >= 5 && Lb.rpc * Lb.tpr <= LM4_THREADS && Lb.total + (size_t)LM4_THREADS * 10 * 8 <= budget) {
        bool v6 = false;
        if (solve_lm_impl() >= 6 && M <= 32 * LM6_BITW) {
            const Lm6Layout L6 = lm6_layout(M, 0, ncta);
            const size_t budget6 = (size_t)220 * 1024;                                  // 227 KB minus v6's static shared memory (5.5 KB)
            if (L6.total + (size_t)LM4_THREADS * 10 * 6 <= budget6) {                   // room for at least 6 entries per lane
                const int cap6 = (int)((budget6 - L6.total - 32) / ((size_t)LM4_THREADS * 10));
                const Lm6Layout Lc6 = lm6_layout(M, cap6, ncta);
                using K6 = void (*)(float *, int, const void *, SolveWs, int, int, double *, int, int);
                const K6 k6 = ncta == 16 ? (K6)solve_lm_v6_kernel<16> : (K6)solve_lm_v6_kernel<8>;
                static const int trace = [] { const char *e = getenv("DF_SOLVE_TRACE"); return e ? atoi(e) : 0; }();
                static const int force_fb = [] { const char *e = getenv("DF_SOLVE_V6_FORCE_FALLBACK"); return e ? atoi(e) : 0; }();
                const cudaError_t le = launch_cluster(k6, budget6, Lc6.total, nodes, M, node_grid, ws, nonlinear_iters, linear_iters, stats_dev, cap6, balanced | (force_fb ? 2 : 0) | (trace ? 4 : 0));
                if (le != cudaSuccess) return (int)le;
                v6 = true;
            }
        }
        const int cap = (int)((budget - Lb.total - 16) / ((size_t)LM4_THREADS * 10));
        const Lm4Layout Lc = lm4_layout(M, cap, ncta);
        static const int merged = [] { const char *e = getenv("DF_SOLVE_MERGED"); return e ? atoi(e) : 1; }();
        using KernelT = void (*)(float *, int, const void *, SolveWs, int, int, double *, int, int, int);
        const KernelT kern = ncta == 16 ? (merged ? (KernelT)solve_lm_v5_kernel<16, true> : (KernelT)solve_lm_v5_kernel<16, false>)
                                        : (merged ? (KernelT)solve_lm_v5_kernel<8, true> : (KernelT)solve_lm_v5_kernel<8, false>);
        const cudaError_t le = launch_cluster(kern, budget, Lc.total, nodes, M, node_grid, ws, nonlinear_iters, linear_iters, stats_dev, cap, balanced, v6 ? 1 : 0);
        if (le != cudaSuccess) return (int)le;
    } else {
        solve_lm_kernel<<<1, LM_THREADS, 0, s>>>(nodes, M, ws, nonlinear_iters, linear_iters, stats_dev);
    }
    DF_LAUNCH_CHECK();
    return 0;
}
