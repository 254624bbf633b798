// nodegrid.cu -- builds the uniform grid over the warp nodes' vertices (layout: warp_common.cuh, NodeGridHeader).
// Replaces WarpField::buildKDTree (kfusion/src/warp_field.cpp:275-282, nanoflann index over nodes_).  Built once per node
// set (node vertices are immutable after WarpField::init); one 1024-thread block, deterministic output: nodes are stored
// cell by cell and, inside a cell, in ascending node index.
#include "warp_common.cuh"

using namespace dfb;

namespace {

__global__ void __launch_bounds__(1024) build_node_grid_kernel(const float *__restrict__ nodes, int M, void *grid, int *cid_tmp, int *order, int *slot,
                                                               float4 *bvh_box, float4 *bvh_leaf, int L)
{
    __shared__ float smin[3][32], smax[3][32];
    __shared__ NodeGridHeader h;
    __shared__ int partial[1024];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;

    // 1. bounding box of the vertices
    float mn[3] = {3.4e38f, 3.4e38f, 3.4e38f}, mx[3] = {-3.4e38f, -3.4e38f, -3.4e38f};
    for (int i = t; i < M; i += 1024)
        for (int c = 0; c < 3; ++c) { const float v = nodes[(size_t)i * DF_NODE_STRIDE + c]; mn[c] = fminf(mn[c], v); mx[c] = fmaxf(mx[c], v); }
    for (int c = 0; c < 3; ++c) {
        for (int o = 16; o > 0; o >>= 1) { mn[c] = fminf(mn[c], __shfl_xor_sync(0xffffffffu, mn[c], o)); mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o)); }
        if (lane == 0) { smin[c][warp] = mn[c]; smax[c][warp] = mx[c]; }
    }
    __syncthreads();
    if (t == 0) {
        float lo[3], hi[3];
        for (int c = 0; c < 3; ++c) {
            lo[c] = smin[c][0]; hi[c] = smax[c][0];
            for (int w = 1; w < 32; ++w) { lo[c] = fminf(lo[c], smin[c][w]); hi[c] = fmaxf(hi[c], smax[c][w]); }
        }
        const float ext = fmaxf(fmaxf(hi[0] - lo[0], hi[1] - lo[1]), hi[2] - lo[2]);
        // nodes sample a surface: ~sqrt(M) nodes along the longest extent; ~3 node spacings per cell, so that the 8th
        // neighbour (about 1.7 spacings away) is usually confirmed after the first shell (27 cells)
        int res = (int)ceilf(sqrtf((float)M) / 3.0f);
        res = max(1, min(res, NODEGRID_MAX_RES));
        const float cell = ext > 0.f ? ext / (float)res * 1.0001f : 1.f;
        h.ox = lo[0]; h.oy = lo[1]; h.oz = lo[2]; h.cell = cell; h.inv_cell = 1.f / cell;
        h.gx = min(NODEGRID_MAX_RES, (int)((hi[0] - lo[0]) * h.inv_cell) + 1);
        h.gy = min(NODEGRID_MAX_RES, (int)((hi[1] - lo[1]) * h.inv_cell) + 1);
        h.gz = min(NODEGRID_MAX_RES, (int)((hi[2] - lo[2]) * h.inv_cell) + 1);
        h.M = M; h.ncell = h.gx * h.gy * h.gz;
        for (int i = 0; i < 6; ++i) h.pad[i] = 0;
        *reinterpret_cast<NodeGridHeader *>(grid) = h;
    }
    __syncthreads();
    int *cell_start = reinterpret_cast<int *>(reinterpret_cast<char *>(grid) + 64);
    float4 *sorted = reinterpret_cast<float4 *>(reinterpret_cast<char *>(grid) + 64 + (((size_t)(h.ncell + 1) * 4 + 15) & ~(size_t)15));

    // 2. cell of every node, per-cell counts
    for (int i = t; i <= h.ncell; i += 1024) cell_start[i] = 0;
    __syncthreads();
    for (int i = t; i < M; i += 1024) {
        const float *v = nodes + (size_t)i * DF_NODE_STRIDE;
        const int cx = min(max((int)floorf((v[0] - h.ox) * h.inv_cell), 0), h.gx - 1);
        const int cy = min(max((int)floorf((v[1] - h.oy) * h.inv_cell), 0), h.gy - 1);
        const int cz = min(max((int)floorf((v[2] - h.oz) * h.inv_cell), 0), h.gz - 1);
        const int cid = cx + h.gx * (cy + h.gy * cz);
        cid_tmp[i] = cid;
        atomicAdd(cell_start + cid + 1, 1);         // counts shifted by one: the inclusive scan below yields the starts
    }
    __syncthreads();
    // 3. inclusive scan of cell_start[1..ncell] (chunked per thread + block scan of chunk sums)
    const int n = h.ncell;
    const int per = (n + 1023) / 1024;
    const int b = min(n, t * per) + 1, e = min(n, t * per + per) + 1;
    int s = 0;
    for (int i = b; i < e; ++i) s += cell_start[i];
    partial[t] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = t >= o ? partial[t - o] : 0;
        __syncthreads();
        partial[t] += v;
        __syncthreads();
    }
    int run = partial[t] - s;
    for (int i = b; i < e; ++i) { run += cell_start[i]; cell_start[i] = run; }
    __syncthreads();
    // 4. deterministic placement: rank inside the cell = number of lower-indexed nodes in the same cell
    for (int i = t; i < M; i += 1024) {
        const int cid = cid_tmp[i];
        int rank = 0;
        for (int j = 0; j < i; ++j) rank += (cid_tmp[j] == cid);
        const float *v = nodes + (size_t)i * DF_NODE_STRIDE;
        sorted[cell_start[cid] + rank] = make_float4(v[0], v[1], v[2], __int_as_float(i));
    }
    // 5. spatial (Morton) order of the nodes for the solver: consecutive slots are neighbours in space, so a CTA that owns a
    //    contiguous range of slots couples almost only to its own rows (solve.cu, v4).  order[rank] = node, slot[node] = rank.
    if (order) {
        __syncthreads();
        const float q = h.inv_cell * (1024.f / (float)max(max(h.gx, h.gy), h.gz));
        for (int i = t; i < M; i += 1024) {
            const float *v = nodes + (size_t)i * DF_NODE_STRIDE;
            unsigned c[3];
            c[0] = (unsigned)min(max((int)((v[0] - h.ox) * q), 0), 1023);
            c[1] = (unsigned)min(max((int)((v[1] - h.oy) * q), 0), 1023);
            c[2] = (unsigned)min(max((int)((v[2] - h.oz) * q), 0), 1023);
            unsigned key = 0;
            for (int b = 0; b < 10; ++b)
                for (int a = 0; a < 3; ++a) key |= ((c[a] >> b) & 1u) << (3 * b + a);
            cid_tmp[i] = (int)key;
        }
        __syncthreads();
        for (int i = t; i < M; i += 1024) {
            const int key = cid_tmp[i];
            int rank = 0;
            for (int j = 0; j < M; ++j) { const int kj = cid_tmp[j]; rank += (kj < key) || (kj == key && j < i); }
            order[rank] = i; slot[i] = rank;
        }
        if (t == 0) {
            NodeGridHeader *hg = reinterpret_cast<NodeGridHeader *>(grid);
            hg->pad[0] = (int)(reinterpret_cast<char *>(order) - reinterpret_cast<char *>(grid));
            hg->pad[1] = (int)(reinterpret_cast<char *>(slot) - reinterpret_cast<char *>(grid));
        }
        // 6. bounding-volume hierarchy for queries that lie far from every node and for the per-voxel searches of fusion.cu (warp_common.cuh,
        //    knn8_bvh / knn8_bvh_seeded): leaves = NODEGRID_BVH_LEAF nodes, implicit complete binary tree of L leaves, boxes bottom-up.
        //    Leaf membership = a k-d median split: the entries of every segment (the whole array, then halves, quarters, ... down to 16)
        //    are sorted along the segment's widest axis and the segment is cut in the middle, so a leaf is a compact patch of eight nodes.
        //    (Runs of eight in Morton order made long, overlapping leaf boxes at Z-curve jumps: ~10 leaves entered per query of the fusion
        //    kernel, most of its instructions in leaf-entry and box tests.)  Segments are aligned
        //    power-of-two blocks, so one bitonic network run up to block size S sorts all of them at once; ties break on the node index.
        //    The search result never depends on this order (boxes are built from whatever the leaves hold; ranking is by (distance, index)).
        if (bvh_box) {
            __syncthreads();
            const float inf = __int_as_float(0x7f800000);
            const int Mpad = L * NODEGRID_BVH_LEAF;
            for (int sidx = t; sidx < Mpad; sidx += 1024) {
                float4 e = make_float4(inf, inf, inf, __int_as_float(0x7fffffff));
                if (sidx < M) { const float *v = nodes + (size_t)sidx * DF_NODE_STRIDE; e = make_float4(v[0], v[1], v[2], __int_as_float(sidx)); }
                bvh_leaf[sidx] = e;
            }
            for (int S = Mpad; S >= 2 * NODEGRID_BVH_LEAF; S >>= 1) {
                __syncthreads();
                // widest axis of every segment (one warp per segment; padding entries are skipped); partial[] holds the axes
                const int nseg = Mpad / S;
                for (int seg = warp; seg < nseg; seg += 32) {
                    float lo[3] = {inf, inf, inf}, hi[3] = {-inf, -inf, -inf};
                    for (int k = lane; k < S; k += 32) {
                        const float4 e = bvh_leaf[seg * S + k];
                        if (__float_as_int(e.w) == 0x7fffffff) continue;
                        lo[0] = fminf(lo[0], e.x); hi[0] = fmaxf(hi[0], e.x);
                        lo[1] = fminf(lo[1], e.y); hi[1] = fmaxf(hi[1], e.y);
                        lo[2] = fminf(lo[2], e.z); hi[2] = fmaxf(hi[2], e.z);
                    }
                    for (int c = 0; c < 3; ++c)
                        for (int o = 16; o > 0; o >>= 1) { lo[c] = fminf(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o)); hi[c] = fmaxf(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o)); }
                    if (lane == 0) {
                        const float ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];      // NaN (empty segment: inf - inf) compares false: axis 0
                        partial[seg] = (ey > ex && ey >= ez) ? 1 : ((ez > ex && ez > ey) ? 2 : 0);
                    }
                }
                __syncthreads();
                for (int k = 2; k <= S; k <<= 1)
                    for (int j = k >> 1; j > 0; j >>= 1) {
                        for (int i = t; i < Mpad; i += 1024) {
                            const int partner = i ^ j;
                            if (partner > i) {
                                const int axis = partial[i / S];
                                const bool up = (k == S) || ((i & k) == 0);           // every segment ends ascending
                                const float4 a = bvh_leaf[i], b = bvh_leaf[partner];
                                const float ka = axis == 0 ? a.x : (axis == 1 ? a.y : a.z), kb = axis == 0 ? b.x : (axis == 1 ? b.y : b.z);
                                const int ia = __float_as_int(a.w), ib = __float_as_int(b.w);
                                const bool a_after_b = ka > kb || (ka == kb && ia > ib);      // padding: key inf, index INT_MAX -> sorts last
                                if (a_after_b == up) { bvh_leaf[i] = b; bvh_leaf[partner] = a; }
                            }
                        }
                        __syncthreads();
                    }
            }
            __syncthreads();
            for (int l = t; l < L; l += 1024) {
                float3 lo = make_float3(inf, inf, inf), hi = make_float3(-inf, -inf, -inf);
                for (int k = 0; k < NODEGRID_BVH_LEAF; ++k) {
                    const float4 e = bvh_leaf[l * NODEGRID_BVH_LEAF + k];
                    if (__float_as_int(e.w) == 0x7fffffff) continue;
                    lo = make_float3(fminf(lo.x, e.x), fminf(lo.y, e.y), fminf(lo.z, e.z));
                    hi = make_float3(fmaxf(hi.x, e.x), fmaxf(hi.y, e.y), fmaxf(hi.z, e.z));
                }
                bvh_box[2 * (L - 1 + l)] = make_float4(lo.x, lo.y, lo.z, 0.f);
                bvh_box[2 * (L - 1 + l) + 1] = make_float4(hi.x, hi.y, hi.z, 0.f);
            }
            for (int width = L / 2; width >= 1; width /= 2) {          // internal nodes [width - 1, 2 * width - 1), one level per pass
                __syncthreads();
                for (int k = t; k < width; k += 1024) {
                    const int i = width - 1 + k;
                    const float4 alo = bvh_box[2 * (2 * i + 1)], ahi = bvh_box[2 * (2 * i + 1) + 1];
                    const float4 blo = bvh_box[2 * (2 * i + 2)], bhi = bvh_box[2 * (2 * i + 2) + 1];
                    bvh_box[2 * i] = make_float4(fminf(alo.x, blo.x), fminf(alo.y, blo.y), fminf(alo.z, blo.z), 0.f);
                    bvh_box[2 * i + 1] = make_float4(fmaxf(ahi.x, bhi.x), fmaxf(ahi.y, bhi.y), fmaxf(ahi.z, bhi.z), 0.f);
                }
            }
            if (t == 0) {
                NodeGridHeader *hg = reinterpret_cast<NodeGridHeader *>(grid);
                hg->pad[2] = (int)(reinterpret_cast<char *>(bvh_box) - reinterpret_cast<char *>(grid));
                hg->pad[3] = (int)(reinterpret_cast<char *>(bvh_leaf) - reinterpret_cast<char *>(grid));
                hg->pad[4] = L;
            }
        }
    }
}

}  // namespace

static int bvh_leaves(int M)
{
    int L = 1;
    while (L * NODEGRID_BVH_LEAF < M) L *= 2;
    return L;
}
static size_t bvh_bytes(int M) { return M <= NODEGRID_ORDER_MAX_M ? (size_t)bvh_leaves(M) * (2 * 32 + NODEGRID_BVH_LEAF * 16) : 0; }

extern "C" size_t df_node_grid_bytes(int M)
{
    const size_t ncell = (size_t)NODEGRID_MAX_RES * NODEGRID_MAX_RES * NODEGRID_MAX_RES;
    const size_t m = (size_t)(M > 0 ? M : 1);
    // header, cell starts, cell-sorted nodes, [BVH boxes + leaves], cell ids / order / slot
    return 64 + (((ncell + 1) * 4 + 15) & ~(size_t)15) + m * 16 + bvh_bytes((int)m) + 3 * ((m * 4 + 15) & ~(size_t)15) + 256;
}

extern "C" int df_build_node_grid(const float *nodes, int M, void *grid, void *stream)
{
    if (M <= 0) return (int)cudaErrorInvalidValue;
    // three int[M] arrays at the very end of the buffer: scratch cell ids / Morton keys, order, slot
    const size_t arr = ((size_t)M * 4 + 15) & ~(size_t)15;
    char *tail = reinterpret_cast<char *>(grid) + df_node_grid_bytes(M) - 3 * arr - 128;
    int *cid_tmp = reinterpret_cast<int *>(tail);
    const bool want_order = M <= NODEGRID_ORDER_MAX_M;        // the ranking is O(M^2) in one block
    int *order = want_order ? reinterpret_cast<int *>(tail + arr) : nullptr;
    int *slot = want_order ? reinterpret_cast<int *>(tail + 2 * arr) : nullptr;
    const int L = bvh_leaves(M);
    float4 *bvh_box = want_order ? reinterpret_cast<float4 *>(tail - bvh_bytes(M)) : nullptr;      // 16-byte aligned: every block above is
    float4 *bvh_leaf = want_order ? bvh_box + 4 * (size_t)L : nullptr;
    build_node_grid_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(nodes, M, grid, cid_tmp, order, slot, bvh_box, bvh_leaf, L);
    DF_LAUNCH_CHECK();
    return 0;
}
