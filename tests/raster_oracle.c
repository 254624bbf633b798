/* raster_oracle.c -- plain C statement of the rasteriser's rule (include/dfusion.h, df_raster_mesh): a loop over triangles and the pixels of
 * their bounding boxes, test infrastructure only.  Compiled with -ffp-contract=off so that every float operation is the one the rule
 * names; fmaf only where the rule writes fma.  ro_raster is the renderer; ro_coverage counts, per pixel, the front-facing triangles that
 * cover its sample, without the depth test. */
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "oracle_util.h"

#define NEAR 0.01f
#define GUARD 16777216.f
#define SMALL 8

typedef struct { float R[9]; float t[3]; } aff;
typedef struct { float fx, fy, cx, cy; } intr;

typedef struct {
    long long ax[3], ay[3], dx[3], dy[3];
    int bias[3];
    int x0, x1, y0, y1;
    float n[3], num;
} tri_t;

static void cross(const float *a, const float *b, float *o)
{
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }

/* camera frame and fixed-point position of every vertex; fix[2i] = INT_MIN marks a skipped vertex */
static void vertices(const float *verts, int n, int vstride, const aff *w, const intr *K, float *cam, int *fix)
{
    for (int i = 0; i < n; ++i) {
        const float *v = verts + (size_t)i * vstride;
        const float x = v[0], y = v[1], z = v[2];
        float *c = cam + 3 * (size_t)i;
        c[0] = w->R[0] * x + w->R[1] * y + w->R[2] * z + w->t[0];
        c[1] = w->R[3] * x + w->R[4] * y + w->R[5] * z + w->t[1];
        c[2] = w->R[6] * x + w->R[7] * y + w->R[8] * z + w->t[2];
        fix[2 * i] = fix[2 * i + 1] = INT_MIN;
        if (isfinite(c[0]) && isfinite(c[1]) && isfinite(c[2]) && c[2] >= NEAR) {
            const float su = fmaf(K->fx, c[0] / c[2], K->cx) * 256.f, sv = fmaf(K->fy, c[1] / c[2], K->cy) * 256.f;
            if (fabsf(su) <= GUARD && fabsf(sv) <= GUARD) { fix[2 * i] = (int)lrintf(su); fix[2 * i + 1] = (int)lrintf(sv); }
        }
    }
}

/* 0 draw, 1 back-facing or zero area, 2 skipped */
static int setup(const int32_t *tris, int t, int n_verts, const float *cam, const int *fix, int cols, int rows, tri_t *T)
{
    const int32_t *ix = tris + 3 * (size_t)t;
    for (int k = 0; k < 3; ++k)
        if (ix[k] < 0 || ix[k] >= n_verts) return 2;
    for (int k = 0; k < 3; ++k)
        if (fix[2 * ix[k]] == INT_MIN) return 2;
    const long long U0 = fix[2 * ix[0]], V0 = fix[2 * ix[0] + 1], U1 = fix[2 * ix[1]], V1 = fix[2 * ix[1] + 1];
    const long long U2 = fix[2 * ix[2]], V2 = fix[2 * ix[2] + 1];
    const long long area = (U1 - U0) * (V2 - V0) - (V1 - V0) * (U2 - U0);
    if (area >= 0) return 1;
    const long long U[3] = {U0, U2, U1}, V[3] = {V0, V2, V1};
    for (int k = 0; k < 3; ++k) {
        const int e = (k + 1) % 3;
        T->ax[k] = U[k]; T->ay[k] = V[k];
        T->dx[k] = U[e] - U[k]; T->dy[k] = V[e] - V[k];
        T->bias[k] = (T->dy[k] < 0 || (T->dy[k] == 0 && T->dx[k] > 0)) ? 0 : 1;
    }
    const int mnx = (int)(U0 < U1 ? (U0 < U2 ? U0 : U2) : (U1 < U2 ? U1 : U2)), mxx = (int)(U0 > U1 ? (U0 > U2 ? U0 : U2) : (U1 > U2 ? U1 : U2));
    const int mny = (int)(V0 < V1 ? (V0 < V2 ? V0 : V2) : (V1 < V2 ? V1 : V2)), mxy = (int)(V0 > V1 ? (V0 > V2 ? V0 : V2) : (V1 > V2 ? V1 : V2));
    /* ceil / floor of a division by 256 (gcc's >> of a negative int is arithmetic) */
    T->x0 = imax((mnx + 255) >> 8, 0); T->x1 = imin(mxx >> 8, cols - 1);
    T->y0 = imax((mny + 255) >> 8, 0); T->y1 = imin(mxy >> 8, rows - 1);
    const float *c0 = cam + 3 * (size_t)ix[0], *c1 = cam + 3 * (size_t)ix[1], *c2 = cam + 3 * (size_t)ix[2];
    const float e1[3] = {c1[0] - c0[0], c1[1] - c0[1], c1[2] - c0[2]}, e2[3] = {c2[0] - c0[0], c2[1] - c0[1], c2[2] - c0[2]};
    cross(e1, e2, T->n);
    T->num = dot(T->n, c0);
    return 0;
}

static int covers(const tri_t *T, int i, int j)
{
    const long long px = (long long)i * 256, py = (long long)j * 256;
    for (int k = 0; k < 3; ++k)
        if (!(T->dx[k] * (py - T->ay[k]) - T->dy[k] * (px - T->ax[k]) >= T->bias[k])) return 0;
    return 1;
}

static void ray(const intr *K, float finvx, float finvy, int i, int j, float *d)
{
    d[0] = ((float)i - K->cx) * finvx;
    d[1] = ((float)j - K->cy) * finvy;
    d[2] = 1.f;
}

/* the renderer: tri_ids (cols*rows, may be NULL), points and normals (cols*rows*4 floats), stats (5, may be NULL); returns 0, or -1 when
 * out of memory */
int ro_raster(const float *verts, int n_verts, int vstride, const int32_t *tris, int n_tris, const float *w12, const float *k4, int cols,
              int rows, int32_t *tri_ids, float *points, float *normals, unsigned long long *stats)
{
    aff w; intr K;
    memcpy(w.R, w12, 36); memcpy(w.t, w12 + 9, 12);
    K.fx = k4[0]; K.fy = k4[1]; K.cx = k4[2]; K.cy = k4[3];
    const float finvx = 1.f / K.fx, finvy = 1.f / K.fy;
    float *cam = malloc(((size_t)n_verts * 3 + 1) * sizeof(float));
    int *fix = malloc(((size_t)n_verts * 2 + 1) * sizeof(int));
    unsigned long long *z = malloc((size_t)cols * rows * sizeof(unsigned long long));
    if (!cam || !fix || !z) { free(cam); free(fix); free(z); return -1; }
    unsigned long long st[5] = {0, 0, 0, 0, 0};
    vertices(verts, n_verts, vstride, &w, &K, cam, fix);
    for (size_t p = 0; p < (size_t)cols * rows; ++p) z[p] = ~0ull;
    for (int t = 0; t < n_tris; ++t) {
        tri_t T;
        const int s = setup(tris, t, n_verts, cam, fix, cols, rows, &T);
        if (s) { ++st[s - 1]; continue; }
        ++st[(T.x1 - T.x0 < SMALL && T.y1 - T.y0 < SMALL) ? 2 : 3];
        for (int j = T.y0; j <= T.y1; ++j)
            for (int i = T.x0; i <= T.x1; ++i) {
                if (!covers(&T, i, j)) continue;
                float d[3];
                ray(&K, finvx, finvy, i, j, d);
                const float tz = T.num / dot(T.n, d);
                if (!(tz > 0.f && tz < INFINITY)) continue;
                const unsigned long long key = ((unsigned long long)float_bits(tz) << 32) | (uint32_t)t;
                if (key < z[(size_t)j * cols + i]) z[(size_t)j * cols + i] = key;
            }
    }
    const uint32_t nan_bits = 0x7fffffffu;                  /* the NaN the CUDA kernels write */
    float nanv;
    memcpy(&nanv, &nan_bits, 4);
    for (int j = 0; j < rows; ++j)
        for (int i = 0; i < cols; ++i) {
            const size_t p = (size_t)j * cols + i;
            float *P = points + 4 * p, *N = normals + 4 * p;
            if (z[p] == ~0ull) {
                for (int k = 0; k < 4; ++k) P[k] = N[k] = nanv;
                if (tri_ids) tri_ids[p] = -1;
                continue;
            }
            ++st[4];
            const int t = (int)(uint32_t)z[p];
            const int32_t *ix = tris + 3 * (size_t)t;
            const float *c0 = cam + 3 * (size_t)ix[0], *c1 = cam + 3 * (size_t)ix[1], *c2 = cam + 3 * (size_t)ix[2];
            const float e1[3] = {c1[0] - c0[0], c1[1] - c0[1], c1[2] - c0[2]}, e2[3] = {c2[0] - c0[0], c2[1] - c0[1], c2[2] - c0[2]};
            float n[3], d[3];
            cross(e1, e2, n);
            ray(&K, finvx, finvy, i, j, d);
            const float tz = dot(n, c0) / dot(n, d);
            const float len = sqrtf(dot(n, n));
            P[0] = d[0] * tz; P[1] = d[1] * tz; P[2] = tz; P[3] = 0.f;
            N[0] = n[0] / len; N[1] = n[1] / len; N[2] = n[2] / len; N[3] = 0.f;
            if (tri_ids) tri_ids[p] = t;
        }
    if (stats) memcpy(stats, st, sizeof st);
    free(cam); free(fix); free(z);
    return 0;
}

/* per pixel, the number of drawn (front-facing, not skipped) triangles whose sample test covers it; no depth test */
int ro_coverage(const float *verts, int n_verts, int vstride, const int32_t *tris, int n_tris, const float *w12, const float *k4, int cols,
                int rows, int32_t *count)
{
    aff w; intr K;
    memcpy(w.R, w12, 36); memcpy(w.t, w12 + 9, 12);
    K.fx = k4[0]; K.fy = k4[1]; K.cx = k4[2]; K.cy = k4[3];
    float *cam = malloc(((size_t)n_verts * 3 + 1) * sizeof(float));
    int *fix = malloc(((size_t)n_verts * 2 + 1) * sizeof(int));
    if (!cam || !fix) { free(cam); free(fix); return -1; }
    vertices(verts, n_verts, vstride, &w, &K, cam, fix);
    memset(count, 0, (size_t)cols * rows * sizeof(int32_t));
    for (int t = 0; t < n_tris; ++t) {
        tri_t T;
        if (setup(tris, t, n_verts, cam, fix, cols, rows, &T)) continue;
        for (int j = T.y0; j <= T.y1; ++j)
            for (int i = T.x0; i <= T.x1; ++i)
                if (covers(&T, i, j)) ++count[(size_t)j * cols + i];
    }
    free(cam); free(fix);
    return 0;
}
