/* reloc_oracle.c -- the relocaliser's rules (include/dfusion.h, DF_KINFU_RELOCALISE) stated again in plain C, test infrastructure only:
 * the fern table, the codes, the match with its top-K and harvest, and the gate's counts in double with the pixels a float evaluation
 * could decide the other way counted apart. */
#include <math.h>
#include <stdint.h>
#include <string.h>

static uint64_t next(uint64_t *s)
{
    *s += 0x9e3779b97f4a7c15ull;
    uint64_t z = *s;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

void rc_fern_table(uint64_t seed, int cols, int rows, int n_ferns, int near_mm, int far_mm, int32_t *out)
{
    uint64_t s = seed;
    for (int i = 0; i < n_ferns * 4; ++i) {
        out[3 * i] = (int32_t)(next(&s) % (uint64_t)cols);
        out[3 * i + 1] = (int32_t)(next(&s) % (uint64_t)rows);
        out[3 * i + 2] = (int32_t)(near_mm + (int64_t)(next(&s) % (uint64_t)(far_mm - near_mm)));
    }
}

/* depth: rows x cols u16 with `stride` elements per row */
void rc_encode(const uint16_t *depth, int stride, int cols, int rows, const int32_t *table, int n_ferns, uint8_t *codes)
{
    for (int f = 0; f < n_ferns; ++f) {
        int code = 0;
        for (int j = 0; j < 4; ++j) {
            const int32_t *t = table + 12 * f + 3 * j;
            if (t[0] < 0 || t[1] < 0 || t[0] >= cols || t[1] >= rows) continue;
            const int d = depth[(size_t)t[1] * stride + t[0]];
            if (d != 0 && d < t[2]) code += 1 << j;
        }
        codes[f] = (uint8_t)code;
    }
}

int rc_dissimilarity(const uint8_t *a, const uint8_t *b, int n_ferns)
{
    int d = 0;
    for (int f = 0; f < n_ferns; ++f) d += a[f] != b[f];
    return d;
}

/* the lookup (k candidates, index -1 / dissimilarity n_ferns + 1 past the count) and, when append, the harvest; returns 1 when the frame
 * was appended (db then holds it at row `*count`, and *count grows) */
int rc_match(uint8_t *db, int *count, int capacity, const uint8_t *code, int n_ferns, int k, int harvest, int append, int *index, int *dis)
{
    for (int r = 0; r < k; ++r) { index[r] = -1; dis[r] = n_ferns + 1; }
    for (int i = 0; i < *count; ++i) {
        const int d = rc_dissimilarity(db + (size_t)i * n_ferns, code, n_ferns);
        /* insertion into the ranked list: strictly smaller dissimilarity goes first, ties keep the lower index first */
        int r = k;
        while (r > 0 && (index[r - 1] < 0 || d < dis[r - 1])) --r;
        if (r >= k) continue;
        for (int q = k - 1; q > r; --q) { index[q] = index[q - 1]; dis[q] = dis[q - 1]; }
        index[r] = i; dis[r] = d;
    }
    const int add = append && *count < capacity && (*count == 0 || dis[0] > harvest);
    if (add) {
        memcpy(db + (size_t)*count * n_ferns, code, (size_t)n_ferns);
        ++*count;
    }
    return add;
}

/* the gate's counts at one level, in double: vertex and normal maps dense float4 rows x cols; T 12 floats (R row-major, t).
 * out_counts: n_valid, n_in, n_ambiguous; *sum_sq the double sum of r^2 over the associated pixels.  A pixel is ambiguous when a float
 * evaluation could decide one of its tests the other way: its squared distance or its |cosine| within 1e-5 relative of the threshold, or
 * a projected coordinate within 1e-5 relative of a pixel boundary (the sampled pixel) */
void rc_gate(const float *vc, const float *nc, const float *vp, const float *np, int cols, int rows, float fx, float fy, float cx, float cy,
             const float *T, float dist_thres, float angle_thres, int *out_counts, double *sum_sq)
{
    const double dist2 = (double)(dist_thres * dist_thres), min_cos = (double)cosf(angle_thres);
    int n_valid = 0, n_in = 0, n_amb = 0;
    double sum = 0.0;
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x) {
            const float *v = vc + ((size_t)y * cols + x) * 4, *n = nc + ((size_t)y * cols + x) * 4;
            if (isnan(v[0])) continue;
            ++n_valid;
            double s[3], ns[3];
            for (int i = 0; i < 3; ++i) {
                s[i] = (double)T[3 * i] * v[0] + (double)T[3 * i + 1] * v[1] + (double)T[3 * i + 2] * v[2] + T[9 + i];
                ns[i] = (double)T[3 * i] * n[0] + (double)T[3 * i + 1] * n[1] + (double)T[3 * i + 2] * n[2];
            }
            if (s[2] <= 0) continue;
            const double u = fx * (s[0] / s[2]) + cx, w = fy * (s[1] / s[2]) + cy;
            int amb = 0;
            const double fu = u - floor(u), fw = w - floor(w), tol_u = 1e-5 * (fabs(u) + 1.0), tol_w = 1e-5 * (fabs(w) + 1.0);
            if (fu < tol_u || 1.0 - fu < tol_u || fw < tol_w || 1.0 - fw < tol_w) amb = 1;
            if (!(u >= 0 && w >= 0 && u < cols && w < rows)) { n_amb += amb; continue; }
            const int iu = (int)u, iw = (int)w;
            const float *d = vp + ((size_t)iw * cols + iu) * 4, *nd = np + ((size_t)iw * cols + iu) * 4;
            if (isnan(d[0])) { n_amb += amb; continue; }
            const double df[3] = {s[0] - d[0], s[1] - d[1], s[2] - d[2]};
            const double dd = df[0] * df[0] + df[1] * df[1] + df[2] * df[2];
            if (fabs(dd - dist2) <= 1e-5 * dist2) amb = 1;
            const double c = fabs(ns[0] * nd[0] + ns[1] * nd[1] + ns[2] * nd[2]);
            if (fabs(c - min_cos) <= 1e-5) amb = 1;
            n_amb += amb;
            if (dd > dist2 || c < min_cos) continue;
            ++n_in;
            const double r = nd[0] * (d[0] - s[0]) + nd[1] * (d[1] - s[1]) + nd[2] * (d[2] - s[2]);
            sum += r * r;
        }
    out_counts[0] = n_valid; out_counts[1] = n_in; out_counts[2] = n_amb;
    *sum_sq = sum;
}

/* the gate's decision (DF_RELOC_MIN_VALID, DF_RELOC_MIN_INLIER_FRAC, DF_RELOC_MAX_RMS passed in) */
int rc_accepts(int ok, int n_valid, int n_in, double sum_sq, int min_valid, float min_frac, float max_rms)
{
    if (!ok || n_valid < min_valid || n_in < 1) return 0;
    if ((float)n_in < min_frac * (float)n_valid) return 0;
    return sqrt(sum_sq / n_in) <= (double)max_rms;
}
