/* mesh_oracle.c -- CPU restatement of the mesh extraction (dfusion.h df_mesh_*, csrc/mesh.cu) for the tests: a plain loop over the cubes in
 * the documented order.  Vertex indices come from a dense per-(voxel, axis) map of the cloud, numbered in the order the cloud extraction
 * emits its points (ascending (z, y, x), then +x, +y, +z) and under its conditions (orc_extract_cloud, oracle/orc_tsdf.c; the tests check
 * the map against that function's output point by point).  Built and loaded by tests/mesh_oracle.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include "df_mc_table.h"
#include "oracle_util.h"

static const signed char TRIS[256][DF_MC_ROW] = DF_MC_TRIANGLES_INIT;
static const signed char CORNER[8][3] = DF_MC_CORNER_INIT;
static const signed char OWNER[12][4] = DF_MC_EDGE_OWNER_INIT;

typedef struct { uint32_t *data; int dims[3]; } mo_volume;

/* a voxel takes part in extraction iff W != 0 && F != 1 */
static int active(uint32_t v, float *F)
{
    *F = half_to_float((uint16_t)(v & 0xffffu));
    return (v >> 16) != 0 && *F != 1.f;
}

/* map[3 * voxel + axis] = index of the cloud point that voxel emits on that axis, -1 where it emits none; returns the number of points */
long long mo_vertex_map(mo_volume vol, int32_t *map)
{
    const int Dx = vol.dims[0], Dy = vol.dims[1], Dz = vol.dims[2];
    const size_t sy = (size_t)Dx, sz = (size_t)Dx * Dy;
    long long count = 0;
    for (size_t i = 0; i < 3 * sz * (size_t)Dz; ++i) map[i] = -1;
    for (int z = 0; z < Dz - 1; ++z)
        for (int y = 0; y < Dy; ++y)
            for (int x = 0; x < Dx; ++x) {
                const size_t v = x + sy * y + sz * z;
                float F, Fn;
                if (!active(vol.data[v], &F)) continue;
                for (int axis = 0; axis < 3; ++axis) {
                    const int nx = x + (axis == 0), ny = y + (axis == 1), nz = z + (axis == 2);
                    if (nx >= Dx || ny >= Dy) continue;
                    if (!active(vol.data[nx + sy * ny + sz * nz], &Fn)) continue;
                    if (!((F > 0 && Fn < 0) || (F < 0 && Fn > 0))) continue;
                    map[3 * v + axis] = (int32_t)count++;
                }
            }
    return count;
}

/* the triangles (3 x int32 each, at most `capacity` written); returns their number, or -1 when the volume has not cloud_count points */
long long mo_mesh(mo_volume vol, long long cloud_count, int32_t *tris, long long capacity)
{
    const int Dx = vol.dims[0], Dy = vol.dims[1], Dz = vol.dims[2];
    const size_t sy = (size_t)Dx, sz = (size_t)Dx * Dy;
    int32_t *map = (int32_t *)malloc(3 * sz * (size_t)Dz * sizeof(int32_t));
    if (!map) return -1;
    if (mo_vertex_map(vol, map) != cloud_count) { free(map); return -1; }
    long long n = 0;
    for (int z = 0; z <= Dz - 3; ++z)
        for (int y = 0; y <= Dy - 2; ++y)
            for (int x = 0; x <= Dx - 2; ++x) {
                int cs = 0, ok = 1;
                for (int i = 0; i < 8 && ok; ++i) {
                    float F;
                    ok = active(vol.data[(x + CORNER[i][0]) + sy * (y + CORNER[i][1]) + sz * (z + CORNER[i][2])], &F) && (F < 0.f || F > 0.f);
                    if (F < 0.f) cs |= 1 << i;
                }
                if (!ok) continue;
                for (int k = 0; k < DF_MC_ROW && TRIS[cs][k] >= 0; k += 3) {
                    for (int m = 0; m < 3; ++m) {
                        const signed char *o = OWNER[TRIS[cs][k + m]];
                        const size_t v = (x + o[0]) + sy * (y + o[1]) + sz * (z + o[2]);
                        if (n < capacity) tris[3 * n + m] = map[3 * v + o[3]];
                    }
                    ++n;
                }
            }
    free(map);
    return n;
}
