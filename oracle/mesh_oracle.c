/* mesh_oracle.c — scalar C restatement of the meshing (DESIGN.md §24), the checker of gpm_tsdf_integrate and
 * gpm_mesh_extract.
 *
 * TEST INFRASTRUCTURE, never part of the product.  Same fp32 operations in the same order as gipuma_b200/csrc/gpm_mesh.cu;
 * compiled with -fno-fast-math -ffp-contract=off like fusion_oracle.c, so every operation is one IEEE round-to-nearest step.
 * The extraction is written the other way round from the kernels: it walks the cubes and their tetrahedra in order, marks
 * the crossing edges of every meshed tetrahedron, numbers the marked edges in (point, direction) order, and walks the
 * tetrahedra again to emit the faces.
 */
#include "../include/gipuma_b200.h"

#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static const int PERM[6][3] = {{0, 1, 2}, {0, 2, 1}, {1, 0, 2}, {1, 2, 0}, {2, 0, 1}, {2, 1, 0}};
static const int DIR_MASK[7] = {1, 2, 4, 3, 5, 6, 7};          /* x, y, z, x+y, x+z, y+z, x+y+z */

static float centre(float o, int i, float s) { return o + ((float)i + 0.5f) * s; }

static float nan_bits(void)
{
    const uint32_t u = 0x7fffffffu;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

/* Voxels of z-slices k0 .. k1-1 of the box (D and Wt hold those slices only).  threads: OpenMP threads over slices. */
void gpo_tsdf(int n, int W, int H, const float* depth, const gpm_fuse_camera* cams, const float origin[3], float s,
              const int dims[3], float trunc, float dmin, float dmax, int k0, int k1, float* D, uint16_t* Wt, int threads)
{
    const int nx = dims[0], ny = dims[1];
    const size_t npix = (size_t)W * H;
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads > 0 ? threads : 1)
    for (int k = k0; k < k1; k++)
        for (int j = 0; j < ny; j++)
            for (int i = 0; i < nx; i++) {
                const float X[3] = {centre(origin[0], i, s), centre(origin[1], j, s), centre(origin[2], k, s)};
                float S = 0.f;
                int w = 0;
                for (int v = 0; v < n; v++) {
                    const float* P = cams[v].P;
                    float h[3];
                    for (int r = 0; r < 3; r++) h[r] = ((P[4 * r] * X[0] + P[4 * r + 1] * X[1]) + P[4 * r + 2] * X[2]) + P[4 * r + 3];
                    const float z = h[2];
                    if (!(z > 0.f)) continue;
                    const float u = floorf(h[0] / z + 0.5f), y = floorf(h[1] / z + 0.5f);
                    if (!(u >= 0.f && u < (float)W && y >= 0.f && y < (float)H)) continue;
                    const float d = depth[v * npix + (size_t)y * W + (size_t)u];
                    if (!(d > 0.f && d >= dmin && d <= dmax)) continue;
                    const float sdf = d - z;
                    if (sdf < -trunc) continue;
                    S = S + (sdf < trunc ? sdf : trunc) / trunc;
                    w++;
                }
                const size_t o = ((size_t)(k - k0) * ny + j) * nx + i;
                D[o] = w ? S / (float)w : nan_bits();
                Wt[o] = (uint16_t)w;
            }
}

typedef struct {
    const float* D;
    const uint16_t* Wt;
    int nx, ny, nz, minw;
    float o[3], s;
    uint8_t* mark;                                              /* per point: bit r = edge (p, direction r) is a vertex */
    int64_t* id;                                                /* per point: id of its first vertex */
} mo_vol;

static int64_t mo_index(const mo_vol* V, int i, int j, int k) { return ((int64_t)k * V->ny + j) * V->nx + i; }
static int mo_valid(const mo_vol* V, int64_t p) { return V->Wt[p] >= V->minw; }
static int mo_inside(const mo_vol* V, int64_t p) { return V->D[p] < 0.f; }

static int dir_of(int mask)
{
    for (int r = 0; r < 7; r++)
        if (DIR_MASK[r] == mask) return r;
    return -1;
}

/* corner masks of tetrahedron t in chain order */
static void tet(int t, int c[4])
{
    c[0] = 0;
    c[1] = 1 << PERM[t][0];
    c[2] = c[1] | 1 << PERM[t][1];
    c[3] = 7;
}

static int64_t corner(const mo_vol* V, int i, int j, int k, int m) { return mo_index(V, i + (m & 1), j + (m >> 1 & 1), k + (m >> 2 & 1)); }

/* inside bits (in chain order) of cube (i, j, k)'s tetrahedron t, or -1 if it is not meshed */
static int tet_inside(const mo_vol* V, int i, int j, int k, const int c[4])
{
    int in4 = 0;
    for (int r = 0; r < 4; r++) {
        const int64_t q = corner(V, i, j, k, c[r]);
        if (!mo_valid(V, q)) return -1;
        in4 |= mo_inside(V, q) << r;
    }
    return in4;
}

/* sign of the permutation seq of 0..3 */
static int parity4(const int seq[4])
{
    int inv = 0;
    for (int x = 0; x < 4; x++)
        for (int y = x + 1; y < 4; y++) inv += seq[x] > seq[y];
    return (inv & 1) ? -1 : 1;
}

static int perm_sign(int t)
{
    const int seq[4] = {PERM[t][0], PERM[t][1], PERM[t][2], 3};
    return parity4(seq);
}

/* vertex id of the edge between chain corners a < b of tetrahedron c of cube (i, j, k) */
static int64_t edge_id(const mo_vol* V, int i, int j, int k, const int c[4], int a, int b)
{
    const int64_t p = corner(V, i, j, k, c[a]);
    const int r = dir_of(c[b] ^ c[a]);
    int64_t id = V->id[p];
    for (int x = 0; x < r; x++) id += (V->mark[p] >> x) & 1;
    return id;
}

/* Marching tetrahedra.  Writes up to vcap vertices and fcap faces; *nv and *nf receive the counts.  Returns 0, or -1 when
 * out of memory. */
int gpo_mesh_extract(const float* D, const uint16_t* Wt, const int dims[3], const float origin[3], float s, int min_weight,
                     float* verts, int64_t vcap, int32_t* faces, int64_t fcap, int64_t* nv, int64_t* nf)
{
    mo_vol V = {D, Wt, dims[0], dims[1], dims[2], min_weight, {origin[0], origin[1], origin[2]}, s, NULL, NULL};
    const int64_t npts = (int64_t)V.nx * V.ny * V.nz;
    V.mark = (uint8_t*)calloc((size_t)npts, 1);
    V.id = (int64_t*)malloc(sizeof(int64_t) * (size_t)npts);
    if (!V.mark || !V.id) { free(V.mark);  free(V.id);  return -1; }
    /* mark the crossing edges of every meshed tetrahedron */
    for (int k = 0; k + 1 < V.nz; k++)
        for (int j = 0; j + 1 < V.ny; j++)
            for (int i = 0; i + 1 < V.nx; i++)
                for (int t = 0; t < 6; t++) {
                    int c[4];
                    tet(t, c);
                    const int in4 = tet_inside(&V, i, j, k, c);
                    if (in4 <= 0 || in4 == 15) continue;
                    for (int a = 0; a < 4; a++)
                        for (int b = a + 1; b < 4; b++)
                            if (((in4 >> a) & 1) != ((in4 >> b) & 1))
                                V.mark[corner(&V, i, j, k, c[a])] |= (uint8_t)(1u << dir_of(c[b] ^ c[a]));
                }
    /* number them and place the vertices */
    int64_t count = 0;
    for (int k = 0; k < V.nz; k++)
        for (int j = 0; j < V.ny; j++)
            for (int i = 0; i < V.nx; i++) {
                const int64_t p = mo_index(&V, i, j, k);
                V.id[p] = count;
                for (int r = 0; r < 7; r++) {
                    if (!((V.mark[p] >> r) & 1)) continue;
                    const int m = DIR_MASK[r];
                    const int c[3] = {i, j, k}, e[3] = {m & 1, m >> 1 & 1, m >> 2 & 1};
                    const int64_t q = mo_index(&V, i + e[0], j + e[1], k + e[2]);
                    const float t = D[p] / (D[p] - D[q]);
                    if (count < vcap)
                        for (int ax = 0; ax < 3; ax++) {
                            const float xp = centre(V.o[ax], c[ax], s), xq = centre(V.o[ax], c[ax] + e[ax], s);
                            verts[3 * count + ax] = xp + t * (xq - xp);
                        }
                    count++;
                }
            }
    *nv = count;
    /* faces, in (cube, tetrahedron) order */
    int64_t f = 0;
#define PUT(x, y, z)                                                                                       \
    do {                                                                                                   \
        if (f < fcap) { faces[3 * f] = (int32_t)(x);  faces[3 * f + 1] = (int32_t)(y);  faces[3 * f + 2] = (int32_t)(z); } \
        f++;                                                                                               \
    } while (0)
    for (int k = 0; k + 1 < V.nz; k++)
        for (int j = 0; j + 1 < V.ny; j++)
            for (int i = 0; i + 1 < V.nx; i++)
                for (int t = 0; t < 6; t++) {
                    int c[4];
                    tet(t, c);
                    const int in4 = tet_inside(&V, i, j, k, c);
                    if (in4 <= 0 || in4 == 15) continue;
                    int in[4], out[4], ki = 0, ko = 0;
                    for (int r = 0; r < 4; r++) {
                        if ((in4 >> r) & 1) in[ki++] = r;
                        else out[ko++] = r;
                    }
#define E(a, b) ((a) < (b) ? edge_id(&V, i, j, k, c, a, b) : edge_id(&V, i, j, k, c, b, a))
                    if (ki == 1 || ki == 3) {
                        /* the lone corner and the other three in chain order; the triangle faces away from an inside
                           lone corner and towards an outside one */
                        const int lone = ki == 1 ? in[0] : out[0];
                        int o[3], n = 0;
                        for (int r = 0; r < 4; r++)
                            if (r != lone) o[n++] = r;
                        const int seq[4] = {lone, o[0], o[1], o[2]};
                        const int away = perm_sign(t) * parity4(seq) > 0;
                        if ((ki == 1) == away) PUT(E(lone, o[0]), E(lone, o[1]), E(lone, o[2]));
                        else PUT(E(lone, o[0]), E(lone, o[2]), E(lone, o[1]));
                    } else {
                        const int seq[4] = {in[0], in[1], out[0], out[1]};
                        const int64_t q0 = E(in[0], out[0]), q1 = E(in[0], out[1]), q2 = E(in[1], out[1]), q3 = E(in[1], out[0]);
                        if (perm_sign(t) * parity4(seq) > 0) { PUT(q0, q1, q2);  PUT(q0, q2, q3); }
                        else { PUT(q0, q3, q2);  PUT(q0, q2, q1); }
                    }
#undef E
                }
#undef PUT
    *nf = f;
    free(V.mark);
    free(V.id);
    return 0;
}
