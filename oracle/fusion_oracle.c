/* fusion_oracle.c — scalar C restatement of the depth-map fusion (DESIGN.md §12), the checker of gpm_fuse.
 *
 * TEST INFRASTRUCTURE, never part of the product.  Same fp32 operations in the same order as gipuma_b200/csrc/gpm_fuse.cu;
 * compiled with -fno-fast-math -ffp-contract=off, so every operation is one IEEE round-to-nearest step, like the kernels'
 * explicit __f*_rn intrinsics.  A pass is computed in two steps: the candidate vertex of every pixel (rows in parallel when
 * OpenMP is there; the result does not depend on it), then emission and marking in (y, x) order on one thread.
 */
#include "../include/gipuma_b200.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    const float* norm4;
    const float* images;
    int n, W, H, channels;
    float dmin, dmax, disp_thresh, cos_thresh;
    const gpm_fuse_camera* cams;
} fo_args;

static float fo_dot3(const float* a, float x, float y, float z) { return (a[0] * x + a[1] * y) + a[2] * z; }

static void fo_backproject(const gpm_fuse_camera* c, float x, float y, float d, float X[3])
{
    const float a = d * x - c->P[3], b = d * y - c->P[7], e = d - c->P[11];
    for (int i = 0; i < 3; i++) X[i] = fo_dot3(c->M_inv + 3 * i, a, b, e);
}

/* target pixel of view j consistent with (X, n), or -1; u, v: its coordinates */
static long fo_consistent(const fo_args* A, int j, const float X[3], const float* n, const float** tgt, float* u, float* v)
{
    const gpm_fuse_camera* c = A->cams + j;
    const float hx = fo_dot3(c->P, X[0], X[1], X[2]) + c->P[3];
    const float hy = fo_dot3(c->P + 4, X[0], X[1], X[2]) + c->P[7];
    const float hz = fo_dot3(c->P + 8, X[0], X[1], X[2]) + c->P[11];
    if (!(hz > 0.f)) return -1;
    const float fu = floorf(hx / hz + 0.5f), fv = floorf(hy / hz + 0.5f);
    if (!(fu >= 0.f && fu < (float)A->W && fv >= 0.f && fv < (float)A->H)) return -1;
    const long q = (long)fv * A->W + (long)fu;
    const float* t = A->norm4 + ((size_t)j * A->W * A->H + q) * 4;
    if (!(t[3] >= A->dmin && t[3] <= A->dmax)) return -1;
    const float fb = c->f * 0.54f;
    if (!(fabsf(fb / hz - fb / t[3]) < A->disp_thresh)) return -1;
    if (!((n[0] * t[0] + n[1] * t[1]) + n[2] * t[2] > A->cos_thresh)) return -1;
    *tgt = t;  *u = fu;  *v = fv;
    return q;
}

static void fo_colour(const fo_args* A, int view, long q, float s[3])
{
    if (!A->images) return;
    const size_t i = (size_t)view * A->W * A->H + q;
    if (A->channels == 1) {
        const float g = A->images[i];
        s[0] = s[0] + g;  s[1] = s[1] + g;  s[2] = s[2] + g;
    } else {
        const float* c = A->images + 4 * i;
        s[0] = s[0] + c[0];  s[1] = s[1] + c[1];  s[2] = s[2] + c[2];
    }
}

static unsigned char fo_uchar(float s, float cnt)
{
    float m = s / cnt;
    m = m >= 0.f ? (m <= 255.f ? m : 255.f) : 0.f;
    return (unsigned char)floorf(m + 0.5f);
}

/* Pixel p of view r as a reference (its used mark aside): returns the number of consistent views (-1: depth out of range)
 * and, when `out` is given and at least num_consistent views are consistent, writes the packed vertex. */
static int fo_vertex(const fo_args* A, int r, long p, int num_consistent, unsigned char* out)
{
    const float* n = A->norm4 + ((size_t)r * A->W * A->H + p) * 4;
    if (!(n[3] >= A->dmin && n[3] <= A->dmax)) return -1;
    float X[3], s[3], sn[3] = {n[0], n[1], n[2]}, col[3] = {0.f, 0.f, 0.f};
    fo_backproject(A->cams + r, (float)(p % A->W), (float)(p / A->W), n[3], X);
    s[0] = X[0];  s[1] = X[1];  s[2] = X[2];
    fo_colour(A, r, p, col);
    int cnt = 0;
    for (int j = 0; j < A->n; j++) {
        if (j == r) continue;
        const float* t;
        float u, v, Xj[3];
        const long q = fo_consistent(A, j, X, n, &t, &u, &v);
        if (q < 0) continue;
        fo_backproject(A->cams + j, u, v, t[3], Xj);
        for (int k = 0; k < 3; k++) s[k] = s[k] + Xj[k];
        for (int k = 0; k < 3; k++) sn[k] = sn[k] + t[k];
        fo_colour(A, j, q, col);
        cnt++;
    }
    if (!out || cnt < num_consistent) return cnt;
    const float m = (float)(cnt + 1);
    const float len = sqrtf((sn[0] * sn[0] + sn[1] * sn[1]) + sn[2] * sn[2]);
    float v[6] = {s[0] / m, s[1] / m, s[2] / m, 0.f, 0.f, 0.f};
    if (len > 0.f)
        for (int k = 0; k < 3; k++) v[3 + k] = sn[k] / len;
    memcpy(out, v, 24);                                         /* little-endian host, like the PLY */
    for (int k = 0; k < 3; k++) out[24 + k] = A->images ? fo_uchar(col[k], m) : 0;
    return cnt;
}

/* Passes r0 .. r1-1 of the fusion, starting from the masks in `used` (n*H*W bytes, updated in place).  Writes up to
 * `capacity` vertices and (view, pixel) sources; returns the number of vertices emitted.  `threads`: OpenMP threads of the
 * candidate step. */
long long gpo_fuse(int n, int W, int H, const float* norm4, const float* images, int channels, const gpm_fuse_camera* cams,
                   float depth_min, float depth_max, float disp_thresh, float normal_thresh, int num_consistent, int r0, int r1,
                   unsigned char* used, unsigned char* vertices, int* source, long long capacity, int threads)
{
    fo_args A = {norm4, images, n, W, H, channels, depth_min, depth_max, disp_thresh,
                 (float)cos((double)normal_thresh * M_PI / 180.0), cams};
    const long npix = (long)W * H;
    int* cnt = (int*)malloc(sizeof(int) * npix);
    long long total = 0;
    for (int r = r0; r < r1; r++) {
        const unsigned char* ur = used + (size_t)r * npix;
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads > 0 ? threads : 1)
        for (int y = 0; y < H; y++)
            for (long p = (long)y * W; p < (long)(y + 1) * W; p++)
                cnt[p] = ur[p] ? -1 : fo_vertex(&A, r, p, num_consistent, NULL);
        for (long p = 0; p < npix; p++) {
            if (cnt[p] < num_consistent) continue;
            if (total < capacity) {
                if (vertices) fo_vertex(&A, r, p, num_consistent, vertices + total * GPM_FUSE_VERTEX_BYTES);
                if (source) { source[2 * total] = r;  source[2 * total + 1] = (int)p; }
            }
            total++;
            const float* nr = norm4 + ((size_t)r * npix + p) * 4;
            float X[3];
            fo_backproject(cams + r, (float)(p % W), (float)(p / W), nr[3], X);
            used[(size_t)r * npix + p] = 1;
            for (int j = 0; j < n; j++) {
                if (j == r) continue;
                const float* t;
                float u, v;
                const long q = fo_consistent(&A, j, X, nr, &t, &u, &v);
                if (q >= 0) used[(size_t)j * npix + q] = 1;
            }
        }
    }
    free(cnt);
    return total;
}
