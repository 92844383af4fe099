/* fusion_rule_oracle.c — scalar C restatement of the depth-map fusion under either consistency rule (DESIGN.md §12, §22),
 * the checker of gpm_fuse_with_rule.
 *
 * TEST INFRASTRUCTURE, never part of the product.  It builds on fusion_oracle.c (included: cameras, back-projection, colour)
 * and restates the passes with the rule-aware test; with GPM_FUSE_DISPARITY it computes what gpo_fuse computes.  Compiled
 * like fusion_oracle.c (-fno-fast-math -ffp-contract=off): every operation one IEEE round-to-nearest step, in the order of
 * gipuma_b200/csrc/gpm_fuse.cu.
 */
#include "fusion_oracle.c"

typedef struct {
    fo_args A;
    int kind;
    float reproj_px, depth_rel;
} fr_args;

/* target pixel of view j consistent with reference pixel (x, y) of view r (depth dr, point X, normal n), or -1 */
static long fr_consistent(const fr_args* R, int r, float x, float y, float dr, int j, const float X[3], const float* n,
                          const float** tgt, float* u, float* v)
{
    const fo_args* A = &R->A;
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
    if (R->kind == GPM_FUSE_DISPARITY) {
        const float fb = c->f * 0.54f;
        if (!(fabsf(fb / hz - fb / t[3]) < A->disp_thresh)) return -1;
    } else {
        const gpm_fuse_camera* cr = A->cams + r;
        float Xj[3];
        fo_backproject(c, fu, fv, t[3], Xj);
        const float gx = fo_dot3(cr->P, Xj[0], Xj[1], Xj[2]) + cr->P[3];
        const float gy = fo_dot3(cr->P + 4, Xj[0], Xj[1], Xj[2]) + cr->P[7];
        const float gz = fo_dot3(cr->P + 8, Xj[0], Xj[1], Xj[2]) + cr->P[11];
        if (!(gz > 0.f)) return -1;
        const float dx = gx / gz - x, dy = gy / gz - y;
        if (!(sqrtf(dx * dx + dy * dy) < R->reproj_px)) return -1;
        if (!(fabsf(gz - dr) / dr < R->depth_rel)) return -1;
    }
    if (!((n[0] * t[0] + n[1] * t[1]) + n[2] * t[2] > A->cos_thresh)) return -1;
    *tgt = t;  *u = fu;  *v = fv;
    return q;
}

/* fo_vertex under the rule */
static int fr_vertex(const fr_args* R, int r, long p, int num_consistent, unsigned char* out)
{
    const fo_args* A = &R->A;
    const float* n = A->norm4 + ((size_t)r * A->W * A->H + p) * 4;
    if (!(n[3] >= A->dmin && n[3] <= A->dmax)) return -1;
    const float x = (float)(p % A->W), y = (float)(p / A->W);
    float X[3], s[3], sn[3] = {n[0], n[1], n[2]}, col[3] = {0.f, 0.f, 0.f};
    fo_backproject(A->cams + r, x, y, n[3], X);
    s[0] = X[0];  s[1] = X[1];  s[2] = X[2];
    fo_colour(A, r, p, col);
    int cnt = 0;
    for (int j = 0; j < A->n; j++) {
        if (j == r) continue;
        const float* t;
        float u, v, Xj[3];
        const long q = fr_consistent(R, r, x, y, n[3], j, X, n, &t, &u, &v);
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

/* gpo_fuse under the rule `kind` (GPM_FUSE_DISPARITY: reproj_px and depth_rel are not read; GPM_FUSE_REPROJECTION:
 * disp_thresh is not read). */
long long gpo_fuse_rule(int n, int W, int H, const float* norm4, const float* images, int channels, const gpm_fuse_camera* cams,
                        float depth_min, float depth_max, float disp_thresh, float normal_thresh, int num_consistent, int kind,
                        float reproj_px, float depth_rel, int r0, int r1, unsigned char* used, unsigned char* vertices,
                        int* source, long long capacity, int threads)
{
    fr_args R = {{norm4, images, n, W, H, channels, depth_min, depth_max, disp_thresh,
                  (float)cos((double)normal_thresh * M_PI / 180.0), cams}, kind, reproj_px, depth_rel};
    const long npix = (long)W * H;
    int* cnt = (int*)malloc(sizeof(int) * npix);
    long long total = 0;
    for (int r = r0; r < r1; r++) {
        const unsigned char* ur = used + (size_t)r * npix;
#pragma omp parallel for schedule(dynamic, 1) num_threads(threads > 0 ? threads : 1)
        for (int y = 0; y < H; y++)
            for (long p = (long)y * W; p < (long)(y + 1) * W; p++)
                cnt[p] = ur[p] ? -1 : fr_vertex(&R, r, p, num_consistent, NULL);
        for (long p = 0; p < npix; p++) {
            if (cnt[p] < num_consistent) continue;
            if (total < capacity) {
                if (vertices) fr_vertex(&R, r, p, num_consistent, vertices + total * GPM_FUSE_VERTEX_BYTES);
                if (source) { source[2 * total] = r;  source[2 * total + 1] = (int)p; }
            }
            total++;
            const float* nr = norm4 + ((size_t)r * npix + p) * 4;
            const float x = (float)(p % W), y = (float)(p / W);
            float X[3];
            fo_backproject(cams + r, x, y, nr[3], X);
            used[(size_t)r * npix + p] = 1;
            for (int j = 0; j < n; j++) {
                if (j == r) continue;
                const float* t;
                float u, v;
                const long q = fr_consistent(&R, r, x, y, nr[3], j, X, nr, &t, &u, &v);
                if (q >= 0) used[(size_t)j * npix + q] = 1;
            }
        }
    }
    free(cnt);
    return total;
}
