// gpm_host.cpp — host-side callers and data formats either side of the hot path (SURVEY.md §8f, rows f1-f3), plain C++,
// no OpenCV, no CUDA.  C-ABI declared in include/gipuma_b200.h.
//   f1  gpm_prepare_cameras   cameraGeometryUtils.h:174-353  P -> K,R,t (RQ), re-base on the reference, Camera_cu fields
//   f2  gpm_select_views      main.cpp:430-499               angle filter on the central rays (deterministic) + depth range
//   f3  gpm_write_dmb / gpm_read_dmb   fileIoUtils.h:247-368 depth / normal maps for the external `fusibile` fusion
#include "../../include/gipuma_b200.h"

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {

struct M3 { double m[9]; };
struct V3 { double v[3]; };

M3 mul(const M3& a, const M3& b)
{
    M3 r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
    return r;
}
V3 mulv(const M3& a, const V3& x)
{
    V3 r;
    for (int i = 0; i < 3; i++) r.v[i] = a.m[3 * i] * x.v[0] + a.m[3 * i + 1] * x.v[1] + a.m[3 * i + 2] * x.v[2];
    return r;
}
double det(const M3& a)
{
    const double* m = a.m;
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}
M3 inv(const M3& a)
{
    const double* m = a.m;
    const double d = det(a);
    M3 r;
    r.m[0] = (m[4] * m[8] - m[5] * m[7]) / d;  r.m[1] = (m[2] * m[7] - m[1] * m[8]) / d;  r.m[2] = (m[1] * m[5] - m[2] * m[4]) / d;
    r.m[3] = (m[5] * m[6] - m[3] * m[8]) / d;  r.m[4] = (m[0] * m[8] - m[2] * m[6]) / d;  r.m[5] = (m[2] * m[3] - m[0] * m[5]) / d;
    r.m[6] = (m[3] * m[7] - m[4] * m[6]) / d;  r.m[7] = (m[1] * m[6] - m[0] * m[7]) / d;  r.m[8] = (m[0] * m[4] - m[1] * m[3]) / d;
    return r;
}
M3 transpose(const M3& a)
{
    M3 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * j + i];
    return r;
}

// RQ decomposition M = K R (K upper triangular with positive diagonal, R a rotation) by Givens rotations — the role
// cv::decomposeProjectionMatrix / RQDecomp3x3 plays at cameraGeometryUtils.h:252.
void rq3(const M3& M, M3& K, M3& R)
{
    M3 A = M, Q = {{1, 0, 0, 0, 1, 0, 0, 0, 1}};
    auto givens = [&](int col_a, int col_b, int row) {         // rotate columns a, b so that A[row][a] becomes 0
        const double x = A.m[3 * row + col_a], y = A.m[3 * row + col_b];
        const double n = std::sqrt(x * x + y * y);
        if (n == 0) return;
        const double c = y / n, s = x / n;
        M3 G = {{1, 0, 0, 0, 1, 0, 0, 0, 1}};
        G.m[3 * col_a + col_a] = c;  G.m[3 * col_a + col_b] = s;
        G.m[3 * col_b + col_a] = -s; G.m[3 * col_b + col_b] = c;
        A = mul(A, G);
        Q = mul(transpose(G), Q);
    };
    givens(1, 2, 2);      // A[2][1] = 0
    givens(0, 2, 2);      // A[2][0] = 0
    givens(0, 1, 1);      // A[1][0] = 0
    for (int i = 0; i < 3; i++)                                 // make the diagonal of K positive
        if (A.m[3 * i + i] < 0) {
            for (int r = 0; r < 3; r++) A.m[3 * r + i] = -A.m[3 * r + i];
            for (int c = 0; c < 3; c++) Q.m[3 * i + c] = -Q.m[3 * i + c];
        }
    K = A;
    R = Q;
}

void store9(float* dst, const M3& a) { for (int i = 0; i < 9; i++) dst[i] = (float)a.m[i]; }

void view_vector(const gpm_camera& c, double x, double y, double v[3])     // cameraGeometryUtils.h:68-77
{
    const double p[3] = {x - c.P_col34[0], y - c.P_col34[1], 1.0 - c.P_col34[2]};
    double n = 0;
    for (int i = 0; i < 3; i++) {
        v[i] = c.M_inv[3 * i] * p[0] + c.M_inv[3 * i + 1] * p[1] + c.M_inv[3 * i + 2] * p[2] - c.C[i];
        n += v[i] * v[i];
    }
    n = std::sqrt(n);
    for (int i = 0; i < 3; i++) v[i] /= n;
}

}  // namespace

// P: n row-major 3x4 projection matrices (doubles), index 0 = reference view.  cam_scale as --cam_scale (K divided by it).
extern "C" int gpm_prepare_cameras(const double* P, int n, double cam_scale, gpm_camera* out)
{
    if (!P || !out || n < 1 || !(cam_scale > 0)) return GPM_E_ARG;
    std::vector<M3> K(n), R(n);
    std::vector<V3> t(n);
    for (int i = 0; i < n; i++) {
        const double* p = P + 12 * i;
        double sgn = 1.0;
        M3 M = {{p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]}};
        if (det(M) < 0) { sgn = -1.0;  for (double& v : M.m) v = -v; }
        rq3(M, K[i], R[i]);
        const double k22 = K[i].m[8];
        for (double& v : K[i].m) v /= k22;
        const V3 p4 = {{sgn * p[3], sgn * p[7], sgn * p[11]}};
        const V3 C = mulv(inv(M), V3{{-p4.v[0], -p4.v[1], -p4.v[2]}});          // camera centre
        const V3 rc = mulv(R[i], C);
        t[i] = V3{{-rc.v[0], -rc.v[1], -rc.v[2]}};                               // t = -R C (:260)
    }
    auto scaleK = [&](M3 k) { k.m[0] /= cam_scale;  k.m[4] /= cam_scale;  k.m[2] /= cam_scale;  k.m[5] /= cam_scale;  return k; };   // :136-147
    const M3 Kref = scaleK(K[0]);
    // transform = [R0 | t0]^-1 (:282-283): X_new = R0 X + t0
    const M3 R0T = transpose(R[0]);
    for (int i = 0; i < n; i++) {
        const M3 Rn = mul(R[i], R0T);                                             // rotation part of [Ri|ti] * [R0|t0]^-1
        const V3 rt0 = mulv(Rn, t[0]);
        const V3 tn = {{t[i].v[0] - rt0.v[0], t[i].v[1] - rt0.v[1], t[i].v[2] - rt0.v[2]}};
        const M3 Mn = mul(Kref, Rn);                                              // P = Kref [Rn | tn] (:124)
        const V3 p4 = mulv(Kref, tn);
        const M3 Minv = inv(Mn);
        const V3 C = mulv(Minv, V3{{-p4.v[0], -p4.v[1], -p4.v[2]}});
        gpm_camera& c = out[i];
        memset(&c, 0, sizeof(c));
        const M3 Ki = scaleK(K[i]);
        store9(c.K, Ki);  store9(c.K_inv, inv(Ki));  store9(c.R, Rn);  store9(c.M_inv, Minv);  store9(c.R_orig_inv, inv(R[i]));
        for (int k = 0; k < 3; k++) { c.t[k] = (float)tn.v[k];  c.C[k] = (float)C.v[k];  c.P_col34[k] = (float)p4.v[k]; }
        c.fx = (float)Kref.m[0];  c.fy = (float)Kref.m[4];  c.f = (float)Kref.m[0];
        c.alpha = c.fx / c.fy;                                                    // :318
        c.baseline = 0.54f;                                                       // :305
    }
    return GPM_OK;
}

// The fusion's cameras: the same decomposition as above without the re-basing (transformP = false), each view with its own
// scaled K — the camera its depth map was computed with when it was the reference view.
extern "C" int gpm_fuse_cameras(const double* P, int n, double cam_scale, gpm_fuse_camera* out)
{
    if (!P || !out || n < 1 || !(cam_scale > 0)) return GPM_E_ARG;
    for (int i = 0; i < n; i++) {
        const double* p = P + 12 * i;
        double sgn = 1.0;
        M3 M = {{p[0], p[1], p[2], p[4], p[5], p[6], p[8], p[9], p[10]}};
        if (det(M) < 0) { sgn = -1.0;  for (double& v : M.m) v = -v; }
        if (det(M) == 0) return GPM_E_ARG;
        M3 K, R;
        rq3(M, K, R);
        const double k22 = K.m[8];
        for (double& v : K.m) v /= k22;
        K.m[0] /= cam_scale;  K.m[4] /= cam_scale;  K.m[2] /= cam_scale;  K.m[5] /= cam_scale;
        const V3 p4 = {{sgn * p[3], sgn * p[7], sgn * p[11]}};
        const V3 C = mulv(inv(M), V3{{-p4.v[0], -p4.v[1], -p4.v[2]}});
        const V3 rc = mulv(R, C);
        const V3 t = {{-rc.v[0], -rc.v[1], -rc.v[2]}};
        const M3 Mn = mul(K, R);
        const V3 col = mulv(K, t);
        gpm_fuse_camera& c = out[i];
        store9(c.M_inv, inv(Mn));
        for (int r = 0; r < 3; r++) {
            for (int k = 0; k < 3; k++) c.P[4 * r + k] = (float)Mn.m[3 * r + k];
            c.P[4 * r + 3] = (float)col.v[r];
        }
        c.f = (float)K.m[0];
    }
    return GPM_OK;
}

// Deterministic selectViews (main.cpp:430-499): cameras whose central ray makes an angle in (min_angle, max_angle) degrees
// with the reference's; at most max_views of them, in index order (the reference shuffles with srand(time(0)) instead).
// depth_range[0..1] receives the min/max depth estimate of main.cpp:470-474 (or is left untouched if NULL).
extern "C" int gpm_select_views(const gpm_camera* cams, int n, int cols, int rows, float min_angle, float max_angle,
                                int max_views, int* subset, float* depth_range)
{
    if (!cams || !subset || n < 1) return GPM_E_ARG;
    const double x = cols / 2, y = rows / 2;
    double v0[3];
    view_vector(cams[0], x, y, v0);
    const double lo = min_angle * M_PI / 180.0, hi = max_angle * M_PI / 180.0;
    float min_depth = 9999.f, max_depth = 0.f;
    int count = 0;
    for (int i = 1; i < n; i++) {
        double v[3];
        view_vector(cams[i], x, y, v);
        double d = v0[0] * v[0] + v0[1] * v[1] + v0[2] * v[2];
        d = d > 1 ? 1 : (d < -1 ? -1 : d);
        const double angle = std::acos(d);
        if (angle > lo && angle < hi) {
            double b = 0;
            for (int k = 0; k < 3; k++) b += (double)(cams[0].C[k] - cams[i].C[k]) * (cams[0].C[k] - cams[i].C[k]);
            b = std::sqrt(b);
            const float min_range = (float)((b / 2.0) / std::sin(hi / 2.0)), max_range = (float)((b / 2.0) / std::sin(lo / 2.0));
            if (min_range < min_depth) min_depth = min_range;
            if (max_range > max_depth) max_depth = max_range;
            if (count < max_views) subset[count++] = i;
        }
    }
    if (depth_range) { depth_range[0] = min_depth;  depth_range[1] = max_depth; }
    return count;
}

// .dmb: int32 type (1 = float), int32 h, int32 w, int32 channels, then h*w*channels floats row-major (fileIoUtils.h:320-368).
extern "C" int gpm_write_dmb(const char* path, const float* data, int rows, int cols, int channels)
{
    if (!path || !data || rows < 1 || cols < 1 || channels < 1) return GPM_E_ARG;
    FILE* f = fopen(path, "wb");
    if (!f) return GPM_E_ARG;
    const int32_t hdr[4] = {1, rows, cols, channels};
    const size_t n = (size_t)rows * cols * channels;
    const bool ok = fwrite(hdr, sizeof(int32_t), 4, f) == 4 && fwrite(data, sizeof(float), n, f) == n;
    fclose(f);
    return ok ? GPM_OK : GPM_E_ARG;
}

extern "C" int gpm_read_dmb(const char* path, float* data, size_t capacity_floats, int* rows, int* cols, int* channels)
{
    if (!path || !rows || !cols || !channels) return GPM_E_ARG;
    FILE* f = fopen(path, "rb");
    if (!f) return GPM_E_ARG;
    int32_t hdr[4] = {-1, 0, 0, 0};
    if (fread(hdr, sizeof(int32_t), 4, f) != 4 || hdr[0] != 1) { fclose(f);  return GPM_E_ARG; }     // only float is supported (:262-266)
    *rows = hdr[1];  *cols = hdr[2];  *channels = hdr[3];
    const size_t n = (size_t)hdr[1] * hdr[2] * hdr[3];
    int rc = GPM_OK;
    if (data) rc = (n <= capacity_floats && fread(data, sizeof(float), n, f) == n) ? GPM_OK : GPM_E_ARG;
    fclose(f);
    return rc;
}

// Depth map (1 channel) and world-normal map (3 channels) of a finished run in the layout the reference writes next to
// its results for fusibile (main.cpp:1040-1070 -> writeDmb / writeDmbNormal).  norm4: rows*cols*4 (gpm_get_state).
extern "C" int gpm_write_result_dmb(const char* depth_path, const char* normal_path, const float* norm4, int rows, int cols)
{
    if (!norm4) return GPM_E_ARG;
    const size_t n = (size_t)rows * cols;
    std::vector<float> d(n), nm(3 * n);
    for (size_t i = 0; i < n; i++) {
        d[i] = norm4[4 * i + 3];
        nm[3 * i] = norm4[4 * i];  nm[3 * i + 1] = norm4[4 * i + 1];  nm[3 * i + 2] = norm4[4 * i + 2];
    }
    int rc = GPM_OK;
    if (depth_path) rc = gpm_write_dmb(depth_path, d.data(), rows, cols, 1);
    if (rc == GPM_OK && normal_path) rc = gpm_write_dmb(normal_path, nm.data(), rows, cols, 3);
    return rc;
}

// Point cloud in the layout storePlyFileBinary writes (displayUtils.h:84-142), with the real vertex count in the header.
extern "C" int gpm_write_ply(const char* path, const unsigned char* vertices, long long count)
{
    if (!path || count < 0 || (count > 0 && !vertices)) return GPM_E_ARG;
    FILE* f = fopen(path, "wb");
    if (!f) return GPM_E_ARG;
    fprintf(f, "ply\nformat binary_little_endian 1.0\nelement vertex %lld\n"
               "property float x\nproperty float y\nproperty float z\n"
               "property float nx\nproperty float ny\nproperty float nz\n"
               "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n", count);
    const size_t n = (size_t)count * GPM_FUSE_VERTEX_BYTES;
    const bool ok = fwrite(vertices, 1, n, f) == n;
    return (fclose(f) == 0 && ok) ? GPM_OK : GPM_E_ARG;
}
