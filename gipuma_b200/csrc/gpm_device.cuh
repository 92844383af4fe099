// gpm_device.cuh — device code of the PatchMatch hot path (sm_90a, H100).
//
// What is computed is the reference's algorithm (kysucix/gipuma, gipuma.cu); how it is computed is not:
//   * one WARP per pixel instead of one thread per pixel: lanes own (view, sample) pairs of the
//     support window, so all 32 lanes of a texture instruction fall into one small source patch and a
//     hypothesis can be abandoned warp-uniformly (no divergence) as soon as an exact lower bound on its
//     final cost reaches the pixel's current cost;
//   * close (+-1 px), far (+-5 px) propagation and plane refinement of one checkerboard colour are fused
//     into ONE launch (legal: a colour only reads the other colour's planes — gipuma.cu:1439-1446,
//     1560-1567), the reference window is staged in shared memory once instead of three times;
//   * per-sample quantities that do not depend on the hypothesis or the view (support weight,
//     reference value, reference gradients) are computed once per pixel, not once per (hypothesis, view);
//   * candidate planes that are bit-identical to the current plane or to an already rejected candidate
//     are skipped (their cost is a pure function of (pixel, plane)).
// None of this changes a single output bit: per-view costs are accumulated by the same sequential
// FMA chain in the same sample order as gipuma.cu:633-677, and every floating-point operation below
// reproduces the operation the reference executes when compiled for sm_100a (nvcc 12.9, -O3 --use_fast_math), i.e. its
// SASS after ptxas' multiply-add fusion — explicit round-to-nearest, flush-to-zero intrinsics are used
// throughout so that neither nvcc nor ptxas can re-associate or re-fuse them.  The file:line comments
// name the reference statement each block follows.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace gpm {

#define GPM_MAXCOST 1000.0f                    // config.h:22
#define GPM_TILE 32                            // pixels per tile side (reference: 32x16 threads = 32x32 px of one colour)
#define GPM_DSTRIDE 33                         // row stride of the per-warp dissimilarity buffer (odd: conflict-free)
#define GPM_APRON 16                           // replicate-padding of the staged reference image (>= (GPM_MAX_BOX+1)/2)
#define GPM_FULL 0xffffffffu
#define GPM_MAX_ROUNDS 16
#define GPM_MEMO_REFINE 0x80000000u   // memo_mask bit: refseen[] is valid (bits 0..19: seen[] entries)
// Rounding variants (eval_plane's `rt`) of the 21 inlined call sites — 20 candidates in source order, then the refinement —
// of gipuma_black_cu / gipuma_red_cu in the reference build, for T = float and T = float4; black and red agree.  Read off
// the reference build with tools/fused_probe.py: e.g. site 9 of the float4 kernels rounds
// the X and Y rows of H x-term first and the Z row y-term first.
#define GPM_FUSED_SITES_FLOAT  {1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1}
#define GPM_FUSED_SITES_FLOAT4 {0, 0, 0, 0, 0, 0, 0, 0, 0, 9, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1}
#define GPM_PROV_UNKNOWN 0xff        // prov[]: cost of unknown rounding variant (else bit 0 = x-first, bit 1 = gradient folding)
#define GPM_PROV_NCC 0x10            // prov[]: an NCC cost (DESIGN.md §15), which has one rounding variant at every call site
#define GPM_PROV_JVS 0x20            // prov[]: a cost weighted by joint view selection (DESIGN.md §17): not a pure function of the plane

// ---- exact-arithmetic primitives -------------------------------------------------------------
// With --use_fast_math these lower to {mul,add,sub,fma}.rn.ftz.f32, which ptxas never fuses.
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float frcp(float a) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }      // MUFU.RCP
__device__ __forceinline__ float frsq(float a) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }    // MUFU.RSQ
__device__ __forceinline__ float fsqrt_(float a) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }   // MUFU.SQRT
__device__ __forceinline__ float fex2(float a) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a)); return r; }      // MUFU.EX2
__device__ __forceinline__ float fmin_(float a, float b) { float r; asm("min.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ float fmax_(float a, float b) { float r; asm("max.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b)); return r; }
// a.x*b.x + a.y*b.y + a.z*b.z as the reference evaluates it: (y-term) then fma(x-term) then fma(z-term)
__device__ __forceinline__ float dot3(float ax, float ay, float az, float bx, float by, float bz)
{
    return ffma(az, bz, ffma(ax, bx, fmul(ay, by)));
}

// ---- constant data ---------------------------------------------------------------------------
struct ViewCam {                // per source view: what getHomography_cu reads (gipuma.cu:339-356)
    float K[9];
    float R[9];
    float t[3];
};
#define GPM_VIEWCAM_FLOATS 21

struct RefCam {                 // reference camera (cameras[REFERENCE])
    float K_inv[9];
    float M_inv[9];
    float R_orig_inv[9];
    float P34[3];
    float C[3];
    float fx, alpha, K2, K5;    // K[2], K[5]: principal point
    float f, baseline;          // CameraParameters_cu::f (refinement, gipuma.cu:904), cameras[0].baseline
    float f_cam;                // cameras[0].f (initialisation, gipuma.cu:1031)
    float depthMin, depthMax;
};

struct KParams {
    int W, H, V;
    int rad;                    // window radius: (box-1)/2 in the sweeps (gipuma.cu:1474), box/2 at init (:1012)
    int nside, ns;              // samples per side (stride WIN_INCREMENT=2, gipuma.cu:28,633-634) and per window
    int halo;                   // (box+1)/2 = WIN_RADIUS (gipuma.cu:1844-1847)
    int tile_w;                 // 32 + 2*halo (SHARED_SIZE_W)
    int tile_stride;            // texels per row of the staged window in shared memory: tile_w rounded up to 16 (TMA box rows of 64-byte multiples)
    int tile_xo;                // texels between the start of the staged rows and the window's first column: the TMA box must start on a
                                // 16-byte boundary of the padded image, so it starts (16 - halo) mod 4 texels early (0 for float4 texels)
    int nrounds;                // sample rounds; after each one an exact lower bound of the final cost is tested
    unsigned char round_end[16];// cumulative sample count at the end of each round (whole window columns)
    int ns_pad;                 // ns rounded up to a multiple of 4
    int nwarps;
    float tau_color, tau_gradient, alpha, gamma;
    float min_disp, max_disp;
    int n_best, cost_comb;
    float good_factor;
    int prune, dedupe_self, dedupe_cand;
    int color;                  // 1: float4 (RGB) images — the reference's -color_processing path (T = float4)
    int memo;                   // 1: skip candidates / refinements already known to be rejected at this pixel (see k_sweep)
    int cost_variant;           // k_cost_eval: 0 = init/refine rounding, 1 = propagation rounding (see eval_plane)
    int ncand;                  // propagation candidates per pixel: 8 (close + far kernels) or 20 (fused kernel, gipuma.cu:1122-1351)
    unsigned char site[24];     // fused kernel: rounding variant (eval_plane's rt) of each inlined call site: 0..19 candidates, 20 refinement
    int cost_rt;                // k_cost_eval: full runtime variant (used when it has bits beyond cost_variant / grad_variant)
    int grad_variant;           // colour only: which of l1(gradX)/3, l1(gradY)/3 ptxas folded into the FMA (1 at initialisation)
    int rng_mode;
    int quadperm;               // 1: lanes of a sampling round are permuted so that every hardware quad (lanes 4q..4q+3) samples a 2x2 block
    unsigned char perm[GPM_MAX_ROUNDS][32];   // sample (relative to the round's first) evaluated by each lane; identity without quadperm
    RefCam ref;
};

// Geometric-consistency term (DESIGN.md §14): what the k_sweep / k_cost_eval variants with GEO = true read besides KParams.
// The per-view K, R and t are those of the photometric homography (ViewCam in shared memory).  The NCC variants read
// min_std (DESIGN.md §15) from here too: it fills the struct's tail padding, so the other kernels' parameters stay as they were.
struct GeoParams {
    const float* depth;         // [V][H][W] each source view's depth map, along that view's own optical axis
    const float* kinv;          // [V][9] K^-1 of each source view
    float Kref[9];              // the reference camera's K
    float weight, max_err;
    float min_std;              // NCC: a window whose weighted standard deviation is below this, in grey levels, costs 2
};

enum { ST_LAUNCH = 0, ST_HYP = 1, ST_SKIP = 2, ST_PRUNED = 3, ST_PAIRS = 4, ST_PAIRS_FULL = 5 };

// ---- per-warp scratch in shared memory -------------------------------------------------------
struct WarpScratch {
    float4* A;      // [ns_pad] per sample: x = float(p.x+i), y = float(p.y+j)   (pt = __int2float_rn, gipuma.cu:210-211)
                    //                      z = gx1 = right-left (:258),          w = gy1 = down-up (:259)
    float* left;    // [ns_pad] reference value at the sample          (leftValue, gipuma.cu:655)
    float* w;       // [ns_pad] support weight                         (weight_cu, gipuma.cu:186-193)
    float4* L4;     // colour mode: [ns_pad] reference RGB at the sample, [ns_pad] gx1 RGB, [ns_pad] gy1 RGB
    float4* GX4;
    float4* GY4;
    float* H;       // [V][12]  homographies of the current hypothesis (rows of 3, 16-byte aligned)
    float* D;       // [V][GPM_DSTRIDE] dissimilarities of the current round
    const unsigned char* perm;   // [GPM_MAX_ROUNDS][32] lane -> sample of the round (block-wide table in shared memory)
    float* a;       // NCC only: [ns_pad] a_s = w_s * r_s
    float* sums;    // NCC only: [4] the window's W = sum w_s, Sr = sum a_s, Srr = sum a_s * r_s (DESIGN.md §15)
};

// multiple of 4 floats so that every warp's block stays 16-byte aligned; ncc: the NCC variants' a_s and pixel sums;
// extra: floats a kernel variant keeps per warp after the common block (joint view selection's cost rows, jvs_floats)
__host__ __device__ inline int warp_scratch_floats(int ns_pad, int V, int color, bool ncc = false, int extra = 0)
{
    return ((6 * ns_pad + (color ? 12 * ns_pad : 0) + V * 12 + V * GPM_DSTRIDE + (ncc ? ns_pad + 4 : 0) + 3) & ~3) + ((extra + 3) & ~3);
}

__device__ __forceinline__ WarpScratch carve(float* base, int ns_pad, int V, int color, const unsigned char* perm, bool ncc = false)
{
    WarpScratch s;
    s.perm = perm;
    s.A = reinterpret_cast<float4*>(base);
    s.L4 = s.A + ns_pad;           s.GX4 = s.L4 + (color ? ns_pad : 0);      s.GY4 = s.GX4 + (color ? ns_pad : 0);
    float* f = base + 4 * ns_pad + (color ? 12 * ns_pad : 0);
    s.left = f;                    s.w = s.left + ns_pad;
    s.H = s.w + ns_pad;            s.D = s.H + V * 12;
    s.a = ncc ? s.D + V * GPM_DSTRIDE : nullptr;
    s.sums = ncc ? s.a + ns_pad : nullptr;
    return s;
}

// depth of plane (n, d) at pixel p — getDisparity_cu / getDepthFromPlane3_cu, gipuma.cu:694-715
__device__ __forceinline__ float plane_depth(const RefCam& c, float nx, float ny, float nz, float d, float px, float py)
{
    if (d != d) return 1000.0f;
    float t = fmul(ny, fsub(py, c.K5));
    t = fmul(c.alpha, t);
    t = ffma(nx, fsub(px, c.K2), t);
    t = ffma(nz, c.fx, t);
    return fmul(fmul(d, -c.fx), frcp(t));
}

// plane distance d = -n . X(p, depth) — getD_cu, gipuma.cu:96-111
__device__ __forceinline__ float plane_d(const RefCam& c, float nx, float ny, float nz, float px, float py, float depth)
{
    const float X = ffma(depth, px, -c.P34[0]);
    const float Y = ffma(depth, py, -c.P34[1]);
    const float Z = fsub(depth, c.P34[2]);
    const float* M = c.M_inv;
    const float wx = ffma(M[2], Z, ffma(M[0], X, fmul(M[1], Y)));
    const float wy = ffma(M[5], Z, ffma(M[3], X, fmul(M[4], Y)));
    const float wz = ffma(M[8], Z, ffma(M[6], X, fmul(M[7], Y)));
    return -dot3(nx, ny, nz, wx, wy, wz);
}

// unit viewing ray through pixel p — getViewVector_cu, gipuma.cu:122-130 (get3Dpoint_cu1, normalize_cu)
__device__ __forceinline__ void view_vector(const RefCam& c, float px, float py, float& vx, float& vy, float& vz)
{
    const float a = fsub(px, c.P34[0]), b = fsub(py, c.P34[1]), e = fsub(1.0f, c.P34[2]);
    const float* M = c.M_inv;
    const float x = fsub(ffma(e, M[2], ffma(a, M[0], fmul(b, M[1]))), c.C[0]);
    const float y = fsub(ffma(e, M[5], ffma(a, M[3], fmul(b, M[4]))), c.C[1]);
    const float z = fsub(ffma(e, M[8], ffma(a, M[6], fmul(b, M[7]))), c.C[2]);
    const float rs = frsq(ffma(z, z, ffma(x, x, fmul(y, y))));
    vx = fmul(x, rs);  vy = fmul(y, rs);  vz = fmul(z, rs);
}

// XORWOW step — curand() of curand_kernel.h (curandStateXORWOW), used by gipuma.cu:138-141
struct Xorwow { unsigned v0, v1, v2, v3, v4, d; };
__device__ __forceinline__ unsigned xorwow_next(Xorwow& s)
{
    const unsigned t = s.v0 ^ (s.v0 >> 2);
    s.v0 = s.v1;  s.v1 = s.v2;  s.v2 = s.v3;  s.v3 = s.v4;
    s.v4 = (s.v4 ^ (s.v4 << 4)) ^ (t ^ (t << 1));
    s.d += 362437u;
    return s.v4 + s.d;
}
// curand_uniform: x * 2^-32 + 2^-33 (one FMA in the reference binary)
__device__ __forceinline__ float xorwow_uniform(Xorwow& s)
{
    return ffma(__uint2float_rn(xorwow_next(s)), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
}

// ---- multi-view combination — pmCostMultiview_cu, gipuma.cu:770-805 --------------------------
// c0/c1: (partial) costs of views lane and lane+32.  Returns the combined cost, identical on all lanes.
// Monotone in every argument, so applied to partial sums it is an exact lower bound of the final value.
__device__ __forceinline__ float combine_views(const KParams& P, float c0, float c1, unsigned lane)
{
    const bool has0 = (int)lane < P.V, has1 = (int)lane + 32 < P.V;
    // "if ( c < MAXCOST ) numValidViews++; else c = MAXCOST;"
    const int num_valid = __popc(__ballot_sync(GPM_FULL, has0 && c0 < GPM_MAXCOST)) +
                          __popc(__ballot_sync(GPM_FULL, has1 && c1 < GPM_MAXCOST));
    unsigned b0 = has0 ? __float_as_uint(fmin_(c0, GPM_MAXCOST)) : 0x7f800000u;   // costs are >= +0: order == uint order
    unsigned b1 = has1 ? __float_as_uint(fmin_(c1, GPM_MAXCOST)) : 0x7f800000u;
    int num_best = num_valid;
    if (P.cost_comb == 1) num_best = min(num_best, P.n_best);      // COMB_BEST_N
    if (P.cost_comb == 3) num_best = P.V;                          // COMB_GOOD
    float sum = 0.0f, thresh = 0.0f;
    for (int i = 0; i < num_best; i++) {                           // ascending order == sort_small + loop :779-797
        const unsigned m = __reduce_min_sync(GPM_FULL, min(b0, b1));
        float c = __uint_as_float(m);
        if (i == 0) thresh = fmul(c, P.good_factor);
        if (P.cost_comb == 3) c = fmin_(thresh, c);
        sum = fadd(sum, c);
        const unsigned hit0 = __ballot_sync(GPM_FULL, b0 == m);    // retire exactly one instance of the minimum
        if (hit0) { if (lane == (unsigned)(__ffs(hit0) - 1)) b0 = 0x7f800000u; }
        else { const unsigned hit1 = __ballot_sync(GPM_FULL, b1 == m); if (lane == (unsigned)(__ffs(hit1) - 1)) b1 = 0x7f800000u; }
    }
    float cost = fmul(frcp(__int2float_rn(num_best)), sum);        // cost / (float)numConsidered
    if (num_best < 1) cost = GPM_MAXCOST;
    if (cost != cost || cost > GPM_MAXCOST || cost < 0.0f) cost = GPM_MAXCOST;
    return cost;
}

// View-shard mode (multi-GPU): the ascending n_best smallest of this rank's view costs, padded with +inf.
// Every lane returns the same values; out[i] is written by lane 0.  (COMB_BEST_N only.)
__device__ __forceinline__ void local_topn(const KParams& P, float c0, float c1, unsigned lane, float* out)
{
    const bool has0 = (int)lane < P.V, has1 = (int)lane + 32 < P.V;
    unsigned b0 = has0 ? __float_as_uint(fmin_(c0, GPM_MAXCOST)) : 0x7f800000u;
    unsigned b1 = has1 ? __float_as_uint(fmin_(c1, GPM_MAXCOST)) : 0x7f800000u;
    for (int i = 0; i < P.n_best; i++) {
        const unsigned m = __reduce_min_sync(GPM_FULL, min(b0, b1));
        if (lane == 0) out[i] = __uint_as_float(m);
        const unsigned hit0 = __ballot_sync(GPM_FULL, b0 == m);
        if (m != 0x7f800000u) {
            if (hit0) { if (lane == (unsigned)(__ffs(hit0) - 1)) b0 = 0x7f800000u; }
            else { const unsigned hit1 = __ballot_sync(GPM_FULL, b1 == m); if (lane == (unsigned)(__ffs(hit1) - 1)) b1 = 0x7f800000u; }
        }
    }
}

struct WarpStats { unsigned hyp, skip, pruned; unsigned long long pairs, pairs_full; };

// ---- geometric-consistency cost of one source view — DESIGN.md §14 ----------------------------------------------
// IEEE round-to-nearest multiply, add, divide and square root only (no FMA, no approximate reciprocal), each product sum
// evaluated as (a0 b0 + a1 b1) + a2 b2, so that a numpy restatement in float32 reproduces every bit (oracle/pygeo.py).
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float sum3(const float* m, float x, float y, float z)
{
    return fadd(fadd(fmul(m[0], x), fmul(m[1], y)), fmul(m[2], z));
}

// g_j = weight * min(err, max_err) of view v (camera `vc`: K, R, t as ViewCam) for plane (n, d) at pixel (px, py):
// the plane's point on the pixel's ray goes into view j, to the nearest pixel (floor(x + 0.5)), back out at that pixel's
// depth in view j's depth map, and into the reference image; err is the distance from p.  weight * max_err where that
// pixel is off-image, its depth is not in [depthMin, depthMax] (0 included), or a point lies behind a camera.
__device__ __forceinline__ float geo_cost(const KParams& P, const GeoParams& G, const float* __restrict__ vc, int v,
                                          float nx, float ny, float nz, float d, float px, float py)
{
    const float* K = vc;
    const float* R = vc + 9;
    const float* t = vc + 18;
    const float far = fmul(G.weight, G.max_err);
    // the point X of the plane on the ray of p (the point the homography H_j maps p through): X = z K_ref^-1 (px, py, 1)
    const float* Ki = P.ref.K_inv;
    const float rx = sum3(Ki, px, py, 1.0f), ry = sum3(Ki + 3, px, py, 1.0f), rz = sum3(Ki + 6, px, py, 1.0f);
    const float z = fdiv(-d, fadd(fadd(fmul(nx, rx), fmul(ny, ry)), fmul(nz, rz)));
    if (!(z > 0.0f)) return far;
    const float X = fmul(z, rx), Y = fmul(z, ry), Z = fmul(z, rz);
    // into view j: Xj = R X + t, (u, v) = K Xj, rounded to the nearest pixel
    const float xj = fadd(sum3(R, X, Y, Z), t[0]), yj = fadd(sum3(R + 3, X, Y, Z), t[1]), zj = fadd(sum3(R + 6, X, Y, Z), t[2]);
    if (!(zj > 0.0f)) return far;
    const float qz = sum3(K + 6, xj, yj, zj);
    const float u = floorf(fadd(fdiv(sum3(K, xj, yj, zj), qz), 0.5f));
    const float w = floorf(fadd(fdiv(sum3(K + 3, xj, yj, zj), qz), 0.5f));
    if (!(u >= 0.0f && u <= (float)(P.W - 1) && w >= 0.0f && w <= (float)(P.H - 1))) return far;
    const float D = __ldg(G.depth + ((size_t)v * P.H + (int)w) * P.W + (int)u);
    if (!(D > 0.0f && D >= P.ref.depthMin && D <= P.ref.depthMax)) return far;
    // back through view j's camera: Y = D K_j^-1 (u', v', 1), X' = R^T (Y - t); then into the reference image
    const float* Kj = G.kinv + 9 * v;
    const float ax = fsub(fmul(D, sum3(Kj, u, w, 1.0f)), t[0]);
    const float ay = fsub(fmul(D, sum3(Kj + 3, u, w, 1.0f)), t[1]);
    const float az = fsub(fmul(D, sum3(Kj + 6, u, w, 1.0f)), t[2]);
    const float bx = fadd(fadd(fmul(R[0], ax), fmul(R[3], ay)), fmul(R[6], az));
    const float by = fadd(fadd(fmul(R[1], ax), fmul(R[4], ay)), fmul(R[7], az));
    const float bz = fadd(fadd(fmul(R[2], ax), fmul(R[5], ay)), fmul(R[8], az));
    if (!(bz > 0.0f)) return far;
    const float pz = sum3(G.Kref + 6, bx, by, bz);
    const float ex = fsub(fdiv(sum3(G.Kref, bx, by, bz), pz), px);
    const float ey = fsub(fdiv(sum3(G.Kref + 3, bx, by, bz), pz), py);
    const float err = __fsqrt_rn(fadd(fmul(ex, ex), fmul(ey, ey)));
    return fmul(G.weight, err < G.max_err ? err : G.max_err);      // a NaN err counts as max_err
}

// ---- NCC cost of one source view from the window sums — DESIGN.md §15 ---------------------------------------------
// Same arithmetic rules as geo_cost (oracle/pyncc.py restates it).  Wsum, Sr, Srr: the pixel's sums (setup_window);
// St, Stt, Srt: the view's sums for the hypothesis; min_var = min_std * min_std.
__device__ __forceinline__ float ncc_cost(float Wsum, float Sr, float Srr, float St, float Stt, float Srt, float min_var)
{
    const float mr = fdiv(Sr, Wsum), mt = fdiv(St, Wsum);
    const float vr = fsub(fdiv(Srr, Wsum), fmul(mr, mr));
    const float vt = fsub(fdiv(Stt, Wsum), fmul(mt, mt));
    const float c = fsub(fdiv(Srt, Wsum), fmul(mr, mt));
    if (!(Wsum > 0.0f) || !(vr >= min_var) || !(vt >= min_var)) return 2.0f;     // flat window, or one-pass cancellation
    const float x = fsub(1.0f, fdiv(c, __fsqrt_rn(fmul(vr, vt))));
    if (x != x) return 2.0f;
    return x < 0.0f ? 0.0f : (x > 2.0f ? 2.0f : x);
}

// ---- planar prior — DESIGN.md §18 --------------------------------------------------------------------------------
// What the k_sweep / k_cost_eval variants with PRIOR = true read besides KParams: one plane per pixel (the prior map,
// n.xyz and d in the state's layout; a pixel has a prior where the plane's depth is in [depthMin, depthMax]) and the term's
// parameters.  A kernel parameter of its own, so that KParams, GeoParams and JvsParams keep their layout.
// The variants with the geometric term's mask (DESIGN.md §21), which exclude the prior, read geo_mask in map's place.
struct PriorParams {
    union {
        const float4* map;                  // [H*W]
        const unsigned char* geo_mask;      // [H*W] nonzero: the geometric term is off at the pixel
    };
    float weight;               // the term's saturation value
    float depth_sigma;          // sigma_d, in depth units
    float normal_scale;         // 1 - cos(sigma_n), rounded once from double on the host
};

// a stored or evaluated cost with the prior term: MAXCOST (no valid view) stays MAXCOST
__device__ __forceinline__ float with_prior(float c, float prior) { return c == GPM_MAXCOST ? c : fadd(c, prior); }

// Depth of plane (n, d) at pixel p by plane_depth's formula, in IEEE round-to-nearest multiply, add and divide (no FMA, no
// approximate reciprocal), so that the prior's depths, its has-a-prior test and the support points' depth test are
// reproducible bit for bit in float32 numpy.  A NaN d gives NaN, which is in no depth range.
__device__ __forceinline__ float prior_depth(const RefCam& c, float nx, float ny, float nz, float d, float px, float py)
{
    const float t = __fadd_rn(__fadd_rn(__fmul_rn(nx, __fsub_rn(px, c.K2)), __fmul_rn(c.alpha, __fmul_rn(ny, __fsub_rn(py, c.K5)))),
                              __fmul_rn(nz, c.fx));
    return __fdiv_rn(__fmul_rn(d, -c.fx), t);
}

// prior(p, h) = weight * q / (1 + q), q = ((depth_h - depth_pi) / sigma_d)^2 + max(0, 1 - n_h . n_pi) / (1 - cos sigma_n):
// a bounded Geman-McClure penalty, 0 at the prior plane, saturating at weight (also where q is not finite).  IEEE
// round-to-nearest multiply, add, subtract and divide only, the dot product as (a0 b0 + a1 b1) + a2 b2, so that a float32
// numpy restatement reproduces every bit (oracle/pyprior.py).  pd: the prior plane's prior_depth at the pixel, hd: the
// hypothesis'.
__device__ __forceinline__ float prior_cost(const PriorParams& R, const float4& pi, float pd, float nx, float ny, float nz, float hd)
{
    const float delta = __fdiv_rn(__fsub_rn(hd, pd), R.depth_sigma);
    const float dot = __fadd_rn(__fadd_rn(__fmul_rn(nx, pi.x), __fmul_rn(ny, pi.y)), __fmul_rn(nz, pi.z));
    const float off = __fsub_rn(1.0f, dot);
    const float a = __fdiv_rn(off > 0.0f ? off : 0.0f, R.normal_scale);
    const float q = __fadd_rn(__fmul_rn(delta, delta), a);
    return __fmul_rn(R.weight, q < 1e30f ? __fdiv_rn(q, __fadd_rn(1.0f, q)) : 1.0f);
}

// homographies H_v = K_v (R_v - t_v n^T / d) K_ref^-1 of plane (n, d) for every view into H[v * 12 ...] (rows of 3,
// 16-byte aligned) — getHomography_cu, gipuma.cu:339-356
__device__ __forceinline__ void homographies(const KParams& P, const float* __restrict__ sCam, float* H, float nx, float ny, float nz,
                                             float d, unsigned lane)
{
    const float rd = frcp(d);
    const float* Ki = P.ref.K_inv;
    for (int v = lane; v < P.V; v += 32) {
        const float* K = sCam + v * GPM_VIEWCAM_FLOATS;
        const float* R = K + 9;
        const float* t = K + 18;
        float A[9], T[9];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            A[3 * i + 0] = ffma(-fmul(t[i], nx), rd, R[3 * i + 0]);
            A[3 * i + 1] = ffma(-fmul(t[i], ny), rd, R[3 * i + 1]);
            A[3 * i + 2] = ffma(-fmul(t[i], nz), rd, R[3 * i + 2]);
        }
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++)
                T[3 * i + j] = ffma(A[3 * i + 2], Ki[6 + j], ffma(A[3 * i], Ki[j], fmul(A[3 * i + 1], Ki[3 + j])));
        float* Hv = H + v * 12;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++)
                Hv[3 * i + j] = ffma(K[3 * i + 2], T[6 + j], ffma(K[3 * i], T[j], fmul(K[3 * i + 1], T[3 + j])));
    }
}

// dissimilarity of one grey sample against one view — pmCostComputation_shared, gipuma.cu:253-274
__device__ __forceinline__ float dissim_grey(const KParams& P, float one_minus_alpha, float gx1, float gy1, float left, float gx2,
                                             float gy2, float t_c)
{
    const float gradX = fsub(gx1, gx2);
    const float gradY = fsub(gy1, gy2);
    const float gradDis = fmin_(P.tau_gradient, fmul(fadd(fabsf(gradX), fabsf(gradY)), 0.0625f));
    const float colDis = fmin_(P.tau_color, fabsf(fsub(left, t_c)));
    return ffma(colDis, one_minus_alpha, fmul(P.alpha, gradDis));
}

// getCorrespondingPoint_cu (gipuma.cu:207-217): H (x, y, 1)^T, then / z — the division's multiply is fused with
// the +-1 / +0.5 texel offsets in the reference binary (FFMA X, rcp(Z), {0.5, 1, -1}); then the source-view taps
// of gipuma.cu:251-253: gx2 = tex(x+1,y) - tex(x-1,y), gy2 = tex(x,y+1) - tex(x,y-1), centre.  The three flags are the
// rounding variant of each row of H (see eval_plane).
__device__ __forceinline__ void fetch_sample_grey(cudaTextureObject_t src, const float4& h0, const float4& h1, const float4& h2, float ax,
                                                  float ay, int v, bool XFIRST, bool YFIRSTX, bool ZFIRSTX, float& gx2, float& gy2,
                                                  float& t_c)
{
    const float X = XFIRST ? fadd(h0.z, ffma(h0.y, ay, fmul(h0.x, ax))) : fadd(h0.z, ffma(h0.x, ax, fmul(h0.y, ay)));
    const float Y = YFIRSTX ? fadd(h1.y, ffma(h1.x, ay, fmul(h0.w, ax))) : fadd(h1.y, ffma(h0.w, ax, fmul(h1.x, ay)));
    const float Z = ZFIRSTX ? fadd(h2.x, ffma(h1.w, ay, fmul(h1.z, ax))) : fadd(h2.x, ffma(h1.z, ax, fmul(h1.w, ay)));
    const float r = frcp(Z);
    const float cx = ffma(X, r, 0.5f), cy = ffma(Y, r, 0.5f);
    const float cxp = fadd(ffma(X, r, 1.0f), 0.5f), cxm = fadd(ffma(X, r, -1.0f), 0.5f);
    const float cyp = fadd(ffma(Y, r, 1.0f), 0.5f), cym = fadd(ffma(Y, r, -1.0f), 0.5f);
    t_c = tex2DLayered<float>(src, cx, cy, v);
    const float t_xp = tex2DLayered<float>(src, cxp, cy, v);
    const float t_xm = tex2DLayered<float>(src, cxm, cy, v);
    const float t_yp = tex2DLayered<float>(src, cx, cyp, v);
    const float t_ym = tex2DLayered<float>(src, cx, cym, v);
    gx2 = fsub(t_xp, t_xm);
    gy2 = fsub(t_yp, t_ym);
}

// ---- cost of one plane hypothesis at the warp's pixel ---------------------------------------
// pmCostMultiview_cu (gipuma.cu:720-806) over pmCost_shared (:585-680) / pmCostComputation_shared (:223-277).
// Returns the exact combined cost, or — if `bound` is finite and an exact lower bound of the final cost
// reaches it — some value >= bound (the caller only tests `< bound`).
// XFIRST selects which of the two roundings of  H0*x + H1*y + H2  the reference binary uses at the call site:
//   false: H2 + fma(H0, x, H1*y)   — gipuma_init_cu2 and the planeRefine kernels;
//   true : H2 + fma(H1, y, H0*x)   — the spatialPropClose/Far kernels, where nvcc hoisted the x products out of
//          the inner (y) loop of gipuma.cu:633-634.  (Both are contractions of the same source line, gipuma.cu:213.)
// XF = 2 takes the variant from `rt` at run time (the fused 20-neighbour kernels, whose inlined call sites differ).
// GEO: every view's cost is fadd(photometric cost, geo_cost) (DESIGN.md §14); (gpx, gpy) is the pixel.  The geometric terms
// are computed before the first round and added to the partial costs of every bound test as well: g >= 0 and a rounded
// add is monotone, so the bound stays an exact lower bound.
// NCC: the photometric cost of every view is the NCC cost (DESIGN.md §15, grey images only; G->min_std).  XF and `rt` are
// ignored: every call site uses one rounding variant.  No bound is tested (partial sums bound nothing); `bound` is ignored.
// ROWS (NCC only; joint view selection, DESIGN.md §17): nothing is combined; view v's NCC cost goes to per_view0[v] and,
// with GEO, its geometric term to per_view1[v] (written by lanes v and v + 32), and the result is 0.
// PRIOR (planar prior, DESIGN.md §18): the result is with_prior(cost, prior), and the bound test compares fadd(b, prior):
// prior >= 0 and a rounded add is monotone, so that stays an exact lower bound of the final value.
// geo_on false (GEO only; the pixel is masked, DESIGN.md §21): no geometric term is computed and the result is exactly that
// of GEO = false; ROWS writes no geometric term.
template <int XF, bool COLOR, bool GEO = false, bool NCC = false, bool ROWS = false, bool PRIOR = false>
__device__ __forceinline__ float eval_plane(const KParams& P, const float* __restrict__ sCam, const WarpScratch& ws,
                                            cudaTextureObject_t src, float nx, float ny, float nz, float d,
                                            float bound, unsigned lane, WarpStats& st,
                                            float* per_view0 = nullptr, float* per_view1 = nullptr, unsigned rt = 0u,
                                            const GeoParams* G = nullptr, float gpx = 0.0f, float gpy = 0.0f, float prior = 0.0f,
                                            bool geo_on = true)
{
    static_assert(!ROWS || NCC, "per-view cost rows are built for the NCC cost only");
    // XF = 0 / 1: compile-time variant; XF = 2: per call, rt bit 0 = x-term first, bit 1 = gradient folding variant,
    // bits 2 / 3 = the Y / Z row of H deviates from bit 0 (ptxas chose per row in one inlined site of the fused kernel)
    const bool XFIRST = XF == 2 ? (rt & 1u) != 0u : XF == 1;
    const bool YFIRSTX = XF == 2 ? (((rt >> 2) ^ rt) & 1u) != 0u : XF == 1;
    const bool ZFIRSTX = XF == 2 ? (((rt >> 3) ^ rt) & 1u) != 0u : XF == 1;
    const int grad_variant = XF == 2 ? (int)((rt >> 1) & 1u) : P.grad_variant;

    homographies(P, sCam, ws.H, nx, ny, nz, d, lane);
    __syncwarp();
    float g0 = 0.0f, g1 = 0.0f;          // geometric terms of views lane and lane + 32
    if constexpr (GEO) if (geo_on) {
        if ((int)lane < P.V) g0 = geo_cost(P, *G, sCam + lane * GPM_VIEWCAM_FLOATS, (int)lane, nx, ny, nz, d, gpx, gpy);
        if ((int)lane + 32 < P.V) g1 = geo_cost(P, *G, sCam + (lane + 32) * GPM_VIEWCAM_FLOATS, (int)lane + 32, nx, ny, nz, d, gpx, gpy);
    }
    if constexpr (NCC) {
        static_assert(!COLOR, "the NCC cost is built for grey images only");
        st.hyp++;
        st.pairs_full += (unsigned long long)P.V * P.ns;
        // t_s of view v at sample s: one fetch at the PM cost's centre tap, the x-term first in every row of H
        auto fetch_centre = [&](int v, int s) {
            const float4* H4 = reinterpret_cast<const float4*>(ws.H + v * 12);
            const float4 h0 = H4[0], h1 = H4[1], h2 = H4[2];
            const float4 a = ws.A[s];
            const float X = fadd(h0.z, ffma(h0.y, a.y, fmul(h0.x, a.x)));
            const float Y = fadd(h1.y, ffma(h1.x, a.y, fmul(h0.w, a.x)));
            const float Z = fadd(h2.x, ffma(h1.w, a.y, fmul(h1.z, a.x)));
            const float r = frcp(Z);
            return tex2DLayered<float>(src, ffma(X, r, 0.5f), ffma(Y, r, 0.5f), v);
        };
        // lane handles pair q = (view v, sample k of the round) of N consecutive groups of 32 pairs, all fetches in flight
        // before D[v][k] = t is written.  In a round of 32 samples lane = sample, and a step covers N views.  Two views per
        // step measured fastest (DESIGN.md §15: 4 and 8 hold more fetches in flight but cost registers and were slower).
        auto ncc_steps = [&](auto nconst, int q0, int s0, int len, int npairs, unsigned M, const unsigned char* prow) {
            constexpr int N = decltype(nconst)::value;
            float t[N];
            int dst[N];
#pragma unroll
            for (int u = 0; u < N; u++) {
                const int q = q0 + u * 32 + (int)lane;
                const int qc = min(q, npairs - 1);
                const int v = (int)(((unsigned)qc * M) >> 20);                       // qc / len
                const int k = prow[qc - v * len];
                t[u] = fetch_centre(v, s0 + k);
                dst[u] = (q < npairs) ? v * GPM_DSTRIDE + k : -1;
            }
#pragma unroll
            for (int u = 0; u < N; u++)
                if (dst[u] >= 0) ws.D[dst[u]] = t[u];
        };
        // the three sums of views lane and lane + 32, sequential in sample order
        float St0 = 0.0f, Stt0 = 0.0f, Srt0 = 0.0f, St1 = 0.0f, Stt1 = 0.0f, Srt1 = 0.0f;
        int s0 = 0;
        for (int r = 0; r < P.nrounds; r++) {
            const int s1 = P.round_end[r];
            const int len = s1 - s0;
            const int npairs = P.V * len;
            const unsigned M = (1u << 20) / (unsigned)len + 1u;
            const unsigned char* prow = ws.perm + r * 32;
            int q0 = 0;
            for (; q0 + 32 < npairs; q0 += 64) ncc_steps(std::integral_constant<int, 2>(), q0, s0, len, npairs, M, prow);
            if (q0 < npairs) ncc_steps(std::integral_constant<int, 1>(), q0, s0, len, npairs, M, prow);
            st.pairs += npairs;
            __syncwarp();
            const float* w = ws.w + s0;
            const float* a = ws.a + s0;
            const float* D0 = ws.D + lane * GPM_DSTRIDE;
            if ((int)lane < P.V)
                for (int k = 0; k < len; k++) {
                    const float t = D0[k], wt = fmul(w[k], t);
                    St0 = fadd(St0, wt);  Stt0 = fadd(Stt0, fmul(wt, t));  Srt0 = fadd(Srt0, fmul(a[k], t));
                }
            if ((int)lane + 32 < P.V) {
                const float* D1 = D0 + 32 * GPM_DSTRIDE;
                for (int k = 0; k < len; k++) {
                    const float t = D1[k], wt = fmul(w[k], t);
                    St1 = fadd(St1, wt);  Stt1 = fadd(Stt1, fmul(wt, t));  Srt1 = fadd(Srt1, fmul(a[k], t));
                }
            }
            __syncwarp();
            s0 = s1;
        }
        const float Wsum = ws.sums[0], Sr = ws.sums[1], Srr = ws.sums[2];
        const float min_var = fmul(G->min_std, G->min_std);
        const float c0 = ncc_cost(Wsum, Sr, Srr, St0, Stt0, Srt0, min_var);
        const float c1 = ncc_cost(Wsum, Sr, Srr, St1, Stt1, Srt1, min_var);
        if constexpr (ROWS) {
            if ((int)lane < P.V) { per_view0[lane] = c0;  if (GEO && geo_on) per_view1[lane] = g0; }
            if ((int)lane + 32 < P.V) { per_view0[lane + 32] = c1;  if (GEO && geo_on) per_view1[lane + 32] = g1; }
            return 0.0f;
        }
        if constexpr (PRIOR) return with_prior(GEO ? combine_views(P, fadd(c0, g0), fadd(c1, g1), lane) : combine_views(P, c0, c1, lane), prior);
        else if constexpr (GEO) return geo_on ? combine_views(P, fadd(c0, g0), fadd(c1, g1), lane) : combine_views(P, c0, c1, lane);
        else return combine_views(P, c0, c1, lane);
    }

    const float one_minus_alpha = fsub(1.0f, P.alpha);
    float c0 = 0.0f, c1 = 0.0f;
    st.hyp++;
    st.pairs_full += (unsigned long long)P.V * P.ns;

    auto dissim = [&](float gx1, float gy1, float left, float gx2, float gy2, float t_c) {
        return dissim_grey(P, one_minus_alpha, gx1, gy1, left, gx2, gy2, t_c);
    };
    auto fetch_sample = [&](const float4& h0, const float4& h1, const float4& h2, float ax, float ay, int v,
                            float& gx2, float& gy2, float& t_c) {
        fetch_sample_grey(src, h0, h1, h2, ax, ay, v, XFIRST, YFIRSTX, ZFIRSTX, gx2, gy2, t_c);
    };

    // ---- colour (T = float4) variants: pmCostComputation_shared<float4>, l1_norm(float4) = (|x|+|y|+|z|) * 0.3333333f
    // (gipuma.cu:174-179).  Operation order and the one FMA ptxas forms ( l1(gradX) + l1(gradY) ) follow the reference's SASS.
    struct C3 { float x, y, z; };
    auto l1sum = [&](float x, float y, float z) { return fadd(fabsf(z), fadd(fabsf(x), fabsf(y))); };
    auto dissim_c = [&](const float4& gx1, const float4& gy1, const float4& left, const C3& gx2, const C3& gy2, const C3& tc) {
        const float sX = l1sum(fsub(gx1.x, gx2.x), fsub(gx1.y, gx2.y), fsub(gx1.z, gx2.z));
        const float sY = l1sum(fsub(gy1.x, gy2.x), fsub(gy1.y, gy2.y), fsub(gy1.z, gy2.z));
        // sweep kernels: FFMA(sY, 1/3, FMUL(sX, 1/3)); gipuma_init_cu2<float4>: FFMA(sX, 1/3, FMUL(sY, 1/3))
        const float third = 0.3333333134651184082f;
        const float g = fmul(grad_variant ? ffma(sX, third, fmul(sY, third)) : ffma(sY, third, fmul(sX, third)), 0.0625f);
        const float gradDis = fmin_(P.tau_gradient, g);
        const float colDiff = fmul(l1sum(fsub(left.x, tc.x), fsub(left.y, tc.y), fsub(left.z, tc.z)), 0.3333333134651184082f);
        const float colDis = fmin_(P.tau_color, colDiff);
        return ffma(colDis, one_minus_alpha, fmul(P.alpha, gradDis));
    };
    auto fetch_sample_c = [&](const float4& h0, const float4& h1, const float4& h2, float ax, float ay, int v,
                              C3& gx2, C3& gy2, C3& tc) {
        const float X = XFIRST ? fadd(h0.z, ffma(h0.y, ay, fmul(h0.x, ax))) : fadd(h0.z, ffma(h0.x, ax, fmul(h0.y, ay)));
        const float Y = YFIRSTX ? fadd(h1.y, ffma(h1.x, ay, fmul(h0.w, ax))) : fadd(h1.y, ffma(h0.w, ax, fmul(h1.x, ay)));
        const float Z = ZFIRSTX ? fadd(h2.x, ffma(h1.w, ay, fmul(h1.z, ax))) : fadd(h2.x, ffma(h1.z, ax, fmul(h1.w, ay)));
        const float r = frcp(Z);
        const float cx = ffma(X, r, 0.5f), cy = ffma(Y, r, 0.5f);
        const float cxp = fadd(ffma(X, r, 1.0f), 0.5f), cxm = fadd(ffma(X, r, -1.0f), 0.5f);
        const float cyp = fadd(ffma(Y, r, 1.0f), 0.5f), cym = fadd(ffma(Y, r, -1.0f), 0.5f);
        // the reference's tex2D<float4> filters each channel with the same weights: three R32F fetches per tap from the
        // channel planes of view v are bit-identical and cost three R32F fetches instead of one RGBA32F fetch
        const int l = 3 * v;
        const float xp0 = tex2DLayered<float>(src, cxp, cy, l), xp1 = tex2DLayered<float>(src, cxp, cy, l + 1), xp2 = tex2DLayered<float>(src, cxp, cy, l + 2);
        const float xm0 = tex2DLayered<float>(src, cxm, cy, l), xm1 = tex2DLayered<float>(src, cxm, cy, l + 1), xm2 = tex2DLayered<float>(src, cxm, cy, l + 2);
        const float yp0 = tex2DLayered<float>(src, cx, cyp, l), yp1 = tex2DLayered<float>(src, cx, cyp, l + 1), yp2 = tex2DLayered<float>(src, cx, cyp, l + 2);
        const float ym0 = tex2DLayered<float>(src, cx, cym, l), ym1 = tex2DLayered<float>(src, cx, cym, l + 1), ym2 = tex2DLayered<float>(src, cx, cym, l + 2);
        tc.x = tex2DLayered<float>(src, cx, cy, l);  tc.y = tex2DLayered<float>(src, cx, cy, l + 1);  tc.z = tex2DLayered<float>(src, cx, cy, l + 2);
        gx2.x = fsub(xp0, xm0);  gx2.y = fsub(xp1, xm1);  gx2.z = fsub(xp2, xm2);
        gy2.x = fsub(yp0, ym0);  gy2.y = fsub(yp1, ym1);  gy2.z = fsub(yp2, ym2);
    };

    // Generic sampling step (short rounds): lane handles pair q = (view v, sample k of the round); pairs of several
    // views share one instruction.  N steps are issued back to back before any result is consumed.
    auto steps = [&](auto nconst, int q0, int s0, int len, int npairs, unsigned M, const unsigned char* prow) {
        constexpr int N = decltype(nconst)::value;
        float gx2[N], gy2[N], t_c[N], gx1[N], gy1[N];
        int dst[N], sidx[N];
#pragma unroll
        for (int u = 0; u < N; u++) {
            const int q = q0 + u * 32 + (int)lane;
            const int qc = min(q, npairs - 1);
            const int v = (int)(((unsigned)qc * M) >> 20);                       // qc / len
            const int k = prow[qc - v * len];
            const int s = s0 + k;
            const float4* H4 = reinterpret_cast<const float4*>(ws.H + v * 12);
            const float4 a = ws.A[s];
            sidx[u] = s;
            dst[u] = (q < npairs) ? v * GPM_DSTRIDE + k : -1;
            if (COLOR) {
                C3 cgx, cgy, ctc;
                fetch_sample_c(H4[0], H4[1], H4[2], a.x, a.y, v, cgx, cgy, ctc);
                const float dis = dissim_c(ws.GX4[s], ws.GY4[s], ws.L4[s], cgx, cgy, ctc);
                if (dst[u] >= 0) ws.D[dst[u]] = dis;
            } else {
                fetch_sample(H4[0], H4[1], H4[2], a.x, a.y, v, gx2[u], gy2[u], t_c[u]);
                gx1[u] = a.z;  gy1[u] = a.w;
            }
        }
        if (!COLOR) {
#pragma unroll
            for (int u = 0; u < N; u++) {
                const float dis = dissim(gx1[u], gy1[u], ws.left[sidx[u]], gx2[u], gy2[u], t_c[u]);
                if (dst[u] >= 0) ws.D[dst[u]] = dis;
            }
        }
    };

    // Full rounds (32 samples): lane = sample, one view per step — every texture instruction reads one compact
    // source patch, homography loads are shared-memory broadcasts.  Two views are in flight per lane.
    auto full_round = [&](int s0, int k) {          // k: this lane's sample of the round (a permutation of 0..31, see KParams::perm)
        if (COLOR) {                      // one view per step; the 5 float4 fetches already are 20 texel reads in flight
            const float4 a = ws.A[s0 + k];
            const float4 l4 = ws.L4[s0 + k], gx4 = ws.GX4[s0 + k], gy4 = ws.GY4[s0 + k];
            for (int v = 0; v < P.V; v++) {
                const float4* Ha = reinterpret_cast<const float4*>(ws.H + v * 12);
                C3 cgx, cgy, ctc;
                fetch_sample_c(Ha[0], Ha[1], Ha[2], a.x, a.y, v, cgx, cgy, ctc);
                ws.D[v * GPM_DSTRIDE + k] = dissim_c(gx4, gy4, l4, cgx, cgy, ctc);
            }
            return;
        }
        const float4 a = ws.A[s0 + k];
        const float left = ws.left[s0 + k];
        float* Dl = ws.D + k;
        int v = 0;
        for (; v + 1 < P.V; v += 2) {
            const float4* Ha = reinterpret_cast<const float4*>(ws.H + v * 12);
            const float4* Hb = Ha + 3;
            float gxa, gya, ca, gxb, gyb, cb;
            fetch_sample(Ha[0], Ha[1], Ha[2], a.x, a.y, v, gxa, gya, ca);
            fetch_sample(Hb[0], Hb[1], Hb[2], a.x, a.y, v + 1, gxb, gyb, cb);
            Dl[v * GPM_DSTRIDE] = dissim(a.z, a.w, left, gxa, gya, ca);
            Dl[(v + 1) * GPM_DSTRIDE] = dissim(a.z, a.w, left, gxb, gyb, cb);
        }
        if (v < P.V) {
            const float4* Ha = reinterpret_cast<const float4*>(ws.H + v * 12);
            float gxa, gya, ca;
            fetch_sample(Ha[0], Ha[1], Ha[2], a.x, a.y, v, gxa, gya, ca);
            Dl[v * GPM_DSTRIDE] = dissim(a.z, a.w, left, gxa, gya, ca);
        }
    };

    int s0 = 0;
    for (int r = 0; r < P.nrounds; r++) {
        const int s1 = P.round_end[r];
        const int len = s1 - s0;
        const int npairs = P.V * len;
        const unsigned M = (1u << 20) / (unsigned)len + 1u;
        const unsigned char* prow = ws.perm + r * 32;
        if (len == 32) {
            full_round(s0, (int)prow[lane]);
        } else {
            int q0 = 0;
            for (; q0 + 32 < npairs; q0 += 64) steps(std::integral_constant<int, 2>(), q0, s0, len, npairs, M, prow);
            if (q0 < npairs) steps(std::integral_constant<int, 1>(), q0, s0, len, npairs, M, prow);
        }
        st.pairs += npairs;
        __syncwarp();
        // cost = cost + w * dis, sample after sample in the reference's order (gipuma.cu:633-677)
        {
            const float* w = ws.w + s0;
            const float* D0 = ws.D + lane * GPM_DSTRIDE;
            if (P.V <= 32) {
                if ((int)lane < P.V)
                    for (int k = 0; k < len; k++) c0 = ffma(w[k], D0[k], c0);
            } else {
                const float* D1 = D0 + 32 * GPM_DSTRIDE;
                const bool has1 = (int)lane + 32 < P.V;
                for (int k = 0; k < len; k++) {
                    const float wk = w[k];
                    c0 = ffma(wk, D0[k], c0);
                    if (has1) c1 = ffma(wk, D1[k], c1);
                }
            }
        }
        __syncwarp();
        const bool last = (r == P.nrounds - 1);
        if (per_view0) {                       // view-shard mode: hand back the exact per-view costs, combine elsewhere
            if (last) { *per_view0 = c0;  *per_view1 = c1;  return 0.0f; }
        } else if (last || P.prune) {
            float b;
            if constexpr (GEO) b = geo_on ? combine_views(P, fadd(c0, g0), fadd(c1, g1), lane) : combine_views(P, c0, c1, lane);
            else b = combine_views(P, c0, c1, lane);
            if constexpr (PRIOR) {
                if (last) return with_prior(b, prior);
                b = fadd(b, prior);
            } else if (last) return b;
            if (b >= bound) { st.pruned++; return b; }
        }
        s0 = s1;
    }
    return GPM_MAXCOST;   // not reached (nrounds >= 1)
}

// ---- per-pixel, hypothesis-independent window data ------------------------------------------
// NCC: also a_s = w_s * r_s and the pixel's sums W, Sr, Srr (DESIGN.md §15), added from +0 in sample order.
template <bool COLOR, bool NCC = false>
__device__ __forceinline__ void setup_window(const KParams& P, const float* __restrict__ tile, const WarpScratch& ws,
                                             int px, int py, int tile_x0, int tile_y0, unsigned lane)
{
    const int tw = P.tile_stride;
    const int cxi = px - tile_x0, cyi = py - tile_y0;
    if (COLOR) {
        const float4* t4 = reinterpret_cast<const float4*>(tile);
        const float4 center = t4[cyi * tw + cxi];
        const float rg = frcp(P.gamma);
        for (int s = lane; s < P.ns; s += 32) {
            const int ii = s / P.nside, jj = s - ii * P.nside;
            const int i = -P.rad + 2 * ii, j = -P.rad + 2 * jj;
            const float4* t = t4 + (cyi + j) * tw + (cxi + i);
            const float4 left = t[0], r = t[1], l = t[-1], dn = t[tw], up = t[-tw];
            ws.A[s] = make_float4(__int2float_rn(px + i), __int2float_rn(py + j), 0.f, 0.f);
            ws.L4[s] = left;
            ws.GX4[s] = make_float4(fsub(r.x, l.x), fsub(r.y, l.y), fsub(r.z, l.z), 0.f);          // gx1 = right - left
            ws.GY4[s] = make_float4(fsub(dn.x, up.x), fsub(dn.y, up.y), fsub(dn.z, up.z), 0.f);    // gy1 = down - up
            // weight_cu<float4>: expf(-l1_norm(left - center) / gamma) = ex2(((sum * -1/3) * rcp(gamma)) * log2 e) in the reference binary
            const float sum = fadd(fabsf(fsub(left.z, center.z)), fadd(fabsf(fsub(left.x, center.x)), fabsf(fsub(left.y, center.y))));
            ws.w[s] = fex2(fmul(fmul(fmul(sum, -0.3333333134651184082f), rg), 1.4426950216293334961f));
        }
        __syncwarp();
        return;
    }
    const float center = tile[cyi * tw + cxi];                     // centerValue, gipuma.cu:626
    const float nrg = -frcp(P.gamma);
    for (int s = lane; s < P.ns; s += 32) {
        const int ii = s / P.nside, jj = s - ii * P.nside;         // i (x offset) outer, j (y offset) inner, :633-634
        const int i = -P.rad + 2 * ii, j = -P.rad + 2 * jj;
        const float* t = tile + (cyi + j) * tw + (cxi + i);
        const float left = t[0];
        ws.A[s] = make_float4(__int2float_rn(px + i), __int2float_rn(py + j),
                              fsub(t[1], t[-1]),                   // gx1 = right - left, :258
                              fsub(t[tw], t[-tw]));                // gy1 = down - up, :259
        ws.left[s] = left;
        // expf(-|left - center| / gamma) under --use_fast_math: (|.| * -rcp(gamma)) * log2(e) -> ex2
        ws.w[s] = fex2(fmul(fmul(fabsf(fsub(left, center)), nrg), 1.4426950216293334961f));
        if constexpr (NCC) ws.a[s] = fmul(ws.w[s], left);
    }
    __syncwarp();
    if constexpr (NCC) {
        if (lane == 0) {
            float Wsum = 0.0f, Sr = 0.0f, Srr = 0.0f;
            for (int s = 0; s < P.ns; s++) {
                const float a = ws.a[s];
                Wsum = fadd(Wsum, ws.w[s]);  Sr = fadd(Sr, a);  Srr = fadd(Srr, fmul(a, ws.left[s]));
            }
            ws.sums[0] = Wsum;  ws.sums[1] = Sr;  ws.sums[2] = Srr;
        }
        __syncwarp();
    }
}

}  // namespace gpm
