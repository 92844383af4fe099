// gpm_fuse.cu — depth-map fusion (DESIGN.md §12, §22): N per-view world-frame depth + normal maps -> one point cloud.
// Compiled on its own, without --use_fast_math (gipuma_b200/build.py): every fp32 operation below is an explicit
// round-to-nearest intrinsic, denormals are kept, and oracle/fusion_oracle.c (the disparity rule) and
// oracle/fusion_rule_oracle.c (either rule) restate the same operations in the same order, so the GPU and the restatements
// agree bit for bit.
//
// Per reference view r (ascending), three launches on the fusion's own stream:
//   k_fuse_pixels   one thread per pixel of view r: consistency test against every other view (the disparity or the
//                   reprojection rule, DESIGN.md §22, a template argument), running sums in registers,
//                   the candidate vertex staged per pixel, used marks written for fused pixels, a per-block count
//   k_scan_blocks   one block: exclusive scan of the per-block counts (fixed order, no atomics)
//   k_compact       order-preserving scatter of the staged vertices into packed 27-byte PLY records + (view, pixel) sources
// The used masks need no second buffer: a pass reads the mask of view r only, at the thread's own pixel, and writes marks
// into other views' masks or at the thread's own pixel, so a mark made in pass r is first read in a later pass.
#include "../../include/gipuma_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

namespace gpm { int set_last_error(int code, const std::string& msg); }

namespace {

constexpr int kBlock = 256;
constexpr int kCamFloats = 22;                     // gpm_fuse_camera: M_inv[9], P[12], f

struct FuseArgs {
    const float4* norm4;                           // n * npix
    const float* images;                           // NULL or n * npix * channels
    unsigned char* used;                           // n * npix
    float4* stage;                                 // 2 * npix: (x, y, z, nx), (ny, nz, rgb bits, -)
    unsigned char* flag;                           // npix
    int* block_count;                              // blocks
    int n, W, H, channels, num_consistent;
    float dmin, dmax;
    float thresh;                                  // disparity rule: disp_thresh; reprojection rule: reproj_px
    float cos_thresh;
    float depth_rel;                               // reprojection rule only
};
// depth_rel fills what was tail padding: the kernel's parameters, and so the disparity rule's code, stay as they were
static_assert(sizeof(FuseArgs) == 88, "FuseArgs: depth_rel must fit the tail padding");

__device__ __forceinline__ float dot3(const float* a, float x, float y, float z)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(a[0], x), __fmul_rn(a[1], y)), __fmul_rn(a[2], z));
}

// get3Dpoint (cameraGeometryUtils.h:51-61): X = M_inv (depth (x, y, 1) - P_col34)
__device__ __forceinline__ void backproject(const float* cam, float x, float y, float d, float X[3])
{
    const float a = __fsub_rn(__fmul_rn(d, x), cam[9 + 3]);
    const float b = __fsub_rn(__fmul_rn(d, y), cam[9 + 7]);
    const float c = __fsub_rn(d, cam[9 + 11]);
    for (int i = 0; i < 3; i++) X[i] = dot3(cam + 3 * i, a, b, c);
}

// Projection of X into the view of `cam`, rounded to the nearest pixel: u = floor(x/z + 0.5), v likewise.  Returns the pixel
// index, or -1 when X is not in front of the camera (z > 0) or the pixel lies outside the image.  *z receives X's depth.
__device__ __forceinline__ int project(const float* cam, const float X[3], int W, int H, float* z, float* u, float* v)
{
    const float* P = cam + 9;
    const float hx = __fadd_rn(dot3(P, X[0], X[1], X[2]), P[3]);
    const float hy = __fadd_rn(dot3(P + 4, X[0], X[1], X[2]), P[7]);
    const float hz = __fadd_rn(dot3(P + 8, X[0], X[1], X[2]), P[11]);
    *z = hz;
    if (!(hz > 0.f)) return -1;
    const float fu = floorf(__fadd_rn(__fdiv_rn(hx, hz), 0.5f));
    const float fv = floorf(__fadd_rn(__fdiv_rn(hy, hz), 0.5f));
    if (!(fu >= 0.f && fu < (float)W && fv >= 0.f && fv < (float)H)) return -1;
    *u = fu;  *v = fv;
    return (int)fv * W + (int)fu;
}

// Consistency of view j (camera `cam`) with the reference point X of normal n, back-projected from pixel (x, y) of view r
// (camera `cr`) at depth dr: the target pixel, or -1.  Rule: GPM_FUSE_DISPARITY or GPM_FUSE_REPROJECTION.
template <int Rule>
__device__ __forceinline__ int consistent(const FuseArgs& a, int j, const float* cam, const float* cr,
                                          const float X[3], float x, float y, float dr, const float4 n, float4* tgt, float* u,
                                          float* v)
{
    float z;
    const int q = project(cam, X, a.W, a.H, &z, u, v);
    if (q < 0) return -1;
    const float4 t = a.norm4[(size_t)j * a.W * a.H + q];
    if (!(t.w >= a.dmin && t.w <= a.dmax)) return -1;
    if (Rule == GPM_FUSE_DISPARITY) {
        const float fb = __fmul_rn(cam[21], 0.54f);                                // baseline constant, cameraGeometryUtils.h:305
        if (!(fabsf(__fsub_rn(__fdiv_rn(fb, z), __fdiv_rn(fb, t.w))) < a.thresh)) return -1;
    } else {
        // the target's own point, projected back into view r: pixel distance to (x, y) and relative depth difference
        float Xj[3];
        backproject(cam, *u, *v, t.w, Xj);
        const float* P = cr + 9;
        const float hx = __fadd_rn(dot3(P, Xj[0], Xj[1], Xj[2]), P[3]);
        const float hy = __fadd_rn(dot3(P + 4, Xj[0], Xj[1], Xj[2]), P[7]);
        const float hz = __fadd_rn(dot3(P + 8, Xj[0], Xj[1], Xj[2]), P[11]);
        if (!(hz > 0.f)) return -1;
        const float dx = __fsub_rn(__fdiv_rn(hx, hz), x), dy = __fsub_rn(__fdiv_rn(hy, hz), y);
        if (!(__fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) < a.thresh)) return -1;
        if (!(__fdiv_rn(fabsf(__fsub_rn(hz, dr)), dr) < a.depth_rel)) return -1;
    }
    const float c = __fadd_rn(__fadd_rn(__fmul_rn(n.x, t.x), __fmul_rn(n.y, t.y)), __fmul_rn(n.z, t.z));
    if (!(c > a.cos_thresh)) return -1;
    *tgt = t;
    return q;
}

__device__ __forceinline__ void add_colour(const FuseArgs& a, int view, int q, float s[3])
{
    if (!a.images) return;
    const size_t i = (size_t)view * a.W * a.H + q;
    if (a.channels == 1) {
        const float g = a.images[i];
        s[0] = __fadd_rn(s[0], g);  s[1] = __fadd_rn(s[1], g);  s[2] = __fadd_rn(s[2], g);
    } else {
        const float4 c = reinterpret_cast<const float4*>(a.images)[i];
        s[0] = __fadd_rn(s[0], c.x);  s[1] = __fadd_rn(s[1], c.y);  s[2] = __fadd_rn(s[2], c.z);
    }
}

// mean colour -> uchar: clamp to [0, 255] (NaN -> 0), round half up
__device__ __forceinline__ unsigned to_uchar(float s, float cnt)
{
    float m = __fdiv_rn(s, cnt);
    m = m >= 0.f ? (m <= 255.f ? m : 255.f) : 0.f;
    return (unsigned)floorf(__fadd_rn(m, 0.5f));
}

template <int Rule>
__global__ void __launch_bounds__(kBlock) k_fuse_pixels(FuseArgs a, const float* __restrict__ cams_g, int r)
{
    extern __shared__ float cams[];
    for (int i = threadIdx.x; i < a.n * kCamFloats; i += blockDim.x) cams[i] = cams_g[i];
    __syncthreads();
    const int npix = a.W * a.H;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    int fused = 0;
    if (p < npix && !a.used[(size_t)r * npix + p]) {
        const float4 n = a.norm4[(size_t)r * npix + p];
        if (n.w >= a.dmin && n.w <= a.dmax) {
            const float* cr = cams + r * kCamFloats;
            const float x = (float)(p % a.W), y = (float)(p / a.W);
            float X[3], s[3], sn[3] = {n.x, n.y, n.z}, col[3] = {0.f, 0.f, 0.f};
            backproject(cr, x, y, n.w, X);
            s[0] = X[0];  s[1] = X[1];  s[2] = X[2];
            add_colour(a, r, p, col);
            int cnt = 0;
            for (int j = 0; j < a.n; j++) {
                if (j == r) continue;
                const float* cj = cams + j * kCamFloats;
                float4 t;
                float u, v, Xj[3];
                const int q = consistent<Rule>(a, j, cj, cr, X, x, y, n.w, n, &t, &u, &v);
                if (q < 0) continue;
                backproject(cj, u, v, t.w, Xj);
                for (int k = 0; k < 3; k++) s[k] = __fadd_rn(s[k], Xj[k]);
                sn[0] = __fadd_rn(sn[0], t.x);  sn[1] = __fadd_rn(sn[1], t.y);  sn[2] = __fadd_rn(sn[2], t.z);
                add_colour(a, j, q, col);
                cnt++;
            }
            if (cnt >= a.num_consistent) {
                fused = 1;
                const float m = (float)(cnt + 1);
                const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(sn[0], sn[0]), __fmul_rn(sn[1], sn[1])), __fmul_rn(sn[2], sn[2])));
                float nn[3] = {0.f, 0.f, 0.f};
                if (len > 0.f)
                    for (int k = 0; k < 3; k++) nn[k] = __fdiv_rn(sn[k], len);
                const unsigned rgb = a.images ? (to_uchar(col[0], m) | to_uchar(col[1], m) << 8 | to_uchar(col[2], m) << 16) : 0u;
                a.stage[2 * (size_t)p] = make_float4(__fdiv_rn(s[0], m), __fdiv_rn(s[1], m), __fdiv_rn(s[2], m), nn[0]);
                a.stage[2 * (size_t)p + 1] = make_float4(nn[1], nn[2], __uint_as_float(rgb), 0.f);
                // marks: the same test again, now that the pixel is known to fuse (plain stores: several pixels may mark one target)
                a.used[(size_t)r * npix + p] = 1;
                for (int j = 0; j < a.n; j++) {
                    if (j == r) continue;
                    float4 t;
                    float u, v;
                    const int q = consistent<Rule>(a, j, cams + j * kCamFloats, cr, X, x, y, n.w, n, &t, &u, &v);
                    if (q >= 0) a.used[(size_t)j * npix + q] = 1;
                }
            }
        }
    }
    if (p < npix) a.flag[p] = (unsigned char)fused;
    const int c = __syncthreads_count(fused);
    if (threadIdx.x == 0) a.block_count[blockIdx.x] = c;
}

// Exclusive scan of the per-block counts in one block (ascending chunks of 1024); total in offs[nblocks].
__global__ void __launch_bounds__(1024) k_scan_blocks(const int* __restrict__ count, int* __restrict__ offs, int nblocks)
{
    __shared__ int warp_sum[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int base = 0; base < nblocks; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nblocks ? count[i] : 0;
        int x = v;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sum[w] = x;
        __syncthreads();
        if (w == 0) {
            int s = warp_sum[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += y;
            }
            warp_sum[lane] = s;                                  // inclusive over warps
        }
        __syncthreads();
        const int incl = x + (w > 0 ? warp_sum[w - 1] : 0) + carry;
        if (i < nblocks) offs[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) offs[nblocks] = carry;
}

__global__ void __launch_bounds__(kBlock) k_compact(const unsigned char* __restrict__ flag, const float4* __restrict__ stage,
                                                   const int* __restrict__ offs, int npix, int r,
                                                   unsigned char* __restrict__ out, int* __restrict__ src)
{
    __shared__ int warp_cnt[kBlock / 32];
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const int f = p < npix ? flag[p] : 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, f);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) warp_cnt[w] = __popc(ballot);
    __syncthreads();
    if (!f) return;
    int pos = offs[blockIdx.x] + __popc(ballot & ((1u << lane) - 1u));
    for (int k = 0; k < w; k++) pos += warp_cnt[k];
    const float4 a = stage[2 * (size_t)p], b = stage[2 * (size_t)p + 1];
    const float v[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
    unsigned char* o = out + (size_t)pos * GPM_FUSE_VERTEX_BYTES;
    for (int k = 0; k < 6; k++) {
        const unsigned bits = __float_as_uint(v[k]);
        for (int i = 0; i < 4; i++) o[4 * k + i] = (unsigned char)(bits >> (8 * i));
    }
    const unsigned rgb = __float_as_uint(b.z);
    o[24] = (unsigned char)rgb;  o[25] = (unsigned char)(rgb >> 8);  o[26] = (unsigned char)(rgb >> 16);
    src[2 * pos] = r;
    src[2 * pos + 1] = p;
}

struct Buffers {
    int dev_prev = -1;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    void* norm4 = nullptr;
    void* images = nullptr;
    void* used = nullptr;
    void* stage = nullptr;
    void* flag = nullptr;
    void* counts = nullptr;
    void* offs = nullptr;
    void* out = nullptr;
    void* src = nullptr;
    void* cams = nullptr;
    int* host_total = nullptr;
    ~Buffers()
    {
        if (stream) cudaStreamSynchronize(stream);
        for (void* p : {norm4, images, used, stage, flag, counts, offs, out, src, cams}) if (p) cudaFree(p);
        if (host_total) cudaFreeHost(host_total);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
        if (dev_prev >= 0) cudaSetDevice(dev_prev);
    }
};

int fail(int code, const std::string& m) { return gpm::set_last_error(code, "gpm_fuse: " + m); }

#define FU(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(GPM_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

}  // namespace

extern "C" int gpm_fuse(const gpm_fuse_desc* d, gpm_fuse_result* res) { return gpm_fuse_with_rule(d, nullptr, res); }

extern "C" int gpm_fuse_with_rule(const gpm_fuse_desc* d, const gpm_fuse_rule* rule, gpm_fuse_result* res)
{
    // every argument is checked before the first CUDA call
    if (!d || !res) return fail(GPM_E_ARG, "null descriptor or result");
    const int kind = rule ? rule->kind : GPM_FUSE_DISPARITY;
    if (kind != GPM_FUSE_DISPARITY && kind != GPM_FUSE_REPROJECTION) return fail(GPM_E_ARG, "unknown rule kind");
    if (kind == GPM_FUSE_REPROJECTION) {
        if (!(std::isfinite(rule->reproj_px) && rule->reproj_px > 0.f)) return fail(GPM_E_ARG, "reproj_px must be finite and > 0");
        if (!(std::isfinite(rule->depth_rel) && rule->depth_rel > 0.f)) return fail(GPM_E_ARG, "depth_rel must be finite and > 0");
    }
    if (d->n_views < 2 || d->n_views > GPM_FUSE_MAX_VIEWS) return fail(GPM_E_ARG, "n_views must be in [2, GPM_FUSE_MAX_VIEWS]");
    if (d->width < 1 || d->height < 1 || (long long)d->width * d->height > (1LL << 30))
        return fail(GPM_E_ARG, "bad image size");
    if (!d->norm4 || !d->P) return fail(GPM_E_ARG, "norm4 and P are required");
    if (d->images && d->channels != 1 && d->channels != 4) return fail(GPM_E_ARG, "channels must be 1 or 4");
    if (!(d->depth_min >= 0.f && d->depth_max > d->depth_min)) return fail(GPM_E_ARG, "need 0 <= depth_min < depth_max");
    if (kind == GPM_FUSE_DISPARITY && !(d->disp_thresh > 0.f)) return fail(GPM_E_ARG, "disp_thresh must be > 0");
    if (!(d->normal_thresh > 0.f && d->normal_thresh <= 180.f)) return fail(GPM_E_ARG, "normal_thresh must be in (0, 180] degrees");
    if (d->num_consistent < 1) return fail(GPM_E_ARG, "num_consistent must be >= 1");
    if (res->capacity < 0 || (res->capacity > 0 && !res->vertices && !res->source)) return fail(GPM_E_ARG, "bad result buffers");
    const int n = d->n_views, W = d->width, H = d->height;
    std::vector<gpm_fuse_camera> cams(n);
    if (gpm_fuse_cameras(d->P, n, d->cam_scale, cams.data()) != GPM_OK) return fail(GPM_E_ARG, "bad projection matrix or cam_scale");
    static_assert(sizeof(gpm_fuse_camera) == kCamFloats * sizeof(float), "camera table layout");
    res->count = 0;  res->fuse_ms = 0.f;  res->upload_ms = 0.f;

    const size_t npix = (size_t)W * H, nall = (size_t)n * npix;
    const int nblocks = (int)((npix + kBlock - 1) / kBlock);
    const size_t img_bytes = d->images ? nall * d->channels * sizeof(float) : 0;
    Buffers b;
    int dev_prev = 0;
    FU(cudaGetDevice(&dev_prev));
    FU(cudaSetDevice(d->device));
    b.dev_prev = dev_prev;
    FU(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
    for (auto& e : b.ev) FU(cudaEventCreate(&e));
    FU(cudaMalloc(&b.used, nall));
    FU(cudaMalloc(&b.stage, 2 * npix * sizeof(float4)));
    FU(cudaMalloc(&b.flag, npix));
    FU(cudaMalloc(&b.counts, nblocks * sizeof(int)));
    FU(cudaMalloc(&b.offs, (nblocks + 1) * sizeof(int)));
    FU(cudaMalloc(&b.out, npix * GPM_FUSE_VERTEX_BYTES));
    FU(cudaMalloc(&b.src, npix * 2 * sizeof(int)));
    FU(cudaMalloc(&b.cams, n * sizeof(gpm_fuse_camera)));
    FU(cudaHostAlloc((void**)&b.host_total, sizeof(int), cudaHostAllocDefault));

    const float4* norm4 = reinterpret_cast<const float4*>(d->norm4);
    const float* images = d->images;
    FU(cudaEventRecord(b.ev[0], b.stream));
    if (!d->on_device) {
        FU(cudaMalloc(&b.norm4, nall * sizeof(float4)));
        FU(cudaMemcpyAsync(b.norm4, d->norm4, nall * sizeof(float4), cudaMemcpyHostToDevice, b.stream));
        norm4 = static_cast<const float4*>(b.norm4);
        if (d->images) {
            FU(cudaMalloc(&b.images, img_bytes));
            FU(cudaMemcpyAsync(b.images, d->images, img_bytes, cudaMemcpyHostToDevice, b.stream));
            images = static_cast<const float*>(b.images);
        }
    }
    FU(cudaEventRecord(b.ev[1], b.stream));
    FU(cudaMemcpyAsync(b.cams, cams.data(), n * sizeof(gpm_fuse_camera), cudaMemcpyHostToDevice, b.stream));
    FU(cudaMemsetAsync(b.used, 0, nall, b.stream));

    FuseArgs a;
    a.norm4 = norm4;  a.images = images;  a.used = static_cast<unsigned char*>(b.used);
    a.stage = static_cast<float4*>(b.stage);  a.flag = static_cast<unsigned char*>(b.flag);
    a.block_count = static_cast<int*>(b.counts);
    a.n = n;  a.W = W;  a.H = H;  a.channels = d->images ? d->channels : 0;  a.num_consistent = d->num_consistent;
    a.dmin = d->depth_min;  a.dmax = d->depth_max;
    a.thresh = kind == GPM_FUSE_DISPARITY ? d->disp_thresh : rule->reproj_px;
    a.depth_rel = kind == GPM_FUSE_DISPARITY ? 0.f : rule->depth_rel;
    a.cos_thresh = (float)std::cos((double)d->normal_thresh * M_PI / 180.0);       // angle < thresh  <=>  dot > cos(thresh)
    const size_t smem = n * sizeof(gpm_fuse_camera);
    long long total = 0;
    for (int r = 0; r < n; r++) {
        if (kind == GPM_FUSE_DISPARITY)
            k_fuse_pixels<GPM_FUSE_DISPARITY><<<nblocks, kBlock, smem, b.stream>>>(a, static_cast<const float*>(b.cams), r);
        else
            k_fuse_pixels<GPM_FUSE_REPROJECTION><<<nblocks, kBlock, smem, b.stream>>>(a, static_cast<const float*>(b.cams), r);
        FU(cudaGetLastError());
        k_scan_blocks<<<1, 1024, 0, b.stream>>>(a.block_count, static_cast<int*>(b.offs), nblocks);
        FU(cudaGetLastError());
        k_compact<<<nblocks, kBlock, 0, b.stream>>>(a.flag, a.stage, static_cast<const int*>(b.offs), (int)npix, r,
                                                    static_cast<unsigned char*>(b.out), static_cast<int*>(b.src));
        FU(cudaGetLastError());
        FU(cudaMemcpyAsync(b.host_total, static_cast<int*>(b.offs) + nblocks, sizeof(int), cudaMemcpyDeviceToHost, b.stream));
        FU(cudaStreamSynchronize(b.stream));
        const long long c = *b.host_total;
        const long long fit = total >= res->capacity ? 0 : std::min(c, res->capacity - total);
        if (fit > 0 && res->vertices)
            FU(cudaMemcpyAsync(res->vertices + total * GPM_FUSE_VERTEX_BYTES, b.out, fit * GPM_FUSE_VERTEX_BYTES,
                               cudaMemcpyDeviceToHost, b.stream));
        if (fit > 0 && res->source)
            FU(cudaMemcpyAsync(res->source + total * 2, b.src, fit * 2 * sizeof(int), cudaMemcpyDeviceToHost, b.stream));
        total += c;
    }
    FU(cudaEventRecord(b.ev[2], b.stream));
    if (res->used) FU(cudaMemcpyAsync(res->used, b.used, nall, cudaMemcpyDeviceToHost, b.stream));
    FU(cudaStreamSynchronize(b.stream));
    if (!d->on_device) FU(cudaEventElapsedTime(&res->upload_ms, b.ev[0], b.ev[1]));
    FU(cudaEventElapsedTime(&res->fuse_ms, b.ev[1], b.ev[2]));
    res->count = total;
    if (total > res->capacity)
        return fail(GPM_E_ARG, "result capacity " + std::to_string(res->capacity) + " < " + std::to_string(total) + " vertices");
    return GPM_OK;
}
