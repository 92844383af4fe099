// gpm_scale.cu — the two per-pixel steps of the coarse-to-fine scheme (DESIGN.md §19): one level of the image pyramid
// (gpm_downsample) and the joint bilateral upsampling of a coarse level's planes (the kernel behind gpm_upsample_planes,
// whose context side is in gpm_api.cu).
// Compiled on its own, without --use_fast_math (gipuma_b200/build.py): every fp32 operation below is an explicit
// round-to-nearest intrinsic, denormals are kept and nothing is contracted, so oracle/pyscale.py's numpy float32 restatement
// reproduces every output bit.
#include "../../include/gipuma_b200.h"
#include "gpm_scale.cuh"

#include <cuda_runtime.h>

#include <string>

namespace gpm { int set_last_error(int code, const std::string& msg); }

namespace {

// (0.25 a + 0.5 b) + 0.25 c, one rounding per operation
__device__ __forceinline__ float binomial(float a, float b, float c)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(0.25f, a), __fmul_rn(0.5f, b)), __fmul_rn(0.25f, c));
}

// Coarse pixel (xc, yc) is the [1 2 1]/4 x [1 2 1]/4 average around fine pixel (2 xc, 2 yc), borders replicated: per channel,
// the horizontal pass of each of the three source rows, then the vertical pass.
__global__ void k_downsample(const float* __restrict__ src, size_t pitch, int W, int H, int ch, float* __restrict__ dst,
                             int Wc, int Hc)
{
    const int xc = blockIdx.x * blockDim.x + threadIdx.x, yc = blockIdx.y * blockDim.y + threadIdx.y;
    if (xc >= Wc || yc >= Hc) return;
    const int x = 2 * xc, y = 2 * yc;
    const int xs[3] = {max(x - 1, 0), x, min(x + 1, W - 1)};
    const int ys[3] = {max(y - 1, 0), y, min(y + 1, H - 1)};
    for (int c = 0; c < ch; c++) {
        float h[3];
        for (int k = 0; k < 3; k++) {
            const float* row = src + (size_t)ys[k] * pitch;
            h[k] = binomial(row[xs[0] * ch + c], row[xs[1] * ch + c], row[xs[2] * ch + c]);
        }
        dst[((size_t)yc * Wc + xc) * ch + c] = binomial(h[0], h[1], h[2]);
    }
}

__device__ __forceinline__ float dot3(float a0, float a1, float a2, float x, float y, float z)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, x), __fmul_rn(a1, y)), __fmul_rn(a2, z));
}

// squared guide difference I(p) - I(q) of two texels of the padded guide
__device__ __forceinline__ float guide_d2(const gpm::JbuArgs& a, size_t p, size_t q)
{
    if (!a.color) {
        const float d = __fsub_rn(a.guide[p], a.guide[q]);
        return __fmul_rn(d, d);
    }
    const float4 u = reinterpret_cast<const float4*>(a.guide)[p], v = reinterpret_cast<const float4*>(a.guide)[q];
    const float dx = __fsub_rn(u.x, v.x), dy = __fsub_rn(u.y, v.y), dz = __fsub_rn(u.z, v.z);
    return dot3(dx, dy, dz, dx, dy, dz);
}

// One thread per fine pixel p: the planes of the coarse pixels within `radius` of c = p / 2, weighted by a spatial table
// and a Cauchy range weight on the fine guide, averaged as depth along p's ray and as normal (DESIGN.md §19).
__global__ void __launch_bounds__(256) k_jbu(const gpm::JbuArgs a)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const float px = (float)x, py = (float)y;
    const float rx = dot3(a.kinv[0], a.kinv[1], a.kinv[2], px, py, 1.f);
    const float ry = dot3(a.kinv[3], a.kinv[4], a.kinv[5], px, py, 1.f);
    const float rz = dot3(a.kinv[6], a.kinv[7], a.kinv[8], px, py, 1.f);
    const int cx = x >> 1, cy = y >> 1;
    const float* ws = a.ws + ((y & 1) * 2 + (x & 1)) * gpm::kJbuSide * gpm::kJbuSide;
    const size_t gp = (size_t)(y + a.apron) * a.guide_pitch + (x + a.apron);
    float sw = 0.f, swz = 0.f, nx = 0.f, ny = 0.f, nz = 0.f;
    for (int j = -a.radius; j <= a.radius; j++) {
        const int qy = cy + j;
        if (qy < 0 || qy >= a.Hc) continue;
        for (int i = -a.radius; i <= a.radius; i++) {
            const int qx = cx + i;
            if (qx < 0 || qx >= a.Wc) continue;
            const float4 n = a.coarse[(size_t)qy * a.Wc + qx];
            const float z = __fdiv_rn(-n.w, dot3(n.x, n.y, n.z, rx, ry, rz));
            if (!(isfinite(z) && z >= a.depth_min && z <= a.depth_max)) continue;
            const size_t gq = (size_t)(2 * qy + a.apron) * a.guide_pitch + (2 * qx + a.apron);
            const float wr = __fdiv_rn(1.f, __fadd_rn(1.f, __fmul_rn(guide_d2(a, gp, gq), a.k_range)));
            const float w = __fmul_rn(ws[(j + gpm::kJbuMaxRadius) * gpm::kJbuSide + i + gpm::kJbuMaxRadius], wr);
            sw = __fadd_rn(sw, w);
            swz = __fadd_rn(swz, __fmul_rn(w, z));
            nx = __fadd_rn(nx, __fmul_rn(w, n.x));
            ny = __fadd_rn(ny, __fmul_rn(w, n.y));
            nz = __fadd_rn(nz, __fmul_rn(w, n.z));
        }
    }
    const float len = __fsqrt_rn(dot3(nx, ny, nz, nx, ny, nz));
    float4 out;
    float depth;
    if (sw > 0.f && len > 0.f) {
        const float Z = __fdiv_rn(swz, sw);
        out.x = __fdiv_rn(nx, len);  out.y = __fdiv_rn(ny, len);  out.z = __fdiv_rn(nz, len);
        out.w = -dot3(out.x, out.y, out.z, __fmul_rn(Z, rx), __fmul_rn(Z, ry), __fmul_rn(Z, rz));
        depth = Z;
    } else {                                             // nothing to average: c's plane, no depth
        out = a.coarse[(size_t)cy * a.Wc + cx];
        depth = 0.f;
    }
    const size_t p = (size_t)y * a.W + x;
    if (a.planes) a.planes[p] = out;
    if (a.depth) a.depth[p] = depth;
}

struct Buffers {
    int dev_prev = -1;
    cudaStream_t stream = nullptr;
    void* src = nullptr;
    void* dst = nullptr;
    ~Buffers()
    {
        if (stream) cudaStreamSynchronize(stream);
        cudaFree(src);  cudaFree(dst);
        if (stream) cudaStreamDestroy(stream);
        if (dev_prev >= 0) cudaSetDevice(dev_prev);
    }
};

int fail(int code, const std::string& m) { return gpm::set_last_error(code, "gpm_downsample: " + m); }

#define DS(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(GPM_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

}  // namespace

namespace gpm {
cudaError_t launch_jbu(const JbuArgs& a, cudaStream_t stream)
{
    const dim3 b(32, 8), g((a.W + 31) / 32, (a.H + 7) / 8);
    k_jbu<<<g, b, 0, stream>>>(a);
    return cudaGetLastError();
}
}  // namespace gpm

extern "C" int gpm_downsample(int device, const float* src, size_t pitch_bytes, int width, int height, int channels, float* dst,
                              int on_device)
{
    if (!src || !dst) return fail(GPM_E_ARG, "null image");
    if (width < 1 || height < 1 || (long long)width * height > (1LL << 30)) return fail(GPM_E_ARG, "bad image size");
    if (channels != 1 && channels != 4) return fail(GPM_E_ARG, "channels must be 1 or 4");
    const size_t row = (size_t)width * channels * sizeof(float);
    if (pitch_bytes == 0) pitch_bytes = row;
    if (pitch_bytes < row || pitch_bytes % sizeof(float)) return fail(GPM_E_ARG, "pitch_bytes must be >= the row size and a multiple of 4");
    const int Wc = (width + 1) / 2, Hc = (height + 1) / 2;
    const size_t out_bytes = (size_t)Wc * Hc * channels * sizeof(float);
    Buffers b;
    int dev_prev = 0;
    DS(cudaGetDevice(&dev_prev));
    DS(cudaSetDevice(device));
    b.dev_prev = dev_prev;
    DS(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
    const float* s = src;
    float* d = dst;
    size_t pitch = pitch_bytes / sizeof(float);
    if (!on_device) {
        DS(cudaMalloc(&b.src, row * height));
        DS(cudaMalloc(&b.dst, out_bytes));
        DS(cudaMemcpy2DAsync(b.src, row, src, pitch_bytes, row, height, cudaMemcpyHostToDevice, b.stream));
        s = static_cast<const float*>(b.src);
        d = static_cast<float*>(b.dst);
        pitch = row / sizeof(float);
    }
    const dim3 blk(32, 8), grid((Wc + 31) / 32, (Hc + 7) / 8);
    k_downsample<<<grid, blk, 0, b.stream>>>(s, pitch, width, height, channels, d, Wc, Hc);
    DS(cudaGetLastError());
    if (!on_device) DS(cudaMemcpyAsync(dst, d, out_bytes, cudaMemcpyDeviceToHost, b.stream));
    DS(cudaStreamSynchronize(b.stream));
    return GPM_OK;
}
