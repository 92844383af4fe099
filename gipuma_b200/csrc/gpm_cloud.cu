// gpm_cloud.cu — exact nearest-neighbour distances between two point clouds (DESIGN.md §13).
// Compiled on its own, without --use_fast_math, with the flags of gpm_fuse.cu (gipuma_b200/build.py): d2 is computed with
// explicit round-to-nearest intrinsics, denormals are kept, and nothing is contracted.
//
// One call:
//   k_scan_points   finiteness of every coordinate and the bounding box of the data (order-independent atomics on
//                   order-preserving integer encodings)
//   k_cell_keys     per data point its cell (cx, cy, cz) of a uniform grid, computed in fp64, packed into a 63-bit key
//   CUB radix sort of (key, index), run-length encoding of the sorted keys, exclusive scan of the run lengths
//   k_gather        the data in cell order as float4
//   k_hash_insert   the occupied cells into an open-addressing hash table: key -> (first point, count)
//   k_query         thread per query: rings of cells around the query's cell, stopping when a conservative lower bound on
//                   the computed d2 of every unsearched point reaches the best d2 found or the smallest d2 whose root
//                   exceeds max_dist
#include "../../include/gipuma_b200.h"

#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace gpm { int set_last_error(int code, const std::string& msg); }

namespace {

constexpr int kBlock = 256;
constexpr int kAxisBits = 21;                                  // cells per axis < 2^21: a key fits 63 bits
constexpr unsigned long long kEmpty = ~0ull;                   // no key has bit 63 set
// cell size rule (DESIGN.md §13): at least twice the mean spacing of the data spread over its bounding box's largest face,
// at least 1/kCapCells of min(max_dist, largest extent) so that a search out to max_dist visits at most about
// (2 kCapCells + 3)^3 cells, and at least 2^-20 of the largest extent so that the key fits
constexpr double kCapCells = 16.0;

struct Grid {
    const float4* pts;                                         // data in cell order, w unused
    const unsigned long long* hkey;                            // hash slots: cell key or kEmpty
    const int2* hrange;                                        // (first point, count) of the slot's cell
    unsigned long long mask;                                   // slots - 1
    double o[3];                                               // grid origin: the data's bounding-box minimum
    double inv_h;                                              // 1 / cell size
    int G[3];                                                  // cells per axis
};

// float -> unsigned whose order is the float order (for finite values)
__device__ __forceinline__ unsigned ordered(float f)
{
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ unsigned long long mix(unsigned long long x)
{
    x ^= x >> 33;  x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;  x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

// box: NULL, or 6 unsigneds (ordered min x y z, then ~ordered max x y z, all reduced with atomicMin)
__global__ void __launch_bounds__(kBlock) k_scan_points(const float* __restrict__ p, long long n, int* __restrict__ bad,
                                                       unsigned* __restrict__ box)
{
    unsigned lo[3] = {~0u, ~0u, ~0u}, hi[3] = {~0u, ~0u, ~0u};
    int nonfinite = 0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        for (int k = 0; k < 3; k++) {
            const float v = p[3 * i + k];
            if (!isfinite(v)) nonfinite = 1;
            lo[k] = min(lo[k], ordered(v));
            hi[k] = min(hi[k], ~ordered(v));
        }
    if (__any_sync(0xffffffffu, nonfinite) && (threadIdx.x & 31) == 0) atomicOr(bad, 1);
    if (!box) return;
    for (int k = 0; k < 3; k++) {
        const unsigned a = __reduce_min_sync(0xffffffffu, lo[k]), b = __reduce_min_sync(0xffffffffu, hi[k]);
        if ((threadIdx.x & 31) == 0) { atomicMin(box + k, a);  atomicMin(box + 3 + k, b); }
    }
}

// t = (p - o) / h per axis in fp64; the same expression gives the query's position in k_query and the grid size on the host
__device__ __forceinline__ double cell_pos(float p, double o, double inv_h) { return ((double)p - o) * inv_h; }

__global__ void __launch_bounds__(kBlock) k_cell_keys(const float* __restrict__ p, int n, Grid g, unsigned long long* __restrict__ key,
                                                     int* __restrict__ idx)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long k = 0;
    for (int a = 0; a < 3; a++)
        k |= (unsigned long long)floor(cell_pos(p[3 * (size_t)i + a], g.o[a], g.inv_h)) << (kAxisBits * a);
    key[i] = k;
    idx[i] = i;
}

__global__ void __launch_bounds__(kBlock) k_gather(const float* __restrict__ p, const int* __restrict__ idx, int n, float4* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t j = 3 * (size_t)idx[i];
    out[i] = make_float4(p[j], p[j + 1], p[j + 2], 0.f);
}

__global__ void __launch_bounds__(kBlock) k_hash_insert(const unsigned long long* __restrict__ ukey, const int* __restrict__ start,
                                                       const int* __restrict__ count, int ncells, unsigned long long* hkey,
                                                       int2* hrange, unsigned long long mask)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ncells) return;
    const unsigned long long k = ukey[i];
    for (unsigned long long s = mix(k) & mask;; s = (s + 1) & mask)
        if (atomicCAS(hkey + s, kEmpty, k) == kEmpty) {        // keys are unique: a slot taken is another cell's
            hrange[s] = make_int2(start[i], count[i]);
            return;
        }
}

__device__ __forceinline__ void visit(const Grid& g, int x, int y, int z, float qx, float qy, float qz, float& best)
{
    const unsigned long long k = (unsigned long long)x | (unsigned long long)y << kAxisBits | (unsigned long long)z << (2 * kAxisBits);
    for (unsigned long long s = mix(k) & g.mask;; s = (s + 1) & g.mask) {
        const unsigned long long h = g.hkey[s];
        if (h == kEmpty) return;
        if (h != k) continue;
        const int2 r = g.hrange[s];
        for (int j = r.x; j < r.x + r.y; j++) {
            const float4 b = g.pts[j];
            const float dx = __fsub_rn(qx, b.x), dy = __fsub_rn(qy, b.y), dz = __fsub_rn(qz, b.z);
            const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
            best = fminf(best, d2);
        }
        return;
    }
}

// vstar: the smallest float whose correctly rounded square root exceeds max_dist (a d2 >= vstar can only give +inf)
__global__ void __launch_bounds__(kBlock) k_query(Grid g, const float* __restrict__ q, int n, float max_dist, float vstar,
                                                 float* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float qv[3] = {q[3 * (size_t)i], q[3 * (size_t)i + 1], q[3 * (size_t)i + 2]};
    double t[3], e = 0.0;
    int c[3];
    for (int a = 0; a < 3; a++) {
        t[a] = cell_pos(qv[a], g.o[a], g.inv_h);
        c[a] = (int)fmin(fmax(floor(t[a]), -1.0), (double)g.G[a]);        // clamped to one cell outside the grid
        e = fmax(e, fabs(t[a]));
    }
    // fp64 error of t, of the data's t (|t| <= 2^21) and of the gaps below, in cells (DESIGN.md §13)
    e = (e + 1.0) * 0x1p-50 + 0x1p-28;
    float best = __int_as_float(0x7f800000);
    for (int k = 0;; k++) {
        // after the rings < k, an unsearched point has, on some axis, a cell >= c + k or <= c - k
        double gap = INFINITY;
        for (int a = 0; a < 3; a++) {
            if (c[a] + k <= g.G[a] - 1) gap = fmin(gap, (double)(c[a] + k) - t[a]);
            if (c[a] - k >= 0) gap = fmin(gap, t[a] - (double)(c[a] - k + 1));
        }
        if (gap == INFINITY) break;                                        // the rings cover the whole grid
        const double r = fmax(gap - e, 0.0) / g.inv_h;                     // lower bound on the true distance
        const double lb = r * r * (1.0 - 1e-6) - 1e-44;                    // lower bound on the computed d2
        if (lb >= (double)fminf(best, vstar)) break;
        const int z0 = max(c[2] - k, 0), z1 = min(c[2] + k, g.G[2] - 1);
        const int y0 = max(c[1] - k, 0), y1 = min(c[1] + k, g.G[1] - 1);
        const int x0 = max(c[0] - k, 0), x1 = min(c[0] + k, g.G[0] - 1);
        for (int z = z0; z <= z1; z++) {
            const bool zs = z == c[2] - k || z == c[2] + k;
            for (int y = y0; y <= y1; y++) {
                if (zs || y == c[1] - k || y == c[1] + k) {
                    for (int x = x0; x <= x1; x++) visit(g, x, y, z, qv[0], qv[1], qv[2], best);
                } else {
                    if (c[0] - k >= 0 && c[0] - k < g.G[0]) visit(g, c[0] - k, y, z, qv[0], qv[1], qv[2], best);
                    if (k > 0 && c[0] + k >= 0 && c[0] + k < g.G[0]) visit(g, c[0] + k, y, z, qv[0], qv[1], qv[2], best);
                }
            }
        }
    }
    const float D = __fsqrt_rn(best);
    out[i] = D <= max_dist ? D : __int_as_float(0x7f800000);
}

struct Buffers {
    int dev_prev = -1;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    void* p[14] = {};
    void* host = nullptr;
    ~Buffers()
    {
        if (stream) cudaStreamSynchronize(stream);
        for (void* x : p) if (x) cudaFree(x);
        if (host) cudaFreeHost(host);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
        if (dev_prev >= 0) cudaSetDevice(dev_prev);
    }
};

int fail(int code, const std::string& m) { return gpm::set_last_error(code, "gpm_nearest_dist: " + m); }

#define CC(call)                                                                                   \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(GPM_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

template <class T>
cudaError_t alloc(Buffers& b, int& used, T** ptr, size_t count)
{
    void* v = nullptr;
    const cudaError_t e = cudaMalloc(&v, std::max<size_t>(count, 1) * sizeof(T));
    b.p[used++] = v;
    *ptr = static_cast<T*>(v);
    return e;
}

// inverse of ordered()
float decode(unsigned u)
{
    const unsigned bits = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
    float f;
    std::memcpy(&f, &bits, sizeof f);
    return f;
}

// the smallest float v with sqrt_rn(v) > m (the host's sqrtf is IEEE correctly rounded, as __fsqrt_rn)
float sqrt_threshold(float m)
{
    float v = m * m;
    if (std::sqrt(v) > m) {
        while (v > 0.f && std::sqrt(std::nextafter(v, 0.f)) > m) v = std::nextafter(v, 0.f);
    } else {
        while (!(std::sqrt(v) > m)) v = std::nextafter(v, INFINITY);
    }
    return v;
}

}  // namespace

extern "C" int gpm_nearest_dist(const gpm_nn_desc* d, gpm_nn_result* res)
{
    // every argument, and the coordinates of host inputs, are checked before the first CUDA call
    if (!d || !res) return fail(GPM_E_ARG, "null descriptor or result");
    if (d->n_query < 0 || d->n_data < 0 || d->n_query > INT_MAX || d->n_data > INT_MAX)
        return fail(GPM_E_ARG, "n_query and n_data must be in [0, 2^31 - 1]");
    if ((d->n_query > 0 && (!d->query || !res->dist)) || (d->n_data > 0 && !d->data)) return fail(GPM_E_ARG, "null point or result buffer");
    if (!(std::isfinite(d->max_dist) && d->max_dist > 0.f)) return fail(GPM_E_ARG, "max_dist must be finite and > 0");
    if (!d->on_device) {
        for (long long i = 0; i < 3 * d->n_query; i++)
            if (!std::isfinite(d->query[i])) return fail(GPM_E_ARG, "non-finite query coordinate");
        for (long long i = 0; i < 3 * d->n_data; i++)
            if (!std::isfinite(d->data[i])) return fail(GPM_E_ARG, "non-finite data coordinate");
    }
    res->upload_ms = res->build_ms = res->query_ms = 0.f;
    res->cell_size = 0.f;
    res->n_cells = 0;
    if (d->n_query == 0) return GPM_OK;
    const int nq = (int)d->n_query, nd = (int)d->n_data;

    Buffers b;
    int dev_prev = 0, used = 0;
    CC(cudaGetDevice(&dev_prev));
    CC(cudaSetDevice(d->device));
    b.dev_prev = dev_prev;
    CC(cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
    for (auto& e : b.ev) CC(cudaEventCreate(&e));
    CC(cudaHostAlloc(&b.host, 16 * sizeof(unsigned), cudaHostAllocDefault));
    unsigned* hbuf = static_cast<unsigned*>(b.host);

    const float* query = d->query;
    const float* data = d->data;
    float* out = d->on_device ? res->dist : nullptr;
    CC(cudaEventRecord(b.ev[0], b.stream));
    if (!d->on_device) {
        float *q = nullptr, *p = nullptr;
        CC(alloc(b, used, &q, 3 * (size_t)nq));
        CC(alloc(b, used, &p, 3 * (size_t)nd));
        CC(alloc(b, used, &out, (size_t)nq));
        CC(cudaMemcpyAsync(q, d->query, 3 * (size_t)nq * sizeof(float), cudaMemcpyHostToDevice, b.stream));
        if (nd) CC(cudaMemcpyAsync(p, d->data, 3 * (size_t)nd * sizeof(float), cudaMemcpyHostToDevice, b.stream));
        query = q;
        data = p;
    }
    CC(cudaEventRecord(b.ev[1], b.stream));

    // validation and bounding box: [0] bad flag, [1..6] box
    unsigned* dscan = nullptr;
    CC(alloc(b, used, &dscan, 8));
    CC(cudaMemsetAsync(dscan, 0, sizeof(unsigned), b.stream));
    CC(cudaMemsetAsync(dscan + 1, 0xff, 6 * sizeof(unsigned), b.stream));
    const int scan_blocks = 4 * 132;
    k_scan_points<<<scan_blocks, kBlock, 0, b.stream>>>(query, nq, reinterpret_cast<int*>(dscan), nullptr);
    CC(cudaGetLastError());
    if (nd) {
        k_scan_points<<<scan_blocks, kBlock, 0, b.stream>>>(data, nd, reinterpret_cast<int*>(dscan), dscan + 1);
        CC(cudaGetLastError());
    }
    CC(cudaMemcpyAsync(hbuf, dscan, 7 * sizeof(unsigned), cudaMemcpyDeviceToHost, b.stream));
    CC(cudaStreamSynchronize(b.stream));
    if (hbuf[0]) return fail(GPM_E_ARG, "non-finite coordinate");

    Grid g{};
    g.inv_h = 1.0;
    int ncells = 0;
    if (nd) {
        float lo[3], hi[3];
        double ext[3];
        for (int a = 0; a < 3; a++) {
            lo[a] = decode(hbuf[1 + a]);
            hi[a] = decode(~hbuf[4 + a]);
            g.o[a] = lo[a];
            ext[a] = (double)hi[a] - (double)lo[a];
        }
        std::sort(ext, ext + 3);
        const double L1 = ext[2], L2 = ext[1];
        const double spacing = std::max(std::sqrt(L1 * L2 / nd), L1 / nd);
        double h = std::max({2.0 * spacing, std::min((double)d->max_dist, L1) / kCapCells, L1 * 0x1p-20});
        if (!(h > 0.0)) h = d->max_dist;                                    // all data points identical
        g.inv_h = 1.0 / h;
        for (int a = 0; a < 3; a++) g.G[a] = (int)std::floor(((double)hi[a] - g.o[a]) * g.inv_h) + 1;
        res->cell_size = (float)h;

        unsigned long long *key = nullptr, *key2 = nullptr, *ukey = nullptr, *hkey = nullptr;
        int *idx = nullptr, *idx2 = nullptr, *count = nullptr, *start = nullptr, *nruns = nullptr;
        float4* pts = nullptr;
        CC(alloc(b, used, &key, nd));
        CC(alloc(b, used, &key2, nd));
        CC(alloc(b, used, &idx, nd));
        CC(alloc(b, used, &idx2, nd));
        CC(alloc(b, used, &pts, nd));
        const int blocks = (nd + kBlock - 1) / kBlock;
        k_cell_keys<<<blocks, kBlock, 0, b.stream>>>(data, nd, g, key, idx);
        CC(cudaGetLastError());
        // one temporary allocation serves the sort, the run-length encoding and the scan
        size_t t_sort = 0, t_rle = 0, t_scan = 0;
        CC(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, key, key2, idx, idx2, nd, 0, 3 * kAxisBits, b.stream));
        CC(cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, key2, key, idx, idx, nd, b.stream));
        CC(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, idx, idx, nd, b.stream));
        unsigned char* tmp = nullptr;
        const size_t t_bytes = std::max({t_sort, t_rle, t_scan});
        CC(alloc(b, used, &tmp, t_bytes));
        size_t tb = t_bytes;
        CC(cub::DeviceRadixSort::SortPairs(tmp, tb, key, key2, idx, idx2, nd, 0, 3 * kAxisBits, b.stream));
        k_gather<<<blocks, kBlock, 0, b.stream>>>(data, idx2, nd, pts);
        CC(cudaGetLastError());
        ukey = key;                                                         // the unsorted keys are no longer needed
        count = idx;
        CC(alloc(b, used, &nruns, 1));
        tb = t_bytes;
        CC(cub::DeviceRunLengthEncode::Encode(tmp, tb, key2, ukey, count, nruns, nd, b.stream));
        CC(cudaMemcpyAsync(hbuf + 8, nruns, sizeof(int), cudaMemcpyDeviceToHost, b.stream));
        CC(cudaStreamSynchronize(b.stream));
        ncells = (int)hbuf[8];
        start = idx2;
        tb = t_bytes;
        CC(cub::DeviceScan::ExclusiveSum(tmp, tb, count, start, ncells, b.stream));
        unsigned long long slots = 1;
        while (slots < 2ull * (unsigned long long)ncells) slots <<= 1;
        int2* hrange = nullptr;
        CC(alloc(b, used, &hkey, slots));
        CC(alloc(b, used, &hrange, slots));
        CC(cudaMemsetAsync(hkey, 0xff, slots * sizeof(unsigned long long), b.stream));
        k_hash_insert<<<(ncells + kBlock - 1) / kBlock, kBlock, 0, b.stream>>>(ukey, start, count, ncells, hkey, hrange, slots - 1);
        CC(cudaGetLastError());
        g.pts = pts;  g.hkey = hkey;  g.hrange = hrange;  g.mask = slots - 1;
    }
    res->n_cells = ncells;
    CC(cudaEventRecord(b.ev[2], b.stream));
    k_query<<<(nq + kBlock - 1) / kBlock, kBlock, 0, b.stream>>>(g, query, nq, d->max_dist, sqrt_threshold(d->max_dist), out);
    CC(cudaGetLastError());
    CC(cudaEventRecord(b.ev[3], b.stream));
    if (!d->on_device) CC(cudaMemcpyAsync(res->dist, out, (size_t)nq * sizeof(float), cudaMemcpyDeviceToHost, b.stream));
    CC(cudaStreamSynchronize(b.stream));
    if (!d->on_device) CC(cudaEventElapsedTime(&res->upload_ms, b.ev[0], b.ev[1]));
    CC(cudaEventElapsedTime(&res->build_ms, b.ev[1], b.ev[2]));
    CC(cudaEventElapsedTime(&res->query_ms, b.ev[2], b.ev[3]));
    return GPM_OK;
}
