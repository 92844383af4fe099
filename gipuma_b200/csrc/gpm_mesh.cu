// gpm_mesh.cu — meshing of depth maps (DESIGN.md §24): TSDF integration into a box of voxels, then marching tetrahedra.
// Compiled on its own, without --use_fast_math, with the flags of gpm_fuse.cu (gipuma_b200/build.py): every fp32 operation
// below is an explicit round-to-nearest intrinsic, denormals are kept, nothing is contracted, and oracle/mesh_oracle.c
// restates the same operations in the same order, so the GPU and the restatement agree bit for bit.
//
// gpm_tsdf_integrate, one launch:
//   k_tsdf          one thread per voxel: every view in ascending order, the sums in registers, the camera table in shared
//                   memory as k_fuse_pixels keeps it
// gpm_mesh_extract, on the lattice of voxel centres (point p = cube p's lowest corner):
//   k_cubes         per point: which of its cube's 6 tetrahedra are meshed (a bit each); per-block face counts
//   k_edges         per point: which of its 7 outgoing edges carry a vertex (a bit each); per-block vertex counts
//   k_scan_blocks   one block: exclusive scans of the per-block counts (64-bit, fixed order, no atomics)
//   k_vertices      per point: its first vertex id (block offset + block scan), its vertices written at their ids
//   k_faces         per point: its cube's faces written at block offset + block scan, in tetrahedron order
#include "../../include/gipuma_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace gpm { int set_last_error(int code, const std::string& msg); }

namespace {

constexpr int kBlock = 256;
constexpr int kCamFloats = 22;                     // gpm_fuse_camera: M_inv[9], P[12], f
constexpr unsigned kNaN = 0x7fffffffu;             // D where no view contributed

// Corners of a cube as 3-bit masks (bit 0: +x, bit 1: +y, bit 2: +z).  Kuhn tetrahedron t of the axis permutation
// (a, b, c) has the corners 0, e_a, e_a + e_b, 7: a chain of masks, each the one before plus one axis.
__constant__ unsigned char kPerm[6][2] = {{0, 1}, {0, 2}, {1, 0}, {1, 2}, {2, 0}, {2, 1}};     // (a, b) of xyz .. zyx
__constant__ signed char kParity[6] = {1, -1, -1, 1, 1, -1};                                  // sign of (a, b, c)
// direction mask -> direction index in the order x, y, z, x+y, x+z, y+z, x+y+z (mask 0 unused)
__constant__ unsigned char kDirIndex[8] = {0, 0, 1, 3, 2, 4, 5, 6};
__constant__ unsigned char kDirMask[7] = {1, 2, 4, 3, 5, 6, 7};

__device__ __forceinline__ void tet_corners(int t, unsigned char c[4])
{
    const int a = 1 << kPerm[t][0], b = 1 << kPerm[t][1];
    c[0] = 0;  c[1] = (unsigned char)a;  c[2] = (unsigned char)(a | b);  c[3] = 7;
}

__device__ __forceinline__ float dot3(const float* a, float x, float y, float z)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(a[0], x), __fmul_rn(a[1], y)), __fmul_rn(a[2], z));
}

// the centre of lattice index i on one axis: origin + (i + 0.5) * s
__device__ __forceinline__ float centre(float o, int i, float s) { return __fadd_rn(o, __fmul_rn(__fadd_rn((float)i, 0.5f), s)); }

struct Box {
    int nx, ny, nz;
    float o[3], s;
};

struct TsdfArgs {
    const float* depth;                            // n * H * W
    float* D;
    unsigned short* Wt;
    int n, W, H;
    float dmin, dmax, trunc;
    Box box;
};

__global__ void __launch_bounds__(kBlock) k_tsdf(TsdfArgs a, const float* __restrict__ cams_g)
{
    extern __shared__ float cams[];
    for (int i = threadIdx.x; i < a.n * kCamFloats; i += blockDim.x) cams[i] = cams_g[i];
    __syncthreads();
    const long long nvox = (long long)a.box.nx * a.box.ny * a.box.nz;
    const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nvox) return;
    const int i = (int)(v % a.box.nx), j = (int)((v / a.box.nx) % a.box.ny), k = (int)(v / ((long long)a.box.nx * a.box.ny));
    const float X0 = centre(a.box.o[0], i, a.box.s), X1 = centre(a.box.o[1], j, a.box.s), X2 = centre(a.box.o[2], k, a.box.s);
    const size_t npix = (size_t)a.W * a.H;
    float S = 0.f;
    int w = 0;
    for (int n = 0; n < a.n; n++) {
        const float* P = cams + n * kCamFloats + 9;
        const float hz = __fadd_rn(dot3(P + 8, X0, X1, X2), P[11]);
        if (!(hz > 0.f)) continue;
        const float hx = __fadd_rn(dot3(P, X0, X1, X2), P[3]);
        const float hy = __fadd_rn(dot3(P + 4, X0, X1, X2), P[7]);
        const float fu = floorf(__fadd_rn(__fdiv_rn(hx, hz), 0.5f));
        const float fv = floorf(__fadd_rn(__fdiv_rn(hy, hz), 0.5f));
        if (!(fu >= 0.f && fu < (float)a.W && fv >= 0.f && fv < (float)a.H)) continue;
        const float d = a.depth[n * npix + (size_t)fv * a.W + (size_t)fu];
        if (!(d > 0.f && d >= a.dmin && d <= a.dmax)) continue;
        const float sdf = __fsub_rn(d, hz);
        if (sdf < -a.trunc) continue;                                      // behind the surface
        S = __fadd_rn(S, __fdiv_rn(fminf(sdf, a.trunc), a.trunc));
        w++;
    }
    a.D[v] = w ? __fdiv_rn(S, (float)w) : __uint_as_float(kNaN);
    a.Wt[v] = (unsigned short)w;
}

struct MeshArgs {
    const float* D;
    const unsigned short* Wt;
    int min_weight;
    Box box;
    unsigned char* tets;                           // per point: bit t = tetrahedron t of its cube is meshed
    unsigned char* edges;                          // per point: bit r = its edge in direction r carries a vertex
    int* vbase;                                    // per point: its first vertex id
    int* block_count;
    const long long* offs;
    float* verts;
    int* faces;
};

__device__ __forceinline__ void coords(const Box& b, long long p, int c[3])
{
    c[0] = (int)(p % b.nx);  c[1] = (int)((p / b.nx) % b.ny);  c[2] = (int)(p / ((long long)b.nx * b.ny));
}

__device__ __forceinline__ long long offset(const Box& b, int m)
{
    return (long long)(m & 1) + (long long)((m >> 1) & 1) * b.nx + (long long)((m >> 2) & 1) * b.nx * b.ny;
}

// valid / inside bits of the 8 corners of cube p (whose lowest corner is p; the caller checks the cube exists)
__device__ __forceinline__ void cube_bits(const MeshArgs& a, long long p, unsigned& valid, unsigned& inside)
{
    valid = inside = 0;
    for (int m = 0; m < 8; m++) {
        const long long q = p + offset(a.box, m);
        if (a.Wt[q] >= a.min_weight) valid |= 1u << m;
        if (a.D[q] < 0.f) inside |= 1u << m;
    }
}

__device__ __forceinline__ bool has_cube(const Box& b, const int c[3]) { return c[0] < b.nx - 1 && c[1] < b.ny - 1 && c[2] < b.nz - 1; }

// faces of a meshed tetrahedron from its corners' inside bits (in chain order): 1 or 3 inside -> 1, 2 -> 2
__device__ __forceinline__ int tet_faces(int in4) { const int n = __popc(in4); return n == 2 ? 2 : (n & 1); }

// Exclusive block scan of one int per thread (kBlock threads); returns the thread's prefix.
__device__ __forceinline__ int block_scan(int x, int* warp_sum)
{
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int s = x;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
    }
    if (lane == 31) warp_sum[w] = s;
    __syncthreads();
    int before = 0;
    for (int k = 0; k < w; k++) before += warp_sum[k];
    return before + s - x;
}

__global__ void __launch_bounds__(kBlock) k_cubes(MeshArgs a, long long npts)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int faces = 0;
    if (p < npts) {
        int c[3];
        coords(a.box, p, c);
        unsigned tets = 0;
        if (has_cube(a.box, c)) {
            unsigned valid, inside;
            cube_bits(a, p, valid, inside);
            for (int t = 0; t < 6; t++) {
                unsigned char cc[4];
                tet_corners(t, cc);
                bool ok = true;
                int in4 = 0;
                for (int r = 0; r < 4; r++) {
                    ok = ok && ((valid >> cc[r]) & 1u);
                    in4 |= (int)((inside >> cc[r]) & 1u) << r;
                }
                if (!ok) continue;
                tets |= 1u << t;
                faces += tet_faces(in4);
            }
        }
        a.tets[p] = (unsigned char)tets;
    }
    const int c = __reduce_add_sync(0xffffffffu, faces);
    __shared__ int warp_sum[kBlock / 32];
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int k = 0; k < kBlock / 32; k++) s += warp_sum[k];
        a.block_count[blockIdx.x] = s;
    }
}

// Edge (p, direction r) carries a vertex when both ends are valid, exactly one is inside, and a meshed tetrahedron has it:
// a tetrahedron of cube p - c1 (c1 a corner mask disjoint from the direction's) whose chain holds both c1 and c1 | dir.
__global__ void __launch_bounds__(kBlock) k_edges(MeshArgs a, long long npts)
{
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned bits = 0;
    if (p < npts && a.Wt[p] >= a.min_weight) {
        int c[3];
        coords(a.box, p, c);
        const int n[3] = {a.box.nx, a.box.ny, a.box.nz};
        const bool in_p = a.D[p] < 0.f;
        for (int r = 0; r < 7; r++) {
            const int m = kDirMask[r];
            bool ok = true;
            for (int ax = 0; ax < 3; ax++) ok = ok && c[ax] + ((m >> ax) & 1) < n[ax];
            if (!ok) continue;
            const long long q = p + offset(a.box, m);
            if (!(a.Wt[q] >= a.min_weight) || (a.D[q] < 0.f) == in_p) continue;
            bool used = false;
            for (int c1 = 0; c1 < 8 && !used; c1++) {
                if (c1 & m) continue;
                bool inb = true;
                for (int ax = 0; ax < 3; ax++) inb = inb && c[ax] - ((c1 >> ax) & 1) >= 0;
                if (!inb) continue;
                const long long o = p - offset(a.box, c1);
                const unsigned tets = a.tets[o];
                for (int t = 0; t < 6 && !used; t++) {
                    if (!((tets >> t) & 1u)) continue;
                    unsigned char cc[4];
                    tet_corners(t, cc);
                    bool h1 = false, h2 = false;
                    for (int k = 0; k < 4; k++) { h1 = h1 || cc[k] == c1;  h2 = h2 || cc[k] == (c1 | m); }
                    used = h1 && h2;
                }
            }
            if (used) bits |= 1u << r;
        }
    }
    if (p < npts) a.edges[p] = (unsigned char)bits;
    const int c = __reduce_add_sync(0xffffffffu, __popc(bits));
    __shared__ int warp_sum[kBlock / 32];
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int k = 0; k < kBlock / 32; k++) s += warp_sum[k];
        a.block_count[blockIdx.x] = s;
    }
}

// Exclusive scan of the per-block counts in one block (ascending chunks of 1024), in 64 bits; total in offs[nblocks].
__global__ void __launch_bounds__(1024) k_scan_blocks(const int* __restrict__ count, long long* __restrict__ offs, long long nblocks)
{
    __shared__ long long warp_sum[32];
    __shared__ long long carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (long long base = 0; base < nblocks; base += 1024) {
        const long long i = base + threadIdx.x;
        const long long v = i < nblocks ? count[i] : 0;
        long long x = v;
        for (int o = 1; o < 32; o <<= 1) {
            const long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sum[w] = x;
        __syncthreads();
        if (w == 0) {
            long long s = warp_sum[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const long long y = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += y;
            }
            warp_sum[lane] = s;
        }
        __syncthreads();
        const long long incl = x + (w > 0 ? warp_sum[w - 1] : 0) + carry;
        if (i < nblocks) offs[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) offs[nblocks] = carry;
}

// the vertex of edge (p, direction mask m): x_p + t (x_q - x_p) per axis, t = D_p / (D_p - D_q)
__device__ __forceinline__ void edge_vertex(const MeshArgs& a, long long p, const int c[3], int m, float out[3])
{
    const long long q = p + offset(a.box, m);
    const float dp = a.D[p], dq = a.D[q];
    const float t = __fdiv_rn(dp, __fsub_rn(dp, dq));
    for (int ax = 0; ax < 3; ax++) {
        const float xp = centre(a.box.o[ax], c[ax], a.box.s);
        const float xq = centre(a.box.o[ax], c[ax] + ((m >> ax) & 1), a.box.s);
        out[ax] = __fadd_rn(xp, __fmul_rn(t, __fsub_rn(xq, xp)));
    }
}

__global__ void __launch_bounds__(kBlock) k_vertices(MeshArgs a, long long npts)
{
    __shared__ int warp_sum[kBlock / 32];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned bits = p < npts ? a.edges[p] : 0u;
    const int base = (int)(a.offs[blockIdx.x] + block_scan(__popc(bits), warp_sum));    // < 2^31: checked on the host
    if (p >= npts) return;
    a.vbase[p] = base;
    if (!bits) return;
    int c[3];
    coords(a.box, p, c);
    int id = base;
    for (int r = 0; r < 7; r++) {
        if (!((bits >> r) & 1u)) continue;
        float X[3];
        edge_vertex(a, p, c, kDirMask[r], X);
        for (int ax = 0; ax < 3; ax++) a.verts[3 * (size_t)id + ax] = X[ax];
        id++;
    }
}

// id of the vertex on the edge between corner masks lo and hi (lo a subset of hi) of cube p
__device__ __forceinline__ int vertex_id(const MeshArgs& a, long long p, int lo, int hi)
{
    const long long q = p + offset(a.box, lo);
    const int r = kDirIndex[hi ^ lo];
    return a.vbase[q] + __popc((unsigned)a.edges[q] & ((1u << r) - 1u));
}

__device__ __forceinline__ void put(const MeshArgs& a, long long f, int x, int y, int z)
{
    a.faces[3 * f] = x;  a.faces[3 * f + 1] = y;  a.faces[3 * f + 2] = z;
}

// The faces of cube p's meshed tetrahedra, in tetrahedron order.  Corners in chain order c[0..3]; orientation sign of the
// tetrahedron (c0, c1, c2, c3) = the permutation's parity.  A triangle (E_ab, E_ac, E_ad) cut from the edges at corner a
// faces away from a when (a, b, c, d) is positively oriented.  Two inside corners i1 < i2, outside o1 < o2: the quad
// E(i1,o1), E(i1,o2), E(i2,o2), E(i2,o1) is split along E(i1,o1) - E(i2,o2), and faces out when (i1, i2, o1, o2) is
// positively oriented; otherwise both triangles are reversed.
__global__ void __launch_bounds__(kBlock) k_faces(MeshArgs a, long long npts)
{
    __shared__ int warp_sum[kBlock / 32];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned tets = p < npts ? a.tets[p] : 0u;
    unsigned inside = 0, valid = 0;
    if (tets) cube_bits(a, p, valid, inside);
    int count = 0;
    for (int t = 0; t < 6; t++) {
        if (!((tets >> t) & 1u)) continue;
        unsigned char cc[4];
        tet_corners(t, cc);
        int in4 = 0;
        for (int r = 0; r < 4; r++) in4 |= (int)((inside >> cc[r]) & 1u) << r;
        count += tet_faces(in4);
    }
    long long f = a.offs[blockIdx.x] + block_scan(count, warp_sum);
    if (!count) return;
    for (int t = 0; t < 6; t++) {
        if (!((tets >> t) & 1u)) continue;
        unsigned char cc[4];
        tet_corners(t, cc);
        int in4 = 0;
        for (int r = 0; r < 4; r++) in4 |= (int)((inside >> cc[r]) & 1u) << r;
        const int nin = __popc(in4);
        if (nin == 0 || nin == 4) continue;
        const int par = kParity[t];
        auto E = [&](int u, int v) { return u < v ? vertex_id(a, p, cc[u], cc[v]) : vertex_id(a, p, cc[v], cc[u]); };
        if (nin != 2) {
            // the lone corner: the inside one of 1, the outside one of 3
            const int lone = __ffs(nin == 1 ? in4 : (~in4 & 15)) - 1;
            int o[3], k = 0;
            for (int r = 0; r < 4; r++) if (r != lone) o[k++] = r;
            // (lone, o0, o1, o2) has the orientation par * (-1)^lone; the triangle must face away from an inside lone
            // corner and towards an outside one
            const bool away = (par * ((lone & 1) ? -1 : 1)) > 0;
            const bool keep = (nin == 1) == away;
            const int e0 = E(lone, o[0]), e1 = E(lone, o[1]), e2 = E(lone, o[2]);
            if (keep) put(a, f, e0, e1, e2); else put(a, f, e0, e2, e1);
            f++;
        } else {
            int in[2], out[2], ki = 0, ko = 0;
            for (int r = 0; r < 4; r++) { if ((in4 >> r) & 1) in[ki++] = r; else out[ko++] = r; }
            // parity of the permutation (in0, in1, out0, out1) of (0, 1, 2, 3): its inversions
            const int seq[4] = {in[0], in[1], out[0], out[1]};
            int inv = 0;
            for (int x = 0; x < 4; x++) for (int y = x + 1; y < 4; y++) inv += seq[x] > seq[y];
            const bool pos = (par * ((inv & 1) ? -1 : 1)) > 0;
            const int q0 = E(in[0], out[0]), q1 = E(in[0], out[1]), q2 = E(in[1], out[1]), q3 = E(in[1], out[0]);
            if (pos) { put(a, f, q0, q1, q2);  put(a, f + 1, q0, q2, q3); }
            else     { put(a, f, q0, q3, q2);  put(a, f + 1, q0, q2, q1); }
            f += 2;
        }
    }
}

struct Buffers {
    int dev_prev = -1;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    void* p[12] = {};
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

template <class T>
cudaError_t alloc(Buffers& b, int& used, T** ptr, size_t count)
{
    void* v = nullptr;
    const cudaError_t e = cudaMalloc(&v, std::max<size_t>(count, 1) * sizeof(T));
    b.p[used++] = v;
    *ptr = static_cast<T*>(v);
    return e;
}

int fail(const char* who, int code, const std::string& m) { return gpm::set_last_error(code, std::string(who) + ": " + m); }

#define MC(who, call)                                                                              \
    do {                                                                                           \
        cudaError_t e_ = (call);                                                                   \
        if (e_ != cudaSuccess) return fail(who, GPM_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

// the box rules shared by both stages; "" when the box is good
std::string check_box(const float origin[3], float voxel, const int dims[3])
{
    for (int a = 0; a < 3; a++) {
        if (dims[a] < 2 || dims[a] > GPM_MESH_MAX_DIM) return "dims must be in [2, GPM_MESH_MAX_DIM]";
        if (!std::isfinite(origin[a])) return "origin must be finite";
    }
    if ((long long)dims[0] * dims[1] * dims[2] > INT_MAX) return "more than 2^31 - 1 voxels";
    if (!(std::isfinite(voxel) && voxel > 0.f)) return "voxel must be finite and > 0";
    return "";
}

Box make_box(const float origin[3], float voxel, const int dims[3])
{
    Box b;
    b.nx = dims[0];  b.ny = dims[1];  b.nz = dims[2];
    for (int a = 0; a < 3; a++) b.o[a] = origin[a];
    b.s = voxel;
    return b;
}

}  // namespace

extern "C" int gpm_tsdf_integrate(const gpm_tsdf_desc* d, gpm_tsdf_result* res)
{
    const char* who = "gpm_tsdf_integrate";
    // every argument is checked before the first CUDA call
    if (!d || !res) return fail(who, GPM_E_ARG, "null descriptor or result");
    if (d->n_views < 1 || d->n_views > GPM_FUSE_MAX_VIEWS) return fail(who, GPM_E_ARG, "n_views must be in [1, GPM_FUSE_MAX_VIEWS]");
    if (d->width < 1 || d->height < 1 || (long long)d->width * d->height > (1LL << 30)) return fail(who, GPM_E_ARG, "bad image size");
    if (!d->depth || !d->P || !res->D || !res->weight) return fail(who, GPM_E_ARG, "depth, P, D and weight are required");
    const std::string box = check_box(d->origin, d->voxel, d->dims);
    if (!box.empty()) return fail(who, GPM_E_ARG, box);
    if (!(std::isfinite(d->trunc) && d->trunc > 0.f)) return fail(who, GPM_E_ARG, "trunc must be finite and > 0");
    if (!(std::isfinite(d->depth_min) && std::isfinite(d->depth_max) && d->depth_min >= 0.f && d->depth_max > d->depth_min))
        return fail(who, GPM_E_ARG, "need finite 0 <= depth_min < depth_max");
    const int n = d->n_views;
    std::vector<gpm_fuse_camera> cams(n);
    if (gpm_fuse_cameras(d->P, n, d->cam_scale, cams.data()) != GPM_OK) return fail(who, GPM_E_ARG, "bad projection matrix or cam_scale");
    static_assert(sizeof(gpm_fuse_camera) == kCamFloats * sizeof(float), "camera table layout");
    res->upload_ms = res->integrate_ms = 0.f;

    const size_t nall = (size_t)n * d->width * d->height;
    const long long nvox = (long long)d->dims[0] * d->dims[1] * d->dims[2];
    Buffers b;
    int dev_prev = 0, used = 0;
    MC(who, cudaGetDevice(&dev_prev));
    MC(who, cudaSetDevice(d->device));
    b.dev_prev = dev_prev;
    MC(who, cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
    for (auto& e : b.ev) MC(who, cudaEventCreate(&e));
    float* cams_d = nullptr;
    MC(who, alloc(b, used, &cams_d, n * (size_t)kCamFloats));
    TsdfArgs a;
    a.depth = d->depth;  a.D = res->D;  a.Wt = res->weight;
    MC(who, cudaEventRecord(b.ev[0], b.stream));
    if (!d->on_device) {
        float* dep = nullptr;
        MC(who, alloc(b, used, &dep, nall));
        MC(who, alloc(b, used, &a.D, (size_t)nvox));
        MC(who, alloc(b, used, &a.Wt, (size_t)nvox));
        MC(who, cudaMemcpyAsync(dep, d->depth, nall * sizeof(float), cudaMemcpyHostToDevice, b.stream));
        a.depth = dep;
    }
    MC(who, cudaEventRecord(b.ev[1], b.stream));
    MC(who, cudaMemcpyAsync(cams_d, cams.data(), n * sizeof(gpm_fuse_camera), cudaMemcpyHostToDevice, b.stream));
    a.n = n;  a.W = d->width;  a.H = d->height;
    a.dmin = d->depth_min;  a.dmax = d->depth_max;  a.trunc = d->trunc;
    a.box = make_box(d->origin, d->voxel, d->dims);
    MC(who, cudaEventRecord(b.ev[2], b.stream));
    const long long nblocks = (nvox + kBlock - 1) / kBlock;
    k_tsdf<<<(unsigned)nblocks, kBlock, n * sizeof(gpm_fuse_camera), b.stream>>>(a, cams_d);
    MC(who, cudaGetLastError());
    MC(who, cudaEventRecord(b.ev[3], b.stream));
    if (!d->on_device) {
        MC(who, cudaMemcpyAsync(res->D, a.D, nvox * sizeof(float), cudaMemcpyDeviceToHost, b.stream));
        MC(who, cudaMemcpyAsync(res->weight, a.Wt, nvox * sizeof(unsigned short), cudaMemcpyDeviceToHost, b.stream));
    }
    MC(who, cudaStreamSynchronize(b.stream));
    if (!d->on_device) MC(who, cudaEventElapsedTime(&res->upload_ms, b.ev[0], b.ev[1]));
    MC(who, cudaEventElapsedTime(&res->integrate_ms, b.ev[2], b.ev[3]));
    return GPM_OK;
}

extern "C" int gpm_mesh_extract(const gpm_mesh_desc* d, gpm_mesh_result* res)
{
    const char* who = "gpm_mesh_extract";
    if (!d || !res) return fail(who, GPM_E_ARG, "null descriptor or result");
    if (!d->D || !d->weight) return fail(who, GPM_E_ARG, "D and weight are required");
    const std::string box = check_box(d->origin, d->voxel, d->dims);
    if (!box.empty()) return fail(who, GPM_E_ARG, box);
    if (d->min_weight < 1) return fail(who, GPM_E_ARG, "min_weight must be >= 1");
    if (res->vertex_capacity < 0 || res->face_capacity < 0 || (res->vertex_capacity > 0 && !res->vertices) ||
        (res->face_capacity > 0 && !res->faces))
        return fail(who, GPM_E_ARG, "bad result buffers");
    res->n_vertices = res->n_faces = 0;
    res->upload_ms = res->extract_ms = 0.f;

    const long long npts = (long long)d->dims[0] * d->dims[1] * d->dims[2];
    const long long nblocks = (npts + kBlock - 1) / kBlock;
    Buffers b;
    int dev_prev = 0, used = 0;
    MC(who, cudaGetDevice(&dev_prev));
    MC(who, cudaSetDevice(d->device));
    b.dev_prev = dev_prev;
    MC(who, cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking));
    for (auto& e : b.ev) MC(who, cudaEventCreate(&e));
    MC(who, cudaHostAlloc(&b.host, 2 * sizeof(long long), cudaHostAllocDefault));
    long long* totals = static_cast<long long*>(b.host);

    MeshArgs a{};
    a.D = d->D;  a.Wt = d->weight;
    a.min_weight = d->min_weight;
    a.box = make_box(d->origin, d->voxel, d->dims);
    int *fcount = nullptr, *vcount = nullptr;
    long long *foffs = nullptr, *voffs = nullptr;
    MC(who, alloc(b, used, &a.tets, (size_t)npts));
    MC(who, alloc(b, used, &a.edges, (size_t)npts));
    MC(who, alloc(b, used, &a.vbase, (size_t)npts));
    MC(who, alloc(b, used, &fcount, (size_t)nblocks));
    MC(who, alloc(b, used, &vcount, (size_t)nblocks));
    MC(who, alloc(b, used, &foffs, (size_t)nblocks + 1));
    MC(who, alloc(b, used, &voffs, (size_t)nblocks + 1));
    MC(who, cudaEventRecord(b.ev[0], b.stream));
    if (!d->on_device) {
        float* D = nullptr;
        unsigned short* W = nullptr;
        MC(who, alloc(b, used, &D, (size_t)npts));
        MC(who, alloc(b, used, &W, (size_t)npts));
        MC(who, cudaMemcpyAsync(D, d->D, npts * sizeof(float), cudaMemcpyHostToDevice, b.stream));
        MC(who, cudaMemcpyAsync(W, d->weight, npts * sizeof(unsigned short), cudaMemcpyHostToDevice, b.stream));
        a.D = D;  a.Wt = W;
    }
    MC(who, cudaEventRecord(b.ev[1], b.stream));
    const unsigned grid = (unsigned)nblocks;
    a.block_count = fcount;
    k_cubes<<<grid, kBlock, 0, b.stream>>>(a, npts);
    MC(who, cudaGetLastError());
    a.block_count = vcount;
    k_edges<<<grid, kBlock, 0, b.stream>>>(a, npts);
    MC(who, cudaGetLastError());
    k_scan_blocks<<<1, 1024, 0, b.stream>>>(fcount, foffs, nblocks);
    MC(who, cudaGetLastError());
    k_scan_blocks<<<1, 1024, 0, b.stream>>>(vcount, voffs, nblocks);
    MC(who, cudaGetLastError());
    MC(who, cudaMemcpyAsync(totals, voffs + nblocks, sizeof(long long), cudaMemcpyDeviceToHost, b.stream));
    MC(who, cudaMemcpyAsync(totals + 1, foffs + nblocks, sizeof(long long), cudaMemcpyDeviceToHost, b.stream));
    MC(who, cudaStreamSynchronize(b.stream));
    const long long nv = totals[0], nf = totals[1];
    res->n_vertices = nv;
    res->n_faces = nf;
    if (nv > INT_MAX) return fail(who, GPM_E_ARG, std::to_string(nv) + " vertices: ids at or above 2^31 are not supported");
    MC(who, alloc(b, used, &a.verts, 3 * (size_t)nv));
    MC(who, alloc(b, used, &a.faces, 3 * (size_t)nf));
    a.offs = voffs;
    k_vertices<<<grid, kBlock, 0, b.stream>>>(a, npts);
    MC(who, cudaGetLastError());
    a.offs = foffs;
    k_faces<<<grid, kBlock, 0, b.stream>>>(a, npts);
    MC(who, cudaGetLastError());
    MC(who, cudaEventRecord(b.ev[2], b.stream));
    const long long vfit = std::min(nv, res->vertex_capacity), ffit = std::min(nf, res->face_capacity);
    if (vfit > 0) MC(who, cudaMemcpyAsync(res->vertices, a.verts, 3 * vfit * sizeof(float), cudaMemcpyDeviceToHost, b.stream));
    if (ffit > 0) MC(who, cudaMemcpyAsync(res->faces, a.faces, 3 * ffit * sizeof(int), cudaMemcpyDeviceToHost, b.stream));
    MC(who, cudaStreamSynchronize(b.stream));
    if (!d->on_device) MC(who, cudaEventElapsedTime(&res->upload_ms, b.ev[0], b.ev[1]));
    MC(who, cudaEventElapsedTime(&res->extract_ms, b.ev[1], b.ev[2]));
    if (nv > res->vertex_capacity || nf > res->face_capacity)
        return fail(who, GPM_E_ARG, "result capacity (" + std::to_string(res->vertex_capacity) + " vertices, " +
                                    std::to_string(res->face_capacity) + " faces) < " + std::to_string(nv) + " vertices, " +
                                    std::to_string(nf) + " faces");
    return GPM_OK;
}

extern "C" int gpm_write_ply_mesh(const char* path, const float* vertices, long long nv, const int* faces, long long nf)
{
    const char* who = "gpm_write_ply_mesh";
    if (!path || nv < 0 || nf < 0 || (nv > 0 && !vertices) || (nf > 0 && !faces)) return fail(who, GPM_E_ARG, "bad arguments");
    for (long long i = 0; i < 3 * nf; i++)
        if (faces[i] < 0 || faces[i] >= nv) return fail(who, GPM_E_ARG, "face index out of range");
    FILE* f = fopen(path, "wb");
    if (!f) return fail(who, GPM_E_ARG, std::string("cannot open ") + path);
    fprintf(f, "ply\nformat binary_little_endian 1.0\nelement vertex %lld\nproperty float x\nproperty float y\n"
               "property float z\nelement face %lld\nproperty list uchar int vertex_indices\nend_header\n", nv, nf);
    bool ok = fwrite(vertices, sizeof(float), 3 * (size_t)nv, f) == 3 * (size_t)nv;
    std::vector<unsigned char> rec(13 * 4096);
    for (long long i0 = 0; ok && i0 < nf; i0 += 4096) {
        const long long k = std::min(nf - i0, 4096LL);
        for (long long i = 0; i < k; i++) {
            rec[13 * i] = 3;
            std::memcpy(&rec[13 * i + 1], faces + 3 * (i0 + i), 12);           // little-endian host
        }
        ok = fwrite(rec.data(), 1, 13 * k, f) == (size_t)(13 * k);
    }
    return (fclose(f) == 0 && ok) ? GPM_OK : fail(who, GPM_E_ARG, std::string("cannot write ") + path);
}
