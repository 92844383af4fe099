// gpm_kernels.cuh — __global__ kernels of the PatchMatch hot path (sm_90a).  See gpm_device.cuh.
#pragma once
#include "gpm_device.cuh"
#include <cuda.h>                 // CUtensorMap (type only; the encoder is fetched through cudaGetDriverEntryPoint)
#include <curand_kernel.h>

namespace gpm {

__host__ __device__ inline int tile_floats(const KParams& P) { return P.tile_stride * P.tile_w * (P.color ? 4 : 1); }
__host__ __device__ inline int fixed_smem_floats(const KParams& P) { return (tile_floats(P) + P.V * GPM_VIEWCAM_FLOATS + 3) & ~3; }
// ncc, extra: the NCC kernels' larger per-warp scratch and a variant's extra floats per warp (warp_scratch_floats)
__device__ __forceinline__ unsigned long long* block_mbar(const KParams& P, float* smem_base, bool ncc = false, int extra = 0)
{
    return reinterpret_cast<unsigned long long*>(smem_base + fixed_smem_floats(P) + (size_t)P.nwarps * warp_scratch_floats(P.ns_pad, P.V, P.color, ncc, extra) + 2);
}
__device__ __forceinline__ unsigned char* block_perm(const KParams& P, float* smem_base, bool ncc = false, int extra = 0)
{
    return reinterpret_cast<unsigned char*>(smem_base + fixed_smem_floats(P) + (size_t)P.nwarps * warp_scratch_floats(P.ns_pad, P.V, P.color, ncc, extra) + 4);
}

// ---- TMA (cp.async.bulk.tensor) + mbarrier primitives -------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, unsigned long long* bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity)
{
    unsigned done = 0;
    for (int spin = 0; !done; spin++) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (spin > (1 << 22)) __trap();          // a lost TMA transaction must fail loudly, not hang the GPU
    }
}

// Stage the (32+2*halo)^2 reference window of tile (bx, by) and the per-view camera table in shared memory.
// Unlike the reference's loader (gipuma.cu:1510-1525, skipped by threads that left early — SURVEY.md §7),
// the whole window is always defined.  One elected thread issues a single 2-D TMA box copy (cp.async.bulk.tensor) from
// the replicate-padded reference image and the block waits on its mbarrier while the other threads copy the camera and
// lane tables.  `phase` = parity of the barrier's current phase (0 for the first / only tile of a block).
__device__ __forceinline__ void stage_block(const KParams& P, const CUtensorMap* tmap, const ViewCam* __restrict__ cams,
                                            float* tile, float* sCam, int tile_x0, int tile_y0, unsigned phase = 0u, bool ncc = false,
                                            int extra = 0)
{
    unsigned long long* bar = block_mbar(P, tile, ncc, extra);
    if (threadIdx.x == 0) {
        if (phase == 0u) mbar_init(bar, 1);
        mbar_arrive_expect_tx(bar, (unsigned)(tile_floats(P) * sizeof(float)));
        tma_load_2d(tile, tmap, (tile_x0 + GPM_APRON - P.tile_xo) * (P.color ? 4 : 1), tile_y0 + GPM_APRON, bar);
    }
    const float* c = reinterpret_cast<const float*>(cams);
    for (int e = threadIdx.x; e < P.V * GPM_VIEWCAM_FLOATS; e += blockDim.x) sCam[e] = c[e];
    // lane -> sample table of the sampling rounds (KParams::perm), word by word
    unsigned* sp = reinterpret_cast<unsigned*>(block_perm(P, tile, ncc, extra));
    const unsigned* gp = reinterpret_cast<const unsigned*>(&P.perm[0][0]);
    for (int e = threadIdx.x; e < GPM_MAX_ROUNDS * 8; e += blockDim.x) sp[e] = gp[e];
    __syncthreads();                                // tables visible; mbarrier initialised before anyone waits on it
    mbar_wait(bar, phase & 1u);
}

__device__ __forceinline__ void flush_stats(unsigned long long* stats, const WarpStats& st, unsigned lane)
{
    if (lane == 0 && stats) {
        atomicAdd(stats + ST_HYP, (unsigned long long)st.hyp);
        atomicAdd(stats + ST_SKIP, (unsigned long long)st.skip);
        atomicAdd(stats + ST_PRUNED, (unsigned long long)st.pruned);
        atomicAdd(stats + ST_PAIRS, st.pairs);
        atomicAdd(stats + ST_PAIRS_FULL, st.pairs_full);
    }
}

// shared memory: [tile tile_stride*tile_w][cams V*21][pad to 16 B][nwarps * warp_scratch][4 ints: work counter, unused, mbarrier (8 B)][lane permutation table, GPM_MAX_ROUNDS x 32 bytes]
__host__ __device__ inline size_t block_smem_bytes(const KParams& P, bool ncc = false, int extra = 0)
{
    size_t fl = (size_t)fixed_smem_floats(P) + (size_t)P.nwarps * warp_scratch_floats(P.ns_pad, P.V, P.color, ncc, extra) + 4 + GPM_MAX_ROUNDS * 8;
    return fl * sizeof(float);
}

// ---- joint view selection (ACMH's multi-hypothesis view selection, DESIGN.md §17) ------------------------------------
// What the JVS variants of k_sweep read besides KParams: the per-pixel selected-views masks and the launch's thresholds.
// A kernel parameter of its own, so that KParams and GeoParams keep their layout in every other kernel.
struct JvsParams {
    unsigned long long* mask;   // [H*W] bit j: view j was selected at this pixel by the last JVS launch
    float tau_t;                // good threshold of this launch: tau_init * exp(-t^2 / alpha), computed on the host
    float kb;                   // -log2(e) / (2 beta^2): conf(m) = ex2(m * m * kb)
    float tau_bad, w_keep;
    int n_good, n_bad;
};

// per-warp floats of the JVS variants after the common scratch: 9 rows of V photometric costs (8 candidates, then the
// current plane or the refinement candidate), as many geometric terms with GEO, and the V view weights
__host__ __device__ inline int jvs_floats(int V, bool geo) { return (geo ? 18 : 9) * V + V; }

// ---- sweep modes: which combinations have kernels --------------------------------------------------------------------
// A context's mode: colour images, the fused 20-neighbour sweep (option neighbours = 20), the geometric-consistency term
// (§14), the NCC cost (§15), adaptive checkerboard sampling (§16), joint view selection (§17), the planar prior (§18) and
// the per-pixel mask of the geometric term (§21) and ACMH's refinement (§23).
// Kernels are instantiated (gpm_api.cu, kernel tables) and setters accept a change (gpm_set_*) exactly for the modes
// mode_conflict() passes.
struct Mode {
    bool color, fused, geo, ncc, adaptive, jvs, prior, geomask, refine_acmh;
    __host__ __device__ constexpr int bits() const
    {
        return color | fused << 1 | geo << 2 | ncc << 3 | adaptive << 4 | jvs << 5 | prior << 6 | geomask << 7 | refine_acmh << 8;
    }
    __host__ __device__ static constexpr Mode of(int b)
    {
        return Mode{bool(b & 1), bool(b & 2), bool(b & 4), bool(b & 8), bool(b & 16), bool(b & 32), bool(b & 64), bool(b & 128),
                    bool(b & 256)};
    }
};
constexpr int GPM_MODES = 512;
// k_cost_eval and k_shard_stage never read refine_acmh (the highest bit): their tables cover the other eight bits
constexpr int GPM_EVAL_MODES = 256;

enum class ModeConflict { none, fused, jvs_needs_ncc_grey, ncc_colour, prior, geomask, refine_fused };

// The one rule: the fused sweep has none of the five modes; joint view selection needs the NCC cost (on grey images);
// the NCC cost needs grey images; the planar prior needs grey images and excludes joint view selection; the geometric
// term's mask needs the term and excludes the planar prior; ACMH's refinement excludes the fused sweep.  The first
// conflict found is the reason a refusal gives.
__host__ __device__ constexpr ModeConflict mode_conflict(Mode m)
{
    if (m.fused && (m.geo || m.ncc || m.adaptive || m.jvs || m.prior)) return ModeConflict::fused;
    if (m.jvs && (!m.ncc || m.color)) return ModeConflict::jvs_needs_ncc_grey;
    if (m.ncc && m.color) return ModeConflict::ncc_colour;
    if (m.prior && (m.color || m.jvs)) return ModeConflict::prior;
    if (m.geomask && (!m.geo || m.prior)) return ModeConflict::geomask;
    if (m.refine_acmh && m.fused) return ModeConflict::refine_fused;
    return ModeConflict::none;
}

// The source-view shard (k_shard_stage) exchanges top-n lists of the 8-neighbour sweep's PM costs, step by step of
// Gipuma's refinement: no geometric term, NCC cost, joint view selection, planar prior, fused sweep or ACMH's refinement.
__host__ __device__ constexpr bool shard_supports(Mode m)
{
    return mode_conflict(m) == ModeConflict::none && !m.geo && !m.ncc && !m.jvs && !m.prior && !m.fused && !m.refine_acmh;
}

// ---- ACMH's refinement (Xu & Tao 2019; DESIGN.md §23) --------------------------------------------------------------------
// What the REFINE_ACMH variants of k_sweep read besides KParams: the draws' key and the perturbation.  A kernel parameter of
// its own, the last one, so that every other kernel parameter keeps its place.
struct AcmhRefine {
    unsigned seed;              // (uint32)seed ^ (uint32)(seed >> 32) of gpm_set_rng's 64-bit seed
    unsigned counter;           // r: k_sweep launches with refinement since gpm_init / gpm_init_planes / gpm_set_rng
    float eps;                  // perturbation, in (0, 1)
};

// lowbias32 (C. Wellons, hash-prospector; public domain): a 32-bit integer hash with a strong avalanche
__host__ __device__ constexpr unsigned acmh_mix(unsigned x)
{
    x ^= x >> 16;  x *= 0x7feb352du;  x ^= x >> 15;  x *= 0x846ca68bu;  x ^= x >> 16;
    return x;
}
// key of pixel i in launch r; draw k is acmh_mix(key ^ k), mapped to (0, 1] as xorwow_uniform maps its words
__host__ __device__ constexpr unsigned acmh_key(unsigned seed, unsigned i, unsigned r) { return acmh_mix(acmh_mix(acmh_mix(seed) ^ i) ^ r); }
__device__ __forceinline__ float acmh_draw(unsigned key, unsigned k)
{
    return ffma(__uint2float_rn(acmh_mix(key ^ k)), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
}

// Candidate j (0..4) of the refinement of the plane `n` at pixel (px, py): (d_r, n), (d, n_r), (d_r, n_r), (d, n_t), (d_t, n).
// d is n's depth at p (prior_depth); draws 0 (d_t), 1..3 (n_t), 4 (d_r), 5, 6, ... (n_r, Marsaglia pairs).  Every operation
// is an IEEE float32 one (no approximate reciprocal or square root), so oracle/pyrefine.py restates it bit for bit.
__device__ __forceinline__ float4 acmh_candidate(const KParams& P, const AcmhRefine& F, unsigned key, const float4& n, int j, float fpx,
                                                 float fpy)
{
    const RefCam& c = P.ref;
    const float d = prior_depth(c, n.x, n.y, n.z, n.w, fpx, fpy);
    // the ray through p, view_vector's formula without the normalisation: a normal faces the camera where n . ray <= 0
    const float a = fsub(fpx, c.P34[0]), b = fsub(fpy, c.P34[1]), e = fsub(1.0f, c.P34[2]);
    const float* M = c.M_inv;
    const float vx = fsub(ffma(e, M[2], ffma(a, M[0], fmul(b, M[1]))), c.C[0]);
    const float vy = fsub(ffma(e, M[5], ffma(a, M[3], fmul(b, M[4]))), c.C[1]);
    const float vz = fsub(ffma(e, M[8], ffma(a, M[6], fmul(b, M[7]))), c.C[2]);
    float nx = n.x, ny = n.y, nz = n.z, depth = d;
    if (j == 0 || j == 2) {                         // d_r: uniform in disparity, as k_init_planes draws
        const float disp = ffma(fsub(P.max_disp, P.min_disp), acmh_draw(key, 4u), P.min_disp);
        depth = __fdiv_rn(fmul(c.f_cam, c.baseline), disp);
    } else if (j == 4) {                            // d_t
        const float s = ffma(acmh_draw(key, 0u), 2.0f, -1.0f);
        depth = fmin_(c.depthMax, fmax_(c.depthMin, fmul(d, ffma(F.eps, s, 1.0f))));
    }
    if (j == 1 || j == 2) {                         // n_r: Marsaglia's sphere sampler
        unsigned k = 5u;
        float u, v, sum;
        do {
            u = ffma(acmh_draw(key, k), 2.0f, -1.0f);
            v = ffma(acmh_draw(key, k + 1u), 2.0f, -1.0f);
            k += 2u;
            sum = ffma(u, u, fmul(v, v));
        } while (sum >= 1.0f);
        const float sq = __fsqrt_rn(fsub(1.0f, sum));
        nx = fmul(fadd(u, u), sq);  ny = fmul(fadd(v, v), sq);  nz = fsub(1.0f, fadd(sum, sum));
    } else if (j == 3) {                            // n_t: n + U(-eps pi, eps pi) per component, normalised
        const float dn = fmul(F.eps, 3.14159274f), two = fadd(dn, dn);
        const float tx = fadd(n.x, ffma(acmh_draw(key, 1u), two, -dn));
        const float ty = fadd(n.y, ffma(acmh_draw(key, 2u), two, -dn));
        const float tz = fadd(n.z, ffma(acmh_draw(key, 3u), two, -dn));
        const float rs = __fdiv_rn(1.0f, __fsqrt_rn(ffma(tz, tz, ffma(tx, tx, fmul(ty, ty)))));
        nx = fmul(tx, rs);  ny = fmul(ty, rs);  nz = fmul(tz, rs);
    }
    if ((j == 1 || j == 2 || j == 3) && dot3(nx, ny, nz, vx, vy, vz) > 0.0f) { nx = -nx;  ny = -ny;  nz = -nz; }
    return make_float4(nx, ny, nz, plane_d(c, nx, ny, nz, fpx, fpy, depth));
}

// GEOMASK variants (§21): whether the geometric term is on at the pixel `at` — off where the mask byte is nonzero.  The mask
// travels in PriorParams::geo_mask, which only the prior variants read otherwise: the mask excludes the prior
// (mode_conflict), so every kernel keeps its parameter layout.
template <bool GEOMASK>
__device__ __forceinline__ bool geo_at(const PriorParams& R, size_t at) { return !GEOMASK || R.geo_mask[at] == 0; }

// ---- exact memo of rejected work: plane identities ------------------------------------------------------------
// Every plane carries a 32-bit identity: pid[p] = p + 1 at initialisation, a fresh number (atomic counter) whenever a
// refinement creates a new plane, and COPIED when a plane propagates to a neighbour (gipuma.cu:867-871 copies the plane
// verbatim).  Equal identity therefore implies bit-identical planes, so "this neighbour still holds the plane I was offered
// before" is one 4-byte compare instead of a 16-byte one, the per-pixel memo shrinks from 8 x 16 + 16 to 8 x 4 + 4 bytes,
// and a neighbour whose identity is remembered is skipped without even loading its plane.  (Planes that are equal by value
// but were created independently have different identities: a skip is lost, never a decision.)
struct Memo {
    unsigned* pid;        // [H*W]       identity of the stored plane
    unsigned* seen;       // [H*W*NC]    identity last offered to each pixel from each propagation direction
    unsigned* refseen;    // [H*W]       identity of the plane from which the last all-rejected refinement started
    unsigned* mask;       // [H*W]       validity bits of seen (0..19) and refseen (GPM_MEMO_REFINE)
    unsigned* next_id;    // device counter of fresh identities
};

// ---- random plane initialisation — gipuma_init_cu2, gipuma.cu:996-1036 ----------------------
__global__ void k_fill_ids(unsigned* __restrict__ pid, unsigned n)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pid[i] = i + 1u;
}

__global__ void k_init_planes(const __grid_constant__ KParams P, unsigned long long seed, float4* __restrict__ planes,
                              unsigned* __restrict__ rng_state, unsigned* __restrict__ pid)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= P.W || y >= P.H) return;
    curandState st;
    curand_init(seed, y, x, &st);                                    // :1019 (reference seed: clock64())
    Xorwow r;
    r.v0 = st.v[0];  r.v1 = st.v[1];  r.v2 = st.v[2];  r.v3 = st.v[3];  r.v4 = st.v[4];  r.d = st.d;
    const float px = __int2float_rn(x), py = __int2float_rn(y);
    float vx, vy, vz;
    view_vector(P.ref, px, py, vx, vy, vz);                         // :1025
    // disp_now = curand_between(mind, maxd)                           :1028
    const float disp = ffma(fsub(P.max_disp, P.min_disp), xorwow_uniform(r), P.min_disp);
    // rndUnitVectorSphereMarsaglia_cu, :148-164
    float a, b, sum;
    do {
        a = ffma(xorwow_uniform(r), 2.0f, -1.0f);
        b = ffma(xorwow_uniform(r), 2.0f, -1.0f);
        sum = ffma(a, a, fmul(b, b));
    } while (sum >= 1.0f);
    const float sq = fsqrt_(fsub(1.0f, sum));
    float nx = fmul(fadd(a, a), sq), ny = fmul(fadd(b, b), sq), nz = fsub(1.0f, fadd(sum, sum));
    if (dot3(nx, ny, nz, vx, vy, vz) > 0.0f) { nx = -nx;  ny = -ny;  nz = -nz; }   // vecOnHemisphere_cu :131-137
    // depth = f * baseline / disp (:1031), d = getD_cu (:1034)
    const float depth = fmul(fmul(P.ref.f_cam, P.ref.baseline), frcp(disp));
    const float d = plane_d(P.ref, nx, ny, nz, px, py, depth);
    planes[(size_t)y * P.W + x] = make_float4(nx, ny, nz, d);
    pid[(size_t)y * P.W + x] = (unsigned)(y * P.W + x) + 1u;
    if (rng_state) {
        unsigned* o = rng_state + ((size_t)y * P.W + x) * 6;
        o[0] = r.v0;  o[1] = r.v1;  o[2] = r.v2;  o[3] = r.v3;  o[4] = r.v4;  o[5] = r.d;
    }
}

// ---- planar prior at one pixel (DESIGN.md §18) ------------------------------------------------------------------------
// The pixel's prior plane and its depth (prior_depth), read once per pixel; of() is the term of a hypothesis, 0 where the
// pixel has no prior (the prior plane's depth is not in [depthMin, depthMax]; an all-zero entry never is).
struct PixelPrior {
    float4 pi;
    float pd;
    bool has;
    __device__ __forceinline__ float of(const KParams& P, const PriorParams& R, const float4& h, float fpx, float fpy) const
    {
        return has ? prior_cost(R, pi, pd, h.x, h.y, h.z, prior_depth(P.ref, h.x, h.y, h.z, h.w, fpx, fpy)) : 0.0f;
    }
};
__device__ __forceinline__ PixelPrior pixel_prior(const KParams& P, const PriorParams& R, size_t at, float fpx, float fpy)
{
    PixelPrior q;
    q.pi = R.map[at];
    q.pd = prior_depth(P.ref, q.pi.x, q.pi.y, q.pi.z, q.pi.w, fpx, fpy);
    q.has = q.pd >= P.ref.depthMin && q.pd <= P.ref.depthMax;
    return q;
}

// ---- cost of the stored (or supplied) plane at every pixel — gipuma.cu:1040-1049 and gpm_cost_eval ----
#ifndef GPM_LB_THREADS
#define GPM_LB_THREADS 512       // max threads per block of the warp-per-pixel kernels (16 warps)
#define GPM_LB_BLOCKS 1
#endif
// GEO: the cost with the geometric-consistency term (DESIGN.md §14); NCC: the NCC photometric cost (§15, grey only).
// G is only read in those variants.  PRIOR: with the planar prior's term (§18, grey only); R is only read there.
// GEOMASK (with GEO): the term is off at the pixels R.geo_mask marks (§21).
template <bool COLOR, bool GEO = false, bool NCC = false, bool PRIOR = false, bool GEOMASK = false>
__global__ void __launch_bounds__(GPM_LB_THREADS, GPM_LB_BLOCKS)
k_cost_eval(const __grid_constant__ KParams P, const __grid_constant__ CUtensorMap tmap, const ViewCam* __restrict__ cams,
            cudaTextureObject_t src, const float4* __restrict__ planes, float* __restrict__ cost, unsigned long long* __restrict__ stats,
            const __grid_constant__ GeoParams G, const PriorParams R)
{
    extern __shared__ __align__(128) float smem[];
    float* tile = smem;
    float* sCam = tile + tile_floats(P);
    float* scratch = smem + fixed_smem_floats(P);
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile_x0 = blockIdx.x * GPM_TILE - P.halo, tile_y0 = blockIdx.y * GPM_TILE - P.halo;
    stage_block(P, &tmap, cams, tile, sCam, tile_x0, tile_y0, 0u, NCC);
    const WarpScratch ws = carve(scratch + (size_t)warp * warp_scratch_floats(P.ns_pad, P.V, P.color, NCC), P.ns_pad, P.V, P.color,
                                 block_perm(P, smem, NCC), NCC);
    WarpStats st = {0, 0, 0, 0, 0};
    for (int idx = warp; idx < GPM_TILE * GPM_TILE; idx += P.nwarps) {
        const int px = blockIdx.x * GPM_TILE + (idx & 31), py = blockIdx.y * GPM_TILE + (idx >> 5);
        if (px >= P.W || py >= P.H) continue;
        setup_window<COLOR, NCC>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);
        const float4 n = planes[(size_t)py * P.W + px];
        const float inf = __int_as_float(0x7f800000);
        const GeoParams* g = (GEO || NCC) ? &G : nullptr;
        const float fpx = __int2float_rn(px), fpy = __int2float_rn(py);
        float pr = 0.0f;
        if constexpr (PRIOR) pr = pixel_prior(P, R, (size_t)py * P.W + px, fpx, fpy).of(P, R, n, fpx, fpy);
        const bool gon = geo_at<GEOMASK>(R, (size_t)py * P.W + px);
        float c;
        if constexpr (NCC) c = eval_plane<1, COLOR, GEO, true, false, PRIOR>(P, sCam, ws, src, n.x, n.y, n.z, n.w, inf, lane, st, nullptr, nullptr, 0u, g, fpx, fpy, pr, gon);
        else c = (P.cost_rt & 12) ? eval_plane<2, COLOR, GEO, false, false, PRIOR>(P, sCam, ws, src, n.x, n.y, n.z, n.w, inf, lane, st, nullptr, nullptr, (unsigned)P.cost_rt, g, fpx, fpy, pr, gon)
                 : P.cost_variant ? eval_plane<1, COLOR, GEO, false, false, PRIOR>(P, sCam, ws, src, n.x, n.y, n.z, n.w, inf, lane, st, nullptr, nullptr, 0u, g, fpx, fpy, pr, gon)
                                  : eval_plane<0, COLOR, GEO, false, false, PRIOR>(P, sCam, ws, src, n.x, n.y, n.z, n.w, inf, lane, st, nullptr, nullptr, 0u, g, fpx, fpy, pr, gon);
        if (lane == 0) cost[(size_t)py * P.W + px] = c;
    }
    flush_stats(stats, st, lane);
}

// ---- one checkerboard colour: close + far propagation + refinement, fused --------------------
// gipuma_{black,red}_spatialPropClose_cu / spatialPropFar_cu / planeRefine_cu, gipuma.cu:1353-1823.
// colour 0 = black, 1 = red; phase_mask bit0 close, bit1 far, bit2 refine.
// Candidate table of the fused 20-neighbour kernel gipuma_checkerboard_cu (gipuma.cu:1236-1330): offset of candidate k
// and the reference's own border guards, written as margins  x >= gx0, x <= W-1-gx1, y >= gy0, y <= H-1-gy1
// (they are not the tightest ones: e.g. `left - cols*2` is guarded by p.y > 2, gipuma.cu:1313-1317).
__device__ const signed char kFusedDx[20]  = { 0,  0,  0, 0, 0, 0, -1, -3, -5, 1, 3, 5,  2, 2, -2, -2, -1,  1, -1, 1};
__device__ const signed char kFusedDy[20]  = {-1, -3, -5, 1, 3, 5,  0,  0,  0, 0, 0, 0, -1, 1, -1,  1, -2, -2,  2, 2};
__device__ const signed char kFusedGx0[20] = { 0,  0,  0, 0, 0, 0,  1,  3,  5, 0, 0, 0,  0, 0,  2,  2,  1,  0,  1, 0};
__device__ const signed char kFusedGx1[20] = { 0,  0,  0, 0, 0, 0,  0,  0,  0, 1, 3, 5,  2, 2,  0,  0,  0,  1,  0, 1};
__device__ const signed char kFusedGy0[20] = { 1,  3,  5, 0, 0, 0,  0,  0,  0, 0, 0, 0,  1, 0,  1,  0,  3,  3,  0, 0};
__device__ const signed char kFusedGy1[20] = { 0,  0,  0, 1, 3, 5,  0,  0,  0, 0, 0, 0,  0, 1,  0,  1,  0,  0,  2, 2};

// Pixel of checkerboard colour `colour` at index idx (0..511) of this block's tile — gipuma.cu:1730-1734 / 1786-1790.
__device__ __forceinline__ void colour_pixel(int idx, int colour, int& px, int& py)
{
    const int tx = idx & 31, ty = idx >> 5;
    px = blockIdx.x * GPM_TILE + tx;
    py = blockIdx.y * GPM_TILE + 2 * ty + (((tx & 1) ^ colour) & 1);
}

// Candidate k of the 8-neighbour sweep: 0..3 = up, down, left, right at 1 px (gipuma.cu:1571-1582), 4..7 the same at 5 px
// (:1450-1462).  (qx, qy) is the neighbour; the result is the reference's border guard (false: the candidate is not offered).
// px and py are taken by reference only so that k_sweep compiles to the same instructions as with the guard written inline:
// by value, the compiler canonicalises `py < H - dist` to `H - dist > py` before inlining.
__device__ __forceinline__ bool close_far_neighbour(int k, const int& px, const int& py, int W, int H, int& qx, int& qy)
{
    const int dist = k < 4 ? 1 : 5, dir = k & 3;
    qx = px;  qy = py;
    bool ok;
    if (dir == 0)      { ok = py > dist - 1;  qy = py - dist; }
    else if (dir == 1) { ok = py < H - dist;  qy = py + dist; }
    else if (dir == 2) { ok = px > dist - 1;  qx = px - dist; }
    else               { ok = px < W - dist;  qx = px + dist; }
    return ok;
}

// Candidate k of the adaptive checkerboard sampling (ACMH, Xu & Tao 2019; DESIGN.md §16): the pixel with the lowest stored
// cost of region k, NaN counting as +inf and a tie going to the earliest offset of the region's scan order.  Regions 0..3
// (near up, down, left, right) are V shapes of 7 offsets: the 1 px neighbour, then (a, ±(a - 1)) for a = 2, 3, 4 along the
// direction; regions 4..7 (far) are the 11 axial offsets 3, 5, ..., 23 px.  Every offset has odd |dy| + |dx|, so region
// pixels are of the other checkerboard colour, whose planes and costs a launch never writes.  false: no offset lies in the
// image (the candidate is not offered); (qx, qy) is then (px, py).
__device__ __forceinline__ bool acs_neighbour(int k, int px, int py, int W, int H, const float* cost, int& qx, int& qy)
{
    const int dir = k & 3, n = k < 4 ? 7 : 11, sgn = (dir == 0 || dir == 2) ? -1 : 1;
    qx = px;  qy = py;
    float best = 0.0f;
    bool found = false;
    for (int j = 0; j < n; j++) {
        const int i = (j + 1) >> 1;
        const int a = k < 4 ? 1 + i : 3 + 2 * j;                   // distance along the direction
        const int b = k < 4 ? ((j & 1) ? -i : i) : 0;              // offset across it
        const int x = px + (dir < 2 ? b : sgn * a), y = py + (dir < 2 ? sgn * a : b);
        if (x < 0 || x >= W || y < 0 || y >= H) continue;
        float c = cost[(size_t)y * W + x];
        if (c != c) c = __int_as_float(0x7f800000);
        if (!found || c < best) { best = c;  qx = x;  qy = y;  found = true; }
    }
    return found;
}

// The sweep's and the shard's neighbour choice: the fixed neighbour of direction k (with the reference's border guard) or,
// ADAPTIVE, the cheapest pixel of region k by the costs the launch started from.
template <bool ADAPTIVE>
__device__ __forceinline__ bool sweep_neighbour(int k, const int& px, const int& py, int W, int H, const float* cost, int& qx, int& qy)
{
    if constexpr (ADAPTIVE) return acs_neighbour(k, px, py, W, H, cost, qx, qy);
    else return close_far_neighbour(k, px, py, W, H, qx, qy);
}

// ---- shared propagation samples (DESIGN.md §4) ------------------------------------------------------------------------
// In the sweep mode with none of the options of Mode — grey images, PM cost, the fixed 8-neighbour sweep — k_sweep costs the
// propagated candidates plane-major before its per-pixel loop.  A launch of colour c never writes a plane of colour 1 - c, and
// each such plane q is offered to q +- (0, 1), q +- (0, 5) (its column group) and q +- (1, 0), q +- (5, 0) (its row group).
// The four windows of a group lie on one stride-2 lattice, and a sample's dissimilarity against view v is a function of the
// plane, the view and the sample's absolute texel alone (the propagation sites all use rounding variant 1), so one warp
// fetches each lattice texel of a group once and runs every target pixel's own chain over it.  The pass serves either
// refinement (§23): it only changes how the propagation pass gets its costs, and the refinement follows it unchanged.
__host__ __device__ constexpr bool shares_samples(Mode m) { return (m.bits() & (GPM_EVAL_MODES - 1)) == 0; }

// Per-warp layout of the plane-major pass, in floats from the warp's scratch (which it overlays: the pass ends before the
// per-pixel loop starts).  L texels of the union lattice (nside x (nside + 5)); A/left/pos: per fetched texel in fetch order,
// its (x, y, gx1, gy1), its reference value and its place in D; lines: the lattice lines the needed windows cover; w: the
// support weights of up to four targets; cv: their per-view costs; D: the dissimilarities of C views (views in chunks, so
// that D does not grow with V).
struct ShareLayout { int L, LS, WS, C, A, H, left, pos, lines, w, cv, D, total; };
__host__ __device__ inline ShareLayout share_layout(const KParams& P)
{
    ShareLayout s;
    s.L = P.nside * (P.nside + 5);
    s.LS = s.L | 1;
    s.WS = P.ns | 1;
    const int chunks = (P.V + 7) / 8;
    s.C = (P.V + chunks - 1) / chunks;
    s.A = 0;
    s.H = 4 * s.L;
    s.left = s.H + 12 * P.V;
    s.pos = s.left + s.L;
    s.lines = s.pos + s.L;
    s.w = s.lines + 20;
    s.cv = s.w + 4 * s.WS;
    s.D = s.cv + 4 * P.V;
    s.total = s.D + s.C * s.LS;
    return s;
}
// floats per warp the pass needs beyond the common warp scratch (block_smem_bytes' `extra`)
__host__ __device__ inline int share_extra_floats(const KParams& P)
{
    const int d = share_layout(P).total - warp_scratch_floats(P.ns_pad, P.V, 0);
    return d > 0 ? d : 0;
}
// after the block's usual shared memory: the costs cand_cost[pixel][k] of the tile's 512 pixels of the launch's colour,
// then each pixel's need mask (bit k: candidate k is evaluated)
#define GPM_SHARE_TABLE_BYTES (GPM_TILE * GPM_TILE / 2 * (8 * 4 + 1))

__device__ __forceinline__ int nth_set_bit(unsigned m, int i)
{
    for (; i > 0; i--) m &= m - 1u;
    return __ffs(m) - 1;
}

// Need masks of the slice's pixels, from the state at launch start only: candidate k of pixel p is evaluated unless it is
// not offered (border guard, phase mask), one of p's 8 remembered identities (memo), its depth at p is out of range, it is
// p's own plane with p's cost of the same rounding variant (dedupe_self), or an earlier candidate of p has its identity
// (dedupe_cand).  Each skip is exact: cost(p, plane) is a pure function and p's cost only decreases, so a skipped candidate
// could not be accepted at any point of p's candidate scan.  Lanes 8m..8m+7 hold the 8 candidates of pixel m of 4.
__device__ __forceinline__ void share_need_masks(const KParams& P, const float4* __restrict__ planes, const unsigned char* __restrict__ prov,
                                                 const Memo& M, int colour, int phase_mask, int idx_begin, int idx_end,
                                                 unsigned char* need, unsigned lane, unsigned warp)
{
    const int j = (int)(lane & 7);
    // two groups of 4 pixels per step, every load of a step issued before any is used (the pass is latency bound)
    for (int base = idx_begin + 8 * (int)warp; base < idx_end; base += 8 * P.nwarps) {
        int idx[2], px[2], py[2];
        bool valid[2], offered[2];
        unsigned id[2], old_id[2], own[2], mmask[2];
        unsigned char pv[2];
        float4 n[2];
#pragma unroll
        for (int u = 0; u < 2; u++) {
            idx[u] = base + 4 * u + (int)(lane >> 3);
            colour_pixel(idx[u], colour, px[u], py[u]);
            valid[u] = idx[u] < idx_end && px[u] < P.W && py[u] < P.H;
            const size_t center = valid[u] ? (size_t)py[u] * P.W + px[u] : 0;
            int qx = px[u], qy = py[u];
            offered[u] = valid[u] && ((phase_mask >> (j >> 2)) & 1) && close_far_neighbour(j, px[u], py[u], P.W, P.H, qx, qy);
            const size_t at = (size_t)qy * P.W + qx;
            id[u] = offered[u] ? M.pid[at] : 0u;
            n[u] = offered[u] ? planes[at] : make_float4(0.f, 0.f, 0.f, 0.f);
            mmask[u] = P.memo && valid[u] ? M.mask[center] : 0u;
            old_id[u] = P.memo && valid[u] ? M.seen[center * 8 + j] : 0u;
            own[u] = valid[u] ? M.pid[center] : 0u;
            pv[u] = valid[u] ? prov[center] : (unsigned char)0;
        }
#pragma unroll
        for (int u = 0; u < 2; u++) {
            const bool old_ok = (mmask[u] >> j) & 1u;
            bool known = false, dup = false;
            for (int i = 0; i < 8; i++) {
                const bool oi = __shfl_sync(GPM_FULL, old_ok, i, 8);
                const unsigned idi = __shfl_sync(GPM_FULL, old_id[u], i, 8);
                const bool ci = __shfl_sync(GPM_FULL, offered[u], i, 8);
                const unsigned cid = __shfl_sync(GPM_FULL, id[u], i, 8);
                known |= oi && idi == id[u];
                dup |= i < j && ci && cid == id[u];
            }
            const float d = plane_depth(P.ref, n[u].x, n[u].y, n[u].z, n[u].w, __int2float_rn(px[u]), __int2float_rn(py[u]));   // gipuma.cu:829-830
            const bool ok = offered[u] && !known && !(P.dedupe_cand && dup) && !(P.dedupe_self && pv[u] == 1 && id[u] == own[u]) &&
                            d >= P.ref.depthMin && d <= P.ref.depthMax;
            const unsigned b = __ballot_sync(GPM_FULL, ok);
            if (j == 0 && idx[u] < idx_end) need[idx[u]] = (unsigned char)(b >> (lane & 24));
        }
    }
}

// The plane-major pass: every needed (pixel, candidate) of the slice gets its exact cost in table[idx * 8 + k].  Work items
// are (plane q, group) over the other colour's pixels of the slice's rows plus the 5-pixel halo, taken dynamically by the
// warps (counter).  `tile` is the staged reference window (already offset by tile_xo).
__device__ __forceinline__ void share_costs(const KParams& P, const float* __restrict__ sCam, const float* __restrict__ tile,
                                            float* wbase, cudaTextureObject_t src, const float4* __restrict__ planes, int colour,
                                            int idx_begin, int idx_end, int tile_x0, int tile_y0, const unsigned char* need,
                                            float* table, int* counter, unsigned long long* stats, unsigned lane, WarpStats& st)
{
    const ShareLayout S = share_layout(P);
    float4* Ae = reinterpret_cast<float4*>(wbase + S.A);
    float* Hs = wbase + S.H;
    float* le = wbase + S.left;
    int* pe = reinterpret_cast<int*>(wbase + S.pos);
    int* lines = reinterpret_cast<int*>(wbase + S.lines);
    float* wt = wbase + S.w;
    float* cv = wbase + S.cv;
    float* Dc = wbase + S.D;
    const int nside = P.nside, rad = P.rad, tw = P.tile_stride, V = P.V;
    const int bx0 = blockIdx.x * GPM_TILE, by0 = blockIdx.y * GPM_TILE;
    // tile rows of the slice, and the items: column groups of its rows +- 5, then row groups of its rows (the row groups'
    // columns run one lattice step past the halo on each side so that every row has 22 planes of the other colour)
    const int ylo = by0 + 2 * (idx_begin >> 5), yhi = by0 + 2 * ((idx_end - 1) >> 5) + 1;
    const int ncol = (yhi - ylo + 11) * 16, nitems = ncol + (yhi - ylo + 1) * 22;
    const float nrg = -frcp(P.gamma);
    const float one_minus_alpha = fsub(1.0f, P.alpha);
    auto texel = [&](int x, int y) { return tile + (y - tile_y0) * tw + (x - tile_x0); };
    auto plane_of = [&](int it, bool& col, int& qx, int& qy) {
        col = it < ncol;
        const int r = col ? it >> 4 : (it - ncol) / 22;
        const int jq = col ? it & 15 : it - ncol - r * 22;
        qy = col ? ylo - 5 + r : ylo + r;
        qx = (col ? bx0 : bx0 - 6) + 2 * jq + ((1 + colour + qy) & 1);
    };
    // the warps take 8 items at a time; lane 4i + m tests target m of item i: q + off along the group's axis, of which q is
    // candidate kk
    int base = 8 * (int)(threadIdx.x >> 5);
    while (base < nitems) {
        const int m = (int)(lane & 3);
        const int off = m == 0 ? -5 : m == 1 ? -1 : m == 2 ? 1 : 5;
        int idx = 0, kk = 0;
        bool mine = false;
        if (base + (int)(lane >> 2) < nitems) {
            bool col;
            int qx, qy;
            plane_of(base + (int)(lane >> 2), col, qx, qy);
            kk = col ? (m == 0 ? 5 : m == 1 ? 1 : m == 2 ? 0 : 4) : (m == 0 ? 7 : m == 1 ? 3 : m == 2 ? 2 : 6);
            const int tx = (col ? qx : qx + off) - bx0, ty = (col ? qy + off : qy) - by0;
            idx = (ty >> 1) * GPM_TILE + tx;
            mine = tx >= 0 && tx < GPM_TILE && ty >= 0 && ty < GPM_TILE && idx >= idx_begin && idx < idx_end && ((need[idx] >> kk) & 1);
        }
        for (unsigned bm = __ballot_sync(GPM_FULL, mine); bm; ) {
            const int it = (__ffs(bm) - 1) >> 2;
            const unsigned nm = (bm >> (4 * it)) & 15u;
            bm &= ~(15u << (4 * it));
            bool col;
            int qx, qy;
            plane_of(base + it, col, qx, qy);
            const int nneed = __popc(nm);
            const float4 pl = planes[(size_t)qy * P.W + qx];
            homographies(P, sCam, Hs, pl.x, pl.y, pl.z, pl.w, lane);
            unsigned lm = 0u;                                    // lattice lines covered by the needed windows
            for (int i = 0; i < 4; i++)
                if ((nm >> i) & 1u) lm |= ((1u << nside) - 1u) << (i == 0 ? 0 : i == 1 ? 2 : i == 2 ? 3 : 5);
            const int nl = __popc(lm), NY = col ? nside + 5 : nside;
            if ((int)lane < nside + 5 && ((lm >> lane) & 1u)) lines[__popc(lm & ((1u << lane) - 1u))] = (int)lane;
            const int x0 = col ? qx - rad : qx - 5 - rad, y0 = col ? qy - 5 - rad : qy - rad;
            __syncwarp();
            // the fetch order: pairs of covered lines, 2 x 2 lattice blocks per hardware quad
            const int n = nl * nside;
            for (int e = (int)lane; e < n; e += 32) {
                const int p2 = e / (2 * nside), rem = e - p2 * 2 * nside;
                const bool pair = 2 * p2 + 1 < nl;
                const int line = lines[pair ? 2 * p2 + (rem & 1) : 2 * p2], b = pair ? rem >> 1 : rem;
                const int lx = col ? b : line, ly = col ? line : b;
                const int x = x0 + 2 * lx, y = y0 + 2 * ly;
                const float* t = texel(x, y);
                Ae[e] = make_float4(__int2float_rn(x), __int2float_rn(y), fsub(t[1], t[-1]), fsub(t[tw], t[-tw]));   // as setup_window
                le[e] = t[0];
                pe[e] = lx * NY + ly;
            }
            for (int f = (int)lane; f < nneed * P.ns; f += 32) {  // support weights of the needed targets, as setup_window
                const int i = f / P.ns, s = f - i * P.ns;
                const int mi = nth_set_bit(nm, i);
                const int o = mi == 0 ? -5 : mi == 1 ? -1 : mi == 2 ? 1 : 5;
                const int cx = col ? qx : qx + o, cy = col ? qy + o : qy;
                const int ii = s / nside, jj = s - ii * nside;
                const float center = *texel(cx, cy), left = *texel(cx - rad + 2 * ii, cy - rad + 2 * jj);
                wt[i * S.WS + s] = fex2(fmul(fmul(fabsf(fsub(left, center)), nrg), 1.4426950216293334961f));
            }
            __syncwarp();
            const unsigned Mg = (1u << 20) / (unsigned)n + 1u;
            for (int v0 = 0; v0 < V; v0 += S.C) {
                const int Cc = min(S.C, V - v0), npairs = Cc * n;
                // lane handles pair (view v0 + vi, texel e); N steps in flight before any result is consumed (as eval_plane)
                auto fetch = [&](auto nconst, int q0) {
                    constexpr int N = decltype(nconst)::value;
                    float gx2[N], gy2[N], tc[N];
                    float4 a[N];
                    int dst[N], ei[N];
#pragma unroll
                    for (int u = 0; u < N; u++) {
                        const int q = q0 + u * 32 + (int)lane;
                        const int qc = min(q, npairs - 1);
                        const int vi = (int)(((unsigned)qc * Mg) >> 20);           // qc / n
                        const int e = qc - vi * n;
                        const float4* H4 = reinterpret_cast<const float4*>(Hs + (v0 + vi) * 12);
                        a[u] = Ae[e];
                        ei[u] = e;
                        dst[u] = q < npairs ? vi * S.LS + pe[e] : -1;
                        fetch_sample_grey(src, H4[0], H4[1], H4[2], a[u].x, a[u].y, v0 + vi, true, true, true, gx2[u], gy2[u], tc[u]);
                    }
#pragma unroll
                    for (int u = 0; u < N; u++) {
                        const float dis = dissim_grey(P, one_minus_alpha, a[u].z, a[u].w, le[ei[u]], gx2[u], gy2[u], tc[u]);
                        if (dst[u] >= 0) Dc[dst[u]] = dis;
                    }
                };
                int q0 = 0;
                for (; q0 + 32 < npairs; q0 += 64) fetch(std::integral_constant<int, 2>(), q0);
                if (q0 < npairs) fetch(std::integral_constant<int, 1>(), q0);
                __syncwarp();
                // lane = (needed target i, view vi): the target's chain  c = c + w_s * D_s  in its own sample order
                if ((int)lane < nneed * Cc) {
                    const int i = (int)lane / Cc, vi = (int)lane - i * Cc;
                    const int mi = nth_set_bit(nm, i);
                    const int o = mi == 0 ? 0 : mi == 1 ? 2 : mi == 2 ? 3 : 5;
                    const float* w = wt + i * S.WS;
                    const float* D = Dc + vi * S.LS + (col ? o : o * nside);
                    float c = 0.0f;
                    for (int ii = 0; ii < nside; ii++)
                        for (int jj = 0; jj < nside; jj++) c = ffma(w[ii * nside + jj], D[ii * NY + jj], c);
                    cv[i * V + v0 + vi] = c;
                }
                __syncwarp();
            }
            for (int i = 0; i < nneed; i++) {
                const float c0 = (int)lane < V ? cv[i * V + lane] : 0.0f;
                const float c1 = (int)lane + 32 < V ? cv[i * V + lane + 32] : 0.0f;
                const float c = combine_views(P, c0, c1, lane);
                const int mi = nth_set_bit(nm, i);
                const int ti = __shfl_sync(GPM_FULL, idx, 4 * it + mi), tk = __shfl_sync(GPM_FULL, kk, 4 * it + mi);
                if (lane == 0) table[ti * 8 + tk] = c;
            }
            st.hyp += nneed;
            st.pairs_full += (unsigned long long)nneed * V * P.ns;
#ifndef GPM_SHARE_COUNT_FETCHES
            st.pairs += (unsigned long long)nneed * V * P.ns;
#else
            // counting build of tools/share_bench.py: `pairs` counts the (view, texel) pairs really fetched, and slot 7 (no
            // counter) the pass's pairs as `pairs` counts them otherwise
            st.pairs += (unsigned long long)n * V;
            if (lane == 0 && stats) atomicAdd(stats + 7, (unsigned long long)nneed * V * P.ns);
#endif
            __syncwarp();
        }
        if (lane == 0) base = atomicAdd(counter, 8);
        base = __shfl_sync(GPM_FULL, base, 0);
    }
}

// One pixel of a joint-view-selection launch (ACMH, Xu & Tao 2019; DESIGN.md §17): NCC cost, grey images, 8-neighbour
// sweep.  The steps as §17 numbers them: (1) the per-view cost rows of the current plane and of every offered candidate
// whose depth is in range (E), a candidate whose identity equals the current plane's or an earlier candidate's reusing
// that row; (2, 3) lane j reduces view j's column over E into good_j, bad_j and s_j and forms the weight w_j; (4) every
// hypothesis is scored sum_j w_j c_j / sum_j w_j, both sums sequential from +0 (lane 0), or by combine_views where
// sum_j w_j = 0; (5) the fold starts at the current plane's re-scored cost.  Weighted costs are not a pure function of the
// plane, so neither memo nor the duplicate-of-current skip is used, and the stored cost is tagged GPM_PROV_JVS.  The
// refinement restates k_sweep's loop body line for line (see shard_refine_candidate).
// REFINE_ACMH: ACMH's five candidates (§23) instead of Gipuma's steps, scored with the same weights.
template <bool GEO, bool ADAPTIVE, bool REFINE_ACMH = false>
__device__ __forceinline__ void jvs_pixel(const KParams& P, const JvsParams& J, const GeoParams* g, const float* __restrict__ sCam,
                                          const float* __restrict__ tile, const WarpScratch& ws, float* __restrict__ jv,
                                          cudaTextureObject_t src, float4* __restrict__ planes, float* __restrict__ cost,
                                          unsigned* __restrict__ rng_state, unsigned char* __restrict__ prov, const Memo& M,
                                          int px, int py, int tile_x0, int tile_y0, int phase_mask, unsigned lane, WarpStats& st,
                                          bool geo_on, const AcmhRefine F)
{
    const RefCam& cam = P.ref;
    const bool with_geo = GEO && geo_on;            // false at a pixel the geometric term's mask marks (§21)
    const int W = P.W, H = P.H, V = P.V;
    const size_t center = (size_t)py * W + px;
    const float fpx = __int2float_rn(px), fpy = __int2float_rn(py);
    const float inf = __int_as_float(0x7f800000);
    float* Mr = jv;                                  // [9][V] photometric costs: rows 0..7 candidates, 8 current / refinement
    float* Gr = jv + 9 * V;                          // GEO: [9][V] geometric terms
    float* wv = jv + (GEO ? 18 : 9) * V;             // [V] view weights
    float4 norm_now = planes[center];
    unsigned own_id = M.pid[center];
    const unsigned long long remembered = J.mask[center];

    // candidate k in lane k, its depth at p and the range test (gipuma.cu:829-830)
    float4 mine = make_float4(0.f, 0.f, 0.f, 0.f);
    bool mine_ok = false, in_range = false;
    float mine_disp = 0.0f;
    size_t mine_at = center;
    if (lane < 8) {
        const bool phase_on = (phase_mask >> (lane >> 2)) & 1;
        int qx, qy;
        const bool ok = sweep_neighbour<ADAPTIVE>((int)lane, px, py, W, H, cost, qx, qy);
        mine_ok = ok && phase_on;
        mine_at = (size_t)qy * W + qx;
    }
    const unsigned mine_id = mine_ok ? M.pid[mine_at] : 0u;
    if (mine_ok) {
        mine = planes[mine_at];
        mine_disp = plane_depth(cam, mine.x, mine.y, mine.z, mine.w, fpx, fpy);
        in_range = mine_disp >= cam.depthMin && mine_disp <= cam.depthMax;
    }
    const unsigned offered = __ballot_sync(GPM_FULL, mine_ok), E = __ballot_sync(GPM_FULL, in_range);
    st.skip += __popc(offered & ~E);

    setup_window<false, true>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);
    auto eval_row = [&](float nx, float ny, float nz, float nd, int r) {
        eval_plane<1, false, GEO, true, true>(P, sCam, ws, src, nx, ny, nz, nd, inf, lane, st, Mr + r * V, Gr + r * V, 0u, g, fpx, fpy, 0.0f, geo_on);
    };
    // (1) rows: 4 bits per candidate k name the row that holds its costs
    eval_row(norm_now.x, norm_now.y, norm_now.z, norm_now.w, 8);
    unsigned rows = 0u;
    for (int k = 0; k < 8; k++) {
        if (!((E >> k) & 1)) continue;
        const unsigned cand_id = __shfl_sync(GPM_FULL, mine_id, k);
        const unsigned earlier = __ballot_sync(GPM_FULL, (int)lane < k && in_range && mine_id == cand_id);
        int r = k;
        if (P.dedupe_self && cand_id == own_id) r = 8;
        else if (P.dedupe_cand && earlier) r = (int)((rows >> (4 * (__ffs(earlier) - 1))) & 15u);
        const float nx = __shfl_sync(GPM_FULL, mine.x, k), ny = __shfl_sync(GPM_FULL, mine.y, k);
        const float nz = __shfl_sync(GPM_FULL, mine.z, k), nd = __shfl_sync(GPM_FULL, mine.w, k);
        if (r == k) eval_row(nx, ny, nz, nd, k);
        else st.skip++;
        rows |= (unsigned)r << (4 * k);
    }
    __syncwarp();
    // (2, 3) view statistics over E and the weights; the new selected-views mask is {j : w_j > 0}
    auto weight = [&](int j) {
        int good = 0, bad = 0;
        float s = 0.0f;
        for (int k = 0; k < 8; k++) {
            if (!((E >> k) & 1)) continue;
            const float m = Mr[(int)((rows >> (4 * k)) & 15u) * V + j];
            if (m < J.tau_t) { good++;  s = fadd(s, fex2(fmul(fmul(m, m), J.kb))); }
            if (m > J.tau_bad) bad++;
        }
        if (good >= J.n_good && bad < J.n_bad) return fdiv(s, __int2float_rn(good));
        if (((remembered >> j) & 1ull) && bad < J.n_bad) return J.w_keep;
        return 0.0f;
    };
    float w0 = 0.0f, w1 = 0.0f;
    if ((int)lane < V) { w0 = weight((int)lane);  wv[lane] = w0; }
    if ((int)lane + 32 < V) { w1 = weight((int)lane + 32);  wv[lane + 32] = w1; }
    const unsigned long long selected = (unsigned long long)__ballot_sync(GPM_FULL, w0 > 0.0f) |
                                        ((unsigned long long)__ballot_sync(GPM_FULL, w1 > 0.0f) << 32);
    __syncwarp();
    float wsum = 0.0f;
    if (lane == 0) for (int j = 0; j < V; j++) wsum = fadd(wsum, wv[j]);
    wsum = __shfl_sync(GPM_FULL, wsum, 0);
    // (4) the cost of the hypothesis in row r
    auto score = [&](int r) {
        const float* m = Mr + r * V;
        const float* gr = Gr + r * V;
        if (wsum == 0.0f) {                          // no reliable view: today's NCC cost
            float c0 = 0.0f, c1 = 0.0f;
            if ((int)lane < V) c0 = with_geo ? fadd(m[lane], gr[lane]) : m[lane];
            if ((int)lane + 32 < V) c1 = with_geo ? fadd(m[lane + 32], gr[lane + 32]) : m[lane + 32];
            return combine_views(P, c0, c1, lane);
        }
        float num = 0.0f;
        if (lane == 0) for (int j = 0; j < V; j++) num = fadd(num, fmul(wv[j], with_geo ? fadd(m[j], gr[j]) : m[j]));
        return __shfl_sync(GPM_FULL, fdiv(num, wsum), 0);
    };
    // (5) the fold: strict <, candidates in k order (gipuma.cu:867-871)
    float cost_now = score(8);
    float disp_now = plane_depth(cam, norm_now.x, norm_now.y, norm_now.z, norm_now.w, fpx, fpy);
    for (int k = 0; k < 8; k++) {
        if (!((E >> k) & 1)) continue;
        const float c = score((int)((rows >> (4 * k)) & 15u));
        float4 nb;
        nb.x = __shfl_sync(GPM_FULL, mine.x, k);  nb.y = __shfl_sync(GPM_FULL, mine.y, k);
        nb.z = __shfl_sync(GPM_FULL, mine.z, k);  nb.w = __shfl_sync(GPM_FULL, mine.w, k);
        const float d = __shfl_sync(GPM_FULL, mine_disp, k);
        const unsigned id = __shfl_sync(GPM_FULL, mine_id, k);
        if (c < cost_now) { norm_now = nb;  cost_now = c;  disp_now = d;  own_id = id; }      // a copy keeps its identity
    }
    if constexpr (REFINE_ACMH) {
        if (phase_mask & 4) {
            bool any_accept = false;
            const float4 start = norm_now;
            const unsigned key = acmh_key(F.seed, (unsigned)center, F.counter);
            for (int j = 0; j < 5; j++) {
                const float4 cand = acmh_candidate(P, F, key, start, j, fpx, fpy);
                eval_row(cand.x, cand.y, cand.z, cand.w, 8);
                __syncwarp();
                const float c = score(8);
                if (c < cost_now) { any_accept = true;  cost_now = c;  norm_now = cand; }
            }
            if (any_accept) {                                 // a new plane: one fresh identity
                unsigned fresh = 0u;
                if (lane == 0) fresh = atomicAdd(M.next_id, 1u);
                own_id = __shfl_sync(GPM_FULL, fresh, 0);
            }
        }
    } else if (phase_mask & 4) {                     // planeRefinement_cu, gipuma.cu:928-994, scored with the same weights
        bool any_accept = false;
        Xorwow r = {0u, 0u, 0u, 0u, 0u, 0u};
        if (P.rng_mode == 1) {
            const unsigned* in = rng_state + center * 6;
            r.v0 = in[0];  r.v1 = in[1];  r.v2 = in[2];  r.v3 = in[3];  r.v4 = in[4];  r.d = in[5];
        }
        float vx, vy, vz;
        view_vector(cam, fpx, fpy, vx, vy, vz);
        const float fb = fmul(cam.baseline, cam.f);
        float deltaN = 1.0f;
        for (float deltaZ = fmul(P.max_disp, 0.5f); deltaZ >= 0.01f; deltaZ = fmul(deltaZ, 0.1f)) {
            const float rdisp = frcp(disp_now);
            const float hi = fmin_(ffma(rdisp, -fb, P.max_disp), deltaZ);
            const float lo = fmin_(ffma(rdisp, fb, P.min_disp), deltaZ);
            const float dz = ffma(xorwow_uniform(r), fadd(lo, hi), -lo);
            float dnew = ffma(rdisp, fb, dz);
            dnew = fmin_(P.max_disp, fmax_(P.min_disp, dnew));
            const float depth_new = fmul(frcp(dnew), fb);
            const float twoN = fadd(deltaN, deltaN);
            const float ax = fadd(norm_now.x, ffma(xorwow_uniform(r), twoN, -deltaN));
            const float ay = fadd(norm_now.y, ffma(twoN, xorwow_uniform(r), -deltaN));
            const float az = fadd(norm_now.z, ffma(twoN, xorwow_uniform(r), -deltaN));
            const float rs = frsq(ffma(az, az, ffma(ax, ax, fmul(ay, ay))));
            float4 cand;
            cand.x = fmul(ax, rs);  cand.y = fmul(ay, rs);  cand.z = fmul(az, rs);
            if (dot3(cand.x, cand.y, cand.z, vx, vy, vz) > 0.0f) { cand.x = -cand.x;  cand.y = -cand.y;  cand.z = -cand.z; }
            cand.w = plane_d(cam, cand.x, cand.y, cand.z, fpx, fpy, depth_new);
            eval_row(cand.x, cand.y, cand.z, cand.w, 8);
            __syncwarp();
            const float c = score(8);
            if (c < cost_now) {                                                          // no depth-range test (:986-990)
                any_accept = true;
                cost_now = c;
                disp_now = depth_new;
                norm_now = cand;
            }
            deltaN = fmul(deltaN, 0.25f);
        }
        if (P.rng_mode == 1 && lane == 0) {
            unsigned* o = rng_state + center * 6;
            o[0] = r.v0;  o[1] = r.v1;  o[2] = r.v2;  o[3] = r.v3;  o[4] = r.v4;  o[5] = r.d;
        }
        if (any_accept) {                                 // a new plane: one fresh identity
            unsigned fresh = 0u;
            if (lane == 0) fresh = atomicAdd(M.next_id, 1u);
            own_id = __shfl_sync(GPM_FULL, fresh, 0);
        }
    }
    if (lane == 0) {
        cost[center] = cost_now;
        planes[center] = norm_now;
        prov[center] = (unsigned char)GPM_PROV_JVS;
        M.pid[center] = own_id;
        J.mask[center] = selected;
    }
}

// GEO: the cost with the geometric-consistency term (DESIGN.md §14; 8-neighbour sweep only); NCC: the NCC photometric cost
// (§15; 8-neighbour sweep, grey images only).  G is only read in those variants.  ADAPTIVE: adaptive checkerboard sampling
// (§16; 8-neighbour sweep), candidate k is acs_neighbour's choice instead of the fixed neighbour.  JVS: joint view
// selection (§17; NCC only), every pixel goes through jvs_pixel; J is only read in those variants.  PRIOR: every
// hypothesis' cost carries the planar prior's term (§18; grey, no joint view selection); R is only read there.  GEOMASK
// (with GEO, without PRIOR): every hypothesis of a pixel R.geo_mask marks costs what it costs without the term (§21).
// REFINE_ACMH (not FUSED): the refinement tries ACMH's five candidates (§23) instead of Gipuma's steps; F is only read there.
template <bool COLOR, bool FUSED, bool GEO = false, bool NCC = false, bool ADAPTIVE = false, bool JVS = false, bool PRIOR = false,
          bool GEOMASK = false, bool REFINE_ACMH = false>
__global__ void __launch_bounds__(GPM_LB_THREADS, GPM_LB_BLOCKS)
k_sweep(const __grid_constant__ KParams P, const __grid_constant__ CUtensorMap tmap, const ViewCam* __restrict__ cams,
        cudaTextureObject_t src, float4* __restrict__ planes, float* __restrict__ cost,
        unsigned* __restrict__ rng_state, unsigned char* __restrict__ prov, Memo M, int colour, int phase_mask,
        unsigned long long* __restrict__ stats, const __grid_constant__ GeoParams G, const JvsParams J, const PriorParams R,
        const AcmhRefine F)
{
    static_assert(mode_conflict(Mode{COLOR, FUSED, GEO, NCC, ADAPTIVE, JVS, PRIOR, GEOMASK, REFINE_ACMH}) == ModeConflict::none, "no such sweep mode (mode_conflict)");
    constexpr bool SHARE = shares_samples(Mode{COLOR, FUSED, GEO, NCC, ADAPTIVE, JVS, PRIOR, GEOMASK, REFINE_ACMH});
    const GeoParams* g = (GEO || NCC) ? &G : nullptr;
    extern __shared__ __align__(128) float smem[];
    float* tile = smem;
    float* sCam = tile + tile_floats(P);
    float* scratch = smem + fixed_smem_floats(P);
    const int extra = JVS ? jvs_floats(P.V, GEO) : SHARE ? share_extra_floats(P) : 0;
    int* counter = reinterpret_cast<int*>(scratch + (size_t)P.nwarps * warp_scratch_floats(P.ns_pad, P.V, P.color, NCC, extra));
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile_x0 = blockIdx.x * GPM_TILE - P.halo, tile_y0 = blockIdx.y * GPM_TILE - P.halo;
    if (threadIdx.x == 0) counter[0] = P.nwarps;
    if constexpr (SHARE) if (threadIdx.x == 0) counter[1] = 8 * P.nwarps;
    stage_block(P, &tmap, cams, tile, sCam, tile_x0, tile_y0, 0u, NCC, extra);
    float* warp_base = scratch + (size_t)warp * warp_scratch_floats(P.ns_pad, P.V, P.color, NCC, extra);
    const WarpScratch ws = carve(warp_base, P.ns_pad, P.V, P.color, block_perm(P, smem, NCC, extra), NCC);
    const RefCam& cam = P.ref;
    WarpStats st = {0, 0, 0, 0, 0};
    const int W = P.W, H = P.H;
    constexpr int NC = FUSED ? 20 : 8;

    // gridDim.z slices of the tile's 512 pixels of this colour (small images: more, smaller work units -> no idle SMs in
    // the last wave); inside a slice the warps take pixels dynamically
    const int per_slice = (GPM_TILE * GPM_TILE / 2 + (int)gridDim.z - 1) / (int)gridDim.z;
    const int idx_begin = (int)blockIdx.z * per_slice;
    const int idx_end = min(GPM_TILE * GPM_TILE / 2, idx_begin + per_slice);
    // SHARE: the propagated candidates' costs come from the plane-major pass (share_costs) through cand_cost
    float* const cand_cost = smem + block_smem_bytes(P, NCC, extra) / sizeof(float);
    unsigned char* const cand_need = reinterpret_cast<unsigned char*>(cand_cost + GPM_TILE * GPM_TILE / 2 * 8);
    if constexpr (SHARE) {
        share_need_masks(P, planes, prov, M, colour, phase_mask, idx_begin, idx_end, cand_need, lane, warp);
        __syncthreads();
        share_costs(P, sCam, tile + P.tile_xo, warp_base, src, planes, colour, idx_begin, idx_end, tile_x0, tile_y0, cand_need, cand_cost,
                    counter + 1, stats, lane, st);
        __syncthreads();
    }
    int idx = idx_begin + (int)warp;
    while (idx < idx_end) {
        int px, py;
        colour_pixel(idx, colour, px, py);
        if constexpr (JVS) {
            if (px < W && py < H)
                jvs_pixel<GEO, ADAPTIVE, REFINE_ACMH>(P, J, g, sCam, tile, ws, warp_base + warp_scratch_floats(P.ns_pad, P.V, P.color, NCC), src,
                                                      planes, cost, rng_state, prov, M, px, py, tile_x0, tile_y0, phase_mask, lane, st,
                                                      geo_at<GEOMASK>(R, (size_t)py * W + px), F);
        } else if (px < W && py < H) {
            const size_t center = (size_t)py * W + px;
            bool window_ready = false;          // the per-pixel window data is only built if something gets evaluated
            const float fpx = __int2float_rn(px), fpy = __int2float_rn(py);
            float4 norm_now = planes[center];
            float cost_now = cost[center];
            float disp_now = plane_depth(cam, norm_now.x, norm_now.y, norm_now.z, norm_now.w, fpx, fpy);   // :1530
            // which rounding variant of the cost function produced cost_now: eval_plane's rt (0 = y-first, 1 = x-first, ...), 0xff = unknown
            int prov_now = prov[center];
            PixelPrior pp{};
            if constexpr (PRIOR) pp = pixel_prior(P, R, center, fpx, fpy);
            const bool gon = geo_at<GEOMASK>(R, center);

            // candidate k lives in lane k: 0..3 = up, down, left, right at 1 px (:1571-1582), 4..7 at 5 px (:1450-1462);
            // fused kernel: the 20 candidates of gipuma.cu:1236-1330 in source order
            constexpr unsigned NCMASK = (1u << NC) - 1u;
            float4 mine = make_float4(0.f, 0.f, 0.f, 0.f);
            bool mine_ok = false;
            size_t mine_at = center;
            if (FUSED) {
                if (lane < NC) {
                    mine_ok = (phase_mask & 1) && px >= kFusedGx0[lane] && px <= W - 1 - kFusedGx1[lane] &&
                              py >= kFusedGy0[lane] && py <= H - 1 - kFusedGy1[lane];
                    mine_at = (size_t)(py + kFusedDy[lane]) * W + (px + kFusedDx[lane]);
                }
            } else if (lane < 8) {
                const bool phase_on = (phase_mask >> (lane >> 2)) & 1;
                int qx, qy;
                const bool ok = sweep_neighbour<ADAPTIVE>((int)lane, px, py, W, H, cost, qx, qy);
                mine_ok = ok && phase_on;
                mine_at = (size_t)qy * W + qx;
            }
            const unsigned mine_id = mine_ok ? M.pid[mine_at] : 0u;
            unsigned own_id = M.pid[center];
            // Memo of rejected work.  A pixel's cost only ever decreases (gipuma.cu:867,986), and cost(p, plane) is a pure
            // function, so a neighbour plane this pixel has already been offered — accepted or not — can never be
            // accepted later: seen[p][k] holds the last plane offered from direction k; an unchanged neighbour is skipped
            // without evaluation, in every later iteration.  Exact, not a heuristic.
            // the cost function of the fused kernel differs between its inlined call sites (P.site): the duplicate / memo
            // shortcuts below only pair candidates of sites with the same rounding variant
            // (NCC costs have a provenance code of their own, GPM_PROV_NCC)
            const unsigned my_site = NCC ? GPM_PROV_NCC : FUSED ? (unsigned)P.site[lane < NC ? lane : 0] : (COLOR ? 0u : 1u);
            unsigned mmask = P.memo ? M.mask[center] : 0u;
            const bool old_ok = P.memo && lane < NC && ((mmask >> lane) & 1);
            const unsigned old_id = old_ok ? M.seen[center * NC + lane] : 0u;
            const bool memo_hit = old_ok && mine_ok && old_id == mine_id;
            if (SHARE ? ((cand_need[idx] >> lane) & 1u) != 0u : mine_ok && !memo_hit) mine = planes[mine_at];   // a remembered neighbour is skipped below without its plane
            const unsigned cand_mask = __ballot_sync(GPM_FULL, mine_ok);
            if constexpr (SHARE) {
                // share_need_masks decided every skip from the launch-start state, share_costs evaluated the rest; the scan,
                // in candidate order with strict <, is the one below.  A needed candidate whose identity the pixel took by an
                // accept in this scan costs exactly cost_now, so taking its cost instead of skipping it decides the same.
                const unsigned need = cand_need[idx];
                for (int k = 0; k < NC; k++) {
                    if (!((cand_mask >> k) & 1)) continue;
                    if (!((need >> k) & 1)) { st.skip++; continue; }
                    float4 nb;
                    nb.x = __shfl_sync(GPM_FULL, mine.x, k);  nb.y = __shfl_sync(GPM_FULL, mine.y, k);
                    nb.z = __shfl_sync(GPM_FULL, mine.z, k);  nb.w = __shfl_sync(GPM_FULL, mine.w, k);
                    const unsigned cand_id = __shfl_sync(GPM_FULL, mine_id, k);
                    const float c = cand_cost[idx * 8 + k];
                    if (c < cost_now) {                                                          // :867-871
                        disp_now = plane_depth(cam, nb.x, nb.y, nb.z, nb.w, fpx, fpy);
                        norm_now = nb;
                        cost_now = c;
                        prov_now = 1;
                        own_id = cand_id;
                    }
                }
            } else for (int k = 0; k < NC; k++) {
                if (!((cand_mask >> k) & 1)) continue;
                // rounding variant of this call site: x-first for float images, y-first for float4 (DESIGN.md §2); the fused
                // kernel's inlined sites are looked up (bit 0 = x-first, bit 1 = gradient folding)
                const unsigned site = NCC ? GPM_PROV_NCC : FUSED ? (unsigned)P.site[k] : (COLOR ? 0u : 1u);
                float4 nb;
                nb.x = __shfl_sync(GPM_FULL, mine.x, k);  nb.y = __shfl_sync(GPM_FULL, mine.y, k);
                nb.z = __shfl_sync(GPM_FULL, mine.z, k);  nb.w = __shfl_sync(GPM_FULL, mine.w, k);
                const unsigned cand_id = __shfl_sync(GPM_FULL, mine_id, k);
                // already offered to this pixel before, from ANY direction (the 8 memo entries double as a history)?
                const bool known = old_ok && my_site == site && cand_id == old_id;
                if (__any_sync(GPM_FULL, known)) { st.skip++; continue; }
                // spatialPropagation_cu, gipuma.cu:832-874
                const float disp_before = plane_depth(cam, nb.x, nb.y, nb.z, nb.w, fpx, fpy);
                const bool in_range = disp_before >= cam.depthMin && disp_before <= cam.depthMax;   // :829-830, :865
                // exact duplicates: cost(p, plane) is a pure function, so a plane equal to the current one or to an
                // earlier candidate of this pixel cannot be accepted (`cost_before < *cost_now` is false)
                const bool same_now = P.dedupe_self && prov_now == (int)site && cand_id == own_id;
                const bool same_mine = P.dedupe_cand && mine_ok && (int)lane < k && my_site == site && cand_id == mine_id;
                const bool dup = __any_sync(GPM_FULL, same_mine);
                if (!in_range || same_now || dup) { st.skip++; continue; }
                if (!window_ready) { setup_window<COLOR, NCC>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);  window_ready = true; }
                float pr = 0.0f;
                if constexpr (PRIOR) pr = pp.of(P, R, nb, fpx, fpy);
                const float c = FUSED ? eval_plane<2, COLOR>(P, sCam, ws, src, nb.x, nb.y, nb.z, nb.w, cost_now, lane, st, nullptr, nullptr, site)
                                      : eval_plane<(COLOR ? 0 : 1), COLOR, GEO, NCC, false, PRIOR>(P, sCam, ws, src, nb.x, nb.y, nb.z, nb.w, cost_now, lane, st,
                                                                                nullptr, nullptr, 0u, g, fpx, fpy, pr, gon);
                if (c < cost_now) {                                                              // :867-871
                    disp_now = disp_before;
                    norm_now = nb;
                    cost_now = c;
                    prov_now = (int)site;
                    own_id = cand_id;                                                            // a copy keeps its identity
                }
            }

            if (P.memo && mine_ok && !memo_hit) {            // every candidate offered above is now known to this pixel
                M.seen[center * NC + lane] = mine_id;
            }
            unsigned new_mask = mmask | (cand_mask & NCMASK);
            // The refinement candidates are a pure function of (pixel, plane at refinement start) in GPM_RNG_REFERENCE
            // mode (zero-state stream; disp_now == plane_depth(norm_now) here), so a refinement that rejected all its steps
            // from exactly this plane before would reject them again.  ACMH's candidates also depend on the launch counter:
            // that refinement neither reads nor writes this memo (§23).
            bool refine = (phase_mask & 4) != 0;
            if (!REFINE_ACMH && refine && P.memo && P.rng_mode == 0 && (mmask & GPM_MEMO_REFINE)) {
                if (M.refseen[center] == own_id) {
                    refine = false;
                    st.skip += 3;
                }
            }
            if (REFINE_ACMH && refine) {
                if (!window_ready) { setup_window<COLOR, NCC>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);  window_ready = true; }
                bool any_accept = false;
                const unsigned rsite = NCC ? GPM_PROV_NCC : 0u;
                const float4 start = norm_now;
                const unsigned key = acmh_key(F.seed, (unsigned)center, F.counter);
                for (int j = 0; j < 5; j++) {               // in order, strict <, as the propagation (gipuma.cu:986-990)
                    const float4 cand = acmh_candidate(P, F, key, start, j, fpx, fpy);
                    float pr = 0.0f;
                    if constexpr (PRIOR) pr = pp.of(P, R, cand, fpx, fpy);
                    const float c = eval_plane<0, COLOR, GEO, NCC, false, PRIOR>(P, sCam, ws, src, cand.x, cand.y, cand.z, cand.w, cost_now, lane,
                                                                                 st, nullptr, nullptr, 0u, g, fpx, fpy, pr, gon);
                    if (c < cost_now) {
                        prov_now = (int)rsite;
                        any_accept = true;
                        cost_now = c;
                        norm_now = cand;
                    }
                }
                if (any_accept) {                                 // a new plane: one fresh identity for the pixel's final plane
                    unsigned fresh = 0u;
                    if (lane == 0) fresh = atomicAdd(M.next_id, 1u);
                    own_id = __shfl_sync(GPM_FULL, fresh, 0);
                }
            } else if (refine) {
                if (!window_ready) { setup_window<COLOR, NCC>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);  window_ready = true; }
                const unsigned id_start = own_id;
                bool any_accept = false;
                // planeRefinement_cu, gipuma.cu:928-994 with getRndDispAndUnitVector_cu, :890-927
                Xorwow r = {0u, 0u, 0u, 0u, 0u, 0u};       // GPM_RNG_REFERENCE: gs.cs is never written (gipuma.cu:1840,1608)
                if (P.rng_mode == 1) {
                    const unsigned* in = rng_state + center * 6;
                    r.v0 = in[0];  r.v1 = in[1];  r.v2 = in[2];  r.v3 = in[3];  r.v4 = in[4];  r.d = in[5];
                }
                float vx, vy, vz;
                view_vector(cam, fpx, fpy, vx, vy, vz);                                          // :948
                const float fb = fmul(cam.baseline, cam.f);
                float deltaN = 1.0f;
                for (float deltaZ = fmul(P.max_disp, 0.5f); deltaZ >= 0.01f; deltaZ = fmul(deltaZ, 0.1f)) {   // :958-959
                    const float rdisp = frcp(disp_now);                   // disp = f*baseline/depth (:904), kept fused
                    const float hi = fmin_(ffma(rdisp, -fb, P.max_disp), deltaZ);        // maxDelta (:910)
                    const float lo = fmin_(ffma(rdisp, fb, P.min_disp), deltaZ);         // -minDelta (:909)
                    const float dz = ffma(xorwow_uniform(r), fadd(lo, hi), -lo);        // curand_between(minDelta, maxDelta) :914
                    float dnew = ffma(rdisp, fb, dz);                                    // disp + deltaZ
                    dnew = fmin_(P.max_disp, fmax_(P.min_disp, dnew));                   // :916
                    const float depth_new = fmul(frcp(dnew), fb);                        // :918
                    const float twoN = fadd(deltaN, deltaN);
                    const float ax = fadd(norm_now.x, ffma(xorwow_uniform(r), twoN, -deltaN));   // :921-923
                    const float ay = fadd(norm_now.y, ffma(twoN, xorwow_uniform(r), -deltaN));
                    const float az = fadd(norm_now.z, ffma(twoN, xorwow_uniform(r), -deltaN));
                    const float rs = frsq(ffma(az, az, ffma(ax, ax, fmul(ay, ay))));     // normalize_cu :113-120
                    float4 cand;
                    cand.x = fmul(ax, rs);  cand.y = fmul(ay, rs);  cand.z = fmul(az, rs);
                    if (dot3(cand.x, cand.y, cand.z, vx, vy, vz) > 0.0f) { cand.x = -cand.x;  cand.y = -cand.y;  cand.z = -cand.z; }
                    cand.w = plane_d(cam, cand.x, cand.y, cand.z, fpx, fpy, depth_new);   // :969
                    const unsigned rsite = NCC ? GPM_PROV_NCC : FUSED ? (unsigned)P.site[20] : 0u;
                    float pr = 0.0f;
                    if constexpr (PRIOR) pr = pp.of(P, R, cand, fpx, fpy);
                    const float c = FUSED ? eval_plane<2, COLOR>(P, sCam, ws, src, cand.x, cand.y, cand.z, cand.w, cost_now, lane, st, nullptr, nullptr, rsite)
                                          : eval_plane<0, COLOR, GEO, NCC, false, PRIOR>(P, sCam, ws, src, cand.x, cand.y, cand.z, cand.w, cost_now, lane, st,
                                                                      nullptr, nullptr, 0u, g, fpx, fpy, pr, gon);
                    if (c < cost_now) {                                                          // :986-990 (no depth-range test)
                        prov_now = (int)rsite;
                        any_accept = true;
                        cost_now = c;
                        disp_now = depth_new;
                        norm_now = cand;
                    }
                    deltaN = fmul(deltaN, 0.25f);                                                // :992
                }
                if (P.rng_mode == 1 && lane == 0) {
                    unsigned* o = rng_state + center * 6;
                    o[0] = r.v0;  o[1] = r.v1;  o[2] = r.v2;  o[3] = r.v3;  o[4] = r.v4;  o[5] = r.d;
                }
                if (any_accept) {                                 // a new plane: one fresh identity for the pixel's final plane
                    unsigned fresh = 0u;
                    if (lane == 0) fresh = atomicAdd(M.next_id, 1u);
                    own_id = __shfl_sync(GPM_FULL, fresh, 0);
                }
                if (P.memo && P.rng_mode == 0) {
                    if (!any_accept) { if (lane == 0) M.refseen[center] = id_start;  new_mask |= GPM_MEMO_REFINE; }
                    else new_mask &= ~GPM_MEMO_REFINE;
                }
            }
            if (P.memo && lane == 0 && new_mask != mmask) M.mask[center] = new_mask;
            if (lane == 0) {                                                                     // :1585-1587
                cost[center] = cost_now;
                planes[center] = norm_now;
                prov[center] = (unsigned char)prov_now;
                M.pid[center] = own_id;
            }
        }
        if (lane == 0) idx = idx_begin + atomicAdd(&counter[0], 1);
        idx = __shfl_sync(GPM_FULL, idx, 0);
    }
    flush_stats(stats, st, lane);
}

// ============================================================================================================
// Source-view sharding across GPUs (SURVEY.md §8e, BASELINE configs 4 / 5, north_star's strong-scaling axis).
// Every rank holds the full plane/cost state and a SUBSET of the source views.  Per-view costs are independent
// (gipuma.cu:742-778); only the combination needs all views.  For COMB_BEST_N the n_best smallest costs over all views
// are the n_best smallest of the union of every rank's n_best smallest, so each rank exports, per pixel and hypothesis
// slot, its ascending local top-n_best; the lists of all ranks are exchanged (an all-gather between two launches of
// k_shard_stage) and every rank merges them, sums in ascending order — the reference's order (gipuma.cu:779-797) — and
// applies the accept logic redundantly.  All ranks therefore keep bit-identical state, identical to a single-GPU run over
// all views.
//   stage 0        initial cost of the stored planes        (1 slot,  radius box/2, both colours)
//   stage 1        close + far propagation candidates       (8 slots)
//   stage 2 + s    refinement step s                         (1 slot; sequential: step s+1 depends on step s' accept)
// The accept of stage s is FUSED into the evaluation of stage s+1 (shard_stage_pixel): a colour costs 1 + S evaluation
// passes plus one closing accept instead of 2 (1 + S) launches.  The exact shortcuts of k_sweep that depend only on the
// shared state are kept — direction memo, history, duplicates (incl. the current plane), refinement memo — so every rank
// skips the same work and the skipped slots simply carry +inf lists.
// Exchange index of pixel (x, y): y * ceil(W/2) + x/2 (pixels of one colour have distinct x/2 within a row).  A rank's
// lists of one stage are dense: (stage == 1 ? 8 : 1) slots of n_best floats per exchange index (stage 0: one such plane
// per colour); the gathered lists are those of every rank, rank-major.
// ============================================================================================================
#define GPM_SF_SKIP_REFINE 1u     // sflags: the refinement of this colour pass is known to reject every step (memo)
#define GPM_SF_ACCEPTED    2u     // sflags: some refinement step of this colour pass was accepted

struct ShardState {
    float* dispbuf;               // disp_now carried between the stages of one colour
    float4* candbuf;              // refinement candidate of the step being exchanged
    float* canddepth;
    unsigned char* sflags;
};

// merged cost of one slot: the n_best smallest over all ranks' lists, summed ascending, / count  (gipuma.cu:779-803).
// A slot that every rank skipped (not offered, out of range, memo hit, duplicate) has only +inf entries and merges to +inf,
// so that no accept can take it whatever the pixel's cost; an evaluated slot always has finite entries (local_topn clamps
// every cost to MAXCOST), and MAXCOST when none of them is below MAXCOST.
__device__ __forceinline__ float shard_merge(const float* __restrict__ g, size_t rank_stride, int world, int nb)
{
    int pos[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    float sum = 0.0f;
    int taken = 0;
    for (int i = 0; i < nb; i++) {
        float best = __int_as_float(0x7f800000);
        int br = -1;
        for (int r = 0; r < world; r++) {
            if (pos[r] < nb) { const float v = __ldcg(g + r * rank_stride + pos[r]); if (v < best) { best = v;  br = r; } }
        }
        if (br < 0 && i == 0) return __int_as_float(0x7f800000);      // no rank has a finite entry: the slot was skipped
        if (br < 0 || !(best < GPM_MAXCOST)) break;        // only views with c < MAXCOST count (numValidViews)
        pos[br]++;
        sum = fadd(sum, best);
        taken++;
    }
    float cost = fmul(frcp(__int2float_rn(taken)), sum);
    if (taken < 1) cost = GPM_MAXCOST;
    if (cost != cost || cost > GPM_MAXCOST || cost < 0.0f) cost = GPM_MAXCOST;
    return cost;
}

__device__ __forceinline__ bool same_bits(const float4& a, const float4& b)
{
    return __float_as_uint(a.x) == __float_as_uint(b.x) && __float_as_uint(a.y) == __float_as_uint(b.y) &&
           __float_as_uint(a.z) == __float_as_uint(b.z) && __float_as_uint(a.w) == __float_as_uint(b.w);
}

// refinement candidate of step `sidx` from (norm_now, disp_now) — getRndDispAndUnitVector_cu, gipuma.cu:890-927, with the
// reference's zero-state stream (pin P2) advanced by 4 draws per earlier step.  The step restates k_sweep's refinement loop
// body line for line, and a fix to one must go to both: k_sweep keeps its own copy because calling a shared helper there
// changes the register allocation of its colour instantiations.
__device__ __forceinline__ float4 shard_refine_candidate(const KParams& P, const float4& norm_now, float disp_now, float fpx, float fpy,
                                                         int sidx, float& depth_new)
{
    const RefCam& cam = P.ref;
    Xorwow r = {0u, 0u, 0u, 0u, 0u, 0u};
    float deltaZ = fmul(P.max_disp, 0.5f), deltaN = 1.0f;
    for (int i = 0; i < sidx; i++) { for (int j = 0; j < 4; j++) xorwow_next(r);  deltaZ = fmul(deltaZ, 0.1f);  deltaN = fmul(deltaN, 0.25f); }
    float vx, vy, vz;
    view_vector(cam, fpx, fpy, vx, vy, vz);
    const float fb = fmul(cam.baseline, cam.f);
    const float rdisp = frcp(disp_now);
    const float hi = fmin_(ffma(rdisp, -fb, P.max_disp), deltaZ);
    const float lo = fmin_(ffma(rdisp, fb, P.min_disp), deltaZ);
    const float dz = ffma(xorwow_uniform(r), fadd(lo, hi), -lo);
    float dnew = ffma(rdisp, fb, dz);
    dnew = fmin_(P.max_disp, fmax_(P.min_disp, dnew));
    depth_new = fmul(frcp(dnew), fb);
    const float twoN = fadd(deltaN, deltaN);
    const float ax = fadd(norm_now.x, ffma(xorwow_uniform(r), twoN, -deltaN));
    const float ay = fadd(norm_now.y, ffma(twoN, xorwow_uniform(r), -deltaN));
    const float az = fadd(norm_now.z, ffma(twoN, xorwow_uniform(r), -deltaN));
    const float rs = frsq(ffma(az, az, ffma(ax, ax, fmul(ay, ay))));
    float4 cand;
    cand.x = fmul(ax, rs);  cand.y = fmul(ay, rs);  cand.z = fmul(az, rs);
    if (dot3(cand.x, cand.y, cand.z, vx, vy, vz) > 0.0f) { cand.x = -cand.x;  cand.y = -cand.y;  cand.z = -cand.z; }
    cand.w = plane_d(cam, cand.x, cand.y, cand.z, fpx, fpy, depth_new);
    return cand;
}

// Accept of stage `stage` at pixel (px, py) from the exchanged lists (one warp; every lane returns the same state).
// stage 1: the 8 propagation slots in the reference's order (gipuma.cu:1571-1582, 1450-1462; accept rule :867-871);
// stage >= 2: one refinement step (:986-990).  ADAPTIVE: slot k is acs_neighbour's choice, re-derived from the costs of the
// other colour, which no stage of this colour writes, so it is the pixel stage 1 evaluated.
template <bool ADAPTIVE>
__device__ __forceinline__ void shard_accept_pixel(const KParams& P, const float4* __restrict__ planes, const float* __restrict__ cost,
                                                   const ShardState& S, const Memo& M,
                                                   int px, int py, int stage, const float* __restrict__ gathered, int world,
                                                   float4& norm_now, float& cost_now, float& disp_now, int& prov_now, unsigned& sf,
                                                   unsigned& own_id, unsigned lane)
{
    const int W = P.W, H = P.H, Wh = (W + 1) >> 1, nb = P.n_best;
    const size_t center = (size_t)py * W + px;
    const int slots = stage == 1 ? 8 : 1;
    const size_t per_rank = (size_t)H * Wh * slots * nb;
    const float* g = gathered + ((size_t)py * Wh + (px >> 1)) * slots * nb;
    const float fpx = __int2float_rn(px), fpy = __int2float_rn(py);
    if (stage == 1) {
        float mine = GPM_MAXCOST;
        if (lane < 8) mine = shard_merge(g + lane * nb, per_rank, world, nb);
        for (int k = 0; k < 8; k++) {
            const float c = __shfl_sync(GPM_FULL, mine, k);
            if (c < cost_now) {
                int qx, qy;
                sweep_neighbour<ADAPTIVE>(k, px, py, W, H, cost, qx, qy);   // offered, so inside the border guard / region
                norm_now = planes[(size_t)qy * W + qx];                 // other colour: not written during this colour's stages
                own_id = M.pid[(size_t)qy * W + qx];                    // a copy keeps its identity
                disp_now = plane_depth(P.ref, norm_now.x, norm_now.y, norm_now.z, norm_now.w, fpx, fpy);
                cost_now = c;
                prov_now = P.color ? 0 : 1;
            }
        }
    } else if (!(sf & GPM_SF_SKIP_REFINE)) {
        const float c = shard_merge(g, per_rank, world, nb);
        if (c < cost_now) {
            cost_now = c;  norm_now = S.candbuf[center];  disp_now = S.canddepth[center];  prov_now = 0;
            sf |= GPM_SF_ACCEPTED;
        }
    }
}

// One stage of one pixel: [accept of stage-1's exchange] + evaluation of `stage` on this rank's views -> local top-n lists.
template <bool COLOR, bool ADAPTIVE>
__device__ __forceinline__ void shard_stage_pixel(const KParams& P, const float* __restrict__ sCam, const float* __restrict__ tile,
                                                  const WarpScratch& ws, cudaTextureObject_t src, float4* __restrict__ planes, float* __restrict__ cost, unsigned char* __restrict__ prov,
                                                  const ShardState& S, const Memo& M, int px, int py, int tile_x0, int tile_y0,
                                                  int stage, int last_stage, const float* __restrict__ gathered_prev, int world,
                                                  float* __restrict__ xchg, unsigned lane, WarpStats& st)
{
    const RefCam& cam = P.ref;
    const int W = P.W, H = P.H, Wh = (W + 1) >> 1, nb = P.n_best;
    const size_t center = (size_t)py * W + px;
    const float inf = __int_as_float(0x7f800000);
    const float fpx = __int2float_rn(px), fpy = __int2float_rn(py);
    float c0, c1;
    float4 norm_now = planes[center];
    if (stage == 0) {                                       // initial costs (gipuma.cu:1040-1049), both colours: two half-resolution planes
        float* out = xchg + ((size_t)((px + py) & 1) * H * Wh + (size_t)py * Wh + (px >> 1)) * nb;
        setup_window<COLOR>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);
        eval_plane<(COLOR ? 1 : 0), COLOR>(P, sCam, ws, src, norm_now.x, norm_now.y, norm_now.z, norm_now.w, inf, lane, st, &c0, &c1);
        local_topn(P, c0, c1, lane, out);
        return;
    }
    float cost_now = cost[center];
    int prov_now = prov[center];
    unsigned sf = stage >= 2 ? (unsigned)S.sflags[center] : 0u;
    float disp_now = stage >= 2 ? S.dispbuf[center] : plane_depth(cam, norm_now.x, norm_now.y, norm_now.z, norm_now.w, fpx, fpy);
    unsigned mmask = P.memo ? M.mask[center] : 0u;
    unsigned new_mask = mmask;
    unsigned own_id = M.pid[center];
    if (stage >= 2) {
        shard_accept_pixel<ADAPTIVE>(P, planes, cost, S, M, px, py, stage - 1, gathered_prev, world, norm_now, cost_now, disp_now, prov_now, sf, own_id, lane);
        if (stage == 2) {
            // refinement memo (see k_sweep): the S candidates are a pure function of (pixel, plane at refinement start)
            sf = 0u;
            if (P.memo && P.rng_mode == 0) {
                if ((mmask & GPM_MEMO_REFINE) && M.refseen[center] == own_id) sf = GPM_SF_SKIP_REFINE;
                else { if (lane == 0) M.refseen[center] = own_id;  new_mask &= ~GPM_MEMO_REFINE; }
            }
        }
    }
    float* out = xchg + ((size_t)py * Wh + (px >> 1)) * (stage == 1 ? 8 : 1) * nb;
    if (stage > last_stage) {                               // closing pass of a colour: only the accept of the last refinement step
        if (P.memo && P.rng_mode == 0 && !(sf & (GPM_SF_SKIP_REFINE | GPM_SF_ACCEPTED))) new_mask |= GPM_MEMO_REFINE;
        if (sf & GPM_SF_ACCEPTED) {                         // the refinement created a new plane: one fresh identity
            unsigned fresh = 0u;
            if (lane == 0) fresh = atomicAdd(M.next_id, 1u);
            own_id = __shfl_sync(GPM_FULL, fresh, 0);
        }
    } else if (stage == 1) {
        float4 mine = make_float4(0.f, 0.f, 0.f, 0.f);
        bool mine_ok = false;
        size_t mine_at = center;
        if (lane < 8) {
            int qx, qy;
            mine_ok = sweep_neighbour<ADAPTIVE>((int)lane, px, py, W, H, cost, qx, qy);
            mine_at = (size_t)qy * W + qx;
        }
        const unsigned mine_id = mine_ok ? M.pid[mine_at] : 0u;
        const bool old_ok = P.memo && lane < 8 && ((mmask >> lane) & 1);
        const unsigned old_id = old_ok ? M.seen[center * 8 + lane] : 0u;
        const bool memo_hit = old_ok && mine_ok && old_id == mine_id;
        if (mine_ok && !memo_hit) mine = planes[mine_at];
        const unsigned cand_mask = __ballot_sync(GPM_FULL, mine_ok);
        const int site = COLOR ? 0 : 1;
        bool window_ready = false;
        for (int k = 0; k < 8; k++) {
            float4 nbp;
            nbp.x = __shfl_sync(GPM_FULL, mine.x, k);  nbp.y = __shfl_sync(GPM_FULL, mine.y, k);
            nbp.z = __shfl_sync(GPM_FULL, mine.z, k);  nbp.w = __shfl_sync(GPM_FULL, mine.w, k);
            const unsigned cand_id = __shfl_sync(GPM_FULL, mine_id, k);
            bool skip = !((cand_mask >> k) & 1);
            if (!skip) skip = __any_sync(GPM_FULL, old_ok && cand_id == old_id);            // offered before, from any direction
            if (!skip) {
                const float d = plane_depth(cam, nbp.x, nbp.y, nbp.z, nbp.w, fpx, fpy);
                const bool in_range = d >= cam.depthMin && d <= cam.depthMax;
                // a plane equal to the current one (cost of the same rounding variant) or to an earlier slot can never pass
                // `cost < cost_now`: cost_now only decreases while the slots are accepted in order
                const bool same_now = P.dedupe_self && prov_now == site && cand_id == own_id;
                const bool same_mine = P.dedupe_cand && mine_ok && (int)lane < k && cand_id == mine_id;
                skip = !in_range || same_now || __any_sync(GPM_FULL, same_mine);
            }
            if (skip) { st.skip++;  if ((int)lane < nb) out[k * nb + lane] = inf;  __syncwarp();  continue; }
            if (!window_ready) { setup_window<COLOR>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);  window_ready = true; }
            eval_plane<(COLOR ? 0 : 1), COLOR>(P, sCam, ws, src, nbp.x, nbp.y, nbp.z, nbp.w, inf, lane, st, &c0, &c1);
            local_topn(P, c0, c1, lane, out + k * nb);
        }
        if (P.memo && mine_ok && !memo_hit) M.seen[center * 8 + lane] = mine_id;
        new_mask |= (cand_mask & 0xffu);
    } else {
        if (sf & GPM_SF_SKIP_REFINE) {
            st.skip++;
            if ((int)lane < nb) out[lane] = inf;
        } else {
            float depth_new;
            const float4 cand = shard_refine_candidate(P, norm_now, disp_now, fpx, fpy, stage - 2, depth_new);
            if (lane == 0) { S.candbuf[center] = cand;  S.canddepth[center] = depth_new; }
            setup_window<COLOR>(P, tile + P.tile_xo, ws, px, py, tile_x0, tile_y0, lane);
            eval_plane<0, COLOR>(P, sCam, ws, src, cand.x, cand.y, cand.z, cand.w, inf, lane, st, &c0, &c1);
            local_topn(P, c0, c1, lane, out);
        }
    }
    if (lane == 0) {
        if (stage >= 2) { planes[center] = norm_now;  cost[center] = cost_now;  prov[center] = (unsigned char)prov_now;  M.pid[center] = own_id; }
        if (stage >= 1) { S.dispbuf[center] = disp_now;  S.sflags[center] = (unsigned char)sf; }
        if (P.memo && new_mask != mmask) M.mask[center] = new_mask;
    }
}

// One exchange stage over the whole image (the all-gather runs between two launches of this kernel).
// stage 0: both colours; 1 .. last_stage: one colour; last_stage + 1: closing accept of the colour.
// ADAPTIVE: adaptive checkerboard sampling (DESIGN.md §16); the exchange format is the same.
template <bool COLOR, bool ADAPTIVE = false>
__global__ void __launch_bounds__(GPM_LB_THREADS, GPM_LB_BLOCKS)
k_shard_stage(const __grid_constant__ KParams P, const __grid_constant__ CUtensorMap tmap, const ViewCam* __restrict__ cams,
              cudaTextureObject_t src, float4* __restrict__ planes, float* __restrict__ cost,
              unsigned char* __restrict__ prov, ShardState S, Memo M, int colour, int stage, int last_stage, const float* __restrict__ gathered_prev,
              int world, float* __restrict__ xchg, unsigned long long* __restrict__ stats)
{
    extern __shared__ __align__(128) float smem[];
    float* tile = smem;
    float* sCam = tile + tile_floats(P);
    float* scratch = smem + fixed_smem_floats(P);
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile_x0 = blockIdx.x * GPM_TILE - P.halo, tile_y0 = blockIdx.y * GPM_TILE - P.halo;
    if (stage <= last_stage) stage_block(P, &tmap, cams, tile, sCam, tile_x0, tile_y0);
    const WarpScratch ws = carve(scratch + (size_t)warp * warp_scratch_floats(P.ns_pad, P.V, P.color), P.ns_pad, P.V, P.color, block_perm(P, smem));
    WarpStats st = {0, 0, 0, 0, 0};
    // stage 0 visits every pixel (both colours, like gipuma_init_cu2); the others one colour
    const int npix = (stage == 0) ? GPM_TILE * GPM_TILE : GPM_TILE * GPM_TILE / 2;
    // gridDim.z slices of the tile's pixel list, as in k_sweep
    const int per_slice = (npix + (int)gridDim.z - 1) / (int)gridDim.z;
    const int idx_end = min(npix, ((int)blockIdx.z + 1) * per_slice);
    for (int idx = (int)blockIdx.z * per_slice + (int)warp; idx < idx_end; idx += P.nwarps) {
        int px, py;
        if (stage == 0) { px = blockIdx.x * GPM_TILE + (idx & 31);  py = blockIdx.y * GPM_TILE + (idx >> 5); }
        else colour_pixel(idx, colour, px, py);
        if (px >= P.W || py >= P.H) continue;
        shard_stage_pixel<COLOR, ADAPTIVE>(P, sCam, tile, ws, src, planes, cost, prov, S, M, px, py,
                                 tile_x0, tile_y0, stage, last_stage, gathered_prev, world, xchg, lane, st);
    }
    flush_stats(stats, st, lane);
}

// closing accept of stage 0: merged initial costs for both colours (thread per half-row position)
__global__ void k_shard_accept0(const __grid_constant__ KParams P, float* __restrict__ cost, unsigned char* __restrict__ prov,
                                const float* __restrict__ gathered, int world)
{
    const int W = P.W, H = P.H, Wh = (W + 1) >> 1, nb = P.n_best;
    const int hx = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (hx >= Wh || py >= H) return;
    const size_t per_rank = (size_t)2 * H * Wh * nb;
    for (int col = 0; col < 2; col++) {
        const int px = 2 * hx + ((py + col) & 1);                      // the pixel of this colour with x/2 == hx in row py
        if (px >= W) continue;
        const size_t center = (size_t)py * W + px;
        const float* g = gathered + ((size_t)col * H * Wh + (size_t)py * Wh + hx) * nb;
        cost[center] = shard_merge(g, per_rank, world, nb);
        prov[center] = P.color ? 3 : 0;          // initialisation variant
    }
}

// ---- planar prior construction and offer (DESIGN.md §18) ------------------------------------------------------------
// Support point of each step x step cell (one thread per cell): the pixel with the smallest stored cost, NaN never winning
// and a tie going to the lower (y, x), kept when its cost < support_cost and its plane's prior_depth is in range.
// at[cell] = its pixel index or -1, plane[cell] = its plane.
__global__ void k_prior_support(const __grid_constant__ KParams P, const float4* __restrict__ planes, const float* __restrict__ cost,
                                int step, float support_cost, int cells_x, int cells_y, int* __restrict__ at, float4* __restrict__ plane)
{
    const int cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y;
    if (cx >= cells_x || cy >= cells_y) return;
    int best = -1;
    float best_c = 0.0f;
    for (int y = cy * step; y < min(P.H, cy * step + step); y++)
        for (int x = cx * step; x < min(P.W, cx * step + step); x++) {
            const float c = cost[(size_t)y * P.W + x];
            if (c == c && (best < 0 || c < best_c)) { best = y * P.W + x;  best_c = c; }
        }
    int keep = -1;
    float4 pl = make_float4(0.f, 0.f, 0.f, 0.f);
    if (best >= 0 && best_c < support_cost) {
        pl = planes[best];
        const float dep = prior_depth(P.ref, pl.x, pl.y, pl.z, pl.w, __int2float_rn(best % P.W), __int2float_rn(best / P.W));
        if (dep >= P.ref.depthMin && dep <= P.ref.depthMax) keep = best;
    }
    at[cy * cells_x + cx] = keep;
    plane[cy * cells_x + cx] = pl;
}

// Rasterisation of the triangles (one thread per triangle over its bounding box).  tri[t] = three counter-clockwise
// (orient > 0) integer vertices x0 y0 x1 y1 x2 y2.  Pixel p belongs to a triangle when every edge a -> b has
// orient(a, b, p) > 0, or = 0 and the edge is top-left (b.y > a.y, or b.y == a.y and b.x < a.x): an interior edge is
// top-left in exactly one of its two triangles, so every pixel inside the hull belongs to exactly one triangle.  The pixel
// gets the triangle's plane where that plane's prior_depth is in range (counted in *with_prior), and stays all-zero else.
__global__ void k_prior_raster(const __grid_constant__ KParams P, const int* __restrict__ tri, const float4* __restrict__ tri_plane,
                               int ntri, float4* __restrict__ map, unsigned long long* __restrict__ with_prior)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntri) return;
    const int* v = tri + 6 * t;
    const float4 pl = tri_plane[t];
    if (pl.x == 0.f && pl.y == 0.f && pl.z == 0.f && pl.w == 0.f) return;            // no plane (degenerate triangle)
    const int x0 = min(v[0], min(v[2], v[4])), x1 = max(v[0], max(v[2], v[4]));
    const int y0 = min(v[1], min(v[3], v[5])), y1 = max(v[1], max(v[3], v[5]));
    unsigned long long n = 0;
    for (int y = y0; y <= y1; y++)
        for (int x = x0; x <= x1; x++) {
            bool in = true;
            for (int e = 0; e < 3 && in; e++) {
                const long long ax = v[2 * e], ay = v[2 * e + 1], bx = v[(2 * e + 2) % 6], by = v[(2 * e + 3) % 6];
                const long long o = (bx - ax) * ((long long)y - ay) - (by - ay) * ((long long)x - ax);
                in = o > 0 || (o == 0 && (by > ay || (by == ay && bx < ax)));
            }
            if (!in) continue;
            const float dep = prior_depth(P.ref, pl.x, pl.y, pl.z, pl.w, __int2float_rn(x), __int2float_rn(y));
            if (dep >= P.ref.depthMin && dep <= P.ref.depthMax) { map[(size_t)y * P.W + x] = pl;  n++; }
        }
    if (n) atomicAdd(with_prior, n);
}

// gpm_offer_prior: pixel p with a prior takes its prior plane when that plane's cost c_prior[p] (k_cost_eval under the
// context's mode) is strictly below the stored cost.  An accepted plane gets the fresh identity *next_id + p; the caller
// then advances the counter by W*H, so the identities do not depend on the order in which the threads run.
__global__ void k_offer_prior(const __grid_constant__ KParams P, const float4* __restrict__ map, const float* __restrict__ c_prior,
                              float4* __restrict__ planes, float* __restrict__ cost, unsigned char* __restrict__ prov, unsigned site,
                              unsigned* __restrict__ pid, const unsigned* __restrict__ next_id)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= P.W || y >= P.H) return;
    const size_t at = (size_t)y * P.W + x;
    const float4 pi = map[at];
    const float dep = prior_depth(P.ref, pi.x, pi.y, pi.z, pi.w, __int2float_rn(x), __int2float_rn(y));
    if (!(dep >= P.ref.depthMin && dep <= P.ref.depthMax) || !(c_prior[at] < cost[at])) return;
    planes[at] = pi;
    cost[at] = c_prior[at];
    prov[at] = (unsigned char)site;
    pid[at] = *next_id + (unsigned)at;
}

__global__ void k_advance_ids(unsigned* __restrict__ next_id, unsigned n) { *next_id += n; }

// ---- final depth / world normal — gipuma_compute_disp, gipuma.cu:1080-1103 ------------------
__global__ void k_finalize(const __grid_constant__ KParams P, float4* __restrict__ planes, const float* __restrict__ cost)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= P.W || y >= P.H) return;
    const size_t center = (size_t)y * P.W + x;
    const float4 n = planes[center];
    const float* R = P.ref.R_orig_inv;
    float4 o;
    o.x = ffma(n.z, R[2], ffma(n.x, R[0], fmul(n.y, R[1])));
    o.y = ffma(n.z, R[5], ffma(n.x, R[3], fmul(n.y, R[4])));
    o.z = ffma(n.z, R[8], ffma(n.x, R[6], fmul(n.y, R[7])));
    o.w = (cost[center] != GPM_MAXCOST) ? plane_depth(P.ref, n.x, n.y, n.z, n.w, __int2float_rn(x), __int2float_rn(y)) : 0.0f;
    planes[center] = o;
}

// Ceiling of the unit that bounds this path, measured in process: filtered R32F fetches per second of the texture unit in its
// best case — 32 lanes = 16 x 2 adjacent texels (every hardware quad a 2x2 block; 1143 Gfetch/s in tools/texbench.cu), the five
// taps of the reference's sample pattern, one layer per warp — on the context's own layered texture.  bench.py divides the
// fetch rate it achieves by this number (roofline.binding_unit).
__global__ void k_fetch_peak(cudaTextureObject_t src, int xmask, int ymask, int V, int reps, float* __restrict__ sink)
{
    const int lane = threadIdx.x & 31, warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const float dx = (float)(lane >> 1), dy = (float)(lane & 1);
    const int v = warp % V;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
    unsigned h = (unsigned)warp * 2654435761u + 12345u;
    for (int r = 0; r < reps; r++) {
        h = h * 1664525u + 1013904223u;
        const float x = 8.37f + (float)((h >> 8) & (unsigned)xmask) + dx;
        const float y = 8.61f + (float)((h >> 20) & (unsigned)ymask) + dy;
        a0 += tex2DLayered<float>(src, x, y, v);
        a1 += tex2DLayered<float>(src, x + 1.0f, y, v);
        a2 += tex2DLayered<float>(src, x - 1.0f, y, v);
        a3 += tex2DLayered<float>(src, x, y + 1.0f, v);
        a4 += tex2DLayered<float>(src, x, y - 1.0f, v);
    }
    const float a = a0 + a1 + a2 + a3 + a4;
    if (a == 12345.678f) sink[0] = a;
}

// Colour source views are sampled from three R32F planes (layer 3v + channel) instead of one RGBA32F layer.
__global__ void k_split_channels(const float4* __restrict__ in, size_t pitch_elems, int W, int H, float* __restrict__ out)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    const float4 p = in[(size_t)y * pitch_elems + x];
    const size_t plane = (size_t)W * H, o = (size_t)y * W + x;
    out[o] = p.x;  out[plane + o] = p.y;  out[2 * plane + o] = p.z;
}

// replicate-pad the reference image (T = float or float4 texels) by GPM_APRON on the left / top and out to the end of the
// allocation on the right / bottom (== the texture's clamp addressing, main.cpp:644-645): the window of the last tile row /
// column reaches roundup(size, 32) + halo + GPM_APRON, past size + 2 * GPM_APRON whenever size % 32 is small
template <typename T>
__global__ void k_pad_reference(const T* __restrict__ img, size_t pitch_elems, int W, int H, T* __restrict__ out, int out_pitch, int out_rows)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= out_pitch || y >= out_rows) return;
    const int sx = min(max(x - GPM_APRON, 0), W - 1), sy = min(max(y - GPM_APRON, 0), H - 1);
    out[(size_t)y * out_pitch + x] = img[(size_t)sy * pitch_elems + sx];
}

}  // namespace gpm
