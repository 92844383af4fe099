// gpm_api.cu — host side of libgipuma_b200.so: the C-ABI declared in include/gipuma_b200.h.
// Replaces the host launcher gipuma<T>() (reference gipuma.cu:1825-1960) and, through the adapter in
// runcuda_adapter.cu, int runcuda(GlobalState&) (gipuma.cu:1962-1970).
//
// Device memory layout (everything resident in HBM for the life of the context):
//   planes   float4[H*W]   (n.xyz, d) row-major, stride W   — LineState::norm4 layout (linestate.h:10)
//   cost     float [H*W]                                      — LineState::c
//   refpad   float [(H+32) x pitch]  reference image, replicate-padded by 16 px, pitch multiple of 32 texels
//   src      cudaArray (layered, R32F, W x H x max_views) + one texture object: Linear filter, the
//            reference's addressing (Wrap + unnormalised, main.cpp:642-648), element read mode
//            (refpad and src are allocated by the first image upload; colour: float4 texels, 3 x max_views layers)
//   cams     ViewCam[max_views]  (K, R, t per source view) — copied to shared memory by every block
//   rng      uint32[H*W*6]  XORWOW state per pixel (GPM_RNG_STATEFUL only)
// No CPU fallback exists: every entry point needs a CUDA device and reports GPM_E_CUDA otherwise.
#include "../../include/gipuma_b200.h"
#include "gpm_kernels.cuh"
#include "gpm_scale.cuh"

#include <algorithm>
#include <array>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

using namespace gpm;

static thread_local std::string g_err;

static int fail(int code, const std::string& msg)
{
    g_err = msg;
    return code;
}

namespace gpm {
int set_last_error(int code, const std::string& msg) { return fail(code, msg); }     // for gpm_fuse.cu and gpm_cloud.cu

// The planar prior's bound (DESIGN.md §18): the largest valid cost of parameters p (PM: ns at the initialisation window
// times the largest dissimilarity; NCC: 2) plus the geometric term's largest value plus the prior's weight stays below
// MAXCOST, so that a valid cost with the term never reaches MAXCOST.  Checked by every setter that changes one of them,
// and by the multi-level driver before any CUDA call (gpm_batch.cpp).
bool prior_bound_ok(const gpm_params& p, bool ncc, float geo_weight, float geo_max_err, float prior_weight)
{
    if (prior_weight <= 0.f) return true;
    const int nside = p.box_hsize / 2 + 1;
    const float top = ncc ? 2.0f : (float)(nside * nside) * ((1.0f - p.alpha) * p.tau_color + p.alpha * p.tau_gradient);
    return top + geo_weight * geo_max_err + prior_weight < GPM_MAXCOST;
}
}

#define CU(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess)                                                                        \
            return fail(GPM_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));              \
    } while (0)

struct gpm_ctx {
    int device = 0, W = 0, H = 0, maxV = 0, V = 0;
    int color = -1;                  // -1 undecided, 0 float images, 1 float4 (RGB) images — fixed by the first image upload
    gpm_params prm{};
    bool have_params = false, have_ref = false;
    std::vector<char> have_view;
    float4* planes = nullptr;
    float* cost = nullptr;
    unsigned* rng = nullptr;
    float* dispbuf = nullptr;        // view-shard mode: disp_now carried between the stages of one colour
    float4* candbuf = nullptr;       // view-shard mode: refinement candidate of the current step
    float* canddepth = nullptr;
    unsigned char* sflags = nullptr; // view-shard mode: per-pixel flags of the current colour pass (GPM_SF_*)
    float* xchg = nullptr;           // view-shard mode: this rank's lists of the current stage / all ranks' lists (gpm_shard_run)
    float* gath = nullptr;
    size_t xchg_floats = 0;
    int gath_world = 0;
    void* comm = nullptr;            // ncclComm_t of the shard group
    bool comm_owned = false;
    int shard_rank = 0, shard_world = 0;
    unsigned long long collectives = 0;
    // Setters only mark state stale; build_kparams clears it once, at the next launch (reset_state_tags)
    bool inputs_dirty = false;       // the cost function or its inputs changed: stored costs (prov) and memo are stale
    bool memo_dirty = false;         // only what the memo may assume changed: the memo is stale
    unsigned* seen = nullptr;        // [H*W*ncand] identity of the plane last offered to each pixel from each of the 8 (fused kernel: 20) propagation directions
    int seen_slots = 8;
    unsigned* refseen = nullptr;     // [H*W]   identity of the plane from which the last all-rejected refinement started
    unsigned* pid = nullptr;         // [H*W]   identity of the stored plane (gpm_kernels.cuh, struct Memo)
    unsigned* next_id = nullptr;     // device counter of fresh identities
    unsigned* memo_mask = nullptr;   // [H*W] validity bits of seen (0-19) and refseen (GPM_MEMO_REFINE)
    unsigned char* prov = nullptr;   // per pixel: which rounding variant of the cost function produced cost[] (see k_sweep)
    // image storage, allocated by the first upload for the context's image type (ensure_color); texel = float, colour: float4
    float* refpad = nullptr;         // padded reference image: refrows x refpitch texels
    int refpitch = 0, refrows = 0;
    CUtensorMap tmap{};              // 2-D TMA descriptor of the padded reference image for the current box size
    int tmap_box = 0;
    float* staging = nullptr;        // W*H texels, upload scratch
    // source views, layered R32F: one layer per view; colour: 3 channel planes per view, layer 3v + ch (an RGBA32F fetch
    // costs several R32F ones, tools/texbench.cu)
    cudaArray_t srcArr = nullptr;
    cudaTextureObject_t srcTex = 0;
    float* planar = nullptr;         // colour only: [3][H][W] split target
    ViewCam* d_cams = nullptr;
    std::vector<ViewCam> h_cams;
    bool cams_dirty = true;
    RefCam ref{};
    unsigned long long seed = 0xC0FFEEULL;
    int rng_mode = GPM_RNG_REFERENCE;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    unsigned long long* d_stats = nullptr;
    unsigned long long launches = 0;
    int opt_prune = 1, opt_dedupe = 1, opt_trust_state = 0, opt_nwarps = 0;
    int opt_cost_variant = -1, opt_memo = 1, opt_quadperm = 1;
    int opt_neighbours = 8;                      // 20: the reference's fused kernel (built when SMALLKERNEL is not defined)
    int opt_site[21];                            // diagnostics: override the fused kernel's call-site variants (-1 = table)
    int smem_optin = 0, num_sms = 132;
    // geometric-consistency mode (DESIGN.md §14): on while geo_weight > 0 (gpm_set_geometric)
    float geo_weight = 0.f, geo_max_err = 1.f;
    float* geo_depth = nullptr;      // [maxV][H][W] source views' depth maps, allocated by the first gpm_set_view_depth
    float* geo_kinv = nullptr;       // [maxV][9]    K^-1 of each source view (copied with the camera table, sync_cams)
    std::vector<char> have_depth;
    std::vector<float> h_kinv;
    float ref_K[9] = {0.f};
    // photometric cost (DESIGN.md §15): GPM_PHOTO_PM, the reference's, or GPM_PHOTO_NCC (gpm_set_photometric)
    int photo = GPM_PHOTO_PM;
    float ncc_min_std = 0.f;
    // propagation (DESIGN.md §16): GPM_PROP_FIXED, the reference's neighbours, or GPM_PROP_ADAPTIVE (gpm_set_propagation)
    int propagation = GPM_PROP_FIXED;
    // view selection (DESIGN.md §17): GPM_VSEL_OFF or GPM_VSEL_JOINT with its parameters (gpm_set_view_selection)
    gpm_view_sel vsel{GPM_VSEL_OFF, 0.f, 0.f, 0.f, 0, 0, 0.f, 0.f};
    unsigned long long* vsel_mask = nullptr;   // [H*W] selected-views masks, allocated by the first switch to JOINT
    int vsel_t = 0;                            // iterations of gpm_sweep since gpm_init / gpm_set_state
    // planar prior (DESIGN.md §18): on while prior_weight > 0 (gpm_set_prior); the map is uploaded or built
    float4* prior_map = nullptr;               // [H*W], allocated by the first gpm_set_planar_prior / gpm_build_planar_prior
    float* prior_cost = nullptr;               // [H*W] gpm_offer_prior's costs of the prior planes
    float prior_weight = 0.f, prior_depth_sigma = 1.f, prior_normal_deg = 5.f;
    bool have_state = false;                   // gpm_init, gpm_run or gpm_set_state has given every pixel a plane and a cost
    // the geometric term's per-pixel mask (DESIGN.md §21): nonzero bytes switch the term off; read while geo_mask_set
    unsigned char* geo_mask = nullptr;         // [H*W], allocated by the first gpm_set_geo_mask
    bool geo_mask_set = false;
    // refinement (DESIGN.md §23): GPM_REFINE_GIPUMA, the reference's, or GPM_REFINE_ACMH (gpm_set_refinement)
    int refine_kind = GPM_REFINE_GIPUMA;
    float refine_eps = 0.02f;
    unsigned refine_count = 0;                 // r: k_sweep launches with refinement since gpm_init / gpm_init_planes / gpm_set_rng
};

namespace {

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// 2-D TMA descriptor (cuTensorMapEncodeTiled, fetched through the runtime so that the library links only cudart) of the
// padded reference image: box = one tile's window, tile_stride x tile_w texels (float4 images: 4 floats per texel).
int ensure_tensor_map(gpm_ctx* c, const KParams& P)
{
    const int box = c->prm.box_hsize;
    if (c->tmap_box == box) return GPM_OK;
    typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    static EncodeTiled encode = nullptr;
    if (!encode) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        CU(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        if (!fn || qres != cudaDriverEntryPointSuccess) return fail(GPM_E_CUDA, "cuTensorMapEncodeTiled is not available in this driver");
        encode = (EncodeTiled)fn;
    }
    const int comps = P.color ? 4 : 1;
    const cuuint64_t gdim[2] = {(cuuint64_t)c->refpitch * comps, (cuuint64_t)c->refrows};
    const cuuint64_t gstride[1] = {(cuuint64_t)c->refpitch * comps * sizeof(float)};
    const cuuint32_t bdim[2] = {(cuuint32_t)(P.tile_stride * comps), (cuuint32_t)P.tile_w};
    const cuuint32_t estr[2] = {1, 1};
    if (bdim[0] > 256 || bdim[1] > 256) return fail(GPM_E_ARG, "window too large for one TMA box");
    const CUresult r = encode(&c->tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, c->refpad, gdim, gstride, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(GPM_E_CUDA, "cuTensorMapEncodeTiled failed: " + std::to_string((int)r));
    c->tmap_box = box;
    return GPM_OK;
}

const int PROV_KEEP = -1;

// The stored state's tags: prov[] (which rounding variant produced cost[]; PROV_KEEP leaves it alone) and the memo's
// validity bits.  Every transition that makes them stale goes through here.
int reset_state_tags(gpm_ctx* c, int prov)
{
    const size_t n = (size_t)c->W * c->H;
    if (prov != PROV_KEEP) CU(cudaMemsetAsync(c->prov, prov, n, c->stream));
    CU(cudaMemsetAsync(c->memo_mask, 0, n * sizeof(unsigned), c->stream));
    return GPM_OK;
}

// the geometric-consistency mode's precondition at weight `weight`: a depth map for every used source view
int check_depth_maps(const gpm_ctx* c, float weight)
{
    if (weight <= 0.f) return GPM_OK;
    for (int v = 0; v < c->V; v++)
        if (!c->have_depth[v]) return fail(GPM_E_STATE, "geometric-consistency mode: source view " + std::to_string(v) + " has no depth map (gpm_set_view_depth)");
    return GPM_OK;
}

bool ncc_on(const gpm_ctx* c) { return c->photo == GPM_PHOTO_NCC; }
bool jvs_on(const gpm_ctx* c) { return c->vsel.kind == GPM_VSEL_JOINT; }

// The context's sweep mode.  Every setter of one of its fields refuses a change that mode_conflict() would not pass, so it
// always names a mode with kernels.
Mode ctx_mode(const gpm_ctx* c)
{
    return Mode{c->color == 1, c->opt_neighbours == 20, c->geo_weight > 0.f, ncc_on(c), c->propagation == GPM_PROP_ADAPTIVE, jvs_on(c),
                c->prior_weight > 0.f, c->geo_weight > 0.f && c->geo_mask_set, c->refine_kind == GPM_REFINE_ACMH};
}

// the index of the context's mode in the tables of k_cost_eval and k_shard_stage, which do not read refine_acmh
int eval_bits(const gpm_ctx* c) { return ctx_mode(c).bits() & (GPM_EVAL_MODES - 1); }

const char* conflict_text(ModeConflict k)
{
    switch (k) {
    case ModeConflict::fused: return "the geometric-consistency mode, the NCC cost, adaptive sampling, joint view selection and the planar prior support the 8-neighbour sweep only (option neighbours = 8)";
    case ModeConflict::jvs_needs_ncc_grey: return "joint view selection is built for the NCC cost (GPM_PHOTO_NCC) on grey images";
    case ModeConflict::ncc_colour: return "the NCC photometric cost supports grey images only";
    case ModeConflict::prior: return "the planar prior supports grey images without joint view selection";
    case ModeConflict::geomask: return "the geometric term's mask and the planar prior exclude each other";
    case ModeConflict::refine_fused: return "ACMH's refinement supports the 8-neighbour sweep only (option neighbours = 8)";
    default: return nullptr;
    }
}

// Refuses the call `fn` if setting `field` of the context's mode to `on` gives a mode mode_conflict() does not pass.  Such a
// refusal is GPM_E_ARG, but GPM_E_STATE for a colour image upload while only the NCC cost is on (include/gipuma_b200.h).
int refuse_change(const gpm_ctx* c, const char* fn, bool Mode::*field, bool on)
{
    Mode m = ctx_mode(c);
    m.*field = on;
    const ModeConflict k = mode_conflict(m);
    if (k == ModeConflict::none) return GPM_OK;
    return fail(field == &Mode::color && k == ModeConflict::ncc_colour ? GPM_E_STATE : GPM_E_ARG, std::string(fn) + ": " + conflict_text(k));
}

// per-warp floats of the JVS kernel variant the context launches (0 without view selection)
int jvs_extra(const gpm_ctx* c) { return jvs_on(c) ? jvs_floats(c->V, c->geo_weight > 0.f) : 0; }

// k_sweep's per-warp floats beyond the common scratch, and its shared memory per block: the JVS rows, or the plane-major
// pass's scratch and candidate cost table in the mode that shares propagation samples (shares_samples)
int sweep_extra(const gpm_ctx* c, const KParams& P) { return shares_samples(ctx_mode(c)) ? share_extra_floats(P) : jvs_extra(c); }
size_t sweep_smem_bytes(const gpm_ctx* c, const KParams& P)
{
    return block_smem_bytes(P, ncc_on(c), sweep_extra(c, P)) + (shares_samples(ctx_mode(c)) ? GPM_SHARE_TABLE_BYTES : 0);
}

// selected-views masks back to "none selected" (gpm_init, gpm_set_state, a switch to JOINT)
int clear_vsel_masks(gpm_ctx* c)
{
    if (c->vsel_mask) CU(cudaMemsetAsync(c->vsel_mask, 0, (size_t)c->W * c->H * sizeof(unsigned long long), c->stream));
    return GPM_OK;
}

// provenance of costs from an initialisation evaluation (gpm_init, or a trusted gpm_set_state)
int init_prov(const gpm_ctx* c) { return ncc_on(c) ? GPM_PROV_NCC : c->color == 1 ? 3 : 0; }

int build_kparams(gpm_ctx* c, bool init_phase, KParams& P, bool eval_call = false)
{
    if (!c->have_params) return fail(GPM_E_STATE, "gpm_set_params has not been called");
    if (!c->have_ref) return fail(GPM_E_STATE, "gpm_set_reference has not been called");
    if (c->V < 1) return fail(GPM_E_STATE, "no source views (gpm_set_num_views)");
    for (int v = 0; v < c->V; v++)
        if (!c->have_view[v]) return fail(GPM_E_STATE, "source view " + std::to_string(v) + " has not been set");
    if (const int rc = check_depth_maps(c, c->geo_weight)) return rc;
    if (c->inputs_dirty || c->memo_dirty) {     // one clearing for a whole scene upload instead of two memsets per setter
        const int rc = reset_state_tags(c, c->inputs_dirty ? GPM_PROV_UNKNOWN : PROV_KEEP);
        if (rc) return rc;
        c->inputs_dirty = c->memo_dirty = false;
    }
    const gpm_params& p = c->prm;
    memset(&P, 0, sizeof(P));
    P.W = c->W;  P.H = c->H;  P.V = c->V;
    const int box = p.box_hsize;
    P.rad = init_phase ? box / 2 : (box - 1) / 2;          // gipuma.cu:1012 vs :1474
    P.nside = P.rad + 1;                                    // i = -rad, -rad+2, ... <= rad
    P.ns = P.nside * P.nside;
    P.ns_pad = (P.ns + 3) & ~3;
    P.halo = (box + 1) / 2;                                 // gipuma.cu:1844-1847
    P.tile_w = GPM_TILE + 2 * P.halo;
    P.tile_stride = (P.tile_w + 15) & ~15;                  // 48 or 64 texels per staged row
    // a TMA box must start on a 16-byte boundary of the image (boxes starting at byte offsets 12, 28, 40, 44 have
    // faulted although cuTensorMapEncodeTiled accepts the descriptor): tile_x0 + GPM_APRON = 32 bx + 16 - halo, so the box starts (16 - halo) mod 4 texels early
    P.tile_xo = (c->color == 1) ? 0 : ((GPM_APRON - P.halo) & 3);
    // rounds of 32 consecutive samples (one per lane); the remainder forms a last, shorter round whose (view, sample) pairs
    // share an instruction across several views
    {
        int r = 0;
        for (int e = 32; e < P.ns && r < 15; e += 32) P.round_end[r++] = (unsigned char)e;
        P.round_end[r++] = (unsigned char)P.ns;
        P.nrounds = r;
    }
    // lane -> sample table of each round.  The texture unit filters a warp's fetches one hardware quad (lanes 4q..4q+3) at a
    // time and is fastest when a quad's four footprints form a compact 2x2 block (tools/texbench.cu): with
    // "quadperm" the samples of a round are dealt to the lanes as 2x2 blocks (x offset i, i+2; y offset j, j+2) where the
    // round contains them, leftovers in window order.  Only WHICH lane evaluates a sample changes; the per-view FMA chain
    // still consumes the dissimilarities in the reference's order.
    P.quadperm = c->opt_quadperm;
    {
        int s0 = 0;
        for (int r = 0; r < P.nrounds; r++) {
            const int s1 = P.round_end[r], len = s1 - s0;
            unsigned char* row = P.perm[r];
            for (int l = 0; l < 32; l++) row[l] = (unsigned char)(l < len ? l : 0);
            if (P.quadperm && len >= 4 && len <= 32) {
                bool used[32] = {false};
                int n = 0;
                for (int k = 0; k < len; k++) {
                    if (used[k]) continue;
                    const int s = s0 + k, jj = s % P.nside;
                    const int kr = k + P.nside, kd = k + 1, kx = k + P.nside + 1;
                    if (jj + 1 < P.nside && kx < len && !used[kr] && !used[kd] && !used[kx]) {
                        row[n++] = (unsigned char)k;  row[n++] = (unsigned char)kr;  row[n++] = (unsigned char)kd;  row[n++] = (unsigned char)kx;
                        used[k] = used[kr] = used[kd] = used[kx] = true;
                    }
                }
                for (int k = 0; k < len; k++) if (!used[k]) row[n++] = (unsigned char)k;
            }
            s0 = s1;
        }
    }
    P.tau_color = p.tau_color;  P.tau_gradient = p.tau_gradient;  P.alpha = p.alpha;  P.gamma = p.gamma;
    P.min_disp = p.min_disparity;  P.max_disp = p.max_disparity;
    P.n_best = p.n_best;  P.cost_comb = p.cost_comb;  P.good_factor = p.good_factor;
    P.prune = c->opt_prune;
    // The lower bound counts a view as valid from its PARTIAL cost; a view whose final cost reaches MAXCOST (then excluded,
    // gipuma.cu:771-774) would make the bound exceed the final value.  Unreachable while ns * max dissimilarity < MAXCOST.
    // The geometric term adds at most weight * max_err to a view's final cost (0 outside that mode).
    // The planar prior adds less than its weight (DESIGN.md §18).
    if ((float)P.ns * ((1.0f - p.alpha) * p.tau_color + p.alpha * p.tau_gradient) + c->geo_weight * c->geo_max_err + c->prior_weight >= GPM_MAXCOST) P.prune = 0;
    if (ncc_on(c)) P.prune = 0;                             // partial NCC sums bound nothing (DESIGN.md §15)
    P.dedupe_self = c->opt_dedupe ? 1 : 0;
    // rounding variant of k_cost_eval: at initialisation the reference's binary is y-first for float, x-first for float4;
    // gpm_cost_eval defaults to the variant of the propagation kernels (x-first for float, y-first for float4)
    // For float4 the initialisation kernel additionally folds the other gradient term into the FMA (grad_variant).
    // Option cost_variant: bit 0 = x-term first, bit 1 = gradient folding (float4 only).
    const int cv = eval_call ? c->opt_cost_variant : -1;          // the option only steers gpm_cost_eval
    P.cost_rt = 0;
    if (init_phase) { P.cost_variant = c->color == 1 ? 1 : 0;  P.grad_variant = c->color == 1 ? 1 : 0; }
    else if (cv >= 0) { P.cost_variant = cv & 1;  P.grad_variant = (c->color == 1) ? ((cv >> 1) & 1) : 0;  P.cost_rt = c->color == 1 ? cv : (cv & ~2); }
    else { P.cost_variant = c->color == 1 ? 0 : 1;  P.grad_variant = 0; }
    P.ncand = c->opt_neighbours == 20 ? 20 : 8;
    // call-site variants of the fused kernels, read off the reference build (tools/fused_probe.py)
    {
        static const unsigned char kSitesFloat[21] = GPM_FUSED_SITES_FLOAT, kSitesFloat4[21] = GPM_FUSED_SITES_FLOAT4;
        for (int k = 0; k < 21; k++)
            P.site[k] = c->opt_site[k] >= 0 ? (unsigned char)c->opt_site[k] : (c->color == 1 ? kSitesFloat4[k] : kSitesFloat[k]);
    }
    P.color = c->color == 1 ? 1 : 0;
    P.memo = c->opt_memo;
    P.dedupe_cand = c->opt_dedupe ? 1 : 0;
    P.rng_mode = c->rng_mode;
    P.ref = c->ref;
    P.ref.depthMin = p.depthMin;  P.ref.depthMax = p.depthMax;
    // warps per block: as many as fit (<= 16).  The kernels use 128 registers per thread, so one 16-warp block fills an SM
    // anyway; shared memory may therefore be spent up to the per-block opt-in limit.
    const size_t per_warp = (size_t)warp_scratch_floats(P.ns_pad, P.V, P.color, ncc_on(c), sweep_extra(c, P)) * sizeof(float);
    const size_t fixed = ((size_t)fixed_smem_floats(P) + 4) * sizeof(float) + (shares_samples(ctx_mode(c)) ? GPM_SHARE_TABLE_BYTES : 0);
    int nw = GPM_LB_THREADS / 32;
    const size_t budget = (size_t)c->smem_optin > 16 * 1024 ? (size_t)c->smem_optin - 8 * 1024 : 40 * 1024;
    while (nw > 2 && fixed + nw * per_warp > budget) nw--;
    if (c->opt_nwarps > 0) nw = c->opt_nwarps;
    if (nw > GPM_LB_THREADS / 32) nw = GPM_LB_THREADS / 32;
    P.nwarps = nw;
    if (sweep_smem_bytes(c, P) > (size_t)c->smem_optin)
        return fail(GPM_E_ARG, "configuration needs more shared memory per block than the device offers");
    return ensure_tensor_map(c, P);
}

// identities 1 .. W*H belong to the pixels' initial planes; fresh ones start above
int reset_next_id(gpm_ctx* c)
{
    const unsigned first = (unsigned)((size_t)c->W * c->H) + 1u;
    CU(cudaMemcpyAsync(c->next_id, &first, sizeof(first), cudaMemcpyHostToDevice, c->stream));
    return GPM_OK;
}

int fill_ids(gpm_ctx* c)
{
    const unsigned n = (unsigned)((size_t)c->W * c->H);
    k_fill_ids<<<(n + 255) / 256, 256, 0, c->stream>>>(c->pid, n);
    CU(cudaGetLastError());
    return reset_next_id(c);
}

int sync_cams(gpm_ctx* c)
{
    if (!c->cams_dirty) return GPM_OK;
    CU(cudaMemcpyAsync(c->d_cams, c->h_cams.data(), sizeof(ViewCam) * c->maxV, cudaMemcpyHostToDevice, c->stream));
    if (c->geo_kinv) CU(cudaMemcpyAsync(c->geo_kinv, c->h_kinv.data(), sizeof(float) * 9 * c->maxV, cudaMemcpyHostToDevice, c->stream));
    c->cams_dirty = false;
    return GPM_OK;
}

// one block per 32 x 32 tile; at least ~8 waves of blocks over the SMs: gridDim.z splits each tile's pixel list into up
// to 8 slices for small images
dim3 tile_grid(const gpm_ctx* c)
{
    dim3 grid((c->W + GPM_TILE - 1) / GPM_TILE, (c->H + GPM_TILE - 1) / GPM_TILE);
    int split = 1;
    while (split < 8 && (long long)grid.x * grid.y * split < 8LL * c->num_sms) split *= 2;
    grid.z = split;
    return grid;
}

GeoParams geo_params(const gpm_ctx* c)
{
    GeoParams G{};
    G.depth = c->geo_depth;  G.kinv = c->geo_kinv;
    memcpy(G.Kref, c->ref_K, sizeof(G.Kref));
    G.weight = c->geo_weight;  G.max_err = c->geo_max_err;
    G.min_std = c->ncc_min_std;
    return G;
}

// JVS launches' parameters at the context's iteration count t (DESIGN.md §17); thresholds in double, rounded once
JvsParams jvs_params(const gpm_ctx* c)
{
    JvsParams J{};
    if (!jvs_on(c)) return J;
    const gpm_view_sel& v = c->vsel;
    const double t = (double)c->vsel_t, beta = (double)v.beta;
    J.mask = c->vsel_mask;
    J.tau_t = (float)((double)v.tau_init * std::exp(-t * t / (double)v.alpha));
    J.kb = (float)(-1.4426950408889634 / (2.0 * beta * beta));
    J.tau_bad = v.tau_bad;  J.w_keep = v.w_keep;  J.n_good = v.n_good;  J.n_bad = v.n_bad;
    return J;
}

// the planar prior's parameters (DESIGN.md §18): 1 - cos(sigma_n) in double, rounded once
PriorParams prior_params(const gpm_ctx* c)
{
    PriorParams R{};
    if (ctx_mode(c).geomask) R.geo_mask = c->geo_mask;       // the masked variants read the mask in the map's place
    else R.map = c->prior_map;
    R.weight = c->prior_weight;
    R.depth_sigma = c->prior_depth_sigma;
    R.normal_scale = (float)(1.0 - std::cos((double)c->prior_normal_deg * 3.14159265358979323846 / 180.0));
    return R;
}

// Kernel tables: entry Mode::bits() is the family's kernel for that mode, nullptr (refused, never launched) where it has
// none.  k_sweep and k_cost_eval exist for the modes mode_conflict() passes (k_cost_eval reads neither the propagation, the
// view selection nor the fused sweep), k_shard_stage for those shard_supports() passes.
template <class Entry, int... B>
auto make_table(Entry entry, std::integer_sequence<int, B...>) { return std::array{entry(std::integral_constant<int, B>{})...}; }

const auto kSweep = make_table([](auto b) -> decltype(&k_sweep<false, false>) {
    constexpr Mode m = Mode::of(decltype(b)::value);
    if constexpr (mode_conflict(m) == ModeConflict::none)
        return k_sweep<m.color, m.fused, m.geo, m.ncc, m.adaptive, m.jvs, m.prior, m.geomask, m.refine_acmh>;
    else return nullptr;
}, std::make_integer_sequence<int, GPM_MODES>{});

const auto kCostEval = make_table([](auto b) -> decltype(&k_cost_eval<false>) {
    constexpr Mode m = Mode::of(decltype(b)::value);
    if constexpr (mode_conflict(m) == ModeConflict::none) return k_cost_eval<m.color, m.geo, m.ncc, m.prior, m.geomask>; else return nullptr;
}, std::make_integer_sequence<int, GPM_EVAL_MODES>{});

const auto kShardStage = make_table([](auto b) -> decltype(&k_shard_stage<false>) {
    constexpr Mode m = Mode::of(decltype(b)::value);
    if constexpr (shard_supports(m)) return k_shard_stage<m.color, m.adaptive>; else return nullptr;
}, std::make_integer_sequence<int, GPM_EVAL_MODES>{});

int launch_colour(gpm_ctx* c, const KParams& P, int colour, int mask)
{
    const auto kern = kSweep[ctx_mode(c).bits()];
    if (!kern) return fail(GPM_E_STATE, "k_sweep has no kernel for this context's mode");
    kern<<<tile_grid(c), P.nwarps * 32, sweep_smem_bytes(c, P), c->stream>>>(P, c->tmap, c->d_cams, c->srcTex, c->planes,
        c->cost, c->rng, c->prov, Memo{c->pid, c->seen, c->refseen, c->memo_mask, c->next_id}, colour, mask, c->d_stats, geo_params(c),
        jvs_params(c), prior_params(c), AcmhRefine{(unsigned)c->seed ^ (unsigned)(c->seed >> 32), c->refine_count, c->refine_eps});
    c->launches++;
    if (mask & 4) c->refine_count++;
    CU(cudaGetLastError());
    return GPM_OK;
}

// cost of `planes` at every pixel into `cost` (k_cost_eval: one block per tile, no slices)
int launch_cost_eval(gpm_ctx* c, const KParams& P, const float4* planes, float* cost)
{
    const auto kern = kCostEval[eval_bits(c)];
    if (!kern) return fail(GPM_E_STATE, "k_cost_eval has no kernel for this context's mode");
    dim3 grid((P.W + GPM_TILE - 1) / GPM_TILE, (P.H + GPM_TILE - 1) / GPM_TILE);
    kern<<<grid, P.nwarps * 32, block_smem_bytes(P, ncc_on(c)), c->stream>>>(P, c->tmap, c->d_cams, c->srcTex, planes, cost, nullptr, geo_params(c),
                                                                            prior_params(c));
    c->launches++;
    CU(cudaGetLastError());
    return GPM_OK;
}

// random planes (gipuma.cu:1870-1875) and their identities; the XORWOW states are kept in GPM_RNG_STATEFUL mode.  ACMH's
// refinement counts its launches from here (§23).
int init_planes(gpm_ctx* c, const KParams& P)
{
    c->refine_count = 0;
    dim3 b(16, 16), gr((c->W + 15) / 16, (c->H + 15) / 16);
    k_init_planes<<<gr, b, 0, c->stream>>>(P, c->seed, c->planes, c->rng_mode == GPM_RNG_STATEFUL ? c->rng : nullptr, c->pid);
    c->launches++;
    CU(cudaGetLastError());
    return reset_next_id(c);
}

// source views: layered array, Linear filter, the reference's addressing (Wrap + unnormalised, main.cpp:642-648), element reads
cudaError_t make_layered_texture(cudaArray_t arr, cudaTextureObject_t* tex)
{
    cudaResourceDesc res;  memset(&res, 0, sizeof(res));
    res.resType = cudaResourceTypeArray;  res.res.array.array = arr;
    cudaTextureDesc td;  memset(&td, 0, sizeof(td));
    td.addressMode[0] = cudaAddressModeWrap;  td.addressMode[1] = cudaAddressModeWrap;   // main.cpp:644-645
    td.addressMode[2] = cudaAddressModeClamp;
    td.filterMode = cudaFilterModeLinear;  td.readMode = cudaReadModeElementType;  td.normalizedCoords = 0;
    return cudaCreateTextureObject(tex, &res, &td, NULL);
}

void set_view_camera(gpm_ctx* c, int v, const gpm_camera* cam)
{
    ViewCam& vc = c->h_cams[v];
    memcpy(vc.K, cam->K, sizeof(vc.K));
    memcpy(vc.R, cam->R, sizeof(vc.R));
    memcpy(vc.t, cam->t, sizeof(vc.t));
    memcpy(&c->h_kinv[9 * (size_t)v], cam->K_inv, 9 * sizeof(float));
    c->cams_dirty = true;
    c->have_view[v] = 1;
    c->inputs_dirty = true;
}

// The first image upload fixes the context's image type (0 float, 1 float4) and allocates the image storage for that type
// only.  A failed allocation is retried by the next upload.
int ensure_color(gpm_ctx* c, int want)
{
    if (c->color == -1) c->color = want;
    if (c->color != want) return fail(GPM_E_STATE, "a context holds either float or float4 images, not both");
    const size_t comps = want ? 4 : 1, n = (size_t)c->W * c->H;
    const cudaChannelFormatDesc desc = cudaCreateChannelDesc(32, 0, 0, 0, cudaChannelFormatKindFloat);
    if (!c->srcArr) CU(cudaMalloc3DArray(&c->srcArr, &desc, make_cudaExtent(c->W, c->H, (want ? 3 : 1) * (size_t)c->maxV), cudaArrayLayered));
    if (!c->srcTex) CU(make_layered_texture(c->srcArr, &c->srcTex));
    if (!c->refpad) CU(cudaMalloc(&c->refpad, (size_t)c->refpitch * c->refrows * comps * sizeof(float)));
    if (!c->staging) CU(cudaMalloc(&c->staging, n * comps * sizeof(float)));
    if (want && !c->planar) CU(cudaMalloc(&c->planar, 3 * n * sizeof(float)));
    return GPM_OK;
}

// row pitch, in texels of type T, of a caller's image of W texels per row (pitch_bytes 0: rows are packed)
template <typename T>
int image_pitch(const gpm_ctx* c, size_t pitch_bytes, size_t* pitch_elems)
{
    if (pitch_bytes == 0) pitch_bytes = (size_t)c->W * sizeof(T);
    if (pitch_bytes % sizeof(T))
        return fail(GPM_E_ARG, sizeof(T) == sizeof(float) ? "pitch_bytes must be a multiple of 4" : "pitch_bytes must be a multiple of 16 for float4 images");
    *pitch_elems = pitch_bytes / sizeof(T);
    return GPM_OK;
}

// the caller's image in device memory: a device image in place, a host image copied into `staging`
template <typename T>
int upload_image(gpm_ctx* c, const float* img, size_t pitch_bytes, int on_device, const T** dev_img, size_t* dev_pitch_elems)
{
    const int rc = image_pitch<T>(c, pitch_bytes, dev_pitch_elems);
    if (rc) return rc;
    *dev_img = reinterpret_cast<const T*>(img);
    if (on_device) return GPM_OK;
    CU(cudaMemcpy2DAsync(c->staging, (size_t)c->W * sizeof(T), img, *dev_pitch_elems * sizeof(T), (size_t)c->W * sizeof(T), c->H,
                         cudaMemcpyHostToDevice, c->stream));
    *dev_img = reinterpret_cast<const T*>(c->staging);
    *dev_pitch_elems = c->W;
    return GPM_OK;
}

}  // namespace

static void set_ref_camera(gpm_ctx* c, const gpm_camera* cam)
{
    RefCam& r = c->ref;
    memcpy(r.K_inv, cam->K_inv, sizeof(r.K_inv));
    memcpy(r.M_inv, cam->M_inv, sizeof(r.M_inv));
    memcpy(r.R_orig_inv, cam->R_orig_inv, sizeof(r.R_orig_inv));
    memcpy(r.P34, cam->P_col34, sizeof(r.P34));
    memcpy(r.C, cam->C, sizeof(r.C));
    r.fx = cam->fx;  r.alpha = cam->alpha;  r.K2 = cam->K[2];  r.K5 = cam->K[5];
    r.f = cam->f;  r.f_cam = cam->f;  r.baseline = cam->baseline;
    memcpy(c->ref_K, cam->K, sizeof(c->ref_K));
    c->have_ref = true;
}

extern "C" const char* gpm_last_error(void) { return g_err.c_str(); }
extern "C" const char* gpm_version(void) { return "gipuma_b200 0.1 (sm_90a)"; }

extern "C" int gpm_create(gpm_ctx** out, int device, int width, int height, int max_views)
{
    if (!out || width < 8 || height < 8 || max_views < 1 || max_views > GPM_MAX_VIEWS)
        return fail(GPM_E_ARG, "gpm_create: bad arguments (max_views must be 1.." + std::to_string(GPM_MAX_VIEWS) + ")");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev < 1)
        return fail(GPM_E_CUDA, std::string("no CUDA device: ") + cudaGetErrorString(e) + " (gipuma_b200 has no CPU fallback)");
    if (device < 0 || device >= ndev) return fail(GPM_E_ARG, "gpm_create: no such device");
    DeviceGuard g(device);
    gpm_ctx* c = new gpm_ctx;
    for (int& v : c->opt_site) v = -1;
    c->device = device;  c->W = width;  c->H = height;  c->maxV = max_views;
    c->have_view.assign(max_views, 0);
    c->h_cams.assign(max_views, ViewCam{});
    c->have_depth.assign(max_views, 0);
    c->h_kinv.assign((size_t)max_views * 9, 0.f);
    const size_t n = (size_t)width * height;
    // the staged window of the last tile row / column reaches roundup(size, 32) + halo + GPM_APRON (+ 3 texels of TMA row padding)
    c->refpitch = (((width + 31) & ~31) + 2 * GPM_APRON + 4 + 31) & ~31;
    c->refrows = ((height + 31) & ~31) + 2 * GPM_APRON;
    cudaError_t err = cudaSuccess;
    auto ok = [&](cudaError_t r) { if (err == cudaSuccess && r != cudaSuccess) err = r; return r == cudaSuccess; };
    ok(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    ok(cudaEventCreate(&c->ev0));
    ok(cudaEventCreate(&c->ev1));
    ok(cudaMalloc(&c->planes, n * sizeof(float4)));
    ok(cudaMalloc(&c->cost, n * sizeof(float)));
    ok(cudaMalloc(&c->prov, n));
    ok(cudaMalloc(&c->seen, n * 8 * sizeof(unsigned)));
    ok(cudaMalloc(&c->refseen, n * sizeof(unsigned)));
    ok(cudaMalloc(&c->pid, n * sizeof(unsigned)));
    ok(cudaMalloc(&c->next_id, sizeof(unsigned)));
    ok(cudaMalloc(&c->memo_mask, n * sizeof(unsigned)));
    ok(cudaMalloc(&c->d_cams, sizeof(ViewCam) * max_views));
    ok(cudaMalloc(&c->d_stats, 8 * sizeof(unsigned long long)));
    if (err == cudaSuccess) {
        ok(cudaMemsetAsync(c->planes, 0, n * sizeof(float4), c->stream));      // LineState::resize zeroes (linestate.h:19-24)
        ok(cudaMemsetAsync(c->cost, 0, n * sizeof(float), c->stream));
        ok(cudaMemsetAsync(c->d_stats, 0, 8 * sizeof(unsigned long long), c->stream));
        if (reset_state_tags(c, GPM_PROV_UNKNOWN) != GPM_OK || fill_ids(c) != GPM_OK) err = cudaErrorUnknown;
    }
    if (err == cudaSuccess) {
        ok(cudaDeviceGetAttribute(&c->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        ok(cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device));
        auto optin = [&](const auto& table) {
            for (const auto kern : table)
                if (kern) ok(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, c->smem_optin));
        };
        optin(kSweep);  optin(kCostEval);  optin(kShardStage);
    }
    if (err != cudaSuccess) {
        std::string m = std::string("gpm_create: ") + cudaGetErrorString(err);
        gpm_destroy(c);
        return fail(GPM_E_CUDA, m);
    }
    *out = c;
    return GPM_OK;
}

static void gpm_shard_comm_destroy_(gpm_ctx* c);

extern "C" void gpm_destroy(gpm_ctx* c)
{
    if (!c) return;
    DeviceGuard g(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->comm && c->comm_owned) gpm_shard_comm_destroy_(c);
    if (c->srcTex) cudaDestroyTextureObject(c->srcTex);
    if (c->srcArr) cudaFreeArray(c->srcArr);
    cudaFree(c->planar);
    cudaFree(c->planes);  cudaFree(c->cost);  cudaFree(c->prov);  cudaFree(c->seen);  cudaFree(c->refseen);  cudaFree(c->pid);  cudaFree(c->next_id);  cudaFree(c->memo_mask);  cudaFree(c->rng);  cudaFree(c->dispbuf);  cudaFree(c->candbuf);  cudaFree(c->canddepth);  cudaFree(c->sflags);  cudaFree(c->xchg);  cudaFree(c->gath);  cudaFree(c->refpad);  cudaFree(c->staging);  cudaFree(c->geo_depth);  cudaFree(c->geo_kinv);  cudaFree(c->vsel_mask);
    cudaFree(c->prior_map);  cudaFree(c->prior_cost);  cudaFree(c->geo_mask);
    cudaFree(c->d_cams);  cudaFree(c->d_stats);
    if (c->ev0) cudaEventDestroy(c->ev0);
    if (c->ev1) cudaEventDestroy(c->ev1);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" int gpm_set_params(gpm_ctx* c, const gpm_params* p)
{
    if (!c || !p) return fail(GPM_E_ARG, "gpm_set_params: null argument");
    if (p->box_hsize != p->box_vsize)
        return fail(GPM_E_ARG, "box_hsize != box_vsize: the reference's tile loader (gipuma.cu:1517) is only defined for square windows");
    if (p->box_hsize < 3 || p->box_hsize > GPM_MAX_BOX || !(p->box_hsize & 1))
        return fail(GPM_E_ARG, "box size must be odd, 3.." + std::to_string(GPM_MAX_BOX));
    if (p->cost_comb < 0 || p->cost_comb > 3) return fail(GPM_E_ARG, "cost_comb must be 0..3");
    if (p->iterations < 0) return fail(GPM_E_ARG, "iterations must be >= 0");
    if (!prior_bound_ok(*p, ncc_on(c), c->geo_weight, c->geo_max_err, c->prior_weight))
        return fail(GPM_E_ARG, "gpm_set_params: with the planar prior's weight a valid cost could reach MAXCOST");
    c->prm = *p;
    c->have_params = true;
    c->inputs_dirty = true;                          // the cost function depends on the parameters: stored costs / memo are stale
    return GPM_OK;
}

extern "C" int gpm_set_num_views(gpm_ctx* c, int n)
{
    if (!c || n < 1 || n > c->maxV) return fail(GPM_E_ARG, "gpm_set_num_views: out of range");
    if (n != c->V) c->inputs_dirty = true;           // the cost function changes with the view count: stored costs / memo are stale
    c->V = n;
    return GPM_OK;
}

extern "C" int gpm_set_rng(gpm_ctx* c, unsigned long long seed, int mode)
{
    if (!c || (mode != GPM_RNG_REFERENCE && mode != GPM_RNG_STATEFUL)) return fail(GPM_E_ARG, "gpm_set_rng: bad mode");
    DeviceGuard g(c->device);
    c->seed = seed;
    c->rng_mode = mode;
    c->refine_count = 0;
    c->memo_dirty = true;                            // the refinement memo assumes the random stream it was built under
    if (mode == GPM_RNG_STATEFUL && !c->rng) {
        CU(cudaMalloc(&c->rng, (size_t)c->W * c->H * 6 * sizeof(unsigned)));
        CU(cudaMemsetAsync(c->rng, 0, (size_t)c->W * c->H * 6 * sizeof(unsigned), c->stream));
    }
    return GPM_OK;
}

// Image uploads, T = float (grey) or float4 (colour: the reference's -color_processing path, main.cpp:560-605).  Each
// returns after a stream synchronisation: the caller may reuse its buffer.
template <typename T>
static int set_reference(const char* fn, gpm_ctx* c, const float* img, size_t pitch_bytes, int on_device, const gpm_camera* cam)
{
    if (!c || !img || !cam) return fail(GPM_E_ARG, std::string(fn) + ": null argument");
    if (const int rc = refuse_change(c, fn, &Mode::color, sizeof(T) == sizeof(float4))) return rc;
    DeviceGuard g(c->device);
    int rc = ensure_color(c, sizeof(T) == sizeof(float4));
    if (rc) return rc;
    const T* d = nullptr;
    size_t pe = 0;
    rc = upload_image<T>(c, img, pitch_bytes, on_device, &d, &pe);
    if (rc) return rc;
    dim3 b(32, 8), gr((c->refpitch + 31) / 32, (c->refrows + 7) / 8);
    k_pad_reference<T><<<gr, b, 0, c->stream>>>(d, pe, c->W, c->H, reinterpret_cast<T*>(c->refpad), c->refpitch, c->refrows);
    CU(cudaGetLastError());
    set_ref_camera(c, cam);
    c->inputs_dirty = true;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

template <typename T>
static int set_view(const char* fn, gpm_ctx* c, int v, const float* img, size_t pitch_bytes, int on_device, const gpm_camera* cam)
{
    if (!c || !img || !cam) return fail(GPM_E_ARG, std::string(fn) + ": null argument");
    if (v < 0 || v >= c->maxV) return fail(GPM_E_ARG, std::string(fn) + ": view index out of range");
    constexpr bool color = sizeof(T) == sizeof(float4);
    if (const int rc = refuse_change(c, fn, &Mode::color, color)) return rc;
    DeviceGuard g(c->device);
    int rc = ensure_color(c, color);
    if (rc) return rc;
    cudaMemcpy3DParms m;  memset(&m, 0, sizeof(m));
    m.dstArray = c->srcArr;
    if (!color) {                   // the image goes straight into its layer of the array: no staging copy
        size_t pe = 0;
        rc = image_pitch<T>(c, pitch_bytes, &pe);
        if (rc) return rc;
        m.srcPtr = make_cudaPitchedPtr(const_cast<float*>(img), pe * sizeof(T), c->W, c->H);
        m.dstPos = make_cudaPos(0, 0, v);
        m.extent = make_cudaExtent(c->W, c->H, 1);
        m.kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    } else {                        // three channel planes, layers 3v .. 3v + 2
        const T* d = nullptr;
        size_t pe = 0;
        rc = upload_image<T>(c, img, pitch_bytes, on_device, &d, &pe);
        if (rc) return rc;
        dim3 b(32, 8), gr((c->W + 31) / 32, (c->H + 7) / 8);
        k_split_channels<<<gr, b, 0, c->stream>>>(reinterpret_cast<const float4*>(d), pe, c->W, c->H, c->planar);
        CU(cudaGetLastError());
        m.srcPtr = make_cudaPitchedPtr(c->planar, c->W * sizeof(float), c->W, c->H);
        m.dstPos = make_cudaPos(0, 0, 3 * (size_t)v);
        m.extent = make_cudaExtent(c->W, c->H, 3);
        m.kind = cudaMemcpyDeviceToDevice;
    }
    CU(cudaMemcpy3DAsync(&m, c->stream));
    set_view_camera(c, v, cam);
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_set_reference(gpm_ctx* c, const float* img, size_t pitch_bytes, int on_device, const gpm_camera* cam)
{
    return set_reference<float>("gpm_set_reference", c, img, pitch_bytes, on_device, cam);
}

extern "C" int gpm_set_reference_color(gpm_ctx* c, const float* rgba, size_t pitch_bytes, int on_device, const gpm_camera* cam)
{
    return set_reference<float4>("gpm_set_reference_color", c, rgba, pitch_bytes, on_device, cam);
}

extern "C" int gpm_set_view(gpm_ctx* c, int v, const float* img, size_t pitch_bytes, int on_device, const gpm_camera* cam)
{
    return set_view<float>("gpm_set_view", c, v, img, pitch_bytes, on_device, cam);
}

extern "C" int gpm_set_view_color(gpm_ctx* c, int v, const float* rgba, size_t pitch_bytes, int on_device, const gpm_camera* cam)
{
    return set_view<float4>("gpm_set_view_color", c, v, rgba, pitch_bytes, on_device, cam);
}

extern "C" int gpm_set_view_depth(gpm_ctx* c, int v, const float* depth, size_t pitch_bytes, int on_device)
{
    if (!c || !depth) return fail(GPM_E_ARG, "gpm_set_view_depth: null argument");
    if (v < 0 || v >= c->maxV) return fail(GPM_E_ARG, "gpm_set_view_depth: view index out of range");
    size_t pe = 0;
    int rc = image_pitch<float>(c, pitch_bytes, &pe);
    if (rc) return rc;
    if (pe < (size_t)c->W) return fail(GPM_E_ARG, "gpm_set_view_depth: pitch_bytes is shorter than a row");
    DeviceGuard g(c->device);
    const size_t n = (size_t)c->W * c->H;
    if (!c->geo_depth) CU(cudaMalloc(&c->geo_depth, n * c->maxV * sizeof(float)));
    if (!c->geo_kinv) {
        CU(cudaMalloc(&c->geo_kinv, sizeof(float) * 9 * c->maxV));
        c->cams_dirty = true;                        // sync_cams copies the K^-1 table with the cameras
    }
    CU(cudaMemcpy2DAsync(c->geo_depth + n * v, (size_t)c->W * sizeof(float), depth, pe * sizeof(float), (size_t)c->W * sizeof(float), c->H,
                         on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    c->have_depth[v] = 1;
    c->inputs_dirty = true;                          // the geometric term reads it: stored costs / memo are stale
    return GPM_OK;
}

// What the setters refuse for their arguments alone; the batch drivers check the same before any CUDA call (job_refusal).
namespace gpm {
const char* photometric_refusal(int kind, float min_std)
{
    if (kind != GPM_PHOTO_PM && kind != GPM_PHOTO_NCC) return "kind must be GPM_PHOTO_PM or GPM_PHOTO_NCC";
    if (kind == GPM_PHOTO_NCC && !(std::isfinite(min_std) && min_std > 0.f)) return "min_std must be finite and > 0";
    return nullptr;
}

const char* propagation_refusal(int kind)
{
    return kind != GPM_PROP_FIXED && kind != GPM_PROP_ADAPTIVE ? "propagation must be GPM_PROP_FIXED or GPM_PROP_ADAPTIVE" : nullptr;
}

const char* view_sel_refusal(const gpm_view_sel* v)
{
    if (!v) return "vsel is NULL";
    if (v->kind != GPM_VSEL_OFF && v->kind != GPM_VSEL_JOINT) return "kind must be GPM_VSEL_OFF or GPM_VSEL_JOINT";
    if (v->kind == GPM_VSEL_OFF) return nullptr;
    auto positive = [](float x) { return std::isfinite(x) && x > 0.f; };
    if (!positive(v->tau_init) || !positive(v->alpha) || !positive(v->tau_bad) || !positive(v->beta))
        return "tau_init, alpha, tau_bad and beta must be finite and > 0";
    if (!std::isfinite(v->w_keep) || v->w_keep < 0.f) return "w_keep must be finite and >= 0";
    if (v->n_good < 1 || v->n_good > 8) return "n_good must be 1..8";
    if (v->n_bad < 1 || v->n_bad > 9) return "n_bad must be 1..9";
    return nullptr;
}

const char* prior_refusal(float weight, float depth_sigma, float normal_sigma_deg);
const char* prior_build_refusal(const gpm_prior_build* b);

// The batch drivers' prior stage (NULL: none): gpm_set_prior's and gpm_build_planar_prior's argument rules, and iterations.
const char* prior_opts_refusal(const gpm_prior_opts* p)
{
    if (!p) return nullptr;
    if (const char* bad = prior_refusal(p->weight, p->depth_sigma, p->normal_sigma_deg)) return bad;
    const gpm_prior_build b{p->step, p->support_cost};
    if (const char* bad = prior_build_refusal(&b)) return bad;
    return p->iterations < 0 ? "prior iterations must be >= 0" : nullptr;
}

// gpm_set_refinement's argument rules (the fused sweep aside), also those of a batch driver's gpm_refine_opts
const char* refine_refusal(int kind, float perturbation)
{
    if (kind != GPM_REFINE_GIPUMA && kind != GPM_REFINE_ACMH) return "unknown refinement kind";
    if (!std::isfinite(perturbation) || !(perturbation > 0.f && perturbation < 1.f)) return "perturbation must be finite and in (0, 1)";
    return nullptr;
}

// What the batch drivers refuse for a job's options before any CUDA call: the setters' argument checks and the mode rule,
// for grey (channels 1) or colour (channels 4) images; a prior stage counts as the planar-prior mode.
const char* job_refusal(const gpm_job_opts* o, const gpm_view_sel* v, const gpm_prior_opts* prior, int channels)
{
    if (!o) return "opts is NULL";
    if (const char* bad = photometric_refusal(o->photometric, o->ncc_min_std)) return bad;
    if (const char* bad = propagation_refusal(o->propagation)) return bad;
    if (const char* bad = view_sel_refusal(v)) return bad;
    if (const char* bad = prior_opts_refusal(prior)) return bad;
    return conflict_text(mode_conflict(Mode{channels == 4, false, false, o->photometric == GPM_PHOTO_NCC,
                                            o->propagation == GPM_PROP_ADAPTIVE, v->kind == GPM_VSEL_JOINT, prior != nullptr}));
}
}  // namespace gpm

extern "C" int gpm_set_geometric(gpm_ctx* c, float weight, float max_err)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_geometric: null context");
    if (!std::isfinite(weight) || weight < 0.f) return fail(GPM_E_ARG, "gpm_set_geometric: weight must be finite and >= 0");
    if (!std::isfinite(max_err) || max_err <= 0.f) return fail(GPM_E_ARG, "gpm_set_geometric: max_err must be finite and > 0");
    if (weight > 0.f && c->shard_world > 0) return fail(GPM_E_STATE, "gpm_set_geometric: view sharding does not support the geometric-consistency mode");
    if (const int rc = refuse_change(c, "gpm_set_geometric", &Mode::geo, weight > 0.f)) return rc;
    if (const int rc = check_depth_maps(c, weight)) return rc;
    if (c->have_params && !prior_bound_ok(c->prm, ncc_on(c), weight, max_err, c->prior_weight))
        return fail(GPM_E_ARG, "gpm_set_geometric: with the planar prior's weight a valid cost could reach MAXCOST");
    if (weight != c->geo_weight || max_err != c->geo_max_err) c->inputs_dirty = true;
    c->geo_weight = weight;
    c->geo_max_err = max_err;
    return GPM_OK;
}

// The mask is copied (W x H bytes, compacted); NULL clears it.  The masked kernels read it only while the term is on, so
// only then does a change make stored costs and the memo stale.
extern "C" int gpm_set_geo_mask(gpm_ctx* c, const unsigned char* mask, size_t pitch_bytes, int on_device)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_geo_mask: null context");
    if (mask && c->prior_weight > 0.f) return fail(GPM_E_ARG, std::string("gpm_set_geo_mask: ") + conflict_text(ModeConflict::geomask));
    if (pitch_bytes == 0) pitch_bytes = (size_t)c->W;
    if (mask && pitch_bytes < (size_t)c->W) return fail(GPM_E_ARG, "gpm_set_geo_mask: pitch_bytes is smaller than a row");
    if (mask) {
        DeviceGuard g(c->device);
        if (!c->geo_mask) CU(cudaMalloc(&c->geo_mask, (size_t)c->W * c->H));
        CU(cudaMemcpy2DAsync(c->geo_mask, (size_t)c->W, mask, pitch_bytes, (size_t)c->W, c->H,
                             on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    if (c->geo_weight > 0.f && (mask || c->geo_mask_set)) c->inputs_dirty = true;
    c->geo_mask_set = mask != nullptr;
    return GPM_OK;
}

extern "C" int gpm_set_photometric(gpm_ctx* c, int kind, float min_std)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_photometric: null context");
    if (const char* bad = photometric_refusal(kind, min_std)) return fail(GPM_E_ARG, std::string("gpm_set_photometric: ") + bad);
    if (const int rc = refuse_change(c, "gpm_set_photometric", &Mode::ncc, kind == GPM_PHOTO_NCC)) return rc;
    if (c->have_params && !prior_bound_ok(c->prm, kind == GPM_PHOTO_NCC, c->geo_weight, c->geo_max_err, c->prior_weight))
        return fail(GPM_E_ARG, "gpm_set_photometric: with the planar prior's weight a valid cost could reach MAXCOST");
    if (kind == GPM_PHOTO_PM) min_std = 0.f;         // not read by the PM cost
    if (kind != c->photo || min_std != c->ncc_min_std) c->inputs_dirty = true;
    c->photo = kind;
    c->ncc_min_std = min_std;
    return GPM_OK;
}

// Only which plane is offered from each direction changes; the accept rule and cost(p, plane) do not, so stored costs, their
// provenance and the memo stay valid across a switch.
extern "C" int gpm_set_propagation(gpm_ctx* c, int kind)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_propagation: null context");
    if (const char* bad = propagation_refusal(kind)) return fail(GPM_E_ARG, std::string("gpm_set_propagation: ") + bad);
    if (const int rc = refuse_change(c, "gpm_set_propagation", &Mode::adaptive, kind == GPM_PROP_ADAPTIVE)) return rc;
    c->propagation = kind;
    return GPM_OK;
}

// Only the refinement's candidates change; the accept rule and cost(p, plane) do not, so nothing is marked stale.
extern "C" int gpm_set_refinement(gpm_ctx* c, int kind, float perturbation)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_refinement: null context");
    if (const char* bad = refine_refusal(kind, perturbation)) return fail(GPM_E_ARG, std::string("gpm_set_refinement: ") + bad);
    if (const int rc = refuse_change(c, "gpm_set_refinement", &Mode::refine_acmh, kind == GPM_REFINE_ACMH)) return rc;
    c->refine_kind = kind;
    c->refine_eps = perturbation;
    return GPM_OK;
}

// A switch either way changes what the stored costs mean (weighted or combined): they and the memo are marked stale.
extern "C" int gpm_set_view_selection(gpm_ctx* c, const gpm_view_sel* vsel)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_view_selection: null context");
    if (const char* bad = view_sel_refusal(vsel)) return fail(GPM_E_ARG, std::string("gpm_set_view_selection: ") + bad);
    if (const int rc = refuse_change(c, "gpm_set_view_selection", &Mode::jvs, vsel->kind == GPM_VSEL_JOINT)) return rc;
    if (vsel->kind == GPM_VSEL_JOINT && !jvs_on(c)) {
        DeviceGuard g(c->device);
        if (!c->vsel_mask) CU(cudaMalloc(&c->vsel_mask, (size_t)c->W * c->H * sizeof(unsigned long long)));
        const int rc = clear_vsel_masks(c);
        if (rc) return rc;
    }
    if (vsel->kind != c->vsel.kind) c->inputs_dirty = true;
    c->vsel = *vsel;
    return GPM_OK;
}

extern "C" int gpm_get_view_masks(gpm_ctx* c, unsigned long long* masks)
{
    if (!c || !masks) return fail(GPM_E_ARG, "gpm_get_view_masks: null argument");
    DeviceGuard g(c->device);
    const size_t n = (size_t)c->W * c->H;
    if (!c->vsel_mask) { memset(masks, 0, n * sizeof(unsigned long long));  return GPM_OK; }
    CU(cudaMemcpyAsync(masks, c->vsel_mask, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

// ---- planar prior (DESIGN.md §18) ---------------------------------------------------------------------------------
namespace gpm {
std::vector<std::array<int, 3>> delaunay(const std::vector<int>& xy);
std::array<float, 4> triangle_plane(const float* Kinv, const int* x, const int* y, const float* const* plane);

const char* prior_refusal(float weight, float depth_sigma, float normal_sigma_deg)
{
    if (!std::isfinite(weight) || weight < 0.f) return "weight must be finite and >= 0";
    if (!std::isfinite(depth_sigma) || depth_sigma <= 0.f) return "depth_sigma must be finite and > 0";
    if (!std::isfinite(normal_sigma_deg) || normal_sigma_deg <= 0.f || normal_sigma_deg > 90.f) return "normal_sigma_deg must be in (0, 90]";
    return nullptr;
}

const char* prior_build_refusal(const gpm_prior_build* b)
{
    if (!b) return "build is NULL";
    if (b->step < 1 || b->step > 64) return "step must be 1..64";
    if (b->support_cost != b->support_cost) return "support_cost must not be NaN";
    return nullptr;
}
}  // namespace gpm

static int ensure_prior_map(gpm_ctx* c)
{
    if (c->prior_map) return GPM_OK;
    const size_t n = (size_t)c->W * c->H;
    CU(cudaMalloc(&c->prior_map, n * sizeof(float4)));
    CU(cudaMemsetAsync(c->prior_map, 0, n * sizeof(float4), c->stream));
    return GPM_OK;
}

extern "C" int gpm_set_planar_prior(gpm_ctx* c, const float* planes, size_t pitch_bytes, int on_device)
{
    if (!c || !planes) return fail(GPM_E_ARG, "gpm_set_planar_prior: null argument");
    const size_t row = (size_t)c->W * sizeof(float4);
    if (pitch_bytes == 0) pitch_bytes = row;
    if (pitch_bytes < row) return fail(GPM_E_ARG, "gpm_set_planar_prior: pitch_bytes is smaller than a row");
    DeviceGuard g(c->device);
    if (const int rc = ensure_prior_map(c)) return rc;
    CU(cudaMemcpy2DAsync(c->prior_map, row, planes, pitch_bytes, row, c->H, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                         c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (c->prior_weight > 0.f) c->inputs_dirty = true;     // the cost function reads the map: stored costs / memo are stale
    return GPM_OK;
}

extern "C" int gpm_get_planar_prior(gpm_ctx* c, float* planes, int on_device)
{
    if (!c || !planes) return fail(GPM_E_ARG, "gpm_get_planar_prior: null argument");
    if (!c->prior_map) return fail(GPM_E_STATE, "gpm_get_planar_prior: no prior map (gpm_set_planar_prior or gpm_build_planar_prior)");
    DeviceGuard g(c->device);
    CU(cudaMemcpyAsync(planes, c->prior_map, (size_t)c->W * c->H * sizeof(float4), on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost,
                       c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_set_prior(gpm_ctx* c, float weight, float depth_sigma, float normal_sigma_deg)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_prior: null context");
    if (const char* bad = prior_refusal(weight, depth_sigma, normal_sigma_deg)) return fail(GPM_E_ARG, std::string("gpm_set_prior: ") + bad);
    if (weight > 0.f && c->shard_world > 0) return fail(GPM_E_STATE, "gpm_set_prior: view sharding does not support the planar prior");
    if (const int rc = refuse_change(c, "gpm_set_prior", &Mode::prior, weight > 0.f)) return rc;
    if (weight > 0.f && c->geo_mask_set) return fail(GPM_E_ARG, std::string("gpm_set_prior: ") + conflict_text(ModeConflict::geomask));
    if (weight > 0.f && !c->prior_map) return fail(GPM_E_STATE, "gpm_set_prior: no prior map (gpm_set_planar_prior or gpm_build_planar_prior)");
    if (c->have_params && !prior_bound_ok(c->prm, ncc_on(c), c->geo_weight, c->geo_max_err, weight))
        return fail(GPM_E_ARG, "gpm_set_prior: weight would let a valid cost reach MAXCOST");
    if (weight != c->prior_weight || (weight > 0.f && (depth_sigma != c->prior_depth_sigma || normal_sigma_deg != c->prior_normal_deg)))
        c->inputs_dirty = true;
    c->prior_weight = weight;
    c->prior_depth_sigma = depth_sigma;
    c->prior_normal_deg = normal_sigma_deg;
    return GPM_OK;
}

// Support points (GPU), Delaunay triangulation and triangle planes (host), rasterisation (GPU), from the stored state.
extern "C" int gpm_build_planar_prior(gpm_ctx* c, const gpm_prior_build* b, gpm_prior_info* info)
{
    if (!c) return fail(GPM_E_ARG, "gpm_build_planar_prior: null context");
    if (const char* bad = prior_build_refusal(b)) return fail(GPM_E_ARG, std::string("gpm_build_planar_prior: ") + bad);
    if (c->W > 4097 || c->H > 4097) return fail(GPM_E_ARG, "gpm_build_planar_prior: images wider or taller than 4097 pixels are not supported");
    if (!c->have_params || !c->have_ref) return fail(GPM_E_STATE, "gpm_build_planar_prior: gpm_set_params and gpm_set_reference first");
    if (!c->have_state) return fail(GPM_E_STATE, "gpm_build_planar_prior: no state to build from (gpm_init, gpm_run or gpm_set_state)");
    DeviceGuard g(c->device);
    KParams P{};
    P.W = c->W;  P.H = c->H;
    P.ref = c->ref;
    P.ref.depthMin = c->prm.depthMin;  P.ref.depthMax = c->prm.depthMax;
    const int step = b->step, cells_x = (c->W + step - 1) / step, cells_y = (c->H + step - 1) / step, ncell = cells_x * cells_y;
    int* d_at = nullptr;
    float4* d_pl = nullptr;
    int* d_tri = nullptr;
    float4* d_tpl = nullptr;
    unsigned long long* d_cnt = nullptr;
    auto release = [&]() { cudaFree(d_at);  cudaFree(d_pl);  cudaFree(d_tri);  cudaFree(d_tpl);  cudaFree(d_cnt); };
    auto cuda = [&](cudaError_t e, const char* what) -> int {
        if (e == cudaSuccess) return GPM_OK;
        release();
        return fail(GPM_E_CUDA, std::string("gpm_build_planar_prior: ") + what + ": " + cudaGetErrorString(e));
    };
    if (int rc = ensure_prior_map(c)) return rc;
    if (int rc = cuda(cudaMalloc(&d_at, ncell * sizeof(int)), "cudaMalloc")) return rc;
    if (int rc = cuda(cudaMalloc(&d_pl, ncell * sizeof(float4)), "cudaMalloc")) return rc;
    if (int rc = cuda(cudaMalloc(&d_cnt, sizeof(unsigned long long)), "cudaMalloc")) return rc;
    dim3 blk(16, 16), grd((cells_x + 15) / 16, (cells_y + 15) / 16);
    k_prior_support<<<grd, blk, 0, c->stream>>>(P, c->planes, c->cost, step, b->support_cost, cells_x, cells_y, d_at, d_pl);
    c->launches++;
    if (int rc = cuda(cudaGetLastError(), "k_prior_support")) return rc;
    std::vector<int> at(ncell);
    std::vector<float4> pl(ncell);
    if (int rc = cuda(cudaMemcpyAsync(at.data(), d_at, ncell * sizeof(int), cudaMemcpyDeviceToHost, c->stream), "cudaMemcpy")) return rc;
    if (int rc = cuda(cudaMemcpyAsync(pl.data(), d_pl, ncell * sizeof(float4), cudaMemcpyDeviceToHost, c->stream), "cudaMemcpy")) return rc;
    if (int rc = cuda(cudaStreamSynchronize(c->stream), "support points")) return rc;
    std::vector<int> xy;
    std::vector<float4> spl;
    for (int k = 0; k < ncell; k++)
        if (at[k] >= 0) { xy.push_back(at[k] % c->W);  xy.push_back(at[k] / c->W);  spl.push_back(pl[k]); }
    std::vector<std::array<int, 3>> tris;
    try { tris = delaunay(xy); } catch (const std::exception& e) { release();  return fail(GPM_E_STATE, std::string("gpm_build_planar_prior: triangulation failed: ") + e.what()); }
    const int ntri = (int)tris.size();
    std::vector<int> tv(6 * (size_t)std::max(ntri, 1));
    std::vector<float4> tp(std::max(ntri, 1));
    for (int t = 0; t < ntri; t++) {
        int x[3], y[3];
        const float* pp[3];
        for (int i = 0; i < 3; i++) {
            x[i] = xy[2 * tris[t][i]];  y[i] = xy[2 * tris[t][i] + 1];
            pp[i] = &spl[tris[t][i]].x;
            tv[6 * t + 2 * i] = x[i];  tv[6 * t + 2 * i + 1] = y[i];
        }
        const std::array<float, 4> q = triangle_plane(c->ref.K_inv, x, y, pp);
        tp[t] = make_float4(q[0], q[1], q[2], q[3]);
    }
    if (int rc = cuda(cudaMemsetAsync(c->prior_map, 0, (size_t)c->W * c->H * sizeof(float4), c->stream), "cudaMemset")) return rc;
    if (int rc = cuda(cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long), c->stream), "cudaMemset")) return rc;
    if (ntri > 0) {
        if (int rc = cuda(cudaMalloc(&d_tri, tv.size() * sizeof(int)), "cudaMalloc")) return rc;
        if (int rc = cuda(cudaMalloc(&d_tpl, tp.size() * sizeof(float4)), "cudaMalloc")) return rc;
        if (int rc = cuda(cudaMemcpyAsync(d_tri, tv.data(), tv.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream), "cudaMemcpy")) return rc;
        if (int rc = cuda(cudaMemcpyAsync(d_tpl, tp.data(), tp.size() * sizeof(float4), cudaMemcpyHostToDevice, c->stream), "cudaMemcpy")) return rc;
        k_prior_raster<<<(ntri + 127) / 128, 128, 0, c->stream>>>(P, d_tri, d_tpl, ntri, c->prior_map, d_cnt);
        c->launches++;
        if (int rc = cuda(cudaGetLastError(), "k_prior_raster")) return rc;
    }
    unsigned long long with = 0;
    if (int rc = cuda(cudaMemcpyAsync(&with, d_cnt, sizeof(with), cudaMemcpyDeviceToHost, c->stream), "cudaMemcpy")) return rc;
    if (int rc = cuda(cudaStreamSynchronize(c->stream), "rasterisation")) return rc;
    release();
    if (c->prior_weight > 0.f) c->inputs_dirty = true;
    if (info) { info->support = (long long)spl.size();  info->triangles = ntri;  info->with_prior = (long long)with; }
    return GPM_OK;
}

// Every pixel with a prior takes its prior plane where that plane's cost under the context's mode is strictly lower.
extern "C" int gpm_offer_prior(gpm_ctx* c)
{
    if (!c) return fail(GPM_E_ARG, "gpm_offer_prior: null context");
    if (!c->prior_map) return fail(GPM_E_STATE, "gpm_offer_prior: no prior map (gpm_set_planar_prior or gpm_build_planar_prior)");
    DeviceGuard g(c->device);
    KParams P;
    int rc = build_kparams(c, false, P);
    if (rc) return rc;
    rc = sync_cams(c);
    if (rc) return rc;
    if (!c->prior_cost) CU(cudaMalloc(&c->prior_cost, (size_t)c->W * c->H * sizeof(float)));
    rc = launch_cost_eval(c, P, c->prior_map, c->prior_cost);
    if (rc) return rc;
    dim3 b(16, 16), gr((c->W + 15) / 16, (c->H + 15) / 16);
    // provenance: the rounding variant k_cost_eval just used (bit 0 x-first, bit 1 gradient folding), or NCC's own tag
    const unsigned site = ncc_on(c) ? GPM_PROV_NCC : (unsigned)(P.cost_variant | (P.grad_variant << 1));
    k_offer_prior<<<gr, b, 0, c->stream>>>(P, c->prior_map, c->prior_cost, c->planes, c->cost, c->prov, site, c->pid, c->next_id);
    c->launches++;
    CU(cudaGetLastError());
    k_advance_ids<<<1, 1, 0, c->stream>>>(c->next_id, (unsigned)((size_t)c->W * c->H));
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_set_state(gpm_ctx* c, const float* norm4, const float* cost, int on_device)
{
    if (!c) return fail(GPM_E_ARG, "gpm_set_state: null context");
    DeviceGuard g(c->device);
    const size_t n = (size_t)c->W * c->H;
    const cudaMemcpyKind k = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    if (norm4) {
        CU(cudaMemcpyAsync(c->planes, norm4, n * sizeof(float4), k, c->stream));
        int rc = fill_ids(c);               // caller-supplied planes: every pixel's plane is its own (equal values are simply not recognised as such)
        if (rc) return rc;
    }
    if (cost) CU(cudaMemcpyAsync(c->cost, cost, n * sizeof(float), k, c->stream));
    if (norm4 && cost) c->have_state = true;
    // provenance of the supplied costs is unknown (GPM_PROV_UNKNOWN) unless the caller vouches that they came from an
    // initialisation / refinement evaluation of exactly these planes ("trust_state": 0)
    int rc = reset_state_tags(c, c->opt_trust_state ? init_prov(c) : GPM_PROV_UNKNOWN);
    if (rc) return rc;
    rc = clear_vsel_masks(c);                        // a new start state: no view selected, t = 0
    if (rc) return rc;
    c->vsel_t = 0;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_get_state(gpm_ctx* c, float* norm4, float* cost, int on_device)
{
    if (!c) return fail(GPM_E_ARG, "gpm_get_state: null context");
    DeviceGuard g(c->device);
    const size_t n = (size_t)c->W * c->H;
    const cudaMemcpyKind k = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (norm4) CU(cudaMemcpyAsync(norm4, c->planes, n * sizeof(float4), k, c->stream));
    if (cost) CU(cudaMemcpyAsync(cost, c->cost, n * sizeof(float), k, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

// Joint bilateral upsampling (DESIGN.md §19): reads the parameters' depth range, the reference's K^-1 and the reference image
// as staged for the sweep; the state, costs, memo and counters are left as they are.
extern "C" int gpm_upsample_planes(gpm_ctx* c, const float* coarse, int coarse_w, int coarse_h, int on_device,
                                   const gpm_jbu_params* jbu, float* planes, float* depth)
{
    if (!c || !coarse || !jbu) return fail(GPM_E_ARG, "gpm_upsample_planes: null argument");
    if (coarse_w != (c->W + 1) / 2 || coarse_h != (c->H + 1) / 2)
        return fail(GPM_E_ARG, "gpm_upsample_planes: the coarse level must be ((W + 1) / 2) x ((H + 1) / 2) of the context's");
    if (jbu->radius < 0 || jbu->radius > kJbuMaxRadius) return fail(GPM_E_ARG, "gpm_upsample_planes: radius must be 0..4");
    if (!(std::isfinite(jbu->sigma_space) && jbu->sigma_space > 0.f) || !(std::isfinite(jbu->sigma_range) && jbu->sigma_range > 0.f))
        return fail(GPM_E_ARG, "gpm_upsample_planes: sigma_space and sigma_range must be finite and > 0");
    if (!c->have_params || !c->have_ref) return fail(GPM_E_STATE, "gpm_upsample_planes: gpm_set_params and gpm_set_reference first");
    DeviceGuard g(c->device);
    JbuArgs a{};
    a.Wc = coarse_w;  a.Hc = coarse_h;  a.W = c->W;  a.H = c->H;  a.radius = jbu->radius;
    a.guide = c->refpad;  a.guide_pitch = c->refpitch;  a.apron = GPM_APRON;  a.color = c->color == 1;
    memcpy(a.kinv, c->ref.K_inv, sizeof(a.kinv));
    a.depth_min = c->prm.depthMin;  a.depth_max = c->prm.depthMax;
    const double ss = jbu->sigma_space, sr = jbu->sigma_range;
    a.k_range = (float)(1.0 / (sr * sr));
    for (int by = 0; by < 2; by++)
        for (int bx = 0; bx < 2; bx++)
            for (int j = -kJbuMaxRadius; j <= kJbuMaxRadius; j++)
                for (int i = -kJbuMaxRadius; i <= kJbuMaxRadius; i++) {
                    const double dx = 2 * i - bx, dy = 2 * j - by;       // (2 q - p) in fine pixels
                    a.ws[((by * 2 + bx) * kJbuSide + j + kJbuMaxRadius) * kJbuSide + i + kJbuMaxRadius] =
                        (float)std::exp(-(dx * dx + dy * dy) / (2.0 * ss * ss));
                }
    const size_t nc = (size_t)coarse_w * coarse_h, n = (size_t)c->W * c->H;
    void *d_coarse = nullptr, *d_planes = nullptr, *d_depth = nullptr;
    cudaError_t e = cudaSuccess;
    if (on_device) {
        a.coarse = reinterpret_cast<const float4*>(coarse);
        a.planes = reinterpret_cast<float4*>(planes);
        a.depth = depth;
    } else {
        e = cudaMalloc(&d_coarse, nc * sizeof(float4));
        if (e == cudaSuccess && planes) e = cudaMalloc(&d_planes, n * sizeof(float4));
        if (e == cudaSuccess && depth) e = cudaMalloc(&d_depth, n * sizeof(float));
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_coarse, coarse, nc * sizeof(float4), cudaMemcpyHostToDevice, c->stream);
        a.coarse = static_cast<const float4*>(d_coarse);
        a.planes = static_cast<float4*>(d_planes);
        a.depth = static_cast<float*>(d_depth);
    }
    if (e == cudaSuccess) e = launch_jbu(a, c->stream);
    if (e == cudaSuccess && !on_device && planes) e = cudaMemcpyAsync(planes, d_planes, n * sizeof(float4), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess && !on_device && depth) e = cudaMemcpyAsync(depth, d_depth, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    cudaFree(d_coarse);  cudaFree(d_planes);  cudaFree(d_depth);
    if (e != cudaSuccess) return fail(GPM_E_CUDA, std::string("gpm_upsample_planes: ") + cudaGetErrorString(e));
    return GPM_OK;
}

static int do_init(gpm_ctx* c)
{
    KParams P;
    int rc = build_kparams(c, true, P);
    if (rc) return rc;
    rc = sync_cams(c);
    if (rc) return rc;
    rc = init_planes(c, P);
    if (rc) return rc;
    rc = launch_cost_eval(c, P, c->planes, c->cost);
    if (rc) return rc;
    rc = clear_vsel_masks(c);                      // view selection starts over: no view selected, t = 0
    if (rc) return rc;
    c->vsel_t = 0;
    c->have_state = true;
    return reset_state_tags(c, init_prov(c));     // costs now come from the init-variant evaluation (float4: x-first + gradient folding 1; NCC: its own)
}

static int do_sweeps(gpm_ctx* c, int iterations)
{
    KParams P;
    int rc = build_kparams(c, false, P);
    if (rc) return rc;
    rc = sync_cams(c);
    if (rc) return rc;
    for (int it = 0; it < iterations; it++) {                                  // gipuma.cu:1911-1941
        rc = launch_colour(c, P, 0, 7);
        if (rc) return rc;
        rc = launch_colour(c, P, 1, 7);
        if (rc) return rc;
        c->vsel_t++;                                                           // view selection's iteration count (§17)
    }
    return GPM_OK;
}

static int do_finalize(gpm_ctx* c)
{
    KParams P;
    int rc = build_kparams(c, false, P);
    if (rc) return rc;
    dim3 b(16, 16), gr((c->W + 15) / 16, (c->H + 15) / 16);
    k_finalize<<<gr, b, 0, c->stream>>>(P, c->planes, c->cost);
    c->launches++;
    CU(cudaGetLastError());
    return reset_state_tags(c, GPM_PROV_UNKNOWN);          // planes are world-frame outputs now
}

extern "C" int gpm_init(gpm_ctx* c)
{
    if (!c) return fail(GPM_E_ARG, "null context");
    DeviceGuard g(c->device);
    int rc = do_init(c);
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_sweep(gpm_ctx* c, int iterations)
{
    if (!c || iterations < 0) return fail(GPM_E_ARG, "gpm_sweep: bad arguments");
    DeviceGuard g(c->device);
    int rc = do_sweeps(c, iterations);
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_phase(gpm_ctx* c, int colour, int phase_mask)
{
    if (!c || colour < 0 || colour > 1 || phase_mask < 1 || phase_mask > 7) return fail(GPM_E_ARG, "gpm_phase: bad arguments");
    DeviceGuard g(c->device);
    KParams P;
    int rc = build_kparams(c, false, P);
    if (rc) return rc;
    rc = sync_cams(c);
    if (rc) return rc;
    rc = launch_colour(c, P, colour, phase_mask);
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_finalize(gpm_ctx* c)
{
    if (!c) return fail(GPM_E_ARG, "null context");
    DeviceGuard g(c->device);
    int rc = do_finalize(c);
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_cost_eval(gpm_ctx* c, const float* planes, float* out_cost, int on_device)
{
    if (!c || !planes || !out_cost) return fail(GPM_E_ARG, "gpm_cost_eval: null argument");
    DeviceGuard g(c->device);
    KParams P;
    int rc = build_kparams(c, false, P, true);
    if (rc) return rc;
    rc = sync_cams(c);
    if (rc) return rc;
    const size_t n = (size_t)c->W * c->H;
    float4* d_pl = nullptr;
    float* d_out = nullptr;
    if (on_device) { d_pl = (float4*)planes;  d_out = out_cost; }
    else {
        cudaError_t e1 = cudaMalloc(&d_pl, n * sizeof(float4));
        if (e1 == cudaSuccess) e1 = cudaMalloc(&d_out, n * sizeof(float));
        if (e1 == cudaSuccess) e1 = cudaMemcpyAsync(d_pl, planes, n * sizeof(float4), cudaMemcpyHostToDevice, c->stream);
        if (e1 != cudaSuccess) { cudaFree(d_pl);  cudaFree(d_out);  return fail(GPM_E_CUDA, std::string("gpm_cost_eval: ") + cudaGetErrorString(e1)); }
    }
    rc = launch_cost_eval(c, P, d_pl, d_out);
    cudaError_t e = cudaSuccess;
    if (rc == GPM_OK && !on_device) e = cudaMemcpyAsync(out_cost, d_out, n * sizeof(float), cudaMemcpyDeviceToHost, c->stream);
    if (rc == GPM_OK && e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (!on_device) { cudaFree(d_pl);  cudaFree(d_out); }
    if (rc) return rc;
    if (e != cudaSuccess) return fail(GPM_E_CUDA, std::string("gpm_cost_eval: ") + cudaGetErrorString(e));
    return GPM_OK;
}

extern "C" int gpm_run(gpm_ctx* c, float* sweep_ms)
{
    if (!c) return fail(GPM_E_ARG, "null context");
    DeviceGuard g(c->device);
    CU(cudaMemsetAsync(c->d_stats, 0, 8 * sizeof(unsigned long long), c->stream));
    c->launches = 0;
    int rc = do_init(c);
    if (rc) return rc;
    CU(cudaEventRecord(c->ev0, c->stream));                                    // gipuma.cu:1908
    rc = do_sweeps(c, c->prm.iterations);
    if (rc) return rc;
    rc = do_finalize(c);
    if (rc) return rc;
    CU(cudaEventRecord(c->ev1, c->stream));                                    // gipuma.cu:1946
    CU(cudaEventSynchronize(c->ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
    if (sweep_ms) *sweep_ms = ms;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}


// ---- source-view sharding (multi-GPU) -------------------------------------------------------------------------
static int shard_refine_steps(const gpm_params& p)
{
    int n = 0;
    for (float dz = p.max_disparity * 0.5f; dz >= 0.01f; dz = dz * 0.1f) n++;      // gipuma.cu:958-959
    return n;
}

// Every shard call taking a context refuses a mode shard_supports() does not pass, before anything is launched: with
// GPM_E_STATE here, but the fused sweep only where it launches (shard_common), with GPM_E_ARG.
static int shard_refuses_state(gpm_ctx* c)
{
    if (c->refine_kind != GPM_REFINE_GIPUMA) return fail(GPM_E_STATE, "view sharding supports Gipuma's refinement only (GPM_REFINE_GIPUMA)");
    Mode m = ctx_mode(c);
    m.fused = false;
    return shard_supports(m) ? GPM_OK : fail(GPM_E_STATE, "view sharding supports neither the geometric-consistency mode, the NCC cost, joint view selection nor the planar prior");
}

extern "C" int gpm_shard_num_stages(gpm_ctx* c)
{
    if (!c || !c->have_params) { fail(GPM_E_STATE, "gpm_shard_num_stages: parameters not set");  return -1; }
    if (shard_refuses_state(c)) return -1;
    return 2 + shard_refine_steps(c->prm);
}

extern "C" long long gpm_shard_stage_floats(gpm_ctx* c, int stage)
{
    if (!c || !c->have_params || stage < 0) { fail(GPM_E_ARG, "gpm_shard_stage_floats: bad arguments");  return -1; }
    if (shard_refuses_state(c)) return -1;
    const long long half = (long long)c->H * ((c->W + 1) / 2);
    const int slots = stage == 1 ? 8 : 1;
    return (stage == 0 ? 2 : 1) * half * slots * c->prm.n_best;
}

static int shard_common(gpm_ctx* c, int stage, KParams& P)
{
    if (const int rc = shard_refuses_state(c)) return rc;
    if (c->prm.cost_comb != GPM_COMB_BEST_N) return fail(GPM_E_ARG, "view sharding supports cost_comb = best_n only");
    if (!shard_supports(ctx_mode(c))) return fail(GPM_E_ARG, "view sharding supports the 8-neighbour sweep only (option neighbours = 8)");
    if (c->prm.n_best < 1 || c->prm.n_best > 32) return fail(GPM_E_ARG, "view sharding needs 1 <= n_best <= 32");
    if (c->rng_mode != GPM_RNG_REFERENCE) return fail(GPM_E_ARG, "view sharding implements the reference's zero-state refinement stream only (GPM_RNG_REFERENCE)");
    const int last = 1 + shard_refine_steps(c->prm);
    if (stage < 0 || stage > last + 1) return fail(GPM_E_ARG, "no such stage");
    int rc = build_kparams(c, stage == 0, P);
    if (rc) return rc;
    rc = sync_cams(c);
    if (rc) return rc;
    if (!c->dispbuf) {
        const size_t n = (size_t)c->W * c->H;
        CU(cudaMalloc(&c->dispbuf, n * sizeof(float)));
        CU(cudaMalloc(&c->candbuf, n * sizeof(float4)));
        CU(cudaMalloc(&c->canddepth, n * sizeof(float)));
        CU(cudaMalloc(&c->sflags, n));
        CU(cudaMemsetAsync(c->sflags, 0, n, c->stream));
    }
    return GPM_OK;
}

// enqueue one stage kernel (stage 0 .. last+1) on the context's stream
static int shard_launch_stage(gpm_ctx* c, const KParams& P, int colour, int stage, const float* gathered_prev, int world, float* xchg)
{
    const auto kern = kShardStage[eval_bits(c)];
    if (!kern) return fail(GPM_E_STATE, "k_shard_stage has no kernel for this context's mode");
    const int last = 1 + shard_refine_steps(c->prm);
    ShardState S{c->dispbuf, c->candbuf, c->canddepth, c->sflags};
    kern<<<tile_grid(c), P.nwarps * 32, block_smem_bytes(P), c->stream>>>(P, c->tmap, c->d_cams,
        c->srcTex, c->planes, c->cost, c->prov, S, Memo{c->pid, c->seen, c->refseen, c->memo_mask, c->next_id}, colour, stage, last,
        gathered_prev, world, xchg, c->d_stats);
    c->launches++;
    CU(cudaGetLastError());
    return GPM_OK;
}

// closing accept of stage 0: the merged initial costs (the kernel sets their provenance to the initialisation variant)
static int shard_accept0(gpm_ctx* c, const KParams& P, const float* gathered, int world)
{
    dim3 b(32, 8), gr(((P.W + 1) / 2 + 31) / 32, (P.H + 7) / 8);
    k_shard_accept0<<<gr, b, 0, c->stream>>>(P, c->cost, c->prov, gathered, world);
    c->launches++;
    CU(cudaGetLastError());
    return reset_state_tags(c, PROV_KEEP);
}

extern "C" int gpm_shard_stage(gpm_ctx* c, int colour, int stage, const float* gathered_prev_dev, int world, float* xchg_dev)
{
    if (!c || colour < 0 || colour > 1 || world < 1 || world > 8) return fail(GPM_E_ARG, "gpm_shard_stage: bad arguments");
    DeviceGuard g(c->device);
    KParams P;
    int rc = shard_common(c, stage, P);
    if (rc) return rc;
    const int last = 1 + shard_refine_steps(c->prm);
    if (stage >= 2 && !gathered_prev_dev) return fail(GPM_E_ARG, "gpm_shard_stage: stages >= 2 need the gathered lists of the previous stage");
    if (stage <= last && !xchg_dev) return fail(GPM_E_ARG, "gpm_shard_stage: no exchange buffer");
    rc = shard_launch_stage(c, P, colour, stage, gathered_prev_dev, world, xchg_dev);
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));       // the caller's collective may run on another stream
    return GPM_OK;
}

extern "C" int gpm_shard_finish_init(gpm_ctx* c, const float* gathered_dev, int world)
{
    if (!c || !gathered_dev || world < 1 || world > 8) return fail(GPM_E_ARG, "gpm_shard_finish_init: bad arguments");
    DeviceGuard g(c->device);
    KParams P;
    int rc = shard_common(c, 0, P);
    if (rc) return rc;
    rc = shard_accept0(c, P, gathered_dev, world);
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

// ---- the exchange behind the C-ABI: NCCL, loaded at run time (a C++ host needs no torch) ---------------------------
#include <dlfcn.h>
namespace {
struct NcclId { char internal[128]; };
struct NcclApi {
    void* h = nullptr;
    int (*GetUniqueId)(NcclId*) = nullptr;
    int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    int (*GetVersion)(int*) = nullptr;
};
NcclApi* nccl_api()
{
    static NcclApi api;
    static bool tried = false;
    if (!tried) {
        tried = true;
        const char* names[] = {getenv("GPM_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n) continue;
            api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.h) break;
        }
        if (api.h) {
            api.GetUniqueId = (int (*)(NcclId*))dlsym(api.h, "ncclGetUniqueId");
            api.CommInitRank = (int (*)(void**, int, NcclId, int))dlsym(api.h, "ncclCommInitRank");
            api.CommDestroy = (int (*)(void*))dlsym(api.h, "ncclCommDestroy");
            api.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(api.h, "ncclAllGather");
            api.GetErrorString = (const char* (*)(int))dlsym(api.h, "ncclGetErrorString");
            api.GetVersion = (int (*)(int*))dlsym(api.h, "ncclGetVersion");
            if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllGather) { dlclose(api.h);  api.h = nullptr; }
        }
    }
    return api.h ? &api : nullptr;
}
}  // namespace

#define NC(call)                                                                                                        \
    do {                                                                                                                \
        int e_ = (call);                                                                                                \
        if (e_ != 0) return fail(GPM_E_CUDA, std::string(#call) + ": NCCL error " + (nccl_api() && nccl_api()->GetErrorString ? nccl_api()->GetErrorString(e_) : "?")); \
    } while (0)

static void gpm_shard_comm_destroy_(gpm_ctx* c)
{
    if (c->comm && c->comm_owned && nccl_api()) nccl_api()->CommDestroy(c->comm);
    c->comm = nullptr;  c->comm_owned = false;
}

extern "C" int gpm_shard_unique_id(void* id128)
{
    if (!id128) return fail(GPM_E_ARG, "gpm_shard_unique_id: null argument");
    NcclApi* n = nccl_api();
    if (!n) return fail(GPM_E_STATE, "NCCL (libnccl.so.2) could not be loaded; set GPM_NCCL_LIB");
    NC(n->GetUniqueId((NcclId*)id128));
    return GPM_OK;
}

static int shard_alloc_exchange(gpm_ctx* c)
{
    long long mx = 0;
    const int ns = gpm_shard_num_stages(c);
    for (int st = 0; st < ns; st++) { const long long f = gpm_shard_stage_floats(c, st);  if (f > mx) mx = f; }
    if (c->xchg && c->xchg_floats >= (size_t)mx && c->gath_world >= c->shard_world) return GPM_OK;
    CU(cudaStreamSynchronize(c->stream));
    cudaFree(c->xchg);  cudaFree(c->gath);  c->xchg = c->gath = nullptr;
    CU(cudaMalloc(&c->xchg, (size_t)mx * sizeof(float)));
    CU(cudaMalloc(&c->gath, (size_t)mx * sizeof(float) * c->shard_world));
    c->xchg_floats = (size_t)mx;  c->gath_world = c->shard_world;
    return GPM_OK;
}

extern "C" int gpm_shard_comm_init(gpm_ctx* c, const void* id128, int rank, int world)
{
    if (!c || world < 1 || world > 8 || rank < 0 || rank >= world) return fail(GPM_E_ARG, "gpm_shard_comm_init: bad arguments (1 <= world <= 8)");
    if (const int rc = shard_refuses_state(c)) return rc;
    DeviceGuard g(c->device);
    gpm_shard_comm_destroy_(c);
    c->shard_rank = rank;  c->shard_world = world;
    if (world > 1) {
        if (!id128) return fail(GPM_E_ARG, "gpm_shard_comm_init: null unique id");
        NcclApi* n = nccl_api();
        if (!n) return fail(GPM_E_STATE, "NCCL (libnccl.so.2) could not be loaded; set GPM_NCCL_LIB");
        NcclId id;  memcpy(&id, id128, sizeof(id));
        NC(n->CommInitRank(&c->comm, world, id, rank));
        c->comm_owned = true;
    }
    return GPM_OK;
}

extern "C" int gpm_shard_comm_attach(gpm_ctx* c, void* nccl_comm, int rank, int world)
{
    if (!c || world < 1 || world > 8 || rank < 0 || rank >= world || (world > 1 && !nccl_comm)) return fail(GPM_E_ARG, "gpm_shard_comm_attach: bad arguments");
    if (const int rc = shard_refuses_state(c)) return rc;
    if (world > 1 && !nccl_api()) return fail(GPM_E_STATE, "NCCL (libnccl.so.2) could not be loaded; set GPM_NCCL_LIB");
    gpm_shard_comm_destroy_(c);
    c->comm = nccl_comm;  c->shard_rank = rank;  c->shard_world = world;
    return GPM_OK;
}

// all-gather of this rank's lists of one stage (rank-major result), on the context's stream
static int shard_exchange(gpm_ctx* c, int stage)
{
    const size_t n = (size_t)gpm_shard_stage_floats(c, stage);
    if (c->shard_world == 1) { CU(cudaMemcpyAsync(c->gath, c->xchg, n * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));  return GPM_OK; }
    NC(nccl_api()->AllGather(c->xchg, c->gath, n, 7 /* ncclFloat32 */, c->comm, c->stream));
    c->collectives++;
    return GPM_OK;
}

// runcuda() with the source views sharded over the ranks of the attached communicator.  Every rank calls it with the same
// parameters, reference image and seed and ITS views; all work — kernels and collectives — is enqueued on the context's
// stream, one host synchronisation at the end.
extern "C" int gpm_shard_run(gpm_ctx* c, float* sweep_ms)
{
    if (!c) return fail(GPM_E_ARG, "null context");
    if (c->shard_world < 1) return fail(GPM_E_STATE, "gpm_shard_run: no communicator (gpm_shard_comm_init / gpm_shard_comm_attach)");
    DeviceGuard g(c->device);
    KParams P0, P;
    int rc = shard_common(c, 0, P0);
    if (rc) return rc;
    rc = shard_common(c, 1, P);
    if (rc) return rc;
    rc = shard_alloc_exchange(c);
    if (rc) return rc;
    const int world = c->shard_world, last = 1 + shard_refine_steps(c->prm);
    CU(cudaMemsetAsync(c->d_stats, 0, 8 * sizeof(unsigned long long), c->stream));
    c->launches = 0;  c->collectives = 0;
    if (world > 1 && !c->comm) return fail(GPM_E_STATE, "gpm_shard_run: no NCCL communicator is attached");
    rc = init_planes(c, P0);
    if (rc) return rc;
    rc = shard_launch_stage(c, P0, 0, 0, nullptr, world, c->xchg);
    if (rc) return rc;
    rc = shard_exchange(c, 0);
    if (rc) return rc;
    rc = shard_accept0(c, P0, c->gath, world);
    if (rc) return rc;
    CU(cudaEventRecord(c->ev0, c->stream));
    for (int it = 0; it < c->prm.iterations; it++)
        for (int colour = 0; colour < 2; colour++) {
            for (int stage = 1; stage <= last; stage++) {
                rc = shard_launch_stage(c, P, colour, stage, c->gath, world, c->xchg);
                if (rc) return rc;
                rc = shard_exchange(c, stage);
                if (rc) return rc;
            }
            rc = shard_launch_stage(c, P, colour, last + 1, c->gath, world, c->xchg);     // closing accept of the colour
            if (rc) return rc;
        }
    rc = do_finalize(c);
    if (rc) return rc;
    CU(cudaEventRecord(c->ev1, c->stream));
    CU(cudaEventSynchronize(c->ev1));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
    if (sweep_ms) *sweep_ms = ms;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

// random planes only (stage 0 of the sharded flow computes the initial cost over all ranks' views)
extern "C" int gpm_init_planes(gpm_ctx* c)
{
    if (!c) return fail(GPM_E_ARG, "null context");
    DeviceGuard g(c->device);
    KParams P;
    int rc = build_kparams(c, true, P);
    if (rc) return rc;
    rc = init_planes(c, P);
    if (rc) return rc;
    rc = reset_state_tags(c, GPM_PROV_UNKNOWN);                // every plane is new: costs and memo are stale
    if (rc) return rc;
    CU(cudaStreamSynchronize(c->stream));
    return GPM_OK;
}

extern "C" int gpm_measure_fetch_peak(gpm_ctx* c, double* gfetch_per_s)
{
    if (!c || !gfetch_per_s) return fail(GPM_E_ARG, "gpm_measure_fetch_peak: null argument");
    if (c->V < 1 || c->color < 0) return fail(GPM_E_STATE, "gpm_measure_fetch_peak: no source views");
    DeviceGuard g(c->device);
    float* sink = reinterpret_cast<float*>(c->d_stats + 7);         // d_stats[7] holds no counter: it is only k_fetch_peak's sink
    const int blocks = c->num_sms * 16, threads = 256, reps = 2048;
    const int layers = c->color == 1 ? 3 * c->V : c->V;       // colour: three R32F channel planes per view
    // random positions inside a window of at most 512 x 512 texels of at most 4 layers: the UNIT's ceiling is wanted, so the
    // working set must stay in L2 whatever the image size (a 3200 x 2400 x 64-layer array would make this a DRAM test)
    int xmask = 1, ymask = 1;
    while (2 * xmask + 1 < c->W - 48 && xmask < 511) xmask = 2 * xmask + 1;
    while (2 * ymask + 1 < c->H - 24 && ymask < 511) ymask = 2 * ymask + 1;
    k_fetch_peak<<<blocks, threads, 0, c->stream>>>(c->srcTex, xmask, ymask, layers, 64, sink);        // warm-up
    double best = 0.0;
    for (int rep = 0; rep < 3; rep++) {
        CU(cudaEventRecord(c->ev0, c->stream));
        k_fetch_peak<<<blocks, threads, 0, c->stream>>>(c->srcTex, xmask, ymask, layers, reps, sink);
        CU(cudaEventRecord(c->ev1, c->stream));
        CU(cudaEventSynchronize(c->ev1));
        CU(cudaGetLastError());
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
        const double g = (double)blocks * threads * reps * 5.0 / (ms * 1e6);
        if (g > best) best = g;
    }
    *gfetch_per_s = best;
    return GPM_OK;
}

extern "C" int gpm_get_stats(gpm_ctx* c, unsigned long long stats[8])
{
    if (!c || !stats) return fail(GPM_E_ARG, "gpm_get_stats: null argument");
    DeviceGuard g(c->device);
    CU(cudaMemcpyAsync(stats, c->d_stats, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    stats[ST_LAUNCH] = c->launches;
    stats[6] = c->collectives;
    return GPM_OK;
}

extern "C" int gpm_reset_stats(gpm_ctx* c)
{
    if (!c) return fail(GPM_E_ARG, "null context");
    DeviceGuard g(c->device);
    CU(cudaMemsetAsync(c->d_stats, 0, 8 * sizeof(unsigned long long), c->stream));
    c->launches = 0;
    return GPM_OK;
}

extern "C" int gpm_set_option(gpm_ctx* c, const char* name, int value)
{
    if (!c || !name) return fail(GPM_E_ARG, "gpm_set_option: null argument");
    const std::string n(name);
    if (n == "prune") c->opt_prune = value != 0;
    else if (n == "dedupe") c->opt_dedupe = value != 0;
    else if (n == "trust_state") c->opt_trust_state = value != 0;
    else if (n == "nwarps") c->opt_nwarps = value;
    else if (n == "cost_variant") c->opt_cost_variant = value < 0 ? -1 : (value & 15);
    else if (n.rfind("site", 0) == 0 && n.size() > 4 && n.size() <= 6 && std::isdigit((unsigned char)n[4])) {
        const int k = std::atoi(n.c_str() + 4);             // "site<k>": variant of call site k of the fused kernel (diagnostics)
        if (k < 0 || k > 20) return fail(GPM_E_ARG, "site index out of range");
        c->opt_site[k] = value < 0 ? -1 : (value & 15);
    }
    else if (n == "neighbours") {
        if (value != 8 && value != 20) return fail(GPM_E_ARG, "neighbours must be 8 (close + far kernels) or 20 (fused kernel)");
        if (const int rc = refuse_change(c, "gpm_set_option", &Mode::fused, value == 20)) return rc;
        DeviceGuard g(c->device);
        const int slots = value == 20 ? 20 : 8;
        if (slots != c->seen_slots) {
            CU(cudaStreamSynchronize(c->stream));
            cudaFree(c->seen);  c->seen = nullptr;
            CU(cudaMalloc(&c->seen, (size_t)c->W * c->H * slots * sizeof(unsigned)));
            c->seen_slots = slots;
        }
        c->memo_dirty = true;
        c->opt_neighbours = value;
    }
    else if (n == "memo") c->opt_memo = value != 0;
    else if (n == "quadperm") c->opt_quadperm = value != 0;
    else return fail(GPM_E_ARG, "gpm_set_option: unknown option '" + n + "'");
    return GPM_OK;
}

extern "C" void* gpm_stream(gpm_ctx* c) { return c ? (void*)c->stream : nullptr; }
