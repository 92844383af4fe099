/* gipuma_b200.h — C-ABI of the PatchMatch hot path (CUDA, sm_90a / H100).
 *
 * This library replaces exactly one thing in kysucix/gipuma: the work behind
 *      int runcuda(GlobalState &gs);                     (reference gipuma.h:2, gipuma.cu:1962-1970)
 * i.e. gipuma<T>() (gipuma.cu:1825-1960): random plane initialisation, red/black checkerboard
 * spatial propagation (close +-1 px, far +-5 px), plane refinement, the multi-view
 * adaptive-support-weight photo-consistency cost, and the final depth / world-normal output.
 *
 * Plain C, no torch / CUDA types in the signatures: device pointers are passed as void* plus an
 * `on_device` flag.  Every entry point returns 0 on success or a negative GPM_E_* code;
 * gpm_last_error() returns a thread-local description.  One gpm_ctx per device / per reference view;
 * contexts are independent (one per rank in multi-GPU runs).
 *
 * The runcuda() adapter that flattens the reference's managed GlobalState into these calls lives in
 * gipuma_b200/csrc/runcuda_adapter.cu (it is the only code that knows GlobalState); see INTEGRATION.md.
 */
#ifndef GIPUMA_B200_H
#define GIPUMA_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GPM_MAX_VIEWS 64          /* source views per reference view (reference: costVector[32], gipuma.cu:736) */
#define GPM_MAX_BOX   25          /* window size limit of the reference's tile loader (gipuma.cu:1513-1522) */

enum {
    GPM_OK = 0,
    GPM_E_ARG = -1,               /* bad argument / unsupported parameter */
    GPM_E_CUDA = -2,              /* a CUDA call failed; see gpm_last_error() */
    GPM_E_STATE = -3              /* call sequence error (e.g. sweep before views are set) */
};

/* cost combination — algorithmparameters.h:17 */
enum { GPM_COMB_ALL = 0, GPM_COMB_BEST_N = 1, GPM_COMB_ANGLE = 2, GPM_COMB_GOOD = 3 };

/* RNG behaviour of the plane-refinement step.
 * GPM_RNG_REFERENCE reproduces what the reference does: gs.cs is cudaMalloc'ed and never written
 * (gipuma.cu:1840, 1608, 1702), so every refinement kernel starts each pixel from an all-zero XORWOW
 * state.  GPM_RNG_STATEFUL keeps a per-pixel XORWOW state seeded at init and advanced by every draw
 * (what the code evidently intended); it has no reference output to compare against. */
enum { GPM_RNG_REFERENCE = 0, GPM_RNG_STATEFUL = 1 };

/* The AlgorithmParameters fields the device path reads (algorithmparameters.h:53-84). */
typedef struct gpm_params {
    int   box_hsize, box_vsize;         /* odd, equal, <= GPM_MAX_BOX */
    float tau_color, tau_gradient;
    float alpha, gamma;
    float min_disparity, max_disparity; /* = f*baseline/depthMax, f*baseline/depthMin (main.cpp:905-906) */
    int   iterations;
    int   n_best;
    int   cost_comb;                    /* GPM_COMB_* */
    float good_factor;
    float depthMin, depthMax;           /* cameras[REFERENCE].depthMin/Max (main.cpp:898-903) */
} gpm_params;

/* The Camera_cu fields the device path reads (camera.h:7-62), 3x3 matrices row-major. */
typedef struct gpm_camera {
    float K[9], K_inv[9], R[9], M_inv[9], R_orig_inv[9];
    float t[3], C[3], P_col34[3];
    float fx, fy, f, alpha, baseline;
} gpm_camera;

typedef struct gpm_ctx gpm_ctx;

/* Create a context on CUDA device `device` for width x height images and up to `max_views`
 * source views.  Replaces the allocations of gipuma<T>() (gipuma.cu:1840) and main.cpp:927-933. */
int gpm_create(gpm_ctx** out, int device, int width, int height, int max_views);
void gpm_destroy(gpm_ctx* ctx);

int gpm_set_params(gpm_ctx* ctx, const gpm_params* p);

/* Reference image + camera (index REFERENCE=0 of gs.imgs / gs.cameras->cameras, config.h:21).
 * `img` is row-major float, `pitch_bytes` between rows; host or device memory. */
int gpm_set_reference(gpm_ctx* ctx, const float* img, size_t pitch_bytes, int on_device, const gpm_camera* cam);

/* Source view `v` (0-based position in viewSelectionSubset, main.cpp:888-892). */
int gpm_set_view(gpm_ctx* ctx, int v, const float* img, size_t pitch_bytes, int on_device, const gpm_camera* cam);

/* Colour images: the reference's -color_processing path (T = float4, gipuma.cu:1965-1966; images built at
 * main.cpp:560-605).  `rgba` is row-major float4 per pixel (x, y, z = the three colour channels, w ignored — the
 * reference's float4 operators drop it, vector_operations.h:3-38).  A context holds either float or float4 images. */
int gpm_set_reference_color(gpm_ctx* ctx, const float* rgba, size_t pitch_bytes, int on_device, const gpm_camera* cam);
int gpm_set_view_color(gpm_ctx* ctx, int v, const float* rgba, size_t pitch_bytes, int on_device, const gpm_camera* cam);

/* Number of source views actually used (viewSelectionSubsetNumber, main.cpp:918). */
int gpm_set_num_views(gpm_ctx* ctx, int n_views);

/* ---- mode compatibility -------------------------------------------------------------------------------------------------
 * A context sweeps in one mode of nine fields: colour images (fixed by the first image upload), the fused 20-neighbour
 * sweep (option "neighbours" = 20), the geometric-consistency term, the NCC cost, adaptive sampling, joint view selection,
 * the planar prior (DESIGN.md §14–§18), the geometric term's per-pixel mask (§21; it counts while the term is on) and
 * ACMH's refinement (§23).
 * Every combination exists except:
 *   - the fused sweep with the geometric term, the NCC cost, adaptive sampling, joint view selection or the planar prior;
 *   - joint view selection without the NCC cost, and so with colour images;
 *   - the NCC cost with colour images;
 *   - the planar prior with colour images or with joint view selection;
 *   - a geometric term's mask with the planar prior (whether the term is on or not);
 *   - ACMH's refinement with the fused sweep.
 * A call that would make one of these is refused and changes nothing.  gpm_set_geometric, gpm_set_photometric,
 * gpm_set_propagation, gpm_set_view_selection, gpm_set_prior, gpm_set_geo_mask, gpm_set_refinement and
 * gpm_set_option("neighbours") return
 * GPM_E_ARG, whichever of the two fields is set last.  A colour image upload (gpm_set_reference_color, gpm_set_view_color) returns GPM_E_ARG
 * while joint view selection or the planar prior is on and GPM_E_STATE while only the NCC cost is.  The batch drivers
 * refuse the same combinations of their job options and image type with GPM_E_ARG before any CUDA call.
 * The source-view shard runs neither the geometric term, the NCC cost, joint view selection nor the planar prior: while one
 * is on, every
 * gpm_shard_* call taking a context returns GPM_E_STATE (gpm_shard_num_stages and gpm_shard_stage_floats return -1), and
 * gpm_set_geometric refuses to turn the term on with GPM_E_STATE once a shard communicator is set.  gpm_shard_stage,
 * gpm_shard_finish_init and gpm_shard_run refuse the fused sweep with GPM_E_ARG.  The shard exchanges Gipuma's refinement
 * steps one by one: while ACMH's refinement is on, every gpm_shard_* call taking a context returns GPM_E_STATE as well. */

/* ---- geometric consistency (DESIGN.md §14) ----------------------------------------------------------------------------
 * A second PatchMatch pass may score each hypothesis against the source views' own depth maps as well: with weight > 0 the
 * cost of view j becomes photo_j + g_j, g_j = weight * min(err, max_err), where err is the forward-backward reprojection
 * error in pixels of the hypothesis' point through view j's depth map (weight * max_err where that depth is missing, out of
 * [depthMin, depthMax] or the point is off-image or behind a camera).  The views are combined as before.  Every cost the
 * context computes (gpm_init, gpm_sweep, gpm_phase, gpm_cost_eval, gpm_run) uses it while it is on.
 * gpm_set_view_depth: view v's depth map, width x height floats (pitch_bytes between rows, 0 = packed; host or device
 *   memory), each pixel's depth along view v's own optical axis as gpm_finalize writes it (0 = no depth).  The cameras are
 *   those of gpm_set_view (K^-1 included) and the reference's K.  Storage is allocated by the first call.
 * gpm_set_geometric: weight 0 (the default) turns the mode off and gives exactly the photometric cost.  Refused with
 *   GPM_E_ARG: weight negative or not finite, max_err not finite or <= 0; with GPM_E_STATE: a used view (0 .. n_views-1)
 *   without a depth map — also at the next launch, if gpm_set_num_views adds one.  Other modes: "mode compatibility". */
int gpm_set_view_depth(gpm_ctx* ctx, int v, const float* depth, size_t pitch_bytes, int on_device);
int gpm_set_geometric(gpm_ctx* ctx, float weight, float max_err);

/* gpm_set_geo_mask (DESIGN.md §21): a per-pixel mask of the geometric term, width x height bytes (pitch_bytes between rows,
 * 0 = packed; host or device memory), copied.  While the term is on, every cost the context computes (gpm_init, gpm_sweep,
 * gpm_phase, gpm_cost_eval, gpm_run) is at a pixel whose byte is nonzero exactly the cost with the term off, and elsewhere
 * exactly the cost with it on.  NULL clears the mask (the default: no mask).  While the term is off the mask has no
 * effect; while it is on, setting, changing or clearing the mask marks stored costs and the memo stale.  Refused with
 * GPM_E_ARG: a mask while the planar prior is on, pitch_bytes smaller than width.  A refused call changes nothing;
 * gpm_set_prior refuses to turn the prior on while a mask is set. */
int gpm_set_geo_mask(gpm_ctx* ctx, const unsigned char* mask, size_t pitch_bytes, int on_device);

/* ---- photometric cost (DESIGN.md §15) ---------------------------------------------------------------------------------
 * GPM_PHOTO_PM (the default) is the reference's adaptive-support-weight cost.  GPM_PHOTO_NCC replaces each view's cost by
 * 1 - the support-weighted normalised cross-correlation of the window (clamped to [0, 2]), which a gain and an offset of the
 * source image leave unchanged; a window whose weighted standard deviation, in the reference or the source view, is below
 * min_std grey levels costs 2.  Grey images and the 8-neighbour sweep only.  With the geometric mode on, view j's cost is
 * ncc_j + g_j.  The lower-bound early-out (option "prune") has no effect on NCC costs.  min_std is ignored for PM.
 * Refused with GPM_E_ARG: an unknown kind; NCC with min_std not finite or <= 0.  Other modes: "mode compatibility".  A
 * refused call changes nothing. */
enum { GPM_PHOTO_PM = 0, GPM_PHOTO_NCC = 1 };
int gpm_set_photometric(gpm_ctx* ctx, int kind, float min_std);

/* ---- propagation (DESIGN.md §16) ----------------------------------------------------------------------------------------
 * GPM_PROP_FIXED (the default) offers each pixel the reference's 8 neighbours: the other-colour pixels at 1 px (close) and
 * 5 px (far) up, down, left and right.  GPM_PROP_ADAPTIVE is the adaptive checkerboard sampling of ACMH (Xu & Tao, CVPR
 * 2019): candidate k is instead the pixel with the lowest stored cost, at the start of the launch, in region k: four
 * V-shaped regions of 7 pixels reaching 4 px (close) and four axial strips of 11 pixels at 3, 5, .., 23 px (far).  NaN
 * costs count as +inf and a tie goes to the earliest pixel of the region's scan order.  The accept rule, the refinement and
 * every cost are unchanged, so the mode may be switched at any point of a run and works with every cost mode, grey or
 * colour, and with the source-view shard (gpm_shard_*).
 * Refused with GPM_E_ARG: an unknown kind.  Other modes: "mode compatibility".  A refused call changes nothing. */
enum { GPM_PROP_FIXED = 0, GPM_PROP_ADAPTIVE = 1 };
int gpm_set_propagation(gpm_ctx* ctx, int kind);

/* ---- view selection (DESIGN.md §17) ------------------------------------------------------------------------------------
 * GPM_VSEL_OFF (the default) scores every hypothesis by the combination rule of gpm_params (cost_comb, n_best): each
 * hypothesis picks its own views.  GPM_VSEL_JOINT is the multi-hypothesis joint view selection of ACMH (Xu & Tao, CVPR
 * 2019): per pixel and launch, the per-view NCC costs m[k][j] of the offered in-range candidates k decide one weight per
 * view j.  With good_j = #{k : m < tau_t}, bad_j = #{k : m > tau_bad} and s_j the sum of exp(-m^2 / (2 beta^2)) over the good
 * entries, w_j = s_j / good_j if good_j >= n_good and bad_j < n_bad; else w_keep if view j was selected at this pixel by the
 * last JVS launch and bad_j < n_bad; else 0.  tau_t = tau_init * exp(-t^2 / alpha), where t counts the iterations of
 * gpm_sweep since gpm_init or gpm_set_state.  Every hypothesis of the pixel, the current plane included, then costs
 * sum_j w_j c_j / sum_j w_j (c_j = m_j + g_j with the geometric term), or the combination rule where every w_j is 0.  The
 * selected-views masks are cleared by gpm_init, gpm_set_state and a switch from OFF to JOINT; a switch either way marks the
 * stored costs stale.  NCC cost, grey images and the 8-neighbour sweep only; fixed or adaptive propagation, with or without
 * the geometric term.
 * Refused with GPM_E_ARG: a NULL `vsel`, an unknown kind; for JOINT, tau_init, alpha, tau_bad or beta not finite or <= 0,
 * w_keep not finite or < 0, n_good outside 1..8, n_bad outside 1..9.  Other modes: "mode compatibility".  A refused call
 * changes nothing. */
enum { GPM_VSEL_OFF = 0, GPM_VSEL_JOINT = 1 };
typedef struct gpm_view_sel {
    int kind;                          /* GPM_VSEL_OFF or GPM_VSEL_JOINT */
    float tau_init;                    /* starting good threshold (ACMH: 0.8) */
    float alpha;                       /* how fast the good threshold shrinks (90) */
    float tau_bad;                     /* bad threshold (1.2) */
    int n_good;                        /* a view needs at least n_good good candidates (3) */
    int n_bad;                         /* ... and fewer than n_bad bad ones (3) */
    float beta;                        /* width of the confidence function (0.3) */
    float w_keep;                      /* weight of a remembered view (0.2) */
} gpm_view_sel;
int gpm_set_view_selection(gpm_ctx* ctx, const gpm_view_sel* vsel);
/* The selected-views mask of every pixel ([height*width], bit j = view j), host memory; all zero before the first JOINT
 * launch. */
int gpm_get_view_masks(gpm_ctx* ctx, unsigned long long* masks);

/* ---- refinement (DESIGN.md §23) ----------------------------------------------------------------------------------------
 * GPM_REFINE_GIPUMA (the default) refines each pixel with Gipuma's steps of shrinking random offsets (gipuma.cu:928-994),
 * drawn as gpm_set_rng's mode says.  GPM_REFINE_ACMH is the multi-hypothesis refinement of ACMH (Xu & Tao, CVPR 2019): from
 * the pixel's plane (n, depth d at the pixel) at the start of its refinement it tries, in this order, (d_r, n), (d, n_r),
 * (d_r, n_r), (d, n_t), (d_t, n), each accepted when its cost is strictly below the running cost: d_r uniform in disparity
 * on [min_disparity, max_disparity], n_r a uniform camera-facing unit normal, d_t = clamp(d (1 + perturbation U(-1, 1)),
 * depthMin, depthMax), n_t = n + perturbation * pi * U(-1, 1) per component, normalised and facing the camera.  Its draws
 * are a stateless hash of (gpm_set_rng's seed, pixel, launch counter, draw index), the same in both RNG modes; the launch
 * counter counts the gpm_sweep / gpm_phase launches with refinement since gpm_init, gpm_init_planes or gpm_set_rng.  Every
 * cost mode, grey or colour, and both propagation modes; not the fused sweep or the source-view shard.  A switch marks
 * nothing stale: only the candidates change.
 * Refused with GPM_E_ARG: an unknown kind, a perturbation not finite or outside (0, 1).  Other modes: "mode
 * compatibility".  A refused call changes nothing. */
enum { GPM_REFINE_GIPUMA = 0, GPM_REFINE_ACMH = 1 };
int gpm_set_refinement(gpm_ctx* ctx, int kind, float perturbation);

/* Seed of the per-pixel curand_init(seed, y, x) at initialisation (gipuma.cu:1019; the reference uses
 * clock64()) and the refinement RNG mode. */
int gpm_set_rng(gpm_ctx* ctx, unsigned long long seed, int mode);

/* Overwrite / read the raw per-pixel state: planes [height*width] float4 (n.xyz in the reference
 * camera frame, w = plane distance d) and costs [height*width] float, both row-major with stride =
 * width — the LineState layout (linestate.h:8-24).  Either pointer may be NULL. */
int gpm_set_state(gpm_ctx* ctx, const float* norm4, const float* cost, int on_device);
int gpm_get_state(gpm_ctx* ctx, float* norm4, float* cost, int on_device);

/* gipuma_init_cu2 (gipuma.cu:996-1051): random plane + initial cost for every pixel. */
int gpm_init(gpm_ctx* ctx);

/* `iterations` red/black sweeps (gipuma.cu:1911-1941).  One iteration = black{close,far,refine} then
 * red{close,far,refine}; the three phases of a colour are fused into one launch. */
int gpm_sweep(gpm_ctx* ctx, int iterations);

/* One phase of one colour, for step-level parity tests: colour 0 = black, 1 = red;
 * phase_mask bit0 = close (gipuma.cu:1471-1588), bit1 = far (:1353-1468), bit2 = refine (:1590-1711). */
int gpm_phase(gpm_ctx* ctx, int colour, int phase_mask);

/* gipuma_compute_disp (gipuma.cu:1080-1103): normals to world frame, w <- depth (0 where cost == MAXCOST). */
int gpm_finalize(gpm_ctx* ctx);

/* Multi-view cost of caller-supplied planes at every pixel (no accept logic) — pmCostMultiview_cu
 * (gipuma.cu:720-806) through the iteration-time path; `planes`/`out_cost` like gpm_set_state. */
int gpm_cost_eval(gpm_ctx* ctx, const float* planes, float* out_cost, int on_device);

/* Whole job as runcuda() does it: init, params.iterations sweeps, finalize; results are left in the
 * context (gpm_get_state).  `sweep_ms` (may be NULL) receives the CUDA-event time from the first sweep
 * kernel to the end of the final kernel — the reference's own timed span (gipuma.cu:1908-1952). */
int gpm_run(gpm_ctx* ctx, float* sweep_ms);

/* ---- source-view sharding across GPUs (SURVEY.md §8e; cost_comb = best_n only) --------------------------------
 * The reference is single-GPU (main.cpp:658-692); what is preserved is pmCostMultiview_cu's combination over ALL views
 * (gipuma.cu:742-806).  Each rank creates a context holding ALL of the state but only ITS subset of the source views
 * (gpm_set_view / gpm_set_num_views with the local views; same parameters, reference image and seed everywhere).
 *
 * High level — the whole runcuda() flow, exchange included, behind the C-ABI (a C++ host needs nothing else):
 *   gpm_shard_unique_id(id)           rank 0: 128-byte NCCL unique id; distribute it to the other ranks by any means
 *   gpm_shard_comm_init(ctx, id, r, n) every rank: ncclCommInitRank on the context's device (n = 1: no communicator)
 *   gpm_shard_comm_attach(ctx, comm, r, n)   alternative: use an existing ncclComm_t of the shard group
 *   gpm_shard_run(ctx, &ms)           init planes, initial costs, params.iterations sweeps, final kernel; per exchange
 *                                     stage one ncclAllGather of the local top-n_best lists on the context's stream; no
 *                                     host synchronisation in between.  Output bit-identical to gpm_run over all views.
 * NCCL is loaded at run time (dlopen "libnccl.so.2", override with GPM_NCCL_LIB); the library itself links only cudart.
 *
 * Low level (tests, custom transports): per stage, gpm_shard_stage applies the accept of the PREVIOUS stage from
 * `gathered_prev_dev` (rank-major concatenation of every rank's lists; ignored for stages 0 and 1) and writes this
 * rank's ascending n_best smallest per-view costs per pixel and hypothesis slot of THIS stage into `xchg_dev`
 * (gpm_shard_stage_floats(stage) floats, device memory).  Stages per colour: 1 (8 propagation candidates), then
 * 2 .. gpm_shard_num_stages()-1 (refinement steps, sequential), then gpm_shard_num_stages() (closing accept only, no
 * output).  Stage 0 evaluates the initial costs after gpm_init_planes (both colours at once; `colour` ignored) and is
 * closed by gpm_shard_finish_init. */
int gpm_init_planes(gpm_ctx* ctx);
int gpm_shard_num_stages(gpm_ctx* ctx);
long long gpm_shard_stage_floats(gpm_ctx* ctx, int stage);
int gpm_shard_stage(gpm_ctx* ctx, int colour, int stage, const float* gathered_prev_dev, int world, float* xchg_dev);
int gpm_shard_finish_init(gpm_ctx* ctx, const float* gathered_dev, int world);
int gpm_shard_unique_id(void* id128);
int gpm_shard_comm_init(gpm_ctx* ctx, const void* id128, int rank, int world);
int gpm_shard_comm_attach(gpm_ctx* ctx, void* nccl_comm, int rank, int world);
int gpm_shard_run(gpm_ctx* ctx, float* sweep_ms);

/* Counters of the last gpm_sweep/gpm_run: [0] kernels launched, [1] hypotheses offered,
 * [2] hypotheses skipped as exact duplicates / out of depth range, [3] hypotheses cut short by the
 * exact lower bound, [4] (view,sample) evaluations done, [5] (view,sample) evaluations a full run would do,
 * [6] collectives issued by gpm_shard_run. */
int gpm_get_stats(gpm_ctx* ctx, unsigned long long stats[8]);
int gpm_reset_stats(gpm_ctx* ctx);

/* Measured ceiling of the unit that bounds this path: filtered R32F fetches per second (in 1e9) of the texture unit for
 * dense footprints on this context's own source-view texture (a ~30 ms microbenchmark; needs the views set).
 * bench.py's roofline.binding_unit divides the achieved fetch rate by it. */
int gpm_measure_fetch_peak(gpm_ctx* ctx, double* gfetch_per_s);

/* Tuning / diagnostics; results are bit-identical for every setting.
 * "prune" (1): exact lower-bound early-out; "dedupe" (1): skip bit-identical candidate planes;
 * "trust_state" (0): treat a state loaded with gpm_set_state as cost-consistent; "nwarps" (0 = auto): warps per block;
 * "memo" (1): skip candidates / refinements this pixel is already known to reject (exact); "cost_variant" (-1 = auto):
 * which of the reference binary's rounding variants gpm_cost_eval reproduces (DESIGN.md §2): bit 0 = x-term first (float: 1 in the propagation kernels, 0 at init / refinement; float4: 0 in
 * all six sweep kernels), bit 1 = float4 gradient folding (float4 initialisation = 3); auto = the propagation kernels' form;
 * "quadperm" (1): deal the samples of a round to the lanes as 2x2 blocks per hardware quad (texture-unit locality);
 * "neighbours" (8): 20 selects the reference's fused sweep — the kernels it launches when built without SMALLKERNEL
 * (gipuma.cu:1122-1351, 1913-1940): 12 axial + 8 knight-move neighbours, then refinement, one launch per colour; bit-exact
 * like the default (view sharding stays 8-neighbour only). */
int gpm_set_option(gpm_ctx* ctx, const char* name, int value);

/* The CUDA stream all work of this context is enqueued on (as a void*), for event timing by callers. */
void* gpm_stream(gpm_ctx* ctx);

/* ---- callers and data formats either side of the hot path (SURVEY.md §8f rows f1-f3; plain host C++, no CUDA) ------
 * gpm_prepare_cameras: n row-major 3x4 projection matrices (index 0 = reference) -> the Camera_cu field values, without
 *   OpenCV (cameraGeometryUtils.h:174-353: RQ decomposition, re-basing so that the reference is K[I|0], baseline 0.54).
 * gpm_select_views: deterministic selectViews (main.cpp:430-499); returns the number of views written to `subset`.
 * gpm_write_dmb / gpm_read_dmb / gpm_write_result_dmb: the .dmb depth / normal maps consumed by `fusibile`
 *   (fileIoUtils.h:247-368; scripts/dtu_fast.sh:57). */
int gpm_prepare_cameras(const double* P, int n, double cam_scale, gpm_camera* out);
int gpm_select_views(const gpm_camera* cams, int n, int cols, int rows, float min_angle, float max_angle, int max_views,
                     int* subset, float* depth_range);
int gpm_write_dmb(const char* path, const float* data, int rows, int cols, int channels);
int gpm_read_dmb(const char* path, float* data, size_t capacity_floats, int* rows, int* cols, int* channels);
int gpm_write_result_dmb(const char* depth_path, const char* normal_path, const float* norm4, int rows, int cols);

/* ---- reference-view batch driver (SURVEY.md §8f row f2): replaces the shell loop that starts one `gipuma` process per
 * reference image (scripts/dtu_fast.sh:30-55) and the view selection of main.cpp:430-499 ------------------------------
 * One process, a worker thread + gpm_ctx per listed device, ONE page-locked copy of the image set shared by all of them
 * (each image is registered once, uploaded asynchronously by whichever device needs it), reference views taken from a
 * common queue.  Per reference view: cameras re-based on it (gpm_prepare_cameras), source views selected
 * (gpm_select_views), depth range as main.cpp:480-483 / 898-906, gpm_run, result returned and / or written as
 * <out_dir>/<ref, 8 digits>/{disp,normals}.dmb (main.cpp:1002-1003) for the external fusibile. */
typedef struct gpm_batch_desc {
    int n_images, width, height;
    const float* const* images;        /* n_images host pointers, row-major float, pitch_bytes between rows (0 = width*4) */
    size_t pitch_bytes;
    const double* P;                   /* n_images row-major 3x4 projection matrices */
    double cam_scale;                  /* --cam_scale (K divided by it); <= 0 means 1 */
    gpm_params params;                 /* depthMin / depthMax <= 0: taken from the view selection; disparities are derived */
    float min_angle, max_angle;        /* degrees (scripts/dtu_fast.sh:18-19) */
    int max_views;                     /* scripts/dtu_fast.sh:21 */
    const int* ref_indices;            /* reference views to process (NULL: 0 .. n_refs-1) */
    int n_refs;
    const int* devices;                /* CUDA device ordinals, one worker each */
    int n_devices;
    unsigned long long seed;
    const char* out_dir;               /* NULL: no files; else list each reference view once (a repeated one is written by two jobs, possibly at once) */
    float* out_norm4;                  /* NULL or n_refs * height*width*4 floats (world normal + depth per job) */
    float* out_cost;                   /* NULL or n_refs * height*width floats */
} gpm_batch_desc;
typedef struct gpm_batch_stats {
    int jobs_done;
    double sweep_ms_total;             /* sum of the jobs' device times (reference's own span) */
    float* per_job_sweep_ms;           /* NULL or n_refs entries */
    int* per_job_views;                /* NULL or n_refs entries: source views selected */
    int* per_job_device;               /* NULL or n_refs entries: device that ran the job */
} gpm_batch_stats;
int gpm_batch_run(const gpm_batch_desc* desc, gpm_batch_stats* stats);
const char* gpm_batch_last_error(void);

/* Two-pass geometric-consistency batch (DESIGN.md §14) on the same worker pool and shared image cache.  Pass 1, for the
 * reference views and every view their selection picks (not recursive), on whichever worker takes the view: gpm_batch_run's
 * per-view setup, gpm_init, gpm_sweep(params.iterations), gpm_get_state (raw planes, reference views only), gpm_finalize,
 * gpm_get_state (depth map), kept in one page-locked host store for the call (about 4 + 16 bytes per pixel and view).  All
 * workers finish pass 1 before any pass-2 job starts.  Pass 2, per reference view: the same setup, gpm_set_view_depth of
 * every selected view's pass-1 depth map, gpm_set_geometric(weight, max_err), gpm_cost_eval of the raw planes and
 * gpm_set_state of the planes with those costs, gpm_sweep(geo_iterations), gpm_finalize, gpm_get_state into out_norm4 /
 * out_cost, the .dmb files as gpm_batch_run writes them, gpm_set_geometric(0, max_err).  Sweep times are CUDA events on
 * gpm_stream around each gpm_sweep.
 * Refused with GPM_E_ARG before any CUDA call: what gpm_batch_run refuses, a reference index out of range (without
 * ref_indices: n_refs > n_images), a reference view listed twice while out_dir is set, channels other than 1 or 4,
 * geo_iterations < 0, weight / max_err that gpm_set_geometric refuses.  GPM_E_STATE, also before any CUDA call: a pass-1
 * view with no source view passing the angle filter (named in gpm_batch_last_error()).  A failure during the run (e.g.
 * negative params.iterations, which gpm_set_params refuses) stops every worker with GPM_E_STATE; the contexts, the image
 * registrations and the host store are released on every path. */
typedef struct gpm_geo_batch_desc {
    gpm_batch_desc batch;              /* as gpm_batch_run; batch.params.iterations = pass-1 iterations; out_norm4 / out_cost /
                                          out_dir receive the pass-2 results */
    int channels;                      /* 1: batch.images are float images; 4: RGBA float4 images (pitch_bytes 0 = width*16) */
    int geo_iterations;                /* pass-2 sweeps, >= 0 */
    float weight, max_err;             /* as gpm_set_geometric */
} gpm_geo_batch_desc;
typedef struct gpm_geo_batch_stats {
    gpm_batch_stats batch;             /* per reference job: pass-2 sweep ms, views selected, device */
    int n_pass1;                       /* views pass 1 ran */
    int* pass1_views;                  /* NULL or n_images entries: those views, ascending */
    float* pass1_sweep_ms;             /* NULL or n_images entries, in the order of pass1_views */
    int* ref_views;                    /* NULL or n_refs * max_views image indices of each job's selected views, -1 after the last */
} gpm_geo_batch_stats;
int gpm_geo_batch_run(const gpm_geo_batch_desc* desc, gpm_geo_batch_stats* stats);

/* The batch drivers with a choice of photometric cost: every job's context gets gpm_set_photometric(kind, min_std) in the
 * per-view setup (both passes of the geometric driver).  gpm_batch_run and gpm_geo_batch_run are these with GPM_PHOTO_PM.
 * Refused with GPM_E_ARG before any CUDA call, besides what those refuse: what gpm_set_photometric refuses for its
 * arguments, and the combinations "mode compatibility" excludes. */
int gpm_batch_run_photo(const gpm_batch_desc* desc, int kind, float min_std, gpm_batch_stats* stats);
int gpm_geo_batch_run_photo(const gpm_geo_batch_desc* desc, int kind, float min_std, gpm_geo_batch_stats* stats);

/* The batch drivers with per-job options: every job's context gets gpm_set_photometric(photometric, ncc_min_std) and
 * gpm_set_propagation(propagation) in the per-view setup (both passes of the geometric driver).  The _photo twins are these
 * with GPM_PROP_FIXED.  Refused with GPM_E_ARG before any CUDA call, besides what those refuse: what the two setters refuse
 * for their arguments, and a NULL `opts`. */
typedef struct gpm_job_opts {
    int photometric;                   /* GPM_PHOTO_PM or GPM_PHOTO_NCC */
    float ncc_min_std;                 /* as gpm_set_photometric (ignored for PM) */
    int propagation;                   /* GPM_PROP_FIXED or GPM_PROP_ADAPTIVE */
} gpm_job_opts;
int gpm_batch_run_opts(const gpm_batch_desc* desc, const gpm_job_opts* opts, gpm_batch_stats* stats);
int gpm_geo_batch_run_opts(const gpm_geo_batch_desc* desc, const gpm_job_opts* opts, gpm_geo_batch_stats* stats);

/* The batch drivers with a view selection (DESIGN.md §17): every job's context also gets gpm_set_view_selection(vsel) in
 * the per-view setup (both passes of the geometric driver; pass 2 starts at t = 0 after its gpm_set_state).  vsel = NULL
 * is GPM_VSEL_OFF: the _opts drivers are these with NULL.  Refused with GPM_E_ARG before any CUDA call, besides what the
 * _opts drivers refuse: what gpm_set_view_selection refuses for its arguments. */
int gpm_batch_run_vsel(const gpm_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel, gpm_batch_stats* stats);
int gpm_geo_batch_run_vsel(const gpm_geo_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                           gpm_geo_batch_stats* stats);

/* ---- depth-map fusion: the per-view world-frame outputs (norm4 of gpm_batch_run, or its .dmb files) -> one point cloud;
 * what the reference's scripts hand to the external `fusibile` (scripts/dtu_fast.sh:56-57).  Deterministic: the same inputs
 * give the same vertices, in the same order, on every run.  The algorithm is specified in DESIGN.md §12; in short, views are
 * processed in ascending order as reference; a valid, unused reference pixel back-projects to X (get3Dpoint in the un-rebased
 * world frame), X is projected into every other view j and rounded to the nearest pixel, and j is consistent when that pixel
 * is inside the image, X is in front of camera j, the pixel's depth is in [depth_min, depth_max], the disparities
 * f_j*0.54/z of X and of the pixel differ by less than disp_thresh and the normals are less than normal_thresh degrees apart
 * (the disparity rule; gpm_fuse_with_rule below selects the scale-free reprojection rule instead).
 * With at least num_consistent consistent views one vertex is emitted (mean position, normalised normal sum, mean colour)
 * and the pixels involved are marked used; a mark only stops a pixel from being a reference in later passes.
 * Vertices are emitted in (reference view, y, x) order. */
#define GPM_FUSE_MAX_VIEWS   256      /* views held in one block's shared-memory camera table */
#define GPM_FUSE_VERTEX_BYTES 27      /* float x, y, z, nx, ny, nz; uchar red, green, blue; packed, little-endian (storePlyFileBinary) */

/* Per-view camera of the fusion, in the un-rebased world frame (getCameraParameters(..., transformP = false),
 * cameraGeometryUtils.h:174-353): P = K_scaled [R | t] with K[2][2] = 1 and K's focal lengths and principal point divided
 * by cam_scale as gpm_prepare_cameras does; M_inv = inverse of P's left 3x3; f = K_scaled[0][0]. */
typedef struct gpm_fuse_camera {
    float M_inv[9];
    float P[12];                       /* row-major 3x4 */
    float f;
} gpm_fuse_camera;
int gpm_fuse_cameras(const double* P, int n, double cam_scale, gpm_fuse_camera* out);

typedef struct gpm_fuse_desc {
    int n_views, width, height;        /* 2 <= n_views <= GPM_FUSE_MAX_VIEWS */
    const float* norm4;                /* n_views * height*width * 4 floats: world normal xyz + depth (0 = invalid) per pixel */
    const float* images;               /* NULL (black vertices) or n_views * height*width * channels floats, values in [0, 255] */
    int channels;                      /* 1 = grey (red = green = blue), 4 = RGBA float4 (x, y, z -> red, green, blue; w unused) */
    int on_device;                     /* norm4 and images are device pointers on `device` (1) or host memory (0) */
    const double* P;                   /* n_views row-major 3x4 projection matrices, as passed to gpm_batch_run */
    double cam_scale;                  /* > 0, as gpm_prepare_cameras */
    float depth_min, depth_max;        /* 0 <= depth_min < depth_max */
    float disp_thresh;                 /* > 0, in pixels of disparity */
    float normal_thresh;               /* degrees, in (0, 180] */
    int num_consistent;                /* >= 1 other views */
    int device;                        /* CUDA device ordinal */
} gpm_fuse_desc;

/* Caller-sized result.  `count` always receives the number of fused vertices.  Up to `capacity` vertices are written to
 * `vertices` (capacity * GPM_FUSE_VERTEX_BYTES bytes) and their sources to `source` (2 ints each: reference view,
 * y*width + x); when count > capacity the call returns GPM_E_ARG after the whole fusion, so a caller may retry with
 * capacity = count.  The number of pixels with depth in [depth_min, depth_max] always suffices.  `used` (NULL or
 * n_views * height*width bytes) receives the final used masks (1 = fused into some vertex).  `fuse_ms` receives the
 * CUDA-event time from the end of the input uploads to the last vertex download, `upload_ms` the time of the uploads of
 * norm4 and images (0 for device inputs).  Fusion allocates its own buffers and stream and frees them before returning. */
typedef struct gpm_fuse_result {
    long long count;
    long long capacity;
    unsigned char* vertices;           /* NULL or capacity * GPM_FUSE_VERTEX_BYTES bytes */
    int* source;                       /* NULL or capacity * 2 ints */
    unsigned char* used;               /* NULL or n_views * height*width bytes */
    float fuse_ms, upload_ms;
} gpm_fuse_result;
int gpm_fuse(const gpm_fuse_desc* desc, gpm_fuse_result* result);

/* The consistency rule of the fusion (DESIGN.md §22).  GPM_FUSE_DISPARITY is the rule above (gpm_fuse).  Under
 * GPM_FUSE_REPROJECTION, view j is consistent with reference pixel p = (x, y) of view r, depth d_r, when X projects into j
 * as above (z > 0, in the image, the pixel's depth in [depth_min, depth_max]) and the back-projection X_j of that pixel
 * (u, v) at its depth, projected back into view r to (x', y') at depth z', satisfies: z' > 0,
 * sqrt(dx*dx + dy*dy) < reproj_px with dx = x' - x, dy = y' - y, |z' - d_r| / d_r < depth_rel, and the normal test above.
 * Every operation of this rule is homogeneous in the world's scale, so its decisions do not depend on it; disp_thresh is
 * not read.  Everything else (cameras, passes, marks, vertex order and averaging) is gpm_fuse's. */
#define GPM_FUSE_DISPARITY    0
#define GPM_FUSE_REPROJECTION 1
typedef struct gpm_fuse_rule {
    int kind;                          /* GPM_FUSE_DISPARITY or GPM_FUSE_REPROJECTION */
    float reproj_px;                   /* REPROJECTION: finite, > 0, in pixels of view r */
    float depth_rel;                   /* REPROJECTION: finite, > 0, relative to d_r */
} gpm_fuse_rule;
/* gpm_fuse under `rule`; a NULL rule is gpm_fuse.  Refused with GPM_E_ARG before any CUDA call, besides what gpm_fuse
 * refuses (except disp_thresh under REPROJECTION): an unknown kind; for REPROJECTION, reproj_px or depth_rel not finite
 * or <= 0. */
int gpm_fuse_with_rule(const gpm_fuse_desc* desc, const gpm_fuse_rule* rule, gpm_fuse_result* result);

/* Binary little-endian PLY with the header of storePlyFileBinary (displayUtils.h:84-97) and `count` packed vertices. */
int gpm_write_ply(const char* path, const unsigned char* vertices, long long count);

/* ---- point-cloud distances: the exact distance from every query point to its nearest data point, the one operation behind
 * accuracy / completeness / F-score of a reconstructed cloud against ground truth (DESIGN.md §13).  fp32, one IEEE
 * round-to-nearest step per operation: dx = q.x - b.x (likewise y, z), d2 = (dx*dx + dy*dy) + dz*dz, m = min over the data
 * of d2, D = sqrt(m); dist = D if D <= max_dist, else +inf (also for an empty data set).  The search skips data only under a
 * provably conservative bound, so every finite output equals a brute-force evaluation bit for bit; m is a minimum over a set,
 * so the output does not depend on the order of the data, on the run, or on where the inputs live.  Refused with GPM_E_ARG
 * before any search: null pointers, counts outside [0, 2^31 - 1], max_dist not finite and > 0, a non-finite coordinate. */
typedef struct gpm_nn_desc {
    long long n_query, n_data;
    const float* query;                /* n_query * 3 floats: x y z per point */
    const float* data;                 /* n_data * 3 floats */
    int on_device;                     /* query, data and result->dist are device pointers on `device` (1) or host memory (0) */
    int device;                        /* CUDA device ordinal */
    float max_dist;                    /* finite, > 0 */
} gpm_nn_desc;

/* `dist` (n_query floats) is caller memory of the inputs' kind.  The times are CUDA events: upload_ms the host-to-device
 * copies of query and data (0 for device inputs), build_ms the validation pass and the grid over the data, query_ms the
 * search.  cell_size and n_cells describe the grid that was built.  The call allocates its own buffers and stream and frees
 * them before returning. */
typedef struct gpm_nn_result {
    float* dist;
    float upload_ms, build_ms, query_ms;
    float cell_size;
    long long n_cells;
} gpm_nn_result;
int gpm_nearest_dist(const gpm_nn_desc* desc, gpm_nn_result* result);

/* ---- meshing (DESIGN.md §24): depth maps -> truncated signed distance volume -> triangle mesh.  Both stages are fp32, one
 * IEEE round-to-nearest step per operation in the order DESIGN.md §24 states, so they are deterministic and independent of
 * where the inputs live.  The volume is an axis-aligned box of nx * ny * nz voxels (each in 2..2048, at most 2^31 - 1 in
 * all) of edge `voxel`; voxel (i, j, k) has its centre at origin + ((i, j, k) + 0.5) * voxel and is element
 * (k * ny + j) * nx + i of every volume (x fastest). */
#define GPM_MESH_MAX_DIM 2048

/* TSDF integration.  Per voxel centre X and view n in ascending order: h = P_n [X, 1] (the fusion's camera, gpm_fuse_cameras)
 * and z = h_2; the view is skipped unless z > 0, the pixel u = floor(h0/z + 0.5), v = floor(h1/z + 0.5) is in the image, its
 * depth d is > 0 and in [depth_min, depth_max], and sdf = d - z >= -trunc.  Otherwise S += min(sdf, trunc) / trunc and
 * Wt += 1.  D = S / Wt, a NaN (bits 0x7fffffff) where Wt = 0. */
typedef struct gpm_tsdf_desc {
    int n_views, width, height;        /* 1 <= n_views <= GPM_FUSE_MAX_VIEWS */
    const float* depth;                /* n_views * height*width floats: depth along each camera's z axis (norm4.w) */
    int on_device;                     /* depth, result->D and result->weight are device pointers on `device` (1) or host (0) */
    const double* P;                   /* n_views row-major 3x4 projection matrices, as passed to gpm_batch_run */
    double cam_scale;                  /* > 0, as gpm_fuse_cameras */
    float depth_min, depth_max;        /* finite, 0 <= depth_min < depth_max */
    float origin[3];                   /* finite: the corner of the box, world units */
    float voxel;                       /* finite, > 0 */
    int dims[3];                       /* nx, ny, nz */
    float trunc;                       /* finite, > 0, world units */
    int device;                        /* CUDA device ordinal */
} gpm_tsdf_desc;

/* D (nz*ny*nx floats) and weight (nz*ny*nx uint16) are caller memory of the inputs' kind.  upload_ms: the depth maps'
 * host-to-device copy (0 for device inputs); integrate_ms: the integration kernel.  CUDA events. */
typedef struct gpm_tsdf_result {
    float* D;
    unsigned short* weight;
    float upload_ms, integrate_ms;
} gpm_tsdf_result;
/* Refused with GPM_E_ARG before any CUDA call: null pointers, n_views outside 1..GPM_FUSE_MAX_VIEWS, an image size < 1 or
 * over 2^30 pixels, dims outside 2..GPM_MESH_MAX_DIM or over 2^31 - 1 voxels, voxel or trunc not finite or <= 0, a
 * non-finite origin, a bad depth range, a projection matrix gpm_fuse_cameras refuses.  The call allocates its own stream
 * and buffers and frees them before returning; an allocation failure is GPM_E_CUDA. */
int gpm_tsdf_integrate(const gpm_tsdf_desc* desc, gpm_tsdf_result* result);

/* Surface extraction by marching tetrahedra on the lattice of voxel centres.  A point is valid when weight >= min_weight
 * and inside when D < 0 (so -0.0 is outside).  Each cube of 8 neighbouring points splits into the 6 Kuhn tetrahedra
 * 0, e_a, e_a + e_b, 1 for the axis permutations (a, b, c) = xyz, xzy, yxz, yzx, zxy, zyx in that order; a tetrahedron is
 * meshed when its 4 corners are valid.  Each crossing edge (one corner inside, one outside) of a meshed tetrahedron gives
 * one vertex, identified by its lower end p and its direction (x, y, z, x+y, x+z, y+z, x+y+z), at x_p + t (x_q - x_p)
 * per axis with t = D_p / (D_p - D_q); vertex ids run in (lattice index of p, direction) order.  A meshed tetrahedron with
 * 1 or 3 inside corners gives 1 triangle, with 2 gives 2 (the split of DESIGN.md §24); faces wind counter-clockwise seen
 * from outside and come in (cube, tetrahedron) order. */
typedef struct gpm_mesh_desc {
    const float* D;                    /* nz*ny*nx floats */
    const unsigned short* weight;      /* nz*ny*nx */
    int on_device;                     /* D and weight are device pointers on `device` (1) or host memory (0) */
    float origin[3];                   /* finite */
    float voxel;                       /* finite, > 0 */
    int dims[3];                       /* nx, ny, nz */
    int min_weight;                    /* >= 1 */
    int device;                        /* CUDA device ordinal */
} gpm_mesh_desc;

/* Caller-sized host result.  n_vertices and n_faces always receive the counts.  Up to vertex_capacity vertices (3 floats
 * x, y, z each) and face_capacity faces (3 vertex ids each) are written; when a count exceeds its capacity the call
 * returns GPM_E_ARG after the whole extraction, so a caller may retry with the counts.  A mesh of 2^31 or more vertices is
 * refused with GPM_E_ARG (ids are int).  upload_ms: the volumes' host-to-device copies (0 for device inputs); extract_ms:
 * the extraction kernels, up to the downloads.  CUDA events. */
typedef struct gpm_mesh_result {
    long long n_vertices, n_faces;
    long long vertex_capacity, face_capacity;
    float* vertices;                   /* NULL or vertex_capacity * 3 floats */
    int* faces;                        /* NULL or face_capacity * 3 ints */
    float upload_ms, extract_ms;
} gpm_mesh_result;
/* Refused with GPM_E_ARG before any CUDA call: null pointers, dims outside 2..GPM_MESH_MAX_DIM or over 2^31 - 1 points,
 * voxel not finite or <= 0, a non-finite origin, min_weight < 1, a negative capacity or a missing buffer for a positive
 * one.  The call allocates its own stream and buffers and frees them before returning; an allocation failure is
 * GPM_E_CUDA. */
int gpm_mesh_extract(const gpm_mesh_desc* desc, gpm_mesh_result* result);

/* Binary little-endian PLY: `float x, y, z` per vertex, `property list uchar int vertex_indices` per face.  Refused with
 * GPM_E_ARG: negative counts, missing buffers, a face index outside [0, n_vertices). */
int gpm_write_ply_mesh(const char* path, const float* vertices, long long n_vertices, const int* faces, long long n_faces);

const char* gpm_last_error(void);
const char* gpm_version(void);

/* ---- planar prior (DESIGN.md §18) -------------------------------------------------------------------------------------
 * ACMP's planar prior (Xu & Tao, AAAI 2020) as an opt-in mode: a prior map holds one plane per pixel (float4 n.xyz, d in
 * the state's layout; a pixel has a prior where that plane's depth lies in [depthMin, depthMax], so an all-zero entry has
 * none).  While the mode is on (weight > 0), every cost the context computes (gpm_init, gpm_sweep, gpm_phase, gpm_cost_eval,
 * gpm_run, gpm_offer_prior) is c + weight * q / (1 + q) at a pixel with a prior, q = ((depth_h - depth_prior) /
 * depth_sigma)^2 + max(0, 1 - n_h . n_prior) / (1 - cos normal_sigma), and c where c = MAXCOST or the pixel has none.
 * gpm_set_planar_prior: width x height float4 (pitch_bytes between rows, 0 = packed; host or device memory).
 * gpm_get_planar_prior: the map (GPM_E_STATE if none was set or built).
 * gpm_build_planar_prior: the map from the stored planes and costs: per step x step cell the pixel with the smallest cost,
 *   kept if its cost < support_cost and its depth is in range; the Delaunay triangulation of those pixels; each triangle's
 *   plane through the three pixels' points on their own planes, rasterised with the top-left rule.  `info` (may be NULL)
 *   receives the counts.  Refused with GPM_E_ARG: step outside 1..64, support_cost NaN, an image wider or taller than 4097
 *   pixels; with GPM_E_STATE: before gpm_set_params and gpm_set_reference.
 * gpm_set_prior: weight 0 (the default) turns the mode off.  Refused with GPM_E_ARG: weight negative or not finite,
 *   depth_sigma not finite or <= 0, normal_sigma_deg outside (0, 90], a weight with which a valid cost of the current
 *   parameters could reach MAXCOST; with GPM_E_STATE: weight > 0 without a map.  Other modes: "mode compatibility".
 * gpm_offer_prior: every pixel with a prior takes its prior plane (with a fresh identity) where that plane's cost under
 *   the context's mode is strictly below the stored cost.  GPM_E_STATE without a map.
 * A refused call changes nothing. */
typedef struct gpm_prior_build {
    int   step;                        /* cell size in pixels (5) */
    float support_cost;                /* a cell's cheapest pixel is a support point when its cost is below this */
} gpm_prior_build;
typedef struct gpm_prior_info {
    long long support;                 /* support points */
    long long triangles;
    long long with_prior;              /* pixels with a prior */
} gpm_prior_info;
int gpm_set_planar_prior(gpm_ctx* ctx, const float* planes, size_t pitch_bytes, int on_device);
int gpm_get_planar_prior(gpm_ctx* ctx, float* planes, int on_device);
int gpm_build_planar_prior(gpm_ctx* ctx, const gpm_prior_build* build, gpm_prior_info* info);
int gpm_set_prior(gpm_ctx* ctx, float weight, float depth_sigma, float normal_sigma_deg);
int gpm_offer_prior(gpm_ctx* ctx);

/* The batch drivers' prior stage (DESIGN.md §18).  In every photometric job (each job of gpm_batch_run_prior, pass 1 of
 * gpm_geo_batch_run_prior), after params.iterations sweeps: gpm_build_planar_prior (step, support_cost), gpm_set_prior
 * (weight, depth_sigma, normal_sigma_deg), gpm_cost_eval + gpm_set_state of the current planes, gpm_offer_prior,
 * gpm_sweep(iterations); then gpm_finalize and the term off.  Pass 2 of the geometric driver has no prior.  info (may be
 * NULL): one gpm_prior_info per job (gpm_batch_run_prior) or per pass-1 view, in stats->pass1_views' order
 * (gpm_geo_batch_run_prior).  Refused with GPM_E_ARG before any CUDA call: gpm_set_prior's and gpm_build_planar_prior's
 * argument rules, iterations < 0, and the planar prior's mode conflicts (colour images, joint view selection).  The
 * _vsel drivers are these with prior = NULL. */
typedef struct gpm_prior_opts {
    float weight, depth_sigma, normal_sigma_deg;
    int   step;
    float support_cost;
    int   iterations;                  /* sweeps with the prior */
    gpm_prior_info* info;
} gpm_prior_opts;
int gpm_batch_run_prior(const gpm_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel, const gpm_prior_opts* prior,
                        gpm_batch_stats* stats);
int gpm_geo_batch_run_prior(const gpm_geo_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                            const gpm_prior_opts* prior, gpm_geo_batch_stats* stats);

/* ---- coarse-to-fine multi-scale PatchMatch (DESIGN.md §19) ------------------------------------------------------------
 * ACMM's multi-scale scheme (Xu & Tao, CVPR 2019): solve a coarse copy of the images, carry the planes up one level at a
 * time with joint bilateral upsampling, and refine with the geometric term at every level.  Every arithmetic step below is
 * one IEEE fp32 round-to-nearest operation, without contraction, so oracle/pyscale.py restates it bit for bit.
 *
 * gpm_downsample: one pyramid level.  The coarse image is ((width + 1) / 2) x ((height + 1) / 2); coarse pixel (xc, yc) is
 *   centred on fine pixel (2 xc, 2 yc), which is what K / 2 (cam_scale * 2 of gpm_prepare_cameras) describes.  Per channel,
 *   a separable [1, 2, 1] / 4 filter with replicated borders: the horizontal pass of each source row, then the vertical pass,
 *   each (0.25 a + 0.5 b) + 0.25 c.  channels 1 (grey) or 4 (RGBA float4, w filtered like the others); src has pitch_bytes
 *   between rows (0 = packed), dst is packed.  Host or device memory (on_device), on `device`.  Uses its own stream, is
 *   synchronous and frees what it allocates.  Refused with GPM_E_ARG: null pointers, sizes < 1, other channel counts, a pitch
 *   below the row size or not a multiple of 4. */
int gpm_downsample(int device, const float* src, size_t pitch_bytes, int width, int height, int channels, float* dst,
                   int on_device);

/* gpm_upsample_planes: joint bilateral upsampling of a coarse level's raw planes (gpm_get_state's layout, the reference
 *   camera frame, which only K's scale distinguishes between levels) to the level of `ctx`, whose gpm_set_params and
 *   reference (image and camera) give the depth range, the rays and the guide.  For fine pixel p = (x, y) with ray
 *   r = K_inv (x, y, 1): candidates q = (x >> 1, y >> 1) + (i, j), |i|, |j| <= radius, inside the coarse image, visited j
 *   outer, i inner; z_q = -d_q / (n_q . r), used when finite and in [depthMin, depthMax]; w_q = ws * wr with ws =
 *   exp(-((2 q.x - x)^2 + (2 q.y - y)^2) / (2 sigma_space^2)) computed in double and rounded once, and wr = 1 / (1 + dI^2 k),
 *   k = fp32(1 / sigma_range^2), dI = I(p) - I(2 q) in the reference image as uploaded (colour: dI^2 = (dx^2 + dy^2) + dz^2
 *   of x, y, z).  Z = sum w z / sum w, N = sum w n, n = N / |N|, d = -(n . (Z r)); depth Z.  Where the weights sum to 0 (no
 *   candidate) or |N| is not > 0, the pixel gets the plane of (x >> 1, y >> 1) unchanged and depth 0 ("no depth" for
 *   gpm_set_view_depth).  `planes` (W x H float4) and `depth` (W x H float) are caller memory of the input's kind; either
 *   may be NULL.  The context's state, costs, memo, modes and counters are not read or changed.  Refused with GPM_E_ARG:
 *   coarse_w != (W + 1) / 2 or coarse_h != (H + 1) / 2, radius outside 0..4, a sigma not finite or <= 0; GPM_E_STATE:
 *   before gpm_set_params and gpm_set_reference. */
typedef struct gpm_jbu_params {
    int   radius;                      /* coarse pixels either side, 0..4 */
    float sigma_space;                 /* fine pixels, > 0 */
    float sigma_range;                 /* grey levels, > 0 */
} gpm_jbu_params;
int gpm_upsample_planes(gpm_ctx* ctx, const float* coarse, int coarse_w, int coarse_h, int on_device, const gpm_jbu_params* jbu,
                        float* planes, float* depth);

/* gpm_ms_batch_run: the multi-level batch driver, on gpm_batch_run's worker pool and shared image cache.  Planned on the
 * calling thread before any CUDA call: the view set V, the transitive closure of the references' selections (so every view
 * refined at a level has its neighbours' maps of that level), and per view of V its selection and depth range, chosen once on
 * the full-size images and kept at every level; the disparities follow each level's f.  Level l uses cam_scale * 2^l and
 * images downsampled l times with gpm_downsample.  Run, with every worker finishing a stage before the next starts:
 *   1. the pyramid of every image of V, into one page-locked host store;
 *   2. coarsest level, every v in V: gpm_init, params.iterations sweeps, the raw planes kept, gpm_finalize, the depth kept;
 *   3. coarsest level, every v in V: the neighbours' depth maps, gpm_set_geometric(weight, max_err), gpm_cost_eval +
 *      gpm_set_state of the raw planes, geo_iterations sweeps, the raw planes kept;
 *   4. each finer level l, every v in V: gpm_upsample_planes of v's level-(l + 1) planes into planes and a depth map D_l(v);
 *      then every v in V (at level 0 the reference views only, since nothing reads the others' results) as in 3, against
 *      the neighbours' D_l: a Jacobi step, so the result depends neither on scheduling nor on the number of workers.
 * After level 0 each reference view is finalized into out_norm4 / out_cost and the .dmb files, as gpm_geo_batch_run leaves
 * them.  One context per worker and level.  Host store: the raw planes of two adjacent levels, a depth map per view of V
 * and the pyramid, about 1.25 * 16 + 4 + 1.33 * channels bytes per pixel and view.  Refused with GPM_E_ARG before any CUDA
 * call: what gpm_geo_batch_run_vsel refuses, levels outside 1..4, a coarsest level below 8 x 8, gpm_upsample_planes' JBU
 * rules; GPM_E_STATE: a view of V with no source view passing the angle filter, named in gpm_batch_last_error().  A failure
 * during the run stops every worker with GPM_E_STATE, the failing view named; contexts, registrations and stores are
 * released on every path. */
#define GPM_MS_MAX_LEVELS 4
typedef struct gpm_ms_batch_desc {
    gpm_geo_batch_desc geo;            /* batch.params.iterations: photometric sweeps at the coarsest level; geo_iterations:
                                          sweeps with the term at every level; out_* receive the level-0 results */
    int levels;                        /* 1..GPM_MS_MAX_LEVELS; 1 is gpm_geo_batch_run over V */
    gpm_jbu_params jbu;
} gpm_ms_batch_desc;
typedef struct gpm_ms_batch_stats {
    gpm_batch_stats batch;             /* per reference job: level-0 sweep ms, views selected, device */
    int n_views;                       /* |V| */
    int* views;                        /* NULL or n_images entries: V, ascending */
    double level_sweep_ms[GPM_MS_MAX_LEVELS];     /* CUDA-event sweep time summed over the views, per level (0 = full size) */
    double level_upsample_ms[GPM_MS_MAX_LEVELS];  /* host time of the gpm_upsample_planes calls, summed, per level */
} gpm_ms_batch_stats;
int gpm_ms_batch_run(const gpm_ms_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                     gpm_ms_batch_stats* stats);

/* gpm_ms_batch_run_prior: gpm_ms_batch_run with the planar prior (ACMMP: Xu, Kong, Zuo & Tao, TPAMI 2022; DESIGN.md §20).
 * Each stage given is the batch drivers' prior stage (gpm_prior_opts above: build, gpm_set_prior, gpm_cost_eval +
 * gpm_set_state of the current planes, gpm_offer_prior, `iterations` sweeps), and touches only its own view's context, so
 * every level stays a Jacobi step.
 *   photometric: at the coarsest level, in step 2 of gpm_ms_batch_run, after the params.iterations sweeps; then the raw planes
 *     kept, gpm_finalize, the term off, the depth map kept: the coarsest geometric stage reads depth maps made with the prior.
 *   geometric: at every level, in each geometric stage, after the geo_iterations sweeps with the geometric term; then the raw
 *     planes kept (levels > 0) or gpm_finalize and the outputs (level 0); then the term off and the geometric term off.  Its
 *     support points are chosen by the stored costs, which include the geometric term, so support_cost is in those units: a
 *     pixel that is photometrically cheap but geometrically inconsistent is not a support point.
 * info of a stage (NULL or caller memory): photometric n_images entries, by image index; geometric GPM_MS_MAX_LEVELS *
 * n_images entries, [level * n_images + image].  Entries of views or levels that ran no stage are zeroed.  The prior
 * sweeps count in stats->level_sweep_ms and the level-0 per-job sweep ms; level_build_ms receives the host time of the
 * gpm_build_planar_prior calls of both stages, summed over the views, per level.  prior NULL, or both stages NULL, is
 * gpm_ms_batch_run.  Refused with GPM_E_ARG before any CUDA call, besides what gpm_ms_batch_run refuses: per stage given,
 * what gpm_batch_run_prior refuses of its options (so colour images and joint view selection), a weight with which a valid
 * cost could reach MAXCOST (photometric: without the geometric term; geometric: with weight * max_err), and a level that
 * gpm_build_planar_prior refuses, wider or taller than 4097 pixels (photometric: the coarsest; geometric: level 0). */
typedef struct gpm_ms_prior_opts {
    const gpm_prior_opts* photometric; /* NULL: no stage */
    const gpm_prior_opts* geometric;   /* NULL: no stage */
    double level_build_ms[GPM_MS_MAX_LEVELS];     /* out: host time of the gpm_build_planar_prior calls, summed, per level */
} gpm_ms_prior_opts;
int gpm_ms_batch_run_prior(const gpm_ms_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                           gpm_ms_prior_opts* prior, gpm_ms_batch_stats* stats);

/* gpm_ms_batch_run_restore: gpm_ms_batch_run_prior with ACMM's detail restorer (Xu & Tao, CVPR 2019), as the project's own
 * rule (DESIGN.md §21).  Only the level-0 job of each reference view changes, and all of it runs in that job's context:
 *   1. photometric-only estimate: load_view with the geometric term off, gpm_init and photo_iterations sweeps, with the
 *      setup and seed of gpm_geo_batch_run's pass 1 for the view; its raw planes PH kept;
 *   2. the level-0 geometric stage as in gpm_ms_batch_run_prior, the geometric prior stage included; then the prior off
 *      and the raw planes MS kept;
 *   3. detection, with the geometric term off: gpm_cost_eval of MS and of PH gives c_ms and c_ph; a pixel is a detail pixel
 *      where fsub(c_ms, c_ph) > threshold in fp32 (a NaN never is);
 *   4. restore: PH at detail pixels, MS elsewhere; gpm_set_geo_mask of the detail pixels, the term on, gpm_cost_eval +
 *      gpm_set_state of the merged planes, `iterations` sweeps;
 *   5. gpm_finalize, the outputs and .dmb files as before; the mask cleared and the term off.
 * The sweeps of steps 1 and 4 count in level_sweep_ms[0] and the job's sweep ms.  restore NULL is gpm_ms_batch_run_prior.
 * Refused with GPM_E_ARG before any CUDA call, besides what gpm_ms_batch_run_prior refuses: photo_iterations < 1,
 * iterations < 0, a threshold that is not finite.  Memory per worker: one W x H float4 buffer, two W x H cost buffers and
 * the mask, on the host; the host store does not grow. */
typedef struct gpm_ms_restore_opts {
    int   photo_iterations;            /* sweeps of the photometric-only estimate, >= 1 */
    float threshold;                   /* detection threshold, in units of the photometric cost */
    int   iterations;                  /* sweeps after the restore, >= 0 */
    int*  restored;                    /* out, NULL or n_refs entries: detail pixels per reference job */
} gpm_ms_restore_opts;
int gpm_ms_batch_run_restore(const gpm_ms_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                             gpm_ms_prior_opts* prior, const gpm_ms_restore_opts* restore, gpm_ms_batch_stats* stats);

/* ---- the batch drivers' refinement (DESIGN.md §23) ----------------------------------------------------------------------
 * Each _refine entry is the newest entry of its family with gpm_set_refinement(kind, perturbation) in every job's setup,
 * so that every sweep of the job uses it: both passes of the geometric driver, and every level and every stage
 * (photometric, geometric, prior and restorer sweeps) of the multi-level one.  refine NULL is Gipuma's refinement:
 * gpm_batch_run_prior, gpm_geo_batch_run_prior and gpm_ms_batch_run_restore are these with NULL.  Refused with GPM_E_ARG
 * before any CUDA call, besides what those refuse: what gpm_set_refinement refuses of its arguments. */
typedef struct gpm_refine_opts {
    int   kind;                        /* GPM_REFINE_GIPUMA or GPM_REFINE_ACMH */
    float perturbation;                /* in (0, 1); ACMH: 0.02 */
} gpm_refine_opts;
int gpm_batch_run_refine(const gpm_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel, const gpm_prior_opts* prior,
                         const gpm_refine_opts* refine, gpm_batch_stats* stats);
int gpm_geo_batch_run_refine(const gpm_geo_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                             const gpm_prior_opts* prior, const gpm_refine_opts* refine, gpm_geo_batch_stats* stats);
int gpm_ms_batch_run_refine(const gpm_ms_batch_desc* desc, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                            gpm_ms_prior_opts* prior, const gpm_ms_restore_opts* restore, const gpm_refine_opts* refine,
                            gpm_ms_batch_stats* stats);

#ifdef __cplusplus
}
#endif
#endif /* GIPUMA_B200_H */
