// gpm_batch.cpp — reference-view batch driver (SURVEY.md §8f row f2): what the reference does with a shell loop that starts
// one `gipuma` process per reference image (scripts/dtu_fast.sh:30-55 — each of them re-reading every image from disk,
// main.cpp:741-745) done by ONE process: a pool of worker threads, one gpm_ctx per device, that share a single page-locked
// copy of the image set (the "shared image cache": every image is registered once and uploaded with asynchronous copies by
// whichever device needs it) and take reference views from a common queue.  Per reference view the driver re-bases the
// cameras on it (gpm_prepare_cameras, cameraGeometryUtils.h:174-353), selects the source views (gpm_select_views,
// main.cpp:430-499, deterministic), derives the depth / disparity range as main.cpp:480-483 and :898-906 do, runs the job
// (gpm_run) and hands back / writes the result (disp.dmb + normals.dmb, main.cpp:1002-1003, for the external fusibile).
// gpm_geo_batch_run runs the two-pass geometric-consistency flow (DESIGN.md §14) on the same pool and image cache.  The
// _photo twins of both choose the photometric cost (DESIGN.md §15), the _opts ones every per-job option (gpm_job_opts):
// the photometric cost and the propagation mode (§16), the _vsel ones the view selection besides (§17), and the _prior
// ones a planar-prior stage in every photometric job besides (§18).  gpm_ms_batch_run runs the coarse-to-fine multi-scale
// flow (§19) on the same pool: a pyramid of the images, then per level a Jacobi step of upsampling and geometric refinement;
// its _prior twin adds prior stages at the coarsest level's photometric stage and in every geometric stage (§20), and its
// _restore twin the detail restorer at level 0 (§21).
// Host C++ over the C-ABI; the only CUDA calls are page-locking, the geometric drivers' host stores and their sweep events.
#include "../../include/gipuma_b200.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include <sys/stat.h>

namespace gpm {
const char* job_refusal(const gpm_job_opts* o, const gpm_view_sel* v, const gpm_prior_opts* prior, int channels);     // gpm_api.cu
bool prior_bound_ok(const gpm_params& p, bool ncc, float geo_weight, float geo_max_err, float prior_weight);        // gpm_api.cu
const char* refine_refusal(int kind, float perturbation);                                                         // gpm_api.cu
}

namespace {
std::mutex g_err_mutex;
std::string g_batch_err;
void set_err(const std::string& m) { std::lock_guard<std::mutex> l(g_err_mutex);  if (g_batch_err.empty()) g_batch_err = m; }
void clear_err() { std::lock_guard<std::mutex> l(g_err_mutex);  g_batch_err.clear(); }

bool batch_desc_ok(const gpm_batch_desc* d)
{
    return d && d->images && d->P && d->n_images >= 2 && d->width >= 8 && d->height >= 8 && d->n_devices >= 1 && d->devices &&
           d->n_refs >= 1 && d->max_views >= 1 && d->max_views <= GPM_MAX_VIEWS;
}

// One view's job as the reference's main.cpp sets it up: cameras re-based on the view (main.cpp: img_filenames[0] is the
// reference image), the selected source views and the parameters with the depth / disparity range.  Host only.
struct ViewSetup {
    std::vector<double> P;
    std::vector<gpm_camera> cams;       // cams[k]: camera of image order[k], re-based on order[0]
    std::vector<int> order, subset;     // subset[0 .. nv-1]: positions in `order` of the selected source views
    int nv = 0;
    gpm_params p{};
    int source(int v) const { return order[subset[v]]; }
};

// false: no source view passes the angle filter (or the cameras cannot be prepared)
bool plan_view(const gpm_batch_desc* d, int ref, ViewSetup& s)
{
    const int n = d->n_images, W = d->width, H = d->height;
    s.P.resize((size_t)n * 12);  s.cams.resize(n);  s.order.resize(n);  s.subset.resize(n);
    s.order[0] = ref;
    for (int i = 0, k = 1; i < n; i++) if (i != ref) s.order[k++] = i;
    for (int i = 0; i < n; i++) memcpy(&s.P[(size_t)i * 12], d->P + (size_t)s.order[i] * 12, 12 * sizeof(double));
    const int rc = gpm_prepare_cameras(s.P.data(), n, d->cam_scale > 0 ? d->cam_scale : 1.0, s.cams.data());
    float range[2] = {0.f, 0.f};
    s.nv = rc == GPM_OK ? gpm_select_views(s.cams.data(), n, W, H, d->min_angle, d->max_angle, d->max_views, s.subset.data(), range) : -1;
    if (s.nv < 1) return false;
    s.p = d->params;
    if (s.p.depthMin <= 0) s.p.depthMin = range[0];                                   // main.cpp:480-483
    if (s.p.depthMax <= 0) s.p.depthMax = range[1];
    s.p.min_disparity = s.cams[0].f * s.cams[0].baseline / s.p.depthMax;             // main.cpp:905-906
    s.p.max_disparity = s.cams[0].f * s.cams[0].baseline / s.p.depthMin;
    return true;
}

// the options of the _photo twins
gpm_job_opts photo_opts(int kind, float min_std) { return gpm_job_opts{kind, min_std, GPM_PROP_FIXED}; }

const gpm_view_sel kVselOff{GPM_VSEL_OFF, 0.f, 0.f, 0.f, 0, 0, 0.f, 0.f};
const gpm_refine_opts kRefineGipuma{GPM_REFINE_GIPUMA, 0.02f};      // a NULL gpm_refine_opts

// what the _refine drivers refuse of their refinement before any CUDA call, or NULL
const char* refine_opts_refusal(const gpm_refine_opts* r) { return r ? gpm::refine_refusal(r->kind, r->perturbation) : nullptr; }

// The per-view setup of a job: photometric cost, propagation, view selection, refinement, parameters, reference and source
// images (images[i]: image i, grey: channels 1, RGBA: 4), view count, RNG.
int load_view(gpm_ctx* ctx, const gpm_batch_desc* d, const float* const* images, int channels, size_t pitch, const ViewSetup& s,
              const gpm_job_opts& o, const gpm_view_sel& v, const gpm_refine_opts& r)
{
    auto set_reference = channels == 4 ? gpm_set_reference_color : gpm_set_reference;
    auto set_view = channels == 4 ? gpm_set_view_color : gpm_set_view;
    int rc = gpm_set_photometric(ctx, o.photometric, o.ncc_min_std);
    if (rc == GPM_OK) rc = gpm_set_propagation(ctx, o.propagation);
    if (rc == GPM_OK) rc = gpm_set_view_selection(ctx, &v);
    if (rc == GPM_OK) rc = gpm_set_refinement(ctx, r.kind, r.perturbation);
    if (rc == GPM_OK) rc = gpm_set_params(ctx, &s.p);
    if (rc == GPM_OK) rc = set_reference(ctx, images[s.order[0]], pitch, 0, &s.cams[0]);
    for (int v = 0; v < s.nv && rc == GPM_OK; v++) rc = set_view(ctx, v, images[s.source(v)], pitch, 0, &s.cams[s.subset[v]]);
    if (rc == GPM_OK) rc = gpm_set_num_views(ctx, s.nv);
    if (rc == GPM_OK) rc = gpm_set_rng(ctx, d->seed, GPM_RNG_REFERENCE);
    return rc;
}

// <out_dir>/<ref as 8 digits>/disp.dmb, normals.dmb — what the per-image processes of the script leave for fusibile
int write_result(const char* out_dir, int ref, const float* norm4, int H, int W)
{
    char dir[1024];
    snprintf(dir, sizeof(dir), "%s/%08d", out_dir, ref);
    mkdir(out_dir, 0777);  mkdir(dir, 0777);
    const std::string dp = std::string(dir) + "/disp.dmb", np_ = std::string(dir) + "/normals.dmb";
    return gpm_write_result_dmb(dp.c_str(), np_.c_str(), norm4, H, W);
}

// The shared image cache: every image page-locked once (cudaHostRegisterPortable: usable from every device's context) for
// the lifetime of this object.  An image that was already pinned (or cannot be) is simply used as it is.
class PinnedImages {
public:
    PinnedImages(const gpm_batch_desc* d, size_t bytes) : d_(d), registered_(d->n_images, 0)
    {
        for (int i = 0; i < d->n_images; i++)
            registered_[i] = cudaHostRegister(const_cast<float*>(d->images[i]), bytes, cudaHostRegisterPortable) == cudaSuccess;
        cudaGetLastError();
    }
    ~PinnedImages() { for (int i = 0; i < d_->n_images; i++) if (registered_[i]) cudaHostUnregister(const_cast<float*>(d_->images[i])); }
    PinnedImages(const PinnedImages&) = delete;
    PinnedImages& operator=(const PinnedImages&) = delete;
private:
    const gpm_batch_desc* d_;
    std::vector<char> registered_;
};

// One worker thread and context per listed device; body(ctx, dev) runs on that thread.  A worker whose context cannot be
// created records the error, counts as failed and still runs body with ctx = nullptr, so that it reaches any barrier in it;
// take_jobs checks `failed` before every job, so such a body never gets to use the context.
template <class Body>
void run_workers(const gpm_batch_desc* d, std::atomic<int>& failed, Body body)
{
    auto worker = [&](int dev) {
        gpm_ctx* ctx = nullptr;
        if (gpm_create(&ctx, dev, d->width, d->height, d->max_views) != GPM_OK) {
            set_err(std::string("gpm_create: ") + gpm_last_error());
            failed++;
            ctx = nullptr;
        }
        body(ctx, dev);
        if (ctx) gpm_destroy(ctx);
    };
    std::vector<std::thread> pool;
    for (int k = 0; k < d->n_devices; k++) pool.emplace_back(worker, d->devices[k]);
    for (auto& t : pool) t.join();
}

// Jobs 0 .. n-1 from the shared counter `next` until they run out or any worker has failed; fn(job) returns false after
// recording its error.
template <class Fn>
void take_jobs(std::atomic<int>& next, int n, std::atomic<int>& failed, Fn fn)
{
    for (;;) {
        const int job = next.fetch_add(1);
        if (job >= n || failed.load()) return;
        if (!fn(job)) { failed++;  return; }
    }
}
}  // namespace

extern "C" const char* gpm_batch_last_error(void)
{
    std::lock_guard<std::mutex> l(g_err_mutex);
    static thread_local std::string copy;
    copy = g_batch_err;
    return copy.c_str();
}

// ---- two-pass geometric-consistency batch (DESIGN.md §14) -----------------------------------------------------------------
namespace {
// Page-locked host memory (portable: every device's context may copy from it) for the lifetime of this object.
class PinnedStore {
public:
    explicit PinnedStore(size_t floats) { if (cudaHostAlloc(&p_, floats * sizeof(float), cudaHostAllocPortable) != cudaSuccess) p_ = nullptr; }
    ~PinnedStore() { if (p_) cudaFreeHost(p_); }
    PinnedStore(const PinnedStore&) = delete;
    PinnedStore& operator=(const PinnedStore&) = delete;
    float* get() const { return static_cast<float*>(p_); }
private:
    void* p_ = nullptr;
};

// Every worker of the pool waits in arrive_and_wait until all of them have arrived; the barrier may be passed any number of
// times (each pass is one generation).
class Barrier {
public:
    explicit Barrier(int n) : n_(n), left_(n) {}
    void arrive_and_wait()
    {
        std::unique_lock<std::mutex> l(m_);
        const unsigned gen = gen_;
        if (--left_ == 0) { left_ = n_;  gen_++;  cv_.notify_all(); }
        else cv_.wait(l, [&] { return gen_ != gen; });
    }
private:
    std::mutex m_;
    std::condition_variable cv_;
    const int n_;
    int left_;
    unsigned gen_ = 0;
};

// CUDA-event time of one gpm_sweep, from an event recorded on the context's stream before it to one recorded after it.
// The events are created by the first sweep, on the calling thread's current device, which must be the context's.
class SweepTimer {
public:
    SweepTimer() = default;
    ~SweepTimer() { if (a_) cudaEventDestroy(a_);  if (b_) cudaEventDestroy(b_); }
    SweepTimer(const SweepTimer&) = delete;
    SweepTimer& operator=(const SweepTimer&) = delete;
    int sweep(gpm_ctx* ctx, int iterations, float* ms)
    {
        cudaStream_t s = static_cast<cudaStream_t>(gpm_stream(ctx));
        if (!a_ && cudaEventCreate(&a_) != cudaSuccess) { a_ = nullptr;  return cuda_fail(); }
        if (!b_ && cudaEventCreate(&b_) != cudaSuccess) { b_ = nullptr;  return cuda_fail(); }
        if (cudaEventRecord(a_, s) != cudaSuccess) return cuda_fail();
        const int rc = gpm_sweep(ctx, iterations);
        if (rc != GPM_OK) return rc;
        if (cudaEventRecord(b_, s) != cudaSuccess || cudaEventSynchronize(b_) != cudaSuccess || cudaEventElapsedTime(ms, a_, b_) != cudaSuccess)
            return cuda_fail();
        return GPM_OK;
    }
    std::string error;
private:
    int cuda_fail() { error = std::string("sweep event: ") + cudaGetErrorString(cudaGetLastError());  return GPM_E_CUDA; }
    cudaEvent_t a_ = nullptr, b_ = nullptr;
};

// The prior stage of a photometric job (DESIGN.md §18), after its params.iterations sweeps: the prior map built from the
// state, the term on, the state re-scored under it (gpm_cost_eval + gpm_set_state), the prior planes offered, and
// prior->iterations more sweeps.  The caller finalizes and then turns the term off (prior_off).  build_ms (may be NULL)
// receives the host time of the build.
int prior_stage(gpm_ctx* ctx, const gpm_prior_opts* p, gpm_prior_info* info, std::vector<float>& n4, std::vector<float>& cost,
                SweepTimer& timer, float* ms, float* build_ms = nullptr)
{
    const gpm_prior_build b{p->step, p->support_cost};
    const auto t0 = std::chrono::steady_clock::now();
    int rc = gpm_build_planar_prior(ctx, &b, info);
    if (build_ms) *build_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (rc == GPM_OK) rc = gpm_set_prior(ctx, p->weight, p->depth_sigma, p->normal_sigma_deg);
    if (rc == GPM_OK) rc = gpm_get_state(ctx, n4.data(), nullptr, 0);
    if (rc == GPM_OK) rc = gpm_cost_eval(ctx, n4.data(), cost.data(), 0);
    if (rc == GPM_OK) rc = gpm_set_state(ctx, n4.data(), cost.data(), 0);
    if (rc == GPM_OK) rc = gpm_offer_prior(ctx);
    if (rc == GPM_OK) rc = timer.sweep(ctx, p->iterations, ms);
    return rc;
}
int prior_off(gpm_ctx* ctx, const gpm_prior_opts* p) { return gpm_set_prior(ctx, 0.f, p->depth_sigma, p->normal_sigma_deg); }
}  // namespace

// gpm_batch_run and its _photo / _opts / _vsel / _prior twins; `fn` names the entry point in error messages
static int batch_run(const char* fn, const gpm_batch_desc* d, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                     const gpm_prior_opts* prior, const gpm_refine_opts* refine, gpm_batch_stats* stats)
{
    clear_err();
    if (!batch_desc_ok(d)) {
        set_err(std::string(fn) + ": bad arguments");
        return GPM_E_ARG;
    }
    const char* bad_refine = refine_opts_refusal(refine);
    if (const char* bad = bad_refine ? bad_refine : gpm::job_refusal(opts, vsel, prior, 1)) {
        set_err(std::string(fn) + ": bad arguments: " + bad);
        return GPM_E_ARG;
    }
    if (!refine) refine = &kRefineGipuma;
    const int n = d->n_images, W = d->width, H = d->height;
    const size_t pitch = d->pitch_bytes ? d->pitch_bytes : (size_t)W * sizeof(float);
    const size_t npix = (size_t)W * H;
    PinnedImages pinned(d, pitch * H);

    std::atomic<int> next(0), failed(0);
    std::vector<double> sweep_ms(d->n_refs, 0.0);
    std::vector<int> views_used(d->n_refs, 0), device_of(d->n_refs, -1);
    run_workers(d, failed, [&](gpm_ctx* ctx, int dev) {
        if (ctx && prior) cudaSetDevice(dev);            // the prior stage's sweep events live on the context's device
        ViewSetup s;
        SweepTimer timer;
        std::vector<float> n4, cost(ctx && prior ? npix : 0);
        if (ctx && prior) n4.resize(npix * 4);
        take_jobs(next, d->n_refs, failed, [&](int job) {
            const int ref = d->ref_indices ? d->ref_indices[job] : job;
            if (ref < 0 || ref >= n) { set_err(std::string(fn) + ": reference index out of range");  return false; }
            if (!plan_view(d, ref, s)) { set_err(std::string(fn) + ": no source view passes the angle filter for reference " + std::to_string(ref));  return false; }
            int rc = load_view(ctx, d, d->images, 1, pitch, s, *opts, *vsel, *refine);
            float ms = 0.f, ms2 = 0.f;
            if (!prior) {
                if (rc == GPM_OK) rc = gpm_run(ctx, &ms);
            } else {                                     // gpm_run's steps with the prior stage before the finalize
                if (rc == GPM_OK) rc = gpm_init(ctx);
                if (rc == GPM_OK) rc = timer.sweep(ctx, d->params.iterations, &ms);
                if (rc == GPM_OK) rc = prior_stage(ctx, prior, prior->info ? prior->info + job : nullptr, n4, cost, timer, &ms2);
                if (rc == GPM_OK) rc = gpm_finalize(ctx);
                if (rc == GPM_OK) rc = prior_off(ctx, prior);
                ms += ms2;
            }
            if (rc != GPM_OK) {
                set_err(std::string("reference view ") + std::to_string(ref) + ": " +
                        (rc == GPM_E_CUDA && !timer.error.empty() ? timer.error : std::string(gpm_last_error())));
                return false;
            }
            sweep_ms[job] = ms;  views_used[job] = s.nv;  device_of[job] = dev;
            float* o4 = d->out_norm4 ? d->out_norm4 + (size_t)job * npix * 4 : nullptr;
            float* oc = d->out_cost ? d->out_cost + (size_t)job * npix : nullptr;
            if (d->out_dir && !o4) { n4.resize(npix * 4);  o4 = n4.data(); }
            if (o4 || oc) rc = gpm_get_state(ctx, o4, oc, 0);
            if (rc == GPM_OK && d->out_dir) rc = write_result(d->out_dir, ref, o4, H, W);
            if (rc != GPM_OK) { set_err(std::string(fn) + ": could not store the result of reference view " + std::to_string(ref));  return false; }
            return true;
        });
    });
    if (stats) {
        stats->jobs_done = 0;  stats->sweep_ms_total = 0.0;
        for (int j = 0; j < d->n_refs; j++) if (device_of[j] >= 0) { stats->jobs_done++;  stats->sweep_ms_total += sweep_ms[j]; }
        if (stats->per_job_sweep_ms) for (int j = 0; j < d->n_refs; j++) stats->per_job_sweep_ms[j] = (float)sweep_ms[j];
        if (stats->per_job_views) for (int j = 0; j < d->n_refs; j++) stats->per_job_views[j] = views_used[j];
        if (stats->per_job_device) for (int j = 0; j < d->n_refs; j++) stats->per_job_device[j] = device_of[j];
    }
    return failed.load() ? GPM_E_STATE : GPM_OK;
}

extern "C" int gpm_batch_run(const gpm_batch_desc* d, gpm_batch_stats* stats)
{
    const gpm_job_opts o = photo_opts(GPM_PHOTO_PM, 0.f);
    return batch_run("gpm_batch_run", d, &o, &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_batch_run_photo(const gpm_batch_desc* d, int kind, float min_std, gpm_batch_stats* stats)
{
    const gpm_job_opts o = photo_opts(kind, min_std);
    return batch_run("gpm_batch_run_photo", d, &o, &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_batch_run_opts(const gpm_batch_desc* d, const gpm_job_opts* opts, gpm_batch_stats* stats)
{
    return batch_run("gpm_batch_run_opts", d, opts, &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_batch_run_vsel(const gpm_batch_desc* d, const gpm_job_opts* opts, const gpm_view_sel* vsel, gpm_batch_stats* stats)
{
    return batch_run("gpm_batch_run_vsel", d, opts, vsel ? vsel : &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_batch_run_prior(const gpm_batch_desc* d, const gpm_job_opts* opts, const gpm_view_sel* vsel, const gpm_prior_opts* prior,
                                   gpm_batch_stats* stats)
{
    return batch_run("gpm_batch_run_prior", d, opts, vsel ? vsel : &kVselOff, prior, nullptr, stats);
}

extern "C" int gpm_batch_run_refine(const gpm_batch_desc* d, const gpm_job_opts* opts, const gpm_view_sel* vsel, const gpm_prior_opts* prior,
                                    const gpm_refine_opts* refine, gpm_batch_stats* stats)
{
    return batch_run("gpm_batch_run_refine", d, opts, vsel ? vsel : &kVselOff, prior, refine, stats);
}


namespace {
// What the geometric and the multi-level drivers refuse in a descriptor, or NULL; is_ref[i] = 1 for every reference view i.
// Every reference index must be an image (without ref_indices: n_refs <= n_images); with out_dir each must be listed once,
// or two workers would write the same files.
const char* geo_desc_refusal(const gpm_geo_batch_desc* g, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                             const gpm_prior_opts* prior, std::vector<char>& is_ref)
{
    if (!g || !batch_desc_ok(&g->batch)) return "the batch descriptor is refused as gpm_batch_run refuses it";
    if (g->channels != 1 && g->channels != 4) return "channels must be 1 or 4";
    if (g->geo_iterations < 0) return "geo_iterations must be >= 0";
    if (!std::isfinite(g->weight) || g->weight < 0.f) return "weight must be finite and >= 0";
    if (!std::isfinite(g->max_err) || g->max_err <= 0.f) return "max_err must be finite and > 0";
    if (const char* bad = gpm::job_refusal(opts, vsel, prior, g->channels)) return bad;
    const gpm_batch_desc* d = &g->batch;
    is_ref.assign(d->n_images, 0);
    for (int j = 0; j < d->n_refs; j++) {
        const int r = d->ref_indices ? d->ref_indices[j] : j;
        if (r < 0 || r >= d->n_images) return "reference index out of range";
        if (is_ref[r] && d->out_dir) return "a reference view is listed twice while out_dir is set";
        is_ref[r] = 1;
    }
    return nullptr;
}
}  // namespace

// gpm_geo_batch_run and its _photo / _opts / _vsel twins; `fn` names the entry point in error messages
static int geo_batch_run(const char* fn, const gpm_geo_batch_desc* g, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                         const gpm_prior_opts* prior, const gpm_refine_opts* refine, gpm_geo_batch_stats* stats)
{
    clear_err();
    std::vector<char> is_ref;
    const char* bad_refine = refine_opts_refusal(refine);
    if (const char* bad = bad_refine ? bad_refine : geo_desc_refusal(g, opts, vsel, prior, is_ref)) {
        set_err(std::string(fn) + ": bad arguments: " + bad);
        return GPM_E_ARG;
    }
    if (!refine) refine = &kRefineGipuma;
    const gpm_batch_desc* d = &g->batch;
    const int n = d->n_images, W = d->width, H = d->height, n_refs = d->n_refs;
    const size_t pitch = d->pitch_bytes ? d->pitch_bytes : (size_t)W * sizeof(float) * g->channels;
    const size_t npix = (size_t)W * H;
    auto ref_of = [&](int job) { return d->ref_indices ? d->ref_indices[job] : job; };
    std::vector<char> in_pass1(n, 0);

    // Pass-1 set: the reference views and every view their selection picks (not recursive), planned on the host before
    // anything runs, so that a view without source views is refused before any CUDA call.
    std::vector<ViewSetup> setup(n);
    for (int pass = 0; pass < 2; pass++)
        for (int i = 0; i < n; i++) {
            if (!(pass == 0 ? is_ref[i] : in_pass1[i] && !is_ref[i])) continue;
            if (!plan_view(d, i, setup[i])) {
                set_err(std::string(fn) + ": no source view passes the angle filter for " +
                        (is_ref[i] ? "reference view " : "source view ") + std::to_string(i));
                return GPM_E_STATE;
            }
            in_pass1[i] = 1;
            if (pass == 0) for (int v = 0; v < setup[i].nv; v++) in_pass1[setup[i].source(v)] = 1;
        }
    std::vector<int> pass1, depth_slot(n, -1), raw_slot(n, -1);
    int n_raw = 0;
    for (int i = 0; i < n; i++)
        if (in_pass1[i]) {
            depth_slot[i] = (int)pass1.size();
            pass1.push_back(i);
            if (is_ref[i]) raw_slot[i] = n_raw++;
        }
    const int n_pass1 = (int)pass1.size();

    // The host store: a pass-1 depth map per pass-1 view, then the raw pass-1 planes of every reference view.
    PinnedImages pinned(d, pitch * H);
    PinnedStore store((size_t)n_pass1 * npix + (size_t)n_raw * npix * 4);
    if (!store.get()) {
        set_err(std::string(fn) + ": cannot allocate the page-locked host store: " + cudaGetErrorString(cudaGetLastError()));
        return GPM_E_CUDA;
    }
    float* depth_store = store.get();
    float* raw_store = depth_store + (size_t)n_pass1 * npix;

    std::atomic<int> next1(0), next2(0), failed(0);
    std::vector<float> pass1_ms(n_pass1, 0.f), pass2_ms(n_refs, 0.f);
    std::vector<int> device_of(n_refs, -1);
    Barrier barrier(d->n_devices);
    run_workers(d, failed, [&](gpm_ctx* ctx, int dev) {
        if (ctx) cudaSetDevice(dev);                     // a worker thread of its own: the sweep events live on its device
        SweepTimer timer;
        std::vector<float> n4(ctx ? npix * 4 : 0), cost(ctx ? npix : 0);
        auto fail_at = [&](const char* what, int view, int rc) {
            set_err(std::string(fn) + ": " + what + " view " + std::to_string(view) + ": " +
                    (rc == GPM_E_CUDA && !timer.error.empty() ? timer.error : std::string(gpm_last_error())));
            return false;
        };
        take_jobs(next1, n_pass1, failed, [&](int job) {          // pass 1: photometric
            const int r = pass1[job];
            int rc = load_view(ctx, d, d->images, g->channels, pitch, setup[r], *opts, *vsel, *refine);
            if (rc == GPM_OK) rc = gpm_init(ctx);
            if (rc == GPM_OK) rc = timer.sweep(ctx, d->params.iterations, &pass1_ms[job]);
            float ms2 = 0.f;
            if (rc == GPM_OK && prior) rc = prior_stage(ctx, prior, prior->info ? prior->info + job : nullptr, n4, cost, timer, &ms2);
            pass1_ms[job] += ms2;
            if (rc == GPM_OK && raw_slot[r] >= 0) rc = gpm_get_state(ctx, raw_store + (size_t)raw_slot[r] * npix * 4, nullptr, 0);
            if (rc == GPM_OK) rc = gpm_finalize(ctx);
            if (rc == GPM_OK && prior) rc = prior_off(ctx, prior);     // pass 2 has no prior
            if (rc == GPM_OK) rc = gpm_get_state(ctx, n4.data(), nullptr, 0);
            if (rc != GPM_OK) return fail_at("pass 1 of", r, rc);
            float* dep = depth_store + (size_t)depth_slot[r] * npix;
            for (size_t k = 0; k < npix; k++) dep[k] = n4[k * 4 + 3];
            return true;
        });
        barrier.arrive_and_wait();                                  // every depth map exists before any pass-2 job starts
        take_jobs(next2, n_refs, failed, [&](int job) {            // pass 2: geometric, seeded with the pass-1 planes
            const int r = ref_of(job);
            const ViewSetup& s = setup[r];
            const float* raw = raw_store + (size_t)raw_slot[r] * npix * 4;
            int rc = load_view(ctx, d, d->images, g->channels, pitch, s, *opts, *vsel, *refine);
            for (int v = 0; v < s.nv && rc == GPM_OK; v++) rc = gpm_set_view_depth(ctx, v, depth_store + (size_t)depth_slot[s.source(v)] * npix, 0, 0);
            if (rc == GPM_OK) rc = gpm_set_geometric(ctx, g->weight, g->max_err);
            if (rc == GPM_OK) rc = gpm_cost_eval(ctx, raw, cost.data(), 0);
            if (rc == GPM_OK) rc = gpm_set_state(ctx, raw, cost.data(), 0);
            if (rc == GPM_OK) rc = timer.sweep(ctx, g->geo_iterations, &pass2_ms[job]);
            if (rc == GPM_OK) rc = gpm_finalize(ctx);
            float* o4 = d->out_norm4 ? d->out_norm4 + (size_t)job * npix * 4 : nullptr;
            float* oc = d->out_cost ? d->out_cost + (size_t)job * npix : nullptr;
            if (d->out_dir && !o4) o4 = n4.data();
            if (rc == GPM_OK && (o4 || oc)) rc = gpm_get_state(ctx, o4, oc, 0);
            if (rc == GPM_OK && d->out_dir && write_result(d->out_dir, r, o4, H, W) != GPM_OK) {
                set_err(std::string(fn) + ": could not store the result of reference view " + std::to_string(r));
                return false;
            }
            if (rc == GPM_OK) rc = gpm_set_geometric(ctx, 0.f, g->max_err);
            if (rc != GPM_OK) return fail_at("pass 2 of reference", r, rc);
            device_of[job] = dev;
            return true;
        });
    });
    if (stats) {
        gpm_batch_stats* b = &stats->batch;
        b->jobs_done = 0;  b->sweep_ms_total = 0.0;
        for (int j = 0; j < n_refs; j++) if (device_of[j] >= 0) { b->jobs_done++;  b->sweep_ms_total += pass2_ms[j]; }
        if (b->per_job_sweep_ms) for (int j = 0; j < n_refs; j++) b->per_job_sweep_ms[j] = pass2_ms[j];
        if (b->per_job_views) for (int j = 0; j < n_refs; j++) b->per_job_views[j] = setup[ref_of(j)].nv;
        if (b->per_job_device) for (int j = 0; j < n_refs; j++) b->per_job_device[j] = device_of[j];
        stats->n_pass1 = n_pass1;
        if (stats->pass1_views) std::copy(pass1.begin(), pass1.end(), stats->pass1_views);
        if (stats->pass1_sweep_ms) std::copy(pass1_ms.begin(), pass1_ms.end(), stats->pass1_sweep_ms);
        if (stats->ref_views)
            for (int j = 0; j < n_refs; j++) {
                const ViewSetup& s = setup[ref_of(j)];
                for (int v = 0; v < d->max_views; v++) stats->ref_views[(size_t)j * d->max_views + v] = v < s.nv ? s.source(v) : -1;
            }
    }
    return failed.load() ? GPM_E_STATE : GPM_OK;
}

extern "C" int gpm_geo_batch_run(const gpm_geo_batch_desc* g, gpm_geo_batch_stats* stats)
{
    const gpm_job_opts o = photo_opts(GPM_PHOTO_PM, 0.f);
    return geo_batch_run("gpm_geo_batch_run", g, &o, &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_geo_batch_run_photo(const gpm_geo_batch_desc* g, int kind, float min_std, gpm_geo_batch_stats* stats)
{
    const gpm_job_opts o = photo_opts(kind, min_std);
    return geo_batch_run("gpm_geo_batch_run_photo", g, &o, &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_geo_batch_run_opts(const gpm_geo_batch_desc* g, const gpm_job_opts* opts, gpm_geo_batch_stats* stats)
{
    return geo_batch_run("gpm_geo_batch_run_opts", g, opts, &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_geo_batch_run_vsel(const gpm_geo_batch_desc* g, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                      gpm_geo_batch_stats* stats)
{
    return geo_batch_run("gpm_geo_batch_run_vsel", g, opts, vsel ? vsel : &kVselOff, nullptr, nullptr, stats);
}

extern "C" int gpm_geo_batch_run_prior(const gpm_geo_batch_desc* g, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                       const gpm_prior_opts* prior, gpm_geo_batch_stats* stats)
{
    return geo_batch_run("gpm_geo_batch_run_prior", g, opts, vsel ? vsel : &kVselOff, prior, nullptr, stats);
}

extern "C" int gpm_geo_batch_run_refine(const gpm_geo_batch_desc* g, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                        const gpm_prior_opts* prior, const gpm_refine_opts* refine, gpm_geo_batch_stats* stats)
{
    return geo_batch_run("gpm_geo_batch_run_refine", g, opts, vsel ? vsel : &kVselOff, prior, refine, stats);
}


// ---- coarse-to-fine multi-scale batch (DESIGN.md §19) ---------------------------------------------------------------------
namespace {
int level_size(int s, int level) { for (int k = 0; k < level; k++) s = (s + 1) / 2;  return s; }

// The detail restorer's detection (DESIGN.md §21): pixel p is a detail pixel where the geometric stage's plane costs more
// than `threshold` above the photometric-only plane, both costed photometrically: fsub(c_ms, c_ph) > threshold, one fp32
// rounding (a NaN is never a detail pixel).  Returns the number of detail pixels.
long long detect_details(const float* c_ms, const float* c_ph, float threshold, size_t n, unsigned char* detail)
{
    long long count = 0;
    for (size_t p = 0; p < n; p++) {
        detail[p] = c_ms[p] - c_ph[p] > threshold ? 1 : 0;
        count += detail[p];
    }
    return count;
}

// planes <- the photometric-only plane at detail pixels, unchanged elsewhere
void merge_planes(float* planes, const float* photo, const unsigned char* detail, size_t n)
{
    for (size_t p = 0; p < n; p++)
        if (detail[p]) memcpy(planes + 4 * p, photo + 4 * p, 4 * sizeof(float));
}

// A view's setup at a coarser level: the level-0 selection, order and depth range, the cameras at `cam_scale` and the
// disparities of their f.
bool rescale_view(const ViewSetup& s0, int n, double cam_scale, ViewSetup& s)
{
    s = s0;
    if (gpm_prepare_cameras(s.P.data(), n, cam_scale, s.cams.data()) != GPM_OK) return false;
    s.p.min_disparity = s.cams[0].f * s.cams[0].baseline / s.p.depthMax;
    s.p.max_disparity = s.cams[0].f * s.cams[0].baseline / s.p.depthMin;
    return true;
}

const char* ms_refusal(const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel, std::vector<char>& is_ref)
{
    if (!m) return "null descriptor";
    if (const char* bad = geo_desc_refusal(&m->geo, opts, vsel, nullptr, is_ref)) return bad;
    if (m->levels < 1 || m->levels > GPM_MS_MAX_LEVELS) return "levels must be 1..4";
    if (level_size(m->geo.batch.width, m->levels - 1) < 8 || level_size(m->geo.batch.height, m->levels - 1) < 8)
        return "the coarsest level is below 8 x 8 pixels";
    if (m->jbu.radius < 0 || m->jbu.radius > 4) return "jbu.radius must be 0..4";
    if (!(std::isfinite(m->jbu.sigma_space) && m->jbu.sigma_space > 0.f) || !(std::isfinite(m->jbu.sigma_range) && m->jbu.sigma_range > 0.f))
        return "jbu.sigma_space and jbu.sigma_range must be finite and > 0";
    return nullptr;
}

// What the multi-level driver refuses in its prior stages (DESIGN.md §20), after ms_refusal passed: each given stage's
// options and mode rule; a weight with which a valid cost could reach MAXCOST, which gpm_set_prior would refuse only
// during the run (photometric stage: without the geometric term; geometric stage: with weight * max_err); a level whose
// build gpm_build_planar_prior refuses (photometric stage: the coarsest; geometric stage: level 0, the largest).
std::string ms_prior_refusal(const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel, const gpm_ms_prior_opts* prior)
{
    if (!prior) return "";
    const gpm_geo_batch_desc* g = &m->geo;
    const bool ncc = opts->photometric == GPM_PHOTO_NCC;
    const struct { const char* name; const gpm_prior_opts* p; float geo_weight; int level; } stages[2] = {
        {"photometric", prior->photometric, 0.f, m->levels - 1}, {"geometric", prior->geometric, g->weight, 0}};
    for (const auto& s : stages) {
        if (!s.p) continue;
        if (const char* bad = gpm::job_refusal(opts, vsel, s.p, g->channels)) return std::string(s.name) + " prior stage: " + bad;
        if (!gpm::prior_bound_ok(g->batch.params, ncc, s.geo_weight, g->max_err, s.p->weight))
            return std::string(s.name) + " prior stage: with its weight a valid cost could reach MAXCOST";
        if (level_size(g->batch.width, s.level) > 4097 || level_size(g->batch.height, s.level) > 4097)
            return std::string(s.name) + " prior stage: its level " + std::to_string(s.level) + " is wider or taller than 4097 pixels";
    }
    return "";
}

// What the multi-level driver refuses of the detail restorer's options (DESIGN.md §21); NULL: no restorer.
const char* ms_restore_refusal(const gpm_ms_restore_opts* r)
{
    if (!r) return nullptr;
    if (r->photo_iterations < 1) return "detail restorer: photo_iterations must be >= 1";
    if (r->iterations < 0) return "detail restorer: iterations must be >= 0";
    if (!std::isfinite(r->threshold)) return "detail restorer: threshold must be finite";
    return nullptr;
}
}  // namespace

// gpm_ms_batch_run, gpm_ms_batch_run_prior and gpm_ms_batch_run_restore; `fn` names the entry point in error messages
static int ms_batch_run(const char* fn_name, const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                        gpm_ms_prior_opts* prior, const gpm_ms_restore_opts* restore, const gpm_refine_opts* refine,
                        gpm_ms_batch_stats* stats)
{
    const std::string fn = fn_name;
    clear_err();
    if (!vsel) vsel = &kVselOff;
    std::vector<char> is_ref;
    if (const char* bad = ms_refusal(m, opts, vsel, is_ref)) {
        set_err(fn + ": bad arguments: " + bad);
        return GPM_E_ARG;
    }
    const std::string bad_prior = ms_prior_refusal(m, opts, vsel, prior);
    if (!bad_prior.empty()) {
        set_err(fn + ": bad arguments: " + bad_prior);
        return GPM_E_ARG;
    }
    if (const char* bad = ms_restore_refusal(restore)) {
        set_err(fn + ": bad arguments: " + bad);
        return GPM_E_ARG;
    }
    if (const char* bad = refine_opts_refusal(refine)) {
        set_err(fn + ": bad arguments: " + bad);
        return GPM_E_ARG;
    }
    if (!refine) refine = &kRefineGipuma;
    const gpm_prior_opts* P_photo = prior ? prior->photometric : nullptr;
    const gpm_prior_opts* P_geo = prior ? prior->geometric : nullptr;
    const gpm_geo_batch_desc* g = &m->geo;
    const gpm_batch_desc* d = &g->batch;
    const int n = d->n_images, n_refs = d->n_refs, ch = g->channels, L = m->levels, top = L - 1;
    if (P_photo && P_photo->info) memset(P_photo->info, 0, (size_t)n * sizeof(gpm_prior_info));
    if (P_geo && P_geo->info) memset(P_geo->info, 0, (size_t)GPM_MS_MAX_LEVELS * n * sizeof(gpm_prior_info));
    auto ref_of = [&](int job) { return d->ref_indices ? d->ref_indices[job] : job; };

    // V: the transitive closure of the references' selections, planned at level 0 before any CUDA call.
    std::vector<ViewSetup> setup0(n);
    std::vector<char> in_v(n, 0);
    std::vector<int> queue;
    for (int i = 0; i < n; i++) if (is_ref[i]) { in_v[i] = 1;  queue.push_back(i); }
    for (size_t q = 0; q < queue.size(); q++) {
        const int i = queue[q];
        if (!plan_view(d, i, setup0[i])) {
            set_err(fn + ": no source view passes the angle filter for " + (is_ref[i] ? "reference view " : "source view ") + std::to_string(i));
            return GPM_E_STATE;
        }
        for (int v = 0; v < setup0[i].nv; v++) {
            const int s = setup0[i].source(v);
            if (!in_v[s]) { in_v[s] = 1;  queue.push_back(s); }
        }
    }
    std::vector<int> views, slot(n, -1), refs;
    for (int i = 0; i < n; i++) {
        if (in_v[i]) { slot[i] = (int)views.size();  views.push_back(i); }
        if (is_ref[i]) refs.push_back(i);
    }
    const int nV = (int)views.size(), nR = (int)refs.size();

    // Per level: size, setups (selection and depth range of level 0; cameras and disparities of the level), image pitch.
    const double scale0 = d->cam_scale > 0 ? d->cam_scale : 1.0;
    std::vector<int> Wl(L), Hl(L);
    std::vector<size_t> npix(L), pitch(L);
    std::vector<std::vector<ViewSetup>> setup(L);
    for (int l = 0; l < L; l++) {
        Wl[l] = level_size(d->width, l);  Hl[l] = level_size(d->height, l);
        npix[l] = (size_t)Wl[l] * Hl[l];
        pitch[l] = l == 0 && d->pitch_bytes ? d->pitch_bytes : (size_t)Wl[l] * ch * sizeof(float);
        if (l == 0) { setup[0] = std::move(setup0);  continue; }
        setup[l].resize(n);
        for (int i : views)
            if (!rescale_view(setup[0][i], n, scale0 * (double)(1 << l), setup[l][i])) {
                set_err(fn + ": bad arguments: the cameras cannot be prepared at level " + std::to_string(l));
                return GPM_E_ARG;
            }
    }

    // The host store: the pyramid levels 1 .. L-1 of every view of V; the raw planes of even levels (level-0 size) and of odd
    // levels (level-1 size), so that a level's upsampling reads the next coarser level's planes while it writes its own; one
    // depth map per view of V, of the current level.
    std::vector<size_t> pyr_off(L, 0);
    size_t floats = 0;
    for (int l = 1; l < L; l++) { pyr_off[l] = floats;  floats += (size_t)nV * npix[l] * ch; }
    const size_t raw_even = floats;
    floats += (size_t)nV * npix[0] * 4;
    const size_t raw_odd = floats;
    if (L > 1) floats += (size_t)nV * npix[1] * 4;
    const size_t depth_off = floats;
    floats += (size_t)nV * npix[0];
    PinnedImages pinned(d, pitch[0] * d->height);
    PinnedStore store(floats);
    if (!store.get()) {
        set_err(fn + ": cannot allocate the page-locked host store: " + cudaGetErrorString(cudaGetLastError()));
        return GPM_E_CUDA;
    }
    float* const base = store.get();
    auto pyr = [&](int l, int k) { return base + pyr_off[l] + (size_t)k * npix[l] * ch; };
    auto raw = [&](int l, int k) { return base + (l % 2 ? raw_odd + (size_t)k * npix[1] * 4 : raw_even + (size_t)k * npix[0] * 4); };
    auto dep = [&](int k) { return base + depth_off + (size_t)k * npix[0]; };
    std::vector<std::vector<const float*>> imgs(L, std::vector<const float*>(n, nullptr));
    for (int i = 0; i < n; i++) imgs[0][i] = d->images[i];
    for (int l = 1; l < L; l++) for (int k = 0; k < nV; k++) imgs[l][views[k]] = pyr(l, k);

    const int n_stages = 2 + 2 * L;
    std::vector<std::atomic<int>> next(n_stages);
    for (auto& a : next) a.store(0);
    std::atomic<int> failed(0);
    std::vector<std::vector<float>> sweep_ms(L, std::vector<float>(nV, 0.f)), up_ms(L, std::vector<float>(nV, 0.f)),
        build_ms(L, std::vector<float>(nV, 0.f));
    std::vector<int> device_of(n_refs, -1), restored(n_refs, 0);
    std::vector<float> job_ms(n_refs, 0.f);
    Barrier barrier(d->n_devices);
    run_workers(d, failed, [&](gpm_ctx* ctx, int dev) {
        if (ctx) cudaSetDevice(dev);                     // a worker thread of its own: the sweep events live on its device
        std::vector<gpm_ctx*> lc(L, nullptr);            // one context per level
        lc[0] = ctx;
        for (int l = 1; l < L && ctx; l++)
            if (gpm_create(&lc[l], dev, Wl[l], Hl[l], d->max_views) != GPM_OK) {
                set_err(fn + ": gpm_create at level " + std::to_string(l) + ": " + gpm_last_error());
                failed++;
                lc[l] = nullptr;
            }
        SweepTimer timer;
        std::vector<float> n4(ctx ? npix[0] * 4 : 0), cost(ctx ? npix[0] : 0);
        // the detail restorer's buffers: the photometric-only planes, both detection costs and the detail mask
        const bool rs = restore && ctx;
        std::vector<float> ph4(rs ? npix[0] * 4 : 0), c_ms(rs ? npix[0] : 0), c_ph(rs ? npix[0] : 0);
        std::vector<unsigned char> detail(rs ? npix[0] : 0);
        auto fail_at = [&](const char* stage, int l, int view, int rc) {
            set_err(fn + ": level " + std::to_string(l) + " " + stage + " of view " + std::to_string(view) + ": " +
                    (rc == GPM_E_CUDA && !timer.error.empty() ? timer.error : std::string(gpm_last_error())));
            return false;
        };
        take_jobs(next[0], L > 1 ? nV : 0, failed, [&](int k) {              // 1. the pyramid
            const float* src = d->images[views[k]];
            for (int l = 1; l < L; l++) {
                const int rc = gpm_downsample(dev, src, pitch[l - 1], Wl[l - 1], Hl[l - 1], ch, pyr(l, k), 0);
                if (rc != GPM_OK) return fail_at("pyramid", l, views[k], rc);
                src = pyr(l, k);
            }
            return true;
        });
        barrier.arrive_and_wait();
        take_jobs(next[1], nV, failed, [&](int k) {                           // 2. coarsest level, photometric
            const int i = views[k];
            gpm_ctx* c = lc[top];
            int rc = load_view(c, d, imgs[top].data(), ch, pitch[top], setup[top][i], *opts, *vsel, *refine);
            if (rc == GPM_OK) rc = gpm_init(c);
            if (rc == GPM_OK) rc = timer.sweep(c, d->params.iterations, &sweep_ms[top][k]);
            float ms2 = 0.f, bms = 0.f;                                       // the photometric prior stage (§20)
            if (rc == GPM_OK && P_photo)
                rc = prior_stage(c, P_photo, P_photo->info ? P_photo->info + i : nullptr, n4, cost, timer, &ms2, &bms);
            sweep_ms[top][k] += ms2;  build_ms[top][k] += bms;
            if (rc == GPM_OK) rc = gpm_get_state(c, raw(top, k), nullptr, 0);
            if (rc == GPM_OK) rc = gpm_finalize(c);
            if (rc == GPM_OK && P_photo) rc = prior_off(c, P_photo);
            if (rc == GPM_OK) rc = gpm_get_state(c, n4.data(), nullptr, 0);
            if (rc != GPM_OK) return fail_at("photometric stage", top, i, rc);
            float* D = dep(k);
            for (size_t p = 0; p < npix[top]; p++) D[p] = n4[p * 4 + 3];
            return true;
        });
        barrier.arrive_and_wait();
        for (int l = top; l >= 0; l--) {
            if (l < top) {
                take_jobs(next[2 + 2 * l], nV, failed, [&](int k) {           // upsampling of level l + 1 into level l
                    const int i = views[k];
                    const ViewSetup& s = setup[l][i];
                    auto set_reference = ch == 4 ? gpm_set_reference_color : gpm_set_reference;
                    int rc = gpm_set_params(lc[l], &s.p);
                    if (rc == GPM_OK) rc = set_reference(lc[l], imgs[l][i], pitch[l], 0, &s.cams[0]);
                    const auto t0 = std::chrono::steady_clock::now();
                    if (rc == GPM_OK) rc = gpm_upsample_planes(lc[l], raw(l + 1, k), Wl[l + 1], Hl[l + 1], 0, &m->jbu, raw(l, k), dep(k));
                    up_ms[l][k] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
                    return rc == GPM_OK ? true : fail_at("upsampling", l, i, rc);
                });
                barrier.arrive_and_wait();                                    // every D_l exists before any view refines
            }
            const int n_jobs = l == 0 ? nR : nV;                              // at level 0 only the references' results are read
            take_jobs(next[3 + 2 * l], n_jobs, failed, [&](int job) {         // geometric stage of level l
                const int i = l == 0 ? refs[job] : views[job], k = slot[i];
                const ViewSetup& s = setup[l][i];
                gpm_ctx* c = lc[l];
                const bool restoring = restore && l == 0;
                float ms = 0.f;
                int rc = load_view(c, d, imgs[l].data(), ch, pitch[l], s, *opts, *vsel, *refine);
                // restorer step 1 (§21): the photometric-only estimate, with the term off, in the view's context as loaded.
                // The geometric stage below replaces the whole state (gpm_set_state), so the view is loaded once.  With one
                // level this repeats the coarsest photometric stage when photo_iterations = params.iterations and there is
                // no photometric prior stage; it is run anyway rather than special-cased.
                if (rc == GPM_OK && restoring) {
                    float ms1 = 0.f;
                    rc = gpm_init(c);
                    if (rc == GPM_OK) rc = timer.sweep(c, restore->photo_iterations, &ms1);
                    if (rc == GPM_OK) rc = gpm_get_state(c, ph4.data(), nullptr, 0);
                    ms += ms1;
                    if (rc != GPM_OK) return fail_at("detail restorer's photometric estimate", l, i, rc);
                }
                for (int v = 0; v < s.nv && rc == GPM_OK; v++) rc = gpm_set_view_depth(c, v, dep(slot[s.source(v)]), 0, 0);
                if (rc == GPM_OK) rc = gpm_set_geometric(c, g->weight, g->max_err);
                if (rc == GPM_OK) rc = gpm_cost_eval(c, raw(l, k), cost.data(), 0);
                if (rc == GPM_OK) rc = gpm_set_state(c, raw(l, k), cost.data(), 0);
                if (rc == GPM_OK) rc = timer.sweep(c, g->geo_iterations, &ms);
                float ms2 = 0.f, bms = 0.f;                                   // the geometric prior stage (§20)
                if (rc == GPM_OK && P_geo)
                    rc = prior_stage(c, P_geo, P_geo->info ? P_geo->info + (size_t)l * n + i : nullptr, n4, cost, timer, &ms2, &bms);
                ms += ms2;
                long long n_detail = 0;
                if (rc == GPM_OK && restoring) {                              // restorer steps 2 (end) to 4 (§21)
                    float ms4 = 0.f;
                    if (P_geo) rc = prior_off(c, P_geo);
                    if (rc == GPM_OK) rc = gpm_get_state(c, n4.data(), nullptr, 0);                 // the planes of the geometric stage
                    if (rc == GPM_OK) rc = gpm_set_geometric(c, 0.f, g->max_err);                  // detection: photometric costs
                    if (rc == GPM_OK) rc = gpm_cost_eval(c, n4.data(), c_ms.data(), 0);
                    if (rc == GPM_OK) rc = gpm_cost_eval(c, ph4.data(), c_ph.data(), 0);
                    if (rc == GPM_OK) {
                        n_detail = detect_details(c_ms.data(), c_ph.data(), restore->threshold, npix[0], detail.data());
                        merge_planes(n4.data(), ph4.data(), detail.data(), npix[0]);
                        rc = gpm_set_geo_mask(c, detail.data(), 0, 0);
                    }
                    if (rc == GPM_OK) rc = gpm_set_geometric(c, g->weight, g->max_err);
                    if (rc == GPM_OK) rc = gpm_cost_eval(c, n4.data(), cost.data(), 0);
                    if (rc == GPM_OK) rc = gpm_set_state(c, n4.data(), cost.data(), 0);
                    if (rc == GPM_OK) rc = timer.sweep(c, restore->iterations, &ms4);
                    ms += ms4;
                }
                sweep_ms[l][k] += ms;  build_ms[l][k] += bms;
                if (rc == GPM_OK && l > 0) rc = gpm_get_state(c, raw(l, k), nullptr, 0);
                if (rc == GPM_OK && l == 0) {
                    rc = gpm_finalize(c);
                    if (rc == GPM_OK) rc = gpm_get_state(c, n4.data(), cost.data(), 0);
                    for (int j = 0; j < n_refs && rc == GPM_OK; j++) {
                        if (ref_of(j) != i) continue;
                        if (d->out_norm4) memcpy(d->out_norm4 + (size_t)j * npix[0] * 4, n4.data(), npix[0] * 4 * sizeof(float));
                        if (d->out_cost) memcpy(d->out_cost + (size_t)j * npix[0], cost.data(), npix[0] * sizeof(float));
                        device_of[j] = dev;  job_ms[j] = ms;  restored[j] = (int)n_detail;
                    }
                    if (rc == GPM_OK && d->out_dir && write_result(d->out_dir, i, n4.data(), d->height, d->width) != GPM_OK) {
                        set_err(fn + ": could not store the result of reference view " + std::to_string(i));
                        return false;
                    }
                }
                if (rc == GPM_OK && P_geo && !restoring) rc = prior_off(c, P_geo);
                if (rc == GPM_OK && restoring) rc = gpm_set_geo_mask(c, nullptr, 0, 0);
                if (rc == GPM_OK) rc = gpm_set_geometric(c, 0.f, g->max_err);
                return rc == GPM_OK ? true : fail_at("geometric stage", l, i, rc);
            });
            barrier.arrive_and_wait();
        }
        for (int l = 1; l < L; l++) if (lc[l]) gpm_destroy(lc[l]);
    });
    if (stats) {
        gpm_batch_stats* b = &stats->batch;
        b->jobs_done = 0;  b->sweep_ms_total = 0.0;
        for (int j = 0; j < n_refs; j++) if (device_of[j] >= 0) { b->jobs_done++;  b->sweep_ms_total += job_ms[j]; }
        if (b->per_job_sweep_ms) for (int j = 0; j < n_refs; j++) b->per_job_sweep_ms[j] = job_ms[j];
        if (b->per_job_views) for (int j = 0; j < n_refs; j++) b->per_job_views[j] = setup[0][ref_of(j)].nv;
        if (b->per_job_device) for (int j = 0; j < n_refs; j++) b->per_job_device[j] = device_of[j];
        stats->n_views = nV;
        if (stats->views) std::copy(views.begin(), views.end(), stats->views);
        for (int l = 0; l < GPM_MS_MAX_LEVELS; l++) {
            stats->level_sweep_ms[l] = stats->level_upsample_ms[l] = 0.0;
            for (int k = 0; l < L && k < nV; k++) { stats->level_sweep_ms[l] += sweep_ms[l][k];  stats->level_upsample_ms[l] += up_ms[l][k]; }
        }
    }
    if (restore && restore->restored) std::copy(restored.begin(), restored.end(), restore->restored);
    if (prior)
        for (int l = 0; l < GPM_MS_MAX_LEVELS; l++) {
            prior->level_build_ms[l] = 0.0;
            for (int k = 0; l < L && k < nV; k++) prior->level_build_ms[l] += build_ms[l][k];
        }
    return failed.load() ? GPM_E_STATE : GPM_OK;
}

extern "C" int gpm_ms_batch_run(const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                gpm_ms_batch_stats* stats)
{
    return ms_batch_run("gpm_ms_batch_run", m, opts, vsel, nullptr, nullptr, nullptr, stats);
}

extern "C" int gpm_ms_batch_run_prior(const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                      gpm_ms_prior_opts* prior, gpm_ms_batch_stats* stats)
{
    return ms_batch_run("gpm_ms_batch_run_prior", m, opts, vsel, prior, nullptr, nullptr, stats);
}

extern "C" int gpm_ms_batch_run_restore(const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                        gpm_ms_prior_opts* prior, const gpm_ms_restore_opts* restore, gpm_ms_batch_stats* stats)
{
    return ms_batch_run("gpm_ms_batch_run_restore", m, opts, vsel, prior, restore, nullptr, stats);
}

extern "C" int gpm_ms_batch_run_refine(const gpm_ms_batch_desc* m, const gpm_job_opts* opts, const gpm_view_sel* vsel,
                                       gpm_ms_prior_opts* prior, const gpm_ms_restore_opts* restore, const gpm_refine_opts* refine,
                                       gpm_ms_batch_stats* stats)
{
    return ms_batch_run("gpm_ms_batch_run_refine", m, opts, vsel, prior, restore, refine, stats);
}
