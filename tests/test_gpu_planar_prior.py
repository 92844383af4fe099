"""Planar prior (DESIGN.md §18) on the GPU, checked exactly against oracle/pyprior.py.

gpm_build_planar_prior must equal pyprior.build (support points, triangles, prior map and counts) bit for bit at ragged
sizes; gpm_cost_eval must equal the cost without the prior plus pyprior's term; every close and far launch must follow
oracle/pypropagate.py's rule with the prior cost (fixed and adaptive propagation, the lower bound cutting hypotheses
short), and twins without the memo, the early-out or the duplicate skips must stay bit-identical; gpm_offer_prior must
equal its restatement; weight 0 and a switch back to 0 must give the run of a context that never had a prior; refusals
must change nothing."""
import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_adaptive_sampling import decision_chain
from test_gpu_sweep_any_size import cost_of

pytestmark = pytest.mark.gpu

f32 = np.float32
MIN_STD, GEO_W, GEO_ERR = 4.0, 0.3, 6.0


def make_scene(rows, cols, views=4, box=9, seed=None):
    from gipuma_b200 import scene as S
    sc = S.make_config(2, rows=rows, cols=cols, n_views=views, iterations=2, seed=seed or rows * 1000 + cols)
    sc.params.box_hsize = sc.params.box_vsize = box
    return sc


def open_ctx(sc, ncc=False, geo=False, adaptive=False, options=None, seed=7):
    from gipuma_b200 import api
    from test_gpu_geometric import depth_maps
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    if ncc:
        ctx.set_photometric("ncc", MIN_STD)
    ctx.load_scene(sc, seed=seed)
    if geo:
        for v, d in enumerate(depth_maps(sc, 3)):
            ctx.set_view_depth(v, d)
        ctx.set_geometric(GEO_W, GEO_ERR)
    if adaptive:
        ctx.set_propagation("adaptive")
    return ctx


def sigma(sc):
    return (sc.params.depthMax - sc.params.depthMin) / 64.0


@pytest.mark.parametrize("rows,cols,step", [(53, 75, 5), (31, 33, 3), (97, 65, 7), (550, 1000, 5)])
def test_build_equals_restatement(rows, cols, step):
    from oracle import pyprior
    sc = make_scene(rows, cols)
    ctx = open_ctx(sc)
    ctx.init()
    ctx.sweep(1)
    planes, cost = ctx.get_state()
    support_cost = float(np.nanpercentile(cost, 60))
    info = ctx.build_planar_prior(step, support_cost)
    got = ctx.planar_prior()
    pts, tris, want, counts = pyprior.build(planes, cost, step, support_cost, sc.cameras[0], sc.params.depthMin, sc.params.depthMax)
    assert (info["support"], info["triangles"], info["with_prior"]) == counts
    assert counts[1] > 0 and counts[2] > 0
    assert bits_equal(got, want) == 0
    # the state is untouched by a build
    p2, c2 = ctx.get_state()
    assert bits_equal(p2, planes) == 0 and bits_equal(c2, cost) == 0


def built_ctx(sc, weight, **kw):
    ctx = open_ctx(sc, **kw)
    ctx.init()
    ctx.sweep(1)
    ctx.build_planar_prior(5, float(np.nanpercentile(ctx.get_state()[1], 60)))
    if weight:
        ctx.set_prior(weight, sigma(sc), 5.0)
    return ctx


@pytest.mark.parametrize("ncc,geo", [(False, False), (False, True), (True, False), (True, True)])
def test_cost_eval_equals_restatement(ncc, geo):
    from oracle import pyprior
    sc = make_scene(61, 83)
    ctx = built_ctx(sc, 0.0, ncc=ncc, geo=geo)
    pm = ctx.planar_prior()
    planes, _ = ctx.get_state()
    rng = np.random.default_rng(1)
    near = pm.copy()
    near[..., 3] *= f32(1.0) + rng.normal(0, 0.01, pm.shape[:2]).astype(f32)        # close to the prior: unsaturated terms
    w = 0.4
    for hyp in (planes, near):
        hyp = np.where((pm == 0).all(-1, keepdims=True), planes, hyp).astype(f32)
        c0 = ctx.cost_eval(hyp)
        ctx.set_prior(w, sigma(sc), 5.0)
        c1 = ctx.cost_eval(hyp)
        ctx.set_prior(0.0, sigma(sc), 5.0)
        want = pyprior.with_prior(c0, hyp, pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax, w, sigma(sc), 5.0)
        assert bits_equal(c1, want) == 0
        has, _ = pyprior.has_prior(pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax)
        assert (c1[has] > c0[has]).any() and bits_equal(c1[~has], c0[~has]) == 0


@pytest.mark.parametrize("ncc,geo,adaptive", [(False, False, False), (False, False, True), (False, True, False),
                                              (True, False, True), (True, True, False)])
def test_sweep_decisions_exact_with_prior(ncc, geo, adaptive):
    sc = make_scene(53, 75, box=15)                  # two sampling rounds: the lower bound is tested once per hypothesis
    w = 0.3 if ncc else 2.0
    A = built_ctx(sc, w, ncc=ncc, geo=geo, adaptive=adaptive)
    A.offer_prior()
    planes, cost = A.get_state()
    twins = []
    for opts in ({"memo": 0}, {"prune": 0}, {"dedupe": 0}, None):
        t = built_ctx(sc, w, ncc=ncc, geo=geo, adaptive=adaptive, options=opts or {})
        t.set_planar_prior(A.planar_prior())
        t.set_state(planes, cost)
        twins.append((t, opts))
    A.set_state(planes, cost)
    A.reset_stats()
    decision_chain(sc, False, A, twins, iterations=2, adaptive=adaptive)
    if not ncc:
        assert A.stats()["pruned"] > 0


@pytest.mark.parametrize("fresh", [False, True])
def test_offer_equals_restatement(fresh):
    """fresh: the stored costs re-scored under the prior first (cost_eval + set_state), as the drivers' prior stage does"""
    from oracle import pyprior
    sc = make_scene(53, 75)
    ctx = built_ctx(sc, 0.5)
    pm = ctx.planar_prior()
    if fresh:
        p, _ = ctx.get_state()
        ctx.set_state(p, ctx.cost_eval(p))
    before = ctx.get_state()
    c_prior = ctx.cost_eval(pm)
    ctx.offer_prior()
    planes, cost = ctx.get_state()
    has, _ = pyprior.has_prior(pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax)
    take = has & (c_prior < before[1])
    assert take.sum() > 0
    assert bits_equal(planes, np.where(take[..., None], pm, before[0])) == 0
    assert bits_equal(cost, np.where(take, c_prior, before[1])) == 0


def test_weight_zero_and_switch_off_give_the_plain_run():
    sc = make_scene(64, 96)
    fresh = open_ctx(sc)
    fresh.run()
    want = fresh.get_state()
    a = open_ctx(sc)
    rng = np.random.default_rng(0)
    a.set_planar_prior(rng.normal(0, 1, (sc.rows, sc.cols, 4)).astype(f32))
    a.set_prior(0.0, 1.0, 5.0)
    a.run()
    b = built_ctx(sc, 0.5)
    b.run()
    with_prior = b.get_state()
    b.set_prior(0.0, sigma(sc), 5.0)
    b.run()
    for got in (a.get_state(), b.get_state()):
        assert bits_equal(got[0], want[0]) == 0 and bits_equal(got[1], want[1]) == 0
    assert bits_equal(with_prior[1], want[1]) != 0


def test_refusals_change_nothing():
    from gipuma_b200 import api
    sc = make_scene(40, 48)
    ctx = open_ctx(sc)
    ctx.init()
    before, launches = ctx.get_state(), ctx.stats()["launches"]
    with pytest.raises(api.GipumaError, match="-3"):
        ctx.set_prior(0.5, 1.0, 5.0)                                   # no map
    with pytest.raises(api.GipumaError, match="-3"):
        ctx.offer_prior()
    ctx.build_planar_prior(5, 1e30)
    launches = ctx.stats()["launches"]
    with pytest.raises(api.GipumaError, match="-1"):
        ctx.set_prior(1e6, 1.0, 5.0)                                   # a valid cost could reach MAXCOST
    ctx.set_photometric("ncc", MIN_STD)
    ctx.set_view_selection("joint")
    with pytest.raises(api.GipumaError, match="-1"):
        ctx.set_prior(0.5, 1.0, 5.0)                                   # joint view selection
    ctx.set_view_selection("off")
    ctx.set_prior(0.3, 1.0, 5.0)
    with pytest.raises(api.GipumaError, match="-1"):
        ctx.set_view_selection("joint")
    with pytest.raises(api.GipumaError, match="-1"):
        ctx.set_option("neighbours", 20)
    with pytest.raises(api.GipumaError, match="-3"):
        ctx.shard_stage(0, 0, None, 1, None)
    assert ctx.stats()["launches"] == launches
    after = ctx.get_state()
    assert bits_equal(after[0], before[0]) == 0 and bits_equal(after[1], before[1]) == 0
    col = api.Context(sc.cols, sc.rows, sc.n_views)
    from gipuma_b200 import scene as S
    csc = S.colorize(make_scene(40, 48))
    col.load_scene(csc)
    col.set_planar_prior(np.zeros((sc.rows, sc.cols, 4), f32))
    with pytest.raises(api.GipumaError, match="-1"):
        col.set_prior(0.5, 1.0, 5.0)


# ---- drivers ----------------------------------------------------------------------------------------------------------
PRIOR = {"weight": 2.0, "depth_sigma": 0.05, "normal_sigma_deg": 5.0, "step": 5, "support_cost": 1e30, "iterations": 2}


def _prior_flow(m, params, made):
    """Context calls that restate the drivers' prior stage: after the params.iterations sweeps of a job that started with
    init (batch jobs, geometric pass 1), build, set_prior, cost_eval + set_state, offer, PRIOR["iterations"] sweeps; the
    term off after that job's finalize."""
    from gipuma_b200 import api
    base_init, base_sweep, base_finalize = api.Context.init, api.Context.sweep, api.Context.finalize

    def init(self):
        base_init(self)
        self._photo_job = True

    def sweep(self, iterations):
        base_sweep(self, iterations)
        if getattr(self, "_photo_job", False):
            assert iterations == params.iterations
            made.append(self.build_planar_prior(PRIOR["step"], PRIOR["support_cost"]))
            self.set_prior(PRIOR["weight"], PRIOR["depth_sigma"], PRIOR["normal_sigma_deg"])
            p, _ = self.get_state()
            self.set_state(p, self.cost_eval(p))
            self.offer_prior()
            base_sweep(self, PRIOR["iterations"])

    def finalize(self):
        base_finalize(self)
        if getattr(self, "_photo_job", False):
            self.set_prior(0.0, PRIOR["depth_sigma"], PRIOR["normal_sigma_deg"])
            self._photo_job = False

    def run(self):
        self.init()
        self.sweep(params.iterations)
        self.finalize()
        return 0.0
    for name, fn in (("init", init), ("sweep", sweep), ("finalize", finalize), ("run", run)):
        m.setattr(api.Context, name, fn)


@pytest.mark.parametrize("name,photometric", [("fusion", "pm"), ("ragged", "ncc")])
def test_batch_run_prior_equals_the_context_flow(name, photometric, monkeypatch):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    import test_gpu_ncc as tn
    c = gb._case(name, False)
    counts = []
    with monkeypatch.context() as m:
        if photometric == "pm":                    # the restated flow sets NCC; keep the PM cost
            m.setattr(api.Context, "set_photometric", lambda self, kind="pm", min_std=0.0: None)
        _prior_flow(m, c["params"], counts)
        w4, wc = tn._restated_batch(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], **gb.KW)
    assert len(counts) == len(c["refs"]) and all(k["with_prior"] > 0 for k in counts)
    kw = dict(photometric="ncc", ncc_min_std=tn.MIN_STD) if photometric == "ncc" else {}
    for devices in ((0,), (0, 0)):
        n4, cost, st = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], devices=devices, cam_scale=c["scale"],
                                     planar_prior=PRIOR, **kw, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
        assert st["prior"] == counts, devices
    off, _, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], cam_scale=c["scale"], **kw, **gb.KW)
    assert bits_equal(off, w4) > 0                                        # the stage reached the jobs


@pytest.mark.parametrize("name", ["fusion", "ragged"])
def test_geometric_pass_prior_equals_the_context_flow(name, monkeypatch):
    """The prior stage in pass 1 only; pass 2 (no init) starts from the pass-1 planes without the term."""
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case(name, False)
    counts = []
    with monkeypatch.context() as m:
        _prior_flow(m, c["params"], counts)
        w4, wc, w_pass1, w_views = gb._restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                                max_err=api.GEO_MAX_ERR, **gb.KW)
    for devices in ((0,), (0, 0)):
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, planar_prior=PRIOR, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views, devices
        assert sorted(k["with_prior"] for k in info["prior"]) == sorted(k["with_prior"] for k in counts)


def test_drivers_refuse_before_any_cuda_call():
    import ctypes as C
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case("fusion", False)
    with pytest.raises(ValueError, match="joint view selection"):
        api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], photometric="ncc", view_selection="joint", planar_prior=PRIOR)
    L = api.load_library()
    imgs = np.ascontiguousarray(c["images"], dtype=f32)
    d, _keep = api._batch_desc(imgs, c["Ps"], c["params"], c["refs"], (0,), c["scale"], 5.0, 45.0, 6, 1, None, None, None)
    bad = api.GpmPriorOpts(2.0, 0.0, 5.0, 5, 1.0, 2, None)                  # depth_sigma 0
    assert L.gpm_batch_run_prior(C.byref(d), C.byref(api.job_opts()), C.byref(api.view_sel()), C.byref(bad), None) == -1
    assert "depth_sigma" in L.gpm_batch_last_error().decode()
    joint = api.view_sel("joint")
    ncc = api.job_opts("ncc")
    ok = api.GpmPriorOpts(2.0, 0.05, 5.0, 5, 1.0, 2, None)
    assert L.gpm_batch_run_prior(C.byref(d), C.byref(ncc), C.byref(joint), C.byref(ok), None) == -1
    assert "planar prior" in L.gpm_batch_last_error().decode()
