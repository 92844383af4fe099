"""The planar prior (DESIGN.md §18) on the GPU at the inputs where its construction and its bookkeeping break, exactly.

- gpm_build_planar_prior equals pyprior.build (support points, triangles, map and counts) bit for bit, and leaves the state
  untouched, on adversarial states: constant costs on one plane (a lattice of support points, every quadrilateral
  cocircular), NaN costs and ties, support sets with 0, 1, 2, only collinear or exactly 3 points, support planes out of
  the depth range, a support plane that almost contains its pixel's ray (its triangles leave the range partway), steps 1
  and 64, a step that divides neither size, the 4097-pixel limit and 1600 x 1200; a 4098-pixel context is refused;
- planes offered by gpm_offer_prior keep the identities the offer gave them (no renumbering gpm_set_state) through the
  sweeps that follow: twins without the memo, the duplicate skips or the early-out, with mask-7 launches or 3 warps stay
  bit-identical, also after a second build and offer and after an offer of an empty map;
- gpm_init with the term on stores the init-variant cost plus exactly pyprior's term;
- the prior sweep follows pypropagate's rule at 33 and 64 source views, windows 3 and 25 and fewer than 16 warps;
- the batch drivers with a prior stage that finds no support point equal the restated context flow."""
import time

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_adaptive_sampling import decision_chain
from test_gpu_planar_prior import make_scene, open_ctx, sigma

pytestmark = pytest.mark.gpu

f32 = np.float32


def smooth_plane(sc, n=(0.1, -0.2, -1.0), depth=500.0):
    """[4] plane (n, d) in the reference camera's frame through depth `depth` on the ray of the image centre, facing the
    camera"""
    Kinv = np.asarray(sc.cameras[0].K_inv, np.float32).astype(np.float64).reshape(3, 3)
    X0 = depth * (Kinv @ np.array([sc.cols / 2.0, sc.rows / 2.0, 1.0]))
    n = np.asarray(n, np.float64) / np.linalg.norm(n)
    if n @ X0 > 0:
        n = -n
    return np.array([*n, -n @ X0], f32)


def tiled(sc, plane):
    return np.ascontiguousarray(np.tile(plane, (sc.rows, sc.cols, 1)), dtype=f32)


def check_build(ctx, sc, planes, cost, step, support_cost):
    """set_state, build: counts, map and untouched state equal pyprior.build; returns its (points, triangles, map, counts)"""
    from oracle import pyprior
    planes, cost = np.ascontiguousarray(planes, f32), np.ascontiguousarray(cost, f32)
    ctx.set_state(planes, cost)
    info = ctx.build_planar_prior(step, support_cost)
    got = ctx.planar_prior()
    pts, tris, want, counts = pyprior.build(planes, cost, step, support_cost, sc.cameras[0], sc.params.depthMin, sc.params.depthMax)
    assert (info["support"], info["triangles"], info["with_prior"]) == counts, (step, support_cost)
    assert bits_equal(got, want) == 0, (step, support_cost, int((got != want).any(-1).sum()))
    p2, c2 = ctx.get_state()
    assert bits_equal(p2, planes) == 0 and bits_equal(c2, cost) == 0
    if counts[1] == 0:
        assert not got.view(np.uint32).any() and counts[2] == 0
    return pts, tris, want, counts


def cells(sc, step):
    return (sc.cols + step - 1) // step, (sc.rows + step - 1) // step


# ---- (a) constant costs: a lattice ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,step", [(53, 75, 5), (61, 83, 7), (44, 100, 6)])
def test_constant_cost_gives_the_lattice(rows, cols, step):
    """W - 1 and H - 1 are no multiples of the step: the last cells are partial.  Every tie goes to the cell's first pixel."""
    sc = make_scene(rows, cols)
    with open_ctx(sc) as ctx:
        planes = tiled(sc, smooth_plane(sc))
        pts, tris, _, counts = check_build(ctx, sc, planes, np.full((rows, cols), f32(0.25)), step, 1.0)
    cx, cy = cells(sc, step)
    assert pts == [(x * step, y * step) for y in range(cy) for x in range(cx)]
    assert counts[1] == 2 * (cx - 1) * (cy - 1) and counts[2] > 0


# ---- (b) NaN costs ---------------------------------------------------------------------------------------------------------
def test_nan_costs_never_win_a_cell():
    sc = make_scene(53, 75)
    step = 5
    rng = np.random.default_rng(3)
    cost = rng.uniform(0.1, 1.0, (sc.rows, sc.cols)).astype(f32)
    want_at = {}
    cost[0:5, 0:5] = np.nan                                       # whole cells of NaN: no support point
    cost[20:25, 35:40] = np.nan
    cost[50:53, 70:75] = np.nan                                   # the last, partial cell
    for cy, cx in ((1, 1), (2, 6), (9, 3)):                       # NaN where the cell's minimum was
        c = cost[cy * 5:cy * 5 + 5, cx * 5:cx * 5 + 5]
        i = np.unravel_index(np.argmin(c), c.shape)
        c[i] = np.nan
        c2 = np.where(np.isnan(c), np.inf, c)
        j = np.unravel_index(np.argmin(c2), c.shape)
        want_at[(cy, cx)] = (cx * 5 + j[1], cy * 5 + j[0])
    c = cost[5:10, 20:25]                                         # a tie after a NaN first pixel: the second pixel wins
    c[:] = f32(0.05)
    c[0, 0] = np.nan
    want_at[(1, 4)] = (21, 5)
    c = cost[30:35, 10:15]                                        # a tie with a NaN in the middle: the first pixel wins
    c[:] = f32(0.05)
    c[2, 3] = np.nan
    want_at[(6, 2)] = (10, 30)
    c = cost[40:45, 60:65]                                        # NaN everywhere but the last pixel
    c[:] = np.nan
    c[4, 4] = f32(0.5)
    want_at[(8, 12)] = (64, 44)
    with open_ctx(sc) as ctx:
        planes = tiled(sc, smooth_plane(sc))
        pts, tris, _, counts = check_build(ctx, sc, planes, cost, step, 2.0)
    cx, cy = cells(sc, step)
    assert counts[0] == cx * cy - 3 and counts[1] > 0
    for (y, x), p in want_at.items():
        assert p in pts, ((y, x), p)
    assert not any(np.isnan(cost[y, x]) for x, y in pts)


# ---- (c) chosen support sets ---------------------------------------------------------------------------------------------
def test_support_sets_without_triangles_give_an_empty_map():
    sc = make_scene(53, 75)
    rng = np.random.default_rng(4)
    base = rng.uniform(0.5, 1.0, (sc.rows, sc.cols)).astype(f32)
    planes = tiled(sc, smooth_plane(sc))
    row = base.copy()
    for cx in range(15):                                          # one row of cells, every support point on row 22
        row[22, cx * 5 + cx % 5] = f32(0.1)
    chosen = [base.copy()]                                        # the cheap pixels one at a time: 1, 2, 3 points
    for y, x in ((7, 12), (41, 20), (18, 66)):
        chosen.append(chosen[-1].copy())
        chosen[-1][y, x] = f32(0.1)
    with open_ctx(sc) as ctx:
        full = check_build(ctx, sc, planes, base, 5, 2.0)        # a full map first: every build below must clear it
        assert full[3][2] > 0
        got = [check_build(ctx, sc, planes, cost, 5, 0.2)[3] for cost in chosen[:3] + [row, chosen[3]]]
    assert [g[0] for g in got] == [0, 1, 2, 15, 3]
    assert [g[1] for g in got] == [0, 0, 0, 0, 1]
    assert got[-1][2] > 0


# ---- (d) out-of-range support planes ---------------------------------------------------------------------------------------
def grazing_plane(sc, x, y, depth_f32, lo, hi, seed):
    """A plane that almost contains the ray of pixel (x, y): its float32 prior_depth there is depth_f32 (in range), while
    the double back-projection of the triangle planes puts the point at a depth in (lo, hi)."""
    from oracle import pyprior
    cam = sc.cameras[0]
    Kinv = np.asarray(cam.K_inv, np.float32).astype(np.float64).reshape(3, 3)
    r = Kinv @ np.array([x, y, 1.0])
    rng = np.random.default_rng(seed)
    for _ in range(100000):
        t = np.cross(r, rng.normal(0, 1, 3))
        n = (t / np.linalg.norm(t) + rng.uniform(-2e-7, 2e-7) * r / np.linalg.norm(r)).astype(f32)
        unit = pyprior.prior_depth(np.array([*n, 1.0], f32), cam, f32(x), f32(y))
        if not np.isfinite(unit) or unit == 0:
            continue
        pl = np.array([*n, f32(depth_f32 / float(unit))], f32)
        d_f32 = float(pyprior.prior_depth(pl, cam, f32(x), f32(y)))
        d_f64 = -float(pl[3]) / (n.astype(np.float64) @ r)
        if sc.params.depthMin <= d_f32 <= sc.params.depthMax and lo < d_f64 < hi:
            return pl
    raise AssertionError("no grazing plane found")


def test_support_planes_out_of_range():
    from oracle import pyprior
    sc = make_scene(53, 75)
    step, lo, hi = 5, sc.params.depthMin, sc.params.depthMax
    P0 = smooth_plane(sc)
    planes = tiled(sc, P0)
    cost = np.full((sc.rows, sc.cols), f32(0.25))
    # the winners (each cell's first pixel) of four cells get planes out of range: beyond depthMax, before depthMin,
    # all-zero (NaN depth) and behind the camera
    far, near = smooth_plane(sc, depth=2.0 * hi), smooth_plane(sc, depth=0.5 * lo)
    planes[5, 5], planes[20, 35], planes[50, 70], planes[0, 40] = far, near, 0.0, [*far[:3], -far[3]]
    with open_ctx(sc) as ctx:
        pts, _, _, counts = check_build(ctx, sc, planes, cost, step, 1.0)
        cx, cy = cells(sc, step)
        assert counts[0] == cx * cy - 4
        assert not {(5, 5), (35, 20), (70, 50), (40, 0)} & set(pts)
        # a support plane almost containing its ray: in range in float32 at its pixel, beyond depthMax where the
        # triangle planes put it, so the triangles around it cross depthMax partway
        g = planes.copy()
        g[25, 35] = grazing_plane(sc, 35, 25, 0.9 * hi, 1.5 * hi, 4.5 * hi, 0)
        pts, tris, pm, counts = check_build(ctx, sc, g, cost, step, 1.0)
    assert (35, 25) in pts
    owner, _ = pyprior.raster_cover(pts, tris, sc.rows, sc.cols)
    has, _ = pyprior.has_prior(pm, sc.cameras[0], lo, hi)
    v = pts.index((35, 25))
    partial = [t for t, tri in enumerate(tris) if v in tri and has[owner == t].any() and not has[owner == t].all()]
    assert partial and int((owner >= 0).sum()) > counts[2]


# ---- (e) steps ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,step", [(37, 53, 1), (40, 130, 64), (40, 50, 64), (53, 75, 7)])
def test_steps(rows, cols, step):
    sc = make_scene(rows, cols)
    rng = np.random.default_rng(rows + cols + step)
    with open_ctx(sc) as ctx:
        ctx.init()
        init_planes, _ = ctx.get_state()
        smooth = tiled(sc, smooth_plane(sc))
        smooth[..., 3] *= (1.0 + rng.normal(0, 0.002, (rows, cols))).astype(f32)
        cost = rng.uniform(0.0, 1.0, (rows, cols)).astype(f32)
        for planes in (smooth, init_planes):
            _, _, _, counts = check_build(ctx, sc, planes, cost, step, 2.0)
            cx, cy = cells(sc, step)
            if planes is smooth:
                assert counts[0] == cx * cy
    if step == 1:
        assert counts[0] > 0.5 * rows * cols


# ---- (f) the 4097-pixel limit ----------------------------------------------------------------------------------------------
def test_width_limit():
    from gipuma_b200 import api
    sc = make_scene(32, 4097)
    rng = np.random.default_rng(9)
    planes = tiled(sc, smooth_plane(sc, n=(0.02, -0.05, -1.0)))
    with open_ctx(sc) as ctx:
        for cost in (np.full((32, 4097), f32(0.25)), rng.uniform(0, 1, (32, 4097)).astype(f32)):
            pts, _, _, counts = check_build(ctx, sc, planes, cost, 8, 2.0)
            assert max(x for x, _ in pts) == 4096 and counts[1] > 0 and counts[2] > 0
    wide = make_scene(32, 4098)
    with open_ctx(wide) as ctx:
        planes = tiled(wide, smooth_plane(wide, n=(0.02, -0.05, -1.0)))
        cost = np.full((32, 4098), f32(0.25))
        ctx.set_state(planes, cost)
        launches = ctx.stats()["launches"]
        with pytest.raises(api.GipumaError, match="-1"):
            ctx.build_planar_prior(8, 2.0)
        assert ctx.stats()["launches"] == launches
        with pytest.raises(api.GipumaError, match="-3"):            # no map was allocated
            ctx.planar_prior()
        p2, c2 = ctx.get_state()
        assert bits_equal(p2, planes) == 0 and bits_equal(c2, cost) == 0


# ---- (g) the measured size -------------------------------------------------------------------------------------------------
def test_build_at_1600x1200():
    t0 = time.perf_counter()
    sc = make_scene(1200, 1600)
    with open_ctx(sc) as ctx:
        ctx.init()
        ctx.sweep(1)
        planes, cost = ctx.get_state()
        _, _, _, counts = check_build(ctx, sc, planes, cost, 8, float(np.nanpercentile(cost, 60)))
    assert counts[1] > 0 and counts[2] > 0
    print("\n1600x1200 step 8: %s, %.1f s" % (counts, time.perf_counter() - t0))


# ---- identities after an offer ---------------------------------------------------------------------------------------------
# twins: the memo, the duplicate skips and the early-out off one at a time, one mask-7 launch per colour, 3 warps
TWINS = [{"memo": 0}, {"dedupe": 0}, {"prune": 0}, None, {"nwarps": 3}]


def offered_ctx(sc, ncc, adaptive, options, empty):
    """init, one sweep, build (empty: support_cost below every cost), the term on, the costs re-scored under it
    (cost_eval + set_state), then the offer: the offered planes keep the identities the offer gave them"""
    ctx = open_ctx(sc, ncc=ncc, adaptive=adaptive, options=options or {})
    ctx.init()
    ctx.sweep(1)
    info = ctx.build_planar_prior(5, -1.0 if empty else float(np.nanpercentile(ctx.get_state()[1], 60)))
    assert (info["triangles"] == 0) == empty
    ctx.set_prior(0.3 if ncc else 2.0, sigma(sc), 5.0)
    p, _ = ctx.get_state()
    ctx.set_state(p, ctx.cost_eval(p))
    before = ctx.get_state()
    ctx.offer_prior()
    after = ctx.get_state()
    changed = bits_equal(after[0], before[0]) + bits_equal(after[1], before[1])
    assert (changed == 0) == empty
    return ctx


def rebuild_and_offer(ctxs):
    """a second build from the swept state and a second offer, without set_state; all contexts stay bit-identical"""
    support_cost = float(np.nanpercentile(ctxs[0].get_state()[1], 60))
    before = ctxs[0].get_state()
    for ctx in ctxs:
        ctx.build_planar_prior(5, support_cost)
        ctx.offer_prior()
    ref = ctxs[0].get_state()
    assert bits_equal(ref[1], before[1]) > 0
    for ctx in ctxs[1:]:
        p, c = ctx.get_state()
        assert bits_equal(p, ref[0]) == 0 and bits_equal(c, ref[1]) == 0


@pytest.mark.parametrize("ncc,adaptive,variant", [(n, a, v) for v in ("once", "twice") for n in (False, True) for a in (False, True)] +
                                                 [(False, True, "empty"), (True, False, "empty")])
def test_offered_identities_hold_through_the_sweep(ncc, adaptive, variant):
    """once: the offer, two iterations; twice: the offer, one iteration, a second build and offer, two iterations.  An
    offered identity that collides with a later fresh one or an earlier one makes the memo or a duplicate skip drop a
    plane that pypropagate's rule accepts."""
    t0 = time.perf_counter()
    sc = make_scene(53, 75, box=15)
    empty = variant == "empty"
    A = offered_ctx(sc, ncc, adaptive, None, empty)
    twins = [(offered_ctx(sc, ncc, adaptive, o, empty), o) for o in TWINS]
    try:
        ref = A.get_state()
        for t, o in twins:
            p, c = t.get_state()
            assert bits_equal(p, ref[0]) == 0 and bits_equal(c, ref[1]) == 0, o
        A.reset_stats()
        if variant == "twice":
            decision_chain(sc, False, A, twins, iterations=1, adaptive=adaptive)
            rebuild_and_offer([A] + [t for t, _ in twins])
            decision_chain(sc, False, A, twins, iterations=2, adaptive=adaptive)
        else:
            decision_chain(sc, False, A, twins, iterations=2, adaptive=adaptive)
        st = A.stats()
    finally:
        for ctx in [A] + [t for t, _ in twins]:
            ctx.close()
    print("\noffer %s ncc=%s adaptive=%s: skipped %d of %d, %.2f s" % (variant, ncc, adaptive, st["skipped"], st["hypotheses"],
                                                                       time.perf_counter() - t0))


# ---- init with the term on -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ncc,geo", [(False, False), (False, True), (True, False), (True, True)])
def test_init_adds_exactly_the_term(ncc, geo):
    from oracle import pyprior
    sc = make_scene(61, 83)
    w = 0.3 if ncc else 2.0
    with open_ctx(sc, ncc=ncc, geo=geo) as off, open_ctx(sc, ncc=ncc, geo=geo) as on:
        off.init()
        off.sweep(1)
        off.build_planar_prior(5, float(np.nanpercentile(off.get_state()[1], 60)))
        pm = off.planar_prior()
        off.init()
        on.set_planar_prior(pm)
        on.set_prior(w, sigma(sc), 5.0)
        on.init()
        p_off, c_off = off.get_state()
        p_on, c_on = on.get_state()
    assert bits_equal(p_on, p_off) == 0
    want = pyprior.with_prior(c_off, p_off, pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax, w, sigma(sc), 5.0)
    assert bits_equal(c_on, want) == 0
    has, _ = pyprior.has_prior(pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax)
    assert (c_on[has] > c_off[has]).sum() > 0.5 * has.sum()


# ---- many views, windows 3 and 25, fewer warps -----------------------------------------------------------------------------
def shape_ctx(sc, ncc, geo, adaptive, options=None, weight=0.0):
    ctx = open_ctx(sc, ncc=ncc, geo=geo, adaptive=adaptive, options=options or {})
    ctx.init()
    ctx.sweep(1)
    ctx.build_planar_prior(5, float(np.nanpercentile(ctx.get_state()[1], 60)))
    if weight:
        ctx.set_prior(weight, sigma(sc), 5.0)
    return ctx


# views, box, NCC, geometric term, adaptive
SHAPES = [(33, 25, False, True, True), (64, 3, True, True, False), (64, 25, False, False, False), (64, 25, True, False, True),
          (33, 3, False, False, False)]


@pytest.mark.parametrize("views,box,ncc,geo,adaptive", SHAPES)
def test_prior_sweep_at_many_views(views, box, ncc, geo, adaptive):
    """test_gpu_planar_prior's chain with twins; box 25 is six sampling rounds, box 3 one"""
    from test_gpu_geometric import make_scene as rig_scene
    t0 = time.perf_counter()
    sc = rig_scene(40, 60, views, box=box)
    w = 0.3 if ncc else 2.0
    A = shape_ctx(sc, ncc, geo, adaptive, weight=w)
    A.offer_prior()
    planes, cost = A.get_state()
    twins = []
    for opts in ({"memo": 0}, {"prune": 0}, {"dedupe": 0}, None, {"nwarps": 3 if views == 64 else 7}):
        t = shape_ctx(sc, ncc, geo, adaptive, opts or {}, weight=w)
        t.set_planar_prior(A.planar_prior())
        t.set_state(planes, cost)
        twins.append((t, opts))
    try:
        A.set_state(planes, cost)
        A.reset_stats()
        decision_chain(sc, False, A, twins, iterations=2, adaptive=adaptive)
        st = A.stats()
    finally:
        for ctx in [A] + [t for t, _ in twins]:
            ctx.close()
    print("\nprior sweep %d views box %d ncc=%s geo=%s adaptive=%s: pruned %d of %d, %.2f s" %
          (views, box, ncc, geo, adaptive, st["pruned"], st["hypotheses"], time.perf_counter() - t0))
    if not ncc:
        if box == 25:
            assert st["pruned"] > 0                   # the bound with the prior term cuts hypotheses short
        else:
            assert st["pruned"] == 0                  # one round: the bound is the final cost


@pytest.mark.parametrize("ncc", [False, True])
def test_cost_eval_at_64_views_box_25(ncc):
    from oracle import pyprior
    from test_gpu_geometric import make_scene as rig_scene
    sc = rig_scene(40, 60, 64, box=25)
    w = 0.3 if ncc else 2.0
    with shape_ctx(sc, ncc, True, False) as ctx:
        pm = ctx.planar_prior()
        planes, _ = ctx.get_state()
        rng = np.random.default_rng(2)
        near = pm.copy()
        near[..., 3] *= f32(1.0) + rng.normal(0, 0.01, pm.shape[:2]).astype(f32)
        for hyp in (planes, np.where((pm == 0).all(-1, keepdims=True), planes, near).astype(f32)):
            c0 = ctx.cost_eval(hyp)
            ctx.set_prior(w, sigma(sc), 5.0)
            c1 = ctx.cost_eval(hyp)
            ctx.set_prior(0.0, sigma(sc), 5.0)
            want = pyprior.with_prior(c0, hyp, pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax, w, sigma(sc), 5.0)
            assert bits_equal(c1, want) == 0
            has, _ = pyprior.has_prior(pm, sc.cameras[0], sc.params.depthMin, sc.params.depthMax)
            assert (c1[has] > c0[has]).any() and bits_equal(c1[~has], c0[~has]) == 0


# ---- drivers with an empty prior -------------------------------------------------------------------------------------------
def empty_prior():
    import test_gpu_planar_prior as tp
    return dict(tp.PRIOR, support_cost=-1.0)                       # below every cost: no support point, an empty map


def test_batch_run_with_an_empty_prior(monkeypatch):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    import test_gpu_ncc as tn
    import test_gpu_planar_prior as tp
    c = gb._case("ragged", False)
    prior = empty_prior()
    counts = []
    with monkeypatch.context() as m:
        m.setattr(tp, "PRIOR", prior)
        tp._prior_flow(m, c["params"], counts)
        w4, wc = tn._restated_batch(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], **gb.KW)
    assert len(counts) == len(c["refs"]) and all(k["with_prior"] == 0 and k["triangles"] == 0 for k in counts)
    for devices in ((0,), (0, 0)):
        n4, cost, st = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], devices=devices, cam_scale=c["scale"],
                                     planar_prior=prior, photometric="ncc", ncc_min_std=tn.MIN_STD, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, devices
        assert st["prior"] == counts and all(k["with_prior"] == 0 for k in st["prior"]), devices


def test_geometric_pass_with_an_empty_prior(monkeypatch):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    import test_gpu_planar_prior as tp
    c = gb._case("fusion", False)
    prior = empty_prior()
    counts = []
    with monkeypatch.context() as m:
        m.setattr(tp, "PRIOR", prior)
        tp._prior_flow(m, c["params"], counts)
        w4, wc, w_pass1, w_views = gb._restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                                max_err=api.GEO_MAX_ERR, **gb.KW)
    assert counts and all(k["with_prior"] == 0 for k in counts)
    for devices in ((0,), (0, 0)):
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, planar_prior=prior, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, devices
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views, devices
        assert len(info["prior"]) == len(counts) and all(k["with_prior"] == 0 for k in info["prior"]), devices
