"""Joint view selection (DESIGN.md §17) on the GPU, checked against oracle/pyjvs.py.

With beta = 1e30 every confidence is exactly 1 and every operation of a launch is IEEE-exact, so every close, far and
combined propagation launch must equal pyjvs.expected() bit for bit in planes, costs and selected-views masks outside the
ambiguous pixels, with fixed and adaptive propagation, with and without the geometric term, at t = 0 and after sweeps, at
ragged sizes with gridDim.z splits and on adversarial states.  The per-view cost rows come from one-view contexts'
gpm_cost_eval of the candidate plane maps, the combination rule's fallback from the checked context's own gpm_cost_eval.
Refinement is checked by its invariants.  With beta = 0.3 the launches must agree wherever the decision is clear of the
MUFU.EX2 error bound.  Twins without memo, prune or dedupe stay bit-identical; mode switches follow each mode's rule; the
batch drivers equal the Context-call flows; refusals change nothing."""
import time

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

f32 = np.float32
WEIGHT, MAX_ERR, MIN_STD = 0.3, 6.0, 4.0
EXACT = {"beta": 1e30}
# ex2.approx.ftz.f32 (MUFU.EX2) has a relative error below 2^-22 (PTX ISA).  A confidence, and so s_j and a rule weight w_j,
# is then off by a relative delta <= 2^-21 after the roundings; a weighted mean sum w c / sum w moves by at most
# 2 delta max|c_j - mean| <= 2 delta * 4 (c_j = NCC + geometric term <= 2 + WEIGHT * MAX_ERR < 4), and the two sequential
# sums of up to V terms, on inputs that differ in the last bits, may round differently by V ulp of 4.  With V <= 10:
# 8 * 2^-21 + 10 * 4 * 2^-23 < 9e-6, a factor of 10 under TOL; at GPM_MAX_VIEWS = 64: 8 * 2^-21 + 64 * 4 * 2^-23 < 3.5e-5, a
# factor of 2.9 under TOL.
TOL = 1e-4
REPORT = {}

# id: (rows, cols, views, box, geometric term, adaptive propagation, sweeps before the checked launches[, parameters over
# EXACT]).  33 and 64 views put a second view in every lane (views lane + 32) and the upper half in the 64-bit masks; at
# 64 views and box 25 with the geometric term each warp keeps the largest scratch of any kernel.
CASES = {
    "fixed_53x75": (53, 75, 4, 15, False, False, 0),
    "adaptive_53x75_t2": (53, 75, 4, 15, False, True, 2),
    "geo_fixed_53x75_t2": (53, 75, 4, 15, True, False, 2),
    "geo_adaptive_45x71": (45, 71, 4, 9, True, True, 0),
    "fixed_8x8": (8, 8, 2, 9, False, False, 0),
    "adaptive_31x33_t5": (31, 33, 3, 11, False, True, 5),
    "adaptive_550x1000_t1": (550, 1000, 3, 9, False, True, 1),
    "fixed_33v_box25": (40, 60, 33, 25, False, False, 0),
    "geo_adaptive_64v_box3": (40, 60, 64, 3, True, True, 0),
    "geo_fixed_64v_box25": (40, 60, 64, 25, True, False, 0),
    "fixed_1v_good1_t2": (53, 75, 1, 15, False, False, 2, {"n_good": 1}),
    "fixed_1v_t2": (53, 75, 1, 15, False, False, 2),
}
MANY = ["fixed_33v_box25", "geo_adaptive_64v_box3", "geo_fixed_64v_box25"]
TWINS = [{"memo": 0}, {"prune": 0}, {"dedupe": 0}]


def make_scene(case):
    import test_gpu_geometric as tg
    return tg.make_scene(*CASES[case][:4])


def exact(case):
    """EXACT with the case's own parameters on top."""
    return dict(EXACT, **(CASES[case][7] if len(CASES[case]) > 7 else {}))


def twins_of(case):
    """The twins' options; at many views or the largest window the host picks fewer than 16 warps, so one more twin runs
    at another warp count."""
    views, box = CASES[case][2:4]
    return TWINS + ([{"nwarps": 3 if views == 64 else 7}] if views > 32 or box == 25 else [])


def upper_masks_reached(masks):
    """Bits >= 32 set, and not the same set at every pixel."""
    hi = np.asarray(masks, np.uint64) >> np.uint64(32)
    return bool((hi != 0).any()) and len(np.unique(hi)) > 1


def open_jvs(case, sc, seed, options=None, params=EXACT, kind="joint"):
    from gipuma_b200 import api
    from test_gpu_geometric import depth_maps
    geo, adaptive = CASES[case][4:6]
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    ctx.set_photometric("ncc", MIN_STD)
    ctx.load_scene(sc, seed=seed)
    if geo:
        for v, d in enumerate(depth_maps(sc, 3)):
            ctx.set_view_depth(v, d)
        ctx.set_geometric(WEIGHT, MAX_ERR)
    ctx.set_propagation("adaptive" if adaptive else "fixed")
    ctx.set_view_selection(kind, **params)
    return ctx


class Rows:
    """Per-view rows of a plane map from one-view contexts: (m, c) [H, W, V], c = m + g with the geometric term."""

    def __init__(self, case, sc):
        from test_gpu_geometric import depth_maps, open_ctx
        geo = CASES[case][4]
        depths = depth_maps(sc, 3) if geo else None
        self.m = [open_ctx(sc, views=[v]) for v in range(sc.n_views)]
        self.c = [open_ctx(sc, depths=depths, weight=WEIGHT, views=[v]) for v in range(sc.n_views)] if geo else []
        for ctx in self.m + self.c:
            ctx.set_photometric("ncc", MIN_STD)

    def __call__(self, planes):
        m = np.stack([ctx.cost_eval(planes) for ctx in self.m], axis=-1)
        c = np.stack([ctx.cost_eval(planes) for ctx in self.c], axis=-1) if self.c else m
        return m, c

    def close(self):
        for ctx in self.m + self.c:
            ctx.close()


def state(ctx):
    p, c = ctx.get_state()
    return p, c, ctx.view_masks()


def same_state(a, b):
    """Byte-equal planes, costs and masks (device outputs against device outputs)."""
    return all(np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8)) for x, y in zip(a, b))


def check_launch(A, rows, sc, case, colour, mask, t, params=EXACT, tol=None):
    """One launch of A against pyjvs.expected; returns (compared, ambiguous, accepted) pixel counts of this colour."""
    from oracle import pyjvs
    adaptive = CASES[case][5]
    cam, prm = sc.cameras[0], sc.params
    before = state(A)
    det = {}
    want = pyjvs.expected(before[0], before[1], before[2], colour, mask & 3, rows, A.cost_eval, cam, prm.depthMin,
                          prm.depthMax, params, t, adaptive=adaptive, details=det)
    A.phase(colour, mask)
    got = state(A)
    H, W = sc.rows, sc.cols
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    amb = want[3].copy()
    if tol is not None:                                  # the decision must be clear of the ex2 error
        vals = np.stack([det["start"]] + det["scores"])
        for i in range(len(vals)):
            for j in range(i + 1, len(vals)):
                d = np.abs(vals[i] - vals[j])
                amb |= (d > 0) & (d <= 2 * tol)
    assert np.array_equal(got[2][~amb], want[2][~amb]), ("masks", case, colour, mask)
    assert not (got[2][~mine] != before[2][~mine]).any()
    if mask & 4:                                         # refinement: invariants under the launch's weights
        changed = (got[0].view(np.uint32) != before[0].view(np.uint32)).any(axis=-1)
        m, c = rows(got[0])
        rescored = pyjvs.weighted(det["w"], c, A.cost_eval(got[0]))
        ok = mine & ~amb
        if tol is None:
            assert bits_equal(got[1][ok], rescored[ok]) == 0, ("refined cost", case, colour)
        assert np.all(got[1][ok] <= want[1][ok] + (tol or 0.0))
        assert bits_equal(got[0][~mine], before[0][~mine]) == 0
        n = got[0][changed & mine][:, :3].astype(np.float64)
        assert np.all(np.abs(np.linalg.norm(n, axis=-1) - 1.0) <= 1e-5)
        return int((mine & ~amb).sum()), int((mine & amb).sum()), int((changed & mine).sum())
    bad = (got[0].view(np.uint32) != want[0].view(np.uint32)).any(axis=-1)
    if tol is None:
        bad |= got[1].view(np.uint32) != want[1].view(np.uint32)
    else:
        bad |= ~(np.abs(got[1] - want[1]) <= tol)
    bad &= ~amb
    assert not bad.any(), (case, colour, mask, int(bad.sum()), np.argwhere(bad)[:8].tolist())
    accepted = mine & (got[0].view(np.uint32) != before[0].view(np.uint32)).any(axis=-1)
    return int((mine & ~amb).sum()), int((mine & amb).sum()), int(accepted.sum())


def chain(case, sc, A, twins, rows, t, params=EXACT, tol=None, masks=(1, 2, 3, 4)):
    stats = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}
    for colour in (0, 1):
        for mask in masks:
            n, a, acc = check_launch(A, rows, sc, case, colour, mask, t, params, tol)
            stats["compared"] += n
            stats["ambiguous"] += a
            stats["refined" if mask == 4 else "accepted"] += acc
            ref = state(A)
            for ctx in twins:
                ctx.phase(colour, mask)
                assert same_state(state(ctx), ref), ("twin", colour, mask)
    return stats


@pytest.mark.parametrize("case", list(CASES))
def test_jvs_launches_exact(case):
    t0 = time.perf_counter()
    sc = make_scene(case)
    sweeps = CASES[case][6]
    seed = 7000 + sc.rows + sc.cols
    A = open_jvs(case, sc, seed, params=exact(case))
    twins = [open_jvs(case, sc, seed, o, params=exact(case)) for o in twins_of(case)]
    rows = Rows(case, sc)
    try:
        for ctx in [A] + twins:
            ctx.init()
            ctx.sweep(sweeps)
        assert same_state(state(A), state(twins[0]))
        if sweeps:
            assert A.view_masks().any()
        A.reset_stats()
        st = chain(case, sc, A, twins, rows, sweeps, params=exact(case))
        s = A.stats()
        assert s["pruned"] == 0 and (s["skipped"] > 0 or sc.rows * sc.cols < 1000)
        if sc.n_views > 32:
            assert upper_masks_reached(A.view_masks())
    finally:
        rows.close()
        for ctx in [A] + twins:
            ctx.close()
    total = st["compared"] + st["ambiguous"]
    assert st["accepted"] > 0 and (st["refined"] > 0 or sweeps >= 5)          # late refinements may all be rejected
    assert st["ambiguous"] <= max(4, 0.005 * total), st
    REPORT[case] = dict(st, seconds=round(time.perf_counter() - t0, 2))
    print("\n%s: %s" % (case, REPORT[case]))


def hostile(sc, A, rng):
    """adversarial_state's planes (bit-equal neighbours, out of range, NaN / +inf costs) with tied costs on top."""
    from test_gpu_sweep_any_size import adversarial_state, cost_of
    n0, _ = A.get_state()
    pl, cost = adversarial_state(sc, n0, cost_of(A), rng, False, False)
    H, W = cost.shape
    tie = rng.random((H, W)) < 0.33
    cost[tie] = np.round(cost[tie] * 8) / 8
    cost[rng.random((H, W)) < 0.02] = np.nan
    cost[rng.random((H, W)) < 0.02] = np.inf
    return pl, cost.astype(f32)


@pytest.mark.parametrize("case", ["fixed_53x75", "adaptive_53x75_t2", "geo_adaptive_45x71"] + MANY)
def test_jvs_launches_exact_on_adversarial_states(case):
    t0 = time.perf_counter()
    sc = make_scene(case)
    A = open_jvs(case, sc, 77, params=exact(case))
    twins = [open_jvs(case, sc, 77, o, params=exact(case)) for o in twins_of(case)]
    rows = Rows(case, sc)
    try:
        A.init()
        pl, cost = hostile(sc, A, np.random.default_rng(11))
        for ctx in [A] + twins:
            ctx.set_state(pl, cost)
        assert not A.view_masks().any()                      # gpm_set_state clears the masks (and t)
        st = chain(case, sc, A, twins, rows, 0, params=exact(case))
        if sc.n_views > 32:
            assert upper_masks_reached(A.view_masks())
        st2 = chain(case, sc, A, twins, rows, 0, params=exact(case))   # now with remembered views
    finally:
        rows.close()
        for ctx in [A] + twins:
            ctx.close()
    assert st["accepted"] + st2["accepted"] > 0
    REPORT["adversarial_" + case] = (st, st2, round(time.perf_counter() - t0, 2))
    print("\nadversarial %s: %s" % (case, REPORT["adversarial_" + case]))


@pytest.mark.parametrize("case", ["fixed_53x75", "geo_adaptive_45x71", "geo_adaptive_64v_box3"])
def test_jvs_launches_within_the_ex2_tolerance(case):
    """beta = 0.3 (the default): the device's MUFU.EX2 and numpy's exp2 differ in the last bits, so costs agree within TOL
    and decisions wherever every pair of competing weighted costs is more than 2 TOL apart."""
    from gipuma_b200 import api
    sc = make_scene(case)
    A = open_jvs(case, sc, 91, params={})
    rows = Rows(case, sc)
    try:
        A.init()
        A.sweep(1)
        st = chain(case, sc, A, [], rows, 1, params=api.JVS_DEFAULTS, tol=TOL)
    finally:
        rows.close()
        A.close()
    total = st["compared"] + st["ambiguous"]
    # a weighted mean over 64 views puts competing scores closer together, so more decisions fall within 2 TOL of each
    # other: 3.3 % of the pixels on an H100 80GB HBM3 (700 W) at 64 views, under 2 % at 4
    assert st["accepted"] > 0 and st["ambiguous"] <= (0.05 if sc.n_views > 32 else 0.02) * total, st
    REPORT["tolerance_" + case] = st
    print("\ntolerance %s: %s" % (case, st))


def test_mask7_launches_and_sweeps_equal_the_twins():
    """One mask-7 launch per colour, and gpm_sweep, in joint mode: twins without memo, prune or dedupe hold the same bits."""
    case = "adaptive_53x75_t2"
    sc = make_scene(case)
    ctxs = [open_jvs(case, sc, 5)] + [open_jvs(case, sc, 5, o) for o in TWINS]
    try:
        for ctx in ctxs:
            ctx.init()
            ctx.sweep(1)
            ctx.phase(0, 7)
            ctx.phase(1, 7)
            ctx.sweep(2)
        ref = state(ctxs[0])
        for ctx in ctxs[1:]:
            assert same_state(state(ctx), ref)
    finally:
        for ctx in ctxs:
            ctx.close()


def test_switching_off_joint_off_follows_each_rule_and_back_to_off_matches_a_fresh_context():
    from oracle import pyacs
    from test_gpu_sweep_any_size import cost_of
    case = "adaptive_53x75_t2"
    sc = make_scene(case)
    prm, cam = sc.params, sc.cameras[0]
    A, fresh = open_jvs(case, sc, 31, kind="off"), open_jvs(case, sc, 31, kind="off")
    rows = Rows(case, sc)
    try:
        A.init()
        A.sweep(1)
        for step, kind in enumerate(["joint", "off", "joint", "off"]):
            A.set_view_selection(kind, **EXACT)
            colour = step & 1
            for mask in (1, 2, 3):
                if kind == "joint":
                    check_launch(A, rows, sc, case, colour, mask, 1)
                else:
                    before = A.get_state()
                    want = pyacs.expected(before[0], before[1], colour, mask, cost_of(A), cam, prm.depthMin, prm.depthMax)
                    A.phase(colour, mask)
                    got = A.get_state()
                    bad = ((got[0].view(np.uint32) != want[0].view(np.uint32)).any(axis=-1) |
                           (got[1].view(np.uint32) != want[1].view(np.uint32))) & ~want[2]
                    assert not bad.any(), (step, mask, int(bad.sum()))
            A.phase(colour, 4)
        A.set_view_selection("joint")
        A.run()
        A.set_view_selection("off")
        A.run()
        fresh.run()
        assert same_state(A.get_state(), fresh.get_state())
    finally:
        rows.close()
        A.close()
        fresh.close()


def test_joint_run_differs_from_off():
    case = "fixed_53x75"
    sc = make_scene(case)
    with open_jvs(case, sc, 5, params={}) as a, open_jvs(case, sc, 5, kind="off") as b:
        a.run()
        b.run()
        assert bits_equal(a.get_state()[0], b.get_state()[0]) > 0


# ---- drivers ----------------------------------------------------------------------------------------------------------
def _joint_contexts(monkeypatch, min_std):
    from gipuma_b200 import api
    made = []

    class JointContext(api.Context):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.set_photometric("ncc", min_std)
            self.set_view_selection("joint")
            made.append(self)
    monkeypatch.setattr(api, "Context", JointContext)
    return made


@pytest.mark.parametrize("name", ["fusion", "ragged"])
def test_batch_run_joint_equals_the_context_flow(name, monkeypatch):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    import test_gpu_ncc as tn
    c = gb._case(name, False)
    with monkeypatch.context() as m:
        made = _joint_contexts(m, tn.MIN_STD)
        w4, wc = tn._restated_batch(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], **gb.KW)
    assert len(made) == 1
    for devices in ((0,), (0, 0)):
        n4, cost, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], devices=devices, cam_scale=c["scale"],
                                    photometric="ncc", ncc_min_std=tn.MIN_STD, view_selection="joint", **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
    off, _, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], cam_scale=c["scale"], photometric="ncc",
                              ncc_min_std=tn.MIN_STD, **gb.KW)
    assert bits_equal(off, w4) > 0                                        # the mode reached the jobs


@pytest.mark.parametrize("name,propagation", [("fusion", "fixed"), ("ragged", "adaptive")])
def test_geometric_pass_joint_equals_the_context_flow(name, propagation, monkeypatch):
    """Both passes in joint mode; pass 2 starts at t = 0 after its gpm_set_state."""
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case(name, False)
    with monkeypatch.context() as m:
        made = _joint_contexts(m, api.NCC_MIN_STD)
        base_init = api.Context.__init__

        def with_propagation(self, *a, **k):
            base_init(self, *a, **k)
            self.set_propagation(propagation)
        m.setattr(api.Context, "__init__", with_propagation)
        w4, wc, w_pass1, w_views = gb._restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                                max_err=api.GEO_MAX_ERR, **gb.KW)
    assert len(made) == 1
    for devices in ((0,), (0, 0)):
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, photometric="ncc", propagation=propagation,
                                            view_selection="joint", **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views, devices


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals_leave_launch_count_and_state_untouched():
    import ctypes as C
    from gipuma_b200 import api
    E_ARG, E_STATE = -1, -3
    case = "fixed_53x75"
    sc = make_scene(case)
    with open_jvs(case, sc, 3) as ctx, open_jvs(case, sc, 3) as twin:
        L, h = ctx.lib, ctx.h
        ctx.init()
        ctx.sweep(1)
        before, launches = state(ctx), ctx.stats()["launches"]
        colour = np.zeros((sc.rows, sc.cols, 4), f32)
        cam = api.pack_camera(sc.cameras[0])
        bad = [api.GpmViewSel(2, 0.8, 90, 1.2, 3, 3, 0.3, 0.2), api.GpmViewSel(1, -0.8, 90, 1.2, 3, 3, 0.3, 0.2),
               api.GpmViewSel(1, 0.8, 90, 1.2, 9, 3, 0.3, 0.2), api.GpmViewSel(1, 0.8, 90, 1.2, 3, 3, float("nan"), 0.2)]
        calls = [(lambda v=v: L.gpm_set_view_selection(h, C.byref(v)), E_ARG) for v in bad]
        calls += [(lambda: L.gpm_set_view_selection(h, None), E_ARG),
                  (lambda: L.gpm_set_photometric(h, 0, C.c_float(0.0)), E_ARG),           # PM while joint
                  (lambda: L.gpm_set_option(h, b"neighbours", 20), E_ARG),
                  (lambda: L.gpm_set_reference_color(h, C.c_void_p(colour.ctypes.data), 0, 0, C.byref(cam)), E_ARG),
                  (lambda: L.gpm_shard_stage(h, 0, 1, None, 1, None), E_STATE),
                  (lambda: L.gpm_shard_finish_init(h, C.c_void_p(1), 1), E_STATE),
                  (lambda: L.gpm_shard_comm_attach(h, None, 0, 1), E_STATE),
                  (lambda: L.gpm_shard_comm_init(h, None, 0, 1), E_STATE),
                  (lambda: L.gpm_shard_run(h, None), E_STATE)]
        for call, code in calls:
            assert call() == code, L.gpm_last_error().decode()
        assert L.gpm_shard_num_stages(h) == -1 and L.gpm_shard_stage_floats(h, 1) == -1
        with pytest.raises(api.GipumaError, match="grey"):
            ctx.set_view(0, colour, sc.cameras[sc.subset[0]])
        assert ctx.stats()["launches"] == launches
        assert same_state(state(ctx), before)
        ctx.sweep(1)                                                         # still joint, still NCC, 8 neighbours
        twin.init()
        twin.sweep(2)
        assert same_state(state(ctx), state(twin))
        with pytest.raises(ValueError):
            ctx.set_view_selection("acmh")
        with pytest.raises(ValueError):
            ctx.set_view_selection("joint", n_bad=0)
        ctx.set_view_selection("off")
        ctx.set_photometric("pm")
        ctx.set_option("neighbours", 20)
        assert L.gpm_set_view_selection(h, C.byref(api.view_sel("joint"))) == E_ARG          # joint with PM, 20 neighbours
        ctx.set_option("neighbours", 8)
        assert L.gpm_set_view_selection(h, C.byref(api.view_sel("joint"))) == E_ARG          # joint with PM
        ctx.set_photometric("ncc", MIN_STD)
        ctx.set_view_selection("joint")
        assert ctx.stats()["launches"] == launches + 2
    sc4 = make_scene(case)
    from gipuma_b200 import scene as S
    sc4 = S.colorize(sc4)
    from test_gpu_geometric import open_ctx
    with open_ctx(sc4) as c4:
        assert c4.lib.gpm_set_view_selection(c4.h, C.byref(api.view_sel("joint"))) == E_ARG  # PM cost, colour images
