"""ACMH's refinement (DESIGN.md §23) on the GPU, bit for bit against oracle/pyrefine.py.

- after ctx.phase(colour, 4), planes and costs equal the restatement: the five candidates generated in numpy from the
  launch-start state, each costed with gpm_cost_eval at the refinement's rounding variant, accepted in order with strict <;
  at ragged sizes and a whole tile multiple, with PM (grey, colour), NCC, NCC + geometric term, geometric term + mask, the
  planar prior and adaptive propagation, 4, 33 and 64 views, and on adversarial states (ties, costs above MAXCOST, NaN);
- twins with the memo, the lower-bound early-out and the duplicate skips off, and with 5 warps per block, stay bit-identical;
- joint view selection, whose costs are not a pure function of the plane: determinism, and every changed plane is one of
  its pixel's five candidates;
- consecutive refinement launches draw different candidates, and gpm_set_rng reproduces the first;
- every refusal leaves the state and the launch count unchanged;
- each driver with refinement= equals its flow restated through Context calls, with 1-3 workers; None and "gipuma" equal
  today's outputs."""
import ctypes as C

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_sweep_any_size import cost_of

pytestmark = pytest.mark.gpu

f32 = np.float32
MAXCOST = f32(1000.0)
EPS = 0.02
GEO_W, GEO_ERR, MIN_STD = 0.3, 6.0, 4.0
E_ARG, E_STATE = -1, -3

# id: (rows, cols, views, mode)
CASES = {
    "pm_grey_53x75_v4": (53, 75, 4, "pm"),
    "pm_grey_64x96_v4": (64, 96, 4, "pm"),
    "pm_colour_53x75_v4": (53, 75, 4, "colour"),
    "ncc_150x101_v4": (101, 150, 4, "ncc"),
    "ncc_geo_53x75_v4": (53, 75, 4, "ncc_geo"),
    "geo_mask_53x75_v4": (53, 75, 4, "geo_mask"),
    "prior_53x75_v4": (53, 75, 4, "prior"),
    "adaptive_53x75_v4": (53, 75, 4, "adaptive"),
    "pm_grey_40x60_v33": (40, 60, 33, "pm"),
    "ncc_geo_40x60_v64": (40, 60, 64, "ncc_geo"),
    "pm_grey_64x64_v64": (64, 64, 64, "pm"),
}


def make_scene(rows, cols, views, colour=False):
    from test_gpu_geometric import make_scene as mk
    return mk(rows, cols, views, 9, colour)


def open_mode(sc, mode, seed=31, options=None, refinement="acmh"):
    from gipuma_b200 import api
    from test_gpu_geometric import depth_maps
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    if mode.startswith("ncc"):
        ctx.set_photometric("ncc", MIN_STD)
    ctx.load_scene(sc, seed=seed)
    if "geo" in mode:
        for v, d in enumerate(depth_maps(sc, 3)):
            ctx.set_view_depth(v, d)
        ctx.set_geometric(GEO_W, GEO_ERR)
    if mode == "geo_mask":
        ctx.set_geo_mask((np.random.default_rng(4).random((sc.rows, sc.cols)) < 0.5).astype(np.uint8))
    if mode == "adaptive":
        ctx.set_propagation("adaptive")
    ctx.set_refinement(refinement, EPS)
    return ctx


def start(ctx, sc, mode):
    """init, one iteration, and for the prior mode the prior built from that state and turned on.  Returns the launch
    counter r of the next refinement launch (2: the iteration's two launches)."""
    ctx.init()
    ctx.sweep(1)
    if mode == "prior":
        ctx.build_planar_prior(5, float(np.nanpercentile(ctx.get_state()[1], 60)))
        ctx.set_prior(1.0, (sc.params.depthMax - sc.params.depthMin) / 64.0, 5.0)
        p, _ = ctx.get_state()
        ctx.set_state(p, ctx.cost_eval(p))
    return 2


def restated(ctx, sc, colour, r, seed=31, before=None, eps=EPS):
    """The state the restatement expects after phase(colour, 4) in launch r, and the five candidates with their costs."""
    from gipuma_b200 import api
    from oracle import pyrefine as R
    p0, c0 = before if before is not None else ctx.get_state()
    prm = sc.params
    cand = R.candidates(p0, api.pack_camera(sc.cameras[0]), prm.min_disparity, prm.max_disparity, prm.depthMin, prm.depthMax,
                        eps, seed, r)
    f = cost_of(ctx)
    costs = np.stack([f(np.ascontiguousarray(cand[j]), 0) for j in range(5)])
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    mine = ((xs + ys) & 1) == colour
    want_p, want_c, changed = R.accept(p0, c0, cand, costs, mine)
    return want_p, want_c, changed, cand, costs


def same(a, b):
    return bits_equal(a[0], b[0]) == 0 and bits_equal(a[1], b[1]) == 0


@pytest.mark.parametrize("case", list(CASES))
def test_refinement_equals_the_restatement(case):
    rows, cols, views, mode = CASES[case]
    sc = make_scene(rows, cols, views, colour=mode == "colour")
    A = open_mode(sc, mode)
    twins = [open_mode(sc, mode, options={"memo": 0, "prune": 0, "dedupe": 0}), open_mode(sc, mode, options={"nwarps": 5})]
    accepted = 0
    try:
        r = [start(c, sc, mode) for c in [A] + twins][0]
        for it in range(2):
            for colour in (0, 1):
                want_p, want_c, changed, _, _ = restated(A, sc, colour, r)
                A.phase(colour, 4)
                got = A.get_state()
                bad = (got[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) | (got[1].view(np.uint32) != want_c.view(np.uint32))
                assert not bad.any(), (case, it, colour, int(bad.sum()), np.argwhere(bad)[:8].tolist())
                accepted += int(changed.sum())
                for t in twins:
                    t.phase(colour, 4)
                    assert same(t.get_state(), got), (case, it, colour)
                r += 1
                for c in [A] + twins:                      # propagation in between: no refinement, r unchanged
                    c.phase(1 - colour, 3)
                assert all(same(t.get_state(), A.get_state()) for t in twins)
        assert accepted > 0, case
    finally:
        for c in [A] + twins:
            c.close()


@pytest.mark.parametrize("mode", ["pm", "ncc_geo"])
def test_refinement_exact_on_adversarial_states(mode):
    sc = make_scene(53, 75, 4)
    A = open_mode(sc, mode)
    try:
        start(A, sc, mode)
        p0, c0 = A.get_state()
        rng = np.random.default_rng(9)
        H, W = c0.shape
        # the next launch's candidate costs, to make ties (rejected) with candidate 0 and 3 at some pixels
        A.set_state(p0, c0)
        _, _, _, cand, costs = restated(A, sc, 0, 2, before=(p0, c0))
        c1 = c0.copy()
        tie0, tie3 = rng.random((H, W)) < 0.1, rng.random((H, W)) < 0.1
        c1[tie0] = costs[0][tie0]
        c1[tie3 & ~tie0] = costs[3][tie3 & ~tie0]
        c1[rng.random((H, W)) < 0.05] = f32(2000.0)                       # above MAXCOST: every candidate below wins
        c1[rng.random((H, W)) < 0.03] = MAXCOST
        c1[rng.random((H, W)) < 0.02] = f32(np.nan)                       # NaN: no candidate is accepted
        p1 = p0.copy()
        p1[rng.random((H, W)) < 0.02, 3] = f32(np.nan)
        A.set_state(p1, c1)                              # gpm_set_state leaves r as it is
        for colour, r in ((0, 2), (1, 3)):
            want_p, want_c, _, _, _ = restated(A, sc, colour, r)
            A.phase(colour, 4)
            got = A.get_state()
            assert bits_equal(got[0], want_p) == 0 and bits_equal(got[1], want_c) == 0, (mode, colour)
    finally:
        A.close()


def test_joint_view_selection_is_deterministic_and_takes_candidates():
    from gipuma_b200 import api
    from oracle import pyrefine as R
    sc = make_scene(53, 75, 4)

    def jvs():
        c = open_mode(sc, "ncc")
        c.set_view_selection("joint")
        return c
    A, B, G = jvs(), jvs(), open_mode(sc, "ncc", refinement="gipuma")
    G.set_view_selection("joint")
    try:
        for c in (A, B, G):
            start(c, sc, "ncc")
        assert same(A.get_state(), B.get_state())
        assert not same(A.get_state(), G.get_state())
        r, taken = 2, 0
        prm = sc.params
        for colour in (0, 1):
            p0, c0 = A.get_state()
            cand = R.candidates(p0, api.pack_camera(sc.cameras[0]), prm.min_disparity, prm.max_disparity, prm.depthMin,
                                prm.depthMax, EPS, 31, r)
            A.phase(colour, 4)
            B.phase(colour, 4)
            p1, c1 = A.get_state()
            assert same((p1, c1), B.get_state())
            changed = (p1.view(np.uint32) != p0.view(np.uint32)).any(axis=-1)
            is_cand = np.zeros_like(changed)
            for j in range(5):
                is_cand |= (p1.view(np.uint32) == cand[j].view(np.uint32)).all(axis=-1)
            assert np.all(is_cand[changed])               # the launch re-weights every cost, so costs are not compared
            taken += int(changed.sum())
            r += 1
        assert taken > 0
    finally:
        for c in (A, B, G):
            c.close()


def test_consecutive_launches_differ_and_set_rng_reproduces():
    sc = make_scene(53, 75, 4)
    A = open_mode(sc, "pm", seed=5)
    try:
        A.init()
        s0 = A.get_state()
        A.phase(0, 4)
        s1 = A.get_state()
        A.set_state(*s0)
        A.phase(0, 4)                                     # r = 1: other candidates
        s2 = A.get_state()
        assert (s1[0].view(np.uint32) != s2[0].view(np.uint32)).any(axis=-1).sum() > 50
        A.set_rng(5)                                      # r back to 0
        A.set_state(*s0)
        A.phase(0, 4)
        assert same(A.get_state(), s1)
        A.init()                                          # gpm_init resets r as well
        A.phase(0, 4)
        assert same(A.get_state(), s1)
    finally:
        A.close()


def test_refusals_change_nothing():
    from gipuma_b200 import api
    sc = make_scene(53, 75, 4)
    A = open_mode(sc, "pm")
    T = open_mode(sc, "pm")
    lib = A.lib
    try:
        for c in (A, T):
            c.init()
            c.phase(0, 4)
        before, launches = A.get_state(), A.stats()["launches"]
        bad = [(5, 0.02), (-1, 0.02), (1, 0.0), (1, 1.0), (1, -0.5), (1, float("nan")), (1, float("inf")), (0, 2.0)]
        for kind, eps in bad:
            assert lib.gpm_set_refinement(A.h, kind, eps) == E_ARG, (kind, eps)
        with pytest.raises(api.GipumaError, match="-1"):
            A.set_option("neighbours", 20)                 # the fused sweep refuses ACMH's refinement
        # while ACMH's refinement is on, every shard call taking a context refuses with GPM_E_STATE
        assert lib.gpm_shard_num_stages(A.h) == -1 and lib.gpm_shard_stage_floats(A.h, 0) == -1
        assert lib.gpm_shard_stage(A.h, 0, 0, None, 1, None) == E_STATE
        import torch
        gathered = torch.zeros(2 * sc.rows * ((sc.cols + 1) // 2) * sc.params.n_best, device="cuda")
        assert lib.gpm_shard_finish_init(A.h, C.c_void_p(gathered.data_ptr()), 1) == E_STATE
        assert lib.gpm_shard_run(A.h, None) == E_STATE
        assert lib.gpm_shard_comm_attach(A.h, None, 0, 1) == E_STATE
        uid = (C.c_char * 128)()
        assert lib.gpm_shard_comm_init(A.h, uid, 0, 1) == E_STATE
        assert "Gipuma's refinement" in lib.gpm_last_error().decode()
        assert same(A.get_state(), before) and A.stats()["launches"] == launches
        # nothing changed: the next refinement launch equals the untouched twin's
        A.phase(1, 4)
        T.phase(1, 4)
        assert same(A.get_state(), T.get_state())
        # the fused sweep refuses the switch in the other direction
        F = open_mode(sc, "pm", refinement="gipuma", options={"neighbours": 20})
        try:
            with pytest.raises(api.GipumaError, match="-1"):
                F.set_refinement("acmh", EPS)
            F.init()
            F.phase(0, 7)
        finally:
            F.close()
        # back to Gipuma's refinement: the shard accepts the context again
        A.set_refinement("gipuma", EPS)
        assert lib.gpm_shard_num_stages(A.h) > 0
    finally:
        A.close()
        T.close()


# ---- drivers ----------------------------------------------------------------------------------------------------------

def _acmh_flow(m):
    """The drivers' job setup with ACMH's refinement, restated: set_refinement next to every set_rng of the flow (the
    switch resets nothing, so its order with set_rng does not matter)."""
    from gipuma_b200 import api
    base = api.Context.set_rng

    def set_rng(self, seed, mode=api.GPM_RNG_REFERENCE):
        self.set_refinement("acmh", EPS)
        base(self, seed, mode)
    m.setattr(api.Context, "set_rng", set_rng)


def test_batch_run_refine_equals_the_context_flow(monkeypatch):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    import test_gpu_ncc as tn
    c = gb._case("ragged", False)
    with monkeypatch.context() as m:
        m.setattr(api.Context, "set_photometric", lambda self, kind="pm", min_std=0.0: None)
        _acmh_flow(m)
        w4, wc = tn._restated_batch(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], **gb.KW)
    for devices in ((0,), (0, 0), (0, 0, 0)):
        n4, cost, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], devices=devices, cam_scale=c["scale"],
                                    refinement={"kind": "acmh", "perturbation": EPS}, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, devices
    ref, rc, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], cam_scale=c["scale"], **gb.KW)
    assert bits_equal(ref, w4) > 0
    for refinement in (None, "gipuma"):
        n4, cost, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], cam_scale=c["scale"], refinement=refinement,
                                    devices=(0, 0), **gb.KW)
        assert bits_equal(n4, ref) == 0 and bits_equal(cost, rc) == 0, refinement


def test_geometric_pass_refine_equals_the_context_flow(monkeypatch):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case("ragged", False)
    with monkeypatch.context() as m:
        _acmh_flow(m)
        w4, wc, w_pass1, w_views = gb._restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                                max_err=api.GEO_MAX_ERR, **gb.KW)
    for devices in ((0,), (0, 0, 0)):
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, refinement="acmh", **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, devices
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views
    ref = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                             cam_scale=c["scale"], **gb.KW)
    got = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                             cam_scale=c["scale"], refinement="gipuma", devices=(0, 0), **gb.KW)
    assert bits_equal(got[0], ref[0]) == 0 and bits_equal(got[1], ref[1]) == 0


def test_multiscale_pass_refine_equals_the_context_flow(monkeypatch):
    from gipuma_b200 import api
    import test_gpu_multiscale as tm
    from test_gpu_geometric_batch import _case
    c = _case("ragged", False)
    levels = 2
    with monkeypatch.context() as m:
        _acmh_flow(m)
        w4, wc, wV = tm._restated(c["images"], c["Ps"], c["params"], c["refs"], levels, c["scale"], weight=api.GEO_WEIGHT,
                                  max_err=api.GEO_MAX_ERR, jbu=tm.JBU, **tm.KW)
    c["modes"] = {}
    for devices in ((0,), (0, 0)):
        n4, cost, info = tm._run(c, levels, devices=devices, refinement="acmh")
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, devices
        assert info["views"] == wV
    ref = tm._run(c, levels)
    got = tm._run(c, levels, refinement="gipuma", devices=(0, 0, 0))
    assert bits_equal(got[0], ref[0]) == 0 and bits_equal(got[1], ref[1]) == 0
    assert bits_equal(ref[0], w4) > 0
