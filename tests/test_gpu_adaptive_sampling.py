"""Adaptive checkerboard sampling (DESIGN.md §16) on the GPU, checked exactly against oracle/pyacs.py.

A propagation launch in this mode is still a pure function of its start state (region pixels are of the other colour,
whose planes and costs a launch never writes), so every close, far and combined launch must equal pyacs.expected() bit
for bit outside the ambiguous pixels, at ragged sizes, with gridDim.z splits, in every cost mode, and on adversarial
states.  Refinement is checked by its invariants.  Twins without the memo, the lower-bound early-out or the duplicate
skips, and a twin with one mask-7 launch per colour, must stay bit-identical.  The mode may be switched mid-run.  The
source-view shard, ranks simulated on one GPU, must equal the single context stage by stage; the batch drivers must equal
the Context-call flows; refusals must change nothing."""
import os
import time

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_sweep_any_size import adversarial_state, check_launch, cost_of

pytestmark = pytest.mark.gpu

f32 = np.float32
WEIGHT, MAX_ERR, MIN_STD = 0.3, 6.0, 4.0
REPORT = {}

# id: (rows, cols, views, box, colour images, NCC, geometric term, stateful RNG)
CASES = {
    "grey_53x75": (53, 75, 4, 9, False, False, False, False),           # 6 tiles: gridDim.z = 8
    "grey_8x8_box25": (8, 8, 2, 25, False, False, False, False),        # every region partly off the image
    "grey_31x33": (31, 33, 3, 15, False, False, False, False),
    "grey_97x65": (97, 65, 6, 3, False, False, False, False),
    "grey_480x640": (480, 640, 10, 15, False, False, False, False),     # gridDim.z = 4 on 132 SMs
    "grey_550x1000": (550, 1000, 10, 15, False, False, False, False),   # gridDim.z = 2 on 132 SMs
    "colour_53x75": (53, 75, 4, 9, True, False, False, False),
    "colour_31x33_box25": (31, 33, 3, 25, True, False, False, False),
    "ncc_53x75": (53, 75, 4, 15, False, True, False, False),
    "ncc_geo_53x75": (53, 75, 4, 15, False, True, True, False),
    "geo_colour_45x71": (45, 71, 4, 9, True, False, True, False),
    "stateful_53x75": (53, 75, 4, 9, False, False, False, True),
}
# twins of the checked context: the exact shortcuts off one at a time, and one mask-7 launch per colour
TWINS = [{"memo": 0}, {"prune": 0}, {"dedupe": 0}, None]


def make_scene(case):
    from gipuma_b200 import scene as S
    rows, cols, views, box, color, ncc, geo, stateful = CASES[case]
    sc = S.make_config(2, rows=rows, cols=cols, n_views=views, iterations=2, seed=rows * 1000 + cols)
    sc.params.box_hsize = sc.params.box_vsize = box
    return S.colorize(sc) if color else sc


def open_acs(case, sc, seed, options=None, propagation="adaptive"):
    from gipuma_b200 import api
    from test_gpu_geometric import depth_maps
    rows, cols, views, box, color, ncc, geo, stateful = CASES[case]
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    if ncc:
        ctx.set_photometric("ncc", MIN_STD)
    ctx.load_scene(sc, seed=seed, rng_mode=api.GPM_RNG_STATEFUL if stateful else api.GPM_RNG_REFERENCE)
    if geo:
        for v, d in enumerate(depth_maps(sc, 3)):
            ctx.set_view_depth(v, d)
        ctx.set_geometric(WEIGHT, MAX_ERR)
    ctx.set_propagation(propagation)
    return ctx


def assert_rule(got, want, colour, what):
    want_p, want_c, amb = want
    bad = (got[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) | (got[1].view(np.uint32) != want_c.view(np.uint32))
    bad &= ~amb
    assert not bad.any(), (what, colour, int(bad.sum()), np.argwhere(bad)[:8].tolist())
    return amb


def finite_or_inf(state):
    """NaN costs as +inf, for check_launch's `cost never increases` (a NaN cost is never replaced: c < NaN is false)."""
    return state[0], np.where(np.isnan(state[1]), f32(np.inf), state[1])


def decision_chain(sc, color, A, twins, iterations=2, adaptive=True):
    """A runs phase(c, 1), phase(c, 2), phase(c, 4) with every propagation decision checked against pyacs.expected; twins
    run the same masks (options) or one mask-7 launch per colour (None) and must hold A's bits after every colour."""
    from oracle import pyacs
    f = cost_of(A)
    cam, prm = sc.cameras[0], sc.params
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    stats = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}
    for _ in range(iterations):
        for colour in (0, 1):
            mine = ((xs + ys) & 1) == colour
            for mask in (1, 2, 4):
                before = A.get_state()
                A.phase(colour, mask)
                after = A.get_state()
                if mask != 4:
                    want = pyacs.expected(before[0], before[1], colour, mask, f, cam, prm.depthMin, prm.depthMax,
                                          color_images=color, adaptive=adaptive)
                    amb = assert_rule(after, want, colour, "mask %d" % mask)
                    stats["compared"] += int((mine & ~amb).sum())
                    stats["ambiguous"] += int((mine & amb).sum())
                    stats["accepted"] += int((mine & (after[1] < before[1])).sum())
                    check_launch(finite_or_inf(before), finite_or_inf(after), colour)
                else:
                    stats["refined"] += check_launch(finite_or_inf(before), finite_or_inf(after), colour, f, sc, 0)
                for ctx, opts in twins:
                    if opts is not None:
                        ctx.phase(colour, mask)
            for ctx, opts in twins:
                if opts is None:
                    ctx.phase(colour, 7)
            ref_p, ref_c = A.get_state()
            for ctx, opts in twins:
                p, c = ctx.get_state()
                assert bits_equal(p, ref_p) == 0 and bits_equal(c, ref_c) == 0, ("twin", opts, colour)
    assert stats["accepted"] > 0 and stats["refined"] > 0
    total = stats["compared"] + stats["ambiguous"]
    assert stats["ambiguous"] <= max(4, 0.005 * total), stats
    return dict(stats, ambiguous_share=stats["ambiguous"] / max(1, total))


@pytest.mark.parametrize("case", list(CASES))
def test_adaptive_decisions_exact(case):
    t0 = time.perf_counter()
    sc = make_scene(case)
    color = CASES[case][4]
    seed = 6000 + sc.rows + sc.cols
    A = open_acs(case, sc, seed)
    twins = [(open_acs(case, sc, seed, o), o) for o in TWINS]
    try:
        for ctx in [A] + [t for t, _ in twins]:
            ctx.init()
        A.reset_stats()
        REPORT[case] = decision_chain(sc, color, A, twins)
        REPORT[case]["stats"] = {k: v for k, v in A.stats().items() if k in ("hypotheses", "skipped", "pairs")}
    finally:
        for ctx in [A] + [t for t, _ in twins]:
            ctx.close()
    REPORT[case]["seconds"] = round(time.perf_counter() - t0, 2)
    print("\n%s: %s" % (case, REPORT[case]))


def hostile_costs(sc, cost, rng):
    """On top of adversarial_state: tied costs (a third of them rounded to 1/8), NaN and +inf costs (2 % each)."""
    c = cost.copy()
    H, W = c.shape
    tie = rng.random((H, W)) < 0.33
    c[tie] = np.round(c[tie] * 8) / 8
    c[rng.random((H, W)) < 0.02] = np.nan
    c[rng.random((H, W)) < 0.02] = np.inf
    return c.astype(f32)


@pytest.mark.parametrize("case,trust", [("grey_53x75", 1), ("grey_53x75", 0), ("colour_53x75", 0), ("ncc_53x75", 0)])
def test_adaptive_decisions_exact_on_adversarial_states(case, trust):
    """Ties inside regions, NaN / +inf / MAXCOST costs, out-of-range and bit-equal planes: the choice and the accept rule
    both decide some pixels."""
    sc = make_scene(case)
    color = CASES[case][4]
    opts = {"trust_state": trust}
    A = open_acs(case, sc, 77, opts)
    twins = [(open_acs(case, sc, 77, dict(opts, **o) if o else opts), o) for o in TWINS]
    try:
        A.init()
        n0, _ = A.get_state()
        rng = np.random.default_rng(11)
        pl, cost = adversarial_state(sc, n0, cost_of(A), rng, False, color)
        cost = hostile_costs(sc, cost, rng)
        for ctx in [A] + [t for t, _ in twins]:
            ctx.set_state(pl, cost)
        REPORT["adversarial_" + case] = decision_chain(sc, color, A, twins)
    finally:
        for ctx in [A] + [t for t, _ in twins]:
            ctx.close()
    print("\nadversarial %s trust=%d: %s" % (case, trust, REPORT["adversarial_" + case]))


@pytest.mark.parametrize("case", ["grey_53x75", "colour_53x75", "ncc_geo_53x75"])
def test_switching_mid_run_follows_the_rule_and_back_to_fixed_matches_a_fresh_context(case):
    from oracle import pyacs
    sc = make_scene(case)
    color = CASES[case][4]
    with open_acs(case, sc, 31, propagation="fixed") as A, open_acs(case, sc, 31, propagation="fixed") as fresh:
        A.init()
        A.sweep(1)
        f = cost_of(A)
        prm, cam = sc.params, sc.cameras[0]
        for step, mode in enumerate(["adaptive", "fixed", "adaptive", "fixed"]):
            A.set_propagation(mode)
            colour = step & 1
            for mask in (1, 2, 3):
                before = A.get_state()
                want = pyacs.expected(before[0], before[1], colour, mask, f, cam, prm.depthMin, prm.depthMax,
                                      color_images=color, adaptive=mode == "adaptive")
                A.phase(colour, mask)
                assert_rule(A.get_state(), want, colour, (mode, mask))
            A.phase(colour, 4)
        A.set_propagation("adaptive")
        A.run()
        A.set_propagation("fixed")
        A.run()
        fresh.run()
        assert bits_equal(A.get_state()[0], fresh.get_state()[0]) == 0 and bits_equal(A.get_state()[1], fresh.get_state()[1]) == 0


def test_adaptive_run_differs_from_fixed():
    """The mode is not a no-op: on a real scene a run picks other planes."""
    sc = make_scene("grey_97x65")
    with open_acs("grey_97x65", sc, 5) as a, open_acs("grey_97x65", sc, 5, propagation="fixed") as b:
        a.run()
        b.run()
        assert bits_equal(a.get_state()[1], b.get_state()[1]) > 0


# ---- source-view shard ------------------------------------------------------------------------------------------------
SHARD_CASES = {
    "53x75": ((53, 75, 7, 3, 9, False, 2), (2, 3)),
    "colour_45x71": ((45, 71, 5, 3, 11, True, 2), (2,)),
    "97x65": ((97, 65, 6, 2, 7, False, 1), (3,)),
    "colour_31x33": ((31, 33, 4, 3, 15, True, 1), (2, 3)),
}


def _adaptive_not_offered_are_inf(g, world, H, W, nb, colour):
    """Stage 1 in adaptive mode: a direction whose region lies wholly off the image holds +inf in every rank's list."""
    from oracle import pyacs
    import test_gpu_view_shard_any_size as A
    u = A.lists_view(g, world, H, W, nb, 1)
    ys, px, valid = A.pixel_of(H, W, colour)
    pxc = np.minimum(px, W - 1)
    for k, _, _, ok in pyacs.choose(np.zeros((H, W), f32), H, W, 3):
        off = valid & ~ok[ys, pxc]
        if off.any():
            assert np.all(u[:, off, k, :] == A.INF), (colour, k)


@pytest.mark.parametrize("case", list(SHARD_CASES))
def test_view_shard_adaptive_stages_equal_the_single_context(case, monkeypatch):
    import test_gpu_view_shard_any_size as A
    from test_gpu_view_shard import SimulatedShard
    (rows, cols, views, n_best, box, colour, iterations), worlds = SHARD_CASES[case]
    sc = A.make_scene(rows, cols, views, n_best, box, colour, iterations)

    class Checker(A.Checker):
        def expected(self, before, colour_, mask):
            from oracle import pyacs
            prm = self.sc.params
            return pyacs.expected(before[0], before[1], colour_, mask, self.cost, self.sc.cameras[0], prm.depthMin,
                                  prm.depthMax, color_images=self.colour_images)

    monkeypatch.setattr(A, "assert_not_offered_are_inf", _adaptive_not_offered_are_inf)
    single = A.open_single(sc)
    single.set_propagation("adaptive")
    groups = [SimulatedShard(sc, w, A.SEED) for w in sorted(worlds, reverse=True)]
    twin = SimulatedShard(sc, max(worlds), A.SEED, {"memo": 0, "dedupe": 0})
    for grp in groups + [twin]:
        for ctx in grp.ctxs:
            ctx.set_propagation("adaptive")
    try:
        chk = Checker(sc, colour, single, groups[0], groups[1:], [twin], single_vs_rule=True)
        chk.init()
        REPORT["shard_" + case] = chk.run(iterations)
    finally:
        for g in groups + [twin]:
            g.close()
        single.close()
    assert REPORT["shard_" + case]["accepted"] > 0 and REPORT["shard_" + case]["refined"] > 0
    print("\nshard %s: %s" % (case, REPORT["shard_" + case]))


@pytest.mark.parametrize("colour", [False, True])
def test_view_shard_runner_adaptive_world1_equals_gpm_run(colour):
    """multigpu.ViewShardRunner(propagation="adaptive") at world size 1 (gpm_shard_run) = an adaptive gpm_run."""
    import test_gpu_view_shard_any_size as A
    from gipuma_b200 import multigpu as M
    sc = A.make_scene(61, 83, 5, 3, 9, colour, 2)
    single = A.open_single(sc)
    single.set_propagation("adaptive")
    run = M.ViewShardRunner(sc, 0, 1, seed=A.SEED, propagation="adaptive")
    try:
        single.run()
        n4, c = run.run()
        s4, s1 = single.get_state()
    finally:
        run.close()
        single.close()
    assert bits_equal(n4, s4) == 0 and bits_equal(c, s1) == 0


def test_view_shard_adaptive_over_two_real_ranks_equals_single_gpu():
    """One real two-rank NCCL run (gpm_shard_run) in adaptive mode, bit-identical to gpm_run.  Needs 2 GPUs."""
    import test_gpu_view_shard_nccl as N
    if N._gpus() < 2:
        pytest.skip("needs 2 GPUs")
    out = N._torchrun(2, [os.path.join("tools", "run_shard_nccl.py"), "--config", "2", "--rows", "353", "--cols", "481",
                          "--views", "7", "--iters", "2", "--propagation", "adaptive"])
    assert out["propagation"] == "adaptive" and out["collectives"] > 0
    assert out["bit_identical_to_single_gpu"] is True


# ---- drivers ----------------------------------------------------------------------------------------------------------
def _adaptive_contexts(monkeypatch):
    from gipuma_b200 import api
    base, made = api.Context, []

    def adaptive_context(*a, **k):
        ctx = base(*a, **k)
        ctx.set_propagation("adaptive")
        made.append(ctx)
        return ctx
    monkeypatch.setattr(api, "Context", adaptive_context)
    return made


@pytest.mark.parametrize("name", ["fusion", "ragged"])
def test_batch_run_adaptive_equals_the_context_flow(name, monkeypatch):
    """batch_run(photometric="ncc", propagation="adaptive") against the NCC tests' restatement of a batch job through
    Context calls (at that restatement's min_std), on a context switched to adaptive sampling; one worker and two."""
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    import test_gpu_ncc as tn
    c = gb._case(name, False)
    with monkeypatch.context() as m:
        made = _adaptive_contexts(m)
        w4, wc = tn._restated_batch(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], **gb.KW)
    assert len(made) == 1
    for devices in ((0,), (0, 0)):
        n4, cost, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], devices=devices, cam_scale=c["scale"],
                                    photometric="ncc", ncc_min_std=tn.MIN_STD, propagation="adaptive", **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
    fixed, _, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], cam_scale=c["scale"], photometric="ncc",
                                ncc_min_std=tn.MIN_STD, **gb.KW)
    assert bits_equal(fixed, w4) > 0                                      # the mode reached the jobs


@pytest.mark.parametrize("name,colour", [("fusion", False), ("ragged", True)])
def test_geometric_pass_adaptive_equals_the_context_flow(name, colour, monkeypatch):
    """geometric_pass(propagation="adaptive") against test_gpu_geometric_batch's restatement of the two-pass flow on
    contexts switched to adaptive sampling (both passes); one worker and two."""
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case(name, colour)
    with monkeypatch.context() as m:
        made = _adaptive_contexts(m)
        w4, wc, w_pass1, w_views = gb._restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                                max_err=api.GEO_MAX_ERR, **gb.KW)
    assert len(made) == 1
    for devices in ((0,), (0, 0)):
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, propagation="adaptive", **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views, devices


# ---- refusals ---------------------------------------------------------------------------------------------------------
def test_refusals_leave_launch_count_and_state_untouched():
    E_ARG = -1
    sc = make_scene("grey_53x75")
    with open_acs("grey_53x75", sc, 3) as ctx, open_acs("grey_53x75", sc, 3) as twin:
        L, h = ctx.lib, ctx.h
        ctx.init()
        ctx.sweep(1)
        state, launches = ctx.get_state(), ctx.stats()["launches"]
        for call in (lambda: L.gpm_set_propagation(h, 2), lambda: L.gpm_set_propagation(h, -1),
                     lambda: L.gpm_set_option(h, b"neighbours", 20)):          # the fused sweep has no adaptive variant
            assert call() == E_ARG, L.gpm_last_error().decode()
        assert ctx.stats()["launches"] == launches
        s = ctx.get_state()
        assert bits_equal(s[0], state[0]) == 0 and bits_equal(s[1], state[1]) == 0
        ctx.sweep(1)                                                         # still adaptive, still 8 neighbours
        twin.init()
        twin.sweep(2)
        assert bits_equal(ctx.get_state()[1], twin.get_state()[1]) == 0
        with pytest.raises(ValueError):
            ctx.set_propagation("acmh")
        ctx.set_propagation("fixed")
        ctx.set_option("neighbours", 20)
        assert L.gpm_set_propagation(h, 1) == E_ARG                        # ADAPTIVE while neighbours = 20
        assert L.gpm_set_propagation(h, 0) == 0
        ctx.set_option("neighbours", 8)
        ctx.set_propagation("adaptive")
        assert ctx.stats()["launches"] == launches + 2
