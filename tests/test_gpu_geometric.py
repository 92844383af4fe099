"""The geometric-consistency mode (DESIGN.md §14) on the GPU.

- weight 0 with depth maps uploaded changes nothing: gpm_run is bit-identical to a context without them;
- gpm_cost_eval in the mode equals the numpy restatement bit for bit at ragged sizes: one view (photometric cost at
  weight 0 plus oracle/pygeo.geo_cost), and several views (each view's photometric cost from a one-view context, plus its
  g_j, combined by pygeo.combine under the best_n / all / good rules; the device's reciprocals of the view counts are
  read off the weight-0 combination of the same sums' photometric parts);
- every propagation decision equals oracle/pypropagate.expected() with this cost, refinement keeps its invariants, and
  twins without memo, lower-bound early-out and duplicate skips, or with one mask-7 launch per colour, stay bit-identical;
- every refusal leaves the launch count and the state untouched;
- the two-pass driver runs on the fusion test's dataset and its output fuses and scores."""
import ctypes
import time

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_sweep_any_size import cost_of, check_launch

pytestmark = pytest.mark.gpu

f32 = np.float32
MAXCOST = f32(1000.0)
WEIGHT, MAX_ERR = 0.3, 6.0


def make_scene(rows, cols, views, box=9, color=False):
    """A rendered scene: the DTU rig up to 10 source views, the templeRing rig (any number of views) above.  At 40 x 60 the
    64-view synthetic rig (config 5) accepts almost no refinement, in every mode; the templeRing rig accepts thousands."""
    from gipuma_b200 import scene as S
    cfg = 2 if views <= 10 else 4
    sc = S.make_config(cfg, rows=rows, cols=cols, n_views=views, iterations=2, seed=rows * 1000 + cols)
    sc.params.box_hsize = sc.params.box_vsize = box
    return S.colorize(sc) if color else sc


def depth_maps(sc, seed):
    """A smooth depth map per source view inside the depth range, with holes (0) and patches outside the range."""
    rng = np.random.default_rng(seed)
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    lo, hi = sc.params.depthMin, sc.params.depthMax
    out = []
    for v in range(sc.n_views):
        a, b = rng.uniform(0.02, 0.08, 2)
        d = 0.5 * (lo + hi) * (1.0 + 0.15 * np.sin(a * xs + v) * np.cos(b * ys))
        d[rng.random(d.shape) < 0.05] = 0.0
        d[rng.random(d.shape) < 0.03] = 1.5 * hi
        out.append(np.ascontiguousarray(d, dtype=f32))
    return out


def open_ctx(sc, seed=99, depths=None, weight=0.0, views=None, options=None):
    """A context over `sc`, or over the listed views of its subset only."""
    from gipuma_b200 import api
    sub = sc.subset if views is None else [sc.subset[v] for v in views]
    ctx = api.Context(sc.cols, sc.rows, len(sub))
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    ctx.set_params(sc.params)
    ctx.set_reference(sc.images[0], sc.cameras[0])
    for v, idx in enumerate(sub):
        ctx.set_view(v, sc.images[idx], sc.cameras[idx])
    ctx.set_num_views(len(sub))
    ctx.set_rng(seed)
    if depths is not None:
        for v, d in enumerate(depths if views is None else [depths[v] for v in views]):
            ctx.set_view_depth(v, d)
        ctx.set_geometric(weight, MAX_ERR)
    return ctx


def restated_g(sc, planes, depths, v, weight=WEIGHT):
    from oracle import pygeo
    p = sc.params
    return pygeo.geo_cost(planes, sc.cameras[0], sc.cameras[sc.subset[v]], depths[v], weight, MAX_ERR, p.depthMin, p.depthMax)


@pytest.mark.parametrize("color", [False, True])
def test_weight_zero_changes_nothing(color):
    sc = make_scene(53, 75, 4, color=color)
    depths = depth_maps(sc, 1)
    outs = []
    for d in (None, depths):
        with open_ctx(sc, depths=d) as ctx:
            if d is not None:                    # on and off again: weight 0 is exactly the photometric cost
                ctx.set_geometric(WEIGHT, MAX_ERR)
                ctx.set_geometric(0.0, MAX_ERR)
            ctx.run()
            outs.append(ctx.get_state())
    assert bits_equal(outs[0][0], outs[1][0]) == 0 and bits_equal(outs[0][1], outs[1][1]) == 0


def planes_to_score(sc, seed):
    """Initial planes and the planes after one sweep (photometric), both as raw reference-frame planes."""
    with open_ctx(sc, seed) as ctx:
        ctx.init()
        p0 = ctx.get_state()[0]
        ctx.sweep(1)
        return [p0, ctx.get_state()[0]]


@pytest.mark.parametrize("rows,cols,color", [(53, 75, False), (31, 33, False), (97, 65, False), (53, 75, True), (29, 41, True)])
def test_cost_of_one_view_equals_the_restatement(rows, cols, color):
    sc = make_scene(rows, cols, 1, color=color)
    depths = depth_maps(sc, rows)
    n_near = 0
    for planes in planes_to_score(sc, rows):
        for variant in (-1, 0, 1):
            with open_ctx(sc, depths=depths, weight=0.0, options={"cost_variant": variant}) as ctx:
                photo = ctx.cost_eval(planes)
                ctx.set_geometric(WEIGHT, MAX_ERR)
                got = ctx.cost_eval(planes)
            g = restated_g(sc, planes, depths, 0)
            s = (photo + g).astype(f32)
            want = np.where(s < MAXCOST, s, MAXCOST).astype(f32)
            assert bits_equal(got, want) == 0, (rows, cols, variant, np.argwhere(got.view(np.uint32) != want.view(np.uint32))[:5])
            n_near += int((g < f32(WEIGHT) * f32(MAX_ERR)).sum())
    assert n_near > 0                             # some hypotheses are scored by an actual reprojection error


def learn_rcp(k, s, combined):
    """The device's float32 reciprocal of each view count k, from combined = rcp(k) * s on the pixels with that count."""
    rcp = {}
    for kk in np.unique(k[k >= 1]):
        m = (k == kk) & (combined < MAXCOST)
        r0 = f32(1.0) / f32(kk)
        fits = [r for r in (r0, np.nextafter(r0, f32(0)), np.nextafter(r0, f32(1))) if bits_equal((r * s[m]).astype(f32), combined[m]) == 0]
        assert len(fits) >= 1, ("no reciprocal of %d reproduces the combination" % kk)
        rcp[int(kk)] = fits[0]
    return rcp


# rows, cols, views, colour, cost_comb, n_best: 33 and 64 views put a second view in every lane (views lane + 32)
MANY = [(53, 75, 4, False, 1, 2), (31, 33, 4, False, 0, 2), (97, 65, 4, False, 3, 2), (53, 75, 4, True, 1, 3),
        (29, 41, 4, True, 0, 2), (40, 60, 33, False, 1, 3), (40, 60, 33, True, 3, 2), (40, 60, 64, False, 0, 2),
        (40, 60, 64, False, 3, 2), (40, 60, 64, True, 1, 40)]


@pytest.mark.parametrize("rows,cols,views,color,comb,n_best", MANY)
def test_cost_of_many_views_equals_the_restatement(rows, cols, views, color, comb, n_best):
    from oracle import pygeo
    t0 = time.perf_counter()
    sc = make_scene(rows, cols, views, color=color)
    sc.params.cost_comb, sc.params.n_best = comb, n_best
    depths = depth_maps(sc, rows + 7)
    n_near = 0
    for planes in planes_to_score(sc, rows):
        photo = []
        for v in range(sc.n_views):
            with open_ctx(sc, depths=depths, views=[v]) as one:
                photo.append(one.cost_eval(planes))
        photo = np.stack(photo)
        with open_ctx(sc, depths=depths) as ctx:
            c0 = ctx.cost_eval(planes)
            ctx.set_geometric(WEIGHT, MAX_ERR)
            got = ctx.cost_eval(planes)
        s0, k0 = pygeo.combine_sum(photo, comb, n_best, sc.params.good_factor)
        rcp = learn_rcp(k0, s0, c0)
        assert bits_equal(pygeo.combine(photo, comb, n_best, sc.params.good_factor, rcp), c0) == 0
        g = np.stack([restated_g(sc, planes, depths, v) for v in range(sc.n_views)])
        sums = (photo + g).astype(f32)
        want = pygeo.combine(sums, comb, n_best, sc.params.good_factor, rcp)
        known = ~np.isnan(want)
        assert known.mean() > 0.98, known.mean()
        assert bits_equal(got[known], want[known]) == 0, (rows, cols, comb, np.argwhere((got != want) & known)[:5])
        n_near += int((g[32:] < f32(WEIGHT) * f32(MAX_ERR)).sum())
    if views > 32:
        assert n_near > 0                         # views lane + 32 are scored by an actual reprojection error
    print("\ngeometric cost, %dx%d, %d views, colour %s, comb %d, n_best %d: %d near views >= 32, %.2f s" %
          (rows, cols, views, color, comb, n_best, n_near, time.perf_counter() - t0))


# box 15: 64 samples, two rounds, so the lower bound is tested; box 25: six rounds; box 3: one round of 4 samples, the
# lower bound has nothing to cut short
@pytest.mark.parametrize("rows,cols,views,box,color", [(53, 75, 4, 15, False), (97, 65, 4, 15, False), (53, 75, 4, 15, True),
                                                       (31, 33, 4, 15, True), (40, 60, 33, 3, False), (40, 60, 33, 25, False),
                                                       (40, 60, 64, 3, False), (40, 60, 64, 25, False), (40, 60, 64, 25, True)])
def test_sweep_decisions_exact(rows, cols, views, box, color):
    from oracle import pypropagate as pp
    t0 = time.perf_counter()
    sc = make_scene(rows, cols, views, box=box, color=color)
    depths = depth_maps(sc, 3)
    seed = 4000 + rows + cols
    ctxs = [open_ctx(sc, seed, depths, WEIGHT),
            open_ctx(sc, seed, depths, WEIGHT, options={"memo": 0, "prune": 0, "dedupe": 0}),
            open_ctx(sc, seed, depths, WEIGHT)]
    # at many views or the largest window the host picks fewer than 16 warps: a twin at another count holds the same bits
    if views > 32 or box == 25:
        ctxs.append(open_ctx(sc, seed, depths, WEIGHT, options={"nwarps": 3 if views == 64 else 7}))
    A = ctxs[0]
    stepped = ctxs[1:2] + ctxs[3:]
    f = cost_of(A)
    cam = sc.cameras[0]
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    stats = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}
    try:
        for ctx in ctxs:
            ctx.init()
        n0, c0 = A.get_state()
        for ctx in ctxs[1:]:
            assert bits_equal(ctx.get_state()[0], n0) == 0 and bits_equal(ctx.get_state()[1], c0) == 0
        A.reset_stats()
        for _ in range(2):
            for colour in (0, 1):
                for mask in (1, 2, 4):
                    before = A.get_state()
                    if mask != 4:
                        want_p, want_c, amb = pp.expected(before[0], before[1], colour, mask, f, cam, sc.params.depthMin,
                                                          sc.params.depthMax, color_images=color)
                    A.phase(colour, mask)
                    after = A.get_state()
                    for other in stepped:
                        other.phase(colour, mask)
                    for other in ctxs[3:]:                          # the warp-count twin, launch by launch
                        p, c = other.get_state()
                        assert bits_equal(p, after[0]) == 0 and bits_equal(c, after[1]) == 0, ("nwarps", colour, mask)
                    if mask != 4:
                        bad = ((after[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) |
                               (after[1].view(np.uint32) != want_c.view(np.uint32))) & ~amb
                        assert not bad.any(), (colour, mask, int(bad.sum()), np.argwhere(bad)[:8].tolist())
                        mine = ((xs + ys) & 1) == colour
                        stats["compared"] += int((mine & ~amb).sum())
                        stats["ambiguous"] += int((mine & amb).sum())
                        stats["accepted"] += int((mine & (after[1] < before[1])).sum())
                        check_launch(before, after, colour)
                    else:
                        stats["refined"] += check_launch(before, after, colour, f, sc, pp.refine_site(False, color))
                ctxs[2].phase(colour, 7)
                ref_p, ref_c = A.get_state()
                for other in ctxs[1:]:
                    p, c = other.get_state()
                    assert bits_equal(p, ref_p) == 0 and bits_equal(c, ref_c) == 0, colour
        st = A.stats()
    finally:
        for ctx in ctxs:
            ctx.close()
    share = stats["ambiguous"] / max(1, stats["compared"] + stats["ambiguous"])
    print("\ngeometric %dx%d, %d views, box %d, colour=%s: %s, ambiguous %.4f, pruned %d of %d, %.2f s" %
          (rows, cols, views, box, color, stats, share, st["pruned"], st["hypotheses"], time.perf_counter() - t0))
    assert stats["accepted"] > 0 and stats["refined"] > 0 and share <= 0.005
    ns = ((box - 1) // 2 + 1) ** 2
    assert st["pairs_full"] == st["hypotheses"] * views * ns           # box 25: 169 samples, 5 x 32 + 9, six rounds
    if ns > 32:
        assert st["pruned"] > 0                   # the lower bound with the geometric term does cut hypotheses short
    else:
        assert st["pruned"] == 0                  # one round: the bound is the final cost


def test_refusals_leave_launch_count_and_state_untouched():
    from gipuma_b200 import api
    sc = make_scene(53, 75, 3)
    depths = depth_maps(sc, 5)
    E_ARG, E_STATE = -1, -3
    with open_ctx(sc, depths=depths[:2], views=[0, 1]) as ctx:
        L, h = ctx.lib, ctx.h
        ctx.init()
        ctx.sweep(1)
        state, launches = ctx.get_state(), ctx.stats()["launches"]
        d = np.ascontiguousarray(depths[0])
        dp = ctypes.c_void_p(d.ctypes.data)
        cf = ctypes.c_float
        calls = [
            (lambda: L.gpm_set_geometric(h, cf(-0.5), cf(1.0)), E_ARG),
            (lambda: L.gpm_set_geometric(h, cf(float("nan")), cf(1.0)), E_ARG),
            (lambda: L.gpm_set_geometric(h, cf(float("inf")), cf(1.0)), E_ARG),
            (lambda: L.gpm_set_geometric(h, cf(1.0), cf(0.0)), E_ARG),
            (lambda: L.gpm_set_geometric(h, cf(1.0), cf(-2.0)), E_ARG),
            (lambda: L.gpm_set_view_depth(h, 2, dp, 0, 0), E_ARG),                 # max_views is 2
            (lambda: L.gpm_set_view_depth(h, -1, dp, 0, 0), E_ARG),
            (lambda: L.gpm_set_view_depth(h, 0, dp, 6, 0), E_ARG),                 # pitch not a multiple of 4
        ]
        for call, want in calls:
            assert call() == want, L.gpm_last_error().decode()
        with api.Context(sc.cols, sc.rows, 3) as c3:              # a used view without a depth map
            c3.set_params(sc.params)
            c3.set_reference(sc.images[0], sc.cameras[0])
            for v in range(3):
                c3.set_view(v, sc.images[sc.subset[v]], sc.cameras[sc.subset[v]])
            c3.set_num_views(2)
            for v in range(2):
                c3.set_view_depth(v, depths[v])
            c3.init()
            s3, l3 = c3.get_state(), c3.stats()["launches"]
            c3.set_num_views(3)
            assert c3.lib.gpm_set_geometric(c3.h, cf(WEIGHT), cf(MAX_ERR)) == E_STATE
            c3.set_num_views(2)
            c3.set_geometric(WEIGHT, MAX_ERR)
            c3.set_num_views(3)                                   # the next launch refuses
            for fn in (lambda: c3.sweep(1), lambda: c3.init(), lambda: c3.phase(0, 7), lambda: c3.cost_eval(s3[0])):
                with pytest.raises(api.GipumaError, match="depth map"):
                    fn()
            assert c3.stats()["launches"] == l3 and bits_equal(c3.get_state()[0], s3[0]) == 0 and bits_equal(c3.get_state()[1], s3[1]) == 0
        ctx.set_geometric(WEIGHT, MAX_ERR)
        geo_calls = [
            (lambda: L.gpm_set_option(h, b"neighbours", 20), E_ARG),
            (lambda: L.gpm_shard_stage(h, 0, 1, None, 1, None), E_STATE),
            (lambda: L.gpm_shard_finish_init(h, dp, 1), E_STATE),
            (lambda: L.gpm_shard_run(h, None), E_STATE),
            (lambda: L.gpm_shard_comm_init(h, None, 0, 1), E_STATE),
            (lambda: L.gpm_shard_comm_attach(h, None, 0, 1), E_STATE),
            (lambda: L.gpm_shard_num_stages(h), -1),
            (lambda: L.gpm_shard_stage_floats(h, 1), -1),
        ]
        for call, want in geo_calls:
            assert call() == want, L.gpm_last_error().decode()
        ctx.set_geometric(0.0, MAX_ERR)
        ctx.set_option("neighbours", 20)
        assert L.gpm_set_geometric(h, cf(WEIGHT), cf(MAX_ERR)) == E_ARG                # the fused sweep has no such variant
        assert ctx.stats()["launches"] == launches
        after = ctx.get_state()
        assert bits_equal(after[0], state[0]) == 0 and bits_equal(after[1], state[1]) == 0


def test_two_pass_driver_runs_fuses_and_scores():
    from gipuma_b200 import api, scene as S
    from test_gpu_fusion import FUSE, REFS, _dataset, _params
    Ps, scale, images, hf = _dataset()
    fPs = [Ps[r] for r in REFS]
    H, W = images.shape[1:]
    gt = S.gt_points(fPs, scale, H, W, hf)
    unit = hf.unit
    taus = (0.25 * unit, 0.5 * unit, unit)
    p = _params()
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    photo, _, _ = api.batch_run(images, Ps, p, REFS, **kw)
    p.iterations = 2
    n4, cost, info = api.geometric_pass(images, Ps, p, REFS, geo_iterations=1, **kw)
    assert n4.shape == photo.shape and cost.shape == photo.shape[:3]
    assert set(REFS) <= set(info["pass1_views"]) and len(info["pass2_sweep_s"]) == len(REFS)
    assert np.all(np.isfinite(n4)) and (n4[..., 3] > 0).mean() > 0.5
    scores = {}
    for name, maps in (("photometric 3", photo), ("photometric 2 + geometric 1", n4)):
        v, _ = api.fuse(maps, fPs, cam_scale=scale, **FUSE)
        s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=taus)
        scores[name] = {k: s[k] for k in ("accuracy_mean", "completeness_mean", "f_score")}
        assert len(v) > 1000 and np.isfinite(s["accuracy_mean"]) and s["f_score"][2] > 0.5
    print("\n%s" % scores)
