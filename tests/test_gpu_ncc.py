"""The NCC photometric cost (DESIGN.md §15) on the GPU.

- the default is unchanged: a context switched PM -> NCC -> PM runs bit-identical to a fresh one (grey, geometric), and a
  colour context whose switch was refused too;
- the arithmetic is bit-exact: with cameras that make every homography an integer translation and gamma = 1e30 (w_s = 1),
  gpm_cost_eval equals oracle/pyncc + oracle/pygeo.combine bit for bit (1 and 4 views, best_n / all / good, geometric term);
- on rendered scenes at ragged sizes the per-view costs agree with the float64 restatement within a measured tolerance,
  which most PM costs and most costs of another view fall outside; a per-view gain and offset moves NCC costs within it
  and PM costs by far more;
- every propagation decision equals oracle/pypropagate.expected() with this cost, refinement keeps its invariants, and
  twins without memo and duplicate skips, or with one mask-7 launch per colour, stay bit-identical;
- every refusal leaves the launch count and the state untouched;
- batch_run and geometric_pass with photometric="ncc" equal the same flows restated through Context calls (the geometric
  one is test_gpu_geometric_batch's restatement on NCC contexts), on the fusion test's dataset and a ragged one, with one and
  two workers, and the NCC cloud beats the PM cloud on the fusion test's dataset under a per-view gain and offset."""
import ctypes
import time
from types import SimpleNamespace

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_sweep_any_size import cost_of, check_launch
from test_gpu_geometric import depth_maps, learn_rcp, make_scene, open_ctx

pytestmark = pytest.mark.gpu

f32 = np.float32
MIN_STD = 2.0
WEIGHT, MAX_ERR = 0.3, 6.0
# |device - float64 restatement| of one view's NCC cost: at most 0.0034 measured on an H100 80GB HBM3 (700 W) over the scenes
# of test_cost_agrees_with_float64_within_tolerance (the texture unit's 8-bit filter weights are the only expected
# difference); PM costs and swapped views differ from the restatement by more than 1.6 there
TOL = 0.02


def ncc_ctx(sc, seed=99, depths=None, weight=0.0, views=None, options=None, min_std=MIN_STD):
    ctx = open_ctx(sc, seed, depths, weight, views, options)
    ctx.set_photometric("ncc", min_std)
    return ctx


# ---- 1. the default is unchanged ------------------------------------------------------------------------------------
@pytest.mark.parametrize("geo", [False, True])
def test_switching_back_to_pm_changes_nothing(geo):
    sc = make_scene(53, 75, 4)
    depths = depth_maps(sc, 1) if geo else None
    outs = []
    for switch in (False, True):
        with open_ctx(sc, depths=depths, weight=WEIGHT if geo else 0.0) as ctx:
            if switch:
                ctx.set_photometric("ncc", 3.0)
                ctx.run()
                ctx.set_photometric("pm")
            ctx.run()
            outs.append(ctx.get_state())
    assert bits_equal(outs[0][0], outs[1][0]) == 0 and bits_equal(outs[0][1], outs[1][1]) == 0


def test_refused_switch_on_colour_context_changes_nothing():
    from gipuma_b200 import api
    sc = make_scene(53, 75, 3, color=True)
    outs = []
    for switch in (False, True):
        with open_ctx(sc) as ctx:
            if switch:
                assert ctx.lib.gpm_set_photometric(ctx.h, 1, ctypes.c_float(MIN_STD)) == -1
                with pytest.raises(api.GipumaError, match="grey"):
                    ctx.set_photometric("ncc")
            ctx.run()
            outs.append(ctx.get_state())
    assert bits_equal(outs[0][0], outs[1][0]) == 0 and bits_equal(outs[0][1], outs[1][1]) == 0


# ---- 2. bit-exact arithmetic on integer translations ----------------------------------------------------------------
F, CX, CY = 64.0, 40.0, 30.0


def translation_cam(sx, sy):
    """R = I, K = [[64, 0, 40], [0, 64, 30], [0, 0, 1]], t = (sx, sy, 0) / 64: the plane n = (0, 0, 1), d = -1 maps pixel
    (x, y) to (x + sx, y + sy) exactly (d = -2: half the shift, d = -0.5: twice it)."""
    from gipuma_b200 import api
    K = np.array([[F, 0, CX], [0, F, CY], [0, 0, 1]], np.float64)
    Ki = np.linalg.inv(K)
    g = api.GpmCamera()
    g.K[:], g.K_inv[:], g.R[:] = K.ravel().tolist(), Ki.ravel().tolist(), np.eye(3).ravel().tolist()
    g.M_inv[:], g.R_orig_inv[:] = Ki.ravel().tolist(), np.eye(3).ravel().tolist()
    g.t[:] = [sx / F, sy / F, 0.0]
    g.fx = g.fy = g.f = F
    g.alpha, g.baseline = 1.0, 0.54
    ns = SimpleNamespace(K=K.astype(f32), K_inv=Ki.astype(f32), R=np.eye(3, dtype=f32), t=np.array([sx / F, sy / F, 0], f32))
    return g, ns


def _rig(n=64, seed=2024):
    """Shifts and (gain, offset) of up to GPM_MAX_VIEWS = 64 views: four fixed ones, then distinct even shifts in
    [-8, 8]^2 (even: the d = -2 and -0.5 planes stay on integer texels) with a seeded gain and offset each."""
    rng = np.random.default_rng(seed)
    shifts = [(4, 0), (-8, 4), (0, -4), (12, 8)]
    light = [(1.0, 0.0), (2.0, -60.0), (0.5, 17.0), (1.0, 0.0)]
    pool = [(x, y) for x in range(-8, 9, 2) for y in range(-8, 9, 2) if (x, y) != (0, 0) and (x, y) not in shifts]
    shifts += [pool[i] for i in rng.permutation(len(pool))[:n - 4]]
    light += [(float(rng.uniform(0.5, 2.0)), float(rng.uniform(-60.0, 40.0))) for _ in range(n - 4)]
    return shifts, light


SHIFTS, LIGHT = _rig()


def translation_case(rows, cols, views, box, seed):
    from gipuma_b200 import scene as S
    rng = np.random.default_rng(seed)
    ref = rng.integers(0, 256, (rows, cols)).astype(f32)
    ys, xs = np.mgrid[0:rows, 0:cols]
    imgs = []
    for v in range(views):
        sx, sy = SHIFTS[v]
        src = ref[np.clip(ys - sy, 0, rows - 1), np.clip(xs - sx, 0, cols - 1)]          # content of ref moved by (sx, sy)
        gain, off = LIGHT[v]
        img = np.clip(gain * src + off + rng.integers(-20, 21, src.shape) * (v % 4 == 3), 0, 255)       # noise on every 4th
        imgs.append(np.floor(img).astype(f32))
    p = S.AlgorithmParameters(box_hsize=box, box_vsize=box, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N, gamma=1e30)
    p.depthMin, p.depthMax = 0.1, 100.0
    d = rng.choice(np.array([-1.0, -2.0, -0.5], f32), (rows, cols))
    planes = np.stack([np.zeros_like(d), np.zeros_like(d), np.ones_like(d), d], axis=-1).astype(f32)
    return ref, imgs, p, planes


def translation_ctx(ref, imgs, p, views, min_std=MIN_STD):
    from gipuma_b200 import api
    rows, cols = ref.shape
    ctx = api.Context(cols, rows, views)
    ctx.set_params(p)
    ctx.set_reference(ref, translation_cam(0, 0)[0])
    for v in range(views):
        ctx.set_view(v, imgs[v], translation_cam(*SHIFTS[v])[0])
    ctx.set_num_views(views)
    ctx.set_photometric("ncc", min_std)
    return ctx


def restated_translation(ref, imgs, planes, box, views, min_std=MIN_STD):
    """Per-view costs [V, H, W] of pyncc with w = 1: r and t read off the images at the (clamped) integer sample pixels."""
    from oracle import pyncc
    rows, cols = ref.shape
    ys, xs = np.mgrid[0:rows, 0:cols]
    offs = pyncc.window_offsets(box)
    r = np.stack([ref[np.clip(ys + j, 0, rows - 1), np.clip(xs + i, 0, cols - 1)] for i, j in offs], axis=-1)
    scale = (-1.0 / planes[..., 3]).astype(np.float64)                 # d = -1: 1, -2: 0.5, -0.5: 2
    out = []
    for v in range(views):
        sx, sy = SHIFTS[v]
        tx, ty = (xs + sx * scale).astype(np.int64), (ys + sy * scale).astype(np.int64)
        t = np.stack([imgs[v][np.clip(ty + j, 0, rows - 1), np.clip(tx + i, 0, cols - 1)] for i, j in offs], axis=-1)
        out.append(pyncc.ncc_cost(np.ones_like(r), r, t, min_std))
    return np.stack(out)


def ns_of(box):
    """Samples of a propagation window: box 3 is one 4-sample round, 11 is 32 + 4, 15 is 32 + 32, 25 is 5 x 32 + 9."""
    return ((box - 1) // 2 + 1) ** 2


@pytest.mark.parametrize("box", [3, 11, 15, 25])
def test_cost_of_one_view_is_bit_exact(box):
    ref, imgs, p, planes = translation_case(45, 70, 1, box, box)
    with translation_ctx(ref, imgs, p, 1) as ctx:
        got = ctx.cost_eval(planes)
    want = restated_translation(ref, imgs, planes, box, 1)[0]
    assert bits_equal(got, want) == 0, np.argwhere(got != want)[:5]
    assert 0.05 < (want < 0.5).mean() < 0.999                          # correlated windows and others


# views, box, cost_comb, n_best, geometric term: 33 and 64 views put a second view in every lane (views lane + 32)
MANY = [(4, 15, 1, 2, False), (4, 11, 0, 2, False), (4, 15, 3, 2, False), (4, 11, 1, 2, True),
        (33, 3, 1, 2, False), (64, 25, 1, 3, False), (64, 11, 1, 40, False), (40, 15, 0, 2, False), (40, 15, 3, 2, False),
        (64, 9, 1, 3, True), (33, 25, 0, 2, True)]


@pytest.mark.parametrize("views,box,comb,n_best,geo", MANY)
def test_cost_of_many_views_is_bit_exact(views, box, comb, n_best, geo):
    from oracle import pygeo
    t0 = time.perf_counter()
    ref, imgs, p, planes = translation_case(45, 70, views, box, 100 + box + comb + views)
    p.cost_comb, p.n_best = comb, n_best
    per_view = restated_translation(ref, imgs, planes, box, views)
    if views > 32:          # a view read in place of its lane partner (j <-> j - 32) would change the sums
        assert (per_view[32:] != per_view[:views - 32]).mean() > 0.5
    with translation_ctx(ref, imgs, p, views) as ctx:
        c0 = ctx.cost_eval(planes)
        s0, k0 = pygeo.combine_sum(per_view, comb, n_best, p.good_factor)
        rcp = learn_rcp(k0, s0, c0)
        assert bits_equal(pygeo.combine(per_view, comb, n_best, p.good_factor, rcp), c0) == 0
        if geo:
            depths = [np.full(ref.shape, 5.0, f32) * (1 + 0.1 * v) for v in range(views)]
            depths[1][::3] = 0.0
            for v in range(views):
                ctx.set_view_depth(v, depths[v])
            ctx.set_geometric(WEIGHT, MAX_ERR)
            got = ctx.cost_eval(planes)
            rc = translation_cam(0, 0)[1]
            g = np.stack([pygeo.geo_cost(planes, rc, translation_cam(*SHIFTS[v])[1], depths[v], WEIGHT, MAX_ERR,
                                         p.depthMin, p.depthMax) for v in range(views)])
            want = pygeo.combine((per_view + g).astype(f32), comb, n_best, p.good_factor, rcp)
            known = ~np.isnan(want)
            assert known.mean() > 0.98 and bits_equal(got[known], want[known]) == 0
            assert (g < f32(WEIGHT * MAX_ERR)).any()
            if views > 32:
                assert (g[32:] < f32(WEIGHT * MAX_ERR)).any()               # views lane + 32 score a real error
    print("\nNCC translation rig, %d views, box %d, comb %d, n_best %d, geo %s: %.2f s" %
          (views, box, comb, n_best, geo, time.perf_counter() - t0))


# ---- 3, 4. general scenes: float64 tolerance and gain invariance ----------------------------------------------------
def per_view_costs(sc, planes, photometric, images=None):
    out = []
    for v in range(sc.n_views):
        with open_ctx(sc, views=[v]) as one:
            if images is not None:
                one.set_view(0, images[sc.subset[v]], sc.cameras[sc.subset[v]])
            if photometric == "ncc":
                one.set_photometric("ncc", MIN_STD)
            out.append(one.cost_eval(planes))
    return np.stack(out)


def random_planes(sc, seed):
    with open_ctx(sc, seed) as ctx:
        ctx.init()
        p0 = ctx.get_state()[0]
        ctx.sweep(1)
        return [p0, ctx.get_state()[0]]


def lit(sc, seed):
    """The scene's images under a seeded per-view gain and offset (the reference image untouched)."""
    rng = np.random.default_rng(seed)
    imgs = sc.images.copy()
    for i in range(1, len(imgs)):
        imgs[i] = rng.uniform(0.6, 1.4) * imgs[i] + rng.uniform(-40, 40)
    return imgs.astype(f32)


@pytest.mark.parametrize("rows,cols", [(53, 75), (37, 61)])
def test_cost_agrees_with_float64_within_tolerance(rows, cols):
    from oracle import pyncc
    sc = make_scene(rows, cols, 3, box=11)
    p = sc.params
    errs, pm_errs, swap_errs, n_sharp = [], [], [], 0
    for planes in random_planes(sc, rows):
        got = per_view_costs(sc, planes, "ncc")
        pm = per_view_costs(sc, planes, "pm")
        w, r, t = pyncc.sample_views64(sc.images[0], [sc.images[i] for i in sc.subset], sc.cameras[0],
                                       [sc.cameras[i] for i in sc.subset], planes, p.box_hsize, p.gamma)
        want = pyncc.ncc_cost64(w, r, t, MIN_STD)
        # windows at the variance floor may go either way: compared where both variances clear it by 1 %
        vr = (w * (r - ((w * r).sum(-1) / w.sum(-1))[..., None]) ** 2).sum(-1) / w.sum(-1)
        vt = (w * (t - ((w * t).sum(-1) / w.sum(-1))[..., None]) ** 2).sum(-1) / w.sum(-1)
        clear = (vr[None] > 1.01 * MIN_STD ** 2) & (vt > 1.01 * MIN_STD ** 2)
        e = np.abs(got - want)[clear]
        errs.append(e)
        pm_errs.append(np.abs(pm - want)[clear])
        swap_errs.append(np.abs(np.roll(got, 1, axis=0) - want)[clear])       # every view scored against another's
        n_sharp += int((want < 0.5).sum())
    e, epm, esw = (np.concatenate(x) for x in (errs, pm_errs, swap_errs))
    share_pm, share_swap = (epm > TOL).mean(), (esw > TOL).mean()
    print("\nNCC vs float64 %dx%d: max %.5f p99.9 %.5f; beyond the tolerance: PM %.4f, swapped views %.4f of %d view costs" %
          (rows, cols, e.max(), np.percentile(e, 99.9), share_pm, share_swap, len(e)))
    assert e.max() <= TOL and n_sharp > 0
    # the tolerance tells the costs apart: most PM costs and most costs of the wrong view fall outside it
    assert share_pm > 0.9 and share_swap > 0.5, (share_pm, share_swap)


def test_gain_and_offset_move_ncc_within_tolerance_and_pm_far():
    sc = make_scene(53, 75, 3, box=11)
    imgs = lit(sc, 5)
    dn, dp = [], []
    for planes in random_planes(sc, 5):
        dn.append(np.abs(per_view_costs(sc, planes, "ncc") - per_view_costs(sc, planes, "ncc", imgs)).ravel())
        dp.append(np.abs(per_view_costs(sc, planes, "pm") - per_view_costs(sc, planes, "pm", imgs)).ravel())
    dn, dp = np.concatenate(dn), np.concatenate(dp)
    # NCC: only windows near the variance floor (which the gain moves across) or clipped pixels may move more
    moved = (dn > TOL).mean()
    print("\ngain: NCC moved > tol %.4f, NCC median %.5f; PM median %.3f" % (moved, np.median(dn), np.median(dp)))
    assert moved < 0.02 and np.median(dn) < TOL / 4 and np.median(dp) > 20 * np.median(dn)


# ---- 5. decisions ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols,views,box,geo", [(53, 75, 4, 15, False), (97, 65, 4, 15, False), (53, 75, 4, 15, True),
                                                     (31, 33, 4, 15, True), (40, 60, 33, 3, False), (40, 60, 33, 25, True),
                                                     (40, 60, 64, 3, True), (40, 60, 64, 25, False)])
def test_sweep_decisions_exact(rows, cols, views, box, geo):
    from oracle import pypropagate as pp
    t0 = time.perf_counter()
    sc = make_scene(rows, cols, views, box=box)
    depths = depth_maps(sc, 3) if geo else None
    wgt = WEIGHT if geo else 0.0
    seed = 5000 + rows + cols
    ctxs = [ncc_ctx(sc, seed, depths, wgt), ncc_ctx(sc, seed, depths, wgt, options={"memo": 0, "dedupe": 0}),
            ncc_ctx(sc, seed, depths, wgt)]
    # at many views or the largest window the host picks fewer than 16 warps: a twin at another count holds the same bits
    if views > 32 or box == 25:
        ctxs.append(ncc_ctx(sc, seed, depths, wgt, options={"nwarps": 3 if views == 64 else 7}))
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
        # an NCC cost in [0, 2] plus a geometric term in [0, weight * max_err], up to the float32 roundings of the sum and
        # of the mean (at box 3 whole windows are flat, NCC 2, and project nowhere, g = weight * max_err)
        assert np.all((c0 >= 0) & (c0 <= (2 + WEIGHT * MAX_ERR) * (1 + 2 ** -20)))
        for ctx in ctxs[1:]:
            assert bits_equal(ctx.get_state()[0], n0) == 0 and bits_equal(ctx.get_state()[1], c0) == 0
        A.reset_stats()
        for _ in range(2):
            for colour in (0, 1):
                for mask in (1, 2, 4):
                    before = A.get_state()
                    if mask != 4:
                        want_p, want_c, amb = pp.expected(before[0], before[1], colour, mask, f, cam, sc.params.depthMin,
                                                          sc.params.depthMax)
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
                        stats["refined"] += check_launch(before, after, colour, f, sc, 0)
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
    print("\nNCC %dx%d, %d views, box %d, geo=%s: %s, ambiguous %.4f, %s, %.2f s" %
          (rows, cols, views, box, geo, stats, share, st, time.perf_counter() - t0))
    assert stats["accepted"] > 0 and stats["refined"] > 0 and share <= 0.005
    assert st["pruned"] == 0 and st["pairs"] == st["pairs_full"]          # no early-out on NCC costs
    assert st["pairs_full"] == st["hypotheses"] * views * ns_of(box)      # every hypothesis ran all rounds_of(box) rounds


# ---- 6. refusals ----------------------------------------------------------------------------------------------------
def test_refusals_leave_launch_count_and_state_untouched():
    sc = make_scene(53, 75, 2)
    gsc = make_scene(53, 75, 2, color=True)
    E_ARG, E_STATE = -1, -3
    cf = ctypes.c_float
    with ncc_ctx(sc) as ctx:
        L, h = ctx.lib, ctx.h
        ctx.init()
        ctx.sweep(1)
        state, launches = ctx.get_state(), ctx.stats()["launches"]
        rgba = np.ascontiguousarray(gsc.images[1])
        rp = ctypes.c_void_p(rgba.ctypes.data)
        from gipuma_b200 import api
        g = api.pack_camera(sc.cameras[1])
        calls = [
            (lambda: L.gpm_set_photometric(h, 2, cf(MIN_STD)), E_ARG),
            (lambda: L.gpm_set_photometric(h, -1, cf(MIN_STD)), E_ARG),
            (lambda: L.gpm_set_photometric(h, 1, cf(0.0)), E_ARG),
            (lambda: L.gpm_set_photometric(h, 1, cf(-1.0)), E_ARG),
            (lambda: L.gpm_set_photometric(h, 1, cf(float("nan"))), E_ARG),
            (lambda: L.gpm_set_photometric(h, 1, cf(float("inf"))), E_ARG),
            (lambda: L.gpm_set_option(h, b"neighbours", 20), E_ARG),
            (lambda: L.gpm_set_view_color(h, 0, rp, 0, 0, ctypes.byref(g)), E_STATE),
            (lambda: L.gpm_set_reference_color(h, rp, 0, 0, ctypes.byref(g)), E_STATE),
            (lambda: L.gpm_shard_stage(h, 0, 1, None, 1, None), E_STATE),
            (lambda: L.gpm_shard_finish_init(h, rp, 1), E_STATE),
            (lambda: L.gpm_shard_run(h, None), E_STATE),
            (lambda: L.gpm_shard_comm_init(h, None, 0, 1), E_STATE),
            (lambda: L.gpm_shard_comm_attach(h, None, 0, 1), E_STATE),
            (lambda: L.gpm_shard_num_stages(h), -1),
            (lambda: L.gpm_shard_stage_floats(h, 1), -1),
        ]
        for call, want in calls:
            assert call() == want, L.gpm_last_error().decode()
        ctx.sweep(1)                                    # still NCC, still grey, same stored state: identical to a twin
        with ncc_ctx(sc) as twin:
            twin.init()
            twin.sweep(2)
            assert bits_equal(ctx.get_state()[1], twin.get_state()[1]) == 0
        ctx.set_photometric("pm")
        ctx.set_option("neighbours", 20)
        assert L.gpm_set_photometric(h, 1, cf(MIN_STD)) == E_ARG           # the fused sweep has no NCC variant
        ctx.set_option("neighbours", 8)
        ctx.set_photometric("ncc", MIN_STD)
        assert ctx.stats()["launches"] == launches + 2
    with open_ctx(gsc) as cctx:                                           # NCC on a colour context
        cctx.init()
        s, n = cctx.get_state(), cctx.stats()["launches"]
        assert cctx.lib.gpm_set_photometric(cctx.h, 1, cf(MIN_STD)) == E_ARG
        assert cctx.stats()["launches"] == n and bits_equal(cctx.get_state()[1], s[1]) == 0


# ---- 7, 8. drivers and quality ----------------------------------------------------------------------------------------
def _restated_batch(images, Ps, params, refs, cam_scale, min_angle, max_angle, max_views, seed):
    """batch_run's per-reference job through Context calls: cameras re-based on the reference, view selection, depth and
    disparity range in the driver's float arithmetic (main.cpp:480-483, 905-906), uploads, gpm_run."""
    import ctypes as C
    from gipuma_b200 import api
    n, H, W = images.shape[:3]
    n4 = np.empty((len(refs), H, W, 4), f32)
    cc = np.empty((len(refs), H, W), f32)
    with api.Context(W, H, max_views) as ctx:
        ctx.set_photometric("ncc", MIN_STD)
        for j, ref in enumerate(refs):
            order = [ref] + [i for i in range(n) if i != ref]
            cams = api.prepare_cameras([Ps[i] for i in order], cam_scale)
            subset, (lo, hi) = api.select_views(cams, W, H, min_angle, max_angle, max_views)
            p = api.GpmParams.from_buffer_copy(api.pack_params(params))
            p.depthMin = p.depthMin if p.depthMin > 0 else lo
            p.depthMax = p.depthMax if p.depthMax > 0 else hi
            fb = f32(cams[0].f) * f32(cams[0].baseline)
            p.min_disparity, p.max_disparity = float(fb / f32(p.depthMax)), float(fb / f32(p.depthMin))
            ctx._check(ctx.lib.gpm_set_params(ctx.h, C.byref(p)))
            ctx.set_reference(images[ref], cams[0])
            for v, k in enumerate(subset):
                ctx.set_view(v, images[order[k]], cams[k])
            ctx.set_num_views(len(subset))
            ctx.set_rng(seed, api.GPM_RNG_REFERENCE)
            ctx.run()
            n4[j], cc[j] = ctx.get_state()
    return n4, cc


@pytest.mark.parametrize("name", ["fusion", "ragged"])
def test_photometric_driver_equals_the_context_flow(name):
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case(name, False)
    w4, wc = _restated_batch(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], **gb.KW)
    for devices in ((0,), (0, 0)):
        n4, cost, _ = api.batch_run(c["images"], c["Ps"], c["params"], c["refs"], devices=devices, cam_scale=c["scale"],
                                    photometric="ncc", ncc_min_std=MIN_STD, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)


@pytest.mark.parametrize("name", ["fusion", "ragged"])
def test_geometric_driver_equals_the_context_flow(name, monkeypatch):
    """geometric_pass(photometric="ncc") against test_gpu_geometric_batch's restatement of the two-pass flow, run on
    contexts switched to the NCC cost (both passes, including the cost_eval of the pass-1 planes under NCC + geometric)."""
    from gipuma_b200 import api
    import test_gpu_geometric_batch as gb
    c = gb._case(name, False)
    base, made = api.Context, []

    def ncc_context(*a, **k):                       # the driver sets the same cost for every job
        ctx = base(*a, **k)
        ctx.set_photometric("ncc", MIN_STD)
        made.append(ctx)
        return ctx
    with monkeypatch.context() as m:
        m.setattr(api, "Context", ncc_context)
        w4, wc, w_pass1, w_views = gb._restated(c["images"], c["Ps"], c["params"], c["refs"], c["scale"], weight=api.GEO_WEIGHT,
                                                max_err=api.GEO_MAX_ERR, **gb.KW)
    assert len(made) == 1
    for devices in ((0,), (0, 0)):
        n4, cost, info = api.geometric_pass(c["images"], c["Ps"], c["params"], c["refs"], geo_iterations=gb.GEO_ITERATIONS,
                                            cam_scale=c["scale"], devices=devices, photometric="ncc", ncc_min_std=MIN_STD, **gb.KW)
        assert bits_equal(n4, w4) == 0 and bits_equal(cost, wc) == 0, (name, devices)
        assert info["pass1_views"] == w_pass1 and info["views"] == w_views, devices


def test_ncc_cloud_beats_pm_under_gain_and_offset():
    from gipuma_b200 import api, scene as S
    from test_gpu_fusion import FUSE, REFS, _dataset, _params
    Ps, scale, images, hf = _dataset()
    rng = np.random.default_rng(9)
    lit_imgs = np.stack([rng.uniform(0.6, 1.4) * im + rng.uniform(-40, 40) for im in images]).astype(f32)
    fPs = [Ps[r] for r in REFS]
    H, W = images.shape[1:]
    gt = S.gt_points(fPs, scale, H, W, hf)
    unit = hf.unit
    kw = dict(cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    f1 = {}
    for name in ("pm", "ncc"):
        n4, _, _ = api.batch_run(lit_imgs, Ps, _params(), REFS, photometric=name, **kw)
        v, _ = api.fuse(n4, fPs, cam_scale=scale, **FUSE)
        s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=(0.25 * unit, 0.5 * unit, unit))
        f1[name] = s["f_score"][2]
    print("\nlit fusion dataset F-score at one unit: %s" % f1)
    assert f1["ncc"] > f1["pm"] + 0.05                  # measured on an H100: 0.853 against 0.731
