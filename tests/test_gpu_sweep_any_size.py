"""Every decision of k_sweep checked exactly at image sizes that are not whole tiles, and in the colour, fused and
stateful-RNG modes, without any reference output.

A propagation launch is a pure function of the planes and costs it starts from, so the state after it must equal
oracle/pypropagate.expected() — the acceptance rule folded in numpy over gpm_cost_eval's costs of the neighbour-shifted
plane maps, with each call site's rounding variant — bit for bit, outside the few pixels whose depth-range test is
ambiguous.  That holds whatever memo, provenance or identity history the context carries, so the exact shortcuts
(memo of rejected work, duplicates, lower-bound early-out) are checked with it too, also on adversarial states with ties,
out-of-range candidates, equal-cost candidates with different bits and MAXCOST plateaus.  gpm_cost_eval shares its
window staging and cost code with the sweep, so its costs are compared with the scalar oracle at the same shapes.
Refinement launches are checked by their invariants (cost of every new plane = its evaluation, unit camera-facing
normals, nothing else changes), the only exact checks GPM_RNG_STATEFUL has.  Contexts that run the same chain as one
mask-7 launch per colour, without the exact shortcuts, with other warp counts, or without the interleaved gpm_cost_eval
calls must stay bit-identical."""
import time

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

MAXCOST = np.float32(1000.0)
REPORT = {}

# id: (rows, cols, views, box, colour images, fused, stateful RNG, params overrides, nwarps)
CASES = {
    "grey_53x75": (53, 75, 4, 9, False, False, False, {}, None),
    "grey_8x8_box25": (8, 8, 2, 25, False, False, False, {}, None),          # window larger than the image
    "grey_31x33": (31, 33, 3, 15, False, False, False, {}, None),
    "grey_40x200": (40, 200, 5, 11, False, False, False, {}, None),
    "grey_97x65": (97, 65, 6, 3, False, False, False, {}, None),
    "grey_480x640": (480, 640, 10, 15, False, False, False, {}, None),      # 300 tiles: gridDim.z = 4 on 132 SMs
    "grey_550x1000": (550, 1000, 10, 15, False, False, False, {}, None),    # 576 tiles: gridDim.z = 2 on 132 SMs
    "colour_53x75": (53, 75, 4, 9, True, False, False, {}, None),
    "colour_31x33_box25": (31, 33, 3, 25, True, False, False, {}, None),
    "fused_grey_53x75": (53, 75, 4, 9, False, True, False, {}, None),
    "fused_colour_53x75": (53, 75, 4, 9, True, True, False, {}, None),
    "fused_grey_29x41": (29, 41, 3, 7, False, True, False, {}, None),
    "fused_colour_29x41": (29, 41, 3, 7, True, True, False, {}, None),
    "stateful_53x75": (53, 75, 4, 9, False, False, True, {}, None),
    "stateful_97x65": (97, 65, 6, 3, False, False, True, {}, None),
    "nbest_above_views_53x75": (53, 75, 4, 9, False, False, False, {"n_best": 6}, None),
    "comb_all_53x75": (53, 75, 4, 9, False, False, False, {"cost_comb": 0}, None),
    "comb_good_53x75": (53, 75, 4, 9, False, False, False, {"cost_comb": 3}, None),
    "nwarps5_53x75": (53, 75, 4, 9, False, False, False, {}, 5),
    "nwarps16_53x75": (53, 75, 4, 9, False, False, False, {}, 16),
}


def make_scene(case):
    from gipuma_b200 import scene as S
    rows, cols, views, box, color, fused, stateful, prm, nwarps = CASES[case]
    sc = S.make_config(2, rows=rows, cols=cols, n_views=views, iterations=2, seed=rows * 1000 + cols)
    sc.params.box_hsize = sc.params.box_vsize = box
    for k, v in prm.items():
        setattr(sc.params, k, v)
    return S.colorize(sc) if color else sc


def open_context(case, sc, seed, options=None):
    from gipuma_b200 import api
    rows, cols, views, box, color, fused, stateful, prm, nwarps = CASES[case]
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    opts = {"neighbours": 20 if fused else 8}
    if nwarps:
        opts["nwarps"] = nwarps
    opts.update(options or {})
    for k, v in opts.items():
        ctx.set_option(k, v)
    ctx.load_scene(sc, seed=seed, rng_mode=api.GPM_RNG_STATEFUL if stateful else api.GPM_RNG_REFERENCE)
    return ctx


def cost_of(ctx):
    """gpm_cost_eval with the rounding variant of one call site; the option is reset to automatic afterwards."""
    def f(planes, site):
        ctx.set_option("cost_variant", site)
        try:
            return ctx.cost_eval(planes)
        finally:
            ctx.set_option("cost_variant", -1)
    return f


def bands(H):
    """Rows [0, 6) and the last 6 rows (part of the last, partial tile row unless H is a multiple of 32)."""
    b = min(H, 6)
    return [(0, b), (H - b, H)] if H > b else [(0, H)]


def assert_close_to_oracle(got, want, y0, y1, what):
    err = np.abs(got[y0:y1] - want[y0:y1]) / np.maximum(1.0, want[y0:y1])       # the bound of test_oracle.py
    assert np.percentile(err, 99) < 2e-3 and err.max() < 5e-2, (what, y0, float(np.percentile(err, 99)), float(err.max()))


def view_rays(cam, H, W):
    """Direction of each pixel's ray (getViewVector_cu, gipuma.cu:122-130) in float64."""
    ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
    p4 = cam.P[:, 3].astype(np.float64)
    pt = np.stack([xs - p4[0], ys - p4[1], np.full_like(xs, 1.0 - p4[2])], axis=-1)
    return pt @ cam.M_inv.astype(np.float64).T - cam.C.astype(np.float64)


def check_launch(before, after, colour, cost_fn=None, sc=None, site=None):
    """Invariants of any launch of one colour; for a refinement launch (cost_fn given) also those of refinement."""
    (p0, c0), (p1, c1) = before, after
    H, W = c0.shape
    ys, xs = np.mgrid[0:H, 0:W]
    other = ((xs + ys) & 1) != colour
    assert bits_equal(p1[other], p0[other]) == 0 and bits_equal(c1[other], c0[other]) == 0
    assert np.all(c1 <= c0)                                                   # the cost never increases
    if cost_fn is None:
        return 0
    changed = (p1.view(np.uint32) != p0.view(np.uint32)).any(axis=-1)
    assert bits_equal(c1[~changed], c0[~changed]) == 0
    if changed.any():
        assert bits_equal(c1[changed], cost_fn(p1, site)[changed]) == 0
        n = p1[changed][:, :3].astype(np.float64)
        assert np.all(np.abs(np.linalg.norm(n, axis=-1) - 1.0) <= 1e-5)
        v = view_rays(sc.cameras[0], H, W)[changed]
        assert np.all(np.einsum("ij,ij->i", n, v) <= 1e-6 * np.linalg.norm(v, axis=-1))   # faces the camera
    return int(changed.sum())


def decision_chain(case, sc, ctxs, iterations=2):
    """Context 0 runs phase(c, 1), phase(c, 2), phase(c, 4) with every decision checked against the restatement and
    gpm_cost_eval calls in between; context 1 (if any) runs the same separate masks without any gpm_cost_eval; the others
    one mask-7 launch per colour.  All must hold bit-identical states after every colour."""
    from oracle import pypropagate as pp
    rows, cols, views, box, color, fused, stateful, prm, nwarps = CASES[case]
    A = ctxs[0]
    f = cost_of(A)
    cam = sc.cameras[0]
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    stats = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}
    for _ in range(iterations):
        for colour in (0, 1):
            for mask in (1, 2, 4):
                before = A.get_state()
                if mask != 4:
                    want_p, want_c, amb = pp.expected(before[0], before[1], colour, mask, f, cam, sc.params.depthMin,
                                                      sc.params.depthMax, fused=fused, color_images=color)
                A.phase(colour, mask)
                after = A.get_state()
                if mask != 4:
                    keep = ~amb
                    bad = (after[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) | \
                          (after[1].view(np.uint32) != want_c.view(np.uint32))
                    bad &= keep
                    assert not bad.any(), (case, colour, mask, int(bad.sum()), np.argwhere(bad)[:8].tolist())
                    mine = ((xs + ys) & 1) == colour
                    stats["compared"] += int((mine & keep).sum())
                    stats["ambiguous"] += int((mine & amb).sum())
                    stats["accepted"] += int((mine & (after[1] < before[1])).sum())
                    check_launch(before, after, colour)
                else:
                    stats["refined"] += check_launch(before, after, colour, f, sc, pp.refine_site(fused, color))
                if len(ctxs) > 1:
                    ctxs[1].phase(colour, mask)
            for other in ctxs[2:]:
                other.phase(colour, 7)
            ref_p, ref_c = A.get_state()
            for i, other in enumerate(ctxs[1:], start=1):
                p, c = other.get_state()
                assert bits_equal(p, ref_p) == 0 and bits_equal(c, ref_c) == 0, (case, "context %d" % i, colour)
    assert stats["accepted"] > 0 and stats["refined"] > 0
    share = stats["ambiguous"] / max(1, stats["compared"] + stats["ambiguous"])
    assert share <= 0.005, share
    return dict(stats, ambiguous_share=share)


@pytest.mark.parametrize("case", list(CASES))
def test_sweep_decisions_exact_at_any_size(case):
    from oracle.pyoracle import Oracle
    t0 = time.perf_counter()
    sc = make_scene(case)
    nwarps = CASES[case][8]
    seed = 4000 + sc.rows + sc.cols
    ctxs = [open_context(case, sc, seed),
            open_context(case, sc, seed),
            open_context(case, sc, seed),
            open_context(case, sc, seed, {"memo": 0, "prune": 0, "dedupe": 0, "quadperm": 0, "nwarps": 3 if nwarps != 3 else 7})]
    try:
        for ctx in ctxs:
            ctx.init()
        n0, c0 = ctxs[0].get_state()
        for ctx in ctxs[1:]:
            n, c = ctx.get_state()
            assert bits_equal(n, n0) == 0 and bits_equal(c, c0) == 0
        # 1. the cost function against the scalar oracle (which clamps the reference image and knows nothing of tiles)
        o = Oracle(sc)
        o.set_threads(8)
        ev = ctxs[0].cost_eval(n0)
        for y0, y1 in bands(sc.rows):
            assert_close_to_oracle(c0, o.cost_eval(n0, y0, y1, init_radius=True), y0, y1, "init cost")
            assert_close_to_oracle(ev, o.cost_eval(n0, y0, y1), y0, y1, "gpm_cost_eval")
        # 2-4. every decision of two iterations, the launch invariants, and the twin contexts
        REPORT[case] = decision_chain(case, sc, ctxs)
    finally:
        for ctx in ctxs:
            ctx.close()
    REPORT[case]["seconds"] = round(time.perf_counter() - t0, 2)
    print("\n%s: %s" % (case, REPORT[case]))


def adversarial_state(sc, planes, cost_fn, rng, fused, color):
    """Planes and costs that make every part of the acceptance rule decide some pixels:
    - 20 % random planes, strongly tilted, through a depth within 3 % of a range bound: out of range at some neighbours;
    - 10 % bit-equal copies of a neighbour's plane (set_state gives them different identities);
    - pairs of candidates with equal costs but different bits (+0.0 / -0.0 normal component) offered to one pixel whose
      cost is MAXCOST, so the candidate order decides which plane it takes;
    - 10 % of the costs set exactly to the cost of the close-up or far-up candidate: ties that must be rejected;
    - 6x6 patches of cost MAXCOST."""
    from oracle import pypropagate as pp
    cam, prm = sc.cameras[0], sc.params
    H, W = planes.shape[:2]
    pl = np.array(planes, dtype=np.float32, copy=True)
    ys, xs = np.mgrid[0:H, 0:W]
    wild = rng.random((H, W)) < 0.2
    n = rng.normal(size=(H, W, 3))
    n[..., 2] = -np.abs(n[..., 2]) - 0.15
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    bound = np.where(rng.random((H, W)) < 0.5, prm.depthMin * (1 + 0.03 * rng.random((H, W))),
                     prm.depthMax * (1 - 0.03 * rng.random((H, W))))
    t = n[..., 0] * (xs - cam.K[0, 2]) + n[..., 1] * (ys - cam.K[1, 2]) * cam.alpha + n[..., 2] * cam.fx
    pl[wild] = np.concatenate([n, (-bound * t / cam.fx)[..., None]], axis=-1)[wild].astype(np.float32)
    copy = rng.random((H, W)) < 0.1
    for (dy, dx) in [(-1, 0), (0, 1), (5, 0), (0, -5)]:
        part = copy & (rng.random((H, W)) < 0.25) & (ys + dy >= 0) & (ys + dy < H) & (xs + dx >= 0) & (xs + dx < W)
        pl[part] = pl[(ys + dy)[part], (xs + dx)[part]]
    pair = np.zeros((H, W), bool)
    pick = rng.random((H, W)) < 0.04
    pick[:5] = False
    pick &= ~np.roll(pick, 1, axis=0) & ~np.roll(pick, 4, axis=0) & ~np.roll(pick, -4, axis=0)
    for py, px in zip(*np.nonzero(pick)):
        up = pl[py - 1, px].copy()
        up[0] = np.float32(0.0)
        pl[py - 1, px] = up
        up[0] = np.float32(-0.0)
        pl[py - 5, px] = up
        pair[py, px] = True
    cost = np.asarray(cost_fn(pl, pp.propagation_site(0, fused, color)), dtype=np.float32).copy()
    ties = [pp.candidates(H, W, 1, True)[0], pp.candidates(H, W, 1, True)[2]] if fused else \
           [pp.candidates(H, W, 1)[0], pp.candidates(H, W, 2)[0]]
    for k, dy, dx, ok in ties:
        tie = ok & (rng.random((H, W)) < 0.05)
        c = np.asarray(cost_fn(pp.shifted(pl, dy, dx, ok), pp.propagation_site(k, fused, color)))
        cost[tie] = c[tie]
    for _ in range(max(1, H * W // 600)):
        y0, x0 = int(rng.integers(0, H)), int(rng.integers(0, W))
        cost[y0:y0 + 6, x0:x0 + 6] = MAXCOST
    cost[pair] = MAXCOST
    return pl, cost


@pytest.mark.parametrize("case", ["grey_53x75", "fused_grey_53x75"])
def test_sweep_decisions_exact_on_adversarial_states(case):
    t0 = time.perf_counter()
    sc = make_scene(case)
    fused, color = CASES[case][5], CASES[case][4]
    ctxs = [open_context(case, sc, 77), open_context(case, sc, 77), open_context(case, sc, 77)]
    try:
        ctxs[0].init()
        n0, _ = ctxs[0].get_state()
        pl, cost = adversarial_state(sc, n0, cost_of(ctxs[0]), np.random.default_rng(5), fused, color)
        for ctx in ctxs:
            ctx.set_state(pl, cost)
        REPORT["adversarial_" + case] = decision_chain(case, sc, ctxs)
    finally:
        for ctx in ctxs:
            ctx.close()
    REPORT["adversarial_" + case]["seconds"] = round(time.perf_counter() - t0, 2)
    print("\nadversarial %s: %s" % (case, REPORT["adversarial_" + case]))
