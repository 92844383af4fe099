"""The sweep mode that costs propagated planes plane-major (grey images, PM cost, fixed 8-neighbour propagation; DESIGN.md
§4, shared propagation samples) checked launch by launch.

Every propagation launch must leave the state oracle/pypropagate.expected() restates — the acceptance rule folded over
gpm_cost_eval's costs of the neighbour-shifted plane maps — bit for bit outside the pixels whose depth-range test is
ambiguous, and twin contexts with the memo, the lower bound and the duplicate skips switched off one at a time (and all
together, at another warp count) must hold bit-identical states after every launch.  The sizes are ragged and small, so
that tiles are partial and gridDim.z splits tiles into slices; windows 3 to 25 and 1 to 64 source views cover one and two
lanes of views and one to eight views per chunk.  Without the memo and the duplicate skips a propagation launch evaluates
exactly the offered candidates whose depth is in range, so its hypothesis count is checked against that number too."""
import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

# id: (rows, cols, views, box)
CASES = {
    "v1_box3_37x45": (37, 45, 1, 3),
    "v2_box11_70x41": (70, 41, 2, 11),
    "v10_box15_97x130": (97, 130, 10, 15),
    "v10_box15_480x640": (480, 640, 10, 15),       # 300 tiles: gridDim.z = 4 on 132 SMs
    "v32_box25_45x66": (45, 66, 32, 25),
    "v33_box15_40x60": (40, 60, 33, 15),
    "v64_box11_35x50": (35, 50, 64, 11),
    "v10_box25_8x8": (8, 8, 10, 25),               # window larger than the image
}
TWINS = [{"memo": 0}, {"prune": 0}, {"dedupe": 0}, {"memo": 0, "prune": 0, "dedupe": 0, "nwarps": 5}]


def make_scene(case):
    from gipuma_b200 import scene as S
    rows, cols, views, box = CASES[case]
    cfg = 2 if views <= 10 else 4                  # the DTU rig up to 10 source views, the templeRing rig (any number) above
    sc = S.make_config(cfg, rows=rows, cols=cols, n_views=views, iterations=2, seed=rows * 1000 + cols + views)
    sc.params.box_hsize = sc.params.box_vsize = box
    return sc


def open_ctx(sc, seed, options=None):
    from gipuma_b200 import api
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    ctx.load_scene(sc, seed=seed)
    return ctx


def cost_of(ctx):
    def f(planes, site):
        ctx.set_option("cost_variant", site)
        try:
            return ctx.cost_eval(planes)
        finally:
            ctx.set_option("cost_variant", -1)
    return f


def in_range_count(planes, colour, mask, cam, lo, hi):
    """(sure, unsure): offered candidates of one propagation launch whose depth is in [lo, hi], and those whose range test
    pypropagate calls ambiguous."""
    from oracle import pypropagate as pp
    H, W = planes.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    lo, hi = float(np.float32(lo)), float(np.float32(hi))
    sure = unsure = 0
    for k, dy, dx, ok in pp.candidates(H, W, mask):
        offered = ok & mine
        depth, cond = pp.depth64(pp.shifted(planes, dy, dx, offered), cam)
        with np.errstate(invalid="ignore"):
            band = np.maximum(pp.DEPTH_BAND, 2.0 ** -20 * (cond + 1.0))
            near = (np.abs(depth - lo) <= band * abs(lo)) | (np.abs(depth - hi) <= band * abs(hi))
            inside = (depth >= lo) & (depth <= hi)
        sure += int((offered & inside & ~near).sum())
        unsure += int((offered & near).sum())
    return sure, unsure


def chain(sc, ctxs, iterations=2):
    """ctxs[0]: every propagation launch against the restatement; all contexts bit-identical after every launch.  The
    last twin runs without memo and duplicate skips: its propagation launches' hypothesis counts are checked."""
    from oracle import pypropagate as pp
    A, plain = ctxs[0], ctxs[-1]
    f = cost_of(A)
    cam, prm = sc.cameras[0], sc.params
    ys, xs = np.mgrid[0:sc.rows, 0:sc.cols]
    n = {"compared": 0, "ambiguous": 0, "accepted": 0}
    for _ in range(iterations):
        for colour in (0, 1):
            for mask in (1, 2, 4):
                before = A.get_state()
                if mask != 4:
                    want_p, want_c, amb = pp.expected(before[0], before[1], colour, mask, f, cam, prm.depthMin, prm.depthMax)
                    sure, unsure = in_range_count(before[0], colour, mask, cam, prm.depthMin, prm.depthMax)
                hyp0 = plain.stats()["hypotheses"]
                for ctx in ctxs:
                    ctx.phase(colour, mask)
                p, c = A.get_state()
                for i, ctx in enumerate(ctxs[1:], start=1):
                    p1, c1 = ctx.get_state()
                    assert bits_equal(p1, p) == 0 and bits_equal(c1, c) == 0, ("twin %d" % i, colour, mask)
                if mask == 4:
                    continue
                bad = ((p.view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) | (c.view(np.uint32) != want_c.view(np.uint32))) & ~amb
                assert not bad.any(), (colour, mask, int(bad.sum()), np.argwhere(bad)[:8].tolist())
                hyp = plain.stats()["hypotheses"] - hyp0
                assert sure <= hyp <= sure + unsure, (colour, mask, hyp, sure, unsure)
                mine = ((xs + ys) & 1) == colour
                n["compared"] += int((mine & ~amb).sum())
                n["ambiguous"] += int((mine & amb).sum())
                n["accepted"] += int((mine & (c < before[1])).sum())
    assert n["accepted"] > 0
    assert n["ambiguous"] <= 0.02 * (n["compared"] + n["ambiguous"])          # small images: a few pixels weigh more
    return n


def check_counters(sc, ctxs):
    ns = ((sc.params.box_hsize + 1) // 2) ** 2
    st = [ctx.stats() for ctx in ctxs]
    for s in st:
        assert s["pairs_full"] == s["hypotheses"] * sc.n_views * ns
    off = st[-1]
    assert off["pruned"] == 0 and off["pairs"] == off["pairs_full"]
    assert st[0]["pairs"] < off["pairs"]


@pytest.mark.parametrize("case", list(CASES))
def test_shared_samples_exact_every_launch(case):
    sc = make_scene(case)
    seed = 900 + sc.rows + sc.cols
    ctxs = [open_ctx(sc, seed)] + [open_ctx(sc, seed, o) for o in TWINS]
    try:
        for ctx in ctxs:
            ctx.init()
            ctx.reset_stats()
        n = chain(sc, ctxs)
        check_counters(sc, ctxs)
        print("\n%s: %s" % (case, n))
    finally:
        for ctx in ctxs:
            ctx.close()


def adversarial(sc, planes, cost_fn, rng):
    """The any-size suite's adversarial state (out-of-range tilted planes, bit-equal copies with other identities, equal
    costs with different bits, exact ties, MAXCOST patches), plus planes with a NaN distance or a NaN normal."""
    from test_gpu_sweep_any_size import adversarial_state
    pl, cost = adversarial_state(sc, planes, cost_fn, rng, False, False)
    H, W = cost.shape
    nan_d = rng.random((H, W)) < 0.03
    nan_n = (rng.random((H, W)) < 0.02) & ~nan_d
    pl[nan_d, 3] = np.float32(np.nan)
    pl[nan_n, 0] = np.float32(np.nan)
    return pl, cost


@pytest.mark.parametrize("case", ["v2_box11_70x41", "v10_box15_97x130", "v33_box15_40x60"])
def test_shared_samples_exact_on_adversarial_states(case):
    """One iteration builds memo entries, identities and provenance; gpm_set_state then installs the adversarial state
    (new identities: every remembered one is stale) and two more iterations are checked."""
    sc = make_scene(case)
    seed = 77 + sc.cols
    ctxs = [open_ctx(sc, seed)] + [open_ctx(sc, seed, o) for o in TWINS]
    try:
        for ctx in ctxs:
            ctx.init()
        chain(sc, ctxs, iterations=1)
        n1, _ = ctxs[0].get_state()
        pl, cost = adversarial(sc, n1, cost_of(ctxs[0]), np.random.default_rng(11))
        for ctx in ctxs:
            ctx.set_state(pl, cost)
            ctx.reset_stats()
        n = chain(sc, ctxs)
        check_counters(sc, ctxs)
        print("\nadversarial %s: %s" % (case, n))
    finally:
        for ctx in ctxs:
            ctx.close()
