"""Every sweep mode the mode rule admits, launch by launch, against the restated decision rules.

A mode is a choice of colour images, the fused sweep, the geometric term, the NCC cost, adaptive propagation, joint view
selection (JVS), the planar prior, the geometric term's mask and ACMH's refinement (mode_conflict() in gpm_kernels.cuh).
Each admitted combination is its own k_sweep instantiation, with its own scratch layout, so each is checked here:

- the rule, restated: 66 sweep modes (34 with Gipuma's refinement, 32 with ACMH's) and 13 k_cost_eval modes; over all 512
  bit patterns the setters accept exactly the admitted ones and refuse every other with GPM_E_ARG (GPM_E_STATE for a
  colour upload while the NCC cost is on), leaving state and launch count unchanged; gpm_shard_num_stages accepts exactly
  the modes shard_supports() passes once the fused sweep, which only a shard launch refuses, is set aside;
- every admitted mode at three shapes (ragged tiles, a window larger than the image, 64 views with the largest scratch):
  init, one sweep, then per colour separate close, far and refinement launches, each against the restatement of its
  mode: oracle/pypropagate.py or oracle/pyacs.py for propagation, oracle/pyjvs.py under JVS, oracle/pyrefine.py for ACMH's
  refinement (with or without JVS), and the launch invariants for Gipuma's refinement, which has no exact restatement under
  the reference RNG.  A twin without memo, prune or dedupe at 2 warps per block stays bit-identical after every launch,
  and one running a single mask-7 launch per colour at 3 warps equals the chain (the automatic count is at least 2, so
  one of them or both run at another count than the checked context).  Under JVS, where a launch's weights depend on the
  candidates it is offered, the mask-7 twin is checked against the restatement of its own launch;
- a seeded walk of single-setter toggles across the modes on one context, each admitted mode checked launch by launch
  and each refused toggle changing nothing.

The parametrisation comes from the restated rule, and a test checks it covers every admitted mode at every shape."""
import time

import numpy as np
import pytest

from conftest import bits_equal

f32 = np.float32
E_ARG, E_STATE = -1, -3
BITS = ("color", "fused", "geo", "ncc", "adaptive", "jvs", "prior", "geomask", "refine_acmh")
COLOR, FUSED, GEO, NCC, ADAPTIVE, JVS, PRIOR, GEOMASK, ACMH = (1 << i for i in range(9))
WEIGHT, MAX_ERR, MIN_STD, EPS, SEED = 0.3, 6.0, 4.0, 0.02, 31
EXACT = {"beta": 1e30}                   # every JVS confidence exactly 1 (test_gpu_view_selection.EXACT)

# id: (rows, cols, views, box, most ambiguous pixels a mode may leave unchecked: 0.5 % of its compared pixels, the bound of
# test_gpu_sweep_any_size, or a count).  A pixel is ambiguous where an offered plane's depth lies within
# pypropagate.DEPTH_BAND of a range bound, and both refinements clamp depths to the bounds exactly.  An 8 x 8 image has
# 32 pixels per colour, so one such pixel is already 0.5 % of a mode's 192 compared pixels; up to 17 were measured
# (geo + prior with Gipuma's refinement), and the bound there is 20 of 192.
SHAPES = {
    "53x75_v4_box9": (53, 75, 4, 9, 0.005),      # ragged partial tiles
    "8x8_v2_box25": (8, 8, 2, 25, 20),           # the window is larger than the image
    "40x60_v64_box25": (40, 60, 64, 25, 0.005),  # the largest scratch: 64 views, box 25 (test_gpu_view_selection's rig)
}


def ambiguous_bound(shape, total):
    b = SHAPES[shape][4]
    return b * total if isinstance(b, float) else b


# ---- the mode rule, restated ------------------------------------------------------------------------------------------

def conflict(b: int):
    """mode_conflict() of gpm_kernels.cuh: the first conflict's name, None for an admitted mode."""
    on = lambda f: bool(b & f)
    if on(FUSED) and (on(GEO) or on(NCC) or on(ADAPTIVE) or on(JVS) or on(PRIOR)):
        return "fused"
    if on(JVS) and (not on(NCC) or on(COLOR)):
        return "jvs_needs_ncc_grey"
    if on(NCC) and on(COLOR):
        return "ncc_colour"
    if on(PRIOR) and (on(COLOR) or on(JVS)):
        return "prior"
    if on(GEOMASK) and (not on(GEO) or on(PRIOR)):
        return "geomask"
    if on(ACMH) and on(FUSED):
        return "refine_fused"
    return None


def shard_supports(b: int) -> bool:
    """shard_supports(): the plain 8-neighbour PM sweep with Gipuma's refinement, grey or colour, fixed or adaptive."""
    return conflict(b) is None and not b & (GEO | NCC | JVS | PRIOR | FUSED | ACMH)


def mode_name(b: int) -> str:
    return "+".join(n for i, n in enumerate(BITS) if b >> i & 1) or "pm_grey"


ADMITTED = [b for b in range(512) if conflict(b) is None]
MATRIX = [(shape, b) for shape in SHAPES for b in ADMITTED]        # the parametrisation of the sweep test
EVAL_MODES = sorted({b & (COLOR | GEO | NCC | PRIOR | GEOMASK) for b in ADMITTED})   # what k_cost_eval reads


def test_the_rule_admits_66_sweep_and_13_cost_eval_modes():
    assert len(ADMITTED) == 66
    assert sum(1 for b in ADMITTED if not b & ACMH) == 34 and sum(1 for b in ADMITTED if b & ACMH) == 32
    assert len(EVAL_MODES) == 13
    assert len({b & 255 for b in ADMITTED}) == 34          # the k_cost_eval / k_shard_stage tables' index space
    assert sorted(b for b in ADMITTED if shard_supports(b)) == [0, COLOR, ADAPTIVE, COLOR | ADAPTIVE]


# ---- scenes and contexts ----------------------------------------------------------------------------------------------

_SCENES = {}


def scene(shape, colour=False):
    key = (shape, bool(colour))
    if key not in _SCENES:
        from test_gpu_geometric import depth_maps, make_scene
        rows, cols, views, box = SHAPES[shape][:4]
        sc = make_scene(rows, cols, views, box, bool(colour))
        _SCENES[key] = (sc, depth_maps(sc, 3), (np.random.default_rng(4).random((rows, cols)) < 0.5).astype(np.uint8))
    return _SCENES[key]


def open_mode(shape, b, options=None):
    """A context over the shape's scene in mode b, its setters in the order of the mode's bits."""
    from gipuma_b200 import api
    sc, depths, gmask = scene(shape, b & COLOR)
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    opts = dict({"neighbours": 20} if b & FUSED else {}, **(options or {}))
    for k, v in opts.items():
        ctx.set_option(k, v)
    if b & NCC:
        ctx.set_photometric("ncc", MIN_STD)
    ctx.load_scene(sc, seed=SEED)
    if b & GEO:
        for v, d in enumerate(depths):
            ctx.set_view_depth(v, d)
        ctx.set_geometric(WEIGHT, MAX_ERR)
    if b & GEOMASK:
        ctx.set_geo_mask(gmask)
    if b & ADAPTIVE:
        ctx.set_propagation("adaptive")
    if b & JVS:
        ctx.set_view_selection("joint", **EXACT)
    if b & ACMH:
        ctx.set_refinement("acmh", EPS)
    return ctx


def start(ctx, sc, b):
    """init and one sweep; with the prior, the prior built from that state and turned on (test_gpu_refine_acmh.start).
    Returns (t, r): JVS's iteration count and the refinement counter of the next launch."""
    ctx.init()
    ctx.sweep(1)
    if b & PRIOR:
        ctx.build_planar_prior(5, float(np.nanpercentile(ctx.get_state()[1], 60)))
        ctx.set_prior(1.0, (sc.params.depthMax - sc.params.depthMin) / 64.0, 5.0)
        p, _ = ctx.get_state()
        ctx.set_state(p, ctx.cost_eval(p))              # gpm_set_state resets t, not r
        return 0, 2
    return 1, 2


class Rows:
    """Per-view rows (m, c) [H, W, V] of a plane map from one-view NCC contexts: c = m + g with the geometric term, m at
    the pixels its mask marks.  Shared by every JVS mode of a shape."""

    def __init__(self, shape):
        from test_gpu_geometric import open_ctx
        self.sc, self.depths, self.gmask = scene(shape)
        n = self.sc.n_views
        self.m = [open_ctx(self.sc, views=[v]) for v in range(n)]
        self.g = [open_ctx(self.sc, depths=self.depths, weight=WEIGHT, views=[v]) for v in range(n)]
        for ctx in self.m + self.g:
            ctx.set_photometric("ncc", MIN_STD)

    def of(self, b):
        def rows(planes):
            m = np.stack([ctx.cost_eval(planes) for ctx in self.m], axis=-1)
            if not b & GEO:
                return m, m
            c = np.stack([ctx.cost_eval(planes) for ctx in self.g], axis=-1)
            if b & GEOMASK:
                c = np.where(self.gmask[..., None] != 0, m, c).astype(f32)
            return m, c
        return rows

    def close(self):
        for ctx in self.m + self.g:
            ctx.close()


_ROWS = {}


@pytest.fixture(scope="module", autouse=True)
def _close_rows():
    yield
    for r in _ROWS.values():
        r.close()
    _ROWS.clear()


def rows_for(shape):
    if shape not in _ROWS:
        _ROWS[shape] = Rows(shape)
    return _ROWS[shape]


def state(ctx, b):
    p, c = ctx.get_state()
    return (p, c, ctx.view_masks()) if b & JVS else (p, c)


def same_state(a, b):
    return all(np.array_equal(np.ascontiguousarray(x).view(np.uint8), np.ascontiguousarray(y).view(np.uint8)) for x, y in zip(a, b))


# ---- one launch against the restatement of its mode -------------------------------------------------------------------

def check_launch(ctx, sc, b, colour, mask, t, r, rows=None):
    """Runs ctx.phase(colour, mask) and checks it against the restatement of mode b.  Returns the counts of this colour's
    pixels (compared, ambiguous, accepted, refined)."""
    from gipuma_b200 import api
    from oracle import pyacs, pyjvs, pypropagate as pp, pyrefine
    from test_gpu_sweep_any_size import check_launch as invariants, cost_of
    cam, prm = sc.cameras[0], sc.params
    H, W = sc.rows, sc.cols
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    color, fused, adaptive = bool(b & COLOR), bool(b & FUSED), bool(b & ADAPTIVE)
    f = cost_of(ctx)
    before = state(ctx, b)
    p0, c0 = before[0], before[1]
    refine_args = (api.pack_camera(cam), prm.min_disparity, prm.max_disparity, prm.depthMin, prm.depthMax, EPS, SEED, r)
    exact = not (mask & 4) or b & ACMH
    refined = np.zeros((H, W), bool)
    if b & JVS:
        rows_of = rows.of(b)
        det = {}
        if not (mask & 4 and b & ACMH):
            want_p, want_c, want_m, amb = pyjvs.expected(p0, c0, before[2], colour, mask & 3, rows_of, ctx.cost_eval, cam,
                                                         prm.depthMin, prm.depthMax, EXACT, t, adaptive=adaptive, details=det)
        else:
            want_p, want_c, want_m, amb, refined = pyrefine.jvs_expected(p0, c0, before[2], colour, mask, rows_of, ctx.cost_eval,
                                                                         cam, *refine_args[:-1], r, EXACT, t, adaptive=adaptive)
    elif mask & 3:
        if adaptive:
            want_p, want_c, amb = pyacs.expected(p0, c0, colour, mask, f, cam, prm.depthMin, prm.depthMax, color_images=color)
        else:
            want_p, want_c, amb = pp.expected(p0, c0, colour, mask, f, cam, prm.depthMin, prm.depthMax, fused=fused,
                                              color_images=color)
    else:
        want_p, want_c, amb = p0, c0, np.zeros((H, W), bool)
    if not b & JVS and mask & 4 and b & ACMH:               # ACMH's refinement after the propagation (mask 7 twins)
        cand = pyrefine.candidates(want_p, *refine_args)
        costs = [f(np.ascontiguousarray(cand[j]), 0) for j in range(len(cand))]
        want_p, want_c, refined = pyrefine.accept(want_p, want_c, cand, costs, mine)
    ctx.phase(colour, mask)
    got = state(ctx, b)
    keep = ~amb
    if b & JVS:
        assert np.array_equal(got[2][keep], want_m[keep]), ("view masks", mode_name(b), colour, mask)
        assert np.array_equal(got[2][~mine], before[2][~mine])
    if exact:
        bad = (got[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) | (got[1].view(np.uint32) != want_c.view(np.uint32))
        bad &= keep
        assert not bad.any(), (mode_name(b), colour, mask, int(bad.sum()), np.argwhere(bad)[:8].tolist())
    changed = (got[0].view(np.uint32) != p0.view(np.uint32)).any(axis=-1)
    if mask & 4 and not b & ACMH:                            # Gipuma's refinement: the launch invariants
        if b & JVS:                                          # every cost is its plane's cost under the launch's weights
            assert bits_equal(got[0][~mine], p0[~mine]) == 0 and bits_equal(got[1][~mine], c0[~mine]) == 0
            _, c = rows.of(b)(got[0])
            rescored = pyjvs.weighted(det["w"], c, ctx.cost_eval(got[0]))
            assert bits_equal(got[1][mine & keep], rescored[mine & keep]) == 0, (mode_name(b), colour, mask)
            assert np.all(got[1][mine & keep] <= want_c[mine & keep])
            n = got[0][changed & mine][:, :3].astype(np.float64)
            assert np.all(np.abs(np.linalg.norm(n, axis=-1) - 1.0) <= 1e-5)
            refined = mine & keep & (got[1] < want_c)
        else:
            assert not mask & 3                              # the chain's refinement launches run alone
            invariants((p0, c0), (got[0], got[1]), colour, f, sc, pp.refine_site(fused, color))
            refined = changed & mine
    elif not b & JVS:
        invariants((p0, c0), (got[0], got[1]), colour)
    accepted = mine & keep & changed if mask == 1 or mask == 2 else np.zeros((H, W), bool)
    return int((mine & keep).sum()), int((mine & amb).sum()), int(accepted.sum()), int((refined & mine).sum())


# ---- every admitted mode at every shape -------------------------------------------------------------------------------

def test_the_matrix_is_every_admitted_mode_at_every_shape():
    """The sweep test's parameters, checked when they are generated: every admitted mode at every shape, each once."""
    assert len(MATRIX) == 66 * 3 and len(set(MATRIX)) == len(MATRIX)
    for shape in SHAPES:
        assert {b for s, b in MATRIX if s == shape} == {b for b in range(512) if conflict(b) is None}
    ids = ["%s-%s" % (s, mode_name(b)) for s, b in MATRIX]
    assert len(set(ids)) == len(ids)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,b", MATRIX, ids=["%s-%s" % (s, mode_name(b)) for s, b in MATRIX])
def test_mode_launches_equal_the_restatement(shape, b):
    t0 = time.perf_counter()
    sc = scene(shape, b & COLOR)[0]
    rows = rows_for(shape) if b & JVS else None
    A = open_mode(shape, b)
    # the automatic warp count is at least 2 (build_kparams): at 2 and 3 warps, one twin or both run at another count
    twin = open_mode(shape, b, {"memo": 0, "prune": 0, "dedupe": 0, "nwarps": 2})
    seven = open_mode(shape, b, {"nwarps": 3})
    ctxs = (A, twin, seven)
    st = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}
    try:
        t, r = [start(c, sc, b) for c in ctxs][0]
        assert same_state(state(twin, b), state(A, b)) and same_state(state(seven, b), state(A, b))
        for colour in (0, 1):
            for mask in (1, 2, 4):
                n, a, acc, ref = check_launch(A, sc, b, colour, mask, t, r, rows)
                st["compared"] += n
                st["ambiguous"] += a
                st["accepted"] += acc
                st["refined"] += ref
                twin.phase(colour, mask)
                assert same_state(state(twin, b), state(A, b)), ("twin", mode_name(b), colour, mask)
                r += mask == 4
            if b & JVS:                                   # one launch's weights see all 8 candidates: its own restatement
                check_launch(seven, sc, b, colour, 7, t, r - 1, rows)
            else:
                seven.phase(colour, 7)
                assert same_state(state(seven, b), state(A, b)), ("mask 7", mode_name(b), colour)
    finally:
        for c in ctxs:
            c.close()
    share = st["ambiguous"] / max(1, st["compared"] + st["ambiguous"])
    report = dict(st, ambiguous_share=round(share, 5), seconds=round(time.perf_counter() - t0, 2))
    print("\n%-16s %-40s %s" % (shape, mode_name(b), report))
    assert st["accepted"] > 0, (shape, mode_name(b), st)
    assert st["refined"] > 0 or not b & ACMH, (shape, mode_name(b), st)
    assert st["ambiguous"] <= ambiguous_bound(shape, st["compared"] + st["ambiguous"]), (shape, mode_name(b), st)


# ---- k_cost_eval in its 13 modes, against the composition of its terms -----------------------------------------------

_ONE_VIEW = {}


def one_view_rows(shape, colour, ncc, planes):
    """[V, H, W] photometric costs of `planes` against each source view alone (one-view contexts, as
    test_gpu_ncc.per_view_costs), the contexts kept for the module."""
    key = (shape, bool(colour), bool(ncc))
    if key not in _ONE_VIEW:
        from test_gpu_geometric import open_ctx
        sc = scene(shape, colour)[0]
        ctxs = [open_ctx(sc, views=[v]) for v in range(sc.n_views)]
        for ctx in ctxs:
            if ncc:
                ctx.set_photometric("ncc", MIN_STD)
        _ONE_VIEW[key] = ctxs
    return np.stack([ctx.cost_eval(planes) for ctx in _ONE_VIEW[key]])


@pytest.fixture(scope="module", autouse=True)
def _close_one_view():
    yield
    for ctxs in _ONE_VIEW.values():
        for ctx in ctxs:
            ctx.close()
    _ONE_VIEW.clear()


def check_photometric_rows(shape, sc, b, planes, photo, combined):
    """The photometric costs at every pixel against high-precision references: the combined PM cost against the scalar
    oracle within test_oracle.py's bound, the per-view NCC costs against the float64 restatement within test_gpu_ncc.TOL
    (where both windows' variances clear the floor by 1 %; at 64 views for views 0, 1, 32 and 63, which cover both lanes
    of the views' split)."""
    from oracle import pyncc
    from test_gpu_ncc import TOL
    H = sc.rows
    if not b & NCC:
        from oracle.pyoracle import Oracle
        from test_gpu_sweep_any_size import assert_close_to_oracle
        o = Oracle(sc)
        o.set_threads(8)
        assert_close_to_oracle(combined, o.cost_eval(planes, 0, H), 0, H, (shape, mode_name(b)))
        return
    views = list(range(sc.n_views)) if sc.n_views <= 8 else [0, 1, 32, sc.n_views - 1]
    p = sc.params
    w, r, t = pyncc.sample_views64(sc.images[0], [sc.images[sc.subset[v]] for v in views], sc.cameras[0],
                                   [sc.cameras[sc.subset[v]] for v in views], planes, p.box_hsize, p.gamma)
    want = pyncc.ncc_cost64(w, r, t, MIN_STD)
    mean = lambda x: ((w * x).sum(-1) / w.sum(-1))
    vr = mean((r - mean(r)[..., None]) ** 2)
    vt = mean((t - mean(t)[..., None]) ** 2)
    clear = (vr[None] > 1.01 * MIN_STD ** 2) & (vt > 1.01 * MIN_STD ** 2)
    err = np.abs(photo[views] - want)[clear]
    assert clear.mean() > 0.5 and err.max() <= TOL, (shape, float(clear.mean()), float(err.max()))


@pytest.mark.gpu
@pytest.mark.parametrize("b", EVAL_MODES, ids=[mode_name(b) for b in EVAL_MODES])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_cost_eval_equals_the_composition_of_its_terms(shape, b):
    """gpm_cost_eval in mode b equals, bit for bit, the composition of its terms in numpy: each view's photometric cost
    from a one-view context, plus pygeo.geo_cost's term with the geometric term, combined by pygeo.combine with the
    device's reciprocals (learned as test_gpu_geometric.learn_rcp does), the per-pixel select of pyrestore.masked_cost with
    the mask, and pyprior.with_prior's term with the prior.  Two plane maps: the state after one sweep, and its pixels
    permuted (planes that do not fit the scene)."""
    from oracle import pygeo, pyprior, pyrestore
    from test_gpu_geometric import learn_rcp
    sc, depths, gmask = scene(shape, b & COLOR)
    prm, cam = sc.params, sc.cameras[0]
    base = b & (COLOR | NCC)                          # the photometric mode alone
    P = open_mode(shape, base)
    A = open_mode(shape, b & ~PRIOR)
    try:
        P.init()
        P.sweep(1)
        p1 = P.get_state()[0]
        perm = np.random.default_rng(SEED).permutation(p1.reshape(-1, 4)).reshape(p1.shape)
        sigma = (prm.depthMax - prm.depthMin) / 64.0
        prior_map = None
        if b & PRIOR:
            A.set_state(p1, P.get_state()[1])
            A.build_planar_prior(5, float(np.nanpercentile(P.get_state()[1], 60)))
            A.set_prior(1.0, sigma, 5.0)
            prior_map = A.planar_prior()
            assert (prior_map != 0).any()
        compared = 0
        for planes in (p1, np.ascontiguousarray(perm)):
            photo = one_view_rows(shape, b & COLOR, b & NCC, planes)
            combined = P.cost_eval(planes)
            s0, k0 = pygeo.combine_sum(photo, prm.cost_comb, prm.n_best, prm.good_factor)
            rcp = learn_rcp(k0, s0, combined)
            want = pygeo.combine(photo, prm.cost_comb, prm.n_best, prm.good_factor, rcp)
            assert bits_equal(want, combined) == 0, (shape, mode_name(b))
            if b & GEO:
                g = np.stack([pygeo.geo_cost(planes, cam, sc.cameras[sc.subset[v]], depths[v], WEIGHT, MAX_ERR, prm.depthMin,
                                             prm.depthMax) for v in range(sc.n_views)])
                on = pygeo.combine((photo + g).astype(f32), prm.cost_comb, prm.n_best, prm.good_factor, rcp)
                want = pyrestore.masked_cost(on, want, gmask) if b & GEOMASK else on
            if b & PRIOR:
                want = pyprior.with_prior(want, planes, prior_map, cam, prm.depthMin, prm.depthMax, 1.0, sigma, 5.0)
            got = A.cost_eval(planes)
            known = ~np.isnan(want)
            assert known.mean() > 0.98, known.mean()
            bad = (got.view(np.uint32) != want.view(np.uint32)) & known
            assert not bad.any(), (shape, mode_name(b), int(bad.sum()), np.argwhere(bad)[:5].tolist())
            if b & GEO:
                assert bits_equal(got, combined) > 0              # the term is on
            compared += int(known.sum())
            if not b & (GEO | PRIOR):
                check_photometric_rows(shape, sc, b, planes, photo, combined)
    finally:
        P.close()
        A.close()
    print("\ncost_eval %-16s %-28s %d pixels compared" % (shape, mode_name(b), compared))


# ---- the setters accept exactly the admitted modes --------------------------------------------------------------------

# A context's images are grey or colour from their first upload on ("a context holds either float or float4 images, not
# both"), so the colour bit is chosen by the upload that follows the options and the photometric cost, and each pattern
# gets a fresh context.  NCC before the upload: a colour upload then meets the NCC cost.
ORDER = (FUSED, NCC, COLOR, GEO, ADAPTIVE, JVS, PRIOR, GEOMASK, ACMH)


def effective(requested: int) -> int:
    """The mode in force for the requested bits: the mask is stored without the term, but only acts with it (ctx_mode)."""
    return requested if requested & GEO else requested & ~GEOMASK


def predicted_rc(requested: int, bit: int, on: bool) -> int:
    """What the setter of `bit` returns when switching it `on` from the requested bits: GPM_E_ARG for a mode the rule
    refuses, GPM_E_STATE for a colour upload while the NCC cost is on (refuse_change), GPM_E_ARG for the mask and the prior
    together even while the term is off (gpm_set_geo_mask, gpm_set_prior)."""
    new = requested | bit if on else requested & ~bit
    k = conflict(effective(new))
    if k is None:
        return E_ARG if new & PRIOR and new & GEOMASK else 0
    return E_STATE if bit == COLOR and on and k == "ncc_colour" else E_ARG


class Setters:
    """The C-ABI setter of each mode bit but the colour, on one context."""

    def __init__(self, ctx, shape):
        from gipuma_b200 import api
        self.api, self.ctx, self.lib, self.h, self.shape = api, ctx, ctx.lib, ctx.h, shape
        self.grey, self.depths, gmask = scene(shape)
        self.gmask = np.ascontiguousarray(gmask)
        self.sigma = (self.grey.params.depthMax - self.grey.params.depthMin) / 64.0

    def upload(self, colour: bool) -> int:
        """Parameters and the grey or colour images; then the random state, the depth maps and a prior map, so that
        only the rule decides the setters that follow.  Returns the first image upload's code."""
        import ctypes as C
        api, lib, h, ctx = self.api, self.lib, self.h, self.ctx
        sc = scene(self.shape, colour)[0]
        ctx.set_params(sc.params)
        img = np.ascontiguousarray(sc.images[0])
        rc = (lib.gpm_set_reference_color if colour else lib.gpm_set_reference)(h, C.c_void_p(img.ctypes.data), 0, 0,
                                                                                 C.byref(api.pack_camera(sc.cameras[0])))
        if rc:
            return rc
        for v, i in enumerate(sc.subset):
            ctx.set_view(v, sc.images[i], sc.cameras[i])
        ctx.set_num_views(len(sc.subset))
        ctx.set_rng(SEED)
        self.prepare()
        ctx.init()
        ctx.set_planar_prior(ctx.get_state()[0])
        return 0

    def prepare(self):
        for v, d in enumerate(self.depths):
            self.ctx.set_view_depth(v, d)

    def set(self, bit: int, on: bool) -> int:
        import ctypes as C
        api, lib, h = self.api, self.lib, self.h
        if bit == FUSED:
            return lib.gpm_set_option(h, b"neighbours", 20 if on else 8)
        if bit == GEO:
            return lib.gpm_set_geometric(h, WEIGHT if on else 0.0, MAX_ERR)
        if bit == NCC:
            return lib.gpm_set_photometric(h, api.check_photometric("ncc" if on else "pm", MIN_STD), MIN_STD if on else 0.0)
        if bit == ADAPTIVE:
            return lib.gpm_set_propagation(h, api.check_propagation("adaptive" if on else "fixed"))
        if bit == JVS:
            v = api.view_sel("joint", **EXACT) if on else api.view_sel("off")
            return lib.gpm_set_view_selection(h, C.byref(v))
        if bit == PRIOR:
            return lib.gpm_set_prior(h, 1.0 if on else 0.0, self.sigma, 5.0)
        if bit == GEOMASK:
            return lib.gpm_set_geo_mask(h, C.c_void_p(self.gmask.ctypes.data) if on else None, 0, 0)
        if bit == ACMH:
            k, e = api.check_refinement("acmh" if on else "gipuma", EPS)
            return lib.gpm_set_refinement(h, k, e)
        raise ValueError(bit)


def snapshot(ctx, initialised=True):
    p, c = ctx.get_state() if initialised else (np.zeros(0, f32), np.zeros(0, f32))
    return p, c, ctx.stats()["launches"]


def unchanged(ctx, snap, initialised=True):
    p, c, n = snapshot(ctx, initialised)
    return bits_equal(p, snap[0]) == 0 and bits_equal(c, snap[1]) == 0 and n == snap[2]


@pytest.mark.gpu
def test_setters_accept_exactly_the_admitted_modes():
    """Each of the 512 patterns on a fresh context, its setters in ORDER from the all-off mode: exactly the admitted modes
    are accepted, each launches, and gpm_shard_num_stages accepts exactly those shard_supports() passes but for the fused
    sweep, which only a shard launch refuses; every other
    pattern is refused by the setter the restated rule names, with the code it names, and the refusal changes neither
    state nor launch count."""
    from gipuma_b200 import api
    shape = "8x8_v2_box25"
    sc = scene(shape)[0]
    accepted, refused = set(), {E_ARG: 0, E_STATE: 0}
    for pattern in range(512):
        ctx = api.Context(sc.cols, sc.rows, sc.n_views)
        try:
            S = Setters(ctx, shape)
            requested, ready = 0, False
            for bit in ORDER:
                if bit != COLOR and not pattern & bit:
                    continue
                on = bool(pattern & bit)
                want = predicted_rc(requested, bit, on)
                snap = snapshot(ctx, ready)
                rc = S.upload(on) if bit == COLOR else S.set(bit, True)
                assert rc == want, (mode_name(pattern), mode_name(bit), rc, ctx.lib.gpm_last_error().decode())
                if rc:
                    assert unchanged(ctx, snap, ready), (mode_name(pattern), mode_name(bit))
                    refused[rc] += 1
                    break
                ready |= bit == COLOR
                requested |= bit if on else 0
            if requested == pattern:
                m = effective(pattern)
                assert conflict(m) is None
                accepted.add(m)
                n = ctx.stats()["launches"]
                ctx.phase(0, 3)                                   # the mode has a kernel
                assert ctx.stats()["launches"] == n + 1
                stages = ctx.lib.gpm_shard_num_stages(ctx.h)
                # the fused sweep is refused only where a shard stage launches (shard_common), with GPM_E_ARG
                assert (stages > 0) == shard_supports(m & ~FUSED), (mode_name(m), stages)
            else:
                assert conflict(effective(pattern)) is not None or pattern & PRIOR and pattern & GEOMASK
        finally:
            ctx.close()
    assert accepted == set(ADMITTED)
    assert refused[E_ARG] > 0 and refused[E_STATE] > 0
    print("\nsetters: %d admitted modes, refusals %s" % (len(accepted), refused))


# ---- switching modes mid-run ------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_mode_walk_checks_every_launch_of_the_mode_in_force():
    """About 40 single-setter toggles on one context: each refused toggle changes nothing, after each accepted one a
    close, a far and a refinement launch equal the restatement of the mode now in force.  Every fifth toggle switches the
    refinement, after Gipuma's refinement memo (GPM_MEMO_REFINE) has been set by rejected refinements.  The images, and so
    the colour bit, are fixed from a context's first upload: the walk is on grey images."""
    shape = "53x75_v4_box9"
    grey = scene(shape)[0]
    rows = rows_for(shape)
    ctx = open_mode(shape, 0)
    rng = np.random.default_rng(2024)
    walked, refusals, modes = 0, 0, set()
    try:
        S = Setters(ctx, shape)
        S.prepare()
        t, r = start(ctx, grey, 0)
        ctx.build_planar_prior(5, float(np.nanpercentile(ctx.get_state()[1], 60)))
        # two Gipuma refinement launches of one colour from the same state: the second skips the pixels whose refinement
        # the first rejected entirely (GPM_MEMO_REFINE), so the memo is set before the walk's first refinement switch
        skipped = []
        for _ in range(2):
            s0 = ctx.stats()["skipped"]
            check_launch(ctx, grey, 0, 0, 4, t, r, rows)
            r += 1
            skipped.append(ctx.stats()["skipped"] - s0)
        assert skipped[1] > 0, skipped
        requested = 0
        for step in range(40):
            bit = ACMH if step % 5 == 4 else int(rng.choice([o for o in ORDER if o != COLOR]))
            on = not requested & bit
            want = predicted_rc(requested, bit, on)
            snap = snapshot(ctx)
            rc = S.set(bit, on)
            assert rc == want, (step, mode_name(requested), mode_name(bit), on, rc, ctx.lib.gpm_last_error().decode())
            if rc:
                assert unchanged(ctx, snap), (step, mode_name(bit))
                refusals += 1
                continue
            requested = requested | bit if on else requested & ~bit
            b = effective(requested)
            modes.add(b)
            for mask in (1, 2, 4):
                check_launch(ctx, grey, b, step & 1, mask, t, r, rows)
                r += mask == 4
            walked += 1
    finally:
        ctx.close()
    print("\nwalk: %d toggles checked, %d refused, %d distinct modes" % (walked, refusals, len(modes)))
    assert walked >= 20 and refusals > 0 and any(m & ACMH for m in modes) and any(not m & ACMH for m in modes)
