"""Adaptive checkerboard sampling (DESIGN.md §16) without a GPU: the region table's properties, the choice's known answers
on hand-made cost maps, the restatement against the fixed mode's where the two must agree, the gpm_job_opts layout, and the
refusals of the drivers and the Python entry points, all before any CUDA call."""
import ctypes as C

import numpy as np
import pytest

from test_geo_batch_args import _desc

E_ARG = -1
f32 = np.float32


def test_region_table_properties():
    from oracle import pyacs, pypropagate as pp
    R = pyacs.REGIONS
    assert [len(r) for r in R] == [7] * 4 + [11] * 4
    every = [o for r in R for o in r]
    assert len(set(every)) == len(every)                                  # no two regions share an offset
    assert all((abs(dy) + abs(dx)) & 1 for dy, dx in every)               # every offset lands on the other colour
    for k in range(4):                                                    # the fixed neighbours, first in scan order
        assert R[k][0] == pp.CLOSE[k] and pp.FAR[k] in R[4 + k]
    assert R[1] == [(-dy, dx) for dy, dx in R[0]] and R[5] == [(-dy, dx) for dy, dx in R[4]]
    assert R[2] == [(dx, dy) for dy, dx in R[0]] and R[6] == [(dx, dy) for dy, dx in R[4]]
    assert R[3] == [(dy, -dx) for dy, dx in R[2]] and R[7] == [(dy, -dx) for dy, dx in R[6]]
    assert R[0] == [(-1, 0), (-2, -1), (-2, 1), (-3, -2), (-3, 2), (-4, -3), (-4, 3)]
    assert R[2] == [(0, -1), (-1, -2), (1, -2), (-2, -3), (2, -3), (-3, -4), (3, -4)]
    assert R[4] == [(-a, 0) for a in range(3, 24, 2)]


def _choice(cost, k, y, x, mask=3):
    from oracle import pyacs
    H, W = cost.shape
    for kk, sy, sx, ok in pyacs.choose(cost, H, W, mask):
        if kk == k:
            return (int(sy[y, x]), int(sx[y, x])) if ok[y, x] else None
    return None


def test_choice_ties_go_to_the_earliest_offset():
    cost = np.full((30, 30), f32(5.0))
    y, x = 15, 15
    assert _choice(cost, 0, y, x) == (14, 15)                             # all equal: the 1 px neighbour
    assert _choice(cost, 4, y, x) == (12, 15)                             # far: the 3 px one
    cost[13, 14] = cost[13, 16] = f32(1.0)                                # (-2, -1) and (-2, +1) tie
    assert _choice(cost, 0, y, x) == (13, 14)
    cost[15, 10] = cost[15, 4] = f32(0.25)                                # far left: 5 px and 11 px tie
    assert _choice(cost, 6, y, x) == (15, 10)
    cost[15, 4] = f32(0.125)                                              # strictly cheaper later: it wins
    assert _choice(cost, 6, y, x) == (15, 4)
    cost[15, 12] = f32(-0.0)                                              # -0 ties with +0 below: the earlier one
    cost[15, 8] = f32(0.0)
    assert _choice(cost, 6, y, x) == (15, 12)


def test_choice_nan_never_beats_a_number():
    cost = np.full((30, 30), np.nan, f32)
    y, x = 15, 15
    assert _choice(cost, 1, y, x) == (16, 15)                             # all NaN: the earliest offset
    cost[19, 12] = f32(999.0)                                             # the last offset of near down, a number
    assert _choice(cost, 1, y, x) == (19, 12)
    cost[16, 15] = np.inf                                                 # +inf ties with NaN, loses to the number
    assert _choice(cost, 1, y, x) == (19, 12)
    cost = np.full((30, 30), np.inf, f32)
    cost[18, 13] = np.nan                                                 # +inf first, NaN later: the tie keeps +inf
    assert _choice(cost, 1, y, x) == (16, 15)


def test_choice_partly_off_image_picks_among_the_pixels_inside():
    cost = np.full((12, 40), f32(9.0))
    cost[0, 6] = f32(3.0)                                                 # (-2, -1) from (2, 7): inside
    assert _choice(cost, 0, 2, 7) == (0, 6)                               # rows -1 and -2 are off the image
    cost[1, 7] = f32(-1.0)
    assert _choice(cost, 0, 2, 7) == (1, 7)
    # far up from row 4: only the 3 px offset is inside
    assert _choice(cost, 4, 4, 7) == (1, 7)
    # a pixel in column 0: near left's (±1, -2), (±2, -3) ... are all off, (0, -1) too
    assert _choice(cost, 2, 5, 0) is None
    # column 1: only (0, -1) is inside
    assert _choice(cost, 2, 5, 1) == (5, 0)


def test_choice_fully_off_image_is_not_offered_and_phase_bits_select():
    from oracle import pyacs
    cost = np.zeros((8, 8), f32)
    got = {k: ok for k, _, _, ok in pyacs.choose(cost, 8, 8, 3)}
    assert not got[0][0].any() and got[0][1:].all()                       # near up: row 0 has nothing above it
    assert not got[4][:3].any() and got[4][3:].all()                      # far up: rows 0-2 have nothing 3 px above
    assert not got[7][:, 5:].any() and got[7][:, :5].all()
    assert [k for k, *_ in pyacs.choose(cost, 8, 8, 1)] == [0, 1, 2, 3]
    assert [k for k, *_ in pyacs.choose(cost, 8, 8, 2)] == [4, 5, 6, 7]
    assert pyacs.choose(cost, 8, 8, 4) == []


def _toy_cost_of(planes, site):
    """A pure cost of a plane at a pixel, with the site folded in."""
    p = planes.astype(np.float64)
    return (np.abs(p[..., 0] * 3.1 + p[..., 1] * 1.7 - p[..., 2]) * 10.0 + (p[..., 3] % 7.0) + 0.01 * site).astype(f32)


def _toy_state(H, W, rng):
    from types import SimpleNamespace
    n = rng.normal(size=(H, W, 3))
    n[..., 2] = -np.abs(n[..., 2]) - 1.0
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    cam = SimpleNamespace(fx=f32(500.0), alpha=f32(1.0), K=np.array([[500, 0, W / 2], [0, 500, H / 2], [0, 0, 1]], f32))
    ys, xs = np.mgrid[0:H, 0:W]
    depth = rng.uniform(400.0, 700.0, size=(H, W))
    t = n[..., 0] * (xs - W / 2) + n[..., 1] * (ys - H / 2) + n[..., 2] * 500.0
    planes = np.concatenate([n, (-depth * t / 500.0)[..., None]], axis=-1).astype(f32)
    return planes, cam


@pytest.mark.parametrize("H,W", [(23, 37), (48, 48), (9, 60)])
@pytest.mark.parametrize("colour", [0, 1])
@pytest.mark.parametrize("mask", [1, 2, 3])
def test_adaptive_equals_fixed_where_each_fixed_neighbour_is_strictly_cheapest(H, W, colour, mask):
    """Where each fixed neighbour is strictly the cheapest pixel of its region, the adaptive restatement equals the fixed one
    bit for bit.  Random costs in [1, 2) with the fixed neighbours of a lattice of pixels (48 px apart, so that their
    regions do not overlap) lowered to 0.5; the comparison covers every pixel whose regions all pick the fixed neighbour
    (or where neither mode offers direction k), the lattice among them."""
    from oracle import pyacs, pypropagate as pp
    rng = np.random.default_rng(H * W + colour)
    planes, cam = _toy_state(H, W, rng)
    ys, xs = np.mgrid[0:H, 0:W]
    mine = ((xs + ys) & 1) == colour
    cost = rng.uniform(1.0, 2.0, size=(H, W)).astype(f32)
    lattice = mine & (ys % 48 == min(H - 1, 7)) & (xs % 48 // 2 == 12)
    assert lattice.any()
    for y, x in zip(*np.nonzero(lattice)):
        for dy, dx in pp.CLOSE + pp.FAR:
            if 0 <= y + dy < H and 0 <= x + dx < W:
                cost[y + dy, x + dx] = f32(0.5)
    fixed = {k: ok for k, _, _, ok in pp.candidates(H, W, mask)}
    agree = mine.copy()
    for k, sy, sx, ok in pyacs.choose(cost, H, W, mask):
        dy, dx = (pp.CLOSE + pp.FAR)[k]
        agree &= (fixed[k] & (sy == ys + dy) & (sx == xs + dx)) | (~fixed[k] & ~ok)
    assert agree[lattice & (ys >= 5) & (ys < H - 5) & (xs >= 5) & (xs < W - 5)].all()
    assert agree.sum() >= lattice.sum()
    want = pp.expected(planes, cost, colour, mask, _toy_cost_of, cam, 450.0, 650.0)
    got = pyacs.expected(planes, cost, colour, mask, _toy_cost_of, cam, 450.0, 650.0, adaptive=True)
    assert (got[0][agree].view(np.uint32) == want[0][agree].view(np.uint32)).all()
    assert (got[1][agree].view(np.uint32) == want[1][agree].view(np.uint32)).all()
    assert (got[2][agree] == want[2][agree]).all()
    assert got[1][~mine].tobytes() == cost[~mine].tobytes()
    assert pyacs.expected(planes, cost, colour, mask, _toy_cost_of, cam, 450.0, 650.0, adaptive=False)[1].tobytes() == \
        want[1].tobytes()


def test_job_opts_layout_matches_the_header():
    from gipuma_b200 import api
    assert C.sizeof(api.GpmJobOpts) == 12
    assert [getattr(api.GpmJobOpts, n).offset for n in ("photometric", "ncc_min_std", "propagation")] == [0, 4, 8]
    o = api.job_opts("ncc", 3.0, "adaptive")
    assert (o.photometric, o.ncc_min_std, o.propagation) == (1, 3.0, 1)
    o = api.job_opts("pm", float("nan"))
    assert (o.photometric, o.ncc_min_std, o.propagation) == (0, 0.0, 0)
    assert api.PROPAGATION == {"fixed": 0, "adaptive": 1}


@pytest.mark.parametrize("opts,msg", [((0, 0.0, 2), "propagation"), ((0, 0.0, -1), "propagation"), ((2, 1.0, 0), "kind"),
                                      ((1, 0.0, 1), "min_std"), (None, "opts")])
def test_opts_drivers_refuse_bad_arguments_without_a_device(opts, msg):
    from gipuma_b200 import api
    lib = api.load_library()
    g, _keep = _desc()
    o = C.byref(api.GpmJobOpts(*opts)) if opts else None
    rc = lib.gpm_geo_batch_run_opts(C.byref(g), o, None)
    err = lib.gpm_batch_last_error().decode()
    assert rc == E_ARG and err.startswith("gpm_geo_batch_run_opts: bad arguments") and msg in err, (rc, err)
    rc = lib.gpm_batch_run_opts(C.byref(g.batch), o, None)
    err = lib.gpm_batch_last_error().decode()
    assert rc == E_ARG and err.startswith("gpm_batch_run_opts: bad arguments") and msg in err, (rc, err)


def test_opts_drivers_refuse_ncc_on_colour_and_bad_descriptors_without_a_device():
    from gipuma_b200 import api
    lib = api.load_library()
    g, _keep = _desc(channels=4)
    assert lib.gpm_geo_batch_run_opts(C.byref(g), C.byref(api.GpmJobOpts(1, 2.0, 1)), None) == E_ARG
    assert "grey" in lib.gpm_batch_last_error().decode()
    assert lib.gpm_batch_run_opts(None, C.byref(api.GpmJobOpts(0, 0.0, 1)), None) == E_ARG
    assert lib.gpm_batch_last_error().decode() == "gpm_batch_run_opts: bad arguments"
    assert lib.gpm_geo_batch_run_opts(None, C.byref(api.GpmJobOpts(0, 0.0, 1)), None) == E_ARG


def test_set_propagation_refuses_a_null_context_without_a_device():
    from gipuma_b200 import api
    lib = api.load_library()
    assert lib.gpm_set_propagation(None, 1) == E_ARG


@pytest.mark.parametrize("kw", [dict(propagation="acmh"), dict(propagation=1), dict(propagation=None),
                                dict(propagation="adaptive", photometric="census")])
@pytest.mark.parametrize("entry", ["batch_run", "geometric_pass"])
def test_api_refuses_bad_propagation_before_loading_the_library(monkeypatch, kw, entry):
    from gipuma_b200 import api, scene as S

    def no_library():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(api, "load_library", no_library)
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1)
    with pytest.raises(ValueError):
        getattr(api, entry)(np.zeros((3, 16, 16), np.float32), [np.eye(3, 4)] * 3, params, [0], **kw)


def test_shard_runner_refuses_bad_propagation_before_creating_a_context(monkeypatch):
    from types import SimpleNamespace
    from gipuma_b200 import api, multigpu
    monkeypatch.setattr(api, "Context", lambda *a, **k: (_ for _ in ()).throw(AssertionError("a context was created")))
    sc = SimpleNamespace(n_views=4, cols=16, rows=16)
    with pytest.raises(ValueError, match="propagation"):
        multigpu.ViewShardRunner(sc, 0, 1, propagation="acmh")
    with pytest.raises(ValueError, match="propagation"):
        multigpu.run_hybrid(lambda r: sc, 1, 0, 1, 1, propagation="ACMH")
