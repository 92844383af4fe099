"""oracle/pypropagate.py — the acceptance rule of one propagation launch in numpy — against the oracle's own restatement
of the reference's kernels (gpo_phase), bit for bit.  Fed with the oracle's cost function, the numpy fold must reproduce
gpo_phase exactly outside the pixels whose range test is ambiguous, at image sizes that are not whole tiles, in the
close, far, close + far and fused 20-candidate launches, for grey and colour images.  The start states contain ties
(a pixel's cost equal to a candidate's), candidates with equal costs but different plane bits, planes far outside the
depth range and MAXCOST patches, so that the order of the candidates, the strict `<` and the guards all decide pixels.
The GPU's sweep is checked against this restatement in test_gpu_sweep_any_size.py."""
import numpy as np
import pytest

from conftest import bits_equal

MAXCOST = np.float32(1000.0)
SHAPES = [(53, 75), (31, 33), (8, 8), (29, 41)]          # rows x cols
MASKS = [1, 2, 3, 8]


def _scene(rows, cols, color):
    from gipuma_b200 import scene as S
    sc = S.make_config(2, rows=rows, cols=cols, n_views=3, iterations=1, seed=rows * 100 + cols)
    sc.params.box_hsize = sc.params.box_vsize = 7
    return S.colorize(sc) if color else sc


def adversarial_state(sc, planes, cost_of, rng):
    """Planes and costs that make every part of the acceptance rule decide some pixels (cost_of(planes, site) -> costs).
    - 20 % random planes, strongly tilted, through a depth within 3 % of a range bound: out of range at some neighbours;
    - 10 % bit-equal copies of a neighbour's plane;
    - pairs of candidates with equal costs but different bits (+0.0 / -0.0 normal component) offered to one pixel whose
      cost is MAXCOST, so the candidate order decides which plane it takes;
    - 10 % of the costs set exactly to the cost of the first close or far candidate: ties that must be rejected;
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
    d = -bound * t / cam.fx
    pl[wild] = np.concatenate([n, d[..., None]], axis=-1)[wild].astype(np.float32)
    copy = rng.random((H, W)) < 0.1
    for (dy, dx) in [(-1, 0), (0, 1), (5, 0), (0, -5)]:
        part = copy & (rng.random((H, W)) < 0.25) & (ys + dy >= 0) & (ys + dy < H) & (xs + dx >= 0) & (xs + dx < W)
        pl[part] = pl[(ys + dy)[part], (xs + dx)[part]]
    # equal-cost pairs: pixel p gets close-up (p - 1 row) with n.x = +0 and far-up (p - 5 rows) with n.x = -0
    pair = np.zeros((H, W), bool)
    if H > 5:
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
    color = sc.images.ndim == 4
    cost = np.asarray(cost_of(pl, pp.propagation_site(0, False, color)), dtype=np.float32).copy()
    for mask in (1, 2):
        k, dy, dx, ok = pp.candidates(H, W, mask)[0]
        tie = ok & (rng.random((H, W)) < 0.05)
        c = np.asarray(cost_of(pp.shifted(pl, dy, dx, ok), pp.propagation_site(k, False, color)))
        cost[tie] = c[tie]
    for _ in range(max(1, H * W // 600)):
        y0, x0 = int(rng.integers(0, H)), int(rng.integers(0, W))
        cost[y0:y0 + 6, x0:x0 + 6] = MAXCOST
    cost[pair] = MAXCOST
    return pl, cost


@pytest.mark.parametrize("color", [False, True], ids=["grey", "colour"])
@pytest.mark.parametrize("rows,cols", SHAPES, ids=["%dx%d" % s for s in SHAPES])
def test_restatement_matches_oracle_phase(rows, cols, color):
    from oracle import pypropagate as pp
    from oracle.pyoracle import Oracle
    sc = _scene(rows, cols, color)
    o = Oracle(sc)
    rng = np.random.default_rng(rows * 7 + cols + int(color))
    b = min(rows, 7)
    bands = [(0, b), (rows - b, rows)] if rows > b else [(0, rows)]
    planes0 = o.init_planes(1000 + rows)
    start = adversarial_state(sc, planes0, lambda pl, site: o.cost_eval(pl), rng)
    changed = compared = ambiguous = 0
    for state in ((planes0, o.cost_eval(planes0, init_radius=True)), start):
        for mask in MASKS:
            for colour in (0, 1):
                for y0, y1 in bands:
                    want_p, want_c = o.phase(state[0], state[1], colour, mask, y0, y1)
                    got_p, got_c, amb = pp.expected(state[0], state[1], colour, mask, lambda pl, site: o.cost_eval(pl, y0, y1),
                                                    sc.cameras[0], sc.params.depthMin, sc.params.depthMax,
                                                    color_images=color)
                    keep = np.zeros((rows, cols), bool)
                    keep[y0:y1] = True
                    keep &= ~amb
                    assert bits_equal(got_p[keep], want_p[keep]) == 0, (mask, colour, y0)
                    assert bits_equal(got_c[keep], want_c[keep]) == 0, (mask, colour, y0)
                    mine = np.zeros((rows, cols), bool)
                    mine[y0:y1] = True
                    other = mine & (((np.mgrid[0:rows, 0:cols].sum(0)) & 1) != colour)
                    assert bits_equal(got_p[other], state[0][other]) == 0
                    changed += int((got_p[keep] != state[0][keep]).any(axis=-1).sum())
                    compared += int(keep.sum())
                    ambiguous += int((amb & mine).sum())
    assert changed > 0.05 * compared                       # many decisions are taken, not just confirmed
    assert ambiguous <= 0.005 * (compared + ambiguous)


def test_fused_candidates_and_guards_match_the_kernel_tables():
    """The fused candidate table here and the one in gpm_kernels.cuh (kFused*) describe the same offsets and margins."""
    import os
    import re
    from oracle import pypropagate as pp
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gipuma_b200", "csrc",
                            "gpm_kernels.cuh")).read()

    def table(name):
        m = re.search(r"kFused%s\[20\]\s*=\s*\{([^}]*)\}" % name, src)
        return [int(v) for v in m.group(1).split(",")]
    assert table("Dy") == [dy for (dy, dx), g in pp.FUSED] and table("Dx") == [dx for (dy, dx), g in pp.FUSED]
    for i, name in enumerate(["Gx0", "Gx1", "Gy0", "Gy1"]):
        assert table(name) == [g[i] for _, g in pp.FUSED]
    dev = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gipuma_b200", "csrc",
                            "gpm_device.cuh")).read()
    for name, want in (("FLOAT", pp.FUSED_SITES_FLOAT), ("FLOAT4", pp.FUSED_SITES_FLOAT4)):
        m = re.search(r"#define GPM_FUSED_SITES_%s\s+\{([^}]*)\}" % name, dev)
        assert tuple(int(v) for v in m.group(1).split(",")) == want


def test_ambiguous_band_marks_depths_at_the_bounds():
    """A candidate whose depth at the pixel is (to float64 precision) a range bound is ambiguous; one well inside is not."""
    from oracle import pypropagate as pp
    sc = _scene(8, 8, False)
    cam, prm = sc.cameras[0], sc.params
    H = W = 8
    ys, xs = np.mgrid[0:H, 0:W]
    pl = np.zeros((H, W, 4), np.float32)
    pl[..., 2] = -1.0
    pl[..., 3] = 0.5 * (prm.depthMin + prm.depthMax)
    pl[3, 4, 3] = prm.depthMax                       # fronto-parallel: depth == d at every pixel
    cost = np.full((H, W), MAXCOST, np.float32)
    _, _, amb = pp.expected(pl, cost, 0, 1, lambda p, s: np.zeros((H, W), np.float32), cam, prm.depthMin, prm.depthMax)
    want = np.zeros((H, W), bool)
    for dy, dx in pp.CLOSE:                          # the pixels that are offered the plane of (3, 4)
        want[3 - dy, 4 - dx] = True
    assert np.array_equal(amb, want & (((xs + ys) & 1) == 0)) and amb.sum() == 4
