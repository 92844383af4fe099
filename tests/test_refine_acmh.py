"""ACMH's refinement (DESIGN.md §23) without a GPU: the hash's known answers, the candidates' properties and draw order in the
float32 restatement oracle/pyrefine.py, the header's gpm_refine_opts layout, and every refusal of the Python API (raised
before the library loads) and of the C-ABI's _refine drivers (raised before any CUDA call)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_multiscale import _ms_desc, _no_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_ARG = -1
f32 = np.float32


def _mix_int(x):
    """lowbias32 on Python integers, independent of numpy's uint32 arithmetic."""
    x &= 0xFFFFFFFF
    x ^= x >> 16
    x = (x * 0x7FEB352D) & 0xFFFFFFFF
    x ^= x >> 15
    x = (x * 0x846CA68B) & 0xFFFFFFFF
    x ^= x >> 16
    return x


def test_hash_known_answers():
    from oracle import pyrefine as R
    kat = {0: 0x0, 1: 0x688990C0, 2: 0xD1132181, 0xDEADBEEF: 0xE628C683, 0xFFFFFFFF: 0x6768824A}
    for x, want in kat.items():
        assert _mix_int(x) == want
        assert int(R.mix(np.uint32(x))) == want
    rng = np.random.default_rng(1)
    xs = rng.integers(0, 2 ** 32, 1000, dtype=np.uint64).astype(np.uint32)
    assert [int(v) for v in R.mix(xs)] == [_mix_int(int(v)) for v in xs]
    # the key chains seed, pixel and launch; the 64-bit seed is folded to 32 bits by xor
    seed, i, r = 0x1234_5678_9ABC_DEF0, 4321, 7
    s = (seed & 0xFFFFFFFF) ^ (seed >> 32)
    assert R.seed32(seed) == s
    assert int(R.key(seed, np.uint32(i), r)) == _mix_int(_mix_int(_mix_int(s) ^ i) ^ r)
    # words map to (0, 1] as xorwow_uniform maps them: 0 -> 2^-33, 2^32 - 1 -> 1
    assert R.uniform(np.uint32(0)) == f32(2.0 ** -33)
    assert R.uniform(np.uint32(0xFFFFFFFF)) == f32(1.0)
    u = R.uniform(R.mix(xs))
    assert u.dtype == np.float32 and np.all((u > 0) & (u <= 1))


def test_fma32_rounds_once():
    from oracle import pyrefine as R
    rng = np.random.default_rng(3)
    a, b, c = (rng.normal(size=20000).astype(np.float32) for _ in range(3))
    got = R.fma32(a, b, c)
    # exact reference: the product and sum in rational arithmetic, rounded to float32 by comparing neighbours
    from fractions import Fraction
    for k in range(0, 20000, 97):
        exact = Fraction(float(a[k])) * Fraction(float(b[k])) + Fraction(float(c[k]))
        g = got[k]
        lo, hi = np.nextafter(g, f32(-np.inf)), np.nextafter(g, f32(np.inf))
        assert abs(Fraction(float(g)) - exact) <= abs(Fraction(float(lo)) - exact)
        assert abs(Fraction(float(g)) - exact) <= abs(Fraction(float(hi)) - exact)
    # (1 + 2^-23) + 2^-24 - 2^-70 lands on a float32 midpoint once rounded to float64, where ties-to-even would round
    # up; the exact value is below the midpoint
    one_ulp = f32(1.0 + 2.0 ** -23)
    assert R.fma32(one_ulp, f32(2.0 ** -24 * (1 - 2.0 ** -23)), one_ulp) == one_ulp


def _scene():
    from gipuma_b200 import api, scene as S
    sc = S.make_config(2, rows=40, cols=56, n_views=3, iterations=1, seed=11)
    return sc, api.pack_camera(sc.cameras[0])


def _start_planes(sc, cam, rng):
    """Random camera-facing planes through depths inside the range."""
    from oracle import pyrefine as R
    H, W = sc.rows, sc.cols
    n = rng.normal(size=(H, W, 3))
    n[..., 2] = -np.abs(n[..., 2]) - 0.3
    n /= np.linalg.norm(n, axis=-1, keepdims=True)
    n = n.astype(np.float32)
    ys, xs = np.mgrid[0:H, 0:W]
    depth = rng.uniform(sc.params.depthMin * 1.05, sc.params.depthMax * 0.95, (H, W)).astype(np.float32)
    c = R._cam(cam)
    d = R.plane_d(c, n[..., 0], n[..., 1], n[..., 2], xs.astype(f32), ys.astype(f32), depth)
    return np.concatenate([n, d[..., None]], axis=-1).astype(np.float32)


def _cands(sc, cam, planes, eps=0.02, seed=99, r=3):
    from oracle import pyrefine as R
    p = sc.params
    return R.candidates(planes, cam, p.min_disparity, p.max_disparity, p.depthMin, p.depthMax, eps, seed, r)


def test_candidates_are_unit_camera_facing_and_in_range():
    from oracle import pyrefine as R
    sc, cam = _scene()
    planes = _start_planes(sc, cam, np.random.default_rng(5))
    p = sc.params
    for eps in (0.02, 0.3, 0.999):
        cand = _cands(sc, cam, planes, eps=eps)
        assert cand.shape == (5,) + planes.shape and cand.dtype == np.float32
        H, W = planes.shape[:2]
        ys, xs = np.mgrid[0:H, 0:W]
        c = R._cam(cam)
        v = np.stack(R.ray(c, xs.astype(f32), ys.astype(f32)), axis=-1).astype(np.float64)
        for j in (1, 2, 3):                                   # n_r, n_r, n_t: unit and facing the camera
            n = cand[j, ..., :3].astype(np.float64)
            assert np.all(np.abs(np.linalg.norm(n, axis=-1) - 1) <= 4e-7 * 3)
            assert np.all(np.einsum("hwi,hwi->hw", n, v) <= 1e-6 * np.linalg.norm(v, axis=-1))
        for j in (0, 4):                                      # the start normal, bit for bit
            assert np.array_equal(cand[j, ..., :3].view(np.uint32), planes[..., :3].view(np.uint32))
        assert np.array_equal(cand[1, ..., :3].view(np.uint32), cand[2, ..., :3].view(np.uint32))
        d, d_r, d_t = R.candidate_depths(planes, cam, p.min_disparity, p.max_disparity, p.depthMin, p.depthMax, eps, 99, 3)
        fb = float(f32(cam.f)) * float(f32(cam.baseline))
        lo, hi = fb / float(f32(p.max_disparity)), fb / float(f32(p.min_disparity))
        assert np.all((d_r >= lo * (1 - 1e-6)) & (d_r <= hi * (1 + 1e-6)))
        assert np.all((d_t >= f32(p.depthMin)) & (d_t <= f32(p.depthMax)))
        rel = np.abs(d_t.astype(np.float64) / d.astype(np.float64) - 1.0)
        inside = (d.astype(np.float64) * (1 - eps) >= p.depthMin) & (d.astype(np.float64) * (1 + eps) <= p.depthMax)
        assert (inside.mean() > 0.5 or eps > 0.1) and np.all(rel[inside] <= eps * (1 + 1e-6) + 3e-7)
        # each candidate's plane passes through its depth at the pixel (up to float32 cancellation at grazing planes)
        for j, want in ((0, d_r), (1, d), (2, d_r), (3, d), (4, d_t)):
            err = np.abs(R.prior_depth(c, cand[j], xs.astype(f32), ys.astype(f32)).astype(np.float64) / want - 1)
            assert np.percentile(err, 99) <= 1e-4 and err.max() <= 1e-2, (j, float(err.max()))


def test_draw_order_including_rejected_marsaglia_pairs():
    from oracle import pyrefine as R
    sc, cam = _scene()
    planes = _start_planes(sc, cam, np.random.default_rng(6))
    H, W = planes.shape[:2]
    ys, xs = np.mgrid[0:H, 0:W]
    seed, r, eps = 99, 3, f32(0.02)
    k = R.key(seed, (ys * W + xs).astype(np.uint32), r)
    _, _, _, pairs = R.marsaglia(k)
    assert (pairs == 1).any() and (pairs == 2).any() and (pairs >= 3).any()
    c = R._cam(cam)
    v = R.ray(c, xs.astype(f32), ys.astype(f32))
    cand = _cands(sc, cam, planes, eps=eps, seed=seed, r=r)
    for want_pairs in (1, 2, 3):
        y, x = np.argwhere(pairs == want_pairs)[0]
        kk = k[y, x]
        u = [float(R.draw(kk, j)) for j in range(5 + 2 * want_pairs)]
        # every earlier pair was rejected, the last one accepted
        a = [2 * u[5 + 2 * m] - 1 for m in range(want_pairs)]
        b = [2 * u[6 + 2 * m] - 1 for m in range(want_pairs)]
        assert all(a[m] ** 2 + b[m] ** 2 >= 1 - 1e-6 for m in range(want_pairs - 1))
        s = a[-1] ** 2 + b[-1] ** 2
        n = np.array([2 * a[-1] * np.sqrt(1 - s), 2 * b[-1] * np.sqrt(1 - s), 1 - 2 * s])
        vv = np.array([float(t[y, x]) for t in v])
        if n @ vv > 0:
            n = -n
        assert np.allclose(cand[1, y, x, :3], n, atol=2e-6), (want_pairs, cand[1, y, x, :3], n)
    # d_t takes draw 0, n_t draws 1..3 and d_r draw 4: moving one key changes exactly the candidates that read it
    y, x = 7, 9
    d, _, _ = R.candidate_depths(planes, cam, sc.params.min_disparity, sc.params.max_disparity, sc.params.depthMin,
                                 sc.params.depthMax, eps, seed, r)
    u0 = float(R.draw(k[y, x], 0))
    assert np.isclose(float(R.prior_depth(c, cand[4], xs.astype(f32), ys.astype(f32))[y, x]),
                      min(max(float(d[y, x]) * (1 + float(eps) * (2 * u0 - 1)), sc.params.depthMin), sc.params.depthMax), rtol=1e-5)
    u4 = float(R.draw(k[y, x], 4))
    disp = (sc.params.max_disparity - sc.params.min_disparity) * u4 + sc.params.min_disparity
    assert np.isclose(float(R.prior_depth(c, cand[0], xs.astype(f32), ys.astype(f32))[y, x]), cam.f * cam.baseline / disp, rtol=1e-5)
    t = np.array([float(planes[y, x, i]) + float(eps) * np.pi * (2 * float(R.draw(k[y, x], 1 + i)) - 1) for i in range(3)])
    t /= np.linalg.norm(t)
    vv = np.array([float(q[y, x]) for q in v])
    assert np.allclose(cand[3, y, x, :3], -t if t @ vv > 0 else t, atol=2e-6)


def test_launches_and_pixels_draw_different_candidates():
    sc, cam = _scene()
    planes = _start_planes(sc, cam, np.random.default_rng(8))
    a, b, c = _cands(sc, cam, planes, r=0), _cands(sc, cam, planes, r=1), _cands(sc, cam, planes, seed=100, r=0)
    assert np.array_equal(a.view(np.uint32), _cands(sc, cam, planes, r=0).view(np.uint32))
    for other in (b, c):
        assert (a[1].view(np.uint32) != other[1].view(np.uint32)).any(axis=-1).mean() > 0.99
    # two pixels with the same plane draw different candidates
    flat = np.broadcast_to(planes[5, 5], planes.shape).copy()
    d = _cands(sc, cam, flat)
    assert len({tuple(d[1, y, x].view(np.uint32)) for y in range(4) for x in range(4)}) == 16


def test_accept_is_in_order_and_strict():
    from oracle import pyrefine as R
    planes = np.zeros((1, 4, 4), np.float32)
    cost = np.array([[1.0, 1.0, 1.0, np.nan]], np.float32)
    cand = np.stack([np.full((1, 4, 4), j + 1, np.float32) for j in range(5)])
    cc = np.array([[[1.0, 0.5, 2.0, 0.1]], [[0.9, 0.5, 2.0, 0.1]], [[0.9, 0.4, 2.0, 0.1]], [[0.8, 0.4, 2.0, 0.1]],
                   [[0.8, 0.4, 2.0, 0.1]]], np.float32)
    p, c, changed = R.accept(planes, cost, cand, cc, np.ones((1, 4), bool))
    assert c[0, :3].tolist() == [f32(0.8), f32(0.4), 1.0] and np.isnan(c[0, 3])
    assert p[0, :, 0].tolist() == [4.0, 3.0, 0.0, 0.0]             # ties keep the earlier plane; NaN accepts nothing
    assert changed.tolist() == [[True, True, False, False]]


def test_jvs_accept_scores_with_the_launch_weights():
    """Under joint view selection each candidate costs sum w c / sum w over its own row (the combination rule's cost
    where sum w = 0), accepted in order with strict <: a tie keeps the running plane, a NaN anywhere in a row (0 * NaN is
    NaN) rejects the candidate, a NaN running cost accepts nothing, and pixels outside `where` keep their state."""
    from oracle import pyrefine as R
    V = 3
    w = np.array([[[0.5, 0.0, 0.5], [0.5, 0.0, 0.5], [0.0, 0.0, 0.0], [0.5, 0.0, 0.5], [0.5, 0.5, 0.5], [0.5, 0.0, 0.5]]], f32)
    cost = np.array([[1.0, 1.0, 1.0, np.nan, 1.0, 1.0]], f32)
    planes = np.zeros((1, 6, 4), f32)
    cand = np.stack([np.full((1, 6, 4), j + 1, f32) for j in range(5)])
    rows = np.full((5, 1, 6, V), 3.0, f32)
    fb = np.full((5, 1, 6), 3.0, f32)
    # pixel 0: candidate 1 ties the running cost (0.5 * 1 + 0.5 * 1) / 1 = 1, candidate 3 is strictly below, 4 ties it
    rows[1, 0, 0] = [1.0, 9.0, 1.0]
    rows[3, 0, 0] = [0.5, 9.0, 0.25]
    rows[4, 0, 0] = [0.25, 9.0, 0.5]
    # pixel 1: NaN in the unweighted view of candidate 0 rejects it; candidate 2 wins
    rows[0, 0, 1] = [0.0, np.nan, 0.0]
    rows[2, 0, 1] = [0.5, 0.0, 0.5]
    # pixel 2: no weight, so the fallback decides: candidate 4's 0.25
    fb[4, 0, 2] = 0.25
    rows[0, 0, 2] = 0.0                                        # a row the weights ignore
    # pixel 3: NaN running cost; pixel 4: outside `where`; pixel 5: nothing below 1
    rows[:, 0, 3] = 0.0
    rows[:, 0, 4] = 0.0
    where = np.array([[True, True, True, True, False, True]])
    p, c, changed = R.jvs_accept(w, planes, cost, cand, rows, fb, where)
    assert c[0, 0] == f32(0.375) and p[0, 0, 0] == 4.0          # 0.5 * 0.5 + 0.5 * 0.25 = 0.375, the tie of 4 rejected
    assert c[0, 1] == f32(0.5) and p[0, 1, 0] == 3.0
    assert c[0, 2] == f32(0.25) and p[0, 2, 0] == 5.0
    assert np.isnan(c[0, 3]) and c[0, 4] == 1.0 and c[0, 5] == 1.0
    assert changed.tolist() == [[True, True, True, False, False, False]]
    assert not p[0, 3:].any()


def test_jvs_expected_refinement_alone_keeps_remembered_views():
    """A launch of the refinement alone (mask 4) offers no candidate, so E is empty: every remembered view weighs w_keep,
    the others 0, the new masks equal the remembered ones at the launch's colour, and the five candidates are scored with
    those weights from the start plane; a pixel with no remembered view falls back to the combination rule."""
    from oracle import pyjvs, pyrefine as R
    sc, cam = _scene()
    H, W, V = sc.rows, sc.cols, 3
    rng = np.random.default_rng(17)
    planes = _start_planes(sc, cam, rng)
    masks = rng.integers(0, 8, (H, W)).astype(np.uint64)
    ys, xs = np.mgrid[0:H, 0:W]

    def rows_of(pl):                                           # a deterministic per-view cost of each plane
        b = pl.view(np.uint32).astype(np.uint64).sum(axis=-1)
        m = np.stack([((b * (2 * j + 3)) % 1009).astype(f32) / f32(500.0) for j in range(V)], axis=-1).astype(f32)
        return m, m

    def fallback_of(pl):
        return rows_of(pl)[0].mean(axis=-1).astype(f32)
    cost = pyjvs.weighted(pyjvs.weights(np.zeros((0, H, W, V), f32), np.zeros((0, H, W), bool), pyjvs.mask_bits(masks, V),
                                        {}, 1), rows_of(planes)[1], fallback_of(planes))
    prm = sc.params
    for colour in (0, 1):
        mine = ((xs + ys) & 1) == colour
        args = (rows_of, fallback_of, sc.cameras[0], cam, prm.min_disparity, prm.max_disparity, prm.depthMin, prm.depthMax,
                0.02, 99, 5, {}, 1)
        p, c, m, amb, refined = R.jvs_expected(planes, cost, masks, colour, 4, *args)
        assert not amb.any() and np.array_equal(m, masks)
        w = np.where(pyjvs.mask_bits(masks, V), f32(pyjvs.DEFAULTS["w_keep"]), f32(0.0)).astype(f32)
        cand = R.candidates(planes, cam, prm.min_disparity, prm.max_disparity, prm.depthMin, prm.depthMax, 0.02, 99, 5)
        want_c = cost.copy()
        want_p = planes.copy()
        for j in range(5):
            cj = pyjvs.weighted(w, rows_of(cand[j])[1], fallback_of(cand[j]))
            take = mine & (cj < want_c)
            want_c = np.where(take, cj, want_c)
            want_p = np.where(take[..., None], cand[j], want_p)
        assert np.array_equal(p.view(np.uint32), want_p.view(np.uint32)) and np.array_equal(c.view(np.uint32), want_c.view(np.uint32))
        assert refined.any() and not refined[~mine].any() and (masks == 0).any()
        # the other colour is untouched
        assert np.array_equal(p[~mine].view(np.uint32), planes[~mine].view(np.uint32))


def test_struct_layout_matches_ctypes(tmp_path):
    from gipuma_b200 import api
    fields = ["kind", "perturbation"]
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%%zu\\n", '
                   'sizeof(gpm_refine_opts)); %s printf("%%d %%d\\n", GPM_REFINE_GIPUMA, GPM_REFINE_ACMH); return 0; }\n' %
                   " ".join('printf("%%zu\\n", offsetof(gpm_refine_opts, %s));' % f for f in fields))
    exe = str(tmp_path / "s")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.GpmRefineOpts)] + [getattr(api.GpmRefineOpts, f).offset for f in fields] + \
        [api.REFINEMENT["gipuma"], api.REFINEMENT["acmh"]]


BAD = ["bad", 1, {"kind": "acmh", "perturbation": 0.0}, {"kind": "acmh", "perturbation": 1.0},
       {"kind": "acmh", "perturbation": -0.1}, {"kind": "acmh", "perturbation": float("nan")},
       {"kind": "acmh", "perturbation": float("inf")}, {"kind": "acmh", "perturbation": 1 - 1e-9},
       {"kind": "acmh", "perturbation": True}, {"kind": "gipuma", "perturbation": 2.0}, {"perturbation": 0.1},
       {"kind": "acmh", "eps": 0.1}, {"kind": "ACMH"}]
BAD_IDS = ["kind_str", "kind_int", "eps_0", "eps_1", "eps_neg", "eps_nan", "eps_inf", "eps_rounds_to_1", "eps_bool",
           "gipuma_eps_2", "no_kind", "unknown_key", "kind_case"]


@pytest.mark.parametrize("refinement", BAD, ids=BAD_IDS)
@pytest.mark.parametrize("driver", ["batch_run", "geometric_pass", "multiscale_pass"])
def test_python_refuses_bad_refinement_before_the_library_loads(monkeypatch, driver, refinement):
    from gipuma_b200 import api, scene as S
    _no_library(monkeypatch)
    p = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N)
    p.depthMin, p.depthMax = 300.0, 800.0
    args = dict(images=np.zeros((3, 48, 64), np.float32), Ps=[np.eye(3, 4)] * 3, params=p, refs=[0])
    if driver == "multiscale_pass":
        args["levels"] = 2
    with pytest.raises(ValueError):
        getattr(api, driver)(refinement=refinement, **args)


@pytest.mark.parametrize("kind,eps", [("bad", 0.02), ("acmh", 0.0), ("acmh", 1.0), ("acmh", float("nan")), ("gipuma", -1.0),
                                      ("acmh", "0.1"), ("acmh", None)],
                         ids=["kind", "eps_0", "eps_1", "eps_nan", "gipuma_eps_neg", "eps_str", "eps_none"])
def test_context_set_refinement_refuses_before_the_library(kind, eps):
    from gipuma_b200 import api
    ctx = api.Context.__new__(api.Context)        # no library, no device: the check must come first
    with pytest.raises(ValueError):
        ctx.set_refinement(kind, eps)


def test_good_refinement_values_pack():
    from gipuma_b200 import api
    assert api.refine_opts(None) is None
    o = api.refine_opts("acmh")
    assert (o.kind, o.perturbation) == (1, f32(0.02))
    o = api.refine_opts({"kind": "gipuma", "perturbation": 0.5})
    assert (o.kind, o.perturbation) == (0, 0.5)
    assert api.REFINE_DEFAULTS == {"perturbation": 0.02}


# ---- the C-ABI's _refine drivers refuse bad options before any CUDA call ------------------------------------------------

@pytest.mark.parametrize("kind,eps", [(2, 0.02), (-1, 0.02), (1, 0.0), (1, 1.0), (1, float("nan")), (0, float("inf"))],
                         ids=["kind_2", "kind_-1", "eps_0", "eps_1", "eps_nan", "gipuma_eps_inf"])
@pytest.mark.parametrize("driver", ["batch", "geo", "ms"])
def test_c_drivers_refuse_bad_refinement(driver, kind, eps):
    from gipuma_b200 import api
    lib = api.load_library()
    m, _keep = _ms_desc()
    r = api.GpmRefineOpts(kind, eps)
    opts = api.job_opts()
    if driver == "batch":
        rc = lib.gpm_batch_run_refine(C.byref(m.geo.batch), C.byref(opts), None, None, C.byref(r), None)
    elif driver == "geo":
        rc = lib.gpm_geo_batch_run_refine(C.byref(m.geo), C.byref(opts), None, None, C.byref(r), None)
    else:
        po = api.GpmMsPriorOpts(None, None)
        rc = lib.gpm_ms_batch_run_refine(C.byref(m), C.byref(opts), None, C.byref(po), None, C.byref(r), None)
    msg = lib.gpm_batch_last_error().decode()
    name = {"batch": "gpm_batch_run_refine", "geo": "gpm_geo_batch_run_refine", "ms": "gpm_ms_batch_run_refine"}[driver]
    assert rc == E_ARG and msg.startswith(name + ": bad arguments"), (rc, msg)
    assert ("refinement kind" in msg) if kind not in (0, 1) else ("perturbation" in msg), msg


def test_set_refinement_refuses_a_null_context():
    from gipuma_b200 import api
    lib = api.load_library()
    assert lib.gpm_set_refinement(None, 1, 0.02) == E_ARG
