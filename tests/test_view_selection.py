"""Joint view selection (DESIGN.md §17) without a GPU: known answers of the restatement oracle/pyjvs.py, the gpm_view_sel
layout, and every refusal of the C-ABI, the batch drivers and the Python API before anything reaches a device."""
import ctypes as C
import math

import numpy as np
import pytest

from test_geo_batch_args import _desc

E_ARG, E_STATE = -1, -3
f32 = np.float32
EXACT = {"beta": 1e30}                         # kb = -0: every confidence is exactly 1


def _rows(*cols):
    """[K, 1, V] rows from K lists of V per-view costs (one pixel)."""
    return np.asarray(cols, f32)[:, None, :]


def _w(rows, in_e=None, remembered=None, t=0, **params):
    from oracle import pyjvs
    K, _, V = rows.shape
    in_e = np.ones((K, 1), bool) if in_e is None else np.asarray(in_e, bool)[:, None]
    rem = np.zeros((1, V), bool) if remembered is None else np.asarray(remembered, bool)[None]
    return pyjvs.weights(rows, in_e, rem, dict(EXACT, **params), t)[0]


def test_beta_1e30_gives_kb_minus_zero_and_unit_confidences():
    from oracle import pyjvs
    k = pyjvs.kb(1e30)
    assert k == 0 and math.copysign(1.0, float(k)) == -1.0
    m = np.array([0.0, 0.3, 0.79, 1.5, 2.0], f32)
    assert np.all(pyjvs.conf(m, k) == f32(1.0))
    # every rule weight is exactly 1: s_j = good_j
    w = _w(_rows([0.1, 0.5, 1.9], [0.2, 0.6, 0.1], [0.3, 0.7, 0.0], [0.4, 0.1, 1.3]))
    assert w.tolist() == [1.0, 1.0, 0.0]


def test_confidence_with_a_finite_beta():
    from oracle import pyjvs
    k = pyjvs.kb(0.3)
    assert k == f32(-math.log2(math.e) / (2 * f32(0.3) ** 2))
    c = pyjvs.conf(np.array([0.0, 0.3], f32), k)
    assert c[0] == 1.0 and abs(float(c[1]) - math.exp(-0.5)) < 1e-6


@pytest.mark.parametrize("n_good", [2, 3, 4])
def test_n_good_boundary(n_good):
    """Three good entries: a weight from n_good <= 3 on, none at n_good = 4."""
    w = _w(_rows([0.1], [0.2], [0.3], [1.0]), n_good=n_good)
    assert w.tolist() == ([1.0] if n_good <= 3 else [0.0])


@pytest.mark.parametrize("n_bad", [1, 2, 3])
def test_n_bad_boundary(n_bad):
    """Two bad entries (> tau_bad = 1.2) and three good ones: a weight only while bad_j = 2 < n_bad."""
    w = _w(_rows([0.1], [0.2], [0.3], [1.3], [2.0], [1.2]), n_bad=n_bad)
    assert w.tolist() == ([1.0] if n_bad == 3 else [0.0])


def test_thresholds_are_strict():
    from oracle import pyjvs
    tt = pyjvs.tau_t(0.8, 90, 0)
    w = _w(_rows([tt], [tt], [tt], [1.2]))                  # m = tau_t is not good; m = tau_bad is not bad
    assert w.tolist() == [0.0]
    w = _w(_rows([tt], [tt], [tt], [1.2]), remembered=[True])
    assert w.tolist() == [float(f32(0.2))]


def test_w_keep_applies_only_to_remembered_views_with_few_bad_entries():
    rows = _rows([0.9, 0.9, 1.5, 0.1], [1.0, 1.3, 1.5, 0.2], [1.0, 1.4, 1.6, 0.3])
    w = _w(rows, remembered=[True, True, True, False], w_keep=0.25)
    # view 0: no good, no bad, remembered -> w_keep; view 1: 2 bad, remembered -> w_keep; view 2: 3 bad -> 0;
    # view 3: three good -> rule weight 1
    assert w.tolist() == [0.25, 0.25, 0.0, 1.0]
    assert _w(rows, w_keep=0.25).tolist() == [0.0, 0.0, 0.0, 1.0]


def test_rule_weight_is_the_mean_confidence_of_the_good_entries():
    from oracle import pyjvs
    rows = _rows([0.1], [0.2], [0.5], [0.79])
    w = _w(rows, beta=0.3)
    k = pyjvs.kb(0.3)
    s = f32(0)
    for m in (0.1, 0.2, 0.5, 0.79):
        s = f32(s + pyjvs.conf(np.array([m], f32), k)[0])
    assert w.tolist() == [float(f32(s / f32(4)))]


def test_excluded_rows_do_not_count_and_duplicates_count_per_occurrence():
    rows = _rows([0.1, 0.1], [0.1, 0.1], [0.1, 1.5], [0.1, 1.5])
    # candidates 2 and 3 not in E (not offered or out of range): view 0 has 2 good entries only
    assert _w(rows, in_e=[True, True, False, False]).tolist() == [0.0, 0.0]
    # the same row twice (a duplicate plane) counts twice
    assert _w(_rows([0.1], [0.1], [0.1]), in_e=[True, True, True]).tolist() == [1.0]


def test_tau_t_at_t_0_1_5():
    from oracle import pyjvs
    for t in (0, 1, 5):
        want = f32(float(f32(0.8)) * math.exp(-t * t / 90.0))
        assert pyjvs.tau_t(0.8, 90, t) == want
    assert pyjvs.tau_t(0.8, 90, 0) == f32(0.8)
    assert pyjvs.tau_t(0.8, 90, 5) < pyjvs.tau_t(0.8, 90, 1) < pyjvs.tau_t(0.8, 90, 0)


def test_weighted_cost_is_sequential_and_falls_back_to_the_combination_rule():
    from oracle import pyjvs, pygeo
    rng = np.random.default_rng(3)
    c = rng.random((5, 7, 6)).astype(f32) * 2
    w = np.where(rng.random((5, 7, 6)) < 0.5, f32(0.2), f32(1.0)).astype(f32)
    w[0, :] = 0.0                                       # a row of pixels without any reliable view
    rcp = {k: f32(1.0) / f32(k) for k in range(1, 7)}
    fb = pygeo.combine(np.moveaxis(c, -1, 0), 1, 3, 1.8, rcp)
    got = pyjvs.weighted(w, c, fb)
    assert np.array_equal(got[0].view(np.uint32), fb[0].view(np.uint32))          # sum w = 0: combine_views
    num, den = f32(0), f32(0)
    for j in range(6):
        num, den = f32(num + f32(w[3, 2, j] * c[3, 2, j])), f32(den + w[3, 2, j])
    assert got[3, 2] == f32(num / den)


def test_masks_round_trip():
    from oracle import pyjvs
    sel = np.zeros((2, 64), bool)
    sel[0, [0, 5, 63]] = True
    m = pyjvs.pack_mask(sel)
    assert m[0] == (1 | 32 | (1 << 63)) and m[1] == 0
    assert np.array_equal(pyjvs.mask_bits(m, 64), sel)


def test_launch_restatement_on_a_toy_state():
    """pyjvs.expected on a 6x6 state with hand-made rows: the weights come from the candidates in E only, the current plane
    is re-scored, a cheaper weighted candidate is accepted and the new mask is written at this colour's pixels only."""
    from types import SimpleNamespace
    from oracle import pyjvs
    H = W = 6
    V = 3
    ys, xs = np.mgrid[0:H, 0:W]
    planes = np.zeros((H, W, 4), f32)
    planes[..., 2] = -1.0
    planes[..., 3] = (1.0 + (ys * W + xs)).astype(f32)           # depth grows with the pixel index; identifies the plane
    cost = np.full((H, W), 1.0, f32)
    cam = SimpleNamespace(fx=1.0, alpha=1.0, K=np.eye(3, dtype=f32))

    def rows_of(pl):
        d = pl[..., 3].astype(np.int64)
        m = np.stack([(d % 7) * f32(0.1), (d % 5) * f32(0.1), np.full(d.shape, 1.5, f32)], axis=-1).astype(f32)
        return m, m

    def fallback_of(pl):
        return np.full(pl.shape[:2], 9.0, f32)
    masks = np.zeros((H, W), np.uint64)
    p1, c1, m1, amb = pyjvs.expected(planes, cost, masks, 0, 1, rows_of, fallback_of, cam, 0.5, 100.0, {"n_good": 2, **EXACT}, 0)
    mine = ((xs + ys) & 1) == 0
    assert not amb.any()
    assert np.array_equal(p1[~mine], planes[~mine]) and np.array_equal(c1[~mine], cost[~mine]) and not m1[~mine].any()
    # view 2 (cost 1.5 everywhere) is bad in every candidate: never selected
    assert not (m1 & np.uint64(4)).any()
    assert (m1[mine] != 0).any()
    m0, _ = rows_of(planes)
    w = pyjvs.weights(np.stack([rows_of(pl)[0] for _, pl, _ in pyjvs.candidate_maps(planes, cost, 0, 1, False)]),
                      np.stack([off for _, _, off in pyjvs.candidate_maps(planes, cost, 0, 1, False)]),
                      pyjvs.mask_bits(masks, V), {"n_good": 2, **EXACT}, 0)
    rescored = pyjvs.weighted(w, m0, fallback_of(planes))
    assert np.all(c1[mine] <= rescored[mine])


def test_view_sel_layout_matches_the_header():
    from gipuma_b200 import api
    assert C.sizeof(api.GpmViewSel) == 32
    names = ("kind", "tau_init", "alpha", "tau_bad", "n_good", "n_bad", "beta", "w_keep")
    assert [getattr(api.GpmViewSel, n).offset for n in names] == [0, 4, 8, 12, 16, 20, 24, 28]
    v = api.view_sel("joint")
    assert (v.kind, v.n_good, v.n_bad) == (1, 3, 3)
    assert [v.tau_init, v.alpha, v.tau_bad, v.beta, v.w_keep] == [float(f32(x)) for x in (0.8, 90, 1.2, 0.3, 0.2)]
    assert api.VIEW_SELECTION == {"off": 0, "joint": 1}
    assert api.JVS_DEFAULTS == {"tau_init": 0.8, "alpha": 90.0, "tau_bad": 1.2, "n_good": 3, "n_bad": 3, "beta": 0.3,
                                "w_keep": 0.2}
    import re
    import os
    hdr = open(os.path.join(os.path.dirname(api.__file__), "..", "include", "gipuma_b200.h")).read()
    body = re.search(r"typedef struct gpm_view_sel \{(.*?)\} gpm_view_sel;", hdr, re.S).group(1)
    assert re.findall(r"(int|float) (\w+);", body) == [("int", "kind"), ("float", "tau_init"), ("float", "alpha"),
                                                       ("float", "tau_bad"), ("int", "n_good"), ("int", "n_bad"),
                                                       ("float", "beta"), ("float", "w_keep")]


BAD_VSEL = [((2, 0.8, 90, 1.2, 3, 3, 0.3, 0.2), "kind"), ((-1, 0.8, 90, 1.2, 3, 3, 0.3, 0.2), "kind"),
            ((1, 0.0, 90, 1.2, 3, 3, 0.3, 0.2), "tau_init"), ((1, math.nan, 90, 1.2, 3, 3, 0.3, 0.2), "tau_init"),
            ((1, 0.8, -1, 1.2, 3, 3, 0.3, 0.2), "alpha"), ((1, 0.8, 90, math.inf, 3, 3, 0.3, 0.2), "tau_bad"),
            ((1, 0.8, 90, 1.2, 3, 3, 0.0, 0.2), "beta"), ((1, 0.8, 90, 1.2, 3, 3, 0.3, -0.1), "w_keep"),
            ((1, 0.8, 90, 1.2, 3, 3, 0.3, math.inf), "w_keep"), ((1, 0.8, 90, 1.2, 0, 3, 0.3, 0.2), "n_good"),
            ((1, 0.8, 90, 1.2, 9, 3, 0.3, 0.2), "n_good"), ((1, 0.8, 90, 1.2, 3, 0, 0.3, 0.2), "n_bad"),
            ((1, 0.8, 90, 1.2, 3, 10, 0.3, 0.2), "n_bad")]


@pytest.mark.parametrize("vsel,msg", BAD_VSEL)
def test_vsel_drivers_refuse_bad_arguments_without_a_device(vsel, msg):
    from gipuma_b200 import api
    lib = api.load_library()
    g, _keep = _desc()
    o = C.byref(api.GpmJobOpts(1, 2.0, 0))
    v = C.byref(api.GpmViewSel(*vsel))
    rc = lib.gpm_geo_batch_run_vsel(C.byref(g), o, v, None)
    err = lib.gpm_batch_last_error().decode()
    assert rc == E_ARG and err.startswith("gpm_geo_batch_run_vsel: bad arguments") and msg in err, (rc, err)
    rc = lib.gpm_batch_run_vsel(C.byref(g.batch), o, v, None)
    err = lib.gpm_batch_last_error().decode()
    assert rc == E_ARG and err.startswith("gpm_batch_run_vsel: bad arguments") and msg in err, (rc, err)
    # the context setter refuses the same before looking at the context
    assert lib.gpm_set_view_selection(None, v) == E_ARG


def test_vsel_drivers_refuse_joint_with_pm_or_colour_without_a_device():
    from gipuma_b200 import api
    lib = api.load_library()
    joint = C.byref(api.view_sel("joint"))
    g, _keep = _desc()
    assert lib.gpm_batch_run_vsel(C.byref(g.batch), C.byref(api.GpmJobOpts(0, 0.0, 0)), joint, None) == E_ARG
    assert "NCC" in lib.gpm_batch_last_error().decode()
    assert lib.gpm_geo_batch_run_vsel(C.byref(g), C.byref(api.GpmJobOpts(0, 0.0, 1)), joint, None) == E_ARG
    assert "NCC" in lib.gpm_batch_last_error().decode()
    g4, _keep4 = _desc(channels=4)
    assert lib.gpm_geo_batch_run_vsel(C.byref(g4), C.byref(api.GpmJobOpts(1, 2.0, 0)), joint, None) == E_ARG
    assert "grey" in lib.gpm_batch_last_error().decode()
    # a NULL vsel is the off mode: what is left to refuse is the job options
    assert lib.gpm_batch_run_vsel(C.byref(g.batch), None, None, None) == E_ARG
    assert "opts" in lib.gpm_batch_last_error().decode()
    assert lib.gpm_batch_run_vsel(None, C.byref(api.GpmJobOpts(1, 2.0, 0)), joint, None) == E_ARG
    assert lib.gpm_batch_last_error().decode() == "gpm_batch_run_vsel: bad arguments"


def test_context_calls_refuse_null_arguments_without_a_device():
    from gipuma_b200 import api
    lib = api.load_library()
    assert lib.gpm_set_view_selection(None, C.byref(api.view_sel("joint"))) == E_ARG
    assert lib.gpm_get_view_masks(None, None) == E_ARG


@pytest.mark.parametrize("kw", [dict(view_selection="acmh"), dict(view_selection=1), dict(view_selection=None),
                                dict(view_selection="joint"),                                  # with the PM cost
                                dict(view_selection="joint", photometric="ncc", jvs_params={"tau_init": -1}),
                                dict(view_selection="joint", photometric="ncc", jvs_params={"n_good": 9}),
                                dict(view_selection="joint", photometric="ncc", jvs_params={"n_bad": 2.5}),
                                dict(view_selection="joint", photometric="ncc", jvs_params={"w_keep": float("nan")}),
                                dict(view_selection="joint", photometric="ncc", jvs_params={"gamma": 1.0})])
@pytest.mark.parametrize("entry", ["batch_run", "geometric_pass"])
def test_api_refuses_bad_view_selection_before_loading_the_library(monkeypatch, kw, entry):
    from gipuma_b200 import api, scene as S

    def no_library():
        raise AssertionError("the library was loaded")
    monkeypatch.setattr(api, "load_library", no_library)
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1)
    with pytest.raises(ValueError):
        getattr(api, entry)(np.zeros((3, 16, 16), np.float32), [np.eye(3, 4)] * 3, params, [0], **kw)


def test_geometric_pass_refuses_joint_on_colour_before_loading_the_library(monkeypatch):
    from gipuma_b200 import api, scene as S
    monkeypatch.setattr(api, "load_library", lambda: (_ for _ in ()).throw(AssertionError("the library was loaded")))
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1)
    with pytest.raises(ValueError):
        api.geometric_pass(np.zeros((3, 16, 16, 4), np.float32), [np.eye(3, 4)] * 3, params, [0], photometric="ncc",
                           view_selection="joint")


def test_shard_runners_refuse_joint_before_creating_a_context(monkeypatch):
    from types import SimpleNamespace
    from gipuma_b200 import api, multigpu
    monkeypatch.setattr(api, "Context", lambda *a, **k: (_ for _ in ()).throw(AssertionError("a context was created")))
    sc = SimpleNamespace(n_views=4, cols=16, rows=16)
    for kind in ("joint", "acmh"):
        with pytest.raises(ValueError, match="view selection|view_selection"):
            multigpu.ViewShardRunner(sc, 0, 1, view_selection=kind)
        with pytest.raises(ValueError, match="view selection|view_selection"):
            multigpu.run_hybrid(lambda r: sc, 1, 0, 1, 1, view_selection=kind)
