"""The planar prior inside the multi-level driver (DESIGN.md §20) without a GPU: the header's gpm_ms_prior_opts layout, and
every refusal of gpm_ms_batch_run_prior and of multiscale_pass's planar_prior / geo_prior, raised before any device is
needed."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from test_multiscale import _ms_desc, _no_library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_ARG, E_STATE = -1, -3

# Box 9, alpha 0.9, tau_color 10, tau_gradient 2: the largest valid PM cost is 25 * 2.8 = 70, and the geometric term of
# _ms_desc (weight 0.5, max_err 3) adds at most 1.5.  A prior weight of 929 keeps 70 + 929 below MAXCOST (1000) but not
# 70 + 1.5 + 929; with NCC (largest cost 2) the same holds for 997.
W_PM, W_NCC = 929.0, 997.0


def test_struct_layout_matches_ctypes(tmp_path):
    from gipuma_b200 import api
    fields = ["photometric", "geometric", "level_build_ms"]
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%%zu\\n", '
                   'sizeof(gpm_ms_prior_opts)); %s return 0; }\n' %
                   " ".join('printf("%%zu\\n", offsetof(gpm_ms_prior_opts, %s));' % f for f in fields))
    exe = str(tmp_path / "s")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.GpmMsPriorOpts)] + [getattr(api.GpmMsPriorOpts, f).offset for f in fields]


# ---- gpm_ms_batch_run_prior ----------------------------------------------------------------------------------------------

def _stage(weight=2.0, depth_sigma=5.0, normal_sigma_deg=5.0, step=5, support_cost=0.5, iterations=1):
    from gipuma_b200 import api
    return api.GpmPriorOpts(weight, depth_sigma, normal_sigma_deg, step, support_cost, iterations, None)


def _run(m, photometric=None, geometric=None, opts=None, vsel=None, prior=True):
    from gipuma_b200 import api
    lib = api.load_library()
    po = api.GpmMsPriorOpts(C.pointer(photometric) if photometric else None, C.pointer(geometric) if geometric else None)
    opts = opts or api.job_opts()
    rc = lib.gpm_ms_batch_run_prior(C.byref(m), C.byref(opts), C.byref(vsel) if vsel else None,
                                    C.byref(po) if prior else None, None)
    return rc, lib.gpm_batch_last_error().decode()


def _refused(rc, msg, *words):
    assert rc == E_ARG and msg.startswith("gpm_ms_batch_run_prior: bad arguments"), (rc, msg)
    for w in words:
        assert w in msg, (w, msg)


@pytest.mark.parametrize("stage", ["photometric", "geometric"])
@pytest.mark.parametrize("kw,word", [(dict(weight=-1.0), "weight"), (dict(weight=float("nan")), "weight"),
                                     (dict(depth_sigma=0.0), "depth_sigma"), (dict(normal_sigma_deg=91.0), "normal_sigma"),
                                     (dict(step=0), "step"), (dict(step=65), "step"),
                                     (dict(support_cost=float("nan")), "support_cost"), (dict(iterations=-1), "iterations")],
                         ids=["weight_-1", "weight_nan", "depth_sigma_0", "normal_sigma_91", "step_0", "step_65",
                              "support_cost_nan", "iterations_-1"])
def test_bad_stage_options_are_refused_before_any_cuda_call(stage, kw, word):
    m, _keep = _ms_desc()
    rc, msg = _run(m, **{stage: _stage(**kw)})
    _refused(rc, msg, stage + " prior stage", word)


@pytest.mark.parametrize("stage", ["photometric", "geometric"])
def test_colour_images_and_joint_view_selection_are_refused_with_either_stage(stage):
    from gipuma_b200 import api
    m, _keep = _ms_desc(channels=4)
    rc, msg = _run(m, **{stage: _stage()})
    _refused(rc, msg, stage + " prior stage", "planar prior")
    m, _keep = _ms_desc()
    rc, msg = _run(m, opts=api.job_opts("ncc"), vsel=api.view_sel("joint"), **{stage: _stage()})
    _refused(rc, msg, stage + " prior stage", "planar prior")
    rc, msg = _run(m, opts=api.job_opts("ncc"), vsel=api.view_sel("joint"))      # no stage: the multi-level driver runs JVS
    assert rc != E_ARG, msg


@pytest.mark.parametrize("photometric,weight", [("pm", W_PM), ("ncc", W_NCC)])
def test_the_geometric_stage_bound_includes_the_geometric_term(photometric, weight):
    from gipuma_b200 import api
    opts = api.job_opts(photometric)
    m, _keep = _ms_desc()
    rc, msg = _run(m, opts=opts, geometric=_stage(weight=weight))
    _refused(rc, msg, "geometric prior stage", "MAXCOST")
    rc, msg = _run(m, opts=opts, photometric=_stage(weight=weight))             # the same weight without the term
    assert rc != E_ARG, msg
    rc, msg = _run(m, opts=opts, photometric=_stage(weight=weight + 2.0))
    _refused(rc, msg, "photometric prior stage", "MAXCOST")
    m0, _keep0 = _ms_desc(weight=0.0)                                            # the term off: the bound is the photometric one
    rc, msg = _run(m0, opts=opts, geometric=_stage(weight=weight))
    assert rc != E_ARG, msg


def test_a_4098_wide_level_0_is_refused_with_the_geometric_stage_only():
    m, _keep = _ms_desc(levels=2, width=4098, height=64)
    rc, msg = _run(m, geometric=_stage())
    _refused(rc, msg, "geometric prior stage", "4097")
    rc, msg = _run(m, photometric=_stage())                                      # the coarsest level is 2049 x 32
    assert rc != E_ARG, msg
    m1, _keep1 = _ms_desc(levels=1, width=4098, height=64)                       # one level: the coarsest is level 0
    rc, msg = _run(m1, photometric=_stage())
    _refused(rc, msg, "photometric prior stage", "4097")
    m2, _keep2 = _ms_desc(levels=2, width=64, height=8196)                      # 4098 tall at the coarsest level
    rc, msg = _run(m2, photometric=_stage())
    _refused(rc, msg, "photometric prior stage", "4097")
    m3, _keep3 = _ms_desc(levels=2, width=64, height=8194)                      # 4097: accepted
    rc, msg = _run(m3, photometric=_stage())
    assert rc != E_ARG, msg


@pytest.mark.parametrize("kw", [dict(levels=0), dict(radius=5), dict(channels=2), dict(weight=float("nan")),
                                dict(ref_indices=(C.c_int * 2)(0, 3))],
                         ids=["levels_0", "radius_5", "channels_2", "weight_nan", "ref_out_of_range"])
@pytest.mark.parametrize("prior", [False, True], ids=["prior_null", "stages_null"])
def test_what_gpm_ms_batch_run_refuses_is_refused(kw, prior):
    m, _keep = _ms_desc(**kw)
    rc, msg = _run(m, prior=prior)
    _refused(rc, msg)


def test_a_view_without_source_views_is_named_before_any_cuda_call():
    m, _keep = _ms_desc(min_angle=0.1, max_angle=0.2)
    rc, msg = _run(m, photometric=_stage(), geometric=_stage())
    assert rc == E_STATE and msg.endswith("reference view 0"), (rc, msg)


def test_valid_stages_pass_every_check():
    m, _keep = _ms_desc(levels=3, width=128, height=96)
    rc, msg = _run(m, photometric=_stage(), geometric=_stage(support_cost=1.0))
    assert rc != E_ARG and rc != E_STATE, msg                 # runs on a GPU; without one it fails for want of a device


# ---- multiscale_pass -----------------------------------------------------------------------------------------------------

def _args(**kw):
    from gipuma_b200 import scene as S
    p = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N)
    p.depthMin, p.depthMax = 300.0, 800.0
    a = dict(images=np.zeros((3, 48, 64), np.float32), Ps=[np.eye(3, 4)] * 3, params=p, refs=[0], levels=2)
    a.update(kw)
    return a


@pytest.mark.parametrize("kw", [dict(planar_prior={"weight": -1.0}), dict(geo_prior={"depth_sigma": 0.0}),
                                dict(planar_prior={"step": 0}), dict(geo_prior={"support_cost": float("nan")}),
                                dict(geo_prior={"iterations": -1}), dict(planar_prior={"sigma": 1.0}),
                                dict(geo_prior={}, images=np.zeros((3, 48, 64, 4), np.float32)),
                                dict(planar_prior={}, images=np.zeros((3, 48, 64, 4), np.float32)),
                                dict(geo_prior={}, photometric="ncc", view_selection="joint"),
                                dict(planar_prior={}, photometric="ncc", view_selection="joint"),
                                dict(geo_prior={"weight": W_PM}), dict(planar_prior={"weight": W_PM + 2.0}),
                                dict(geo_prior={"weight": W_NCC}, photometric="ncc"),
                                dict(geo_prior={}, images=np.zeros((3, 64, 4098), np.float32)),
                                dict(planar_prior={}, levels=1, images=np.zeros((3, 64, 4098), np.float32))],
                         ids=["weight_-1", "depth_sigma_0", "step_0", "support_cost_nan", "iterations_-1", "unknown_key",
                              "geo_colour", "photo_colour", "geo_jvs", "photo_jvs", "geo_bound_pm", "photo_bound_pm",
                              "geo_bound_ncc", "geo_4098_wide", "photo_4098_wide_one_level"])
def test_multiscale_pass_refuses_bad_stages_before_loading_the_library(monkeypatch, kw):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    with pytest.raises(ValueError):
        api.multiscale_pass(**_args(**kw))


@pytest.mark.parametrize("kw", [dict(planar_prior={"weight": W_PM}), dict(geo_prior={"weight": W_PM}, weight=0.0),
                                dict(planar_prior={}, images=np.zeros((3, 64, 4098), np.float32)),
                                dict(planar_prior={}, geo_prior={"support_cost": 1.0})],
                         ids=["photo_bound_pm", "geo_bound_without_the_term", "photo_4098_wide", "both"])
def test_multiscale_pass_passes_valid_stages_to_the_library(monkeypatch, kw):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    with pytest.raises(AssertionError, match="the library was reached"):
        api.multiscale_pass(**_args(**kw))


def test_the_bound_restatement_agrees_with_the_library_bound():
    """check_prior_bound raises exactly where gpm_ms_batch_run_prior refuses the weight (the bound in float32)."""
    from gipuma_b200 import api
    m, _keep = _ms_desc()
    p = SimpleNamespace(box_hsize=9, alpha=0.9, tau_color=10.0, tau_gradient=2.0)
    for photometric in ("pm", "ncc"):
        top = 70.0 if photometric == "pm" else 2.0
        for w in np.nextafter(np.float32(1000.0 - top - 1.5), np.float32([0, 2000])).tolist() + [1000.0 - top - 1.5]:
            try:
                api.check_prior_bound(p, photometric, 0.5, 3.0, w)
                ok = True
            except ValueError:
                ok = False
            rc, msg = _run(m, opts=api.job_opts(photometric), geometric=_stage(weight=w))
            assert ok == (rc != E_ARG), (photometric, w, rc, msg)
