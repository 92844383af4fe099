"""The detail restorer (DESIGN.md §21) without a GPU: the header's gpm_ms_restore_opts layout, every refusal of
gpm_ms_batch_run_restore and of multiscale_pass's detail_restorer, raised before any device is needed, gpm_set_geo_mask's
refusal of a null context, and the known answers of the float32 restatement oracle/pyrestore.py."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from test_multiscale import _ms_desc, _no_library
from test_multiscale_prior import _args, _stage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_ARG, E_STATE = -1, -3
f32 = np.float32


def test_struct_layout_matches_ctypes(tmp_path):
    from gipuma_b200 import api
    fields = ["photo_iterations", "threshold", "iterations", "restored"]
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%%zu\\n", '
                   'sizeof(gpm_ms_restore_opts)); %s return 0; }\n' %
                   " ".join('printf("%%zu\\n", offsetof(gpm_ms_restore_opts, %s));' % f for f in fields))
    exe = str(tmp_path / "s")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.GpmMsRestoreOpts)] + [getattr(api.GpmMsRestoreOpts, f).offset for f in fields]


# ---- gpm_ms_batch_run_restore --------------------------------------------------------------------------------------------

def _restore(photo_iterations=2, threshold=1.0, iterations=2):
    from gipuma_b200 import api
    return api.GpmMsRestoreOpts(photo_iterations, threshold, iterations, None)


def _run(m, restore=None, geometric=None, opts=None, vsel=None):
    from gipuma_b200 import api
    lib = api.load_library()
    po = api.GpmMsPriorOpts(None, C.pointer(geometric) if geometric else None)
    opts = opts or api.job_opts()
    rc = lib.gpm_ms_batch_run_restore(C.byref(m), C.byref(opts), C.byref(vsel) if vsel else None, C.byref(po),
                                      C.byref(restore) if restore else None, None)
    return rc, lib.gpm_batch_last_error().decode()


def _refused(rc, msg, *words):
    assert rc == E_ARG and msg.startswith("gpm_ms_batch_run_restore: bad arguments"), (rc, msg)
    for w in words:
        assert w in msg, (w, msg)


@pytest.mark.parametrize("kw,word", [(dict(photo_iterations=0), "photo_iterations must be >= 1"),
                                     (dict(photo_iterations=-3), "photo_iterations must be >= 1"),
                                     (dict(iterations=-1), "iterations must be >= 0"),
                                     (dict(threshold=float("nan")), "threshold must be finite"),
                                     (dict(threshold=float("inf")), "threshold must be finite"),
                                     (dict(threshold=float("-inf")), "threshold must be finite")],
                         ids=["photo_iterations_0", "photo_iterations_-3", "iterations_-1", "threshold_nan", "threshold_inf",
                              "threshold_-inf"])
def test_bad_restorer_options_are_refused_before_any_cuda_call(kw, word):
    m, _keep = _ms_desc()
    rc, msg = _run(m, _restore(**kw))
    _refused(rc, msg, "detail restorer", word)


@pytest.mark.parametrize("kw", [dict(levels=0), dict(radius=5), dict(channels=2), dict(weight=float("nan")),
                                dict(ref_indices=(C.c_int * 2)(0, 3))],
                         ids=["levels_0", "radius_5", "channels_2", "weight_nan", "ref_out_of_range"])
@pytest.mark.parametrize("with_restore", [False, True], ids=["restore_null", "restore"])
def test_what_gpm_ms_batch_run_prior_refuses_is_refused(kw, with_restore):
    m, _keep = _ms_desc(**kw)
    rc, msg = _run(m, _restore() if with_restore else None)
    _refused(rc, msg)


def test_a_bad_prior_stage_is_refused_with_the_restorer():
    m, _keep = _ms_desc()
    rc, msg = _run(m, _restore(), geometric=_stage(step=0))
    _refused(rc, msg, "geometric prior stage", "step")


def test_a_view_without_source_views_is_named_before_any_cuda_call():
    m, _keep = _ms_desc(min_angle=0.1, max_angle=0.2)
    rc, msg = _run(m, _restore())
    assert rc == E_STATE and msg.endswith("reference view 0"), (rc, msg)


@pytest.mark.parametrize("kw", [dict(), dict(photo_iterations=1, iterations=0, threshold=-1e30)])
def test_valid_options_pass_every_check(kw):
    m, _keep = _ms_desc(levels=3, width=128, height=96)
    rc, msg = _run(m, _restore(**kw), geometric=_stage())
    assert rc != E_ARG and rc != E_STATE, msg                 # runs on a GPU; without one it fails for want of a device


def test_gpm_set_geo_mask_refuses_a_null_context():
    from gipuma_b200 import api
    lib = api.load_library()
    mask = np.zeros(16, np.uint8)
    assert lib.gpm_set_geo_mask(None, C.c_void_p(mask.ctypes.data), 4, 0) == E_ARG
    assert "null context" in lib.gpm_last_error().decode()


# ---- multiscale_pass -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("restorer,word", [({"photo_iterations": 0}, "photo_iterations"), ({"photo_iterations": 1.5}, "photo_iterations"),
                                           ({"photo_iterations": True}, "photo_iterations"), ({"iterations": -1}, "iterations"),
                                           ({"iterations": "2"}, "iterations"), ({"threshold": float("nan")}, "threshold"),
                                           ({"threshold": float("inf")}, "threshold"), ({"threshold": None}, "threshold"),
                                           ({"threshold": {"pm": float("nan"), "ncc": 0.1}}, "threshold"),
                                           ({"threshold": 1e39}, "finite in float32"), ({"threshold": -1e39}, "finite in float32"),
                                           ({"threshold": 10 ** 400}, "finite in float32"),
                                           ({"photo_iterations": 2 ** 31}, "photo_iterations"), ({"iterations": 2 ** 40}, "iterations"),
                                           ({"thresold": 1.0}, "unknown")],
                         ids=["photo_iterations_0", "photo_iterations_float", "photo_iterations_bool", "iterations_-1",
                              "iterations_str", "threshold_nan", "threshold_inf", "threshold_none", "threshold_dict_nan",
                              "threshold_1e39", "threshold_-1e39", "threshold_huge_int", "photo_iterations_2^31",
                              "iterations_2^40", "unknown_key"])
def test_multiscale_pass_refuses_a_bad_restorer_before_loading_the_library(monkeypatch, restorer, word):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    with pytest.raises(ValueError, match=word):
        api.multiscale_pass(**_args(detail_restorer=restorer))


def test_a_threshold_dict_without_the_cost_in_use_is_refused_before_loading_the_library(monkeypatch):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    with pytest.raises(ValueError, match="no entry for photometric='ncc'"):
        api.multiscale_pass(**_args(detail_restorer={"threshold": {"pm": 2.0}}, photometric="ncc"))
    with pytest.raises(AssertionError, match="the library was reached"):        # the entry of the cost in use is enough
        api.multiscale_pass(**_args(detail_restorer={"threshold": {"ncc": 0.2}}, photometric="ncc"))


def test_the_largest_float32_threshold_passes():
    from gipuma_b200 import api
    from types import SimpleNamespace
    big = float(np.finfo(np.float32).max)
    o, _ = api.restore_opts({"threshold": -big}, SimpleNamespace(iterations=1), 1)
    assert o.threshold == -big


def test_multiscale_pass_refuses_zero_photo_iterations_from_the_parameters(monkeypatch):
    """photo_iterations defaults to params.iterations, and that default is checked too."""
    from gipuma_b200 import api
    _no_library(monkeypatch)
    a = _args(detail_restorer={})
    a["params"].iterations = 0
    with pytest.raises(ValueError, match="photo_iterations"):
        api.multiscale_pass(**a)


@pytest.mark.parametrize("restorer", [{}, {"threshold": -5.0, "iterations": 0, "photo_iterations": 3}, {"threshold": {"pm": 2.0}}])
def test_multiscale_pass_passes_a_valid_restorer_to_the_library(monkeypatch, restorer):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    with pytest.raises(AssertionError, match="the library was reached"):
        api.multiscale_pass(**_args(detail_restorer=restorer))


def test_restore_opts_fills_the_defaults():
    from gipuma_b200 import api
    from types import SimpleNamespace
    p = SimpleNamespace(iterations=5)
    for kind in ("pm", "ncc"):
        o, restored = api.restore_opts({}, p, 3, kind)
        assert (o.photo_iterations, o.iterations) == (5, api.RESTORE_DEFAULTS["iterations"])
        assert o.threshold == f32(api.RESTORE_DEFAULTS["threshold"][kind])
        assert len(restored) == 3
    assert api.restore_opts(None, p, 3) == (None, None)


# ---- oracle/pyrestore.py -------------------------------------------------------------------------------------------------

def test_equal_costs_give_no_detail_pixel():
    from oracle import pyrestore
    c = np.random.default_rng(1).uniform(0, 50, (7, 9)).astype(f32)
    assert not pyrestore.detect(c, c.copy(), 0.0).any()
    assert pyrestore.detect(c, c.copy(), -1e-30).all()


def test_the_comparison_is_strict():
    from oracle import pyrestore
    c_ph = f32([[1.0, 2.0, 3.0]])
    c_ms = f32([[1.5, 2.5, 3.25]])
    assert pyrestore.detect(c_ms, c_ph, 0.5).tolist() == [[0, 0, 0]]          # differences 0.5, 0.5, 0.25: none above 0.5
    assert pyrestore.detect(c_ms, c_ph, np.nextafter(f32(0.5), f32(0))).tolist() == [[1, 1, 0]]


def test_the_difference_is_rounded_once_in_float32():
    from oracle import pyrestore
    # 1 + 2^-23 - 1 is exact in float32, 2^-24 is not representable as a difference of these two in float64 terms either;
    # 16777217 (float64) - 1 = 16777216 in float32 because the cost itself is float32
    c_ms = f32([np.float32(1.0) + np.float32(2.0 ** -23)])
    c_ph = f32([1.0])
    assert pyrestore.detect(c_ms, c_ph, 2.0 ** -24).tolist() == [1]
    assert pyrestore.detect(c_ms, c_ph, 2.0 ** -23).tolist() == [0]
    big = f32([3.0e38]), f32([-3.0e38])                     # the float32 difference overflows to +inf
    assert pyrestore.detect(big[0], big[1], 1e38).tolist() == [1]


def test_nan_costs_are_never_detail_pixels():
    from oracle import pyrestore
    nan = f32(np.nan)
    c_ms = f32([nan, 5.0, nan, np.inf])
    c_ph = f32([0.0, nan, nan, np.inf])                      # inf - inf is NaN too
    assert pyrestore.detect(c_ms, c_ph, -1e30).tolist() == [0, 0, 0, 0]


def test_the_merge_takes_x_and_y_in_order_on_a_non_square_image():
    from oracle import pyrestore
    H, W = 3, 5
    ys, xs = np.mgrid[0:H, 0:W]
    ms = np.stack([xs, ys, np.zeros_like(xs), np.full_like(xs, 1)], -1).astype(f32)
    ph = np.stack([xs, ys, np.zeros_like(xs), np.full_like(xs, 2)], -1).astype(f32)
    detail = np.zeros((H, W), np.uint8)
    detail[2, 4] = detail[0, 3] = 1                         # (x 4, y 2) and (x 3, y 0)
    out = pyrestore.merge(ms, ph, detail)
    assert out.dtype == np.float32 and out.shape == (H, W, 4)
    assert (out[..., 3] == 2).sum() == 2 and out[2, 4, 3] == 2 and out[0, 3, 3] == 2
    assert (out[..., :2] == ms[..., :2]).all()              # x and y of every pixel are where they were


def test_the_masked_cost_is_a_per_pixel_select():
    from oracle import pyrestore
    on = f32([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]])
    off = f32([[-1.0, -2.0], [-3.0, -4.0], [-5.0, -6.0]])
    mask = np.uint8([[0, 7], [1, 0], [0, 255]])
    assert pyrestore.masked_cost(on, off, mask).tolist() == [[1.0, -2.0], [-3.0, 4.0], [5.0, -6.0]]
    assert (pyrestore.masked_cost(on, off, np.zeros_like(mask)) == on).all()
    assert (pyrestore.masked_cost(on, off, np.ones_like(mask)) == off).all()
