"""The coarse-to-fine scheme (DESIGN.md §19) without a GPU: known answers of the numpy restatement oracle/pyscale.py, the
header's struct layouts, and every argument refusal of multiscale_pass, Context.upsample_planes, gpm_downsample and
gpm_ms_batch_run, raised before any device is needed."""
import ctypes as C
import os
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import pyscale

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_ARG, E_STATE = -1, -3
f32 = np.float32


# ---- known answers of the restatement ------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(7, 9), (8, 10), (5, 6, 4)])
def test_constant_image_downsamples_to_itself(shape):
    img = np.full(shape, 37.25, f32)
    out = pyscale.downsample(img)
    assert out.shape == ((shape[0] + 1) // 2, (shape[1] + 1) // 2) + shape[2:]
    assert np.all(out == f32(37.25))


@pytest.mark.parametrize("W,H", [(9, 7), (10, 8), (1, 1), (2, 3), (1601, 1201)])
def test_sizes_round_up(W, H):
    assert pyscale.downsample(np.zeros((H, W), f32)).shape == ((H + 1) // 2, (W + 1) // 2)


def test_linear_ramp_is_sampled_at_even_pixels_away_from_the_border():
    H, W = 11, 14
    ys, xs = np.mgrid[0:H, 0:W]
    img = (3.0 * xs + 5.0 * ys + 1.0).astype(f32)          # exact in float32, and so is every filter step
    out = pyscale.downsample(img)
    yc, xc = np.mgrid[0:out.shape[0], 0:out.shape[1]]
    want = (3.0 * 2 * xc + 5.0 * 2 * yc + 1.0).astype(f32)
    inner = (2 * xc + 1 <= W - 1) & (2 * yc + 1 <= H - 1) & (xc > 0) & (yc > 0)
    assert np.array_equal(out[inner], want[inner])
    assert not np.array_equal(out[0, 1:], want[0, 1:])     # the replicated top border pulls row 0 towards the image


def _plane_scene(H=12, W=16, depth=5.0, tilt=0.1):
    """K_inv of a pinhole camera and the raw plane (n.xyz, d) n . X + d = 0 that a coarse level stores at every pixel."""
    K = np.array([[20.0, 0, W / 2], [0, 20.0, H / 2], [0, 0, 1]])
    Kinv = np.linalg.inv(K).astype(f32)
    n = np.array([tilt, -0.5 * tilt, -1.0])
    n /= np.linalg.norm(n)
    d = -n[2] * depth                                        # the plane through (0, 0, depth)
    coarse = np.tile(np.array([n[0], n[1], n[2], d], f32), ((H + 1) // 2, (W + 1) // 2, 1))
    return K, Kinv, coarse


@pytest.mark.parametrize("radius", [0, 2, 4])
def test_one_plane_is_reproduced(radius):
    H, W = 12, 16
    _, Kinv, coarse = _plane_scene(H, W)
    guide = np.random.default_rng(1).uniform(0, 255, (H, W)).astype(f32)
    planes, depth = pyscale.jbu(coarse, guide, Kinv, 1.0, 100.0, radius, 2.0, 10.0)
    ys, xs = np.mgrid[0:H, 0:W]
    r = np.stack([xs, ys, np.ones_like(xs)], -1).astype(np.float64) @ Kinv.astype(np.float64).T
    n = coarse[0, 0, :3].astype(np.float64)
    z = -coarse[0, 0, 3] / (r @ n)
    assert np.all(np.abs(depth - z) <= 8 * np.spacing(z.astype(f32)))
    assert np.all(np.abs(planes[..., :3] - coarse[0, 0, :3]) <= 4e-7)
    assert np.all(np.abs(planes[..., 3] - coarse[0, 0, 3]) <= 8 * np.spacing(abs(coarse[0, 0, 3])))


def test_unusable_candidates_are_skipped_and_the_fallback_is_c_with_no_depth():
    H, W = 10, 12
    _, Kinv, coarse = _plane_scene(H, W)
    bad = coarse.copy()
    bad[..., :] = 0.0                                        # all-zero planes: z = -0 / 0 = NaN
    bad[1, 2] = [np.nan, 0, -1, 3]
    bad[3, 3] = coarse[3, 3] * np.array([1, 1, 1, 1000], f32)  # depth x 1000: out of range
    bad[2, 4] = -coarse[2, 4]                                 # n and d negated: the same depth, in range
    guide = np.zeros((H, W), f32)
    planes, depth = pyscale.jbu(bad, guide, Kinv, 1.0, 100.0, 0, 2.0, 10.0)
    ys, xs = np.mgrid[0:H, 0:W]
    fallback = ~((ys >> 1 == 2) & (xs >> 1 == 4))
    assert np.all(depth[fallback] == 0)
    assert np.array_equal(planes[fallback].view(np.uint32), bad[ys >> 1, xs >> 1][fallback].view(np.uint32))
    assert np.all(depth[~fallback] > 0)
    # a behind-camera plane (z < 0) and an out-of-range one are skipped; with radius 1 the neighbours' good plane is used
    only = np.zeros_like(coarse)
    only[2, 4] = coarse[2, 4]
    only[2, 3] = coarse[2, 3] * np.array([1, 1, 1, -1], f32)          # behind the camera
    planes1, depth1 = pyscale.jbu(only, guide, Kinv, 1.0, 100.0, 1, 2.0, 10.0)
    assert np.all(depth1[4:6, 6:10] > 0)
    assert np.all(np.abs(planes1[4:6, 6:10, :3] - coarse[2, 4, :3]) <= 4e-7)


def test_a_guide_edge_keeps_the_other_sides_plane_out_within_the_cauchy_bound():
    H, W = 16, 16
    _, Kinv, near = _plane_scene(H, W, depth=5.0, tilt=0.0)
    _, _, far = _plane_scene(H, W, depth=9.0, tilt=0.0)
    coarse = near.copy()
    coarse[:, 4:] = far[:, 4:]                                # coarse columns >= 4 (fine x >= 8) are far
    guide = np.where(np.arange(W)[None, :] >= 8, 200.0, 0.0).astype(f32).repeat(H, 0)
    sr = 5.0
    _, depth = pyscale.jbu(coarse, guide, Kinv, 1.0, 100.0, 2, 4.0, sr)
    bound = 1.0 / (1.0 + 200.0 ** 2 / sr ** 2)                # largest range weight across the edge
    # x = 6, 7 (near side, c.x = 3): at most 25 far candidates of range weight <= bound against c's own of range weight 1
    ws = pyscale.spatial_table(4.0)
    for x in (6, 7):
        share = (depth[:, x] - 5.0) / (9.0 - 5.0)
        assert np.all(share >= -1e-6) and np.all(share <= 25 * bound / ws[:, :, 4, 4].min() + 1e-6)
        assert np.any(share > 0)                              # the far side does leak in, within the bound
    assert np.all(np.abs(depth[:, 12:] - 9.0) <= 1e-5 * 9)   # every candidate far: the far plane


def test_colour_guide_uses_xyz_only():
    H, W = 8, 8
    _, Kinv, near = _plane_scene(H, W, depth=5.0, tilt=0.0)
    _, _, far = _plane_scene(H, W, depth=9.0, tilt=0.0)
    coarse = near.copy()
    coarse[:, 2:] = far[:, 2:]
    g = np.random.default_rng(3).uniform(0, 255, (H, W, 4)).astype(f32)
    g2 = g.copy()
    g2[..., 3] = 0
    a = pyscale.jbu(coarse, g, Kinv, 1.0, 100.0, 2, 2.0, 10.0)
    b = pyscale.jbu(coarse, g2, Kinv, 1.0, 100.0, 2, 2.0, 10.0)
    assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))


# ---- struct layouts ------------------------------------------------------------------------------------------------------

def test_struct_layouts_match_ctypes(tmp_path):
    from gipuma_b200 import api
    fields = {"gpm_jbu_params": ["radius", "sigma_space", "sigma_range"],
              "gpm_ms_batch_desc": ["geo", "levels", "jbu"],
              "gpm_ms_batch_stats": ["batch", "n_views", "views", "level_sweep_ms", "level_upsample_ms"]}
    lines = ['printf("%%zu\\n", sizeof(%s));' % s + "".join(' printf("%%zu\\n", offsetof(%s, %s));' % (s, f) for f in fs)
             for s, fs in fields.items()]
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%%d\\n", '
                   'GPM_MS_MAX_LEVELS); %s return 0; }\n' % " ".join(lines))
    exe = str(tmp_path / "s")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = [api.MS_MAX_LEVELS]
    for cls, fs in ((api.GpmJbuParams, fields["gpm_jbu_params"]), (api.GpmMsBatchDesc, fields["gpm_ms_batch_desc"]),
                    (api.GpmMsBatchStats, fields["gpm_ms_batch_stats"])):
        want += [C.sizeof(cls)] + [getattr(cls, f).offset for f in fs]
    assert got == want


# ---- refusals ------------------------------------------------------------------------------------------------------------

def _no_library(monkeypatch):
    from gipuma_b200 import api

    def no_library(*a, **k):
        raise AssertionError("the library was reached with arguments that must be refused")
    monkeypatch.setattr(api, "load_library", no_library)


@pytest.mark.parametrize("kw", [dict(levels=0), dict(levels=5), dict(levels=2.5), dict(levels=4),
                                dict(jbu=dict(radius=-1)), dict(jbu=dict(radius=5)), dict(jbu=dict(sigma_space=0.0)),
                                dict(jbu=dict(sigma_range=float("nan"))), dict(jbu=dict(sigma=1.0)),
                                dict(weight=-0.1), dict(max_err=0.0), dict(refs=[3]), dict(refs=[]), dict(geo_iterations=-1),
                                dict(geo_iterations=1.5), dict(images=np.zeros((3, 48, 64, 3), np.float32)),
                                dict(Ps=[np.eye(3, 4)] * 2), dict(max_views=0), dict(photometric="ncc", view_selection="joint",
                                images=np.zeros((3, 48, 64, 4), np.float32)), dict(view_selection="joint")],
                         ids=["levels_0", "levels_5", "levels_2.5", "coarsest_8x6", "radius_-1", "radius_5", "sigma_space_0",
                              "sigma_range_nan", "unknown_jbu_key", "weight", "max_err", "ref_out_of_range", "no_refs",
                              "geo_iterations_-1", "geo_iterations_1.5", "three_channels", "too_few_Ps", "max_views_0",
                              "jvs_colour", "jvs_pm"])
def test_multiscale_pass_refuses_bad_arguments_before_loading_the_library(monkeypatch, kw):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    args = dict(images=np.zeros((3, 48, 64), np.float32), Ps=[np.eye(3, 4)] * 3, params=SimpleNamespace(iterations=1), refs=[0],
                levels=3)
    args.update(kw)
    with pytest.raises(ValueError):
        api.multiscale_pass(**args)


@pytest.mark.parametrize("kw", [dict(radius=-1), dict(radius=5), dict(sigma_space=0.0), dict(sigma_space=float("nan")),
                                dict(sigma_range=0.0), dict(sigma_range=float("nan")), dict(shape=(5, 8, 4))])
def test_upsample_planes_refuses_bad_arguments_before_any_device(monkeypatch, kw):
    from gipuma_b200 import api
    _no_library(monkeypatch)
    ctx = object.__new__(api.Context)                        # a context's Python side without a device behind it
    ctx.W, ctx.H, ctx.h, ctx.lib = 16, 12, None, None
    coarse = np.zeros(kw.pop("shape", (6, 8, 4)), np.float32)
    with pytest.raises(ValueError):
        ctx.upsample_planes(coarse, **kw)


@pytest.mark.parametrize("args", [dict(src=None), dict(dst=None), dict(width=0), dict(height=0), dict(channels=3),
                                  dict(channels=2), dict(pitch_bytes=12), dict(pitch_bytes=66)])
def test_downsample_refuses_bad_arguments_before_any_cuda_call(args):
    from gipuma_b200 import api
    lib = api.load_library()
    img, out = np.zeros((6, 4), np.float32), np.zeros((3, 2), np.float32)
    a = dict(device=0, src=img.ctypes.data, pitch_bytes=0, width=4, height=6, channels=1, dst=out.ctypes.data, on_device=0)
    a.update(args)
    rc = lib.gpm_downsample(a["device"], a["src"], a["pitch_bytes"], a["width"], a["height"], a["channels"], a["dst"], a["on_device"])
    assert rc == E_ARG and lib.gpm_last_error().decode().startswith("gpm_downsample")


def _ms_desc(levels=2, radius=2, sigma_space=2.0, sigma_range=10.0, width=96, height=64, **kw):
    """A valid descriptor over 3 DTU cameras (grey), then the fields of `kw` overwritten."""
    from gipuma_b200 import api, scene as S
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N)
    params.depthMin, params.depthMax = 300.0, 800.0
    Ps = [S.load_dtu_projections()[i] for i in range(3)]
    imgs = np.zeros((3, height, width), np.float32)
    d, keep = api._batch_desc(imgs, Ps, params, [0, 2], (0,), 1600.0 / width, 5.0, 45.0, 2, 7, None, None, None)
    m = api.GpmMsBatchDesc(api.GpmGeoBatchDesc(d, 1, 1, 0.5, 3.0), levels, api.GpmJbuParams(radius, sigma_space, sigma_range))
    for name, value in kw.items():
        setattr(m.geo.batch if hasattr(m.geo.batch, name) else m.geo, name, value)
    return m, keep


def _ms_run(m):
    from gipuma_b200 import api
    lib = api.load_library()
    opts = api.job_opts()
    rc = lib.gpm_ms_batch_run(C.byref(m) if m is not None else None, C.byref(opts), None, None)
    return rc, lib.gpm_batch_last_error().decode()


@pytest.mark.parametrize("kw", [dict(levels=0), dict(levels=5), dict(levels=4, width=64, height=48), dict(radius=-1),
                                dict(radius=5), dict(sigma_space=0.0), dict(sigma_range=float("nan")), dict(images=None),
                                dict(channels=2), dict(geo_iterations=-1), dict(weight=float("nan")), dict(max_err=0.0),
                                dict(max_views=65), dict(n_devices=0), dict(ref_indices=(C.c_int * 2)(0, 3)),
                                dict(ref_indices=(C.c_int * 2)(2, 2), out_dir=b"unused")],
                         ids=["levels_0", "levels_5", "coarsest_8x6", "radius_-1", "radius_5", "sigma_space_0", "sigma_range_nan",
                              "null_images", "channels_2", "geo_iterations_-1", "weight_nan", "max_err_0", "max_views_65",
                              "n_devices_0", "ref_out_of_range", "repeated_ref_with_out_dir"])
def test_ms_batch_run_refuses_bad_descriptors_before_any_cuda_call(kw):
    m, _keep = _ms_desc(**kw)
    rc, msg = _ms_run(m)
    assert rc == E_ARG and msg.startswith("gpm_ms_batch_run: bad arguments"), (rc, msg)


def test_ms_batch_run_accepts_the_smallest_coarsest_level():
    m, _keep = _ms_desc(levels=4, width=64, height=57)        # 8 x 8 at level 3
    rc, msg = _ms_run(m)
    assert rc != E_ARG, msg                                   # runs on a GPU; without one it fails for want of a device


def test_ms_batch_run_refuses_a_null_descriptor():
    rc, msg = _ms_run(None)
    assert rc == E_ARG and "bad arguments" in msg


def test_ms_batch_run_names_a_view_without_source_views_before_any_cuda_call():
    m, _keep = _ms_desc(min_angle=0.1, max_angle=0.2)
    rc, msg = _ms_run(m)
    assert rc == E_STATE and msg.endswith("reference view 0"), (rc, msg)
