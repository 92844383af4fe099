"""Depth-map fusion (DESIGN.md §12) without a GPU: the C restatement on hand-made scenes with known answers, the fusion's
cameras, the PLY writer / reader, and the refusal of bad descriptors before any CUDA call."""
import ctypes as C
import os
import subprocess

import numpy as np

F, W, H, Z0 = 100.0, 40, 24, 10.0          # focal length, image size, plane depth


def _P(cx_world, f=F):
    """Camera with R = I at (cx_world, 0, 0), principal point at the image centre."""
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1.0]])
    return K @ np.hstack([np.eye(3), np.array([[-cx_world], [0.0], [0.0]])])


def _plane(n_views, normal=(0.0, 0.0, -1.0)):
    """Every camera looks down +z at the plane z = Z0: depth Z0 everywhere, normal facing the cameras."""
    n4 = np.zeros((n_views, H, W, 4), np.float32)
    n4[..., :3] = normal
    n4[..., 3] = Z0
    return n4


# camera 1 sits 0.5 to the right: a plane point seen at column x in view 0 is at column x - 5 in view 1
SHIFT = 5
PS2 = [_P(0.0), _P(0.5)]
ARGS = dict(depth_min=1.0, depth_max=100.0, disp_thresh=0.1, normal_thresh=30.0)


def _fuse(n4, Ps, num_consistent=1, **kw):
    from gipuma_b200 import api
    from oracle import pyfusion
    args = dict(ARGS, **{k: kw.pop(k) for k in list(kw) if k in ARGS})
    return pyfusion.fuse(n4, api.fuse_cameras(Ps), num_consistent=num_consistent, **args, **kw)


def test_fusion_cameras_are_the_un_rebased_projections():
    from gipuma_b200 import api, scene as S
    Ps = [S.load_dtu_projections()[i] for i in (0, 9, 30)]
    for P, c in zip(Ps, api.fuse_cameras(Ps, 4.0)):
        K, R, Cc = S.decompose_projection(P)
        K = S.scale_K(K / K[2, 2], 4.0)
        want = K @ np.hstack([R, (-R @ Cc)[:, None]])
        got = np.array(c.P[:], dtype=np.float64).reshape(3, 4)
        assert np.allclose(got, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
        assert np.allclose(np.array(c.M_inv[:]).reshape(3, 3) @ want[:, :3], np.eye(3), atol=1e-5)
        assert c.f == np.float32(K[0, 0])


def test_two_cameras_on_a_plane_fuse_every_overlapping_pixel():
    verts, src, used = _fuse(_plane(2), PS2)
    xs = src[:, 1] % W
    assert len(verts) == H * (W - SHIFT)                       # view 0's columns SHIFT.. see the plane in view 1
    assert (src[:, 0] == 0).all() and (xs >= SHIFT).all()
    assert np.array_equal(src[:, 1], np.sort(src[:, 1]))       # (view, y, x) order
    assert used[0, :, SHIFT:].all() and not used[0, :, :SHIFT].any()
    assert used[1, :, :W - SHIFT].all() and not used[1, :, W - SHIFT:].any()
    ys = src[:, 1] // W
    assert np.allclose(verts["x"], (xs - W / 2) * Z0 / F, atol=1e-4) and np.allclose(verts["y"], (ys - H / 2) * Z0 / F, atol=1e-4)
    assert np.allclose(verts["z"], Z0, atol=1e-5) and (verts["nz"] == -1.0).all()
    assert (verts["red"] == 0).all()                           # no images: black


def test_too_few_other_views_gives_no_vertex():
    verts, _, used = _fuse(_plane(3), PS2 + [_P(-0.5)], num_consistent=3)       # N - 1 = 2 < 3
    assert len(verts) == 0 and not used.any()


def test_a_view_off_by_more_than_disp_thresh_contributes_nothing():
    n4 = _plane(3)
    n4[2, ..., 3] = Z0 * 1.3                                   # view 2 disagrees: disparity 5.4 vs 4.15 px
    Ps = PS2 + [_P(-0.5)]
    verts, src, used = _fuse(n4, Ps, refs=(0, 1))
    v2, s2, _ = _fuse(_plane(2), PS2, refs=(0, 1))
    assert not used[2].any()
    assert np.array_equal(src, s2) and verts.tobytes() == v2.tobytes()


def test_a_flipped_normal_is_rejected():
    n4 = _plane(2)
    n4[1, ..., :3] *= -1
    verts, _, used = _fuse(n4, PS2)
    assert len(verts) == 0 and not used.any()
    n4[1, ..., :3] = (0.0, np.sin(np.radians(25.0)), -np.cos(np.radians(25.0)))    # 25 degrees apart: still consistent
    assert len(_fuse(n4, PS2)[0]) == H * (W - SHIFT)


def test_marks_apply_from_the_next_pass():
    """A mark stops a pixel from being a reference in later passes only: the targets' masks never change the current pass."""
    Ps = PS2 + [_P(1.0)]
    v0, s0, u0 = _fuse(_plane(3), Ps, refs=(0, 1))
    pre = np.zeros((3, H, W), np.uint8)
    pre[1:] = 1
    v1, s1, u1 = _fuse(_plane(3), Ps, refs=(0, 1), used=pre)   # every target already marked: pass 0 unchanged
    assert v0.tobytes() == v1.tobytes() and np.array_equal(s0, s1)
    assert np.array_equal(u1[0], u0[0])
    # all passes: views 1 and 2 only add pixels view 0 did not mark
    v, s, u = _fuse(_plane(3), Ps)
    assert v[: len(v0)].tobytes() == v0.tobytes()
    later = s[len(v0):]
    assert len(later) > 0 and not u0[later[:, 0], later[:, 1] // W, later[:, 1] % W].any()
    assert u.sum() >= u0.sum()


def test_grey_and_rgba_colour_is_the_rounded_mean():
    n4 = _plane(2)
    grey = np.zeros((2, H, W), np.float32)
    grey[0], grey[1] = 100.0, 103.0                            # mean 101.5 -> 102 (half up)
    verts, _, _ = _fuse(n4, PS2, images=grey)
    assert (verts["red"] == 102).all() and (verts["green"] == 102).all() and (verts["blue"] == 102).all()
    rgba = np.zeros((2, H, W, 4), np.float32)
    rgba[0] = (10.0, 300.0, -5.0, 77.0)
    rgba[1] = (20.0, 300.0, -5.0, 77.0)
    verts, _, _ = _fuse(n4, PS2, images=rgba)
    assert (verts["red"] == 15).all() and (verts["green"] == 255).all() and (verts["blue"] == 0).all()


def test_ply_round_trip_and_header(tmp_path):
    from gipuma_b200 import api
    rng = np.random.default_rng(5)
    v = np.zeros(17, dtype=api.PLY_VERTEX)
    for k in ("x", "y", "z", "nx", "ny", "nz"):
        v[k] = rng.normal(size=17).astype(np.float32)
    for k in ("red", "green", "blue"):
        v[k] = rng.integers(0, 256, 17)
    path = str(tmp_path / "cloud.ply")
    api.write_ply(path, v)
    header = (b"ply\nformat binary_little_endian 1.0\nelement vertex 17\nproperty float x\nproperty float y\n"
              b"property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
              b"property uchar green\nproperty uchar blue\nend_header\n")
    data = open(path, "rb").read()
    assert data == header + v.tobytes() and len(data) == len(header) + 17 * 27
    assert api.read_ply(path).tobytes() == v.tobytes()
    api.write_ply(path, v[:0])
    assert len(api.read_ply(path)) == 0


def test_bad_descriptors_are_refused_before_any_cuda_call():
    from gipuma_b200 import api
    lib = api.load_library()
    n4 = _plane(2)
    P = np.ascontiguousarray(np.stack(PS2).reshape(-1))

    def call(**kw):
        d = api.GpmFuseDesc(2, W, H, n4.ctypes.data, None, 0, 0, P.ctypes.data_as(C.POINTER(C.c_double)), 1.0,
                            1.0, 100.0, 0.1, 30.0, 1, 0)
        for k, v in kw.items():
            setattr(d, k, v)
        r = api.GpmFuseResult(0, 0, None, None, None, 0.0, 0.0)
        return lib.gpm_fuse(C.byref(d), C.byref(r)), lib.gpm_last_error().decode()

    for bad in (dict(n_views=1), dict(P=None), dict(norm4=None), dict(disp_thresh=0.0), dict(disp_thresh=-1.0),
                dict(normal_thresh=0.0), dict(normal_thresh=200.0), dict(num_consistent=0), dict(depth_max=0.5),
                dict(cam_scale=0.0), dict(images=n4.ctypes.data, channels=3), dict(width=0)):
        rc, msg = call(**bad)
        assert rc == -1 and msg.startswith("gpm_fuse:"), (bad, rc, msg)
    from conftest import have_cuda
    if not have_cuda():
        rc, msg = call()                                       # a valid descriptor needs a device: no CPU path
        assert rc == -2, msg


def test_fusion_struct_layouts_match_ctypes(tmp_path):
    from gipuma_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%zu %zu %zu %zu %zu\\n", '
                   'sizeof(gpm_fuse_camera), sizeof(gpm_fuse_desc), sizeof(gpm_fuse_result), offsetof(gpm_fuse_desc, device), '
                   'offsetof(gpm_fuse_result, upload_ms)); return 0; }\n')
    exe = str(tmp_path / "t")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(root, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.GpmFuseCamera), C.sizeof(api.GpmFuseDesc), C.sizeof(api.GpmFuseResult),
                   api.GpmFuseDesc.device.offset, api.GpmFuseResult.upload_ms.offset]
