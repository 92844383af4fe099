"""The float64 references of oracle/pyrecon64.py against the C restatements, without a GPU: the fusion's first pass under
both rules on hand-made rigs and a rendered scene, TSDF integration, and the marching-tetrahedra vertices.  The GPU
files check the kernels against the same references (tests/test_gpu_fusion_edges.py, tests/test_gpu_mesh_edges.py)."""
import numpy as np
import pytest

F, W, H, Z0 = 100.0, 40, 24, 10.0
RULES = [("disparity", dict(disp_thresh=0.1)), ("reprojection", dict(reproj_px=1.0, depth_rel=0.01))]


def _P(C, f=F, w=W, h=H, R=np.eye(3)):
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1.0]])
    return K @ np.hstack([R, (-R @ np.asarray(C, np.float64))[:, None]])


def _plane(n, h=H, w=W):
    n4 = np.zeros((n, h, w, 4), np.float32)
    n4[..., :3] = (0.0, 0.0, -1.0)
    n4[..., 3] = Z0
    return n4


def _restated_first_pass(n4, Ps, rule, kw, num_consistent, images=None, **thr):
    from gipuma_b200 import api
    from oracle import pyfusion_rule
    args = dict(depth_min=1.0, depth_max=100.0, disp_thresh=kw.get("disp_thresh", 0.1), normal_thresh=30.0)
    args.update(thr)
    return pyfusion_rule.fuse(n4, api.fuse_cameras(Ps), num_consistent=num_consistent, images=images, refs=(0, 1), rule=rule,
                              reproj_px=kw.get("reproj_px", 2.0), depth_rel=kw.get("depth_rel", 0.01), **args)


def _float64_first_pass(n4, Ps, rule, kw, num_consistent, images=None, **thr):
    from gipuma_b200 import api
    from oracle import pyrecon64
    args = dict(depth_min=1.0, depth_max=100.0, normal_thresh=30.0)
    args.update(thr)
    return pyrecon64.first_pass(n4, api.fuse_cameras(Ps), num_consistent=num_consistent, images=images, rule=rule, **args,
                                **kw)


def _hand_made():
    """Planes seen by cameras shifted along x and y, one view at a disagreeing depth, one with noisy normals, an invalid
    patch, and random grey images."""
    rng = np.random.default_rng(4)
    Ps = [_P((0, 0, 0)), _P((0.5, 0, 0)), _P((-0.5, 0.3, 0)), _P((0.3, -0.2, 0))]
    n4 = _plane(4)
    n4[2, ..., 3] = Z0 * 1.001
    n4[3, ..., :3] += rng.normal(0, 0.3, (H, W, 3)).astype(np.float32)
    n4[0, 3:6, 5:9, 3] = 0.0
    grey = rng.integers(0, 256, (4, H, W)).astype(np.float32)
    return n4, Ps, grey


def _rendered(n_views=5, rows=45, cols=61):
    """synthetic_rig around a height field, rendered ground truth (invalid where the ray cast did not converge)."""
    from gipuma_b200 import scene as S
    K = np.array([[cols * 1.2, 0, cols / 2], [0, cols * 1.2, rows / 2], [0, 0, 1.0]])
    Ps = S.synthetic_rig(n_views - 1, K, 500.0, 5.0, 25.0, seed=3)
    cams = S.prepare_cameras(Ps)
    hf = S.HeightField(z0=500.0, unit=500.0 / cams[0].fx, seed=9)
    return S.render_norm4(Ps, 1.0, rows, cols, hf), Ps


@pytest.mark.parametrize("rule,kw", RULES)
@pytest.mark.parametrize("num_consistent", [1, 2])
def test_float64_first_pass_agrees_with_the_restatement_on_hand_made_rigs(rule, kw, num_consistent):
    from oracle import pyrecon64
    n4, Ps, grey = _hand_made()
    v, src, _ = _restated_first_pass(n4, Ps, rule, kw, num_consistent, images=grey)
    ref = _float64_first_pass(n4, Ps, rule, kw, num_consistent, images=grey)
    checked = pyrecon64.check_first_pass(ref, v, src, W, images=True)
    assert checked > 0.9 * H * W and ref["fused"].any() and not ref["fused"].all()


@pytest.mark.parametrize("rule,kw", [("disparity", dict(disp_thresh=0.1)), ("reprojection", dict(reproj_px=1.0, depth_rel=0.005))])
def test_float64_first_pass_agrees_with_the_restatement_on_a_rendered_scene(rule, kw):
    from oracle import pyrecon64
    n4, Ps = _rendered()
    v, src, _ = _restated_first_pass(n4, Ps, rule, kw, 2, depth_min=300.0, depth_max=800.0)
    ref = _float64_first_pass(n4, Ps, rule, kw, 2, depth_min=300.0, depth_max=800.0)
    checked = pyrecon64.check_first_pass(ref, v, src, n4.shape[2])
    assert checked > 0.9 * n4.shape[1] * n4.shape[2] and ref["fused"].sum() > 100 and not ref["fused"][ref["certain"]].all()


def test_the_float64_decisions_are_uncertain_exactly_on_an_edge():
    """A target depth on the disparity threshold's edge cannot be decided in float64; one well away from it can."""
    from gipuma_b200 import api
    from oracle import pyrecon64
    Ps = [_P((0, 0, 0)), _P((0.5, 0, 0))]
    n4 = _plane(2)
    fb = np.float32(F) * np.float32(0.54)
    z = np.float32(Z0)
    edge = np.float64(fb) / (np.float64(fb) / np.float64(z) - np.float64(np.float32(0.1)))
    n4[1, 0, :, 3] = np.float32(edge)
    n4[1, 1, :, 3] = np.float32(edge * 1.01)
    n4[1, 2, :, 3] = np.float32(edge * 0.99)
    dec = pyrecon64.fusion_decisions(n4, api.fuse_cameras(Ps), 0, 1.0, 100.0, 30.0, disp_thresh=0.1)
    row = lambda y: slice(y * W + 10, y * W + W)                      # columns whose target lies in the image
    assert not dec["certain"][1, row(0)].any()
    assert dec["certain"][1, row(1)].all() and not dec["ok"][1, row(1)].any()
    assert dec["certain"][1, row(2)].all() and dec["ok"][1, row(2)].all()


def _tsdf_rig():
    n4, Ps = _rendered(4)
    from gipuma_b200 import scene as S
    g = S.gt_points(Ps, 1.0, n4.shape[1], n4.shape[2], None, norm4=n4)
    lo, hi = g.min(axis=0), g.max(axis=0)
    voxel = float(np.float32((hi - lo).max() / 20))
    origin = tuple(float(np.float32(x)) for x in lo - 2 * voxel)
    return np.ascontiguousarray(n4[..., 3]), Ps, origin, voxel, (24, 23, 22)


@pytest.mark.parametrize("trunc_vox", [1.0, 3.0])
def test_float64_tsdf_agrees_with_the_restatement(trunc_vox):
    from gipuma_b200 import api
    from oracle import pymesh, pyrecon64
    dep, Ps, origin, voxel, dims = _tsdf_rig()
    dep[1, 5:9, 5:20] = np.float32("nan")
    dep[2, 10:12, :] = np.float32(-0.0)
    cams = api.fuse_cameras(Ps)
    trunc = trunc_vox * voxel
    D, Wt = pymesh.tsdf(dep, cams, origin, voxel, dims, trunc, 300.0, 800.0)
    ref = pyrecon64.tsdf(dep, cams, origin, voxel, dims, trunc, 300.0, 800.0)
    assert pyrecon64.check_tsdf(ref, D, Wt) > 0.99 * np.prod(dims)
    assert (Wt > 0).mean() > 0.05 and (D[Wt > 0] < 0).any() and (D[Wt > 0] > 0).any()


def test_float64_mesh_vertices_agree_with_the_restatement():
    from oracle import pymesh, pyrecon64
    n = (21, 19, 17)
    o, s = (-1.25, 0.5, 2.0), 0.37
    x, y, z = (np.float32(o[a]) + (np.arange(n[a], dtype=np.float32) + np.float32(0.5)) * np.float32(s) for a in range(3))
    Z, Y, X = np.meshgrid(z, y, x, indexing="ij")
    D = (np.sqrt((X - 2.2) ** 2 + (Y - 3.9) ** 2 + (Z - 5.1) ** 2) - 2.4).astype(np.float32)
    D[3, 4, 5] = np.float32(-0.0)
    v, f = pymesh.extract(D, np.ones(D.shape, np.uint16), o, s, 1)
    assert pyrecon64.check_mesh_vertices(D, o, s, v) > 100
