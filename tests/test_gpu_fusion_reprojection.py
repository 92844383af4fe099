"""The reprojection rule of the depth-map fusion on the GPU (gpm_fuse_with_rule, DESIGN.md §22): equal bit for bit to the C
restatement (oracle/fusion_rule_oracle.c) on PatchMatch outputs and on ground truth at several thresholds, in grey and RGBA;
independent of where its inputs live and of any live PatchMatch context; unchanged in its decisions by a change of the
world's scale; and at the DTU size."""
import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

FUSE = dict(depth_min=300.0, depth_max=800.0, disp_thresh=0.1, normal_thresh=30.0, num_consistent=2, rule="reprojection",
            reproj_px=2.0, depth_rel=0.01)
REFS = list(range(0, 24, 3))
SETTINGS = [dict(), dict(reproj_px=1.0, depth_rel=0.005, normal_thresh=10.0, num_consistent=3),
            dict(reproj_px=4.0, depth_rel=0.02, num_consistent=1), dict(reproj_px=0.5, depth_rel=0.05, num_consistent=2)]


def _dataset(rows=96, cols=128, n_cams=24):
    """Images of the first `n_cams` DTU positions looking at one height field (world = frame of camera 0)."""
    from gipuma_b200 import scene as S
    Ps = [S.load_dtu_projections()[i] for i in range(n_cams)]
    scale = 1600.0 / cols
    cams = S.prepare_cameras(Ps, scale)
    hf = S.HeightField(z0=550.0, unit=550.0 / cams[0].fx, seed=77)
    images = np.stack([S.render_view(c, rows, cols, hf)[0] for c in cams])
    return Ps, scale, images, hf


@pytest.fixture(scope="module")
def batch(tmp_path_factory):
    """PatchMatch outputs of the reference views REFS (in memory and as the batch driver's .dmb directory) and their
    ground truth."""
    from gipuma_b200 import api, scene as S
    Ps, scale, images, hf = _dataset()
    p = S.AlgorithmParameters(box_hsize=11, box_vsize=11, iterations=3, n_best=3, cost_comb=S.COMB_BEST_N, gamma=10.0)
    p.depthMin, p.depthMax = 300.0, 800.0
    out_dir = str(tmp_path_factory.mktemp("batch"))
    n4, _, _ = api.batch_run(images, Ps, p, REFS, cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242,
                             out_dir=out_dir)
    fPs = [Ps[r] for r in REFS]
    gt = S.render_norm4(fPs, scale, images.shape[1], images.shape[2], hf)
    return dict(Ps=Ps, scale=scale, images=images, hf=hf, n4=n4, gt=gt, out_dir=out_dir, fPs=fPs)


def _oracle(n4, Ps, scale, images=None, **kw):
    from gipuma_b200 import api
    from oracle import pyfusion_rule
    args = dict(FUSE, **kw)
    return pyfusion_rule.fuse(n4, api.fuse_cameras(Ps, scale), images=images, threads=8, **args)


def _same(v, info, ov, osrc, oused):
    assert len(v) == len(ov) and info["count"] == len(ov)
    assert np.array_equal(info["source"], osrc)
    assert v.tobytes() == ov.tobytes()
    assert np.array_equal(info["used"], oused)


def _surface_error(hf, Ps, v):
    """Height of each vertex above the height field, in the frame re-based on camera 0."""
    from gipuma_b200 import scene as S
    R0, t0 = S.ref0_frame(Ps)
    X = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float64) @ R0.T + t0
    return X[:, 2] - hf.height(X[:, 0], X[:, 1])


@pytest.mark.parametrize("maps", ["n4", "gt"])
@pytest.mark.parametrize("setting", range(len(SETTINGS)))
def test_gpu_reprojection_rule_equals_the_c_restatement(batch, maps, setting):
    from gipuma_b200 import api
    kw = dict(FUSE, **SETTINGS[setting])
    v, info = api.fuse(batch[maps], batch["fPs"], cam_scale=batch["scale"], **kw)
    _same(v, info, *_oracle(batch[maps], batch["fPs"], batch["scale"], **kw))
    assert len(v) > 100
    err = np.abs(_surface_error(batch["hf"], batch["fPs"], v)) / batch["hf"].z0
    print("%s, %s: %d vertices, %.4f within 0.5 %% of depth, max %.2g z0" % (maps, SETTINGS[setting], len(v),
                                                                           (err < 0.005).mean(), err.max()))


@pytest.mark.parametrize("colour", ["grey", "rgba"])
def test_gpu_reprojection_rule_colour_equals_the_c_restatement(batch, colour):
    from gipuma_b200 import api
    g = batch["images"][REFS]
    imgs = np.ascontiguousarray(g if colour == "grey" else
                                np.stack([g, 255.0 - g, 0.5 * g, np.full_like(g, 99.0)], axis=-1), dtype=np.float32)
    v, info = api.fuse(batch["n4"], batch["fPs"], images=imgs, cam_scale=batch["scale"], **FUSE)
    _same(v, info, *_oracle(batch["n4"], batch["fPs"], batch["scale"], images=imgs))
    assert (v["red"] != 0).any()


def test_gpu_reprojection_rule_is_the_same_for_host_device_and_dmb_inputs(batch, tmp_path):
    import torch
    from gipuma_b200 import api
    imgs = np.ascontiguousarray(batch["images"][REFS])
    v1, i1 = api.fuse(batch["n4"], batch["fPs"], images=imgs, cam_scale=batch["scale"], **FUSE)
    v2, i2 = api.fuse(torch.from_numpy(batch["n4"]).cuda(), batch["fPs"], images=torch.from_numpy(imgs).cuda(),
                      cam_scale=batch["scale"], **FUSE)
    assert i2["upload_ms"] == 0.0
    api.write_ply(str(tmp_path / "a.ply"), v1)
    api.write_ply(str(tmp_path / "b.ply"), v2)
    assert open(tmp_path / "a.ply", "rb").read() == open(tmp_path / "b.ply", "rb").read()
    assert np.array_equal(i2["source"], i1["source"]) and np.array_equal(i2["used"], i1["used"])
    v3, i3 = api.fuse_batch_dir(batch["out_dir"], REFS, batch["Ps"], images=batch["images"], cam_scale=batch["scale"], **FUSE)
    assert v3.tobytes() == v1.tobytes() and np.array_equal(i3["source"], i1["source"])


def test_gpu_reprojection_rule_leaves_a_live_context_untouched(batch):
    from gipuma_b200 import api, scene as S
    sc = S.make_config(1, rows=64, cols=96)
    with api.Context(sc.cols, sc.rows, sc.n_views) as ctx:
        ctx.load_scene(sc)
        ctx.run()
        a4, ac = ctx.get_state()
        api.fuse(batch["n4"], batch["fPs"], cam_scale=batch["scale"], **FUSE)
        ctx.run()
        b4, bc = ctx.get_state()
    assert bits_equal(a4, b4) == 0 and bits_equal(ac, bc) == 0


@pytest.mark.parametrize("maps", ["n4", "gt"])
def test_gpu_reprojection_rule_does_not_depend_on_the_worlds_scale(batch, maps):
    """The world times s = 2^-10 (P's fourth column, the depths, the depth range): the reprojection rule gives the same
    sources and masks, positions times s bit for bit, the same normals and colours.  The disparity rule, at the same
    disp_thresh, does not."""
    from gipuma_b200 import api
    s = 2.0 ** -10
    sPs = [np.hstack([np.asarray(P, np.float64)[:, :3], np.asarray(P, np.float64)[:, 3:] * s]) for P in batch["fPs"]]
    n4 = batch[maps]
    sn4 = n4.copy()
    sn4[..., 3] *= np.float32(s)
    imgs = np.ascontiguousarray(batch["images"][REFS])
    srange = dict(depth_min=FUSE["depth_min"] * s, depth_max=FUSE["depth_max"] * s)
    v, i = api.fuse(n4, batch["fPs"], images=imgs, cam_scale=batch["scale"], **FUSE)
    sv, si = api.fuse(sn4, sPs, images=imgs, cam_scale=batch["scale"], **dict(FUSE, **srange))
    assert len(v) > 500 and np.array_equal(si["source"], i["source"]) and np.array_equal(si["used"], i["used"])
    for k in ("x", "y", "z"):
        assert np.array_equal(sv[k].view(np.uint32), (v[k] * np.float32(s)).view(np.uint32))
    for k in ("nx", "ny", "nz", "red", "green", "blue"):
        assert np.array_equal(sv[k], v[k])
    d = dict(FUSE, rule="disparity", reproj_px=None, depth_rel=None)
    dv, di = api.fuse(n4, batch["fPs"], cam_scale=batch["scale"], **d)
    sdv, sdi = api.fuse(sn4, sPs, cam_scale=batch["scale"], **dict(d, **srange))
    print("%s: reprojection %d vertices at both scales; disparity %d -> %d" % (maps, len(v), len(dv), len(sdv)))
    assert not np.array_equal(sdi["source"], di["source"])


def test_gpu_reprojection_rule_at_dtu_size():
    """49 DTU cameras at 1600x1200, ground truth maps: the first passes must equal the restatement exactly, and on a seeded
    sample of later reference views every vertex must be the restatement's candidate of its pixel, and every candidate
    the GPU did not emit must have been marked by an earlier pass."""
    from gipuma_b200 import api, scene as S
    from oracle import pyfusion_rule
    Ps = [S.load_dtu_projections()[i] for i in range(49)]
    H, W = 1200, 1600
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1])[0].fx, seed=77)
    gt = S.render_norm4(Ps, 1.0, H, W, hf)
    prm = dict(FUSE, num_consistent=3)
    v, info = api.fuse(gt, Ps, **prm)
    cams = api.fuse_cameras(Ps)
    src = info["source"]
    print("DTU size, reprojection rule: %d vertices, fusion %.1f ms, upload %.1f ms" % (len(v), info["fuse_ms"], info["upload_ms"]))
    ov, osrc, _ = pyfusion_rule.fuse(gt, cams, refs=(0, 2), threads=32, **prm)
    k = int((src[:, 0] < 2).sum())
    assert k == len(ov) and np.array_equal(src[:k], osrc) and v[:k].tobytes() == ov.tobytes()
    for r in np.random.default_rng(2026).choice(np.arange(2, 49), 3, replace=False):
        cv, csrc, _ = pyfusion_rule.fuse(gt, cams, refs=(int(r), int(r) + 1), threads=32, **prm)
        mine = src[:, 0] == r
        pos = np.searchsorted(csrc[:, 1], src[mine, 1])
        assert (pos < len(csrc)).all() and np.array_equal(csrc[pos, 1], src[mine, 1])
        assert v[mine].tobytes() == cv[pos].tobytes()
        missed = np.setdiff1d(csrc[:, 1], src[mine, 1])
        assert info["used"][r].reshape(-1)[missed].all()
    # the disparity rule's vertices here lie up to 4.9e-3 z0 off the surface (test_gpu_fusion_at_dtu_size): a consistent
    # pixel may show another surface point at a similar depth.  The reprojection rule asks the target's point to land back
    # on the reference pixel: in the restatement's run of all 49 passes (5,098,710 vertices) every vertex lies within
    # 4.3e-5 z0 of the surface
    err = np.abs(_surface_error(hf, Ps, v)) / hf.z0
    print("DTU size, reprojection rule: %.5f of the vertices within 1e-3 z0 of the surface, max %.2g z0 "
          "(disparity rule: 0.996 and 4.9e-3 z0)" % ((err < 1e-3).mean(), err.max()))
    assert err.max() < 5e-5
