"""Nearest-neighbour distances on the GPU (gpm_nearest_dist, DESIGN.md §13): equal bit for bit to the brute-force
restatement on adversarial sets and to the certified restatement at 10^6 points, deterministic, and, end to end, the scores
of fused clouds against the ground truth of the synthetic scenes."""
import numpy as np
import pytest

from oracle import pycloud

pytestmark = pytest.mark.gpu


def _check(q, b, max_dist, want=None):
    from gipuma_b200 import api
    q = np.ascontiguousarray(q, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    got, info = api.nearest_distance(q, b, max_dist)
    want = pycloud.brute(q, b, max_dist) if want is None else want
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert len(bad) == 0, "%d of %d differ, first %s: GPU %r, restatement %r (cell %g)" % (
        len(bad), len(q), bad[:3], got[bad[:3]], want[bad[:3]], info["cell_size"])
    return got, info


def _lattice(n, step=1.0):
    g = np.arange(n + 1, dtype=np.float32) * np.float32(step)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3)


def test_lattice_on_cell_boundaries_and_one_ulp_either_side():
    # a 17^3 lattice of step 1 spanning 16 with max_dist 16: the cell size is exactly 1 (min(max_dist, extent) / 16), so
    # every lattice coordinate is a cell boundary; the copies one ulp below and above straddle it
    L = _lattice(16)
    up, down = np.nextafter(L, np.float32(np.inf)), np.nextafter(L, np.float32(-np.inf))
    data = np.concatenate([L[::3], up[1::3], down[2::3]])
    rng = np.random.default_rng(1)
    query = np.concatenate([L[::2] + np.float32(0.5), up[::5], down[::7], L[1::4], rng.uniform(-3, 19, (4000, 3))])
    for md in (16.0, 0.5, 1.0, 0.70710677):
        _, info = _check(query, data, md)
        if md == 16.0:
            assert info["cell_size"] == 1.0


def test_identical_points_and_a_single_point():
    rng = np.random.default_rng(2)
    q = rng.normal(3.0, 2.0, (5000, 3))
    same = np.tile(np.float32([3.25, -1.5, 7.0]), (2000, 1))
    for md in (0.01, 2.0, 50.0):
        _check(q, same, md)
        _check(q, same[:1], md)
    _check(same[:10], same, 1.0)                               # zero distance


def test_queries_far_outside_the_data_are_inf():
    rng = np.random.default_rng(3)
    data = rng.uniform(0, 1, (3000, 3))
    far = rng.uniform(-1, 1, (2000, 3)) * 1e6 + np.array([3e6, 0, 0])
    got, _ = _check(far, data, 10.0)
    assert np.isinf(got).all()
    got, _ = _check(far[:200], data, 3e38)                     # a cap beyond float range of d2: every distance finite
    assert np.isfinite(got).all()


def test_empty_sets():
    from gipuma_b200 import api
    q = np.ones((7, 3), np.float32)
    got, info = api.nearest_distance(q, np.zeros((0, 3), np.float32), 5.0)
    assert np.isinf(got).all() and info["n_cells"] == 0
    got, _ = api.nearest_distance(np.zeros((0, 3), np.float32), q, 5.0)
    assert got.shape == (0,)


def test_max_dist_below_the_spacing_and_beyond_the_extent():
    rng = np.random.default_rng(4)
    data = _lattice(20, 1.0) + rng.uniform(-0.05, 0.05, (21 ** 3, 3)).astype(np.float32)
    q = rng.uniform(-2, 22, (20000, 3))
    got, _ = _check(q, data, 0.3)
    assert np.isinf(got).any() and np.isfinite(got).any()
    got, _ = _check(q, data, 1e3)
    assert np.isfinite(got).all()
    small = rng.uniform(0, 1, (500, 3))
    _check(q, small, 1e5)


def test_plane_with_a_hole_probed_one_ulp_either_side_of_max_dist():
    g = np.arange(-20, 20.01, 0.5, dtype=np.float32)
    X, Y = np.meshgrid(g, g, indexing="ij")
    keep = X ** 2 + Y ** 2 > 5.0 ** 2
    data = np.stack([X[keep], Y[keep], np.zeros(keep.sum(), np.float32)], axis=1)
    rng = np.random.default_rng(5)
    q = np.concatenate([np.stack([rng.uniform(-4, 4, 3000), rng.uniform(-4, 4, 3000), rng.uniform(-3, 3, 3000)], axis=1),
                        rng.uniform(-25, 25, (3000, 3))]).astype(np.float32)
    exact = pycloud.brute(q, data, 1e3)
    for j in (0, 1, 2, 3000):
        D = exact[j]
        for md in (D, np.nextafter(D, np.float32(0)), np.nextafter(D, np.float32(np.inf))):
            got, _ = _check(q, data, float(md))
            assert (got[j] == D) == (md >= D)


def test_coordinates_offset_by_1e4_so_that_dx_rounds():
    rng = np.random.default_rng(6)
    data = (1e4 + rng.uniform(0, 3, (30000, 3))).astype(np.float32)
    q = (1e4 + rng.uniform(-0.5, 3.5, (20000, 3))).astype(np.float32)
    got, _ = _check(q, data, 0.2)
    # the restatement really exercises rounding here: float64 distances differ from the fp32 specification
    exact = np.sqrt(((q[:50, None, :].astype(np.float64) - data[None].astype(np.float64)) ** 2).sum(-1).min(1))
    assert (exact.astype(np.float32) != got[:50]).any()


def _surface(n, rng):
    """Points on a wavy surface with 1 % noise: the shape of a scanned object."""
    u = rng.uniform(-200, 200, (n, 2))
    z = 500 + 20 * np.sin(u[:, 0] / 37) * np.cos(u[:, 1] / 23) + rng.normal(0, 0.2, n)
    return np.column_stack([u, z]).astype(np.float32)


def test_a_million_points_equal_the_certified_restatement():
    rng = np.random.default_rng(7)
    data, q = _surface(1_100_000, rng), _surface(1_000_000, rng)
    q[:50000] += rng.normal(0, 5, (50000, 3)).astype(np.float32)       # some far from the surface
    want, cert = pycloud.certified(q, data, 2.0)
    print("certified %.4f of %d queries" % (cert.mean(), len(q)))
    got, info = _check(q, data, 2.0, want)
    print("1e6 x 1.1e6: build %.2f ms, query %.2f ms, %d cells of %.3g" % (info["build_ms"], info["query_ms"], info["n_cells"],
                                                                       info["cell_size"]))


def test_deterministic_over_runs_permutations_and_memory_kinds():
    import torch
    from gipuma_b200 import api
    rng = np.random.default_rng(8)
    data, q = _surface(200_000, rng), _surface(150_000, rng)
    a, _ = api.nearest_distance(q, data, 3.0)
    b, _ = api.nearest_distance(q, data, 3.0)
    c, _ = api.nearest_distance(q, np.ascontiguousarray(data[rng.permutation(len(data))]), 3.0)
    d, info = api.nearest_distance(torch.from_numpy(q).cuda(), torch.from_numpy(data).cuda(), 3.0)
    assert info["upload_ms"] == 0.0 and d.is_cuda
    for x in (b, c, d.cpu().numpy()):
        assert x.tobytes() == a.tobytes()
    # the vertex records of fuse / read_ply are taken by their x, y, z fields
    v = np.zeros(len(q), dtype=api.PLY_VERTEX)
    v["x"], v["y"], v["z"] = q[:, 0], q[:, 1], q[:, 2]
    assert api.nearest_distance(v, data, 3.0)[0].tobytes() == a.tobytes()


def test_non_finite_device_coordinates_are_refused():
    import torch
    from gipuma_b200 import api
    q = torch.zeros((100, 3), device="cuda")
    b = torch.ones((100, 3), device="cuda")
    b[57, 1] = float("nan")
    with pytest.raises(api.GipumaError, match="non-finite"):
        api.nearest_distance(q, b, 1.0)
    b[57, 1] = 0.0
    q[3, 2] = float("inf")
    with pytest.raises(api.GipumaError, match="non-finite"):
        api.nearest_distance(q, b, 1.0)


# ---- end to end: fused clouds of the fusion test's dataset against the scene's ground truth ---------------------------

def test_scores_of_fused_clouds_on_the_fusion_dataset():
    from gipuma_b200 import api, scene as S
    from test_gpu_fusion import FUSE, REFS, _dataset, _params
    Ps, scale, images, hf = _dataset()
    fPs = [Ps[r] for r in REFS]
    H, W = images.shape[1:]
    gt_maps = S.render_norm4(fPs, scale, H, W, hf)
    gt = S.gt_points(fPs, scale, H, W, hf, norm4=gt_maps)
    unit = hf.unit                                             # one reference pixel at z0: 2.4 here
    taus = (0.25 * unit, 0.5 * unit, unit)
    # ground truth fused: the vertices are means of a few views' surface points, so their distance to the nearest
    # ground-truth sample is set by the samples' spacing; a frame mismatch would put them tens of units away
    v, _ = api.fuse(gt_maps, fPs, cam_scale=scale, **FUSE)
    s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=taus)
    print("GT fused (%d vertices, %d GT points): %s" % (len(v), len(gt), {k: s[k] for k in (
        "accuracy_mean", "accuracy_median", "completeness_mean", "completeness_median", "precision", "recall", "f_score")}))
    # recorded on an H100: accuracy 0.127 unit (0.302), precision at a quarter unit 0.955
    assert s["accuracy_outliers"] == 0.0 and s["accuracy_mean"] < 0.2 * unit and s["precision"][0] > 0.93
    # PatchMatch fused
    n4, _, _ = api.batch_run(images, Ps, _params(), REFS, cam_scale=scale, min_angle=5.0, max_angle=45.0, max_views=6, seed=4242)
    v, _ = api.fuse(n4, fPs, cam_scale=scale, **FUSE)
    s = api.evaluate_cloud(v, gt, max_dist=10 * unit, taus=taus)
    print("PatchMatch fused (%d vertices): %s" % (len(v), {k: s[k] for k in (
        "accuracy_mean", "accuracy_median", "completeness_mean", "completeness_median", "accuracy_outliers",
        "completeness_outliers", "precision", "recall", "f_score")}))
    # recorded on an H100: accuracy 0.587 unit, completeness 0.857 unit, F-score at one unit 0.857; asserted with a 20 % margin
    assert s["accuracy_mean"] < 0.70 * unit and s["completeness_mean"] < 1.03 * unit and s["f_score"][2] > 0.69


def test_dtu_size_ground_truth_fusion_equals_the_certified_restatement_on_a_sample():
    """49 DTU cameras at 1600x1200: the ground-truth-fused cloud (about 5.1 M vertices) against gt_points of every third row
    and column; seeded samples of 10^5 queries in each direction must equal the certified restatement."""
    from gipuma_b200 import api, scene as S
    from test_gpu_fusion import FUSE
    Ps = [S.load_dtu_projections()[i] for i in range(49)]
    H, W = 1200, 1600
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1])[0].fx, seed=77)
    maps = S.render_norm4(Ps, 1.0, H, W, hf)
    v, _ = api.fuse(maps, Ps, **dict(FUSE, disp_thresh=0.1, num_consistent=3))
    gt = S.gt_points(Ps, 1.0, H, W, hf, stride=3, norm4=maps)
    del maps
    rec = np.ascontiguousarray(np.stack([v["x"], v["y"], v["z"]], axis=1))
    rng = np.random.default_rng(2026)
    for name, q, b in (("accuracy", rec, gt), ("completeness", gt, rec)):
        d, info = api.nearest_distance(q, b, 20.0)
        pick = np.sort(rng.choice(len(q), 100_000, replace=False))
        want, cert = pycloud.certified(q[pick], b, 20.0)
        assert d[pick].tobytes() == want.tobytes(), name
        print("DTU size %s: %d queries x %d points, build %.1f ms, query %.1f ms, %.4f certified, mean %.4f" % (
            name, len(q), len(b), info["build_ms"], info["query_ms"], cert.mean(), float(np.mean(d[np.isfinite(d)]))))
