"""Point-cloud evaluation (DESIGN.md §13) without a GPU: the two restatements of the nearest distance agree, cloud_scores on
hand-made distances with known answers, gt_points on the height field, and the refusal of bad descriptors before any CUDA
call."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from oracle import pycloud


def _sets(kind, rng):
    if kind == "random":
        return rng.uniform(-50, 50, (3000, 3)), rng.uniform(-50, 50, (4000, 3))
    if kind == "clustered":
        centres = rng.uniform(-100, 100, (6, 3))
        data = centres[rng.integers(0, 6, 5000)] + rng.normal(0, 0.3, (5000, 3))
        query = centres[rng.integers(0, 6, 3000)] + rng.normal(0, 2.0, (3000, 3))
        return query, data
    # duplicates: every data point three times, the first 300 five times; queries on and between them, far from the origin
    # so that dx rounds
    base = (1e4 + rng.integers(-40, 40, (1200, 3)) * 0.25 + rng.uniform(0, 1e-3, (1200, 3))).astype(np.float32)
    data = np.concatenate([base] * 3 + [base[:300]] * 2)
    query = np.concatenate([base[:1000], base[:1000] + 0.125])
    return query, data


@pytest.mark.parametrize("kind", ["random", "clustered", "duplicates"])
@pytest.mark.parametrize("max_dist", [0.2, 3.0, 1e3])
def test_certified_restatement_equals_brute_force(kind, max_dist):
    q, b = (x.astype(np.float32) for x in _sets(kind, np.random.default_rng(len(kind))))
    want = pycloud.brute(q, b, max_dist)
    got, cert = pycloud.certified(q, b, max_dist, k=4, workers=1)
    assert got.view(np.uint32).tobytes() == want.view(np.uint32).tobytes()
    assert cert.mean() > 0.5                                   # the certificate does most of the work
    if kind == "duplicates":
        assert (~cert).any()                                   # five equal points tie for the k = 4 candidates
    if max_dist == 1e3:
        assert np.isfinite(want).all()


def test_brute_force_is_the_specification():
    q = np.array([[0, 0, 0], [1e4, 0, 0], [3, 4, 12]], np.float32)
    b = np.array([[3, 4, 0], [1e4 + 1e-3, 0, 0]], np.float32)
    d2 = pycloud.brute_d2(q, b)
    assert d2[0] == np.float32(25) and d2[2] == np.float32(144)
    dx = np.float32(1e4) - np.float32(1e4 + 1e-3)               # dx rounds: 1e4 + 1e-3 is not a float32
    assert d2[1] == dx * dx
    assert np.isinf(pycloud.brute(q, b[:0], 1.0)).all()
    d = pycloud.brute(q, b, 12.0)
    assert d[0] == 5 and d[2] == 12 and np.isinf(pycloud.brute(q, b, np.nextafter(np.float32(12), np.float32(0)))[2])


def test_sqrt_threshold():
    for m in (1e-30, 0.37, 1.0, 20.0, 3.1e5, 1e19):
        v = pycloud.sqrt_threshold(m)
        assert np.sqrt(v) > np.float32(m) and not np.sqrt(np.nextafter(v, np.float32(0))) > np.float32(m)


def test_cloud_scores_known_answers():
    from gipuma_b200 import api
    inf = float("inf")
    s = api.cloud_scores([0.1, 0.3, 2.0, 25.0, inf], [0.2, 0.4, inf, inf], max_dist=20.0, taus=(0.25, 1.0, 20.0))
    assert s["accuracy_mean"] == pytest.approx((0.1 + 0.3 + 2.0) / 3) and s["accuracy_median"] == pytest.approx(0.3)
    assert s["completeness_mean"] == pytest.approx(0.3) and s["completeness_median"] == pytest.approx(0.3)
    assert s["overall"] == pytest.approx(0.5 * (0.8 + 0.3))
    assert s["accuracy_outliers"] == pytest.approx(0.4) and s["completeness_outliers"] == pytest.approx(0.5)
    assert s["precision"] == pytest.approx([0.2, 0.4, 0.6]) and s["recall"] == pytest.approx([0.25, 0.5, 0.5])
    assert s["f_score"][1] == pytest.approx(2 * 0.4 * 0.5 / 0.9)
    # the cap is "< max_dist": a distance of exactly max_dist is an outlier
    s = api.cloud_scores([20.0, 1.0], [1.0], max_dist=20.0, taus=(20.0,))
    assert s["accuracy_mean"] == 1.0 and s["accuracy_outliers"] == 0.5 and s["precision"] == [0.5]
    # F-score 0: nothing within tau in either direction
    s = api.cloud_scores([5.0], [6.0], max_dist=20.0, taus=(1.0,))
    assert s["precision"] == [0.0] and s["recall"] == [0.0] and s["f_score"] == [0.0]


def test_cloud_scores_sums_in_index_order():
    from gipuma_b200 import api
    x = np.array([1.0] + [1e-16] * 1000)                       # each 1e-16 is lost against the running sum; numpy's
    s = api.cloud_scores(x, x, max_dist=2.0, taus=())           # pairwise sum would keep them
    assert s["accuracy_mean"] == 1.0 / len(x) and s["completeness_mean"] == 1.0 / len(x)


def test_cloud_scores_refuses_tau_beyond_max_dist_and_handles_empty_sets():
    from gipuma_b200 import api
    with pytest.raises(ValueError):
        api.cloud_scores([1.0], [1.0], max_dist=20.0, taus=(20.5,))
    with pytest.raises(ValueError):
        api.cloud_scores([1.0], [1.0], max_dist=float("inf"))
    s = api.cloud_scores([], [], max_dist=20.0, taus=(1.0,))
    assert all(math.isnan(s[k]) for k in ("accuracy_mean", "accuracy_median", "completeness_mean", "completeness_median", "overall"))
    assert s["accuracy_outliers"] == 0.0 and s["completeness_outliers"] == 0.0
    assert s["precision"] == [0.0] and s["recall"] == [0.0] and s["f_score"] == [0.0]
    s = api.cloud_scores([30.0, float("inf")], [0.5], max_dist=20.0, taus=(1.0,))
    assert math.isnan(s["accuracy_mean"]) and s["accuracy_outliers"] == 1.0 and s["completeness_mean"] == 0.5


def test_gt_points_lie_on_the_height_field():
    from gipuma_b200 import scene as S
    Ps = [S.load_dtu_projections()[i] for i in (0, 5, 20)]
    rows, cols = 48, 64
    scale = 1600.0 / cols
    hf = S.HeightField(z0=550.0, unit=550.0 / S.prepare_cameras(Ps[:1], scale)[0].fx, seed=77)
    n4 = S.render_norm4(Ps, scale, rows, cols, hf)
    pts = S.gt_points(Ps, scale, rows, cols, hf, norm4=n4)
    assert pts.dtype == np.float32 and pts.shape == (int((n4[..., 3] > 0).sum()), 3)
    R0, t0 = S.ref0_frame(Ps)
    X = pts.astype(np.float64) @ R0.T + t0
    err = np.abs(X[:, 2] - hf.height(X[:, 0], X[:, 1]))
    # the maps' ray casts used float32 cameras: 2.4e-5 z0 at most here (view 0 alone, whose camera is exact: 6e-8 z0)
    assert err.max() < 5e-5 * hf.z0 and err[: int((n4[0, ..., 3] > 0).sum())].max() < 1e-6 * hf.z0
    half = S.gt_points(Ps, scale, rows, cols, hf, stride=2, norm4=n4)
    assert len(half) == int((n4[:, ::2, ::2, 3] > 0).sum())
    assert np.array_equal(half, S.gt_points(Ps, scale, rows, cols, hf, stride=2))


def test_bad_descriptors_are_refused_before_any_cuda_call():
    from gipuma_b200 import api
    lib = api.load_library()
    q = np.zeros((4, 3), np.float32)
    b = np.ones((5, 3), np.float32)
    out = np.empty(4, np.float32)

    def call(res=True, **kw):
        d = api.GpmNnDesc(4, 5, q.ctypes.data, b.ctypes.data, 0, 0, 1.0)
        for k, v in kw.items():
            setattr(d, k, v)
        r = api.GpmNnResult(out.ctypes.data, 0.0, 0.0, 0.0, 0.0, 0)
        rc = lib.gpm_nearest_dist(C.byref(d), C.byref(r) if res else None)
        return rc, lib.gpm_last_error().decode()

    nan_q = q.copy()
    nan_q[2, 1] = np.nan
    inf_b = b.copy()
    inf_b[4, 2] = -np.inf
    for bad in (dict(n_query=-1), dict(n_data=-3), dict(n_query=1 << 31), dict(query=None), dict(data=None),
                dict(max_dist=0.0), dict(max_dist=-1.0), dict(max_dist=float("inf")), dict(max_dist=float("nan")),
                dict(query=nan_q.ctypes.data), dict(data=inf_b.ctypes.data), dict(res=False)):
        rc, msg = call(**bad)
        assert rc == -1 and msg.startswith("gpm_nearest_dist:"), (bad, rc, msg)
    assert call(n_query=0, query=None)[0] == 0                 # nothing to compute
    with pytest.raises(ValueError):
        api.nearest_distance(np.zeros((3, 2), np.float32), b, 1.0)
    with pytest.raises(TypeError):
        api.nearest_distance(q.astype(np.float64), b, 1.0)
    from conftest import have_cuda
    if not have_cuda():
        rc, msg = call()                                       # a valid descriptor needs a device: no CPU path
        assert rc == -2, msg


def test_cloud_struct_layouts_match_ctypes(tmp_path):
    from gipuma_b200 import api
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "gipuma_b200.h"\nint main(void){ printf("%zu %zu %zu %zu %zu\\n", '
                   'sizeof(gpm_nn_desc), sizeof(gpm_nn_result), offsetof(gpm_nn_desc, max_dist), offsetof(gpm_nn_result, cell_size), '
                   'offsetof(gpm_nn_result, n_cells)); return 0; }\n')
    exe = str(tmp_path / "t")
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I" + os.path.join(root, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(api.GpmNnDesc), C.sizeof(api.GpmNnResult), api.GpmNnDesc.max_dist.offset,
                   api.GpmNnResult.cell_size.offset, api.GpmNnResult.n_cells.offset]
