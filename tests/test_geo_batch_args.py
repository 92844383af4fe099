"""gpm_geo_batch_run (the two-pass geometric-consistency batch driver, DESIGN.md §14) without a GPU: its descriptor structs
have the header's layout, every bad descriptor is refused with GPM_E_ARG and a message before any CUDA call, a view whose
angle filter passes nothing is refused with GPM_E_STATE naming it before any CUDA call, and there is no CPU path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E_ARG, E_STATE = -1, -3


def _desc(**kw):
    """A valid descriptor over 3 DTU cameras at 96x64 (grey), then the fields of `kw` overwritten."""
    from gipuma_b200 import api, scene as S
    params = S.AlgorithmParameters(box_hsize=9, box_vsize=9, iterations=1, n_best=2, cost_comb=S.COMB_BEST_N)
    params.depthMin, params.depthMax = 300.0, 800.0
    Ps = [S.load_dtu_projections()[i] for i in range(3)]
    imgs = np.zeros((3, 64, 96), np.float32)
    d, keep = api._batch_desc(imgs, Ps, params, [0, 2], (0,), 1600.0 / 96, 5.0, 45.0, 2, 7, None, None, None)
    g = api.GpmGeoBatchDesc(d, 1, 1, 0.5, 3.0)
    for name, value in kw.items():
        setattr(g.batch if hasattr(g.batch, name) else g, name, value)
    return g, keep


def _run(g):
    from gipuma_b200 import api
    lib = api.load_library()
    rc = lib.gpm_geo_batch_run(C.byref(g) if g is not None else None, None)
    return rc, lib.gpm_batch_last_error().decode()


@pytest.mark.parametrize("kw", [dict(images=None), dict(channels=2), dict(geo_iterations=-1), dict(weight=float("nan")),
                                dict(weight=-1.0), dict(max_err=0.0), dict(max_views=0), dict(max_views=65),
                                dict(n_devices=0), dict(ref_indices=(C.c_int * 2)(0, 3)), dict(ref_indices=None, n_refs=5),
                                dict(ref_indices=(C.c_int * 2)(2, 2), out_dir=b"unused")],
                         ids=["null_images", "channels_2", "geo_iterations_-1", "weight_nan", "weight_-1", "max_err_0",
                              "max_views_0", "max_views_65", "n_devices_0", "ref_out_of_range", "implicit_refs_beyond_images",
                              "repeated_ref_with_out_dir"])
def test_bad_descriptors_are_refused_before_any_cuda_call(kw):
    g, _keep = _desc(**kw)
    rc, msg = _run(g)
    assert rc == E_ARG and msg.startswith("gpm_geo_batch_run: bad arguments"), (rc, msg)


def test_repeated_reference_without_out_dir_is_accepted():
    g, _keep = _desc(ref_indices=(C.c_int * 2)(2, 2))
    rc, msg = _run(g)
    assert rc != E_ARG, msg                                   # runs on a GPU; without one it fails for want of a device


@pytest.mark.parametrize("kw", [dict(weight=-0.1), dict(max_err=0.0), dict(refs=[3]), dict(refs=[]), dict(geo_iterations=-1),
                                dict(geo_iterations=1.5), dict(images=np.zeros((3, 16, 16, 3), np.float32)),
                                dict(Ps=[np.eye(3, 4)] * 2), dict(max_views=0)])
def test_geometric_pass_refuses_bad_arguments_before_loading_the_library(monkeypatch, kw):
    from types import SimpleNamespace
    from gipuma_b200 import api

    def no_library(*a, **k):
        raise AssertionError("the library was reached with arguments that must be refused")
    monkeypatch.setattr(api, "load_library", no_library)
    args = dict(images=np.zeros((3, 16, 16), np.float32), Ps=[np.eye(3, 4)] * 3, params=SimpleNamespace(iterations=1), refs=[0])
    args.update(kw)
    with pytest.raises(ValueError):
        api.geometric_pass(**args)


def test_null_descriptor_is_refused():
    rc, msg = _run(None)
    assert rc == E_ARG and "bad arguments" in msg


def test_a_view_without_source_views_is_refused_by_name_before_any_cuda_call():
    g, _keep = _desc(min_angle=0.1, max_angle=0.2)             # no camera within 0.1 .. 0.2 degrees of another
    rc, msg = _run(g)
    assert rc == E_STATE and msg.endswith("reference view 0"), (rc, msg)


def test_no_cpu_fallback_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA device present: covered by tests/test_gpu_geometric_batch.py")
    g, _keep = _desc()
    rc, msg = _run(g)
    assert rc != 0 and ("CUDA" in msg or "device" in msg), (rc, msg)


def test_struct_layouts_match_ctypes(tmp_path):
    from gipuma_b200 import api
    fields = {"gpm_geo_batch_desc": ["batch", "channels", "geo_iterations", "weight", "max_err"],
              "gpm_geo_batch_stats": ["batch", "n_pass1", "pass1_views", "pass1_sweep_ms", "ref_views"]}
    lines = ['printf("%%zu\\n", sizeof(%s));' % s + "".join(' printf("%%zu\\n", offsetof(%s, %s));' % (s, f) for f in fs)
             for s, fs in fields.items()]
    src = tmp_path / "s.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gipuma_b200.h"\nint main(void){ %s return 0; }\n'
                   % " ".join(lines))
    exe = str(tmp_path / "s")
    subprocess.check_call(["gcc", "-I" + os.path.join(ROOT, "include"), str(src), "-o", exe])
    got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = []
    for cls, fs in ((api.GpmGeoBatchDesc, fields["gpm_geo_batch_desc"]), (api.GpmGeoBatchStats, fields["gpm_geo_batch_stats"])):
        want += [C.sizeof(cls)] + [getattr(cls, f).offset for f in fs]
    assert got == want
