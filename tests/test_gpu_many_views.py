"""Many source views (33 .. GPM_MAX_VIEWS = 64) on the GPU, where every lane of a warp holds a second view (lane + 32).

- at 64 views and box 25 with joint view selection and the geometric term (the largest per-warp scratch of any kernel) a
  context with the automatic warp count runs, and a forced count of 16 warps, whose shared memory no H100 offers, is
  refused with GPM_E_ARG before any launch, leaving the launch count and the state untouched;
- a whole gpm_run is bit-identical when the source views are handed to the context in another order (images, cameras
  and depth maps moved together): combine_views sums the selected costs in ascending order of value and memo, duplicate
  skips and the lower bound are exact shortcuts, so any per-view mis-indexing that the restatements' shapes miss shows
  here.  PM and NCC, each with and without the geometric term, fixed and adaptive propagation, under best_n / all / good.
  Joint view selection is left out: its weighted sums run in view order, so a permutation may change the last bit."""
import ctypes
import time

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_geometric import WEIGHT, depth_maps, make_scene, open_ctx

pytestmark = pytest.mark.gpu

E_ARG = -1


def test_sixteen_warps_refused_at_the_largest_scratch():
    import test_gpu_view_selection as tv
    case = "geo_fixed_64v_box25"
    sc = tv.make_scene(case)
    with tv.open_jvs(case, sc, 13) as ctx, tv.open_jvs(case, sc, 13) as twin:
        L, h = ctx.lib, ctx.h
        ctx.init()
        ctx.sweep(1)                                                   # the automatic warp count runs
        before, launches = tv.state(ctx), ctx.stats()["launches"]
        assert before[2].any()
        planes, out = np.ascontiguousarray(before[0]), np.empty_like(before[1])
        ctx.set_option("nwarps", 16)
        calls = [lambda: L.gpm_init(h), lambda: L.gpm_sweep(h, 1), lambda: L.gpm_phase(h, 0, 7), lambda: L.gpm_phase(h, 1, 3),
                 lambda: L.gpm_cost_eval(h, ctypes.c_void_p(planes.ctypes.data), ctypes.c_void_p(out.ctypes.data), 0)]
        for call in calls:
            assert call() == E_ARG
            assert "shared memory" in L.gpm_last_error().decode()
        assert ctx.stats()["launches"] == launches and tv.same_state(tv.state(ctx), before)
        ctx.set_option("nwarps", 0)
        ctx.sweep(1)
        twin.init()
        twin.sweep(2)
        assert tv.same_state(tv.state(ctx), tv.state(twin))


# views, box, cost_comb, n_best (every window of two rounds or more, so the lower bound has something to cut)
COMBOS = [(33, 11, 1, 3), (64, 15, 1, 40), (33, 25, 0, 2), (64, 13, 3, 2)]
MODES = ["pm", "pm_geo", "ncc", "ncc_geo"]


def permutations(V):
    """Reverse, rotate by 32, and swap the first and last view: each moves views across the lane / lane + 32 boundary."""
    return {"reverse": list(range(V))[::-1], "rotate32": [(v + 32) % V for v in range(V)],
            "swap_ends": [V - 1] + list(range(1, V - 1)) + [0]}


@pytest.mark.parametrize("propagation", ["fixed", "adaptive"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("views,box,comb,n_best", COMBOS)
def test_run_is_invariant_under_view_order(views, box, comb, n_best, mode, propagation):
    t0 = time.perf_counter()
    sc = make_scene(40, 60, views, box=box)
    sc.params.cost_comb, sc.params.n_best = comb, n_best
    geo = mode.endswith("_geo")
    depths = depth_maps(sc, 21) if geo else None
    seed = 300 + views + box

    def run(order):
        with open_ctx(sc, seed, depths, WEIGHT if geo else 0.0, views=order) as ctx:
            if mode.startswith("ncc"):
                ctx.set_photometric("ncc", 2.0)
            ctx.set_propagation(propagation)
            ctx.run()
            return ctx.get_state(), ctx.stats()

    (n0, c0), st = run(list(range(views)))
    assert st["hypotheses"] > 0 and np.isfinite(c0).mean() > 0.99
    if mode == "pm_geo":
        assert st["pruned"] > 0                                        # the lower bound with the geometric term acts
    for name, order in permutations(views).items():
        assert sorted(order) == list(range(views)) and order != list(range(views))
        (n1, c1), _ = run(order)
        assert bits_equal(n1, n0) == 0 and bits_equal(c1, c0) == 0, (name, bits_equal(n1, n0), bits_equal(c1, c0))
    print("\nview order, %d views, box %d, comb %d, n_best %d, %s, %s: pruned %d of %d, %.2f s" %
          (views, box, comb, n_best, mode, propagation, st["pruned"], st["hypotheses"], time.perf_counter() - t0))
