"""Context state across setter calls: a parameter change makes the stored costs stale, and the first image upload fixes the
context's image type."""
import dataclasses

import numpy as np
import pytest

from conftest import bits_equal

pytestmark = pytest.mark.gpu

SEED = 4711
NO_SHORTCUTS = {"memo": 0, "dedupe": 0, "prune": 0}


def small_scene(color):
    from gipuma_b200 import scene as S
    sc = S.make_config(2, rows=240, cols=320, n_views=4, iterations=2, seed=31)
    return S.colorize(sc) if color else sc


def sweep_through_param_change(sc, options):
    """init + 2 sweeps under the scene's parameters, then 2 more under the same parameters with tau_color and tau_gradient
    halved.  Truncation at a smaller tau can only lower a cost, so every cost stored before the change is too high."""
    from gipuma_b200 import api
    with api.Context(sc.cols, sc.rows, sc.n_views) as ctx:
        for k, v in options.items():
            ctx.set_option(k, v)
        ctx.load_scene(sc, seed=SEED)
        ctx.init()
        ctx.sweep(2)
        ctx.set_params(dataclasses.replace(sc.params, tau_color=sc.params.tau_color / 2,
                                           tau_gradient=sc.params.tau_gradient / 2))
        ctx.sweep(2)
        return ctx.get_state()


@pytest.mark.parametrize("color", [False, True], ids=["grey", "colour"])
def test_parameter_change_between_sweeps_matches_the_run_without_shortcuts(color):
    """The exact shortcuts (duplicate skip, memo, lower bound) must not trust costs computed under other parameters: the
    default options and the run with every shortcut off give the same planes and costs, bit for bit."""
    sc = small_scene(color)
    n4, c = sweep_through_param_change(sc, {})
    m4, mc = sweep_through_param_change(sc, NO_SHORTCUTS)
    assert bits_equal(n4, m4) == 0, "planes differ from the run without shortcuts"
    assert bits_equal(c, mc) == 0, "costs differ from the run without shortcuts"


def test_first_upload_fixes_the_image_type():
    from gipuma_b200 import api
    grey, colour = small_scene(False), small_scene(True)
    ref = lambda s: np.ascontiguousarray(s.images[0])                          # noqa: E731
    view = lambda s, v: np.ascontiguousarray(s.images[s.subset[v]])          # noqa: E731
    with api.Context(grey.cols, grey.rows, grey.n_views) as ctx:
        ctx.set_params(grey.params)
        ctx.set_reference(ref(grey), grey.cameras[0])
        with pytest.raises(api.GipumaError):
            ctx.set_view(0, view(colour, 0), colour.cameras[colour.subset[0]])
        ctx.load_scene(grey, seed=SEED)                                        # the grey context still takes grey images
        ctx.init()
    with api.Context(colour.cols, colour.rows, colour.n_views) as ctx:
        ctx.set_params(colour.params)
        ctx.set_view(0, view(colour, 0), colour.cameras[colour.subset[0]])
        with pytest.raises(api.GipumaError):
            ctx.set_reference(ref(grey), grey.cameras[0])
        ctx.load_scene(colour, seed=SEED)
        ctx.init()
