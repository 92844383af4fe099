"""The source-view shard checked exactly at ragged and odd image sizes, stage by stage.

The shard runs on kernels of its own (k_shard_stage, k_shard_accept0) with their own pixel indexing:
half-row lists (Wh = ceil(W / 2)), the colour parity, stage 0's two parity planes, 8 * n_best floats per pixel in stage
1, and their own tile-slice loop and accept.  The ranks are simulated by contexts on one GPU (test_gpu_view_shard's
SimulatedShard, all-gather = torch.cat), next to one context holding every view, all with the same seed.  After every
stage:
- init: every rank's costs after shard_finish_init equal ctx.init() of the single context;
- propagation (accepted by stage 2): planes and costs equal oracle/pypropagate.expected(mask=3), outside the pixels whose
  depth-range test is ambiguous, and equal the single context after phase(colour, 1) and phase(colour, 2) everywhere;
- lists: the slots the border guards do not offer are +inf on every rank, and the n_best smallest of the union of the
  gathered lists are the same bits for every world size (selections only: the merge divides with an approximate
  reciprocal, so its mean is not restated);
- each refinement step: a changed pixel's cost equals its gpm_cost_eval at the refinement's call site, its normal is a
  unit vector facing the camera, nothing else changes;
- closing accept: the state equals the single context after phase(colour, 4);
- twin groups without memo and duplicate shortcuts, and with 5 warps per block, stay bit-identical after every colour.
The cases cover every gridDim.z split (1, 2, 4, 8 on 132 SMs), odd widths, partial tiles, n_best above the views of a
rank, > 32 views on one rank and world sizes 1 .. 8.  Adversarial states (ties, out-of-range planes, costs above
MAXCOST) go through set_state, and the refusals of the stage entry points are checked."""
import time

import numpy as np
import pytest

from conftest import bits_equal
from test_gpu_sweep_any_size import adversarial_state, bands, check_launch, cost_of
from test_gpu_view_shard import SimulatedShard, open_ranks

pytestmark = pytest.mark.gpu

MAXCOST = np.float32(1000.0)
INF = np.uint32(0x7f800000)
SEED = 0xC0FFEE
TILE = 32
REPORT = {}

# id: (rows, cols, views, world sizes, n_best, box, colour images, iterations, lists checked on the edge rows only)
CASES = {
    "53x75": (53, 75, 7, (1, 2, 3), 3, 9, False, 2, False),                 # 3 + 2 + 2 views at world 3
    "colour_45x71": (45, 71, 5, (2,), 3, 11, True, 2, False),
    "8x8_box25": (8, 8, 2, (2,), 3, 25, False, 2, False),                   # window larger than the image; n_best > views per rank
    "31x33_world8_nbest1": (31, 33, 9, (8,), 1, 15, False, 2, False),       # world at the limit
    "31x33_world8_nbest8": (31, 33, 9, (8,), 8, 15, False, 2, False),
    "37x41_40views": (37, 41, 40, (1,), 3, 7, False, 2, False),             # > 32 views on one rank
    "473x599": (473, 599, 6, (2,), 3, 15, False, 1, False),                 # 285 tiles
    "663x853": (663, 853, 6, (3,), 3, 15, False, 1, False),                 # 567 tiles
    "1045x1051": (1045, 1051, 4, (2,), 3, 9, False, 1, True),               # 1089 tiles
}


def make_scene(rows, cols, views, n_best, box, colour, iterations):
    from gipuma_b200 import scene as S
    sc = S.make_config(2, rows=rows, cols=cols, n_views=views, iterations=iterations, seed=rows * 1000 + cols)
    sc.params.box_hsize = sc.params.box_vsize = box
    sc.params.n_best = n_best
    return S.colorize(sc) if colour else sc


def case_scene(case):
    rows, cols, views, worlds, n_best, box, colour, iterations, _ = CASES[case]
    return make_scene(rows, cols, views, n_best, box, colour, iterations)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tiles(rows, cols):
    return -(-rows // TILE) * -(-cols // TILE)


def grid_split(rows, cols, sms):
    """gridDim.z of the tile kernels: the smallest power of two <= 8 with tiles * split >= 8 * SMs."""
    z = 1
    while z < 8 and tiles(rows, cols) * z < 8 * sms:
        z *= 2
    return z


def open_single(sc):
    from gipuma_b200 import api
    ctx = api.Context(sc.cols, sc.rows, sc.n_views)
    ctx.load_scene(sc, seed=SEED)
    return ctx


def pixel_of(H, W, parity):
    """Pixel x of every half-row slot (py, hx) of the pixels with (x + y) & 1 == parity, and whether it lies in the image."""
    ys, hx = np.mgrid[0:H, 0:(W + 1) // 2]
    px = 2 * hx + ((ys + parity) & 1)
    return ys, px, px < W


def lists_view(g, world, H, W, nb, st):
    """The gathered lists of stage `st` as uint32 [world, ..., n_best]: stage 0 [2, H, Wh], stage 1 [H, Wh, 8], later [H, Wh]."""
    Wh = (W + 1) // 2
    shape = (2, H, Wh) if st == 0 else (H, Wh, 8) if st == 1 else (H, Wh)
    return g.cpu().numpy().view(np.uint32).reshape((world,) + shape + (nb,))


def selection(g, world, H, W, nb, st, colour, rows):
    """The n_best smallest entries of the union of all ranks' lists of every slot (bits; 0 where no pixel is), on `rows`."""
    u = lists_view(g, world, H, W, nb, st)
    u = np.moveaxis(u, 0, -2)
    sel = np.sort(u.reshape(u.shape[:-2] + (world * nb,)), axis=-1)[..., :nb]
    if st == 0:
        valid = np.stack([pixel_of(H, W, p)[2] for p in (0, 1)])
        sel = np.where(valid[..., None], sel, 0)[:, rows]
    else:
        valid = pixel_of(H, W, colour)[2]
        sel = np.where(valid.reshape(valid.shape + (1,) * (sel.ndim - 2)), sel, 0)[rows]
    return sel


def edge_rows(H, edges_only):
    return np.concatenate([np.arange(a, b) for a, b in bands(H)]) if edges_only else np.arange(H)


def assert_not_offered_are_inf(g, world, H, W, nb, colour):
    """Stage 1: a slot the border guards do not offer holds +inf in every rank's list."""
    from oracle import pypropagate as pp
    u = lists_view(g, world, H, W, nb, 1)
    ys, px, valid = pixel_of(H, W, colour)
    pxc = np.minimum(px, W - 1)
    for k, dy, dx, ok in pp.candidates(H, W, 3):
        off = valid & ~ok[ys, pxc]
        if off.any():
            assert np.all(u[:, off, k, :] == INF), (colour, k, int((u[:, off, k, :] != INF).sum()))


def group_state(grp):
    """The state of rank 0, after checking that every rank holds the same bits."""
    p0, c0 = grp.ctxs[0].get_state()
    for ctx in grp.ctxs[1:]:
        p, c = ctx.get_state()
        assert bits_equal(p, p0) == 0 and bits_equal(c, c0) == 0
    return p0, c0


def assert_same_state(a, b, what):
    bad = (a[0].view(np.uint32) != b[0].view(np.uint32)).any(axis=-1) | (a[1].view(np.uint32) != b[1].view(np.uint32))
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:8].tolist())


class Checker:
    """Runs the checked group, its list peers and twins through colours with every stage checked."""

    def __init__(self, sc, colour_images, single, checked, list_peers=(), twins=(), edges_only=False, single_vs_rule=False):
        self.sc, self.colour_images, self.single, self.checked = sc, colour_images, single, checked
        self.list_peers, self.twins = list(list_peers), list(twins)
        self.rows = edge_rows(sc.rows, edges_only)
        self.single_vs_rule = single_vs_rule
        self.cost = cost_of(single)
        self.stats = {"compared": 0, "ambiguous": 0, "accepted": 0, "refined": 0}

    def expected(self, before, colour, mask):
        from oracle import pypropagate as pp
        prm = self.sc.params
        return pp.expected(before[0], before[1], colour, mask, self.cost, self.sc.cameras[0], prm.depthMin, prm.depthMax,
                           fused=False, color_images=self.colour_images)

    def assert_rule(self, got, want, colour, what):
        """got == want outside the ambiguous pixels; returns the ambiguous mask."""
        want_p, want_c, amb = want
        bad = (got[0].view(np.uint32) != want_p.view(np.uint32)).any(axis=-1) | (got[1].view(np.uint32) != want_c.view(np.uint32))
        bad &= ~amb
        assert not bad.any(), (what, colour, int(bad.sum()), np.argwhere(bad)[:8].tolist())
        return amb

    def lists(self, grp, st, g, colour, sels):
        sc = self.sc
        nb = sc.params.n_best
        sel = selection(g, grp.world, sc.rows, sc.cols, nb, st, colour, self.rows)
        if st in sels:
            assert np.array_equal(sel, sels[st]), ("lists", "world %d" % grp.world, "stage %d" % st, colour,
                                                   int((sel != sels[st]).any(axis=-1).sum()))
        else:
            sels[st] = sel

    def init(self):
        sc, sels = self.sc, {}
        self.single.init()
        want = self.single.get_state()
        for grp in [self.checked] + self.list_peers + self.twins:
            g0 = grp.init()
            assert_same_state(group_state(grp), want, "init, world %d" % grp.world)
            if grp is self.checked or grp in self.list_peers:
                self.lists(grp, 0, g0, 0, sels)

    def colour(self, colour):
        sc, single = self.sc, self.single
        H, W = sc.rows, sc.cols
        ys, xs = np.mgrid[0:H, 0:W]
        mine = ((xs + ys) & 1) == colour
        before = group_state(self.checked)
        assert_same_state(before, single.get_state(), "colour start")
        sels = {}
        last = {"state": before}

        def on_checked(st, g):
            after = group_state(self.checked)
            if st == 1:                                        # evaluation only: the state is untouched
                assert_same_state(after, before, "stage 1")
                assert_not_offered_are_inf(g, self.checked.world, H, W, sc.params.n_best, colour)
            elif st == 2:                                      # the accept of the propagation slots
                amb = self.assert_rule(after, self.expected(before, colour, 3), colour, "propagation")
                check_launch(before, after, colour)
                self.stats["compared"] += int((mine & ~amb).sum())
                self.stats["ambiguous"] += int((mine & amb).sum())
                self.stats["accepted"] += int((mine & (after[1] < before[1])).sum())
                for mask in (1, 2):
                    s0 = single.get_state()
                    single.phase(colour, mask)
                    if self.single_vs_rule:
                        self.assert_rule(single.get_state(), self.expected(s0, colour, mask), colour, "single, mask %d" % mask)
                assert_same_state(after, single.get_state(), "propagation vs single")
            else:                                              # the accept of one refinement step
                self.stats["refined"] += check_launch(last["state"], after, colour, self.cost, sc, 0)
            if st == self.checked.n_stages:                    # closing accept: the whole refinement
                single.phase(colour, 4)
                assert_same_state(after, single.get_state(), "closing accept vs single")
            if g is not None:
                self.lists(self.checked, st, g, colour, sels)
            last["state"] = after

        self.checked.colour(colour, on_checked)
        for grp in self.list_peers:
            grp.colour(colour, lambda st, g, grp=grp: g is not None and self.lists(grp, st, g, colour, sels))
        for grp in self.twins:
            grp.colour(colour)
        ref = single.get_state()
        for grp in self.list_peers + self.twins:
            assert_same_state(group_state(grp), ref, "world %d after colour %d" % (grp.world, colour))

    def run(self, iterations):
        for _ in range(iterations):
            for colour in (0, 1):
                self.colour(colour)
        # at most 0.5 % of the decisions are left out of the comparison with the rule (they are still compared with the
        # single context); at 8x8 (128 decisions) one ambiguous pixel is already 0.8 %, so a few are allowed there
        st = self.stats
        total = st["compared"] + st["ambiguous"]
        assert st["ambiguous"] <= max(4, 0.005 * total), st
        return dict(st, ambiguous_share=st["ambiguous"] / max(1, total))


def test_cases_cover_every_grid_split():
    sms = sm_count()
    z = {case: grid_split(c[0], c[1], sms) for case, c in CASES.items()}
    print("\nSMs %d, gridDim.z per case: %s" % (sms, z))
    assert {1, 2, 4, 8} <= set(z.values()), z


@pytest.mark.parametrize("case", list(CASES))
def test_view_shard_stages_exact_at_any_size(case):
    t0 = time.perf_counter()
    rows, cols, views, worlds, n_best, box, colour, iterations, edges_only = CASES[case]
    sc = case_scene(case)
    single = open_single(sc)
    groups = [SimulatedShard(sc, w, SEED) for w in sorted(worlds, reverse=True)]     # the largest world is checked stage by stage
    twin_memo = SimulatedShard(sc, max(worlds), SEED, {"memo": 0, "dedupe": 0})
    # 5 warps per block, at world 1 where the case has no world-1 group: its lists also pin the selections across world sizes
    twin_warps = SimulatedShard(sc, 1 if 1 not in worlds else max(worlds), SEED, {"nwarps": 5})
    try:
        chk = Checker(sc, colour, single, groups[0], groups[1:] + [twin_warps], [twin_memo], edges_only)
        chk.init()
        REPORT[case] = chk.run(iterations)
    finally:
        for g in groups + [twin_memo, twin_warps]:
            g.close()
        single.close()
    assert REPORT[case]["accepted"] > 0 and REPORT[case]["refined"] > 0
    REPORT[case]["z"] = grid_split(rows, cols, sm_count())
    REPORT[case]["seconds"] = round(time.perf_counter() - t0, 2)
    print("\n%s: %s" % (case, REPORT[case]))


@pytest.mark.parametrize("case", ["53x75", "1045x1051"])
def test_view_shard_runner_world1_equals_single_run(case):
    """multigpu.ViewShardRunner at world size 1 (gpm_shard_run, the exchange a device copy) = gpm_run, bit for bit."""
    from gipuma_b200 import api, multigpu as M
    sc = case_scene(case)
    single, _, _ = api.runcuda(sc, seed=SEED)
    run = M.ViewShardRunner(sc, 0, 1, seed=SEED)
    try:
        n4, c = run.run()
    finally:
        run.close()
    assert bits_equal(n4, single.norm4) == 0 and bits_equal(c, single.c) == 0


@pytest.mark.parametrize("case,world", [("53x75", 3), ("colour_45x71", 2)])
def test_view_shard_on_adversarial_states(case, world):
    """adversarial_state of the sweep tests (ties, bit-equal copies, out-of-range planes, MAXCOST patches) set through
    set_state, and 5 % of the pixels at least 5 px inside every border given a cost of 2 * MAXCOST or +inf, some of them
    with every neighbour out of range: a slot every rank skipped must never be accepted, as k_sweep never compares a
    skipped candidate.  (The costs above MAXCOST stay away from the borders, so a flow that did accept such a slot would
    still read planes inside the image.)  The shard and the single context must both follow the acceptance rule."""
    t0 = time.perf_counter()
    sc = case_scene(case)
    H, W = sc.rows, sc.cols
    single = open_single(sc)
    grp = SimulatedShard(sc, world, SEED)
    try:
        single.init()
        n0, _ = single.get_state()
        rng = np.random.default_rng(11)
        pl, cost = adversarial_state(sc, n0, cost_of(single), rng, False, CASES[case][6])
        ys, xs = np.mgrid[0:H, 0:W]
        inner = (ys >= 5) & (ys < H - 5) & (xs >= 5) & (xs < W - 5)
        high = inner & (rng.random((H, W)) < 0.05)
        cost[high] = np.where(rng.random((H, W)) < 0.5, 2 * MAXCOST, np.float32(np.inf))[high]
        # around 30 % of them, every neighbour 1 and 5 px away holds a fronto-parallel plane at depth 2 * depthMax: out of
        # range, so every rank skips all 8 slots, and a skipped slot accepted in place of none would show
        from oracle import pypropagate as pp
        lonely = high & (rng.random((H, W)) < 0.3)
        far = np.array([0.0, 0.0, -1.0, 2 * sc.params.depthMax], np.float32)
        nbr = np.zeros((H, W), bool)
        for dy, dx in pp.CLOSE + pp.FAR:
            nbr[(ys + dy)[lonely], (xs + dx)[lonely]] = True
        pl[nbr] = far
        nbr &= ~high
        cost[nbr] = cost_of(single)(pl, pp.propagation_site(0, False, CASES[case][6]))[nbr]
        assert lonely.sum() > 0
        grp.init()
        for ctx in grp.ctxs:
            ctx.set_state(pl, cost)
        single.set_state(pl, cost)
        chk = Checker(sc, CASES[case][6], single, grp, single_vs_rule=True)
        REPORT["adversarial_" + case] = chk.run(2)
    finally:
        grp.close()
        single.close()
    REPORT["adversarial_" + case]["seconds"] = round(time.perf_counter() - t0, 2)
    print("\nadversarial %s: %s" % (case, REPORT["adversarial_" + case]))


def test_view_shard_refusals_come_before_any_launch():
    """Configurations the shard does not implement and bad stage arguments are refused, and nothing was launched: the
    launch count, the state and the exchange buffer are untouched."""
    import torch
    from gipuma_b200 import api
    sc = make_scene(45, 71, 4, 3, 9, False, 1)

    def refused(setup, call):
        ctx = open_ranks(sc, 1, SEED)[0]
        try:
            ctx.init()
            setup(ctx)
            state = ctx.get_state()
            launches = ctx.stats()["launches"]
            n = max(ctx.shard_stage_floats(s) for s in range(ctx.shard_num_stages()))
            buf = torch.full((max(n, 1) * 2,), 12345.0, dtype=torch.float32, device="cuda")
            with pytest.raises(api.GipumaError):
                call(ctx, buf)
            torch.cuda.synchronize()
            assert ctx.stats()["launches"] == launches
            assert bool((buf == 12345.0).all())
            assert_same_state(ctx.get_state(), state, "refused call")
        finally:
            ctx.close()

    def params(**kw):
        def setup(ctx):
            prm = sc.params
            old = {k: getattr(prm, k) for k in kw}
            for k, v in kw.items():
                setattr(prm, k, v)
            try:
                ctx.set_params(prm)
            finally:
                for k, v in old.items():
                    setattr(prm, k, v)
        return setup

    def none(ctx):
        pass

    stage1 = lambda ctx, buf: ctx.shard_stage(0, 1, None, 1, buf)            # noqa: E731
    stage0 = lambda ctx, buf: ctx.shard_stage(0, 0, None, 1, buf)            # noqa: E731
    finish = lambda ctx, buf: ctx.shard_finish_init(buf, 1)                  # noqa: E731
    for setup in (lambda ctx: ctx.set_option("neighbours", 20), lambda ctx: ctx.set_rng(SEED, api.GPM_RNG_STATEFUL),
                  params(n_best=0), params(n_best=33)):
        for call in (stage0, stage1, finish):
            refused(setup, call)
    refused(none, lambda ctx, buf: ctx.shard_stage(0, 1, None, 9, buf))
    refused(none, lambda ctx, buf: ctx.shard_finish_init(buf, 9))
    refused(none, lambda ctx, buf: ctx.shard_stage(0, ctx.shard_num_stages() + 1, buf, 1, buf))
    refused(none, lambda ctx, buf: ctx.shard_stage(1, -1, None, 1, buf))
