#!/usr/bin/env python
"""GPU parity probe (development tool): gipuma_b200 vs the pinned reference build, level by level.

  cost   : same planes -> multi-view cost, bitwise
  init   : random planes + initial cost
  steps  : each of the six sweep kernels of one iteration from the reference's own state
  full   : whole runcuda()
Usage: python tools/gpu_probe2.py [--case small|v10|b25|v47|cfg2] ...
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from gipuma_b200 import scene as S, api          # noqa: E402
from oracle import pyref                          # noqa: E402


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def cmp(name, a, b, out):
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    neq = bits(a) != bits(b)
    both_nan = np.isnan(a) & np.isnan(b)
    neq &= ~both_nan
    n = int(neq.sum())
    rec = {"n": int(a.size), "mismatch": n}
    if n:
        d = np.abs(a.astype(np.float64) - b.astype(np.float64))
        rel = d / np.maximum(1e-30, np.abs(b.astype(np.float64)))
        rec["max_abs"] = float(np.nanmax(d[neq]))
        rec["max_rel"] = float(np.nanmax(rel[neq]))
        idx = np.argwhere(neq)[:3].tolist()
        rec["first"] = [(i, float(a[tuple(i)]), float(b[tuple(i)])) for i in idx]
    out[name] = rec
    return n


def make_case(name):
    if name == "small":
        return S.make_config(1)
    if name == "v10":
        return S.make_config(2, rows=352, cols=480)
    if name == "b25":
        return S.make_config(3, rows=256, cols=320, n_views=30)
    if name == "v47":
        return S.make_config(4, rows=256, cols=320)
    if name == "cfg2":
        return S.make_config(2)
    if name == "cfg3":
        return S.make_config(3)
    raise ValueError(name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", nargs="+", default=["small", "v10"])
    ap.add_argument("--levels", nargs="+", default=["cost", "init", "steps", "full"])
    ap.add_argument("--time", action="store_true")
    args = ap.parse_args()
    for case in args.case:
        sc = make_case(case)
        ref = pyref.Harness("ref64" if sc.n_views > 32 else "ref")
        out = {"case": case, "rows": sc.rows, "cols": sc.cols, "V": sc.n_views, "box": sc.params.box_hsize}
        ctx = api.Context(sc.cols, sc.rows, sc.n_views)
        ctx.load_scene(sc)
        # reference init state
        r_n4, r_c, _ = ref.steps(sc, [pyref.STEP_INIT])
        if "cost" in args.levels:
            rc = ref.cost_eval(sc, r_n4)
            mc = ctx.cost_eval(r_n4)
            cmp("cost_eval(mine vs ref)", mc, rc, out)
            cmp("ref: init cost vs sweep-path cost", r_c, rc, out)
        if "init" in args.levels:
            ctx.init()
            m_n4, m_c = ctx.get_state()
            cmp("init planes", m_n4, r_n4, out)
            cmp("init cost", m_c, r_c, out)
        if "steps" in args.levels:
            names = ["black_close", "black_far", "black_refine", "red_close", "red_far", "red_refine"]
            mine_map = [(0, 1), (0, 2), (0, 4), (1, 1), (1, 2), (1, 4)]
            s_n4, s_c = r_n4, r_c
            for k, nm in enumerate(names):
                n_n4, n_c, _ = ref.steps(sc, [k + 1], norm4=s_n4, cost=s_c)
                for trust in (0, 1):
                    ctx.set_option("trust_state", trust)
                    ctx.set_state(s_n4, s_c)
                    ctx.phase(*mine_map[k])
                    m_n4, m_c = ctx.get_state()
                    cmp("%s planes (trust=%d)" % (nm, trust), m_n4, n_n4, out)
                    cmp("%s cost (trust=%d)" % (nm, trust), m_c, n_c, out)
                s_n4, s_c = n_n4, n_c
            # fused colour launch vs three reference kernels
            b_n4, b_c, _ = ref.steps(sc, [1, 2, 3], norm4=r_n4, cost=r_c)
            ctx.set_option("trust_state", 1)
            ctx.set_state(r_n4, r_c)
            ctx.phase(0, 7)
            m_n4, m_c = ctx.get_state()
            cmp("black fused planes", m_n4, b_n4, out)
            cmp("black fused cost", m_c, b_c, out)
            fin_n4, fin_c, _ = ref.steps(sc, [7], norm4=b_n4, cost=b_c)
            ctx.finalize()
            m_n4, m_c = ctx.get_state()
            cmp("finalize planes", m_n4, fin_n4, out)
            ctx.set_option("trust_state", 0)
        if "full" in args.levels:
            f_n4, f_c, printed_s, wall_ms = ref.run(sc)
            for opts in ({}, {"prune": 0, "dedupe": 0, "memo": 0}):
                ls, ms, st = api.runcuda(sc, options=opts)
                tag = "full%s" % ("" if not opts else " (no prune/dedupe)")
                cmp(tag + " norm4", ls.norm4, f_n4, out)
                cmp(tag + " cost", ls.c, f_c, out)
                out[tag + " ms"] = ms
                out[tag + " stats"] = st
            out["ref printed_s"] = printed_s
            out["speedup_vs_ref"] = printed_s * 1000.0 / out["full ms"]
            try:
                drop = pyref.Harness("dropin")
                d_n4, d_c, d_s, d_ms = drop.run(sc)
                cmp("dropin harness norm4", d_n4, f_n4, out)
                cmp("dropin harness cost", d_c, f_c, out)
                out["dropin printed_s"] = d_s
            except Exception as e:      # noqa: BLE001
                out["dropin error"] = repr(e)
        print(json.dumps(out, indent=1))
        ctx.close()


if __name__ == "__main__":
    main()
