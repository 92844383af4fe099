#!/usr/bin/env python
"""Which optimisation switch changes the output at full size?  (development tool)"""
import json, os, sys
import numpy as np
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from gipuma_b200 import scene as S, api
cfg = int(sys.argv[1]) if len(sys.argv) > 1 else 2
sc = S.make_config(cfg)
base, _, _ = api.runcuda(sc, options={"prune": 0, "dedupe": 0, "memo": 0})
for name, opts in [("repeat", {"prune": 0, "dedupe": 0, "memo": 0}), ("prune", {"dedupe": 0, "memo": 0}),
                   ("dedupe", {"prune": 0, "memo": 0}), ("memo", {"prune": 0, "dedupe": 0}), ("all", {})]:
    o, ms, st = api.runcuda(sc, options=opts)
    neq = (o.norm4.view(np.uint32) != base.norm4.view(np.uint32)).any(axis=-1) | (o.c.view(np.uint32) != base.c.view(np.uint32))
    ys, xs = np.nonzero(neq)
    print(json.dumps({"switch": name, "ms": ms, "mismatched_pixels": int(neq.sum()),
                      "first": [[int(y), int(x), float(o.c[y, x]), float(base.c[y, x])] for y, x in list(zip(ys, xs))[:5]]}))
