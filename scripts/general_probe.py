"""Stage timings of the general matcher flavour (float cost slab, optional -wl/-wr weights) on one C2 tile,
next to the census / 8-bit cost hot path.  Usage on the GPU box: python scripts/general_probe.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from s2p_b200.engine import Engine, default_params
from s2p_b200.synth import make_pair

eng = Engine(0)
H = W = int(os.environ.get("SIZE", 1024))
dmin, dmax = -64, 63
ref, sec, _ = make_pair(H, W, dmin, dmax, seed=0)
rng = np.random.default_rng(0)
wl = np.maximum(rng.uniform(0, 1, (H, W)) ** 2, 0.1).astype(np.float32)
wr = np.maximum(rng.uniform(0, 1, (H, W)) ** 2, 0.1).astype(np.float32)
for name, kw, wts in [("census (hot path)", {}, None), ("census + weights", {}, (wl, wr)), ("ad", {"cost": "ad"}, None),
                      ("btad", {"cost": "btad"}, None), ("ncc 5x5", {"cost": "ncc"}, None), ("ncc 7x7", {"cost": "ncc", "census_win": 7}, None)]:
    p = default_params("mgm", **kw)
    for _ in range(3):
        out = eng.mgm(ref, sec, dmin, dmax, p, weights=wts)
    t = eng.last_timings(0)
    print("%-18s" % name, " ".join("%s %.3f" % (k, v) for k, v in t.items()), "ms; valid %.3f" % np.isfinite(out["disp"]).mean(), flush=True)
