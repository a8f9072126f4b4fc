"""The folded workspace layout on the device: the C2-like tile resident and forced folded (CUDA-event time per tile, identical
outputs), then the 2100 x 2020 x 400-label tile with no limit, which only fits folded (time and peak device memory).

    python scripts/fold_probe.py [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from s2p_b200.engine import Engine, default_params, workspace_bytes  # noqa: E402
from s2p_b200.synth import make_pair  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(eng, reps, call):
    import torch
    out, ms = None, []
    for _ in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return out, sorted(ms[1:])[len(ms[1:]) // 2]        # median after one warm-up


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for fold_probe.json (default: print only)")
    a = ap.parse_args()
    import torch
    res = {"card": card()}
    eng = Engine(0)
    p = default_params("mgm")
    # C2-like: 1024 x 1024, 128 labels
    h = w = 1024
    dmin, dmax = -64, 63
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=2, nan_border=0.0)
    r, t_res = timed(eng, a.reps, lambda: eng.mgm(ref, sec, dmin, dmax, p, want_right=True))
    eng.set_workspace_limit(workspace_bytes(w, h, dmax - dmin + 1) - 1)
    n0 = eng.folded_calls()
    f, t_fold = timed(eng, a.reps, lambda: eng.mgm(ref, sec, dmin, dmax, p, want_right=True))
    eng.set_workspace_limit(0)
    same = all(np.array_equal(r[k], f[k], equal_nan=k != "mask") for k in ("disp", "conf", "mask", "disp_right"))
    res["c2"] = dict(tile=[w, h, dmax - dmin + 1], resident_ms=t_res, folded_ms=t_fold, folded_calls=eng.folded_calls() - n0,
                     identical=same, resident_gib=workspace_bytes(w, h, 128) / 2 ** 30,
                     folded_gib=workspace_bytes(w, h, 128, folded=True) / 2 ** 30)
    eng.close()
    # the large tile: 2100 x 2020 x 400 labels, no limit; a fresh engine so that the peak is this tile's
    eng = Engine(0)
    w, h, dmin, dmax = 2100, 2020, -200, 199
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=3, nan_border=0.0)
    torch.cuda.synchronize()
    free0, total = torch.cuda.mem_get_info()
    n0 = eng.folded_calls()
    out, t_big = timed(eng, 1, lambda: eng.mgm(ref, sec, dmin, dmax, p))
    free1, _ = torch.cuda.mem_get_info()
    res["large"] = dict(tile=[w, h, dmax - dmin + 1], ms=t_big, folded_calls=eng.folded_calls() - n0,
                        device_bytes_in_use_after=int(free0 - free1), total_bytes=int(total),
                        resident_gib=workspace_bytes(w, h, 400) / 2 ** 30, folded_gib=workspace_bytes(w, h, 400, folded=True) / 2 ** 30,
                        valid_fraction=float(np.isfinite(out["disp"]).mean()))
    eng.close()
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fold_probe.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
