"""Writes tests/golden/census_windows.npz: outputs of the reference `mgm` binary (oracle/_ref/mgm, OMP_NUM_THREADS=1) at
CENSUS_NCC_WIN 4, 9 and 11 on one seeded pair with no-data strips, so that machines without the reference's sources have a
fixed target for the census windows beyond 7 and the even ones.  Run from the repository root where oracle/_ref is built:

    python tests/golden/make_golden_census_windows.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import oracle as O            # noqa: E402
from s2p_b200.synth import make_pair      # noqa: E402

WINS = (4, 9, 11)
DMIN, DMAX = -12, 11


def main():
    if not O.have_ref():
        raise SystemExit("oracle/_ref/mgm is not built")
    ref, sec, _ = make_pair(48, 96, DMIN, DMAX, seed=21, nan_border=0.04)
    out = dict(ref=ref, sec=sec, dmin=np.int32(DMIN), dmax=np.int32(DMAX), wins=np.array(WINS, np.int32))
    for win in WINS:
        r = O.run_ref(ref, sec, DMIN, DMAX, O.mgm_params(census_win=win), threads=1)
        for k in ("disp", "conf", "dispR"):
            out["%s_%d" % (k, win)] = r[k]
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "census_windows.npz"), **out)


if __name__ == "__main__":
    main()
