"""The claims the pruned WTA's pass 0 rests on (wta_pruned_kernel, DESIGN.md 3.2), checked on the CPU: from the survivors
{d : C[d] <= S[d0]} dilated by one slot alone, the winner, the three values of the sub-pixel fit and every pass's last
arg-minimum equal those from the full vectors.  Pass volumes from scripts/wta_prune_model.py's numpy restatement of the scan, pinned to the oracle's S."""
import os
import sys

import numpy as np
import pytest

from s2p_b200.synth import make_pair

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))


@pytest.mark.parametrize("win,tsgm,fix,nanb", [(5, 3, 1, 0.0), (5, 4, 1, 0.1), (3, 3, 1, 0.0), (7, 2, 0, 0.1), (5, 1, 0, 0.0)])
def test_survivors_decide_winner_consensus_and_fit(oracle, win, tsgm, fix, nanb):
    import wta_prune_model as M
    h, w, dmin, dmax = 9, 34, -10, 13
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=win + tsgm, nan_border=nanb)
    nl = np.isnan(ref)
    lo = np.full((h, w), dmin, np.int32)
    hi = np.where(nl, dmin + 1, dmax).astype(np.int32)
    u, v = np.nan_to_num(ref, nan=0.0), np.nan_to_num(sec, nan=0.0)
    D = dmax - dmin + 1
    C = oracle.port.costvolume(u, v, lo, hi, dmin, D, win)
    So = oracle.port.aggregate(C, lo, hi, dmin, 8.0, 32.0, 8, tsgm, fix)[0]
    Ls = M.pass_volumes(C, 8.0, 32.0, tsgm)
    if win == 5:            # integer costs: the numpy sums are the oracle's bit for bit (scaled costs round in the fma)
        fin = np.isfinite(So)
        assert np.array_equal(M.sum_passes(Ls, C, fix)[fin], So[fin])
    for L in Ls:
        assert np.all(L >= C)
    assert np.all(So[np.isfinite(So)] >= C[np.isfinite(So)] * np.float32(1 - 2.0 ** -18))
    for rule in ("cmin", "best", "cmin+prev"):
        s, d = M.survivors(C, M.probe_value(C, So, rule))
        M.check_claims(C, So, d, Ls)
