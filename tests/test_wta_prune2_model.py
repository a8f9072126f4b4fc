"""The claims the two-stage pruned WTA rests on (wta_pruned_kernel, DESIGN.md 3.2), checked on the CPU: pass 0 read on the
dilated survivors {d : C[d] <= S[d0]}, passes 1-7 on {d : L_0[d] <= S[d0]} dilated and {d : C[d] <= L_q[d0]}; from those
reads alone the winner, the three values of the sub-pixel fit and every pass's last arg-minimum equal those from the full
vectors.  Census 3x3 and 7x7 (scaled costs) are where the 2^-16 slack of the bound matters."""
import os
import sys

import numpy as np
import pytest

from s2p_b200.synth import make_pair

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))


@pytest.mark.parametrize("win,tsgm,fix,nanb", [(5, 3, 1, 0.0), (5, 4, 1, 0.1), (3, 3, 1, 0.0), (3, 2, 1, 0.1),
                                               (7, 3, 1, 0.0), (7, 2, 0, 0.1), (5, 1, 0, 0.0)])
def test_two_stage_reads_decide_winner_consensus_and_fit(oracle, win, tsgm, fix, nanb):
    import wta_prune_model as M
    h, w, dmin, dmax = 9, 34, -10, 13
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=win + tsgm + 1, nan_border=nanb)
    nl = np.isnan(ref)
    lo = np.full((h, w), dmin, np.int32)
    hi = np.where(nl, dmin + 1, dmax).astype(np.int32)
    u, v = np.nan_to_num(ref, nan=0.0), np.nan_to_num(sec, nan=0.0)
    D = dmax - dmin + 1
    C = oracle.port.costvolume(u, v, lo, hi, dmin, D, win)
    So = oracle.port.aggregate(C, lo, hi, dmin, 8.0, 32.0, 8, tsgm, fix)[0]
    Ls = M.pass_volumes(C, 8.0, 32.0, tsgm)
    fin = np.isfinite(So)
    # S >= L_0 within the slack the kernel allows (exact for the integer costs of 5x5)
    assert np.all(So[fin] >= Ls[0][fin] * np.float32(1 - 2.0 ** -18))
    masks = M.two_stage(C, M.probe_value(C, So, "cmin"), Ls)
    assert len(masks) == 8
    M.check_claims(C, So, masks, Ls)
