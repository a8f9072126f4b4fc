"""The CPU oracle against the reference binary for the float-cost flavour beyond 512 labels: what
tests/test_gpu_wide_general.py compares the GPU with.  The binary's digests are kept in
tests/golden/wide_general_ref_outputs.json; where oracle/_ref is built the binary also runs live and must still give them."""
import json
import os

import numpy as np
import pytest

from s2p_b200.synth import make_pair

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wide_general_ref_outputs.json")


def _weights(shape, seed, ones=0.6):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0, 255, shape)
    w = np.maximum(((255 - x) / 255) ** 2, 0.1).astype(np.float32)
    w[rng.random(shape) < ones] = 1.0
    return w


@pytest.mark.parametrize("cost,tsgm,dmin,dmax", [(4, 3, -300, 299), (1, 4, -600, 500)])
def test_port_weighted_distance_beyond_512_labels_matches_reference_binary(oracle, cost, tsgm, dmin, dmax):
    h, w = 20, 640
    ref, sec, _ = make_pair(h, w, dmin, dmax, seed=17 + cost, nan_border=0.03)
    wl, wr = _weights((h, w), 21), _weights((h, w), 22, 0.3)
    P = oracle.mgm_params(dct_shift=1, cost=cost, tsgm=tsgm, P1=12.0, P2=48.0)
    want = json.load(open(GOLDEN))["%s-tsgm%d-[%d,%d]" % (oracle.COSTS[cost], tsgm, dmin, dmax)]
    if os.access(os.path.join(oracle.REF_DIR, "mgm"), os.X_OK):
        assert oracle.ref_mgm_outputs(ref, sec, dmin, dmax, P, wl=wl, wr=wr) == want, "the reference binary no longer gives the recorded digests"
    d, c, dr = oracle.port.mgm(ref, sec, dmin, dmax, P, wl, wr)
    ours = dict(disp=d, conf=c, dispR=dr)
    assert sorted(want) == sorted(ours)
    bad = [k for k in sorted(ours) if oracle.digest(ours[k]) != want[k]]
    assert not bad, "differs from the reference binary: %s" % ", ".join(bad)
