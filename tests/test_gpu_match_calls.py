"""Matcher calls that run at the same time on different slots of one context keep to themselves: a call's timeout aborts only
its own slot, and the PKR images of one call are written by that call alone.  s2pb_rectify_match equals its two steps."""
import threading

import numpy as np
import pytest

from s2p_b200.synth import make_pair
from util import same

pytestmark = pytest.mark.gpu
LONG_MS = 600000     # the timeout bench.py gives every call


def _device_mgm(engine, torch, slot, ref, sec, dmin, dmax, params, stream):
    """Engine.mgm_device on `slot` and `stream` -> (disp, conf, mask) on the host; S2pbError propagates"""
    h, w = ref.shape
    with torch.cuda.stream(stream):
        a, b = torch.from_numpy(ref).cuda(), torch.from_numpy(sec).cuda()
        disp = torch.empty((h, w), dtype=torch.float32, device="cuda")
        conf = torch.empty_like(disp)
        mask = torch.empty((h, w), dtype=torch.uint8, device="cuda")
    stream.synchronize()
    engine.mgm_device(slot, a.data_ptr(), b.data_ptr(), w, h, dmin, dmax, params, disp.data_ptr(), conf.data_ptr(),
                      mask.data_ptr(), nodata_hint=0, stream=stream.cuda_stream)
    stream.synchronize()
    return disp.cpu().numpy(), conf.cpu().numpy(), mask.cpu().numpy()


def _run_both(fa, fb):
    """fa and fb on two host threads at once -> (result or exception of fa, result or exception of fb)"""
    out = [None, None]

    def run(k, f):
        try:
            out[k] = f()
        except Exception as e:      # noqa: BLE001 - handed to the test
            out[k] = e
    th = [threading.Thread(target=run, args=(k, f)) for k, f in enumerate((fa, fb))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return out


def _same_outputs(got, want):
    return all(same(g, w) if g.dtype != np.uint8 else np.array_equal(g, w) for g, w in zip(got, want))


@pytest.mark.parametrize("algo", ["mgm", "mgm_multi"])
def test_timeout_aborts_only_its_own_slot(engine, algo):
    import torch
    from s2p_b200 import _lib
    from s2p_b200.engine import S2pbError, default_params
    big, big_sec, _ = make_pair(512, 512, -100, 100, seed=1)
    ref, sec, _ = make_pair(192, 256, -24, 23, seed=4)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    pb = default_params(algo, timeout_ms=LONG_MS)
    small = _device_mgm(engine, torch, 0, big[:96, :128].copy(), big_sec[:96, :128].copy(), -12, 12, pb, sa)
    solo = _device_mgm(engine, torch, 1, ref, sec, -24, 23, pb, sb)
    a, b = _run_both(lambda: _device_mgm(engine, torch, 0, big, big_sec, -100, 100, default_params(algo, timeout_ms=1), sa),
                     lambda: _device_mgm(engine, torch, 1, ref, sec, -24, 23, pb, sb))
    assert isinstance(a, S2pbError) and a.code == _lib.ERR_TIMEOUT, a
    assert not isinstance(b, Exception), b
    assert _same_outputs(b, solo), "the call on slot 1 changed when slot 0 timed out"
    again = _device_mgm(engine, torch, 0, big[:96, :128].copy(), big_sec[:96, :128].copy(), -12, 12, pb, sa)
    assert _same_outputs(again, small), "slot 0 is not right after its timeout"


@pytest.mark.parametrize("algo", ["mgm", "mgm_multi"])
def test_pkr_images_belong_to_their_call(engine, algo):
    import torch
    from s2p_b200.engine import default_params
    ref, sec, _ = make_pair(160, 224, -20, 19, seed=6)
    ref2, sec2, _ = make_pair(192, 256, -24, 23, seed=7)
    p = default_params(algo)
    sb = torch.cuda.Stream()
    solo_pkr = engine.mgm(ref, sec, -20, 19, p, want_right=True, want_pkr=True)
    solo_dev = _device_mgm(engine, torch, 1, ref2, sec2, -24, 23, p, sb)
    a, b = _run_both(lambda: engine.mgm(ref, sec, -20, 19, p, want_right=True, want_pkr=True),
                     lambda: _device_mgm(engine, torch, 1, ref2, sec2, -24, 23, p, sb))
    assert not isinstance(a, Exception), a
    assert not isinstance(b, Exception), b
    for k in ("disp", "conf", "mask", "disp_right", "pkr_left", "pkr_right"):
        assert np.array_equal(a[k], solo_pkr[k], equal_nan=True), k
    assert _same_outputs(b, solo_dev), "the call on slot 1 changed beside a PKR call"


def test_rectify_match_equals_its_two_steps(engine):
    from s2p_b200 import _lib
    from s2p_b200.engine import S2pbError, default_params
    from util import load_real_pair
    z = load_real_pair()
    comp = lambda Hm, xy: np.asarray(Hm, np.float64) @ np.array([[1, 0, xy[0]], [0, 1, xy[1]], [0, 0, 1.0]])  # noqa: E731
    H1, H2 = comp(z["H1"], z["xy1"]), comp(z["H2"], z["xy2"])
    src1, src2 = z["crop1"].astype(np.float32), z["crop2"].astype(np.float32)
    h, w = z["rectified_ref"].shape
    p = default_params("mgm")
    r1, r2 = engine.homography(src1, H1, w, h), engine.homography(src2, H2, w, h)
    want = engine.mgm(r1, r2, -41, 30, p, want_right=True)
    got = engine.rectify_match(src1, H1, src2, H2, w, h, -41, 30, p, want_right=True)
    assert np.array_equal(got["rect1"], r1, equal_nan=True) and np.array_equal(got["rect2"], r2, equal_nan=True)
    for k in ("disp", "conf", "mask", "disp_right"):
        assert np.array_equal(got[k], want[k], equal_nan=True), k
    big, big_sec, _ = make_pair(512, 512, -100, 100, seed=1)
    with pytest.raises(S2pbError) as e:
        engine.rectify_match(big, np.eye(3), big_sec, np.eye(3), 512, 512, -100, 100, default_params("mgm", timeout_ms=1))
    assert e.value.code == _lib.ERR_TIMEOUT
    again = engine.rectify_match(src1, H1, src2, H2, w, h, -41, 30, p, want_right=True)
    for k in ("rect1", "rect2", "disp", "conf", "mask", "disp_right"):
        assert np.array_equal(again[k], got[k], equal_nan=True), k
