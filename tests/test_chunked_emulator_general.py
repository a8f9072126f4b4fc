"""The chunk-skipping aggregation's general flavour (float costs, a weight image, penalties P*w with the reference build's
rounding) replayed on the CPU by scripts/chunked_emulator.py with the kernel's warps and pipeline depth for the slab:
the emulated volume must equal the oracle's weighted aggregation bit for bit, and the chunk-skipping WTA its result."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("dp,h,w,tsgm", [(576, 12, 14, 1), (640, 11, 13, 2), (1056, 9, 11, 3), (1088, 10, 9, 4)])
def test_emulated_general_kernel_equals_oracle(dp, h, w, tsgm):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "chunked_emulator.py"), str(dp), str(h), str(w), str(tsgm), "4"],
                       capture_output=True, text=True, env=dict(os.environ, EMU_GENERAL="1"), timeout=250)
    assert r.returncode == 0, r.stderr[-1500:]
    out = r.stdout
    assert "general, DP %d" % dp in out and "(%d warps, 2 stages)" % (8 if dp <= 1024 else 2) in out, out
    assert ": 0 of " in out and "skipped chunks untouched: True" in out, out
    assert "chunk-skipping WTA: 0 disparities and 0 confidences" in out, out
