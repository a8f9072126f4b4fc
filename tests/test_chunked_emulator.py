"""The experimental chunk-skipping aggregation kernel (s2p_b200/csrc/agg_chunked.cuh) replayed on the CPU by
scripts/chunked_emulator.py -- same ring slots, guards, spans, staging slots and range words -- must reproduce the
oracle's aggregated volume bit for bit; the first version of the kernel's neighbour masking must not."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(args, env=None):
    e = dict(os.environ, **(env or {}))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "chunked_emulator.py")] + [str(a) for a in args],
                       capture_output=True, text=True, env=e, timeout=250)
    assert r.returncode == 0, r.stderr[-1500:]
    return r.stdout


@pytest.mark.parametrize("dp,h,w,tsgm", [(64, 20, 24, 3), (96, 18, 35, 4), (512, 17, 20, 2), (64, 33, 9, 1)])
def test_emulated_kernel_equals_oracle(dp, h, w, tsgm):
    out = _run([dp, h, w, tsgm, 3])                              # skipped chunks are left untouched (chunk-skipping WTA)
    assert ": 0 of " in out and "skipped chunks untouched: True" in out, out
    assert "chunk-skipping WTA: 0 disparities and 0 confidences" in out, out


def test_emulator_catches_the_chunk_edge_bug():
    out = _run([64, 20, 24, 3, 0], env={"EMU_BUGGY": "1"})
    assert ": 0 of " not in out
