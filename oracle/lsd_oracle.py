"""TEST INFRASTRUCTURE ONLY: the regularity weights of algo == 'mgm_multi_lsd', run as the reference runs them.

``ref_lsd_pipeline`` runs the shell pipeline of s2p/block_matching.py:202-217,

    qauto IM | lsd - - | cut -d' ' -f1,2,3,4 | pview segments W H | plambda - "255 x - 255 / 2 pow 0.1 fmax" -o OUT

with /bin/sh and oracle/_ref (oracle/lsd.mk) first on PATH.  Two `tee`s record what flows between the stages without
changing it: the bytes qauto writes into its pipe and the text lsd writes into its own.  The image goes in as a PFM file
and the weights come back as one (iio is built without the image libraries); the stages between them see what they see
in s2p, because iio picks the format of a stream written to "-" from the data, not from a file name.

``ref_lsd_on_pgm`` runs lsd on qauto's output saved as a PGM file, the only format lsd_cmd.c reads: the segments the
detector finds in the quantised image when it is given one it can read.
"""
import os
import shutil
import subprocess
import tempfile

import numpy as np

from . import oracle as O

TOOLS = ("qauto", "lsd", "pview", "plambda")
WEIGHT_LAW = "255 x - 255 / 2 pow 0.1 fmax"


def have_ref_lsd():
    return all(os.access(os.path.join(O.REF_DIR, t), os.X_OK) for t in TOOLS)


def _env():
    env = dict(os.environ)
    env["PATH"] = O.REF_DIR + os.pathsep + env.get("PATH", "")
    env.pop("LINN", None)                # pview reads it from the environment; s2p never sets it (70)
    return env


def ref_lsd_pipeline(img):
    """-> dict: ``weights`` float32 (h, w), what plambda wrote; ``qauto_out`` bytes, what qauto wrote into the pipe;
    ``lsd_out`` / ``lsd_err`` str, what lsd wrote to stdout / stderr; ``status``, the pipeline's exit status (that of
    its last command, as /bin/sh reports it to common.run)."""
    img = np.asarray(img, np.float32)
    h, w = img.shape
    tmp = tempfile.mkdtemp(prefix="s2pb_lsd_")
    try:
        im, out = os.path.join(tmp, "im.pfm"), os.path.join(tmp, "w.pfm")
        qo, lo, le = (os.path.join(tmp, f) for f in ("qauto.out", "lsd.out", "lsd.err"))
        O.write_pfm(im, img)
        cmd = ("qauto %s | tee %s | lsd  -  - 2>%s | tee %s | cut -d' ' -f1,2,3,4 | pview segments %d %d | "
               "plambda -  \"%s\" -o %s" % (im, qo, le, lo, w, h, WEIGHT_LAW, out))
        r = subprocess.run(cmd, shell=True, executable="/bin/sh", env=_env(),
                           stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        res = dict(status=r.returncode, weights=O.read_pfm(out) if os.path.exists(out) else None)
        with open(qo, "rb") as f:
            res["qauto_out"] = f.read()
        for k, p in (("lsd_out", lo), ("lsd_err", le)):
            with open(p) as f:
                res[k] = f.read()
        return res
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def ref_lsd_on_pgm(img):
    """-> str: lsd's output (7 columns per segment) on ``qauto IM q.pgm``."""
    tmp = tempfile.mkdtemp(prefix="s2pb_lsd_")
    try:
        im, q = os.path.join(tmp, "im.pfm"), os.path.join(tmp, "q.pgm")
        O.write_pfm(im, np.asarray(img, np.float32))
        tool = lambda t: os.path.join(O.REF_DIR, t)
        subprocess.run([tool("qauto"), im, q], env=_env(), check=True,
                       stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        return subprocess.run([tool("lsd"), q, "-"], env=_env(), check=True,
                              stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
