"""Records what the reference's weight-map pipeline of algo == 'mgm_multi_lsd' computes for the cases of
tests/lsd_cases.py, for the machines where oracle/_ref is not built (it needs the reference's sources):
tests/golden/lsd_weights.npz holds, per case, the digest of the input image, the pipeline's exit status, the first bytes
qauto writes into its pipe, lsd's stdout and stderr, the weights plambda writes, and the segments lsd finds when it is
given qauto's output as a PGM file.
    python tests/golden/make_golden_lsd.py        (after __graft_entry__.build() has built oracle/_ref)
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))


def main():
    import lsd_cases as C
    from oracle import lsd_oracle as L
    from oracle import oracle as O
    assert L.have_ref_lsd(), "oracle/_ref is not built"
    rec = {}
    for name, make in sorted(C.CASES.items()):
        img = make()
        r = L.ref_lsd_pipeline(img)
        pgm = L.ref_lsd_on_pgm(img) if np.isfinite(img).sum() > round(0.05 * img.size) else ""
        rec[name + "/digest"] = np.array(O.digest(img))
        rec[name + "/status"] = np.array(r["status"])
        rec[name + "/qauto_head"] = np.array(r["qauto_out"][:6])
        rec[name + "/lsd_out"] = np.array(r["lsd_out"])
        rec[name + "/lsd_err"] = np.array(r["lsd_err"])
        rec[name + "/weights"] = r["weights"]
        rec[name + "/pgm_segments"] = np.array(len(pgm.splitlines()))
        print("%-22s %4dx%-4d status %d, qauto %r, lsd %r, %d segments from a PGM, weights in [%g, %g]" % (
            name, img.shape[1], img.shape[0], r["status"], r["qauto_out"][:6], r["lsd_err"].strip(),
            len(pgm.splitlines()), r["weights"].min(), r["weights"].max()))
    np.savez_compressed(C.RECORDED, **rec)


if __name__ == "__main__":
    main()
