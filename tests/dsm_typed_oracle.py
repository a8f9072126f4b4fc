"""TEST INFRASTRUCTURE ONLY -- the PLY vertex records of tests/dsm_oracle.py with every property type the DSM rasterisation
reads: double, float and uchar, and the integer types s2p writes for the colours of a `clr` image in its own type (char,
short, ushort, int, uint).  Each property is decoded as astype(np.float64) gives it; dsm_oracle.plyflatten folds the result."""
import numpy as np

from dsm_oracle import F32, F64, U8

I8, I16, U16, I32, U32 = 16, 17, 18, 19, 20                  # S2PB_PLY_* of the integer colour types
NUMPY = {F64: "<f8", F32: "<f4", U8: "u1", I8: "i1", I16: "<i2", U16: "<u2", I32: "<i4", U32: "<u4"}
PLY_NAME = {F64: "double", F32: "float", U8: "uchar", I8: "char", I16: "short", U16: "ushort", I32: "int", U32: "uint"}


def record_dtype(names, types):
    return np.dtype({"names": list(names), "formats": [NUMPY[int(t)] for t in types]})


def columns(records, names, types):
    """(n, nprops) float64: every property of the (n, record_bytes) uint8 records, as astype(np.float64) gives it"""
    v = np.ascontiguousarray(records).view(record_dtype(names, types)).reshape(-1)
    return np.stack([v[n].astype(np.float64) for n in names], axis=1) if len(v) else np.zeros((0, len(names)))


def records_of(props, types):
    """(n, nprops) values -> (n, record_bytes) uint8 records with the given S2PB_PLY_* types"""
    names = ["p%d" % k for k in range(len(types))]
    rec = np.zeros(len(props), record_dtype(names, types))
    for k, n in enumerate(names):
        rec[n] = props[:, k]
    return rec.view(np.uint8).reshape(len(props), -1)


def write_ply(path, records, names, types, comments=()):
    head = ["ply", "format binary_little_endian 1.0"] + ["comment %s" % c for c in comments]
    head += ["element vertex %d" % len(records)] + ["property %s %s" % (PLY_NAME[int(t)], n) for n, t in zip(names, types)]
    head += ["end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        f.write(np.ascontiguousarray(records, np.uint8).tobytes())
