"""CPU checks of the clouds coloured from a `clr` image in its own type: the PLY header of every colour type, the PLY reader's
integer colour properties, and the decoding of integer columns by tests/dsm_typed_oracle.py."""
import numpy as np
import pytest

import dsm_oracle as DO
import dsm_typed_oracle as D
import ply_oracle as P

# numpy colour type -> the PLY type name plyfile writes for it
PLY_NAMES = {np.int8: "char", np.uint8: "uchar", np.int16: "short", np.uint16: "ushort", np.int32: "int", np.uint32: "uint",
             np.float32: "float", np.float64: "double"}
COMMENTS = ["created by S2P", "projection: CRS epsg:32740"]


@pytest.mark.parametrize("dtype", sorted(PLY_NAMES, key=lambda t: np.dtype(t).str))
def test_header_of_every_colour_type(dtype):
    from s2p_b200 import cloud
    from s2p_b200.engine import Engine
    for nb in (1, 3, 4):
        for conf in (False, True):
            records = np.zeros(17, Engine.ply_dtype(nb, conf, dtype))
            assert records.dtype == P.ply_dtype(nb, conf, dtype)
            assert cloud.ply_header(records, COMMENTS) == P.ply_header(17, COMMENTS, nb, conf, PLY_NAMES[dtype])


def test_engine_dtype_is_the_literal_writer_dtype():
    """the record the literal writer builds for colours of each type, band count and confidence"""
    from s2p_b200.engine import Engine
    xyz = np.zeros((2, 3, 3))
    for dtype in PLY_NAMES:
        for nb in (1, 3, 4):
            for conf in (None, np.ones((2, 3), np.float32)):
                want = P.ply_records_literal(xyz, np.zeros((nb, 2, 3), dtype), conf).dtype
                assert Engine.ply_dtype(nb, conf is not None, dtype) == want


def _ply(tmp_path, props):
    p = tmp_path / "c.ply"
    p.write_bytes(b"ply\nformat binary_little_endian 1.0\nelement vertex 0\n" +
                  b"".join(b"property %s %s\n" % (t.encode(), n.encode()) for t, n in props) + b"end_header\n")
    return str(p)


@pytest.mark.parametrize("ctype", ["char", "short", "ushort", "int", "uint", "int8", "int16", "uint16", "int32", "uint32"])
def test_reader_accepts_integer_colours(tmp_path, ctype):
    from s2p_b200 import rasterization as R
    for nb in (3, 4):
        props = [("double", "x"), ("double", "y"), ("double", "z")] + [(ctype, c) for c in ("red", "green", "blue", "ir")[:nb]]
        cloud = R.read_ply(_ply(tmp_path, props + [("float", "confidence")]))
        assert cloud.names == [n for _, n in props] + ["confidence"]
        size = np.dtype(D.NUMPY[cloud.types[3]]).itemsize
        assert cloud.dtype.itemsize == 24 + nb * size + 4


@pytest.mark.parametrize("prop", [("int", "x"), ("ushort", "y"), ("short", "z"), ("ushort", "confidence"), ("uint", "alpha"),
                                  ("char", "nx")])
def test_reader_refuses_other_integer_properties(tmp_path, prop):
    from s2p_b200 import rasterization as R
    props = [("double", "x"), ("double", "y"), ("double", "z"), ("ushort", "red"), ("ushort", "green"), ("ushort", "blue")]
    props = [prop if n == prop[1] else (t, n) for t, n in props]
    if prop not in props:
        props.append(prop)
    with pytest.raises(R.UnsupportedPly):
        R.read_ply(_ply(tmp_path, props))


def test_integer_columns_decode_as_astype_float64(tmp_path):
    """the typed oracle and the reader turn every integer colour type into float64 as astype(np.float64) does, extremes included"""
    from s2p_b200 import rasterization as R
    rng = np.random.default_rng(4)
    for t in (D.I8, DO.U8, D.I16, D.U16, D.I32, D.U32):
        info = np.iinfo(np.dtype(D.NUMPY[t]))
        vals = np.r_[info.min, info.max, 0, rng.integers(info.min, int(info.max) + 1, 50)].astype(D.NUMPY[t])
        types = [DO.F64, DO.F64, DO.F64, t, t, t]
        props = np.stack([rng.normal(0, 1, len(vals)), rng.normal(0, 1, len(vals)), rng.normal(0, 1, len(vals)), vals,
                          vals[::-1], np.roll(vals, 3)], axis=1)
        rec = D.records_of(props, types)
        names = ["x", "y", "z", "red", "green", "blue"]
        cols = D.columns(rec, names, types)
        assert np.array_equal(cols[:, 3], vals.astype(np.float64))
        assert np.array_equal(cols[:, 4], vals[::-1].astype(np.float64))
        p = tmp_path / ("c%d.ply" % t)
        D.write_ply(p, rec, names, types)
        cloud = R.read_ply(str(p))
        assert cloud.types == types
        assert np.array_equal(np.stack([cloud.column(k) for k in range(6)], 1), cols)


def test_typed_oracle_agrees_with_the_dsm_oracle():
    """on double, float and uchar, the typed oracle's records and columns are those of tests/dsm_oracle.py"""
    types = DO.S2P_CONF_TYPES
    vals = DO.seeded_cloud(2, 300, 1000.0, 2000.0, 0.5, 30, 20, types=types)
    names = ["x", "y", "z", "red", "green", "blue", "confidence"]
    rec = DO.records_of(vals, types)
    assert np.array_equal(D.records_of(vals, types), rec)
    assert np.array_equal(D.columns(rec, names, types), DO.columns(rec, names, types))
