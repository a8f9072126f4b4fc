"""The UTM oracle (tests/utm_oracle.py) on the CPU: the 50-digit truth against facts that need no series, the float64
restatement of the kernel against the truth, and the reading of output CRSs (s2p_b200.projection)."""
import mpmath as mp
import numpy as np
import pytest

import utm_oracle as U


def _lonlat(seed, n, zone, dlon=4.0):
    rng = np.random.default_rng(seed)
    return np.stack([U.lon0_of(zone) + rng.uniform(-dlon, dlon, n), rng.uniform(-80.0, 84.0, n)], axis=1)


@pytest.mark.parametrize("lat", [0.0, 1e-7, 7.5, 45.0, -33.25, 60.0, 80.0, -80.0, 84.0, 89.999])
def test_truth_central_meridian_is_k0_times_the_arc(lat):
    for south in (False, True):
        x, y = U.truth(U.lon0_of(40), lat, 40, south)
        with mp.workdps(U.DPS):
            assert abs(x - U.FE) < mp.mpf("1e-30")
            assert abs(y - (U.FN_SOUTH if south else 0) - U.K0 * U.meridian_arc_quad(lat)) < mp.mpf("1e-12")


def test_truth_origin_of_the_zone():
    for zone in (1, 31, 60):
        x, y = U.truth(U.lon0_of(zone), 0.0, zone, False)
        assert float(x) == 500000.0 and abs(y) < mp.mpf("1e-30")
        x, y = U.truth(U.lon0_of(zone), 0.0, zone, True)
        assert float(x) == 500000.0 and float(y) == 10000000.0


@pytest.mark.parametrize("dlon,lat", [(0.5, 10.0), (3.0, -45.0), (4.0, 70.0), (2.25, 0.0)])
def test_truth_easting_is_antisymmetric(dlon, lat):
    zone = 17
    xe, ye = U.truth(U.lon0_of(zone) + dlon, lat, zone, False)
    xw, yw = U.truth(U.lon0_of(zone) - dlon, lat, zone, False)
    with mp.workdps(U.DPS):
        assert xe > U.FE
        assert abs((xe - U.FE) + (xw - U.FE)) < mp.mpf("1e-30")
        assert abs(ye - yw) < mp.mpf("1e-30")


def test_host_coefficients_are_the_exact_series():
    """the order-6 polynomials in n the host evaluates against the coefficients the truth computes at 50 digits (Krueger's
    alpha) or here by the same Fourier projection (chi - phi as a function of phi): they differ by O(n^7) ~ 4e-20"""
    cbg, gtu, _ = U.coefficients()
    _, alpha = U._series()
    for j in range(6):
        assert abs(float(alpha[j]) - gtu[j]) < 2e-19, j
    with mp.workdps(U.DPS):
        N = 64
        samples = []
        for k in range(N):
            p = mp.pi * k / N
            if k in (0, N // 2):
                v = mp.mpf(0)
            elif p < mp.pi / 2:
                v = U._chi(p) - p
            else:
                v = -(U._chi(mp.pi - p) - (mp.pi - p))
            samples.append((p, v))
        for j in range(6):
            c = 2 * mp.fsum(v * mp.sin(2 * (j + 1) * p) for p, v in samples) / N
            assert abs(float(c) - cbg[j]) < 5e-19, j


@pytest.mark.parametrize("zone,south", [(1, False), (31, False), (40, True), (60, True)])
def test_restatement_within_1e7_m_of_the_truth(zone, south):
    ll = _lonlat(zone, 120, zone)
    ll = np.concatenate([ll, [[U.lon0_of(zone) + 4.0, -80.0], [U.lon0_of(zone) - 4.0, 84.0], [U.lon0_of(zone) + 3.0, 0.0]]])
    got = U.restate(np.concatenate([ll, np.zeros((len(ll), 1))], axis=1), zone, south)
    want = U.truth_array(ll, zone, south)
    assert np.abs(got[:, :2] - want).max() < 1e-7


def test_restatement_nan_inf_and_altitude():
    p = np.array([[3.0, 45.0, 123.456], [np.nan, 45.0, 1.0], [3.0, np.nan, 1.0], [3.0, 45.0, np.nan], [3.0, 91.0, 5.0],
                  [3.0 + 360.0 - 1.0, 10.0, -7.0]])
    out = U.restate(p, 31, False)
    assert out[0, 2] == 123.456
    assert np.isnan(out[1:4]).all()
    assert np.isposinf(out[4]).all()
    assert np.abs(out[5, :2] - U.restate(np.array([[2.0, 10.0, -7.0]]), 31, False)[0, :2]).max() < 1e-6
    assert out[5, 2] == -7.0


class _Crs:
    def __init__(self, code):
        self.code = code

    def to_epsg(self):
        return self.code


def test_output_crs_targets():
    from s2p_b200.projection import epsg_of, utm_target
    assert epsg_of("epsg:32740") == 32740 and epsg_of("EPSG:4326") == 4326 and epsg_of(32631) == 32631
    assert epsg_of(np.int64(4979)) == 4979 and epsg_of(_Crs(32601)) == 32601
    assert epsg_of("epsg:32740+5773") is None and epsg_of(_Crs(None)) is None and epsg_of(True) is None
    assert utm_target(None) == (0, False) and utm_target("") == (0, False)
    assert utm_target("epsg:4979") == (0, False) and utm_target(4326) == (0, False)
    assert utm_target("epsg:32601") == (1, False) and utm_target("Epsg:32660") == (60, False)
    assert utm_target("epsg:32701") == (1, True) and utm_target(_Crs(32740)) == (40, True) and utm_target(32760) == (60, True)
    for other in ("epsg:32740+5773", "epsg:32600", "epsg:32661", "epsg:32700", "epsg:32761", 2154, "+proj=utm +zone=40",
                  _Crs(None), _Crs(3857)):
        assert utm_target(other) is None, other
