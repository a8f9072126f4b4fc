"""Statements of the maps of S2PB_ZONE_PROJ (csrc/projection_kernels.cuh, projection.cu) on any ellipsoid.

* Lambert conic conformal, two standard parallels (EPSG method 9802):
  - ``lcc_params`` / ``lcc_restate``: the host's float64 constants and lcc_forward's arithmetic in numpy, in its operation
    order;
  - ``lcc_truth``: the formulas of IOGP Guidance Note 7-2 (sec. 3.1.1.1) as written there, m, t, n, F, r, theta, in 50-digit
    mpmath.
* Transverse Mercator (EPSG method 9807), the map of the ETRS89 UTM zones: ``tm_coefficients`` / ``tm_restate`` restate
  utm_params and utm_forward for an ellipsoid (a, f), scale k0 and origin; ``tm_truth`` is the 50-digit truth of
  tests/utm_oracle.py with the ellipsoid as a parameter.  On WGS84 they are utm_oracle's, which the tests check.

A projection is the tuple of s2p_b200.projection.Projection (method, a, rf, lon0, lat0, lat1, lat2, k0, x0, y0).
"""
import functools

import mpmath as mp
import numpy as np

DPS = 50
ORDER = 6
PI = 3.141592653589793
D2R = 0.017453292519943295
TM, LCC = 1, 2


# ------------------------------------------------------------------ float64 restatements

def lcc_params(proj):
    """(e, n, aF, rho0) of projection.cu's lcc_params, in the same float64 operations"""
    _, a, rf, _, lat0, lat1, lat2 = proj[:7]
    f = 1.0 / rf
    e2 = f * (2.0 - f)
    e = np.sqrt(e2)

    def m(phi):
        s = np.sin(phi)
        return np.cos(phi) / np.sqrt(1.0 - e2 * s * s)

    def psi(phi):
        return np.arcsinh(np.tan(phi)) - e * np.arctanh(e * np.sin(phi))
    phi1, phi2, phi0 = lat1 * D2R, lat2 * D2R, lat0 * D2R
    n = np.sin(phi1) if lat1 == lat2 else (np.log(m(phi1)) - np.log(m(phi2))) / (psi(phi2) - psi(phi1))
    aF = a * (m(phi1) * np.exp(n * psi(phi1)) / n)
    rho0 = 0.0 if abs(lat0) == 90.0 else aF * np.exp(-(n * psi(phi0)))
    return float(e), float(n), float(aF), float(rho0)


def _wrap(lam):
    return np.where(np.abs(lam) > PI, lam - 2 * PI * np.floor((lam + PI) / (2 * PI)), lam)


def lcc_restate(lonlatalt, proj):
    """(..., 3) float64 (lon, lat in degrees, alt) -> (..., 3) float64 (x, y, alt), lcc_forward's arithmetic.  NaN in any
    coordinate -> NaN in all three; |lat| > 90 or the pole away from the cone -> +inf in all three."""
    e, n, aF, rho0 = lcc_params(proj)
    lon0, x0, y0 = proj[3], proj[8], proj[9]
    p = np.asarray(lonlatalt, np.float64)
    lon, lat, alt = p[..., 0], p[..., 1], p[..., 2]
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        lam = _wrap((lon - lon0) * D2R)
        phi = lat * D2R
        pole = np.abs(np.abs(phi) - 1.5707963267948966) < 1e-10
        psi = np.arcsinh(np.tan(phi)) - e * np.arctanh(e * np.sin(phi))
        rho = np.where(pole, 0.0, aF * np.exp(-(n * psi)))
        theta = n * lam
        x = x0 + rho * np.sin(theta)
        y = y0 + (rho0 - rho * np.cos(theta))
        out = np.stack([x, y, alt], axis=-1)
        bad = ~(np.abs(lat) <= 90.0) | (pole & (phi * n <= 0.0))
    out[bad] = np.inf
    out[np.isnan(p).any(axis=-1)] = np.nan
    return out


def tm_coefficients(a, f, k0):
    """(cbg, gtu, qa) of projection.cu's tm_params, in the same float64 operations"""
    n = f / (2.0 - f)
    cbg, gtu = [0.0] * 6, [0.0] * 6
    np_ = n
    cbg[0] = n * (-2 + n * (2 / 3.0 + n * (4 / 3.0 + n * (-82 / 45.0 + n * (32 / 45.0 + n * (4642 / 4725.0))))))
    gtu[0] = n * (0.5 + n * (-2 / 3.0 + n * (5 / 16.0 + n * (41 / 180.0 + n * (-127 / 288.0 + n * (7891 / 37800.0))))))
    np_ *= n
    cbg[1] = np_ * (5 / 3.0 + n * (-16 / 15.0 + n * (-13 / 9.0 + n * (904 / 315.0 + n * (-1522 / 945.0)))))
    gtu[1] = np_ * (13 / 48.0 + n * (-3 / 5.0 + n * (557 / 1440.0 + n * (281 / 630.0 + n * (-1983433 / 1935360.0)))))
    np_ *= n
    cbg[2] = np_ * (-26 / 15.0 + n * (34 / 21.0 + n * (8 / 5.0 + n * (-12686 / 2835.0))))
    gtu[2] = np_ * (61 / 240.0 + n * (-103 / 140.0 + n * (15061 / 26880.0 + n * (167603 / 181440.0))))
    np_ *= n
    cbg[3] = np_ * (1237 / 630.0 + n * (-12 / 5.0 + n * (-24832 / 14175.0)))
    gtu[3] = np_ * (49561 / 161280.0 + n * (-179 / 168.0 + n * (6601661 / 7257600.0)))
    np_ *= n
    cbg[4] = np_ * (-734 / 315.0 + n * (109598 / 31185.0))
    gtu[4] = np_ * (34729 / 80640.0 + n * (-3418889 / 1995840.0))
    np_ *= n
    cbg[5] = np_ * (444337 / 155925.0)
    gtu[5] = np_ * (212378941 / 319334400.0)
    n2 = n * n
    qa = a * (k0 / (1 + n) * (1 + n2 * (1 / 4.0 + n2 * (1 / 64.0 + n2 / 256.0))))
    return cbg, gtu, qa


def tm_restate(lonlatalt, proj):
    """(..., 3) float64 -> (..., 3) float64, utm_forward's arithmetic with the coefficients of tm_params for proj"""
    _, a, rf, lon0, _, _, _, k0, x0, y0 = proj
    cbg, gtu, qa = tm_coefficients(a, 1.0 / rf, k0)
    p = np.asarray(lonlatalt, np.float64)
    lon, lat, alt = p[..., 0], p[..., 1], p[..., 2]
    with np.errstate(invalid="ignore", over="ignore"):
        lam = _wrap((lon - lon0) * D2R)
        phi = lat * D2R
        s2, c2 = np.sin(2.0 * phi), np.cos(2.0 * phi)
        tc2 = 2.0 * c2
        h1, h2 = np.full_like(phi, cbg[ORDER - 1]), np.zeros_like(phi)
        h = h1
        for k in range(ORDER - 2, -1, -1):
            h = -h2 + tc2 * h1 + cbg[k]
            h2, h1 = h1, h
        chi = phi + h * s2
        sc, cc, sl, cl = np.sin(chi), np.cos(chi), np.sin(lam), np.cos(lam)
        ccl = cc * cl
        xip = np.arctan2(sc, ccl)
        inv_d = 1.0 / np.hypot(sc, ccl)
        sinh_e = sl * cc * inv_d
        etap = np.arcsinh(sinh_e)
        two_inv_d = 2.0 * inv_d
        two_inv_d2 = two_inv_d * inv_d
        t = ccl * two_inv_d2
        sin2x, cos2x = sc * t, ccl * t - 1.0
        sinh2e, cosh2e = sinh_e * two_inv_d, two_inv_d2 - 1.0
        r, q = 2.0 * cos2x * cosh2e, -2.0 * sin2x * sinh2e
        hr, hi = np.full_like(phi, gtu[ORDER - 1]), np.zeros_like(phi)
        hr1, hi1 = np.zeros_like(phi), np.zeros_like(phi)
        for k in range(ORDER - 2, -1, -1):
            hr2, hi2, hr1, hi1 = hr1, hi1, hr, hi
            hr = -hr2 + r * hr1 - q * hi1 + gtu[k]
            hi = -hi2 + q * hr1 + r * hi1
        sr, si = sin2x * cosh2e, cos2x * sinh2e
        xi = xip + (sr * hr - si * hi)
        eta = etap + (sr * hi + si * hr)
        x = qa * eta + x0
        y = qa * xi + y0
        bad = ~(np.abs(lat) <= 90.0) | (np.abs(eta) > 2.623395162778)
        out = np.stack([x, y, alt], axis=-1)
    out[bad] = np.inf
    out[np.isnan(p).any(axis=-1)] = np.nan
    return out


def restate(lonlatalt, proj):
    """the device's map of proj, by its method"""
    return (tm_restate if proj[0] == TM else lcc_restate)(lonlatalt, proj)


# ------------------------------------------------------------------ 50-digit truths

def _ell(a, rf):
    f = 1 / mp.mpf(rf)
    e2 = f * (2 - f)
    return mp.mpf(a), e2, mp.sqrt(e2)


def lcc_truth(lon, lat, proj):
    """(x, y) in metres, as mpf, of (lon, lat) in degrees (floats, taken exactly): Guidance Note 7-2's LCC 2SP formulas
    m = cos phi / sqrt(1 - e^2 sin^2 phi), t = tan(pi/4 - phi/2) / ((1 - e sin phi) / (1 + e sin phi))^(e/2),
    n = (ln m1 - ln m2) / (ln t1 - ln t2), F = m1 / (n t1^n), r = a F t^n, theta = n (lambda - lambda_F),
    E = E_F + r sin theta, N = N_F + r_F - r cos theta; longitudes reduced to [-180, 180] from lambda_F as PROJ reduces them"""
    _, a_, rf, lon0, lat0, lat1, lat2, _, x0, y0 = proj
    with mp.workdps(DPS):
        a, e2, e = _ell(a_, rf)
        rad = mp.pi / 180

        def m(phi):
            return mp.cos(phi) / mp.sqrt(1 - e2 * mp.sin(phi) ** 2)

        def t(phi):
            s = mp.sin(phi)
            return mp.tan(mp.pi / 4 - phi / 2) / ((1 - e * s) / (1 + e * s)) ** (e / 2)
        p1, p2, pf = mp.mpf(lat1) * rad, mp.mpf(lat2) * rad, mp.mpf(lat0) * rad
        n = mp.sin(p1) if lat1 == lat2 else (mp.log(m(p1)) - mp.log(m(p2))) / (mp.log(t(p1)) - mp.log(t(p2)))
        F = m(p1) / (n * t(p1) ** n)
        rF = a * F * t(pf) ** n
        dl = mp.mpf(lon) - mp.mpf(lon0)
        dl = dl - 360 * mp.floor((dl + 180) / 360)
        r = a * F * t(mp.mpf(lat) * rad) ** n
        theta = n * dl * rad
        return x0 + r * mp.sin(theta), y0 + rF - r * mp.cos(theta)


def _arc(phi, a, e2):
    s, c = mp.sin(phi), mp.cos(phi)
    return a * (mp.ellipe(phi, e2) - e2 * s * c / mp.sqrt(1 - e2 * s * s))


def _chi(phi, e):
    return mp.atan(mp.sinh(mp.asinh(mp.tan(phi)) - e * mp.atanh(e * mp.sin(phi))))


@functools.lru_cache(maxsize=None)
def _series(a_, rf):
    """(A, alpha_1..alpha_8) of the ellipsoid (a_, 1/rf): the rectifying radius and Krueger's coefficients at DPS digits, by
    the Fourier projection of tests/utm_oracle.py"""
    with mp.workdps(DPS + 10):
        a, e2, e = _ell(a_, rf)
        half_pi = mp.pi / 2
        A = _arc(half_pi, a, e2) / half_pi

        def g(chi):                     # mu - chi on [-pi/2, pi/2]
            if chi == 0 or abs(chi) == half_pi:
                return mp.mpf(0)
            phi = mp.findroot(lambda p: _chi(p, e) - chi, chi)
            return _arc(phi, a, e2) / A - chi
        N = 64
        samples = []
        for k in range(N):
            chi = mp.pi * k / N
            samples.append((chi, g(chi) if chi <= half_pi else -g(mp.pi - chi)))
        alpha = [2 * mp.fsum(v * mp.sin(2 * j * c) for c, v in samples) / N for j in range(1, 9)]
        return A, alpha


def tm_truth(lon, lat, proj):
    """(x, y) in metres, as mpf, of (lon, lat) in degrees (floats, taken exactly) in the transverse Mercator proj"""
    _, a_, rf, lon0, _, _, _, k0, x0, y0 = proj
    A, alpha = _series(float(a_), float(rf))
    with mp.workdps(DPS):
        _, _, e = _ell(a_, rf)
        dl = mp.mpf(lon) - mp.mpf(lon0)
        dl = dl - 360 * mp.floor((dl + 180) / 360)
        lam = dl * mp.pi / 180
        phi = mp.mpf(lat) * mp.pi / 180
        chi = _chi(phi, e) if abs(lat) < 90 else phi
        sc, cc = mp.sin(chi), mp.cos(chi)
        xip = mp.atan2(sc, cc * mp.cos(lam))
        etap = mp.asinh(mp.sin(lam) * cc / mp.hypot(sc, cc * mp.cos(lam)))
        zp = mp.mpc(xip, etap)
        z = zp + mp.fsum(alpha[j - 1] * mp.sin(2 * j * zp) for j in range(1, 9))
        return x0 + mp.mpf(k0) * A * z.imag, y0 + mp.mpf(k0) * A * z.real


def truth_array(lonlat, proj):
    """(n, 2) degrees -> (n, 2) float64 metres"""
    fn = tm_truth if proj[0] == TM else lcc_truth
    return np.array([[float(v) for v in fn(float(lo), float(la), proj)] for lo, la in np.asarray(lonlat)])


# ------------------------------------------------------------------ a stand-in for pyproj

def fake_pyproj(shift=0.0, codes=None):
    """A module with pyproj's ``Transformer.from_crs(src, dst, always_xy=True).transform(lon, lat, z)`` for EPSG:4979 to the
    codes of s2p_b200.projection.PROJECTED (or ``codes``, a dict of them), by the float64 restatement above, x and y moved by
    ``shift`` metres: PROJ agreeing with the device (shift 0), or applying a datum shift (shift of a few decimetres)."""
    import types
    from s2p_b200.projection import PROJECTED
    table = PROJECTED if codes is None else codes
    calls = []

    class Transformer:
        def __init__(self, proj):
            self.proj = proj

        @staticmethod
        def from_crs(src, dst, always_xy=False):
            calls.append((src, dst))
            code = int(str(dst).lower().replace("epsg:", ""))
            if str(src).lower() != "epsg:4979" or not always_xy or code not in table:
                raise ValueError("no transformation from %s to %s" % (src, dst))
            return Transformer(table[code])

        def transform(self, lon, lat, z):
            out = restate(np.stack([np.asarray(lon, np.float64), np.asarray(lat, np.float64), np.asarray(z, np.float64)], -1),
                          self.proj)
            return out[..., 0] + shift, out[..., 1] + shift, out[..., 2]
    m = types.ModuleType("pyproj")
    m.Transformer = Transformer
    m.calls = calls
    return m
