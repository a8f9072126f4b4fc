"""Two statements of the WGS84 -> UTM projection (EPSG:4979 -> EPSG:326zz / 327zz) that projection_kernels.cuh computes.

* ``truth``: the transverse Mercator in 50-digit mpmath, written without the truncated series in n that the kernel uses.
  The conformal latitude and the spherical transverse Mercator are exact closed forms.  Krueger's series
  xi + i eta = zeta' + sum_j alpha_j sin(2 j zeta') is carried to j = 8, with each alpha_j computed here, at 50 digits, as the
  Fourier sine coefficient of mu - chi (rectifying minus conformal latitude, as functions of chi) that it is on the central
  meridian; mu comes from the meridian arc by the elliptic integral of the second kind.  alpha_9 is of order n^9 ~ 1e-25,
  so the truncation is far below a nanometre.  The tests check this truth against facts that need no series: the
  northing on the central meridian is k0 times the meridian arc (mpmath.quad), the origin of the zone maps to
  (500 000, 0), the easting is antisymmetric about the central meridian.
* ``restate``: the kernel's float64 arithmetic in numpy, step for step and in its operation order (Poder / Engsager, as
  PROJ runs it for +proj=utm; Karney 2011), with the coefficients the host computes.
"""
import functools

import mpmath as mp
import numpy as np

A_WGS84 = 6378137.0
F_WGS84 = 1 / 298.257223563
K0 = 0.9996
FE = 500000.0
FN_SOUTH = 10000000.0
ORDER = 6
DPS = 50


def lon0_of(zone):
    return 6.0 * zone - 183.0


# ------------------------------------------------------------------ float64 restatement of the kernel

def coefficients():
    """(cbg, gtu, qa) of projection.cu's utm_params, in the same float64 operations"""
    f = F_WGS84
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
    qa = A_WGS84 * (K0 / (1 + n) * (1 + n2 * (1 / 4.0 + n2 * (1 / 64.0 + n2 / 256.0))))
    return cbg, gtu, qa


def restate(lonlatalt, zone, south):
    """(..., 3) float64 (lon, lat in degrees, alt) -> (..., 3) float64 (x, y, alt), the kernel's arithmetic.  NaN in any
    coordinate -> NaN in all three; outside the domain -> +inf in all three."""
    cbg, gtu, qa = coefficients()
    p = np.asarray(lonlatalt, np.float64)
    lon, lat, alt = p[..., 0], p[..., 1], p[..., 2]
    d2r = 0.017453292519943295
    with np.errstate(invalid="ignore", over="ignore"):
        lam = (lon - lon0_of(zone)) * d2r
        lam = np.where(np.abs(lam) > 3.141592653589793,
                       lam - 6.283185307179586 * np.floor((lam + 3.141592653589793) / 6.283185307179586), lam)
        phi = lat * d2r
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
        x = qa * eta + FE
        y = qa * xi + (FN_SOUTH if south else 0.0)
        bad = ~(np.abs(lat) <= 90.0) | (np.abs(eta) > 2.623395162778)
        out = np.stack([x, y, alt], axis=-1)
    out[bad] = np.inf
    out[np.isnan(p).any(axis=-1)] = np.nan
    return out


# ------------------------------------------------------------------ 50-digit truth

def _ell():
    f = mp.mpf(1) / mp.mpf("298.257223563")
    e2 = f * (2 - f)
    return mp.mpf(6378137), e2, mp.sqrt(e2)


def meridian_arc_quad(lat):
    """meridian arc from the equator to latitude lat (degrees, a float taken exactly), by quadrature of the radius of
    curvature of the meridian"""
    with mp.workdps(DPS):
        a, e2, _ = _ell()
        phi = mp.mpf(lat) * mp.pi / 180
        return mp.quad(lambda t: a * (1 - e2) / (1 - e2 * mp.sin(t) ** 2) ** mp.mpf(1.5), [0, phi])


def _arc(phi):
    a, e2, _ = _ell()
    s, c = mp.sin(phi), mp.cos(phi)
    return a * (mp.ellipe(phi, e2) - e2 * s * c / mp.sqrt(1 - e2 * s * s))


def _chi(phi):
    """conformal latitude, exact"""
    _, _, e = _ell()
    return mp.atan(mp.sinh(mp.asinh(mp.tan(phi)) - e * mp.atanh(e * mp.sin(phi))))


@functools.lru_cache(maxsize=None)
def _series():
    """(A, alpha_1..alpha_8): the rectifying radius and Krueger's coefficients, at DPS digits"""
    with mp.workdps(DPS + 10):
        half_pi = mp.pi / 2
        quad_arc = _arc(half_pi)
        A = quad_arc / half_pi

        def g(chi):                     # mu - chi on [-pi/2, pi/2]
            if chi == 0 or abs(chi) == half_pi:
                return mp.mpf(0)
            phi = mp.findroot(lambda p: _chi(p) - chi, chi)
            return _arc(phi) / A - chi

        N = 64
        samples = []
        for k in range(N):
            chi = mp.pi * k / N
            samples.append((chi, g(chi) if chi <= half_pi else -g(mp.pi - chi)))
        alpha = [2 * mp.fsum(v * mp.sin(2 * j * c) for c, v in samples) / N for j in range(1, 9)]
        return A, alpha


def truth(lon, lat, zone, south):
    """(x, y) in metres, as mpf, of the point (lon, lat) in degrees (floats, taken exactly)"""
    A, alpha = _series()
    with mp.workdps(DPS):
        dl = mp.mpf(lon) - mp.mpf(lon0_of(zone))
        dl = dl - 360 * mp.floor((dl + 180) / 360)
        lam = dl * mp.pi / 180
        phi = mp.mpf(lat) * mp.pi / 180
        chi = _chi(phi) if abs(lat) < 90 else phi
        sc, cc = mp.sin(chi), mp.cos(chi)
        xip = mp.atan2(sc, cc * mp.cos(lam))
        etap = mp.asinh(mp.sin(lam) * cc / mp.hypot(sc, cc * mp.cos(lam)))
        zp = mp.mpc(xip, etap)
        z = zp + mp.fsum(alpha[j - 1] * mp.sin(2 * j * zp) for j in range(1, 9))
        x = FE + K0 * A * z.imag
        y = (FN_SOUTH if south else 0) + K0 * A * z.real
        return x, y


def truth_array(lonlat, zone, south):
    """(n, 2) degrees -> (n, 2) float64 metres"""
    return np.array([[float(v) for v in truth(float(lo), float(la), zone, south)] for lo, la in np.asarray(lonlat)])
