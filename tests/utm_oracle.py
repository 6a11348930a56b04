"""Test helper: the WGS84 UTM transverse Mercator restated in mpmath (40 digits) as Krüger's series of order 6 in n
(Karney 2011, "Transverse Mercator with an accuracy of a few nanometers", eqs 7-9, 11, 15, 35, 36), the oracle of
amb_import_raster_lonlat's positions (include/aerial_mapper_b200.h).  The coefficients are exact fractions; the
conformal-to-geodetic latitude step is solved to full precision.  test_lonlat_import_cpu.py pins the oracle to the exact
projection (meridian arc, conformality, round trip)."""
from fractions import Fraction as F

import mpmath as mp

mp.mp.dps = 40

A_WGS84 = mp.mpf(6378137)
F_WGS84 = 1 / mp.mpf("298.257223563")
K0 = mp.mpf("0.9996")
FE = mp.mpf(500000)
N3 = F_WGS84 / (2 - F_WGS84)
E2 = F_WGS84 * (2 - F_WGS84)
E = mp.sqrt(E2)
RECT = A_WGS84 / (1 + N3) * (1 + N3 ** 2 / 4 + N3 ** 4 / 64 + N3 ** 6 / 256)   # rectifying radius A

# Karney 2011, eq 35 (alpha, forward) and eq 36 (beta, inverse): coefficient of n^1 .. n^6
ALPHA = [[F(1, 2), F(-2, 3), F(5, 16), F(41, 180), F(-127, 288), F(7891, 37800)],
         [0, F(13, 48), F(-3, 5), F(557, 1440), F(281, 630), F(-1983433, 1935360)],
         [0, 0, F(61, 240), F(-103, 140), F(15061, 26880), F(167603, 181440)],
         [0, 0, 0, F(49561, 161280), F(-179, 168), F(6601661, 7257600)],
         [0, 0, 0, 0, F(34729, 80640), F(-3418889, 1995840)],
         [0, 0, 0, 0, 0, F(212378941, 319334400)]]
BETA = [[F(1, 2), F(-2, 3), F(37, 96), F(-1, 360), F(-81, 512), F(96199, 604800)],
        [0, F(1, 48), F(1, 15), F(-437, 1440), F(46, 105), F(-1118711, 3870720)],
        [0, 0, F(17, 480), F(-37, 840), F(-209, 4480), F(5569, 90720)],
        [0, 0, 0, F(4397, 161280), F(-11, 504), F(-830251, 7257600)],
        [0, 0, 0, 0, F(4583, 161280), F(-108847, 3991680)],
        [0, 0, 0, 0, 0, F(20648693, 638668800)]]


def _series(rows):
    return [sum(mp.mpf(c.numerator) / c.denominator * N3 ** (m + 1) for m, c in enumerate(r)) for r in rows]


ALPHA_N = _series(ALPHA)
BETA_N = _series(BETA)


def zone_of(epsg):
    """(central meridian in degrees, false northing) of a WGS84 UTM EPSG code."""
    south = 32701 <= epsg <= 32760
    assert south or 32601 <= epsg <= 32660, epsg
    return 6 * (epsg % 100) - 183, (mp.mpf(10000000) if south else mp.mpf(0))


def taup_of_tau(tau):
    """tan(conformal latitude) of tan(geodetic latitude)."""
    tau1 = mp.sqrt(1 + tau * tau)
    sig = mp.sinh(E * mp.atanh(E * tau / tau1))
    return mp.sqrt(1 + sig * sig) * tau - sig * tau1


def tau_of_taup(taup):
    tau = taup / (1 - E2)
    for _ in range(60):
        d = (taup - taup_of_tau(tau)) * (1 + (1 - E2) * tau * tau) / \
            ((1 - E2) * mp.sqrt(1 + tau * tau) * mp.sqrt(1 + taup_of_tau(tau) ** 2))
        tau += d
        if abs(d) < mp.mpf(10) ** (-mp.mp.dps + 3) * (1 + abs(tau)):
            break
    return tau


def inverse(easting, northing, epsg):
    """(lon, lat) in degrees (mpf) of a UTM position, by the order-6 series."""
    lon0, fn = zone_of(epsg)
    xi = (mp.mpf(northing) - fn) / (K0 * RECT)
    eta = (mp.mpf(easting) - FE) / (K0 * RECT)
    xip = xi - sum(b * mp.sin(2 * k * xi) * mp.cosh(2 * k * eta) for k, b in enumerate(BETA_N, 1))
    etap = eta - sum(b * mp.cos(2 * k * xi) * mp.sinh(2 * k * eta) for k, b in enumerate(BETA_N, 1))
    taup = mp.sin(xip) / mp.sqrt(mp.sinh(etap) ** 2 + mp.cos(xip) ** 2)
    lat = mp.degrees(mp.atan(tau_of_taup(taup)))
    lon = lon0 + mp.degrees(mp.atan2(mp.sinh(etap), mp.cos(xip)))
    return lon, lat


def forward(lon, lat, epsg):
    """(easting, northing) of (lon, lat) in degrees, by the order-6 alpha series."""
    lon0, fn = zone_of(epsg)
    phi, lam = mp.radians(mp.mpf(lat)), mp.radians(mp.mpf(lon) - lon0)
    taup = taup_of_tau(mp.tan(phi))
    xip = mp.atan2(taup, mp.cos(lam))
    etap = mp.asinh(mp.sin(lam) / mp.sqrt(taup * taup + mp.cos(lam) ** 2))
    xi = xip + sum(a * mp.sin(2 * k * xip) * mp.cosh(2 * k * etap) for k, a in enumerate(ALPHA_N, 1))
    eta = etap + sum(a * mp.cos(2 * k * xip) * mp.sinh(2 * k * etap) for k, a in enumerate(ALPHA_N, 1))
    return FE + K0 * RECT * eta, fn + K0 * RECT * xi


def meridian_arc(lat):
    """The exact meridian arc from the equator to latitude `lat` (degrees), by quadrature."""
    phi = mp.radians(mp.mpf(lat))
    return mp.quad(lambda p: A_WGS84 * (1 - E2) / (1 - E2 * mp.sin(p) ** 2) ** mp.mpf(1.5), [0, phi])


def isometric_latitude(lat):
    """psi = asinh(tan(chi)) of a geodetic latitude in degrees."""
    return mp.asinh(taup_of_tau(mp.tan(mp.radians(mp.mpf(lat)))))
