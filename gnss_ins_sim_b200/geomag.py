"""World Magnetic Model on the host: the reference's geomag.GeoMag (gnss_ins_sim/geoparams/geomag.py:23-283)
restated, and the geomagnetic field path_gen uses (pathgen.py:164-171).

The synthesis keeps the reference's operation order, its decimal-year rule (year + days since 1 January
/ 365.0) and its branch at the geographic poles, so that bx, by, bz are bit-identical to it.  It runs
once per trajectory, at the initial position: plain Python is enough.

No coefficient file ships with this package.  `field_ned` takes the path of a NOAA `.COF` file, or
uses the `geoparams/WMM.COF` of an installed gnss_ins_sim package (located, not imported).
"""
import importlib.util
import math
import os
from datetime import date

MAXORD = 12


def read_cof(path):
    """NOAA .COF file -> (epoch, rows): rows are (n, m, gnm, hnm, dgnm, dhnm) tuples in file order
    (geomag.py:255-271: a 3-field line is the header, a 6-field line a coefficient, others are ignored)."""
    epoch, rows = None, []
    with open(path) as f:
        for line in f:
            v = line.strip().split()
            if len(v) == 3:
                epoch = float(v[0])
            elif len(v) == 6:
                rows.append((int(float(v[0])), int(float(v[1])), float(v[2]), float(v[3]),
                             float(v[4]), float(v[5])))
    if epoch is None or not rows:
        raise ValueError('%s is not a WMM coefficient file (.COF)' % path)
    return epoch, rows


def decimal_year(day):
    """geomag.py:24: year + whole days since 1 January / 365.0 (also in leap years)."""
    return day.year + ((day - date(day.year, 1, 1)).days / 365.0)


class GeoMag:
    """Degree-12 spherical-harmonic synthesis from Schmidt-normalised Gauss coefficients."""

    def __init__(self, epoch, rows):
        z13, z14 = lambda: [0.0] * 13, lambda: [0.0] * 14     # noqa: E731
        self.epoch = float(epoch)
        self.c = [z14() for _ in range(14)]
        self.cd = [z14() for _ in range(14)]
        for n, m, gnm, hnm, dgnm, dhnm in rows:
            if m <= n:
                self.c[m][n] = gnm
                self.cd[m][n] = dgnm
                if m != 0:
                    self.c[n][m - 1] = hnm
                    self.cd[n][m - 1] = dhnm
        # Schmidt-normalised -> unnormalised (geomag.py:258-283)
        self.snorm = [z13() for _ in range(13)]
        self.snorm[0][0] = 1.0
        self.k = [z13() for _ in range(13)]
        self.fn = [0.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0, 10.0, 11.0, 12.0, 13.0]
        self.fm = [0.0, 1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0, 8.0, 9.0, 10.0, 11.0, 12.0]
        for n in range(1, MAXORD + 1):
            self.snorm[0][n] = self.snorm[0][n - 1] * (2.0 * n - 1) / n
            j = 2.0
            for m in range(0, n + 1):
                self.k[m][n] = (((n - 1) * (n - 1)) - (m * m)) / ((2.0 * n - 1) * (2.0 * n - 3.0))
                if m > 0:
                    flnmj = ((n - m + 1.0) * j) / (n + m)
                    self.snorm[m][n] = self.snorm[m - 1][n] * math.sqrt(flnmj)
                    j = 1.0
                    self.c[n][m - 1] = self.snorm[m][n] * self.c[n][m - 1]
                    self.cd[n][m - 1] = self.snorm[m][n] * self.cd[n][m - 1]
                self.c[m][n] = self.snorm[m][n] * self.c[m][n]
                self.cd[m][n] = self.snorm[m][n] * self.cd[m][n]

    @classmethod
    def from_file(cls, path):
        return cls(*read_cof(path))

    def field(self, dlat, dlon, h, day):
        """(bx, by, bz) [nT], north / east / down, at geodetic latitude and longitude [deg], height h [m]
        above the ellipsoid and a datetime.date (geomag.py:23-160)."""
        a, b, re = 6378.137, 6356.7523142, 6371.2
        a2, b2 = a * a, b * b
        c2 = a2 - b2
        a4, b4 = a2 * a2, b2 * b2
        c4 = a4 - b4
        t = decimal_year(day)
        alt = h / 1000.0
        dt = t - self.epoch
        rlat, rlon = math.radians(dlat), math.radians(dlon)
        srlon, srlat = math.sin(rlon), math.sin(rlat)
        crlon, crlat = math.cos(rlon), math.cos(rlat)
        srlat2, crlat2 = srlat * srlat, crlat * crlat
        sp = [0.0] * 14
        cp = [0.0] * 14
        cp[0] = 1.0
        sp[1], cp[1] = srlon, crlon
        pp = [0.0] * 13
        pp[0] = 1.0
        p = [[0.0] * 14 for _ in range(14)]
        p[0][0] = 1.0
        dp = [[0.0] * 13 for _ in range(14)]
        tc = [[0.0] * 13 for _ in range(14)]
        # geodetic -> spherical coordinates
        q = math.sqrt(a2 - c2 * srlat2)
        q1 = alt * q
        q2 = ((q1 + a2) / (q1 + b2)) * ((q1 + a2) / (q1 + b2))
        ct = srlat / math.sqrt(q2 * crlat2 + srlat2)
        st = math.sqrt(1.0 - (ct * ct))
        r2 = (alt * alt) + 2.0 * q1 + (a4 - c4 * srlat2) / (q * q)
        r = math.sqrt(r2)
        d = math.sqrt(a2 * crlat2 + b2 * srlat2)
        ca = (alt + d) / r
        sa = c2 * crlat * srlat / (r * d)
        for m in range(2, MAXORD + 1):
            sp[m] = sp[1] * cp[m - 1] + cp[1] * sp[m - 1]
            cp[m] = cp[1] * cp[m - 1] - sp[1] * sp[m - 1]
        aor = re / r
        ar = aor * aor
        br = bt = bp = bpp = 0.0
        k, c, cd, fm, fn = self.k, self.c, self.cd, self.fm, self.fn
        for n in range(1, MAXORD + 1):
            ar = ar * aor
            for m in range(0, n + 1):
                # unnormalised associated Legendre functions and derivatives by recursion
                if n == m:
                    p[m][n] = st * p[m - 1][n - 1]
                    dp[m][n] = st * dp[m - 1][n - 1] + ct * p[m - 1][n - 1]
                elif n == 1 and m == 0:
                    p[m][n] = ct * p[m][n - 1]
                    dp[m][n] = ct * dp[m][n - 1] - st * p[m][n - 1]
                elif n > 1 and n != m:
                    if m > n - 2:
                        p[m][n - 2] = 0
                        dp[m][n - 2] = 0.0
                    p[m][n] = ct * p[m][n - 1] - k[m][n] * p[m][n - 2]
                    dp[m][n] = ct * dp[m][n - 1] - st * p[m][n - 1] - k[m][n] * dp[m][n - 2]
                # time-adjusted Gauss coefficients
                tc[m][n] = c[m][n] + dt * cd[m][n]
                if m != 0:
                    tc[n][m - 1] = c[n][m - 1] + dt * cd[n][m - 1]
                # accumulate the spherical-harmonic expansions
                par = ar * p[m][n]
                if m == 0:
                    temp1 = tc[m][n] * cp[m]
                    temp2 = tc[m][n] * sp[m]
                else:
                    temp1 = tc[m][n] * cp[m] + tc[n][m - 1] * sp[m]
                    temp2 = tc[m][n] * sp[m] - tc[n][m - 1] * cp[m]
                bt = bt - ar * temp1 * dp[m][n]
                bp = bp + (fm[m] * temp2 * par)
                br = br + (fn[n] * temp1 * par)
                # geographic poles: the east component from the m = 1 terms
                if st == 0.0 and m == 1:
                    if n == 1:
                        pp[n] = pp[n - 1]
                    else:
                        pp[n] = ct * pp[n - 1] - k[m][n] * pp[n - 2]
                    parp = ar * pp[n]
                    bpp = bpp + (fm[m] * temp2 * parp)
        if st == 0.0:
            bp = bpp
        else:
            bp = bp / st
        # spherical -> geodetic components
        bx = -bt * ca - br * sa
        by = bp
        bz = bt * sa - br * ca
        return bx, by, bz


class CoefficientsMissing(ValueError, NotImplementedError):
    """No WMM coefficient file was given and none is installed.  A ValueError that says how to pass one; also a
    NotImplementedError, which is what path_gen(..., magnet=True) raised before it generated magnetometer output,
    so callers that caught that keep working where no coefficients are available."""


def installed_cof():
    """geoparams/WMM.COF of an installed gnss_ins_sim package (found without importing it), or None."""
    spec = importlib.util.find_spec('gnss_ins_sim')
    if spec is None or not spec.submodule_search_locations:
        return None
    for d in spec.submodule_search_locations:
        path = os.path.join(d, 'geoparams', 'WMM.COF')
        if os.path.isfile(path):
            return path
    return None


def field_ned(ini, ref_frame, wmm_file=None, wmm_date=None):
    """The geomagnetic field path_gen rotates into the body frame (pathgen.py:164-171): WMM at the initial
    position ini[0:3] (lat, lon [rad], h [m]) on wmm_date (default: today), nT -> uT; in ref_frame 1 the
    horizontal part is put on the x axis, [sqrt(bx^2 + by^2), 0, bz]."""
    if wmm_file is None:
        wmm_file = installed_cof()
        if wmm_file is None:
            raise CoefficientsMissing('a 9-axis IMU needs World Magnetic Model coefficients: pass wmm_file=<path of a '
                                      'NOAA .COF file> (no installed gnss_ins_sim package provides geoparams/WMM.COF)')
    if not os.path.isfile(wmm_file):
        raise ValueError('WMM coefficient file %r does not exist' % (wmm_file,))
    d2r = math.pi / 180
    gm = GeoMag.from_file(wmm_file)
    bx, by, bz = gm.field(ini[0] / d2r, ini[1] / d2r, ini[2], date.today() if wmm_date is None else wmm_date)
    g = [bx / 1000.0, by / 1000.0, bz / 1000.0]
    if ref_frame == 1:
        g[0] = math.sqrt(g[0] * g[0] + g[1] * g[1])
        g[1] = 0.0
    return g
