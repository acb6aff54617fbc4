"""Generate tests/golden/mag_90deg.npz by running the UNMODIFIED reference (the helpers and the reference
import of gen_golden.py).  Test infrastructure only.

    python oracle/gen_golden_mag.py

Frozen:
  * Both reference frames on motion_def-90deg_turn.csv at 100 Hz, IMU(axis=9) with a dict accuracy (a
    non-identity, non-symmetric mag_si, a non-zero mag_hi, a different mag_std per axis), algorithm=None,
    R runs with the b2ins normals injected into np.random.randn in loop A's call order (acc_gen, gyro_gen,
    mag_gen per run; ins_sim.py:490-506): ref_mag, mag per run, and the NED field path_gen used.
  * The reference's date pinned by rebinding GeoMag.GeoMag's default `time` argument (bound to
    date.today() at import, so the reference's ref_mag changes from day to day).
  * geomag.GeoMag(...).GeoMag(lat, lon, h, date) -> (bx, by, bz) nT on a grid that includes the poles
    (the st == 0 branch), 100 km altitude, both hemispheres and two dates.
  * The WMM.COF coefficient table as arrays, so that tests evaluate the restatement without the reference.
"""
import itertools
import os
from datetime import date

import numpy as np

from gen_golden import MOTION, OUT, RandnQueue, inject_stream, read_ini, ins_sim, imu_model
from gnss_ins_sim.geoparams import geomag
import mag_np

FS = 100.0
DATE = date(2017, 7, 2)
ACCURACY = {
    'gyro_b': np.array([1.0, -2.0, 0.5]), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
    'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
    'accel_b': np.array([2.0e-3, 1.0e-3, -3.0e-3]), 'accel_vrw': np.array([0.03, 0.03, 0.03]),
    'accel_b_stability': np.array([4.0e-5, 4.0e-5, 4.0e-5]), 'accel_b_corr': np.array([200.0, 200.0, 200.0]),
    'mag_si': np.array([[1.02, 0.03, -0.01], [-0.02, 0.97, 0.05], [0.04, -0.06, 1.01]]),
    'mag_hi': np.array([10.0, -7.5, 3.0]),
    'mag_std': np.array([0.2, 0.35, 0.5]),
}


def read_table(path):
    epoch, model, modeldate, rows = None, None, None, []
    with open(path) as f:
        for line in f:
            v = line.strip().split()
            if len(v) == 3:
                epoch, model, modeldate = float(v[0]), v[1], v[2]
            elif len(v) == 6:
                rows.append([float(x) for x in v])
    return epoch, model, modeldate, np.array(rows)


def gen_mag(R=4, seed=20240):
    geomag.GeoMag.GeoMag.__defaults__ = (0, DATE)
    csv = os.path.join(MOTION, 'motion_def-90deg_turn.csv')
    ini = read_ini(csv)
    cof = os.path.join(os.path.dirname(geomag.__file__), 'WMM.COF')
    epoch, model, modeldate, rows = read_table(cof)
    out = {'fs': FS, 'seed': seed, 'run_ids': np.arange(R), 'ini': ini,
           'date': np.array([DATE.year, DATE.month, DATE.day]),
           'mag_si': ACCURACY['mag_si'], 'mag_hi': ACCURACY['mag_hi'], 'mag_std': ACCURACY['mag_std'],
           'cof_epoch': epoch, 'cof_model': model, 'cof_modeldate': modeldate, 'cof_rows': rows}
    for rf in (0, 1):
        imu = imu_model.IMU(accuracy=dict(ACCURACY), axis=9, gps=False)
        probe = ins_sim.Sim([FS, 0.0, 0.0], csv, ref_frame=rf, imu=imu, algorithm=None)
        real = np.random.randn
        np.random.randn = lambda *s: np.zeros(s)
        try:
            probe.run(1)
        finally:
            np.random.randn = real
        n = probe.dmgr.time.data.shape[0]
        zmag = mag_np.mag_normals(n, np.arange(R), seed)
        q = RandnQueue()
        for r in range(R):
            inject_stream(q, n, [r], seed)
            q.push(zmag[r])
        sim = ins_sim.Sim([FS, 0.0, 0.0], csv, ref_frame=rf, imu=imu, algorithm=None)
        np.random.randn = q
        try:
            sim.run(R)
        finally:
            np.random.randn = real
        assert not q.q, 'unused queued normals: %d' % len(q.q)
        d = sim.dmgr
        # the field path_gen rotates (pathgen.py:164-171)
        g = geomag.GeoMag('WMM.COF').GeoMag(ini[0] / (np.pi / 180), ini[1] / (np.pi / 180), ini[2])
        gn = np.array([g.bx, g.by, g.bz]) / 1000.0
        if rf == 1:
            gn[0] = np.sqrt(gn[0] * gn[0] + gn[1] * gn[1])
            gn[1] = 0.0
        out['geo_mag_n_rf%d' % rf] = gn
        out['ref_mag_rf%d' % rf] = d.ref_mag.data
        out['mag_rf%d' % rf] = np.stack([d.mag.data[r] for r in range(R)])
        out['ref_att_rf%d' % rf] = d.ref_att_euler.data
        assert np.allclose(out['mag_rf%d' % rf], mag_np.mag_gen(d.ref_mag.data, imu.mag_err, zmag),
                           rtol=0, atol=1e-12)
    # GeoMag on a grid: poles, both hemispheres, 100 km, two dates
    grid = []
    gm = geomag.GeoMag('WMM.COF')
    for lat, lon, h, day in itertools.product((-90.0, -63.5, -12.25, 0.0, 31.2, 89.0, 90.0),
                                              (-179.5, -75.3, 0.0, 121.47),
                                              (0.0, 2500.0, 100000.0),
                                              (date(2015, 1, 1), date(2019, 10, 15))):
        m = gm.GeoMag(lat, lon, h, day)
        grid.append([lat, lon, h, day.year, day.month, day.day, m.bx, m.by, m.bz])
    out['grid'] = np.array(grid)
    np.savez_compressed(os.path.join(OUT, 'mag_90deg.npz'), **out)


if __name__ == '__main__':
    gen_mag()
