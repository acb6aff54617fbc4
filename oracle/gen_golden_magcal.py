"""Generate tests/golden/magcal.npz from the UNMODIFIED reference: its Sim with
demo_algorithms.mag_calibrate.MagCal, and its libmagcal.so called directly.  Test infrastructure only.

    python oracle/gen_golden_magcal.py

Frozen:
  * Sim: tests/golden/motion_def-mag_cal.csv (three 720-degree rotations about body x, y and z at 45 deg/s,
    3 s pauses) at 100 Hz, ref_frame 1, IMU(axis=9) with a dict accuracy (a non-identity mag_si, a non-zero
    mag_hi, a different mag_std per axis), R runs with the b2ins normals injected into np.random.randn in loop
    A's call order (as gen_golden_mag.py), builtins.input answering the six segment indices, matplotlib's
    plot / grid / show as no-ops (a stand-in module where matplotlib is not installed): soft_iron, hard_iron and
    every MAG_CAL_STRIDE-th row of mag_cal per run, every REF_MAG_STRIDE-th row of ref_mag.  The samples are not
    stored: tests rebuild ref_mag with the path generator and mag from its normals (mag_np.mag_gen, asserted
    here to 1e-12 uT of the reference's).  The two off-axis true gyro channels are asserted zero inside each
    segment.
  * libmagcal.so MagCalibrate on synthetic cases (each segment on its own copy of the rows): single-axis
    rotations of unequal lengths (3 to 20 000 rows), noise 0 to 1 uT, hard iron up to 100 x |b|, overlapping
    segments, and degenerate input (noise-free samples from a plane through the origin, a NaN sample, a constant
    segment).  Stored: each case's recipe for magcal_np.synthetic_mag (inputs rounded to 2^-24 uT, so they are
    rebuilt bit for bit) and the reference's soft_iron and hard_iron.
"""
import builtins
import ctypes
import os
import sys
import types
from datetime import date

import numpy as np

try:
    import matplotlib
    matplotlib.use('Agg')
except ImportError:     # the plugin only plots; a stand-in keeps its import and its calls working
    _mpl = types.ModuleType('matplotlib')
    _mpl.pyplot = types.ModuleType('matplotlib.pyplot')
    _mpl.mlab = types.ModuleType('matplotlib.mlab')
    for _f in ('plot', 'grid', 'show'):
        setattr(_mpl.pyplot, _f, lambda *a, **k: None)
    sys.modules.update({'matplotlib': _mpl, 'matplotlib.pyplot': _mpl.pyplot, 'matplotlib.mlab': _mpl.mlab})

from gen_golden import OUT, REF, RandnQueue, inject_stream, read_ini, ins_sim, imu_model  # noqa: E402
from gnss_ins_sim.geoparams import geomag  # noqa: E402
from demo_algorithms import mag_calibrate  # noqa: E402
import mag_np  # noqa: E402
import magcal_np as mc  # noqa: E402

FS = 100.0
DATE = date(2017, 7, 2)
MOTION = os.path.join(OUT, 'motion_def-mag_cal.csv')
SEGMENTS = ((343, 1900), (2243, 3800), (4143, 5700))
ACCURACY = {
    'gyro_b': np.zeros(3), 'gyro_arw': np.full(3, 0.25), 'gyro_b_stability': np.full(3, 3.5),
    'gyro_b_corr': np.full(3, 100.0), 'accel_b': np.zeros(3), 'accel_vrw': np.full(3, 0.03),
    'accel_b_stability': np.full(3, 4e-5), 'accel_b_corr': np.full(3, 200.0),
    'mag_si': np.array([[1.05, 0.04, -0.02], [-0.03, 0.96, 0.06], [0.05, -0.07, 1.02]]),
    'mag_hi': np.array([12.0, -8.5, 4.0]),
    'mag_std': np.array([0.2, 0.35, 0.5]),
}
REF_MAG_STRIDE = 200      # rows kept of ref_mag: tests rebuild it (path generator + WMM) and check these
MAG_CAL_STRIDE = 8        # rows kept of mag_cal: tests rebuild mag from its normals (mag_np) and check these
LIB = os.path.join(REF, 'demo_algorithms', 'mag_calibrate_lib', 'libmagcal.so')


def gen_sim(R=3, seed=777):
    geomag.GeoMag.GeoMag.__defaults__ = (0, DATE)
    ini = read_ini(MOTION)
    imu = imu_model.IMU(accuracy=dict(ACCURACY), axis=9, gps=False)
    probe = ins_sim.Sim([FS, 0.0, 0.0], MOTION, ref_frame=1, imu=imu, algorithm=None)
    real = np.random.randn
    np.random.randn = lambda *s: np.zeros(s)
    try:
        probe.run(1)
    finally:
        np.random.randn = real
    d = probe.dmgr
    n = d.time.data.shape[0]
    for a, (lo, hi) in enumerate(SEGMENTS):
        off = [c for c in range(3) if c != a]
        assert np.abs(d.ref_gyro.data[lo:hi][:, off]).max() <= 1e-12, 'segment %d is not a clean rotation' % a
        assert (hi - lo) * np.abs(d.ref_gyro.data[lo:hi, a]).min() / FS >= 2 * np.pi
    zmag = mag_np.mag_normals(n, np.arange(R), seed)
    q = RandnQueue()
    for r in range(R):
        inject_stream(q, n, [r], seed)
        q.push(zmag[r])
    answers = [str(v) for _ in range(R) for pair in SEGMENTS for v in pair]
    real_input = builtins.input
    builtins.input = lambda prompt='': answers.pop(0)
    sim = ins_sim.Sim([FS, 0.0, 0.0], MOTION, ref_frame=1, imu=imu, algorithm=mag_calibrate.MagCal())
    np.random.randn = q
    try:
        sim.run(R)
    finally:
        np.random.randn = real
        builtins.input = real_input
    assert not q.q and not answers
    d = sim.dmgr
    mag = np.stack([d.mag.data[r] for r in range(R)])
    assert np.allclose(mag, mag_np.mag_gen(d.ref_mag.data, imu.mag_err, zmag), rtol=0, atol=1e-12)
    g = geomag.GeoMag('WMM.COF').GeoMag(ini[0] / (np.pi / 180), ini[1] / (np.pi / 180), ini[2])
    return {'fs': FS, 'seed': seed, 'run_ids': np.arange(R), 'date': np.array([DATE.year, DATE.month, DATE.day]),
            'segments': np.array(SEGMENTS), 'mag_si': ACCURACY['mag_si'], 'mag_hi': ACCURACY['mag_hi'],
            'mag_std': ACCURACY['mag_std'], 'geo_mag_n': np.array([g.bx, g.by, g.bz]) / 1000.0,
            'ref_mag_rows': d.ref_mag.data[::REF_MAG_STRIDE],
            'soft_iron': np.stack([d.soft_iron.data['algo0_%d' % r] for r in range(R)]),
            'hard_iron': np.stack([d.hard_iron.data['algo0_%d' % r] for r in range(R)]),
            'mag_cal_rows': np.stack([d.mag_cal.data['algo0_%d' % r][::MAG_CAL_STRIDE] for r in range(R)])}


def ref_calibrate(mag, seg):
    """MagCalibrate of the reference library, each segment on its own copy."""
    lib = ctypes.CDLL(LIB)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)     # noqa: E731
    si, hi = np.zeros((3, 3)), np.zeros((1, 4))
    xs = [np.ascontiguousarray(mag[a:b], dtype=np.float64).copy() for a, b in seg]
    rows = np.array([b - a for a, b in seg], dtype=np.int32)
    lib.MagCalibrate(P(si), P(hi), P(xs[0]), P(xs[1]), P(xs[2]), P(rows))
    return si, hi[0], np.concatenate(xs)


def gen_synthetic():
    """kind 0: ordinary; 1: hard iron 10 to 100 x |b|; 2: degenerate (the reference gives NaN).  Stored: each
    case's recipe (magcal_np.synthetic_mag) and the reference's result on the samples it makes."""
    rng = np.random.default_rng(2026)
    specs = []
    for ns, noise, hm, kind in [((5, 7, 9), 0.5, 10.0, 0), ((3, 3, 3), 0.1, 10.0, 0),
                                ((1000, 2000, 3000), 0.3, 10.0, 0), ((20000, 300, 3), 1.0, 10.0, 0),
                                ((1000, 1000, 1000), 0.0, 10.0, 0), ((800, 900, 700), 0.2, 470.0, 1),
                                ((1000, 1000, 1000), 0.2, 4700.0, 1), ((3000, 2000, 1000), 1.0, 4700.0, 1),
                                ((1200, 1100, 1000), 0.3, 20.0, 0)]:
        b = rng.standard_normal(3)
        b *= 47.0 / np.linalg.norm(b)
        si = np.eye(3) + 0.1 * rng.standard_normal((3, 3))
        hi = rng.standard_normal(3)
        hi *= hm / np.linalg.norm(hi)
        e = np.cumsum([0] + list(ns))
        seg = [(int(e[k]), int(e[k + 1])) for k in range(3)]
        specs.append({'shape': mc.SYN_ROTATIONS, 'ns': np.array(ns), 'noise': noise, 'b': b, 'si': si, 'hi': hi,
                      'run': len(specs), 'seg': np.array(seg), 'kind': kind})
    specs[-1]['seg'] = np.array([(0, 1500), (1000, 2300), (2000, 3300)])     # overlapping segments
    n = 200
    for shape in (mc.SYN_PLANE, mc.SYN_PLANE_NAN, mc.SYN_PLANE_CONST):
        specs.append({'shape': shape, 'ns': np.array([n, n, n]), 'noise': 0.0, 'b': np.zeros(3), 'si': np.eye(3),
                      'hi': np.zeros(3), 'run': len(specs), 'seg': np.array([(0, n), (n, 2 * n), (2 * n, 3 * n)]),
                      'kind': 2})
    out = {}
    for i, spec in enumerate(specs):
        out.update({'syn%d_%s' % (i, k): v for k, v in spec.items()})
        mag, seg, kind = mc.golden_synthetic(out, i)
        si, hi, _ = ref_calibrate(mag, seg)
        if kind == 2:
            assert np.isnan(si).all() and np.isnan(hi).all(), 'degenerate case %d' % i
        else:
            assert np.isfinite(si).all() and np.isfinite(hi).all(), 'case %d' % i
        out.update({'syn%d_soft_iron' % i: si, 'syn%d_hard_iron' % i: hi, 'syn%d_nansum' % i: np.nansum(mag)})
    out['syn_count'] = len(specs)
    return out


if __name__ == '__main__':
    out = gen_sim()
    out.update(gen_synthetic())
    np.savez_compressed(os.path.join(OUT, 'magcal.npz'), **out)
