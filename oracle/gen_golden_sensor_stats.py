"""Generate tests/golden/sensor_stats_90deg.npz by running the UNMODIFIED reference (the helpers and the
reference import of gen_golden.py, the pinned WMM date of gen_golden_mag.py).  Test infrastructure only.

    python oracle/gen_golden_sensor_stats.py

Frozen, for the 90 deg turn at 100 Hz with R = 8 runs of a 9-axis IMU with GPS at 10 Hz, the b2ins normals
injected into np.random.randn in loop A's call order (acc_gen, gyro_gen, gps_gen, mag_gen per run;
ins_sim.py:490-506), in five cases: both reference frames, random vibration (ref_frame 1), sinusoidal
vibration (ref_frame 0) and white bias drift (tau = inf, ref_frame 0):
  * get_error_stats(name, start, use_output_units=ou) of the reference for gyro, accel, mag and gps, starts
    -1, 0, 2.5 s and past the end (gps: -1 and 0 only -- the reference indexes GPS rows with the IMU time
    index, ins_data_manager.py:774-783), ou False and True, and the units strings;
  * the truth and the error models, so that the statistics can be recomputed without the reference.
For both frames without vibration, the att_euler / pos / vel statistics of the two plugins of
sensor_stats_plugins (starts -1, 0 and 2.5 s; pos also with extra_opt 'ned' and 'ecef' in ref_frame 0) and
the error-statistics block of results().  The reference caches the error array of a data name at the first
call (ins_data_manager.py:427-431): every extra_opt gets a fresh Sim.
"""
import copy
import os

import numpy as np

from gen_golden import MOTION, OUT, RandnQueue, read_ini, ins_sim, imu_model
from gen_golden_mag import DATE
from gnss_ins_sim.geoparams import geomag
import oracle_np as onp
import mag_np
import sensor_stats_np as ssn
import sensor_stats_plugins as plugins

FS, FS_GPS, R, SEED = 100.0, 10.0, 8, 8086
CSV = os.path.join(MOTION, 'motion_def-90deg_turn.csv')
GPS_ERR = {'stdp': np.array([5.0, 5.0, 7.0]), 'stdv': np.array([0.05, 0.05, 0.05])}
ACCURACY = {
    'gyro_b': np.array([1.0, -2.0, 0.5]), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
    'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
    'accel_b': np.array([2.0e-3, 1.0e-3, -3.0e-3]), 'accel_vrw': np.array([0.03, 0.03, 0.03]),
    'accel_b_stability': np.array([4.0e-5, 4.0e-5, 4.0e-5]), 'accel_b_corr': np.array([200.0, 200.0, 200.0]),
    'mag_si': np.array([[1.02, 0.03, -0.01], [-0.02, 0.97, 0.05], [0.04, -0.06, 1.01]]),
    'mag_hi': np.array([10.0, -7.5, 3.0]), 'mag_std': np.array([0.2, 0.35, 0.5]),
}
# tag -> (ref_frame, env, white bias drift)
CASES = {
    'rf0': (0, None, False),
    'rf1': (1, None, False),
    'vibrand_rf1': (1, {'acc': '[0.03 0.001 0.01]-random', 'gyro': '[6 5 4]d-random'}, False),
    'vibsin_rf0': (0, {'acc': '[0.03 0.001 0.01]g-3Hz-sinusoidal', 'gyro': '[6 5 4]d-0.5Hz-sinusoidal'}, False),
    'whitedrift_rf0': (0, None, True),
}
STARTS = np.array([-1.0, 0.0, 2.5, 1.0e6])
GPS_STARTS = np.array([-1.0, 0.0])
PLUGIN_STARTS = np.array([-1.0, 0.0, 2.5])


def accuracy(white):
    acc = copy.deepcopy(ACCURACY)
    if white:
        del acc['gyro_b_corr'], acc['accel_b_corr']
    return acc


def run_reference(rf, env, white, algorithm=None):
    """One reference Sim.run(R) on the b2ins stream; the module tables imu_model writes into are restored."""
    saved = copy.deepcopy((imu_model.gyro_low_accuracy, imu_model.accel_low_accuracy))
    try:
        imu = imu_model.IMU(accuracy=accuracy(white), axis=9, gps=True, gps_opt=GPS_ERR)
        sim = ins_sim.Sim([FS, FS_GPS, 0.0], CSV, ref_frame=rf, imu=imu, env=copy.deepcopy(env),
                          algorithm=algorithm)
        n, m = 1000, 100
        run_ids = np.arange(R)
        vib_acc = sim._Sim__parse_env(env['acc']) if env else None
        vib_gyro = sim._Sim__parse_env(env['gyro']) if env else None
        z = onp.noise_normals(n, run_ids, SEED)
        zva, zvg = onp.vib_normals(n, run_ids, SEED)
        zg = onp.gps_normals(m, run_ids, SEED)
        zm = mag_np.mag_normals(n, run_ids, SEED)
        q = RandnQueue()
        for r in range(R):
            for gm, w, vib, zv in ((z['acc_gm'], z['acc_w'], vib_acc, zva), (z['gyr_gm'], z['gyr_w'], vib_gyro, zvg)):
                for i in range(3):
                    if white:
                        q.push(gm[r, :, i])          # drift[i] * randn(n), pathgen.py:591-593
                    else:
                        blk = np.full((n, 3), np.nan)
                        blk[:, i] = gm[r, :, i]
                        q.push(blk)
                if vib is not None and vib['type'] == 'random':
                    for i in range(3):
                        q.push(zv[r, :, i])
                q.push(w[r])
            q.push(zg[r, :, 0:3])
            q.push(zg[r, :, 3:6])
            q.push(zm[r])
        phases = onp.gyro_vib_phase_uniforms(run_ids, SEED)
        pq = [phases[r, c] for r in range(R) for c in range(3)]
        real_randn, real_rand = np.random.randn, np.random.rand
        np.random.randn = q
        np.random.rand = lambda *s: np.array([pq.pop(0)])
        try:
            sim.run(R)
        finally:
            np.random.randn, np.random.rand = real_randn, real_rand
        assert not q.q, 'unused queued normals: %d' % len(q.q)
        # imu.gyro_err / accel_err ARE the module tables restored below: keep copies
        errs = {'gyro': copy.deepcopy(imu.gyro_err), 'accel': copy.deepcopy(imu.accel_err),
                'mag': copy.deepcopy(imu.mag_err)}
        return sim, errs, vib_acc, vib_gyro
    finally:
        imu_model.gyro_low_accuracy.clear()
        imu_model.gyro_low_accuracy.update(saved[0])
        imu_model.accel_low_accuracy.clear()
        imu_model.accel_low_accuracy.update(saved[1])


def put_stats(out, prefix, st):
    for k in ('max', 'avg', 'std'):
        v = st[k]
        out['%s_%s' % (prefix, k)] = np.stack([v[key] for key in sorted(v)]) if isinstance(v, dict) else np.asarray(v)
    out[prefix + '_units'] = np.array(st['units'])


def gen_case(out, tag):
    rf, env, white = CASES[tag]
    sim, errs, vib_acc, vib_gyro = run_reference(rf, env, white)
    d = sim.dmgr
    out[tag + '_ref_frame'] = rf
    for k in ('time', 'ref_gyro', 'ref_accel', 'ref_mag', 'ref_gps', 'gps_time', 'ref_pos', 'ref_vel',
              'ref_att_euler'):
        out['%s_%s' % (tag, k)] = getattr(d, k).data
    for sensor in ('gyro', 'accel'):
        e = errs[sensor]
        for k, v in e.items():
            out['%s_%s_%s' % (tag, sensor, k)] = np.asarray(v, dtype=np.float64)
    for k in ('si', 'hi', 'std'):
        out['%s_mag_%s' % (tag, k)] = np.asarray(errs['mag'][k], dtype=np.float64)
    for v, k in ((vib_acc, 'vib_acc'), (vib_gyro, 'vib_gyro')):
        if v is not None:
            out['%s_%s_type' % (tag, k)] = np.array(v['type'])
            out['%s_%s_amp' % (tag, k)] = np.array([v['x'], v['y'], v['z']])
            out['%s_%s_freq' % (tag, k)] = float(v.get('freq', 0.0))
    # the reference's data themselves agree with the oracle's
    og, oa = ssn.imu(FS, d.ref_gyro.data, d.ref_accel.data, errs['gyro'], errs['accel'], SEED, np.arange(R),
                     vib_acc, vib_gyro)
    assert np.allclose(np.stack([d.gyro.data[r] for r in range(R)]), og, rtol=0, atol=1e-12)
    assert np.allclose(np.stack([d.accel.data[r] for r in range(R)]), oa, rtol=0, atol=1e-12)
    for name in ('gyro', 'accel', 'mag', 'gps'):
        for i, s in enumerate(GPS_STARTS if name == 'gps' else STARTS):
            for ou in (0, 1):
                st = d.get_error_stats(name, err_stats_start=s, angle=False, use_output_units=bool(ou))
                put_stats(out, '%s_%s_s%d_ou%d' % (tag, name, i, ou), st)


def gen_plugins(out, tag):
    rf, env, white = CASES[tag]
    for pname, cls in (('full', plugins.FullRate), ('half', plugins.HalfRate)):
        # results() first, on a fresh Sim: its statistics block
        sim = run_reference(rf, env, white, cls())[0]
        sim.results(err_stats_start=-1 if pname == 'full' else 2.5)
        out['%s_%s_results' % (tag, pname)] = np.array(sim.sum[sim.sum.index('The following are error statistics.'):])
        for opt in ([''] + (['ned', 'ecef'] if rf == 0 else [])):
            sim = run_reference(rf, env, white, cls())[0]
            for name in (('att_euler', 'pos', 'vel') if opt == '' else ('pos',)):
                for i, s in enumerate(PLUGIN_STARTS):
                    for ou in (0, 1):
                        st = sim.dmgr.get_error_stats(name, err_stats_start=s, angle=(name == 'att_euler'),
                                                      use_output_units=bool(ou), extra_opt=opt)
                        put_stats(out, '%s_%s_%s%s_s%d_ou%d' % (tag, pname, name, opt and '_' + opt, i, ou), st)


def main():
    geomag.GeoMag.GeoMag.__defaults__ = (0, DATE)
    out = {'fs': FS, 'fs_gps': FS_GPS, 'seed': SEED, 'run_ids': np.arange(R), 'ini': read_ini(CSV),
           'stdp': GPS_ERR['stdp'], 'stdv': GPS_ERR['stdv'], 'date': np.array([DATE.year, DATE.month, DATE.day]),
           'starts': STARTS, 'gps_starts': GPS_STARTS, 'plugin_starts': PLUGIN_STARTS,
           'cases': np.array(sorted(CASES))}
    for tag in CASES:
        gen_case(out, tag)
    for tag in ('rf0', 'rf1'):
        gen_plugins(out, tag)
    np.savez_compressed(os.path.join(OUT, 'sensor_stats_90deg.npz'), **out)


if __name__ == '__main__':
    main()
