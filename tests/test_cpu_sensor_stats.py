"""Error statistics of sensor data and of reference-style plugins, on the host: the NumPy oracle
(sensor_stats_np) and Sim's logged-data path against the reference's get_error_stats / results() output
frozen in tests/golden/sensor_stats_90deg.npz (oracle/gen_golden_sensor_stats.py)."""
import numpy as np
import pytest

import sensor_stats_np as ssn
import sensor_stats_plugins as plugins
from conftest import load_golden, assert_close

G = load_golden('sensor_stats_90deg.npz')
R = len(G['run_ids'])
SEED = int(G['seed'])
UNITS = {'gyro': (['rad/s'] * 3, ['deg/s'] * 3), 'accel': (['m/s^2'] * 3, ['m/s^2'] * 3),
         'mag': (['uT'] * 3, ['uT'] * 3)}


def gps_units(rf):
    if rf == 1:
        return ['m', 'm', 'm', 'm/s', 'm/s', 'm/s'], ['m', 'm', 'm', 'm/s', 'm/s', 'm/s']
    return ['rad', 'rad', 'm', 'm/s', 'm/s', 'm/s'], ['deg', 'deg', 'm', 'm/s', 'm/s', 'm/s']


def err_model(tag, sensor):
    white = 'arw' if sensor == 'gyro' else 'vrw'
    return {k: G['%s_%s_%s' % (tag, sensor, k)] for k in ('b', 'b_drift', 'b_corr', white)}


def vib(tag, k):
    if '%s_%s_type' % (tag, k) not in G:
        return None
    a = G['%s_%s_amp' % (tag, k)]
    return {'type': str(G['%s_%s_type' % (tag, k)]), 'x': a[0], 'y': a[1], 'z': a[2],
            'freq': float(G['%s_%s_freq' % (tag, k)])}


def sensor_data(tag):
    """{name: (x [R, m, C], ref [m, C], row times)} of one golden case, made by the oracle."""
    g = lambda k: G['%s_%s' % (tag, k)]                              # noqa: E731
    rf = int(g('ref_frame'))
    gyro, accel = ssn.imu(float(G['fs']), g('ref_gyro'), g('ref_accel'), err_model(tag, 'gyro'),
                          err_model(tag, 'accel'), SEED, G['run_ids'], vib(tag, 'vib_acc'), vib(tag, 'vib_gyro'))
    mag = ssn.mag(g('ref_mag'), {k: g('mag_' + k) for k in ('si', 'hi', 'std')}, SEED, G['run_ids'])
    gps = ssn.gps(g('ref_gps'), {'stdp': G['stdp'], 'stdv': G['stdv']}, rf, SEED, G['run_ids'])
    t = g('time')
    return {'gyro': (gyro, g('ref_gyro'), t), 'accel': (accel, g('ref_accel'), t),
            'mag': (mag, g('ref_mag'), t), 'gps': (gps, g('ref_gps'), g('gps_time'))}


def starts(name):
    return G['gps_starts'] if name == 'gps' else G['starts']


@pytest.mark.parametrize('tag', [str(c) for c in G['cases']])
def test_oracle_reproduces_reference(tag):
    rf = int(G[tag + '_ref_frame'])
    for name, (x, ref, t) in sensor_data(tag).items():
        units, out_units = gps_units(rf) if name == 'gps' else UNITS[name]
        for i, s in enumerate(starts(name)):
            end, proc = ssn.stats(x, ref, ssn.first_at(t, s))
            st = end if s == -1 else proc
            for ou in (0, 1):
                key = '%s_%s_s%d_ou%d' % (tag, name, i, ou)
                scale = ssn.output_scale(units, out_units) if ou else 1.0
                for k in ('max', 'avg', 'std'):
                    assert_close(st[k] * scale, G['%s_%s' % (key, k)], 1e-12, 1e-9, key + ' ' + k)
                assert str(G[key + '_units']) == str(out_units)


def write_dir(path, tag):
    """A logged-data directory in the reference's file format with the oracle's sensor data of one case."""
    from gnss_ins_sim_b200 import logged
    rf = int(G[tag + '_ref_frame'])
    g = lambda k: G['%s_%s' % (tag, k)]                              # noqa: E731
    data = sensor_data(tag)
    for k in ('time', 'ref_pos', 'ref_vel', 'ref_att_euler', 'ref_gyro', 'ref_accel', 'ref_mag', 'ref_gps',
              'gps_time'):
        logged.write_data(str(path), k, g(k), rf)
    for name in ('gyro', 'accel', 'mag', 'gps'):
        logged.write_data(str(path), name, {r: data[name][0][r] for r in range(R)}, rf)
    return str(path)


def logged_sim(path, tag, algorithm=None):
    from gnss_ins_sim_b200.sim import Sim
    sim = Sim([float(G['fs']), float(G['fs_gps']), 0.0], path, ref_frame=int(G[tag + '_ref_frame']),
              algorithm=algorithm)
    sim.run(R)
    return sim


@pytest.mark.parametrize('tag', ['rf0', 'rf1'])
def test_logged_sensor_stats_match_reference(tag, tmp_path):
    sim = logged_sim(write_dir(tmp_path, tag), tag)
    for name in ('gyro', 'accel', 'mag', 'gps'):
        for i, s in enumerate(starts(name)):
            for ou in (0, 1):
                st = sim.get_error_stats(name, err_stats_start=s, use_output_units=bool(ou))
                key = '%s_%s_s%d_ou%d' % (tag, name, i, ou)
                for k in ('max', 'avg', 'std'):
                    got = st[k] if s == -1 else np.stack([st[k][r] for r in range(R)])
                    assert_close(got, G['%s_%s' % (key, k)], 1e-9, 1e-6, key + ' ' + k)
                if ou:
                    assert st['units'] == str(G[key + '_units'])


@pytest.mark.parametrize('tag', ['rf0', 'rf1'])
@pytest.mark.parametrize('pname', ['full', 'half'])
def test_logged_plugin_stats_match_reference(tag, pname, tmp_path):
    rf = int(G[tag + '_ref_frame'])
    cls = plugins.FullRate if pname == 'full' else plugins.HalfRate
    sim = logged_sim(write_dir(tmp_path, tag), tag, cls())
    for opt in [''] + (['ned', 'ecef'] if rf == 0 else []):
        for name in (('att_euler', 'pos', 'vel') if opt == '' else ('pos',)):
            for i, s in enumerate(G['plugin_starts']):
                for ou in (0, 1):
                    st = sim.get_error_stats(name, err_stats_start=s, angle=(name == 'att_euler'),
                                             use_output_units=bool(ou), extra_opt=opt)
                    key = '%s_%s_%s%s_s%d_ou%d' % (tag, pname, name, opt and '_' + opt, i, ou)
                    for k in ('max', 'avg', 'std'):
                        got = st[k] if s == -1 else np.stack([st[k]['algo0_%d' % r] for r in range(R)])
                        # NED / ECEF metres: lla2ecef of ~6.4e6 m rounds at 1e-9 m
                        assert_close(got, G['%s_%s' % (key, k)], 1e-9, 1.0 if opt else 1e-3, key + ' ' + k)
                    if ou:
                        assert st['units'] == str(G[key + '_units'])


def _numbers(block):
    return np.array([float(v) for v in block.replace('[', ' ').replace(']', ' ').split()])


@pytest.mark.parametrize('pname,start', [('full', -1), ('half', 2.5)])
def test_results_prints_plugin_block(pname, start, tmp_path, capsys):
    cls = plugins.FullRate if pname == 'full' else plugins.HalfRate
    sim = logged_sim(write_dir(tmp_path, 'rf0'), 'rf0', cls())
    sim.results(err_stats_start=start)
    text = capsys.readouterr().out
    want = str(G['rf0_%s_results' % pname])
    got = text[text.index('The following are error statistics.'):].rstrip('\n')
    # the same lines: headers verbatim, numbers to printing precision
    wl, gl = want.rstrip('\n').split('\n'), got.split('\n')
    assert len(wl) == len(gl)
    for a, b in zip(wl, gl):
        if 'error:' in a:
            assert a.split(':')[0] == b.split(':')[0]
            assert_close(_numbers(b.split(':', 1)[1]), _numbers(a.split(':', 1)[1]), 1e-6, 1e-12, a)
        else:
            assert a == b


def test_odo_has_no_error_statistics():
    from gnss_ins_sim_b200.sim import Sim
    sim = Sim(100.0, {'ref_pos': np.zeros((4, 3)), 'ref_vel': np.zeros((4, 3)), 'ref_att': np.zeros((4, 3)),
                      'ref_accel': np.zeros((4, 3)), 'ref_gyro': np.zeros((4, 3))})
    with pytest.raises(ValueError, match='odo has no error statistics'):
        sim.get_error_stats('odo', 0)
    with pytest.raises(ValueError, match='error statistics exist for'):
        sim.get_error_stats('wb', 0)
