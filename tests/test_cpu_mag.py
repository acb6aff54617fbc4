"""Magnetometer output without a GPU: the restated World Magnetic Model, path_gen's true field in the body
frame and the NumPy magnetometer generator against the reference's golden (tests/golden/mag_90deg.npz), the
argument errors that must come before any device work, the path_gen entry points and the data files."""
import ctypes
import os
from datetime import date

import numpy as np
import pytest

import mag_np
from conftest import ROOT, load_golden

MOTION = """ini lat (deg),ini lon (deg),ini alt (m),ini vx_body (m/s),ini vy_body (m/s),ini vz_body (m/s),ini yaw (deg),ini pitch (deg),ini roll (deg)
32,120,0,0,0,0,0,0,0
command type,yaw (deg),pitch (deg),roll (deg),vx_body (m/s),vy_body (m/s),vz_body (m/s),command duration (s),GPS visibility
1,0,0,0,0,0,0,2,1
5,90,0,0,10,0,0,5,1
1,0,0,0,0,0,0,3,1
"""


def write_cof(g, path):
    """The golden's coefficient table as a NOAA .COF file (repr keeps every float exact)."""
    with open(path, 'w') as f:
        f.write('    %r            %s        %s\n' % (float(g['cof_epoch']), str(g['cof_model']),
                                                     str(g['cof_modeldate'])))
        for r in g['cof_rows']:
            f.write('%3d %2d %r %r %r %r\n' % (int(r[0]), int(r[1]), *map(float, r[2:])))
        f.write('9' * 48 + '\n')
    return path


def golden_date(g):
    return date(*map(int, g['date']))


def mag_err(g):
    return {'si': g['mag_si'], 'hi': g['mag_hi'], 'std': g['mag_std']}


def test_wmm_matches_reference_grid():
    """GeoMag on the golden's grid (poles, both hemispheres, 0 / 2.5 / 100 km, two dates): bit-identical."""
    from gnss_ins_sim_b200 import geomag
    g = load_golden('mag_90deg.npz')
    gm = geomag.GeoMag(float(g['cof_epoch']), [(int(r[0]), int(r[1]), *r[2:]) for r in g['cof_rows']])
    assert np.any(np.abs(g['grid'][:, 0]) == 90.0) and g['grid'][:, 2].max() == 100000.0
    for row in g['grid']:
        b = np.array(gm.field(row[0], row[1], row[2], date(*map(int, row[3:6]))))
        ref = row[6:9]
        assert np.abs(b - ref).max() <= 1e-12 * np.linalg.norm(ref), row[:6]
        assert np.array_equal(b, ref), row[:6]


def test_cof_file_round_trip(tmp_path):
    from gnss_ins_sim_b200 import geomag
    g = load_golden('mag_90deg.npz')
    epoch, rows = geomag.read_cof(write_cof(g, str(tmp_path / 'w.COF')))
    assert epoch == float(g['cof_epoch'])
    assert np.array_equal(np.array(rows, dtype=np.float64), g['cof_rows'])
    assert geomag.decimal_year(date(2017, 7, 2)) == 2017 + 182 / 365.0


@pytest.mark.parametrize('rf', [0, 1])
def test_path_gen_reproduces_reference_ref_mag(rf, tmp_path):
    """path_gen(..., magnet=True) on motion_def-90deg_turn.csv: the field and every ref_mag row bit-identical
    to the reference's; in ref_frame 1 the field is [h, 0, v]."""
    from gnss_ins_sim_b200 import geomag, pathgen
    g = load_golden('mag_90deg.npz')
    cof = write_cof(g, str(tmp_path / 'w.COF'))
    ini, cmd = pathgen.parse_motion(os.path.join(ROOT, 'tests', 'golden', 'motion_def-90deg_turn.csv'))
    assert np.array_equal(ini, g['ini'])
    field = np.array(geomag.field_ned(ini, rf, cof, golden_date(g)))
    assert np.array_equal(field, g['geo_mag_n_rf%d' % rf])
    if rf == 1:
        assert field[1] == 0.0 and field[0] > 0.0
    r = pathgen.path_gen(ini, cmd, np.array([[1.0, 100.0], [-1.0, 100.0], [-1.0, 100.0]]),
                         pathgen.HIGH_MOBILITY, rf, True, cof, golden_date(g))
    ref = g['ref_mag_rf%d' % rf]
    assert r['mag'].shape == (ref.shape[0], 4)
    assert np.array_equal(r['mag'][:, 0], r['imu'][:, 0])
    assert np.abs(r['mag'][:, 1:4] - ref).max() <= 1e-12 * np.abs(ref).max()
    assert np.array_equal(r['mag'][:, 1:4], ref)
    # a rotation keeps the field strength
    assert np.allclose(np.linalg.norm(ref, axis=1), np.linalg.norm(field), rtol=1e-14)


@pytest.mark.parametrize('rf', [0, 1])
def test_oracle_reproduces_reference_mag(rf):
    g = load_golden('mag_90deg.npz')
    ref = g['ref_mag_rf%d' % rf]
    z = mag_np.mag_normals(ref.shape[0], g['run_ids'], int(g['seed']))
    o = mag_np.mag_gen(ref, mag_err(g), z)
    assert np.abs(o - g['mag_rf%d' % rf]).max() <= 1e-12 * np.abs(g['mag_rf%d' % rf]).max()


def test_nine_axis_without_coefficients_raises_before_device_work(monkeypatch, tmp_path):
    import importlib.util
    from gnss_ins_sim_b200 import engine, imu_model, sim
    calls = []
    monkeypatch.setattr(engine, 'mag_noise', lambda *a, **k: calls.append(a))
    monkeypatch.setattr(engine, 'to_device', lambda *a, **k: calls.append(a))
    real = importlib.util.find_spec
    monkeypatch.setattr(importlib.util, 'find_spec', lambda name, *a: None if name == 'gnss_ins_sim' else real(name, *a))
    imu = imu_model.IMU('low-accuracy', axis=9, gps=False)
    with pytest.raises(ValueError, match='wmm_file'):
        sim.Sim([100.0, 0.0, 0.0], MOTION, imu=imu).run(2)
    with pytest.raises(ValueError, match='does not exist'):
        sim.Sim([100.0, 0.0, 0.0], MOTION, imu=imu, wmm_file=str(tmp_path / 'none.COF')).run(2)
    # a trajectory dict without ref_mag
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    traj = {k: t[k] for k in ('ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    with pytest.raises(ValueError, match='ref_mag'):
        sim.Sim([100.0, 0.0, 0.0], traj, imu=imu).run(2)
    assert not calls


def test_path_gen_entry_points_agree_without_field():
    """b2ins_path_gen_host and b2ins_path_gen_ex_host with a null field: identical imu / nav / gps / odo rows."""
    from gnss_ins_sim_b200 import _lib, pathgen
    lib = _lib.load()
    ini, cmd = pathgen.parse_motion(MOTION)
    cmd = np.ascontiguousarray(cmd)
    mob = pathgen.HIGH_MOBILITY.copy()
    for rf in (0, 1):
        rows = lib.b2ins_path_rows(_lib.host_ptr(cmd), cmd.shape[0], 100.0)
        outs = []
        for ex in (False, True):
            imu, nav, gps, odo = np.zeros((rows, 7)), np.zeros((rows, 10)), np.zeros((rows, 8)), np.zeros((rows, 5))
            ng = ctypes.c_int64(0)
            args = (_lib.host_ptr(ini), _lib.host_ptr(cmd), cmd.shape[0], 100.0, 1.0, 10.0, 100.0,
                    _lib.host_ptr(mob), rf, rows, _lib.host_ptr(imu), _lib.host_ptr(nav), _lib.host_ptr(gps),
                    ctypes.byref(ng), _lib.host_ptr(odo))
            n = lib.b2ins_path_gen_ex_host(*args, None, None) if ex else lib.b2ins_path_gen_host(*args)
            assert n == rows
            outs.append((imu, nav, gps[:ng.value], odo))
        for a, b in zip(*outs):
            assert np.array_equal(a, b)
        # a field without an output buffer is an argument error
        mag = np.zeros((rows, 4))
        field = np.array([20.0, 1.0, 40.0])
        n = lib.b2ins_path_gen_ex_host(*args[:10], _lib.host_ptr(imu), _lib.host_ptr(nav), None, None, None,
                                       _lib.host_ptr(field), None)
        assert n < 0
        n = lib.b2ins_path_gen_ex_host(*args[:10], _lib.host_ptr(imu), _lib.host_ptr(nav), None, None, None,
                                       _lib.host_ptr(field), _lib.host_ptr(mag))
        assert n == rows and np.array_equal(imu, outs[0][0])
        assert np.allclose(np.linalg.norm(mag[:, 1:4], axis=1), np.linalg.norm(field), rtol=1e-14)


def test_dict_trajectory_carries_ref_mag():
    from gnss_ins_sim_b200 import sim
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    traj = {k: t[k] for k in ('ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    n = traj['ref_gyro'].shape[0]
    out = sim.load_trajectory(dict(traj, ref_mag=np.ones((n, 3))))
    assert out['ref_mag'].shape == (n, 3)
    with pytest.raises(ValueError, match='ref_mag'):
        sim.load_trajectory(dict(traj, ref_mag=np.ones((n, 2))))


def test_write_data_mag_header_and_read_back(tmp_path):
    from gnss_ins_sim_b200 import logged
    rng = np.random.default_rng(3)
    ref = rng.standard_normal((50, 3)) * 30.0
    runs = {0: ref + 0.1, 1: ref - 0.2}
    logged.write_data(str(tmp_path), 'ref_mag', ref, 0)
    logged.write_data(str(tmp_path), 'mag', runs, 1)
    with open(tmp_path / 'mag-0.csv') as f:
        assert f.readline().strip() == 'mag_x (uT),mag_y (uT),mag_z (uT)'
    with open(tmp_path / 'ref_mag.csv') as f:
        assert f.readline().strip() == 'ref_mag_x (uT),ref_mag_y (uT),ref_mag_z (uT)'
    d = logged.read_data_dir(str(tmp_path), 0)
    assert np.array_equal(d['ref_mag'], np.genfromtxt(tmp_path / 'ref_mag.csv', delimiter=',', skip_header=1))
    assert np.abs(d['ref_mag'] - ref).max() <= 1e-15 * np.abs(ref).max() * 10
    for k in (0, 1):
        assert np.abs(d['mag'][k] - runs[k]).max() <= 1e-14 * np.abs(runs[k]).max()
