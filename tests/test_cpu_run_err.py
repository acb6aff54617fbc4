"""Run-to-run bias, scale-factor and misalignment errors of the IMU model without a GPU: the IMU's units and checks,
the C struct and its argument checks, the oracle (oracle/run_err_np.py) and the law of its draws, and the plugins
that cannot take the errors."""
import ctypes
import math
import os

import numpy as np
import pytest

import noise952_np as nz
import oracle_np as onp
import run_err_np as rx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D2R = math.pi / 180.0
BASE = {'gyro_b': [0.0] * 3, 'gyro_b_stability': [1.0] * 3, 'gyro_arw': [0.1] * 3, 'gyro_b_corr': [100.0] * 3,
        'accel_b': [0.0] * 3, 'accel_b_stability': [1e-4] * 3, 'accel_vrw': [0.05] * 3, 'accel_b_corr': [100.0] * 3}
OFF = 1.0 - np.eye(3)


def test_imu_run_errors_in_si_units():
    from gnss_ins_sim_b200.imu_model import IMU
    ma = [[0.0, 0.1, 0.2], [0.3, 0.0, 0.4], [0.5, 0.6, 0.0]]
    imu = IMU(dict(BASE, gyro_b_std=[3.6, 7.2, 10.8], gyro_sf=1000.0, gyro_ma=0.05, accel_b_std=0.01,
                   accel_sf=[100.0, 200.0, 300.0], accel_ma=ma))
    np.testing.assert_allclose(imu.gyro_err['b_std'], np.array([3.6, 7.2, 10.8]) * D2R / 3600.0, rtol=1e-15)
    np.testing.assert_allclose(imu.gyro_err['sf'], [1e-3] * 3, rtol=1e-15)
    np.testing.assert_allclose(imu.gyro_err['ma'], 0.05 * D2R * OFF, rtol=1e-15)     # scalar -> off-diagonals
    assert imu.gyro_err['ma'].shape == (3, 3) and np.all(np.diag(imu.gyro_err['ma']) == 0.0)
    np.testing.assert_allclose(imu.accel_err['b_std'], [0.01] * 3, rtol=1e-15)
    np.testing.assert_allclose(imu.accel_err['sf'], [1e-4, 2e-4, 3e-4], rtol=1e-15)
    np.testing.assert_allclose(imu.accel_err['ma'], np.array(ma) * D2R, rtol=1e-15)
    # absent keys are not stored; grades and dicts without the keys gain none
    only = IMU(dict(BASE, gyro_sf=[5.0] * 3))
    assert 'sf' in only.gyro_err and not {'b_std', 'ma'} & set(only.gyro_err)
    assert not {'b_std', 'sf', 'ma'} & set(only.accel_err)
    for grade in ('low-accuracy', 'mid-accuracy', 'high-accuracy'):
        g = IMU(grade)
        assert set(g.gyro_err) == {'b', 'b_drift', 'b_corr', 'arw'}
        assert set(g.accel_err) == {'b', 'b_drift', 'b_corr', 'vrw'}
    assert set(IMU(dict(BASE)).gyro_err) == {'b', 'b_drift', 'b_corr', 'arw'}


def test_imu_run_error_keys_are_validated():
    from gnss_ins_sim_b200.imu_model import IMU
    for key, bad in (('gyro_b_std', -1.0), ('gyro_sf', float('nan')), ('accel_sf', float('inf')),
                     ('accel_b_std', -0.1), ('gyro_ma', -0.5), ('accel_ma', float('nan')),
                     ('gyro_b_std', float('-inf'))):
        with pytest.raises(ValueError, match=key):
            IMU(dict(BASE, **{key: [bad] * 3 if 'ma' not in key else bad}))
    with pytest.raises(ValueError, match='gyro_ma must have a zero diagonal'):
        IMU(dict(BASE, gyro_ma=np.eye(3)))
    with pytest.raises(ValueError, match='accel_ma'):
        IMU(dict(BASE, accel_ma=[[0.0, 1.0, 1.0], [1.0, 0.0, np.inf], [1.0, 1.0, 0.0]]))
    # the setters take the stored SI keys, with the same checks
    imu = IMU('mid-accuracy')
    imu.set_gyro_error({'sf': 1e-3, 'ma': 1e-4, 'b_std': np.full(3, 2e-6)})
    imu.set_accel_error({'b_std': np.full(3, 1e-3)})
    assert imu.gyro_err['sf'].shape == (3,) and np.array_equal(imu.gyro_err['ma'], 1e-4 * OFF)
    assert imu.accel_err['b_std'][0] == 1e-3
    with pytest.raises(ValueError, match='sf must be finite and >= 0'):
        imu.set_gyro_error({'sf': -1e-3})
    with pytest.raises(ValueError, match='ma must have a zero diagonal'):
        imu.set_accel_error({'ma': np.full((3, 3), 1e-3)})
    with pytest.raises(ValueError, match='unsupported key'):
        imu.set_gyro_error({'sf_x': 1.0})


def test_run_err_struct_matches_header():
    from gnss_ins_sim_b200 import _lib
    assert ctypes.sizeof(_lib.RunErr) == 120
    assert (_lib.RunErr.b.offset, _lib.RunErr.sf.offset, _lib.RunErr.ma.offset) == (0, 24, 48)
    with open(os.path.join(ROOT, 'include', 'b2ins.h')) as f:
        h = f.read()
    assert 'typedef struct b2ins_run_err {\n  double b[3];\n  double sf[3];\n  double ma[3][3];\n} b2ins_run_err;' in h
    # absent or zero keys pass NULL: the _rx entry points then launch what the _ex ones do
    assert _lib.run_err({'b': np.ones(3)}) is None
    assert _lib.run_err({'b_std': np.zeros(3), 'sf': 0.0, 'ma': np.zeros((3, 3))}) is None
    assert _lib.set_run_errors({'sf': [0.0, 1e-6, 0.0], 'ma': 0.0}) == ['sf']
    e = _lib.run_err({'sf': np.array([1.0, 2.0, 3.0]), 'ma': 0.5})
    assert list(e.sf) == [1.0, 2.0, 3.0] and list(e.b) == [0.0] * 3
    assert [list(r) for r in e.ma] == (0.5 * OFF).tolist()
    m = np.arange(9.0).reshape(3, 3) * OFF
    assert [list(r) for r in _lib.run_err({'ma': m}).ma] == m.tolist()


def _pins():
    """(name, call, expected (rc, text)) of the new entry points' argument checks, decided before any CUDA call."""
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    n, R = 10, 2
    x = np.zeros((R, n, 3))
    ref = np.zeros((n, 3))
    hp = _lib.host_ptr
    se = _lib.sensor_err({'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf),
                          'arw': np.zeros(3)}, 'arw')
    vib = _lib.vib(None)
    good = _lib.run_err({'sf': 1e-3, 'ma': 1e-4, 'b_std': 1e-5})
    neg, nan, diag = (_lib.run_err({'sf': 1e-3}) for _ in range(3))
    neg.b[1] = -1.0
    nan.ma[2][0] = float('nan')
    diag.ma[1][1] = 1e-3
    fake = ctypes.c_void_p(0x1000)           # a device pointer never dereferenced: the checks come first
    B = ctypes.byref

    def noise(rg=good, ra=None, fs=100.0, runs=R, layout=0):
        return lib.b2ins_imu_noise_rx_f64(fs, runs, n, fake, fake, B(se), B(se), None, None, B(vib), B(vib), 1, 0,
                                          layout, fake, fake, None, rg, ra, None)

    def host(rg=good, ra=None, runs=R):
        return lib.b2ins_imu_noise_rx_f64_host(100.0, runs, n, hp(ref), hp(ref), B(se), B(se), None, None, B(vib),
                                               B(vib), 1, 0, 0, hp(x), hp(x.copy()), None, rg, ra)

    def stats(rg=good, ra=None, start=-1):
        return lib.b2ins_imu_err_stats_rx_f64(100.0, R, n, fake, fake, B(se), B(se), None, None, B(vib), B(vib), 1,
                                              0, start, fake, None, rg, ra, None)

    def table(rg=good, ra=None, runs=R, out=fake):
        return lib.b2ins_imu_run_err_f64(1, runs, 0, rg, ra, out, None)

    arg = lambda t: (_lib.ERR_ARG, t)  # noqa: E731
    bad_sigma = arg('run errors: b, sf and ma must be finite and >= 0')
    bad_diag = arg('run errors: the diagonal of ma must be 0')
    return [
        ('noise neg b', lambda: noise(rg=B(neg)), bad_sigma),
        ('noise nan ma accel', lambda: noise(rg=None, ra=B(nan)), bad_sigma),
        ('noise diag', lambda: noise(rg=B(diag)), bad_diag),
        ('noise fs', lambda: noise(rg=B(good), fs=0.0), arg('fs must be positive')),
        ('noise layout', lambda: noise(rg=B(good), layout=3), arg('layout must be B2INS_LAYOUT_*')),
        ('noise runs 0', lambda: noise(rg=B(good), runs=0), (_lib.OK, None)),
        ('host neg b', lambda: host(rg=B(neg)), bad_sigma),
        ('host diag accel', lambda: host(rg=None, ra=B(diag)), bad_diag),
        ('host runs 0', lambda: host(rg=B(good), runs=0), (_lib.OK, None)),
        ('stats nan', lambda: stats(rg=B(nan)), bad_sigma),
        ('stats diag', lambda: stats(ra=B(diag)), bad_diag),
        ('stats start', lambda: stats(rg=B(good), start=n), arg('stats_start must be < n')),
        ('table neg', lambda: table(rg=B(neg)), bad_sigma),
        ('table diag', lambda: table(rg=None, ra=B(diag)), bad_diag),
        ('table runs', lambda: table(rg=B(good), runs=-1), arg('runs must be non-negative')),
        ('table null', lambda: table(rg=B(good), out=None), arg('null buffer')),
        ('table runs 0', lambda: table(rg=B(good), runs=0), (_lib.OK, None)),
    ], {'noise': lambda: noise(rg=B(good)), 'host': lambda: host(rg=B(good)),
        'stats': lambda: stats(rg=B(good)), 'table': lambda: table(rg=B(good))}


def test_new_entry_points_check_their_arguments():
    """Each bad argument gives B2INS_ERR_ARG and its b2ins_last_error() text before any CUDA call; without a device,
    valid calls reach CUDA and report B2INS_ERR_CUDA."""
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    pins, valid = _pins()
    for name, call, (rc, text) in pins:
        got = call()
        assert got == rc, (name, got, lib.b2ins_last_error())
        if text is not None:
            assert lib.b2ins_last_error().decode() == text, name
    if lib.b2ins_device_count() == 0:
        for name, call in valid.items():
            assert call() == _lib.ERR_CUDA, name


def _errs(**kw):
    g = {'b': np.array([1e-4, 0.0, -2e-4]), 'b_drift': np.full(3, 1e-5), 'b_corr': np.array([100.0, np.inf, 5.0]),
         'arw': np.full(3, 1e-4)}
    a = {'b': np.array([0.01, 0.0, -0.02]), 'b_drift': np.full(3, 1e-3), 'b_corr': np.array([np.inf, 50.0, 1.0]),
         'vrw': np.full(3, 1e-3)}
    return dict(g, **kw), dict(a, **kw)


def test_oracle_with_zero_run_errors_is_noise952():
    n = 300
    rng = np.random.default_rng(3)
    rg, ra = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
    for extra in ({}, {'b_std': np.zeros(3), 'sf': np.zeros(3), 'ma': np.zeros((3, 3))}):
        ge, ae = _errs(rrw=np.full(3, 1e-4), **extra)
        g0, a0 = nz.imu_noise(100.0, rg, ra, ge, ae, 9, [0, 5, 2 ** 33])
        g1, a1 = rx.imu_noise(100.0, rg, ra, ge, ae, 9, [0, 5, 2 ** 33])
        assert np.array_equal(g0, g1) and np.array_equal(a0, a1)


def test_oracle_delta_is_s_ref_plus_b():
    """Per sample: the oracle's measurement minus noise952's is b_run + S ref, with S and b_run drawn as the
    spec says (pair by pair from normal_pair), and sigma 0 gives exactly 0."""
    n, seed, runs = 50, 77, [4, 2 ** 32 + 1, 2 ** 32 - 1]
    rng = np.random.default_rng(5)
    rg, ra = rng.standard_normal((n, 3)), rng.standard_normal((n, 3)) + [0.0, 0.0, -9.8]
    ma = np.array([[0.0, 1e-3, 0.0], [2e-3, 0.0, 3e-3], [0.0, 4e-3, 0.0]])
    ge, ae = _errs(b_std=np.array([1e-5, 0.0, 3e-5]), sf=np.array([1e-3, 2e-3, 0.0]), ma=ma)
    g0, a0 = nz.imu_noise(100.0, rg, ra, ge, ae, seed, runs)
    g1, a1 = rx.imu_noise(100.0, rg, ra, ge, ae, seed, runs)
    for sensor, err, ref, d in ((1, ge, rg, g1 - g0), (0, ae, ra, a1 - a0)):
        tab = rx.table(err, sensor, seed, runs)
        for ri, run in enumerate(runs):
            S, b = np.zeros((3, 3)), np.zeros(3)
            for j in range(6):
                z0, z1 = onp.normal_pair(rx.RUN_ERR_T, rx.DRAW_RUN_ERR + 6 * sensor + j, run, seed)
                if j < 3:
                    b[j], S[j, j] = err['b_std'][j] * z0, err['sf'][j] * z1
                else:
                    (c0, c1), i = rx.OFF_DIAG[j - 3], j - 3
                    S[i, c0], S[i, c1] = err['ma'][i, c0] * z0, err['ma'][i, c1] * z1
            assert np.array_equal(tab[ri, :, :3], S) and np.array_equal(tab[ri, :, 3], b)
            assert S[2, 2] == 0.0 and S[0, 2] == 0.0 and b[1] == 0.0      # sigma 0 -> 0
            want = b[None] + ref.dot(S.T)
            np.testing.assert_allclose(d[ri], want, rtol=0.0, atol=1e-15 * max(1.0, np.abs(ref).max()) * 16)


def test_run_error_draws_follow_their_law():
    """Over 20 000 oracle runs each of the 24 parameters is N(0, sigma^2): its sample variance / sigma^2 inside a
    chi-square bound (6 standard deviations of the ratio), its mean within 6 standard errors, and no two
    parameters correlated beyond 5 / sqrt(R)."""
    R = 20000
    sig = {'b_std': np.array([1.0, 2.0, 3.0]), 'sf': np.array([4.0, 5.0, 6.0]),
           'ma': np.array([[0.0, 7.0, 8.0], [9.0, 0.0, 10.0], [11.0, 12.0, 0.0]])}
    runs = np.arange(R, dtype=np.uint64) + np.uint64(2 ** 31)
    cols, scale = [], []
    for sensor in (0, 1):
        t = rx.table(sig, sensor, 1234, runs)
        for i in range(3):
            for j in range(3):
                cols.append(t[:, i, j])
                scale.append(sig['sf'][i] if i == j else sig['ma'][i, j])
            cols.append(t[:, i, 3])
            scale.append(sig['b_std'][i])
    X = np.stack(cols, axis=1) / np.array(scale)
    assert X.shape == (R, 24)
    ratio = np.mean(X * X, axis=0)              # chi^2_R / R: mean 1, sd sqrt(2 / R)
    assert np.all(np.abs(ratio - 1.0) <= 6.0 * math.sqrt(2.0 / R)), ratio
    assert np.all(np.abs(X.mean(0)) <= 6.0 / math.sqrt(R)), X.mean(0)
    C = np.corrcoef(X, rowvar=False)
    off = np.abs(C - np.diag(np.diag(C)))
    assert off.max() <= 5.0 / math.sqrt(R), off.max()


@pytest.mark.parametrize('plugin', ['ins_loose', 'odo'])
def test_sim_refuses_plugins_whose_kernels_make_no_run_errors(plugin):
    from gnss_ins_sim_b200.imu_model import IMU
    from gnss_ins_sim_b200.sim import Sim
    n = 8
    traj = {k: np.zeros((n, 3)) for k in ('ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro')}
    traj['ref_odo'] = np.zeros(n)
    if plugin == 'ins_loose':
        from gnss_ins_sim_b200.ins_loose import InsLoose
        algo = InsLoose(np.zeros(9))
    else:
        from gnss_ins_sim_b200.free_integration_odo import FreeIntegration as FreeIntegrationOdo
        algo = FreeIntegrationOdo(np.zeros(9))
    imu = IMU(dict(BASE, gyro_sf=[100.0] * 3, accel_ma=0.01), odo=True)
    sim = Sim(100.0, traj, imu=imu, algorithm=algo)
    with pytest.raises(ValueError, match='scale-factor') as e:
        sim.run(1)
    assert "'gyro sf'" in str(e.value) and "'accel ma'" in str(e.value)
    assert 'gyro' not in sim.data and 'accel' not in sim.data      # refused before anything was reset
