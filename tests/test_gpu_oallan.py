"""K4o, the overlapping Allan variance, on the GPU: against the NumPy oracle (oracle/oallan_np.py) on the
golden series, ragged lengths, both plugin layouts and series built to defeat an uncompensated prefix;
bit-identical results whatever the batch; the white-noise law through Sim; Sim and the logged-data
directory against the plugin on the same arrays."""
import numpy as np
import pytest

import oallan_np as oa
import oracle_np as onp
from conftest import assert_close, load_golden, write_logged_dir

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _oallan(eng, fs, x):
    """x: numpy [S, n] -> (avar [S, ntau], tau) on the device, as numpy."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    avar, tau = eng.oallan(fs, eng.to_device(x), x.shape[1], x.shape[0])
    torch.cuda.synchronize()
    return avar.cpu().numpy(), tau.cpu().numpy()


def _against_oracle(avar, tau, x, fs, what, rel=1e-9):
    for s in range(x.shape[0]):
        o, ot = oa.oallan_var(x[s], fs)
        assert np.array_equal(tau, ot), what
        assert_close(avar[s], o, rel, 0.0, '%s, series %d' % (what, s))


def test_golden_series(eng):
    g = load_golden('allan.npz')
    for key, fs in (('x', float(g['fs'])), ('x2', float(g['fs2']))):
        x = np.asarray(g[key], dtype=np.float64)[None]
        avar, tau = _oallan(eng, fs, x)
        assert avar.shape == (1, len(onp.allan_multipliers(x.shape[1], fs))) and avar.shape[1] > 0
        _against_oracle(avar, tau, x, fs, key)
        _, t_k4 = eng.allan(fs, eng.to_device(x[0]), x.shape[1], 1)
        assert np.array_equal(tau, t_k4.cpu().numpy())      # the same grid as the non-overlapping curve


@pytest.mark.parametrize('n', [9000, 5 * 2048 - 1, 5 * 2048 + 1, 7 * 2304 - 1, 7 * 2304 + 1, 90, 9])
def test_ragged_lengths(eng, n):
    x = np.random.default_rng(n).standard_normal((3, n)) + 0.5
    avar, tau = _oallan(eng, 1.0, x)
    _against_oracle(avar, tau, x, 1.0, 'n=%d' % n)


def test_too_short_is_empty(eng):
    avar, tau = _oallan(eng, 100.0, np.random.default_rng(0).standard_normal((2, 800)))
    assert avar.shape == (2, 0) and tau.shape == (0,)


def test_plugin_layouts(eng):
    """Allan(overlapping=True): channel-major [R, 3, n] and the interleaved [R, n, 3] triads read in place."""
    from gnss_ins_sim_b200.allan_analysis import Allan
    R, n, fs = 3, 20011, 50.0
    rng = np.random.default_rng(7)
    acm = rng.standard_normal((R, 3, n)) * 0.02 + np.array([0.1, -0.2, -9.8])[None, :, None]
    gcm = rng.standard_normal((R, 3, n)) * 1e-3
    al = Allan(overlapping=True)
    tau, a1, g1 = al.run_batch(fs, acm, gcm, channel_major=True)
    _, a2, g2 = al.run_batch(fs, acm.transpose(0, 2, 1), gcm.transpose(0, 2, 1))
    assert a1.shape == (R, len(tau), 3) and np.array_equal(a1, a2) and np.array_equal(g1, g2)
    for r in range(R):
        for c in range(3):
            o, ot = oa.oallan_var(acm[r, c], fs)
            assert_close(a1[r, :, c], np.sqrt(o), 1e-9, 0.0, 'ad_accel %d %d' % (r, c))
            o, _ = oa.oallan_var(gcm[r, c], fs)
            assert_close(g1[r, :, c], np.sqrt(o), 1e-9, 0.0, 'ad_gyro %d %d' % (r, c))
    assert np.array_equal(tau, ot)
    al.run([fs, acm[1].T, gcm[1].T])
    t, ada, adg = al.get_results()
    assert np.array_equal(t, tau) and np.array_equal(ada, a1[1]) and np.array_equal(adg, g1[1])
    # the default is still the reference's estimator
    _, b1, _ = Allan().run_batch(fs, acm, gcm, channel_major=True)
    o, _ = onp.allan_var(acm[0, 2], fs)
    assert_close(b1[0, :, 2], np.sqrt(o), 1e-9, 0.0, 'Allan() is allan_var')


def test_adversarial_precision(eng):
    """n = 1e6 at 100 Hz: white noise of 1e-3 on a 1e4 offset, an accelerometer z with gravity, and the
    drifting series x_i = 1e4 + 1e-3 i + noise that a plain float64 prefix gets wrong by 3e-8 at m = 1
    (tests/test_cpu_oallan.py shows it on the CPU)."""
    n, fs = 10 ** 6, 100.0
    rng = np.random.default_rng(1)
    ramp = 1e4 + 1e-3 * np.arange(n) + 1e-3 * rng.standard_normal(n)
    off = 1e4 + 1e-3 * rng.standard_normal(n)
    accz = -9.80665 + 0.01 * rng.standard_normal(n)
    x = np.stack([ramp, off, accz])
    avar, tau = _oallan(eng, fs, x)
    _against_oracle(avar, tau, x, fs, 'adversarial')
    f64, _ = oa.oallan_var_prefix64(ramp, fs)
    o, _ = oa.oallan_var(ramp, fs)
    assert abs(f64[0] / o[0] - 1.0) > 1e-8    # the tolerance above would catch a naive prefix


def test_config4_length_channel(eng):
    """One accelerometer z channel at BASELINE config-4 length (14.4 M samples @400 Hz), K1's own draw."""
    from gnss_ins_sim_b200 import imu_model
    n, fs = 14400000, 400.0
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    ref_gyro = eng.to_device(np.zeros((n, 3)))
    ref_accel = eng.to_device(np.tile([0.0, 0.0, -9.8], (n, 1)))
    gyro, accel = eng.imu_noise(fs, 1, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, 5,
                                layout=eng.LAYOUT_CHANNEL_MAJOR)
    z = accel[0, 2:3].contiguous()
    avar, tau = eng.oallan(fs, z, n, 1)
    avar, tau = avar.cpu().numpy(), tau.cpu().numpy()
    del gyro, accel, ref_gyro, ref_accel
    assert avar.shape == (1, 55) and abs(tau[-1] - 2500.0) < 1e-9
    _against_oracle(avar, tau, z.cpu().numpy(), fs, 'config-4 accel z')


def test_constant_series_is_exactly_zero(eng):
    x = np.stack([np.full(50000, v) for v in (3.7, -9.80665, 1e4, 0.0)])
    avar, _ = _oallan(eng, 10.0, x)
    assert avar.size > 0 and np.all(avar == 0.0)


def test_non_finite_samples(eng):
    """Short series with NaN and +-inf samples, in one batch with finite ones, against the definition."""
    n, fs = 400, 1.0
    rng = np.random.default_rng(3)
    rows = []
    for spots in ([(123, np.nan)], [(7, np.inf)], [(0, -np.inf)], [(399, np.inf)],
                  [(200, np.inf), (201, -np.inf)], [(200, np.inf), (204, -np.inf)],
                  [(150, -np.inf), (163, np.inf)], [(50, np.inf), (80, np.inf)],
                  [(10, np.nan), (300, np.inf)], []):
        x = rng.standard_normal(n)
        for i, v in spots:
            x[i] = v
        rows.append(x)
    x = np.stack(rows)
    avar, tau = _oallan(eng, fs, x)
    for s in range(x.shape[0]):
        b, _ = oa.oallan_var_brute(x[s], fs)
        if np.isfinite(x[s]).all():
            assert_close(avar[s], b, 1e-9, 0.0, 'finite series beside the non-finite ones')
        else:
            assert np.array_equal(np.isnan(avar[s]), np.isnan(b)), s
            assert np.array_equal(avar[s][~np.isnan(b)], b[~np.isnan(b)]), s


def test_bit_identical_whatever_the_batch(eng):
    n, fs = 50003, 20.0
    rng = np.random.default_rng(11)
    mine = rng.standard_normal((4, n)) * 0.3 + 2.0
    others = rng.standard_normal((7, n))
    alone = np.concatenate([_oallan(eng, fs, mine[s:s + 1])[0] for s in range(4)])
    batch, _ = _oallan(eng, fs, mine)
    mixed, _ = _oallan(eng, fs, np.concatenate([others[:3], mine, others[3:]]))
    assert np.array_equal(alone, batch) and np.array_equal(alone, mixed[3:7])
    # the interleaved triad layout reads the same samples: the same bits
    tri = np.ascontiguousarray(np.concatenate([mine, others[:2]]).reshape(2, 3, n).transpose(0, 2, 1))
    av, _ = eng.oallan(fs, eng.to_device(tri), n, 6, inner=3, outer_stride=3 * n, sample_stride=3)
    assert np.array_equal(av.cpu().numpy()[:4], alone)


def _white_imu():
    from gnss_ins_sim_b200 import imu_model
    z = np.zeros(3)
    return imu_model.IMU(accuracy={'gyro_b': z, 'gyro_b_stability': z, 'gyro_arw': np.array([0.3, 0.2, 0.25]),
                                   'accel_b': z, 'accel_b_stability': z, 'accel_vrw': np.array([0.05, 0.04, 0.06])},
                         axis=6, gps=False)


def _static(n):
    z = np.zeros((n, 3))
    return {'ref_pos': z, 'ref_vel': z, 'ref_att': z, 'ref_accel': np.tile([0.0, 0.0, -9.8], (n, 1)),
            'ref_gyro': z}


def _sim_ad(sim, R):
    ada, adg, t = sim.get_data(['ad_accel', 'ad_gyro', 'algo_time'])
    return (np.stack([ada['algo0_%d' % r] for r in range(R)]), np.stack([adg['algo0_%d' % r] for r in range(R)]),
            t['algo0_0'])


def test_white_noise_law_through_sim(eng):
    """256 runs of a white-noise-only IMU: mean avar_o(m) within 4 standard errors of sigma^2 / m at every
    tau, and at the two longest tau a smaller spread over the runs than the non-overlapping estimator."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    n, fs, R, seed = 20000, 100.0, 256, 17
    imu = _white_imu()
    out = {}
    for ov in (True, False):
        sim = Sim([fs, 0.0, 0.0], _static(n), ref_frame=1, imu=imu, algorithm=Allan(overlapping=ov), seed=seed)
        sim.run(R)
        out[ov] = _sim_ad(sim, R)
    ada, adg, tau = out[True]
    m = np.rint(tau * fs)
    for ad, sig2 in ((ada, imu.accel_err['vrw'] ** 2 * fs), (adg, imu.gyro_err['arw'] ** 2 * fs)):
        av = ad ** 2                                   # [R, ntau, 3]
        mean, se = av.mean(0), av.std(0, ddof=1) / np.sqrt(R)
        law = sig2[None, :] / m[:, None]
        assert (np.abs(mean - law) <= 4.0 * se).all(), np.abs(mean - law) / se
    for o, no in ((ada, out[False][0]), (adg, out[False][1])):
        assert (o[:, -2:, :].std(0) < no[:, -2:, :].std(0)).all()


def test_sim_equals_the_plugin_on_the_materialised_series(eng, monkeypatch):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    from gnss_ins_sim_b200 import imu_model
    n, fs, R, seed = 30011, 100.0, 5, 23
    imu = imu_model.IMU('low-accuracy', axis=6, gps=False)
    traj = _static(n)
    sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(overlapping=True), seed=seed)
    sim.run(R)
    ada, adg, tau = _sim_ad(sim, R)
    gyro, accel = eng.imu_noise(fs, R, eng.to_device(traj['ref_gyro']), eng.to_device(traj['ref_accel']),
                                imu.gyro_err, imu.accel_err, seed, layout=eng.LAYOUT_CHANNEL_MAJOR)
    t2, a2, g2 = Allan(overlapping=True).run_batch(fs, accel, gyro, channel_major=True)
    assert np.array_equal(tau, t2) and np.array_equal(ada, a2) and np.array_equal(adg, g2)
    # small run blocks: the same bits
    monkeypatch.setattr(Sim, '_allan_block', lambda self, *a: 2)
    sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(overlapping=True), seed=seed)
    sim.run(R)
    b_a, b_g, _ = _sim_ad(sim, R)
    assert np.array_equal(b_a, ada) and np.array_equal(b_g, adg)


def test_logged_data_directory(eng, tmp_path):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    g = load_golden('logged_bosch.npz')
    d = write_logged_dir(str(tmp_path / 'bosch'), g)
    sim = Sim([100.0, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=Allan(overlapping=True))
    sim.run(1)
    ada, adg, tau = (sim.get_data([k])[0]['algo0_0'] for k in ('ad_accel', 'ad_gyro', 'algo_time'))
    t2, a2, g2 = Allan(overlapping=True).run_batch(100.0, g['accel'][None], g['gyro'][None])
    assert np.array_equal(tau, t2) and a2.shape[1] > 0
    assert_close(ada, a2[0], 1e-9, 0.0, 'logged accel')
    assert_close(adg, g2[0], 1e-9, 0.0, 'logged gyro')
