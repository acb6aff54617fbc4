"""K4o's Hadamard form, the overlapping Hadamard variance, on the GPU: against the NumPy oracle
(oracle/ohadamard_np.py) on the golden series, ragged lengths, both plugin layouts and series built to defeat an
uncompensated prefix; exact zeros on constants and integer ramps; the IEEE non-finite rule; bit-identical results
whatever the batch; the white-noise law through Sim; Sim with Allan(overlapping=True) and Hadamard() against the
plugins on the same series; a logged directory whose gyro drifts."""
import numpy as np
import pytest

import oallan_np as oa
import ohadamard_np as oh
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


def _ohad(eng, fs, x):
    """x: numpy [S, n] -> (hvar [S, ntau], tau) on the device, as numpy."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    hvar, tau = eng.ohadamard(fs, eng.to_device(x), x.shape[1], x.shape[0])
    torch.cuda.synchronize()
    return hvar.cpu().numpy(), tau.cpu().numpy()


def _against_oracle(hvar, tau, x, fs, what, rel=1e-9):
    for s in range(x.shape[0]):
        o, ot = oh.ohadamard_var(x[s], fs)
        assert np.array_equal(tau, ot), what
        assert_close(hvar[s], o, rel, 0.0, '%s, series %d' % (what, s))


def test_golden_series(eng):
    g = load_golden('allan.npz')
    for key, fs in (('x', float(g['fs'])), ('x2', float(g['fs2']))):
        x = np.asarray(g[key], dtype=np.float64)[None]
        hvar, tau = _ohad(eng, fs, x)
        assert hvar.shape == (1, len(onp.allan_multipliers(x.shape[1], fs))) and hvar.shape[1] > 0
        _against_oracle(hvar, tau, x, fs, key)
        _, t_k4 = eng.allan(fs, eng.to_device(x[0]), x.shape[1], 1)
        assert np.array_equal(tau, t_k4.cpu().numpy())      # the same grid as the Allan curves


@pytest.mark.parametrize('n', [9000, 5 * 2048 - 1, 5 * 2048 + 1, 7 * 2304 - 1, 7 * 2304 + 1, 90, 9])
def test_ragged_lengths(eng, n):
    x = np.random.default_rng(n).standard_normal((3, n)) + 0.5
    hvar, tau = _ohad(eng, 1.0, x)
    _against_oracle(hvar, tau, x, 1.0, 'n=%d' % n)


def test_too_short_is_empty(eng):
    hvar, tau = _ohad(eng, 100.0, np.random.default_rng(0).standard_normal((2, 800)))
    assert hvar.shape == (2, 0) and tau.shape == (0,)


def test_plugin_layouts(eng):
    """Hadamard(): channel-major [R, 3, n] and the interleaved [R, n, 3] triads read in place."""
    from gnss_ins_sim_b200.allan_analysis import Hadamard
    R, n, fs = 3, 20011, 50.0
    rng = np.random.default_rng(7)
    acm = rng.standard_normal((R, 3, n)) * 0.02 + np.array([0.1, -0.2, -9.8])[None, :, None]
    gcm = rng.standard_normal((R, 3, n)) * 1e-3 + 1e-6 * np.arange(n)
    h = Hadamard()
    tau, a1, g1 = h.run_batch(fs, acm, gcm, channel_major=True)
    _, a2, g2 = h.run_batch(fs, acm.transpose(0, 2, 1), gcm.transpose(0, 2, 1))
    assert a1.shape == (R, len(tau), 3) and np.array_equal(a1, a2) and np.array_equal(g1, g2)
    for r in range(R):
        for c in range(3):
            o, ot = oh.ohadamard_var(acm[r, c], fs)
            assert_close(a1[r, :, c], np.sqrt(o), 1e-9, 0.0, 'hd_accel %d %d' % (r, c))
            o, _ = oh.ohadamard_var(gcm[r, c], fs)
            assert_close(g1[r, :, c], np.sqrt(o), 1e-9, 0.0, 'hd_gyro %d %d' % (r, c))
    assert np.array_equal(tau, ot)
    h.run([fs, acm[1].T, gcm[1].T])
    t, hda, hdg = h.get_results()
    assert np.array_equal(t, tau) and np.array_equal(hda, a1[1]) and np.array_equal(hdg, g1[1])


def test_adversarial_precision(eng):
    """n = 1e6 at 100 Hz: white noise of 1e-3 on a 1e4 offset, an accelerometer z with gravity, and the
    drifting series x_i = 1e4 + 1e-3 i + noise that a plain float64 prefix gets badly wrong
    (tests/test_cpu_ohadamard.py shows it on the CPU).  Against the exact fixed-point form: at long tau the
    long-double oracle's own prefix rounding reaches 4.5e-9 of hvar on the drifting series (the drift cancels,
    the prefix does not); it holds the other two, and every tau up to 10^4, to 1e-9."""
    n, fs = 10 ** 6, 100.0
    rng = np.random.default_rng(1)
    ramp = 1e4 + 1e-3 * np.arange(n) + 1e-3 * rng.standard_normal(n)
    off = 1e4 + 1e-3 * rng.standard_normal(n)
    accz = -9.80665 + 0.01 * rng.standard_normal(n)
    x = np.stack([ramp, off, accz])
    hvar, tau = _ohad(eng, fs, x)
    m = np.rint(tau * fs)
    for s in range(3):
        ex, t_ex = oh.ohadamard_var_fixed(x[s], fs)
        assert np.array_equal(tau, t_ex)
        assert_close(hvar[s], ex, 1e-9, 0.0, 'adversarial, series %d, exact form' % s)
        ld, _ = oh.ohadamard_var(x[s], fs)
        keep = (m <= 10 ** 4) if s == 0 else np.ones(m.size, bool)
        assert_close(hvar[s][keep], ld[keep], 1e-9, 0.0, 'adversarial, series %d, long double' % s)
    f64, _ = oh.ohadamard_var_prefix64(ramp, fs)
    o, _ = oh.ohadamard_var_fixed(ramp, fs)
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
    hvar, tau = eng.ohadamard(fs, z, n, 1)
    hvar, tau = hvar.cpu().numpy(), tau.cpu().numpy()
    del gyro, accel, ref_gyro, ref_accel
    assert hvar.shape == (1, 55) and abs(tau[-1] - 2500.0) < 1e-9
    _against_oracle(hvar, tau, z.cpu().numpy(), fs, 'config-4 accel z')


def test_constant_and_integer_ramp_are_exactly_zero(eng):
    n = 50000
    x = np.stack([np.full(n, 3.7), np.full(n, -9.80665), np.full(n, 1e4), np.zeros(n),
                  3.0 * np.arange(n), -7.0 * np.arange(n) + 12.0])
    hvar, _ = _ohad(eng, 10.0, x)
    assert hvar.size > 0 and np.all(hvar == 0.0)
    av, _ = eng.oallan(10.0, eng.to_device(x[4:5]), n, 1)     # the Allan variance keeps the ramp: b^2 m^2 / 2
    m = np.asarray(onp.allan_multipliers(n, 10.0), dtype=np.float64)
    assert_close(av.cpu().numpy()[0], 9.0 * m * m / 2.0, 1e-12, 0.0, 'oallan of 3 i')


def test_non_finite_samples(eng):
    """Short series with NaN and +-inf samples, in one batch with finite ones, against the definition: every
    sign pattern of the rule (a window with both signs, S2 and S0 of opposite signs, S1 with the sign of S2
    or S0) at several distances."""
    n, fs = 400, 1.0
    rng = np.random.default_rng(3)
    rows = []
    for spots in ([(123, np.nan)], [(7, np.inf)], [(0, -np.inf)], [(399, np.inf)],
                  [(200, np.inf), (201, -np.inf)], [(200, np.inf), (204, -np.inf)],
                  [(100, np.inf), (110, -np.inf)], [(100, np.inf), (110, np.inf)],
                  [(100, -np.inf), (105, -np.inf)], [(100, np.inf), (105, -np.inf)],
                  [(150, -np.inf), (163, np.inf)], [(50, np.inf), (80, np.inf)], [(50, np.inf), (140, -np.inf)],
                  [(10, np.nan), (300, np.inf)], []):
        x = rng.standard_normal(n)
        for i, v in spots:
            x[i] = v
        rows.append(x)
    x = np.stack(rows)
    hvar, tau = _ohad(eng, fs, x)
    mixed = 0
    for s in range(x.shape[0]):
        b, _ = oh.ohadamard_var_brute(x[s], fs)
        if np.isfinite(x[s]).all():
            assert_close(hvar[s], b, 1e-9, 0.0, 'finite series beside the non-finite ones')
        else:
            assert np.array_equal(np.isnan(hvar[s]), np.isnan(b)), s
            assert np.array_equal(hvar[s][~np.isnan(b)], b[~np.isnan(b)]), s
            mixed += np.isnan(b).any() and not np.isnan(b).all()
    assert mixed >= 5      # the patterns give +inf at some tau and NaN at others


def test_bit_identical_whatever_the_batch(eng):
    n, fs = 50003, 20.0
    rng = np.random.default_rng(11)
    mine = rng.standard_normal((4, n)) * 0.3 + 2.0
    others = rng.standard_normal((7, n))
    alone = np.concatenate([_ohad(eng, fs, mine[s:s + 1])[0] for s in range(4)])
    batch, _ = _ohad(eng, fs, mine)
    mixed, _ = _ohad(eng, fs, np.concatenate([others[:3], mine, others[3:]]))
    assert np.array_equal(alone, batch) and np.array_equal(alone, mixed[3:7])
    # the interleaved triad layout reads the same samples: the same bits
    tri = np.ascontiguousarray(np.concatenate([mine, others[:2]]).reshape(2, 3, n).transpose(0, 2, 1))
    hv, _ = eng.ohadamard(fs, eng.to_device(tri), n, 6, inner=3, outer_stride=3 * n, sample_stride=3)
    assert np.array_equal(hv.cpu().numpy()[:4], alone)


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


def _sim_out(sim, R, names, algo):
    a, g, t = sim.get_data(list(names) + ['algo_time'])
    key = '%s_%%d' % algo
    return (np.stack([a[key % r] for r in range(R)]), np.stack([g[key % r] for r in range(R)]), t[key % 0])


def test_white_noise_law_through_sim(eng):
    """256 runs of a white-noise-only IMU: mean hvar(m) within 4 standard errors of sigma^2 / m at every tau."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Hadamard
    n, fs, R, seed = 20000, 100.0, 256, 17
    imu = _white_imu()
    sim = Sim([fs, 0.0, 0.0], _static(n), ref_frame=1, imu=imu, algorithm=Hadamard(), seed=seed)
    sim.run(R)
    hda, hdg, tau = _sim_out(sim, R, ('hd_accel', 'hd_gyro'), 'algo0')
    assert 'ad_accel' not in sim.data and 'ad_gyro' not in sim.data
    m = np.rint(tau * fs)
    for hd, sig2 in ((hda, imu.accel_err['vrw'] ** 2 * fs), (hdg, imu.gyro_err['arw'] ** 2 * fs)):
        hv = hd ** 2                                   # [R, ntau, 3]
        mean, se = hv.mean(0), hv.std(0, ddof=1) / np.sqrt(R)
        law = sig2[None, :] / m[:, None]
        assert (np.abs(mean - law) <= 4.0 * se).all(), np.abs(mean - law) / se


def test_sim_with_both_estimators_equals_the_plugins(eng, monkeypatch):
    """Allan(overlapping=True) and Hadamard() in one Sim: both curves from the same series, each equal to its
    plugin on K1's materialised series; small run blocks give the same bits."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan, Hadamard
    from gnss_ins_sim_b200 import imu_model
    n, fs, R, seed = 30011, 100.0, 5, 23
    imu = imu_model.IMU('low-accuracy', axis=6, gps=False)
    traj = _static(n)
    sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=[Allan(overlapping=True), Hadamard()],
              seed=seed)
    sim.run(R)
    ada, adg, tau = _sim_out(sim, R, ('ad_accel', 'ad_gyro'), 'algo0')
    hda, hdg, tau1 = _sim_out(sim, R, ('hd_accel', 'hd_gyro'), 'algo1')
    assert sorted(sim.get_data(['algo_time'])[0]) == sorted(['algo%d_%d' % (a, r) for a in (0, 1) for r in range(R)])
    assert sorted(sim.get_data(['ad_gyro'])[0]) == ['algo0_%d' % r for r in range(R)]
    assert sorted(sim.get_data(['hd_gyro'])[0]) == ['algo1_%d' % r for r in range(R)]
    gyro, accel = eng.imu_noise(fs, R, eng.to_device(traj['ref_gyro']), eng.to_device(traj['ref_accel']),
                                imu.gyro_err, imu.accel_err, seed, layout=eng.LAYOUT_CHANNEL_MAJOR)
    t2, a2, g2 = Allan(overlapping=True).run_batch(fs, accel, gyro, channel_major=True)
    t3, a3, g3 = Hadamard().run_batch(fs, accel, gyro, channel_major=True)
    assert np.array_equal(tau, t2) and np.array_equal(ada, a2) and np.array_equal(adg, g2)
    assert np.array_equal(tau1, t3) and np.array_equal(hda, a3) and np.array_equal(hdg, g3)
    assert not np.array_equal(a2, a3)
    # the reverse order and small run blocks: the same bits
    monkeypatch.setattr(Sim, '_allan_block', lambda self, *a: 2)
    sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=[Hadamard(), Allan(overlapping=True)],
              seed=seed)
    sim.run(R)
    b_a, b_g, _ = _sim_out(sim, R, ('hd_accel', 'hd_gyro'), 'algo0')
    assert np.array_equal(b_a, hda) and np.array_equal(b_g, hdg)
    b_a, b_g, _ = _sim_out(sim, R, ('ad_accel', 'ad_gyro'), 'algo1')
    assert np.array_equal(b_a, ada) and np.array_equal(b_g, adg)
    assert len(sim.get_data(['algo_time'])[0]) == 2 * R


def test_logged_directory_with_a_drifting_gyro(eng, tmp_path):
    """A static recording whose gyro x drifts linearly (b per sample): Hadamard() stays on the white-noise law at
    long tau, Allan(overlapping=True) follows b^2 m^2 / 2 there; both equal their plugins on the arrays."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan, Hadamard
    n, fs, sig, b = 200000, 100.0, 1e-3, 1e-7
    rng = np.random.default_rng(29)
    gyro = sig * rng.standard_normal((n, 3))
    gyro[:, 0] += b * np.arange(n)
    accel = 0.02 * rng.standard_normal((n, 3)) + np.array([0.0, 0.0, -9.8])
    d = write_logged_dir(str(tmp_path / 'drift'), {'fs': fs, 'gyro': gyro, 'accel': accel})
    sim = Sim([fs, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=[Allan(overlapping=True), Hadamard()])
    sim.run(1)
    adg, hdg, hda, tau = (sim.get_data([k])[0][a] for k, a in (('ad_gyro', 'algo0_0'), ('hd_gyro', 'algo1_0'),
                                                                ('hd_accel', 'algo1_0'), ('algo_time', 'algo1_0')))
    t2, a2, g2 = Hadamard().run_batch(fs, accel[None], gyro[None])
    _, _, g3 = Allan(overlapping=True).run_batch(fs, accel[None], gyro[None])
    assert np.array_equal(tau, t2) and tau.size > 0
    assert_close(hdg, g2[0], 1e-9, 0.0, 'logged hd_gyro')
    assert_close(hda, a2[0], 1e-9, 0.0, 'logged hd_accel')
    assert_close(adg, g3[0], 1e-9, 0.0, 'logged ad_gyro')
    m = np.rint(tau * fs)[-3:]
    white = sig ** 2 / m
    hv, av = hdg[-3:, 0] ** 2, adg[-3:, 0] ** 2
    assert ((hv / white > 0.25) & (hv / white < 4.0)).all(), hv / white
    assert (np.abs(av / (b * b * m * m / 2.0) - 1.0) < 0.2).all(), av / (b * b * m * m / 2.0)
    assert (av / white > 1e3).all()
    # the channels without drift: the two estimators agree to within their spread
    assert ((hdg[-3:, 1:] / adg[-3:, 1:]) ** 2 > 0.2).all() and ((hdg[-3:, 1:] / adg[-3:, 1:]) ** 2 < 5.0).all()
