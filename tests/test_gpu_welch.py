"""Welch power spectral density (K11) on the GPU: against the NumPy oracle (oracle/welch_np.py) over the grid of
lengths, overlaps, ragged series and windows, including one config-4-length channel; the same bits whatever the
batch, position and layout; the non-finite rule; K5's vibration synthesis inverted exactly; a sinusoidal
environment's power; the white-noise law through Sim; Sim with Psd against the plugin, a logged directory and
save_data."""
import os

import numpy as np
import pytest

import welch_np as wn
from conftest import write_logged_dir

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _welch(eng, fs, x, N, D, window):
    """x: numpy [S, n] channel-major -> (psd [S, L], freq [L]) as numpy."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    psd, freq = eng.welch(fs, eng.to_device(x), x.shape[1], x.shape[0], N, D, np.asarray(window, dtype=np.float64))
    torch.cuda.synchronize()
    return psd.cpu().numpy(), freq.cpu().numpy()


def _bound(got, ref, what):
    tol = 1e-9 * np.abs(ref) + 1e-11 * np.abs(ref).max()
    err = np.abs(got - ref)
    assert (err <= tol).all(), '%s: worst |d|/tol = %.3g' % (what, (err / tol).max())


def _overlaps(N):
    return sorted({0, N // 2, N - 1, N // 2 - 3 if (N // 2) % 2 == 0 else N // 2})


@pytest.mark.parametrize('N', [16, 256, 1000, 4096, 6000, 16384])
def test_against_the_oracle_on_the_grid(eng, N):
    rng = np.random.default_rng(N)
    fs = 200.0
    for D in _overlaps(N):
        S = N - D
        for n in (N, N + S - 1):
            x = rng.standard_normal((3, n)) * np.array([[0.3], [2.0], [1e-3]]) + np.array([[5.0], [-9.8], [0.0]])
            for window in (wn.hann(N), rng.uniform(0.2, 1.0, N)):
                psd, freq = _welch(eng, fs, x, N, D, window)
                for s in range(3):
                    f, p = wn.welch(x[s], fs, N, D, window)
                    assert np.array_equal(freq, f)
                    _bound(psd[s], p, 'N=%d D=%d n=%d series %d' % (N, D, n, s))


@pytest.mark.parametrize('N, n', [(256, 300000), (6000, 300000), (1000, 250001)])
def test_several_chunks_per_series(eng, N, n):
    """Series long enough that their segments are split over several CTAs (radix-2 and Bluestein forms)."""
    x = np.random.default_rng(n + N).standard_normal((2, n)) + 1.0
    psd, _ = _welch(eng, 100.0, x, N, N // 2, wn.hann(N))
    for s in range(2):
        _bound(psd[s], wn.welch(x[s], 100.0, N)[1], 'N=%d n=%d' % (N, n))


def test_config4_length_channel(eng):
    """One accelerometer z channel at config-4 length (14.4 M samples @400 Hz), K1's own draw, N = 16384."""
    from gnss_ins_sim_b200 import imu_model
    n, fs, N = 14400000, 400.0, 16384
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    ref_gyro = eng.to_device(np.zeros((n, 3)))
    ref_accel = eng.to_device(np.tile([0.0, 0.0, -9.8], (n, 1)))
    gyro, accel = eng.imu_noise(fs, 1, ref_gyro, ref_accel, imu.gyro_err, imu.accel_err, 5,
                                layout=eng.LAYOUT_CHANNEL_MAJOR)
    z = accel[0, 2:3].contiguous()
    psd, freq = eng.welch(fs, z, n, 1, N, N // 2, wn.hann(N))
    psd, freq, z = psd.cpu().numpy()[0], freq.cpu().numpy(), z.cpu().numpy()[0]
    del gyro, accel, ref_gyro, ref_accel
    f, p = wn.welch(z, fs, N)
    assert np.array_equal(freq, f)
    _bound(psd, p, 'config-4 accel z')


def test_same_bits_whatever_the_batch_and_layout(eng):
    n, fs = 5000, 50.0
    rng = np.random.default_rng(7)
    for N in (256, 1000, 4096):
        mine = rng.standard_normal((3, n)) * 0.2 + 1.0
        others = rng.standard_normal((999, n))
        alone = np.concatenate([_welch(eng, fs, mine[s:s + 1], N, N // 2, wn.hann(N))[0] for s in range(3)])
        for pos in (0, 1, 517, 996):
            x = np.concatenate([others[:pos], mine, others[pos:997]])
            assert x.shape[0] == 1000
            batch, _ = _welch(eng, fs, x, N, N // 2, wn.hann(N))
            assert np.array_equal(batch[pos:pos + 3], alone), (N, pos)
        # the interleaved (n, 3) layout of one run reads the same samples
        tri = eng.to_device(np.ascontiguousarray(mine.T[None]))
        p, _ = eng.welch(fs, tri, n, 3, N, N // 2, wn.hann(N), inner=3, outer_stride=3 * n, sample_stride=3)
        assert np.array_equal(p.cpu().numpy(), alone), N


def test_non_finite_and_zero_series(eng):
    N, D, n = 256, 128, 1000
    rng = np.random.default_rng(9)
    K, S = wn.segments(n, N, D)
    tail = S * (K - 1) + N
    base = rng.standard_normal(n)
    rows = [base]
    for bad in (np.nan, np.inf, -np.inf):
        for i in (0, 300, tail - 1):
            y = base.copy()
            y[i] = bad
            rows.append(y)
        y = base.copy()
        y[tail:] = bad
        rows.append(y)
    rows.append(np.zeros(n))
    psd, _ = _welch(eng, 10.0, np.stack(rows), N, D, wn.hann(N))
    for b in range(3):
        for j in range(3):
            assert np.all(np.isnan(psd[1 + 4 * b + j]))
        assert np.array_equal(psd[4 + 4 * b], psd[0])      # the unused tail is never read
    assert np.all(psd[-1] == 0.0)
    with pytest.raises(ValueError):
        _welch(eng, 10.0, np.zeros((1, 255)), 256, 128, wn.hann(256))
    for N in (255, 8194, 32768, 8):
        with pytest.raises(ValueError):
            _welch(eng, 10.0, np.zeros((1, 40000)), N, N // 2, np.ones(N))


def _zero_imu():
    from gnss_ins_sim_b200 import imu_model
    z = np.zeros(3)
    return imu_model.IMU(accuracy={'gyro_b': z, 'gyro_b_stability': z, 'gyro_arw': z,
                                   'accel_b': z, 'accel_b_stability': z, 'accel_vrw': z}, axis=6, gps=False)


def _static(n):
    z = np.zeros((n, 3))
    return {'ref_pos': z, 'ref_vel': z, 'ref_att': z, 'ref_accel': np.tile([0.0, 0.0, -9.8], (n, 1)),
            'ref_gyro': z}


def _sim_out(sim, R, algo='algo0'):
    a, g, f = sim.get_data(['psd_accel', 'psd_gyro', 'algo_freq'])
    key = '%s_%%d' % algo
    return np.stack([a[key % r] for r in range(R)]), np.stack([g[key % r] for r in range(R)]), f[key % 0]


@pytest.mark.parametrize('n', [4096, 6000])
def test_k5_vibration_inverted_exactly(eng, n):
    """A PSD environment on a noise-free IMU: one boxcar segment of the whole (period-n) series returns the
    interpolated table at every interior bin (radix-2 and Bluestein forms of K5 and K11)."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.psd_analysis import Psd
    fs, R = 100.0, 3
    tf = np.linspace(0.0, fs / 2, 7)
    tab = np.array([[1e-4, 3e-3, 5e-4, 2e-3, 1e-5, 4e-4, 1e-4], [2e-4] * 7, [5e-5, 1e-3, 1e-3, 1e-4, 1e-4, 2e-3, 2e-3]])
    env = np.column_stack([tf, tab.T])
    sim = Sim([fs, 0.0, 0.0], _static(n), ref_frame=1, imu=_zero_imu(), env={'acc': env},
              algorithm=Psd(nperseg=n, window=np.ones(n)), seed=4)
    sim.run(R)
    pa, _, freq = _sim_out(sim, R)
    for c in range(3):
        want = np.interp(freq, tf, tab[c])[1:-1]
        got = pa[:, 1:-1, c]
        assert (np.abs(got / want - 1) <= 1e-9).all(), np.abs(got / want - 1).max()


def test_sinusoidal_environment_power(eng):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.psd_analysis import Psd
    fs, N, k0, A, n = 400.0, 1024, 100, 0.7, 40 * 1024
    f0 = k0 * fs / N
    sim = Sim([fs, 0.0, 0.0], _static(n), ref_frame=1, imu=_zero_imu(),
              env={'acc': '[%r %r %r]-%rHz-sinusoidal' % (A, A / 2, A / 4, f0)}, algorithm=Psd(nperseg=N), seed=4)
    sim.run(2)
    pa, _, freq = _sim_out(sim, 2)
    assert abs(freq[k0] - f0) <= 1e-12 * f0
    for c, amp in enumerate((A, A / 2, A / 4)):
        power = pa[:, k0 - 1:k0 + 2, c].sum(axis=1) * fs / N
        assert (np.abs(power / (amp * amp / 2) - 1) <= 1e-9).all(), power


def test_white_noise_law_through_sim(eng):
    """An IMU with only ARW and VRW: the mean over runs and interior bins is 2 arw^2 (2 vrw^2) within 5 standard
    errors of the per-run spread."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.psd_analysis import Psd
    from gnss_ins_sim_b200 import imu_model
    n, fs, R = 40000, 100.0, 64
    z = np.zeros(3)
    imu = imu_model.IMU(accuracy={'gyro_b': z, 'gyro_b_stability': z, 'gyro_arw': np.array([0.3, 0.2, 0.25]),
                                  'accel_b': z, 'accel_b_stability': z, 'accel_vrw': np.array([0.05, 0.04, 0.06])},
                        axis=6, gps=False)
    sim = Sim([fs, 0.0, 0.0], _static(n), ref_frame=1, imu=imu, algorithm=Psd(nperseg=512), seed=31)
    sim.run(R)
    pa, pg, _ = _sim_out(sim, R)
    for p, rw in ((pa, imu.accel_err['vrw']), (pg, imu.gyro_err['arw'])):
        per_run = p[:, 1:-1, :].mean(axis=1)                      # [R, 3]
        mean, se = per_run.mean(0), per_run.std(0, ddof=1) / np.sqrt(R)
        assert (np.abs(mean - 2 * rw ** 2) <= 5 * se).all(), (mean, 2 * rw ** 2, se)


def test_sim_equals_the_plugin_and_logged_and_save_data(eng, monkeypatch, tmp_path):
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.psd_analysis import Psd
    from gnss_ins_sim_b200 import imu_model
    n, fs, R, seed = 30011, 100.0, 5, 23
    imu = imu_model.IMU('low-accuracy', axis=6, gps=False)
    traj = _static(n)
    sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Psd(nperseg=1000, noverlap=300), seed=seed)
    sim.run(R)
    pa, pg, freq = _sim_out(sim, R)
    gyro, accel = eng.imu_noise(fs, R, eng.to_device(traj['ref_gyro']), eng.to_device(traj['ref_accel']),
                                imu.gyro_err, imu.accel_err, seed, layout=eng.LAYOUT_CHANNEL_MAJOR)
    f2, a2, g2 = Psd(nperseg=1000, noverlap=300).run_batch(fs, accel, gyro, channel_major=True)
    assert np.array_equal(freq, f2) and np.array_equal(pa, a2) and np.array_equal(pg, g2)
    assert 'algo_time' not in sim.data
    # small run blocks: the same bits
    monkeypatch.setattr(Sim, '_allan_block', lambda self, *a: 2)
    sim2 = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Psd(nperseg=1000, noverlap=300), seed=seed)
    sim2.run(R)
    b_a, b_g, _ = _sim_out(sim2, R)
    assert np.array_equal(b_a, pa) and np.array_equal(b_g, pg)
    with pytest.raises(ValueError):
        sim2.get_error_stats('psd_gyro')
    # save_data round trip of the spectra
    out = str(tmp_path / 'out')
    sim.save_data(out, names=['algo_freq', 'psd_accel', 'psd_gyro'])
    back = np.genfromtxt(os.path.join(out, 'psd_gyro-algo0_3.csv'), delimiter=',', skip_header=1)
    assert np.array_equal(back, pg[3])
    fb = np.genfromtxt(os.path.join(out, 'algo_freq-algo0_0.csv'), delimiter=',', skip_header=1)
    assert np.array_equal(fb, freq)
    with open(os.path.join(out, 'psd_accel-algo0_0.csv')) as fp:
        assert fp.readline().strip() == ('PSD_accel_x (m^2/s^4/Hz),PSD_accel_y (m^2/s^4/Hz),'
                                         'PSD_accel_z (m^2/s^4/Hz)')
    # a logged directory filters the same as its arrays
    rng = np.random.default_rng(3)
    lg = 1e-3 * rng.standard_normal((20000, 3))
    la = 0.02 * rng.standard_normal((20000, 3)) + np.array([0.0, 0.0, -9.8])
    d = write_logged_dir(str(tmp_path / 'logged'), {'fs': fs, 'gyro': lg, 'accel': la}, deg=False)
    sim3 = Sim([fs, 0.0, 0.0], d, ref_frame=0, imu=None, algorithm=Psd(nperseg=2048))
    sim3.run(1)
    la3, lg3, lf3 = _sim_out(sim3, 1)
    f4, a4, g4 = Psd(nperseg=2048).run_batch(fs, la[None], lg[None])
    assert np.array_equal(lf3, f4) and np.array_equal(la3, a4) and np.array_equal(lg3, g4)
