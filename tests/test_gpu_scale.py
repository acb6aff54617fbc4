"""GPU parity at BASELINE config-3 / config-4 sizes (n = 193 036 samples @200 Hz, ref_frame 0;
Allan over millions of samples): the CUDA path against the plain-C oracle (oracle/oracle.c,
itself pinned to the reference's golden vectors) on synthetic trajectories, plus
size-independent properties."""
import numpy as np
import pytest

import oracle_c
import oracle_np as onp
from conftest import assert_close

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

LOW_G = {'b': np.zeros(3), 'b_drift': np.full(3, 10.0 * np.pi / 180 / 3600),
         'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.75 * np.pi / 180 / 60)}
LOW_A = {'b': np.zeros(3), 'b_drift': np.full(3, 2.0e-4), 'b_corr': np.full(3, 100.0),
         'vrw': np.full(3, 0.05 / 60)}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def synthetic_drive(n, fs):
    """A smooth, singularity-free 'drive': gentle turns and accelerations (true IMU output
    only has to be an input series for parity; it need not come from path_gen)."""
    t = np.arange(n) / fs
    gyro = np.stack([0.01 * np.sin(0.11 * t), 0.008 * np.sin(0.07 * t + 1.0),
                     0.05 * np.sin(0.013 * t)], axis=1)
    accel = np.stack([0.3 * np.sin(0.05 * t), 0.2 * np.cos(0.03 * t),
                      -9.794 + 0.05 * np.sin(0.2 * t)], axis=1)
    ini = np.array([31.5 * np.pi / 180, 120.4 * np.pi / 180, 10.0, 5.0, 0.0, 0.0, 3.19, 0.01, -0.02])
    nav_end = np.zeros(9)
    nav_end[3:6] = ini[0:3]
    return np.ascontiguousarray(gyro), np.ascontiguousarray(accel), ini, nav_end


@pytest.mark.parametrize('lanes', [1, 8, 32])
def test_config3_length_fused_mc_vs_c_oracle(eng, lanes):
    n, fs, R, seed = 193036, 200.0, 5, 20240922
    gyro, accel, ini, nav_end = synthetic_drive(n, fs)
    nav = np.zeros((n, 9))
    nav[-1] = nav_end
    o_err, _ = oracle_c.mc_free_integration(0, fs, R, 7, gyro, accel, nav_end, LOW_G, LOW_A, seed,
                                            ini[None], threads=0)
    cfg = eng.make_mc_config(0, fs, n, R, seed, LOW_G, LOW_A, 1, 9, run_offset=7, lanes_per_run=lanes)
    res = eng.mc_free_integration(cfg, eng.to_device(gyro), eng.to_device(accel), eng.to_device(nav),
                                  eng.to_device(ini[None]))
    err = res.end_err.cpu().numpy()
    # contract: 1e-6 relative (scale 1 rad / 1 m/s; lat/lon errors are ~1e-4 rad here)
    assert_close(err[:, 0:3], o_err[:, 0:3], 1e-6, 1.0, 'att')
    assert_close(err[:, 6:9], o_err[:, 6:9], 1e-6, 1.0, 'vel')
    assert_close(err[:, 5], o_err[:, 5], 1e-6, 1.0, 'alt')
    assert_close(err[:, 3:5] * 6.4e6, o_err[:, 3:5] * 6.4e6, 1e-6, 1.0, 'lat/lon in metres')
    # and what it really achieves after 1.9e5 steps
    assert np.abs(err[:, 6:9] - o_err[:, 6:9]).max() < 1e-7
    assert np.abs((err[:, 3:5] - o_err[:, 3:5]) * 6.4e6).max() < 1e-5


def test_config3_length_fed_vs_c_oracle(eng):
    """K2 with supplied noise at n = 193 036, ref_frame 0 and 1, histories compared at strides."""
    n, fs, R = 193036, 200.0, 2
    gyro, accel, ini, _ = synthetic_drive(n, fs)
    g, a = oracle_c.imu_noise(fs, gyro, accel, LOW_G, LOW_A, 99, np.arange(R))
    for rf in (0, 1):
        o_att, o_pos, o_vel = oracle_c.free_integration(rf, fs, g, a, np.tile(ini, (R, 1)))
        att, pos, vel = eng.free_integration(rf, fs, eng.to_device(g), eng.to_device(a),
                                             eng.to_device(ini[None]), lanes_per_run=16)
        sl = slice(None, None, 997)
        assert np.abs(att.cpu().numpy()[:, sl] - o_att[:, sl]).max() < 1e-7
        assert_close(vel.cpu().numpy()[:, sl], o_vel[:, sl], 1e-6, 1.0, 'vel')
        scale = 1.0 if rf == 1 else 1.0 / 6.4e6
        assert_close(pos.cpu().numpy()[:, sl], o_pos[:, sl], 1e-6, scale, 'pos')


def test_k1_long_series_gm_carry(eng):
    """The Gauss-Markov carry across 750+ tiles of the time-parallel generator."""
    n, fs, R = 193036, 200.0, 3
    gyro, accel, ini, _ = synthetic_drive(n, fs)
    g, a = eng.imu_noise(fs, R, eng.to_device(gyro), eng.to_device(accel), LOW_G, LOW_A, 5, 11)
    og, oa = oracle_c.imu_noise(fs, gyro, accel, LOW_G, LOW_A, 5, np.arange(11, 11 + R))
    assert_close(g.cpu().numpy(), og, 1e-11, 1.0, 'gyro')
    assert_close(a.cpu().numpy(), oa, 1e-11, 1.0, 'accel')
    # short correlation times only: the carry pass looks at the tail of each segment (the drives
    # older than ~46 correlation times have decayed below 1e-20 of the state)
    fast_g = dict(LOW_G, b_corr=np.array([0.5, 2.0, np.inf]))
    fast_a = dict(LOW_A, b_corr=np.array([1.0, 1.0, 3.0]))
    g, a = eng.imu_noise(fs, R, eng.to_device(gyro), eng.to_device(accel), fast_g, fast_a, 3, 40)
    og, oa = oracle_c.imu_noise(fs, gyro, accel, fast_g, fast_a, 3, np.arange(40, 40 + R))
    assert_close(g.cpu().numpy(), og, 1e-11, 1.0, 'gyro, truncated carry pass')
    assert_close(a.cpu().numpy(), oa, 1e-11, 1.0, 'accel, truncated carry pass')


def test_k4_allan_millions_of_samples(eng):
    """Four decade levels, ragged length, a constant offset 10^4 times the noise."""
    rng = np.random.RandomState(4)
    n, fs = 2000003, 400.0
    x = np.empty((2, n, 3))
    for r in range(2):
        for c in range(3):
            x[r, :, c] = -9.79 + 1e-3 * rng.randn(n) + np.cumsum(1e-6 * rng.randn(n))
    avar, tau = eng.allan(fs, eng.to_device(x), n, 6, inner=3, outer_stride=3 * n, sample_stride=3)
    avar = avar.cpu().numpy().reshape(2, 3, -1)
    assert avar.shape[2] == len(onp.allan_multipliers(n, fs)) and avar.shape[2] > 40
    for r in range(2):
        for c in range(3):
            o, t = oracle_c.allan_var(x[r, :, c], fs)
            assert_close(avar[r, c], o, 1e-9, 0.0, 'avar')
    assert_close(tau.cpu().numpy(), t, 1e-15, 0.0, 'tau')


@pytest.mark.parametrize('n', [200004, 150001])
def test_k4_allan_contiguous_series_both_front_ends(eng, n):
    """Contiguous series: even n keeps every row 16-byte aligned (persistent bulk-copy front end,
    several tiles per CTA: 8 x 39 tiles on 132 SMs), odd n does not (per-thread loads)."""
    rng = np.random.RandomState(n % 1000)
    nser, fs = 8, 200.0
    x = 3.7 + 1e-2 * rng.randn(nser, n) + np.cumsum(1e-5 * rng.randn(nser, n), axis=1)
    avar, tau = eng.allan(fs, eng.to_device(x), n, nser)
    avar = avar.cpu().numpy()
    for r in range(nser):
        o, t = oracle_c.allan_var(np.ascontiguousarray(x[r]), fs)
        assert_close(avar[r], o, 1e-9, 0.0, 'avar %d' % r)
    assert_close(tau.cpu().numpy(), t, 1e-15, 0.0, 'tau')


def test_lane_group_forms_agree_at_the_wave_boundary(eng):
    """The same runs through every form of the fused kernel: 1200 runs are 150 CTAs at G = 16 (just
    over one wave: the single-warp form is launched), 75 at G = 8 and 38 at G = 4 (warp-specialised
    form), 10 at G = 1; automatic choice included.  Per-run end-point errors must agree."""
    from conftest import load_golden
    g = load_golden('traj_90deg_turn_100hz_rf1.npz')
    nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
    dev = [eng.to_device(a) for a in (g['ref_gyro'], g['ref_accel'], nav, g['ini'][None])]
    ref = None
    for lanes in (1, 16, 8, 4, 0):
        cfg = eng.make_mc_config(1, 100.0, nav.shape[0], 1200, 5, LOW_G, LOW_A, 1, 9, lanes_per_run=lanes)
        err = eng.mc_free_integration(cfg, *dev).end_err.cpu().numpy()
        if ref is None:
            ref = err
        else:
            assert_close(err, ref, 1e-9, 1e-3, 'lanes %d' % lanes)


def test_large_ensemble_properties(eng):
    """BASELINE-size ensembles without an oracle: (i) two disjoint halves of 2^16 runs have
    statistically identical error statistics, (ii) end-point std grows like the white-noise
    random walk predicts (velocity error std ~ vrw*sqrt(T) within 20 %)."""
    n, fs = 2000, 100.0
    t = np.arange(n) / fs
    gyro = np.zeros((n, 3))
    accel = np.zeros((n, 3))
    ini = np.array([0.55, 2.09, 0.0, 0.0, 0.0, 0.0, 0.3, 0.0, 0.0, 9.8])   # gravity override
    accel[:, 2] = -9.8
    nav = np.zeros((n, 9))
    nav[:, 0] = 0.3
    nav[:, 3:6] = onp.lla2ecef(ini[0:3])
    quiet_g = {'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, 100.0), 'arw': np.zeros(3)}
    acc = {'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, 100.0),
           'vrw': np.full(3, 0.05 / 60)}
    dev = [eng.to_device(a) for a in (gyro, accel, nav, ini[None])]
    st = []
    for off in (0, 65536):
        cfg = eng.make_mc_config(1, fs, n, 65536, 77, quiet_g, acc, 1, 10, run_offset=off)
        st.append(eng.error_stats(eng.mc_free_integration(cfg, *dev).end_err).cpu().numpy())
    a, b = st
    assert (np.abs(a[2, 6:9] / b[2, 6:9] - 1) < 0.03).all()
    expect = 0.05 / 60 * np.sqrt(n / fs)            # vrw * sqrt(T)
    assert (np.abs(a[2, 6:9] / expect - 1) < 0.2).all()
    assert (np.abs(a[1, 6:9]) < 5 * a[2, 6:9] / np.sqrt(65536)).all()


def test_config4_length_allan_through_sim(eng):
    """BASELINE config 4 shape: static 10 h @400 Hz (n = 14.4 M), 'low-accuracy' IMU, the Allan
    plugin through Sim (K1 noise + K4), 4 runs here instead of 256; one run/channel is checked
    against the C oracle's noise + allan_var, all channels against the white-noise law."""
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.allan_analysis import Allan
    n, fs, R, seed = 14400000, 400.0, 4, 5
    ref_gyro = np.zeros((n, 3))
    ref_accel = np.tile(np.array([4.9, 0.0, -8.487]), (n, 1))        # 30 deg pitch, static
    traj = {'ref_pos': np.zeros((n, 3)), 'ref_vel': np.zeros((n, 3)), 'ref_att': np.zeros((n, 3)),
            'ref_accel': ref_accel, 'ref_gyro': ref_gyro}
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    sim = Sim([fs, 0.0, 0.0], traj, ref_frame=1, imu=imu, algorithm=Allan(), seed=seed)
    sim.run(R)
    tau, ada, adg = sim.get_data(['algo_time', 'ad_accel', 'ad_gyro'])
    t = tau['algo0_0']
    assert t.shape == (55,) and abs(t[-1] - 2500.0) < 1e-9 and ada['algo0_3'].shape == (55, 3)
    # run 2, gyro z and accel x against the oracle (noise from oracle.c, Allan from oracle.c)
    og, oa = oracle_c.imu_noise(fs, ref_gyro, ref_accel, LOW_G, LOW_A, seed, [2])
    av, ot = oracle_c.allan_var(np.ascontiguousarray(og[0, :, 2]), fs)
    assert_close(adg['algo0_2'][:, 2], np.sqrt(av), 1e-8, 0.0, 'ad_gyro z')
    av, _ = oracle_c.allan_var(np.ascontiguousarray(oa[0, :, 0]), fs)
    assert_close(ada['algo0_2'][:, 0], np.sqrt(av), 1e-8, 0.0, 'ad_accel x')
    assert_close(t, ot, 1e-12, 0.0, 'tau')
    # ... and against the unmodified reference's allan_var on the same series (oracle/gen_golden.py:
    # gen_allan_config4; same seed, run and IMU as here)
    from conftest import load_golden
    ref = load_golden('allan_config4_full_length.npz')
    assert int(ref['n']) == n and int(ref['seed']) == seed and int(ref['run']) == 2
    assert_close(t, ref['tau'], 1e-12, 0.0, 'tau (reference)')
    assert_close(adg['algo0_2'][:, 2], np.sqrt(ref['avar_gyro_z']), 1e-8, 0.0, 'ad_gyro z (reference)')
    # (accel x rides on a 4.9 m/s^2 offset: summation order shows at 1e-8 of the variance)
    assert_close(ada['algo0_2'][:, 0], np.sqrt(ref['avar_accel_x']), 1e-6, 0.0, 'ad_accel x (reference)')
    # white-noise regime (tau << bias correlation time): AD(tau) = arw / sqrt(tau)
    arw = LOW_G['arw'][0]
    k = np.where((t >= 0.01) & (t <= 1.0))[0]
    for r in range(R):
        ratio = adg['algo0_%d' % r][k, :] / (arw / np.sqrt(t[k]))[:, None]
        assert (np.abs(ratio - 1) < 0.05).all()


def test_config3_true_long_drive_through_sim(eng):
    """BASELINE config 3 end to end on its true trajectory: motion_def-long_drive.csv @200 Hz
    (193 036 samples from the host path generator), 'low-accuracy' IMU, ref_frame 0, through Sim;
    a handful of runs against the C oracle."""
    import os
    from conftest import ROOT
    from gnss_ins_sim_b200 import imu_model, pathgen
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    csv = os.path.join(ROOT, 'tests', 'golden', 'motion_def-long_drive.csv')
    ini, _ = pathgen.parse_motion(csv)
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    sim = Sim([200.0, 0.0, 0.0], csv, ref_frame=0, imu=imu, algorithm=FreeIntegration(ini), seed=11)
    R = 5
    sim.run(R)
    t = sim._traj
    assert t['ref_gyro'].shape == (193036, 3)
    nav_end = np.concatenate([t['ref_att'][-1], t['ref_pos'][-1], t['ref_vel'][-1]])
    o_err, _ = oracle_c.mc_free_integration(0, 200.0, R, 0, t['ref_gyro'], t['ref_accel'], nav_end,
                                            imu.gyro_err, imu.accel_err, 11, ini[None], threads=0)
    err = sim.end_point_errors()
    assert_close(err[:, 0:3], o_err[:, 0:3], 1e-6, 1.0, 'att')
    assert_close(err[:, 6:9], o_err[:, 6:9], 1e-6, 1.0, 'vel')
    assert_close(err[:, 3:5] * 6.4e6, o_err[:, 3:5] * 6.4e6, 1e-6, 1.0, 'lat/lon [m]')
    assert_close(err[:, 5], o_err[:, 5], 1e-6, 1.0, 'alt')
    st = sim.get_error_stats('pos', -1, extra_opt='ned')
    assert st['units'] == "['m', 'm', 'm']" and np.isfinite(st['std']).all()


def test_k1_time_segmented_path(eng):
    """Few runs + long series: K1 splits the time axis into segments (two-pass Gauss-Markov
    carry).  Same numbers as the serial oracle, including across segment boundaries."""
    n, fs, R = 700001, 100.0, 2
    gyro, accel, ini, _ = synthetic_drive(n, fs)
    fast_g = dict(LOW_G, b_corr=np.array([0.5, 100.0, np.inf]))     # fast, slow and white drift
    g, a = eng.imu_noise(fs, R, eng.to_device(gyro), eng.to_device(accel), fast_g, LOW_A, 3, 40)
    og, oa = oracle_c.imu_noise(fs, gyro, accel, fast_g, LOW_A, 3, np.arange(40, 40 + R))
    assert_close(g.cpu().numpy(), og, 1e-11, 1.0, 'gyro')
    assert_close(a.cpu().numpy(), oa, 1e-11, 1.0, 'accel')


def test_config3_full_length_against_the_reference(eng):
    """BASELINE config 3 at its full length against the UNMODIFIED REFERENCE: motion_def-long_drive.csv
    @200 Hz (193 036 samples), 'low-accuracy' IMU, ref_frame 0 through Sim -- end points and the histories
    at every 2000th sample against what the reference reached with the same injected normals
    (philox_config3_long_drive_rf0.npz, oracle/gen_golden.py: gen_philox_config3)."""
    import os
    from conftest import ROOT, load_golden, wrap_pi
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('philox_config3_long_drive_rf0.npz')
    csv = os.path.join(ROOT, 'tests', 'golden', 'motion_def-long_drive.csv')
    imu = imu_model.IMU(accuracy='low-accuracy', axis=6, gps=False)
    R, stride = len(g['run_ids']), int(g['stride'])
    sim = Sim([float(g['fs']), 0.0, 0.0], csv, ref_frame=0, imu=imu, algorithm=FreeIntegration(g['ini']),
              seed=int(g['seed']))
    sim.run(R)
    assert sim._traj['ref_gyro'].shape[0] == int(g['n'])
    want = g['end_state'] - g['ref_end'][None]
    want[:, 0:3] = wrap_pi(want[:, 0:3])
    err = sim.end_point_errors()
    # contract 1e-6 relative (the end points are ~1e3 m and ~30 m/s off the truth after 965 s)
    assert np.abs(wrap_pi(err[:, 0:3] - want[:, 0:3])).max() < 1e-9
    assert np.abs(err[:, 6:9] - want[:, 6:9]).max() < 1e-5
    assert np.abs((err[:, 3:5] - want[:, 3:5]) * 6.4e6).max() < 1e-3 and np.abs(err[:, 5] - want[:, 5]).max() < 1e-3
    h = sim.histories(stride=stride)
    att, pos, vel = (np.asarray(h[k]) for k in ('att_euler', 'pos', 'vel'))       # [R, rows, 3] host arrays
    m = g['att'].shape[1]
    assert np.abs(wrap_pi(att[:, :m] - g['att'])).max() < 1e-9
    assert np.abs(vel[:, :m] - g['vel']).max() < 1e-5
    assert np.abs((pos[:, :m, 0:2] - g['pos'][:, :, 0:2]) * 6.4e6).max() < 1e-3
    assert np.abs(pos[:, :m, 2] - g['pos'][:, :, 2]).max() < 1e-3
