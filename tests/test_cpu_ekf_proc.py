"""The spec of the loosely-coupled filter's process-error statistics (oracle/ekf_proc_np.py).

The spec's statistics are the reference's formulas applied to the filter spec's histories: wrapped attitude
errors, LLA / NED / ECEF position errors, plain velocity errors, max|e|, mean and std with ddof 0 from the
start sample; a start on the last sample reduces to the end-point error."""
import numpy as np
import pytest

from conftest import load_golden
import ekf_np
import ekf_proc_np
import oracle_np as onp

DEMO_IMU = {'gyro_b': np.zeros(3), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
            'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
            'accel_b': np.zeros(3), 'accel_vrw': np.array([0.03119, 0.03009, 0.04779]),
            'accel_b_stability': np.array([4.29e-5, 5.72e-5, 8.02e-5]),
            'accel_b_corr': np.array([200.0, 200.0, 200.0])}       # demo_ins_loose.py:28-37
FS = 100.0
N = 700
RUNS = np.arange(3, 8)


def _case():
    """The 90-degree turn in ref_frame 0, cut to N samples, with its 10 Hz GPS truth, all visible."""
    from gnss_ins_sim_b200 import imu_model
    t = load_golden('traj_90deg_turn_100hz_rf0.npz')
    g = load_golden('gps_90deg_rf0.npz')
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)[:N]
    idx = np.rint(g['gps_time'] * 100.0).astype(np.int64)
    keep = idx < N
    imu = imu_model.IMU(accuracy=DEMO_IMU, axis=6, gps=True)
    args = (FS, t['ref_gyro'][:N], t['ref_accel'][:N], nav, g['ref_gps'][keep], idx[keep],
            np.ones(int(keep.sum())), imu.gyro_err, imu.accel_err, imu.gps_err, 11, RUNS, t['ini'])
    return args, nav


@pytest.fixture(scope='module')
def spec():
    args, nav = _case()
    return args, nav, ekf_np.ins_loose(*args, want_hist=True, vel_rw=0.02)


def _by_hand(h, nav, start, frame):
    """The statistics written out: errors of rows >= start, then max|e|, mean, std (ddof 0)."""
    r = nav[start:]
    att = (h['att'][:, start:] - r[None, :, 0:3] + np.pi) % (2.0 * np.pi) - np.pi
    x = h['pos'][:, start:]
    if frame == '':
        pos = x - r[None, :, 3:6]
    else:
        d = onp.lla2ecef(x) - onp.lla2ecef(r[:, 3:6])[None]
        if frame == 'ecef':
            pos = d
        else:
            sl, cl, so, co = np.sin(r[:, 3]), np.cos(r[:, 3]), np.sin(r[:, 4]), np.cos(r[:, 4])
            pos = np.stack([-sl * co * d[..., 0] - sl * so * d[..., 1] + cl * d[..., 2],
                            -so * d[..., 0] + co * d[..., 1],
                            -cl * co * d[..., 0] - cl * so * d[..., 1] - sl * d[..., 2]], axis=-1)
    vel = h['vel'][:, start:] - r[None, :, 6:9]
    e = np.concatenate([att, pos, vel], axis=2)
    return np.stack([np.abs(e).max(1), e.mean(1), np.sqrt(((e - e.mean(1, keepdims=True)) ** 2).mean(1))], 1)


@pytest.mark.parametrize('frame', ekf_proc_np.FRAMES)
def test_spec_is_the_reference_statistics_of_the_filter_histories(spec, frame):
    args, nav, h = spec
    for start in (0, 345):
        ps = ekf_proc_np.process_stats(h['att'], h['pos'], h['vel'], nav, start, frame)
        ref = _by_hand(h, nav, start, frame)
        assert ps.shape == (RUNS.size, 3, 9)
        assert np.allclose(ps, ref, rtol=1e-9, atol=1e-12 if frame == '' else 1e-7), (frame, start)
    out = ekf_proc_np.ins_loose(*args, proc_start=345, pos_frame=frame, vel_rw=0.02)
    for k in ('end_err', 'end_bias', 'nees', 'inside3', 'att', 'pos', 'vel'):
        assert np.array_equal(out[k], h[k]), k
    assert np.array_equal(out['proc_stats'], ekf_proc_np.process_stats(h['att'], h['pos'], h['vel'], nav, 345,
                                                                      frame))


@pytest.mark.parametrize('frame', ekf_proc_np.FRAMES)
def test_start_on_the_last_sample_is_the_end_point_error(spec, frame):
    args, nav, h = spec
    ps = ekf_proc_np.process_stats(h['att'], h['pos'], h['vel'], nav, N - 1, frame)
    end = h['end_err'].copy()
    if frame:
        from proc_pos_np import lla_array_error
        end[:, 3:6] = lla_array_error(h['pos'][:, -1], nav[-1, 3:6], frame)
    assert np.all(ps[:, 2] == 0.0)
    assert np.array_equal(ps[:, 1], end)
    assert np.array_equal(ps[:, 0], np.abs(end))
