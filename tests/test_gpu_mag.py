"""K8, the magnetometer measurement generator (b2ins_mag_noise_f64, engine.mag_noise), and the 9-axis IMU
through Sim, against the reference's golden (tests/golden/mag_90deg.npz) and the NumPy oracle (mag_np).

Tolerance: the contract |x - ref| <= 1e-6 * max(|ref|, 1 uT), and 1e-9 of the same.  K8 computes the same
products as the reference's (ref_mag + hi) si^T + std z, in FP64 with the device's own rounding (FMA
contraction, Box-Muller with the device's log / sincos), so agreement near 1e-14 uT is expected."""
import ctypes
import os

import numpy as np
import pytest

import mag_np
from conftest import GOLDEN, load_golden, assert_close
from test_cpu_mag import write_cof, golden_date, mag_err

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')
MOTION = os.path.join(GOLDEN, 'motion_def-90deg_turn.csv')


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _imu(g, axis=9):
    from gnss_ins_sim_b200 import imu_model
    acc = {'gyro_b': np.zeros(3), 'gyro_arw': np.full(3, 0.25), 'gyro_b_stability': np.full(3, 3.5),
           'gyro_b_corr': np.full(3, 100.0), 'accel_b': np.zeros(3), 'accel_vrw': np.full(3, 0.03),
           'accel_b_stability': np.full(3, 4e-5), 'accel_b_corr': np.full(3, 200.0),
           'mag_si': g['mag_si'], 'mag_hi': g['mag_hi'], 'mag_std': g['mag_std']}
    return imu_model.IMU(accuracy=acc, axis=axis, gps=False)


@pytest.mark.parametrize('rf', [0, 1])
def test_k8_matches_reference_and_oracle(eng, rf):
    g = load_golden('mag_90deg.npz')
    ref, want = g['ref_mag_rf%d' % rf], g['mag_rf%d' % rf]
    R, n, _ = want.shape
    out = eng.mag_noise(R, eng.to_device(ref), mag_err(g), int(g['seed'])).cpu().numpy()
    assert_close(out, want, 1e-6, 1.0, 'mag (contract)')
    assert_close(out, want, 1e-9, 1.0, 'mag')
    # the normals themselves: (out - si (ref + hi)) / std against the oracle's
    mean = (ref + g['mag_hi']).dot(g['mag_si'].T)
    z = (out - mean[None]) / g['mag_std']
    zo = mag_np.mag_normals(n, g['run_ids'], int(g['seed']))
    assert np.abs(z - zo).max() <= 1e-13 * max(1.0, np.abs(zo).max())


@pytest.mark.parametrize('R,n', [(1, 1000), (33, 777), (1000, 101), (3, 193036)])
def test_k8_ragged_launches(eng, R, n):
    rng = np.random.default_rng(R * 7 + n)
    ref = rng.standard_normal((n, 3)) * 30.0
    err = {'si': np.eye(3) + 0.05 * rng.standard_normal((3, 3)), 'hi': rng.standard_normal(3),
           'std': np.array([0.1, 0.2, 0.3])}
    seed, off = 99, 5
    out = eng.mag_noise(R, eng.to_device(ref), err, seed, run_offset=off).cpu().numpy()
    runs = np.arange(off, off + R) if R <= 33 else np.array([off, off + R // 2, off + R - 1])
    o = mag_np.mag_gen(ref, err, mag_np.mag_normals(n, runs, seed))
    assert_close(out[runs - off], o, 1e-9, 1.0, 'ragged R=%d n=%d' % (R, n))
    assert eng.mag_noise(0, eng.to_device(ref), err, seed).shape == (0, n, 3)


def test_k8_blocking_invariance(eng):
    rng = np.random.default_rng(5)
    ref = eng.to_device(rng.standard_normal((513, 3)) * 40.0)
    err = {'si': np.eye(3), 'hi': np.zeros(3), 'std': np.ones(3)}
    whole = eng.mag_noise(12, ref, err, 7).cpu().numpy()
    part = eng.mag_noise(4, ref, err, 7, run_offset=5).cpu().numpy()
    assert np.array_equal(part, whole[5:9])


def test_k8_noise_statistics(eng):
    """4096 runs x 1000 samples: per axis, mag - si (ref + hi) has mean 0 and std `std` within 5 standard
    errors (of the mean: std / sqrt(N); of the std: std / sqrt(2N))."""
    rng = np.random.default_rng(11)
    n, R = 1000, 4096
    ref = rng.standard_normal((n, 3)) * 30.0
    err = {'si': np.array([[1.02, 0.03, -0.01], [-0.02, 0.97, 0.05], [0.04, -0.06, 1.01]]),
           'hi': np.array([10.0, -7.5, 3.0]), 'std': np.array([0.2, 0.35, 0.5])}
    out = eng.mag_noise(R, eng.to_device(ref), err, 2024)
    e = (out - torch.from_numpy((ref + err['hi']).dot(err['si'].T)).cuda()[None]).reshape(-1, 3)
    N = e.shape[0]
    mean, std = e.mean(0).cpu().numpy(), e.std(0).cpu().numpy()
    assert (np.abs(mean) <= 5 * err['std'] / np.sqrt(N)).all(), mean
    assert (np.abs(std - err['std']) <= 5 * err['std'] / np.sqrt(2 * N)).all(), std
    # the three axes are independent draws
    c = np.corrcoef(e.cpu().numpy().T)
    assert np.abs(c[np.triu_indices(3, 1)]).max() <= 5 / np.sqrt(N)


def test_k8_argument_errors(eng):
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    ref = eng.to_device(np.ones((10, 3)))
    out = torch.empty((2, 10, 3), dtype=torch.float64, device='cuda')
    si, hi, std = np.eye(3).copy(), np.zeros(3), np.ones(3)
    P = lambda a: _lib.host_ptr(a)                                   # noqa: E731
    D = lambda t: ctypes.c_void_p(t.data_ptr())                      # noqa: E731
    call = lambda runs, n, r, o, s_i, h_i, s_d: lib.b2ins_mag_noise_f64(runs, n, r, s_i, h_i, s_d, 1, 0, o, None)  # noqa: E731
    assert call(2, 10, D(ref), D(out), P(si), P(hi), P(std)) == _lib.OK
    assert call(-1, 10, D(ref), D(out), P(si), P(hi), P(std)) == _lib.ERR_ARG
    assert call(2, -1, D(ref), D(out), P(si), P(hi), P(std)) == _lib.ERR_ARG
    assert call(2, 10, None, D(out), P(si), P(hi), P(std)) == _lib.ERR_ARG
    assert call(2, 10, D(ref), None, P(si), P(hi), P(std)) == _lib.ERR_ARG
    assert call(2, 10, D(ref), D(out), None, P(hi), P(std)) == _lib.ERR_ARG
    assert call(2, 10, D(ref), D(out), P(si), None, P(std)) == _lib.ERR_ARG
    assert call(2, 10, D(ref), D(out), P(si), P(hi), None) == _lib.ERR_ARG
    for bad in (-1.0, np.nan, np.inf):
        assert call(2, 10, D(ref), D(out), P(si), P(hi), P(np.array([1.0, bad, 1.0]))) == _lib.ERR_ARG
    torch.cuda.synchronize()


def _sim(g, cof, rf, algorithm=None, axis=9, **kw):
    from gnss_ins_sim_b200.sim import Sim
    return Sim([100.0, 0.0, 0.0], MOTION, ref_frame=rf, imu=_imu(g, axis), algorithm=algorithm,
               seed=int(g['seed']), wmm_file=cof, wmm_date=golden_date(g), **kw)


@pytest.mark.parametrize('rf', [0, 1])
def test_sim_nine_axis_matches_reference(eng, rf, tmp_path):
    g = load_golden('mag_90deg.npz')
    cof = write_cof(g, str(tmp_path / 'w.COF'))
    R = len(g['run_ids'])
    sim = _sim(g, cof, rf)
    sim.run(R)
    ref_mag, mag = sim.get_data(['ref_mag', 'mag'])
    assert np.array_equal(ref_mag, g['ref_mag_rf%d' % rf])
    assert sorted(mag.keys()) == list(range(R))
    for r in range(R):
        assert_close(mag[r], g['mag_rf%d' % rf][r], 1e-9, 1.0, 'Sim mag run %d' % r)
    # blocking: history_block 7 and 32 give the same runs bit for bit
    a, b = _sim(g, cof, rf, history_block=7), _sim(g, cof, rf, history_block=32)
    a.run(12)
    b.run(12)
    for r in range(12):
        assert np.array_equal(a.get_data(['mag'])[0][r], b.get_data(['mag'])[0][r])
    # save_data -> a logged-data directory reads back the same values
    d = str(tmp_path / 'saved')
    sim.save_data(d, names=['time', 'ref_mag', 'mag'])
    from gnss_ins_sim_b200.sim import Sim
    back = Sim([100.0, 0.0, 0.0], d, ref_frame=rf)
    back.run(R)
    rb, mb = back.get_data(['ref_mag', 'mag'])
    assert_close(rb, ref_mag, 1e-15, 1.0, 'ref_mag read back')
    for r in range(R):
        assert_close(mb[r], mag[r], 1e-15, 1.0, 'mag read back')


@pytest.mark.parametrize('rf', [0, 1])
def test_nine_axis_leaves_other_outputs_unchanged(eng, rf, tmp_path):
    """The magnetometer draws are separate: free integration with IMU(axis=9) equals axis=6 exactly."""
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    g = load_golden('mag_90deg.npz')
    cof = write_cof(g, str(tmp_path / 'w.COF'))
    out = []
    for axis in (9, 6):
        sim = _sim(g, cof, rf, algorithm=FreeIntegration(g['ini']), axis=axis)
        sim.run(40)
        st = [sim.get_error_stats(k) for k in ('att_euler', 'pos', 'vel')]
        proc = sim.get_error_stats('vel', err_stats_start=2.0)
        hist = sim.get_data(['pos'])[0]['algo0_3']
        out.append((sim.end_point_errors(), st, proc, hist, sim.get_data(['accel'])[0][5]))
    assert np.array_equal(out[0][0], out[1][0])
    for s9, s6 in zip(out[0][1], out[1][1]):
        for k in ('max', 'avg', 'std'):
            assert np.array_equal(s9[k], s6[k])
    for k in ('max', 'avg', 'std'):
        for key in out[0][2][k]:
            assert np.array_equal(out[0][2][k][key], out[1][2][k][key])
    assert np.array_equal(out[0][3], out[1][3]) and np.array_equal(out[0][4], out[1][4])


class _MagPlugin:
    """A reference-style plugin that takes the magnetometer (the mag_calibrate case)."""
    input = ['fs', 'mag']
    output = ['algo_time']

    def __init__(self):
        self.seen = []

    def reset(self):
        pass

    def run(self, set_of_input):
        self.seen.append(set_of_input[1])
        self.n = set_of_input[1].shape[0]

    def get_results(self):
        return [np.arange(self.n) / 100.0]


def test_plugin_receives_the_mag_get_data_returns(eng, tmp_path):
    g = load_golden('mag_90deg.npz')
    cof = write_cof(g, str(tmp_path / 'w.COF'))
    plug = _MagPlugin()
    sim = _sim(g, cof, 0, algorithm=plug, history_block=3)
    sim.run(5)
    mag = sim.get_data(['mag'])[0]
    assert len(plug.seen) == 5
    for r in range(5):
        assert np.array_equal(plug.seen[r], mag[r])
    assert_close(np.stack([mag[r] for r in range(4)]), g['mag_rf0'], 1e-9, 1.0, 'plugin mag')
