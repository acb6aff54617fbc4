"""K10, the magnetometer calibration (b2ins_magcal_f64 / b2ins_magcal_fed_f64, engine.mag_calibrate[_mc]), and
MagCal through Sim, against the reference's golden (tests/golden/magcal.npz) and the NumPy oracle (magcal_np).

Tolerances: the contract |x - ref| <= 1e-6 * max(|ref|, scale) and 1e-9 of the same, hard iron on the scale
of the field it estimates (as in test_cpu_magcal).  K10 computes calibrate_moments's formulation with its own
order of additions."""
import ctypes

import numpy as np
import pytest

import magcal_np as mc
from conftest import GOLDEN, load_golden, assert_close
from test_cpu_magcal import radius_cancellation, golden_inputs, MAG_CAL_STRIDE, REF_MAG_STRIDE
from test_cpu_mag import write_cof, golden_date

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')
MOTION = GOLDEN + '/motion_def-mag_cal.csv'


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _golden():
    """The golden with its Sim inputs rebuilt: ref_mag, ref_gyro [n, 3] and mag [R, n, 3]."""
    g = load_golden('magcal.npz')
    g['ref_mag'], g['ref_gyro'], g['mag'] = golden_inputs(g)
    return g


def _synthetic(g, i):
    return mc.golden_synthetic(g, i)


def _err(g, std=None):
    return {'si': g['mag_si'], 'hi': g['mag_hi'], 'std': g['mag_std'] if std is None else std}


def _sim(g, tmp_path, algorithm, std=None, **kw):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    acc = {'gyro_b': np.zeros(3), 'gyro_arw': np.full(3, 0.25), 'gyro_b_stability': np.full(3, 3.5),
           'gyro_b_corr': np.full(3, 100.0), 'accel_b': np.zeros(3), 'accel_vrw': np.full(3, 0.03),
           'accel_b_stability': np.full(3, 4e-5), 'accel_b_corr': np.full(3, 200.0),
           'mag_si': g['mag_si'], 'mag_hi': g['mag_hi'], 'mag_std': g['mag_std'] if std is None else std}
    cof = write_cof(load_golden('mag_90deg.npz'), str(tmp_path / 'w.COF'))
    return Sim([100.0, 0.0, 0.0], MOTION, ref_frame=1, imu=imu_model.IMU(accuracy=acc, axis=9, gps=False),
               algorithm=algorithm, seed=int(g['seed']), wmm_file=cof, wmm_date=golden_date(g), **kw)


def _magcal(g):
    from gnss_ins_sim_b200.mag_calibrate import MagCal
    return MagCal(segments=tuple(map(tuple, g['segments'])))


def _check(S, h, si, hi, rel, what):
    assert_close(S, si, rel, 1.0, what + ' soft_iron')
    assert_close(h[..., 0:3], hi[..., 0:3], rel, abs(hi.reshape(-1)[3]), what + ' hard_iron')
    assert_close(h[..., 3], hi[..., 3], rel * radius_cancellation(hi.reshape(-1)), 1.0, what + ' radius')


def test_sim_matches_reference(eng, tmp_path):
    g = _golden()
    R = len(g['run_ids'])
    sim = _sim(g, tmp_path, _magcal(g))
    sim.run(R)
    assert_close(sim.get_data(['ref_mag'])[0][::REF_MAG_STRIDE], g['ref_mag_rows'], 1e-12, 1.0, 'ref_mag')
    si, hi, cal, mag = sim.get_data(['soft_iron', 'hard_iron', 'mag_cal', 'mag'])
    assert sorted(si.keys()) == ['algo0_%d' % r for r in range(R)]
    for r in range(R):
        k = 'algo0_%d' % r
        assert si[k].shape == (3, 3) and hi[k].shape == (1, 4) and cal[k].shape == (sum(b - a for a, b in g['segments']), 3)
        for rel in (1e-6, 1e-9):
            _check(si[k], hi[k], g['soft_iron'][r], g['hard_iron'][r], rel, 'run %d' % r)
            assert_close(cal[k][::MAG_CAL_STRIDE], g['mag_cal_rows'][r], rel, 1.0, 'mag_cal run %d' % r)
        # mag_cal is exactly what the fed form makes of get_data(['mag'])
        res = eng.mag_calibrate(g['segments'], eng.to_device(mag[r][None]), want_cal=True)
        assert np.array_equal(res.mag_cal.cpu().numpy()[0], cal[k])
    sim.results()
    assert 'statistics for soft_iron' in sim.sum and 'statistics for hard_iron' in sim.sum


def test_fed_matches_oracle_on_synthetic_cases(eng):
    g = _golden()
    for i in range(int(g['syn_count'])):
        mag, seg, kind = _synthetic(g, i)
        res = eng.mag_calibrate(seg, eng.to_device(mag[None]), want_cal=True)
        S, h = res.soft_iron.cpu().numpy()[0], res.hard_iron.cpu().numpy()[0]
        cal = res.mag_cal.cpu().numpy()[0]
        if kind == 2:
            assert np.isnan(S).all() and np.isnan(h).all() and np.isnan(cal).all(), i
            continue
        oS, oh = mc.calibrate_moments(mag, seg)
        _check(S, h, g['syn%d_soft_iron' % i], g['syn%d_hard_iron' % i], 1e-6, 'case %d (reference)' % i)
        _check(S, h, oS, oh, 1e-9, 'case %d (oracle)' % i)
        assert_close(cal, mc.apply(mag, seg, S, h), 1e-12, abs(h[3]), 'case %d mag_cal' % i)


def test_generated_equals_fed_on_k8_output(eng):
    g = _golden()
    ref = eng.to_device(g['ref_mag'])
    for off in (0, 37):
        gen = eng.mag_calibrate_mc(50, g['segments'], ref, _err(g), 123, run_offset=off)
        fed = eng.mag_calibrate(g['segments'], eng.mag_noise(50, ref, _err(g), 123, run_offset=off))
        assert torch.equal(gen.soft_iron, fed.soft_iron) and torch.equal(gen.hard_iron, fed.hard_iron)


def test_run_result_independent_of_batch_and_offset(eng):
    g = _golden()
    ref = eng.to_device(g['ref_mag'])
    whole = eng.mag_calibrate_mc(1000, g['segments'], ref, _err(g), 9)
    si, hi, err = (t.cpu().numpy() for t in (whole.soft_iron, whole.hard_iron, whole.err))
    for R, off in ((1, 0), (1, 999), (7, 3), (7, 500), (1000, 0)):
        part = eng.mag_calibrate_mc(R, g['segments'], ref, _err(g), 9, run_offset=off)
        assert np.array_equal(part.soft_iron.cpu().numpy(), si[off:off + R])
        assert np.array_equal(part.hard_iron.cpu().numpy(), hi[off:off + R])
        assert np.array_equal(part.err.cpu().numpy(), err[off:off + R])
    # the error against the model, as the oracle computes it from the outputs
    b = np.linalg.norm(g['ref_mag'][0])
    for r in (0, 511, 999):
        e = mc.calibration_error(si[r], hi[r], g['mag_si'], g['mag_hi'], b)
        assert_close(err[r], e, 1e-12, 1.0, 'err run %d' % r)


def test_degenerate_runs_give_nan_and_complete(eng):
    g = _golden()
    idx = [i for i in range(int(g['syn_count'])) if int(g['syn%d_kind' % i]) == 2]
    good = _synthetic(g, idx[0])[0].copy()
    good[:, 0] += 10.0
    good += 0.3 * np.random.default_rng(1).standard_normal(good.shape)
    batch = np.stack([_synthetic(g, i)[0] for i in idx] + [good])
    res = eng.mag_calibrate(g['syn%d_seg' % idx[0]], eng.to_device(batch), want_cal=True)
    torch.cuda.synchronize()
    S, h = res.soft_iron.cpu().numpy(), res.hard_iron.cpu().numpy()
    assert np.isnan(S[:-1]).all() and np.isnan(h[:-1]).all()
    assert np.isfinite(S[-1]).all() and np.isfinite(h[-1]).all()


def test_plugin_run_equals_run_batch(eng):
    g = _golden()
    a = _magcal(g)
    a.reset()
    a.run([g['mag'][1]])
    si, hi, cal = a.get_results()
    bs, bh, bc = a.run_batch(g['mag'][1:2])
    assert si.shape == (3, 3) and hi.shape == (1, 4)
    assert np.array_equal(si, bs[0]) and np.array_equal(hi[0], bh[0]) and np.array_equal(cal, bc[0])


def test_saved_directory_calibrates_like_the_generated_runs(eng, tmp_path):
    from gnss_ins_sim_b200.sim import Sim
    g = _golden()
    sim = _sim(g, tmp_path, _magcal(g))
    sim.run(4)
    d = str(tmp_path / 'saved')
    sim.save_data(d, names=['time', 'ref_mag', 'mag'])
    back = Sim([100.0, 0.0, 0.0], d, ref_frame=1, algorithm=_magcal(g))
    back.run(4)
    for k in ('soft_iron', 'hard_iron'):
        a, b = sim.get_data([k])[0], back.get_data([k])[0]
        for r in range(4):
            assert_close(b['algo0_%d' % r], a['algo0_%d' % r], 1e-9, 1.0, '%s run %d read back' % (k, r))
    with pytest.raises(ValueError):
        back.get_error_stats('soft_iron')


def test_error_stats_match_host_statistics(eng, tmp_path):
    g = _golden()
    sim = _sim(g, tmp_path, _magcal(g))
    sim.run(200)
    si, hi = sim.get_data(['soft_iron', 'hard_iron'])
    b = np.linalg.norm(g['ref_mag'][0])
    e = np.stack([mc.calibration_error(si['algo0_%d' % r], hi['algo0_%d' % r], g['mag_si'], g['mag_hi'], b)
                  for r in range(200)])
    for name, cols in (('soft_iron', slice(0, 9)), ('hard_iron', slice(9, 13))):
        st = sim.get_error_stats(name)
        assert st['units'] == str(['-'] * 9 if name == 'soft_iron' else ['uT'] * 4)
        for k, ref in (('max', np.abs(e[:, cols]).max(0)), ('avg', e[:, cols].mean(0)), ('std', e[:, cols].std(0))):
            assert_close(st[k], ref, 1e-9, 1e-12, '%s %s' % (name, k))
        with pytest.raises(ValueError):
            sim.get_error_stats(name, err_stats_start=1.0)


def _zero_noise_error(eng, g, runs=1):
    ref = eng.to_device(g['ref_mag'])
    return eng.mag_calibrate_mc(runs, g['segments'], ref, _err(g, np.zeros(3)), 1).err.cpu().numpy()


def test_zero_noise_error_within_sampling_bound(eng):
    """Noise-free samples of the clean rotations: the ranges come from sampled extremes, which miss the true
    ones by at most r (1 - cos(w dt / 2)), so |E| and |e_hi| / |hi| stay below (w dt)^2 / 8."""
    g = _golden()
    e = _zero_noise_error(eng, g)[0]
    w_dt = np.abs(g['ref_gyro']).max() / float(g['fs'])
    bound = w_dt * w_dt / 8.0
    assert np.abs(e[0:9]).max() < bound, (e, bound)
    assert np.abs(e[9:12]).max() / np.linalg.norm(g['mag_hi']) < bound, (e, bound)


def test_noisy_ensemble_mean_matches_oracle(eng):
    """32768 noisy runs reduced by K3: every mean calibration error agrees with the oracle's mean over 256 runs
    of the same model within 3 standard errors of the difference.  The mean is not the noise-free value: noise
    widens the sampled ranges the sensitivities come from, which biases E (about 1e-2 on its first entry here)."""
    g = _golden()
    R, Ro = 32768, 256
    ref = eng.to_device(g['ref_mag'])
    res = eng.mag_calibrate_mc(R, g['segments'], ref, _err(g), 2024)
    st = eng.error_stats(res.err).cpu().numpy()
    mag = eng.mag_noise(Ro, ref, _err(g), 2024, run_offset=R).cpu().numpy()
    b = np.linalg.norm(g['ref_mag'][0])
    eo = np.stack([mc.calibration_error(*mc.calibrate_moments(m, g['segments']), g['mag_si'], g['mag_hi'], b)
                   for m in mag])
    se = np.sqrt(st[2] ** 2 / R + eo.std(0) ** 2 / Ro)
    assert (np.abs(st[1] - eo.mean(0)) <= 3.0 * se).all(), (st[1] - eo.mean(0), se)
    e0 = _zero_noise_error(eng, g)[0]
    assert abs(st[1][0] - e0[0]) > 10.0 * st[2][0] / np.sqrt(R)       # the range bias is resolved


def test_argument_errors(eng):
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    x = torch.zeros((2, 30, 3), dtype=torch.float64, device='cuda')
    out9 = torch.empty((2, 9), dtype=torch.float64, device='cuda')
    out4 = torch.empty((2, 4), dtype=torch.float64, device='cuda')
    D = lambda t: ctypes.c_void_p(t.data_ptr())                      # noqa: E731

    def call(seg, runs=2, n=30, mag=x, sstride=3, si=out9, hi=out4):
        s = np.ascontiguousarray(seg, dtype=np.int64)
        return lib.b2ins_magcal_fed_f64(runs, n, s.ctypes.data_as(_lib.c_int64_p), None if mag is None else D(mag),
                                        3 * n, sstride, None if si is None else D(si), D(hi), None, None)
    assert call([0, 10, 10, 20, 20, 30]) == _lib.OK
    for seg in ([0, 2, 10, 20, 20, 30], [-1, 10, 10, 20, 20, 30], [0, 10, 10, 20, 20, 31], [5, 4, 10, 20, 20, 30]):
        assert call(seg) == _lib.ERR_ARG, seg
    assert call([0, 10, 10, 20, 20, 30], runs=-1) == _lib.ERR_ARG
    assert call([0, 10, 10, 20, 20, 30], mag=None) == _lib.ERR_ARG
    assert call([0, 10, 10, 20, 20, 30], si=None) == _lib.ERR_ARG
    assert call([0, 10, 10, 20, 20, 30], sstride=2) == _lib.ERR_ARG
    assert lib.b2ins_magcal_fed_f64(2, 30, None, D(x), 90, 3, D(out9), D(out4), None, None) == _lib.ERR_ARG
    torch.cuda.synchronize()
    # the host form equals the device form
    rng = np.random.default_rng(3)
    m = np.ascontiguousarray(rng.standard_normal((2, 30, 3)) * 40.0 + 5.0)
    seg = np.array([0, 10, 10, 20, 20, 30], dtype=np.int64)
    hs, hh, hc = np.empty((2, 9)), np.empty((2, 4)), np.empty((2, 30, 3))
    assert lib.b2ins_magcal_fed_f64_host(2, 30, seg.ctypes.data_as(_lib.c_int64_p), _lib.host_ptr(m), 90, 3,
                                         _lib.host_ptr(hs), _lib.host_ptr(hh), _lib.host_ptr(hc)) == _lib.OK
    res = eng.mag_calibrate(seg.reshape(3, 2), eng.to_device(m), want_cal=True)
    assert np.array_equal(hs, res.soft_iron.cpu().numpy().reshape(2, 9), equal_nan=True)
    assert np.array_equal(hh, res.hard_iron.cpu().numpy(), equal_nan=True)
    assert np.array_equal(hc, res.mag_cal.cpu().numpy(), equal_nan=True)
