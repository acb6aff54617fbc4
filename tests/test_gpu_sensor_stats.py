"""Error statistics of sensor data on the device: K9 (IMU error statistics reduced inside the noise generator,
b2ins_imu_err_stats_f64) and K3p (per-run statistics of a device array, b2ins_proc_stats_f64), through
engine and Sim.get_error_stats, against the reference's golden (tests/golden/sensor_stats_90deg.npz), the
NumPy oracle and NumPy statistics of the same Sim's get_data histories.

Tolerance against the reference: the contract |x - ref| <= 1e-6 * max(|ref|, scale), and 1e-9 of the same.
Against K1's own histories: 1e-12 -- the errors are the same numbers, only the summation order differs."""
import copy
import os

import numpy as np
import pytest

import sensor_stats_np as ssn
from conftest import GOLDEN, ROOT, load_golden, assert_close
from test_cpu_mag import write_cof, golden_date
from test_cpu_sensor_stats import G, R, SEED, starts

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')
MOTION = os.path.join(GOLDEN, 'motion_def-90deg_turn.csv')
# the error models and environments of oracle/gen_golden_sensor_stats.py
ACCURACY = {
    'gyro_b': np.array([1.0, -2.0, 0.5]), 'gyro_arw': np.array([0.25, 0.25, 0.25]),
    'gyro_b_stability': np.array([3.5, 3.5, 3.5]), 'gyro_b_corr': np.array([100.0, 100.0, 100.0]),
    'accel_b': np.array([2.0e-3, 1.0e-3, -3.0e-3]), 'accel_vrw': np.array([0.03, 0.03, 0.03]),
    'accel_b_stability': np.array([4.0e-5, 4.0e-5, 4.0e-5]), 'accel_b_corr': np.array([200.0, 200.0, 200.0]),
    'mag_si': np.array([[1.02, 0.03, -0.01], [-0.02, 0.97, 0.05], [0.04, -0.06, 1.01]]),
    'mag_hi': np.array([10.0, -7.5, 3.0]), 'mag_std': np.array([0.2, 0.35, 0.5]),
}
ENV = {'vibrand_rf1': {'acc': '[0.03 0.001 0.01]-random', 'gyro': '[6 5 4]d-random'},
       'vibsin_rf0': {'acc': '[0.03 0.001 0.01]g-3Hz-sinusoidal', 'gyro': '[6 5 4]d-0.5Hz-sinusoidal'}}
MID_G = {'b': np.array([1e-5, -2e-5, 3e-6]), 'b_drift': np.full(3, 3.5 * np.pi / 180 / 3600),
         'b_corr': np.full(3, 100.0), 'arw': np.full(3, 0.25 * np.pi / 180 / 60)}
MID_A = {'b': np.array([2e-3, -1e-3, 5e-4]), 'b_drift': np.full(3, 5e-5), 'b_corr': np.full(3, 100.0),
         'vrw': np.full(3, 0.03 / 60)}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


@pytest.fixture(scope='module')
def cof(tmp_path_factory):
    return write_cof(load_golden('mag_90deg.npz'), str(tmp_path_factory.mktemp('wmm') / 'w.COF'))


def _sim(tag, cof, algorithm=None, env=None, **kw):
    """Sim of one golden case: the 90 deg turn, a 9-axis IMU with GPS at 10 Hz and the case's error model."""
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    acc = copy.deepcopy(ACCURACY)
    if tag.startswith('whitedrift'):
        del acc['gyro_b_corr'], acc['accel_b_corr']
    imu = imu_model.IMU(accuracy=acc, axis=9, gps=True, gps_opt={'stdp': G['stdp'], 'stdv': G['stdv']})
    return Sim([float(G['fs']), float(G['fs_gps']), 0.0], MOTION, ref_frame=int(G[tag + '_ref_frame']), imu=imu,
               env=env if env is not None else ENV.get(tag), algorithm=algorithm, seed=SEED, wmm_file=cof,
               wmm_date=golden_date(load_golden('mag_90deg.npz')), **kw)


def _per_run(st, k, runs):
    return np.stack([st[k][r] for r in range(runs)])


@pytest.mark.parametrize('tag', [str(c) for c in G['cases']])
def test_sim_matches_reference(eng, cof, tag):
    sim = _sim(tag, cof)
    sim.run(R)
    assert_close(sim.data['ref_gyro'], G[tag + '_ref_gyro'], 1e-12, 1e-9, 'ref_gyro')
    for name in ('gyro', 'accel', 'mag', 'gps'):
        for i, s in enumerate(starts(name)):
            for ou in (0, 1):
                st = sim.get_error_stats(name, err_stats_start=s, use_output_units=bool(ou))
                key = '%s_%s_s%d_ou%d' % (tag, name, i, ou)
                for k in ('max', 'avg', 'std'):
                    got = st[k] if s == -1 else _per_run(st, k, R)
                    assert_close(got, G['%s_%s' % (key, k)], 1e-6, 1e-6, key + ' contract')
                    assert_close(got, G['%s_%s' % (key, k)], 1e-9, 1e-6, key)
                if ou:
                    assert st['units'] == str(G[key + '_units'])


def _oracle_check(eng, R_, n, run_offset, start, rng_seed, vib_acc=None, vib_gyro=None, check_runs=None):
    rng = np.random.default_rng(rng_seed)
    ref_g, ref_a = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0 + [0, 0, -9.8]
    end, proc = eng.imu_err_stats(100.0, R_, eng.to_device(ref_g), eng.to_device(ref_a), MID_G, MID_A, 77,
                                  run_offset=run_offset, vib_gyro=vib_gyro, vib_accel=vib_acc, stats_start=start)
    end, proc = end.cpu().numpy(), proc.cpu().numpy()
    runs = np.arange(R_) if check_runs is None else np.asarray(check_runs)
    og, oa = ssn.imu(100.0, ref_g, ref_a, MID_G, MID_A, 77, runs + run_offset, vib_acc, vib_gyro)
    x = np.concatenate([oa, og], axis=2)
    ref = np.concatenate([ref_a, ref_g], axis=1)
    _, p = ssn.stats(x, ref, start)
    e = x[:, -1] - ref[-1]
    assert_close(end[runs], e, 1e-9, 1e-6, 'end_err R=%d n=%d' % (R_, n))
    for k, s in enumerate(('max', 'avg', 'std')):
        assert_close(proc[runs, k], p[s], 1e-9, 1e-6, '%s R=%d n=%d' % (s, R_, n))


@pytest.mark.parametrize('R_,n,start', [(1, 1000, 0), (33, 2000, 250), (1000, 1000, 999)])
def test_k9_matches_oracle(eng, R_, n, start):
    _oracle_check(eng, R_, n, 5, start, R_, check_runs=None if R_ <= 33 else [0, 1, 500, 999])
    _oracle_check(eng, R_, n, 5, start, R_ + 1, vib_acc={'type': 'random', 'x': 0.1, 'y': 0.2, 'z': 0.3},
                  vib_gyro={'type': 'sinusoidal', 'x': 0.01, 'y': 0.02, 'z': 0.03, 'freq': 2.0},
                  check_runs=None if R_ <= 33 else [0, 999])


def _k1_reference(eng, R_, n, start, vib_gyro=None, vib_accel=None, seed=3):
    """K9 and NumPy statistics of K1's materialised measurements for the same arguments."""
    rng = np.random.default_rng(n)
    rg = eng.to_device(rng.standard_normal((n, 3)) * 0.3)
    ra = eng.to_device(rng.standard_normal((n, 3)) * 3.0)
    end, proc = eng.imu_err_stats(100.0, R_, rg, ra, MID_G, MID_A, seed, run_offset=2, vib_gyro=vib_gyro,
                                  vib_accel=vib_accel, stats_start=start)
    gyro, accel = eng.imu_noise(100.0, R_, rg, ra, MID_G, MID_A, seed, run_offset=2, vib_gyro=vib_gyro,
                                vib_accel=vib_accel)
    e = torch.cat([accel - ra[None], gyro - rg[None]], dim=2).cpu().numpy()
    return end.cpu().numpy(), proc.cpu().numpy(), e


def _seg_len(n, runs):
    """Samples per time segment of K1 and K9 (noise_prepare, b2ins_api.cu): with fewer runs than two per SM and
    n >= 2^18 the time axis is split, in whole 896-sample tiles; otherwise one segment of n."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if runs >= 2 * sms or n < (1 << 18):
        return n
    nseg = max(1, min(-(-2 * sms // runs), n // (1 << 16)))
    return -(-(-(-n // nseg)) // 896) * 896


def test_k9_segmented_path(eng):
    """3 runs x 300 000 samples take the time-segmented path: pass 1 (a fast Gauss-Markov channel whose pass 1
    covers only the tail of a segment, slow ones, white drift), the carry chain, K9's pass 0 from every segment's
    carry, the per-segment partials and err_stats_fold_kernel.  Starts in the first segment, on a segment
    boundary, inside a later segment (earlier segments count nothing) and in the last segment.  Against NumPy
    statistics of K1's series of the same call (the same numbers: 1e-12, end points bit for bit) and against the
    serial C oracle, which knows nothing of segments."""
    import oracle_c
    n, R_, fs, seed = 300000, 3, 100.0, 3
    seg = _seg_len(n, R_)
    assert -(-n // seg) >= 3, 'not segmented: %d samples per segment' % seg
    gerr = dict(MID_G, b_corr=np.array([0.5, 100.0, np.inf]))
    aerr = dict(MID_A, b_corr=np.array([np.inf, 0.3, 200.0]))
    rng = np.random.default_rng(8)
    ref_g, ref_a = rng.standard_normal((n, 3)) * 0.3, rng.standard_normal((n, 3)) * 3.0
    rg, ra = eng.to_device(ref_g), eng.to_device(ref_a)
    gyro, accel = eng.imu_noise(fs, R_, rg, ra, gerr, aerr, seed, run_offset=2)
    e = torch.cat([accel - ra[None], gyro - rg[None]], dim=2).cpu().numpy()
    del gyro, accel
    og, oa = oracle_c.imu_noise(fs, ref_g, ref_a, gerr, aerr, seed, np.arange(2, 2 + R_))
    eo = np.concatenate([oa - ref_a[None], og - ref_g[None]], axis=2)
    stat = lambda x: (np.max(np.abs(x), 1), np.average(x, 1), np.std(x, 1))     # noqa: E731
    for start in (0, seg, 2 * seg + 123, n - 5):
        end, proc = eng.imu_err_stats(fs, R_, rg, ra, gerr, aerr, seed, run_offset=2, stats_start=start)
        end, proc = end.cpu().numpy(), proc.cpu().numpy()
        assert np.array_equal(end, e[:, -1])            # the values K1 stores, bit for bit
        assert_close(end, eo[:, -1], 1e-9, 1.0, 'end_err vs oracle')
        for k, (v, vo) in enumerate(zip(stat(e[:, start:]), stat(eo[:, start:]))):
            assert_close(proc[:, k], v, 1e-12, 1e-9, 'start %d stat %d vs K1' % (start, k))
            assert_close(proc[:, k], vo, 1e-9, 1.0, 'start %d stat %d vs oracle' % (start, k))
        end2, proc2 = eng.imu_err_stats(fs, R_, rg, ra, gerr, aerr, seed, run_offset=2, stats_start=start)
        assert np.array_equal(proc, proc2.cpu().numpy()) and np.array_equal(end, end2.cpu().numpy())


def test_k9_psd_vibration_equals_k1(eng):
    tab = np.linspace(0.0, 50.0, 60)
    v = {'type': 'psd', 'freq': tab, 'x': np.full(60, 1e-3), 'y': np.full(60, 2e-3), 'z': np.full(60, 5e-4)}
    series, N = eng.psd_series(100.0, 3000, 4, 0, v, 3, run_offset=2)
    sg, Ng = eng.psd_series(100.0, 3000, 4, 1, v, 3, run_offset=2)
    end, proc, e = _k1_reference(eng, 4, 3000, 100, vib_gyro=eng.vib_series(sg, Ng),
                                 vib_accel=eng.vib_series(series, N))
    assert np.array_equal(end, e[:, -1])
    es = e[:, 100:]
    for k, v in enumerate((np.max(np.abs(es), 1), np.average(es, 1), np.std(es, 1))):
        assert_close(proc[:, k], v, 1e-12, 1e-9, 'psd stat %d' % k)


@pytest.mark.parametrize('vib', ['none', 'random', 'sinusoidal', 'psd'])
def test_k9_end_err_is_k1_sample_bit_for_bit(eng, vib):
    """Unsegmented path: K9's end points are K1's last stored samples minus the truth, bit for bit, with every
    vibration type and a white-drift channel (b_corr = inf) next to Gauss-Markov ones."""
    R_, n = 5, 2000
    gerr = dict(MID_G, b_corr=np.array([100.0, np.inf, 50.0]))
    aerr = dict(MID_A, b_corr=np.array([np.inf, 200.0, 100.0]))
    vg = va = None
    if vib == 'random':
        va = {'type': 'random', 'x': 0.1, 'y': 0.2, 'z': 0.3}
        vg = {'type': 'random', 'x': 0.01, 'y': 0.02, 'z': 0.03}
    elif vib == 'sinusoidal':
        va = {'type': 'sinusoidal', 'x': 0.1, 'y': 0.2, 'z': 0.3, 'freq': 3.0}
        vg = {'type': 'sinusoidal', 'x': 0.01, 'y': 0.02, 'z': 0.03, 'freq': 2.0}
    elif vib == 'psd':
        tab = np.linspace(0.0, 50.0, 60)
        v = {'type': 'psd', 'freq': tab, 'x': np.full(60, 1e-3), 'y': np.full(60, 2e-3), 'z': np.full(60, 5e-4)}
        va = eng.vib_series(*eng.psd_series(100.0, n, R_, 0, v, 3, run_offset=2))
        vg = eng.vib_series(*eng.psd_series(100.0, n, R_, 1, v, 3, run_offset=2))
    rng = np.random.default_rng(11)
    rg = eng.to_device(rng.standard_normal((n, 3)) * 0.3)
    ra = eng.to_device(rng.standard_normal((n, 3)) * 3.0)
    end, _ = eng.imu_err_stats(100.0, R_, rg, ra, gerr, aerr, 3, run_offset=2, vib_gyro=vg, vib_accel=va)
    gyro, accel = eng.imu_noise(100.0, R_, rg, ra, gerr, aerr, 3, run_offset=2, vib_gyro=vg, vib_accel=va)
    e = torch.cat([accel[:, -1] - ra[-1], gyro[:, -1] - rg[-1]], dim=1).cpu().numpy()
    assert np.array_equal(end.cpu().numpy(), e)


def test_k3p_matches_numpy(eng):
    rng = np.random.default_rng(4)
    for R_, m, C, start in ((1, 1, 1, 0), (7, 1000, 3, 0), (5, 777, 6, 300), (300, 101, 8, 100)):
        x, ref = rng.standard_normal((R_, m, C)) + 3.0, rng.standard_normal((m, C))
        end, proc = eng.proc_stats(eng.to_device(x), eng.to_device(ref), start)
        st = ssn.stats(x, ref, start)[1]
        assert np.array_equal(end.cpu().numpy(), x[:, -1] - ref[-1])
        for k, s in enumerate(('max', 'avg', 'std')):
            assert_close(proc.cpu().numpy()[:, k], st[s], 1e-12, 1e-9, 'K3p %s' % s)


def test_abi_rejects_bad_arguments(eng):
    import ctypes
    from gnss_ins_sim_b200 import _lib
    lib = _lib.load()
    x = eng.to_device(np.ones((2, 10, 3)))
    out = eng.to_device(np.zeros((2, 3, 9)))
    D = lambda t: ctypes.c_void_p(t.data_ptr())                      # noqa: E731
    call = lambda runs, m, nc, xp, start, ep, pp: lib.b2ins_proc_stats_f64(runs, m, nc, xp, D(x), start, ep, pp, None)  # noqa: E731
    assert call(2, 10, 3, D(x), 0, D(out), D(out)) == _lib.OK
    for bad in ((-1, 10, 3, D(x), 0, D(out), D(out)), (2, -1, 3, D(x), 0, D(out), D(out)),
                (2, 10, 0, D(x), 0, D(out), D(out)), (2, 10, 9, D(x), 0, D(out), D(out)),
                (2, 10, 3, None, 0, D(out), D(out)), (2, 10, 3, D(x), 10, D(out), D(out)),
                (2, 10, 3, D(x), -1, D(out), D(out)), (2, 10, 3, D(x), 0, None, D(out)),
                (2, 10, 3, D(x), 0, D(out), None)):
        assert call(*bad) == _lib.ERR_ARG, bad
    ge, ae = _lib.sensor_err(MID_G, 'arw'), _lib.sensor_err(MID_A, 'vrw')
    vn = _lib.vib(None)
    ref = eng.to_device(np.zeros((10, 3)))
    k9 = lambda runs, n, start, ep, pp, r=D(ref): lib.b2ins_imu_err_stats_f64(  # noqa: E731
        100.0, runs, n, r, r, ctypes.byref(ge), ctypes.byref(ae), ctypes.byref(vn), ctypes.byref(vn), 1, 0, start,
        ep, pp, None)
    assert k9(2, 10, 0, D(out), D(out)) == _lib.OK
    assert k9(2, 10, -1, D(out), None) == _lib.OK
    for bad in ((-1, 10, 0, D(out), D(out)), (2, -1, 0, D(out), D(out)), (2, 10, 0, None, D(out)),
                (2, 10, 0, D(out), None), (2, 10, 10, D(out), D(out))):
        assert k9(*bad) == _lib.ERR_ARG, bad
    assert k9(2, 10, 0, D(out), D(out), None) == _lib.ERR_ARG
    torch.cuda.synchronize()


def _hist_stats(sim, name, runs, start_row):
    ref = sim.data['ref_' + name]
    x = np.stack([sim.get_data([name])[0][r] for r in range(runs)])
    end, proc = ssn.stats(x, ref, start_row)
    return end, proc


@pytest.mark.parametrize('rf,env', [(0, None), (1, {'acc': np.array([[0.0, 1e-4, 1e-4, 1e-4], [50.0, 1e-4, 2e-4, 3e-4]]),
                                                    'gyro': '[0.5 0.4 0.3]d-random'})])
def test_sim_equals_numpy_of_histories(eng, cof, rf, env):
    tag = 'rf%d' % rf
    sim = _sim(tag, cof, env=env, history_block=7)
    sim.run(20)
    for name in ('gyro', 'accel', 'mag', 'gps'):
        t = sim.data['gps_time'] if name == 'gps' else sim.data['time']
        for s in (-1, 0, 2.5):
            if name == 'gps' and s == 2.5:
                s = 2.55      # between GPS epochs: the first GPS row at or after it
            st = sim.get_error_stats(name, err_stats_start=s)
            end, proc = _hist_stats(sim, name, 20, ssn.first_at(t, s))
            for k in ('max', 'avg', 'std'):
                if s == -1:
                    assert_close(st[k], end[k], 1e-12, 1e-9, '%s end %s' % (name, k))
                else:
                    assert_close(_per_run(st, k, 20), proc[k], 1e-12, 1e-9, '%s %s %s' % (name, s, k))


def test_run_base_split_equals_one_sim(eng, cof):
    one = _sim('rf0', cof)
    one.run(12)
    a, b = _sim('rf0', cof), _sim('rf0', cof, run_base=5)
    a.run(5)
    b.run(7)
    for name in ('gyro', 'accel', 'mag', 'gps'):
        whole = one.get_error_stats(name, err_stats_start=0)
        pa, pb = a.get_error_stats(name, err_stats_start=0), b.get_error_stats(name, err_stats_start=0)
        for k in ('max', 'avg', 'std'):
            assert np.array_equal(_per_run(whole, k, 12), np.concatenate([_per_run(pa, k, 5), _per_run(pb, k, 7)]))


def test_launches(eng, cof, monkeypatch):
    """One K9 launch serves gyro and accel at one start, end points reuse it, nothing runs K12, and a
    repeated call launches nothing."""
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    calls = []
    for nm in ('imu_err_stats', 'imu_noise', 'mc_free_integration', 'proc_stats', 'mag_noise', 'gps_noise'):
        def wrap(*a, _real=getattr(eng, nm), _nm=nm, **k):
            calls.append(_nm)
            return _real(*a, **k)
        monkeypatch.setattr(eng, nm, wrap)
    sim = _sim('rf0', cof, algorithm=FreeIntegration(G['ini']))
    sim.run(9)
    calls.clear()
    sim.get_error_stats('gyro', 2.5)
    sim.get_error_stats('accel', 2.5)
    sim.get_error_stats('gyro', -1)
    sim.get_error_stats('accel', -1, use_output_units=True)
    assert calls == ['imu_err_stats']
    sim.get_error_stats('mag', 0)
    sim.get_error_stats('mag', -1)
    sim.get_error_stats('gps', 0)
    assert calls == ['imu_err_stats', 'mag_noise', 'proc_stats', 'gps_noise', 'proc_stats']
    calls.clear()
    for name in ('gyro', 'accel', 'mag', 'gps'):
        sim.get_error_stats(name, 0 if name in ('mag', 'gps') else 2.5)
    assert calls == []


def _worker(rank, world, port, tmp, cof):
    import sys
    import torch.distributed as td
    sys.path.insert(0, ROOT)
    torch.cuda.set_device(rank)
    td.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                          device_id=torch.device('cuda', rank))
    sim = _sim('rf0', cof)
    sim.run(13)
    out = {}
    for name in ('gyro', 'mag', 'gps'):
        for s in (-1, 0):
            st = sim.get_error_stats(name, s)
            for k in ('max', 'avg', 'std'):
                out['%s_%d_%s' % (name, s, k)] = st[k] if s == -1 else _per_run(st, k, 13)
    np.savez(os.path.join(tmp, 'r%d.npz' % rank), **out)
    td.destroy_process_group()


def test_sharded_matches_single_gpu(cof, tmp_path):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    import torch.multiprocessing as mp
    port = 29800 + (os.getpid() % 1000)
    mp.spawn(_worker, args=(2, port, str(tmp_path), cof), nprocs=2, join=True)
    sim = _sim('rf0', cof)
    sim.run(13)
    for r in range(2):
        z = np.load(os.path.join(str(tmp_path), 'r%d.npz' % r))
        for name in ('gyro', 'mag', 'gps'):
            for s in (-1, 0):
                st = sim.get_error_stats(name, s)
                for k in ('max', 'avg', 'std'):
                    one = st[k] if s == -1 else _per_run(st, k, 13)
                    assert_close(z['%s_%d_%s' % (name, s, k)], one, 1e-12, 1e-9, '%s %d %s' % (name, s, k))
