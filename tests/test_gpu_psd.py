"""K5 (csrc/psd_kernel.cuh) on every transform plan, and every consumer of its series where the series wraps.

K5 turns a PSD table into one vibration series of period N per run and axis, by the direct cosine synthesis
(N <= 14 and 8194 <= N <= 16382), a radix-2 transform (N / 2 a power of two) or Bluestein (the other N / 2 up
to 4095); b2ins_diag_psd_plan says which, and tests/test_cpu_psd.py holds the lengths below to their plans.
Every series is held to time_series_from_psd on the same Philox phases at 1e-12 of its maximum (the oracle
itself is certified against an exact synthesis at 1e-14 on the CPU); the worst error per plan is printed.

The consumers (K1, K12 in every launch shape, K7, K9, Sim) read a series of period N at t % N.  They run on a
stationary trajectory of 40001 samples (two periods of 16384 and 7233 samples more), where a series that
does not wrap gives other numbers: the same launch over the series unrolled to n samples on the host must
give identical bits, and the measurement histories must equal the oracle's noise plus its tiled series."""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, load_golden, assert_close
import oracle_np as onp

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

TOL = 1e-12
WORST = {}                    # plan -> (worst |d| / max|x| over every series checked, where)
FS = 100.0


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    yield engine
    if WORST:
        print('\nK5 vs time_series_from_psd, worst |d| / max|x| per plan:')
        for plan, (rel, what) in sorted(WORST.items()):
            print('  %-16s %.2e  (%s)' % (plan, rel, what))


def _golden_vib():
    """The golden table (8193 rows up to 100 Hz, fs = 200 Hz) on three axes."""
    g = load_golden('psd.npz')
    f, s = g['freq_a'], g['sxx_a']
    return float(g['fs_a']), {'type': 'psd', 'freq': f, 'x': s, 'y': 2.0 * s, 'z': 0.5 * s + 1e-6}


def _tile(s, n):
    """[..., N] -> [..., n]: the series read at t % N."""
    N = s.shape[-1]
    reps = np.tile(s, (1,) * (s.ndim - 1) + (n // N,))
    return np.concatenate([reps, s[..., :n % N]], axis=-1)


def _oracle(vib, fs, n, run_ids, seed, sensor):
    """time_series_from_psd of every run and axis on K5's phase normals: [R, 3, n]."""
    N = min(n + n % 2, 16384)
    z = onp.psd_phase_normals(N // 2 + 1, np.asarray(run_ids, dtype=np.uint64), seed, sensor)
    out = np.empty((len(run_ids), 3, n))
    for r in range(len(run_ids)):
        for c, key in enumerate('xyz'):
            ok, out[r, c] = onp.time_series_from_psd(vib[key], vib['freq'], fs, n, z[r, c])
            assert ok
    return out


def _check(series, ref, plan, what):
    """series [R, 3, N] (device or host) against ref [R, 3, n] at TOL of each series' maximum."""
    s = series.cpu().numpy() if hasattr(series, 'cpu') else series
    got = _tile(s, ref.shape[-1])
    scale = np.abs(ref).max(axis=-1, keepdims=True)
    d = np.abs(got - ref)
    assert np.isfinite(got).all(), what
    bad = d > TOL * scale
    with np.errstate(divide='ignore', invalid='ignore'):
        rel = np.where(scale > 0, d / scale, np.where(d > 0, np.inf, 0.0))
    if float(rel.max()) >= WORST.get(plan, (0.0, ''))[0]:
        WORST[plan] = (float(rel.max()), what)
    assert not bad.any(), '%s: %d samples off, worst %.3e of max|x| (series %s)' % (
        what, bad.sum(), rel.max(), np.unravel_index(np.argmax(rel), rel.shape)[:2])


def _plan(n):
    from gnss_ins_sim_b200 import _lib
    return _lib.psd_plan(n)[0]


# ------------------------------------------------------------------------------------------ K5 itself ----
# The worst direct-plan error is at N = 2 (~3e-13): a series of two bins whose phases sit near +-pi/2 is small
# beside its bins, and the last bit in which the device's and NumPy's phase normals may differ shows through.
LENGTHS = [1, 2, 3, 5, 14,                     # direct, N = 2 .. 14 (N = 2: L = 2, no interior bin)
           16, 32,                             # the smallest radix-2 lengths
           18, 34, 777, 1000,                  # the smallest Bluestein lengths, and P = 1024
           2050, 4098, 8186, 8190,             # Bluestein up to P = 8192 (M = 4093 prime, M = 4095)
           8192,                               # radix-2, M = 4096
           8193, 8194, 10000, 16382,           # direct, M = 4097 .. 8191 (8191 prime)
           16383, 16384, 16385, 40001]         # radix-2, N = 16384


@pytest.mark.parametrize('n', LENGTHS)
def test_k5_every_length_matches_the_oracle(eng, n):
    fs, vib = _golden_vib()
    R, seed, run0 = 3, 99, 5
    plan = _plan(n)
    for sensor in (0, 1):
        series, N = eng.psd_series(fs, n, R, sensor, vib, seed, run0)
        assert N == min(n + n % 2, 16384) and tuple(series.shape) == (R, 3, N)
        _check(series, _oracle(vib, fs, n, range(run0, run0 + R), seed, sensor), plan,
               'n=%d sensor %d (%s)' % (n, sensor, plan))


@pytest.mark.parametrize('n', [16384, 8190, 10000])
def test_k5_many_series_per_cta(eng, n):
    """300 runs = 900 series, more than two per persistent CTA of the transforms (2 x 132 CTAs): the work array
    and the Bluestein chirp transform are reused across series; every series is checked."""
    fs, vib = _golden_vib()
    R, seed, run0 = 300, 4, 11
    series, N = eng.psd_series(fs, n, R, 1, vib, seed, run0)
    _check(series, _oracle(vib, fs, n, range(run0, run0 + R), seed, 1), _plan(n), 'n=%d, %d runs' % (n, R))


def test_k5_run_ids_across_the_philox_high_word(eng):
    fs, vib = _golden_vib()
    r0 = 2 ** 32 - 2
    for n in (14, 1000, 40001):
        series, N = eng.psd_series(fs, n, 4, 0, vib, 21, r0)
        _check(series, _oracle(vib, fs, n, range(r0, r0 + 4), 21, 0), _plan(n), 'n=%d runs 2^32-2 ..' % n)


def test_k5_run_split_of_large_launches(eng):
    """16390 runs at n = 64 cross psd_series' 16384-run launch split: the rows either side of it are the
    oracle's and those of a call that starts at run 16384."""
    fs, vib = _golden_vib()
    n, seed = 64, 8
    series, N = eng.psd_series(fs, n, 16390, 1, vib, seed, 0)
    assert tuple(series.shape) == (16390, 3, N)
    rows = [0, 16383, 16384, 16389]
    s = series.cpu().numpy()
    _check(s[rows], _oracle(vib, fs, n, rows, seed, 1), _plan(n), 'rows about the launch split')
    tail, _ = eng.psd_series(fs, n, 6, 1, vib, seed, 16384)
    assert np.array_equal(tail.cpu().numpy(), s[16384:16390])


def _tables():
    f = FS / 2
    step = np.array([1e-4, 1e-4, 4e-4, 4e-4])
    return {
        'left end clamps': (np.linspace(5.0, f, 10), np.stack([np.linspace(1e-4, 1e-3, 10), np.full(10, 2e-4),
                                                               np.geomspace(1e-5, 1e-3, 10)])),
        'right end clamps': (np.linspace(0.0, 30.0, 7), np.stack([np.linspace(1e-3, 1e-4, 7), np.full(7, 3e-4),
                                                                  np.linspace(0.0, 1e-3, 7)])),
        'step at a grid frequency': (np.array([0.0, 10.0, 10.0, f]), np.stack([step, 2 * step, step[::-1]])),
        'two rows': (np.array([0.0, f]), np.array([[1e-4, 3e-4], [2e-4, 2e-4], [5e-4, 0.0]])),
        'zero bins': (np.array([0.0, 10.0, 20.0, 30.0, f]), np.array([[0.0, 0.0, 1e-4, 0.0, 0.0], np.zeros(5),
                                                                      [1e-4, 0.0, 0.0, 0.0, 1e-4]])),
    }


@pytest.mark.parametrize('n', [14, 1000, 40001])
def test_k5_tables_follow_np_interp(eng, n):
    """Tables np.interp clamps at either end, a step (a repeated breakpoint) a grid frequency lands on, two
    rows, zero bins and a table of exactly L rows (used as it is), each against the oracle; the caller's
    arrays are left as they were."""
    N = min(n + n % 2, 16384)
    L = N // 2 + 1
    grid = np.linspace(0.0, FS / 2, L)
    tabs = _tables()
    if n == 1000:
        assert 10.0 in grid                                  # the step's breakpoint is a grid frequency
    tabs['exactly L rows'] = (grid, np.stack([np.interp(grid, [0.0, 50.0], [1e-4, 5e-4]), np.full(L, 1e-4),
                                              np.where(np.arange(L) % 3 == 0, 2e-4, 0.0)]))
    for name, (f, s) in tabs.items():
        vib = {'type': 'psd', 'freq': f, 'x': s[0], 'y': s[1], 'z': s[2]}
        keep = {k: np.array(v, copy=True) for k, v in vib.items() if k != 'type'}
        series, _ = eng.psd_series(FS, n, 2, 0, vib, 13, 40)
        for k, v in keep.items():
            assert np.array_equal(vib[k], v), (name, k)
        ref = _oracle(vib, FS, n, [40, 41], 13, 0)
        _check(series, ref, _plan(n), '%s, n=%d' % (name, n))
        if name == 'zero bins':
            assert not series[:, 1].any()                    # an all-zero axis is zero
        for k, v in keep.items():
            assert np.array_equal(vib[k], v), (name, k, 'after the oracle')


_CHILD = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from gnss_ins_sim_b200 import _lib, engine
d = dict(np.load(sys.argv[2]))
vib = {'type': 'psd', 'freq': d['freq'], 'x': d['x'], 'y': d['y'], 'z': d['z']}
out = {}
for n in d['lengths']:
    assert _lib.psd_plan(int(n)) == ('direct', 0), n
    s, N = engine.psd_series(float(d['fs']), int(n), 2, 1, vib, 99, 5)
    out['n%d' % n] = s.cpu().numpy()
np.savez(sys.argv[3], **out)
'''


def test_k5_direct_synthesis_at_transform_lengths(eng, tmp_path):
    """B2INS_PSD_DIRECT (read once per process) sends every length to the direct synthesis: in a child
    process, for lengths the transforms take here, the series equal the transforms' and the oracle's."""
    fs, vib = _golden_vib()
    lengths = np.array([16, 1000, 8190, 16384])
    args = tmp_path / 'args.npz'
    np.savez(args, fs=fs, freq=vib['freq'], x=vib['x'], y=vib['y'], z=vib['z'], lengths=lengths)
    env = dict(os.environ, B2INS_PSD_DIRECT='1')
    out = subprocess.run([sys.executable, '-c', _CHILD, ROOT, str(args), str(tmp_path / 'direct.npz')],
                         env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-4000:]
    direct = np.load(tmp_path / 'direct.npz')
    for n in lengths:
        assert _plan(n) != 'direct', n
        fft, _ = eng.psd_series(fs, int(n), 2, 1, vib, 99, 5)
        d = direct['n%d' % n]
        _check(d, _tile(fft.cpu().numpy(), int(n)), 'direct (forced)', 'direct vs %s, n=%d' % (_plan(n), n))
        _check(d, _oracle(vib, fs, int(n), [5, 6], 99, 1), 'direct (forced)', 'forced direct n=%d' % n)


# ----------------------------------------------------------------------------------- consumers ----
N_WRAP, R_WRAP, R0_WRAP, SEED = 40001, 9, 1000, 7
PSD_ACC = {'type': 'psd', 'freq': np.linspace(0.0, 50.0, 26), 'x': np.full(26, 1e-3),
           'y': np.linspace(1e-3, 4e-3, 26), 'z': np.full(26, 2e-3)}
PSD_GYRO = {k: (v * 1e-4 if k in 'xyz' else v) for k, v in PSD_ACC.items()}
SHAPES = [(1, '3,1,0'), (1, '6,1,0'), (1, '0'), (2, '3,1,0'), (2, '6,1,0'), (4, '3,1,0'), (4, '3,1,1'),
          (4, '6,1,0'), (4, '6,1,1'), (4, '6,2,0'), (8, '6,1,0'), (8, '6,2,0'), (8, '1,2,0'), (16, '1,4,0'),
          (16, '1,4,1'), (32, '1,4,1'), (32, '0')]       # test_gpu_r02.SHAPES
_CACHE = {}


def _mid():
    from gnss_ins_sim_b200 import imu_model
    return imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)


def _still(rf, n=N_WRAP):
    """The first sample of the 90-degree turn held for n samples: ref_gyro, ref_accel [n, 3], nav [n, 9], ini."""
    g = load_golden('traj_90deg_turn_100hz_rf%d.npz' % rf)
    nav0 = np.concatenate([g['ref_att'][0], g['ref_pos'][0], g['ref_vel'][0]])
    return (np.tile(g['ref_gyro'][0], (n, 1)), np.tile(g['ref_accel'][0], (n, 1)), np.tile(nav0, (n, 1)),
            g['ini'])


def _vibs(eng, n, runs, r0):
    """(wrapped, unrolled) Vib pairs (accel, gyro) over K5's series of runs r0 .., and the host series."""
    out = {}
    for sensor, v in ((0, PSD_ACC), (1, PSD_GYRO)):
        s, N = eng.psd_series(FS, n, runs, sensor, v, SEED, r0)
        host = s.cpu().numpy()
        u = eng.to_device(_tile(host, n))
        out[sensor] = (eng.vib_series(s, N), eng.vib_series(u, n), host)
    return (out[0][0], out[1][0]), (out[0][1], out[1][1]), (out[0][2], out[1][2])


def _oracle_imu(rf, n=N_WRAP, runs=R_WRAP, r0=R0_WRAP):
    """oracle_np measurements of the mid-accuracy IMU with the oracle's PSD series added: gyro, accel [R, n, 3]."""
    key = (rf, n, runs, r0)
    if key not in _CACHE:
        rg, ra, _, _ = _still(rf, n)
        imu = _mid()
        ids = np.arange(r0, r0 + runs)
        og, oa = onp.imu_noise(FS, rg, ra, imu.gyro_err, imu.accel_err, SEED, ids)
        va = _oracle(PSD_ACC, FS, n, ids, SEED, 0).transpose(0, 2, 1)
        vg = _oracle(PSD_GYRO, FS, n, ids, SEED, 1).transpose(0, 2, 1)
        _CACHE[key] = (og + vg, oa + va)
    return _CACHE[key]


def test_k5_series_of_the_wrap_case(eng):
    """The series every consumer test below reads: radix-2, N = 16384, against the oracle."""
    for sensor, v in ((0, PSD_ACC), (1, PSD_GYRO)):
        s, N = eng.psd_series(FS, N_WRAP, R_WRAP, sensor, v, SEED, R0_WRAP)
        assert N == 16384 and N_WRAP == 2 * N + 7233
        _check(s, _oracle(v, FS, N_WRAP, range(R0_WRAP, R0_WRAP + R_WRAP), SEED, sensor), _plan(N_WRAP),
               'wrap case sensor %d' % sensor)


def test_k1_reads_the_series_at_t_mod_n(eng):
    rg, ra, _, _ = _still(1)
    imu = _mid()
    wrapped, unrolled, _ = _vibs(eng, N_WRAP, R_WRAP, R0_WRAP)
    og, oa = _oracle_imu(1)
    dev = eng.to_device(rg), eng.to_device(ra)
    back = {eng.LAYOUT_RUN_MAJOR: lambda t: t, eng.LAYOUT_TIME_MAJOR: lambda t: t.permute(2, 0, 1),
            eng.LAYOUT_CHANNEL_MAJOR: lambda t: t.permute(0, 2, 1)}
    for layout, to_rnc in back.items():
        out = []
        for va, vg in (wrapped, unrolled):
            g, a = eng.imu_noise(FS, R_WRAP, *dev, imu.gyro_err, imu.accel_err, SEED, R0_WRAP,
                                 vib_gyro=vg, vib_accel=va, layout=layout)
            out.append((to_rnc(g).cpu().numpy(), to_rnc(a).cpu().numpy()))
        (g, a), (gu, au) = out
        assert np.array_equal(g, gu) and np.array_equal(a, au), layout
        assert_close(g, og, TOL, 1.0, 'K1 gyro layout %d' % layout)
        assert_close(a, oa, TOL, 1.0, 'K1 accel layout %d' % layout)


def _k12(eng, rf, lanes, vib, dev, odo=None):
    imu = _mid()
    kw = {} if odo is None else {'odo_err': {'scale': 0.999, 'stdv': 0.01}, 'ref_odo': odo}
    cfg = eng.make_mc_config(rf, FS, N_WRAP, R_WRAP, SEED, imu.gyro_err, imu.accel_err, 1, 9,
                             run_offset=R0_WRAP, vib_accel=vib[0], vib_gyro=vib[1], lanes_per_run=lanes,
                             dump_runs=R_WRAP, **kw)
    res = eng.mc_free_integration(cfg, *dev, dump_imu=True)
    return (res.end_err.cpu().numpy(), res.gyro.cpu().numpy(), res.accel.cpu().numpy(),
            None if res.odo is None else res.odo.cpu().numpy())


@pytest.mark.parametrize('rf', [1, 0])
def test_k12_every_shape_reads_the_series_at_t_mod_n(eng, rf, monkeypatch):
    """Every launch shape of the fused Monte-Carlo kernel: histories against the oracle, the wrapped series
    against the unrolled one bit for bit, and the end-point errors of all shapes within 1e-10 (positions in
    ref_frame 1: within the resolution of the ECEF coordinates they are differences of)."""
    rg, ra, nav, ini = _still(rf)
    dev = [eng.to_device(a) for a in (rg, ra, nav, ini[None])]
    wrapped, unrolled, _ = _vibs(eng, N_WRAP, R_WRAP, R0_WRAP)
    og, oa = _oracle_imu(rf)
    # end-point errors agree within 1e-10; the position errors of ref_frame 1 are differences of ECEF
    # coordinates of ~6e6 m, whose last bits (2^-31 .. 2^-30 m) the shapes may round differently over 400 s
    tol = np.full(9, 1e-10)
    tol[3:6] += 2 * np.spacing(np.abs(nav[:, 3:6]).max())
    first, ran = None, 0
    for lanes, shape in SHAPES:
        monkeypatch.setenv('B2INS_MC_SHAPE', shape)
        try:
            w = _k12(eng, rf, lanes, wrapped, dev)
        except ValueError as e:
            assert 'no specialised kernel' in str(e), (lanes, shape, e)
            continue
        u = _k12(eng, rf, lanes, unrolled, dev)
        what = 'rf %d lanes %d shape %s' % (rf, lanes, shape)
        for a, b in zip(w[:3], u[:3]):
            assert np.array_equal(a, b), what + ': wrapped and unrolled series differ'
        assert_close(w[1], og, TOL, 1.0, what + ' gyro')
        assert_close(w[2], oa, TOL, 1.0, what + ' accel')
        if first is None:
            first = w[0]
        assert (np.abs(w[0] - first) < tol).all(), (what, np.abs(w[0] - first).max(0))
        ran += 1
    monkeypatch.delenv('B2INS_MC_SHAPE')
    assert ran >= 10
    # the odometer variant
    odo = eng.to_device(np.zeros(N_WRAP))
    for lanes in (1, 4, 32):
        w, u = _k12(eng, rf, lanes, wrapped, dev, odo), _k12(eng, rf, lanes, unrolled, dev, odo)
        for a, b in zip(w, u):
            assert np.array_equal(a, b), ('odometer', rf, lanes)
        assert_close(w[1], og, TOL, 1.0, 'odometer rf %d lanes %d gyro' % (rf, lanes))
        assert_close(w[2], oa, TOL, 1.0, 'odometer rf %d lanes %d accel' % (rf, lanes))


@pytest.mark.parametrize('tag', ['90deg_mid_rf1_vibrand', '90deg_mid_rf0_vibsin'])
def test_k12_every_shape_on_the_vibration_goldens(eng, tag, monkeypatch):
    """Random and sinusoidal vibration through every launch shape against the reference's histories."""
    g = load_golden('philox_%s.npz' % tag)
    ge = {'b': g['gyro_b'], 'b_drift': g['gyro_b_drift'], 'b_corr': g['gyro_b_corr'], 'arw': g['gyro_arw']}
    ae = {'b': g['accel_b'], 'b_drift': g['accel_b_drift'], 'b_corr': g['accel_b_corr'], 'vrw': g['accel_vrw']}
    vib = {}
    for key in ('vib_acc', 'vib_gyro'):
        a = g[key + '_amp']
        vib[key] = {'type': str(g[key + '_type']), 'x': a[0], 'y': a[1], 'z': a[2], 'freq': float(g[key + '_freq'])}
    R, n, rf = g['gyro'].shape[0], g['gyro'].shape[1], int(g['ref_frame'])
    nav = np.concatenate([g['ref_att'], g['ref_pos'], g['ref_vel']], axis=1)
    dev = [eng.to_device(a) for a in (g['ref_gyro'], g['ref_accel'], nav, g['ini'][None])]
    ran = 0
    for lanes, shape in SHAPES:
        monkeypatch.setenv('B2INS_MC_SHAPE', shape)
        cfg = eng.make_mc_config(rf, float(g['fs']), n, R, int(g['seed']), ge, ae, 1, 9,
                                 run_offset=int(g['run_ids'][0]), vib_gyro=vib['vib_gyro'],
                                 vib_accel=vib['vib_acc'], lanes_per_run=lanes, dump_runs=R)
        try:
            res = eng.mc_free_integration(cfg, *dev, dump_imu=True)
        except ValueError as e:
            assert 'no specialised kernel' in str(e), (lanes, shape, e)
            continue
        what = '%s lanes %d shape %s' % (tag, lanes, shape)
        assert_close(res.gyro.cpu().numpy(), g['gyro'], TOL, 1.0, what + ' gyro')
        assert_close(res.accel.cpu().numpy(), g['accel'], TOL, 1.0, what + ' accel')
        ran += 1
    monkeypatch.delenv('B2INS_MC_SHAPE')
    assert ran >= 10


def test_k7_reads_the_series_at_t_mod_n(eng):
    """The loosely-coupled filter on motion_def-ins.csv (73 250 samples, 10 Hz GPS): the wrapped and the
    unrolled series give the same end-point errors, consistency record and bias estimates, and not the quiet
    run's."""
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import trajectory_from_motion_def
    t = trajectory_from_motion_def(FS, os.path.join(GOLDEN, 'motion_def-ins.csv'), 0, gps=True, fs_gps=10.0)
    n = t['ref_gyro'].shape[0]
    assert n > 4 * 16384
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=True)
    nav = np.concatenate([t['ref_att'], t['ref_pos'], t['ref_vel']], axis=1)
    idx = torch.from_numpy(np.rint(t['gps_time'] * FS).astype(np.int64)).cuda()
    dev = [eng.to_device(a) for a in (t['ref_gyro'], t['ref_accel'], nav, t['ref_gps'], t['gps_visibility'])]
    R, r0 = 8, 3
    wrapped, unrolled, _ = _vibs(eng, n, R, r0)

    def run(vib):
        kw = {} if vib is None else {'vib_accel': vib[0], 'vib_gyro': vib[1]}
        res = eng.ins_loose(FS, R, SEED, imu.gyro_err, imu.accel_err, imu.gps_err, t['ini'], dev[0], dev[1],
                            dev[2], dev[3], idx, dev[4], run_offset=r0, **kw)
        return [x.cpu().numpy() for x in (res.end_err, res.consist, res.end_bias)]

    w, u, q = run(wrapped), run(unrolled), run(None)
    for a, b, name in zip(w, u, ('end_err', 'consist', 'end_bias')):
        assert np.array_equal(a, b), name
    assert np.abs(w[0] - q[0]).max() > 0.0 and np.isfinite(w[0]).all()


def test_k9_reads_the_series_at_t_mod_n(eng):
    """Sensor error statistics of the wrapped and unrolled series agree bit for bit, and equal those of K1's
    histories."""
    rg, ra, _, _ = _still(1)
    imu = _mid()
    dev = eng.to_device(rg), eng.to_device(ra)
    wrapped, unrolled, _ = _vibs(eng, N_WRAP, R_WRAP, R0_WRAP)
    start = 100
    out = []
    for va, vg in (wrapped, unrolled):
        end, proc = eng.imu_err_stats(FS, R_WRAP, *dev, imu.gyro_err, imu.accel_err, SEED, R0_WRAP,
                                      vib_gyro=vg, vib_accel=va, stats_start=start)
        out.append((end.cpu().numpy(), proc.cpu().numpy()))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
    g, a = eng.imu_noise(FS, R_WRAP, *dev, imu.gyro_err, imu.accel_err, SEED, R0_WRAP,
                         vib_gyro=wrapped[1], vib_accel=wrapped[0])
    e = torch.cat([a - dev[1][None], g - dev[0][None]], dim=2).cpu().numpy()
    end, proc = out[0]
    assert np.array_equal(end, e[:, -1])
    es = e[:, start:]
    for k, v in enumerate((np.max(np.abs(es), 1), np.average(es, 1), np.std(es, 1))):
        assert_close(proc[:, k], v, TOL, 1e-9, 'psd stat %d' % k)


def test_sim_psd_environment_end_to_end(eng):
    """Sim(env = PSD tables) on the stationary trajectory of 20001 samples, run_base 7: the gyro and accel
    data of two runs are the oracle's noise plus its PSD series."""
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    n, base, R = 20001, 7, 2
    rg, ra, nav, ini = _still(1, n)
    traj = {'time': np.arange(n) / FS, 'ref_att': nav[:, 0:3], 'ref_pos': nav[:, 3:6], 'ref_vel': nav[:, 6:9],
            'ref_accel': ra, 'ref_gyro': rg}
    table = lambda v: np.column_stack([v['freq'], v['x'], v['y'], v['z']])      # noqa: E731
    sim = Sim([FS, 0.0, 0.0], traj, ref_frame=1, imu=_mid(), env={'acc': table(PSD_ACC), 'gyro': table(PSD_GYRO)},
              algorithm=FreeIntegration(ini), seed=SEED, run_base=base)
    sim.run(R)
    gyro, accel = sim.get_data(['gyro', 'accel'])
    og, oa = _oracle_imu(1, n, R, base)
    for r in range(R):
        assert_close(gyro[r], og[r], TOL, 1.0, 'Sim gyro run %d' % r)
        assert_close(accel[r], oa[r], TOL, 1.0, 'Sim accel run %d' % r)
