"""The speculative blocks of the fused Monte-Carlo kernels, on the host: mc_av_kernel's attitude /
velocity split (att_step<true> in blocks of four, restore and redo with att_step<false>, att_exact after
a warm block ending on a kResync sample, vel_step on the old and new sin/cos) and mc_spec_kernel's
nav_step<RF, false, ODO, true> blocks (tools/step_host.cu, the code the kernels compile).

A block that goes cold -- an increment above kRotMax, the pitch leaving +-pi/2, a NaN -- must leave
exactly what the plain step loop leaves, and non-finite inputs must make the same samples NaN as in
the reference (oracle_np): for every sample and each of att, pos and vel, the row holds a NaN exactly
when the oracle's does.  (Within a row the elements may differ: ref_frame 1 takes c_bn [0, 0, g]
from the third column only, so a NaN yaw does not reach vel.z as the reference's 0 * NaN does.)
Needs nvcc (host pass only); no GPU."""
import ctypes

import numpy as np
import pytest

from conftest import load_golden
from test_cpu_step import host, run as run_step   # noqa: F401  (host: the module fixture that builds the library)
import oracle_np as onp

ROT_MAX = 2.0 ** -5          # kRotMax in csrc/mech.cuh
RESYNC = 64                  # kResync
ANGLE_TOL = 1e-9


@pytest.fixture(scope='module')
def lib(host):               # noqa: F811
    P = ctypes.c_void_p
    host.step_host_av_blocks.argtypes = [ctypes.c_int64, ctypes.c_double, P, P, P, ctypes.c_int, P, P, P]
    host.step_host_spec_blocks.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_double, ctypes.c_int,
                                           ctypes.c_int, P, P, P, ctypes.c_int, P, P, P]
    assert host.step_host_resync_default() == RESYNC
    return host


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def run_blocks(lib, form, rf, fs, gyro, accel, ini, earth_rot=True, odo=False):
    """form 'av': mc_av_kernel's split (ref_frame 1, free integration); 'spec': mc_spec_kernel's blocks."""
    gyro = np.ascontiguousarray(gyro, dtype=np.float64)
    accel = np.ascontiguousarray(accel, dtype=np.float64)
    ini = np.ascontiguousarray(ini, dtype=np.float64)
    n = gyro.shape[0]
    out = [np.full((n, 3), -7.0) for _ in range(3)]
    if form == 'av':
        assert rf == 1 and not odo
        lib.step_host_av_blocks(n, float(fs), _p(gyro), _p(accel), _p(ini), ini.shape[0], *[_p(o) for o in out])
    else:
        lib.step_host_spec_blocks(int(rf), n, float(fs), int(earth_rot), int(odo), _p(gyro), _p(accel), _p(ini),
                                  ini.shape[0], *[_p(o) for o in out])
    return out


def oracle(rf, fs, gyro, accel, ini, odo=False):
    with np.errstate(invalid='ignore', over='ignore'):      # the non-finite cases
        if odo:
            return [a[0] for a in onp.free_integration_odo(rf, fs, gyro[None], accel[None, :, 0], ini[None])]
        return [a[0] for a in onp.free_integration(rf, fs, gyro[None], accel[None], ini[None])]


# ---- checks shared with tests/test_gpu_exact_path.py ---------------------------------------------------
def assert_angles(att, o_att, what, tol=ANGLE_TOL, wrapped=(0, 2), pitch=True):
    """Raw angles, not modulo 2 pi: within tol of the oracle's, or exactly 2 pi off where the oracle's
    angle is within tol of +-pi (the one wrap decided by rounding); the `wrapped` columns (yaw, roll) in
    [-pi, pi] wherever the oracle's are, and the pitch always in [-pi/2, pi/2].  Non-finite oracle
    elements are skipped (the NaN contract is checked on its own)."""
    att, o_att = np.asarray(att), np.asarray(o_att)
    assert att.shape == o_att.shape, (what, att.shape, o_att.shape)
    fin = np.isfinite(o_att)
    with np.errstate(invalid='ignore'):
        d = np.abs(np.where(fin, att - o_att, 0.0))
    flip = (np.abs(d - 2 * np.pi) <= tol) & (np.abs(np.abs(o_att) - np.pi) <= tol)
    if pitch:
        flip[..., 1] = False
    bad = ~((d <= tol) | flip) | (fin & ~np.isfinite(att))
    assert not bad.any(), '%s: %d angles off, worst %.3e at %s' % (what, bad.sum(), d[bad].max(),
                                                                   np.argwhere(bad)[0])
    for k in wrapped:
        inside = fin[..., k] & (np.abs(o_att[..., k]) <= np.pi)
        assert (np.abs(att[..., k][inside]) <= np.pi).all(), (what, 'yaw/roll left [-pi, pi]', k)
    if pitch:
        p = att[..., 1][np.isfinite(att[..., 1])]
        assert (np.abs(p) <= np.pi / 2).all(), (what, 'pitch left [-pi/2, pi/2]', np.abs(p).max())


def nan_rows(x):
    return np.isnan(x).any(axis=-1)


def assert_nan_rows(got, ref, what):
    """For every sample of att, pos and vel: a NaN in got's row exactly when ref's row has one."""
    for name, g, r in zip(('att', 'pos', 'vel'), got, ref):
        gn, rn = nan_rows(g), nan_rows(r)
        assert np.array_equal(gn, rn), '%s %s: NaN rows %d (first %s) against the oracle\'s %d (first %s)' % (
            what, name, gn.sum(), np.argmax(gn) if gn.any() else None, rn.sum(), np.argmax(rn) if rn.any() else None)


def assert_same(got, ref, what):
    for name, g, r in zip(('att', 'pos', 'vel'), got, ref):
        assert np.array_equal(g, r, equal_nan=True), '%s %s: %d elements differ' % (
            what, name, (~((g == r) | (np.isnan(g) & np.isnan(r)))).sum())


# ---- inputs --------------------------------------------------------------------------------------------
INI = np.array([0.55, 2.09, 30.0, 5.0, 0.0, 0.0, 0.1, 0.05, -0.2])


def hard_case(rf):
    """tests/test_cpu_step.py's hard case: increments above kRotMax, yaw and roll wrapping, the pitch
    through +-pi/2, 6000 samples."""
    rng = np.random.default_rng(11 + rf)
    fs, n = 100.0, 6000
    t = np.arange(n) / fs
    ini = np.array([0.55, 2.09, 30.0, 5.0, 0.0, 0.0, 3.0, 0.2, -3.0])
    gyro = np.stack([1.7 * np.sin(0.9 * t) + 0.8, 0.35 * np.cos(0.31 * t), 2.5 * np.cos(0.23 * t) - 0.6], 1)
    gyro += 0.01 * rng.standard_normal((n, 3))
    gyro[2000:2100] *= 4.0
    accel = np.stack([0.3 * np.sin(0.2 * t), 0.2 * np.cos(0.15 * t), -9.8 + 0.1 * np.sin(0.4 * t)], 1)
    return fs, gyro, accel, ini


def reflection_case():
    """tests/test_cpu_step.py's pitch reflection: a pure pitch rate across +pi/2 with roll = 0."""
    fs, n = 100.0, 400
    gyro = np.zeros((n, 3))
    gyro[:, 1] = 0.5
    accel = np.tile([0.0, 0.0, -9.8], (n, 1))
    return fs, gyro, accel, np.array([0.55, 2.09, 30.0, 0.0, 0.0, 0.0, 0.1, 1.45, 0.0])


def gentle(n=300, fs=100.0, seed=3):
    """Slow rotations: no step is cold but for what a test injects."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / fs
    gyro = np.stack([0.2 * np.sin(0.7 * t), 0.1 * np.cos(0.5 * t), 0.3 + 0.05 * np.sin(t)], 1)
    gyro += 1e-3 * rng.standard_normal((n, 3))
    accel = np.stack([0.3 * np.sin(0.2 * t), 0.2 * np.cos(0.15 * t), -9.8 + 0.1 * np.sin(0.4 * t)], 1)
    return fs, gyro, accel


def forms(rf, odo=False):
    return ['spec'] + (['av'] if rf == 1 and not odo else [])


def big_steps(o_att):
    """Steps i -> i + 1 of the oracle with an Euler-angle increment above kRotMax (wraps taken out):
    cold in the kernels."""
    d = np.diff(o_att, axis=0)
    d = (d + np.pi) % (2 * np.pi) - np.pi
    return (np.abs(d) > ROT_MAX).any(1)


# ---- the blocks equal the step loop --------------------------------------------------------------------
@pytest.mark.parametrize('case', ['hard_rf1', 'hard_rf0', 'reflection_rf1', 'reflection_rf0',
                                  'logged_bosch', 'logged_nxp'])
def test_blocks_equal_the_step_loop(lib, case):
    """The hard cases of test_cpu_step.py (cold blocks, pitch reflections, wraps) and logged data: the block
    forms leave bit for bit what the step-by-step loop leaves."""
    if case.startswith('logged'):
        g = load_golden(case + '.npz')
        fs, gyro, accel, ini = float(g['fs']), g['gyro'], g['accel'], g['ini']
        frames = (0, 1)                  # the fixtures are ref_frame 0 data; lat/lon/alt serve ref_frame 1 too
    else:
        frames = (int(case[-1]),)
        fs, gyro, accel, ini = hard_case(frames[0]) if case.startswith('hard') else reflection_case()
        o = oracle(frames[0], fs, gyro, accel, ini)
        if case.startswith('hard'):
            assert big_steps(o[0]).sum() >= 50
        else:
            assert (np.diff(o[0][:, 1]) < 0).any() and np.abs(o[0][:, 1]).max() <= np.pi / 2   # reflected
    for rf in frames:
        step = run_step(lib, rf, fs, gyro, accel, ini)
        for form in forms(rf):
            assert_same(run_blocks(lib, form, rf, fs, gyro, accel, ini), step, '%s %s rf %d' % (case, form, rf))


@pytest.mark.parametrize('rf', [1, 0])
@pytest.mark.parametrize('at', [100, 101, 102, 103, 127, 191, 252, 297])
def test_one_cold_step_at_each_block_position(lib, rf, at):
    """One roll burst above kRotMax at step `at`: positions 0-3 of a block, the last step of a block that
    ends on a kResync sample (127, 191), the first of one (252: block 252..255, 256 = 4 * 64) and a single
    step after the last whole block (n = 300)."""
    fs, gyro, accel = gentle()
    gyro = gyro.copy()
    gyro[at, 0] = 6.0                      # 0.06 rad in one step
    o = oracle(rf, fs, gyro, accel, INI)
    assert np.flatnonzero(big_steps(o[0])).tolist() == [at]
    step = run_step(lib, rf, fs, gyro, accel, INI)
    assert_angles(step[0], o[0], 'step rf %d' % rf)
    for form in forms(rf):
        got = run_blocks(lib, form, rf, fs, gyro, accel, INI)
        assert_same(got, step, '%s rf %d cold at %d' % (form, rf, at))
        assert_angles(got[0], o[0], '%s rf %d' % (form, rf))
        np.testing.assert_allclose(got[2], o[2], rtol=1e-9, atol=1e-9)


def test_warm_blocks_take_the_time_based_reevaluation(lib):
    """Without the re-evaluation every kResync samples the incremental sin/cos drift by about one ulp of
    the increment per step; a long warm series ends bit-equal to the step loop only if the block forms
    re-evaluate on the same samples."""
    fs, n = 100.0, 1283
    t = np.arange(n) / fs
    _, _, accel = gentle(n)
    # a roll rate of ~2.5 rad/s (0.027 rad per step, five turns), small pitch and yaw rates: warm throughout
    gyro = np.stack([2.5 + 0.2 * np.sin(t), np.full(n, 0.05), np.full(n, 0.03)], 1)
    gyro += 1e-3 * np.random.default_rng(5).standard_normal((n, 3))
    o = oracle(1, fs, gyro, accel, INI)
    assert not big_steps(o[0]).any() and np.abs(o[0][:, 1]).max() < 1.0
    assert np.abs(np.diff(o[0][:, 2])).max() > 6.0                  # roll wraps
    step = run_step(lib, 1, fs, gyro, accel, INI)
    never = run_step(lib, 1, fs, gyro, accel, INI, resync=0)
    assert not np.array_equal(never[0], step[0])
    for rf in (1, 0):
        step = run_step(lib, rf, fs, gyro, accel, INI)
        for form in forms(rf):
            assert_same(run_blocks(lib, form, rf, fs, gyro, accel, INI), step, '%s rf %d' % (form, rf))


# ---- non-finite inputs -----------------------------------------------------------------------------------
NONFINITE = {
    'nan_gyro': lambda g, ini: g.__setitem__((101, 2), np.nan),
    'inf_gyro': lambda g, ini: g.__setitem__((130, 0), np.inf),
    'nan_yaw': lambda g, ini: ini.__setitem__(6, np.nan),
    'nan_pitch': lambda g, ini: ini.__setitem__(7, np.nan),
}


@pytest.mark.parametrize('odo', [False, True])
@pytest.mark.parametrize('rf', [1, 0])
@pytest.mark.parametrize('case', sorted(NONFINITE))
def test_non_finite_inputs_propagate_like_the_reference(lib, case, rf, odo):
    """A NaN or Inf gyro sample, a NaN initial yaw or pitch: the step loop and both block forms make the
    same samples NaN as the oracle (the run is invalid from there on), and agree with it before."""
    fs, gyro, accel = gentle()
    gyro, ini = gyro.copy(), INI.copy()
    NONFINITE[case](gyro, ini)
    if odo:
        accel = accel.copy()
        accel[:, 0] = 3.0 + 0.5 * np.sin(np.arange(accel.shape[0]) / 50.0)    # odometer speed in accel.x
    o = oracle(rf, fs, gyro, accel, ini, odo)
    assert nan_rows(o[0]).any() and nan_rows(o[1]).any() and nan_rows(o[2]).any(), 'the oracle goes NaN'
    first = min(int(np.argmax(nan_rows(x))) for x in o)
    got = {'step': run_step(lib, rf, fs, gyro, accel, ini, odo=odo)}
    for form in forms(rf, odo):
        got[form] = run_blocks(lib, form, rf, fs, gyro, accel, ini, odo=odo)
    for form, out in got.items():
        what = '%s %s rf %d odo %d' % (case, form, rf, odo)
        assert_nan_rows(out, o, what)
        if first > 0:
            assert_angles(out[0][:first], o[0][:first], what)
            np.testing.assert_allclose(out[2][:first], o[2][:first], rtol=1e-9, atol=1e-9, err_msg=what)
    for form in forms(rf, odo):
        assert_same(got[form], got['step'], '%s %s rf %d odo %d' % (case, form, rf, odo))
