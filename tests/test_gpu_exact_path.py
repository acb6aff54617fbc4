"""The exact-path fallback of the fused Monte-Carlo kernels on the GPU.

mc_av_kernel (ref_frame 1, groups of 4 and 8) and mc_spec_kernel (groups of 4 and 8) step in blocks of
four without the exact-path branch; a block in which any lane of the warp went cold (an increment above
kRotMax, the pitch leaving +-pi/2, the latitude moving more than 2^-10 rad, a NaN) is restored and redone
step by step, and yaw and roll are wrapped only when the exact path runs.  A warp that writes histories
runs the plain step loop instead, so every case is launched three times: histories of every run (plain
loop) against the oracle; end points only (blocks), bit-equal to the first launch's; and histories of a
few runs of the first warp only (some warps speculate, some do not), bit-equal to the second.

The IMU has no error (b, drift, white noise all 0, no vibration) except in the noisy scenario, so that the
kernels integrate the reference gyro / accel exactly, and every run has its own initial state, so lanes
of one warp go cold at different steps.  Angles are compared raw, not modulo 2 pi."""
import numpy as np
import pytest

from conftest import assert_close
from test_cpu_exact_path import ROT_MAX, assert_angles, nan_rows
from test_gpu_r02 import SHAPES
import oracle_np as onp

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

SEED = 1234
LAT_ROT_MAX = 2.0 ** -10          # kLatRotMax
TOL = 1e-9


@pytest.fixture(scope='module')
def gpu():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    return True


def launch_cases(rf):
    """(lanes, B2INS_MC_SHAPE): every shape of test_gpu_r02 (the split form '6,2,0' is ref_frame 1 only)
    and the default shape of every lane-group width ('')."""
    return ([(g, s) for g, s in SHAPES if not (rf == 0 and s == '6,2,0')] +
            [(g, '') for g in (1, 2, 4, 8, 16, 32)])


def no_error(white):
    return {'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf), white: np.zeros(3)}


class Scenario:
    def __init__(self, rf, fs, gyro, accel, ini, gerr=None, aerr=None, earth_rot=True):
        self.rf, self.fs, self.earth_rot = rf, fs, earth_rot
        self.gyro, self.accel, self.ini = gyro, accel, np.ascontiguousarray(ini)
        self.n, self.R = gyro.shape[0], ini.shape[0]
        self.gerr, self.aerr = gerr or no_error('arw'), aerr or no_error('vrw')
        self.exact_imu = gerr is None and aerr is None
        p0 = onp.lla2ecef(ini[0, :3]) if rf == 1 else ini[0, :3]
        self.nav = np.zeros((self.n, 9))
        self.nav[-1] = np.concatenate([[0.3, 0.2, -0.1], p0, [1.0, 2.0, 3.0]])
        self._dev = None
        self.o = None

    @property
    def dev(self):
        if self._dev is None:
            self._dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (self.gyro, self.accel, self.nav,
                                                                                  self.ini)]
        return self._dev

    def oracle(self, gyro=None, accel=None):
        gyro = np.broadcast_to(self.gyro, (self.R,) + self.gyro.shape) if gyro is None else gyro
        accel = np.broadcast_to(self.accel, (self.R,) + self.accel.shape) if accel is None else accel
        with np.errstate(invalid='ignore', over='ignore'):
            self.o = onp.free_integration(self.rf, self.fs, gyro, accel, self.ini, self.earth_rot)
        return self.o

    def launch(self, monkeypatch, lanes, shape, dump):
        from gnss_ins_sim_b200 import engine
        if shape:
            monkeypatch.setenv('B2INS_MC_SHAPE', shape)
        else:
            monkeypatch.delenv('B2INS_MC_SHAPE', raising=False)
        cfg = engine.make_mc_config(self.rf, self.fs, self.n, self.R, SEED, self.gerr, self.aerr, self.R, 9,
                                    earth_rot=self.earth_rot, lanes_per_run=lanes, dump_runs=dump)
        res = engine.mc_free_integration(cfg, *self.dev, want_state=True, dump_nav=dump > 0, dump_imu=dump > 0)
        monkeypatch.delenv('B2INS_MC_SHAPE', raising=False)
        out = {'end_err': res.end_err.cpu().numpy(), 'end_state': res.end_state.cpu().numpy()}
        if dump:
            for k in ('att', 'pos', 'vel', 'gyro', 'accel'):
                out[k] = getattr(res, k).cpu().numpy()
        return out


def warps_of(R, lanes):
    per = max(1, 32 // lanes)
    return [np.arange(w, min(w + per, R)) for w in range(0, R, per)]


def assert_mixed(flag, lanes, what):
    """Some warp of `lanes`-lane groups holds runs with and without `flag`."""
    assert any(flag[w].any() and not flag[w].all() for w in warps_of(flag.size, lanes)), (what, lanes)


def end_oracle(sc, o):
    r = sc.nav[-1]
    att, pos, vel = (x[:, -1] for x in o)
    with np.errstate(invalid='ignore'):
        err = np.concatenate([onp.angle_range_pi(att - r[0:3]), pos - r[3:6], vel - r[6:9]], 1)
    return err, np.concatenate([att, pos, vel], 1)


def check_nav(sc, att, pos, vel, o, runs, upto, what):
    """Histories of `runs` against the oracle up to sample upto[r] (finite runs), or by the NaN contract."""
    o_att, o_pos, o_vel = o
    for r in runs:
        w = '%s run %d' % (what, r)
        if nan_rows(o_att[r]).any() or nan_rows(o_pos[r]).any() or nan_rows(o_vel[r]).any():
            for name, g, x in (('att', att, o_att), ('pos', pos, o_pos), ('vel', vel, o_vel)):
                assert np.array_equal(nan_rows(g[r]), nan_rows(x[r])), (w, name, 'NaN rows')
            u = min(int(np.argmax(nan_rows(x[r]))) for x in o)
        else:
            u = upto[r]
        assert_angles(att[r, :u], o_att[r, :u], w)
        assert_close(vel[r, :u], o_vel[r, :u], TOL, 1.0, w + ' vel')
        if sc.rf == 1:
            assert_close(pos[r, :u] - pos[r, :1], o_pos[r, :u] - o_pos[r, :1], TOL, 1.0, w + ' pos')
        else:
            assert_close(pos[r, :u, :2], o_pos[r, :u, :2], TOL, 1e-3, w + ' lat/lon')
            assert_close(pos[r, :u, 2], o_pos[r, :u, 2], TOL, 1.0, w + ' alt')


def check_end(sc, out, o, runs, what):
    """end_err and end_state of `runs` against the oracle's last sample; NaN contract per third."""
    o_err, o_state = end_oracle(sc, o)
    for key, ref in (('end_err', o_err), ('end_state', o_state)):
        got = out[key]
        for r in runs:
            w = '%s %s run %d' % (what, key, r)
            for k in range(3):
                assert np.isnan(got[r, 3 * k:3 * k + 3]).any() == np.isnan(ref[r, 3 * k:3 * k + 3]).any(), (w, k)
            if np.isnan(ref[r]).any():
                continue
            if key == 'end_err':
                assert_angles(got[r, :3], ref[r, :3], w, wrapped=(0, 1, 2), pitch=False)
            else:
                assert_angles(got[r, :3], ref[r, :3], w)
            scale = np.maximum(np.abs(o_state[r, 3:]), 1.0)
            assert (np.abs(got[r, 3:] - ref[r, 3:]) <= TOL * scale).all(), (w, got[r, 3:] - ref[r, 3:])


def last_bits_only(rf, lanes, shape):
    """Launches whose history loop and loop without histories are not bit-identical on an H100: in ref_frame 1
    the compiler contracts the two inlined copies of the step into FMAs differently where the group has 8 or more
    lanes and the step is not split over two warps, and in the single-warp form with one lane.  Measured: up to
    35 differing end values of 37 runs, at most 2e-14 rad / 5e-10 m (a 1.5 rad per step burst amplifies the last
    bits).  Every ref_frame 0 launch and the ref_frame 1 split form and groups of 1 to 4 lanes in the specialised
    form are bit-identical, and are held to that."""
    if rf != 1:
        return False
    split = shape == '6,2,0' or (shape == '' and lanes in (4, 8))
    return (lanes >= 8 and not split) or (lanes == 1 and shape == '0')


def assert_same_end(a, b, rf, lanes, shape, what):
    if not last_bits_only(rf, lanes, shape):
        assert np.array_equal(a, b, equal_nan=True), what
        return
    assert np.array_equal(np.isnan(a), np.isnan(b)), what
    with np.errstate(invalid='ignore'):
        bad = np.abs(a - b) > TOL * np.maximum(np.abs(b), 1.0)
    assert not bad.any(), (what, np.nanmax(np.abs(a - b)))


def run_cases(monkeypatch, sc, what=''):
    """The three launches of every launch case; the oracle from the first launch's IMU if the IMU has errors.
    Returns {case: end results of the speculating launch}."""
    R, n = sc.R, sc.n
    upto = np.full(R, n)
    if sc.exact_imu and sc.o is None:
        sc.oracle()
    imu0, ends = None, {}
    for lanes, shape in launch_cases(sc.rf):
        w = '%s lanes %d shape %r' % (what, lanes, shape)
        full = sc.launch(monkeypatch, lanes, shape, R)
        if sc.exact_imu:
            assert np.array_equal(full['gyro'], np.broadcast_to(sc.gyro, full['gyro'].shape)), w
            assert np.array_equal(full['accel'], np.broadcast_to(sc.accel, full['accel'].shape)), w
        elif imu0 is None:
            imu0 = (full['gyro'], full['accel'])
            sc.oracle(*imu0)
            upto = upto_of(sc.o)
        else:
            assert np.array_equal(full['gyro'], imu0[0]) and np.array_equal(full['accel'], imu0[1]), w
        check_nav(sc, full['att'], full['pos'], full['vel'], sc.o, range(R), upto, w)
        whole = [r for r in range(R) if upto[r] == n]
        check_end(sc, full, sc.o, whole, w + ' launch 1')
        spec = sc.launch(monkeypatch, lanes, shape, 0)
        few = sc.launch(monkeypatch, lanes, shape, max(1, (32 // lanes) // 2))
        for k in ('end_err', 'end_state'):
            assert_same_end(spec[k], full[k], sc.rf, lanes, shape, (w, k, 'without histories against with them'))
            assert_same_end(few[k], spec[k], sc.rf, lanes, shape, (w, k, 'histories of part of the first warp'))
        ends[(lanes, shape)] = spec
    return ends


def upto_of(o):
    """Per run, the samples before the first one with |cos(pitch)| < 0.05: beyond it 1/cos amplifies the
    last bits and a random walk is chaotic."""
    near = np.abs(np.cos(o[0][:, :, 1])) < 0.05
    return np.where(near.any(1), np.argmax(near, 1), o[0].shape[1])


def check_k2(sc, gyro, accel, upto, what):
    """The fed single-warp form (K2) of the same runs against the same oracle."""
    from gnss_ins_sim_b200 import engine
    g, a = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (gyro, accel))
    for lanes in (0, 1, 4, 32):
        att, pos, vel = (x.cpu().numpy() for x in engine.free_integration(
            sc.rf, sc.fs, g, a, sc.dev[3], earth_rot=sc.earth_rot, lanes_per_run=lanes))
        check_nav(sc, att, pos, vel, sc.o, range(sc.R), upto, '%s K2 lanes %d' % (what, lanes))


def tiled(sc):
    return (np.broadcast_to(sc.gyro, (sc.R,) + sc.gyro.shape), np.broadcast_to(sc.accel, (sc.R,) + sc.accel.shape))


# ---- A: the pitch through +-pi/2 at a different step in each run ------------------------------------------
def pitch_scenario(rf):
    fs, n, delta = 100.0, 777, 0.01                 # 0.01 rad of pitch per step
    # the step at which each crossing run goes through +-pi/2 (the step from sample s to s + 1): every
    # position in a block and a round, the last step of a kResync period and of a tile, the last step
    targets = [0, 1, 2, 3, 4, 5, 6, 7, 63, 64, 65, 127, 128, 129, 191, 255, 256, 300, 319, 383, 447, 511, 512,
               575, 639, 700, 701, 702, 767, n - 2]
    never = set(range(2, 37, 5))                    # runs that never cross: mixed warps
    R = len(targets) + len(never)
    gyro = np.zeros((n, 3))
    gyro[:, 1] = delta * fs
    accel = np.tile([0.1, -0.2, -9.6], (n, 1))
    ini = np.zeros((R, 9))
    ini[:, :3] = [0.55, 2.09, 30.0]
    ini[:, 6] = np.linspace(-3.0, 3.0, R)
    it = iter(targets)
    for r in range(R):
        if r in never:
            ini[r, 8] = np.pi / 2 if r % 2 else -np.pi / 2       # theta_dot = w_y cos(roll) = 0
            continue
        s = next(it)
        # unfolded pitch p0 + k delta passes pi/2 + m pi half way through step s
        u = (s + 0.5) * delta
        m = np.floor(u / np.pi)
        p0 = np.pi / 2 + m * np.pi - u
        up = r % 2 == 0
        ini[r, 7] = p0 if up else -p0
        ini[r, 8] = 0.0 if up else np.pi
    return Scenario(rf, fs, gyro, accel, ini), np.array(sorted(never)), targets


@pytest.mark.parametrize('rf', [1, 0])
def test_pitch_through_the_singularity_at_every_step_position(gpu, rf, monkeypatch):
    sc, never, targets = pitch_scenario(rf)
    o_att = sc.oracle()[0]
    # reflections: yaw and roll jump by pi
    jump = np.abs(((np.diff(o_att[:, :, 2], axis=1) + np.pi) % (2 * np.pi)) - np.pi) > 3.0
    steps = np.unique(np.nonzero(jump)[1])
    crossing = jump.any(1)
    assert not crossing[never].any() and crossing.sum() == sc.R - never.size
    assert set(steps % 4) == set(range(4)) and set(steps % 8) == set(range(8))
    assert (steps % 64 == 63).any() and (steps % 128 == 127).any() and (sc.n - 2) in steps
    assert set(targets) <= set(steps.tolist())
    assert (np.pi / 2 - np.abs(o_att[:, :, 1])).min() >= 1e-3       # closest approach
    for lanes in (4, 8):
        assert_mixed(crossing, lanes, 'crossing')
    assert (np.abs(np.diff(o_att[never][:, :, 0], axis=1)) > 6.0).any()   # lazily wrapped yaw of the others
    run_cases(monkeypatch, sc, what='pitch rf %d' % rf)
    check_k2(sc, *tiled(sc), np.full(sc.R, sc.n), 'pitch rf %d' % rf)


# ---- B: fast rotations -------------------------------------------------------------------------------------
BIG = {50: 30.0, 51: 150.0, 301: 80.0, 302: 45.0, 303: 120.0, 430: 60.0, 639: 100.0, 767: 35.0, 1000: 90.0,
       1101: 140.0, 1102: 55.0}                       # rad/s on x: 0.3 to 1.5 rad in one step
EDGE = [200, 201, 202, 203, 555, 556, 890, 1279]       # 3.5 rad/s on y: cold or not by the run's roll


def fast_scenario(rf, n=1283, R=203):
    fs = 100.0
    t = np.arange(n) / fs
    gyro = np.stack([2.2 + 0.2 * np.sin(0.8 * t), 0.05 * np.cos(0.3 * t), 0.04 * np.sin(0.5 * t)], 1)
    for s, w in BIG.items():
        if s < n - 1:
            gyro[s, 0] += w
    for s in EDGE:
        if s < n - 1:
            gyro[s, 1] += 3.5
    accel = np.stack([0.3 * np.sin(0.2 * t), 0.2 * np.cos(0.15 * t), -9.8 + 0.1 * np.sin(0.4 * t)], 1)
    ini = np.zeros((R, 9))
    ini[:, :3] = [0.55, 2.09, 30.0]
    ini[:, 3] = 5.0
    ini[:, 6] = np.linspace(-3.0, 3.0, R)
    ini[:, 7] = 0.1 * np.sin(np.arange(R))
    ini[:, 8] = np.linspace(-np.pi, np.pi, R, endpoint=False)
    return Scenario(rf, fs, gyro, accel, ini)


def check_fast_coverage(sc):
    o_att = sc.oracle()[0]
    d = np.abs((np.diff(o_att, axis=1) + np.pi) % (2 * np.pi) - np.pi)
    cold = (d > ROT_MAX).any(2)                                     # [R, n - 1]
    big = [s for s in BIG if s < sc.n - 1]
    assert cold[:, big].all()
    edge = [s for s in EDGE if s < sc.n - 1]
    for s in edge:
        assert cold[:, s].any() and not cold[:, s].all(), s          # the same burst: cold in some lanes only
    assert set(np.array(edge) % 4) == set(range(4))
    assert_mixed(cold[:, edge[0]], 4, 'edge burst')
    assert_mixed(cold[:, edge[0]], 8, 'edge burst')
    turns = np.abs(np.unwrap(o_att[:, :, 2], axis=1)[:, -1] - o_att[:, 0, 2]) / (2 * np.pi)
    assert turns.min() >= 3.0
    assert np.abs(o_att[:, :, 1]).max() < 1.2


@pytest.mark.parametrize('rf', [1, 0])
def test_fast_rotations(gpu, rf, monkeypatch):
    sc = fast_scenario(rf)
    check_fast_coverage(sc)
    run_cases(monkeypatch, sc, what='fast rf %d' % rf)
    check_k2(sc, *tiled(sc), np.full(sc.R, sc.n), 'fast rf %d' % rf)


# ---- C: noisy Monte-Carlo runs -------------------------------------------------------------------------------
@pytest.mark.parametrize('rf', [1, 0])
def test_noisy_monte_carlo_runs(gpu, rf, monkeypatch):
    """White gyro noise of 0.015 rad per sample: increments fall on both sides of kRotMax at random."""
    fs, n, R = 100.0, 777, 37
    gyro = np.tile([0.3, 0.1, -0.2], (n, 1))
    accel = np.tile([0.2, -0.1, -9.8], (n, 1))
    ini = np.zeros((R, 9))
    ini[:, :3] = [0.55, 2.09, 30.0]
    ini[:, 6] = np.linspace(-3.0, 3.0, R)
    ini[:, 8] = np.linspace(-1.0, 1.0, R)
    gerr = {'b': np.array([0.01, -0.02, 0.005]), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf),
            'arw': np.full(3, 0.15)}
    aerr = {'b': np.zeros(3), 'b_drift': np.zeros(3), 'b_corr': np.full(3, np.inf), 'vrw': np.full(3, 0.05)}
    sc = Scenario(rf, fs, gyro, accel, ini, gerr, aerr)
    run_cases(monkeypatch, sc, what='noisy rf %d' % rf)
    o_att = sc.o[0]
    upto = upto_of(sc.o)
    assert (upto == n).sum() >= R // 2
    d = np.abs((np.diff(o_att, axis=1) + np.pi) % (2 * np.pi) - np.pi)
    cold = (d > ROT_MAX).any(2)
    assert 0.02 < cold.mean() < 0.5
    blocks = cold[:, :(n - 1) // 4 * 4].reshape(R, -1, 4).any(2)     # [R, blocks]: cold blocks per run
    for lanes in (4, 8):
        assert any((blocks[w].any(0) & ~blocks[w].all(0)).any() for w in warps_of(R, lanes))


# ---- D: a non-finite run among finite ones -----------------------------------------------------------------
@pytest.mark.parametrize('rf', [1, 0])
@pytest.mark.parametrize('what', ['yaw', 'pitch'])
def test_nan_run_propagates_and_leaves_its_warp_alone(gpu, rf, what, monkeypatch):
    """Run 10 (in the middle of a CTA of every shape) starts with a NaN angle: from the samples the oracle
    makes NaN on, its rows are NaN, its end_err too; every other run equals a launch without the NaN
    bit for bit (the NaN lane is cold in every block, so its warp redoes every block)."""
    sc = fast_scenario(rf, n=777, R=37)
    finite = run_cases(monkeypatch, sc, what='finite rf %d' % rf)
    bad = 10
    ini = sc.ini.copy()
    ini[bad, 6 if what == 'yaw' else 7] = np.nan
    sc_nan = Scenario(rf, sc.fs, sc.gyro, sc.accel, ini)
    o = sc_nan.oracle()
    assert nan_rows(o[0][bad]).all() and nan_rows(o[2][bad]).any()
    assert not any(nan_rows(x[np.arange(sc.R) != bad]).any() for x in o)
    ends = run_cases(monkeypatch, sc_nan, what='NaN %s rf %d' % (what, rf))
    others = np.arange(sc.R) != bad
    for case, out in ends.items():
        for k in ('end_err', 'end_state'):
            assert_same_end(out[k][others], finite[case][k][others], rf, *case, (case, k, 'runs beside the NaN run'))
            assert np.isnan(out[k][bad]).any()
    check_k2(sc_nan, *tiled(sc_nan), np.full(sc.R, sc.n), 'NaN %s rf %d' % (what, rf))


# ---- E: ref_frame 0, the latitude's increment above 2^-10 rad ---------------------------------------------
def test_latitude_increment_takes_the_exact_path(gpu, monkeypatch):
    """At 1 Hz a northward speed of ~6.2 km/s moves the latitude 2^-10 rad per step: runs from 4 to 8 km/s,
    some cold on the latitude alone, others not."""
    fs, n, R = 1.0, 777, 37
    gyro = np.zeros((n, 3))
    accel = np.tile([0.0, 0.0, -9.8], (n, 1))
    ini = np.zeros((R, 9))
    ini[:, :3] = [0.2, 1.0, 100.0]
    ini[:, 3] = 4000.0 + 4000.0 * ((np.arange(R) * 7) % R) / (R - 1)     # shuffled: mixed warps
    sc = Scenario(0, fs, gyro, accel, ini)
    o_att, o_pos, _ = sc.oracle()
    dlat = np.abs(np.diff(o_pos[:, :, 0], axis=1))
    d = np.abs((np.diff(o_att, axis=1) + np.pi) % (2 * np.pi) - np.pi)
    assert (d <= ROT_MAX).all() and np.abs(o_att[:, :, 1]).max() < 1.2   # the latitude is the only trigger
    lat_cold = (dlat > LAT_ROT_MAX).any(1)
    assert lat_cold.any() and not lat_cold.all()
    for lanes in (4, 8):
        assert_mixed(lat_cold, lanes, 'latitude')
    run_cases(monkeypatch, sc, what='latitude')
    check_k2(sc, *tiled(sc), np.full(sc.R, sc.n), 'latitude')
