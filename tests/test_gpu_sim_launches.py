"""Which kernel launches and uploads Sim makes for its lazy data, counted by wrapping the engine entry
points: history blocks, the histories() arrays, the odometer, GPS and magnetometer histories, the filter,
re-running a Sim with two plugins, and that a dropped Sim is freed without the cyclic collector."""
import gc
import weakref

import numpy as np
import pytest

from conftest import load_golden

torch = pytest.importorskip('torch')
gpu = pytest.mark.gpu


@pytest.fixture
def eng():
    if not torch.cuda.is_available():
        pytest.skip('no CUDA device')
    from gnss_ins_sim_b200 import engine
    return engine


def _traj(g):
    return {k: g[k] for k in ('time', 'ref_pos', 'ref_vel', 'ref_att', 'ref_accel', 'ref_gyro', 'ini')}


def _ini():
    return load_golden('philox_90deg_mid_rf0.npz')['ini']


def _count(monkeypatch, eng, *names):
    """Wrap engine.<name> for each name; returns the list of (name, args, kwargs) of every call."""
    calls = []
    for nm in names:
        def wrap(*a, _real=getattr(eng, nm), _nm=nm, **k):
            calls.append((_nm, a, k))
            return _real(*a, **k)
        monkeypatch.setattr(eng, nm, wrap)
    return calls


def _k12(calls):
    """(runs, run_offset, dump_runs, algo) of each K12 launch."""
    return [(a[0].runs, a[0].run_offset, a[0].dump_runs, a[0].algo) for nm, a, k in calls
            if nm == 'mc_free_integration']


def _sim(algorithm=None, **kw):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    g = load_golden('philox_90deg_mid_rf0.npz')
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False)
    return Sim([100.0, 0.0, 0.0], _traj(g), ref_frame=0, imu=imu, algorithm=algorithm, seed=int(g['seed']), **kw)


def _gps_mag_sim(algorithm=None, **kw):
    """ref_frame 0, a 9-axis IMU with GPS: the 90-degree turn with its GPS rows and magnetic field."""
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    g, gp, m = (load_golden(f) for f in ('philox_90deg_mid_rf0.npz', 'gps_90deg_rf0.npz', 'mag_90deg.npz'))
    traj = dict(_traj(g), ref_gps=gp['ref_gps'], gps_time=gp['gps_time'], gps_visibility=gp['gps_visibility'],
                ref_mag=m['ref_mag_rf0'])
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=9, gps=True)
    return Sim([100.0, 10.0, 0.0], traj, ref_frame=0, imu=imu, algorithm=algorithm, seed=5, **kw), traj


@gpu
def test_free_integration_history_blocks(eng, monkeypatch):
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    sim = _sim(FreeIntegration(_ini()))
    sim.run(40)
    calls = _count(monkeypatch, eng, 'mc_free_integration', 'imu_noise')
    pos = sim.get_data(['pos'])[0]
    pos['algo0_0'], pos['algo0_31']
    assert _k12(calls) == [(32, 0, 32, 0)] and len(calls) == 1
    pos['algo0_32']
    assert _k12(calls) == [(32, 0, 32, 0), (8, 32, 8, 0)] and len(calls) == 2
    # the K12 history block also holds the runs' IMU samples and every navigation output
    sim.get_data(['gyro'])[0][5], sim.get_data(['att_euler'])[0]['algo0_0']
    assert len(calls) == 2


@gpu
def test_histories_serve_get_data(eng, monkeypatch):
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    sim = _sim(FreeIntegration(_ini()))
    sim.run(12)
    calls = _count(monkeypatch, eng, 'mc_free_integration', 'imu_noise')
    h = sim.histories()
    assert len(calls) == 1
    assert np.array_equal(sim.get_data(['vel'])[0]['algo0_7'], h['vel'][7])
    assert len(calls) == 1
    sim.run(12)
    sim.histories(stride=10)
    assert len(calls) == 2
    sim.get_data(['vel'])[0]['algo0_7']
    assert _k12(calls)[2] == (12, 0, 12, 0)


@gpu
def test_odo_histories_come_from_the_odometer_plugin(eng, monkeypatch):
    from gnss_ins_sim_b200 import imu_model
    from gnss_ins_sim_b200.sim import Sim
    from gnss_ins_sim_b200.free_integration_odo import FreeIntegration as FreeIntegrationOdo
    g = load_golden('philox_90deg_mid_rf0_odo.npz')
    imu = imu_model.IMU(accuracy='mid-accuracy', axis=6, gps=False, odo=True,
                        odo_opt={'scale': float(g['odo_scale']), 'stdv': float(g['odo_stdv'])})
    sim = Sim([100.0, 0.0, 0.0], dict(_traj(g), ref_odo=g['ref_odo']), ref_frame=0, imu=imu,
              algorithm=FreeIntegrationOdo(g['ini']), seed=int(g['seed']))
    sim.run(6)
    calls = _count(monkeypatch, eng, 'mc_free_integration', 'imu_noise')
    sim.get_data(['odo'])[0][3]
    assert _k12(calls) == [(6, 0, 6, 1)] and len(calls) == 1
    sim.get_data(['gyro'])[0][3], sim.get_data(['pos'])[0]['algo0_1']
    assert len(calls) == 1


@gpu
def test_gps_and_mag_history_blocks(eng, monkeypatch):
    sim, traj = _gps_mag_sim(history_block=4)
    calls = _count(monkeypatch, eng, 'gps_noise', 'mag_noise', 'imu_noise', 'to_device')
    sim.run(10)
    gps, mag = sim.get_data(['gps', 'mag'])
    for r in (0, 3, 5, 9):
        gps[r], mag[r]
    for r in (1, 6):
        gps[r], mag[r]
    for nm in ('gps_noise', 'mag_noise'):
        assert [k.get('run_offset') for n, a, k in calls if n == nm] == [0, 4, 8]
    assert not [c for c in calls if c[0] == 'imu_noise']
    for key in ('ref_gps', 'ref_mag'):
        ups = [a for n, a, k in calls if n == 'to_device' and isinstance(a[0], np.ndarray)
               and a[0].shape == traj[key].shape and np.array_equal(a[0], traj[key])]
        assert len(ups) <= 1, key


@gpu
def test_filter_history_block(eng, monkeypatch):
    from gnss_ins_sim_b200.ins_loose import InsLoose
    sim = _gps_mag_sim(InsLoose(_ini()))[0]
    sim.run(6)
    calls = _count(monkeypatch, eng, 'ins_loose', 'mc_free_integration', 'imu_noise')
    sim.get_data(['wb'])[0]['algo0_2']
    assert [(c[0], c[2].get('dump_runs')) for c in calls] == [('ins_loose', 6)]
    sim.get_data(['pos'])[0]['algo0_3']
    assert len(calls) == 1


@gpu
def test_second_run_publishes_only_its_own_outputs(eng):
    from gnss_ins_sim_b200.free_integration import FreeIntegration
    sim = _sim([FreeIntegration(_ini()), FreeIntegration(_ini())])
    sim.run(8)
    sim.run(4)
    pos = sim.get_data(['pos'])[0]
    assert len(pos) == 8
    assert sorted(pos) == ['algo%d_%d' % (a, r) for a in (0, 1) for r in range(4)]
    assert 'algo0_5' not in pos


def _freed(make):
    """Whether the Sim that make() builds and uses is freed by reference counting alone."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        return make() is None
    finally:
        if enabled:
            gc.enable()


def test_sim_without_device_work_is_freed_without_the_cyclic_collector():
    def make():
        sim = _sim()
        sim.run(3)
        sim.get_data(['gyro', 'ref_att_quat'])
        return weakref.ref(sim)
    assert _freed(lambda: make()())


@gpu
def test_sim_is_freed_without_the_cyclic_collector(eng):
    from gnss_ins_sim_b200.free_integration import FreeIntegration

    def make():
        sim = _sim(FreeIntegration(_ini()))
        sim.run(5)
        sim.get_data(['pos'])[0]['algo0_1']
        sim.get_data(['gyro'])[0][2]
        sim.histories()
        return weakref.ref(sim)
    assert _freed(lambda: make()())
