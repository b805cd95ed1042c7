"""The reference's numpy dynamics path (use_numba=False; QuadrotorDynamics.step1 + floor_interaction,
quadrotor_dynamics.py:225-346, 389-457; include/quadswarm.h, qs_set_numpy_dynamics): the oracle pinned to the reference's
own trajectories (tests/golden/numpy_path_*.npz, written by oracle/gen_golden_numpy_path.py), the keyed landing-yaw draws,
the host-side keyword handling, and on the GPU the kernels against the oracle with planted floor states in every launch
shape, rollout against single steps, and what the floor model does to a sliding drone."""
import glob
import math
import os
import re
import types

import numpy as np
import pytest
from scipy import stats

from oracle import numpy_path_oracle as npo
from oracle import philox as px
from oracle import quadswarm_oracle as qo
from oracle import sensor_noise_oracle as sno

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
FILES = sorted(glob.glob(os.path.join(GOLDEN, 'numpy_path_*.npz')))
TOL = dict(rtol=1e-9, atol=1e-9)
ARM = qo.QuadParams.arm


def _make_scenario(mode, cfg, rng):
    from quad_swarm_rl_b200.scenarios import create_scenario
    sc = create_scenario(mode, cfg.num_agents, room_dims=cfg.room_dims, rng=np.random.RandomState(0),
                         ep_time=cfg.ep_time, use_obstacles=cfg.use_obstacles)
    sc.rng = rng
    return sc


def test_fixtures_present():
    assert [os.path.basename(f) for f in FILES] == ['numpy_path_c3_obstacles_8.npz', 'numpy_path_defaultquad_drag_4.npz',
                                                    'numpy_path_floor_8.npz', 'numpy_path_wall_gyro_bias_6.npz']


_REPLAYS = {}


def _replay(path):
    if path not in _REPLAYS:
        _REPLAYS[path] = npo.replay_numpy_path_golden(np.load(path, allow_pickle=False), _make_scenario)
    return _REPLAYS[path]


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[len('numpy_path_'):-4] for f in FILES])
def test_oracle_replays_reference_numpy_path(path):
    """Observations, rewards, reward terms, dones, goals, every recorded state and the episode statistics to 1e-9."""
    import json
    g = np.load(path, allow_pickle=False)
    out, env = _replay(path)
    assert env.cfg.use_numba is False
    np.testing.assert_allclose(out['obs0'], g['obs0'], **TOL)
    assert np.array_equal(out['dones'], g['dones'])
    np.testing.assert_allclose(out['rewards'], g['rewards'], **TOL)
    np.testing.assert_allclose(out['goals'], g['goals'], **TOL)
    m = ~np.isnan(g['infos'])
    assert np.array_equal(np.isnan(out['infos']), ~m)
    np.testing.assert_allclose(out['infos'][m], g['infos'][m], **TOL)
    np.testing.assert_allclose(out['obs'], g['obs'], **TOL)
    for k in ('pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou'):
        np.testing.assert_allclose(out['state_' + k], g['state_' + k], err_msg=k, **TOL)
    assert np.array_equal(out['state_on_floor'], g['state_on_floor'])
    ref_stats = json.loads(str(g['ep_stats_json']))
    assert len(ref_stats) >= 1 and [t for t, _ in out['ep_stats']] == [t for t, _ in ref_stats]
    for (_, mine), (_, ref) in zip(out['ep_stats'], ref_stats):
        for k, v in ref.items():
            assert mine[k] == pytest.approx(v, rel=1e-9, abs=1e-9), k


def test_fixtures_exercise_the_numpy_floor_model():
    """Together the fixtures hold drones resting on the floor between the arm and 0.05 m (the njit path would have them in
    the air), sliding sub-steps, the vx = vy = 0 friction corner, and upside-down landings whose yaw loop retried (counted by
    the oracle, whose replay of numpy's stream would lose step at the first try it missed or invented)."""
    seen = dict(between=0, slides=0, corner=0, landings=0, retries=0)
    for path in FILES:
        g = np.load(path)
        z = g['state_pos'][..., 2]
        seen['between'] += int(np.sum(g['state_on_floor'] & (z > ARM + 1e-3)))
        for d in _replay(path)[1].drones:
            seen['slides'] += getattr(d, 'slides', 0)
            seen['corner'] += getattr(d, 'slide_corner', 0)
            seen['landings'] += getattr(d, 'landings_upside_down', 0)
            seen['retries'] += getattr(d, 'landing_yaw_tries', 0) - getattr(d, 'landings_upside_down', 0)
    print(seen)
    assert all(v > 0 for v in seen.values()), seen
    assert np.all(np.load(os.path.join(GOLDEN, 'numpy_path_floor_8.npz'))['state_pos'][..., 2] >= 0.05 - 1e-12)


def test_landing_yaw_is_keyed_at_site_23():
    """The keyed landing yaw: try k of sub-step j of drone i is word k % 4 of Philox block (env, step, 23 | i << 8 | j << 16,
    k // 4) (qs_rng.cuh, SITE_FLOOR_YAW_NP); the first try whose body x-axis lies within 60 deg of the direction to the
    origin is taken, at most 64 tries.  Over many landings: accepted yaws uniform in that +-60 deg cone, tries geometric
    with p = 1/3."""
    assert npo.SITE_FLOOR_YAW_NP == 23 and npo.FLOOR_YAW_MAX_TRIES == 64
    src = open(os.path.join(ROOT, 'quad_swarm_rl_b200', 'csrc', 'qs_rng.cuh')).read()
    assert re.search(r'SITE_FLOOR_YAW_NP = 23,', src)
    rng = qo.PhiloxRng(20261016)
    offsets, tries = [], []
    for n in range(3000):
        env, step, i, sub = n % 37, n // 37, n % 8, n % 2
        rng.begin(env, step)
        d = qo.Drone()
        ang = 0.37 * n
        d.pos = np.array([3.0 * math.cos(ang), 3.0 * math.sin(ang), 0.05])
        rot, k = npo.landing_yaw(d, rng, i, sub)
        # the same tries from the raw generator
        for t in range(k):
            blk = px.philox4x32_10(env, step, (23 | i << 8 | sub << 16), t // 4, 20261016 & px.MASK, 0)
            th = -math.pi + 2 * math.pi * px.u01(blk[t % 4])
            ok = math.cos(th) * -math.cos(ang) + math.sin(th) * -math.sin(ang) >= 0.5
            assert ok == (t == k - 1), (n, t)
        assert rot[0, 0] == pytest.approx(math.cos(th), abs=1e-15) and rot[1, 0] == pytest.approx(math.sin(th), abs=1e-15)
        offsets.append((math.atan2(rot[1, 0], rot[0, 0]) - (ang + math.pi) + math.pi) % (2 * math.pi) - math.pi)
        tries.append(k)
    assert np.max(np.abs(offsets)) <= math.pi / 3 + 1e-12
    assert stats.kstest(offsets, 'uniform', args=(-math.pi / 3, 2 * math.pi / 3)).pvalue > 1e-3
    assert np.mean(tries) == pytest.approx(3.0, rel=0.08)


def test_numpy_stream_routing_and_ou_constants():
    """NumpyReplayRng serves the thrust noise, the sensor noise and the landing yaw from numpy's global stream; the
    collision responses keep numba's.  OUNoise keeps theta = 0.15 and sigma = 0.01 in float64."""
    rng = npo.NumpyReplayRng(1, 2, [3])
    for site in (px.SITE_OU, px.SITE_SENSOR0, px.SITE_SENSOR1, px.SITE_SENSOR_RESET, npo.SITE_FLOOR_YAW_NP,
                 sno.SITE_NOISE_N, sno.SITE_NOISE_U, sno.SITE_GYRO_BIAS):
        assert rng._stream(site) is rng.py, site
    for site in (px.SITE_PAIR_N, px.SITE_PAIR_U, px.SITE_OBST_U):
        assert rng._stream(site) is rng.nb, site
    cfg = npo.enable(qo.EnvConfig(num_agents=1))
    env = qo.OracleEnv(cfg, npo.NumpyReplayRng(5, 6, [7]), qo.TableEpisodeSource([dict(goals=np.zeros((1, 3)), spawn=np.zeros((1, 3)), obst_xy=None)]))
    d = env.drones[0]
    d.ou = np.array([0.1, -0.2, 0.3, 0.0])
    ou = qo.ou_noise_step(d, env.P, env.rng, 0)
    rs = np.random.RandomState(5)
    x = np.array([0.1, -0.2, 0.3, 0.0])
    np.testing.assert_array_equal(ou, x + (0.15 * (0 - x) + 0.2 * 0.05 * rs.randn(4)))


def test_header_declares_and_lib_binds_the_entry_point():
    import ctypes
    from quad_swarm_rl_b200 import _lib as L
    hdr = open(os.path.join(ROOT, 'include', 'quadswarm.h')).read()
    decl = re.search(r'int qs_set_numpy_dynamics\(([^)]*)\);', hdr).group(1)
    assert [a.strip().rsplit(' ', 1)[0] for a in decl.split(',')] == ['QsHandle*', 'int']
    assert L.EXPORTS['qs_set_numpy_dynamics'] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int])


def test_entry_point_rejects_a_null_handle_without_gpu():
    import sys
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from quad_swarm_rl_b200 import _lib as L
    lib = L.load()
    assert lib.qs_set_numpy_dynamics(None, 1) == -1 and b'null' in lib.qs_last_error()


def test_numpy_path_kernels_fit_like_the_default_ones():
    """The numpy path has its own step kernels, one per default instantiation, built from the same body; the ones that can
    carry the courier warp keep its budget (<= 128 registers, no local memory: two CTAs of consecutive steps per SM)."""
    from tests.parity_util import kernel_resources
    usage = kernel_resources(r'qs_step_kernel(_npy)?ILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE')
    default = sorted(k[1:] for k in usage if not k[0])
    assert len(default) == 84 and sorted(k[1:] for k in usage if k[0]) == default
    courier = {k: v for k, v in usage.items() if k[0] and k[1] < 16 and k[2:] == (0, 0, 1, 0, 0)}
    assert sorted(k[1] for k in courier) == [1, 2, 4, 8]
    for k, v in courier.items():
        assert v['REG'] <= 128 and v['LOCAL'] == 0, (k, v)


class _Captured(Exception):
    pass


def _cfg(**extra):
    return types.SimpleNamespace(**dict(dict(
        quads_num_agents=4, quads_episode_duration=1.0, quads_obs_repr='xyz_vxyz_R_omega', quads_neighbor_visible_num=2,
        quads_neighbor_obs_type='pos_vel', quads_collision_hitbox_radius=2.0, quads_collision_falloff_radius=4.0,
        quads_use_obstacles=False, quads_obst_density=0.2, quads_obst_size=0.6, quads_obst_spawn_area=[8.0, 8.0],
        quads_use_downwash=False, quads_mode='static_same_goal', quads_room_dims=[10., 10., 10.], seed=3), **extra))


@pytest.mark.parametrize('flag,expect', [(None, True), (True, True), (False, False)])
def test_factory_reads_quads_use_numba(flag, expect, monkeypatch):
    """make_quadrotor_env_multi_batched passes --quads_use_numba on; an object without the attribute keeps the njit path."""
    from quad_swarm_rl_b200 import env as env_mod
    from quad_swarm_rl_b200.wrappers import make_quadrotor_env_multi_batched

    def fake(**kw):
        raise _Captured(kw)
    monkeypatch.setattr(env_mod, 'QuadrotorEnvMultiBatched', fake)
    cfg = _cfg() if flag is None else _cfg(quads_use_numba=flag)
    with pytest.raises(_Captured) as e:
        make_quadrotor_env_multi_batched(cfg, num_envs=2)
    assert e.value.args[0]['use_numba'] is expect


@pytest.mark.parametrize('use_numba', [False, True])
def test_env_objects_forward_use_numba_to_the_engine(use_numba, monkeypatch):
    from quad_swarm_rl_b200 import env as env_mod

    def fake(**kw):
        raise _Captured(kw)
    monkeypatch.setattr(env_mod, 'QuadSwarmEngine', fake)
    kw = dict(num_agents=4, ep_time=1.0, rew_coeff=None, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=2,
              neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0, use_obstacles=False,
              obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0], use_downwash=False, use_numba=use_numba,
              quads_mode='static_same_goal', room_dims=[10., 10., 10.], use_replay_buffer=False, quads_view_mode=['topdown'],
              quads_render=False, dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
              dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
              init_random_state=False, seed=3)
    for make in (lambda: env_mod.QuadrotorEnvMulti(**kw),
                 lambda: env_mod.QuadrotorEnvMultiBatched(num_envs=2, num_agents=4, use_numba=use_numba, seed=3)):
        with pytest.raises(_Captured) as e:
            make()
        assert e.value.args[0]['use_numba'] is use_numba
    with pytest.raises(_Captured) as e:
        env_mod.QuadrotorEnvMultiBatched(num_envs=2, num_agents=4, seed=3)
    assert e.value.args[0]['use_numba'] is True


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
KW = dict(num_agents=8, neighbor_visible_num=2, ep_time=0.9, obs_repr='xyz_vxyz_R_omega_floor', use_numba=False)
C3_FULL = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True, use_downwash=True,
               ep_time=0.9, use_numba=False)
C2_FULL = dict(num_agents=8, neighbor_visible_num=6, ep_time=0.9, use_numba=False)
C4_FULL = dict(num_agents=32, neighbor_visible_num=6, ep_time=0.6, use_numba=False)
NOISE = dict(gyro_norm_std=0.1, quat_norm_std=0.01, pos_unif_range=0.01)
C3_REW = dict(quadcol_bin=5.0, quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
PLANT_AT = (0, 20, 40, 60)


def _rotz(a):
    return np.array([[math.cos(a), -math.sin(a), 0.], [math.sin(a), math.cos(a), 0.], [0., 0., 1.]])


def _rotx(a):
    return np.array([[1., 0., 0.], [0., math.cos(a), -math.sin(a)], [0., math.sin(a), math.cos(a)]])


def _plant_floor(pair, t, counts):
    """Planted floor states on the oracle side, copied to the device: per drone, in turn, airborne between the arm and
    0.05 m, an upside-down landing away from the origin, sliding on the floor, pushed straight down on the floor.  Before
    every step, the crashed_floor masks of the previous one are compared where that step was decided away from thresholds."""
    from quad_swarm_rl_b200 import _lib as L
    from tests.parity_util import MARGIN_EPS
    if t > 0:
        fl = pair.device_fields()['flags']
        for e, o in enumerate(pair.oracles):
            if o.step_margin > MARGIN_EPS and o.tick > 0:
                dev = (fl[e] & L.FLAG_CRASHED_FLOOR) != 0
                assert np.array_equal(dev, [d.crashed_floor for d in o.drones]), f'crashed_floor differs before step {t} env {e}'
                counts['crashed_floor'] += int(dev.sum())
    if t not in PLANT_AT:
        return
    rs = np.random.RandomState(1000 + t)
    for o in pair.oracles:
        for i, d in enumerate(o.drones):
            kind = (i + PLANT_AT.index(t)) % 4
            r, a = rs.uniform(1.0, 4.0), rs.uniform(-math.pi, math.pi)
            x, y = r * math.cos(a), r * math.sin(a)
            yaw = rs.uniform(-math.pi, math.pi)
            d.omega = np.zeros(3)
            if kind == 0:
                d.pos, d.vel, d.rot, d.on_floor = np.array([x, y, rs.uniform(ARM + 5e-4, 0.05 - 5e-4)]), \
                    np.array([rs.uniform(-0.5, 0.5), rs.uniform(-0.5, 0.5), 0.]), _rotz(yaw), False
            elif kind == 1:
                d.pos, d.vel, d.rot, d.on_floor = np.array([x, y, 0.06]), np.array([0., 0., -1.5]), \
                    _rotz(yaw) @ _rotx(math.pi - rs.uniform(0, 0.4)), False
            elif kind == 2:
                d.pos, d.vel, d.rot, d.on_floor = np.array([x, y, 0.05]), \
                    np.array([rs.uniform(-1, 1), rs.uniform(-1, 1), 0.]), _rotz(yaw), True
            else:
                d.pos, d.vel, d.rot, d.on_floor = np.array([x, y, 0.05]), np.array([0., 0., -0.3]), _rotz(yaw), True
            z = d.pos[2]                        # 0.05 stays exact: the device's 0.05f is on the floor too
            d.pos = d.pos.astype(np.float32).astype(np.float64)
            d.pos[2] = z if z == 0.05 else d.pos[2]
            d.vel = d.vel.astype(np.float32).astype(np.float64)
            d.rot = d.rot.astype(np.float32).astype(np.float64)
            d.crashed_floor = False
            d.acc = np.zeros(3)
    pair.sync_device_from_oracle()


def _drag_rows(pair):
    """Every drone flies DefaultQuad with rotor drag and rolling moment (qs_set_dynamics -> DYN kernels), on both sides."""
    from quad_swarm_rl_b200 import quad_models as qm
    from quad_swarm_rl_b200.quad_models import DYN_FIELDS
    row = qm.constants_row(qm.defaultquad_params()).copy()
    row[DYN_FIELDS.index('c_drag')], row[DYN_FIELDS.index('c_roll')] = 0.01, 0.001
    rows = np.broadcast_to(row, (pair.engine.E, pair.N, len(row))).astype(np.float32).copy()
    pair.engine.set_dynamics(rows)
    P = qo.quad_params_from_constants(dict(zip(DYN_FIELDS, row.astype(np.float32).astype(np.float64))))
    for o in pair.oracles:
        o.Ps = [P] * pair.N
        o.P = P


SHAPES = ['wait', 'handover', 'split', 'balanced_c2', 'courier_c3', 'multiwave_c4', 'dyn', 'nz']


@pytest.mark.gpu
@pytest.mark.parametrize('shape', SHAPES)
def test_kernel_matches_oracle_with_planted_floor_states(shape, monkeypatch):
    """Kernel (keyed draws) against the oracle on the numpy path with planted floor states: the grid-wide wait and the
    per-block hand-over (QS_PDL), the split kernels (QS_SPLIT), chained full-size grids in the balanced, courier (c3) and
    multi-wave (c4) shapes, per-drone constants with rotor drag (DYN) and a noise dict with the gyro-bias model (NZ).
    States within 1e-4 + 1e-4 |ref|, on_floor / crashed_floor masks bit-exact away from the thresholds."""
    from oracle.scenario_gen import DeviceORandomSource, DeviceScenarioSource
    from tests import parity_util as pu
    if shape in ('wait', 'handover'):
        monkeypatch.setenv('QS_PDL', '2' if shape == 'wait' else '3')
    if shape == 'split':
        monkeypatch.setenv('QS_SPLIT', '1')
    if shape == 'balanced_c2':
        pair = pu.SampledPair(1024, [0, 511, 1023], C2_FULL, seed=7101, device_scenario='static_same_goal',
                              source_factory=lambda: DeviceScenarioSource('static_same_goal'), chained=True)
    elif shape == 'courier_c3':
        pair = pu.SampledPair(4096, [0, 2048, 4095], C3_FULL, seed=7102, device_scenario='o_random',
                              source_factory=lambda: DeviceORandomSource(), chained=True, rew_coeff=C3_REW)
    elif shape == 'multiwave_c4':
        pair = pu.SampledPair(2048, [0, 1024, 2047], C4_FULL, seed=7103, device_scenario='static_same_goal',
                              source_factory=lambda: DeviceScenarioSource('static_same_goal'), chained=True,
                              rew_coeff=dict(quadcol_bin=5.0, quadcol_bin_smooth_max=10.0))
    elif shape == 'nz':
        pair = pu.Pair(6, dict(KW, sense_noise=NOISE), seed=7104, table_seed=7105)
        pair.ocfg.noise = sno.noise_model(NOISE)
    else:
        pair = pu.Pair(6, KW, seed=7106 + SHAPES.index(shape), table_seed=7110)
        if shape in ('wait', 'handover'):
            pair.engine.set_chained(True)               # the grid-wide wait / the per-block hand-over between step grids
    npo.enable(pair.ocfg)
    if shape == 'dyn':
        _drag_rows(pair)
    counts = dict(crashed_floor=0)
    rep = pu.run_parity(pair, 80, np.random.RandomState(31), resync=10, hook=lambda p, t: _plant_floor(p, t, counts))
    ds = [d for o in pair.oracles for d in o.drones]
    seen = dict(slides=sum(getattr(d, 'slides', 0) for d in ds), corner=sum(getattr(d, 'slide_corner', 0) for d in ds),
                landings=sum(getattr(d, 'landings_upside_down', 0) for d in ds),
                tries=sum(getattr(d, 'landing_yaw_tries', 0) for d in ds))
    frac = rep['skipped_env_steps'] / max(1, rep['skipped_env_steps'] + rep['compared_env_steps'])
    print(shape, rep, seen, counts, f'skipped {100 * frac:.1f} %')
    # drones resting on the floor lift off by micrometres whenever their random thrust exceeds their weight: those env-steps
    # decide the 0.05 m threshold within float32 resolution and are skipped (and re-synchronised), more of them with 32 drones
    assert rep['floor'] > 0 and counts['crashed_floor'] > 0 and frac <= (0.35 if pair.N <= 8 else 0.6), (rep, counts)
    assert seen['slides'] > 0 and seen['corner'] > 0 and seen['tries'] > seen['landings'] > 0, seen
    assert pair.engine.handover_timeouts == 0
    pair.engine.close()


def _engine(E, kw, seed=5, **extra):
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    kw = dict(kw)
    dev_scn = 'o_random' if kw.get('use_obstacles') else 'static_same_goal'
    return QuadSwarmEngine(num_envs=E, seed=seed, device_scenario=dev_scn, **kw, **extra)


def _acts(T, E, N, seed=0, lo=-1.0, hi=1.0):
    import torch
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    return (torch.rand((T, E, N, 4), device='cuda', generator=g) * (hi - lo) + lo).contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize('kw', [KW, C3_FULL, dict(KW, sense_noise=NOISE)], ids=['floor_obs', 'c3', 'noise'])
def test_rollout_equals_single_steps(kw):
    """rollout(T) gives, bit for bit, what T single steps give on the numpy path, through floor contacts and auto-resets
    (weak, lopsided thrust: the drones tumble onto the floor); the njit path gives something else."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    E, T, N = 256, 150, kw['num_agents']
    e1, e2, e3 = _engine(E, kw), _engine(E, kw), _engine(E, dict(kw, use_numba=True))
    a = _acts(T, E, N, seed=4, lo=-1.0, hi=0.2)
    e1.reset(); e2.reset(); e3.reset()
    obs1 = torch.empty((T, E, N, e1.D), device='cuda'); rew1 = torch.empty((T, E, N), device='cuda')
    dn1 = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    floor = 0
    for t in range(T):
        e1.step(a[t], obs_out=obs1[t], rewards_out=rew1[t], dones_out=dn1[t])
        floor += int(((e1.get_state()['agent_u32'][..., 0] & L.FLAG_CRASHED_FLOOR) != 0).sum())
    o2, r2, d2 = e2.rollout(a)
    o3, _, _ = e3.rollout(a)
    torch.cuda.synchronize()
    assert torch.equal(obs1, o2) and torch.equal(rew1, r2) and torch.equal(dn1, d2)
    assert int(dn1.sum()) > 0 and floor > E
    assert not torch.equal(o2, o3)
    s1, s2 = e1.get_state(), e2.get_state()
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        assert torch.equal(s1[k], s2[k]), k
    for e in (e1, e2, e3):
        e.close()


@pytest.mark.gpu
def test_sliding_drone_gains_speed_on_the_numpy_path():
    """A drone sliding on the floor under less thrust than its weight: the numpy path's friction points along the velocity
    and speeds it up; the njit path's points against it and slows it down (quadrotor_dynamics.py:419-422 / :601-604)."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    from quad_swarm_rl_b200.engine import STATE_F32_FIELDS as F
    speeds = {}
    for use_numba in (False, True):
        e = _engine(64, dict(num_agents=4, neighbor_visible_num=2, ep_time=15.0, sense_noise=None, use_numba=use_numba))
        e.reset()
        st = e.get_state()
        af, au = st['agent_f32'], st['agent_u32']
        af[..., F['pos'][0] + 2] = float(np.float32(ARM))          # on the floor in both paths
        af[..., F['vel'][0]:F['vel'][1]] = torch.tensor([0.5, 0.0, 0.0], device=af.device)
        af[..., F['rot'][0]:F['rot'][1]] = torch.eye(3, device=af.device).reshape(9)
        af[..., F['omega'][0]:F['omega'][1]] = 0.
        au[..., 0] = (au[..., 0] & ~(L.FLAG_ON_FLOOR | L.FLAG_CRASHED_FLOOR)) | L.FLAG_ON_FLOOR      # resting on it already
        e.set_state(st)
        a = torch.full((64, 4, 4), -0.5, device='cuda')
        for _ in range(10):
            e.step(a)
        v = e.get_state()['agent_f32'][..., F['vel'][0]].cpu().numpy()
        speeds[use_numba] = v
        e.close()
    assert np.all(speeds[False] > 0.6) and np.all(speeds[True] < 0.4), (speeds[False].min(), speeds[True].max())


@pytest.mark.gpu
def test_option_fixed_after_the_first_reset_and_off_is_the_default():
    """qs_set_numpy_dynamics fails once a reset ran; enable = 0 after enable = 1 gives the default path bit for bit."""
    import torch
    kw = dict(KW, use_numba=True)
    e1, e2 = _engine(128, kw), _engine(128, kw)
    assert e2.lib.qs_set_numpy_dynamics(e2.h, 1) == 0 and e2.lib.qs_set_numpy_dynamics(e2.h, 0) == 0
    a = _acts(60, 128, 8, seed=2, lo=-1.0, hi=0.2)
    e1.reset(); e2.reset()
    o1, r1, d1 = e1.rollout(a)
    o2, r2, d2 = e2.rollout(a)
    assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2)
    assert e1.lib.qs_set_numpy_dynamics(e1.h, 1) == -1 and b'first reset' in e1.lib.qs_last_error()
    e1.close(); e2.close()


@pytest.mark.gpu
def test_wrapped_steps_take_the_numpy_path():
    """The batched factory's wrapped steps (qs_wrap_step) with --quads_use_numba=False run the numpy path: the same config
    on the njit path gives the same reset and different steps once drones reach the floor."""
    import torch
    from quad_swarm_rl_b200.wrappers import make_quadrotor_env_multi_batched
    obs = {}
    for flag in (False, True):
        cfg = _cfg(quads_use_numba=flag, quads_num_agents=8, quads_obs_repr='xyz_vxyz_R_omega_floor', quads_use_downwash=True,
                   replay_buffer_sample_prob=0.0, quads_collision_reward=5.0, quads_collision_smooth_max_penalty=4.0,
                   quads_obst_collision_reward=5.0, anneal_collision_steps=0.0)
        env = make_quadrotor_env_multi_batched(cfg, num_envs=64)
        assert env.engine.use_numba is flag
        o0, _ = env.reset()
        g = torch.Generator(device='cuda')
        g.manual_seed(5)
        seq = [o0.clone()]
        for _ in range(95):                             # weak thrust: the drones fall to the floor within the episode
            o, *_ = env.step(torch.rand((env.num_agents, 4), device='cuda', generator=g) * 0.5 - 1)
            seq.append(o.clone())
        obs[flag] = seq
        env.close()
    assert torch.equal(obs[False][0], obs[True][0])
    assert not torch.equal(obs[False][-1], obs[True][-1])
