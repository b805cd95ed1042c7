"""The reference's other controllers (QuadrotorEnvMulti(raw_control=False): NonlinearPositionController; raw_control_zero_middle
=False: RawControl with actions in [0, 1]; include/quadswarm.h, qs_set_control): the oracle pinned to the reference's own
trajectories (tests/golden/control_*.npz, written by oracle/gen_golden_control.py), its Jinv against the reference's, the
action spaces and keyword handling, and on the GPU the kernels against the oracle, the bit-exact execution paths, the
wrapped step and what the controller does to the goal distance."""
import glob
import json
import os
import re

import numpy as np
import pytest

from oracle import control_oracle as co
from oracle import numpy_path_oracle as npo
from oracle import quadswarm_oracle as qo
from oracle import sensor_noise_oracle as sno

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
FILES = sorted(glob.glob(os.path.join(GOLDEN, 'control_*.npz')))
TOL = dict(rtol=1e-9, atol=1e-9)


def _make_scenario(mode, cfg, rng):
    from quad_swarm_rl_b200.scenarios import create_scenario
    sc = create_scenario(mode, cfg.num_agents, room_dims=cfg.room_dims, rng=np.random.RandomState(0),
                         ep_time=cfg.ep_time, use_obstacles=cfg.use_obstacles)
    sc.rng = rng
    return sc


def test_fixtures_present():
    assert [os.path.basename(f) for f in FILES] == ['control_c3_numpy_8.npz', 'control_corners_6.npz',
                                                    'control_randomquad_5.npz', 'control_raw_unit_wall_6.npz',
                                                    'control_swap_goals_8.npz']


_REPLAYS = {}


def _replay(path):
    """(replay output, oracle env, motor commands of every drone and step) of a fixture; cached."""
    if path not in _REPLAYS:
        cmds = []
        saved = co.position_command

        def recording(d, P):
            c = saved(d, P)
            cmds.append(c.copy())
            return c
        co.position_command = recording
        try:
            out, env = co.replay_control_golden(np.load(path, allow_pickle=False), _make_scenario)
        finally:
            co.position_command = saved
        _REPLAYS[path] = out, env, np.array(cmds)
    return _REPLAYS[path]


def _case(path):
    return json.loads(str(np.load(path, allow_pickle=False)['case_json']))


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[len('control_'):-4] for f in FILES])
def test_oracle_replays_reference_controllers(path):
    """Observations, rewards, reward terms, dones, goals, every recorded state and the episode statistics to 1e-9."""
    g = np.load(path, allow_pickle=False)
    out, env, _ = _replay(path)
    kw = _case(path)['kw']
    assert env.cfg.control == (co.POSITION if kw.get('raw_control', True) is False else co.RAW_UNIT)
    assert getattr(env.cfg, 'use_numba', True) is kw.get('use_numba', True)
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


def test_fixtures_exercise_the_controllers():
    """The fixtures hold what the controllers have to get right: saturated commands at both bounds, the clamp of the goal
    distance, upside-down attitudes, floor contacts, goal switches within an episode, actions beyond both bounds of [0, 1]."""
    _, env, cmds = _replay(os.path.join(GOLDEN, 'control_corners_6.npz'))
    assert (cmds == 0).any() and (cmds == 1).any() and ((cmds > 0) & (cmds < 1)).any()
    g = np.load(os.path.join(GOLDEN, 'control_corners_6.npz'))
    far = np.linalg.norm(g['goals'][:-1] - g['state_pos'][:-1], axis=-1) > 4.0
    assert far.any() and (g['state_rot'][..., 2, 2] < 0).any() and g['state_on_floor'].any()
    g = np.load(os.path.join(GOLDEN, 'control_swap_goals_8.npz'))
    ep = g['goals'][:251]
    assert (np.abs(np.diff(ep, axis=0)) > 0.1).any() and g['dones'][:, 0].sum() == 2
    g = np.load(os.path.join(GOLDEN, 'control_c3_numpy_8.npz'))
    infos = g['infos'][..., 16]                      # rewraw_quadcol_obstacle
    assert (infos < 0).any() and g['state_on_floor'].any()
    g = np.load(os.path.join(GOLDEN, 'control_raw_unit_wall_6.npz'))
    assert (g['actions'] < 0).any() and (g['actions'] > 1).any()
    g = np.load(os.path.join(GOLDEN, 'control_randomquad_5.npz'))
    assert len(np.unique(g['dyn_rows'][:, :, 0])) > 5     # masses: per drone and per episode


def _reference_or_skip():
    from oracle import ref_harness as rh
    if not rh.reference_available():
        pytest.skip('reference tree not available')
    return rh


@pytest.mark.parametrize('model', ['Crazyflie', 'DefaultQuad', 'MediumQuad', 'RandomQuad'])
def test_oracle_jinv_matches_the_reference(model):
    """The oracle's Jinv from the derived constants equals np.linalg.inv(quadrotor_jacobian(dynamics)) of the reference."""
    import contextlib
    import io
    rh = _reference_or_skip()
    from quad_swarm_rl_b200.quad_models import DYN_FIELDS
    np.random.seed(11)
    kw = dict(dyn_sampler_1={'class': 'RelativeSampler', 'noise_ratio': 0.05, 'sampler': 'normal'}) if model == 'RandomQuad' else {}
    env = rh.make_reference_env(num_agents=3, neighbor_visible_num=2, dynamics_params=model, **kw)
    from gym_art.quadrotor_multi.quadrotor_control import quadrotor_jacobian      # on the path once the env is built
    rows = rh.dynamics_rows(env)
    for e, row in zip(env.envs, rows):
        with contextlib.redirect_stdout(io.StringIO()):
            ref = np.linalg.inv(quadrotor_jacobian(e.dynamics))
        P = qo.QuadParams() if model == 'Crazyflie' else qo.quad_params_from_constants(dict(zip(DYN_FIELDS, [row[k] for k in DYN_FIELDS])))
        np.testing.assert_allclose(co.jacobian_inverse(P), ref, rtol=1e-12, atol=1e-12 * np.abs(ref).max())


@pytest.mark.parametrize('model', ['Crazyflie', 'DefaultQuad'])
@pytest.mark.parametrize('raw_control,zero_middle', [(True, True), (True, False), (False, True), (False, False)])
def test_action_spaces_equal_the_reference(model, raw_control, zero_middle):
    _reference_or_skip()
    import contextlib
    import io
    from quad_swarm_rl_b200 import quad_models as qm
    from quad_swarm_rl_b200.spaces import make_action_space
    from oracle.gen_golden_control import make_reference_env
    with contextlib.redirect_stdout(io.StringIO()):
        env = make_reference_env(num_agents=2, neighbor_visible_num=1, dynamics_params=model, raw_control=raw_control,
                                 raw_control_zero_middle=zero_middle)
    t2w = qm.SAMPLERS[model]().sample(rs=np.random.RandomState(0))['motor']['thrust_to_weight']
    mine = make_action_space(raw_control, zero_middle, t2w)
    assert np.array_equal(mine.low, env.action_space.low) and np.array_equal(mine.high, env.action_space.high)
    assert mine.dtype == env.action_space.dtype


def test_default_action_space_is_unchanged():
    from quad_swarm_rl_b200.spaces import make_action_space
    s = make_action_space()
    assert np.array_equal(s.low, -np.ones(4, np.float32)) and np.array_equal(s.high, np.ones(4, np.float32))


class _Captured(Exception):
    pass


@pytest.mark.parametrize('raw_control,zero_middle', [(True, True), (True, False), (False, True), (False, False)])
def test_env_objects_forward_the_controller_keywords(raw_control, zero_middle, monkeypatch):
    from quad_swarm_rl_b200 import env as env_mod

    def fake(**kw):
        raise _Captured(kw)
    monkeypatch.setattr(env_mod, 'QuadSwarmEngine', fake)
    kw = dict(num_agents=4, ep_time=1.0, rew_coeff=None, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=2,
              neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0, use_obstacles=False,
              obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0], use_downwash=False, use_numba=True,
              quads_mode='static_same_goal', room_dims=[10., 10., 10.], use_replay_buffer=False, quads_view_mode=['topdown'],
              quads_render=False, dynamics_params='Crazyflie', raw_control=raw_control, raw_control_zero_middle=zero_middle,
              dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
              init_random_state=False, seed=3)
    for make in (lambda: env_mod.QuadrotorEnvMulti(**kw),
                 lambda: env_mod.QuadrotorEnvMultiBatched(num_envs=2, num_agents=4, raw_control=raw_control,
                                                          raw_control_zero_middle=zero_middle, seed=3)):
        with pytest.raises(_Captured) as e:
            make()
        assert e.value.args[0]['raw_control'] is raw_control and e.value.args[0]['raw_control_zero_middle'] is zero_middle
    with pytest.raises(_Captured) as e:
        env_mod.QuadrotorEnvMultiBatched(num_envs=2, num_agents=4, seed=3)
    assert e.value.args[0]['raw_control'] is True and e.value.args[0]['raw_control_zero_middle'] is True


def test_header_declares_and_lib_binds_the_entry_point():
    import ctypes
    from quad_swarm_rl_b200 import _lib as L
    hdr = open(os.path.join(ROOT, 'include', 'quadswarm.h')).read()
    decl = re.search(r'int qs_set_control\(([^)]*)\);', hdr).group(1)
    assert [a.strip().rsplit(' ', 1)[0] for a in decl.split(',')] == ['QsHandle*', 'int']
    for name, v in (('QS_CONTROL_RAW', 0), ('QS_CONTROL_RAW_UNIT', 1), ('QS_CONTROL_POSITION', 2)):
        assert re.search(rf'#define {name} {v}\b', hdr) and getattr(L, name) == v
    assert L.EXPORTS['qs_set_control'] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int])


def test_entry_point_rejects_a_null_handle_without_gpu():
    import sys
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from quad_swarm_rl_b200 import _lib as L
    lib = L.load()
    assert lib.qs_set_control(None, 2) == -1 and b'null' in lib.qs_last_error()


def test_control_kernels_instantiate_the_grid_wide_wait_shape_only():
    """Per dynamics path: NP in {1, ..., 32} x SCN x DYN x NZ, never the split or hand-over shapes; no local memory beyond
    the stack frame."""
    from tests.parity_util import kernel_resources
    usage = kernel_resources(r'qs_step_kernel_pc(_npy)?ILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE')
    for npy in (False, True):
        keys = sorted(k[1:] for k in usage if bool(k[0]) is npy)
        assert keys == sorted((NP, 0, scn, 0, dyn, nz) for NP in (1, 2, 4, 8, 16, 32) for scn in (0, 1)
                              for dyn in (0, 1) for nz in (0, 1))
    for k, v in usage.items():
        assert v['LOCAL'] == 0, (k, v)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
C2 = dict(num_agents=8, neighbor_visible_num=6, ep_time=1.0)
C3 = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True, use_downwash=True,
          ep_time=1.0)
C3_REW = dict(quadcol_bin=5.0, quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
NOISE = dict(gyro_norm_std=0.1, quat_norm_std=0.01, pos_unif_range=0.01)
MODES = {'position': dict(raw_control=False), 'raw_unit': dict(raw_control_zero_middle=False)}


def _random_rows(pair, seed):
    """RandomQuad + RelativeSampler constants for every drone (qs_set_dynamics -> DYN kernels), on both sides."""
    from quad_swarm_rl_b200.quad_models import DYN_FIELDS, DynamicsSource
    rs = np.random.RandomState(seed)
    src = DynamicsSource('RandomQuad', None, {'class': 'RelativeSampler', 'noise_ratio': 0.05, 'sampler': 'normal'}, rs=rs)
    rows = np.stack([src.sample_row() for _ in range(pair.engine.E * pair.N)]).reshape(pair.engine.E, pair.N, -1)
    pair.engine.set_dynamics(rows.astype(np.float32))
    for e, o in enumerate(pair.oracles):
        o.Ps = [qo.quad_params_from_constants(dict(zip(DYN_FIELDS, r.astype(np.float32).astype(np.float64)))) for r in rows[e]]
        o.P = o.Ps[0]


PARITY = [
    ('position', 'c2_wait', False), ('position', 'numpy_floor', False), ('position', 'dyn_randomquad', False),
    ('position', 'nz_gyro_bias', False), ('position', 'numpy_dyn_nz', False), ('position', 'swap_goals_device', False),
    ('position', 'c2_full', True), ('position', 'c3_full', True), ('position', 'c3_full_unchained', True),
    ('raw_unit', 'c2_wait', False), ('raw_unit', 'numpy_floor', False), ('raw_unit', 'dyn_randomquad', False),
    ('raw_unit', 'c3_full', True),
]


@pytest.mark.gpu
@pytest.mark.parametrize('mode,case,full', PARITY, ids=[f'{m}-{c}' for m, c, _ in PARITY])
def test_kernel_matches_oracle(mode, case, full):
    """Kernel (keyed draws) against the oracle with each controller: small configs on both dynamics paths, per-drone RandomQuad
    constants (DYN), a noise dict with the gyro bias (NZ), a device scenario with goal events and auto-resets, and full-size
    c2 (8 x 1024) / c3 (8 x 4096) grids, chained and unchained, checked on sampled envs.  States within 1e-4 + 1e-4 |ref|
    with teacher forcing every 20 steps, masks bit-exact under the threshold-margin rule."""
    from oracle.scenario_gen import DeviceORandomSource, DeviceScenarioSource
    from tests import parity_util as pu
    ctl = MODES[mode]
    rew = None
    if case == 'c2_full':
        pair = pu.SampledPair(1024, [0, 511, 1023], dict(C2, **ctl), seed=8101, device_scenario='swap_goals',
                              source_factory=lambda: DeviceScenarioSource('swap_goals'), chained=True)
    elif case in ('c3_full', 'c3_full_unchained'):
        pair = pu.SampledPair(4096, [0, 2048, 4095], dict(C3, **ctl), seed=8102, device_scenario='o_random',
                              source_factory=lambda: DeviceORandomSource(), chained=case == 'c3_full', rew_coeff=C3_REW)
        rew = C3_REW
    elif case == 'swap_goals_device':
        pair = pu.DevicePair(16, dict(C2, ep_time=2.5, **ctl), seed=8103, device_scenario='swap_goals',
                             source_factory=lambda: DeviceScenarioSource('swap_goals'))
    else:
        kw = dict(C3 if case == 'numpy_floor' else C2, **ctl)
        if case in ('numpy_floor', 'numpy_dyn_nz'):
            kw['use_numba'] = False
        if case in ('nz_gyro_bias', 'numpy_dyn_nz'):
            kw['sense_noise'] = NOISE
        pair = pu.Pair(6, kw, seed=8110 + [c for _, c, _ in PARITY].index(case), table_seed=8120,
                       rew_coeff=C3_REW if case == 'numpy_floor' else None)
        if case == 'c2_wait':
            pair.engine.set_chained(True)
        if 'sense_noise' in kw:
            pair.ocfg.noise = sno.noise_model(NOISE)
        if case in ('dyn_randomquad', 'numpy_dyn_nz'):
            _random_rows(pair, 8130)
    if pair.kw.get('use_numba', True) is False:
        npo.enable(pair.ocfg)
    co.enable(pair.ocfg, **ctl)
    assert rew is None or pair.ocfg.rew_coeff['quadcol_bin_smooth_max'] == 4.0
    T = 270 if case == 'swap_goals_device' else 120
    rep = pu.run_parity(pair, T, np.random.RandomState(41), resync=20, action_scale=1.5 if mode == 'raw_unit' else 1.0)
    print(mode, case, rep)
    assert rep['steps'] == T and rep['dones'] >= 1 and rep['compared_env_steps'] > 0.5 * T * pair.E, rep
    assert pair.engine.handover_timeouts == 0
    pair.engine.close()


def _engine(E, kw, seed=5, **extra):
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    kw = dict(kw)
    dev_scn = 'o_random' if kw.get('use_obstacles') else 'swap_goals'
    return QuadSwarmEngine(num_envs=E, seed=seed, device_scenario=dev_scn, **kw, **extra)


def _acts(T, E, N, seed=0, lo=-1.0, hi=1.0):
    import torch
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    return (torch.rand((T, E, N, 4), device='cuda', generator=g) * (hi - lo) + lo).contiguous()


EXEC = [('position', C2), ('position', dict(C3, use_numba=False)), ('raw_unit', C3), ('raw_unit', dict(C2, use_numba=False))]


@pytest.mark.gpu
@pytest.mark.parametrize('mode,kw', EXEC, ids=['position-c2', 'position-c3-numpy', 'raw_unit-c3', 'raw_unit-c2-numpy'])
def test_execution_paths_are_bit_exact(mode, kw):
    """rollout(T) == T single steps; a CUDA graph of T chained steps == one rollout; the host-buffer entry point == the
    device one — bit for bit, through goal events and auto-resets.  The default controller gives something else."""
    import torch
    E, T, N = 512, 120, kw['num_agents']
    kw = dict(kw, **MODES[mode])
    e1, e2, e3, e4 = (_engine(E, kw) for _ in range(4))
    e0 = _engine(E, {k: v for k, v in kw.items() if k not in MODES[mode]})
    a = _acts(T, E, N, seed=4, lo=-0.5, hi=1.5)
    for e in (e0, e1, e2, e3, e4):
        e.reset()
    obs1 = torch.empty((T, E, N, e1.D), device='cuda'); rew1 = torch.empty((T, E, N), device='cuda')
    dn1 = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    for t in range(T):
        e1.step(a[t], obs_out=obs1[t], rewards_out=rew1[t], dones_out=dn1[t])
    o2, r2, d2 = e2.rollout(a)
    o0, _, _ = e0.rollout(a)
    torch.cuda.synchronize()
    assert torch.equal(obs1, o2) and torch.equal(rew1, r2) and torch.equal(dn1, d2)
    assert int(dn1.sum()) > 0 and not torch.equal(o2, o0)
    # a CUDA graph of chained steps (after three warm-up steps outside the capture)
    e3.set_chained(True)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    obs3 = torch.empty_like(obs1); rew3 = torch.empty_like(rew1); dn3 = torch.empty_like(dn1)
    with torch.cuda.stream(st):
        for t in range(3):
            e3.step(a[t], obs_out=obs3[t], rewards_out=rew3[t], dones_out=dn3[t])
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for t in range(3, T):
                e3.step(a[t], obs_out=obs3[t], rewards_out=rew3[t], dones_out=dn3[t])
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(obs3, o2) and torch.equal(rew3, r2) and torch.equal(dn3, d2)
    # host buffers
    an = a.cpu().numpy()
    ob = np.empty((E, N, e4.D), np.float32); rw = np.empty((E, N), np.float32); dn = np.empty((E, N), np.uint8)
    for t in range(T):
        e4.step_host(an[t], ob, rw, dn)
    assert np.array_equal(ob, o2[-1].cpu().numpy()) and np.array_equal(rw, r2[-1].cpu().numpy())
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        s = e2.get_state()[k]
        assert torch.equal(e1.get_state()[k], s) and torch.equal(e3.get_state()[k], s) and torch.equal(e4.get_state()[k], s), k
    for e in (e0, e1, e2, e3, e4):
        e.close()


@pytest.mark.gpu
def test_set_control_is_checked_and_raw_is_the_default():
    """Unknown modes and calls after the first reset fail with QS_ERR_INVALID_ARG; QS_CONTROL_RAW set explicitly gives the
    default bit for bit."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    e1, e2 = _engine(128, C2), _engine(128, C2)
    assert e2.lib.qs_set_control(e2.h, 3) == -1 and b'unknown control mode' in e2.lib.qs_last_error()
    assert e2.lib.qs_set_control(e2.h, -1) == -1
    assert e2.lib.qs_set_control(e2.h, L.QS_CONTROL_POSITION) == 0 and e2.lib.qs_set_control(e2.h, L.QS_CONTROL_RAW) == 0
    a = _acts(60, 128, 8, seed=2)
    e1.reset(); e2.reset()
    o1, r1, d1 = e1.rollout(a)
    o2, r2, d2 = e2.rollout(a)
    assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2)
    for e in (e1, e2):
        assert e.lib.qs_set_control(e.h, L.QS_CONTROL_POSITION) == -1 and b'first reset' in e.lib.qs_last_error()
        e.close()


@pytest.mark.gpu
def test_wrapped_steps_with_the_controller():
    """qs_wrap_step (training.BatchedTrainingEnv) with the controller: the wrappers do not perturb the env, and their
    statistics are those of the unwrapped terms and of the raw caller actions."""
    import torch
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    from quad_swarm_rl_b200.training import BatchedTrainingEnv
    mk = lambda: QuadrotorEnvMultiBatched(num_envs=24, num_agents=8, ep_time=0.4, seed=5, raw_control=False,
                                          quads_mode='static_same_goal')
    env, twin = mk(), mk()
    w = BatchedTrainingEnv(env, reward_shaping_scheme=dict(quad_rewards=dict(pos=1.0)), stats_every=1 << 30)
    w.reset(); twin.reset()
    E, N = 24, 8
    raw_sum = torch.zeros((E, N, 8), device='cuda')
    acts = []
    g = torch.Generator(device='cuda'); g.manual_seed(1)
    for t in range(41):
        a = torch.rand((E * N, 4), device='cuda', generator=g) * 2 - 1
        obs, rew, term, trunc, infos = w.step(a)
        o2, r2, t2, _, _ = twin.step(a, with_terms=True)
        assert torch.equal(obs, o2) and torch.equal(rew, r2) and torch.equal(term, t2)
        raw_sum += twin.engine.rew_terms
        acts.append(a.view(E, N, 4))
        if term.any():
            break
    assert t == 40 and term.all()
    st = w.flush_stats()['episode_extra_stats']
    np.testing.assert_allclose(st['rewraw_pos'], raw_sum[..., 0].mean().item(), rtol=1e-5)
    np.testing.assert_allclose(st['rewraw_action'], raw_sum[..., 1].mean().item(), rtol=1e-5)
    np.testing.assert_allclose(st['z_action2_mean'], torch.stack(acts)[..., 2].mean().item(), atol=1e-5)
    env.close(); twin.close()


@pytest.mark.gpu
def test_controller_flies_the_drones_to_their_goals():
    """Under the controller the mean goal distance of 256 envs falls over an episode, as in the reference, and follows the
    oracle's (the oracle on the keyed draws of the first envs, without teacher forcing)."""
    import torch
    from oracle.scenario_gen import DeviceScenarioSource
    from tests import parity_util as pu
    pair = pu.SampledPair(256, list(range(4)), dict(num_agents=4, neighbor_visible_num=2, ep_time=2.0, raw_control=False),
                          seed=8201, device_scenario='static_same_goal',
                          source_factory=lambda: DeviceScenarioSource('static_same_goal'))
    co.enable(pair.ocfg, raw_control=False)
    pair.reset()
    zero = np.zeros((4, 4, 4), np.float32)
    dev, orc = [], []
    for t in range(150):
        pair.step(zero)
        f = pair.engine.get_state()['agent_f32']
        from quad_swarm_rl_b200.engine import STATE_F32_FIELDS as F
        pos = f[..., F['pos'][0]:F['pos'][1]]
        goal = f[..., F['goal'][0]:F['goal'][1]]
        dev.append(float(torch.linalg.norm(goal - pos, dim=-1).mean()))
        orc.append(float(np.mean([np.linalg.norm(d.goal[:3] - d.pos) for o in pair.oracles for d in o.drones])))
    dev, orc = np.array(dev), np.array(orc)
    print('goal distance', dev[[0, 50, 100, 149]], orc[[0, 50, 100, 149]])
    assert dev[-1] < 0.5 * dev[0] and orc[-1] < 0.5 * orc[0]
    assert np.abs(dev[-1] - orc[-1]) < 0.1 + 0.2 * orc[-1]
    pair.engine.close()
