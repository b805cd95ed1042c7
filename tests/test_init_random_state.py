"""Random initial states (init_random_state=True, quadrotor_single.py:405-423; include/quadswarm.h, qs_set_init_random_state):
the oracle pinned to the reference's own trajectories (tests/golden/init_state_*.npz, written by
oracle/gen_golden_init_state.py), the distributions of the keyed draws, the host-side keyword handling, and on the GPU the
kernels against the oracle in every launch shape, the bit-exact equivalences of the launch paths with the option on, and
full-size statistics of the spawn states the kernels draw."""
import ctypes
import glob
import os
import re
import subprocess

import numpy as np
import pytest
from scipy import stats

from oracle import init_state_oracle as iso
from oracle import quadswarm_oracle as qo
from oracle import sensor_noise_oracle as sno

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
FILES = sorted(glob.glob(os.path.join(GOLDEN, 'init_state_*.npz')))
TOL = dict(rtol=1e-9, atol=1e-9)
TWO_PI = 2 * np.pi


def _make_scenario(mode, cfg, rng):
    from quad_swarm_rl_b200.scenarios import create_scenario
    sc = create_scenario(mode, cfg.num_agents, room_dims=cfg.room_dims, rng=np.random.RandomState(0),
                         ep_time=cfg.ep_time, use_obstacles=cfg.use_obstacles)
    sc.rng = rng
    return sc


def test_fixtures_present():
    assert len(FILES) >= 4, FILES


_REPLAYS = {}


def _replay(path):
    if path not in _REPLAYS:
        _REPLAYS[path] = iso.replay_init_state_golden(np.load(path, allow_pickle=False), _make_scenario)
    return _REPLAYS[path]


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[len('init_state_'):-4] for f in FILES])
def test_oracle_replays_reference_with_random_initial_states(path):
    g = np.load(path, allow_pickle=False)
    out, env = _replay(path)
    assert env.cfg.init_random_state and env.init_resets >= 4 * env.num_agents      # explicit reset + >= 3 auto-resets
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


def test_fixtures_exercise_random_initial_states():
    """Every fixture runs through >= 3 auto-resets with moving, spinning spawns; together they hold upside-down spawns
    (R[2,2] < 0), fwd re-draws of rand_uniform_rot3d (counted by the oracle, whose replay of the reference's numpy stream
    would lose step at the first re-draw it missed or invented), and drones on the floor within 40 steps of their spawn
    (not planted there)."""
    seen = dict(inverted=0, redraw=0, floor=0)
    for path in FILES:
        g = np.load(path)
        assert list(g['obs_t']) == list(g['state_t']) == list(range(len(g['obs_t'])))
        done = np.where(g['dones'][:, 0])[0]
        assert len(done) >= 3, path
        # spawn states: the explicit reset (its observation) and the state after every auto-reset
        rot = np.concatenate([g['obs0'][:, 6:15].reshape(-1, 3, 3), g['state_rot'][done].reshape(-1, 3, 3)])
        vel = np.concatenate([g['obs0'][:, 3:6], g['state_vel'][done].reshape(-1, 3)])
        om = g['state_omega'][done].reshape(-1, 3)
        assert np.all(np.linalg.norm(vel, axis=1) > 0) and np.all(np.linalg.norm(om, axis=1) > 0), path
        assert np.linalg.norm(om, axis=1).max() <= TWO_PI * (1 + 1e-6) and np.linalg.norm(g['state_vel'][done], axis=2).max() <= 1 + 1e-6
        seen['inverted'] += int(np.sum(rot[:, 2, 2] < 0))
        seen['redraw'] += _replay(path)[1].init_redraws
        for s in [0] + [int(t) + 1 for t in done]:
            planted = set(int(i) for t, i in zip(g['plant_t'], g['plant_i']) if s <= t < s + 40)
            floor = g['state_on_floor'][s:s + 40].any(axis=0)
            seen['floor'] += sum(1 for i in np.where(floor)[0] if i not in planted)
    print(seen)
    assert all(v > 0 for v in seen.values()), seen


def _keyed_spawns(n, vel_max=1.0, omega_max=TWO_PI):
    """n spawn states from the keyed generator (PhiloxRng, the kernels' draws): drones 0..7 of envs / episodes."""
    rng = qo.PhiloxRng(20261015)
    out, tries = [], 0
    for k in range(n // 8):
        rng.begin_episode(k % 97, 1 + k // 97)
        for i in range(8):
            vel, rot, om, t, _ = iso.random_state(rng, i, vel_max, omega_max)
            out.append((vel, rot, om))
            tries += t - 1
    return out, tries


def test_keyed_draws_follow_the_reference_distributions():
    """|vel| ~ U(0, vel_max), |omega| ~ U(0, omega_max); R is Haar-uniform (the re-draw rule keeps the joint law of (up, fwd)
    rotation invariant), so the z components of its columns are U(-1, 1); R is orthonormal in float64."""
    spawns, redraws = _keyed_spawns(4000)
    vel = np.array([s[0] for s in spawns])
    rot = np.array([s[1] for s in spawns])
    om = np.array([s[2] for s in spawns])
    assert stats.kstest(np.linalg.norm(vel, axis=1), 'uniform', args=(0, 1)).pvalue > 1e-3
    assert stats.kstest(np.linalg.norm(om, axis=1), 'uniform', args=(0, TWO_PI)).pvalue > 1e-3
    for col in (0, 1, 2):
        assert stats.kstest(rot[:, 2, col], 'uniform', args=(-1, 2)).pvalue > 1e-3, col
    assert np.abs(np.einsum('nji,njk->nik', rot, rot) - np.eye(3)).max() < 1e-12
    assert np.all(np.abs(vel) <= 1.0) and np.all(np.abs(om) <= TWO_PI)
    assert 10 <= redraws <= 200, redraws                  # p(re-draw) = P(fwd.up > 0.95) = 2.5 %
    assert np.mean(rot[:, 2, 2] < 0) == pytest.approx(0.5, abs=0.03)


def test_reference_order_of_the_numpy_draws():
    """ReplayRng consumes numpy's global stream in random_state's order (quadrotor_dynamics.py:193-206): 3 discarded
    position uniforms, vel (3 + 1), omega (3 + 1), then rand_uniform_rot3d's normals (quad_utils.py:94-104), restated here
    with numpy's own vector calls."""
    for seed in range(40):
        rng = qo.ReplayRng(seed, seed + 1, [0])
        vel, rot, om, tries, _ = iso.random_state(rng, 0)
        rs = np.random.RandomState(seed)
        rs.uniform(low=-np.array([10., 10., 10.]), high=np.array([10., 10., 10.]), size=(3,))
        v = rs.uniform(low=-1.0, high=1.0, size=(3,))
        v = rs.uniform(low=0., high=1.0) / (np.linalg.norm(v) + 1e-6) * v
        w = rs.uniform(low=-TWO_PI, high=TWO_PI, size=(3,))
        w = rs.uniform(low=0., high=TWO_PI) / (np.linalg.norm(w) + 1e-6) * w
        unit = lambda: (lambda x: x / (x[0] ** 2 + x[1] ** 2 + x[2] ** 2) ** 0.5)(rs.normal(size=(3,)))
        up, fwd, t = unit(), unit(), 1
        while np.dot(fwd, up) > 0.95:
            fwd, t = unit(), t + 1
        left = np.cross(up, fwd)
        left = left / (left[0] ** 2 + left[1] ** 2 + left[2] ** 2) ** 0.5
        np.testing.assert_array_equal(vel, v)
        np.testing.assert_array_equal(om, w)
        np.testing.assert_allclose(rot, np.column_stack([fwd, left, np.cross(fwd, left)]), rtol=0, atol=1e-15)
        assert tries == t
        assert rng.py.random_sample() == rs.random_sample()          # both streams end at the same place


# ---- host-side keyword handling and the C ABI (no GPU)
def test_env_objects_accept_init_random_state():
    """QuadrotorEnvMulti(..., init_random_state=True) passes the keyword check (it used to raise NotImplementedError);
    without a GPU the engine then refuses to start."""
    import torch
    from quad_swarm_rl_b200.env import QuadrotorEnvMulti, QuadrotorEnvMultiBatched
    kw = dict(num_agents=4, ep_time=1.0, rew_coeff=None, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=2,
              neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0, use_obstacles=False,
              obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0], use_downwash=False, use_numba=True,
              quads_mode='static_same_goal', room_dims=[10., 10., 10.], use_replay_buffer=False, quads_view_mode=['topdown'],
              quads_render=False, dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
              dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
              init_random_state=True, seed=3)
    if torch.cuda.is_available():
        env = QuadrotorEnvMulti(**kw)
        assert env.engine.init_random_state
        env.close()
        env = QuadrotorEnvMultiBatched(num_envs=2, num_agents=4, init_random_state=True, seed=3)
        assert env.engine.init_random_state
        env.close()
    else:
        for make in (lambda: QuadrotorEnvMulti(**kw),
                     lambda: QuadrotorEnvMultiBatched(num_envs=2, num_agents=4, init_random_state=True, seed=3)):
            with pytest.raises(RuntimeError, match='CUDA device'):
                make()


def _c_values(tmp_path, exprs):
    src = tmp_path / 'v.c'
    fmt = ' '.join(['%lld'] * len(exprs))
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "quadswarm.h"\nint main(){printf("' + fmt + '\\n", ' +
                   ', '.join(f'(long long)({e})' for e in exprs) + ');return 0;}\n')
    exe = tmp_path / 'v'
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    return [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]


def test_abi_layouts_unchanged_and_prototype_matches_header(tmp_path):
    """The option adds one entry point: QsConfig's layout and the QS_STATE_* row sizes are those of the previous release,
    and the ctypes prototype follows the header's declaration."""
    from quad_swarm_rl_b200 import _lib as L
    vals = _c_values(tmp_path, ['sizeof(QsConfig)', 'offsetof(QsConfig, seed)', 'QS_STATE_F32', 'QS_STATE_U32',
                                'QS_STATE_ENV_I32'])
    assert vals == [ctypes.sizeof(L.QsConfig), L.QsConfig.seed.offset, L.QS_STATE_F32, L.QS_STATE_U32, L.QS_STATE_ENV_I32]
    assert vals == [104, 80, 43, 4, 36]
    hdr = open(os.path.join(ROOT, 'include', 'quadswarm.h')).read()
    decl = re.search(r'int qs_set_init_random_state\(([^)]*)\);', hdr).group(1)
    assert [a.strip().rsplit(' ', 1)[0] for a in decl.split(',')] == ['QsHandle*', 'int', 'float', 'float']
    assert L.EXPORTS['qs_set_init_random_state'] == (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_float])


def test_entry_point_rejects_bad_arguments_without_gpu():
    import sys
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from quad_swarm_rl_b200 import _lib as L
    lib = L.load()
    assert lib.qs_set_init_random_state(None, 1, 1.0, TWO_PI) == -1 and b'null' in lib.qs_last_error()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
KW_SAME = dict(num_agents=8, neighbor_visible_num=6, ep_time=0.4)
KW_C3 = dict(num_agents=8, neighbor_visible_num=2, ep_time=0.5, use_obstacles=True, use_downwash=True,
             obs_repr='xyz_vxyz_R_omega_floor')
NOISE = dict(pos_unif_range=0.01, quat_norm_std=0.01, gyro_noise_density=0.001)
KW_WALL = dict(num_agents=6, neighbor_visible_num=2, ep_time=0.4, obs_repr='xyz_vxyz_R_omega_wall', sense_noise=NOISE)
KW_DQ = dict(num_agents=4, neighbor_visible_num=2, ep_time=0.4)
C3_REW = dict(quadcol_bin=5.0, quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)


def _on(kw):
    return dict(kw, init_random_state=True)


def _arm_oracles(pair, kw):
    """Attach the option (and a noise dict's model) to the oracle config every oracle env of the pair shares."""
    iso.enable(pair.ocfg)
    if isinstance(kw.get('sense_noise'), dict):
        pair.ocfg.noise = sno.noise_model(kw['sense_noise'])
    return pair


def _defaultquad(pair):
    """Every drone flies DefaultQuad (qs_set_dynamics), on both sides."""
    from quad_swarm_rl_b200 import quad_models as qm
    from quad_swarm_rl_b200.quad_models import DYN_FIELDS
    row = qm.constants_row(qm.defaultquad_params())
    rows = np.broadcast_to(row, (pair.engine.E, pair.N, len(row))).astype(np.float32).copy()
    pair.engine.set_dynamics(rows)
    P = qo.quad_params_from_constants(dict(zip(DYN_FIELDS, row.astype(np.float32).astype(np.float64))))
    for o in pair.oracles:
        o.Ps = [P] * pair.N
        o.P = P


def _report(name, pair, rep):
    resets = sum(getattr(o, 'init_resets', 0) for o in pair.oracles)
    near = sum(getattr(o, 'init_near', 0) for o in pair.oracles)
    frac = rep['skipped_env_steps'] / max(1, rep['skipped_env_steps'] + rep['compared_env_steps'])
    print(f'{name}: {rep}; drone resets {resets}, fwd re-draws {sum(getattr(o, "init_redraws", 0) for o in pair.oracles)}, '
          f'near the re-draw threshold {near} ({100 * near / max(1, resets):.3f} %); skipped env-steps {100 * frac:.2f} %')
    return resets, frac


def _device_pair(kw, E, seed):
    from oracle.scenario_gen import DeviceORandomSource, DeviceScenarioSource
    from tests import parity_util as pu
    if kw.get('use_obstacles'):
        return pu.DevicePair(E, _on(kw), seed, 'o_random', lambda: DeviceORandomSource())
    mode = 'static_diff_goal' if kw is KW_WALL or kw is KW_DQ else 'static_same_goal'
    return pu.DevicePair(E, _on(kw), seed, mode, lambda: DeviceScenarioSource(mode))


@pytest.mark.gpu
@pytest.mark.parametrize('source', ['host_tables', 'device'])
@pytest.mark.parametrize('name', ['same_goal_8', 'c3_obstacles_8', 'wall_noise_6', 'defaultquad_4'])
def test_kernel_matches_oracle_with_random_initial_states(name, source):
    """The four golden configurations (wall_noise_6: the custom noise model, NZ kernels; defaultquad_4: per-drone
    constants, DYN kernels), host tables and device-side scenarios, through auto-resets and two explicit resets."""
    from tests import parity_util as pu
    kw = dict(same_goal_8=KW_SAME, c3_obstacles_8=KW_C3, wall_noise_6=KW_WALL, defaultquad_4=KW_DQ)[name]
    E, seed = 8, 4100 + len(name)
    pair = pu.Pair(E, _on(kw), seed=seed, table_seed=seed + 1) if source == 'host_tables' else _device_pair(kw, E, seed)
    _arm_oracles(pair, kw)
    if name == 'defaultquad_4':
        _defaultquad(pair)
    total = dict(dones=0, floor=0, skipped=0, compared=0)
    for r in range(2):                                  # run_parity starts with an explicit reset
        if r and source == 'host_tables':               # the second run walks the tables from the first again, on both sides
            pair._push_table(0)
            for o in pair.oracles:
                o.source.k = -1
        rep = pu.run_parity(pair, 100, np.random.RandomState(seed + r), resync=10)
        for k, k2 in (('dones', 'dones'), ('floor', 'floor'), ('skipped', 'skipped_env_steps'), ('compared', 'compared_env_steps')):
            total[k] += rep[k2]
        _report(f'{name}/{source} run {r}', pair, rep)
    resets, _ = _report(name, pair, dict(rep, skipped_env_steps=total['skipped'], compared_env_steps=total['compared']))
    assert total['dones'] >= 2 * E and resets == (2 * E + total['dones']) * pair.N, (total, resets)
    assert total['skipped'] <= 0.10 * (total['skipped'] + total['compared']), total
    pair.engine.close()


def _engine(E, kw, seed=5, **extra):
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    kw = dict(kw)
    dev_scn = 'o_random' if kw.get('use_obstacles') else 'static_same_goal'
    return QuadSwarmEngine(num_envs=E, seed=seed, device_scenario=dev_scn, **kw, **extra)


def _acts(T, E, N, seed=0):
    import torch
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    return (torch.rand((T, E, N, 4), device='cuda', generator=g) * 2 - 1).contiguous()


def _state_equal(e1, e2):
    import torch
    s1, s2 = e1.get_state(), e2.get_state()
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        assert torch.equal(s1[k], s2[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('kw', [KW_SAME, KW_C3, KW_WALL], ids=['same_goal', 'c3', 'noise'])
def test_rollout_equals_steps_and_host_buffers_and_shards(kw):
    """With the option on, across auto-resets: rollout(T) == T single steps; qs_step_host == qs_step on device buffers;
    two shards (env_id_offset) == one engine."""
    import torch
    E, T, N = 64, 90, kw['num_agents']
    e1, e2, host = _engine(E, _on(kw)), _engine(E, _on(kw)), _engine(E, _on(kw))
    s0, s1 = _engine(E // 2, _on(kw)), _engine(E // 2, _on(kw), env_id_offset=E // 2)
    a = _acts(T, E, N, seed=3)
    e1.reset(); e2.reset(); s0.reset(); s1.reset()
    obs_np = np.zeros((E, N, host.D), np.float32)
    host.reset_host(obs_np)
    assert np.array_equal(obs_np, e1.obs.cpu().numpy())
    assert torch.equal(torch.cat([s0.obs, s1.obs]), e1.obs)
    rew_np, dn_np = np.zeros((E, N), np.float32), np.zeros((E, N), np.uint8)
    obs1 = torch.empty((T, E, N, e1.D), device='cuda'); rew1 = torch.empty((T, E, N), device='cuda')
    dn1 = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    for t in range(T):
        e1.step(a[t], obs_out=obs1[t], rewards_out=rew1[t], dones_out=dn1[t])
        host.step_host(a[t].cpu().numpy(), obs_np, rew_np, dn_np)
        o0, r0, d0 = s0.step(a[t, :E // 2].contiguous())
        o1, r1, d1 = s1.step(a[t, E // 2:].contiguous())
        assert np.array_equal(obs_np, obs1[t].cpu().numpy()) and np.array_equal(rew_np, rew1[t].cpu().numpy()), t
        assert torch.equal(torch.cat([o0, o1]), obs1[t]) and torch.equal(torch.cat([r0, r1]), rew1[t]), t
        assert torch.equal(torch.cat([d0, d1]), dn1[t]), t
    o2, r2, d2 = e2.rollout(a)
    torch.cuda.synchronize()
    assert torch.equal(obs1, o2) and torch.equal(rew1, r2) and torch.equal(dn1, d2)
    assert int(dn1.sum()) > 0
    _state_equal(e1, e2)
    _state_equal(e1, host)
    for e in (e1, e2, host, s0, s1):
        e.close()


C2_FULL = dict(num_agents=8, neighbor_visible_num=6, obs_repr='xyz_vxyz_R_omega')
C3_FULL = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True, use_downwash=True)
C4_FULL = dict(num_agents=32, neighbor_visible_num=6, obs_repr='xyz_vxyz_R_omega')


@pytest.mark.gpu
@pytest.mark.parametrize('name,kw,E,dev_scn,pdl,chained', [
    ('c3_handover', C3_FULL, 4096, 'o_random', '3', True), ('c3_auto', C3_FULL, 4096, 'o_random', None, True),
    ('c3_wait', C3_FULL, 300, 'o_random', '2', True), ('c3_unchained', C3_FULL, 4096, 'o_random', None, False),
    ('c2_split', C2_FULL, 1024, 'swap_goals', None, True), ('c2_courier', C2_FULL, 1024, 'swap_goals', None, True),
    ('c4_multiwave_handover', C4_FULL, 2048, 'swarm_vs_swarm', None, True), ('c3_host_tables', C3_FULL, 37, None, '3', True)])
def test_chained_graph_equals_one_rollout(name, kw, E, dev_scn, pdl, chained, monkeypatch):
    """A CUDA graph of 96 step launches (every chaining mode: per-block hand-over, grid-wide wait, unchained; split,
    courier and multi-wave shapes) gives, bit for bit, what one rollout launch gives, over replays and auto-resets."""
    import torch
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    if pdl is not None:
        monkeypatch.setenv('QS_PDL', pdl)
    if 'split' in name:
        monkeypatch.setenv('QS_SPLIT', '1')
    T, R, N = 96, 3, kw['num_agents']

    def mk():
        e = QuadSwarmEngine(num_envs=E, seed=9, ep_time=0.3, device_scenario=dev_scn, init_random_state=True, **kw)
        if dev_scn is None:
            from tests.parity_util import make_tables
            t = make_tables(np.random.RandomState(1), E, N, e.M, True, episodes=1)[0]
            e.set_next_episode(t['goals'], t['spawn'], t['obst'])
        return e
    e1, e2 = mk(), mk()
    e1.set_chained(chained)
    e2.set_chained(chained)
    a = _acts(T, E, N)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    obs = torch.empty((T, E, N, e1.D), device='cuda'); rew = torch.empty((T, E, N), device='cuda')
    dn = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    with torch.cuda.stream(st):
        e1.reset()
        for t in range(3):
            e1.step(a[t], obs_out=obs[t], rewards_out=rew[t], dones_out=dn[t])
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for t in range(T):
                e1.step(a[t], obs_out=obs[t], rewards_out=rew[t], dones_out=dn[t])
    e2.reset()
    for t in range(3):
        e2.step(a[t])
    for r in range(R):
        g.replay()
        torch.cuda.synchronize()
        o2, r2, d2 = e2.rollout(a)
        torch.cuda.synchronize()
        assert torch.equal(obs, o2) and torch.equal(rew, r2) and torch.equal(dn, d2), f'replay {r}'
        _state_equal(e1, e2)
    assert int(dn.sum()) > 0
    assert e1.handover_timeouts == 0 and e2.handover_timeouts == 0
    e1.close(); e2.close()


@pytest.mark.gpu
def test_pregenerated_record_equals_inline_generation(monkeypatch):
    """An auto-reset that copies its episode's record (qs_pregen_kernel ran before every step launch, QS_PREGEN=1) and
    one that generates the episode inline (a graph of steps that never refills a record, QS_PREGEN=0) spawn the same
    random states: the draws are keyed by the episode, not by where they are made."""
    import torch
    E, T, N = 512, 120, 8
    monkeypatch.setenv('QS_PREGEN', '1')
    e1 = _engine(E, _on(dict(KW_C3, ep_time=0.3)))
    monkeypatch.setenv('QS_PREGEN', '0')
    e2 = _engine(E, _on(dict(KW_C3, ep_time=0.3)))
    a = _acts(T, E, N, seed=8)
    obs1 = torch.empty((T, E, N, e1.D), device='cuda'); dn1 = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    obs2, dn2 = torch.empty_like(obs1), torch.empty_like(dn1)
    e1.reset()
    for t in range(T):
        e1.step(a[t], obs_out=obs1[t], dones_out=dn1[t])
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        e2.reset()
        for t in range(3):                  # warm-up launches before the capture
            e2.step(a[t], obs_out=obs2[t], dones_out=dn2[t])
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for t in range(3, T):
                e2.step(a[t], obs_out=obs2[t], dones_out=dn2[t])
    g.replay()
    torch.cuda.synchronize()
    assert int(dn1.sum()) >= 2 * E * N
    assert torch.equal(obs1, obs2) and torch.equal(dn1, dn2)
    _state_equal(e1, e2)
    e1.close(); e2.close()


@pytest.mark.gpu
def test_env_snapshot_restore_with_random_initial_states():
    """snapshot()/restore(keep_rng_counters=False) continues bit-identically across auto-resets with random spawns."""
    from quad_swarm_rl_b200.env import QuadrotorEnvMulti
    env = QuadrotorEnvMulti(num_agents=8, ep_time=0.2, rew_coeff=None, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=6,
                            neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0,
                            use_obstacles=False, obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0],
                            use_downwash=False, use_numba=True, quads_mode='static_same_goal', room_dims=[10., 10., 10.],
                            use_replay_buffer=True, quads_view_mode=['topdown'], quads_render=False,
                            dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
                            dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
                            init_random_state=True, seed=12)
    obs0 = env.reset()
    assert np.abs(obs0[:, 3:6]).max() > 0 and np.abs(obs0[:, 15:18]).max() > 0.01       # moving, spinning spawns
    acts = np.random.RandomState(0).uniform(-1, 1, (70, 8, 4)).astype(np.float32)
    for t in range(10):
        env.step(acts[t])
    snap = env.snapshot()
    first, dones = [], 0
    for t in range(10, 70):
        o, _, d, _ = env.step(acts[t])
        first.append(o.copy())
        dones += int(d[0])
    assert dones >= 2
    env.restore(snap, keep_rng_counters=False)
    for t, ref in zip(range(10, 70), first):
        assert np.array_equal(env.step(acts[t])[0], ref), t
    env.close()


@pytest.mark.gpu
def test_option_off_is_bit_identical_and_fixed_after_the_first_reset():
    """enable = 0 (after a call with 1) is the default path; the option cannot change once a reset or step ran."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    for kw in (KW_SAME, KW_C3):
        e1, e2 = _engine(256, kw), _engine(256, kw)
        assert e2.lib.qs_set_init_random_state(e2.h, 1, 0.5, 1.0) == 0
        assert e2.lib.qs_set_init_random_state(e2.h, 0, 1.0, TWO_PI) == 0
        a = _acts(80, 256, kw['num_agents'], seed=2)
        e1.reset(); e2.reset()
        assert torch.equal(e1.obs, e2.obs)
        o1, r1, d1 = e1.rollout(a)
        o2, r2, d2 = e2.rollout(a)
        assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2) and int(d1.sum()) > 0
        _state_equal(e1, e2)
        assert e1.lib.qs_set_init_random_state(e1.h, 1, 1.0, TWO_PI) == -1 and b'first reset' in e1.lib.qs_last_error()
        e1.close(); e2.close()
    e = _engine(4, KW_SAME)
    for bad in ((1, -1.0, 1.0), (1, 1.0, float('nan')), (1, float('inf'), 1.0)):
        assert e.lib.qs_set_init_random_state(e.h, *bad) == -1
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize('shape', ['split', 'courier', 'c4_multiwave'])
def test_launch_shapes_match_oracle(shape, monkeypatch):
    """The option in the step shapes the golden-configuration test does not reach at its size: the split physics /
    observer kernel (QS_SPLIT=1), the balanced shape with the courier warp (c3, 4096 envs, chained) and the multi-wave
    per-block hand-over (c4, 32 drones x 2048 envs, chained); sampled envs checked against the oracle."""
    from oracle.scenario_gen import DeviceORandomSource, DeviceScenarioSource
    from tests import parity_util as pu
    if shape == 'split':
        monkeypatch.setenv('QS_SPLIT', '1')
        pair = pu.Pair(6, _on(dict(KW_C3, ep_time=0.4)), seed=5151, table_seed=5152)
        T = 120
    elif shape == 'courier':
        pair = pu.SampledPair(4096, [0, 2048, 4095], _on(dict(C3_FULL, ep_time=0.4)), seed=5252, device_scenario='o_random',
                              source_factory=lambda: DeviceORandomSource(), chained=True, rew_coeff=C3_REW)
        T = 100
    else:
        pair = pu.SampledPair(2048, [0, 1024, 2047], _on(dict(C4_FULL, ep_time=0.3)), seed=5353, device_scenario='swarm_vs_swarm',
                              source_factory=lambda: DeviceScenarioSource('swarm_vs_swarm'), chained=True,
                              rew_coeff=dict(quadcol_bin=5.0, quadcol_bin_smooth_max=10.0))
        T = 70
    _arm_oracles(pair, {})
    rep = pu.run_parity(pair, T, np.random.RandomState(13), resync=10)
    resets, frac = _report(shape, pair, rep)
    assert rep['dones'] >= 2 * pair.E and frac <= 0.10, rep
    assert pair.engine.handover_timeouts == 0
    pair.engine.close()


@pytest.mark.gpu
def test_full_size_spawn_statistics():
    """8 drones x 4096 envs after one reset: |v| <= vel_max, |omega| <= omega_max, R orthonormal to float32 precision, and
    the same distributions as the keyed CPU twin (KS tests); a non-default vel_max / omega_max scales them."""
    from quad_swarm_rl_b200.engine import STATE_F32_FIELDS as F
    E, N = 4096, 8
    for vmax, wmax in ((1.0, TWO_PI), (2.5, 3.0)):
        e = _engine(E, dict(KW_SAME, ep_time=15.0), init_random_state=True, init_vel_max=vmax, init_omega_max=wmax)
        e.reset()
        af = e.get_state()['agent_f32'].cpu().numpy().astype(np.float64).reshape(E * N, -1)
        vel = af[:, F['vel'][0]:F['vel'][1]]
        om = af[:, F['omega'][0]:F['omega'][1]]
        R = af[:, F['rot'][0]:F['rot'][1]].reshape(-1, 3, 3)
        v, w = np.linalg.norm(vel, axis=1), np.linalg.norm(om, axis=1)
        assert v.max() <= vmax * (1 + 1e-5) and w.max() <= wmax * (1 + 1e-5)
        assert np.abs(np.einsum('nji,njk->nik', R, R) - np.eye(3)).max() <= 1e-5
        assert stats.kstest(v, 'uniform', args=(0, vmax)).pvalue > 1e-3
        assert stats.kstest(w, 'uniform', args=(0, wmax)).pvalue > 1e-3
        for col in (0, 2):
            assert stats.kstest(R[:, 2, col], 'uniform', args=(-1, 2)).pvalue > 1e-3, col
        assert np.abs(vel).max() <= vmax and np.mean(R[:, 2, 2] < 0) == pytest.approx(0.5, abs=0.01)
        e.close()
