"""Configurable sensor noise (sense_noise = a dict of SensorNoise parameters, sensor_noise.py:69-110; include/quadswarm.h,
qs_set_sensor_noise): the oracle pinned to the reference's own trajectories (tests/golden/sensor_noise_*.npz, written by
oracle/gen_golden_noise.py), the host-side keyword handling, and on the GPU the kernels against the oracle, the bit-exact
equivalences of the launch paths with the model on, and full-size statistics of the noise the kernels draw."""
import ctypes
import glob
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import sensor_noise_oracle as sno
from oracle.gen_golden import INFO_KEYS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
FILES = sorted(glob.glob(os.path.join(GOLDEN, 'sensor_noise_*.npz')))
TOL = dict(rtol=1e-9, atol=1e-9)


def _make_scenario(mode, cfg, rng):
    from quad_swarm_rl_b200.scenarios import create_scenario
    sc = create_scenario(mode, cfg.num_agents, room_dims=cfg.room_dims, rng=np.random.RandomState(0),
                         ep_time=cfg.ep_time, use_obstacles=cfg.use_obstacles)
    sc.rng = rng
    return sc


def test_fixtures_present():
    assert len(FILES) >= 3, FILES


@pytest.mark.parametrize('path', FILES, ids=[os.path.basename(f)[len('sensor_noise_'):-4] for f in FILES])
def test_oracle_replays_reference_with_noise_dict(path):
    g = np.load(path, allow_pickle=False)
    out, env = sno.replay_noise_golden(g, _make_scenario)
    assert env.cfg.noise is not None
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
    np.testing.assert_allclose(out['gyro_bias'], g['gyro_bias'], err_msg='gyro bias', **TOL)


def test_fixtures_exercise_the_noise_model():
    """Re-draws after contact responses, auto-resets, a perturbed observed rotation and a non-zero gyro bias all occur."""
    k = {name: i for i, name in enumerate(INFO_KEYS)}
    seen = dict(redraw=False, reset=False, rotation=False, bias=False)
    for path in FILES:
        g = np.load(path)
        inf = g['infos']
        contact = np.nanmin(inf[..., k['rewraw_quadcol']]) < 0
        if not np.all(np.isnan(inf[..., k['rewraw_quadcol_obstacle']])):
            contact |= np.nanmin(inf[..., k['rewraw_quadcol_obstacle']]) < 0
        seen['redraw'] |= bool(contact)
        seen['reset'] |= bool(g['dones'][:, 0].sum() >= 2)
        kw = json.loads(str(g['case_json']))['kw']
        assert list(g['obs_t']) == list(g['state_t']) == list(range(len(g['obs_t'])))
        rot_err = np.abs(g['obs'][:, :, 6:15] - g['state_rot'].reshape(g['obs'].shape[0], -1, 9)).max()
        if kw['sense_noise'].get('quat_norm_std', 0) or kw['sense_noise'].get('quat_unif_range', 0):
            assert rot_err > 1e-6, path
            seen['rotation'] = True
        if kw['sense_noise'].get('gyro_norm_std', 0):
            assert np.abs(g['gyro_bias']).max() > 1e-3, path
            seen['bias'] = True
    assert all(seen.values()), seen


# ---- host-side keyword handling (no GPU: resolve_sense_noise is what the env objects and the engine call first)
def test_sense_noise_keyword_resolution():
    from quad_swarm_rl_b200.engine import resolve_sense_noise, SENSOR_NOISE_FIELDS
    assert resolve_sense_noise('default') == 'default'
    assert resolve_sense_noise(None) is None
    with pytest.raises(TypeError, match='pos_std'):
        resolve_sense_noise(dict(pos_std=0.1))                       # SensorNoise(**d) rejects an unknown keyword
    with pytest.raises(ValueError):
        resolve_sense_noise('loud')
    assert resolve_sense_noise(dict(bypass=True)) is None
    assert resolve_sense_noise(dict(bypass=True, pos_norm_std=1.0)) is None
    assert resolve_sense_noise({}) == 'default'
    assert resolve_sense_noise(dict(pos_norm_std=0.005, vel_norm_std=0.01)) == 'default'
    assert resolve_sense_noise(dict(acc_static_noise_std=0.3, acc_dynamic_noise_ratio=0.1, use_numba=True)) == 'default'
    # the bias parameters matter only with the gyro model on
    assert resolve_sense_noise(dict(gyro_random_walk=0.5, gyro_bias_correlation_time=3.0)) == 'default'
    m = resolve_sense_noise(dict(gyro_norm_std=1.0))
    assert isinstance(m, dict) and set(m) == set(SENSOR_NOISE_FIELDS) and m['gyro_random_walk'] == 0.0105
    m = resolve_sense_noise(dict(quat_unif_range=0.02))
    assert m['quat_unif_range'] == 0.02 and m['pos_norm_std'] == 0.005


def test_env_objects_reject_unknown_noise_keys_before_touching_the_gpu():
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    with pytest.raises(TypeError):
        QuadrotorEnvMultiBatched(num_envs=2, num_agents=2, sense_noise=dict(gyro=1.0))


def test_qssensornoise_layout_matches_c(tmp_path):
    from quad_swarm_rl_b200 import _lib as L
    src = tmp_path / 'sz.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "quadswarm.h"\nint main(){printf("%zu %zu %zu\\n", '
                   'sizeof(QsSensorNoise), offsetof(QsSensorNoise, gyro_noise_density), '
                   'offsetof(QsSensorNoise, gyro_bias_correlation_time));return 0;}\n')
    exe = tmp_path / 'sz'
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    c = L.QsSensorNoise
    assert [int(x) for x in out] == [ctypes.sizeof(c), c.gyro_noise_density.offset, c.gyro_bias_correlation_time.offset]


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
NOISE_A = dict(pos_norm_std=0.01, pos_unif_range=0.02, vel_norm_std=0.02, vel_unif_range=0.05, quat_norm_std=0.02,
               quat_unif_range=0.03, gyro_noise_density=0.001)
NOISE_B = dict(gyro_norm_std=0.1, quat_norm_std=0.01)
NOISE_C = dict(gyro_norm_std=1.0, gyro_bias_correlation_time=0.05, gyro_noise_density=0.005, gyro_random_walk=0.02,
               pos_unif_range=0.01)
KW_A = dict(num_agents=8, neighbor_visible_num=6, ep_time=0.5, sense_noise=NOISE_A)
KW_B = dict(num_agents=8, neighbor_visible_num=2, ep_time=0.8, use_obstacles=True, use_downwash=True,
            obs_repr='xyz_vxyz_R_omega_floor', sense_noise=NOISE_B)
KW_C = dict(num_agents=6, neighbor_visible_num=2, ep_time=0.6, obs_repr='xyz_vxyz_R_omega_wall', sense_noise=NOISE_C)


def _noise_pair(E, kw, seed):
    from tests.parity_util import Pair

    class NoisePair(Pair):
        """Pair whose teacher forcing also carries the gyro bias."""

        def sync_device_from_oracle(self):
            super().sync_device_from_oracle()
            if self.engine.gyro_model:
                self.engine.set_gyro_bias(self.oracle_bias().astype(np.float32))

        def oracle_bias(self):
            return np.array([[sno.gyro_bias(d) for d in o.drones] for o in self.oracles])

    pair = NoisePair(E, kw, seed=seed, table_seed=seed + 1)
    pair.ocfg.noise = sno.noise_model(kw['sense_noise'])         # every oracle env shares this config object
    return pair


@pytest.mark.gpu
@pytest.mark.parametrize('kw', [KW_A, KW_B, KW_C], ids=['unif_quat_8', 'c3_gyro_bias_8', 'wall_gyro_bias_6'])
def test_kernel_matches_oracle_with_noise_model(kw):
    from tests.parity_util import run_parity
    pair = _noise_pair(6, kw, seed=31)
    bias_err = [0.0]

    def check_bias(p, t):                  # the bias after the previous step (or the reset), every step
        if p.engine.gyro_model:
            ref = p.oracle_bias()
            dev = p.engine.get_gyro_bias().cpu().numpy().astype(np.float64)
            err = np.abs(dev - ref)
            assert (err <= 1e-4 + 1e-4 * np.abs(ref)).all(), f'gyro bias before step {t}: {err.max():.3e}'
            bias_err[0] = max(bias_err[0], float(err.max()))
    def hook(p, t):
        check_bias(p, t)
        if t % 40 == 5:
            # contact responses (and with them the re-draw of every drone's noise): two drones flying into each other and
            # one into the +x wall, planted into the oracle and copied to the device
            for o in p.oracles:
                a, b, c = o.drones[0], o.drones[1], o.drones[2]
                a.pos, a.vel = np.array([0.5, 0.3, 2.0]), np.array([1.0, 0.0, 0.0])
                b.pos, b.vel = np.array([0.56, 0.31, 2.02]), np.array([-1.0, 0.1, 0.0])
                c.pos, c.vel = np.array([o.room_box[1][0] - 0.004, -1.0, 3.0]), np.array([2.5, 0.2, 0.1])
            p.sync_device_from_oracle()
    rep = run_parity(pair, 120, np.random.RandomState(4), resync=10, hook=hook)
    check_bias(pair, 120)
    assert rep['dones'] >= 6 and rep['kicked'] >= 6, rep
    if pair.engine.gyro_model:
        assert np.abs(pair.oracle_bias()).max() > 1e-4
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
    for k in ('agent_f32', 'agent_u32', 'env_i32', 'gyro_bias'):
        if k in s1 or k in s2:
            assert torch.equal(s1[k], s2[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('kw', [KW_A, KW_B], ids=['unif_quat', 'c3_gyro_bias'])
def test_rollout_graph_and_steps_are_bit_identical(kw):
    """rollout(T) == T single steps == a CUDA graph of T chained steps, with the model on, across auto-resets."""
    import torch
    E, T = 300, 100
    N = kw['num_agents']
    e1, e2 = _engine(E, kw), _engine(E, kw)
    assert e1.gyro_model == ('gyro_norm_std' in kw['sense_noise'])
    a = _acts(T, E, N)
    e1.reset(); e2.reset()
    obs1 = torch.empty((T, E, N, e1.D), device='cuda'); rew1 = torch.empty((T, E, N), device='cuda')
    dn1 = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    for t in range(T):
        e1.step(a[t], obs_out=obs1[t], rewards_out=rew1[t], dones_out=dn1[t])
    o2, r2, d2 = e2.rollout(a)
    torch.cuda.synchronize()
    assert torch.equal(obs1, o2) and torch.equal(rew1, r2) and torch.equal(dn1, d2)
    assert int(dn1.sum()) > 0
    _state_equal(e1, e2)
    # chained graph of steps (the launcher keeps the single-warp shape with the grid-wide wait for this model); e1 has
    # launched before, so the capture records steady-state launches only
    e3 = e1
    e3.set_chained(True)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    obs3 = torch.empty_like(obs1); rew3 = torch.empty_like(rew1); dn3 = torch.empty_like(dn1)
    with torch.cuda.stream(st):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for t in range(T):
                e3.step(a[t], obs_out=obs3[t], rewards_out=rew3[t], dones_out=dn3[t])
    for r in range(2):                      # both continue from the same state
        g.replay()
        o2, r2, d2 = e2.rollout(a)
        torch.cuda.synchronize()
        assert torch.equal(obs3, o2) and torch.equal(rew3, r2) and torch.equal(dn3, d2), r
        _state_equal(e2, e3)
    e1.close(); e2.close()


@pytest.mark.gpu
def test_host_buffers_and_shards_are_bit_identical():
    """qs_step_host == qs_step on device buffers; two shards (env_id_offset) == one engine, gyro bias included."""
    import torch
    kw = KW_B
    E, T, N = 64, 90, KW_B['num_agents']
    full, host = _engine(E, kw), _engine(E, kw)
    s0, s1 = _engine(E // 2, kw), _engine(E // 2, kw, env_id_offset=E // 2)
    a = _acts(T, E, N, seed=3)
    full.reset(); s0.reset(); s1.reset()
    obs_np = np.zeros((E, N, host.D), np.float32)
    host.reset_host(obs_np)
    assert np.array_equal(obs_np, full.obs.cpu().numpy())
    rew_np, dn_np = np.zeros((E, N), np.float32), np.zeros((E, N), np.uint8)
    for t in range(T):
        o, r, d = full.step(a[t])
        host.step_host(a[t].cpu().numpy(), obs_np, rew_np, dn_np)
        o0, r0, d0 = s0.step(a[t, :E // 2].contiguous())
        o1, r1, d1 = s1.step(a[t, E // 2:].contiguous())
        assert np.array_equal(obs_np, o.cpu().numpy()) and np.array_equal(rew_np, r.cpu().numpy()), t
        assert torch.equal(torch.cat([o0, o1]), o) and torch.equal(torch.cat([r0, r1]), r) and torch.equal(torch.cat([d0, d1]), d), t
    b = full.get_gyro_bias()
    assert torch.equal(torch.cat([s0.get_gyro_bias(), s1.get_gyro_bias()]), b) and float(b.abs().max()) > 0
    assert torch.equal(host.get_gyro_bias(), b)
    for e in (full, host, s0, s1):
        e.close()


@pytest.mark.gpu
def test_env_snapshot_restore_with_gyro_bias():
    """snapshot()/restore(): the gyro bias is part of the snapshot (the reference's deepcopy copies SensorNoise.gyro_bias).
    keep_rng_counters=False continues bit-identically; the default rewinds the bias too but draws fresh noise."""
    from quad_swarm_rl_b200.env import QuadrotorEnvMulti
    env = QuadrotorEnvMulti(num_agents=8, ep_time=4.0, rew_coeff=None, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=6,
                            neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0,
                            use_obstacles=False, obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0],
                            use_downwash=False, use_numba=True, quads_mode='static_same_goal', room_dims=[10., 10., 10.],
                            use_replay_buffer=True, quads_view_mode=['topdown'], quads_render=False,
                            dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
                            dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise=NOISE_C,
                            init_random_state=False, seed=12)
    env.reset()
    acts = np.random.RandomState(0).uniform(-1, 1, (40, 8, 4)).astype(np.float32)
    for t in range(10):
        env.step(acts[t])
    snap = env.snapshot()
    b_snap = snap['device']['gyro_bias'].clone()
    first = [env.step(acts[t])[0].copy() for t in range(10, 40)]
    b_end = env.engine.get_gyro_bias().clone()
    assert not np.array_equal(b_end.cpu().numpy(), b_snap.cpu().numpy())
    env.restore(snap, keep_rng_counters=False)
    assert np.array_equal(env.engine.get_gyro_bias().cpu().numpy(), b_snap.cpu().numpy())
    for t, ref in zip(range(10, 40), first):
        assert np.array_equal(env.step(acts[t])[0], ref)
    assert np.array_equal(env.engine.get_gyro_bias().cpu().numpy(), b_end.cpu().numpy())
    env.restore(snap)
    assert np.array_equal(env.engine.get_gyro_bias().cpu().numpy(), b_snap.cpu().numpy())
    env.close()


@pytest.mark.gpu
def test_default_and_defaults_equal_dict_are_bit_identical():
    import torch
    kw = dict(num_agents=8, neighbor_visible_num=6, ep_time=0.5)
    e1 = _engine(256, dict(kw, sense_noise='default'))
    e2 = _engine(256, dict(kw, sense_noise=dict(pos_norm_std=0.005, acc_static_noise_std=0.5, gyro_random_walk=3.0)))
    assert e2.sense_noise == 'default'
    a = _acts(80, 256, 8, seed=2)
    e1.reset(); e2.reset()
    o1, r1, d1 = e1.rollout(a)
    o2, r2, d2 = e2.rollout(a)
    assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2)
    e1.close(); e2.close()


@pytest.mark.gpu
def test_noise_model_is_fixed_after_the_first_reset():
    from quad_swarm_rl_b200 import _lib as L
    e = _engine(4, KW_A)
    e.reset()
    sn = L.QsSensorNoise(**{k: 0.0 for k, _ in L.QsSensorNoise._fields_})
    assert e.lib.qs_set_sensor_noise(e.h, ctypes.byref(sn)) == -1 and b'first reset' in e.lib.qs_last_error()
    e.close()
    e = _engine(4, dict(KW_A, sense_noise='default'))
    assert e.lib.qs_set_gyro_bias(e.h, None, ctypes.c_void_p(e.obs.data_ptr()), None) == -1      # model off: no bias
    e.close()


def _true_and_observed(engine):
    """(true pos, vel, rot, omega, goal) of every drone and the self part of its last observation."""
    from quad_swarm_rl_b200.engine import STATE_F32_FIELDS as F
    af = engine.get_state()['agent_f32'].cpu().numpy().astype(np.float64)
    f = lambda k: af[..., F[k][0]:F[k][1]]
    return f('pos'), f('vel'), f('rot').reshape(*af.shape[:2], 3, 3), f('omega'), f('goal'), \
        engine.obs.cpu().numpy().astype(np.float64)


@pytest.mark.gpu
def test_full_size_noise_statistics():
    """8 drones x 4096 envs: the per-component spread of observation - true state is sqrt(sigma^2 + r^2 / 3) (normal plus
    uniform part) within 2 %, a purely uniform part stays inside its range, the rotation-residual angle has the std of theta
    per axis, and the gyro bias has the closed-form variance of its AR(1) process.  An independent check of the draw layout
    (sites, blocks, lanes) at the benchmark size."""
    import torch
    E, N = 4096, 8
    noise = dict(pos_norm_std=0.01, pos_unif_range=0.02, vel_norm_std=0.0, vel_unif_range=0.05, quat_norm_std=0.02,
                 quat_unif_range=0.03, gyro_noise_density=0.003)
    kw = dict(num_agents=N, neighbor_visible_num=6, ep_time=15.0, sense_noise=noise)
    e = _engine(E, kw)
    e.reset()
    a = torch.zeros((E, N, 4), device='cuda')
    dp, dv, dw, th = [], [], [], []
    for t in range(6):
        e.step(a)
        pos, vel, rot, om, goal, obs = _true_and_observed(e)
        dp.append((obs[..., 0:3] + goal - pos).reshape(-1, 3))
        dv.append((obs[..., 3:6] - vel).reshape(-1, 3))
        dw.append((obs[..., 15:18] - om).reshape(-1, 3))
        Rn = obs[..., 6:15].reshape(E, N, 3, 3)
        Rt = np.einsum('enji,enjk->enik', rot, Rn)                    # R^T R~ = R(theta)
        th.append(0.5 * np.stack([Rt[..., 2, 1] - Rt[..., 1, 2], Rt[..., 0, 2] - Rt[..., 2, 0],
                                  Rt[..., 1, 0] - Rt[..., 0, 1]], -1).reshape(-1, 3))
    dp, dv, dw, th = (np.concatenate(x) for x in (dp, dv, dw, th))
    for name, x, sd in (('pos', dp, np.hypot(0.01, 0.02 / 3 ** 0.5)), ('vel', dv, 0.05 / 3 ** 0.5), ('gyro', dw, 0.003),
                        ('theta', th, np.hypot(0.02, 0.03 / 3 ** 0.5))):
        std = x.std(axis=0)
        assert np.all(np.abs(std / sd - 1) < 0.02), (name, std, sd)
        assert np.all(np.abs(x.mean(axis=0)) < 0.02 * sd), (name, x.mean(axis=0))
    assert np.abs(dv).max() <= 0.05 * (1 + 1e-5) + 1e-6 and np.abs(dv).max() > 0.049
    e.close()
    # gyro bias: b_n = pi b_(n-1) + sigma_b n; after many observations Var(b) = sigma_b^2 / (1 - pi^2) (stationary AR(1))
    tau, gnd = 0.02, 0.004
    e = _engine(E, dict(kw, sense_noise=dict(gyro_norm_std=1.0, gyro_bias_correlation_time=tau, gyro_noise_density=gnd)))
    e.reset()
    for t in range(60):
        e.step(a)
    b = e.get_gyro_bias().cpu().numpy().astype(np.float64).reshape(-1, 3)
    dt = 0.005
    pi = np.exp(-dt / tau)
    sigma_b2 = -(gnd ** 2 / dt) * (tau / 2) * np.expm1(-2 * dt / tau)
    var = sigma_b2 / (1 - pi ** 2)
    assert np.all(np.abs(b.var(axis=0) / var - 1) < 0.04), (b.var(axis=0), var)
    e.close()
