"""Per-episode pillar size on host tables (qs_set_next_obstacle_radius; QuadrotorEnvMulti.reset(obst_density, obst_size),
quadrotor_multi.py:339-351): the oracle pinned to the reference driven through a sequence of reset(obst_density, obst_size)
calls (tests/golden/obst_size_o_random_8.npz, written by oracle/gen_golden_obst_size.py), the entry point's argument
checks and the resources of the kernels it changes, and on the GPU the kernels against the oracle with a different size in
every env and episode, the golden through QuadrotorEnvMulti, the env's reset / snapshot / restore and the batched env."""
import json
import os
import re

import numpy as np
import pytest

from oracle import obst_size_oracle as oso
from oracle.gen_golden import INFO_KEYS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'obst_size_o_random_8.npz')
TOL = dict(rtol=1e-9, atol=1e-9)
OBST_TERM = INFO_KEYS.index('rewraw_quadcol_obstacle')


def _make_scenario(mode, cfg, rng):
    from quad_swarm_rl_b200.scenarios import create_scenario
    sc = create_scenario(mode, cfg.num_agents, room_dims=cfg.room_dims, rng=np.random.RandomState(0),
                         ep_time=cfg.ep_time, use_obstacles=cfg.use_obstacles)
    sc.rng = rng
    return sc


# ---- CPU ----
def test_fixture_hits_pillars_of_every_size():
    g = np.load(GOLDEN)
    hit = g['obst_term'] < 0
    sizes = {float(s): int(hit[g['sizes'] == s].sum()) for s in np.unique(g['sizes'])}
    assert sorted(sizes) == [0.3, 0.4, 0.5, 0.6] and all(v > 0 for v in sizes.values()), sizes
    assert sorted(np.unique(g['reset_density']).tolist()) == [0.05, 0.1, 0.15, 0.2]
    assert g['dones'][:, 0].sum() >= len(g['reset_t'])             # every segment runs past an auto-reset


def test_oracle_replays_reference_reset_sequence():
    g = np.load(GOLDEN, allow_pickle=False)
    out, _ = oso.replay_obst_size_golden(g, _make_scenario)
    np.testing.assert_array_equal(out['sizes'], g['sizes'])         # auto-resets keep the size of the explicit reset
    np.testing.assert_allclose(out['obs0'], g['obs0'], **TOL)
    assert np.array_equal(out['dones'], g['dones'])
    np.testing.assert_allclose(out['goals'], g['goals'], **TOL)
    np.testing.assert_allclose(out['rewards'], g['rewards'], **TOL)
    np.testing.assert_array_equal(out['infos'][..., OBST_TERM], g['obst_term'])
    infos = out['infos'][g['obs_t']]                 # the fixture keeps the reward terms of the steps it has observations of
    assert np.array_equal(np.isnan(infos), np.isnan(g['infos']))
    m = ~np.isnan(g['infos'])
    np.testing.assert_allclose(infos[m], g['infos'][m], **TOL)
    np.testing.assert_allclose(out['obs'], g['obs'], **TOL)
    for k in ('pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou'):
        np.testing.assert_allclose(out['state_' + k], g['state_' + k], err_msg=k, **TOL)
    assert np.array_equal(out['state_on_floor'], g['state_on_floor'])
    ref_stats = json.loads(str(g['ep_stats_json']))
    assert [t for t, _ in ref_stats] == [t for t, _ in out['ep_stats']]
    for (_, s0), (_, s1) in zip(ref_stats, out['ep_stats']):
        assert set(s0) == set(s1)
        for k in s0:
            np.testing.assert_allclose(s1[k], s0[k], err_msg=k, **TOL)


def test_header_declares_and_lib_binds_the_entry_point():
    import ctypes
    from quad_swarm_rl_b200 import _lib as L
    hdr = open(os.path.join(ROOT, 'include', 'quadswarm.h')).read()
    decl = re.search(r'int qs_set_next_obstacle_radius\(([^)]*)\);', hdr).group(1)
    assert [a.strip().rsplit(' ', 1)[0] for a in decl.split(',')] == ['QsHandle*', 'const uint8_t*', 'const float*', 'void*']
    assert L.EXPORTS['qs_set_next_obstacle_radius'] == (ctypes.c_int, [ctypes.c_void_p] * 4)


def _lib():
    import sys
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    from quad_swarm_rl_b200 import _lib as L
    return L.load()


def test_entry_point_rejects_null_arguments_without_gpu():
    import ctypes
    lib = _lib()
    r = (ctypes.c_float * 1)(0.2)
    assert lib.qs_set_next_obstacle_radius(None, None, r, None) == -1 and b'null' in lib.qs_last_error()
    assert lib.qs_set_next_obstacle_radius(ctypes.c_void_p(1), None, None, None) == -1 and b'null' in lib.qs_last_error()


def test_changed_kernels_use_no_local_memory():
    """The latch sits in the reset path every step and reset kernel inlines.  The kernels that had no local memory keep
    none: the ones that can carry the courier warp (<= 128 registers), every reset kernel, and the new table kernel."""
    from tests.parity_util import kernel_resources
    _lib()
    step = kernel_resources(r'qs_step_kernel(_npy)?ILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE')
    courier = {k: v for k, v in step.items() if k[1] < 16 and k[2:] == (0, 0, 1, 0, 0)}
    assert len(courier) == 8, sorted(courier)
    for k, v in courier.items():
        assert v['REG'] <= 128 and v['LOCAL'] == 0, (k, v)
    reset = kernel_resources(r'(qs_reset_kernel\w*)')
    assert reset and all(v['LOCAL'] == 0 for v in reset.values()), reset
    table = kernel_resources(r'(k_set_next_obstacle_radius)')
    assert table and all(v['LOCAL'] == 0 and v['STACK'] == 0 for v in table.values()), table


# ---- GPU ----
KW_C3 = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True,
             use_downwash=True, ep_time=0.6)


def _sized_pair(E, kw, seed, sizes):
    """parity_util.Pair whose episode k of env e has pillar size sizes[k][e] on both sides."""
    from tests import parity_util as pu

    class SizedPair(pu.Pair):
        def _push_table(self, k):
            super()._push_table(k)
            s = sizes[min(k, len(sizes) - 1)]
            self.engine.set_next_obstacle_radius(np.array([x / 2.0 for x in s], np.float32))

    pair = SizedPair(E, kw, seed=seed, table_seed=seed + 1, episodes=len(sizes))
    for e, o in enumerate(pair.oracles):
        eps = [dict(ep, obst_size=sizes[k][e]) for k, ep in enumerate(o.source.episodes)]
        o.source = oso.SizedTableEpisodeSource(eps, approch_goal_metric=0.5)
    return pair


def _fly_into_pillars(pair, t):
    """Every 25 steps, drones 0 and 1 of each env start just outside a pillar's collision distance, flying at it (on the
    oracle, then written into the device): random actions alone rarely reach a pillar."""
    if t % 25 != 5:
        return
    for o in pair.oracles:
        for i in (0, 1):
            c = o.obst_xy[i]
            r = o.obst_size / 2.0 + o.env_arm + 0.02
            d = o.drones[i]
            d.pos = np.array([c[0] + r, c[1], 2.0])
            d.vel = np.array([-1.5, 0.0, 0.0])
    pair.sync_device_from_oracle()


@pytest.mark.gpu
def test_kernels_match_oracle_with_a_size_per_env_and_episode():
    """Four envs, four episodes (explicit resets and auto-resets), a different size in every env and episode: observations,
    rewards, state and the collision / done masks against the oracle (run_parity: masks bit-exact)."""
    from tests import parity_util as pu
    sizes = [[0.3, 0.4, 0.5, 0.6], [0.6, 0.3, 0.4, 0.5], [0.5, 0.6, 0.3, 0.4], [0.4, 0.5, 0.6, 0.3]]
    pair = _sized_pair(4, KW_C3, 2468, sizes)
    obstcol, dones = 0, 0
    for r in range(2):
        if r:                                      # the second run walks the tables from the first again, on both sides
            pair._push_table(0)
            for o in pair.oracles:
                o.source.k = -1
        rep = pu.run_parity(pair, 200, np.random.RandomState(31 + r), resync=10, hook=_fly_into_pillars)
        obstcol += rep['obstcol']
        dones += rep['dones']
        assert rep['skipped_env_steps'] <= 0.05 * (rep['skipped_env_steps'] + rep['compared_env_steps']), rep
    assert dones >= 8 and obstcol > 0, (dones, obstcol)
    # the radius of the running episode is what the device latched: scn_f[0].x of each env row
    base = 4 + pu.L.QS_NUM_ENV_STATS
    r_dev = pair.engine.get_state()['env_i32'][:, base + 4].cpu().numpy().view(np.float32)
    np.testing.assert_array_equal(r_dev, [np.float32(o.obst_size / 2.0) for o in pair.oracles])
    pair.engine.close()


def _env(**over):
    from quad_swarm_rl_b200.env import QuadrotorEnvMulti
    kw = dict(num_agents=8, ep_time=0.6, rew_coeff=None, obs_repr='xyz_vxyz_R_omega_floor', neighbor_visible_num=2,
              neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0, use_obstacles=True,
              obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0], use_downwash=True, use_numba=True,
              quads_mode='o_random', room_dims=[10., 10., 10.], use_replay_buffer=False, quads_view_mode=['topdown'],
              quads_render=False, dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
              dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
              init_random_state=False, seed=21)
    kw.update(over)
    return QuadrotorEnvMulti(**kw)


@pytest.mark.gpu
def test_golden_through_the_env_object():
    """The fixture's reset(obst_density, obst_size) sequence through QuadrotorEnvMulti.  Every step whose starting state the
    fixture holds starts from the reference's state and pillars, with the previous step's pillar contacts taken from the
    reference's geometry; the radius the device uses is the one its resets latched, so the 3x3 distance patch and the
    obstacle collision mask of that step follow the reference's.  The device draws its own noise, so drones within BAND
    of a pillar's collision distance, before or after the step, are not compared."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    from quad_swarm_rl_b200.engine import STATE_F32_FIELDS as F
    g = np.load(GOLDEN)
    kw = json.loads(str(g['case_json']))['kw']
    env = _env(rew_coeff=kw['rew_coeff'], sense_noise=None)
    n, T, BAND = 8, g['actions'].shape[0], 5e-3
    arm = 0.04596194077712559
    resets = {int(t): (float(d), float(s)) for t, d, s in zip(g['reset_t'], g['reset_density'], g['reset_size'])}
    ep_of = np.searchsorted(g['obst_t'], np.arange(T), side='right') - 1
    state_row = {int(t): k for k, t in enumerate(g['state_t'])}
    obs_row = {int(t): k for k, t in enumerate(g['obs_t'])}

    def pillar_gap(xy, t):
        """distance of each drone to its nearest pillar minus the collision distance of step t's size"""
        pil = g['obst_xy'][ep_of[t]]
        return np.min(np.linalg.norm(xy[:, None, :2] - pil[None, :, :], axis=2), axis=1) - (g['sizes'][t] / 2.0 + arm)

    compared = steps = hits = 0
    hit_sizes = set()
    max_sdf = 0.0
    for t in range(T):
        if t in resets:
            env.reset(*resets[t])
            assert env.obst_size == resets[t][1]
        fresh = t in resets or (t > 0 and g['dones'][t - 1, 0])
        check = t in obs_row and (t - 1) in state_row and not fresh and not g['dones'][t, 0]
        if check:                                  # the reference's state after step t - 1 (and this step's plants)
            k0 = state_row[t - 1]
            gap_before = pillar_gap(g['state_pos'][k0], t - 1)
            st = env.engine.get_state()
            af = st['agent_f32'][0].cpu().numpy()
            for k in ('pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou'):
                a, b = F[k]
                af[:, a:b] = g['state_' + k][k0].reshape(n, -1)
            for k in np.where(g['plant_t'] == t)[0]:
                i = int(g['plant_i'][k])
                af[i, 0:3], af[i, 3:6] = g['plant_pos'][k], g['plant_vel'][k]
                af[i, 6:15], af[i, 15:18] = g['plant_rot'][k].reshape(-1), g['plant_omega'][k]
            fl = st['agent_u32'][0].cpu().numpy().view(np.uint32)
            fl[:, 0] &= np.uint32(~L.FLAG_PREV_OBST & 0xffffffff)
            fl[:, 0] |= np.where(gap_before < 0, L.FLAG_PREV_OBST, 0).astype(np.uint32)
            st['agent_f32'][0] = torch.from_numpy(af)
            st['agent_u32'][0] = torch.from_numpy(fl.view(np.int32))
            st['obst_xy'][0] = torch.from_numpy(g['obst_xy'][ep_of[t]].astype(np.float32))
            env.engine.set_state(st)
        obs, _, dones, infos = env.step(g['actions'][t])
        assert dones[0] == bool(g['dones'][t, 0]), t
        if not check:
            continue
        size = g['sizes'][t]
        assert size == env.obst_size
        k1 = obs_row[t]
        ok = (np.abs(pillar_gap(g['obs_pos'][k1], t)) > BAND) & (np.abs(gap_before) > BAND)
        err = np.abs(obs[:, -9:] - g['obs'][k1][:, -9:])
        assert (err[ok] < BAND).all(), (t, err.max())
        max_sdf = max(max_sdf, float(err[ok].max(initial=0.0)))
        dev_hit = np.array([infos[i]['rewards']['rewraw_quadcol_obstacle'] for i in range(n)]) < 0
        ref_hit = g['obst_term'][t] < 0
        assert np.array_equal(dev_hit[ok], ref_hit[ok]), t
        steps += 1
        compared += int(ok.sum())
        hits += int(ref_hit[ok].sum())
        if ref_hit[ok].any():
            hit_sizes.add(float(size))
    assert steps >= 80 and compared > 0.9 * n * steps and len(hit_sizes) >= 2, (steps, compared, hits, hit_sizes)
    print(f'[obst_size golden] {steps} steps, {compared} drone-steps compared, {hits} pillar hits at sizes '
          f'{sorted(hit_sizes)}, max 3x3 patch error {max_sdf:.2e}')
    env.close()


@pytest.mark.gpu
def test_env_reset_accepts_a_size_and_still_rejects_a_density_above_the_table():
    env = _env()
    env.reset()
    assert env.obst_size == 0.6 and env._pushed_obst_size is None          # never changed: the handle is untouched
    env.reset(obst_density=0.1, obst_size=0.4)
    assert env.obst_size == 0.4 and env.obst_density == 0.1
    env.reset()                                                              # kept for later episodes, as the reference
    assert env.obst_size == 0.4
    with pytest.raises(NotImplementedError):
        env.reset(obst_density=0.3, obst_size=0.5)
    env.close()


@pytest.mark.gpu
def test_snapshot_restore_across_size_changes_continues_bit_identically():
    env = _env()
    rs = np.random.RandomState(3)
    acts = rs.uniform(-1, 1, (200, 8, 4)).astype(np.float32)
    run = lambda ts: [tuple(np.copy(x) for x in env.step(acts[t])[:3]) for t in ts]

    def same(a, b):
        for x, y in zip(a, b):
            assert all(np.array_equal(u, v) for u, v in zip(x, y))
    env.reset()
    run(range(20))
    snap0 = env.snapshot()                         # construction size, before the handle switched
    first0 = run(range(20, 50))
    env.reset(obst_size=0.4)
    run(range(20))
    snap1 = env.snapshot()
    first1 = run(range(20, 90))                    # an auto-reset at 60 keeps 0.4
    env.reset(obst_size=0.3)
    run(range(10))
    env.restore(snap1, keep_rng_counters=False)
    assert env.obst_size == 0.4
    same(run(range(20, 90)), first1)
    env.restore(snap0, keep_rng_counters=False)
    assert env.obst_size == 0.6
    same(run(range(20, 50)), first0)
    env.close()


@pytest.mark.gpu
def test_batched_host_tables_with_a_radius_per_env():
    """QuadrotorEnvMultiBatched(device_scenarios=False): radii per env through the engine, one mask at a time; the 3x3
    distance patch of every drone against the oracle's get_surround_sdfs with the env's radius, after the reset and every
    step, across an auto-reset that keeps the radius."""
    from oracle.quadswarm_oracle import get_surround_sdfs
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    import torch
    E, N = 6, 8
    env = QuadrotorEnvMultiBatched(E, N, ep_time=0.3, use_obstacles=True, quads_mode='o_random', device_scenarios=False,
                                   obs_repr='xyz_vxyz_R_omega_floor', neighbor_visible_num=2, seed=9)
    radii = np.full(E, 0.3, np.float32)
    r_new = np.array([0.15, 0.2, 0.25, 0.3, 0.15, 0.2], np.float32)
    mask = np.array([1, 1, 1, 0, 0, 1], np.uint8)
    env.engine.set_next_obstacle_radius(r_new, env_mask=mask)
    radii[mask == 1] = r_new[mask == 1]
    obs, _ = env.reset()
    gen = torch.Generator(device='cuda')
    gen.manual_seed(5)
    worst = 0.0
    for t in range(70):                            # ep_len 30: two auto-resets
        if t:
            a = torch.rand((E * N, 4), device='cuda', generator=gen) * 2 - 1
            obs = env.step(a)[0]
        st = env.engine.get_state()
        pos = st['agent_f32'][..., 0:3].double().cpu().numpy()
        pil = st['obst_xy'].double().cpu().numpy()
        o = obs.view(E, N, -1)[..., -9:].double().cpu().numpy()
        for e in range(E):
            ref = get_surround_sdfs(pos[e, :, :2], pil[e], float(radii[e]))
            err = np.abs(o[e] - ref)
            assert err.max() < 1e-4, (t, e, err.max())
            worst = max(worst, float(err.max()))
    env.close()
