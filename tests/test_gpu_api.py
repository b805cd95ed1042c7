"""GPU tests of the C-ABI surface and the reference-facing env objects: API equivalences that hold bit-exactly
(one launch vs many, host vs device buffers, shard invariance, snapshot / restore) and size-independent properties at
BASELINE.json's full sizes (rotation orthonormality, episode length, bounds, determinism)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

C3 = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True, use_downwash=True)
C2 = dict(num_agents=8, neighbor_visible_num=6, obs_repr='xyz_vxyz_R_omega')


def _engine(E, kw, seed=3, ep_time=0.5, **extra):
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    from tests.parity_util import make_tables
    eng = QuadSwarmEngine(num_envs=E, seed=seed, ep_time=ep_time, **kw, **extra)
    t = make_tables(np.random.RandomState(11), E, kw['num_agents'], eng.M, kw.get('use_obstacles', False), episodes=1)[0]
    eng.set_next_episode(t['goals'], t['spawn'], t['obst'])
    return eng, t


def _actions(T, E, N, seed=5):
    g = torch.Generator(device='cuda'); g.manual_seed(seed)
    return (torch.rand((T, E, N, 4), device='cuda', generator=g) * 2 - 1).contiguous()


@pytest.mark.parametrize('kw', [C3, C2], ids=['c3', 'c2'])
def test_rollout_equals_repeated_steps(kw):
    """qs_rollout(T) == T x qs_step, bit for bit (same kernel, state kept in registers), across an auto-reset."""
    T, E = 70, 37
    a = _actions(T, E, kw['num_agents'])
    e1, _ = _engine(E, kw); e2, _ = _engine(E, kw)
    o1 = e1.reset().clone(); o2 = e2.reset().clone()
    assert torch.equal(o1, o2)
    obs_s, rew_s, done_s = [], [], []
    for t in range(T):
        o, r, d = e1.step(a[t])
        obs_s.append(o.clone()); rew_s.append(r.clone()); done_s.append(d.clone())
    obs_r, rew_r, done_r = e2.rollout(a)
    assert torch.equal(torch.stack(obs_s), obs_r) and torch.equal(torch.stack(rew_s), rew_r) and torch.equal(torch.stack(done_s), done_r)
    assert int(done_r.sum()) == E * kw['num_agents']          # ep_len = 50 -> exactly one episode end inside 70 steps
    s1, s2 = e1.get_state(), e2.get_state()
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        assert torch.equal(s1[k], s2[k]), k
    e3, _ = _engine(E, kw); e3.reset()
    o_last, _, _ = e3.rollout(a, last_obs_only=True)
    assert torch.equal(o_last[0], obs_r[-1])
    for e in (e1, e2, e3):
        e.close()


@pytest.mark.parametrize('pinned', [False, True], ids=['pageable_copies', 'pinned_zero_copy'])
def test_host_buffer_step_equals_device_step(pinned):
    """qs_step_host == qs_step, bit for bit: pageable numpy buffers go through staging copies, page-locked ones are
    read / written by the kernel itself (zero-copy over PCIe)."""
    E, kw = 19, C3
    e1, _ = _engine(E, kw); e2, _ = _engine(E, kw)
    e1.reset(); e2.reset()
    a = _actions(12, E, 8)

    def host(shape, dtype):
        t = torch.zeros(shape, dtype=dtype)
        return (t.pin_memory() if pinned else t).numpy()

    obs_h, rew_h, dn_h = host((E, 8, e1.D), torch.float32), host((E, 8), torch.float32), host((E, 8), torch.uint8)
    terms_h = host((E, 8, 8), torch.float32)
    a_h = host((E, 8, 4), torch.float32)
    for t in range(12):
        o, r, d = e1.step(a[t], with_terms=True)
        a_h[...] = a[t].cpu().numpy()
        e2.step_host(a_h, obs_h, rew_h, dn_h, terms_h)
        assert np.array_equal(o.cpu().numpy(), obs_h) and np.array_equal(r.cpu().numpy(), rew_h)
        assert np.array_equal(d.cpu().numpy(), dn_h) and np.array_equal(e1.rew_terms.cpu().numpy(), terms_h)
    e1.close(); e2.close()


def test_shard_invariance():
    """Results depend on the GLOBAL env id only: one engine of 8 envs == two engines of 4 envs with offsets 0 and 4."""
    kw = C3
    whole, t = _engine(8, kw)
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    parts = []
    for r in range(2):
        p = QuadSwarmEngine(num_envs=4, seed=3, ep_time=0.5, env_id_offset=4 * r, **kw)
        p.set_next_episode(t['goals'][4 * r:4 * r + 4], t['spawn'][4 * r:4 * r + 4], t['obst'][4 * r:4 * r + 4])
        parts.append(p)
    ow = whole.reset()
    op = torch.cat([p.reset() for p in parts])
    assert torch.equal(ow, op)
    a = _actions(60, 8, 8)
    for t_ in range(60):
        ow, rw, dw = whole.step(a[t_])
        outs = [p.step(a[t_, 4 * r:4 * r + 4].contiguous()) for r, p in enumerate(parts)]
        assert torch.equal(ow, torch.cat([o[0] for o in outs])) and torch.equal(rw, torch.cat([o[1] for o in outs]))
    whole.close(); [p.close() for p in parts]


def test_snapshot_restore_replays_identically():
    """qs_get_state / qs_set_state: restoring a snapshot and replaying the same actions reproduces the same outputs
    (what deepcopy(env) gives the reference's replay wrapper, quad_experience_replay.py:99-104)."""
    eng, _ = _engine(16, C3); eng.reset()
    a = _actions(30, 16, 8)
    for t in range(10):
        eng.step(a[t])
    snap = {k: v.clone() for k, v in eng.get_state().items()}
    first = [tuple(x.clone() for x in eng.step(a[t])) for t in range(10, 30)]
    eng.set_state(snap)
    for t, ref in zip(range(10, 30), first):
        out = eng.step(a[t])
        assert all(torch.equal(x, y) for x, y in zip(out, ref))
    eng.close()


def test_masked_reset_only_touches_selected_envs():
    eng, _ = _engine(6, C2); eng.reset()
    a = _actions(5, 6, 8)
    for t in range(5):
        eng.step(a[t])
    before = eng.get_state()
    obs_before = eng.obs.clone()
    mask = np.array([0, 1, 0, 0, 1, 0], np.uint8)
    eng.reset(env_mask=mask)
    after = eng.get_state()
    keep = torch.tensor(mask == 0, device='cuda')
    assert torch.equal(before['agent_f32'][keep], after['agent_f32'][keep]) and torch.equal(obs_before[keep], eng.obs[keep])
    assert (after['env_i32'][~keep, 0] == 0).all() and (after['env_i32'][keep, 0] == 5).all()
    eng.close()


@pytest.mark.parametrize('cfg', ['c2', 'c3', 'c4'])
def test_full_size_properties(cfg):
    """BASELINE.json sizes: properties that need no oracle.  R stays orthonormal, positions stay in the room, rewards are
    finite and bounded, every env ends its episode on tick ep_len + 1, and a second run is bit-identical."""
    import bench
    from quad_swarm_rl_b200.engine import QuadSwarmEngine, STATE_F32_FIELDS as F
    c = bench.CONFIGS[cfg]
    E, kw = c['E'], c['kw']
    N = kw['num_agents']
    runs = []
    for rep in range(2):
        eng = QuadSwarmEngine(num_envs=E, seed=9, ep_time=0.4, rew_coeff=c['rew'], **kw)
        g, s, o = bench.make_episode_tables(c, 64, seed=1)
        tile = lambda x: None if x is None else np.tile(x, (E // 64, 1, 1))
        eng.set_next_episode(tile(g), tile(s), tile(o))
        eng.reset()
        a = _actions(45, E, N, seed=21)
        obs, rew, done = eng.rollout(a)
        st = eng.get_state()
        runs.append((obs, rew, done, st['agent_f32'].clone()))
        if rep == 0:
            af = st['agent_f32']
            R = af[..., F['rot'][0]:F['rot'][1]].reshape(E, N, 3, 3)
            eye = torch.eye(3, device='cuda').expand(E, N, 3, 3)
            assert (R @ R.transpose(-1, -2) - eye).abs().max() < 1e-4
            pos = af[..., 0:3]
            assert (pos[..., :2].abs() <= 5.0).all() and (pos[..., 2] >= 0.0459).all() and (pos[..., 2] <= 10.0).all()
            assert torch.isfinite(obs).all() and torch.isfinite(rew).all() and (rew.abs() < 6.0).all()
            d = done.view(45, E, N)
            assert d[40].all() and int(d.sum()) == E * N          # ep_len = 40: done exactly once, on step 41
            # (|omega| may exceed the 40 rad/s clip right after a contact response: the kick lands after the clip)
        eng.close()
    for x, y in zip(runs[0], runs[1]):
        assert torch.equal(x, y)


def test_reference_style_env_object():
    """QuadrotorEnvMulti keeps the reference's protocol: types, shapes, info keys, auto-reset, mutable rew_coeff."""
    from quad_swarm_rl_b200.env import QuadrotorEnvMulti
    env = QuadrotorEnvMulti(
        num_agents=8, ep_time=0.3, rew_coeff=None, obs_repr='xyz_vxyz_R_omega_floor', neighbor_visible_num=2,
        neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0, use_obstacles=True,
        obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0], use_downwash=True, use_numba=True,
        quads_mode='o_random', room_dims=[10., 10., 10.], use_replay_buffer=False, quads_view_mode=['topdown'],
        quads_render=False, dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
        dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
        init_random_state=False, seed=4)
    assert env.num_agents == 8 and env.is_multiagent and env.observation_space.shape == (40,)
    obs = env.reset()
    assert isinstance(obs, np.ndarray) and obs.shape == (8, 40) and obs.dtype == np.float64
    env.rew_coeff['quadcol_bin_obst'] = 7.0              # wrappers mutate this dict mid-run
    saw_done = False
    for t in range(35):
        obs, rewards, dones, infos = env.step([env.action_space.sample() for _ in range(8)])
        assert obs.shape == (8, 40) and len(rewards) == 8 and isinstance(rewards[0], float) and isinstance(dones[0], bool)
        keys = set(infos[0]['rewards'])
        assert {'rew_main', 'rewraw_main', 'rew_quadcol', 'rew_proximity', 'rewraw_quadcol', 'rew_quadcol_obstacle'} <= keys
        total = sum(infos[3]['rewards'][k] for k in ('rew_pos', 'rew_action', 'rew_crash', 'rew_orient', 'rew_spin',
                                                      'rew_quadcol', 'rew_proximity', 'rew_quadcol_obstacle'))
        assert total == pytest.approx(rewards[3], abs=2e-6)
        if dones[0]:
            saw_done = True
            assert all(dones) and env.envs[0].tick == 0
            st = infos[0]['episode_extra_stats']
            assert 'num_collisions' in st and 'o_random/distance_to_goal_1s' in st and 'metric/agent_success_rate' in st
        else:
            assert env.envs[0].tick == (t + 1) % 31
    assert saw_done and env.scenario.name() == 'Scenario_o_random'
    env.close()


@pytest.mark.parametrize('device_scenarios', [False, True])
def test_batched_env_and_dynamic_scenario(device_scenarios):
    """swarm_vs_swarm behind the batched env: goals stay put until an env's swap tick (400..599), some envs have swapped
    by tick 449, every env ends on its 451st step.  With device_scenarios the host does nothing per tick or per episode."""
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    env = QuadrotorEnvMultiBatched(num_envs=16, num_agents=8, ep_time=4.5, neighbor_visible_num=6, quads_mode='swarm_vs_swarm',
                                   seed=2, device_scenarios=device_scenarios)
    assert env.device_scenario == ('swarm_vs_swarm' if device_scenarios else None)
    obs, info = env.reset()
    assert obs.is_cuda and obs.shape == (128, 54) and env.num_agents == 128

    def goals():
        return env.engine.get_state()['agent_f32'][..., 30:33].cpu().numpy().copy()

    snaps = {0: goals()}
    ended = []
    for t in range(455):
        obs, rew, term, trunc, infos = env.step(torch.rand((128, 4), device='cuda') * 2 - 1)
        if term.any():
            assert term.all() and not trunc.any()
            ended.append(t)
        if t + 1 in (399, 449, 455):
            snaps[t + 1] = goals()
    assert ended == [450]                                       # ep_len = 450 -> every env ends on its 451st step
    assert np.array_equal(snaps[0], snaps[399])                 # no goal event before tick 400
    swapped = (snaps[399] != snaps[449]).any(axis=(1, 2))
    assert swapped.any() and not swapped.all()                  # periods are U(4, 6) s: some envs have swapped by 4.49 s
    assert (snaps[449] != snaps[455]).any(axis=(1, 2)).all()    # new episode, new formations everywhere
    if device_scenarios:
        es, _ = env.engine.episode_stats()
        assert set(es[:, 12].cpu().numpy().tolist()) == {9}      # QS_SCENARIO_SWARM_VS_SWARM latched with the statistics
    env.close()


def test_batched_env_obstacle_mix_on_device():
    """The obstacle baseline's `--quads_mode=mix` with pillars (runs/obstacles/quad_obstacle_baseline.py:12): both obstacle
    scenarios are drawn and generated on the device, no host work per episode."""
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    env = QuadrotorEnvMultiBatched(num_envs=48, num_agents=8, ep_time=0.2, neighbor_visible_num=2, quads_mode='mix', seed=9,
                                   use_obstacles=True, obs_repr='xyz_vxyz_R_omega_floor', use_downwash=True)
    assert env.device_scenario == 'mix' and env.engine.M == 12
    env.reset()
    for t in range(22):
        obs, rew, term, trunc, _ = env.step(torch.rand((384, 4), device='cuda') * 2 - 1)
    es, _ = env.engine.episode_stats()
    assert set(es[:, 12].cpu().numpy().tolist()) == {1, 11}
    goals = env.engine.get_state()['agent_f32'][..., 30:33].cpu().numpy()
    same = np.array([np.all(g == g[0]) for g in goals])
    assert same.any() and not same.all()                         # o_static_same_goal envs share one goal, o_random envs do not
    assert torch.isfinite(obs).all()
    env.close()


def test_batched_env_mix_on_device_reports_scenario_names():
    """quads_mode='mix' with the device-side generators: every episode draws its scenario on the device; the single-env
    API reports it in the episode statistics' key prefix (reward_shaping.py:95-98 consumes those keys)."""
    from quad_swarm_rl_b200 import _lib as L
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    env = QuadrotorEnvMultiBatched(num_envs=64, num_agents=4, ep_time=0.2, neighbor_visible_num=2, quads_mode='mix', seed=5)
    assert env.device_scenario == 'mix'
    env.reset()
    seen = set()
    for t in range(64):
        env.step(torch.rand((256, 4), device='cuda') * 2 - 1)
        if (t + 1) % 21 == 0:
            es, _ = env.engine.episode_stats()
            seen |= set(es[:, 12].cpu().numpy().tolist())
    assert seen == set(range(2, 10)) | {12}                     # all nine obstacle-free scenarios of scenarios/utils.py:7-10 were drawn
    stats = env._episode_stats(0, 'Scenario_mix')
    es, _ = env.engine.episode_stats()
    name = L.SCENARIO_NAMES[int(es[0, 12])]
    assert f'{name}/num_collisions' in stats[0] and f'{name}/distance_to_goal_1s' in stats[0]
    env.close()


@pytest.mark.parametrize('E,dev_scn', [(4096, 'o_random'), (None, 'o_random'), (300, 'o_static_same_goal')])
def test_chained_step_grids_into_one_output_array(E, dev_scn):
    """Early hand-over of the courier warp: a block publishes its env state before its observation rows are written, and its
    successor starts on that.  When the caller gives every step the SAME output arrays, the rows of step t+1 must still land
    after those of step t (the `done` word, qs_step.cuh).  A graph of chained launches into one array must leave exactly what
    stepping with a synchronisation after every launch leaves.  E = None: two physics warps per SM, a batch for which the
    launcher picks the balanced shape with the courier warp whatever the SM count."""
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    T, N = 80, C3['num_agents']
    if E is None:
        E = 2 * (32 // N) * torch.cuda.get_device_properties(0).multi_processor_count
    mk = lambda: QuadSwarmEngine(num_envs=E, seed=4, ep_time=0.5, device_scenario=dev_scn, **C3)
    e1, e2 = mk(), mk()
    e1.set_chained(True); e2.set_chained(True)
    a = _actions(T, E, N)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())     # the tables / actions above were enqueued on the default stream
    with torch.cuda.stream(st):
        e1.reset()
        e1.step(a[0])
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for t in range(1, T):
                e1.step(a[t])                       # engine-owned obs / rewards / dones arrays: the same every step
        for _ in range(3):
            g.replay()
        st.synchronize()
    e2.reset()
    e2.step(a[0])
    for _ in range(3):
        for t in range(1, T):
            e2.step(a[t])
            torch.cuda.synchronize()
    assert torch.equal(e1.obs, e2.obs) and torch.equal(e1.rewards, e2.rewards) and torch.equal(e1.dones, e2.dones)
    s1, s2 = e1.get_state(), e2.get_state()
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        assert torch.equal(s1[k], s2[k]), k
    assert e1.handover_timeouts == 0 and e2.handover_timeouts == 0
    e1.close(); e2.close()


C4 = dict(num_agents=32, neighbor_visible_num=6, obs_repr='xyz_vxyz_R_omega')


@pytest.mark.parametrize('name,kw,E,dev_scn,pdl,chained', [
    ('c3_handover', C3, 4096, 'o_random', '3', True), ('c3_auto', C3, 4096, 'o_random', None, True),
    ('c2_split_handover', C2, 1024, 'swap_goals', None, True), ('c2_courier', C2, 1024, 'swap_goals', None, True),
    ('c4_multiwave_handover', C4, 2048, 'swarm_vs_swarm', None, True),
    ('c3_small', C3, 37, None, '3', True), ('c3_wait', C3, 300, None, '2', True),
    ('c3_unchained', C3, 4096, 'o_random', None, False), ('c4_unchained', C4, 2048, 'swarm_vs_swarm', None, False),
    ('c2_vector_stores', C2, 1024, 'swap_goals', None, True)])
def test_back_to_back_step_grids_equal_one_rollout(name, kw, E, dev_scn, pdl, chained, monkeypatch):
    """Consecutive step launches overlap on the GPU (programmatic dependent launch with a per-block hand-over instead of a
    grid-wide wait).  Replaying a CUDA graph of 96 step launches — no host gap between them — must give, bit for bit,
    what ONE launch that keeps the env block in registers gives, over several replays and across auto-resets."""
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    if pdl is not None:
        monkeypatch.setenv('QS_PDL', pdl)           # read by each engine when it is created
    if 'split' in name:
        monkeypatch.setenv('QS_SPLIT', '1')         # a chained handle of this size would use the balanced shape with a courier warp
    if name.endswith('vector_stores'):
        monkeypatch.setenv('QS_OBS_BULK', '0')      # observation tiles leave with vector stores instead of the copy engine
    T, R = 96, 3
    N = kw['num_agents']
    mk = lambda: (QuadSwarmEngine(num_envs=E, seed=9, ep_time=1.0, device_scenario=dev_scn, **kw) if dev_scn else _engine(E, kw, ep_time=1.0)[0])
    e1, e2 = mk(), mk()
    e1.set_chained(chained)                         # step grids follow each other directly (qs_set_chained)
    e2.set_chained(chained)                         # same kernel instantiation on both sides (hand-over / wait variants are
                                                    # separate template instances: identical source, but only equal builds are bit-equal)
    a = _actions(T, E, N)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())     # the tables / actions above were enqueued on the default stream
    obs = torch.empty((T, E, N, e1.D), device='cuda'); rew = torch.empty((T, E, N), device='cuda')
    dn = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
    with torch.cuda.stream(st):
        e1.reset()
        for t in range(3):                                   # warm-up launches before capture (not part of the comparison)
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
        s1, s2 = e1.get_state(), e2.get_state()
        for k in ('agent_f32', 'agent_u32', 'env_i32'):
            assert torch.equal(s1[k], s2[k]), (r, k)
    assert int(dn.sum()) > 0 or T * R < e1.ep_len
    assert e1.handover_timeouts == 0 and e2.handover_timeouts == 0
    e1.close(); e2.close()


def _ref_style_env(**over):
    from quad_swarm_rl_b200.env import QuadrotorEnvMulti
    kw = dict(num_agents=8, ep_time=4.0, rew_coeff=None, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=6,
              neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0, collision_falloff_radius=4.0, use_obstacles=False,
              obst_density=0.2, obst_size=0.6, obst_spawn_area=[8.0, 8.0], use_downwash=False, use_numba=True,
              quads_mode='static_same_goal', room_dims=[10., 10., 10.], use_replay_buffer=True, quads_view_mode=['topdown'],
              quads_render=False, dynamics_params='Crazyflie', raw_control=True, raw_control_zero_middle=True,
              dynamics_randomize_every=None, dynamics_change=None, dyn_sampler_1=None, sense_noise='default',
              init_random_state=False, seed=12)
    kw.update(over)
    return QuadrotorEnvMulti(**kw)


def test_env_snapshot_restore():
    """env.snapshot()/restore() (device SoA state + host episode state): with the RNG counters rewound the continuation is
    bit-identical; by default they stay live (what a replayed event needs: same physics, fresh noise).  The collision-event
    replay itself runs in the wrapper kernel: tests/test_gpu_batched.py."""
    env = _ref_style_env()
    env.reset()
    rs = np.random.RandomState(0)
    acts = rs.uniform(-1, 1, (40, 8, 4)).astype(np.float32)
    for t in range(10):
        env.step(acts[t])
    snap = env.snapshot()
    first = [env.step(acts[t])[0].copy() for t in range(10, 40)]
    env.restore(snap, keep_rng_counters=False)         # everything rewound, the keyed RNG counters included
    assert env.envs[0].tick == 10
    for t, ref in zip(range(10, 40), first):
        assert np.array_equal(env.step(acts[t])[0], ref)
    # default (what the replay wrapper uses): state rewound, RNG counters live -> same physics, fresh noise
    env.restore(snap)
    assert env.envs[0].tick == 10
    o = env.step(acts[10])[0]
    d = np.abs(o - first[0])
    assert d.max() > 0 and d[:, :3].max() < 0.05 and d[:, 6:15].max() < 0.01 and d.max() < 1.0, d.max()   # fresh OU / sensor noise only
    env.close()



def test_env_objects_with_other_physical_models():
    """dynamics_params / dyn_sampler_1 / dynamics_randomize_every of the reference's constructor (quadrotor_single.py:99-211):
    the env objects sample one airframe per drone on the host (quad_models.py, pinned to the reference) and upload the
    constants; resampled constants are latched by the env's next auto-reset."""
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    from quad_swarm_rl_b200.quad_models import DYN_FIELDS
    env = QuadrotorEnvMultiBatched(num_envs=6, num_agents=4, ep_time=0.3, neighbor_visible_num=2, quads_mode='static_diff_goal', seed=9,
                                   dynamics_params='RandomQuad', dynamics_randomize_every=1,
                                   dyn_sampler_1={'class': 'RelativeSampler', 'noise_ratio': 0.05, 'sampler': 'normal'})
    rows0 = env._dyn_rows.copy()
    assert len(np.unique(rows0[..., DYN_FIELDS.index('mass')])) == 24               # every drone its own airframe
    assert env.quad_arm == pytest.approx(float(rows0[0, 0, DYN_FIELDS.index('arm')]))
    obs, _ = env.reset()
    for t in range(70):
        obs, rew, term, trunc, _ = env.step(torch.rand((24, 4), device='cuda') * 2 - 1)
        assert torch.isfinite(obs).all() and torch.isfinite(rew).all()
    assert not np.array_equal(env._dyn_rows, rows0)                                  # resampled after the first episode
    env.close()
    single = _ref_style_env(dynamics_params='DefaultQuad', ep_time=0.3)
    single.reset()
    for t in range(35):
        o, r, d, i = single.step(np.random.RandomState(t).uniform(-1, 1, (8, 4)).astype(np.float32))
    assert np.isfinite(o).all() and single.quad_arm == pytest.approx(0.12 * 2 ** 0.5)
    single.close()
