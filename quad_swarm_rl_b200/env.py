"""Reference-facing environment objects on top of the CUDA engine.

`QuadrotorEnvMulti` keeps the object protocol of `gym_art.quadrotor_multi.quadrotor_multi.QuadrotorEnvMulti`
(constructor keywords, reset()/step() signatures and return types, `rew_coeff`, `scenario`, `envs[i].tick`, ...;
reference quadrotor_multi.py:23-724) so that the reference's wrappers and Sample Factory's rollout workers can
consume it unchanged — the env step itself runs as one CUDA kernel launch (include/quadswarm.h).

`QuadrotorEnvMultiBatched` is the same env with E independent copies behind one object: `num_agents = E * N`,
observations / rewards / dones stay on the device as torch tensors (what a batched sampler wants).

Episode generation (goal formations, spawn points, pillar placement) stays on the host (scenarios.py): the tables of
the NEXT episode are uploaded one episode ahead, because the device auto-resets inside the step kernel.
"""
import copy
from collections import deque

import numpy as np
import torch

from . import _lib as L
from .engine import QuadSwarmEngine, resolve_sense_noise
from .scenarios import create_scenario, obstacle_map_given_density
from .spaces import make_observation_space, make_action_space

QUADS_OBS_REPR = L.OBS_SELF_SIZE
L_TERM_RAW_QUADCOL, L_TERM_RAW_QUADCOL_OBST = 5, 7          # QS_TERM_* in include/quadswarm.h
ARM = 0.04596194077712559          # Crazyflie motor arm, quadrotor_dynamics.py:158


class _DroneView:
    """`env.envs[i]`: the handful of per-drone attributes wrappers and scenarios read (quadrotor_single.py:98-234)."""

    def __init__(self, parent, env_idx, i):
        self._p, self._e, self._i = parent, env_idx, i
        self.control_freq = parent.control_freq
        self.dt = 0.005
        self.sim_steps = 2
        self.ep_time = parent.ep_time
        self.ep_len = parent.ep_len
        self.box = parent.box
        self.use_obstacles = parent.use_obstacles
        self.room_box = parent.room_box

    @property
    def tick(self):
        return int(self._p._tick[self._e])

    @property
    def time_remain(self):
        return self.ep_len - self.tick

    @property
    def goal(self):
        return self._p._goals[self._e, self._i]

    @property
    def dynamics(self):
        return _DynamicsView(self._p, self._e, self._i)


class _DynamicsView:
    """Read-only rigid-body state of one drone, fetched from the device on access (qs_get_state)."""

    def __init__(self, parent, e, i):
        st = parent.engine.get_state()
        af = st['agent_f32'][e, i].cpu().numpy().astype(np.float64)
        fl = int(st['agent_u32'][e, i, 0].item()) & 0xffffffff
        self.pos, self.vel, self.rot, self.omega = af[0:3], af[3:6], af[6:15].reshape(3, 3), af[15:18]
        self.thrust_rot_damp, self.thrust_cmds_damp = af[18:22], af[22:26]
        self.on_floor = bool(fl & L.FLAG_ON_FLOOR)
        self.crashed_floor = bool(fl & L.FLAG_CRASHED_FLOOR)
        self.crashed_wall = bool(fl & L.FLAG_CRASHED_WALL)
        self.crashed_ceiling = bool(fl & L.FLAG_CRASHED_CEILING)
        self.arm = ARM


class _EnvBase:
    """Shared construction: reference keyword set (quadrotor_multi.py:24-41) -> engine + host scenarios."""

    def __init__(self, num_envs, num_agents, ep_time, rew_coeff, obs_repr,
                 neighbor_visible_num, neighbor_obs_type, collision_hitbox_radius, collision_falloff_radius,
                 use_obstacles, obst_density, obst_size, obst_spawn_area,
                 use_downwash, use_numba, quads_mode, room_dims, use_replay_buffer, quads_view_mode, quads_render,
                 dynamics_params, raw_control, raw_control_zero_middle, dynamics_randomize_every, dynamics_change,
                 dyn_sampler_1, sense_noise, init_random_state, render_mode='human', device=0, seed=None,
                 env_id_offset=0, device_scenario=None, device_dynamics=False):
        # the env factory's fixed choices (swarm_rl/env_wrappers/quad_utils.py:22-31) are the only supported ones
        from .quad_models import SAMPLERS
        if isinstance(dynamics_params, str) and dynamics_params not in SAMPLERS:
            raise AttributeError(f"module 'quadrotor_randomization' has no attribute {dynamics_params!r}")     # getattr(quad_rand, name)
        if quads_render:
            raise NotImplementedError("rendering is out of scope")
        resolve_sense_noise(sense_noise)                     # 'default', None or a dict of SensorNoise parameters
        self.num_envs = int(num_envs)
        self.num_agents_per_env = int(num_agents)
        self.is_multiagent = True                           # quadrotor_multi.py:54
        self.room_dims = room_dims
        self.quads_view_mode = quads_view_mode
        self.quads_mode = quads_mode
        self.use_numba = use_numba                          # False: the physics of the reference's numpy path (floor model)
        # RawControl with actions in [-1, 1] / [0, 1], or (raw_control=False) the NonlinearPositionController, which flies
        # every drone to its goal and ignores the actions (quadrotor_single.py:259-273)
        self.raw_control, self.raw_control_zero_middle = bool(raw_control), bool(raw_control_zero_middle)
        self.use_obstacles = bool(use_obstacles)
        self.use_downwash = bool(use_downwash)
        self.use_replay_buffer = use_replay_buffer
        self.obst_density, self.obst_size, self.obst_spawn_area = obst_density, obst_size, obst_spawn_area
        self._obst_size0 = obst_size                        # the size of the engine's construction radius
        self._pushed_obst_size = None                       # the size last sent with set_next_obstacle_radius, None: never
        self.ep_time = ep_time
        self.control_freq = 100.0                           # sim_freq / sim_steps, quadrotor_single.py:160
        self.control_dt = 1.0 / self.control_freq
        self.quad_arm = ARM
        self.box = 0.1 if self.use_obstacles else 2.0       # quadrotor_single.py:215-218
        self.room_box = np.array([[-room_dims[0] / 2., -room_dims[1] / 2., 0.], [room_dims[0] / 2., room_dims[1] / 2., room_dims[2]]])
        self.collisions_grace_period_seconds = 1.5
        self.collisions_grace_period_steps = 1.5 * self.control_freq
        self.collision_threshold = collision_hitbox_radius * ARM
        self.collision_falloff_threshold = collision_falloff_radius * ARM
        self.activate_replay_buffer = False
        self.saved_in_replay_buffer = False
        self.crashes_in_recent_episodes = deque([], maxlen=100)     # quadrotor_multi.py:174-175
        self.crashes_last_episode = 0
        self.render_mode = render_mode
        self.scenes = []
        obs_self_size = QUADS_OBS_REPR[obs_repr]             # KeyError on unknown names, as the reference
        if neighbor_obs_type not in ('none', 'pos_vel'):
            raise KeyError(neighbor_obs_type)
        if neighbor_visible_num == -1:
            self.num_use_neighbor_obs = num_agents - 1
        else:
            self.num_use_neighbor_obs = neighbor_visible_num
        k_eff = self.num_use_neighbor_obs if neighbor_obs_type == 'pos_vel' else 0
        if k_eff > 0 and not (k_eff == num_agents - 1 or 1 <= k_eff < num_agents - 1):
            raise RuntimeError("Incorrect number of neigbors")      # quadrotor_multi.py:274
        if seed is None:
            seed = int(np.random.SeedSequence().entropy % (2 ** 62))
        self.seed_value = seed
        self._host_rng = np.random.RandomState(seed % (2 ** 32))
        # physical model of every drone (quadrotor_single.py:186-211): the Crazyflie constants compiled into the kernels, or one
        # dynamics source per drone (parameter set -> dynamics_change -> samplers -> limits -> derived constants) whose rows
        # are uploaded with qs_set_dynamics; `dynamics_randomize_every` resamples them every that many episodes
        factory_change = dict(noise=dict(thrust_noise_ratio=0.05), damp=dict(vel=0, omega_quadratic=0))      # quad_utils.py:31
        self.dynamics_randomize_every = dynamics_randomize_every
        self._dyn_sources = None
        dyn_spec, t2w = None, None
        quad_arm = 0.0
        if dynamics_params != 'Crazyflie' or dyn_sampler_1 is not None or dynamics_randomize_every is not None or \
                (dynamics_change is not None and dynamics_change != factory_change):
            from .quad_models import DynamicsSource, DYN_FIELDS, GRAV, dynamics_sampler_spec
            if device_dynamics:
                # the sampler runs on the device (qs_set_dynamics_sampler); quad_arm and envs[0]'s thrust-to-weight come from
                # the construction row of env 0, drone 0.  That row depends on (seed, env id, episode 0, drone 0) only, so a
                # one-env handle with the same seed and env id computes it before the real handle, whose QsConfig.quad_arm
                # needs it.  The thrust-to-weight is recovered from the float32 row (sum of thrust_max / (g mass)): it
                # differs from the parameter itself by about 1e-7 relative (it only sets the position controller's action
                # bounds).
                dyn_spec = dynamics_sampler_spec(dynamics_params, dynamics_change, dyn_sampler_1)
                probe = QuadSwarmEngine(num_envs=1, num_agents=num_agents, seed=seed, device=device, env_id_offset=env_id_offset,
                                        dynamics_sampler=dyn_spec)
                row0 = probe.get_dynamics()[0, 0].double().cpu().numpy()
                probe.close()
                F = DYN_FIELDS.index
                t2w = float(row0[F('thrust_max0'):F('thrust_max3') + 1].sum() / (GRAV * row0[F('mass')]))
            else:
                self._dyn_sources = [DynamicsSource(dynamics_params, dynamics_change, dyn_sampler_1, rs=self._host_rng)
                                     for _ in range(self.num_envs * num_agents)]
                self._dyn_rows = np.stack([src.sample_row() for src in self._dyn_sources]).reshape(self.num_envs, num_agents, -1)
                row0 = self._dyn_rows[0, 0]
                t2w = self._dyn_sources[0].params['motor']['thrust_to_weight']
            quad_arm = float(row0[DYN_FIELDS.index('arm')])          # quadrotor_multi.py:81: envs[0].dynamics.arm
            self.quad_arm = quad_arm
            self.collision_threshold = collision_hitbox_radius * quad_arm
            self.collision_falloff_threshold = collision_falloff_radius * quad_arm
        self._traj_count = np.zeros(self.num_envs, np.int64)
        self.engine = QuadSwarmEngine(
            num_envs=self.num_envs, num_agents=num_agents, obs_repr=obs_repr, neighbor_visible_num=neighbor_visible_num,
            neighbor_obs_type=neighbor_obs_type, use_obstacles=use_obstacles, obst_density=obst_density,
            obst_size=obst_size, obst_spawn_area=obst_spawn_area, use_downwash=use_downwash, room_dims=room_dims,
            ep_time=ep_time, collision_hitbox_radius=collision_hitbox_radius,
            collision_falloff_radius=collision_falloff_radius, sense_noise=sense_noise, rew_coeff=rew_coeff,
            seed=seed, device=device, env_id_offset=env_id_offset, device_scenario=device_scenario, quad_arm=quad_arm,
            init_random_state=init_random_state, use_numba=bool(use_numba), raw_control=self.raw_control,
            raw_control_zero_middle=self.raw_control_zero_middle, dynamics_sampler=dyn_spec,
            dynamics_randomize_every=dynamics_randomize_every,
            # scenario.approch_goal_metric (o_base.py:16: 1.0 for the goal-sharing obstacle scenarios, else 0.5); with the
            # host-side `mix` over obstacle scenarios the value of o_random is used for every episode
            approch_goal_metric=1.0 if quads_mode in ('o_static_same_goal', 'o_dynamic_same_goal', 'o_swap_goals',
                                                       'o_ep_rand_bezier') else 0.5)
        if quads_mode == 'mix' and use_obstacles and device_scenario is None:
            import warnings
            warnings.warn("quads_mode='mix' with obstacles on host tables: the reached-goal radius (approch_goal_metric) of "
                          "o_random, 0.5, is used for every episode, also for the o_static_same_goal ones (the reference: 1.0). "
                          "The device-side generator (device_scenarios=True, the default of QuadrotorEnvMultiBatched) keeps it "
                          "per episode.")
        if self._dyn_sources is not None:
            self.engine.set_dynamics(self._dyn_rows)
        self.device_scenario = device_scenario
        self.rew_coeff = self.engine.rew_coeff               # the live, mutable dict (reward_shaping.py:55-61 writes it)
        self.ep_len = self.engine.ep_len
        self.num_obstacles = self.engine.M
        self.observation_space = make_observation_space(obs_repr, k_eff, self.use_obstacles, room_dims)
        # envs[0]'s action space (quadrotor_multi.py): the position controller's bounds depend on its model's thrust_to_weight
        if t2w is None:
            from .quad_models import crazyflie_params
            t2w = crazyflie_params()['motor']['thrust_to_weight']
        self.action_space = make_action_space(self.raw_control, self.raw_control_zero_middle, t2w)
        assert self.observation_space.shape[0] == self.engine.D == obs_self_size + 6 * k_eff + (9 if self.use_obstacles else 0)
        # host-side episode generators: the scenario of the current episode and of the next one, per env
        mk = lambda: create_scenario(quads_mode, num_agents, room_dims=room_dims, rng=self._host_rng, ep_time=ep_time,
                                     use_obstacles=self.use_obstacles)
        self._scenarios = [mk() for _ in range(self.num_envs)]
        self._next_scenarios = [mk() for _ in range(self.num_envs)]
        self._make_scenario = mk
        E, N = self.num_envs, num_agents
        self._tick = np.zeros(E, dtype=np.int64)
        self._goals = np.zeros((E, N, 3))
        self._next = dict(goals=np.zeros((E, N, 3), np.float32), spawn=np.zeros((E, N, 3), np.float32),
                          obst=np.zeros((E, max(self.num_obstacles, 1), 2), np.float32))
        self.envs = [_DroneView(self, 0, i) for i in range(N)]
        self.last_step_unique_collisions = np.array([], dtype=int)
        self.curr_quad_col = np.array([], dtype=int)

    # ---- episode tables
    def _generate_episode(self, scenario, e):
        """Run scenario.reset() (and pillar placement) for env e; fill the staging tables."""
        if self.use_obstacles:
            obst_map, pos_arr, cells = obstacle_map_given_density(self._host_rng, self.obst_spawn_area, self.obst_density,
                                                                  room_height=self.room_dims[2])
            scenario.reset(obst_map=obst_map, cell_centers=cells)
            xy = np.asarray(pos_arr, dtype=np.float32)[:, :2]
            self._next['obst'][e, :] = 1e6            # unused slots sit far outside the room
            self._next['obst'][e, :len(xy)] = xy[:self.num_obstacles]
        else:
            scenario.reset()
        self._next['goals'][e] = scenario.goals
        self._next['spawn'][e] = scenario.goals if scenario.spawn_points is None else scenario.spawn_points

    def _push_next(self, mask=None):
        self.engine.set_next_episode(self._next['goals'], self._next['spawn'],
                                     self._next['obst'][:, :self.num_obstacles] if self.use_obstacles else None, env_mask=mask)

    def _push_obst_size(self, force=False):
        """self.obst_size for every episode that starts from now on (engine.set_next_obstacle_radius, radius = size / 2 as
        obstacles.py:9-10).  Unless forced, a handle that never leaves its construction size is never switched to
        per-episode radii."""
        if not self.use_obstacles:
            return
        if not force and (self._pushed_obst_size == self.obst_size or
                          (self._pushed_obst_size is None and self.obst_size == self._obst_size0)):
            return
        self.engine.set_next_obstacle_radius(np.full(self.num_envs, self.obst_size / 2.0, np.float32))
        self._pushed_obst_size = self.obst_size

    def can_drones_fly(self):
        """quadrotor_multi.py:281-287: fewer than one floor crash per episode on average over >= 10 episodes."""
        return abs(np.mean(self.crashes_in_recent_episodes)) < 1 and len(self.crashes_in_recent_episodes) >= 10

    def _begin_episodes(self, envs):
        """Host bookkeeping after the device (auto-)reset of `envs`: current scenario <- next, generate the one after."""
        if self.use_replay_buffer and not self.activate_replay_buffer:          # quadrotor_multi.py:356-359
            self.crashes_in_recent_episodes.append(self.crashes_last_episode)
            self.activate_replay_buffer = self.can_drones_fly()
            self.crashes_last_episode = 0
        self._traj_count[list(envs)] += 1
        self.resample_dynamics(list(envs))            # constants for the reset that will END the episode starting now
        if self.device_scenario is not None:          # episodes are generated inside the kernels: only the tick restarts
            self._tick[list(envs)] = 0
            return
        for e in envs:
            self._scenarios[e], self._next_scenarios[e] = self._next_scenarios[e], self._make_scenario()
            self._goals[e] = self._next['goals'][e]
            self._tick[e] = 0
            self._generate_episode(self._next_scenarios[e], e)
        mask = np.zeros(self.num_envs, np.uint8)
        mask[list(envs)] = 1
        self._push_next(mask)

    def _reset_all(self):
        if self.device_scenario is not None:
            obs = self.engine.reset()
            self._tick[:] = 0
            return obs
        for e in range(self.num_envs):
            self._generate_episode(self._next_scenarios[e], e)
        self._push_next()
        obs = self.engine.reset()
        self._begin_episodes(range(self.num_envs))
        return obs

    def _scenario_ticks(self):
        """scenario.step() for every env (quadrotor_multi.py:590); uploads goals that moved."""
        if self.device_scenario is not None:          # goals move inside the step kernel
            return
        changed = []
        for e, sc in enumerate(self._scenarios):
            if not sc.dynamic:
                continue
            before = sc.goals
            sc.step(int(self._tick[e]))
            if sc.goals is not before or not np.array_equal(sc.goals, self._goals[e]):
                self._goals[e] = sc.goals
                changed.append(e)
        if changed:
            mask = np.zeros(self.num_envs, np.uint8)
            mask[changed] = 1
            self.engine.set_goals(self._goals.astype(np.float32), env_mask=mask)

    @property
    def scenario(self):
        return self._scenarios[0]

    def close(self):
        self.engine.close()

    def render(self, *a, **k):
        raise NotImplementedError("rendering is out of scope of the CUDA env step")

    # ---- infos
    def _reward_dicts(self, terms, coeff):
        """infos[i]['rewards'] of quadrotor_single.py:68-85 + quadrotor_multi.py:533-540 from the raw device terms."""
        out = []
        for t in terms:
            d = {
                'rew_main': coeff['pos'] * t[0], 'rew_pos': coeff['pos'] * t[0], 'rew_action': coeff['effort'] * t[1],
                'rew_crash': coeff['crash'] * t[2], 'rew_orient': coeff['orient'] * t[3], 'rew_spin': coeff['spin'] * t[4],
                'rewraw_main': t[0], 'rewraw_pos': t[0], 'rewraw_action': t[1], 'rewraw_crash': t[2],
                'rewraw_orient': t[3], 'rewraw_spin': t[4],
                'rew_quadcol': coeff['quadcol_bin'] * t[5], 'rew_proximity': t[6], 'rewraw_quadcol': t[5],
            }
            if self.use_obstacles:
                d['rew_quadcol_obstacle'] = coeff['quadcol_bin_obst'] * t[7]
                d['rewraw_quadcol_obstacle'] = t[7]
            out.append({'rewards': {k: float(v) for k, v in d.items()}})
        return out

    def _episode_stats(self, e, scenario_name):
        """episode_extra_stats of quadrotor_multi.py:626-718 for env e from the statistics latched on the device."""
        es, ags = self.engine.episode_stats()
        es, ags = es[e].cpu().numpy(), ags[e].cpu().numpy()
        N = self.num_agents_per_env
        name = scenario_name[9:]
        if self.device_scenario is not None:          # the scenario of the episode that ended (for mix: the one drawn)
            name = L.SCENARIO_NAMES.get(int(es[L.ENV_STAT_KEYS.index('scenario')]), name)
        common = {
            'num_collisions': int(es[0]), 'num_collisions_with_room': int(es[3]), 'num_collisions_with_floor': int(es[4]),
            'num_collisions_with_wall': int(es[5]), 'num_collisions_with_ceiling': int(es[6]),
            'num_collisions_after_settle': int(es[1]), f'{name}/num_collisions': int(es[1]),
            'num_collisions_final_5_s': int(es[2]), f'{name}/num_collisions_final_5_s': int(es[2]),
        }
        if self.use_obstacles:
            common.update({
                'num_collisions_obst_quad': int(es[7]), 'num_collisions_obst_quad_after_settle': int(es[8]),
                f'{name}/num_collisions_obst': int(es[7]), 'num_collisions_obst_quad_3_5': int(es[9]),
                f'{name}/num_collisions_obst_quad_3_5': int(es[9]), 'num_collisions_obst_quad_5': int(es[10]),
                f'{name}/num_collisions_obst_quad_5': int(es[10]),
            })
        flags = ags[:, 3].astype(np.int64)
        no_col_agent, no_col_obst, reached = (flags & 1) != 0, (flags & 2) != 0, (flags & 4) != 0
        col_flag = np.logical_and(no_col_agent, no_col_obst)
        rates = {
            'agent_success_rate': 1.0 * np.sum(np.logical_and(col_flag, reached)) / N,
            'agent_deadlock_rate': 1.0 * np.sum(np.logical_and(col_flag, ~reached)) / N,
            'agent_col_rate': 1.0 - np.sum(col_flag) / N,
            'agent_neighbor_col_rate': 1.0 - np.sum(no_col_agent) / N,
            'agent_obst_col_rate': 1.0 - np.sum(no_col_obst) / N,
        }
        out = []
        for i in range(N):
            s = dict(common)
            for k, col in (('1s', 0), ('3s', 1), ('5s', 2)):
                s[f'distance_to_goal_{k}'] = float(ags[i, col])
                s[f'{name}/distance_to_goal_{k}'] = float(ags[i, col])
            for k, v in rates.items():
                s[f'metric/{k}'] = float(v)
                s[f'{name}/{k}'] = float(v)
            out.append(s)
        return out


class QuadrotorEnvMulti(_EnvBase):
    """Drop-in for the reference's QuadrotorEnvMulti: one env of N drones, numpy in / numpy + python lists out."""

    def __init__(self, num_agents, ep_time, rew_coeff, obs_repr,
                 neighbor_visible_num, neighbor_obs_type, collision_hitbox_radius, collision_falloff_radius,
                 use_obstacles, obst_density, obst_size, obst_spawn_area,
                 use_downwash, use_numba, quads_mode, room_dims, use_replay_buffer, quads_view_mode, quads_render,
                 dynamics_params, raw_control, raw_control_zero_middle, dynamics_randomize_every, dynamics_change,
                 dyn_sampler_1, sense_noise, init_random_state, render_mode='human', device=0, seed=None):
        super().__init__(1, num_agents, ep_time, rew_coeff, obs_repr, neighbor_visible_num, neighbor_obs_type,
                         collision_hitbox_radius, collision_falloff_radius, use_obstacles, obst_density, obst_size,
                         obst_spawn_area, use_downwash, use_numba, quads_mode, room_dims, use_replay_buffer,
                         quads_view_mode, quads_render, dynamics_params, raw_control, raw_control_zero_middle,
                         dynamics_randomize_every, dynamics_change, dyn_sampler_1, sense_noise, init_random_state,
                         render_mode=render_mode, device=device, seed=seed)
        self.num_agents = num_agents
        N, D = num_agents, self.engine.D
        self._a = np.zeros((1, N, 4), np.float32)
        self._obs = np.zeros((1, N, D), np.float32)
        self._rew = np.zeros((1, N), np.float32)
        self._done = np.zeros((1, N), np.uint8)
        self._terms = np.zeros((1, N, L.QS_NUM_TERMS), np.float32)

    @property
    def unwrapped(self):
        return self

    def reset(self, obst_density=None, obst_size=None):
        """quadrotor_multi.py:339-411 -> obs ndarray [N, D] float64."""
        if obst_density:
            if int(obst_density * self.obst_spawn_area[0] * self.obst_spawn_area[1]) > self.num_obstacles:
                raise NotImplementedError("obst_density above the construction-time density needs a larger pillar table")
            self.obst_density = obst_density
        if obst_size:                            # kept for the later episodes too, as the reference's self.obst_size
            self.obst_size = obst_size
        self._push_obst_size()
        obs = self._reset_all()
        return obs[0].cpu().numpy().astype(np.float64)

    def step(self, actions):
        """quadrotor_multi.py:413-724 -> (obs[N,D] float64, rewards list, dones list, infos list)."""
        N = self.num_agents
        self._a[0] = np.asarray(actions, dtype=np.float32).reshape(N, 4)
        coeff = dict(self.rew_coeff)              # the coefficients in force for this step
        self.engine.step_host(self._a, self._obs, self._rew, self._done, self._terms)
        self._tick[0] += 1
        done = bool(self._done[0, 0])
        infos = self._reward_dicts(self._terms[0].astype(np.float64), coeff)
        # ids penalised this step (quadrotor_multi.py:440,467); differs from the reference only when drone 0 alone is
        # new, which the reference lists but never penalises (SURVEY Appendix D-3)
        self.last_step_unique_collisions = np.where(self._terms[0, :, L_TERM_RAW_QUADCOL] < 0)[0]
        self.curr_quad_col = np.where(self._terms[0, :, L_TERM_RAW_QUADCOL_OBST] < 0)[0]
        if self.use_replay_buffer and not self.activate_replay_buffer:          # quadrotor_multi.py:611-612
            self.crashes_last_episode += infos[0]['rewards']['rew_crash']
        if done:
            stats = self._episode_stats(0, self._scenarios[0].name())
            for i in range(N):
                if self.saved_in_replay_buffer:                               # quadrotor_multi.py:629-633
                    infos[i]['episode_extra_stats'] = {
                        'num_collisions_replay': stats[i]['num_collisions'],
                        'num_collisions_obst_replay': stats[i].get('num_collisions_obst_quad', 0)}
                else:
                    infos[i]['episode_extra_stats'] = stats[i]
            self._begin_episodes([0])
        else:
            self._scenario_ticks()
        obs = self._obs[0].astype(np.float64)
        rewards = [float(r) for r in self._rew[0]]
        dones = [done] * N
        return obs, rewards, dones, infos


    # ---- snapshot / restore: what deepcopy(env) gives the reference's replay wrapper (quad_experience_replay.py:99-104)
    def snapshot(self):
        st = self.engine.get_state()
        return dict(device={k: (v.clone() if v is not None else None) for k, v in st.items()},
                    scenarios=copy.deepcopy((self._scenarios, self._next_scenarios)), tick=self._tick.copy(),
                    goals=self._goals.copy(), next={k: v.copy() for k, v in self._next.items()},
                    obst_density=self.obst_density, obst_size=self.obst_size,
                    obst_size_per_episode=self._pushed_obst_size is not None, saved_in_replay_buffer=True,
                    activate_replay_buffer=self.activate_replay_buffer)

    def restore(self, snap, zero_collision_counters=False, keep_rng_counters=True):
        """keep_rng_counters (default, what the replay wrapper needs): the RNG step counter, the episode index and the
        episode number stay those of the LIVE env — the reference's deepcopy does not rewind numpy's global generators
        either, so a replayed event sees fresh noise.  False restores them too: the continuation is then bit-identical to
        what followed the snapshot."""
        dev = {k: (v.clone() if v is not None else None) for k, v in snap['device'].items()}
        if zero_collision_counters:          # quad_experience_replay.py:188-190: accurate per-replay statistics
            for k in (0, 1, 7, 8):           # QS_STAT_NUM_COLLISIONS, _AFTER_SETTLE, _OBST, _OBST_AFTER_SETTLE
                dev['env_i32'][:, 4 + k] = 0
        # counters a replayed snapshot must not rewind: the RNG step counter (a replay would re-draw the noise it drew the
        # first time), the episode index and the episode number that keys the episode-generation draws
        if keep_rng_counters:
            live = self.engine.get_state()['env_i32']
            for col in (1, 3, 4 + L.QS_NUM_ENV_STATS + 16):
                dev['env_i32'][:, col] = live[:, col]
        # the snapshot's pillar size: that of its running episode travels in the device state (scn_f[0].x), the one of the
        # episodes after it is set again; a snapshot from before the first size change holds radius 0 there
        if snap['obst_size_per_episode'] or self._pushed_obst_size is not None:
            if not snap['obst_size_per_episode']:
                r0 = np.array([self._obst_size0 / 2.0], np.float32).view(np.int32)[0]
                dev['env_i32'][:, 4 + L.QS_NUM_ENV_STATS + 4] = int(r0)
            self.obst_size = snap['obst_size']
            self._push_obst_size(force=self._pushed_obst_size is None)
        self.engine.set_state(dev)
        self._scenarios, self._next_scenarios = copy.deepcopy(snap['scenarios'])
        for sc in self._scenarios + self._next_scenarios:
            sc.rng = self._host_rng
            if hasattr(sc, 'scenario') and sc.scenario is not None:
                sc.scenario.rng = self._host_rng
        self._tick = snap['tick'].copy()
        self._goals = snap['goals'].copy()
        self._next = {k: v.copy() for k, v in snap['next'].items()}
        self._push_next()
        self.obst_density = snap['obst_density']
        self.saved_in_replay_buffer = snap['saved_in_replay_buffer']


def _resample_dynamics(self, env_ids):
    """QuadrotorSingle._reset, quadrotor_single.py:387-390: every `dynamics_randomize_every`-th episode of an env its drones get
    freshly sampled constants; they are uploaded now and latched by the env's (auto-)reset (qs_set_dynamics, at_next_reset)."""
    if self._dyn_sources is None or self.dynamics_randomize_every is None:
        return
    N = self.num_agents_per_env
    mask = np.zeros(self.num_envs, np.uint8)
    for e in env_ids:
        if (self._traj_count[e] + 1) % self.dynamics_randomize_every == 0:
            for i in range(N):
                self._dyn_rows[e, i] = self._dyn_sources[e * N + i].sample_row()
            mask[e] = 1
    if mask.any():
        self.engine.set_dynamics(self._dyn_rows, env_mask=mask, at_next_reset=True)


_EnvBase.resample_dynamics = _resample_dynamics


class QuadrotorEnvMultiBatched(_EnvBase):
    """E independent envs behind one object for a batched sampler: `num_agents = E * N`; device tensors in and out
    (gymnasium 5-tuple step API, terminated = dones, truncated all False as in swarm_rl/env_wrappers/compatibility.py)."""

    def __init__(self, num_envs, num_agents=8, ep_time=15.0, rew_coeff=None, obs_repr='xyz_vxyz_R_omega',
                 neighbor_visible_num=-1, neighbor_obs_type='pos_vel', collision_hitbox_radius=2.0,
                 collision_falloff_radius=4.0, use_obstacles=False, obst_density=0.2, obst_size=0.6,
                 obst_spawn_area=(8.0, 8.0), use_downwash=False, quads_mode='static_same_goal',
                 room_dims=(10., 10., 10.), sense_noise='default', device=0, seed=None, env_id_offset=0,
                 device_scenarios=True, dynamics_params='Crazyflie', dynamics_randomize_every=None, dynamics_change=None,
                 dyn_sampler_1=None, init_random_state=False, use_numba=True, raw_control=True,
                 raw_control_zero_middle=True, device_dynamics=False):
        """device_dynamics: who produces the per-drone physical constants, like device_scenarios for the episodes.  False:
        one host quad_models.DynamicsSource per drone, re-uploaded every ep_len + 1 steps when dynamics_randomize_every is
        set.  True: the device samples every drone's row at construction and at each env's own resets
        (qs_set_dynamics_sampler); nothing is sampled or uploaded on the host."""
        # device-side generators (no host work per episode or per tick): o_random with obstacles, the goal-formation
        # family and mix without; every other mode uses host tables
        dev_scn = None
        if device_scenarios and quads_mode in L.DEVICE_SCENARIOS and \
                (quads_mode == 'mix' or (quads_mode in L.OBSTACLE_SCENARIOS) == bool(use_obstacles)) and \
                not (quads_mode == 'run_away' and num_agents < 2):      # host class: fails at the first event, as the reference
            dev_scn = quads_mode
        super().__init__(num_envs, num_agents, ep_time, rew_coeff, obs_repr, neighbor_visible_num, neighbor_obs_type,
                         collision_hitbox_radius, collision_falloff_radius, use_obstacles, obst_density, obst_size,
                         obst_spawn_area, use_downwash, use_numba, quads_mode, room_dims, False, ['topdown'], False,
                         dynamics_params, raw_control, raw_control_zero_middle, dynamics_randomize_every, dynamics_change, dyn_sampler_1, sense_noise,
                         init_random_state, device=device, seed=seed, env_id_offset=env_id_offset, device_scenario=dev_scn,
                         device_dynamics=device_dynamics)
        self.num_agents = num_envs * num_agents
        self._truncated = torch.zeros(self.num_agents, dtype=torch.bool, device=self.engine.device)

    def reset(self, seed=None, options=None):
        obs = self._reset_all()
        return obs.view(self.num_agents, -1), {}

    def step(self, actions, with_terms=False, wrapped=False):
        """with_terms: also fill engine.rew_terms [E,N,QS_NUM_TERMS] (raw reward terms of this step); wrapped: the step
        runs with the training wrappers' kernel behind it (training.BatchedTrainingEnv, engine.wrap_enable)."""
        a = torch.as_tensor(actions, dtype=torch.float32, device=self.engine.device).reshape(self.num_envs, self.num_agents_per_env, 4)
        if wrapped:
            obs, rew, done = self.engine.wrap_step(a.contiguous())
        else:
            obs, rew, done = self.engine.step(a.contiguous(), with_terms=with_terms)
        if self.device_scenario is not None:           # nothing to do on the host: episodes and goal events live in the kernels
            if self._dyn_sources is not None and self.dynamics_randomize_every is not None:
                # dynamics randomisation without reading `dones` back: envs that never left lock-step end their episodes every
                # ep_len + 1 steps; replayed episodes (training.BatchedTrainingEnv) just latch the pending constants later
                self._steps_since_upload = getattr(self, '_steps_since_upload', 0) + 1
                if self._steps_since_upload >= self.ep_len + 1:
                    self._steps_since_upload = 0
                    self._traj_count += 1
                    self.resample_dynamics(range(self.num_envs))
            return obs.view(self.num_agents, -1), rew.view(-1), done.view(-1).bool(), self._truncated, {}
        self._tick += 1
        finished = np.nonzero(self._tick > self.ep_len)[0]           # lock-step episodes: known on the host without a sync
        if len(finished):
            self._begin_episodes(finished)
        self._scenario_ticks()
        return obs.view(self.num_agents, -1), rew.view(-1), done.view(-1).bool(), self._truncated, {}
