"""Batched device engine: E envs x N drones stepped by one CUDA kernel launch per control step.

Thin Python owner of a `QsHandle` (include/quadswarm.h).  PyTorch is used only as the device-memory
and stream plumbing: every tensor handed to the C ABI is a plain device pointer.  The reference-facing
object protocol (QuadrotorEnvMulti.reset()/step()) lives in env.py on top of this class.
"""
import ctypes as C
import math

import numpy as np
import torch

from . import _lib as L

DEFAULT_REW_COEFF = dict(pos=1., effort=0.05, action_change=0., crash=1., orient=1., yaw=0., rot=0., attitude=0.,
                         spin=0.1, vel=0., quadcol_bin=5., quadcol_bin_smooth_max=4., quadcol_bin_obst=5.)  # quadrotor_multi.py:91-94


# SensorNoise.__init__ keywords and their defaults, sensor_noise.py:69-76
SENSOR_NOISE_DEFAULTS = dict(pos_norm_std=0.005, pos_unif_range=0., vel_norm_std=0.01, vel_unif_range=0., quat_norm_std=0.,
                             quat_unif_range=0., gyro_norm_std=0., gyro_noise_density=0.000175, gyro_random_walk=0.0105,
                             gyro_bias_correlation_time=1000., bypass=False, acc_static_noise_std=0.002,
                             acc_dynamic_noise_ratio=0.005, use_numba=False)
# the parameters that reach an observation (the accelerometer is never observed): the fields of QsSensorNoise
SENSOR_NOISE_FIELDS = tuple(k for k, _ in L.QsSensorNoise._fields_)


def resolve_sense_noise(sense_noise):
    """The `sense_noise` keyword of QuadrotorEnvMulti (quadrotor_single.py:236-247) -> None (no noise), 'default' (the set
    compiled into the kernels) or a dict of the SENSOR_NOISE_FIELDS (the custom model, qs_set_sensor_noise).  A dict takes
    the keywords of SensorNoise(**sense_noise): an unknown key raises TypeError like that call; bypass=True is None; a dict
    whose observed parameters equal the defaults, without the gyro bias model, is 'default'."""
    if sense_noise is None or (isinstance(sense_noise, str) and sense_noise == 'default'):
        return sense_noise
    if not isinstance(sense_noise, dict):
        raise ValueError("ERROR: QuadEnv: sense_noise parameter is of unknown type: " + str(sense_noise))
    for k in sense_noise:
        if k not in SENSOR_NOISE_DEFAULTS:
            raise TypeError(f"SensorNoise.__init__() got an unexpected keyword argument '{k}'")
    p = dict(SENSOR_NOISE_DEFAULTS, **sense_noise)
    if p['bypass']:
        return None
    model = {k: float(p[k]) for k in SENSOR_NOISE_FIELDS}
    defaults = ('pos_norm_std', 'pos_unif_range', 'vel_norm_std', 'vel_unif_range', 'quat_norm_std', 'quat_unif_range',
                'gyro_noise_density')
    if model['gyro_norm_std'] == 0. and all(model[k] == SENSOR_NOISE_DEFAULTS[k] for k in defaults):
        return 'default'
    return model


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class QuadSwarmEngine:
    def __init__(self, num_envs, num_agents=8, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=-1,
                 neighbor_obs_type='pos_vel', use_obstacles=False, obst_density=0.2, obst_size=0.6,
                 obst_spawn_area=(8.0, 8.0), use_downwash=False, room_dims=(10., 10., 10.), ep_time=15.0,
                 collision_hitbox_radius=2.0, collision_falloff_radius=4.0, sense_noise='default',
                 approch_goal_metric=0.5, rew_coeff=None, seed=0, device=0, env_id_offset=0,
                 device_scenario=None, quad_arm=0.0, init_random_state=False, init_vel_max=1.0, init_omega_max=2 * math.pi,
                 use_numba=True, raw_control=True, raw_control_zero_middle=True, dynamics_sampler=None,
                 dynamics_randomize_every=None):
        if not torch.cuda.is_available():
            raise RuntimeError("QuadSwarmEngine needs a CUDA device (the env step has no CPU path)")
        self.lib = L.load()
        self.device = torch.device('cuda', device)
        self.E, self.N = int(num_envs), int(num_agents)
        if neighbor_obs_type != 'pos_vel':
            neighbor_visible_num = 0                      # QUADS_NEIGHBOR_OBS_TYPE 'none' -> 0 floats, quad_utils.py:36-39
        self.num_obstacles = int(obst_density * obst_spawn_area[0] * obst_spawn_area[1]) if use_obstacles else 0  # quadrotor_multi.py:128
        cfg = L.QsConfig()
        cfg.num_envs, cfg.num_agents = self.E, self.N
        cfg.obs_repr = L.OBS_REPR[obs_repr]
        cfg.neighbor_visible_num = int(neighbor_visible_num)
        cfg.use_obstacles = int(bool(use_obstacles))
        cfg.num_obstacles = self.num_obstacles
        cfg.use_downwash = int(bool(use_downwash))
        self.sense_noise = resolve_sense_noise(sense_noise)
        cfg.sense_noise = 0 if self.sense_noise is None else 1
        cfg.obst_size = float(obst_size)
        cfg.room_dims = (C.c_float * 3)(*[float(x) for x in room_dims])
        cfg.ep_time = float(ep_time)
        cfg.collision_hitbox_radius = float(collision_hitbox_radius)
        cfg.collision_falloff_radius = float(collision_falloff_radius)
        cfg.approch_goal_metric = float(approch_goal_metric)
        cfg.env_id_offset = int(env_id_offset)
        if device_scenario is not None and device_scenario not in L.DEVICE_SCENARIOS:
            raise ValueError(f"no device-side generator for scenario {device_scenario!r} (host tables handle it)")
        if device_scenario not in (None, 'mix') and (device_scenario in L.OBSTACLE_SCENARIOS) != bool(use_obstacles):
            raise ValueError(f"device-side scenario {device_scenario!r} does not match use_obstacles={use_obstacles}")
        cfg.scenario = L.DEVICE_SCENARIOS[device_scenario] if device_scenario is not None else L.SCENARIO_HOST_TABLES
        cfg.obst_grid = (C.c_int32 * 2)(int(obst_spawn_area[0]), int(obst_spawn_area[1]))
        cfg.seed = int(seed)
        cfg.quad_arm = float(quad_arm)          # 0 = Crazyflie; envs[0].dynamics.arm of the model in use otherwise (quadrotor_multi.py:81)
        self.device_scenario = device_scenario
        self.cfg = cfg
        h = C.c_void_p()
        L.check(self.lib.qs_create(C.byref(cfg), int(device), C.byref(h)))
        self.h = h
        # stateful gyro model on: get_state() / set_state() carry the per-drone gyro bias
        self.gyro_model = isinstance(self.sense_noise, dict) and self.sense_noise['gyro_norm_std'] != 0.
        if isinstance(self.sense_noise, dict):
            L.check(self.lib.qs_set_sensor_noise(h, C.byref(L.QsSensorNoise(**self.sense_noise))))
        # QuadrotorSingle(init_random_state=True): every spawn starts from a random velocity, body rate and attitude
        # (max_init_vel / max_init_omega, quadrotor_single.py:181-182)
        self.init_random_state = bool(init_random_state)
        if self.init_random_state:
            L.check(self.lib.qs_set_init_random_state(h, 1, float(init_vel_max), float(init_omega_max)))
        # QuadrotorEnvMulti(use_numba=False): the physics of the reference's numpy path, whose floor model differs
        # (QuadrotorDynamics.step1 + floor_interaction, quadrotor_dynamics.py:225-346, 389-457)
        self.use_numba = bool(use_numba)
        if not self.use_numba:
            L.check(self.lib.qs_set_numpy_dynamics(h, 1))
        # QuadrotorSingle(raw_control, raw_control_zero_middle) (quadrotor_single.py:259-273): RawControl with actions in
        # [-1, 1] (the default) or [0, 1], or the NonlinearPositionController, which ignores the actions
        self.raw_control, self.raw_control_zero_middle = bool(raw_control), bool(raw_control_zero_middle)
        if not self.raw_control:
            L.check(self.lib.qs_set_control(h, L.QS_CONTROL_POSITION))
        elif not self.raw_control_zero_middle:
            L.check(self.lib.qs_set_control(h, L.QS_CONTROL_RAW_UNIT))
        # dynamics randomisation on the device (quad_models.dynamics_sampler_spec): every drone's row is sampled at
        # construction and at the resets `dynamics_randomize_every` names (quadrotor_single.py:186-211,359-390)
        if dynamics_sampler is not None:
            spec = L.dyn_sampler_struct(dynamics_sampler)
            L.check(self.lib.qs_set_dynamics_sampler(h, C.byref(spec), int(dynamics_randomize_every or 0)))
        self.D = self.lib.qs_obs_dim(h)
        self.M = self.lib.qs_num_obstacles(h)
        self.ep_len = self.lib.qs_ep_len(h)
        self.K = (self.N - 1) if neighbor_visible_num == -1 else int(neighbor_visible_num)
        self.S = L.OBS_SELF_SIZE[obs_repr]
        dev = self.device
        E, N, D = self.E, self.N, self.D
        self.obs = torch.zeros((E, N, D), dtype=torch.float32, device=dev)
        self.rewards = torch.zeros((E, N), dtype=torch.float32, device=dev)
        self.dones = torch.zeros((E, N), dtype=torch.uint8, device=dev)
        self.rew_terms = torch.zeros((E, N, L.QS_NUM_TERMS), dtype=torch.float32, device=dev)
        self.rew_coeff = dict(DEFAULT_REW_COEFF)
        if rew_coeff:
            assert set(rew_coeff.keys()).issubset(set(self.rew_coeff.keys()))       # quadrotor_multi.py:97-106
            self.rew_coeff.update({k: float(v) for k, v in rew_coeff.items()})
        self._pushed_coeff = None
        self.push_reward_coeffs()

    # ---- lifetime
    def close(self):
        if getattr(self, 'h', None):
            self.lib.qs_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # ---- reward coefficients are runtime-mutable (annealing / PBT write them mid-run)
    def push_reward_coeffs(self):
        vals = tuple(float(self.rew_coeff[k]) for k in L.REW_KEYS)
        if vals != self._pushed_coeff:
            arr = (C.c_float * L.QS_NUM_REW_COEFF)(*vals)
            L.check(self.lib.qs_set_reward_coeffs(self.h, arr))
            self._pushed_coeff = vals

    # ---- episode tables
    def _dev_f32(self, x, shape):
        if x is None:
            return None
        t = torch.as_tensor(np.asarray(x, dtype=np.float32) if not torch.is_tensor(x) else x, dtype=torch.float32)
        t = t.to(self.device).contiguous()
        assert tuple(t.shape) == tuple(shape), (tuple(t.shape), tuple(shape))
        return t

    def _dev_mask(self, mask):
        if mask is None:
            return None
        t = torch.as_tensor(np.asarray(mask).astype(np.uint8) if not torch.is_tensor(mask) else mask.to(torch.uint8))
        t = t.to(self.device).contiguous()
        assert tuple(t.shape) == (self.E,)
        return t

    def set_next_episode(self, goals, spawn=None, obst_xy=None, env_mask=None):
        g = self._dev_f32(goals, (self.E, self.N, 3))
        s = self._dev_f32(spawn, (self.E, self.N, 3))
        o = self._dev_f32(obst_xy, (self.E, self.M, 2)) if obst_xy is not None else None
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_set_next_episode(self.h, _ptr(m), _ptr(g), _ptr(s), _ptr(o), self._stream()))

    def set_next_obstacle_radius(self, radius, env_mask=None):
        """Pillar radius [E] (size / 2) of each masked env's next episode on a host-table handle (include/quadswarm.h,
        qs_set_next_obstacle_radius): latched by the env's next (auto-)reset like the tables of set_next_episode, and kept
        by its later episodes until it changes.  The first call switches the handle to per-episode radii; every env keeps
        the construction radius until a radius of its own is latched.  A state taken with get_state() before that call
        holds radius 0 for its running episode."""
        r = self._dev_f32(radius, (self.E,))
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_set_next_obstacle_radius(self.h, _ptr(m), _ptr(r), self._stream()))

    def set_goals(self, goals, env_mask=None):
        g = self._dev_f32(goals, (self.E, self.N, 3))
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_set_goals(self.h, _ptr(m), _ptr(g), self._stream()))

    # ---- reset / step on device tensors
    def reset(self, env_mask=None):
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_reset(self.h, _ptr(m), _ptr(self.obs), self._stream()))
        return self.obs

    def step(self, actions, with_terms=False, obs_out=None, rewards_out=None, dones_out=None):
        """actions: float32 CUDA tensor [E,N,4] (raw policy outputs).  Returns views of the engine's output buffers
        (or the caller's, e.g. slots of a rollout ring)."""
        assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()
        assert tuple(actions.shape) == (self.E, self.N, 4)
        obs = self.obs if obs_out is None else obs_out
        rew = self.rewards if rewards_out is None else rewards_out
        done = self.dones if dones_out is None else dones_out
        self.push_reward_coeffs()
        L.check(self.lib.qs_step(self.h, _ptr(actions), _ptr(obs), _ptr(rew), _ptr(done),
                                 _ptr(self.rew_terms) if with_terms else C.c_void_p(0), self._stream()))
        return obs, rew, done

    def rollout(self, actions, obs_out=None, rewards_out=None, dones_out=None, last_obs_only=False):
        """T control steps in one launch.  actions [T,E,N,4]."""
        T = actions.shape[0]
        assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()
        dev = self.device
        if obs_out is None:
            obs_out = torch.empty(((1 if last_obs_only else T), self.E, self.N, self.D), dtype=torch.float32, device=dev)
        if rewards_out is None:
            rewards_out = torch.empty((T, self.E, self.N), dtype=torch.float32, device=dev)
        if dones_out is None:
            dones_out = torch.empty((T, self.E, self.N), dtype=torch.uint8, device=dev)
        self.push_reward_coeffs()
        L.check(self.lib.qs_rollout(self.h, int(T), _ptr(actions), _ptr(obs_out), _ptr(rewards_out), _ptr(dones_out),
                                    int(bool(last_obs_only)), self._stream()))
        return obs_out, rewards_out, dones_out

    # ---- host-buffer entry points (numpy in / out, copies inside)
    def step_host(self, actions_np, obs_np, rewards_np, dones_np, terms_np=None):
        self.push_reward_coeffs()
        L.check(self.lib.qs_step_host(self.h, actions_np.ctypes.data_as(C.c_void_p), obs_np.ctypes.data_as(C.c_void_p),
                                      rewards_np.ctypes.data_as(C.c_void_p), dones_np.ctypes.data_as(C.c_void_p),
                                      terms_np.ctypes.data_as(C.c_void_p) if terms_np is not None else C.c_void_p(0)))

    def step_host_async(self, actions_np, obs_np, rewards_np, dones_np, terms_np=None):
        """step_host without the final synchronisation (page-locked buffers only); wait() completes it."""
        self.push_reward_coeffs()
        L.check(self.lib.qs_step_host_async(self.h, actions_np.ctypes.data_as(C.c_void_p), obs_np.ctypes.data_as(C.c_void_p),
                                            rewards_np.ctypes.data_as(C.c_void_p), dones_np.ctypes.data_as(C.c_void_p),
                                            terms_np.ctypes.data_as(C.c_void_p) if terms_np is not None else C.c_void_p(0)))

    def wait(self):
        L.check(self.lib.qs_wait(self.h))

    def reset_host(self, obs_np, env_mask_np=None):
        L.check(self.lib.qs_reset_host(self.h, env_mask_np.ctypes.data_as(C.c_void_p) if env_mask_np is not None else C.c_void_p(0),
                                       obs_np.ctypes.data_as(C.c_void_p)))

    # ---- state snapshot / restore
    def get_state(self):
        dev = self.device
        af = torch.empty((self.E, self.N, L.QS_STATE_F32), dtype=torch.float32, device=dev)
        au = torch.empty((self.E, self.N, L.QS_STATE_U32), dtype=torch.int32, device=dev)
        ei = torch.empty((self.E, L.QS_STATE_ENV_I32), dtype=torch.int32, device=dev)
        ob = torch.empty((self.E, max(self.M, 1), 2), dtype=torch.float32, device=dev)
        L.check(self.lib.qs_get_state(self.h, _ptr(af), _ptr(au), _ptr(ei), _ptr(ob), self._stream()))
        st = dict(agent_f32=af, agent_u32=au, env_i32=ei, obst_xy=ob[:, :self.M])
        if self.gyro_model:
            st['gyro_bias'] = self.get_gyro_bias()
        return st

    def set_state(self, state, env_mask=None):
        af = state['agent_f32'].to(self.device, torch.float32).contiguous()
        au = state['agent_u32'].to(self.device, torch.int32).contiguous()
        ei = state['env_i32'].to(self.device, torch.int32).contiguous()
        ob = state.get('obst_xy')
        ob = ob.to(self.device, torch.float32).contiguous() if (ob is not None and self.M > 0) else None
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_set_state(self.h, _ptr(m), _ptr(af), _ptr(au), _ptr(ei), _ptr(ob), self._stream()))
        if self.gyro_model and state.get('gyro_bias') is not None:
            self.set_gyro_bias(state['gyro_bias'], env_mask=env_mask)

    def get_gyro_bias(self):
        """Gyro bias of every drone [E,N,3] (zeros unless the stateful gyro model is on)."""
        b = torch.empty((self.E, self.N, 3), dtype=torch.float32, device=self.device)
        L.check(self.lib.qs_get_gyro_bias(self.h, _ptr(b), self._stream()))
        return b

    def set_gyro_bias(self, bias, env_mask=None):
        b = self._dev_f32(bias, (self.E, self.N, 3))
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_set_gyro_bias(self.h, _ptr(m), _ptr(b), self._stream()))

    def episode_stats(self):
        dev = self.device
        es = torch.empty((self.E, L.QS_NUM_ENV_STATS), dtype=torch.int32, device=dev)
        ags = torch.empty((self.E, self.N, L.QS_NUM_AGENT_STATS), dtype=torch.float32, device=dev)
        L.check(self.lib.qs_read_episode_stats(self.h, _ptr(es), _ptr(ags), self._stream()))
        return es, ags

    def get_dynamics(self):
        """The live per-drone rows [E,N,QS_DYN_ROW] (qs_get_dynamics)."""
        out = torch.empty((self.E, self.N, L.QS_DYN_ROW), dtype=torch.float32, device=self.device)
        L.check(self.lib.qs_get_dynamics(self.h, _ptr(out), self._stream()))
        return out

    def set_dynamics(self, rows, env_mask=None, at_next_reset=False):
        """Per-drone physical constants (include/quadswarm.h, qs_set_dynamics): rows [E,N,QS_DYN_ROW] float32, the layout
        of quad_models.DYN_FIELDS.  at_next_reset: latched by each masked env's next (auto-)reset, like the reference's
        resample_dynamics inside _reset."""
        r = self._dev_f32(rows, (self.E, self.N, L.QS_DYN_ROW))
        m = self._dev_mask(env_mask)
        L.check(self.lib.qs_set_dynamics(self.h, _ptr(m), _ptr(r), int(bool(at_next_reset)), self._stream()))

    # ---- the training wrappers as kernels (include/quadswarm.h, qs_wrap_*)
    def wrap_enable(self, use_replay=False, replay_buffer_size=20, replay_prob=0.75, replay_always_active=False):
        c = L.QsWrapConfig()
        c.use_replay, c.replay_buffer_size = int(bool(use_replay)), int(replay_buffer_size)
        c.replay_prob, c.replay_always_active = float(replay_prob), int(bool(replay_always_active))
        L.check(self.lib.qs_wrap_enable(self.h, C.byref(c)))
        self._agg = np.zeros(L.QS_WRAP_AGG, np.float32)
        self._true_reward = torch.zeros((self.E, self.N), dtype=torch.float32, device=self.device)

    def wrap_step(self, actions, obs_out=None, rewards_out=None, dones_out=None):
        assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous()
        obs = self.obs if obs_out is None else obs_out
        rew = self.rewards if rewards_out is None else rewards_out
        done = self.dones if dones_out is None else dones_out
        self.push_reward_coeffs()
        L.check(self.lib.qs_wrap_step(self.h, _ptr(actions), _ptr(obs), _ptr(rew), _ptr(done), self._stream()))
        return obs, rew, done

    def wrap_apply(self, actions, terms, dones, obs=None):
        """The wrappers' kernel alone on caller-supplied per-step inputs (include/quadswarm.h, qs_wrap_apply)."""
        obs = self.obs if obs is None else obs
        self.push_reward_coeffs()
        L.check(self.lib.qs_wrap_apply(self.h, _ptr(actions), _ptr(terms), _ptr(obs), _ptr(dones), self._stream()))

    def wrap_read(self, reset=True):
        L.check(self.lib.qs_wrap_read(self.h, self._agg.ctypes.data_as(C.c_void_p), int(bool(reset)), self._stream()))
        return self._agg.copy()

    def wrap_true_reward(self):
        L.check(self.lib.qs_wrap_true_reward(self.h, _ptr(self._true_reward), self._stream()))
        return self._true_reward

    def set_obstacle_randomization(self, densities, sizes):
        """Per-episode pillar density / size drawn on the device from these choice lists (include/quadswarm.h,
        qs_set_obstacle_randomization); the engine must have been built with obst_density = the largest one."""
        d = (C.c_float * len(densities))(*[float(x) for x in densities])
        z = (C.c_float * len(sizes))(*[float(x) for x in sizes])
        L.check(self.lib.qs_set_obstacle_randomization(self.h, d, len(densities), z, len(sizes)))

    def set_chained(self, on=True):
        """Promise (or retract) that consecutive step() / rollout() calls follow each other directly on the stream
        (include/quadswarm.h, qs_set_chained): rollouts with pre-generated actions, CUDA graphs of steps."""
        L.check(self.lib.qs_set_chained(self.h, int(bool(on))))

    @property
    def launch_count(self):
        return int(self.lib.qs_launch_count(self.h))

    @property
    def handover_timeouts(self):
        """Hand-over waits between overlapping step grids that hit their bound (0 in a healthy run); synchronises."""
        return int(self.lib.qs_handover_timeouts(self.h))


# field offsets inside agent_f32 rows (include/quadswarm.h, qs_get_state)
STATE_F32_FIELDS = dict(pos=(0, 3), vel=(3, 6), rot=(6, 15), omega=(15, 18), thrust_rot_damp=(18, 22),
                        thrust_cmds_damp=(22, 26), ou=(26, 30), goal=(30, 33), dist_ring=(33, 37), dist_sums=(37, 40),
                        stale_vel=(40, 43))
