"""Wrapper semantics of swarm_rl/env_wrappers (reward shaping + annealing, 5-tuple compatibility) and the env factory.

Sample Factory and gymnasium are not installed in this image, so the wrappers are plain delegating objects that
follow the same protocol (`reset`, `step`, `unwrapped`, attribute forwarding).  When Sample Factory is present the
factory below can be registered as is: `register_env("quadrotor_multi", make_quadrotor_env)` (swarm_rl/train.py:18).
"""
import copy

import numpy as np

# swarm_rl/env_wrappers/reward_shaping.py:7-16
DEFAULT_QUAD_REWARD_SHAPING_SINGLE = dict(
    quad_rewards=dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0),
)
DEFAULT_QUAD_REWARD_SHAPING = copy.deepcopy(DEFAULT_QUAD_REWARD_SHAPING_SINGLE)
DEFAULT_QUAD_REWARD_SHAPING['quad_rewards'].update(dict(quadcol_bin=0.0, quadcol_bin_smooth_max=0.0, quadcol_bin_obst=0.0))


class AnnealSchedule:                      # swarm_rl/env_wrappers/quad_utils.py:13-17
    def __init__(self, coeff_name, final_value, anneal_env_steps):
        self.coeff_name = coeff_name
        self.final_value = final_value
        self.anneal_env_steps = anneal_env_steps


class Wrapper:
    """Delegating wrapper with the gymnasium.Wrapper surface the reference relies on."""

    def __init__(self, env):
        self.env = env

    def __getattr__(self, name):
        if name.startswith('_'):
            raise AttributeError(name)
        return getattr(self.env, name)

    @property
    def unwrapped(self):
        return self.env.unwrapped

    def close(self):
        return self.env.close()


class QuadsTrainingEnv(Wrapper):
    """What QuadsRewardShapingWrapper(ExperienceReplayWrapper(QuadrotorEnvMulti)) is to the reference's callers
    (reward_shaping.py:19-123, quad_experience_replay.py:66-209) — old 4-tuple API, numpy observations, lists of per-agent
    rewards / dones / info dicts — as a thin adapter over `training.BatchedTrainingEnv` with ONE env: the wrappers' work
    itself runs in the kernel behind the step kernel (csrc/qs_wrap.cuh).  At an episode end every agent's info carries
    `true_reward` and `episode_extra_stats` (the env's statistics are means over its agents, which is also how Sample
    Factory aggregates them); the per-step `info['rewards']` dicts of the raw env are not produced here."""

    def __init__(self, benv):
        super().__init__(benv)
        self.num_agents = benv.env.num_agents_per_env
        self.is_multiagent = True
        self.training_info = benv.training_info

    def reset(self):
        obs, _ = self.env.reset()
        return obs.cpu().numpy().astype(np.float64)

    def step(self, action):
        import torch
        benv = self.env
        a = torch.as_tensor(np.asarray(action, dtype=np.float32), device=benv.engine.device)
        obs, rew, term, _, _ = benv.step(a)
        dones = term.cpu().numpy().astype(bool)
        infos = [dict() for _ in range(self.num_agents)]
        if dones[0]:
            fin = benv.flush_stats()
            if fin:
                tr = fin['true_reward'].cpu().numpy().reshape(-1)
                for i, info in enumerate(infos):
                    info['true_reward'] = float(tr[i])
                    info['episode_extra_stats'] = dict(fin['episode_extra_stats'])
        return obs.cpu().numpy().astype(np.float64), [float(x) for x in rew.cpu().numpy()], [bool(d) for d in dones], infos


class QuadEnvCompatibility(Wrapper):
    """Old 4-tuple API -> gymnasium 5-tuple (compatibility.py:10-57): terminated = dones, truncated all False."""

    def reset(self, seed=None, options=None):
        return self.env.reset(), {}

    def step(self, action):
        obs, reward, done, info = self.env.step(action)
        if isinstance(info, dict) and isinstance(done, bool):
            done = [done]
        terminated = np.array(done, dtype=bool)
        truncated = np.zeros_like(terminated)
        return obs, reward, terminated, truncated, info

    def render(self):
        return self.env.render()


def _shaping_and_annealing(cfg):
    """quad_utils.py:72-90: reward coefficients from the CLI flags, linear annealing of the collision terms."""
    reward_shaping = copy.deepcopy(DEFAULT_QUAD_REWARD_SHAPING)
    reward_shaping['quad_rewards']['quadcol_bin'] = cfg.quads_collision_reward
    reward_shaping['quad_rewards']['quadcol_bin_smooth_max'] = cfg.quads_collision_smooth_max_penalty
    reward_shaping['quad_rewards']['quadcol_bin_obst'] = cfg.quads_obst_collision_reward
    annealing = None
    if cfg.anneal_collision_steps > 0:
        names = {'quadcol_bin': cfg.quads_collision_reward, 'quadcol_bin_smooth_max': cfg.quads_collision_smooth_max_penalty,
                 'quadcol_bin_obst': cfg.quads_obst_collision_reward}
        for k in names:
            reward_shaping['quad_rewards'][k] = 0.0
        annealing = [AnnealSchedule(k, v, cfg.anneal_collision_steps) for k, v in names.items()]
    return reward_shaping, annealing


def make_quadrotor_env_multi_batched(cfg, num_envs, env_id_offset=0, stats_every=None):
    """swarm_rl/env_wrappers/quad_utils.py:20-110 for a batched sampler: `num_envs` envs behind one object, CUDA tensors in and
    out.  Episodes, goal events, reward-shaping statistics and the collision-event replay all run in kernels
    (training.BatchedTrainingEnv); `cfg` is any object carrying the `--quads_*` attributes of quadrotor_params.py:15-121."""
    from .env import QuadrotorEnvMultiBatched
    from .training import BatchedTrainingEnv
    if getattr(cfg, 'visualize_v_value', False):
        raise NotImplementedError("V-value visualisation is out of scope")
    env = QuadrotorEnvMultiBatched(
        num_envs=num_envs, num_agents=cfg.quads_num_agents, ep_time=cfg.quads_episode_duration,
        rew_coeff=dict(DEFAULT_QUAD_REWARD_SHAPING['quad_rewards']), obs_repr=cfg.quads_obs_repr,
        neighbor_visible_num=cfg.quads_neighbor_visible_num, neighbor_obs_type=cfg.quads_neighbor_obs_type,
        collision_hitbox_radius=cfg.quads_collision_hitbox_radius, collision_falloff_radius=cfg.quads_collision_falloff_radius,
        use_obstacles=cfg.quads_use_obstacles,
        # the pillar table is sized for the largest density the randomisation can draw
        obst_density=(max(cfg.quads_obst_density, float(np.arange(cfg.quads_obst_density_min, cfg.quads_obst_density_max, 0.05).max()))
                      if (getattr(cfg, 'quads_domain_random', False) and getattr(cfg, 'quads_obst_density_random', False)) else cfg.quads_obst_density),
        obst_size=cfg.quads_obst_size,
        obst_spawn_area=cfg.quads_obst_spawn_area, use_downwash=cfg.quads_use_downwash, quads_mode=cfg.quads_mode,
        room_dims=cfg.quads_room_dims, device=getattr(cfg, 'quads_device', 0), seed=getattr(cfg, 'seed', None),
        env_id_offset=env_id_offset,
        # --quads_use_numba (quadrotor_params.py:88, default False); an object without the attribute keeps the njit path
        use_numba=getattr(cfg, 'quads_use_numba', True))
    # quad_utils.py:67-70: domain randomisation of the pillar field (per fresh episode, on the device)
    if cfg.quads_use_obstacles and getattr(cfg, 'quads_domain_random', False) and env.device_scenario is not None:
        dens = [cfg.quads_obst_density]
        sizes = [cfg.quads_obst_size]
        if getattr(cfg, 'quads_obst_density_random', False):
            dens = list(np.arange(cfg.quads_obst_density_min, cfg.quads_obst_density_max, 0.05))
        if getattr(cfg, 'quads_obst_size_random', False):
            sizes = list(np.arange(cfg.quads_obst_size_min, cfg.quads_obst_size_max, 0.1))
        env.engine.set_obstacle_randomization(dens, sizes)
    reward_shaping, annealing = _shaping_and_annealing(cfg)
    return BatchedTrainingEnv(env, reward_shaping_scheme=reward_shaping, annealing=annealing,
                              replay_buffer_sample_prob=cfg.replay_buffer_sample_prob, stats_every=stats_every)


def make_quadrotor_env_multi(cfg, render_mode=None, **kwargs):
    """The same factory for ONE env with the reference's object protocol (numpy in / out, lists of per-agent values):
    QuadEnvCompatibility(QuadsTrainingEnv(BatchedTrainingEnv(one env)))."""
    if getattr(cfg, 'quads_render', False):
        raise NotImplementedError("rendering is out of scope")
    benv = make_quadrotor_env_multi_batched(cfg, num_envs=1, stats_every=1 << 30)
    return QuadEnvCompatibility(QuadsTrainingEnv(benv))


def make_quadrotor_env(env_name, cfg=None, _env_config=None, render_mode=None, **kwargs):
    """Sample Factory env factory, same signature as swarm_rl/env_wrappers/quad_utils.py:113-117."""
    if env_name == 'quadrotor_multi':
        return make_quadrotor_env_multi(cfg, render_mode, **kwargs)
    raise NotImplementedError
