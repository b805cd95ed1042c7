"""CPU oracle of the configurable sensor-noise model — TEST INFRASTRUCTURE ONLY.

`sense_noise` may be a dict of SensorNoise parameters (quadrotor_single.py:236-247 -> SensorNoise(**sense_noise),
sensor_noise.py:69-231) instead of 'default'.  This module extends oracle/quadswarm_oracle.py with that model without
changing it: an EnvConfig that carries a `noise` attribute (a SensorNoiseModel) has its self observations drawn by
noisy_state() below; every other EnvConfig keeps the oracle's default path.  Importing the module installs the dispatch.

Random sources, as in the oracle:
  * ReplayRng – NoiseReplayRng adds the njit draws of the model to the numba stream; the gyro-bias draws
                (add_noise_to_omega) stay on numpy's global stream, after the njit draws of the same call;
  * PhiloxRng – keyed draws at the sites below, the twins of qs_rng.cuh (full-precision layout of philox.KeyedDraws).
"""
from dataclasses import dataclass
import json
import math

import numpy as np

from . import philox as px
from . import quadswarm_oracle as qo
from .gen_golden import INFO_KEYS
from .replay import config_from_case

# ---- draw sites of the model (must match qs_rng.cuh); j = which observation of the step: 0 its own, 1 the re-draw after
# a contact response, 2 an (auto-)reset
SITE_NOISE_N = 18      # (i,j)  normals v0..2 pos, v4..6 vel, v8..10 gyro, v12..14 rotation angle   sensor_noise.py:241-256
SITE_NOISE_U = 19      # (i,j)  uniforms v0..2 pos, v4..6 vel, v8..10 rotation angle
SITE_GYRO_BIAS = 20    # (i,j)  normals v0..2 bias innovation, v4..6 random walk (numpy-global stream)  sensor_noise.py:221-231
_KIND = {px.SITE_SENSOR0: 0, px.SITE_SENSOR1: 1, px.SITE_SENSOR_RESET: 2}


@dataclass(frozen=True)
class SensorNoiseModel:
    """The SensorNoise(**sense_noise) parameters that reach an observation (sensor_noise.py:69-110), with its defaults.
    gyro_norm_std != 0 switches on the stateful gyro model (add_noise_to_omega, :221-231)."""
    pos_norm_std: float = 0.005
    pos_unif_range: float = 0.0
    vel_norm_std: float = 0.01
    vel_unif_range: float = 0.0
    quat_norm_std: float = 0.0
    quat_unif_range: float = 0.0
    gyro_norm_std: float = 0.0
    gyro_noise_density: float = 0.000175
    gyro_random_walk: float = 0.0105
    gyro_bias_correlation_time: float = 1000.0
    dt: float = 0.005                   # QuadrotorSingle.dt, passed by get_state.py to add_noise_numba

    def bias_coefficients(self):
        """(pi, sigma_b) of the bias update b <- pi b + sigma_b N(0, 1), sensor_noise.py:224-229."""
        sigma_g_d = self.gyro_noise_density / (self.dt ** 0.5)
        tau = self.gyro_bias_correlation_time
        sigma_b = (-(sigma_g_d ** 2) * (tau / 2) * (math.exp(-2 * self.dt / tau) - 1)) ** 0.5
        return math.exp(-self.dt / tau), sigma_b


def noise_model(sense_noise):
    """SensorNoise(**sense_noise) of a dict (its observed parameters), else None; bypass=True means no noise at all."""
    if not isinstance(sense_noise, dict) or sense_noise.get('bypass', False):
        return None
    names = set(SensorNoiseModel.__dataclass_fields__) - {'dt'}
    return SensorNoiseModel(**{k: float(v) for k, v in sense_noise.items() if k in names})


class NoiseReplayRng(qo.ReplayRng):
    """ReplayRng whose numba stream also serves the model's njit draws."""

    def _stream(self, site):
        return self.nb if site in (SITE_NOISE_N, SITE_NOISE_U) else super()._stream(site)


def gyro_bias(d):
    """SensorNoise.gyro_bias of drone d (sensor_noise.py:101): zero until the gyro model first advances it, never reset."""
    return getattr(d, 'gyro_bias', np.zeros(3))


def quat_from_small_angle(theta):
    """sensor_noise.py:11-23."""
    q_squared = np.linalg.norm(theta) ** 2 / 4.0
    if q_squared < 1:
        q = np.array([(1 - q_squared) ** 0.5, theta[0] * 0.5, theta[1] * 0.5, theta[2] * 0.5])
    else:
        w = 1.0 / (1 + q_squared) ** 0.5
        f = 0.5 * w
        q = np.array([w, theta[0] * f, theta[1] * f, theta[2] * f])
    return q / np.linalg.norm(q)


def quat_x_quat(q, p):
    """quatXquat, quad_utils.py:148-159."""
    return np.array([q[0] * p[0] - q[1] * p[1] - q[2] * p[2] - q[3] * p[3],
                     q[0] * p[1] + q[1] * p[0] - q[2] * p[3] + q[3] * p[2],
                     q[0] * p[2] + q[1] * p[3] + q[2] * p[0] - q[3] * p[1],
                     q[0] * p[3] - q[1] * p[2] + q[2] * p[1] + q[3] * p[0]])


def noisy_state(d, m, rng, i, kind):
    """SensorNoise(**dict).add_noise_numba (sensor_noise.py:172-218, njit :235-261) for a rotation-matrix state, plus
    add_noise_to_omega (:221-231) when m.gyro_norm_std != 0.  The njit draws (numba stream) in their order: pos normal,
    pos uniform, vel normal, vel uniform, gyro normal, theta normal, theta uniform, accelerometer (never observed); then the
    gyro model's two normal triples on numpy's global stream.  uniform(lo, hi) is lo + (hi - lo) u, as numba computes it."""
    N, U = SITE_NOISE_N, SITE_NOISE_U
    nrm = lambda blk: np.array([rng.normal(N, i, kind, 4 * blk + c) for c in range(3)])
    uni = lambda blk, r: np.array([-r + (r - (-r)) * rng.uniform(U, i, kind, 4 * blk + c) for c in range(3)])
    pos = d.pos + m.pos_norm_std * nrm(0) + uni(0, m.pos_unif_range)
    vel = d.vel + m.vel_norm_std * nrm(1) + uni(1, m.vel_unif_range)
    omega = d.omega + m.gyro_noise_density * nrm(2)
    theta = m.quat_norm_std * nrm(3) + uni(2, m.quat_unif_range)
    rng.skip_normal(N, 6)            # accelerometer noise: computed by the reference, never observed
    if m.gyro_norm_std != 0.:
        B = SITE_GYRO_BIAS
        pi_g_d, sigma_b = m.bias_coefficients()
        d.gyro_bias = pi_g_d * gyro_bias(d) + sigma_b * np.array([rng.normal(B, i, kind, c) for c in range(3)])
        omega = d.omega + d.gyro_bias + m.gyro_random_walk * np.array([rng.normal(B, i, kind, 4 + c) for c in range(3)])
    q = quat_x_quat(qo.rot2quat(d.rot), quat_from_small_angle(theta))
    return pos, vel, qo.quat2R(q[0], q[1], q[2], q[3]), omega


_default_self_observation = qo.self_observation


def self_observation(d, cfg, P, room_box, rng, i, site):
    """get_state.py:6-72 under the configured model; the oracle's own function for every other config."""
    m = getattr(cfg, 'noise', None)
    if m is None or not cfg.sense_noise:
        return _default_self_observation(d, cfg, P, room_box, rng, i, site)
    pos, vel, rot, omega = noisy_state(d, m, rng, i, _KIND[site])
    parts = [pos - d.goal[:3], vel, rot.flatten(), omega]
    if cfg.obs_repr == 'xyz_vxyz_R_omega_floor':
        parts.append((pos[2],))
    elif cfg.obs_repr == 'xyz_vxyz_R_omega_wall':
        parts.append(np.clip(pos - room_box[0], 0.0, 5.0))
        parts.append(np.clip(room_box[1] - pos, 0.0, 5.0))
    return np.concatenate(parts)


qo.self_observation = self_observation          # OracleEnv.reset / step look the function up in their module


def noise_config(kw):
    """EnvConfig of a fixture's keyword set, with its noise model attached."""
    cfg = config_from_case(kw)
    cfg.sense_noise = kw.get('sense_noise', 'default') is not None
    cfg.noise = noise_model(kw.get('sense_noise', 'default'))
    return cfg


def replay_noise_golden(g, make_scenario):
    """oracle/replay.py's replay for the fixtures of oracle/gen_golden_noise.py (Crazyflie, noise dict), recording the
    gyro bias of every drone after every step as well.  make_scenario(mode, cfg, rng) -> host scenario object."""
    case = json.loads(str(g['case_json']))
    kw, T, seed = case['kw'], case['T'], case['seed']
    cfg = noise_config(kw)
    n = cfg.num_agents
    rng = NoiseReplayRng(seed, seed + 1, [seed + 100 + i for i in range(n)])
    env = qo.OracleEnv(cfg, rng, qo.ReferenceEpisodeSource(make_scenario(kw.get('quads_mode', 'static_same_goal'), cfg, rng.py)))
    out = dict(obs0=env.reset())
    keys = ('pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou', 'on_floor')
    rec = dict(rewards=np.zeros((T, n)), dones=np.zeros((T, n), dtype=bool), goals=np.zeros((T, n, 3)),
               infos=np.full((T, n, len(INFO_KEYS)), np.nan), gyro_bias=np.zeros((T, n, 3)))
    obs, states = {}, {k: {} for k in keys}
    want_obs, want_state = set(int(t) for t in g['obs_t']), set(int(t) for t in g['state_t'])
    for t in range(T):
        for k in np.where(g['plant_t'] == t)[0]:
            d = env.drones[int(g['plant_i'][k])]
            d.pos, d.vel = g['plant_pos'][k].copy(), g['plant_vel'][k].copy()
            d.rot, d.omega = g['plant_rot'][k].copy(), g['plant_omega'][k].astype(np.float32).astype(np.float64)
            d.acc = np.zeros(3)
            d.accelerometer = np.array([0., 0., 9.81])
        o, r, dn, inf = env.step(g['actions'][t])
        if t in want_obs:
            obs[t] = o
        rec['rewards'][t], rec['dones'][t] = r, dn
        for i in range(n):
            for k, key in enumerate(INFO_KEYS):
                if key in inf[i]['rewards']:
                    rec['infos'][t, i, k] = inf[i]['rewards'][key]
        rec['goals'][t] = np.array([d.goal for d in env.drones])
        rec['gyro_bias'][t] = np.array([gyro_bias(d) for d in env.drones])
        if t in want_state:
            for k in keys:
                states[k][t] = np.array([getattr(d, k) for d in env.drones])
    out.update(rec, obs=np.array([obs[int(t)] for t in g['obs_t']]),
               **{'state_' + k: np.array([states[k][int(t)] for t in g['state_t']]) for k in keys})
    return out, env
