"""CPU oracle of random initial states (init_random_state=True) — TEST INFRASTRUCTURE ONLY.

QuadrotorSingle(init_random_state=True) (quadrotor_single.py:405-423, 3-D) spawns every drone, at every reset, from
QuadrotorDynamics.random_state (quadrotor_dynamics.py:193-206) instead of a level attitude facing the origin at rest.
This module extends oracle/quadswarm_oracle.py with that option without changing it: an EnvConfig that carries
`init_random_state = True` (and `init_vel_max` / `init_omega_max`) has its drones reset by reset_drone() below; every
other EnvConfig keeps the oracle's default path.  Importing the module installs the dispatch.

Random sources, as in the oracle:
  * ReplayRng – numpy's global stream, in the reference's order: the discarded position (3 uniforms), vel direction (3)
                and magnitude (1), omega direction (3) and magnitude (1), then rand_uniform_rot3d's normals (up, fwd,
                fwd re-draws).  randyaw() is not drawn in this branch.
  * PhiloxRng – keyed draws at the sites below, the twins of qs_rng.cuh, keyed by the episode like the spawn jitter.
"""
import numpy as np

from . import philox as px
from . import quadswarm_oracle as qo
from . import replay
from . import sensor_noise_oracle as sno

# ---- draw sites (must match qs_rng.cuh)
SITE_INIT_U = 21       # (i)  uniforms v0..2 vel direction, v3 vel magnitude, v4..6 omega direction, v7 omega magnitude
SITE_INIT_N = 22       # (i)  normals v0..2 up, v[4(t+1)..4(t+1)+2] fwd of try t
INIT_ROT_MAX_TRIES = 16     # cap of the fwd re-draw loop (the reference's is unbounded)
EPS = 1e-6                  # quadrotor_dynamics.py:13
MAX_INIT_VEL, MAX_INIT_OMEGA = 1.0, 2 * np.pi    # QuadrotorSingle.max_init_vel / max_init_omega, quadrotor_single.py:181-182
NEAR_DOT = 1e-5             # |fwd.up - 0.95| below this: float32 normals may decide the re-draw test the other way


def _uniform(rng, i, v):
    return rng.episode_draws.uniform(SITE_INIT_U, i, 0, v) if rng.keyed else rng.uniform(SITE_INIT_U, i, 0, v)


def _normal(rng, i, v):
    return rng.episode_draws.normal(SITE_INIT_N, i, 0, v) if rng.keyed else rng.normal(SITE_INIT_N, i, 0, v)


def _normalize(x):
    """quad_utils.py:80-86."""
    n = (x[0] ** 2 + x[1] ** 2 + x[2] ** 2) ** 0.5
    return x if n < 0.00001 else x / n


def random_state(rng, i, vel_max=MAX_INIT_VEL, omega_max=MAX_INIT_OMEGA):
    """QuadrotorDynamics.random_state without the position it returns (discarded by _reset, but drawn by ReplayRng) ->
    (vel, rot, omega, tries, margin): tries = fwd draws made, margin = smallest |fwd.up - 0.95| of the tries."""
    rng.skip_uniform(SITE_INIT_U, 3)                 # pos = np.random.uniform(-box, box, 3)
    lo, hi = -vel_max, vel_max
    vel = np.array([lo + (hi - lo) * _uniform(rng, i, v) for v in range(3)])
    vel = (0. + (vel_max - 0.) * _uniform(rng, i, 3)) / (np.linalg.norm(vel) + EPS) * vel
    lo, hi = -omega_max, omega_max
    omega = np.array([lo + (hi - lo) * _uniform(rng, i, 4 + v) for v in range(3)])
    omega = (0. + (omega_max - 0.) * _uniform(rng, i, 7)) / (np.linalg.norm(omega) + EPS) * omega
    # rand_uniform_rot3d, quad_utils.py:94-104
    up = _normalize(np.array([_normal(rng, i, v) for v in range(3)]))
    t, margin = 0, np.inf
    while True:
        fwd = _normalize(np.array([_normal(rng, i, 4 * (t + 1) + v) for v in range(3)]))
        t += 1
        dot = float(np.dot(fwd, up))
        margin = min(margin, abs(dot - 0.95))
        if not dot > 0.95 or (rng.keyed and t >= INIT_ROT_MAX_TRIES):
            break
    left = _normalize(_cross(up, fwd))
    up = _cross(fwd, left)
    return vel, np.column_stack([fwd, left, up]), omega, t, margin


def _cross(a, b):
    """quad_utils.cross."""
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


_default_reset_drone = qo.OracleEnv._reset_drone


def reset_drone(self, i, site_obs):
    """QuadrotorSingle._reset (quadrotor_single.py:387-447) with init_random_state; the oracle's own method otherwise.
    Counts on the env: init_resets (drone resets) and init_redraws (fwd re-draws); sets step_margin = 0 when a re-draw test sat within
    NEAR_DOT of its threshold (a parity test then skips the step's comparison and re-synchronises)."""
    cfg = self.cfg
    if not getattr(cfg, 'init_random_state', False):
        return _default_reset_drone(self, i, site_obs)
    d = self.drones[i]
    rng = self.rng
    box = self.box
    jitter = np.array([-box + (box - (-box)) * rng.uniform(px.SITE_SPAWN_U, i, 0, v) for v in range(3)])
    x, y, z = jitter + d.spawn_point
    if z < 0.75:
        z = 0.75
    vel, rot, omega, tries, margin = random_state(rng, i, cfg.init_vel_max, cfg.init_omega_max)
    self.init_resets = getattr(self, 'init_resets', 0) + 1
    self.init_redraws = getattr(self, 'init_redraws', 0) + tries - 1
    if margin < NEAR_DOT:
        self.init_near = getattr(self, 'init_near', 0) + 1
        self.step_margin = 0.0
    d.pos = np.array([x, y, z])
    d.vel = vel
    d.acc = np.zeros(3)
    d.accelerometer = np.array([0., 0., qo.GRAV])
    d.rot = rot
    d.omega = omega.astype(np.float32).astype(np.float64)      # set_state stores omega as float32 (quadrotor_dynamics.py:188)
    d.thrust_cmds_damp = np.zeros(4)
    d.thrust_rot_damp = np.zeros(4)
    d.on_floor = False
    d.crashed_floor = d.crashed_wall = d.crashed_ceiling = False
    return qo.self_observation(d, cfg, self.P, self.room_box, rng, i, site_obs)


qo.OracleEnv._reset_drone = reset_drone


def enable(cfg, vel_max=MAX_INIT_VEL, omega_max=MAX_INIT_OMEGA):
    """Attach the option to an EnvConfig (shared by every OracleEnv built on it)."""
    cfg.init_random_state = True
    cfg.init_vel_max, cfg.init_omega_max = float(vel_max), float(omega_max)
    return cfg


def replay_init_state_golden(g, make_scenario):
    """oracle/replay.py's replay for the fixtures of oracle/gen_golden_init_state.py: the same replay, on a config that
    carries the option (and the noise model of a sense_noise dict, oracle/sensor_noise_oracle.py)."""
    saved = replay.config_from_case, replay.ReplayRng
    replay.config_from_case = lambda kw: enable(sno.noise_config(kw))
    replay.ReplayRng = sno.NoiseReplayRng
    try:
        return replay.replay_golden(g, make_scenario)
    finally:
        replay.config_from_case, replay.ReplayRng = saved
