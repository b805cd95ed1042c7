"""CPU oracle of the reference's numpy dynamics path (use_numba=False) — TEST INFRASTRUCTURE ONLY.

QuadrotorEnvMulti(use_numba=False) steps every drone with QuadrotorDynamics.step1 + floor_interaction
(quadrotor_dynamics.py:225-346, 389-457) instead of the njit step1_numba + floor_interaction_numba (:348-383, :569-639),
draws its thrust noise from OUNoise (quad_utils.py:253-279) and its observations from SensorNoise.add_noise
(sensor_noise.py:112-170).  This module extends oracle/quadswarm_oracle.py with that path without changing it: an
EnvConfig that carries `use_numba = False` gets the numpy path; every other EnvConfig keeps the oracle's default path.
Importing the module installs the dispatch (after oracle/sensor_noise_oracle.py's and oracle/init_state_oracle.py's, so
the three combine).

What differs from the njit path:
  * floor threshold and snap height 0.05 for every drone (:75, :392-393) instead of the arm (:378); the threshold margin
    is measured against 0.05;
  * at rest only when |vel| == 0 (:406) instead of |vel| < 1e-6 (:586);
  * sliding friction (cos, sin)(atan2(-vy, -vx)), subtracted (:419-422): it pushes along the velocity;
  * an upside-down first contact re-draws randyaw() until rot[:, 0] . to_xyhat(-pos) >= 0.5 (:434-437);
  * OUNoise keeps theta and sigma in float64 (the njit OUNoiseNumba stores them as float32);
  * SensorNoise.add_noise draws the gyro normal only when the gyro-bias model is off (:138-142), and the bias draws come
    in the middle of the call, before the rotation noise.
Rotor drag (:260-289) is the term the oracle already applies for a model with C_drag / C_roll != 0.

Random sources, as in the oracle:
  * ReplayRng – NumpyReplayRng: OU, sensor noise (default set and a noise dict) and the landing yaw come from numpy's
                global stream (py), in the reference's order; the collision responses keep their streams;
  * PhiloxRng – keyed draws; the landing yaw at SITE_FLOOR_YAW_NP (j = sub-step, v = try), the twin of qs_rng.cuh.  OU
                and sensor noise keep their sites.
"""
import math

import numpy as np

from . import philox as px
from . import quadswarm_oracle as qo
from . import replay
from . import sensor_noise_oracle as sno
from . import init_state_oracle  # noqa: F401  (its dispatch is installed first; this module wraps it)

SITE_FLOOR_YAW_NP = 23     # (i,j) uniforms v[k], j = sub-step, k = rejection try of randyaw()   quadrotor_dynamics.py:434-437
FLOOR_YAW_MAX_TRIES = px.RESET_YAW_MAX_TRIES     # cap of the keyed loop (the reference's is unbounded)
FLOOR_THRESHOLD = 0.05     # QuadrotorDynamics.floor_threshold, quadrotor_dynamics.py:75
OU_THETA, OU_SIGMA = 0.15, 0.2 * 0.05            # OUNoise(4, sigma=0.2 * thrust_noise_ratio), quad_utils.py:256; :171-173
_NP_SITES = {px.SITE_OU, SITE_FLOOR_YAW_NP, px.SITE_SENSOR0, px.SITE_SENSOR1, px.SITE_SENSOR_RESET,
             sno.SITE_NOISE_N, sno.SITE_NOISE_U, sno.SITE_GYRO_BIAS}


class NumpyReplayRng(qo.ReplayRng):
    """ReplayRng of the numpy path: the draws that the njit path takes from numba's stream and that the numpy path takes
    from numpy's global one (thrust noise, sensor noise, landing yaw) are served by `py`."""

    def _stream(self, site):
        return self.py if site in _NP_SITES else super()._stream(site)


def _numpy_path(d):
    """The drone's env runs on a config with use_numba = False (read at every call: enable() may come after the envs)."""
    return getattr(getattr(d, 'env_cfg', None), 'use_numba', True) is False


_default_ou_noise_step = qo.ou_noise_step


def ou_noise_step(d, P, rng, i):
    """OUNoise.noise, quad_utils.py:275-279: theta and sigma in float64.  A drone with the default constants has the
    float32 sigma of OUNoiseNumba in its QuadParams; the numpy path's value is 0.2 * 0.05."""
    if not _numpy_path(d):
        return _default_ou_noise_step(d, P, rng, i)
    sigma = OU_SIGMA if P.ou_sigma == qo.QuadParams.ou_sigma else P.ou_sigma
    z = np.array([rng.normal(px.SITE_OU, i, 0, v) for v in range(4)])
    d.ou = d.ou + (OU_THETA * (P.ou_mu - d.ou) + sigma * z)
    return d.ou


def landing_yaw(d, rng, i, substep):
    """randyaw() until rot[:, 0] . to_xyhat(-pos) >= 0.5 (quadrotor_dynamics.py:434-437, quad_utils.py:120-124, 207-209);
    keyed: at most FLOOR_YAW_MAX_TRIES tries.  Returns (rot, tries); records the margin of every test on the drone."""
    v = -d.pos.copy()
    v[2] = 0
    n = (v[0] ** 2 + v[1] ** 2 + v[2] ** 2) ** 0.5
    xyhat = v if n < 0.00001 else v / n
    k = 0
    while True:
        theta = -np.pi + (np.pi - (-np.pi)) * rng.uniform(SITE_FLOOR_YAW_NP, i, substep, k)
        c, s = np.cos(theta), np.sin(theta)
        rot = np.array([[c, -s, 0.], [s, c, 0.], [0., 0., 1.]])
        k += 1
        dot = float(np.dot(rot[:, 0], xyhat))
        d.margin = min(d.margin, abs(dot - 0.5))
        if dot >= 0.5 or (rng.keyed and k >= FLOOR_YAW_MAX_TRIES):
            return rot, k


_default_dynamics_substep = qo.dynamics_substep


def dynamics_substep(d, P, cmd, thr_noise, room_box, rng, i, substep):
    """QuadrotorDynamics.step1 (quadrotor_dynamics.py:225-346) with floor_interaction (:389-457) for a drone on the numpy
    path; the oracle's njit sub-step otherwise.  Counts on the drone: landing_yaw_tries (randyaw draws of upside-down
    first contacts), landings_upside_down, slides (sliding-friction sub-steps), slide_corner (of those, vx = vy = 0)."""
    if not _numpy_path(d):
        return _default_dynamics_substep(d, P, cmd, thr_noise, room_box, rng, i, substep)
    dt = P.dt
    inertia = np.array(P.inertia)
    thrust_cmds = np.clip(cmd, 0., 1.)
    motor_tau = P.motor_tau_up * np.ones(4)
    motor_tau[thrust_cmds < d.thrust_cmds_damp] = P.motor_tau_down
    motor_tau[motor_tau > 1.] = 1.
    thrust_rot = thrust_cmds ** 0.5
    d.thrust_rot_damp = motor_tau * (thrust_rot - d.thrust_rot_damp) + d.thrust_rot_damp
    d.thrust_cmds_damp = d.thrust_rot_damp ** 2
    d.thrust_cmds_damp = np.clip(d.thrust_cmds_damp + thrust_cmds * thr_noise, 0.0, 1.0)
    lin = P.motor_linearity
    thrusts = P.thrust_max * ((1 - lin) * d.thrust_cmds_damp ** 2 + lin * d.thrust_cmds_damp)    # angvel2thrust, :95-102
    torques = np.array(P.prop_crossproducts) * thrusts[:, None]
    torques[:, 2] += P.torque_max * np.array(P.prop_ccw) * d.thrust_cmds_damp
    torque = np.sum(torques, axis=0)
    rotor_drag_force = np.zeros(3)
    if P.c_drag != 0 or P.c_roll != 0:          # :260-289
        prop_pos = np.array(P.prop_pos)
        vel_body = d.rot.T @ d.vel
        v_rotor = vel_body + np.cross(d.omega, prop_pos)
        v_rotor[:, 2] = 0.
        sq = np.sqrt(d.thrust_cmds_damp)[:, None]
        rotor_drag_fi = -P.c_drag * sq * v_rotor
        rotor_drag_force = np.sum(rotor_drag_fi, axis=0)
        rotor_drag_torque = np.sum(np.cross(rotor_drag_fi, prop_pos), axis=0)
        rotor_roll_torque = np.sum(-P.c_roll * np.array(P.prop_ccw)[:, None] * sq * v_rotor, axis=0)
        rotor_visc_torque = rotor_drag_torque + rotor_roll_torque
        vel_norm = np.linalg.norm(vel_body)
        rdf_norm = np.linalg.norm(rotor_drag_force)
        rdf_norm_clip = np.clip(rdf_norm, 0., vel_norm * P.mass / (2 * dt))
        if rdf_norm > qo.EPS_DYN:
            rotor_drag_force = (rotor_drag_force / rdf_norm) * rdf_norm_clip
        rvt_norm = np.linalg.norm(rotor_visc_torque)
        rvt_norm_clipped = np.clip(rvt_norm, 0., np.linalg.norm(d.omega * inertia) / (2 * dt))
        if rvt_norm > qo.EPS_DYN:
            rotor_visc_torque = (rotor_visc_torque / rvt_norm) * rvt_norm_clipped
        torque = torque + rotor_visc_torque
    thrust = np.array([0., 0., np.sum(thrusts)])

    omega_vec = d.rot @ d.omega                 # :298-306
    wx, wy, wz = omega_vec
    omega_norm = np.linalg.norm(omega_vec)
    if omega_norm != 0:
        K = np.array([[0, -wz, wy], [wz, 0, -wx], [-wy, wx, 0]]) / omega_norm
        rot_angle = omega_norm * dt
        d.rot = (np.eye(3) + np.sin(rot_angle) * K + (1. - np.cos(rot_angle)) * (K @ K)) @ d.rot
    d.since_last_svd += dt                      # :309-314
    if d.since_last_svd > P.since_last_svd_limit:
        u, s, v = np.linalg.svd(d.rot)
        d.rot = u @ v
        d.since_last_svd = 0
    omega = d.omega                             # :319-325
    omega_dot = (1.0 / inertia) * (qo_cross(-omega, inertia * omega) + torque)
    omega_damp_quadratic = np.clip(P.damp_omega_quadratic * omega ** 2, 0.0, 1.0)
    d.omega = np.clip(omega + (1.0 - omega_damp_quadratic) * dt * omega_dot, -P.omega_max, P.omega_max)
    d.pos = d.pos + dt * d.vel                  # :329-336
    pos_before_clip = d.pos.copy()
    _m = np.abs(np.concatenate([pos_before_clip - room_box[0], pos_before_clip - room_box[1]]))
    _m = _m[_m > 0]
    if len(_m):
        d.margin = min(d.margin, float(np.min(_m)))
    d.pos = np.clip(d.pos, room_box[0], room_box[1])
    d.crashed_wall = not np.array_equal(pos_before_clip[:2], d.pos[:2])
    d.crashed_ceiling = bool(pos_before_clip[2] > d.pos[2])

    # --- floor_interaction, :389-457
    sum_thr_drag = thrust + rotor_drag_force
    d.crashed_floor = False
    if d.pos[2] != FLOOR_THRESHOLD and d.pos[2] != room_box[0][2]:
        d.margin = min(d.margin, abs(float(d.pos[2]) - FLOOR_THRESHOLD))
    if d.pos[2] <= FLOOR_THRESHOLD:
        d.pos = np.array((d.pos[0], d.pos[1], FLOOR_THRESHOLD))
        force = d.rot @ sum_thr_drag
        if d.on_floor:
            d.rot = qo.yaw_only(d.rot)
            force_xy_magn = np.linalg.norm(np.array([force[0], force[1]]))
            friction_xy_magn = P.mu * (P.mass * qo.GRAV - force[2])
            if np.linalg.norm(d.vel) == 0.0:
                if force_xy_magn != friction_xy_magn:
                    # at rest or not on the next sub-step is decided by this difference
                    d.margin = min(d.margin, abs(force_xy_magn - friction_xy_magn))
                force_xy_magn = max(force_xy_magn - friction_xy_magn, 0.)
                if force_xy_magn == 0.:
                    force[0] = 0.
                    force[1] = 0.
                else:
                    force_angle = math.atan2(force[1], force[0])
                    force[0] = force_xy_magn * math.cos(force_angle)
                    force[1] = force_xy_magn * math.sin(force_angle)
            else:
                friction_xy_angle = np.arctan2(-1.0 * d.vel[1], -1.0 * d.vel[0])
                force[0] = force[0] - np.cos(friction_xy_angle) * friction_xy_magn
                force[1] = force[1] - np.sin(friction_xy_angle) * friction_xy_magn
                d.slides = getattr(d, 'slides', 0) + 1
                if d.vel[0] == 0. and d.vel[1] == 0.:
                    d.slide_corner = getattr(d, 'slide_corner', 0) + 1
        else:
            d.on_floor = True
            d.crashed_floor = True
            d.vel = np.zeros(3)
            d.omega = np.zeros(3)                # float32 zeros in the reference (:430, set_state :188)
            if d.rot[2, 2] < 0:
                d.rot, tries = landing_yaw(d, rng, i, substep)
                d.landings_upside_down = getattr(d, 'landings_upside_down', 0) + 1
                d.landing_yaw_tries = getattr(d, 'landing_yaw_tries', 0) + tries
            else:
                d.rot = qo.yaw_only(d.rot)
            d.thrust_cmds_damp = np.zeros(4)
            d.thrust_rot_damp = np.zeros(4)
        d.acc = np.array((0., 0., -qo.GRAV)) + (1.0 / P.mass) * force
        d.acc[2] = np.maximum(0, d.acc[2])
    else:
        if d.on_floor:
            d.on_floor = False
        force = d.rot @ sum_thr_drag
        d.acc = np.array((0., 0., -qo.GRAV)) + (1.0 / P.mass) * force
    d.vel = (1.0 - P.vel_damp) * d.vel + dt * d.acc          # :342-346
    d.accelerometer = d.rot.T @ (d.acc + np.array([0., 0., qo.GRAV]))


def qo_cross(a, b):
    """quad_utils.cross."""
    return np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def noisy_state(d, m, rng, i, kind):
    """SensorNoise(**dict).add_noise (sensor_noise.py:112-170) for a rotation-matrix state: the twin of
    sensor_noise_oracle.noisy_state in the numpy call order — pos normal, pos uniform, vel normal, vel uniform, then either
    the gyro model's two normal triples (add_noise_to_omega, :221-231) or the gyro normal, theta normal, theta uniform,
    accelerometer (never observed).  The keyed draws are those of the njit model (same sites)."""
    N, U = sno.SITE_NOISE_N, sno.SITE_NOISE_U
    nrm = lambda blk: np.array([rng.normal(N, i, kind, 4 * blk + c) for c in range(3)])
    uni = lambda blk, r: np.array([-r + (r - (-r)) * rng.uniform(U, i, kind, 4 * blk + c) for c in range(3)])
    pos = d.pos + m.pos_norm_std * nrm(0) + uni(0, m.pos_unif_range)
    vel = d.vel + m.vel_norm_std * nrm(1) + uni(1, m.vel_unif_range)
    if m.gyro_norm_std != 0.:
        B = sno.SITE_GYRO_BIAS
        pi_g_d, sigma_b = m.bias_coefficients()
        d.gyro_bias = pi_g_d * sno.gyro_bias(d) + sigma_b * np.array([rng.normal(B, i, kind, c) for c in range(3)])
        omega = d.omega + d.gyro_bias + m.gyro_random_walk * np.array([rng.normal(B, i, kind, 4 + c) for c in range(3)])
    else:
        omega = d.omega + m.gyro_noise_density * nrm(2)
    theta = m.quat_norm_std * nrm(3) + uni(2, m.quat_unif_range)
    rng.skip_normal(N, 6)
    q = sno.quat_x_quat(qo.rot2quat(d.rot), sno.quat_from_small_angle(theta))
    return pos, vel, qo.quat2R(q[0], q[1], q[2], q[3]), omega


_noise_self_observation = qo.self_observation


def self_observation(d, cfg, P, room_box, rng, i, site):
    """get_state.py:6-72 over SensorNoise.add_noise for a noise dict on the numpy path.  The default set draws what the njit
    call draws, in the same order (NumpyReplayRng moves it to numpy's stream), so it keeps the oracle's function."""
    m = getattr(cfg, 'noise', None)
    if not _numpy_path(d) or m is None or not cfg.sense_noise:
        return _noise_self_observation(d, cfg, P, room_box, rng, i, site)
    pos, vel, rot, omega = noisy_state(d, m, rng, i, sno._KIND[site])
    parts = [pos - d.goal[:3], vel, rot.flatten(), omega]
    if cfg.obs_repr == 'xyz_vxyz_R_omega_floor':
        parts.append((pos[2],))
    elif cfg.obs_repr == 'xyz_vxyz_R_omega_wall':
        parts.append(np.clip(pos - room_box[0], 0.0, 5.0))
        parts.append(np.clip(room_box[1] - pos, 0.0, 5.0))
    return np.concatenate(parts)


_default_init = qo.OracleEnv.__init__


def _init(self, cfg, *args, **kwargs):
    """OracleEnv.__init__; every drone also keeps its env's config, which selects the path."""
    _default_init(self, cfg, *args, **kwargs)
    for d in self.drones:
        d.env_cfg = cfg


qo.ou_noise_step = ou_noise_step
qo.dynamics_substep = dynamics_substep
qo.self_observation = self_observation
qo.OracleEnv.__init__ = _init


def enable(cfg):
    """Put an EnvConfig on the numpy path (shared by every OracleEnv built on it)."""
    cfg.use_numba = False
    return cfg


def replay_numpy_path_golden(g, make_scenario):
    """oracle/replay.py's replay for the fixtures of oracle/gen_golden_numpy_path.py: the same replay, on a config on the
    numpy path (with the noise model of a sense_noise dict) and on the numpy path's streams."""
    saved = replay.config_from_case, replay.ReplayRng
    replay.config_from_case = lambda kw: enable(sno.noise_config(kw))
    replay.ReplayRng = NumpyReplayRng
    try:
        return replay.replay_golden(g, make_scenario)
    finally:
        replay.config_from_case, replay.ReplayRng = saved
