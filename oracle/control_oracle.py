"""CPU oracle of the reference's other controllers — TEST INFRASTRUCTURE ONLY.

QuadrotorEnvMulti(raw_control=False) steps every drone with NonlinearPositionController (quadrotor_control.py:253-330, the
Mellinger controller, tf_control = False): it ignores the action and computes the motor commands from the drone's state
and goal.  QuadrotorEnvMulti(raw_control_zero_middle=False) keeps RawControl with actions in [0, 1]: clip(action, 0, 1)
is the motor command (:37-57).  Rewards keep the raw action in both (quadrotor_single.py:347-349).

This module extends oracle/quadswarm_oracle.py with both without changing it: an EnvConfig that carries
`control = POSITION` or `control = RAW_UNIT` gets that controller; every other EnvConfig keeps RawControl with
zero_action_middle.  Importing the module installs the dispatch (after the sensor-noise, initial-state and numpy-path
extensions, so that all of them combine).
"""
import numpy as np

from . import quadswarm_oracle as qo
from . import replay
from . import sensor_noise_oracle as sno
from . import numpy_path_oracle as npo     # its dispatch is installed first; this module wraps it

RAW, RAW_UNIT, POSITION = 'raw', 'raw_unit', 'position'
KP_P, KD_P = 4.5, 3.5                    # quadrotor_control.py:266
KP_A, KD_A = 200.0, 50.0                 # :267
PROP_CCW = np.array([-1., 1., -1., 1.])  # quadrotor_dynamics.py:47


def jacobian(P):
    """quadrotor_jacobian(dynamics), quadrotor_control.py:158-169, of a QuadParams (thrust_max / torque_max scalar or per
    motor)."""
    thrust_max = np.broadcast_to(np.asarray(P.thrust_max, dtype=np.float64), (4,))
    torque_max = np.broadcast_to(np.asarray(P.torque_max, dtype=np.float64), (4,))
    torque = thrust_max * np.array(P.prop_crossproducts).T
    torque[2, :] = torque_max * np.array(P.prop_ccw)
    thrust = thrust_max * np.ones((1, 4))
    dw = (1.0 / np.array(P.inertia))[:, None] * torque
    dv = thrust / P.mass
    return np.vstack([dv, dw])


def jacobian_inverse(P):
    """NonlinearPositionController.Jinv, quadrotor_control.py:257-258."""
    return np.linalg.inv(jacobian(P))


def _normalize(x):
    """quad_utils.normalize, :80-86."""
    n = (x[0] ** 2 + x[1] ** 2 + x[2] ** 2) ** 0.5
    return x if n < 0.00001 else x / n


def position_command(d, P):
    """NonlinearPositionController.step, quadrotor_control.py:282-330: the motor commands of drone `d` (state at the start
    of the control step, its goal) under constants P."""
    to_goal = d.goal[:3] - d.pos
    n = (to_goal[0] ** 2 + to_goal[1] ** 2 + to_goal[2] ** 2) ** 0.5
    e_p = -(to_goal if n <= 4.0 else (4.0 / n) * to_goal)                 # clamp_norm, quad_utils.py:112-116
    acc_des = -KP_P * e_p - KD_P * d.vel + np.array([0, 0, qo.GRAV])
    zb_des = _normalize(acc_des)
    yb_des = _normalize(np.cross(zb_des, np.array([1.0, 0.0, 0.0])))
    xb_des = np.cross(yb_des, zb_des)
    R_des = np.column_stack((xb_des, yb_des, zb_des))
    R = d.rot
    M = R_des.T @ R - R.T @ R_des
    e_R = 0.5 * np.array([M[2, 1], M[0, 2], M[1, 0]])
    e_R[2] *= 0.2
    dw_des = -KP_A * e_R - KD_A * d.omega
    thrust_mag = np.dot(acc_des, R[:, 2])
    thrusts = np.matmul(jacobian_inverse(P), np.append(thrust_mag, dw_des))
    thrusts[thrusts < 0] = 0
    thrusts[thrusts > 1] = 1
    return thrusts


def _control(d):
    return getattr(getattr(d, 'env_cfg', None), 'control', RAW)


_default_step = qo.OracleEnv.step


def _step(self, actions):
    """OracleEnv.step; every drone also keeps its raw action of this step (RAW_UNIT maps it itself)."""
    for d, a in zip(self.drones, actions):
        d.action = np.asarray(a, dtype=np.float64)
    return _default_step(self, actions)


_default_dynamics_substep = qo.dynamics_substep


def dynamics_substep(d, P, cmd, thr_noise, room_box, rng, i, substep):
    """The sub-step of the drone's dynamics path with the command of its env's controller: computed once per control step,
    at the first sub-step, from the state at the start of the step (QuadrotorSingle._step, quadrotor_single.py:345)."""
    mode = _control(d)
    if mode != RAW:
        if substep == 0:
            d.control_cmd = position_command(d, P) if mode == POSITION else np.clip(d.action, 0.0, 1.0)
        cmd = d.control_cmd
    return _default_dynamics_substep(d, P, cmd, thr_noise, room_box, rng, i, substep)


qo.OracleEnv.step = _step
qo.dynamics_substep = dynamics_substep


def enable(cfg, raw_control=True, raw_control_zero_middle=True):
    """Give an EnvConfig the controller of QuadrotorEnvMulti(raw_control, raw_control_zero_middle)."""
    cfg.control = POSITION if not raw_control else (RAW if raw_control_zero_middle else RAW_UNIT)
    return cfg


def config_from_case(kw):
    """replay.config_from_case with the case's noise model, dynamics path and controller."""
    cfg = sno.noise_config(kw)
    if kw.get('use_numba', True) is False:
        npo.enable(cfg)
    return enable(cfg, kw.get('raw_control', True), kw.get('raw_control_zero_middle', True))


def replay_control_golden(g, make_scenario):
    """oracle/replay.py's replay for the fixtures of oracle/gen_golden_control.py."""
    import json
    kw = json.loads(str(g['case_json']))['kw']
    saved = replay.config_from_case, replay.ReplayRng
    replay.config_from_case = config_from_case
    if kw.get('use_numba', True) is False:
        replay.ReplayRng = npo.NumpyReplayRng
    try:
        return replay.replay_golden(g, make_scenario)
    finally:
        replay.config_from_case, replay.ReplayRng = saved
