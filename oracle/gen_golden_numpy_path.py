"""Generate tests/golden/numpy_path_*.npz by running the UNMODIFIED reference with use_numba=False — TEST INFRASTRUCTURE
ONLY.

Run in a container where /root/reference is mounted:  python -m oracle.gen_golden_numpy_path
Same recording as oracle/gen_golden.py (seeds, actions, planted states, the reference's observations / rewards / dones /
reward terms / states); every env is built with use_numba=False, so the drones step QuadrotorDynamics.step1 +
floor_interaction (quadrotor_dynamics.py:225-346, 389-457) and draw their thrust and sensor noise from numpy's global
stream.  The `floor` plants (case floor_8) put drones between the arm and 0.05 m above the floor, slide them on it, push
one straight down on it with no horizontal velocity (the atan2(-0, -0) friction direction) and land others upside down away
from the origin, so that the landing-yaw loop retries (tests/test_numpy_path.py checks that the fixture holds all of it).
"""
import os
import sys

import numpy as np

from . import gen_golden
from .gen_golden import rotx, rotz

C3_REW = dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0, quadcol_bin=5.0,
              quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
FLOOR_PLANT_AT = [0, 30, 70]
CASES = [
    # planted floor states (below)
    dict(name='floor_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=1.0, quads_mode='static_diff_goal',
                                 obs_repr='xyz_vxyz_R_omega_floor', use_numba=False),
         T=160, seed=401, obs_stride=1, plant='floor', plant_at=FLOOR_PLANT_AT),
    # c3: pillars, downwash, floor observation (the responses' numpy-stream draws interleave with the noise draws)
    dict(name='c3_obstacles_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=1.0, use_obstacles=True,
                                        use_downwash=True, quads_mode='o_random', obs_repr='xyz_vxyz_R_omega_floor',
                                        rew_coeff=C3_REW, use_numba=False),
         T=170, seed=402, obs_stride=1, plant='obst', plant_at=[5, 120]),
    # a sense_noise dict with the gyro-bias model, wall observation, planted room contacts
    dict(name='wall_gyro_bias_6', kw=dict(num_agents=6, neighbor_visible_num=2, ep_time=0.6, quads_mode='static_diff_goal',
                                          obs_repr='xyz_vxyz_R_omega_wall', use_numba=False,
                                          sense_noise=dict(gyro_norm_std=1.0, gyro_bias_correlation_time=0.05,
                                                           gyro_noise_density=0.005, gyro_random_walk=0.02,
                                                           pos_unif_range=0.01, quat_norm_std=0.01)),
         T=130, seed=403, obs_stride=1, plant='room', plant_at=[0, 65]),
    # another physical model with rotor drag and rolling moment (dynamics_change), planted room and floor contacts
    dict(name='defaultquad_drag_4', kw=dict(num_agents=4, neighbor_visible_num=2, ep_time=0.6, quads_mode='static_diff_goal',
                                            dynamics_params='DefaultQuad', use_numba=False,
                                            dynamics_change=dict(noise=dict(thrust_noise_ratio=0.05),
                                                                 damp=dict(vel=0, omega_quadratic=0),
                                                                 motor=dict(C_drag=0.01, C_roll=0.001))),
         T=130, seed=404, obs_stride=1, plant='room4', plant_at=[0, 60]),
]


def _plants_floor(env, rs):
    """One call per entry of FLOOR_PLANT_AT.  First: two drones between the arm and 0.05 m (the numpy path's floor, the
    njit path's air), two upright landings, three upside-down landings away from the origin.  Then: drones on the floor
    pushed sideways (sliding friction) and one pushed straight down (vx = vy = +0).  Last: more upside-down landings."""
    k = _plants_floor.calls
    _plants_floor.calls += 1
    up, down = rotz(rs.uniform(-3, 3)), rotz(rs.uniform(-3, 3)) @ rotx(np.pi - 0.3)
    if k == 0:
        return [dict(i=0, pos=[1.0, -1.5, 0.048], vel=[0.3, 0.1, 0.0], rot=up, omega=[0., 0., 0.]),
                dict(i=1, pos=[-0.5, 2.0, 0.0495], vel=[0.0, 0.0, 0.0], rot=rotz(0.7), omega=[0., 0., 0.2]),
                dict(i=2, pos=[3.0, 2.0, 0.06], vel=[0.0, 0.0, -2.0], rot=down, omega=[0.1, 0., 0.]),
                dict(i=3, pos=[-2.5, 3.5, 0.07], vel=[0.2, -0.1, -1.5], rot=rotz(2.0) @ rotx(np.pi), omega=[0., 0.3, 0.]),
                dict(i=4, pos=[4.0, -1.0, 0.055], vel=[0.0, 0.0, -1.0], rot=rotz(-1.0) @ rotx(2.9), omega=[0., 0., 0.]),
                dict(i=5, pos=[-3.0, -3.0, 0.06], vel=[1.0, -0.5, -1.0], rot=up, omega=[0., 0., 0.])]
    if k == 1:
        return [dict(i=0, pos=[1.2, -1.4, 0.05], vel=[0.8, -0.4, 0.0], rot=rotz(0.2), omega=[0., 0., 0.]),
                dict(i=1, pos=[-0.5, 2.0, 0.05], vel=[0.0, 0.0, -0.2], rot=rotz(0.7), omega=[0., 0., 0.]),
                dict(i=2, pos=[3.0, 2.0, 0.05], vel=[-0.5, 0.6, 0.0], rot=rotz(-2.0), omega=[0., 0., 0.]),
                dict(i=5, pos=[-3.0, -3.0, 0.05], vel=[0.0, 1.2, -0.1], rot=rotz(1.0), omega=[0., 0., 0.])]
    return [dict(i=3, pos=[-4.0, 0.5, 0.06], vel=[0.0, 0.0, -1.0], rot=down, omega=[0., 0., 0.]),
            dict(i=4, pos=[2.0, 4.0, 0.052], vel=[0.0, 0.0, -0.5], rot=rotz(1.5) @ rotx(np.pi - 0.1), omega=[0., 0., 0.]),
            dict(i=6, pos=[-1.0, -4.0, 0.06], vel=[0.3, 0.0, -1.0], rot=rotz(-0.5) @ rotx(np.pi), omega=[0., 0., 0.]),
            dict(i=7, pos=[3.5, -3.5, 0.058], vel=[0.0, 0.0, -1.0], rot=rotz(0.1) @ rotx(np.pi - 0.4), omega=[0., 0., 0.])]


def run_case(case):
    """gen_golden.run_reference_case; the `floor` plants go through its obstacle-plant hook."""
    if case.get('plant') != 'floor':
        return gen_golden.run_reference_case(case)
    saved = gen_golden._plants_obst
    _plants_floor.calls = 0
    gen_golden._plants_obst = _plants_floor
    try:
        return gen_golden.run_reference_case(case)
    finally:
        gen_golden._plants_obst = saved


def main(argv=None):
    only = set(sys.argv[1:] if argv is None else argv)
    for case in CASES:
        if only and case['name'] not in only:
            continue
        out = run_case(case)
        path = os.path.join(gen_golden.GOLDEN_DIR, f"numpy_path_{case['name']}.npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: T={case['T']} D={out['obs0'].shape[1]} -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == '__main__':
    main()
