"""Generate tests/golden/init_state_*.npz by running the UNMODIFIED reference with init_random_state=True — TEST
INFRASTRUCTURE ONLY.

Run in a container where /root/reference is mounted:  python -m oracle.gen_golden_init_state
Same recording as oracle/gen_golden.py (seeds, actions, planted states, the reference's observations / rewards / dones /
reward terms / states).  The reference's env factory hard-codes init_random_state=False, so the option is switched on in
every QuadrotorSingle after construction (quadrotor_single.py:149; it is read only in _reset, :407).  Short episodes: every
case runs through several auto-resets.  The seeds are chosen so that the fixtures hold upside-down spawns, fwd re-draws of
rand_uniform_rot3d and floor contacts right after a spawn (tests/test_init_random_state.py checks all three).
"""
import os
import sys

import numpy as np

from . import gen_golden
from . import ref_harness as rh

C3_REW = dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0, quadcol_bin=5.0,
              quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
CASES = [
    dict(name='same_goal_8', kw=dict(num_agents=8, neighbor_visible_num=6, ep_time=0.4, quads_mode='static_same_goal'),
         T=130, seed=301, obs_stride=1),
    # c3-like: pillars, downwash, floor observation
    dict(name='c3_obstacles_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=0.5, use_obstacles=True, use_downwash=True,
                                        quads_mode='o_random', obs_repr='xyz_vxyz_R_omega_floor', rew_coeff=C3_REW),
         T=160, seed=302, obs_stride=1),
    # wall observation, planted room contacts, a sense_noise dict (the custom noise model)
    dict(name='wall_noise_6', kw=dict(num_agents=6, neighbor_visible_num=2, ep_time=0.4, quads_mode='static_diff_goal',
                                      obs_repr='xyz_vxyz_R_omega_wall',
                                      sense_noise=dict(pos_unif_range=0.01, quat_norm_std=0.01, gyro_noise_density=0.001)),
         T=130, seed=303, obs_stride=1, plant='room', plant_at=[0, 65]),
    # another physical model (per-drone constants)
    dict(name='defaultquad_4', kw=dict(num_agents=4, neighbor_visible_num=2, ep_time=0.4, quads_mode='static_diff_goal',
                                       dynamics_params='DefaultQuad'), T=130, seed=304, obs_stride=1),
]


def run_case(case):
    """gen_golden.run_reference_case on an env whose drones spawn in random initial states."""
    make = rh.make_reference_env

    def make_random_init(**kw):
        env = make(**kw)
        for e in env.envs:
            e.init_random_state = True
        return env

    rh.make_reference_env = make_random_init
    try:
        return gen_golden.run_reference_case(case)
    finally:
        rh.make_reference_env = make


def main(argv=None):
    only = set(sys.argv[1:] if argv is None else argv)
    for case in CASES:
        if only and case['name'] not in only:
            continue
        out = run_case(case)
        path = os.path.join(gen_golden.GOLDEN_DIR, f"init_state_{case['name']}.npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: T={case['T']} D={out['obs0'].shape[1]} -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == '__main__':
    main()
