"""Generate tests/golden/sensor_noise_*.npz by running the UNMODIFIED reference with dicts of SensorNoise parameters — TEST
INFRASTRUCTURE ONLY.

Run in a container where /root/reference is mounted:  python -m oracle.gen_golden_noise
Same recording as oracle/gen_golden.py (seeds, actions, planted states, the reference's observations / rewards / dones /
reward terms / states), plus the gyro bias of every drone after every step (SensorNoise.gyro_bias, sensor_noise.py:101,228).
The files are not named ref_*.npz: tests/test_oracle_vs_reference.py replays those with the default noise set.
"""
import os
import sys

import numpy as np

from . import gen_golden
from . import ref_harness as rh

CASES = [
    # uniform ranges and rotation noise; planted collision clusters (contact re-draws) and 0.5 s episodes (auto-resets)
    dict(name='cluster_8_unif_quat', kw=dict(num_agents=8, neighbor_visible_num=6, ep_time=0.5, quads_mode='static_same_goal',
                                             sense_noise=dict(pos_norm_std=0.01, pos_unif_range=0.02, vel_norm_std=0.02,
                                                              vel_unif_range=0.05, quat_norm_std=0.02, quat_unif_range=0.03,
                                                              gyro_noise_density=0.001)),
         T=130, seed=201, obs_stride=1, plant='cluster', plant_at=[0, 40, 80]),
    # c3-like env (pillars, downwash, floor observation) with the stateful gyro model and rotation noise
    dict(name='c3_gyro_bias_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=0.8, use_obstacles=True, use_downwash=True,
                                        quads_mode='o_random', obs_repr='xyz_vxyz_R_omega_floor',
                                        rew_coeff=dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0,
                                                       quadcol_bin=5.0, quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0),
                                        sense_noise=dict(gyro_norm_std=0.1, quat_norm_std=0.01, acc_static_noise_std=0.01)),
         T=180, seed=202, obs_stride=1, plant='obst', plant_at=[5, 100]),
    # wall observation, room contacts, a short bias correlation time: the bias matters within the run
    dict(name='wall_gyro_bias_6', kw=dict(num_agents=6, neighbor_visible_num=2, ep_time=0.6, quads_mode='static_diff_goal',
                                          obs_repr='xyz_vxyz_R_omega_wall',
                                          sense_noise=dict(gyro_norm_std=1.0, gyro_bias_correlation_time=0.05,
                                                           gyro_noise_density=0.005, gyro_random_walk=0.02,
                                                           pos_unif_range=0.01)),
         T=130, seed=203, obs_stride=1, plant='room', plant_at=[0, 65]),
]


def run_case(case):
    """gen_golden.run_reference_case with the gyro bias recorded after every step."""
    log = []
    make = rh.make_reference_env

    def make_recording(**kw):
        env = make(**kw)
        step = env.step

        def recorded_step(actions):
            r = step(actions)
            log.append(np.array([e.sense_noise.gyro_bias for e in env.envs], dtype=np.float64))
            return r
        env.step = recorded_step
        return env

    rh.make_reference_env = make_recording
    try:
        out = gen_golden.run_reference_case(case)
    finally:
        rh.make_reference_env = make
    out['gyro_bias'] = np.array(log)
    return out


def main(argv=None):
    only = set(sys.argv[1:] if argv is None else argv)
    for case in CASES:
        if only and case['name'] not in only:
            continue
        out = run_case(case)
        path = os.path.join(gen_golden.GOLDEN_DIR, f"sensor_noise_{case['name']}.npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: T={case['T']} D={out['obs0'].shape[1]} -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == '__main__':
    main()
