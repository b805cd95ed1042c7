"""Generate tests/golden/control_*.npz by running the UNMODIFIED reference with its other controllers — TEST
INFRASTRUCTURE ONLY.

Run in a container where /root/reference is mounted:  python -m oracle.gen_golden_control
Same recording as oracle/gen_golden.py (seeds, actions, planted states, the reference's observations / rewards / dones /
reward terms / states), on envs built with raw_control=False (NonlinearPositionController, quadrotor_control.py:253-330)
or raw_control_zero_middle=False (RawControl with actions in [0, 1]).  NonlinearPositionController.__init__ imports
tensorflow; oracle/stubs/tensorflow stands in for it.

Every planted state has omega = 0: set_state stores omega as float32 (quadrotor_dynamics.py:188), and the controller's
-kd_a * omega (:318) then rounds to float32 in the reference until the next sub-step; zero stays exact.
"""
import contextlib
import io
import os
import sys

import numpy as np

from . import gen_golden
from . import ref_harness as rh
from .gen_golden import rotx, rotz

C3_REW = dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0, quadcol_bin=5.0,
              quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
FACTORY_CHANGE = dict(noise=dict(thrust_noise_ratio=0.05), damp=dict(vel=0, omega_quadratic=0))
ZERO = [0., 0., 0.]


def make_reference_env(num_agents=8, ep_time=15.0, obs_repr='xyz_vxyz_R_omega', neighbor_visible_num=6,
                       neighbor_obs_type='pos_vel', use_obstacles=False, obst_density=0.2, obst_size=0.6,
                       obst_spawn_area=(8.0, 8.0), use_downwash=False, use_numba=True, quads_mode='static_same_goal',
                       room_dims=(10., 10., 10.), rew_coeff=None, collision_hitbox_radius=2.0,
                       collision_falloff_radius=4.0, sense_noise='default', quiet=True, dynamics_params='Crazyflie',
                       dyn_sampler_1=None, dynamics_change=None, dynamics_randomize_every=None, raw_control=True,
                       raw_control_zero_middle=True):
    """ref_harness.make_reference_env with the controller keywords of QuadrotorEnvMulti."""
    rh._ensure_path()
    from gym_art.quadrotor_multi.quadrotor_multi import QuadrotorEnvMulti
    if rew_coeff is None:
        rew_coeff = dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0,
                         quadcol_bin=5.0, quadcol_bin_smooth_max=10.0, quadcol_bin_obst=5.0)
    with contextlib.redirect_stdout(io.StringIO()) if quiet else contextlib.nullcontext():
        return QuadrotorEnvMulti(
            num_agents=num_agents, ep_time=ep_time, rew_coeff=rew_coeff, obs_repr=obs_repr,
            neighbor_visible_num=neighbor_visible_num, neighbor_obs_type=neighbor_obs_type,
            collision_hitbox_radius=collision_hitbox_radius, collision_falloff_radius=collision_falloff_radius,
            use_obstacles=use_obstacles, obst_density=obst_density, obst_size=obst_size,
            obst_spawn_area=list(obst_spawn_area), use_downwash=use_downwash, use_numba=use_numba,
            quads_mode=quads_mode, room_dims=list(room_dims), use_replay_buffer=False,
            quads_view_mode=['topdown'], quads_render=False, dynamics_params=dynamics_params, raw_control=raw_control,
            raw_control_zero_middle=raw_control_zero_middle, dynamics_randomize_every=dynamics_randomize_every,
            dynamics_change=dynamics_change if dynamics_change is not None else FACTORY_CHANGE,
            dyn_sampler_1=dyn_sampler_1, sense_noise=sense_noise, init_random_state=False)


def _plants_pillars(env, rs):
    """Drones flying into pillars (one already inside a pillar's footprint) and one landing on the floor."""
    obst = np.array(env.obstacles.pos_arr)
    P = []
    for k in range(min(4, len(obst))):
        o = obst[k]
        ang = rs.uniform(-np.pi, np.pi)
        r = 0.3 + 0.046 + 0.01 if k else 0.2
        pos = [o[0] + r * np.cos(ang), o[1] + r * np.sin(ang), rs.uniform(1.0, 3.0)]
        P.append(dict(i=k, pos=pos, vel=[-1.5 * np.cos(ang), -1.5 * np.sin(ang), 0.1], rot=rotz(rs.uniform(-3, 3)),
                      omega=ZERO))
    P.append(dict(i=5, pos=[0.5, -0.5, 0.07], vel=[0.3, 0.2, -2.5], rot=rotz(0.4) @ rotx(0.3), omega=ZERO))
    return P


def _plants_corners(env, rs):
    """Upside down in the air and on the floor, resting on the floor, far (> 4 m) from the goal, against a wall."""
    return [dict(i=0, pos=[1.0, 1.0, 3.0], vel=[0.5, 0.0, 0.0], rot=rotz(0.3) @ rotx(np.pi), omega=ZERO),
            dict(i=1, pos=[-0.5, 0.8, 0.0], vel=ZERO, rot=rotz(1.1), omega=ZERO),
            dict(i=2, pos=[-4.8, -4.8, 0.4], vel=[0.0, 0.0, 0.0], rot=rotz(-2.0), omega=ZERO),
            dict(i=3, pos=[4.9, 4.7, 9.5], vel=[1.0, 0.5, 2.0], rot=rotz(2.5) @ rotx(0.4), omega=ZERO),
            dict(i=4, pos=[2.0, -1.0, 0.06], vel=[0.0, 0.0, -1.0], rot=rotz(0.8) @ rotx(np.pi - 0.2), omega=ZERO),
            dict(i=5, pos=[0.0, 0.0, 2.0], vel=[0.0, 0.0, 2.8], rot=rotx(np.pi / 2), omega=ZERO)]


def _plants_models(env, rs):
    """Drones of different airframes thrown off their hover."""
    return [dict(i=k, pos=[rs.uniform(-3, 3), rs.uniform(-3, 3), rs.uniform(0.5, 4.0)], vel=rs.uniform(-1.5, 1.5, 3),
                 rot=rotz(rs.uniform(-3, 3)) @ rotx(rs.uniform(-0.8, 0.8)), omega=ZERO) for k in range(2)]


CASES = [
    # the controller chasing swapped goals over two episodes (njit path)
    dict(name='swap_goals_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=2.5, quads_mode='swap_goals',
                                      raw_control=False),
         T=510, seed=501, obs_stride=10),
    # c3 on the numpy path: pillars, downwash, floor observation; contact responses and floor contacts
    dict(name='c3_numpy_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=1.0, use_obstacles=True,
                                    use_downwash=True, quads_mode='o_random', obs_repr='xyz_vxyz_R_omega_floor',
                                    rew_coeff=C3_REW, use_numba=False, raw_control=False),
         T=170, seed=502, obs_stride=1, plant=_plants_pillars, plant_at=[5, 120]),
    # RandomQuad + RelativeSampler resampled every episode: a Jinv per drone, rebuilt at every reset
    dict(name='randomquad_5', kw=dict(num_agents=5, neighbor_visible_num=2, ep_time=0.6, quads_mode='static_diff_goal',
                                      dynamics_params='RandomQuad', use_downwash=True,
                                      dyn_sampler_1={'class': 'RelativeSampler', 'noise_ratio': 0.05, 'sampler': 'normal'},
                                      dynamics_randomize_every=1, raw_control=False),
         T=140, seed=503, obs_stride=1, plant=_plants_models, plant_at=[20, 90], construct_seed=778),
    # planted corners: saturated commands, upside-down attitudes, the clamp of the goal distance, floor contacts
    dict(name='corners_6', kw=dict(num_agents=6, neighbor_visible_num=2, ep_time=1.0, quads_mode='static_same_goal',
                                   obs_repr='xyz_vxyz_R_omega_floor', raw_control=False),
         T=120, seed=504, obs_stride=1, plant=_plants_corners, plant_at=[0, 60]),
    # RawControl with actions in [0, 1]: the recorded actions span [-1.3, 1.3], so both clip bounds occur
    dict(name='raw_unit_wall_6', kw=dict(num_agents=6, neighbor_visible_num=2, ep_time=0.6, quads_mode='static_diff_goal',
                                         obs_repr='xyz_vxyz_R_omega_wall', raw_control_zero_middle=False),
         T=130, seed=505, obs_stride=1),
]


def run_case(case):
    """gen_golden.run_reference_case on an env with the case's controller; a case's plants go through its obstacle-plant
    hook."""
    case = dict(case)
    plants = case.pop('plant', None)
    if plants is not None:
        case['plant'] = 'obst'
    saved = rh.make_reference_env, gen_golden._plants_obst
    rh.make_reference_env = make_reference_env
    if plants is not None:
        gen_golden._plants_obst = plants
    try:
        return gen_golden.run_reference_case(case)
    finally:
        rh.make_reference_env, gen_golden._plants_obst = saved


def main(argv=None):
    only = set(sys.argv[1:] if argv is None else argv)
    for case in CASES:
        if only and case['name'] not in only:
            continue
        out = run_case(case)
        path = os.path.join(gen_golden.GOLDEN_DIR, f"control_{case['name']}.npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: T={case['T']} D={out['obs0'].shape[1]} -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == '__main__':
    main()
