"""Generate tests/golden/obst_size_*.npz by driving the UNMODIFIED reference through a fixed sequence of
reset(obst_density, obst_size) calls — TEST INFRASTRUCTURE ONLY.

Run in a container where /root/reference is mounted:  python -m oracle.gen_golden_obst_size
What ExperienceReplayWrapper.new_episode does with --quads_domain_random (quad_experience_replay.py:195-206): every
explicit reset draws a pillar density and size, and the env keeps both for its auto-resets (quadrotor_multi.py:339-351).
Each segment starts with such a reset, runs past one auto-reset, and plants drones flying into pillars shortly after the
reset, so that drones hit pillars of every size.  The recording is that of oracle/gen_golden.py (seeds, actions, planted
states, the reference's observations / rewards / dones / reward terms / states / episode statistics) plus the reset
sequence and the pillar positions and size of every episode.  To keep the file small, the states are stored after every
STRIDE-th step and before every step in which a drone hits a pillar, and the observations, reward terms and positions after
the step that follows each of them: pairs that let a test start a step from the reference's state and compare what it
produces.  Rewards,
dones, goals, sizes and the obstacle-collision term are stored for every step.
"""
import json
import os
import sys

import numpy as np

from . import ref_harness as rh
from .gen_golden import GOLDEN_DIR, INFO_KEYS, _plants_obst

C3_REW = dict(pos=1.0, effort=0.05, spin=0.1, vel=0.0, crash=1.0, orient=1.0, yaw=0.0, quadcol_bin=5.0,
              quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
CASES = [
    # (density, size, steps) per explicit reset; the table of the construction density (0.2: 12 pillars) holds them all
    dict(name='o_random_8', kw=dict(num_agents=8, neighbor_visible_num=2, ep_time=0.6, use_obstacles=True, obst_density=0.2,
                                    obst_size=0.6, use_downwash=True, quads_mode='o_random', obs_repr='xyz_vxyz_R_omega_floor',
                                    rew_coeff=C3_REW),
         segments=[(0.2, 0.3, 70), (0.05, 0.6, 70), (0.1, 0.4, 70), (0.15, 0.5, 70)], plant_after=3,
         seed=501),
]
STRIDE = 3
STATE_KEYS = ['pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou', 'on_floor']


def run_case(case):
    kw = dict(case['kw'])
    env = rh.make_reference_env(**kw)
    n, seed = kw['num_agents'], case['seed']
    rh.seed_reference(env, seed, seed + 1, [seed + 100 + i for i in range(n)])
    act_rs, plant_rs = np.random.RandomState(seed + 7), np.random.RandomState(seed + 9)
    T = sum(s for _, _, s in case['segments'])
    actions, rewards = np.zeros((T, n, 4)), np.zeros((T, n))
    dones = np.zeros((T, n), dtype=bool)
    infos = np.full((T, n, len(INFO_KEYS)), np.nan)
    goals, sizes = np.zeros((T, n, 3)), np.zeros(T)
    obs0, obs, plants, ep_stats, obst_log = [], [], [], [], []
    states = {k: [] for k in STATE_KEYS}
    reset_t, t = [], 0
    for density, size, steps in case['segments']:
        reset_t.append(t)
        obs0.append(np.array(env.reset(obst_density=density, obst_size=size), dtype=np.float64))
        obst_log.append((t, np.array(env.obstacles.pos_arr)[:, :2].copy(), float(env.obst_size)))
        for k in range(steps):
            if k == case['plant_after']:
                for p in _plants_obst(env, plant_rs):
                    rh.plant_state(env, p['i'], p['pos'], p['vel'], p['rot'], p['omega'])
                    plants.append((t, p['i'], np.array(p['pos'], float), np.array(p['vel'], float),
                                   np.array(p['rot'], float), np.array(p['omega'], float)))
            a = ((1.3 if t % 7 == 3 else 1.0) * act_rs.uniform(-1, 1, size=(n, 4))).astype(np.float32).astype(np.float64)
            actions[t] = a
            sizes[t] = float(env.obst_size)
            o, r, d, inf = env.step([a[i] for i in range(n)])
            obs.append(np.array(o, dtype=np.float64))
            rewards[t], dones[t] = np.array(r, dtype=np.float64), d
            for i in range(n):
                for j, key in enumerate(INFO_KEYS):
                    if key in inf[i]['rewards']:
                        infos[t, i, j] = float(inf[i]['rewards'][key])
            goals[t] = np.array([e.goal for e in env.envs])
            snap = rh.snapshot(env)
            for key in STATE_KEYS:
                states[key].append(snap[key])
            if d[0]:
                ep_stats.append((t, {key: float(v) for key, v in inf[0]['episode_extra_stats'].items()}))
                obst_log.append((t + 1, np.array(env.obstacles.pos_arr)[:, :2].copy(), float(env.obst_size)))
            t += 1
    M = int(kw['obst_density'] * 64)
    obst_xy = np.full((len(obst_log), M, 2), 1e6)              # fewer pillars than the table: the rest far outside the room
    for k, (_, xy, _) in enumerate(obst_log):
        obst_xy[k, :len(xy)] = xy
    term = infos[..., INFO_KEYS.index('rewraw_quadcol_obstacle')]
    hit_t = np.where((term < 0).any(axis=1))[0]
    state_t = np.union1d(np.arange(0, T - 1, STRIDE), hit_t[hit_t > 0] - 1)
    obs_t = state_t + 1
    out = dict(obs0=np.array(obs0), actions=actions.astype(np.float32), rewards=rewards, dones=dones, goals=goals,
               sizes=sizes, obst_term=term,
               obs_t=obs_t, obs=np.array(obs)[obs_t], infos=infos[obs_t], obs_pos=np.array(states['pos'])[obs_t],
               state_t=state_t,
               reset_t=np.array(reset_t, dtype=int), reset_density=np.array([d for d, _, _ in case['segments']]),
               reset_size=np.array([s for _, s, _ in case['segments']]),
               plant_t=np.array([p[0] for p in plants], dtype=int), plant_i=np.array([p[1] for p in plants], dtype=int),
               plant_pos=np.array([p[2] for p in plants]).reshape(-1, 3),
               plant_vel=np.array([p[3] for p in plants]).reshape(-1, 3),
               plant_rot=np.array([p[4] for p in plants]).reshape(-1, 3, 3),
               plant_omega=np.array([p[5] for p in plants]).reshape(-1, 3),
               ep_stats_json=np.array(json.dumps(ep_stats)),
               obst_t=np.array([o[0] for o in obst_log], dtype=int), obst_xy=obst_xy,
               obst_n=np.array([len(o[1]) for o in obst_log], dtype=int), obst_size=np.array([o[2] for o in obst_log]),
               case_json=np.array(json.dumps(dict(name=case['name'], kw=kw, T=T, seed=seed, D=int(obs0[0].shape[1])))))
    out.update({'state_' + k: np.array(v)[state_t] for k, v in states.items()})
    return out


def main(argv=None):
    only = set(sys.argv[1:] if argv is None else argv)
    for case in CASES:
        if only and case['name'] not in only:
            continue
        out = run_case(case)
        path = os.path.join(GOLDEN_DIR, f"obst_size_{case['name']}.npz")
        np.savez_compressed(path, **out)
        print(f"{case['name']}: T={out['actions'].shape[0]} D={out['obs0'].shape[2]} -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == '__main__':
    main()
