"""Per-episode pillar size on host tables (QuadrotorEnvMulti.reset(obst_density, obst_size), quadrotor_multi.py:339-351) in
the CPU oracle — TEST INFRASTRUCTURE ONLY.

* SizedTableEpisodeSource: the table source of the GPU parity tests with an optional `obst_size` per episode, the twin of
  qs_set_next_obstacle_radius.  The device keeps the radius size / 2 in float32, so the oracle's size is twice that float.
  An episode without the key keeps the size of the one before, as an env the calls never mask keeps its radius.
* replay_obst_size_golden: replays tests/golden/obst_size_*.npz (oracle/gen_golden_obst_size.py), where the unmodified
  reference was driven through a sequence of explicit reset(obst_density, obst_size) calls, with the reference's own random
  streams (ReplayRng) like oracle/replay.py.
"""
import json

import numpy as np

from .gen_golden import INFO_KEYS
from .quadswarm_oracle import OracleEnv, ReferenceEpisodeSource, ReplayRng, TableEpisodeSource
from .replay import config_from_case

STATE_KEYS = ('pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou', 'on_floor')


def device_size(size):
    """The pillar size the device flies for `size`: twice its float32 radius."""
    return 2.0 * float(np.float32(size / 2.0))


class SizedTableEpisodeSource(TableEpisodeSource):
    def reset(self, env):
        out = super().reset(env)
        if self.cur.get('obst_size') is not None:
            env.obst_size = device_size(self.cur['obst_size'])
        return out


def replay_obst_size_golden(g, make_scenario):
    """g: the loaded golden npz; make_scenario(mode, cfg, rng) -> the host scenario object under test.  Returns the oracle's
    obs0 of every explicit reset, and its per-step rewards / dones / infos / goals / obs / states / episode statistics in
    the fixture's layout, plus the pillar size in force at every step."""
    case = json.loads(str(g['case_json']))
    kw, seed = case['kw'], case['seed']
    cfg = config_from_case(kw)
    n = cfg.num_agents
    rng = ReplayRng(seed, seed + 1, [seed + 100 + i for i in range(n)])
    scenario = make_scenario(kw['quads_mode'], cfg, rng.py)
    env = OracleEnv(cfg, rng, ReferenceEpisodeSource(scenario))
    T = int(g['actions'].shape[0])
    out = dict(obs0=[], rewards=np.zeros((T, n)), dones=np.zeros((T, n), dtype=bool),
               infos=np.full((T, n, len(INFO_KEYS)), np.nan), goals=np.zeros((T, n, 3)), sizes=np.zeros(T), ep_stats=[])
    obs, states = {}, {k: {} for k in STATE_KEYS}
    resets = {int(t): (float(d), float(s)) for t, d, s in zip(g['reset_t'], g['reset_density'], g['reset_size'])}
    want_obs, want_state = set(int(t) for t in g['obs_t']), set(int(t) for t in g['state_t'])
    for t in range(T):
        if t in resets:                        # reset(obst_density, obst_size): both kept for the later episodes
            cfg.obst_density, env.obst_size = resets[t]
            out['obs0'].append(env.reset())
        for k in np.where(g['plant_t'] == t)[0]:
            d = env.drones[int(g['plant_i'][k])]
            d.pos, d.vel = g['plant_pos'][k].copy(), g['plant_vel'][k].copy()
            d.rot, d.omega = g['plant_rot'][k].copy(), g['plant_omega'][k].astype(np.float32).astype(np.float64)
            d.acc = np.zeros(3)
            d.accelerometer = np.array([0., 0., 9.81])
        out['sizes'][t] = env.obst_size
        o, r, dn, inf = env.step(g['actions'][t])
        if t in want_obs:
            obs[t] = o
        out['rewards'][t] = r
        out['dones'][t] = dn
        for i in range(n):
            for k, key in enumerate(INFO_KEYS):
                if key in inf[i]['rewards']:
                    out['infos'][t, i, k] = inf[i]['rewards'][key]
        out['goals'][t] = np.array([d.goal for d in env.drones])
        if t in want_state:
            for k in states:
                states[k][t] = np.array([getattr(d, k) for d in env.drones])
        if dn[0]:
            out['ep_stats'].append((t, {k: float(v) for k, v in inf[0]['episode_extra_stats'].items()}))
    out['obs0'] = np.array(out['obs0'])
    out['obs'] = np.array([obs[int(t)] for t in g['obs_t']])
    out.update({'state_' + k: np.array([states[k][int(t)] for t in g['state_t']]) for k in states})
    return out, env
