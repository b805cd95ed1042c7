"""Shared machinery of the GPU parity tests: drive the CUDA engine and the CPU oracle with identical seeds
(keyed Philox draws), identical actions and identical episode tables, and compare step by step.

The oracle is float64, the kernels float32.  Trajectories are teacher-forced: every `resync` steps (and after
any step whose discrete decisions sat closer to their thresholds than float32 can resolve) the oracle's state is
written into the engine with qs_set_state, so the comparison measures per-step error, not chaotic divergence.

Also the resource usage of the built library's kernels (kernel_resources), which the CPU tests check.
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import quadswarm_oracle as qo
from quad_swarm_rl_b200 import _lib as L
from quad_swarm_rl_b200.engine import QuadSwarmEngine, STATE_F32_FIELDS

MARGIN_EPS = 2e-5        # float32 resolution of positions in a 10 m room (ulp(10) ~ 1e-6) with head-room
NEIGHBOR_GAP_EPS = 3e-5


def make_tables(rs, E, N, M, use_obst, episodes=3, spread=1.5):
    """Random per-env episode tables (goals, spawn points, pillar positions on the 1 m grid)."""
    eps = []
    cells = qo.get_cell_centers(8, 8)
    for _ in range(episodes):
        goals = np.zeros((E, N, 3), np.float32)
        spawn = np.zeros((E, N, 3), np.float32)
        obst = np.zeros((E, max(M, 1), 2), np.float32)
        for e in range(E):
            c = rs.uniform(-2, 2, 3) + np.array([0, 0, 3.0])
            goals[e] = (c + rs.uniform(-spread, spread, (N, 3))).astype(np.float32)
            goals[e, :, 2] = np.maximum(goals[e, :, 2], 0.5)
            if use_obst:
                idx = rs.choice(64, M + N, replace=False)
                obst[e, :M] = cells[idx[:M]]
                spawn[e, :, :2] = cells[idx[M:]]
                spawn[e, :, 2] = rs.uniform(1.0, 3.0, N)
            else:
                spawn[e] = (c + rs.uniform(-0.4, 0.4, (N, 3))).astype(np.float32)
        eps.append(dict(goals=goals, spawn=spawn, obst=obst[:, :M] if use_obst else None))
    return eps


def cfg_to_oracle(kw):
    return qo.EnvConfig(
        num_agents=kw['num_agents'], ep_time=kw.get('ep_time', 15.0), obs_repr=kw.get('obs_repr', 'xyz_vxyz_R_omega'),
        neighbor_visible_num=kw.get('neighbor_visible_num', -1), neighbor_obs_type=kw.get('neighbor_obs_type', 'pos_vel'),
        use_obstacles=kw.get('use_obstacles', False), obst_density=kw.get('obst_density', 0.2),
        obst_size=kw.get('obst_size', 0.6), obst_spawn_area=tuple(kw.get('obst_spawn_area', (8.0, 8.0))),
        use_downwash=kw.get('use_downwash', False), room_dims=tuple(kw.get('room_dims', (10., 10., 10.))),
        sense_noise=kw.get('sense_noise', 'default') is not None)


class Pair:
    """One CUDA engine + E oracle envs on the same seeds and tables."""

    def __init__(self, E, kw, seed=1234, table_seed=5, episodes=3, env_id_offset=0, rew_coeff=None):
        self.E, self.kw = E, dict(kw)
        self.N = kw['num_agents']
        self.engine = QuadSwarmEngine(num_envs=E, seed=seed, env_id_offset=env_id_offset, rew_coeff=rew_coeff, **kw)
        self.ocfg = cfg_to_oracle(kw)
        if rew_coeff:
            self.ocfg.rew_coeff.update(rew_coeff)
        M = self.engine.M
        rs = np.random.RandomState(table_seed)
        self.tables = make_tables(rs, E, self.N, M, kw.get('use_obstacles', False), episodes=episodes)
        self.table_idx = 0
        self.oracles = []
        for e in range(E):
            eps = [dict(goals=t['goals'][e].astype(np.float64), spawn=t['spawn'][e].astype(np.float64),
                        obst_xy=None if t['obst'] is None else t['obst'][e].astype(np.float64)) for t in self.tables]
            src = qo.TableEpisodeSource(eps, approch_goal_metric=0.5)
            self.oracles.append(qo.OracleEnv(self.ocfg, qo.PhiloxRng(seed), src, env_id=env_id_offset + e))
        self._push_table(0)

    def _push_table(self, k):
        t = self.tables[min(k, len(self.tables) - 1)]
        self.engine.set_next_episode(t['goals'], t['spawn'], t['obst'])

    def reset(self):
        obs_o = np.stack([o.reset() for o in self.oracles])
        obs_d = self.engine.reset().cpu().numpy().astype(np.float64)
        self.table_idx = 1
        self._push_table(1)           # the NEXT auto-reset consumes table 1
        return obs_d, obs_o

    def step(self, actions):
        """actions float32 [E,N,4]"""
        a_dev = torch.as_tensor(actions, device=self.engine.device).contiguous()
        obs, rew, done = self.engine.step(a_dev, with_terms=True)
        out_d = dict(obs=obs.cpu().numpy().astype(np.float64), rewards=rew.cpu().numpy().astype(np.float64),
                     dones=done.cpu().numpy().astype(bool), terms=self.engine.rew_terms.cpu().numpy().astype(np.float64))
        res = [o.step(actions[e].astype(np.float64)) for e, o in enumerate(self.oracles)]
        out_o = dict(obs=np.stack([r[0] for r in res]), rewards=np.array([[float(x) for x in r[1]] for r in res]),
                     dones=np.array([r[2] for r in res], dtype=bool), infos=[r[3] for r in res])
        if out_o['dones'].any():
            self.table_idx += 1
            self._push_table(self.table_idx)
        return out_d, out_o

    # ---- teacher forcing: oracle state -> device
    def oracle_state(self):
        E, N = self.E, self.N
        af = np.zeros((E, N, L.QS_STATE_F32), np.float32)
        au = np.zeros((E, N, L.QS_STATE_U32), np.int64)
        ei = np.zeros((E, L.QS_STATE_ENV_I32), np.int32)
        M = self.engine.M
        ob = np.zeros((E, max(M, 1), 2), np.float32)
        F = STATE_F32_FIELDS
        for e, o in enumerate(self.oracles):
            for i, d in enumerate(o.drones):
                row = af[e, i]
                row[F['pos'][0]:F['pos'][1]] = d.pos
                row[F['vel'][0]:F['vel'][1]] = d.vel
                row[F['rot'][0]:F['rot'][1]] = d.rot.reshape(-1)
                row[F['omega'][0]:F['omega'][1]] = d.omega
                row[F['thrust_rot_damp'][0]:F['thrust_rot_damp'][1]] = d.thrust_rot_damp
                row[F['thrust_cmds_damp'][0]:F['thrust_cmds_damp'][1]] = d.thrust_cmds_damp
                row[F['ou'][0]:F['ou'][1]] = d.ou
                row[F['goal'][0]:F['goal'][1]] = d.goal
                hist = [x / o.P.dt for x in o.distance_to_goal[i]]
                ring = (hist[::-1] + [0.0] * 4)[:4]
                row[F['dist_ring'][0]:F['dist_ring'][1]] = ring
                L_ = o.ep_len + 1
                sums = []
                for w in (100, 300, 500):
                    w = min(w, L_)
                    sums.append(sum(h for t, h in enumerate(hist, start=1) if t > L_ - w))
                row[F['dist_sums'][0]:F['dist_sums'][1]] = sums
                row[F['stale_vel'][0]:F['stale_vel'][1]] = o.vel[i]
                fl = 0
                fl |= L.FLAG_ON_FLOOR if d.on_floor else 0
                fl |= L.FLAG_CRASHED_FLOOR if d.crashed_floor else 0
                fl |= L.FLAG_CRASHED_WALL if d.crashed_wall else 0
                fl |= L.FLAG_CRASHED_CEILING if d.crashed_ceiling else 0
                fl |= L.FLAG_PREV_WALL if i in list(o.prev_crashed_walls) else 0
                fl |= L.FLAG_PREV_CEILING if i in list(o.prev_crashed_ceiling) else 0
                fl |= L.FLAG_PREV_ROOM if i in list(o.prev_crashed_room) else 0
                fl |= L.FLAG_PREV_OBST if i in list(o.prev_obst_quad_collisions) else 0
                fl |= L.FLAG_NO_COL_AGENT if o.agent_col_agent[i] else 0
                fl |= L.FLAG_NO_COL_OBST if o.agent_col_obst[i] else 0
                fl |= L.FLAG_REACHED_GOAL if o.reached_goal[i] else 0
                prev = 0
                for (a, b) in o.prev_drone_collisions:
                    if a == i:
                        prev |= 1 << b
                    if b == i:
                        prev |= 1 << a
                au[e, i, 0] = fl
                au[e, i, 1] = prev
            svd = int(round(o.drones[0].since_last_svd / o.P.dt))
            ei[e, :4] = [o.tick, o.step_count, svd, 0]
            ei[e, 4 + L.QS_NUM_ENV_STATS + 16] = o.epi              # episode number (keys the episode-generation draws)
            ei[e, 4:4 + 11] = [o.collisions_per_episode, o.collisions_after_settle, o.collisions_final_5s,
                               o.collisions_room_per_episode, o.collisions_floor_per_episode,
                               o.collisions_wall_per_episode, o.collisions_ceiling_per_episode,
                               o.obst_quad_collisions_per_episode, o.obst_quad_collisions_after_settle,
                               o.distance_to_goal_3_5, o.distance_to_goal_5]
            if M > 0 and o.obst_xy is not None:
                ob[e, :] = 1.0e4                                    # unused table slots stand far outside the room
                ob[e, :len(o.obst_xy)] = o.obst_xy
                base = 4 + L.QS_NUM_ENV_STATS
                if getattr(o.source, 'densities', None) is not None:      # per-episode pillar radius / count (scn_f[0].xy)
                    ei[e, base + 4:base + 6] = np.array([o.obst_size / 2.0, float(len(o.obst_xy))], np.float32).view(np.int32)
            sc = getattr(o.source, 's', None)                 # twin of the device-side scenario state (scenario_gen.py)
            if sc is not None:
                base = 4 + L.QS_NUM_ENV_STATS
                ei[e, base:base + 4] = [sc['mode'], sc['period'], sc['next'], sc['f'] | (sc['growing'] << 8)]
                fl32 = np.array([sc['size'], sc['layer'], sc['hi'], sc['speed'], *sc['c1'], 0.0, *sc['c2'], 0.0], np.float32)
                ei[e, base + 4:base + 16] = fl32.view(np.int32)
        au32 = au.astype(np.uint32).view(np.int32)
        return dict(agent_f32=torch.from_numpy(af), agent_u32=torch.from_numpy(au32.copy()), env_i32=torch.from_numpy(ei),
                    obst_xy=torch.from_numpy(ob[:, :M].copy()) if M > 0 else None)

    def sync_device_from_oracle(self):
        st = self.oracle_state()
        cur = self.engine.get_state()
        st['env_i32'][:, 3] = cur['env_i32'][:, 3].cpu()          # episode_idx is engine-private
        if getattr(self.oracles[0].source, 's', None) is None:    # no twin of the scenario state: keep the device's
            base = 4 + L.QS_NUM_ENV_STATS
            st['env_i32'][:, base:] = cur['env_i32'][:, base:].cpu()
        self.engine.set_state(st)

    def device_fields(self):
        st = self.engine.get_state()
        af = st['agent_f32'].cpu().numpy().astype(np.float64)
        au = st['agent_u32'].cpu().numpy().view(np.uint32)
        out = {k: af[..., a:b] for k, (a, b) in STATE_F32_FIELDS.items()}
        out['flags'] = au[..., 0]
        out['prev_col'] = au[..., 1]
        out['env_i32'] = st['env_i32'].cpu().numpy()
        return out

    def oracle_fields(self):
        o = self.oracles
        f = lambda name: np.array([[getattr(d, name) for d in e.drones] for e in o], dtype=np.float64)
        return dict(pos=f('pos'), vel=f('vel'), rot=f('rot').reshape(self.E, self.N, 9), omega=f('omega'),
                    thrust_rot_damp=f('thrust_rot_damp'), thrust_cmds_damp=f('thrust_cmds_damp'), ou=f('ou'),
                    goal=f('goal'),
                    on_floor=np.array([[d.on_floor for d in e.drones] for e in o], dtype=bool))


class DevicePair(Pair):
    """Engine with a device-side episode generator + oracle envs fed by its CPU twin (oracle/scenario_gen.py): no host
    tables on either side."""

    def __init__(self, E, kw, seed, device_scenario, source_factory, env_id_offset=0):
        self.E, self.kw, self.N = E, dict(kw), kw['num_agents']
        self.engine = QuadSwarmEngine(num_envs=E, seed=seed, device_scenario=device_scenario,
                                      env_id_offset=env_id_offset, **kw)
        self.ocfg = cfg_to_oracle(kw)
        self.oracles = [qo.OracleEnv(self.ocfg, qo.PhiloxRng(seed), source_factory(), env_id=env_id_offset + e)
                        for e in range(E)]
        self.table_idx = 0

    def _push_table(self, k):
        pass


class SampledPair(Pair):
    """Full-size engine (E_total envs, the BASELINE shapes) checked against the oracle on a SAMPLE of its envs: the keyed
    random draws make env e's trajectory a function of (seed, global env id, actions) only, so `OracleEnv(env_id=e)`
    reproduces exactly what the engine's env e must do while all the other envs run beside it.  The engine therefore runs
    the kernel instantiation, grid shape and launch chaining of the benchmark; run_parity() sees only the sampled rows.
    `device_scenario` / `source_factory` as in DevicePair (no host tables), or host tables when both are None."""

    def __init__(self, E_total, sample, kw, seed, device_scenario=None, source_factory=None, chained=False, table_seed=5,
                 rew_coeff=None):
        self.E_total = E_total
        self.sample = list(sample)
        self.E, self.kw, self.N = len(self.sample), dict(kw), kw['num_agents']
        self.engine = QuadSwarmEngine(num_envs=E_total, seed=seed, device_scenario=device_scenario, rew_coeff=rew_coeff, **kw)
        self.engine.set_chained(chained)
        self.ocfg = cfg_to_oracle(kw)
        if rew_coeff:
            self.ocfg.rew_coeff.update(rew_coeff)
        self.table_idx = 0
        self.tables = None
        if device_scenario is None:
            rs = np.random.RandomState(table_seed)
            self.tables = make_tables(rs, E_total, self.N, self.engine.M, kw.get('use_obstacles', False), episodes=3)
        self.oracles = []
        for e in self.sample:
            if device_scenario is None:
                eps = [dict(goals=t['goals'][e].astype(np.float64), spawn=t['spawn'][e].astype(np.float64),
                            obst_xy=None if t['obst'] is None else t['obst'][e].astype(np.float64)) for t in self.tables]
                src = qo.TableEpisodeSource(eps, approch_goal_metric=0.5)
            else:
                src = source_factory()
            self.oracles.append(qo.OracleEnv(self.ocfg, qo.PhiloxRng(seed), src, env_id=e))
        self._gen = torch.Generator(device=self.engine.device)
        self._gen.manual_seed(seed + 77)
        self._idx = torch.as_tensor(self.sample, device=self.engine.device, dtype=torch.long)
        self._mask = torch.zeros(E_total, dtype=torch.uint8, device=self.engine.device)
        self._mask[self._idx] = 1
        if self.tables is not None:
            self._push_table(0)

    def _push_table(self, k):
        if self.tables is not None:
            t = self.tables[min(k, len(self.tables) - 1)]
            self.engine.set_next_episode(t['goals'], t['spawn'], t['obst'])

    def reset(self):
        obs_o = np.stack([o.reset() for o in self.oracles])
        obs_d = self.engine.reset()[self._idx].cpu().numpy().astype(np.float64)
        self.table_idx = 1
        self._push_table(1)
        return obs_d, obs_o

    def step(self, actions):
        """actions float32 [len(sample),N,4]; every other env gets its own random actions"""
        dev = self.engine.device
        a_all = torch.rand((self.E_total, self.N, 4), device=dev, generator=self._gen) * 2 - 1
        a_all[self._idx] = torch.as_tensor(actions, device=dev)
        obs, rew, done = self.engine.step(a_all.contiguous(), with_terms=True)
        ix = self._idx
        out_d = dict(obs=obs[ix].cpu().numpy().astype(np.float64), rewards=rew[ix].cpu().numpy().astype(np.float64),
                     dones=done[ix].cpu().numpy().astype(bool), terms=self.engine.rew_terms[ix].cpu().numpy().astype(np.float64))
        res = [o.step(actions[e].astype(np.float64)) for e, o in enumerate(self.oracles)]
        out_o = dict(obs=np.stack([r[0] for r in res]), rewards=np.array([[float(x) for x in r[1]] for r in res]),
                     dones=np.array([r[2] for r in res], dtype=bool), infos=[r[3] for r in res])
        if out_o['dones'].any():
            self.table_idx += 1
            self._push_table(self.table_idx)
        return out_d, out_o

    def sync_device_from_oracle(self):
        st = self.oracle_state()                       # rows of the sampled envs
        cur = self.engine.get_state()
        ix = self._idx.cpu()
        st['env_i32'][:, 3] = cur['env_i32'][ix.to(cur['env_i32'].device), 3].cpu()
        if getattr(self.oracles[0].source, 's', None) is None:
            base = 4 + L.QS_NUM_ENV_STATS
            st['env_i32'][:, base:] = cur['env_i32'][ix.to(cur['env_i32'].device), base:].cpu()
        dev = self.engine.device
        for k in ('agent_f32', 'agent_u32', 'env_i32'):
            cur[k][self._idx] = st[k].to(dev)
        if st.get('obst_xy') is not None and self.engine.M > 0:
            ob = cur['obst_xy'].clone()
            ob[self._idx] = st['obst_xy'].to(dev)
            cur['obst_xy'] = ob
        self.engine.set_state(cur, env_mask=self._mask)

    def device_fields(self):
        st = self.engine.get_state()
        ix = self._idx
        af = st['agent_f32'][ix].cpu().numpy().astype(np.float64)
        au = st['agent_u32'][ix].cpu().numpy().view(np.uint32)
        out = {k: af[..., a:b] for k, (a, b) in STATE_F32_FIELDS.items()}
        out['flags'] = au[..., 0]
        out['prev_col'] = au[..., 1]
        out['env_i32'] = st['env_i32'][ix].cpu().numpy()
        return out


def run_parity(pair, T, rs, resync=20, rtol=1e-4, atol=1e-4, action_scale=1.0, check_state=True, hook=None,
               margin_eps=MARGIN_EPS, gap_eps=NEIGHBOR_GAP_EPS):
    """Step both sides T times; returns a report dict.  Raises AssertionError on a real mismatch.
    resync = 1 with margin_eps ~ 3e-6 is the TIGHT mode: the device is teacher-forced from the oracle after every step, so
    the two sides differ by one step of fp32 arithmetic only (positions: ulp(5 m) = 4.8e-7) and the discrete masks are
    compared on every env-step whose decisions sit further than that from their thresholds."""
    E, N = pair.E, pair.N
    obs_d, obs_o = pair.reset()
    np.testing.assert_allclose(obs_d, obs_o, rtol=rtol, atol=atol, err_msg='reset obs')
    rep = dict(steps=0, skipped_env_steps=0, max_obs_err=0.0, max_rew_err=0.0, max_state_err=0.0, dones=0,
               quadcol=0, obstcol=0, kicked=0, floor=0, compared_env_steps=0)
    for t in range(T):
        if hook:
            hook(pair, t)
        a = (action_scale * rs.uniform(-1, 1, size=(E, N, 4))).astype(np.float32)
        d, o = pair.step(a)
        assert np.array_equal(d['dones'], o['dones']), f'dones differ at step {t}'
        rep['dones'] += int(o['dones'][:, 0].sum())
        dev = pair.device_fields() if check_state else None
        orc = pair.oracle_fields() if check_state else None
        need_sync = (t + 1) % resync == 0
        for e, oe in enumerate(pair.oracles):
            ok = oe.step_margin > margin_eps and (pair.engine.K in (0, N - 1) or oe.step_neighbor_gap > gap_eps)
            if not ok:
                rep['skipped_env_steps'] += 1
                need_sync = True
                continue
            rep['compared_env_steps'] += 1
            err = np.abs(d['obs'][e] - o['obs'][e])
            tol = atol + rtol * np.abs(o['obs'][e])
            assert (err <= tol).all(), (f'obs mismatch step {t} env {e}: max err {err.max():.3e} at '
                                        f'{np.unravel_index(err.argmax(), err.shape)}; margin {oe.step_margin:.2e}')
            rep['max_obs_err'] = max(rep['max_obs_err'], float(err.max()))
            rerr = np.abs(d['rewards'][e] - o['rewards'][e])
            assert (rerr <= atol + rtol * np.abs(o['rewards'][e])).all(), f'reward mismatch step {t} env {e}: {rerr.max():.3e}'
            rep['max_rew_err'] = max(rep['max_rew_err'], float(rerr.max()))
            # bit-exact masks
            raw_q = np.array([o['infos'][e][i]['rewards']['rewraw_quadcol'] for i in range(N)])
            assert np.array_equal(d['terms'][e][:, 5], raw_q), f'quadcol mask differs step {t} env {e}'
            rep['quadcol'] += int((raw_q < 0).sum())
            if pair.engine.M > 0:
                raw_ob = np.array([o['infos'][e][i]['rewards']['rewraw_quadcol_obstacle'] for i in range(N)])
                assert np.array_equal(d['terms'][e][:, 7], raw_ob), f'obstacle mask differs step {t} env {e}'
                rep['obstcol'] += int((raw_ob < 0).sum())
            if check_state and not o['dones'][e, 0]:
                fl = dev['flags'][e]
                assert np.array_equal((fl & L.FLAG_ON_FLOOR) != 0, orc['on_floor'][e]), f'on_floor differs step {t} env {e}'
                assert bool(fl[0] & L.FLAG_KICKED) == bool(oe.kicked), f'kicked flag differs step {t} env {e}'
                rep['kicked'] += int(bool(oe.kicked))
                rep['floor'] += int(orc['on_floor'][e].sum())
                for k in ('pos', 'vel', 'rot', 'omega', 'thrust_rot_damp', 'thrust_cmds_damp', 'ou', 'goal'):
                    serr = np.abs(dev[k][e] - orc[k][e])
                    assert (serr <= atol + rtol * np.abs(orc[k][e])).all(), \
                        f'state {k} mismatch step {t} env {e}: {serr.max():.3e}'
                    rep['max_state_err'] = max(rep['max_state_err'], float(serr.max()))
                assert dev['env_i32'][e, 0] == oe.tick
        rep['steps'] += 1
        if need_sync:
            pair.sync_device_from_oracle()
    return rep


def kernel_resources(pattern):
    """Registers, stack frame and local memory of the built library's kernels (`cuobjdump --dump-resource-usage`):
    {key: {'REG': n, 'STACK': n, 'LOCAL': n}} for every function whose mangled name matches the regex `pattern`, keyed by
    the match's groups, digit groups as ints.  Skips the test when cuobjdump or the library is not there."""
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not (os.path.exists(tool) and os.path.exists(L.LIB_PATH)):
        pytest.skip('cuobjdump or the library not available')
    out = subprocess.run([tool, '--dump-resource-usage', L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    usage, key = {}, None
    for line in out.splitlines():
        if 'Function' in line:
            m = re.search(pattern, line)
            key = tuple(int(g) if g and g.isdigit() else g for g in m.groups()) if m else None
        elif key is not None and 'REG:' in line:
            usage[key] = {k: int(v) for k, v in re.findall(r'(REG|STACK|LOCAL):(\d+)', line)}
            key = None
    return usage
