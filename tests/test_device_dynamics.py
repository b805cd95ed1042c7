"""Dynamics randomisation on the device (qs_set_dynamics_sampler, csrc/qs_dyn_sampler.cuh; QuadrotorEnvMultiBatched(
device_dynamics=True)).

CPU: the RandomState stand-in of the twin (oracle/dyn_sampler_oracle.py) consumes draws in the host pipeline's order for
every supported combination; the flat spec round-trips and rejects what the device cannot run; the twin's rows have the
distribution of the host pipeline's.  GPU: the device rows equal the twin's after construction and after every reset, change
exactly at the resets the cadence names, do not depend on how the steps are launched, and fly like rows uploaded with
qs_set_dynamics(at_next_reset)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.dyn_sampler_oracle import ForwardingDraws, twin_row, twin_source          # noqa: E402
from quad_swarm_rl_b200 import _lib as L                                               # noqa: E402
from quad_swarm_rl_b200 import quad_models as Q                                       # noqa: E402


def _custom_dict():
    """A user's parameter dict: another key order, densities instead of masses, no arms.l."""
    p = Q.defaultquad_params()
    g = p['geom']
    g['body'] = {'w': 0.1, 'h': 0.08, 'l': 0.12, 'm': 0.45}
    g['payload'] = {'density': 900.0, 'l': 0.1, 'w': 0.1, 'h': 0.03}
    g['arms'] = {'w': 0.015, 'h': 0.015, 'density': 1200.0}
    p['motor'] = dict(reversed(list(p['motor'].items())))
    return {'motor': p['motor'], 'geom': g, 'noise': p['noise'], 'damp': p['damp']}


BASES = {'Crazyflie': 'Crazyflie', 'DefaultQuad': 'DefaultQuad', 'MediumQuad': 'MediumQuad', 'dict': _custom_dict(),
         'RandomQuad': 'RandomQuad'}
CHANGE = {'motor': {'thrust_to_weight': 2.2}, 'damp': {'vel': 0.0}}
SAMPLERS = {
    'none': None,
    'rel_normal': {'class': 'RelativeSampler', 'noise_ratio': 0.1, 'sampler': 'normal'},
    'rel_uniform_custom': {'class': 'RelativeSampler', 'noise_ratio': 0.05, 'sampler': 'uniform',
                           'noise_ratio_custom': {'motor': {'thrust_to_weight': 0.2, 'assymetry': 0.02}, 'geom': {'body': {'w': 0.3}}}},
    'const': {'class': 'ConstValueSampler', 'params_change': {'motor': {'torque_to_thrust': 0.01}, 'noise': {'thrust_noise_ratio': 0.03}}},
}
COMBOS = [(b, c, s1, s2) for b in BASES for c in (False, True) for s1 in SAMPLERS for s2 in SAMPLERS]


def _args(base, change, s1, s2):
    return BASES[base], (CHANGE if change else None), SAMPLERS[s1], SAMPLERS[s2]


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('base,change,s1,s2', COMBOS)
def test_standin_draws_in_pipeline_order(base, change, s1, s2):
    """A stand-in that splits every call into scalar draws of a real RandomState gives DynamicsSource's own rows."""
    args = _args(base, change, s1, s2)
    ref = Q.DynamicsSource(*args, rs=np.random.RandomState(11))
    alt = Q.DynamicsSource(*args, rs=ForwardingDraws(np.random.RandomState(11)))
    for _ in range(3):
        np.testing.assert_array_equal(alt.sample_row(), ref.sample_row())


@pytest.mark.parametrize('base,change,s1,s2', COMBOS)
def test_flat_spec_round_trips(base, change, s1, s2):
    spec = Q.dynamics_sampler_spec(*_args(base, change, s1, s2))
    back = L.dyn_sampler_spec_of(L.dyn_sampler_struct(spec))
    assert back['base'] == spec['base'] and list(back['sampler']) == list(spec['sampler'])
    np.testing.assert_array_equal(back['order'], spec['order'])
    for a, b in [(back['params'], spec['params']), (back['change'], spec['change'])] + list(zip(back['samp'], spec['samp'])):
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[1], b[1])
    if spec['base'] == Q.DYN_BASE_FIXED:           # the leaves rebuild the base tree, key order included
        tree = Q.unflatten_tree(*spec['params'], spec['order'])
        base_tree = twin_source(*_args(base, False, 'none', 'none'))._base()
        assert Q.flatten_tree(tree)[2] == Q.flatten_tree(base_tree)[2]
        assert Q.constants_row(tree).tobytes() == Q.constants_row(base_tree).tobytes()
    assert len(spec['order']) == int(spec['params'][0].sum())


@pytest.mark.parametrize('kw,match', [
    (dict(dynamics_params='SmallQuad'), 'unknown dynamics_params'),
    (dict(dyn_sampler_1={'class': 'AbsoluteSampler'}), 'RelativeSampler and ConstValueSampler'),
    (dict(dyn_sampler_2={'class': 'RandomQuad'}), 'RelativeSampler and ConstValueSampler'),
    (dict(dyn_sampler_1={'class': 'RelativeSampler', 'noise_ratio': 0.1, 'sampler': 'lognormal'}), 'normal'),
    (dict(dynamics_params={**Q.crazyflie_params(), 'extra': {'x': 1.0}}), 'no leaf extra.x'),
    (dict(dynamics_change={'motor': {'thrust_to_weight': float('nan')}}), 'finite'),
    (dict(dynamics_change={'motor': {'not_a_leaf': 1.0}}), 'cannot build'),
    (dict(dynamics_change={'geom': {'motor_pos': {'xyz': [0.1, 0.1]}}}), '3 numbers'),
    (dict(dyn_sampler_1={'class': 'ConstValueSampler', 'params_change': {'motor': {'linearity': 'full'}}}), 'finite number'),
])
def test_unsupported_specs_raise(kw, match):
    with pytest.raises(ValueError, match=match):
        Q.dynamics_sampler_spec(**kw)


def test_ctypes_layout_matches_c(tmp_path):
    src = tmp_path / 'sz.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "quadswarm.h"\nint main(){printf("%zu %zu %zu %zu %zu %d\\n", '
                   'sizeof(QsDynSampler), offsetof(QsDynSampler, params), offsetof(QsDynSampler, change), '
                   'offsetof(QsDynSampler, samp), sizeof(QsDynLeaves), QS_DYN_LEAVES);return 0;}\n')
    exe = tmp_path / 'sz'
    subprocess.run(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)], check=True)
    out = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = L.QsDynSampler
    assert out == [ctypes.sizeof(S), S.params.offset, S.change.offset, S.samp.offset, ctypes.sizeof(L.QsDynLeaves),
                   Q.DYN_NUM_LEAVES]


@pytest.mark.parametrize('base,s1', [('RandomQuad', 'none'), ('Crazyflie', 'rel_normal')])
def test_twin_has_the_pipeline_distribution(base, s1):
    """Two-sample KS test per row field: the twin's keyed draws (envs 0..n-1, episode 1) against the host pipeline's
    RandomState rows."""
    from scipy.stats import ks_2samp
    n = 1200
    args = _args(base, False, s1, 'none')
    src = twin_source(*args)
    twin = np.stack([twin_row(src, 123, e, 1, 0) for e in range(n)])
    ref_src = Q.DynamicsSource(*args, rs=np.random.RandomState(5))
    ref = np.stack([ref_src.sample_row() for _ in range(n)])
    for k, name in enumerate(Q.DYN_FIELDS):
        if np.all(ref[:, k] == ref[0, k]):
            assert np.all(twin[:, k] == ref[0, k]), name
            continue
        assert ks_2samp(twin[:, k], ref[:, k]).pvalue > 1e-3, name


# ---------------------------------------------------------------------------------------------------------------- GPU
EPI_COL = 4 + L.QS_NUM_ENV_STATS + 16           # episode number in the env_i32 state row
SPECS = {1: ('DefaultQuad', True, 'const', 'none'), 5: ('RandomQuad', False, 'none', 'none'),
         8: ('Crazyflie', False, 'rel_normal', 'rel_uniform_custom'), 32: ('RandomQuad', True, 'rel_normal', 'none')}


def _engine(E, N, spec_args, every, seed=3, **kw):
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    return QuadSwarmEngine(num_envs=E, num_agents=N, ep_time=0.05, seed=seed, neighbor_visible_num=min(N - 1, 2),
                           dynamics_sampler=Q.dynamics_sampler_spec(*_args(*spec_args)), dynamics_randomize_every=every, **kw)


def _actions(T, E, N, seed=0):
    import torch
    g = torch.Generator(device='cpu').manual_seed(seed)
    return (torch.rand((T, E, N, 4), generator=g) * 2 - 1).cuda().contiguous()


class _Expected:
    """Twin rows of the last resampling episode of each env (episode 0 = construction)."""

    def __init__(self, spec_args, seed, N, every, env_id_offset=0):
        self.src, self.seed, self.N, self.every, self.off = twin_source(*_args(*spec_args)), seed, N, every, env_id_offset
        self.cache = {}

    def last_due(self, g):
        if not self.every:
            return 0
        return (g // self.every) * self.every

    def rows(self, episodes, envs=None):
        """Rows [len(envs), N, 40] of `envs` (default: all), env envs[k] in episode episodes[k]."""
        out = []
        for e, g in zip(range(len(episodes)) if envs is None else envs, episodes):
            key = (int(e), self.last_due(int(g)))
            if key not in self.cache:
                self.cache[key] = np.stack([twin_row(self.src, self.seed, self.off + key[0], key[1], i) for i in range(self.N)])
            out.append(self.cache[key])
        return np.stack(out)


def _ulps(dev, ref):
    """|dev - ref| in float32 ulp of ref (exact zeros must match exactly)."""
    return np.abs(dev.astype(np.float64) - ref.astype(np.float64)) / np.spacing(np.abs(ref)).astype(np.float64)


def _rows_follow_the_twin(N, spec_args, every, use_numba=True):
    """Staggered envs (explicit masked resets at different steps), >= 3 auto-resets each: after construction and after every
    step the live rows are the twin's rows of each env's last resampling episode, to 2 float32 ulp."""
    import torch
    E, T, seed = 6, 30, 3
    eng = _engine(E, N, spec_args, every, seed=seed, use_numba=use_numba)
    exp = _Expected(spec_args, seed, N, every)
    worst = 0.0

    def check():
        nonlocal worst
        torch.cuda.synchronize()
        epi = eng.get_state()['env_i32'][:, EPI_COL].cpu().numpy()
        rows = eng.get_dynamics().cpu().numpy()
        u = _ulps(rows, exp.rows(epi))
        worst = max(worst, float(u.max()))
        assert u.max() <= 2.0, (epi, np.unravel_index(np.argmax(u), u.shape))
        return epi

    check()
    eng.reset()
    check()
    a = _actions(T, E, N)
    for t in range(T):
        eng.step(a[t])
        if t in (2, 4, 7):                     # explicit resets of some envs: the envs leave lock-step
            mask = np.zeros(E, np.uint8)
            mask[[t % E, (t + 3) % E]] = 1
            eng.reset(env_mask=mask)
        epi = check()
    assert epi.min() >= 4, epi                 # construction + first reset + >= 3 auto-resets per env
    print(f'[dyn twin] N={N} {spec_args} every={every} numba={use_numba}: max |device - twin| = {worst:.2f} ulp')
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 5, 8, 32])
@pytest.mark.parametrize('every', [None, 1, 3])
@pytest.mark.parametrize('use_numba', [True, False])
def test_rows_equal_the_twin_at_every_reset(N, every, use_numba):
    if not use_numba and N not in (5, 32):
        pytest.skip('the numpy dynamics path: two swarm sizes suffice')
    _rows_follow_the_twin(N, SPECS[N], every, use_numba)


@pytest.mark.gpu
@pytest.mark.parametrize('spec_args', [('dict', True, 'rel_normal', 'none'), ('MediumQuad', False, 'rel_uniform_custom', 'const')])
def test_fixed_base_sets_equal_the_twin(spec_args):
    """The other fixed base sets: a user dict with `m` on some parts and `density` on others and no arms.l (both branches of
    the part mass inside one row, the arm length from the geometry), and MediumQuad."""
    _rows_follow_the_twin(5, spec_args, 1)


@pytest.mark.gpu
def test_rewound_episode_number_does_not_latch_a_stale_row():
    """A row prepared for episode 2 (tag pending) must not be latched by a full reset after the episode number was set back:
    that reset starts episode 1, which `every = 2` does not resample, so every drone keeps its construction row."""
    import torch
    E, N, seed = 4, 3, 5
    spec = ('RandomQuad', False, 'none', 'none')
    eng = _engine(E, N, spec, 2, seed=seed)
    exp = _Expected(spec, seed, N, 2)
    eng.reset()                                # episode 1; the generator behind the reset prepares the rows of episode 2
    st = eng.get_state()
    st['env_i32'][:, EPI_COL] = 0
    eng.set_state(st)
    eng.reset()                                # episode 1 again, full mask
    torch.cuda.synchronize()
    epi = eng.get_state()['env_i32'][:, EPI_COL].cpu().numpy()
    assert (epi == 1).all(), epi
    assert _ulps(eng.get_dynamics().cpu().numpy(), exp.rows([0] * E)).max() <= 2.0
    eng.close()


@pytest.mark.gpu
def test_a_row_not_prepared_is_sampled_behind_the_step_grid():
    """A step whose reset finds no prepared row for its episode (the episode number was moved since the row was prepared)
    gets it right behind its grid: the rows after that step are the twin's rows of the new episode."""
    import torch
    E, N, seed = 4, 3, 6
    spec = ('Crazyflie', False, 'rel_normal', 'none')
    eng = _engine(E, N, spec, 1, seed=seed)
    exp = _Expected(spec, seed, N, 1)
    eng.reset()
    a = _actions(3, E, N)
    eng.step(a[0])
    st = eng.get_state()
    epi0 = st['env_i32'][:, EPI_COL].clone()
    st['env_i32'][:, EPI_COL] = epi0 + 5             # the prepared row is the one of episode epi0 + 1
    st['env_i32'][:, 0] = eng.ep_len                 # tick: every env ends its episode in the next step
    eng.set_state(st)
    eng.step(a[1])
    torch.cuda.synchronize()
    epi = eng.get_state()['env_i32'][:, EPI_COL].cpu().numpy()
    assert (epi == epi0.cpu().numpy() + 6).all(), epi
    assert _ulps(eng.get_dynamics().cpu().numpy(), exp.rows(epi)).max() <= 2.0
    eng.close()


def _run_steps(eng, a, mode, chunk=5):
    """Step `eng` through actions a [T,E,N,4] after a reset: one qs_step per step ('step'), one qs_rollout ('rollout'), or
    the first step, then a chained CUDA graph of `chunk` steps replayed over the rest ('graph', (T - 1) % chunk == 0).
    Returns the per-step (obs, rewards, dones) (graph: of the last step of each replay) and the final rows."""
    import torch
    T = a.shape[0]
    eng.reset()
    if mode == 'rollout':
        obs, rew, done = eng.rollout(a)
        return [(obs[t], rew[t], done[t]) for t in range(T)], eng.get_dynamics()
    outs = []
    if mode == 'graph':
        eng.set_chained(True)
        st = torch.cuda.Stream()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            o, r, d = eng.step(a[0])
            outs.append((o.clone(), r.clone(), d.clone()))
            buf = a[1:1 + chunk].clone()
            st.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                for t in range(chunk):
                    o, r, d = eng.step(buf[t])
            for c in range((T - 1) // chunk):
                buf.copy_(a[1 + c * chunk:1 + (c + 1) * chunk])
                g.replay()
                outs.append((o.clone(), r.clone(), d.clone()))
            st.synchronize()
        torch.cuda.synchronize()
        return outs, eng.get_dynamics()
    for t in range(T):
        o, r, d = eng.step(a[t])
        outs.append((o.clone(), r.clone(), d.clone()))
    return outs, eng.get_dynamics()


def _same(outs, ref, steps=None):
    import torch
    steps = range(len(ref)) if steps is None else steps
    return all(torch.equal(x, y) for o, t in zip(outs, steps) for x, y in zip(o, ref[t]))


@pytest.mark.gpu
def test_results_do_not_depend_on_how_steps_are_launched(monkeypatch):
    """qs_step vs qs_rollout vs a chained CUDA graph, QS_PREGEN=0 vs the default cadence, two shards vs one handle: the
    same observations, rewards, dones and rows, bit for bit."""
    import torch
    E, N, T, seed = 24, 8, 41, 9
    spec = SPECS[32]
    a = _actions(T, E, N, seed=1)
    base, base_rows = _run_steps(_engine(E, N, spec, 1, seed=seed), a, 'step')
    outs, rows = _run_steps(_engine(E, N, spec, 1, seed=seed), a, 'rollout')
    assert _same(outs, base) and torch.equal(rows, base_rows)
    outs, rows = _run_steps(_engine(E, N, spec, 1, seed=seed), a, 'graph')
    assert _same(outs, base, steps=range(0, T, 5)) and torch.equal(rows, base_rows)
    for cadence in ('0', '1'):             # every row sampled inside the resets / the generator before every step
        monkeypatch.setenv('QS_PREGEN', cadence)
        outs, rows = _run_steps(_engine(E, N, spec, 1, seed=seed), a, 'step')
        monkeypatch.delenv('QS_PREGEN')
        assert _same(outs, base) and torch.equal(rows, base_rows), cadence
    # two shards of E / 2 envs (env_id_offset keys the draws), both with the collision radii of one quad_arm
    h = E // 2
    arm = float(base_rows[0, 0, Q.DYN_FIELDS.index('arm')])
    shards = [_run_steps(_engine(h, N, spec, 1, seed=seed, env_id_offset=k * h, quad_arm=arm), a[:, k * h:(k + 1) * h].contiguous(),
                         'step') for k in range(2)]
    one, one_rows = _run_steps(_engine(E, N, spec, 1, seed=seed, quad_arm=arm), a, 'step')
    for t in range(T):
        for q in range(3):
            assert torch.equal(torch.cat([shards[0][0][t][q], shards[1][0][t][q]]), one[t][q]), (t, q)
    assert torch.equal(torch.cat([shards[0][1], shards[1][1]]), one_rows)


@pytest.mark.gpu
def test_rows_uploaded_at_the_same_resets_fly_the_same():
    """A handle without the sampler that receives the sampler's rows through qs_set_dynamics(at_next_reset) before the
    resets that latch them flies bit-identical trajectories."""
    import torch
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    E, N, T, seed = 8, 8, 36, 4
    spec = SPECS[8]
    A = _engine(E, N, spec, 3, seed=seed)
    B = QuadSwarmEngine(num_envs=E, num_agents=N, ep_time=0.05, seed=seed, neighbor_visible_num=2)
    B.set_dynamics(A.get_dynamics())
    a = _actions(T, E, N, seed=2)
    A.reset(); B.reset()
    A2 = _engine(E, N, spec, 3, seed=seed)          # runs one step ahead of A to know which envs latch new rows
    A2.reset()
    for t in range(T):
        before = A.get_dynamics()
        A2.step(a[t])
        after = A2.get_dynamics()
        changed = (after != before).flatten(1).any(1).to(torch.uint8)
        if bool(changed.any()):
            B.set_dynamics(after, env_mask=changed, at_next_reset=True)
        oa, ra, da = A.step(a[t])
        ob, rb, db = B.step(a[t])
        assert torch.equal(oa, ob) and torch.equal(ra, rb) and torch.equal(da, db), t
        assert torch.equal(A.get_dynamics(), B.get_dynamics()), t
    assert int(A.get_state()['env_i32'][:, EPI_COL].min()) >= 4


@pytest.mark.gpu
def test_entry_point_validation():
    import torch
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    lib = L.load()
    good = L.dyn_sampler_struct(Q.dynamics_sampler_spec('RandomQuad'))

    def fresh():
        return QuadSwarmEngine(num_envs=2, num_agents=3, ep_time=0.05, seed=1)

    e = fresh()
    out = torch.empty((2, 3, L.QS_DYN_ROW), device='cuda')
    assert lib.qs_get_dynamics(e.h, ctypes.c_void_p(out.data_ptr()), None) == -1      # no per-drone rows yet
    assert lib.qs_set_dynamics_sampler(e.h, None, 0) == -1
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(good), -1) == -1
    bad = [('base', 7), ('n_order', 3)]
    for field, v in bad:
        s = L.dyn_sampler_struct(Q.dynamics_sampler_spec('RandomQuad'))
        setattr(s, field, v)
        assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(s), 0) == -1, field
    s = L.dyn_sampler_struct(Q.dynamics_sampler_spec('Crazyflie'))
    s.params.value[Q.DYN_LEAVES.index((('motor', 'thrust_to_weight'), None))] = float('inf')
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(s), 0) == -1
    s = L.dyn_sampler_struct(Q.dynamics_sampler_spec('Crazyflie'))
    s.sampler[1] = 9
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(s), 0) == -1
    s = L.dyn_sampler_struct(Q.dynamics_sampler_spec('Crazyflie'))
    s.params.present[Q.DYN_LEAVES.index((('geom', 'body', 'w'), None))] = 0
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(s), 0) == -1
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(good), 2) == 0
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(good), 2) == -1           # once
    e.get_dynamics()
    with pytest.raises(L.QsError, match='sampler'):
        e.set_dynamics(np.zeros((2, 3, L.QS_DYN_ROW), np.float32))              # the sampler owns the rows
    e.close()
    e = fresh()
    e.reset()
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(good), 0) == -1           # after the first reset
    e.close()
    e = fresh()
    e.set_dynamics(np.tile(Q.constants_row(Q.crazyflie_params()), (2, 3, 1)))
    assert lib.qs_set_dynamics_sampler(e.h, ctypes.byref(good), 0) == -1           # rows from qs_set_dynamics
    e.close()


@pytest.mark.gpu
def test_batched_training_env_with_replay_c3():
    """c3-sized (4096 envs x 8 drones, obstacles, o_random) wrapped training env with collision-event replay and device-side
    RandomQuad rows resampled every episode.  A collision planted in every other env puts an event in its buffer; over four
    episodes the outputs stay finite, events are replayed, and every env's live rows are the twin's rows of its episode
    number: a replayed event keeps the env's live constants, and replay never rewinds the episode number."""
    import torch
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    from quad_swarm_rl_b200.training import BatchedTrainingEnv
    E, N, seed = 4096, 8, 21
    env = QuadrotorEnvMultiBatched(E, num_agents=N, ep_time=2.5, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor',
                                   use_obstacles=True, use_downwash=True, quads_mode='o_random', seed=seed,
                                   dynamics_params='RandomQuad', dynamics_randomize_every=1, device_dynamics=True)
    assert env._dyn_sources is None
    w = BatchedTrainingEnv(env, replay_buffer_sample_prob=0.75, replay_always_active=True, stats_every=1 << 30)
    w.reset()
    g = torch.Generator(device='cuda')
    g.manual_seed(2)
    planted = torch.arange(E, device='cuda') % 2 == 0
    for t in range(4 * (env.ep_len + 1)):
        if t == 200:                                         # drone 1 onto drone 0: a collision 1.5 s after a checkpoint
            st = env.engine.get_state()
            st['agent_f32'][planted, 1, 0:3] = st['agent_f32'][planted, 0, 0:3] + 0.01
            env.engine.set_state(st, env_mask=planted)
        act = 0.05 + 0.3 * (torch.rand((E * N, 4), device='cuda', generator=g) * 2 - 1)
        obs, rew, term, trunc, infos = w.step(act)
        assert torch.isfinite(obs).all() and torch.isfinite(rew).all(), t
    torch.cuda.synchronize()
    w.flush_stats()
    assert w.totals['replayed_events'] > 0
    epi = env.engine.get_state()['env_i32'][:, EPI_COL].cpu().numpy()
    assert epi.min() >= 4
    rows = env.engine.get_dynamics().cpu().numpy()
    exp = _Expected(('RandomQuad', False, 'none', 'none'), seed, N, 1)
    pick = np.arange(0, E, 64)                               # planted envs
    assert _ulps(rows[pick], exp.rows(epi[pick], envs=pick)).max() <= 2.0
    # quad_arm: the construction row of env 0, drone 0
    arm = Q.DYN_FIELDS.index('arm')
    assert _ulps(np.float32(env.quad_arm), exp.rows([0])[0, 0, arm]) <= 2.0
    env.engine.close()
