"""Swarm sizes 9 to 31: the 16-lane kernel group (N = 9..16) and the partly filled 32-lane group (N = 17..31) against the CPU
oracle.  A swarm of N drones runs on a lane group of NP = next_pow2(N) lanes and every kernel is templated on NP, so these
sizes run instantiations (and idle-lane patterns) that N <= 8 and N = 32 never reach: 16-bit group ballots, the k-nearest
argsort over 16 / 32 candidates with idle lanes at +inf, pair bits >= 16, two envs per physics / observer warp pair in the
split shape, warp tiles of 18..32 observation rows, 16-lane wrapper reductions.

Tolerances are the suite's: observations, rewards and state within 1e-4 + 1e-4 |ref|; collision, pillar, floor and kick
masks bit for bit on every env-step that run_parity compares.  Every case states its bound on the env-steps run_parity
skips (decisions closer to a threshold than float32 resolves; drones resting against each other, a wall or the floor sit
there), asserts a minimum number of compared env-steps, and asserts that its events (episode ends, collisions, kicks, floor
and pillar contacts, goal events) actually happened.

CPU: every step-kernel instantiation NP = 16 / 32 can select is in the library and uses no local memory."""
import re
import subprocess

import numpy as np
import pytest

from tests.parity_util import DevicePair, Pair, SampledPair, kernel_resources, run_parity
from tests.test_gpu_parity import _cluster_hook, _dyn_rows, _obst_hook, _params_of, _room_hook
from tests.test_init_random_state import _arm_oracles, _on
from tests.test_numpy_path import _plant_floor
from tests.test_sensor_noise import _noise_pair
from tests.test_step_shape import ROOT, _stagger

FLOOR = 'xyz_vxyz_R_omega_floor'
WALL = 'xyz_vxyz_R_omega_wall'
COL_REW = dict(quadcol_bin=5.0, quadcol_bin_smooth_max=10.0)


def _np(n):
    return 1 << (n - 1).bit_length()


def _spread(n):
    """Half-width of a planted cluster: the 8-drone clusters of test_gpu_parity.py (0.12 m) at the same drone density."""
    return 0.12 * (n / 8) ** 0.5


def _events_hook(n, every=36, extra=None):
    """Clusters flying at each other (collisions, kicks, downwash) every `every` steps and, half-way between them, drones
    planted on walls, ceiling and floor."""
    cluster = _cluster_hook((0.0, 0.0, 3.0), _spread(n), 0.6, every)
    room = _room_hook(every)

    def hook(p, t):
        cluster(p, t)
        room(p, t + every // 2)
        if extra is not None:
            extra(p, t)
    return hook


def _parity(pair, T, seed, **kw):
    rep = run_parity(pair, T, np.random.RandomState(seed), **kw)
    total = rep['skipped_env_steps'] + rep['compared_env_steps']
    rep['skipped_frac'] = rep['skipped_env_steps'] / max(1, total)
    print(f'N={pair.N} E={pair.E} T={T}: {rep}')
    return rep


def _check(rep, bound, min_compared, **at_least):
    assert rep['skipped_frac'] <= bound, rep
    assert rep['compared_env_steps'] >= min_compared, rep
    for k, v in at_least.items():
        assert rep[k] >= v, (k, rep)


# The launch shape is read from a profiler trace (test_step_shape._step_grid_shape) of a twin engine in a process of its
# own: in one process, only the first few profiler sessions record the kernels.
_PROBE = """
import json, pathlib, sys
import torch
from quad_swarm_rl_b200.engine import QuadSwarmEngine
from tests.test_step_shape import _step_grid_shape
a = json.loads(sys.argv[1])
eng = QuadSwarmEngine(**a['kw'])
eng.set_chained(a['chained'])
eng.reset()
x = torch.zeros((eng.E, eng.N, 4), device='cuda')
eng.step(x)
grid, block = _step_grid_shape(torch, eng, x, pathlib.Path(a['tmp']))
names = [e['name'] for e in json.load(open(pathlib.Path(a['tmp']) / 'trace.json'))['traceEvents']
         if 'qs_step_kernel' in e.get('name', '') and 'grid' in e.get('args', {})]
print(json.dumps([grid, block, names[-1]]))
"""
# template arguments <NP, SPLIT, SCN, HO, DYN, NZ> of a step kernel, demangled or mangled
_TARGS = (re.compile(r'qs_step_kernel(?:_npy)?<(\d+), (true|false), (true|false), (true|false), (true|false), (true|false)>'),
          re.compile(r'qs_step_kernel(?:_npy)?ILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELb([01])E'))


def _launch(kw, E, tmp_path, chained=False, device_scenario=None):
    """(grid, block, kernel name) of a step launch of an engine built like the test's (same config, same QS_* switches)."""
    import json
    import sys
    arg = json.dumps(dict(kw=dict(kw, num_envs=E, seed=1, device_scenario=device_scenario), chained=chained,
                          tmp=str(tmp_path)))
    out = subprocess.run([sys.executable, '-c', _PROBE, arg], capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-3000:]
    return tuple(json.loads(out.stdout.strip().splitlines()[-1]))


def _grid_block(kw, E, tmp_path, **launch):
    return _launch(kw, E, tmp_path, **launch)[:2]


def _hand_over(name):
    """HO template argument of the launched step kernel: per-block hand-over (True) or grid-wide wait (False)."""
    for rx in _TARGS:
        m = rx.search(name)
        if m:
            return m.group(4) in ('true', '1')
    raise AssertionError(f'no template arguments in {name!r}')


def _shape(E, n, split):
    """(grid, block) of the split shape (one env group per physics / observer warp pair) or the single-warp shape (two
    warps of env groups per 64-thread CTA)."""
    per_block = (32 if split else 64) // _np(n)
    return (E + per_block - 1) // per_block, 64


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# 1. parity over swarm sizes, in both small-batch shapes
# ---------------------------------------------------------------------------------------------------------------------
# (id, config, E, D, observation write-out of the staged shapes)
ROWS = [
    ('n9_k1', dict(num_agents=9, neighbor_visible_num=1), 7, 24, 'tensor store'),
    ('n12_k6_floor_pillars_downwash', dict(num_agents=12, neighbor_visible_num=6, obs_repr=FLOOR, use_obstacles=True,
                                           use_downwash=True), 8, 64, 'tensor store, 24-row box'),
    ('n12_all', dict(num_agents=12, neighbor_visible_num=-1), 9, 84, 'unstaged'),
    ('n16_k6', dict(num_agents=16, neighbor_visible_num=6), 6, 54, 'linear bulk copy'),
    ('n16_k14_wall', dict(num_agents=16, neighbor_visible_num=14, obs_repr=WALL), 4, 108, 'unstaged'),
    ('n17_k2_floor_pillars', dict(num_agents=17, neighbor_visible_num=2, obs_repr=FLOOR, use_obstacles=True), 5, 40,
     'tensor store, 17-row box'),
    ('n24_k6_wall_downwash', dict(num_agents=24, neighbor_visible_num=6, obs_repr=WALL, use_downwash=True), 4, 60,
     'tensor store, 24-row box'),
    ('n31_k3_floor', dict(num_agents=31, neighbor_visible_num=3, obs_repr=FLOOR), 3, 37, 'linear bulk copy (odd D)'),
]
MATRIX = [(r, s) for r in ROWS for s in (('0', '1') if r[3] <= 72 else (None,))]


@pytest.mark.gpu
@pytest.mark.parametrize('row,split', MATRIX, ids=[f'{r[0]}-{"auto" if s is None else ("split" if s == "1" else "single")}'
                                                   for r, s in MATRIX])
def test_parity_over_swarm_sizes(row, split, monkeypatch, tmp_path):
    """Pair + run_parity(resync=20), with planted clusters, wall / ceiling / floor contacts and (with pillars) pillar
    contacts.  Rows of D <= 72 run in the split shape (QS_SPLIT=1) and in the single-warp shape (QS_SPLIT=0); wider rows
    are never staged and take the single-warp shape.  Skip bound: 10 % of the env-steps for N <= 16, 20 % for N > 16 (more
    drones rest against each other after a planted collision); at least half of them compared."""
    name, cfg, E, D, _ = row
    if split is not None:
        monkeypatch.setenv('QS_SPLIT', split)
    n, T = cfg['num_agents'], 72
    kw = dict(cfg, ep_time=0.3)
    pair = Pair(E, kw, seed=9000 + n, table_seed=9100 + n, rew_coeff=COL_REW)
    assert pair.engine.D == D
    obst = kw.get('use_obstacles', False)
    rep = _parity(pair, T, 9200 + n, resync=20, hook=_events_hook(n, extra=_obst_hook(24) if obst else None))
    _check(rep, 0.10 if n <= 16 else 0.20, 0.5 * E * T, dones=2 * E, quadcol=1, kicked=1, floor=1, obstcol=1 if obst else 0)
    assert _grid_block(kw, E, tmp_path) == _shape(E, n, split == '1')
    pair.engine.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. tight masks in dense clusters
# ---------------------------------------------------------------------------------------------------------------------
def _pair_tracker(pairs_seen, multi):
    """Hook part that reads every oracle env's colliding pairs (prev_drone_collisions) after each step: the pairs that are
    new in that step, and the env-steps that resolve more than one new pair."""
    last = {}

    def hook(p, t):
        for e, o in enumerate(p.oracles):
            cur = set(tuple(sorted(map(int, q))) for q in o.prev_drone_collisions)
            new = cur - last.get(e, set())
            pairs_seen.update(new)
            multi[0] += int(len(new) > 1)
            last[e] = cur
    return hook


TIGHT = [
    ('cluster_16', dict(num_agents=16, neighbor_visible_num=6, use_downwash=True, ep_time=2.0), 6),
    ('cluster_24', dict(num_agents=24, neighbor_visible_num=6, use_downwash=True, ep_time=2.0), 4),
    ('room_12', dict(num_agents=12, neighbor_visible_num=2, ep_time=1.0), 6),
]


@pytest.mark.gpu
@pytest.mark.parametrize('name,kw,E', TIGHT, ids=[c[0] for c in TIGHT])
def test_masks_bit_exact_in_dense_swarms(name, kw, E):
    """Teacher forcing after every step (resync=1, margin 3e-6, neighbour gap 5e-6): collision / floor / kick masks bit for
    bit on at least 98 % of the env-steps (skip bound 2 %; 4 % for the room contacts of 12 drones, see below).  The clusters make new pairs among drones 8..15 and, at N = 24,
    pairs with an index >= 16, and env-steps with several new pairs (the pair-resolution loop runs more than once)."""
    n, T = kw['num_agents'], 110
    pairs, multi = set(), [0]
    track = _pair_tracker(pairs, multi)
    if name.startswith('cluster'):
        plant = _cluster_hook((0.0, 0.0, 3.0), _spread(n), 0.6, 25)
    else:
        plant = _room_hook(30)

    def hook(p, t):
        track(p, t)
        plant(p, t)
    pair = Pair(E, kw, seed=4242 + n, table_seed=4243 + n, rew_coeff=COL_REW)
    rep = _parity(pair, T, 4244 + n, resync=1, margin_eps=3e-6, gap_eps=5e-6, hook=hook)
    print(name, 'new pairs', sorted(pairs), 'env-steps with several new pairs', multi[0])
    if name.startswith('cluster'):
        _check(rep, 0.02, 0.9 * E * T, quadcol=1, kicked=1)
        assert any(min(q) >= 8 for q in pairs), sorted(pairs)
        if n > 16:
            assert any(max(q) >= 16 for q in pairs), sorted(pairs)
        assert multi[0] >= 1
    else:
        # the room hook plants every drone on a wall, the ceiling or the floor; a drone resting on a surface sits on that
        # threshold while it rests, so the skipped env-steps grow with the drones per env: the 6-drone case of
        # test_gpu_parity.py keeps 2 %, twice the drones 4 %
        _check(rep, 0.04, 0.9 * E * T, kicked=1, floor=1, dones=E)
    pair.engine.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. launch shapes at the batch sizes users run
# ---------------------------------------------------------------------------------------------------------------------
SAMPLED = [
    # (id, N, E, scenario, chained, QS_PDL, split shape on 132 SMs, per-block hand-over)
    ('n16_e1000_split_chained', 16, 1000, 'static_same_goal', True, None, True, True),
    ('n16_e2048_single_chained_pillars', 16, 2048, 'o_random', True, None, False, True),
    ('n16_e8192_multiwave_chained', 16, 8192, 'static_same_goal', True, None, False, True),
    ('n16_e2048_unchained', 16, 2048, 'static_same_goal', False, None, False, False),
    ('n16_e2048_chained_wait_pillars', 16, 2048, 'o_random', True, '2', False, False),
    ('n24_e512_split_chained', 24, 512, 'swarm_vs_swarm', True, None, True, True),
    ('n24_e1024_single_chained_pillars', 24, 1024, 'o_random', True, None, False, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize('name,n,E,scn,chained,pdl,split,ho', SAMPLED, ids=[c[0] for c in SAMPLED])
def test_sampled_envs_in_full_size_launch_shapes(name, n, E, scn, chained, pdl, split, ho, monkeypatch, tmp_path):
    """SampledPair: envs 0, E/2 and E-1 against the oracle while all E envs run, in the shape plan_step picks: the split
    shape while E*NP/32 <= 4 x SMs, the single-warp shape above.  Between chained step grids the split shape and pillar
    tables take the per-block hand-over, and so does a grid of several waves (8192 envs: 2048 CTAs); a single-wave grid
    without pillars takes the grid-wide wait, and QS_PDL=2 forces the wait on a batch with pillars.  An unchained handle
    never hands over.  The grid, block and HO template argument of the launched kernel are asserted (132 SMs).  Planted
    clusters and contacts; skip bound 15 %, at least 80 % of the sampled env-steps compared; no hand-over timed out."""
    from oracle.scenario_gen import DeviceORandomSource, DeviceScenarioSource
    if pdl is not None:
        monkeypatch.setenv('QS_PDL', pdl)
    obst = scn == 'o_random'
    kw = dict(num_agents=n, neighbor_visible_num=6 if n == 16 else 4, ep_time=0.3)
    if obst:
        kw.update(obs_repr=FLOOR, use_obstacles=True, use_downwash=True)
        fac = lambda: DeviceORandomSource()
    else:
        fac = lambda: DeviceScenarioSource(scn)
    T = 70
    pair = SampledPair(E, [0, E // 2, E - 1], kw, seed=31000 + E + n, device_scenario=scn, source_factory=fac,
                       chained=chained, rew_coeff=dict(COL_REW, quadcol_bin_obst=5.0) if obst else COL_REW)
    rep = _parity(pair, T, 13, resync=20, hook=_events_hook(n, extra=_obst_hook(24) if obst else None))
    _check(rep, 0.15, 0.8 * 3 * T, dones=3, quadcol=1, kicked=1, floor=1, obstcol=1 if obst else 0)
    if _sms() == 132:
        grid, block, kernel = _launch(kw, E, tmp_path, chained=chained, device_scenario=scn)
        print(kernel)
        assert (grid, block) == _shape(E, n, split) and _hand_over(kernel) == ho
    assert pair.engine.handover_timeouts == 0
    pair.engine.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. feature kernels at NP = 16 and partly filled NP = 32
# ---------------------------------------------------------------------------------------------------------------------
FEAT_KW = {12: dict(num_agents=12, neighbor_visible_num=2, obs_repr=WALL, use_downwash=True),
           24: dict(num_agents=24, neighbor_visible_num=6, obs_repr=FLOOR)}


@pytest.mark.gpu
@pytest.mark.parametrize('n', [12, 24])
def test_per_drone_dynamics_at_swarm_sizes(n):
    """DYN kernels: 'zoo' airframes (every model in every env), replaced with at_next_reset=True at step 30 and latched at
    each env's auto-reset (single-warp kernels with the grid-wide wait).  Skip bound 10 % (N = 12), 20 % (N = 24)."""
    E, T = 4, 100
    kw = dict(FEAT_KW[n], ep_time=0.4)
    rows0, rows1 = _dyn_rows(E, n, 1), _dyn_rows(E, n, 2)
    pair = Pair(E, kw, seed=777 + n, table_seed=778 + n, rew_coeff=COL_REW)
    pair.engine.set_dynamics(rows0)
    P0, P1 = _params_of(rows0), _params_of(rows1)
    pending = [[False] * n for _ in range(E)]
    for e, o in enumerate(pair.oracles):
        o.Ps = list(P0[e])
        o.P = o.Ps[0]

        def src(i, e=e):
            if pending[e][i]:
                pending[e][i] = False
                return P1[e][i]
            return None
        o.dyn_source = src

    def swap(p, t):
        if t == 30:
            p.engine.set_dynamics(rows1, at_next_reset=True)
            for e in range(E):
                pending[e] = [True] * n
    rep = _parity(pair, T, 3, resync=20, hook=_events_hook(n, extra=swap))
    _check(rep, 0.10 if n <= 16 else 0.20, 0.5 * E * T, dones=2 * E, quadcol=1, kicked=1, floor=1)
    assert not any(any(x) for x in pending)                   # every env latched the new constants
    pair.engine.close()


NOISE_GYRO = dict(gyro_norm_std=1.0, gyro_bias_correlation_time=0.05, gyro_noise_density=0.005, gyro_random_walk=0.02,
                  pos_unif_range=0.01, quat_norm_std=0.01)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [12, 24])
def test_noise_model_with_gyro_bias_at_swarm_sizes(n):
    """NZ kernels: a noise dict with the gyro-bias model; the bias of every drone is compared before every step
    (1e-4 + 1e-4 |ref|); single-warp kernels with the grid-wide wait.  Skip bound 10 % (N = 12), 20 % (N = 24)."""
    E, T = 4, 90
    kw = dict(FEAT_KW[n], ep_time=0.4, sense_noise=NOISE_GYRO)
    pair = _noise_pair(E, kw, seed=31 + n)
    assert pair.engine.gyro_model
    checked = [0]

    def check_bias(p, t):
        ref = p.oracle_bias()
        dev = p.engine.get_gyro_bias().cpu().numpy().astype(np.float64)
        err = np.abs(dev - ref)
        assert (err <= 1e-4 + 1e-4 * np.abs(ref)).all(), f'gyro bias before step {t}: {err.max():.3e}'
        checked[0] += 1
    rep = _parity(pair, T, 4, resync=10, hook=_events_hook(n, extra=check_bias))
    check_bias(pair, T)
    _check(rep, 0.10 if n <= 16 else 0.20, 0.5 * E * T, dones=2 * E, quadcol=1, kicked=1, floor=1)
    assert checked[0] == T + 1 and np.abs(pair.oracle_bias()).max() > 1e-4
    pair.engine.close()


@pytest.mark.gpu
@pytest.mark.parametrize('split', ['0', '1'], ids=['single', 'split'])
@pytest.mark.parametrize('n', [12, 24])
def test_numpy_dynamics_path_at_swarm_sizes(n, split, monkeypatch):
    """qs_step_kernel_npy (use_numba=False) with planted floor states, against oracle/numpy_path_oracle.py, in the split and
    the single-warp shape.  on_floor / crashed_floor masks bit for bit away from thresholds.  Skip bound 60 %, as for the
    32-drone numpy-path case of test_numpy_path.py: drones resting on the floor lift off by micrometres whenever their
    random thrust exceeds their weight, and those env-steps decide the 0.05 m threshold within float32 resolution."""
    from oracle import numpy_path_oracle as npo
    monkeypatch.setenv('QS_SPLIT', split)
    E, T = 4, 80
    kw = dict(num_agents=n, neighbor_visible_num=2 if n == 12 else 6, ep_time=0.9, obs_repr=FLOOR, use_numba=False)
    pair = Pair(E, kw, seed=7200 + n, table_seed=7210 + n)
    npo.enable(pair.ocfg)
    counts = dict(crashed_floor=0)
    rep = _parity(pair, T, 31, resync=10, hook=lambda p, t: _plant_floor(p, t, counts))
    ds = [d for o in pair.oracles for d in o.drones]
    seen = dict(slides=sum(getattr(d, 'slides', 0) for d in ds), corner=sum(getattr(d, 'slide_corner', 0) for d in ds),
                landings=sum(getattr(d, 'landings_upside_down', 0) for d in ds),
                tries=sum(getattr(d, 'landing_yaw_tries', 0) for d in ds))
    print(seen, counts)
    _check(rep, 0.6, 0.3 * E * T, floor=1)
    assert counts['crashed_floor'] > 0
    assert seen['slides'] > 0 and seen['corner'] > 0 and seen['tries'] > seen['landings'] > 0, seen
    pair.engine.close()


@pytest.mark.gpu
@pytest.mark.parametrize('n', [12, 24])
def test_random_initial_states_at_swarm_sizes(n):
    """qs_reset_kernel<NP, *, true>: random spawn velocity, body rate and attitude at the explicit reset and every
    auto-reset, against the oracle with the option on.  Skip bound 10 % (N = 12), 20 % (N = 24)."""
    E, T = 4, 100
    kw = _on(dict(FEAT_KW[n], ep_time=0.4))
    pair = _arm_oracles(Pair(E, kw, seed=4100 + n, table_seed=4101 + n, rew_coeff=COL_REW), kw)
    rep = _parity(pair, T, 4102 + n, resync=10, hook=_events_hook(n))
    resets = sum(getattr(o, 'init_resets', 0) for o in pair.oracles)
    _check(rep, 0.10 if n <= 16 else 0.20, 0.5 * E * T, dones=2 * E, quadcol=1, kicked=1, floor=1)
    assert resets == (E + rep['dones']) * n, (resets, rep)
    pair.engine.close()


@pytest.mark.gpu
def test_per_episode_pillar_randomisation_16_drones():
    """qs_set_obstacle_randomization at N = 16: per-episode pillar count and radius drawn on the device equal the twin's, and
    the trajectories stay in parity across auto-resets.  Skip bound 10 %."""
    from oracle.scenario_gen import DeviceORandomSource
    from quad_swarm_rl_b200 import _lib as L
    dens = [0.05, 0.1, 0.15000000000000002, 0.2]
    sizes = [0.3, 0.4, 0.5, 0.6000000000000001, 0.7000000000000002]
    kw = dict(num_agents=16, neighbor_visible_num=2, obs_repr=FLOOR, use_obstacles=True, use_downwash=True, ep_time=0.4)
    E, T = 6, 130
    pair = DevicePair(E, kw, 1357, 'o_random', lambda: DeviceORandomSource(densities=dens, sizes=sizes))
    pair.engine.set_obstacle_randomization(dens, sizes)
    seen_m, seen_r = set(), set()

    def check(p, t):
        if t % 41 == 5:
            st = p.engine.get_state()
            base = 4 + L.QS_NUM_ENV_STATS
            rad_m = st['env_i32'][:, base + 4:base + 6].cpu().numpy().view(np.float32)
            for e, o in enumerate(p.oracles):
                assert rad_m[e, 0] == np.float32(o.obst_size / 2) and int(rad_m[e, 1]) == len(o.obst_xy) == o.source.num_pillars
                ob = st['obst_xy'][e].cpu().numpy()
                assert np.array_equal(ob[:len(o.obst_xy)], o.obst_xy.astype(np.float32)) and (ob[len(o.obst_xy):] == 1.0e4).all()
                seen_m.add(len(o.obst_xy))
                seen_r.add(float(rad_m[e, 0]))
    rep = _parity(pair, T, 8, resync=20, hook=check)
    print(sorted(seen_m), sorted(seen_r))
    _check(rep, 0.10, 0.5 * E * T, dones=3 * E)
    assert len(seen_m) >= 3 and len(seen_r) >= 3
    pair.engine.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. device-side scenarios
# ---------------------------------------------------------------------------------------------------------------------
SCENARIOS = [
    ('swarm_vs_swarm', 13, 2), ('swarm_vs_swarm', 24, 2), ('dynamic_formations', 16, 3), ('ep_lissajous3D', 16, 3),
    # run_away at 16 drones: at step 112 a drone sliding on the floor stops within a sub-step and its friction direction
    # comes from a velocity of 1.2e-6 m/s, which float32 does not resolve; the oracle's step margin covers that decision
    ('run_away', 16, 3),
    ('o_random', 16, 4), ('o_ep_rand_bezier', 16, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize('mode,n,E', SCENARIOS, ids=[f'{m}-{n}' for m, n, _ in SCENARIOS])
def test_device_scenarios_at_swarm_sizes(mode, n, E):
    """Episodes, goals and goal events generated inside the kernels equal oracle/scenario_gen.py's twin; goals are
    compared every step (state 'goal') across goal events and auto-resets.  Every drone observes all its neighbours: the
    goal formations put drones at equal distances from each other, a k-nearest order that float32 does not resolve, and
    with k < N - 1 most env-steps would be skipped.  Skip bound 60 %, at least 40 % compared: under random actions most
    drones come to rest on the floor within the episode, and a resting drone lifts off by micrometres whenever its random
    thrust exceeds its weight, which decides the floor threshold within float32 resolution; with 13 to 24 drones per env
    one of them does so in about half of the env-steps (36 % at N = 13, 54 % at N = 24 measured on an H100).  Goals are
    also compared directly at the end, whatever was skipped."""
    from oracle.scenario_gen import DeviceORandomSource, DeviceScenarioSource
    from quad_swarm_rl_b200 import _lib as L
    periodic = mode in ('swarm_vs_swarm', 'o_ep_rand_bezier')           # first goal event after 4-6 s
    kw = dict(num_agents=n, neighbor_visible_num=-1, ep_time=6.3 if periodic else (0.5 if mode == 'o_random' else 1.2))
    if mode.startswith('o_'):
        kw.update(obs_repr=FLOOR, use_obstacles=True, use_downwash=True)
        fac = lambda: DeviceORandomSource(scenario=mode)
    else:
        fac = lambda: DeviceScenarioSource(mode)
    T = 660 if periodic else (130 if mode == 'o_random' else 260)
    pair = DevicePair(E, kw, 97531 + n, mode, fac)
    rep = _parity(pair, T, 11, resync=10)
    _check(rep, 0.60, 0.4 * E * T, dones=E)
    if mode != 'o_random':
        assert all(o.source.events >= 1 for o in pair.oracles)
    st = pair.engine.get_state()
    goals = st['agent_f32'][..., 30:33].cpu().numpy()
    for e, o in enumerate(pair.oracles):
        np.testing.assert_allclose(goals[e], np.array([d.goal for d in o.drones]), rtol=1e-5, atol=1e-5)
        if kw.get('use_obstacles'):
            assert np.array_equal(st['obst_xy'][e].cpu().numpy(), o.obst_xy.astype(np.float32))
    es, _ = pair.engine.episode_stats()
    assert {int(x) for x in es[:, 12].cpu().numpy()} == {L.DEVICE_SCENARIOS[mode]}
    pair.engine.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. bit-identity of the execution paths
# ---------------------------------------------------------------------------------------------------------------------
PATHS = [
    # (id, config, E, device scenario): E*NP/32 <= 528 takes the split shape, above the single-warp one
    ('n16_floor_pillars_d64', dict(num_agents=16, neighbor_visible_num=6, obs_repr=FLOOR, use_obstacles=True,
                                   use_downwash=True), 301, 'o_random'),
    ('n24_wall_d60', dict(num_agents=24, neighbor_visible_num=6, obs_repr=WALL, use_downwash=True), 1100, 'static_same_goal'),
    ('n31_floor_d37', dict(num_agents=31, neighbor_visible_num=3, obs_repr=FLOOR), 301, 'static_same_goal'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('name,cfg,E,scn', PATHS, ids=[c[0] for c in PATHS])
def test_execution_paths_are_bit_identical(name, cfg, E, scn, monkeypatch):
    """With staggered episode ticks (auto-resets inside every chain), torch.equal on observations, rewards, dones and the
    state between: rollout(T); T single steps; a CUDA graph of T chained steps; the host-buffer path (qs_step_host);
    rollout(T, last_obs_only=True); a rollout with QS_OBS_BULK=0 (vector stores instead of the copy engine: at D = 37 the
    1-wide stores); a CUDA graph of chained steps that all write the engine's own output arrays."""
    import torch
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    n, T = cfg['num_agents'], 60

    def mk():
        e = QuadSwarmEngine(num_envs=E, seed=21, ep_time=0.3, device_scenario=scn, **cfg)
        e.reset()
        _stagger(torch, e, 77)
        e.step(torch.zeros((E, n, 4), device='cuda'))       # the launch decisions are made before any graph capture
        return e
    ref, steps, graph, host, last, same = (mk() for _ in range(6))
    monkeypatch.setenv('QS_OBS_BULK', '0')
    vec = mk()
    monkeypatch.delenv('QS_OBS_BULK')
    g = torch.Generator(device='cuda')
    g.manual_seed(5)
    a = (torch.rand((T, E, n, 4), device='cuda', generator=g) * 2 - 1).contiguous()
    o_r, r_r, d_r = ref.rollout(a)
    torch.cuda.synchronize()
    assert int(d_r.sum()) > E * n                                  # auto-resets inside the chain

    def same_state(e):
        s1, s2 = ref.get_state(), e.get_state()
        for k in ('agent_f32', 'agent_u32', 'env_i32', 'obst_xy'):
            assert torch.equal(s1[k], s2[k]), k

    # T single steps
    o1, r1, d1 = torch.empty_like(o_r), torch.empty_like(r_r), torch.empty_like(d_r)
    for t in range(T):
        steps.step(a[t], obs_out=o1[t], rewards_out=r1[t], dones_out=d1[t])
    assert torch.equal(o1, o_r) and torch.equal(r1, r_r) and torch.equal(d1, d_r)
    same_state(steps)
    # CUDA graphs of chained steps: into a ring of outputs, and into the engine's own arrays
    o3, r3, d3 = torch.empty_like(o_r), torch.empty_like(r_r), torch.empty_like(d_r)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        graphs = []
        for eng, ring in ((graph, True), (same, False)):
            eng.set_chained(True)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=st):
                for t in range(T):
                    if ring:
                        eng.step(a[t], obs_out=o3[t], rewards_out=r3[t], dones_out=d3[t])
                    else:
                        eng.step(a[t])
            graphs.append(gr)
        for gr in graphs:
            gr.replay()
        st.synchronize()
    assert torch.equal(o3, o_r) and torch.equal(r3, r_r) and torch.equal(d3, d_r)
    assert torch.equal(same.obs, o_r[-1]) and torch.equal(same.rewards, r_r[-1]) and torch.equal(same.dones, d_r[-1])
    same_state(graph)
    same_state(same)
    assert graph.handover_timeouts == 0 and same.handover_timeouts == 0
    # host buffers
    obs_np, rew_np, dn_np = np.zeros((E, n, host.D), np.float32), np.zeros((E, n), np.float32), np.zeros((E, n), np.uint8)
    a_np = a.cpu().numpy()
    for t in range(T):
        host.step_host(a_np[t], obs_np, rew_np, dn_np)
        assert np.array_equal(obs_np, o_r[t].cpu().numpy()) and np.array_equal(rew_np, r_r[t].cpu().numpy()), t
        assert np.array_equal(dn_np, d_r[t].cpu().numpy()), t
    same_state(host)
    # the last observation only; vector stores instead of the bulk copy
    o4, r4, d4 = last.rollout(a, last_obs_only=True)
    o5, r5, d5 = vec.rollout(a)
    torch.cuda.synchronize()
    assert torch.equal(o4[0], o_r[-1]) and torch.equal(r4, r_r) and torch.equal(d4, d_r)
    assert torch.equal(o5, o_r) and torch.equal(r5, r_r) and torch.equal(d5, d_r)
    same_state(last)
    same_state(vec)
    for e in (ref, steps, graph, host, last, same, vec):
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. wrappers and episode statistics
# ---------------------------------------------------------------------------------------------------------------------
def _batched(**kw):
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    base = dict(num_envs=24, ep_time=0.4, neighbor_visible_num=6, quads_mode='static_same_goal', seed=4)
    base.update(kw)
    return QuadrotorEnvMultiBatched(**base)


@pytest.mark.gpu
@pytest.mark.parametrize('n', [12, 16])
def test_reward_shaping_statistics_at_swarm_sizes(n):
    """The wrapper kernel's cumulative reward terms, true_reward, action statistics (z_action*_mean / _std: reductions over
    16-lane groups, with idle lanes at N = 12) and latched episode statistics, against sums taken from a twin engine that
    steps the same envs without the wrappers."""
    import torch
    from quad_swarm_rl_b200.training import BatchedTrainingEnv
    from quad_swarm_rl_b200.wrappers import AnnealSchedule
    E = 24
    env, twin = _batched(num_agents=n), _batched(num_agents=n)
    scheme = dict(quad_rewards=dict(quadcol_bin=0.0, pos=1.0))
    w = BatchedTrainingEnv(env, reward_shaping_scheme=scheme, annealing=[AnnealSchedule('quadcol_bin', 5.0, 1000.0)],
                           stats_every=1 << 30)
    w.training_info['approx_total_training_steps'] = 400
    w.reset(); twin.reset()
    twin.engine.rew_coeff.update(scheme['quad_rewards'])
    raw_sum = torch.zeros((E, n, 8), device='cuda')
    acts = []
    g = torch.Generator(device='cuda'); g.manual_seed(1)
    for t in range(41):
        # per-drone offsets make the action statistics of every drone (and lane) different
        a = torch.rand((E * n, 4), device='cuda', generator=g) * 2 - 1
        a = (a * 0.5 + torch.linspace(-0.5, 0.5, n, device='cuda').repeat(E)[:, None]).contiguous()
        obs, rew, term, trunc, infos = w.step(a)
        o2, r2, t2, _, _ = twin.step(a, with_terms=True)
        assert torch.equal(obs, o2) and torch.equal(rew, r2) and torch.equal(term, t2)
        raw_sum += twin.engine.rew_terms
        acts.append(a.view(E, n, 4))
        if term.any():
            break
    assert t == 40 and term.all()
    fin = w.flush_stats()
    st = fin['episode_extra_stats']
    assert fin['episodes_finished'] == E
    np.testing.assert_allclose(st['rewraw_pos'], raw_sum[..., 0].mean().item(), rtol=1e-5)
    np.testing.assert_allclose(st['rew_proximity'], raw_sum[..., 6].mean().item(), rtol=1e-4, atol=1e-7)
    true_reward = raw_sum[..., 0] + 1000.0 * raw_sum[..., 5]
    assert torch.allclose(fin['true_reward'], true_reward, rtol=1e-5, atol=1e-3)
    np.testing.assert_allclose(st['rewraw_main'], true_reward.mean().item(), rtol=1e-4)
    A = torch.stack(acts)
    for k in range(4):
        np.testing.assert_allclose(st[f'z_action{k}_mean'], A[..., k].mean().item(), atol=1e-5)
        joint = A[..., k].permute(1, 0, 2).reshape(E, -1).std(dim=1, unbiased=False).mean().item()
        np.testing.assert_allclose(st[f'z_action{k}_std'], joint, rtol=1e-4)
    es, ags = twin.engine.episode_stats()
    np.testing.assert_allclose(st['num_collisions'], es[:, 0].float().mean().item(), rtol=1e-6)
    np.testing.assert_allclose(st['distance_to_goal_1s'], ags[..., 0].mean().item(), rtol=1e-5)
    env.close(); twin.close()


@pytest.mark.gpu
@pytest.mark.parametrize('n', [16, 24])
def test_episode_stats_latch_at_swarm_sizes(n):
    """The statistics latched at episode end (counters built from __popc of 16-bit and partly filled 32-bit ballots) equal
    the oracle's episode_extra_stats.  The device is teacher-forced after every step but keeps its own counters, so the
    increments of every step are the kernel's; only an env-step that decided a threshold closer than 3e-6 takes the oracle's
    counters.  Planted clusters and pillars make the drone and pillar collision counters non-zero.  Envs whose last step was
    such an env-step are left out; at least half of them are compared."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    kw = dict(num_agents=n, neighbor_visible_num=2, obs_repr=FLOOR, use_obstacles=True, use_downwash=True, ep_time=0.4)
    E = 6
    pair = Pair(E, kw, seed=900 + n, table_seed=901 + n)
    pair.reset()
    rs = np.random.RandomState(902)
    plant = _events_hook(n, every=20)
    eng = pair.engine

    def keeping_counters(fn, keep):
        """Teacher forcing (fn) that leaves the device's episode counters of the envs in `keep` as they were."""
        cnt = eng.get_state()['env_i32'][:, 4:4 + 11].clone()
        fn()
        st = eng.get_state()
        k = torch.as_tensor(keep, device=cnt.device)
        st['env_i32'][k, 4:4 + 11] = cnt[k]
        eng.set_state(st)

    stats, clean = None, np.ones(E, bool)
    for t in range(41):
        keeping_counters(lambda: plant(pair, t), np.ones(E, bool))
        d, o = pair.step(rs.uniform(-1, 1, (E, n, 4)).astype(np.float32))
        clean = np.array([oe.step_margin > 3e-6 for oe in pair.oracles])
        if o['dones'].any():
            stats = o['infos']
            break
        keeping_counters(pair.sync_device_from_oracle, clean)
    assert stats is not None and t == 40
    es, ags = eng.episode_stats()
    es, ags = es.cpu().numpy(), ags.cpu().numpy()
    print('compared envs', clean, 'latched', es[:, :11].tolist())
    assert clean.sum() >= E // 2
    nonzero = set()
    for e in np.where(clean)[0]:
        s0 = stats[e][0]['episode_extra_stats']
        for k, key in enumerate(L.ENV_STAT_KEYS[:11]):
            assert es[e, k] == s0[key], (e, key, es[e, k], s0[key])
            if es[e, k]:
                nonzero.add(key)
        for i in range(n):
            si = stats[e][i]['episode_extra_stats']
            np.testing.assert_allclose(ags[e, i, :3], [si['distance_to_goal_1s'], si['distance_to_goal_3s'],
                                                       si['distance_to_goal_5s']], rtol=1e-4)
    print('non-zero counters', sorted(nonzero))
    assert {'num_collisions', 'num_collisions_obst_quad'} <= nonzero, nonzero
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('n,pair_ids', [(16, (14, 15)), (24, (20, 21))])
def test_replay_stores_collisions_of_high_lanes(n, pair_ids):
    """A collision planted between drones 14 and 15 (N = 16) or 20 and 21 (N = 24), lanes the wrapper's col_any ballot must
    see, is stored as a replay event and replayed from the checkpoint 1.5 s before it (quad_experience_replay.py)."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    from quad_swarm_rl_b200.training import BatchedTrainingEnv
    E = 32
    env = _batched(num_envs=E, num_agents=n, ep_time=3.0, seed=7)
    w = BatchedTrainingEnv(env, replay_buffer_sample_prob=1.0, replay_always_active=True, stats_every=1 << 30)
    w.reset()
    g = torch.Generator(device='cuda'); g.manual_seed(2)
    hover = torch.zeros((E * n, 4), device='cuda') + 0.05
    planted = torch.arange(E, device='cuda') % 2 == 0
    i, j = pair_ids
    state_at, quiet = {}, None
    for t in range(301):
        if t == 200:
            st = env.engine.get_state()
            quiet = st['env_i32'][:, 4] == 0                   # no collision so far in this episode
            st['agent_f32'][planted, j, 0:3] = st['agent_f32'][planted, i, 0:3] + 0.01
            env.engine.set_state(st, env_mask=planted)
        obs, rew, term, trunc, infos = w.step(hover + 0.3 * (torch.rand((E * n, 4), device='cuda', generator=g) * 2 - 1))
        if t + 1 == 100:
            state_at = {k: v.clone() for k, v in env.engine.get_state().items() if v is not None}
            obs_at = obs.view(E, n, -1).clone()
        if term.any():
            break
    assert t == 300 and term.all()
    agg = env.engine.wrap_read(reset=False)
    assert agg[L.WA['EVENTS_STORED']] >= int(planted.sum())
    stc = env.engine.get_state()
    ticks = stc['env_i32'][:, 0]
    replayed = ticks > 0
    assert replayed[planted].all() and agg[L.WA['REPLAYED_EVENTS']] == int(replayed.sum())
    assert ((ticks[replayed] % 50) == 0).all()
    # envs whose only collision of the episode is the planted one (none before the plant, one in the latched episode count)
    # restart from the checkpoint 1.5 s before tick 201: tick 100
    es, _ = env.engine.episode_stats()
    only = quiet & (es[:, 0] == 1)
    ridx = torch.nonzero(planted & only).flatten()
    print('planted envs whose only collision is the planted one:', len(ridx), 'of', int(planted.sum()))
    assert len(ridx) >= int(planted.sum()) // 2, es[:, 0]
    assert (ticks[ridx] == 100).all()
    assert torch.equal(stc['agent_f32'][ridx], state_at['agent_f32'][ridx])
    assert torch.equal(obs.view(E, n, -1)[ridx], obs_at[ridx])
    env.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. CPU: the NP = 16 / 32 instantiations in the built library
# ---------------------------------------------------------------------------------------------------------------------
def _usage():
    """Resource usage of the step kernels {(path, NP, SPLIT, SCN, HO, DYN, NZ): {REG, STACK, LOCAL}} and of the NP = 16 / 32
    reset, pre-generation and wrapper kernels {(name, NP, other template arguments): ...} in the built library."""
    steps = kernel_resources(r'qs_step_kernel(_npy)?ILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE')
    other = kernel_resources(r'(qs_reset_kernel|qs_pregen_kernel|qs_wrap_kernel)ILi(16|32)E(\w*?)EEvN')
    return {('npy' if k[0] else 'default',) + k[1:]: v for k, v in steps.items()}, other


def test_np16_np32_step_instantiations_present_without_local_memory():
    """For NP in {16, 32}, every instantiation step_kernel<NP> (qs_step_select.cuh) can return, SPLIT / SCN / HO / DYN / NZ
    in its 14 reachable combinations, is in the library for the default and the numpy dynamics path (56 kernels), and none
    of them, nor the NP = 16 / 32 reset, pre-generation and wrapper kernels, uses local memory beyond its stack frame.
    Registers and stack frames are printed so that a change to them shows up in review."""
    steps, other = _usage()
    reach = set()
    for scn in (0, 1):
        for dyn in (0, 1):
            reach.add((0, scn, 0, dyn, 1))                     # NZ, with or without DYN
        reach.add((0, scn, 0, 1, 0))                           # DYN
        for split in (0, 1):
            for ho in (0, 1):
                reach.add((split, scn, ho, 0, 0))
    assert len(reach) == 14
    want = {(path, NP) + c for path in ('default', 'npy') for NP in (16, 32) for c in reach}
    assert len(want) == 56
    missing = want - set(steps)
    assert not missing, sorted(missing)
    for k in sorted(want):
        v = steps[k]
        print('qs_step_kernel%s<NP=%d, SPLIT=%d, SCN=%d, HO=%d, DYN=%d, NZ=%d>' % ((('_npy' if k[0] == 'npy' else ''),) + k[1:]),
              'REG', v['REG'], 'STACK', v['STACK'], 'LOCAL', v['LOCAL'])
        assert v['LOCAL'] == 0, (k, v)
    # qs_reset_kernel<NP, NZ, RND> (4 each), qs_pregen_kernel<NP>, qs_wrap_kernel<NP>
    assert sorted((name, NP) for name, NP, _ in other) == sorted(
        [(name, NP) for NP in (16, 32) for name in ['qs_reset_kernel'] * 4 + ['qs_pregen_kernel', 'qs_wrap_kernel']])
    for k, v in sorted(other.items()):
        print(k, 'REG', v['REG'], 'STACK', v['STACK'], 'LOCAL', v['LOCAL'])
        assert v['LOCAL'] == 0, (k, v)
