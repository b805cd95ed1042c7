"""Small workload for compute-sanitizer (memcheck / racecheck / synccheck / initcheck): both step-kernel shapes, both
launch-chaining modes, resets, contacts, every device-side scenario id, rollout, state and statistics kernels, the
pre-generated episode records, per-drone dynamics, obstacle randomisation and the training-wrapper kernel (replay on), the courier-warp hand-over of balanced grids, and the step kernels of the
control modes (position controller, [0, 1] actions) on both dynamics paths."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from quad_swarm_rl_b200.engine import QuadSwarmEngine
from tests.parity_util import make_tables

OBST = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True, use_downwash=True)
WALL = dict(num_agents=5, neighbor_visible_num=-1, obs_repr='xyz_vxyz_R_omega_wall')
WIDE = dict(num_agents=32, neighbor_visible_num=6)


def run(kw, E, scn, steps=14, chained=True):
    eng = QuadSwarmEngine(num_envs=E, seed=1, ep_time=0.12, device_scenario=scn, **kw)
    if scn is None:
        t = make_tables(np.random.RandomState(2), E, kw['num_agents'], eng.M, kw.get('use_obstacles', False), episodes=1, spread=0.05)[0]
        t['spawn'] = t['goals'].copy() if not kw.get('use_obstacles') else t['spawn']     # tight clusters -> contacts
        eng.set_next_episode(t['goals'], t['spawn'], t['obst'])
    eng.set_chained(chained)
    eng.reset()
    a = torch.rand((steps + 8, E, kw['num_agents'], 4), device='cuda') * 2 - 1
    for k in range(steps):
        eng.step(a[k].contiguous(), with_terms=True)
    eng.rollout(a[steps:].contiguous())
    st = eng.get_state(); eng.set_state(st); eng.episode_stats()
    assert eng.handover_timeouts == 0
    torch.cuda.synchronize()
    eng.close()


for split in ('0', '1'):
    os.environ['QS_SPLIT'] = split
    os.environ['QS_PDL'] = '3'                       # per-block hand-over between step grids
    for kw, E, scn in ((OBST, 13, None), (OBST, 13, 'mix'), (WALL, 7, None), (WIDE, 3, 'mix')):
        run(kw, E, scn, steps=10)
os.environ['QS_SPLIT'] = '0'
os.environ['QS_PDL'] = '2'                           # grid-wide wait
run(OBST, 13, 'o_static_same_goal', steps=10)
os.environ['QS_PDL'] = '3'
for scn in ('static_same_goal', 'static_diff_goal', 'dynamic_same_goal', 'dynamic_diff_goal', 'swap_goals', 'dynamic_formations',
            'ep_lissajous3D', 'swarm_vs_swarm', 'ep_rand_bezier'):
    run(dict(num_agents=8, neighbor_visible_num=3), 5, scn, steps=4, chained=False)


def run_extras(E=9, steps=40, chained=False, dynamics=True):
    """Round-2 kernels: dynamics rows latched at reset, obstacle density / size per episode, wrapper epilogue with replay."""
    from quad_swarm_rl_b200 import quad_models as qm
    kw = dict(OBST, obst_density=0.8)
    eng = QuadSwarmEngine(num_envs=E, seed=3, ep_time=0.1, device_scenario='o_random', **kw)
    eng.set_obstacle_randomization([0.2, 0.8], [0.6, 0.85])
    rows = np.stack([np.stack([qm.constants_row(qm.crazyflie_params()) for _ in range(8)]) for _ in range(E)])
    if dynamics:
        eng.set_dynamics(rows.astype(np.float32), at_next_reset=True)
    eng.wrap_enable(use_replay=True, replay_buffer_size=4, replay_prob=0.75, replay_always_active=True)
    eng.set_chained(chained)
    eng.reset()
    a = torch.rand((steps, E, 8, 4), device='cuda') * 2 - 1
    for k in range(steps):
        eng.wrap_step(a[k].contiguous())
    eng.wrap_read()
    torch.cuda.synchronize()
    eng.close()


run_extras()
os.environ.pop('QS_PDL', None)                       # default launch rule: balanced CTAs with a courier warp (>= 2 warps per SM)
run(OBST, 600, 'o_random', steps=8)
run(dict(num_agents=8, neighbor_visible_num=6), 600, 'swap_goals', steps=8)
run_extras(E=600, steps=30, chained=True, dynamics=False)      # wrapped control steps, block-chained with the wrapper kernel
# the control modes of qs_set_control on both dynamics paths (qs_step_pc.cu, qs_step_pc_npy.cu)
for ctl in (dict(raw_control=False), dict(raw_control_zero_middle=False)):
    for use_numba in (True, False):
        run(dict(OBST, use_numba=use_numba, **ctl), 13, 'o_random', steps=10)
        run(dict(num_agents=8, neighbor_visible_num=6, use_numba=use_numba, **ctl), 600, 'swap_goals', steps=8)
print('sanitize workload done')
