"""Cost of a per-episode pillar size on host tables (qs_set_next_obstacle_radius) on the c3 workload.

Times c3 (8 drones x 4096 envs, o_random pillars, downwash) with its episodes taken from host tables (bench.py
--host-tables), two ways — the construction radius for every episode, and a radius per env (sizes 0.3 / 0.4 / 0.5 / 0.6,
latched at every reset) — with bench.py's method (chained step launches in CUDA graphs over rings larger than L2, median
step time over the blocks), in alternating rounds so that the spread between rounds shows beside the difference.  Prints
one JSON line with the card name and its power limit.
Usage: python scripts/bench_obstacle_size.py [--steps K] [--warmup W] [--rounds R]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from bench_sensor_noise import gpu_info  # noqa: E402
from quad_swarm_rl_b200.engine import QuadSwarmEngine  # noqa: E402

SIZES = (0.3, 0.4, 0.5, 0.6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=2048)
    ap.add_argument('--warmup', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    plain_set_next_episode = QuadSwarmEngine.set_next_episode

    def with_radii(self, goals, spawn=None, obst_xy=None, env_mask=None):
        # the bench runner uploads its tables once, right before its reset: the radii go with them
        plain_set_next_episode(self, goals, spawn, obst_xy, env_mask)
        self.set_next_obstacle_radius(np.array([SIZES[e % len(SIZES)] / 2.0 for e in range(self.E)], np.float32))

    res = {}
    for r in range(a.rounds):
        for var in ('fixed', 'per_episode'):
            QuadSwarmEngine.set_next_episode = with_radii if var == 'per_episode' else plain_set_next_episode
            args = argparse.Namespace(envs=0, config='c3', no_graph=False, lockstep=False, host_tables=True, seed=0,
                                      ep_time=15.0, warmup=a.warmup)
            m = bench.measure_workload(torch, None, 'c3', args, 0, 0, 1, a.steps)
            m['runner'].close()
            res.setdefault(var, []).append(m['us_per_step'])
            torch.cuda.empty_cache()
    QuadSwarmEngine.set_next_episode = plain_set_next_episode
    base = np.median(res['fixed'])
    out = dict(gpu_info(), workload='c3 host tables', steps=a.steps, rounds=a.rounds,
               us_per_step={var: dict(median=float(np.median(v)), rounds=[round(x, 3) for x in v],
                                      vs_fixed=float(np.median(v) / base)) for var, v in res.items()})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
