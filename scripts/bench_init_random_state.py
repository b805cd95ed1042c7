"""Cost of random initial states (init_random_state=True, qs_set_init_random_state) on the benchmark workloads c2 and c3.

Times each workload with the option off and on, with bench.py's method (chained step launches in CUDA graphs over rings
larger than L2, staggered episode ticks, median step time over the blocks), in alternating rounds so that the spread between
rounds shows beside the difference.  The option only acts at a reset: with 15 s episodes c3 resets about 4096 / 1500 ~ 3
envs per step.  Prints one JSON line with the card name, its power limit and SM clock.
Usage: python scripts/bench_init_random_state.py [--steps K] [--warmup W] [--rounds R]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402
from bench_sensor_noise import gpu_info  # noqa: E402

VARIANTS = {'off': False, 'on': True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=2048)
    ap.add_argument('--warmup', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--configs', default='c2,c3')
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    res = {}
    for r in range(a.rounds):
        for cfg_name in a.configs.split(','):
            for var, on in VARIANTS.items():
                name = f'{cfg_name}_{var}'
                cfg = dict(bench.CONFIGS[cfg_name])
                cfg['kw'] = dict(cfg['kw'], init_random_state=on)
                bench.CONFIGS[name] = cfg
                args = argparse.Namespace(envs=0, config=name, no_graph=False, lockstep=False, host_tables=False, seed=0,
                                          ep_time=15.0, warmup=a.warmup)
                m = bench.measure_workload(torch, None, name, args, 0, 0, 1, a.steps)
                m['runner'].close()
                res.setdefault(name, []).append(m['us_per_step'])
                torch.cuda.empty_cache()
    out = dict(gpu_info(), steps=a.steps, rounds=a.rounds, us_per_step={})
    for cfg_name in a.configs.split(','):
        base = np.median(res[f'{cfg_name}_off'])
        for var in VARIANTS:
            v = res[f'{cfg_name}_{var}']
            out['us_per_step'][f'{cfg_name}_{var}'] = dict(median=float(np.median(v)), rounds=[round(x, 2) for x in v],
                                                           vs_off=float(np.median(v) / base))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
