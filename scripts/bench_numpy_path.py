"""Cost of the numpy dynamics path (use_numba=False, qs_set_numpy_dynamics) on the benchmark workloads c2 and c3.

Times each workload on the njit path (the default) and on the numpy path, with bench.py's method (chained step launches in
CUDA graphs over rings larger than L2, staggered episode ticks, median step time over the blocks), in alternating rounds so
that the spread between rounds shows beside the difference.  The numpy path runs its own kernel instantiations; only their
floor-contact code differs.  Prints one JSON line with the card name, its power limit and SM clock.
Usage: python scripts/bench_numpy_path.py [--steps K] [--warmup W] [--rounds R] [--configs c2,c3]
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

VARIANTS = {'numba': True, 'numpy': False}       # value: use_numba


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=2048)
    ap.add_argument('--warmup', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--configs', default='c2,c3')
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    res = {}
    for r in range(a.rounds):
        for cfg_name in a.configs.split(','):
            for var, use_numba in VARIANTS.items():
                name = f'{cfg_name}_{var}'
                cfg = dict(bench.CONFIGS[cfg_name])
                cfg['kw'] = dict(cfg['kw'], use_numba=use_numba)
                bench.CONFIGS[name] = cfg
                args = argparse.Namespace(envs=0, config=name, no_graph=False, lockstep=False, host_tables=False, seed=0,
                                          ep_time=15.0, warmup=a.warmup)
                m = bench.measure_workload(torch, None, name, args, 0, 0, 1, a.steps)
                m['runner'].close()
                res.setdefault(name, []).append(m['us_per_step'])
                torch.cuda.empty_cache()
    out = dict(gpu_info(), steps=a.steps, rounds=a.rounds, us_per_step={})
    for cfg_name in a.configs.split(','):
        base = np.median(res[f'{cfg_name}_numba'])
        for var in VARIANTS:
            v = res[f'{cfg_name}_{var}']
            out['us_per_step'][f'{cfg_name}_{var}'] = dict(median=float(np.median(v)), rounds=[round(x, 3) for x in v],
                                                           spread=float(np.max(v) - np.min(v)), vs_numba=float(np.median(v) / base))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
