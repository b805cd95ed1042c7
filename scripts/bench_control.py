"""Cost of the control modes of qs_set_control on the benchmark workloads c2 and c3: RawControl with actions in [-1, 1] (the
default, `raw`), RawControl with actions in [0, 1] (`raw_unit`, raw_control_zero_middle=False) and the position controller
(`position`, raw_control=False).

Times each workload in each mode with bench.py's method (chained step launches in CUDA graphs over rings larger than L2,
staggered episode ticks, median step time over the blocks), in alternating rounds so that the spread between rounds shows
beside the difference.  The two other modes run their own kernel instantiations, in the single-warp shape with the grid-wide
wait only, so part of their cost is that shape's, not the controller's.  Prints one JSON line with the card name, its power
limit and SM clock.
Usage: python scripts/bench_control.py [--steps K] [--warmup W] [--rounds R] [--configs c2,c3]
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

VARIANTS = {'raw': {}, 'raw_unit': dict(raw_control_zero_middle=False), 'position': dict(raw_control=False)}


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
            for var, ctl in VARIANTS.items():
                name = f'{cfg_name}_{var}'
                cfg = dict(bench.CONFIGS[cfg_name])
                cfg['kw'] = dict(cfg['kw'], **ctl)
                bench.CONFIGS[name] = cfg
                args = argparse.Namespace(envs=0, config=name, no_graph=False, lockstep=False, host_tables=False, seed=0,
                                          ep_time=15.0, warmup=a.warmup)
                m = bench.measure_workload(torch, None, name, args, 0, 0, 1, a.steps)
                m['runner'].close()
                res.setdefault(name, []).append(m['us_per_step'])
                torch.cuda.empty_cache()
    out = dict(gpu_info(), steps=a.steps, rounds=a.rounds, us_per_step={})
    for cfg_name in a.configs.split(','):
        base = np.median(res[f'{cfg_name}_raw'])
        for var in VARIANTS:
            v = res[f'{cfg_name}_{var}']
            out['us_per_step'][f'{cfg_name}_{var}'] = dict(median=float(np.median(v)), rounds=[round(x, 3) for x in v],
                                                           spread=float(np.max(v) - np.min(v)), vs_raw=float(np.median(v) / base))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
