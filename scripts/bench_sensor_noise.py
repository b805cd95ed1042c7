"""Cost of the custom sensor-noise model (qs_set_sensor_noise) on the benchmark workloads c2 and c3.

Times each workload three ways — sense_noise='default', a custom dict without the gyro bias model, and one with it — with
bench.py's method (chained step launches in CUDA graphs over rings larger than L2, median step time over the blocks), in
alternating rounds so that the spread between rounds shows beside the differences.  Prints one JSON line with the card name
and its power limit.  Usage: python scripts/bench_sensor_noise.py [--steps K] [--warmup W] [--rounds R]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

VARIANTS = {
    'default': 'default',
    'custom': dict(pos_unif_range=0.01, vel_unif_range=0.02, quat_norm_std=0.02, quat_unif_range=0.01),
    'custom_gyro_bias': dict(pos_unif_range=0.01, vel_unif_range=0.02, quat_norm_std=0.02, quat_unif_range=0.01,
                             gyro_norm_std=1.0),
}


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(',')]
        return dict(gpu=name, power_limit=power, sm_max_clock=clk)
    except Exception as e:          # the numbers stay valid; only the label is missing
        return dict(gpu=f'unknown ({e})')


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
            for var, noise in VARIANTS.items():
                name = f'{cfg_name}_{var}'
                cfg = dict(bench.CONFIGS[cfg_name])
                cfg['kw'] = dict(cfg['kw'], sense_noise=noise)
                bench.CONFIGS[name] = cfg
                args = argparse.Namespace(envs=0, config=name, no_graph=False, lockstep=False, host_tables=False, seed=0,
                                          ep_time=15.0, warmup=a.warmup)
                m = bench.measure_workload(torch, None, name, args, 0, 0, 1, a.steps)
                m['runner'].close()
                res.setdefault(name, []).append(m['us_per_step'])
                torch.cuda.empty_cache()
    out = dict(gpu_info(), steps=a.steps, rounds=a.rounds, us_per_step={})
    for cfg_name in a.configs.split(','):
        base = np.median(res[f'{cfg_name}_default'])
        for var in VARIANTS:
            v = res[f'{cfg_name}_{var}']
            out['us_per_step'][f'{cfg_name}_{var}'] = dict(median=float(np.median(v)), rounds=[round(x, 2) for x in v],
                                                           vs_default=float(np.median(v) / base))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
