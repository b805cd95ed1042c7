"""Cost of per-drone dynamics sampled on the device (qs_set_dynamics_sampler) on the c3 workload, and what it saves at
construction.

Step time: bench.py's method (chained step launches in CUDA graphs over rings larger than L2, staggered episode ticks, median
step time over the blocks), in alternating rounds, for
  * `default`:    the Crazyflie constants compiled into the kernels (no per-drone rows), for reference;
  * `fixed`:      per-drone rows (Crazyflie + RelativeSampler(0.1, normal)) sampled once at construction, never again;
  * `every1`:     the same sampler, every drone resampled at each of its env's resets (dynamics_randomize_every=1);
  * `randomquad`: RandomQuad airframes resampled at each reset.
With ep_time = 15 s and staggered episodes, about E / 1501 envs reset per step.
Construction: a 4096 x 8 QuadrotorEnvMultiBatched with RandomQuad and dynamics_randomize_every=1, host pipeline
(quad_models.DynamicsSource per drone) vs device_dynamics=True, wall time to the end of the constructor plus a device
synchronisation.  Prints one JSON line with the card name, its power limit and SM clock.
Usage: python scripts/bench_device_dynamics.py [--steps K] [--warmup W] [--rounds R] [--no-construction]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

import bench  # noqa: E402
from bench_sensor_noise import gpu_info  # noqa: E402
from quad_swarm_rl_b200.quad_models import dynamics_sampler_spec  # noqa: E402

REL = {'class': 'RelativeSampler', 'noise_ratio': 0.1, 'sampler': 'normal'}
VARIANTS = {'default': {},
            'fixed': dict(dynamics_sampler=dynamics_sampler_spec('Crazyflie', None, REL), dynamics_randomize_every=None),
            'every1': dict(dynamics_sampler=dynamics_sampler_spec('Crazyflie', None, REL), dynamics_randomize_every=1),
            'randomquad': dict(dynamics_sampler=dynamics_sampler_spec('RandomQuad'), dynamics_randomize_every=1)}


def construction_seconds(torch, device_dynamics):
    from quad_swarm_rl_b200.env import QuadrotorEnvMultiBatched
    kw = dict(bench.CONFIGS['c3']['kw'])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    env = QuadrotorEnvMultiBatched(bench.CONFIGS['c3']['E'], quads_mode='o_random', seed=0, dynamics_params='RandomQuad',
                                   dynamics_randomize_every=1, device_dynamics=device_dynamics, **kw)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    env.engine.close()
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=2048)
    ap.add_argument('--warmup', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--no-construction', action='store_true')
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    res = {}
    for r in range(a.rounds):
        for var, extra in VARIANTS.items():
            name = f'c3_{var}'
            cfg = dict(bench.CONFIGS['c3'])
            cfg['kw'] = dict(cfg['kw'], **extra)
            bench.CONFIGS[name] = cfg
            args = argparse.Namespace(envs=0, config=name, no_graph=False, lockstep=False, host_tables=False, seed=0,
                                      ep_time=15.0, warmup=a.warmup)
            m = bench.measure_workload(torch, None, name, args, 0, 0, 1, a.steps)
            m['runner'].close()
            res.setdefault(var, []).append(m['us_per_step'])
            torch.cuda.empty_cache()
    out = dict(gpu_info(), steps=a.steps, rounds=a.rounds, us_per_step={})
    base = np.median(res['default'])
    for var in VARIANTS:
        v = res[var]
        out['us_per_step'][var] = dict(median=float(np.median(v)), rounds=[round(x, 3) for x in v],
                                       spread=float(np.max(v) - np.min(v)), vs_default=float(np.median(v) / base))
    if not a.no_construction:
        out['construction_s'] = dict(device=construction_seconds(torch, True), host=construction_seconds(torch, False))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
