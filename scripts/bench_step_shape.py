"""Step time of two builds of the library side by side: the launch shape of the chained step grid (plan_step) and the
register budget of the step kernel decide how many CTAs of consecutive steps an SM holds at once.

Each build is loaded through QS_LIB in a process of its own, and the builds alternate over the rounds, so that the spread
between rounds shows beside the difference.  Every process times, with bench.py's method (chained step launches in CUDA
graphs over rings larger than L2, staggered episode ticks, median step time over the blocks): c3, c2, c4, c5, c3 with the
training wrappers (qs_wrap_step), the c3 rollout (64 steps per launch) and c3 with 4x the envs.  Prints one JSON line with
the card name, its power limit and SM clock.
Usage: python scripts/bench_step_shape.py old=PATH new=PATH [--steps K] [--warmup W] [--rounds R]
       A build may carry environment settings for its processes: name=PATH:VAR=VALUE[:VAR=VALUE...]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

CASES = ('c3', 'c2', 'c4', 'c5', 'c3_wrapped', 'c3_rollout', 'c3_x4')


def worker(steps, warmup):
    """One process, one build (QS_LIB): every case once, microseconds per control step."""
    import torch
    import bench
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    if not torch.cuda.is_available():
        raise SystemExit('needs a CUDA device')
    out = {}

    def args_for(name, envs=0):
        return argparse.Namespace(envs=envs, config=name, no_graph=False, lockstep=False, host_tables=False, seed=0,
                                  ep_time=15.0, warmup=warmup)

    for case in CASES:
        name = case.split('_')[0]
        cfg = bench.CONFIGS[name]
        if case == 'c3_rollout':
            E, N, kw = cfg['E'], cfg['kw']['num_agents'], cfg['kw']
            T = 64
            eng = QuadSwarmEngine(num_envs=E, seed=0, device=0, rew_coeff=cfg['rew'], ep_time=15.0, device_scenario=cfg['mode'], **kw)
            eng.reset()
            g = torch.Generator(device='cuda'); g.manual_seed(3)
            acts = (torch.rand((T, E, N, 4), device='cuda', generator=g) * 2 - 1).contiguous()
            o = torch.empty((T, E, N, eng.D), device='cuda'); r = torch.empty((T, E, N), device='cuda')
            d = torch.empty((T, E, N), dtype=torch.uint8, device='cuda')
            for _ in range(2):
                eng.rollout(acts, obs_out=o, rewards_out=r, dones_out=d)
            reps = max(4, steps // T)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                eng.rollout(acts, obs_out=o, rewards_out=r, dones_out=d)
            e1.record()
            torch.cuda.synchronize()
            out[case] = e0.elapsed_time(e1) * 1e3 / (reps * T)
            eng.close()
            del o, r, d, acts
        else:
            envs = 4 * cfg['E'] if case == 'c3_x4' else 0
            m = bench.measure_workload(torch, None, name, args_for(name, envs), 0, 0, 1, steps, wrapped=(case == 'c3_wrapped'))
            timeouts = m['runner'].eng.handover_timeouts
            m['runner'].close()
            if timeouts:
                raise RuntimeError(f'{case}: a per-block hand-over timed out')
            out[case] = m['us_per_step']
        torch.cuda.empty_cache()
    print('RESULT ' + json.dumps(out), flush=True)


def parse_build(spec):
    name, rest = spec.split('=', 1)
    parts = rest.split(':')
    env = dict(kv.split('=', 1) for kv in parts[1:])
    return name, os.path.abspath(parts[0]), env


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('builds', nargs='*', help='name=PATH[:VAR=VALUE...] (default: old / new are required)')
    ap.add_argument('--steps', type=int, default=2048)
    ap.add_argument('--warmup', type=int, default=256)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.steps, a.warmup)
        return
    if len(a.builds) < 2:
        raise SystemExit('give at least two builds, e.g. old=PATH new=PATH')
    from bench_sensor_noise import gpu_info
    builds = [parse_build(b) for b in a.builds]
    for _, path, _ in builds:
        if not os.path.exists(path):
            raise SystemExit(f'{path} does not exist')
    res = {name: {c: [] for c in CASES} for name, _, _ in builds}
    for r in range(a.rounds):
        order = builds if r % 2 == 0 else builds[::-1]
        for name, path, env in order:
            penv = dict(os.environ, QS_LIB=path, **env)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', '--steps', str(a.steps), '--warmup', str(a.warmup)],
                               env=penv, capture_output=True, text=True, cwd=ROOT)
            line = [ln for ln in p.stdout.splitlines() if ln.startswith('RESULT ')]
            if p.returncode != 0 or not line:
                raise SystemExit(f'{name} round {r} failed:\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}')
            for c, v in json.loads(line[-1][7:]).items():
                res[name][c].append(v)
            print(f'round {r} {name}: ' + ' '.join(f'{c}={v[-1]:.2f}' for c, v in res[name].items()), file=sys.stderr, flush=True)
    ref = builds[0][0]
    out = dict(gpu_info(), steps=a.steps, rounds=a.rounds, builds={n: p for n, p, _ in builds}, us_per_step={})
    for name, _, env in builds:
        out['us_per_step'][name] = {}
        for c in CASES:
            v = np.array(res[name][c])
            med = float(np.median(v))
            out['us_per_step'][name][c] = dict(median=round(med, 3), spread=round(float(v.max() - v.min()), 3),
                                               rounds=[round(x, 2) for x in v],
                                               vs_first=round(med / float(np.median(res[ref][c])), 4))
        if env:
            out['us_per_step'][name]['env'] = env
    print(json.dumps(out))


if __name__ == '__main__':
    main()
