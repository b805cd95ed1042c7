"""Timeline of the step kernel's phases (debug build tune/libquadswarm_tl.so, -DQS_TIMELINE): %globaltimer stamps of
warp 0 of every block at 8 points, for the 20 chained launches of a CUDA graph.  Usage (GPU box):
    QS_LIB=$PWD/tune/libquadswarm_tl.so python scripts/gpu_timeline.py [c3|c2|c4] [stagger]"""
import ctypes as C
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from quad_swarm_rl_b200 import _lib as L
from quad_swarm_rl_b200.engine import QuadSwarmEngine

name = sys.argv[1] if len(sys.argv) > 1 else 'c3'
stagger = len(sys.argv) > 2 and sys.argv[2] == 'stagger'
cfg = bench.CONFIGS[name]
E, kw = cfg['E'], cfg['kw']
N = kw['num_agents']
eng = QuadSwarmEngine(num_envs=E, seed=0, rew_coeff=cfg['rew'], device_scenario=cfg['mode'], **kw)
eng.reset()
if stagger:
    st = eng.get_state()
    st['env_i32'][:, 0] = torch.randint(0, eng.ep_len + 1, (E,), device='cuda', dtype=torch.int32)
    eng.set_state(st)
eng.set_chained(True)
K = 20
act = (torch.rand((K, E, N, 4), device='cuda') * 2 - 1).contiguous()
obs = torch.empty((K, E, N, eng.D), device='cuda'); rew = torch.empty((K, E, N), device='cuda')
dn = torch.empty((K, E, N), dtype=torch.uint8, device='cuda')
s = torch.cuda.Stream()
lib = L.load()
lib.qs_debug_timeline.argtypes = [C.c_void_p, C.c_void_p]
lib.qs_debug_timeline_rewind.argtypes = [C.c_void_p]
with torch.cuda.stream(s):
    for t in range(3):
        eng.step(act[t], obs_out=obs[t], rewards_out=rew[t], dones_out=dn[t])
    s.synchronize()
    lib.qs_debug_timeline_rewind(eng.h)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for t in range(K):
            eng.step(act[t], obs_out=obs[t], rewards_out=rew[t], dones_out=dn[t])
    for _ in range(30):
        g.replay()
    s.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(50):
        g.replay()
    e1.record(s)
    s.synchronize()
print(f'{name} stagger={stagger} PDL={os.environ.get("QS_PDL")}: {e0.elapsed_time(e1) / 50 / K * 1e3:.2f} us/step (instrumented build)')
buf = np.zeros((64, 4096, 16), np.uint64)
L.check(lib.qs_debug_timeline(eng.h, buf.ctypes.data_as(C.c_void_p)))
tl = buf[:K].astype(np.int64)
nb = int((tl[0, :, 0] > 0).sum())
smid = tl[:, :nb, 8].copy()
rst = tl[:, :nb, 9:12].copy()
tl = tl[:, :nb, :8]
t0 = tl[:, :, 0].min()
tl = (tl - t0) / 1e3          # us
names = ['entry', 'waited', 'loaded', 'dyn', 'pairs', 'obs', 'emit', 'exit']
print(f'blocks {nb}; per step: median over blocks of (stamp - first entry of the step), then the step-to-step spacing')
for k in range(2, K):
    ent = tl[k, :, 0].min()
    row = ' '.join(f'{names[j]}={np.median(tl[k, :, j]) - ent:6.2f}' for j in range(1, 8))
    print(f'step {k:2d}: first entry at {ent:8.2f} (+{ent - tl[k - 1, :, 0].min():5.2f} after the previous one); last exit +{tl[k, :, 7].max() - ent:6.2f}; '
          f'entry spread {tl[k, :, 0].max() - ent:5.2f} | {row}')
d = tl[2:]
ph = [np.median(d[:, :, j] - d[:, :, j - 1]) for j in range(1, 8)]
print('median phase durations (us): ' + ' '.join(f'{names[j]}-{names[j - 1]}={ph[j - 1]:.2f}' for j in range(1, 8)))
print('p95 phase durations (us):    ' + ' '.join(f'{np.percentile(d[:, :, j] - d[:, :, j - 1], 95):.2f}' for j in range(1, 8)))
print('max block duration entry->exit per step (us):', np.round((d[:, :, 7] - d[:, :, 0]).max(axis=1), 2))
# blocks by how many blocks share their SM in that step
dur = d[:, :, 7] - d[:, :, 1]
sm = smid[2:]
for k in (5, 12):
    cnt = np.bincount(sm[k], minlength=160)
    per = cnt[sm[k]]
    print(f'step {k + 2}: blocks per SM histogram {np.bincount(cnt)[1:].tolist()} | median waited->exit by #blocks on the SM: ' +
          ' '.join(f'{c}:{np.median(dur[k][per == c]):.2f}(n={int((per == c).sum())})' for c in np.unique(per)))
print('waited->exit percentiles (us) 50/90/99/max:', np.round(np.percentile(dur, [50, 90, 99, 100]), 2))
# SM time by what the SM holds, between the first entry of the 2nd and the last exit of the next-to-last recorded step:
# no CTA, one CTA that still waits for its predecessor (entry -> waited), one working CTA, two or more CTAs
w0, w1 = d[1, :, 0].min(), d[-2, :, 7].max()
share = np.zeros(4)
for s_ in np.unique(sm):
    m = sm == s_
    ent, wt, ex = d[:, :, 0][m], d[:, :, 1][m], d[:, :, 7][m]
    pts = np.unique(np.clip(np.concatenate([ent, wt, ex, [w0, w1]]), w0, w1))
    mid, ln = (pts[:-1] + pts[1:]) / 2, np.diff(pts)
    res = ((ent[None] <= mid[:, None]) & (ex[None] > mid[:, None])).sum(1)
    waiting = ((ent[None] <= mid[:, None]) & (wt[None] > mid[:, None])).sum(1)
    share += [ln[res == 0].sum(), ln[(res == 1) & (waiting == 1)].sum(), ln[(res == 1) & (waiting == 0)].sum(), ln[res >= 2].sum()]
share /= share.sum()
print('SM time shares: idle {:.3f} | one CTA, waiting for its predecessor {:.3f} | one CTA, working {:.3f} | two or more CTAs {:.3f}'.format(*share))
slow = np.argsort(dur[5])[-8:]
print('slowest blocks of step 7:', [(int(b), int(sm[5][b]), round(float(dur[5][b]), 2), np.round(np.diff(d[5, b, 1:8]), 2).tolist()) for b in slow])
# reset path of the blocks that had one (stamps 9..11: start of the episode-end branch, after reset_env, after the redraw)
for k in range(2, K):
    for b in range(nb):
        if rst[k, b, 0] > 0 and rst[k, b, 2] >= rst[k, b, 0] and buf[k, b, 4] > 0:
            t4, t5 = int(buf[k, b, 4]), int(buf[k, b, 5])
            if t4 <= rst[k, b, 0] <= t5:
                print(f'reset in step {k} block {b}: pairs->branch {(rst[k, b, 0] - t4) / 1e3:.2f} us, stats+reset_env {(rst[k, b, 1] - rst[k, b, 0]) / 1e3:.2f}, '
                      f'noise+dmin {(rst[k, b, 2] - rst[k, b, 1]) / 1e3:.2f}, rest to obs {(t5 - rst[k, b, 2]) / 1e3:.2f}')
                break
print('globaltimer resolution check: distinct diffs', np.unique(np.diff(np.sort(tl[5].ravel())))[:6])
eng.close()
