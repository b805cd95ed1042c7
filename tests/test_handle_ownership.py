"""Every buffer of a handle has one owner (csrc/quadswarm.cu): the device and page-locked host buffers are allocated only
by dev_alloc / host_alloc, which record them in the handle, and freed only by dev_release / release_handle, so that a
failed qs_create, qs_wrap_enable or qs_set_dynamics leaks nothing.  On the GPU: handles whose options allocate and free
buffers before the first reset step exactly like handles given the final options once."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'quad_swarm_rl_b200', 'csrc', 'quadswarm.cu')


def _callers(call):
    """Names of the top-level definitions of quadswarm.cu whose bodies contain a call matching `call` ('#define' for a
    macro, None outside any function)."""
    text = open(SRC).read()
    # comments and literals in one left-to-right pass (a comment may hold a quote, a string a '//')
    text = re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"|\'(?:\\.|[^\'\\\n])*\'',
                  lambda m: '""' if m.group(0)[0] in '"\'' else ' ', text, flags=re.S)
    call_re = re.compile(r'\b(?:' + call + r')\s*\(')
    directive = re.compile(r'^[ \t]*#(?:[^\n]*\\\n)*[^\n]*', flags=re.M)
    owners = ['#define' for d in directive.findall(text) if call_re.search(d)]
    text = directive.sub(' ', text)
    depth, head, name = 0, 0, None
    for m in re.finditer(r'[{};]|' + call_re.pattern, text):
        tok = m.group(0)
        if tok == '{':
            if depth == 0:
                sig = re.search(r'(\w+)\s*\(', text[head:m.start()])
                name = sig.group(1) if sig else None
            depth += 1
        elif tok in ('}', ';'):
            if tok == '}':
                depth -= 1
            if depth == 0:               # the next top-level definition starts after this
                head, name = m.end(), None
        else:
            owners.append(name)
    return owners


def test_only_the_allocation_helpers_allocate():
    assert set(_callers(r'cudaMalloc\w*|cudaHostAlloc')) == {'dev_alloc', 'host_alloc'}


def test_only_the_teardown_frees():
    assert set(_callers(r'cudaFree\w*')) == {'dev_release', 'release_handle'}


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
KW = dict(num_agents=8, neighbor_visible_num=2, ep_time=0.3, use_obstacles=True, use_downwash=True,
          obs_repr='xyz_vxyz_R_omega_floor', sense_noise=dict(gyro_norm_std=0.1, quat_norm_std=0.01))


def _dyn_rows(E, N):
    """Crazyflies and DefaultQuads, alternating drone by drone."""
    from quad_swarm_rl_b200 import quad_models as qm
    cf, dq = qm.constants_row(qm.crazyflie_params()), qm.constants_row(qm.defaultquad_params())
    return np.stack([np.stack([cf if (e + i) % 2 else dq for i in range(N)]) for e in range(E)]).astype(np.float32)


@pytest.mark.gpu
def test_handles_reallocating_before_the_first_reset_step_like_fresh_ones():
    """The gyro-bias model switched off and on again before the first reset (its buffer freed and allocated anew), then
    wrappers with replay and per-drone dynamics: each such handle steps bit-identically to one given those options once."""
    import ctypes
    import torch
    from quad_swarm_rl_b200 import _lib as L
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    E, T, N = 12, 45, KW['num_agents']
    rows = _dyn_rows(E, N)
    for seed in range(3):
        toggled, fresh = (QuadSwarmEngine(num_envs=E, seed=seed, device_scenario='o_random', **KW) for _ in range(2))
        assert toggled.gyro_model
        on = L.QsSensorNoise(**toggled.sense_noise)
        off = L.QsSensorNoise(**dict(toggled.sense_noise, gyro_norm_std=0.0))
        for sn in (off, on):
            L.check(toggled.lib.qs_set_sensor_noise(toggled.h, ctypes.byref(sn)))
        for e in (toggled, fresh):
            e.set_dynamics(rows)
            e.wrap_enable(use_replay=True, replay_buffer_size=4, replay_prob=0.9, replay_always_active=True)
            e.reset()
        g = torch.Generator(device='cuda')
        g.manual_seed(seed)
        a = (torch.rand((T, E, N, 4), device='cuda', generator=g) * 2 - 1).contiguous()
        dones = 0
        for t in range(T):
            o1, r1, d1 = (x.clone() for x in toggled.wrap_step(a[t]))
            o2, r2, d2 = fresh.wrap_step(a[t])
            assert torch.equal(o1, o2) and torch.equal(r1, r2) and torch.equal(d1, d2), (seed, t)
            dones += int(d2.sum())
        assert dones > 0
        s1, s2 = toggled.get_state(), fresh.get_state()
        for k in ('agent_f32', 'agent_u32', 'env_i32', 'gyro_bias'):
            assert torch.equal(s1[k], s2[k]), (seed, k)
        assert float(s1['gyro_bias'].abs().max()) > 0
        # the aggregate's sums are float atomics: their order, and so their last bits, differ from run to run
        g1, g2 = toggled.wrap_read(), fresh.wrap_read()
        np.testing.assert_allclose(g1, g2, rtol=1e-5, atol=1e-6)
        assert g1[L.WA['EPISODES_TOTAL']] == g2[L.WA['EPISODES_TOTAL']] > 0
        toggled.close()
        fresh.close()
