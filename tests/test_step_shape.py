"""Launch shape of chained step grids with the courier warp (plan_step, quadswarm.cu): the instantiations that can carry the
courier are capped at 128 registers, so that two CTAs of consecutive steps fit on one SM, and the c3-sized chain takes a
shape whose CTAs do.  CPU: the register budget of the built library.  GPU: chained step grids in that shape give, bit for
bit, what one rollout gives (staggered episode ticks, so that auto-resets and pre-generated episode records occur), also
when every step writes the same output arrays, and a wrapped chain gives what synchronised wrapped steps give."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.environ.get('QS_LIB') or os.path.join(ROOT, 'quad_swarm_rl_b200', 'libquadswarm.so')
C3 = dict(num_agents=8, neighbor_visible_num=2, obs_repr='xyz_vxyz_R_omega_floor', use_obstacles=True, use_downwash=True)
C3_REW = dict(quadcol_bin=5.0, quadcol_bin_smooth_max=4.0, quadcol_bin_obst=5.0)
# qs_step_kernel<NP, SPLIT, SCN, HO, DYN, NZ>
KERNEL = re.compile(r'qs_step_kernelILi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])ELb([01])EE')


def _resource_usage():
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(tool):
        pytest.skip('cuobjdump not available')
    if not os.path.exists(LIB):
        pytest.skip('library not built')
    out = subprocess.run([tool, '--dump-resource-usage', LIB], capture_output=True, text=True, check=True).stdout
    usage, name = {}, None
    for line in out.splitlines():
        m = KERNEL.search(line) if 'Function' in line else None
        if m:
            name = tuple(int(x) for x in m.groups())
        elif name is not None and 'REG:' in line:
            usage[name] = {k: int(v) for k, v in re.findall(r'(REG|STACK|LOCAL):(\d+)', line)}
            name = None
    return usage


def test_courier_instantiations_fit_two_ctas_per_sm():
    """Every step instantiation that can carry the courier warp (NP < 16, single-warp, hand-over, no DYN / NZ / SCN) uses at
    most 128 registers and no local memory: two 256-thread CTAs, or three 160-thread ones, fit the 64 K registers of an SM."""
    usage = _resource_usage()
    courier = {k: v for k, v in usage.items() if k[0] < 16 and k[1:] == (0, 0, 1, 0, 0)}
    assert sorted(k[0] for k in courier) == [1, 2, 4, 8], sorted(usage)
    for k, v in courier.items():
        assert v['REG'] <= 128 and v['LOCAL'] == 0, (k, v)


def _stagger(torch, eng, seed):
    """Every env at its own point of the episode, as in bench.py: auto-resets in every step."""
    st = eng.get_state()
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    st['env_i32'][:, 0] = torch.randint(0, eng.ep_len + 1, (eng.E,), device='cuda', generator=g, dtype=torch.int32)
    eng.set_state(st)


def _pair(torch, E, T, ep_time=1.0, wrapped=False):
    from quad_swarm_rl_b200.engine import QuadSwarmEngine
    mk = lambda: QuadSwarmEngine(num_envs=E, seed=21, ep_time=ep_time, device_scenario='o_random', rew_coeff=C3_REW, **C3)
    e1, e2 = mk(), mk()
    for e in (e1, e2):
        if wrapped:
            e.wrap_enable(use_replay=True, replay_buffer_size=8, replay_prob=0.75, replay_always_active=True)
        e.set_chained(True)               # the same kernel instantiation on both sides (only equal builds are bit-equal)
        e.reset()
        _stagger(torch, e, 77)
    g = torch.Generator(device='cuda')
    g.manual_seed(5)
    a = (torch.rand((T, E, 8, 4), device='cuda', generator=g) * 2 - 1).contiguous()
    return e1, e2, a


def _step_grid_shape(torch, eng, a, tmp_path):
    """(grid, block) of the step kernel of one chained launch, from a profiler trace."""
    import json
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.step(a)
        torch.cuda.synchronize()
    path = str(tmp_path / 'trace.json')
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))['traceEvents'] if 'qs_step_kernel' in e.get('name', '') and 'grid' in e.get('args', {})]
    assert ev, 'no step kernel in the trace'
    return ev[-1]['args']['grid'][0], ev[-1]['args']['block'][0]


def _expected_shape(torch):
    """The c3 shape plan_step picks on a 132-SM H100 SXM (None elsewhere: other SM counts give other shapes)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return (256, 160) if sms == 132 else None


@pytest.mark.gpu
@pytest.mark.parametrize('same_output', [False, True], ids=['ring', 'same_output_array'])
def test_chained_graph_in_step_shape_equals_one_rollout(same_output, tmp_path):
    """A CUDA graph of 240 chained c3 step launches (4096 envs, staggered ticks, 1 s episodes: about 40 auto-resets per step,
    and a next-episode generator launch every 25 steps, so that resets use both pre-generated and inline episodes) gives
    what one rollout launch gives, bit for bit.  With `same_output` every step writes the engine's own output arrays, so
    the observation rows of consecutive steps land on the same addresses; the last step must still win."""
    import torch
    T, E = 240, 4096
    e1, e2, a = _pair(torch, E, T)
    expect = _expected_shape(torch)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    obs = torch.empty((T, E, 8, e1.D), device='cuda'); rew = torch.empty((T, E, 8), device='cuda')
    dn = torch.empty((T, E, 8), dtype=torch.uint8, device='cuda')
    with torch.cuda.stream(st):
        warm = a[:2].clone()
        e1.step(warm[0])
        if expect is not None:
            assert _step_grid_shape(torch, e1, warm[1], tmp_path) == expect
        else:
            e1.step(warm[1])
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for t in range(T):
                if same_output:
                    e1.step(a[t])
                else:
                    e1.step(a[t], obs_out=obs[t], rewards_out=rew[t], dones_out=dn[t])
        g.replay()
        st.synchronize()
    e2.step(warm[0]); e2.step(warm[1])
    o2, r2, d2 = e2.rollout(a)
    torch.cuda.synchronize()
    if same_output:
        assert torch.equal(e1.obs, o2[-1]) and torch.equal(e1.rewards, r2[-1]) and torch.equal(e1.dones, d2[-1])
    else:
        assert torch.equal(obs, o2) and torch.equal(rew, r2) and torch.equal(dn, d2)
    assert int(d2.sum()) > 8 * T                      # auto-resets all along the chain
    s1, s2 = e1.get_state(), e2.get_state()
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        assert torch.equal(s1[k], s2[k]), k
    assert e1.handover_timeouts == 0 and e2.handover_timeouts == 0
    e1.close(); e2.close()


@pytest.mark.gpu
def test_wrapped_chain_in_step_shape_equals_synchronised_steps():
    """qs_wrap_step at the c3 size in the same shape: the wrapper kernel's blocks follow the step grid's env -> block mapping
    (StepParams.wrap_chain).  A CUDA graph of 200 wrapped control steps (replay on) leaves what the same launches with a
    device synchronisation after every one leave."""
    import torch
    from quad_swarm_rl_b200 import _lib as L
    T, E = 200, 4096
    e1, e2, a = _pair(torch, E, T, wrapped=True)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        e1.wrap_step(a[0])
        st.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            for t in range(1, T):
                e1.wrap_step(a[t])
        gr.replay()
        st.synchronize()
    e2.wrap_step(a[0])
    for t in range(1, T):
        e2.wrap_step(a[t])
        torch.cuda.synchronize()
    assert torch.equal(e1.obs, e2.obs) and torch.equal(e1.rewards, e2.rewards) and torch.equal(e1.dones, e2.dones)
    s1, s2 = e1.get_state(), e2.get_state()
    for k in ('agent_f32', 'agent_u32', 'env_i32'):
        assert torch.equal(s1[k], s2[k]), k
    g1, g2 = e1.wrap_read(), e2.wrap_read()
    assert g1[L.WA['EPISODES_TOTAL']] == g2[L.WA['EPISODES_TOTAL']] > 0
    np.testing.assert_allclose(g1, g2, rtol=2e-4, atol=1e-3)             # float atomics: the order of the additions differs
    assert e1.handover_timeouts == 0 and e2.handover_timeouts == 0
    e1.close(); e2.close()
