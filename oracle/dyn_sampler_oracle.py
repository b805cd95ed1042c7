"""CPU twin of the device-side dynamics sampler (qs_set_dynamics_sampler; quad_swarm_rl_b200/csrc/qs_dyn_sampler.cuh).

TEST INFRASTRUCTURE ONLY.  The twin adds no second restatement of the physics: it feeds the UNMODIFIED host pipeline,
`quad_models.DynamicsSource` (pinned to the reference by tests/golden/dyn_models.json and ref_randomquad_relsampler_5.npz),
with a numpy `RandomState` stand-in whose `uniform` / `normal` return the keyed draws of site SITE_DYN in sequence:

    draw k of drone i of env e in episode g = Philox block (e, EPISODE_KEY_BIT | g, SITE_DYN | i << 8, k), key = seed
    uniform(low, high) = low + (high - low) u01(word 0)
    normal(loc, scale) = loc + scale sqrt(-2 ln u1) cos(2 pi u2),  u1, u2 of words (0, 1) as philox.normal_pair

Calls with array arguments or `size` are split into scalar draws in C order, which is how numpy's RandomState consumes its
stream; `ForwardingDraws` does the same split on a real RandomState, so that a test can show the split keeps the pipeline's
draw order (its rows equal DynamicsSource's own).  Episode 0 is the construction sample.
"""
import math

import numpy as np

from quad_swarm_rl_b200.quad_models import DynamicsSource

from .philox import EPISODE_KEY_BIT, MASK, philox4x32_10

SITE_DYN = 24


class ScalarDraws:
    """RandomState stand-in: every uniform / normal call becomes scalar draws in C order (subclasses give the scalars)."""

    def __init__(self):
        self.count = 0

    def _draw(self, fn, a, b, size):
        a_arr, b_arr = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
        if size is not None:
            a_arr, b_arr = np.broadcast_to(a_arr, size), np.broadcast_to(b_arr, size)
        vals = []
        for x, y in zip(a_arr.ravel(), b_arr.ravel()):
            vals.append(fn(float(x), float(y)))          # self.count = index of this scalar in the drone's sequence
            self.count += 1
        out = np.array(vals, np.float64)
        if size is None and a_arr.ndim == 0:
            return float(out[0])
        return out.reshape(a_arr.shape)

    def uniform(self, low=0.0, high=1.0, size=None):
        return self._draw(self.scalar_uniform, low, high, size)

    def normal(self, loc=0.0, scale=1.0, size=None):
        return self._draw(self.scalar_normal, loc, scale, size)


class ForwardingDraws(ScalarDraws):
    """Scalar draws from a real RandomState (one call per scalar)."""

    def __init__(self, rs):
        super().__init__()
        self.rs = rs

    def scalar_uniform(self, low, high):
        return self.rs.uniform(low, high)

    def scalar_normal(self, loc, scale):
        return self.rs.normal(loc, scale)


class KeyedDraws(ScalarDraws):
    """The device's draws of one drone: scalar k comes from Philox block k of SITE_DYN."""

    def __init__(self, seed, env_id, episode, drone):
        super().__init__()
        self.k0, self.k1 = seed & MASK, (seed >> 32) & MASK
        self.c0, self.c1, self.c2 = env_id & MASK, EPISODE_KEY_BIT | episode, SITE_DYN | (drone << 8)

    def _block(self):
        return philox4x32_10(self.c0, self.c1, self.c2, self.count, self.k0, self.k1)

    def scalar_uniform(self, low, high):
        x = self._block()[0]
        return low + (high - low) * ((x >> 8) * 2.0 ** -24)

    def scalar_normal(self, loc, scale):
        xa, xb = self._block()[:2]
        u1 = ((xa >> 9) + 0.5) * 2.0 ** -23
        u2 = (xb >> 8) * 2.0 ** -24
        return loc + scale * (math.sqrt(-2.0 * math.log(u1)) * math.cos(2.0 * math.pi * u2))


def twin_source(dynamics_params='Crazyflie', dynamics_change=None, dyn_sampler_1=None, dyn_sampler_2=None):
    """A DynamicsSource whose construction draws (structure only) come from a throw-away RandomState."""
    return DynamicsSource(dynamics_params, dynamics_change, dyn_sampler_1, dyn_sampler_2, rs=np.random.RandomState(0))


def twin_row(src, seed, env_id, episode, drone):
    """The float32 row the device writes for drone `drone` of global env `env_id` in episode `episode`."""
    src.rs = KeyedDraws(seed, env_id, episode, drone)
    return src.sample_row()


def twin_rows(src, seed, episodes, num_agents, env_id_offset=0):
    """Rows [E, N, 40] of envs env_id_offset + e, each in its episode episodes[e]."""
    return np.stack([np.stack([twin_row(src, seed, env_id_offset + e, int(g), i) for i in range(num_agents)])
                     for e, g in enumerate(episodes)])
