"""`Box` space used for observation_space / action_space.

gymnasium's `spaces.Box` is used when gymnasium is importable (so Sample Factory sees the real thing); this image has
no gymnasium, so a minimal stand-in with the same attributes (low, high, shape, dtype, sample, contains) is provided.
"""
import numpy as np

try:                                    # pragma: no cover - not installed in the build image
    from gymnasium.spaces import Box    # noqa: F401
except Exception:                       # ImportError or a stub without Box
    class Box:
        def __init__(self, low, high, shape=None, dtype=np.float32):
            low = np.asarray(low, dtype=dtype)
            high = np.asarray(high, dtype=dtype)
            if shape is not None:
                low = np.broadcast_to(low, shape).copy()
                high = np.broadcast_to(high, shape).copy()
            self.low, self.high = low, high
            self.shape = low.shape
            self.dtype = np.dtype(dtype)
            self._rng = np.random.default_rng()

        def seed(self, seed=None):
            self._rng = np.random.default_rng(seed)

        def sample(self):
            return self._rng.uniform(self.low, self.high).astype(self.dtype)

        def contains(self, x):
            x = np.asarray(x)
            return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

        def __repr__(self):
            return f"Box({self.shape}, {self.dtype})"


def make_observation_space(obs_repr, num_use_neighbor_obs, use_obstacles, room_dims, neighbor_obs_type='pos_vel'):
    """Bounds of QuadrotorSingle.make_observation_space (quadrotor_single.py:278-335) for the components in use."""
    room_range = np.array(room_dims, dtype=np.float64)          # room_box[1] - room_box[0]
    vxyz_max, omega_max = 3.0, 40.0                             # quadrotor_dynamics.py:49-50
    comp = {
        'xyz': (-room_range, room_range), 'vxyz': (-vxyz_max * np.ones(3), vxyz_max * np.ones(3)),
        'R': (-np.ones(9), np.ones(9)), 'omega': (-omega_max * np.ones(3), omega_max * np.ones(3)),
        'floor': (np.zeros(1), room_dims[2] * np.ones(1)), 'wall': (np.zeros(6), 5.0 * np.ones(6)),
        'rxyz': (-room_range, room_range), 'rvxyz': (-2.0 * vxyz_max * np.ones(3), 2.0 * vxyz_max * np.ones(3)),
        'octmap': (-10 * np.ones(9), 10 * np.ones(9)),
    }
    names = obs_repr.split('_')
    if neighbor_obs_type == 'pos_vel' and num_use_neighbor_obs > 0:
        names = names + ['rxyz', 'rvxyz'] * num_use_neighbor_obs
    if use_obstacles:
        names = names + ['octmap']
    low = np.concatenate([comp[n][0] for n in names])
    high = np.concatenate([comp[n][1] for n in names])
    return Box(low, high, dtype=np.float32)


def make_action_space(raw_control=True, raw_control_zero_middle=True, thrust_to_weight=None):
    """The controller's action_space (quadrotor_single.py:259-273): RawControl with zero_action_middle [-1, 1], without it
    [0, 1] (quadrotor_control.py:37-49); NonlinearPositionController (raw_control=False) the bounds of its unused action,
    (-1, -10 pi, -10 pi, -2 pi) .. (thrust_to_weight - 1, 10 pi, 10 pi, 2 pi) of the drone's model (:482-490)."""
    if not raw_control:
        max_rp, max_yaw = 5 * 2 * np.pi, 2 * np.pi
        return Box(np.array([-1.0, -max_rp, -max_rp, -max_yaw]),
                   np.array([thrust_to_weight - 1.0, max_rp, max_rp, max_yaw]), dtype=np.float32)
    if not raw_control_zero_middle:
        return Box(np.zeros(4), np.ones(4), dtype=np.float32)
    return Box(-np.ones(4), np.ones(4), dtype=np.float32)
