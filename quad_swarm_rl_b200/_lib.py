"""ctypes binding of include/quadswarm.h (the C ABI of the CUDA env step).

The shared library is built in-tree by `__graft_entry__.build()` (nvcc, sm_90a).  There is no CPU
fallback: if the library is missing, loading fails loudly.
"""
import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('QS_LIB') or os.path.join(_PKG, 'libquadswarm.so')     # QS_LIB: tuning builds only

QS_OK = 0
QS_NUM_REW_COEFF = 8
QS_NUM_TERMS = 8
QS_NUM_ENV_STATS = 13
QS_NUM_AGENT_STATS = 4
QS_STATE_F32 = 43
QS_STATE_U32 = 4
QS_STATE_ENV_I32 = 36
QS_MAX_AGENTS = 32
QS_DYN_ROW = 40
QS_DYN_LEAVES = 45
QS_CONTROL_RAW, QS_CONTROL_RAW_UNIT, QS_CONTROL_POSITION = 0, 1, 2
SCENARIO_HOST_TABLES, SCENARIO_O_RANDOM = 0, 1
# scenarios with a device-side generator (QS_SCENARIO_* of include/quadswarm.h), by their reference names
DEVICE_SCENARIOS = {'o_random': 1, 'static_same_goal': 2, 'static_diff_goal': 3, 'dynamic_same_goal': 4,
                    'dynamic_diff_goal': 5, 'swap_goals': 6, 'dynamic_formations': 7, 'ep_lissajous3D': 8,
                    'swarm_vs_swarm': 9, 'mix': 10, 'o_static_same_goal': 11, 'ep_rand_bezier': 12,
                    'o_dynamic_same_goal': 13, 'o_swap_goals': 14, 'o_ep_rand_bezier': 15, 'run_away': 16}
OBSTACLE_SCENARIOS = ('o_random', 'o_static_same_goal', 'o_dynamic_same_goal', 'o_swap_goals', 'o_ep_rand_bezier')
SCENARIO_NAMES = {v: k for k, v in DEVICE_SCENARIOS.items()}

REW_KEYS = ('pos', 'effort', 'crash', 'orient', 'spin', 'quadcol_bin', 'quadcol_bin_smooth_max', 'quadcol_bin_obst')
OBS_REPR = {'xyz_vxyz_R_omega': 0, 'xyz_vxyz_R_omega_floor': 1, 'xyz_vxyz_R_omega_wall': 2}
OBS_SELF_SIZE = {'xyz_vxyz_R_omega': 18, 'xyz_vxyz_R_omega_floor': 19, 'xyz_vxyz_R_omega_wall': 24}

FLAG_ON_FLOOR, FLAG_CRASHED_FLOOR, FLAG_CRASHED_WALL, FLAG_CRASHED_CEILING = 1 << 0, 1 << 1, 1 << 2, 1 << 3
FLAG_PREV_WALL, FLAG_PREV_CEILING, FLAG_PREV_ROOM, FLAG_PREV_OBST = 1 << 4, 1 << 5, 1 << 6, 1 << 7
FLAG_NO_COL_AGENT, FLAG_NO_COL_OBST, FLAG_REACHED_GOAL = 1 << 8, 1 << 9, 1 << 10
FLAG_KICKED, FLAG_NEW_QUADCOL, FLAG_NEW_OBSTCOL = 1 << 11, 1 << 12, 1 << 13

ENV_STAT_KEYS = ('num_collisions', 'num_collisions_after_settle', 'num_collisions_final_5_s', 'num_collisions_with_room',
                 'num_collisions_with_floor', 'num_collisions_with_wall', 'num_collisions_with_ceiling',
                 'num_collisions_obst_quad', 'num_collisions_obst_quad_after_settle', 'num_collisions_obst_quad_3_5',
                 'num_collisions_obst_quad_5', 'episodes_done', 'scenario')


class QsConfig(C.Structure):
    _fields_ = [
        ('num_envs', C.c_int32), ('num_agents', C.c_int32), ('obs_repr', C.c_int32),
        ('neighbor_visible_num', C.c_int32), ('use_obstacles', C.c_int32), ('num_obstacles', C.c_int32),
        ('use_downwash', C.c_int32), ('sense_noise', C.c_int32), ('obst_size', C.c_float),
        ('room_dims', C.c_float * 3), ('ep_time', C.c_float), ('collision_hitbox_radius', C.c_float),
        ('collision_falloff_radius', C.c_float), ('approch_goal_metric', C.c_float),
        ('env_id_offset', C.c_int32), ('scenario', C.c_int32), ('obst_grid', C.c_int32 * 2), ('seed', C.c_uint64),
        ('quad_arm', C.c_float), ('reserved_', C.c_int32 * 3),
    ]


class QsSensorNoise(C.Structure):
    _fields_ = [(k, C.c_double) for k in ('pos_norm_std', 'pos_unif_range', 'vel_norm_std', 'vel_unif_range', 'quat_norm_std',
                                           'quat_unif_range', 'gyro_noise_density', 'gyro_norm_std', 'gyro_random_walk',
                                           'gyro_bias_correlation_time')]


class QsWrapConfig(C.Structure):
    _fields_ = [('use_replay', C.c_int32), ('replay_buffer_size', C.c_int32), ('replay_prob', C.c_float),
                ('replay_always_active', C.c_int32), ('reserved_', C.c_int32 * 4)]


class QsDynLeaves(C.Structure):
    _fields_ = [('value', C.c_double * QS_DYN_LEAVES), ('present', C.c_uint8 * QS_DYN_LEAVES), ('reserved_', C.c_uint8 * 3)]


class QsDynSampler(C.Structure):
    _fields_ = [('base', C.c_int32), ('sampler', C.c_int32 * 2), ('n_order', C.c_int32), ('order', C.c_int32 * QS_DYN_LEAVES),
                ('params', QsDynLeaves), ('change', QsDynLeaves), ('samp', QsDynLeaves * 2)]


def _leaves(present_value):
    out = QsDynLeaves()
    present, value = present_value
    out.present[:] = [int(x) for x in present]
    out.value[:] = [float(x) for x in value]
    return out


def dyn_sampler_struct(spec):
    """quad_models.dynamics_sampler_spec(...) -> QsDynSampler."""
    out = QsDynSampler()
    out.base = int(spec['base'])
    out.sampler[:] = [int(k) for k in spec['sampler']]
    out.n_order = len(spec['order'])
    out.order[:len(spec['order'])] = [int(k) for k in spec['order']]
    out.params, out.change = _leaves(spec['params']), _leaves(spec['change'])
    out.samp[0], out.samp[1] = _leaves(spec['samp'][0]), _leaves(spec['samp'][1])
    return out


def dyn_sampler_spec_of(st):
    """QsDynSampler -> the spec dict of quad_models.dynamics_sampler_spec."""
    import numpy as np
    leaves = lambda l: (np.array(l.present[:], np.uint8), np.array(l.value[:], np.float64))
    return dict(base=st.base, order=np.array(st.order[:st.n_order], np.int32), params=leaves(st.params), change=leaves(st.change),
                sampler=list(st.sampler), samp=[leaves(st.samp[0]), leaves(st.samp[1])])


QS_WRAP_AGG = 149
WA = dict(AGENT_EPISODES=0, TRUE_REWARD=1, RAW0=2, REW0=10, ACT_MEAN0=18, ACT_STD0=22, ENV_EPISODES=26, ENV_STAT0=27, DIST0=38,
          SUCCESS=41, DEADLOCK=42, COL=43, NEIGHBOR_COL=44, OBST_COL=45, REPLAY_ENV_EPISODES=46, REPLAY_COLLISIONS=47,
          REPLAY_COLLISIONS_OBST=48, EPISODES_TOTAL=49, REPLAYED_EVENTS=50, EVENTS_STORED=51, CHECKPOINTS=52, SCN0=53)

EXPORTS = {
    # name: (restype, argtypes)
    'qs_create': (C.c_int, [C.POINTER(QsConfig), C.c_int, C.POINTER(C.c_void_p)]),
    'qs_destroy': (C.c_int, [C.c_void_p]),
    'qs_last_error': (C.c_char_p, []),
    'qs_obs_dim': (C.c_int, [C.c_void_p]),
    'qs_num_envs': (C.c_int, [C.c_void_p]),
    'qs_num_agents': (C.c_int, [C.c_void_p]),
    'qs_num_obstacles': (C.c_int, [C.c_void_p]),
    'qs_ep_len': (C.c_int, [C.c_void_p]),
    'qs_set_reward_coeffs': (C.c_int, [C.c_void_p, C.POINTER(C.c_float)]),
    'qs_set_next_episode': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_next_obstacle_radius': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_goals': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_reset': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_step': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_step_host': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_reset_host': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_step_host_async': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_wait': (C.c_int, [C.c_void_p]),
    'qs_rollout': (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    'qs_get_state': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_state': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_read_episode_stats': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_chained': (C.c_int, [C.c_void_p, C.c_int]),
    'qs_set_obstacle_randomization': (C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_float), C.c_int]),
    'qs_set_dynamics': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    'qs_set_dynamics_sampler': (C.c_int, [C.c_void_p, C.POINTER(QsDynSampler), C.c_int]),
    'qs_get_dynamics': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_sensor_noise': (C.c_int, [C.c_void_p, C.POINTER(QsSensorNoise)]),
    'qs_get_gyro_bias': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_gyro_bias': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_set_init_random_state': (C.c_int, [C.c_void_p, C.c_int, C.c_float, C.c_float]),
    'qs_set_numpy_dynamics': (C.c_int, [C.c_void_p, C.c_int]),
    'qs_set_control': (C.c_int, [C.c_void_p, C.c_int]),
    'qs_wrap_enable': (C.c_int, [C.c_void_p, C.POINTER(QsWrapConfig)]),
    'qs_wrap_step': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_wrap_apply': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_wrap_read': (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    'qs_wrap_true_reward': (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    'qs_launch_count': (C.c_int64, [C.c_void_p]),
    'qs_handover_timeouts': (C.c_int64, [C.c_void_p]),
}

_lib = None


def load():
    """dlopen the in-tree CUDA library and declare every entry point of include/quadswarm.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: the CUDA extension has not been built. Run "
            "`python -c 'import __graft_entry__ as g; g.build()'` from the repo root (needs nvcc). "
            "There is no CPU fallback for the env step.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class QsError(RuntimeError):
    pass


def check(rc):
    if rc != QS_OK:
        msg = load().qs_last_error()
        raise QsError(f"quadswarm error {rc}: {msg.decode() if msg else '?'}")
