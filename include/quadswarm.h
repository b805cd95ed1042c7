/*
 * quadswarm.h — C ABI of the H100-native QuadSwarm vectorised environment step.
 *
 * The reference (Zhehui-Huang/quad-swarm-rl) has NO FFI: its hot path is a Python object protocol
 * (SURVEY.md §8b).  This header is the boundary a binding would target; every entry point names the
 * reference interface it replaces (paths under gym_art/quadrotor_multi/ unless stated otherwise).
 * `quad_swarm_rl_b200/env.py` binds it with ctypes and re-exposes the reference's
 * QuadrotorEnvMulti.reset()/step() surface on top; INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *   - Plain C types only.  All *_dev pointers are caller-owned DEVICE memory on the handle's GPU,
 *     *_host pointers are host memory.  Nothing is allocated per step.
 *   - E = envs on this GPU, N = drones per env (<= 32), A = E*N agents, D = qs_obs_dim(),
 *     M = qs_num_obstacles().  Agent index a = env*N + i everywhere.
 *   - Work is enqueued on the cudaStream_t passed as `stream` (a void*; NULL = default stream);
 *     only the *_host entry points synchronise.  The *_host entry points run on a private stream of the
 *     handle and order themselves after the most recent asynchronous call of the handle (whatever stream it
 *     used), so e.g. qs_set_goals(stream) followed by qs_step_host() is race-free.
 *   - Return value: 0 = QS_OK, negative = error; qs_last_error() gives the message (thread-local).
 *   - One handle per GPU; a handle is not thread-safe.
 */
#ifndef QUADSWARM_H_
#define QUADSWARM_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QS_OK 0
#define QS_ERR_INVALID_ARG (-1)
#define QS_ERR_UNSUPPORTED (-2)
#define QS_ERR_CUDA (-3)

#define QS_MAX_AGENTS 32
#define QS_MAX_OBST_CHOICES 16

/* obs_repr: quad_utils.py:30-34 (QUADS_OBS_REPR) */
#define QS_OBS_XYZ_VXYZ_R_OMEGA 0       /* 18 floats */
#define QS_OBS_XYZ_VXYZ_R_OMEGA_FLOOR 1 /* 19 floats */
#define QS_OBS_XYZ_VXYZ_R_OMEGA_WALL 2  /* 24 floats */

/* Episode generation (goal / spawn points, pillar placement), the job of scenario.reset() +
 * obst_generation_given_density() in the reference (quadrotor_multi.py:304-325,347-353):
 *   HOST_TABLES  the host uploads tables with qs_set_next_episode (any scenario of scenarios/*.py);
 *   O_RANDOM     generated on the device at every (auto-)reset: M distinct pillar cells, N distinct free spawn cells and
 *                N distinct free goal cells, z ~ U(1,3) (scenarios/obstacles/o_random.py:27-52, o_base.py:71-83);
 *                needs use_obstacles.  No host work per episode. */
#define QS_SCENARIO_HOST_TABLES 0
#define QS_SCENARIO_O_RANDOM 1
/* The obstacle-free scenario family, generated and TICKED on the device (formation picks, goal formations, the timed
 * goal switches every 4-6 s, per-tick goal motion; `mix` draws one of the eight per episode; scenarios/base.py:39-150,
 * dynamic_same_goal.py, dynamic_diff_goal.py, swap_goals.py, dynamic_formations.py, ep_lissajous3D.py,
 * swarm_vs_swarm.py, mix.py:37-93).  Ids 2..9 need use_obstacles = 0 and are contiguous on purpose. */
#define QS_SCENARIO_STATIC_SAME_GOAL 2
#define QS_SCENARIO_STATIC_DIFF_GOAL 3
#define QS_SCENARIO_DYNAMIC_SAME_GOAL 4
#define QS_SCENARIO_DYNAMIC_DIFF_GOAL 5
#define QS_SCENARIO_SWAP_GOALS 6
#define QS_SCENARIO_DYNAMIC_FORMATIONS 7
#define QS_SCENARIO_EP_LISSAJOUS3D 8
#define QS_SCENARIO_SWARM_VS_SWARM 9
#define QS_SCENARIO_MIX 10                  /* use_obstacles = 0: one of 2..9 and 12 per episode (scenarios/utils.py:7-16); = 1: o_random or
                                               o_static_same_goal (mix.py:45-57, utils.py:18) */
/* obstacles/o_static_same_goal.py: pillars and spawn cells as o_random, one common goal above the centre of the
 * largest free square of the pillar grid (o_base.py:123-153), approch_goal_metric 1.0.  Needs use_obstacles. */
#define QS_SCENARIO_O_STATIC_SAME_GOAL 11
/* scenarios/ep_rand_bezier.py: one common goal that follows quadratic Bezier segments, two control points re-drawn 5..10 m
 * away every 5 s (and at tick 1) until both lie inside the room.  Obstacle-free family; part of `mix`. */
#define QS_SCENARIO_EP_RAND_BEZIER 12
/* The evaluation scenarios of the obstacle family (scenarios/utils.py:18-20), generated and ticked on the device; pillars
 * and spawn cells as o_random; all need use_obstacles and have approch_goal_metric 1.0 (o_base.py:16):
 *   O_DYNAMIC_SAME_GOAL  common goal above the centre of the largest free square; at tick 1 and then every 4-6 s it hops to a
 *                        random free cell at most 4 m away, z ~ U(0.75, 3) (o_dynamic_same_goal.py:17-51);
 *   O_SWAP_GOALS         a formation around that centre, permuted among the drones every 4-6 s (o_swap_goals.py);
 *   O_EP_RAND_BEZIER     common goal above a random free cell, then quadratic Bezier segments of 6 s whose two control
 *                        points lie 2..5 m away and inside x, y in (-4.5, 4.5), z in (2, 2.5) (o_ep_rand_bezier.py:14-57). */
#define QS_SCENARIO_O_DYNAMIC_SAME_GOAL 13
#define QS_SCENARIO_O_SWAP_GOALS 14
#define QS_SCENARIO_O_EP_RAND_BEZIER 15
/* scenarios/run_away.py: a shuffled goal formation around (0, 0, 2); every second (tick % 100 == 0, tick > 0) the goals of
 * drones 0 and 1 jump onto the goals of two random drones drawn from 1..N-1 (run_away.py:14-25).  Obstacle-free family,
 * not part of `mix` (scenarios/utils.py:7-10); needs num_agents >= 2, as the reference's randint(1, N). */
#define QS_SCENARIO_RUN_AWAY 16
#define QS_SCENARIO_LAST QS_SCENARIO_RUN_AWAY
#define QS_SCENARIO_DEVICE_FAMILY_FIRST QS_SCENARIO_STATIC_SAME_GOAL

/* reward coefficient slots: the subset of QuadrotorEnvMulti.rew_coeff (quadrotor_multi.py:91-94) with a
 * non-zero default or a CLI override (swarm_rl/env_wrappers/reward_shaping.py:7-16). */
enum {
    QS_REW_POS = 0, QS_REW_EFFORT, QS_REW_CRASH, QS_REW_ORIENT, QS_REW_SPIN,
    QS_REW_QUADCOL_BIN, QS_REW_QUADCOL_BIN_SMOOTH_MAX, QS_REW_QUADCOL_BIN_OBST,
    QS_NUM_REW_COEFF
};

/* per-agent raw reward terms written by qs_step when rew_terms_dev != NULL; these are the `rewraw_*`
 * entries of infos[i]['rewards'] (quadrotor_single.py:68-85, quadrotor_multi.py:533-540), from which the
 * host rebuilds every `rew_*` key by multiplying with the coefficient in force for that step. */
enum {
    QS_TERM_RAW_POS = 0,     /* rewraw_pos  = -dt*|goal-pos|  (== rewraw_main) */
    QS_TERM_RAW_ACTION,      /* rewraw_action = -dt*|a| */
    QS_TERM_RAW_CRASH,       /* rewraw_crash  = -dt*on_floor */
    QS_TERM_RAW_ORIENT,      /* rewraw_orient */
    QS_TERM_RAW_SPIN,        /* rewraw_spin */
    QS_TERM_RAW_QUADCOL,     /* rewraw_quadcol (0 / -1) */
    QS_TERM_PROXIMITY,       /* rew_proximity (already weighted: depends on quadcol_bin_smooth_max) */
    QS_TERM_RAW_QUADCOL_OBST,/* rewraw_quadcol_obstacle (0 / -1) */
    QS_NUM_TERMS
};

/* per-env episode statistics latched when an episode ends (quadrotor_multi.py:626-718) */
enum {
    QS_STAT_NUM_COLLISIONS = 0, QS_STAT_NUM_COLLISIONS_AFTER_SETTLE, QS_STAT_NUM_COLLISIONS_FINAL_5S,
    QS_STAT_NUM_COLLISIONS_ROOM, QS_STAT_NUM_COLLISIONS_FLOOR, QS_STAT_NUM_COLLISIONS_WALL,
    QS_STAT_NUM_COLLISIONS_CEILING, QS_STAT_NUM_COLLISIONS_OBST, QS_STAT_NUM_COLLISIONS_OBST_AFTER_SETTLE,
    QS_STAT_NUM_COLLISIONS_OBST_3_5, QS_STAT_NUM_COLLISIONS_OBST_5, QS_STAT_EPISODES_DONE,
    QS_STAT_SCENARIO,        /* QS_SCENARIO_* of the episode that ended (for `mix`: the scenario drawn for it) */
    QS_NUM_ENV_STATS
};
/* per-agent episode statistics latched with them */
enum {
    QS_ASTAT_DIST_1S = 0, QS_ASTAT_DIST_3S, QS_ASTAT_DIST_5S,
    QS_ASTAT_FLAGS,          /* bit0 agent_col_agent (1 = never collided after settle), bit1 agent_col_obst, bit2 reached_goal */
    QS_NUM_AGENT_STATS
};

/* Construction arguments = the keyword set of QuadrotorEnvMulti.__init__ that the hot path reads
 * (quadrotor_multi.py:24-41), with the fixed choices of the env factory
 * (swarm_rl/env_wrappers/quad_utils.py:22-31: Crazyflie, raw control, default sensor noise,
 * thrust_noise_ratio 0.05, use_numba=True) baked in. */
typedef struct QsConfig {
    int32_t num_envs;                /* E on this GPU */
    int32_t num_agents;              /* N, 1..32 */
    int32_t obs_repr;                /* QS_OBS_* */
    int32_t neighbor_visible_num;    /* -1 = all others, 0 = none, else K (quadrotor_multi.py:47-50) */
    int32_t use_obstacles;
    int32_t num_obstacles;           /* M = int(density * area) (quadrotor_multi.py:128) */
    int32_t use_downwash;
    int32_t sense_noise;             /* 1 = 'default' (sensor_noise.py:70-76) or the set of qs_set_sensor_noise, 0 = bypass */
    float obst_size;                 /* pillar diameter */
    float room_dims[3];
    float ep_time;                   /* seconds; ep_len = int(ep_time / 0.01) (quadrotor_single.py:158) */
    float collision_hitbox_radius;   /* in arm lengths (quadrotor_multi.py:154) */
    float collision_falloff_radius;  /* in arm lengths (quadrotor_multi.py:155) */
    float approch_goal_metric;       /* scenario.approch_goal_metric (scenarios/base.py:31) */
    int32_t env_id_offset;           /* global id of env 0 (multi-GPU shards: rank * E); keys the RNG */
    int32_t scenario;                /* QS_SCENARIO_*: who generates the episodes consumed by (auto-)resets */
    int32_t obst_grid[2];            /* pillar grid cells along x / y = int(obst_spawn_area) (quadrotor_multi.py:305) */
    uint64_t seed;
    float quad_arm;                  /* QuadrotorEnvMulti.quad_arm = envs[0].dynamics.arm at construction (quadrotor_multi.py:81);
                                        0 = Crazyflie (0.04596194 m).  Scales the collision / proximity / pillar radii. */
    int32_t reserved_[3];
} QsConfig;

typedef struct QsHandle QsHandle;

/* replaces QuadrotorEnvMulti.__init__ (quadrotor_multi.py:24-207) */
int qs_create(const QsConfig* cfg, int device, QsHandle** out);
int qs_destroy(QsHandle* h);
const char* qs_last_error(void);

int qs_obs_dim(const QsHandle* h);        /* D = S + 6K (+9), quadrotor_single.py:311-316 */
int qs_num_envs(const QsHandle* h);
int qs_num_agents(const QsHandle* h);
int qs_num_obstacles(const QsHandle* h);
int qs_ep_len(const QsHandle* h);

/* replaces writes to env.unwrapped.rew_coeff (swarm_rl/env_wrappers/reward_shaping.py:55-61,110-118).
 * coeffs_host[QS_NUM_REW_COEFF]; takes effect at the next qs_step. */
int qs_set_reward_coeffs(QsHandle* h, const float* coeffs_host);

/* Episode tables consumed by the next (auto-)reset of each env — what scenario.reset() and
 * obst_generation_given_density() hand to QuadrotorEnvMulti.reset (quadrotor_multi.py:347-367).
 * goals_dev [E,N,3]; spawn_dev [E,N,3] or NULL (spawn at the goal, :363-364); obst_xy_dev [E,M,2] or NULL.
 * env_mask_dev [E] bytes or NULL (= all).  Tables persist until overwritten. */
int qs_set_next_episode(QsHandle* h, const uint8_t* env_mask_dev, const float* goals_dev, const float* spawn_dev,
                        const float* obst_xy_dev, void* stream);

/* Pillar radius of the next episode of each env on a host-table handle — the obst_size of
 * QuadrotorEnvMulti.reset(obst_density, obst_size) (quadrotor_multi.py:339-351; obstacles.py:9-10: radius = size / 2).
 * radius_dev [E] floats, env_mask_dev [E] bytes or NULL (= all).  Same contract as qs_set_next_episode: each masked env's
 * next (auto-)reset latches its value, which then sets the collision test, the contact response and the 3x3 distance
 * patch of that episode; it persists until overwritten.  The first call switches the handle to per-episode radii: every
 * env's running episode keeps the construction radius (QsConfig.obst_size / 2), and so does every later episode of an env
 * the calls never mask.  From then on the handle steps without the split step shape, like qs_set_obstacle_randomization.
 * qs_get_state / qs_set_state carry the running episode's radius (scenario state, scn_f[0].x).  Copies the radii to the
 * host and synchronises `stream` to check them: every one of the E values must be finite and >= 0.  Fails with
 * QS_ERR_INVALID_ARG without use_obstacles, or on a handle with a device-side scenario (which draws its sizes with
 * qs_set_obstacle_randomization). */
int qs_set_next_obstacle_radius(QsHandle* h, const uint8_t* env_mask_dev, const float* radius_dev, void* stream);

/* replaces `env.goal = ...` assignments made by scenario.step() (e.g. scenarios/swarm_vs_swarm.py:84-85). */
int qs_set_goals(QsHandle* h, const uint8_t* env_mask_dev, const float* goals_dev, void* stream);

/* replaces QuadrotorEnvMulti.reset (quadrotor_multi.py:339-411) for the masked envs; obs_dev [E,N,D]
 * (rows of unmasked envs are left untouched). */
int qs_reset(QsHandle* h, const uint8_t* env_mask_dev, float* obs_dev, void* stream);

/* replaces QuadrotorEnvMulti.step (quadrotor_multi.py:413-724): one control step of every env, auto-reset
 * included.  actions_dev [E,N,4] raw policy outputs; obs_dev [E,N,D]; rewards_dev [E,N]; dones_dev [E,N]
 * bytes; rew_terms_dev [E,N,QS_NUM_TERMS] or NULL.  One kernel launch. */
int qs_step(QsHandle* h, const float* actions_dev, float* obs_dev, float* rewards_dev, uint8_t* dones_dev,
            float* rew_terms_dev, void* stream);

/* same step with HOST buffers: H2D of actions, the step kernel, D2H of obs/rewards/dones(/terms), then a
 * stream synchronise — the call a non-batched rollout worker makes.  Pageable buffers go through the handle's
 * page-locked staging.  When every buffer is page-locked and mapped, the kernel reads the actions from and writes its
 * outputs to the host buffers itself (zero-copy over PCIe, no separate copy launches; QS_ZERO_COPY=0 in the environment
 * forces explicit cudaMemcpyAsync on the page-locked buffers instead). */
int qs_step_host(QsHandle* h, const float* actions_host, float* obs_host, float* rewards_host, uint8_t* dones_host,
                 float* rew_terms_host);
int qs_reset_host(QsHandle* h, const uint8_t* env_mask_host, float* obs_host);
/* The same step without the final synchronisation (page-locked buffers only): the call returns once the work is enqueued on
 * the handle's private stream; qs_wait blocks until the outputs are in the host buffers.  With two handles (two halves of
 * the envs, double-buffered sampling as Sample Factory runs its rollout workers) the kernel of one half overlaps the
 * PCIe transfer of the other:  A.async; B.async; A.wait -> policy on A's observations; B.wait -> ... */
int qs_step_host_async(QsHandle* h, const float* actions_host, float* obs_host, float* rewards_host, uint8_t* dones_host,
                       float* rew_terms_host);
int qs_wait(QsHandle* h);

/* T consecutive control steps in ONE launch (persistent CTAs keep the env block in registers):
 * actions_dev [T,E,N,4], obs_dev [T,E,N,D] or, when last_obs_only != 0, [E,N,D]; rewards_dev [T,E,N];
 * dones_dev [T,E,N].  Same results as T calls of qs_step. */
int qs_rollout(QsHandle* h, int num_steps, const float* actions_dev, float* obs_dev, float* rewards_dev,
               uint8_t* dones_dev, int last_obs_only, void* stream);

/* State snapshot / restore — what deepcopy(env) gives the replay wrapper (quad_experience_replay.py:99-104)
 * and what parity tests use for teacher forcing.  agent_f32_dev [E,N,QS_STATE_F32]: pos3 vel3 rot9(row-major)
 * omega3 thrust_rot_damp4 thrust_cmds_damp4 ou4 goal3 dist_ring4 dist_sums3 stale_vel3;
 * agent_u32_dev [E,N,QS_STATE_U32]: flags, prev_collision_row, 0, 0;
 * env_i32_dev [E,QS_STATE_ENV_I32]: tick, step_count, svd_count, episode_idx, the QS_NUM_ENV_STATS running counters,
 * then the device-side scenario state (4 ints: scenario, period, next event tick, formation | growing << 8; 12 floats as
 * bit patterns: formation size, layer distance, largest size, speed, centre 1 xyz_, centre 2 xyz_). */
#define QS_STATE_F32 43
#define QS_STATE_U32 4
#define QS_STATE_ENV_I32 36
int qs_get_state(QsHandle* h, float* agent_f32_dev, uint32_t* agent_u32_dev, int32_t* env_i32_dev,
                 float* obst_xy_dev, void* stream);
int qs_set_state(QsHandle* h, const uint8_t* env_mask_dev, const float* agent_f32_dev, const uint32_t* agent_u32_dev,
                 const int32_t* env_i32_dev, const float* obst_xy_dev, void* stream);

/* Per-drone physical constants — replaces QuadrotorSingle.update_dynamics / resample_dynamics (quadrotor_single.py:249-258,
 * 359-385) and QuadrotorDynamics.update_model (quadrotor_dynamics.py:104-166).  rows_dev [E,N,QS_DYN_ROW] floats, one row per
 * drone with the constants the integrator reads (host side: quad_swarm_rl_b200/quad_models.py derives them from a parameter
 * set / the dynamics-randomisation samplers):
 *   0 mass, 1 1/mass, 2-4 inertia diagonal, 5-7 its inverse, 8-11 thrust_max per motor, 12-15 torque_max per motor,
 *   16-23 propeller (x, y) per motor, 24-27 propeller z per motor (relative to the centre of mass), 28 motor_tau_up,
 *   29 motor_tau_down, 30 motor linearity, 31 OU sigma (0.2 * thrust_noise_ratio), 32 C_drag, 33 C_roll (rotor drag /
 *   rolling moment: numpy path of the reference only, quadrotor_dynamics.py:256-289), 34 vel_damp, 35 omega_quadratic,
 *   36 arm (= floor threshold, :378), 37-39 reserved.
 * at_next_reset = 0: the rows take effect now (construction); != 0: every masked env latches them at its next (auto-)reset,
 * where its OU state and SVD counter restart like those of the reference's fresh QuadrotorDynamics object.
 * Until the first call every drone uses the Crazyflie constants compiled into the kernels.  The env-level collision radii
 * (collision_hitbox_radius * arm etc.) stay those of QsConfig.quad_arm, as the reference fixes them at construction
 * (quadrotor_multi.py:81,154-155). */
#define QS_DYN_ROW 40
int qs_set_dynamics(QsHandle* h, const uint8_t* env_mask_dev, const float* rows_dev, int at_next_reset, void* stream);

/* Dynamics randomisation on the device — replaces the dynamics_params / dynamics_change / dyn_sampler_1 / dyn_sampler_2 /
 * dynamics_randomize_every pipeline of QuadrotorSingle (quadrotor_single.py:186-211,359-390; quadrotor_randomization.py).
 * Every drone's row is sampled on the device, in float64, and rounded to float32 once: base set (a fixed parameter tree or
 * RandomQuad, quadrotor_randomization.py:142-243) -> dynamics_change -> sampler 1 -> sampler 2 -> check_quad_param_limits ->
 * the link inertia model and the derived constants of qs_set_dynamics' row.  The row of drone i of env e in episode k is a
 * function of (seed, env_id_offset + e, k, i) only (draw site 24, episode-keyed): k = 0 is the construction sample, an
 * (auto-)reset that starts episode k >= 1 resamples when randomize_every > 0 and k % randomize_every == 0 (the reference's
 * (traj_count + 1) % every == 0 with traj_count = k - 1), and the drone keeps its row otherwise.
 *
 * The parameter tree is a flat vector of QS_DYN_LEAVES leaves, each a presence flag plus a float64 value; array leaves are
 * one leaf per element.  Leaf ids (QS_DL_*) name the tree's paths; `order` lists the present leaves in the order the tree
 * is walked (dict order of the host pipeline), which is the order RelativeSampler draws in. */
enum {
    QS_DL_BODY_L = 0, QS_DL_BODY_W, QS_DL_BODY_H, QS_DL_BODY_M, QS_DL_BODY_DENSITY,                          /* geom.body */
    QS_DL_PAYLOAD_L, QS_DL_PAYLOAD_W, QS_DL_PAYLOAD_H, QS_DL_PAYLOAD_M, QS_DL_PAYLOAD_DENSITY,                /* geom.payload */
    QS_DL_ARMS_L, QS_DL_ARMS_W, QS_DL_ARMS_H, QS_DL_ARMS_M, QS_DL_ARMS_DENSITY,                              /* geom.arms */
    QS_DL_MOTORS_H, QS_DL_MOTORS_R, QS_DL_MOTORS_M, QS_DL_MOTORS_DENSITY,                                    /* geom.motors */
    QS_DL_PROPS_H, QS_DL_PROPS_R, QS_DL_PROPS_M, QS_DL_PROPS_DENSITY,                                        /* geom.propellers */
    QS_DL_MOTOR_POS_X, QS_DL_MOTOR_POS_Y, QS_DL_MOTOR_POS_Z,                                                 /* geom.motor_pos.xyz */
    QS_DL_ARMS_ANGLE, QS_DL_ARMS_Z,                                                                          /* geom.arms_pos */
    QS_DL_PAYLOAD_X, QS_DL_PAYLOAD_Y, QS_DL_PAYLOAD_Z_SIGN,                                                  /* geom.payload_pos */
    QS_DL_DAMP_VEL, QS_DL_DAMP_OMEGA_QUADRATIC,                                                              /* damp */
    QS_DL_THRUST_NOISE_RATIO,                                                                                /* noise */
    QS_DL_THRUST_TO_WEIGHT, QS_DL_ASSYMETRY0, QS_DL_ASSYMETRY1, QS_DL_ASSYMETRY2, QS_DL_ASSYMETRY3,         /* motor */
    QS_DL_TORQUE_TO_THRUST, QS_DL_LINEARITY, QS_DL_C_DRAG, QS_DL_C_ROLL, QS_DL_DAMP_TIME_UP, QS_DL_DAMP_TIME_DOWN,
    QS_DYN_LEAVES
};
typedef struct QsDynLeaves {
    double value[QS_DYN_LEAVES];
    uint8_t present[QS_DYN_LEAVES];
    uint8_t reserved_[3];
} QsDynLeaves;
#define QS_DYN_BASE_FIXED 0             /* `params` is the base set (Crazyflie, DefaultQuad, MediumQuad, a dict) */
#define QS_DYN_BASE_RANDOM_QUAD 1       /* RandomQuad: 31 draws; `params.present` is its tree (values unused) */
#define QS_DYN_SAMPLER_NONE 0
#define QS_DYN_SAMPLER_RELATIVE_NORMAL 1    /* RelativeSampler(sampler='normal'): value ~ N(v, (ratio / 2 |v|)^2), one draw per leaf */
#define QS_DYN_SAMPLER_RELATIVE_UNIFORM 2   /* RelativeSampler(sampler='uniform'): value ~ U(v - v ratio, v + v ratio) */
#define QS_DYN_SAMPLER_CONST 3              /* ConstValueSampler: every present leaf of `samp` replaces the tree's value */
typedef struct QsDynSampler {
    int32_t base;                   /* QS_DYN_BASE_* */
    int32_t sampler[2];             /* QS_DYN_SAMPLER_* of dyn_sampler_1, dyn_sampler_2 */
    int32_t n_order;
    int32_t order[QS_DYN_LEAVES];   /* the present leaves of the tree in walk order (n_order of them) */
    QsDynLeaves params;             /* the tree: which leaves exist, and for QS_DYN_BASE_FIXED their values */
    QsDynLeaves change;             /* dynamics_change: present leaves override the base set's values */
    QsDynLeaves samp[2];            /* relative samplers: the noise ratio of every leaf of the tree; const: the new values */
} QsDynSampler;
/* Call after qs_create and before the first qs_reset / qs_step: allocates the per-drone tables and writes every drone's
 * construction sample.  randomize_every = 0 is the reference's None (the construction sample only).  Later calls, a handle
 * that already has rows from qs_set_dynamics, malformed specs (unknown kinds, leaves outside the tree, missing leaves the
 * model needs) and non-finite values fail with QS_ERR_INVALID_ARG.  qs_set_dynamics fails on such a handle: the sampler owns
 * the rows.  The sampling runs ahead of the resets where it can (beside the next-episode generator); the new rows are
 * latched right behind the step grid or the qs_reset that started their episode, and sampled there if none were prepared,
 * with the same results.  A sampler handle steps with the DYN kernels of qs_set_dynamics (single-warp shape, grid-wide
 * wait), one control step per grid: its qs_rollout launches num_steps grids. */
int qs_set_dynamics_sampler(QsHandle* h, const QsDynSampler* spec_host, int randomize_every);
/* The live rows of every drone, rows_dev [E,N,QS_DYN_ROW] floats (device -> device copy on `stream`).  Fails on a handle
 * without per-drone rows (neither qs_set_dynamics nor qs_set_dynamics_sampler was called). */
int qs_get_dynamics(QsHandle* h, float* rows_dev, void* stream);

/* Per-episode pillar density / size randomisation — replaces ExperienceReplayWrapper's domain randomisation
 * (gym_art/quadrotor_multi/quad_experience_replay.py:76-88,108-118,196-205: np.random.choice over np.arange(min, max, step))
 * and QuadrotorEnvMulti.reset(obst_density, obst_size) (quadrotor_multi.py:339-351).  densities_host [n_densities] and
 * sizes_host [n_sizes] (pillar diameters) are the choice lists; every (auto-)reset of an env draws one of each, places
 * int(density * area) pillars (at most QsConfig.num_obstacles, the table size) and uses size / 2 as the pillar radius for the
 * collision test, the contact response and the 3x3 distance patch of that episode.  Needs a device-side obstacle scenario.
 * n_densities = n_sizes = 0 switches the randomisation off. */
int qs_set_obstacle_randomization(QsHandle* h, const float* densities_host, int n_densities, const float* sizes_host, int n_sizes);

/* Sensor-noise model — replaces SensorNoise(**sense_noise) (sensor_noise.py:69-110; quadrotor_single.py:236-247), one
 * parameter set for every drone of the handle.  Per observation of a drone (get_state.py:6-72, numba path):
 *   pos~ = pos + N(0, pos_norm_std) + U(-pos_unif_range, pos_unif_range), vel~ likewise,
 *   omega~ = omega + N(0, gyro_noise_density),
 *   R~ = quat2R(rot2quat(R) x quat_from_small_angle(theta)), theta = N(0, quat_norm_std) + U(-quat_unif_range, quat_unif_range).
 * gyro_norm_std != 0 switches on the stateful gyro model (add_noise_to_omega, sensor_noise.py:221-231, dt = 0.005 s):
 * omega~ = omega + b + gyro_random_walk N(0, 1) after b <- pi b + sigma_b N(0, 1), with one bias b per drone that starts at
 * zero, is never reset and advances once per observation (a step draws up to three: its own, the re-draw after a contact
 * response, the observation of an auto-reset).  The accelerometer parameters are not part of the struct: it is never observed.
 * Every std and range must be finite and >= 0; gyro_bias_correlation_time > 0 when the gyro model is on.
 * Call after qs_create and before the first qs_reset / qs_step; later calls fail with QS_ERR_INVALID_ARG (the reference sets
 * the noise only in its constructor), as does a call on a handle whose QsConfig.sense_noise = 0.  Without a call the
 * 'default' set (QsConfig.sense_noise = 1) is compiled into the kernels.  The custom model runs in the single-warp step shape
 * with the grid-wide wait between steps. */
typedef struct QsSensorNoise {
    double pos_norm_std, pos_unif_range;
    double vel_norm_std, vel_unif_range;
    double quat_norm_std, quat_unif_range;
    double gyro_noise_density;
    double gyro_norm_std;                 /* != 0: stateful gyro bias */
    double gyro_random_walk;
    double gyro_bias_correlation_time;    /* seconds */
} QsSensorNoise;
int qs_set_sensor_noise(QsHandle* h, const QsSensorNoise* noise_host);

/* Gyro bias of every drone, [E,N,3] floats (zeros while the gyro model is off; set fails then).  Part of the env state for
 * snapshots: qs_get_state / qs_set_state do not carry it. */
int qs_get_gyro_bias(QsHandle* h, float* bias_dev, void* stream);
int qs_set_gyro_bias(QsHandle* h, const uint8_t* env_mask_dev, const float* bias_dev, void* stream);

/* Random initial states — replaces QuadrotorSingle(init_random_state=True) (quadrotor_single.py:405-423, 3-D): every spawn of
 * every drone, explicit reset or auto-reset, starts from QuadrotorDynamics.random_state (quadrotor_dynamics.py:193-206)
 * instead of a level attitude facing the origin at rest:
 *   vel = m / (|d| + 1e-6) d, d ~ U(-vel_max, vel_max)^3, m ~ U(0, vel_max); omega likewise with omega_max;
 *   R = rand_uniform_rot3d() (quad_utils.py:94-104), uniform over SO(3), upside down included.
 * The position is the usual spawn jitter (z >= 0.75); the neighbour block of a reset observation still sees the stale
 * velocities (QuadrotorEnvMulti.reset does not refresh self.vel).  The reference's values are vel_max = 1 m/s and
 * omega_max = 2 pi rad/s (QuadrotorSingle.max_init_vel / max_init_omega, quadrotor_single.py:181-182); both must be finite
 * and >= 0.  enable = 0 restores the default.  Call after qs_create and before the first qs_reset / qs_step; later calls fail
 * with QS_ERR_INVALID_ARG (the reference fixes the option in its constructor).  Works in every step shape. */
int qs_set_init_random_state(QsHandle* h, int enable, float vel_max, float omega_max);

/* Dynamics path — replaces QuadrotorEnvMulti(use_numba=False) (quadrotor_multi.py:67 -> QuadrotorSingle -> QuadrotorDynamics,
 * quadrotor_dynamics.py:211-214): enable = 1 steps the physics of the reference's numpy path, QuadrotorDynamics.step1 +
 * floor_interaction (:225-346, :389-457), instead of its njit path (step1_numba + floor_interaction_numba, :348-383, :569-639),
 * which is the default.  Only the floor model differs:
 *   - floor threshold and snap height 0.05 for every drone (:75, :392-393), not the drone's arm (:378);
 *   - at rest only when all three velocity components are exactly 0 (:406), not |vel| < 1e-6 (:586);
 *   - sliding friction (cos, sin)(atan2(-vy, -vx)), subtracted (:419-422): it pushes the drone along its velocity;
 *   - an upside-down first contact re-draws randyaw() until the body x-axis points within 60 deg of the origin (:434-437),
 *     at most 64 tries (draw site 23), instead of one uniform yaw (:616-619).
 * The thrust noise and sensor noise keep their keyed draws (same distributions in both paths); the per-drone constants of
 * qs_set_dynamics apply their rotor drag in both paths.  enable = 0 restores the default.  Call after qs_create and before the
 * first qs_reset / qs_step; later calls fail with QS_ERR_INVALID_ARG (the reference fixes use_numba in its constructor).
 * Works in every step shape. */
int qs_set_numpy_dynamics(QsHandle* h, int enable);

/* Control mode — replaces QuadrotorEnvMulti(raw_control=..., raw_control_zero_middle=...) (quadrotor_single.py:259-273):
 *   QS_CONTROL_RAW (default): RawControl(zero_action_middle=True), motor command 0.5 (clip(action, -1, 1) + 1)
 *     (quadrotor_control.py:37-57);
 *   QS_CONTROL_RAW_UNIT: RawControl(zero_action_middle=False), motor command clip(action, 0, 1) (scale 1, bias 0, :37-49);
 *   QS_CONTROL_POSITION: NonlinearPositionController with tf_control = False (:253-330), the Mellinger controller.  It
 *     ignores the action and flies each drone to its current goal from the state at the start of the control step: the
 *     desired acceleration 4.5 clamp_norm(goal - pos, 4) - 3.5 vel + (0, 0, g), the attitude error against the thrust
 *     direction with the body x-axis towards (1, 0, 0), torques -200 e_R - 50 omega, and motor commands
 *     clip(Jinv (thrust, torques), 0, 1) with Jinv = inv(quadrotor_jacobian(dynamics)) (:157-171) of each drone's
 *     constants (the Crazyflie set, or the rows of qs_set_dynamics).
 * Rewards and the wrapper statistics keep seeing the caller's raw action in every mode (quadrotor_single.py:347-349).
 * Steps with a mode other than QS_CONTROL_RAW run in the single-warp shape with the grid-wide wait, on either dynamics path.
 * Call after qs_create and before the first qs_reset / qs_step; later calls and unknown modes fail with QS_ERR_INVALID_ARG
 * (the reference fixes the controller in its constructor). */
#define QS_CONTROL_RAW 0
#define QS_CONTROL_RAW_UNIT 1
#define QS_CONTROL_POSITION 2
int qs_set_control(QsHandle* h, int mode);

/* flag bits in agent_u32[.,0] */
#define QS_FLAG_ON_FLOOR (1u << 0)
#define QS_FLAG_CRASHED_FLOOR (1u << 1)
#define QS_FLAG_CRASHED_WALL (1u << 2)
#define QS_FLAG_CRASHED_CEILING (1u << 3)
#define QS_FLAG_PREV_WALL (1u << 4)
#define QS_FLAG_PREV_CEILING (1u << 5)
#define QS_FLAG_PREV_ROOM (1u << 6)
#define QS_FLAG_PREV_OBST (1u << 7)
#define QS_FLAG_NO_COL_AGENT (1u << 8)
#define QS_FLAG_NO_COL_OBST (1u << 9)
#define QS_FLAG_REACHED_GOAL (1u << 10)
#define QS_FLAG_KICKED (1u << 11)          /* a contact response / downwash changed this env's state this step */
#define QS_FLAG_NEW_QUADCOL (1u << 12)     /* agent is in last_step_unique_collisions this step */
#define QS_FLAG_NEW_OBSTCOL (1u << 13)     /* agent is in curr_quad_col this step */

/* episode statistics of the most recently finished episode of each env:
 * env_stats_dev [E,QS_NUM_ENV_STATS] (int32), agent_stats_dev [E,N,QS_NUM_AGENT_STATS] (float) */
int qs_read_episode_stats(QsHandle* h, int32_t* env_stats_dev, float* agent_stats_dev, void* stream);

/* Launch chaining between consecutive step grids.  Off (default): every qs_step grid waits for the complete stream
 * predecessor (griddepcontrol.wait) before it touches anything — correct after ANY kernel, e.g. the policy network
 * that wrote actions_dev.  On: the caller promises that between two consecutive qs_step / qs_rollout calls of this
 * handle nothing else is enqueued on `stream` (pre-generated action rollouts, benchmarks, CUDA graphs of steps); the
 * first step after any other call of the handle still does the full wait.  Chained grids prefetch their actions before
 * the dependency wait and hand their envs over per CTA instead of waiting grid-wide: block b of a step starts as soon as
 * block b of the previous step has stored its env state — before that block has written its observation rows (DESIGN.md,
 * "Launch chaining").  The output arrays of consecutive chained steps may be the same ones (the rows of a block are
 * ordered by a second per-block word); with qs_wrap_step the wrapper kernel takes part in the same per-block protocol.
 * Environment QS_CHAINED=1 sets the initial value.
 * There is no reference counterpart (Sample Factory steps its envs from Python, one at a time). */
int qs_set_chained(QsHandle* h, int on);

/* ---- the training wrappers as kernels (SURVEY 8f-2, 8f-3) -------------------------------------------------------------
 * Replaces QuadsRewardShapingWrapper.step (swarm_rl/env_wrappers/reward_shaping.py:52-123: cumulative reward terms, action
 * statistics, true_reward, episode_extra_stats) and ExperienceReplayWrapper.step / new_episode
 * (gym_art/quadrotor_multi/quad_experience_replay.py:66-209: checkpoint every 0.5 s, the checkpoint from 1.5 s before a
 * collision goes into the env's event buffer, finished envs replay a buffered event with probability p once the drones can
 * fly, quadrotor_multi.py:281-287,356-359).  qs_wrap_step = the step kernel + ONE epilogue kernel; no host
 * synchronisation: statistics of finished episodes are accumulated on the device and fetched with qs_wrap_read whenever
 * the trainer logs.  The env "deep copy" of the reference is a copy of the env's state rows (what qs_get_state exports). */
typedef struct QsWrapConfig {
    int32_t use_replay;              /* cfg.replay_buffer_sample_prob > 0 (swarm_rl/env_wrappers/quad_utils.py:67-70) */
    int32_t replay_buffer_size;      /* events per env; the reference keeps 20 per wrapped env (quad_experience_replay.py:16-21) */
    float replay_prob;               /* replay_buffer_sample_prob */
    int32_t replay_always_active;    /* 1: skip the can_drones_fly gate (tests) */
    int32_t reserved_[4];
} QsWrapConfig;
int qs_wrap_enable(QsHandle* h, const QsWrapConfig* cfg);
/* one control step of the wrapped envs: qs_step, then the wrappers' bookkeeping for this step (rows of obs_dev of envs that
 * restart from a replayed event are overwritten with the event's observation, as ExperienceReplayWrapper.step returns it) */
int qs_wrap_step(QsHandle* h, const float* actions_dev, float* obs_dev, float* rewards_dev, uint8_t* dones_dev, void* stream);
/* the wrappers' kernel alone, on caller-supplied per-step inputs (what qs_step would have produced): actions_dev [E,N,4],
 * rew_terms_dev [E,N,QS_NUM_TERMS], dones_dev [E,N]; obs_dev [E,N,D] as in qs_wrap_step.  For callers that step the envs
 * themselves (qs_step with rew_terms_dev) and for parity tests against the reference's wrappers on recorded inputs. */
int qs_wrap_apply(QsHandle* h, const float* actions_dev, const float* rew_terms_dev, float* obs_dev, const uint8_t* dones_dev, void* stream);
/* sums over the episodes finished since the last read with reset != 0, layout QS_WA_* below; synchronises `stream`.
 * A mean statistic = its sum / the matching episode count (QS_WA_AGENT_EPISODES or QS_WA_ENV_EPISODES). */
#define QS_WRAP_AGG 149
enum {
    QS_WA_AGENT_EPISODES = 0, QS_WA_TRUE_REWARD = 1, QS_WA_RAW0 = 2, QS_WA_REW0 = 10, QS_WA_ACT_MEAN0 = 18, QS_WA_ACT_STD0 = 22,
    QS_WA_ENV_EPISODES = 26, QS_WA_ENV_STAT0 = 27, QS_WA_DIST0 = 38, QS_WA_SUCCESS = 41, QS_WA_DEADLOCK = 42, QS_WA_COL = 43,
    QS_WA_NEIGHBOR_COL = 44, QS_WA_OBST_COL = 45, QS_WA_REPLAY_ENV_EPISODES = 46, QS_WA_REPLAY_COLLISIONS = 47,
    QS_WA_REPLAY_COLLISIONS_OBST = 48, QS_WA_EPISODES_TOTAL = 49, QS_WA_REPLAYED_EVENTS = 50, QS_WA_EVENTS_STORED = 51,
    QS_WA_CHECKPOINTS = 52, QS_WA_SCN0 = 53           /* + 6 * scenario id: agent-episodes, rew_pos, rew_crash, env-episodes,
                                                         num_collisions_after_settle, distance_to_goal_1s */
};
int qs_wrap_read(QsHandle* h, float* agg_host, int reset, void* stream);
/* infos['true_reward'] of the most recently finished episode of every agent, [E,N] floats (device -> device copy) */
int qs_wrap_true_reward(QsHandle* h, float* out_dev, void* stream);

/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t qs_launch_count(const QsHandle* h);

/* Consecutive qs_step / qs_rollout launches of a handle may overlap on the GPU: a CTA of the later grid waits for the
 * CTA of the earlier grid that owns the same envs (per-block hand-over, DESIGN.md).  The wait is bounded (~1 s); this
 * returns how many waits ran into the bound since qs_create — always 0 unless the device state was corrupted.
 * A timed-out wait also latches a sticky error: every later qs_step / qs_rollout / qs_step_host of the handle returns
 * QS_ERR_CUDA.  Synchronises the device. */
int64_t qs_handover_timeouts(QsHandle* h);

#ifdef __cplusplus
}
#endif
#endif /* QUADSWARM_H_ */
