// Device-side building blocks of the QuadSwarm env step (sm_90a, fp32).
//
// Each function states the reference behaviour it reproduces (file:line under
// gym_art/quadrotor_multi/ of Zhehui-Huang/quad-swarm-rl); the float64 restatement the parity tests
// compare against is oracle/quadswarm_oracle.py.  This is a from-scratch data-parallel design:
// one thread owns one drone, the drones of an env sit in adjacent lanes of one warp, and every
// all-pairs quantity is exchanged with warp shuffles (N <= 32), never through global memory.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/quadswarm.h"
#include "qs_rng.cuh"

// Loads of mutable env state inside the step kernels.  QS_LD: always through L2 (rare paths).  ld_state<CG>: the hot
// loads; CG = true in the step-kernel instantiations that hand over per block (qs_step.cuh: no kernel boundary, hence no
// L1 invalidation, lies between the writer and the reader of a slot), plain cached loads otherwise (faster).
#define QS_LD(ptr) __ldcg(ptr)

namespace qs {

template <bool CG, typename T>
__device__ __forceinline__ T ld_state(const T* ptr) { return CG ? __ldcg(ptr) : *ptr; }

// ---- Crazyflie constants (SURVEY.md Appendix B; oracle.QuadParams; tests/golden/crazyflie_constants.json) ----
constexpr float GRAV = 9.81f;
constexpr float MASS = 0.028000000000000008f;
constexpr float INV_MASS = (float)(1.0 / 0.028000000000000008);
constexpr float IXX = 1.3669232142857143e-05f, IYY = 1.4356732142857143e-05f, IZZ = 2.656158333333334e-05f;
constexpr float INV_IXX = (float)(1.0 / 1.3669232142857143e-05), INV_IYY = (float)(1.0 / 1.4356732142857143e-05),
                INV_IZZ = (float)(1.0 / 2.656158333333334e-05);
constexpr float THRUST_MAX = 0.13047300000000003f;
constexpr float TORQUE_MAX = 0.0007828380000000002f;
constexpr float PROP_ARM_XY = 0.0325f;            // |prop_crossproducts| components, quadrotor_dynamics.py:141
constexpr float ARM = 0.04596194077712559f;       // quadrotor_dynamics.py:158 (also the njit floor threshold, :378)
constexpr float MOTOR_TAU_UP = 0.13333244445037035f, MOTOR_TAU_DOWN = 0.13333244445037035f;
constexpr float OMEGA_MAX = 40.0f;
constexpr float FLOOR_MU = 0.6f;
// QS_NUMPY_DYNAMICS = 1 (set by qs_step_npy.cu only): the floor model of the reference's numpy path (use_numba=False;
// QuadrotorDynamics.floor_interaction, quadrotor_dynamics.py:389-457) in physics_substep().
#ifndef QS_NUMPY_DYNAMICS
#define QS_NUMPY_DYNAMICS 0
#endif
#if QS_NUMPY_DYNAMICS
constexpr float FLOOR_THRESHOLD_NP = 0.05f;       // floor threshold and snap height of the numpy path, every model (:75)
#endif
// QS_CONTROL_MODES = 1 (set by qs_step_pc.cu only): the step maps actions to motor commands by StepParams.control
// (QS_CONTROL_RAW_UNIT or QS_CONTROL_POSITION, position_control() below) instead of RawControl with zero_action_middle.
#ifndef QS_CONTROL_MODES
#define QS_CONTROL_MODES 0
#endif
constexpr float SIM_DT = 0.005f;                  // quadrotor_single.py:157
constexpr float CONTROL_DT = 0.01f;               // quadrotor_multi.py:83
constexpr int SIM_STEPS = 2;                      // quadrotor_single.py:102
constexpr int SVD_PERIOD = 100;                   // sub-steps between re-orthogonalisations: the float64 accumulator
                                                  // of quadrotor_dynamics.py:547-551 first exceeds 0.5 on its 100th += 0.005
constexpr float OU_THETA = 0.15f, OU_SIGMA = 0.01f;   // float32 in the reference too (numba_utils.py:69-71)
constexpr float POS_NOISE_STD = 0.005f, VEL_NOISE_STD = 0.01f, GYRO_NOISE_STD = 0.000175f;   // sensor_noise.py:70-76
constexpr float EPS_DYN = 1e-6f;                  // quadrotor_dynamics.py:13
constexpr float EPS_COL = 1e-5f;                  // quad_utils.py:10
constexpr float PI_F = 3.14159265358979323846f;
constexpr float VXYZ_MAX = 3.0f;                  // quadrotor_dynamics.py:50 (neighbour rel-vel clip = 2x, quadrotor_single.py:295)

// ---- state slots: struct-of-arrays of float4, slot-major [NUM_SLOTS][A_pad] -> one LDG.128 per slot per thread ----
enum Slot {
    SL_POS_VX = 0,   // pos.xyz, vel.x
    SL_V_OM,         // vel.y, vel.z, omega.x, omega.y
    SL_OM_R0,        // omega.z, R00, R01, R02
    SL_R1_R20,       // R10, R11, R12, R20
    SL_R2_FLAGS,     // R21, R22, flags(u32), prev_collision_row(u32)
    SL_ROT_DAMP,     // thrust_rot_damp[4]
    SL_CMDS_DAMP,    // thrust_cmds_damp[4]
    SL_OU,           // OU noise state[4]
    SL_DIST_RING,    // previous 4 goal distances, newest first
    NUM_RW_SLOTS,    // ---- slots above are read+written every step ----
    SL_GOAL = NUM_RW_SLOTS,   // goal.xyz, 0   (read every step, written by reset / set_goals)
    SL_DIST_SUMS,    // running sums of the goal distance over the last 1 s / 3 s / 5 s of the episode
    SL_STALE_VEL,    // QuadrotorEnvMulti.self.vel as a reset following a reset would see it (Appendix D-6)
    NUM_SLOTS
};

struct DevState {
    float4* slots;          // [NUM_SLOTS][A_pad]
    long long a_pad;
    int4* env_ctr;          // [E] tick, step_count, svd_count, episode_idx
    int32_t* env_cnt;       // [E][QS_NUM_ENV_STATS] running episode counters
    float2* obst;           // [E][M]
    float4* next_goal;      // [A]  host tables: goal; device-generated record: goal, w = cos(yaw) of the spawn pose
    float4* next_spawn;     // [A]  host tables: spawn point (w = 1: use it, w = 0: spawn at the goal); record: final spawn
                            //      position (jitter applied), w = sin(yaw)
    float2* next_obst;      // [E][M]
    int32_t* stats_env;     // [E][QS_NUM_ENV_STATS]  latched at episode end
    float4* stats_agent;    // [A]                     latched at episode end
    int* ready;             // [E + 1] per step-kernel block: 1 = the block's env state is complete in L2 (per-block hand-over);
                            //         ready[E] counts hand-over waits that timed out
    int2* epi;              // [E] x = number of the episode the env is running (every reset, explicit or automatic, starts the
                            //     next one; keys the episode-generation draws), y = episode number the next-episode RECORD
                            //     (next_goal / next_spawn / next_obst / next_scn_*) was generated for, 0 = none (qs_pregen_kernel)
    int4* next_scn_i;       // [E]     scenario state of the pre-generated next episode
    float4* next_scn_f;     // [E][3]
    float4* dyn;            // [A][QS_DYN_ROW / 4] per-drone physical constants (qs_set_dynamics), or null: Crazyflie constants
    float4* next_dyn;       // [A][QS_DYN_ROW / 4] constants latched by the env's next (auto-)reset when dyn_pending[env] != 0;
                            //     dynamics sampler: the rows qs_dyn_pregen_kernel prepared for episode dyn_pending[E + env]
    int* dyn_pending;       // [E]; dynamics sampler: [2][E], row 0 always 0 (the step and reset kernels latch nothing),
                            //     row 1 the episode whose rows next_dyn holds, 0 = none
    int* err_flag;          // mapped page-locked host word: set to 1 by a step kernel whose hand-over wait timed out (sticky)
    int4* scn_i;            // [E]     device-side scenario state: scenario, period, next event tick, formation | growing << 8
    float4* scn_f;          // [E][3]  formation size / layer distance / largest size / speed; centre 1; centre 2
};

// Custom sensor-noise model (qs_set_sensor_noise); read only by the NZ kernel instantiations.  bias_pi / bias_sigma are the
// per-observation factors of add_noise_to_omega (sensor_noise.py:224-229), computed on the host in float64.
struct NoiseModel {
    float pos_std, pos_range, vel_std, vel_range, gyro_std, quat_std, quat_range;
    float bias_pi, bias_sigma, random_walk;
    int rot;                // quat_std or quat_range != 0: the observed rotation is perturbed
};

// qs_set_dynamics_sampler's arguments, in device memory (read only at resampling resets)
struct DynSampler {
    QsDynSampler spec;
    int every;              // randomize_every: resample at the reset that starts episode g when g % every == 0; 0 = never
};

struct StepParams {
    alignas(64) unsigned char obs_map[128];     // CUtensorMap of the caller's observation array (obs_bulk == 1), see quadswarm.cu
    DevState st;
    const float4* actions;  // [T][A]
    float* obs;             // [T][A][D] or [A][D]
    float* rewards;         // [T][A]
    uint8_t* dones;         // [T][A]
    float* rew_terms;       // [T][A][QS_NUM_TERMS] or null
    const uint8_t* env_mask;    // reset / set_state kernels only
    int E, N, K, D, S, M;
    int obs_repr, use_obst, use_downwash, sense_noise;
    int ep_len, T, last_obs_only;
    float room_lo[3], room_hi[3];
    float col_thr, falloff_thr, obst_radius, obst_col_thr, obst_half_size;
    float col_thr2, falloff_thr2, quad_arm;     // col_thr^2, falloff_thr^2, obst_col_thr - obst_half_size: kernel operands, not registers
    float grace_steps, final_steps, approach_metric;
    float rew[QS_NUM_REW_COEFF];
    uint32_t seed_lo, seed_hi;
    int env_id_offset;
    // observation staging (coalesced write-out): vector width V, Q = D / V, padded row stride Dp, magic = ceil(2^20 / Q)
    int obs_stage, obs_v, obs_q, obs_dp, obs_magic, smem_tile_off;
    int obs_bulk;                       // write-out of the staged tile: 0 vector stores, 1 one TMA tensor store per warp tile
                                        // (obs_map, D % 4 == 0), 2 one linear cp.async.bulk per warp tile (unpadded rows)
#ifdef QS_TIMELINE
    unsigned long long* tl;             // debug build only: [64 slots][4096 blocks][8] %globaltimer stamps of warp 0 of every block
    int tl_slot;
#endif
    // per-episode pillar density / size randomisation (qs_set_obstacle_randomization): the number of pillars and their radius
    // are drawn per env at every reset from these lists; the env's values live in scn_f[3 env].xy (radius, count)
    int obst_random, n_obst_counts, n_obst_radii;
    int obst_counts[QS_MAX_OBST_CHOICES];
    float obst_radii[QS_MAX_OBST_CHOICES];
    int chained;                        // 1: the stream predecessor of this launch is a step grid of the same handle (qs_set_chained):
                                        //    actions are prefetched before the dependency wait; hand-over kernels skip the grid-wide wait
    int courier;            // per-block hand-over with a courier warp (last warp of the block, no envs): early release of the state
    int wrap_chain;         // courier launch inside qs_wrap_step: block-chained with the wrapper kernel (see qs_wrap_kernel)
    int scenario, grid_l, grid_w;       // QS_SCENARIO_*, pillar grid cells along x / y
    NoiseModel nz;                      // custom sensor-noise model (NZ instantiations)
    float4* gyro_bias;                  // [A] xyz: gyro bias of the stateful gyro model (qs_set_sensor_noise), or null: model off
                                        // (not in DevState: the scenario functions take that by value)
    int init_random;                    // qs_set_init_random_state: every spawn gets a random vel / omega / R (random_init_state)
    float init_vel_max, init_omega_max;
    int control;                        // qs_set_control: QS_CONTROL_*; read only by the kernels of qs_step_pc.cu
    const DynSampler* dyn;              // qs_set_dynamics_sampler (qs_dyn_sampler.cuh), or null; read only by the
                                        // sampler's kernels (quadswarm.cu).  It takes the last 8 bytes of the
                                        // struct's padding: every other kernel keeps its parameter layout.
};

struct Agent {
    float pos[3], vel[3], R[9], om[3];
    float rd[4], cd[4], ou[4];
    float goal[3];
    float ring[4];
    uint32_t flags, prev_col;
};

// ---- small helpers ----
struct V3 { float x, y, z; };
struct KickVO { V3 vel; V3 dom; };         // new velocity, delta omega
struct PairOut { V3 v1, v2, dom; };        // new velocities of both drones, +/- delta omega
struct ResetPose { V3 pos; float cs, sn; };
struct Noise9 { float p[3], v[3], w[3]; }; // scaled sensor noise: position, velocity, gyro

__device__ __forceinline__ float clampf(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
__device__ __forceinline__ float norm3(float x, float y, float z) { return fsqrt(x * x + y * y + z * z); }

template <int NP>
__device__ __forceinline__ float shfl(float v, int src) { return __shfl_sync(0xffffffffu, v, src, NP); }
template <int NP>
__device__ __forceinline__ uint32_t shfl_u(uint32_t v, int src) { return __shfl_sync(0xffffffffu, v, src, NP); }
template <int NP>
__device__ __forceinline__ uint32_t group_ballot(bool pred) {
    const uint32_t b = __ballot_sync(0xffffffffu, pred);
    if (NP == 32) return b;
    const int base = (threadIdx.x & 31) & ~(NP - 1);
    return (b >> base) & ((1u << (NP & 31)) - 1u);
}

template <bool CG = false>
__device__ __forceinline__ void load_agent(const DevState& st, long long a, Agent& s) {
    const float4* p = st.slots + a;
    const float4 q0 = ld_state<CG>(p + SL_POS_VX * st.a_pad), q1 = ld_state<CG>(p + SL_V_OM * st.a_pad),
                 q2 = ld_state<CG>(p + SL_OM_R0 * st.a_pad), q3 = ld_state<CG>(p + SL_R1_R20 * st.a_pad),
                 q4 = ld_state<CG>(p + SL_R2_FLAGS * st.a_pad), q5 = ld_state<CG>(p + SL_ROT_DAMP * st.a_pad),
                 q6 = ld_state<CG>(p + SL_CMDS_DAMP * st.a_pad), q7 = ld_state<CG>(p + SL_OU * st.a_pad),
                 q8 = ld_state<CG>(p + SL_DIST_RING * st.a_pad), q9 = ld_state<CG>(p + SL_GOAL * st.a_pad);
    s.pos[0] = q0.x; s.pos[1] = q0.y; s.pos[2] = q0.z; s.vel[0] = q0.w;
    s.vel[1] = q1.x; s.vel[2] = q1.y; s.om[0] = q1.z; s.om[1] = q1.w;
    s.om[2] = q2.x; s.R[0] = q2.y; s.R[1] = q2.z; s.R[2] = q2.w;
    s.R[3] = q3.x; s.R[4] = q3.y; s.R[5] = q3.z; s.R[6] = q3.w;
    s.R[7] = q4.x; s.R[8] = q4.y; s.flags = __float_as_uint(q4.z); s.prev_col = __float_as_uint(q4.w);
    s.rd[0] = q5.x; s.rd[1] = q5.y; s.rd[2] = q5.z; s.rd[3] = q5.w;
    s.cd[0] = q6.x; s.cd[1] = q6.y; s.cd[2] = q6.z; s.cd[3] = q6.w;
    s.ou[0] = q7.x; s.ou[1] = q7.y; s.ou[2] = q7.z; s.ou[3] = q7.w;
    s.ring[0] = q8.x; s.ring[1] = q8.y; s.ring[2] = q8.z; s.ring[3] = q8.w;
    s.goal[0] = q9.x; s.goal[1] = q9.y; s.goal[2] = q9.z;
}

__device__ __forceinline__ void store_agent(const DevState& st, long long a, const Agent& s, bool store_goal) {
    float4* p = st.slots + a;
    p[SL_POS_VX * st.a_pad] = make_float4(s.pos[0], s.pos[1], s.pos[2], s.vel[0]);
    p[SL_V_OM * st.a_pad] = make_float4(s.vel[1], s.vel[2], s.om[0], s.om[1]);
    p[SL_OM_R0 * st.a_pad] = make_float4(s.om[2], s.R[0], s.R[1], s.R[2]);
    p[SL_R1_R20 * st.a_pad] = make_float4(s.R[3], s.R[4], s.R[5], s.R[6]);
    p[SL_R2_FLAGS * st.a_pad] = make_float4(s.R[7], s.R[8], __uint_as_float(s.flags), __uint_as_float(s.prev_col));
    p[SL_ROT_DAMP * st.a_pad] = make_float4(s.rd[0], s.rd[1], s.rd[2], s.rd[3]);
    p[SL_CMDS_DAMP * st.a_pad] = make_float4(s.cd[0], s.cd[1], s.cd[2], s.cd[3]);
    p[SL_OU * st.a_pad] = make_float4(s.ou[0], s.ou[1], s.ou[2], s.ou[3]);
    p[SL_DIST_RING * st.a_pad] = make_float4(s.ring[0], s.ring[1], s.ring[2], s.ring[3]);
    if (store_goal) p[SL_GOAL * st.a_pad] = make_float4(s.goal[0], s.goal[1], s.goal[2], 0.f);
}

// state of a lane without a drone: at rest, level, and far from every other lane (it takes part in the shuffles of its warp)
__device__ __forceinline__ void idle_agent(Agent& s, int i) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { s.pos[k] = 1e9f + 1e6f * i; s.vel[k] = 0.f; s.om[k] = 0.f; s.goal[k] = 0.f; }
#pragma unroll
    for (int k = 0; k < 9; ++k) s.R[k] = (k % 4 == 0) ? 1.f : 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) { s.rd[k] = 0.f; s.cd[k] = 0.f; s.ou[k] = 0.f; s.ring[k] = 0.f; }
    s.flags = 0u; s.prev_col = 0u;
}

// new velocity and body-rate increment of a contact response (obstacle, wall, ceiling)
__device__ __forceinline__ void apply_kick(Agent& s, const KickVO& o) {
    s.vel[0] = o.vel.x; s.vel[1] = o.vel.y; s.vel[2] = o.vel.z;
    s.om[0] += o.dom.x; s.om[1] += o.dom.y; s.om[2] += o.dom.z;
}

// R -> pure yaw (quadrotor_dynamics.py:579-581, :614-621): theta = atan2(R10, R00 + eps), then (cos, sin) of it.
// cos(atan2(y, x)) = x / hypot, so no trigonometry is needed; atan2(0, 0) = 0 gives the identity.
__device__ __forceinline__ void yaw_only(float R[9]) {
    const float x = R[0] + EPS_DYN, y = R[3];
    const float h2 = x * x + y * y;
    float c = 1.f, s = 0.f;
    if (h2 > 0.f) {
        const float inv = frsqrt(h2);
        c = x * inv; s = y * inv;
    }
    R[0] = c; R[1] = -s; R[2] = 0.f; R[3] = s; R[4] = c; R[5] = 0.f; R[6] = 0.f; R[7] = 0.f; R[8] = 1.f;
}

// Nearest orthogonal matrix (polar factor) = U V^T of the SVD the reference takes every 0.5 s
// (quadrotor_dynamics.py:547-551).  R is orthogonal to rounding on entry, so two Newton steps
// X <- (X + X^-T) / 2 reach fp32 precision; no LAPACK-style SVD is needed on the device.
struct M3 { float m[9]; };
__device__ __noinline__ M3 orthonormalize(M3 in) {
    float* R = in.m;
#pragma unroll 1
    for (int it = 0; it < 2; ++it) {
        const float c00 = R[4] * R[8] - R[5] * R[7], c01 = R[5] * R[6] - R[3] * R[8], c02 = R[3] * R[7] - R[4] * R[6];
        const float c10 = R[2] * R[7] - R[1] * R[8], c11 = R[0] * R[8] - R[2] * R[6], c12 = R[1] * R[6] - R[0] * R[7];
        const float c20 = R[1] * R[5] - R[2] * R[4], c21 = R[2] * R[3] - R[0] * R[5], c22 = R[0] * R[4] - R[1] * R[3];
        const float det = R[0] * c00 + R[1] * c01 + R[2] * c02;
        const float h = 0.5f / det;     // X^-T = cofactor / det
        R[0] = 0.5f * R[0] + h * c00; R[1] = 0.5f * R[1] + h * c01; R[2] = 0.5f * R[2] + h * c02;
        R[3] = 0.5f * R[3] + h * c10; R[4] = 0.5f * R[4] + h * c11; R[5] = 0.5f * R[5] + h * c12;
        R[6] = 0.5f * R[6] + h * c20; R[7] = 0.5f * R[7] + h * c21; R[8] = 0.5f * R[8] + h * c22;
    }
    return in;
}

// cold half of the floor contact: upside-down first contact draws a random yaw (quadrotor_dynamics.py:616-619)
__device__ __noinline__ float2 floor_random_yaw(RngKey key, int i, int sub) {
    const float4 u = rng_uniform4(key, SITE_FLOOR_YAW, i, 0, 0);
    const float th = -PI_F + (PI_F - (-PI_F)) * (sub == 0 ? u.x : u.y);
    float s, c;
    sincosf(th, &s, &c);
    return make_float2(c, s);
}

#if QS_NUMPY_DYNAMICS
__device__ __noinline__ float2 floor_yaw_numpy(RngKey key, int i, int sub, float x, float y);      // below

// Sliding-friction direction of the numpy path, (cos, sin)(atan2(-vy, -vx)) (quadrotor_dynamics.py:419-422), from the njit
// path's (ca, sa) = v_xy / |v_xy|: the friction is subtracted along the velocity there, so it pushes the drone on.  With no
// horizontal velocity atan2 sees signed zeros: atan2(-0, -0) = -pi for vx = +0 (direction (-1, 0)), atan2(-0, +0) = -0 for
// vx = -0 (direction (1, 0)); the sin(-pi) = -1.2e-16 of the first is dropped.
__device__ __forceinline__ void friction_dir_numpy(float vx, float h2, float& ca, float& sa) {
    if (h2 > 0.f) { ca = -ca; sa = -sa; }
    else ca = copysignf(1.f, -vx);
}
#endif

// ---- per-drone physical constants (SURVEY 8f-4: dynamics randomisation, non-Crazyflie models, rotor drag) ----
// Row layout = QS_DYN_* of include/quadswarm.h = quad_models.DYN_FIELDS: what QuadrotorDynamics.update_model derives
// (quadrotor_dynamics.py:104-166).  Kernels instantiated with DYN = false keep the compile-time Crazyflie constants above.
struct Phys {
    float mass, inv_mass, ixx, iyy, izz, inv_ixx, inv_iyy, inv_izz;
    float thrust_max[4], torque_max[4];
    float px[4], py[4], pz[4];
    float tau_up, tau_down, linearity, ou_sigma, c_drag, c_roll, vel_damp, omega_quadratic, arm;
};

__device__ __forceinline__ void load_phys(const float4* rows, long long a, Phys& ph) {
    const float4* r = rows + a * (QS_DYN_ROW / 4);
    const float4 q0 = QS_LD(r + 0), q1 = QS_LD(r + 1), q2 = QS_LD(r + 2), q3 = QS_LD(r + 3), q4 = QS_LD(r + 4), q5 = QS_LD(r + 5),
                 q6 = QS_LD(r + 6), q7 = QS_LD(r + 7), q8 = QS_LD(r + 8), q9 = QS_LD(r + 9);
    ph.mass = q0.x; ph.inv_mass = q0.y; ph.ixx = q0.z; ph.iyy = q0.w;
    ph.izz = q1.x; ph.inv_ixx = q1.y; ph.inv_iyy = q1.z; ph.inv_izz = q1.w;
    ph.thrust_max[0] = q2.x; ph.thrust_max[1] = q2.y; ph.thrust_max[2] = q2.z; ph.thrust_max[3] = q2.w;
    ph.torque_max[0] = q3.x; ph.torque_max[1] = q3.y; ph.torque_max[2] = q3.z; ph.torque_max[3] = q3.w;
    ph.px[0] = q4.x; ph.py[0] = q4.y; ph.px[1] = q4.z; ph.py[1] = q4.w;
    ph.px[2] = q5.x; ph.py[2] = q5.y; ph.px[3] = q5.z; ph.py[3] = q5.w;
    ph.pz[0] = q6.x; ph.pz[1] = q6.y; ph.pz[2] = q6.z; ph.pz[3] = q6.w;
    ph.tau_up = q7.x; ph.tau_down = q7.y; ph.linearity = q7.z; ph.ou_sigma = q7.w;
    ph.c_drag = q8.x; ph.c_roll = q8.y; ph.vel_damp = q8.z; ph.omega_quadratic = q8.w;
    ph.arm = q9.x;
}

#if QS_CONTROL_MODES
// inv(quadrotor_jacobian(dynamics)) (quadrotor_control.py:157-171, :257-258), in float64 like np.linalg.inv.  J maps the
// normalised motor thrusts to (acceleration along the body z-axis, angular accelerations):
//   J[0][k] = thrust_max_k / mass, J[1][k] = thrust_max_k py_k / Ixx, J[2][k] = -thrust_max_k px_k / Iyy,
//   J[3][k] = torque_max_k prop_ccw_k / Izz, prop_ccw = (-1, 1, -1, 1) (quadrotor_dynamics.py:47).
// DYN = false: the compile-time Crazyflie constants (the compiler folds the inverse); DYN = true: the drone's row, so a row
// latched at a reset is inverted from the next step on.  The inverse is the adjugate over the determinant: J of an
// X-frame has zero leading minors, which Gauss-Jordan elimination would have to pivot around.
template <bool DYN>
__device__ __forceinline__ void jacobian_inverse(const Phys& ph, double Ji[16]) {
    constexpr float CF_PX[4] = {PROP_ARM_XY, -PROP_ARM_XY, -PROP_ARM_XY, PROP_ARM_XY};
    constexpr float CF_PY[4] = {-PROP_ARM_XY, -PROP_ARM_XY, PROP_ARM_XY, PROP_ARM_XY};
    double m[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double tm = DYN ? ph.thrust_max[k] : THRUST_MAX, qm = DYN ? ph.torque_max[k] : TORQUE_MAX;
        const double px = DYN ? ph.px[k] : CF_PX[k], py = DYN ? ph.py[k] : CF_PY[k];
        m[0][k] = tm / (double)(DYN ? ph.mass : MASS);
        m[1][k] = tm * py / (double)(DYN ? ph.ixx : IXX);
        m[2][k] = -tm * px / (double)(DYN ? ph.iyy : IYY);
        m[3][k] = ((k & 1) ? qm : -qm) / (double)(DYN ? ph.izz : IZZ);
    }
    // 2 x 2 minors of rows 0-1 (s) and rows 2-3 (c)
    const double s0 = m[0][0] * m[1][1] - m[1][0] * m[0][1], s1 = m[0][0] * m[1][2] - m[1][0] * m[0][2];
    const double s2 = m[0][0] * m[1][3] - m[1][0] * m[0][3], s3 = m[0][1] * m[1][2] - m[1][1] * m[0][2];
    const double s4 = m[0][1] * m[1][3] - m[1][1] * m[0][3], s5 = m[0][2] * m[1][3] - m[1][2] * m[0][3];
    const double c5 = m[2][2] * m[3][3] - m[3][2] * m[2][3], c4 = m[2][1] * m[3][3] - m[3][1] * m[2][3];
    const double c3 = m[2][1] * m[3][2] - m[3][1] * m[2][2], c2 = m[2][0] * m[3][3] - m[3][0] * m[2][3];
    const double c1 = m[2][0] * m[3][2] - m[3][0] * m[2][2], c0 = m[2][0] * m[3][1] - m[3][0] * m[2][1];
    const double inv_det = 1.0 / (s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0);
    Ji[0] = (m[1][1] * c5 - m[1][2] * c4 + m[1][3] * c3) * inv_det;
    Ji[1] = (-m[0][1] * c5 + m[0][2] * c4 - m[0][3] * c3) * inv_det;
    Ji[2] = (m[3][1] * s5 - m[3][2] * s4 + m[3][3] * s3) * inv_det;
    Ji[3] = (-m[2][1] * s5 + m[2][2] * s4 - m[2][3] * s3) * inv_det;
    Ji[4] = (-m[1][0] * c5 + m[1][2] * c2 - m[1][3] * c1) * inv_det;
    Ji[5] = (m[0][0] * c5 - m[0][2] * c2 + m[0][3] * c1) * inv_det;
    Ji[6] = (-m[3][0] * s5 + m[3][2] * s2 - m[3][3] * s1) * inv_det;
    Ji[7] = (m[2][0] * s5 - m[2][2] * s2 + m[2][3] * s1) * inv_det;
    Ji[8] = (m[1][0] * c4 - m[1][1] * c2 + m[1][3] * c0) * inv_det;
    Ji[9] = (-m[0][0] * c4 + m[0][1] * c2 - m[0][3] * c0) * inv_det;
    Ji[10] = (m[3][0] * s4 - m[3][1] * s2 + m[3][3] * s0) * inv_det;
    Ji[11] = (-m[2][0] * s4 + m[2][1] * s2 - m[2][3] * s0) * inv_det;
    Ji[12] = (-m[1][0] * c3 + m[1][1] * c1 - m[1][2] * c0) * inv_det;
    Ji[13] = (m[0][0] * c3 - m[0][1] * c1 + m[0][2] * c0) * inv_det;
    Ji[14] = (-m[3][0] * s3 + m[3][1] * s1 - m[3][2] * s0) * inv_det;
    Ji[15] = (m[2][0] * s3 - m[2][1] * s1 + m[2][2] * s0) * inv_det;
}

// normalize(), quad_utils.py:80-86: x / |x|, or x unchanged when |x| < 1e-5
__device__ __forceinline__ void normalize3(float v[3]) {
    const float n = norm3(v[0], v[1], v[2]);
    if (n >= 1e-5f) { v[0] /= n; v[1] /= n; v[2] /= n; }
}

// NonlinearPositionController.step, quadrotor_control.py:282-330 (tf_control = False): the motor commands that fly the drone
// towards its goal, from its state at the start of the control step.  The action is not read.
template <bool DYN>
__device__ __forceinline__ void position_control(const Agent& s, const Phys& ph, float cmd[4]) {
    float acc[3] = {s.goal[0] - s.pos[0], s.goal[1] - s.pos[1], s.goal[2] - s.pos[2]};
    const float gd = norm3(acc[0], acc[1], acc[2]);
    const float sc = gd <= 4.f ? 1.f : 4.f / gd;                             // -e_p = clamp_norm(goal - pos, 4.0), :287
#pragma unroll
    for (int k = 0; k < 3; ++k) acc[k] = 4.5f * (sc * acc[k]) - 3.5f * s.vel[k];   // kp_p = 4.5, kd_p = 3.5, :266, :290
    acc[2] += GRAV;
    float zb[3] = {acc[0], acc[1], acc[2]};
    normalize3(zb);
    float yb[3] = {0.f, zb[2], -zb[1]};                                       // cross(zb, rot_des[:, 0] = (1, 0, 0))
    normalize3(yb);
    const float xb[3] = {yb[1] * zb[2] - yb[2] * zb[1], yb[2] * zb[0] - yb[0] * zb[2], yb[0] * zb[1] - yb[1] * zb[0]};
    // e_R = 0.5 vee(R_des^T R - R^T R_des); with A = R_des^T R, A_ij = (column i of R_des) . (column j of R)
    auto rcol = [&](const float d[3], int j) { return d[0] * s.R[j] + d[1] * s.R[3 + j] + d[2] * s.R[6 + j]; };
    const float e0 = 0.5f * (rcol(zb, 1) - rcol(yb, 2));
    const float e1 = 0.5f * (rcol(xb, 2) - rcol(zb, 0));
    const float e2 = 0.2f * (0.5f * (rcol(yb, 0) - rcol(xb, 1)));              // e_R[2] *= 0.2, :315
    const float des[4] = {acc[0] * s.R[2] + acc[1] * s.R[5] + acc[2] * s.R[8],   // thrust_mag = acc_des . R[:, 2], :320
                          -200.f * e0 - 50.f * s.om[0], -200.f * e1 - 50.f * s.om[1], -200.f * e2 - 50.f * s.om[2]};
    double Ji[16];
    jacobian_inverse<DYN>(ph, Ji);
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const double t = Ji[4 * r] * des[0] + Ji[4 * r + 1] * des[1] + Ji[4 * r + 2] * des[2] + Ji[4 * r + 3] * des[3];
        cmd[r] = clampf((float)t, 0.f, 1.f);                                   // :325-327
    }
}
#endif

// One 5 ms physics sub-step of the njit path: step1_numba, quadrotor_dynamics.py:348-383
// (calculate_torque_integrate_rotations_and_update_omega :497-566, room clip :360-367,
//  floor_interaction_numba :569-639, compute_velocity_and_acceleration :642-649).
// `cmd` is the RawControl output in [0,1]; the OU state s.ou is the thrust noise of this control step.
// DYN = false: the compile-time Crazyflie constants; `ph` is not read.  DYN = true: the per-drone constants `ph` — general
// motor asymmetry / linearity / propeller positions / damping — plus the rotor-drag and rolling-moment term that only the
// reference's numpy path has (step1, quadrotor_dynamics.py:256-289; all shipped models have C_drag = C_roll = 0).
// The Crazyflie arms are not the general formulas with constant values: IEEE arithmetic does not fold terms such as
// (1 - linearity) cd^2 or 1 - clamp(0 ox^2) away, so those would change the default kernels' arithmetic.
// QS_NUMPY_DYNAMICS: the floor model of the numpy path instead (floor_interaction, :389-457).
template <bool DYN, bool FMA_FRICTION>
__device__ __forceinline__ void physics_substep(Agent& s, const float cmd[4], bool do_svd, const StepParams& p,
                                                const RngKey& key, int i, int sub, const Phys& ph) {
    static_assert(!(DYN && FMA_FRICTION), "the fused friction form is written with the Crazyflie mass");
    float thr[4];
    float tq0, tq1, tq2, thrust_z;
    float drag_fx = 0.f, drag_fy = 0.f, drag_fz = 0.f;      // body-frame rotor drag (DYN)
    if constexpr (DYN) {
        tq0 = 0.f; tq1 = 0.f; tq2 = 0.f; thrust_z = 0.f;
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const float c = cmd[m];
            const float tau = fminf((c < s.cd[m]) ? ph.tau_down : ph.tau_up, 1.f);
            s.rd[m] = tau * (fsqrt(c) - s.rd[m]) + s.rd[m];
            s.cd[m] = clampf(s.rd[m] * s.rd[m] + c * s.ou[m], 0.f, 1.f);
            thr[m] = ph.thrust_max[m] * ((1.f - ph.linearity) * s.cd[m] * s.cd[m] + ph.linearity * s.cd[m]);   // numba_utils.py:58-60
            // prop_crossproducts = cross(prop_pos, z) = (py, -px, 0) (quadrotor_dynamics.py:141); prop_ccw = (-1, 1, -1, 1)
            tq0 += ph.py[m] * thr[m];
            tq1 += -ph.px[m] * thr[m];
            tq2 += ((m & 1) ? 1.f : -1.f) * ph.torque_max[m] * s.cd[m];
            thrust_z += thr[m];
        }
        if (ph.c_drag != 0.f || ph.c_roll != 0.f) {
            // body-frame velocity of every rotor hub, projected on the rotor plane
            const float vbx = s.R[0] * s.vel[0] + s.R[3] * s.vel[1] + s.R[6] * s.vel[2];
            const float vby = s.R[1] * s.vel[0] + s.R[4] * s.vel[1] + s.R[7] * s.vel[2];
            const float vbz = s.R[2] * s.vel[0] + s.R[5] * s.vel[1] + s.R[8] * s.vel[2];
            float tx = 0.f, ty = 0.f, tz = 0.f;
#pragma unroll
            for (int m = 0; m < 4; ++m) {
                const float vrx = vbx + (s.om[1] * ph.pz[m] - s.om[2] * ph.py[m]);       // v + omega x prop_pos
                const float vry = vby + (s.om[2] * ph.px[m] - s.om[0] * ph.pz[m]);
                const float sq = sqrtf(s.cd[m]);
                const float fix = -ph.c_drag * sq * vrx, fiy = -ph.c_drag * sq * vry;     // drag force of rotor m (z component 0)
                drag_fx += fix; drag_fy += fiy;
                // torque = f_i x prop_pos, plus the rolling moment -C_roll ccw sqrt(c) v_rotor
                tx += fiy * ph.pz[m]; ty += -fix * ph.pz[m]; tz += fix * ph.py[m] - fiy * ph.px[m];
                const float ccw = (m & 1) ? 1.f : -1.f;
                tx += -ph.c_roll * ccw * sq * vrx; ty += -ph.c_roll * ccw * sq * vry;
            }
            const float dt2 = 2.f * SIM_DT;
            const float vel_norm = norm3(vbx, vby, vbz);
            const float rdf = sqrtf(drag_fx * drag_fx + drag_fy * drag_fy);
            if (rdf > EPS_DYN) {
                const float sc = fminf(rdf, vel_norm * ph.mass / dt2) / rdf;
                drag_fx *= sc; drag_fy *= sc;
            }
            const float rvt = sqrtf(tx * tx + ty * ty + tz * tz);
            if (rvt > EPS_DYN) {
                const float lim = norm3(s.om[0] * ph.ixx, s.om[1] * ph.iyy, s.om[2] * ph.izz) / dt2;
                const float sc = fminf(rvt, lim) / rvt;
                tx *= sc; ty *= sc; tz *= sc;
            }
            tq0 += tx; tq1 += ty; tq2 += tz;
        }
    } else {
        // motor lag on sqrt(thrust) + OU thrust noise (:504-517); linearity = 1 so thrust = thrust_max * cmds_damp
#pragma unroll
        for (int m = 0; m < 4; ++m) {
            const float c = cmd[m];                       // already in [0,1]; the second np.clip (:504) is a no-op
            const float tau = fminf((c < s.cd[m]) ? MOTOR_TAU_DOWN : MOTOR_TAU_UP, 1.f);
            s.rd[m] = tau * (fsqrt(c) - s.rd[m]) + s.rd[m];
            s.cd[m] = clampf(s.rd[m] * s.rd[m] + c * s.ou[m], 0.f, 1.f);
            thr[m] = THRUST_MAX * s.cd[m];
        }
        // torques: prop_crossproducts x thrust, plus rotor reaction torque about z (:520-526); rotor drag is zero (:529)
        tq0 = PROP_ARM_XY * ((thr[2] + thr[3]) - (thr[0] + thr[1]));
        tq1 = PROP_ARM_XY * ((thr[1] + thr[2]) - (thr[0] + thr[3]));
        tq2 = TORQUE_MAX * ((s.cd[1] + s.cd[3]) - (s.cd[0] + s.cd[2]));
        thrust_z = (thr[0] + thr[1]) + (thr[2] + thr[3]);
    }

    // Rodrigues rotation by the world-frame angular velocity w (:537-544):
    //   R <- (I + sin(t) K + (1 - cos(t)) K^2) R,  K = [w]x / |w|,  t = |w| dt
    // written as R + a (w x r) + b (w (w.r) - r |w|^2) per column r, with a = dt sin(t)/t and b = dt^2 (1-cos t)/t^2
    // evaluated as polynomials in t^2 (t <= 40 sqrt(3) dt = 0.35): no sqrt, no division, exact identity at w = 0
    // (the reference skips the update when |w| == 0).
    {
        const float wx = s.R[0] * s.om[0] + s.R[1] * s.om[1] + s.R[2] * s.om[2];
        const float wy = s.R[3] * s.om[0] + s.R[4] * s.om[1] + s.R[5] * s.om[2];
        const float wz = s.R[6] * s.om[0] + s.R[7] * s.om[1] + s.R[8] * s.om[2];
        const float w2 = wx * wx + wy * wy + wz * wz;
        const float t2 = w2 * (SIM_DT * SIM_DT);
        const float ca = SIM_DT * (1.f + t2 * (-1.f / 6.f + t2 * (1.f / 120.f + t2 * (-1.f / 5040.f))));
        const float cb = (SIM_DT * SIM_DT) * (0.5f + t2 * (-1.f / 24.f + t2 * (1.f / 720.f + t2 * (-1.f / 40320.f))));
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float vx = s.R[c], vy = s.R[3 + c], vz = s.R[6 + c];
            const float wd = wx * vx + wy * vy + wz * vz;
            s.R[c] = vx + ca * (wy * vz - wz * vy) + cb * (wx * wd - vx * w2);
            s.R[3 + c] = vy + ca * (wz * vx - wx * vz) + cb * (wy * wd - vy * w2);
            s.R[6 + c] = vz + ca * (wx * vy - wy * vx) + cb * (wz * wd - vz * w2);
        }
    }
    if (do_svd) {
        M3 m;
#pragma unroll
        for (int k = 0; k < 9; ++k) m.m[k] = s.R[k];
        m = orthonormalize(m);
#pragma unroll
        for (int k = 0; k < 9; ++k) s.R[k] = m.m[k];
    }

    // Euler step of the body rates with gyroscopic term (:555-560); the Crazyflie's quadratic damping is zero
    if constexpr (DYN) {
        const float ox = s.om[0], oy = s.om[1], oz = s.om[2];
        const float ix = ph.ixx * ox, iy = ph.iyy * oy, iz = ph.izz * oz;
        const float cxx = oz * iy - oy * iz, cyy = ox * iz - oz * ix, czz = oy * ix - ox * iy;
        const float dx = 1.f - clampf(ph.omega_quadratic * ox * ox, 0.f, 1.f), dy = 1.f - clampf(ph.omega_quadratic * oy * oy, 0.f, 1.f),
                    dz = 1.f - clampf(ph.omega_quadratic * oz * oz, 0.f, 1.f);
        s.om[0] = clampf(ox + dx * SIM_DT * (ph.inv_ixx * (cxx + tq0)), -OMEGA_MAX, OMEGA_MAX);
        s.om[1] = clampf(oy + dy * SIM_DT * (ph.inv_iyy * (cyy + tq1)), -OMEGA_MAX, OMEGA_MAX);
        s.om[2] = clampf(oz + dz * SIM_DT * (ph.inv_izz * (czz + tq2)), -OMEGA_MAX, OMEGA_MAX);
    } else {
        const float ox = s.om[0], oy = s.om[1], oz = s.om[2];
        const float ix = IXX * ox, iy = IYY * oy, iz = IZZ * oz;
        const float cxx = oz * iy - oy * iz;          // cross(-omega, I omega)
        const float cyy = ox * iz - oz * ix;
        const float czz = oy * ix - ox * iy;
        s.om[0] = clampf(ox + SIM_DT * (INV_IXX * (cxx + tq0)), -OMEGA_MAX, OMEGA_MAX);
        s.om[1] = clampf(oy + SIM_DT * (INV_IYY * (cyy + tq1)), -OMEGA_MAX, OMEGA_MAX);
        s.om[2] = clampf(oz + SIM_DT * (INV_IZZ * (czz + tq2)), -OMEGA_MAX, OMEGA_MAX);
    }
    // position with the OLD velocity (:563), room clip and wall / ceiling flags (:360-367)
    const float px = s.pos[0] + SIM_DT * s.vel[0], py = s.pos[1] + SIM_DT * s.vel[1], pz = s.pos[2] + SIM_DT * s.vel[2];
    s.pos[0] = clampf(px, p.room_lo[0], p.room_hi[0]);
    s.pos[1] = clampf(py, p.room_lo[1], p.room_hi[1]);
    s.pos[2] = clampf(pz, p.room_lo[2], p.room_hi[2]);
    uint32_t fl = s.flags & ~(QS_FLAG_CRASHED_WALL | QS_FLAG_CRASHED_CEILING | QS_FLAG_CRASHED_FLOOR);
    if (px != s.pos[0] || py != s.pos[1]) fl |= QS_FLAG_CRASHED_WALL;
    if (pz > s.pos[2]) fl |= QS_FLAG_CRASHED_CEILING;

    // force in the world frame: R (thrust + rotor drag)
    const float r22 = s.R[8];
    float fx, fy, fz;
    if constexpr (DYN) {
        fx = s.R[0] * drag_fx + s.R[1] * drag_fy + s.R[2] * (thrust_z + drag_fz);
        fy = s.R[3] * drag_fx + s.R[4] * drag_fy + s.R[5] * (thrust_z + drag_fz);
        fz = s.R[6] * drag_fx + s.R[7] * drag_fy + s.R[8] * (thrust_z + drag_fz);
    } else {
        fx = s.R[2] * thrust_z; fy = s.R[5] * thrust_z; fz = r22 * thrust_z;
    }
    const float mass = DYN ? ph.mass : MASS, inv_mass = DYN ? ph.inv_mass : INV_MASS;
    const float keep = DYN ? 1.f - ph.vel_damp : 1.f;      // the Crazyflie's vel_damp is zero, and 1.f * v is exact

    // floor contact / friction, threshold = the arm (:569-639, :378).  Numpy path: threshold 0.05 (:75), exact at-rest
    // test (:406), friction along the velocity (:419-422), re-drawn landing yaw (:434-437)
#if QS_NUMPY_DYNAMICS
    const float floor_z = FLOOR_THRESHOLD_NP;
#else
    const float floor_z = DYN ? ph.arm : ARM;
#endif
    if (s.pos[2] <= floor_z) {
        s.pos[2] = floor_z;
        if (fl & QS_FLAG_ON_FLOOR) {
            yaw_only(s.R);
            // FMA_FRICTION: MASS * GRAV - fz with one rounding, written out.  The compiler fused it in these kernels before
            // their register cap and no longer does; the other kernels keep the expression (and the compiler's choice) as it was.
            const float fric = FLOOR_MU * (FMA_FRICTION ? __fmaf_rn(-r22, thrust_z, MASS * GRAV) : mass * GRAV - fz);
#if QS_NUMPY_DYNAMICS
            if (s.vel[0] == 0.f && s.vel[1] == 0.f && s.vel[2] == 0.f) {       // :406
#else
            const float v2 = s.vel[0] * s.vel[0] + s.vel[1] * s.vel[1] + s.vel[2] * s.vel[2];
            if (v2 < EPS_DYN * EPS_DYN) {
#endif
                // at rest: static friction eats the horizontal force (direction kept: cos/sin of atan2(fy, fx))
                const float f2 = fx * fx + fy * fy;
                const float fm = fsqrt(f2);
                const float mag = fmaxf(fm - fric, 0.f);
                if (fm > 0.f) {
                    const float sc = mag * frcp(fm);
                    fx *= sc; fy *= sc;
                } else {                                // atan2(0, 0) = 0: the residual force points along +x
                    fx = mag; fy = 0.f;
                }
            } else {
                // sliding: friction against the horizontal velocity direction.  With no horizontal velocity atan2(vy, vx)
                // sees signed zeros: atan2(+-0, +0) = +-0 -> direction (1, 0), atan2(+-0, -0) = +-pi -> (-1, 0) (the
                // sin(+-pi) = +-1.2e-16 is dropped)
                const float h2 = s.vel[0] * s.vel[0] + s.vel[1] * s.vel[1];
                float ca = copysignf(1.f, s.vel[0]), sa = 0.f;
                if (h2 > 0.f) {
                    const float inv = frsqrt(h2);
                    ca = s.vel[0] * inv; sa = s.vel[1] * inv;
                }
#if QS_NUMPY_DYNAMICS
                friction_dir_numpy(s.vel[0], h2, ca, sa);
#endif
                fx -= ca * fric; fy -= sa * fric;
            }
        } else {
            fl |= QS_FLAG_ON_FLOOR | QS_FLAG_CRASHED_FLOOR;
            s.vel[0] = s.vel[1] = s.vel[2] = 0.f;
            s.om[0] = s.om[1] = s.om[2] = 0.f;
            if (s.R[8] < 0.f) {                         // upside down: random yaw (:616-619; numpy path :434-437)
#if QS_NUMPY_DYNAMICS
                const float2 cs = floor_yaw_numpy(key, i, sub, s.pos[0], s.pos[1]);
#else
                const float2 cs = floor_random_yaw(key, i, sub);
#endif
                s.R[0] = cs.x; s.R[1] = -cs.y; s.R[2] = 0.f; s.R[3] = cs.y; s.R[4] = cs.x; s.R[5] = 0.f;
                s.R[6] = 0.f; s.R[7] = 0.f; s.R[8] = 1.f;
            } else {
                yaw_only(s.R);
            }
#pragma unroll
            for (int m = 0; m < 4; ++m) { s.rd[m] = 0.f; s.cd[m] = 0.f; }
        }
        // the force was taken with the pre-flattening rotation (:576), as here
        s.vel[0] = keep * s.vel[0] + SIM_DT * (inv_mass * fx);
        s.vel[1] = keep * s.vel[1] + SIM_DT * (inv_mass * fy);
        s.vel[2] = keep * s.vel[2] + SIM_DT * fmaxf(0.f, -GRAV + inv_mass * fz);
    } else {
        fl &= ~QS_FLAG_ON_FLOOR;
        s.vel[0] = keep * s.vel[0] + SIM_DT * (inv_mass * fx);
        s.vel[1] = keep * s.vel[1] + SIM_DT * (inv_mass * fy);
        s.vel[2] = keep * s.vel[2] + SIM_DT * (-GRAV + inv_mass * fz);
    }
    s.flags = fl;
    // velocity used the NEW acceleration (:645).  The accelerometer reading (:648) is never observed.
}

// The default step kernels: Crazyflie constants, inlined into the kernel.
template <bool FMA_FRICTION = false>
__device__ __forceinline__ void dynamics_substep(Agent& s, const float cmd[4], bool do_svd, const StepParams& p,
                                                 const RngKey& key, int i, int sub) {
    physics_substep<false, FMA_FRICTION>(s, cmd, do_svd, p, key, i, sub, Phys{});
}

// The DYN step kernels: per-drone constants, out of line.
__device__ __noinline__ void dynamics_substep_dyn(Agent& s, const float cmd[4], bool do_svd, const StepParams& p, const RngKey& key,
                                                  int i, int sub, const Phys& ph) {
    physics_substep<true, false>(s, cmd, do_svd, p, key, i, sub, ph);
}

// Observed rotation quat2R(rot2quat(R) x qt) (sensor_noise.py:34-63,205-210; quad_utils.py:133-159); qt is the
// rotation-noise quaternion.  The default noise set has qt = identity and emits R directly instead (write_observation).
__device__ __forceinline__ void observed_rotation(const float R[9], const float qt[4], float out[9]) {
    const float trace = R[0] + R[4] + R[8];
    float qw, qx, qy, qz;
    if (trace > 0.f) {
        const float S = fsqrt(trace + 1.0f) * 2.f, iS = frcp(S);
        qw = 0.25f * S; qx = (R[7] - R[5]) * iS; qy = (R[2] - R[6]) * iS; qz = (R[3] - R[1]) * iS;
    } else if (R[0] > R[4] && R[0] > R[8]) {
        const float S = fsqrt(1.0f + R[0] - R[4] - R[8]) * 2.f, iS = frcp(S);
        qw = (R[7] - R[5]) * iS; qx = 0.25f * S; qy = (R[1] + R[3]) * iS; qz = (R[2] + R[6]) * iS;
    } else if (R[4] > R[8]) {
        const float S = fsqrt(1.0f + R[4] - R[0] - R[8]) * 2.f, iS = frcp(S);
        qw = (R[2] - R[6]) * iS; qx = (R[1] + R[3]) * iS; qy = 0.25f * S; qz = (R[5] + R[7]) * iS;
    } else {
        const float S = fsqrt(1.0f + R[8] - R[0] - R[4]) * 2.f, iS = frcp(S);
        qw = (R[3] - R[1]) * iS; qx = (R[2] + R[6]) * iS; qy = (R[5] + R[7]) * iS; qz = 0.25f * S;
    }
    {   // quatXquat(quat, qt), quad_utils.py:148-159
        const float w = qw * qt[0] - qx * qt[1] - qy * qt[2] - qz * qt[3];
        const float x = qw * qt[1] + qx * qt[0] - qy * qt[3] + qz * qt[2];
        const float y = qw * qt[2] + qx * qt[3] + qy * qt[0] - qz * qt[1];
        const float z = qw * qt[3] - qx * qt[2] + qy * qt[1] + qz * qt[0];
        qw = w; qx = x; qy = y; qz = z;
    }
    const float xx = 2.f * qx * qx, yy = 2.f * qy * qy, zz = 2.f * qz * qz;
    const float xy = 2.f * qx * qy, xz = 2.f * qx * qz, yz = 2.f * qy * qz;
    const float wx = 2.f * qx * qw, wy = 2.f * qy * qw, wz = 2.f * qz * qw;
    out[0] = 1.0f - yy - zz; out[1] = xy - wz; out[2] = xz + wy;
    out[3] = xy + wz; out[4] = 1.0f - xx - zz; out[5] = yz - wx;
    out[6] = xz - wy; out[7] = yz + wx; out[8] = 1.0f - xx - yy;
}

// fresh sensor-noise draw for a non-default site (after a contact response / a reset): the compact layout of the hot
// draws (qs_rng.cuh, normal_pair16) — normal n of the site lives in half n % 2 of word n / 2 of its blocks 0 and 1
__device__ __noinline__ Noise9 sensor_noise(RngKey key, uint32_t site, int i) {
    uint4 blk[2];
    philox4x32_10_x2(key.env, key.step, rng_c2(site, i, 0), key.k0, key.k1, blk);
    float n[10];
    normal_pair16(blk[0].x, n[0], n[1]);
    normal_pair16(blk[0].y, n[2], n[3]);
    normal_pair16(blk[0].z, n[4], n[5]);
    normal_pair16(blk[0].w, n[6], n[7]);
    normal_pair16(blk[1].x, n[8], n[9]);
    Noise9 o;
    o.p[0] = POS_NOISE_STD * n[0]; o.p[1] = POS_NOISE_STD * n[1]; o.p[2] = POS_NOISE_STD * n[2];
    o.v[0] = VEL_NOISE_STD * n[3]; o.v[1] = VEL_NOISE_STD * n[4]; o.v[2] = VEL_NOISE_STD * n[5];
    o.w[0] = GYRO_NOISE_STD * n[6]; o.w[1] = GYRO_NOISE_STD * n[7]; o.w[2] = GYRO_NOISE_STD * n[8];
    return o;
}

// the 'default' set's first sensor-noise draw of a step, scaled from the hot normals (SITE_HOT); zero with sensor noise off
__device__ __forceinline__ Noise9 default_noise(const HotNormals& hn, int sense_noise) {
    const float on = sense_noise ? 1.f : 0.f;
    Noise9 nz;
    nz.p[0] = on * POS_NOISE_STD * hn.sn[0]; nz.p[1] = on * POS_NOISE_STD * hn.sn[1]; nz.p[2] = on * POS_NOISE_STD * hn.sn[2];
    nz.v[0] = on * VEL_NOISE_STD * hn.sn[3]; nz.v[1] = on * VEL_NOISE_STD * hn.sn[4]; nz.v[2] = on * VEL_NOISE_STD * hn.sn[5];
    nz.w[0] = on * GYRO_NOISE_STD * hn.sn[6]; nz.w[1] = on * GYRO_NOISE_STD * hn.sn[7]; nz.w[2] = on * GYRO_NOISE_STD * hn.sn[8];
    return nz;
}

// One observation's noise under the custom model (qs_set_sensor_noise; add_noise_numba + add_noise_to_omega,
// sensor_noise.py:172-231): offsets of position / velocity / gyro, the rotation-noise quaternion, and the gyro bias after this
// observation.  kind = j of the draws (qs_rng.cuh, SITE_NOISE_*).  A block whose scale is zero is not drawn: the draws are
// keyed, so skipping one changes no other.  Uniforms follow numba's low + (high - low) u.
struct SensedNoise { Noise9 n; float q[4]; float3 bias; };
__device__ __noinline__ SensedNoise sensor_noise_model(const NoiseModel& m, RngKey key, uint32_t kind, int i, float3 bias,
                                                       bool gyro_model) {
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    SensedNoise o;
    {
        const float4 n = m.pos_std != 0.f ? rng_normal4(key, SITE_NOISE_N, i, kind, 0) : zero;
        const float4 u = m.pos_range != 0.f ? rng_uniform4(key, SITE_NOISE_U, i, kind, 0) : zero;
        const float lo = -m.pos_range, w = m.pos_range - lo;
        o.n.p[0] = m.pos_std * n.x + (lo + w * u.x); o.n.p[1] = m.pos_std * n.y + (lo + w * u.y); o.n.p[2] = m.pos_std * n.z + (lo + w * u.z);
    }
    {
        const float4 n = m.vel_std != 0.f ? rng_normal4(key, SITE_NOISE_N, i, kind, 1) : zero;
        const float4 u = m.vel_range != 0.f ? rng_uniform4(key, SITE_NOISE_U, i, kind, 1) : zero;
        const float lo = -m.vel_range, w = m.vel_range - lo;
        o.n.v[0] = m.vel_std * n.x + (lo + w * u.x); o.n.v[1] = m.vel_std * n.y + (lo + w * u.y); o.n.v[2] = m.vel_std * n.z + (lo + w * u.z);
    }
    if (gyro_model) {
        // b <- pi b + sigma_b N(0, 1); omega~ = omega + b + random_walk N(0, 1) (sensor_noise.py:228-231)
        const float4 nb = rng_normal4(key, SITE_GYRO_BIAS, i, kind, 0), nw = rng_normal4(key, SITE_GYRO_BIAS, i, kind, 1);
        bias.x = m.bias_pi * bias.x + m.bias_sigma * nb.x;
        bias.y = m.bias_pi * bias.y + m.bias_sigma * nb.y;
        bias.z = m.bias_pi * bias.z + m.bias_sigma * nb.z;
        o.n.w[0] = bias.x + m.random_walk * nw.x; o.n.w[1] = bias.y + m.random_walk * nw.y; o.n.w[2] = bias.z + m.random_walk * nw.z;
    } else {
        const float4 n = m.gyro_std != 0.f ? rng_normal4(key, SITE_NOISE_N, i, kind, 2) : zero;
        o.n.w[0] = m.gyro_std * n.x; o.n.w[1] = m.gyro_std * n.y; o.n.w[2] = m.gyro_std * n.z;
    }
    o.bias = bias;
    o.q[0] = 1.f; o.q[1] = 0.f; o.q[2] = 0.f; o.q[3] = 0.f;
    if (m.rot) {
        const float4 n = m.quat_std != 0.f ? rng_normal4(key, SITE_NOISE_N, i, kind, 3) : zero;
        const float4 u = m.quat_range != 0.f ? rng_uniform4(key, SITE_NOISE_U, i, kind, 2) : zero;
        const float lo = -m.quat_range, w = m.quat_range - lo;
        const float tx = m.quat_std * n.x + (lo + w * u.x), ty = m.quat_std * n.y + (lo + w * u.y), tz = m.quat_std * n.z + (lo + w * u.z);
        // quat_from_small_angle, sensor_noise.py:11-23
        const float q2 = (tx * tx + ty * ty + tz * tz) * 0.25f;
        float qw, f;
        if (q2 < 1.f) { qw = sqrtf(1.f - q2); f = 0.5f; }
        else { qw = rsqrtf(1.f + q2); f = 0.5f * qw; }
        const float qx = tx * f, qy = ty * f, qz = tz * f;
        const float inv = rsqrtf(qw * qw + qx * qx + qy * qy + qz * qz);
        o.q[0] = qw * inv; o.q[1] = qx * inv; o.q[2] = qy * inv; o.q[3] = qz * inv;
    }
    return o;
}

// compute_new_vel, collisions/utils.py:8-18
__device__ __forceinline__ V3 compute_new_vel(float u, float max_vel_magn, V3 vel, V3 shift, float low, float high) {
    const float decay = low + (high - low) * u;
    const float nx = vel.x + shift.x, ny = vel.y + shift.y, nz = vel.z + shift.z;
    float mag = sqrtf(nx * nx + ny * ny + nz * nz);
    const float den = (mag == 0.f) ? mag + EPS_COL : mag;
    const float dx = nx / den, dy = ny / den, dz = nz / den;
    mag = fminf(mag * decay, max_vel_magn);
    V3 out;
    out.x = vel.x + (dx * mag - vel.x); out.y = vel.y + (dy * mag - vel.y); out.z = vel.z + (dz * mag - vel.z);
    return out;
}

// compute_new_omega, collisions/utils.py:22-33 (three direction uniforms, one magnitude uniform)
__device__ __forceinline__ V3 compute_new_omega(float u0, float u1, float u2, float um, float magn_scale) {
    const float omega_max = magn_scale * PI_F;
    const float x = -1.f + 2.f * u0, y = -1.f + 2.f * u1, z = -1.f + 2.f * u2;
    const float mag = sqrtf(x * x + y * y + z * z);
    const float den = (mag == 0.f) ? mag + EPS_COL : mag;
    const float lo = omega_max * 0.5f;
    const float m = lo + (omega_max - lo) * um;
    V3 out;
    out.x = x / den * m; out.y = y / den * m; out.z = z / den * m;
    return out;
}

// perform_collision_between_drones, collisions/quadrotors.py:24-59.  Every lane of the env evaluates the pair
// (a < b) from shuffled copies of both drones and keyed draws, lanes a and b keep their half of the result.
__device__ __noinline__ PairOut pair_response(RngKey key, int a, int b, V3 p1, V3 v1, V3 p2, V3 v2) {
    float nx = p1.x - p2.x, ny = p1.y - p2.y, nz = p1.z - p2.z;
    const float nm = sqrtf(nx * nx + ny * ny + nz * nz);
    const float den = (nm == 0.f) ? nm + EPS_COL : nm;
    nx /= den; ny /= den; nz /= den;
    const float v1n = v1.x * nx + v1.y * ny + v1.z * nz;
    const float v2n = v2.x * nx + v2.y * ny + v2.z * nz;
    const float ch[3] = {(v2n - v1n) * nx, (v2n - v1n) * ny, (v2n - v1n) * nz};
    V3 s1 = {ch[0], ch[1], ch[2]}, s2 = {-ch[0], -ch[1], -ch[2]};
#pragma unroll 1
    for (int t = 0; t < 3; ++t) {
        const float4 n0 = rng_normal4(key, SITE_PAIR_N, a, b, 3 * t), n1 = rng_normal4(key, SITE_PAIR_N, a, b, 3 * t + 1),
                     n2 = rng_normal4(key, SITE_PAIR_N, a, b, 3 * t + 2);
        s1.x = ch[0] + (0.8f * n0.x + 0.15f * n0.w); s1.y = ch[1] + (0.8f * n0.y + 0.15f * n1.x); s1.z = ch[2] + (0.8f * n0.z + 0.15f * n1.y);
        s2.x = -ch[0] + (-0.8f * n0.x + 0.15f * n1.z); s2.y = -ch[1] + (-0.8f * n0.y + 0.15f * n1.w); s2.z = -ch[2] + (-0.8f * n0.z + 0.15f * n2.x);
        const float d1 = (v1.x + s1.x) * nx + (v1.y + s1.y) * ny + (v1.z + s1.z) * nz;
        const float d2 = (v2.x + s2.x) * nx + (v2.y + s2.y) * ny + (v2.z + s2.z) * nz;
        if (d1 > 0.f && 0.f > d2) break;
    }
    const float maxv = fmaxf(sqrtf(v1.x * v1.x + v1.y * v1.y + v1.z * v1.z), sqrtf(v2.x * v2.x + v2.y * v2.y + v2.z * v2.z));
    const float4 u0 = rng_uniform4(key, SITE_PAIR_U, a, b, 0), u1 = rng_uniform4(key, SITE_PAIR_U, a, b, 1);
    PairOut o;
    o.v1 = compute_new_vel(u0.x, maxv, v1, s1, 0.2f, 0.8f);
    o.v2 = compute_new_vel(u0.y, maxv, v2, s2, 0.2f, 0.8f);
    o.dom = compute_new_omega(u0.z, u0.w, u1.x, u1.y, 20.0f);
    return o;
}

// perform_collision_with_obstacle, collisions/obstacles.py:23-50 (obstacle z = room_height / 2, quadrotor_multi.py:322)
__device__ __noinline__ KickVO obstacle_response(RngKey key, int i, V3 pos, V3 vel, float ox, float oy, float oz,
                                                 float obst_half_size) {
    float nx = pos.x - ox, ny = pos.y - oy;
    const float nm = sqrtf(nx * nx + ny * ny);
    const float den = (nm == 0.f) ? nm + EPS_COL : nm;
    nx /= den; ny /= den;
    const float vmag = sqrtf(vel.x * vel.x + vel.y * vel.y + vel.z * vel.z);
    const float nvx = vmag * nx, nvy = vmag * ny;
    float noise[3] = {0.f, 0.f, 0.f};
#pragma unroll 1
    for (int t = 0; t < 3; ++t) {
        const float4 n0 = rng_normal4(key, SITE_OBST_N, i, 0, 2 * t), n1 = rng_normal4(key, SITE_OBST_N, i, 0, 2 * t + 1);
        const float tx = 0.1f * n0.x + 0.05f * n0.w, ty = 0.1f * n0.y + 0.05f * n1.x, tz = 0.1f * n0.z + 0.05f * n1.y;
        if ((nvx + tx) * nx + (nvy + ty) * ny > 0.f) {
            noise[0] = tx; noise[1] = ty; noise[2] = tz;
            break;
        }
    }
    const float4 u0 = rng_uniform4(key, SITE_OBST_U, i, 0, 0), u1 = rng_uniform4(key, SITE_OBST_U, i, 0, 1);
    const V3 shift = {nvx - vel.x + noise[0], nvy - vel.y + noise[1], 0.f - vel.z + noise[2]};
    const float dx = pos.x - ox, dy = pos.y - oy, dz = pos.z - oz;
    const bool inside = sqrtf(dx * dx + dy * dy + dz * dz) < obst_half_size;
    KickVO o;
    o.vel = compute_new_vel(u0.x, vmag, vel, shift, inside ? 1.0f : 0.2f, inside ? 1.0f : 0.8f);
    o.dom = compute_new_omega(u0.y, u0.z, u0.w, u1.x, 1.0f);
    return o;
}

__device__ __forceinline__ V3 room_omega_kick(float u0, float u1, float u2, float um) {
    const float omega_max = 20.f * PI_F;
    const float x = -1.f + 2.f * u0, y = -1.f + 2.f * u1, z = -1.f + 2.f * u2;
    const float inv = 1.f / (sqrtf(x * x + y * y + z * z) + 1e-5f);
    const float lo = omega_max * 0.5f;
    const float m = lo + (omega_max - lo) * um;
    V3 o = {x * inv * m, y * inv * m, z * inv * m};
    return o;
}

// perform_collision_with_wall, collisions/room.py:6-44.  touch_* say which wall the clipped position sits on.
__device__ __noinline__ KickVO wall_response(RngKey key, int i, V3 vel, int touch_x, int touch_y) {
    const float4 u0 = rng_uniform4(key, SITE_WALL_U, i, 0, 0), u1 = rng_uniform4(key, SITE_WALL_U, i, 0, 1),
                 u2 = rng_uniform4(key, SITE_WALL_U, i, 0, 2);
    const float speed = sqrtf(vel.x * vel.x + vel.y * vel.y + vel.z * vel.z);
    const float lo = 0.2f * speed, hi = 0.8f * speed;
    const float real_speed = clampf(lo + (hi - lo) * u0.x, 0.1f, 6.0f);
    float dx = -1.f + 2.f * u0.y, dy = -1.f + 2.f * u0.z;
    if (touch_x < 0) dx = 0.1f + (1.0f - 0.1f) * u1.x;
    else if (touch_x > 0) dx = -1.0f + (-0.1f - -1.0f) * u1.x;
    if (touch_y < 0) dy = 0.1f + (1.0f - 0.1f) * u1.y;
    else if (touch_y > 0) dy = -1.0f + (-0.1f - -1.0f) * u1.y;
    const float dz = -1.0f + (-0.5f - -1.0f) * u1.z;
    const float inv = 1.f / (sqrtf(dx * dx + dy * dy + dz * dz) + 1e-5f);
    KickVO o;
    o.vel.x = real_speed * (dx * inv); o.vel.y = real_speed * (dy * inv); o.vel.z = real_speed * (dz * inv);
    o.dom = room_omega_kick(u1.w, u2.x, u2.y, u2.z);
    return o;
}

// perform_collision_with_ceiling, collisions/room.py:91-113
__device__ __noinline__ KickVO ceiling_response(RngKey key, int i, V3 vel) {
    const float4 u0 = rng_uniform4(key, SITE_CEIL_U, i, 0, 0), u1 = rng_uniform4(key, SITE_CEIL_U, i, 0, 1),
                 u2 = rng_uniform4(key, SITE_CEIL_U, i, 0, 2);
    const float speed = sqrtf(vel.x * vel.x + vel.y * vel.y + vel.z * vel.z);
    const float lo = 0.2f * speed, hi = 0.8f * speed;
    const float real_speed = clampf(lo + (hi - lo) * u0.x, 0.1f, 6.0f);
    const float dx = -1.f + 2.f * u0.y, dy = -1.f + 2.f * u0.z;
    const float dz = -1.0f + (-0.5f - -1.0f) * u1.x;
    const float inv = 1.f / (sqrtf(dx * dx + dy * dy + dz * dz) + 1e-5f);
    KickVO o;
    o.vel.x = real_speed * (dx * inv); o.vel.y = real_speed * (dy * inv); o.vel.z = real_speed * (dz * inv);
    o.dom = room_omega_kick(u1.y, u1.z, u1.w, u2.x);
    return o;
}

// downwash push on drone `me` sitting in the cylinder below drone `other` (aerodynamics/downwash.py:27-66);
// d = |p_me - p_other|, (zx, zy, zz) = body z-axis of `other`.  Returns delta velocity / delta omega.
__device__ __noinline__ KickVO downwash_kick(RngKey key, int other, int me, float d, float zx, float zy, float zz) {
    const float4 ui = rng_uniform4(key, SITE_DW_I, other, 0, 0);
    const float4 u0 = rng_uniform4(key, SITE_DW_IJ, other, me, 0), u1 = rng_uniform4(key, SITE_DW_IJ, other, me, 1);
    const float acc = fmaxf(1e-6f, (6.f / 17.f) * (-10.f * d + 7.f) + (-0.1f + 0.2f * ui.x));
    const float omd = fmaxf(1e-6f, 0.3f * (d - 1.f) * (d - 1.f) + (-0.01f + 0.02f * ui.y));
    float ax = zx + (-0.1f + 0.2f * u0.x), ay = zy + (-0.1f + 0.2f * u0.y), az = zz + (-0.1f + 0.2f * u0.z);
    float mag = sqrtf(ax * ax + ay * ay + az * az);
    float den = (mag == 0.f) ? mag + 1e-6f : mag;
    ax = -(ax / den); ay = -(ay / den); az = -(az / den);
    const float bx = -1.f + 2.f * u0.w, by = -1.f + 2.f * u1.x, bz = -1.f + 2.f * u1.y;
    mag = sqrtf(bx * bx + by * by + bz * bz);
    den = (mag == 0.f) ? mag + 1e-6f : mag;
    KickVO o;
    o.vel.x = acc * ax * CONTROL_DT; o.vel.y = acc * ay * CONTROL_DT; o.vel.z = acc * az * CONTROL_DT;
    o.dom.x = omd * (bx / den) * CONTROL_DT; o.dom.y = omd * (by / den) * CONTROL_DT; o.dom.z = omd * (bz / den) * CONTROL_DT;
    return o;
}

// ---- device-side episode generator: o_random (scenarios/obstacles/o_random.py:27-52, o_base.py:71-83,
//      quadrotor_multi.py:304-325).  Sequential uniform sampling without replacement over the grid cells with a
//      64-bit occupancy mask; every lane of the env runs the same deterministic selection and keeps its own picks, so no
//      exchange is needed.  Keyed draws (SITE_SCENARIO_U): value v = 0..M-1 pillar cells, 64.. spawn cells, 128.. spawn z,
//      192.. goal cells, 256.. goal z.  Cell (rid, cid) sits at (cid + 0.5 - L/2, W - 1 - rid + 0.5 - W/2) like the
//      reference's get_cell_centers / obst_map indexing.  Twin: oracle/scenario_gen.py.
// position of the r-th (0-based) set bit of x; r < popc(x).  Binary search on popcounts (~25 instructions; the fns
// instruction is emulated by a loop over the bits).
__device__ __forceinline__ int nth_set_bit32(uint32_t x, int r) {
    int pos = 0;
    int c = __popc(x & 0xffffu);
    if (r >= c) { r -= c; pos += 16; x >>= 16; }
    c = __popc(x & 0xffu);
    if (r >= c) { r -= c; pos += 8; x >>= 8; }
    c = __popc(x & 0xfu);
    if (r >= c) { r -= c; pos += 4; x >>= 4; }
    c = __popc(x & 0x3u);
    if (r >= c) { r -= c; pos += 2; x >>= 2; }
    if (r >= (int)(x & 1u)) pos += 1;
    return pos;
}

__device__ __forceinline__ int nth_free_cell(unsigned long long mask, int r, int cells) {
    // index of the r-th (0-based) clear bit of `mask` among bits [0, cells); `cells` if there is none
    const unsigned long long lim = cells >= 64 ? ~0ull : ((1ull << cells) - 1ull);
    const unsigned long long fr = ~mask & lim;
    const uint32_t lo = (uint32_t)fr, hi = (uint32_t)(fr >> 32);
    const int nlo = __popc(lo);
    if (r < nlo) return nth_set_bit32(lo, r);
    if (r - nlo < __popc(hi)) return 32 + nth_set_bit32(hi, r - nlo);
    return cells;
}

__device__ __forceinline__ float scenario_u(const RngKey& key, int v) {
    const float4 u = rng_uniform4(key, SITE_SCENARIO_U, 0, 0, v >> 2);
    const int w = v & 3;
    return w == 0 ? u.x : (w == 1 ? u.y : (w == 2 ? u.z : u.w));
}

// floor(u * n) for u = k / 2^24, in integer arithmetic so that the fp32 kernel and the fp64 oracle agree exactly
__device__ __forceinline__ int scenario_pick(const RngKey& key, int v, int n) {
    const uint32_t k = (uint32_t)(scenario_u(key, v) * 16777216.0f);
    return (int)((k * (uint32_t)n) >> 24);
}

__device__ __forceinline__ float2 cell_center(int cell, int L, int W) {
    const int rid = cell / W, cid = cell - rid * W;
    return make_float2((float)cid + 0.5f - (float)(L / 2), (float)(W - 1 - rid) + 0.5f - (float)(W / 2));
}

struct ORandomEpisode { V3 spawn, goal; int mode; unsigned long long mask; };

// word w of a uniform block
__device__ __forceinline__ float u4_word(const float4& u, int w) { return w == 0 ? u.x : (w == 1 ? u.y : (w == 2 ? u.z : u.w)); }
// floor(u * n) for a uniform already drawn (same integer arithmetic as scenario_pick)
__device__ __forceinline__ int pick_of(float u, int n) {
    const uint32_t k = (uint32_t)(u * 16777216.0f);
    return (int)((k * (uint32_t)n) >> 24);
}

// o_base.py:123-153 (max_square_area_center): dynamic programme over the pillar map; returns the map cell (row * W + col)
// at the centre of the largest free square.  Reference quirks kept: the first row / column of the table hold the MAP
// values (an occupied border cell counts as a square of size 1), only strictly larger squares replace the best one.
__device__ __noinline__ int largest_free_square_cell(unsigned long long mask, int L, int W) {
    unsigned char dp[64];
    int best = 0, cx = 0, cy = 0;
    for (int j = 0; j < W; ++j) dp[j] = (unsigned char)((mask >> j) & 1ull);
    for (int i = 1; i < L; ++i) {
        dp[i * W] = (unsigned char)((mask >> (i * W)) & 1ull);
        for (int j = 1; j < W; ++j) {
            int v = 0;
            if (!((mask >> (i * W + j)) & 1ull)) {
                v = min(min((int)dp[(i - 1) * W + j], (int)dp[i * W + j - 1]), (int)dp[(i - 1) * W + j - 1]) + 1;
                if (v > best) { best = v; cx = i - (best - 1) / 2; cy = j - (best - 1) / 2; }
            }
            dp[i * W + j] = (unsigned char)v;
        }
    }
    return cx * W + cy;
}

// pillar table of the env -> `obst_out[m]` for m = lane, lane + stride, ... ; this lane's spawn / goal returned
// `scenario`: QS_SCENARIO_O_RANDOM, QS_SCENARIO_O_STATIC_SAME_GOAL, QS_SCENARIO_MIX (one of the two per episode, slot 321) or one
// of the ticked obstacle scenarios (their goals are finished by o_episode_extras, qs_scenario.cuh).
// The draws are the keyed values scenario_u(key, v) (one Philox block serves four consecutive v: it is computed once
// per four picks here, not once per pick).
__device__ __noinline__ ORandomEpisode o_random_episode(RngKey key, int scenario, int i, int n_agents, int M, int L, int W, int lane_i,
                                                        int stride, float2* obst_smem, float2* obst_glob, int M_table) {
    const int cells = L * W;
    // the table keeps M_table slots; with fewer pillars this episode (density randomisation) the rest stand far outside
    // the room, where no test or distance can see them
    for (int m = M + lane_i; m < M_table; m += stride) {
        const float2 far = make_float2(1.0e4f, 1.0e4f);
        if (obst_smem != nullptr) obst_smem[m] = far;
        obst_glob[m] = far;
    }
    unsigned long long mask = 0ull;
    float4 ub = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int m = 0; m < M; ++m) {
        if ((m & 3) == 0) ub = rng_uniform4(key, SITE_SCENARIO_U, 0, 0, m >> 2);
        const int r = pick_of(u4_word(ub, m & 3), cells - m);
        const int c = nth_free_cell(mask, r, cells);
        mask |= 1ull << c;
        if ((m % stride) == lane_i) {
            const float2 xy = cell_center(c, L, W);
            if (obst_smem != nullptr) obst_smem[m] = xy;
            obst_glob[m] = xy;
        }
    }
    ORandomEpisode ep;
    ep.mode = scenario;
    if (scenario == QS_SCENARIO_MIX) ep.mode = scenario_pick(key, 321, 2) == 0 ? QS_SCENARIO_O_RANDOM : QS_SCENARIO_O_STATIC_SAME_GOAL;
    const int free_cells = cells - M;
    unsigned long long ms = mask, mg = mask;
    float4 us = ub, ug = ub;
    int cs = 0, cg = 0;
    const int kend = min(i, n_agents - 1);
#pragma unroll 1
    for (int k = 0; k <= kend; ++k) {
        if ((k & 3) == 0) {
            us = rng_uniform4(key, SITE_SCENARIO_U, 0, 0, (64 + k) >> 2);
            ug = rng_uniform4(key, SITE_SCENARIO_U, 0, 0, (192 + k) >> 2);
        }
        cs = nth_free_cell(ms, pick_of(u4_word(us, k & 3), free_cells - k), cells);
        ms |= 1ull << cs;
        cg = nth_free_cell(mg, pick_of(u4_word(ug, k & 3), free_cells - k), cells);
        mg |= 1ull << cg;
    }
    {
        const int k = kend;
        const float2 a = cell_center(cs, L, W), b = cell_center(cg, L, W);
        ep.spawn.x = a.x; ep.spawn.y = a.y; ep.spawn.z = 1.0f + (3.0f - 1.0f) * scenario_u(key, 128 + k);
        ep.goal.x = b.x; ep.goal.y = b.y; ep.goal.z = 1.0f + (3.0f - 1.0f) * scenario_u(key, 256 + k);
    }
    ep.mask = mask;
    if (ep.mode == QS_SCENARIO_O_STATIC_SAME_GOAL || ep.mode == QS_SCENARIO_O_DYNAMIC_SAME_GOAL || ep.mode == QS_SCENARIO_O_SWAP_GOALS) {
        // one goal for the whole swarm (o_static_same_goal.py:44-52; the start of o_dynamic_same_goal.py:45, the formation
        // centre of o_swap_goals.py:46)
        const float2 c = cell_center(largest_free_square_cell(mask, L, W), L, W);
        ep.goal.x = c.x; ep.goal.y = c.y; ep.goal.z = 1.5f + (3.0f - 1.5f) * scenario_u(key, 320);
    }
    return ep;
}

// QuadrotorSingle._reset, quadrotor_single.py:387-447: spawn jitter, z >= 0.75, random yaw facing the origin.
__device__ __noinline__ ResetPose reset_pose(RngKey key, int i, V3 spawn, float box) {
    const float4 u = rng_uniform4(key, SITE_SPAWN_U, i, 0, 0);
    ResetPose r;
    r.pos.x = (-box + (box - (-box)) * u.x) + spawn.x;
    r.pos.y = (-box + (box - (-box)) * u.y) + spawn.y;
    r.pos.z = fmaxf((-box + (box - (-box)) * u.z) + spawn.z, 0.75f);
    // to_xyhat(-pos), quad_utils.py:75-82,112-116
    float hx = -r.pos.x, hy = -r.pos.y;
    const float n = sqrtf(hx * hx + hy * hy);
    if (!(n < 0.00001f)) { hx /= n; hy /= n; }
    float sn = 0.f, cs = 1.f;
    float4 uy = u;
#pragma unroll 1
    for (int k = 0; k < RESET_YAW_MAX_TRIES; ++k) {
        if ((k & 3) == 0) uy = rng_uniform4(key, SITE_RESET_YAW_U, i, 0, k >> 2);
        const float uu = u4_word(uy, k & 3);
        sincosf(-PI_F + (PI_F - (-PI_F)) * uu, &sn, &cs);
        if (cs * hx + sn * hy >= 0.5f) break;          // rotation[:, 0] = (cos, sin, 0)
    }
    r.cs = cs; r.sn = sn;
    return r;
}

// apply a reset pose: zero rates and motor state, cleared contact flags.  OU state and the SVD counter are NOT
// reset (Appendix D-9).
__device__ __forceinline__ void apply_reset(Agent& s, const ResetPose& r) {
    s.pos[0] = r.pos.x; s.pos[1] = r.pos.y; s.pos[2] = r.pos.z;
    s.R[0] = r.cs; s.R[1] = -r.sn; s.R[2] = 0.f; s.R[3] = r.sn; s.R[4] = r.cs; s.R[5] = 0.f; s.R[6] = 0.f; s.R[7] = 0.f; s.R[8] = 1.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) { s.vel[k] = 0.f; s.om[k] = 0.f; }
#pragma unroll
    for (int m = 0; m < 4; ++m) { s.rd[m] = 0.f; s.cd[m] = 0.f; s.ring[m] = 0.f; }
    s.flags = QS_FLAG_NO_COL_AGENT | QS_FLAG_NO_COL_OBST;
    s.prev_col = 0u;
}

// normalize(), quad_utils.py:80-86: a vector shorter than 1e-5 is returned unchanged
__device__ __forceinline__ V3 normalize_ref(V3 v) {
    const float n = sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
    if (n < 0.00001f) return v;
    v.x /= n; v.y /= n; v.z /= n;
    return v;
}

// The initial state of a spawn with init_random_state (quadrotor_single.py:405-423): QuadrotorDynamics.random_state
// (quadrotor_dynamics.py:193-206).  Velocity and body rate: a direction from a uniform cube, scaled to a uniform magnitude,
// x = mag / (|d| + EPS) d with EPS = 1e-6 (:13); attitude: rand_uniform_rot3d (quad_utils.py:94-104), R = [fwd | left | up].
// random_state's position draw is discarded by _reset and not drawn here.  The fwd re-draw loop is capped at
// INIT_ROT_MAX_TRIES (DESIGN, deviations).  Keyed by the episode, like the spawn jitter: applied after apply_reset.
struct InitState { float vel[3], om[3], R[9]; };
__device__ __noinline__ InitState random_init_state(RngKey key, int i, float vel_max, float omega_max) {
    InitState o;
    const float4 u0 = rng_uniform4(key, SITE_INIT_U, i, 0, 0), u1 = rng_uniform4(key, SITE_INIT_U, i, 0, 1);
    {
        const float lo = -vel_max, w = vel_max - lo;
        const float dx = lo + w * u0.x, dy = lo + w * u0.y, dz = lo + w * u0.z;
        const float f = (vel_max * u0.w) / (sqrtf(dx * dx + dy * dy + dz * dz) + 1e-6f);
        o.vel[0] = f * dx; o.vel[1] = f * dy; o.vel[2] = f * dz;
    }
    {
        const float lo = -omega_max, w = omega_max - lo;
        const float dx = lo + w * u1.x, dy = lo + w * u1.y, dz = lo + w * u1.z;
        const float f = (omega_max * u1.w) / (sqrtf(dx * dx + dy * dy + dz * dz) + 1e-6f);
        o.om[0] = f * dx; o.om[1] = f * dy; o.om[2] = f * dz;
    }
    const float4 nu = rng_normal4(key, SITE_INIT_N, i, 0, 0);
    V3 up = normalize_ref(V3{nu.x, nu.y, nu.z}), fwd;
#pragma unroll 1
    for (int t = 0; t < INIT_ROT_MAX_TRIES; ++t) {
        const float4 nf = rng_normal4(key, SITE_INIT_N, i, 0, t + 1);
        fwd = normalize_ref(V3{nf.x, nf.y, nf.z});
        if (!(fwd.x * up.x + fwd.y * up.y + fwd.z * up.z > 0.95f)) break;
    }
    const V3 left = normalize_ref(V3{up.y * fwd.z - up.z * fwd.y, up.z * fwd.x - up.x * fwd.z, up.x * fwd.y - up.y * fwd.x});
    up = V3{fwd.y * left.z - fwd.z * left.y, fwd.z * left.x - fwd.x * left.z, fwd.x * left.y - fwd.y * left.x};
    o.R[0] = fwd.x; o.R[1] = left.x; o.R[2] = up.x;
    o.R[3] = fwd.y; o.R[4] = left.y; o.R[5] = up.y;
    o.R[6] = fwd.z; o.R[7] = left.z; o.R[8] = up.z;
    return o;
}

#if QS_NUMPY_DYNAMICS
// The landing yaw of the numpy path (floor_interaction, quadrotor_dynamics.py:434-437): randyaw() is re-drawn until the body
// x-axis points within 60 deg of the origin, seen from the snapped position (x, y) — to_xyhat(-pos), quad_utils.py:120-124.
// Capped at RESET_YAW_MAX_TRIES like reset_pose (DESIGN, deviations).
__device__ __noinline__ float2 floor_yaw_numpy(RngKey key, int i, int sub, float x, float y) {
    float hx = -x, hy = -y;
    const float n = sqrtf(hx * hx + hy * hy);
    if (!(n < 0.00001f)) { hx /= n; hy /= n; }
    float sn = 0.f, cs = 1.f;
    float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int k = 0; k < RESET_YAW_MAX_TRIES; ++k) {
        if ((k & 3) == 0) u = rng_uniform4(key, SITE_FLOOR_YAW_NP, i, sub, k >> 2);
        sincosf(-PI_F + (PI_F - (-PI_F)) * u4_word(u, k & 3), &sn, &cs);
        if (cs * hx + sn * hy >= 0.5f) break;          // rot[:, 0] = (cos, sin, 0)
    }
    return make_float2(cs, sn);
}
#endif

}  // namespace qs
