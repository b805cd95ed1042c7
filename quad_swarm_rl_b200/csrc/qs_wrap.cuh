// The wrapper stack of the reference's training env, as ONE epilogue kernel behind the step kernel (SURVEY.md 8f-2, 8f-3):
//
//   QuadsRewardShapingWrapper.step   swarm_rl/env_wrappers/reward_shaping.py:52-123
//       cumulative rew_* / rewraw_* terms and action statistics of the running episode; at an episode end the
//       `true_reward`, the `episode_extra_stats` keys (incl. the env's own statistics, quadrotor_multi.py:626-718) and the
//       per-scenario copies of the headline keys;
//   ExperienceReplayWrapper.step / new_episode   gym_art/quadrotor_multi/quad_experience_replay.py:66-209
//       a checkpoint of the env every 0.5 s, the checkpoint from 1.5 s before a collision goes into the env's 20-slot event
//       buffer, a finished env restarts from a buffered event with probability p (can_drones_fly gate,
//       quadrotor_multi.py:281-287,356-359).
//
// The reference walks Python lists of dicts per agent and deep-copies the env; here everything is per-env / per-agent
// device state, the env "deep copy" is a copy of the env's SoA rows, and nothing crosses PCIe per step: finished-episode
// statistics are ACCUMULATED on the device (sums + counts) and read whenever the trainer logs (qs_wrap_read).  No host
// synchronisation, no PyTorch: qs_wrap_step = step kernel + this kernel.
#pragma once
#include "qs_step.cuh"

namespace qs {

// ---- aggregate of the finished episodes since the last qs_wrap_read (all float sums) ----
enum WrapAgg {
    WA_AGENT_EPISODES = 0,       // agent-episodes of FRESH episodes summed below (replayed episodes only feed WA_REPLAY_*)
    WA_TRUE_REWARD,              // rewraw_main (reward_shaping.py:80-84: rewraw_pos + 1000 rewraw_quadcol ... as batched.py)
    WA_RAW0,                     // 8 cumulative raw terms, QS_TERM_* order
    WA_REW0 = WA_RAW0 + 8,       // 8 cumulative weighted terms
    WA_ACT_MEAN0 = WA_REW0 + 8,  // z_action{k}_mean
    WA_ACT_STD0 = WA_ACT_MEAN0 + 4,
    WA_ENV_EPISODES = WA_ACT_STD0 + 4,
    WA_ENV_STAT0,                // QS_STAT_NUM_COLLISIONS .. QS_STAT_NUM_COLLISIONS_OBST_5 (11 counters), per env-episode
    WA_DIST0 = WA_ENV_STAT0 + 11,    // distance_to_goal_1s / 3s / 5s, per agent-episode
    WA_SUCCESS = WA_DIST0 + 3, WA_DEADLOCK, WA_COL, WA_NEIGHBOR_COL, WA_OBST_COL,
    WA_REPLAY_ENV_EPISODES, WA_REPLAY_COLLISIONS, WA_REPLAY_COLLISIONS_OBST,
    WA_EPISODES_TOTAL, WA_REPLAYED_EVENTS, WA_EVENTS_STORED, WA_CHECKPOINTS,
    WA_SCN0,                     // per scenario id s (0..15): 6 floats: agent-episodes, rew_pos, rew_crash, env-episodes,
                                 //                            num_collisions_after_settle, distance_to_goal_1s
    WA_COUNT = WA_SCN0 + 16 * 6
};
static_assert(WA_COUNT == QS_WRAP_AGG, "QS_WRAP_AGG of include/quadswarm.h");

constexpr int RP_KEEP = 6;       // 3 s of checkpoints, one every 0.5 s (quad_experience_replay.py:17-21,84)
constexpr int RP_CP_EVERY = 50;
constexpr int RP_STEPS_AGO = 3;  // the checkpoint from 1.5 s before the collision (:87,:157)
constexpr int RP_COOLDOWN = 500; // one event per 5 s (:154)
constexpr int RP_MAX_REPLAYS = 10;
constexpr int RP_GRACE = 150;    // collisions_grace_period_seconds * control_freq
constexpr int SNAP_BATCH = 32;   // observation words in flight per lane in a snapshot copy (a row of c3 is 40 words: 2 round trips)
constexpr int SNAP_ENV_I32 = 40; // env_ctr 4, env_cnt 13, scn_i 4, scn_f 12 (bit patterns), spare
constexpr uint32_t SITE_REPLAY_U = 17;     // (env) uniforms v0 replay?, v1 which event   quad_experience_replay.py:176-178

struct WrapState {
    // reward shaping
    float4* acc;                 // [6][A]: raw 0-3, raw 4-7, rew 0-3, rew 4-7, action sums, action square sums
    int* ep_steps;               // [E]
    float* true_reward;          // [A]  latched at the episode end (infos['true_reward'])
    float* agg;                  // [WA_COUNT]
    // replay
    int slots;                   // RP_KEEP + buffer size
    int buffer;                  // events per env
    float4* snap_slots;          // [E][slots][NUM_SLOTS][N]
    float* snap_obs;             // [E][slots][N][D]
    int32_t* snap_env;           // [E][slots][SNAP_ENV_I32]
    float2* snap_obst;           // [E][slots][M]
    int4* rp;                    // [E]  ring_pos, ring_cnt, buf_pos, last_added tick
    int4* rq;                    // [E]  saved (this episode is a replay), active (can_drones_fly), crash_n, 0
    float* crash_now;            // [E]
    float* crash_hist;           // [E][100]
    int32_t* ev_state;           // [E][buffer]  -1 empty, else how often the event was replayed
    float replay_prob;
    int replay_on, always_active;
};

// kernel parameters of the stand-alone wrapper kernel (qs_wrap_apply, and qs_wrap_step behind the split step shape)
struct WrapParams {
    StepParams sp;               // sp.actions / sp.rew_terms / sp.dones / sp.obs: this control step's arrays
    WrapState w;
    int chain;                   // 1: per-block hand-over with the step grids (see qs_wrap_kernel)
};
// what the body works on
struct WrapView {
    const StepParams* sp;
    const WrapState* w;
    const float4* actions;
    const float* terms;          // [A][QS_NUM_TERMS] written by the step of this control step
    const uint8_t* dones;        // [A]
    float* obs;                  // [A][D]  (rows of replayed envs are overwritten)
    const int* rows;             // block-chained launch: counter Rw of the block (else null) and the value it must reach before rows
    int rows_want;               // of q.obs are read or overwritten
};

__device__ __forceinline__ void agg_add(float* agg, int k, float v) { if (v != 0.f) atomicAdd(agg + k, v); }

// Block-chained launch: the body starts when the step block has stored state, rewards, dones and reward terms; its
// observation rows may still be on their way.  Called by whole warps right before they read or overwrite rows of q.obs.
__device__ __forceinline__ void wait_rows(const WrapView& q) {
    if (q.rows == nullptr) return;
    if ((threadIdx.x & 31) == 0) poll_acquire<counter_below>(q.rows, q.rows_want);    // a lost count is caught (and reported) at the end of the kernel
    __syncwarp();
}

// copy the rows of env `env` between the live state and snapshot slot `slot` (all lanes of the env take part)
template <bool TO_SNAP>
__device__ __forceinline__ void snap_copy(const WrapView& q, int env, int i, bool valid, int slot, bool keep_live_counters) {
    const StepParams& p = *q.sp;
    const DevState& st = p.st;
    const WrapState& w = *q.w;
    const long long a = (long long)env * p.N + i;
    const long long sbase = ((long long)env * w.slots + slot);
    // All loads of a copy are issued before its first store (the compiler must assume the two sides alias, so a load -> store
    // loop would pay one memory round trip per element: 12 slots + N D / N observation words = ~50 serialized round trips).
    if (valid) {
        float4* sn = w.snap_slots + (sbase * NUM_SLOTS) * p.N + i;
        float4 v[NUM_SLOTS];
#pragma unroll
        for (int k = 0; k < NUM_SLOTS; ++k) v[k] = TO_SNAP ? __ldcg(st.slots + (long long)k * st.a_pad + a) : __ldcg(sn + (long long)k * p.N);
#pragma unroll
        for (int k = 0; k < NUM_SLOTS; ++k) {
            if (TO_SNAP) sn[(long long)k * p.N] = v[k];
            else st.slots[(long long)k * st.a_pad + a] = v[k];
        }
    }
    // observation rows and pillar table: the env's lanes stride over them, SNAP_BATCH words in flight per lane
    float* so = w.snap_obs + sbase * p.N * p.D;
    float* lo = q.obs + (long long)env * p.N * p.D;
    const float* src = TO_SNAP ? lo : so;
    float* dst = TO_SNAP ? so : lo;
    if (valid) {
        const int total = p.N * p.D;
        for (int k0 = i; k0 < total; k0 += SNAP_BATCH * p.N) {
            float t[SNAP_BATCH];
#pragma unroll
            for (int u = 0; u < SNAP_BATCH; ++u) { const int k = k0 + u * p.N; t[u] = k < total ? __ldcg(src + k) : 0.f; }
#pragma unroll
            for (int u = 0; u < SNAP_BATCH; ++u) { const int k = k0 + u * p.N; if (k < total) dst[k] = t[u]; }
        }
    }
    if (p.M > 0 && valid) {
        float2* sb = w.snap_obst + sbase * p.M;
        float2* lb = st.obst + (long long)env * p.M;
        float2 t[8];
        for (int m0 = i; m0 < p.M; m0 += 8 * p.N) {
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int m = m0 + u * p.N; t[u] = m < p.M ? __ldcg((TO_SNAP ? lb : sb) + m) : make_float2(0.f, 0.f); }
#pragma unroll
            for (int u = 0; u < 8; ++u) { const int m = m0 + u * p.N; if (m < p.M) (TO_SNAP ? sb : lb)[m] = t[u]; }
        }
    }
    if (valid && i == 0) {
        int32_t* se = w.snap_env + sbase * SNAP_ENV_I32;
        if (TO_SNAP) {
            const int4 c = __ldcg(st.env_ctr + env);
            const int4 si = __ldcg(st.scn_i + env);
            int32_t cn[QS_NUM_ENV_STATS];
            float4 f[3];
#pragma unroll
            for (int k = 0; k < QS_NUM_ENV_STATS; ++k) cn[k] = __ldcg(st.env_cnt + (long long)env * QS_NUM_ENV_STATS + k);
#pragma unroll
            for (int r = 0; r < 3; ++r) f[r] = __ldcg(st.scn_f + 3 * (long long)env + r);
            se[0] = c.x; se[1] = c.y; se[2] = c.z; se[3] = c.w;
#pragma unroll
            for (int k = 0; k < QS_NUM_ENV_STATS; ++k) se[4 + k] = cn[k];
            se[17] = si.x; se[18] = si.y; se[19] = si.z; se[20] = si.w;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                se[21 + 4 * r] = __float_as_int(f[r].x); se[22 + 4 * r] = __float_as_int(f[r].y);
                se[23 + 4 * r] = __float_as_int(f[r].z); se[24 + 4 * r] = __float_as_int(f[r].w);
            }
        } else {
            // counters a replay must not rewind: the RNG step counter, the episode index (and the episode number, which is
            // not part of the snapshot at all)
            const int4 live = __ldcg(st.env_ctr + env);
            int32_t sv[SNAP_ENV_I32];
#pragma unroll
            for (int k = 0; k < 33; ++k) sv[k] = __ldcg(se + k);
            st.env_ctr[env] = keep_live_counters ? make_int4(sv[0], live.y, sv[2], live.w) : make_int4(sv[0], sv[1], sv[2], sv[3]);
#pragma unroll
            for (int k = 0; k < QS_NUM_ENV_STATS; ++k) {
                // quad_experience_replay.py:188-190: the replayed episode counts its collisions from zero
                const bool zero = k == QS_STAT_NUM_COLLISIONS || k == QS_STAT_NUM_COLLISIONS_AFTER_SETTLE ||
                                  k == QS_STAT_NUM_COLLISIONS_OBST || k == QS_STAT_NUM_COLLISIONS_OBST_AFTER_SETTLE;
                st.env_cnt[(long long)env * QS_NUM_ENV_STATS + k] = zero ? 0 : sv[4 + k];
            }
            st.scn_i[env] = make_int4(sv[17], sv[18], sv[19], sv[20]);
#pragma unroll
            for (int r = 0; r < 3; ++r)
                st.scn_f[3 * (long long)env + r] = make_float4(__int_as_float(sv[21 + 4 * r]), __int_as_float(sv[22 + 4 * r]),
                                                               __int_as_float(sv[23 + 4 * r]), __int_as_float(sv[24 + 4 * r]));
        }
    }
}

// snapshot slot -> snapshot slot of the same env (checkpoint ring -> event buffer)
__device__ __forceinline__ void snap_move(const WrapView& q, int env, int i, bool valid, int src, int dst) {
    const StepParams& p = *q.sp;
    const WrapState& w = *q.w;
    const long long sb = ((long long)env * w.slots + src), db = ((long long)env * w.slots + dst);
    if (valid) {
        float4 v[NUM_SLOTS];
#pragma unroll
        for (int k = 0; k < NUM_SLOTS; ++k) v[k] = __ldcg(w.snap_slots + (sb * NUM_SLOTS + k) * p.N + i);
#pragma unroll
        for (int k = 0; k < NUM_SLOTS; ++k) w.snap_slots[(db * NUM_SLOTS + k) * p.N + i] = v[k];
        const int total = p.N * p.D;
        for (int k0 = i; k0 < total; k0 += SNAP_BATCH * p.N) {
            float t[SNAP_BATCH];
#pragma unroll
            for (int u = 0; u < SNAP_BATCH; ++u) { const int k = k0 + u * p.N; t[u] = k < total ? __ldcg(w.snap_obs + sb * total + k) : 0.f; }
#pragma unroll
            for (int u = 0; u < SNAP_BATCH; ++u) { const int k = k0 + u * p.N; if (k < total) w.snap_obs[db * total + k] = t[u]; }
        }
        for (int m = i; m < p.M; m += p.N) w.snap_obst[db * p.M + m] = __ldcg(w.snap_obst + sb * p.M + m);
        for (int k = i; k < SNAP_ENV_I32; k += p.N) w.snap_env[db * SNAP_ENV_I32 + k] = __ldcg(w.snap_env + sb * SNAP_ENV_I32 + k);
    }
}

template <int NP>
__device__ __forceinline__ void wrap_body(const WrapView& q, int env, int i) {
    const StepParams& p = *q.sp;
    const DevState& st = p.st;
    const WrapState& w = *q.w;
    const int lane = threadIdx.x & 31;
    const bool env_ok = env < p.E;
    const bool valid = env_ok && i < p.N;
    const long long a = (long long)env * p.N + i;
    const long long A = (long long)p.E * p.N;

    // (all loads of state that another block instance wrote go through L2 — __ldcg: with block-chained launches there is no
    // kernel boundary, hence no L1 invalidation, between the writer and this reader)
    // env-level words: issued here, together with the per-agent loads below (one memory round trip for everything; loaded
    // where they are used, behind the shuffle, they added two serialised ones to every block's chain)
    int steps_prev = 0;
    int4 rp = make_int4(0, 0, 0, -(1 << 30)), rq = make_int4(0, 0, 0, 0), ctr_now = make_int4(0, 0, 0, 0);
    if (env_ok) {
        steps_prev = __ldcg(w.ep_steps + env);
        if (w.replay_on) { rp = __ldcg(w.rp + env); rq = __ldcg(w.rq + env); ctr_now = __ldcg(st.env_ctr + env); }
    }

    // ---- reward shaping: accumulate this step (reward_shaping.py:66-78) ----
    float raw[QS_NUM_TERMS], rwd[QS_NUM_TERMS];
    float4 act = make_float4(0.f, 0.f, 0.f, 0.f), asum = act, asq = act;
    bool done = false;
    float term_quadcol = 0.f, term_obst = 0.f, term_crash = 0.f;
#pragma unroll
    for (int k = 0; k < QS_NUM_TERMS; ++k) { raw[k] = 0.f; rwd[k] = 0.f; }
    if (valid) {
        const float4* t4 = reinterpret_cast<const float4*>(q.terms + a * QS_NUM_TERMS);
        const float4 ta = __ldcg(t4), tb = __ldcg(t4 + 1);      // written by the step grid that may still be running: L2, not L1
        const float tt[QS_NUM_TERMS] = {ta.x, ta.y, ta.z, ta.w, tb.x, tb.y, tb.z, tb.w};
        term_quadcol = tt[QS_TERM_RAW_QUADCOL]; term_obst = tt[QS_TERM_RAW_QUADCOL_OBST]; term_crash = tt[QS_TERM_RAW_CRASH];
        const float cf[QS_NUM_TERMS] = {p.rew[QS_REW_POS], p.rew[QS_REW_EFFORT], p.rew[QS_REW_CRASH], p.rew[QS_REW_ORIENT],
                                        p.rew[QS_REW_SPIN], p.rew[QS_REW_QUADCOL_BIN], 1.0f, p.rew[QS_REW_QUADCOL_BIN_OBST]};
        float4 r0 = __ldcg(w.acc + 0 * A + a), r1 = __ldcg(w.acc + 1 * A + a), w0 = __ldcg(w.acc + 2 * A + a), w1 = __ldcg(w.acc + 3 * A + a);
        asum = __ldcg(w.acc + 4 * A + a); asq = __ldcg(w.acc + 5 * A + a);
        act = __ldcs(q.actions + a);
        r0.x += tt[0]; r0.y += tt[1]; r0.z += tt[2]; r0.w += tt[3]; r1.x += tt[4]; r1.y += tt[5]; r1.z += tt[6]; r1.w += tt[7];
        w0.x += tt[0] * cf[0]; w0.y += tt[1] * cf[1]; w0.z += tt[2] * cf[2]; w0.w += tt[3] * cf[3];
        w1.x += tt[4] * cf[4]; w1.y += tt[5] * cf[5]; w1.z += tt[6] * cf[6]; w1.w += tt[7] * cf[7];
        asum.x += act.x; asum.y += act.y; asum.z += act.z; asum.w += act.w;
        asq.x += act.x * act.x; asq.y += act.y * act.y; asq.z += act.z * act.z; asq.w += act.w * act.w;
        raw[0] = r0.x; raw[1] = r0.y; raw[2] = r0.z; raw[3] = r0.w; raw[4] = r1.x; raw[5] = r1.y; raw[6] = r1.z; raw[7] = r1.w;
        rwd[0] = w0.x; rwd[1] = w0.y; rwd[2] = w0.z; rwd[3] = w0.w; rwd[4] = w1.x; rwd[5] = w1.y; rwd[6] = w1.z; rwd[7] = w1.w;
        done = __ldcg(q.dones + a) != 0;
        if (!done) {
            w.acc[0 * A + a] = r0; w.acc[1 * A + a] = r1; w.acc[2 * A + a] = w0; w.acc[3 * A + a] = w1;
            w.acc[4 * A + a] = asum; w.acc[5 * A + a] = asq;
        }
    }
    const bool env_done = __shfl_sync(0xffffffffu, done, lane & ~(NP - 1)) && env_ok;      // all agents of an env end together
    int steps = env_ok ? steps_prev + 1 : 0;
    const bool saved = rq.x != 0;                              // the episode that ran this step is a replay
    int ev_dst = 0;

    // ---- episode end: statistics of the finished episode (reward_shaping.py:80-118, quadrotor_multi.py:626-718) ----
    if (__any_sync(0xffffffffu, env_done)) {
        // action sums of the whole env (all lanes of the warp take part in the shuffles)
        float4 env_asum = valid ? asum : make_float4(0.f, 0.f, 0.f, 0.f), env_asq = valid ? asq : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int o = NP / 2; o > 0; o >>= 1) {
            env_asum.x += __shfl_xor_sync(0xffffffffu, env_asum.x, o, NP); env_asum.y += __shfl_xor_sync(0xffffffffu, env_asum.y, o, NP);
            env_asum.z += __shfl_xor_sync(0xffffffffu, env_asum.z, o, NP); env_asum.w += __shfl_xor_sync(0xffffffffu, env_asum.w, o, NP);
            env_asq.x += __shfl_xor_sync(0xffffffffu, env_asq.x, o, NP); env_asq.y += __shfl_xor_sync(0xffffffffu, env_asq.y, o, NP);
            env_asq.z += __shfl_xor_sync(0xffffffffu, env_asq.z, o, NP); env_asq.w += __shfl_xor_sync(0xffffffffu, env_asq.w, o, NP);
        }
        if (env_done && valid) {
            const float true_reward = raw[QS_TERM_RAW_POS] + 1000.0f * raw[QS_TERM_RAW_QUADCOL];
            w.true_reward[a] = true_reward;
            const int ncol_settle = __ldcg(st.stats_env + (long long)env * QS_NUM_ENV_STATS + QS_STAT_NUM_COLLISIONS_AFTER_SETTLE);
            const int scn = min(max(__ldcg(st.stats_env + (long long)env * QS_NUM_ENV_STATS + QS_STAT_SCENARIO), 0), 15);
            if (!saved) {
                agg_add(w.agg, WA_AGENT_EPISODES, 1.0f);
                agg_add(w.agg, WA_TRUE_REWARD, true_reward);
#pragma unroll
                for (int k = 0; k < QS_NUM_TERMS; ++k) { agg_add(w.agg, WA_RAW0 + k, raw[k]); agg_add(w.agg, WA_REW0 + k, rwd[k]); }
                // z_action{k}_mean / _std: over ALL agents and steps of the env's episode jointly (reward_shaping.py:100-106
                // transposes the [T, N, 4] action log to [4, N, T] and takes np.mean / np.std of each of the 4 slices)
                const float inv = 1.0f / (float)(max(steps, 1) * p.N);
                const float am[4] = {env_asum.x * inv, env_asum.y * inv, env_asum.z * inv, env_asum.w * inv};
                const float aq[4] = {env_asq.x * inv, env_asq.y * inv, env_asq.z * inv, env_asq.w * inv};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    agg_add(w.agg, WA_ACT_MEAN0 + k, am[k]);
                    agg_add(w.agg, WA_ACT_STD0 + k, sqrtf(fmaxf(aq[k] - am[k] * am[k], 0.f)));
                }
                const float4 ags = __ldcg(st.stats_agent + a);
                agg_add(w.agg, WA_DIST0, ags.x); agg_add(w.agg, WA_DIST0 + 1, ags.y); agg_add(w.agg, WA_DIST0 + 2, ags.z);
                const uint32_t fb = __float_as_uint(ags.w);
                const bool no_col_agent = fb & 1u, no_col_obst = (fb & 2u) != 0u, reached = (fb & 4u) != 0u;
                const bool col_flag = no_col_agent && no_col_obst;
                agg_add(w.agg, WA_SUCCESS, (col_flag && reached) ? 1.f : 0.f);
                agg_add(w.agg, WA_DEADLOCK, (col_flag && !reached) ? 1.f : 0.f);
                agg_add(w.agg, WA_COL, col_flag ? 0.f : 1.f);
                agg_add(w.agg, WA_NEIGHBOR_COL, no_col_agent ? 0.f : 1.f);
                agg_add(w.agg, WA_OBST_COL, no_col_obst ? 0.f : 1.f);
                float* sc = w.agg + WA_SCN0 + 6 * scn;
                agg_add(sc, 0, 1.0f); agg_add(sc, 1, rwd[QS_TERM_RAW_POS]); agg_add(sc, 2, rwd[QS_TERM_RAW_CRASH]); agg_add(sc, 5, ags.x);
                if (i == 0) {
                    agg_add(w.agg, WA_ENV_EPISODES, 1.0f);
                    agg_add(sc, 3, 1.0f); agg_add(sc, 4, (float)ncol_settle);
                    for (int k = 0; k < 11; ++k)
                        agg_add(w.agg, WA_ENV_STAT0 + k, (float)__ldcg(st.stats_env + (long long)env * QS_NUM_ENV_STATS + k));
                }
            } else if (i == 0) {
                // a replayed episode only reports its collision counts (quadrotor_multi.py:640-649)
                agg_add(w.agg, WA_REPLAY_ENV_EPISODES, 1.0f);
                agg_add(w.agg, WA_REPLAY_COLLISIONS, (float)ncol_settle);
                agg_add(w.agg, WA_REPLAY_COLLISIONS_OBST, (float)__ldcg(st.stats_env + (long long)env * QS_NUM_ENV_STATS + QS_STAT_NUM_COLLISIONS_OBST_AFTER_SETTLE));
            }
            if (i == 0) agg_add(w.agg, WA_EPISODES_TOTAL, 1.0f);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < 6; ++k) w.acc[(long long)k * A + a] = z;
        }
        if (env_done) steps = 0;
    }
    if (env_ok && i == 0) w.ep_steps[env] = steps;
    if (!w.replay_on) return;

    // ---- collision-event replay (quad_experience_replay.py:120-209), per env, masked.  Every phase is entered by the whole
    //      warp (warp-uniform `any`), the per-env predicate selects the lanes that act; no collective sits in divergent code.
    const int gbase = lane & ~(NP - 1);
    const int tick = ctr_now.x, step_count = ctr_now.y;
    // crashes_last_episode += infos[0]['rewards']['rew_crash'] (quadrotor_multi.py:611-612): agent 0's weighted term
    const float crash = __shfl_sync(0xffffffffu, term_crash, gbase) * p.rew[QS_REW_CRASH];
    const bool col_any = group_ballot<NP>(valid && (term_quadcol < 0.f || term_obst < 0.f)) != 0u;
    const bool active = rq.y != 0;
    const bool running = env_ok && !env_done;
    bool dirty = false;

    // 1. checkpoint every 0.5 s (not while replaying an event), :140-142
    const bool cp = running && active && !saved && tick > 0 && (tick % RP_CP_EVERY) == 0;
    if (__any_sync(0xffffffffu, cp)) {
        wait_rows(q);
        if (cp) {
            snap_copy<true>(q, env, i, valid, rp.x, false);
            if (i == 0) agg_add(w.agg, WA_CHECKPOINTS, 1.0f);
            rp.x = (rp.x + 1) % RP_KEEP;
            rp.y = min(rp.y + 1, RP_KEEP);
            dirty = true;
        }
        __syncwarp();
    }
    // 2. a collision after the grace period stores the checkpoint from 1.5 s earlier, at most one event per 5 s (:144-163).
    //    The live episode goes on unflagged: only the stored copy carries saved_in_replay_buffer (:24-28).
    const bool ev = running && col_any && active && !saved && tick > RP_GRACE && tick - rp.w > RP_COOLDOWN && rp.y >= RP_STEPS_AGO;
    if (__any_sync(0xffffffffu, ev)) {
        if (ev) {
            int dst = -1;
            for (int b = 0; b < w.buffer; ++b)                       // first free slot, else round-robin (:36-45)
                if (dst < 0 && __ldcg(w.ev_state + (long long)env * w.buffer + b) < 0) dst = b;
            if (dst < 0) dst = rp.z;
            const int src = (rp.x - RP_STEPS_AGO + RP_KEEP) % RP_KEEP;
            snap_move(q, env, i, valid, src, RP_KEEP + dst);
            rp.z = (dst + 1) % w.buffer;
            rp.w = tick;
            dirty = true;
            ev_dst = dst;
        }
        __syncwarp();
        if (ev && i == 0) {
            w.ev_state[(long long)env * w.buffer + ev_dst] = 0;
            agg_add(w.agg, WA_EVENTS_STORED, 1.0f);
        }
    }
    if (running && i == 0 && crash != 0.f) w.crash_now[env] = __ldcg(w.crash_now + env) + crash;

    // 3. a finished env: can_drones_fly bookkeeping (quadrotor_multi.py:281-287,356-359), then a buffered event is replayed
    //    with probability p instead of the fresh episode the step kernel has already started (:167-209)
    if (__any_sync(0xffffffffu, env_done)) {
        wait_rows(q);                                            // a replayed event overwrites rows of this step's observation
        float mean = 0.f;
        if (env_done && i == 0) {
            const float cn = __ldcg(w.crash_now + env) + crash;
            w.crash_hist[(long long)env * 100 + (rq.z % 100)] = cn;
            w.crash_now[env] = 0.f;
            const int cnt = min(rq.z + 1, 100);
            if (cnt >= 10 && !rq.y) {
                for (int k = 0; k < cnt; ++k) mean += __ldcg(w.crash_hist + (long long)env * 100 + k);
                mean /= (float)cnt;
            }
        }
        mean = __shfl_sync(0xffffffffu, mean, gbase);
        int pick = -1;
        if (env_done) {
            rq.z += 1;
            if (w.always_active || (min(rq.z, 100) >= 10 && fabsf(mean) < 1.0f)) rq.y = 1;
            rp.y = 0; rp.w = -(1 << 30);                         // fresh-episode defaults (new_episode, :167-174)
            rq.x = 0;
            int n_valid = 0;
            for (int b = 0; b < w.buffer; ++b) n_valid += __ldcg(w.ev_state + (long long)env * w.buffer + b) >= 0 ? 1 : 0;
            const float4 u = rng_uniform4(step_key(p, env, step_count), SITE_REPLAY_U, 0, 0, 0);
            if (n_valid > 0 && rq.y && u.x < w.replay_prob) {
                int want = min((int)(u.y * (float)n_valid), n_valid - 1);
                for (int b = 0; b < w.buffer; ++b) {
                    if (__ldcg(w.ev_state + (long long)env * w.buffer + b) >= 0) {
                        if (want == 0) { pick = b; break; }
                        --want;
                    }
                }
                snap_copy<false>(q, env, i, valid, RP_KEEP + pick, true);
                rq.x = 1;                                        // the stored copy carries saved_in_replay_buffer = True
            }
            dirty = true;
        }
        __syncwarp();
        if (env_done && pick >= 0 && i == 0) {
            const int r = __ldcg(w.ev_state + (long long)env * w.buffer + pick) + 1;
            w.ev_state[(long long)env * w.buffer + pick] = r >= RP_MAX_REPLAYS ? -1 : r;          // cleanup (:56-57)
            agg_add(w.agg, WA_REPLAYED_EVENTS, 1.0f);
        }
    }
    if (env_ok && i == 0 && dirty) { w.rp[env] = rp; w.rq[env] = rq; }
}

// q.chain = 0: the kernel follows the step grid with a grid-wide wait (any launch shape; qs_wrap_apply).
// q.chain = 1: launched with the step grid's env -> block mapping behind a courier step launch (qs_wrap_step on a chained
// handle): block b takes the `done` word of step block b (all of its stores are out), does the wrappers' work for the
// block's envs — which may rewrite their state (replay) — and then hands the block to the next step grid (`ready`).  No
// grid-wide barrier is left in a wrapped control step; a block lets its dependents launch once it holds its `turn` (block b
// of the previous wrapper grid is through), see the courier warp of the step kernel.
#ifdef QS_TIMELINE
#define QS_WTL(k) do { if (threadIdx.x == 0 && blockIdx.x < 4096) q.sp.tl[((long long)q.sp.tl_slot * 4096 + blockIdx.x) * 16 + 12 + (k)] = gtime(); } while (0)
#else
#define QS_WTL(k) do { } while (0)
#endif

template <int NP>
__global__ void __launch_bounds__(256) qs_wrap_kernel(const __grid_constant__ WrapParams q) {
    const DevState& st = q.sp.st;
    __shared__ int s_ticket;
    QS_WTL(0);
    if (q.chain) {
        // instance j of wrapper block b (ticket from Tw) waits for the j-th wrapped step instance of block b to have stored its
        // state, rewards, dones and reward terms (Dw > j); its own predecessor finished before that step instance could start
        // (counters: qs_step.cuh).  The step block may still be writing its observation rows: see wait_rows.
        if (threadIdx.x == 0) s_ticket = atomicAdd(hw_word(st, q.sp.E, HW_TW), 1);
        __syncthreads();
        asm volatile("griddepcontrol.launch_dependents;");
        if (threadIdx.x == 0) counter_wait(hw_word(st, q.sp.E, HW_DW), (int)((unsigned)s_ticket + 1u), st.ready + q.sp.E, st.err_flag);
        __syncthreads();
    } else {
        asm volatile("griddepcontrol.launch_dependents;");
        asm volatile("griddepcontrol.wait;" ::: "memory");        // the step grid of this control step is complete
    }
    WrapView v;
    v.sp = &q.sp; v.w = &q.w; v.actions = q.sp.actions; v.terms = q.sp.rew_terms; v.dones = q.sp.dones; v.obs = q.sp.obs;
    v.rows = q.chain ? hw_word(st, q.sp.E, HW_RW) : nullptr;
    v.rows_want = q.chain ? (int)((unsigned)s_ticket + 1u) : 0;
    const int lane = threadIdx.x & 31;
    QS_WTL(1);
    wrap_body<NP>(v, blockIdx.x * (blockDim.x / NP) + threadIdx.x / NP, lane & (NP - 1));
    QS_WTL(2);
    if (q.chain) {
        __syncthreads();
        if (threadIdx.x == 0) {
            counter_wait(hw_word(st, q.sp.E, HW_RW), v.rows_want, st.ready + q.sp.E, st.err_flag);      // the step block is through: its rows are out
            counter_inc(hw_word(st, q.sp.E, HW_S));                  // the block's state goes to the next step instance
        }
    }
    QS_WTL(3);
}

}  // namespace qs
