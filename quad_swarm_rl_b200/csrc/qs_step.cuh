// The fused env-step kernel: per-drone dynamics -> all-pairs collision / proximity / downwash ->
// contact responses -> observation assembly -> episode bookkeeping and auto-reset, ONE launch per
// control step (or T control steps per launch for qs_rollout, state kept in registers).
//
// Thread mapping: NP = next power of two >= N lanes per env, 32/NP envs per warp; lane i of a group owns
// drone i.  All cross-drone traffic is __shfl_sync within the group; the env's pillar table is staged in
// shared memory.  Follows QuadrotorEnvMulti.step, quadrotor_multi.py:413-724 (see DESIGN.md for the map).
//
// Shape of the code: at the benchmark sizes the GPU holds < 2 warps per SM sub-partition, so the kernel
// is bound by instruction fetch and dependent-issue latency, not by HBM or issue slots.  Hence: rolled
// loops (small instruction footprint), SFU approximations instead of the branchy IEEE sqrt/div
// sequences, trigonometry-free contact code, and every rare path (contact responses, random yaw, reset,
// re-drawn sensor noise) out of line.
#pragma once
#include "qs_device.cuh"
#include "qs_scenario.cuh"
#include "qs_dyn_sampler.cuh"

namespace qs {

#ifdef QS_TIMELINE
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
#define QS_TL(k) do { if (threadIdx.x == 0 && blockIdx.x < 4096) { p.tl[((long long)p.tl_slot * 4096 + blockIdx.x) * 16 + (k)] = gtime(); \
    if ((k) == 0) { unsigned sm; asm volatile("mov.u32 %0, %smid;" : "=r"(sm)); p.tl[((long long)p.tl_slot * 4096 + blockIdx.x) * 16 + 8] = sm; } } } while (0)
#else
#define QS_TL(k) do { } while (0)
#endif

struct EnvCtr {
    int tick, step_count, svd_count, episode_idx;
};

// smallest squared centre distance from the drone to a pillar of its env
__device__ __forceinline__ float min_pillar_dist2(const StepParams& p, const Agent& s, const float2* s_obst_env) {
    float dmin2 = 1e4f;
#pragma unroll 4
    for (int m = 0; m < p.M; ++m) {
        const float2 ob = s_obst_env[m];
        const float dx = s.pos[0] - ob.x, dy = s.pos[1] - ob.y;
        dmin2 = fminf(dmin2, dx * dx + dy * dy);
    }
    return dmin2;
}

// Observation row of one drone: get_state.py:6-72 (self part), quadrotor_multi.py:233-274 (neighbours),
// obstacles/utils.py:5-27 (3x3 SDF).  `nvel` is the velocity the neighbour block sees (stale after a reset,
// SURVEY Appendix D-6); `nz` is the scaled sensor noise of this observation.
// `row` points either at the drone's row in global memory or at its row of the warp's shared-memory staging tile
// (see flush_observation_tile).
// Hand-off arrays of the split (physics warp -> observer warp) kernel: 24 arrays of 32 floats in shared memory.
enum Hand { H_PX = 0, H_PY, H_PZ, H_VX, H_VY, H_VZ, H_NVX, H_NVY, H_NVZ, H_R0, H_OX = H_R0 + 9, H_OY, H_OZ, H_GX, H_GY, H_GZ, H_COUNT };
constexpr int HAND_FLOATS = 2 * H_COUNT * 32 + 32;      // post-integration buffer, final-state buffer, one flag word per lane
constexpr uint32_t HF_KICKED = 1u, HF_RESET = 2u;

// value of drone j of my env: from the hand-off arrays (SM) or by warp shuffle from the lane that owns it
template <int NP, bool SM>
__device__ __forceinline__ float nbv(float mine, const float* hand, int arr, int gbase, int j) {
    if (SM) return hand[32 * arr + gbase + j];
    return __shfl_sync(0xffffffffu, mine, j, NP);
}

template <int NP, bool SM = false>
__device__ __forceinline__ void write_observation(const StepParams& p, const Agent& s, const float nvel[3], const Noise9& nz,
                                                  int i, bool valid, const float2* s_obst_env, float dmin2,
                                                  float* __restrict__ row, float obst_r, const float* hand = nullptr, int gbase = 0) {
    // ---- self observation
    {
        const float px = s.pos[0] + nz.p[0], py = s.pos[1] + nz.p[1], pz = s.pos[2] + nz.p[2];
        // The reference observes quat2R(rot2quat(R)) (sensor_noise.py:205-210); with the default noise set the rotation
        // noise is exactly zero, the round trip is the identity up to rounding (<= 4e-16 in float64, SURVEY Appendix D-8),
        // so R is emitted directly.  The custom model's rotation noise (NZ) passes s.R = observed_rotation() in.
        const float* rot = s.R;
        if (valid) {
            row[0] = px - s.goal[0]; row[1] = py - s.goal[1]; row[2] = pz - s.goal[2];
            row[3] = s.vel[0] + nz.v[0]; row[4] = s.vel[1] + nz.v[1]; row[5] = s.vel[2] + nz.v[2];
#pragma unroll
            for (int k = 0; k < 9; ++k) row[6 + k] = rot[k];
            row[15] = s.om[0] + nz.w[0]; row[16] = s.om[1] + nz.w[1]; row[17] = s.om[2] + nz.w[2];
            if (p.obs_repr == QS_OBS_XYZ_VXYZ_R_OMEGA_FLOOR) {
                row[18] = pz;
            } else if (p.obs_repr == QS_OBS_XYZ_VXYZ_R_OMEGA_WALL) {
                row[18] = clampf(px - p.room_lo[0], 0.f, 5.f); row[19] = clampf(py - p.room_lo[1], 0.f, 5.f);
                row[20] = clampf(pz - p.room_lo[2], 0.f, 5.f);
                row[21] = clampf(p.room_hi[0] - px, 0.f, 5.f); row[22] = clampf(p.room_hi[1] - py, 0.f, 5.f);
                row[23] = clampf(p.room_hi[2] - pz, 0.f, 5.f);
            }
        }
    }

    // ---- neighbour block: K nearest by distance + closing speed, or all others in index order
    if (NP > 1 && p.K > 0) {
        const float rx = p.room_hi[0] - p.room_lo[0], ry = p.room_hi[1] - p.room_lo[1], rz = p.room_hi[2] - p.room_lo[2];
        const float rv = 2.0f * VXYZ_MAX;
        float* nrow = row + p.S;
        if (p.K == p.N - 1) {
            int slot = 0;
#pragma unroll 1
            for (int j = 0; j < p.N; ++j) {
                const float qx = nbv<NP, SM>(s.pos[0], hand, H_PX, gbase, j), qy = nbv<NP, SM>(s.pos[1], hand, H_PY, gbase, j), qz = nbv<NP, SM>(s.pos[2], hand, H_PZ, gbase, j);
                const float wx = nbv<NP, SM>(nvel[0], hand, H_NVX, gbase, j), wy = nbv<NP, SM>(nvel[1], hand, H_NVY, gbase, j), wz = nbv<NP, SM>(nvel[2], hand, H_NVZ, gbase, j);
                if (j != i && valid) {
                    float* d = nrow + 6 * slot;
                    d[0] = clampf(qx - s.pos[0], -rx, rx); d[1] = clampf(qy - s.pos[1], -ry, ry);
                    d[2] = clampf(qz - s.pos[2], -rz, rz);
                    d[3] = clampf(wx - nvel[0], -rv, rv); d[4] = clampf(wy - nvel[1], -rv, rv);
                    d[5] = clampf(wz - nvel[2], -rv, rv);
                    ++slot;
                }
            }
        } else {
            // score_j = max(|dp|, 0.01) + dp_hat . dv (quadrotor_multi.py:259-266); kept in registers
            float score[NP];
#pragma unroll
            for (int j = 0; j < NP; ++j) {
                const float dx = nbv<NP, SM>(s.pos[0], hand, H_PX, gbase, j) - s.pos[0], dy = nbv<NP, SM>(s.pos[1], hand, H_PY, gbase, j) - s.pos[1],
                            dz = nbv<NP, SM>(s.pos[2], hand, H_PZ, gbase, j) - s.pos[2];
                const float ux = nbv<NP, SM>(nvel[0], hand, H_NVX, gbase, j) - nvel[0], uy = nbv<NP, SM>(nvel[1], hand, H_NVY, gbase, j) - nvel[1],
                            uz = nbv<NP, SM>(nvel[2], hand, H_NVZ, gbase, j) - nvel[2];
                const float dist = fmaxf(norm3(dx, dy, dz), 0.01f);
                const float sc = dist + (dx * ux + dy * uy + dz * uz) * frcp(dist);
                score[j] = (j < p.N && j != i) ? sc : __int_as_float(0x7f800000);   // +inf: never selected
            }
#pragma unroll 1
            for (int k = 0; k < p.K; ++k) {
                // stable argsort: strictly smaller score wins, ties keep the lower index (Appendix D-11); a taken
                // candidate's score is overwritten with +inf; K <= N - 2 guarantees a finite score remains
                float best = score[0];
                int bj = 0;
#pragma unroll
                for (int j = 1; j < NP; ++j) {
                    const bool better = score[j] < best;
                    best = better ? score[j] : best;
                    bj = better ? j : bj;
                }
                const int src = bj;
#pragma unroll
                for (int j = 0; j < NP; ++j) score[j] = (j == src) ? __int_as_float(0x7f800000) : score[j];
                const float qx = nbv<NP, SM>(s.pos[0], hand, H_PX, gbase, src), qy = nbv<NP, SM>(s.pos[1], hand, H_PY, gbase, src), qz = nbv<NP, SM>(s.pos[2], hand, H_PZ, gbase, src);
                const float wx = nbv<NP, SM>(nvel[0], hand, H_NVX, gbase, src), wy = nbv<NP, SM>(nvel[1], hand, H_NVY, gbase, src), wz = nbv<NP, SM>(nvel[2], hand, H_NVZ, gbase, src);
                if (valid) {
                    float* d = nrow + 6 * k;
                    d[0] = clampf(qx - s.pos[0], -rx, rx); d[1] = clampf(qy - s.pos[1], -ry, ry);
                    d[2] = clampf(qz - s.pos[2], -rz, rz);
                    d[3] = clampf(wx - nvel[0], -rv, rv); d[4] = clampf(wy - nvel[1], -rv, rv);
                    d[5] = clampf(wz - nvel[2], -rv, rv);
                }
            }
        }
    }

    // ---- 3x3 signed-distance patch around the drone (resolution 0.1 m, obstacles/utils.py:5-27):
    //      cell value = min over pillars of |cell - pillar| - radius.  A pillar whose CENTRE distance exceeds the
    //      smallest centre distance by more than 2 sqrt(2) * 0.1 cannot be the nearest pillar of any of the 9 cells
    //      (triangle inequality), so only the few qualifying pillars get the 9-cell update; the min is taken on
    //      squared distances and one square root per cell follows (sqrt is monotone).
    if (p.use_obst) {
        const float res = 0.1f;
        const float lim = fsqrt(dmin2) + (2.0f * 1.41421356f * res + 1e-4f);
        const float lim2 = lim * lim;
        uint32_t cand = 0u;
        const int Mb = min(p.M, 32);
#pragma unroll 4
        for (int m = 0; m < Mb; ++m) {
            const float2 ob = s_obst_env[m];
            const float dx = s.pos[0] - ob.x, dy = s.pos[1] - ob.y;
            cand |= (dx * dx + dy * dy <= lim2) ? (1u << m) : 0u;
        }
        const float gx0 = s.pos[0] - res, gx1 = s.pos[0], gx2 = s.pos[0] + res;
        const float gy0 = s.pos[1] - res, gy1 = s.pos[1], gy2 = s.pos[1] + res;
        float b0 = 1e4f, b1 = 1e4f, b2 = 1e4f, b3 = 1e4f, b4 = 1e4f, b5 = 1e4f, b6 = 1e4f, b7 = 1e4f, b8 = 1e4f;
#define QS_SDF_UPDATE(ob)                                                                                                  \
        {                                                                                                                  \
            const float ex0 = (gx0 - ob.x) * (gx0 - ob.x), ex1 = (gx1 - ob.x) * (gx1 - ob.x), ex2 = (gx2 - ob.x) * (gx2 - ob.x); \
            const float ey0 = (gy0 - ob.y) * (gy0 - ob.y), ey1 = (gy1 - ob.y) * (gy1 - ob.y), ey2 = (gy2 - ob.y) * (gy2 - ob.y); \
            b0 = fminf(b0, ex0 + ey0); b1 = fminf(b1, ex0 + ey1); b2 = fminf(b2, ex0 + ey2);                                \
            b3 = fminf(b3, ex1 + ey0); b4 = fminf(b4, ex1 + ey1); b5 = fminf(b5, ex1 + ey2);                                \
            b6 = fminf(b6, ex2 + ey0); b7 = fminf(b7, ex2 + ey1); b8 = fminf(b8, ex2 + ey2);                                \
        }
        while (cand != 0u) {
            const int m = __ffs(cand) - 1;
            cand &= cand - 1u;
            const float2 ob = s_obst_env[m];
            QS_SDF_UPDATE(ob)
        }
        for (int m = 32; m < p.M; ++m) {        // tables with more than 32 pillars: plain scan of the tail
            const float2 ob = s_obst_env[m];
            QS_SDF_UPDATE(ob)
        }
#undef QS_SDF_UPDATE
        if (valid) {
            float* srow = row + p.S + 6 * p.K;
            const float r = obst_r;
            srow[0] = fsqrt(b0) - r; srow[1] = fsqrt(b1) - r; srow[2] = fsqrt(b2) - r;
            srow[3] = fsqrt(b3) - r; srow[4] = fsqrt(b4) - r; srow[5] = fsqrt(b5) - r;
            srow[6] = fsqrt(b6) - r; srow[7] = fsqrt(b7) - r; srow[8] = fsqrt(b8) - r;
        }
    }
}

// Coalesced write-out of a warp's observation tile.  The rows of the drones a warp owns are contiguous in global
// memory ([A][D] row-major, consecutive agents), so the tile staged in shared memory (row stride Dp) is copied out
// with full-width vector stores: chunk c of V floats -> row c / Q, column (c % Q) * V, Q = D / V.
__device__ __forceinline__ void flush_observation_tile(const StepParams& p, const float* tile, float* __restrict__ gdst, int n_rows,
                                                       int lane) {
    const int Q = p.obs_q, V = p.obs_v, Dp = p.obs_dp;
    const int total = n_rows * Q;
    if (V == 4) {
#pragma unroll 2
        for (int c = lane; c < total; c += 32) {
            const int r = (int)(((unsigned)c * (unsigned)p.obs_magic) >> 20);
            const int q = c - r * Q;
            __stcs(reinterpret_cast<float4*>(gdst + 4 * c), *reinterpret_cast<const float4*>(tile + r * Dp + 4 * q));
        }
    } else if (V == 2) {
#pragma unroll 2
        for (int c = lane; c < total; c += 32) {
            const int r = (int)(((unsigned)c * (unsigned)p.obs_magic) >> 20);
            const int q = c - r * Q;
            __stcs(reinterpret_cast<float2*>(gdst + 2 * c), *reinterpret_cast<const float2*>(tile + r * Dp + 2 * q));
        }
    } else {
#pragma unroll 2
        for (int c = lane; c < total; c += 32) {
            const int r = (int)(((unsigned)c * (unsigned)p.obs_magic) >> 20);
            const int q = c - r * Q;
            __stcs(gdst + c, tile[r * Dp + q]);
        }
    }
}

// ---- asynchronous write-out of a staged observation tile (bulk-copy / TMA engine, shared -> global) ----
// A warp's rows are one contiguous span of the [T][A][D] observation array.  Instead of the copy loop above (161 executed
// instructions per warp and step on c3, plus the LSU round trip), ONE elected lane hands the tile to the copy engine:
//   obs_bulk 1 (D % 4 == 0): cp.async.bulk.tensor.3d store through a tensor map of the caller's observation array
//               ([T][A][D] floats, box = [1][rows per tile][Dp]).  The box is as wide as the PADDED shared-memory row
//               (Dp > D keeps the row writes at the 4-way bank-conflict optimum of 16-byte aligned rows); columns >= D
//               and rows >= A lie outside the tensor and are clipped by the engine, so ragged last tiles need no code.
//   obs_bulk 2 (otherwise): rows are staged unpadded (stride D: 2-way conflicts for D = 54) and the tile leaves with one
//               linear cp.async.bulk when its byte count and global address are multiples of 16; the copy loop covers
//               the rare remainder.
// The generic-proxy writes of the lanes are ordered before the async proxy's reads by fence.proxy.async + __syncwarp; the
// tile may be rewritten (or the CTA may exit) only after cp.async.bulk.wait_group.read 0 — bulk_drain() below.
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// the observation stream is written once and read by another kernel much later: L2 evict-first, so that it does not push
// the env state (re-read every step) out of the cache
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(gdst), "r"(smem_u32(ssrc)),
                 "r"(bytes), "l"(l2_evict_first_policy())
                 : "memory");
}
__device__ __forceinline__ void tensor_s2g_3d(const void* tmap, const void* ssrc, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%1, %2, %3}], [%4], %5;" ::"l"(tmap),
                 "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(ssrc)), "l"(l2_evict_first_policy())
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_drain() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// rows [0, n_rows) of `tile` -> row `row0` of step `t` of the observation array (gdst = its address)
__device__ __forceinline__ void emit_observation_tile(const StepParams& p, const float* tile, float* __restrict__ gdst, int row0, int t,
                                                      int n_rows, int lane) {
    if (p.obs_bulk == 1) {
        fence_async_smem();
        __syncwarp();
        if (lane == 0) {
            tensor_s2g_3d(&p.obs_map, tile, 0, row0, t);
            bulk_commit();
        }
        return;
    }
    if (p.obs_bulk == 2) {
        const uint32_t bytes = (uint32_t)(n_rows * p.D) * 4u;
        if (((bytes | (uint32_t)(uintptr_t)gdst) & 15u) == 0u) {
            fence_async_smem();
            __syncwarp();
            if (lane == 0) {
                bulk_s2g(gdst, tile, bytes);
                bulk_commit();
            }
            return;
        }
    }
    __syncwarp();
    flush_observation_tile(p, tile, gdst, n_rows, lane);
}

// ---- episodes ----
// An episode (pillar table, goals, spawn poses, scenario state) is a function of (seed, env id, episode number): its draws
// are keyed by the episode number (qs_rng.cuh, EPISODE_KEY_BIT).  generate_episode() is therefore the same whether it runs
// inside the reset path of a step / reset kernel or ahead of time in qs_pregen_kernel, which fills the env's NEXT-episode
// record (next_goal / next_spawn / next_obst / next_scn_*) off the step's critical path; an (auto-)reset that finds the
// record of its episode only copies it.  (Envs that reset in different steps, as in training with collision-event replay,
// would otherwise put one ~20 k-instruction generator on the critical path of EVERY step.)
struct EpisodeLane { V3 goal; ResetPose pose; int scn_next; float approach; float obst_r; };

// key of the draws of env `env` in the step with the env's step counter `step`
__device__ __forceinline__ RngKey step_key(const StepParams& p, int env, uint32_t step) {
    RngKey k;
    k.k0 = p.seed_lo; k.k1 = p.seed_hi;
    k.env = (uint32_t)(p.env_id_offset + env);
    k.step = step;
    return k;
}

// (the episode word is set last: as step_key's argument it is computed first, which changes the reset path's register allocation)
__device__ __forceinline__ RngKey episode_key(const StepParams& p, int env, int episode) {
    RngKey k = step_key(p, env, 0u);
    k.step = EPISODE_KEY_BIT | (uint32_t)episode;
    return k;
}

// true when the kernels generate the episodes (no host tables)
template <bool SCN>
__device__ __forceinline__ bool device_generated(const StepParams& p) {
    return (p.use_obst && p.scenario != QS_SCENARIO_HOST_TABLES && (SCN || !ticked_obstacle_scenario(p.scenario))) ||
           (SCN && !p.use_obst && p.scenario >= QS_SCENARIO_DEVICE_FAMILY_FIRST);
}

// this lane's share of the env's next episode; the env-level parts go to (obst_smem,) obst_dst, scn_i_dst, scn_f_dst
template <bool SCN>
__device__ __forceinline__ EpisodeLane generate_episode(const StepParams& p, const RngKey& ekey, int i, float2* obst_smem,
                                                        float2* obst_dst, int4* scn_i_dst, float4* scn_f_dst) {
    EpisodeLane e;
    e.scn_next = SCN_NEVER;
    e.approach = p.approach_metric;
    e.obst_r = p.obst_radius;
    V3 spawn;
    if (p.use_obst) {
        // pillar count and size of this episode (ExperienceReplayWrapper's domain randomisation, quad_experience_replay.py:
        // 108-118 -> reset(obst_density, obst_size), quadrotor_multi.py:339-351): uniform picks from the configured lists
        int M_e = p.M;
        if (p.obst_random) {
            M_e = p.obst_counts[scenario_pick(ekey, 322, p.n_obst_counts)];
            e.obst_r = p.obst_radii[scenario_pick(ekey, 323, p.n_obst_radii)];
        }
        // o_random / o_static_same_goal / their mix; every lane also writes its share of the pillar table
        const ORandomEpisode ep = o_random_episode(ekey, p.scenario, i, p.N, M_e, p.grid_l, p.grid_w, i, p.N, obst_smem, obst_dst, p.M);
        e.goal = ep.goal;
        spawn = ep.spawn;
        if (p.scenario != QS_SCENARIO_O_RANDOM)           // per-episode scenario id + its approch_goal_metric (o_base.py:16)
            e.approach = ep.mode == QS_SCENARIO_O_RANDOM ? 0.5f : 1.0f;
        if (SCN && ticked_obstacle_scenario(ep.mode)) {
            const ScnOut o = o_episode_extras(ekey, ep.mode, p.N, i, ep.mask, p.grid_l, p.grid_w, ep.goal, e.obst_r, M_e, scn_i_dst, scn_f_dst);
            e.goal = o.goal;
            e.scn_next = o.next;
        } else if (i == 0) {
            scn_i_dst[0] = make_int4(ep.mode, 0, SCN_NEVER, 0);
            scn_f_dst[0] = make_float4(e.obst_r, (float)M_e, 0.f, 0.f);
            scn_f_dst[1] = make_float4(0.f, 0.f, 0.f, e.approach);
            scn_f_dst[2] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    } else if (SCN) {
        // goal formation of the env's scenario; drones spawn around their goals
        const ScnOut o = scenario_reset(ekey, p.scenario, p.N, i, scn_i_dst, scn_f_dst);
        e.goal = o.goal;
        spawn = o.goal;
        e.scn_next = o.next;
    } else {
        e.goal.x = 0.f; e.goal.y = 0.f; e.goal.z = 2.f;      // not reached: device_generated<SCN>() is false
        spawn = e.goal;
    }
    e.pose = reset_pose(ekey, i, spawn, p.use_obst ? 0.1f : 2.0f);      // box: quadrotor_single.py:215-218
    return e;
}

// Start the next episode of one env and respawn its drones (QuadrotorEnvMulti.reset, quadrotor_multi.py:339-411).
// Called by ALL lanes of a warp (the branch around it is warp-uniform); `do_reset` is per env.  Sets nvel to the velocity
// the neighbour block must see.  init_random: the spawns get random initial states (p.init_random; a compile-time constant
// in the reset kernel).
template <int NP, bool SCN>
__device__ __forceinline__ void reset_env(const StepParams& p, const RngKey& key, Agent& s, long long a, int env, int i,
                                          bool do_reset, bool valid, int tick_before_reset, float2* s_obst_env,
                                          float nvel[3], int& scn_next, float& approach, float& obst_r, bool init_random) {
    const DevState& st = p.st;
    if (do_reset && valid) {
        // stale velocity (Appendix D-6): the multi-env's self.vel is only refreshed by step()
        if (tick_before_reset > 0) {
            nvel[0] = s.vel[0]; nvel[1] = s.vel[1]; nvel[2] = s.vel[2];
        } else {
            const float4 sv = QS_LD(st.slots + SL_STALE_VEL * st.a_pad + a);
            nvel[0] = sv.x; nvel[1] = sv.y; nvel[2] = sv.z;
        }
        st.slots[SL_STALE_VEL * st.a_pad + a] = make_float4(nvel[0], nvel[1], nvel[2], 0.f);
        const int2 ep = QS_LD(st.epi + env);
        const int g = ep.x + 1;                                   // number of the episode that starts now
        ResetPose rp;
        if (device_generated<SCN>(p)) {
            const long long e3 = 3 * (long long)env;
            if (ep.y == g) {
                // the episode was generated ahead of time: copy its record
                const float4 ng = QS_LD(st.next_goal + a), ns = QS_LD(st.next_spawn + a);
                s.goal[0] = ng.x; s.goal[1] = ng.y; s.goal[2] = ng.z;
                rp.pos.x = ns.x; rp.pos.y = ns.y; rp.pos.z = ns.z; rp.cs = ng.w; rp.sn = ns.w;
                if (p.use_obst) {
                    for (int m = i; m < p.M; m += p.N) {
                        const float2 ob = QS_LD(st.next_obst + (long long)env * p.M + m);
                        st.obst[(long long)env * p.M + m] = ob;
                        if (s_obst_env != nullptr) s_obst_env[m] = ob;
                    }
                }
                const int4 nsi = QS_LD(st.next_scn_i + env);
                const float4 f1 = QS_LD(st.next_scn_f + e3 + 1);
                if (p.obst_random) obst_r = QS_LD(st.next_scn_f + e3).x;
                scn_next = nsi.z;
                if (p.use_obst && p.scenario != QS_SCENARIO_O_RANDOM) approach = f1.w;
                if (i == 0) {
                    st.scn_i[env] = nsi;
                    st.scn_f[e3] = QS_LD(st.next_scn_f + e3);
                    st.scn_f[e3 + 1] = f1;
                    st.scn_f[e3 + 2] = QS_LD(st.next_scn_f + e3 + 2);
                }
            } else {
                const EpisodeLane e = generate_episode<SCN>(p, episode_key(p, env, g), i, s_obst_env, st.obst + (long long)env * p.M,
                                                            st.scn_i + env, st.scn_f + e3);
                s.goal[0] = e.goal.x; s.goal[1] = e.goal.y; s.goal[2] = e.goal.z;
                rp = e.pose;
                scn_next = e.scn_next;
                obst_r = e.obst_r;
                if (p.use_obst && p.scenario != QS_SCENARIO_O_RANDOM) approach = e.approach;
            }
        } else {
            // host tables (qs_set_next_episode); the spawn jitter / yaw draws are episode-keyed like everywhere
            const float4 gq = st.next_goal[a], sp = st.next_spawn[a];
            s.goal[0] = gq.x; s.goal[1] = gq.y; s.goal[2] = gq.z;
            V3 spawn;
            spawn.x = sp.w != 0.f ? sp.x : gq.x; spawn.y = sp.w != 0.f ? sp.y : gq.y; spawn.z = sp.w != 0.f ? sp.z : gq.z;
            rp = reset_pose(episode_key(p, env, g), i, spawn, p.use_obst ? 0.1f : 2.0f);
            if (p.obst_random) {        // the pillar radius of this episode (qs_set_next_obstacle_radius)
                const float4 nr = QS_LD(st.next_scn_f + 3 * (long long)env);
                obst_r = nr.x;
                if (i == 0) st.scn_f[3 * (long long)env] = nr;
            }
        }
        if (i == 0) st.epi[env] = make_int2(g, ep.y);
        apply_reset(s, rp);
        if (init_random) {          // a handle-wide setting; episode-keyed, so a pre-generated record needs no extra field
            const InitState r = random_init_state(episode_key(p, env, g), i, p.init_vel_max, p.init_omega_max);
#pragma unroll
            for (int k = 0; k < 3; ++k) { s.vel[k] = r.vel[k]; s.om[k] = r.om[k]; }
#pragma unroll
            for (int k = 0; k < 9; ++k) s.R[k] = r.R[k];
        }
        st.slots[SL_DIST_SUMS * st.a_pad + a] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (p.use_obst) {
        if (do_reset && p.scenario == QS_SCENARIO_HOST_TABLES) {
            for (int m = i; m < p.M; m += NP) {
                const float2 ob = st.next_obst[(long long)env * p.M + m];
                st.obst[(long long)env * p.M + m] = ob;
                if (s_obst_env != nullptr) s_obst_env[m] = ob;
            }
        }
        __syncwarp();
    }
}

// Largest balanced CTA: 8 worker warps + the courier, or 9 worker warps without it (plan_step, quadswarm.cu).
#define QS_LB 288
// Register budget of the step instantiations.  The ones that can carry the courier warp (NP < 16, single-warp, per-block
// hand-over, no DYN / NZ / SCN) get 128 registers per thread: plan_step gives c3 / c5 (1024 physics warps, 132 SMs on H100)
// 256 CTAs of 4 workers + courier = 160 threads, and 160 x 128 = 20,480 registers let three such CTAs share an SM's 65,536,
// so the successor's CTA of a block starts on an SM beside this step's (at 152 allocated registers, 288-thread CTAs of
// 8 + 1 warps fit once: 43,776).  The bound is written as 512 threads per CTA (65,536 / 512 = 128) rather than (256, 2):
// the same instantiations also run the 288-thread balanced CTAs.  The other instantiations (split, DYN, NZ, SCN with its
// scenario generators, NP >= 16) keep one 288-thread (or 128-thread) CTA as their bound.
template <int NP, bool SPLIT, bool SCN, bool HO, bool DYN, bool NZ>
__host__ __device__ constexpr bool courier_capable() { return NP < 16 && !SPLIT && !SCN && HO && !DYN && !NZ; }
template <int NP, bool SPLIT, bool SCN, bool HO, bool DYN, bool NZ>
__host__ __device__ constexpr int step_max_threads() { return courier_capable<NP, SPLIT, SCN, HO, DYN, NZ>() ? 512 : (NP >= 16 ? 128 : QS_LB); }
// named barriers of the split kernel (physics warp <-> observer warp, 64 threads).  Both warps use bar.sync: the
// observer reaches barrier 1 first, the physics warp reaches barrier 2 first and has only its stores left to do.
// Out of line on purpose: both warps then execute the SAME bar.sync instruction (what compute-sanitizer's synccheck
// expects of a CTA-wide barrier), and the call boundary keeps the compiler from moving shared-memory traffic across it.
__device__ __noinline__ void bar_sync(int id) {
    __syncwarp();          // bar.sync is warp-aligned: lanes that diverged in the preceding code must reconverge first
    asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory");
}
// Barriers between the worker warps and the courier warp (single-warp shapes): producer / consumer pairs on named barriers —
// the side that has something to wait for executes bar.sync, the side that only reports executes bar.arrive and goes on.
// `n` = all threads of the CTA.  (Ids: 1 state may be loaded, 4 ... in a wrapped chain, 2 state stored, 3 all stores issued.)
__device__ __forceinline__ void named_sync(int id, int n) {
    __syncwarp();
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}
// threads of the CTA and this thread's index, read where they are used (volatile: not kept in registers across the step
// body of the courier-capable kernels, whose register budget is tight)
__device__ __forceinline__ int block_threads() {
    int n;
    asm volatile("mov.u32 %0, %%ntid.x;" : "=r"(n));
    return n;
}
__device__ __forceinline__ int thread_index() {
    int n;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(n));
    return n;
}
__device__ __forceinline__ void named_arrive(int id, int n) {
    __syncwarp();
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}
// one-shot shared-memory mbarrier (one arrival): the courier tells the workers something without making them wait for each other
__device__ __forceinline__ void mbar_init(unsigned long long* b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* b) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"((unsigned)__cvta_generic_to_shared(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, int parity) {
    int ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.s32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"((unsigned)__cvta_generic_to_shared(b)), "r"(parity) : "memory");
    } while (!ok);
}

// running episode counter += v.  A reduction (RED.ADD, no return value): a load + store pair per counter put one L2
// round trip per counter on the critical path of every warp with a discrete event.
__device__ __forceinline__ void cnt_add(int32_t* c, int k, int v) { if (v != 0) atomicAdd(c + k, v); }

// Polls a hand-over word with acquire loads while WAITING(value, want) holds, at most 2^24 times with a 40 ns back-off (~1 s:
// a lost hand-over must not hang the GPU).  Returns whether it gave up.  A flag is waited for until it is set, a counter
// until it reaches `want` (compared as a difference: the counters wrap around after 2^32 steps).
__device__ __forceinline__ bool flag_unset(int v, int) { return v == 0; }
__device__ __forceinline__ bool counter_below(int v, int want) { return v - want < 0; }
template <bool (*WAITING)(int, int)>
__device__ __forceinline__ bool poll_acquire(const int* word, int want) {
    int v = 0, spins = 0;
    do {
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(word) : "memory");
        if (WAITING(v, want)) __nanosleep(40);
    } while (WAITING(v, want) && ++spins < (1 << 24));
    return WAITING(v, want);
}
// A hand-over that timed out: the env block is stepped from state that may be incomplete.  Counted (qs_handover_timeouts) and
// latched in the handle's sticky error word: every later qs_step fails.
__device__ __forceinline__ void report_handover_timeout(int* timeouts, int* err_flag) {
    atomicAdd(timeouts, 1);
    if (err_flag != nullptr) *reinterpret_cast<volatile int*>(err_flag) = 1;
    __threadfence_system();
}

// ---- per-block hand-over between consecutive step grids (HO kernels) ----
// Envs are independent, so block b of step t+1 only needs block b of step t.  Every step launch carries the programmatic
// stream-serialization attribute; instead of griddepcontrol.wait (a grid-wide barrier: every step then costs the launch
// latency plus the SLOWEST warp of the grid) a block waits for its own predecessor's `ready` word, takes it, and only
// then lets the next grid start launching — so at most two step grids overlap and a block of step t+2 can never see the
// word block b(t) left for b(t+1).  The writer publishes with barrier + st.release; the reader acquires
// and reads the state with ld.global.cg (L1 is not coherent across the grids).  Any other kernel / copy on the stream
// never triggers early, so it still sees, and is seen by, whole step grids.  (This flag protocol, run by thread 0, serves the
// split and the multi-wave shapes; balanced single-wave grids use the counters of the courier warp below.)
__device__ __forceinline__ void handover_acquire(int* ready, int* timeouts, int* err_flag) {
    if (poll_acquire<flag_unset>(ready, 0)) report_handover_timeout(timeouts, err_flag);
    asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(ready), "r"(0) : "memory");
}
// st.release = fence + store (SASS: MEMBAR.ALL.GPU; STG.E.STRONG.GPU); an extra __threadfence() in front of it was a second,
// sequentially consistent membar on the block's critical path.  The writes of the block's other threads are ordered before
// it by the barrier they arrived at (cumulativity).
__device__ __forceinline__ void handover_release(int* ready) {
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(ready), "r"(1) : "memory");
}
// ---- courier warps: the same hand-over with COUNTERS instead of flags ----
// A block publishes its env state BEFORE it writes the observation rows ("early hand-over", see the kernel), and a block lets
// its dependents launch the moment it starts — so several generations of block b can be resident and waiting at once, which
// a flag with one waiter cannot express.  Per block b, all monotonic (a replayed CUDA graph repeats its kernel parameters,
// so nothing here comes from the host):
//   T  tickets: instance k of block b takes k = T++ when it starts (before it lets the next grid launch, so tickets follow
//      the launch order);
//   S  states handed on: instance k waits for S >= k, and S becomes k + 1 when the state it left may be used — by the block
//      itself as soon as the state is stored, or by the wrapper kernel's block in a wrapped control step;
//   D  instances whose LAST store is out: instance k waits for D >= k before its own observation rows may be written
//      (same addresses when the caller reuses one array);
//   Tw / Dw / Rw  the wrapper kernel's tickets, the number of wrapped step instances whose state (and rewards, dones, reward
//      terms) is stored, and the number of those whose last store is out (qs_wrap_kernel).
// At rest T = S = D and Tw = Dw = Rw; an unchained launch needs no special case.
enum { HW_READY = 0, HW_T = 1, HW_S = 2, HW_D = 3, HW_TW = 4, HW_DW = 5, HW_RW = 6, HW_ROWS = 7 };     // rows of DevState::ready, [E + 1] each
__device__ __forceinline__ int* hw_word(const DevState& st, int E, int row) { return st.ready + (long long)row * (E + 1) + blockIdx.x; }
// poll_acquire<counter_below> written out: called through it, the NP = 32 hand-over step kernels compile to different code
__device__ __forceinline__ void counter_wait(const int* c, int want, int* timeouts, int* err_flag) {
    int v = 0, spins = 0;
    do {
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(c) : "memory");
        if (v - want < 0) __nanosleep(40);
    } while (v - want < 0 && ++spins < (1 << 24));    // ~1 s: a lost hand-over must not hang the GPU
    if (v - want < 0) report_handover_timeout(timeouts, err_flag);
}
__device__ __forceinline__ void counter_set(int* c, int v) { asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(c), "r"(v) : "memory"); }
__device__ __forceinline__ void counter_inc(int* c) { asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(c), "r"(1) : "memory"); }
__device__ __forceinline__ void bulk_drain_writes() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// physics warp -> shared hand-off arrays
__device__ __forceinline__ void hand_store(float* hand, int lane, const Agent& s, const float nvel[3]) {
    hand[32 * H_PX + lane] = s.pos[0]; hand[32 * H_PY + lane] = s.pos[1]; hand[32 * H_PZ + lane] = s.pos[2];
    hand[32 * H_VX + lane] = s.vel[0]; hand[32 * H_VY + lane] = s.vel[1]; hand[32 * H_VZ + lane] = s.vel[2];
    hand[32 * H_NVX + lane] = nvel[0]; hand[32 * H_NVY + lane] = nvel[1]; hand[32 * H_NVZ + lane] = nvel[2];
#pragma unroll
    for (int k = 0; k < 9; ++k) hand[32 * (H_R0 + k) + lane] = s.R[k];
    hand[32 * H_OX + lane] = s.om[0]; hand[32 * H_OY + lane] = s.om[1]; hand[32 * H_OZ + lane] = s.om[2];
    hand[32 * H_GX + lane] = s.goal[0]; hand[32 * H_GY + lane] = s.goal[1]; hand[32 * H_GZ + lane] = s.goal[2];
}

__device__ __forceinline__ void hand_load(const float* hand, int lane, Agent& s, float nvel[3]) {
    s.pos[0] = hand[32 * H_PX + lane]; s.pos[1] = hand[32 * H_PY + lane]; s.pos[2] = hand[32 * H_PZ + lane];
    s.vel[0] = hand[32 * H_VX + lane]; s.vel[1] = hand[32 * H_VY + lane]; s.vel[2] = hand[32 * H_VZ + lane];
    nvel[0] = hand[32 * H_NVX + lane]; nvel[1] = hand[32 * H_NVY + lane]; nvel[2] = hand[32 * H_NVZ + lane];
#pragma unroll
    for (int k = 0; k < 9; ++k) s.R[k] = hand[32 * (H_R0 + k) + lane];
    s.om[0] = hand[32 * H_OX + lane]; s.om[1] = hand[32 * H_OY + lane]; s.om[2] = hand[32 * H_OZ + lane];
    s.goal[0] = hand[32 * H_GX + lane]; s.goal[1] = hand[32 * H_GY + lane]; s.goal[2] = hand[32 * H_GZ + lane];
}

// The step kernel.  SPLIT = false: one warp does everything for its 32 drones.  SPLIT = true (blocks of 64 threads):
// warp 0 ("physics") integrates, detects and resolves contacts and keeps the books; warp 1 ("observer") draws the
// sensor noise while the physics warp integrates, then builds the observation rows from the hand-off arrays in shared
// memory — speculatively from the post-integration state, re-done only in the rare steps where a contact response or a
// reset changed it.  The two halves of a drone's ~2.7 k-instruction dependency chain overlap.
// SCN = true: the env's goals come from the device-side scenario family (qs_scenario.cuh); the other instantiations do
// not carry that code (instruction-cache footprint of the hot loop: +1.3 % step time on c3 when it was compiled in).
// HO = true: per-block hand-over between consecutive step grids instead of the grid-wide wait (handover_acquire above);
// chosen by the launcher when a step grid does not fit the GPU in one wave or the split shape is used.
// DYN = true: per-drone physical constants (qs_set_dynamics; SURVEY 8f-4) instead of the compile-time Crazyflie set — only
// instantiated for the single-warp shape with the grid-wide wait.
// NZ = true: the custom sensor-noise model (qs_set_sensor_noise, p.nz) instead of the compile-time 'default' set; the gyro
// bias (p.gyro_bias, when that model is on) rides in registers across the steps of a launch.  Same shape as DYN.
// qs_step_npy.cu compiles this kernel once more, as qs_step_kernel_npy, with the floor model of the reference's numpy path
// (QS_NUMPY_DYNAMICS, qs_set_numpy_dynamics).  qs_step_pc.cu / qs_step_pc_npy.cu compile it as qs_step_kernel_pc /
// qs_step_kernel_pc_npy with the control modes of qs_set_control (QS_CONTROL_MODES; same shape as DYN).
template <int NP, bool SPLIT, bool SCN, bool HO, bool DYN = false, bool NZ = false>
__global__ void __launch_bounds__(step_max_threads<NP, SPLIT, SCN, HO, DYN, NZ>()) qs_step_kernel(const __grid_constant__ StepParams p) {
    static_assert(!(DYN || NZ || QS_CONTROL_MODES) || (!SPLIT && !HO),
                  "per-drone constants, the custom sensor-noise model and the control modes run in the single-warp shape with "
                  "the grid-wide wait");
    extern __shared__ __align__(128) float2 s_obst[];
    __shared__ int s_late;          // courier launches: a block with a goal event behind the observation is released at its end
    __shared__ unsigned long long s_rows;      // courier launches: mbarrier, completes when the previous instance's observation rows are out
    const DevState& st = p.st;
    const int lane = threadIdx.x & 31;
    const int i = lane & (NP - 1);
    const int role = SPLIT ? (threadIdx.x >> 5) : 0;                 // 0 physics (or everything), 1 observer
    const int tid = SPLIT ? lane : threadIdx.x;
    // courier warp (p.courier, single-warp shape with the per-block hand-over): the last warp of the block carries no envs;
    // it takes the predecessor's state word, waits for the predecessor's observation rows, publishes this block's state as
    // soon as the workers have stored it (before they build the observation) and the block's completion at the end — the
    // fences and flag round trips of the hand-over then cost the worker warps nothing.
    const bool has_courier = HO && !SPLIT && p.courier != 0;
    const int work_threads = has_courier ? (int)blockDim.x - 32 : (int)blockDim.x;
    const int envs_per_block = (SPLIT ? 32 : work_threads) / NP;
    const int env_local = tid / NP;
    const int env = blockIdx.x * envs_per_block + env_local;
    if (has_courier && (int)threadIdx.x >= work_threads) {
        int* const tmo = st.ready + p.E;
        const int nthr = (int)blockDim.x;
        if (!p.chained) asm volatile("griddepcontrol.wait;" ::: "memory");      // after a foreign kernel: its writes formally visible
        int k = 0;
        if (lane == 0) {
            s_late = 0;
            mbar_init(&s_rows, 1);
            k = atomicAdd(hw_word(st, p.E, HW_T), 1);                 // this instance's ticket ...
        }
        named_arrive(5, nthr);                                        // ... is taken before any thread of the block lets the next grid launch
        asm volatile("griddepcontrol.launch_dependents;");
        if (lane == 0) counter_wait(hw_word(st, p.E, HW_S), k, tmo, st.err_flag);
        named_arrive(1, nthr);                                        // the workers start loading the state
        if (lane == 0) {
            // the predecessor's observation rows are out (in a wrapped chain the wrapper kernel has waited for that)
            if (!p.wrap_chain) counter_wait(hw_word(st, p.E, HW_D), k, tmo, st.err_flag);
            mbar_arrive(&s_rows);
        }
        named_sync(2, nthr);                                          // the workers have stored the block's state (and do not wait here)
        const int late = *reinterpret_cast<volatile int*>(&s_late);
        const int k1 = (int)((unsigned)k + 1u);                       // the counters wrap around after 2^32 steps; waits compare differences
        // plain chain: the next instance may start.  Wrapped chain: the wrapper kernel's block may start on the stored state
        // (it waits for Rw where it needs this step's observation rows, and before it hands the state on).
        if (!late && lane == 0) {
            if (p.wrap_chain) counter_inc(hw_word(st, p.E, HW_DW)); else counter_set(hw_word(st, p.E, HW_S), k1);
        }
        named_sync(3, nthr);                                          // the workers' last stores (bulk copies drained) are issued
        if (lane == 0) {
            if (p.wrap_chain) {
                if (late) counter_inc(hw_word(st, p.E, HW_DW));
                counter_inc(hw_word(st, p.E, HW_RW));
            } else if (late) counter_set(hw_word(st, p.E, HW_S), k1);
            counter_set(hw_word(st, p.E, HW_D), k1);
        }
        return;
    }
    const bool env_ok = env < p.E;
    const bool valid = env_ok && i < p.N;
    const long long a = (long long)env * p.N + i;
    const long long A = (long long)p.E * p.N;

    // The actions of the first step are never written by a step grid, and whatever wrote them completed before the
    // PREDECESSOR of this grid passed its own wait: they are loaded before the dependency wait (HBM latency hidden
    // behind the predecessor's tail).
    // Only for CHAINED launches (qs_set_chained: the stream predecessor is a step grid of this handle); otherwise the
    // predecessor may be the kernel that produced the actions and the load follows the wait.
    QS_TL(0);
    float4 av0 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.chained && valid && role == 0) av0 = __ldcs(p.actions + a);          // streaming: read once

    // Programmatic dependent launch: wait here for the PREVIOUS step's grid to complete (and flush) before touching any
    // state; the trigger that lets the NEXT step's grid start launching is issued just before this grid's final stores
    // (hides part of the launch latency of each step; triggering at kernel start is SLOWER because the early grid competes
    // for issue slots while it spins).  Without the launch attribute both are no-ops.
    if (HO) {
        // not chained: the stream predecessor may be a foreign kernel (it never triggers early, so this grid starts when
        // it has completed; the wait makes its writes formally visible).  Chained step grids (qs_set_chained) skip it.
        if (!p.chained) asm volatile("griddepcontrol.wait;" ::: "memory");
        if (has_courier) {
            named_sync(5, (int)blockDim.x);                          // the courier has taken the block's ticket
            asm volatile("griddepcontrol.launch_dependents;");
            named_sync(1, (int)blockDim.x);                          // the state of the previous instance has been handed on
        } else {
            if (threadIdx.x == 0) handover_acquire(st.ready + blockIdx.x, st.ready + p.E, st.err_flag);
            __syncthreads();
            asm volatile("griddepcontrol.launch_dependents;");
        }
    } else {
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }

    QS_TL(1);
    if (!p.chained && valid && role == 0) av0 = __ldcs(p.actions + a);

    // shared memory: [envs_per_block][M] pillar table, then one observation staging tile per warp
    float2* s_obst_env = s_obst + env_local * p.M;
    float* s_tile = reinterpret_cast<float*>(s_obst) + p.smem_tile_off + (SPLIT ? 0 : (threadIdx.x >> 5)) * (32 * p.obs_dp);
    float* s_hand = reinterpret_cast<float*>(s_obst) + p.smem_tile_off + 32 * p.obs_dp;      // SPLIT only
    float* s_hand2 = s_hand + 32 * H_COUNT;                                                  // final state after a response / reset
    uint32_t* s_hflag = reinterpret_cast<uint32_t*>(s_hand2 + 32 * H_COUNT);

    Agent s;
    EnvCtr ctr = {0, 0, 0, 0};
    if (valid && role == 0) load_agent<HO>(st, a, s);      // state loads are issued before the pillar staging barrier
    // running sums of the goal distance over the last 1 / 3 / 5 s of the episode: loaded with the state (an env in its last
    // 5 s — a third of all envs when they run out of phase — would otherwise pay a dependent L2 round trip mid-step)
    float4 dsum = make_float4(0.f, 0.f, 0.f, 0.f);
    bool dsum_dirty = false;
    if (valid && role == 0) dsum = ld_state<HO>(st.slots + SL_DIST_SUMS * st.a_pad + a);
    Phys ph;
    if (DYN) load_phys(st.dyn, valid ? a : 0, ph);
    const bool gyro_model = NZ && p.gyro_bias != nullptr;
    float3 gb = make_float3(0.f, 0.f, 0.f);
    if (gyro_model && valid) {
        const float4 b = QS_LD(p.gyro_bias + a);
        gb = make_float3(b.x, b.y, b.z);
    }
    float qt[4] = {1.f, 0.f, 0.f, 0.f};      // rotation-noise quaternion of the observation (NZ)
    // env-level words: issued together with the state loads, BEFORE the pillar staging below waits for its own loads (one
    // L2 round trip for everything instead of two serialized ones)
    int4 ctr_raw = make_int4(0, 0, 0, 0);
    if (env_ok) ctr_raw = ld_state<HO>(st.env_ctr + env);
    // An env whose episode ends in this step (known from the tick just loaded) will need its next-episode record and its
    // running statistics at the END of the step: their lines are pulled into L2 now (they were written long ago and have
    // usually been evicted by the observation stream), behind the whole step's arithmetic.
    if (env_ok && role == 0 && ctr_raw.x + p.T > p.ep_len && valid) {
        prefetch_l2(st.epi + env);
        prefetch_l2(st.next_goal + a);
        prefetch_l2(st.next_spawn + a);
        prefetch_l2(st.slots + SL_STALE_VEL * st.a_pad + a);
        if (i == 0) {
            prefetch_l2(st.env_cnt + (long long)env * QS_NUM_ENV_STATS);
            prefetch_l2(st.next_scn_i + env);
            prefetch_l2(st.next_scn_f + 3 * (long long)env);
            if (p.use_obst) prefetch_l2(st.next_obst + (long long)env * p.M);
        }
    }
    // device-side scenarios: the tick of the env's next goal event (qs_scenario.cuh); never for the other scenarios
    constexpr bool dev_scn = SCN;
    int scn_next = SCN_NEVER;
    if (dev_scn && env_ok && role == 0) scn_next = QS_LD(st.scn_i + env).z;
    // approch_goal_metric is a property of the episode's scenario where the obstacle scenarios are drawn on the device
    const bool env_metric = p.use_obst && p.scenario > QS_SCENARIO_O_RANDOM;
    float approach = p.approach_metric;
    if (env_metric && env_ok && role == 0) approach = QS_LD(st.scn_f + 3 * (long long)env + 1).w;
    float obst_r = p.obst_radius;                 // per-episode pillar radius where the size is randomised
    if (p.obst_random && env_ok) obst_r = QS_LD(st.scn_f + 3 * (long long)env).x;
    // stage the pillar tables in shared memory.  Single-warp shape: every warp stages the tables of ITS envs (a contiguous
    // [32 / NP][M] float2 span) and only a warp-level barrier follows; split shape: the block's two warps share them.
    if (p.use_obst) {
        if (SPLIT) {
            const long long base = (long long)blockIdx.x * envs_per_block * p.M;
            const long long total = (long long)p.E * p.M;
            for (int k = threadIdx.x; k < envs_per_block * p.M; k += blockDim.x)
                if (base + k < total) s_obst[k] = ld_state<HO>(st.obst + base + k);
            __syncthreads();
        } else {
            const int wenv = (threadIdx.x >> 5) * (32 / NP);                      // first env (block-local) of this warp
            const long long base = ((long long)blockIdx.x * envs_per_block + wenv) * p.M;
            const long long total = (long long)p.E * p.M;
            float2* dst = s_obst + wenv * p.M;
            for (int k = lane; k < (32 / NP) * p.M; k += 32)
                if (base + k < total) dst[k] = ld_state<HO>(st.obst + base + k);
            __syncwarp();
        }
    }
    if (!valid) idle_agent(s, i);
    ctr.tick = ctr_raw.x; ctr.step_count = ctr_raw.y; ctr.svd_count = ctr_raw.z; ctr.episode_idx = ctr_raw.w;
#ifdef QS_TIMELINE
    if (ctr.tick + __float_as_int(s.pos[0]) == 0x7fffffff) QS_TL(7);      // depends on the loaded state: stamp 2 follows the loads
    QS_TL(2);
#endif
    if (SPLIT && role == 1) {
        // ============================ observer warp ============================
        const int gbase = lane & ~(NP - 1);
        const int slot = (lane / NP) * p.N + i;                       // row of this drone inside the warp's tile
        const int env_first = blockIdx.x * envs_per_block;
        const int envs_here = min(envs_per_block, p.E - env_first);
#pragma unroll 1
        for (int t = 0; t < p.T; ++t) {
            const RngKey key = step_key(p, env, ctr.step_count);
            const bool want = !p.last_obs_only || t == p.T - 1;
            // first sensor-noise draw (SITE_HOT, 2 Philox blocks), overlapped with the physics warp's integration
            Noise9 nz = default_noise(hot_normals(key, i), p.sense_noise);
            Agent o;
            float nvel[3];
            bar_sync(1);                                              // post-integration state is in the hand-off arrays
            if (want) {
                hand_load(s_hand, lane, o, nvel);
                const float dmin2 = p.use_obst ? min_pillar_dist2(p, o, s_obst_env) : 1e4f;
                write_observation<NP, true>(p, o, nvel, nz, i, valid, s_obst_env, dmin2, s_tile + slot * p.obs_dp, p.obst_radius, s_hand, gbase);
            }
            bar_sync(2);                                              // final state + flags
            const uint32_t hf = s_hflag[gbase];
            if (p.use_obst && __any_sync(0xffffffffu, (hf & HF_RESET) != 0u)) {
                // a reset replaced this env's pillars: the physics warp wrote them to global memory only, the observer
                // refreshes the shared-memory table (the physics warp reads it again only after barrier 3)
                if (hf & HF_RESET) {
                    for (int m = i; m < p.M; m += NP) s_obst_env[m] = QS_LD(st.obst + (long long)env * p.M + m);
                }
                __syncwarp();
            }
            if (want && hf != 0u) {                                   // contact response or reset: rebuild the rows of this env
                hand_load(s_hand2, lane, o, nvel);
                if (p.sense_noise) nz = sensor_noise(key, (hf & HF_RESET) ? SITE_SENSOR_RESET : SITE_SENSOR1, i);
                const float dmin2 = p.use_obst ? min_pillar_dist2(p, o, s_obst_env) : 1e4f;
                write_observation<NP, true>(p, o, nvel, nz, i, valid, s_obst_env, dmin2, s_tile + slot * p.obs_dp, p.obst_radius, s_hand2, gbase);
            }
            if (want) {
                float* gbase_ptr = p.obs + (p.last_obs_only ? 0 : (long long)t * A) * p.D;
                if (envs_here > 0)
                    emit_observation_tile(p, s_tile, gbase_ptr + (long long)env_first * p.N * p.D, env_first * p.N,
                                          p.last_obs_only ? 0 : t, envs_here * p.N, lane);
                if (p.obs_bulk) bulk_drain();                         // the tile is rewritten in the next step
            }
            ctr.step_count += 1;
            bar_sync(3);                                              // hand-off arrays and tile are free again
        }
        if (!HO) asm volatile("griddepcontrol.launch_dependents;");
        if (HO) bar_sync(4);                                          // the physics warp publishes the block's state
        return;
    }

    bool goal_dirty = false;
    bool late_goal = false;                            // goal event after the last observation (the single-warp shape stores the
                                                       // state before it, at t = T - 1)

#pragma unroll 1
    for (int t = 0; t < p.T; ++t) {
        const RngKey key = step_key(p, env, ctr.step_count);

        // the draws every drone needs every step: OU thrust noise + first sensor-noise draw (SITE_HOT: 2 Philox blocks)
        Noise9 nz;
        float4 ou_z;
        if (SPLIT) {
            const uint4 b0 = rng_block(key, SITE_HOT, i, 0, 0);
            normal_pair16(b0.x, ou_z.x, ou_z.y);
            normal_pair16(b0.y, ou_z.z, ou_z.w);
#pragma unroll
            for (int k = 0; k < 3; ++k) { nz.p[k] = 0.f; nz.v[k] = 0.f; nz.w[k] = 0.f; }
        } else {
            const HotNormals hn = hot_normals(key, i);
            ou_z = make_float4(hn.ou[0], hn.ou[1], hn.ou[2], hn.ou[3]);
            nz = default_noise(hn, p.sense_noise);
            if (NZ) {
                const SensedNoise sn = sensor_noise_model(p.nz, key, 0, i, gb, gyro_model);
                nz = sn.n; gb = sn.bias;
#pragma unroll
                for (int k = 0; k < 4; ++k) qt[k] = sn.q[k];
            }
        }

        // ================= per-drone part: QuadrotorSingle._step, quadrotor_single.py:341-357 =================
        float act[4] = {0.f, 0.f, 0.f, 0.f};
        if (valid) {
            const float4 av = (t == 0) ? av0 : __ldcs(p.actions + ((long long)t * A + a));
            act[0] = av.x; act[1] = av.y; act[2] = av.z; act[3] = av.w;
        }
        av0 = make_float4(0.f, 0.f, 0.f, 0.f);         // used by the first step only: not live across the rest of the loop
        float cmd[4];
#if QS_CONTROL_MODES
        if (p.control == QS_CONTROL_POSITION) {                     // warp-uniform (one mode per handle)
            position_control<DYN>(s, ph, cmd);
        } else {
#pragma unroll
            for (int m = 0; m < 4; ++m) cmd[m] = clampf(act[m], 0.f, 1.f);    // RawControl(zero_action_middle=False), :37-57
        }
#else
#pragma unroll
        for (int m = 0; m < 4; ++m) cmd[m] = 0.5f * (clampf(act[m], -1.f, 1.f) + 1.f);    // RawControl.step, quadrotor_control.py:53-57
#endif
        // OU thrust noise, once per control step (numba_utils.py:101-105, quadrotor_dynamics.py:209)
        const float ou_sigma = DYN ? ph.ou_sigma : OU_SIGMA;
        s.ou[0] += OU_THETA * (0.f - s.ou[0]) + ou_sigma * ou_z.x;
        s.ou[1] += OU_THETA * (0.f - s.ou[1]) + ou_sigma * ou_z.y;
        s.ou[2] += OU_THETA * (0.f - s.ou[2]) + ou_sigma * ou_z.z;
        s.ou[3] += OU_THETA * (0.f - s.ou[3]) + ou_sigma * ou_z.w;
#pragma unroll 1
        for (int sub = 0; sub < SIM_STEPS; ++sub) {
            ctr.svd_count += 1;
            const bool do_svd = ctr.svd_count >= SVD_PERIOD;
            if (do_svd) ctr.svd_count = 0;
            if (DYN) dynamics_substep_dyn(s, cmd, do_svd, p, key, i, sub, ph);
            else dynamics_substep<courier_capable<NP, SPLIT, SCN, HO, DYN, NZ>()>(s, cmd, do_svd, p, key, i, sub);
        }
        if (SPLIT) {                                                   // positions are final from here on
            hand_store(s_hand, lane, s, s.vel);
            bar_sync(1);
        }
#ifdef QS_TIMELINE
        if (__float_as_int(s.pos[0]) == 0x7fffffff) QS_TL(7);
        QS_TL(3);
#endif
        // compute_reward_weighted, quadrotor_single.py:34-92 (dt = SIM dt, raw unclipped action)
        const bool on_floor = (s.flags & QS_FLAG_ON_FLOOR) != 0u;
        const float dist = norm3(s.goal[0] - s.pos[0], s.goal[1] - s.pos[1], s.goal[2] - s.pos[2]);
        const float raw_effort = fsqrt(act[0] * act[0] + act[1] * act[1] + act[2] * act[2] + act[3] * act[3]);
        const float raw_orient = on_floor ? 1.0f : -s.R[8];
        const float raw_spin = norm3(s.om[0], s.om[1], s.om[2]);
        const float raw_crash = on_floor ? 1.0f : 0.0f;
        float reward = -SIM_DT * (p.rew[QS_REW_POS] * dist + p.rew[QS_REW_EFFORT] * raw_effort + p.rew[QS_REW_CRASH] * raw_crash +
                                  p.rew[QS_REW_ORIENT] * raw_orient + p.rew[QS_REW_SPIN] * raw_spin);
        const long long ta = (long long)t * A + a;
        if (valid && p.rew_terms) {              // the per-drone terms leave now: they are not kept live across the env part
            float* tr = p.rew_terms + ta * QS_NUM_TERMS;
            tr[QS_TERM_RAW_POS] = SIM_DT * -dist;
            tr[QS_TERM_RAW_ACTION] = SIM_DT * -raw_effort;
            tr[QS_TERM_RAW_CRASH] = SIM_DT * -raw_crash;
            tr[QS_TERM_RAW_ORIENT] = SIM_DT * -raw_orient;
            tr[QS_TERM_RAW_SPIN] = SIM_DT * -raw_spin;
        }
        const int tick_before = ctr.tick;
        const int time_remain = p.ep_len - tick_before;
        ctr.tick = tick_before + 1;
        const bool done = ctr.tick > p.ep_len;

        // ================= env part: all-pairs pass (positions only) =================
        // calculate_collision_matrix (collisions/quadrotors.py:63-91), proximity penalties (:95-103), downwash
        // detection (aerodynamics/downwash.py:4-51) — drone i scans every other drone j of its env.  Thresholds are
        // compared on squared distances (same predicate, no square root on the common path).
        uint32_t cur_col = 0u;
        float prox = 0.f;
        bool dw_applied = false;
        float dw_dv[3] = {0.f, 0.f, 0.f}, dw_dw[3] = {0.f, 0.f, 0.f};
        if (NP > 1) {
            const float max_pen = p.rew[QS_REW_QUADCOL_BIN_SMOOTH_MAX];
            const float pen_ratio = -max_pen / p.falloff_thr;
#pragma unroll 2
            for (int j = 0; j < p.N; ++j) {
                const float dx = s.pos[0] - shfl<NP>(s.pos[0], j), dy = s.pos[1] - shfl<NP>(s.pos[1], j),
                            dz = s.pos[2] - shfl<NP>(s.pos[2], j);
                const float d2 = dx * dx + dy * dy + dz * dz;
                const bool other = (j != i) && valid;
                if (other && d2 <= p.falloff_thr2) {
                    const float d = fsqrt(d2);
                    if (d2 <= p.col_thr2) cur_col |= 1u << j;
                    prox += pen_ratio * d + max_pen;
                }
                // the downwash cylinder (|rel_z| < 0.7, rel_xy < 0.1) lies inside the ball d^2 < 0.5: the z-axis
                // exchange and the cylinder test run only when some drone of the warp is that close to drone j
                if (p.use_downwash && __any_sync(0xffffffffu, other && d2 < 0.5f)) {
                    const float zx = shfl<NP>(s.R[2], j), zy = shfl<NP>(s.R[5], j), zz = shfl<NP>(s.R[8], j);
                    // is drone i (me) inside the downwash cylinder below drone j?  -0.7 < rel_z < 0 and rel_xy < 0.1
                    const float rel_z = dx * zx + dy * zy + dz * zz;
                    const float rxy2 = d2 - rel_z * rel_z;                 // negative -> sqrt is NaN in numpy -> false
                    if (other && -0.7f < rel_z && rel_z < 0.f && rxy2 >= 0.f && rxy2 < 0.1f * 0.1f) {
                        const KickVO k = downwash_kick(key, j, i, fsqrt(d2), zx, zy, zz);
                        dw_dv[0] += k.vel.x; dw_dv[1] += k.vel.y; dw_dv[2] += k.vel.z;
                        dw_dw[0] += k.dom.x; dw_dw[1] += k.dom.y; dw_dw[2] += k.dom.z;
                        dw_applied = true;
                    }
                }
            }
        }
        // obstacles: first pillar in index order within arm + radius (obstacles/utils.py:31-43)
        int hit = -1;
        float dmin2 = 1e4f;                          // smallest squared centre distance to a pillar (prunes the SDF pass)
        if (p.use_obst) {
            const float obst_thr = p.obst_random ? p.quad_arm + obst_r : p.obst_col_thr;
            const float obst_thr2 = obst_thr * obst_thr;
#pragma unroll 4
            for (int m = p.M - 1; m >= 0; --m) {
                const float2 ob = s_obst_env[m];
                const float dx = s.pos[0] - ob.x, dy = s.pos[1] - ob.y;
                const float d2 = dx * dx + dy * dy;
                hit = (d2 <= obst_thr2) ? m : hit;      // obst_thr2 = (quad_arm + radius)^2, obstacles/utils.py:33
                dmin2 = fminf(dmin2, d2);
            }
        }

        // ---- discrete events of this step.  Almost every step is "quiet" for all 32 drones of a warp (no contact now or
        //      on the previous tick, no crash flag, no downwash): then the whole bookkeeping below collapses to defaults.
        float raw_quadcol = 0.f, raw_obst = 0.f;
        uint32_t new_pairs = 0u;
        bool new_obst = false, wall_c = false, ceil_c = false, kicked = false;
        const uint32_t busy_flags = QS_FLAG_CRASHED_FLOOR | QS_FLAG_CRASHED_WALL | QS_FLAG_CRASHED_CEILING | QS_FLAG_PREV_WALL |
                                    QS_FLAG_PREV_CEILING | QS_FLAG_PREV_ROOM | QS_FLAG_PREV_OBST;
        const bool quiet = cur_col == 0u && s.prev_col == 0u && hit < 0 && (s.flags & busy_flags) == 0u && !dw_applied;
        const bool settled = (float)ctr.tick >= p.grace_steps;
        s.flags &= ~(QS_FLAG_KICKED | QS_FLAG_NEW_QUADCOL | QS_FLAG_NEW_OBSTCOL);
        if (!__all_sync(0xffffffffu, quiet)) {
            // collision bookkeeping, quadrotor_multi.py:433-459 (quirks D-2..D-4 reproduced)
            const bool in_u = (cur_col != 0u) && (s.prev_col == 0u);                     // flattened-id set difference
            const uint32_t u_mask = group_ballot<NP>(in_u && valid);
            const int col_curr_tick = __popc(u_mask) / 2;
            const bool u_any = (u_mask & ~1u) != 0u;                                      // ids.any(): id 0 alone is falsy
            raw_quadcol = (u_any && in_u) ? -1.0f : 0.0f;
            new_pairs = cur_col & ~s.prev_col;                                            // pair-level novelty (:437-438)
            if (col_curr_tick > 0 && settled && in_u) s.flags &= ~QS_FLAG_NO_COL_AGENT;
            s.prev_col = cur_col;

            // pillar contacts, :462-488
            new_obst = (hit >= 0) && !(s.flags & QS_FLAG_PREV_OBST) && valid;
            const uint32_t obst_mask = p.use_obst ? group_ballot<NP>(new_obst) : 0u;
            raw_obst = new_obst ? -1.0f : 0.0f;
            s.flags = (hit >= 0) ? (s.flags | QS_FLAG_PREV_OBST) : (s.flags & ~QS_FLAG_PREV_OBST);
            bool far35 = false, far5 = false;
            if (new_obst && settled) {
                s.flags &= ~QS_FLAG_NO_COL_OBST;
                // distance to goal of the FIRST-draw noisy position (quadrotor_multi.py:474)
                if (SPLIT && p.sense_noise) {
                    const uint4 b0 = rng_block(key, SITE_HOT, i, 0, 0);
                    float n0, n1, n2, n3;
                    normal_pair16(b0.z, n0, n1);
                    normal_pair16(b0.w, n2, n3);
                    nz.p[0] = POS_NOISE_STD * n0; nz.p[1] = POS_NOISE_STD * n1; nz.p[2] = POS_NOISE_STD * n2;
                }
                const float q = norm3((s.pos[0] + nz.p[0]) - s.goal[0], (s.pos[1] + nz.p[1]) - s.goal[1], (s.pos[2] + nz.p[2]) - s.goal[2]);
                far35 = q > 3.5f; far5 = q > 5.0f;
            }

            // room, quadrotor_multi.py:289-302,491-497 (quirk D-5: novelty against the previously RETURNED lists)
            const bool floor_c = (s.flags & QS_FLAG_CRASHED_FLOOR) != 0u && valid;
            wall_c = (s.flags & QS_FLAG_CRASHED_WALL) && !(s.flags & QS_FLAG_PREV_WALL) && valid;
            ceil_c = (s.flags & QS_FLAG_CRASHED_CEILING) && !(s.flags & QS_FLAG_PREV_CEILING) && valid;
            const bool room_c = (floor_c || wall_c || ceil_c) && !(s.flags & QS_FLAG_PREV_ROOM);
            s.flags &= ~(QS_FLAG_PREV_WALL | QS_FLAG_PREV_CEILING | QS_FLAG_PREV_ROOM);
            if (wall_c) s.flags |= QS_FLAG_PREV_WALL;
            if (ceil_c) s.flags |= QS_FLAG_PREV_CEILING;
            if (room_c) s.flags |= QS_FLAG_PREV_ROOM;
            if (u_any && in_u) s.flags |= QS_FLAG_NEW_QUADCOL;
            if (new_obst) s.flags |= QS_FLAG_NEW_OBSTCOL;

            // ballots of this step's discrete events.  NB: none of them may sit behind a short-circuit `||` / `&&` whose
            // left side differs between the envs of a warp.
            const uint32_t floor_m = group_ballot<NP>(floor_c), wall_m = group_ballot<NP>(wall_c),
                           ceil_m = group_ballot<NP>(ceil_c), room_m = group_ballot<NP>(room_c);
            const uint32_t dw_m = p.use_downwash ? group_ballot<NP>(dw_applied) : 0u;
            const uint32_t new_pair_m = group_ballot<NP>(new_pairs != 0u && valid);
            const uint32_t f35 = group_ballot<NP>(far35), f5 = group_ballot<NP>(far5);
            kicked = (dw_m | new_pair_m | obst_mask | wall_m | ceil_m) != 0u;             // self_state_update_flag, :549-587

            // episode counters (lane 0 of the env), quadrotor_multi.py:448-456,468-478,522-526
            const int n_obst = __popc(obst_mask);
            const bool any_event = col_curr_tick > 0 || n_obst > 0 || ((floor_m | wall_m | ceil_m | room_m) != 0u && settled);
            if (any_event && i == 0 && env_ok) {
                int32_t* c = st.env_cnt + (long long)env * QS_NUM_ENV_STATS;
                cnt_add(c, QS_STAT_NUM_COLLISIONS, col_curr_tick);
                if (col_curr_tick > 0 && settled) cnt_add(c, QS_STAT_NUM_COLLISIONS_AFTER_SETTLE, col_curr_tick);
                if (col_curr_tick > 0 && (float)time_remain <= p.final_steps) cnt_add(c, QS_STAT_NUM_COLLISIONS_FINAL_5S, col_curr_tick);
                cnt_add(c, QS_STAT_NUM_COLLISIONS_OBST, n_obst);
                if (settled) {
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_OBST_AFTER_SETTLE, n_obst);
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_OBST_3_5, __popc(f35));
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_OBST_5, __popc(f5));
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_ROOM, __popc(room_m));
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_FLOOR, __popc(floor_m));
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_WALL, __popc(wall_m));
                    cnt_add(c, QS_STAT_NUM_COLLISIONS_CEILING, __popc(ceil_m));
                }
            }
        }

#ifdef QS_TIMELINE
        if (__float_as_int(prox) == 0x7fffffff) QS_TL(7);
        QS_TL(4);
#endif
        // rewards, quadrotor_multi.py:499-540
        const float rew_prox = -1.0f * (CONTROL_DT * prox);
        reward += p.rew[QS_REW_QUADCOL_BIN] * raw_quadcol;
        reward += rew_prox;
        if (p.use_obst) reward += p.rew[QS_REW_QUADCOL_BIN_OBST] * raw_obst;

        // goal-distance log and reached_goal, quadrotor_multi.py:542-546
        {
            const float m5 = (dist + s.ring[0] + s.ring[1] + s.ring[2] + s.ring[3]) * 0.2f;
            if (ctr.tick >= 5 && m5 < approach) s.flags |= QS_FLAG_REACHED_GOAL;
            s.ring[3] = s.ring[2]; s.ring[2] = s.ring[1]; s.ring[1] = s.ring[0]; s.ring[0] = dist;
            const int len = p.ep_len + 1;
            const int w5 = min(len, 500);
            if (valid && ctr.tick > len - w5) {
                if (ctr.tick > len - min(len, 100)) dsum.x += dist;
                if (ctr.tick > len - min(len, 300)) dsum.y += dist;
                dsum.z += dist;
                dsum_dirty = true;
            }
        }

        // ================= contact responses, quadrotor_multi.py:548-587 (rare: one warp-uniform branch) =================
        if (__any_sync(0xffffffffu, kicked)) {
            if (dw_applied) {
#pragma unroll
                for (int k = 0; k < 3; ++k) { s.vel[k] += dw_dv[k]; s.om[k] += dw_dw[k]; }
            }
            if (NP > 1) {
                // new colliding pairs, lexicographic order, one at a time (the second response of a drone sees the first)
                uint32_t pending = new_pairs & ~((2u << i) - 1u);      // partners j > i: lane i owns pair (i, j)
                if (!valid) pending = 0u;
                while (__any_sync(0xffffffffu, pending != 0u)) {
                    // every lane of the warp runs the same shuffles; groups without a pending pair just idle
                    const uint32_t owners = group_ballot<NP>(pending != 0u);
                    const bool act_pair = owners != 0u;
                    const int pa = act_pair ? __ffs(owners) - 1 : 0;
                    const uint32_t pend_a = shfl_u<NP>(pending, pa);
                    const int pb = act_pair ? __ffs(pend_a) - 1 : 0;
                    V3 p1, v1, p2, v2;
                    p1.x = shfl<NP>(s.pos[0], pa); p1.y = shfl<NP>(s.pos[1], pa); p1.z = shfl<NP>(s.pos[2], pa);
                    v1.x = shfl<NP>(s.vel[0], pa); v1.y = shfl<NP>(s.vel[1], pa); v1.z = shfl<NP>(s.vel[2], pa);
                    p2.x = shfl<NP>(s.pos[0], pb); p2.y = shfl<NP>(s.pos[1], pb); p2.z = shfl<NP>(s.pos[2], pb);
                    v2.x = shfl<NP>(s.vel[0], pb); v2.y = shfl<NP>(s.vel[1], pb); v2.z = shfl<NP>(s.vel[2], pb);
                    if (act_pair && (i == pa || i == pb)) {
                        const PairOut o = pair_response(key, pa, pb, p1, v1, p2, v2);
                        if (i == pa) {
                            s.vel[0] = o.v1.x; s.vel[1] = o.v1.y; s.vel[2] = o.v1.z;
                            s.om[0] += o.dom.x; s.om[1] += o.dom.y; s.om[2] += o.dom.z;
                            pending &= ~(1u << pb);
                        } else {
                            s.vel[0] = o.v2.x; s.vel[1] = o.v2.y; s.vel[2] = o.v2.z;
                            s.om[0] -= o.dom.x; s.om[1] -= o.dom.y; s.om[2] -= o.dom.z;
                        }
                    }
                }
            }
            if (new_obst) {
                const float2 ob = s_obst_env[hit];
                V3 pos = {s.pos[0], s.pos[1], s.pos[2]}, vel = {s.vel[0], s.vel[1], s.vel[2]};
                const KickVO o = obstacle_response(key, i, pos, vel, ob.x, ob.y, 0.5f * (p.room_hi[2] - p.room_lo[2]) + p.room_lo[2],
                                                   obst_r);
                apply_kick(s, o);
            }
            if (wall_c) {
                V3 vel = {s.vel[0], s.vel[1], s.vel[2]};
                const int tx = s.pos[0] == p.room_lo[0] ? -1 : (s.pos[0] == p.room_hi[0] ? 1 : 0);
                const int ty = s.pos[1] == p.room_lo[1] ? -1 : (s.pos[1] == p.room_hi[1] ? 1 : 0);
                apply_kick(s, wall_response(key, i, vel, tx, ty));
            }
            if (ceil_c) {
                V3 vel = {s.vel[0], s.vel[1], s.vel[2]};
                apply_kick(s, ceiling_response(key, i, vel));
            }
            if (kicked) {
                s.flags |= QS_FLAG_KICKED;
                if (NZ) {
                    const SensedNoise sn = sensor_noise_model(p.nz, key, 1, i, gb, gyro_model);
                    nz = sn.n; gb = sn.bias;
#pragma unroll
                    for (int k = 0; k < 4; ++k) qt[k] = sn.q[k];
                } else if (!SPLIT && p.sense_noise) nz = sensor_noise(key, SITE_SENSOR1, i);      // fresh noise for every drone of the env (:598-599)
            }
        }

        // ================= scenario tick, quadrotor_multi.py:590 (reads the post-increment tick) =================
        // The observation of this step shows the NEW goal only if a contact response forces its re-computation
        // (quadrotor_multi.py:598-599); otherwise it was computed before the tick.  Single-warp kernel: event envs without
        // a response are ticked after the observation instead (site B below).  An env that ends its episode now is reset.
        const bool scn_ev = dev_scn && env_ok && ctr.tick == scn_next && !done;
        if (dev_scn && __any_sync(0xffffffffu, scn_ev && (SPLIT || kicked))) {
            const V3 g = {s.goal[0], s.goal[1], s.goal[2]};
            const bool act = scn_ev && (SPLIT || kicked);
            const ScnOut o = p.use_obst ? obstacle_scenario_tick<NP>(key, p.N, i, ctr.tick, g, act, st, env, p.grid_l, p.grid_w, p.M)
                                         : scenario_tick<NP>(key, p.N, i, ctr.tick, g, act, st, env);
            if (act) {
                s.goal[0] = o.goal.x; s.goal[1] = o.goal.y; s.goal[2] = o.goal.z;
                scn_next = o.next;
                goal_dirty = true;
            }
        }

        // ================= outputs of this step =================
        if (valid) {
            __stcs(p.rewards + ta, reward);
            __stcs(p.dones + ta, (uint8_t)(done ? 1 : 0));
            if (p.rew_terms) {
                float* tr = p.rew_terms + ta * QS_NUM_TERMS;
                tr[QS_TERM_RAW_QUADCOL] = raw_quadcol;
                tr[QS_TERM_PROXIMITY] = rew_prox;
                tr[QS_TERM_RAW_QUADCOL_OBST] = raw_obst;
            }
        }

        // ================= episode end: latch statistics, auto-reset (quadrotor_multi.py:626-722) =================
        float nvel[3] = {s.vel[0], s.vel[1], s.vel[2]};
        const bool do_reset = done && env_ok;
        if (__any_sync(0xffffffffu, do_reset)) {          // warp-uniform branch
            QS_TL(9);
            if (do_reset && valid) {
                const float4 sums = dsum;
                dsum = make_float4(0.f, 0.f, 0.f, 0.f);           // reset_env zeroes the slot
                dsum_dirty = false;
                const int len = p.ep_len + 1;
                const uint32_t fbits = ((s.flags & QS_FLAG_NO_COL_AGENT) ? 1u : 0u) | ((s.flags & QS_FLAG_NO_COL_OBST) ? 2u : 0u) |
                                       ((s.flags & QS_FLAG_REACHED_GOAL) ? 4u : 0u);
                st.stats_agent[a] = make_float4(sums.x / (float)min(len, 100), sums.y / (float)min(len, 300),
                                                sums.z / (float)min(len, 500), __uint_as_float(fbits));
            }
            if (do_reset && i == 0) {
                int32_t* c = st.env_cnt + (long long)env * QS_NUM_ENV_STATS;
                int32_t* o = st.stats_env + (long long)env * QS_NUM_ENV_STATS;
                // all loads first, then the stores: a load behind a store to the same line waits for the store's round trip
                int32_t v[QS_NUM_ENV_STATS];
#pragma unroll
                for (int k = 0; k < QS_NUM_ENV_STATS; ++k) v[k] = QS_LD(c + k);
#pragma unroll
                for (int k = 0; k < QS_NUM_ENV_STATS; ++k) { o[k] = v[k]; c[k] = 0; }
                o[QS_STAT_EPISODES_DONE] = ctr.episode_idx + 1;
                o[QS_STAT_SCENARIO] = (dev_scn || env_metric) ? QS_LD(st.scn_i + env).x : p.scenario;
            }
            reset_env<NP, SCN>(p, key, s, a, env, i, do_reset, valid, ctr.tick, SPLIT ? nullptr : s_obst_env, nvel, scn_next, approach, obst_r,
                               p.init_random != 0);
            if (DYN) {
                // resample_dynamics inside _reset (quadrotor_single.py:387-390): constants uploaded with at_next_reset are
                // latched now; update_dynamics builds a fresh QuadrotorDynamics, so OU state and SVD counter restart.  A
                // handle with the device-side sampler never has a row pending: qs_dyn_pregen_kernel latches its rows.
                const int pend = do_reset ? QS_LD(st.dyn_pending + env) : 0;
                if (pend != 0) {
                    if (valid) {
                        for (int q = 0; q < QS_DYN_ROW / 4; ++q)
                            st.dyn[a * (QS_DYN_ROW / 4) + q] = QS_LD(st.next_dyn + a * (QS_DYN_ROW / 4) + q);
                        load_phys(st.next_dyn, a, ph);
#pragma unroll
                        for (int k = 0; k < 4; ++k) s.ou[k] = 0.f;
                    }
                    ctr.svd_count = 0;
                }
                __syncwarp();
                if (pend != 0 && i == 0) st.dyn_pending[env] = 0;
            }
#ifdef QS_TIMELINE
            if (__float_as_int(s.pos[0]) == 0x7fffffff) QS_TL(7);
            QS_TL(10);
#endif
            if (do_reset) {
                ctr.tick = 0;
                ctr.episode_idx += 1;
                goal_dirty = true;
                if (NZ) {
                    const SensedNoise sn = sensor_noise_model(p.nz, key, 2, i, gb, gyro_model);
                    nz = sn.n; gb = sn.bias;
#pragma unroll
                    for (int k = 0; k < 4; ++k) qt[k] = sn.q[k];
                }
                if (!SPLIT) {
                    if (!NZ && p.sense_noise) nz = sensor_noise(key, SITE_SENSOR_RESET, i);
                    dmin2 = min_pillar_dist2(p, s, s_obst_env);          // new pose, new pillar table
                }
            }
#ifdef QS_TIMELINE
            if (__float_as_int(nz.p[0] + dmin2) == 0x7fffffff) QS_TL(7);
            QS_TL(11);
#endif
        }
        if (SPLIT) {
            // hand-off 2: final velocities / rates (and the whole state after a reset) + per-env flags
            const uint32_t hf = (kicked ? HF_KICKED : 0u) | (do_reset ? HF_RESET : 0u);
            if (hf != 0u) hand_store(s_hand2, lane, s, nvel);
            s_hflag[lane] = hf;
            bar_sync(2);
        }

        // The env state is final here (only a goal event at site B below touches it again): its stores are issued before
        // the observation is built, so that the fence of the per-block hand-over at the end of the kernel finds them
        // acknowledged instead of waiting a memory round trip for them.
        if (!SPLIT && t == p.T - 1) {
            if (valid) store_agent(st, a, s, goal_dirty);
            if (valid && dsum_dirty) st.slots[SL_DIST_SUMS * st.a_pad + a] = dsum;
            if (env_ok && i == 0) st.env_ctr[env] = make_int4(ctr.tick, ctr.step_count + 1, ctr.svd_count, ctr.episode_idx);
            if (gyro_model && valid) p.gyro_bias[a] = make_float4(gb.x, gb.y, gb.z, 0.f);
            if (has_courier) {
                // Early hand-over: the successor block only needs this block's env STATE, which is complete now; the
                // observation rows still to be written belong to this step's output arrays (the courier has made sure that
                // the predecessor's rows are complete).  A goal event that must run after the observation (site B) keeps
                // the state open: such a block (rare) is released at the end.
                if (dev_scn && scn_ev && !kicked) *reinterpret_cast<volatile int*>(&s_late) = 1;
                named_arrive(2, block_threads());
                // the rows of the previous instance are out (checked by the courier long ago: this does not spin in practice)
                mbar_wait(&s_rows, 0);
            }
        }

        // ================= observation (of the post-response, or freshly reset, state) =================
        if (SPLIT) {
            bar_sync(3);                                               // observer is done with this step's hand-off
        } else if (!p.last_obs_only || t == p.T - 1) {
            float* gbase = p.obs + (p.last_obs_only ? 0 : (long long)t * A) * p.D;
            // rotation noise (NZ): the observation is built with the perturbed rotation in s.R, which is restored after it
            float R_true[9];
            if (NZ && p.nz.rot) {
#pragma unroll
                for (int k = 0; k < 9; ++k) R_true[k] = s.R[k];
                observed_rotation(R_true, qt, s.R);
            }
            if (p.obs_stage) {
                // rows go to the warp's shared-memory tile, then out through the bulk-copy engine (or coalesced vector stores)
                const int slot = (lane / NP) * p.N + i;               // row of this drone inside the warp's tile
                if (p.obs_bulk && p.T > 1) bulk_drain();              // the previous step's copy has read the tile
                float* const tile = reinterpret_cast<float*>(s_obst) + p.smem_tile_off + (thread_index() >> 5) * (32 * p.obs_dp);  // = s_tile
                write_observation<NP>(p, s, nvel, nz, i, valid, s_obst_env, dmin2, tile + slot * p.obs_dp, obst_r);
                QS_TL(5);
                const int env_first = env - (thread_index() & 31) / NP;                   // first env of this warp
                const int envs_here = min(32 / NP, p.E - env_first);
                if (envs_here > 0)
                    emit_observation_tile(p, tile, gbase + (long long)env_first * p.N * p.D, env_first * p.N,
                                          p.last_obs_only ? 0 : t, envs_here * p.N, lane);
                __syncwarp();
            } else {
                write_observation<NP>(p, s, nvel, nz, i, valid, s_obst_env, dmin2, gbase + a * p.D, obst_r);
            }
            if (NZ && p.nz.rot) {
#pragma unroll
                for (int k = 0; k < 9; ++k) s.R[k] = R_true[k];
            }
        }
        if (!SPLIT && dev_scn && __any_sync(0xffffffffu, scn_ev && !kicked)) {      // scenario tick, site B
            const V3 g = {s.goal[0], s.goal[1], s.goal[2]};
            const bool act = scn_ev && !kicked;
            const ScnOut o = p.use_obst ? obstacle_scenario_tick<NP>(key, p.N, i, ctr.tick, g, act, st, env, p.grid_l, p.grid_w, p.M)
                                         : scenario_tick<NP>(key, p.N, i, ctr.tick, g, act, st, env);
            if (act) {
                s.goal[0] = o.goal.x; s.goal[1] = o.goal.y; s.goal[2] = o.goal.z;
                scn_next = o.next;
                goal_dirty = true;
                late_goal = true;
            }
        }
        ctr.step_count += 1;
    }

    if (!HO) asm volatile("griddepcontrol.launch_dependents;");                 // late trigger: overlap only the launch latency
    QS_TL(6);
    if (SPLIT || late_goal) {
        if (valid) store_agent(st, a, s, goal_dirty);
        if (valid && dsum_dirty) st.slots[SL_DIST_SUMS * st.a_pad + a] = dsum;
        if (env_ok && i == 0) st.env_ctr[env] = make_int4(ctr.tick, ctr.step_count, ctr.svd_count, ctr.episode_idx);
        if (gyro_model && valid) p.gyro_bias[a] = make_float4(gb.x, gb.y, gb.z, 0.f);
    }
    if (!SPLIT && p.obs_bulk) {
        if (has_courier) bulk_drain_writes();         // ... and the `done` word promises that the rows are written
        else bulk_drain();                            // shared memory must outlive the bulk copy's reads
    }
    if (HO) {
        if (has_courier) named_arrive(3, block_threads());
        else {
            if (SPLIT) bar_sync(4); else __syncthreads();
            if (threadIdx.x == 0) handover_release(st.ready + blockIdx.x);
        }
    }
    QS_TL(7);
}

// Explicit reset of the masked envs: QuadrotorEnvMulti.reset, quadrotor_multi.py:339-411.  NZ: custom sensor-noise model.
// RND: random initial states (qs_set_init_random_state).
template <int NP, bool NZ = false, bool RND = false>
__global__ void __launch_bounds__(128) qs_reset_kernel(const __grid_constant__ StepParams p) {
    extern __shared__ __align__(128) float2 s_obst[];
    const DevState& st = p.st;
    const int lane = threadIdx.x & 31;
    const int i = lane & (NP - 1);
    const int envs_per_block = blockDim.x / NP;
    const int env_local = threadIdx.x / NP;
    const int env = blockIdx.x * envs_per_block + env_local;
    const bool env_ok = env < p.E && (p.env_mask == nullptr || p.env_mask[env] != 0);
    const bool valid = env_ok && i < p.N;
    const long long a = (long long)env * p.N + i;
    float2* s_obst_env = s_obst + env_local * p.M;

    Agent s;
    if (valid) load_agent(st, a, s);
    else idle_agent(s, i);
    EnvCtr ctr = {0, 0, 0, 0};
    if (env_ok) {
        const int4 c = st.env_ctr[env];
        ctr.tick = c.x; ctr.step_count = c.y; ctr.svd_count = c.z; ctr.episode_idx = c.w;
    }
    const RngKey key = step_key(p, env, ctr.step_count);
    float nvel[3] = {0.f, 0.f, 0.f};
    // every lane of the warp takes part in the shuffles below; lanes of unmasked envs write nothing
    int scn_next = SCN_NEVER;
    float approach = p.approach_metric;
    float obst_r = p.obst_radius;
    reset_env<NP, true>(p, key, s, a, env, i, env_ok, valid, ctr.tick, s_obst_env, nvel, scn_next, approach, obst_r, RND);
    if (st.dyn != nullptr) {          // pending physical constants are latched by explicit resets too
        const int pend = env_ok ? QS_LD(st.dyn_pending + env) : 0;
        if (pend != 0) {
            if (valid) {
                for (int q = 0; q < QS_DYN_ROW / 4; ++q)
                    st.dyn[a * (QS_DYN_ROW / 4) + q] = QS_LD(st.next_dyn + a * (QS_DYN_ROW / 4) + q);
#pragma unroll
                for (int k = 0; k < 4; ++k) s.ou[k] = 0.f;
            }
            ctr.svd_count = 0;
        }
        __syncwarp();
        if (pend != 0 && i == 0) st.dyn_pending[env] = 0;
    }
    if (env_ok && i == 0) {
        int32_t* c = st.env_cnt + (long long)env * QS_NUM_ENV_STATS;
        for (int k = 0; k < QS_NUM_ENV_STATS; ++k) c[k] = 0;
        st.env_ctr[env] = make_int4(0, ctr.step_count + 1, ctr.svd_count, ctr.episode_idx);
    }
    Noise9 nz;
#pragma unroll
    for (int k = 0; k < 3; ++k) { nz.p[k] = 0.f; nz.v[k] = 0.f; nz.w[k] = 0.f; }
    if (NZ) {
        const bool gyro_model = p.gyro_bias != nullptr;
        float3 gb = make_float3(0.f, 0.f, 0.f);
        if (gyro_model && valid) {
            const float4 b = p.gyro_bias[a];
            gb = make_float3(b.x, b.y, b.z);
        }
        const SensedNoise sn = sensor_noise_model(p.nz, key, 2, i, gb, gyro_model);
        nz = sn.n;
        if (gyro_model && valid) p.gyro_bias[a] = make_float4(sn.bias.x, sn.bias.y, sn.bias.z, 0.f);
        if (valid) store_agent(st, a, s, true);
        if (p.nz.rot) observed_rotation(s.R, sn.q, s.R);       // s.R is stored; only the observation sees the perturbed one
    } else if (p.sense_noise) nz = sensor_noise(key, SITE_SENSOR_RESET, i);
    write_observation<NP>(p, s, nvel, nz, i, valid, s_obst_env, p.use_obst ? min_pillar_dist2(p, s, s_obst_env) : 1e4f,
                          p.obs + a * p.D, obst_r);
    if (!NZ && valid) store_agent(st, a, s, true);
}

// Generates, for every env that does not hold one yet, the record of its NEXT episode (see generate_episode above).  Launched
// by the library every few hundred steps between two step launches, and after every explicit reset: an env's record is
// consumed at most once per episode, so the (expensive, latency-bound) generators never run inside a step.
template <int NP>
__global__ void __launch_bounds__(128) qs_pregen_kernel(const __grid_constant__ StepParams p) {
    const DevState& st = p.st;
    const int lane = threadIdx.x & 31;
    const int i = lane & (NP - 1);
    const int env = blockIdx.x * (blockDim.x / NP) + threadIdx.x / NP;
    const bool valid = env < p.E && i < p.N;
    const long long a = (long long)env * p.N + i;
    int2 ep = make_int2(0, 0);
    if (valid) ep = st.epi[env];
    const int g = ep.x + 1;
    const bool work = valid && ep.y != g;
    if (work) {
        const long long e3 = 3 * (long long)env;
        const EpisodeLane e = generate_episode<true>(p, episode_key(p, env, g), i, nullptr, st.next_obst + (long long)env * p.M,
                                                     st.next_scn_i + env, st.next_scn_f + e3);
        st.next_goal[a] = make_float4(e.goal.x, e.goal.y, e.goal.z, e.pose.cs);
        st.next_spawn[a] = make_float4(e.pose.pos.x, e.pose.pos.y, e.pose.pos.z, e.pose.sn);
    }
    __syncwarp();
    if (work && i == 0) st.epi[env] = make_int2(ep.x, g);
}

}  // namespace qs
