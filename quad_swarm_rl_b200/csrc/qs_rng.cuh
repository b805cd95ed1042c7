// Keyed Philox4x32-10 draws for the QuadSwarm step kernels (sm_90a).
//
// Device twin of oracle/philox.py: both define the same function
//   (seed, env, step_count, site, i, j, value_index) -> random value
// so the CPU oracle and these kernels consume identical random numbers.  The reference
// (gym_art/quadrotor_multi) draws from two order-dependent Mersenne-Twister streams
// (SURVEY.md Appendix C), which a data-parallel kernel cannot replay; the site table below
// names every draw site of the reference instead and gives it a fixed counter.
//
//   counter = (env_id, step_count, site | i << 8 | j << 16, block)   key = (seed_lo, seed_hi)
//   uniform01(x) = (x >> 8) * 2^-24                       (exact in fp32)
//   normal pair (xa, xb): u1 = ((xa >> 9) + 0.5) * 2^-23, u2 = (xb >> 8) * 2^-24,
//                         r = sqrt(-2 ln u1), n0 = r cos(2 pi u2), n1 = r sin(2 pi u2)
//   value index v lives in block v / 4, word v % 4; words (0,1) and (2,3) form the normal pairs.
//
// The integer part is bit-exact with the oracle.  The Box-Muller transcendentals use the SFU
// approximations (lg2 / sqrt / sin / cos .approx, each with an ABSOLUTE error bound).  lg2's sets the error
// of r = sqrt(-2 ln u1) where r is small (dr ~ 0.7 dlg2 / r).  Measured on an H100 over every value of u1
// and of u2 (tests/test_device_functions.py): |n - n_float64| <= 1.8e-4 for normal_pair, <= 1.2e-5 for
// normal_pair16, and every value is finite (at u1 = 1 - 2^-24, log2 u1 = -8.6e-8, r stays >= 0).  A drawn
// value sigma n is off by sigma times that: <= 1.2e-7 for the hot draws (sigma <= 0.01), 1.8e-4 sigma at the
// full-precision sites (contact responses, random initial states, a sensor-noise model with any sigma).
#pragma once
#include <cstdint>

namespace qs {

enum Site : uint32_t {
    SITE_OU = 0,            // (i)   normals v0..3                               numba_utils.py:103
    SITE_FLOOR_YAW = 1,     // (i)   uniforms v0 / v1 = sub-step 0 / 1           quadrotor_dynamics.py:617
    SITE_SENSOR0 = 2,       // (i)   normals v0..2 pos, v3..5 vel, v6..8 gyro    sensor_noise.py:241-251
    SITE_SENSOR1 = 3,       // (i)   re-draw after a contact response            quadrotor_multi.py:598-599
    SITE_SENSOR_RESET = 4,  // (i)   observation returned by an (auto-)reset
    SITE_DW_I = 5,          // (i)   uniforms v0 acc noise, v1 omega noise       downwash.py:30,35
    SITE_DW_IJ = 6,         // (i,j) uniforms v0..2 z-axis noise, v3..5 omega dir downwash.py:56,62
    SITE_PAIR_N = 7,        // (i<j) normals, try t: v[12t..12t+8]               collisions/quadrotors.py:36-38
    SITE_PAIR_U = 8,        // (i<j) uniforms v0,v1 decay, v2..4 omega dir, v5 omega mag  collisions/utils.py
    SITE_OBST_N = 9,        // (i)   normals, try t: v[8t..8t+5]                 collisions/obstacles.py:33-34
    SITE_OBST_U = 10,       // (i)   uniforms v0 decay, v1..3 omega dir, v4 omega mag
    SITE_WALL_U = 11,       // (i)   uniforms v0 speed, v1..3 dir, v4 x, v5 y, v6 z, v7..9 omega dir, v10 mag  collisions/room.py:10-40
    SITE_CEIL_U = 12,       // (i)   uniforms v0 speed, v1..3 dir, v4 z, v5..7 omega dir, v8 mag               collisions/room.py:94-110
    SITE_SPAWN_U = 13,      // (i)   uniforms v0..2                              quadrotor_single.py:394
    SITE_RESET_YAW_U = 14,  // (i)   uniforms v[k], k = rejection try            quadrotor_single.py:432-434
    SITE_SCENARIO_U = 15,   // (slot) env-level scenario generators
    SITE_HOT = 16,          // (i)   the draws every drone needs every step (OU + first sensor draw), compact layout below
    // 17 = SITE_REPLAY_U (qs_wrap.cuh).  The custom sensor-noise model (qs_set_sensor_noise) draws full-precision values from
    // its own sites (CPU twin: oracle/sensor_noise_oracle.py); j = which observation of the step: 0 its own, 1 the re-draw
    // after a contact response, 2 an (auto-)reset.
    SITE_NOISE_N = 18,      // (i,j) normals v0..2 pos, v4..6 vel, v8..10 gyro, v12..14 rotation angle   sensor_noise.py:241-256
    SITE_NOISE_U = 19,      // (i,j) uniforms v0..2 pos, v4..6 vel, v8..10 rotation angle
    SITE_GYRO_BIAS = 20,    // (i,j) normals v0..2 bias innovation, v4..6 random walk                    sensor_noise.py:221-231
    // Random initial state of a spawn (qs_set_init_random_state; QuadrotorDynamics.random_state, quadrotor_dynamics.py:193-206),
    // episode-keyed like SITE_SPAWN_U.  Full-precision draws; CPU twin: oracle/init_state_oracle.py.
    SITE_INIT_U = 21,       // (i)   uniforms v0..2 vel direction, v3 vel magnitude, v4..6 omega direction, v7 omega magnitude
    SITE_INIT_N = 22,       // (i)   normals v0..2 up, v[4(t+1)..4(t+1)+2] fwd of try t        rand_uniform_rot3d, quad_utils.py:94-104
    // Upside-down first floor contact of the numpy dynamics path (qs_set_numpy_dynamics; floor_interaction,
    // quadrotor_dynamics.py:434-437), step-keyed like SITE_FLOOR_YAW.  CPU twin: oracle/numpy_path_oracle.py.
    SITE_FLOOR_YAW_NP = 23, // (i,j) uniforms v[k], j = sub-step, k = rejection try of randyaw()
    // Per-drone physical constants of the device-side dynamics sampler (qs_set_dynamics_sampler, qs_dyn_sampler.cuh),
    // episode-keyed like SITE_SPAWN_U (episode 0 = the construction sample).  Draw k of drone i is block k: a uniform is
    // low + (high - low) u01(word 0), a normal is the float64 Box-Muller n0 of words (0, 1).  CPU twin:
    // oracle/dyn_sampler_oracle.py.
    SITE_DYN = 24,          // (i)   block k = the k-th scalar the host pipeline draws
};

constexpr int RESET_YAW_MAX_TRIES = 64;     // also caps the SITE_FLOOR_YAW_NP loop (reference: unbounded; p(re-draw) = 2/3)
constexpr int INIT_ROT_MAX_TRIES = 16;      // fwd re-draws of rand_uniform_rot3d (reference: unbounded; p(re-draw) ~ 2.5 %)

struct RngKey {
    uint32_t k0, k1;      // seed
    uint32_t env;         // global env id
    uint32_t step;        // per-env step counter
};

// Draws that define an EPISODE (pillar / spawn / goal generation, formation picks, spawn jitter, reset yaw) are keyed by the
// env's episode number, not by its step counter: counter word 1 = EPISODE_KEY_BIT | episode number.  An episode is then a
// function of (seed, env id, episode number) only, whenever and wherever it is generated — inside the reset path of the
// step kernel, or ahead of time by qs_pregen_kernel.  Sites: SITE_SCENARIO_U streams 0 / 1, SITE_SPAWN_U, SITE_RESET_YAW_U,
// SITE_INIT_U, SITE_INIT_N.
constexpr uint32_t EPISODE_KEY_BIT = 0x80000000u;

constexpr uint32_t PHILOX_M0 = 0xD2511F53u, PHILOX_M1 = 0xCD9E8D57u, PHILOX_W0 = 0x9E3779B9u, PHILOX_W1 = 0xBB67AE85u;

// One block.  The round loop stays rolled: the kernel is instruction-fetch bound, not issue bound.
__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                               uint32_t k0, uint32_t k1) {
#pragma unroll 1
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(PHILOX_M0, c0), lo0 = PHILOX_M0 * c0;
        const uint32_t hi1 = __umulhi(PHILOX_M1, c2), lo1 = PHILOX_M1 * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += PHILOX_W0;
        k1 += PHILOX_W1;
    }
    return make_uint4(c0, c1, c2, c3);
}

// Four independent blocks in one rolled loop (4-way ILP on the multiply chain): the per-step draws every
// drone always needs (OU thrust noise + three sensor-noise blocks).
__device__ __forceinline__ void philox4x32_10_x4(uint32_t c0, uint32_t c1, const uint32_t c2[4], const uint32_t c3[4],
                                                 uint32_t k0, uint32_t k1, uint4 out[4]) {
    uint32_t a[4], b[4], c[4], d[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { a[q] = c0; b[q] = c1; c[q] = c2[q]; d[q] = c3[q]; }
#pragma unroll 1
    for (int r = 0; r < 10; ++r) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint32_t hi0 = __umulhi(PHILOX_M0, a[q]), lo0 = PHILOX_M0 * a[q];
            const uint32_t hi1 = __umulhi(PHILOX_M1, c[q]), lo1 = PHILOX_M1 * c[q];
            a[q] = hi1 ^ b[q] ^ k0;
            b[q] = lo1;
            c[q] = hi0 ^ d[q] ^ k1;
            d[q] = lo0;
        }
        k0 += PHILOX_W0;
        k1 += PHILOX_W1;
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) out[q] = make_uint4(a[q], b[q], c[q], d[q]);
}

// Two independent blocks in one rolled loop: the hot per-step draws (SITE_HOT, see hot_normals below).
__device__ __forceinline__ void philox4x32_10_x2(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t k0, uint32_t k1, uint4 out[2]) {
    // blocks 0 and 1 of counter word 3
    uint32_t a[2] = {c0, c0}, b[2] = {c1, c1}, c[2] = {c2, c2}, d[2] = {0u, 1u};
#pragma unroll 1
    for (int r = 0; r < 10; ++r) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const uint32_t hi0 = __umulhi(PHILOX_M0, a[q]), lo0 = PHILOX_M0 * a[q];
            const uint32_t hi1 = __umulhi(PHILOX_M1, c[q]), lo1 = PHILOX_M1 * c[q];
            a[q] = hi1 ^ b[q] ^ k0;
            b[q] = lo1;
            c[q] = hi0 ^ d[q] ^ k1;
            d[q] = lo0;
        }
        k0 += PHILOX_W0;
        k1 += PHILOX_W1;
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) out[q] = make_uint4(a[q], b[q], c[q], d[q]);
}

__device__ __forceinline__ uint32_t rng_c2(uint32_t site, uint32_t i, uint32_t j) { return site | (i << 8) | (j << 16); }

__device__ __forceinline__ uint4 rng_block(const RngKey& k, uint32_t site, uint32_t i, uint32_t j, uint32_t block) {
    return philox4x32_10(k.env, k.step, rng_c2(site, i, j), block, k.k0, k.k1);
}

__device__ __forceinline__ float u01(uint32_t x) { return (float)(x >> 8) * 5.9604644775390625e-08f; }  // 2^-24

// SFU approximations (PTX *.approx.ftz.f32): one MUFU instruction each, no slow-path branches
__device__ __forceinline__ float fsqrt(float x) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float frcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float frsqrt(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float flg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fsin(float x) { float r; asm("sin.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fcos(float x) { float r; asm("cos.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

__device__ __forceinline__ void normal_pair(uint32_t xa, uint32_t xb, float& n0, float& n1) {
    const float u1 = ((float)(xa >> 9) + 0.5f) * 1.1920928955078125e-07f;   // 2^-23, exact
    const float u2 = (float)(xb >> 8) * 5.9604644775390625e-08f;
    const float r = fsqrt(-1.3862943611198906f * flg2(u1));                 // -2 ln u1 = -2 ln2 * lg2 u1
    // angle folded into [-pi, pi) where sin/cos.approx are most accurate: cos(2 pi u2) = -cos(2 pi (u2 - 1/2))
    const float ang = 6.283185307179586f * (u2 - 0.5f);
    n0 = -r * fcos(ang);
    n1 = -r * fsin(ang);
}

// Compact normal pair of ONE word (hot per-step draws): u1 = ((x >> 16) + 0.5) 2^-16, u2 = (x & 0xffff) 2^-16.
// |n| <= sqrt(2 ln 2^17) = 4.85; the two draws every drone makes every step (OU thrust noise, sigma 0.01, and the
// sensor noise, sigma <= 0.01) then need 7 words = 2 Philox blocks instead of 4.  Twin: oracle/philox.py hot_normal.
__device__ __forceinline__ void normal_pair16(uint32_t x, float& n0, float& n1) {
    const float u1 = ((float)(x >> 16) + 0.5f) * 1.52587890625e-05f;        // 2^-16, exact
    const float u2 = (float)(x & 0xffffu) * 1.52587890625e-05f;
    const float r = fsqrt(-1.3862943611198906f * flg2(u1));
    const float ang = 6.283185307179586f * (u2 - 0.5f);
    n0 = -r * fcos(ang);
    n1 = -r * fsin(ang);
}

// SITE_HOT layout (drone i, blocks 0 and 1 of counter word 3):
//   block 0: word 0 -> OU normals 0,1; word 1 -> OU 2,3; word 2 -> sensor 0,1 (pos x, y); word 3 -> sensor 2,3 (pos z, vel x)
//   block 1: word 0 -> sensor 4,5 (vel y, z); word 1 -> sensor 6,7 (gyro x, y); word 2 -> sensor 8 (gyro z), spare
struct HotNormals { float ou[4]; float sn[9]; };
__device__ __forceinline__ HotNormals hot_normals(const RngKey& k, uint32_t i) {
    uint4 blk[2];
    philox4x32_10_x2(k.env, k.step, rng_c2(SITE_HOT, i, 0), k.k0, k.k1, blk);
    HotNormals h;
    float spare;
    normal_pair16(blk[0].x, h.ou[0], h.ou[1]);
    normal_pair16(blk[0].y, h.ou[2], h.ou[3]);
    normal_pair16(blk[0].z, h.sn[0], h.sn[1]);
    normal_pair16(blk[0].w, h.sn[2], h.sn[3]);
    normal_pair16(blk[1].x, h.sn[4], h.sn[5]);
    normal_pair16(blk[1].y, h.sn[6], h.sn[7]);
    normal_pair16(blk[1].z, h.sn[8], spare);
    return h;
}

// 4 uniforms / 4 normals of one block
__device__ __forceinline__ float4 uniform4_of(const uint4 b) { return make_float4(u01(b.x), u01(b.y), u01(b.z), u01(b.w)); }
__device__ __forceinline__ float4 normal4_of(const uint4 b) {
    float4 n;
    normal_pair(b.x, b.y, n.x, n.y);
    normal_pair(b.z, b.w, n.z, n.w);
    return n;
}
__device__ __forceinline__ float4 rng_uniform4(const RngKey& k, uint32_t site, uint32_t i, uint32_t j, uint32_t block) {
    return uniform4_of(rng_block(k, site, i, j, block));
}
__device__ __forceinline__ float4 rng_normal4(const RngKey& k, uint32_t site, uint32_t i, uint32_t j, uint32_t block) {
    return normal4_of(rng_block(k, site, i, j, block));
}

}  // namespace qs
