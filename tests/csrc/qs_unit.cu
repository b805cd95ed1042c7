// Test-only device harness: one __global__ wrapper per device function of qs_device.cuh / qs_rng.cuh, one element per
// thread, so that tests/test_device_functions.py can feed chosen inputs to each function and compare it with its float64
// twin in oracle/.  The production header is included unchanged and no device code is copied.
//
// Every entry point takes caller-owned device pointers (torch tensors), the element count and a stream, and returns the
// launch's cudaError_t; the harness allocates nothing.  Counter words of keyed draws come per element as
// ctr[t] = (env, step, i, j) with the seed (k0, k1) shared.  Agents travel as their raw struct (AGENT_WORDS 32-bit words,
// layout of qs::Agent), physical constants as QS_DYN_ROW-float rows (the qs_set_dynamics layout read by load_phys).
//
// Built twice by __graft_entry__.build() with the product's NVCC_FLAGS: libqs_unit.so (QS_CONTROL_MODES=1) and
// libqs_unit_npy.so (QS_NUMPY_DYNAMICS=1 QS_CONTROL_MODES=1, the numpy path's floor model).  The product never loads them.
#include "../../quad_swarm_rl_b200/csrc/qs_device.cuh"

using namespace qs;

constexpr int AGENT_WORDS = 39;
static_assert(sizeof(Agent) == AGENT_WORDS * 4, "tests/test_device_functions.py mirrors the Agent layout");

namespace {

constexpr int BLOCK = 256;
inline int grid_of(int n) { return (n + BLOCK - 1) / BLOCK; }

__device__ __forceinline__ int tid() { return blockIdx.x * blockDim.x + threadIdx.x; }
__device__ __forceinline__ RngKey key_of(uint32_t k0, uint32_t k1, const uint4* ctr, int t) {
    return RngKey{k0, k1, ctr[t].x, ctr[t].y};
}
__device__ __forceinline__ V3 v3(const float* p) { return V3{p[0], p[1], p[2]}; }
__device__ __forceinline__ void put(float* o, V3 v) { o[0] = v.x; o[1] = v.y; o[2] = v.z; }
__device__ __forceinline__ void put_kick(float* o, const KickVO& k) { put(o, k.vel); put(o + 3, k.dom); }

// ---- RNG ----
__global__ void k_philox(const uint4* ctr, const uint2* key, uint4* out, int n) {
    const int t = tid(); if (t >= n) return;
    const uint4 c = ctr[t];
    out[t] = philox4x32_10(c.x, c.y, c.z, c.w, key[t].x, key[t].y);
}
// blocks 0 and 1 of counter word 3 for counter words (c0, c1, c2) = ctr[t].xyz
__global__ void k_philox_x2(const uint4* ctr, const uint2* key, uint4* out, int n) {
    const int t = tid(); if (t >= n) return;
    const uint4 c = ctr[t];
    uint4 o[2];
    philox4x32_10_x2(c.x, c.y, c.z, key[t].x, key[t].y, o);
    out[2 * t] = o[0]; out[2 * t + 1] = o[1];
}
// four blocks: counter words 0, 1 shared = c01[t], words 2 / 3 of block q = c2[4 t + q] / c3[4 t + q]
__global__ void k_philox_x4(const uint2* c01, const uint32_t* c2, const uint32_t* c3, const uint2* key, uint4* out, int n) {
    const int t = tid(); if (t >= n) return;
    uint4 o[4];
    philox4x32_10_x4(c01[t].x, c01[t].y, c2 + 4 * t, c3 + 4 * t, key[t].x, key[t].y, o);
    for (int q = 0; q < 4; ++q) out[4 * t + q] = o[q];
}
__global__ void k_u01(const uint32_t* x, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    out[t] = u01(x[t]);
}
__global__ void k_normal_pair(const uint32_t* xa, const uint32_t* xb, float2* out, int n) {
    const int t = tid(); if (t >= n) return;
    float a, b;
    normal_pair(xa[t], xb[t], a, b);
    out[t] = make_float2(a, b);
}
__global__ void k_normal_pair16(const uint32_t* x, float2* out, int n) {
    const int t = tid(); if (t >= n) return;
    float a, b;
    normal_pair16(x[t], a, b);
    out[t] = make_float2(a, b);
}

// ---- rotation ----
__global__ void k_orthonormalize(const float* in, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    M3 m;
    for (int k = 0; k < 9; ++k) m.m[k] = in[9 * t + k];
    m = orthonormalize(m);
    for (int k = 0; k < 9; ++k) out[9 * t + k] = m.m[k];
}
__global__ void k_observed_rotation(const float* R, const float* qt, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    float r[9], q[4], o[9];
    for (int k = 0; k < 9; ++k) r[k] = R[9 * t + k];
    for (int k = 0; k < 4; ++k) q[k] = qt[4 * t + k];
    observed_rotation(r, q, o);
    for (int k = 0; k < 9; ++k) out[9 * t + k] = o[k];
}
__global__ void k_yaw_only(const float* in, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    float r[9];
    for (int k = 0; k < 9; ++k) r[k] = in[9 * t + k];
    yaw_only(r);
    for (int k = 0; k < 9; ++k) out[9 * t + k] = r[k];
}

// ---- physics sub-step: variant 0 dynamics_substep<false>, 1 dynamics_substep<true> (FMA_FRICTION), 2 dynamics_substep_dyn
// with row t of `rows`.  ctr[t] = (env, step, i, sub).
__global__ void k_substep(int variant, Agent* s, const float* cmd, const int* do_svd, const float* room, uint32_t k0,
                          uint32_t k1, const uint4* ctr, const float4* rows, int n) {
    const int t = tid(); if (t >= n) return;
    StepParams p;
    for (int k = 0; k < 3; ++k) { p.room_lo[k] = room[k]; p.room_hi[k] = room[3 + k]; }
    const RngKey key = key_of(k0, k1, ctr, t);
    const int i = (int)ctr[t].z, sub = (int)ctr[t].w;
    Agent a = s[t];
    float c[4];
    for (int m = 0; m < 4; ++m) c[m] = cmd[4 * t + m];
    if (variant == 0) {
        dynamics_substep<false>(a, c, do_svd[t] != 0, p, key, i, sub);
    } else if (variant == 1) {
        dynamics_substep<true>(a, c, do_svd[t] != 0, p, key, i, sub);
    } else {
        Phys ph;
        load_phys(rows, t, ph);
        dynamics_substep_dyn(a, c, do_svd[t] != 0, p, key, i, sub, ph);
    }
    s[t] = a;
}

// ---- controller ----
__global__ void k_jacobian_inverse(const float4* rows, double* out, int n) {
    const int t = tid(); if (t >= n) return;
    Phys ph;
    load_phys(rows, t, ph);
    double ji[16];
    jacobian_inverse<true>(ph, ji);
    for (int k = 0; k < 16; ++k) out[16 * t + k] = ji[k];
}
// rows == nullptr: position_control<false> (Crazyflie constants), else position_control<true> with row t
__global__ void k_position_control(const Agent* s, const float4* rows, float* cmd, int n) {
    const int t = tid(); if (t >= n) return;
    const Agent a = s[t];
    float c[4];
    if (rows == nullptr) {
        position_control<false>(a, Phys{}, c);
    } else {
        Phys ph;
        load_phys(rows, t, ph);
        position_control<true>(a, ph, c);
    }
    for (int m = 0; m < 4; ++m) cmd[4 * t + m] = c[m];
}

// ---- contact responses ----
// in[t] = p1, v1, p2, v2; out[t] = new v1, new v2, delta omega (+ for a, - for b); ctr[t] = (env, step, a, b)
__global__ void k_pair_response(uint32_t k0, uint32_t k1, const uint4* ctr, const float* in, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    const float* q = in + 12 * t;
    const PairOut o = pair_response(key_of(k0, k1, ctr, t), (int)ctr[t].z, (int)ctr[t].w, v3(q), v3(q + 3), v3(q + 6), v3(q + 9));
    put(out + 9 * t, o.v1); put(out + 9 * t + 3, o.v2); put(out + 9 * t + 6, o.dom);
}
// in[t] = pos, vel, obstacle xyz, obstacle half size; out[t] = new vel, delta omega
__global__ void k_obstacle_response(uint32_t k0, uint32_t k1, const uint4* ctr, const float* in, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    const float* q = in + 10 * t;
    put_kick(out + 6 * t, obstacle_response(key_of(k0, k1, ctr, t), (int)ctr[t].z, v3(q), v3(q + 3), q[6], q[7], q[8], q[9]));
}
__global__ void k_wall_response(uint32_t k0, uint32_t k1, const uint4* ctr, const float* vel, const int2* touch, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    put_kick(out + 6 * t, wall_response(key_of(k0, k1, ctr, t), (int)ctr[t].z, v3(vel + 3 * t), touch[t].x, touch[t].y));
}
__global__ void k_ceiling_response(uint32_t k0, uint32_t k1, const uint4* ctr, const float* vel, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    put_kick(out + 6 * t, ceiling_response(key_of(k0, k1, ctr, t), (int)ctr[t].z, v3(vel + 3 * t)));
}
// in[t] = distance, body z-axis of `other`; ctr[t] = (env, step, other, me)
__global__ void k_downwash_kick(uint32_t k0, uint32_t k1, const uint4* ctr, const float* in, float* out, int n) {
    const int t = tid(); if (t >= n) return;
    const float* q = in + 4 * t;
    put_kick(out + 6 * t, downwash_kick(key_of(k0, k1, ctr, t), (int)ctr[t].z, (int)ctr[t].w, q[0], q[1], q[2], q[3]));
}

}  // namespace

#define QS_UNIT_LAUNCH(kernel, ...)                                                            \
    do {                                                                                       \
        if (n <= 0) return cudaSuccess;                                                        \
        kernel<<<grid_of(n), BLOCK, 0, stream>>>(__VA_ARGS__);                                 \
        return cudaGetLastError();                                                             \
    } while (0)

extern "C" {

int qs_unit_agent_words() { return AGENT_WORDS; }
int qs_unit_numpy_dynamics() { return QS_NUMPY_DYNAMICS; }

cudaError_t qs_unit_philox(const void* ctr, const void* key, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_philox, (const uint4*)ctr, (const uint2*)key, (uint4*)out, n);
}
cudaError_t qs_unit_philox_x2(const void* ctr, const void* key, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_philox_x2, (const uint4*)ctr, (const uint2*)key, (uint4*)out, n);
}
cudaError_t qs_unit_philox_x4(const void* c01, const void* c2, const void* c3, const void* key, void* out, int n,
                              cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_philox_x4, (const uint2*)c01, (const uint32_t*)c2, (const uint32_t*)c3, (const uint2*)key, (uint4*)out, n);
}
cudaError_t qs_unit_u01(const void* x, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_u01, (const uint32_t*)x, (float*)out, n);
}
cudaError_t qs_unit_normal_pair(const void* xa, const void* xb, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_normal_pair, (const uint32_t*)xa, (const uint32_t*)xb, (float2*)out, n);
}
cudaError_t qs_unit_normal_pair16(const void* x, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_normal_pair16, (const uint32_t*)x, (float2*)out, n);
}
cudaError_t qs_unit_orthonormalize(const void* in, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_orthonormalize, (const float*)in, (float*)out, n);
}
cudaError_t qs_unit_observed_rotation(const void* R, const void* qt, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_observed_rotation, (const float*)R, (const float*)qt, (float*)out, n);
}
cudaError_t qs_unit_yaw_only(const void* in, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_yaw_only, (const float*)in, (float*)out, n);
}
cudaError_t qs_unit_substep(int variant, void* agents, const void* cmd, const void* do_svd, const void* room, uint32_t k0,
                            uint32_t k1, const void* ctr, const void* rows, int n, cudaStream_t stream) {
    if (variant < 0 || variant > 2 || (variant == 2 && rows == nullptr)) return cudaErrorInvalidValue;
    QS_UNIT_LAUNCH(k_substep, variant, (Agent*)agents, (const float*)cmd, (const int*)do_svd, (const float*)room, k0, k1,
                   (const uint4*)ctr, (const float4*)rows, n);
}
cudaError_t qs_unit_jacobian_inverse(const void* rows, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_jacobian_inverse, (const float4*)rows, (double*)out, n);
}
cudaError_t qs_unit_position_control(const void* agents, const void* rows, void* cmd, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_position_control, (const Agent*)agents, (const float4*)rows, (float*)cmd, n);
}
cudaError_t qs_unit_pair_response(uint32_t k0, uint32_t k1, const void* ctr, const void* in, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_pair_response, k0, k1, (const uint4*)ctr, (const float*)in, (float*)out, n);
}
cudaError_t qs_unit_obstacle_response(uint32_t k0, uint32_t k1, const void* ctr, const void* in, void* out, int n,
                                      cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_obstacle_response, k0, k1, (const uint4*)ctr, (const float*)in, (float*)out, n);
}
cudaError_t qs_unit_wall_response(uint32_t k0, uint32_t k1, const void* ctr, const void* vel, const void* touch, void* out, int n,
                                  cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_wall_response, k0, k1, (const uint4*)ctr, (const float*)vel, (const int2*)touch, (float*)out, n);
}
cudaError_t qs_unit_ceiling_response(uint32_t k0, uint32_t k1, const void* ctr, const void* vel, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_ceiling_response, k0, k1, (const uint4*)ctr, (const float*)vel, (float*)out, n);
}
cudaError_t qs_unit_downwash_kick(uint32_t k0, uint32_t k1, const void* ctr, const void* in, void* out, int n, cudaStream_t stream) {
    QS_UNIT_LAUNCH(k_downwash_kick, k0, k1, (const uint4*)ctr, (const float*)in, (float*)out, n);
}

}  // extern "C"
