// Device-side dynamics randomisation (qs_set_dynamics_sampler): the whole host pipeline of quad_models.DynamicsSource
// for one drone — base set or RandomQuad (quadrotor_randomization.py:142-243), dynamics_change, up to two samplers
// (:50-110, :345-377), check_quad_param_limits (:16-48), the link inertia model (inertia.py:182-310) and
// QuadrotorDynamics.update_model (quadrotor_dynamics.py:104-166) — in float64, rounded to the float32 row once.
// Every operation follows quad_models.py in the same order, so that this function and its CPU twin (the unmodified
// host pipeline fed with the same keyed draws, oracle/dyn_sampler_oracle.py) agree to float64 rounding.  Rare path: runs
// once per drone at a resampling reset, never on a step's common path.
#pragma once
#include "qs_device.cuh"

namespace qs {

// resample at the reset that starts episode g (>= 1): the reference's (traj_count + 1) % every == 0, traj_count = g - 1
__host__ __device__ __forceinline__ bool dyn_due(int g, int every) { return every > 0 && g % every == 0; }

// The keyed draws of one drone: draw k is block k of SITE_DYN.
struct DynDraws {
    RngKey key;
    uint32_t i, k;
    __device__ double uniform(double lo, double hi) {
        const uint4 b = rng_block(key, SITE_DYN, i, 0, k++);
        return lo + (hi - lo) * ((double)(b.x >> 8) * 5.9604644775390625e-08);
    }
    __device__ double normal(double loc, double scale) {
        const uint4 b = rng_block(key, SITE_DYN, i, 0, k++);
        const double u1 = ((double)(b.x >> 9) + 0.5) * 1.1920928955078125e-07;
        const double u2 = (double)(b.y >> 8) * 5.9604644775390625e-08;
        return loc + scale * (sqrt(-2.0 * log(u1)) * cos(2.0 * 3.141592653589793 * u2));
    }
};

__device__ __forceinline__ double dclip_lo(double x, double lo) { return fmax(x, lo); }
__device__ __forceinline__ double dclip(double x, double lo, double hi) { return fmin(fmax(x, lo), hi); }

// randomquad_parameters (quad_models.py:202-240) without its final limits check; draws in its order
__device__ __forceinline__ void randomquad_leaves(double* L, DynDraws& d) {
    const double dlo[5] = {500., 200., 500., 500., 200.}, dhi[5] = {2000., 2000., 2000., 4500., 300.};
    const int dens[5] = {QS_DL_BODY_DENSITY, QS_DL_PAYLOAD_DENSITY, QS_DL_ARMS_DENSITY, QS_DL_MOTORS_DENSITY, QS_DL_PROPS_DENSITY};
#pragma unroll 1
    for (int k = 0; k < 5; ++k) L[dens[k]] = d.uniform(dlo[k], dhi[k]);
    const double total_w = d.uniform(0.05, 0.2);
    const double total_l = dclip_lo(d.normal(1., 0.1), 1.0) * total_w;
    const double motor_z = d.normal(0., total_w / 8.);
    L[QS_DL_MOTOR_POS_X] = total_w / 2.; L[QS_DL_MOTOR_POS_Y] = total_l / 2.; L[QS_DL_MOTOR_POS_Z] = motor_z;
    L[QS_DL_MOTORS_R] = total_w * d.normal(0.1, 0.01);
    L[QS_DL_MOTORS_H] = L[QS_DL_MOTORS_R] * d.normal(1.0, 0.05);
    const double w_low = 0.25, w_high = 0.5;
    const double w_coeff = d.uniform(w_low, w_high);
    L[QS_DL_BODY_W] = w_coeff * total_w;
    const double l_scale = (1. - (w_coeff - w_low) / (w_high - w_low));
    L[QS_DL_BODY_L] = dclip_lo(d.normal(1., l_scale), 1.0) * L[QS_DL_BODY_W];
    L[QS_DL_BODY_H] = d.uniform(0.1, 1.5) * L[QS_DL_BODY_W];
    const double pl0 = d.uniform(0.25, 1.0), pl1 = d.uniform(0.25, 1.0), pl2 = d.uniform(0.25, 1.0);
    L[QS_DL_PAYLOAD_W] = pl0 * L[QS_DL_BODY_W];
    L[QS_DL_PAYLOAD_L] = pl1 * L[QS_DL_BODY_L];
    L[QS_DL_PAYLOAD_H] = pl2 * L[QS_DL_BODY_H];
    L[QS_DL_PAYLOAD_X] = d.normal(0., L[QS_DL_BODY_W] / 10.);
    L[QS_DL_PAYLOAD_Y] = d.normal(0., L[QS_DL_BODY_W] / 10.);
    const double zs = d.uniform(-1., 1.);
    L[QS_DL_PAYLOAD_Z_SIGN] = zs > 0. ? 1. : (zs < 0. ? -1. : 0.);
    L[QS_DL_ARMS_W] = total_w * d.normal(0.05, 0.005);
    L[QS_DL_ARMS_H] = total_w * d.normal(0.05, 0.005);
    L[QS_DL_ARMS_ANGLE] = d.normal(45., 10.);
    L[QS_DL_ARMS_Z] = motor_z - L[QS_DL_MOTORS_H] / 2.;
    const double t2w = d.uniform(1.5, 3.5);
    L[QS_DL_PROPS_H] = 0.01;
    L[QS_DL_PROPS_R] = 0.3 * total_w * sqrt(t2w / 2.0);
    L[QS_DL_THRUST_NOISE_RATIO] = d.uniform(0.01, 0.05);
    const double damp_up = d.uniform(0.15, 0.2);
    const double damp_down_scale = d.uniform(1.0, 1.0);
    L[QS_DL_THRUST_TO_WEIGHT] = t2w;
    L[QS_DL_TORQUE_TO_THRUST] = d.uniform(0.005, 0.025);
#pragma unroll 1
    for (int k = 0; k < 4; ++k) L[QS_DL_ASSYMETRY0 + k] = d.uniform(0.9, 1.1);
    L[QS_DL_LINEARITY] = 1.0; L[QS_DL_C_DRAG] = 0.; L[QS_DL_C_ROLL] = 0.;
    L[QS_DL_DAMP_TIME_UP] = damp_up; L[QS_DL_DAMP_TIME_DOWN] = damp_down_scale * damp_up;
    L[QS_DL_DAMP_VEL] = 0.; L[QS_DL_DAMP_OMEGA_QUADRATIC] = 0.;
}

// check_quad_param_limits (quad_models.py:176-198); init = the tree before the sampler (propeller-radius rescale) or null
__device__ __forceinline__ void check_limits(double* L, const uint8_t* P, const double* init) {
#pragma unroll 1
    for (int k = QS_DL_BODY_L; k <= QS_DL_PROPS_DENSITY; ++k)
        if (P[k]) L[k] = dclip_lo(L[k], 0.);
    L[QS_DL_MOTOR_POS_X] = dclip_lo(L[QS_DL_MOTOR_POS_X], 0.005);
    L[QS_DL_MOTOR_POS_Y] = dclip_lo(L[QS_DL_MOTOR_POS_Y], 0.005);
    const double bw = L[QS_DL_BODY_W];
    L[QS_DL_PAYLOAD_X] = dclip(L[QS_DL_PAYLOAD_X], -bw / 4., bw / 4.);
    L[QS_DL_PAYLOAD_Y] = dclip(L[QS_DL_PAYLOAD_Y], -bw / 4., bw / 4.);
    L[QS_DL_ARMS_ANGLE] = dclip(L[QS_DL_ARMS_ANGLE], 0., 90.);
    L[QS_DL_DAMP_VEL] = dclip(L[QS_DL_DAMP_VEL], 0., 1.);
    L[QS_DL_DAMP_OMEGA_QUADRATIC] = dclip(L[QS_DL_DAMP_OMEGA_QUADRATIC], 0., 1.);
    L[QS_DL_THRUST_TO_WEIGHT] = dclip_lo(L[QS_DL_THRUST_TO_WEIGHT], 1.2);
    L[QS_DL_TORQUE_TO_THRUST] = dclip(L[QS_DL_TORQUE_TO_THRUST], 0.001, 1.);
    L[QS_DL_LINEARITY] = dclip(L[QS_DL_LINEARITY], 0., 1.);
#pragma unroll 1
    for (int k = 0; k < 4; ++k) L[QS_DL_ASSYMETRY0 + k] = dclip(L[QS_DL_ASSYMETRY0 + k], 0.9, 1.1);
    L[QS_DL_C_DRAG] = dclip_lo(L[QS_DL_C_DRAG], 0.);
    L[QS_DL_C_ROLL] = dclip_lo(L[QS_DL_C_ROLL], 0.);
    L[QS_DL_DAMP_TIME_UP] = dclip_lo(L[QS_DL_DAMP_TIME_UP], 0.);
    L[QS_DL_DAMP_TIME_DOWN] = dclip_lo(L[QS_DL_DAMP_TIME_DOWN], 0.);
    if (init != nullptr)
        L[QS_DL_PROPS_R] = init[QS_DL_PROPS_R] * sqrt(init[QS_DL_THRUST_TO_WEIGHT] / L[QS_DL_THRUST_TO_WEIGHT]);
}

// _mass (quad_models.py:58): `m` when the part has one, else density * volume
__device__ __forceinline__ double part_mass(const double* L, const uint8_t* P, int m_leaf, double volume) {
    return P[m_leaf] ? L[m_leaf] : L[m_leaf + 1] * volume;
}

// Link j of quad_link's 14 (body, payload, arms 0-3, motors 0-3, propellers 0-3): mass, own inertia diagonal, z-rotation,
// position.  Motors and arms in the order front-right, back-right, back-left, front-left (x signs + - - +, y signs - - + +).
__device__ __forceinline__ void quad_link_part(const double* L, const uint8_t* P, int j, double angle, double arms_l,
                                               double* t) {
    const int k = j < 2 ? 0 : (j - 2) & 3;
    const double sx = (k == 0 || k == 3) ? 1. : -1., sy = k < 2 ? -1. : 1.;
    const double mx = L[QS_DL_MOTOR_POS_X], my = L[QS_DL_MOTOR_POS_Y], mz = L[QS_DL_MOTOR_POS_Z];
    double m, I0, I1, I2, a = 0., x, y, z;
    if (j < 6) {            // boxes: body, payload, arms
        const int b = j == 0 ? QS_DL_BODY_L : (j == 1 ? QS_DL_PAYLOAD_L : QS_DL_ARMS_L);
        const double l = j < 2 ? L[b] : arms_l, w = L[b + 1], h = L[b + 2];
        m = part_mass(L, P, b + 3, l * w * h);
        I0 = m / 12. * (h * h + w * w); I1 = m / 12. * (l * l + h * h); I2 = m / 12. * (w * w + l * l);
        if (j == 0) {
            x = 0.; y = 0.; z = 0.;
        } else if (j == 1) {
            const double zs = L[QS_DL_PAYLOAD_Z_SIGN];
            x = L[QS_DL_PAYLOAD_X]; y = L[QS_DL_PAYLOAD_Y];
            z = (zs > 0. ? 1. : (zs < 0. ? -1. : 0.)) * (L[QS_DL_BODY_H] + L[QS_DL_PAYLOAD_H]) / 2;
        } else {
            const double delta_y = my - L[QS_DL_BODY_W] / 2.;
            a = (k % 2 == 0) ? -angle : angle;
            x = sx * (mx - delta_y / (2 * tan(angle))); y = sy * (my - delta_y / 2); z = L[QS_DL_ARMS_Z];
        }
    } else {                // cylinders: motors, propellers
        const int b = j < 10 ? QS_DL_MOTORS_H : QS_DL_PROPS_H;
        const double h = L[b], r = L[b + 1];
        m = part_mass(L, P, b + 2, 3.141592653589793 * h * (r * r));
        I0 = m / 12. * (3 * (r * r) + h * h); I1 = I0; I2 = 0.5 * m * (r * r);
        x = sx * mx; y = sy * my; z = j < 10 ? mz : mz + (L[QS_DL_MOTORS_H] / 2. + L[QS_DL_PROPS_H]);
    }
    t[0] = m; t[1] = I0; t[2] = I1; t[3] = I2; t[4] = a; t[5] = x; t[6] = y; t[7] = z;
}

// quad_link + derive_constants (quad_models.py:62-143) -> the row (DYN_FIELDS), still in float64.  The 14 links go through
// a table in local memory and rolled loops: a rare path, kept to few registers.
__device__ __forceinline__ void derive_row(const double* L, const uint8_t* P, double* row) {
    double angle = L[QS_DL_ARMS_ANGLE] / 180. * 3.141592653589793;
    if (angle == 0.) angle = 0.01;
    const double mx = L[QS_DL_MOTOR_POS_X], my = L[QS_DL_MOTOR_POS_Y], mz = L[QS_DL_MOTOR_POS_Z];
    const double arms_l = P[QS_DL_ARMS_L] ? L[QS_DL_ARMS_L] : (my - L[QS_DL_BODY_W] / 2.) / sin(angle);
    double t[14][8];
#pragma unroll 1
    for (int j = 0; j < 14; ++j) quad_link_part(L, P, j, angle, arms_l, t[j]);
    // np.sum of the 14 masses (numpy's pairwise summation: eight partial sums, then the rest in order)
    double mass = ((t[0][0] + t[1][0]) + (t[2][0] + t[3][0])) + ((t[4][0] + t[5][0]) + (t[6][0] + t[7][0]));
#pragma unroll 1
    for (int j = 8; j < 14; ++j) mass += t[j][0];
    double com[3] = {0., 0., 0.};
#pragma unroll 1
    for (int j = 0; j < 14; ++j) {
        com[0] = com[0] + t[j][0] * t[j][5]; com[1] = com[1] + t[j][0] * t[j][6]; com[2] = com[2] + t[j][0] * t[j][7];
    }
    com[0] = com[0] / mass; com[1] = com[1] / mass; com[2] = com[2] / mass;
    double I[3] = {0., 0., 0.};
#pragma unroll 1
    for (int j = 0; j < 14; ++j) {
        double c = 1.0, s = 0.0;
        if (t[j][4] != 0.) { c = cos(t[j][4]); s = sin(t[j][4]); }
        const double m = t[j][0], x = t[j][5] - com[0], y = t[j][6] - com[1], z = t[j][7] - com[2];
        I[0] += (c * c * t[j][1] + s * s * t[j][2]) + m * (y * y + z * z);
        I[1] += (s * s * t[j][1] + c * c * t[j][2]) + m * (x * x + z * z);
        I[2] += t[j][3] + m * (x * x + y * y);
    }
    // derive_constants
    double asum = 0.;
#pragma unroll 1
    for (int k = 0; k < 4; ++k) asum += L[QS_DL_ASSYMETRY0 + k];
    const double dt = 0.005, EPS = 1e-6, G = 9.81;
    row[0] = mass; row[1] = 1.0 / mass;
#pragma unroll 1
    for (int c = 0; c < 3; ++c) { row[2 + c] = I[c]; row[5 + c] = 1.0 / I[c]; }
#pragma unroll 1
    for (int k = 0; k < 4; ++k) {
        const double asym = L[QS_DL_ASSYMETRY0 + k] * 4. / asum;
        const double tm = G * mass * L[QS_DL_THRUST_TO_WEIGHT] * asym / 4.0;
        row[8 + k] = tm;
        row[12 + k] = L[QS_DL_TORQUE_TO_THRUST] * tm;
        row[16 + 2 * k] = ((k == 0 || k == 3) ? 1. : -1.) * mx - com[0];
        row[17 + 2 * k] = (k < 2 ? -1. : 1.) * my - com[1];
        row[24 + k] = mz - com[2];
    }
    row[28] = 4 * dt / (L[QS_DL_DAMP_TIME_UP] + EPS);
    row[29] = 4 * dt / (L[QS_DL_DAMP_TIME_DOWN] + EPS);
    row[30] = L[QS_DL_LINEARITY];
    row[31] = 0.2 * L[QS_DL_THRUST_NOISE_RATIO];
    row[32] = L[QS_DL_C_DRAG]; row[33] = L[QS_DL_C_ROLL];
    row[34] = L[QS_DL_DAMP_VEL]; row[35] = L[QS_DL_DAMP_OMEGA_QUADRATIC];
    row[36] = sqrt(mx * mx + my * my);
    row[37] = 0.; row[38] = 0.; row[39] = 0.;
}

// DynamicsSource.sample() + derive_constants for drone i under `key` (the episode key of the env's episode that starts, or
// episode 0 for the construction sample); writes the float32 row to `out` (QS_DYN_ROW / 4 float4).  Called by the sampler's
// own kernels only (k_dyn_construct, qs_dyn_pregen_kernel), never by a step kernel.
__device__ __noinline__ void sample_dyn_row(const DynSampler* __restrict__ dyn, RngKey key, int i, float4* out) {
    const QsDynSampler* __restrict__ spec = &dyn->spec;
    double L[QS_DYN_LEAVES], L0[QS_DYN_LEAVES];
    uint8_t P[QS_DYN_LEAVES];
    DynDraws d;
    d.key = key; d.i = (uint32_t)i; d.k = 0u;
#pragma unroll 1
    for (int k = 0; k < QS_DYN_LEAVES; ++k) { L[k] = spec->params.value[k]; P[k] = spec->params.present[k]; }
    if (spec->base == QS_DYN_BASE_RANDOM_QUAD) {
        randomquad_leaves(L, d);
        check_limits(L, P, nullptr);
    }
#pragma unroll 1
    for (int k = 0; k < QS_DYN_LEAVES; ++k)
        if (spec->change.present[k]) L[k] = spec->change.value[k];
#pragma unroll 1
    for (int s = 0; s < 2; ++s) {
        const int kind = spec->sampler[s];
        const QsDynLeaves& q = spec->samp[s];
        if (kind == QS_DYN_SAMPLER_RELATIVE_NORMAL || kind == QS_DYN_SAMPLER_RELATIVE_UNIFORM) {
#pragma unroll 1
            for (int k = 0; k < QS_DYN_LEAVES; ++k) L0[k] = L[k];
#pragma unroll 1
            for (int o = 0; o < spec->n_order; ++o) {
                const int k = spec->order[o];
                const double v = L[k], ratio = q.value[k];
                L[k] = kind == QS_DYN_SAMPLER_RELATIVE_NORMAL ? d.normal(v, fabs((ratio / 2) * v))
                                                             : d.uniform(v - v * ratio, v + v * ratio);
            }
            check_limits(L, P, L0);
        } else if (kind == QS_DYN_SAMPLER_CONST) {
#pragma unroll 1
            for (int k = 0; k < QS_DYN_LEAVES; ++k)
                if (q.present[k]) L[k] = q.value[k];
        }
    }
    check_limits(L, P, nullptr);
    double row[QS_DYN_ROW];
    derive_row(L, P, row);
#pragma unroll 1
    for (int q = 0; q < QS_DYN_ROW / 4; ++q)
        out[q] = make_float4((float)row[4 * q], (float)row[4 * q + 1], (float)row[4 * q + 2], (float)row[4 * q + 3]);
}

}  // namespace qs
