/*
 * policy_obs_oracle.c -- TEST INFRASTRUCTURE: the CPU twin of the policy observation table (wl_set_policy_terms,
 * wl_policy_observe_kernel; DESIGN.md 6q) on the unchanged oracle's generator, Box-Muller and rotations.
 *
 * For every env i and output column j: the library float src[j] of the state groups st [WL_NUM_GROUPS][n][4] (the
 * device state's layout), then, when corrupt, the column's additive noise keyed as the header documents, then the clip
 * (r_clamp), then the scale -- each fp32 operation in the kernel's order (no fma).  Built by tests/policy_obs_oracle.py
 * with the oracle's own flags (fp32, no contraction), so it is bit-exact with the kernel.
 */
#include "../oracle/wl_oracle.c"

#define RNG_POLICY_OBS 16u
#define POBS_NOISE_GAUSSIAN 1
#define POBS_NOISE_UNIFORM 2

/* the 32 library floats of env i: the critic library's 29 (root_pos_w, root_euler_xyz, base_lin_vel, base_ang_vel,
 * last_action, joint_vel, joint_pos, wheel_friction, base_mass, motor_damping) then projected_gravity */
static void pobs_library(const float* st, int32_t n, int i, float o[32]) {
    const float* g[WL_NUM_GROUPS];
    for (int k = 0; k < WL_NUM_GROUPS; ++k) g[k] = st + ((size_t)k * n + i) * 4;
    const real q[4] = {g[WL_G_QUAT][0], g[WL_G_QUAT][1], g[WL_G_QUAT][2], g[WL_G_QUAT][3]};
    real R[9], eu[3], vb[3], wb[3], gb[3];
    const real v[3] = {g[WL_G_LINVEL][0], g[WL_G_LINVEL][1], g[WL_G_LINVEL][2]};
    const real w[3] = {g[WL_G_ANGVEL][0], g[WL_G_ANGVEL][1], g[WL_G_ANGVEL][2]};
    const real down[3] = {0.0f, 0.0f, -1.0f};
    rotmat(q, R);
    euler_xyz(q, eu);
    rotT(R, v, vb);
    rotT(R, w, wb);
    rotT(R, down, gb);
    for (int k = 0; k < 3; ++k) {
        o[k] = g[WL_G_POS][k]; o[3 + k] = eu[k]; o[6 + k] = vb[k]; o[9 + k] = wb[k]; o[29 + k] = gb[k];
    }
    o[12] = g[WL_G_ACTION][0]; o[13] = g[WL_G_ACTION][1];
    for (int k = 0; k < 4; ++k) {
        o[14 + k] = g[WL_G_WHEEL][k]; o[20 + k] = g[WL_G_PMU_D][k]; o[25 + k] = g[WL_G_PKD][k];
    }
    o[18] = g[WL_G_STEER][0]; o[19] = g[WL_G_STEER][1];
    o[24] = g[WL_G_PMASS][0];
}

/* library [n][32] of every env, for the numpy restatement */
void wlo_policy_library(const float* st, int32_t n, float* out) {
    for (int i = 0; i < n; ++i) pobs_library(st, n, i, out + (size_t)i * 32);
}

/* the noise draw of column j: z ~ N(0, 1) (Gaussian) or u in [0, 1) (uniform), keyed as the header documents */
float wlo_policy_obs_draw(uint64_t seed, uint32_t gid, uint32_t t, int32_t call_idx, int32_t j, int32_t kind) {
    uint32_t r[4];
    if (kind == POBS_NOISE_GAUSSIAN && j < 12)
        philox4x32(seed, gid, t, call_idx < 0 ? RNG_OBS : RNG_OBS_EXTRA, (call_idx < 0 ? 0u : 3u * (uint32_t)call_idx) + (uint32_t)(j / 4), r);
    else
        philox4x32(seed, gid, t, RNG_POLICY_OBS, 16u * (uint32_t)(call_idx + 1) + (kind == POBS_NOISE_UNIFORM ? 8u : 0u) + (uint32_t)(j / 4), r);
    const int w = j % 4;
    if (kind == POBS_NOISE_UNIFORM) return u01(r[w]);
    float z0, z1;
    box_muller(r[w < 2 ? 0 : 2], r[w < 2 ? 1 : 3], &z0, &z1);
    return (w & 1) ? z1 : z0;
}

/* out [n][dp]; per column: src, noise (0 none, 1 Gaussian (na, nb) = (mean, std), 2 uniform (na, nb) = (n_min, n_max - n_min)),
 * clip flag with [lo, hi], scale flag with scale.  call_idx = -1: the row after the step at t; >= 0: an observe call. */
void wlo_policy_observe(uint64_t seed, int32_t env_id_offset, int32_t n, const float* st, int32_t dp, const uint8_t* src,
                        const uint8_t* noise, const float* na, const float* nb, const uint8_t* has_clip, const float* lo,
                        const float* hi, const uint8_t* has_scale, const float* scale, int32_t corrupt, uint32_t t,
                        int32_t call_idx, float* out) {
    for (int i = 0; i < n; ++i) {
        float lib[32];
        pobs_library(st, n, i, lib);
        const uint32_t gid = (uint32_t)(env_id_offset + i);
        for (int j = 0; j < dp; ++j) {
            float x = lib[src[j]];
            if (corrupt && noise[j]) {
                const float d = wlo_policy_obs_draw(seed, gid, t, call_idx, j, noise[j]);
                if (noise[j] == POBS_NOISE_GAUSSIAN) {
                    const float v = x + na[j];
                    const float s = nb[j] * d;
                    x = v + s;
                } else {
                    const float s = d * nb[j];
                    const float v = x + s;
                    x = v + na[j];
                }
            }
            if (has_clip[j]) x = r_clamp(x, lo[j], hi[j]);
            if (has_scale[j]) x = x * scale[j];
            out[(size_t)i * dp + j] = x;
        }
    }
}
