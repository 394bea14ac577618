// wl_reset_dr.cuh -- reset-mode domain randomisation (IsaacLab EventTermCfg mode="reset", DESIGN 6n), included by wl_api.cu
// ahead of wl_startup_kernel (decode_step, the state groups).
//
// The start-up events draw each env's friction buckets, motor damping and masses once.  wl_reset_dr_kernel draws them again
// for the envs a call reset, with the start-up formulas and a key of its own, and writes only the groups of the events the
// handle's mask names.  It is a launch of its own after the calls that reset envs: the step kernels are not touched.
#pragma once

#define WL_RESET_DR_BS 128

// The DR parameters of one env from its four Philox blocks (wl_startup_kernel's and wl_reset_dr_kernel's draw): r0 friction
// buckets, r1 actuator gains, r2 base mass, r3 wheel masses.  The total mass starts from the nominal mass every time (randomize_rigid_body_mass applies to the default mass):
// base term first, then the four wheel terms.
struct DrParams {
    float D[4], C[4], kd[4];
    float mass, inv_mass;
    float inv_Iw[4];
};
__device__ __forceinline__ void dr_params(const wl_config& c, uint4 r0, uint4 r1, uint4 r2, uint4 r3, DrParams& p) {
    const uint32_t rb[4] = {r0.x, r0.y, r0.z, r0.w}, rk[4] = {r1.x, r1.y, r1.z, r1.w}, rm[4] = {r3.x, r3.y, r3.z, r3.w};
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        uint32_t bk = 0;
        if (c.dr_enable && c.dr_num_buckets > 1) bk = __umulhi(rb[w], (uint32_t)c.dr_num_buckets);
        p.D[w] = c.dr_bucket_D[bk]; p.C[w] = c.dr_bucket_C[bk];
        p.kd[w] = c.dc_damping[w];
        if (c.dr_enable && ((c.dr_kd_mask >> w) & 1)) p.kd[w] = uniform(rk[w], c.dr_kd_range[0], c.dr_kd_range[1]);
    }
    // randomize_rigid_body_mass: "add" -> base_link mass += U; "abs" -> base_link mass := U (mushr_visual_env_cfg.py:280-288);
    // wheel links := U (:290-299), their spin inertia rescaled by the mass ratio
    float mass = c.mass_nominal;
    float inv_Iw[4] = {c.d_inv_Iw, c.d_inv_Iw, c.d_inv_Iw, c.d_inv_Iw};
    if (c.dr_enable) {
        const float u = uniform(r2.x, c.dr_mass_add[0], c.dr_mass_add[1]);
        if (c.dr_mass_mode == 0) mass = mass + u;
        else mass = (mass - c.dr_base_mass_nominal) + u;
        if (c.dr_wheel_mass_enable) {
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                const float mw = uniform(rm[w], c.dr_wheel_mass[0], c.dr_wheel_mass[1]);
                mass = mass + (mw - c.wheel_mass_nominal);
                inv_Iw[w] = c.d_inv_Iw * (c.wheel_mass_nominal / mw);
            }
        }
    }
    float inv_mass = 1.0f / mass;
    p.mass = mass; p.inv_mass = inv_mass;
#pragma unroll
    for (int w = 0; w < 4; ++w) p.inv_Iw[w] = inv_Iw[w];
}

// block k of env gid's draw: the reset key (counter t, stream RNG_RESET_DR) when event k is in reset mode, else the start-up
// key, so that a start-up-mode component is recomputed to its start-up value
__device__ __forceinline__ uint4 dr_block(const wl_config& c, uint32_t gid, uint32_t t, uint32_t mask, uint32_t k) {
    return ((mask >> k) & 1u) ? philox4x32(c.seed, gid, t, RNG_RESET_DR, k) : philox4x32(c.seed, gid, 0u, RNG_STARTUP, k);
}

// One thread per env (after_step) or per listed id (after wl_reset; ids == null: every env).  After a step the envs it reset
// are those whose episode_length_buf it left at 0 (every step kernel counts an env up by one, then a reset sets it to 0), and
// t is that step's counter, decoded as the step decoded it; after wl_reset t is wl_reset's counter as wl_reset_kernel uses it.
// Launched without the PDL attribute and without an early trigger: it starts once the step has finished, and a step launched
// after it with PDL starts only when it has completed (a chained duo step, which skips its griddepcontrol.wait, included:
// DESIGN.md 6e).
__global__ void __launch_bounds__(WL_RESET_DR_BS)
wl_reset_dr_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, const wl_globals* __restrict__ gl,
                   const int64_t* __restrict__ ids, int n_ids, uint32_t t_arg, bool after_step, uint32_t mask) {
    const int n = c.num_envs;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_ids) return;
    const int i = ids ? (int)ids[k] : k;
    if (i < 0 || i >= n) return;
    if (after_step && __float_as_int(ldg4(st, WL_G_POS, n, i).w) != 0) return;
    const uint32_t t = after_step ? decode_step(gl, t_arg) : t_arg;
    const uint32_t gid = (uint32_t)(c.env_id_offset + i);
    const bool material = mask & WL_RESET_EV_MATERIAL, gains = mask & WL_RESET_EV_ACTUATOR_GAINS;
    const bool mass = mask & (WL_RESET_EV_BASE_MASS | WL_RESET_EV_WHEEL_MASS);
    const uint4 z = make_uint4(0u, 0u, 0u, 0u);
    const uint4 r0 = material ? dr_block(c, gid, t, mask, 0u) : z;
    const uint4 r1 = gains ? dr_block(c, gid, t, mask, 1u) : z;
    const uint4 r2 = mass ? dr_block(c, gid, t, mask, 2u) : z;
    const uint4 r3 = (mass && c.dr_wheel_mass_enable) ? dr_block(c, gid, t, mask, 3u) : z;
    DrParams p;
    dr_params(c, r0, r1, r2, r3, p);
    if (material) {
        stg4(st, WL_G_PMU_D, n, i, make_float4(p.D[0], p.D[1], p.D[2], p.D[3]));
        stg4(st, WL_G_PMU_C, n, i, make_float4(p.C[0], p.C[1], p.C[2], p.C[3]));
    }
    if (gains) stg4(st, WL_G_PKD, n, i, make_float4(p.kd[0], p.kd[1], p.kd[2], p.kd[3]));
    if (mass) stg4(st, WL_G_PMASS, n, i, make_float4(p.mass, p.inv_mass, 0.0f, 0.0f));
    if (mask & WL_RESET_EV_WHEEL_MASS) stg4(st, WL_G_PIW, n, i, make_float4(p.inv_Iw[0], p.inv_Iw[1], p.inv_Iw[2], p.inv_Iw[3]));
}
