/*
 * reset_dr_oracle.c -- TEST INFRASTRUCTURE: the CPU twin of the reset-mode DR events (wl_set_reset_events,
 * wl_reset_dr_kernel; DESIGN.md 6n) on top of the unchanged oracle.
 *
 * This translation unit compiles oracle/wl_oracle.c as it is, with its wlo_step, wlo_step_terms, wlo_reset and wlo_destroy
 * renamed, and exports those four names again: each calls the oracle's own function, then applies the redraw at the point
 * the library launches wl_reset_dr_kernel -- after a step to the envs it left at episode length 0, after a reset to its ids.
 * wlo_set_reset_events stores a handle's mask (the refusals of wl_set_reset_events).  Built by tests/reset_dr_oracle.py with
 * the oracle's own flags, so that it is bit-exact with the kernel in the fp32 build.
 */
#define wlo_step wlo_step_oracle
#define wlo_step_terms wlo_step_terms_oracle
#define wlo_reset wlo_reset_oracle
#define wlo_destroy wlo_destroy_oracle
#include "../oracle/wl_oracle.c"
#undef wlo_step
#undef wlo_step_terms
#undef wlo_reset
#undef wlo_destroy

#define RNG_RESET_DR 12u

/* the handles' masks (the oracle's handle has no field for it) */
#define MAX_HANDLES 1024
static struct { const wlo_sim* s; uint32_t mask; } g_masks[MAX_HANDLES];

static uint32_t mask_of(const wlo_sim* s) {
    for (int k = 0; k < MAX_HANDLES; ++k) if (g_masks[k].s == s) return g_masks[k].mask;
    return 0u;
}

/* wl_set_reset_events: the same refusals (WL_EINVAL, the mask unchanged) */
int wlo_set_reset_events(wlo_sim* s, uint32_t mask) {
    const wl_config* c = &s->cfg;
    const uint32_t all = WL_RESET_EV_MATERIAL | WL_RESET_EV_ACTUATOR_GAINS | WL_RESET_EV_BASE_MASS | WL_RESET_EV_WHEEL_MASS;
    if ((mask & ~all) || (mask && !c->dr_enable) || ((mask & WL_RESET_EV_ACTUATOR_GAINS) && c->dr_kd_mask == 0) ||
        ((mask & WL_RESET_EV_WHEEL_MASS) && !c->dr_wheel_mass_enable))
        return WL_EINVAL;
    int free_slot = -1;
    for (int k = 0; k < MAX_HANDLES; ++k) {
        if (g_masks[k].s == s) { g_masks[k].mask = mask; return 0; }
        if (!g_masks[k].s && free_slot < 0) free_slot = k;
    }
    if (free_slot < 0) return WL_EINVAL;
    g_masks[free_slot].s = s;
    g_masks[free_slot].mask = mask;
    return 0;
}

/* the DR parameters of one env from its four Philox blocks: r0 friction buckets, r1 actuator gains, r2 base mass, r3 wheel
 * masses -- wlo_startup's formulas (and wl_reset_dr_kernel's dr_params) */
static void dr_draw(const wl_config* c, wlo_env* e, const uint32_t r0[4], const uint32_t r1[4], const uint32_t r2[4], const uint32_t r3[4]) {
    for (int i = 0; i < 4; ++i) {
        uint32_t bk = 0;
        if (c->dr_enable && c->dr_num_buckets > 1) bk = (uint32_t)(((uint64_t)r0[i] * (uint64_t)c->dr_num_buckets) >> 32);
        e->D[i] = (real)c->dr_bucket_D[bk];
        e->C[i] = (real)c->dr_bucket_C[bk];
        e->kd[i] = (real)c->dc_damping[i];
        if (c->dr_enable && ((c->dr_kd_mask >> i) & 1)) e->kd[i] = uniform(r1[i], (real)c->dr_kd_range[0], (real)c->dr_kd_range[1]);
    }
    e->mass = (real)c->mass_nominal;
    for (int i = 0; i < 4; ++i) e->inv_Iw[i] = (real)c->d_inv_Iw;
    if (c->dr_enable) {
        real u = uniform(r2[0], (real)c->dr_mass_add[0], (real)c->dr_mass_add[1]);
        if (c->dr_mass_mode == 0) e->mass = e->mass + u;
        else e->mass = (e->mass - (real)c->dr_base_mass_nominal) + u;
        if (c->dr_wheel_mass_enable)
            for (int i = 0; i < 4; ++i) {
                real mw = uniform(r3[i], (real)c->dr_wheel_mass[0], (real)c->dr_wheel_mass[1]);
                e->mass = e->mass + (mw - (real)c->wheel_mass_nominal);
                e->inv_Iw[i] = (real)c->d_inv_Iw * ((real)c->wheel_mass_nominal / mw);
            }
    }
    e->inv_mass = K(1.0) / e->mass;
}

/* wl_reset_dr_kernel for env li reset by the call with counter t: block k from the reset key when event k is in reset mode,
 * else from the start-up key; only the named events' parameters are written */
static void reset_dr_env(wlo_sim* s, uint32_t m, int li, uint32_t t) {
    const wl_config* c = &s->cfg;
    const uint32_t gid = (uint32_t)(c->env_id_offset + li);
    uint32_t r[4][4];
    for (uint32_t k = 0; k < 4; ++k) {
        if ((m >> k) & 1u) philox4x32(c->seed, gid, t, RNG_RESET_DR, k, r[k]);
        else philox4x32(c->seed, gid, 0u, RNG_STARTUP, k, r[k]);
    }
    wlo_env* e = &s->env[li];
    wlo_env d = *e;
    dr_draw(c, &d, r[0], r[1], r[2], r[3]);
    if (m & WL_RESET_EV_MATERIAL) for (int i = 0; i < 4; ++i) { e->D[i] = d.D[i]; e->C[i] = d.C[i]; }
    if (m & WL_RESET_EV_ACTUATOR_GAINS) for (int i = 0; i < 4; ++i) e->kd[i] = d.kd[i];
    if (m & (WL_RESET_EV_BASE_MASS | WL_RESET_EV_WHEEL_MASS)) { e->mass = d.mass; e->inv_mass = d.inv_mass; e->spare0 = e->spare1 = K(0.0); }
    if (m & WL_RESET_EV_WHEEL_MASS) for (int i = 0; i < 4; ++i) e->inv_Iw[i] = d.inv_Iw[i];
}

static void redraw_after_step(wlo_sim* s, int64_t step_counter) {
    const uint32_t m = mask_of(s);
    if (!m) return;
    for (int li = 0; li < s->cfg.num_envs; ++li)
        if (s->env[li].ep_len == 0) reset_dr_env(s, m, li, (uint32_t)step_counter);
}

int wlo_step(wlo_sim* s, const float* action, float* obs, float* rew, uint8_t* terminated, uint8_t* truncated,
             int64_t step_counter, int nthreads) {
    int rc = wlo_step_oracle(s, action, obs, rew, terminated, truncated, step_counter, nthreads);
    redraw_after_step(s, step_counter);
    return rc;
}

int wlo_step_terms(wlo_sim* s, const float* action, float* obs, float* rew, uint8_t* terminated, uint8_t* truncated,
                   int64_t step_counter, int nthreads) {
    int rc = wlo_step_terms_oracle(s, action, obs, rew, terminated, truncated, step_counter, nthreads);
    redraw_after_step(s, step_counter);
    return rc;
}

int wlo_reset(wlo_sim* s, const int64_t* env_ids, int32_t n_ids, int64_t step_counter) {
    int rc = wlo_reset_oracle(s, env_ids, n_ids, step_counter);
    const uint32_t m = mask_of(s);
    const int n = env_ids ? n_ids : s->cfg.num_envs;
    if (m)
        for (int k = 0; k < n; ++k) reset_dr_env(s, m, env_ids ? (int)env_ids[k] : k, (uint32_t)step_counter);
    return rc;
}

void wlo_destroy(wlo_sim* s) {
    for (int k = 0; k < MAX_HANDLES; ++k) if (g_masks[k].s == s) { g_masks[k].s = NULL; g_masks[k].mask = 0u; }
    wlo_destroy_oracle(s);
}
