/*
 * row_terms_oracle.c -- TEST INFRASTRUCTURE: the CPU twin of the row terms on the Elevation / Visual rows
 * (wl_set_row_terms, wl_scan_row_kernel, wl_visual_row_kernel; DESIGN.md 6r), on the unchanged oracle's ray arithmetic,
 * generator, Box-Muller and rotations.  Built by tests/row_terms_oracle.py with the oracle's own flags (fp32, no
 * contraction), so it is bit-exact with the kernels; the library also carries the whole oracle (wlo_create, wlo_step, ...).
 */
#include "../oracle/wl_oracle.c"

#define RNG_ROW_TERMS 17u

/* the raw columns of env li: Elevation 689 (elev_obs's values without its clips; a ray that misses is +inf), Visual the 8
 * tail floats (visual_obs's without the last action's clip) */
static void row_raw(const wlo_sim* s, const wlo_env* e, float* o) {
    const wl_config* c = &s->cfg;
    real R[9]; rotmat(e->q, R);
    real vb[3], wb[3]; rotT(R, e->v, vb); rotT(R, e->w, wb);
    if (c->task == WL_TASK_VISUAL) {
        for (int k = 0; k < 3; ++k) { o[k] = (float)vb[k]; o[3 + k] = (float)wb[k]; }
        o[6] = (float)e->action[0]; o[7] = (float)e->action[1];
        return;
    }
    real eu[3]; euler_xyz(e->q, eu);
    real gx = e->cmdb[0] - e->p[0], gy = e->cmdb[1] - e->p[1];
    o[0] = (float)((gx != gx) ? K(0.0) : gx); o[1] = (float)((gy != gy) ? K(0.0) : gy);
    for (int k = 0; k < 3; ++k) { o[2 + k] = (float)eu[k]; o[5 + k] = (float)vb[k]; o[8 + k] = (float)wb[k]; }
    o[11] = (float)e->action[0]; o[12] = (float)e->action[1];
    real bx = fm((real)c->base_link_z, R[2], e->p[0]), by = fm((real)c->base_link_z, R[5], e->p[1]), bz = fm((real)c->base_link_z, R[8], e->p[2]);
    real cy, sy; yaw_cs(e, &cy, &sy);
    for (int k = 0; k < WL_SCAN_RAYS; ++k) {
        int rx = k % WL_SCAN_SIDE, ry = k / WL_SCAN_SIDE;
        real lx = fm((real)rx, (real)c->scan_res, -(real)c->scan_half), ly = fm((real)ry, (real)c->scan_res, -(real)c->scan_half);
        real wx = fm(cy, lx, fm(-sy, ly, bx)), wy = fm(sy, lx, fm(cy, ly, by));
        real hit, gxx, gyy;
        if (hf_sample(s, wx, wy, &hit, &gxx, &gyy)) {
            real hs = bz - hit - (real)c->scan_offset;
            o[13 + k] = (float)(-hs + (e->p[2] - (real)c->scan_plane_init));
        } else {
            o[13 + k] = INFINITY;
        }
    }
}
/* the noise draw of row column j: z ~ N(0, 1) (WL_NOISE_GAUSSIAN) or u in [0, 1) (WL_NOISE_UNIFORM), keyed as the header
 * documents */
float wlo_row_draw(uint64_t seed, uint32_t gid, uint32_t t, int32_t call_idx, int32_t j, int32_t kind) {
    uint32_t r[4];
    philox4x32(seed, gid, t, RNG_ROW_TERMS, 512u * (uint32_t)(call_idx + 1) + (kind == WL_NOISE_UNIFORM ? 256u : 0u) + (uint32_t)(j / 4), r);
    const int w = j % 4;
    if (kind == WL_NOISE_UNIFORM) return (float)u01(r[w]);
    real z0, z1;
    box_muller(r[w < 2 ? 0 : 2], r[w < 2 ? 1 : 3], &z0, &z1);
    return (float)((w & 1) ? z1 : z0);
}
/* raw [N][689] (Elevation) or [N][8] (Visual) of the oracle's current state */
int wlo_row_raw(const wlo_sim* s, float* raw) {
    const int w = s->cfg.task == WL_TASK_VISUAL ? 8 : WL_OBS_DIM_ELEV;
    for (int li = 0; li < s->cfg.num_envs; ++li) row_raw(s, &s->env[li], raw + (size_t)w * li);
    return 0;
}
/* The row of every env under the row terms `terms` (the wl_set_row_terms table, n_terms = the task's count): the raw column,
 * then the term's noise (only with the config's enable_corruption), clip and scale, each one fp32 operation in
 * ObservationManager.compute's order, with the parameters rounded as wl_set_row_terms rounds them.  obs is [N][row floats]
 * of the task (Visual: the camera floats are left as they are).  call_idx -1: the row of the step at step_counter. */
int wlo_row_observe(wlo_sim* s, const wl_policy_term* terms, int32_t n_terms, int64_t step_counter, int32_t call_idx, float* obs) {
    const wl_config* c = &s->cfg;
    const int vis = c->task == WL_TASK_VISUAL, w = vis ? 8 : WL_OBS_DIM_ELEV;
    const int camf = vis ? vis_cam_floats(c) : 0, stride = vis ? WL_OBS_DIM_VISUAL + camf : WL_OBS_DIM_ELEV;
    int term_of[WL_OBS_DIM_ELEV], first[8];
    for (int k = 0, j = 0; k < n_terms; ++k) {
        const int width = terms[k].kind == WL_ROW_WORLD_HEIGHT_MAP ? WL_SCAN_RAYS : terms[k].kind == WL_ROW_GOAL_RELATIVE_XYZ ? 2 :
                          (terms[k].kind == WL_CRITIC_LAST_ACTION ? 2 : 3);
        first[k] = j;
        for (int q = 0; q < width && j < w; ++q) term_of[j++] = k;
    }
    float* raw = (float*)malloc(sizeof(float) * w);
    for (int li = 0; li < c->num_envs; ++li) {
        row_raw(s, &s->env[li], raw);
        float* row = obs + (size_t)stride * li + camf;
        for (int j = 0; j < w; ++j) {
            const wl_policy_term* d = &terms[term_of[j]];
            float x = raw[j];
            if (c->enable_corruption && d->noise != WL_NOISE_NONE) {
                const float na = (float)d->noise_params[0];
                const float nb = d->noise == WL_NOISE_UNIFORM ? (float)(d->noise_params[1] - d->noise_params[0]) : (float)d->noise_params[1];
                const float z = wlo_row_draw(c->seed, (uint32_t)(c->env_id_offset + li), (uint32_t)step_counter, call_idx, j, d->noise);
                if (d->noise == WL_NOISE_GAUSSIAN) {
                    const float v = x + na;
                    const float e = nb * z;
                    x = v + e;
                } else {
                    const float e = z * nb;
                    const float v = x + e;
                    x = v + na;
                }
            }
            if (d->clip) x = (float)r_clamp(x, (float)d->clip_range[0], (float)d->clip_range[1]);
            if (d->n_scale) x = x * (float)d->scale[d->n_scale == 1 ? 0 : j - first[term_of[j]]];
            row[j] = x;
        }
    }
    free(raw);
    return 0;
}

