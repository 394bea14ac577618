// wl_terms.cuh -- device terms: the reward / termination functions that the reference's task files define but do not
// register (elevation/mushr_elevation_env_cfg.py, visual/mushr_visual_env_cfg.py), evaluated on the device between
// the two halves of the staged step (wl_step_terms, DESIGN.md 6l).
//
// Semantics = the reference's function registered as a Python term through env.staged_step: terminations first
// (a termination fires when its value is nonzero), then rewards in registration order, each adding
// fp32(f) * fp32(weight * step_dt) to the step reward and to the term's per-episode sum (weight 0: skipped, not
// evaluated).  Every operation is fp32, in the order the torch expression evaluates it; Python scalars enter as the
// fp32 constants torch converts them to (the host folds each term's parameters into those constants,
// wl_set_device_terms).  One thread per env, no float atomics: the episode-log entries are reduced in a fixed tree
// order (wl_terms_kernel per CTA, wl_terms_log_kernel over the CTAs), so results are bit-identical run to run.
#pragma once
#include "wl_step.cuh"

namespace wl {

// the kernel's copy of the term table (wl_set_device_terms fills it; passed by value as a __grid_constant__)
struct TermTable {
    int32_t n;
    int32_t kind[WL_MAX_DEVICE_TERMS];
    int32_t role[WL_MAX_DEVICE_TERMS];
    float scale[WL_MAX_DEVICE_TERMS];      // reward: fp32(weight * step_dt)
    int32_t skip[WL_MAX_DEVICE_TERMS];     // a reward term of weight 0: not evaluated
    float p[WL_MAX_DEVICE_TERMS][4];       // the parameters as the fp32 constants the torch expression uses
};
// per-env buffers of the device terms (one allocation per handle, see wl_set_device_terms)
struct TermBufs {
    float* sums;              // [WL_MAX_DEVICE_TERMS][N] per-episode sums of the reward terms
    float* prev;              // [N] elevation_continuity's previous elevation (NaN: not called yet)
    uint8_t* extra_term;      // [N] a termination term fired
    uint8_t* extra_to;        // [N] a time-out term fired
    uint8_t* fired;           // [N] bit k: term k fired (TerminationManager.get_term)
    float* part;              // [CTAs][16] per-CTA partial sums of the episode-log entries
};

#define WL_TERMS_BS 128

// TraversabilityHashmapUtil.get_traversability at the root (x, y): the lookup visual_terms makes (quirk Q14)
__device__ __forceinline__ bool term_traversable(const wl_config& c, const VisualMap& vm, float x, float y) {
    int xi = (int)((x + c.vis_width / 2.0f + c.vis_row_spacing / 2.0f) / c.vis_row_spacing);
    int yi = (int)((y + c.vis_height / 2.0f + c.vis_col_spacing / 2.0f) / c.vis_col_spacing);
    xi = xi < 0 ? 0 : (xi > c.vis_rows - 1 ? c.vis_rows - 1 : xi);
    yi = yi < 0 ? 0 : (yi > c.vis_cols - 1 ? c.vis_cols - 1 : yi);
    return __ldg(vm.map + (size_t)yi * c.vis_cols + xi) != 0;
}

// The pre-reset quantities the terms read, formed once per env
struct TermIn {
    V3 p, vw, vb, wb;            // root_pos_w, root_lin_vel_w, base_lin_vel, base_ang_vel
    float qw, qx, qy, qz;
    float spin;                  // sum of the 4 throttle joint velocities
};

// value of term `kind` with parameters p; `prev` is elevation_continuity's state (updated in place)
__device__ __forceinline__ float term_value(const wl_config& c, const VisualMap& vm, int kind, const float p[4], const TermIn& s,
                                            uint32_t t, float& prev) {
    switch (kind) {
    case WL_TERM_E_FORWARD_VEL: return r_min(s.vb.x, 1.2f);                                   // clamp(v_b.x, max=1.2)
    case WL_TERM_E_FORWARD_WHEEL_SPIN: return r_min(s.spin, 200.0f);                          // clamp(sum, max=200)
    case WL_TERM_E_CHANGE_IN_ELEVATION: return (s.vw.z > 0.0f) ? s.vw.z : 0.0f;
    case WL_TERM_E_ASCENDING: return r_max(s.vw.z, 0.0f);
    case WL_TERM_E_STEEP_PENALTY: {
        // pitch as euler_xyz_from_quat returns it, wrapped to [0, 2 pi): a nose-down car has a pitch near 2 pi (the quirk)
        const float pitch = euler_xyz(s.qw, s.qx, s.qy, s.qz).y;
        return r_max(pitch - p[0], 0.0f);
    }
    case WL_TERM_E_ELEVATION_CONTINUITY: {
        const float z = s.p.z - 0.19f;
        const float d = z - ((prev != prev) ? z : prev);            // first call: prev = z
        prev = z;
        return (z > p[0] && d != 0.0f) ? fabsf(50.0f * d) : 0.0f;
    }
    case WL_TERM_E_YAW_CHANGE_ON_ELEV: {
        const float z = s.p.z - 0.19f, a = fabsf(s.wb.z);
        return (z > p[1] && a > p[0]) ? 2.0f * (a * a) : 0.0f;
    }
    case WL_TERM_E_UPRIGHT_PENALTY: {
        // matrix_from_quat's R22 (normalised by |q|^2), arccos in degrees; arccos of |x| > 1 is NaN -> 0 (torch.where)
        const float two_s = 2.0f / (((s.qw * s.qw + s.qx * s.qx) + s.qy * s.qy) + s.qz * s.qz);
        const float r22 = 1.0f - two_s * (s.qx * s.qx + s.qy * s.qy);
        if (!(fabsf(r22) <= 1.0f)) return 0.0f;
        const float deg = det_atan2(sqrtf((1.0f - r22) * (1.0f + r22)), r22) * 57.29577951308232f;
        return (deg > p[0]) ? deg - p[0] : 0.0f;
    }
    case WL_TERM_E_ROLL_ON_ELEV: {
        const float z = s.p.z - 0.19f, a = fabsf(s.wb.x);
        return (z > p[0] && a > p[1]) ? a * 2.0f : 0.0f;
    }
    case WL_TERM_E_LOW_VEL_PENALTY: return (s.vb.x < p[0]) ? 1.0f : 0.0f;
    case WL_TERM_V_IS_TRAVERSABLE: return term_traversable(c, vm, s.p.x, s.p.y) ? 1.0f : 0.0f;
    case WL_TERM_V_IS_TRAVERSABLE_SPEED_SCALED: return (term_traversable(c, vm, s.p.x, s.p.y) ? 1.0f : 0.0f) * s.vb.x;
    case WL_TERM_V_VEL_REW_TRAV: {
        const float target = term_traversable(c, vm, s.p.x, s.p.y) ? p[0] : p[1];
        const float sp = sqrtf((s.vb.x * s.vb.x + s.vb.y * s.vb.y) + s.vb.z * s.vb.z);
        const float d = sp - target;
        const float sd = -(d * d) + target * target;
        return (sd > 0.0f) ? sd : 0.0f;
    }
    case WL_TERM_V_LOW_SPEED_PENALTY: {
        const float sp = sqrtf((s.vb.x * s.vb.x + s.vb.y * s.vb.y) + s.vb.z * s.vb.z);
        return (sp < p[0]) ? 1.0f : 0.0f;
    }
    case WL_TERM_V_OFF_TRACK: {       // p = straight, corner_out_radius, corner_out_radius**2 (squared in double, as Python does)
        const float x = s.p.x, y = s.p.y;
        bool out;
        if (fabsf(y) < p[0]) out = fabsf(x) > p[1];
        else if (y > 0.0f) { const float a = y - p[0]; out = a * a + x * x > p[2]; }
        else { const float a = y + p[0]; out = a * a + x * x > p[2]; }
        return out ? 1.0f : 0.0f;
    }
    case WL_TERM_V_BOOL_IS_NOT_TRAVERSABLE:
        // common_step_counter // max_episode_length < 1000: the counter the step runs at (host or device counter)
        if (t / (uint32_t)c.max_episode_length < 1000u) return 0.0f;
        return term_traversable(c, vm, s.p.x, s.p.y) ? 0.0f : 1.0f;
    case WL_TERM_V_ROLL_OVER: {
        const float roll = euler_xyz(s.qw, s.qx, s.qy, s.qz).x - 3.14159265358979323846f;
        return (roll < 1.57079632679489661923f && roll > -1.57079632679489661923f) ? 1.0f : 0.0f;
    }
    default: return 0.0f;
    }
}

// One thread per env, between stage a (which left the pre-reset state and the built-in reward / bits) and stage b.
// Adds the reward terms to d_rew, raises the extra termination / time-out bytes stage b reads, keeps the per-episode
// sums (zeroed for the envs done in this step) and, with `part`, writes the CTA's partial log sums: [k] the done envs'
// episode sums (reward term k) or fired count (termination term k), [8] the done count.
__global__ void __launch_bounds__(WL_TERMS_BS)
wl_terms_kernel(const __grid_constant__ TermTable tt, const __grid_constant__ wl_config c, const float4* __restrict__ st,
                const wl_globals* __restrict__ gl, const float* __restrict__ aux, uint32_t t_arg, float* __restrict__ rew,
                const uint8_t* __restrict__ tbits, TermBufs b, bool with_log) {
    __shared__ float red[9][WL_TERMS_BS];
    const int n = c.num_envs;
    const int i = blockIdx.x * WL_TERMS_BS + threadIdx.x;
    const uint32_t t = decode_step(gl, t_arg);
    const VisualMap vm = (c.task == WL_TASK_VISUAL) ? visual_map(c, aux) : VisualMap{nullptr, nullptr};
    float contrib[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) contrib[k] = 0.0f;
    if (i < n) {
        TermIn s;
        float4 g = ldg4(st, WL_G_POS, n, i); s.p = V3{g.x, g.y, g.z};
        g = ldg4(st, WL_G_QUAT, n, i); s.qw = g.x; s.qx = g.y; s.qy = g.z; s.qz = g.w;
        g = ldg4(st, WL_G_LINVEL, n, i); s.vw = V3{g.x, g.y, g.z};
        g = ldg4(st, WL_G_ANGVEL, n, i); const V3 ww{g.x, g.y, g.z};
        g = ldg4(st, WL_G_WHEEL, n, i); s.spin = (g.x + g.y) + (g.z + g.w);
        const M3 R = rotmat(s.qw, s.qx, s.qy, s.qz);
        s.vb = rotT(R, s.vw); s.wb = rotT(R, ww);
        float prev = b.prev[i];
        // terminations first (TerminationManager.compute runs before RewardManager.compute)
        uint32_t fired = 0u;
        bool x_term = false, x_to = false;
#pragma unroll
        for (int k = 0; k < WL_MAX_DEVICE_TERMS; ++k) {
            if (k >= tt.n || tt.role[k] == WL_TERM_ROLE_REWARD) continue;
            if (term_value(c, vm, tt.kind[k], tt.p[k], s, t, prev) != 0.0f) {
                fired |= 1u << k;
                if (tt.role[k] == WL_TERM_ROLE_TIME_OUT) x_to = true; else x_term = true;
            }
        }
        float r = rew[i];
        float sums[WL_MAX_DEVICE_TERMS];
#pragma unroll
        for (int k = 0; k < WL_MAX_DEVICE_TERMS; ++k) {
            sums[k] = 0.0f;
            if (k >= tt.n || tt.role[k] != WL_TERM_ROLE_REWARD || tt.skip[k]) continue;
            const float val = term_value(c, vm, tt.kind[k], tt.p[k], s, t, prev) * tt.scale[k];
            r += val;
            sums[k] = b.sums[(size_t)k * n + i] + val;
        }
        rew[i] = r;
        b.prev[i] = prev;
        b.extra_term[i] = x_term ? 1 : 0;
        b.extra_to[i] = x_to ? 1 : 0;
        b.fired[i] = (uint8_t)fired;
        const bool done = (tbits[i] != 0) || x_term || x_to;
#pragma unroll
        for (int k = 0; k < WL_MAX_DEVICE_TERMS; ++k) {
            if (k >= tt.n) continue;
            if (tt.role[k] != WL_TERM_ROLE_REWARD) { contrib[k] = (done && ((fired >> k) & 1u)) ? 1.0f : 0.0f; continue; }
            if (tt.skip[k]) continue;
            contrib[k] = done ? sums[k] : 0.0f;
            b.sums[(size_t)k * n + i] = done ? 0.0f : sums[k];
        }
        contrib[8] = done ? 1.0f : 0.0f;
    }
    if (!with_log) return;
    // fixed-order tree over the CTA's 128 envs
#pragma unroll
    for (int k = 0; k < 9; ++k) red[k][threadIdx.x] = contrib[k];
    __syncthreads();
    for (int h = WL_TERMS_BS / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) {
#pragma unroll
            for (int k = 0; k < 9; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + h];
        }
        __syncthreads();
    }
    if (threadIdx.x < 9) b.part[(size_t)blockIdx.x * 16 + threadIdx.x] = red[threadIdx.x][0];
}

// The device terms' Episode_* entries of the step from the per-CTA partials: warp k sums column k over the CTAs
// (lane-strided, then a butterfly: a fixed order).  Reward term: sum / max(count, 1) / max_episode_length_s
// (RewardManager.reset); termination term: the count of done envs where it fired.
__global__ void __launch_bounds__(9 * 32)
wl_terms_log_kernel(const __grid_constant__ TermTable tt, const __grid_constant__ wl_config c, const float* __restrict__ part,
                    int ctas, float* __restrict__ term_log) {
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float v = 0.0f;
    for (int g = lane; g < ctas; g += 32) v += part[(size_t)g * 16 + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __shared__ float col[9];
    if (lane == 0) col[k] = v;
    __syncthreads();
    if (threadIdx.x < tt.n) {
        const int j = threadIdx.x;
        term_log[j] = (tt.role[j] == WL_TERM_ROLE_REWARD) ? col[j] / r_max(col[8], 1.0f) / c.episode_length_s : col[j];
    }
    if (threadIdx.x >= tt.n && threadIdx.x < WL_MAX_DEVICE_TERMS) term_log[threadIdx.x] = 0.0f;
}

}   // namespace wl
