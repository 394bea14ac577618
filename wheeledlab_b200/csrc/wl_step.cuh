// wl_step.cuh -- the per-env fused step: action map -> DC-motor / PD actuators ->
// chassis + 4-wheel integrator with Pacejka-style slip forces -> terminations ->
// rewards -> auto-reset -> interval pushes -> observations (+ Gaussian noise).
// One env's whole step lives in registers; HBM is touched once per group on the way in
// and once on the way out (DESIGN.md "Kernels").
//
// Reference behaviour restated here (file:line under the reference's source/ directory):
//   action term     wheeledlab/wheeledlab/envs/mdp/actions/ackermann_actions.py:119-145,150-201
//                   wheeledlab/wheeledlab/envs/mdp/actions/rc_car_actions.py:12-29,36-64
//   actuators       wheeledlab_assets/wheeledlab_assets/hound.py:4-52
//   terminations    wheeledlab_tasks/wheeledlab_tasks/drifting/mushr_drift_env_cfg.py:201-217,343-362
//   rewards         .../drifting/mushr_drift_env_cfg.py:160-299
//   reset           .../drifting/mdp/events.py:102-133
//   pushes          .../drifting/mushr_drift_env_cfg.py:121-143
//   observations    wheeledlab_tasks/wheeledlab_tasks/common/observations.py:19-56
#pragma once
#include "wl_device.cuh"

namespace wl {

struct EnvState {
    V3 p; float qw, qx, qy, qz; V3 v; V3 w;
    float omega[4]; float steer[2], steer_vel[2];
    float action[2], prev_action[2];
    int ep_len; float t_hf, t_lf;
    float sums[WL_MAX_REW_TERMS];
    float mass, inv_mass, spare0, spare1;
    float D[4], C[4], kd[4];
    float inv_Iw[4];  // 1 / wheel spin inertia (read from WL_G_PIW only when the wheel-mass DR is on)
    float cmd[4];     // elevation: goal x,y (world), heading_w, command time_left
    float cmdb[4];    // elevation: command in the yaw frame x,y, heading_b, spare
};

__device__ __forceinline__ void load_env(const float4* __restrict__ st, int n, int i, EnvState& e, bool with_cmd, bool with_iw = false,
                                         float inv_Iw_nominal = 0.0f) {
    float4 g;
    if (with_iw) { g = ldg4(st, WL_G_PIW, n, i); e.inv_Iw[0] = g.x; e.inv_Iw[1] = g.y; e.inv_Iw[2] = g.z; e.inv_Iw[3] = g.w; }
    else { e.inv_Iw[0] = e.inv_Iw[1] = e.inv_Iw[2] = e.inv_Iw[3] = inv_Iw_nominal; }
    g = ldg4(st, WL_G_POS, n, i); e.p = V3{g.x, g.y, g.z}; e.ep_len = __float_as_int(g.w);
    g = ldg4(st, WL_G_QUAT, n, i); e.qw = g.x; e.qx = g.y; e.qy = g.z; e.qz = g.w;
    g = ldg4(st, WL_G_LINVEL, n, i); e.v = V3{g.x, g.y, g.z}; e.t_hf = g.w;
    g = ldg4(st, WL_G_ANGVEL, n, i); e.w = V3{g.x, g.y, g.z}; e.t_lf = g.w;
    g = ldg4(st, WL_G_WHEEL, n, i); e.omega[0] = g.x; e.omega[1] = g.y; e.omega[2] = g.z; e.omega[3] = g.w;
    g = ldg4(st, WL_G_STEER, n, i); e.steer[0] = g.x; e.steer[1] = g.y; e.steer_vel[0] = g.z; e.steer_vel[1] = g.w;
    g = ldg4(st, WL_G_ACTION, n, i); e.action[0] = g.x; e.action[1] = g.y; e.prev_action[0] = g.z; e.prev_action[1] = g.w;
    g = ldg4(st, WL_G_SUM0, n, i); e.sums[0] = g.x; e.sums[1] = g.y; e.sums[2] = g.z; e.sums[3] = g.w;
    g = ldg4(st, WL_G_SUM1, n, i); e.sums[4] = g.x; e.sums[5] = g.y; e.sums[6] = g.z; e.sums[7] = g.w;
    g = ldg4(st, WL_G_PMASS, n, i); e.mass = g.x; e.inv_mass = g.y; e.spare0 = g.z; e.spare1 = g.w;
    g = ldg4(st, WL_G_PMU_D, n, i); e.D[0] = g.x; e.D[1] = g.y; e.D[2] = g.z; e.D[3] = g.w;
    g = ldg4(st, WL_G_PMU_C, n, i); e.C[0] = g.x; e.C[1] = g.y; e.C[2] = g.z; e.C[3] = g.w;
    g = ldg4(st, WL_G_PKD, n, i); e.kd[0] = g.x; e.kd[1] = g.y; e.kd[2] = g.z; e.kd[3] = g.w;
    if (with_cmd) {
        g = ldg4(st, WL_G_CMD, n, i); e.cmd[0] = g.x; e.cmd[1] = g.y; e.cmd[2] = g.z; e.cmd[3] = g.w;
        g = ldg4(st, WL_G_CMDB, n, i); e.cmdb[0] = g.x; e.cmdb[1] = g.y; e.cmdb[2] = g.z; e.cmdb[3] = g.w;
    }
}
// dynamic state only (params are read-only in the step)
__device__ __forceinline__ void store_env(float4* __restrict__ st, int n, int i, const EnvState& e, bool with_cmd) {
    stg4(st, WL_G_POS, n, i, make_float4(e.p.x, e.p.y, e.p.z, __int_as_float(e.ep_len)));
    stg4(st, WL_G_QUAT, n, i, make_float4(e.qw, e.qx, e.qy, e.qz));
    stg4(st, WL_G_LINVEL, n, i, make_float4(e.v.x, e.v.y, e.v.z, e.t_hf));
    stg4(st, WL_G_ANGVEL, n, i, make_float4(e.w.x, e.w.y, e.w.z, e.t_lf));
    stg4(st, WL_G_WHEEL, n, i, make_float4(e.omega[0], e.omega[1], e.omega[2], e.omega[3]));
    stg4(st, WL_G_STEER, n, i, make_float4(e.steer[0], e.steer[1], e.steer_vel[0], e.steer_vel[1]));
    stg4(st, WL_G_ACTION, n, i, make_float4(e.action[0], e.action[1], e.prev_action[0], e.prev_action[1]));
    stg4(st, WL_G_SUM0, n, i, make_float4(e.sums[0], e.sums[1], e.sums[2], e.sums[3]));
    stg4(st, WL_G_SUM1, n, i, make_float4(e.sums[4], e.sums[5], e.sums[6], e.sums[7]));
    if (with_cmd) {
        stg4(st, WL_G_CMD, n, i, make_float4(e.cmd[0], e.cmd[1], e.cmd[2], e.cmd[3]));
        stg4(st, WL_G_CMDB, n, i, make_float4(e.cmdb[0], e.cmdb[1], e.cmdb[2], e.cmdb[3]));
    }
}

// ---- quad (4 lanes per env) state access: lane w = wheel [bl,br,fl,fr][w].  Per-wheel scalars live in slot [0]
// of the lane's EnvState (omega, D, C, kd) and front lanes keep THEIR steer joint in steer[0]/steer_vel[0].
// Two phases: quad_issue_loads() puts every load in flight into a register block and quad_unpack() consumes it -- whatever is
// written between the two calls (the observation noise) executes under the shadow of the loads.
struct QuadRaw { float4 pos, quat, linvel, angvel, action, sum0, sum1, pmass, steer, cmd, cmdb; float omega, D, C, kd, inv_Iw; };
__device__ __forceinline__ void quad_issue_loads(const float4* __restrict__ st, int n, int i, int w, QuadRaw& r, bool with_cmd, bool with_iw,
                                                 bool with_sums = true) {
    r.pos = ldg4(st, WL_G_POS, n, i); r.quat = ldg4(st, WL_G_QUAT, n, i);
    r.linvel = ldg4(st, WL_G_LINVEL, n, i); r.angvel = ldg4(st, WL_G_ANGVEL, n, i);
    r.action = ldg4(st, WL_G_ACTION, n, i);
    if (with_sums) { r.sum0 = ldg4(st, WL_G_SUM0, n, i); r.sum1 = ldg4(st, WL_G_SUM1, n, i); }
    else { r.sum0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f); r.sum1 = r.sum0; }
    r.pmass = ldg4(st, WL_G_PMASS, n, i); r.steer = ldg4(st, WL_G_STEER, n, i);
    const float* f = reinterpret_cast<const float*>(st);
    const size_t lane_off = (size_t)i * 4 + w;                       // 32 lanes -> 128 contiguous bytes
    r.omega = f[(size_t)WL_G_WHEEL * n * 4 + lane_off];
    r.D = f[(size_t)WL_G_PMU_D * n * 4 + lane_off];
    r.C = f[(size_t)WL_G_PMU_C * n * 4 + lane_off];
    r.kd = f[(size_t)WL_G_PKD * n * 4 + lane_off];
    r.inv_Iw = with_iw ? f[(size_t)WL_G_PIW * n * 4 + lane_off] : 0.0f;
    if (with_cmd) { r.cmd = ldg4(st, WL_G_CMD, n, i); r.cmdb = ldg4(st, WL_G_CMDB, n, i); }
}
__device__ __forceinline__ void quad_unpack(const QuadRaw& r, int w, EnvState& e, bool with_cmd, bool with_iw, float inv_Iw_nominal) {
    float4 g;
    e.inv_Iw[0] = with_iw ? r.inv_Iw : inv_Iw_nominal;
    g = r.pos; e.p = V3{g.x, g.y, g.z}; e.ep_len = __float_as_int(g.w);
    g = r.quat; e.qw = g.x; e.qx = g.y; e.qy = g.z; e.qz = g.w;
    g = r.linvel; e.v = V3{g.x, g.y, g.z}; e.t_hf = g.w;
    g = r.angvel; e.w = V3{g.x, g.y, g.z}; e.t_lf = g.w;
    g = r.action; e.action[0] = g.x; e.action[1] = g.y; e.prev_action[0] = g.z; e.prev_action[1] = g.w;
    g = r.sum0; e.sums[0] = g.x; e.sums[1] = g.y; e.sums[2] = g.z; e.sums[3] = g.w;
    g = r.sum1; e.sums[4] = g.x; e.sums[5] = g.y; e.sums[6] = g.z; e.sums[7] = g.w;
    g = r.pmass; e.mass = g.x; e.inv_mass = g.y; e.spare0 = g.z; e.spare1 = g.w;
    e.omega[0] = r.omega; e.D[0] = r.D; e.C[0] = r.C; e.kd[0] = r.kd;
    g = r.steer;
    e.steer[0] = (w == 3) ? g.y : g.x; e.steer_vel[0] = (w == 3) ? g.w : g.z;   // lanes 0-2 see the LEFT joint, lane 3 the right
    e.steer[1] = g.y; e.steer_vel[1] = g.w;
    if (with_cmd) {
        g = r.cmd; e.cmd[0] = g.x; e.cmd[1] = g.y; e.cmd[2] = g.z; e.cmd[3] = g.w;
        g = r.cmdb; e.cmdb[0] = g.x; e.cmdb[1] = g.y; e.cmdb[2] = g.z; e.cmdb[3] = g.w;
    }
}
__device__ __forceinline__ void load_env_quad(const float4* __restrict__ st, int n, int i, int w, EnvState& e, bool with_cmd,
                                              bool with_iw = false, float inv_Iw_nominal = 0.0f) {
    QuadRaw r;
    quad_issue_loads(st, n, i, w, r, with_cmd, with_iw);
    quad_unpack(r, w, e, with_cmd, with_iw, inv_Iw_nominal);
}
__device__ __forceinline__ void store_env_quad(float4* __restrict__ st, int n, int i, int w, const EnvState& e, bool with_cmd,
                                               bool with_sums = true) {
    float* f = reinterpret_cast<float*>(st);
    f[(size_t)WL_G_WHEEL * n * 4 + (size_t)i * 4 + w] = e.omega[0];
    if (w >= 2) {                                                      // own steer joint: pos at [w-2], vel at [2 + w-2]
        f[(size_t)WL_G_STEER * n * 4 + (size_t)i * 4 + (w - 2)] = e.steer[0];
        f[(size_t)WL_G_STEER * n * 4 + (size_t)i * 4 + w] = e.steer_vel[0];
    }
    if (w == 0) {
        stg4(st, WL_G_POS, n, i, make_float4(e.p.x, e.p.y, e.p.z, __int_as_float(e.ep_len)));
        stg4(st, WL_G_QUAT, n, i, make_float4(e.qw, e.qx, e.qy, e.qz));
        stg4(st, WL_G_LINVEL, n, i, make_float4(e.v.x, e.v.y, e.v.z, e.t_hf));
        stg4(st, WL_G_ANGVEL, n, i, make_float4(e.w.x, e.w.y, e.w.z, e.t_lf));
    } else if (w == 1) {
        stg4(st, WL_G_ACTION, n, i, make_float4(e.action[0], e.action[1], e.prev_action[0], e.prev_action[1]));
        if (with_sums) {
            stg4(st, WL_G_SUM0, n, i, make_float4(e.sums[0], e.sums[1], e.sums[2], e.sums[3]));
            stg4(st, WL_G_SUM1, n, i, make_float4(e.sums[4], e.sums[5], e.sums[6], e.sums[7]));
        }
        if (with_cmd) {
            stg4(st, WL_G_CMD, n, i, make_float4(e.cmd[0], e.cmd[1], e.cmd[2], e.cmd[3]));
            stg4(st, WL_G_CMDB, n, i, make_float4(e.cmdb[0], e.cmdb[1], e.cmdb[2], e.cmdb[3]));
        }
    }
}
// store_env_quad for the duo kernel's fixed specs (no command, no sums), with no lane-divergent region: the chassis is the
// same in the quad's four lanes, so lane w writes state group w (position, quaternion, linear, angular velocity), lane 0
// also the actions and lanes 2 / 3 their steer joint.  Every store is predicated on its lane's condition.
__device__ __forceinline__ void st_global_if(float* p, float v, bool pred) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %2, 0;\n @p st.global.f32 [%0], %1;\n}" ::"l"(p), "f"(v), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void st_global_if(float4* p, float4 v, bool pred) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %5, 0;\n @p st.global.v4.f32 [%0], {%1, %2, %3, %4};\n}"
                 ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void st_global_if(uint8_t* p, uint32_t v, bool pred) {
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %2, 0;\n @p st.global.u8 [%0], %1;\n}" ::"l"(p), "r"(v), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void store_env_quad_sel(float4* __restrict__ st, int n, int i, int w, const EnvState& e, bool live) {
    float* f = reinterpret_cast<float*>(st);
    const bool w0 = w == 0, w1 = w == 1, w2 = w == 2;
    const float4 g = make_float4(sel(w0, e.p.x, sel(w1, e.qw, sel(w2, e.v.x, e.w.x))), sel(w0, e.p.y, sel(w1, e.qx, sel(w2, e.v.y, e.w.y))),
                                 sel(w0, e.p.z, sel(w1, e.qy, sel(w2, e.v.z, e.w.z))),
                                 sel(w0, __int_as_float(e.ep_len), sel(w1, e.qz, sel(w2, e.t_hf, e.t_lf))));
    st_global_if(st + (size_t)w * n + i, g, live);                                 // WL_G_POS + w
    st_global_if(st + (size_t)WL_G_ACTION * n + i, make_float4(e.action[0], e.action[1], e.prev_action[0], e.prev_action[1]),
                 live && w == 0);
    st_global_if(f + (size_t)WL_G_WHEEL * n * 4 + (size_t)i * 4 + w, e.omega[0], live);
    const int js = (w >= 2) ? w - 2 : 0;
    st_global_if(f + (size_t)WL_G_STEER * n * 4 + (size_t)i * 4 + js, e.steer[0], live && w >= 2);
    st_global_if(f + (size_t)WL_G_STEER * n * 4 + (size_t)i * 4 + 2 + js, e.steer_vel[0], live && w >= 2);
}

// ---- step spec: the config fields that pick a branch or set a trip count in the Drift-family step ----------------------
// A kernel templated on a packed spec key K != 0 reads these fields as constants, so the branches it does not take and the
// sub-step loop's trip count are resolved at compile time.  K == 0 is the generic instantiation: every field is read from
// the config at run time.
struct StepSpec { int32_t action_kind, bounding, no_reverse, push_enable, noise, wheel_mass, decimation, substeps; };

__host__ __device__ constexpr StepSpec step_spec(const wl_config& c) {
    return StepSpec{c.action_kind, c.bounding, c.no_reverse != 0, c.push_enable != 0, c.enable_corruption != 0,
                    c.dr_wheel_mass_enable != 0, c.decimation, c.substeps};
}
// bit 31 set, [0,2) action kind, [2,4) bounding, 4..7 the flags, [8,16) decimation, [16,24) substeps; 0 if a field does not fit
__host__ __device__ constexpr uint32_t spec_key(const StepSpec& s) {
    return (s.action_kind < 0 || s.action_kind > 3 || s.bounding < 0 || s.bounding > 3 || s.decimation < 1 || s.decimation > 255 ||
            s.substeps < 1 || s.substeps > 255) ? 0u
         : 0x80000000u | (uint32_t)s.action_kind | ((uint32_t)s.bounding << 2) | ((uint32_t)s.no_reverse << 4) |
           ((uint32_t)s.push_enable << 5) | ((uint32_t)s.noise << 6) | ((uint32_t)s.wheel_mass << 7) |
           ((uint32_t)s.decimation << 8) | ((uint32_t)s.substeps << 16);
}
template <uint32_t K>
struct Spec {
    static constexpr bool fixed = K != 0u;
    __device__ __forceinline__ static int action_kind(const wl_config& c) { return fixed ? (int)(K & 3u) : c.action_kind; }
    __device__ __forceinline__ static int bounding(const wl_config& c) { return fixed ? (int)((K >> 2) & 3u) : c.bounding; }
    __device__ __forceinline__ static bool no_reverse(const wl_config& c) { return fixed ? ((K >> 4) & 1u) != 0u : c.no_reverse != 0; }
    __device__ __forceinline__ static bool push_enable(const wl_config& c) { return fixed ? ((K >> 5) & 1u) != 0u : c.push_enable != 0; }
    __device__ __forceinline__ static bool noise(const wl_config& c) { return fixed ? ((K >> 6) & 1u) != 0u : c.enable_corruption != 0; }
    __device__ __forceinline__ static bool wheel_mass(const wl_config& c) { return fixed ? ((K >> 7) & 1u) != 0u : c.dr_wheel_mass_enable != 0; }
    __device__ __forceinline__ static int decimation(const wl_config& c) { return fixed ? (int)((K >> 8) & 0xFFu) : c.decimation; }
    __device__ __forceinline__ static int substeps(const wl_config& c) { return fixed ? (int)((K >> 16) & 0xFFu) : c.substeps; }
};

// ---- A. action term ---------------------------------------------------------------
template <uint32_t K = 0>
__device__ __forceinline__ void process_action(const wl_config& c, float a0, float a1, float wheel_target[4], float steer_target[2]) {
    using S = Spec<K>;
    if (S::bounding(c) == WL_BOUND_CLIP) { a0 = r_clamp(a0, -1.0f, 1.0f); a1 = r_clamp(a1, -1.0f, 1.0f); }
    else if (S::bounding(c) == WL_BOUND_TANH) { a0 = det_tanh(a0); a1 = det_tanh(a1); }      // ackermann_actions.py:126-127
    float v = a0 * c.act_scale[0] + c.act_offset[0];
    float delta = a1 * c.act_scale[1] + c.act_offset[1];
    if (S::no_reverse(c)) v = r_max(v, 0.0f);
    float tan_d = det_tan(delta);
    float L = c.base_length, W = c.base_width, r = c.wheel_radius_cfg;
    if (S::action_kind(c) == WL_ACT_RWD) {
        float wt = v * c.d_inv_wheel_radius_cfg;
        wheel_target[WL_BL] = wt; wheel_target[WL_BR] = wt; wheel_target[WL_FL] = 0.0f; wheel_target[WL_FR] = 0.0f;
        steer_target[0] = tan_d; steer_target[1] = tan_d;      // quirk Q1
        return;
    }
    float Rt = (tan_d == 0.0f) ? 1.0e6f : L / tan_d;
    float hw = W / 2.0f;
    float Rl = Rt - hw, Rr = Rt + hw;
    float Rrl = sqrtf(Rl * Rl + L * L), Rrr = sqrtf(Rr * Rr + L * L);
    float rden = 1.0f / (Rt * r);
    wheel_target[WL_FL] = v * fabsf(Rrl * rden);
    wheel_target[WL_FR] = v * fabsf(Rrr * rden);
    wheel_target[WL_BL] = v * fabsf(Rl * rden);
    wheel_target[WL_BR] = v * fabsf(Rr * rden);
    if (S::action_kind(c) == WL_ACT_4WD) { steer_target[0] = tan_d; steer_target[1] = tan_d; }
    else { steer_target[0] = det_atan(L / Rl); steer_target[1] = det_atan(L / Rr); }
}

// ---- a7 DC motor -------------------------------------------------------------------
__device__ __forceinline__ float dc_motor(const wl_config& c, float kd, float effort_limit, float target, float omega) {
    if (!(effort_limit > 0.0f)) return 0.0f;
    float tau = kd * (target - omega);
    float ratio = omega * c.d_inv_dc_vel_limit;
    float max_eff = r_clamp(c.dc_saturation * (1.0f - ratio), 0.0f, effort_limit);
    float min_eff = r_clamp(c.dc_saturation * (-1.0f - ratio), -effort_limit, 0.0f);
    return r_clamp(tau, min_eff, max_eff);
}

// DCMotor speed-dependent effort limits (the clip of dc_motor), evaluated once per physics step like IsaacLab does
__device__ __forceinline__ void dc_limits(const wl_config& c, float effort_limit, float omega, float& lo, float& hi) {
    if (!(effort_limit > 0.0f)) { lo = 0.0f; hi = 0.0f; return; }
    float ratio = omega * c.d_inv_dc_vel_limit;
    hi = r_clamp(c.dc_saturation * (1.0f - ratio), 0.0f, effort_limit);
    lo = r_clamp(c.dc_saturation * (-1.0f - ratio), -effort_limit, 0.0f);
}
// the same limits as a select instead of an early return (no divergent region where it runs inside the sub-step loop)
__device__ __forceinline__ void dc_limits_sel(const wl_config& c, float effort_limit, float omega, float& lo, float& hi) {
    const bool on = effort_limit > 0.0f;
    const float ratio = omega * c.d_inv_dc_vel_limit;
    const float h = r_clamp(c.dc_saturation * (1.0f - ratio), 0.0f, effort_limit);
    const float l = r_clamp(c.dc_saturation * (-1.0f - ratio), -effort_limit, 0.0f);
    hi = on ? h : 0.0f; lo = on ? l : 0.0f;
}

// ---- terrain -----------------------------------------------------------------------
struct Terrain { const float* __restrict__ hf; };

// bilinear height-field sample at world (x, y): returns false outside the raster (a "miss" for the ray-caster,
// the z = hf_outside_z ground plane for the wheels).  gx, gy = d z / d x, d z / d y.
__device__ __forceinline__ bool hf_sample(const wl_config& c, const float* __restrict__ hf, float x, float y, float& z, float& gx,
                                          float& gy) {
    const float inv = c.d_inv_hf_cell;
    float fx = (x - c.hf_x0) * inv, fy = (y - c.hf_y0) * inv;
    if (!((fx >= 0.0f) && (fy >= 0.0f) && (fx <= (float)(c.hf_nx - 1)) && (fy <= (float)(c.hf_ny - 1)))) return false;
    int ix = (int)floorf(fx), iy = (int)floorf(fy);
    if (ix > c.hf_nx - 2) ix = c.hf_nx - 2;
    if (iy > c.hf_ny - 2) iy = c.hf_ny - 2;
    float tx = fx - (float)ix, ty = fy - (float)iy;
    const float* row0 = hf + (size_t)iy * c.hf_pitch + ix;
    const float* row1 = row0 + c.hf_pitch;
    float z00 = __ldg(row0), z10 = __ldg(row0 + 1), z01 = __ldg(row1), z11 = __ldg(row1 + 1);
    float za = fm(z10 - z00, tx, z00), zb = fm(z11 - z01, tx, z01);
    z = fm(zb - za, ty, za);
    gx = fm((z11 - z01) - (z10 - z00), ty, z10 - z00) * inv;
    gy = (zb - za) * inv;
    return true;
}
// height z and unit normal n (world) under world point (x, y).  FLAT tasks never call this.
__device__ __forceinline__ void heightfield_at(const wl_config& c, const Terrain& T, float x, float y, float& z, V3& n) {
    float gx, gy;
    if (T.hf != nullptr && hf_sample(c, T.hf, x, y, z, gx, gy)) {
        float ninv = fdiv_norm(1.0f, fsqrt_norm(fm(gx, gx, fm(gy, gy, 1.0f))));       // argument >= 1: normal range
        n = V3{-gx * ninv, -gy * ninv, ninv};
        return;
    }
    z = (T.hf != nullptr) ? c.hf_outside_z : 0.0f;
    n = V3{0.0f, 0.0f, 1.0f};
}

// ---- a8 integrator sub-step ----------------------------------------------------------
struct Chassis { V3 pc; float qw, qx, qy, qz; V3 v; V3 wb; };
// per-env invariants of the env step: chassis inertia (DR mass ratio) and, per wheel (LANES == 4: slot 0 = this lane's
// wheel), h / I_w and 1 / (1 + h kd / I_w) of the implicit DC-motor damper
struct StepConsts { float I[3], invI[3]; float hI[4], idk[4], fxk[4]; };

template <int NW, uint32_t K = 0>
__device__ __forceinline__ StepConsts make_step_consts(const wl_config& c, const EnvState& e) {
    StepConsts k;
    const float mass = e.mass, inv_mass = e.inv_mass;
#pragma unroll
    for (int i = 0; i < NW; ++i) {
        k.hI[i] = Spec<K>::wheel_mass(c) ? c.d_h * e.inv_Iw[i] : c.d_hI;
        // hI > 0 and the damping kd >= 0, so the divisor is >= 1 and the quotient normal: a fixed spec skips the slow-path check
        k.idk[i] = Spec<K>::fixed ? fdiv_norm(1.0f, fm(k.hI[i], e.kd[i], 1.0f)) : 1.0f / fm(k.hI[i], e.kd[i], 1.0f);
        // longitudinal stick cap (tire_mx / h) with this wheel's own spin inertia
        k.fxk[i] = Spec<K>::wheel_mass(c) ? c.d_inv_h / fm(c.wheel_radius * c.wheel_radius, e.inv_Iw[i], c.tire_mx_rest) : c.d_fxk;
    }
    float ms = mass * c.d_inv_mass_nominal;          // inertia scales with the DR mass ratio (a14)
    float ms_inv = c.mass_nominal * inv_mass;
#pragma unroll
    for (int a = 0; a < 3; ++a) { k.I[a] = c.inertia_nominal[a] * ms; k.invI[a] = c.d_invI_nominal[a] * ms_inv; }
    return k;
}

// steer joint j (0 left, 1 right): implicit PD step, returns sin/cos of the new angle
__device__ __forceinline__ void steer_step(const wl_config& c, float target, float& pos, float& vel, float& sn, float& cs) {
    float v = fm(c.d_hkp, target - pos, c.steer_inertia * vel) * c.d_sden;
    v = r_clamp(v, -c.steer_vel_limit, c.steer_vel_limit);
    float p = r_clamp(fm(c.d_h, v, pos), -c.steer_pos_limit, c.steer_pos_limit);
    vel = v; pos = p;
    det_sincos(p, sn, cs);
}

struct WheelOut { V3 F, Tq; float omega; };

// one wheel: contact, Pacejka slip force with the implicit-stick cap, spin update.  `i` = wheel index
// [bl, br, fl, fr]; (sn, cs) = sin/cos of its steer angle (front wheels only).  SEL: the front / rear tyre direction is a
// select between both forms, not a branch on i (for a warp whose lanes hold different wheels)
template <int TASK, bool SEL = false>
__device__ __forceinline__ WheelOut wheel_force(const wl_config& c, const Terrain& T, const StepConsts& k, const M3& R,
                                                const Chassis& b, V3 vb, int i, float sn, float cs, float omega, float target,
                                                float eff_lo, float eff_hi, float kd, float hI, float idk, float fxk, float Dmu, float Cmu) {
    const float rw = c.wheel_radius;
    V3 rho{((i >= 2) ? c.hub_x_front : c.hub_x_rear) - c.com[0], ((i & 1) ? -c.hub_y : c.hub_y) - c.com[1], c.hub_z - c.com[2]};
    float comp; V3 nb;
    if (TASK == WL_TASK_ELEVATION) {
        V3 hubw = rot(R, rho);
        hubw.x += b.pc.x; hubw.y += b.pc.y; hubw.z += b.pc.z;
        float zt; V3 nw; heightfield_at(c, T, hubw.x, hubw.y, zt, nw);
        comp = fm(-(hubw.z - zt), nw.z, rw);
        nb = rotT(R, nw);
    } else {                                     // plane z = 0, normal (0,0,1)
        float hz = dot3(R.r[6], R.r[7], R.r[8], rho.x, rho.y, rho.z) + b.pc.z;
        comp = rw - hz;
        nb = V3{R.r[6], R.r[7], R.r[8]};
    }
    WheelOut o;
    // drive torque first.  The DCMotor damper tau = kd (w_t - w) is stiff (kd h / I_w >> 1): implicit in the new wheel
    // speed; when that torque leaves the motor's effort limits the clipped torque is applied explicitly instead
    const float os = fm(hI, fm(kd, target, -(c.wheel_damping * omega)), omega) * idk;
    const float t_imp = kd * (target - os);
    const float tc = r_clamp(t_imp, eff_lo, eff_hi);
    float om_star = (tc == t_imp) ? os : fm(hI, tc - c.wheel_damping * omega, omega);
    V3 rc = axpy(rho, -rw, nb);
    V3 vc = cross(b.wb, rc);
    vc.x += vb.x; vc.y += vb.y; vc.z += vb.z;
    float sdot = -dot(nb, vc);
    float ce = r_min(comp, c.comp_max);                       // depenetration cap (spawn inside a ramp, hard landings)
    float Fz = fm(c.susp_k, ce, c.susp_c * sdot);
    if (ce > c.susp_travel) Fz = fm(c.bump_k, ce - c.susp_travel, Fz);
    Fz = (comp > 0.0f) ? r_max(Fz, 0.0f) : 0.0f;
    V3 ft;
    if (SEL) {
        const float df = fm(cs, nb.x, sn * nb.y), dr = nb.x;
        const bool front = i >= 2;
        ft.x = front ? fm(-df, nb.x, cs) : fm(-dr, nb.x, 1.0f);
        ft.y = front ? fm(-df, nb.y, sn) : -(dr * nb.y);
        ft.z = front ? -(df * nb.z) : -(dr * nb.z);
    } else if (i >= 2) { float d = fm(cs, nb.x, sn * nb.y); ft = V3{fm(-d, nb.x, cs), fm(-d, nb.y, sn), -(d * nb.z)}; }
    else { float d = nb.x; ft = V3{fm(-d, nb.x, 1.0f), -(d * nb.y), -(d * nb.z)}; }
    // |ft|^2 = 1 - d^2: normalise with the binomial series of (1 - e)^(-1/2), e = 1 - |ft|^2 (no sqrt, no division)
    float en = 1.0f - dot(ft, ft);
    float finv = fm(fm(fm(fm(0.2734375f, en, 0.3125f), en, 0.375f), en, 0.5f), en, 1.0f);
    ft.x *= finv; ft.y *= finv; ft.z *= finv;
    V3 lt = cross(nb, ft);
    float vx = dot(vc, ft), vy = dot(vc, lt);
    float sx = fm(om_star, rw, -vx), sy = -vy;               // slip velocity of the tyre surface
    // |s| >= 1e-12 keeps every operand below in the normal range (the fast IEEE sequences need no slow path); at exactly
    // zero slip the force is zero through sx = sy = 0 either way
    float smag = fsqrt_norm(r_max(fm(sx, sx, sy * sy), 1.0e-24f));
    float den = r_max(fabsf(vx), c.tire_v0);
    float sm = det_sin_0_pi(Cmu * det_atan_ratio<true>(c.tire_B * smag, den));
    float Fmag = Fz * (Dmu * sm);
    float inv_s = fdiv_norm(1.0f, r_max(smag, 1.0e-9f));
    float Fx = (Fmag * sx) * inv_s, Fy = (Fmag * sy) * inv_s;
    float fxm = fxk * fabsf(sx), fym = c.d_fyk * fabsf(sy);  // implicit-stick cap
    Fx = r_clamp(Fx, -fxm, fxm); Fy = r_clamp(Fy, -fym, fym);
    o.F = V3{fm(Fz, nb.x, fm(Fx, ft.x, Fy * lt.x)), fm(Fz, nb.y, fm(Fx, ft.y, Fy * lt.y)), fm(Fz, nb.z, fm(Fx, ft.z, Fy * lt.z))};
    o.Tq = cross(rc, o.F);
    o.omega = fm(-hI, rw * Fx, om_star);
    return o;
}

// chassis: semi-implicit Euler; Euler's equations in the body frame (gyroscopic term on, mushr.py:28)
__device__ __forceinline__ void chassis_integrate(const wl_config& c, const StepConsts& k, const M3& R, Chassis& b, V3 Fb, V3 Tb,
                                                  float inv_mass) {
    const float h = c.d_h;
    V3 Fw = rot(R, Fb);
    b.v.x = fm(h, Fw.x * inv_mass, b.v.x);
    b.v.y = fm(h, Fw.y * inv_mass, b.v.y);
    b.v.z = fm(h, fm(Fw.z, inv_mass, -c.gravity), b.v.z);
    V3 Iw3{k.I[0] * b.wb.x, k.I[1] * b.wb.y, k.I[2] * b.wb.z};
    V3 g = cross(b.wb, Iw3);
    b.wb.x = fm(h, (Tb.x - g.x) * k.invI[0], b.wb.x);
    b.wb.y = fm(h, (Tb.y - g.y) * k.invI[1], b.wb.y);
    b.wb.z = fm(h, (Tb.z - g.z) * k.invI[2], b.wb.z);
    b.pc = axpy(b.pc, h, b.v);
    float hh = 0.5f * h;
    float qw = b.qw, qx = b.qx, qy = b.qy, qz = b.qz, ox = b.wb.x, oy = b.wb.y, oz = b.wb.z;
    float nqw = fm(-hh, dot3(qx, qy, qz, ox, oy, oz), qw);
    float nqx = fm(hh, fm(qw, ox, fm(qy, oz, -(qz * oy))), qx);
    float nqy = fm(hh, fm(qw, oy, fm(qz, ox, -(qx * oz))), qy);
    float nqz = fm(hh, fm(qw, oz, fm(qx, oy, -(qy * ox))), qz);
    // renormalise with the series of (1 + e)^(-1/2), e = |q|^2 - 1 = O(h^2 |w|^2) (no sqrt, no division)
    float eq = fm(nqw, nqw, fm(nqx, nqx, fm(nqy, nqy, nqz * nqz))) - 1.0f;
    float qinv = fm(fm(fm(-0.3125f, eq, 0.375f), eq, -0.5f), eq, 1.0f);
    b.qw = nqw * qinv; b.qx = nqx * qinv; b.qy = nqy * qinv; b.qz = nqz * qinv;
}

// LANES == 1: one thread owns the env and loops over the 4 wheels.
// LANES == 4: four adjacent lanes own one env; lane (l & 3) owns wheel l & 3, the chassis is integrated
//             redundantly (bit-identically) in all four, forces are summed with two butterfly shuffles.
// Both sum as (F0 + F1) + (F2 + F3), the order the oracle uses.  SEL (LANES == 4): no divergent region in the pass.
template <int TASK, int LANES, bool SEL = false>
__device__ __forceinline__ void physics_substep(const wl_config& c, const Terrain& T, EnvState& e, Chassis& b,
                                                const float wheel_target[4], const float eff_lo[4], const float eff_hi[4],
                                                const float steer_target[2], const StepConsts& k) {
    M3 R = rotmat(b.qw, b.qx, b.qy, b.qz);
    V3 vb = rotT(R, b.v);
    V3 Fb, Tb;
    if (LANES == 1) {
        float sn[2], cs[2];
        steer_step(c, steer_target[0], e.steer[0], e.steer_vel[0], sn[0], cs[0]);
        steer_step(c, steer_target[1], e.steer[1], e.steer_vel[1], sn[1], cs[1]);
        WheelOut w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
            w[i] = wheel_force<TASK>(c, T, k, R, b, vb, i, (i >= 2) ? sn[i - 2] : 0.0f, (i >= 2) ? cs[i - 2] : 1.0f, e.omega[i],
                                     wheel_target[i], eff_lo[i], eff_hi[i], e.kd[i], k.hI[i], k.idk[i], k.fxk[i], e.D[i], e.C[i]);
#pragma unroll
        for (int i = 0; i < 4; ++i) e.omega[i] = w[i].omega;
        Fb = V3{(w[0].F.x + w[1].F.x) + (w[2].F.x + w[3].F.x), (w[0].F.y + w[1].F.y) + (w[2].F.y + w[3].F.y),
                (w[0].F.z + w[1].F.z) + (w[2].F.z + w[3].F.z)};
        Tb = V3{(w[0].Tq.x + w[1].Tq.x) + (w[2].Tq.x + w[3].Tq.x), (w[0].Tq.y + w[1].Tq.y) + (w[2].Tq.y + w[3].Tq.y),
                (w[0].Tq.z + w[1].Tq.z) + (w[2].Tq.z + w[3].Tq.z)};
    } else {
        const int i = threadIdx.x & 3;
        float sn, cs;
        // every lane steps the joint it holds (rear lanes carry a copy of the left joint that is never stored): no divergent
        // region inside the sub-step; rear wheels then take (sin, cos) = (0, 1)
        steer_step(c, steer_target[0], e.steer[0], e.steer_vel[0], sn, cs);
        sn = (i >= 2) ? sn : 0.0f; cs = (i >= 2) ? cs : 1.0f;
        WheelOut w = wheel_force<TASK, SEL>(c, T, k, R, b, vb, i, sn, cs, e.omega[0], wheel_target[0], eff_lo[0], eff_hi[0], e.kd[0],
                                       k.hI[0], k.idk[0], k.fxk[0], e.D[0], e.C[0]);
        e.omega[0] = w.omega;
        float v6[6] = {w.F.x, w.F.y, w.F.z, w.Tq.x, w.Tq.y, w.Tq.z};
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            v6[q] += __shfl_xor_sync(0xffffffffu, v6[q], 1);
            v6[q] += __shfl_xor_sync(0xffffffffu, v6[q], 2);
        }
        Fb = V3{v6[0], v6[1], v6[2]}; Tb = V3{v6[3], v6[4], v6[5]};
    }
    chassis_integrate(c, k, R, b, Fb, Tb, e.inv_mass);
}

// ---- B. decimation x (actuators -> integrator) on the chassis at the centre of mass ------------------------------------
__device__ __forceinline__ Chassis chassis_from_env(const wl_config& c, const EnvState& e) {
    const M3 R = rotmat(e.qw, e.qx, e.qy, e.qz);
    const V3 cw = rot(R, V3{c.com[0], c.com[1], c.com[2]});
    Chassis b;
    b.pc = V3{e.p.x + cw.x, e.p.y + cw.y, e.p.z + cw.z};
    b.v = e.v; b.qw = e.qw; b.qx = e.qx; b.qy = e.qy; b.qz = e.qz;
    b.wb = rotT(R, e.w);
    return b;
}
// effort: the DC-motor effort limit per wheel (LANES == 4: slot 0 = this lane's wheel); the speed-dependent limits are
// formed once per physics step.  With a fixed spec (K != 0) the trip counts are constants but the loops stay rolled: fully
// unrolled, the 4 x 1 Drift sub-steps were no faster on H100 (DESIGN.md 6e) and cost ~900 more static instructions
// SEL: the pass has no divergent region (dc_limits_sel, physics_substep<..., SEL>).  `pass_done` is called after every
// sub-step (the duo kernel's phase trace, WL_DUO_TRACE; empty otherwise).
struct NoPassHook { __device__ __forceinline__ void operator()(const EnvState&) const {} };
template <int TASK, int LANES, uint32_t K = 0, bool SEL = false, typename PassHook = NoPassHook>
__device__ __forceinline__ void run_substeps(const wl_config& c, const Terrain& T, EnvState& e, Chassis& b, const float target[4],
                                             const float effort[4], const float steer_target[2], const StepConsts& kc,
                                             PassHook pass_done = {}) {
    using S = Spec<K>;
    for (int d = 0; d < S::decimation(c); ++d) {
        float lo[4], hi[4];
#pragma unroll
        for (int w = 0; w < 4 / LANES; ++w) {
            if (SEL) dc_limits_sel(c, effort[w], e.omega[w], lo[w], hi[w]);
            else dc_limits(c, effort[w], e.omega[w], lo[w], hi[w]);
        }
        for (int j = 0; j < S::substeps(c); ++j) {
            physics_substep<TASK, LANES, SEL>(c, T, e, b, target, lo, hi, steer_target, kc);
            pass_done(e);
        }
    }
}
// back to the root frame: writes e.p / v / q / w, returns the rotation of the new attitude
__device__ __forceinline__ M3 env_from_chassis(const wl_config& c, EnvState& e, const Chassis& b) {
    const M3 R = rotmat(b.qw, b.qx, b.qy, b.qz);
    const V3 cw = rot(R, V3{c.com[0], c.com[1], c.com[2]});
    e.p = V3{b.pc.x - cw.x, b.pc.y - cw.y, b.pc.z - cw.z};
    e.v = b.v; e.qw = b.qw; e.qx = b.qx; e.qy = b.qy; e.qz = b.qz;
    e.w = rot(R, b.wb);
    return R;
}

// ---- drift terminations / rewards -----------------------------------------------------
__device__ __forceinline__ bool drift_off_track(const wl_config& c, float x, float y) {
    float st = c.trk_straight, ro = c.trk_corner_out, ri = c.trk_corner_in;
    bool off, in;
    if (fabsf(y) < st) { off = fabsf(x) > ro; in = fabsf(x) < ri; }
    else if (y > 0.0f) { float d2 = (y - st) * (y - st) + x * x; off = d2 > ro * ro; in = d2 < ri * ri; }
    else { float d2 = (y + st) * (y + st) + x * x; off = d2 > ro * ro; in = d2 < ri * ri; }
    return off || in;
}

// `slip_atan` = det_atan2(vb.y, vb.x) (computed by the caller so that the quad kernel can batch its atan2 calls)
// SEL: no divergent region and no slow-path call: the roots through fsqrt_sel, both cross-track cases evaluated and selected.
template <bool SEL = false>
__device__ __forceinline__ void drift_reward_terms(const wl_config& c, float steer_l, float steer_r, float slip_atan, V3 p, V3 vb,
                                                   V3 wb, float wz_world, bool out_of_bounds, bool time_out,
                                                   float f[WL_MAX_REW_TERMS]) {
    if (SEL) {
        const float slip = fabsf(slip_atan);
        float valid = (fabsf(vb.x) < c.slip_min_vel_x || slip > c.slip_max_thresh) ? 0.0f : slip;
        f[WL_DR_SIDE_SLIP] = (valid < c.slip_min_thresh) ? 0.0f : valid;
        const float dv = fsqrt_sel(vb.x * vb.x + vb.y * vb.y) - c.vel_speed_target;
        f[WL_DR_VEL] = dv * dv + c.vel_offset;
        f[WL_DR_PROGRESS] = wz_world;
        const float sm = (steer_l + steer_r) / 2.0f;
        const float av = r_clamp(wb.z, -c.tlgr_ang_vel_thresh, c.tlgr_ang_vel_thresh);
        f[WL_DR_TLGR] = r_max(sm * av * -1.0f, 0.0f);
        const float sp = fsqrt_sel(vb.x * vb.x + vb.y * vb.y + vb.z * vb.z);
        f[WL_DR_TURN_ENERGY] = (fabsf(p.y) > c.energy_straight) ? sp * sp : 0.0f;
        const float st = c.trk_straight, tr = c.ctd_track_radius;
        const float ds = (p.x > 0.0f) ? (p.x - tr) : (p.x + tr);
        const float yy = (p.y > 0.0f) ? (p.y - st) : (p.y + st);
        const float dc = fsqrt_sel(yy * yy + p.x * p.x) - tr;
        f[WL_DR_CROSS_TRACK] = fsqrt_sel(sel(fabsf(p.y) < st, ds * ds, dc * dc)) + c.ctd_offset;
        f[WL_DR_TERM_PENS] = (out_of_bounds && !time_out) ? 1.0f : 0.0f;
        f[7] = 0.0f;
        return;
    }
    float slip = fabsf(slip_atan);
    float valid = (fabsf(vb.x) < c.slip_min_vel_x || slip > c.slip_max_thresh) ? 0.0f : slip;
    if (valid < c.slip_min_thresh) valid = 0.0f;
    f[WL_DR_SIDE_SLIP] = valid;
    float gs = sqrtf(vb.x * vb.x + vb.y * vb.y);
    float dv = gs - c.vel_speed_target;
    f[WL_DR_VEL] = dv * dv + c.vel_offset;
    f[WL_DR_PROGRESS] = wz_world;
    float sm = (steer_l + steer_r) / 2.0f;
    float av = r_clamp(wb.z, -c.tlgr_ang_vel_thresh, c.tlgr_ang_vel_thresh);
    float tl = sm * av * -1.0f;
    f[WL_DR_TLGR] = r_max(tl, 0.0f);
    float sp = sqrtf(vb.x * vb.x + vb.y * vb.y + vb.z * vb.z);
    f[WL_DR_TURN_ENERGY] = (fabsf(p.y) > c.energy_straight) ? sp * sp : 0.0f;
    float st = c.trk_straight, tr = c.ctd_track_radius, sq;
    if (fabsf(p.y) < st) { float d = (p.x > 0.0f) ? (p.x - tr) : (p.x + tr); sq = d * d; }
    else { float yy = (p.y > 0.0f) ? (p.y - st) : (p.y + st); float d = sqrtf(yy * yy + p.x * p.x) - tr; sq = d * d; }
    f[WL_DR_CROSS_TRACK] = sqrtf(sq) + c.ctd_offset;
    f[WL_DR_TERM_PENS] = (out_of_bounds && !time_out) ? 1.0f : 0.0f;
    f[7] = 0.0f;
}
// drift termination mask: bit 0 time_out, bit 1 out of bounds
__device__ __forceinline__ uint32_t drift_term_mask(bool time_out, bool oob) { return (time_out ? 1u : 0u) | (oob ? 2u : 0u); }

// ---- elevation task (elevation/mushr_elevation_env_cfg.py) -------------------------------------------------
// terminations :339-376 -> mask bits [0 time_out, 1 cart_out_of_bounds, 2 stuck, 3 rollover, 4 at_goal]; rewards :155-305
// (active terms :283-305).  The command is the yaw-frame vector stored at the previous command update (quirk Q5:
// the reference subtracts the WORLD position from it).
__device__ __forceinline__ uint32_t elev_terms(const wl_config& c, const EnvState& e, const M3& R, V3 vb, float sum_omega,
                                               bool time_out, float f[WL_MAX_REW_TERMS]) {
    float gx = e.cmdb[0] - e.p.x, gy = e.cmdb[1] - e.p.y;
    float gn = sqrtf(fm(gx, gx, gy * gy));
    bool oob = e.p.z < c.elev_min_height;                                   // root_height_below_minimum :354-357
    bool stuck = (r_min(vb.x, 1.2f) < c.elev_stuck_min_vel) && (sum_omega > c.elev_stuck_spin);   // :342-347 (2nd def wins, Q6)
    bool roll = R.r[8] < c.elev_rollover_cos;                               // upright_bool :217-222,339-340
    bool goal = gn < c.elev_goal_dist;                                      // close_to_goal :268-273
    f[WL_ER_GOAL_RATE] = 5.0f + fm(e.v.x, gx, e.v.y * gy) / gn;             // goal_progress_rate :239-249
    float zv = e.p.z - c.elev_plane_z;                                      // higher_elevation :166-173
    float he = ((zv > 0.1f) && (vb.x > 0.1f)) ? zv : 0.0f;
    f[WL_ER_HEIGHT_Z] = r_clamp(he, 0.0f, 1.0f);
    f[WL_ER_FALLING] = (vb.z > c.elev_fall_vel) ? 1.0f : 0.0f;              // is_falling_penalty :251-254 (2nd def, Q6)
    f[WL_ER_TERM_PEN] = (stuck && !time_out) ? 1.0f : 0.0f;                 // is_terminated_term("stuck")
    f[4] = f[5] = f[6] = f[7] = 0.0f;
    return (time_out ? 1u : 0u) | (oob ? 2u : 0u) | (stuck ? 4u : 0u) | (roll ? 8u : 0u) | (goal ? 16u : 0u);
}
// reset_root_state_uniform (:409-419) on the default root state (z = 0.25, :97,147-149) + manager resets +
// command reset (UniformPose2dCommand resample, :425-435)
__device__ __forceinline__ void elev_reset_env(const wl_config& c, EnvState& e, uint32_t gid, uint32_t t) {
    uint4 r = philox4x32(c.seed, gid, t, RNG_RESET, 0u);
    uint4 r2 = philox4x32(c.seed, gid, t, RNG_RESET, 1u);
    e.p.x = uniform(r.x, c.elev_reset_xy[0], c.elev_reset_xy[1]);
    e.p.y = uniform(r.y, c.elev_reset_xy[0], c.elev_reset_xy[1]);
    e.p.z = c.elev_spawn_z;
    float yaw = uniform(r.z, -c.elev_reset_yaw, c.elev_reset_yaw);
    float sh, ch; det_sincos(yaw * 0.5f, sh, ch);
    e.qw = ch; e.qx = 0.0f; e.qy = 0.0f; e.qz = sh;
    e.v = V3{uniform(r.w, c.elev_reset_vel[0], c.elev_reset_vel[1]), uniform(r2.x, c.elev_reset_vel[0], c.elev_reset_vel[1]), 0.0f};
    e.w = V3{0.0f, 0.0f, 0.0f};
    e.ep_len = 0;
#pragma unroll
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) e.sums[k] = 0.0f;
    e.action[0] = e.action[1] = e.prev_action[0] = e.prev_action[1] = 0.0f;
    e.cmd[0] = uniform(r2.y, c.cmd_pos_range[0], c.cmd_pos_range[1]);
    e.cmd[1] = uniform(r2.z, c.cmd_pos_range[0], c.cmd_pos_range[1]);
    e.cmd[2] = 0.0f;
    e.cmd[3] = c.cmd_resample_s;
}
// cos/sin of the root yaw (quat_apply_yaw): normalised (1-2(y^2+z^2), 2(wz+xy))
__device__ __forceinline__ void yaw_cs(const EnvState& e, float& cy, float& sy) {
    float cr = fm(-2.0f, fm(e.qy, e.qy, e.qz * e.qz), 1.0f), sr = 2.0f * fm(e.qw, e.qz, e.qx * e.qy);
    float rinv = 1.0f / sqrtf(fm(cr, cr, sr * sr));
    cy = cr * rinv; sy = sr * rinv;
}
// CommandManager.compute(dt): timer, resample, then the yaw-frame command (UniformPose2dCommand._update_command)
__device__ __forceinline__ void elev_command_update(const wl_config& c, EnvState& e, uint32_t gid, uint32_t t, float step_dt) {
    e.cmd[3] = e.cmd[3] - step_dt;
    if (e.cmd[3] <= 0.0f) {
        uint4 r = philox4x32(c.seed, gid, t, RNG_CMD, 0u);
        e.cmd[0] = uniform(r.x, c.cmd_pos_range[0], c.cmd_pos_range[1]);
        e.cmd[1] = uniform(r.y, c.cmd_pos_range[0], c.cmd_pos_range[1]);
        e.cmd[3] = c.cmd_resample_s;
    }
    float cy, sy; yaw_cs(e, cy, sy);
    float dx = e.cmd[0] - e.p.x, dy = e.cmd[1] - e.p.y;
    e.cmdb[0] = fm(cy, dx, sy * dy);             // rotate by -yaw
    e.cmdb[1] = fm(cy, dy, -(sy * dx));
    e.cmdb[2] = 0.0f; e.cmdb[3] = 0.0f;
}
// proprioceptive head of the elevation observation (:57-72): 13 floats, no noise (:85); `eu` = euler_xyz
__device__ __forceinline__ void elev_proprio(const wl_config& c, const EnvState& e, V3 eu, float o[13]) {
    M3 R = rotmat(e.qw, e.qx, e.qy, e.qz);
    V3 vb = rotT(R, e.v), wb = rotT(R, e.w);
    float gx = e.cmdb[0] - e.p.x, gy = e.cmdb[1] - e.p.y;
    o[0] = (gx != gx) ? 0.0f : gx; o[1] = (gy != gy) ? 0.0f : gy;          // nan_to_num(nan=0)
    o[2] = eu.x; o[3] = eu.y; o[4] = eu.z;
    o[5] = r_clamp(vb.x, -c.obs_clip, c.obs_clip); o[6] = r_clamp(vb.y, -c.obs_clip, c.obs_clip); o[7] = r_clamp(vb.z, -c.obs_clip, c.obs_clip);
    o[8] = r_clamp(wb.x, -c.obs_clip, c.obs_clip); o[9] = r_clamp(wb.y, -c.obs_clip, c.obs_clip); o[10] = r_clamp(wb.z, -c.obs_clip, c.obs_clip);
    o[11] = r_clamp(e.action[0], -1.0f, 1.0f); o[12] = r_clamp(e.action[1], -1.0f, 1.0f);
}

// ---- visual task, physics side (visual/mushr_visual_env_cfg.py; the RTX camera observation is out of scope) -------
struct VisualMap { const int32_t* __restrict__ cells; const uint8_t* __restrict__ map; };
__device__ __forceinline__ VisualMap visual_map(const wl_config& c, const float* aux) {
    const char* b = reinterpret_cast<const char*>(aux);
    return VisualMap{reinterpret_cast<const int32_t*>(b), reinterpret_cast<const uint8_t*>(b + (((size_t)c.vis_n_trav * 4 + 15) & ~(size_t)15))};
}
// rewards :304-387 (traversable_reward, forward_vel), terminations :392-409 (time_out, out_of_map);
// map lookup = TraversabilityHashmapUtil.get_map_id (utils/traversability_utils.py:83-88: +spacing/2, truncation,
// clamp, indexed [y_idx, x_idx]; quirk Q14)
// ---- visual task, camera term (software pinhole camera over the 2-colour plane mesh; restated in oracle/wl_oracle.c) ----
__host__ __device__ __forceinline__ int vis_cam_floats(const wl_config& c) { return c.vis_cam ? c.vis_cam_w * (c.vis_cam_h - c.vis_cam_row0) : 0; }
// floats per observation row of the task (the visual row is the camera floats followed by the proprioceptive ones)
__host__ __device__ __forceinline__ int obs_row_floats(const wl_config& c, int task) {
    return task == WL_TASK_ELEVATION ? WL_OBS_DIM_ELEV : task == WL_TASK_VISUAL ? WL_OBS_DIM_VISUAL + vis_cam_floats(c) : WL_OBS_DIM_BLIND;
}
// torchvision rgb_to_grayscale of a grey pixel (r = g = b = v): the weights sum to 0.9999, not 1
__device__ __forceinline__ float cam_gray(float v) { return fm(0.114f, v, fm(0.587f, v, 0.2989f * v)); }
__device__ __forceinline__ float cam_clamp01(float v) { return r_min(r_max(v, 0.0f), 1.0f); }
struct CamAug { float v0, v1, w0, w1, w2; };      // values of the black / white class after ColorJitter; 5-tap Gaussian weights
// ColorJitter + GaussianBlur parameters of one camera frame (one draw per call for the WHOLE batch, like torchvision's
// transforms on a [B,3,H,W] tensor); `aug` != null overrides the draw (golden-vector tests).  A 2-valued grey image stays
// 2-valued under the point operations, so the jitter is tracked on the two class values; p = fraction of white pixels.
__device__ __forceinline__ CamAug cam_aug_params(const wl_config& c, uint32_t t, uint32_t stream, uint32_t sub, const float* aug, float p) {
    CamAug A; A.v0 = 0.0f; A.v1 = 1.0f; A.w0 = 1.0f; A.w1 = 0.0f; A.w2 = 0.0f;
    if (c.vis_cam != 2) return A;
    float b, ct, sa, sigma; int order[4] = {0, 1, 2, 3};
    if (aug != nullptr) {
        b = aug[0]; ct = aug[1]; sa = aug[2]; sigma = aug[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) order[k] = (int)aug[5 + k];
    } else {
        const uint4 r = philox4x32(c.seed, 0u, t, stream, 2u * sub), q = philox4x32(c.seed, 0u, t, stream, 2u * sub + 1u);
        b = uniform(r.x, r_max(0.0f, 1.0f - c.vis_aug_brightness), 1.0f + c.vis_aug_brightness);
        ct = uniform(r.y, r_max(0.0f, 1.0f - c.vis_aug_contrast), 1.0f + c.vis_aug_contrast);
        sa = uniform(r.z, r_max(0.0f, 1.0f - c.vis_aug_saturation), 1.0f + c.vis_aug_saturation);
        sigma = uniform(r.w, c.vis_aug_sigma[0], c.vis_aug_sigma[1]);
        const uint32_t rq[3] = {q.x, q.y, q.z};            // Fisher-Yates (torch.randperm(4) stand-in)
#pragma unroll
        for (int i = 3; i >= 1; --i) { const int j = (int)__umulhi(rq[3 - i], (uint32_t)(i + 1)); const int tmp = order[i]; order[i] = order[j]; order[j] = tmp; }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int op = order[k];
        if (op == 0) { A.v0 = cam_clamp01(b * A.v0); A.v1 = cam_clamp01(b * A.v1); }
        else if (op == 1) {
            const float m = fm(p, cam_gray(A.v1), (1.0f - p) * cam_gray(A.v0));          // mean of the grey-scale image
            A.v0 = cam_clamp01(fm(ct, A.v0, (1.0f - ct) * m)); A.v1 = cam_clamp01(fm(ct, A.v1, (1.0f - ct) * m));
        } else if (op == 2) {
            A.v0 = cam_clamp01(fm(sa, A.v0, (1.0f - sa) * cam_gray(A.v0))); A.v1 = cam_clamp01(fm(sa, A.v1, (1.0f - sa) * cam_gray(A.v1)));
        }                                                  // op 3 = hue: the identity on grey pixels
    }
    const float e1 = det_exp(-0.5f / (sigma * sigma)), e2 = (e1 * e1) * (e1 * e1);       // exp(-x^2 / 2 sigma^2), x = 1, 2
    const float S = fm(2.0f, e1 + e2, 1.0f);
    A.w0 = 1.0f / S; A.w1 = e1 / S; A.w2 = e2 / S;
    return A;
}
__device__ __forceinline__ uint32_t visual_terms(const wl_config& c, const VisualMap& vm, const EnvState& e, V3 vb, bool time_out,
                                                 float f[WL_MAX_REW_TERMS]) {
    int xi = (int)((e.p.x + c.vis_width / 2.0f + c.vis_row_spacing / 2.0f) / c.vis_row_spacing);
    int yi = (int)((e.p.y + c.vis_height / 2.0f + c.vis_col_spacing / 2.0f) / c.vis_col_spacing);
    xi = xi < 0 ? 0 : (xi > c.vis_rows - 1 ? c.vis_rows - 1 : xi);
    yi = yi < 0 ? 0 : (yi > c.vis_cols - 1 ? c.vis_cols - 1 : yi);
    const bool trav = __ldg(vm.map + (size_t)yi * c.vis_cols + xi) != 0;
    f[WL_VR_TRAVERSABLE] = trav ? 1.0f : -1.0f;
    f[WL_VR_FORWARD_VEL] = vb.x;
    f[2] = f[3] = f[4] = f[5] = f[6] = f[7] = 0.0f;
    const bool out = (e.p.x > c.vis_width / 2.0f) || (e.p.x < -c.vis_width / 2.0f) || (e.p.y > c.vis_height / 2.0f) ||
                     (e.p.y < -c.vis_height / 2.0f);
    return (time_out ? 1u : 0u) | (out ? 2u : 0u);
}
// reset_root_state (visual/mdp/events.py:11-42) with generate_random_poses (utils/__init__.py:188-202): a uniformly
// random traversable cell, yaw U(0,360) deg, z = 0.1, zero velocity
__device__ __forceinline__ void visual_reset_env(const wl_config& c, const VisualMap& vm, EnvState& e, uint32_t gid, uint32_t t) {
    uint4 r = philox4x32(c.seed, gid, t, RNG_RESET, 0u);
    const int cell = __ldg(vm.cells + __umulhi(r.x, (uint32_t)c.vis_n_trav));
    const int ys = cell / c.vis_cols, xs = cell - ys * c.vis_cols;
    e.p.x = ((float)xs - (float)(c.vis_cols / 2)) * c.vis_row_spacing;
    e.p.y = ((float)ys - (float)(c.vis_rows / 2)) * c.vis_col_spacing;
    e.p.z = c.vis_spawn_z;
    float yaw = (360.0f * u01(r.y)) * 0.017453292519943295f;
    float sh, ch; det_sincos(yaw * 0.5f, sh, ch);
    e.qw = ch; e.qx = 0.0f; e.qy = 0.0f; e.qz = sh;
    e.v = V3{0.0f, 0.0f, 0.0f}; e.w = V3{0.0f, 0.0f, 0.0f};
    e.ep_len = 0;
#pragma unroll
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) e.sums[k] = 0.0f;
    e.action[0] = e.action[1] = e.prev_action[0] = e.prev_action[1] = 0.0f;
}
// VisualObsCfg.PolicyCfg minus the camera term (:43-57; enable_corruption False): 8 floats
__device__ __forceinline__ void visual_proprio(const wl_config& c, const EnvState& e, float o[8]) {
    M3 R = rotmat(e.qw, e.qx, e.qy, e.qz);
    V3 vb = rotT(R, e.v), wb = rotT(R, e.w);
    o[0] = vb.x; o[1] = vb.y; o[2] = vb.z; o[3] = wb.x; o[4] = wb.y; o[5] = wb.z;
    o[6] = r_clamp(e.action[0], -1.0f, 1.0f); o[7] = r_clamp(e.action[1], -1.0f, 1.0f);
}

// ---- E. reward weighting and done flags ----------------------------------------------------
// value = f * w * dt per term, terms with w == 0 skipped; adds each value to the episode sums, returns the step reward
// SEL: every term is weighed and the sums take it by select (the same operations in the same order, so the same bits)
template <bool SEL = false>
__device__ __forceinline__ float weigh_rewards(const wl_config& c, const float wts[WL_MAX_REW_TERMS], const float f[WL_MAX_REW_TERMS],
                                               float sums[WL_MAX_REW_TERMS]) {
    float total = 0.0f;
#pragma unroll
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) {
        if (SEL) {
            const float val = f[k] * wts[k] * c.d_step_dt;
            const bool on = k < c.num_rew_terms && wts[k] != 0.0f;
            total = sel(on, total + val, total); sums[k] = sel(on, sums[k] + val, sums[k]);
        } else if (k < c.num_rew_terms) {
            float w = wts[k];
            if (w != 0.0f) { float val = f[k] * w * c.d_step_dt; total += val; sums[k] += val; }
        }
    }
    return total;
}
// terminated / truncated bytes of a termination mask: bit 0 (time_out) truncates, every other bit terminates
struct DoneBytes { uint8_t terminated, truncated; };
__device__ __forceinline__ DoneBytes done_bytes(uint32_t tmask) { return DoneBytes{(uint8_t)((tmask & ~1u) ? 1 : 0), (uint8_t)((tmask & 1u) ? 1 : 0)}; }

// ---- reset / pushes / observations -----------------------------------------------------
// The drift reset in two parts: the draw (a function of (seed, env id, step) and the config only, never of the state) and
// its application to the state.  The duo kernel draws in its aux warp and applies in its env warp.
struct DriftReset { float px, py, qw, qz, t_hf, t_lf; };
__device__ __forceinline__ DriftReset drift_reset_draw(const wl_config& c, uint32_t gid, uint32_t t) {
    uint4 r = philox4x32(c.seed, gid, t, RNG_RESET, 0u);
    uint32_t idx = __umulhi(r.x, (uint32_t)c.num_ref_poses);
    float nx = (2.0f * u01(r.y) - 1.0f) * c.reset_pos_noise;
    float ny = (2.0f * u01(r.z) - 1.0f) * c.reset_pos_noise;
    float nyaw = (2.0f * u01(r.w) - 1.0f) * c.reset_yaw_noise;
    float px = c.ref_poses[3 * idx + 0] + nx;
    float py = c.ref_poses[3 * idx + 1] + ny;
    float yaw = c.ref_poses[3 * idx + 2] * 0.017453292519943295f + nyaw;
    float sh, ch; det_sincos(yaw * 0.5f, sh, ch);
    uint4 r2 = philox4x32(c.seed, gid, t, RNG_RESET, 1u);
    return DriftReset{px, py, ch, sh, uniform(r2.x, c.push_hf_interval[0], c.push_hf_interval[1]),
                      uniform(r2.y, c.push_lf_interval[0], c.push_lf_interval[1])};
}
__device__ __forceinline__ void drift_reset_apply(const DriftReset& d, EnvState& e) {
    e.p.x = d.px; e.p.y = d.py; e.p.z = 0.0f;
    e.qw = d.qw; e.qx = 0.0f; e.qy = 0.0f; e.qz = d.qz;
    e.v = V3{0.0f, 0.0f, 0.0f}; e.w = V3{0.0f, 0.0f, 0.0f};
    e.ep_len = 0;
#pragma unroll
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) e.sums[k] = 0.0f;
    e.action[0] = e.action[1] = e.prev_action[0] = e.prev_action[1] = 0.0f;
    e.t_hf = d.t_hf; e.t_lf = d.t_lf;
}
__device__ __forceinline__ void drift_reset_env(const wl_config& c, EnvState& e, uint32_t gid, uint32_t t) {
    drift_reset_apply(drift_reset_draw(c, gid, t), e);
}
// the task's reset; vm is read by the visual task only
__device__ __forceinline__ void reset_env(const wl_config& c, int task, const VisualMap& vm, EnvState& e, uint32_t gid, uint32_t t) {
    if (task == WL_TASK_ELEVATION) elev_reset_env(c, e, gid, t);
    else if (task == WL_TASK_VISUAL) visual_reset_env(c, vm, e, gid, t);
    else drift_reset_env(c, e, gid, t);
}
// returns true when a push changed the velocities
__device__ __forceinline__ bool interval_pushes(const wl_config& c, EnvState& e, uint32_t gid, uint32_t t, float step_dt) {
    if (!c.push_enable) return false;
    bool fired = false;
    e.t_hf = e.t_hf - step_dt;
    if (e.t_hf < 1.0e-6f) {
        uint4 r = philox4x32(c.seed, gid, t, RNG_PUSH_HF, 0u);
        e.v.x = e.v.x + uniform(r.x, -c.push_hf_range[0], c.push_hf_range[0]);
        e.v.y = e.v.y + uniform(r.y, -c.push_hf_range[1], c.push_hf_range[1]);
        e.w.z = e.w.z + uniform(r.z, -c.push_hf_range[2], c.push_hf_range[2]);
        e.t_hf = uniform(r.w, c.push_hf_interval[0], c.push_hf_interval[1]);
        fired = true;
    }
    e.t_lf = e.t_lf - step_dt;
    if (e.t_lf < 1.0e-6f) {
        uint4 r = philox4x32(c.seed, gid, t, RNG_PUSH_LF, 0u);
        e.w.z = e.w.z + uniform(r.x, -c.push_lf_yaw, c.push_lf_yaw);
        e.t_lf = uniform(r.y, c.push_lf_interval[0], c.push_lf_interval[1]);
        fired = true;
    }
    return fired;
}
// writes 14 floats (obs must be 8-byte aligned: 14 floats = 7 x float2 per env)
__device__ __forceinline__ void blind_obs(const wl_config& c, const EnvState& e, uint32_t gid, uint32_t t, uint32_t stream,
                                          uint32_t sub0, float* __restrict__ obs) {
    M3 R = rotmat(e.qw, e.qx, e.qy, e.qz);
    V3 vb = rotT(R, e.v), wb = rotT(R, e.w), eu = euler_xyz(e.qw, e.qx, e.qy, e.qz);
    float z[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) z[k] = 0.0f;
    if (c.enable_corruption) {
#pragma unroll
        for (uint32_t k = 0; k < 3; ++k) {
            uint4 r = philox4x32(c.seed, gid, t, stream, sub0 + k);
            box_muller(r.x, r.y, z[4 * k + 0], z[4 * k + 1]);
            box_muller(r.z, r.w, z[4 * k + 2], z[4 * k + 3]);
        }
    }
    float o[14];
    o[0] = e.p.x + c.noise_std[0] * z[0]; o[1] = e.p.y + c.noise_std[0] * z[1]; o[2] = e.p.z + c.noise_std[0] * z[2];
    o[3] = eu.x + c.noise_std[1] * z[3]; o[4] = eu.y + c.noise_std[1] * z[4]; o[5] = eu.z + c.noise_std[1] * z[5];
    o[6] = vb.x + c.noise_std[2] * z[6]; o[7] = vb.y + c.noise_std[2] * z[7]; o[8] = vb.z + c.noise_std[2] * z[8];
    o[9] = wb.x + c.noise_std[3] * z[9]; o[10] = wb.y + c.noise_std[3] * z[10]; o[11] = wb.z + c.noise_std[3] * z[11];
    o[12] = r_clamp(e.action[0], -1.0f, 1.0f); o[13] = r_clamp(e.action[1], -1.0f, 1.0f);
    float2* o2 = reinterpret_cast<float2*>(obs);
#pragma unroll
    for (int k = 0; k < 7; ++k) o2[k] = make_float2(o[2 * k], o[2 * k + 1]);
}

// ---- fused rollout-slab fan-out over NVLink peer memory (SURVEY 8e): every output row of the step (observation, reward,
// done masks) is stored locally AND at the same offset of every peer's symmetric buffer (delta = peer base - local base),
// so the learner-facing "all-gather" is done by the time the step kernels are: no separate collective, no staging copy.
#define WL_MAX_PEERS 8
struct PeerFan { int32_t n; int32_t mc; long long delta[WL_MAX_PEERS]; long long mc_delta; };
template <typename TT>
__device__ __forceinline__ void fan_store(const PeerFan& pf, TT* p, TT v) {
    *p = v;
    for (int k = 0; k < pf.n; ++k) *reinterpret_cast<TT*>(reinterpret_cast<char*>(p) + pf.delta[k]) = v;
}
// NVSwitch multicast form (pf.mc, wl_set_multicast_fanout): ONE multimem.st to the multicast alias of the buffer, which the
// switch replicates into every rank's copy -- the GPU's NVLink egress is 1x the row instead of (world-1)x, and the kernel issues
// one remote store instead of world-1.  The local copy is also stored directly, so readers on this GPU never depend on the
// loop through the switch (the multicast write lands on the same bytes with the same value).  16- and 8-byte pieces only.
// MC_ONLY: the host has checked that every row of the launch is full and aligned -- no per-peer path in the kernel at all
template <bool MC_ONLY = false>
__device__ __forceinline__ void fan_store16(const PeerFan& pf, float4* p, float4 v) {
    if (MC_ONLY || pf.mc) {
        *p = v;
        asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                     ::"l"(reinterpret_cast<char*>(p) + pf.mc_delta), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    } else {
        fan_store(pf, p, v);
    }
}
template <bool MC_ONLY = false>
__device__ __forceinline__ void fan_store8(const PeerFan& pf, float2* p, float2 v) {
    if (MC_ONLY || pf.mc) {
        *p = v;
        asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};"
                     ::"l"(reinterpret_cast<char*>(p) + pf.mc_delta), "f"(v.x), "f"(v.y) : "memory");
    } else {
        fan_store(pf, p, v);
    }
}

// quad version: lane k in {0,1,2} owns Philox block k (4 normals, drawn by quad_obs_noise at the TOP of the kernel, under
// the shadow of the state loads) and writes obs[4k..4k+3]; lane 3 writes the last action.  `eu_k` = this lane's euler angle
// (lane0 roll, lane1 pitch, lane2 yaw), already wrapped.
template <uint32_t K = 0>
__device__ __forceinline__ void quad_obs_noise(const wl_config& c, int w, uint32_t gid, uint32_t t, uint32_t stream, uint32_t sub0, float z[4]) {
    z[0] = z[1] = z[2] = z[3] = 0.0f;
    if (Spec<K>::noise(c)) {
        uint4 r = philox4x32(c.seed, gid, t, stream, sub0 + (uint32_t)(w < 3 ? w : 0));
        box_muller(r.x, r.y, z[0], z[1]);
        box_muller(r.z, r.w, z[2], z[3]);
    }
}
// this lane's slice of the 14-float row: lanes 0..2 four floats (obs[4w..4w+3], noise added), lane 3 the two last-action floats
// SEL: every lane evaluates the same sums and selects its slice, with no lane-divergent region.
template <bool SEL = false>
__device__ __forceinline__ float4 blind_obs_quad_values(const wl_config& c, const EnvState& e, int w, float eu_k, V3 vb, V3 wb, const float z[4]) {
    const unsigned base = (threadIdx.x & 31u) & ~3u;
    float eu1 = __shfl_sync(0xffffffffu, eu_k, base + 1), eu2 = __shfl_sync(0xffffffffu, eu_k, base + 2);
    if (SEL) {
        const bool w0 = w == 0, w1 = w == 1;
        const float n0 = c.noise_std[0], n1 = c.noise_std[1], n2 = c.noise_std[2], n3 = c.noise_std[3];
        const float4 v = make_float4((w0 ? e.p.x : w1 ? eu1 : vb.z) + (w0 ? n0 : w1 ? n1 : n2) * z[0],
                                     (w0 ? e.p.y : w1 ? eu2 : wb.x) + (w0 ? n0 : w1 ? n1 : n3) * z[1],
                                     (w0 ? e.p.z : w1 ? vb.x : wb.y) + (w0 ? n0 : w1 ? n2 : n3) * z[2],
                                     (w0 ? eu_k : w1 ? vb.y : wb.z) + (w0 ? n1 : w1 ? n2 : n3) * z[3]);
        return (w == 3) ? make_float4(r_clamp(e.action[0], -1.0f, 1.0f), r_clamp(e.action[1], -1.0f, 1.0f), 0.0f, 0.0f) : v;
    }
    float b0, b1, b2, b3, s0, s1, s2, s3;
    if (w == 0) { b0 = e.p.x; b1 = e.p.y; b2 = e.p.z; b3 = eu_k; s0 = s1 = s2 = c.noise_std[0]; s3 = c.noise_std[1]; }
    else if (w == 1) { b0 = eu1; b1 = eu2; b2 = vb.x; b3 = vb.y; s0 = s1 = c.noise_std[1]; s2 = s3 = c.noise_std[2]; }
    else if (w == 2) { b0 = vb.z; b1 = wb.x; b2 = wb.y; b3 = wb.z; s0 = c.noise_std[2]; s1 = s2 = s3 = c.noise_std[3]; }
    else { return make_float4(r_clamp(e.action[0], -1.0f, 1.0f), r_clamp(e.action[1], -1.0f, 1.0f), 0.0f, 0.0f); }
    return make_float4(b0 + s0 * z[0], b1 + s1 * z[1], b2 + s2 * z[2], b3 + s3 * z[3]);
}
__device__ __forceinline__ void blind_obs_quad(const wl_config& c, const EnvState& e, int w, float eu_k, V3 vb, V3 wb, const float z[4],
                                               float* __restrict__ obs, bool live, const PeerFan& pf) {
    const float4 v = blind_obs_quad_values(c, e, w, eu_k, vb, wb, z);
    float2* o2 = reinterpret_cast<float2*>(obs + 4 * w);
    if (!live) return;
    fan_store(pf, &o2[0], make_float2(v.x, v.y));
    if (w < 3) fan_store(pf, &o2[1], make_float2(v.z, v.w));
}
__device__ __forceinline__ void blind_obs_quad(const wl_config& c, const EnvState& e, int w, float eu_k, V3 vb, V3 wb, const float z[4],
                                               float* __restrict__ obs, bool live) {
    const float4 v = blind_obs_quad_values(c, e, w, eu_k, vb, wb, z);
    float2* o2 = reinterpret_cast<float2*>(obs + 4 * w);
    if (!live) return;
    o2[0] = make_float2(v.x, v.y);
    if (w < 3) o2[1] = make_float2(v.z, v.w);
}

}  // namespace wl
