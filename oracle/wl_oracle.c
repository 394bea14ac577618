/*
 * wl_oracle.c -- CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * A plain-C, one-env-at-a-time restatement of the vectorised WheeledLab step that
 * wheeledlab_b200's CUDA kernels implement.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference leg may load this library; the
 * product path never does.
 *
 * PARITY STATUS (see DESIGN.md "Oracle"):
 *   - MDP term math (actions, rewards, terminations, reset poses, curriculum, obs
 *     assembly) follows the reference files cited at each function and is PINNED by
 *     golden vectors generated from the reference's own Python
 *     (tests/golden/, tests/golden/make_golden.py).
 *   - The rigid-body / tyre / actuator integrator stands in for PhysX-5 (closed
 *     binary, absent from the reference sources and not installable offline): PARITY UNPINNED at
 *     the PhysX boundary.  The model is builder-defined (DESIGN.md "Physics model").
 *   - Visual task camera: the post-processing (crop, ColorJitter, GaussianBlur, Grayscale, Normalize) is PINNED by
 *     golden vectors from the reference's own torchvision functions; the renderer that feeds it stands in for the RTX
 *     tiled camera (not available): PARITY UNPINNED at the pixel level (DESIGN.md 6c).
 *
 * Arithmetic contract shared with the CUDA path (so results are bit-identical):
 * IEEE fp32, no FMA contraction (-ffp-contract=off here, -fmad=false there),
 * correctly rounded / and sqrt, and the polynomial sin/cos/atan/log below instead
 * of libm.  Build with -DWLO_DOUBLE for a float64 "truth" variant (libm) used by the
 * tolerance tests.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <stddef.h>

#include "../include/wheeledlab_b200.h"

#ifdef WLO_DOUBLE
typedef double real;
#define K(x) x
#define r_sqrt sqrt
#define r_fabs fabs
#define r_floor floor
#else
typedef float real;
#define K(x) x##f
#define r_sqrt sqrtf
#define r_fabs fabsf
#define r_floor floorf
#endif

#define PI_R K(3.14159265358979323846)
#define TWO_PI_R K(6.28318530717958647692)
#define HALF_PI_R K(1.57079632679489661923)

static inline real r_min(real a, real b) { return a < b ? a : b; }
static inline real r_max(real a, real b) { return a > b ? a : b; }
static inline real r_clamp(real x, real lo, real hi) { return r_min(r_max(x, lo), hi); }

/* ------------------------------------------------------------------------- */
/* Philox4x32-10 (Salmon et al. 2011), counter = (global env id, step, stream, sub) */
/* ------------------------------------------------------------------------- */
#define RNG_OBS 0u
#define RNG_RESET 1u
#define RNG_PUSH_HF 3u
#define RNG_PUSH_LF 4u
#define RNG_ACTION 5u
#define RNG_STARTUP 6u
#define RNG_OBS_EXTRA 7u
#define RNG_CMD 8u
#define RNG_CAM 10u
#define RNG_CAM_EXTRA 11u

static void philox4x32(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t out[4]) {
    uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
/* [0,1) with 24 random bits (exact in fp32) */
static inline real u01(uint32_t x) { return (real)(x >> 8) * K(5.9604644775390625e-08); }
/* (0,1] */
static inline real u01_open(uint32_t x) { return (real)((x >> 8) + 1u) * K(5.9604644775390625e-08); }
/* fm(a,b,c) = round(a*b + c), one rounding: mirrors __fmaf_rn on the device */
#ifdef WLO_DOUBLE
static inline real fm(real a, real b, real c) { return fma(a, b, c); }
#else
static inline real fm(real a, real b, real c) { return fmaf(a, b, c); }
#endif
static inline real uniform(uint32_t x, real lo, real hi) { return fm(hi - lo, u01(x), lo); }

/* ------------------------------------------------------------------------- */
/* deterministic elementary functions (cephes single-precision kernels)      */
/* ------------------------------------------------------------------------- */
#ifdef WLO_DOUBLE
static void det_sincos(real x, real* s, real* c) { *s = sin(x); *c = cos(x); }
static real det_atan(real x) { return atan(x); }
static real det_atan_ratio(real num, real den) { return atan(num / den); }
static real det_sin_0_pi(real x) { return sin(x); }
static real det_atan2(real y, real x) { return atan2(y, x); }
static real det_log(real x) { return log(x); }
static real det_exp(real x) { return exp(x); }
#else
static void det_sincos(float x, float* s, float* c) {
    float q = floorf(fm(x, 0.63661977236758134f, 0.5f));
    float y = fm(-q, 1.5703125f, x);
    y = fm(-q, 4.837512969970703125e-4f, y);
    y = fm(-q, 7.54978995489188216e-8f, y);
    int qi = (int)q;
    float z = y * y;
    float ps = fm(fm(-1.9515295891e-4f, z, 8.3321608736e-3f), z, -1.6666654611e-1f);
    float sp = fm(ps * z, y, y);
    float pc = fm(fm(2.443315711809948e-5f, z, -1.388731625493765e-3f), z, 4.166664568298827e-2f);
    float cp = fm(pc * z, z, fm(-0.5f, z, 1.0f));
    switch (qi & 3) {
        case 0: *s = sp; *c = cp; break;
        case 1: *s = cp; *c = -sp; break;
        case 2: *s = -sp; *c = -cp; break;
        default: *s = -cp; *c = sp; break;
    }
}
/* sin(x), x in [0, pi]: fold to [0, pi/2], degree-9 odd polynomial (|err| <= 1.5e-7) */
static float det_sin_0_pi(float x) {
    float xr = (x > 1.57079632679489661923f) ? (3.14159265358979323846f - x) : x;
    float z = xr * xr;
    float q = fm(fm(fm(2.590488293208182e-06f, z, -1.9800897280219942e-04f), z, 8.332899771630764e-03f), z, -1.6666647791862488e-01f);
    return fm(xr * z, q, xr);
}
/* atan(num/den), num >= 0, den > 0, with one division (cephes ranges applied to the ratio) */
static float det_atan_ratio(float num, float den) {
    float y0, x;
    if (num > 2.414213562373095f * den) { y0 = 1.5707963267948966f; x = -(den / num); }
    else if (num > 0.4142135623730950f * den) { y0 = 0.7853981633974483f; x = (num - den) / (num + den); }
    else { y0 = 0.0f; x = num / den; }
    float z = x * x;
    float p = fm(fm(fm(8.05374449538e-2f, z, -1.38776856032e-1f), z, 1.99777106478e-1f), z, -3.33329491539e-1f);
    return y0 + fm(p * z, x, x);
}
static float det_atan(float xx) {
    float r = det_atan_ratio(fabsf(xx), 1.0f);
    return (xx < 0.0f) ? -r : r;
}
static float det_atan2(float y, float x) {
    if (x == 0.0f) {
        if (y > 0.0f) return 1.5707963267948966f;
        if (y < 0.0f) return -1.5707963267948966f;
        return 0.0f;
    }
    float r = det_atan_ratio(fabsf(y), fabsf(x));
    if ((y < 0.0f) != (x < 0.0f)) r = -r;
    if (x < 0.0f) r = (y >= 0.0f) ? r + 3.14159265358979323846f : r - 3.14159265358979323846f;
    return r;
}
static float det_log(float xin) {
    uint32_t bits; memcpy(&bits, &xin, 4);
    int e = (int)((bits >> 23) & 0xffu) - 126;
    bits = (bits & 0x807fffffu) | 0x3f000000u;
    float x; memcpy(&x, &bits, 4);
    if (x < 0.707106781186547524f) { e -= 1; x = x + x - 1.0f; } else { x = x - 1.0f; }
    float z = x * x;
    float p = fm(7.0376836292e-2f, x, -1.1514610310e-1f);
    p = fm(p, x, 1.1676998740e-1f); p = fm(p, x, -1.2420140846e-1f); p = fm(p, x, 1.4249322787e-1f);
    p = fm(p, x, -1.6668057665e-1f); p = fm(p, x, 2.0000714765e-1f); p = fm(p, x, -2.4999993993e-1f);
    p = fm(p, x, 3.3333331174e-1f);
    float y = p * x * z;
    float fe = (float)e;
    y = fm(-2.12194440e-4f, fe, y);
    y = fm(-0.5f, z, y);
    float r = x + y;
    return fm(0.693359375f, fe, r);
}
/* exp(x), x <= 0 (cephes expf) */
static float det_exp(float x) {
    if (x < -87.0f) return 0.0f;
    float n = floorf(fm(x, 1.44269504088896341f, 0.5f));
    float r = fm(-n, 0.693359375f, x);
    r = fm(n, 2.12194440e-4f, r);
    float z = r * r;
    float p = fm(1.9875691500e-4f, r, 1.3981999507e-3f);
    p = fm(p, r, 8.3334519073e-3f); p = fm(p, r, 4.1665795894e-2f); p = fm(p, r, 1.6666665459e-1f); p = fm(p, r, 5.0000001201e-1f);
    float y = fm(p, z, r) + 1.0f;
    uint32_t bits = (uint32_t)((int)n + 127) << 23;
    float sc; memcpy(&sc, &bits, 4);
    return y * sc;
}
#endif
static real det_tan(real x) { real s, c; det_sincos(x, &s, &c); return s / c; }
static real det_asin(real x) { return det_atan2(x, r_sqrt((K(1.0) - x) * (K(1.0) + x))); }
/* tanh (cephes tanhf): odd polynomial below 0.625, 1 - 2 / (exp(2|x|) + 1) above, +-1 beyond 9 */
#ifdef WLO_DOUBLE
static real det_tanh(real x) { return tanh(x); }
#else
static float det_tanh(float x) {
    float a = fabsf(x), r;
    if (a > 9.0f) r = 1.0f;
    else if (a >= 0.625f) { float e = det_exp(a + a); r = 1.0f - 2.0f / (e + 1.0f); }
    else {
        float z = a * a;
        float p = fm(fm(fm(fm(-5.70498872745e-3f, z, 2.06390887954e-2f), z, -5.37397155531e-2f), z, 1.33314422036e-1f), z, -3.33332819422e-1f);
        r = fm(p * z, a, a);
    }
    return (x < 0.0f) ? -r : r;
}
#endif

/* two standard normals from two u32 (Box-Muller) */
static void box_muller(uint32_t a, uint32_t b, real* z0, real* z1) {
    real u1 = u01_open(a), u2 = u01(b);
    real r = r_sqrt(K(-2.0) * det_log(u1));
    real s, c; det_sincos(TWO_PI_R * u2, &s, &c);
    *z0 = r * c; *z1 = r * s;
}

/* ------------------------------------------------------------------------- */
/* per-env state (AoS here on purpose: readable; the product is AoSoA float4)  */
/* ------------------------------------------------------------------------- */
typedef struct {
    real p[3], q[4], v[3], w[3];            /* root link pos, quat wxyz, COM lin vel (world), ang vel (world) */
    real omega[4];                          /* wheel spin [bl,br,fl,fr] */
    real steer[2], steer_vel[2];            /* front left/right steer joint */
    real action[2], prev_action[2];
    int32_t ep_len;
    real t_hf, t_lf;
    real sums[WL_MAX_REW_TERMS];
    real mass, inv_mass, spare0, spare1;
    real D[4], C[4], kd[4];
    real inv_Iw[4];   /* 1 / wheel spin inertia (wheel-mass DR, visual :290-299) */
    real cmd[4];      /* elevation: goal x,y (world), heading_w, command time_left */
    real cmdb[4];     /* elevation: command in the yaw frame x,y, heading_b, spare */
} wlo_env;

typedef struct wlo_sim {
    wl_config cfg;
    wlo_env* env;
    real rew_weight[WL_MAX_REW_TERMS];
    double log_sum[WL_MAX_REW_TERMS];     /* last step: sum over reset envs of episode sums */
    double log_term[8];                   /* last step: #reset, then per termination term counts */
    int32_t any_reset_last;
    float* hf;
    int32_t* vis_cells;       /* visual: spawn-candidate cell ids */
    uint8_t* vis_map;         /* visual: traversability map [rows, cols] */
} wlo_sim;

static inline real dot3(real ax, real ay, real az, real bx, real by, real bz) { return fm(ax, bx, fm(ay, by, az * bz)); }
static void rotmat(const real q[4], real R[9]) {
    real w = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = fm(K(-2.0), fm(y, y, z * z), K(1.0)); R[1] = K(2.0) * fm(x, y, -(w * z)); R[2] = K(2.0) * fm(x, z, w * y);
    R[3] = K(2.0) * fm(x, y, w * z); R[4] = fm(K(-2.0), fm(x, x, z * z), K(1.0)); R[5] = K(2.0) * fm(y, z, -(w * x));
    R[6] = K(2.0) * fm(x, z, -(w * y)); R[7] = K(2.0) * fm(y, z, w * x); R[8] = fm(K(-2.0), fm(x, x, y * y), K(1.0));
}
/* out = R a   /   out = R^T a */
static void rot(const real R[9], const real a[3], real o[3]) {
    o[0] = dot3(R[0], R[1], R[2], a[0], a[1], a[2]);
    o[1] = dot3(R[3], R[4], R[5], a[0], a[1], a[2]);
    o[2] = dot3(R[6], R[7], R[8], a[0], a[1], a[2]);
}
static void rotT(const real R[9], const real a[3], real o[3]) {
    o[0] = dot3(R[0], R[3], R[6], a[0], a[1], a[2]);
    o[1] = dot3(R[1], R[4], R[7], a[0], a[1], a[2]);
    o[2] = dot3(R[2], R[5], R[8], a[0], a[1], a[2]);
}
static void cross(const real a[3], const real b[3], real o[3]) {
    o[0] = fm(a[1], b[2], -(a[2] * b[1]));
    o[1] = fm(a[2], b[0], -(a[0] * b[2]));
    o[2] = fm(a[0], b[1], -(a[1] * b[0]));
}
static inline real vdot(const real a[3], const real b[3]) { return dot3(a[0], a[1], a[2], b[0], b[1], b[2]); }

/* ------------------------------------------------------------------------- */
/* terrain: height z and unit normal n at world (x,y)                          */
/* Drift/Visual: plane z=0 (mushr_drift_env_cfg.py:39-51).                     */
/* Elevation: bilinear height-field (raster of Terrains/huge_compact.usd or    */
/* procedural), ground plane hf_outside_z outside the raster                   */
/* (elevation/mushr_elevation_env_cfg.py:95-128).                              */
/* ------------------------------------------------------------------------- */
static inline real hf_at(const wlo_sim* s, int ix, int iy) { return (real)s->hf[(size_t)iy * s->cfg.hf_pitch + ix]; }

/* returns 1 when (x,y) is inside the raster */
static int hf_sample(const wlo_sim* s, real x, real y, real* z, real* gx, real* gy) {
    const wl_config* c = &s->cfg;
    real inv = K(1.0) / (real)c->hf_cell;
    real fx = (x - (real)c->hf_x0) * inv, fy = (y - (real)c->hf_y0) * inv;
    if (!(fx >= K(0.0)) || !(fy >= K(0.0)) || !(fx <= (real)(c->hf_nx - 1)) || !(fy <= (real)(c->hf_ny - 1))) return 0;
    int ix = (int)r_floor(fx), iy = (int)r_floor(fy);
    if (ix > c->hf_nx - 2) ix = c->hf_nx - 2;
    if (iy > c->hf_ny - 2) iy = c->hf_ny - 2;
    real tx = fx - (real)ix, ty = fy - (real)iy;
    real z00 = hf_at(s, ix, iy), z10 = hf_at(s, ix + 1, iy), z01 = hf_at(s, ix, iy + 1), z11 = hf_at(s, ix + 1, iy + 1);
    real za = fm(z10 - z00, tx, z00), zb = fm(z11 - z01, tx, z01);
    *z = fm(zb - za, ty, za);
    *gx = fm((z11 - z01) - (z10 - z00), ty, z10 - z00) * inv;
    *gy = (zb - za) * inv;
    return 1;
}
static void terrain(const wlo_sim* s, real x, real y, real* z, real n[3]) {
    if (s->cfg.task == WL_TASK_ELEVATION && s->hf) {
        real gx, gy;
        if (hf_sample(s, x, y, z, &gx, &gy)) {
            real inv = K(1.0) / r_sqrt(fm(gx, gx, fm(gy, gy, K(1.0))));
            n[0] = -gx * inv; n[1] = -gy * inv; n[2] = inv;
            return;
        }
        *z = (real)s->cfg.hf_outside_z;
    } else {
        *z = K(0.0);
    }
    n[0] = K(0.0); n[1] = K(0.0); n[2] = K(1.0);
}

/* ------------------------------------------------------------------------- */
/* A. action term.  ackermann_actions.py:119-133 (process), :136-145 (apply), */
/*    rc_car_actions.py:12-29 (RWD), :36-64 (4WD), ackermann_actions.py:150-201 */
/* ------------------------------------------------------------------------- */
static int process_action(const wl_config* c, const float a_in[2], real wheel_target[4], real steer_target[2]) {
    real a0 = (real)a_in[0], a1 = (real)a_in[1];
    if (c->bounding == WL_BOUND_CLIP) { a0 = r_clamp(a0, K(-1.0), K(1.0)); a1 = r_clamp(a1, K(-1.0), K(1.0)); }
    else if (c->bounding == WL_BOUND_TANH) { a0 = det_tanh(a0); a1 = det_tanh(a1); }      /* ackermann_actions.py:126-127 */
    else if (c->bounding != WL_BOUND_NONE) return WL_EUNSUPPORTED;
    real v = a0 * (real)c->act_scale[0] + (real)c->act_offset[0];
    real delta = a1 * (real)c->act_scale[1] + (real)c->act_offset[1];
    if (c->no_reverse) v = r_max(v, K(0.0));
    real tan_d = det_tan(delta);
    real L = (real)c->base_length, W = (real)c->base_width, r = (real)c->wheel_radius_cfg;
    if (c->action_kind == WL_ACT_RWD) {
        real wt = v * (real)c->d_inv_wheel_radius_cfg;
        wheel_target[WL_BL] = wt; wheel_target[WL_BR] = wt; wheel_target[WL_FL] = K(0.0); wheel_target[WL_FR] = K(0.0);
        steer_target[0] = tan_d; steer_target[1] = tan_d;      /* quirk Q1: tan(delta) is the position target */
        return 0;
    }
    real Rt = (tan_d == K(0.0)) ? K(1.0e6) : L / tan_d;
    real hw = W / K(2.0);
    real Rl = Rt - hw, Rr = Rt + hw;
    real Rrl = r_sqrt(Rl * Rl + L * L), Rrr = r_sqrt(Rr * Rr + L * L);
    real rden = K(1.0) / (Rt * r);
    wheel_target[WL_FL] = v * r_fabs(Rrl * rden);
    wheel_target[WL_FR] = v * r_fabs(Rrr * rden);
    wheel_target[WL_BL] = v * r_fabs(Rl * rden);
    wheel_target[WL_BR] = v * r_fabs(Rr * rden);
    if (c->action_kind == WL_ACT_4WD) { steer_target[0] = tan_d; steer_target[1] = tan_d; }
    else { steer_target[0] = det_atan(L / Rl); steer_target[1] = det_atan(L / Rr); }
    return 0;
}

/* ------------------------------------------------------------------------- */
/* a7 DC motor (hound.py:13-21,40-43; IsaacLab DCMotor._clip_effort [UPSTREAM-RECALL]) */
/* ------------------------------------------------------------------------- */
static real dc_motor(const wl_config* c, real kd, real effort_limit, real target, real omega) {
    if (!(effort_limit > K(0.0))) return K(0.0);        /* passive joint, hound.py:44-51 */
    real tau = kd * (target - omega);                    /* stiffness = 0 */
    real sat = (real)c->dc_saturation;
    real ratio = omega * (real)c->d_inv_dc_vel_limit;
    real max_eff = r_clamp(sat * (K(1.0) - ratio), K(0.0), effort_limit);
    real min_eff = r_clamp(sat * (K(-1.0) - ratio), -effort_limit, K(0.0));
    return r_clamp(tau, min_eff, max_eff);
}

/* ------------------------------------------------------------------------- */
/* a8 one integrator sub-step of length h (builder-defined model, DESIGN.md)    */
/* body-frame quantities: vb, wb; pc = COM position (world)                     */
/* ------------------------------------------------------------------------- */
typedef struct { real pc[3]; real q[4]; real v[3]; real wb[3]; } chassis_t;
/* mass-dependent per-env invariants; everything else comes from the d_* derived config fields */
typedef struct { real I[3], invI[3]; real hI[4], idk[4], fxk[4]; } step_consts;

static void make_step_consts(const wl_config* c, const wlo_env* e, step_consts* k) {
    real ms = e->mass * (real)c->d_inv_mass_nominal;     /* inertia scales with the mass ratio (a14) */
    real ms_inv = (real)c->mass_nominal * e->inv_mass;
    for (int a = 0; a < 3; ++a) { k->I[a] = (real)c->inertia_nominal[a] * ms; k->invI[a] = (real)c->d_invI_nominal[a] * ms_inv; }
    /* implicit DC-motor damper (DESIGN.md 3): h / I_w per wheel and 1 / (1 + h kd / I_w), constant over the env step */
    for (int i = 0; i < 4; ++i) {
        k->hI[i] = c->dr_wheel_mass_enable ? (real)c->d_h * e->inv_Iw[i] : (real)c->d_hI;
        k->idk[i] = K(1.0) / fm(k->hI[i], e->kd[i], K(1.0));
        /* longitudinal stick cap (tire_mx / h) with this wheel's own spin inertia */
        k->fxk[i] = c->dr_wheel_mass_enable
                        ? (real)c->d_inv_h / fm((real)c->wheel_radius * (real)c->wheel_radius, e->inv_Iw[i], (real)c->tire_mx_rest)
                        : (real)c->d_fxk;
    }
}
/* DCMotor speed-dependent effort limits (same clip as dc_motor), evaluated once per physics step like IsaacLab does */
static void dc_limits(const wl_config* c, real effort_limit, real omega, real* lo, real* hi) {
    if (!(effort_limit > K(0.0))) { *lo = K(0.0); *hi = K(0.0); return; }
    real sat = (real)c->dc_saturation;
    real ratio = omega * (real)c->d_inv_dc_vel_limit;
    *hi = r_clamp(sat * (K(1.0) - ratio), K(0.0), effort_limit);
    *lo = r_clamp(sat * (K(-1.0) - ratio), -effort_limit, K(0.0));
}

/* derived constants: same fp32 operations, same order, as wl_config_finalize() in the product library */
static void config_finalize(wl_config* c) {
    c->d_h = c->sim_dt / (float)c->substeps;
    c->d_inv_h = 1.0f / c->d_h;
    c->d_step_dt = c->sim_dt * (float)c->decimation;
    c->d_hkp = c->d_h * c->steer_kp;
    c->d_sden = 1.0f / fmaf(c->d_h, c->d_hkp, fmaf(c->d_h, c->steer_kd, c->steer_inertia));
    c->d_inv_Iw = 1.0f / c->wheel_inertia;
    c->d_hI = c->d_h * c->d_inv_Iw;
    c->d_inv_hf_cell = c->hf_cell > 0.0f ? 1.0f / c->hf_cell : 0.0f;
    c->d_fxk = c->tire_mx * c->d_inv_h;
    c->d_fyk = c->tire_my * c->d_inv_h;
    c->d_inv_wheel_radius_cfg = 1.0f / c->wheel_radius_cfg;
    c->d_inv_dc_vel_limit = 1.0f / c->dc_vel_limit;
    c->d_inv_mass_nominal = 1.0f / c->mass_nominal;
    for (int a = 0; a < 3; ++a) c->d_invI_nominal[a] = 1.0f / c->inertia_nominal[a];
    c->d_vis_mesh_inv_dx = c->vis_mesh_dx > 0.0f ? 1.0f / c->vis_mesh_dx : 0.0f;
    c->d_vis_mesh_inv_dy = c->vis_mesh_dy > 0.0f ? 1.0f / c->vis_mesh_dy : 0.0f;
}

static void physics_substep(const wlo_sim* s, wlo_env* e, chassis_t* b, const real wheel_target[4], const real eff_lo[4],
                            const real eff_hi[4], const real steer_target[2], const step_consts* k) {
    const wl_config* c = &s->cfg;
    real h = (real)c->d_h;
    real R[9]; rotmat(b->q, R);
    /* steering: implicit PD on the steer joint (hound.py:5-12) */
    real sn[2], cs[2];
    for (int j = 0; j < 2; ++j) {
        real vel = fm((real)c->d_hkp, steer_target[j] - e->steer[j], (real)c->steer_inertia * e->steer_vel[j]) * (real)c->d_sden;
        vel = r_clamp(vel, -(real)c->steer_vel_limit, (real)c->steer_vel_limit);
        real pos = r_clamp(fm(h, vel, e->steer[j]), -(real)c->steer_pos_limit, (real)c->steer_pos_limit);
        e->steer_vel[j] = vel; e->steer[j] = pos;
        det_sincos(pos, &sn[j], &cs[j]);
    }
    real vb[3]; rotT(R, b->v, vb);
    real F[4][3], T[4][3];
    real rw = (real)c->wheel_radius, bw = (real)c->wheel_damping;
    for (int i = 0; i < 4; ++i) {
        real rho[3];
        rho[0] = ((i >= 2) ? (real)c->hub_x_front : (real)c->hub_x_rear) - (real)c->com[0];
        rho[1] = ((i & 1) ? -(real)c->hub_y : (real)c->hub_y) - (real)c->com[1];
        rho[2] = (real)c->hub_z - (real)c->com[2];
        real comp, nb[3];
        if (c->task == WL_TASK_ELEVATION) {
            real hubw[3]; rot(R, rho, hubw);
            hubw[0] += b->pc[0]; hubw[1] += b->pc[1]; hubw[2] += b->pc[2];
            real zt, nw[3]; terrain(s, hubw[0], hubw[1], &zt, nw);
            comp = fm(-(hubw[2] - zt), nw[2], rw);
            rotT(R, nw, nb);
        } else {                                     /* plane z = 0 */
            real hz = dot3(R[6], R[7], R[8], rho[0], rho[1], rho[2]) + b->pc[2];
            comp = rw - hz;
            nb[0] = R[6]; nb[1] = R[7]; nb[2] = R[8];
        }
        /* drive torque first, then friction against the resulting slip (implicit stick, DESIGN.md).  The DCMotor damper
         * tau = kd (w_t - w) is stiff (kd h / I_w >> 1), so it is integrated implicitly in the new wheel speed; when the
         * resulting torque leaves the motor's effort limits the clipped torque is applied explicitly instead. */
        real os = fm(k->hI[i], fm(e->kd[i], wheel_target[i], -(bw * e->omega[i])), e->omega[i]) * k->idk[i];
        real t_imp = e->kd[i] * (wheel_target[i] - os);
        real tc = r_clamp(t_imp, eff_lo[i], eff_hi[i]);
        real om_star = (tc == t_imp) ? os : fm(k->hI[i], tc - bw * e->omega[i], e->omega[i]);
        real rc[3] = {fm(-rw, nb[0], rho[0]), fm(-rw, nb[1], rho[1]), fm(-rw, nb[2], rho[2])};
        real vc[3]; cross(b->wb, rc, vc);
        vc[0] += vb[0]; vc[1] += vb[1]; vc[2] += vb[2];
        real sdot = -vdot(nb, vc);
        real ce = r_min(comp, (real)c->comp_max);     /* depenetration cap */
        real Fz = fm((real)c->susp_k, ce, (real)c->susp_c * sdot);
        if (ce > (real)c->susp_travel) Fz = fm((real)c->bump_k, ce - (real)c->susp_travel, Fz);
        Fz = (comp > K(0.0)) ? r_max(Fz, K(0.0)) : K(0.0);
        real ft[3];
        if (i >= 2) {
            real d = fm(cs[i - 2], nb[0], sn[i - 2] * nb[1]);
            ft[0] = fm(-d, nb[0], cs[i - 2]); ft[1] = fm(-d, nb[1], sn[i - 2]); ft[2] = -(d * nb[2]);
        } else {
            real d = nb[0];
            ft[0] = fm(-d, nb[0], K(1.0)); ft[1] = -(d * nb[1]); ft[2] = -(d * nb[2]);
        }
        /* |ft|^2 = 1 - d^2: binomial series of (1 - e)^(-1/2), e = 1 - |ft|^2 */
        real en = K(1.0) - vdot(ft, ft);
        real finv = fm(fm(fm(fm(K(0.2734375), en, K(0.3125)), en, K(0.375)), en, K(0.5)), en, K(1.0));
        ft[0] *= finv; ft[1] *= finv; ft[2] *= finv;
        real lt[3]; cross(nb, ft, lt);
        real vx = vdot(vc, ft), vy = vdot(vc, lt);
        real sx = fm(om_star, rw, -vx), sy = -vy;     /* slip velocity of the tyre surface */
        real smag = r_sqrt(r_max(fm(sx, sx, sy * sy), K(1.0e-24)));   /* |s| >= 1e-12: all operands below stay normal-range */
        real den = r_max(r_fabs(vx), (real)c->tire_v0);
        real sm = det_sin_0_pi(e->C[i] * det_atan_ratio((real)c->tire_B * smag, den));
        real Fmag = Fz * (e->D[i] * sm);
        real inv_s = K(1.0) / r_max(smag, K(1.0e-9));
        real Fx = (Fmag * sx) * inv_s, Fy = (Fmag * sy) * inv_s;
        real fxm = k->fxk[i] * r_fabs(sx), fym = (real)c->d_fyk * r_fabs(sy);
        Fx = r_clamp(Fx, -fxm, fxm); Fy = r_clamp(Fy, -fym, fym);
        for (int a = 0; a < 3; ++a) F[i][a] = fm(Fz, nb[a], fm(Fx, ft[a], Fy * lt[a]));
        cross(rc, F[i], T[i]);
        e->omega[i] = fm(-k->hI[i], rw * Fx, om_star);
    }
    real Fb[3], Tb[3];
    for (int a = 0; a < 3; ++a) { Fb[a] = (F[0][a] + F[1][a]) + (F[2][a] + F[3][a]); Tb[a] = (T[0][a] + T[1][a]) + (T[2][a] + T[3][a]); }
    /* chassis: semi-implicit Euler, Euler's equations in the body frame (gyroscopic term on, mushr.py:28) */
    real Fw[3]; rot(R, Fb, Fw);
    b->v[0] = fm(h, Fw[0] * e->inv_mass, b->v[0]);
    b->v[1] = fm(h, Fw[1] * e->inv_mass, b->v[1]);
    b->v[2] = fm(h, fm(Fw[2], e->inv_mass, -(real)c->gravity), b->v[2]);
    real Iw3[3] = {k->I[0] * b->wb[0], k->I[1] * b->wb[1], k->I[2] * b->wb[2]};
    real g[3]; cross(b->wb, Iw3, g);
    b->wb[0] = fm(h, (Tb[0] - g[0]) * k->invI[0], b->wb[0]);
    b->wb[1] = fm(h, (Tb[1] - g[1]) * k->invI[1], b->wb[1]);
    b->wb[2] = fm(h, (Tb[2] - g[2]) * k->invI[2], b->wb[2]);
    b->pc[0] = fm(h, b->v[0], b->pc[0]);
    b->pc[1] = fm(h, b->v[1], b->pc[1]);
    b->pc[2] = fm(h, b->v[2], b->pc[2]);
    real hh = K(0.5) * h;
    real qw = b->q[0], qx = b->q[1], qy = b->q[2], qz = b->q[3];
    real ox = b->wb[0], oy = b->wb[1], oz = b->wb[2];
    real nqw = fm(-hh, dot3(qx, qy, qz, ox, oy, oz), qw);
    real nqx = fm(hh, fm(qw, ox, fm(qy, oz, -(qz * oy))), qx);
    real nqy = fm(hh, fm(qw, oy, fm(qz, ox, -(qx * oz))), qy);
    real nqz = fm(hh, fm(qw, oz, fm(qx, oy, -(qy * ox))), qz);
    /* renormalise with the series of (1 + e)^(-1/2), e = |q|^2 - 1 */
    real eq = fm(nqw, nqw, fm(nqx, nqx, fm(nqy, nqy, nqz * nqz))) - K(1.0);
    real qinv = fm(fm(fm(K(-0.3125), eq, K(0.375)), eq, K(-0.5)), eq, K(1.0));
    b->q[0] = nqw * qinv; b->q[1] = nqx * qinv; b->q[2] = nqy * qinv; b->q[3] = nqz * qinv;
}

/* ------------------------------------------------------------------------- */
/* euler_xyz_from_quat [UPSTREAM-RECALL isaaclab.utils.math], each angle % 2pi */
/* used by root_euler_xyz, wheeledlab/envs/mdp/observations.py:9-12            */
/* ------------------------------------------------------------------------- */
static inline real wrap_2pi(real a) { return (a < K(0.0)) ? a + TWO_PI_R : a; }
static void euler_xyz(const real q[4], real e[3]) {
    real w = q[0], x = q[1], y = q[2], z = q[3];
    real sin_roll = K(2.0) * fm(w, x, y * z), cos_roll = fm(K(-2.0), fm(x, x, y * y), K(1.0));
    real sin_pitch = K(2.0) * fm(w, y, -(z * x));
    real sin_yaw = K(2.0) * fm(w, z, x * y), cos_yaw = fm(K(-2.0), fm(y, y, z * z), K(1.0));
    real pitch;
    if (r_fabs(sin_pitch) >= K(1.0)) pitch = (sin_pitch < K(0.0)) ? -HALF_PI_R : HALF_PI_R;
    else pitch = det_asin(sin_pitch);
    e[0] = wrap_2pi(det_atan2(sin_roll, cos_roll));
    e[1] = wrap_2pi(pitch);
    e[2] = wrap_2pi(det_atan2(sin_yaw, cos_yaw));
}

/* ------------------------------------------------------------------------- */
/* drift terminations.  mushr_drift_env_cfg.py:201-217 (in_range/off_track),  */
/* :343-348 (cart_off_track)                                                   */
/* ------------------------------------------------------------------------- */
static int drift_off_track(const wl_config* c, real x, real y) {
    real st = (real)c->trk_straight, ro = (real)c->trk_corner_out, ri = (real)c->trk_corner_in;
    int off, in;
    if (r_fabs(y) < st) { off = r_fabs(x) > ro; in = r_fabs(x) < ri; }
    else if (y > K(0.0)) {
        real d2 = (y - st) * (y - st) + x * x;
        off = d2 > ro * ro; in = d2 < ri * ri;
    } else {
        real d2 = (y + st) * (y + st) + x * x;
        off = d2 > ro * ro; in = d2 < ri * ri;
    }
    return off || in;
}

/* drift reward terms, mushr_drift_env_cfg.py:160-240; returns f_i (unweighted) */
static void drift_reward_terms(const wl_config* c, const wlo_env* e, const real p[3], const real vb[3], const real wb[3],
                               real wz_world, int out_of_bounds, int time_out, real f[WL_MAX_REW_TERMS]) {
    /* side_slip :219-230 (params :246-254) */
    real slip = r_fabs(det_atan2(vb[1], vb[0]));
    real valid = (r_fabs(vb[0]) < (real)c->slip_min_vel_x || slip > (real)c->slip_max_thresh) ? K(0.0) : slip;
    if (valid < (real)c->slip_min_thresh) valid = K(0.0);
    f[WL_DR_SIDE_SLIP] = valid;
    /* vel_dist :167-171 */
    real gs = r_sqrt(vb[0] * vb[0] + vb[1] * vb[1]);
    real dv = gs - (real)c->vel_speed_target;
    f[WL_DR_VEL] = dv * dv + (real)c->vel_offset;
    /* track_progress_rate :160-165: world yaw rate */
    f[WL_DR_PROGRESS] = wz_world;
    /* turn_left_go_right :232-240 */
    real sm = (e->steer[0] + e->steer[1]) / K(2.0);
    real av = r_clamp(wb[2], -(real)c->tlgr_ang_vel_thresh, (real)c->tlgr_ang_vel_thresh);
    real tl = sm * av * K(-1.0);
    f[WL_DR_TLGR] = r_max(tl, K(0.0));
    /* energy_through_turn :195-199 (3-D body speed, quirk Q7) */
    real sp = r_sqrt(vb[0] * vb[0] + vb[1] * vb[1] + vb[2] * vb[2]);
    f[WL_DR_TURN_ENERGY] = (r_fabs(p[1]) > (real)c->energy_straight) ? sp * sp : K(0.0);
    /* cross_track_dist :173-193 (p = 1) */
    real st = (real)c->trk_straight, tr = (real)c->ctd_track_radius, sq;
    if (r_fabs(p[1]) < st) {
        real d = (p[0] > K(0.0)) ? (p[0] - tr) : (p[0] + tr);
        sq = d * d;
    } else {
        real yy = (p[1] > K(0.0)) ? (p[1] - st) : (p[1] + st);
        real d = r_sqrt(yy * yy + p[0] * p[0]) - tr;
        sq = d * d;
    }
    f[WL_DR_CROSS_TRACK] = r_sqrt(sq) + (real)c->ctd_offset;
    /* is_terminated_term(["out_of_bounds"]) :295-299 [UPSTREAM-RECALL: * ~time_outs] */
    f[WL_DR_TERM_PENS] = (out_of_bounds && !time_out) ? K(1.0) : K(0.0);
    f[7] = K(0.0);
}

/* ------------------------------------------------------------------------- */
/* reset_root_state_along_track.__call__, drifting/mdp/events.py:102-133       */
/* ------------------------------------------------------------------------- */
static void sample_interval_timers(const wl_config* c, wlo_env* e, uint32_t a, uint32_t b) {
    e->t_hf = uniform(a, (real)c->push_hf_interval[0], (real)c->push_hf_interval[1]);
    e->t_lf = uniform(b, (real)c->push_lf_interval[0], (real)c->push_lf_interval[1]);
}
/* pose part of __call__ (events.py:119-131) from the raw draws: idx, u_x, u_y, u_yaw in [0,1) */
static void drift_reset_pose(const wl_config* c, wlo_env* e, uint32_t idx, real ux, real uy, real uyaw) {
    real nx = (K(2.0) * ux - K(1.0)) * (real)c->reset_pos_noise;
    real ny = (K(2.0) * uy - K(1.0)) * (real)c->reset_pos_noise;
    real nyaw = (K(2.0) * uyaw - K(1.0)) * (real)c->reset_yaw_noise;
    e->p[0] = (real)c->ref_poses[3 * idx + 0] + nx;
    e->p[1] = (real)c->ref_poses[3 * idx + 1] + ny;
    e->p[2] = K(0.0);
    real yaw = (real)c->ref_poses[3 * idx + 2] * K(0.017453292519943295) + nyaw;   /* deg2rad, :126 */
    real sh, ch; det_sincos(yaw * K(0.5), &sh, &ch);
    e->q[0] = ch; e->q[1] = K(0.0); e->q[2] = K(0.0); e->q[3] = sh;                 /* roll = pitch = 0 */
}
static void drift_reset_env(const wl_config* c, wlo_env* e, uint32_t gid, int64_t t) {
    uint32_t r[4], r2[4];
    philox4x32(c->seed, gid, (uint32_t)t, RNG_RESET, 0u, r);
    uint32_t idx = (uint32_t)(((uint64_t)r[0] * (uint64_t)c->num_ref_poses) >> 32);
    drift_reset_pose(c, e, idx, u01(r[1]), u01(r[2]), u01(r[3]));
    for (int k = 0; k < 3; ++k) { e->v[k] = K(0.0); e->w[k] = K(0.0); }
    /* joint state untouched (quirk Q3).  manager resets [UPSTREAM-RECALL Appendix B]: */
    e->ep_len = 0;
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) e->sums[k] = K(0.0);
    e->action[0] = e->action[1] = e->prev_action[0] = e->prev_action[1] = K(0.0);
    philox4x32(c->seed, gid, (uint32_t)t, RNG_RESET, 1u, r2);
    sample_interval_timers(c, e, r2[0], r2[1]);
}

/* ------------------------------------------------------------------------- */
/* elevation task, elevation/mushr_elevation_env_cfg.py                          */
/* ------------------------------------------------------------------------- */
/* terminations :339-376 -> mask bits [0 time_out,1 cart_out_of_bounds,2 stuck,3 rollover,4 at_goal]; rewards :283-305 */
static uint32_t elev_terms(const wl_config* c, const wlo_env* e, const real R[9], const real vb[3], real sum_omega, int time_out,
                           real f[WL_MAX_REW_TERMS]) {
    real gx = e->cmdb[0] - e->p[0], gy = e->cmdb[1] - e->p[1];        /* quirk Q5: yaw-frame command minus WORLD position */
    real gn = r_sqrt(fm(gx, gx, gy * gy));
    int oob = e->p[2] < (real)c->elev_min_height;                     /* root_height_below_minimum :354-357 */
    int stuck = (r_min(vb[0], K(1.2)) < (real)c->elev_stuck_min_vel) && (sum_omega > (real)c->elev_stuck_spin); /* :342-347 */
    int roll = R[8] < (real)c->elev_rollover_cos;                     /* upright_bool :217-222,339-340 */
    int goal = gn < (real)c->elev_goal_dist;                          /* close_to_goal :268-273 */
    f[WL_ER_GOAL_RATE] = K(5.0) + fm(e->v[0], gx, e->v[1] * gy) / gn; /* goal_progress_rate :239-249 */
    real zv = e->p[2] - (real)c->elev_plane_z;                        /* higher_elevation :166-173 */
    real he = ((zv > K(0.1)) && (vb[0] > K(0.1))) ? zv : K(0.0);
    f[WL_ER_HEIGHT_Z] = r_clamp(he, K(0.0), K(1.0));
    f[WL_ER_FALLING] = (vb[2] > (real)c->elev_fall_vel) ? K(1.0) : K(0.0);   /* is_falling_penalty :251-254 (2nd def) */
    f[WL_ER_TERM_PEN] = (stuck && !time_out) ? K(1.0) : K(0.0);      /* is_terminated_term("stuck") */
    f[4] = f[5] = f[6] = f[7] = K(0.0);
    return (time_out ? 1u : 0u) | (oob ? 2u : 0u) | (stuck ? 4u : 0u) | (roll ? 8u : 0u) | (goal ? 16u : 0u);
}
/* reset_root_state_uniform :409-419 on default root z 0.25 (:97,147-149) + manager resets + command resample :425-435 */
static void elev_reset_env(const wl_config* c, wlo_env* e, uint32_t gid, int64_t t) {
    uint32_t r[4], r2[4];
    philox4x32(c->seed, gid, (uint32_t)t, RNG_RESET, 0u, r);
    philox4x32(c->seed, gid, (uint32_t)t, RNG_RESET, 1u, r2);
    e->p[0] = uniform(r[0], (real)c->elev_reset_xy[0], (real)c->elev_reset_xy[1]);
    e->p[1] = uniform(r[1], (real)c->elev_reset_xy[0], (real)c->elev_reset_xy[1]);
    e->p[2] = (real)c->elev_spawn_z;
    real yaw = uniform(r[2], -(real)c->elev_reset_yaw, (real)c->elev_reset_yaw);
    real sh, ch; det_sincos(yaw * K(0.5), &sh, &ch);
    e->q[0] = ch; e->q[1] = K(0.0); e->q[2] = K(0.0); e->q[3] = sh;
    e->v[0] = uniform(r[3], (real)c->elev_reset_vel[0], (real)c->elev_reset_vel[1]);
    e->v[1] = uniform(r2[0], (real)c->elev_reset_vel[0], (real)c->elev_reset_vel[1]);
    e->v[2] = K(0.0);
    e->w[0] = e->w[1] = e->w[2] = K(0.0);
    e->ep_len = 0;
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) e->sums[k] = K(0.0);
    e->action[0] = e->action[1] = e->prev_action[0] = e->prev_action[1] = K(0.0);
    e->cmd[0] = uniform(r2[1], (real)c->cmd_pos_range[0], (real)c->cmd_pos_range[1]);
    e->cmd[1] = uniform(r2[2], (real)c->cmd_pos_range[0], (real)c->cmd_pos_range[1]);
    e->cmd[2] = K(0.0);
    e->cmd[3] = (real)c->cmd_resample_s;
}
static void yaw_cs(const wlo_env* e, real* cy, real* sy) {
    real cr = fm(K(-2.0), fm(e->q[2], e->q[2], e->q[3] * e->q[3]), K(1.0)), sr = K(2.0) * fm(e->q[0], e->q[3], e->q[1] * e->q[2]);
    real rinv = K(1.0) / r_sqrt(fm(cr, cr, sr * sr));
    *cy = cr * rinv; *sy = sr * rinv;
}
/* CommandManager.compute(dt) [UPSTREAM-RECALL]: timer, resample, yaw-frame command */
static void elev_command_update(const wl_config* c, wlo_env* e, uint32_t gid, int64_t t, real step_dt) {
    e->cmd[3] = e->cmd[3] - step_dt;
    if (e->cmd[3] <= K(0.0)) {
        uint32_t r[4]; philox4x32(c->seed, gid, (uint32_t)t, RNG_CMD, 0u, r);
        e->cmd[0] = uniform(r[0], (real)c->cmd_pos_range[0], (real)c->cmd_pos_range[1]);
        e->cmd[1] = uniform(r[1], (real)c->cmd_pos_range[0], (real)c->cmd_pos_range[1]);
        e->cmd[3] = (real)c->cmd_resample_s;
    }
    real cy, sy; yaw_cs(e, &cy, &sy);
    real dx = e->cmd[0] - e->p[0], dy = e->cmd[1] - e->p[1];
    e->cmdb[0] = fm(cy, dx, sy * dy);
    e->cmdb[1] = fm(cy, dy, -(sy * dx));
    e->cmdb[2] = K(0.0); e->cmdb[3] = K(0.0);
}
static void euler_xyz(const real q[4], real e[3]);
/* ElevationObsCfg (:50-88): 13 proprioceptive floats + 676-ray height map, all clipped, no noise */
static void elev_obs(const wlo_sim* s, const wlo_env* e, float* obs) {
    const wl_config* c = &s->cfg;
    real R[9]; rotmat(e->q, R);
    real vb[3], wb[3], eu[3]; rotT(R, e->v, vb); rotT(R, e->w, wb); euler_xyz(e->q, eu);
    real gx = e->cmdb[0] - e->p[0], gy = e->cmdb[1] - e->p[1];
    real cl = (real)c->obs_clip;
    obs[0] = (float)((gx != gx) ? K(0.0) : gx); obs[1] = (float)((gy != gy) ? K(0.0) : gy);
    for (int k = 0; k < 3; ++k) {
        obs[2 + k] = (float)eu[k];
        obs[5 + k] = (float)r_clamp(vb[k], -cl, cl);
        obs[8 + k] = (float)r_clamp(wb[k], -cl, cl);
    }
    obs[11] = (float)r_clamp(e->action[0], K(-1.0), K(1.0));
    obs[12] = (float)r_clamp(e->action[1], K(-1.0), K(1.0));
    /* ray-caster :132-142: 26x26 grid on base_link, yaw-only alignment, vertical rays vs the terrain raster */
    real bx = fm((real)c->base_link_z, R[2], e->p[0]), by = fm((real)c->base_link_z, R[5], e->p[1]), bz = fm((real)c->base_link_z, R[8], e->p[2]);
    real cy, sy; yaw_cs(e, &cy, &sy);
    for (int k = 0; k < WL_SCAN_RAYS; ++k) {
        int rx = k % WL_SCAN_SIDE, ry = k / WL_SCAN_SIDE;
        real lx = fm((real)rx, (real)c->scan_res, -(real)c->scan_half), ly = fm((real)ry, (real)c->scan_res, -(real)c->scan_half);
        real wx = fm(cy, lx, fm(-sy, ly, bx)), wy = fm(sy, lx, fm(cy, ly, by));
        real hit, gxx, gyy, v;
        if (hf_sample(s, wx, wy, &hit, &gxx, &gyy)) {
            real hs = bz - hit - (real)c->scan_offset;                              /* mdp.height_scan */
            v = r_clamp(-hs + (e->p[2] - (real)c->scan_plane_init), -cl, cl);       /* world_height_map :44-48 */
        } else {
            v = cl;                                                                 /* miss: +inf, clipped */
        }
        obs[13 + k] = (float)v;
    }
}

/* ------------------------------------------------------------------------- */
/* visual task, physics side (visual/mushr_visual_env_cfg.py; camera out of scope) */
/* ------------------------------------------------------------------------- */
/* rewards :304-387, terminations :392-409; map lookup = TraversabilityHashmapUtil.get_map_id
 * (utils/traversability_utils.py:83-88: +spacing/2, truncation toward zero, clamp, indexed [y_idx, x_idx]) */
static uint32_t visual_terms(const wlo_sim* s, const wlo_env* e, const real vb[3], int time_out, real f[WL_MAX_REW_TERMS]) {
    const wl_config* c = &s->cfg;
    int xi = (int)((e->p[0] + (real)c->vis_width / K(2.0) + (real)c->vis_row_spacing / K(2.0)) / (real)c->vis_row_spacing);
    int yi = (int)((e->p[1] + (real)c->vis_height / K(2.0) + (real)c->vis_col_spacing / K(2.0)) / (real)c->vis_col_spacing);
    xi = xi < 0 ? 0 : (xi > c->vis_rows - 1 ? c->vis_rows - 1 : xi);
    yi = yi < 0 ? 0 : (yi > c->vis_cols - 1 ? c->vis_cols - 1 : yi);
    int trav = s->vis_map[(size_t)yi * c->vis_cols + xi] != 0;
    f[WL_VR_TRAVERSABLE] = trav ? K(1.0) : K(-1.0);                       /* traversable_reward :309-312 */
    f[WL_VR_FORWARD_VEL] = vb[0];                                         /* forward_vel :371-372 */
    for (int k = 2; k < WL_MAX_REW_TERMS; ++k) f[k] = K(0.0);
    int out = (e->p[0] > (real)c->vis_width / K(2.0)) || (e->p[0] < -(real)c->vis_width / K(2.0)) ||
              (e->p[1] > (real)c->vis_height / K(2.0)) || (e->p[1] < -(real)c->vis_height / K(2.0));   /* out_of_map :392-400 */
    return (time_out ? 1u : 0u) | (out ? 2u : 0u);
}
/* reset_root_state (visual/mdp/events.py:11-42) + generate_random_poses (utils/__init__.py:188-202) */
static void visual_reset_env(const wlo_sim* s, wlo_env* e, uint32_t gid, int64_t t) {
    const wl_config* c = &s->cfg;
    uint32_t r[4]; philox4x32(c->seed, gid, (uint32_t)t, RNG_RESET, 0u, r);
    int cell = s->vis_cells[(uint32_t)(((uint64_t)r[0] * (uint64_t)c->vis_n_trav) >> 32)];
    int ys = cell / c->vis_cols, xs = cell - ys * c->vis_cols;
    e->p[0] = ((real)xs - (real)(c->vis_cols / 2)) * (real)c->vis_row_spacing;
    e->p[1] = ((real)ys - (real)(c->vis_rows / 2)) * (real)c->vis_col_spacing;
    e->p[2] = (real)c->vis_spawn_z;
    real yaw = (K(360.0) * u01(r[1])) * K(0.017453292519943295);
    real sh, ch; det_sincos(yaw * K(0.5), &sh, &ch);
    e->q[0] = ch; e->q[1] = K(0.0); e->q[2] = K(0.0); e->q[3] = sh;
    for (int k = 0; k < 3; ++k) { e->v[k] = K(0.0); e->w[k] = K(0.0); }
    e->ep_len = 0;
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) e->sums[k] = K(0.0);
    e->action[0] = e->action[1] = e->prev_action[0] = e->prev_action[1] = K(0.0);
}
static void visual_obs(const wlo_env* e, float* obs) {
    real R[9]; rotmat(e->q, R);
    real vb[3], wb[3]; rotT(R, e->v, vb); rotT(R, e->w, wb);
    for (int k = 0; k < 3; ++k) { obs[k] = (float)vb[k]; obs[3 + k] = (float)wb[k]; }
    obs[6] = (float)r_clamp(e->action[0], K(-1.0), K(1.0)); obs[7] = (float)r_clamp(e->action[1], K(-1.0), K(1.0));
}

/* ---- visual task, camera term: software pinhole camera over the 2-colour plane mesh ----------------------------------
 * Follows camera_data_rgb_flattened[_aug] (visual/mdp_sensors/observations.py:64-87): keep rows [H//3, H), (ColorJitter,
 * GaussianBlur(5),) Grayscale, Normalize(0.5, 0.5), flatten.  The RTX renderer is replaced by a ray / plane intersection
 * against the coloured mesh of utils/__init__.py:8-89 (unlit albedo; background = vis_cam_bg) -- the rendering model is
 * builder-defined (parity unpinned); the post-processing is pinned to the reference function by tests/golden. */
static int vis_cam_floats(const wl_config* c) { return c->vis_cam ? c->vis_cam_w * (c->vis_cam_h - c->vis_cam_row0) : 0; }
static real cam_gray(real v) { return fm(K(0.114), v, fm(K(0.587), v, K(0.2989) * v)); }
static real cam_clamp01(real v) { return r_min(r_max(v, K(0.0)), K(1.0)); }
typedef struct { real v0, v1, w0, w1, w2; } cam_aug_t;
static cam_aug_t cam_aug_params(const wl_config* c, uint32_t t, uint32_t stream, uint32_t sub, const float* aug, real p) {
    cam_aug_t A; A.v0 = K(0.0); A.v1 = K(1.0); A.w0 = K(1.0); A.w1 = K(0.0); A.w2 = K(0.0);
    if (c->vis_cam != 2) return A;
    real b, ct, sa, sigma; int order[4] = {0, 1, 2, 3};
    if (aug) {
        b = (real)aug[0]; ct = (real)aug[1]; sa = (real)aug[2]; sigma = (real)aug[4];
        for (int k = 0; k < 4; ++k) order[k] = (int)aug[5 + k];
    } else {
        uint32_t r[4], q[4];
        philox4x32(c->seed, 0u, t, stream, 2u * sub, r); philox4x32(c->seed, 0u, t, stream, 2u * sub + 1u, q);
        b = uniform(r[0], r_max(K(0.0), K(1.0) - (real)c->vis_aug_brightness), K(1.0) + (real)c->vis_aug_brightness);
        ct = uniform(r[1], r_max(K(0.0), K(1.0) - (real)c->vis_aug_contrast), K(1.0) + (real)c->vis_aug_contrast);
        sa = uniform(r[2], r_max(K(0.0), K(1.0) - (real)c->vis_aug_saturation), K(1.0) + (real)c->vis_aug_saturation);
        sigma = uniform(r[3], (real)c->vis_aug_sigma[0], (real)c->vis_aug_sigma[1]);
        for (int i = 3; i >= 1; --i) {
            int j = (int)(((uint64_t)q[3 - i] * (uint64_t)(i + 1)) >> 32);
            int tmp = order[i]; order[i] = order[j]; order[j] = tmp;
        }
    }
    for (int k = 0; k < 4; ++k) {
        int op = order[k];
        if (op == 0) { A.v0 = cam_clamp01(b * A.v0); A.v1 = cam_clamp01(b * A.v1); }
        else if (op == 1) {
            real m = fm(p, cam_gray(A.v1), (K(1.0) - p) * cam_gray(A.v0));
            A.v0 = cam_clamp01(fm(ct, A.v0, (K(1.0) - ct) * m)); A.v1 = cam_clamp01(fm(ct, A.v1, (K(1.0) - ct) * m));
        } else if (op == 2) {
            A.v0 = cam_clamp01(fm(sa, A.v0, (K(1.0) - sa) * cam_gray(A.v0))); A.v1 = cam_clamp01(fm(sa, A.v1, (K(1.0) - sa) * cam_gray(A.v1)));
        }
    }
    real e1 = det_exp(K(-0.5) / (sigma * sigma)), e2 = (e1 * e1) * (e1 * e1);
    real S = fm(K(2.0), e1 + e2, K(1.0));
    A.w0 = K(1.0) / S; A.w1 = e1 / S; A.w2 = e2 / S;
    return A;
}
static int cam_pixel_white(const wl_config* c, const uint8_t* map, const real R[9], const real pc[3], int u, int v) {
    real xo = ((real)u + K(0.5) - (real)c->vis_cam_cx) / (real)c->vis_cam_fx;
    real yo = ((real)v + K(0.5) - (real)c->vis_cam_cy) / (real)c->vis_cam_fy;
    real dx = fm(-R[2], yo, fm(-R[1], xo, R[0]));
    real dy = fm(-R[5], yo, fm(-R[4], xo, R[3]));
    real dz = fm(-R[8], yo, fm(-R[7], xo, R[6]));
    int bg = c->vis_cam_bg >= 0.5f;
    if (!(dz < K(0.0)) || !(pc[2] > K(0.0))) return bg;
    real tt = pc[2] / (-dz);
    if (tt > K(100.0)) return bg;
    real hx = fm(tt, dx, pc[0]), hy = fm(tt, dy, pc[1]);
    real fx = r_floor((hx - (real)c->vis_mesh_x0) * (real)c->d_vis_mesh_inv_dx), fy = r_floor((hy - (real)c->vis_mesh_y0) * (real)c->d_vis_mesh_inv_dy);
    if (!(fx >= K(0.0)) || !(fy >= K(0.0)) || !(fx < (real)(c->vis_cols - 1)) || !(fy < (real)(c->vis_rows - 1))) return 0;
    return map[(size_t)(int)fy * c->vis_cols + (int)fx] != 0;
}
/* post-processing of one frame given its white mask [rows*W]: jitter on the class values, separable blur, gray, normalise */
static void camera_post(const wl_config* c, const uint8_t* white, uint32_t t, uint32_t stream, uint32_t sub, const float* aug, float* out) {
    const int W = c->vis_cam_w, rows = c->vis_cam_h - c->vis_cam_row0, npix = W * rows;
    int nw = 0;
    for (int k = 0; k < npix; ++k) nw += white[k] ? 1 : 0;
    cam_aug_t A = cam_aug_params(c, t, stream, sub, aug, (real)nw / (real)npix);
    if (c->vis_cam != 2) {
        for (int k = 0; k < npix; ++k) out[k] = (float)fm(K(2.0), cam_gray(white[k] ? K(1.0) : K(0.0)), K(-1.0));
        return;
    }
    /* blur the MASK (separable 5 taps, reflect padding), then map through the jittered class values: the blur is affine
     * in the mask, J = v0 + (v1 - v0) w */
    real* Hb = (real*)malloc(sizeof(real) * (size_t)npix);
    for (int r = 0; r < rows; ++r)
        for (int u = 0; u < W; ++u) {
#define WLO_JV(x_) (white[r * W + ((x_) < 0 ? -(x_) : ((x_) >= W ? 2 * W - 2 - (x_) : (x_)))] ? K(1.0) : K(0.0))
            real acc = A.w0 * WLO_JV(u);
            acc = fm(A.w1, WLO_JV(u - 1) + WLO_JV(u + 1), acc);
            acc = fm(A.w2, WLO_JV(u - 2) + WLO_JV(u + 2), acc);
            Hb[r * W + u] = acc;
#undef WLO_JV
        }
    const real dv = A.v1 - A.v0;
    for (int r = 0; r < rows; ++r)
        for (int u = 0; u < W; ++u) {
#define WLO_HR(y_) Hb[((y_) < 0 ? -(y_) : ((y_) >= rows ? 2 * rows - 2 - (y_) : (y_))) * W + u]
            real acc = A.w0 * WLO_HR(r);
            acc = fm(A.w1, WLO_HR(r - 1) + WLO_HR(r + 1), acc);
            acc = fm(A.w2, WLO_HR(r - 2) + WLO_HR(r + 2), acc);
            out[r * W + u] = (float)fm(K(2.0), cam_gray(fm(dv, acc, A.v0)), K(-1.0));
#undef WLO_HR
        }
    free(Hb);
}
static void camera_render(const wl_config* c, const uint8_t* map, const wlo_env* e, uint8_t* white) {
    const int W = c->vis_cam_w, rows = c->vis_cam_h - c->vis_cam_row0;
    real R[9]; rotmat(e->q, R);
    real cp[3] = {(real)c->vis_cam_pos[0], (real)c->vis_cam_pos[1], (real)c->vis_cam_pos[2]}, off[3];
    rot(R, cp, off);
    real pc[3] = {e->p[0] + off[0], e->p[1] + off[1], e->p[2] + off[2]};
    for (int r = 0; r < rows; ++r)
        for (int u = 0; u < W; ++u) white[r * W + u] = (uint8_t)cam_pixel_white(c, map, R, pc, u, c->vis_cam_row0 + r);
}
static void camera_obs(const wlo_sim* s, const wlo_env* e, uint32_t t, uint32_t stream, uint32_t sub, const float* aug, float* out) {
    uint8_t white[WL_CAM_MAX_PIXELS];
    camera_render(&s->cfg, s->vis_map, e, white);
    camera_post(&s->cfg, white, t, stream, sub, aug, out);
}

/* interval pushes, mushr_drift_env_cfg.py:121-143; push_by_setting_velocity (+=) [UPSTREAM-RECALL a13] */
static void interval_pushes(const wl_config* c, wlo_env* e, uint32_t gid, int64_t t, real step_dt) {
    if (!c->push_enable) return;
    e->t_hf = e->t_hf - step_dt;
    if (e->t_hf < K(1.0e-6)) {
        uint32_t r[4]; philox4x32(c->seed, gid, (uint32_t)t, RNG_PUSH_HF, 0u, r);
        e->v[0] = e->v[0] + uniform(r[0], -(real)c->push_hf_range[0], (real)c->push_hf_range[0]);
        e->v[1] = e->v[1] + uniform(r[1], -(real)c->push_hf_range[1], (real)c->push_hf_range[1]);
        e->w[2] = e->w[2] + uniform(r[2], -(real)c->push_hf_range[2], (real)c->push_hf_range[2]);
        e->t_hf = uniform(r[3], (real)c->push_hf_interval[0], (real)c->push_hf_interval[1]);
    }
    e->t_lf = e->t_lf - step_dt;
    if (e->t_lf < K(1.0e-6)) {
        uint32_t r[4]; philox4x32(c->seed, gid, (uint32_t)t, RNG_PUSH_LF, 0u, r);
        e->w[2] = e->w[2] + uniform(r[0], -(real)c->push_lf_yaw, (real)c->push_lf_yaw);
        e->t_lf = uniform(r[1], (real)c->push_lf_interval[0], (real)c->push_lf_interval[1]);
    }
}

/* BlindObsCfg.PolicyCfg, wheeledlab_tasks/common/observations.py:19-56 */
static void blind_obs(const wl_config* c, const wlo_env* e, uint32_t gid, uint32_t t, uint32_t stream, uint32_t sub0, float* obs) {
    real R[9]; rotmat(e->q, R);
    real vb[3], wb[3], eu[3]; rotT(R, e->v, vb); rotT(R, e->w, wb); euler_xyz(e->q, eu);
    real z[12];
    for (int k = 0; k < 12; ++k) z[k] = K(0.0);
    if (c->enable_corruption) {
        for (uint32_t k = 0; k < 3; ++k) {
            uint32_t r[4]; philox4x32(c->seed, gid, t, stream, sub0 + k, r);
            box_muller(r[0], r[1], &z[4 * k + 0], &z[4 * k + 1]);
            box_muller(r[2], r[3], &z[4 * k + 2], &z[4 * k + 3]);
        }
    }
    for (int k = 0; k < 3; ++k) {
        obs[0 + k] = (float)(e->p[k] + (real)c->noise_std[0] * z[0 + k]);   /* root_pos_w - env_origin(=0) */
        obs[3 + k] = (float)(eu[k] + (real)c->noise_std[1] * z[3 + k]);
        obs[6 + k] = (float)(vb[k] + (real)c->noise_std[2] * z[6 + k]);
        obs[9 + k] = (float)(wb[k] + (real)c->noise_std[3] * z[9 + k]);
    }
    obs[12] = (float)r_clamp(e->action[0], K(-1.0), K(1.0));               /* last_action, clip (-1,1), no noise */
    obs[13] = (float)r_clamp(e->action[1], K(-1.0), K(1.0));
}

/* ------------------------------------------------------------------------- */
/* one env.step() for one env -- ordering per SURVEY 3.3 A..I                  */
/* ------------------------------------------------------------------------- */
typedef struct { double sum[WL_MAX_REW_TERMS]; double n_reset; double n_term[WL_MAX_TERM_TERMS]; int any; } step_log;

static int env_step(wlo_sim* s, int li, const float* a_in, int64_t t, float* obs, float* rew, uint8_t* term_o,
                    uint8_t* trunc_o, step_log* lg) {
    const wl_config* c = &s->cfg;
    wlo_env* e = &s->env[li];
    uint32_t gid = (uint32_t)(c->env_id_offset + li);
    /* A. action manager: prev <- action <- raw */
    e->prev_action[0] = e->action[0]; e->prev_action[1] = e->action[1];
    e->action[0] = (real)a_in[0]; e->action[1] = (real)a_in[1];
    real wheel_target[4], steer_target[2];
    int rc = process_action(c, a_in, wheel_target, steer_target);
    if (rc) return rc;
    /* B. decimation x (actuators -> physics) */
    chassis_t b;
    real R[9]; rotmat(e->q, R);
    real cw[3]; { real cc[3] = {(real)c->com[0], (real)c->com[1], (real)c->com[2]}; rot(R, cc, cw); }
    for (int k = 0; k < 3; ++k) { b.pc[k] = e->p[k] + cw[k]; b.v[k] = e->v[k]; }
    for (int k = 0; k < 4; ++k) b.q[k] = e->q[k];
    rotT(R, e->w, b.wb);
    step_consts kc; make_step_consts(c, e, &kc);
    for (int d = 0; d < c->decimation; ++d) {
        real lo[4], hi[4];
        for (int i = 0; i < 4; ++i) dc_limits(c, (real)c->dc_effort[i], e->omega[i], &lo[i], &hi[i]);
        for (int j = 0; j < c->substeps; ++j) physics_substep(s, e, &b, wheel_target, lo, hi, steer_target, &kc);
    }
    rotmat(b.q, R);
    { real cc[3] = {(real)c->com[0], (real)c->com[1], (real)c->com[2]}; rot(R, cc, cw); }
    for (int k = 0; k < 3; ++k) { e->p[k] = b.pc[k] - cw[k]; e->v[k] = b.v[k]; }
    for (int k = 0; k < 4; ++k) e->q[k] = b.q[k];
    rot(R, b.wb, e->w);
    /* C. counters */
    e->ep_len += 1;
    /* D. terminations (time_out first in cfg order) */
    int time_out = e->ep_len >= c->max_episode_length;
    uint32_t tmask;
    real step_dt = (real)c->d_step_dt;
    real f[WL_MAX_REW_TERMS];
    real vb[3]; rotT(R, e->v, vb);
    if (c->task == WL_TASK_DRIFT) {
        int oob = drift_off_track(c, e->p[0], e->p[1]);
        drift_reward_terms(c, e, e->p, vb, b.wb, e->w[2], oob, time_out, f);
        tmask = (time_out ? 1u : 0u) | (oob ? 2u : 0u);
    } else if (c->task == WL_TASK_ELEVATION) {
        tmask = elev_terms(c, e, R, vb, (e->omega[0] + e->omega[1]) + (e->omega[2] + e->omega[3]), time_out, f);
    } else if (c->task == WL_TASK_VISUAL) {
        tmask = visual_terms(s, e, vb, time_out, f);
    } else {
        return WL_EUNSUPPORTED;
    }
    tmask &= (uint32_t)c->term_enable;     /* play cfgs: terminations = None */
    /* E. reward manager [UPSTREAM-RECALL Appendix B]: value = f*w*dt, skip w==0 */
    real total = K(0.0);
    for (int k = 0; k < c->num_rew_terms; ++k) {
        if (s->rew_weight[k] == K(0.0)) continue;
        real val = f[k] * s->rew_weight[k] * step_dt;
        total += val;
        e->sums[k] += val;
    }
    *rew = (float)total;
    *term_o = (uint8_t)((tmask & ~1u) ? 1 : 0); *trunc_o = (uint8_t)(tmask & 1u);
    /* F. auto reset */
    if (tmask) {
        lg->any = 1; lg->n_reset += 1.0;
        for (int j = 0; j < WL_MAX_TERM_TERMS; ++j) lg->n_term[j] += ((tmask >> j) & 1u) ? 1.0 : 0.0;
        for (int k = 0; k < WL_MAX_REW_TERMS; ++k) lg->sum[k] += (double)e->sums[k];
        if (c->task == WL_TASK_ELEVATION) elev_reset_env(c, e, gid, t);
        else if (c->task == WL_TASK_VISUAL) visual_reset_env(s, e, gid, t);
        else drift_reset_env(c, e, gid, t);
    }
    if (c->task == WL_TASK_VISUAL) {      /* PolicyCfg order: camera, base_lin_vel, base_ang_vel, last_action (:45-52) */
        if (c->vis_cam) camera_obs(s, e, (uint32_t)t, RNG_CAM, 0u, NULL, obs);
        visual_obs(e, obs + vis_cam_floats(c));
        return 0;
    }
    if (c->task == WL_TASK_ELEVATION) {
        /* G. commands; I. observations */
        elev_command_update(c, e, gid, t, step_dt);
        elev_obs(s, e, obs);
        return 0;
    }
    /* H. interval events on the post-reset state */
    interval_pushes(c, e, gid, t, step_dt);
    /* I. observations */
    blind_obs(c, e, gid, (uint32_t)t, RNG_OBS, 0u, obs);
    return 0;
}

/* ------------------------------------------------------------------------- */
/* exported API (host pointers)                                                */
/* ------------------------------------------------------------------------- */
wlo_sim* wlo_create(const wl_config* cfg, const float* heightfield) {
    wlo_sim* s = (wlo_sim*)calloc(1, sizeof(wlo_sim));
    s->cfg = *cfg;
    config_finalize(&s->cfg);
    s->env = (wlo_env*)calloc((size_t)cfg->num_envs, sizeof(wlo_env));
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) s->rew_weight[k] = (real)cfg->rew_weight[k];
    if (heightfield && cfg->task == WL_TASK_VISUAL) {        /* aux = int32 cells[n_trav] | pad16 | uint8 map[rows*cols] */
        size_t off = ((size_t)cfg->vis_n_trav * 4 + 15) & ~(size_t)15, nm = (size_t)cfg->vis_rows * cfg->vis_cols;
        s->vis_cells = (int32_t*)malloc((size_t)cfg->vis_n_trav * 4);
        s->vis_map = (uint8_t*)malloc(nm);
        memcpy(s->vis_cells, heightfield, (size_t)cfg->vis_n_trav * 4);
        memcpy(s->vis_map, (const char*)heightfield + off, nm);
    } else if (heightfield && cfg->hf_nx > 0) {
        size_t n = (size_t)cfg->hf_pitch * cfg->hf_ny;
        s->hf = (float*)malloc(n * sizeof(float));
        memcpy(s->hf, heightfield, n * sizeof(float));
    }
    for (int i = 0; i < cfg->num_envs; ++i) s->env[i].q[0] = K(1.0);
    return s;
}
void wlo_destroy(wlo_sim* s) { if (s) { free(s->env); free(s->hf); free(s->vis_cells); free(s->vis_map); free(s); } }
int wlo_is_double(void) {
#ifdef WLO_DOUBLE
    return 1;
#else
    return 0;
#endif
}

/* startup events a14: material buckets, actuator gains, base mass; initial interval timers */
int wlo_startup(wlo_sim* s) {
    const wl_config* c = &s->cfg;
    for (int li = 0; li < c->num_envs; ++li) {
        wlo_env* e = &s->env[li];
        uint32_t gid = (uint32_t)(c->env_id_offset + li);
        uint32_t r0[4], r1[4], r2[4], r3[4];
        philox4x32(c->seed, gid, 0u, RNG_STARTUP, 0u, r0);
        philox4x32(c->seed, gid, 0u, RNG_STARTUP, 1u, r1);
        philox4x32(c->seed, gid, 0u, RNG_STARTUP, 2u, r2);
        philox4x32(c->seed, gid, 0u, RNG_STARTUP, 3u, r3);
        for (int i = 0; i < 4; ++i) {
            uint32_t bk = 0;
            if (c->dr_enable && c->dr_num_buckets > 1) bk = (uint32_t)(((uint64_t)r0[i] * (uint64_t)c->dr_num_buckets) >> 32);
            e->D[i] = (real)c->dr_bucket_D[bk];
            e->C[i] = (real)c->dr_bucket_C[bk];
            e->kd[i] = (real)c->dc_damping[i];
            if (c->dr_enable && ((c->dr_kd_mask >> i) & 1)) e->kd[i] = uniform(r1[i], (real)c->dr_kd_range[0], (real)c->dr_kd_range[1]);
        }
        /* randomize_rigid_body_mass [UPSTREAM-RECALL]: "add" -> base_link mass += U; "abs" -> base_link mass := U
         * (mushr_visual_env_cfg.py:280-288); wheel links := U (:290-299), their inertia rescaled by the mass ratio */
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
        sample_interval_timers(c, e, r2[1], r2[2]);
        e->q[0] = K(1.0); e->q[1] = e->q[2] = e->q[3] = K(0.0);
    }
    return 0;
}

int wlo_reset(wlo_sim* s, const int64_t* env_ids, int32_t n_ids, int64_t step_counter) {
    const wl_config* c = &s->cfg;
    int n = env_ids ? n_ids : c->num_envs;
    for (int k = 0; k < n; ++k) {
        int li = env_ids ? (int)env_ids[k] : k;
        if (c->task == WL_TASK_ELEVATION) elev_reset_env(c, &s->env[li], (uint32_t)(c->env_id_offset + li), step_counter);
        else if (c->task == WL_TASK_VISUAL) visual_reset_env(s, &s->env[li], (uint32_t)(c->env_id_offset + li), step_counter);
        else drift_reset_env(c, &s->env[li], (uint32_t)(c->env_id_offset + li), step_counter);
    }
    return 0;
}

int wlo_step(wlo_sim* s, const float* action, float* obs, float* rew, uint8_t* terminated, uint8_t* truncated,
             int64_t step_counter, int nthreads) {
    const wl_config* c = &s->cfg;
    int od = (c->task == WL_TASK_ELEVATION) ? WL_OBS_DIM_ELEV : (c->task == WL_TASK_VISUAL) ? WL_OBS_DIM_VISUAL + vis_cam_floats(c) : WL_OBS_DIM_BLIND;
    step_log tot; memset(&tot, 0, sizeof tot);
    int err = 0;
    (void)nthreads;
#ifdef _OPENMP
#pragma omp parallel num_threads(nthreads > 0 ? nthreads : 1)
#endif
    {
        step_log lg; memset(&lg, 0, sizeof lg);
#ifdef _OPENMP
#pragma omp for schedule(static)
#endif
        for (int li = 0; li < c->num_envs; ++li) {
            int rc = env_step(s, li, action + 2 * (size_t)li, step_counter, obs + (size_t)od * li, rew + li, terminated + li,
                              truncated + li, &lg);
            if (rc) err = rc;
        }
#ifdef _OPENMP
#pragma omp critical
#endif
        {
            for (int k = 0; k < WL_MAX_REW_TERMS; ++k) tot.sum[k] += lg.sum[k];
            tot.n_reset += lg.n_reset; tot.any |= lg.any;
            for (int j = 0; j < WL_MAX_TERM_TERMS; ++j) tot.n_term[j] += lg.n_term[j];
        }
    }
    if (tot.any) {      /* extras["log"] is rebuilt inside _reset_idx only: a step without a reset keeps the previous row */
        for (int k = 0; k < WL_MAX_REW_TERMS; ++k) s->log_sum[k] = tot.sum[k];
        s->log_term[0] = tot.n_reset;
        for (int j = 0; j < WL_MAX_TERM_TERMS; ++j) s->log_term[1 + j] = tot.n_term[j];
    }
    s->any_reset_last = tot.any;
    /* common_step_counter += 1, then the curriculum terms (curriculums.py:23-35), only if >= 1 env reset this step */
    {
        int64_t cn = step_counter + 1;
        if (c->curr_n > 0 && tot.any && (cn % c->max_episode_length) == 0) {
            int E = (int)(cn / c->max_episode_length);
            for (int k = 0; k < c->curr_n; ++k) {
                if (E / c->curr_every[k] > c->curr_max[k]) continue;
                if ((E + 1) % c->curr_every[k] == 0) s->rew_weight[c->curr_slot[k]] += (real)c->curr_inc[k];
            }
        }
    }
    return err;
}

int wlo_observe(wlo_sim* s, float* obs, int64_t step_counter, int32_t call_idx) {
    const wl_config* c = &s->cfg;
    if (c->task == WL_TASK_ELEVATION) {
        for (int li = 0; li < c->num_envs; ++li) elev_obs(s, &s->env[li], obs + (size_t)WL_OBS_DIM_ELEV * li);
        return 0;
    }
    if (c->task == WL_TASK_VISUAL) {
        const int camf = vis_cam_floats(c);
        for (int li = 0; li < c->num_envs; ++li) {
            float* row = obs + (size_t)(WL_OBS_DIM_VISUAL + camf) * li;
            if (camf) camera_obs(s, &s->env[li], (uint32_t)step_counter, RNG_CAM_EXTRA, (uint32_t)call_idx, NULL, row);
            visual_obs(&s->env[li], row + camf);
        }
        return 0;
    }
    for (int li = 0; li < c->num_envs; ++li)
        blind_obs(c, &s->env[li], (uint32_t)(c->env_id_offset + li), (uint32_t)step_counter, RNG_OBS_EXTRA,
                  3u * (uint32_t)call_idx, obs + (size_t)WL_OBS_DIM_BLIND * li);
    return 0;
}

/* curriculum, wheeledlab/envs/mdp/curriculums.py:10-35 -- the counter conditions are
 * evaluated by the caller (fire_mask); the "called only when >=1 env reset" condition
 * (SURVEY a11) is applied here from the last step's any_reset flag. */
int wlo_curriculum(wlo_sim* s, int32_t n_terms, const int32_t* slots, const float* increases, uint32_t fire_mask) {
    if (!s->any_reset_last) return 0;
    for (int t = 0; t < n_terms; ++t)
        if ((fire_mask >> t) & 1u) s->rew_weight[slots[t]] += (real)increases[t];
    return 0;
}

int wlo_synth_actions(const wl_config* c, float* action, int64_t step_counter, int32_t dist) {
    for (int li = 0; li < c->num_envs; ++li) {
        uint32_t r[4]; philox4x32(c->seed, (uint32_t)(c->env_id_offset + li), (uint32_t)step_counter, RNG_ACTION, 0u, r);
        if (dist == 0) {
            action[2 * li + 0] = (float)(K(2.0) * u01(r[0]) - K(1.0));
            action[2 * li + 1] = (float)(K(2.0) * u01(r[1]) - K(1.0));
        } else {
            real z0, z1; box_muller(r[0], r[1], &z0, &z1);
            action[2 * li + 0] = (float)r_clamp(z0, K(-1.0), K(1.0));
            action[2 * li + 1] = (float)r_clamp(z1, K(-1.0), K(1.0));
        }
    }
    return 0;
}

/* ---- packed state import / export in the product's AoSoA layout ------------- */
static inline float* grp(float* buf, int g, int n, int i) { return buf + ((size_t)g * n + i) * 4; }
void wlo_export_state(const wlo_sim* s, float* buf) {
    int n = s->cfg.num_envs;
    for (int i = 0; i < n; ++i) {
        const wlo_env* e = &s->env[i];
        float* g;
        g = grp(buf, WL_G_POS, n, i); g[0] = (float)e->p[0]; g[1] = (float)e->p[1]; g[2] = (float)e->p[2]; memcpy(&g[3], &e->ep_len, 4);
        g = grp(buf, WL_G_QUAT, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->q[k];
        g = grp(buf, WL_G_LINVEL, n, i); for (int k = 0; k < 3; ++k) g[k] = (float)e->v[k]; g[3] = (float)e->t_hf;
        g = grp(buf, WL_G_ANGVEL, n, i); for (int k = 0; k < 3; ++k) g[k] = (float)e->w[k]; g[3] = (float)e->t_lf;
        g = grp(buf, WL_G_WHEEL, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->omega[k];
        g = grp(buf, WL_G_STEER, n, i); g[0] = (float)e->steer[0]; g[1] = (float)e->steer[1]; g[2] = (float)e->steer_vel[0]; g[3] = (float)e->steer_vel[1];
        g = grp(buf, WL_G_ACTION, n, i); g[0] = (float)e->action[0]; g[1] = (float)e->action[1]; g[2] = (float)e->prev_action[0]; g[3] = (float)e->prev_action[1];
        g = grp(buf, WL_G_SUM0, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->sums[k];
        g = grp(buf, WL_G_SUM1, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->sums[4 + k];
        g = grp(buf, WL_G_PMASS, n, i); g[0] = (float)e->mass; g[1] = (float)e->inv_mass; g[2] = (float)e->spare0; g[3] = (float)e->spare1;
        g = grp(buf, WL_G_PMU_D, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->D[k];
        g = grp(buf, WL_G_PMU_C, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->C[k];
        g = grp(buf, WL_G_PKD, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->kd[k];
        g = grp(buf, WL_G_CMD, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->cmd[k];
        g = grp(buf, WL_G_CMDB, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->cmdb[k];
        g = grp(buf, WL_G_PIW, n, i); for (int k = 0; k < 4; ++k) g[k] = (float)e->inv_Iw[k];
    }
}
void wlo_import_state(wlo_sim* s, const float* cbuf) {
    int n = s->cfg.num_envs; float* buf = (float*)cbuf;
    for (int i = 0; i < n; ++i) {
        wlo_env* e = &s->env[i];
        const float* g;
        g = grp(buf, WL_G_POS, n, i); e->p[0] = g[0]; e->p[1] = g[1]; e->p[2] = g[2]; memcpy(&e->ep_len, &g[3], 4);
        g = grp(buf, WL_G_QUAT, n, i); for (int k = 0; k < 4; ++k) e->q[k] = g[k];
        g = grp(buf, WL_G_LINVEL, n, i); for (int k = 0; k < 3; ++k) e->v[k] = g[k]; e->t_hf = g[3];
        g = grp(buf, WL_G_ANGVEL, n, i); for (int k = 0; k < 3; ++k) e->w[k] = g[k]; e->t_lf = g[3];
        g = grp(buf, WL_G_WHEEL, n, i); for (int k = 0; k < 4; ++k) e->omega[k] = g[k];
        g = grp(buf, WL_G_STEER, n, i); e->steer[0] = g[0]; e->steer[1] = g[1]; e->steer_vel[0] = g[2]; e->steer_vel[1] = g[3];
        g = grp(buf, WL_G_ACTION, n, i); e->action[0] = g[0]; e->action[1] = g[1]; e->prev_action[0] = g[2]; e->prev_action[1] = g[3];
        g = grp(buf, WL_G_SUM0, n, i); for (int k = 0; k < 4; ++k) e->sums[k] = g[k];
        g = grp(buf, WL_G_SUM1, n, i); for (int k = 0; k < 4; ++k) e->sums[4 + k] = g[k];
        g = grp(buf, WL_G_PMASS, n, i); e->mass = g[0]; e->inv_mass = g[1]; e->spare0 = g[2]; e->spare1 = g[3];
        g = grp(buf, WL_G_PMU_D, n, i); for (int k = 0; k < 4; ++k) e->D[k] = g[k];
        g = grp(buf, WL_G_PMU_C, n, i); for (int k = 0; k < 4; ++k) e->C[k] = g[k];
        g = grp(buf, WL_G_PKD, n, i); for (int k = 0; k < 4; ++k) e->kd[k] = g[k];
        g = grp(buf, WL_G_CMD, n, i); for (int k = 0; k < 4; ++k) e->cmd[k] = g[k];
        g = grp(buf, WL_G_CMDB, n, i); for (int k = 0; k < 4; ++k) e->cmdb[k] = g[k];
        g = grp(buf, WL_G_PIW, n, i); for (int k = 0; k < 4; ++k) e->inv_Iw[k] = g[k];
    }
}
void wlo_get_weights(const wlo_sim* s, float* w) { for (int k = 0; k < WL_MAX_REW_TERMS; ++k) w[k] = (float)s->rew_weight[k]; }
void wlo_set_weights(wlo_sim* s, const float* w) { for (int k = 0; k < WL_MAX_REW_TERMS; ++k) s->rew_weight[k] = (real)w[k]; }
/* the d_log row of the last step (RewardManager.reset, Appendix B): [0..7] mean episode sum over the reset envs /
 * max_episode_length_s, [8] n_reset, [9] n_terminated, [10] n_timeout */
void wlo_get_log(const wlo_sim* s, double* out) {
    double cnt = s->log_term[0] > 1.0 ? s->log_term[0] : 1.0;
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) out[k] = s->log_sum[k] / (cnt * (double)s->cfg.episode_length_s);
    for (int j = 0; j < 8; ++j) out[8 + j] = s->log_term[j];
}

int wlo_any_reset_last(const wlo_sim* s) { return s->any_reset_last; }

/* ---- unit-level hooks for golden-vector and det-math tests -------------------- */
int wlo_detmath(int32_t op, const float* in, const float* in2, float* out, int32_t n) {
    for (int i = 0; i < n; ++i) {
        real x = (real)in[i], s, c;
        switch (op) {
            case 0: det_sincos(x, &s, &c); out[i] = (float)s; break;
            case 1: det_sincos(x, &s, &c); out[i] = (float)c; break;
            case 2: out[i] = (float)det_atan(x); break;
            case 3: out[i] = (float)det_atan2((real)in2[i], x); break;
            case 4: out[i] = (float)det_log(x); break;
            case 5: out[i] = (float)det_tan(x); break;
            case 6: out[i] = (float)det_asin(x); break;
            case 7: out[i] = (float)det_exp(x); break;
            case 8: out[i] = (float)det_tanh(x); break;
            default: return WL_EINVAL;
        }
    }
    return 0;
}
/* DCMotor torque (a7) for given gains / targets / joint speeds: out[i] = clip(kd (target - omega), speed-dependent limits) */
int wlo_dc_motor(const wl_config* c_in, float kd, float effort_limit, const float* target, const float* omega, float* out, int32_t n) {
    wl_config cc = *c_in; config_finalize(&cc);
    for (int i = 0; i < n; ++i) out[i] = (float)dc_motor(&cc, (real)kd, (real)effort_limit, (real)target[i], (real)omega[i]);
    return 0;
}
/* camera term alone: aug = NULL draws the parameters; obs rows have the full visual stride */
int wlo_camera(wlo_sim* s, float* obs, int64_t step_counter, const float* aug) {
    const wl_config* c = &s->cfg;
    if (c->task != WL_TASK_VISUAL || !c->vis_cam) return WL_EUNSUPPORTED;
    const int camf = vis_cam_floats(c);
    for (int li = 0; li < c->num_envs; ++li)
        camera_obs(s, &s->env[li], (uint32_t)step_counter, RNG_CAM, 0u, aug, obs + (size_t)(WL_OBS_DIM_VISUAL + camf) * li);
    return 0;
}
/* post-processing only (golden vectors of camera_data_rgb_flattened[_aug]): white [n, rows*W] u8, aug 9 floats, out [n, rows*W] */
int wlo_camera_post(const wl_config* c_in, const uint8_t* white, const float* aug, float* out, int32_t n) {
    wl_config cc = *c_in; config_finalize(&cc);
    const int npix = vis_cam_floats(&cc);
    if (npix <= 0 || npix > WL_CAM_MAX_PIXELS) return WL_EINVAL;
    for (int i = 0; i < n; ++i) camera_post(&cc, white + (size_t)i * npix, 0u, RNG_CAM, 0u, aug, out + (size_t)i * npix);
    return 0;
}
/* raw render of env li: white mask [rows*W] */
int wlo_camera_render(wlo_sim* s, int32_t li, uint8_t* white) {
    if (s->cfg.task != WL_TASK_VISUAL || !s->cfg.vis_cam || li < 0 || li >= s->cfg.num_envs) return WL_EINVAL;
    camera_render(&s->cfg, s->vis_map, &s->env[li], white);
    return 0;
}
int wlo_philox(uint64_t seed, uint32_t c0_base, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t* out, int32_t n) {
    for (int i = 0; i < n; ++i) philox4x32(seed, c0_base + (uint32_t)i, c1, c2, c3, out + 4 * (size_t)i);
    return 0;
}
/* action map only: out wheel targets [n,4] (bl,br,fl,fr) and steer targets [n,2] */
int wlo_action_map(const wl_config* c_in, const float* action, float* wheel, float* steer, int32_t n) {
    wl_config cc = *c_in; config_finalize(&cc); const wl_config* c = &cc;
    for (int i = 0; i < n; ++i) {
        real wt[4], st[2];
        int rc = process_action(c, action + 2 * i, wt, st);
        if (rc) return rc;
        for (int k = 0; k < 4; ++k) wheel[4 * i + k] = (float)wt[k];
        steer[2 * i] = (float)st[0]; steer[2 * i + 1] = (float)st[1];
    }
    return 0;
}
/* drift MDP terms on given root states: in[n,13] = pos3 quat4 linvel_w3 angvel_w3, steer[n,2];
 * out f[n,8] unweighted terms, term[n] out_of_bounds */
int wlo_drift_terms(const wl_config* c, const float* root, const float* steer, const int32_t* ep_len, float* f_out,
                    uint8_t* oob, int32_t n) {
    for (int i = 0; i < n; ++i) {
        wlo_env e; memset(&e, 0, sizeof e);
        const float* r = root + 13 * i;
        real p[3] = {r[0], r[1], r[2]}, q[4] = {r[3], r[4], r[5], r[6]}, v[3] = {r[7], r[8], r[9]}, w[3] = {r[10], r[11], r[12]};
        e.steer[0] = steer[2 * i]; e.steer[1] = steer[2 * i + 1];
        real R[9]; rotmat(q, R);
        real vb[3], wb[3]; rotT(R, v, vb); rotT(R, w, wb);
        int t = drift_off_track(c, p[0], p[1]);
        int to = ep_len[i] >= c->max_episode_length;
        real f[WL_MAX_REW_TERMS];
        drift_reward_terms(c, &e, p, vb, wb, w[2], t, to, f);
        for (int k = 0; k < WL_MAX_REW_TERMS; ++k) f_out[WL_MAX_REW_TERMS * i + k] = (float)f[k];
        oob[i] = (uint8_t)t;
    }
    return 0;
}
/* reset pose from explicit draws: pose[n,7] = pos3 quat4 */
int wlo_drift_reset_pose(const wl_config* c, const int32_t* idx, const float* u_xy, const float* u_yaw, float* pose, int32_t n) {
    for (int i = 0; i < n; ++i) {
        wlo_env e; memset(&e, 0, sizeof e);
        drift_reset_pose(c, &e, (uint32_t)idx[i], (real)u_xy[2 * i], (real)u_xy[2 * i + 1], (real)u_yaw[i]);
        for (int k = 0; k < 3; ++k) pose[7 * i + k] = (float)e.p[k];
        for (int k = 0; k < 4; ++k) pose[7 * i + 3 + k] = (float)e.q[k];
    }
    return 0;
}
/* elevation MDP terms on given states: root[n,13] = pos3 quat4 linvel_w3 angvel_w3, cmdb[n,2], omega[n,4];
 * out f[n,8] unweighted reward terms, mask[n] termination bits, proprio[n,13] observation head */
int wlo_elev_terms(const wl_config* c_in, const float* root, const float* cmdb, const float* omega, const float* action,
                   const int32_t* ep_len, float* f_out, uint32_t* mask, float* proprio, int32_t n) {
    wl_config cc = *c_in; config_finalize(&cc); const wl_config* c = &cc;
    for (int i = 0; i < n; ++i) {
        wlo_env e; memset(&e, 0, sizeof e);
        const float* r = root + 13 * i;
        for (int k = 0; k < 3; ++k) { e.p[k] = r[k]; e.v[k] = r[7 + k]; e.w[k] = r[10 + k]; }
        for (int k = 0; k < 4; ++k) { e.q[k] = r[3 + k]; e.omega[k] = omega[4 * i + k]; }
        e.cmdb[0] = cmdb[2 * i]; e.cmdb[1] = cmdb[2 * i + 1];
        e.action[0] = action[2 * i]; e.action[1] = action[2 * i + 1];
        real R[9]; rotmat(e.q, R);
        real vb[3]; rotT(R, e.v, vb);
        real f[WL_MAX_REW_TERMS];
        mask[i] = elev_terms(c, &e, R, vb, (e.omega[0] + e.omega[1]) + (e.omega[2] + e.omega[3]), ep_len[i] >= c->max_episode_length, f);
        for (int k = 0; k < WL_MAX_REW_TERMS; ++k) f_out[WL_MAX_REW_TERMS * i + k] = (float)f[k];
        /* proprio head only (no height-field needed) */
        real wb[3], eu[3]; rotT(R, e.w, wb); euler_xyz(e.q, eu);
        real gx = e.cmdb[0] - e.p[0], gy = e.cmdb[1] - e.p[1], cl = (real)c->obs_clip;
        float* o = proprio + 13 * i;
        o[0] = (float)((gx != gx) ? K(0.0) : gx); o[1] = (float)((gy != gy) ? K(0.0) : gy);
        for (int k = 0; k < 3; ++k) { o[2 + k] = (float)eu[k]; o[5 + k] = (float)r_clamp(vb[k], -cl, cl); o[8 + k] = (float)r_clamp(wb[k], -cl, cl); }
        o[11] = (float)r_clamp(e.action[0], K(-1.0), K(1.0)); o[12] = (float)r_clamp(e.action[1], K(-1.0), K(1.0));
    }
    return 0;
}
int wlo_euler_xyz(const float* quat, float* out, int32_t n) {
    for (int i = 0; i < n; ++i) {
        real q[4] = {quat[4 * i], quat[4 * i + 1], quat[4 * i + 2], quat[4 * i + 3]}, e[3];
        euler_xyz(q, e);
        out[3 * i] = (float)e[0]; out[3 * i + 1] = (float)e[1]; out[3 * i + 2] = (float)e[2];
    }
    return 0;
}

/* same X-macro descriptor as the product library, so tests can cross-check the layouts */
const char* wlo_config_describe(void) {
    static char buf[16384];
    if (buf[0] == 0) {
        size_t off = 0;
#define WL_XS(type, tag, name) off += (size_t)snprintf(buf + off, sizeof buf - off, "%s:%s:1:%zu;", #name, #tag, offsetof(wl_config, name));
#define WL_XA(type, tag, name, n) off += (size_t)snprintf(buf + off, sizeof buf - off, "%s:%s:%d:%zu;", #name, #tag, (int)(n), offsetof(wl_config, name));
        WL_CONFIG_FIELDS(WL_XS, WL_XA)
#undef WL_XS
#undef WL_XA
        snprintf(buf + off, sizeof buf - off, "sizeof:%zu", sizeof(wl_config));
    }
    return buf;
}
