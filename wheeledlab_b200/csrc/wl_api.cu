// wl_api.cu -- kernels + the extern "C" ABI declared in include/wheeledlab_b200.h.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -fmad=false -lineinfo -O3 (see build.py).
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include <cuda.h>

#include "wl_step.cuh"

using namespace wl;

#include "wl_critic.cuh"
#include "wl_policy_obs.cuh"
#include "wl_row_terms.cuh"
#include "wl_events.cuh"

// ---------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------
struct wl_sim {
    wl_config cfg;
    float4* state;          // groups
    wl_globals* globals;    // device
    const float* hf;        // device height-field or null
    size_t state_bytes;
    int64_t launches;
    int64_t chained_steps;  // wl_step launches of the duo kernel that ran chained (wl_chained_step_count)
    int64_t deep_steps;     // (of those, the ones that ran deep: wl_deep_step_count)
    int64_t last_t;         // counter of the most recent step launched through this handle (-1: none); host mirror
    int64_t base_host;      // host mirror of wl_globals.step_base
    uint8_t* term_bits;     // optional per-env termination-term bits output of wl_step (wl_set_term_bits)
    PeerFan fan;            // peers every output row of wl_step is also stored to (wl_set_peer_fanout); n = 0: none
    const void* hp_host[8]; // wl_step_host_zero_copy: pinned host blocks already resolved to their device alias
    void* hp_dev[8];
    int hp_n;
    int device;             // CUDA device ordinal the handle lives on
    int obs_dim;
    int variant;            // 0 auto, 1 thread-per-env, 4 quad-per-env
    CUtensorMap tmap;       // 2-D tensor map over the height-field (elevation task)
    bool has_tmap;
    int scan_mode;          // ray-cast tile staging: 1 one TMA tile per CTA (default), 2 TMA producer/consumer pipeline, 0 plain loads (A/B)
    uint32_t spec;          // spec_key(step_spec(cfg)): picks the duo kernel's instantiation (see with_spec)
    const void* duo_kernel; // the duo kernel duo_threads was sized for (see duo_block)
    int duo_threads;
    int step_variant;       // what the most recent wl_step launched (wl_step_launch_info): variant after the automatic choice
    int step_specialised;   // (the duo kernel ran a spec instantiation, not its generic body)
    int step_threads;       // (threads per CTA)
    struct DevTerms* dterms;   // wl_set_device_terms: the term table and its per-env state (null: none)
    CriticTable critic;        // wl_set_critic_terms: the critic observation's columns (n_cols = 0: none)
    uint32_t reset_ev;         // wl_set_reset_events: WL_RESET_EV_* bits of the events redrawn at every reset (0: none)
    EventTable events;         // wl_set_event_timers: the interval terms' ranges and per-env timers (n = 0: none)
    struct DevEvents* devents; // wl_set_device_events: the device event terms and their timers (null: none)
    PolicyObsTable pobs;       // wl_set_policy_terms: the policy observation's columns (n_cols = 0: none)
    RowTable rows;             // wl_set_row_terms: noise, clip and scale of the Elevation / Visual row (n_terms = 0: none)
    RowTable crit_rows;        // wl_set_row_critic: clip and scale of the critic's copy of the Elevation row (n_terms = 0: none)
    CriticTable crit_extra;    // wl_set_row_critic: the critic-library columns after it
};

// SMs of the H100 SXM the launch geometry is sized for
#define WL_NUM_SMS 132
// below this many envs one thread/env cannot fill the SMs x 4 schedulers; use 4 lanes per env
#define WL_QUAD_MAX_ENVS (WL_NUM_SMS * 4 * 32 * 2)

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
static int cuda_check(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return 0;
    return fail(WL_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

// every kernel launch made through a handle is counted (wl_launch_count) and checked here
static int launched(wl_sim* sim, const char* what, int count = 1) {
    sim->launches += count;
    return cuda_check(cudaGetLastError(), what);
}
// the step counter of an entry that does not advance it: a host value below 2^31, or WL_DEVICE_COUNTER_PLUS(k)
static int check_counter(const std::string& fn, int64_t step_counter) {
    if (step_counter < ((int64_t)1 << 31) && step_counter >= -((int64_t)1 << 31)) return WL_OK;
    return fail(WL_EINVAL, fn + ": step counter out of range (< 2^31, or WL_DEVICE_COUNTER_PLUS(k))");
}
// Raise KERNEL's dynamic shared-memory limit to `bytes` on device `dev`, once per device.  It must happen before the kernel's
// first launch and outside any graph capture: every entry calls this before it launches, and the PPO workspace queries reach
// it before the first update (see ppo_workspace).
template <auto KERNEL>
static int raise_smem(int dev, size_t bytes, const char* fn) {
    static bool done[64] = {false};
    if (dev < 0 || dev >= 64 || done[dev]) return WL_OK;
    if (int rc = cuda_check(cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes), fn)) return rc;
    done[dev] = true;
    return WL_OK;
}
// f(std::integral_constant<int, T>{}) for the first listed task T equal to `task`, else for WL_TASK_DRIFT: a caller
// instantiates its kernel for the tasks it lists only
template <int... TASKS, typename F>
static void with_task(int task, F&& f) {
    if (!((task == TASKS && (f(std::integral_constant<int, TASKS>{}), true)) || ...)) f(std::integral_constant<int, WL_TASK_DRIFT>{});
}

// The step specs of the shipped Drift-family configs (make_task("drift") / "hound_4wd" / "f1tenth_drift" and the lowered Drift
// and F1Tenth train / play cfgs): RWD or 4WD action map, clip bounding, no reverse, pushes and observation noise on, no
// wheel-mass DR, decimation 4 x 1 sub-step.  The duo kernel is instantiated for these; every other config runs its generic body.
static constexpr uint32_t SPEC_DRIFT_RWD = spec_key(StepSpec{WL_ACT_RWD, WL_BOUND_CLIP, 1, 1, 1, 0, 4, 1});
static constexpr uint32_t SPEC_DRIFT_4WD = spec_key(StepSpec{WL_ACT_4WD, WL_BOUND_CLIP, 1, 1, 1, 0, 4, 1});
// f(std::integral_constant<uint32_t, K>{}) for the listed spec key K equal to `spec`, else for K = 0 (the generic instantiation)
template <uint32_t... KS, typename F>
static void with_spec(uint32_t spec, F&& f) {
    if (!((spec == KS && (f(std::integral_constant<uint32_t, KS>{}), true)) || ...)) f(std::integral_constant<uint32_t, 0u>{});
}

static inline void ensure_device(const wl_sim* sim) {
    int cur = -1;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != sim->device) cudaSetDevice(sim->device);   // launches go to the handle's device
}
static inline size_t groups_bytes(int n) { return (size_t)WL_NUM_GROUPS * (size_t)n * 16u; }
static inline size_t align256(size_t x) { return (x + 255u) & ~(size_t)255u; }

// ---------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------
// ---- per-step bookkeeping without a grid-wide sync (layout + protocol: wl_globals in the header) ---------------------
// step counter of this launch: the host's value, or (negative host value = -1 - k) device base + k
__device__ __forceinline__ uint32_t decode_step(const wl_globals* __restrict__ gl, uint32_t t_arg) {
    return ((int32_t)t_arg < 0) ? __ldcg(&gl->step_base) + (0xFFFFFFFFu - t_arg) : t_arg;
}
// Programmatic dependent launch (sm_90+): a step kernel lets the next launch of the stream start its prologue right away
// (launch_dependents first thing) and itself waits for the previous kernel's memory to be final (wait) before the first
// read of anything a previous launch may have written.  Both are no-ops for a launch without the PDL attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// W(t): the weights step t-1 used, plus increase_reward_weight_over_time (curriculums.py:23-35) for the counter value t
// reached by the step that just ended -- the reference calls it from _reset_idx, i.e. only if >= 1 env reset in step t-1.
// Every thread of the launch evaluates this identically (no thread writes what another one reads here).
__device__ __forceinline__ void load_weights(const wl_config& c, const wl_globals* __restrict__ gl, uint32_t t, float wts[WL_MAX_REW_TERMS]) {
    const float4* wp = reinterpret_cast<const float4*>(gl->rew_weight[(t + 1u) & 1u]);
    const float4 w0 = __ldcg(wp), w1 = __ldcg(wp + 1);
    wts[0] = w0.x; wts[1] = w0.y; wts[2] = w0.z; wts[3] = w0.w; wts[4] = w1.x; wts[5] = w1.y; wts[6] = w1.z; wts[7] = w1.w;
    if (c.curr_n > 0 && t != 0u && (t % (uint32_t)c.max_episode_length) == 0u) {
        if (__ldcg(&gl->acc[(t + 2u) % 3u][8]) > 0.0f && __ldcg(&gl->curr_applied_t) != t) {     // (not already applied in place by the host path)
            const int E = (int)(t / (uint32_t)c.max_episode_length);
            for (int k = 0; k < c.curr_n; ++k) {
                if (E / c.curr_every[k] > c.curr_max[k]) continue;
                if ((E + 1) % c.curr_every[k] == 0) {
                    const int slot = c.curr_slot[k];
#pragma unroll
                    for (int q = 0; q < WL_MAX_REW_TERMS; ++q) if (q == slot) wts[q] += c.curr_inc[k];
                }
            }
        }
    }
}
// extras["log"] row of the step whose accumulators are `row`: means of the episode sums over the reset envs divided by
// max_episode_length_s (RewardManager.reset), then the counts.  Lanes 0..15 of one warp, one element each.
__device__ __forceinline__ void publish_log_row(const wl_config& c, wl_globals* __restrict__ gl, uint32_t row, int lane) {
    const float v = (lane < 16) ? __ldcg(&gl->acc[row][lane]) : 0.0f;
    const float cnt = __shfl_sync(0xffffffffu, v, 8);
    float* lp = gl->log_ptr[row];
    float out = (lane < WL_MAX_REW_TERMS) ? v / (r_max(cnt, 1.0f) * c.episode_length_s) : v;
    if (lane < 16) {
        if (cnt > 0.0f) gl->last_log[lane] = out;            // extras["log"] persists until the next step that resets an env
        else out = gl->last_log[lane];
        if (lp != nullptr) lp[lane] = out;
    }
}
// The janitor: ONE warp of the launch -- the first warp of an EXTRA CTA appended to the grid (blockIdx.x == gridDim.x - 1)
// that owns no envs, so that no env warp starts its dependent chain late.
__device__ __forceinline__ void janitor(const wl_config& c, wl_globals* __restrict__ gl, uint32_t t, const float wts[WL_MAX_REW_TERMS],
                                        float* __restrict__ d_log) {
    const int lane = threadIdx.x & 31;
    if (t != 0u) publish_log_row(c, gl, (t + 2u) % 3u, lane);          // step t-1 (complete: its kernel has finished)
    if (lane < 16) gl->acc[(t + 1u) % 3u][lane] = 0.0f;                // re-arm the row step t+1 will use
    float w = wts[0];
#pragma unroll
    for (int q = 1; q < WL_MAX_REW_TERMS; ++q) w = (lane == q) ? wts[q] : w;
    if (lane < WL_MAX_REW_TERMS) gl->rew_weight[t & 1u][lane] = w;     // W(t), read by step t+1
    if (lane == 0) gl->log_ptr[t % 3u] = d_log;
}
// true in the janitor CTA, whose first warp has then run the janitor.  wts: W(t) when the caller has already loaded it.
__device__ __forceinline__ bool janitor_cta(const wl_config& c, wl_globals* __restrict__ gl, uint32_t t, float* __restrict__ d_log,
                                            const float* wts = nullptr) {
    if (blockIdx.x != gridDim.x - 1) return false;
    if (threadIdx.x < 32) {
        float wj[WL_MAX_REW_TERMS];
        if (wts == nullptr) { load_weights(c, gl, t, wj); wts = wj; }
        janitor(c, gl, t, wts, d_log);
    }
    return true;
}
template <int WIDTH = 32>
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = WIDTH / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// Finished envs -> this step's accumulator row: warp-shuffle reduce, one RED set per warp (no fence, no ticket: the
// kernel boundary publishes the row to the next launch).  acc layout: [0..7] episode sums, [8] #reset, [9+j] #envs whose
// termination term j fired (tmask bit j).  WIDTH = 8: only lanes 0..7 can contribute, and the lanes above add zeros to the
// full butterfly, so three steps give lanes 0..7 the same nonzero sums; lanes 0..15 then issue the 16 REDs side by side.
// SPREAD (WIDTH = 32): likewise lanes 0..15 issue the REDs, by select and predicate rather than 16 branches in lane 0.
template <int WIDTH = 32, bool SPREAD = false>
__device__ __forceinline__ bool log_accumulate(float* __restrict__ acc, bool contrib, uint32_t tmask,
                                               const float sums[WL_MAX_REW_TERMS]) {
    const unsigned any_c = __ballot_sync(0xffffffffu, contrib);
    if (!any_c) return false;
    float vals[16];
#pragma unroll
    for (int k = 0; k < WL_MAX_REW_TERMS; ++k) vals[k] = contrib ? sums[k] : 0.0f;
    vals[8] = contrib ? 1.0f : 0.0f;
#pragma unroll
    for (int j = 0; j < WL_MAX_TERM_TERMS; ++j) vals[9 + j] = (contrib && ((tmask >> j) & 1u)) ? 1.0f : 0.0f;
#pragma unroll
    for (int k = 0; k < 16; ++k) vals[k] = warp_sum<WIDTH>(vals[k]);
    if (WIDTH < 32) {
        const int lane = threadIdx.x & 31, m = lane & 7;
        float a = vals[0], b = vals[8];
#pragma unroll
        for (int k = 1; k < 8; ++k) { a = sel(m == k, vals[k], a); b = sel(m == k, vals[8 + k], b); }
        a = __shfl_sync(0xffffffffu, a, m); b = __shfl_sync(0xffffffffu, b, m);
        const float v = (lane < 8) ? a : b;                   // lane k < 16: element k, as lanes 0..7 hold it
        if (lane < 16 && v != 0.0f) atomicAdd(&acc[lane], v);
    } else if (SPREAD) {
        const int lane = threadIdx.x & 31;
        float v = vals[0];
#pragma unroll
        for (int k = 1; k < 16; ++k) v = sel(lane == k, vals[k], v);
        if (lane < 16 && v != 0.0f) atomicAdd(&acc[lane], v);
    } else if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 16; ++k) if (vals[k] != 0.0f) atomicAdd(&acc[k], vals[k]);
    }
    return true;
}

// One thread per env.  TASK selects the MDP + terrain at compile time.
#ifndef WL_STEP_MIN_BLOCKS
#define WL_STEP_MIN_BLOCKS 4      // 4 CTAs x 128 threads / SM (<= 128 registers); overridable for occupancy A/B builds
#endif
// STAGE 0: the whole env.step.  STAGE 1 / 2: the same code cut after section E (wl_step_stage_a / wl_step_stage_b), so that
// host-side (Python) reward and termination terms can run between "rewards" and "reset" exactly where the reference's
// managers would call them; the state round-trips through HBM losslessly, so 1 + 2 == 0 bit for bit.
// STAGE 3 / 4: stage 2 cut once more, after the interval pushes (wl_step_stage_b1: F, H) and before the commands and the
// observation (wl_step_stage_b2: G, I), so that host-side event terms run in between (DESIGN 6o).  Stage 4 reads nothing
// but the state buffer: whatever the host wrote there in between is what its command and observation are formed from.
struct StageIO { uint8_t* tmask; const uint8_t* extra_terminated; const uint8_t* extra_truncated; };
template <int TASK, int STAGE = 0>
__global__ void __launch_bounds__(128, WL_STEP_MIN_BLOCKS)
wl_step_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, wl_globals* __restrict__ gl, Terrain T,
               const float2* __restrict__ action, float* __restrict__ obs, float* __restrict__ rew,
               uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o, float* __restrict__ d_log, uint32_t t_arg,
               StageIO sio = StageIO{nullptr, nullptr, nullptr}) {
    constexpr bool ELEV = (TASK == WL_TASK_ELEVATION), VIS = (TASK == WL_TASK_VISUAL);
    pdl_trigger();
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    pdl_wait();
    const uint32_t t = decode_step(gl, t_arg);
    const VisualMap vm = VIS ? visual_map(c, T.hf) : VisualMap{nullptr, nullptr};
    bool done = false;
    uint32_t tmask = 0u;
    EnvState e;
    float wts[WL_MAX_REW_TERMS];            // W(t): issued with the state loads so the latency hides behind the integrator
    if (STAGE != 4) load_weights(c, gl, t, wts);
    if (STAGE != 1 && STAGE != 4 && janitor_cta(c, gl, t, d_log, wts)) return;
    if (STAGE == 4) {
        if (i < n) load_env(st, n, i, e, ELEV, c.dr_wheel_mass_enable != 0, c.d_inv_Iw);
    } else if (STAGE == 2 || STAGE == 3) {
        if (i < n) {
            load_env(st, n, i, e, ELEV, c.dr_wheel_mass_enable != 0, c.d_inv_Iw);
            tmask = sio.tmask[i];
            if (sio.extra_truncated && sio.extra_truncated[i]) tmask |= 1u;            // host-side time-out style term
            if (sio.extra_terminated && sio.extra_terminated[i]) tmask |= 0x80u;       // host-side termination term
            const DoneBytes db = done_bytes(tmask);
            terminated_o[i] = db.terminated;
            truncated_o[i] = db.truncated;
            done = tmask != 0u;
        }
    } else if (i < n) {
        load_env(st, n, i, e, ELEV, c.dr_wheel_mass_enable != 0, c.d_inv_Iw);
        // A. action manager
        float2 a = action[i];
        e.prev_action[0] = e.action[0]; e.prev_action[1] = e.action[1];
        e.action[0] = a.x; e.action[1] = a.y;
        float wheel_target[4], steer_target[2];
        process_action(c, a.x, a.y, wheel_target, steer_target);
        // B. decimation x (actuators -> integrator)
        Chassis b = chassis_from_env(c, e);
        StepConsts kc = make_step_consts<4>(c, e);
        run_substeps<TASK, 1>(c, T, e, b, wheel_target, c.dc_effort, steer_target, kc);
        const M3 R = env_from_chassis(c, e, b);
        // C. counters   D. terminations   E. rewards
        e.ep_len += 1;
        const bool time_out = e.ep_len >= c.max_episode_length;
        float f[WL_MAX_REW_TERMS];
        V3 vb = rotT(R, e.v);
        if (ELEV) {
            tmask = elev_terms(c, e, R, vb, (e.omega[0] + e.omega[1]) + (e.omega[2] + e.omega[3]), time_out, f);
        } else if (VIS) {
            tmask = visual_terms(c, vm, e, vb, time_out, f);
        } else {
            const bool oob = drift_off_track(c, e.p.x, e.p.y);
            drift_reward_terms(c, e.steer[0], e.steer[1], det_atan2(vb.y, vb.x), e.p, vb, b.wb, e.w.z, oob, time_out, f);
            tmask = drift_term_mask(time_out, oob);
        }
        tmask &= (uint32_t)c.term_enable;
        rew[i] = weigh_rewards(c, wts, f, e.sums);
        if (STAGE == 1) {                    // cut: state (with this step's episode sums) back to HBM, term bits for stage 2
            sio.tmask[i] = (uint8_t)tmask;
            store_env(st, n, i, e, ELEV);
            return;
        }
        const DoneBytes db = done_bytes(tmask);
        terminated_o[i] = db.terminated;
        truncated_o[i] = db.truncated;
        if (STAGE == 0 && sio.tmask != nullptr) sio.tmask[i] = (uint8_t)tmask;      // per-term masks (wl_set_term_bits)
        done = tmask != 0u;
    }
    if (STAGE == 1) return;
    // F. auto-reset + per-step episode log (warp-shuffle reduction over the finished envs)
    if (STAGE != 4) log_accumulate(gl->acc[t % 3u], done, tmask, e.sums);
    if (i < n) {
        const uint32_t gid = (uint32_t)(c.env_id_offset + i);
        if (done) reset_env(c, TASK, vm, e, gid, t);
        if (STAGE == 3) {                    // cut: H, then the post-reset, post-push state back to HBM for stage 4
            if (!VIS && !ELEV) interval_pushes(c, e, gid, t, c.d_step_dt);
            store_env(st, n, i, e, ELEV);
            return;
        }
        // G. commands   H. interval events (post-reset state)   I. observations
        if (VIS) {
            float o[8]; visual_proprio(c, e, o);
            const int camf = vis_cam_floats(c);              // the camera floats come first (wl_camera_kernel fills them)
            float4* row = reinterpret_cast<float4*>(obs + (size_t)(WL_OBS_DIM_VISUAL + camf) * i + camf);
            row[0] = make_float4(o[0], o[1], o[2], o[3]); row[1] = make_float4(o[4], o[5], o[6], o[7]);
        } else if (ELEV) {
            elev_command_update(c, e, gid, t, c.d_step_dt);
            float o[13]; elev_proprio(c, e, euler_xyz(e.qw, e.qx, e.qy, e.qz), o);
            float* row = obs + (size_t)WL_OBS_DIM_ELEV * i;
#pragma unroll
            for (int k = 0; k < 13; ++k) row[k] = o[k];
        } else {
            if (STAGE != 4) interval_pushes(c, e, gid, t, c.d_step_dt);
            blind_obs(c, e, gid, t, RNG_OBS, 0u, obs + (size_t)WL_OBS_DIM_BLIND * i);
        }
        if (STAGE != 4 || ELEV) store_env(st, n, i, e, ELEV);     // (stage 4 changes the command groups only)
    }
}

// Four lanes per env (lane = wheel).  Same arithmetic, same results; the per-wheel work runs in parallel and the
// chassis is integrated redundantly in the 4 lanes.  Used when N is too small to fill the chip with one thread/env.
// quad_env_step = sections A..I of ONE env.step() on register-resident state `e` (lane-local view, see load_env_quad).
// lane w of an env's quad computes ONE of the three euler angles (lane 0 roll, 1 pitch, 2 and 3 yaw), wrapped to [0, 2 pi)
// SEL: the pitch override, the atan2 zero cases and the wrap as selects, with no lane-divergent region.  The pitch root is
// needed only for |sin_pitch| < 1, where (1 - s)(1 + s) >= 2^-24 is normal, so the fast-path root is the IEEE one.
template <bool SEL = false>
__device__ __forceinline__ float euler_lane(float qw, float qx, float qy, float qz, int w) {
    float sin_roll = 2.0f * fm(qw, qx, qy * qz), cos_roll = fm(-2.0f, fm(qx, qx, qy * qy), 1.0f);
    float sin_pitch = 2.0f * fm(qw, qy, -(qz * qx));
    float sin_yaw = 2.0f * fm(qw, qz, qx * qy), cos_yaw = fm(-2.0f, fm(qy, qy, qz * qz), 1.0f);
    float ay = (w == 0) ? sin_roll : (w == 1) ? sin_pitch : sin_yaw;
    if (SEL) {
        const float ax = sel(w == 1, fsqrt_norm((1.0f - sin_pitch) * (1.0f + sin_pitch)), (w == 0) ? cos_roll : cos_yaw);
        const float ovr = (sin_pitch < 0.0f) ? -1.57079632679489661923f : 1.57079632679489661923f;
        return wrap_2pi(sel(w == 1 && fabsf(sin_pitch) >= 1.0f, ovr, det_atan2_sel(ay, ax)));
    }
    float ax = (w == 0) ? cos_roll : (w == 1) ? sqrtf((1.0f - sin_pitch) * (1.0f + sin_pitch)) : cos_yaw;
    float ang = det_atan2(ay, ax);
    if (w == 1 && fabsf(sin_pitch) >= 1.0f) ang = (sin_pitch < 0.0f) ? -1.57079632679489661923f : 1.57079632679489661923f;
    return wrap_2pi(ang);
}

// lane w of the quad of env i (n = c.num_envs).  A whole quad is live or not; a dead quad shadows the last env (ii, gid; it
// stores nothing) so that the quad shuffles stay convergent.  base = the quad's first lane in the warp.
struct QuadLane { int i, w; bool live; int ii; uint32_t gid; unsigned base; };
__device__ __forceinline__ QuadLane quad_lane(const wl_config& c, int n, int i, int w) {
    const bool live = i < n;
    const int ii = live ? i : n - 1;
    return QuadLane{i, w, live, ii, (uint32_t)(c.env_id_offset + ii), (threadIdx.x & 31u) & ~3u};
}

template <int TASK>
__device__ __forceinline__ void quad_env_step(const wl_config& c, const Terrain& T, const VisualMap& vm, float* __restrict__ acc_row,
                                              const float wts[WL_MAX_REW_TERMS], EnvState& e, const QuadLane& L, uint32_t t, float2 a,
                                              const float znoise[4], float* __restrict__ obs_row, float* __restrict__ rew,
                                              uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o,
                                              uint8_t* __restrict__ term_bits = nullptr) {
    constexpr bool ELEV = (TASK == WL_TASK_ELEVATION), VIS = (TASK == WL_TASK_VISUAL);
    const int i = L.i, w = L.w;
    const bool live = L.live;
    const uint32_t gid = L.gid;
    const unsigned base = L.base;
    // A. action manager (redundant in the 4 lanes)
    e.prev_action[0] = e.action[0]; e.prev_action[1] = e.action[1];
    e.action[0] = a.x; e.action[1] = a.y;
    float wheel_target[4], steer_target[2];
    process_action(c, a.x, a.y, wheel_target, steer_target);
    const float my_target = (w == 0) ? wheel_target[0] : (w == 1) ? wheel_target[1] : (w == 2) ? wheel_target[2] : wheel_target[3];
    const float my_effort = (w == 0) ? c.dc_effort[0] : (w == 1) ? c.dc_effort[1] : (w == 2) ? c.dc_effort[2] : c.dc_effort[3];
    float my_steer_target[2] = {(w == 3) ? steer_target[1] : steer_target[0], 0.0f};
    // B. decimation x (actuators -> integrator)
    Chassis b = chassis_from_env(c, e);
    StepConsts kc = make_step_consts<1>(c, e);
    const float my_targets[4] = {my_target, 0.0f, 0.0f, 0.0f}, my_efforts[4] = {my_effort, 0.0f, 0.0f, 0.0f};
    run_substeps<TASK, 4>(c, T, e, b, my_targets, my_efforts, my_steer_target, kc);
    M3 R = env_from_chassis(c, e, b);
    // C./D./E. counters, terminations, rewards (redundant in the 4 lanes)
    e.ep_len += 1;
    const bool time_out = e.ep_len >= c.max_episode_length;
    V3 vb = rotT(R, e.v);
    uint32_t tmask;
    float f[WL_MAX_REW_TERMS];
    if (ELEV) {
        float o01 = e.omega[0] + __shfl_xor_sync(0xffffffffu, e.omega[0], 1);      // (w0+w1), (w2+w3)
        float osum = o01 + __shfl_xor_sync(0xffffffffu, o01, 2);                   // (w0+w1)+(w2+w3)
        tmask = elev_terms(c, e, R, vb, osum, time_out, f);
    } else if (VIS) {
        tmask = visual_terms(c, vm, e, vb, time_out, f);
    } else {
        const float steer_l = __shfl_sync(0xffffffffu, e.steer[0], base + 2), steer_r = __shfl_sync(0xffffffffu, e.steer[0], base + 3);
        const bool oob = drift_off_track(c, e.p.x, e.p.y);
        drift_reward_terms(c, steer_l, steer_r, det_atan2(vb.y, vb.x), e.p, vb, b.wb, e.w.z, oob, time_out, f);
        tmask = drift_term_mask(time_out, oob);
    }
    // I'. observation inputs from the post-physics state, formed HERE so that this lane's euler atan2 overlaps the reward
    // terms' atan2 / sqrt chains in one basic block; an env that resets (or gets pushed) redoes them below -- the rare path
    float eu_k = 0.0f;
    V3 wbo{0.0f, 0.0f, 0.0f};
    if (!VIS) eu_k = euler_lane(e.qw, e.qx, e.qy, e.qz, w);
    if (!VIS && !ELEV) wbo = rotT(R, e.w);                        // (R^T of the WORLD rate, as the oracle forms it: not b.wb bit for bit)
    tmask &= (uint32_t)c.term_enable;
    const float total = weigh_rewards(c, wts, f, e.sums);
    const bool done = tmask != 0u;
    if (live && w == 0) {
        const DoneBytes db = done_bytes(tmask);
        rew[i] = total; terminated_o[i] = db.terminated; truncated_o[i] = db.truncated;
        if (term_bits != nullptr) term_bits[i] = (uint8_t)tmask;      // per-term masks for TerminationManager.get_term
    }
    // F. per-step episode log: one contribution per env (lane 0 of each live quad), then auto-reset
    log_accumulate(acc_row, done && live && (w == 0), tmask, e.sums);
    if (done) {
        reset_env(c, TASK, vm, e, gid, t);
        if (!VIS) eu_k = euler_lane(e.qw, e.qx, e.qy, e.qz, w);
        if (!VIS && !ELEV) { R = rotmat(e.qw, e.qx, e.qy, e.qz); vb = rotT(R, e.v); wbo = rotT(R, e.w); }   // (the oracle's own operations: signed zeros)
    }
    if (ELEV) elev_command_update(c, e, gid, t, c.d_step_dt);
    else if (!VIS) {
        // H. interval pushes: never on the step an env resets (fresh timers exceed step_dt), so R is still the rotation of e.q
        if (interval_pushes(c, e, gid, t, c.d_step_dt)) { vb = rotT(R, e.v); wbo = rotT(R, e.w); }
    }
    if (VIS) {      // 8 proprioceptive floats, no noise, no euler: lanes 0 and 1 write one float4 each
        float o[8]; visual_proprio(c, e, o);
        if (live && w < 2) {
            float4* row = reinterpret_cast<float4*>(obs_row + vis_cam_floats(c));
            row[w] = (w == 0) ? make_float4(o[0], o[1], o[2], o[3]) : make_float4(o[4], o[5], o[6], o[7]);
        }
    } else if (ELEV) {
        V3 eu{__shfl_sync(0xffffffffu, eu_k, base + 0), __shfl_sync(0xffffffffu, eu_k, base + 1), __shfl_sync(0xffffffffu, eu_k, base + 2)};
        float o[13]; elev_proprio(c, e, eu, o);
        if (live) {
            // lane w writes o[w], o[w+4], o[w+8] (and lane 0 also o[12]): 4-byte rows, scalar stores
            const float v0 = (w == 0) ? o[0] : (w == 1) ? o[1] : (w == 2) ? o[2] : o[3];
            const float v1 = (w == 0) ? o[4] : (w == 1) ? o[5] : (w == 2) ? o[6] : o[7];
            const float v2 = (w == 0) ? o[8] : (w == 1) ? o[9] : (w == 2) ? o[10] : o[11];
            obs_row[w] = v0; obs_row[w + 4] = v1; obs_row[w + 8] = v2;
            if (w == 0) obs_row[12] = o[12];
        }
    } else {
        // blind_obs_quad shuffles: every lane of the warp calls it, dead quads only skip the stores
        blind_obs_quad(c, e, w, eu_k, vb, wbo, znoise, obs_row, live);
    }
}

template <int TASK>
__global__ void __launch_bounds__(128)
wl_step_quad_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, wl_globals* __restrict__ gl, Terrain T,
                    const float2* __restrict__ action, float* __restrict__ obs, float* __restrict__ rew,
                    uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o, float* __restrict__ d_log, uint32_t t_arg,
                    uint8_t* __restrict__ term_bits) {
    constexpr bool ELEV = (TASK == WL_TASK_ELEVATION), VIS = (TASK == WL_TASK_VISUAL);
    pdl_trigger();
    const VisualMap vm = VIS ? visual_map(c, T.hf) : VisualMap{nullptr, nullptr};
    const int n = c.num_envs;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const QuadLane L = quad_lane(c, n, tid >> 2, tid & 3);      // (blockDim is a multiple of 4)
    pdl_wait();
    const uint32_t t = decode_step(gl, t_arg);
    if (janitor_cta(c, gl, t, d_log)) return;
    EnvState e;
    QuadRaw raw;
    quad_issue_loads(st, n, L.ii, L.w, raw, ELEV, c.dr_wheel_mass_enable != 0);
    const float2 a = action[L.ii];
    float wts[WL_MAX_REW_TERMS];
    load_weights(c, gl, t, wts);
    // the observation noise depends on (env id, step) only: drawn here, while the state loads are in flight (nothing above
    // has consumed a loaded value yet)
    float zn[4];
    if (!ELEV && !VIS) quad_obs_noise(c, L.w, L.gid, t, RNG_OBS, 0u, zn); else zn[0] = zn[1] = zn[2] = zn[3] = 0.0f;
    quad_unpack(raw, L.w, e, ELEV, c.dr_wheel_mass_enable != 0, c.d_inv_Iw);
    quad_env_step<TASK>(c, T, vm, gl->acc[t % 3u], wts, e, L, t, a, zn, obs + (size_t)obs_row_floats(c, TASK) * L.ii, rew, terminated_o, truncated_o, term_bits);
    if (L.live) store_env_quad(st, n, L.i, L.w, e, ELEV);
}

// ---------------------------------------------------------------------------------------
// Drift-family step in the latency-optimised geometry for small N: CTA = 2 warps for 8 envs.  Warp 0 (the "env warp")
// is the quad (lane = wheel) and carries ONLY what is on the dependent chain: state loads -> integrator sub-steps ->
// terminations -> reset -> pushes -> observations -> state stores.  Warp 1 (the "aux warp", lane = env) does everything
// that is not on that chain, concurrently on another scheduler: the action map (ready before the first sub-step needs the
// targets), the observation-noise and push draws (counter based: functions of (env, step) only) and -- once the env warp
// has published the post-physics state in shared memory -- reward terms, episode sums, reward / done stores and the
// episode log.  Hand-offs are named barriers (bar.arrive / bar.sync), each used once per launch.  Same arithmetic as
// wl_step_quad_kernel, operation for operation.
// ---------------------------------------------------------------------------------------
#define WL_DUO_ENVS 8
// A CTA is the env warp, the aux warp and, when the whole grid is resident at once with it (duo_block), a third "spacer" warp
// that exits at once.  The warps of an SM's CTAs take consecutive scheduler (sub-partition) slots: with 2-warp CTAs the
// env warps of the ~4 CTAs per SM at 4096 envs sat two per scheduler on two of the four schedulers; with 3 slots per CTA
// each env warp has a scheduler of its own (measured with %warpid on H100, DESIGN.md 6e).  The spacer warp holds
// registers, so at 8192 envs it would leave CTAs waiting for a second wave: there the CTA stays at 2 warps.
#define WL_DUO_THREADS 96
// The deep-chained step's CTA: four env warps (warps 0..3, 8 envs each) and one aux warp (warp 4, lane = env) for 32 envs.
// Its grids share the SMs with the grids before them, so CTA slots and registers per env bound how many are in flight:
// one aux warp per 32 envs instead of per 8 holds 440 instead of 704 registers per env (DESIGN.md 6e).
#define WL_DEEP_ENV_WARPS 4
#define WL_DEEP_ENVS (WL_DUO_ENVS * WL_DEEP_ENV_WARPS)
#define WL_DEEP_THREADS (32 * (WL_DEEP_ENV_WARPS + 1))
// how a single-GPU duo step runs (duo_chain_mode, DESIGN.md 6e): wl_step_duo_kernel waiting at entry / chained (skips
// that wait; the aux warp waits, then triggers) / wl_step_duo_deep_kernel (triggers at entry, waits before exit)
enum { WL_CHAIN_NONE = 0, WL_CHAIN_SHALLOW = 1, WL_CHAIN_DEEP = 2 };
// the staging of a CTA of E envs: row q0 + q belongs to quad q of the env warp whose first row is q0
template <int E>
struct DuoShared {
    float tgt[E][8];                // wheel_target[4], steer_target[2]
    float noise[E][12];             // observation noise normals (Philox blocks 0..2)
    float push[E][8];               // hf fired, dvx, dvy, dwz_hf, t_hf_new, lf fired, dwz_lf, t_lf_new
    float fin[E][16];               // post-physics: p(3) vb(3) wb(3) wz_world steer_l steer_r raw-tmask(bits)
    __align__(16) float rst[E][16];             // reset outcome: px py qw qz t_hf t_lf (DriftReset, timers after this step) vb(3) wbo(3) euler[wheel lane]
    __align__(16) float obs[E * WL_OBS_DIM_BLIND];              // the observation rows of the CTA, staged for 128-bit stores
    __align__(16) float rewrow[E];                              // the CTA's rewards and done bytes, staged the same way
    __align__(8) uint8_t maskrow[2][E];
};
// NT: the threads that meet at the barrier (every warp of the CTA but the spacer)
template <int NT>
__device__ __forceinline__ void bar_arrive(int id) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "n"(NT) : "memory"); }
template <int NT>
__device__ __forceinline__ void bar_sync(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(NT) : "memory"); }

// ---- phase trace of the duo kernel (diagnostic build only: -DWL_DUO_TRACE, tools/duo_trace.py; without the macro the
// kernel's machine code is unchanged).  Every warp that owns envs stamps %globaltimer at its hand-offs and appends one
// record.  A stamp takes a value as `dep` and is predicated on it, so it is issued only once that value has arrived.
#ifdef WL_DUO_TRACE
// (the aux warp stamps TR_BAR1 at its bar.arrive 1 and TR_ARRIVE2 once it passes bar.sync 2)
enum { TR_ENTRY, TR_PARAMS, TR_WAITED, TR_LOADS, TR_BAR1, TR_PASS0, TR_ARRIVE2 = TR_PASS0 + 8, TR_LAST, TR_AUX_ARRIVE3, TR_AUX_WAITED, TR_EXIT, TR_N };
struct DuoTraceRec {
    unsigned long long st;          // the env set (state buffer) of the launch
    uint32_t t, cta, smid, warpid;  // step counter, blockIdx.x, %smid, %warpid
    uint32_t role, passes, warp, pad;   // 0 env warp, 1 aux warp; sub-step passes stamped; warp index in the CTA
    unsigned long long ts[TR_N];    // %globaltimer, ns (0: not stamped)
    uint32_t ck[6];                 // env warp: %clock (SM cycles) at bar.sync 1 and at the end of sub-step passes 0..3; pad
};
__device__ DuoTraceRec* g_duo_trace;
__device__ unsigned int g_duo_trace_cap, g_duo_trace_n;
__device__ __forceinline__ unsigned long long tr_now(uint32_t dep) {
    unsigned long long ts;
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %1, 0x7fc00001;\n mov.u64 %0, 0;\n @p mov.u64 %0, %%globaltimer;\n}"
                 : "=l"(ts) : "r"(dep) : "memory");
    return ts;
}
__device__ __forceinline__ uint32_t tr_clock(uint32_t dep) {
    uint32_t ck;
    asm volatile("{\n .reg .pred p;\n setp.ne.u32 p, %1, 0x7fc00001;\n mov.u32 %0, 0;\n @p mov.u32 %0, %%clock;\n}"
                 : "=r"(ck) : "r"(dep) : "memory");
    return ck;
}
#define TR_DECL unsigned long long tr_[TR_N] = {}; uint32_t tr_pass_ = 0, tr_ck_[6] = {}
#define TR(k, dep) (tr_[k] = tr_now((uint32_t)(dep)))
#define TR_CK_BAR1(dep) (tr_ck_[0] = tr_clock((uint32_t)(dep)))
#define TR_PASS_HOOK , [&](const EnvState& es) { \
    if (tr_pass_ < 4) tr_ck_[1 + tr_pass_] = tr_clock(__float_as_uint(es.omega[0])); \
    if (tr_pass_ < 8) tr_[TR_PASS0 + tr_pass_] = tr_now(__float_as_uint(es.omega[0])); ++tr_pass_; }
__device__ __forceinline__ void tr_commit(const unsigned long long* ts, uint32_t passes, const float4* st, uint32_t t, uint32_t role,
                                          const uint32_t* ck) {
    if ((threadIdx.x & 31) != 0 || g_duo_trace == nullptr) return;
    const unsigned int k = atomicAdd(&g_duo_trace_n, 1u);
    if (k >= g_duo_trace_cap) return;
    DuoTraceRec& r = g_duo_trace[k];
    uint32_t smid, warpid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%warpid;" : "=r"(warpid));
    r.st = reinterpret_cast<unsigned long long>(st); r.t = t; r.cta = blockIdx.x; r.smid = smid; r.warpid = warpid;
    r.role = role; r.passes = passes; r.warp = threadIdx.x >> 5;
    for (int i = 0; i < TR_N; ++i) r.ts[i] = ts[i];
    for (int i = 0; i < 6; ++i) r.ck[i] = ck[i];
}
#define TR_COMMIT(role) tr_commit(tr_, tr_pass_, st, t, role, tr_ck_)
#else
#define TR_DECL
#define TR(k, dep)
#define TR_CK_BAR1(dep)
#define TR_PASS_HOOK
#define TR_COMMIT(role)
#endif

// lane g < 13: the line of state group g holding envs env0..env0+7 (8 x 16 bytes); lane 13: their actions; lane 14: the
// wheel-inertia group when the wheel-mass DR reads it.  An L2 prefetch is safe before griddepcontrol.wait: L2 is the
// point of coherence, so a line the previous kernel writes afterwards is not left stale there.
__device__ __forceinline__ void duo_prefetch_l2(const float4* st, const float2* action, int n, int env0, int lane, bool wm) {
    const void* p = (lane < 13) ? static_cast<const void*>(st + (size_t)lane * n + env0)
                  : (lane == 13) ? static_cast<const void*>(action + env0)
                  : (lane == 14 && wm) ? static_cast<const void*>(st + (size_t)WL_G_PIW * n + env0) : nullptr;
    if (p != nullptr) asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// FAN = 0: no peer: the fan-out / multicast / packed-row code is not in the kernel at all (the dependent stream of one warp per
// scheduler also pays for instruction fetch: several hundred static instructions fewer on the single-GPU path).
// FAN = 2: multicast only -- the host has checked that num_envs is a multiple of 8 and the output rows are aligned, so every row
// is a full wide store: local copy + ONE multimem.st, no per-peer loops, no element-wise fallback in the instruction stream.
// FAN = 1: the general fan-out (per-peer stores; multicast for the rows that qualify).
// K: the step spec key (wl_step.cuh, Spec).  The single-GPU path (FAN = 0) is instantiated for the shipped Drift-family specs
// (with_spec): their action map, bounding, push and noise branches are folded and the sub-step trip counts are constants;
// K = 0 reads the config at run time (every other config, and FAN = 1 / 2).
// Launch bounds: 4 CTAs per SM hold the 4096-env grid with the spacer warp (duo_block); without the minimum, ptxas traded
// a register spill in the env warp for an occupancy no launch here needs.
// DEEP: the deep-chained form (wl_step_duo_deep_kernel, FAN = 0 only), in CTAs of WL_DEEP_ENV_WARPS env warps and one aux
// warp; otherwise warp 0 is the env warp and warp 1 the aux warp.
template <int FAN, uint32_t K, bool DEEP>
__device__ __forceinline__ void duo_step(const wl_config& c, float4* __restrict__ st, wl_globals* __restrict__ gl,
                                         const float2* __restrict__ action, float* __restrict__ obs, float* __restrict__ rew,
                                         uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o, float* __restrict__ d_log,
                                         uint32_t t_arg, uint8_t* __restrict__ term_bits, const PeerFan& pf, int chained) {
    using S = Spec<K>;
    constexpr int EW = DEEP ? WL_DEEP_ENV_WARPS : 1;            // env warps; the aux warp is warp EW
    constexpr int ENVS = WL_DUO_ENVS * EW, NT = 32 * (EW + 1);
    __shared__ DuoShared<ENVS> sh;
    TR_DECL;
    TR(TR_ENTRY, 0);
    if (!DEEP && threadIdx.x >= 64) return;                     // the spacer warp
    const int n = c.num_envs;
    TR(TR_PARAMS, n);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int env0 = blockIdx.x * ENVS;
    const int q0 = DEEP ? WL_DUO_ENVS * warp : 0;               // an env warp's first env in the CTA (and staging row)
    // Launched with PDL, this prologue runs while the previous step's tail is still running: up to the wait it reads only
    // kernel parameters and requests into L2 the lines both warps load first (the janitor CTA owns no envs).
    if ((DEEP ? warp < EW : warp == 0) && env0 + q0 < n) duo_prefetch_l2(st, action, n, env0 + q0, lane, S::wheel_mass(c));
    // chained (FAN = 0 only; duo_chain_mode): every launch that may still run beside this grid is a duo step of another env
    // set that touches none of this launch's buffers, and this set's previous step has completed (the host checks).  The
    // env CTAs then start on entry.  Shallow (chained != 0): the aux warp waits before the weights and the episode log
    // (wl_globals: janitor t-1) and before its trigger, and the janitor CTA waits here, so every CTA triggers only once the
    // grid before has completed.  Deep: every CTA, the janitor's included, triggers here and nothing waits until the aux
    // warp's and the janitor's last instruction, so the next grid launches once this one is resident; the wait before exit
    // keeps a grid from completing before its predecessor.  DESIGN.md 6e.
    constexpr bool deep = DEEP;
    const bool early = FAN == 0 && (deep || chained != 0) && blockIdx.x != gridDim.x - 1;
    if (deep) pdl_trigger();
    else if (!early) pdl_wait();
    TR(TR_WAITED, n);
    const uint32_t t = decode_step(gl, t_arg);
    if (janitor_cta(c, gl, t, d_log)) {
        if (deep) pdl_wait();
        return;
    }
    const Terrain T{nullptr};
    if (warp == EW) {
        // ================= aux warp: lane j < ENVS <-> env env0 + j =================
        const int j = DEEP ? lane : lane & 7;
        const int i = env0 + j;
        const bool live = (lane < ENVS) && (i < n);
        const int ii = (i < n) ? i : n - 1;
        const uint32_t gid = (uint32_t)(c.env_id_offset + ii);
        float2 a = make_float2(0.0f, 0.0f);
        float4 s0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), s1 = s0;
        float t_hf = 0.0f, t_lf = 0.0f;
        if (lane < ENVS) {
            a = action[ii];
            s0 = ldg4(st, WL_G_SUM0, n, ii); s1 = ldg4(st, WL_G_SUM1, n, ii);
            const float* fst = reinterpret_cast<const float*>(st);
            t_hf = fst[((size_t)WL_G_LINVEL * n + ii) * 4 + 3]; t_lf = fst[((size_t)WL_G_ANGVEL * n + ii) * 4 + 3];
        }
        float wts[WL_MAX_REW_TERMS];
        if (!S::fixed) {
            if (early && !deep) {
                pdl_wait();
                TR(TR_AUX_WAITED, n);
            }
            load_weights(c, gl, t, wts);
        }
        TR(TR_LOADS, __float_as_uint(a.x) ^ __float_as_uint(s1.w) ^ __float_as_uint(t_lf));
        // A. action map -> targets of the whole env step
        if (lane < ENVS) {
            float wt[4], stt[2];
            process_action<K>(c, a.x, a.y, wt, stt);
            sh.tgt[j][0] = wt[0]; sh.tgt[j][1] = wt[1]; sh.tgt[j][2] = wt[2]; sh.tgt[j][3] = wt[3];
            sh.tgt[j][4] = stt[0]; sh.tgt[j][5] = stt[1];
        }
        bar_arrive<NT>(1);
        TR(TR_BAR1, __float_as_uint(sh.tgt[j][0]));
        // N. observation noise: lane = (env, Philox block); deep, lane = env and its three blocks as independent chains
        if (DEEP) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float z[4];
                quad_obs_noise<K>(c, k, gid, t, RNG_OBS, 0u, z);
                sh.noise[j][4 * k + 0] = z[0]; sh.noise[j][4 * k + 1] = z[1]; sh.noise[j][4 * k + 2] = z[2]; sh.noise[j][4 * k + 3] = z[3];
            }
        } else if (lane < 24) {
            const int jn = lane / 3, k = lane - 3 * jn;
            const int in_ = (env0 + jn < n) ? env0 + jn : n - 1;
            float z[4];
            quad_obs_noise<K>(c, k, (uint32_t)(c.env_id_offset + in_), t, RNG_OBS, 0u, z);
            sh.noise[jn][4 * k + 0] = z[0]; sh.noise[jn][4 * k + 1] = z[1]; sh.noise[jn][4 * k + 2] = z[2]; sh.noise[jn][4 * k + 3] = z[3];
        }
        // P. interval pushes of an env that does NOT reset this step (the env warp ignores them otherwise)
        if (lane < ENVS) {
            float hf = 0.0f, dvx = 0.0f, dvy = 0.0f, dwh = 0.0f, lf = 0.0f, dwl = 0.0f;
            if (S::push_enable(c)) {
                t_hf = t_hf - c.d_step_dt;
                if (t_hf < 1.0e-6f) {
                    uint4 r = philox4x32(c.seed, gid, t, RNG_PUSH_HF, 0u);
                    dvx = uniform(r.x, -c.push_hf_range[0], c.push_hf_range[0]);
                    dvy = uniform(r.y, -c.push_hf_range[1], c.push_hf_range[1]);
                    dwh = uniform(r.z, -c.push_hf_range[2], c.push_hf_range[2]);
                    t_hf = uniform(r.w, c.push_hf_interval[0], c.push_hf_interval[1]);
                    hf = 1.0f;
                }
                t_lf = t_lf - c.d_step_dt;
                if (t_lf < 1.0e-6f) {
                    uint4 r = philox4x32(c.seed, gid, t, RNG_PUSH_LF, 0u);
                    dwl = uniform(r.x, -c.push_lf_yaw, c.push_lf_yaw);
                    t_lf = uniform(r.y, c.push_lf_interval[0], c.push_lf_interval[1]);
                    lf = 1.0f;
                }
            }
            sh.push[j][0] = hf; sh.push[j][1] = dvx; sh.push[j][2] = dvy; sh.push[j][3] = dwh; sh.push[j][4] = t_hf;
            sh.push[j][5] = lf; sh.push[j][6] = dwl; sh.push[j][7] = t_lf;
        }
        // shallow, fixed spec: the wait on the previous grid and the CTA's trigger come before the reset draw, the aux warp's
        // longest draw, rather than after it (Drift measured 7 % faster on H100, DESIGN.md 6e).  Nothing the draw reads is
        // written by another launch; the weights are still loaded after the wait.
        if (S::fixed && early && !deep) {
            pdl_wait();
            TR(TR_AUX_WAITED, n);
            pdl_trigger();
        }
        // Z. the auto-reset outcome of every env, whether it resets or not: lane = (env, wheel) as in the env warp, which
        // only selects it after bar.sync 3.  A reset env is not pushed: its fresh timers exceed step_dt and only count down.
        // (Drawn before the action map, in the shadow of the loads, it delayed bar.arrive 1 and the step took longer.)
        // Deep, lane = env: one draw per env, and the euler angle of each wheel lane.
        if (DEEP) {
            DriftReset d = drift_reset_draw(c, gid, t);
            EnvState z;
            drift_reset_apply(d, z);
            const M3 R = rotmat(z.qw, z.qx, z.qy, z.qz);
            const V3 vb = rotT(R, z.v), wbo = rotT(R, z.w);
            if (S::push_enable(c)) { d.t_hf = d.t_hf - c.d_step_dt; d.t_lf = d.t_lf - c.d_step_dt; }
            float* ro = sh.rst[j];
            reinterpret_cast<float4*>(ro)[0] = make_float4(d.px, d.py, d.qw, d.qz);
            reinterpret_cast<float4*>(ro)[1] = make_float4(d.t_hf, d.t_lf, vb.x, vb.y);
            reinterpret_cast<float4*>(ro)[2] = make_float4(vb.z, wbo.x, wbo.y, wbo.z);
            float eu[4];
#pragma unroll
            for (int w = 0; w < 4; ++w) eu[w] = euler_lane(z.qw, z.qx, z.qy, z.qz, w);
            reinterpret_cast<float4*>(ro)[3] = make_float4(eu[0], eu[1], eu[2], eu[3]);
            TR(TR_AUX_ARRIVE3, __float_as_uint(eu[3]));
        } else {
            const QuadLane Lz = quad_lane(c, n, env0 + (lane >> 2), lane & 3);
            DriftReset d = drift_reset_draw(c, Lz.gid, t);
            EnvState z;
            drift_reset_apply(d, z);
            const float eu = euler_lane(z.qw, z.qx, z.qy, z.qz, Lz.w);
            const M3 R = rotmat(z.qw, z.qx, z.qy, z.qz);
            const V3 vb = rotT(R, z.v), wbo = rotT(R, z.w);
            if (S::push_enable(c)) { d.t_hf = d.t_hf - c.d_step_dt; d.t_lf = d.t_lf - c.d_step_dt; }
            float* ro = sh.rst[lane >> 2];
            if (Lz.w == 0) {
                reinterpret_cast<float4*>(ro)[0] = make_float4(d.px, d.py, d.qw, d.qz);
                reinterpret_cast<float4*>(ro)[1] = make_float4(d.t_hf, d.t_lf, vb.x, vb.y);
                reinterpret_cast<float4*>(ro)[2] = make_float4(vb.z, wbo.x, wbo.y, wbo.z);
            }
            ro[12 + Lz.w] = eu;
            TR(TR_AUX_ARRIVE3, __float_as_uint(eu));
        }
        bar_arrive<NT>(3);
        // (a fixed spec loads the weights only now, off the way to bar.arrive 1: only the rewards below read them)
        if (S::fixed) load_weights(c, gl, t, wts);
        // R. rewards, episode sums, reward / done stores, episode log -- on the post-physics state the env warps publish
        bar_sync<NT>(2);
        TR(TR_ARRIVE2, __float_as_uint(sh.fin[j][0]));
        pdl_trigger();                                          // (see the env warp's trigger)
        uint32_t tmask = 0u;
        float sums[WL_MAX_REW_TERMS] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        bool done = false;
        if (lane < ENVS) {
            const float* fi = sh.fin[j];
            const V3 p{fi[0], fi[1], fi[2]}, vb{fi[3], fi[4], fi[5]}, wb{fi[6], fi[7], fi[8]};
            const uint32_t raw = __float_as_uint(fi[12]);
            const bool time_out = (raw & 1u) != 0u, oob = (raw & 2u) != 0u;
            float f[WL_MAX_REW_TERMS];
            if (S::fixed) drift_reward_terms<true>(c, fi[10], fi[11], det_atan2_sel(vb.y, vb.x), p, vb, wb, fi[9], oob, time_out, f);
            else drift_reward_terms(c, fi[10], fi[11], det_atan2(vb.y, vb.x), p, vb, wb, fi[9], oob, time_out, f);
            tmask = raw & (uint32_t)c.term_enable;
            const float total = weigh_rewards<S::fixed>(c, wts, f, sums);
            done = tmask != 0u;
            // fan-out active, full CTA, aligned rows: 32 + 8 + 8 contiguous bytes leave as four wide stores (one NVLink /
            // multicast write each instead of 24 small ones); otherwise element by element (without peers the staging round
            // trip would sit at the kernel's tail for nothing)
            const bool packed = (FAN == 2) || ((FAN == 1) && ((pf.n | pf.mc) != 0) && (env0 + WL_DUO_ENVS <= n) && ((reinterpret_cast<uintptr_t>(rew + env0) & 15u) == 0) &&
                                (((reinterpret_cast<uintptr_t>(terminated_o + env0) | reinterpret_cast<uintptr_t>(truncated_o + env0)) & 7u) == 0));
            const auto [tb, ub] = done_bytes(tmask);
            if (packed) {
                sh.rewrow[lane] = total; sh.maskrow[0][lane] = tb; sh.maskrow[1][lane] = ub;
                __syncwarp(0xffu);
                if (lane < 2) fan_store16<FAN == 2>(pf, reinterpret_cast<float4*>(rew + env0) + lane, reinterpret_cast<const float4*>(sh.rewrow)[lane]);
                else if (lane == 2) fan_store8<FAN == 2>(pf, reinterpret_cast<float2*>(terminated_o + env0), *reinterpret_cast<const float2*>(sh.maskrow[0]));
                else if (lane == 3) fan_store8<FAN == 2>(pf, reinterpret_cast<float2*>(truncated_o + env0), *reinterpret_cast<const float2*>(sh.maskrow[1]));
            } else if (S::fixed) {
                st_global_if(reinterpret_cast<float*>(rew + i), total, live);
                st_global_if(terminated_o + i, tb, live); st_global_if(truncated_o + i, ub, live);
            } else if (live) {
                if (FAN == 1) { fan_store(pf, &rew[i], total); fan_store(pf, &terminated_o[i], tb); fan_store(pf, &truncated_o[i], ub); }
                else { rew[i] = total; terminated_o[i] = tb; truncated_o[i] = ub; }
            }
            if (live && term_bits != nullptr) term_bits[i] = (uint8_t)tmask;
        }
        if (DEEP) log_accumulate<32, S::fixed>(gl->acc[t % 3u], done && live, tmask, sums);
        else log_accumulate<S::fixed ? 8 : 32>(gl->acc[t % 3u], done && live, tmask, sums);
        if (deep && S::fixed) {                                 // (predicated: no branch ahead of the exit wait below)
#pragma unroll
            for (int k = 0; k < WL_MAX_REW_TERMS; ++k) sums[k] = done ? 0.0f : sums[k];
            st_global_if(st + (size_t)WL_G_SUM0 * n + i, make_float4(sums[0], sums[1], sums[2], sums[3]), live);
            st_global_if(st + (size_t)WL_G_SUM1 * n + i, make_float4(sums[4], sums[5], sums[6], sums[7]), live);
        } else if (live) {
            if (done) {
#pragma unroll
                for (int k = 0; k < WL_MAX_REW_TERMS; ++k) sums[k] = 0.0f;
            }
            stg4(st, WL_G_SUM0, n, i, make_float4(sums[0], sums[1], sums[2], sums[3]));
            stg4(st, WL_G_SUM1, n, i, make_float4(sums[4], sums[5], sums[6], sums[7]));
        }
        TR(TR_LAST, __float_as_uint(sums[7]));
        if (deep) {
            pdl_wait();
            TR(TR_EXIT, n);
        }
        TR_COMMIT(1);
        return;
    }
    // ================= env warp: the quad (lane = wheel), 8 envs from env0 + q0 =================
    const int q = lane >> 2, qs = q0 + q;                       // qs: the quad's staging row
    const int env8 = env0 + q0;
    const QuadLane L = quad_lane(c, n, env8 + q, lane & 3);
    const int i = L.i, w = L.w, ii = L.ii;
    const bool live = L.live;
    const bool wm = S::wheel_mass(c);
    EnvState e;
    QuadRaw raw;
    quad_issue_loads(st, n, ii, w, raw, false, wm, false);
    const float2 a = action[ii];
    TR(TR_LOADS, __float_as_uint(raw.pos.x) ^ __float_as_uint(raw.kd) ^ __float_as_uint(a.y));
    quad_unpack(raw, w, e, false, wm, c.d_inv_Iw);
    // A. action manager: only the bookkeeping; the map itself comes from the aux warp
    e.prev_action[0] = e.action[0]; e.prev_action[1] = e.action[1];
    e.action[0] = a.x; e.action[1] = a.y;
    const float my_effort = (w == 0) ? c.dc_effort[0] : (w == 1) ? c.dc_effort[1] : (w == 2) ? c.dc_effort[2] : c.dc_effort[3];
    // B. decimation x (actuators -> integrator)
    Chassis b = chassis_from_env(c, e);
    StepConsts kc = make_step_consts<1, K>(c, e);
    bar_sync<NT>(1);
    const float my_targets[4] = {sh.tgt[qs][w], 0.0f, 0.0f, 0.0f}, my_efforts[4] = {my_effort, 0.0f, 0.0f, 0.0f};
    const float my_steer_target[2] = {sh.tgt[qs][(w == 3) ? 5 : 4], 0.0f};
    TR(TR_BAR1, __float_as_uint(my_targets[0]));
    TR_CK_BAR1(__float_as_uint(my_targets[0]));
    // with a fixed spec the pass is free of divergent regions (measured faster on H100, DESIGN.md 6e)
    run_substeps<WL_TASK_DRIFT, 4, K, S::fixed>(c, T, e, b, my_targets, my_efforts, my_steer_target, kc TR_PASS_HOOK);
    M3 R = env_from_chassis(c, e, b);
    // C./D. counters, terminations (the env warp needs `done` for the reset; the reward side lives in the aux warp)
    e.ep_len += 1;
    const bool time_out = e.ep_len >= c.max_episode_length;
    V3 vb = rotT(R, e.v);
    const float steer_l = __shfl_sync(0xffffffffu, e.steer[0], L.base + 2), steer_r = __shfl_sync(0xffffffffu, e.steer[0], L.base + 3);
    const bool oob = drift_off_track(c, e.p.x, e.p.y);
    const uint32_t raw_mask = drift_term_mask(time_out, oob);
    if (w == 0) {
        float* fo = sh.fin[qs];
        fo[0] = e.p.x; fo[1] = e.p.y; fo[2] = e.p.z; fo[3] = vb.x; fo[4] = vb.y; fo[5] = vb.z;
        fo[6] = b.wb.x; fo[7] = b.wb.y; fo[8] = b.wb.z; fo[9] = e.w.z; fo[10] = steer_l; fo[11] = steer_r;
        fo[12] = __uint_as_float(raw_mask);
    }
    bar_arrive<NT>(2);
    TR(TR_ARRIVE2, raw_mask);
    // The next step's launch may begin once every CTA is here (the aux warp triggers after bar.sync 2; the spacer warp and
    // the janitor CTA have exited).  Triggering at entry instead let each grid launch the next while only partly resident,
    // and triggering after the last store was slower on H100 (DESIGN.md 6e).  Chained, the env warp does not trigger: a
    // shallow launch's successor relies on every trigger following a wait, and a deep launch has triggered at entry.
    if (!early) pdl_trigger();
    // I'. observation inputs from the post-physics state (an env that resets / gets pushed takes others below)
    float eu_k = euler_lane<S::fixed>(e.qw, e.qx, e.qy, e.qz, w);
    V3 wbo = rotT(R, e.w);
    const bool done = (raw_mask & (uint32_t)c.term_enable) != 0u;
    // F. auto-reset and H. interval pushes: the reset outcome, the push draws and the noise come from the aux warp
    bar_sync<NT>(3);
    if (S::fixed) {
        // as selects over both outcomes, so that a warp with resetting and pushed envs does not split.  The pushed velocities
        // are rotated whether a push fired or not: unpushed, they are the same values, so the same bits.
        const float4* ro = reinterpret_cast<const float4*>(sh.rst[qs]);
        const float4 r0 = ro[0], r1 = ro[1], r2 = ro[2];
        const float eu_r = sh.rst[qs][12 + w];
        EnvState er = e;
        drift_reset_apply(DriftReset{r0.x, r0.y, r0.z, r0.w, r1.x, r1.y}, er);
        V3 vbp = vb, wbp = wbo;
        if (S::push_enable(c)) {
            const float* pu = sh.push[qs];
            const bool hf = pu[0] != 0.0f, lf = pu[5] != 0.0f;
            e.v.x = hf ? e.v.x + pu[1] : e.v.x; e.v.y = hf ? e.v.y + pu[2] : e.v.y;
            e.w.z = hf ? e.w.z + pu[3] : e.w.z; e.w.z = lf ? e.w.z + pu[6] : e.w.z;
            e.t_hf = pu[4]; e.t_lf = pu[7];
            vbp = rotT(R, e.v); wbp = rotT(R, e.w);
        }
        e = done ? er : e;
        vb = done ? V3{r1.z, r1.w, r2.x} : vbp; wbo = done ? V3{r2.y, r2.z, r2.w} : wbp;
        eu_k = done ? eu_r : eu_k;
    } else if (done) {                                                 // (sums and log: aux warp)
        const float4* ro = reinterpret_cast<const float4*>(sh.rst[qs]);
        const float4 r0 = ro[0], r1 = ro[1], r2 = ro[2];
        drift_reset_apply(DriftReset{r0.x, r0.y, r0.z, r0.w, r1.x, r1.y}, e);
        vb = V3{r1.z, r1.w, r2.x}; wbo = V3{r2.y, r2.z, r2.w};
        eu_k = sh.rst[qs][12 + w];
    } else if (S::push_enable(c)) {
        const float* pu = sh.push[qs];
        bool fired = false;
        if (pu[0] != 0.0f) { e.v.x = e.v.x + pu[1]; e.v.y = e.v.y + pu[2]; e.w.z = e.w.z + pu[3]; fired = true; }
        e.t_hf = pu[4];
        if (pu[5] != 0.0f) { e.w.z = e.w.z + pu[6]; fired = true; }
        e.t_lf = pu[7];
        if (fired) { vb = rotT(R, e.v); wbo = rotT(R, e.w); }
    }
    const int k4 = (w < 3) ? 4 * w : 0;
    const float zn[4] = {sh.noise[qs][k4], sh.noise[qs][k4 + 1], sh.noise[qs][k4 + 2], sh.noise[qs][k4 + 3]};
    // the env warp's 8 observation rows are 448 contiguous bytes: staged in shared memory and written as 28 x 128-bit stores
    // (full sectors towards HBM, NVLink peers and -- zero-copy host transport -- PCIe, instead of 8-byte pieces)
    float* orow0 = obs + (size_t)WL_OBS_DIM_BLIND * env8;
    if ((FAN == 2) || (env8 + WL_DUO_ENVS <= n && (reinterpret_cast<uintptr_t>(orow0) & 15u) == 0)) {
        const float4 v = blind_obs_quad_values<S::fixed>(c, e, w, eu_k, vb, wbo, zn);
        float* so = sh.obs + WL_OBS_DIM_BLIND * qs + 4 * w;
        so[0] = v.x; so[1] = v.y;
        if (w < 3) { so[2] = v.z; so[3] = v.w; }
        __syncwarp();
        if (lane < (WL_DUO_ENVS * WL_OBS_DIM_BLIND) / 4)
        {
            if (FAN) fan_store16<FAN == 2>(pf, reinterpret_cast<float4*>(orow0) + lane, reinterpret_cast<const float4*>(sh.obs + WL_OBS_DIM_BLIND * q0)[lane]);
            else reinterpret_cast<float4*>(orow0)[lane] = reinterpret_cast<const float4*>(sh.obs + WL_OBS_DIM_BLIND * q0)[lane];
        }
    } else {
        if (FAN == 1) blind_obs_quad(c, e, w, eu_k, vb, wbo, zn, obs + (size_t)WL_OBS_DIM_BLIND * ii, live, pf);
        else blind_obs_quad(c, e, w, eu_k, vb, wbo, zn, obs + (size_t)WL_OBS_DIM_BLIND * ii, live);
    }
    if (S::fixed) store_env_quad_sel(st, n, i, w, e, live);
    else if (live) store_env_quad(st, n, i, w, e, false, false);
    TR(TR_LAST, __float_as_uint(e.omega[0]));
    TR_COMMIT(0);
}
template <int FAN, uint32_t K>
__global__ void __launch_bounds__(WL_DUO_THREADS, 4)
wl_step_duo_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, wl_globals* __restrict__ gl,
                   const float2* __restrict__ action, float* __restrict__ obs, float* __restrict__ rew,
                   uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o, float* __restrict__ d_log, uint32_t t_arg,
                   uint8_t* __restrict__ term_bits, const __grid_constant__ PeerFan pf, int chained) {
    duo_step<FAN, K, false>(c, st, gl, action, obs, rew, terminated_o, truncated_o, d_log, t_arg, term_bits, pf, chained);
}
// The deep-chained step (FAN = 0) is an entry of its own, so that the machine code of the unchained and shallow steps, which
// single-set rollouts run, carries none of its branches.  Launch bounds: 4 CTAs of 160 threads per SM (at most 96
// registers: 5 warps per scheduler), 128 envs per SM against the 80 of 2-warp CTAs.
template <uint32_t K>
__global__ void __launch_bounds__(WL_DEEP_THREADS, 4)
wl_step_duo_deep_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, wl_globals* __restrict__ gl,
                        const float2* __restrict__ action, float* __restrict__ obs, float* __restrict__ rew,
                        uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o, float* __restrict__ d_log, uint32_t t_arg,
                        uint8_t* __restrict__ term_bits, const __grid_constant__ PeerFan pf) {
    duo_step<0, K, true>(c, st, gl, action, obs, rew, terminated_o, truncated_o, d_log, t_arg, term_bits, pf, 1);
}

// ---------------------------------------------------------------------------------------
// fused policy: actor + critic 64x64 ELU MLPs in front of the quad step (one warp = 8 envs; lane w of a quad owns hidden
// units [16w, 16w+16) of BOTH nets; layer outputs are exchanged through 4 KB of shared memory per warp)
// ---------------------------------------------------------------------------------------
#define WL_HID 64
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
struct PolicyOffsets { int32_t o[13]; };

// critic_obs_dim: the width of the critic's input (the asymmetric network); 0 = obs_dim
static int policy_offsets(int obs_dim, int32_t off[13], int critic_obs_dim = 0) {
    auto al = [](int x) { return (x + 3) & ~3; };
    int p = 0;
    for (int net = 0; net < 2; ++net) {
        const int out = net == 0 ? 2 : 1, in = (net == 1 && critic_obs_dim > 0) ? critic_obs_dim : obs_dim;
        off[net * 6 + 0] = p; p = al(p + al(in) * WL_HID);           // rows padded to a multiple of 4 (zeros)
        off[net * 6 + 1] = p; p = al(p + WL_HID);
        off[net * 6 + 2] = p; p = al(p + WL_HID * WL_HID);
        off[net * 6 + 3] = p; p = al(p + WL_HID);
        off[net * 6 + 4] = p; p = al(p + WL_HID * out);
        off[net * 6 + 5] = p; p = al(p + out);
    }
    off[12] = p; p = al(p + 2);
    return p;
}

// ---- shared-memory mbarriers and TMA copies that complete on them (one definition of each PTX form) --------------------
// mbar_init_fence makes the initialised barriers visible to the async proxy before any copy names them
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect(uint64_t* b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait_parity(uint64_t* b, uint32_t parity) {
    const uint32_t mb = smem_u32(b);
    uint32_t ok = 0;
    while (!ok)
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(mb), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(b)) : "memory");
}
// the box of the 2-D tensor map at element (x, y) -> shared
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* tmap, int x, int y, uint64_t* b) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ float elu(float x) { return x > 0.0f ? x : __expf(x) - 1.0f; }

// one hidden layer for a register tile of 4 units x 4 envs: per 4 inputs, 4 LDS.128 of activations (one per env, a pure
// broadcast: the whole warp shares the env tile) and 4 LDS.128 of input-major weights (conflict-free: the 16 lanes of a
// net read 256 contiguous bytes) feed 64 FMAs; accumulation order per output = bias, then inputs ascending.
// mlp_tile_accum adds inputs 0..nin-1 to acc (nin a multiple of 4), so a layer can also be run in K chunks.
__device__ __forceinline__ void mlp_tile_accum(const float* W, const float* x0, int xstride, int nin, float acc[4][4]) {
#pragma unroll 4
    for (int j = 0; j < nin; j += 4) {
        float xs[4][4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float4 v = *reinterpret_cast<const float4*>(x0 + e * xstride + j);
            xs[e][0] = v.x; xs[e][1] = v.y; xs[e][2] = v.z; xs[e][3] = v.w;
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const float4 w0 = *reinterpret_cast<const float4*>(W + (j + jj) * WL_HID);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float x = xs[e][jj];
                acc[e][0] = fmaf(w0.x, x, acc[e][0]); acc[e][1] = fmaf(w0.y, x, acc[e][1]);
                acc[e][2] = fmaf(w0.z, x, acc[e][2]); acc[e][3] = fmaf(w0.w, x, acc[e][3]);
            }
        }
    }
}
__device__ __forceinline__ void mlp_tile_layer(const float* W, const float* bias, const float* x0, int xstride, int nin, float acc[4][4]) {
    const float4 b0 = *reinterpret_cast<const float4*>(bias);
#pragma unroll
    for (int e = 0; e < 4; ++e) { acc[e][0] = b0.x; acc[e][1] = b0.y; acc[e][2] = b0.z; acc[e][3] = b0.w; }
    mlp_tile_accum(W, x0, xstride, nin, acc);
}

// the policy's Gaussian head (rsl_rl ActorCritic.act): z ~ N(0,1)^2 from the generator's policy stream for (global env,
// step), a = mean + std * z, log-prob summed over the two action dims.  wl_act_step and wl_policy_act share it, so their
// samples agree bit for bit.
__device__ __forceinline__ void policy_noise(uint64_t seed, uint32_t gid, uint32_t t, float& z0, float& z1) {
    const uint4 r = philox4x32(seed, gid, t, RNG_POLICY, 0u);
    box_muller(r.x, r.y, z0, z1);
}
__device__ __forceinline__ void gaussian_head(float m0, float m1, float s0, float s1, float z0, float z1, float2& a, float& lp) {
    a = make_float2(fmaf(s0, z0, m0), fmaf(s1, z1, m1));
    lp = -0.5f * (z0 * z0 + z1 * z1) - __logf(s0) - __logf(s1) - 1.8378770664093453f;   // 2 * 0.5 log(2 pi)
}

__device__ __forceinline__ void mlp_tile_store_elu(float* h0, int hstride, const float acc[4][4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
        *reinterpret_cast<float4*>(h0 + e * hstride) = make_float4(elu(acc[e][0]), elu(acc[e][1]), elu(acc[e][2]), elu(acc[e][3]));
}

#define WL_ACT_ENVS 32                           // envs per CTA: 4096 envs -> 128 CTAs, one per SM
#define WL_ACT_THREADS 256                       // 8 lanes per env for the MLPs (2 warps per scheduler); threads 0..127 = the env quads
#define WL_ACT_XS 20                             // padded observation row
#define WL_ACT_HS (2 * WL_HID + 4)               // padded hidden row, [actor 64 | critic 64 | pad]

// INFER (wl_act_infer_step): the actor mean alone is the action -- no critic, no policy noise, no log-prob; only the actor
// blocks of the blob are copied, and warps 0..3 run the actor with lanes 0-15 and 16-31 on different envs.  Each output
// keeps its summation order, so the actions equal the mean the INFER = false instantiation stores, bit for bit.
template <int TASK, bool INFER = false>
__global__ void __launch_bounds__(WL_ACT_THREADS)
wl_act_step_quad_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, wl_globals* __restrict__ gl, Terrain T,
                        const float* __restrict__ obs_in, const float* __restrict__ blob, int blob_floats, PolicyOffsets po_off,
                        wl_policy_out po, float* __restrict__ obs, float* __restrict__ rew, uint8_t* __restrict__ terminated_o,
                        uint8_t* __restrict__ truncated_o, float* __restrict__ d_log, uint32_t t_arg, int obs_dim) {
    constexpr bool ELEV = (TASK == WL_TASK_ELEVATION), VIS = (TASK == WL_TASK_VISUAL);
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar[2];
    pdl_trigger();
    pdl_wait();
    if (blockIdx.x == gridDim.x - 1) {                       // the janitor CTA; the step is decoded in its branch only
        if (threadIdx.x < 32) {
            const uint32_t tj = decode_step(gl, t_arg);
            float wj[WL_MAX_REW_TERMS];
            load_weights(c, gl, tj, wj); janitor(c, gl, tj, wj, d_log);
        }
        return;
    }
    float* sw = smem;                                        // the whole weight blob (~42 KB)
    float* sx = smem + blob_floats;                          // [32][WL_ACT_XS]
    float* sh = sx + WL_ACT_ENVS * WL_ACT_XS;                // [32][WL_ACT_HS]
    // ---- bulk async copies (TMA, 1-D) bring the blob from L2 into shared memory while the env state loads fly: the two
    // first-layer blocks (7.5 KB) complete on mbar[0], everything else (34 KB) on mbar[1] and lands during layer 1
    if (threadIdx.x == 0) {
        mbar_init(&mbar[0], 1); mbar_init(&mbar[1], 1);
        mbar_init_fence();
        const int a0 = po_off.o[0], a1 = po_off.o[2], c0 = po_off.o[6], c1 = po_off.o[8];
        if constexpr (INFER) {                               // actor W1t | b1, then the rest of the actor
            mbar_expect(&mbar[0], (uint32_t)(a1 - a0) * 4u);
            bulk_g2s(sw + a0, blob + a0, (uint32_t)(a1 - a0) * 4u, &mbar[0]);
            mbar_expect(&mbar[1], (uint32_t)(c0 - a1) * 4u);
            bulk_g2s(sw + a1, blob + a1, (uint32_t)(c0 - a1) * 4u, &mbar[1]);
        } else {
            mbar_expect(&mbar[0], (uint32_t)((a1 - a0) + (c1 - c0)) * 4u);
            bulk_g2s(sw + a0, blob + a0, (uint32_t)(a1 - a0) * 4u, &mbar[0]);
            bulk_g2s(sw + c0, blob + c0, (uint32_t)(c1 - c0) * 4u, &mbar[0]);
            mbar_expect(&mbar[1], (uint32_t)((c0 - a1) + (blob_floats - c1)) * 4u);
            bulk_g2s(sw + a1, blob + a1, (uint32_t)(c0 - a1) * 4u, &mbar[1]);
            bulk_g2s(sw + c1, blob + c1, (uint32_t)(blob_floats - c1) * 4u, &mbar[1]);
        }
    }
    const uint32_t t = decode_step(gl, t_arg);
    const VisualMap vm = VIS ? visual_map(c, T.hf) : VisualMap{nullptr, nullptr};
    const int n = c.num_envs;
    const bool stepper = threadIdx.x < 4 * WL_ACT_ENVS;      // warps 0..3 own the env quads; warps 4..7 only help with the MLPs
    const int q = (threadIdx.x >> 2) & (WL_ACT_ENVS - 1);
    const QuadLane L = quad_lane(c, n, blockIdx.x * WL_ACT_ENVS + q, threadIdx.x & 3);
    EnvState e;
    float wts[WL_MAX_REW_TERMS];
    if (stepper) {
        load_env_quad(st, n, L.ii, L.w, e, ELEV, c.dr_wheel_mass_enable != 0, c.d_inv_Iw);
        load_weights(c, gl, t, wts);
    }
    for (int k = threadIdx.x; k < WL_ACT_ENVS * 16; k += WL_ACT_THREADS) {
        const int eq = k >> 4, j = k & 15, ei = min(blockIdx.x * WL_ACT_ENVS + eq, n - 1);
        sx[eq * WL_ACT_XS + j] = j < obs_dim ? obs_in[(size_t)ei * obs_dim + j] : 0.0f;
    }
    // the policy noise does not depend on the weights: draw it while the copies are in flight
    float z0 = 0.0f, z1 = 0.0f, zn[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (stepper) {
        if constexpr (!INFER) policy_noise(c.seed, L.gid, t, z0, z1);
        if (!ELEV && !VIS) quad_obs_noise(c, L.w, L.gid, t, RNG_OBS, 0u, zn);
    }
    __syncthreads();                                         // mbarrier init visible to every waiter; obs rows written
    mbar_wait_parity(&mbar[0], 0);
    // ---- MLPs: warp k takes envs 4k..4k+3 of the CTA; its 32 lanes tile the 128 (actor | critic) hidden columns 4 at a
    // time, so a lane holds 4 units x 4 envs in registers.  Layer exchanges stay warp-local (__syncwarp).  W1t has obs_dim
    // rows; rows obs_dim..nin1-1 read whatever follows in the blob and meet the zero padding of x.
    if (!INFER || stepper) {                                 // (INFER: warp k takes envs 8k..8k+7, half-warps 4 each)
        const int lane = threadIdx.x & 31, net = INFER ? 0 : lane >> 4, ucol = (lane & 15) * 4;
        const int env0 = INFER ? (threadIdx.x >> 5) * 8 + (lane >> 4) * 4 : (threadIdx.x >> 5) * 4;
        const int nin1 = (obs_dim + 3) & ~3;
        const int oW1 = net ? po_off.o[6] : po_off.o[0], oB1 = net ? po_off.o[7] : po_off.o[1];     // (no dynamic indexing of kernel params)
        const int oW2 = net ? po_off.o[8] : po_off.o[2], oB2 = net ? po_off.o[9] : po_off.o[3];
        float acc[4][4];
        float* h0 = sh + env0 * WL_ACT_HS + net * WL_HID;
        mlp_tile_layer(sw + oW1 + ucol, sw + oB1 + ucol, sx + env0 * WL_ACT_XS, WL_ACT_XS, nin1, acc);
        mlp_tile_store_elu(h0 + ucol, WL_ACT_HS, acc);
        __syncwarp();
        mbar_wait_parity(&mbar[1], 0);                          // layer-2 / head weights have landed (copy overlapped layer 1)
        mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, h0, WL_ACT_HS, WL_HID, acc);
        __syncwarp();                                        // every lane has finished reading layer-1 activations
        mlp_tile_store_elu(h0 + ucol, WL_ACT_HS, acc);
    }
    __syncthreads();                                         // layer-2 activations of all 32 envs are in shared memory
    if (stepper) {
        // output heads: lane w of the env's quad takes hidden units [16w, 16w+16) of both nets, then a quad butterfly
        const float* hrow = sh + q * WL_ACT_HS;
        const float* w3a = sw + po_off.o[4]; const float* w3c = sw + po_off.o[10];
        float m0 = 0.0f, m1 = 0.0f, vv = 0.0f;
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            const int j = 16 * L.w + u;
            if constexpr (INFER) {
                const float xa = hrow[j];
                m0 = fmaf(w3a[2 * j], xa, m0); m1 = fmaf(w3a[2 * j + 1], xa, m1);
            } else {
                const float xa = hrow[j], xc = hrow[WL_HID + j];
                m0 = fmaf(w3a[2 * j], xa, m0); m1 = fmaf(w3a[2 * j + 1], xa, m1);
                vv = fmaf(w3c[j], xc, vv);
            }
        }
        m0 += __shfl_xor_sync(0xffffffffu, m0, 1); m0 += __shfl_xor_sync(0xffffffffu, m0, 2);
        m1 += __shfl_xor_sync(0xffffffffu, m1, 1); m1 += __shfl_xor_sync(0xffffffffu, m1, 2);
        float2 a;
        if constexpr (INFER) {
            m0 += sw[po_off.o[5]]; m1 += sw[po_off.o[5] + 1];
            a = make_float2(m0, m1);
            if (L.live && L.w == 0) reinterpret_cast<float2*>(po.actions)[L.i] = a;
        } else {
            vv += __shfl_xor_sync(0xffffffffu, vv, 1); vv += __shfl_xor_sync(0xffffffffu, vv, 2);
            m0 += sw[po_off.o[5]]; m1 += sw[po_off.o[5] + 1]; vv += sw[po_off.o[11]];
            float lp;
            gaussian_head(m0, m1, sw[po_off.o[12]], sw[po_off.o[12] + 1], z0, z1, a, lp);
            if (L.live && L.w == 0) {
                reinterpret_cast<float2*>(po.actions)[L.i] = a;
                reinterpret_cast<float2*>(po.mean)[L.i] = make_float2(m0, m1);
                po.log_prob[L.i] = lp;
                po.value[L.i] = vv;
            }
        }
        // ---- the env step on the sampled action (INFER: on the mean)
        quad_env_step<TASK>(c, T, vm, gl->acc[t % 3u], wts, e, L, t, a, zn, obs + (size_t)obs_row_floats(c, TASK) * L.ii, rew, terminated_o, truncated_o);
        if (L.live) store_env_quad(st, n, L.i, L.w, e, ELEV);
    }
}

// wl_policy_act_elu: the policy of wl_act_step_quad_kernel<TASK, false> without the env step, for a step that is launched
// separately (the staged step).  The same CTA of 32 envs x 8 lanes, the same blob copies on the two mbarriers, the same
// mlp_tile_layer tiles, quad head butterfly and policy noise (global env id, decoded counter), so actions, mean, log-prob
// and value equal what wl_act_step stores, bit for bit.  No janitor CTA, no env state, no episode log.  It does not trigger
// dependents early: a step launched after it with PDL waits for every action.
// ASYM (wl_policy_act_asym): the critic's first layer reads a second staged row, critic_in [N, critic_dim] padded to
// WL_ACT_XC floats, and the blob's critic W1t block has ceil4(critic_dim) rows; everything else is the same code, so the
// actor's outputs do not depend on the critic input and the critic's keep their summation order.
#define WL_ACT_XC 36                             // padded critic observation row (critic_dim <= 32)
template <bool ASYM>
__device__ __forceinline__ void policy_act_elu_body(const wl_config& c, const wl_globals* __restrict__ gl, const float* __restrict__ obs_in,
                                                    const float* __restrict__ critic_in, int critic_dim, const float* __restrict__ blob,
                                                    int blob_floats, const PolicyOffsets& po_off, const wl_policy_out& po, uint32_t t_arg,
                                                    int obs_dim) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar[2];
    float* sw = smem;                                        // the whole weight blob
    float* sx = smem + blob_floats;                          // [32][WL_ACT_XS]
    float* sh = sx + WL_ACT_ENVS * WL_ACT_XS;                // [32][WL_ACT_HS]
    float* sxc = sh + WL_ACT_ENVS * WL_ACT_HS;               // ASYM: [32][WL_ACT_XC]
    if (threadIdx.x == 0) {                                  // first-layer blocks on mbar[0], the rest on mbar[1]
        mbar_init(&mbar[0], 1); mbar_init(&mbar[1], 1);
        mbar_init_fence();
        const int a0 = po_off.o[0], a1 = po_off.o[2], c0 = po_off.o[6], c1 = po_off.o[8];
        mbar_expect(&mbar[0], (uint32_t)((a1 - a0) + (c1 - c0)) * 4u);
        bulk_g2s(sw + a0, blob + a0, (uint32_t)(a1 - a0) * 4u, &mbar[0]);
        bulk_g2s(sw + c0, blob + c0, (uint32_t)(c1 - c0) * 4u, &mbar[0]);
        mbar_expect(&mbar[1], (uint32_t)((c0 - a1) + (blob_floats - c1)) * 4u);
        bulk_g2s(sw + a1, blob + a1, (uint32_t)(c0 - a1) * 4u, &mbar[1]);
        bulk_g2s(sw + c1, blob + c1, (uint32_t)(blob_floats - c1) * 4u, &mbar[1]);
    }
    const uint32_t t = decode_step(gl, t_arg);
    const int n = c.num_envs;
    const bool head = threadIdx.x < 4 * WL_ACT_ENVS;         // warps 0..3 own the env quads of the heads
    const int q = (threadIdx.x >> 2) & (WL_ACT_ENVS - 1);
    const QuadLane L = quad_lane(c, n, blockIdx.x * WL_ACT_ENVS + q, threadIdx.x & 3);
    for (int k = threadIdx.x; k < WL_ACT_ENVS * 16; k += WL_ACT_THREADS) {
        const int eq = k >> 4, j = k & 15, ei = min(blockIdx.x * WL_ACT_ENVS + eq, n - 1);
        sx[eq * WL_ACT_XS + j] = j < obs_dim ? obs_in[(size_t)ei * obs_dim + j] : 0.0f;
    }
    if constexpr (ASYM) {
        for (int k = threadIdx.x; k < WL_ACT_ENVS * 32; k += WL_ACT_THREADS) {
            const int eq = k >> 5, j = k & 31, ei = min(blockIdx.x * WL_ACT_ENVS + eq, n - 1);
            sxc[eq * WL_ACT_XC + j] = j < critic_dim ? critic_in[(size_t)ei * critic_dim + j] : 0.0f;
        }
    }
    float z0 = 0.0f, z1 = 0.0f;
    if (head) policy_noise(c.seed, L.gid, t, z0, z1);
    __syncthreads();                                         // mbarrier init visible to every waiter; obs rows written
    mbar_wait_parity(&mbar[0], 0);
    {                                                        // warp k: envs 4k..4k+3, lanes tile (actor | critic) 4 units each
        const int lane = threadIdx.x & 31, net = lane >> 4, ucol = (lane & 15) * 4;
        const int env0 = (threadIdx.x >> 5) * 4;
        const int nin1 = (obs_dim + 3) & ~3;
        const int oW1 = net ? po_off.o[6] : po_off.o[0], oB1 = net ? po_off.o[7] : po_off.o[1];
        const int oW2 = net ? po_off.o[8] : po_off.o[2], oB2 = net ? po_off.o[9] : po_off.o[3];
        float acc[4][4];
        float* h0 = sh + env0 * WL_ACT_HS + net * WL_HID;
        if (ASYM && net) mlp_tile_layer(sw + oW1 + ucol, sw + oB1 + ucol, sxc + env0 * WL_ACT_XC, WL_ACT_XC, (critic_dim + 3) & ~3, acc);
        else mlp_tile_layer(sw + oW1 + ucol, sw + oB1 + ucol, sx + env0 * WL_ACT_XS, WL_ACT_XS, nin1, acc);
        mlp_tile_store_elu(h0 + ucol, WL_ACT_HS, acc);
        __syncwarp();
        mbar_wait_parity(&mbar[1], 0);
        mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, h0, WL_ACT_HS, WL_HID, acc);
        __syncwarp();                                        // every lane has finished reading layer-1 activations
        mlp_tile_store_elu(h0 + ucol, WL_ACT_HS, acc);
    }
    __syncthreads();                                         // layer-2 activations of all 32 envs are in shared memory
    if (!head) return;
    const float* hrow = sh + q * WL_ACT_HS;
    const float* w3a = sw + po_off.o[4]; const float* w3c = sw + po_off.o[10];
    float m0 = 0.0f, m1 = 0.0f, vv = 0.0f;
#pragma unroll
    for (int u = 0; u < 16; ++u) {
        const int j = 16 * L.w + u;
        const float xa = hrow[j], xc = hrow[WL_HID + j];
        m0 = fmaf(w3a[2 * j], xa, m0); m1 = fmaf(w3a[2 * j + 1], xa, m1);
        vv = fmaf(w3c[j], xc, vv);
    }
    m0 += __shfl_xor_sync(0xffffffffu, m0, 1); m0 += __shfl_xor_sync(0xffffffffu, m0, 2);
    m1 += __shfl_xor_sync(0xffffffffu, m1, 1); m1 += __shfl_xor_sync(0xffffffffu, m1, 2);
    vv += __shfl_xor_sync(0xffffffffu, vv, 1); vv += __shfl_xor_sync(0xffffffffu, vv, 2);
    m0 += sw[po_off.o[5]]; m1 += sw[po_off.o[5] + 1]; vv += sw[po_off.o[11]];
    float2 a;
    float lp;
    gaussian_head(m0, m1, sw[po_off.o[12]], sw[po_off.o[12] + 1], z0, z1, a, lp);
    if (L.live && L.w == 0) {
        reinterpret_cast<float2*>(po.actions)[L.i] = a;
        reinterpret_cast<float2*>(po.mean)[L.i] = make_float2(m0, m1);
        po.log_prob[L.i] = lp;
        po.value[L.i] = vv;
    }
}
__global__ void __launch_bounds__(WL_ACT_THREADS)
wl_policy_act_elu_kernel(const __grid_constant__ wl_config c, const wl_globals* __restrict__ gl, const float* __restrict__ obs_in,
                         const float* __restrict__ blob, int blob_floats, PolicyOffsets po_off, wl_policy_out po, uint32_t t_arg,
                         int obs_dim) {
    policy_act_elu_body<false>(c, gl, obs_in, nullptr, 0, blob, blob_floats, po_off, po, t_arg, obs_dim);
}
__global__ void __launch_bounds__(WL_ACT_THREADS)
wl_policy_act_asym_kernel(const __grid_constant__ wl_config c, const wl_globals* __restrict__ gl, const float* __restrict__ obs_in,
                          const float* __restrict__ critic_in, int critic_dim, const float* __restrict__ blob, int blob_floats,
                          PolicyOffsets po_off, wl_policy_out po, uint32_t t_arg, int obs_dim) {
    policy_act_elu_body<true>(c, gl, obs_in, critic_in, critic_dim, blob, blob_floats, po_off, po, t_arg, obs_dim);
}

// K consecutive env.step()s in ONE launch (synthetic / scripted-action rollouts, SURVEY 7.7): the state stays in registers
// for the whole rollout, every step still writes its observation / reward / done rows ([K,N,...] slab) and its episode-log
// row.  actions == nullptr => U[-1,1]^2 drawn in-kernel from the counter-based generator (and stored to act_out).
// Bit-identical to K calls of wl_step.  The curriculum is applied by the host-side splitter: [t, t+K) never crosses an
// episode boundary of the global counter when curr_n > 0.
template <int TASK>
__global__ void __launch_bounds__(128)
wl_rollout_quad_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, wl_globals* __restrict__ gl, Terrain T,
                       const float2* __restrict__ action, float2* __restrict__ act_out, float* __restrict__ obs,
                       float* __restrict__ rew, uint8_t* __restrict__ terminated_o, uint8_t* __restrict__ truncated_o,
                       float* __restrict__ d_log, uint32_t t_arg, int K, unsigned* __restrict__ ticket) {
    constexpr bool ELEV = (TASK == WL_TASK_ELEVATION), VIS = (TASK == WL_TASK_VISUAL);
    const uint32_t t0 = decode_step(gl, t_arg);
    const VisualMap vm = VIS ? visual_map(c, T.hf) : VisualMap{nullptr, nullptr};
    const int n = c.num_envs;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const QuadLane L = quad_lane(c, n, tid >> 2, tid & 3);
    EnvState e;
    load_env_quad(st, n, L.ii, L.w, e, ELEV, c.dr_wheel_mass_enable != 0, c.d_inv_Iw);
    float wts[WL_MAX_REW_TERMS];             // W(t0) holds for the whole window (it never crosses an episode boundary)
    load_weights(c, gl, t0, wts);
    if (blockIdx.x == 0 && threadIdx.x < 32) janitor(c, gl, t0, wts, nullptr);      // flushes step t0-1's log row
    const int od = obs_row_floats(c, TASK);
    for (int k = 0; k < K; ++k) {
        const uint32_t t = t0 + (uint32_t)k;
        float2 a;
        if (action != nullptr) a = action[(size_t)k * n + L.ii];
        else {
            uint4 r = philox4x32(c.seed, L.gid, t, RNG_ACTION, 0u);
            a = make_float2(2.0f * u01(r.x) - 1.0f, 2.0f * u01(r.y) - 1.0f);
        }
        if (act_out != nullptr && L.live && L.w == 0) act_out[(size_t)k * n + L.i] = a;
        float zn[4];
        if (!ELEV && !VIS) quad_obs_noise(c, L.w, L.gid, t, RNG_OBS, 0u, zn); else zn[0] = zn[1] = zn[2] = zn[3] = 0.0f;
        quad_env_step<TASK>(c, T, vm, d_log + (size_t)k * WL_LOG_FLOATS, wts, e, L, t, a, zn, obs + ((size_t)k * n + L.ii) * od,
                            rew + (size_t)k * n, terminated_o + (size_t)k * n, truncated_o + (size_t)k * n);
    }
    if (L.live) store_env_quad(st, n, L.i, L.w, e, ELEV);
    // last CTA (ticket, amortised over the K steps of the launch): turn the K accumulator rows into means and leave the
    // globals as K single steps would have: W of the last step in its slot, its raw accumulator row where the next launch
    // looks for it (the curriculum boundary at t0 + K reads its reset count; the next janitor re-publishes it to last_log,
    // which must not then lose the episode sums), nothing pending for the log, the next row re-armed
    if ((threadIdx.x & 31) == 0) __threadfence();
    __syncthreads();
    if (threadIdx.x != 0) return;
    const unsigned tk = atomicAdd(ticket, 1u);
    if (tk != gridDim.x - 1) return;
    __threadfence();
    float last_raw[16];
    for (int k = 0; k < K; ++k) {
        float* row = d_log + (size_t)k * WL_LOG_FLOATS;
        const float cnt = __ldcg(&row[8]);
        if (k == K - 1)
            for (int q = 0; q < 16; ++q) last_raw[q] = __ldcg(&row[q]);
        if (cnt > 0.0f) {
            const float denom = cnt * c.episode_length_s;
            for (int q = 0; q < WL_MAX_REW_TERMS; ++q) row[q] = __ldcg(&row[q]) / denom;
            for (int q = 0; q < 16; ++q) gl->last_log[q] = row[q];
        } else {
            for (int q = 0; q < 16; ++q) row[q] = gl->last_log[q];         // no reset in this step: the previous row persists
        }
    }
    const uint32_t tl = t0 + (uint32_t)K - 1u;
    for (int q = 0; q < WL_MAX_REW_TERMS; ++q) gl->rew_weight[tl & 1u][q] = wts[q];
    for (int q = 0; q < 16; ++q) { gl->acc[tl % 3u][q] = last_raw[q]; gl->acc[(tl + 1u) % 3u][q] = 0.0f; }
    gl->log_ptr[tl % 3u] = nullptr;
    *ticket = 0u;
}

// ---------------------------------------------------------------------------------------
// height-scan observation (ray-caster sensor, elevation/mushr_elevation_env_cfg.py:44-48,74-82,132-142):
// one CTA per env.  The yaw-rotated 2.5 m x 2.5 m footprint fits a WL_TILE x WL_TILE window of the height-field;
// one elected thread pulls that window into shared memory with a single TMA (cp.async.bulk.tensor.2d, completion on
// an mbarrier; out-of-raster elements are zero-filled by the hardware and never read), then 128 threads take the
// 676 vertical rays as bilinear samples from shared memory and write obs[13:689] coalesced.
// ---------------------------------------------------------------------------------------
// window = WL_TILE_W x WL_TILE_H samples.  The footprint needs <= 38 samples per axis; TMA wants the innermost box
// coordinate 16-byte aligned (ox % 4 == 0), so the window starts up to 3 samples early and is 44 wide.
#define WL_TILE_W 44
#define WL_TILE_H 40
#define WL_SCAN_THREADS 128


// The 676 rays of one env out of its shared-memory window: thread t takes rays t, t+128, ... (linear order: all 32 lanes busy,
// fully coalesced stores).  The SIX rays of a thread are independent chains, written branch-free (window indices clamped into
// the tile, the miss value selected at the end) and fully unrolled so that the compiler interleaves them: the loop is bound by
// instruction latency (F2I, LDS, dependent FFMAs), not by bytes.  Per-ray arithmetic unchanged (bit-identical outputs).
struct ScanPose { float bx, by, bz, cy, sy, pz; int ox, oy; };
// the scan constants of env i: ray-caster parent = base_link (root + R (0,0,base_link_z)), yaw of the yaw-aligned rays
// (attach_yaw_only), and the window origin (in samples), which covers base +- (half*sqrt2 + 1 cell)
__device__ __forceinline__ ScanPose scan_pose(const wl_config& c, const float4* __restrict__ st, int n, int i) {
    const float inv = c.d_inv_hf_cell;
    float4 g0 = ldg4(st, WL_G_POS, n, i), g1 = ldg4(st, WL_G_QUAT, n, i);
    EnvState e0; e0.p = V3{g0.x, g0.y, g0.z}; e0.qw = g1.x; e0.qx = g1.y; e0.qy = g1.z; e0.qz = g1.w;
    M3 R = rotmat(e0.qw, e0.qx, e0.qy, e0.qz);
    ScanPose q;
    q.bx = fm(c.base_link_z, R.r[2], e0.p.x); q.by = fm(c.base_link_z, R.r[5], e0.p.y); q.bz = fm(c.base_link_z, R.r[8], e0.p.z);
    yaw_cs(e0, q.cy, q.sy);
    q.pz = e0.p.z;
    const float reach = c.scan_half * 1.41421356237f + c.hf_cell;
    q.ox = ((int)floorf((q.bx - reach - c.hf_x0) * inv)) & ~3;      // two's complement: rounds toward -inf
    q.oy = (int)floorf((q.by - reach - c.hf_y0) * inv);
    return q;
}
// ROW (row terms, DESIGN 6r): the raw world_height_map value (a miss is +inf), then the map term's stages, with the draw of
// ray r at dz[r] (formed before the tile landed)
template <bool ROW = false>
__device__ __forceinline__ void scan_rays(const wl_config& c, const float* __restrict__ tl, const ScanPose& q, float* __restrict__ row, int tid,
                                          const RowStage* __restrict__ ms = nullptr, const float* __restrict__ dz = nullptr) {
    constexpr int ITER = (WL_SCAN_RAYS + WL_SCAN_THREADS - 1) / WL_SCAN_THREADS;
    const float inv = c.d_inv_hf_cell;
    const float fxmax = (float)(c.hf_nx - 1), fymax = (float)(c.hf_ny - 1);
    const float base = q.pz - c.scan_plane_init;
    float v[ITER], tx[ITER], ty[ITER];
    const float* t0[ITER];
    bool inside[ITER];
#pragma unroll
    for (int j = 0; j < ITER; ++j) {                                              // phase 1: ray -> window address, weights
        int r = tid + WL_SCAN_THREADS * j;
        if (r > WL_SCAN_RAYS - 1) r = WL_SCAN_RAYS - 1;                           // the tail threads recompute the last ray (not stored)
        const int ry = (r * 2521) >> 16, rx = r - ry * WL_SCAN_SIDE;             // r / 26, r % 26 for r < 676
        const float lx = fm((float)rx, c.scan_res, -c.scan_half), ly = fm((float)ry, c.scan_res, -c.scan_half);
        const float wx = fm(q.cy, lx, fm(-q.sy, ly, q.bx)), wy = fm(q.sy, lx, fm(q.cy, ly, q.by));
        const float fx = (wx - c.hf_x0) * inv, fy = (wy - c.hf_y0) * inv;
        inside[j] = (fx >= 0.0f) && (fy >= 0.0f) && (fx <= fxmax) && (fy <= fymax);
        int ix = (int)floorf(fx), iy = (int)floorf(fy);
        ix = min(ix, c.hf_nx - 2); iy = min(iy, c.hf_ny - 2);
        tx[j] = fx - (float)ix; ty[j] = fy - (float)iy;
        // (the six F2I/I2F per ray run on the 16-lane pipe, 48 of its cycles per warp-iteration against 64 issue slots: the loop
        //  is issue-bound, and the 2^23-binade tricks that avoid the conversions cost 16 more issue slots per ray -- not taken)
        const int ux = min(max(ix - q.ox, 0), WL_TILE_W - 2), uy = min(max(iy - q.oy, 0), WL_TILE_H - 2);   // no-op for a hit
        t0[j] = tl + uy * WL_TILE_W + ux;
    }
    float z00[ITER], z10[ITER], z01[ITER], z11[ITER];
    asm volatile("" ::: "memory"); __syncwarp();                                  // (compiler fences: keep the phases apart)
#pragma unroll
    for (int j = 0; j < ITER; ++j) {                                              // phase 2: the 24 shared-memory reads in flight together
        z00[j] = t0[j][0]; z10[j] = t0[j][1]; z01[j] = t0[j][WL_TILE_W]; z11[j] = t0[j][WL_TILE_W + 1];
    }
    asm volatile("" ::: "memory"); __syncwarp();
#pragma unroll
    for (int j = 0; j < ITER; ++j) {                                              // phase 3: bilinear sample, height, clip
        const float za = fm(z10[j] - z00[j], tx[j], z00[j]), zb = fm(z11[j] - z01[j], tx[j], z01[j]);
        const float hit = fm(zb - za, ty[j], za);
        const float hs = q.bz - hit - c.scan_offset;                              // mdp.height_scan
        if (ROW) {
            const int r = min(tid + WL_SCAN_THREADS * j, WL_SCAN_RAYS - 1);
            const float h = -hs + base;
            v[j] = row_stage(*ms, inside[j] ? h : __int_as_float(0x7f800000), ms->noise != WL_NOISE_NONE ? dz[r] : 0.0f);
        } else {
        const float hv = r_clamp(-hs + base, -c.obs_clip, c.obs_clip);           // world_height_map, clip
        v[j] = inside[j] ? hv : c.obs_clip;                                       // miss: +inf clipped
        }
    }
#pragma unroll
    for (int j = 0; j < ITER; ++j) {
        const int r = tid + WL_SCAN_THREADS * j;
        if (r < WL_SCAN_RAYS) row[r] = v[j];
    }
}

template <bool USE_TMA>
__global__ void __launch_bounds__(WL_SCAN_THREADS, 8)
wl_scan_kernel(const __grid_constant__ wl_config c, const __grid_constant__ CUtensorMap tmap, const float4* __restrict__ st,
               const float* __restrict__ hf, float* __restrict__ obs) {
    __shared__ __align__(128) float tile[WL_TILE_W * WL_TILE_H];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ ScanPose sp;                  // per-env constants of the scan, formed ONCE by thread 0
    const int i = blockIdx.x;
    if (threadIdx.x == 0) {
        const ScanPose p = scan_pose(c, st, c.num_envs, i);
        sp = p;
        if (USE_TMA) {
            mbar_init(&mbar, 1);
            mbar_init_fence();
            mbar_expect(&mbar, WL_TILE_W * WL_TILE_H * 4);
            tma_load_2d(tile, &tmap, p.ox, p.oy, &mbar);
        }
    }
    __syncthreads();                         // constants + mbarrier visible to everyone
    const ScanPose q = sp;
    if (USE_TMA) {
        mbar_wait_parity(&mbar, 0);          // all threads wait for the bytes
    } else {
        for (int k = threadIdx.x; k < WL_TILE_W * WL_TILE_H; k += WL_SCAN_THREADS) {
            int tx = k % WL_TILE_W, ty = k / WL_TILE_W, gx = q.ox + tx, gy = q.oy + ty;
            tile[k] = (gx >= 0 && gy >= 0 && gx < c.hf_nx && gy < c.hf_ny) ? __ldg(hf + (size_t)gy * c.hf_pitch + gx) : 0.0f;
        }
        __syncthreads();
    }
    scan_rays(c, tile, q, obs + (size_t)WL_OBS_DIM_ELEV * i + 13, threadIdx.x);
}

// ---------------------------------------------------------------------------------------
// The same ray-caster as a TMA producer / consumer PIPELINE (wl_set_scan_tma(2); NOT the default: resident one-tile CTAs per
// SM already hide the set-up + TMA latency, and the ray loop is issue-bound): persistent CTAs (a few per SM) walk the envs; warp 4 is
// the producer -- it reads the next env's pose, forms the per-env constants and issues the cp.async.bulk.tensor.2d of that
// env's window into the other shared-memory stage -- while warps 0..3 take the 676 rays of the current env out of the stage
// that has landed.  full[s] (TMA transaction bytes) and empty[s] (one arrival per consumer warp) are mbarriers; the pose load,
// the constant set-up and the TMA latency of env k+1 hide behind the rays of env k instead of heading every CTA's life.
// Rays are taken in linear order (r = thread + 128 j: all 32 lanes busy, fully coalesced stores).  Same arithmetic.
// ---------------------------------------------------------------------------------------
#define WL_SCAN_STAGES 2
__global__ void __launch_bounds__(WL_SCAN_THREADS + 32)
wl_scan_pipe_kernel(const __grid_constant__ wl_config c, const __grid_constant__ CUtensorMap tmap, const float4* __restrict__ st,
                    float* __restrict__ obs) {
    __shared__ __align__(128) float tile[WL_SCAN_STAGES][WL_TILE_W * WL_TILE_H];
    __shared__ __align__(8) uint64_t full[WL_SCAN_STAGES], empty[WL_SCAN_STAGES];
    __shared__ ScanPose sp[WL_SCAN_STAGES];                  // the scan constants of the env in the stage
    const int n = c.num_envs;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < WL_SCAN_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], WL_SCAN_THREADS / 32);
        }
        mbar_init_fence();
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == WL_SCAN_THREADS / 32) {
        // ---------------- producer ----------------
        if (lane != 0) return;
        int k = 0;
        for (int i = blockIdx.x; i < n; i += gridDim.x, ++k) {
            const int s = k % WL_SCAN_STAGES;
            const uint32_t ph = (uint32_t)(k / WL_SCAN_STAGES) & 1u;
            mbar_wait_parity(&empty[s], ph ^ 1u);                        // stage free (passes at once on its first use)
            const ScanPose p = scan_pose(c, st, n, i);
            sp[s] = p;
            mbar_expect(&full[s], WL_TILE_W * WL_TILE_H * 4);
            tma_load_2d(tile[s], &tmap, p.ox, p.oy, &full[s]);
        }
        return;
    }
    // ---------------- consumers (warps 0..3) ----------------
    int k = 0;
    for (int i = blockIdx.x; i < n; i += gridDim.x, ++k) {
        const int s = k % WL_SCAN_STAGES;
        const uint32_t ph = (uint32_t)(k / WL_SCAN_STAGES) & 1u;
        mbar_wait_parity(&full[s], ph);
        const ScanPose q = sp[s];
        scan_rays(c, tile[s], q, obs + (size_t)WL_OBS_DIM_ELEV * i + 13, threadIdx.x);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);                           // this warp is done with the stage
    }
}

// The ray-caster of a handle with row terms (DESIGN 6r): the whole 689-float row from the state.  Columns 0..12 are the raw
// proprioceptive terms (elev_proprio without its clips), columns 13..688 the raw world_height_map of the 676 rays, each
// through its term's noise, clip and scale.  The draws do not depend on the height-field: every thread forms one or two
// Philox blocks (4 columns each) into shared memory while the tile is in flight, and thread 32 forms the proprioceptive
// values meanwhile.  Same launch shape, tile staging and ray arithmetic as wl_scan_kernel.
// CRITIC (wl_critic_observe on a row critic, DESIGN 6s): the same row through the critic's clips and scales, with no draw
// formed (the critic's stages have no noise), in rows of Dc floats, followed by the extra critic-library columns `ex`; thread 32,
// which loads the state groups, forms their library floats too.
template <bool USE_TMA, bool CRITIC>
__device__ __forceinline__ void scan_row_body(const wl_config& c, const CUtensorMap& tmap, const RowTable& rt, const float4* __restrict__ st,
                                              const float* __restrict__ hf, const wl_globals* __restrict__ gl, uint32_t t_arg,
                                              int32_t call_idx, float* __restrict__ obs, const CriticTable* ex, int Dc) {
    __shared__ __align__(128) float tile[WL_TILE_W * WL_TILE_H];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ ScanPose sp;
    __shared__ __align__(16) float dz[CRITIC ? 4 : 4 * WL_ROW_BLOCKS];  // the noise draw of every column (float4 stores; only when some column is noisy; CRITIC: unused)
    __shared__ float raw[WL_ROW_PROPRIO];    // the raw proprioceptive columns
    __shared__ float lib[CRITIC ? WL_CRITIC_LIB_FLOATS : 1];            // CRITIC: the critic library floats of the extra columns
    const int i = blockIdx.x, n = c.num_envs, tid = threadIdx.x;
    if (tid == 0) {
        const ScanPose p = scan_pose(c, st, n, i);
        sp = p;
        if (USE_TMA) {
            mbar_init(&mbar, 1);
            mbar_init_fence();
            mbar_expect(&mbar, WL_TILE_W * WL_TILE_H * 4);
            tma_load_2d(tile, &tmap, p.ox, p.oy, &mbar);
        }
    } else if (tid == 32) {
        const float4 p = ldg4(st, WL_G_POS, n, i), q = ldg4(st, WL_G_QUAT, n, i), v = ldg4(st, WL_G_LINVEL, n, i),
                     w = ldg4(st, WL_G_ANGVEL, n, i), a = ldg4(st, WL_G_ACTION, n, i), cb = ldg4(st, WL_G_CMDB, n, i);
        const M3 R = rotmat(q.x, q.y, q.z, q.w);
        const V3 vb = rotT(R, V3{v.x, v.y, v.z}), wb = rotT(R, V3{w.x, w.y, w.z}), eu = euler_xyz(q.x, q.y, q.z, q.w);
        const float gx = cb.x - p.x, gy = cb.y - p.y;
        raw[0] = (gx != gx) ? 0.0f : gx; raw[1] = (gy != gy) ? 0.0f : gy;            // nan_to_num(nan=0)
        raw[2] = eu.x; raw[3] = eu.y; raw[4] = eu.z;
        raw[5] = vb.x; raw[6] = vb.y; raw[7] = vb.z; raw[8] = wb.x; raw[9] = wb.y; raw[10] = wb.z;
        raw[11] = a.x; raw[12] = a.y;
        if constexpr (CRITIC) {                                // wl_critic_observe_kernel's library floats (critic_first order)
            const uint32_t G = ex->groups;
            lib[0] = p.x; lib[1] = p.y; lib[2] = p.z;
            lib[3] = eu.x; lib[4] = eu.y; lib[5] = eu.z;
            lib[6] = vb.x; lib[7] = vb.y; lib[8] = vb.z; lib[9] = wb.x; lib[10] = wb.y; lib[11] = wb.z;
            lib[12] = a.x; lib[13] = a.y;
            float4 g;
            if (G & (1u << WL_G_WHEEL)) { g = ldg4(st, WL_G_WHEEL, n, i); lib[14] = g.x; lib[15] = g.y; lib[16] = g.z; lib[17] = g.w; }
            if (G & (1u << WL_G_STEER)) { g = ldg4(st, WL_G_STEER, n, i); lib[18] = g.x; lib[19] = g.y; }
            if (G & (1u << WL_G_PMU_D)) { g = ldg4(st, WL_G_PMU_D, n, i); lib[20] = g.x; lib[21] = g.y; lib[22] = g.z; lib[23] = g.w; }
            if (G & (1u << WL_G_PMASS)) { g = ldg4(st, WL_G_PMASS, n, i); lib[24] = g.x; }
            if (G & (1u << WL_G_PKD)) { g = ldg4(st, WL_G_PKD, n, i); lib[25] = g.x; lib[26] = g.y; lib[27] = g.z; lib[28] = g.w; }
        }
    }
    if (!CRITIC && rt.noisy) {               // in the TMA's shadow
        const uint32_t t = decode_step(gl, t_arg), gid = (uint32_t)(c.env_id_offset + i);
        for (int b = tid; b < WL_ROW_BLOCKS; b += WL_SCAN_THREADS) {
            float d[4];
            if (4 * b >= WL_ROW_PROPRIO) {   // map columns only (the last block's padding draws are not read)
                if (rt.map.noise != WL_NOISE_NONE) row_draws(row_block(c.seed, gid, t, call_idx, rt.map.noise, (uint32_t)b), rt.map.noise, d);
                else d[0] = d[1] = d[2] = d[3] = 0.0f;
            } else {
                int k[4];
#pragma unroll
                for (int w = 0; w < 4; ++w) k[w] = 4 * b + w < WL_ROW_PROPRIO ? rt.col[4 * b + w].noise : rt.map.noise;
                row_mixed_draws(c.seed, gid, t, call_idx, (uint32_t)b, k, d);
            }
            *reinterpret_cast<float4*>(dz + 4 * b) = make_float4(d[0], d[1], d[2], d[3]);
        }
    }
    __syncthreads();                         // constants, mbarrier, draws and raw columns visible to everyone
    const ScanPose q = sp;
    float* row = obs + (size_t)(CRITIC ? Dc : WL_OBS_DIM_ELEV) * i;
    if constexpr (CRITIC) {                  // (wl_set_row_critic refuses noise: every stage is clip and scale)
        if (tid < WL_ROW_PROPRIO) row[tid] = row_stage(rt.col[tid], raw[tid], 0.0f);
        if (tid < ex->n_cols) {
            const float x = lib[ex->src[tid]], cl = ex->clip[tid];
            row[WL_OBS_DIM_ELEV + tid] = cl > 0.0f ? r_clamp(x, -cl, cl) : x;
        }
    } else {
        if (tid < WL_ROW_PROPRIO) row[tid] = row_stage(rt.col[tid], raw[tid], rt.col[tid].noise != WL_NOISE_NONE ? dz[tid] : 0.0f);
    }
    if (USE_TMA) {
        mbar_wait_parity(&mbar, 0);
    } else {
        for (int k = tid; k < WL_TILE_W * WL_TILE_H; k += WL_SCAN_THREADS) {
            int tx = k % WL_TILE_W, ty = k / WL_TILE_W, gx = q.ox + tx, gy = q.oy + ty;
            tile[k] = (gx >= 0 && gy >= 0 && gx < c.hf_nx && gy < c.hf_ny) ? __ldg(hf + (size_t)gy * c.hf_pitch + gx) : 0.0f;
        }
        __syncthreads();
    }
    scan_rays<true>(c, tile, q, row + WL_ROW_PROPRIO, tid, &rt.map, CRITIC ? nullptr : dz + WL_ROW_PROPRIO);
}
template <bool USE_TMA>
__global__ void __launch_bounds__(WL_SCAN_THREADS, 8)
wl_scan_row_kernel(const __grid_constant__ wl_config c, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ RowTable rt,
                   const float4* __restrict__ st, const float* __restrict__ hf, const wl_globals* __restrict__ gl, uint32_t t_arg,
                   int32_t call_idx, float* __restrict__ obs) {
    scan_row_body<USE_TMA, false>(c, tmap, rt, st, hf, gl, t_arg, call_idx, obs, nullptr, 0);
}
// the critic row [N, Dc] of a row critic (rt: the critic's stages, ex: its extra columns)
template <bool USE_TMA>
__global__ void __launch_bounds__(WL_SCAN_THREADS, 8)
wl_scan_critic_row_kernel(const __grid_constant__ wl_config c, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ RowTable rt,
                          const __grid_constant__ CriticTable ex, const float4* __restrict__ st, const float* __restrict__ hf, int Dc,
                          float* __restrict__ obs) {
    scan_row_body<USE_TMA, true>(c, tmap, rt, st, hf, nullptr, 0u, 0, obs, &ex, Dc);
}

#include "wl_reset_dr.cuh"

__global__ void wl_startup_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st) {
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t gid = (uint32_t)(c.env_id_offset + i);
    uint4 r0 = philox4x32(c.seed, gid, 0u, RNG_STARTUP, 0u);
    uint4 r1 = philox4x32(c.seed, gid, 0u, RNG_STARTUP, 1u);
    uint4 r2 = philox4x32(c.seed, gid, 0u, RNG_STARTUP, 2u);
    uint4 r3 = philox4x32(c.seed, gid, 0u, RNG_STARTUP, 3u);
    DrParams p;
    dr_params(c, r0, r1, r2, r3, p);
    stg4(st, WL_G_PIW, n, i, make_float4(p.inv_Iw[0], p.inv_Iw[1], p.inv_Iw[2], p.inv_Iw[3]));
    stg4(st, WL_G_PMASS, n, i, make_float4(p.mass, p.inv_mass, 0.0f, 0.0f));
    stg4(st, WL_G_PMU_D, n, i, make_float4(p.D[0], p.D[1], p.D[2], p.D[3]));
    stg4(st, WL_G_PMU_C, n, i, make_float4(p.C[0], p.C[1], p.C[2], p.C[3]));
    stg4(st, WL_G_PKD, n, i, make_float4(p.kd[0], p.kd[1], p.kd[2], p.kd[3]));
    float t_hf = uniform(r2.y, c.push_hf_interval[0], c.push_hf_interval[1]);
    float t_lf = uniform(r2.z, c.push_lf_interval[0], c.push_lf_interval[1]);
    float4 g;
    g = ldg4(st, WL_G_LINVEL, n, i); g.w = t_hf; stg4(st, WL_G_LINVEL, n, i, g);
    g = ldg4(st, WL_G_ANGVEL, n, i); g.w = t_lf; stg4(st, WL_G_ANGVEL, n, i, g);
    stg4(st, WL_G_QUAT, n, i, make_float4(1.0f, 0.0f, 0.0f, 0.0f));
}

__global__ void wl_reset_kernel(const __grid_constant__ wl_config c, float4* __restrict__ st, const float* __restrict__ aux,
                                const int64_t* __restrict__ ids, int n_ids, uint32_t t) {
    const int n = c.num_envs;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_ids) return;
    const int i = ids ? (int)ids[k] : k;
    if (i < 0 || i >= n) return;
    EnvState e;
    const bool elev = c.task == WL_TASK_ELEVATION;
    load_env(st, n, i, e, elev);
    reset_env(c, c.task, visual_map(c, aux), e, (uint32_t)(c.env_id_offset + i), t);      // (elevation: the command b-frame vector is NOT refreshed by reset())
    store_env(st, n, i, e, elev);
}

__global__ void wl_observe_kernel(const __grid_constant__ wl_config c, const float4* __restrict__ st, float* __restrict__ obs,
                                  uint32_t t, uint32_t call_idx) {
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    EnvState e;
    if (c.task == WL_TASK_VISUAL) {
        load_env(st, n, i, e, false);
        float o[8]; visual_proprio(c, e, o);
        const int camf = vis_cam_floats(c);
        float* row = obs + (size_t)(WL_OBS_DIM_VISUAL + camf) * i + camf;
#pragma unroll
        for (int k = 0; k < 8; ++k) row[k] = o[k];
        return;
    }
    if (c.task == WL_TASK_ELEVATION) {
        load_env(st, n, i, e, true);
        float o[13]; elev_proprio(c, e, euler_xyz(e.qw, e.qx, e.qy, e.qz), o);
        float* row = obs + (size_t)WL_OBS_DIM_ELEV * i;
#pragma unroll
        for (int k = 0; k < 13; ++k) row[k] = o[k];
        return;
    }
    load_env(st, n, i, e, false);
    blind_obs(c, e, (uint32_t)(c.env_id_offset + i), t, RNG_OBS_EXTRA, 3u * call_idx, obs + (size_t)WL_OBS_DIM_BLIND * i);
}

// suspension joint pos / vel are not part of the stored state (DESIGN.md 2): derive them for the articulation view.
// pos = clamp(compression, +-travel) of the wheel's contact spring, vel = compression rate, wheel order [bl,br,fl,fr].
template <int TASK>
__global__ void wl_suspension_kernel(const __grid_constant__ wl_config c, const float4* __restrict__ st, Terrain T,
                                     float4* __restrict__ pos_o, float4* __restrict__ vel_o) {
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    EnvState e;
    load_env(st, n, i, e, false);
    M3 R = rotmat(e.qw, e.qx, e.qy, e.qz);
    V3 cw = rot(R, V3{c.com[0], c.com[1], c.com[2]});
    V3 pc{e.p.x + cw.x, e.p.y + cw.y, e.p.z + cw.z};
    V3 vb = rotT(R, e.v), wb = rotT(R, e.w);
    float sp[4], sv[4];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        V3 rho{((w >= 2) ? c.hub_x_front : c.hub_x_rear) - c.com[0], ((w & 1) ? -c.hub_y : c.hub_y) - c.com[1], c.hub_z - c.com[2]};
        V3 hubw = rot(R, rho);
        hubw.x += pc.x; hubw.y += pc.y; hubw.z += pc.z;
        float zt = 0.0f; V3 nw{0.0f, 0.0f, 1.0f};
        if (TASK == WL_TASK_ELEVATION) heightfield_at(c, T, hubw.x, hubw.y, zt, nw);
        float comp = fm(-(hubw.z - zt), nw.z, c.wheel_radius);
        V3 nb = rotT(R, nw);
        V3 rc = axpy(rho, -c.wheel_radius, nb);
        V3 vc = cross(wb, rc);
        vc.x += vb.x; vc.y += vb.y; vc.z += vb.z;
        sp[w] = r_clamp(comp, -c.susp_travel, c.susp_travel);
        sv[w] = (comp > 0.0f) ? -dot(nb, vc) : 0.0f;
    }
    pos_o[i] = make_float4(sp[0], sp[1], sp[2], sp[3]);
    vel_o[i] = make_float4(sv[0], sv[1], sv[2], sv[3]);
}

struct CurrArgs { int32_t n; int32_t slots[WL_MAX_REW_TERMS]; float inc[WL_MAX_REW_TERMS]; uint32_t fire_mask; uint32_t wslot, row; };
__global__ void wl_curriculum_kernel(wl_globals* __restrict__ gl, CurrArgs a) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (!(gl->acc[a.row][8] > 0.0f)) return;                 // the reference's call site is _reset_idx: only if >= 1 env reset
    for (int t = 0; t < a.n; ++t)
        if ((a.fire_mask >> t) & 1u) gl->rew_weight[a.wslot][a.slots[t]] += a.inc[t];
}
// publish the log row of step t_next - 1 without stepping, then drop its pointer: the caller may free or reuse the row's
// buffer once this has run, so the next step's janitor must not write the row through it again (it still re-publishes
// last_log, with the same values)
__global__ void wl_flush_kernel(const __grid_constant__ wl_config c, wl_globals* __restrict__ gl, uint32_t t_next) {
    if (t_next == 0u) return;
    const uint32_t row = (t_next + 2u) % 3u;
    publish_log_row(c, gl, row, threadIdx.x & 31);
    __syncwarp();                                                      // every lane has read log_ptr[row]
    if (threadIdx.x == 0) gl->log_ptr[row] = nullptr;
}
// counter jump: carry the weights over to the slot the next step reads, clear the accumulators and the pending log
__global__ void wl_rearm_kernel(wl_globals* __restrict__ gl, uint32_t from_slot, uint32_t to_slot) {
    const int lane = threadIdx.x;
    if (lane < WL_MAX_REW_TERMS && from_slot != to_slot) gl->rew_weight[to_slot][lane] = gl->rew_weight[from_slot][lane];
    if (lane < 16) { gl->acc[0][lane] = 0.0f; gl->acc[1][lane] = 0.0f; gl->acc[2][lane] = 0.0f; }
    if (lane < 3) gl->log_ptr[lane] = nullptr;
}
// host-counter path, after a step whose successor counter t_next is a curriculum boundary: apply the terms in place to the
// slot step t_next will read (so the host sees them at once) and mark the boundary as done
__global__ void wl_boundary_kernel(const __grid_constant__ wl_config c, wl_globals* __restrict__ gl, uint32_t t_next) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    float wts[WL_MAX_REW_TERMS];
    load_weights(c, gl, t_next, wts);
    for (int q = 0; q < WL_MAX_REW_TERMS; ++q) gl->rew_weight[(t_next + 1u) & 1u][q] = wts[q];
    gl->curr_applied_t = t_next;
}
__global__ void wl_advance_kernel(wl_globals* __restrict__ gl, uint32_t k) { if (threadIdx.x == 0 && blockIdx.x == 0) gl->step_base += k; }

__global__ void wl_synth_actions_kernel(const __grid_constant__ wl_config c, const wl_globals* __restrict__ gl,
                                        float2* __restrict__ action, uint32_t t_arg, int dist) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.num_envs) return;
    const uint32_t t = decode_step(gl, t_arg);
    uint4 r = philox4x32(c.seed, (uint32_t)(c.env_id_offset + i), t, RNG_ACTION, 0u);
    float a0, a1;
    if (dist == 0) { a0 = 2.0f * u01(r.x) - 1.0f; a1 = 2.0f * u01(r.y) - 1.0f; }
    else { float z0, z1; box_muller(r.x, r.y, z0, z1); a0 = r_clamp(z0, -1.0f, 1.0f); a1 = r_clamp(z1, -1.0f, 1.0f); }
    action[i] = make_float2(a0, a1);
}

// GAE(lambda) over the rollout slab: one thread per env, t = T-1 .. 0; loads are issued WL_GAE_CHUNK steps ahead so the
// reverse scan is bandwidth- rather than latency-bound (17 B read + 8 B written per (t, env)).
#define WL_GAE_CHUNK 8
__global__ void __launch_bounds__(128)
wl_gae_kernel(const float* __restrict__ rew, const float* __restrict__ val, const float* __restrict__ last_val,
              const uint8_t* __restrict__ done, const uint8_t* __restrict__ tout, float gamma, float lam,
              float* __restrict__ ret, float* __restrict__ adv, int T, int N) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float next_v = last_val[i], a = 0.0f;
    for (int t1 = T; t1 > 0; t1 -= WL_GAE_CHUNK) {
        const int t0 = (t1 - WL_GAE_CHUNK > 0) ? t1 - WL_GAE_CHUNK : 0;
        float r[WL_GAE_CHUNK], v[WL_GAE_CHUNK]; uint8_t d[WL_GAE_CHUNK], to[WL_GAE_CHUNK];
#pragma unroll
        for (int k = 0; k < WL_GAE_CHUNK; ++k) {
            const int t = t1 - 1 - k;
            if (t >= t0) {
                const size_t o = (size_t)t * N + i;
                r[k] = rew[o]; v[k] = val[o]; d[k] = done[o]; to[k] = tout ? tout[o] : (uint8_t)0;
            }
        }
#pragma unroll
        for (int k = 0; k < WL_GAE_CHUNK; ++k) {
            const int t = t1 - 1 - k;
            if (t >= t0) {
                const float nt = d[k] ? 0.0f : 1.0f;
                const float rr = to[k] ? r[k] + gamma * v[k] : r[k];           // time-out bootstrap
                const float delta = rr + nt * gamma * next_v - v[k];
                a = delta + nt * gamma * lam * a;
                const size_t o = (size_t)t * N + i;
                ret[o] = a + v[k]; adv[o] = a;
                next_v = v[k];
            }
        }
    }
}

// GAE for SMALL N (the reference's 128 x 4096 rollout): the backward recurrence a_t = delta_t + k_t a_{t+1} is affine, so
// the T steps of an env are cut into segments of WL_GAE_SEG steps, one thread per (env, segment): every thread loads its
// whole segment at once (one exposed memory latency instead of T / WL_GAE_CHUNK), reduces it to (c, p) with
// a_start = c + p * a_in, the S segments of an env are chained through shared memory (S - 1 dependent FMAs), and the
// outputs are formed from registers.  CTA = 32 envs x S segments (warp = segment: every load / store is coalesced over envs).
// Rounding differs from the sequential scan by a few ulp (two-level association).
#define WL_GAE_SEG 16
__global__ void __launch_bounds__(512)
wl_gae_seg_kernel(const float* __restrict__ rew, const float* __restrict__ val, const float* __restrict__ last_val,
                  const uint8_t* __restrict__ done, const uint8_t* __restrict__ tout, float gamma, float lam,
                  float* __restrict__ ret, float* __restrict__ adv, int T, int N) {
    __shared__ float s_c[16][33], s_p[16][33], s_in[16][33];
    const int lane = threadIdx.x & 31, seg = threadIdx.x >> 5, S = blockDim.x >> 5;
    const int i = blockIdx.x * 32 + lane;
    const bool live = i < N;
    const int ii = live ? i : N - 1;
    const int t0 = seg * WL_GAE_SEG;                       // this thread owns steps [t0, t0 + WL_GAE_SEG) intersected with [0, T)
    float r[WL_GAE_SEG], v[WL_GAE_SEG], kk[WL_GAE_SEG];
    uint8_t d[WL_GAE_SEG], to[WL_GAE_SEG];
#pragma unroll
    for (int k = 0; k < WL_GAE_SEG; ++k) {
        const int t = t0 + k;
        if (t < T) {
            const size_t o = (size_t)t * N + ii;
            r[k] = rew[o]; v[k] = val[o]; d[k] = done[o]; to[k] = tout ? tout[o] : (uint8_t)0;
        } else { r[k] = 0.0f; v[k] = 0.0f; d[k] = 1; to[k] = 0; }
    }
    const int t_end = min(t0 + WL_GAE_SEG, T);             // value that follows the segment: V(t_end) or the bootstrap value
    float next_v = (t_end < T) ? val[(size_t)t_end * N + ii] : last_val[ii];
    // backward over the segment: c = contribution with a_in = 0, p = product of the k_t
    float c = 0.0f, p = 1.0f;
#pragma unroll
    for (int k = WL_GAE_SEG - 1; k >= 0; --k) {
        if (t0 + k < T) {
            const float nt = d[k] ? 0.0f : 1.0f;
            const float rr = to[k] ? r[k] + gamma * v[k] : r[k];           // time-out bootstrap
            const float delta = rr + nt * gamma * next_v - v[k];
            const float kt = nt * gamma * lam;
            c = delta + kt * c; p = kt * p;
            r[k] = c; kk[k] = p;                                           // a_t = r[k] + kk[k] * a_in
            next_v = v[k];
        }
    }
    s_c[seg][lane] = c; s_p[seg][lane] = p;
    __syncthreads();
    if (seg == 0) {                                        // chain the env's segments: a_in of segment s = a at the start of segment s + 1
        float a_in = 0.0f;
        for (int q = S - 1; q >= 0; --q) { s_in[q][lane] = a_in; a_in = s_c[q][lane] + s_p[q][lane] * a_in; }
    }
    __syncthreads();
    const float a_in = s_in[seg][lane];
    if (live) {
#pragma unroll
        for (int k = 0; k < WL_GAE_SEG; ++k) {
            const int t = t0 + k;
            if (t < T) {
                const float a = r[k] + kk[k] * a_in;
                const size_t o = (size_t)t * N + i;
                ret[o] = a + v[k]; adv[o] = a;
            }
        }
    }
}

// Data-parallel learner step for the small rsl_rl networks (SURVEY 8f-2): gradient all-reduce FUSED with the Adam update in
// one kernel over peer memory.  Every rank keeps its flat gradient in a symmetric (P2P-mapped) buffer; each thread reads
// element i of every rank's gradient (NVLink loads, fixed rank order -> every rank forms the identical mean), and applies
// Adam to its own replica of the parameters.  10.5 K parameters = 42 KB per rank: one launch instead of NCCL all-reduce +
// optimizer kernels.  The caller brackets the launch with barriers (gradients complete / safe to overwrite).
struct GradPeers { int32_t n; int32_t pad; const float* g[WL_MAX_PEERS]; };
// torch.optim.Adam's update of one parameter (bias corrections bc = 1 - beta^t, complements cb = 1 - beta); shared by every
// optimiser kernel
__device__ __forceinline__ void adam_update(float* param, float* m, float* v, int i, float g, float lr, float beta1, float cb1,
                                            float beta2, float cb2, float eps, float bc1, float bc2) {
    const float p = param[i];
    const float mi = fmaf(beta1, m[i], cb1 * g);
    const float vi = fmaf(beta2, v[i], cb2 * g * g);
    m[i] = mi; v[i] = vi;
    param[i] = p - lr * (mi / bc1) / (sqrtf(vi / bc2) + eps);
}
__global__ void wl_dp_adam_kernel(float* __restrict__ param, float* __restrict__ m, float* __restrict__ v, const __grid_constant__ GradPeers gp,
                                  float lr, float beta1, float cb1, float beta2, float cb2, float eps, float weight_decay, float bc1,
                                  float bc2, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float g = 0.0f;
    for (int r = 0; r < gp.n; ++r) g += __ldcg(gp.g[r] + i);           // (L2-coherent loads: peers have just written)
    g = g / (float)gp.n;
    if (weight_decay != 0.0f) g = fmaf(weight_decay, param[i], g);
    adam_update(param, m, v, i, g, lr, beta1, cb1, beta2, cb2, eps, bc1, bc2);
}

#include "wl_ppo.cuh"
#include "wl_wide.cuh"
#include "wl_actor.cuh"
#include "wl_episode.cuh"
#include "wl_terms.cuh"
#include "wl_dev_events.cuh"
#include "wl_distill.cuh"

// the handle's device terms: the kernel's table and one device allocation holding the per-env state
struct DevTerms {
    TermTable tt;
    TermBufs b;
    uint8_t* tbits;     // [N] stage a's built-in termination bits when the handle records none (wl_set_term_bits)
    void* block;
};
static void free_event_timers(wl_sim* sim) {
    if (sim->events.time_left) cudaFree(sim->events.time_left);
    sim->events = EventTable{};
}
static void free_device_terms(wl_sim* sim) {
    if (!sim->dterms) return;
    cudaFree(sim->dterms->block);
    delete sim->dterms;
    sim->dterms = nullptr;
}
// the handle's device event terms: the kernel's table (its timers point into `block`) and stage a's term bits
struct DevEvents {
    DevEventTable et;
    uint8_t* tbits;     // [N] stage a's built-in termination bits when the handle records none (wl_set_term_bits)
    void* block;
};
static void free_device_events(wl_sim* sim) {
    if (!sim->devents) return;
    cudaFree(sim->devents->block);
    delete sim->devents;
    sim->devents = nullptr;
}
// a call that steps the handle without its device event terms refuses it, before any device work
static int refuse_devents(const wl_sim* sim, const char* fn) {
    if (!sim->devents) return WL_OK;
    return fail(WL_EUNSUPPORTED, std::string(fn) + ": the handle has device event terms, which wl_step_terms applies (wl_set_device_events(0) first)");
}
// a call that hands its next call the built-in policy row refuses a handle with a policy table, before any device work
static int refuse_pobs(const wl_sim* sim, const char* fn) {
    if (sim->pobs.n_cols == 0) return WL_OK;
    return fail(WL_EUNSUPPORTED, std::string(fn) + ": the handle has a policy observation table, whose row wl_policy_observe forms "
                                 "(wl_set_policy_terms(0) first)");
}
// a call that writes the built-in Elevation / Visual row in its own kernel refuses a handle with row terms, before any device work
static int refuse_rows(const wl_sim* sim, const char* fn) {
    if (sim->rows.n_terms == 0) return WL_OK;
    return fail(WL_EUNSUPPORTED, std::string(fn) + ": the handle has row terms, which wl_step writes (wl_set_row_terms(0) first)");
}
// the width of the row the policy kernels read: the policy table's when the handle has one, else the built-in row's
static int policy_in_dim(const wl_sim* sim) { return sim->pobs.n_cols ? sim->pobs.n_cols : sim->obs_dim; }

__global__ void wl_detmath_kernel(int op, const float* __restrict__ in, const float* __restrict__ in2, float* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = in[i], s, c2, r = 0.0f;
    switch (op) {
        case 0: det_sincos(x, s, c2); r = s; break;
        case 1: det_sincos(x, s, c2); r = c2; break;
        case 2: r = det_atan(x); break;
        case 3: r = det_atan2(in2[i], x); break;
        case 4: r = det_log(x); break;
        case 5: r = det_tan(x); break;
        case 6: r = det_asin(x); break;
        case 7: r = det_exp(x); break;
        case 8: r = det_tanh(x); break;
        case 9: r = fdiv_norm(in2[i], x); break;          // in2 / in
        case 10: r = fsqrt_norm(x); break;
        case 11: r = det_atan_ratio<true>(in2[i], x); break;
        case 12: r = det_atan_ratio<false>(in2[i], x); break;
    }
    out[i] = r;
}
__global__ void wl_null_kernel(int* p) { if (p != nullptr && threadIdx.x == 1024) *p = 0; }
__global__ void wl_null_cfg_kernel(const __grid_constant__ wl_config c, int* p) { if (p != nullptr && threadIdx.x == 1024) *p = c.num_envs; }
__global__ void wl_philox_kernel(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint4* __restrict__ out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    out[i] = philox4x32(seed, c0 + (uint32_t)i, c1, c2, c3);
}

// ---------------------------------------------------------------------------------------
// Visual task camera term (mdp_sensors/observations.py:64-87 on a software pinhole camera): one CTA per env renders the
// kept rows of the 80 x 60 frame against the 2-colour plane mesh, applies ColorJitter on the two class values, the 5 x 5
// Gaussian blur (separable, reflect padding) through shared memory, Grayscale + Normalize(0.5, 0.5), and streams the
// 3200 floats out as float4.  HBM: 12.8 KB written per env, the 250 KB map stays in L2.
// ---------------------------------------------------------------------------------------
#define WL_CAM_THREADS 128
#define WL_CAM_MAX_W 128
#define WL_CAM_MAX_ROWS 64
__global__ void __launch_bounds__(WL_CAM_THREADS)
wl_camera_kernel(const __grid_constant__ wl_config c, const float4* __restrict__ st, const wl_globals* __restrict__ gl,
                 const float* __restrict__ aux, float* __restrict__ obs, uint32_t t_arg, uint32_t stream, uint32_t sub,
                 const float* __restrict__ aug) {
    // Thread (u4, rg) owns 4 consecutive columns 4*u4 .. 4*u4+3 of rows rg, rg + RG, ...: row terms are shared by 4 pixels
    // and every shared-memory access is a vector one.  Jp: white mask (bytes) with 4 pad columns on either side
    // (only the inner 2 are used: reflected border); Hp: horizontal pass, with 2 reflected rows above and below.
    __shared__ __align__(16) uint8_t Jp[WL_CAM_MAX_PIXELS + 8 * WL_CAM_MAX_ROWS];     // the mask is kept as bytes: 9 CTAs per SM
    __shared__ CamAug A_s;
    __shared__ __align__(16) float Hp[WL_CAM_MAX_PIXELS + 4 * WL_CAM_MAX_W];
    __shared__ __align__(16) float CX[WL_CAM_MAX_W], CY[WL_CAM_MAX_W], CZ[WL_CAM_MAX_W];   // per-column part of the ray direction
    __shared__ float yo_s[WL_CAM_MAX_ROWS];
    __shared__ int n_white;
    const int i = blockIdx.x, n = c.num_envs, tid = threadIdx.x;
    const int W = c.vis_cam_w, rows = c.vis_cam_h - c.vis_cam_row0, npix = W * rows, WP = W + 8, W4 = W >> 2;
    const int RG = WL_CAM_THREADS / W4;                      // row groups (threads >= RG * W4 idle in the 2-D phases)
    const int rg = tid / W4, u4 = tid - rg * W4;
    const bool act = rg < RG;
    const uint32_t t = decode_step(gl, t_arg);
    const VisualMap vm = visual_map(c, aux);
    const float4 gp = ldg4(st, WL_G_POS, n, i), gq = ldg4(st, WL_G_QUAT, n, i);
    const M3 R = rotmat(gq.x, gq.y, gq.z, gq.w);
    const V3 off = rot(R, V3{c.vis_cam_pos[0], c.vis_cam_pos[1], c.vis_cam_pos[2]});
    const V3 pc{gp.x + off.x, gp.y + off.y, gp.z + off.z};
    if (tid == 0) n_white = 0;
    // pixel-centre coordinates of the optical frame (x right, y down, z forward) and the column part of R (1, -xo, -yo)
    if (tid < W) {
        const float xo = ((float)tid + 0.5f - c.vis_cam_cx) / c.vis_cam_fx;
        CX[tid] = fm(-R.r[1], xo, R.r[0]); CY[tid] = fm(-R.r[4], xo, R.r[3]); CZ[tid] = fm(-R.r[7], xo, R.r[6]);
    }
    if (tid < rows) yo_s[tid] = ((float)(c.vis_cam_row0 + tid) + 0.5f - c.vis_cam_cy) / c.vis_cam_fy;
    const bool bg = c.vis_cam_bg >= 0.5f, above = pc.z > 0.0f;
    const float cmax = (float)(c.vis_cols - 1), rmax = (float)(c.vis_rows - 1);
    __syncthreads();
    // ---- render: ray through the pixel centre -> plane z = 0 -> face of the coloured mesh (utils/__init__.py:8-89)
    int mine = 0;
    if (act) {
        const float4 cx = reinterpret_cast<const float4*>(CX)[u4], cy = reinterpret_cast<const float4*>(CY)[u4], cz = reinterpret_cast<const float4*>(CZ)[u4];
        const float cxs[4] = {cx.x, cx.y, cx.z, cx.w}, cys[4] = {cy.x, cy.y, cy.z, cy.w}, czs[4] = {cz.x, cz.y, cz.z, cz.w};
        for (int r = rg; r < rows; r += RG) {
            const float yo = yo_s[r];
            uint8_t wv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float dz = fm(-R.r[8], yo, czs[j]);
                bool wh = bg;
                if (dz < 0.0f && above) {
                    const float tt = pc.z / (-dz);                                  // depth along the optical axis
                    if (!(tt > 100.0f)) {                                           // clipping_range = (0.01, 1e2)
                        const float hx = fm(tt, fm(-R.r[2], yo, cxs[j]), pc.x), hy = fm(tt, fm(-R.r[5], yo, cys[j]), pc.y);
                        const float fx = floorf((hx - c.vis_mesh_x0) * c.d_vis_mesh_inv_dx), fy = floorf((hy - c.vis_mesh_y0) * c.d_vis_mesh_inv_dy);
                        wh = (fx >= 0.0f) && (fy >= 0.0f) && (fx < cmax) && (fy < rmax) && (__ldg(vm.map + (size_t)(int)fy * c.vis_cols + (int)fx) != 0);
                    }
                }
                wv[j] = wh ? 1 : 0;
                mine += wh ? 1 : 0;
            }
            *reinterpret_cast<uchar4*>(Jp + r * WP + 4 + 4 * u4) = make_uchar4(wv[0], wv[1], wv[2], wv[3]);
        }
    }
    mine = (int)warp_sum((float)mine);           // <= 32 * 64: exact in fp32
    if ((tid & 31) == 0 && mine) atomicAdd(&n_white, mine);
    __syncthreads();
    if (tid == WL_CAM_THREADS - 1)                // one thread draws the frame's ColorJitter / blur parameters for the CTA
        A_s = cam_aug_params(c, t, stream, sub, aug, (float)n_white / (float)npix);
    float4* row4 = reinterpret_cast<float4*>(obs + (size_t)(WL_OBS_DIM_VISUAL + npix) * i);
    if (c.vis_cam != 2) {                        // camera_data_rgb_flattened: grayscale + normalize only
        const float g0 = fm(2.0f, cam_gray(0.0f), -1.0f), g1 = fm(2.0f, cam_gray(1.0f), -1.0f);
        if (act)
            for (int r = rg; r < rows; r += RG) {
                const uchar4 m = *reinterpret_cast<const uchar4*>(Jp + r * WP + 4 + 4 * u4);
                row4[r * W4 + u4] = make_float4(m.x ? g1 : g0, m.y ? g1 : g0, m.z ? g1 : g0, m.w ? g1 : g0);
            }
        return;
    }
    // reflected border columns: -1 -> 1, -2 -> 2, W -> W-2, W+1 -> W-3
    if (tid < rows) {
        uint8_t* jr = Jp + tid * WP + 4;
        jr[-1] = jr[1]; jr[-2] = jr[2]; jr[W] = jr[W - 2]; jr[W + 1] = jr[W - 3];
    }
    __syncthreads();
    const CamAug A = A_s;
    // ---- horizontal 5-tap pass on the mask; padded row rp holds source row reflect(rp - 2)
    if (act)
        for (int rp = rg; rp < rows + 4; rp += RG) {
            int r = rp - 2;
            r = r < 0 ? -r : (r >= rows ? 2 * rows - 2 - r : r);
            const uchar4* j4 = reinterpret_cast<const uchar4*>(Jp + r * WP) + u4;
            const uchar4 Lb = j4[0], Mb = j4[1], Qb = j4[2];
            const float4 L = make_float4(0.0f, 0.0f, (float)Lb.z, (float)Lb.w), M = make_float4((float)Mb.x, (float)Mb.y, (float)Mb.z, (float)Mb.w);
            const float4 Q = make_float4((float)Qb.x, (float)Qb.y, 0.0f, 0.0f);
            float4 o;
            o.x = fm(A.w2, L.z + M.z, fm(A.w1, L.w + M.y, A.w0 * M.x));
            o.y = fm(A.w2, L.w + M.w, fm(A.w1, M.x + M.z, A.w0 * M.y));
            o.z = fm(A.w2, M.x + Q.x, fm(A.w1, M.y + M.w, A.w0 * M.z));
            o.w = fm(A.w2, M.y + Q.y, fm(A.w1, M.z + Q.x, A.w0 * M.w));
            reinterpret_cast<float4*>(Hp + rp * W)[u4] = o;
        }
    __syncthreads();
    // ---- vertical pass, then the ColorJitter class values (blur is affine in the mask: J = v0 + (v1 - v0) w),
    // Grayscale and Normalize((x - 0.5) / 0.5); one STG.128 per thread and row
    if (act) {
        const float dv = A.v1 - A.v0;
        for (int r = rg; r < rows; r += RG) {
            const float4* h = reinterpret_cast<const float4*>(Hp + r * W) + u4;      // padded rows r .. r+4 = source rows r-2 .. r+2
            const float4 a = h[0], b = h[W4], m = h[2 * W4], d = h[3 * W4], e = h[4 * W4];
            float4 o;
            o.x = fm(2.0f, cam_gray(fm(dv, fm(A.w2, a.x + e.x, fm(A.w1, b.x + d.x, A.w0 * m.x)), A.v0)), -1.0f);
            o.y = fm(2.0f, cam_gray(fm(dv, fm(A.w2, a.y + e.y, fm(A.w1, b.y + d.y, A.w0 * m.y)), A.v0)), -1.0f);
            o.z = fm(2.0f, cam_gray(fm(dv, fm(A.w2, a.z + e.z, fm(A.w1, b.z + d.z, A.w0 * m.z)), A.v0)), -1.0f);
            o.w = fm(2.0f, cam_gray(fm(dv, fm(A.w2, a.w + e.w, fm(A.w1, b.w + d.w, A.w0 * m.w)), A.v0)), -1.0f);
            row4[r * W4 + u4] = o;
        }
    }
}

// ---------------------------------------------------------------------------------------
// launch geometry: spread small N over all SMs, use fatter CTAs once the chip is full
// ---------------------------------------------------------------------------------------
// launch with (or without) the programmatic-dependent-launch attribute
// (A kernel launched with it must wait (griddepcontrol.wait) before its first read of anything a previous launch may have
// written.  The single-GPU duo kernel is always launched with it (DESIGN.md 6e); the fan-out forms of the duo kernel share
// its code but are launched without it; the thread, quad and act-step kernels use it only with WL_PDL=1.)
static bool g_pdl = (getenv("WL_PDL") != nullptr) && (atoi(getenv("WL_PDL")) != 0);

// What may still run on a stream, for the single-GPU duo step (DESIGN.md 6e).  A kernel that triggers its dependents
// (griddepcontrol.launch_dependents) releases a PDL-launched successor early, whether it was itself launched with the
// attribute or not; all of them (the step, quad, act-step and duo kernels) are launched through launch_k, which clears the
// record, and the FAN = 0 duo launch then records itself.  Any other kernel lets its successor start only once it has
// completed, and does so only after its own predecessor has, so it leaves nothing running that the record would have to
// describe.  The record holds:
// * the in-flight suffix: the footprints (buffers read or written) of the duo steps since, and including, the most recent
//   one that triggered only after its wait (unchained or shallow).  Such a step's trigger follows the completion of every
//   launch before it, and a deep step triggers at entry, so only the steps of the suffix can run beside the next launch;
// * the env sets (state buffers) of the last WL_DEEP_DISTINCT duo steps;
// * the id of the graph capture it was made in (0: none): launches captured into a graph never ran on the stream, and the
//   first node of a graph starts only once the work before the graph launch has completed.
// Deep chains need the H = WL_DEEP_DISTINCT most recent steps and this one to be of distinct env sets, so that a set that
// recurs within H steps keeps the two-grid protocol (a deep step lengthens the suffix, and a set that recurs inside the
// suffix must wait at entry); the suffix stays shorter than C = WL_DEEP_CAP, which bounds the host's disjointness check.
#ifndef WL_DEEP_DISTINCT
#define WL_DEEP_DISTINCT 4
#endif
#ifndef WL_DEEP_CAP
#define WL_DEEP_CAP 32
#endif
struct Span { uintptr_t lo, hi; };
struct DuoFootprint { Span w[6]; int n_spans; Span act; };
struct DuoPrev {
    unsigned long long capture = 0;
    std::vector<DuoFootprint> suffix;
    uintptr_t recent[WL_DEEP_DISTINCT] = {};       // state buffers of the last duo steps, most recent at [0]; 0: none
};
// (stream handle, device, host thread for cudaStreamPerThread: each host thread's per-thread stream is a stream of its own)
using StreamKey = std::tuple<uintptr_t, int, size_t>;
struct DuoKey { StreamKey stream; unsigned long long capture; };
static std::mutex g_duo_mu;
static std::map<StreamKey, DuoPrev> g_duo_prev;       // one entry per stream ever used (a destroyed stream's entry stays)
static DuoKey duo_key(cudaStream_t cs) {
    int dev = 0;
    cudaGetDevice(&dev);                       // (stream 0 names a different stream on each device)
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    unsigned long long id = 0;
    if (cudaStreamGetCaptureInfo(cs, &st, &id) != cudaSuccess || st != cudaStreamCaptureStatusActive) id = 0;
    const size_t thr = (cs == cudaStreamPerThread) ? std::hash<std::thread::id>{}(std::this_thread::get_id()) : 0;
    return DuoKey{StreamKey{reinterpret_cast<uintptr_t>(cs), dev, thr}, id};
}
static bool spans_meet(Span a, Span b) { return a.lo < b.hi && b.lo < a.hi; }
// true when the footprints are disjoint, reads of the actions by both excepted
static bool footprints_apart(const DuoFootprint& a, const DuoFootprint& b) {
    for (int i = 0; i < a.n_spans; ++i) {
        if (spans_meet(a.w[i], b.act)) return false;
        for (int k = 0; k < b.n_spans; ++k) if (spans_meet(a.w[i], b.w[k])) return false;
    }
    for (int k = 0; k < b.n_spans; ++k) if (spans_meet(b.w[k], a.act)) return false;
    return true;
}
// how a duo step with footprint `fp` runs (wl_step_duo_kernel's `chained`), and the record after it.  Chained: the stream's
// record, in the same capture or outside any, has a suffix and this step touches none of the buffers of any step in it,
// the actions they read excepted; otherwise unchained, and the suffix restarts with this step.  Deep: chained, the last
// WL_DEEP_DISTINCT duo steps and this one are of distinct env sets, and the suffix with this step is shorter than
// WL_DEEP_CAP; otherwise a chained step is shallow and the suffix restarts with it.
static int duo_chain_mode(const DuoKey& key, const DuoFootprint& fp, DuoPrev& next) {
    {
        std::lock_guard<std::mutex> lk(g_duo_mu);
        auto it = g_duo_prev.find(key.stream);
        if (it != g_duo_prev.end() && it->second.capture == key.capture) next = it->second;
    }
    next.capture = key.capture;
    bool apart = !next.suffix.empty();
    for (const DuoFootprint& f : next.suffix) apart = apart && footprints_apart(f, fp);
    const uintptr_t set = fp.w[0].lo;
    bool distinct = true;
    for (int i = 0; i < WL_DEEP_DISTINCT; ++i) {
        if (next.recent[i] == 0) break;
        for (int k = 0; k < i; ++k) distinct = distinct && next.recent[k] != next.recent[i];
        distinct = distinct && next.recent[i] != set;
    }
    const int mode = !apart ? WL_CHAIN_NONE : (distinct && (int)next.suffix.size() + 1 < WL_DEEP_CAP) ? WL_CHAIN_DEEP : WL_CHAIN_SHALLOW;
    if (mode != WL_CHAIN_DEEP) next.suffix.clear();
    next.suffix.push_back(fp);
    for (int i = WL_DEEP_DISTINCT - 1; i > 0; --i) next.recent[i] = next.recent[i - 1];
    next.recent[0] = set;
    return mode;
}
static void set_duo_prev(const DuoKey& key, DuoPrev rec) {
    std::lock_guard<std::mutex> lk(g_duo_mu);
    g_duo_prev[key.stream] = std::move(rec);
}

template <typename... KArgs, typename... Args>
static void launch_k(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t cs, bool pdl, const Args&... args) {
    set_duo_prev(duo_key(cs), DuoPrev{});
    static_assert(sizeof...(KArgs) == sizeof...(Args), "argument count");
    cudaLaunchConfig_t lc;
    memset(&lc, 0, sizeof lc);
    lc.gridDim = dim3((unsigned)grid); lc.blockDim = dim3((unsigned)block); lc.dynamicSmemBytes = smem; lc.stream = cs;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = attr; lc.numAttrs = pdl ? 1 : 0;
    // parameters by address: the 1.5 KB wl_config is read in place by the runtime, not copied through a by-value call chain.
    // (each argument must already have exactly the kernel's parameter type: checked below)
    static_assert((std::is_same<typename std::decay<KArgs>::type, typename std::decay<Args>::type>::value && ...), "argument types must match the kernel's");
    void* ptrs[] = {const_cast<void*>(static_cast<const void*>(&args))...};
    cudaLaunchKernelExC(&lc, reinterpret_cast<const void*>(kernel), ptrs);
}

static inline int pick_block(int n) {
    if (n >= WL_NUM_SMS * 128 * 4) return 128;
    if (n >= WL_NUM_SMS * 64 * 2) return 64;
    return 32;
}

// block size of a duo-kernel launch of `grid` CTAs: with the spacer warp when every CTA is resident at once with it, else 64.
// (A deep-chained launch has CTAs of its own, WL_DEEP_THREADS: it shares the SMs with the grids before it, so CTA slots
// count more than a scheduler per env warp, DESIGN.md 6e.)
template <typename KF>
static int duo_block(wl_sim* sim, KF kernel, int grid) {
    const void* kp = reinterpret_cast<const void*>(kernel);
    if (sim->duo_kernel != kp) {
        int per_sm = 0, sms = 0;
        const bool ok = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, WL_DUO_THREADS, 0) == cudaSuccess &&
                        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, sim->device) == cudaSuccess;
        sim->duo_threads = (ok && grid <= per_sm * sms) ? WL_DUO_THREADS : 64;
        sim->duo_kernel = kp;
    }
    return sim->duo_threads;
}

// t: the step counter (host value or WL_DEVICE_COUNTER_PLUS(k)); call_idx: -1 after a step, wl_observe's otherwise.  Both
// key the row terms' noise only.
static int launch_scan(wl_sim* sim, float* d_obs, uint32_t t, int32_t call_idx, cudaStream_t cs) {
    const int n = sim->cfg.num_envs;
    if (sim->rows.n_terms) {                                 // row terms: the whole row (scan mode 2 is refused with them)
        if (sim->scan_mode >= 1 && sim->has_tmap)
            wl_scan_row_kernel<true><<<n, WL_SCAN_THREADS, 0, cs>>>(sim->cfg, sim->tmap, sim->rows, sim->state, sim->hf, sim->globals, t, call_idx, d_obs);
        else
            wl_scan_row_kernel<false><<<n, WL_SCAN_THREADS, 0, cs>>>(sim->cfg, sim->tmap, sim->rows, sim->state, sim->hf, sim->globals, t, call_idx, d_obs);
        return launched(sim, "wl_scan_row_kernel");
    }
    if (sim->scan_mode == 2 && sim->has_tmap) {              // TMA producer/consumer pipeline, persistent CTAs
        static const int per_sm = [] { const char* e = getenv("WL_SCAN_CTAS_PER_SM"); int v = e ? atoi(e) : 6; return v < 1 ? 1 : (v > 12 ? 12 : v); }();
        const int grid = n < WL_NUM_SMS * per_sm ? n : WL_NUM_SMS * per_sm;    // (WL_SCAN_CTAS_PER_SM: tuning experiments only)
        wl_scan_pipe_kernel<<<grid, WL_SCAN_THREADS + 32, 0, cs>>>(sim->cfg, sim->tmap, sim->state, d_obs);
    } else if (sim->scan_mode >= 1 && sim->has_tmap)
        wl_scan_kernel<true><<<n, WL_SCAN_THREADS, 0, cs>>>(sim->cfg, sim->tmap, sim->state, sim->hf, d_obs);
    else
        wl_scan_kernel<false><<<n, WL_SCAN_THREADS, 0, cs>>>(sim->cfg, sim->tmap, sim->state, sim->hf, d_obs);
    return launched(sim, "wl_scan_kernel");
}
// the Visual tail through the row terms, after every launch that writes the Visual row (nothing without row terms)
static int launch_visual_row(wl_sim* sim, float* d_obs, uint32_t t, int32_t call_idx, cudaStream_t cs) {
    if (!sim->rows.n_terms) return WL_OK;
    const int n = sim->cfg.num_envs;
    wl_visual_row_kernel<<<(n + WL_ROW_VIS_BS - 1) / WL_ROW_VIS_BS, WL_ROW_VIS_BS, 0, cs>>>(
        sim->rows, sim->state, sim->globals, n, vis_cam_floats(sim->cfg), sim->cfg.seed, sim->cfg.env_id_offset, t, call_idx, d_obs);
    return launched(sim, "wl_visual_row_kernel");
}

// ---------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------
static int launch_camera(wl_sim* sim, float* d_obs, uint32_t t, uint32_t stream_id, uint32_t sub, const float* d_aug, cudaStream_t cs) {
    wl_camera_kernel<<<sim->cfg.num_envs, WL_CAM_THREADS, 0, cs>>>(sim->cfg, sim->state, sim->globals, sim->hf, d_obs, t, stream_id, sub, d_aug);
    return launched(sim, "wl_camera_kernel");
}
// The row tail: the kernels that finish the Elevation and Visual built-in rows, after every launch that writes one (nothing on
// the Drift family).  After a step (call_idx -1) the camera draws from RNG_CAM, sub 0; in wl_observe's tail it draws from
// RNG_CAM_EXTRA, sub call_idx, which without row terms may be any value, -1 included: hence the flag.
static int launch_row_tail(wl_sim* sim, float* d_obs, uint32_t t, bool after_step, int32_t call_idx, cudaStream_t cs) {
    if (sim->cfg.task == WL_TASK_ELEVATION) return launch_scan(sim, d_obs, t, call_idx, cs);
    if (sim->cfg.task != WL_TASK_VISUAL) return WL_OK;
    if (sim->cfg.vis_cam)        // t may be device-relative
        if (int rc = launch_camera(sim, d_obs, t, after_step ? RNG_CAM : RNG_CAM_EXTRA, after_step ? 0u : (uint32_t)call_idx, nullptr, cs))
            return rc;
    return launch_visual_row(sim, d_obs, t, call_idx, cs);
}

extern "C" {

const char* wl_last_error(void) { return g_err.c_str(); }
const char* wl_build_info(void) { return "wheeledlab_b200 abi=2 arch=sm_90a fmad=false"; }
size_t wl_config_sizeof(void) { return sizeof(wl_config); }

const char* wl_config_describe(void) {
    static std::string s;
    if (s.empty()) {
        char buf[256];
#define WL_XS(type, tag, name)                                                                  \
    snprintf(buf, sizeof buf, "%s:%s:1:%zu;", #name, #tag, offsetof(wl_config, name)); s += buf;
#define WL_XA(type, tag, name, n)                                                               \
    snprintf(buf, sizeof buf, "%s:%s:%d:%zu;", #name, #tag, (int)(n), offsetof(wl_config, name)); s += buf;
        WL_CONFIG_FIELDS(WL_XS, WL_XA)
#undef WL_XS
#undef WL_XA
        snprintf(buf, sizeof buf, "sizeof:%zu", sizeof(wl_config)); s += buf;
    }
    return s.c_str();
}

int wl_set_step_counter(wl_sim* sim, int64_t value, void* stream) {
    if (!sim) return fail(WL_EINVAL, "wl_set_step_counter: null handle");
    ensure_device(sim);
    const uint32_t v = (uint32_t)value;
    sim->base_host = value;
    return cuda_check(cudaMemcpyAsync(&sim->globals->step_base, &v, sizeof v, cudaMemcpyHostToDevice, (cudaStream_t)stream),
                      "wl_set_step_counter");
}
int wl_advance_counter(wl_sim* sim, int32_t K, void* stream) {
    if (!sim || K < 0) return fail(WL_EINVAL, "wl_advance_counter: bad argument");
    ensure_device(sim);
    wl_advance_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(sim->globals, (uint32_t)K);
    sim->base_host += K;
    return launched(sim, "wl_advance_kernel");
}
int wl_note_device_counter(wl_sim* sim, int64_t value) {
    if (!sim) return fail(WL_EINVAL, "wl_note_device_counter: null handle");
    sim->base_host = value;
    sim->last_t = value - 1;          // the replayed graph ended on step value - 1
    return WL_OK;
}
int wl_log_flush(wl_sim* sim, void* stream) {
    if (!sim) return fail(WL_EINVAL, "wl_log_flush: null handle");
    ensure_device(sim);
    if (sim->last_t < 0) return WL_OK;
    wl_flush_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(sim->cfg, sim->globals, (uint32_t)(sim->last_t + 1));
    return launched(sim, "wl_flush_kernel");
}
float* wl_reward_weights(wl_sim* sim) { return sim ? sim->globals->rew_weight[(uint32_t)sim->last_t & 1u] : nullptr; }

int wl_set_term_bits(wl_sim* sim, uint8_t* d_term_bits) {
    if (!sim) return fail(WL_EINVAL, "wl_set_term_bits: null handle");
    sim->term_bits = d_term_bits;
    return WL_OK;
}
// The packed rows leave as 16-byte stores at pointer + delta, so every delta must keep that alignment.  The multicast delta
// is only a shortcut for the rows that qualify: the others go peer by peer, so it needs the peer deltas set first, and
// switching the peers off switches it off too.
int wl_set_peer_fanout(wl_sim* sim, int32_t n_peers, const int64_t* byte_deltas) {
    if (!sim || n_peers < 0 || n_peers > WL_MAX_PEERS || (n_peers > 0 && !byte_deltas)) return fail(WL_EINVAL, "wl_set_peer_fanout: bad argument");
    if (n_peers > 0 && sim->cfg.task != WL_TASK_DRIFT) return fail(WL_EUNSUPPORTED, "wl_set_peer_fanout: Drift-family tasks only");
    for (int k = 0; k < n_peers; ++k)
        if (byte_deltas[k] % 16 != 0) return fail(WL_EINVAL, "wl_set_peer_fanout: every byte delta must be a multiple of 16");
    const int32_t mc = sim->fan.mc; const long long mcd = sim->fan.mc_delta;
    memset(&sim->fan, 0, sizeof sim->fan);
    if (n_peers > 0) { sim->fan.mc = mc; sim->fan.mc_delta = mcd; }
    sim->fan.n = n_peers;
    for (int k = 0; k < n_peers; ++k) sim->fan.delta[k] = (long long)byte_deltas[k];
    return WL_OK;
}
int wl_set_multicast_fanout(wl_sim* sim, int64_t mc_byte_delta) {
    if (!sim) return fail(WL_EINVAL, "wl_set_multicast_fanout: null handle");
    if (mc_byte_delta != 0 && sim->cfg.task != WL_TASK_DRIFT) return fail(WL_EUNSUPPORTED, "wl_set_multicast_fanout: Drift-family tasks only");
    if (mc_byte_delta != 0 && sim->fan.n == 0) return fail(WL_EINVAL, "wl_set_multicast_fanout: set the peer deltas first (wl_set_peer_fanout)");
    if (mc_byte_delta % 16 != 0) return fail(WL_EINVAL, "wl_set_multicast_fanout: the byte delta must be a multiple of 16");
    sim->fan.mc = mc_byte_delta != 0 ? 1 : 0;
    sim->fan.mc_delta = (long long)mc_byte_delta;
    return WL_OK;
}
int wl_set_seed(wl_sim* sim, uint64_t seed) {
    if (!sim) return fail(WL_EINVAL, "wl_set_seed: null handle");
    sim->cfg.seed = seed;
    return WL_OK;
}

int wl_config_finalize(wl_config* c) {
    if (!c) return fail(WL_EINVAL, "wl_config_finalize: null");
    if (c->substeps <= 0 || !(c->sim_dt > 0.0f)) return fail(WL_EINVAL, "wl_config_finalize: bad sim timing");
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
    return WL_OK;
}

size_t wl_globals_offset(int32_t num_envs) { return align256(groups_bytes(num_envs)); }
size_t wl_state_bytes(int32_t num_envs) { return wl_globals_offset(num_envs) + align256(sizeof(wl_globals)); }

int wl_create(const wl_config* cfg, void* d_state, size_t state_bytes, const float* d_heightfield, wl_sim** out) {
    if (!cfg || !d_state || !out) return fail(WL_EINVAL, "wl_create: null argument");
    if (cfg->abi_version != WL_ABI_VERSION) return fail(WL_EINVAL, "wl_create: abi_version mismatch");
    if (cfg->num_envs <= 0) return fail(WL_EINVAL, "wl_create: num_envs must be > 0");
    if (state_bytes < wl_state_bytes(cfg->num_envs)) return fail(WL_EINVAL, "wl_create: state buffer too small");
    if (((uintptr_t)d_state & 255u) != 0) return fail(WL_EINVAL, "wl_create: state buffer must be 256-byte aligned");
    if (cfg->task != WL_TASK_DRIFT && cfg->task != WL_TASK_ELEVATION && cfg->task != WL_TASK_VISUAL)
        return fail(WL_EUNSUPPORTED, "wl_create: unknown task");
    if (cfg->task == WL_TASK_VISUAL) {
        if (!d_heightfield) return fail(WL_EINVAL, "wl_create: the visual task needs the traversability data (see header)");
        if (cfg->vis_rows < 1 || cfg->vis_cols < 1 || cfg->vis_n_trav < 1) return fail(WL_EINVAL, "wl_create: bad traversability map geometry");
        if (((uintptr_t)d_heightfield & 15u) != 0) return fail(WL_EINVAL, "wl_create: traversability data must be 16-byte aligned");
        if (cfg->vis_cam) {
            const int rows = cfg->vis_cam_h - cfg->vis_cam_row0;
            if (cfg->vis_cam < 0 || cfg->vis_cam > 2 || cfg->vis_cam_w < 4 || (cfg->vis_cam_w & 3) || rows < 3 || cfg->vis_cam_row0 < 0 ||
                cfg->vis_cam_w * rows > WL_CAM_MAX_PIXELS || cfg->vis_cam_w > 128 || rows > 64 || !(cfg->vis_cam_fx > 0.0f) || !(cfg->vis_cam_fy > 0.0f) ||
                !(cfg->vis_mesh_dx > 0.0f) || !(cfg->vis_mesh_dy > 0.0f) || (cfg->vis_cam == 2 && !(cfg->vis_aug_sigma[0] > 0.0f)))
                return fail(WL_EINVAL, "wl_create: bad camera geometry (width % 4 == 0 and <= 128, 3..64 kept rows, <= WL_CAM_MAX_PIXELS pixels)");
        }
    }
    if (cfg->task == WL_TASK_ELEVATION) {
        if (!d_heightfield) return fail(WL_EINVAL, "wl_create: the elevation task needs a height-field");
        if (cfg->hf_nx < 2 || cfg->hf_ny < 2 || cfg->hf_pitch < cfg->hf_nx || (cfg->hf_pitch & 3) || !(cfg->hf_cell > 0.0f))
            return fail(WL_EINVAL, "wl_create: bad height-field geometry (hf_pitch must be >= hf_nx and a multiple of 4)");
        if (((uintptr_t)d_heightfield & 15u) != 0) return fail(WL_EINVAL, "wl_create: height-field must be 16-byte aligned");
        // The height scan reads every ray's 2x2 cell out of a WL_TILE_W x WL_TILE_H window staged in shared memory, and clamps
        // the cell into the window, so a cell outside it is a wrong height, not a fault.  scan_pose starts the window
        // reach = scan_half*sqrt2 + hf_cell below the base (rounded down to a sample; in x down again to a multiple of 4).  The
        // 26 x 26 rays within +-scan_half span up to D = 2*scan_half*sqrt2 / hf_cell cells along an axis (yaw 45 deg), so they
        // touch floor(D) + 2 cells: with the reach's cell and the +1 bilinear neighbour, floor(D) + 4 rows and floor(D) + 7
        // columns.  The 1/64-cell margin absorbs the float32 rounding of the kernel's index arithmetic.  0.1 m at the
        // task's 1.25 m half-width needs 39 of the 40 rows; the smallest cell accepted there is about 0.0956 m.
        if ((WL_SCAN_SIDE - 1) * (double)cfg->scan_res > 2.0 * (double)cfg->scan_half * (1.0 + 1e-6))
            return fail(WL_EINVAL, "wl_create: the height-scan grid must lie within +-scan_half (25 * scan_res <= 2 * scan_half)");
        const int span = (int)floor(2.0 * (double)cfg->scan_half * 1.41421356237 / (double)cfg->hf_cell + 1.0 / 64.0);
        if (span + 4 > WL_TILE_H || span + 7 > WL_TILE_W)
            return fail(WL_EINVAL, "wl_create: hf_cell too small for scan_half: the height scan needs floor(2*scan_half*sqrt2/hf_cell) + 4 <= " +
                                   std::to_string(WL_TILE_H) + " window rows (hf_cell > about scan_half / 13.08: 0.0956 m at scan_half 1.25 m)");
    }
    if (cfg->bounding != WL_BOUND_CLIP && cfg->bounding != WL_BOUND_NONE && cfg->bounding != WL_BOUND_TANH)
        return fail(WL_EUNSUPPORTED, "wl_create: unknown bounding strategy");
    if (cfg->action_kind != WL_ACT_ACKERMANN && cfg->action_kind != WL_ACT_RWD && cfg->action_kind != WL_ACT_4WD)
        return fail(WL_EUNSUPPORTED, "wl_create: unknown action term kind");
    if (cfg->dr_wheel_mass_enable && !(cfg->dr_wheel_mass[0] > 0.0f && cfg->wheel_mass_nominal > 0.0f))
        return fail(WL_EINVAL, "wl_create: wheel-mass DR needs positive masses");
    if (cfg->decimation <= 0 || cfg->substeps <= 0 || !(cfg->sim_dt > 0.0f)) return fail(WL_EINVAL, "wl_create: bad sim timing");
    if (cfg->num_rew_terms < 0 || cfg->num_rew_terms > WL_MAX_REW_TERMS) return fail(WL_EINVAL, "wl_create: num_rew_terms");
    if (cfg->curr_n < 0 || cfg->curr_n > 4) return fail(WL_EINVAL, "wl_create: curr_n must be in [0,4]");
    for (int k = 0; k < cfg->curr_n; ++k)
        if (cfg->curr_every[k] < 1 || cfg->curr_slot[k] < 0 || cfg->curr_slot[k] >= WL_MAX_REW_TERMS)
            return fail(WL_EINVAL, "wl_create: bad curriculum term");
    if (cfg->num_ref_poses <= 0 || cfg->num_ref_poses > WL_MAX_REF_POSES) return fail(WL_EINVAL, "wl_create: num_ref_poses");
    if (cfg->dr_num_buckets < 1 || cfg->dr_num_buckets > WL_MAX_BUCKETS) return fail(WL_EINVAL, "wl_create: dr_num_buckets");
    int dev_count = 0;
    if (int rc = cuda_check(cudaGetDeviceCount(&dev_count), "cudaGetDeviceCount")) return rc;
    if (dev_count == 0) return fail(WL_ECUDA, "wl_create: no CUDA device (this library has no CPU path)");
    wl_sim* s = new (std::nothrow) wl_sim();
    if (!s) return fail(WL_EINVAL, "wl_create: out of host memory");
    s->cfg = *cfg;
    if (int rc = wl_config_finalize(&s->cfg)) { delete s; return rc; }
    s->state = reinterpret_cast<float4*>(d_state);
    s->globals = reinterpret_cast<wl_globals*>(reinterpret_cast<char*>(d_state) + wl_globals_offset(cfg->num_envs));
    s->hf = d_heightfield;
    s->state_bytes = state_bytes;
    s->launches = 0;
    s->chained_steps = 0;
    s->deep_steps = 0;
    s->last_t = -1;
    s->base_host = 0;
    s->term_bits = nullptr;
    memset(&s->fan, 0, sizeof s->fan);
    s->hp_n = 0;
    cudaGetDevice(&s->device);
    s->variant = 0;
    s->has_tmap = false;
    s->scan_mode = 1;
    s->spec = spec_key(step_spec(s->cfg));
    s->duo_kernel = nullptr;
    s->duo_threads = 64;
    s->step_variant = s->step_specialised = s->step_threads = 0;
    s->reset_ev = 0;
    if (cfg->task == WL_TASK_ELEVATION) {
        typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (int rc = cuda_check(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres),
                                "cudaGetDriverEntryPoint(cuTensorMapEncodeTiled)")) { delete s; return rc; }
        if (!fn || qres != cudaDriverEntryPointSuccess) { delete s; return fail(WL_ECUDA, "cuTensorMapEncodeTiled not available"); }
        cuuint64_t gdim[2] = {(cuuint64_t)cfg->hf_nx, (cuuint64_t)cfg->hf_ny};
        cuuint64_t gstride[1] = {(cuuint64_t)cfg->hf_pitch * sizeof(float)};
        cuuint32_t box[2] = {WL_TILE_W, WL_TILE_H}, estr[2] = {1, 1};
        CUresult cr = ((encode_fn)fn)(&s->tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)d_heightfield, gdim, gstride, box, estr,
                                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr != CUDA_SUCCESS) { delete s; return fail(WL_ECUDA, "cuTensorMapEncodeTiled failed (code " + std::to_string((int)cr) + ")"); }
        s->has_tmap = true;
    }
    s->obs_dim = obs_row_floats(*cfg, cfg->task);
    // live reward weights
    for (int slot = 0; slot < 2; ++slot)
        if (int rc = cuda_check(cudaMemcpy(s->globals->rew_weight[slot], cfg->rew_weight, sizeof(float) * WL_MAX_REW_TERMS,
                                           cudaMemcpyHostToDevice), "upload reward weights")) { delete s; return rc; }
    {
        const uint32_t none = 0xFFFFFFFFu;
        if (int rc = cuda_check(cudaMemcpy(&s->globals->curr_applied_t, &none, sizeof none, cudaMemcpyHostToDevice), "init globals")) { delete s; return rc; }
    }
    *out = s;
    return WL_OK;
}

int wl_destroy(wl_sim* sim) { if (sim) { free_device_terms(sim); free_event_timers(sim); free_device_events(sim); } delete sim; return WL_OK; }
int32_t wl_obs_dim(const wl_sim* sim) { return sim ? sim->obs_dim : 0; }
int wl_set_scan_tma(wl_sim* sim, int32_t use_tma) {
    if (!sim) return fail(WL_EINVAL, "wl_set_scan_tma: null handle");
    if (use_tma < 0 || use_tma > 2) return fail(WL_EINVAL, "wl_set_scan_tma: 0, 1 or 2");
    if (use_tma == 2 && sim->rows.n_terms) return fail(WL_EUNSUPPORTED, "wl_set_scan_tma: the pipelined ray-caster (2) has no row-terms variant");
    sim->scan_mode = use_tma;
    return WL_OK;
}
int wl_set_kernel_variant(wl_sim* sim, int32_t lanes_per_env) {
    if (!sim) return fail(WL_EINVAL, "wl_set_kernel_variant: null handle");
    if (lanes_per_env != 0 && lanes_per_env != 1 && lanes_per_env != 4 && lanes_per_env != 8)
        return fail(WL_EINVAL, "wl_set_kernel_variant: 0, 1, 4 or 8");
    sim->variant = lanes_per_env;
    return WL_OK;
}
int64_t wl_launch_count(const wl_sim* sim) { return sim ? sim->launches : 0; }
int64_t wl_chained_step_count(const wl_sim* sim) { return sim ? sim->chained_steps : 0; }
int64_t wl_deep_step_count(const wl_sim* sim) { return sim ? sim->deep_steps : 0; }
int wl_step_launch_info(const wl_sim* sim, int32_t* variant, uint32_t* spec_key, int32_t* specialised, int32_t* threads_per_cta) {
    if (!sim) return fail(WL_EINVAL, "wl_step_launch_info: null handle");
    if (variant) *variant = sim->step_variant;
    if (spec_key) *spec_key = sim->spec;
    if (specialised) *specialised = sim->step_specialised;
    if (threads_per_cta) *threads_per_cta = sim->step_threads;
    return WL_OK;
}

}   // extern "C"
// Steps are issued with consecutive counters (the janitor protocol, see wl_globals).  Resolve this launch's counter on the host
// mirror; on a jump publish the pending log row, carry the weights to the slot the step will read and clear the rows.
static int prep_step(wl_sim* sim, int64_t step_counter, int32_t n_steps, cudaStream_t cs) {
    ensure_device(sim);
    const int64_t t = step_counter >= 0 ? step_counter : sim->base_host + (-1 - step_counter);
    if (t >= ((int64_t)1 << 31) - n_steps) return fail(WL_EINVAL, "step counter out of range (< 2^31)");
    if (t != sim->last_t + 1) {
        if (sim->last_t >= 0) wl_flush_kernel<<<1, 32, 0, cs>>>(sim->cfg, sim->globals, (uint32_t)(sim->last_t + 1));
        wl_rearm_kernel<<<1, 32, 0, cs>>>(sim->globals, (uint32_t)sim->last_t & 1u, (uint32_t)(t - 1) & 1u);
        if (int rc = launched(sim, "wl_rearm_kernel", 2)) return rc;
    }
    sim->last_t = t + n_steps - 1;
    return WL_OK;
}
// The peer / multicast fan-out is carried by wl_step's duo kernel only.  Every other call that writes the rows of a step
// (rollout, act step, staged step, host-transport step) refuses while it is set, before any device work: run without it,
// every peer would keep stale rows with no error.
static bool fan_set(const wl_sim* sim) { return sim->fan.n > 0 || sim->fan.mc; }
static int refuse_fan(const wl_sim* sim, const char* fn) {
    if (!fan_set(sim)) return WL_OK;
    return fail(WL_EUNSUPPORTED, std::string(fn) + ": the peer fan-out is set, and only wl_step carries it (wl_set_peer_fanout(0) first)");
}
// after the step kernel(s): a curriculum boundary reached with a host-supplied counter is applied in place right away
static int post_step(wl_sim* sim, int64_t step_counter, cudaStream_t cs) {
    if (step_counter < 0 || sim->cfg.curr_n <= 0) return WL_OK;
    const int64_t t_next = sim->last_t + 1;
    if (t_next % sim->cfg.max_episode_length != 0) return WL_OK;
    wl_boundary_kernel<<<1, 32, 0, cs>>>(sim->cfg, sim->globals, (uint32_t)t_next);
    return launched(sim, "wl_boundary_kernel");
}
// after a call that reset envs: the reset-mode DR events of the handle (DESIGN 6n).  after_step: the envs the step just
// reset, found by the kernel (n_ids = num_envs, ids = null); otherwise wl_reset's ids.  Mask 0: nothing is launched.
static int reset_dr(wl_sim* sim, const int64_t* ids, int n_ids, int64_t step_counter, bool after_step, cudaStream_t cs) {
    if (!sim->reset_ev) return WL_OK;
    wl_reset_dr_kernel<<<(n_ids + WL_RESET_DR_BS - 1) / WL_RESET_DR_BS, WL_RESET_DR_BS, 0, cs>>>(
        sim->cfg, sim->state, sim->globals, ids, n_ids, (uint32_t)step_counter, after_step, sim->reset_ev);
    return launched(sim, "wl_reset_dr_kernel");
}
// the step epilogue, after the step kernel(s) and the row tail: the reset-mode DR of the envs the step reset, then the
// curriculum boundary
static int end_step(wl_sim* sim, int64_t step_counter, cudaStream_t cs) {
    if (int rc = reset_dr(sim, nullptr, sim->cfg.num_envs, step_counter, true, cs)) return rc;
    return post_step(sim, step_counter, cs);
}
extern "C" {

int wl_startup(wl_sim* sim, void* stream) {
    if (!sim) return fail(WL_EINVAL, "wl_startup: null handle");
    ensure_device(sim);
    const int n = sim->cfg.num_envs, bs = 128;
    wl_startup_kernel<<<(n + bs - 1) / bs, bs, 0, (cudaStream_t)stream>>>(sim->cfg, sim->state);
    return launched(sim, "wl_startup_kernel");
}

int wl_reset(wl_sim* sim, const int64_t* d_env_ids, int32_t n_ids, int64_t step_counter, void* stream) {
    if (!sim) return fail(WL_EINVAL, "wl_reset: null handle");
    ensure_device(sim);
    const int n = d_env_ids ? n_ids : sim->cfg.num_envs;
    if (n <= 0) return WL_OK;
    const int bs = 128;
    wl_reset_kernel<<<(n + bs - 1) / bs, bs, 0, (cudaStream_t)stream>>>(sim->cfg, sim->state, sim->hf, d_env_ids, n, (uint32_t)step_counter);
    if (int rc = launched(sim, "wl_reset_kernel")) return rc;
    return reset_dr(sim, d_env_ids, n, step_counter, false, (cudaStream_t)stream);
}

int wl_step(wl_sim* sim, const float* d_action, float* d_obs, float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated,
            float* d_log, int64_t step_counter, void* stream) {
    if (!sim || !d_action || !d_obs || !d_rew || !d_terminated || !d_truncated) return fail(WL_EINVAL, "wl_step: null argument");
    if (((uintptr_t)d_action & 7u) || ((uintptr_t)d_obs & 7u)) return fail(WL_EINVAL, "wl_step: action/obs must be 8-byte aligned");
    if (int rc = refuse_devents(sim, "wl_step")) return rc;
    const int n = sim->cfg.num_envs;
    Terrain T{sim->hf};
    // 8 = quad + aux warp (Drift family, small N: shortest dependent chain), 4 = quad, 1 = thread per env
    int variant = sim->variant ? sim->variant : ((n <= WL_QUAD_MAX_ENVS) ? ((sim->cfg.task == WL_TASK_DRIFT) ? 8 : 4) : 1);
    if (variant == 8 && sim->cfg.task != WL_TASK_DRIFT) variant = 4;
    if (variant != 8 && fan_set(sim))                         // before prep_step: a refused call leaves the handle as it was
        return fail(WL_EUNSUPPORTED, "wl_step: the peer fan-out is implemented by the Drift-family small-N kernel (variant 8) only");
    const float2* act = reinterpret_cast<const float2*>(d_action);
    cudaStream_t cs = (cudaStream_t)stream;
    const uint32_t t = (uint32_t)step_counter;               // negative (device base + k) stays encoded: see decode_step
    if (int rc = prep_step(sim, step_counter, 1, cs)) return rc;
    StageIO sio0{sim->term_bits, nullptr, nullptr};
    int specialised = 0, cta_threads = 0;
    if (variant == 8) {
        const int grid = (n + WL_DUO_ENVS - 1) / WL_DUO_ENVS + 1;                            // + the janitor CTA
        const bool rows_ok = (n % WL_DUO_ENVS) == 0 && (((uintptr_t)d_obs | (uintptr_t)d_rew) & 15u) == 0 &&
                             (((uintptr_t)d_terminated | (uintptr_t)d_truncated) & 7u) == 0;
        const int unchained = 0;
        if (sim->fan.mc && rows_ok)
            launch_k(wl_step_duo_kernel<2, 0u>, grid, duo_block(sim, wl_step_duo_kernel<2, 0u>, grid), 0, cs, false, sim->cfg, sim->state, sim->globals, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sim->term_bits, sim->fan, unchained);
        else if (fan_set(sim))
            launch_k(wl_step_duo_kernel<1, 0u>, grid, duo_block(sim, wl_step_duo_kernel<1, 0u>, grid), 0, cs, false, sim->cfg, sim->state, sim->globals, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sim->term_bits, sim->fan, unchained);
        else {
            auto span = [](const void* p, size_t bytes) { const uintptr_t a = reinterpret_cast<uintptr_t>(p); return Span{a, a + bytes}; };
            const size_t un = (size_t)n;
            DuoFootprint fp{{span(sim->state, sim->state_bytes), span(d_obs, un * WL_OBS_DIM_BLIND * sizeof(float)), span(d_rew, un * sizeof(float)),
                             span(d_terminated, un), span(d_truncated, un), span(sim->term_bits, sim->term_bits ? un : 0)},
                            6, span(act, un * sizeof(float2))};
            const DuoKey key = duo_key(cs);
            DuoPrev next;
            const int chained = duo_chain_mode(key, fp, next);
            with_spec<SPEC_DRIFT_RWD, SPEC_DRIFT_4WD>(sim->spec, [&](auto k) {
                specialised = k.value != 0u;
                if (chained == WL_CHAIN_DEEP) {
                    cta_threads = WL_DEEP_THREADS;
                    const int deep_grid = (n + WL_DEEP_ENVS - 1) / WL_DEEP_ENVS + 1;                 // + the janitor CTA
                    launch_k(wl_step_duo_deep_kernel<k>, deep_grid, cta_threads, 0, cs, true, sim->cfg, sim->state, sim->globals, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sim->term_bits, sim->fan);
                } else {
                    const int shallow = chained == WL_CHAIN_SHALLOW;
                    cta_threads = duo_block(sim, wl_step_duo_kernel<0, k>, grid);
                    launch_k(wl_step_duo_kernel<0, k>, grid, cta_threads, 0, cs, true, sim->cfg, sim->state, sim->globals, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sim->term_bits, sim->fan, shallow);
                }
            });
            set_duo_prev(key, std::move(next));
            sim->chained_steps += chained != WL_CHAIN_NONE;
            sim->deep_steps += chained == WL_CHAIN_DEEP;
        }
        if (cta_threads == 0) cta_threads = sim->duo_threads;
    } else if (variant == 4) {
#ifndef WL_QUAD_BS
#define WL_QUAD_BS 32
#endif
        const int bs = WL_QUAD_BS, threads = 4 * n, grid = (threads + bs - 1) / bs + 1;      // + the janitor CTA
        with_task<WL_TASK_ELEVATION, WL_TASK_VISUAL>(sim->cfg.task, [&](auto task) {
            launch_k(wl_step_quad_kernel<task>, grid, bs, 0, cs, g_pdl, sim->cfg, sim->state, sim->globals, T, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sim->term_bits);
        });
        cta_threads = bs;
    } else {
        const int bs = pick_block(n), grid = (n + bs - 1) / bs + 1;
        with_task<WL_TASK_ELEVATION, WL_TASK_VISUAL>(sim->cfg.task, [&](auto task) {
            launch_k(wl_step_kernel<task, 0>, grid, bs, 0, cs, g_pdl, sim->cfg, sim->state, sim->globals, T, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sio0);
        });
        cta_threads = bs;
    }
    sim->step_variant = variant; sim->step_specialised = specialised; sim->step_threads = cta_threads;
    if (int rc = launched(sim, "wl_step_kernel")) return rc;
    if (int rc = launch_row_tail(sim, d_obs, t, true, -1, cs)) return rc;
    return end_step(sim, step_counter, cs);
}

#ifdef WL_DUO_TRACE
// phase-trace build only (tools/duo_trace.py): duo-kernel warps append records to `buf` (capacity `cap`) from the next
// launch on; returns the number appended since the last call
int wl_duo_trace_arm(void* buf, uint32_t cap) {
    unsigned int n = 0, zero = 0;
    if (cudaMemcpyFromSymbol(&n, g_duo_trace_n, sizeof n) != cudaSuccess) return -1;
    if (cudaMemcpyToSymbol(g_duo_trace, &buf, sizeof buf) != cudaSuccess || cudaMemcpyToSymbol(g_duo_trace_cap, &cap, sizeof cap) != cudaSuccess ||
        cudaMemcpyToSymbol(g_duo_trace_n, &zero, sizeof zero) != cudaSuccess) return -1;
    return (int)n;
}
#endif

// ---- env.step cut in two (host-side reward / termination terms run in between) ----------------------------------------
}   // extern "C" (templates have C++ linkage)
template <int STAGE>
static int launch_stage(wl_sim* sim, const float2* act, float* d_obs, float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated,
                        float* d_log, uint32_t t, StageIO sio, cudaStream_t cs) {
    const bool jan = STAGE == 2 || STAGE == 3;                                // stage b / b1: + the janitor CTA
    const int n = sim->cfg.num_envs, bs = pick_block(n), grid = (n + bs - 1) / bs + (jan ? 1 : 0);
    Terrain T{sim->hf};
    with_task<WL_TASK_ELEVATION, WL_TASK_VISUAL>(sim->cfg.task, [&](auto task) {
        launch_k(wl_step_kernel<task, STAGE>, grid, bs, 0, cs, false, sim->cfg, sim->state, sim->globals, T, act, d_obs, d_rew, d_terminated, d_truncated, d_log, t, sio);
    });
    static const char* const names[] = {"wl_step_kernel", "wl_step_kernel<stage a>", "wl_step_kernel<stage b>", "wl_step_kernel<stage b1>",
                                        "wl_step_kernel<stage b2>"};
    return launched(sim, names[STAGE]);
}
extern "C" {

int wl_step_stage_a(wl_sim* sim, const float* d_action, float* d_rew, uint8_t* d_term_bits, int64_t step_counter, void* stream) {
    if (!sim || !d_action || !d_rew || !d_term_bits) return fail(WL_EINVAL, "wl_step_stage_a: null argument");
    if ((uintptr_t)d_action & 7u) return fail(WL_EINVAL, "wl_step_stage_a: action must be 8-byte aligned");
    if (step_counter < 0) return fail(WL_EINVAL, "wl_step_stage_a: the staged step takes the host's step counter");
    if (int rc = refuse_fan(sim, "wl_step_stage_a")) return rc;
    if (int rc = refuse_devents(sim, "wl_step_stage_a")) return rc;
    {   // stage a reads W(t) like a full step: re-arm on a counter jump, but the step is only committed by stage b
        const int64_t keep = sim->last_t;
        if (int rc = prep_step(sim, step_counter, 1, (cudaStream_t)stream)) return rc;
        sim->last_t = (keep == step_counter - 1) ? keep : step_counter - 1;
    }
    return launch_stage<1>(sim, reinterpret_cast<const float2*>(d_action), nullptr, d_rew, nullptr, nullptr, nullptr, (uint32_t)step_counter,
                           StageIO{d_term_bits, nullptr, nullptr}, (cudaStream_t)stream);
}

int wl_step_stage_b(wl_sim* sim, const uint8_t* d_term_bits, const uint8_t* d_extra_terminated, const uint8_t* d_extra_truncated,
                    float* d_obs, uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream) {
    if (!sim || !d_term_bits || !d_obs || !d_terminated || !d_truncated) return fail(WL_EINVAL, "wl_step_stage_b: null argument");
    if (step_counter < 0) return fail(WL_EINVAL, "wl_step_stage_b: the staged step takes the host's step counter");
    if (int rc = refuse_fan(sim, "wl_step_stage_b")) return rc;
    if (int rc = prep_step(sim, step_counter, 1, (cudaStream_t)stream)) return rc;
    if (int rc = launch_stage<2>(sim, nullptr, d_obs, nullptr, d_terminated, d_truncated, d_log, (uint32_t)step_counter,
                                 StageIO{const_cast<uint8_t*>(d_term_bits), d_extra_terminated, d_extra_truncated}, (cudaStream_t)stream))
        return rc;
    if (int rc = launch_row_tail(sim, d_obs, (uint32_t)step_counter, true, -1, (cudaStream_t)stream)) return rc;
    return end_step(sim, step_counter, (cudaStream_t)stream);
}

int wl_step_stage_b1(wl_sim* sim, const uint8_t* d_term_bits, const uint8_t* d_extra_terminated, const uint8_t* d_extra_truncated,
                     uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream) {
    if (!sim || !d_term_bits || !d_terminated || !d_truncated) return fail(WL_EINVAL, "wl_step_stage_b1: null argument");
    if (step_counter < 0) return fail(WL_EINVAL, "wl_step_stage_b1: the staged step takes the host's step counter");
    if (int rc = refuse_fan(sim, "wl_step_stage_b1")) return rc;
    if (int rc = prep_step(sim, step_counter, 1, (cudaStream_t)stream)) return rc;
    if (int rc = launch_stage<3>(sim, nullptr, nullptr, nullptr, d_terminated, d_truncated, d_log, (uint32_t)step_counter,
                                 StageIO{const_cast<uint8_t*>(d_term_bits), d_extra_terminated, d_extra_truncated}, (cudaStream_t)stream))
        return rc;
    return end_step(sim, step_counter, (cudaStream_t)stream);
}

int wl_step_stage_b2(wl_sim* sim, float* d_obs, int64_t step_counter, void* stream) {
    if (!sim || !d_obs) return fail(WL_EINVAL, "wl_step_stage_b2: null argument");
    if (step_counter < 0 || step_counter != sim->last_t)
        return fail(WL_EINVAL, "wl_step_stage_b2: step_counter must be that of the wl_step_stage_b1 before it");
    if (int rc = refuse_fan(sim, "wl_step_stage_b2")) return rc;
    ensure_device(sim);
    if (int rc = launch_stage<4>(sim, nullptr, d_obs, nullptr, nullptr, nullptr, nullptr, (uint32_t)step_counter,
                                 StageIO{nullptr, nullptr, nullptr}, (cudaStream_t)stream))
        return rc;
    return launch_row_tail(sim, d_obs, (uint32_t)step_counter, true, -1, (cudaStream_t)stream);
}

int wl_set_event_timers(wl_sim* sim, int32_t n_terms, const float* lo_hi) {
    if (!sim) return fail(WL_EINVAL, "wl_set_event_timers: null handle");
    if (n_terms < 0 || n_terms > WL_MAX_EVENT_TERMS) return fail(WL_EINVAL, "wl_set_event_timers: n_terms must be 0..8");
    if (n_terms > 0 && !lo_hi) return fail(WL_EINVAL, "wl_set_event_timers: null range table");
    if (fan_set(sim)) return fail(WL_EINVAL, "wl_set_event_timers: the peer fan-out is set, and event timers run with the staged step only");
    EventTable et{};
    et.n = n_terms;
    for (int k = 0; k < n_terms; ++k) {
        const float lo = lo_hi[2 * k], hi = lo_hi[2 * k + 1];
        if (!std::isfinite(lo) || !std::isfinite(hi) || lo < 0.0f || lo > hi)
            return fail(WL_EINVAL, "wl_set_event_timers: term " + std::to_string(k) + ": the range must be finite with 0 <= lo <= hi");
        et.lo[k] = lo; et.hi[k] = hi;
    }
    ensure_device(sim);
    if (n_terms == 0) { free_event_timers(sim); return WL_OK; }
    const int n = sim->cfg.num_envs;
    if (int rc = cuda_check(cudaMalloc(&et.time_left, sizeof(float) * (size_t)n_terms * n), "wl_set_event_timers: allocate")) return rc;
    // drawn and finished before returning, so that a step on any stream afterwards sees the timers
    wl_event_timers_init_kernel<<<(n + WL_EVENT_BS - 1) / WL_EVENT_BS, WL_EVENT_BS>>>(sim->cfg, et);
    int rc = launched(sim, "wl_event_timers_init_kernel");
    if (!rc) rc = cuda_check(cudaDeviceSynchronize(), "wl_set_event_timers: draw");
    if (rc) { cudaFree(et.time_left); return rc; }
    free_event_timers(sim);
    sim->events = et;
    return WL_OK;
}

int wl_event_timers(wl_sim* sim, const uint8_t* d_done, uint8_t* d_fired, int64_t step_counter, void* stream) {
    if (!sim || !d_done || !d_fired) return fail(WL_EINVAL, "wl_event_timers: null argument");
    if (step_counter < 0 || step_counter >= ((int64_t)1 << 31)) return fail(WL_EINVAL, "wl_event_timers: step_counter out of range (0 <= t < 2^31)");
    if (sim->events.n < 1) return fail(WL_EINVAL, "wl_event_timers: no event timers (wl_set_event_timers)");
    if (fan_set(sim)) return fail(WL_EINVAL, "wl_event_timers: the peer fan-out is set, and event timers run with the staged step only");
    ensure_device(sim);
    const int n = sim->cfg.num_envs;
    wl_event_timers_kernel<<<(n + WL_EVENT_BS - 1) / WL_EVENT_BS, WL_EVENT_BS, 0, (cudaStream_t)stream>>>(sim->cfg, sim->events, d_done, d_fired,
                                                                                                          (uint32_t)step_counter);
    return launched(sim, "wl_event_timers_kernel");
}

}   // extern "C"
static int launch_device_events(wl_sim* sim, const uint8_t* d_terminated, const uint8_t* d_truncated, uint32_t t, cudaStream_t cs) {
    const int n = sim->cfg.num_envs;
    wl_device_events_kernel<<<(n + WL_DEVICE_EVENTS_BS - 1) / WL_DEVICE_EVENTS_BS, WL_DEVICE_EVENTS_BS, 0, cs>>>(
        sim->cfg, sim->devents->et, sim->state, sim->globals, d_terminated, d_truncated, t);
    return launched(sim, "wl_device_events_kernel");
}
extern "C" {

int wl_set_device_events(wl_sim* sim, const wl_device_event_desc* table, int32_t n_terms) {
    if (!sim) return fail(WL_EINVAL, "wl_set_device_events: null handle");
    if (n_terms < 0 || n_terms > WL_MAX_DEVICE_EVENTS) return fail(WL_EINVAL, "wl_set_device_events: n_terms must be 0..8");
    if (n_terms > 0 && !table) return fail(WL_EINVAL, "wl_set_device_events: null term table");
    if (fan_set(sim)) return fail(WL_EINVAL, "wl_set_device_events: the peer fan-out is set, and device events run with wl_step_terms only");
    DevEventTable et{};
    et.n = n_terms;
    for (int k = 0; k < n_terms; ++k) {
        const wl_device_event_desc& d = table[k];
        const std::string term = "wl_set_device_events: term " + std::to_string(k);
        if (d.mode != WL_EVENT_MODE_RESET && d.mode != WL_EVENT_MODE_INTERVAL) return fail(WL_EINVAL, term + ": unknown mode");
        for (int j = 0; j < 6; ++j) {
            const float lo = d.velocity_range[j][0], hi = d.velocity_range[j][1];
            if (!std::isfinite(lo) || !std::isfinite(hi) || lo > hi)
                return fail(WL_EINVAL, term + ": velocity range " + std::to_string(j) + " must be finite with lo <= hi");
            et.lo[k][j] = lo; et.hi[k][j] = hi;
        }
        et.slot[k] = -1;
        if (d.mode == WL_EVENT_MODE_INTERVAL) {
            const float lo = d.interval_range_s[0], hi = d.interval_range_s[1];
            if (!std::isfinite(lo) || !std::isfinite(hi) || lo < 0.0f || lo > hi)
                return fail(WL_EINVAL, term + ": interval_range_s must be finite with 0 <= lo <= hi");
            et.slot[k] = et.timers.n;
            et.timers.lo[et.timers.n] = lo; et.timers.hi[et.timers.n] = hi;
            ++et.timers.n;
        }
    }
    ensure_device(sim);
    if (n_terms == 0) { free_device_events(sim); return WL_OK; }
    const size_t n = (size_t)sim->cfg.num_envs, o_bits = align256((size_t)et.timers.n * n * 4), bytes = o_bits + align256(n);
    char* blk = nullptr;
    if (int rc = cuda_check(cudaMalloc(&blk, bytes), "wl_set_device_events: allocate")) return rc;
    DevEvents* de = new (std::nothrow) DevEvents();
    if (!de) { cudaFree(blk); return fail(WL_EINVAL, "wl_set_device_events: out of host memory"); }
    et.timers.time_left = et.timers.n ? reinterpret_cast<float*>(blk) : nullptr;
    int rc = cuda_check(cudaMemset(blk + o_bits, 0, n), "wl_set_device_events: clear");
    if (!rc && et.timers.n) {       // the interval timers, drawn as wl_set_event_timers draws them
        wl_event_timers_init_kernel<<<(unsigned)((n + WL_EVENT_BS - 1) / WL_EVENT_BS), WL_EVENT_BS>>>(sim->cfg, et.timers);
        rc = launched(sim, "wl_event_timers_init_kernel");
    }
    // finished before returning, so that a step on any stream afterwards sees the timers
    if (!rc) rc = cuda_check(cudaDeviceSynchronize(), "wl_set_device_events: draw");
    if (rc) { cudaFree(blk); delete de; return rc; }
    de->et = et;
    de->tbits = reinterpret_cast<uint8_t*>(blk + o_bits);
    de->block = blk;
    free_device_events(sim);
    sim->devents = de;
    return WL_OK;
}

int wl_device_events(wl_sim* sim, const uint8_t* d_terminated, const uint8_t* d_truncated, int64_t step_counter, void* stream) {
    if (!sim || !d_terminated || !d_truncated) return fail(WL_EINVAL, "wl_device_events: null argument");
    if (int rc = check_counter("wl_device_events", step_counter)) return rc;
    if (!sim->devents) return fail(WL_EINVAL, "wl_device_events: no device event terms (wl_set_device_events)");
    if (fan_set(sim)) return fail(WL_EINVAL, "wl_device_events: the peer fan-out is set, and device events run with wl_step_terms only");
    ensure_device(sim);
    return launch_device_events(sim, d_terminated, d_truncated, (uint32_t)step_counter, (cudaStream_t)stream);
}

int wl_set_device_terms(wl_sim* sim, const wl_term_desc* terms, int32_t n_terms) {
    if (!sim) return fail(WL_EINVAL, "wl_set_device_terms: null handle");
    if (n_terms < 0 || n_terms > WL_MAX_DEVICE_TERMS) return fail(WL_EINVAL, "wl_set_device_terms: at most 8 device terms");
    if (n_terms > 0 && !terms) return fail(WL_EINVAL, "wl_set_device_terms: null term table");
    TermTable tt;
    memset(&tt, 0, sizeof tt);
    tt.n = n_terms;
    const double step_dt = (double)sim->cfg.sim_dt * (double)sim->cfg.decimation;      // TaskSpec.step_dt
    for (int k = 0; k < n_terms; ++k) {
        const wl_term_desc& d = terms[k];
        if (d.kind < 1 || d.kind >= WL_TERM_KINDS) return fail(WL_EINVAL, "wl_set_device_terms: unknown term kind " + std::to_string(d.kind));
        if (d.role < WL_TERM_ROLE_REWARD || d.role > WL_TERM_ROLE_TIME_OUT) return fail(WL_EINVAL, "wl_set_device_terms: unknown role");
        if (!std::isfinite(d.weight)) return fail(WL_EINVAL, "wl_set_device_terms: non-finite weight");
        for (int j = 0; j < 4; ++j)
            if (!std::isfinite(d.params[j])) return fail(WL_EINVAL, "wl_set_device_terms: non-finite parameter");
        const bool map = d.kind == WL_TERM_V_IS_TRAVERSABLE || d.kind == WL_TERM_V_IS_TRAVERSABLE_SPEED_SCALED ||
                         d.kind == WL_TERM_V_VEL_REW_TRAV || d.kind == WL_TERM_V_BOOL_IS_NOT_TRAVERSABLE;
        if (map && sim->cfg.task != WL_TASK_VISUAL)
            return fail(WL_EUNSUPPORTED, "wl_set_device_terms: a traversability-map term needs the Visual task");
        tt.kind[k] = d.kind;
        tt.role[k] = d.role;
        tt.scale[k] = d.role == WL_TERM_ROLE_REWARD ? (float)(d.weight * step_dt) : 0.0f;
        tt.skip[k] = d.role == WL_TERM_ROLE_REWARD && d.weight == 0.0;
        for (int j = 0; j < 4; ++j) tt.p[k][j] = (float)d.params[j];
        if (d.kind == WL_TERM_V_OFF_TRACK) tt.p[k][2] = (float)(d.params[1] * d.params[1]);     // corner_out_radius**2 in double
    }
    ensure_device(sim);
    if (n_terms == 0) { free_device_terms(sim); return WL_OK; }
    const size_t n = (size_t)sim->cfg.num_envs, ctas = (n + WL_TERMS_BS - 1) / WL_TERMS_BS;
    const size_t o_sums = 0, o_prev = align256(o_sums + WL_MAX_DEVICE_TERMS * n * 4), o_part = align256(o_prev + n * 4),
                 o_bytes = align256(o_part + ctas * 16 * 4), bytes = o_bytes + 4 * align256(n);
    // the new table and state are built completely before the old ones are dropped: a failure leaves the handle as it was
    char* blk = nullptr;
    if (int rc = cuda_check(cudaMalloc(&blk, bytes), "wl_set_device_terms: allocate")) return rc;
    DevTerms* dt = new (std::nothrow) DevTerms();
    if (!dt) { cudaFree(blk); return fail(WL_EINVAL, "wl_set_device_terms: out of host memory"); }
    // cleared and finished before returning, so that a step on any stream afterwards sees the cleared state
    int rc = cuda_check(cudaMemset(blk, 0, bytes), "wl_set_device_terms: clear");
    if (!rc) rc = cuda_check(cudaMemset(blk + o_prev, 0xFF, n * 4), "wl_set_device_terms: clear");    // NaN: not called yet
    if (!rc) rc = cuda_check(cudaDeviceSynchronize(), "wl_set_device_terms: synchronize");
    if (rc) { cudaFree(blk); delete dt; return rc; }
    dt->tt = tt;
    dt->block = blk;
    dt->b.sums = reinterpret_cast<float*>(blk + o_sums);
    dt->b.prev = reinterpret_cast<float*>(blk + o_prev);
    dt->b.part = reinterpret_cast<float*>(blk + o_part);
    dt->b.extra_term = reinterpret_cast<uint8_t*>(blk + o_bytes);
    dt->b.extra_to = dt->b.extra_term + align256(n);
    dt->b.fired = dt->b.extra_to + align256(n);
    dt->tbits = dt->b.fired + align256(n);
    free_device_terms(sim);
    sim->dterms = dt;
    return WL_OK;
}

uint8_t* wl_device_term_masks(const wl_sim* sim) { return (sim && sim->dterms) ? sim->dterms->b.fired : nullptr; }

int wl_step_terms(wl_sim* sim, const float* d_action, float* d_obs, float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated,
                  float* d_log, float* d_term_log, int64_t step_counter, void* stream) {
    if (!sim || !d_action || !d_obs || !d_rew || !d_terminated || !d_truncated) return fail(WL_EINVAL, "wl_step_terms: null argument");
    if (((uintptr_t)d_action & 7u) || ((uintptr_t)d_obs & 7u)) return fail(WL_EINVAL, "wl_step_terms: action/obs must be 8-byte aligned");
    if (int rc = refuse_fan(sim, "wl_step_terms")) return rc;
    cudaStream_t cs = (cudaStream_t)stream;
    DevTerms* dt = sim->dterms;
    DevEvents* de = sim->devents;
    if (!dt && !de) return wl_step(sim, d_action, d_obs, d_rew, d_terminated, d_truncated, d_log, step_counter, stream);   // wl_step itself
    if (int rc = prep_step(sim, step_counter, 1, cs)) return rc;
    const uint32_t t = (uint32_t)step_counter;               // negative (device base + k) stays encoded: see decode_step
    uint8_t* tbits = sim->term_bits ? sim->term_bits : dt ? dt->tbits : de->tbits;
    if (int rc = launch_stage<1>(sim, reinterpret_cast<const float2*>(d_action), nullptr, d_rew, nullptr, nullptr, nullptr, t,
                                 StageIO{tbits, nullptr, nullptr}, cs)) return rc;
    const int n = sim->cfg.num_envs, ctas = (n + WL_TERMS_BS - 1) / WL_TERMS_BS;
    if (dt) {
        wl_terms_kernel<<<ctas, WL_TERMS_BS, 0, cs>>>(dt->tt, sim->cfg, sim->state, sim->globals, sim->hf, t, d_rew, tbits, dt->b,
                                                      d_term_log != nullptr);
        if (int rc = launched(sim, "wl_terms_kernel")) return rc;
        if (d_term_log) {
            wl_terms_log_kernel<<<1, 9 * 32, 0, cs>>>(dt->tt, sim->cfg, dt->b.part, ctas, d_term_log);
            if (int rc = launched(sim, "wl_terms_log_kernel")) return rc;
        }
    }
    const StageIO sio{tbits, dt ? dt->b.extra_term : nullptr, dt ? dt->b.extra_to : nullptr};
    if (de) {   // stage b cut after the reset and the built-in pushes: the reset-mode DR, then the device events, then b2
        if (int rc = launch_stage<3>(sim, nullptr, nullptr, nullptr, d_terminated, d_truncated, d_log, t, sio, cs)) return rc;
        if (int rc = reset_dr(sim, nullptr, n, step_counter, true, cs)) return rc;
        if (int rc = launch_device_events(sim, d_terminated, d_truncated, t, cs)) return rc;
        if (int rc = launch_stage<4>(sim, nullptr, d_obs, nullptr, nullptr, nullptr, nullptr, t, StageIO{nullptr, nullptr, nullptr}, cs)) return rc;
    } else if (int rc = launch_stage<2>(sim, nullptr, d_obs, nullptr, d_terminated, d_truncated, d_log, t, sio, cs)) {
        return rc;
    }
    if (int rc = launch_row_tail(sim, d_obs, t, true, -1, cs)) return rc;
    return de ? post_step(sim, step_counter, cs) : end_step(sim, step_counter, cs);     // (with device events reset_dr ran above)
}

int wl_rollout(wl_sim* sim, int32_t K, const float* d_actions, float* d_actions_out, float* d_obs, float* d_rew,
               uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream) {
    if (!sim || !d_obs || !d_rew || !d_terminated || !d_truncated || !d_log) return fail(WL_EINVAL, "wl_rollout: null argument");
    if (K < 1) return fail(WL_EINVAL, "wl_rollout: K must be >= 1");
    if (int rc = refuse_fan(sim, "wl_rollout")) return rc;
    if (int rc = refuse_devents(sim, "wl_rollout")) return rc;
    if (int rc = refuse_pobs(sim, "wl_rollout")) return rc;
    if (int rc = refuse_rows(sim, "wl_rollout")) return rc;
    if (sim->cfg.task == WL_TASK_ELEVATION) return fail(WL_EUNSUPPORTED, "wl_rollout: the elevation step is two kernels (use wl_step)");
    if (sim->cfg.task == WL_TASK_VISUAL && sim->cfg.vis_cam) return fail(WL_EUNSUPPORTED, "wl_rollout: the camera term is a second kernel (use wl_step)");
    if (sim->reset_ev) return fail(WL_EUNSUPPORTED, "wl_rollout: the reset-mode DR events are a second kernel after each step (use wl_step)");
    if (sim->cfg.curr_n > 0) {
        if (step_counter < 0) return fail(WL_EINVAL, "wl_rollout: with curriculum terms the host must pass the step counter");
        const int64_t L = sim->cfg.max_episode_length;
        // counters after steps 0..K-2 are t+1..t+K-1: none may be an episode boundary (only the last step may end on one)
        if ((step_counter + K - 1) / L != step_counter / L)
            return fail(WL_EINVAL, "wl_rollout: [t, t+K) must end at or before the next episode boundary of the global counter");
    }
    const int n = sim->cfg.num_envs;
    Terrain T{sim->hf};
    const int bs = 32, threads = 4 * n, grid = (threads + bs - 1) / bs;
    cudaStream_t cs = (cudaStream_t)stream;
    ensure_device(sim);
    if (int rc = cuda_check(cudaMemsetAsync(d_log, 0, (size_t)K * WL_LOG_FLOATS * sizeof(float), cs), "wl_rollout: clear log rows")) return rc;
    if (int rc = prep_step(sim, step_counter, K, cs)) return rc;
    const float2* act = reinterpret_cast<const float2*>(d_actions);
    float2* aout = reinterpret_cast<float2*>(d_actions_out);
    with_task<WL_TASK_VISUAL>(sim->cfg.task, [&](auto task) {
        wl_rollout_quad_kernel<task><<<grid, bs, 0, cs>>>(sim->cfg, sim->state, sim->globals, T, act, aout, d_obs, d_rew, d_terminated, d_truncated, d_log, (uint32_t)step_counter, K, &sim->globals->ticket);
    });
    if (int rc = launched(sim, "wl_rollout_quad_kernel")) return rc;
    return post_step(sim, step_counter, cs);
}

size_t wl_result_bytes(int32_t num_envs) { return (size_t)num_envs * 6u; }

int wl_step_host(wl_sim* sim, const float* h_action, float* d_action, float* d_obs, void* d_result, float* d_log,
                 void* h_result, float* h_obs, int64_t step_counter, void* stream) {
    if (!sim || !h_action || !d_action || !d_obs || !d_result || !h_result) return fail(WL_EINVAL, "wl_step_host: null argument");
    if (int rc = refuse_fan(sim, "wl_step_host")) return rc;     // (its rows are the caller's result block, not a slab's)
    const size_t n = (size_t)sim->cfg.num_envs;
    cudaStream_t cs = (cudaStream_t)stream;
    ensure_device(sim);
    if (int rc = cuda_check(cudaMemcpyAsync(d_action, h_action, n * 2 * sizeof(float), cudaMemcpyHostToDevice, cs), "H2D actions")) return rc;
    float* d_rew = reinterpret_cast<float*>(d_result);
    uint8_t* d_term = reinterpret_cast<uint8_t*>(d_result) + n * 4;
    uint8_t* d_trunc = d_term + n;
    if (int rc = wl_step(sim, d_action, d_obs, d_rew, d_term, d_trunc, d_log, step_counter, stream)) return rc;
    if (int rc = cuda_check(cudaMemcpyAsync(h_result, d_result, wl_result_bytes((int32_t)n), cudaMemcpyDeviceToHost, cs), "D2H results")) return rc;
    if (h_obs) {
        if (int rc = cuda_check(cudaMemcpyAsync(h_obs, d_obs, n * (size_t)sim->obs_dim * sizeof(float), cudaMemcpyDeviceToHost, cs), "D2H obs")) return rc;
    }
    return cuda_check(cudaStreamSynchronize(cs), "wl_step_host: stream synchronize");
}

// device alias of a pinned host block (cudaHostGetDevicePointer is a driver call: resolved once per block and cached)
static void* host_alias(wl_sim* sim, const void* h) {
    for (int k = 0; k < sim->hp_n; ++k) if (sim->hp_host[k] == h) return sim->hp_dev[k];
    void* d = nullptr;
    if (cudaHostGetDevicePointer(&d, const_cast<void*>(h), 0) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    const int slot = sim->hp_n < 8 ? sim->hp_n++ : (int)(((uintptr_t)h >> 6) & 7u);
    sim->hp_host[slot] = h; sim->hp_dev[slot] = d;
    return d;
}

int wl_step_host_zero_copy(wl_sim* sim, const float* h_action, float* d_obs, float* d_log, void* h_result,
                           int64_t step_counter, void* stream) {
    if (!sim || !h_action || !d_obs || !h_result) return fail(WL_EINVAL, "wl_step_host_zero_copy: null argument");
    if (int rc = refuse_fan(sim, "wl_step_host_zero_copy")) return rc;
    const size_t n = (size_t)sim->cfg.num_envs;
    const float* da = reinterpret_cast<const float*>(host_alias(sim, h_action));
    void* dr = host_alias(sim, h_result);
    if (!da || !dr) return fail(WL_EINVAL, "wl_step_host_zero_copy: h_action / h_result must be pinned (device-mapped) host memory");
    float* d_rew = reinterpret_cast<float*>(dr);
    uint8_t* d_term = reinterpret_cast<uint8_t*>(dr) + n * 4;
    uint8_t* d_trunc = d_term + n;
    if (int rc = wl_step(sim, da, d_obs, d_rew, d_term, d_trunc, d_log, step_counter, stream)) return rc;
    return cuda_check(cudaStreamSynchronize((cudaStream_t)stream), "wl_step_host_zero_copy: stream synchronize");
}

int wl_observe(wl_sim* sim, float* d_obs, int64_t step_counter, int32_t call_idx, void* stream) {
    if (!sim || !d_obs) return fail(WL_EINVAL, "wl_observe: null argument");
    if (sim->rows.n_terms && (call_idx < 0 || call_idx > WL_ROW_MAX_CALL))
        return fail(WL_EINVAL, "wl_observe: with row terms call_idx must be in 0..2^23-2 (it keys their noise)");
    ensure_device(sim);
    const int n = sim->cfg.num_envs, bs = 128;
    wl_observe_kernel<<<(n + bs - 1) / bs, bs, 0, (cudaStream_t)stream>>>(sim->cfg, sim->state, d_obs, (uint32_t)step_counter,
                                                                         (uint32_t)call_idx);
    if (int rc = launched(sim, "wl_observe_kernel")) return rc;
    return launch_row_tail(sim, d_obs, (uint32_t)step_counter, false, call_idx, (cudaStream_t)stream);
}

int wl_camera(wl_sim* sim, float* d_obs, int64_t step_counter, const float* d_aug, void* stream) {
    if (!sim || !d_obs) return fail(WL_EINVAL, "wl_camera: null argument");
    ensure_device(sim);
    if (sim->cfg.task != WL_TASK_VISUAL || !sim->cfg.vis_cam) return fail(WL_EUNSUPPORTED, "wl_camera: the handle has no camera term");
    return launch_camera(sim, d_obs, (uint32_t)step_counter, RNG_CAM, 0u, d_aug, (cudaStream_t)stream);
}

int wl_curriculum(wl_sim* sim, int32_t n_terms, const int32_t* slots, const float* increases, uint32_t fire_mask,
                  void* stream) {
    if (!sim) return fail(WL_EINVAL, "wl_curriculum: null handle");
    ensure_device(sim);
    if (n_terms < 0 || n_terms > WL_MAX_REW_TERMS) return fail(WL_EINVAL, "wl_curriculum: n_terms");
    if (n_terms == 0 || fire_mask == 0) return WL_OK;
    CurrArgs a; memset(&a, 0, sizeof a);
    a.n = n_terms; a.fire_mask = fire_mask;
    if (sim->last_t < 0) return WL_OK;                       // no step yet: no env has reset
    a.wslot = (uint32_t)sim->last_t & 1u; a.row = (uint32_t)sim->last_t % 3u;
    for (int t = 0; t < n_terms; ++t) {
        if (slots[t] < 0 || slots[t] >= WL_MAX_REW_TERMS) return fail(WL_EINVAL, "wl_curriculum: slot out of range");
        a.slots[t] = slots[t]; a.inc[t] = increases[t];
    }
    wl_curriculum_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(sim->globals, a);
    return launched(sim, "wl_curriculum_kernel");
}

int wl_synth_actions(wl_sim* sim, float* d_action, int64_t step_counter, int32_t dist, void* stream) {
    if (!sim || !d_action) return fail(WL_EINVAL, "wl_synth_actions: null argument");
    ensure_device(sim);
    const int n = sim->cfg.num_envs, bs = 128;
    wl_synth_actions_kernel<<<(n + bs - 1) / bs, bs, 0, (cudaStream_t)stream>>>(sim->cfg, sim->globals, reinterpret_cast<float2*>(d_action),
                                                                               (uint32_t)step_counter, dist);
    return launched(sim, "wl_synth_actions_kernel");
}

int wl_derive_suspension(wl_sim* sim, float* d_susp_pos, float* d_susp_vel, void* stream) {
    if (!sim || !d_susp_pos || !d_susp_vel) return fail(WL_EINVAL, "wl_derive_suspension: null argument");
    ensure_device(sim);
    if (((uintptr_t)d_susp_pos & 15u) || ((uintptr_t)d_susp_vel & 15u)) return fail(WL_EINVAL, "wl_derive_suspension: outputs must be 16-byte aligned");
    const int n = sim->cfg.num_envs, bs = 128;
    Terrain T{sim->hf};
    with_task<WL_TASK_ELEVATION>(sim->cfg.task, [&](auto task) {
        wl_suspension_kernel<task><<<(n + bs - 1) / bs, bs, 0, (cudaStream_t)stream>>>(sim->cfg, sim->state, T, (float4*)d_susp_pos, (float4*)d_susp_vel);
    });
    return launched(sim, "wl_suspension_kernel");
}

int32_t wl_policy_blob_floats(int32_t obs_dim, int32_t offsets[13]) {
    int32_t tmp[13];
    return policy_offsets(obs_dim, offsets ? offsets : tmp);
}
int32_t wl_policy_blob_floats_asym(int32_t obs_dim, int32_t critic_obs_dim, int32_t offsets[13]) {
    int32_t tmp[13];
    return policy_offsets(obs_dim, offsets ? offsets : tmp, critic_obs_dim);
}

int wl_set_critic_terms(wl_sim* sim, const wl_critic_term* terms, int32_t n_terms) {
    if (!sim) return fail(WL_EINVAL, "wl_set_critic_terms: null handle");
    if (n_terms < 0 || n_terms > WL_MAX_CRITIC_TERMS) return fail(WL_EINVAL, "wl_set_critic_terms: at most 16 critic terms");
    if (n_terms > 0 && !terms) return fail(WL_EINVAL, "wl_set_critic_terms: null term table");
    if (sim->cfg.task != WL_TASK_DRIFT) return fail(WL_EUNSUPPORTED, "wl_set_critic_terms: the critic observation is implemented for the Drift family only");
    CriticTable tb;
    memset(&tb, 0, sizeof tb);
    for (int k = 0; k < n_terms; ++k) {
        const wl_critic_term& d = terms[k];
        if (d.kind < 1 || d.kind >= WL_CRITIC_KINDS) return fail(WL_EINVAL, "wl_set_critic_terms: unknown term kind " + std::to_string(d.kind));
        if (!std::isfinite(d.clip) || d.clip < 0.0f) return fail(WL_EINVAL, "wl_set_critic_terms: clip must be finite and >= 0");
        if (tb.n_cols + critic_width(d.kind) > WL_MAX_CRITIC_OBS) return fail(WL_EINVAL, "wl_set_critic_terms: the critic row is wider than 32 floats");
        for (int j = 0; j < critic_width(d.kind); ++j) {
            tb.src[tb.n_cols] = (uint8_t)(critic_first(d.kind) + j);
            tb.clip[tb.n_cols++] = d.clip;
        }
        tb.groups |= critic_groups(d.kind);
    }
    sim->critic = tb;
    return WL_OK;
}
int32_t wl_critic_obs_dim(const wl_sim* sim) {
    if (!sim) return 0;
    return sim->crit_rows.n_terms ? WL_OBS_DIM_ELEV + sim->crit_extra.n_cols : sim->critic.n_cols;
}

int wl_set_policy_terms(wl_sim* sim, const wl_policy_term* terms, int32_t n_terms) {
    const std::string fn = "wl_set_policy_terms: ";
    if (!sim) return fail(WL_EINVAL, fn + "null handle");
    if (n_terms < 0 || n_terms > WL_MAX_POLICY_TERMS) return fail(WL_EINVAL, fn + "at most 16 policy terms");
    if (n_terms > 0 && !terms) return fail(WL_EINVAL, fn + "null term table");
    if (sim->cfg.task != WL_TASK_DRIFT) return fail(WL_EUNSUPPORTED, fn + "a policy observation table is implemented for the Drift family only");
    if (fan_set(sim)) return fail(WL_EUNSUPPORTED, fn + "the peer fan-out is set, and only the built-in row carries it");
    PolicyObsTable tb;
    memset(&tb, 0, sizeof tb);
    for (int k = 0; k < n_terms; ++k) {
        const wl_policy_term& d = terms[k];
        const std::string at = fn + "term " + std::to_string(k) + ": ";
        if (d.kind < 1 || d.kind >= WL_POLICY_OBS_KINDS) return fail(WL_EINVAL, at + "unknown term kind " + std::to_string(d.kind));
        if (d.noise < WL_NOISE_NONE || d.noise > WL_NOISE_UNIFORM) return fail(WL_EINVAL, at + "unknown noise model " + std::to_string(d.noise));
        const int w = policy_obs_width(d.kind);
        if (d.n_scale != 0 && d.n_scale != 1 && d.n_scale != w) return fail(WL_EINVAL, at + "n_scale must be 0, 1 or the term's width");
        bool finite = std::isfinite(d.noise_params[0]) && std::isfinite(d.noise_params[1]) && std::isfinite(d.clip_range[0]) &&
                      std::isfinite(d.clip_range[1]);
        for (int s = 0; s < 4; ++s) finite = finite && std::isfinite(d.scale[s]);
        if (!finite) return fail(WL_EINVAL, at + "a noise, clip or scale parameter is not finite");
        if (tb.n_cols + w > WL_MAX_POLICY_OBS) return fail(WL_EINVAL, fn + "the policy row is wider than 32 floats");
        for (int j = 0; j < w; ++j, ++tb.n_cols) {
            const int c = tb.n_cols;
            tb.src[c] = (uint8_t)(policy_obs_first(d.kind) + j);
            tb.noise[c] = (uint8_t)d.noise;
            tb.na[c] = (float)d.noise_params[0];
            tb.nb[c] = d.noise == WL_NOISE_UNIFORM ? (float)(d.noise_params[1] - d.noise_params[0]) : (float)d.noise_params[1];
            tb.flags[c] = (uint8_t)((d.clip ? WL_POBS_CLIP : 0u) | (d.n_scale ? WL_POBS_SCALE : 0u));
            tb.lo[c] = (float)d.clip_range[0];
            tb.hi[c] = (float)d.clip_range[1];
            tb.scale[c] = d.n_scale ? (float)d.scale[d.n_scale == 1 ? 0 : j] : 1.0f;
        }
        tb.groups |= policy_obs_groups(d.kind);
    }
    sim->pobs = tb;
    return WL_OK;
}
int32_t wl_policy_obs_dim(const wl_sim* sim) { return sim ? sim->pobs.n_cols : 0; }
int wl_policy_observe(wl_sim* sim, int64_t step_counter, int32_t call_idx, float* d_out, void* stream) {
    const std::string fn = "wl_policy_observe: ";
    if (!sim || !d_out) return fail(WL_EINVAL, fn + "null argument");
    if ((uintptr_t)d_out & 3u) return fail(WL_EINVAL, fn + "d_out must be 4-byte aligned");
    if (sim->pobs.n_cols < 1) return fail(WL_EINVAL, fn + "no policy table (wl_set_policy_terms)");
    if (step_counter >= ((int64_t)1 << 31) || step_counter < -((int64_t)1 << 31))
        return fail(WL_EINVAL, fn + "step counter out of range (< 2^31, or WL_DEVICE_COUNTER_PLUS(k))");
    if (call_idx < WL_POLICY_OBS_AFTER_STEP || call_idx >= (1 << 27)) return fail(WL_EINVAL, fn + "call_idx must be in -1..2^27-1");
    if (fan_set(sim)) return fail(WL_EUNSUPPORTED, fn + "the peer fan-out is set, and only the built-in row carries it");
    ensure_device(sim);
    const int n = sim->cfg.num_envs;
    wl_policy_observe_kernel<<<(n + WL_POBS_ENVS - 1) / WL_POBS_ENVS, WL_POBS_THREADS, 0, (cudaStream_t)stream>>>(
        sim->pobs, sim->state, sim->globals, n, sim->cfg.seed, sim->cfg.env_id_offset, sim->cfg.enable_corruption, (uint32_t)step_counter,
        call_idx, d_out);
    return launched(sim, "wl_policy_observe_kernel");
}

// The row table of the Elevation / Visual terms `terms` (n_terms: 0 or the task's count), every term checked before `tb` is
// written; noise kept only when `corrupt`.  Error messages start with fn.
static int row_table(const std::string& fn, int task, const wl_policy_term* terms, int32_t n_terms, bool corrupt, RowTable& out) {
    static const int elev[WL_ROW_TERMS_ELEVATION] = {WL_ROW_GOAL_RELATIVE_XYZ, WL_CRITIC_ROOT_EULER_XYZ, WL_CRITIC_BASE_LIN_VEL,
                                                     WL_CRITIC_BASE_ANG_VEL, WL_CRITIC_LAST_ACTION, WL_ROW_WORLD_HEIGHT_MAP};
    static const int vis[WL_ROW_TERMS_VISUAL] = {WL_CRITIC_BASE_LIN_VEL, WL_CRITIC_BASE_ANG_VEL, WL_CRITIC_LAST_ACTION};
    const int* kinds = task == WL_TASK_ELEVATION ? elev : vis;
    const int count = task == WL_TASK_ELEVATION ? WL_ROW_TERMS_ELEVATION : WL_ROW_TERMS_VISUAL;
    if (n_terms != 0 && n_terms != count)
        return fail(WL_EINVAL, fn + "n_terms must be 0 or the task's " + std::to_string(count) + " terms");
    RowTable tb;
    memset(&tb, 0, sizeof tb);
    int col = 0;
    for (int k = 0; k < n_terms; ++k) {
        const wl_policy_term& d = terms[k];
        const std::string at = fn + "term " + std::to_string(k) + ": ";
        if (d.kind != kinds[k]) return fail(WL_EINVAL, at + "kind " + std::to_string(d.kind) + " is not the row's term " + std::to_string(kinds[k]));
        if (d.noise < WL_NOISE_NONE || d.noise > WL_NOISE_UNIFORM) return fail(WL_EINVAL, at + "unknown noise model " + std::to_string(d.noise));
        const bool map = d.kind == WL_ROW_WORLD_HEIGHT_MAP;
        const int w = map ? WL_SCAN_RAYS : d.kind == WL_ROW_GOAL_RELATIVE_XYZ ? 2 : critic_width(d.kind);
        if (map ? (d.n_scale != 0 && d.n_scale != 1) : (d.n_scale != 0 && d.n_scale != 1 && d.n_scale != w))
            return fail(WL_EINVAL, at + (map ? "n_scale must be 0 or 1 on the height map" : "n_scale must be 0, 1 or the term's width"));
        bool finite = std::isfinite(d.noise_params[0]) && std::isfinite(d.noise_params[1]) && std::isfinite(d.clip_range[0]) &&
                      std::isfinite(d.clip_range[1]);
        for (int s = 0; s < 4; ++s) finite = finite && std::isfinite(d.scale[s]);
        if (!finite) return fail(WL_EINVAL, at + "a noise, clip or scale parameter is not finite");
        for (int j = 0; j < (map ? 1 : w); ++j) {
            RowStage& s = map ? tb.map : tb.col[col++];
            s.noise = corrupt ? d.noise : WL_NOISE_NONE;
            s.na = (float)d.noise_params[0];
            s.nb = d.noise == WL_NOISE_UNIFORM ? (float)(d.noise_params[1] - d.noise_params[0]) : (float)d.noise_params[1];
            s.flags = (d.clip ? WL_ROW_CLIP : 0u) | (d.n_scale ? WL_ROW_SCALE : 0u);
            s.lo = (float)d.clip_range[0];
            s.hi = (float)d.clip_range[1];
            s.sc = d.n_scale ? (float)d.scale[d.n_scale == 1 ? 0 : j] : 1.0f;
            tb.noisy |= s.noise != WL_NOISE_NONE;
        }
    }
    tb.n_terms = n_terms;
    out = tb;
    return WL_OK;
}

int wl_set_row_terms(wl_sim* sim, const wl_policy_term* terms, int32_t n_terms) {
    const std::string fn = "wl_set_row_terms: ";
    if (!sim) return fail(WL_EINVAL, fn + "null handle");
    if (n_terms > 0 && !terms) return fail(WL_EINVAL, fn + "null term table");
    const int task = sim->cfg.task;
    if (task != WL_TASK_ELEVATION && task != WL_TASK_VISUAL)
        return fail(WL_EUNSUPPORTED, fn + "row terms are implemented for the Elevation and Visual tasks (the Drift family's groups go through wl_set_policy_terms)");
    if (fan_set(sim)) return fail(WL_EUNSUPPORTED, fn + "the peer fan-out is set, and only the built-in row carries it");
    if (sim->scan_mode == 2 && task == WL_TASK_ELEVATION)
        return fail(WL_EUNSUPPORTED, fn + "the pipelined ray-caster (wl_set_scan_tma(2)) has no row-terms variant");
    return row_table(fn, task, terms, n_terms, sim->cfg.enable_corruption != 0, sim->rows);
}

int wl_set_row_critic(wl_sim* sim, const wl_policy_term* row_terms, int32_t n_row_terms, const wl_critic_term* extra, int32_t n_extra) {
    const std::string fn = "wl_set_row_critic: ";
    if (!sim) return fail(WL_EINVAL, fn + "null handle");
    if ((n_row_terms > 0 && !row_terms) || (n_extra > 0 && !extra)) return fail(WL_EINVAL, fn + "null term table");
    if (sim->cfg.task != WL_TASK_ELEVATION)
        return fail(WL_EUNSUPPORTED, fn + "a row critic is implemented for the Elevation task only (the Drift family's critic: wl_set_critic_terms)");
    if (n_row_terms == 0 && n_extra != 0) return fail(WL_EINVAL, fn + "extra columns need the row terms");
    if (n_extra < 0 || n_extra > WL_MAX_CRITIC_TERMS) return fail(WL_EINVAL, fn + "at most 16 extra critic terms");
    RowTable rt;
    if (int rc = row_table(fn, WL_TASK_ELEVATION, row_terms, n_row_terms, false, rt)) return rc;
    static const char* const names[WL_ROW_TERMS_ELEVATION] = {"goal_relative_xyz", "root_euler_xyz", "base_lin_vel", "base_ang_vel",
                                                              "last_action", "world_height_map"};
    for (int k = 0; k < n_row_terms; ++k) {
        const std::string at = fn + "term " + std::to_string(k) + " (" + names[k] + "): ";
        if (row_terms[k].noise != WL_NOISE_NONE) return fail(WL_EINVAL, at + "the critic row is noise-free (noise must be WL_NOISE_NONE)");
        if (k == 5 && !row_terms[k].clip) return fail(WL_EINVAL, at + "the critic's height map needs a finite clip (a miss is +inf)");
    }
    CriticTable ex;
    memset(&ex, 0, sizeof ex);
    for (int k = 0; k < n_extra; ++k) {
        const wl_critic_term& d = extra[k];
        const std::string at = fn + "extra term " + std::to_string(k) + ": ";
        if (d.kind < 1 || d.kind >= WL_CRITIC_KINDS) return fail(WL_EINVAL, at + "unknown term kind " + std::to_string(d.kind));
        if (!std::isfinite(d.clip) || d.clip < 0.0f) return fail(WL_EINVAL, at + "clip must be finite and >= 0");
        if (ex.n_cols + critic_width(d.kind) > WL_MAX_CRITIC_OBS) return fail(WL_EINVAL, fn + "the extra columns are wider than 32 floats");
        for (int j = 0; j < critic_width(d.kind); ++j) {
            ex.src[ex.n_cols] = (uint8_t)(critic_first(d.kind) + j);
            ex.clip[ex.n_cols++] = d.clip;
        }
        ex.groups |= critic_groups(d.kind);
    }
    sim->crit_rows = rt;
    sim->crit_extra = ex;
    return WL_OK;
}
int32_t wl_row_terms(const wl_sim* sim) { return sim ? sim->rows.n_terms : 0; }

int wl_set_reset_events(wl_sim* sim, uint32_t mask) {
    if (!sim) return fail(WL_EINVAL, "wl_set_reset_events: null handle");
    const uint32_t all = WL_RESET_EV_MATERIAL | WL_RESET_EV_ACTUATOR_GAINS | WL_RESET_EV_BASE_MASS | WL_RESET_EV_WHEEL_MASS;
    if (mask & ~all) return fail(WL_EINVAL, "wl_set_reset_events: unknown bit(s) " + std::to_string(mask & ~all));
    const wl_config& c = sim->cfg;
    if (mask && !c.dr_enable) return fail(WL_EINVAL, "wl_set_reset_events: the config has no DR events (dr_enable = 0)");
    if ((mask & WL_RESET_EV_ACTUATOR_GAINS) && c.dr_kd_mask == 0)
        return fail(WL_EINVAL, "wl_set_reset_events: the config has no randomize_actuator_gains event (dr_kd_mask = 0)");
    if ((mask & WL_RESET_EV_WHEEL_MASS) && !c.dr_wheel_mass_enable)
        return fail(WL_EINVAL, "wl_set_reset_events: the config has no wheel-mass event (dr_wheel_mass_enable = 0)");
    sim->reset_ev = mask;
    return WL_OK;
}
uint32_t wl_reset_events(const wl_sim* sim) { return sim ? sim->reset_ev : 0u; }
int wl_critic_observe(wl_sim* sim, float* d_critic_obs, void* stream) {
    if (!sim || !d_critic_obs) return fail(WL_EINVAL, "wl_critic_observe: null argument");
    if ((uintptr_t)d_critic_obs & 3u) return fail(WL_EINVAL, "wl_critic_observe: d_critic_obs must be 4-byte aligned");
    if (sim->critic.n_cols < 1 && !sim->crit_rows.n_terms)
        return fail(WL_EINVAL, "wl_critic_observe: no critic table (wl_set_critic_terms / wl_set_row_critic)");
    ensure_device(sim);
    const int n = sim->cfg.num_envs;
    if (sim->crit_rows.n_terms) {                            // the row critic: the ray-caster again, noise-free (DESIGN 6s)
        const int Dc = WL_OBS_DIM_ELEV + sim->crit_extra.n_cols;
        cudaStream_t cs = (cudaStream_t)stream;
        if (sim->scan_mode >= 1 && sim->has_tmap)
            wl_scan_critic_row_kernel<true><<<n, WL_SCAN_THREADS, 0, cs>>>(sim->cfg, sim->tmap, sim->crit_rows, sim->crit_extra, sim->state, sim->hf, Dc, d_critic_obs);
        else
            wl_scan_critic_row_kernel<false><<<n, WL_SCAN_THREADS, 0, cs>>>(sim->cfg, sim->tmap, sim->crit_rows, sim->crit_extra, sim->state, sim->hf, Dc, d_critic_obs);
        return launched(sim, "wl_scan_critic_row_kernel");
    }
    wl_critic_observe_kernel<<<(n + WL_CRITIC_BS - 1) / WL_CRITIC_BS, WL_CRITIC_BS, 0, (cudaStream_t)stream>>>(sim->critic, sim->state, n, d_critic_obs);
    return launched(sim, "wl_critic_observe_kernel");
}

// wl_act_step and wl_act_infer_step: the same launch of wl_act_step_quad_kernel<task, infer> (arguments checked by the caller
// for null)
static int act_step_launch(bool infer, const char* fn, wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out,
                           float* d_obs, float* d_rew, uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter,
                           void* stream) {
    if (int rc = refuse_fan(sim, fn)) return rc;
    if (int rc = refuse_devents(sim, fn)) return rc;
    if (int rc = refuse_pobs(sim, fn)) return rc;
    if (int rc = refuse_rows(sim, fn)) return rc;
    if (sim->cfg.task == WL_TASK_ELEVATION) return fail(WL_EUNSUPPORTED, std::string(fn) + ": blind-observation tasks only (obs_dim <= 16)");
    if (sim->obs_dim > 16) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim > 16");
    if (((uintptr_t)d_policy_blob & 15u) || ((uintptr_t)out.actions & 7u) || ((uintptr_t)out.mean & 7u))
        return fail(WL_EINVAL, std::string(fn) + ": policy blob must be 16-byte aligned, actions/mean 8-byte aligned");
    PolicyOffsets po;
    const int blob_floats = policy_offsets(sim->obs_dim, po.o);
    const int n = sim->cfg.num_envs, grid = (n + WL_ACT_ENVS - 1) / WL_ACT_ENVS + 1;      // + the janitor CTA
    const size_t smem = sizeof(float) * ((size_t)blob_floats + WL_ACT_ENVS * (WL_ACT_XS + WL_ACT_HS));
    Terrain T{sim->hf};
    cudaStream_t cs = (cudaStream_t)stream;
    if (int rc = prep_step(sim, step_counter, 1, cs)) return rc;
    // all four forms on the first call (prep_step made sim->device current), as the other entry may next run inside a capture
    if (int rc = raise_smem<wl_act_step_quad_kernel<WL_TASK_VISUAL>>(sim->device, 96 * 1024, fn)) return rc;
    if (int rc = raise_smem<wl_act_step_quad_kernel<WL_TASK_DRIFT>>(sim->device, 96 * 1024, fn)) return rc;
    if (int rc = raise_smem<wl_act_step_quad_kernel<WL_TASK_VISUAL, true>>(sim->device, 96 * 1024, fn)) return rc;
    if (int rc = raise_smem<wl_act_step_quad_kernel<WL_TASK_DRIFT, true>>(sim->device, 96 * 1024, fn)) return rc;
    with_task<WL_TASK_VISUAL>(sim->cfg.task, [&](auto task) {
        launch_k(infer ? wl_act_step_quad_kernel<task, true> : wl_act_step_quad_kernel<task, false>, grid, WL_ACT_THREADS, smem, cs, g_pdl,
                 sim->cfg, sim->state, sim->globals, T, d_obs_in, d_policy_blob, blob_floats, po, out, d_obs, d_rew, d_terminated,
                 d_truncated, d_log, (uint32_t)step_counter, sim->obs_dim);
    });
    if (int rc = launched(sim, infer ? "wl_act_step_quad_kernel<infer>" : "wl_act_step_quad_kernel")) return rc;
    return end_step(sim, step_counter, cs);
}

int wl_act_step(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out, float* d_obs, float* d_rew,
                uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream) {
    if (!sim || !d_obs_in || !d_policy_blob || !out.actions || !out.mean || !out.log_prob || !out.value || !d_obs || !d_rew ||
        !d_terminated || !d_truncated)
        return fail(WL_EINVAL, "wl_act_step: null argument");
    return act_step_launch(false, "wl_act_step", sim, d_obs_in, d_policy_blob, out, d_obs, d_rew, d_terminated, d_truncated, d_log,
                           step_counter, stream);
}

int wl_act_infer_step(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, float* d_actions, float* d_obs, float* d_rew,
                      uint8_t* d_terminated, uint8_t* d_truncated, float* d_log, int64_t step_counter, void* stream) {
    if (!sim || !d_obs_in || !d_policy_blob || !d_actions || !d_obs || !d_rew || !d_terminated || !d_truncated)
        return fail(WL_EINVAL, "wl_act_infer_step: null argument");
    const wl_policy_out out{d_actions, nullptr, nullptr, nullptr};
    return act_step_launch(true, "wl_act_infer_step", sim, d_obs_in, d_policy_blob, out, d_obs, d_rew, d_terminated, d_truncated, d_log,
                           step_counter, stream);
}

// wl_policy_act_elu and wl_policy_act_asym (asym: the critic reads d_critic_obs_in, critic_obs_dim wide) after their null
// checks: the same checks, blob and shared-memory sizing, and grid
static int policy_act_narrow(bool asym, const char* fn, wl_sim* sim, const float* d_obs_in, const float* d_critic_obs_in,
                             int32_t critic_obs_dim, const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream) {
    if (((uintptr_t)d_policy_blob & 15u) || ((uintptr_t)out.actions & 7u) || ((uintptr_t)out.mean & 7u) || ((uintptr_t)d_obs_in & 3u) ||
        ((uintptr_t)d_critic_obs_in & 3u) || ((uintptr_t)out.log_prob & 3u) || ((uintptr_t)out.value & 3u))
        return fail(WL_EINVAL, std::string(fn) + ": policy blob must be 16-byte aligned, actions/mean 8-byte aligned, " +
                                   (asym ? "obs_in/critic_obs_in/log_prob/value" : "obs_in/log_prob/value") + " 4-byte aligned");
    if (asym && (critic_obs_dim < 1 || critic_obs_dim > WL_MAX_CRITIC_OBS)) return fail(WL_EINVAL, std::string(fn) + ": critic_obs_dim must be in 1..32");
    if (int rc = check_counter(fn, step_counter)) return rc;
    // no step rows are written, but the step that consumes these actions refuses the fan-out: refuse it here already
    if (int rc = refuse_fan(sim, fn)) return rc;
    const int D = policy_in_dim(sim);
    if (D < 1 || D > 16) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim > 16 (the network wl_act_step runs)");
    ensure_device(sim);
    PolicyOffsets po;
    const int blob_floats = policy_offsets(D, po.o, critic_obs_dim);
    const size_t smem = sizeof(float) * ((size_t)blob_floats + WL_ACT_ENVS * (WL_ACT_XS + WL_ACT_HS + (asym ? WL_ACT_XC : 0)));
    if (int rc = asym ? raise_smem<wl_policy_act_asym_kernel>(sim->device, 96 * 1024, fn) : raise_smem<wl_policy_act_elu_kernel>(sim->device, 96 * 1024, fn))
        return rc;
    const int n = sim->cfg.num_envs, grid = (n + WL_ACT_ENVS - 1) / WL_ACT_ENVS;
    if (asym)
        wl_policy_act_asym_kernel<<<grid, WL_ACT_THREADS, smem, (cudaStream_t)stream>>>(
            sim->cfg, sim->globals, d_obs_in, d_critic_obs_in, critic_obs_dim, d_policy_blob, blob_floats, po, out, (uint32_t)step_counter, D);
    else
        wl_policy_act_elu_kernel<<<grid, WL_ACT_THREADS, smem, (cudaStream_t)stream>>>(
            sim->cfg, sim->globals, d_obs_in, d_policy_blob, blob_floats, po, out, (uint32_t)step_counter, D);
    return launched(sim, asym ? "wl_policy_act_asym_kernel" : "wl_policy_act_elu_kernel");
}

int wl_policy_act_asym(wl_sim* sim, const float* d_obs_in, const float* d_critic_obs_in, int32_t critic_obs_dim,
                       const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream) {
    if (!sim || !d_obs_in || !d_critic_obs_in || !d_policy_blob || !out.actions || !out.mean || !out.log_prob || !out.value)
        return fail(WL_EINVAL, "wl_policy_act_asym: null argument");
    return policy_act_narrow(true, "wl_policy_act_asym", sim, d_obs_in, d_critic_obs_in, critic_obs_dim, d_policy_blob, out, step_counter, stream);
}

int wl_policy_act_elu(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream) {
    if (!sim || !d_obs_in || !d_policy_blob || !out.actions || !out.mean || !out.log_prob || !out.value)
        return fail(WL_EINVAL, "wl_policy_act_elu: null argument");
    return policy_act_narrow(false, "wl_policy_act_elu", sim, d_obs_in, nullptr, 0, d_policy_blob, out, step_counter, stream);
}

int wl_gae(const float* d_rewards, const float* d_values, const float* d_last_values, const uint8_t* d_dones,
           const uint8_t* d_time_outs, float gamma, float lam, float* d_returns, float* d_advantages, int32_t T, int32_t N,
           void* stream) {
    if (!d_rewards || !d_values || !d_last_values || !d_dones || !d_returns || !d_advantages) return fail(WL_EINVAL, "wl_gae: null argument");
    if (T < 1 || N < 1) return fail(WL_EINVAL, "wl_gae: T and N must be >= 1");
    const int S = (T + WL_GAE_SEG - 1) / WL_GAE_SEG;
    if (N <= 65536 && S >= 2 && S <= 16)      // small N: latency-bound -> segment-parallel scan; large N: the streaming scan is bandwidth-bound
        wl_gae_seg_kernel<<<(N + 31) / 32, 32 * S, 0, (cudaStream_t)stream>>>(d_rewards, d_values, d_last_values, d_dones, d_time_outs, gamma,
                                                                              lam, d_returns, d_advantages, T, N);
    else
        wl_gae_kernel<<<(N + 127) / 128, 128, 0, (cudaStream_t)stream>>>(d_rewards, d_values, d_last_values, d_dones, d_time_outs, gamma,
                                                                         lam, d_returns, d_advantages, T, N);
    return cuda_check(cudaGetLastError(), "wl_gae_kernel");
}

// workspace of wl_episode_stats: [(return, length) per (t, env)][done word per (t, 32 envs)], 256-byte aligned
static size_t episode_words_off(int32_t T, int32_t N) { return align256(sizeof(float2) * (size_t)T * N); }
size_t wl_episode_stats_workspace_bytes(int32_t T, int32_t N) {
    if (T < 1 || T > WL_EP_MAX_T || N < 1) { fail(WL_EINVAL, "wl_episode_stats_workspace_bytes: T must be in 1..4096 and N >= 1"); return 0; }
    return episode_words_off(T, N) + sizeof(uint32_t) * (size_t)T * ((N + 31) / 32);
}

int wl_episode_stats(const float* d_rewards, const uint8_t* d_terminated, const uint8_t* d_truncated, int32_t T, int32_t N,
                     float* d_cur_return, float* d_cur_length, wl_episode_stats_state* d_stats, void* d_workspace,
                     size_t workspace_bytes, void* stream) {
    if (!d_rewards || !d_terminated || !d_truncated || !d_cur_return || !d_cur_length || !d_stats || !d_workspace)
        return fail(WL_EINVAL, "wl_episode_stats: null argument");
    const size_t need = wl_episode_stats_workspace_bytes(T, N);
    if (need == 0) return fail(WL_EINVAL, "wl_episode_stats: T must be in 1..4096 and N >= 1");
    if (workspace_bytes < need) return fail(WL_EINVAL, "wl_episode_stats: workspace smaller than wl_episode_stats_workspace_bytes(T, N)");
    if (((uintptr_t)d_stats & 7u) != 0 || ((uintptr_t)d_workspace & 255u) != 0)
        return fail(WL_EINVAL, "wl_episode_stats: d_stats must be 8-byte and d_workspace 256-byte aligned");
    cudaStream_t cs = (cudaStream_t)stream;
    float2* ep = reinterpret_cast<float2*>(d_workspace);
    uint32_t* words = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(d_workspace) + episode_words_off(T, N));
    wl_episode_walk_kernel<<<(N + WL_EP_WALK_THREADS - 1) / WL_EP_WALK_THREADS, WL_EP_WALK_THREADS, 0, cs>>>(
        d_rewards, d_terminated, d_truncated, T, N, d_cur_return, d_cur_length, ep, words);
    if (int rc = cuda_check(cudaGetLastError(), "wl_episode_walk_kernel")) return rc;
    wl_episode_ring_kernel<<<1, WL_EP_RING_THREADS, 0, cs>>>(ep, words, T, N, d_stats);
    return cuda_check(cudaGetLastError(), "wl_episode_ring_kernel");
}

int wl_dp_adam_step(float* d_param, float* d_m, float* d_v, int32_t n_ranks, const float* const* d_grads, float lr, double beta1,
                    double beta2, float eps, float weight_decay, int32_t step, int32_t n, void* stream) {
    if (!d_param || !d_m || !d_v || !d_grads || n_ranks < 1 || n_ranks > WL_MAX_PEERS || n < 1 || step < 1)
        return fail(WL_EINVAL, "wl_dp_adam_step: bad argument");
    GradPeers gp; memset(&gp, 0, sizeof gp);
    gp.n = n_ranks;
    for (int r = 0; r < n_ranks; ++r) { if (!d_grads[r]) return fail(WL_EINVAL, "wl_dp_adam_step: null gradient pointer"); gp.g[r] = d_grads[r]; }
    // torch forms 1 - beta^t and 1 - beta from the Python (double) betas, as wl_ppo_step_kernel does; in fp32, 0.999f exceeds
    // 0.999 by 1.3e-8 and 1 - 0.999f^t is ~1.3e-5 off for the first thousand steps
    const float bc1 = (float)(1.0 - pow(beta1, (double)step)), bc2 = (float)(1.0 - pow(beta2, (double)step));
    wl_dp_adam_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(d_param, d_m, d_v, gp, lr, (float)beta1, (float)(1.0 - beta1),
                                                                         (float)beta2, (float)(1.0 - beta2), eps, weight_decay, bc1, bc2, n);
    return cuda_check(cudaGetLastError(), "wl_dp_adam_kernel");
}

// dynamic shared memory of wl_ppo_grad_kernel: the blob (grows with obs_dim), W2 transposed, the tile's rows
static size_t ppo_grad_smem(int obs_dim) {
    int32_t off[13];
    return sizeof(float) * ((size_t)policy_offsets(obs_dim, off) + 2 * WL_HID * WL_HID + WL_HID + WL_PPO_TILE * WL_PPO_XS +
                            4 * WL_PPO_TILE * WL_PPO_HS + WL_PPO_TILE * WL_PPO_SD);
}

// workspace of wl_ppo_update: [reduced row][fp64 block sums of squares][one gradient row per CTA], each 256-byte aligned
struct PpoWorkspace { int blob_floats, rowlen, ctas, norm_parts; size_t norm_off, rows_off, bytes; };
// (wl_ppo_update_wide's: wl_ppo_update's, then H1 and dZ1 of a mini-batch)
struct PpoWideWorkspace { PpoWorkspace w; size_t h1_off, dz_off, bytes; };
static void ppo_rows_layout(int32_t obs_dim, int32_t batch, int32_t num_mini_batches, int sms, PpoWorkspace& w, int32_t critic_obs_dim = 0) {
    int32_t off[13];
    w.blob_floats = policy_offsets(obs_dim, off, critic_obs_dim);
    w.rowlen = (w.blob_floats + WL_PPO_STATS + 3) & ~3;
    const int tiles = (batch / num_mini_batches + WL_PPO_TILE - 1) / WL_PPO_TILE;
    w.ctas = tiles < sms ? tiles : sms;
    w.norm_parts = (w.rowlen + 255) / 256;
    w.norm_off = align256(sizeof(float) * w.rowlen);
    w.rows_off = align256(w.norm_off + sizeof(double) * w.norm_parts);
    w.bytes = w.rows_off + sizeof(float) * (size_t)w.rowlen * w.ctas;
}
// the network an update trains: wl_ppo_update's ELU network, wl_ppo_update_wide's ReLU network, wl_ppo_update_asym's ELU
// network with a critic row of its own, wl_ppo_update_wide_asym's ReLU network with one
enum PpoNet { PPO_NARROW, PPO_WIDE, PPO_ASYM, PPO_WIDE_ASYM };
static size_t ppo_grad_asym_smem(int obs_dim, int critic_obs_dim);
static int wide_attributes(int dev, const char* fn);
static int wide_asym_attributes(int dev, const char* fn);
// The shape checks and the workspace layout of an update of `net` (critic_obs_dim: PPO_ASYM only).  The gradient kernels'
// shared-memory limits are per-device attributes: raised once to what the widest network needs, so updates of any obs_dim
// share them in one process.  The workspace query reaches here before the first update, so callers that query outside a
// graph capture (FusedPPO, PPOIteration.start) never set them inside one.
static int ppo_workspace(const char* fn, PpoNet net, int32_t obs_dim, int32_t critic_obs_dim, int32_t batch, int32_t num_mini_batches,
                         PpoWideWorkspace& x) {
    if (obs_dim < 1 || batch < 1 || num_mini_batches < 1) return fail(WL_EINVAL, std::string(fn) + ": obs_dim, batch and num_mini_batches must be >= 1");
    const bool wide = net == PPO_WIDE || net == PPO_WIDE_ASYM;
    if (wide && obs_dim > WL_WIDE_MAX_OBS) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim > 4096");
    if (!wide && obs_dim > 16) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim > 16 (the network wl_act_step runs)");
    if (net == PPO_ASYM && (critic_obs_dim < 1 || critic_obs_dim > WL_MAX_CRITIC_OBS))
        return fail(WL_EINVAL, std::string(fn) + ": critic_obs_dim must be in 1..32");
    if (net == PPO_WIDE_ASYM && (critic_obs_dim < 1 || critic_obs_dim > WL_WIDE_MAX_OBS))
        return fail(WL_EUNSUPPORTED, std::string(fn) + ": critic_obs_dim must be in 1..4096");
    if (batch % num_mini_batches != 0) return fail(WL_EINVAL, std::string(fn) + ": batch must be a multiple of num_mini_batches");
    int dev = 0, sms = 0;
    if (int rc = cuda_check(cudaGetDevice(&dev), fn)) return rc;
    if (int rc = cuda_check(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev), fn)) return rc;
    if (int rc = net == PPO_WIDE ? wide_attributes(dev, fn)
                 : net == PPO_WIDE_ASYM ? wide_asym_attributes(dev, fn)
                 : net == PPO_ASYM ? raise_smem<wl_ppo_grad_asym_kernel>(dev, ppo_grad_asym_smem(16, WL_MAX_CRITIC_OBS), fn)
                                   : raise_smem<wl_ppo_grad_kernel>(dev, ppo_grad_smem(16), fn))
        return rc;
    ppo_rows_layout(obs_dim, batch, num_mini_batches, sms, x.w, net == PPO_ASYM || net == PPO_WIDE_ASYM ? critic_obs_dim : 0);
    x.bytes = x.w.bytes;
    if (wide) {                 // then H1 and dZ1 of a mini-batch ([tiles * 32][128] fp32 each)
        const size_t hb = sizeof(float) * 2 * WL_HID * (size_t)WL_PPO_TILE * ((batch / num_mini_batches + WL_PPO_TILE - 1) / WL_PPO_TILE);
        x.h1_off = align256(x.w.bytes);
        x.dz_off = align256(x.h1_off + hb);
        x.bytes = x.dz_off + hb;
    }
    return WL_OK;
}

int32_t wl_ppo_state_floats(void) { return 10 + 2 * WL_PPO_MAX_UPDATES; }

size_t wl_ppo_workspace_bytes(int32_t obs_dim, int32_t batch, int32_t num_mini_batches) {
    PpoWideWorkspace x;
    return ppo_workspace("wl_ppo_workspace_bytes", PPO_NARROW, obs_dim, 0, batch, num_mini_batches, x) ? 0 : x.bytes;
}

// the host-side checks of one rank's arguments to a PPO update entry (fn names the entry in the message)
static int ppo_check_args(const char* fn, const wl_ppo_params* p, const wl_ppo_batch* b, const float* d_blob, const float* d_adam_m,
                          const float* d_adam_v, const float* d_state, const void* d_workspace) {
    if (!p || !b) return fail(WL_EINVAL, std::string(fn) + ": null params / batch");
    if (!b->obs || !b->actions || !b->values || !b->log_prob || !b->mean || !b->returns || !b->advantages || !b->perm)
        return fail(WL_EINVAL, std::string(fn) + ": null array in batch");
    if (!d_blob || !d_adam_m || !d_adam_v || !d_state || !d_workspace)
        return fail(WL_EINVAL, std::string(fn) + ": null d_blob / d_adam_m / d_adam_v / d_state / d_workspace");
    if (p->num_learning_epochs < 1) return fail(WL_EINVAL, std::string(fn) + ": num_learning_epochs must be >= 1");
    return WL_OK;
}

// the workspace layout of an update of `net` and the checks against it
static int ppo_check_layout(const char* fn, PpoNet net, int32_t critic_obs_dim, const wl_ppo_params* p, const wl_ppo_batch* b,
                            const float* d_blob, const float* d_adam_m, const float* d_adam_v, const void* d_workspace,
                            size_t workspace_bytes, PpoWideWorkspace& x) {
    if (int rc = ppo_workspace(fn, net, p->obs_dim, critic_obs_dim, p->batch, p->num_mini_batches, x)) return rc;
    if (((uintptr_t)d_blob & 15u) || ((uintptr_t)d_adam_m & 15u) || ((uintptr_t)d_adam_v & 15u))
        return fail(WL_EINVAL, std::string(fn) + ": d_blob / d_adam_m / d_adam_v must be 16-byte aligned");
    if (((uintptr_t)d_workspace & 255u) || ((uintptr_t)b->actions & 7u) || ((uintptr_t)b->mean & 7u))
        return fail(WL_EINVAL, std::string(fn) + ": d_workspace must be 256-byte aligned, actions / mean 8-byte aligned");
    static const char* const query[] = {"wl_ppo_workspace_bytes", "wl_ppo_wide_workspace_bytes", "wl_ppo_asym_workspace_bytes",
                                        "wl_ppo_wide_asym_workspace_bytes"};
    if (workspace_bytes < x.bytes)
        return fail(WL_EINVAL, std::string(fn) + ": workspace_bytes too small (" + query[net] + " gives " + std::to_string(x.bytes) + ")");
    return WL_OK;
}

static size_t ppo_grad_smem(int obs_dim);
static size_t ppo_wide_grad_smem();
static size_t ppo_wide_dw1_smem();
static size_t ppo_wide_dw1_asym_smem();

// The gradient phase of one mini-batch (a.row0): one gradient row per CTA in the workspace.  Narrow: wl_ppo_grad_kernel;
// wide: the gathered layer-1 forward, the layers 2-3 gradient kernel and the split-K dW1 -- with xc, the critic's layer 1
// over xc [batch, Dc] (the asymmetric forward and dW1 kernels; the layers 2-3 kernel is the same).
static void ppo_grad_phase(bool wide, const PpoWideWorkspace& x, const PolicyOffsets& po, const PolicyOffsets& pc, const PpoArgs& a,
                           const float* d_blob, const float* d_state, char* ws, cudaStream_t cs, const float* xc = nullptr, int Dc = 0) {
    const PpoWorkspace& w = x.w;
    float* rows = (float*)(ws + w.rows_off);
    if (!wide) {
        wl_ppo_grad_kernel<<<w.ctas, WL_PPO_THREADS, ppo_grad_smem(a.obs_dim), cs>>>(d_blob, w.blob_floats, po, a, d_state, rows, w.rowlen);
        return;
    }
    float* H1 = (float*)(ws + x.h1_off);
    float* dZ1 = (float*)(ws + x.dz_off);
    const int K = xc && Dc > a.obs_dim ? Dc : a.obs_dim;
    const dim3 dw1_grid((unsigned)((K + WL_DW1_K - 1) / WL_DW1_K), (unsigned)w.ctas);
    if (xc) wl_ppo_wide_fwd_asym_kernel<<<a.tiles, WL_WIDE_THREADS, sizeof(float) * 2 * WL_WIDE_STAGE_ASYM, cs>>>(d_blob, po, a, xc, Dc, H1);
    else wl_ppo_wide_fwd_kernel<<<a.tiles, WL_WIDE_THREADS, sizeof(float) * 2 * WL_WIDE_STAGE, cs>>>(d_blob, po, a, H1);
    wl_ppo_wide_grad_kernel<<<w.ctas, WL_PPO_THREADS, ppo_wide_grad_smem(), cs>>>(d_blob, w.blob_floats, po, pc, a, d_state, H1, dZ1,
                                                                                 rows, w.rowlen);
    if (xc) wl_ppo_wide_dw1_asym_kernel<<<dw1_grid, WL_WIDE_THREADS, ppo_wide_dw1_asym_smem(), cs>>>(po, a, dZ1, rows, w.rowlen, xc, Dc);
    else wl_ppo_wide_dw1_kernel<<<dw1_grid, WL_WIDE_THREADS, ppo_wide_dw1_smem(), cs>>>(po, a, dZ1, rows, w.rowlen);
}

// the per-mini-batch arguments of every update entry
static void ppo_launch_args(const wl_ppo_params* p, const wl_ppo_batch* b, PpoArgs& a, PpoStepArgs& sa) {
    const int B = p->batch / p->num_mini_batches;
    a.b = *b; a.obs_dim = p->obs_dim; a.B = B; a.tiles = (B + WL_PPO_TILE - 1) / WL_PPO_TILE;
    a.clip = p->clip_param; a.vcoef = p->value_loss_coef; a.inv_B = 1.0f / (float)B; a.clipped_value = p->use_clipped_value_loss != 0;
    sa = PpoStepArgs{p->max_grad_norm, p->desired_kl, a.inv_B, p->adaptive != 0, 0};
}

static int wide_compact_offsets(const PolicyOffsets& po, int blob_floats, PolicyOffsets& pc);

// wl_ppo_update (wide false), wl_ppo_update_wide and wl_ppo_update_wide_asym (xc: the critic's rows, Dc wide): rsl_rl's
// update, epochs x mini-batches of the gradient phase, the reduction and the Adam step
static int ppo_update(const char* fn, bool wide, const wl_ppo_params* p, const wl_ppo_batch* b, float* d_blob, float* d_adam_m,
                      float* d_adam_v, float* d_state, void* d_workspace, size_t workspace_bytes, void* stream,
                      const float* xc = nullptr, int Dc = 0) {
    if (int rc = ppo_check_args(fn, p, b, d_blob, d_adam_m, d_adam_v, d_state, d_workspace)) return rc;
    PpoWideWorkspace x;
    const PpoNet net = !wide ? PPO_NARROW : xc ? PPO_WIDE_ASYM : PPO_WIDE;
    if (int rc = ppo_check_layout(fn, net, Dc, p, b, d_blob, d_adam_m, d_adam_v, d_workspace, workspace_bytes, x))
        return rc;
    const PpoWorkspace& w = x.w;
    PolicyOffsets po, pc;
    policy_offsets(p->obs_dim, po.o, Dc);
    if (wide) wide_compact_offsets(po, w.blob_floats, pc);
    else pc = po;
    cudaStream_t cs = (cudaStream_t)stream;
    char* ws = (char*)d_workspace;
    float* red = (float*)ws;
    double* norm_part = (double*)(ws + w.norm_off);
    float* rows = (float*)(ws + w.rows_off);
    wl_ppo_begin_kernel<<<1, WL_PPO_FIN_THREADS, 0, cs>>>(b->advantages, p->batch, d_blob, po.o[12], d_state);
    if (int rc = cuda_check(cudaGetLastError(), "wl_ppo_begin_kernel")) return rc;
    PpoArgs a;
    PpoStepArgs sa;
    ppo_launch_args(p, b, a, sa);
    for (int e = 0; e < p->num_learning_epochs; ++e) {
        for (int i = 0; i < p->num_mini_batches; ++i) {
            a.row0 = (int64_t)i * a.B;
            sa.update_index = e * p->num_mini_batches + i;
            ppo_grad_phase(wide, x, po, pc, a, d_blob, d_state, ws, cs, xc, Dc);
            if (xc) {                                        // the asymmetric parameter lengths (ppo_is_param's critic_dim)
                wl_ppo_reduce_asym_kernel<<<w.norm_parts, 256, 0, cs>>>(rows, w.ctas, w.rowlen, w.blob_floats, po, p->obs_dim, Dc,
                                                                        d_blob, p->entropy_coef, red, norm_part);
                wl_ppo_step_asym_kernel<<<1, WL_PPO_FIN_THREADS, 0, cs>>>(d_blob, d_adam_m, d_adam_v, d_state, red, norm_part, w.norm_parts,
                                                                          w.blob_floats, po, p->obs_dim, Dc, sa);
            } else {
                wl_ppo_reduce_kernel<<<w.norm_parts, 256, 0, cs>>>(rows, w.ctas, w.rowlen, w.blob_floats, po, p->obs_dim, d_blob,
                                                                   p->entropy_coef, red, norm_part);
                wl_ppo_step_kernel<false><<<1, WL_PPO_FIN_THREADS, 0, cs>>>(d_blob, d_adam_m, d_adam_v, d_state, red, norm_part, w.norm_parts,
                                                                            w.blob_floats, po, p->obs_dim, sa, nullptr);
            }
            if (int rc = cuda_check(cudaGetLastError(), wide ? "wl_ppo_update_wide kernels" : "wl_ppo_grad_kernel / wl_ppo_reduce_kernel / wl_ppo_step_kernel"))
                return rc;
        }
    }
    return WL_OK;
}

int wl_ppo_update(const wl_ppo_params* p, const wl_ppo_batch* b, float* d_blob, float* d_adam_m, float* d_adam_v, float* d_state,
                  void* d_workspace, size_t workspace_bytes, void* stream) {
    return ppo_update("wl_ppo_update", false, p, b, d_blob, d_adam_m, d_adam_v, d_state, d_workspace, workspace_bytes, stream);
}

// ---- the asymmetric update (DESIGN 6m): wl_ppo_update's loop over wl_ppo_grad_asym_kernel and the asymmetric blob layout ----
static size_t ppo_grad_asym_smem(int obs_dim, int critic_obs_dim) {
    int32_t off[13];
    return sizeof(float) * ((size_t)policy_offsets(obs_dim, off, critic_obs_dim) + 2 * WL_HID * WL_HID + WL_HID + 2 * WL_PPO_TILE * WL_PPO_XA +
                            4 * WL_PPO_TILE * WL_PPO_HS + WL_PPO_TILE * WL_PPO_SD);
}
size_t wl_ppo_asym_workspace_bytes(int32_t obs_dim, int32_t critic_obs_dim, int32_t batch, int32_t num_mini_batches) {
    PpoWideWorkspace x;
    return ppo_workspace("wl_ppo_asym_workspace_bytes", PPO_ASYM, obs_dim, critic_obs_dim, batch, num_mini_batches, x) ? 0 : x.bytes;
}

int wl_ppo_update_asym(const wl_ppo_params* p, const wl_ppo_batch* b, const float* d_critic_obs, int32_t critic_obs_dim, float* d_blob,
                       float* d_adam_m, float* d_adam_v, float* d_state, void* d_workspace, size_t workspace_bytes, void* stream) {
    const char* fn = "wl_ppo_update_asym";
    if (int rc = ppo_check_args(fn, p, b, d_blob, d_adam_m, d_adam_v, d_state, d_workspace)) return rc;
    if (!d_critic_obs || ((uintptr_t)d_critic_obs & 3u)) return fail(WL_EINVAL, std::string(fn) + ": d_critic_obs is null or not 4-byte aligned");
    PpoWideWorkspace x;
    if (int rc = ppo_check_layout(fn, PPO_ASYM, critic_obs_dim, p, b, d_blob, d_adam_m, d_adam_v, d_workspace, workspace_bytes, x)) return rc;
    const PpoWorkspace& w = x.w;
    PolicyOffsets po;
    policy_offsets(p->obs_dim, po.o, critic_obs_dim);
    cudaStream_t cs = (cudaStream_t)stream;
    char* ws = (char*)d_workspace;
    float* red = (float*)ws;
    double* norm_part = (double*)(ws + w.norm_off);
    float* rows = (float*)(ws + w.rows_off);
    const size_t smem = ppo_grad_asym_smem(p->obs_dim, critic_obs_dim);
    wl_ppo_begin_kernel<<<1, WL_PPO_FIN_THREADS, 0, cs>>>(b->advantages, p->batch, d_blob, po.o[12], d_state);
    if (int rc = cuda_check(cudaGetLastError(), "wl_ppo_begin_kernel")) return rc;
    PpoArgs a;
    PpoStepArgs sa;
    ppo_launch_args(p, b, a, sa);
    for (int e = 0; e < p->num_learning_epochs; ++e) {
        for (int i = 0; i < p->num_mini_batches; ++i) {
            a.row0 = (int64_t)i * a.B;
            sa.update_index = e * p->num_mini_batches + i;
            wl_ppo_grad_asym_kernel<<<w.ctas, WL_PPO_THREADS, smem, cs>>>(d_blob, w.blob_floats, po, a, d_critic_obs, critic_obs_dim, d_state,
                                                                          rows, w.rowlen);
            wl_ppo_reduce_asym_kernel<<<w.norm_parts, 256, 0, cs>>>(rows, w.ctas, w.rowlen, w.blob_floats, po, p->obs_dim, critic_obs_dim,
                                                                    d_blob, p->entropy_coef, red, norm_part);
            wl_ppo_step_asym_kernel<<<1, WL_PPO_FIN_THREADS, 0, cs>>>(d_blob, d_adam_m, d_adam_v, d_state, red, norm_part, w.norm_parts,
                                                                      w.blob_floats, po, p->obs_dim, critic_obs_dim, sa);
            if (int rc = cuda_check(cudaGetLastError(), "wl_ppo_grad_asym_kernel / wl_ppo_reduce_asym_kernel / wl_ppo_step_asym_kernel")) return rc;
        }
    }
    return WL_OK;
}

// ---- the wide (ReLU) actor-critic: wl_policy_act and wl_ppo_update_wide (DESIGN 6g) ----------------------------------
// offsets inside the copy of the blob without its W1t blocks ([o1, o6) | [o7, end)) the wide kernels keep in shared
// memory; returns its float count (the same for every obs_dim)
static int wide_compact_offsets(const PolicyOffsets& po, int blob_floats, PolicyOffsets& pc) {
    const int na = po.o[6] - po.o[1];
    for (int k = 0; k < 13; ++k) pc.o[k] = (k == 0 || k == 6) ? -1 : (k < 6 ? po.o[k] - po.o[1] : na + po.o[k] - po.o[7]);
    return na + blob_floats - po.o[7];
}
static size_t wide_compact_bytes() {
    PolicyOffsets po, pc;
    return sizeof(float) * (size_t)wide_compact_offsets(po, policy_offsets(1, po.o), pc);
}
static size_t policy_act_smem() { return sizeof(float) * (2 * WL_WIDE_STAGE + WL_WIDE_ROWS * WL_PPO_HS) + wide_compact_bytes(); }
static size_t ppo_wide_grad_smem() {
    return wide_compact_bytes() + sizeof(float) * (2 * WL_HID * WL_HID + WL_HID + 4 * WL_PPO_TILE * WL_PPO_HS + WL_PPO_TILE * WL_PPO_SD);
}
static size_t ppo_wide_dw1_smem() { return sizeof(float) * 2 * WL_PPO_TILE * (WL_DW1_K + 2 * WL_HID); }
static size_t policy_act_asym_smem() { return sizeof(float) * (2 * WL_WIDE_STAGE_ASYM + WL_WIDE_ROWS * WL_PPO_HS) + wide_compact_bytes(); }
static size_t ppo_wide_dw1_asym_smem() { return sizeof(float) * 2 * WL_PPO_TILE * (2 * WL_DW1_K + 2 * WL_HID); }

// the dynamic shared-memory limits of the wide kernels, raised together (the sizes do not depend on obs_dim)
static int wide_attributes(int dev, const char* fn) {
    if (int rc = raise_smem<wl_policy_act_kernel>(dev, policy_act_smem(), fn)) return rc;
    if (int rc = raise_smem<wl_ppo_wide_grad_kernel>(dev, ppo_wide_grad_smem(), fn)) return rc;
    return raise_smem<wl_ppo_wide_dw1_kernel>(dev, ppo_wide_dw1_smem(), fn);
}
// the same for the asymmetric kernels (and the wide grad kernel they share)
static int wide_asym_attributes(int dev, const char* fn) {
    if (int rc = wide_attributes(dev, fn)) return rc;
    if (int rc = raise_smem<wl_policy_act_wide_asym_kernel>(dev, policy_act_asym_smem(), fn)) return rc;
    if (int rc = raise_smem<wl_ppo_wide_fwd_asym_kernel>(dev, sizeof(float) * 2 * WL_WIDE_STAGE_ASYM, fn)) return rc;
    return raise_smem<wl_ppo_wide_dw1_asym_kernel>(dev, ppo_wide_dw1_asym_smem(), fn);
}

int wl_policy_act(wl_sim* sim, const float* d_obs_in, const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream) {
    if (!sim || !d_obs_in || !d_policy_blob || !out.actions || !out.mean || !out.log_prob || !out.value)
        return fail(WL_EINVAL, "wl_policy_act: null argument");
    const int D = policy_in_dim(sim), n = sim->cfg.num_envs;
    if (D < 1 || D > WL_WIDE_MAX_OBS) return fail(WL_EUNSUPPORTED, "wl_policy_act: obs_dim must be in 1..4096");
    if (((uintptr_t)d_policy_blob & 15u) || ((uintptr_t)out.actions & 7u) || ((uintptr_t)out.mean & 7u))
        return fail(WL_EINVAL, "wl_policy_act: policy blob must be 16-byte aligned, actions/mean 8-byte aligned");
    ensure_device(sim);
    if (int rc = wide_attributes(sim->device, "wl_policy_act")) return rc;
    PolicyOffsets po, pc;
    const int blob_floats = policy_offsets(D, po.o);
    wide_compact_offsets(po, blob_floats, pc);
    wl_policy_act_kernel<<<(n + WL_WIDE_ROWS - 1) / WL_WIDE_ROWS, WL_WIDE_THREADS, policy_act_smem(), (cudaStream_t)stream>>>(
        d_obs_in, n, D, d_policy_blob, blob_floats, po, pc, out, sim->globals, sim->cfg.seed, sim->cfg.env_id_offset, (uint32_t)step_counter);
    return launched(sim, "wl_policy_act_kernel");
}

int wl_policy_act_wide_asym(wl_sim* sim, const float* d_obs_in, const float* d_critic_obs_in, int32_t critic_obs_dim,
                            const float* d_policy_blob, wl_policy_out out, int64_t step_counter, void* stream) {
    const char* fn = "wl_policy_act_wide_asym";
    if (!sim || !d_obs_in || !d_critic_obs_in || !d_policy_blob || !out.actions || !out.mean || !out.log_prob || !out.value)
        return fail(WL_EINVAL, std::string(fn) + ": null argument");
    const int D = policy_in_dim(sim), n = sim->cfg.num_envs;
    if (D < 1 || D > WL_WIDE_MAX_OBS) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim must be in 1..4096");
    if (critic_obs_dim < 1 || critic_obs_dim > WL_WIDE_MAX_OBS) return fail(WL_EINVAL, std::string(fn) + ": critic_obs_dim must be in 1..4096");
    if (((uintptr_t)d_policy_blob & 15u) || ((uintptr_t)out.actions & 7u) || ((uintptr_t)out.mean & 7u))
        return fail(WL_EINVAL, std::string(fn) + ": policy blob must be 16-byte aligned, actions/mean 8-byte aligned");
    if (((uintptr_t)d_obs_in & 3u) || ((uintptr_t)d_critic_obs_in & 3u))
        return fail(WL_EINVAL, std::string(fn) + ": obs_in / critic_obs_in must be 4-byte aligned");
    ensure_device(sim);
    if (int rc = wide_asym_attributes(sim->device, fn)) return rc;
    PolicyOffsets po, pc;
    const int blob_floats = policy_offsets(D, po.o, critic_obs_dim);
    wide_compact_offsets(po, blob_floats, pc);
    wl_policy_act_wide_asym_kernel<<<(n + WL_WIDE_ROWS - 1) / WL_WIDE_ROWS, WL_WIDE_THREADS, policy_act_asym_smem(), (cudaStream_t)stream>>>(
        d_obs_in, n, D, d_critic_obs_in, critic_obs_dim, d_policy_blob, blob_floats, po, pc, out, sim->globals, sim->cfg.seed,
        sim->cfg.env_id_offset, (uint32_t)step_counter);
    return launched(sim, "wl_policy_act_wide_asym_kernel");
}

int wl_actor_mean(const float* d_obs, int32_t n, int32_t obs_dim, const float* d_policy_blob, int32_t activation, float* d_mean,
                  void* stream) {
    if (!d_obs || !d_policy_blob || !d_mean) return fail(WL_EINVAL, "wl_actor_mean: null argument");
    if (n < 1) return fail(WL_EINVAL, "wl_actor_mean: n must be >= 1");
    if (activation != WL_ACTIVATION_ELU && activation != WL_ACTIVATION_RELU)
        return fail(WL_EINVAL, "wl_actor_mean: activation must be WL_ACTIVATION_ELU or WL_ACTIVATION_RELU");
    if (obs_dim < 1 || obs_dim > WL_WIDE_MAX_OBS) return fail(WL_EUNSUPPORTED, "wl_actor_mean: obs_dim must be in 1..4096");
    if (activation == WL_ACTIVATION_ELU && obs_dim > 16)
        return fail(WL_EUNSUPPORTED, "wl_actor_mean: the ELU network (wl_act_step's) takes obs_dim <= 16");
    if (((uintptr_t)d_policy_blob & 15u) || ((uintptr_t)d_mean & 7u) || ((uintptr_t)d_obs & 3u))
        return fail(WL_EINVAL, "wl_actor_mean: policy blob must be 16-byte aligned, mean 8-byte aligned, obs 4-byte aligned");
    // device guard: the launch goes to the device that holds the output
    cudaPointerAttributes pa;
    if (int rc = cuda_check(cudaPointerGetAttributes(&pa, d_mean), "wl_actor_mean")) return rc;
    if (pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged) return fail(WL_EINVAL, "wl_actor_mean: d_mean is not device memory");
    int cur = -1;
    if (cudaGetDevice(&cur) == cudaSuccess && cur != pa.device) cudaSetDevice(pa.device);
    const size_t smem = actor_mean_smem();
    if (int rc = raise_smem<wl_actor_mean_kernel<false>>(pa.device, smem, "wl_actor_mean")) return rc;
    if (int rc = raise_smem<wl_actor_mean_kernel<true>>(pa.device, smem, "wl_actor_mean")) return rc;
    PolicyOffsets po;
    policy_offsets(obs_dim, po.o);
    const int grid = (n + WL_AM_ROWS - 1) / WL_AM_ROWS;
    if (activation == WL_ACTIVATION_RELU)
        wl_actor_mean_kernel<true><<<grid, WL_AM_THREADS, smem, (cudaStream_t)stream>>>(d_obs, n, obs_dim, d_policy_blob, po, reinterpret_cast<float2*>(d_mean));
    else
        wl_actor_mean_kernel<false><<<grid, WL_AM_THREADS, smem, (cudaStream_t)stream>>>(d_obs, n, obs_dim, d_policy_blob, po, reinterpret_cast<float2*>(d_mean));
    return cuda_check(cudaGetLastError(), "wl_actor_mean_kernel");
}

size_t wl_ppo_wide_workspace_bytes(int32_t obs_dim, int32_t batch, int32_t num_mini_batches) {
    PpoWideWorkspace x;
    return ppo_workspace("wl_ppo_wide_workspace_bytes", PPO_WIDE, obs_dim, 0, batch, num_mini_batches, x) ? 0 : x.bytes;
}

int wl_ppo_update_wide(const wl_ppo_params* p, const wl_ppo_batch* b, float* d_blob, float* d_adam_m, float* d_adam_v, float* d_state,
                       void* d_workspace, size_t workspace_bytes, void* stream) {
    return ppo_update("wl_ppo_update_wide", true, p, b, d_blob, d_adam_m, d_adam_v, d_state, d_workspace, workspace_bytes, stream);
}

size_t wl_ppo_wide_asym_workspace_bytes(int32_t obs_dim, int32_t critic_obs_dim, int32_t batch, int32_t num_mini_batches) {
    PpoWideWorkspace x;
    return ppo_workspace("wl_ppo_wide_asym_workspace_bytes", PPO_WIDE_ASYM, obs_dim, critic_obs_dim, batch, num_mini_batches, x) ? 0 : x.bytes;
}

int wl_ppo_update_wide_asym(const wl_ppo_params* p, const wl_ppo_batch* b, const float* d_critic_obs, int32_t critic_obs_dim, float* d_blob,
                            float* d_adam_m, float* d_adam_v, float* d_state, void* d_workspace, size_t workspace_bytes, void* stream) {
    const char* fn = "wl_ppo_update_wide_asym";
    if (!d_critic_obs || ((uintptr_t)d_critic_obs & 3u)) return fail(WL_EINVAL, std::string(fn) + ": d_critic_obs is null or not 4-byte aligned");
    return ppo_update(fn, true, p, b, d_blob, d_adam_m, d_adam_v, d_state, d_workspace, workspace_bytes, stream, d_critic_obs, critic_obs_dim);
}

// ---- behaviour cloning: rsl_rl's Distillation.update() on the student actor (DESIGN 6t) ------------------------------
// workspace: [reduced row][fp64 block sums of squares][one gradient row per CTA][per-row squared errors of a chunk]
// [H1 of a chunk][dZ1 of a chunk] (the last two are the ReLU network's), each 256-byte aligned.  A row covers the actor,
// blob [0, o6).
struct DistillWorkspace { int rowlen, ctas, tiles, norm_parts; size_t norm_off, rows_off, sq_off, h1_off, dz_off, bytes; };
static size_t distill_grad_smem(bool relu) {
    int32_t off[13];
    policy_offsets(16, off);
    const int nact = relu ? off[6] - off[1] : off[6];
    return sizeof(float) * ((size_t)nact + WL_HID * WL_HID + WL_HID + (relu ? 0 : WL_DS_TILE * WL_DS_XS) + 4 * WL_DS_TILE * WL_DS_HS +
                            WL_DS_TILE * WL_DS_SD);
}
static size_t distill_dw1_smem() { return sizeof(float) * 2 * WL_DS_TILE * (WL_DW1_K + WL_HID); }
static size_t distill_fwd_smem() { return sizeof(float) * 2 * WL_DS_FWD_STAGE; }
static int distill_workspace(const char* fn, int32_t obs_dim, int32_t n_envs, int32_t gradient_length, DistillWorkspace& w) {
    if (obs_dim < 1 || obs_dim > WL_WIDE_MAX_OBS) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim must be in 1..4096");
    if (n_envs < 1 || gradient_length < 1) return fail(WL_EINVAL, std::string(fn) + ": n_envs and gradient_length must be >= 1");
    const int64_t B = (int64_t)n_envs * gradient_length;
    if (B > (int64_t)1 << 30) return fail(WL_EINVAL, std::string(fn) + ": n_envs * gradient_length must be <= 2^30");
    int dev = 0, sms = 0;
    if (int rc = cuda_check(cudaGetDevice(&dev), fn)) return rc;
    if (int rc = cuda_check(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev), fn)) return rc;
    if (int rc = raise_smem<wl_distill_grad_kernel<false>>(dev, distill_grad_smem(false), fn)) return rc;
    if (int rc = raise_smem<wl_distill_grad_kernel<true>>(dev, distill_grad_smem(true), fn)) return rc;
    if (int rc = raise_smem<wl_distill_fwd_kernel>(dev, distill_fwd_smem(), fn)) return rc;
    if (int rc = raise_smem<wl_distill_dw1_kernel>(dev, distill_dw1_smem(), fn)) return rc;
    int32_t off[13];
    policy_offsets(obs_dim, off);
    w.rowlen = off[6];
    w.tiles = (int)((B + WL_DS_TILE - 1) / WL_DS_TILE);
    w.ctas = w.tiles < sms ? w.tiles : sms;
    w.norm_parts = (w.rowlen + 255) / 256;
    w.norm_off = align256(sizeof(float) * w.rowlen);
    w.rows_off = align256(w.norm_off + sizeof(double) * w.norm_parts);
    w.sq_off = align256(w.rows_off + sizeof(float) * (size_t)w.rowlen * w.ctas);
    w.h1_off = align256(w.sq_off + sizeof(float) * (size_t)B);
    const size_t hb = sizeof(float) * WL_HID * (size_t)w.tiles * WL_DS_TILE;
    w.dz_off = align256(w.h1_off + hb);
    w.bytes = w.dz_off + hb;
    return WL_OK;
}

int32_t wl_distill_state_floats(int32_t T, int32_t num_learning_epochs) {
    if (T < 1 || num_learning_epochs < 1 || (int64_t)T * num_learning_epochs > (1 << 24)) {
        fail(WL_EINVAL, "wl_distill_state_floats: T and num_learning_epochs must be >= 1 (T * epochs <= 2^24)");
        return 0;
    }
    return WL_DS_STATE_HEAD + T * num_learning_epochs;
}

size_t wl_distill_workspace_bytes(int32_t obs_dim, int32_t n_envs, int32_t gradient_length) {
    DistillWorkspace w;
    return distill_workspace("wl_distill_workspace_bytes", obs_dim, n_envs, gradient_length, w) ? 0 : w.bytes;
}

int wl_distill_update(const wl_distill_params* p, const float* d_obs, const float* d_teacher_actions, int32_t T, int32_t N,
                      int32_t activation, float* d_blob, float* d_adam_m, float* d_adam_v, float* d_state, void* d_workspace,
                      size_t workspace_bytes, void* stream) {
    const char* fn = "wl_distill_update";
    if (!p) return fail(WL_EINVAL, std::string(fn) + ": null params");
    if (!d_obs || !d_teacher_actions || !d_blob || !d_adam_m || !d_adam_v || !d_state || !d_workspace)
        return fail(WL_EINVAL, std::string(fn) + ": null d_obs / d_teacher_actions / d_blob / d_adam_m / d_adam_v / d_state / d_workspace");
    if (activation != WL_ACTIVATION_ELU && activation != WL_ACTIVATION_RELU)
        return fail(WL_EINVAL, std::string(fn) + ": activation must be WL_ACTIVATION_ELU or WL_ACTIVATION_RELU");
    const int D = p->obs_dim;
    if (D < 1 || D > WL_WIDE_MAX_OBS) return fail(WL_EUNSUPPORTED, std::string(fn) + ": obs_dim must be in 1..4096");
    if (activation == WL_ACTIVATION_ELU && D > 16)
        return fail(WL_EUNSUPPORTED, std::string(fn) + ": the ELU network (wl_act_step's) takes obs_dim <= 16");
    if (p->num_learning_epochs < 1) return fail(WL_EINVAL, std::string(fn) + ": num_learning_epochs must be >= 1");
    if (p->gradient_length < 1) return fail(WL_EINVAL, std::string(fn) + ": gradient_length must be >= 1");
    if (T < 1 || N < 1) return fail(WL_EINVAL, std::string(fn) + ": T and N must be >= 1");
    if (T < p->gradient_length) return fail(WL_EINVAL, std::string(fn) + ": T must be >= gradient_length (no step would cover a chunk)");
    if (wl_distill_state_floats(T, p->num_learning_epochs) == 0) return fail(WL_EINVAL, std::string(fn) + ": T * num_learning_epochs > 2^24");
    if (((uintptr_t)d_blob & 15u) || ((uintptr_t)d_adam_m & 15u) || ((uintptr_t)d_adam_v & 15u))
        return fail(WL_EINVAL, std::string(fn) + ": d_blob / d_adam_m / d_adam_v must be 16-byte aligned");
    if (((uintptr_t)d_workspace & 255u) || ((uintptr_t)d_teacher_actions & 7u) || ((uintptr_t)d_obs & 3u) || ((uintptr_t)d_state & 3u))
        return fail(WL_EINVAL, std::string(fn) + ": d_workspace must be 256-byte aligned, d_teacher_actions 8-byte, d_obs / d_state 4-byte");
    DistillWorkspace w;
    if (int rc = distill_workspace(fn, D, N, p->gradient_length, w)) return rc;
    if (workspace_bytes < w.bytes)
        return fail(WL_EINVAL, std::string(fn) + ": workspace_bytes too small (wl_distill_workspace_bytes gives " + std::to_string(w.bytes) + ")");
    const bool relu = activation == WL_ACTIVATION_RELU;
    PolicyOffsets po;
    policy_offsets(D, po.o);
    cudaStream_t cs = (cudaStream_t)stream;
    char* ws = (char*)d_workspace;
    float* red = (float*)ws;
    double* norm_part = (double*)(ws + w.norm_off);
    float* rows = (float*)(ws + w.rows_off);
    float* H1 = (float*)(ws + w.h1_off);
    float* dZ1 = (float*)(ws + w.dz_off);
    DistillArgs a;
    a.obs = d_obs; a.target = d_teacher_actions; a.sqerr = (float*)(ws + w.sq_off);
    a.D = D; a.N = N; a.T = T; a.inv_N = (float)(1.0 / N);
    // rsl_rl counts the stored steps across epochs: Adam steps after every gradient_length-th step of the E * T, and the
    // steps after the last one are evaluated (their losses are logged) but not stepped
    const int total = T * p->num_learning_epochs, G = p->gradient_length;
    int n_steps = 0;
    for (int k0 = 0; k0 < total; k0 += G) {
        const int g = total - k0 < G ? total - k0 : G;
        const bool step = g == G;
        a.step0 = k0 % T; a.B = g * N; a.tiles = (a.B + WL_DS_TILE - 1) / WL_DS_TILE;
        const int ctas = a.tiles < w.ctas ? a.tiles : w.ctas;
        if (relu) {
            wl_distill_fwd_kernel<<<2 * a.tiles, WL_DS_FWD_THREADS, distill_fwd_smem(), cs>>>(d_blob, po, a, H1);
            wl_distill_grad_kernel<true><<<ctas, WL_DS_THREADS, distill_grad_smem(true), cs>>>(d_blob, po, a, H1, dZ1, rows, w.rowlen);
            if (step) {
                const dim3 grid((unsigned)((D + WL_DW1_K - 1) / WL_DW1_K), (unsigned)ctas);
                wl_distill_dw1_kernel<<<grid, WL_DS_THREADS, distill_dw1_smem(), cs>>>(po, a, dZ1, rows, w.rowlen);
            }
        } else {
            wl_distill_grad_kernel<false><<<ctas, WL_DS_THREADS, distill_grad_smem(false), cs>>>(d_blob, po, a, nullptr, nullptr, rows, w.rowlen);
        }
        wl_distill_loss_kernel<<<g, 256, 0, cs>>>(a.sqerr, N, k0, d_state);
        if (step) {
            wl_distill_reduce_kernel<<<w.norm_parts, 256, 0, cs>>>(rows, ctas, w.rowlen, po, D, red, norm_part);
            wl_distill_step_kernel<<<1, WL_DS_FIN_THREADS, 0, cs>>>(d_blob, d_adam_m, d_adam_v, d_state, red, norm_part, w.norm_parts, po, D,
                                                                   p->max_grad_norm);
            ++n_steps;
        }
        if (int rc = cuda_check(cudaGetLastError(), "wl_distill_update kernels")) return rc;
    }
    wl_distill_finish_kernel<<<1, 1, 0, cs>>>(d_state, total, n_steps);
    return cuda_check(cudaGetLastError(), "wl_distill_finish_kernel");
}

// ---- the data-parallel update (DESIGN 6j) ---------------------------------------------------------------------------
static size_t ppo_dp_slot_bytes(int rowlen) { return align256(sizeof(float) * (size_t)rowlen); }

size_t wl_ppo_dp_exchange_bytes(int32_t obs_dim) {
    if (obs_dim < 1 || obs_dim > WL_WIDE_MAX_OBS) { fail(WL_EINVAL, "wl_ppo_dp_exchange_bytes: obs_dim must be in 1..4096"); return 0; }
    int32_t off[13];
    const int rowlen = (policy_offsets(obs_dim, off) + WL_PPO_STATS + 3) & ~3;
    return WL_PPO_DP_HEADER + 2 * ppo_dp_slot_bytes(rowlen);
}

int wl_ppo_update_dp(const wl_ppo_params* p, int32_t activation, int32_t n_ranks, void* const* d_exchange, int32_t n_local,
                     const int32_t* local_ranks, const wl_ppo_batch* batches, float* const* d_blob, float* const* d_adam_m,
                     float* const* d_adam_v, float* const* d_state, void* const* d_workspace, size_t workspace_bytes, void* stream) {
    static const char* fn = "wl_ppo_update_dp";
    if (!p) return fail(WL_EINVAL, "wl_ppo_update_dp: null params");
    if (activation != WL_ACTIVATION_ELU && activation != WL_ACTIVATION_RELU)
        return fail(WL_EINVAL, "wl_ppo_update_dp: activation must be WL_ACTIVATION_ELU or WL_ACTIVATION_RELU");
    if (n_ranks < 1 || n_ranks > WL_MAX_PEERS) return fail(WL_EINVAL, "wl_ppo_update_dp: n_ranks must be in 1..8 (WL_MAX_PEERS)");
    if (!d_exchange) return fail(WL_EINVAL, "wl_ppo_update_dp: null d_exchange");
    PpoExchange ex; memset(&ex, 0, sizeof ex);
    ex.n = n_ranks;
    for (int r = 0; r < n_ranks; ++r) {
        if (!d_exchange[r] || ((uintptr_t)d_exchange[r] & 255u))
            return fail(WL_EINVAL, "wl_ppo_update_dp: exchange buffer " + std::to_string(r) + " is null or not 256-byte aligned");
        ex.buf[r] = (const char*)d_exchange[r];
    }
    if (n_local < 1 || n_local > n_ranks || !local_ranks) return fail(WL_EINVAL, "wl_ppo_update_dp: n_local must be in 1..n_ranks, local_ranks non-null");
    bool seen[WL_MAX_PEERS] = {false};
    for (int l = 0; l < n_local; ++l) {
        const int r = local_ranks[l];
        if (r < 0 || r >= n_ranks) return fail(WL_EINVAL, "wl_ppo_update_dp: local rank index " + std::to_string(r) + " out of 0..n_ranks-1");
        if (seen[r]) return fail(WL_EINVAL, "wl_ppo_update_dp: local rank " + std::to_string(r) + " given twice");
        seen[r] = true;
    }
    if (!batches || !d_blob || !d_adam_m || !d_adam_v || !d_state || !d_workspace)
        return fail(WL_EINVAL, "wl_ppo_update_dp: null per-rank array");
    for (int l = 0; l < n_local; ++l)
        if (int rc = ppo_check_args(fn, p, &batches[l], d_blob[l], d_adam_m[l], d_adam_v[l], d_state[l], d_workspace[l])) return rc;
    if (activation == WL_ACTIVATION_ELU && p->obs_dim > 16)
        return fail(WL_EUNSUPPORTED, "wl_ppo_update_dp: obs_dim > 16 (the network wl_act_step runs)");
    // every local rank's exchange buffer on one device: the call runs them in one stream
    int dev0 = -1;
    for (int l = 0; l < n_local; ++l) {
        cudaPointerAttributes pa;
        if (cudaPointerGetAttributes(&pa, d_exchange[local_ranks[l]]) != cudaSuccess || pa.type != cudaMemoryTypeDevice) {
            cudaGetLastError();
            return fail(WL_EINVAL, "wl_ppo_update_dp: local exchange buffer " + std::to_string(local_ranks[l]) + " is not device memory");
        }
        if (l == 0) dev0 = pa.device;
        else if (pa.device != dev0) return fail(WL_EINVAL, "wl_ppo_update_dp: local ranks' exchange buffers are on different devices");
    }
    const bool wide = activation == WL_ACTIVATION_RELU;
    PpoWideWorkspace x;
    for (int l = 0; l < n_local; ++l)
        if (int rc = ppo_check_layout(fn, wide ? PPO_WIDE : PPO_NARROW, 0, p, &batches[l], d_blob[l], d_adam_m[l], d_adam_v[l], d_workspace[l], workspace_bytes, x)) return rc;
    const PpoWorkspace& w = x.w;
    PolicyOffsets po, pc;
    policy_offsets(p->obs_dim, po.o);
    if (wide) wide_compact_offsets(po, w.blob_floats, pc);
    else pc = po;
    cudaStream_t cs = (cudaStream_t)stream;
    const size_t slot = ppo_dp_slot_bytes(w.rowlen);
    for (int l = 0; l < n_local; ++l)
        wl_ppo_begin_kernel<<<1, WL_PPO_FIN_THREADS, 0, cs>>>(batches[l].advantages, p->batch, d_blob[l], po.o[12], d_state[l]);
    if (int rc = cuda_check(cudaGetLastError(), "wl_ppo_begin_kernel")) return rc;
    PpoArgs a;
    PpoStepArgs sa;
    ppo_launch_args(p, &batches[0], a, sa);
    const int K = p->num_learning_epochs * p->num_mini_batches;
    for (int k = 0; k < K; ++k) {
        const size_t slot_off = WL_PPO_DP_HEADER + (size_t)(k & 1) * slot;
        a.row0 = (int64_t)(k % p->num_mini_batches) * a.B;
        sa.update_index = k;
        // every local rank publishes before any waits: in the one-process form the waits never spin
        for (int l = 0; l < n_local; ++l) {
            char* ws = (char*)d_workspace[l];
            char* own = (char*)d_exchange[local_ranks[l]];
            a.b = batches[l];
            ppo_grad_phase(wide, x, po, pc, a, d_blob[l], d_state[l], ws, cs);
            wl_ppo_reduce_kernel<<<w.norm_parts, 256, 0, cs>>>((const float*)(ws + w.rows_off), w.ctas, w.rowlen, w.blob_floats, po,
                                                               p->obs_dim, d_blob[l], p->entropy_coef, (float*)(own + slot_off),
                                                               (double*)(ws + w.norm_off));
            wl_ppo_dp_publish_kernel<<<1, 1, 0, cs>>>((uint32_t*)own);
        }
        for (int l = 0; l < n_local; ++l) {
            char* ws = (char*)d_workspace[l];
            uint32_t* own = (uint32_t*)d_exchange[local_ranks[l]];
            wl_ppo_dp_reduce_kernel<<<w.norm_parts, 256, 0, cs>>>(ex, own, slot_off, w.rowlen, w.blob_floats, po, p->obs_dim, a.inv_B,
                                                                  (float*)ws, (double*)(ws + w.norm_off));
            wl_ppo_step_kernel<true><<<1, WL_PPO_FIN_THREADS, 0, cs>>>(d_blob[l], d_adam_m[l], d_adam_v[l], d_state[l], (const float*)ws,
                                                                       (const double*)(ws + w.norm_off), w.norm_parts, w.blob_floats, po,
                                                                       p->obs_dim, sa, own + 1);
        }
        if (int rc = cuda_check(cudaGetLastError(), "wl_ppo_update_dp kernels")) return rc;
    }
    if (K & 1) {       // the no-row round: the next call starts on slot 0 again (see wl_ppo.cuh)
        for (int l = 0; l < n_local; ++l) wl_ppo_dp_publish_kernel<<<1, 1, 0, cs>>>((uint32_t*)d_exchange[local_ranks[l]]);
        for (int l = 0; l < n_local; ++l) wl_ppo_dp_wait_kernel<<<1, 1, 0, cs>>>(ex, (uint32_t*)d_exchange[local_ranks[l]]);
        if (int rc = cuda_check(cudaGetLastError(), "wl_ppo_dp_wait_kernel")) return rc;
    }
    return WL_OK;
}

int wl_test_detmath(int32_t op, const float* d_in, const float* d_in2, float* d_out, int32_t n, void* stream) {
    if (n <= 0) return WL_OK;
    wl_detmath_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(op, d_in, d_in2 ? d_in2 : d_in, d_out, n);
    return cuda_check(cudaGetLastError(), "wl_detmath_kernel");
}
int wl_graph_upload(void* graph_exec, void* stream) {
    if (!graph_exec) return fail(WL_EINVAL, "wl_graph_upload: null graph");
    return cuda_check(cudaGraphUpload((cudaGraphExec_t)graph_exec, (cudaStream_t)stream), "cudaGraphUpload");
}
int wl_test_null(int32_t grid, int32_t block, void* stream) {
    wl_null_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(nullptr);
    return cuda_check(cudaGetLastError(), "wl_null_kernel");
}
int wl_test_null_cfg(wl_sim* sim, int32_t grid, int32_t block, void* stream) {      /* same, carrying the 1.5 KB wl_config parameter */
    if (!sim) return fail(WL_EINVAL, "wl_test_null_cfg: null handle");
    wl_null_cfg_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(sim->cfg, nullptr);
    return cuda_check(cudaGetLastError(), "wl_null_cfg_kernel");
}
int wl_test_philox(uint64_t seed, uint32_t c0_base, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t* d_out, int32_t n,
                   void* stream) {
    if (n <= 0) return WL_OK;
    wl_philox_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(seed, c0_base, c1, c2, c3, reinterpret_cast<uint4*>(d_out), n);
    return cuda_check(cudaGetLastError(), "wl_philox_kernel");
}
int wl_test_device_terms(wl_sim* sim, const float* d_state, const uint8_t* d_done, float* d_rew, float* d_term_log,
                         int64_t step_counter, void* stream) {
    if (!sim || !d_state || !d_done || !d_rew) return fail(WL_EINVAL, "wl_test_device_terms: null argument");
    if ((uintptr_t)d_state & 15u) return fail(WL_EINVAL, "wl_test_device_terms: state must be 16-byte aligned");
    if (step_counter < 0) return fail(WL_EINVAL, "wl_test_device_terms: takes a host step counter");
    DevTerms* dt = sim->dterms;
    if (!dt) return fail(WL_EINVAL, "wl_test_device_terms: the handle has no device terms");
    ensure_device(sim);
    cudaStream_t cs = (cudaStream_t)stream;
    const int n = sim->cfg.num_envs, ctas = (n + WL_TERMS_BS - 1) / WL_TERMS_BS;
    wl_terms_kernel<<<ctas, WL_TERMS_BS, 0, cs>>>(dt->tt, sim->cfg, reinterpret_cast<const float4*>(d_state), sim->globals, sim->hf,
                                                  (uint32_t)step_counter, d_rew, d_done, dt->b, d_term_log != nullptr);
    if (int rc = launched(sim, "wl_terms_kernel")) return rc;
    if (d_term_log) {
        wl_terms_log_kernel<<<1, 9 * 32, 0, cs>>>(dt->tt, sim->cfg, dt->b.part, ctas, d_term_log);
        if (int rc = launched(sim, "wl_terms_log_kernel")) return rc;
    }
    return WL_OK;
}

}  // extern "C"
