// wl_events.cuh -- interval timers of host-side (Python) event terms (IsaacLab EventManager, mode="interval"; DESIGN 6o),
// included by wl_api.cu.
//
// EventManager [UPSTREAM-RECALL], per interval term k with is_global_time=False, restated as the built-in push timers are:
//   _prepare_terms   time_left[k] = rand(N) * (hi - lo) + lo
//   reset(env_ids)   time_left[k][env_ids] = rand(len) * (hi - lo) + lo          (inside _reset_idx, before the interval events)
//   apply("interval", dt)
//                    time_left[k] -= dt; ids = (time_left[k] < 1e-6).nonzero();
//                    time_left[k][ids] = rand(len) * (hi - lo) + lo; func(env, ids, **params)
// The kernel does the redraw of the reset envs, the decrement, the fire test and the fire redraw of every term for one env in
// one thread, and writes one fired byte per (term, env); the host calls each term's function with its fired ids.  Every fp32
// operation is written in the order above (u * (hi - lo) + lo, not an fma), so the test-side twin matches bit for bit.
#pragma once

#define WL_EVENT_BS 128

struct EventTable {
    int32_t n;                          // interval terms (0: none)
    float lo[WL_MAX_EVENT_TERMS], hi[WL_MAX_EVENT_TERMS];
    float* time_left;                   // [n][num_envs], device
};

// torch.rand's U[0, 1) (24 bits) scaled to [lo, hi) as the event manager scales it
__device__ __forceinline__ float event_interval(uint32_t x, float lo, float hi) { return __fadd_rn(__fmul_rn(u01(x), __fsub_rn(hi, lo)), lo); }

// one step of timer k at o = k * num_envs + i with the draws r: redraw a reset env (.x), count down, fire below 1e-6 and
// redraw a fired one (.y); returns whether it fired (also the device event terms' timers, wl_dev_events.cuh)
__device__ __forceinline__ bool event_timer_step(const EventTable& et, int k, size_t o, uint4 r, bool reset, float dt) {
    float tl = et.time_left[o];
    if (reset) tl = event_interval(r.x, et.lo[k], et.hi[k]);
    tl = __fsub_rn(tl, dt);
    const bool f = tl < 1.0e-6f;
    if (f) tl = event_interval(r.y, et.lo[k], et.hi[k]);
    et.time_left[o] = tl;
    return f;
}

// the construction draw: key (seed, global env id, 0, RNG_EVENT_INIT, k)
__global__ void __launch_bounds__(WL_EVENT_BS)
wl_event_timers_init_kernel(const __grid_constant__ wl_config c, const __grid_constant__ EventTable et) {
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t gid = (uint32_t)(c.env_id_offset + i);
    for (int k = 0; k < et.n; ++k)
        et.time_left[(size_t)k * n + i] = event_interval(philox4x32(c.seed, gid, 0u, RNG_EVENT_INIT, (uint32_t)k).x, et.lo[k], et.hi[k]);
}

// one step of every term for env i: key (seed, global env id, t, RNG_EVENT, k); .x redraws a reset env, .y a fired one
__global__ void __launch_bounds__(WL_EVENT_BS)
wl_event_timers_kernel(const __grid_constant__ wl_config c, const __grid_constant__ EventTable et, const uint8_t* __restrict__ done,
                       uint8_t* __restrict__ fired, uint32_t t) {
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t gid = (uint32_t)(c.env_id_offset + i);
    const bool reset = done[i] != 0;
    const float dt = c.d_step_dt;
    for (int k = 0; k < et.n; ++k) {
        const size_t o = (size_t)k * n + i;
        fired[o] = event_timer_step(et, k, o, philox4x32(c.seed, gid, t, RNG_EVENT, (uint32_t)k), reset, dt) ? 1 : 0;
    }
}
