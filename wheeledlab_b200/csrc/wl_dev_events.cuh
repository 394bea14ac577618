// wl_dev_events.cuh -- device event terms: IsaacLab's push_by_setting_velocity in reset and interval mode (DESIGN 6p),
// included by wl_api.cu after decode_step.
//
// push_by_setting_velocity [UPSTREAM-RECALL], per term with velocity_range {x, y, z, roll, pitch, yaw: (lo, hi)}:
//   vel_w = asset.data.root_vel_w[env_ids]
//   vel_w += sample_uniform(ranges[:, 0], ranges[:, 1], vel_w.shape)        (torch.rand * (hi - lo) + lo)
//   asset.write_root_velocity_to_sim(vel_w, env_ids)
// The kernel runs every term of the table for one env in one thread, in table order, on the state stage b1 left: a
// reset-mode term fires where b1 reset the env, an interval-mode term where its timer (the host-side event terms' timer,
// event_timer_step) ran out.  The linear and angular velocity groups are read once and written once, and only when some
// term fired.  Every fp32 operation is written out (u * (hi - lo) + lo, then v + that, no fma) so that the test-side twin
// matches bit for bit.
#pragma once

#define WL_DEVICE_EVENTS_BS 128

struct DevEventTable {
    int32_t n;                                   // terms (0: none)
    int32_t slot[WL_MAX_DEVICE_EVENTS];          // timer index of an interval term; -1: reset mode
    float lo[WL_MAX_DEVICE_EVENTS][6], hi[WL_MAX_DEVICE_EVENTS][6];
    EventTable timers;                           // the interval terms' ranges and per-env timers (timers.n of them)
};

__global__ void __launch_bounds__(WL_DEVICE_EVENTS_BS)
wl_device_events_kernel(const __grid_constant__ wl_config c, const __grid_constant__ DevEventTable et, float4* __restrict__ st,
                        const wl_globals* __restrict__ gl, const uint8_t* __restrict__ terminated,
                        const uint8_t* __restrict__ truncated, uint32_t t_arg) {
    const int n = c.num_envs;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t t = decode_step(gl, t_arg);
    const uint32_t gid = (uint32_t)(c.env_id_offset + i);
    const bool reset = (terminated[i] | truncated[i]) != 0;
    uint32_t fire = 0u;
    for (int k = 0; k < et.n; ++k) {
        const int s = et.slot[k];
        const bool f = s < 0 ? reset
                             : event_timer_step(et.timers, s, (size_t)s * n + i, philox4x32(c.seed, gid, t, RNG_EVENT, (uint32_t)s), reset,
                                                c.d_step_dt);
        fire |= (f ? 1u : 0u) << k;
    }
    if (fire == 0u) return;
    const float4 lv = ldg4(st, WL_G_LINVEL, n, i), av = ldg4(st, WL_G_ANGVEL, n, i);
    float v[6] = {lv.x, lv.y, lv.z, av.x, av.y, av.z};
    for (int k = 0; k < et.n; ++k) {
        if (!((fire >> k) & 1u)) continue;
        const uint4 a = philox4x32(c.seed, gid, t, RNG_DEVICE_EVENT, (uint32_t)k);
        const uint4 b = philox4x32(c.seed, gid, t, RNG_DEVICE_EVENT, (uint32_t)(WL_MAX_DEVICE_EVENTS + k));
        const uint32_t r[6] = {a.x, a.y, a.z, a.w, b.x, b.y};
#pragma unroll
        for (int j = 0; j < 6; ++j) v[j] = __fadd_rn(v[j], event_interval(r[j], et.lo[k][j], et.hi[k][j]));
    }
    stg4(st, WL_G_LINVEL, n, i, make_float4(v[0], v[1], v[2], lv.w));
    stg4(st, WL_G_ANGVEL, n, i, make_float4(v[3], v[4], v[5], av.w));
}
