/*
 * device_events_oracle.c -- TEST INFRASTRUCTURE: the CPU twin of the device event terms (wl_set_device_events,
 * wl_device_events_kernel; DESIGN.md 6p) on the unchanged oracle's generator.
 *
 * IsaacLab's push_by_setting_velocity per term k, in table order: a reset-mode term fires where the env was reset, an
 * interval-mode term where its timer (the interval timers' twin, event_timers_oracle.c, on the term's own timer index)
 * ran out; a fired term adds u * (hi - lo) + lo to each of the six root velocity components, u from the key
 * (seed, env_id_offset + i, t, stream 15, k) for x, y, z, roll and (..., 8 + k) for pitch, yaw.  Each fp32 operation in
 * the kernel's order (no fma).  Built by tests/device_events_oracle.py with the oracle's own flags (fp32, no contraction),
 * so it is bit-exact with the kernel.
 */
#include "event_timers_oracle.c"

#define RNG_DEVICE_EVENT 15u
#define MAX_DEVICE_EVENTS 8

/* vel [n][6] (x, y, z, roll, pitch, yaw) in place; slot[k] the timer index of term k or -1 (reset mode); lo / hi [n_terms][6];
 * timer_lo_hi [n_timers][2] and time_left [n_timers][n] as wlo_event_timers takes them. */
void wlo_device_events(uint64_t seed, int32_t env_id_offset, int32_t n, int32_t n_terms, const int32_t* slot, const float* lo,
                       const float* hi, int32_t n_timers, const float* timer_lo_hi, float step_dt, const uint8_t* done,
                       float* time_left, float* vel, int64_t step_counter) {
    uint8_t* fired = (uint8_t*)calloc((size_t)(n_timers > 0 ? n_timers : 1) * n, 1);
    if (n_timers > 0)
        wlo_event_timers(seed, env_id_offset, n, n_timers, timer_lo_hi, step_dt, done, time_left, fired, step_counter);
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < n_terms; ++k) {
            const int f = slot[k] < 0 ? done[i] != 0 : fired[(size_t)slot[k] * n + i] != 0;
            if (!f) continue;
            uint32_t a[4], b[4];
            philox4x32(seed, (uint32_t)(env_id_offset + i), (uint32_t)step_counter, RNG_DEVICE_EVENT, (uint32_t)k, a);
            philox4x32(seed, (uint32_t)(env_id_offset + i), (uint32_t)step_counter, RNG_DEVICE_EVENT, (uint32_t)(MAX_DEVICE_EVENTS + k), b);
            const uint32_t r[6] = {a[0], a[1], a[2], a[3], b[0], b[1]};
            for (int j = 0; j < 6; ++j)
                vel[(size_t)i * 6 + j] = vel[(size_t)i * 6 + j] + event_interval(r[j], lo[k * 6 + j], hi[k * 6 + j]);
        }
    free(fired);
}
