/*
 * event_timers_oracle.c -- TEST INFRASTRUCTURE: the CPU twin of the interval timers of host-side event terms
 * (wl_set_event_timers, wl_event_timers_kernel; DESIGN.md 6o) on the unchanged oracle's generator.
 *
 * wlo_event_timers_init is the construction draw, wlo_event_timers one step of every term: redraw where done, subtract
 * step_dt, fire below 1e-6, redraw where fired -- each fp32 operation in the kernel's order (u * (hi - lo) + lo, no fma).
 * Built by tests/event_timers_oracle.py with the oracle's own flags (fp32, no contraction), so it is bit-exact with the kernel.
 */
#include "../oracle/wl_oracle.c"

#define RNG_EVENT 13u
#define RNG_EVENT_INIT 14u

static float event_interval(uint32_t x, float lo, float hi) { return (float)u01(x) * (hi - lo) + lo; }

void wlo_event_timers_init(uint64_t seed, int32_t env_id_offset, int32_t n, int32_t n_terms, const float* lo_hi, float* time_left) {
    for (int k = 0; k < n_terms; ++k)
        for (int i = 0; i < n; ++i) {
            uint32_t r[4];
            philox4x32(seed, (uint32_t)(env_id_offset + i), 0u, RNG_EVENT_INIT, (uint32_t)k, r);
            time_left[(size_t)k * n + i] = event_interval(r[0], lo_hi[2 * k], lo_hi[2 * k + 1]);
        }
}

void wlo_event_timers(uint64_t seed, int32_t env_id_offset, int32_t n, int32_t n_terms, const float* lo_hi, float step_dt,
                      const uint8_t* done, float* time_left, uint8_t* fired, int64_t step_counter) {
    for (int k = 0; k < n_terms; ++k)
        for (int i = 0; i < n; ++i) {
            const size_t o = (size_t)k * n + i;
            const float lo = lo_hi[2 * k], hi = lo_hi[2 * k + 1];
            uint32_t r[4];
            philox4x32(seed, (uint32_t)(env_id_offset + i), (uint32_t)step_counter, RNG_EVENT, (uint32_t)k, r);
            float tl = time_left[o];
            if (done[i]) tl = event_interval(r[0], lo, hi);
            tl = tl - step_dt;
            fired[o] = tl < 1.0e-6f;
            if (fired[o]) tl = event_interval(r[1], lo, hi);
            time_left[o] = tl;
        }
}
