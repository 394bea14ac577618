// wl_episode.cuh -- the rsl_rl runner's episode statistics (modified_rsl_rl_runner.py:55-63, :99-109) over one rollout slab
// (DESIGN 6h), included by wl_api.cu.
//
// Two launches, no float atomics, no host values: wl_episode_walk_kernel (one thread per env walks t = 0..T-1: the fp32
// running return and length, each finished episode's (return, length) into the workspace at its (t, env) cell, and one
// ballot word of done flags per (t, 32 envs)) -> wl_episode_ring_kernel (one CTA: per-t done counts from the ballot words,
// the suffix walk that finds the first t whose episodes survive in the last WL_EPISODE_RING, the ranks of the survivors
// from warp suffix scans of the words, the ring writes, and the fp64 means over the ring in age order).
#pragma once

#define WL_EP_WALK_THREADS 64                      // small CTAs: the walk is latency-bound, so spread it over many SMs
#define WL_EP_CHUNK 16                             // rewards / flags loaded WL_EP_CHUNK steps ahead of the dependent sum
#define WL_EP_RING_THREADS 1024
#define WL_EP_MAX_T 4096                           // per-t counts live in shared memory

__global__ void __launch_bounds__(WL_EP_WALK_THREADS)
wl_episode_walk_kernel(const float* __restrict__ rew, const uint8_t* __restrict__ term, const uint8_t* __restrict__ trunc,
                       int T, int N, float* __restrict__ cur_ret, float* __restrict__ cur_len, float2* __restrict__ ep,
                       uint32_t* __restrict__ done_words) {
    const int i = blockIdx.x * WL_EP_WALK_THREADS + threadIdx.x;
    const int W = (N + 31) >> 5, w = i >> 5;
    if (w >= W) return;                            // a warp past the last env (N < the CTA): it owns no done word
    const bool live = i < N;                       // the tail warp's dead lanes still vote (as "not done")
    float c = live ? cur_ret[i] : 0.0f, l = live ? cur_len[i] : 0.0f;
    for (int t0 = 0; t0 < T; t0 += WL_EP_CHUNK) {
        float r[WL_EP_CHUNK];
        bool d[WL_EP_CHUNK];
#pragma unroll
        for (int k = 0; k < WL_EP_CHUNK; ++k) {
            const size_t o = (size_t)(t0 + k) * N + i;
            const bool in = live && t0 + k < T;
            r[k] = in ? rew[o] : 0.0f;
            d[k] = in && (term[o] | trunc[o]) != 0;
        }
#pragma unroll
        for (int k = 0; k < WL_EP_CHUNK; ++k) {
            const int t = t0 + k;
            if (t < T) {                           // (warp-uniform)
                c += r[k];                         // cur_reward_sum += rewards (fp32, in t order)
                l += 1.0f;                         // cur_episode_length += 1
                const uint32_t word = __ballot_sync(0xffffffffu, d[k]);
                if (d[k]) { ep[(size_t)t * N + i] = make_float2(c, l); c = 0.0f; l = 0.0f; }
                if ((threadIdx.x & 31) == 0) done_words[(size_t)t * W + w] = word;
            }
        }
    }
    if (live) { cur_ret[i] = c; cur_len[i] = l; }
}

// One CTA.  The episodes of this call are appended in (t, env id) order, M of them; the one that is k-th from the end
// (k = 0 the last) survives iff k < WL_EPISODE_RING and lands in ring slot (head + M - 1 - k) mod WL_EPISODE_RING.
__global__ void __launch_bounds__(WL_EP_RING_THREADS)
wl_episode_ring_kernel(const float2* __restrict__ ep, const uint32_t* __restrict__ done_words, int T, int N,
                       wl_episode_stats_state* __restrict__ st) {
    __shared__ int s_after[WL_EP_MAX_T];           // done count of row t, then: episodes in the rows after t
    __shared__ int s_part[WL_EP_RING_THREADS / 32];
    __shared__ int s_t0, s_total;
    const int W = (N + 31) >> 5, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int head = st->head;
    for (int t = warp; t < T; t += WL_EP_RING_THREADS / 32) {
        int c = 0;
        for (int w = lane; w < W; w += 32) c += __popc(done_words[(size_t)t * W + w]);
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) s_after[t] = c;
    }
    __syncthreads();
    int part = 0;
    for (int t = threadIdx.x; t < T; t += WL_EP_RING_THREADS) part += s_after[t];
    part = __reduce_add_sync(0xffffffffu, part);
    if (lane == 0) s_part[warp] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        int total = 0;
        for (int k = 0; k < WL_EP_RING_THREADS / 32; ++k) total += s_part[k];
        // walk back from the last row until WL_EPISODE_RING episodes lie behind: rows before that contribute nothing
        int after = 0, t = T - 1;
        for (; t >= 0 && after < WL_EPISODE_RING; --t) { const int c = s_after[t]; s_after[t] = after; after += c; }
        s_t0 = t + 1;
        s_total = total;
    }
    __syncthreads();
    const int t0 = s_t0, M = s_total;
    for (int t = t0 + warp; t < T; t += WL_EP_RING_THREADS / 32) {     // a warp per row, 32 words at a time from the top
        int after = s_after[t];                                        // (warp-uniform)
        for (int hi = W; hi > 0 && after < WL_EPISODE_RING; hi -= 32) {
            const int w = hi - 32 + lane;
            const uint32_t word = w >= 0 ? done_words[(size_t)t * W + w] : 0u;
            const int c = __popc(word);
            int s = c;                                                 // done envs in words w.. of this chunk
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_down_sync(0xffffffffu, s, o); if (lane + o < 32) s += v; }
            int k = after + s - c;                                     // from-the-end index of the word's highest done env
            for (uint32_t m = word; m != 0u && k < WL_EPISODE_RING; ++k) {
                const int b = 31 - __clz(m);
                m &= ~(1u << b);
                const float2 e = ep[(size_t)t * N + w * 32 + b];
                const int slot = (int)(((int64_t)head + M - 1 - k) % WL_EPISODE_RING);
                st->ring_return[slot] = e.x;
                st->ring_length[slot] = e.y;
            }
            after += __shfl_sync(0xffffffffu, s, 0);
        }
    }
    __syncthreads();                                                   // the ring writes are visible to thread 0
    if (threadIdx.x == 0) {
        const int fill = min(WL_EPISODE_RING, st->fill + M);
        const int head2 = (int)(((int64_t)head + M) % WL_EPISODE_RING);
        double sr = 0.0, sl = 0.0;                                     // statistics.mean: fp64, oldest first
        for (int k = 0; k < fill; ++k) {
            const int slot = (head2 - fill + k + WL_EPISODE_RING) % WL_EPISODE_RING;
            sr += (double)st->ring_return[slot];
            sl += (double)st->ring_length[slot];
        }
        st->fill = fill;
        st->head = head2;
        st->finished = M;
        st->mean_return = fill > 0 ? sr / fill : 0.0;
        st->mean_length = fill > 0 ? sl / fill : 0.0;
    }
}
