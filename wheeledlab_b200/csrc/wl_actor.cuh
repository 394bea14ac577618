// wl_actor.cuh -- the actor mean alone (wl_actor_mean, DESIGN 6i): rsl_rl ActorCritic.act_inference, obs -> 64 -> 64 -> 2
// in the blob layout of wl_act_step, for any batch of observation rows and no sim handle.  Included by wl_api.cu after
// wl_wide.cuh (it reuses mlp_tile_*, elu / relu, the cp.async and bulk-copy helpers).
//
// Every output is summed in the order of the kernel that trained or rolled out the network, so playback computes what
// the rollout computed, bit for bit:
//   ELU  (obs_dim <= 16): wl_act_step's order -- bias, then inputs ascending (mlp_tile_layer); the head's quad butterfly
//   ReLU (obs_dim <= 4096): wl_policy_act's order -- layer 1 in K chunks of 32, each summed from zero and added to the
//         running sum, which starts at the bias (wide_layer1); the head's 8-thread butterfly
// With no critic, a lane's 4 x 4 register tile covers 4 rows x 4 actor units, and the two half-warps take different rows:
// warp k of a CTA owns rows 8k..8k+7.  A CTA is 4 warps (32 rows), so up to 132 x 32 rows run at one warp per scheduler.
#pragma once

#define WL_AM_ROWS 32                             // rows per CTA
#define WL_AM_THREADS 128                         // 4 warps x (2 half-warps x 4 rows)
#define WL_AM_XS (WL_WIDE_KC + 4)                 // padded staged observation row
#define WL_AM_STAGE (WL_AM_ROWS * WL_AM_XS + WL_WIDE_KC * WL_HID)      // floats per stage: x rows | the actor's W1t rows
#define WL_AM_HS (WL_HID + 4)                     // padded hidden row

// stage inputs k0 .. k0 + kn - 1 (kn a multiple of 4) of layer 1: rows r0 .. r0 + 31 of x (zero past D and past n) and the
// actor's W1t rows
__device__ __forceinline__ void actor_stage(float* sb, const float* __restrict__ x, int n, int D, int r0, const float* __restrict__ W1t,
                                            int k0, int kn) {
    for (int k = threadIdx.x; k < WL_AM_ROWS * WL_WIDE_KC; k += WL_AM_THREADS) {
        const int r = k / WL_WIDE_KC, j = k % WL_WIDE_KC, col = k0 + j;
        const bool ok = r0 + r < n && col < D;
        cp_async4(sb + r * WL_AM_XS + j, ok ? x + (size_t)(r0 + r) * D + col : x, ok);
    }
    float* sw = sb + WL_AM_ROWS * WL_AM_XS;
    for (int k = threadIdx.x; k < kn * (WL_HID / 4); k += WL_AM_THREADS)
        cp_async16(sw + k * 4, W1t + (size_t)k0 * WL_HID + k * 4);
}

// the actor mean of rows r0 .. r0 + 31 of obs [n, D] -> mean [n] (float2).  RELU: the Elevation / Visual network; else the
// Drift family's ELU network (D <= 16).  Does not trigger dependents early: a step launched after it waits for every mean.
template <bool RELU>
__global__ void __launch_bounds__(WL_AM_THREADS)
wl_actor_mean_kernel(const float* __restrict__ obs, int n, int D, const float* __restrict__ blob, PolicyOffsets po, float2* __restrict__ mean) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    float* stage = smem;                                     // 2 x WL_AM_STAGE
    float* sw = stage + 2 * WL_AM_STAGE;                     // the actor after W1t: blob [o1, o6) = b1 | W2t | b2 | W3t | b3
    float* sh = sw + (po.o[6] - po.o[1]);                    // [32][WL_AM_HS]
    const int tid = threadIdx.x, r0 = blockIdx.x * WL_AM_ROWS;
    if (tid == 0) {
        const uint32_t nb = (uint32_t)(po.o[6] - po.o[1]) * 4u;
        mbar_init(&mbar, 1);
        mbar_init_fence();
        mbar_expect(&mbar, nb);
        bulk_g2s(sw, blob + po.o[1], nb, &mbar);
    }
    const int lane = tid & 31, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 8 + (lane >> 4) * 4;
    const int nin1 = (D + 3) & ~3;
    const float* W1t = blob + po.o[0];
    float acc[4][4];
    if constexpr (RELU) {                                    // wide_layer1's chunking, actor columns only
        const int nch = (nin1 + WL_WIDE_KC - 1) / WL_WIDE_KC;
        const float4 b0 = *reinterpret_cast<const float4*>(blob + po.o[1] + ucol);
#pragma unroll
        for (int e = 0; e < 4; ++e) { acc[e][0] = b0.x; acc[e][1] = b0.y; acc[e][2] = b0.z; acc[e][3] = b0.w; }
        actor_stage(stage, obs, n, D, r0, W1t, 0, min(WL_WIDE_KC, nin1));
        cp_async_commit();
        for (int c = 0; c < nch; ++c) {
            if (c + 1 < nch) {
                const int k1 = (c + 1) * WL_WIDE_KC;
                actor_stage(stage + ((c + 1) & 1) * WL_AM_STAGE, obs, n, D, r0, W1t, k1, min(WL_WIDE_KC, nin1 - k1));
                cp_async_commit();
                cp_async_wait<1>();
            } else {
                cp_async_wait<0>();
            }
            __syncthreads();                                 // chunk c is in shared memory for every thread
            const float* sb = stage + (c & 1) * WL_AM_STAGE;
            float part[4][4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { part[e][0] = 0.0f; part[e][1] = 0.0f; part[e][2] = 0.0f; part[e][3] = 0.0f; }
            mlp_tile_accum(sb + WL_AM_ROWS * WL_AM_XS + ucol, sb + env0 * WL_AM_XS, WL_AM_XS, min(WL_WIDE_KC, nin1 - c * WL_WIDE_KC), part);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[e][q] += part[e][q];
            __syncthreads();                                 // every thread is done with the buffer the next chunk refills
        }
        store_relu(sh + env0 * WL_AM_HS + ucol, WL_AM_HS, acc);
    } else {                                                 // wl_act_step's layer 1: one pass, bias first
        actor_stage(stage, obs, n, D, r0, W1t, 0, nin1);
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        mlp_tile_layer(stage + WL_AM_ROWS * WL_AM_XS + ucol, blob + po.o[1] + ucol, stage + env0 * WL_AM_XS, WL_AM_XS, nin1, acc);
        mlp_tile_store_elu(sh + env0 * WL_AM_HS + ucol, WL_AM_HS, acc);
    }
    float* h0 = sh + env0 * WL_AM_HS;
    mbar_wait_parity(&mbar, 0);                              // b1 .. b3 have landed (the copy overlapped layer 1)
    __syncwarp();
    const int oW2 = po.o[2] - po.o[1], oB2 = po.o[3] - po.o[1], oW3 = po.o[4] - po.o[1], oB3 = po.o[5] - po.o[1];
    mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, h0, WL_AM_HS, WL_HID, acc);
    __syncwarp();                                            // every lane has finished reading layer-1 activations
    if constexpr (RELU) store_relu(h0 + ucol, WL_AM_HS, acc);
    else mlp_tile_store_elu(h0 + ucol, WL_AM_HS, acc);
    __syncthreads();                                         // layer-2 activations of all 32 rows are in shared memory
    const float* w3a = sw + oW3;
    if constexpr (RELU) {                                    // wl_policy_act's head: 8 threads per row, 8 units each
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
            const int s = pass * (WL_AM_THREADS / 8) + (tid >> 3), p = tid & 7, i = r0 + s;
            const float* hrow = sh + s * WL_AM_HS;
            float m0 = 0.0f, m1 = 0.0f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int j = 8 * p + k;
                m0 = fmaf(w3a[2 * j], hrow[j], m0); m1 = fmaf(w3a[2 * j + 1], hrow[j], m1);
            }
#pragma unroll
            for (int x = 1; x < 8; x <<= 1) {
                m0 += __shfl_xor_sync(0xffffffffu, m0, x); m1 += __shfl_xor_sync(0xffffffffu, m1, x);
            }
            if (p == 0 && i < n) mean[i] = make_float2(m0 + sw[oB3], m1 + sw[oB3 + 1]);
        }
    } else {                                                 // wl_act_step's head: 4 threads per row, 16 units each
        const int s = tid >> 2, w = tid & 3, i = r0 + s;
        const float* hrow = sh + s * WL_AM_HS;
        float m0 = 0.0f, m1 = 0.0f;
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            const int j = 16 * w + u;
            const float xa = hrow[j];
            m0 = fmaf(w3a[2 * j], xa, m0); m1 = fmaf(w3a[2 * j + 1], xa, m1);
        }
        m0 += __shfl_xor_sync(0xffffffffu, m0, 1); m0 += __shfl_xor_sync(0xffffffffu, m0, 2);
        m1 += __shfl_xor_sync(0xffffffffu, m1, 1); m1 += __shfl_xor_sync(0xffffffffu, m1, 2);
        if (w == 0 && i < n) mean[i] = make_float2(m0 + sw[oB3], m1 + sw[oB3 + 1]);
    }
}

// dynamic shared memory of wl_actor_mean_kernel (the same for every obs_dim): two stages, the actor after W1t, the hidden rows
static size_t actor_mean_smem() {
    int32_t off[13];
    policy_offsets(1, off);
    return sizeof(float) * ((size_t)2 * WL_AM_STAGE + (off[6] - off[1]) + WL_AM_ROWS * WL_AM_HS);
}
