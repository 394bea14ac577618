// wl_ppo.cuh -- rsl_rl PPO.update() for the Drift-family actor-critic (DESIGN 6f), included by wl_api.cu after the
// policy blob layout, mlp_tile_layer, the bulk-copy helpers and adam_update it reuses.
//
// Per mini-batch: wl_ppo_grad_kernel (persistent CTAs, one gradient row per CTA in blob layout) -> wl_ppo_reduce_kernel
// (rows summed in CTA order per column, fp64 block sums of squares) -> wl_ppo_step_kernel (norm, KL rule, clip, Adam,
// statistics).  No float atomics anywhere: the reduction order is fixed by (batch, SM count).
#pragma once

#define WL_PPO_THREADS 256
#define WL_PPO_TILE 32                            // samples per tile: 8 warps x 4 samples in the mlp_tile_layer geometry
#define WL_PPO_XS 20                              // padded observation row
#define WL_PPO_XA 36                              // asymmetric update: padded row of either input (critic_dim <= 32)
#define WL_PPO_HS (2 * WL_HID + 4)                // padded hidden row, [actor 64 | critic 64 | pad]
#define WL_PPO_SD 8                               // per-sample row: dmu0 dmu1 dV dsigma0 dsigma1 | surrogate value-loss KL
#define WL_PPO_STATS 3                            // columns after the blob in a gradient row: surrogate, value loss, KL sums
#define WL_PPO_FIN_THREADS 1024
#define WL_PPO_LOG_SQRT_2PI 0.91893853320467274f

struct PpoArgs {
    wl_ppo_batch b;
    int64_t row0;                                 // first perm index of this mini-batch
    int obs_dim, B, tiles;
    float clip, vcoef, inv_B;
    int clipped_value;
};

// ELU with an accurate expm1 (torch's fp32 ELU), and its derivative from the activation: elu'(x) = h > 0 ? 1 : h + 1
__device__ __forceinline__ float ppo_elu(float x) { return x > 0.0f ? x : expm1f(x); }
__device__ __forceinline__ float ppo_elu_grad(float h) { return h > 0.0f ? 1.0f : h + 1.0f; }
// torch.max(x, y) backward: the share of the gradient that goes to x (half at ties)
__device__ __forceinline__ float ppo_max_share(float x, float y) { return x > y ? 1.0f : (x == y ? 0.5f : 0.0f); }

// is blob float c a parameter (not alignment padding, not a zero row of W1t)?  critic_dim: the critic's input width
// (obs_dim for the symmetric network)
__device__ __forceinline__ bool ppo_is_param(int c, const PolicyOffsets& po, int obs_dim, int critic_dim) {
    const int len[13] = {obs_dim * WL_HID, WL_HID, WL_HID * WL_HID, WL_HID, WL_HID * 2, 2,
                         critic_dim * WL_HID, WL_HID, WL_HID * WL_HID, WL_HID, WL_HID, 1, 2};
    bool p = false;
#pragma unroll
    for (int k = 0; k < 13; ++k) p |= (c >= po.o[k] && c < po.o[k] + len[k]);
    return p;
}

// the loss terms of mini-batch row `row` (< B) with the network outputs (mu0, mu1, V) = (m0, m1, vv): d[0..4] = dL/dmu0,
// dL/dmu1, dL/dV, dL/dsigma0, dL/dsigma1 (the log-prob part), d[5..7] = surrogate, value loss, KL
__device__ __forceinline__ void ppo_sample_derivs(const PpoArgs& a, int row, float m0, float m1, float vv, float sg_0, float sg_1,
                                                  float so0, float so1, float adv_mean, float adv_den, float* d) {
    const int64_t g = a.b.perm[a.row0 + row];
    const float2 act = reinterpret_cast<const float2*>(a.b.actions)[g];
    const float2 mo = reinterpret_cast<const float2*>(a.b.mean)[g];
    const float A = (a.b.advantages[g] - adv_mean) / adv_den;
    const float R = a.b.returns[g], vo = a.b.values[g];
    // log-prob of the stored action under N(mu, sigma), summed over the two dims (torch Normal.log_prob)
    const float d0 = act.x - m0, d1 = act.y - m1, var0 = sg_0 * sg_0, var1 = sg_1 * sg_1;
    const float lp = (-(d0 * d0) / (2.0f * var0) - logf(sg_0) - WL_PPO_LOG_SQRT_2PI)
                   + (-(d1 * d1) / (2.0f * var1) - logf(sg_1) - WL_PPO_LOG_SQRT_2PI);
    const float ratio = expf(lp - a.b.log_prob[g]);
    const float lo = 1.0f - a.clip, hi = 1.0f + a.clip;
    const float su1 = -A * ratio, su2 = -A * fminf(fmaxf(ratio, lo), hi);
    const float w = ppo_max_share(su1, su2);
    const float in_r = (ratio >= lo && ratio <= hi) ? 1.0f : 0.0f;      // clamp passes the gradient at its bounds
    const float dratio = (w * a.inv_B) * -A + ((1.0f - w) * a.inv_B) * -A * in_r;
    const float dlp = dratio * ratio;
    d[0] = dlp * (d0 / var0);
    d[1] = dlp * (d1 / var1);
    d[3] = dlp * ((d0 * d0) * sg_0 / (var0 * var0) - 1.0f / sg_0);
    d[4] = dlp * ((d1 * d1) * sg_1 / (var1 * var1) - 1.0f / sg_1);
    float vl, dv;
    if (a.clipped_value) {
        const float dvo = vv - vo, vc = vo + fminf(fmaxf(dvo, -a.clip), a.clip);
        const float l1 = (vv - R) * (vv - R), l2 = (vc - R) * (vc - R), wv = ppo_max_share(l1, l2);
        const float in_v = (dvo >= -a.clip && dvo <= a.clip) ? 1.0f : 0.0f;
        dv = (wv * a.inv_B) * (2.0f * (vv - R)) + ((1.0f - wv) * a.inv_B) * (2.0f * (vc - R)) * in_v;
        vl = fmaxf(l1, l2);
    } else {
        dv = a.inv_B * (2.0f * (vv - R));
        vl = (R - vv) * (R - vv);
    }
    d[2] = a.vcoef * dv;
    d[5] = fmaxf(su1, su2);
    d[6] = vl;
    const float e0 = mo.x - m0, e1 = mo.y - m1;
    d[7] = (logf(sg_0 / so0 + 1e-5f) + (so0 * so0 + e0 * e0) / (2.0f * var0) - 0.5f)
         + (logf(sg_1 / so1 + 1e-5f) + (so1 * so1 + e1 * e1) / (2.0f * var1) - 0.5f);
}

__device__ __forceinline__ void ppo_store_elu(float* h0, const float acc[4][4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
        *reinterpret_cast<float4*>(h0 + e * WL_PPO_HS) = make_float4(ppo_elu(acc[e][0]), ppo_elu(acc[e][1]), ppo_elu(acc[e][2]), ppo_elu(acc[e][3]));
}

// One launch per mini-batch.  CTA b takes tiles b, b + grid, ... of 32 samples; per tile: gather through the permutation,
// both forward passes (mlp_tile_layer), the per-sample loss derivatives, back-propagation through shared memory, and
// accumulation of every weight gradient in registers (thread t owns a fixed set of gradient entries for the CTA's whole
// lifetime, summed over samples in order).  At the end it writes its row of the workspace in blob layout.
// wl_ppo_grad_asym_kernel below is this kernel with a critic row of its own: a change to the forward, backward or
// accumulation here belongs there too (tests/test_asym_critic_gpu.py holds the two to the same bits).
__global__ void __launch_bounds__(WL_PPO_THREADS, 1)
wl_ppo_grad_kernel(const float* __restrict__ blob, int blob_floats, PolicyOffsets po, const __grid_constant__ PpoArgs a,
                   const float* __restrict__ state, float* __restrict__ rows, int rowlen) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    float* sw = smem;                                        // the whole blob
    float* sw2t = sw + blob_floats;                          // [net][64 out][64 in]: W2 output-major, for dh1 = dz2 W2
    float* szero = sw2t + 2 * WL_HID * WL_HID;               // the zero "bias" of the backward layer
    float* sx = szero + WL_HID;                              // [32][XS]
    float* sh1 = sx + WL_PPO_TILE * WL_PPO_XS;               // [32][HS] layer-1 activations
    float* sh2 = sh1 + WL_PPO_TILE * WL_PPO_HS;              // layer-2 activations
    float* sg2 = sh2 + WL_PPO_TILE * WL_PPO_HS;              // dL/dz2
    float* sg1 = sg2 + WL_PPO_TILE * WL_PPO_HS;              // dL/dz1
    float* sd = sg1 + WL_PPO_TILE * WL_PPO_HS;               // [32][SD]
    const int tid = threadIdx.x, D = a.obs_dim;
    if (tid == 0) {
        mbar_init(&mbar, 1);
        mbar_init_fence();
        mbar_expect(&mbar, (uint32_t)blob_floats * 4u);
        bulk_g2s(sw, blob, (uint32_t)blob_floats * 4u, &mbar);
    }
    if (tid < WL_HID) szero[tid] = 0.0f;
    const float adv_mean = state[4], adv_den = state[5] + 1e-8f, so0 = state[2], so1 = state[3];
    __syncthreads();
    mbar_wait_parity(&mbar, 0);
    for (int k = tid; k < 2 * WL_HID * WL_HID; k += WL_PPO_THREADS) {
        const int u = (k >> 6) & (WL_HID - 1), i = k & (WL_HID - 1);
        sw2t[k] = sw[(k >> 12 ? po.o[8] : po.o[2]) + i * WL_HID + u];
    }
    const float sg_0 = sw[po.o[12]], sg_1 = sw[po.o[12] + 1];
    // gradient entries this thread owns: net = tid / 128, r = tid % 128
    const int net = tid >> 7, r = tid & 127;
    const int i2 = (r >> 3) * 4, u2 = (r & 7) * 8;           // dW2t rows i2..i2+3, cols u2..u2+7
    const int i1 = (r >> 4) * 2, u1 = (r & 15) * 4;          // dW1t rows i1..i1+1, cols u1..u1+3
    float gW2[4][8], gW1[2][4], gb = 0.0f, gh = 0.0f;        // gb: db1 (r < 64) / db2; gh: head, std or statistic (tid < 200)
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 8; ++q) gW2[k][q] = 0.0f;
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int q = 0; q < 4; ++q) gW1[k][q] = 0.0f;
    // forward geometry (as wl_act_step): warp w takes samples 4w..4w+3, lane = (net, 4 units)
    const int lane = tid & 31, fnet = lane >> 4, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 4, nin1 = (D + 3) & ~3;
    const int oW1 = fnet ? po.o[6] : po.o[0], oB1 = fnet ? po.o[7] : po.o[1];
    const int oW2 = fnet ? po.o[8] : po.o[2], oB2 = fnet ? po.o[9] : po.o[3];
    const float b3a0 = sw[po.o[5]], b3a1 = sw[po.o[5] + 1], b3c = sw[po.o[11]];
    __syncthreads();                                         // sw2t complete

    for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
        const int s0 = tile * WL_PPO_TILE;
        for (int k = tid; k < WL_PPO_TILE * 16; k += WL_PPO_THREADS) {
            const int s = k >> 4, j = k & 15, row = s0 + s;
            float x = 0.0f;
            if (row < a.B && j < D) x = a.b.obs[(size_t)a.b.perm[a.row0 + row] * D + j];
            sx[s * WL_PPO_XS + j] = x;
        }
        __syncthreads();
        {
            float acc[4][4];
            float* h1 = sh1 + env0 * WL_PPO_HS + fnet * WL_HID;
            mlp_tile_layer(sw + oW1 + ucol, sw + oB1 + ucol, sx + env0 * WL_PPO_XS, WL_PPO_XS, nin1, acc);
            ppo_store_elu(h1 + ucol, acc);
            __syncwarp();
            mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, h1, WL_PPO_HS, WL_HID, acc);
            ppo_store_elu(sh2 + env0 * WL_PPO_HS + fnet * WL_HID + ucol, acc);
        }
        __syncthreads();
        {   // heads: 8 threads per sample, 8 hidden units each, then a butterfly; thread 0 of the 8 forms the derivatives
            const int s = tid >> 3, p = tid & 7, row = s0 + s;
            const float* hrow = sh2 + s * WL_PPO_HS;
            const float* w3a = sw + po.o[4]; const float* w3c = sw + po.o[10];
            float m0 = 0.0f, m1 = 0.0f, vv = 0.0f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int j = 8 * p + k;
                m0 = fmaf(w3a[2 * j], hrow[j], m0); m1 = fmaf(w3a[2 * j + 1], hrow[j], m1);
                vv = fmaf(w3c[j], hrow[WL_HID + j], vv);
            }
#pragma unroll
            for (int x = 1; x < 8; x <<= 1) {
                m0 += __shfl_xor_sync(0xffffffffu, m0, x); m1 += __shfl_xor_sync(0xffffffffu, m1, x);
                vv += __shfl_xor_sync(0xffffffffu, vv, x);
            }
            if (p == 0) {
                float* d = sd + s * WL_PPO_SD;
                if (row < a.B) {
                    ppo_sample_derivs(a, row, m0 + b3a0, m1 + b3a1, vv + b3c, sg_0, sg_1, so0, so1, adv_mean, adv_den, d);
                } else {
#pragma unroll
                    for (int k = 0; k < WL_PPO_SD; ++k) d[k] = 0.0f;     // tail of a partial tile: no gradient
                }
            }
        }
        __syncthreads();
        for (int k = tid; k < WL_PPO_TILE * 2 * WL_HID; k += WL_PPO_THREADS) {     // dz2 = (dy W3) * elu'(h2)
            const int s = k >> 7, c = k & 127;
            const float* d = sd + s * WL_PPO_SD;
            const float dh = c < WL_HID ? d[0] * sw[po.o[4] + 2 * c] + d[1] * sw[po.o[4] + 2 * c + 1] : d[2] * sw[po.o[10] + c - WL_HID];
            sg2[s * WL_PPO_HS + c] = dh * ppo_elu_grad(sh2[s * WL_PPO_HS + c]);
        }
        __syncthreads();
        {   // dz1 = (dz2 W2) * elu'(h1): the forward layer routine on the output-major copy of W2, zero bias
            float acc[4][4];
            mlp_tile_layer(sw2t + fnet * WL_HID * WL_HID + ucol, szero + ucol, sg2 + env0 * WL_PPO_HS + fnet * WL_HID, WL_PPO_HS, WL_HID, acc);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int o = (env0 + e) * WL_PPO_HS + fnet * WL_HID + ucol;
                const float4 h = *reinterpret_cast<const float4*>(sh1 + o);
                *reinterpret_cast<float4*>(sg1 + o) = make_float4(acc[e][0] * ppo_elu_grad(h.x), acc[e][1] * ppo_elu_grad(h.y),
                                                                  acc[e][2] * ppo_elu_grad(h.z), acc[e][3] * ppo_elu_grad(h.w));
            }
        }
        __syncthreads();
        // accumulate the weight gradients over the tile's samples, in sample order
        for (int s = 0; s < WL_PPO_TILE; ++s) {
            const float* h1 = sh1 + s * WL_PPO_HS + net * WL_HID;
            const float* g2 = sg2 + s * WL_PPO_HS + net * WL_HID;
            const float* g1 = sg1 + s * WL_PPO_HS + net * WL_HID;
            const float4 hv = *reinterpret_cast<const float4*>(h1 + i2);
            const float4 ga = *reinterpret_cast<const float4*>(g2 + u2), gc = *reinterpret_cast<const float4*>(g2 + u2 + 4);
            const float hk[4] = {hv.x, hv.y, hv.z, hv.w}, gq[8] = {ga.x, ga.y, ga.z, ga.w, gc.x, gc.y, gc.z, gc.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int q = 0; q < 8; ++q) gW2[k][q] = fmaf(hk[k], gq[q], gW2[k][q]);
            const float2 xv = *reinterpret_cast<const float2*>(sx + s * WL_PPO_XS + i1);
            const float4 dz = *reinterpret_cast<const float4*>(g1 + u1);
            const float xk[2] = {xv.x, xv.y}, dq[4] = {dz.x, dz.y, dz.z, dz.w};
#pragma unroll
            for (int k = 0; k < 2; ++k)
#pragma unroll
                for (int q = 0; q < 4; ++q) gW1[k][q] = fmaf(xk[k], dq[q], gW1[k][q]);
            gb += r < WL_HID ? g1[r] : g2[r - WL_HID];
            const float* d = sd + s * WL_PPO_SD;
            if (tid < 128) gh = fmaf(sh2[s * WL_PPO_HS + (tid >> 1)], d[tid & 1], gh);
            else if (tid < 192) gh = fmaf(sh2[s * WL_PPO_HS + tid - 64], d[2], gh);
            else if (tid < 200) gh += d[tid - 192];
        }
        __syncthreads();                                     // the next tile overwrites the shared rows
    }

    float* row = rows + (size_t)blockIdx.x * rowlen;
    const int gW1o = net ? po.o[6] : po.o[0], gB1o = net ? po.o[7] : po.o[1];
    const int gW2o = net ? po.o[8] : po.o[2], gB2o = net ? po.o[9] : po.o[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        *reinterpret_cast<float4*>(row + gW2o + (i2 + k) * WL_HID + u2) = make_float4(gW2[k][0], gW2[k][1], gW2[k][2], gW2[k][3]);
        *reinterpret_cast<float4*>(row + gW2o + (i2 + k) * WL_HID + u2 + 4) = make_float4(gW2[k][4], gW2[k][5], gW2[k][6], gW2[k][7]);
    }
#pragma unroll
    for (int k = 0; k < 2; ++k)
        if (i1 + k < D) *reinterpret_cast<float4*>(row + gW1o + (i1 + k) * WL_HID + u1) = make_float4(gW1[k][0], gW1[k][1], gW1[k][2], gW1[k][3]);
    row[r < WL_HID ? gB1o + r : gB2o + r - WL_HID] = gb;
    if (tid < 128) row[po.o[4] + tid] = gh;                  // dW3t actor, [unit][action]
    else if (tid < 192) row[po.o[10] + tid - 128] = gh;      // dW3t critic
    else if (tid < 194) row[po.o[5] + tid - 192] = gh;       // db3 actor
    else if (tid == 194) row[po.o[11]] = gh;                 // db3 critic
    else if (tid < 197) row[po.o[12] + tid - 195] = gh;      // dsigma (the log-prob part; entropy is added once when reduced)
    else if (tid < 200) row[blob_floats + tid - 197] = gh;   // surrogate / value-loss / KL sums
}

// wl_ppo_grad_kernel for the asymmetric network (wl_ppo_update_asym): the critic's layer 1 and its dW1 run over a second
// gathered row, critic_obs [batch, Dc]; both inputs are staged [net][32][WL_PPO_XA], zero-padded, and a thread owns four dW1t
// rows of its net instead of two.  Everything else is wl_ppo_grad_kernel line for line (a kernel of its own so that the
// symmetric kernel's code is not perturbed): every gradient entry is still one fmaf chain over the samples in order, so with
// Dc == obs_dim and critic_obs == obs the row equals the symmetric kernel's.
__global__ void __launch_bounds__(WL_PPO_THREADS, 1)
wl_ppo_grad_asym_kernel(const float* __restrict__ blob, int blob_floats, PolicyOffsets po, const __grid_constant__ PpoArgs a,
                        const float* __restrict__ critic_obs, int Dc, const float* __restrict__ state, float* __restrict__ rows,
                        int rowlen) {
    constexpr int XS = WL_PPO_XA, R1 = 4;
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    float* sw = smem;                                        // the whole blob
    float* sw2t = sw + blob_floats;                          // [net][64 out][64 in]: W2 output-major, for dh1 = dz2 W2
    float* szero = sw2t + 2 * WL_HID * WL_HID;               // the zero "bias" of the backward layer
    float* sx = szero + WL_HID;                              // [net][32][XS]
    float* sh1 = sx + 2 * WL_PPO_TILE * XS;                  // [32][HS] layer-1 activations
    float* sh2 = sh1 + WL_PPO_TILE * WL_PPO_HS;              // layer-2 activations
    float* sg2 = sh2 + WL_PPO_TILE * WL_PPO_HS;              // dL/dz2
    float* sg1 = sg2 + WL_PPO_TILE * WL_PPO_HS;              // dL/dz1
    float* sd = sg1 + WL_PPO_TILE * WL_PPO_HS;               // [32][SD]
    const int tid = threadIdx.x, D = a.obs_dim;
    if (tid == 0) {
        mbar_init(&mbar, 1);
        mbar_init_fence();
        mbar_expect(&mbar, (uint32_t)blob_floats * 4u);
        bulk_g2s(sw, blob, (uint32_t)blob_floats * 4u, &mbar);
    }
    if (tid < WL_HID) szero[tid] = 0.0f;
    const float adv_mean = state[4], adv_den = state[5] + 1e-8f, so0 = state[2], so1 = state[3];
    __syncthreads();
    mbar_wait_parity(&mbar, 0);
    for (int k = tid; k < 2 * WL_HID * WL_HID; k += WL_PPO_THREADS) {
        const int u = (k >> 6) & (WL_HID - 1), i = k & (WL_HID - 1);
        sw2t[k] = sw[(k >> 12 ? po.o[8] : po.o[2]) + i * WL_HID + u];
    }
    const float sg_0 = sw[po.o[12]], sg_1 = sw[po.o[12] + 1];
    // gradient entries this thread owns: net = tid / 128, r = tid % 128
    const int net = tid >> 7, r = tid & 127;
    const int i2 = (r >> 3) * 4, u2 = (r & 7) * 8;           // dW2t rows i2..i2+3, cols u2..u2+7
    const int i1 = (r >> 4) * R1, u1 = (r & 15) * 4;         // dW1t rows i1..i1+R1-1, cols u1..u1+3
    float gW2[4][8], gW1[R1][4], gb = 0.0f, gh = 0.0f;        // gb: db1 (r < 64) / db2; gh: head, std or statistic (tid < 200)
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 8; ++q) gW2[k][q] = 0.0f;
#pragma unroll
    for (int k = 0; k < R1; ++k)
#pragma unroll
        for (int q = 0; q < 4; ++q) gW1[k][q] = 0.0f;
    // forward geometry (as wl_act_step): warp w takes samples 4w..4w+3, lane = (net, 4 units)
    const int lane = tid & 31, fnet = lane >> 4, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 4;
    const int nin1 = ((fnet ? Dc : D) + 3) & ~3;
    const float* fx = sx + fnet * WL_PPO_TILE * XS;          // the forward lane's input rows
    const float* gx = sx + net * WL_PPO_TILE * XS;           // the gradient thread's input rows
    const int Dn = net ? Dc : D;
    const int oW1 = fnet ? po.o[6] : po.o[0], oB1 = fnet ? po.o[7] : po.o[1];
    const int oW2 = fnet ? po.o[8] : po.o[2], oB2 = fnet ? po.o[9] : po.o[3];
    const float b3a0 = sw[po.o[5]], b3a1 = sw[po.o[5] + 1], b3c = sw[po.o[11]];
    __syncthreads();                                         // sw2t complete

    for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
        const int s0 = tile * WL_PPO_TILE;
        for (int k = tid; k < 2 * WL_PPO_TILE * 32; k += WL_PPO_THREADS) {
            const int xn = k >> 10, s = (k >> 5) & 31, j = k & 31, row = s0 + s;
            float x = 0.0f;
            if (row < a.B) {
                const size_t g = (size_t)a.b.perm[a.row0 + row];
                if (xn == 0) { if (j < D) x = a.b.obs[g * D + j]; }
                else if (j < Dc) x = critic_obs[g * Dc + j];
            }
            sx[(xn * WL_PPO_TILE + s) * XS + j] = x;
        }
        __syncthreads();
        {
            float acc[4][4];
            float* h1 = sh1 + env0 * WL_PPO_HS + fnet * WL_HID;
            mlp_tile_layer(sw + oW1 + ucol, sw + oB1 + ucol, fx + env0 * XS, XS, nin1, acc);
            ppo_store_elu(h1 + ucol, acc);
            __syncwarp();
            mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, h1, WL_PPO_HS, WL_HID, acc);
            ppo_store_elu(sh2 + env0 * WL_PPO_HS + fnet * WL_HID + ucol, acc);
        }
        __syncthreads();
        {   // heads: 8 threads per sample, 8 hidden units each, then a butterfly; thread 0 of the 8 forms the derivatives
            const int s = tid >> 3, p = tid & 7, row = s0 + s;
            const float* hrow = sh2 + s * WL_PPO_HS;
            const float* w3a = sw + po.o[4]; const float* w3c = sw + po.o[10];
            float m0 = 0.0f, m1 = 0.0f, vv = 0.0f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int j = 8 * p + k;
                m0 = fmaf(w3a[2 * j], hrow[j], m0); m1 = fmaf(w3a[2 * j + 1], hrow[j], m1);
                vv = fmaf(w3c[j], hrow[WL_HID + j], vv);
            }
#pragma unroll
            for (int x = 1; x < 8; x <<= 1) {
                m0 += __shfl_xor_sync(0xffffffffu, m0, x); m1 += __shfl_xor_sync(0xffffffffu, m1, x);
                vv += __shfl_xor_sync(0xffffffffu, vv, x);
            }
            if (p == 0) {
                float* d = sd + s * WL_PPO_SD;
                if (row < a.B) {
                    ppo_sample_derivs(a, row, m0 + b3a0, m1 + b3a1, vv + b3c, sg_0, sg_1, so0, so1, adv_mean, adv_den, d);
                } else {
#pragma unroll
                    for (int k = 0; k < WL_PPO_SD; ++k) d[k] = 0.0f;     // tail of a partial tile: no gradient
                }
            }
        }
        __syncthreads();
        for (int k = tid; k < WL_PPO_TILE * 2 * WL_HID; k += WL_PPO_THREADS) {     // dz2 = (dy W3) * elu'(h2)
            const int s = k >> 7, c = k & 127;
            const float* d = sd + s * WL_PPO_SD;
            const float dh = c < WL_HID ? d[0] * sw[po.o[4] + 2 * c] + d[1] * sw[po.o[4] + 2 * c + 1] : d[2] * sw[po.o[10] + c - WL_HID];
            sg2[s * WL_PPO_HS + c] = dh * ppo_elu_grad(sh2[s * WL_PPO_HS + c]);
        }
        __syncthreads();
        {   // dz1 = (dz2 W2) * elu'(h1): the forward layer routine on the output-major copy of W2, zero bias
            float acc[4][4];
            mlp_tile_layer(sw2t + fnet * WL_HID * WL_HID + ucol, szero + ucol, sg2 + env0 * WL_PPO_HS + fnet * WL_HID, WL_PPO_HS, WL_HID, acc);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int o = (env0 + e) * WL_PPO_HS + fnet * WL_HID + ucol;
                const float4 h = *reinterpret_cast<const float4*>(sh1 + o);
                *reinterpret_cast<float4*>(sg1 + o) = make_float4(acc[e][0] * ppo_elu_grad(h.x), acc[e][1] * ppo_elu_grad(h.y),
                                                                  acc[e][2] * ppo_elu_grad(h.z), acc[e][3] * ppo_elu_grad(h.w));
            }
        }
        __syncthreads();
        // accumulate the weight gradients over the tile's samples, in sample order
        for (int s = 0; s < WL_PPO_TILE; ++s) {
            const float* h1 = sh1 + s * WL_PPO_HS + net * WL_HID;
            const float* g2 = sg2 + s * WL_PPO_HS + net * WL_HID;
            const float* g1 = sg1 + s * WL_PPO_HS + net * WL_HID;
            const float4 hv = *reinterpret_cast<const float4*>(h1 + i2);
            const float4 ga = *reinterpret_cast<const float4*>(g2 + u2), gc = *reinterpret_cast<const float4*>(g2 + u2 + 4);
            const float hk[4] = {hv.x, hv.y, hv.z, hv.w}, gq[8] = {ga.x, ga.y, ga.z, ga.w, gc.x, gc.y, gc.z, gc.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int q = 0; q < 8; ++q) gW2[k][q] = fmaf(hk[k], gq[q], gW2[k][q]);
            const float4 xv = *reinterpret_cast<const float4*>(gx + s * XS + i1);
            const float4 dz = *reinterpret_cast<const float4*>(g1 + u1);
            const float xk[4] = {xv.x, xv.y, xv.z, xv.w}, dq[4] = {dz.x, dz.y, dz.z, dz.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int q = 0; q < 4; ++q) gW1[k][q] = fmaf(xk[k], dq[q], gW1[k][q]);
            gb += r < WL_HID ? g1[r] : g2[r - WL_HID];
            const float* d = sd + s * WL_PPO_SD;
            if (tid < 128) gh = fmaf(sh2[s * WL_PPO_HS + (tid >> 1)], d[tid & 1], gh);
            else if (tid < 192) gh = fmaf(sh2[s * WL_PPO_HS + tid - 64], d[2], gh);
            else if (tid < 200) gh += d[tid - 192];
        }
        __syncthreads();                                     // the next tile overwrites the shared rows
    }

    float* row = rows + (size_t)blockIdx.x * rowlen;
    const int gW1o = net ? po.o[6] : po.o[0], gB1o = net ? po.o[7] : po.o[1];
    const int gW2o = net ? po.o[8] : po.o[2], gB2o = net ? po.o[9] : po.o[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        *reinterpret_cast<float4*>(row + gW2o + (i2 + k) * WL_HID + u2) = make_float4(gW2[k][0], gW2[k][1], gW2[k][2], gW2[k][3]);
        *reinterpret_cast<float4*>(row + gW2o + (i2 + k) * WL_HID + u2 + 4) = make_float4(gW2[k][4], gW2[k][5], gW2[k][6], gW2[k][7]);
    }
#pragma unroll
    for (int k = 0; k < R1; ++k)
        if (i1 + k < Dn) *reinterpret_cast<float4*>(row + gW1o + (i1 + k) * WL_HID + u1) = make_float4(gW1[k][0], gW1[k][1], gW1[k][2], gW1[k][3]);
    row[r < WL_HID ? gB1o + r : gB2o + r - WL_HID] = gb;
    if (tid < 128) row[po.o[4] + tid] = gh;                  // dW3t actor, [unit][action]
    else if (tid < 192) row[po.o[10] + tid - 128] = gh;      // dW3t critic
    else if (tid < 194) row[po.o[5] + tid - 192] = gh;       // db3 actor
    else if (tid == 194) row[po.o[11]] = gh;                 // db3 critic
    else if (tid < 197) row[po.o[12] + tid - 195] = gh;      // dsigma (the log-prob part; entropy is added once when reduced)
    else if (tid < 200) row[blob_floats + tid - 197] = gh;   // surrogate / value-loss / KL sums
}

// Column c of the reduced row = sum of the CTAs' rows in CTA order (+ the entropy term's d/dsigma = -entropy_coef / sigma for
// the std entries); each block also writes the fp64 sum of squares of its parameter columns (tree in thread order).
__device__ __forceinline__ void ppo_reduce_body(const float* __restrict__ rows, int nrows, int rowlen, int blob_floats,
                                                const PolicyOffsets& po, int obs_dim, int critic_dim, const float* __restrict__ blob,
                                                float entropy_coef, float* __restrict__ red, double* __restrict__ norm_part) {
    __shared__ double sq[256];
    const int c = blockIdx.x * 256 + threadIdx.x;
    const bool param = c < blob_floats && ppo_is_param(c, po, obs_dim, critic_dim);
    float g = 0.0f;
    if (param || (c >= blob_floats && c < blob_floats + WL_PPO_STATS))
        for (int r = 0; r < nrows; ++r) g += rows[(size_t)r * rowlen + c];
    if (c >= po.o[12] && c < po.o[12] + 2) g -= entropy_coef / blob[c];
    if (c < rowlen) red[c] = g;
    sq[threadIdx.x] = param ? (double)g * (double)g : 0.0;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) sq[threadIdx.x] += sq[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) norm_part[blockIdx.x] = sq[0];
}
__global__ void __launch_bounds__(256)
wl_ppo_reduce_kernel(const float* __restrict__ rows, int nrows, int rowlen, int blob_floats, PolicyOffsets po, int obs_dim,
                     const float* __restrict__ blob, float entropy_coef, float* __restrict__ red, double* __restrict__ norm_part) {
    ppo_reduce_body(rows, nrows, rowlen, blob_floats, po, obs_dim, obs_dim, blob, entropy_coef, red, norm_part);
}
__global__ void __launch_bounds__(256)
wl_ppo_reduce_asym_kernel(const float* __restrict__ rows, int nrows, int rowlen, int blob_floats, PolicyOffsets po, int obs_dim,
                          int critic_dim, const float* __restrict__ blob, float entropy_coef, float* __restrict__ red,
                          double* __restrict__ norm_part) {
    ppo_reduce_body(rows, nrows, rowlen, blob_floats, po, obs_dim, critic_dim, blob, entropy_coef, red, norm_part);
}

struct PpoStepArgs {
    float max_grad_norm, desired_kl, inv_B;
    int adaptive, update_index;
};

// One CTA: global norm -> clip coefficient, KL -> learning rate (before this step, as rsl_rl), statistics, then Adam on every
// parameter of the blob in place (padding entries are never touched).  DP: `red` is the row wl_ppo_dp_reduce_kernel wrote,
// whose KL column already holds the mean over the ranks of each rank's kl_mean; a nonzero exchange error word (a peer wait
// that timed out) leaves everything untouched.
template <bool DP>
__device__ __forceinline__ void ppo_step_body(float* __restrict__ blob, float* __restrict__ m, float* __restrict__ v, float* __restrict__ state,
                                              const float* __restrict__ red, const double* __restrict__ norm_part, int nparts,
                                              int blob_floats, const PolicyOffsets& po, int obs_dim, int critic_dim, const PpoStepArgs& a,
                                              const uint32_t* __restrict__ dp_error) {
    if constexpr (DP) {
        if (*(const volatile uint32_t*)dp_error) return;
    }
    __shared__ float s_coef, s_lr, s_bc1, s_bc2;
    if (threadIdx.x == 0) {
        double n2 = 0.0;
        for (int i = 0; i < nparts; ++i) n2 += norm_part[i];
        const float norm = (float)sqrt(n2);
        const float coef = fminf(a.max_grad_norm / (norm + 1e-6f), 1.0f);         // clip_grad_norm_: always applied
        const float kl = DP ? red[blob_floats + 2] : red[blob_floats + 2] * a.inv_B;
        float lr = state[0];
        if (a.adaptive) {
            if (kl > a.desired_kl * 2.0f) lr = fmaxf(1e-5f, lr / 1.5f);
            else if (kl < a.desired_kl / 2.0f && kl > 0.0f) lr = fminf(1e-2f, lr * 1.5f);
        }
        const float step = state[1] + 1.0f;
        const float s0 = blob[po.o[12]], s1 = blob[po.o[12] + 1];
        state[0] = lr; state[1] = step;
        state[6] += red[blob_floats] * a.inv_B;
        state[7] += red[blob_floats + 1] * a.inv_B;
        state[8] += (0.5f + WL_PPO_LOG_SQRT_2PI + logf(s0)) + (0.5f + WL_PPO_LOG_SQRT_2PI + logf(s1));
        state[9] = kl;
        if (a.update_index < WL_PPO_MAX_UPDATES) { state[10 + 2 * a.update_index] = kl; state[11 + 2 * a.update_index] = lr; }
        s_coef = coef; s_lr = lr;
        // torch forms 1 - beta^t and 1 - beta from the Python (double) betas; in fp32, 1 - 0.999f^t would lose ~1e-5
        s_bc1 = (float)(1.0 - pow(0.9, (double)step)); s_bc2 = (float)(1.0 - pow(0.999, (double)step));
    }
    __syncthreads();
    const float coef = s_coef, lr = s_lr, bc1 = s_bc1, bc2 = s_bc2;
    const float cb1 = (float)(1.0 - 0.9), cb2 = (float)(1.0 - 0.999);
    for (int c = threadIdx.x; c < blob_floats; c += WL_PPO_FIN_THREADS)
        if (ppo_is_param(c, po, obs_dim, critic_dim)) adam_update(blob, m, v, c, red[c] * coef, lr, 0.9f, cb1, 0.999f, cb2, 1e-8f, bc1, bc2);
}
template <bool DP>
__global__ void __launch_bounds__(WL_PPO_FIN_THREADS)
wl_ppo_step_kernel(float* __restrict__ blob, float* __restrict__ m, float* __restrict__ v, float* __restrict__ state,
                   const float* __restrict__ red, const double* __restrict__ norm_part, int nparts, int blob_floats,
                   PolicyOffsets po, int obs_dim, PpoStepArgs a, const uint32_t* __restrict__ dp_error) {
    ppo_step_body<DP>(blob, m, v, state, red, norm_part, nparts, blob_floats, po, obs_dim, obs_dim, a, dp_error);
}
__global__ void __launch_bounds__(WL_PPO_FIN_THREADS)
wl_ppo_step_asym_kernel(float* __restrict__ blob, float* __restrict__ m, float* __restrict__ v, float* __restrict__ state,
                        const float* __restrict__ red, const double* __restrict__ norm_part, int nparts, int blob_floats,
                        PolicyOffsets po, int obs_dim, int critic_dim, PpoStepArgs a) {
    ppo_step_body<false>(blob, m, v, state, red, norm_part, nparts, blob_floats, po, obs_dim, critic_dim, a, nullptr);
}

// Once per update: advantage mean and unbiased std over the whole batch (fp64, fixed order), old sigma snapshot, statistics reset.
__global__ void __launch_bounds__(WL_PPO_FIN_THREADS)
wl_ppo_begin_kernel(const float* __restrict__ adv, int n, const float* __restrict__ blob, int o_std, float* __restrict__ state) {
    __shared__ double sh[WL_PPO_FIN_THREADS];
    __shared__ double s_mean;
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += WL_PPO_FIN_THREADS) s += (double)adv[i];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int k = WL_PPO_FIN_THREADS / 2; k > 0; k >>= 1) {
        if (threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) s_mean = sh[0] / n;
    __syncthreads();
    const double mean = s_mean;
    s = 0.0;
    for (int i = threadIdx.x; i < n; i += WL_PPO_FIN_THREADS) { const double d = (double)adv[i] - mean; s += d * d; }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int k = WL_PPO_FIN_THREADS / 2; k > 0; k >>= 1) {
        if (threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        state[2] = blob[o_std]; state[3] = blob[o_std + 1];
        state[4] = (float)mean;
        state[5] = (float)sqrt(n > 1 ? sh[0] / (n - 1) : 0.0);
        state[6] = 0.0f; state[7] = 0.0f; state[8] = 0.0f; state[9] = 0.0f;
    }
}

// ---- data-parallel update (DESIGN 6j): every rank's reduced row averaged across ranks inside each mini-batch ----------
// Each rank owns an exchange buffer, symmetric across ranks (same layout, P2P-mapped or on one device): a 256-byte header
// (word 0: the rank's epoch, the number of rows it has published; word 1: its error word) and two slots of one reduced row
// each, mini-batch parity.  Per mini-batch: wl_ppo_reduce_kernel writes the rank's own reduced row into slot (k & 1) of its
// buffer, wl_ppo_dp_publish_kernel bumps the epoch, wl_ppo_dp_reduce_kernel waits for every rank's epoch to reach its own
// and averages the R slots into the rank's workspace row, and wl_ppo_step_kernel<true> steps on that average.
//
// Why two slots and one flag per mini-batch are enough: a rank overwrites its slot of mini-batch k + 2 (wl_ppo_reduce_kernel
// of k + 2) only after its DP reduce of k + 1 has passed the wait, i.e. after every peer published k + 1.  A peer publishes
// k + 1 after its reduce of k + 1, which its stream runs after its DP reduce of k -- its last read of anyone's slot of k.
// So nobody still reads the slot being overwritten.  This needs the parity to alternate across calls as well: a call with
// an odd number of mini-batches ends with one more publish / wait round that carries no row (wl_ppo_dp_wait_kernel).
#define WL_PPO_DP_HEADER 256
#define WL_PPO_DP_TIMEOUT_NS 60000000000ull       // 60 s: far beyond any rank skew of a healthy run (a checkpoint write included)

struct PpoExchange { int32_t n; int32_t pad; const char* buf[WL_MAX_PEERS]; };

__device__ __forceinline__ uint32_t ppo_ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t ppo_globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// One thread: bump this rank's epoch, a release store at system scope.  The reduce kernel before it on the stream wrote the
// slot; the fence makes those writes visible system-wide before the flag that a peer acquires over NVLink.
__global__ void wl_ppo_dp_publish_kernel(uint32_t* __restrict__ own) {
    const uint32_t e = *(volatile uint32_t*)own + 1u;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(own), "r"(e) : "memory");
}

// Wait until every rank's epoch has reached this rank's own (acquire loads at system scope), bounded by %globaltimer: on
// timeout, or if an earlier wait timed out, the rank's error word is set and false returned (no trap: the step kernel then
// skips, the host raises when it reads the error word back).
__device__ bool ppo_dp_wait(const PpoExchange& ex, uint32_t* own) {
    volatile uint32_t* err = own + 1;
    if (*err) return false;
    const uint32_t target = *(volatile uint32_t*)own;
    const uint64_t t0 = ppo_globaltimer();
    for (int r = 0; r < ex.n; ++r) {
        const uint32_t* e = reinterpret_cast<const uint32_t*>(ex.buf[r]);
        while ((int32_t)(ppo_ld_acquire_sys(e) - target) < 0) {
            if (ppo_globaltimer() - t0 > WL_PPO_DP_TIMEOUT_NS) { *err = 1u; __threadfence_system(); return false; }
            __nanosleep(256);
        }
    }
    return true;
}

// The no-row round that keeps the slot parity alternating across calls with an odd number of mini-batches.
__global__ void wl_ppo_dp_wait_kernel(const __grid_constant__ PpoExchange ex, uint32_t* __restrict__ own) { ppo_dp_wait(ex, own); }

// One CTA per 256 columns, as wl_ppo_reduce_kernel: column c of `red` = (sum over ranks 0..R-1 of slot c) / R for the
// parameters, in rank order on every rank (so every replica forms the same bits); the fp64 sum of squares of the averaged
// parameter columns per block (tree in thread order); the KL column = (sum_r kl_mean_r) / R with kl_mean_r = slot_r[KL] *
// inv_B; the surrogate / value-loss columns stay this rank's own (rsl_rl reduces neither).
__global__ void __launch_bounds__(256)
wl_ppo_dp_reduce_kernel(const __grid_constant__ PpoExchange ex, uint32_t* __restrict__ own, size_t slot_off, int rowlen,
                        int blob_floats, PolicyOffsets po, int obs_dim, float inv_B, float* __restrict__ red,
                        double* __restrict__ norm_part) {
    __shared__ double sq[256];
    __shared__ int s_ok;
    if (threadIdx.x == 0) {
        s_ok = ppo_dp_wait(ex, own);
        __threadfence_system();
    }
    __syncthreads();
    if (!s_ok) return;
    const int c = blockIdx.x * 256 + threadIdx.x;
    const bool param = c < blob_floats && ppo_is_param(c, po, obs_dim, obs_dim);
    const float rn = (float)ex.n;
    float g = 0.0f;
    if (param) {
        for (int r = 0; r < ex.n; ++r) g += __ldcg(reinterpret_cast<const float*>(ex.buf[r] + slot_off) + c);
        g = g / rn;
    } else if (c == blob_floats + 2) {
        for (int r = 0; r < ex.n; ++r) g += __ldcg(reinterpret_cast<const float*>(ex.buf[r] + slot_off) + c) * inv_B;
        g = g / rn;
    } else if (c >= blob_floats && c < blob_floats + WL_PPO_STATS) {
        g = reinterpret_cast<const float*>(reinterpret_cast<const char*>(own) + slot_off)[c];
    }
    if (c < rowlen) red[c] = g;
    sq[threadIdx.x] = param ? (double)g * (double)g : 0.0;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) sq[threadIdx.x] += sq[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) norm_part[blockIdx.x] = sq[0];
}
