// wl_distill.cuh -- rsl_rl's Distillation.update() for the student actor (DESIGN 6t), included by wl_api.cu after
// wl_actor.cuh (it reuses mlp_tile_*, ppo_elu / relu, the cp.async and bulk-copy helpers and adam_update).
//
// Behaviour cloning: the loss of one stored step is mse(student(obs_t), teacher_action_t), the mean over N x 2 elements,
// and every gradient_length steps the summed loss is back-propagated through the actor and Adam steps the actor alone.
// Per chunk of gradient_length steps (its rows are whole slab steps, no permutation):
//   wl_distill_fwd_kernel      ReLU network: H1 = relu(X W1 + b1) of the chunk's rows, actor only -> workspace
//   wl_distill_grad_kernel     the actor forward (ELU: layer 1 too), the MSE head gradient (mu - a*) / N, back-propagation,
//                              every actor gradient entry but the ReLU network's dW1 in registers (one row per CTA); the
//                              per-row squared errors -> workspace
//   wl_distill_dw1_kernel      ReLU network: dW1 = X^T dZ1, split over samples as the grad kernel's CTAs
//   wl_distill_loss_kernel     each step's loss (fp64 sum over its N rows, fixed order)
//   wl_distill_reduce_kernel   rows summed in CTA order per actor column, fp64 block sums of squares
//   wl_distill_step_kernel     the optional clip_grad_norm_, then Adam on the actor's parameters only
// The critic blocks, the std and every padding float are never read for the loss and never stepped.  No float atomics.
#pragma once

#define WL_DS_THREADS 256
#define WL_DS_TILE 64                             // samples per tile: 8 warps x (2 half-warps x 4 samples), actor only
#define WL_DS_XS 20                               // padded observation row of the ELU network (obs_dim <= 16)
#define WL_DS_HS (WL_HID + 4)                     // padded hidden row
#define WL_DS_SD 4                                // per-sample row: dL/dmu0, dL/dmu1
#define WL_DS_FWD_THREADS 128                     // wl_actor_mean's geometry: 4 warps x (2 half-warps x 4 rows), 32 rows
#define WL_DS_FWD_STAGE (WL_AM_ROWS * WL_AM_XS + WL_WIDE_KC * WL_HID)
#define WL_DS_FIN_THREADS 1024
#define WL_DS_STATE_HEAD 4                        // d_state: lr, Adam steps, mean loss, optimizer steps of the last update

struct DistillArgs {
    const float* obs;                             // [T, N, D] slab order
    const float* target;                          // [T, N, 2] the teacher's actions
    float* sqerr;                                 // [B] per-row squared error of the chunk (workspace)
    int D, N, T, B, step0, tiles;                 // B = rows of the chunk; step0 = its first step's index (mod T: epochs repeat)
    float inv_N;
};

// chunk row r -> slab row: the chunk's step j = r / N is slab step (step0 + j) mod T
__device__ __forceinline__ int64_t distill_row(const DistillArgs& a, int r) {
    const int j = r / a.N, n = r - j * a.N;
    return (int64_t)((a.step0 + j) % a.T) * a.N + n;
}

// is blob float c a parameter of the actor (not padding, not a zero row of W1t)?
__device__ __forceinline__ bool distill_is_actor_param(int c, const PolicyOffsets& po, int D) {
    const int len[6] = {D * WL_HID, WL_HID, WL_HID * WL_HID, WL_HID, WL_HID * 2, 2};
    bool p = false;
#pragma unroll
    for (int k = 0; k < 6; ++k) p |= (c >= po.o[k] && c < po.o[k] + len[k]);
    return p;
}

__device__ __forceinline__ void distill_store_elu(float* h0, const float acc[4][4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
        *reinterpret_cast<float4*>(h0 + e * WL_DS_HS) = make_float4(ppo_elu(acc[e][0]), ppo_elu(acc[e][1]), ppo_elu(acc[e][2]), ppo_elu(acc[e][3]));
}

// ---- the ReLU network's layer 1: wl_actor_mean's K-chunked sums over the chunk's rows --------------------------------
__device__ __forceinline__ void distill_stage(float* sb, const float* __restrict__ x, int D, const int64_t* srow,
                                              const float* __restrict__ W1t, int k0, int kn) {
    for (int k = threadIdx.x; k < WL_AM_ROWS * WL_WIDE_KC; k += WL_DS_FWD_THREADS) {
        const int r = k / WL_WIDE_KC, j = k % WL_WIDE_KC, col = k0 + j;
        const int64_t row = srow[r];
        const bool ok = row >= 0 && col < D;
        cp_async4(sb + r * WL_AM_XS + j, ok ? x + row * D + col : x, ok);
    }
    float* sw = sb + WL_AM_ROWS * WL_AM_XS;
    for (int k = threadIdx.x; k < kn * (WL_HID / 4); k += WL_DS_FWD_THREADS)
        cp_async16(sw + k * 4, W1t + (size_t)k0 * WL_HID + k * 4);
}

// H1[r] = relu(b1 + X[row(r)] W1) for the chunk's rows r (rows past B: relu(b1), never used), [tiles * 64][64]
__global__ void __launch_bounds__(WL_DS_FWD_THREADS)
wl_distill_fwd_kernel(const float* __restrict__ blob, PolicyOffsets po, const __grid_constant__ DistillArgs a, float* __restrict__ H1) {
    extern __shared__ __align__(128) float smem[];           // 2 x WL_DS_FWD_STAGE
    __shared__ int64_t srow[WL_AM_ROWS];
    const int tid = threadIdx.x, r0 = blockIdx.x * WL_AM_ROWS;
    if (tid < WL_AM_ROWS) srow[tid] = r0 + tid < a.B ? distill_row(a, r0 + tid) : -1;
    __syncthreads();
    const int lane = tid & 31, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 8 + (lane >> 4) * 4;
    const int nin1 = (a.D + 3) & ~3, nch = (nin1 + WL_WIDE_KC - 1) / WL_WIDE_KC;
    const float* W1t = blob + po.o[0];
    float acc[4][4];
    const float4 b0 = *reinterpret_cast<const float4*>(blob + po.o[1] + ucol);
#pragma unroll
    for (int e = 0; e < 4; ++e) { acc[e][0] = b0.x; acc[e][1] = b0.y; acc[e][2] = b0.z; acc[e][3] = b0.w; }
    distill_stage(smem, a.obs, a.D, srow, W1t, 0, min(WL_WIDE_KC, nin1));
    cp_async_commit();
    for (int c = 0; c < nch; ++c) {
        if (c + 1 < nch) {
            const int k1 = (c + 1) * WL_WIDE_KC;
            distill_stage(smem + ((c + 1) & 1) * WL_DS_FWD_STAGE, a.obs, a.D, srow, W1t, k1, min(WL_WIDE_KC, nin1 - k1));
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();                                     // chunk c is in shared memory for every thread
        const float* sb = smem + (c & 1) * WL_DS_FWD_STAGE;
        float part[4][4];
#pragma unroll
        for (int e = 0; e < 4; ++e) { part[e][0] = 0.0f; part[e][1] = 0.0f; part[e][2] = 0.0f; part[e][3] = 0.0f; }
        mlp_tile_accum(sb + WL_AM_ROWS * WL_AM_XS + ucol, sb + env0 * WL_AM_XS, WL_AM_XS, min(WL_WIDE_KC, nin1 - c * WL_WIDE_KC), part);
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[e][q] += part[e][q];
        __syncthreads();                                     // every thread is done with the buffer the next chunk refills
    }
    store_relu(H1 + (size_t)(r0 + env0) * WL_HID + ucol, WL_HID, acc);
}

// ---- the gradient of one chunk ---------------------------------------------------------------------------------------
// Persistent CTAs: CTA b takes tiles b, b + grid, ... of 64 samples; thread t owns fixed actor gradient entries for the
// CTA's whole lifetime, summed over the samples in order, and writes them into its row of the workspace (blob layout).
// RELU: layer 1 comes from H1 and its dZ1 goes to the workspace for wl_distill_dw1_kernel; else (ELU) layer 1 and dW1 are
// computed here.  The forward sums in wl_actor_mean's order; the ELU is torch's (expm1), as in wl_ppo_grad_kernel.
template <bool RELU>
__global__ void __launch_bounds__(WL_DS_THREADS, 1)
wl_distill_grad_kernel(const float* __restrict__ blob, PolicyOffsets po, const __grid_constant__ DistillArgs a,
                       const float* __restrict__ H1, float* __restrict__ dZ1, float* __restrict__ rows, int rowlen) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    const int base = RELU ? po.o[1] : 0;                     // the actor from W1t (ELU) or from b1 (ReLU) up to the critic
    const int nact = po.o[6] - base;
    float* sw = smem;
    float* sw2t = sw + nact;                                 // [64 out][64 in]: W2 output-major, for dh1 = dz2 W2
    float* szero = sw2t + WL_HID * WL_HID;                   // the zero "bias" of the backward layer
    float* sx = szero + WL_HID;                              // [64][XS] (ELU)
    float* sh1 = sx + (RELU ? 0 : WL_DS_TILE * WL_DS_XS);    // [64][HS] layer-1 activations
    float* sh2 = sh1 + WL_DS_TILE * WL_DS_HS;                // layer-2 activations
    float* sg2 = sh2 + WL_DS_TILE * WL_DS_HS;                // dL/dz2
    float* sg1 = sg2 + WL_DS_TILE * WL_DS_HS;                // dL/dz1
    float* sd = sg1 + WL_DS_TILE * WL_DS_HS;                 // [64][SD]
    const int tid = threadIdx.x, D = a.D;
    if (tid == 0) {
        mbar_init(&mbar, 1);
        mbar_init_fence();
        mbar_expect(&mbar, (uint32_t)nact * 4u);
        bulk_g2s(sw, blob + base, (uint32_t)nact * 4u, &mbar);
    }
    if (tid < WL_HID) szero[tid] = 0.0f;
    __syncthreads();
    mbar_wait_parity(&mbar, 0);
    const int oW1 = po.o[0] - base, oB1 = po.o[1] - base, oW2 = po.o[2] - base, oB2 = po.o[3] - base;
    const int oW3 = po.o[4] - base, oB3 = po.o[5] - base;
    for (int k = tid; k < WL_HID * WL_HID; k += WL_DS_THREADS) {
        const int u = k >> 6, i = k & (WL_HID - 1);
        sw2t[k] = sw[oW2 + i * WL_HID + u];
    }
    // gradient entries this thread owns
    const int i2 = (tid >> 4) * 4, u2 = (tid & 15) * 4;      // dW2t rows i2..i2+3, cols u2..u2+3
    const int i1 = tid >> 4;                                 // dW1t row i1 (ELU), cols u2..u2+3
    float gW2[4][4], gW1[4], gb = 0.0f, gd = 0.0f;           // gb: db1 / db2 (tid < 128) or dW3t (tid >= 128); gd: db3 (tid < 2)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        gW1[k] = 0.0f;
#pragma unroll
        for (int q = 0; q < 4; ++q) gW2[k][q] = 0.0f;
    }
    const int lane = tid & 31, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 8 + (lane >> 4) * 4, nin1 = (D + 3) & ~3;
    __syncthreads();                                         // sw2t complete

    for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
        const int s0 = tile * WL_DS_TILE;
        if constexpr (RELU) {
            for (int k = tid; k < WL_DS_TILE * (WL_HID / 4); k += WL_DS_THREADS) {
                const int s = k >> 4, q = k & 15;
                *reinterpret_cast<float4*>(sh1 + s * WL_DS_HS + 4 * q) = *reinterpret_cast<const float4*>(H1 + (size_t)(s0 + s) * WL_HID + 4 * q);
            }
        } else {
            for (int k = tid; k < WL_DS_TILE * 16; k += WL_DS_THREADS) {
                const int s = k >> 4, j = k & 15, row = s0 + s;
                float x = 0.0f;
                if (row < a.B && j < D) x = a.obs[distill_row(a, row) * D + j];
                sx[s * WL_DS_XS + j] = x;
            }
        }
        __syncthreads();
        {
            float acc[4][4];
            float* h1 = sh1 + env0 * WL_DS_HS;
            if constexpr (!RELU) {
                mlp_tile_layer(sw + oW1 + ucol, sw + oB1 + ucol, sx + env0 * WL_DS_XS, WL_DS_XS, nin1, acc);
                distill_store_elu(h1 + ucol, acc);
                __syncwarp();
            }
            mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, h1, WL_DS_HS, WL_HID, acc);
            if constexpr (RELU) store_relu(sh2 + env0 * WL_DS_HS + ucol, WL_DS_HS, acc);
            else distill_store_elu(sh2 + env0 * WL_DS_HS + ucol, acc);
        }
        __syncthreads();
        {   // head (wl_actor_mean's butterflies): the MSE derivative and the squared error of each sample
            const float* w3a = sw + oW3;
            constexpr int P = RELU ? 8 : 4, U = WL_HID / P;
#pragma unroll
            for (int pass = 0; pass < (RELU ? 2 : 1); ++pass) {
                const int s = pass * (WL_DS_THREADS / P) + tid / P, p = tid % P, row = s0 + s;
                const float* hrow = sh2 + s * WL_DS_HS;
                float m0 = 0.0f, m1 = 0.0f;
#pragma unroll
                for (int k = 0; k < U; ++k) {
                    const int j = U * p + k;
                    m0 = fmaf(w3a[2 * j], hrow[j], m0); m1 = fmaf(w3a[2 * j + 1], hrow[j], m1);
                }
#pragma unroll
                for (int x = 1; x < P; x <<= 1) {
                    m0 += __shfl_xor_sync(0xffffffffu, m0, x); m1 += __shfl_xor_sync(0xffffffffu, m1, x);
                }
                if (p == 0) {
                    float* d = sd + s * WL_DS_SD;
                    if (row < a.B) {
                        const float2 t = reinterpret_cast<const float2*>(a.target)[distill_row(a, row)];
                        const float e0 = (m0 + sw[oB3]) - t.x, e1 = (m1 + sw[oB3 + 1]) - t.y;
                        d[0] = e0 * a.inv_N;                 // d/dmu of mse over N x 2 elements: 2 (mu - a*) / (2 N)
                        d[1] = e1 * a.inv_N;
                        a.sqerr[row] = e0 * e0 + e1 * e1;
                    } else {
                        d[0] = 0.0f; d[1] = 0.0f;            // tail of a partial tile: no gradient
                    }
                }
            }
        }
        __syncthreads();
        for (int k = tid; k < WL_DS_TILE * WL_HID; k += WL_DS_THREADS) {   // dz2 = (dmu W3) * act'(h2)
            const int s = k >> 6, c = k & (WL_HID - 1);
            const float* d = sd + s * WL_DS_SD;
            const float dh = d[0] * sw[oW3 + 2 * c] + d[1] * sw[oW3 + 2 * c + 1];
            const float h = sh2[s * WL_DS_HS + c];
            sg2[s * WL_DS_HS + c] = RELU ? (h > 0.0f ? dh : 0.0f) : dh * ppo_elu_grad(h);
        }
        __syncthreads();
        {   // dz1 = (dz2 W2) * act'(h1): the forward layer routine on the output-major copy of W2, zero bias
            float acc[4][4];
            mlp_tile_layer(sw2t + ucol, szero + ucol, sg2 + env0 * WL_DS_HS, WL_DS_HS, WL_HID, acc);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int o = (env0 + e) * WL_DS_HS + ucol;
                const float4 h = *reinterpret_cast<const float4*>(sh1 + o);
                float4 g;
                if constexpr (RELU) {
                    g = make_float4(h.x > 0.0f ? acc[e][0] : 0.0f, h.y > 0.0f ? acc[e][1] : 0.0f,
                                    h.z > 0.0f ? acc[e][2] : 0.0f, h.w > 0.0f ? acc[e][3] : 0.0f);
                    *reinterpret_cast<float4*>(dZ1 + (size_t)(s0 + env0 + e) * WL_HID + ucol) = g;
                } else {
                    g = make_float4(acc[e][0] * ppo_elu_grad(h.x), acc[e][1] * ppo_elu_grad(h.y),
                                    acc[e][2] * ppo_elu_grad(h.z), acc[e][3] * ppo_elu_grad(h.w));
                }
                *reinterpret_cast<float4*>(sg1 + o) = g;
            }
        }
        __syncthreads();
        // accumulate the weight gradients over the tile's samples, in sample order
        for (int s = 0; s < WL_DS_TILE; ++s) {
            const float* h1 = sh1 + s * WL_DS_HS;
            const float* g2 = sg2 + s * WL_DS_HS;
            const float* g1 = sg1 + s * WL_DS_HS;
            const float4 hv = *reinterpret_cast<const float4*>(h1 + i2);
            const float4 gv = *reinterpret_cast<const float4*>(g2 + u2);
            const float hk[4] = {hv.x, hv.y, hv.z, hv.w}, gq[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int q = 0; q < 4; ++q) gW2[k][q] = fmaf(hk[k], gq[q], gW2[k][q]);
            if constexpr (!RELU) {
                const float xv = sx[s * WL_DS_XS + i1];
                const float4 dz = *reinterpret_cast<const float4*>(g1 + u2);
                gW1[0] = fmaf(xv, dz.x, gW1[0]); gW1[1] = fmaf(xv, dz.y, gW1[1]);
                gW1[2] = fmaf(xv, dz.z, gW1[2]); gW1[3] = fmaf(xv, dz.w, gW1[3]);
            }
            const float* d = sd + s * WL_DS_SD;
            if (tid < WL_HID) gb += g1[tid];
            else if (tid < 2 * WL_HID) gb += g2[tid - WL_HID];
            else gb = fmaf(sh2[s * WL_DS_HS + ((tid - 2 * WL_HID) >> 1)], d[tid & 1], gb);
            if (tid < 2) gd += d[tid];
        }
        __syncthreads();                                     // the next tile overwrites the shared rows
    }

    float* row = rows + (size_t)blockIdx.x * rowlen;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        *reinterpret_cast<float4*>(row + po.o[2] + (i2 + k) * WL_HID + u2) = make_float4(gW2[k][0], gW2[k][1], gW2[k][2], gW2[k][3]);
    if (!RELU && i1 < D) *reinterpret_cast<float4*>(row + po.o[0] + i1 * WL_HID + u2) = make_float4(gW1[0], gW1[1], gW1[2], gW1[3]);
    if (tid < WL_HID) row[po.o[1] + tid] = gb;               // db1
    else if (tid < 2 * WL_HID) row[po.o[3] + tid - WL_HID] = gb;     // db2
    else row[po.o[4] + tid - 2 * WL_HID] = gb;               // dW3t, [unit][action]
    if (tid < 2) row[po.o[5] + tid] = gd;                    // db3
}

// dW1t[k][u] = sum over the chunk's samples of X[row(s)][k] dZ1[s][u].  Block (kt, split) owns W1t rows 64 kt .. 64 kt + 63
// and the samples of tiles split, split + gridDim.y, ... (the grad kernel's tiles), summed in sample order; it writes its
// partial into gradient row `split`.  Thread: 4 rows x 4 columns.
__global__ void __launch_bounds__(WL_DS_THREADS)
wl_distill_dw1_kernel(PolicyOffsets po, const __grid_constant__ DistillArgs a, const float* __restrict__ dZ1, float* __restrict__ rows,
                      int rowlen) {
    extern __shared__ __align__(128) float smem[];           // 2 stages of [64][64] X | [64][64] dZ1
    constexpr int XF = WL_DS_TILE * WL_DW1_K, SF = XF + WL_DS_TILE * WL_HID;
    const int tid = threadIdx.x, D = a.D, k0 = blockIdx.x * WL_DW1_K;
    const int tk = (tid >> 4) * 4, tu = (tid & 15) * 4;
    auto stage = [&](float* sb, int tile) {
        const int s0 = tile * WL_DS_TILE;
        for (int k = tid; k < XF; k += WL_DS_THREADS) {
            const int s = k / WL_DW1_K, j = k % WL_DW1_K, col = k0 + j;
            const bool ok = s0 + s < a.B && col < D;
            const float* src = ok ? a.obs + distill_row(a, s0 + s) * D + col : a.obs;
            cp_async4(sb + k, src, ok);
        }
        for (int k = tid; k < WL_DS_TILE * (WL_HID / 4); k += WL_DS_THREADS)
            cp_async16(sb + XF + 4 * k, dZ1 + (size_t)s0 * WL_HID + 4 * k);
    };
    float g[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 4; ++q) g[k][q] = 0.0f;
    int it = 0;
    stage(smem, blockIdx.y);
    cp_async_commit();
    for (int tile = blockIdx.y; tile < a.tiles; tile += gridDim.y, ++it) {
        if (tile + (int)gridDim.y < a.tiles) {
            stage(smem + ((it + 1) & 1) * SF, tile + gridDim.y);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float* sx = smem + (it & 1) * SF;
        const float* sz = sx + XF;
        for (int s = 0; s < WL_DS_TILE; ++s) {
            const float4 xv = *reinterpret_cast<const float4*>(sx + s * WL_DW1_K + tk);
            const float4 zv = *reinterpret_cast<const float4*>(sz + s * WL_HID + tu);
            const float xk[4] = {xv.x, xv.y, xv.z, xv.w}, zq[4] = {zv.x, zv.y, zv.z, zv.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int q = 0; q < 4; ++q) g[k][q] = fmaf(xk[k], zq[q], g[k][q]);
        }
        __syncthreads();
    }
    float* row = rows + (size_t)blockIdx.y * rowlen + po.o[0] + tu;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (k0 + tk + k < D) *reinterpret_cast<float4*>(row + (size_t)(k0 + tk + k) * WL_HID) = make_float4(g[k][0], g[k][1], g[k][2], g[k][3]);
}

// one CTA per step j of the chunk: loss of step k0 + j = (sum over its N rows of the squared errors, fp64, tree in thread
// order) / (2 N) -> state[WL_DS_STATE_HEAD + k0 + j]
__global__ void __launch_bounds__(256)
wl_distill_loss_kernel(const float* __restrict__ sqerr, int N, int k0, float* __restrict__ state) {
    __shared__ double sh[256];
    double s = 0.0;
    for (int n = threadIdx.x; n < N; n += 256) s += (double)sqerr[(size_t)blockIdx.x * N + n];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) sh[threadIdx.x] += sh[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) state[WL_DS_STATE_HEAD + k0 + blockIdx.x] = (float)(sh[0] / (2.0 * N));
}

// column c of the reduced row = sum of the CTAs' rows in CTA order (actor parameters only; every other column 0); each
// block also writes the fp64 sum of squares of its columns (tree in thread order)
__global__ void __launch_bounds__(256)
wl_distill_reduce_kernel(const float* __restrict__ rows, int nrows, int rowlen, PolicyOffsets po, int D, float* __restrict__ red,
                         double* __restrict__ norm_part) {
    __shared__ double sq[256];
    const int c = blockIdx.x * 256 + threadIdx.x;
    const bool param = c < rowlen && distill_is_actor_param(c, po, D);
    float g = 0.0f;
    if (param)
        for (int r = 0; r < nrows; ++r) g += rows[(size_t)r * rowlen + c];
    if (c < rowlen) red[c] = g;
    sq[threadIdx.x] = param ? (double)g * (double)g : 0.0;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) sq[threadIdx.x] += sq[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) norm_part[blockIdx.x] = sq[0];
}

// One CTA: the global norm -> clip_grad_norm_'s coefficient (max_grad_norm > 0; else no clip), then Adam (0.9, 0.999, 1e-8,
// the fixed learning rate state[0]) on every actor parameter of the blob in place
__global__ void __launch_bounds__(WL_DS_FIN_THREADS)
wl_distill_step_kernel(float* __restrict__ blob, float* __restrict__ m, float* __restrict__ v, float* __restrict__ state,
                       const float* __restrict__ red, const double* __restrict__ norm_part, int nparts, PolicyOffsets po, int D,
                       float max_grad_norm) {
    __shared__ float s_coef, s_lr, s_bc1, s_bc2;
    if (threadIdx.x == 0) {
        float coef = 1.0f;
        if (max_grad_norm > 0.0f) {
            double n2 = 0.0;
            for (int i = 0; i < nparts; ++i) n2 += norm_part[i];
            coef = fminf(max_grad_norm / ((float)sqrt(n2) + 1e-6f), 1.0f);
        }
        const float step = state[1] + 1.0f;
        state[1] = step;
        s_coef = coef; s_lr = state[0];
        s_bc1 = (float)(1.0 - pow(0.9, (double)step)); s_bc2 = (float)(1.0 - pow(0.999, (double)step));
    }
    __syncthreads();
    const float coef = s_coef, lr = s_lr, bc1 = s_bc1, bc2 = s_bc2;
    const float cb1 = (float)(1.0 - 0.9), cb2 = (float)(1.0 - 0.999);
    for (int c = threadIdx.x; c < po.o[6]; c += WL_DS_FIN_THREADS)
        if (distill_is_actor_param(c, po, D)) adam_update(blob, m, v, c, red[c] * coef, lr, 0.9f, cb1, 0.999f, cb2, 1e-8f, bc1, bc2);
}

// Once per update, after the last chunk: state[2] = the mean of the update's n_losses per-step losses (fp64, in order),
// state[3] = the number of Adam steps it took
__global__ void wl_distill_finish_kernel(float* __restrict__ state, int n_losses, int n_steps) {
    double s = 0.0;
    for (int i = 0; i < n_losses; ++i) s += (double)state[WL_DS_STATE_HEAD + i];
    state[2] = (float)(s / n_losses);
    state[3] = (float)n_steps;
}
