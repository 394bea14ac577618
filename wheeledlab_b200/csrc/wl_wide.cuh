// wl_wide.cuh -- the actor-critic for wide observations (DESIGN 6g): obs -> 64 -> 64 -> (2 | 1) ReLU MLPs in the blob
// layout of wl_act_step, for any obs_dim up to 4096.  Included by wl_api.cu after wl_ppo.cuh (it reuses mlp_tile_*, the
// Gaussian head, the bulk copies, PpoArgs / ppo_sample_derivs and the PPO reduce / step kernels).
//
// Layer 1 ([rows x obs_dim] . [obs_dim x 128], actor and critic side by side) is the one part whose weights do not fit in
// shared memory: it runs as a K-chunked FP32 SGEMM on tiles of 32 rows (wide_layer1), W1t and the observation rows staged
// chunk by chunk with cp.async (two stages).  Everything after layer 1 uses the blob minus its two W1t blocks, held in
// shared memory in a compact layout (compact offsets: wide_compact_offsets on the host).
//   wl_policy_act_kernel       the rollout's policy: layer 1, layer 2, heads, Gaussian sample -> wl_policy_out
//   wl_ppo_wide_fwd_kernel     PPO: H1 = relu(X[perm] W1 + b1) of a mini-batch -> workspace
//   wl_ppo_wide_grad_kernel    PPO: layers 2-3, the loss derivatives, back-propagation to dZ1 -> workspace; dW2, dW3, the
//                              heads, db1, dsigma and the loss sums in registers (one gradient row per CTA, as 6f)
//   wl_ppo_wide_dw1_kernel     PPO: dW1 = X[perm]^T dZ1, split over samples: split s writes gradient row s
// then wl_ppo_reduce_kernel and wl_ppo_step_kernel as for the narrow network.  No float atomics: every sum has a fixed order.
// The asymmetric network (DESIGN 6s) has the critic's layer 1 over a row of its own: wl_policy_act_wide_asym_kernel,
// wl_ppo_wide_fwd_asym_kernel and wl_ppo_wide_dw1_asym_kernel are the kernels above with that second input (the grad
// kernel is shared), followed by the asymmetric reduce and step kernels.
#pragma once

#define WL_WIDE_ROWS 32                           // rows per layer-1 tile (8 warps x 4 rows in the mlp_tile_layer geometry)
#define WL_WIDE_KC 32                             // inputs per staged chunk of layer 1
#define WL_WIDE_XS (WL_WIDE_KC + 4)               // padded staged observation row
#define WL_WIDE_STAGE (WL_WIDE_ROWS * WL_WIDE_XS + 2 * WL_WIDE_KC * WL_HID)     // floats per stage: x rows | W1t actor | W1t critic
#define WL_WIDE_STAGE_ASYM (2 * WL_WIDE_ROWS * WL_WIDE_XS + 2 * WL_WIDE_KC * WL_HID)   // actor rows | critic rows | W1t actor | W1t critic
#define WL_WIDE_THREADS 256
#define WL_WIDE_MAX_OBS 4096
#define WL_DW1_K 64                               // W1t rows per dW1 tile (x 128 columns of both nets)

__device__ __forceinline__ void cp_async4(void* dst, const void* src, bool ok) {      // !ok: zero-fill, nothing read
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(ok ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float relu(float x) { return x > 0.0f ? x : 0.0f; }

// stage inputs k0 .. k0 + kn - 1 (kn a multiple of 4, k0 + kn <= ceil4(D)) of layer 1: the 32 rows' observations (zero past
// D and for rows < 0) and both nets' W1t rows
__device__ __forceinline__ void wide_stage(float* sb, const float* __restrict__ x, int D, const int64_t* srow,
                                           const float* __restrict__ blob, int oWa, int oWc, int k0, int kn) {
    for (int k = threadIdx.x; k < WL_WIDE_ROWS * WL_WIDE_KC; k += WL_WIDE_THREADS) {
        const int r = k / WL_WIDE_KC, j = k % WL_WIDE_KC, col = k0 + j;
        const int64_t row = srow[r];
        const bool ok = row >= 0 && col < D;
        cp_async4(sb + r * WL_WIDE_XS + j, ok ? x + row * D + col : x, ok);
    }
    float* sw = sb + WL_WIDE_ROWS * WL_WIDE_XS;
    const int per_net = kn * (WL_HID / 4);
    for (int k = threadIdx.x; k < 2 * per_net; k += WL_WIDE_THREADS) {
        const int net = k >= per_net, q = k - net * per_net;
        cp_async16(sw + net * WL_WIDE_KC * WL_HID + q * 4, blob + (net ? oWc : oWa) + (size_t)k0 * WL_HID + q * 4);
    }
}
// the asymmetric stage (WL_WIDE_STAGE_ASYM floats: actor rows | critic rows | W1t actor | W1t critic): net `net` stages its
// rows and kn[net] W1t rows from its own input; a net with kn <= 0 (past its last chunk) stages nothing
__device__ __forceinline__ void wide_stage_asym(float* sb, const float* __restrict__ x, int D, const float* __restrict__ xc, int Dc,
                                                const int64_t* srow, const float* __restrict__ blob, int oWa, int oWc, int k0,
                                                int kna, int knc) {
#pragma unroll
    for (int net = 0; net < 2; ++net) {
        const float* xs = net ? xc : x;
        const int Dn = net ? Dc : D, kn = net ? knc : kna;
        if (kn <= 0) continue;
        for (int k = threadIdx.x; k < WL_WIDE_ROWS * WL_WIDE_KC; k += WL_WIDE_THREADS) {
            const int r = k / WL_WIDE_KC, j = k % WL_WIDE_KC, col = k0 + j;
            const int64_t row = srow[r];
            const bool ok = row >= 0 && col < Dn;
            cp_async4(sb + (net * WL_WIDE_ROWS + r) * WL_WIDE_XS + j, ok ? xs + row * Dn + col : xs, ok);
        }
        float* sw = sb + 2 * WL_WIDE_ROWS * WL_WIDE_XS + net * WL_WIDE_KC * WL_HID;
        const float* w = blob + (net ? oWc : oWa) + (size_t)k0 * WL_HID;
        for (int q = threadIdx.x; q < kn * (WL_HID / 4); q += WL_WIDE_THREADS) cp_async16(sw + q * 4, w + q * 4);
    }
}

// layer 1 (pre-activation) of both nets for the 32 rows srow[] of x (-1: a zero row), in the mlp_tile_layer geometry: warp w
// takes rows 4w..4w+3, lane = (net, 4 units).  Each K chunk is summed on its own (inputs ascending) and added to the running
// sum, which starts at the bias: two-level summation keeps the rounding error of a 689-long (3208-long) dot product near
// that of torch's blocked sums.  `stage`: 2 * WL_WIDE_STAGE floats of shared memory (ASYM: 2 * WL_WIDE_STAGE_ASYM).  Ends
// with a __syncthreads.
// ASYM (DESIGN 6s): the critic's inputs are xc [.., Dc] instead of x.  Each net keeps its own chunks of 32 from input 0,
// so a net's sums are those of the symmetric layer on its own input; a net that has run out of chunks adds nothing (not
// zeros: -0 + 0 is +0).
template <bool ASYM = false>
__device__ __forceinline__ void wide_layer1(const float* __restrict__ x, int D, const int64_t* srow, const float* __restrict__ blob,
                                            const PolicyOffsets& po, float* stage, float acc[4][4],
                                            const float* __restrict__ xc = nullptr, int Dc = 0) {
    constexpr int STAGE = ASYM ? WL_WIDE_STAGE_ASYM : WL_WIDE_STAGE;
    const int lane = threadIdx.x & 31, net = lane >> 4, ucol = (lane & 15) * 4, env0 = (threadIdx.x >> 5) * 4;
    const int nina = (D + 3) & ~3, ninc = ASYM ? (Dc + 3) & ~3 : nina;
    const int nin1 = max(nina, ninc), nch = (nin1 + WL_WIDE_KC - 1) / WL_WIDE_KC, ninn = net ? ninc : nina;
    const float4 b0 = *reinterpret_cast<const float4*>(blob + (net ? po.o[7] : po.o[1]) + ucol);
#pragma unroll
    for (int e = 0; e < 4; ++e) { acc[e][0] = b0.x; acc[e][1] = b0.y; acc[e][2] = b0.z; acc[e][3] = b0.w; }
    if (ASYM) wide_stage_asym(stage, x, D, xc, Dc, srow, blob, po.o[0], po.o[6], 0, min(WL_WIDE_KC, nina), min(WL_WIDE_KC, ninc));
    else wide_stage(stage, x, D, srow, blob, po.o[0], po.o[6], 0, min(WL_WIDE_KC, nin1));
    cp_async_commit();
    for (int c = 0; c < nch; ++c) {
        if (c + 1 < nch) {
            const int k1 = (c + 1) * WL_WIDE_KC;
            if (ASYM) wide_stage_asym(stage + ((c + 1) & 1) * STAGE, x, D, xc, Dc, srow, blob, po.o[0], po.o[6], k1,
                                      min(WL_WIDE_KC, nina - k1), min(WL_WIDE_KC, ninc - k1));
            else wide_stage(stage + ((c + 1) & 1) * STAGE, x, D, srow, blob, po.o[0], po.o[6], k1, min(WL_WIDE_KC, nin1 - k1));
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();                                     // chunk c is in shared memory for every thread
        const float* sb = stage + (c & 1) * STAGE;
        const int kn = min(WL_WIDE_KC, ninn - c * WL_WIDE_KC);
        if (!ASYM || kn > 0) {
            const int xoff = ASYM ? (net * WL_WIDE_ROWS + env0) * WL_WIDE_XS : env0 * WL_WIDE_XS;
            float part[4][4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { part[e][0] = 0.0f; part[e][1] = 0.0f; part[e][2] = 0.0f; part[e][3] = 0.0f; }
            mlp_tile_accum(sb + (ASYM ? 2 : 1) * WL_WIDE_ROWS * WL_WIDE_XS + net * WL_WIDE_KC * WL_HID + ucol, sb + xoff, WL_WIDE_XS,
                           kn, part);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[e][q] += part[e][q];
        }
        __syncthreads();                                     // every thread is done with the buffer the next chunk refills
    }
}

// the blob without its W1t blocks, [o1, o6) | [o7, end), into shared memory `sw` (one bulk copy each, completing on mbar)
__device__ __forceinline__ void wide_load_compact(float* sw, const float* __restrict__ blob, int blob_floats, const PolicyOffsets& po,
                                                  uint64_t* mbar) {
    const uint32_t na = (uint32_t)(po.o[6] - po.o[1]), nc = (uint32_t)(blob_floats - po.o[7]);
    mbar_init(mbar, 1);
    mbar_init_fence();
    mbar_expect(mbar, (na + nc) * 4u);
    bulk_g2s(sw, blob + po.o[1], na * 4u, mbar);
    bulk_g2s(sw + na, blob + po.o[7], nc * 4u, mbar);
}

__device__ __forceinline__ void store_relu(float* h0, int hstride, const float acc[4][4]) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
        *reinterpret_cast<float4*>(h0 + e * hstride) = make_float4(relu(acc[e][0]), relu(acc[e][1]), relu(acc[e][2]), relu(acc[e][3]));
}

// ---- the rollout's policy ------------------------------------------------------------------------------------------
// One CTA per 32 envs.  po: blob offsets; pc: the compact offsets of the shared-memory copy.  Does not step the env and
// does not trigger dependents early: a step launched after it with PDL waits for every action.  ASYM (wl_policy_act_wide_asym):
// the critic's layer 1 reads critic_in [n, Dc]; everything after layer 1 is the same code.
template <bool ASYM>
__device__ __forceinline__ void policy_act_wide_body(const float* __restrict__ obs_in, int n, int D, const float* __restrict__ blob,
                                                     int blob_floats, const PolicyOffsets& po, const PolicyOffsets& pc,
                                                     const wl_policy_out& out, const wl_globals* __restrict__ gl, uint64_t seed,
                                                     int env_id_offset, uint32_t t_arg, const float* __restrict__ critic_in, int Dc) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ int64_t srow[WL_WIDE_ROWS];
    float* stage = smem;
    float* sw = stage + 2 * (ASYM ? WL_WIDE_STAGE_ASYM : WL_WIDE_STAGE);   // compact blob
    float* sh = sw + (po.o[6] - po.o[1]) + (blob_floats - po.o[7]);     // [32][WL_PPO_HS]
    const int tid = threadIdx.x, r0 = blockIdx.x * WL_WIDE_ROWS;
    if (tid == 0) wide_load_compact(sw, blob, blob_floats, po, &mbar);
    if (tid < WL_WIDE_ROWS) srow[tid] = r0 + tid < n ? r0 + tid : -1;
    __syncthreads();
    const int lane = tid & 31, net = lane >> 4, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 4;
    float acc[4][4];
    wide_layer1<ASYM>(obs_in, D, srow, blob, po, stage, acc, critic_in, Dc);
    float* h0 = sh + env0 * WL_PPO_HS + net * WL_HID;
    store_relu(h0 + ucol, WL_PPO_HS, acc);
    mbar_wait_parity(&mbar, 0);
    __syncwarp();
    mlp_tile_layer(sw + (net ? pc.o[8] : pc.o[2]) + ucol, sw + (net ? pc.o[9] : pc.o[3]) + ucol, h0, WL_PPO_HS, WL_HID, acc);
    __syncwarp();                                            // every lane has finished reading layer-1 activations
    store_relu(h0 + ucol, WL_PPO_HS, acc);
    __syncthreads();
    // heads: 8 threads per env, 8 hidden units each, then a butterfly
    const int s = tid >> 3, p = tid & 7, i = r0 + s;
    const float* hrow = sh + s * WL_PPO_HS;
    const float* w3a = sw + pc.o[4]; const float* w3c = sw + pc.o[10];
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
    if (p == 0 && i < n) {
        m0 += sw[pc.o[5]]; m1 += sw[pc.o[5] + 1]; vv += sw[pc.o[11]];
        float z0, z1, lp;
        float2 a;
        policy_noise(seed, (uint32_t)(env_id_offset + i), decode_step(gl, t_arg), z0, z1);
        gaussian_head(m0, m1, sw[pc.o[12]], sw[pc.o[12] + 1], z0, z1, a, lp);
        reinterpret_cast<float2*>(out.actions)[i] = a;
        reinterpret_cast<float2*>(out.mean)[i] = make_float2(m0, m1);
        out.log_prob[i] = lp;
        out.value[i] = vv;
    }
}
__global__ void __launch_bounds__(WL_WIDE_THREADS)
wl_policy_act_kernel(const float* __restrict__ obs_in, int n, int D, const float* __restrict__ blob, int blob_floats, PolicyOffsets po,
                     PolicyOffsets pc, wl_policy_out out, const wl_globals* __restrict__ gl, uint64_t seed, int env_id_offset,
                     uint32_t t_arg) {
    policy_act_wide_body<false>(obs_in, n, D, blob, blob_floats, po, pc, out, gl, seed, env_id_offset, t_arg, nullptr, 0);
}
__global__ void __launch_bounds__(WL_WIDE_THREADS)
wl_policy_act_wide_asym_kernel(const float* __restrict__ obs_in, int n, int D, const float* __restrict__ critic_in, int Dc,
                               const float* __restrict__ blob, int blob_floats, PolicyOffsets po, PolicyOffsets pc, wl_policy_out out,
                               const wl_globals* __restrict__ gl, uint64_t seed, int env_id_offset, uint32_t t_arg) {
    policy_act_wide_body<true>(obs_in, n, D, blob, blob_floats, po, pc, out, gl, seed, env_id_offset, t_arg, critic_in, Dc);
}

// ---- PPO update ------------------------------------------------------------------------------------------------------
// H1[row] = relu(layer 1 of X[perm[row0 + row]]) for the mini-batch, [tiles * 32][128] (rows past B: relu(b1), never used)
__global__ void __launch_bounds__(WL_WIDE_THREADS)
wl_ppo_wide_fwd_kernel(const float* __restrict__ blob, PolicyOffsets po, const __grid_constant__ PpoArgs a, float* __restrict__ H1) {
    extern __shared__ __align__(128) float smem[];
    __shared__ int64_t srow[WL_WIDE_ROWS];
    const int tid = threadIdx.x, s0 = blockIdx.x * WL_WIDE_ROWS;
    if (tid < WL_WIDE_ROWS) srow[tid] = s0 + tid < a.B ? a.b.perm[a.row0 + s0 + tid] : -1;
    __syncthreads();
    float acc[4][4];
    wide_layer1(a.b.obs, a.obs_dim, srow, blob, po, smem, acc);
    const int lane = tid & 31, net = lane >> 4, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 4;
    store_relu(H1 + (size_t)(s0 + env0) * (2 * WL_HID) + net * WL_HID + ucol, 2 * WL_HID, acc);
}
// the same with the critic's layer 1 over xc [batch, Dc] (slab order, gathered through the same perm)
__global__ void __launch_bounds__(WL_WIDE_THREADS)
wl_ppo_wide_fwd_asym_kernel(const float* __restrict__ blob, PolicyOffsets po, const __grid_constant__ PpoArgs a, const float* __restrict__ xc,
                            int Dc, float* __restrict__ H1) {
    extern __shared__ __align__(128) float smem[];
    __shared__ int64_t srow[WL_WIDE_ROWS];
    const int tid = threadIdx.x, s0 = blockIdx.x * WL_WIDE_ROWS;
    if (tid < WL_WIDE_ROWS) srow[tid] = s0 + tid < a.B ? a.b.perm[a.row0 + s0 + tid] : -1;
    __syncthreads();
    float acc[4][4];
    wide_layer1<true>(a.b.obs, a.obs_dim, srow, blob, po, smem, acc, xc, Dc);
    const int lane = tid & 31, net = lane >> 4, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 4;
    store_relu(H1 + (size_t)(s0 + env0) * (2 * WL_HID) + net * WL_HID + ucol, 2 * WL_HID, acc);
}

// Layers 2-3 and the loss on H1, back-propagated to dZ1 = dL/d(layer-1 pre-activation) -> workspace.  As wl_ppo_grad_kernel
// (persistent CTAs, tiles b, b + grid, ...; thread t owns fixed gradient entries) without layer 1, with ReLU; its row gets
// every gradient entry except dW1 (wl_ppo_wide_dw1_kernel writes those).  sw: compact blob (offsets pc), po: blob offsets.
__global__ void __launch_bounds__(WL_PPO_THREADS, 1)
wl_ppo_wide_grad_kernel(const float* __restrict__ blob, int blob_floats, PolicyOffsets po, PolicyOffsets pc, const __grid_constant__ PpoArgs a,
                        const float* __restrict__ state, const float* __restrict__ H1, float* __restrict__ dZ1, float* __restrict__ rows,
                        int rowlen) {
    extern __shared__ __align__(128) float smem[];
    __shared__ __align__(8) uint64_t mbar;
    const int cfl = (po.o[6] - po.o[1]) + (blob_floats - po.o[7]);
    float* sw = smem;                                        // compact blob
    float* sw2t = sw + cfl;                                  // [net][64 out][64 in]: W2 output-major, for dh1 = dz2 W2
    float* szero = sw2t + 2 * WL_HID * WL_HID;
    float* sh1 = szero + WL_HID;                             // [32][HS] layer-1 activations
    float* sh2 = sh1 + WL_PPO_TILE * WL_PPO_HS;              // layer-2 activations
    float* sg2 = sh2 + WL_PPO_TILE * WL_PPO_HS;              // dL/dz2
    float* sg1 = sg2 + WL_PPO_TILE * WL_PPO_HS;              // dL/dz1
    float* sd = sg1 + WL_PPO_TILE * WL_PPO_HS;               // [32][SD]
    const int tid = threadIdx.x;
    if (tid == 0) wide_load_compact(sw, blob, blob_floats, po, &mbar);
    if (tid < WL_HID) szero[tid] = 0.0f;
    const float adv_mean = state[4], adv_den = state[5] + 1e-8f, so0 = state[2], so1 = state[3];
    __syncthreads();
    mbar_wait_parity(&mbar, 0);
    for (int k = tid; k < 2 * WL_HID * WL_HID; k += WL_PPO_THREADS) {
        const int u = (k >> 6) & (WL_HID - 1), i = k & (WL_HID - 1);
        sw2t[k] = sw[(k >> 12 ? pc.o[8] : pc.o[2]) + i * WL_HID + u];
    }
    const float sg_0 = sw[pc.o[12]], sg_1 = sw[pc.o[12] + 1];
    const int net = tid >> 7, r = tid & 127;
    const int i2 = (r >> 3) * 4, u2 = (r & 7) * 8;           // dW2t rows i2..i2+3, cols u2..u2+7
    float gW2[4][8], gb = 0.0f, gh = 0.0f;                   // gb: db1 (r < 64) / db2; gh: head, std or statistic (tid < 200)
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 8; ++q) gW2[k][q] = 0.0f;
    const int lane = tid & 31, fnet = lane >> 4, ucol = (lane & 15) * 4, env0 = (tid >> 5) * 4;
    const int oW2 = fnet ? pc.o[8] : pc.o[2], oB2 = fnet ? pc.o[9] : pc.o[3];
    const float b3a0 = sw[pc.o[5]], b3a1 = sw[pc.o[5] + 1], b3c = sw[pc.o[11]];
    __syncthreads();                                         // sw2t complete

    for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
        const int s0 = tile * WL_PPO_TILE;
        for (int k = tid; k < WL_PPO_TILE * 32; k += WL_PPO_THREADS) {
            const int s = k >> 5, q = k & 31;
            *reinterpret_cast<float4*>(sh1 + s * WL_PPO_HS + 4 * q) = *reinterpret_cast<const float4*>(H1 + (size_t)(s0 + s) * (2 * WL_HID) + 4 * q);
        }
        __syncthreads();
        {
            float acc[4][4];
            mlp_tile_layer(sw + oW2 + ucol, sw + oB2 + ucol, sh1 + env0 * WL_PPO_HS + fnet * WL_HID, WL_PPO_HS, WL_HID, acc);
            store_relu(sh2 + env0 * WL_PPO_HS + fnet * WL_HID + ucol, WL_PPO_HS, acc);
        }
        __syncthreads();
        {   // heads: 8 threads per sample, 8 hidden units each, then a butterfly; thread 0 of the 8 forms the derivatives
            const int s = tid >> 3, p = tid & 7, row = s0 + s;
            const float* hrow = sh2 + s * WL_PPO_HS;
            const float* w3a = sw + pc.o[4]; const float* w3c = sw + pc.o[10];
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
        for (int k = tid; k < WL_PPO_TILE * 2 * WL_HID; k += WL_PPO_THREADS) {     // dz2 = (dy W3) * relu'(h2)
            const int s = k >> 7, c = k & 127;
            const float* d = sd + s * WL_PPO_SD;
            const float dh = c < WL_HID ? d[0] * sw[pc.o[4] + 2 * c] + d[1] * sw[pc.o[4] + 2 * c + 1] : d[2] * sw[pc.o[10] + c - WL_HID];
            sg2[s * WL_PPO_HS + c] = sh2[s * WL_PPO_HS + c] > 0.0f ? dh : 0.0f;   // torch threshold_backward: 0 at h == 0
        }
        __syncthreads();
        {   // dz1 = (dz2 W2) * relu'(h1): the forward layer routine on the output-major copy of W2, zero bias
            float acc[4][4];
            mlp_tile_layer(sw2t + fnet * WL_HID * WL_HID + ucol, szero + ucol, sg2 + env0 * WL_PPO_HS + fnet * WL_HID, WL_PPO_HS, WL_HID, acc);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int o = (env0 + e) * WL_PPO_HS + fnet * WL_HID + ucol;
                const float4 h = *reinterpret_cast<const float4*>(sh1 + o);
                const float4 g = make_float4(h.x > 0.0f ? acc[e][0] : 0.0f, h.y > 0.0f ? acc[e][1] : 0.0f,
                                             h.z > 0.0f ? acc[e][2] : 0.0f, h.w > 0.0f ? acc[e][3] : 0.0f);
                *reinterpret_cast<float4*>(sg1 + o) = g;
                *reinterpret_cast<float4*>(dZ1 + (size_t)(s0 + env0 + e) * (2 * WL_HID) + fnet * WL_HID + ucol) = g;
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
            gb += r < WL_HID ? g1[r] : g2[r - WL_HID];
            const float* d = sd + s * WL_PPO_SD;
            if (tid < 128) gh = fmaf(sh2[s * WL_PPO_HS + (tid >> 1)], d[tid & 1], gh);
            else if (tid < 192) gh = fmaf(sh2[s * WL_PPO_HS + tid - 64], d[2], gh);
            else if (tid < 200) gh += d[tid - 192];
        }
        __syncthreads();                                     // the next tile overwrites the shared rows
    }

    float* row = rows + (size_t)blockIdx.x * rowlen;
    const int gB1o = net ? po.o[7] : po.o[1], gW2o = net ? po.o[8] : po.o[2], gB2o = net ? po.o[9] : po.o[3];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        *reinterpret_cast<float4*>(row + gW2o + (i2 + k) * WL_HID + u2) = make_float4(gW2[k][0], gW2[k][1], gW2[k][2], gW2[k][3]);
        *reinterpret_cast<float4*>(row + gW2o + (i2 + k) * WL_HID + u2 + 4) = make_float4(gW2[k][4], gW2[k][5], gW2[k][6], gW2[k][7]);
    }
    row[r < WL_HID ? gB1o + r : gB2o + r - WL_HID] = gb;
    if (tid < 128) row[po.o[4] + tid] = gh;                  // dW3t actor, [unit][action]
    else if (tid < 192) row[po.o[10] + tid - 128] = gh;      // dW3t critic
    else if (tid < 194) row[po.o[5] + tid - 192] = gh;       // db3 actor
    else if (tid == 194) row[po.o[11]] = gh;                 // db3 critic
    else if (tid < 197) row[po.o[12] + tid - 195] = gh;      // dsigma (the log-prob part; entropy is added once when reduced)
    else if (tid < 200) row[blob_floats + tid - 197] = gh;   // surrogate / value-loss / KL sums
}

// dW1t[k][u] (both nets: u < 64 actor, u >= 64 critic) = sum over samples of X[perm[row0 + s]][k] dZ1[s][u].  Block
// (kt, split) owns W1t rows 64 kt .. 64 kt + 63 and the samples of tiles split, split + gridDim.y, ... (the grad kernel's
// tiles), summed in sample order; it writes its partial into gradient row `split`.  Thread: 4 rows x 8 columns.
// ASYM: the critic's columns take their rows from xc [batch, Dc] (staged beside X); gridDim.x covers max(D, Dc).
template <bool ASYM>
__device__ __forceinline__ void ppo_wide_dw1_body(const PolicyOffsets& po, const PpoArgs& a, const float* __restrict__ dZ1,
                                                  float* __restrict__ rows, int rowlen, const float* __restrict__ xc, int Dc) {
    extern __shared__ __align__(128) float smem[];           // 2 stages of [32][64] X (ASYM: and [32][64] Xc) | [32][128] dZ1
    constexpr int XF = WL_PPO_TILE * WL_DW1_K, NX = ASYM ? 2 : 1, SF = NX * XF + WL_PPO_TILE * 2 * WL_HID;
    const int tid = threadIdx.x, D = a.obs_dim, k0 = blockIdx.x * WL_DW1_K;
    const int tk = (tid >> 4) * 4, tu = (tid & 15) * 8;
    auto stage = [&](float* sb, int tile) {
        const int s0 = tile * WL_PPO_TILE;
#pragma unroll
        for (int net = 0; net < NX; ++net) {
            const int Dn = net ? Dc : D;
            for (int k = tid; k < XF; k += WL_WIDE_THREADS) {
                const int s = k / WL_DW1_K, j = k % WL_DW1_K, col = k0 + j;
                const bool ok = s0 + s < a.B && col < Dn;
                const float* src = net ? xc : a.b.obs;
                if (ok) src += (size_t)a.b.perm[a.row0 + s0 + s] * Dn + col;
                cp_async4(sb + net * XF + k, src, ok);
            }
        }
        for (int k = tid; k < WL_PPO_TILE * 32; k += WL_WIDE_THREADS)
            cp_async16(sb + NX * XF + 4 * k, dZ1 + (size_t)s0 * (2 * WL_HID) + 4 * k);
    };
    float g[4][8];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int q = 0; q < 8; ++q) g[k][q] = 0.0f;
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
        const float* sx = smem + (it & 1) * SF + (ASYM && tu >= WL_HID ? XF : 0);
        const float* sz = smem + (it & 1) * SF + NX * XF;
        for (int s = 0; s < WL_PPO_TILE; ++s) {
            const float4 xv = *reinterpret_cast<const float4*>(sx + s * WL_DW1_K + tk);
            const float4 za = *reinterpret_cast<const float4*>(sz + s * 2 * WL_HID + tu), zb = *reinterpret_cast<const float4*>(sz + s * 2 * WL_HID + tu + 4);
            const float xk[4] = {xv.x, xv.y, xv.z, xv.w}, zq[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
                for (int q = 0; q < 8; ++q) g[k][q] = fmaf(xk[k], zq[q], g[k][q]);
        }
        __syncthreads();
    }
    const int Dn = ASYM && tu >= WL_HID ? Dc : D;
    float* row = rows + (size_t)blockIdx.y * rowlen + (tu < WL_HID ? po.o[0] : po.o[6]) + (tu & (WL_HID - 1));
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (k0 + tk + k < Dn) {
            *reinterpret_cast<float4*>(row + (size_t)(k0 + tk + k) * WL_HID) = make_float4(g[k][0], g[k][1], g[k][2], g[k][3]);
            *reinterpret_cast<float4*>(row + (size_t)(k0 + tk + k) * WL_HID + 4) = make_float4(g[k][4], g[k][5], g[k][6], g[k][7]);
        }
}
__global__ void __launch_bounds__(WL_WIDE_THREADS)
wl_ppo_wide_dw1_kernel(PolicyOffsets po, const __grid_constant__ PpoArgs a, const float* __restrict__ dZ1, float* __restrict__ rows, int rowlen) {
    ppo_wide_dw1_body<false>(po, a, dZ1, rows, rowlen, nullptr, 0);
}
__global__ void __launch_bounds__(WL_WIDE_THREADS)
wl_ppo_wide_dw1_asym_kernel(PolicyOffsets po, const __grid_constant__ PpoArgs a, const float* __restrict__ dZ1, float* __restrict__ rows,
                            int rowlen, const float* __restrict__ xc, int Dc) {
    ppo_wide_dw1_body<true>(po, a, dZ1, rows, rowlen, xc, Dc);
}
