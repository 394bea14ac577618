// wl_policy_obs.cuh -- a modified policy observation group of the Drift family (DESIGN 6q), included by wl_api.cu after
// wl_critic.cuh (the critic library's first / width / groups, and through wl_step.cuh rotmat / rotT / euler_xyz / r_clamp).
//
// A handle's policy table (wl_set_policy_terms) lists terms of the critic library plus projected_gravity, each with
// optional additive noise, clip and scale; wl_policy_observe_kernel writes their concatenation, [N, Dp], from the state
// groups the step just left, in ObservationManager.compute's order per term: value, noise (enable_corruption only), clip,
// scale.  Noise keys: the header's wl_policy_term comment.
#pragma once

#define WL_POBS_ENVS 16                           // envs per CTA: N = 4096 is 256 CTAs, and a thread draws at most 4 elements
#define WL_POBS_THREADS 128
#define WL_POBS_GRAVITY_FIRST 29                  // library floats 29..31: projected_gravity (after the critic's 29)
#define WL_POBS_GRAVITY_BIT (1u << 31)            // `groups` bit: form projected_gravity (reads WL_G_QUAT)
#define WL_POBS_CLIP 1u                           // PolicyObsTable.flags bits
#define WL_POBS_SCALE 2u
enum : uint32_t { RNG_POLICY_OBS = 16u };         // columns >= 12 and uniform noise (RNG streams: wl_device.cuh)

// the step counter of a host value or WL_DEVICE_COUNTER_PLUS(k) (defined in wl_api.cu, with the step kernels)
__device__ __forceinline__ uint32_t decode_step(const wl_globals* __restrict__ gl, uint32_t t_arg);

// the kernel's table, per output column j: library float src[j]; noise[j] (WL_NOISE_*) with na / nb = (mean, std) or
// (n_min, n_max - n_min); flags[j] & WL_POBS_CLIP: clamp to [lo, hi]; flags[j] & WL_POBS_SCALE: times scale[j]
struct PolicyObsTable {
    int32_t n_cols;                               // Dp (0: no table)
    uint32_t groups;                              // bit g: state group g is read; WL_POBS_GRAVITY_BIT
    uint8_t src[WL_MAX_POLICY_OBS];
    uint8_t noise[WL_MAX_POLICY_OBS];
    uint8_t flags[WL_MAX_POLICY_OBS];
    float na[WL_MAX_POLICY_OBS], nb[WL_MAX_POLICY_OBS];
    float lo[WL_MAX_POLICY_OBS], hi[WL_MAX_POLICY_OBS];
    float scale[WL_MAX_POLICY_OBS];
};

__host__ __device__ constexpr int policy_obs_first(int kind) { return kind == WL_POLICY_PROJECTED_GRAVITY ? WL_POBS_GRAVITY_FIRST : critic_first(kind); }
__host__ __device__ constexpr int policy_obs_width(int kind) { return kind == WL_POLICY_PROJECTED_GRAVITY ? 3 : critic_width(kind); }
static uint32_t policy_obs_groups(int kind) {
    return kind == WL_POLICY_PROJECTED_GRAVITY ? (WL_POBS_GRAVITY_BIT | (1u << WL_G_QUAT)) : critic_groups(kind);
}

// The noise of column j for the env with global id gid at counter t: (x + mean) + std * z or (x + u * (n_max - n_min)) +
// n_min, IsaacLab's gaussian_noise / uniform_noise with operation "add" [UPSTREAM-RECALL isaaclab.utils.noise].  A Gaussian
// column below 12 takes blind_obs's draw for that column: block j / 4 of (RNG_OBS, 0) after a step, of (RNG_OBS_EXTRA,
// 3 call_idx) for an observe call, lane j % 4 of its two Box-Muller pairs.  Every other noisy column takes block
// 16 (call_idx + 1) + 8 [uniform] + j / 4 of RNG_POLICY_OBS, word j % 4 (a Box-Muller pair for a Gaussian one).
__device__ __forceinline__ float policy_obs_noise(uint64_t seed, uint32_t gid, uint32_t t, int32_t call_idx, int j, int kind, float na,
                                                  float nb, float x) {
    const bool low = kind == WL_NOISE_GAUSSIAN && j < 12;
    const uint32_t ctx = (uint32_t)(call_idx + 1);
    const uint4 r = low ? philox4x32(seed, gid, t, call_idx < 0 ? RNG_OBS : RNG_OBS_EXTRA, (call_idx < 0 ? 0u : 3u * (uint32_t)call_idx) + (uint32_t)(j >> 2))
                        : philox4x32(seed, gid, t, RNG_POLICY_OBS, 16u * ctx + (kind == WL_NOISE_UNIFORM ? 8u : 0u) + (uint32_t)(j >> 2));
    const int w = j & 3;
    if (kind == WL_NOISE_GAUSSIAN) {
        float z0, z1;
        if (w < 2) box_muller(r.x, r.y, z0, z1); else box_muller(r.z, r.w, z0, z1);
        const float z = (w & 1) ? z1 : z0;
        const float v = x + na;
        const float s = nb * z;
        return v + s;
    }
    const uint32_t word = w == 0 ? r.x : w == 1 ? r.y : w == 2 ? r.z : r.w;
    const float s = u01(word) * nb;
    const float v = x + s;
    return v + na;
}

// One thread per env forms the library floats its table needs into shared memory, as wl_critic_observe_kernel does (plus
// projected_gravity = R^T (0, 0, -1)); then the CTA's 128 threads write its 16 rows, contiguous in [N, Dp], as float4 words
// (scalar words when `out` is not 16-byte aligned), each element drawn, clipped and scaled where it is written.  The draws
// are the kernel's cost, so a CTA holds few envs: more CTAs, and fewer draws one after another per thread.
__global__ void __launch_bounds__(WL_POBS_THREADS)
wl_policy_observe_kernel(const __grid_constant__ PolicyObsTable tb, const float4* __restrict__ st, const wl_globals* __restrict__ gl, int n,
                         uint64_t seed, int32_t env_id_offset, int32_t corrupt, uint32_t t_arg, int32_t call_idx, float* __restrict__ out) {
    __shared__ float lib[WL_POBS_ENVS * WL_CRITIC_LS];
    __shared__ int s_src[WL_MAX_POLICY_OBS], s_noise[WL_MAX_POLICY_OBS], s_flags[WL_MAX_POLICY_OBS];
    __shared__ float s_na[WL_MAX_POLICY_OBS], s_nb[WL_MAX_POLICY_OBS], s_lo[WL_MAX_POLICY_OBS], s_hi[WL_MAX_POLICY_OBS], s_sc[WL_MAX_POLICY_OBS];
    const int tid = threadIdx.x, env0 = blockIdx.x * WL_POBS_ENVS, i = env0 + tid;
    if (tid < WL_MAX_POLICY_OBS) {
        s_src[tid] = tb.src[tid]; s_noise[tid] = corrupt ? tb.noise[tid] : WL_NOISE_NONE; s_flags[tid] = tb.flags[tid];
        s_na[tid] = tb.na[tid]; s_nb[tid] = tb.nb[tid]; s_lo[tid] = tb.lo[tid]; s_hi[tid] = tb.hi[tid]; s_sc[tid] = tb.scale[tid];
    }
    if (tid < WL_POBS_ENVS && i < n) {
        float* o = lib + tid * WL_CRITIC_LS;
        const uint32_t G = tb.groups;
        float4 g;
        if (G & (1u << WL_G_POS)) { g = ldg4(st, WL_G_POS, n, i); o[0] = g.x; o[1] = g.y; o[2] = g.z; }
        if (G & (1u << WL_G_QUAT)) {
            g = ldg4(st, WL_G_QUAT, n, i);
            const V3 eu = euler_xyz(g.x, g.y, g.z, g.w);
            o[3] = eu.x; o[4] = eu.y; o[5] = eu.z;
            const M3 R = rotmat(g.x, g.y, g.z, g.w);
            if (G & (1u << WL_G_LINVEL)) {
                const float4 v = ldg4(st, WL_G_LINVEL, n, i);
                const V3 vb = rotT(R, V3{v.x, v.y, v.z});
                o[6] = vb.x; o[7] = vb.y; o[8] = vb.z;
            }
            if (G & (1u << WL_G_ANGVEL)) {
                const float4 v = ldg4(st, WL_G_ANGVEL, n, i);
                const V3 wb = rotT(R, V3{v.x, v.y, v.z});
                o[9] = wb.x; o[10] = wb.y; o[11] = wb.z;
            }
            if (G & WL_POBS_GRAVITY_BIT) {
                const V3 gb = rotT(R, V3{0.0f, 0.0f, -1.0f});
                o[29] = gb.x; o[30] = gb.y; o[31] = gb.z;
            }
        }
        if (G & (1u << WL_G_ACTION)) { g = ldg4(st, WL_G_ACTION, n, i); o[12] = g.x; o[13] = g.y; }
        if (G & (1u << WL_G_WHEEL)) { g = ldg4(st, WL_G_WHEEL, n, i); o[14] = g.x; o[15] = g.y; o[16] = g.z; o[17] = g.w; }
        if (G & (1u << WL_G_STEER)) { g = ldg4(st, WL_G_STEER, n, i); o[18] = g.x; o[19] = g.y; }
        if (G & (1u << WL_G_PMU_D)) { g = ldg4(st, WL_G_PMU_D, n, i); o[20] = g.x; o[21] = g.y; o[22] = g.z; o[23] = g.w; }
        if (G & (1u << WL_G_PMASS)) { g = ldg4(st, WL_G_PMASS, n, i); o[24] = g.x; }
        if (G & (1u << WL_G_PKD)) { g = ldg4(st, WL_G_PKD, n, i); o[25] = g.x; o[26] = g.y; o[27] = g.z; o[28] = g.w; }
    }
    __syncthreads();
    const uint32_t t = decode_step(gl, t_arg);
    const int Dp = tb.n_cols, envs = min(WL_POBS_ENVS, n - env0), floats = envs * Dp;
    float* blk = out + (size_t)env0 * Dp;         // 16 * Dp * 4 bytes per CTA: 16-byte aligned whenever `out` is
    const bool al16 = (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
    auto col = [&](int f) {
        const int e = f / Dp, j = f - e * Dp;
        float x = lib[e * WL_CRITIC_LS + s_src[j]];
        if (s_noise[j] != WL_NOISE_NONE)
            x = policy_obs_noise(seed, (uint32_t)(env_id_offset + env0 + e), t, call_idx, j, s_noise[j], s_na[j], s_nb[j], x);
        if (s_flags[j] & WL_POBS_CLIP) x = r_clamp(x, s_lo[j], s_hi[j]);
        if (s_flags[j] & WL_POBS_SCALE) x = x * s_sc[j];
        return x;
    };
    if (!al16) {                                  // a slab row of an odd N * Dp: scalar stores, still contiguous
        for (int f = tid; f < floats; f += WL_POBS_THREADS) blk[f] = col(f);
        return;
    }
    for (int f = 4 * tid; f + 3 < floats; f += 4 * WL_POBS_THREADS)
        *reinterpret_cast<float4*>(blk + f) = make_float4(col(f), col(f + 1), col(f + 2), col(f + 3));
    if (tid < (floats & 3)) blk[(floats & ~3) + tid] = col((floats & ~3) + tid);
}
