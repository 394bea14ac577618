// wl_critic.cuh -- the privileged critic observation of the Drift family (DESIGN 6m), included by wl_api.cu after
// wl_step.cuh (EnvState's state groups, rotmat / rotT / euler_xyz, r_clamp).
//
// A handle's critic table (wl_set_critic_terms) lists terms of the library below; wl_critic_observe_kernel writes their
// concatenation, [N, Dc], from the state groups the step just left.  No noise, no generator, no counter.
#pragma once

#define WL_CRITIC_LIB_FLOATS 29                   // every library term once, in kind order
#define WL_CRITIC_BS 128                          // envs per CTA
#define WL_CRITIC_LS 33                           // padded library row in shared memory (odd: conflict-free column reads)

// the kernel's table: output column j = library float src[j], clipped to +-clip[j] when clip[j] > 0
struct CriticTable {
    int32_t n_cols;                               // Dc (0: no table)
    uint32_t groups;                              // bit g: state group g is read
    uint8_t src[WL_MAX_CRITIC_OBS];
    float clip[WL_MAX_CRITIC_OBS];
};

// first library float and width of each term kind (index = kind), and the state groups it reads
__host__ __device__ constexpr int critic_first(int kind) {
    constexpr int f[WL_CRITIC_KINDS] = {0, 0, 3, 6, 9, 12, 14, 18, 20, 24, 25};
    return f[kind];
}
__host__ __device__ constexpr int critic_width(int kind) {
    constexpr int w[WL_CRITIC_KINDS] = {0, 3, 3, 3, 3, 2, 4, 2, 4, 1, 4};
    return w[kind];
}
static uint32_t critic_groups(int kind) {
    switch (kind) {
        case WL_CRITIC_ROOT_POS_W: return 1u << WL_G_POS;
        case WL_CRITIC_ROOT_EULER_XYZ: return 1u << WL_G_QUAT;
        case WL_CRITIC_BASE_LIN_VEL: return (1u << WL_G_QUAT) | (1u << WL_G_LINVEL);
        case WL_CRITIC_BASE_ANG_VEL: return (1u << WL_G_QUAT) | (1u << WL_G_ANGVEL);
        case WL_CRITIC_LAST_ACTION: return 1u << WL_G_ACTION;
        case WL_CRITIC_JOINT_VEL: return 1u << WL_G_WHEEL;
        case WL_CRITIC_JOINT_POS: return 1u << WL_G_STEER;
        case WL_CRITIC_WHEEL_FRICTION: return 1u << WL_G_PMU_D;
        case WL_CRITIC_BASE_MASS: return 1u << WL_G_PMASS;
        default: return 1u << WL_G_PKD;
    }
}

// One thread per env forms the library floats its table needs (one 128-bit load per state group, coalesced across the
// warp; groups no term names are not read) into shared memory; then the CTA writes its 128 rows, which are contiguous in
// [N, Dc], as float4 words (scalar words when `out` is not 16-byte aligned).  The shared columns are blind_obs's
// arithmetic without the noise draw: the same rotmat / rotT / euler_xyz / r_clamp on the same state words.
__global__ void __launch_bounds__(WL_CRITIC_BS)
wl_critic_observe_kernel(const __grid_constant__ CriticTable tb, const float4* __restrict__ st, int n, float* __restrict__ out) {
    __shared__ float lib[WL_CRITIC_BS * WL_CRITIC_LS];
    __shared__ int s_src[WL_MAX_CRITIC_OBS];
    __shared__ float s_clip[WL_MAX_CRITIC_OBS];
    const int tid = threadIdx.x, env0 = blockIdx.x * WL_CRITIC_BS, i = env0 + tid;
    if (tid < WL_MAX_CRITIC_OBS) { s_src[tid] = tb.src[tid]; s_clip[tid] = tb.clip[tid]; }
    if (i < n) {
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
        }
        if (G & (1u << WL_G_ACTION)) { g = ldg4(st, WL_G_ACTION, n, i); o[12] = g.x; o[13] = g.y; }
        if (G & (1u << WL_G_WHEEL)) { g = ldg4(st, WL_G_WHEEL, n, i); o[14] = g.x; o[15] = g.y; o[16] = g.z; o[17] = g.w; }
        if (G & (1u << WL_G_STEER)) { g = ldg4(st, WL_G_STEER, n, i); o[18] = g.x; o[19] = g.y; }
        if (G & (1u << WL_G_PMU_D)) { g = ldg4(st, WL_G_PMU_D, n, i); o[20] = g.x; o[21] = g.y; o[22] = g.z; o[23] = g.w; }
        if (G & (1u << WL_G_PMASS)) { g = ldg4(st, WL_G_PMASS, n, i); o[24] = g.x; }
        if (G & (1u << WL_G_PKD)) { g = ldg4(st, WL_G_PKD, n, i); o[25] = g.x; o[26] = g.y; o[27] = g.z; o[28] = g.w; }
    }
    __syncthreads();
    const int Dc = tb.n_cols, envs = min(WL_CRITIC_BS, n - env0), floats = envs * Dc;
    float* blk = out + (size_t)env0 * Dc;         // 128 * Dc * 4 bytes per CTA: 16-byte aligned whenever `out` is
    const bool al16 = (reinterpret_cast<uintptr_t>(out) & 15u) == 0;
    auto col = [&](int f) {
        const int e = f / Dc, j = f - e * Dc;
        const float x = lib[e * WL_CRITIC_LS + s_src[j]], cl = s_clip[j];
        return cl > 0.0f ? r_clamp(x, -cl, cl) : x;
    };
    if (!al16) {                                  // a slab row of an odd N * Dc: scalar stores, still contiguous
        for (int f = tid; f < floats; f += WL_CRITIC_BS) blk[f] = col(f);
        return;
    }
    for (int f = 4 * tid; f + 3 < floats; f += 4 * WL_CRITIC_BS)
        *reinterpret_cast<float4*>(blk + f) = make_float4(col(f), col(f + 1), col(f + 2), col(f + 3));
    if (tid < (floats & 3)) blk[(floats & ~3) + tid] = col((floats & ~3) + tid);
}
