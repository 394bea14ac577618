// wl_row_terms.cuh -- noise, clip and scale on the Elevation and Visual policy rows (DESIGN 6r), included by wl_api.cu after
// wl_policy_obs.cuh (decode_step's declaration; through wl_step.cuh rotmat / rotT / euler_xyz / box_muller / r_clamp).
//
// A handle's row terms (wl_set_row_terms) keep the task's built-in terms and their order and add, per term, what IsaacLab's
// ObservationManager.compute applies after the value: additive noise (enable_corruption only), the clip, the scale.  The
// Elevation row is written whole by wl_scan_row_kernel (wl_api.cu, next to wl_scan_kernel); the eight floats after the
// Visual camera by wl_visual_row_kernel below.  Noise keys: the header's wl_set_row_terms comment.
#pragma once

#define WL_ROW_PROPRIO 13                         // per-column stages: Elevation columns 0..12, Visual tail 0..7
#define WL_ROW_BLOCKS ((WL_OBS_DIM_ELEV + 3) / 4) // Philox blocks of one Elevation row: 173
#define WL_ROW_CLIP 1u                            // RowStage.flags bits
#define WL_ROW_SCALE 2u
#define WL_ROW_VIS_BS 128
#define WL_ROW_MAX_CALL ((1 << 23) - 2)           // wl_observe's call_idx with row terms: 512 (call_idx + 1) + 256 + 172 < 2^32
enum : uint32_t { RNG_ROW_TERMS = 17u };          // (RNG streams: wl_device.cuh)

// one column's stages: noise WL_NOISE_* with (na, nb) = (mean, std) or (n_min, n_max - n_min); clip [lo, hi]; scale sc
struct RowStage {
    int32_t noise;
    uint32_t flags;
    float na, nb, lo, hi, sc;
};
struct RowTable {
    int32_t n_terms;                              // 0: no row terms
    int32_t noisy;                                // some column draws noise (enable_corruption and a noise model)
    RowStage col[WL_ROW_PROPRIO];                 // the proprioceptive columns
    RowStage map;                                 // Elevation: every height-map column
};

// the block of Philox words of row block b (columns 4b..4b+3) for noise of `kind`
__device__ __forceinline__ uint4 row_block(uint64_t seed, uint32_t gid, uint32_t t, int32_t call_idx, int kind, uint32_t b) {
    return philox4x32(seed, gid, t, RNG_ROW_TERMS, 512u * (uint32_t)(call_idx + 1) + (kind == WL_NOISE_UNIFORM ? 256u : 0u) + b);
}
// the four draws of a block: N(0, 1) from two Box-Muller pairs, or U[0, 1)
__device__ __forceinline__ void row_draws(uint4 r, int kind, float d[4]) {
    if (kind == WL_NOISE_GAUSSIAN) {
        box_muller(r.x, r.y, d[0], d[1]);
        box_muller(r.z, r.w, d[2], d[3]);
    } else {
        d[0] = u01(r.x); d[1] = u01(r.y); d[2] = u01(r.z); d[3] = u01(r.w);
    }
}
// the draws of block b whose columns have the noise kinds k[0..3] (WL_NOISE_NONE: no draw, 0): one Philox block per kind
// present, so a column of one kind never shares a word with a column of the other
__device__ __forceinline__ void row_mixed_draws(uint64_t seed, uint32_t gid, uint32_t t, int32_t call_idx, uint32_t b, const int k[4], float d[4]) {
#pragma unroll
    for (int w = 0; w < 4; ++w) d[w] = 0.0f;
#pragma unroll
    for (int kind = WL_NOISE_GAUSSIAN; kind <= WL_NOISE_UNIFORM; ++kind) {
        if (k[0] != kind && k[1] != kind && k[2] != kind && k[3] != kind) continue;
        float e[4];
        row_draws(row_block(seed, gid, t, call_idx, kind, b), kind, e);
#pragma unroll
        for (int w = 0; w < 4; ++w) if (k[w] == kind) d[w] = e[w];
    }
}
// noise, clip, scale of one column, each one fp32 operation in ObservationManager.compute's order (no fma: -fmad=false)
__device__ __forceinline__ float row_stage(const RowStage& s, float x, float d) {
    if (s.noise == WL_NOISE_GAUSSIAN) {
        const float v = x + s.na;
        const float e = s.nb * d;
        x = v + e;
    } else if (s.noise == WL_NOISE_UNIFORM) {
        const float e = d * s.nb;
        const float v = x + e;
        x = v + s.na;
    }
    if (s.flags & WL_ROW_CLIP) x = r_clamp(x, s.lo, s.hi);
    if (s.flags & WL_ROW_SCALE) x = x * s.sc;
    return x;
}

// The eight floats after the camera floats of every Visual row (base_lin_vel, base_ang_vel, last_action), from the state
// the step / reset left, through the row terms.  One thread per env; row stride 8 + camf.
__global__ void __launch_bounds__(WL_ROW_VIS_BS)
wl_visual_row_kernel(const __grid_constant__ RowTable rt, const float4* __restrict__ st, const wl_globals* __restrict__ gl, int n, int camf,
                     uint64_t seed, int32_t env_id_offset, uint32_t t_arg, int32_t call_idx, float* __restrict__ obs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 q = ldg4(st, WL_G_QUAT, n, i), v = ldg4(st, WL_G_LINVEL, n, i), w = ldg4(st, WL_G_ANGVEL, n, i), a = ldg4(st, WL_G_ACTION, n, i);
    const M3 R = rotmat(q.x, q.y, q.z, q.w);
    const V3 vb = rotT(R, V3{v.x, v.y, v.z}), wb = rotT(R, V3{w.x, w.y, w.z});
    const float x[8] = {vb.x, vb.y, vb.z, wb.x, wb.y, wb.z, a.x, a.y};
    float d[8] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    if (rt.noisy) {
        const uint32_t t = decode_step(gl, t_arg), gid = (uint32_t)(env_id_offset + i);
#pragma unroll
        for (int b = 0; b < 2; ++b) {
            const int k[4] = {rt.col[4 * b].noise, rt.col[4 * b + 1].noise, rt.col[4 * b + 2].noise, rt.col[4 * b + 3].noise};
            row_mixed_draws(seed, gid, t, call_idx, (uint32_t)b, k, d + 4 * b);
        }
    }
    float* row = obs + (size_t)(WL_OBS_DIM_VISUAL + camf) * i + camf;
#pragma unroll
    for (int j = 0; j < 8; ++j) row[j] = row_stage(rt.col[j], x[j], d[j]);
}
