// Shared pieces of the GAT kernels (gat_step.cu: K1 recurrence + attention; gat128.cu: the 128-wide recurrence):
// launch arguments, gate-activation constants, packed-fp32 arithmetic and the f16 hi/lo split.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace iplan {

constexpr int H = IPLAN_HID;   // 32 == GAT_hidden_dim == attention_dim
constexpr int G3 = 3 * H;      // gate rows r|z|n
constexpr int GAT_THREADS = 256;           // attend kernel
constexpr int GAT_WARPS = GAT_THREADS / 32;
constexpr int REC_THREADS = 128;           // recurrence kernel: 4 warps = 4 m-tiles of 16 egos
constexpr int REC_WARPS = REC_THREADS / 32;
constexpr int DLP = IPLAN_MAX_SLOTS;       // row pitch of the dl scratch: dl[dir][s][DLP]
constexpr int IN_MAX = 16;     // obs_dim + latent_dim upper bound
constexpr int NT_G = G3 / 8;   // 12 n-tiles of 8 gate columns
constexpr int PP = G3 + 8;     // row pitch of the ego projections P: rows of different chains fall in different banks
constexpr int KB_H = H / 16;   // 2 k-blocks of 16 hidden units

struct GatArgs {
    const float* params; int64_t param_stride;
    iplan_view hist, beh, hprev, out;
    const float* gumbel; float* dbg_hard; float* dl;
    uint64_t seed, counter;
    float inv_tau;
    int n_envs, n_slots, obs_dim, latent_dim;
};

// fast, fp32-accurate-enough gates (abs error ~1e-7): ex2.approx + rcp.approx
// The recurrence keeps its r|z pre-activations scaled by -log2(e) and its n pre-activation by
// 2 log2(e) (the scale is folded into W_hh, b_hh, P and Q once per CTA), so that
//   sigmoid(x) = 1 / (1 + 2^(x'))   and   tanh(x) = 1 - 2 / (1 + 2^(x'))
// cost one ex2.approx + one add + one rcp.approx each (abs error ~1e-7).
constexpr float K_RZ = -1.4426950408889634f;      // -log2(e)
constexpr float K_N = 2.8853900817779268f;        //  2 log2(e)
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// fp32 pairs: an accumulator fragment is two (col, col+1) pairs, so the gate math is written on pairs.
// sm_90 has no packed fp32 instructions; each pair op is two scalar round-to-nearest ops.
typedef float2 f32x2;
__device__ __forceinline__ f32x2 pk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ void upk2(f32x2 v, float& a, float& b) { a = v.x; b = v.y; }
__device__ __forceinline__ f32x2 add2(f32x2 a, f32x2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 sub2(f32x2 a, f32x2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 mul2(f32x2 a, f32x2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f32x2 fma2(f32x2 a, f32x2 b, f32x2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ f32x2 lds64(const float* p) {
    f32x2 v;
    asm volatile("ld.shared.v2.f32 {%0,%1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"((uint32_t)__cvta_generic_to_shared(p)));
    return v;
}

// Four sigmoid denominators with ONE rcp.approx (the XU pipe is the recurrence's busiest unit):
// given ea = 2^xa (pair) and eb = 2^xb (pair), returns ia = 1/(1+ea), ib = 1/(1+eb) from
//   p = (1+ea)(1+eb) per pair,  inv = 1/(p0 p1),  q = (inv p1, inv p0) = 1/p,
//   ia = (1+eb) q,  ib = (1+ea) q.
// Inputs are clamped to x <= 30 so that p0 p1 <= 2^121 stays finite; the clamp moves a sigmoid by
// < 1e-9 (the gate is saturated: pre-activation beyond 20.8).
__device__ __forceinline__ void sigmoid4_den(f32x2 x01, f32x2 x23, f32x2& ia, f32x2& ib) {
    float x0, x1, x2, x3;
    upk2(x01, x0, x1); upk2(x23, x2, x3);
    const f32x2 ea = pk2(ex2_approx(fminf(x0, 30.0f)), ex2_approx(fminf(x1, 30.0f)));
    const f32x2 eb = pk2(ex2_approx(fminf(x2, 30.0f)), ex2_approx(fminf(x3, 30.0f)));
    const f32x2 b = add2(eb, pk2(1.0f, 1.0f));
    const f32x2 p = fma2(ea, b, b);
    float p0, p1;
    upk2(p, p0, p1);
    const float inv = rcp_approx(p0 * p1);
    const f32x2 q = pk2(inv * p1, inv * p0);
    ia = mul2(b, q);
    ib = fma2(ea, q, q);
}
// pair -> packed f16 hi pair and f16 lo (residual) pair
__device__ __forceinline__ void split_f16p(f32x2 v, uint32_t& hi, uint32_t& lo) {
    float x, y;
    upk2(v, x, y);
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    float rx, ry;
    upk2(sub2(v, pk2(hf.x, hf.y)), rx, ry);
    const __half2 l = __floats2half2_rn(rx, ry);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// (x, y) -> packed f16 hi pair and f16 lo (residual) pair
__device__ __forceinline__ void split_f16(float x, float y, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

}  // namespace iplan
