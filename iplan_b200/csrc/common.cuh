// Shared device helpers for the iPLAN sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/iplan_b200.h"

#define IPLAN_WARP 32

namespace iplan {

// ---- error plumbing (host) --------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
int  check_launch(const char* what);
int  sm_count();                 // multiprocessors of the current device (grid sizing)

// ---- deterministic cross-CTA sums ---------------------------------------------------------------
// Float atomics from several CTAs add in the order the CTAs happen to finish, so the rounding of the result changes from run
// to run.  Where several CTAs contribute to one sum, each CTA of the group instead stores its partial into its own slot of
// `part` and arrives at the group's counter; the last CTA to arrive adds the slots in slot order (det_last_arrival), which
// gives the same bits in every run.  det_scratch() returns library-owned device buffers of at least the given sizes, with
// every counter zero between launches (the reducing CTA resets its counter); it grows them on demand, synchronising the
// device when it does.  Launches that use it must be ordered on one stream.
struct DetScratch { float* part; unsigned* count; };
DetScratch det_scratch(size_t part_floats, size_t n_counters);      // part == NULL on failure (error text set)

#define IPLAN_REQUIRE(cond, ...)                 \
    do {                                         \
        if (!(cond)) {                           \
            iplan::set_error(__VA_ARGS__);       \
            return -1;                           \
        }                                        \
    } while (0)

// ---- parameter layouts (shared by host wrappers and kernels) ----------------------
__host__ __device__ inline int64_t pad4(int64_t x) { return (x + 3) & ~int64_t(3); }

struct GatLayout {      // nova/GAT_Net.py:18-39, state_dict order
    int64_t enc_w, enc_b;
    int64_t wih_f, whh_f, bih_f, bhh_f;
    int64_t wih_r, whh_r, bih_r, bhh_r;
    int64_t he_w, he_b;
    int64_t q_w, k_w, v_w, v_b;
    int64_t c_wih, c_whh, c_bih, c_bhh;
    int64_t total;
};
__host__ __device__ inline GatLayout gat_layout(int in_dim) {
    const int H = IPLAN_HID;
    GatLayout L;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t at = o; o = pad4(o + n); return at; };
    L.enc_w = take((int64_t)H * in_dim); L.enc_b = take(H);
    L.wih_f = take(3 * H * 2 * H); L.whh_f = take(3 * H * H); L.bih_f = take(3 * H); L.bhh_f = take(3 * H);
    L.wih_r = take(3 * H * 2 * H); L.whh_r = take(3 * H * H); L.bih_r = take(3 * H); L.bhh_r = take(3 * H);
    L.he_w = take(2 * 2 * H); L.he_b = take(2);
    L.q_w = take(H * H); L.k_w = take(H * H); L.v_w = take(H * H); L.v_b = take(H);
    L.c_wih = take(3 * H * H); L.c_whh = take(3 * H * H); L.c_bih = take(3 * H); L.c_bhh = take(3 * H);
    L.total = o;
    return L;
}

struct BehLayout {      // nova/behavior_net.py:12-15 (EncoderRNN), state_dict order
    int64_t lin_w, lin_b, wih, whh, bih, bhh, out_w, out_b, total;
};
__host__ __device__ inline BehLayout beh_layout(int obs_dim, int latent_dim) {
    const int E = IPLAN_HID;
    BehLayout L;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t at = o; o = pad4(o + n); return at; };
    L.lin_w = take((int64_t)E * obs_dim); L.lin_b = take(E);
    L.wih = take(3 * E * E); L.whh = take(3 * E * E); L.bih = take(3 * E); L.bhh = take(3 * E);
    L.out_w = take((int64_t)latent_dim * E); L.out_b = take(latent_dim);
    L.total = o;
    return L;
}

struct BfcLayout {      // nova/behavior_FC_net.py:6-37 (Encoder_3FC, Decoder_3FC), state_dict order
    int64_t w1, b1, w2, b2, w3, b3, total;
};
__host__ __device__ inline BfcLayout bfc_layout(int in_dim, int hidden, int out_dim) {
    BfcLayout L;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t at = o; o = pad4(o + n); return at; };
    L.w1 = take((int64_t)hidden * in_dim); L.b1 = take(hidden);
    L.w2 = take((int64_t)hidden * hidden); L.b2 = take(hidden);
    L.w3 = take((int64_t)out_dim * hidden); L.b3 = take(out_dim);
    L.total = o;
    return L;
}

// R_Actor / R_Critic trunk (utils/mappo_utils/mlp.py, rnn.py), state_dict order.
struct TrunkLayout {
    int64_t ln0_w, ln0_b;            // base.feature_norm
    int64_t fc1_w, fc1_b, ln1_w, ln1_b;   // base.mlp.fc1.{0,2}
    int64_t fch_w, fch_b, lnh_w, lnh_b;   // base.mlp.fc_h.{0,2}  (dead parameters)
    int64_t fc2_w, fc2_b, ln2_w, ln2_b;   // base.mlp.fc2.0.{0,2}
    int64_t wih, whh, bih, bhh;      // rnn.rnn.*_l0
    int64_t ln3_w, ln3_b;            // rnn.norm
    int64_t head_w, head_b;          // act.action_out.linear  |  v_out.{weight,bias}
    int64_t total;                   // (critic: + stddev, mean, mean_sq, debiasing_term)
};
__host__ __device__ inline TrunkLayout trunk_layout(int feat_dim, int head_out, bool critic) {
    const int R = IPLAN_RNN;
    TrunkLayout L;
    int64_t o = 0;
    auto take = [&](int64_t n) { int64_t at = o; o = pad4(o + n); return at; };
    L.ln0_w = take(feat_dim); L.ln0_b = take(feat_dim);
    L.fc1_w = take((int64_t)R * feat_dim); L.fc1_b = take(R); L.ln1_w = take(R); L.ln1_b = take(R);
    L.fch_w = take(R * R); L.fch_b = take(R); L.lnh_w = take(R); L.lnh_b = take(R);
    L.fc2_w = take(R * R); L.fc2_b = take(R); L.ln2_w = take(R); L.ln2_b = take(R);
    L.wih = take(3 * R * R); L.whh = take(3 * R * R); L.bih = take(3 * R); L.bhh = take(3 * R);
    L.ln3_w = take(R); L.ln3_b = take(R);
    L.head_w = take((int64_t)head_out * R); L.head_b = take(head_out);
    if (critic) { take(1); take(1); take(1); take(1); }
    L.total = o;
    return L;
}

#ifdef __CUDACC__
// Called by every thread of the CTA after it stored its share of the CTA's partial; true in the CTA that reduces the group
// (the partials of the others are then visible to it; read them with __ldcg).
__device__ __forceinline__ bool det_last_arrival(unsigned* counter, unsigned members) {
    __shared__ unsigned s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(counter, 1u);
        s_last = prev == members - 1;
        if (s_last) atomicExch(counter, 0u);
    }
    __syncthreads();
    if (s_last) __threadfence();
    return s_last != 0;
}

// ---- math ---------------------------------------------------------------------------
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float tanhf_acc(float x) { return tanhf(x); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- Philox4x32-10 counter RNG (Salmon et al. 2011) ----------------------------------
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0; key.y += W1;
    }
    return ctr;
}
// uniform in (0,1), never 0 or 1: the top 24 bits plus one half, scaled by 2^-24, capped at the largest float below 1.
// From 2^23 up the sum rounds to even in fp32, and 2^24 - 1 + 0.5 rounds to 2^24, i.e. exactly 1.0 (then log(1 - u) is
// -inf); the cap maps that one input to 1 - 2^-24 and leaves every other value, and so every noise stream, unchanged.
// oracle/philox.py restates this bit for bit.
__device__ __forceinline__ float u01(uint32_t x) { return fminf(((x >> 8) + 0.5f) * (1.0f / 16777216.0f), 0x1.fffffep-1f); }
#endif  // __CUDACC__

}  // namespace iplan
