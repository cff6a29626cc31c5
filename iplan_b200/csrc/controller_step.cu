// K1c — controller step: actor and critic forward for one timestep.
//
// Replaces DcntrlMAC.select_actions_ippo (reference controllers/dcntrl_controller.py:27-58):
// per agent  R_Actor.forward (modules/agents/ippo_actor.py:43-72) and R_Critic.forward
// (modules/critics/ippo_critic.py:47-65), i.e. for both nets
//   LN(F) -> Linear(F,64) -> ReLU -> LN -> Linear(64,64) -> ReLU -> LN      (mlp.py:24-56)
//   -> 1-step GRU(64) from the stored hidden -> LN                             (rnn.py:24-78)
//   actor: Linear(64,n_act), logits[avail==0] = -1e10, Categorical sample/mode, log-prob
//          (act.py:81-85, distributions.py:14-28,64-68);  critic: Linear(64,1) (popart.py:41-46)
// One CTA handles CTRL_ROWS envs of one agent; both nets share the staged input rows.
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>

#include "common.cuh"

namespace iplan {

constexpr int R = IPLAN_RNN;            // 64
constexpr int CTRL_THREADS = 256;
constexpr int CTRL_WARPS = CTRL_THREADS / 32;
constexpr int CTRL_ROWS = 18;            // at the Highway feature width 18 rows are what fits in 227 KB of shared memory
constexpr int CTRL_MT = (CTRL_ROWS + 15) / 16;   // MMA m-tiles per CTA
constexpr float LN_EPS = 1e-5f;

struct CtrlArgs {
    const float* actor; int64_t actor_stride;
    const float* critic; int64_t critic_stride;
    const float* feat; int64_t feat_sa, feat_se;
    const float* rnn_a_in; const float* rnn_c_in; float* rnn_a_out; float* rnn_c_out;
    int64_t rnn_sa, rnn_se, rnn_osa, rnn_ose;
    const uint8_t* avail; const float* uniforms;
    uint64_t seed, counter; int greedy;
    int32_t* actions; float* logp; float* values; float* logits;
    float* next_onehot; float* this_onehot;
    int n_envs, feat_dim, feat_ld, n_actions;
    int allow_vec;          // 0: always the scalar staging path (timing experiments: IPLAN_CTRL_VEC=0)
};

// y[k] = b[k] + sum_j W[k][j] * x[j]  for one output row k (64 inputs, x in shared memory)
__device__ __forceinline__ float dot64(const float* __restrict__ wrow, const float* x, float acc) {
    const float4* w4 = reinterpret_cast<const float4*>(wrow);
    const float4* x4 = reinterpret_cast<const float4*>(x);
#pragma unroll
    for (int q = 0; q < R / 4; ++q) {
        const float4 w = __ldg(w4 + q);
        const float4 v = x4[q];
        acc = fmaf(w.x, v.x, acc); acc = fmaf(w.y, v.y, acc);
        acc = fmaf(w.z, v.z, acc); acc = fmaf(w.w, v.w, acc);
    }
    return acc;
}

// LayerNorm over 64 features held as (v0 = feature lane, v1 = feature lane+32)
__device__ __forceinline__ void ln64(float& v0, float& v1, const float* __restrict__ g, const float* __restrict__ bta, int lane) {
    const float mean = warp_sum(v0 + v1) * (1.0f / R);
    const float d0 = v0 - mean, d1 = v1 - mean;
    const float var = warp_sum(d0 * d0 + d1 * d1) * (1.0f / R);
    const float rstd = 1.0f / sqrtf(var + LN_EPS);
    v0 = d0 * rstd * g[lane] + bta[lane];
    v1 = d1 * rstd * g[lane + 32] + bta[lane + 32];
}

__device__ __forceinline__ void csplit(float x, float y, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void cmma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cldsm(uint32_t (&r)[4], const void* p) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}


constexpr int TAP = R + 8;               // fp32 pitch of the tail's activation rows: conflict-free float2 fragment reads

// out[row][8 nt + c] = bias[8 nt + c] + sum_k A[row][k] * Wg[(8 nt + c) * 64 + k]   for nt in [nt0, nt1), row < CTRL_ROWS
// A: shared memory rows (pitch TAP) of ONE net; Wg / bias: global.  K = 64: 4 k-blocks x 3 MMAs (f16 hi/lo split)
// per accumulator.  The weight fragments are read from global exactly once per CTA (a quad reads 32 contiguous
// bytes of one weight row), instead of once per row as a per-row dot product would.
__device__ __forceinline__ void tail_gemm64(const float* A, const float* __restrict__ Wg, const float* __restrict__ bias,
                                            int nt0, int nt1, float* out, int ldout, int lane) {
    const int gq = lane >> 2, tq = lane & 3;
    uint32_t ah[CTRL_MT][4][4], al[CTRL_MT][4][4];
#pragma unroll
    for (int m = 0; m < CTRL_MT; ++m) {
        const float* x0 = A + min(16 * m + gq, CTRL_ROWS - 1) * TAP + 2 * tq;
        const float* x1 = A + min(16 * m + gq + 8, CTRL_ROWS - 1) * TAP + 2 * tq;
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            const float2 v00 = *reinterpret_cast<const float2*>(x0 + 16 * kb);
            const float2 v10 = *reinterpret_cast<const float2*>(x1 + 16 * kb);
            const float2 v01 = *reinterpret_cast<const float2*>(x0 + 16 * kb + 8);
            const float2 v11 = *reinterpret_cast<const float2*>(x1 + 16 * kb + 8);
            csplit(v00.x, v00.y, ah[m][kb][0], al[m][kb][0]);
            csplit(v10.x, v10.y, ah[m][kb][1], al[m][kb][1]);
            csplit(v01.x, v01.y, ah[m][kb][2], al[m][kb][2]);
            csplit(v11.x, v11.y, ah[m][kb][3], al[m][kb][3]);
        }
    }
    float2 wv[2][8];                                            // weight fragments of the current and the next n-tile
    auto load_w = [&](int nt, float2 (&w)[8]) {
        const float* wr = Wg + (size_t)(8 * nt + gq) * R + 2 * tq;
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            w[2 * kb] = __ldg(reinterpret_cast<const float2*>(wr + 16 * kb));
            w[2 * kb + 1] = __ldg(reinterpret_cast<const float2*>(wr + 16 * kb + 8));
        }
    };
    load_w(nt0, wv[0]);
#pragma unroll 2
    for (int nt = nt0; nt < nt1; ++nt) {
        const int cur = (nt - nt0) & 1;
        if (nt + 1 < nt1) load_w(nt + 1, wv[cur ^ 1]);
        uint32_t bh[4][2], bl[4][2];
#pragma unroll
        for (int kb = 0; kb < 4; ++kb) {
            csplit(wv[cur][2 * kb].x, wv[cur][2 * kb].y, bh[kb][0], bl[kb][0]);
            csplit(wv[cur][2 * kb + 1].x, wv[cur][2 * kb + 1].y, bh[kb][1], bl[kb][1]);
        }
        const int c0 = 8 * nt + 2 * tq;
        const float b0 = bias[c0], b1 = bias[c0 + 1];
#pragma unroll
        for (int m = 0; m < CTRL_MT; ++m) {
            float acc[4] = {b0, b1, b0, b1};
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) {
                cmma(acc, ah[m][kb], bh[kb][0], bh[kb][1]);
                cmma(acc, al[m][kb], bh[kb][0], bh[kb][1]);
                cmma(acc, ah[m][kb], bl[kb][0], bl[kb][1]);
            }
            const int r0 = 16 * m + gq, r1 = r0 + 8;
            if (r0 < CTRL_ROWS) *reinterpret_cast<float2*>(out + r0 * ldout + c0) = make_float2(acc[0], acc[1]);
            if (r1 < CTRL_ROWS) *reinterpret_cast<float2*>(out + r1 * ldout + c0) = make_float2(acc[2], acc[3]);
        }
    }
}

__global__ void __launch_bounds__(CTRL_THREADS, 1) controller_step_kernel(CtrlArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int ag = blockIdx.y, b0 = blockIdx.x * CTRL_ROWS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int F = a.feat_dim;
    const int K16 = (F + 15) & ~15, LDH = K16 + 8;              // f16 row pitch: conflict-free ldmatrix
    __half* s_yh = reinterpret_cast<__half*>(smem_raw);         // [ROWS][LDH] normalised rows, f16 hi
    __half* s_yl = s_yh + CTRL_ROWS * LDH;                      // [ROWS][LDH] ... f16 lo
    // the f16 rows are dead after fc1; the GRU projections of the tail reuse their space (s_gi / s_gh below)
    const size_t stage_bytes = max((size_t)2 * CTRL_ROWS * LDH * sizeof(__half), (size_t)4 * CTRL_ROWS * 3 * R * sizeof(float));
    float* s_z = reinterpret_cast<float*>(smem_raw + stage_bytes);   // [2][ROWS][64] fc1 pre-activations
    float* s_act = s_z + 2 * CTRL_ROWS * R;     // [2*ROWS][TAP] per-task activation rows
    float* s_h0 = s_act + 2 * CTRL_ROWS * TAP;  // [2*ROWS][TAP] per-task hidden input
    float* s_stat = s_h0 + 2 * CTRL_ROWS * TAP; // [ROWS][2] mean, rstd
    float* s_gi = reinterpret_cast<float*>(smem_raw);    // [2*ROWS][192] GRU input projections (aliases s_yh/s_yl: dead after fc1)
    float* s_gh = s_gi + 2 * CTRL_ROWS * 3 * R;          // [2*ROWS][192] GRU hidden projections

    // ---- LayerNorm statistics over the F input features ------------------------------------------------
    // Vector path (rows 16-byte aligned, as in the packed episode store): a warp owns rows warp, warp + 8, ...; a row is read
    // with ONE batch of float4 loads per net (all in flight together), statistics from registers.  The scalar path keeps two
    // passes over L1/L2.
    constexpr int V4 = 20, RPW = (CTRL_ROWS + CTRL_WARPS - 1) / CTRL_WARPS;
    const bool vec = a.allow_vec && (reinterpret_cast<uintptr_t>(a.feat) & 15) == 0 && (a.feat_sa & 3) == 0 && (a.feat_se & 3) == 0 &&
                     a.feat_ld >= ((F + 3) & ~3) && K16 <= 128 * V4 && 2 * K16 <= 4 * CTRL_ROWS * TAP &&
                     ((reinterpret_cast<uintptr_t>(a.actor) | reinterpret_cast<uintptr_t>(a.critic)) & 15) == 0 &&
                     (a.actor_stride & 3) == 0 && (a.critic_stride & 3) == 0;
    float mean_r[RPW], rstd_r[RPW];
#pragma unroll
    for (int k = 0; k < RPW; ++k) { mean_r[k] = 0.0f; rstd_r[k] = 0.0f; }
    if (!vec) {
        for (int r = warp; r < CTRL_ROWS; r += CTRL_WARPS) {
            const int b = min(b0 + r, a.n_envs - 1);
            const float* src = a.feat + ag * a.feat_sa + b * a.feat_se;
            float s = 0.0f;
            for (int f = lane; f < F; f += 32) s += src[f];
            const float mean = warp_sum(s) / (float)F;
            float v = 0.0f;
            for (int f = lane; f < F; f += 32) { const float d = src[f] - mean; v = fmaf(d, d, v); }
            const float var = warp_sum(v) / (float)F;
            if (lane == 0) { s_stat[2 * r] = mean; s_stat[2 * r + 1] = 1.0f / sqrtf(var + LN_EPS); }
        }
        __syncthreads();
    }
    // ---- fc1 for both nets on the tensor cores: [16 rows x K] . W1^T, one 8-output n-tile per warp
    const int gq = lane >> 2, tq = lane & 3;
    for (int net = 0; net < 2; ++net) {
        const float* P = net == 0 ? a.actor + (int64_t)ag * a.actor_stride : a.critic + (int64_t)ag * a.critic_stride;
        const TrunkLayout L = trunk_layout(F, net == 0 ? a.n_actions : 1, net == 1);
        if (vec) {                                               // y = LN(x) as f16 hi + lo, a row per warp pass
            // this net's LayerNorm gamma / beta: staged once in shared memory (the tail's activation rows, unused until both
            // fc1 products are done), so that the row passes below wait for global memory once per row, not once per float4
            float4* g4 = reinterpret_cast<float4*>(s_act);
            float4* bt4 = g4 + K16 / 4;
            {
                const float4* gg4 = reinterpret_cast<const float4*>(P + L.ln0_w);
                const float4* gb4 = reinterpret_cast<const float4*>(P + L.ln0_b);
                const int n4 = (F + 3) >> 2;
                for (int i = tid; i < n4; i += CTRL_THREADS) { g4[i] = __ldg(gg4 + i); bt4[i] = __ldg(gb4 + i); }
            }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < RPW; ++k) {
                const int r = warp + CTRL_WARPS * k;
                if (r < CTRL_ROWS) {
                    const int b = min(b0 + r, a.n_envs - 1);
                    const float4* src4 = reinterpret_cast<const float4*>(a.feat + ag * a.feat_sa + b * a.feat_se);
                    float4 xv[V4];
#pragma unroll
                    for (int j = 0; j < V4; ++j) {
                        const int f = 4 * (lane + 32 * j);
                        xv[j] = f < F ? __ldg(src4 + lane + 32 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (f + 1 >= F) xv[j].y = 0.0f;                 // the row's last float4 may run past F
                        if (f + 2 >= F) xv[j].z = 0.0f;
                        if (f + 3 >= F) xv[j].w = 0.0f;
                    }
                    if (net == 0) {
                        float sm = 0.0f;
#pragma unroll
                        for (int j = 0; j < V4; ++j) sm += (xv[j].x + xv[j].y) + (xv[j].z + xv[j].w);
                        const float mean = warp_sum(sm) / (float)F;
                        float vs = 0.0f;
#pragma unroll
                        for (int j = 0; j < V4; ++j) {
                            const int f = 4 * (lane + 32 * j);
                            const float d0 = xv[j].x - mean, d1 = xv[j].y - mean, d2 = xv[j].z - mean, d3 = xv[j].w - mean;
                            if (f < F) vs = fmaf(d0, d0, vs);
                            if (f + 1 < F) vs = fmaf(d1, d1, vs);
                            if (f + 2 < F) vs = fmaf(d2, d2, vs);
                            if (f + 3 < F) vs = fmaf(d3, d3, vs);
                        }
                        mean_r[k] = mean;
                        rstd_r[k] = 1.0f / sqrtf(warp_sum(vs) / (float)F + LN_EPS);
                    }
                    const float mean = mean_r[k], rstd = rstd_r[k];
#pragma unroll
                    for (int j = 0; j < V4; ++j) {
                        const int f = 4 * (lane + 32 * j);
                        if (f < K16) {
                            float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (f < F) {
                                const float4 g = g4[lane + 32 * j], bt = bt4[lane + 32 * j];
                                y.x = (xv[j].x - mean) * rstd * g.x + bt.x;
                                y.y = f + 1 < F ? (xv[j].y - mean) * rstd * g.y + bt.y : 0.0f;
                                y.z = f + 2 < F ? (xv[j].z - mean) * rstd * g.z + bt.z : 0.0f;
                                y.w = f + 3 < F ? (xv[j].w - mean) * rstd * g.w + bt.w : 0.0f;
                            }
                            uint32_t h0, l0, h1, l1;
                            csplit(y.x, y.y, h0, l0);
                            csplit(y.z, y.w, h1, l1);
                            *reinterpret_cast<uint2*>(s_yh + r * LDH + f) = make_uint2(h0, h1);
                            *reinterpret_cast<uint2*>(s_yl + r * LDH + f) = make_uint2(l0, l1);
                        }
                    }
                }
            }
        } else
        for (int f = tid; f < K16; f += CTRL_THREADS) {          // y = LN(x) as f16 hi + lo
            const float g = f < F ? P[L.ln0_w + f] : 0.0f;
            const float bt = f < F ? P[L.ln0_b + f] : 0.0f;
#pragma unroll 2
            for (int r = 0; r < CTRL_ROWS; ++r) {
                const int b = min(b0 + r, a.n_envs - 1);
                const float x = f < F ? a.feat[ag * a.feat_sa + b * a.feat_se + f] : 0.0f;
                const float y = f < F ? (x - s_stat[2 * r]) * s_stat[2 * r + 1] * g + bt : 0.0f;
                const __half h = __float2half_rn(y);
                s_yh[r * LDH + f] = h;
                s_yl[r * LDH + f] = __float2half_rn(y - __half2float(h));
            }
        }
        __syncthreads();
        float acc[CTRL_MT][4];
#pragma unroll
        for (int m = 0; m < CTRL_MT; ++m) acc[m][0] = acc[m][1] = acc[m][2] = acc[m][3] = 0.0f;
        const float* w1 = P + L.fc1_w + (int64_t)(warp * 8 + gq) * F;       // this lane's weight row
        const __half* ah_base[CTRL_MT];
        const __half* al_base[CTRL_MT];
#pragma unroll
        for (int m = 0; m < CTRL_MT; ++m) {                      // rows past CTRL_ROWS re-read the last row (unused)
            const int row = min(16 * m + (lane & 15), CTRL_ROWS - 1);
            ah_base[m] = s_yh + row * LDH + (lane >> 4) * 8;
            al_base[m] = s_yl + row * LDH + (lane >> 4) * 8;
        }
        const int nkb = K16 >> 4;
        // weights of one chunk (4 k-blocks) as B-fragment scalars; the NEXT chunk's loads are issued before
        // the current chunk's MMAs, so the L2 round trip overlaps the tensor work
        auto load_chunk = [&](int kc, float (&w)[4][4]) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int k0 = 16 * (kc + q) + 2 * tq;
                const bool on = kc + q < nkb;
                w[q][0] = (on && k0 < F) ? __ldg(w1 + k0) : 0.0f;
                w[q][1] = (on && k0 + 1 < F) ? __ldg(w1 + k0 + 1) : 0.0f;
                w[q][2] = (on && k0 + 8 < F) ? __ldg(w1 + k0 + 8) : 0.0f;
                w[q][3] = (on && k0 + 9 < F) ? __ldg(w1 + k0 + 9) : 0.0f;
            }
        };
        float wv[4][4], wn[4][4];
        load_chunk(0, wv);
        for (int kc = 0; kc < nkb; kc += 4) {                    // 4 k-blocks: 12 chained MMAs, then fp32 add
            load_chunk(kc + 4, wn);
            float part[CTRL_MT][4];
#pragma unroll
            for (int m = 0; m < CTRL_MT; ++m) part[m][0] = part[m][1] = part[m][2] = part[m][3] = 0.0f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (kc + q < nkb) {
                    uint32_t bh0, bl0, bh1, bl1;
                    csplit(wv[q][0], wv[q][1], bh0, bl0);
                    csplit(wv[q][2], wv[q][3], bh1, bl1);
#pragma unroll
                    for (int m = 0; m < CTRL_MT; ++m) {
                        uint32_t ah[4], al[4];
                        cldsm(ah, ah_base[m] + 16 * (kc + q));
                        cldsm(al, al_base[m] + 16 * (kc + q));
                        cmma(part[m], ah, bh0, bh1);
                        cmma(part[m], al, bh0, bh1);
                        cmma(part[m], ah, bl0, bl1);
                    }
                }
            }
#pragma unroll
            for (int m = 0; m < CTRL_MT; ++m) {
                acc[m][0] += part[m][0]; acc[m][1] += part[m][1]; acc[m][2] += part[m][2]; acc[m][3] += part[m][3];
            }
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int e = 0; e < 4; ++e) wv[q][e] = wn[q][e];
        }
        const int n0 = warp * 8 + 2 * tq;
#pragma unroll
        for (int m = 0; m < CTRL_MT; ++m)
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
                const int row = 16 * m + gq + 8 * hr;
                if (row < CTRL_ROWS) {
                    s_z[(net * CTRL_ROWS + row) * R + n0] = acc[m][2 * hr] + P[L.fc1_b + n0];
                    s_z[(net * CTRL_ROWS + row) * R + n0 + 1] = acc[m][2 * hr + 1] + P[L.fc1_b + n0 + 1];
                }
            }
        __syncthreads();
    }

    // ---- tails.  Row-wise pieces (LayerNorm, gates, heads): 2*ROWS (net,row) tasks, one warp each;
    //      the 64-wide products (fc2, GRU projections) on the tensor cores, weights read once per CTA.
    const float* const Pa = a.actor + (int64_t)ag * a.actor_stride;
    const float* const Pc = a.critic + (int64_t)ag * a.critic_stride;
    // actor and critic trunks share every offset up to head_w (state_dict order); only head_b differs
    const TrunkLayout L = trunk_layout(F, a.n_actions, false);
    const int64_t critic_head_b = trunk_layout(F, 1, true).head_b;
    for (int task = warp; task < 2 * CTRL_ROWS; task += CTRL_WARPS) {       // ReLU -> LN1; stage h0
        const int net = task / CTRL_ROWS, r = task % CTRL_ROWS;
        const int bc = min(b0 + r, a.n_envs - 1);
        const float* P = net == 0 ? Pa : Pc;
        const float* hin = (net == 0 ? a.rnn_a_in : a.rnn_c_in) + ag * a.rnn_sa + bc * a.rnn_se;
        s_h0[task * TAP + lane] = hin[lane]; s_h0[task * TAP + lane + 32] = hin[lane + 32];
        float v0 = fmaxf(s_z[task * R + lane], 0.0f), v1 = fmaxf(s_z[task * R + lane + 32], 0.0f);
        ln64(v0, v1, P + L.ln1_w, P + L.ln1_b, lane);
        s_act[task * TAP + lane] = v0; s_act[task * TAP + lane + 32] = v1;
    }
    __syncthreads();
    {   // fc2: warp -> (net, two n-tiles); output overwrites s_z
        const int net = warp >> 2, nt0 = 2 * (warp & 3);
        const float* P = net == 0 ? Pa : Pc;
        tail_gemm64(s_act + net * CTRL_ROWS * TAP, P + L.fc2_w, P + L.fc2_b, nt0, nt0 + 2,
                    s_z + net * CTRL_ROWS * R, R, lane);
    }
    __syncthreads();
    for (int task = warp; task < 2 * CTRL_ROWS; task += CTRL_WARPS) {       // ReLU -> LN2
        const int net = task / CTRL_ROWS;
        const float* P = net == 0 ? Pa : Pc;
        float v0 = fmaxf(s_z[task * R + lane], 0.0f), v1 = fmaxf(s_z[task * R + lane + 32], 0.0f);
        ln64(v0, v1, P + L.ln2_w, P + L.ln2_b, lane);
        s_act[task * TAP + lane] = v0; s_act[task * TAP + lane + 32] = v1;
    }
    __syncthreads();
    {   // GRU projections: warp -> (net, input | hidden matrix, half of the 24 n-tiles)
        const int net = warp >> 2, hid = (warp >> 1) & 1, nt0 = 12 * (warp & 1);
        const float* P = net == 0 ? Pa : Pc;
        tail_gemm64((hid ? s_h0 : s_act) + net * CTRL_ROWS * TAP, P + (hid ? L.whh : L.wih),
                    P + (hid ? L.bhh : L.bih), nt0, nt0 + 12,
                    (hid ? s_gh : s_gi) + net * CTRL_ROWS * 3 * R, 3 * R, lane);
    }
    __syncthreads();
    for (int task = warp; task < 2 * CTRL_ROWS; task += CTRL_WARPS) {
        const int net = task / CTRL_ROWS, r = task % CTRL_ROWS;
        const int b = b0 + r;
        const bool live = b < a.n_envs;          // warp-uniform
        const int bc = live ? b : a.n_envs - 1;
        const float* P = net == 0 ? Pa : Pc;
        float* act = s_act + task * TAP;
        const float* h0 = s_h0 + task * TAP;
        const float* gi = s_gi + task * 3 * R;
        const float* gh = s_gh + task * 3 * R;
        // GRU gates: hidden units c = lane, lane+32; gate rows r: c, z: 64+c, n: 128+c
        float hn[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int c = lane + 32 * u;
            const float rg = sigmoidf_acc(gi[c] + gh[c]);
            const float zg = sigmoidf_acc(gi[R + c] + gh[R + c]);
            const float ng = tanhf_acc(gi[2 * R + c] + rg * gh[2 * R + c]);
            hn[u] = (1.0f - zg) * ng + zg * h0[c];
        }
        float v0, v1;
        if (live) {
            float* hout = (net == 0 ? a.rnn_a_out : a.rnn_c_out) + ag * a.rnn_osa + b * a.rnn_ose;
            hout[lane] = hn[0]; hout[lane + 32] = hn[1];
        }
        v0 = hn[0]; v1 = hn[1];
        ln64(v0, v1, P + L.ln3_w, P + L.ln3_b, lane);
        __syncwarp();
        act[lane] = v0; act[lane + 32] = v1;
        __syncwarp();
        const int64_t ob = (int64_t)ag * a.n_envs + bc;
        if (net == 1) {
            const float val = warp_sum(v0 * P[L.head_w + lane] + v1 * P[L.head_w + lane + 32]) + P[critic_head_b];
            if (live && lane == 0) a.values[ob] = val;
        } else {
            const int nA = a.n_actions;
            float lg = -INFINITY;
            if (lane < nA) {
                lg = dot64(P + L.head_w + lane * R, act, P[L.head_b + lane]);
                if (a.avail && a.avail[ob * nA + lane] == 0) lg = -1e10f;
            }
            const float mx = warp_max(lg);
            const float ex = lane < nA ? expf(lg - mx) : 0.0f;
            const float den = warp_sum(ex);
            const float lp = lg - mx - logf(den);            // log-softmax
            const float pr = lane < nA ? expf(lp) : 0.0f;
            int action;
            if (a.greedy) {
                const float pmx = warp_max(pr);
                const unsigned m = __ballot_sync(0xffffffffu, lane < nA && pr == pmx);
                action = __ffs(m) - 1;                       // first maximal index (argmax)
            } else {
                float uu;
                if (a.uniforms) uu = a.uniforms[ob];
                else {
                    const uint4 rnd = philox4x32(make_uint4((uint32_t)ob, (uint32_t)(ob >> 32), (uint32_t)a.counter,
                                                            (uint32_t)(a.counter >> 32)),
                                                 make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32) ^ 0x5bd1e995u));
                    uu = u01(rnd.x);
                }
                float cdf = pr;                              // inclusive scan over the first lanes
#pragma unroll
                for (int o = 1; o < IPLAN_MAX_ACT; o <<= 1) {
                    const float t = __shfl_up_sync(0xffffffffu, cdf, o);
                    if (lane >= o) cdf += t;
                }
                const unsigned m = __ballot_sync(0xffffffffu, lane < nA && uu >= cdf);
                action = min(__popc(m), nA - 1);
            }
            const float lp_a = __shfl_sync(0xffffffffu, lp, action);
            if (live) {
                if (lane == 0) { a.actions[ob] = action; a.logp[ob] = lp_a; }
                if (a.logits && lane < nA) a.logits[ob * nA + lane] = lg;
                if (lane < nA) {
                    const float oh = lane == action ? 1.0f : 0.0f;
                    if (a.next_onehot) a.next_onehot[ag * a.feat_sa + b * a.feat_se + lane] = oh;
                    if (a.this_onehot) a.this_onehot[ag * a.feat_sa + b * a.feat_se + lane] = oh;
                }
            }
        }
        __syncwarp();
    }
}

}  // namespace iplan

extern "C" int iplan_controller_step(const float* actor_params, int64_t actor_stride,
                                     const float* critic_params, int64_t critic_stride,
                                     const float* feat, int64_t feat_stride_agent, int64_t feat_stride_env,
                                     const float* rnn_a_in, const float* rnn_c_in,
                                     float* rnn_a_out, float* rnn_c_out,
                                     int64_t rnn_stride_agent, int64_t rnn_stride_env,
                                     int64_t rnn_out_stride_agent, int64_t rnn_out_stride_env,
                                     const uint8_t* avail, const float* uniforms,
                                     uint64_t seed, uint64_t counter, int greedy,
                                     int32_t* actions, float* logp, float* values, float* logits,
                                     float* next_onehot, float* this_onehot,
                                     int n_envs, int n_agents, int feat_dim, int n_actions,
                                     void* stream) {
    using namespace iplan;
    IPLAN_REQUIRE(n_actions > 0 && n_actions <= IPLAN_MAX_ACT, "controller_step: n_actions %d not in [1,%d]", n_actions, IPLAN_MAX_ACT);
    IPLAN_REQUIRE(n_envs > 0 && n_agents > 0 && n_agents <= 65535 && feat_dim > 0, "controller_step: bad sizes");
    IPLAN_REQUIRE(actor_params && critic_params && feat && rnn_a_in && rnn_c_in && rnn_a_out && rnn_c_out && actions && logp && values,
                  "controller_step: null pointer");
    CtrlArgs a;
    a.actor = actor_params; a.actor_stride = actor_stride; a.critic = critic_params; a.critic_stride = critic_stride;
    a.feat = feat; a.feat_sa = feat_stride_agent; a.feat_se = feat_stride_env;
    a.rnn_a_in = rnn_a_in; a.rnn_c_in = rnn_c_in; a.rnn_a_out = rnn_a_out; a.rnn_c_out = rnn_c_out;
    a.rnn_sa = rnn_stride_agent; a.rnn_se = rnn_stride_env;
    a.rnn_osa = rnn_out_stride_agent; a.rnn_ose = rnn_out_stride_env;
    a.avail = avail; a.uniforms = uniforms; a.seed = seed; a.counter = counter; a.greedy = greedy;
    a.actions = actions; a.logp = logp; a.values = values; a.logits = logits;
    a.next_onehot = next_onehot; a.this_onehot = this_onehot;
    a.n_envs = n_envs; a.feat_dim = feat_dim; a.feat_ld = (feat_dim + 3) & ~3; a.n_actions = n_actions;
    static const int allow_vec = getenv("IPLAN_CTRL_VEC") ? atoi(getenv("IPLAN_CTRL_VEC")) : 1;
    a.allow_vec = allow_vec;
    const size_t ldh = ((feat_dim + 15) & ~15) + 8;
    const size_t stage = std::max((size_t)2 * CTRL_ROWS * ldh * 2, (size_t)4 * CTRL_ROWS * 3 * R * sizeof(float));
    const size_t smem = stage + ((size_t)2 * CTRL_ROWS * R + 4 * CTRL_ROWS * TAP + 2 * CTRL_ROWS) * sizeof(float);
    IPLAN_REQUIRE(smem <= 227 * 1024, "controller_step: feat_dim %d needs %zu B of shared memory", feat_dim, smem);
    static size_t configured = 0;
    if (smem > configured) {
        cudaError_t e = cudaFuncSetAttribute(controller_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("controller_step: smem attr %zu: %s", smem, cudaGetErrorString(e)); return (int)e; }
        configured = smem;
    }
    dim3 grid((n_envs + CTRL_ROWS - 1) / CTRL_ROWS, n_agents);
    controller_step_kernel<<<grid, CTRL_THREADS, smem, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("controller_step");
}
