// K2 and the IPPO update — kernels behind IPPOLearner.train (reference
// learners/ippo_learner.py:227-317) for ALL agents at once (agents are independent
// parameter sets; the reference's Python loop over agents is a grid dimension here).
//
// Rows: agent a owns the matrix X_a[Rall][Fp], Rall = Bf*(T+1), row (b,t) = the controller
// input of episode b at time t (EpisodeBatch packed layout).  "net" = 2*a + {0 actor, 1 critic}.
//
// Per PPO epoch (reference :284-310; num_mini_batch = 1 so a minibatch is every training
// row in permuted order — the permutation only reorders sums; with more mini-batches gather_rows copies each one's
// rows into dense buffers and the same kernels run on those, once per mini-batch):
//   fc1_prep        fold LayerNorm(F) into fc1:  W' = gamma.W1, ws = sum_f W', c = W1.beta + b1
//   fc1_fwd         Z1 = rstd_r (X W'^T - mu_r ws) + c                      (both nets, N=128)
//   ln_relu_fwd     A1 = LN(ReLU(Z1));  linear_fwd Z2 = A1 W2^T + b2;  A2 = LN(ReLU(Z2))
//   linear_fwd      GI = A2 W_ih^T + b_ih ;  GH = H0 W_hh^T + b_hh
//   gru_head        GRU gates -> H1 -> LN -> heads; train mode fuses the PPO losses
//                   (clipped ratio + entropy; clipped one-sided-Huber value loss, :128-159,
//                   :185-197) and their backward through heads, LN and the GRU gates
//   linear_dw/dx, ln_relu_bwd, fc1_bwd, fc1_grad_finish     the rest of the backward
//   grad_norm + adam  clip_grad_norm_(10) and Adam(lr, eps) (:205-223, :74-81)
// Once per train(): row_stats (LayerNorm statistics of X rows, parameter-free), the
// forward pre-pass (values on all T+1 steps, old log-probs) and K2a gae_adv
// (compute_returns :344-365 + advantage moments :272-279).
#include <cuda_fp16.h>

#include <algorithm>
#include <stdlib.h>

#include "common.cuh"

namespace iplan {

constexpr int RH = IPLAN_RNN;       // 64
constexpr int RH3 = 3 * RH;          // 192
constexpr float LEPS = 1e-5f;

// a per-net row buffer: element [agent][type][row][col]
struct RowBuf {
    float* p; int64_t sa, sn; int ld;
    __device__ __forceinline__ float* row(int a, int type, int64_t r) const { return p + a * sa + type * sn + r * ld; }
};

struct NetParams {       // flat parameter / gradient buffers, one per net type
    const float* actor; const float* critic; int64_t actor_stride, critic_stride;
    __device__ __forceinline__ const float* net(int a, int type) const {
        return type == 0 ? actor + a * actor_stride : critic + a * critic_stride;
    }
};
struct NetGrads {
    float* actor; float* critic; int64_t actor_stride, critic_stride;
    __device__ __forceinline__ float* net(int a, int type) const {
        return type == 0 ? actor + a * actor_stride : critic + a * critic_stride;
    }
};

// ---------------------------------------------------------------------------------------
// row_stats: mean / rstd of LayerNorm(F) for every row of X (parameter-free, once per train)
// ---------------------------------------------------------------------------------------
__global__ void row_stats_kernel(const float* __restrict__ X, int64_t x_sa, int ldx, int F, int64_t rows,
                                 float* __restrict__ stat /* [A][rows][2] */) {
    const int a = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = warp; r < rows; r += nwarps) {
        const float* x = X + a * x_sa + r * ldx;
        float s = 0.0f;
        for (int f = lane; f < F; f += 32) s += x[f];
        const float mean = warp_sum(s) / (float)F;
        float v = 0.0f;
        for (int f = lane; f < F; f += 32) { const float d = x[f] - mean; v = fmaf(d, d, v); }
        const float var = warp_sum(v) / (float)F;
        if (lane == 0) {
            stat[(a * rows + r) * 2] = mean;
            stat[(a * rows + r) * 2 + 1] = 1.0f / sqrtf(var + LEPS);
        }
    }
}

// fc1_grad_finish: from G, S = colsum(dZ1), M = sum_r dZ1s*mu  ->  grads of fc1.W, LN0 gamma/beta
//   dW1[k][f] = gamma[f]*(G[k][f] - M[k]) + beta[f]*S[k];  dgamma[f] = sum_k W1[k][f]*(G[k][f]-M[k]);
//   dbeta[f] = sum_k W1[k][f]*S[k]          (fc1.bias grad = S is written by ln_relu_bwd)
__global__ void fc1_grad_finish_kernel(NetParams P, NetGrads Gr, int F, const float* __restrict__ G, int ldg,
                                       const float* __restrict__ SM /* [A][2][128]: S | M */) {
    const int a = blockIdx.y, type = blockIdx.z;
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    const float* p = P.net(a, type);
    float* g = Gr.net(a, type);
    const TrunkLayout L = trunk_layout(F, 1, false);
    const float gam = p[L.ln0_w + f], bet = p[L.ln0_b + f];
    float dg = 0.0f, db = 0.0f;
    for (int k = 0; k < RH; ++k) {
        const int kk = type * 64 + k;
        const float gv = G[((int64_t)a * 128 + kk) * ldg + f] - SM[(a * 2 + 1) * 128 + kk];
        const float s = SM[(a * 2 + 0) * 128 + kk];
        const float w = p[L.fc1_w + (int64_t)k * F + f];
        g[L.fc1_w + (int64_t)k * F + f] = gam * gv + bet * s;
        dg = fmaf(w, gv, dg);
        db = fmaf(w, s, db);
    }
    g[L.ln0_w + f] = dg;
    g[L.ln0_b + f] = db;
}

// Linear layers on 64-wide activations (fc2, GRU projections): tensor-core kernels
#include "lin64_mma.cuh"

// ---------------------------------------------------------------------------------------
// LayerNorm(ReLU(z)) forward / backward on 64-wide rows; one warp per (row), lane owns c, c+32
// ---------------------------------------------------------------------------------------
__global__ void ln_relu_fwd_kernel(RowBuf z, RowBuf out, NetParams P, int64_t g_off, int64_t b_off, int64_t rows, int n_types) {
    const int a = blockIdx.y / n_types, type = blockIdx.y % n_types;
    const int lane = threadIdx.x & 31;
    const float* p = P.net(a, type);
    const float g0 = p[g_off + lane], g1 = p[g_off + lane + 32], b0 = p[b_off + lane], b1 = p[b_off + lane + 32];
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = warp; r < rows; r += nwarps) {
        const float* zr = z.row(a, type, r);
        const float v0 = fmaxf(zr[lane], 0.0f), v1 = fmaxf(zr[lane + 32], 0.0f);
        const float mean = warp_sum(v0 + v1) * (1.0f / RH);
        const float d0 = v0 - mean, d1 = v1 - mean;
        const float rstd = 1.0f / sqrtf(warp_sum(d0 * d0 + d1 * d1) * (1.0f / RH) + LEPS);
        float* o = out.row(a, type, r);
        o[lane] = d0 * rstd * g0 + b0;
        o[lane + 32] = d1 * rstd * g1 + b1;
    }
}

// dz = ReLU'(z) * LNbwd(dout);  z buffer is overwritten with dz (times `scale_r` = rstd of the
// input LayerNorm when this is layer 1, so that fc1_bwd is a plain product);  accumulates
// d gamma, d beta of this LN, the bias gradient of the preceding Linear (colsum dz) and, for
// layer 1, S = colsum(dz) and M = sum_r dz*rstd_r*mean_r.
__global__ void ln_relu_bwd_kernel(RowBuf z, RowBuf dout, NetParams P, NetGrads Gr, int64_t g_off, int64_t b_off,
                                   int64_t lin_b_off, int64_t rows, int n_types,
                                   const float* __restrict__ stat /* NULL or [A][rows][2] */,
                                   float* __restrict__ SM /* NULL or [A][2][128] */) {
    const int a = blockIdx.y / n_types, type = blockIdx.y % n_types;
    const int lane = threadIdx.x & 31;
    const float* p = P.net(a, type);
    const float g0 = p[g_off + lane], g1 = p[g_off + lane + 32];
    float dg0 = 0, dg1 = 0, db0 = 0, db1 = 0, s0 = 0, s1 = 0, m0 = 0, m1 = 0;
    const int64_t warp = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t r = warp; r < rows; r += nwarps) {
        float* zr = z.row(a, type, r);
        const float* dr = dout.row(a, type, r);
        const float z0 = zr[lane], z1 = zr[lane + 32];
        const float v0 = fmaxf(z0, 0.0f), v1 = fmaxf(z1, 0.0f);
        const float mean = warp_sum(v0 + v1) * (1.0f / RH);
        const float c0 = v0 - mean, c1 = v1 - mean;
        const float rstd = 1.0f / sqrtf(warp_sum(c0 * c0 + c1 * c1) * (1.0f / RH) + LEPS);
        const float x0 = c0 * rstd, x1 = c1 * rstd;
        const float dy0 = dr[lane], dy1 = dr[lane + 32];
        dg0 = fmaf(dy0, x0, dg0); dg1 = fmaf(dy1, x1, dg1); db0 += dy0; db1 += dy1;
        const float dx0 = dy0 * g0, dx1 = dy1 * g1;
        const float m1_ = warp_sum(dx0 + dx1) * (1.0f / RH);
        const float m2_ = warp_sum(dx0 * x0 + dx1 * x1) * (1.0f / RH);
        float dz0 = z0 > 0.0f ? rstd * (dx0 - m1_ - x0 * m2_) : 0.0f;
        float dz1 = z1 > 0.0f ? rstd * (dx1 - m1_ - x1 * m2_) : 0.0f;
        s0 += dz0; s1 += dz1;
        if (stat) {
            const float mu = stat[(a * rows + r) * 2], rs = stat[(a * rows + r) * 2 + 1];
            dz0 *= rs; dz1 *= rs;
            m0 = fmaf(dz0, mu, m0); m1 = fmaf(dz1, mu, m1);
        }
        zr[lane] = dz0; zr[lane + 32] = dz1;
    }
    // block reduction of the lane-local accumulators, then one atomic per feature per block
    __shared__ float red[8][64];
    float* g = Gr.net(a, type);
    const int w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    float vals[4][2] = {{dg0, dg1}, {db0, db1}, {s0, s1}, {m0, m1}};
    for (int q = 0; q < 4; ++q) {
        if (q == 3 && !stat) break;
        red[w][lane] = vals[q][0]; red[w][lane + 32] = vals[q][1];
        __syncthreads();
        if (w == 0) {
            float t0 = 0, t1 = 0;
            for (int i = 0; i < nw; ++i) { t0 += red[i][lane]; t1 += red[i][lane + 32]; }
            if (q == 0) { atomicAdd(&g[g_off + lane], t0); atomicAdd(&g[g_off + lane + 32], t1); }
            if (q == 1) { atomicAdd(&g[b_off + lane], t0); atomicAdd(&g[b_off + lane + 32], t1); }
            if (q == 2) {
                atomicAdd(&g[lin_b_off + lane], t0); atomicAdd(&g[lin_b_off + lane + 32], t1);
                if (SM) { atomicAdd(&SM[(a * 2 + 0) * 128 + type * 64 + lane], t0); atomicAdd(&SM[(a * 2 + 0) * 128 + type * 64 + lane + 32], t1); }
            }
            if (q == 3) { atomicAdd(&SM[(a * 2 + 1) * 128 + type * 64 + lane], t0); atomicAdd(&SM[(a * 2 + 1) * 128 + type * 64 + lane + 32], t1); }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------
// gru_head: GRU gates -> H1 -> LN -> policy / value head  [+ PPO losses and backward]
// ---------------------------------------------------------------------------------------
struct HeadArgs {
    RowBuf gi, gh;                 // [192] pre-activations; overwritten with dGI / dGH in train mode
    const float* h0a; const float* h0c; int64_t h0_sa; int h0_ld;     // stored hidden inputs
    NetParams P; NetGrads G;
    int F, n_actions, T1, n_eps, n_train_eps, rows;       // rows = n_eps*T1
    const int32_t* actions;        // [A][rows]
    const uint8_t* avail;          // NULL or [A][rows][n_actions]
    // eval outputs
    float* logp_out; float* ent_out; float* value_out;    // [A][rows] (may be NULL)
    // train inputs
    const float* old_logp; const float* old_value; const float* returns; const float* adv_raw; const float* alive;
    const float* norm;             // [A][4]: adv mean, 1/(adv std + 1e-5), 1/sum(alive over train rows), 1/n_train_rows
    float clip, ent_coef, v_coef, huber_delta;
    float gscale;                  // power-of-two loss scale applied to d loss / d logits|value (undone in adam)
    float* stats;                 // [A][8]: sums of policy-loss, value-loss, entropy, ratio (already normalised)
    const int32_t* train_rows;    // NULL, or [A]: the rows are a gathered mini-batch whose first train_rows[a] rows train
    int train;
};

__device__ __forceinline__ float huber_os(float e, float d) {       // utils/mappo_utils/util.py:33-36
    const float ae = fabsf(e);
    return ae <= d ? 0.5f * e * e : (e > d ? d * (ae - 0.5f * d) : 0.0f);
}
__device__ __forceinline__ float huber_os_grad(float e, float d) {
    return fabsf(e) <= d ? e : (e > d ? d : 0.0f);
}

// 16 lanes per row, two rows per warp: lane `sub` of a half-warp owns the hidden units / features
// c = sub + 16 u (u = 0..3), so the per-row scalar work (soft-max, losses) is shared by 16 lanes instead of 32 and
// a warp carries two independent dependency chains.  Reductions over a row's 64 features = 4 local adds + 4 shuffles.
constexpr int HU = 4;                       // units per lane
constexpr int HEAD_THREADS = 128;
constexpr int HEAD_WARPS = HEAD_THREADS / 32;
// lane-local gradient accumulators flushed through shared memory at the end: per feature-lane values
//   dW[n_out][HU], dg3[HU], db3[HU], dbi[3][HU], dbh[3][HU]  and per-row scalars dB[n_out], 3 statistics

__device__ __forceinline__ float half_sum(float v) {                 // sum over the 16 lanes of a half-warp
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

// TYPE 0 = actor (NOUT >= n_actions head rows kept in registers), TYPE 1 = critic (NOUT = 1); blockIdx.y = agent
template <int TYPE, int NOUT>
__global__ void __launch_bounds__(HEAD_THREADS, 3) gru_head_kernel(HeadArgs h) {
    constexpr int HEAD_NV = NOUT * HU + 2 * HU + 6 * HU;        // vector slots of the gradient flush
    constexpr int HEAD_NS = NOUT + 3;                            // scalar slots
    __shared__ float red_v[HEAD_WARPS][HEAD_NV][32];
    __shared__ float red_s[HEAD_WARPS][2][HEAD_NS];
    const int a = blockIdx.y;
    constexpr int type = TYPE;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int sub = lane & 15, half = lane >> 4;
    const float* p = h.P.net(a, type);
    const TrunkLayout L = trunk_layout(h.F, type == 0 ? h.n_actions : 1, type == 1);
    const int nA = h.n_actions;
    const int n_out = type == 0 ? nA : 1;
    float g3[HU], b3[HU], hw[NOUT][HU], hb[NOUT];
#pragma unroll
    for (int u = 0; u < HU; ++u) { g3[u] = p[L.ln3_w + sub + 16 * u]; b3[u] = p[L.ln3_b + sub + 16 * u]; }
#pragma unroll
    for (int l = 0; l < NOUT; ++l) {
#pragma unroll
        for (int u = 0; u < HU; ++u) hw[l][u] = l < n_out ? p[L.head_w + l * RH + sub + 16 * u] : 0.0f;
        hb[l] = l < n_out ? p[L.head_b + l] : 0.0f;
    }
    float nrm_mean = 0, nrm_istd = 0, inv_msum = 0, inv_rows = 0;
    if (h.train) { nrm_mean = h.norm[a * 4]; nrm_istd = h.norm[a * 4 + 1]; inv_msum = h.norm[a * 4 + 2]; inv_rows = h.norm[a * 4 + 3]; }

    // lane-local gradient accumulators
    float dW[NOUT][HU], dB[NOUT];
#pragma unroll
    for (int l = 0; l < NOUT; ++l) {
        dB[l] = 0.0f;
#pragma unroll
        for (int u = 0; u < HU; ++u) dW[l][u] = 0.0f;
    }
    float dg3[HU], db3[HU], dbi[3][HU], dbh[3][HU];
#pragma unroll
    for (int u = 0; u < HU; ++u) {
        dg3[u] = db3[u] = 0.0f;
#pragma unroll
        for (int q = 0; q < 3; ++q) dbi[q][u] = dbh[q][u] = 0.0f;
    }
    float st_loss = 0, st_ent = 0, st_ratio = 0;

    const int64_t pair0 = ((int64_t)blockIdx.x * HEAD_WARPS + w) * 2;           // first row of this warp's first pair
    const int64_t stride = (int64_t)gridDim.x * HEAD_WARPS * 2;
    for (int64_t rp = pair0; rp < h.rows; rp += stride) {                       // warp-uniform trip count
        const int64_t r_raw = rp + half;
        const bool valid = r_raw < h.rows;                                       // half-uniform
        const int64_t r = valid ? r_raw : h.rows - 1;
        const int b = (int)(r / h.T1), t = (int)(r - (int64_t)b * h.T1);
        float* gi = h.gi.row(a, type, r);
        float* gh = h.gh.row(a, type, r);
        const float* h0 = (type == 0 ? h.h0a : h.h0c) + a * h.h0_sa + r * h.h0_ld;
        float rg[HU], zg[HU], ng[HU], ghn[HU], h1[HU], h0v[HU];
        float s1 = 0.0f;
#pragma unroll
        for (int u = 0; u < HU; ++u) {
            const int c = sub + 16 * u;
            rg[u] = sigmoidf_acc(gi[c] + gh[c]);
            zg[u] = sigmoidf_acc(gi[RH + c] + gh[RH + c]);
            ghn[u] = gh[2 * RH + c];
            ng[u] = tanhf_acc(gi[2 * RH + c] + rg[u] * ghn[u]);
            h0v[u] = h0[c];
            h1[u] = (1.0f - zg[u]) * ng[u] + zg[u] * h0v[u];
            s1 += h1[u];
        }
        const float mean = half_sum(s1) * (1.0f / RH);
        float cen[HU], s2 = 0.0f;
#pragma unroll
        for (int u = 0; u < HU; ++u) { cen[u] = h1[u] - mean; s2 = fmaf(cen[u], cen[u], s2); }
        const float rstd = 1.0f / sqrtf(half_sum(s2) * (1.0f / RH) + LEPS);
        float xh[HU], av[HU];
#pragma unroll
        for (int u = 0; u < HU; ++u) { xh[u] = cen[u] * rstd; av[u] = xh[u] * g3[u] + b3[u]; }
        float outv[NOUT];
#pragma unroll
        for (int l = 0; l < NOUT; ++l) {
            if (l < n_out) {                                                     // block-uniform
                float d = 0.0f;
#pragma unroll
                for (int u = 0; u < HU; ++u) d = fmaf(hw[l][u], av[u], d);
                outv[l] = half_sum(d) + hb[l];
            } else {
                outv[l] = -INFINITY;
            }
        }

        const int64_t ridx = (int64_t)a * h.rows + r;
        const bool train_row = valid && h.train && (h.train_rows ? r < h.train_rows[a] : t < h.T1 - 1 && b < h.n_train_eps);
        float dA[HU];                         // gradient wrt the LN3 output
#pragma unroll
        for (int u = 0; u < HU; ++u) dA[u] = 0.0f;
        if (type == 0) {
            const int act = h.actions[ridx];
            bool masked[NOUT];
            float mx = -INFINITY;
#pragma unroll
            for (int l = 0; l < NOUT; ++l) {
                masked[l] = l < nA && h.avail && h.avail[ridx * nA + l] == 0;
                if (masked[l]) outv[l] = -1e10f;
                if (l < nA) mx = fmaxf(mx, outv[l]);
            }
            float den = 0.0f;
#pragma unroll
            for (int l = 0; l < NOUT; ++l) if (l < nA) den += expf(outv[l] - mx);
            const float lse = mx + logf(den);
            float ent = 0.0f, lp_a = 0.0f, pl[NOUT], lpl[NOUT];
#pragma unroll
            for (int l = 0; l < NOUT; ++l) {
                lpl[l] = l < nA ? outv[l] - lse : 0.0f;
                pl[l] = l < nA ? expf(lpl[l]) : 0.0f;
                ent -= pl[l] * lpl[l];
                if (l == act) lp_a = lpl[l];
            }
            if (!h.train) {                                                      // block-uniform
                if (sub == 0 && valid) {
                    if (h.logp_out) h.logp_out[ridx] = lp_a;
                    if (h.ent_out) h.ent_out[ridx] = ent;
                }
                continue;
            }
            float dl[NOUT];
#pragma unroll
            for (int l = 0; l < NOUT; ++l) dl[l] = 0.0f;
            if (train_row) {
                const float m = h.alive[ridx];
                const float adv = (h.adv_raw[ridx] - nrm_mean) * nrm_istd;
                const float ratio = expf(lp_a - h.old_logp[ridx]);
                const float s1_ = ratio * adv;
                const float s2_ = fminf(fmaxf(ratio, 1.0f - h.clip), 1.0f + h.clip) * adv;
                const bool inside = ratio >= 1.0f - h.clip && ratio <= 1.0f + h.clip;
                float d = 0.0f;                                   // d min(s1,s2) / d logp
                if (s1_ < s2_) d = s1_;
                else if (s1_ == s2_) d = inside ? s1_ : 0.5f * s1_;
                const float g_lp = -m * inv_msum * d * h.gscale;
                const float g_ent = -h.ent_coef * inv_rows * h.gscale;       // d(-c*mean ent)/d ent_row
#pragma unroll
                for (int l = 0; l < NOUT; ++l) {
                    if (l < nA && !masked[l]) {
                        const float dlp = g_lp * ((l == act ? 1.0f : 0.0f) - pl[l]);
                        const float dent = g_ent * (-pl[l] * (lpl[l] + ent));
                        dl[l] = dlp + dent;
                    }
                }
                if (sub == 0) {                                  // per-row scalars: one lane of the half-warp carries them
                    st_loss += -fminf(s1_, s2_) * m * inv_msum;
                    st_ent += ent * inv_rows;
                    st_ratio += ratio * inv_rows;
                }
            }
#pragma unroll
            for (int l = 0; l < NOUT; ++l) {
#pragma unroll
                for (int u = 0; u < HU; ++u) {
                    dA[u] = fmaf(dl[l], hw[l][u], dA[u]);
                    dW[l][u] = fmaf(dl[l], av[u], dW[l][u]);
                }
                if (sub == 0) dB[l] += dl[l];
            }
        } else {
            const float v = outv[0];
            if (!h.train) {
                if (sub == 0 && valid && h.value_out) h.value_out[ridx] = v;
                continue;
            }
            float dv = 0.0f;
            if (train_row) {
                const float m = h.alive[ridx];
                const float vo = h.old_value[ridx], ret = h.returns[ridx];
                const float diff = v - vo;
                const float vc = vo + fminf(fmaxf(diff, -h.clip), h.clip);
                const float eo = ret - v, ec = ret - vc;
                const float lo = huber_os(eo, h.huber_delta), lc = huber_os(ec, h.huber_delta);
                const bool inside = diff >= -h.clip && diff <= h.clip;
                // d max(lo, lc) / d v.  d lo/dv = -h'(eo);  d lc/dv = -h'(ec) where the clamp passes
                // (inside the range), else 0.  Inside the range vc = vo + (v - vo) can differ from v
                // by an ulp, so which of lo / lc is larger is rounding noise there: both branches
                // must carry the same gradient (torch.max splits it evenly on an exact tie).
                const float go = -huber_os_grad(eo, h.huber_delta);
                const float gc = inside ? -huber_os_grad(ec, h.huber_delta) : 0.0f;
                const float g = lo > lc ? go : (lc > lo ? gc : 0.5f * (go + gc));
                dv = h.v_coef * m * inv_msum * g * h.gscale;
                if (sub == 0) st_loss += fmaxf(lo, lc) * m * inv_msum;
            }
#pragma unroll
            for (int u = 0; u < HU; ++u) { dA[u] = dv * hw[0][u]; dW[0][u] = fmaf(dv, av[u], dW[0][u]); }
            if (sub == 0) dB[0] += dv;
        }
        // ---- backward: LN3, GRU gates (rows past the end carry dA = 0 and store nothing) --------
        float dx[HU], t1 = 0.0f, t2 = 0.0f;
#pragma unroll
        for (int u = 0; u < HU; ++u) {
            dg3[u] = fmaf(dA[u], xh[u], dg3[u]); db3[u] += dA[u];
            dx[u] = dA[u] * g3[u];
            t1 += dx[u]; t2 = fmaf(dx[u], xh[u], t2);
        }
        const float m1_ = half_sum(t1) * (1.0f / RH);
        const float m2_ = half_sum(t2) * (1.0f / RH);
#pragma unroll
        for (int u = 0; u < HU; ++u) {
            const int c = sub + 16 * u;
            const float dh = rstd * (dx[u] - m1_ - xh[u] * m2_);
            const float dn = dh * (1.0f - zg[u]);
            const float dz = dh * (h0v[u] - ng[u]);
            const float dan = dn * (1.0f - ng[u] * ng[u]);
            const float dr = dan * ghn[u];
            const float daz = dz * zg[u] * (1.0f - zg[u]);
            const float dar = dr * rg[u] * (1.0f - rg[u]);
            if (valid) {
                gi[c] = dar; gi[RH + c] = daz; gi[2 * RH + c] = dan;
                gh[c] = dar; gh[RH + c] = daz; gh[2 * RH + c] = dan * rg[u];
            }
            dbi[0][u] += dar; dbi[1][u] += daz; dbi[2][u] += dan;
            dbh[0][u] += dar; dbh[1][u] += daz; dbh[2][u] += dan * rg[u];
        }
    }
    if (!h.train) return;

    // ---- one-barrier block reduction of the lane-local accumulators -> global gradient buffers ---------
    {
        int k = 0;
#pragma unroll
        for (int l = 0; l < NOUT; ++l)
#pragma unroll
            for (int u = 0; u < HU; ++u) red_v[w][k++][lane] = dW[l][u];
#pragma unroll
        for (int u = 0; u < HU; ++u) red_v[w][k++][lane] = dg3[u];
#pragma unroll
        for (int u = 0; u < HU; ++u) red_v[w][k++][lane] = db3[u];
#pragma unroll
        for (int q = 0; q < 3; ++q)
#pragma unroll
            for (int u = 0; u < HU; ++u) red_v[w][k++][lane] = dbi[q][u];
#pragma unroll
        for (int q = 0; q < 3; ++q)
#pragma unroll
            for (int u = 0; u < HU; ++u) red_v[w][k++][lane] = dbh[q][u];
        if (sub == 0) {
#pragma unroll
            for (int l = 0; l < NOUT; ++l) red_s[w][half][l] = dB[l];
            red_s[w][half][NOUT] = st_loss; red_s[w][half][NOUT + 1] = st_ent; red_s[w][half][NOUT + 2] = st_ratio;
        }
    }
    __syncthreads();
    float* g = h.G.net(a, type);
    for (int idx = threadIdx.x; idx < HEAD_NV * 16; idx += HEAD_THREADS) {
        const int k = idx >> 4, s16 = idx & 15;
        float t = 0.0f;
#pragma unroll
        for (int i = 0; i < HEAD_WARPS; ++i) t += red_v[i][k][s16] + red_v[i][k][s16 + 16];
        const int u = k % HU, grp = k / HU;                 // grp: 0..7 head rows | 8 dg3 | 9 db3 | 10..12 dbi | 13..15 dbh
        const int c = s16 + 16 * u;
        if (grp < NOUT) { if (grp < n_out) atomicAdd(&g[L.head_w + grp * RH + c], t); }
        else if (grp == NOUT) atomicAdd(&g[L.ln3_w + c], t);
        else if (grp == NOUT + 1) atomicAdd(&g[L.ln3_b + c], t);
        else if (grp < NOUT + 5) atomicAdd(&g[L.bih + (grp - NOUT - 2) * RH + c], t);
        else atomicAdd(&g[L.bhh + (grp - NOUT - 5) * RH + c], t);
    }
    if (threadIdx.x < HEAD_NS) {
        const int q = threadIdx.x;
        float t = 0.0f;
#pragma unroll
        for (int i = 0; i < HEAD_WARPS; ++i) t += red_s[i][0][q] + red_s[i][1][q];
        if (q < NOUT) { if (q < n_out) atomicAdd(&g[L.head_b + q], t); }
        else if (q == NOUT) atomicAdd(&h.stats[a * 8 + (type == 0 ? 0 : 1)], t);   // policy | value loss
        else if (q == NOUT + 1 && type == 0) atomicAdd(&h.stats[a * 8 + 2], t);      // entropy
        else if (q == NOUT + 2 && type == 0) atomicAdd(&h.stats[a * 8 + 3], t);      // ratio
    }
}

// the whole train-mode tail as one kernel
#include "tail_fused.cuh"

// ---------------------------------------------------------------------------------------
// K2a gae_adv: GAE backward scan + raw advantages + their moments (one CTA per agent)
// ---------------------------------------------------------------------------------------
__global__ void gae_adv_kernel(const float* __restrict__ V /* [A][rows] */, const float* __restrict__ reward,
                               const float* __restrict__ alive, float gamma, float lam, int T1, int n_eps, int n_train_eps,
                               float* __restrict__ returns, float* __restrict__ adv_raw,
                               double* __restrict__ moments /* [A][4]: sum adv, sum adv^2, n, sum alive(train rows) */) {
    const int a = blockIdx.x;
    const int T = T1 - 1;
    const int64_t base = (int64_t)a * n_eps * T1;
    double s1 = 0.0, s2 = 0.0, sm = 0.0;
    for (int b = threadIdx.x; b < n_eps; b += blockDim.x) {
        const int64_t o = base + (int64_t)b * T1;
        float gae = 0.0f;
        for (int t = T - 1; t >= 0; --t) {
            const float vt = V[o + t], vn = V[o + t + 1], mn = alive[o + t + 1];
            const float delta = reward[o + t] + gamma * vn * mn - vt;        // :354-356
            gae = delta + gamma * lam * mn * gae;                            // :357
            const float ret = gae + vt;                                      // :358
            returns[o + t] = ret;
            float adv = ret - vt;                                            // :273
            if (alive[o + t] == 0.0f) adv = 0.0f;                            // :277
            adv_raw[o + t] = adv;
            s1 += adv; s2 += (double)adv * adv;
            if (b < n_train_eps) sm += alive[o + t];
        }
        returns[o + T] = 0.0f; adv_raw[o + T] = 0.0f;
    }
    __shared__ double red[3][32];
    auto wsum = [](double v) { for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); return v; };
    s1 = wsum(s1); s2 = wsum(s2); sm = wsum(sm);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane == 0) { red[0][w] = s1; red[1][w] = s2; red[2][w] = sm; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t1 = 0, t2 = 0, t3 = 0;
        for (int i = 0; i < nw; ++i) { t1 += red[0][i]; t2 += red[1][i]; t3 += red[2][i]; }
        moments[a * 4 + 0] = t1; moments[a * 4 + 1] = t2; moments[a * 4 + 2] = (double)n_eps * T; moments[a * 4 + 3] = t3;
    }
}

// finalise (after an optional cross-rank all-reduce of `moments`): unbiased std over all
// Bf*T entries incl. the zeros (:278), and the loss denominators
__global__ void adv_finalize_kernel(const double* __restrict__ moments, double n_train_rows_global, float* __restrict__ norm, int A) {
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A) return;
    const double s1 = moments[a * 4], s2 = moments[a * 4 + 1], n = moments[a * 4 + 2], sm = moments[a * 4 + 3];
    const double mean = s1 / n;
    double var = (s2 - n * mean * mean) / (n - 1.0);
    if (var < 0) var = 0;
    norm[a * 4 + 0] = (float)mean;
    norm[a * 4 + 1] = 1.0f / ((float)sqrt(var) + 1e-5f);
    norm[a * 4 + 2] = (float)(1.0 / sm);
    norm[a * 4 + 3] = (float)(1.0 / n_train_rows_global);
}

// ---------------------------------------------------------------------------------------
// grad_norm + Adam
// ---------------------------------------------------------------------------------------
__global__ void grad_sqnorm_kernel(const float* __restrict__ g, int64_t stride, int64_t total, float inv_gscale,
                                   float* __restrict__ out /* [A] */) {
    const int a = blockIdx.y;
    float s = 0.0f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = g[a * stride + i] * inv_gscale;
        s = fmaf(v, v, s);
    }
    __shared__ float red[32];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0f;
        s = warp_sum(s);
        if (threadIdx.x == 0) atomicAdd(&out[a], s);
    }
}

// torch.optim.Adam step with clip_grad_norm_ folded in:  g *= min(1, max_norm/(norm+1e-6))
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            const float* __restrict__ mask, const float* __restrict__ sqnorm, int64_t stride, int64_t total,
                            float lr, float b1, float b2, float eps, float bc1, float bc2_sqrt, float max_norm,
                            float inv_gscale, float* __restrict__ stats, int stat_col) {
    const int a = blockIdx.y;
    const float norm = sqrtf(sqnorm[a]);
    const float coef = max_norm > 0.0f ? fminf(max_norm / (norm + 1e-6f), 1.0f) : 1.0f;
    if (stats && blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&stats[a * 8 + stat_col], norm);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        if (mask[i] == 0.0f) continue;
        const int64_t j = a * stride + i;
        const float gr = g[j] * inv_gscale * coef;     // undo the power-of-two loss scale (exact)
        const float mm = b1 * m[j] + (1.0f - b1) * gr;
        const float vv = b2 * v[j] + (1.0f - b2) * gr * gr;
        m[j] = mm; v[j] = vv;
        const float denom = sqrtf(vv) / bc2_sqrt + eps;
        p[j] = p[j] - (lr / bc1) * (mm / denom);
    }
}

// ---------------------------------------------------------------------------------------
// gather_rows: one shuffled mini-batch as dense rows, so that the TMA / wgmma fc1 kernels (which load tiles, not row
// lists) and the tail run on it as they run on the packed store.  One warp per destination row: the two f16 operand rows
// as 16-byte vectors, the two stored hidden rows, and the row's scalars.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) gather_rows_kernel(iplan_gather_args g) {
    const int a = blockIdx.y, lane = threadIdx.x & 31;
    const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    const int vec = g.ldx / 8;                                               // uint4 = 8 halves
    for (int64_t j = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); j < g.rows_dst; j += warps) {
        const int64_t d = (int64_t)a * g.rows_dst + j;
        const int32_t i = g.idx[d];
        const int64_t s = (int64_t)a * g.rows_src + (i < 0 ? 0 : i);
        const uint4* xh = reinterpret_cast<const uint4*>(static_cast<const __half*>(g.Xh) + s * g.ldx);
        const uint4* xl = reinterpret_cast<const uint4*>(static_cast<const __half*>(g.Xl) + s * g.ldx);
        uint4* oh = reinterpret_cast<uint4*>(static_cast<__half*>(g.Xh_out) + d * g.ldx);
        uint4* ol = reinterpret_cast<uint4*>(static_cast<__half*>(g.Xl_out) + d * g.ldx);
        for (int v = lane; v < vec; v += 32) { oh[v] = __ldg(xh + v); ol[v] = __ldg(xl + v); }
        if (lane < RH / 4) {
            reinterpret_cast<float4*>(g.rnn_a_out + d * RH)[lane] = __ldg(reinterpret_cast<const float4*>(g.rnn_a + s * RH) + lane);
        } else {
            reinterpret_cast<float4*>(g.rnn_c_out + d * RH)[lane - RH / 4] = __ldg(reinterpret_cast<const float4*>(g.rnn_c + s * RH) + lane - RH / 4);
        }
        if (lane < 5) g.scalars_out[lane][d] = g.scalars[lane][s];
        else if (lane < 7) g.stat_out[d * 2 + lane - 5] = g.stat[s * 2 + lane - 5];
        else if (lane == 7) g.actions_out[d] = g.actions[s];
        else if (lane - 8 < g.n_actions) g.avail_out[d * g.n_actions + lane - 8] = g.avail[s * g.n_actions + lane - 8];
    }
}

}  // namespace iplan

// =======================================================================================
// C ABI
// =======================================================================================
using namespace iplan;

extern "C" int iplan_learner_row_stats(const float* X, int64_t x_stride_agent, int ldx, int feat_dim, int64_t rows,
                                       int n_agents, float* stat, void* stream) {
    IPLAN_REQUIRE(X && stat && rows > 0 && n_agents > 0 && feat_dim > 0 && ldx >= feat_dim, "row_stats: bad arguments");
    dim3 grid((unsigned)std::min<int64_t>((rows + 7) / 8, sm_count() * 16), n_agents);
    row_stats_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(X, x_stride_agent, ldx, feat_dim, rows, stat);
    count_launch();
    return check_launch("row_stats");
}

// everything between Z1 and the heads; train != 0 also runs the loss + backward down to dZ1
// (scaled by rstd) and all gradients except fc1.W / LN0, which iplan_learner_fc1_backward adds.

extern "C" int iplan_learner_tail(const iplan_learner_ctx* c, int train, void* stream_) {
    IPLAN_REQUIRE(c && c->Z1 && c->A1 && c->Z2 && c->A2 && c->GI && c->GH, "learner_tail: null work buffer");
    IPLAN_REQUIRE(c->n_actions > 0 && c->n_actions <= IPLAN_MAX_ACT, "learner_tail: n_actions %d not in [1,%d]", c->n_actions, IPLAN_MAX_ACT);
    IPLAN_REQUIRE(c->n_agents > 0 && c->n_eps > 0 && c->T1 > 0 && c->feat_dim > 0, "learner_tail: bad sizes");
    cudaStream_t st = (cudaStream_t)stream_;
    const int A = c->n_agents;
    const int64_t rows = (int64_t)c->n_eps * c->T1;
    NetParams P{c->actor, c->critic, c->actor_stride, c->critic_stride};
    NetGrads G{c->g_actor, c->g_critic, c->actor_stride, c->critic_stride};
    const TrunkLayout L = trunk_layout(c->feat_dim, 1, false);
    RowBuf z1{c->Z1, rows * 128, 64, 128};
    RowBuf a1{c->A1, 2 * rows * RH, rows * RH, RH}, z2{c->Z2, 2 * rows * RH, rows * RH, RH}, a2{c->A2, 2 * rows * RH, rows * RH, RH};
    RowBuf gi{c->GI, 2 * rows * RH3, rows * RH3, RH3}, gh{c->GH, 2 * rows * RH3, rows * RH3, RH3};
    // the stored hidden inputs: type 0 reads rnn_a, type 1 reads rnn_c -> two launches for GH
    const unsigned rw = (unsigned)std::min<int64_t>((rows + 7) / 8, sm_count() * 8);
    const unsigned mt = (unsigned)((rows + 63) / 64), mt128 = (unsigned)((rows + 127) / 128);
    static bool lin_configured = false;
    if (!lin_configured) {
        cudaFuncSetAttribute(lin64_rows_kernel<64, 64, 128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Lin64Rows<64, 64, 128, false>::SMEM);
        cudaFuncSetAttribute(lin64_rows_kernel<64, 192, 128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Lin64Rows<64, 192, 128, false>::SMEM);
        cudaFuncSetAttribute(lin64_rows_kernel<192, 64, 64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Lin64Rows<192, 64, 64, true>::SMEM);
        cudaFuncSetAttribute(lin64_rows_kernel<64, 64, 128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Lin64Rows<64, 64, 128, true>::SMEM);
        cudaFuncSetAttribute(lin64_dw_kernel<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Lin64Dw<192>::SMEM);
        cudaFuncSetAttribute(lin64_dw_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Lin64Dw<64>::SMEM);
        lin_configured = true;
    }
    int launches = 0;
    HeadArgs h;
    h.gi = gi; h.gh = gh; h.h0a = c->rnn_a; h.h0c = c->rnn_c; h.h0_sa = c->rnn_stride_agent; h.h0_ld = c->rnn_ld;
    h.P = P; h.G = G; h.F = c->feat_dim; h.n_actions = c->n_actions; h.T1 = c->T1; h.n_eps = c->n_eps;
    h.n_train_eps = c->n_train_eps; h.rows = (int)rows; h.actions = c->actions; h.avail = c->avail;
    h.logp_out = c->logp_out; h.ent_out = c->ent_out; h.value_out = c->value_out;
    h.old_logp = c->old_logp; h.old_value = c->old_value; h.returns = c->returns; h.adv_raw = c->adv_raw; h.alive = c->alive;
    h.norm = c->norm; h.clip = c->clip; h.ent_coef = c->ent_coef; h.v_coef = c->v_coef; h.huber_delta = c->huber_delta;
    h.gscale = c->grad_scale > 0.0f ? c->grad_scale : 1.0f;
    h.stats = c->stats; h.train_rows = c->train_rows; h.train = train;
    if (train) IPLAN_REQUIRE(c->g_actor && c->g_critic && c->old_logp && c->old_value && c->returns && c->adv_raw && c->alive && c->norm && c->stats && c->SM && c->stat,
                             "learner_tail: train mode needs gradient/loss buffers");
    static int tail_impl = -1;          // 0 = fused kernel (default), 1 = the twelve separate kernels (cross-check); IPLAN_TAIL_IMPL
    if (tail_impl < 0) { const char* e = getenv("IPLAN_TAIL_IMPL"); tail_impl = (e && e[0] == '1') ? 1 : 0; }
    if (train && tail_impl == 0 && c->n_actions <= TF_NOUT) {
        static bool tf_configured = false;
        if (!tf_configured) {
            cudaError_t e = cudaFuncSetAttribute(tail_fused_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TF_SMEM);
            if (e == cudaSuccess) e = cudaFuncSetAttribute(tail_fused_kernel<TF_NOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TF_SMEM);
            if (e != cudaSuccess) { set_error("learner_tail: fused kernel smem attr %zu: %s", TF_SMEM, cudaGetErrorString(e)); return (int)e; }
            tf_configured = true;
        }
        TfArgs fa;
        fa.h = h; fa.z1 = z1; fa.a1 = a1; fa.z2 = z2; fa.a2 = a2; fa.stat = c->stat; fa.SM = c->SM; fa.rows = rows;
        const int64_t n_tiles16 = (rows + 15) / 16;
        // one CTA per SM: ctas x (2A nets) CTAs, actor and critic tiles side by side
        const int ctas = (int)std::min<int64_t>((n_tiles16 + TF_WARPS - 1) / TF_WARPS, std::max(1, sm_count() / (2 * A)));
        const DetScratch ds = det_scratch((size_t)2 * A * ctas * TF_WARPS * TF_REC, (size_t)2 * A);
        if (!ds.part) return -1;                                      // det_scratch set the error text
        fa.part = ds.part; fa.count = ds.count;
        if (c->n_actions <= 5) tail_fused_kernel<5><<<dim3((unsigned)ctas, 2 * A), TF_THREADS, TF_SMEM, st>>>(fa);
        else tail_fused_kernel<TF_NOUT><<<dim3((unsigned)ctas, 2 * A), TF_THREADS, TF_SMEM, st>>>(fa);
        launches = 1;
        const int64_t n_tiles64 = (rows + 63) / 64;
        const unsigned dw_ctas = (unsigned)std::min<int64_t>(n_tiles64, 32);
        const int dw_tiles = (int)((n_tiles64 + dw_ctas - 1) / dw_ctas);
        // weight gradients (K = rows) + the bias gradients = column sums of the same dY arrays
        if (int rc = launch_lin64_dw<192>(dim3(dw_ctas, 2 * A), st, gi, a2, G, L.wih, rows, dw_tiles, 2, L.bih)) return rc; ++launches;
        {
            RowBuf h0a{const_cast<float*>(c->rnn_a), c->rnn_stride_agent, 0, c->rnn_ld};
            RowBuf h0c{const_cast<float*>(c->rnn_c), c->rnn_stride_agent, 0, c->rnn_ld};
            RowBuf gha{c->GH, 2 * rows * RH3, 0, RH3}, ghc{c->GH + rows * RH3, 2 * rows * RH3, 0, RH3};
            NetGrads Ga{c->g_actor, c->g_actor, c->actor_stride, c->actor_stride};
            NetGrads Gc{c->g_critic, c->g_critic, c->critic_stride, c->critic_stride};
            if (int rc = launch_lin64_dw<192>(dim3(dw_ctas, A), st, gha, h0a, Ga, L.whh, rows, dw_tiles, 1, L.bhh)) return rc; ++launches;
            if (int rc = launch_lin64_dw<192>(dim3(dw_ctas, A), st, ghc, h0c, Gc, L.whh, rows, dw_tiles, 1, L.bhh)) return rc; ++launches;
        }
        if (int rc = launch_lin64_dw<64>(dim3(dw_ctas, 2 * A), st, z2, a1, G, L.fc2_w, rows, dw_tiles, 2, L.fc2_b)) return rc; ++launches;
        tail_beta_kernel<<<2 * A, RH, 0, st>>>(P, G, c->feat_dim, c->n_actions); ++launches;
        count_launch(launches);
        return check_launch("learner_tail(fused)");
    }
    ln_relu_fwd_kernel<<<dim3(rw, 2 * A), 256, 0, st>>>(z1, a1, P, L.ln1_w, L.ln1_b, rows, 2); ++launches;
    lin64_rows_kernel<64, 64, 128, false><<<dim3(mt128, 2 * A), 256, Lin64Rows<64, 64, 128, false>::SMEM, st>>>(a1, z2, P, L.fc2_w, L.fc2_b, rows, 2); ++launches;
    ln_relu_fwd_kernel<<<dim3(rw, 2 * A), 256, 0, st>>>(z2, a2, P, L.ln2_w, L.ln2_b, rows, 2); ++launches;
    lin64_rows_kernel<64, 192, 128, false><<<dim3(mt128, 2 * A), 256, Lin64Rows<64, 192, 128, false>::SMEM, st>>>(a2, gi, P, L.wih, L.bih, rows, 2); ++launches;
    {   // GH = H0 W_hh^T + b_hh ; actor and critic hidden inputs live in different arrays
        RowBuf h0a{const_cast<float*>(c->rnn_a), c->rnn_stride_agent, 0, c->rnn_ld};
        RowBuf h0c{const_cast<float*>(c->rnn_c), c->rnn_stride_agent, 0, c->rnn_ld};
        NetParams Pa{c->actor, c->actor, c->actor_stride, c->actor_stride};
        NetParams Pc{c->critic, c->critic, c->critic_stride, c->critic_stride};
        RowBuf gha{c->GH, 2 * rows * RH3, 0, RH3}, ghc{c->GH + rows * RH3, 2 * rows * RH3, 0, RH3};
        lin64_rows_kernel<64, 192, 128, false><<<dim3(mt128, A), 256, Lin64Rows<64, 192, 128, false>::SMEM, st>>>(h0a, gha, Pa, L.whh, L.bhh, rows, 1); ++launches;
        lin64_rows_kernel<64, 192, 128, false><<<dim3(mt128, A), 256, Lin64Rows<64, 192, 128, false>::SMEM, st>>>(h0c, ghc, Pc, L.whh, L.bhh, rows, 1); ++launches;
    }
    {
        const dim3 hgrid((unsigned)std::min<int64_t>((rows + 7) / 8, sm_count() * 6), A);
        if (c->n_actions <= 5) gru_head_kernel<0, 5><<<hgrid, HEAD_THREADS, 0, st>>>(h);
        else gru_head_kernel<0, IPLAN_MAX_ACT><<<hgrid, HEAD_THREADS, 0, st>>>(h);
        gru_head_kernel<1, 1><<<hgrid, HEAD_THREADS, 0, st>>>(h);
        launches += 2;
    }
    if (train) {
        const int64_t n_tiles64 = (rows + 63) / 64;
        const unsigned dw_ctas = (unsigned)std::min<int64_t>(n_tiles64, 32);
        const int dw_tiles = (int)((n_tiles64 + dw_ctas - 1) / dw_ctas);
        // GRU projections: dW_ih = dGI^T A2, dW_hh = dGH^T H0, dA2 = dGI W_ih (into the A2 buffer)
        if (int rc = launch_lin64_dw<192>(dim3(dw_ctas, 2 * A), st, gi, a2, G, L.wih, rows, dw_tiles, 2)) return rc; ++launches;
        {
            RowBuf h0a{const_cast<float*>(c->rnn_a), c->rnn_stride_agent, 0, c->rnn_ld};
            RowBuf h0c{const_cast<float*>(c->rnn_c), c->rnn_stride_agent, 0, c->rnn_ld};
            RowBuf gha{c->GH, 2 * rows * RH3, 0, RH3}, ghc{c->GH + rows * RH3, 2 * rows * RH3, 0, RH3};
            NetGrads Ga{c->g_actor, c->g_actor, c->actor_stride, c->actor_stride};
            NetGrads Gc{c->g_critic, c->g_critic, c->critic_stride, c->critic_stride};
            if (int rc = launch_lin64_dw<192>(dim3(dw_ctas, A), st, gha, h0a, Ga, L.whh, rows, dw_tiles, 1)) return rc; ++launches;
            if (int rc = launch_lin64_dw<192>(dim3(dw_ctas, A), st, ghc, h0c, Gc, L.whh, rows, dw_tiles, 1)) return rc; ++launches;
        }
        lin64_rows_kernel<192, 64, 64, true><<<dim3(mt, 2 * A), 128, Lin64Rows<192, 64, 64, true>::SMEM, st>>>(gi, a2, P, L.wih, -1, rows, 2); ++launches;
        ln_relu_bwd_kernel<<<dim3(rw, 2 * A), 256, 0, st>>>(z2, a2, P, G, L.ln2_w, L.ln2_b, L.fc2_b, rows, 2, nullptr, nullptr); ++launches;
        if (int rc = launch_lin64_dw<64>(dim3(dw_ctas, 2 * A), st, z2, a1, G, L.fc2_w, rows, dw_tiles, 2)) return rc; ++launches;
        lin64_rows_kernel<64, 64, 128, true><<<dim3(mt128, 2 * A), 256, Lin64Rows<64, 64, 128, true>::SMEM, st>>>(z2, a1, P, L.fc2_w, -1, rows, 2); ++launches;
        ln_relu_bwd_kernel<<<dim3(rw, 2 * A), 256, 0, st>>>(z1, a1, P, G, L.ln1_w, L.ln1_b, L.fc1_b, rows, 2, c->stat, c->SM); ++launches;
    }
    count_launch(launches);
    return check_launch("learner_tail");
}

extern "C" int iplan_learner_gather_rows(const iplan_gather_args* g, void* stream) {
    IPLAN_REQUIRE(g && g->idx && g->Xh && g->Xl && g->Xh_out && g->Xl_out && g->stat && g->stat_out && g->rnn_a && g->rnn_c &&
                  g->rnn_a_out && g->rnn_c_out && g->actions && g->actions_out && g->avail && g->avail_out, "gather_rows: null array");
    for (int i = 0; i < 5; ++i) IPLAN_REQUIRE(g->scalars[i] && g->scalars_out[i], "gather_rows: null scalar array %d", i);
    IPLAN_REQUIRE(g->rows_src > 0 && g->rows_dst > 0 && g->n_agents > 0 && g->ldx > 0 && g->ldx % 8 == 0 &&
                  g->n_actions > 0 && g->n_actions <= IPLAN_MAX_ACT, "gather_rows: bad sizes");
    IPLAN_REQUIRE((((uintptr_t)g->Xh | (uintptr_t)g->Xl | (uintptr_t)g->Xh_out | (uintptr_t)g->Xl_out | (uintptr_t)g->rnn_a |
                    (uintptr_t)g->rnn_c | (uintptr_t)g->rnn_a_out | (uintptr_t)g->rnn_c_out) & 15) == 0, "gather_rows: rows need 16-byte alignment");
    dim3 grid((unsigned)std::min<int64_t>((g->rows_dst + 7) / 8, sm_count() * 8), g->n_agents);
    gather_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*g);
    count_launch();
    return check_launch("gather_rows");
}

namespace iplan {
// fc1.weight / feature_norm gradients from the product G (fc1_mma.cu) and the column sums S | M
int launch_fc1_grad_finish(const float* actor, int64_t actor_stride, const float* critic, int64_t critic_stride,
                           float* g_actor, float* g_critic, int feat_dim, const float* G, int ldg, const float* SM,
                           int n_agents, cudaStream_t st) {
    NetParams P{actor, critic, actor_stride, critic_stride};
    NetGrads Gr{g_actor, g_critic, actor_stride, critic_stride};
    fc1_grad_finish_kernel<<<dim3((feat_dim + 127) / 128, n_agents, 2), 128, 0, st>>>(P, Gr, feat_dim, G, ldg, SM);
    count_launch();
    return check_launch("fc1_grad_finish");
}
}  // namespace iplan

extern "C" int iplan_learner_gae(const float* values, const float* reward, const float* alive, float gamma, float lam,
                                 int T1, int n_eps, int n_train_eps, int n_agents,
                                 float* returns, float* adv_raw, double* moments, void* stream) {
    IPLAN_REQUIRE(values && reward && alive && returns && adv_raw && moments && T1 >= 2 && n_eps > 0, "gae: bad arguments");
    gae_adv_kernel<<<n_agents, 512, 0, (cudaStream_t)stream>>>(values, reward, alive, gamma, lam, T1, n_eps, n_train_eps, returns, adv_raw, moments);
    count_launch();
    return check_launch("gae");
}

extern "C" int iplan_learner_adv_finalize(const double* moments, double n_train_rows_global, float* norm, int n_agents, void* stream) {
    IPLAN_REQUIRE(moments && norm && n_train_rows_global > 0, "adv_finalize: bad arguments");
    adv_finalize_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(moments, n_train_rows_global, norm, n_agents);
    count_launch();
    return check_launch("adv_finalize");
}

extern "C" int iplan_learner_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const float* mask,
                                  float* sqnorm_scratch, int64_t stride, int64_t total, int n_agents,
                                  float lr, float beta1, float beta2, float eps, int step, float max_norm,
                                  float grad_scale, float* stats, int stat_col, void* stream) {
    IPLAN_REQUIRE(params && grads && exp_avg && exp_avg_sq && mask && sqnorm_scratch && step >= 1 && grad_scale > 0.f, "adam: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(sqnorm_scratch, 0, sizeof(float) * n_agents, st);
    if (e != cudaSuccess) { set_error("adam: memset: %s", cudaGetErrorString(e)); return (int)e; }
    const float inv = 1.0f / grad_scale;
    grad_sqnorm_kernel<<<dim3(1, n_agents), 1024, 0, st>>>(grads, stride, total, inv, sqnorm_scratch);   // one block per agent: a fixed summation order
    const double bc1 = 1.0 - pow((double)beta1, step), bc2 = 1.0 - pow((double)beta2, step);
    adam_kernel<<<dim3(128, n_agents), 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, mask, sqnorm_scratch, stride, total,
                                                     lr, beta1, beta2, eps, (float)bc1, (float)sqrt(bc2), max_norm, inv, stats, stat_col);
    count_launch(2);
    return check_launch("adam");
}
