// Prediction_policy.learn — forward, loss and backward of the instant-incentive (GAT) trajectory predictor for one
// minibatch of sampled transitions (reference nova/prediction_policy.py:168-253; SURVEY §8f rank 2).
//
// Per agent-net a and sampled transition p (P = pred_batch_size = 64 per agent, so this is a small job: one CTA per
// (p, a), plain fp32 FFMA — it is ~1 % of a training iteration and its arithmetic is specified line by line by
// oracle/iplan_oracle.py::gat_backward_manual / prediction_decoder):
//   hidden = GAT_Net(x0 | lat0, att0)                       (nova/GAT_Net.py:41-142; gumbel noise explicit or Philox)
//   pred   = Prediction_Decoder(x0, hidden), pl steps fed back on itself, teacher_forcing_ratio = 0
//            (nova/prediction_net.py:37-63: ReLU(linear) -> 1-step GRU -> tanh -> dropout -> out)
//   loss_a = sum |target - pred| * mask / (sum mask + 1e-10) * o * pl                    (:228-230)
//   gradients of loss_a wrt every GAT and decoder parameter, added (atomicAdd) into flat gradient buffers with the
//   parameter buffers' layout; clipping and Adam run afterwards on those buffers (iplan_learner_adam).
// Intermediates that the backward needs (the bi-GRU hidden states, the decoder's per-step vectors) live in a global
// scratch slice per CTA (L2 resident); shared memory holds the working set of the phase at hand.
#include "common.cuh"

namespace iplan {

constexpr int PT = 256;                  // threads per CTA
constexpr int PH = IPLAN_HID;            // 32
constexpr int PG = 3 * PH;               // 96
constexpr int PIN = 16;                  // padded GAT input width

struct PDecLayout { int64_t lin_w, lin_b, wih, whh, bih, bhh, out_w, out_b, total; };
__host__ __device__ inline PDecLayout pdec_layout(int o) {
    PDecLayout L;
    int64_t off = 0;
    auto take = [&](int64_t n) { int64_t at = off; off = pad4(off + n); return at; };
    L.lin_w = take((int64_t)PH * o); L.lin_b = take(PH);
    L.wih = take(PG * PH); L.whh = take(PG * PH); L.bih = take(PG); L.bhh = take(PG);
    L.out_w = take((int64_t)o * PH); L.out_b = take(o);
    L.total = off;
    return L;
}

struct PredArgs {
    const float* gat; int64_t gat_stride; const float* dec; int64_t dec_stride;
    float* g_gat; float* g_dec;
    const float* x0; const float* lat0; const float* att0; const float* target; const float* mask;   // [A][P][N][.]
    const float* gumbel; const uint8_t* keep; const float* scale; float* loss_sum;
    float* scratch; int64_t scratch_per_cta;
    uint64_t seed, counter; float inv_tau, p_drop;
    int P, N, o, L, pl;
};

__device__ __forceinline__ float psig(float x) { return 1.0f / (1.0f + expf(-x)); }

// out[r][c] = act(bias[c] + sum_k in[r][k] * W[c*ldw + k]); in/out anywhere (smem or global), W global
__device__ void cta_dense(float* out, int ldo, const float* in, int ldi, int rows, const float* __restrict__ W, int ldw,
                          const float* __restrict__ bias, int cols, int K, bool relu) {
    for (int idx = threadIdx.x; idx < rows * cols; idx += PT) {
        const int r = idx / cols, c = idx - r * cols;
        float acc = bias ? bias[c] : 0.0f;
        const float* w = W + (int64_t)c * ldw;
        const float* x = in + (int64_t)r * ldi;
        for (int k = 0; k < K; ++k) acc = fmaf(x[k], w[k], acc);
        out[(int64_t)r * ldo + c] = relu ? fmaxf(acc, 0.0f) : acc;
    }
}
// out[r][k] (+)= sum_c d[r][c] * W[c*ldw + k]
__device__ void cta_dense_t(float* out, int ldo, const float* d, int ldd, int rows, const float* __restrict__ W, int ldw,
                            int cols, int K, bool accumulate) {
    for (int idx = threadIdx.x; idx < rows * K; idx += PT) {
        const int r = idx / K, k = idx - r * K;
        float acc = accumulate ? out[(int64_t)r * ldo + k] : 0.0f;
        const float* dr = d + (int64_t)r * ldd;
        for (int c = 0; c < cols; ++c) acc = fmaf(dr[c], W[(int64_t)c * ldw + k], acc);
        out[(int64_t)r * ldo + k] = acc;
    }
}
// G[c*ldg + k] += sum_r d[r][c] * in[r][k]   (atomic: every CTA of an agent adds into the same buffer); gb[c] += sum_r d[r][c]
__device__ void cta_wgrad(float* G, int ldg, float* gb, const float* d, int ldd, const float* in, int ldi, int rows, int cols, int K) {
    for (int idx = threadIdx.x; idx < cols * K; idx += PT) {
        const int c = idx / K, k = idx - c * K;
        float acc = 0.0f;
        for (int r = 0; r < rows; ++r) acc = fmaf(d[(int64_t)r * ldd + c], in[(int64_t)r * ldi + k], acc);
        atomicAdd(G + (int64_t)c * ldg + k, acc);
    }
    if (gb)
        for (int c = threadIdx.x; c < cols; c += PT) {
            float acc = 0.0f;
            for (int r = 0; r < rows; ++r) acc += d[(int64_t)r * ldd + c];
            atomicAdd(gb + c, acc);
        }
}

__global__ void __launch_bounds__(PT, 1) pred_learn_kernel(PredArgs a) {
    extern __shared__ __align__(16) float sm[];
    const int p = blockIdx.x, ag = blockIdx.y, tid = threadIdx.x;
    const int N = a.N, NM1 = N - 1, o = a.o, Ld = a.L, pl = a.pl, in_dim = o + Ld;
    const float* __restrict__ Wg = a.gat + (int64_t)ag * a.gat_stride;
    const float* __restrict__ Wd = a.dec + (int64_t)ag * a.dec_stride;
    float* Gg = a.g_gat + (int64_t)ag * a.gat_stride;
    float* Gd = a.g_dec + (int64_t)ag * a.dec_stride;
    const GatLayout L = gat_layout(in_dim);
    const PDecLayout D = pdec_layout(o);
    const int64_t sample = (int64_t)ag * a.P + p;
    const float* x0 = a.x0 + sample * N * o;
    const float* lat0 = a.lat0 + sample * N * Ld;
    const float* att0 = a.att0 + sample * N * PH;
    const float* target = a.target + sample * N * pl * o;            // [N][pl][o]
    const float gscale = a.mask[sample] * a.scale[ag];                 // d loss / d |err| for this sample's elements

    // ---- shared memory ------------------------------------------------------------------------------------
    float* s_x = sm;                         // [N][PIN]
    float* s_enc = s_x + N * PIN;            // [N][32]  (enc > 0  <=>  its pre-activation > 0)
    float* s_denc = s_enc + N * PH;          // [N][32]
    float* s_dd = s_denc + N * PH;           // [N][N-1] logit difference, later d loss / d (logit difference)
    float* s_hard = s_dd + N * NM1;          // [N][N-1]
    float* s_soft = s_hard + N * NM1;        // [N][N-1]
    float* s_ego = s_soft + N * NM1;         // [N][96]
    float* s_nbr = s_ego + N * PG;           // [N][96]
    float* s_h = s_nbr + N * PG;             // [2][N][32]
    float* s_whh = s_h + 2 * N * PH;         // [96][33] W_hh (padded rows)
    float* s_u = s_whh + PG * 33;            // union region: 448 N floats (the larger, BPTT view)
    // attention-phase view of the union
    float* s_q = s_u;                        // [N][32]
    float* s_k = s_q + N * PH;
    float* s_v = s_k + N * PH;               // ReLU output (v > 0  <=>  pre-activation > 0)
    float* s_xa = s_v + N * PH;
    float* s_hid = s_xa + N * PH;            // [N][32] GAT output = decoder initial hidden
    float* s_gic = s_hid + N * PH;           // [N][96] GRUCell input pre-activation
    float* s_dq = s_gic + N * PG;            // [N][32] ...
    // BPTT-phase view of the union
    float* s_dh = s_u;                       // [N][32]
    float* s_hb = s_dh + N * PH;             // [N][32] hidden before the step
    float* s_dgi = s_hb + N * PH;            // [N][96]
    float* s_dgh = s_dgi + N * PG;           // [N][96]
    float* s_dego = s_dgh + N * PG;          // [N][96]
    float* s_dnbr = s_dego + N * PG;         // [N][96]

    // ---- global scratch ---------------------------------------------------------------------------------------
    float* sc = a.scratch + ((int64_t)ag * a.P + p) * a.scratch_per_cta;
    float* g_hs = sc;                                        // [2][N][N-1][32] bi-GRU hidden after each position
    float* g_dx = g_hs + (int64_t)2 * N * NM1 * PH;          // decoder: x_t [pl][N][o]
    float* g_du = g_dx + (int64_t)pl * N * o;                // u_t [pl][N][32]
    float* g_dhd = g_du + (int64_t)pl * N * PH;              // h_t [pl+1][N][32]
    float* g_dy = g_dhd + (int64_t)(pl + 1) * N * PH;        // y_t [pl][N][32] (after dropout)
    float* g_dout = g_dy + (int64_t)pl * N * PH;             // d out_t [pl][N][o]
    float* g_dgi = g_dout + (int64_t)pl * N * o;             // d gi [pl][N][96]
    float* g_dgh = g_dgi + (int64_t)pl * N * PG;             // d gh [pl][N][96]
    float* g_ddu = g_dgh + (int64_t)pl * N * PG;             // d (pre-ReLU u) [pl][N][32]
    float* g_dhid = g_ddu + (int64_t)pl * N * PH;            // d hidden [N][32]
    float* g_dgc = g_dhid + (int64_t)N * PH;                 // GRUCell d gi [N][96]
    float* g_dgch = g_dgc + (int64_t)N * PG;                 // GRUCell d gh [N][96]

    // ================= forward: GAT =================
    for (int idx = tid; idx < N * PIN; idx += PT) {
        const int n = idx / PIN, c = idx - n * PIN;
        s_x[idx] = c < o ? x0[n * o + c] : (c < in_dim ? lat0[n * Ld + (c - o)] : 0.0f);
    }
    __syncthreads();
    cta_dense(s_enc, PH, s_x, PIN, N, Wg + L.enc_w, in_dim, Wg + L.enc_b, PH, in_dim, true);
    __syncthreads();
    for (int dir = 0; dir < 2; ++dir) {
        const float* wih = Wg + (dir ? L.wih_r : L.wih_f);
        const float* whh = Wg + (dir ? L.whh_r : L.whh_f);
        const float* bhh = Wg + (dir ? L.bhh_r : L.bhh_f);
        cta_dense(s_ego, PG, s_enc, PH, N, wih, 2 * PH, Wg + (dir ? L.bih_r : L.bih_f), PG, PH, false);
        cta_dense(s_nbr, PG, s_enc, PH, N, wih + PH, 2 * PH, nullptr, PG, PH, false);
        for (int idx = tid; idx < PG * PH; idx += PT) s_whh[(idx / PH) * 33 + (idx % PH)] = whh[idx];
        for (int idx = tid; idx < N * PH; idx += PT) s_h[idx] = 0.0f;
        __syncthreads();
        int cur = 0;
        for (int step = 0; step < NM1; ++step) {
            const int s = dir ? NM1 - 1 - step : step;
            const float* hc = s_h + cur * N * PH;
            float* hn = s_h + (cur ^ 1) * N * PH;
            for (int idx = tid; idx < N * PH; idx += PT) {
                const int i = idx >> 5, c = idx & 31;
                const int j = s < i ? s : s + 1;
                const float* hi = hc + i * PH;
                float gh[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const float* w = s_whh + (q * PH + c) * 33;
                    float acc = bhh[q * PH + c];
                    for (int k = 0; k < PH; ++k) acc = fmaf(hi[k], w[k], acc);
                    gh[q] = acc;
                }
                const float* eg = s_ego + i * PG;
                const float* nb = s_nbr + j * PG;
                const float r = psig(eg[c] + nb[c] + gh[0]);
                const float z = psig(eg[PH + c] + nb[PH + c] + gh[1]);
                const float nn = tanhf(eg[2 * PH + c] + nb[2 * PH + c] + r * gh[2]);
                const float hv = (1.0f - z) * nn + z * hi[c];
                hn[idx] = hv;
                g_hs[(((int64_t)dir * N + i) * NM1 + s) * PH + c] = hv;
            }
            cur ^= 1;
            __syncthreads();
        }
    }
    // hard attention: logit difference per edge from the stored hidden states
    {
        const float* he = Wg + L.he_w;                                // [2][64]
        const float db = Wg[L.he_b + 1] - Wg[L.he_b];
        for (int idx = tid; idx < N * NM1; idx += PT) {
            const int i = idx / NM1, s = idx - i * NM1;
            float acc = db;
            for (int dir = 0; dir < 2; ++dir) {
                const float* hv = g_hs + (((int64_t)dir * N + i) * NM1 + s) * PH;
                for (int c = 0; c < PH; ++c) acc = fmaf(hv[c], he[2 * PH + dir * PH + c] - he[dir * PH + c], acc);
            }
            float noise;
            const int64_t edge = (sample * N + i) * NM1 + s;
            if (a.gumbel) noise = a.gumbel[2 * edge + 1] - a.gumbel[2 * edge];
            else {
                const uint4 rnd = philox4x32(make_uint4((uint32_t)edge, (uint32_t)(edge >> 32), (uint32_t)a.counter, (uint32_t)(a.counter >> 32)),
                                             make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)));
                const float uu = u01(rnd.x);
                noise = logf(uu) - logf(1.0f - uu);
            }
            s_hard[idx] = psig((acc + noise) * a.inv_tau);
        }
    }
    cta_dense(s_q, PH, s_enc, PH, N, Wg + L.q_w, PH, nullptr, PH, PH, false);
    cta_dense(s_k, PH, s_enc, PH, N, Wg + L.k_w, PH, nullptr, PH, PH, false);
    cta_dense(s_v, PH, s_enc, PH, N, Wg + L.v_w, PH, Wg + L.v_b, PH, PH, true);
    __syncthreads();
    for (int idx = tid; idx < N * NM1; idx += PT) {                   // scores
        const int i = idx / NM1, s = idx - i * NM1, j = s < i ? s : s + 1;
        float acc = 0.0f;
        for (int c = 0; c < PH; ++c) acc = fmaf(s_q[i * PH + c], s_k[j * PH + c], acc);
        s_soft[idx] = acc / 5.656854249492381f;
    }
    __syncthreads();
    for (int i = tid; i < N; i += PT) {                               // softmax over the N-1 neighbours of ego i
        float mx = -INFINITY;
        for (int s = 0; s < NM1; ++s) mx = fmaxf(mx, s_soft[i * NM1 + s]);
        float den = 0.0f;
        for (int s = 0; s < NM1; ++s) { const float e = expf(s_soft[i * NM1 + s] - mx); s_soft[i * NM1 + s] = e; den += e; }
        for (int s = 0; s < NM1; ++s) s_soft[i * NM1 + s] /= den;
    }
    __syncthreads();
    for (int idx = tid; idx < N * PH; idx += PT) {                    // x_i = sum_s soft * hard * v_j
        const int i = idx >> 5, c = idx & 31;
        float acc = 0.0f;
        for (int s = 0; s < NM1; ++s) acc = fmaf(s_soft[i * NM1 + s] * s_hard[i * NM1 + s], s_v[(s < i ? s : s + 1) * PH + c], acc);
        s_xa[idx] = acc;
    }
    __syncthreads();
    cta_dense(s_gic, PG, s_xa, PH, N, Wg + L.c_wih, PH, Wg + L.c_bih, PG, PH, false);
    __syncthreads();
    for (int idx = tid; idx < N * PH; idx += PT) {                    // GRUCell(x, att0)
        const int i = idx >> 5, c = idx & 31;
        const float* hp = att0 + i * PH;
        float gh[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float* w = Wg + L.c_whh + (q * PH + c) * PH;
            float acc = Wg[L.c_bhh + q * PH + c];
            for (int k = 0; k < PH; ++k) acc = fmaf(hp[k], w[k], acc);
            gh[q] = acc;
        }
        const float* gi = s_gic + i * PG;
        const float r = psig(gi[c] + gh[0]), z = psig(gi[PH + c] + gh[1]);
        const float nn = tanhf(gi[2 * PH + c] + r * gh[2]);
        const float hv = (1.0f - z) * nn + z * hp[c];
        s_hid[idx] = hv;
        g_dhd[idx] = hv;                                              // decoder h_0
    }
    __syncthreads();

    // ================= forward: decoder roll-out (one warp per node, lane = hidden unit) =================
    const int lane = tid & 31, warp = tid >> 5;
    const float keep_scale = 1.0f / (1.0f - a.p_drop);
    auto kept = [&](int t, int n, int c) -> bool {                    // the dropout draw of element (t, n, c), same in both passes
        const int64_t kidx = ((sample * pl + t) * N + n) * PH + c;
        if (a.keep) return a.keep[kidx] != 0;
        const uint4 rnd = philox4x32(make_uint4((uint32_t)kidx, (uint32_t)(kidx >> 32), (uint32_t)a.counter, (uint32_t)(a.counter >> 32)),
                                     make_uint2((uint32_t)a.seed ^ 0x9e3779b9u, (uint32_t)(a.seed >> 32)));
        return u01(rnd.x) >= a.p_drop;
    };
    float loss_local = 0.0f;
    for (int n = warp; n < N; n += PT / 32) {
        for (int c = lane; c < o; c += 32) g_dx[(int64_t)n * o + c] = x0[n * o + c];       // x_0 (layout [t][N][o])
        __syncwarp();
        for (int t = 0; t < pl; ++t) {
            const float* xt = g_dx + ((int64_t)t * N + n) * o;
            float u = Wd[D.lin_b + lane];
            for (int k = 0; k < o; ++k) u = fmaf(Wd[D.lin_w + lane * o + k], xt[k], u);
            u = fmaxf(u, 0.0f);
            g_du[((int64_t)t * N + n) * PH + lane] = u;
            const float* hp = g_dhd + ((int64_t)t * N + n) * PH;
            __syncwarp();
            const float* ut = g_du + ((int64_t)t * N + n) * PH;
            float gi[3], gh[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                float ai = Wd[D.bih + q * PH + lane], ah = Wd[D.bhh + q * PH + lane];
                const float* wi = Wd + D.wih + (q * PH + lane) * PH;
                const float* wh = Wd + D.whh + (q * PH + lane) * PH;
                for (int k = 0; k < PH; ++k) { ai = fmaf(wi[k], ut[k], ai); ah = fmaf(wh[k], hp[k], ah); }
                gi[q] = ai; gh[q] = ah;
            }
            const float r = psig(gi[0] + gh[0]), z = psig(gi[1] + gh[1]);
            const float nn = tanhf(gi[2] + r * gh[2]);
            const float hv = (1.0f - z) * nn + z * hp[lane];
            g_dhd[((int64_t)(t + 1) * N + n) * PH + lane] = hv;
            const bool kp = kept(t, n, lane);
            const float y = kp ? tanhf(hv) * keep_scale : 0.0f;
            g_dy[((int64_t)t * N + n) * PH + lane] = y;
            __syncwarp();
            const float* yt = g_dy + ((int64_t)t * N + n) * PH;
            if (lane < o) {
                float ov = Wd[D.out_b + lane];
                for (int k = 0; k < PH; ++k) ov = fmaf(Wd[D.out_w + lane * PH + k], yt[k], ov);
                if (t + 1 < pl) g_dx[((int64_t)(t + 1) * N + n) * o + lane] = ov;
                const float e = ov - target[((int64_t)n * pl + t) * o + lane];
                loss_local += fabsf(e) * a.mask[sample];
                g_dout[((int64_t)t * N + n) * o + lane] = (e > 0.0f ? 1.0f : (e < 0.0f ? -1.0f : 0.0f)) * gscale;   // d loss / d out_t (own term)
            }
            __syncwarp();
        }
    }
    loss_local = warp_sum(loss_local);
    if (lane == 0) atomicAdd(a.loss_sum + ag, loss_local);

    // ================= backward: decoder (same warp owns the node) =================
    for (int n = warp; n < N; n += PT / 32) {
        float dh = 0.0f;                                              // d loss / d h_t[lane], carried backwards
        for (int t = pl - 1; t >= 0; --t) {
            const float* dot = g_dout + ((int64_t)t * N + n) * o;     // complete: own term + d x_{t+1} (added below)
            const float* hp = g_dhd + ((int64_t)t * N + n) * PH;
            const float* ut = g_du + ((int64_t)t * N + n) * PH;
            const float hv = g_dhd[((int64_t)(t + 1) * N + n) * PH + lane];
            float dy = 0.0f;
            for (int k = 0; k < o; ++k) dy = fmaf(dot[k], Wd[D.out_w + k * PH + lane], dy);
            const float th = tanhf(hv);
            if (kept(t, n, lane)) dh += dy * keep_scale * (1.0f - th * th);                    // dropped units pass nothing
            // recompute the gates of step t
            float gi[3], gh[3];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                float ai = Wd[D.bih + q * PH + lane], ah = Wd[D.bhh + q * PH + lane];
                const float* wi = Wd + D.wih + (q * PH + lane) * PH;
                const float* wh = Wd + D.whh + (q * PH + lane) * PH;
                for (int k = 0; k < PH; ++k) { ai = fmaf(wi[k], ut[k], ai); ah = fmaf(wh[k], hp[k], ah); }
                gi[q] = ai; gh[q] = ah;
            }
            const float r = psig(gi[0] + gh[0]), z = psig(gi[1] + gh[1]);
            const float nn = tanhf(gi[2] + r * gh[2]);
            const float dn = dh * (1.0f - z), dz = dh * (hp[lane] - nn);
            const float dan = dn * (1.0f - nn * nn), daz = dz * z * (1.0f - z), dar = dan * gh[2] * r * (1.0f - r);
            float* dgi = g_dgi + ((int64_t)t * N + n) * PG;
            float* dgh = g_dgh + ((int64_t)t * N + n) * PG;
            dgi[lane] = dar; dgi[PH + lane] = daz; dgi[2 * PH + lane] = dan;
            dgh[lane] = dar; dgh[PH + lane] = daz; dgh[2 * PH + lane] = dan * r;
            __syncwarp();
            float dhp = dh * z, du = 0.0f;
            for (int g = 0; g < PG; ++g) {
                dhp = fmaf(dgh[g], Wd[D.whh + g * PH + lane], dhp);
                du = fmaf(dgi[g], Wd[D.wih + g * PH + lane], du);
            }
            du = ut[lane] > 0.0f ? du : 0.0f;
            g_ddu[((int64_t)t * N + n) * PH + lane] = du;
            __syncwarp();
            if (t > 0 && lane < o) {                                  // x_t = out_{t-1}: its gradient joins d out_{t-1}
                const float* ddu = g_ddu + ((int64_t)t * N + n) * PH;
                float dx = 0.0f;
                for (int c = 0; c < PH; ++c) dx = fmaf(ddu[c], Wd[D.lin_w + c * o + lane], dx);
                g_dout[((int64_t)(t - 1) * N + n) * o + lane] += dx;
            }
            __syncwarp();
            dh = dhp;
        }
        g_dhid[n * PH + lane] = dh;
    }
    __syncthreads();
    // decoder weight gradients: sums over (t, n) of outer products of the stored vectors
    cta_wgrad(Gd + D.out_w, PH, Gd + D.out_b, g_dout, o, g_dy, PH, pl * N, o, PH);
    cta_wgrad(Gd + D.wih, PH, Gd + D.bih, g_dgi, PG, g_du, PH, pl * N, PG, PH);
    cta_wgrad(Gd + D.whh, PH, Gd + D.bhh, g_dgh, PG, g_dhd, PH, pl * N, PG, PH);        // h_{t}, t = 0..pl-1 are the first pl*N rows
    cta_wgrad(Gd + D.lin_w, o, Gd + D.lin_b, g_ddu, PH, g_dx, o, pl * N, PH, o);

    // ================= backward: GRUCell, attention =================
    for (int idx = tid; idx < N * PH; idx += PT) {                    // GRUCell backward (recompute its gates)
        const int i = idx >> 5, c = idx & 31;
        const float* hp = att0 + i * PH;
        float gh[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float* w = Wg + L.c_whh + (q * PH + c) * PH;
            float acc = Wg[L.c_bhh + q * PH + c];
            for (int k = 0; k < PH; ++k) acc = fmaf(hp[k], w[k], acc);
            gh[q] = acc;
        }
        const float* gi = s_gic + i * PG;
        const float r = psig(gi[c] + gh[0]), z = psig(gi[PH + c] + gh[1]);
        const float nn = tanhf(gi[2 * PH + c] + r * gh[2]);
        const float dh = g_dhid[idx];
        const float dn = dh * (1.0f - z), dz = dh * (hp[c] - nn);
        const float dan = dn * (1.0f - nn * nn), daz = dz * z * (1.0f - z), dar = dan * gh[2] * r * (1.0f - r);
        g_dgc[i * PG + c] = dar; g_dgc[i * PG + PH + c] = daz; g_dgc[i * PG + 2 * PH + c] = dan;
        g_dgch[i * PG + c] = dar; g_dgch[i * PG + PH + c] = daz; g_dgch[i * PG + 2 * PH + c] = dan * r;
    }
    __syncthreads();
    cta_wgrad(Gg + L.c_wih, PH, Gg + L.c_bih, g_dgc, PG, s_xa, PH, N, PG, PH);
    cta_wgrad(Gg + L.c_whh, PH, Gg + L.c_bhh, g_dgch, PG, att0, PH, N, PG, PH);
    float* s_dxa = s_dq;                                              // [N][32] d x (aggregated message)
    float* s_dk = s_dxa + N * PH;
    float* s_dv = s_dk + N * PH;
    float* s_dqq = s_dv + N * PH;
    cta_dense_t(s_dxa, PH, g_dgc, PG, N, Wg + L.c_wih, PH, PG, PH, false);
    for (int idx = tid; idx < 3 * N * PH; idx += PT) s_dk[idx] = 0.0f;          // d k, d v, d q
    __syncthreads();
    // per edge: d w = d x_i . v_j ; d soft, d hard ; d v_j += w d x_i (accumulated per j below)
    for (int idx = tid; idx < N * NM1; idx += PT) {
        const int i = idx / NM1, s = idx - i * NM1, j = s < i ? s : s + 1;
        float dw = 0.0f;
        for (int c = 0; c < PH; ++c) dw = fmaf(s_dxa[i * PH + c], s_v[j * PH + c], dw);
        const float so = s_soft[idx], hd = s_hard[idx];
        s_dd[idx] = dw * so * hd * (1.0f - hd) * a.inv_tau;           // d loss / d (logit difference)
        s_ego[idx] = dw * hd;                                          // d soft  (s_ego is free here: N*(N-1) <= N*96)
    }
    __syncthreads();
    for (int i = tid; i < N; i += PT) {                               // softmax backward per ego, scaled by 1/sqrt(D)
        float dot = 0.0f;
        for (int s = 0; s < NM1; ++s) dot = fmaf(s_soft[i * NM1 + s], s_ego[i * NM1 + s], dot);
        for (int s = 0; s < NM1; ++s) s_ego[i * NM1 + s] = s_soft[i * NM1 + s] * (s_ego[i * NM1 + s] - dot) / 5.656854249492381f;   // d score
    }
    __syncthreads();
    for (int idx = tid; idx < N * PH; idx += PT) {                    // d q_i, and the gathers d k_j, d v_j (loop over the egos that see j)
        const int n = idx >> 5, c = idx & 31;
        float dq = 0.0f;
        for (int s = 0; s < NM1; ++s) dq = fmaf(s_ego[n * NM1 + s], s_k[(s < n ? s : s + 1) * PH + c], dq);
        s_dqq[idx] = dq;
        float dk = 0.0f, dv = 0.0f;
        for (int i = 0; i < N; ++i) {                                 // node n is neighbour position s = n (if n < i) or n - 1 (if n > i) of ego i
            if (i == n) continue;
            const int s = n < i ? n : n - 1;
            dk = fmaf(s_ego[i * NM1 + s], s_q[i * PH + c], dk);
            dv = fmaf(s_soft[i * NM1 + s] * s_hard[i * NM1 + s], s_dxa[i * PH + c], dv);
        }
        s_dk[idx] = dk;
        s_dv[idx] = s_v[idx] > 0.0f ? dv : 0.0f;                      // through v = ReLU(.)
    }
    __syncthreads();
    cta_wgrad(Gg + L.q_w, PH, nullptr, s_dqq, PH, s_enc, PH, N, PH, PH);
    cta_wgrad(Gg + L.k_w, PH, nullptr, s_dk, PH, s_enc, PH, N, PH, PH);
    cta_wgrad(Gg + L.v_w, PH, Gg + L.v_b, s_dv, PH, s_enc, PH, N, PH, PH);
    cta_dense_t(s_denc, PH, s_dqq, PH, N, Wg + L.q_w, PH, PH, PH, false);
    __syncthreads();
    cta_dense_t(s_denc, PH, s_dk, PH, N, Wg + L.k_w, PH, PH, PH, true);
    __syncthreads();
    cta_dense_t(s_denc, PH, s_dv, PH, N, Wg + L.v_w, PH, PH, PH, true);
    // hard-attention head: d logits = (-dd, +dd); d W_he[c][dir*32 + k] = sum dd * (+-) h ; d b_he
    {
        {                                                             // thread = (edge group, dir, k): 4 x 2 x 32
            const int grp = tid >> 6, dir = (tid >> 5) & 1, kq = tid & 31;
            float acc = 0.0f;
            for (int e = grp; e < N * NM1; e += 4) acc = fmaf(s_dd[e], g_hs[((int64_t)dir * N * NM1 + e) * PH + kq], acc);
            atomicAdd(Gg + L.he_w + 2 * PH + dir * PH + kq, acc);      // row 1 (+)
            atomicAdd(Gg + L.he_w + dir * PH + kq, -acc);              // row 0 (-)
        }
        if (tid == 0) {
            float acc = 0.0f;
            for (int e = 0; e < N * NM1; ++e) acc += s_dd[e];
            atomicAdd(Gg + L.he_b + 1, acc);
            atomicAdd(Gg + L.he_b, -acc);
        }
    }
    __syncthreads();

    // ================= backward: bidirectional GRU (BPTT), one direction at a time =================
    for (int dir = 0; dir < 2; ++dir) {
        const float* wih = Wg + (dir ? L.wih_r : L.wih_f);
        const float* whh = Wg + (dir ? L.whh_r : L.whh_f);
        const float* bhh = Wg + (dir ? L.bhh_r : L.bhh_f);
        float* g_wih = Gg + (dir ? L.wih_r : L.wih_f);
        float* g_whh = Gg + (dir ? L.whh_r : L.whh_f);
        const float* he = Wg + L.he_w;
        cta_dense(s_ego, PG, s_enc, PH, N, wih, 2 * PH, Wg + (dir ? L.bih_r : L.bih_f), PG, PH, false);
        cta_dense(s_nbr, PG, s_enc, PH, N, wih + PH, 2 * PH, nullptr, PG, PH, false);
        for (int idx = tid; idx < PG * PH; idx += PT) s_whh[(idx / PH) * 33 + (idx % PH)] = whh[idx];
        for (int idx = tid; idx < N * PH; idx += PT) s_dh[idx] = 0.0f;
        for (int idx = tid; idx < 2 * N * PG; idx += PT) s_dego[idx] = 0.0f;    // d ego, d nbr
        // per-thread accumulators of d W_hh: entries (g, k) = tid + q * PT, q < 12
        float accw[(PG * PH + PT - 1) / PT];
#pragma unroll
        for (int q = 0; q < (PG * PH + PT - 1) / PT; ++q) accw[q] = 0.0f;
        float accb = 0.0f;                                            // d b_hh[tid] for tid < 96
        __syncthreads();
        for (int step = NM1 - 1; step >= 0; --step) {                 // positions in reverse processing order
            const int s = dir ? NM1 - 1 - step : step;
            const int s_prev = dir ? s + 1 : s - 1;                   // position processed just before s (none if step == 0)
            for (int idx = tid; idx < N * PH; idx += PT) {
                const int i = idx >> 5, c = idx & 31;
                s_hb[idx] = step > 0 ? g_hs[(((int64_t)dir * N + i) * NM1 + s_prev) * PH + c] : 0.0f;
                s_dh[idx] += s_dd[i * NM1 + s] * (he[2 * PH + dir * PH + c] - he[dir * PH + c]);    // d hh from the logit difference
            }
            __syncthreads();
            for (int idx = tid; idx < N * PH; idx += PT) {            // gates of (ego i, unit c) recomputed, their pre-activation gradients
                const int i = idx >> 5, c = idx & 31;
                const int j = s < i ? s : s + 1;
                const float* hi = s_hb + i * PH;
                float gh[3];
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    const float* w = s_whh + (q * PH + c) * 33;
                    float acc = bhh[q * PH + c];
                    for (int k = 0; k < PH; ++k) acc = fmaf(hi[k], w[k], acc);
                    gh[q] = acc;
                }
                const float* eg = s_ego + i * PG;
                const float* nb = s_nbr + j * PG;
                const float r = psig(eg[c] + nb[c] + gh[0]);
                const float z = psig(eg[PH + c] + nb[PH + c] + gh[1]);
                const float nn = tanhf(eg[2 * PH + c] + nb[2 * PH + c] + r * gh[2]);
                const float dh = s_dh[idx];
                const float dn = dh * (1.0f - z), dz = dh * (hi[c] - nn);
                const float dan = dn * (1.0f - nn * nn), daz = dz * z * (1.0f - z), dar = dan * gh[2] * r * (1.0f - r);
                s_dgi[i * PG + c] = dar; s_dgi[i * PG + PH + c] = daz; s_dgi[i * PG + 2 * PH + c] = dan;
                s_dgh[i * PG + c] = dar; s_dgh[i * PG + PH + c] = daz; s_dgh[i * PG + 2 * PH + c] = dan * r;
                s_dh[idx] = dh * z;                                   // direct path to h_before; the W_hh path is added below
            }
            __syncthreads();
            for (int idx = tid; idx < N * PH; idx += PT) {            // d h_before += d gh W_hh
                const int i = idx >> 5, c = idx & 31;
                float acc = s_dh[idx];
                const float* dg = s_dgh + i * PG;
                for (int g = 0; g < PG; ++g) acc = fmaf(dg[g], s_whh[g * 33 + c], acc);
                s_dh[idx] = acc;
            }
#pragma unroll
            for (int q = 0; q < (PG * PH + PT - 1) / PT; ++q) {       // d W_hh[g][k] += sum_i d gh[i][g] h_before[i][k]
                const int e = tid + q * PT;
                if (e < PG * PH) {
                    const int g = e >> 5, k = e & 31;
                    float acc = accw[q];
                    for (int i = 0; i < N; ++i) acc = fmaf(s_dgh[i * PG + g], s_hb[i * PH + k], acc);
                    accw[q] = acc;
                }
            }
            if (tid < PG) { float acc = accb; for (int i = 0; i < N; ++i) acc += s_dgh[i * PG + tid]; accb = acc; }
            for (int idx = tid; idx < N * PG; idx += PT) s_dego[idx] += s_dgi[idx];          // ego i keeps its own gradient
            for (int idx = tid; idx < 2 * PG; idx += PT) {            // neighbour rows: j = s for egos i > s, j = s + 1 for egos i <= s
                const int which = idx / PG, g = idx - which * PG;
                float acc = 0.0f;
                if (which == 0) { for (int i = s + 1; i < N; ++i) acc += s_dgi[i * PG + g]; s_dnbr[s * PG + g] += acc; }
                else { for (int i = 0; i <= s && i < N; ++i) acc += s_dgi[i * PG + g]; s_dnbr[(s + 1) * PG + g] += acc; }
            }
            __syncthreads();
        }
#pragma unroll
        for (int q = 0; q < (PG * PH + PT - 1) / PT; ++q) {
            const int e = tid + q * PT;
            if (e < PG * PH) atomicAdd(g_whh + e, accw[q]);
        }
        if (tid < PG) atomicAdd(Gg + (dir ? L.bhh_r : L.bhh_f) + tid, accb);
        // input projections: W_ih = [ego part | neighbour part] (row pitch 64), b_ih from the ego part
        cta_wgrad(g_wih, 2 * PH, Gg + (dir ? L.bih_r : L.bih_f), s_dego, PG, s_enc, PH, N, PG, PH);
        cta_wgrad(g_wih + PH, 2 * PH, nullptr, s_dnbr, PG, s_enc, PH, N, PG, PH);
        __syncthreads();
        cta_dense_t(s_denc, PH, s_dego, PG, N, wih, 2 * PH, PG, PH, true);
        __syncthreads();
        cta_dense_t(s_denc, PH, s_dnbr, PG, N, wih + PH, 2 * PH, PG, PH, true);
        __syncthreads();
    }
    // ================= backward: encoder =================
    for (int idx = tid; idx < N * PH; idx += PT) s_denc[idx] = s_enc[idx] > 0.0f ? s_denc[idx] : 0.0f;
    __syncthreads();
    cta_wgrad(Gg + L.enc_w, in_dim, Gg + L.enc_b, s_denc, PH, s_x, PIN, N, PH, in_dim);
}

}  // namespace iplan

extern "C" int64_t iplan_pdec_layout(int obs_dim, int64_t* offsets) {
    const iplan::PDecLayout L = iplan::pdec_layout(obs_dim);
    if (offsets) { const int64_t o[8] = {L.lin_w, L.lin_b, L.wih, L.whh, L.bih, L.bhh, L.out_w, L.out_b}; for (int i = 0; i < 8; ++i) offsets[i] = o[i]; }
    return L.total;
}

namespace iplan {
// dynamic shared memory of pred_learn_kernel at N slots
constexpr size_t pred_learn_smem_bytes(int N) {
    return sizeof(float) * ((size_t)N * PIN + 2 * (size_t)N * PH + 3 * (size_t)N * (N - 1) + 2 * (size_t)N * PG
                            + 2 * (size_t)N * PH + PG * 33 + 2 * (size_t)N * PH + 4 * (size_t)N * PG);
}
static_assert(pred_learn_smem_bytes(IPLAN_PRED_LEARN_MAX_SLOTS) <= 227 * 1024 && pred_learn_smem_bytes(IPLAN_PRED_LEARN_MAX_SLOTS + 1) > 227 * 1024,
              "IPLAN_PRED_LEARN_MAX_SLOTS (include/iplan_b200.h) is not the largest slot count that fits");
}  // namespace iplan

extern "C" int64_t iplan_pred_learn_scratch_floats(int n_agents, int n_samples, int n_slots, int obs_dim, int pred_len) {
    const int64_t N = n_slots, pl = pred_len, o = obs_dim, H = IPLAN_HID, G = 3 * IPLAN_HID;
    const int64_t per = 2 * N * (N - 1) * H + pl * N * o + pl * N * H + (pl + 1) * N * H + pl * N * H + pl * N * o
                        + 2 * pl * N * G + pl * N * H + N * H + 2 * N * G;
    return (int64_t)n_agents * n_samples * ((per + 3) & ~int64_t(3));
}

extern "C" int iplan_pred_learn(const float* gat_params, int64_t gat_stride, const float* dec_params, int64_t dec_stride,
                                float* g_gat, float* g_dec,
                                const float* x0, const float* lat0, const float* att0, const float* target, const float* mask,
                                const float* gumbel, const uint8_t* keep, const float* scale, float* loss_sum,
                                float* scratch, int64_t scratch_floats, uint64_t seed, uint64_t counter, float tau, float p_drop,
                                int n_agents, int n_samples, int n_slots, int obs_dim, int latent_dim, int pred_len, void* stream) {
    using namespace iplan;
    IPLAN_REQUIRE(gat_params && dec_params && g_gat && g_dec && x0 && lat0 && att0 && target && mask && scale && loss_sum && scratch,
                  "pred_learn: null pointer");
    IPLAN_REQUIRE(n_slots >= 2 && n_slots <= IPLAN_MAX_SLOTS && obs_dim > 0 && obs_dim + latent_dim <= PIN && obs_dim <= 32 && pred_len > 0,
                  "pred_learn: bad sizes");
    IPLAN_REQUIRE(n_agents > 0 && n_samples > 0 && tau > 0.f && p_drop >= 0.f && p_drop < 1.f, "pred_learn: bad arguments");
    const int64_t need = iplan_pred_learn_scratch_floats(n_agents, n_samples, n_slots, obs_dim, pred_len);
    IPLAN_REQUIRE(scratch_floats >= need, "pred_learn: scratch too small (%lld floats, need %lld)", (long long)scratch_floats, (long long)need);
    PredArgs a;
    a.gat = gat_params; a.gat_stride = gat_stride; a.dec = dec_params; a.dec_stride = dec_stride; a.g_gat = g_gat; a.g_dec = g_dec;
    a.x0 = x0; a.lat0 = lat0; a.att0 = att0; a.target = target; a.mask = mask; a.gumbel = gumbel; a.keep = keep; a.scale = scale;
    a.loss_sum = loss_sum; a.scratch = scratch; a.scratch_per_cta = need / ((int64_t)n_agents * n_samples);
    a.seed = seed; a.counter = counter; a.inv_tau = 1.0f / tau; a.p_drop = p_drop;
    a.P = n_samples; a.N = n_slots; a.o = obs_dim; a.L = latent_dim; a.pl = pred_len;
    const size_t smem = pred_learn_smem_bytes(n_slots);
    IPLAN_REQUIRE(smem <= 227 * 1024, "pred_learn: n_slots %d needs %zu B of shared memory (at most %d slots fit)", n_slots, smem,
                  IPLAN_PRED_LEARN_MAX_SLOTS);
    static size_t configured = 0;
    if (smem > configured) {
        cudaError_t e = cudaFuncSetAttribute(pred_learn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("pred_learn: smem attr %zu: %s", smem, cudaGetErrorString(e)); return (int)e; }
        configured = smem;
    }
    pred_learn_kernel<<<dim3(n_samples, n_agents), PT, smem, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("pred_learn");
}
