// iPLAN-FC behaviour module (reference nova/behavior_FC_policy.py, nova/behavior_FC_net.py): the fully-connected
// encoder's rollout step and the fused forward + backward of Behavior_policy.learn.  Arithmetic: tools/beh_fc_oracle.py.
//
//   encoder  x (K0 = W o) -> h1 = tanh(W1 x + b1) (E) -> h2 = tanh(W2 h1 + b2) (E) -> z = softmax(W3 h2 + b3) (L)
//   decoder  [x | z_prev] (K0 + L) -> d1 = tanh(V1 . + c1) (Dh) -> d2 = tanh(V2 d1 + c2) (Dh) -> pred = V3 d2 + c3 (K0)
//
// learn: nothing recurs (latent_{j-1} is the encoder's output on the window ending at j-1), so every (agent-net, env,
// slot, position) row is independent.  A CTA owns one agent-net's parameters (staged once in shared memory, both
// orientations where the backward needs them) and walks tiles of 64 consecutive rows (positions of the same chain are
// consecutive, so neighbouring rows share most of their history).  Activations are feature-major [feature][row] fp32 in
// shared memory.  The 64-wide decoder products (forward through V1, V2, V3; input gradients through V3 and V2; weight
// gradients dV1, dV2, dV3) run on the tensor cores: mma.sync.m16n8k16 with both operands split into f16 hi + lo
// (hi*hi + lo*hi + hi*lo, split_mma.cuh), one warp per 16 rows x 32 outputs (or 16 x 32 of dW); the weight operands are
// split once per CTA into fragment order.  The 32-wide encoder products (and the latent columns) are FP32 register-tiled.
// Weight gradients accumulate per thread in registers across all tiles of the CTA, one add of the tile's partial sum per
// tile (a CTA walks over a thousand tiles at 512 envs; Kahan compensation of those sums does not fit the register budget,
// 236 of 255 without it); the loss, one register, is added with Kahan compensation.  At the end each CTA stores its partial sums into its own slot; the last CTA
// of the agent-net adds the slots in CTA order (det_scratch), so the result does not depend on scheduling.  The backward
// runs on d loss / d prediction divided by the loss scale (a sign, so the bias gradient of the output layer is an exact
// integer sum); the reducing CTA multiplies every gradient by the scale once.
#include <cuda_fp16.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>

#include "common.cuh"

namespace iplan {
#include "split_mma.cuh"
namespace {

constexpr int FC_E = 32;            // encoder_rnn_dim
constexpr int FC_DH = 64;           // decoder_rnn_dim
constexpr int FC_KMAX = 64;         // W o + L (decoder input) upper bound
constexpr int FC_LMAX = 8;          // latent_dim upper bound
constexpr int FC_THREADS = 256;
constexpr int FC_R = 64;            // rows per tile
constexpr int FC_RP = FC_R + 4;     // row pitch of the feature-major activations
constexpr int FC_NACC = 63;         // per-thread gradient accumulators (see acc_dst)
static_assert(FC_E == IPLAN_BFC_ENC_HIDDEN && FC_DH == IPLAN_BFC_DEC_HIDDEN && FC_KMAX == IPLAN_BFC_MAX_IN &&
              FC_LMAX == IPLAN_BFC_MAX_LATENT, "iplan_b200.h limits are the kernel's");
static_assert(FC_THREADS == 4 * FC_R && FC_LMAX == 2 * 4, "softmax / latent gradient: four threads per row, two columns each");
static_assert(FC_THREADS == (FC_DH / 4) * (FC_R / 4) && FC_THREADS == (FC_E / 4) * (FC_R / 2), "product thread maps");
static_assert(FC_THREADS == 4 * FC_DH && FC_THREADS == FC_E * FC_LMAX, "bias and W3 gradient thread maps");

struct FcSmem {
    // one agent-net's parameters, zero padded
    float w1t[FC_KMAX][FC_E];       // W1^T [input k][hidden n], k < K0
    float w2t[FC_E][FC_E];          // W2^T
    float w2[FC_E][FC_E];           // W2
    float w3[FC_LMAX][FC_E];        // W3, rows >= L zero
    // B fragments of the 64 x 64 tensor-core products, [operand][hi|lo][n-tile][k-block][lane] (b0 = k 2t, 2t+1 ; b1 =
    // k 2t+8, 2t+9 ; n = lane / 4): VF_V1, VF_V2, VF_V3 give B(k, n) = V[n][k] (forward), VB_V3, VB_V2 give V[k][n]
    // (input gradient); zero outside V1's K0 + L columns and V3's K0 rows
    uint2 vf[5][2][8][4][32];
    float v1lat[FC_DH][FC_LMAX];    // V1[:, K0 + l]
    float b1[FC_E], b2[FC_E], b3[FC_LMAX], c1[FC_DH], c2[FC_DH], c3[FC_KMAX];
    // one tile, feature-major
    float p[FC_KMAX][FC_RP];        // encoder input: window ending at j - 1
    float din[FC_KMAX][FC_RP];      // decoder input: [window ending at j | latent_{j-1} | 0]
    float d1[FC_DH][FC_RP];         // decoder hidden 1, then its gradient G1
    float d2[FC_DH][FC_RP];         // decoder hidden 2, then G2
    float g3[FC_KMAX][FC_RP];       // d loss / d prediction, divided by scale (-1, 0 or 1)
    float h1[FC_E][FC_RP];          // encoder hidden 1, then GE1
    float h2[FC_E][FC_RP];          // encoder hidden 2, then GE2
    float ge3[FC_LMAX][FC_RP];      // d loss / d logits
    int64_t rowoff[FC_R];           // hist offset of the row's chain at t = 0
    int jpos[FC_R];                 // position j; -1 past the last row
    float red[FC_THREADS];
};
static_assert(sizeof(FcSmem) <= 227 * 1024, "one CTA per SM");

enum { VF_V1 = 0, VF_V2, VF_V3, VB_V3, VB_V2 };

struct FcLearnArgs {
    const float* enc; const float* dec; int64_t enc_stride, dec_stride;
    float* g_enc; float* g_dec; const float* hist; float scale; float* b_loss;
    int n_eps, n_steps, n_slots, obs_dim, latent_dim, hist_len, n_pos;
    float* part; unsigned* count;
};

// y[i][b] = sum_{k < kin} Wk[k][n0 + i] X[k][r0 + b]   (FP32, the 32-wide encoder products)
__device__ __forceinline__ void rowmm(const float* Wk, int ldw, const float* X, int kin, int n0, int r0, float (&y)[4][2]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) y[i][0] = y[i][1] = 0.0f;
#pragma unroll 4
    for (int k = 0; k < kin; ++k) {
        const float4 w = *reinterpret_cast<const float4*>(Wk + k * ldw + n0);
        const float2 x = *reinterpret_cast<const float2*>(X + k * FC_RP + r0);
        const float wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            y[i][0] = fmaf(wv[i], x.x, y[i][0]);
            y[i][1] = fmaf(wv[i], x.y, y[i][1]);
        }
    }
}

// acc += x, with the rounding error carried in c (Kahan): the loss runs over every tile of the CTA
__device__ __forceinline__ void kadd(float& acc, float& c, float x) {
    const float y = x - c, t = acc + y;
    c = (t - acc) - y;
    acc = t;
}

// Y[r][n] = sum_{k < 64} X[k][r] B(k, n) on the tensor cores for the warp's 16 rows r = 16 rb + g + 8 (e >> 1) and 32
// outputs n = 32 nh + 8 nt + 2 t + (e & 1) (g = lane / 4, t = lane % 4): y[nt][e].  12 MMAs per output tile.
__device__ __forceinline__ void rowmma(const uint2 (&Bf)[2][8][4][32], const float* X, int rb, int nh, int lane, float (&y)[4][4]) {
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) y[nt][0] = y[nt][1] = y[nt][2] = y[nt][3] = 0.0f;
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
        const float* x = X + (16 * kb + 2 * t) * FC_RP + 16 * rb + g;
        uint32_t ah[4], al[4];
        l64_split(x[0], x[FC_RP], ah[0], al[0]);
        l64_split(x[8], x[FC_RP + 8], ah[1], al[1]);
        l64_split(x[8 * FC_RP], x[9 * FC_RP], ah[2], al[2]);
        l64_split(x[8 * FC_RP + 8], x[9 * FC_RP + 8], ah[3], al[3]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const uint2 bh = Bf[0][4 * nh + nt][kb][lane], bl = Bf[1][4 * nh + nt][kb][lane];
            l64_mma(y[nt], ah, bh.x, bh.y);
            l64_mma(y[nt], al, bh.x, bh.y);
            l64_mma(y[nt], ah, bl.x, bl.y);
        }
    }
}

// acc[OFF + 4 nt + e] += (sum over the tile's 64 rows of G[m][r] X[n][r] on the tensor cores, for the warp's 16 x 32 block
// of a 64 x 64 weight gradient: m = 16 wm + g + 8 (e >> 1), n = 32 wn + 8 nt + 2 t + (e & 1)), one add per tile.
template <int OFF>
__device__ __forceinline__ void dw_mma(float (&acc)[FC_NACC], const float* G, const float* X, int wm, int wn, int lane) {
    const int g = lane >> 2, t = lane & 3;
    float part[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) part[nt][0] = part[nt][1] = part[nt][2] = part[nt][3] = 0.0f;
#pragma unroll
    for (int kb = 0; kb < 4; ++kb) {
        const float* gp = G + (16 * wm + g) * FC_RP + 16 * kb + 2 * t;
        const float2 v00 = *reinterpret_cast<const float2*>(gp), v10 = *reinterpret_cast<const float2*>(gp + 8 * FC_RP);
        const float2 v01 = *reinterpret_cast<const float2*>(gp + 8), v11 = *reinterpret_cast<const float2*>(gp + 8 * FC_RP + 8);
        uint32_t ah[4], al[4];
        l64_split(v00.x, v00.y, ah[0], al[0]);
        l64_split(v10.x, v10.y, ah[1], al[1]);
        l64_split(v01.x, v01.y, ah[2], al[2]);
        l64_split(v11.x, v11.y, ah[3], al[3]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const float* xp = X + (32 * wn + 8 * nt + g) * FC_RP + 16 * kb + 2 * t;
            const float2 b0 = *reinterpret_cast<const float2*>(xp), b1 = *reinterpret_cast<const float2*>(xp + 8);
            uint32_t bh0, bl0, bh1, bl1;
            l64_split(b0.x, b0.y, bh0, bl0);
            l64_split(b1.x, b1.y, bh1, bl1);
            l64_mma(part[nt], ah, bh0, bh1);
            l64_mma(part[nt], al, bh0, bh1);
            l64_mma(part[nt], ah, bl0, bl1);
        }
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[OFF + 4 * nt + e] += part[nt][e];
}

// acc[OFF + i NB + j] += sum over the tile's rows of G[m0 + i][r] X[n0 + nstep j][r]   (rows in order, FP32; the tile's
// partial is added to the running sum)
template <int OFF, int MB, int NB>
__device__ __forceinline__ void dw_acc(float (&acc)[FC_NACC], const float* G, int m0, const float* X, int n0, int nstep) {
    float part[MB * NB];
#pragma unroll
    for (int i = 0; i < MB * NB; ++i) part[i] = 0.0f;
#pragma unroll 1
    for (int r = 0; r < FC_R; r += 4) {
        float4 g[MB], x[NB];
#pragma unroll
        for (int i = 0; i < MB; ++i) g[i] = *reinterpret_cast<const float4*>(G + (m0 + i) * FC_RP + r);
#pragma unroll
        for (int j = 0; j < NB; ++j) x[j] = *reinterpret_cast<const float4*>(X + (n0 + nstep * j) * FC_RP + r);
#pragma unroll
        for (int i = 0; i < MB; ++i)
#pragma unroll
            for (int j = 0; j < NB; ++j) {
                float s = part[i * NB + j];
                s = fmaf(g[i].x, x[j].x, s);
                s = fmaf(g[i].y, x[j].y, s);
                s = fmaf(g[i].z, x[j].z, s);
                s = fmaf(g[i].w, x[j].w, s);
                part[i * NB + j] = s;
            }
    }
#pragma unroll
    for (int i = 0; i < MB * NB; ++i) acc[OFF + i] += part[i];
}

// Where accumulator k of thread tid belongs: offset into the encoder (enc = true) or decoder gradient, -1 for padding.
//   0..47   dV1, dV2, dV3   (dw_mma) warp w, lane l: m = 16 (w / 2) + l / 4 + 8 (e / 2), n = 32 (w % 2) + 8 nt + 2 (l % 4) + e % 2
//   48..55  dW1             m = 2 (tid / 16) + i, n = tid % 16 + 16 j
//   56..59  dW2             m = 2 (tid / 16) + i, n = tid % 16 + 16 j
//   60      dW3             m = tid / 32, n = tid % 32
//   61      bias            c1 | c2 | c3 | b1 | b2 by tid;  62: b3[tid]
__device__ int64_t acc_dst(int k, int tid, int K0, int Ld, const BfcLayout& LE, const BfcLayout& LD, bool& enc) {
    const int hi = tid >> 4, lo = tid & 15;
    enc = false;
    if (k < 48) {
        const int t = k >> 4, nt = (k >> 2) & 3, e = k & 3, w = tid >> 5, l = tid & 31;
        const int m = 16 * (w >> 1) + (l >> 2) + 8 * (e >> 1), n = 32 * (w & 1) + 8 * nt + 2 * (l & 3) + (e & 1);
        if (t == 0) return n < K0 + Ld ? LD.w1 + (int64_t)m * (K0 + Ld) + n : -1;
        if (t == 1) return LD.w2 + (int64_t)m * FC_DH + n;
        return m < K0 ? LD.w3 + (int64_t)m * FC_DH + n : -1;
    }
    if (k == 61 && tid < 3 * FC_DH) {
        const int t = tid >> 6, c = tid & 63;
        return t == 0 ? LD.b1 + c : t == 1 ? LD.b2 + c : (c < K0 ? LD.b3 + c : -1);
    }
    enc = true;
    if (k < 56) {
        const int i = (k - 48) >> 2, j = (k - 48) & 3, m = 2 * hi + i, n = lo + 16 * j;
        return n < K0 ? LE.w1 + (int64_t)m * K0 + n : -1;
    }
    if (k < 60) {
        const int i = (k - 56) >> 1, j = (k - 56) & 1, m = 2 * hi + i, n = lo + 16 * j;
        return LE.w2 + m * FC_E + n;
    }
    if (k == 60) {
        const int m = tid >> 5, n = tid & 31;
        return m < Ld ? LE.w3 + m * FC_E + n : -1;
    }
    if (k == 61) return tid < 3 * FC_DH + FC_E ? LE.b1 + tid - 3 * FC_DH : LE.b2 + tid - 3 * FC_DH - FC_E;
    return tid < Ld ? LE.b3 + tid : -1;
}

__global__ void __launch_bounds__(FC_THREADS, 1) beh_fc_learn_kernel(FcLearnArgs a) {
    extern __shared__ __align__(16) unsigned char fc_raw[];
    FcSmem& S = *reinterpret_cast<FcSmem*>(fc_raw);
    const int ag = blockIdx.y, tid = threadIdx.x;
    const int o = a.obs_dim, Wn = a.hist_len, Ld = a.latent_dim, K0 = Wn * o, N = a.n_slots, n_pos = a.n_pos;
    const int64_t row_step = (int64_t)N * o;                     // one time step of the history
    const BfcLayout LE = bfc_layout(K0, FC_E, Ld), LD = bfc_layout(K0 + Ld, FC_DH, K0);
    const float* __restrict__ PE = a.enc + ag * a.enc_stride;
    const float* __restrict__ PD = a.dec + ag * a.dec_stride;

    for (int idx = tid; idx < FC_KMAX * FC_E; idx += FC_THREADS) {
        const int k = idx / FC_E, n = idx % FC_E;
        S.w1t[k][n] = k < K0 ? PE[LE.w1 + n * K0 + k] : 0.0f;
    }
    for (int idx = tid; idx < FC_E * FC_E; idx += FC_THREADS) {
        const int k = idx / FC_E, n = idx % FC_E;
        S.w2t[k][n] = PE[LE.w2 + n * FC_E + k];
        S.w2[k][n] = PE[LE.w2 + k * FC_E + n];
    }
    for (int idx = tid; idx < FC_LMAX * FC_E; idx += FC_THREADS) {
        const int l = idx / FC_E, n = idx % FC_E;
        S.w3[l][n] = l < Ld ? PE[LE.w3 + l * FC_E + n] : 0.0f;
    }
    for (int idx = tid; idx < 5 * 8 * 4 * 32; idx += FC_THREADS) {
        const int l = idx & 31, kb = (idx >> 5) & 3, nt = (idx >> 7) & 7, which = idx >> 10;
        const int n = 8 * nt + (l >> 2), k0 = 16 * kb + 2 * (l & 3);
        auto bv = [&](int k) -> float {
            switch (which) {
                case VF_V1: return k < K0 + Ld ? PD[LD.w1 + n * (K0 + Ld) + k] : 0.0f;
                case VF_V2: return PD[LD.w2 + n * FC_DH + k];
                case VF_V3: return n < K0 ? PD[LD.w3 + n * FC_DH + k] : 0.0f;
                case VB_V3: return k < K0 ? PD[LD.w3 + k * FC_DH + n] : 0.0f;
                default: return PD[LD.w2 + k * FC_DH + n];
            }
        };
        uint32_t h0, l0, h1, l1;
        l64_split(bv(k0), bv(k0 + 1), h0, l0);
        l64_split(bv(k0 + 8), bv(k0 + 9), h1, l1);
        S.vf[which][0][nt][kb][l] = make_uint2(h0, h1);
        S.vf[which][1][nt][kb][l] = make_uint2(l0, l1);
    }
    for (int idx = tid; idx < FC_DH * FC_LMAX; idx += FC_THREADS) {
        const int n = idx / FC_LMAX, l = idx % FC_LMAX;
        S.v1lat[n][l] = l < Ld ? PD[LD.w1 + n * (K0 + Ld) + K0 + l] : 0.0f;
    }
    if (tid < FC_DH) {
        S.c1[tid] = PD[LD.b1 + tid];
        S.c2[tid] = PD[LD.b2 + tid];
        S.c3[tid] = tid < K0 ? PD[LD.b3 + tid] : 0.0f;
    }
    if (tid < FC_E) { S.b1[tid] = PE[LE.b1 + tid]; S.b2[tid] = PE[LE.b2 + tid]; }
    if (tid < FC_LMAX) S.b3[tid] = tid < Ld ? PE[LE.b3 + tid] : 0.0f;
    {   // activations: padding rows (features past K0 / K0 + L) stay zero for the whole launch
        float* act = &S.p[0][0];
        const int n_act = (int)(&S.ge3[0][0] + FC_LMAX * FC_RP - act);
        for (int i = tid; i < n_act; i += FC_THREADS) act[i] = 0.0f;
    }

    // thread maps of the products: tensor cores -> warp = 16 rows (or dW rows) x 32 outputs; FP32 32 outputs -> 4 outputs x 2 rows
    const int warp = tid >> 5, lane = tid & 31, wr = warp >> 1, wc = warp & 1, lg = lane >> 2, lt = lane & 3;
    const int n32 = 4 * (tid & 7), r32 = 2 * (tid >> 3);
    const int rq = tid >> 2, q = tid & 3, l0 = 2 * q, l1 = 2 * q + 1;      // four threads per row, two latent columns each

    float acc[FC_NACC];
#pragma unroll
    for (int k = 0; k < FC_NACC; ++k) acc[k] = 0.0f;
    float lsum = 0.0f, lcmp = 0.0f;
    const int64_t rows = (int64_t)a.n_eps * N * n_pos;
    const int64_t n_tiles = (rows + FC_R - 1) / FC_R;

    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        __syncthreads();                                          // the previous tile is done with rowoff / jpos / p / din
        if (tid < FC_R) {
            const int64_t qrow = tile * FC_R + tid;
            int j = -1;
            int64_t off = 0;
            if (qrow < rows) {
                const int64_t chain = qrow / n_pos;
                j = (int)(qrow - chain * n_pos);
                const int64_t b = chain / N, n = chain - b * N;
                off = (((int64_t)ag * a.n_eps + b) * a.n_steps) * row_step + n * o;
            }
            S.rowoff[tid] = off;
            S.jpos[tid] = j;
        }
        __syncthreads();
        for (int idx = tid; idx < K0 * FC_R; idx += FC_THREADS) {
            const int k = idx / FC_R, r = idx - k * FC_R;
            const int j = S.jpos[r], w = k / o, c = k - w * o;
            float vp = 0.0f, vc = 0.0f;
            if (j >= 0) {
                const int t = j - Wn + 1 + w;                     // row w of the window ending at j (rows < 0 are zeros)
                const float* base = a.hist + S.rowoff[r] + c;
                if (t >= 0) vc = __ldg(base + t * row_step);
                if (t >= 1) vp = __ldg(base + (t - 1) * row_step);
            }
            S.p[k][r] = vp;
            S.din[k][r] = vc;
        }
        __syncthreads();

        // ---- encoder on the window ending at j - 1 -> latent_{j-1} (rows with j = 0 use 0) ----
        {
            float y[4][2];
            rowmm(&S.w1t[0][0], FC_E, &S.p[0][0], K0, n32, r32, y);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int b = 0; b < 2; ++b) S.h1[n32 + i][r32 + b] = tanhf(y[i][b] + S.b1[n32 + i]);
        }
        __syncthreads();
        {
            float y[4][2];
            rowmm(&S.w2t[0][0], FC_E, &S.h1[0][0], FC_E, n32, r32, y);
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int b = 0; b < 2; ++b) S.h2[n32 + i][r32 + b] = tanhf(y[i][b] + S.b2[n32 + i]);
        }
        __syncthreads();
        {
            float z0 = S.b3[l0], z1 = S.b3[l1];
#pragma unroll 8
            for (int k = 0; k < FC_E; ++k) {
                const float h = S.h2[k][rq];
                z0 = fmaf(S.w3[l0][k], h, z0);
                z1 = fmaf(S.w3[l1][k], h, z1);
            }
            const float v0 = l0 < Ld ? z0 : -INFINITY, v1 = l1 < Ld ? z1 : -INFINITY;
            float mx = fmaxf(v0, v1);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float e0 = l0 < Ld ? expf(v0 - mx) : 0.0f, e1 = l1 < Ld ? expf(v1 - mx) : 0.0f;
            float den = e0 + e1;
            den += __shfl_xor_sync(0xffffffffu, den, 1);
            den += __shfl_xor_sync(0xffffffffu, den, 2);
            const bool live = S.jpos[rq] > 0;
            if (l0 < Ld) S.din[K0 + l0][rq] = live ? e0 / den : 0.0f;
            if (l1 < Ld) S.din[K0 + l1][rq] = live ? e1 / den : 0.0f;
        }
        __syncthreads();

        // ---- decoder on [window ending at j | latent_{j-1}] ----
        // y[nt][e] of a tensor-core product -> (output n, row r) of this thread
#define FC_EACH(...)                                                                             \
        _Pragma("unroll") for (int nt = 0; nt < 4; ++nt)                                          \
            _Pragma("unroll") for (int e = 0; e < 4; ++e) {                                       \
                const int n = 32 * wc + 8 * nt + 2 * lt + (e & 1), r = 16 * wr + lg + 8 * (e >> 1); \
                __VA_ARGS__                                                                      \
            }
        {
            float y[4][4];
            rowmma(S.vf[VF_V1], &S.din[0][0], wr, wc, lane, y);
            FC_EACH(S.d1[n][r] = tanhf(y[nt][e] + S.c1[n]);)
        }
        __syncthreads();
        {
            float y[4][4];
            rowmma(S.vf[VF_V2], &S.d1[0][0], wr, wc, lane, y);
            FC_EACH(S.d2[n][r] = tanhf(y[nt][e] + S.c2[n]);)
        }
        __syncthreads();
        {   // prediction, L1 error against the window ending at j + 1, d loss / d prediction / scale
            float y[4][4], lt_sum = 0.0f;
            rowmma(S.vf[VF_V3], &S.d2[0][0], wr, wc, lane, y);
            FC_EACH(
                const int j = S.jpos[r];
                float g = 0.0f;
                if (j >= 0 && n < K0) {
                    const int w = n / o, c = n - w * o, t = j - Wn + 2 + w;
                    const float nxt = t >= 0 ? __ldg(a.hist + S.rowoff[r] + t * row_step + c) : 0.0f;
                    const float err = nxt - (y[nt][e] + S.c3[n]);
                    lt_sum += fabsf(err);
                    g = err > 0.0f ? -1.0f : (err < 0.0f ? 1.0f : 0.0f);   // unscaled: sums of signs stay exact
                }
                S.g3[n][r] = g;)
            kadd(lsum, lcmp, lt_sum);
        }
        __syncthreads();

        // ---- backward ----
        dw_mma<32>(acc, &S.g3[0][0], &S.d2[0][0], wr, wc, lane);              // dV3 = G3^T D2
        __syncthreads();
        {
            float y[4][4];
            rowmma(S.vf[VB_V3], &S.g3[0][0], wr, wc, lane, y);                       // G2 = (G3 V3) (1 - d2^2), over d2
            FC_EACH(const float d = S.d2[n][r]; S.d2[n][r] = y[nt][e] * (1.0f - d * d);)
        }
        __syncthreads();
        dw_mma<16>(acc, &S.d2[0][0], &S.d1[0][0], wr, wc, lane);              // dV2 = G2^T D1
        __syncthreads();
        {
            float y[4][4];
            rowmma(S.vf[VB_V2], &S.d2[0][0], wr, wc, lane, y);                       // G1 = (G2 V2) (1 - d1^2), over d1
            FC_EACH(const float d = S.d1[n][r]; S.d1[n][r] = y[nt][e] * (1.0f - d * d);)
        }
#undef FC_EACH
        __syncthreads();
        dw_mma<0>(acc, &S.d1[0][0], &S.din[0][0], wr, wc, lane);              // dV1 = G1^T [x | z]
        {   // d loss / d latent_{j-1} = G1 V1[:, K0:], through the soft-max
            float g0 = 0.0f, g1 = 0.0f;
#pragma unroll 8
            for (int n = 0; n < FC_DH; ++n) {
                const float gv = S.d1[n][rq];
                g0 = fmaf(S.v1lat[n][l0], gv, g0);
                g1 = fmaf(S.v1lat[n][l1], gv, g1);
            }
            const float z0 = l0 < Ld ? S.din[K0 + l0][rq] : 0.0f, z1 = l1 < Ld ? S.din[K0 + l1][rq] : 0.0f;
            float s = z0 * g0 + z1 * g1;
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            const bool live = S.jpos[rq] > 0;
            S.ge3[l0][rq] = live ? z0 * (g0 - s) : 0.0f;
            S.ge3[l1][rq] = live ? z1 * (g1 - s) : 0.0f;
        }
        __syncthreads();
        dw_acc<60, 1, 1>(acc, &S.ge3[0][0], tid >> 5, &S.h2[0][0], tid & 31, 0);  // dW3 = GE3^T H2
        __syncthreads();
        {
            float y[4][2];
            rowmm(&S.w3[0][0], FC_E, &S.ge3[0][0], Ld, n32, r32, y);            // GE2 = (GE3 W3) (1 - h2^2), over h2
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int b = 0; b < 2; ++b) {
                    const float h = S.h2[n32 + i][r32 + b];
                    S.h2[n32 + i][r32 + b] = y[i][b] * (1.0f - h * h);
                }
        }
        __syncthreads();
        dw_acc<56, 2, 2>(acc, &S.h2[0][0], 2 * (tid >> 4), &S.h1[0][0], tid & 15, 16);   // dW2 = GE2^T H1
        __syncthreads();
        {
            float y[4][2];
            rowmm(&S.w2[0][0], FC_E, &S.h2[0][0], FC_E, n32, r32, y);           // GE1 = (GE2 W2) (1 - h1^2), over h1
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int b = 0; b < 2; ++b) {
                    const float h = S.h1[n32 + i][r32 + b];
                    S.h1[n32 + i][r32 + b] = y[i][b] * (1.0f - h * h);
                }
        }
        __syncthreads();
        dw_acc<48, 2, 4>(acc, &S.h1[0][0], 2 * (tid >> 4), &S.p[0][0], tid & 15, 16);    // dW1 = GE1^T X_{j-1}
        {   // bias gradients: row sums of G1 | G2 | G3 | GE1 | GE2 (one per thread) and GE3
            const float* src = tid < FC_DH ? S.d1[tid] : tid < 2 * FC_DH ? S.d2[tid - FC_DH] : tid < 3 * FC_DH ? S.g3[tid - 2 * FC_DH]
                             : tid < 3 * FC_DH + FC_E ? S.h1[tid - 3 * FC_DH] : S.h2[tid - 3 * FC_DH - FC_E];
            float s = 0.0f;
#pragma unroll 8
            for (int r = 0; r < FC_R; ++r) s += src[r];
            acc[61] += s;
            if (tid < FC_LMAX) {
                float s3 = 0.0f;
#pragma unroll 8
                for (int r = 0; r < FC_R; ++r) s3 += S.ge3[tid][r];
                acc[62] += s3;
            }
        }
    }

    // ---- this CTA's partial sums -> its slot; the last CTA of the agent-net adds the slots in CTA order ----
    constexpr int V = FC_NACC * FC_THREADS + 1;
    float* slot = a.part + ((int64_t)ag * gridDim.x + blockIdx.x) * V;
#pragma unroll
    for (int k = 0; k < FC_NACC; ++k) slot[k * FC_THREADS + tid] = acc[k];
    S.red[tid] = lsum - lcmp;
    __syncthreads();
    if (tid == 0) {
        float s = 0.0f;
        for (int i = 0; i < FC_THREADS; ++i) s += S.red[i];
        slot[FC_NACC * FC_THREADS] = s;
    }
    if (!det_last_arrival(a.count + ag, gridDim.x)) return;
    const float* slots = a.part + (int64_t)ag * gridDim.x * V;
    float* ge = a.g_enc + ag * a.enc_stride;
    float* gd = a.g_dec + ag * a.dec_stride;
#pragma unroll 1
    for (int k = 0; k < FC_NACC; ++k) {
        bool enc;
        const int64_t off = acc_dst(k, tid, K0, Ld, LE, LD, enc);
        if (off < 0) continue;
        float s = 0.0f;
        for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(slots + (int64_t)c * V + k * FC_THREADS + tid);
        (enc ? ge : gd)[off] += s * a.scale;
    }
    if (tid == 0) {
        float s = 0.0f;
        for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(slots + (int64_t)c * V + FC_NACC * FC_THREADS);
        a.b_loss[ag] += s * a.scale;
    }
}

// ---- rollout step: one warp per node, lane = hidden unit --------------------------------------------------------------
// Simple rather than fast: each node is a serial chain of K0 + 2E shuffle-FMAs, so at 512 envs the step reaches about
// 135 GB/s on its 28 MB of windows, far below the bandwidth it could use (several nodes per warp would close the gap).
constexpr int STEP_THREADS = 256, STEP_NODES_PER_WARP = 8;

struct FcStepArgs {
    const float* params; int64_t param_stride;
    iplan_view window; int64_t win_step; int win_pad;
    iplan_view lat;
    int n_envs, n_slots, obs_dim, latent_dim, hist_len;
};

__global__ void __launch_bounds__(STEP_THREADS) behavior_fc_step_kernel(FcStepArgs a) {
    __shared__ float w1t[FC_KMAX][FC_E], w2t[FC_E][FC_E], w3t[FC_E][FC_LMAX], bias[2 * FC_E + FC_LMAX];
    const int ag = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int o = a.obs_dim, Ld = a.latent_dim, K0 = a.hist_len * o, N = a.n_slots;
    const BfcLayout L = bfc_layout(K0, FC_E, Ld);
    const float* __restrict__ P = a.params + ag * a.param_stride;
    for (int idx = tid; idx < K0 * FC_E; idx += STEP_THREADS) { const int k = idx / FC_E, n = idx % FC_E; w1t[k][n] = P[L.w1 + n * K0 + k]; }
    for (int idx = tid; idx < FC_E * FC_E; idx += STEP_THREADS) { const int k = idx / FC_E, n = idx % FC_E; w2t[k][n] = P[L.w2 + n * FC_E + k]; }
    for (int idx = tid; idx < FC_E * FC_LMAX; idx += STEP_THREADS) {
        const int k = idx / FC_LMAX, l = idx % FC_LMAX;
        w3t[k][l] = l < Ld ? P[L.w3 + l * FC_E + k] : 0.0f;
    }
    if (tid < FC_E) { bias[tid] = P[L.b1 + tid]; bias[FC_E + tid] = P[L.b2 + tid]; }
    if (tid < FC_LMAX) bias[2 * FC_E + tid] = tid < Ld ? P[L.b3 + tid] : 0.0f;
    __syncthreads();

    const int total = a.n_envs * N;
    const int first = (blockIdx.x * (STEP_THREADS / 32) + warp) * STEP_NODES_PER_WARP;
    for (int nd = first; nd < min(first + STEP_NODES_PER_WARP, total); ++nd) {
        const int b = nd / N, n = nd - b * N;
        const float* src = a.window.ptr + ag * a.window.stride_agent + (int64_t)b * a.window.stride_env + (int64_t)n * a.window.stride_slot;
        float x[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = lane + 32 * u;
            float v = 0.0f;
            if (k < K0) {
                if (a.win_step == 0) v = src[k];
                else {
                    const int w = k / o, c = k - w * o;
                    v = w >= a.win_pad ? src[(int64_t)(w - a.win_pad) * a.win_step + c] : 0.0f;
                }
            }
            x[u] = v;
        }
        float h = bias[lane];
        for (int k = 0; k < K0; ++k) h = fmaf(w1t[k][lane], __shfl_sync(0xffffffffu, k < 32 ? x[0] : x[1], k & 31), h);
        const float h1 = tanhf(h);
        h = bias[FC_E + lane];
#pragma unroll 8
        for (int k = 0; k < FC_E; ++k) h = fmaf(w2t[k][lane], __shfl_sync(0xffffffffu, h1, k), h);
        const float h2 = tanhf(h);
        const int l = lane & (FC_LMAX - 1);
        float z = bias[2 * FC_E + l];
#pragma unroll 8
        for (int k = 0; k < FC_E; ++k) z = fmaf(w3t[k][l], __shfl_sync(0xffffffffu, h2, k), z);
        const float v = lane < Ld ? z : -INFINITY;
        const float mx = warp_max(v);
        const float e = lane < Ld ? expf(v - mx) : 0.0f;
        const float den = warp_sum(e);
        if (lane < Ld)
            a.lat.ptr[ag * a.lat.stride_agent + (int64_t)b * a.lat.stride_env + (int64_t)n * a.lat.stride_slot + lane] = e / den;
    }
}

int check_fc_shape(const char* what, int obs_dim, int latent_dim, int hist_len, int enc_hidden) {
    IPLAN_REQUIRE(enc_hidden == FC_E, "%s: enc_hidden %d != %d (Encoder_3FC is built for encoder_rnn_dim %d)", what, enc_hidden, FC_E, FC_E);
    IPLAN_REQUIRE(obs_dim >= 1, "%s: obs_dim %d < 1", what, obs_dim);
    IPLAN_REQUIRE(hist_len >= 1, "%s: hist_len %d < 1", what, hist_len);
    IPLAN_REQUIRE(latent_dim >= 1 && latent_dim <= FC_LMAX, "%s: latent_dim %d not in [1,%d]", what, latent_dim, FC_LMAX);
    IPLAN_REQUIRE((int64_t)hist_len * obs_dim + latent_dim <= FC_KMAX, "%s: hist_len*obs_dim+latent_dim %lld > %d", what,
                  (long long)hist_len * obs_dim + latent_dim, FC_KMAX);
    return 0;
}

}  // namespace
}  // namespace iplan

extern "C" int iplan_behavior_fc_step(const float* enc_params, int64_t param_stride,
                                      iplan_view window, int64_t win_stride_step, int win_pad, iplan_view lat_out,
                                      int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int hist_len, int enc_hidden,
                                      void* stream) {
    using namespace iplan;
    if (check_fc_shape("behavior_fc_step", obs_dim, latent_dim, hist_len, enc_hidden)) return -1;
    IPLAN_REQUIRE(win_pad >= 0 && win_pad < hist_len, "behavior_fc_step: win_pad %d not in [0,%d)", win_pad, hist_len);
    IPLAN_REQUIRE(n_envs > 0 && n_agents > 0 && n_agents <= 65535 && n_slots > 0 && (int64_t)n_envs * n_slots < (1ll << 30),
                  "behavior_fc_step: bad sizes (n_envs %d, n_agents %d, n_slots %d)", n_envs, n_agents, n_slots);
    IPLAN_REQUIRE(enc_params && window.ptr && lat_out.ptr, "behavior_fc_step: null pointer");
    FcStepArgs a;
    a.params = enc_params; a.param_stride = param_stride;
    a.window = window; a.win_step = win_stride_step; a.win_pad = win_stride_step ? win_pad : 0;
    a.lat = lat_out;
    a.n_envs = n_envs; a.n_slots = n_slots; a.obs_dim = obs_dim; a.latent_dim = latent_dim; a.hist_len = hist_len;
    const int per_cta = (STEP_THREADS / 32) * STEP_NODES_PER_WARP;
    dim3 grid((n_envs * n_slots + per_cta - 1) / per_cta, n_agents);
    behavior_fc_step_kernel<<<grid, STEP_THREADS, 0, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("behavior_fc_step");
}

extern "C" int iplan_beh_fc_learn(const float* enc_params, int64_t enc_stride, const float* dec_params, int64_t dec_stride,
                                  float* g_enc, float* g_dec, const float* hist, float scale, float* b_loss,
                                  int n_agents, int n_eps, int n_steps, int n_slots, int obs_dim, int latent_dim, int hist_len,
                                  int enc_hidden, int dec_hidden, void* stream) {
    using namespace iplan;
    if (check_fc_shape("beh_fc_learn", obs_dim, latent_dim, hist_len, enc_hidden)) return -1;
    IPLAN_REQUIRE(dec_hidden == FC_DH, "beh_fc_learn: dec_hidden %d != %d (Decoder_3FC is built for decoder_rnn_dim %d)",
                  dec_hidden, FC_DH, FC_DH);
    const int n_pos = n_steps - 1 - hist_len;
    IPLAN_REQUIRE(n_pos >= 1, "beh_fc_learn: n_pos = n_steps - 1 - hist_len = %d < 1 (episode of %d steps, windows of %d)",
                  n_pos, n_steps, hist_len);
    IPLAN_REQUIRE(n_eps > 0 && n_slots > 0 && n_agents > 0 && n_agents <= 65535, "beh_fc_learn: bad sizes (n_eps %d, n_slots %d, n_agents %d)",
                  n_eps, n_slots, n_agents);
    IPLAN_REQUIRE((int64_t)n_eps * n_slots * n_pos < (1ll << 40), "beh_fc_learn: too many rows");
    IPLAN_REQUIRE(enc_params && dec_params && g_enc && g_dec && hist && b_loss, "beh_fc_learn: null pointer");
    const int64_t rows = (int64_t)n_eps * n_slots * n_pos;
    const int64_t tiles = (rows + FC_R - 1) / FC_R;
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>(tiles, sm_count() / n_agents));
    const DetScratch ds = det_scratch((size_t)gx * n_agents * (FC_NACC * FC_THREADS + 1), n_agents);
    if (!ds.part) return -1;
    static bool configured = false;
    const size_t smem = sizeof(FcSmem);
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(beh_fc_learn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("beh_fc_learn: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    FcLearnArgs a;
    a.enc = enc_params; a.dec = dec_params; a.enc_stride = enc_stride; a.dec_stride = dec_stride;
    a.g_enc = g_enc; a.g_dec = g_dec; a.hist = hist; a.scale = scale; a.b_loss = b_loss;
    a.n_eps = n_eps; a.n_steps = n_steps; a.n_slots = n_slots; a.obs_dim = obs_dim; a.latent_dim = latent_dim;
    a.hist_len = hist_len; a.n_pos = n_pos; a.part = ds.part; a.count = ds.count;
    beh_fc_learn_kernel<<<dim3(gx, n_agents), FC_THREADS, smem, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("beh_fc_learn");
}
