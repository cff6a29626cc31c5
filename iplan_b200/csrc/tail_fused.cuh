// The 64-wide tail of the IPPO update as ONE kernel per epoch (train mode): everything between the fc1 output Z1 and
// its gradient dZ1 stays in registers of the warp that owns the rows.
//
//   forward   a1 = LN(ReLU(z1)); z2 = a1 W2^T + b2; a2 = LN(ReLU(z2)); GRU gates from a2 W_ih^T, h0 W_hh^T -> h1;
//             a3 = LN(h1); policy / value head                          (utils/mappo_utils/mlp.py:50-56, rnn.py:24-78,
//                                                                         act.py:81-85, modules/critics/ippo_critic.py:47-65)
//   loss      clipped-ratio policy loss - entropy bonus | clipped one-sided-Huber value loss
//                                                                        (learners/ippo_learner.py:128-159, :185-197)
//   backward  head -> LN3 -> GRU gates -> dGI, dGH -> dA2 = dGI W_ih -> LN2 -> dZ2 -> dA1 = dZ2 W2 -> LN1 -> dZ1
//
// It replaces ln_relu_fwd x2, lin64_rows x6, gru_head x2 and ln_relu_bwd x2 (12 launches whose 64 / 192-wide
// intermediates each made a round trip through HBM).  What leaves the kernel is what the weight-gradient products need
// (lin64_dw_kernel: dGI with a2, dGH with h0, dZ2 with a1) and dZ1 (scaled by the input LayerNorm's rstd) for the fc1
// backward.  The small gradients: bias gradients are column sums of dGI / dGH / dZ2 and are taken by the weight-gradient
// kernel that reads those arrays anyway; LayerNorm beta gradients follow from them linearly (colsum(dY W) = colsum(dY) W:
// tail_beta_kernel); what remains (LayerNorm gammas, head, the S / M sums of the fc1 backward) is reduced over the eight
// row groups of a warp with shuffles and added to global memory by four lanes (shared-memory float atomics are CAS
// loops on this architecture: the first version of this kernel spent most of its time spinning in them).
//
// One warp = 16 rows; 8 warps per CTA walk the row tiles of one (agent, net).  Every matrix product is
// mma.sync.m16n8k16 on f16 hi/lo splits (hi*hi + lo*hi + hi*lo, chains <= 12, fp32 adds between chains); the accumulator
// fragment of one product is the A fragment of the next (rows g / g+8 of a quad, columns 8 nt + 2 t, +1), so LayerNorm
// statistics are two quad shuffles and activations never move.  The weights live in shared memory as ready-made B
// fragments (hi and lo): W2, W_ih, W_hh for the forward products, W_ih and W2 again in the transposed fragment order for
// the two input-gradient products (176 KB), so a CTA owns an SM.  The gate pre-activations are recomputed in the
// backward sweep (576 MMAs per tile) rather than kept: 384 values per row do not fit in registers.
//
// Included by learner.cu inside namespace iplan, after RowBuf / NetParams / NetGrads / HeadArgs / huber_os.
#pragma once

constexpr int TF_THREADS = 256, TF_WARPS = 8;
constexpr int TF_NOUT = IPLAN_MAX_ACT;             // head rows kept (actor: n_actions <= 8; critic: 1)

struct TfFrag {                                    // B fragments {b0, b1} per (n-tile, k-block, lane), hi and lo
    uint2 w2f[2][8][4][32];                        // z2 = a1 W2^T          n-tile = out column block, k-block = in
    uint2 wihf[2][24][4][32];                      // gi = a2 W_ih^T
    uint2 whhf[2][24][4][32];                      // gh = h0 W_hh^T
    uint2 wihb[2][8][12][32];                      // dA2 = dGI W_ih        n-tile = a2 column block, k-block = gate block
    uint2 w2b[2][8][4][32];                        // dA1 = dZ2 W2
};
// parameter vectors (fp32) and the CTA's gradient accumulators
struct TfVec {
    float ln1_g[RH], ln1_b[RH], b2[RH], ln2_g[RH], ln2_b[RH], bih[RH3], bhh[RH3], ln3_g[RH], ln3_b[RH];
    float head_w[TF_NOUT][RH], head_b[TF_NOUT];
};
// warp-private gradient accumulators: the small gradients (LayerNorm gammas, head, S / M, loss sums) are summed over a warp's
// tiles here and added to global memory once, when the warp is done
constexpr int TF_SLOT_LN1 = 0, TF_SLOT_LN2 = 1, TF_SLOT_LN3 = 2, TF_SLOT_S = 3, TF_SLOT_M = 4, TF_SLOT_HEAD = 5;
constexpr int TF_SLOTS = TF_SLOT_HEAD + TF_NOUT;
constexpr int TF_WARPS_C = 8;
struct TfAcc {
    float v[TF_SLOTS][64];         // vectors over the 64 columns: lane l owns columns 2 l, 2 l + 1
    float s[3 + TF_NOUT][32];      // per-lane running sums of row scalars: loss | entropy | ratio | d head_b[l]
};
constexpr size_t TF_SMEM = sizeof(TfFrag) + sizeof(TfVec) + TF_WARPS_C * sizeof(TfAcc);
// one warp's flushed sums: the slot vectors, then the row scalars; a multiple of 4 floats keeps every record 16-byte aligned
constexpr int TF_REC = (TF_SLOTS * 64 + 3 + TF_NOUT + 3) & ~3;

struct TfArgs {
    HeadArgs h;                    // parameters, targets, loss constants (h.gi / h.gh = the dGI / dGH buffers)
    RowBuf z1, a1, z2, a2;         // Z1 in / dZ1 out (in place) | a1 out | dZ2 out | a2 out
    const float* stat;             // [A][rows][2] mean / rstd of the input LayerNorm
    float* SM;                     // [A][2][128]  S = colsum(dZ1), M = sum_r dZ1 rstd_r mu_r
    int64_t rows;
    float* part;                   // [2A][CTAs][TF_WARPS][TF_REC] the warps' sums, reduced in warp order (det_last_arrival)
    unsigned* count;               // [2A]
};

// gates with ex2.approx / rcp.approx (abs error ~1e-7, as in K1): sigmoid(x) = 1 / (1 + 2^(-x log2 e)), tanh(x) = 1 - 2 / (1 + 2^(2 x log2 e))
__device__ __forceinline__ float tf_ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float tf_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float tf_sigmoid(float x) { return tf_rcp(1.0f + tf_ex2(fminf(-1.4426950408889634f * x, 80.0f))); }
__device__ __forceinline__ float tf_tanh(float x) { return fmaf(-2.0f, tf_rcp(1.0f + tf_ex2(fminf(2.8853900817779268f * x, 80.0f))), 1.0f); }

__device__ __forceinline__ float tf_quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    return v;
}
// v[nt][j] = this thread's partial of column 8 nt + 2 t + j (t = lane & 3).  Sum over the warp's eight row groups g = lane >> 2
// as a reduce-scatter (14 shuffles for 16 columns: each exchange halves what a lane still carries), after which lane l holds
// the totals of columns 2 l and 2 l + 1, and add them to the warp's accumulator slot.
__device__ __forceinline__ void tf_red16(float* slot, int lane, const float (&v)[8][2]) {
    const bool g2 = lane & 16, g1 = lane & 8, g0 = lane & 4;
    float w[4][2], x[2][2], y[2];
#pragma unroll
    for (int n = 0; n < 4; ++n)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float send = g2 ? v[n][j] : v[n + 4][j], keep = g2 ? v[n + 4][j] : v[n][j];
            w[n][j] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
#pragma unroll
    for (int n = 0; n < 2; ++n)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const float send = g1 ? w[n][j] : w[n + 2][j], keep = g1 ? w[n + 2][j] : w[n][j];
            x[n][j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const float send = g0 ? x[0][j] : x[1][j], keep = g0 ? x[1][j] : x[0][j];
        y[j] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    float2* p = reinterpret_cast<float2*>(slot) + lane;          // column pair 8 g + 2 t = 2 lane
    float2 c = *p;
    c.x += y[0]; c.y += y[1];
    *p = c;
}

// A fragments (hi, lo) of k-block kb from a 16 x 64 accumulator-layout array
__device__ __forceinline__ void tf_afrag(const float (&x)[8][4], int kb, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    l64_split(x[2 * kb][0], x[2 * kb][1], hi[0], lo[0]);
    l64_split(x[2 * kb][2], x[2 * kb][3], hi[1], lo[1]);
    l64_split(x[2 * kb + 1][0], x[2 * kb + 1][1], hi[2], lo[2]);
    l64_split(x[2 * kb + 1][2], x[2 * kb + 1][3], hi[3], lo[3]);
}
__device__ __forceinline__ void tf_mma3(float (&d)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], uint2 bh, uint2 bl) {
    l64_mma(d, ah, bh.x, bh.y);
    l64_mma(d, al, bh.x, bh.y);
    l64_mma(d, ah, bl.x, bl.y);
}
// LayerNorm(ReLU(z)) of the two rows a thread holds a quarter of: x_hat, mean / rstd (per row), out = x_hat g + b
__device__ __forceinline__ void tf_ln_relu(const float (&z)[8][4], const float* __restrict__ gam, const float* __restrict__ bet, int t,
                                           float (&xh)[8][4], float (&out)[8][4], float (&rstd)[2]) {
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) { s0 += fmaxf(z[nt][0], 0.f) + fmaxf(z[nt][1], 0.f); s1 += fmaxf(z[nt][2], 0.f) + fmaxf(z[nt][3], 0.f); }
    const float m0 = tf_quad_sum(s0) * (1.0f / RH), m1 = tf_quad_sum(s1) * (1.0f / RH);
    float v0 = 0.f, v1 = 0.f;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        xh[nt][0] = fmaxf(z[nt][0], 0.f) - m0; xh[nt][1] = fmaxf(z[nt][1], 0.f) - m0;
        xh[nt][2] = fmaxf(z[nt][2], 0.f) - m1; xh[nt][3] = fmaxf(z[nt][3], 0.f) - m1;
        v0 = fmaf(xh[nt][0], xh[nt][0], v0); v0 = fmaf(xh[nt][1], xh[nt][1], v0);
        v1 = fmaf(xh[nt][2], xh[nt][2], v1); v1 = fmaf(xh[nt][3], xh[nt][3], v1);
    }
    rstd[0] = 1.0f / sqrtf(tf_quad_sum(v0) * (1.0f / RH) + LEPS);
    rstd[1] = 1.0f / sqrtf(tf_quad_sum(v1) * (1.0f / RH) + LEPS);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        const float2 g2 = *reinterpret_cast<const float2*>(gam + 8 * nt + 2 * t), b2 = *reinterpret_cast<const float2*>(bet + 8 * nt + 2 * t);
        xh[nt][0] *= rstd[0]; xh[nt][1] *= rstd[0]; xh[nt][2] *= rstd[1]; xh[nt][3] *= rstd[1];
        out[nt][0] = xh[nt][0] * g2.x + b2.x; out[nt][1] = xh[nt][1] * g2.y + b2.y;
        out[nt][2] = xh[nt][2] * g2.x + b2.x; out[nt][3] = xh[nt][3] * g2.y + b2.y;
    }
}
// backward of out = LN(ReLU(z)) g + b for the two rows: dz (in place of dy); column sums of dy x_hat (-> d gamma) and, if asked, of dz
// go to the warp's accumulator slots
__device__ __forceinline__ void tf_ln_relu_bwd(const float (&z)[8][4], const float (&xh)[8][4], const float (&rstd)[2],
                                               const float* __restrict__ gam, int t, int lane, float (&dy)[8][4],
                                               float* acc_gam, float* acc_colsum, bool live0, bool live1) {
    float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
    float dx[8][4];
    {
        float gv[8][2];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const float2 g2 = *reinterpret_cast<const float2*>(gam + 8 * nt + 2 * t);
            // rows past the end carry dy = 0 (live = false): they add nothing
            gv[nt][0] = dy[nt][0] * xh[nt][0] + dy[nt][2] * xh[nt][2];
            gv[nt][1] = dy[nt][1] * xh[nt][1] + dy[nt][3] * xh[nt][3];
            dx[nt][0] = dy[nt][0] * g2.x; dx[nt][1] = dy[nt][1] * g2.y; dx[nt][2] = dy[nt][2] * g2.x; dx[nt][3] = dy[nt][3] * g2.y;
            a0 += dx[nt][0] + dx[nt][1]; a1 += dx[nt][2] + dx[nt][3];
            c0 = fmaf(dx[nt][0], xh[nt][0], c0); c0 = fmaf(dx[nt][1], xh[nt][1], c0);
            c1 = fmaf(dx[nt][2], xh[nt][2], c1); c1 = fmaf(dx[nt][3], xh[nt][3], c1);
        }
        tf_red16(acc_gam, lane, gv);
    }
    const float m10 = tf_quad_sum(a0) * (1.0f / RH), m11 = tf_quad_sum(a1) * (1.0f / RH);
    const float m20 = tf_quad_sum(c0) * (1.0f / RH), m21 = tf_quad_sum(c1) * (1.0f / RH);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        dy[nt][0] = (live0 && z[nt][0] > 0.f) ? rstd[0] * (dx[nt][0] - m10 - xh[nt][0] * m20) : 0.f;
        dy[nt][1] = (live0 && z[nt][1] > 0.f) ? rstd[0] * (dx[nt][1] - m10 - xh[nt][1] * m20) : 0.f;
        dy[nt][2] = (live1 && z[nt][2] > 0.f) ? rstd[1] * (dx[nt][2] - m11 - xh[nt][2] * m21) : 0.f;
        dy[nt][3] = (live1 && z[nt][3] > 0.f) ? rstd[1] * (dx[nt][3] - m11 - xh[nt][3] * m21) : 0.f;
    }
    if (acc_colsum) {
        float cv[8][2];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) { cv[nt][0] = dy[nt][0] + dy[nt][2]; cv[nt][1] = dy[nt][1] + dy[nt][3]; }
        tf_red16(acc_colsum, lane, cv);
    }
}

// blockIdx.y = 2 * agent + net type (0 actor: NOUT >= n_actions head rows; 1 critic: one head row): actor and critic tiles
// run side by side so that one launch covers all SMs.  ONE body for both (only the loss section branches on the type):
// two instantiations of this much straight-line code would not stay in the instruction cache.
template <int NOUT>
__global__ void __launch_bounds__(TF_THREADS, 1) tail_fused_kernel(TfArgs A) {
    extern __shared__ __align__(16) unsigned char tf_raw[];
    const int a = blockIdx.y >> 1, type = blockIdx.y & 1;
    TfFrag& F = *reinterpret_cast<TfFrag*>(tf_raw);
    TfVec& V = *reinterpret_cast<TfVec*>(tf_raw + sizeof(TfFrag));
    const HeadArgs& h = A.h;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    static_assert(TF_WARPS == TF_WARPS_C, "accumulator count");
    TfAcc& ACC = reinterpret_cast<TfAcc*>(tf_raw + sizeof(TfFrag) + sizeof(TfVec))[warp];
    for (int i = lane; i < (int)(sizeof(TfAcc) / sizeof(float)); i += 32) reinterpret_cast<float*>(&ACC)[i] = 0.0f;
    const int g = lane >> 2, t = lane & 3;
    const float* __restrict__ p = h.P.net(a, type);
    const TrunkLayout L = trunk_layout(h.F, type == 0 ? h.n_actions : 1, type == 1);
    const int n_out = type == 0 ? h.n_actions : 1;

    // ---- stage the weights as B fragments: b0 = (k = 16 kb + 2t, +1 ; n = 8 nt + g), b1 = the same at k + 8 -----------------
    auto frag = [&](float w00, float w01, float w10, float w11, uint2& hi, uint2& lo) {
        l64_split(w00, w01, hi.x, lo.x);
        l64_split(w10, w11, hi.y, lo.y);
    };
    for (int idx = tid; idx < 8 * 4 * 32; idx += TF_THREADS) {             // W2 forward: B[k = in][n = out] = W2[out][in]
        const int l = idx & 31, kb = (idx >> 5) & 3, nt = idx >> 7, gg = l >> 2, tt = l & 3;
        const float* w = p + L.fc2_w + (8 * nt + gg) * RH + 16 * kb + 2 * tt;
        frag(w[0], w[1], w[8], w[9], F.w2f[0][nt][kb][l], F.w2f[1][nt][kb][l]);
    }
    for (int idx = tid; idx < 2 * 24 * 4 * 32; idx += TF_THREADS) {        // W_ih, W_hh forward
        const int l = idx & 31, kb = (idx >> 5) & 3, nt = (idx >> 7) % 24, m = idx / (24 * 128), gg = l >> 2, tt = l & 3;
        const float* w = p + (m ? L.whh : L.wih) + (8 * nt + gg) * RH + 16 * kb + 2 * tt;
        uint2(*dst)[24][4][32] = m ? F.whhf : F.wihf;
        frag(w[0], w[1], w[8], w[9], dst[0][nt][kb][l], dst[1][nt][kb][l]);
    }
    for (int idx = tid; idx < 8 * 12 * 32; idx += TF_THREADS) {            // W_ih backward: B[k = gate][n = a2 column] = W_ih[gate][column]
        const int l = idx & 31, kb = (idx >> 5) % 12, nt = idx / (12 * 32), gg = l >> 2, tt = l & 3;
        const float* w = p + L.wih + (16 * kb + 2 * tt) * RH + 8 * nt + gg;
        frag(w[0], w[RH], w[8 * RH], w[9 * RH], F.wihb[0][nt][kb][l], F.wihb[1][nt][kb][l]);
    }
    for (int idx = tid; idx < 8 * 4 * 32; idx += TF_THREADS) {             // W2 backward
        const int l = idx & 31, kb = (idx >> 5) & 3, nt = idx >> 7, gg = l >> 2, tt = l & 3;
        const float* w = p + L.fc2_w + (16 * kb + 2 * tt) * RH + 8 * nt + gg;
        frag(w[0], w[RH], w[8 * RH], w[9 * RH], F.w2b[0][nt][kb][l], F.w2b[1][nt][kb][l]);
    }
    for (int c = tid; c < RH; c += TF_THREADS) {
        V.ln1_g[c] = p[L.ln1_w + c]; V.ln1_b[c] = p[L.ln1_b + c]; V.b2[c] = p[L.fc2_b + c];
        V.ln2_g[c] = p[L.ln2_w + c]; V.ln2_b[c] = p[L.ln2_b + c]; V.ln3_g[c] = p[L.ln3_w + c]; V.ln3_b[c] = p[L.ln3_b + c];
    }
    for (int c = tid; c < RH3; c += TF_THREADS) { V.bih[c] = p[L.bih + c]; V.bhh[c] = p[L.bhh + c]; }
    for (int idx = tid; idx < TF_NOUT * RH; idx += TF_THREADS) {
        const int l = idx / RH, c = idx - l * RH;
        V.head_w[l][c] = l < n_out ? p[L.head_w + l * RH + c] : 0.0f;
    }
    if (tid < TF_NOUT) V.head_b[tid] = tid < n_out ? p[L.head_b + tid] : 0.0f;
    __syncthreads();

    const float nrm_mean = h.norm[a * 4], nrm_istd = h.norm[a * 4 + 1], inv_msum = h.norm[a * 4 + 2], inv_rows = h.norm[a * 4 + 3];
    const int64_t rows = A.rows;
    const int64_t n_tiles = (rows + 15) / 16;
    const float* h0base = (type == 0 ? h.h0a : h.h0c) + a * h.h0_sa;
    float* gg = h.G.net(a, type);                                           // this net's gradient buffer
    float* smS = A.SM + (a * 2 + 0) * 128 + type * 64;
    float* smM = A.SM + (a * 2 + 1) * 128 + type * 64;

    for (int64_t tile = (int64_t)blockIdx.x * TF_WARPS + warp; tile < n_tiles; tile += (int64_t)gridDim.x * TF_WARPS) {
        const int64_t r0 = tile * 16 + g, r1 = r0 + 8;
        const bool live0 = r0 < rows, live1 = r1 < rows;
        const int64_t q0 = live0 ? r0 : rows - 1, q1 = live1 ? r1 : rows - 1;
        float* z1p0 = A.z1.row(a, type, q0);
        float* z1p1 = A.z1.row(a, type, q1);

        // ---- forward -----------------------------------------------------------------------------------------
        float act[8][4];
        {
            float z[8][4], xh[8][4], rs1[2];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float2 v0 = *reinterpret_cast<const float2*>(z1p0 + 8 * nt + 2 * t), v1 = *reinterpret_cast<const float2*>(z1p1 + 8 * nt + 2 * t);
                z[nt][0] = v0.x; z[nt][1] = v0.y; z[nt][2] = v1.x; z[nt][3] = v1.y;
            }
            tf_ln_relu(z, V.ln1_g, V.ln1_b, t, xh, act, rs1);              // act = a1
        }
        {
            float* o0 = A.a1.row(a, type, q0);
            float* o1 = A.a1.row(a, type, q1);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                if (live0) *reinterpret_cast<float2*>(o0 + 8 * nt + 2 * t) = make_float2(act[nt][0], act[nt][1]);
                if (live1) *reinterpret_cast<float2*>(o1 + 8 * nt + 2 * t) = make_float2(act[nt][2], act[nt][3]);
            }
        }
        float z2[8][4];
        {
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) tf_afrag(act, kb, ah[kb], al[kb]);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) tf_mma3(d, ah[kb], al[kb], F.w2f[0][nt][kb][lane], F.w2f[1][nt][kb][lane]);
                const float2 b = *reinterpret_cast<const float2*>(V.b2 + 8 * nt + 2 * t);
                z2[nt][0] = d[0] + b.x; z2[nt][1] = d[1] + b.y; z2[nt][2] = d[2] + b.x; z2[nt][3] = d[3] + b.y;
            }
        }
        {
            float xh2[8][4], rs2[2];
            tf_ln_relu(z2, V.ln2_g, V.ln2_b, t, xh2, act, rs2);            // act = a2
        }
        {
            float* o0 = A.a2.row(a, type, q0);
            float* o1 = A.a2.row(a, type, q1);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                if (live0) *reinterpret_cast<float2*>(o0 + 8 * nt + 2 * t) = make_float2(act[nt][0], act[nt][1]);
                if (live1) *reinterpret_cast<float2*>(o1 + 8 * nt + 2 * t) = make_float2(act[nt][2], act[nt][3]);
            }
        }
        // operand fragments of the gate products: a2 and h0 (kept for the backward sweep's recomputation)
        uint32_t a2h[4][4], a2l[4][4], h0h[4][4], h0l[4][4];
        float h0v[8][4];
        {
            const float* hp0 = h0base + q0 * h.h0_ld;
            const float* hp1 = h0base + q1 * h.h0_ld;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float2 v0 = *reinterpret_cast<const float2*>(hp0 + 8 * nt + 2 * t), v1 = *reinterpret_cast<const float2*>(hp1 + 8 * nt + 2 * t);
                h0v[nt][0] = v0.x; h0v[nt][1] = v0.y; h0v[nt][2] = v1.x; h0v[nt][3] = v1.y;
            }
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) { tf_afrag(act, kb, a2h[kb], a2l[kb]); tf_afrag(h0v, kb, h0h[kb], h0l[kb]); }
        }
        // gate pre-activations of hidden-unit tile ut (8 units): gi / gh for r | z | n, biases added
        auto gates = [&](int ut, float (&rg)[4], float (&zg)[4], float (&ng)[4], float (&ghn)[4]) {
            float gi[3][4], gh[3][4];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const int nt = 8 * q + ut;
                gi[q][0] = gi[q][1] = gi[q][2] = gi[q][3] = 0.f;
                gh[q][0] = gh[q][1] = gh[q][2] = gh[q][3] = 0.f;
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) {
                    tf_mma3(gi[q], a2h[kb], a2l[kb], F.wihf[0][nt][kb][lane], F.wihf[1][nt][kb][lane]);
                    tf_mma3(gh[q], h0h[kb], h0l[kb], F.whhf[0][nt][kb][lane], F.whhf[1][nt][kb][lane]);
                }
                const float2 bi = *reinterpret_cast<const float2*>(V.bih + 8 * nt + 2 * t), bh = *reinterpret_cast<const float2*>(V.bhh + 8 * nt + 2 * t);
                gi[q][0] += bi.x; gi[q][1] += bi.y; gi[q][2] += bi.x; gi[q][3] += bi.y;
                gh[q][0] += bh.x; gh[q][1] += bh.y; gh[q][2] += bh.x; gh[q][3] += bh.y;
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                rg[e] = tf_sigmoid(gi[0][e] + gh[0][e]);
                zg[e] = tf_sigmoid(gi[1][e] + gh[1][e]);
                ghn[e] = gh[2][e];
                ng[e] = tf_tanh(gi[2][e] + rg[e] * ghn[e]);
            }
        };
        float h1[8][4];
        // rolled (the body is ~300 instructions; unrolled, the kernel outgrows the instruction cache): the register arrays
        // are indexed by the loop counter through compare-and-select, never through local memory
#pragma unroll 1
        for (int ut = 0; ut < 8; ++ut) {
            float rg[4], zg[4], ng[4], ghn[4];
            gates(ut, rg, zg, ng, ghn);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float h0e = 0.f;
#pragma unroll
                for (int u2 = 0; u2 < 8; ++u2) h0e = u2 == ut ? h0v[u2][e] : h0e;
                const float v = (1.0f - zg[e]) * ng[e] + zg[e] * h0e;
#pragma unroll
                for (int u2 = 0; u2 < 8; ++u2) h1[u2][e] = u2 == ut ? v : h1[u2][e];
            }
        }
        // LN3 (no ReLU) and the head
        float xh3[8][4], a3[8][4], rs3[2];
        {
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) { s0 += h1[nt][0] + h1[nt][1]; s1 += h1[nt][2] + h1[nt][3]; }
            const float m0 = tf_quad_sum(s0) * (1.0f / RH), m1 = tf_quad_sum(s1) * (1.0f / RH);
            float v0 = 0.f, v1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                xh3[nt][0] = h1[nt][0] - m0; xh3[nt][1] = h1[nt][1] - m0; xh3[nt][2] = h1[nt][2] - m1; xh3[nt][3] = h1[nt][3] - m1;
                v0 = fmaf(xh3[nt][0], xh3[nt][0], v0); v0 = fmaf(xh3[nt][1], xh3[nt][1], v0);
                v1 = fmaf(xh3[nt][2], xh3[nt][2], v1); v1 = fmaf(xh3[nt][3], xh3[nt][3], v1);
            }
            rs3[0] = 1.0f / sqrtf(tf_quad_sum(v0) * (1.0f / RH) + LEPS);
            rs3[1] = 1.0f / sqrtf(tf_quad_sum(v1) * (1.0f / RH) + LEPS);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float2 g2 = *reinterpret_cast<const float2*>(V.ln3_g + 8 * nt + 2 * t), b2 = *reinterpret_cast<const float2*>(V.ln3_b + 8 * nt + 2 * t);
                xh3[nt][0] *= rs3[0]; xh3[nt][1] *= rs3[0]; xh3[nt][2] *= rs3[1]; xh3[nt][3] *= rs3[1];
                a3[nt][0] = xh3[nt][0] * g2.x + b2.x; a3[nt][1] = xh3[nt][1] * g2.y + b2.y;
                a3[nt][2] = xh3[nt][2] * g2.x + b2.x; a3[nt][3] = xh3[nt][3] * g2.y + b2.y;
            }
        }
        float out0[NOUT], out1[NOUT];                                 // head outputs of the thread's two rows (quad-uniform)
#pragma unroll
        for (int l = 0; l < NOUT; ++l) {
            float d0 = 0.f, d1 = 0.f;
            if (l < n_out) {
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    const float2 w = *reinterpret_cast<const float2*>(&V.head_w[l][8 * nt + 2 * t]);
                    d0 = fmaf(w.x, a3[nt][0], d0); d0 = fmaf(w.y, a3[nt][1], d0);
                    d1 = fmaf(w.x, a3[nt][2], d1); d1 = fmaf(w.y, a3[nt][3], d1);
                }
                out0[l] = tf_quad_sum(d0) + V.head_b[l];
                out1[l] = tf_quad_sum(d1) + V.head_b[l];
            } else {
                out0[l] = out1[l] = -INFINITY;
            }
        }
        // ---- losses and d loss / d head outputs, per row (all four lanes of a quad compute the same numbers) -------------
        float dl0[NOUT], dl1[NOUT];
        float st_loss = 0.f, st_ent = 0.f, st_ratio = 0.f;
        auto row_loss = [&](int64_t r, bool live, float (&outv)[NOUT], float (&dl)[NOUT]) {
#pragma unroll
            for (int l = 0; l < NOUT; ++l) dl[l] = 0.0f;
            const int b = (int)(r / h.T1), tt = (int)(r - (int64_t)b * h.T1);
            const bool train_row = live && tt < h.T1 - 1 && b < h.n_train_eps;
            const int64_t ridx = (int64_t)a * h.rows + r;
            if (type == 0) {
                const int nA = h.n_actions;
                const int actn = h.actions[ridx];
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
                    if (l == actn) lp_a = lpl[l];
                }
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
                    const float g_ent = -h.ent_coef * inv_rows * h.gscale;
#pragma unroll
                    for (int l = 0; l < NOUT; ++l)
                        if (l < nA && !masked[l])
                            dl[l] = g_lp * ((l == actn ? 1.0f : 0.0f) - pl[l]) + g_ent * (-pl[l] * (lpl[l] + ent));
                    st_loss += -fminf(s1_, s2_) * m * inv_msum;
                    st_ent += ent * inv_rows;
                    st_ratio += ratio * inv_rows;
                }
            } else {
                const float v = outv[0];
                if (train_row) {
                    const float m = h.alive[ridx];
                    const float vo = h.old_value[ridx], ret = h.returns[ridx];
                    const float diff = v - vo;
                    const float vc = vo + fminf(fmaxf(diff, -h.clip), h.clip);
                    const float eo = ret - v, ec = ret - vc;
                    const float lo = huber_os(eo, h.huber_delta), lc = huber_os(ec, h.huber_delta);
                    const bool inside = diff >= -h.clip && diff <= h.clip;
                    const float go = -huber_os_grad(eo, h.huber_delta);
                    const float gc = inside ? -huber_os_grad(ec, h.huber_delta) : 0.0f;
                    const float gg = lo > lc ? go : (lc > lo ? gc : 0.5f * (go + gc));
                    dl[0] = h.v_coef * m * inv_msum * gg * h.gscale;
                    st_loss += fmaxf(lo, lc) * m * inv_msum;
                }
            }
        };
        row_loss(q0, live0, out0, dl0);
        row_loss(q1, live1, out1, dl1);
        {   // per-row scalars (the four lanes of a quad hold the same numbers): per-lane running sums, reduced when the warp is done
            ACC.s[0][lane] += st_loss;                                      // policy | value loss
            if (type == 0) { ACC.s[1][lane] += st_ent; ACC.s[2][lane] += st_ratio; }
#pragma unroll
            for (int l = 0; l < NOUT; ++l) if (l < n_out) ACC.s[3 + l][lane] += dl0[l] + dl1[l];
        }
        // ---- backward: head, LN3 -> dh1 ------------------------------------------------------------------------------
        float dh[8][4];
        {
            float dA[8][4];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) { dA[nt][0] = dA[nt][1] = dA[nt][2] = dA[nt][3] = 0.f; }
#pragma unroll
            for (int l = 0; l < NOUT; ++l) {
                if (l < n_out) {
                    float hv[8][2];
#pragma unroll
                    for (int nt = 0; nt < 8; ++nt) {
                        const float2 w = *reinterpret_cast<const float2*>(&V.head_w[l][8 * nt + 2 * t]);
                        dA[nt][0] = fmaf(dl0[l], w.x, dA[nt][0]); dA[nt][1] = fmaf(dl0[l], w.y, dA[nt][1]);
                        dA[nt][2] = fmaf(dl1[l], w.x, dA[nt][2]); dA[nt][3] = fmaf(dl1[l], w.y, dA[nt][3]);
                        hv[nt][0] = dl0[l] * a3[nt][0] + dl1[l] * a3[nt][2];
                        hv[nt][1] = dl0[l] * a3[nt][1] + dl1[l] * a3[nt][3];
                    }
                    tf_red16(ACC.v[TF_SLOT_HEAD + l], lane, hv);
                }
            }
            float a0 = 0.f, a1 = 0.f, c0 = 0.f, c1 = 0.f;
            {
                float gv[8][2];
#pragma unroll
                for (int nt = 0; nt < 8; ++nt) {
                    gv[nt][0] = dA[nt][0] * xh3[nt][0] + dA[nt][2] * xh3[nt][2];
                    gv[nt][1] = dA[nt][1] * xh3[nt][1] + dA[nt][3] * xh3[nt][3];
                }
                tf_red16(ACC.v[TF_SLOT_LN3], lane, gv);
            }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int c = 8 * nt + 2 * t;
                const float2 g2 = *reinterpret_cast<const float2*>(V.ln3_g + c);
                dA[nt][0] *= g2.x; dA[nt][1] *= g2.y; dA[nt][2] *= g2.x; dA[nt][3] *= g2.y;
                a0 += dA[nt][0] + dA[nt][1]; a1 += dA[nt][2] + dA[nt][3];
                c0 = fmaf(dA[nt][0], xh3[nt][0], c0); c0 = fmaf(dA[nt][1], xh3[nt][1], c0);
                c1 = fmaf(dA[nt][2], xh3[nt][2], c1); c1 = fmaf(dA[nt][3], xh3[nt][3], c1);
            }
            const float m10 = tf_quad_sum(a0) * (1.0f / RH), m11 = tf_quad_sum(a1) * (1.0f / RH);
            const float m20 = tf_quad_sum(c0) * (1.0f / RH), m21 = tf_quad_sum(c1) * (1.0f / RH);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                dh[nt][0] = rs3[0] * (dA[nt][0] - m10 - xh3[nt][0] * m20); dh[nt][1] = rs3[0] * (dA[nt][1] - m10 - xh3[nt][1] * m20);
                dh[nt][2] = rs3[1] * (dA[nt][2] - m11 - xh3[nt][2] * m21); dh[nt][3] = rs3[1] * (dA[nt][3] - m11 - xh3[nt][3] * m21);
            }
        }
        // ---- backward through the GRU gates (recomputed), dGI / dGH out, dA2 = dGI W_ih ---------------------------------
        float da2[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) da2[nt][0] = da2[nt][1] = da2[nt][2] = da2[nt][3] = 0.f;
        float* gi0 = h.gi.row(a, type, q0);
        float* gi1 = h.gi.row(a, type, q1);
        float* gh0 = h.gh.row(a, type, q0);
        float* gh1 = h.gh.row(a, type, q1);
#pragma unroll 1
        for (int up = 0; up < 4; ++up) {                                    // 16 hidden units = one k-block of each gate
            float dgi[3][2][4];                                             // [gate][unit tile of the pair][e]
#pragma unroll
            for (int w2 = 0; w2 < 2; ++w2) {
                const int ut = 2 * up + w2;
                float rg[4], zg[4], ng[4], ghn[4];
                gates(ut, rg, zg, ng, ghn);
                float dghn[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float dhe = 0.f, h0e = 0.f;
#pragma unroll
                    for (int u2 = 0; u2 < 8; ++u2) { dhe = u2 == ut ? dh[u2][e] : dhe; h0e = u2 == ut ? h0v[u2][e] : h0e; }
                    const float dn = dhe * (1.0f - zg[e]);
                    const float dz = dhe * (h0e - ng[e]);
                    const float dan = dn * (1.0f - ng[e] * ng[e]);
                    const float dr = dan * ghn[e];
                    dgi[0][w2][e] = dr * rg[e] * (1.0f - rg[e]);
                    dgi[1][w2][e] = dz * zg[e] * (1.0f - zg[e]);
                    dgi[2][w2][e] = dan;
                    dghn[e] = dan * rg[e];
                }
                const int c = 8 * ut + 2 * t;
#pragma unroll
                for (int q = 0; q < 3; ++q) {
                    if (live0) {
                        *reinterpret_cast<float2*>(gi0 + q * RH + c) = make_float2(dgi[q][w2][0], dgi[q][w2][1]);
                        *reinterpret_cast<float2*>(gh0 + q * RH + c) = q < 2 ? make_float2(dgi[q][w2][0], dgi[q][w2][1]) : make_float2(dghn[0], dghn[1]);
                    }
                    if (live1) {
                        *reinterpret_cast<float2*>(gi1 + q * RH + c) = make_float2(dgi[q][w2][2], dgi[q][w2][3]);
                        *reinterpret_cast<float2*>(gh1 + q * RH + c) = q < 2 ? make_float2(dgi[q][w2][2], dgi[q][w2][3]) : make_float2(dghn[2], dghn[3]);
                    }
                }
            }
            // dA2 += dGI[:, this k-block of each gate] . W_ih   (three k-blocks: a chain of 9 per n-tile, then an fp32 add)
            uint32_t dh_[3][4], dl_[3][4];
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                l64_split(dgi[q][0][0], dgi[q][0][1], dh_[q][0], dl_[q][0]);
                l64_split(dgi[q][0][2], dgi[q][0][3], dh_[q][1], dl_[q][1]);
                l64_split(dgi[q][1][0], dgi[q][1][1], dh_[q][2], dl_[q][2]);
                l64_split(dgi[q][1][2], dgi[q][1][3], dh_[q][3], dl_[q][3]);
            }
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int q = 0; q < 3; ++q) tf_mma3(d, dh_[q], dl_[q], F.wihb[0][nt][4 * q + up][lane], F.wihb[1][nt][4 * q + up][lane]);
                da2[nt][0] += d[0]; da2[nt][1] += d[1]; da2[nt][2] += d[2]; da2[nt][3] += d[3];
            }
        }
        // ---- LN2 backward -> dZ2 (out), dA1 = dZ2 W2, LN1 backward -> dZ1 (scaled by the input LayerNorm's rstd, out) -------
        {
            float xh2[8][4], tmp[8][4], rs2[2];                             // x_hat of LN2 again (cheaper than keeping 32 registers alive)
            tf_ln_relu(z2, V.ln2_g, V.ln2_b, t, xh2, tmp, rs2);
            tf_ln_relu_bwd(z2, xh2, rs2, V.ln2_g, t, lane, da2, ACC.v[TF_SLOT_LN2], nullptr, live0, live1);   // da2 = dZ2 now
        }
        {
            float* o0 = A.z2.row(a, type, q0);
            float* o1 = A.z2.row(a, type, q1);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                if (live0) *reinterpret_cast<float2*>(o0 + 8 * nt + 2 * t) = make_float2(da2[nt][0], da2[nt][1]);
                if (live1) *reinterpret_cast<float2*>(o1 + 8 * nt + 2 * t) = make_float2(da2[nt][2], da2[nt][3]);
            }
        }
        float da1[8][4];
        {
            uint32_t ah[4][4], al[4][4];
#pragma unroll
            for (int kb = 0; kb < 4; ++kb) tf_afrag(da2, kb, ah[kb], al[kb]);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int kb = 0; kb < 4; ++kb) tf_mma3(d, ah[kb], al[kb], F.w2b[0][nt][kb][lane], F.w2b[1][nt][kb][lane]);
                da1[nt][0] = d[0]; da1[nt][1] = d[1]; da1[nt][2] = d[2]; da1[nt][3] = d[3];
            }
        }
        {
            float z[8][4], xh[8][4], tmp[8][4], rs1[2];                     // z1 again (still untouched in global memory) and its LN
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const float2 v0 = *reinterpret_cast<const float2*>(z1p0 + 8 * nt + 2 * t), v1 = *reinterpret_cast<const float2*>(z1p1 + 8 * nt + 2 * t);
                z[nt][0] = v0.x; z[nt][1] = v0.y; z[nt][2] = v1.x; z[nt][3] = v1.y;
            }
            tf_ln_relu(z, V.ln1_g, V.ln1_b, t, xh, tmp, rs1);
            tf_ln_relu_bwd(z, xh, rs1, V.ln1_g, t, lane, da1, ACC.v[TF_SLOT_LN1], ACC.v[TF_SLOT_S], live0, live1);  // da1 = dZ1 now; S = colsum
        }
        {
            const float mu0 = A.stat[(a * rows + q0) * 2], rs0 = A.stat[(a * rows + q0) * 2 + 1];
            const float mu1 = A.stat[(a * rows + q1) * 2], rs1_ = A.stat[(a * rows + q1) * 2 + 1];
            float mv[8][2];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int c = 8 * nt + 2 * t;
                const float v00 = da1[nt][0] * rs0, v01 = da1[nt][1] * rs0, v10 = da1[nt][2] * rs1_, v11 = da1[nt][3] * rs1_;
                mv[nt][0] = v00 * mu0 + v10 * mu1;
                mv[nt][1] = v01 * mu0 + v11 * mu1;
                if (live0) *reinterpret_cast<float2*>(z1p0 + c) = make_float2(v00, v01);
                if (live1) *reinterpret_cast<float2*>(z1p1 + c) = make_float2(v10, v11);
            }
            tf_red16(ACC.v[TF_SLOT_M], lane, mv);
        }
    }
    // ---- the warp's accumulated small gradients -> its record; the net's last CTA adds the records in warp order -------------
    __syncwarp();
    const int64_t n_rec = (int64_t)gridDim.x * TF_WARPS;
    float* rec = A.part + ((int64_t)blockIdx.y * n_rec + (int64_t)blockIdx.x * TF_WARPS + warp) * TF_REC;
    for (int sl = 0; sl < TF_SLOTS; ++sl)
        *reinterpret_cast<float2*>(rec + 64 * sl + 2 * lane) = reinterpret_cast<const float2*>(ACC.v[sl])[lane];
    for (int k = 0; k < 3 + TF_NOUT; ++k) {
        float v = t == 0 ? ACC.s[k][lane] : 0.0f;                           // one lane per quad: the four hold the same sums
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (lane == 0) rec[TF_SLOTS * 64 + k] = v;
    }
    if (!det_last_arrival(A.count + blockIdx.y, gridDim.x)) return;
    const float* recs = A.part + (int64_t)blockIdx.y * n_rec * TF_REC;
    for (int idx = threadIdx.x; idx < TF_REC; idx += TF_THREADS) {
        float* dst;
        float* dst2 = nullptr;
        if (idx < TF_SLOTS * 64) {
            const int sl = idx >> 6, c = idx & 63;
            if (sl >= TF_SLOT_HEAD + n_out) continue;
            dst = sl == TF_SLOT_LN1 ? gg + L.ln1_w + c : sl == TF_SLOT_LN2 ? gg + L.ln2_w + c : sl == TF_SLOT_LN3 ? gg + L.ln3_w + c
                : sl == TF_SLOT_S ? gg + L.fc1_b + c : sl == TF_SLOT_M ? smM + c : gg + L.head_w + (sl - TF_SLOT_HEAD) * RH + c;
            if (sl == TF_SLOT_S) dst2 = smS + c;                            // S = colsum(dZ1) is also the fc1 bias gradient
        } else {
            const int k = idx - TF_SLOTS * 64;                              // loss | entropy | ratio | d head_b[l]
            if (k == 0) dst = &h.stats[a * 8 + (type == 0 ? 0 : 1)];
            else if (k < 3) { if (type != 0) continue; dst = &h.stats[a * 8 + 1 + k]; }
            else { if (k - 3 >= n_out) continue; dst = &gg[L.head_b + k - 3]; }
        }
        float v = 0.0f;
        for (int64_t r = 0; r < n_rec; ++r) v += __ldcg(recs + r * TF_REC + idx);
        *dst += v;
        if (dst2) *dst2 += v;
    }
}

// LayerNorm beta gradients and the rest of the gate-bias bookkeeping, from the column sums the weight-gradient kernels
// left in the bias slots:  d beta2 = (d b_ih) W_ih,  d beta1 = (d b2) W2,  d beta3 = (d head_b) W_head   (colsum(dY W) = colsum(dY) W).
// One CTA per (agent, net); 64 threads.
__global__ void tail_beta_kernel(NetParams P, NetGrads G, int F, int n_actions) {
    const int a = blockIdx.x >> 1, type = blockIdx.x & 1, c = threadIdx.x;
    const float* p = P.net(a, type);
    float* g = G.net(a, type);
    const int n_out = type == 0 ? n_actions : 1;
    const TrunkLayout L = trunk_layout(F, n_out, type == 1);
    float b2 = 0.f, b1 = 0.f, b3 = 0.f;
    for (int k = 0; k < RH3; ++k) b2 = fmaf(g[L.bih + k], p[L.wih + k * RH + c], b2);
    for (int k = 0; k < RH; ++k) b1 = fmaf(g[L.fc2_b + k], p[L.fc2_w + k * RH + c], b1);
    for (int k = 0; k < n_out; ++k) b3 = fmaf(g[L.head_b + k], p[L.head_w + k * RH + c], b3);
    g[L.ln2_b + c] = b2;
    g[L.ln1_b + c] = b1;
    g[L.ln3_b + c] = b3;
}
