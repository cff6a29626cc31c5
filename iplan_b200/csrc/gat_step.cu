// K1 — fused GAT step for one timestep of the rollout.
//
// Replaces Prediction_policy.GAT_latent_update (reference nova/prediction_policy.py:92-118)
// and, inside it, GAT_Net.forward (nova/GAT_Net.py:41-142).  One CTA owns one
// (env b, agent-net a) pair per kernel and keeps every intermediate in shared memory:
//
//   x[n]      = [history_t[n] | behaviour_{t-1}[n]]                       (:102-105)
//   enc[n]    = ReLU(W_e x[n] + b_e)                                       (:50)
//   hard attention: for ego i, a bidirectional GRU runs over the N-1 neighbours
//     j(i,s) = s < i ? s : s+1 with input [enc_i ; enc_j], h0 = 0          (:57-83)
//     -> factored input projection  W_ih[enc_i;enc_j] = P[i] + Q[j]  (SURVEY App. A)
//     -> logits(i,s) = W_he [h_fwd ; h_rev] + b_he, gumbel-softmax tau      (:85-95)
//        only softmax(.)[1] is used, i.e. sigmoid((l1-l0 + g1-g0)/tau)
//   soft attention: softmax_s(q_i . k_j / sqrt(D)), v = ReLU(W_v enc + b)   (:99-129)
//   x_i = sum_s soft * hard * v_j (no renormalisation)                      (:132)
//   out = GRUCell(x_i, h_prev_i)                                            (:140)
//
// The work is the 2N GRU chains of length N-1 (91 % of the FLOPs).  They run on the tensor
// cores: a warp advances 16 chains (egos) of one direction per step as ONE 16x96x32 product
// h . W_hh^T with mma.sync.m16n8k16 (f16 inputs, f32 accumulate).  fp32 accuracy is kept by
// splitting both operands into f16 hi + lo parts and issuing hi*hi + lo*hi + hi*lo (the
// dropped lo*lo term is < 2^-22 relative).  The accumulator fragment of step s is, element
// for element, the A fragment of step s+1, so the hidden state never leaves registers.
//
// Two kernels per step, both on the caller's stream:
//   gat_recur_kernel   grid (B, A, 2 directions), 4 warps: encode, P/Q projections of its
//                      direction, the N chains of that direction; writes the per-edge logit
//                      difference dl[dir][s][i] to a scratch buffer (L2 resident, 27 KB per (b,a)).
//                      56 KB smem, 126 registers -> 4 CTAs (16 warps) per SM, and CTAs in
//                      different phases overlap on an SM.  Gate math on packed fp32 pairs
//                      (FADD2 / FMUL2 / FFMA2), four sigmoid denominators per rcp.approx.
//   gat_attend_kernel  grid (B, A), 8 warps: encode, q|k|v, scores and aggregation as MMA
//                      products around a warp-per-ego soft-max x gumbel gate, GRUCell.
//
// HBM traffic per (b,a): read N*(o+L+32) floats, write N*32 floats; weights (28.8k floats)
// and the dl scratch come from L2.
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "gat_common.cuh"

namespace iplan {

__host__ __device__ inline size_t rec_smem_floats(int N) {
    // s_P | s_Q | union { s_x, s_enc  (prologue) ; W_hh fragments, b_hn, logit weights (recurrence) }
    const size_t pro = (size_t)N * IN_MAX + (size_t)H * IN_MAX + (size_t)N * H, rec = 4 * NT_G * KB_H * 32 + 64 + 32;
    return (size_t)N * PP + (size_t)N * G3 + (pro > rec ? pro : rec);
}
constexpr int QKP = 72;         // row pitch of the q|k buffer: q at columns 0..31, k at columns KOFF..KOFF+31
constexpr int KOFF = 36;        //   (8-byte aligned, (72 g + 2 t) mod 32 distinct over a half-warp: conflict-free fragment reads)
constexpr int WP = 64 + 8;      // attention-weight / V^T row pitch: K = 64 neighbour columns, zero padded
__host__ __device__ inline size_t att_smem_floats(int N) {
    // s_vt (aliases s_x, s_we) | s_enc | s_xa | s_hp | s_gh | region { s_qk, s_dl, s_w }  (s_gi aliases the region)
    // The score product (phase 5a) reads k rows up to the next multiple of 8 past N - 1, so the region holds at least
    // that many q|k rows; below N = 4 this is more than s_qk + s_dl + s_w.
    const size_t region = (size_t)N * QKP + (size_t)N * (N - 1) + (size_t)N * WP;
    const size_t qk_pad = (size_t)((N + 7) & ~7) * QKP;
    const size_t gru = (size_t)N * G3;
    const size_t big = region > qk_pad ? region : qk_pad;
    return (size_t)H * WP + 3 * (size_t)N * H + (size_t)N * G3 + (big > gru ? big : gru);
}

// volatile: the W_hh fragments are loop-invariant, and hoisting them out of the step loop would cost
// 96 registers per thread
__device__ __forceinline__ uint4 lds128(const uint4* p) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "r"((uint32_t)__cvta_generic_to_shared(p)));
    return v;
}

// D = A(16x16, row) * B(16x8, col) + C, f16 x f16 -> f32
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1, const float (&c)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
                 : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(c[3]));
}

// out[n][c] = act( sum_{k<16 KB} in[n][k] * Wg[c*ldw + k] + bias[c] )  for n < N, c < cols (cols % 8 == 0)
// `in` / `out` in shared memory (row pitch ldin / ldout floats), W and bias in global OR shared memory.
// All warps of the CTA cooperate: one task = one 16-node x 8-column tile = 3 KB MMAs (f16 hi/lo
// split, see header).  W is read as B fragments: a quad reads 32 contiguous bytes of one weight row, so
// every sector fetched is fully used.  TRANS_OUT stores out[c][n] instead (row pitch ldout).
struct EpiNone { __device__ __forceinline__ float operator()(int, float v) const { return v; } };

struct StoreNone {};            // default: out[r][c] (or out[c][r] with TRANS_OUT)

template <int NW, int KB = KB_H, bool TRANS_OUT = false, class Epi = EpiNone, class Store = StoreNone>
__device__ __forceinline__ void dense32_mma(const float* in, int ldin, int N, const float* __restrict__ Wg, int ldw,
                                            const float* __restrict__ bias, int cols, float* out, int ldout, bool relu,
                                            int warp, int lane, Epi epi = Epi(), Store store = Store()) {
    const int gq = lane >> 2, tq = lane & 3;
    const int mtiles = (N + 15) >> 4, ntiles = cols >> 3;
    const int mh = (mtiles + 1) >> 1;                 // a task = one n-tile x one half of the m-tiles
    const int ntask = ntiles * 2;
    constexpr int DT = KB == 1 ? 4 : (KB == 2 ? 6 : 1);   // tasks whose weight fragments are fetched together
    for (int base = warp; base < ntask; base += NW * DT) {
        float2 wv[DT][2 * KB];
#pragma unroll
        for (int i = 0; i < DT; ++i) {                // issue every load first: one L2 round trip
            const int task = base + i * NW;
            if (task < ntask) {
                const float* wr = Wg + (size_t)(8 * (task >> 1) + gq) * ldw + 2 * tq;
#pragma unroll
                for (int q = 0; q < 2 * KB; ++q) wv[i][q] = *reinterpret_cast<const float2*>(wr + 8 * q);
            }
        }
#pragma unroll
        for (int i = 0; i < DT; ++i) {
            const int task = base + i * NW;
            if (task >= ntask) break;
            const int nt = task >> 1, half = task & 1;
            const int c0 = 8 * nt + 2 * tq;
            const float b0 = bias ? bias[c0] : 0.0f, b1 = bias ? bias[c0 + 1] : 0.0f;
            uint32_t bh[KB][2], bl[KB][2];
#pragma unroll
            for (int kb = 0; kb < KB; ++kb) {
                split_f16(wv[i][2 * kb].x, wv[i][2 * kb].y, bh[kb][0], bl[kb][0]);
                split_f16(wv[i][2 * kb + 1].x, wv[i][2 * kb + 1].y, bh[kb][1], bl[kb][1]);
            }
            const int mt_end = min(mtiles, (half + 1) * mh);
            for (int mt = half * mh; mt < mt_end; ++mt) {
                const int r0 = mt * 16 + gq, r1 = r0 + 8;
                const float* x0 = in + min(r0, N - 1) * ldin + 2 * tq;
                const float* x1 = in + min(r1, N - 1) * ldin + 2 * tq;
                float acc[4] = {b0, b1, b0, b1};
#pragma unroll
                for (int kb = 0; kb < KB; ++kb) {      // <= 12 MMAs per accumulator chain (KB <= 4)
                    uint32_t ahi[4], alo[4];
                    const float2 v00 = *reinterpret_cast<const float2*>(x0 + 16 * kb);
                    const float2 v10 = *reinterpret_cast<const float2*>(x1 + 16 * kb);
                    const float2 v01 = *reinterpret_cast<const float2*>(x0 + 16 * kb + 8);
                    const float2 v11 = *reinterpret_cast<const float2*>(x1 + 16 * kb + 8);
                    split_f16(v00.x, v00.y, ahi[0], alo[0]);
                    split_f16(v10.x, v10.y, ahi[1], alo[1]);
                    split_f16(v01.x, v01.y, ahi[2], alo[2]);
                    split_f16(v11.x, v11.y, ahi[3], alo[3]);
                    mma16816(acc, ahi, bh[kb][0], bh[kb][1], acc);
                    mma16816(acc, alo, bh[kb][0], bh[kb][1], acc);
                    mma16816(acc, ahi, bl[kb][0], bl[kb][1], acc);
                }
                if (relu) { acc[0] = fmaxf(acc[0], 0.f); acc[1] = fmaxf(acc[1], 0.f); acc[2] = fmaxf(acc[2], 0.f); acc[3] = fmaxf(acc[3], 0.f); }
                acc[0] = epi(c0, acc[0]); acc[1] = epi(c0 + 1, acc[1]); acc[2] = epi(c0, acc[2]); acc[3] = epi(c0 + 1, acc[3]);
                if constexpr (!std::is_same<Store, StoreNone>::value) {       // caller-defined placement: store(row, col, value)
                    if (r0 < N) { store(r0, c0, acc[0]); store(r0, c0 + 1, acc[1]); }
                    if (r1 < N) { store(r1, c0, acc[2]); store(r1, c0 + 1, acc[3]); }
                } else if (TRANS_OUT) {
                    if (r0 < N) { out[c0 * ldout + r0] = acc[0]; out[(c0 + 1) * ldout + r0] = acc[1]; }
                    if (r1 < N) { out[c0 * ldout + r1] = acc[2]; out[(c0 + 1) * ldout + r1] = acc[3]; }
                } else {
                    if (r0 < N) { out[r0 * ldout + c0] = acc[0]; out[r0 * ldout + c0 + 1] = acc[1]; }
                    if (r1 < N) { out[r1 * ldout + c0] = acc[2]; out[r1 * ldout + c0 + 1] = acc[3]; }
                }
            }
        }
    }
}

// phases 0 + 1, shared by both kernels: gather x = [history | behaviour latent] (zero padded to IN_MAX columns),
// enc = ReLU(W_e x + b_e) as one N x 32 x 16 tensor-core product.  s_we: [H][IN_MAX] staging of W_e (zero padded).
template <int NT>
__device__ __forceinline__ void gat_encode(const GatArgs& a, const float* __restrict__ W, const GatLayout& L,
                                           int b, int ag, float* s_x, float* s_we, float* s_enc) {
    const int N = a.n_slots, in_dim = a.obs_dim + a.latent_dim, tid = threadIdx.x;
    const float* hist = a.hist.ptr + ag * a.hist.stride_agent + b * a.hist.stride_env;
    const float* beh = a.beh.ptr + ag * a.beh.stride_agent + b * a.beh.stride_env;
    for (int idx = tid; idx < N * IN_MAX; idx += NT) {
        const int n = idx / IN_MAX, c = idx - n * IN_MAX;
        float v = 0.0f;
        if (c < a.obs_dim) v = hist[n * a.hist.stride_slot + c];
        else if (c < in_dim) v = beh[n * a.beh.stride_slot + (c - a.obs_dim)];
        s_x[idx] = v;
    }
    for (int idx = tid; idx < H * IN_MAX; idx += NT) {
        const int c = idx / IN_MAX, k = idx - c * IN_MAX;
        s_we[idx] = k < in_dim ? W[L.enc_w + c * in_dim + k] : 0.0f;
    }
    __syncthreads();
    dense32_mma<NT / 32, 1>(s_x, IN_MAX, N, s_we, IN_MAX, W + L.enc_b, H, s_enc, H, true, tid >> 5, tid & 31);
    __syncthreads();
}

// ---- kernel 1 of 2: the N GRU chains of one direction for one (env, agent-net) -------------
__global__ void __launch_bounds__(REC_THREADS, 4) gat_recur_kernel(GatArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int b = blockIdx.x, ag = blockIdx.y, dir = blockIdx.z;
    const int N = a.n_slots, NM1 = N - 1;
    const int in_dim = a.obs_dim + a.latent_dim;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* __restrict__ W = a.params + (int64_t)ag * a.param_stride;
    const GatLayout L = gat_layout(in_dim);

    float* s_P = smem;                                  // [N][PP]  ego part + b_ih (+ b_hh for r|z), gate-scaled
    float* s_Q = s_P + N * PP;                          // [N][96]  neighbour part, gate-scaled
    float* s_x = s_Q + N * G3;                          // [N][IN_MAX]   } prologue only; the W_hh fragments below
    float* s_we = s_x + N * IN_MAX;                     // [H][IN_MAX]   } take their place for the recurrence
    float* s_enc = s_we + H * IN_MAX;                   // [N][H]        }
    uint4* s_w4 = reinterpret_cast<uint4*>(s_Q + N * G3);   // [12][2][32] W_hh B fragments {hi0, hi1, lo0, lo1}
    float4* s_bn = reinterpret_cast<float4*>(s_w4 + NT_G * KB_H * 32);   // [4 t4][4 tq] b_hn pair twice = the n tile's initial accumulator
    float2* s_lw = reinterpret_cast<float2*>(s_bn + 16);                 // [4 t4][4 tq] logit-difference weight pair

    gat_encode<REC_THREADS>(a, W, L, b, ag, s_x, s_we, s_enc);

    // ---- phase 2: factored input projections P (ego, + b_ih) and Q (neighbour) ------
    const float* wih = W + (dir ? L.wih_r : L.wih_f);
    const float* bhh = W + (dir ? L.bhh_r : L.bhh_f);
    // the gate-activation scale (and b_hh of r|z) is folded into P and Q as they are produced
    auto epi_p = [bhh](int c, float v) { return c < 2 * H ? K_RZ * (v + bhh[c]) : K_N * v; };
    auto epi_q = [](int c, float v) { return (c < 2 * H ? K_RZ : K_N) * v; };
    dense32_mma<REC_WARPS, KB_H, false>(s_enc, H, N, wih, 2 * H, W + (dir ? L.bih_r : L.bih_f), G3, s_P, PP, false, warp, lane, epi_p);
    dense32_mma<REC_WARPS, KB_H, false>(s_enc, H, N, wih + H, 2 * H, nullptr, G3, s_Q, G3, false, warp, lane, epi_q);
    __syncthreads();                                    // s_enc is dead from here: its space takes the W_hh fragments
    // W_hh B fragments (mma.m16n8k16 "col" operand: b0 = (k=2t,2t+1 ; n=g), b1 = (k=2t+8,2t+9 ; n=g)),
    // B[k][n] = W_hh[gate n][hidden k], gate-activation scale folded in, f16 hi and lo parts.
    {
        const float* whh = W + (dir ? L.whh_r : L.whh_f);
        for (int idx = tid; idx < NT_G * KB_H * 32; idx += REC_THREADS) {
            const int ln = idx & 31, kb = (idx >> 5) & 1, nt = idx >> 6;
            const float* wr = whh + (8 * nt + (ln >> 2)) * H + 16 * kb + 2 * (ln & 3);
            const float2 w0 = *reinterpret_cast<const float2*>(wr);
            const float2 w1 = *reinterpret_cast<const float2*>(wr + 8);
            const float ks = nt < 8 ? K_RZ : K_N;
            uint4 f;
            split_f16(ks * w0.x, ks * w0.y, f.x, f.z);
            split_f16(ks * w1.x, ks * w1.y, f.y, f.w);
            s_w4[idx] = f;
        }
        if (tid < 16) {
            const int c = 8 * (tid >> 2) + 2 * (tid & 3);
            const float b0 = K_N * bhh[2 * H + c], b1 = K_N * bhh[2 * H + c + 1];
            s_bn[tid] = make_float4(b0, b1, b0, b1);
            s_lw[tid] = make_float2(W[L.he_w + 2 * H + dir * H + c] - W[L.he_w + dir * H + c],
                                    W[L.he_w + 2 * H + dir * H + c + 1] - W[L.he_w + dir * H + c + 1]);
        }
    }
    __syncthreads();
    // ---- phase 3: the chains on the tensor cores; warp = m-tile of 16 egos -----------
    const int gq = lane >> 2, tq = lane & 3, mt = warp;
    if (mt * 16 >= N) return;                                           // warp-uniform; no barrier follows
    const int row0 = mt * 16 + gq, row1 = row0 + 8;                     // ego indices of this thread's two rows
    const bool ok0 = row0 < N, ok1 = row1 < N;
    const int i0 = ok0 ? row0 : N - 1, i1 = ok1 ? row1 : N - 1;
    float* dl = a.dl + ((((int64_t)ag * a.n_envs + b) * 2 + dir) * NM1) * DLP;
    const uint4* w4 = s_w4 + lane;
    // per-chain constants in accumulator-fragment layout: element e of tile nt is
    // (row e<2 ? row0 : row1, col 8*nt + 2*tq + (e&1))
    // per-chain constants (ego part of the input projection) stay in shared memory: element e of tile nt is
    // (row e<2 ? row0 : row1, col 8*nt + 2*tq + (e&1)); reading them per step keeps the kernel at 128 registers
    // (4 CTAs = 16 warps per SM)
    const float* p0row = s_P + i0 * PP + 2 * tq;
    const float* p1row = s_P + i1 * PP + 2 * tq;
    // hidden state: h01[t4] = (row0; cols 8 t4 + 2 tq, +1), h23[t4] = the same columns of row1
    f32x2 h01[4], h23[4];
#pragma unroll
    for (int t4 = 0; t4 < 4; ++t4) h01[t4] = h23[t4] = pk2(0.0f, 0.0f);
    const f32x2 one2 = pk2(1.0f, 1.0f), mtwo2 = pk2(-2.0f, -2.0f);

    for (int step = 0; step < NM1; ++step) {
        const int s = dir ? NM1 - 1 - step : step;
        // A fragments from the hidden state (accumulator layout == A layout, see header)
        uint32_t ahi[KB_H][4], alo[KB_H][4];
#pragma unroll
        for (int kb = 0; kb < KB_H; ++kb) {
            split_f16p(h01[2 * kb], ahi[kb][0], alo[kb][0]);          // row g,   k low
            split_f16p(h23[2 * kb], ahi[kb][1], alo[kb][1]);          // row g+8, k low
            split_f16p(h01[2 * kb + 1], ahi[kb][2], alo[kb][2]);      // row g,   k high
            split_f16p(h23[2 * kb + 1], ahi[kb][3], alo[kb][3]);      // row g+8, k high
        }
        // neighbour of ego i at position s is j = s < i ? s : s + 1
        const float* q0 = s_Q + (s < i0 ? s : s + 1) * G3 + 2 * tq;
        const float* q1 = s_Q + (s < i1 ? s : s + 1) * G3 + 2 * tq;
        f32x2 pl01 = pk2(0.0f, 0.0f), pl23 = pl01;
        // Hidden units in groups of 8 (t4): the r|z|n tiles of a group take their six MMA
        // passes (three independent chains), then the group's gate math runs while the
        // next group's MMAs are in flight, so tensor, MUFU and FP32 pipes overlap within one warp.
#pragma unroll
        for (int t4 = 0; t4 < 4; ++t4) {
            float acc[3][4];
            uint4 w[3][KB_H];
            const float4 bn = s_bn[4 * t4 + tq];
#pragma unroll
            for (int gi = 0; gi < 3; ++gi)
#pragma unroll
                for (int kb = 0; kb < KB_H; ++kb) w[gi][kb] = lds128(w4 + ((4 * gi + t4) * KB_H + kb) * 32);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) {
                float c0[4];
                if (gi < 2) {
                    const int nt = 4 * gi + t4;
                    const float2 c01 = *reinterpret_cast<const float2*>(p0row + 8 * nt);
                    const float2 c23 = *reinterpret_cast<const float2*>(p1row + 8 * nt);
                    c0[0] = c01.x; c0[1] = c01.y; c0[2] = c23.x; c0[3] = c23.y;
                }
                else { c0[0] = bn.x; c0[1] = bn.y; c0[2] = bn.z; c0[3] = bn.w; }
                mma16816(acc[gi], ahi[0], w[gi][0].x, w[gi][0].y, c0);
            }
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) mma16816(acc[gi], ahi[1], w[gi][1].x, w[gi][1].y, acc[gi]);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) mma16816(acc[gi], alo[0], w[gi][0].x, w[gi][0].y, acc[gi]);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) mma16816(acc[gi], alo[1], w[gi][1].x, w[gi][1].y, acc[gi]);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) mma16816(acc[gi], ahi[0], w[gi][0].z, w[gi][0].w, acc[gi]);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) mma16816(acc[gi], ahi[1], w[gi][1].z, w[gi][1].w, acc[gi]);
            // gates on (col, col+1) pairs; four reciprocals per rcp.approx (rcp4)
            f32x2 r01, r23, z01, z23, i01, i23;
            sigmoid4_den(add2(pk2(acc[0][0], acc[0][1]), lds64(q0 + 8 * t4)),
                         add2(pk2(acc[0][2], acc[0][3]), lds64(q1 + 8 * t4)), r01, r23);      // r = 1 / (1 + 2^x')
            sigmoid4_den(add2(pk2(acc[1][0], acc[1][1]), lds64(q0 + H + 8 * t4)),
                         add2(pk2(acc[1][2], acc[1][3]), lds64(q1 + H + 8 * t4)), z01, z23);
            sigmoid4_den(fma2(r01, pk2(acc[2][0], acc[2][1]), add2(lds64(p0row + 2 * H + 8 * t4), lds64(q0 + 2 * H + 8 * t4))),
                         fma2(r23, pk2(acc[2][2], acc[2][3]), add2(lds64(p1row + 2 * H + 8 * t4), lds64(q1 + 2 * H + 8 * t4))), i01, i23);
            const f32x2 n01 = fma2(mtwo2, i01, one2), n23 = fma2(mtwo2, i23, one2);   // tanh = 1 - 2 / (1 + 2^x')
            h01[t4] = fma2(z01, sub2(h01[t4], n01), n01);                   // (1 - z) n + z h
            h23[t4] = fma2(z23, sub2(h23[t4], n23), n23);
            const f32x2 lw = lds64(reinterpret_cast<const float*>(s_lw + 4 * t4 + tq));
            pl01 = fma2(lw, h01[t4], pl01);
            pl23 = fma2(lw, h23[t4], pl23);
        }
        // the 32 hidden units of a row live in the 4 lanes of a quad
        float pa, pb;
        upk2(pl01, pa, pb);
        float pl0 = pa + pb;
        upk2(pl23, pa, pb);
        float pl1 = pa + pb;
        pl0 += __shfl_xor_sync(0xffffffffu, pl0, 1); pl0 += __shfl_xor_sync(0xffffffffu, pl0, 2);
        pl1 += __shfl_xor_sync(0xffffffffu, pl1, 1); pl1 += __shfl_xor_sync(0xffffffffu, pl1, 2);
        if (tq == 0) {                                      // dl[s][i]: a warp's 16 egos are one 64-byte segment
            if (ok0) dl[s * DLP + i0] = pl0;
            if (ok1) dl[s * DLP + i1] = pl1;
        }
    }
}

// ---- kernel 2 of 2: q/k/v, hard x soft attention, GRUCell ------------------------------------
__global__ void __launch_bounds__(GAT_THREADS, 2) gat_attend_kernel(GatArgs a) {
    extern __shared__ __align__(16) float smem[];
    const int b = blockIdx.x, ag = blockIdx.y;
    const int N = a.n_slots, NM1 = N - 1;
    const int in_dim = a.obs_dim + a.latent_dim;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* __restrict__ W = a.params + (int64_t)ag * a.param_stride;
    const GatLayout L = gat_layout(in_dim);

    float* s_vt = smem;                                 // [H][WP]  V^T: s_vt[c][j] = v_j[c], columns >= N zero
    float* s_x = smem;                                  // [N][IN_MAX] (dead after the encode; (N+H)*IN_MAX <= H*WP)
    float* s_we = s_x + N * IN_MAX;                     // [H][IN_MAX]  likewise
    float* s_enc = s_vt + H * WP;                       // [N][H]
    float* s_xa = s_enc + N * H;                        // [N][H] aggregated messages
    float* s_hp = s_xa + N * H;                         // [N][H] h_prev
    float* s_gh = s_hp + N * H;                         // [N][96] GRUCell hidden pre-activations
    float* s_qk = s_gh + N * G3;                        // [N][QKP] q | k
    float* s_dl = s_qk + N * QKP;                       // [N][N-1] logit difference, both directions summed
    float* s_w = s_dl + N * NM1;                        // [N][WP] scores, then attention weights over ALL slots j (self = 0)
    float* s_gi = s_qk;                                 // [N][96] GRUCell input pre-activations  (q, k, dl, w are dead by then)

    const float* hprev = a.hprev.ptr + ag * a.hprev.stride_agent + b * a.hprev.stride_env;
    float* outp = a.out.ptr + ag * a.out.stride_agent + b * a.out.stride_env;

    // ---- everything that only depends on the kernel's inputs is fetched first, so its L2 latency overlaps the encode:
    //      h_prev (cp.async) and the recurrence kernel's dl[dir][s][i] (summed over the two directions, transposed)
    for (int idx = tid; idx < N * H; idx += GAT_THREADS) {
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(s_hp + idx);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(hprev + (idx >> 5) * a.hprev.stride_slot + (idx & 31)));
    }
    asm volatile("cp.async.commit_group;");
    {
        const float* dlf = a.dl + (((int64_t)ag * a.n_envs + b) * 2) * NM1 * DLP;
        const float* dlr = dlf + (int64_t)NM1 * DLP;
        for (int idx = tid; idx < NM1 * DLP; idx += GAT_THREADS) {
            const int s = idx / DLP, i = idx - s * DLP;
            if (i < N) s_dl[i * NM1 + s] = dlf[idx] + dlr[idx];
        }
    }
    gat_encode<GAT_THREADS>(a, W, L, b, ag, s_x, s_we, s_enc);

    // ---- phase 4: q | k | v^T as ONE product over the three consecutive weight tensors; gh = h_prev W_hh^T + b_hh ------
    for (int idx = tid; idx < H * WP; idx += GAT_THREADS) s_vt[idx] = 0.0f;       // s_x is dead: gat_encode ends with a barrier
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    {
        const float* vb = W + L.v_b;
        auto store_qkv = [=](int r, int c, float v) {
            if (c < H) s_qk[r * QKP + c] = v;
            else if (c < 2 * H) s_qk[r * QKP + KOFF + (c - H)] = v;
            else s_vt[(c - 2 * H) * WP + r] = fmaxf(v + vb[c - 2 * H], 0.0f);     // v = ReLU(W_v enc + b_v), transposed
        };
        dense32_mma<GAT_WARPS, KB_H, false, EpiNone>(s_enc, H, N, W + L.q_w, H, nullptr, 3 * H, nullptr, 0, false, warp, lane, EpiNone(), store_qkv);
    }
    dense32_mma<GAT_WARPS>(s_hp, H, N, W + L.c_whh, H, W + L.c_bhh, G3, s_gh, G3, false, warp, lane);
    __syncthreads();

    // ---- phase 5a: raw scores S[i][j] = q_i . k_j for every slot pair, on the tensor cores --------
    // (columns are padded to a multiple of 8: rows of the q|k buffer past N-1 are whatever follows in shared memory,
    //  inside the allocation (att_smem_floats); those columns are never read)
    dense32_mma<GAT_WARPS>(s_qk, QKP, N, s_qk + KOFF, QKP, nullptr, (N + 7) & ~7, s_w, WP, false, warp, lane);
    __syncthreads();

    // ---- phase 5b: soft x hard attention weights, one warp per ego; lane -> slots j = lane, lane + 32 ----
    const float db = W[L.he_b + 1] - W[L.he_b + 0];
    for (int i = warp; i < N; i += GAT_WARPS) {
        float sc[2], hd[2];
        uint4 rnd[2] = {make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u)};
        if (!a.gumbel) {                                                  // Philox key (ego, j >> 2), word j & 3
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int64_t key = (((int64_t)ag * a.n_envs + b) * N + i) * 16 + ((lane + 32 * u) >> 2);
                rnd[u] = philox4x32(make_uint4((uint32_t)key, (uint32_t)(key >> 32), (uint32_t)a.counter, (uint32_t)(a.counter >> 32)),
                                    make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)));
            }
        }
        float* wrow = s_w + i * WP;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int j = lane + 32 * u;
            sc[u] = -INFINITY; hd[u] = 0.0f;
            if (j < N && j != i) {
                const int s = j < i ? j : j - 1;                         // position of neighbour j in ego i's sequence
                sc[u] = wrow[j] * 0.17677669529663687f;                  // / np.sqrt(attention_dim), :126
                float noise;
                const int64_t edge = (((int64_t)ag * a.n_envs + b) * N + i) * NM1 + s;
                if (a.gumbel) {
                    noise = a.gumbel[2 * edge + 1] - a.gumbel[2 * edge];
                } else {
                    const int wsel = lane & 3;
                    const float uu = u01(wsel == 0 ? rnd[u].x : (wsel == 1 ? rnd[u].y : (wsel == 2 ? rnd[u].z : rnd[u].w)));
                    noise = __logf(uu) - __logf(1.0f - uu);  // Gumbel - Gumbel ~ Logistic(0,1)
                }
                const float dlog = s_dl[i * NM1 + s] + db;
                hd[u] = __fdividef(1.0f, 1.0f + expf(-(dlog + noise) * a.inv_tau));
                if (a.dbg_hard) a.dbg_hard[edge] = hd[u];
            }
        }
        const float mx = warp_max(fmaxf(sc[0], sc[1]));
        const float e0 = expf(sc[0] - mx);                               // exp(-inf) = 0 for self / padding
        const float e1 = expf(sc[1] - mx);
        const float den = warp_sum(e0 + e1);
        wrow[lane] = (e0 / den) * hd[0];
        wrow[lane + 32] = (e1 / den) * hd[1];
    }
    __syncthreads();

    // ---- phase 5c: x_i = sum_j w[i][j] v_j  =  W (N x 64) . V (64 x 32), on the tensor cores -------
    dense32_mma<GAT_WARPS, 4>(s_w, WP, N, s_vt, WP, nullptr, H, s_xa, H, false, warp, lane);
    __syncthreads();

    // ---- phase 6: GRUCell(x_i, h_prev_i) (:140): gi = x W_ih^T + b_ih (gh was computed in phase 4), gates -----
    dense32_mma<GAT_WARPS>(s_xa, H, N, W + L.c_wih, H, W + L.c_bih, G3, s_gi, G3, false, warp, lane);
    __syncthreads();
    for (int idx = tid; idx < N * H; idx += GAT_THREADS) {
        const int n = idx >> 5, c = idx & 31;
        const float* gi = s_gi + n * G3;
        const float* gh = s_gh + n * G3;
        const float r = sigmoidf_acc(gi[c] + gh[c]);
        const float z = sigmoidf_acc(gi[H + c] + gh[H + c]);
        const float nn = tanhf_acc(gi[2 * H + c] + r * gh[2 * H + c]);
        outp[n * a.out.stride_slot + c] = (1.0f - z) * nn + z * s_hp[idx];
    }
}

}  // namespace iplan

extern "C" int64_t iplan_gat_scratch_floats(int n_envs, int n_agents, int n_slots) {
    return (int64_t)n_envs * n_agents * 2 * (n_slots - 1) * iplan::DLP;
}

extern "C" int iplan_gat_step_ex(const float* gat_params, int64_t param_stride,
                                 iplan_view hist, iplan_view beh_prev, iplan_view h_prev, iplan_view out,
                                 const float* gumbel, uint64_t seed, uint64_t counter,
                                 float tau, float* dbg_hard, float* scratch, int64_t scratch_floats,
                                 int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim,
                                 void* ev_begin, void* ev_mid, void* ev_end, void* stream) {
    using namespace iplan;
    IPLAN_REQUIRE(n_slots >= 2 && n_slots <= IPLAN_MAX_SLOTS, "gat_step: n_slots %d not in [2,%d]", n_slots, IPLAN_MAX_SLOTS);
    IPLAN_REQUIRE(obs_dim + latent_dim <= IN_MAX && obs_dim > 0 && latent_dim >= 0, "gat_step: obs_dim+latent_dim %d > %d", obs_dim + latent_dim, IN_MAX);
    IPLAN_REQUIRE(n_envs > 0 && n_agents > 0 && n_agents <= 65535, "gat_step: bad n_envs/n_agents");
    IPLAN_REQUIRE(gat_params && hist.ptr && beh_prev.ptr && h_prev.ptr && out.ptr, "gat_step: null pointer");
    IPLAN_REQUIRE(tau > 0.f, "gat_step: tau must be > 0");
    IPLAN_REQUIRE(scratch && scratch_floats >= iplan_gat_scratch_floats(n_envs, n_agents, n_slots),
                  "gat_step: scratch too small (%lld floats, need iplan_gat_scratch_floats)", (long long)scratch_floats);
    GatArgs a;
    a.params = gat_params; a.param_stride = param_stride;
    a.hist = hist; a.beh = beh_prev; a.hprev = h_prev; a.out = out;
    a.gumbel = gumbel; a.dbg_hard = dbg_hard; a.dl = scratch; a.seed = seed; a.counter = counter;
    a.inv_tau = 1.0f / tau;
    a.n_envs = n_envs; a.n_slots = n_slots; a.obs_dim = obs_dim; a.latent_dim = latent_dim;
    const size_t smem_r = rec_smem_floats(n_slots) * sizeof(float);
    const size_t smem_a = att_smem_floats(n_slots) * sizeof(float);
    static size_t conf_r = 0, conf_a = 0;
    if (smem_r > conf_r) {
        cudaError_t e = cudaFuncSetAttribute(gat_recur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_r);
        if (e != cudaSuccess) { set_error("gat_step: recur smem attr %zu: %s", smem_r, cudaGetErrorString(e)); return (int)e; }
        conf_r = smem_r;
    }
    if (smem_a > conf_a) {
        cudaError_t e = cudaFuncSetAttribute(gat_attend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_a);
        if (e != cudaSuccess) { set_error("gat_step: attend smem attr %zu: %s", smem_a, cudaGetErrorString(e)); return (int)e; }
        conf_a = smem_a;
    }
    if (ev_begin) cudaEventRecord((cudaEvent_t)ev_begin, (cudaStream_t)stream);
    gat_recur_kernel<<<dim3(n_envs, n_agents, 2), REC_THREADS, smem_r, (cudaStream_t)stream>>>(a);
    count_launch();
    int rc = check_launch("gat_step(recur)");
    if (rc) return rc;
    if (ev_mid) cudaEventRecord((cudaEvent_t)ev_mid, (cudaStream_t)stream);
    gat_attend_kernel<<<dim3(n_envs, n_agents), GAT_THREADS, smem_a, (cudaStream_t)stream>>>(a);
    count_launch();
    rc = check_launch("gat_step(attend)");
    if (ev_end) cudaEventRecord((cudaEvent_t)ev_end, (cudaStream_t)stream);
    return rc;
}

extern "C" int iplan_gat_step(const float* gat_params, int64_t param_stride,
                              iplan_view hist, iplan_view beh_prev, iplan_view h_prev, iplan_view out,
                              const float* gumbel, uint64_t seed, uint64_t counter,
                              float tau, float* dbg_hard, float* scratch, int64_t scratch_floats,
                              int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim,
                              void* stream) {
    return iplan_gat_step_ex(gat_params, param_stride, hist, beh_prev, h_prev, out, gumbel, seed, counter, tau, dbg_hard,
                             scratch, scratch_floats, n_envs, n_agents, n_slots, obs_dim, latent_dim,
                             nullptr, nullptr, nullptr, stream);
}
