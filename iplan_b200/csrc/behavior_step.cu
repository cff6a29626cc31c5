// K1b — behaviour-incentive encoder step.
//
// Replaces Behavior_policy.latent_update (reference nova/stable_behavior_policy.py:83-123)
// and EncoderRNN.forward (nova/behavior_net.py:17-22):
//   u_t   = ReLU(W_l w_t + b_l)                       for the W window rows w_t of a slot
//   h     = GRU(u_1..u_W ; h_carried)                 (one layer, batch_first)
//   z     = softmax(W_o h + b_o)                      latent_dim values
//   new   = (1 - c) * prev + c * z                    soft update (:118), c = soft_update_coef
// A "node" is one (env, agent-net, slot); nodes are independent.  One warp advances 16 nodes;
// every product of a step runs on the tensor cores with mma.sync.m16n8k16 (f16 hi/lo split of
// both operands, three MMAs per product -> fp32-class accuracy, see gat_step.cu):
//   u_t (16x32)  = [w_t | 1 | 0..] (16x16) . [W_l | b_l]^T          -> accumulator layout
//   gates        = u_t . W_ih^T  +  h . W_hh^T                        (accumulator layout of one
//                  product is the A layout of the next: u and h never leave registers)
// The B fragments of W_l, W_ih, W_hh (hi and lo) are staged once per CTA in shared memory.
#include <cuda_fp16.h>

#include <stdlib.h>

#include "common.cuh"
#include "behavior_common.cuh"

namespace iplan {

constexpr int E = IPLAN_HID;       // encoder_rnn_dim
constexpr int E3 = 3 * E;
constexpr int BEH_THREADS = 256;
constexpr int BEH_WARPS = BEH_THREADS / 32;
constexpr int NODES_W = 16;        // nodes per warp (one MMA m-tile)
constexpr int WIN_MAX = 64;        // hist_len * obs_dim upper bound per node
constexpr int LAT_MAX = 8;         // latent_dim upper bound (one MMA n-tile)
constexpr int NT3 = E3 / 8;        // 12 gate n-tiles

struct BehSmem {
    uint2 wih[2][NT3][2][32];       // [hi|lo][n-tile][k-block][lane] B fragments of W_ih
    uint2 whh[2][NT3][2][32];       // ... of W_hh
    uint2 wlin[2][4][32];           // [hi|lo][n-tile][lane] B fragments of [W_l | b_l] (K padded to 16)
    uint2 wout[2][2][32];           // [hi|lo][k-block][lane] B fragments of W_o (N padded to 8)
    float2 bias[16][4];             // accumulator-layout bias pairs: [0..7] b_ih+b_hh (r|z), [8..11] b_in, [12..15] b_hn
    float win[BEH_WARPS][NODES_W][WIN_MAX];
};

__device__ __forceinline__ float bsigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float btanh(float x) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * x)); }

__device__ __forceinline__ void bsplit(float x, float y, uint32_t& hi, uint32_t& lo) {
    const __half2 h = __floats2half2_rn(x, y);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(x - hf.x, y - hf.y);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void bmma(float (&d)[4], const uint32_t (&a)[4], uint2 b, const float (&c)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%11,%12,%13};"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y), "f"(c[0]), "f"(c[1]), "f"(c[2]), "f"(c[3]));
}
// accumulator-layout values v[4 tiles][4] (16 rows x 32 cols) -> A fragments of the two k-blocks
__device__ __forceinline__ void to_afrag(const float (&v)[4][4], uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
    for (int kb = 0; kb < 2; ++kb) {
        bsplit(v[2 * kb][0], v[2 * kb][1], hi[kb][0], lo[kb][0]);
        bsplit(v[2 * kb][2], v[2 * kb][3], hi[kb][1], lo[kb][1]);
        bsplit(v[2 * kb + 1][0], v[2 * kb + 1][1], hi[kb][2], lo[kb][2]);
        bsplit(v[2 * kb + 1][2], v[2 * kb + 1][3], hi[kb][3], lo[kb][3]);
    }
}

__global__ void __launch_bounds__(BEH_THREADS, 2) behavior_step_kernel(BehArgs a) {
    extern __shared__ __align__(16) unsigned char raw[];
    BehSmem& S = *reinterpret_cast<BehSmem*>(raw);
    const int ag = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int gq = lane >> 2, tq = lane & 3;
    const int N = a.n_slots, o = a.obs_dim, Wn = a.hist_len, Ld = a.latent_dim;
    const float* __restrict__ P = a.params + (int64_t)ag * a.param_stride;
    const BehLayout L = beh_layout(o, Ld);
    const int total_nodes = a.n_envs * N;

    // ---- stage the B fragments (b0 = (k=2t,2t+1 ; n=g), b1 = (k=2t+8,2t+9 ; n=g)) --------------
    for (int idx = tid; idx < 2 * NT3 * 2 * 32; idx += BEH_THREADS) {
        const int l = idx & 31, kb = (idx >> 5) & 1, nt = (idx >> 6) % NT3, m = idx / (64 * NT3);
        const int g = l >> 2, t = l & 3;
        const float* wr = P + (m ? L.whh : L.wih) + (8 * nt + g) * E + 16 * kb + 2 * t;
        uint32_t h0, l0, h1, l1;
        bsplit(wr[0], wr[1], h0, l0);
        bsplit(wr[8], wr[9], h1, l1);
        uint2(*dst)[NT3][2][32] = m ? S.whh : S.wih;
        dst[0][nt][kb][l] = make_uint2(h0, h1);
        dst[1][nt][kb][l] = make_uint2(l0, l1);
    }
    for (int idx = tid; idx < 4 * 32; idx += BEH_THREADS) {
        const int l = idx & 31, nt = idx >> 5;
        const int g = l >> 2, t = l & 3;
        const int c = 8 * nt + g;                       // output unit
        auto wl = [&](int k) { return k < o ? P[L.lin_w + c * o + k] : (k == o ? P[L.lin_b + c] : 0.0f); };
        uint32_t h0, l0, h1, l1;
        bsplit(wl(2 * t), wl(2 * t + 1), h0, l0);
        bsplit(wl(2 * t + 8), wl(2 * t + 9), h1, l1);
        S.wlin[0][nt][l] = make_uint2(h0, h1);
        S.wlin[1][nt][l] = make_uint2(l0, l1);
    }
    for (int idx = tid; idx < 2 * 32; idx += BEH_THREADS) {
        const int l = idx & 31, kb = idx >> 5;
        const int g = l >> 2, t = l & 3;
        auto wo = [&](int k) { return g < Ld ? P[L.out_w + g * E + k] : 0.0f; };
        uint32_t h0, l0, h1, l1;
        bsplit(wo(16 * kb + 2 * t), wo(16 * kb + 2 * t + 1), h0, l0);
        bsplit(wo(16 * kb + 2 * t + 8), wo(16 * kb + 2 * t + 9), h1, l1);
        S.wout[0][kb][l] = make_uint2(h0, h1);
        S.wout[1][kb][l] = make_uint2(l0, l1);
    }
    for (int idx = tid; idx < 16 * 4; idx += BEH_THREADS) {      // bias pairs for cols 8*nt + 2*t + {0,1}
        const int t = idx & 3, j = idx >> 2;
        float v[2];
        for (int u = 0; u < 2; ++u) {
            if (j < 8) { const int c = 8 * j + 2 * t + u; v[u] = P[L.bih + c] + P[L.bhh + c]; }
            else if (j < 12) v[u] = P[L.bih + 2 * E + 8 * (j - 8) + 2 * t + u];
            else v[u] = P[L.bhh + 2 * E + 8 * (j - 12) + 2 * t + u];
        }
        S.bias[j][t] = make_float2(v[0], v[1]);
    }

    // ---- this warp's 16 nodes ------------------------------------------------------------------
    const int node_base = (blockIdx.x * BEH_WARPS + warp) * NODES_W;
    const int nd0 = node_base + gq, nd1 = nd0 + 8;
    const bool ok0 = nd0 < total_nodes, ok1 = nd1 < total_nodes;
    const int c0n = ok0 ? nd0 : 0, c1n = ok1 ? nd1 : 0;
    const int b0 = c0n / N, n0 = c0n - b0 * N, b1 = c1n / N, n1 = c1n - b1 * N;
    // stage the 16 windows.  All loads of a batch are issued before the first store (one L2 round trip per batch: the
    // kernel used to spend 40 % of its time in a load -> store -> next load chain here)
    if (a.win_step != 0 && o <= 8) {
        // rows live `win_step` apart (the episode store's time axis): lane -> (node r, window row w) pairs, o floats each
        constexpr int PB = 5, OM = 8;
        const int pairs = NODES_W * Wn;
        for (int p0 = 0; p0 < pairs; p0 += 32 * PB) {
            float v[PB][OM];
            int dsto[PB];
#pragma unroll
            for (int k = 0; k < PB; ++k) {
                const int pp = p0 + 32 * k + lane;
                const bool on = pp < pairs;
                const int r = on ? pp / Wn : 0, w = on ? pp - r * Wn : 0;
                const int nd = min(node_base + r, total_nodes - 1);
                const int bb = nd / N, nn = nd - bb * N;
                const bool ld = on && w >= a.win_pad;
                const float* src = a.window.ptr + ag * a.window.stride_agent + bb * a.window.stride_env + nn * a.window.stride_slot
                                   + (int64_t)(ld ? w - a.win_pad : 0) * a.win_step;
                dsto[k] = on ? r * WIN_MAX + w * o : -1;
#pragma unroll
                for (int c = 0; c < OM; ++c) v[k][c] = (ld && c < o) ? src[c] : 0.0f;
            }
#pragma unroll
            for (int k = 0; k < PB; ++k) {
                if (dsto[k] >= 0) {
                    float* dst = &S.win[warp][0][0] + dsto[k];
#pragma unroll
                    for (int c = 0; c < OM; ++c)
                        if (c < o) dst[c] = v[k][c];
                }
            }
        }
    } else {
        for (int r0 = 0; r0 < NODES_W; r0 += 8) {
            float v[8][2];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int nd = min(node_base + r0 + k, total_nodes - 1);
                const int bb = nd / N, nn = nd - bb * N;
                const float* src = a.window.ptr + ag * a.window.stride_agent + bb * a.window.stride_env + nn * a.window.stride_slot;
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int q = lane + 32 * u;
                    float x = 0.0f;
                    if (q < Wn * o) {
                        if (a.win_step == 0) x = src[q];
                        else { const int w = q / o, c = q - w * o; x = w >= a.win_pad ? src[(int64_t)(w - a.win_pad) * a.win_step + c] : 0.0f; }
                    }
                    v[k][u] = x;
                }
            }
#pragma unroll
            for (int k = 0; k < 8; ++k)
#pragma unroll
                for (int u = 0; u < 2; ++u)
                    if (lane + 32 * u < Wn * o) S.win[warp][r0 + k][lane + 32 * u] = v[k][u];
        }
    }
    float h[4][4];
    {
        const float* h0p = a.hid.ptr + ag * a.hid.stride_agent + b0 * a.hid.stride_env + n0 * a.hid.stride_slot;
        const float* h1p = a.hid.ptr + ag * a.hid.stride_agent + b1 * a.hid.stride_env + n1 * a.hid.stride_slot;
#pragma unroll
        for (int t4 = 0; t4 < 4; ++t4) {
            const float2 v0 = *reinterpret_cast<const float2*>(h0p + 8 * t4 + 2 * tq);
            const float2 v1 = *reinterpret_cast<const float2*>(h1p + 8 * t4 + 2 * tq);
            h[t4][0] = v0.x; h[t4][1] = v0.y; h[t4][2] = v1.x; h[t4][3] = v1.y;
        }
    }
    __syncthreads();
    if (node_base >= total_nodes) return;

    const float zero4[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int t = 0; t < Wn; ++t) {
        // A fragment of [w_t | 1 | 0...]: this thread holds k = 2tq, 2tq+1 of rows gq and gq+8
        uint32_t whi[4], wlo[4];
        {
            const float* w0 = S.win[warp][gq] + t * o;
            const float* w1 = S.win[warp][gq + 8] + t * o;
            const int k0 = 2 * tq, k1 = 2 * tq + 1;
            const float x00 = k0 < o ? w0[k0] : (k0 == o ? 1.0f : 0.0f), x01 = k1 < o ? w0[k1] : (k1 == o ? 1.0f : 0.0f);
            const float x10 = k0 < o ? w1[k0] : (k0 == o ? 1.0f : 0.0f), x11 = k1 < o ? w1[k1] : (k1 == o ? 1.0f : 0.0f);
            bsplit(x00, x01, whi[0], wlo[0]);
            bsplit(x10, x11, whi[1], wlo[1]);
            whi[2] = whi[3] = wlo[2] = wlo[3] = 0u;           // k = 8..15 : zero padding
        }
        float u[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            bmma(u[nt], whi, S.wlin[0][nt][lane], zero4);
            bmma(u[nt], wlo, S.wlin[0][nt][lane], u[nt]);
            bmma(u[nt], whi, S.wlin[1][nt][lane], u[nt]);
#pragma unroll
            for (int e = 0; e < 4; ++e) u[nt][e] = fmaxf(u[nt][e], 0.0f);
        }
        uint32_t uhi[2][4], ulo[2][4], hhi[2][4], hlo[2][4];
        to_afrag(u, uhi, ulo);
        to_afrag(h, hhi, hlo);
        // hidden units in groups of 8 (t4): the group's r|z|n tiles take their MMA passes (independent
        // chains), then its gates run while the next group's MMAs are in flight; only one group's
        // accumulators are live at a time (register budget for 2 CTAs per SM)
#pragma unroll
        for (int t4 = 0; t4 < 4; ++t4) {
            float acc[3][4], ahn[4];
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) {                       // input part from u: bias as C operand
                const int nt = 4 * gi + t4;
                const float2 bb = S.bias[nt][tq];
                const float c[4] = {bb.x, bb.y, bb.x, bb.y};
                bmma(acc[gi], uhi[0], S.wih[0][nt][0][lane], c);
            }
            {
                const float2 bb = S.bias[12 + t4][tq];              // b_hn
                const float c[4] = {bb.x, bb.y, bb.x, bb.y};
                bmma(ahn, hhi[0], S.whh[0][8 + t4][0][lane], c);
            }
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) { const int nt = 4 * gi + t4; bmma(acc[gi], uhi[1], S.wih[0][nt][1][lane], acc[gi]); }
            bmma(ahn, hhi[1], S.whh[0][8 + t4][1][lane], ahn);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) { const int nt = 4 * gi + t4; bmma(acc[gi], ulo[0], S.wih[0][nt][0][lane], acc[gi]); }
            bmma(ahn, hlo[0], S.whh[0][8 + t4][0][lane], ahn);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) { const int nt = 4 * gi + t4; bmma(acc[gi], ulo[1], S.wih[0][nt][1][lane], acc[gi]); }
            bmma(ahn, hlo[1], S.whh[0][8 + t4][1][lane], ahn);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) { const int nt = 4 * gi + t4; bmma(acc[gi], uhi[0], S.wih[1][nt][0][lane], acc[gi]); }
            bmma(ahn, hhi[0], S.whh[1][8 + t4][0][lane], ahn);
#pragma unroll
            for (int gi = 0; gi < 3; ++gi) { const int nt = 4 * gi + t4; bmma(acc[gi], uhi[1], S.wih[1][nt][1][lane], acc[gi]); }
            bmma(ahn, hhi[1], S.whh[1][8 + t4][1][lane], ahn);
            // hidden part of r|z accumulates on top of the input part
#pragma unroll
            for (int gi = 0; gi < 2; ++gi) {
                const int nt = 4 * gi + t4;
                bmma(acc[gi], hhi[0], S.whh[0][nt][0][lane], acc[gi]);
                bmma(acc[gi], hhi[1], S.whh[0][nt][1][lane], acc[gi]);
                bmma(acc[gi], hlo[0], S.whh[0][nt][0][lane], acc[gi]);
                bmma(acc[gi], hlo[1], S.whh[0][nt][1][lane], acc[gi]);
                bmma(acc[gi], hhi[0], S.whh[1][nt][0][lane], acc[gi]);
                bmma(acc[gi], hhi[1], S.whh[1][nt][1][lane], acc[gi]);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float r = bsigmoid(acc[0][e]);
                const float z = bsigmoid(acc[1][e]);
                const float n = btanh(acc[2][e] + r * ahn[e]);
                h[t4][e] = n + z * (h[t4][e] - n);
            }
            asm volatile("" ::: "memory");       // keep the next group's fragment loads from being hoisted (registers)
        }
    }

    // ---- latent = softmax(W_o h + b_o), soft update, stores -----------------------------------------
    uint32_t hhi[2][4], hlo[2][4];
    to_afrag(h, hhi, hlo);
    const int lc0 = 2 * tq, lc1 = 2 * tq + 1;              // latent columns of this thread
    const float bo0 = lc0 < Ld ? P[L.out_b + lc0] : 0.0f, bo1 = lc1 < Ld ? P[L.out_b + lc1] : 0.0f;
    float lg[4] = {bo0, bo1, bo0, bo1};
    bmma(lg, hhi[0], S.wout[0][0][lane], lg);
    bmma(lg, hhi[1], S.wout[0][1][lane], lg);
    bmma(lg, hlo[0], S.wout[0][0][lane], lg);
    bmma(lg, hlo[1], S.wout[0][1][lane], lg);
    bmma(lg, hhi[0], S.wout[1][0][lane], lg);
    bmma(lg, hhi[1], S.wout[1][1][lane], lg);
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {                       // rr = 0: row gq, rr = 1: row gq + 8
        float v0 = lc0 < Ld ? lg[2 * rr] : -INFINITY, v1 = lc1 < Ld ? lg[2 * rr + 1] : -INFINITY;
        float mx = fmaxf(v0, v1);
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float e0 = lc0 < Ld ? expf(v0 - mx) : 0.0f, e1 = lc1 < Ld ? expf(v1 - mx) : 0.0f;
        float den = e0 + e1;
        den += __shfl_xor_sync(0xffffffffu, den, 1);
        den += __shfl_xor_sync(0xffffffffu, den, 2);
        const bool ok = rr ? ok1 : ok0;
        const int bb = rr ? b1 : b0, nn = rr ? n1 : n0;
        if (ok) {
            const int64_t po = ag * a.lat_prev.stride_agent + bb * a.lat_prev.stride_env + nn * a.lat_prev.stride_slot;
            const int64_t oo = ag * a.lat_out.stride_agent + bb * a.lat_out.stride_env + nn * a.lat_out.stride_slot;
            // (1 - c) * prev + z * c, each product rounded as numpy does (:118)
            if (lc0 < Ld) a.lat_out.ptr[oo + lc0] = __fadd_rn(__fmul_rn(1.0f - a.coef, a.lat_prev.ptr[po + lc0]), __fmul_rn(e0 / den, a.coef));
            if (lc1 < Ld) a.lat_out.ptr[oo + lc1] = __fadd_rn(__fmul_rn(1.0f - a.coef, a.lat_prev.ptr[po + lc1]), __fmul_rn(e1 / den, a.coef));
            float* hp = a.hid.ptr + ag * a.hid.stride_agent + bb * a.hid.stride_env + nn * a.hid.stride_slot;
#pragma unroll
            for (int t4 = 0; t4 < 4; ++t4)
                *reinterpret_cast<float2*>(hp + 8 * t4 + 2 * tq) = make_float2(h[t4][2 * rr], h[t4][2 * rr + 1]);
        }
    }
}

}  // namespace iplan

extern "C" int iplan_behavior_step(const float* beh_params, int64_t param_stride,
                                   iplan_view window, iplan_view hid_io, iplan_view lat_prev, iplan_view lat_out,
                                   float soft_coef,
                                   int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int hist_len,
                                   void* stream) {
    return iplan_behavior_step_ex(beh_params, param_stride, window, 0, 0, hid_io, lat_prev, lat_out, soft_coef,
                                  n_envs, n_agents, n_slots, obs_dim, latent_dim, hist_len, stream);
}

extern "C" int iplan_behavior_step_ex(const float* beh_params, int64_t param_stride,
                                      iplan_view window, int64_t win_stride_step, int win_pad,
                                      iplan_view hid_io, iplan_view lat_prev, iplan_view lat_out,
                                      float soft_coef,
                                      int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int hist_len,
                                      void* stream) {
    using namespace iplan;
    IPLAN_REQUIRE(win_pad >= 0 && win_pad < hist_len, "behavior_step: win_pad %d not in [0,%d)", win_pad, hist_len);
    IPLAN_REQUIRE(obs_dim > 0 && obs_dim <= 7, "behavior_step: obs_dim %d not in [1,7]", obs_dim);
    IPLAN_REQUIRE(hist_len > 0 && hist_len * obs_dim <= WIN_MAX, "behavior_step: hist_len*obs_dim %d > %d", hist_len * obs_dim, WIN_MAX);
    IPLAN_REQUIRE(latent_dim > 0 && latent_dim <= LAT_MAX, "behavior_step: latent_dim %d not in [1,%d]", latent_dim, LAT_MAX);
    IPLAN_REQUIRE(n_envs > 0 && n_agents > 0 && n_agents <= 65535 && n_slots > 0, "behavior_step: bad sizes");
    IPLAN_REQUIRE(beh_params && window.ptr && hid_io.ptr && lat_prev.ptr && lat_out.ptr, "behavior_step: null pointer");
    IPLAN_REQUIRE(hid_io.stride_slot % 2 == 0 && hid_io.stride_env % 2 == 0 && hid_io.stride_agent % 2 == 0,
                  "behavior_step: hidden-state strides must be even (8-byte vector access)");
    BehArgs a;
    a.params = beh_params; a.param_stride = param_stride;
    a.window = window; a.hid = hid_io; a.lat_prev = lat_prev; a.lat_out = lat_out;
    a.coef = soft_coef;
    a.n_envs = n_envs; a.n_slots = n_slots; a.obs_dim = obs_dim; a.latent_dim = latent_dim; a.hist_len = hist_len;
    a.win_step = win_stride_step; a.win_pad = win_stride_step ? win_pad : 0;
    const size_t smem = sizeof(BehSmem);
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(behavior_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("behavior_step: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    const int nodes = n_envs * n_slots;
    dim3 grid((nodes + BEH_WARPS * NODES_W - 1) / (BEH_WARPS * NODES_W), n_agents);
    behavior_step_kernel<<<grid, BEH_THREADS, smem, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("behavior_step");
}
