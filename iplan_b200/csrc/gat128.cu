// GAT_Net.forward at GAT_hidden_dim = attention_dim = 128 (the synthetic GAT + GRU microbench, 8192 envs x 32 agent-nets x
// 16 slots x 128-d; the op is reference nova/GAT_Net.py:41-142 with wider layers).
//
// At H = 128 one chain's ego projection is 384 values and the hidden-state weights of one direction (384 x 128) are 96 KB
// per f16 part.  So the product is turned around:
//
//     D^T[gate row (384)][chain (N = 16 = the egos of one item)] = W_hh[384 x 128] . h^T[128 x 16]
//
// and runs on the Hopper warpgroup tensor cores (wgmma.mma_async m64n16k16, f16 inputs, fp32 accumulators in registers):
//   A = W_hh of this (agent-net, direction), f16 hi + lo parts (192 KB), written once per CTA into shared memory as K-major
//       SWIZZLE_128B tiles of [64 gate rows][64 k];
//   B = h^T of the current item, a K-major SWIZZLE_128B tile [16 chains][128 hi | 128 lo] f16 (8 KB), double buffered:
//       step s reads one buffer while the gate math writes h_{s+1} into the other, so one CTA barrier per step suffices.
// fp32 accuracy comes from the hi / lo split: hi*hi + hi*lo + lo*hi (three passes of 8 k-blocks; lo*lo < 2^-22 relative).
// Warpgroup w owns hidden units 64 w .. 64 w + 63 of all three gates (M-tiles r, z, n), so the r, z and n pre-activations of
// a (unit, chain) land in the same thread: two units x four chains per thread.  It adds P (registers, constant over the 15
// steps) and Q (read from L2 while the product runs), applies the gates (ex2 + shared rcp as in K1), keeps h in fp32
// registers and writes its f16 hi / lo halves into the next operand tile.  The per-step hard-attention logit (a sum over
// the 128 units) is a butterfly over the 8 rows of a warp fragment + an 8-warp exchange through shared memory.
//
// The GEMM-shaped parts of the op (encode, the factored input projections P | Q, q | k | v, the GRUCell projections) are
// plain row x weight products over all 4.2 M slots: the host side runs them as library GEMMs (cuBLAS fp32 through
// torch.matmul, iplan_b200/nova/gat128.py); this file holds the recurrence, the attention and the GRUCell gate kernels.
#include "common.cuh"
#include "gat_common.cuh"

namespace iplan {

constexpr int HB = 128, G3B = 3 * HB, NB = 16, STEPS = NB - 1;
constexpr int G8_THREADS = 256;                      // two warpgroups; warpgroup w = hidden units 64 w .. 64 w + 63
constexpr int G8_WTILE = 64 * 128;                   // one [64 rows][64 k] f16 operand tile (rows of 128 B)
constexpr int G8_OFF_W = 0;                          // W_hh tiles [gate 3][warpgroup 2][k half 2][hi | lo]
constexpr int G8_BT_BYTES = 4 * NB * 128;            // h^T operand tile: 4 sub-tiles (hi k<64, hi k>=64, lo, lo) of [16 rows][128 B]
constexpr int G8_OFF_BT = G8_OFF_W + 24 * G8_WTILE;  // 2 buffers
constexpr int G8_OFF_PL = G8_OFF_BT + 2 * G8_BT_BYTES;   // logit exchange [2 parities][8 warps][16 chains]
constexpr size_t G8_SMEM = G8_OFF_PL + 2 * 8 * NB * 4 + 1024;   // + alignment of the base to 1024 B (swizzle atoms)

struct Gat128Args {
    const float* P; const float* Q;                  // [2 dirs][A][items][16][384] gate-scaled ego / neighbour projections (+ biases in Q)
    const float* whh;                                // [A][2][384][128]
    const float* bhn;                                // [A][2][128]  b_hn (unscaled)
    const float* lw;                                 // [A][2][128]  logit-difference weights
    float* dl;                                       // [A][items][2][15][16]
    int n_agents; int64_t n_items; int items_per_cta;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sts16(uint32_t addr, uint16_t v) {
    asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Byte offset of 16-byte chunk `chunk` (0..7) of row `row` in a K-major SWIZZLE_128B tile (rows of 128 B, base 1024-aligned)
__device__ __forceinline__ uint32_t swz128(int row, int chunk) {
    return (uint32_t)(row >> 3) * 1024u + (uint32_t)(row & 7) * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
}
// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_128B tile: rows of 128 B, 8-row groups 1024 B apart (stride
// byte offset); the leading byte offset is unused when K fits one swizzle atom.  A k-block of 16 f16 starts 32 B further.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N_PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N_PENDING) : "memory"); }
// D[64 x 16] += A[64 x 16] . B[16 x 16]^T, both operands K-major in shared memory, f16 in, fp32 accumulate
// accumulate == 0: D = A . B^T (the old contents of d are ignored)
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t da, uint64_t db, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(accumulate) : "memory");
}

__global__ void __launch_bounds__(G8_THREADS, 1) gat128_recur_kernel(Gat128Args a) {
    extern __shared__ unsigned char g8_raw[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wg = warp >> 2, q = lane & 3;
    const int ag = blockIdx.y, dir = blockIdx.z;
    const uint32_t raw_u = smem_u32(g8_raw);
    const uint32_t base = (raw_u + 1023u) & ~1023u;
    float* plx = reinterpret_cast<float*>(g8_raw + (base - raw_u) + G8_OFF_PL);
    auto wtile = [&](int g, int kh, int hl) { return base + G8_OFF_W + (uint32_t)((((g * 2 + wg) * 2 + kh) * 2 + hl) * G8_WTILE); };

    // ---- W_hh -> shared memory, gate-activation scale folded in (see gat_common.cuh), f16 hi and lo tiles -----------------
    {
        const float* whh = a.whh + (int64_t)(ag * 2 + dir) * G3B * HB;
        for (int idx = tid; idx < G3B * (HB / 8); idx += G8_THREADS) {
            const int row = idx >> 4, c16 = idx & 15;                // gate row, chunk of 8 k
            const int g = row >> 7, w = (row >> 6) & 1, r = row & 63, kh = c16 >> 3;
            const float ks = g < 2 ? K_RZ : K_N;
            const float4 x0 = *reinterpret_cast<const float4*>(whh + (int64_t)row * HB + 8 * c16);
            const float4 x1 = *reinterpret_cast<const float4*>(whh + (int64_t)row * HB + 8 * c16 + 4);
            uint32_t hi[4], lo[4];
            split_f16(ks * x0.x, ks * x0.y, hi[0], lo[0]);
            split_f16(ks * x0.z, ks * x0.w, hi[1], lo[1]);
            split_f16(ks * x1.x, ks * x1.y, hi[2], lo[2]);
            split_f16(ks * x1.z, ks * x1.w, hi[3], lo[3]);
            const uint32_t t = base + G8_OFF_W + (uint32_t)((((g * 2 + w) * 2 + kh) * 2) * G8_WTILE) + swz128(r, c16 & 7);
            sts128(t, hi[0], hi[1], hi[2], hi[3]);
            sts128(t + G8_WTILE, lo[0], lo[1], lo[2], lo[3]);
        }
    }
    // this thread's accumulator elements (m64n16 fragment): rows = units u0, u0 + 8; columns = chains 2q, 2q+1 (j = 0) and
    // 8 + 2q, 9 + 2q (j = 1); element 4 j + 2 rr + e = (unit u0 + 8 rr, chain 8 j + 2 q + e)
    const int u0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int uu[2] = {u0, u0 + 8};
    float bn[2], lwu[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        bn[rr] = K_N * a.bhn[(ag * 2 + dir) * HB + uu[rr]];
        lwu[rr] = a.lw[(ag * 2 + dir) * HB + uu[rr]];
    }

    const int64_t it0 = (int64_t)blockIdx.x * a.items_per_cta;
    const int64_t it1 = it0 + a.items_per_cta < a.n_items ? it0 + a.items_per_cta : a.n_items;
    const int64_t pq_stride_dir = (int64_t)a.n_agents * a.n_items * NB * G3B;
    const float* Pd = a.P + dir * pq_stride_dir + (int64_t)ag * a.n_items * NB * G3B;
    const float* Qd = a.Q + dir * pq_stride_dir + (int64_t)ag * a.n_items * NB * G3B;
    const f32x2 one2 = pk2(1.0f, 1.0f), mtwo2 = pk2(-2.0f, -2.0f);
    int buf = 0;
    for (int64_t item = it0; item < it1; ++item) {
        // ---- per item: P into registers, h = 0, operand tile = 0 -----------------------------------------------------------
        f32x2 P2[3][2][2];                                          // [gate][rr][j]: (chain 8 j + 2 q, +1) of unit uu[rr]
        {
            const float* pp = Pd + item * NB * G3B;
#pragma unroll
            for (int g = 0; g < 3; ++g)
#pragma unroll
                for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int c = 8 * j + 2 * q;
                        P2[g][rr][j] = pk2(pp[c * G3B + g * HB + uu[rr]], pp[(c + 1) * G3B + g * HB + uu[rr]]);
                    }
        }
        f32x2 h2[2][2];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) h2[rr][0] = h2[rr][1] = pk2(0.f, 0.f);
        {
            const uint32_t z = base + G8_OFF_BT + buf * G8_BT_BYTES + 32 * tid;     // 8 KB / 256 threads
            sts128(z, 0u, 0u, 0u, 0u);
            sts128(z + 16, 0u, 0u, 0u, 0u);
        }
        fence_proxy_async();
        __syncthreads();
        const float* qt = Qd + item * NB * G3B;
        for (int step = 0; step < STEPS; ++step) {
            const int s = dir ? STEPS - 1 - step : step;
            // neighbour of ego c at position s: j = s < c ? s : s + 1 -> chains 0..s read Q row s+1, chains s+1.. read row s.
            // Issued before the product so that the L2 latency overlaps it.
            float qa[3][2], qb[3][2];
#pragma unroll
            for (int g = 0; g < 3; ++g)
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    qa[g][rr] = qt[s * G3B + g * HB + uu[rr]];
                    qb[g][rr] = qt[(s + 1) * G3B + g * HB + uu[rr]];
                }
            // D^T = W_hh h^T for this warpgroup's 64 units: 3 gates x 3 passes x 8 k-blocks
            float acc[3][8];
            const uint32_t bt = base + G8_OFF_BT + buf * G8_BT_BYTES;
            wgmma_fence();
#pragma unroll
            for (int g = 0; g < 3; ++g)
#pragma unroll
                for (int pass = 0; pass < 3; ++pass) {              // hi*hi, W hi x h lo, W lo x h hi
                    const int hl = pass == 2 ? 1 : 0;
                    const uint32_t hsub = pass == 1 ? 2u : 0u;
#pragma unroll
                    for (int kb = 0; kb < 8; ++kb) {
                        const uint64_t da = wgmma_desc(wtile(g, kb >> 2, hl) + 32u * (kb & 3));
                        const uint64_t db = wgmma_desc(bt + (hsub + (kb >> 2)) * (NB * 128) + 32u * (kb & 3));
                        wgmma_m64n16k16(acc[g], da, db, (pass | kb) != 0);
                    }
                }
            wgmma_commit();
            wgmma_wait<0>();
            // ---- gates on (chain, chain + 1) pairs; four reciprocals per rcp.approx --------------------------------------------
            auto qsel = [&](float qa_, float qb_, int c) { return s < c ? qa_ : qb_; };
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                f32x2 d[3][2], qv[3][2];
#pragma unroll
                for (int g = 0; g < 3; ++g)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int c = 8 * j + 2 * q;
                        d[g][j] = pk2(acc[g][4 * j + 2 * rr], acc[g][4 * j + 2 * rr + 1]);
                        qv[g][j] = pk2(qsel(qa[g][rr], qb[g][rr], c), qsel(qa[g][rr], qb[g][rr], c + 1));
                    }
                const f32x2 bn2 = pk2(bn[rr], bn[rr]);
                f32x2 r0, r1, z0, z1, i0, i1;
                sigmoid4_den(add2(add2(d[0][0], P2[0][rr][0]), qv[0][0]), add2(add2(d[0][1], P2[0][rr][1]), qv[0][1]), r0, r1);
                sigmoid4_den(add2(add2(d[1][0], P2[1][rr][0]), qv[1][0]), add2(add2(d[1][1], P2[1][rr][1]), qv[1][1]), z0, z1);
                sigmoid4_den(fma2(r0, add2(d[2][0], bn2), add2(P2[2][rr][0], qv[2][0])),
                             fma2(r1, add2(d[2][1], bn2), add2(P2[2][rr][1], qv[2][1])), i0, i1);
                const f32x2 n0 = fma2(mtwo2, i0, one2), n1 = fma2(mtwo2, i1, one2);
                h2[rr][0] = fma2(z0, sub2(h2[rr][0], n0), n0);
                h2[rr][1] = fma2(z1, sub2(h2[rr][1], n1), n1);
            }
            // ---- h^T into the other operand tile: element (chain c, k = unit u): sub-tile u >> 6 (hi) / 2 + (u >> 6) (lo) -------
            {
                const uint32_t nt = base + G8_OFF_BT + (buf ^ 1) * G8_BT_BYTES;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const int u = uu[rr];
                    const uint32_t sub = nt + (uint32_t)(u >> 6) * (NB * 128), ch = (uint32_t)(u & 63) >> 3, in = (uint32_t)(u & 7) * 2;
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        uint32_t hh, hl;
                        split_f16p(h2[rr][j], hh, hl);
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const uint32_t c = 8 * j + 2 * q + e;
                            const uint32_t off = (c >> 3) * 1024u + (c & 7) * 128u + ((ch ^ (c & 7)) << 4) + in;
                            sts16(sub + off, (uint16_t)(e ? hh >> 16 : hh & 0xffffu));
                            sts16(sub + 2 * (NB * 128) + off, (uint16_t)(e ? hl >> 16 : hl & 0xffffu));
                        }
                    }
                }
            }
            // ---- hard-attention logit difference of every chain: sum over the 128 units = the 8 fragment rows of a warp, then
            //      the 8 warps through shared memory
            {
                float* plw = plx + (step & 1) * (8 * NB) + warp * NB;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    float pa, pb, ra, rb;
                    upk2(h2[0][j], pa, pb);
                    upk2(h2[1][j], ra, rb);
                    pa = fmaf(lwu[1], ra, lwu[0] * pa);
                    pb = fmaf(lwu[1], rb, lwu[0] * pb);
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) { pa += __shfl_xor_sync(0xffffffffu, pa, o); pb += __shfl_xor_sync(0xffffffffu, pb, o); }
                    if (lane < 4) { plw[8 * j + 2 * q] = pa; plw[8 * j + 2 * q + 1] = pb; }
                }
            }
            fence_proxy_async();
            __syncthreads();
            buf ^= 1;
            if (tid < NB) {                                         // dl[item][dir][s][i]
                const float* px = plx + (step & 1) * (8 * NB) + tid;
                float v = px[0];
#pragma unroll
                for (int w8 = 1; w8 < 8; ++w8) v += px[w8 * NB];
                a.dl[((((int64_t)ag * a.n_items + item) * 2 + dir) * STEPS + s) * NB + tid] = v;
            }
        }
    }
}

// ---- attention over one item (16 slots): scores, gumbel hard gate, soft-max, aggregation ---------------------------------
// qkv [rows][384] (q | k | v, v WITHOUT bias / ReLU), dl [A][items][2][15][16], gumbel NULL or [A][items][16][15][2];
// x out [rows][128].  One warp per ego, 8 warps per CTA = half an item; grid = (2 * items, A).
__global__ void __launch_bounds__(256) gat128_attend_kernel(const float* __restrict__ qkv, const float* __restrict__ v_bias /* [A][128] */,
                                                             const float* __restrict__ dl, const float* __restrict__ he_b /* [A][2] */,
                                                             const float* __restrict__ gumbel, uint64_t seed, uint64_t counter, float inv_tau,
                                                             float* __restrict__ x, int64_t n_items) {
    const int ag = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t item = blockIdx.x >> 1;
    const int i = (blockIdx.x & 1) * 8 + warp;
    const int64_t row0 = ((int64_t)ag * n_items + item) * NB;
    const float* qi = qkv + (row0 + i) * G3B;
    float q4[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) q4[c] = qi[lane + 32 * c];
    const float db = he_b[ag * 2 + 1] - he_b[ag * 2];
    float sc[NB], hd[NB], mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        sc[j] = -INFINITY; hd[j] = 0.0f;
        if (j != i) {
            const float* kj = qkv + (row0 + j) * G3B + HB;
            float d = 0.0f;
#pragma unroll
            for (int c = 0; c < 4; ++c) d = fmaf(q4[c], kj[lane + 32 * c], d);
            d = warp_sum(d);
            sc[j] = d / 11.313708498984761f;                           // sqrt(attention_dim = 128)
            const int s = j < i ? j : j - 1;
            const int64_t e0 = (((int64_t)ag * n_items + item) * 2) * STEPS * NB;
            const float dlog = (dl[e0 + s * NB + i] + dl[e0 + (STEPS + s) * NB + i]) + db;
            const int64_t edge = (row0 + i) * STEPS + s;
            float noise;
            if (gumbel) noise = gumbel[2 * edge + 1] - gumbel[2 * edge];
            else {
                const uint4 rnd = philox4x32(make_uint4((uint32_t)edge, (uint32_t)(edge >> 32), (uint32_t)counter, (uint32_t)(counter >> 32)),
                                             make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
                const float uu = u01(rnd.x);
                noise = __logf(uu) - __logf(1.0f - uu);
            }
            hd[j] = sigmoidf_acc((dlog + noise) * inv_tau);
            mx = fmaxf(mx, sc[j]);
        }
    }
    float den = 0.0f;
#pragma unroll
    for (int j = 0; j < NB; ++j) { sc[j] = expf(sc[j] - mx); den += sc[j]; }
    float xa[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        if (j != i) {
            const float w = (sc[j] / den) * hd[j];
            const float* vj = qkv + (row0 + j) * G3B + 2 * HB;
#pragma unroll
            for (int c = 0; c < 4; ++c) xa[c] = fmaf(w, fmaxf(vj[lane + 32 * c] + v_bias[ag * HB + lane + 32 * c], 0.0f), xa[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) x[(row0 + i) * HB + lane + 32 * c] = xa[c];
}

// ---- GRUCell gates (nova/GAT_Net.py:140): gi, gh [rows][384] (biases included), h_prev / out [rows][128] ----------------------
__global__ void gat128_gates_kernel(const float* __restrict__ gi, const float* __restrict__ gh, const float* __restrict__ hprev,
                                    float* __restrict__ out, int64_t n) {
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx >> 7;
        const int c = (int)(idx & 127);
        const float* a = gi + r * G3B;
        const float* b = gh + r * G3B;
        const float rg = sigmoidf_acc(a[c] + b[c]);
        const float zg = sigmoidf_acc(a[HB + c] + b[HB + c]);
        const float ng = tanhf_acc(a[2 * HB + c] + rg * b[2 * HB + c]);
        out[idx] = (1.0f - zg) * ng + zg * hprev[idx];
    }
}

}  // namespace iplan

using namespace iplan;

extern "C" int iplan_gat128_recur(const float* P, const float* Q, const float* whh, const float* bhn, const float* lw, float* dl,
                                  int n_agents, int64_t n_items, void* stream) {
    IPLAN_REQUIRE(P && Q && whh && bhn && lw && dl && n_agents > 0 && n_agents <= 65535 && n_items > 0, "gat128_recur: bad arguments");
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(gat128_recur_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G8_SMEM);
        if (e != cudaSuccess) { set_error("gat128_recur: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    Gat128Args a;
    a.P = P; a.Q = Q; a.whh = whh; a.bhn = bhn; a.lw = lw; a.dl = dl; a.n_agents = n_agents; a.n_items = n_items;
    // (agent-net, direction) pairs x chunks: about eight waves of CTAs, so that the last, partial wave is short; every CTA
    // stages its W_hh once and then walks its items
    const int pairs = 2 * n_agents;
    int chunks = (sm_count() * 8 + pairs - 1) / pairs;
    if (chunks > n_items) chunks = (int)n_items;
    a.items_per_cta = (int)((n_items + chunks - 1) / chunks);
    chunks = (int)((n_items + a.items_per_cta - 1) / a.items_per_cta);
    gat128_recur_kernel<<<dim3((unsigned)chunks, (unsigned)n_agents, 2), G8_THREADS, G8_SMEM, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("gat128_recur");
}

extern "C" int iplan_gat128_attend(const float* qkv, const float* v_bias, const float* dl, const float* he_b, const float* gumbel,
                                   uint64_t seed, uint64_t counter, float tau, float* x, int n_agents, int64_t n_items, void* stream) {
    IPLAN_REQUIRE(qkv && v_bias && dl && he_b && x && n_agents > 0 && n_items > 0 && tau > 0.f, "gat128_attend: bad arguments");
    IPLAN_REQUIRE(2 * n_items <= 2147483647LL, "gat128_attend: too many items for one launch");
    gat128_attend_kernel<<<dim3((unsigned)(2 * n_items), (unsigned)n_agents), 256, 0, (cudaStream_t)stream>>>(
        qkv, v_bias, dl, he_b, gumbel, seed, counter, 1.0f / tau, x, n_items);
    count_launch();
    return check_launch("gat128_attend");
}

extern "C" int iplan_gat128_gates(const float* gi, const float* gh, const float* hprev, float* out, int64_t rows, void* stream) {
    IPLAN_REQUIRE(gi && gh && hprev && out && rows > 0, "gat128_gates: bad arguments");
    gat128_gates_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(gi, gh, hprev, out, rows * HB);
    count_launch();
    return check_launch("gat128_gates");
}
