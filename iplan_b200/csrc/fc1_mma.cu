// The two large products of the IPPO update on the tensor cores.
//
//   forward   Z1[a][r][0..128) = rstd_r * (X_a[r] . W'_a[n] - mean_r * ws[n]) + cc[n]
//             = LayerNorm(F) + fc1 of the actor (n < 64) and the critic (n >= 64) in ONE pass over
//             the packed episode rows X_a [rows][ldx]  (utils/mappo_utils/mlp.py:50-56)
//   backward  G[a][kk][f] = sum_r dZ1s[a][r][kk] * X_a[r][f]      (fc1.weight / feature_norm grads)
//
// fp32 results from f16 tensor-core MMAs: both operands are split into f16 hi + lo parts and the
// products hi*hi + lo*hi + hi*lo are accumulated in fp32 (error ~2^-22 relative; the dropped lo*lo
// term is below fp32 rounding).  X never changes during a train() call, so its hi/lo split is
// made ONCE (x_split_kernel: 4 bytes per element, like the fp32 original) and both products
// stream the f16 copies; W' is split by fc1_prep, dZ1s by dz_split (scaled by a power of two so
// the small loss gradients sit in f16's normal range).
//
// Kernel shape (both): 128x128 CTA tile, BK = 32, 8 warps (4 x 2, 32x64 warp tiles),
// 3-stage cp.async pipeline, ldmatrix fragment loads (padded rows: conflict-free),
// mma.sync.m16n8k16.f16 -> f32.
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"

namespace iplan {

constexpr int F1_BM = 128, F1_BN = 128, F1_BK = 32, F1_STAGES = 3, F1_THREADS = 256;
constexpr int RHh = IPLAN_RNN;       // 64

struct NetP {
    const float* actor; const float* critic; int64_t actor_stride, critic_stride;
    __device__ __forceinline__ const float* net(int a, int type) const {
        return type == 0 ? actor + a * actor_stride : critic + a * critic_stride;
    }
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], const void* p) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t (&r)[4], const void* p) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}
__device__ __forceinline__ void mma_f16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---------------------------------------------------------------------------------------------
// one-time / per-epoch operand preparation
// ---------------------------------------------------------------------------------------------
__global__ void x_split_kernel(const float* __restrict__ x, int64_t n2, __half2* __restrict__ hi, __half2* __restrict__ lo) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (int64_t)gridDim.x * blockDim.x) {
        const float2 v = reinterpret_cast<const float2*>(x)[i];
        const __half2 h = __floats2half2_rn(v.x, v.y);
        const float2 hf = __half22float2(h);
        hi[i] = h;
        lo[i] = __floats2half2_rn(v.x - hf.x, v.y - hf.y);
    }
}

// W'[a][type*64+k][f] = gamma[f] * W1[k][f] (0 for f >= F) as f16 hi/lo; ws = sum_f W', c = W1.beta + b1
__global__ void fc1_prep16_kernel(NetP P, int F, int ldw, __half* __restrict__ Wh, __half* __restrict__ Wl,
                                  float* __restrict__ ws, float* __restrict__ cc) {
    const int a = blockIdx.y, kk = blockIdx.x;
    const int type = kk >> 6, k = kk & 63;
    const float* p = P.net(a, type);
    const TrunkLayout L = trunk_layout(F, 1, false);
    const float* w1 = p + L.fc1_w + (int64_t)k * F;
    const int64_t ob = ((int64_t)a * 128 + kk) * ldw;
    float s = 0.0f, c = 0.0f;
    for (int f = threadIdx.x; f < ldw; f += blockDim.x) {
        float v = 0.0f;
        if (f < F) {
            const float w = w1[f];
            v = p[L.ln0_w + f] * w;
            c = fmaf(p[L.ln0_b + f], w, c);
        }
        const __half h = __float2half_rn(v);
        Wh[ob + f] = h;
        Wl[ob + f] = __float2half_rn(v - __half2float(h));
        s += v;
    }
    __shared__ float red[2][32];
    s = warp_sum(s); c = warp_sum(c);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s; red[1][threadIdx.x >> 5] = c; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const int nw = blockDim.x >> 5;
        s = threadIdx.x < nw ? red[0][threadIdx.x] : 0.0f;
        c = threadIdx.x < nw ? red[1][threadIdx.x] : 0.0f;
        s = warp_sum(s); c = warp_sum(c);
        if (threadIdx.x == 0) { ws[a * 128 + kk] = s; cc[a * 128 + kk] = c + p[L.fc1_b + k]; }
    }
}

__global__ void absmax_kernel(const float* __restrict__ x, int64_t n_per_agent, unsigned* __restrict__ out /* [A] float bits */) {
    const int a = blockIdx.y;
    float m = 0.0f;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_per_agent; i += (int64_t)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(x[a * n_per_agent + i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) atomicMax(&out[a], __float_as_uint(m));      // non-negative floats order like uints
}

// dZ1s -> f16 hi/lo scaled by 2^e so that max|.| lands near 2^10; gscale[a] = 2^-e for the epilogue
__global__ void dz_split_kernel(const float* __restrict__ x, int64_t n_per_agent, const unsigned* __restrict__ amax,
                                __half* __restrict__ hi, __half* __restrict__ lo, float* __restrict__ gscale) {
    const int a = blockIdx.y;
    const float mx = __uint_as_float(amax[a]);
    int e = 0;
    if (mx > 0.0f && isfinite(mx)) { int ex; frexpf(mx, &ex); e = 10 - ex; }
    e = max(-100, min(100, e));
    const float sc = exp2f((float)e);
    if (blockIdx.x == 0 && threadIdx.x == 0) gscale[a] = exp2f((float)-e);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_per_agent; i += (int64_t)gridDim.x * blockDim.x) {
        const float v = x[a * n_per_agent + i] * sc;
        const __half h = __float2half_rn(v);
        hi[a * n_per_agent + i] = h;
        lo[a * n_per_agent + i] = __float2half_rn(v - __half2float(h));
    }
}

// ---------------------------------------------------------------------------------------------
// forward:  C[128 rows][128 n] = Xtile[128][K] . W'[128 n][K]^T       (both K-contiguous)
// ---------------------------------------------------------------------------------------------
constexpr int FW_PITCH = F1_BK + 8;                 // halves per smem row (80 B: conflict-free ldmatrix)
constexpr int FW_TILE = F1_BM * FW_PITCH;           // halves per operand tile
constexpr int FW_STAGE = 4 * FW_TILE;               // Ahi, Alo, Bhi, Blo
constexpr size_t FW_SMEM = (size_t)F1_STAGES * FW_STAGE * sizeof(__half);

__global__ void __launch_bounds__(F1_THREADS, 1) fc1_fwd_mma_kernel(
    const __half* __restrict__ Xh, const __half* __restrict__ Xl, int64_t x_sa, int ldx, int rows,
    const __half* __restrict__ Wh, const __half* __restrict__ Wl, const float* __restrict__ ws, const float* __restrict__ cc,
    const float* __restrict__ stat, float* __restrict__ Z1) {
    extern __shared__ __align__(16) __half smem_h[];
    const int a = blockIdx.y, m0 = blockIdx.x * F1_BM;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1;                       // 4 x 2 warps, 32 x 64 warp tile
    const __half* gA[2] = {Xh + a * x_sa, Xl + a * x_sa};
    const __half* gB[2] = {Wh + (int64_t)a * 128 * ldx, Wl + (int64_t)a * 128 * ldx};
    const int ktiles = ldx / F1_BK;

    auto load_stage = [&](int st, int kt) {
        __half* base = smem_h + (size_t)st * FW_STAGE;
        // 4 operand tiles x 128 rows x 4 chunks of 16 B = 2048 chunks, 8 per thread
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int c = tid + i * F1_THREADS;
            const int op = c >> 9, r = (c >> 2) & 127, ch = c & 3;
            const __half* src;
            if (op < 2) src = gA[op] + (int64_t)min(m0 + r, rows - 1) * ldx + kt * F1_BK + ch * 8;
            else src = gB[op - 2] + (int64_t)r * ldx + kt * F1_BK + ch * 8;
            cp_async16(base + op * FW_TILE + r * FW_PITCH + ch * 8, src);
        }
    };

    float acc[2][8][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0f;

#pragma unroll
    for (int s = 0; s < F1_STAGES - 1; ++s) {
        if (s < ktiles) load_stage(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < ktiles; ++kt) {
        cp_async_wait<F1_STAGES - 2>();
        __syncthreads();
        if (kt + F1_STAGES - 1 < ktiles) load_stage((kt + F1_STAGES - 1) % F1_STAGES, kt + F1_STAGES - 1);
        cp_async_commit();
        const __half* st = smem_h + (size_t)(kt % F1_STAGES) * FW_STAGE;
        // The tensor core's fp32 accumulation truncates; over hundreds of k-tiles that bias reaches
        // ~1e-5.  Keep each MMA chain to one k-tile (6 MMAs) and add the partials in fp32 (RN) below.
        float part[2][8][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.0f;
#pragma unroll
        for (int kb = 0; kb < F1_BK / 16; ++kb) {
            uint32_t ah[2][4], al[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = wm * 32 + i * 16 + (lane & 15), cpos = kb * 16 + (lane >> 4) * 8;
                ldsm_x4(ah[i], st + 0 * FW_TILE + r * FW_PITCH + cpos);
                ldsm_x4(al[i], st + 1 * FW_TILE + r * FW_PITCH + cpos);
            }
#pragma unroll
            for (int jp = 0; jp < 4; ++jp) {
                uint32_t bh[4], bl[4];
                const int n = wn * 64 + jp * 16 + (lane & 7) + ((lane >> 4) << 3), cpos = kb * 16 + ((lane >> 3) & 1) * 8;
                ldsm_x4(bh, st + 2 * FW_TILE + n * FW_PITCH + cpos);
                ldsm_x4(bl, st + 3 * FW_TILE + n * FW_PITCH + cpos);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    mma_f16(part[i][2 * jp], ah[i], bh[0], bh[1]);
                    mma_f16(part[i][2 * jp + 1], ah[i], bh[2], bh[3]);
                    mma_f16(part[i][2 * jp], al[i], bh[0], bh[1]);
                    mma_f16(part[i][2 * jp + 1], al[i], bh[2], bh[3]);
                    mma_f16(part[i][2 * jp], ah[i], bl[0], bl[1]);
                    mma_f16(part[i][2 * jp + 1], ah[i], bl[2], bl[3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                acc[i][j][0] += part[i][j][0]; acc[i][j][1] += part[i][j][1];
                acc[i][j][2] += part[i][j][2]; acc[i][j][3] += part[i][j][3];
            }
    }
    cp_async_wait<0>();
    // epilogue: fold the LayerNorm statistics
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int r = m0 + wm * 32 + i * 16 + gq + hrow * 8;
            if (r >= rows) continue;
            const float mean = stat[((int64_t)a * rows + r) * 2], rstd = stat[((int64_t)a * rows + r) * 2 + 1];
            float* zr = Z1 + ((int64_t)a * rows + r) * 128;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int n = wn * 64 + j * 8 + 2 * tq;
                float2 o;
                o.x = rstd * (acc[i][j][2 * hrow] - mean * ws[a * 128 + n]) + cc[a * 128 + n];
                o.y = rstd * (acc[i][j][2 * hrow + 1] - mean * ws[a * 128 + n + 1]) + cc[a * 128 + n + 1];
                *reinterpret_cast<float2*>(zr + n) = o;
            }
        }
}

// ---------------------------------------------------------------------------------------------
// backward:  G[128 kk][128 f] += sum_{r in chunk} dZ[r][kk] * X[r][f]    (both r-major: .trans loads)
// ---------------------------------------------------------------------------------------------
constexpr int BW_PITCH = 128 + 8;                   // halves per smem row (272 B: conflict-free ldmatrix)
constexpr int BW_TILE = F1_BK * BW_PITCH;
constexpr int BW_STAGE = 4 * BW_TILE;               // dZhi, dZlo, Xhi, Xlo
constexpr size_t BW_SMEM = (size_t)F1_STAGES * BW_STAGE * sizeof(__half);

__global__ void __launch_bounds__(F1_THREADS, 1) fc1_bwd_mma_kernel(
    const __half* __restrict__ Xh, const __half* __restrict__ Xl, int64_t x_sa, int ldx, int rows, int rows_per_chunk,
    const __half* __restrict__ Dh, const __half* __restrict__ Dl, const float* __restrict__ gscale,
    float* __restrict__ G /* [A][128][ldx] */, float* __restrict__ part /* [A][f tiles][chunks][128][F1_BN] */,
    unsigned* __restrict__ count /* [A][f tiles] */) {
    extern __shared__ __align__(16) __half smem_h[];
    const int a = blockIdx.z, f0 = blockIdx.x * F1_BN;
    const int r0 = blockIdx.y * rows_per_chunk, r1 = min(rows, r0 + rows_per_chunk);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1;
    const __half* gX[2] = {Xh + a * x_sa, Xl + a * x_sa};
    const __half* gD[2] = {Dh + (int64_t)a * rows * 128, Dl + (int64_t)a * rows * 128};
    const int ktiles = (r1 - r0 + F1_BK - 1) / F1_BK;

    auto load_stage = [&](int st, int kt) {
        __half* base = smem_h + (size_t)st * BW_STAGE;
        // 4 tiles x 32 rows x 16 chunks of 16 B = 2048 chunks, 8 per thread; rows past r1 are zero-filled
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int c = tid + i * F1_THREADS;
            const int op = c >> 9, r = (c >> 4) & 31, ch = c & 15;
            const int gr = r0 + kt * F1_BK + r;
            __half* dst = base + op * BW_TILE + r * BW_PITCH + ch * 8;
            if (gr < r1) {
                const __half* src;
                if (op < 2) src = gD[op] + (int64_t)gr * 128 + ch * 8;
                else src = gX[op - 2] + (int64_t)gr * ldx + min(f0 + ch * 8, ldx - 8);
                cp_async16(dst, src);
            } else {
                *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
            }
        }
    };

    float acc[2][8][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0f;

#pragma unroll
    for (int s = 0; s < F1_STAGES - 1; ++s) {
        if (s < ktiles) load_stage(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < ktiles; ++kt) {
        cp_async_wait<F1_STAGES - 2>();
        __syncthreads();
        if (kt + F1_STAGES - 1 < ktiles) load_stage((kt + F1_STAGES - 1) % F1_STAGES, kt + F1_STAGES - 1);
        cp_async_commit();
        const __half* st = smem_h + (size_t)(kt % F1_STAGES) * BW_STAGE;
        // The tensor core's fp32 accumulation truncates; over hundreds of k-tiles that bias reaches
        // ~1e-5.  Keep each MMA chain to one k-tile (6 MMAs) and add the partials in fp32 (RN) below.
        float part[2][8][4];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.0f;
#pragma unroll
        for (int kb = 0; kb < F1_BK / 16; ++kb) {
            // A(m = kk, k = r) is stored [r][kk]: transposed 8x8 loads; matrix q: k-half q>>1, m-half q&1
            uint32_t ah[2][4], al[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int kr = kb * 16 + ((lane >> 4) & 1) * 8 + (lane & 7);
                const int mc = wm * 32 + i * 16 + ((lane >> 3) & 1) * 8;
                ldsm_x4_t(ah[i], st + 0 * BW_TILE + kr * BW_PITCH + mc);
                ldsm_x4_t(al[i], st + 1 * BW_TILE + kr * BW_PITCH + mc);
            }
#pragma unroll
            for (int jp = 0; jp < 4; ++jp) {
                // B(k = r, n = f) stored [r][f]: matrix q: k-half q&1, n-half q>>1
                uint32_t bh[4], bl[4];
                const int kr = kb * 16 + ((lane >> 3) & 1) * 8 + (lane & 7);
                const int nc = wn * 64 + jp * 16 + (lane >> 4) * 8;
                ldsm_x4_t(bh, st + 2 * BW_TILE + kr * BW_PITCH + nc);
                ldsm_x4_t(bl, st + 3 * BW_TILE + kr * BW_PITCH + nc);
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    mma_f16(part[i][2 * jp], ah[i], bh[0], bh[1]);
                    mma_f16(part[i][2 * jp + 1], ah[i], bh[2], bh[3]);
                    mma_f16(part[i][2 * jp], al[i], bh[0], bh[1]);
                    mma_f16(part[i][2 * jp + 1], al[i], bh[2], bh[3]);
                    mma_f16(part[i][2 * jp], ah[i], bl[0], bl[1]);
                    mma_f16(part[i][2 * jp + 1], ah[i], bl[2], bl[3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                acc[i][j][0] += part[i][j][0]; acc[i][j][1] += part[i][j][1];
                acc[i][j][2] += part[i][j][2]; acc[i][j][3] += part[i][j][3];
            }
    }
    cp_async_wait<0>();
    // this chunk's 128 x F1_BN tile of G into its slot; the last chunk of the tile to finish adds the slots in chunk order
    const float unscale = gscale[a];
    const int gq = lane >> 2, tq = lane & 3;
    const int64_t group = (int64_t)a * gridDim.x + blockIdx.x;
    float* slot = part + (group * gridDim.y + blockIdx.y) * (128 * F1_BN);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int kk = wm * 32 + i * 16 + gq + hrow * 8;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int fl = wn * 64 + j * 8 + 2 * tq;
                *reinterpret_cast<float2*>(slot + kk * F1_BN + fl) =
                    make_float2(acc[i][j][2 * hrow] * unscale, acc[i][j][2 * hrow + 1] * unscale);
            }
        }
    if (!det_last_arrival(count + group, gridDim.y)) return;
    const float* slots = part + group * gridDim.y * (128 * F1_BN);
    for (int idx = tid; idx < 128 * F1_BN; idx += F1_THREADS) {
        const int kk = idx / F1_BN, f = f0 + idx % F1_BN;
        if (f >= ldx) continue;
        float s = 0.0f;
        for (unsigned c = 0; c < gridDim.y; ++c) s += __ldcg(slots + (int64_t)c * (128 * F1_BN) + idx);
        G[((int64_t)a * 128 + kk) * ldx + f] += s;
    }
}

}  // namespace iplan

using namespace iplan;

extern "C" int iplan_learner_x_split(const float* X, int64_t n_elems, void* Xh, void* Xl, void* stream) {
    IPLAN_REQUIRE(X && Xh && Xl && n_elems > 0 && n_elems % 2 == 0, "x_split: bad arguments");
    x_split_kernel<<<sm_count() * 8, 256, 0, (cudaStream_t)stream>>>(X, n_elems / 2, (__half2*)Xh, (__half2*)Xl);
    count_launch();
    return check_launch("x_split");
}

extern "C" int iplan_learner_fc1_forward(const float* actor, int64_t actor_stride, const float* critic, int64_t critic_stride,
                                         const void* Xh, const void* Xl, int64_t x_stride_agent, int ldx, int feat_dim,
                                         int64_t rows, int n_agents, const float* stat, void* Wh, void* Wl,
                                         float* ws, float* cc, float* Z1, void* stream) {
    IPLAN_REQUIRE(actor && critic && Xh && Xl && stat && Wh && Wl && ws && cc && Z1, "fc1_forward: null pointer");
    IPLAN_REQUIRE(ldx % F1_BK == 0 && ldx >= feat_dim, "fc1_forward: ldx must be a multiple of %d and >= feat_dim", F1_BK);
    IPLAN_REQUIRE(rows > 0 && rows < (1ll << 31), "fc1_forward: bad row count");
    cudaStream_t st = (cudaStream_t)stream;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(fc1_fwd_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FW_SMEM);
        if (e != cudaSuccess) { set_error("fc1_forward: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    NetP P{actor, critic, actor_stride, critic_stride};
    fc1_prep16_kernel<<<dim3(128, n_agents), 256, 0, st>>>(P, feat_dim, ldx, (__half*)Wh, (__half*)Wl, ws, cc);
    dim3 grid((unsigned)((rows + F1_BM - 1) / F1_BM), n_agents);
    fc1_fwd_mma_kernel<<<grid, F1_THREADS, FW_SMEM, st>>>((const __half*)Xh, (const __half*)Xl, x_stride_agent, ldx, (int)rows,
                                                           (const __half*)Wh, (const __half*)Wl, ws, cc, stat, Z1);
    count_launch(2);
    return check_launch("fc1_forward");
}

// defined in learner.cu
namespace iplan { int launch_fc1_grad_finish(const float*, int64_t, const float*, int64_t, float*, float*, int, const float*, int, const float*, int, cudaStream_t); }

extern "C" int iplan_learner_fc1_backward(const float* actor, int64_t actor_stride, const float* critic, int64_t critic_stride,
                                          float* g_actor, float* g_critic,
                                          const void* Xh, const void* Xl, int64_t x_stride_agent, int ldx, int feat_dim,
                                          int64_t rows, int n_agents,
                                          const float* dZ1, void* Dh, void* Dl, float* gscale /* [A][2] */,
                                          const float* SM, float* G, void* stream) {
    IPLAN_REQUIRE(actor && critic && g_actor && g_critic && Xh && Xl && dZ1 && Dh && Dl && gscale && SM && G, "fc1_backward: null pointer");
    IPLAN_REQUIRE(ldx % 8 == 0 && rows > 0 && rows < (1ll << 31), "fc1_backward: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(fc1_bwd_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BW_SMEM);
        if (e != cudaSuccess) { set_error("fc1_backward: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    cudaError_t e = cudaMemsetAsync(G, 0, sizeof(float) * (size_t)n_agents * 128 * ldx, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(gscale, 0, sizeof(float) * 2 * n_agents, st);
    if (e != cudaSuccess) { set_error("fc1_backward: memset: %s", cudaGetErrorString(e)); return (int)e; }
    unsigned* amax = reinterpret_cast<unsigned*>(gscale);          // [A] max bits | [A] 2^-e
    float* unscale = gscale + n_agents;
    const int64_t npa = rows * 128;
    absmax_kernel<<<dim3(sm_count(), n_agents), 256, 0, st>>>(dZ1, npa, amax);
    dz_split_kernel<<<dim3(sm_count() * 2, n_agents), 256, 0, st>>>(dZ1, npa, amax, (__half*)Dh, (__half*)Dl, unscale);
    const int chunk = 2048;
    dim3 grid((unsigned)((ldx + F1_BN - 1) / F1_BN), (unsigned)((rows + chunk - 1) / chunk), n_agents);
    const DetScratch ds = det_scratch((size_t)grid.x * grid.y * grid.z * 128 * F1_BN, (size_t)grid.x * grid.z);
    if (!ds.part) return -1;                                       // det_scratch set the error text
    fc1_bwd_mma_kernel<<<grid, F1_THREADS, BW_SMEM, st>>>((const __half*)Xh, (const __half*)Xl, x_stride_agent, ldx, (int)rows, chunk,
                                                           (const __half*)Dh, (const __half*)Dl, unscale, G, ds.part, ds.count);
    count_launch(3);
    int rc = check_launch("fc1_backward");
    if (rc) return rc;
    return launch_fc1_grad_finish(actor, actor_stride, critic, critic_stride, g_actor, g_critic, feat_dim, G, ldx, SM, n_agents, st);
}
