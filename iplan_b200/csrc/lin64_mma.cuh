// Tensor-core kernels for the 64-wide layers of the actor / critic trunk (fc2: 64->64, GRU
// projections: 64->192) over row-major activation buffers [rows][64|192]:
//   lin64_rows_kernel   C[r][j] = sum_i A[r][i] * Bm[i][j] (+ bias[j])      forward (Bm = W^T) and
//                       input-gradient (Bm = W) products; one warp = 16 rows x all columns
//   lin64_dw_kernel     dW[n][k] += sum_r dY[r][n] * X[r][k]                 weight gradients;
//                       persistent CTAs accumulate over many 64-row tiles, one atomic pass at the end
// fp32 in / fp32 out; operands are split into f16 hi + lo (hi*hi + lo*hi + hi*lo on
// mma.sync.m16n8k16, fp32 accumulate, tensor-core chains <= 12 MMAs then fp32 RN adds).  The
// weight operand is split once per CTA while it is staged in shared memory; activations are
// staged as fp32 with cp.async and split in registers (each element is used by one warp only).
// Included by learner.cu INSIDE namespace iplan, after RowBuf / NetParams / NetGrads are defined
// (and after <cuda_fp16.h>).
#pragma once

#include "split_mma.cuh"

__device__ __forceinline__ void l64_cp16(void* smem, const void* gmem) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void l64_cp_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
template <int KIN, int NOUT, int ROWS, bool TRANS_W>
struct Lin64Rows {
    static constexpr int THREADS = ROWS * 2;             // one warp per 16 rows
    static constexpr int AP = KIN + 8;                   // fp32 pitch: conflict-free float2 fragment reads
    static constexpr int BP = KIN + 8;                   // f16 pitch (halves)
    static constexpr size_t SMEM = (size_t)ROWS * AP * 4 + 2 * (size_t)NOUT * BP * 2;
    static constexpr int NT = NOUT / 8, KB = KIN / 16;
};

template <int KIN, int NOUT, int ROWS, bool TRANS_W>
__global__ void __launch_bounds__(ROWS * 2) lin64_rows_kernel(RowBuf x, RowBuf y, NetParams P, int64_t w_off, int64_t b_off,
                                                               int64_t rows, int n_types) {
    using C = Lin64Rows<KIN, NOUT, ROWS, TRANS_W>;
    extern __shared__ __align__(16) unsigned char l64_smem[];
    float* As = reinterpret_cast<float*>(l64_smem);
    __half* Bh = reinterpret_cast<__half*>(l64_smem + (size_t)ROWS * C::AP * 4);
    __half* Bl = Bh + (size_t)NOUT * C::BP;
    const int a = blockIdx.y / n_types, type = blockIdx.y % n_types;
    const int64_t r_base = (int64_t)blockIdx.x * ROWS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const float* p = P.net(a, type);
    const float* W = p + w_off;

    // activations: cp.async, 16 B chunks (rows past the end re-read the last row; never stored)
    for (int c = tid; c < ROWS * (KIN / 4); c += C::THREADS) {
        const int r = c / (KIN / 4), ch = c % (KIN / 4);
        const int64_t gr = min(r_base + r, rows - 1);
        l64_cp16(As + r * C::AP + ch * 4, x.row(a, type, gr) + ch * 4);
    }
    // weights: Bt[j][i] = Bm[i][j], split into f16 hi / lo once
    for (int idx = tid; idx < NOUT * KIN; idx += C::THREADS) {
        int i, j;
        if (TRANS_W) { i = idx / NOUT; j = idx % NOUT; } else { j = idx / KIN; i = idx % KIN; }
        const float w = W[idx];
        const __half h = __float2half_rn(w);
        Bh[j * C::BP + i] = h;
        Bl[j * C::BP + i] = __float2half_rn(w - __half2float(h));
    }
    l64_cp_wait_all();
    __syncthreads();

    float acc[C::NT][4];
#pragma unroll
    for (int nt = 0; nt < C::NT; ++nt) {
        const float b0 = b_off >= 0 ? p[b_off + 8 * nt + 2 * t] : 0.0f, b1 = b_off >= 0 ? p[b_off + 8 * nt + 2 * t + 1] : 0.0f;
        acc[nt][0] = b0; acc[nt][1] = b1; acc[nt][2] = b0; acc[nt][3] = b1;
    }
    const float* a0p = As + (warp * 16 + g) * C::AP + 2 * t;
    const float* a1p = a0p + 8 * C::AP;
#pragma unroll 1
    for (int kc = 0; kc < C::KB; kc += 4) {                 // chunks of 4 k-blocks: MMA chains of 12
        float part[C::NT][4];
#pragma unroll
        for (int nt = 0; nt < C::NT; ++nt) part[nt][0] = part[nt][1] = part[nt][2] = part[nt][3] = 0.0f;
#pragma unroll
        for (int kq = 0; kq < 4; ++kq) {
            const int kb = kc + kq;
            uint32_t ah[4], al[4];
            const float2 v00 = *reinterpret_cast<const float2*>(a0p + 16 * kb);
            const float2 v10 = *reinterpret_cast<const float2*>(a1p + 16 * kb);
            const float2 v01 = *reinterpret_cast<const float2*>(a0p + 16 * kb + 8);
            const float2 v11 = *reinterpret_cast<const float2*>(a1p + 16 * kb + 8);
            l64_split(v00.x, v00.y, ah[0], al[0]);
            l64_split(v10.x, v10.y, ah[1], al[1]);
            l64_split(v01.x, v01.y, ah[2], al[2]);
            l64_split(v11.x, v11.y, ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < C::NT; ++nt) {
                const __half* bh = Bh + (8 * nt + g) * C::BP + 16 * kb + 2 * t;
                const __half* bl = Bl + (8 * nt + g) * C::BP + 16 * kb + 2 * t;
                const uint32_t bh0 = *reinterpret_cast<const uint32_t*>(bh), bh1 = *reinterpret_cast<const uint32_t*>(bh + 8);
                const uint32_t bl0 = *reinterpret_cast<const uint32_t*>(bl), bl1 = *reinterpret_cast<const uint32_t*>(bl + 8);
                l64_mma(part[nt], ah, bh0, bh1);
                l64_mma(part[nt], al, bh0, bh1);
                l64_mma(part[nt], ah, bl0, bl1);
            }
        }
#pragma unroll
        for (int nt = 0; nt < C::NT; ++nt) {
            acc[nt][0] += part[nt][0]; acc[nt][1] += part[nt][1]; acc[nt][2] += part[nt][2]; acc[nt][3] += part[nt][3];
        }
    }
    const int64_t r0 = r_base + warp * 16 + g, r1 = r0 + 8;
#pragma unroll
    for (int nt = 0; nt < C::NT; ++nt) {
        if (r0 < rows) *reinterpret_cast<float2*>(y.row(a, type, r0) + 8 * nt + 2 * t) = make_float2(acc[nt][0], acc[nt][1]);
        if (r1 < rows) *reinterpret_cast<float2*>(y.row(a, type, r1) + 8 * nt + 2 * t) = make_float2(acc[nt][2], acc[nt][3]);
    }
}

// ---------------------------------------------------------------------------------------------
template <int NO>
struct Lin64Dw {
    static constexpr int THREADS = 256, TR = 64;         // 64-row tiles
    static constexpr int DP = NO + 4, XP = 64 + 4;       // fp32 pitches: (2t*pitch) mod 32 = 8t
    static constexpr size_t SMEM = (size_t)TR * (DP + XP) * 4;
    static constexpr int MTW = NO / 64;                  // m-tiles per warp (warp grid 4 x 2)
};

// bias_off >= 0: also adds the column sums of dY (the gradient of the layer's bias) to Gr[bias_off + n].
// The CTAs of one net (blockIdx.y) store their partial sums in part[blockIdx.y][blockIdx.x][NO * 64 + NO]; the last of them to
// finish adds those in CTA order (det_last_arrival, count[blockIdx.y]).
template <int NO>
__global__ void __launch_bounds__(256) lin64_dw_kernel(RowBuf dy, RowBuf x, NetGrads Gr, int64_t w_off, int64_t rows,
                                                        int tiles_per_cta, int n_types, int64_t bias_off, float* part, unsigned* count) {
    using C = Lin64Dw<NO>;
    extern __shared__ __align__(16) unsigned char l64_smem[];
    float* Ds = reinterpret_cast<float*>(l64_smem);       // [64][DP]  dY tile
    float* Xs = Ds + C::TR * C::DP;                        // [64][XP]  X tile
    const int a = blockIdx.y / n_types, type = blockIdx.y % n_types;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int wm = warp >> 1, wn = warp & 1;               // 4 x 2 warps: (NO/4) x 32 warp tile
    const int64_t n_tiles = (rows + C::TR - 1) / C::TR;
    const int64_t t0 = (int64_t)blockIdx.x * tiles_per_cta, t1 = min(n_tiles, t0 + tiles_per_cta);

    float acc[C::MTW][4][4];
#pragma unroll
    for (int i = 0; i < C::MTW; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0f;

    float colsum = 0.0f;                                    // thread n < NO: sum_r dY[r][n] over this CTA's tiles
    for (int64_t tile = t0; tile < t1; ++tile) {
        const int64_t r_base = tile * C::TR;
        for (int c = tid; c < C::TR * (NO / 4); c += C::THREADS) {
            const int r = c / (NO / 4), ch = c % (NO / 4);
            float* dst = Ds + r * C::DP + ch * 4;
            if (r_base + r < rows) l64_cp16(dst, dy.row(a, type, r_base + r) + ch * 4);
            else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        for (int c = tid; c < C::TR * 16; c += C::THREADS) {
            const int r = c >> 4, ch = c & 15;
            float* dst = Xs + r * C::XP + ch * 4;
            if (r_base + r < rows) l64_cp16(dst, x.row(a, type, r_base + r) + ch * 4);
            else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        l64_cp_wait_all();
        __syncthreads();
        if (bias_off >= 0 && tid < NO) {
            float cs = 0.0f;
#pragma unroll 8
            for (int r = 0; r < C::TR; ++r) cs += Ds[r * C::DP + tid];
            colsum += cs;
        }
        float part[C::MTW][4][4];
#pragma unroll
        for (int i = 0; i < C::MTW; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) part[i][j][0] = part[i][j][1] = part[i][j][2] = part[i][j][3] = 0.0f;
#pragma unroll
        for (int ks = 0; ks < C::TR / 16; ++ks) {
            const int k0 = 16 * ks + 2 * t;
            uint32_t bh[4][2], bl[4][2];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = wn * 32 + 8 * j + g;
                l64_split(Xs[k0 * C::XP + n], Xs[(k0 + 1) * C::XP + n], bh[j][0], bl[j][0]);
                l64_split(Xs[(k0 + 8) * C::XP + n], Xs[(k0 + 9) * C::XP + n], bh[j][1], bl[j][1]);
            }
#pragma unroll
            for (int i = 0; i < C::MTW; ++i) {
                const int m = wm * (NO / 4) + 16 * i + g;
                uint32_t ah[4], al[4];
                l64_split(Ds[k0 * C::DP + m], Ds[(k0 + 1) * C::DP + m], ah[0], al[0]);
                l64_split(Ds[k0 * C::DP + m + 8], Ds[(k0 + 1) * C::DP + m + 8], ah[1], al[1]);
                l64_split(Ds[(k0 + 8) * C::DP + m], Ds[(k0 + 9) * C::DP + m], ah[2], al[2]);
                l64_split(Ds[(k0 + 8) * C::DP + m + 8], Ds[(k0 + 9) * C::DP + m + 8], ah[3], al[3]);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    l64_mma(part[i][j], ah, bh[j][0], bh[j][1]);
                    l64_mma(part[i][j], al, bh[j][0], bh[j][1]);
                    l64_mma(part[i][j], ah, bl[j][0], bl[j][1]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < C::MTW; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                acc[i][j][0] += part[i][j][0]; acc[i][j][1] += part[i][j][1];
                acc[i][j][2] += part[i][j][2]; acc[i][j][3] += part[i][j][3];
            }
        __syncthreads();
    }
    constexpr int V = NO * 64 + NO;
    float* slot = part + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * V;
    if (tid < NO) slot[NO * 64 + tid] = colsum;
#pragma unroll
    for (int i = 0; i < C::MTW; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = wm * (NO / 4) + 16 * i + g + ((e & 2) ? 8 : 0);
                const int n = wn * 32 + 8 * j + 2 * t + (e & 1);
                slot[m * 64 + n] = acc[i][j][e];
            }
    if (!det_last_arrival(count + blockIdx.y, gridDim.x)) return;
    const float* slots = part + (int64_t)blockIdx.y * gridDim.x * V;
    float* gw = Gr.net(a, type) + w_off;
    for (int idx = tid; idx < V; idx += C::THREADS) {
        if (idx >= NO * 64 && bias_off < 0) break;
        float s = 0.0f;
        for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(slots + (int64_t)c * V + idx);
        if (idx < NO * 64) gw[idx] += s;
        else Gr.net(a, type)[bias_off + idx - NO * 64] += s;
    }
}

// launch with the scratch of the ordered reduction
template <int NO>
int launch_lin64_dw(dim3 grid, cudaStream_t st, RowBuf dy, RowBuf x, NetGrads Gr, int64_t w_off, int64_t rows, int tiles_per_cta,
                    int n_types, int64_t bias_off = -1) {
    const DetScratch ds = det_scratch((size_t)grid.x * grid.y * (NO * 64 + NO), grid.y);
    if (!ds.part) return -1;                                      // det_scratch set the error text
    lin64_dw_kernel<NO><<<grid, 256, Lin64Dw<NO>::SMEM, st>>>(dy, x, Gr, w_off, rows, tiles_per_cta, n_types, bias_off, ds.part, ds.count);
    return 0;
}
