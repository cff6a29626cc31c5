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
// Kernel shape (both): a 128 x 128 output tile per CTA, k-tiles of 64, on the Hopper warpgroup tensor cores
// (wgmma.mma_async m64n128k16, f16 in, fp32 accumulators in registers).  One producer warp streams the four operand parts
// (A hi, A lo, B hi, B lo: 16 KB each) of every k-tile into a 3-stage ring of SWIZZLE_128B shared-memory tiles with TMA
// (cp.async.bulk.tensor, full / empty mbarriers); two consumer warpgroups each own 64 rows of the tile x all 128 columns.
//   forward   A = X rows, B = W' rows: both K-major ([row][k] in memory, one 128-row x 64-k box per part).
//   backward  A = dZ1s^T, B = X, both stored [r][.] with r = k: MN-major (transposed wgmma), two 64-r x 64-wide boxes per
//             part.
// The tensor maps are 3-D [agent][row][column], so a box reaching past the last row (or column) of an agent reads zeros,
// never the next agent's rows: ragged row counts and widths need no clamping, and the backward's sums over rows stay exact.
// Each 64-k tile runs as two MMA chains of 32 k whose fp32 partials are added in k order, and the backward sums chunks of
// 2048 rows: the same groups and order as the mma.sync kernels these replace, so the results are unchanged bit for bit.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "hopper.cuh"

namespace iplan {

constexpr int F1_BM = 128, F1_BN = 128, F1_BK = 64, F1_STAGES = 3;
constexpr int F1_THREADS = 2 * 128 + 32;                 // two consumer warpgroups + one producer warp
constexpr uint32_t F1_PART = F1_BM * F1_BK * 2;          // bytes of one f16 operand part of a k-tile (16 KB)
constexpr uint32_t F1_STAGE = 4 * F1_PART;               // A hi, A lo, B hi, B lo
constexpr size_t F1_SMEM = (size_t)F1_STAGES * F1_STAGE + 1024;   // + alignment of the base to 1024 B (swizzle atoms)

struct NetP {
    const float* actor; const float* critic; int64_t actor_stride, critic_stride;
    __device__ __forceinline__ const float* net(int a, int type) const {
        return type == 0 ? actor + a * actor_stride : critic + a * critic_stride;
    }
};

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
// the shared main loop:  C[128][128] = sum over k-tiles of A[128][64 k] . B[128][64 k]^T
// ---------------------------------------------------------------------------------------------
// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T; TRANS = 1: both operands MN-major in shared memory
template <int TRANS>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, int accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,"
                 "%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,"
                 "%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %67;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
                   "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
                   "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
                   "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
                   "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
                   "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
                   "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
                   "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(accumulate), "n"(TRANS)
                 : "memory");
}

struct F1Maps { CUtensorMap ah, al, bh, bl; };

// Runs the k-tiles [0, ktiles) of agent a.  MN = false (forward): k-tile kt is columns 64 kt.. of rows m0.. (A) and of the
// 128 W' rows (B).  MN = true (backward): k-tile kt is rows r0 + 64 kt.. ; A columns 0..127, B columns n0..n0+127.
// Returns true in the consumer threads, whose acc then holds the tile: element j of warpgroup wg's m64n128 fragment is
// (row 64 wg + 16 (warp & 3) + (lane >> 2) + 8 ((j >> 1) & 1), column 8 (j >> 2) + 2 (lane & 3) + (j & 1)).
template <bool MN>
__device__ __forceinline__ bool f1_mainloop(const F1Maps& M, int a, int m0, int n0, int ktiles, float (&acc)[64]) {
    extern __shared__ unsigned char f1_raw[];
    __shared__ __align__(8) uint64_t bars[2 * F1_STAGES];          // full[s], then empty[s]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t base = (smem_u32(f1_raw) + 1023u) & ~1023u;
    const uint32_t full = smem_u32(bars), empty = full + 8 * F1_STAGES;
    if (tid == 0) {
        for (int s = 0; s < F1_STAGES; ++s) {
            mbar_init(full + 8 * s, 1);                          // the producer's arrive + the TMA bytes
            mbar_init(empty + 8 * s, 8);                         // one arrive per consumer warp
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {                                             // ---- producer ----
        if (lane == 0) {
            tma_prefetch_desc(&M.ah); tma_prefetch_desc(&M.al); tma_prefetch_desc(&M.bh); tma_prefetch_desc(&M.bl);
            for (int kt = 0; kt < ktiles; ++kt) {
                const int s = kt % F1_STAGES;
                mbar_wait(empty + 8 * s, ((kt / F1_STAGES) & 1) ^ 1);
                const uint32_t st = base + s * F1_STAGE, bar = full + 8 * s;
                mbar_arrive_expect_tx(bar, F1_STAGE);
                if (!MN) {
                    tma_load_3d(st, &M.ah, bar, kt * F1_BK, m0, a);
                    tma_load_3d(st + F1_PART, &M.al, bar, kt * F1_BK, m0, a);
                    tma_load_3d(st + 2 * F1_PART, &M.bh, bar, kt * F1_BK, 0, a);
                    tma_load_3d(st + 3 * F1_PART, &M.bl, bar, kt * F1_BK, 0, a);
                } else {
                    const int r = m0 + kt * F1_BK;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        tma_load_3d(st + h * (F1_PART / 2), &M.ah, bar, 64 * h, r, a);
                        tma_load_3d(st + F1_PART + h * (F1_PART / 2), &M.al, bar, 64 * h, r, a);
                        tma_load_3d(st + 2 * F1_PART + h * (F1_PART / 2), &M.bh, bar, n0 + 64 * h, r, a);
                        tma_load_3d(st + 3 * F1_PART + h * (F1_PART / 2), &M.bl, bar, n0 + 64 * h, r, a);
                    }
                }
            }
        }
        return false;
    }

    // ---- consumers: warpgroup wg = rows 64 wg .. 64 wg + 63 of the tile ----
    const int wg = warp >> 2;
    // K-major: 64 rows of 128 B per warpgroup, a k-block of 16 is 32 B further.  MN-major: the 64-wide halves of a part
    // are 8 KB apart (the B operand's leading byte offset), a k-block of 16 is 16 rows of 128 B further.
    const uint32_t oa = wg * (F1_PART / 2), kstep = MN ? 2048u : 32u, lbo = MN ? F1_PART / 2 : 16u;
    float part[64];
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = part[j] = 0.0f;
    for (int kt = 0; kt < ktiles; ++kt) {
        const int s = kt % F1_STAGES;
        mbar_wait(full + 8 * s, (kt / F1_STAGES) & 1);
        const uint32_t st = base + s * F1_STAGE;
        // The tensor core's fp32 accumulation truncates; over hundreds of k-tiles that bias reaches ~1e-5.  Keep each MMA
        // chain to 32 k (hi*hi, lo*hi, hi*lo for each k-block of 16: 6 wgmmas into a fresh accumulator) and add the partials
        // in fp32 (RN) in k order.  The groups of 32 k and their order fix the rounding of the result: the fc1 weight
        // gradient is G - M, a difference of two large sums, so it shows G's rounding magnified.
        // (A second accumulator to overlap the two chains would not fit the registers of a 288-thread CTA; the other
        // consumer warpgroup's chain keeps the tensor cores busy while this one adds.)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            wgmma_fence();
#pragma unroll
            for (int kb = 2 * h; kb < 2 * h + 2; ++kb) {
                const uint64_t ah = wgmma_desc(st + oa + kb * kstep, lbo), al = wgmma_desc(st + F1_PART + oa + kb * kstep, lbo);
                const uint64_t bh = wgmma_desc(st + 2 * F1_PART + kb * kstep, lbo), bl = wgmma_desc(st + 3 * F1_PART + kb * kstep, lbo);
                wgmma_m64n128k16<MN>(part, ah, bh, kb & 1);
                wgmma_m64n128k16<MN>(part, al, bh, 1);
                wgmma_m64n128k16<MN>(part, ah, bl, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (h == 1) {
                __syncwarp();
                if (lane == 0) mbar_arrive(empty + 8 * s);
            }
#pragma unroll
            for (int j = 0; j < 64; ++j) acc[j] += part[j];
        }
    }
    return true;
}

// ---------------------------------------------------------------------------------------------
// forward:  C[128 rows][128 n] = Xtile[128][K] . W'[128 n][K]^T       (both K-contiguous)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(F1_THREADS, 1) fc1_fwd_wgmma_kernel(
    const __grid_constant__ F1Maps M, int ldx, int rows, const float* __restrict__ ws, const float* __restrict__ cc,
    const float* __restrict__ stat, float* __restrict__ Z1) {
    const int a = blockIdx.y, m0 = blockIdx.x * F1_BM;
    float acc[64];
    if (!f1_mainloop<false>(M, a, m0, 0, (ldx + F1_BK - 1) / F1_BK, acc)) return;
    // epilogue: fold the LayerNorm statistics
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gq = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
        const int r = m0 + 16 * warp + gq + hrow * 8;                 // 16 warp = 64 wg + 16 (warp & 3)
        if (r >= rows) continue;
        const float mean = stat[((int64_t)a * rows + r) * 2], rstd = stat[((int64_t)a * rows + r) * 2 + 1];
        float* zr = Z1 + ((int64_t)a * rows + r) * 128;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = j * 8 + 2 * tq;
            float2 o;
            o.x = rstd * (acc[4 * j + 2 * hrow] - mean * ws[a * 128 + n]) + cc[a * 128 + n];
            o.y = rstd * (acc[4 * j + 2 * hrow + 1] - mean * ws[a * 128 + n + 1]) + cc[a * 128 + n + 1];
            *reinterpret_cast<float2*>(zr + n) = o;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// backward:  G[128 kk][128 f] += sum_{r in chunk} dZ[r][kk] * X[r][f]    (both r-major: transposed wgmma)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(F1_THREADS, 1) fc1_bwd_wgmma_kernel(
    const __grid_constant__ F1Maps M, int ldx, int rows, int rows_per_chunk, const float* __restrict__ gscale,
    float* __restrict__ G /* [A][128][ldx] */, float* __restrict__ part /* [A][f tiles][chunks][128][F1_BN] */,
    unsigned* __restrict__ count /* [A][f tiles] */) {
    const int a = blockIdx.z, f0 = blockIdx.x * F1_BN;
    const int r0 = blockIdx.y * rows_per_chunk, r1 = min(rows, r0 + rows_per_chunk);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float acc[64];
    const bool consumer = f1_mainloop<true>(M, a, r0, f0, (r1 - r0 + F1_BK - 1) / F1_BK, acc);
    // this chunk's 128 x F1_BN tile of G into its slot; the last chunk of the tile to finish adds the slots in chunk order
    const int64_t group = (int64_t)a * gridDim.x + blockIdx.x;
    if (consumer) {
        const float unscale = gscale[a];
        const int gq = lane >> 2, tq = lane & 3;
        float* slot = part + (group * gridDim.y + blockIdx.y) * (128 * F1_BN);
#pragma unroll
        for (int hrow = 0; hrow < 2; ++hrow) {
            const int kk = 16 * warp + gq + hrow * 8;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int fl = j * 8 + 2 * tq;
                *reinterpret_cast<float2*>(slot + kk * F1_BN + fl) =
                    make_float2(acc[4 * j + 2 * hrow] * unscale, acc[4 * j + 2 * hrow + 1] * unscale);
            }
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

// ---------------------------------------------------------------------------------------------
// host: tensor maps
// ---------------------------------------------------------------------------------------------
// The driver's tensor-map encoder, looked up through the runtime so the library links no libcuda.
static PFN_cuTensorMapEncodeTiled_v12000 tmap_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    return fn;
}

// Map of the f16 tensor [d2][d1][d0] at p (d0 contiguous, d1 and d2 strides s1 and s2 elements), SWIZZLE_128B boxes of
// {box0, box1, 1}.  Maps are cached by (pointer, shape, box): the learner calls with the same buffers every epoch.
static int tmap_f16(CUtensorMap* out, const void* p, int64_t d0, int64_t d1, int64_t d2, int64_t s1, int64_t s2, int box0, int box1) {
    struct Entry { const void* p; int64_t key[7]; CUtensorMap map; };
    static Entry cache[16];
    static int n_used = 0, next = 0;
    const int64_t key[7] = {d0, d1, d2, s1, s2, box0, box1};
    for (int i = 0; i < n_used; ++i)
        if (cache[i].p == p && std::equal(key, key + 7, cache[i].key)) { *out = cache[i].map; return 0; }
    IPLAN_REQUIRE(((uintptr_t)p & 15) == 0 && s1 % 8 == 0 && s2 % 8 == 0, "fc1: f16 operands need 16-byte aligned rows");
    PFN_cuTensorMapEncodeTiled_v12000 encode = tmap_encoder();
    IPLAN_REQUIRE(encode, "fc1: cuTensorMapEncodeTiled is not available from the driver");
    const cuuint64_t dims[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
    const cuuint64_t strides[2] = {(cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2};
    const cuuint32_t box[3] = {(cuuint32_t)box0, (cuuint32_t)box1, 1}, estr[3] = {1, 1, 1};
    Entry& e = cache[next];
    const CUresult r = encode(&e.map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(p), dims, strides, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { e.p = nullptr; set_error("fc1: cuTensorMapEncodeTiled failed (%d)", (int)r); return -1; }
    e.p = p;
    std::copy(key, key + 7, e.key);
    *out = e.map;
    next = (next + 1) % 16;
    n_used = std::max(n_used, next == 0 ? 16 : next);
    return 0;
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
    IPLAN_REQUIRE(ldx % 32 == 0 && ldx >= feat_dim, "fc1_forward: ldx must be a multiple of 32 and >= feat_dim");
    IPLAN_REQUIRE(rows > 0 && rows < (1ll << 31), "fc1_forward: bad row count");
    cudaStream_t st = (cudaStream_t)stream;
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(fc1_fwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F1_SMEM);
        if (e != cudaSuccess) { set_error("fc1_forward: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    F1Maps M;
    if (tmap_f16(&M.ah, Xh, ldx, rows, n_agents, ldx, x_stride_agent, F1_BK, F1_BM) ||
        tmap_f16(&M.al, Xl, ldx, rows, n_agents, ldx, x_stride_agent, F1_BK, F1_BM) ||
        tmap_f16(&M.bh, Wh, ldx, 128, n_agents, ldx, 128ll * ldx, F1_BK, F1_BN) ||
        tmap_f16(&M.bl, Wl, ldx, 128, n_agents, ldx, 128ll * ldx, F1_BK, F1_BN))
        return -1;                                                 // tmap_f16 set the error text
    NetP P{actor, critic, actor_stride, critic_stride};
    fc1_prep16_kernel<<<dim3(128, n_agents), 256, 0, st>>>(P, feat_dim, ldx, (__half*)Wh, (__half*)Wl, ws, cc);
    dim3 grid((unsigned)((rows + F1_BM - 1) / F1_BM), n_agents);
    fc1_fwd_wgmma_kernel<<<grid, F1_THREADS, F1_SMEM, st>>>(M, ldx, (int)rows, ws, cc, stat, Z1);
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
        cudaError_t e = cudaFuncSetAttribute(fc1_bwd_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F1_SMEM);
        if (e != cudaSuccess) { set_error("fc1_backward: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    F1Maps M;
    if (tmap_f16(&M.ah, Dh, 128, rows, n_agents, 128, rows * 128, 64, F1_BK) ||
        tmap_f16(&M.al, Dl, 128, rows, n_agents, 128, rows * 128, 64, F1_BK) ||
        tmap_f16(&M.bh, Xh, ldx, rows, n_agents, ldx, x_stride_agent, 64, F1_BK) ||
        tmap_f16(&M.bl, Xl, ldx, rows, n_agents, ldx, x_stride_agent, 64, F1_BK))
        return -1;                                                 // tmap_f16 set the error text
    cudaError_t e = cudaMemsetAsync(G, 0, sizeof(float) * (size_t)n_agents * 128 * ldx, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(gscale, 0, sizeof(float) * 2 * n_agents, st);
    if (e != cudaSuccess) { set_error("fc1_backward: memset: %s", cudaGetErrorString(e)); return (int)e; }
    unsigned* amax = reinterpret_cast<unsigned*>(gscale);          // [A] max bits | [A] 2^-e
    float* unscale = gscale + n_agents;
    const int64_t npa = rows * 128;
    absmax_kernel<<<dim3(sm_count(), n_agents), 256, 0, st>>>(dZ1, npa, amax);
    dz_split_kernel<<<dim3(sm_count() * 2, n_agents), 256, 0, st>>>(dZ1, npa, amax, (__half*)Dh, (__half*)Dl, unscale);
    const unsigned ftiles = (unsigned)((ldx + F1_BN - 1) / F1_BN);
    // rows per split-K chunk (a multiple of F1_BK); it sets which rows each partial sums, and so the result's rounding
    const int chunk = 2048;
    dim3 grid(ftiles, (unsigned)((rows + chunk - 1) / chunk), n_agents);
    const DetScratch ds = det_scratch((size_t)grid.x * grid.y * grid.z * 128 * F1_BN, (size_t)grid.x * grid.z);
    if (!ds.part) return -1;                                       // det_scratch set the error text
    fc1_bwd_wgmma_kernel<<<grid, F1_THREADS, F1_SMEM, st>>>(M, ldx, (int)rows, chunk, unscale, G, ds.part, ds.count);
    count_launch(3);
    int rc = check_launch("fc1_backward");
    if (rc) return rc;
    return launch_fc1_grad_finish(actor, actor_stride, critic, critic_stride, g_actor, g_critic, feat_dim, G, ldx, SM, n_agents, st);
}
