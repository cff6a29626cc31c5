// Behavior_policy.learn as register-tiled GEMMs (reference nova/stable_behavior_policy.py:161-279; SURVEY §8f rank 3).
//
// Same arithmetic as beh_learn.cu (the first draft, kept as the cross-check: one warp per chain, lanes = hidden units,
// 1 % of the FMA peak), organised so that the FMA pipe does the work:
//
//   * a CTA owns 64 chains (chain = one history slot of one episode of one agent-net) and walks them in lock step; every
//     GRU step is then a [64 chains] x [3H gate columns] x [K = 2H] product, computed as a register tile of 4 chains x H/16
//     hidden units per thread (all three gates of a unit in one thread, so the gate math is thread-local) against weights
//     that sit in shared memory for the CTA's lifetime ([k][gate column] fp32, row stride = 4 mod 32 so that the
//     transposed reads of the backward sweep are conflict free);
//   * activations live in [feature][chain] tiles (row stride 68 floats): a thread reads its four chains with one LDS.128;
//   * the backward sweep recomputes a window from its boundary state (kept per window position in global memory) and
//     leaves u, h, r, z, n, W_hn h (and the decoder's dropped-out output) of its W steps in an L2-resident slab; each
//     backward step is then three products: the weight gradients dW += dG^T [u | h] (48 + 48 accumulators per thread,
//     registers, for the whole kernel; flushed with one atomic per entry at the end), the data gradients [du | dh] = dG W,
//     and the small input / output layers;
//   * decoder and encoder only meet in the latent: encoder forward (latent_j for every window position j) -> decoder
//     forward + backward (loss, decoder gradients, d loss / d latent_j) -> encoder backward.  Three launches.
//
// Plain fp32 FFMA on purpose: the legacy mma.sync path would need three f16 passes per product for fp32 accuracy
// (2.5 x the FMA peak at best), a tensor-core version is the next step.
#include "common.cuh"

namespace iplan {
namespace blt {

constexpr int NT = 256;      // threads per CTA
constexpr int RC = 64;       // chains per CTA
constexpr int RS = 68;       // row stride (floats) of a [feature][chain] tile in shared memory

template <int H> struct Cfg {
    static constexpr int G = 3 * H;
    static constexpr int WS = 2 * G + 4;     // row stride of the weight tile: [k][W_ih cols | W_hh cols], = 4 (mod 32)
    static constexpr int UPT = H / 16;       // hidden units per thread in the gate / data-gradient products
    static constexpr int GPT = G / 16;       // weight-gradient tile per thread: GPT gate rows x KPT input columns
    static constexpr int KPT = H / 16;
};

__device__ __forceinline__ float sg(float x) { return 1.0f / (1.0f + expf(-x)); }

template <int N> __device__ __forceinline__ void ldv(const float* p, float (&v)[N]) {
    if constexpr (N == 4) { const float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w; }
    else if constexpr (N == 2) { const float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y; }
    else { for (int i = 0; i < N; ++i) v[i] = p[i]; }
}
__device__ __forceinline__ void ld4(const float* p, float (&v)[4]) { ldv<4>(p, v); }
__device__ __forceinline__ void st4(float* p, const float (&v)[4]) { *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]); }

struct Coord {               // thread -> (4 chains, UPT units): warp = 4 chain groups x 8 unit groups
    int c0, ug, lane, warp;
    __device__ Coord() {
        lane = threadIdx.x & 31; warp = threadIdx.x >> 5;
        const int ul = lane & 7, cl = lane >> 3, wc = warp & 3, wu = warp >> 2;
        c0 = 4 * (wc * 4 + cl); ug = wu * 8 + ul;
    }
};
// logical unit of the thread's i-th unit, and its column inside a gate block of the weight tile (a thread's units are
// adjacent columns: one vector load; its rows in the transposed read are adjacent rows: conflict free)
__device__ __forceinline__ int unit_of(int ug, int i) { return ug + 16 * i; }
template <int H> __device__ __forceinline__ int col_to_unit(int p) { return (p % Cfg<H>::UPT) * 16 + p / Cfg<H>::UPT; }

// ---- weights -> shared memory ---------------------------------------------------------------------------------------
// Wf[k][m * G + gate * H + col(unit)] = (m ? W_hh : W_ih)[gate * H + unit][k];  bias[4][H] (column order): b_r, b_z sums, b_in, b_hn
template <int H>
__device__ void stage_gru(float* Wf, float* bias, const float* __restrict__ wih, const float* __restrict__ whh,
                          const float* __restrict__ bih, const float* __restrict__ bhh) {
    constexpr int G = Cfg<H>::G, WS = Cfg<H>::WS, UPT = Cfg<H>::UPT;
    for (int idx = threadIdx.x; idx < 2 * G * H; idx += NT) {
        const int m = idx / (G * H), rem = idx - m * G * H, g = rem / H, k = rem - g * H;
        const int gate = g / H, unit = g - gate * H, col = (unit & 15) * UPT + (unit >> 4);
        Wf[k * WS + m * G + gate * H + col] = (m ? whh : wih)[rem];
    }
    for (int idx = threadIdx.x; idx < H; idx += NT) {
        const int col = (idx & 15) * UPT + (idx >> 4);
        bias[0 * H + col] = bih[idx] + bhh[idx];
        bias[1 * H + col] = bih[H + idx] + bhh[H + idx];
        bias[2 * H + col] = bih[2 * H + idx];
        bias[3 * H + col] = bhh[2 * H + idx];
    }
}

// ---- one GRU step for the thread's 4 chains x UPT units: gates from the u / h tiles ----------------------------------
template <int H>
__device__ __forceinline__ void gru_gates(const float* __restrict__ Wf, const float* __restrict__ bias, const float* __restrict__ us,
                                          const float* __restrict__ hs, const Coord& t, float (&r)[4][Cfg<H>::UPT], float (&z)[4][Cfg<H>::UPT],
                                          float (&nn)[4][Cfg<H>::UPT], float (&ghn)[4][Cfg<H>::UPT]) {
    constexpr int G = Cfg<H>::G, WS = Cfg<H>::WS, UPT = Cfg<H>::UPT;
    float ar[4][UPT], az[4][UPT], ai[4][UPT], ah[4][UPT];
#pragma unroll
    for (int i = 0; i < UPT; ++i) {
        const int col = t.ug * UPT + i;
        const float b0 = bias[col], b1 = bias[H + col], b2 = bias[2 * H + col], b3 = bias[3 * H + col];
#pragma unroll
        for (int c = 0; c < 4; ++c) { ar[c][i] = b0; az[c][i] = b1; ai[c][i] = b2; ah[c][i] = b3; }
    }
    const float* wrow = Wf + t.ug * UPT;
#pragma unroll 4
    for (int k = 0; k < H; ++k) {
        float uv[4], hv[4], wir[UPT], wiz[UPT], win[UPT], whr[UPT], whz[UPT], whn[UPT];
        ld4(us + k * RS + t.c0, uv); ld4(hs + k * RS + t.c0, hv);
        const float* w = wrow + k * WS;
        ldv<UPT>(w, wir); ldv<UPT>(w + H, wiz); ldv<UPT>(w + 2 * H, win);
        ldv<UPT>(w + G, whr); ldv<UPT>(w + G + H, whz); ldv<UPT>(w + G + 2 * H, whn);
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int i = 0; i < UPT; ++i) {
                ar[c][i] = fmaf(uv[c], wir[i], fmaf(hv[c], whr[i], ar[c][i]));
                az[c][i] = fmaf(uv[c], wiz[i], fmaf(hv[c], whz[i], az[c][i]));
                ai[c][i] = fmaf(uv[c], win[i], ai[c][i]);
                ah[c][i] = fmaf(hv[c], whn[i], ah[c][i]);
            }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int i = 0; i < UPT; ++i) {
            r[c][i] = sg(ar[c][i]); z[c][i] = sg(az[c][i]); ghn[c][i] = ah[c][i];
            nn[c][i] = tanhf(ai[c][i] + r[c][i] * ah[c][i]);
        }
}

// ---- data gradients: du[c][unit] = sum_g dgi[g][c] W_ih[g][unit], dhp likewise with dgh and W_hh ---------------------
// DG tile rows (column order): [0,H) d a_r, [H,2H) d a_z, [2H,3H) d a_n (input side), [3H,4H) d a_n * r (hidden side)
template <int H>
__device__ __forceinline__ void gru_bwd_data(const float* __restrict__ Wf, const float* __restrict__ DG, const Coord& t,
                                             float (&du)[4][Cfg<H>::UPT], float (&dhp)[4][Cfg<H>::UPT]) {
    constexpr int G = Cfg<H>::G, WS = Cfg<H>::WS, UPT = Cfg<H>::UPT;
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int i = 0; i < UPT; ++i) { du[c][i] = 0.0f; dhp[c][i] = 0.0f; }
    for (int g4 = 0; g4 < G; g4 += 4) {
        const bool ngate = g4 >= 2 * H;                       // uniform
        float d[4][4], dn[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            ld4(DG + (g4 + q) * RS + t.c0, d[q]);
            if (ngate) ld4(DG + (g4 + q + H) * RS + t.c0, dn[q]);
            else { dn[q][0] = d[q][0]; dn[q][1] = d[q][1]; dn[q][2] = d[q][2]; dn[q][3] = d[q][3]; }
        }
#pragma unroll
        for (int i = 0; i < UPT; ++i) {
            float wi[4], wh[4];
            const float* w = Wf + unit_of(t.ug, i) * WS + g4;
            ld4(w, wi); ld4(w + G, wh);
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    du[c][i] = fmaf(d[q][c], wi[q], du[c][i]);
                    dhp[c][i] = fmaf(dn[q][c], wh[q], dhp[c][i]);
                }
        }
    }
}

// ---- weight gradients: aih[g][k] += sum_c dgi[g][c] u[k][c]; ahh[g][k] += sum_c dgh[g][c] hp[k][c] --------------------
// thread -> gate rows gb * GPT + i (column order), input columns kg + 16 j
template <int H>
__device__ __forceinline__ void gru_dw(const float* __restrict__ DG, const float* __restrict__ us, const float* __restrict__ hps, const Coord& t,
                                       float (&aih)[Cfg<H>::GPT][Cfg<H>::KPT], float (&ahh)[Cfg<H>::GPT][Cfg<H>::KPT]) {
    constexpr int GPT = Cfg<H>::GPT, KPT = Cfg<H>::KPT;
    const int kg = t.lane & 15, gb = t.warp * 2 + (t.lane >> 4);
#pragma unroll 1
    for (int c4 = 0; c4 < RC; c4 += 4) {
        float xu[KPT][4], xh[KPT][4];
#pragma unroll
        for (int j = 0; j < KPT; ++j) { ld4(us + (kg + 16 * j) * RS + c4, xu[j]); ld4(hps + (kg + 16 * j) * RS + c4, xh[j]); }
#pragma unroll
        for (int i = 0; i < GPT; ++i) {
            const int g = gb * GPT + i;
            float di[4], dh[4];
            ld4(DG + g * RS + c4, di);
            ld4(DG + (g < 2 * H ? g : g + H) * RS + c4, dh);
#pragma unroll
            for (int j = 0; j < KPT; ++j) {
                float s = aih[i][j], v = ahh[i][j];
#pragma unroll
                for (int c = 0; c < 4; ++c) { s = fmaf(di[c], xu[j][c], s); v = fmaf(dh[c], xh[j][c], v); }
                aih[i][j] = s; ahh[i][j] = v;
            }
        }
    }
}

template <int H>
__device__ void flush_dw(const float (&aih)[Cfg<H>::GPT][Cfg<H>::KPT], const float (&ahh)[Cfg<H>::GPT][Cfg<H>::KPT], const Coord& t,
                         float* __restrict__ Gih, float* __restrict__ Ghh) {
    constexpr int GPT = Cfg<H>::GPT, KPT = Cfg<H>::KPT;
    const int kg = t.lane & 15, gb = t.warp * 2 + (t.lane >> 4);
#pragma unroll
    for (int i = 0; i < GPT; ++i) {
        const int g = gb * GPT + i, gate = g / H, unit = col_to_unit<H>(g - gate * H);
#pragma unroll
        for (int j = 0; j < KPT; ++j) {
            const int k = kg + 16 * j;
            atomicAdd(Gih + (gate * H + unit) * H + k, aih[i][j]);
            atomicAdd(Ghh + (gate * H + unit) * H + k, ahh[i][j]);
        }
    }
}

// ---- tile copies: global [rows][64] <-> shared [rows][RS] ------------------------------------------------------------
__device__ __forceinline__ void tile_g2s(float* s, const float* __restrict__ g, int rows) {
    for (int idx = threadIdx.x; idx < rows * (RC / 4); idx += NT) {
        const int row = idx >> 4, q = idx & 15;
        *reinterpret_cast<float4*>(s + row * RS + 4 * q) = *reinterpret_cast<const float4*>(g + row * RC + 4 * q);
    }
}
__device__ __forceinline__ void tile_s2g(float* __restrict__ g, const float* s, int rows) {
    for (int idx = threadIdx.x; idx < rows * (RC / 4); idx += NT) {
        const int row = idx >> 4, q = idx & 15;
        *reinterpret_cast<float4*>(g + row * RC + 4 * q) = *reinterpret_cast<const float4*>(s + row * RS + 4 * q);
    }
}
__device__ __forceinline__ void tile_zero(float* s, int rows) {
    for (int idx = threadIdx.x; idx < rows * RS; idx += NT) s[idx] = 0.0f;
}

// sum over the tile's 64 chains of row `row` (x optionally another row)
__device__ __forceinline__ float row_sum(const float* a) {
    float s = 0.0f;
#pragma unroll 4
    for (int c = 0; c < RC; c += 4) { float v[4]; ld4(a + c, v); s += (v[0] + v[1]) + (v[2] + v[3]); }
    return s;
}
__device__ __forceinline__ float row_dot(const float* a, const float* b) {
    float s = 0.0f;
#pragma unroll 4
    for (int c = 0; c < RC; c += 4) {
        float v[4], w[4]; ld4(a + c, v); ld4(b + c, w);
        s = fmaf(v[0], w[0], s); s = fmaf(v[1], w[1], s); s = fmaf(v[2], w[2], s); s = fmaf(v[3], w[3], s);
    }
    return s;
}

struct Args {
    const float* enc; int64_t enc_stride; const float* dec; int64_t dec_stride;
    float* g_enc; float* g_dec;
    const float* hist;        // [A][B][T][N][o]
    const float* mask;        // [A][B][T]
    const float* scale;       // [A][n_pos]
    const uint8_t* keep;      // NULL (Philox) or [A][B][n_pos][N][W][64]
    float* b_loss; float* s_loss;
    float* lat_all;           // [A][tiles][n_pos + 1][L][64]   latent_j per window position (encoder forward)
    float* znew;              // [A][tiles][n_pos][L][64]       soft-max outputs z_j
    float* eh_b;              // [A][tiles][n_pos + 1][32][64]  encoder hidden at window boundaries
    float* dh_b;              // [A][tiles][n_pos][64][64]      decoder hidden at window boundaries
    float* dlat;              // [A][tiles][n_pos][L][64]       d loss / d latent_j through the decoder input
    float* slab;              // [A][tiles][W][slab rows][64]   the window being back-propagated
    uint64_t seed, counter; float p_drop, coef, thres, stab_scale;
    int B, T, N, o, L, W, n_pos, tiles;
};

constexpr int HE = IPLAN_HID, HD = IPLAN_RNN;
// slab rows per step
constexpr int D_U = 0, D_H = 64, D_R = 128, D_Z = 192, D_N = 256, D_GH = 320, D_Y = 384, D_P = 448, D_ROWS = 456;
constexpr int E_U = 0, E_H = 32, E_R = 64, E_Z = 96, E_N = 128, E_GH = 160, E_ROWS = 192;

// chain bookkeeping of a tile (shared memory): offset of hist[b][0][n][0] inside the agent's block, of mask[b][0], validity
struct ChainInfo { int hoff[RC]; int moff[RC]; int gid[RC]; };      // gid = (ag * B + b) * N + n, -1 if the chain does not exist

__device__ void chain_setup(ChainInfo* ci, const Args& a, int tile, int ag) {
    for (int c = threadIdx.x; c < RC; c += NT) {
        const int q = tile * RC + c;
        if (q < a.B * a.N) {
            const int b = q / a.N, n = q - b * a.N;
            ci->hoff[c] = (b * a.T * a.N + n) * a.o; ci->moff[c] = b * a.T; ci->gid[c] = (ag * a.B + b) * a.N + n;
        } else { ci->hoff[c] = 0; ci->moff[c] = 0; ci->gid[c] = -1; }
    }
}

// rows 0..o-1 of the input tile: history step t of every chain (zeros before the episode start and for missing chains)
__device__ __forceinline__ void load_hist_rows(float* xin, const float* __restrict__ hist, const ChainInfo* ci, int t, int N, int o) {
    for (int idx = threadIdx.x; idx < RC * o; idx += NT) {
        const int c = idx / o, kk = idx - c * o;
        xin[kk * RS + c] = (t >= 0 && ci->gid[c] >= 0) ? hist[ci->hoff[c] + (int64_t)t * N * o + kk] : 0.0f;
    }
}

// u[unit][chain] = ReLU(b[unit] + sum_kk w[kk][unit] x[kk][chain]) for the thread's pairs; lw = [kk][H] in shared memory
template <int H>
__device__ __forceinline__ void input_layer(float* us, const float* xin, const float* lw, const float* lb, int in_d, const Coord& t) {
    constexpr int UPT = Cfg<H>::UPT;
    float acc[UPT][4];
#pragma unroll
    for (int i = 0; i < UPT; ++i) { const float b = lb[unit_of(t.ug, i)]; for (int c = 0; c < 4; ++c) acc[i][c] = b; }
    for (int kk = 0; kk < in_d; ++kk) {
        float x[4]; ld4(xin + kk * RS + t.c0, x);
#pragma unroll
        for (int i = 0; i < UPT; ++i) {
            const float w = lw[kk * H + unit_of(t.ug, i)];
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[i][c] = fmaf(w, x[c], acc[i][c]);
        }
    }
#pragma unroll
    for (int i = 0; i < UPT; ++i) {
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[i][c] = fmaxf(acc[i][c], 0.0f);
        st4(us + unit_of(t.ug, i) * RS + t.c0, acc[i]);
    }
}

// gate derivatives for the thread's pairs -> DG tile; returns dh * z in dhz
template <int H>
__device__ __forceinline__ void gate_derivs(float* DG, const Coord& t, const float (&dh)[4][Cfg<H>::UPT], const float* __restrict__ sr, const float* __restrict__ sz,
                                            const float* __restrict__ sn, const float* __restrict__ sgh, const float* __restrict__ shp, float (&dhz)[4][Cfg<H>::UPT]) {
    constexpr int UPT = Cfg<H>::UPT;
#pragma unroll
    for (int i = 0; i < UPT; ++i) {
        const int un = unit_of(t.ug, i), col = t.ug * UPT + i;
        float r[4], z[4], n[4], gh[4], hp[4], dar[4], daz[4], dan[4], dnr[4];
        ld4(sr + un * RC + t.c0, r); ld4(sz + un * RC + t.c0, z); ld4(sn + un * RC + t.c0, n); ld4(sgh + un * RC + t.c0, gh); ld4(shp + un * RC + t.c0, hp);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const float d = dh[c][i];
            const float dn = d * (1.0f - z[c]), dz = d * (hp[c] - n[c]);
            dan[c] = dn * (1.0f - n[c] * n[c]); daz[c] = dz * z[c] * (1.0f - z[c]); dar[c] = dan[c] * gh[c] * r[c] * (1.0f - r[c]);
            dnr[c] = dan[c] * r[c];
            dhz[c][i] = d * z[c];
        }
        st4(DG + col * RS + t.c0, dar); st4(DG + (H + col) * RS + t.c0, daz); st4(DG + (2 * H + col) * RS + t.c0, dan); st4(DG + (3 * H + col) * RS + t.c0, dnr);
    }
}

// =====================================================================================================================
// encoder
// =====================================================================================================================
struct EncSmem {             // offsets in floats
    static constexpr int WF = 0, BIAS = WF + HE * Cfg<HE>::WS, LW = BIAS + 4 * HE, LB = LW + 8 * HE, OW = LB + HE, OB = OW + 8 * HE,
                         CI = OB + 8, XIN = CI + 3 * RC, U = XIN + 8 * RS, HA = U + HE * RS, HB = HA + HE * RS, P = HB + HE * RS, LG = P + HE * RS,
                         DG = LG + 8 * RS, TOTAL = DG + 4 * HE * RS;
};

__device__ void enc_stage(float* sm, const float* __restrict__ We, const BehLayout& E, int o, int L) {
    stage_gru<HE>(sm + EncSmem::WF, sm + EncSmem::BIAS, We + E.wih, We + E.whh, We + E.bih, We + E.bhh);
    for (int idx = threadIdx.x; idx < 8 * HE; idx += NT) {
        const int kk = idx / HE, un = idx - kk * HE;
        sm[EncSmem::LW + idx] = kk < o ? We[E.lin_w + un * o + kk] : 0.0f;
        sm[EncSmem::OW + idx] = kk < L ? We[E.out_w + kk * HE + un] : 0.0f;          // [l][k]
    }
    for (int idx = threadIdx.x; idx < HE; idx += NT) sm[EncSmem::LB + idx] = We[E.lin_b + idx];
    for (int idx = threadIdx.x; idx < 8; idx += NT) sm[EncSmem::OB + idx] = idx < L ? We[E.out_b + idx] : 0.0f;
}

// the W steps of window position j from the boundary state in `hcur`; optionally leaves u, h, r, z, n, W_hn h in the slab.
// Returns the buffer that holds the hidden state after the last step.
template <bool STORE>
__device__ float* enc_window(float* sm, const Args& a, const float* __restrict__ hist, const ChainInfo* ci, const Coord& t, int j, float* hcur,
                             float* __restrict__ slab) {
    float* xin = sm + EncSmem::XIN; float* us = sm + EncSmem::U;
    float* hnext = hcur == sm + EncSmem::HA ? sm + EncSmem::HB : sm + EncSmem::HA;
    for (int w = 0; w < a.W; ++w) {
        load_hist_rows(xin, hist, ci, j - a.W + 1 + w, a.N, a.o);
        __syncthreads();
        input_layer<HE>(us, xin, sm + EncSmem::LW, sm + EncSmem::LB, a.o, t);
        __syncthreads();
        float r[4][2], z[4][2], nn[4][2], gh[4][2];
        gru_gates<HE>(sm + EncSmem::WF, sm + EncSmem::BIAS, us, hcur, t, r, z, nn, gh);
        float* sl = slab + (int64_t)w * E_ROWS * RC;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int un = unit_of(t.ug, i);
            float hp[4], hn[4]; ld4(hcur + un * RS + t.c0, hp);
#pragma unroll
            for (int c = 0; c < 4; ++c) hn[c] = (1.0f - z[c][i]) * nn[c][i] + z[c][i] * hp[c];
            st4(hnext + un * RS + t.c0, hn);
            if (STORE) {
                float v[4];
                st4(sl + (E_H + un) * RC + t.c0, hn);
                for (int c = 0; c < 4; ++c) v[c] = r[c][i]; st4(sl + (E_R + un) * RC + t.c0, v);
                for (int c = 0; c < 4; ++c) v[c] = z[c][i]; st4(sl + (E_Z + un) * RC + t.c0, v);
                for (int c = 0; c < 4; ++c) v[c] = nn[c][i]; st4(sl + (E_N + un) * RC + t.c0, v);
                for (int c = 0; c < 4; ++c) v[c] = gh[c][i]; st4(sl + (E_GH + un) * RC + t.c0, v);
                ld4(us + un * RS + t.c0, v); st4(sl + (E_U + un) * RC + t.c0, v);
            }
        }
        __syncthreads();
        float* tmp = hcur; hcur = hnext; hnext = tmp;
    }
    return hcur;
}

__global__ void __launch_bounds__(NT, 2) enc_fwd_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    const int tile = blockIdx.x, ag = blockIdx.y, tid = threadIdx.x;
    const Coord t;
    const BehLayout E = beh_layout(a.o, a.L);
    const int L = a.L, NP = a.n_pos;
    ChainInfo* ci = reinterpret_cast<ChainInfo*>(sm + EncSmem::CI);
    enc_stage(sm, a.enc + (int64_t)ag * a.enc_stride, E, a.o, L);
    chain_setup(ci, a, tile, ag);
    const float* hist = a.hist + (int64_t)ag * a.B * a.T * a.N * a.o;
    const int64_t tl = (int64_t)ag * a.tiles + tile;
    float* lat_all = a.lat_all + tl * (NP + 1) * L * RC;
    float* znew = a.znew + tl * NP * L * RC;
    float* eh_b = a.eh_b + tl * (NP + 1) * HE * RC;
    float* hcur = sm + EncSmem::HA;
    tile_zero(hcur, HE);
    float lat[8];                                               // thread c < 64: the chain's latent
#pragma unroll
    for (int l = 0; l < 8; ++l) lat[l] = 0.0f;
    if (tid < RC) for (int l = 0; l < L; ++l) lat_all[l * RC + tid] = 0.0f;
    __syncthreads();
    for (int j = 0; j < NP; ++j) {
        tile_s2g(eh_b + (int64_t)j * HE * RC, hcur, HE);
        hcur = enc_window<false>(sm, a, hist, ci, t, j, hcur, a.slab);
        // latent head: logits[l][c] = b[l] + sum_k out_w[l][k] h[k][c]
        {
            const int c = tid & 63, q = tid >> 6;
            float s0 = sm[EncSmem::OB + 2 * q], s1 = sm[EncSmem::OB + 2 * q + 1];
            for (int k = 0; k < HE; ++k) {
                const float hv = hcur[k * RS + c];
                s0 = fmaf(sm[EncSmem::OW + (2 * q) * HE + k], hv, s0);
                s1 = fmaf(sm[EncSmem::OW + (2 * q + 1) * HE + k], hv, s1);
            }
            sm[EncSmem::LG + (2 * q) * RS + c] = s0; sm[EncSmem::LG + (2 * q + 1) * RS + c] = s1;
        }
        __syncthreads();
        if (tid < RC) {
            float lg[8], mx = -INFINITY, den = 0.0f;
#pragma unroll
            for (int l = 0; l < 8; ++l) { lg[l] = l < L ? sm[EncSmem::LG + l * RS + tid] : -INFINITY; mx = fmaxf(mx, lg[l]); }
#pragma unroll
            for (int l = 0; l < 8; ++l) { lg[l] = l < L ? expf(lg[l] - mx) : 0.0f; den += lg[l]; }
#pragma unroll
            for (int l = 0; l < 8; ++l)
                if (l < L) {
                    const float zl = lg[l] / den;
                    znew[((int64_t)j * L + l) * RC + tid] = zl;
                    lat[l] = (1.0f - a.coef) * lat[l] + zl * a.coef;
                    lat_all[((int64_t)(j + 1) * L + l) * RC + tid] = lat[l];
                }
        }
        __syncthreads();
    }
    tile_s2g(eh_b + (int64_t)NP * HE * RC, hcur, HE);
}

__global__ void __launch_bounds__(NT, 2) enc_bwd_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    const int tile = blockIdx.x, ag = blockIdx.y, tid = threadIdx.x;
    const Coord t;
    const BehLayout E = beh_layout(a.o, a.L);
    const int L = a.L, NP = a.n_pos, W = a.W, o = a.o;
    ChainInfo* ci = reinterpret_cast<ChainInfo*>(sm + EncSmem::CI);
    enc_stage(sm, a.enc + (int64_t)ag * a.enc_stride, E, o, L);
    chain_setup(ci, a, tile, ag);
    const float* hist = a.hist + (int64_t)ag * a.B * a.T * a.N * a.o;
    const int64_t tl = (int64_t)ag * a.tiles + tile;
    const float* znew = a.znew + tl * NP * L * RC;
    const float* eh_b = a.eh_b + tl * (NP + 1) * HE * RC;
    const float* dlat = a.dlat + tl * NP * L * RC;
    float* slab = a.slab + tl * W * D_ROWS * RC;                 // the decoder's slab, free again
    float* DG = sm + EncSmem::DG; float* us = sm + EncSmem::U; float* P = sm + EncSmem::P; float* xin = sm + EncSmem::XIN; float* LG = sm + EncSmem::LG;

    float aih[Cfg<HE>::GPT][Cfg<HE>::KPT], ahh[Cfg<HE>::GPT][Cfg<HE>::KPT];
#pragma unroll
    for (int i = 0; i < Cfg<HE>::GPT; ++i)
#pragma unroll
        for (int jx = 0; jx < Cfg<HE>::KPT; ++jx) { aih[i][jx] = 0.0f; ahh[i][jx] = 0.0f; }
    float g_bias = 0.0f;                 // thread tid < 128: column sum of DG row tid
    float g_ow = 0.0f;                   // thread: out_w[l = tid / 32][k = tid % 32]
    float g_ob = 0.0f;                   // tid < 8
    float g_lw = 0.0f;                   // tid < 32 * o: lin_w[unit = tid % 32][kk = tid / 32]
    float g_lb = 0.0f;                   // tid < 32
    float c_lat[8];                      // tid < 64: d loss / d latent_{j+1} of chain tid
#pragma unroll
    for (int l = 0; l < 8; ++l) c_lat[l] = 0.0f;
    float deh[4][2];                     // d loss / d (encoder hidden after window j), carried
#pragma unroll
    for (int c = 0; c < 4; ++c) { deh[c][0] = 0.0f; deh[c][1] = 0.0f; }
    __syncthreads();

    for (int j = NP - 1; j >= 0; --j) {
        float* hcur = sm + EncSmem::HA;
        tile_g2s(hcur, eh_b + (int64_t)j * HE * RC, HE);
        __syncthreads();
        hcur = enc_window<true>(sm, a, hist, ci, t, j, hcur, slab);          // ends with a barrier; hcur = hidden after the window
        // ---- latent recursion and soft-max head -------------------------------------------------------------------
        if (tid < RC) {
            float zl[8], dnl[8], dot = 0.0f;
#pragma unroll
            for (int l = 0; l < 8; ++l)
                if (l < L) {
                    zl[l] = znew[((int64_t)j * L + l) * RC + tid];
                    dnl[l] = a.coef * c_lat[l];
                    c_lat[l] = (1.0f - a.coef) * c_lat[l] + dlat[((int64_t)j * L + l) * RC + tid];
                    dot = fmaf(zl[l], dnl[l], dot);
                }
#pragma unroll
            for (int l = 0; l < 8; ++l) LG[l * RS + tid] = l < L ? zl[l] * (dnl[l] - dot) : 0.0f;
        }
        __syncthreads();
        {   // out_w / out_b gradients, and the head's contribution to deh
            const int l = tid >> 5, k = tid & 31;
            if (l < L) g_ow += row_dot(LG + l * RS, hcur + k * RS);
            if (tid < L) g_ob += row_sum(LG + tid * RS);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int un = unit_of(t.ug, i);
                for (int ll = 0; ll < L; ++ll) {
                    float d[4]; ld4(LG + ll * RS + t.c0, d);
                    const float wv = sm[EncSmem::OW + ll * HE + un];
#pragma unroll
                    for (int c = 0; c < 4; ++c) deh[c][i] = fmaf(d[c], wv, deh[c][i]);
                }
            }
        }
        // ---- BPTT through the window ----------------------------------------------------------------------------------
        for (int w = W - 1; w >= 0; --w) {
            const float* sl = slab + (int64_t)w * E_ROWS * RC;
            const float* hp_g = w > 0 ? slab + (int64_t)(w - 1) * E_ROWS * RC + E_H * RC : eh_b + (int64_t)j * HE * RC;
            float dhz[4][2];
            gate_derivs<HE>(DG, t, deh, sl + E_R * RC, sl + E_Z * RC, sl + E_N * RC, sl + E_GH * RC, hp_g, dhz);
            tile_g2s(us, sl + E_U * RC, HE);
            tile_g2s(P, hp_g, HE);
            load_hist_rows(xin, hist, ci, j - W + 1 + w, a.N, o);
            __syncthreads();
            gru_dw<HE>(DG, us, P, t, aih, ahh);
            float du[4][2], dhp[4][2];
            gru_bwd_data<HE>(sm + EncSmem::WF, DG, t, du, dhp);
            if (tid < 4 * HE) g_bias += row_sum(DG + tid * RS);
            float dli[2][4];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float uv[4]; ld4(us + unit_of(t.ug, i) * RS + t.c0, uv);
#pragma unroll
                for (int c = 0; c < 4; ++c) { dli[i][c] = uv[c] > 0.0f ? du[c][i] : 0.0f; deh[c][i] = dhz[c][i] + dhp[c][i]; }
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < 2; ++i) st4(us + unit_of(t.ug, i) * RS + t.c0, dli[i]);
            __syncthreads();
            if (tid < HE * o) g_lw += row_dot(us + (tid & 31) * RS, xin + (tid >> 5) * RS);
            if (tid < HE) g_lb += row_sum(us + tid * RS);
            __syncthreads();
        }
    }
    // ---- flush -----------------------------------------------------------------------------------------------------------
    float* Ge = a.g_enc + (int64_t)ag * a.enc_stride;
    flush_dw<HE>(aih, ahh, t, Ge + E.wih, Ge + E.whh);
    if (tid < 4 * HE) {
        const int blk = tid / HE, unit = col_to_unit<HE>(tid % HE);
        if (blk < 2) { atomicAdd(Ge + E.bih + blk * HE + unit, g_bias); atomicAdd(Ge + E.bhh + blk * HE + unit, g_bias); }
        else if (blk == 2) atomicAdd(Ge + E.bih + 2 * HE + unit, g_bias);
        else atomicAdd(Ge + E.bhh + 2 * HE + unit, g_bias);
    }
    if ((tid >> 5) < L) atomicAdd(Ge + E.out_w + (tid >> 5) * HE + (tid & 31), g_ow);
    if (tid < L) atomicAdd(Ge + E.out_b + tid, g_ob);
    if (tid < HE * o) atomicAdd(Ge + E.lin_w + (tid & 31) * o + (tid >> 5), g_lw);
    if (tid < HE) atomicAdd(Ge + E.lin_b + tid, g_lb);
}

// =====================================================================================================================
// decoder
// =====================================================================================================================
struct BDecLayout { int64_t lin_w, lin_b, wih, whh, bih, bhh, out_w, out_b, total; };
__host__ __device__ inline BDecLayout bdec_layout(int o, int Ld) {
    BDecLayout L;
    int64_t off = 0;
    auto take = [&](int64_t n) { int64_t at = off; off = pad4(off + n); return at; };
    L.lin_w = take((int64_t)HD * (o + Ld)); L.lin_b = take(HD);
    L.wih = take(3 * HD * HD); L.whh = take(3 * HD * HD); L.bih = take(3 * HD); L.bhh = take(3 * HD);
    L.out_w = take((int64_t)o * HD); L.out_b = take(o);
    L.total = off;
    return L;
}

struct DecSmem {
    static constexpr int WF = 0, BIAS = WF + HD * Cfg<HD>::WS, LW = BIAS + 4 * HD, LB = LW + 16 * HD, OW = LB + HD, OB = OW + 8 * HD,
                         CI = OB + 8, XIN = CI + 3 * RC, U = XIN + 16 * RS, P = U + HD * RS, PART = P + HD * RS, DPR = PART + 32 * RS,
                         OVER = DPR + 8 * RS, HA = OVER, HB = HA + HD * RS, DG = OVER, TOTAL = OVER + 4 * HD * RS;
};

// one Philox call per (chain, position, step, unit group): components 0..3 = units ug, ug + 16, ug + 32, ug + 48
__device__ __forceinline__ void keep_bits(const Args& a, const ChainInfo* ci, const Coord& t, int j, int w, bool (&kp)[4][4]) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const int gid = ci->gid[t.c0 + c];
        if (gid < 0) { for (int i = 0; i < 4; ++i) kp[c][i] = false; continue; }
        if (a.keep) {
            const uint8_t* k = a.keep + ((((int64_t)(gid / a.N) * a.n_pos + j) * a.N + gid % a.N) * a.W + w) * HD;
#pragma unroll
            for (int i = 0; i < 4; ++i) kp[c][i] = k[unit_of(t.ug, i)] != 0;
        } else {
            const uint64_t e = (((uint64_t)gid * a.n_pos + j) * a.W + w) * 16 + t.ug;
            const uint4 rnd = philox4x32(make_uint4((uint32_t)e, (uint32_t)(e >> 32), (uint32_t)a.counter, (uint32_t)(a.counter >> 32)),
                                         make_uint2((uint32_t)a.seed ^ 0x85ebca6bu, (uint32_t)(a.seed >> 32)));
            kp[c][0] = u01(rnd.x) >= a.p_drop; kp[c][1] = u01(rnd.y) >= a.p_drop; kp[c][2] = u01(rnd.z) >= a.p_drop; kp[c][3] = u01(rnd.w) >= a.p_drop;
        }
    }
}

// decoder input tile of (position j, step w): rows 0..o-1 the window row, rows o..o+L-1 latent_j
__device__ __forceinline__ void dec_input(float* xin, const Args& a, const float* __restrict__ hist, const float* __restrict__ lat_j, const ChainInfo* ci, int j, int w) {
    load_hist_rows(xin, hist, ci, j - a.W + 1 + w, a.N, a.o);
    for (int idx = threadIdx.x; idx < a.L * RC; idx += NT) {
        const int l = idx >> 6, c = idx & 63;
        xin[(a.o + l) * RS + c] = lat_j[idx];
    }
}

// the W steps of window position j.  LOSS: accumulate the reconstruction / stability terms; STORE: leave the step's state in the slab.
template <bool LOSS, bool STORE>
__device__ float* dec_window(float* sm, const Args& a, const float* __restrict__ hist, const float* __restrict__ mask, const float* __restrict__ lat_j,
                             const ChainInfo* ci, const Coord& t, int j, float scale_j, float* hcur, float* __restrict__ slab, float& bl, float& sl_acc) {
    float* xin = sm + DecSmem::XIN; float* us = sm + DecSmem::U; float* ys = sm + DecSmem::P; float* part = sm + DecSmem::PART;
    float* hnext = hcur == sm + DecSmem::HA ? sm + DecSmem::HB : sm + DecSmem::HA;
    const float ks = 1.0f / (1.0f - a.p_drop);
    const int tid = threadIdx.x, o = a.o, in_d = a.o + a.L;
    for (int w = 0; w < a.W; ++w) {
        dec_input(xin, a, hist, lat_j, ci, j, w);
        __syncthreads();
        input_layer<HD>(us, xin, sm + DecSmem::LW, sm + DecSmem::LB, in_d, t);
        __syncthreads();
        float r[4][4], z[4][4], nn[4][4], gh[4][4];
        gru_gates<HD>(sm + DecSmem::WF, sm + DecSmem::BIAS, us, hcur, t, r, z, nn, gh);
        bool kp[4][4];
        keep_bits(a, ci, t, j, w, kp);
        float* sl = slab + (int64_t)w * D_ROWS * RC;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int un = unit_of(t.ug, i);
            float hp[4], hn[4], y[4]; ld4(hcur + un * RS + t.c0, hp);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                hn[c] = (1.0f - z[c][i]) * nn[c][i] + z[c][i] * hp[c];
                y[c] = kp[c][i] ? tanhf(hn[c]) * ks : 0.0f;
            }
            st4(hnext + un * RS + t.c0, hn);
            st4(ys + un * RS + t.c0, y);
            if (STORE) {
                float v[4];
                st4(sl + (D_H + un) * RC + t.c0, hn); st4(sl + (D_Y + un) * RC + t.c0, y);
                for (int c = 0; c < 4; ++c) v[c] = r[c][i]; st4(sl + (D_R + un) * RC + t.c0, v);
                for (int c = 0; c < 4; ++c) v[c] = z[c][i]; st4(sl + (D_Z + un) * RC + t.c0, v);
                for (int c = 0; c < 4; ++c) v[c] = nn[c][i]; st4(sl + (D_N + un) * RC + t.c0, v);
                for (int c = 0; c < 4; ++c) v[c] = gh[c][i]; st4(sl + (D_GH + un) * RC + t.c0, v);
                ld4(us + un * RS + t.c0, v); st4(sl + (D_U + un) * RC + t.c0, v);
            }
        }
        __syncthreads();
        {   // prediction: quarter q of the hidden units of chain c, all o outputs
            const int c = tid & 63, q = tid >> 6;
            float acc[8];
#pragma unroll
            for (int oo = 0; oo < 8; ++oo) acc[oo] = 0.0f;
            for (int k = 16 * q; k < 16 * q + 16; ++k) {
                const float yv = ys[k * RS + c];
#pragma unroll
                for (int oo = 0; oo < 8; ++oo) acc[oo] = fmaf(sm[DecSmem::OW + oo * HD + k], yv, acc[oo]);
            }
#pragma unroll
            for (int oo = 0; oo < 8; ++oo) part[(q * 8 + oo) * RS + c] = acc[oo];
        }
        __syncthreads();
        if (tid < RC) {
            const int c = tid;
            const bool valid = ci->gid[c] >= 0;
            float e2 = 0.0f;
            for (int oo = 0; oo < o; ++oo) {
                const float pv = sm[DecSmem::OB + oo] + ((part[oo * RS + c] + part[(8 + oo) * RS + c]) + (part[(16 + oo) * RS + c] + part[(24 + oo) * RS + c]));
                if (STORE) sl[(D_P + oo) * RC + c] = pv;
                if (LOSS && valid) {
                    const float nx = hist[ci->hoff[c] + (int64_t)(j + 1 + w) * a.N * o + oo];
                    bl += fabsf(nx - pv) * mask[ci->moff[c] + j + 1 + w] * scale_j;
                    const float dcur = xin[oo * RS + c] - pv;
                    e2 = fmaf(dcur, dcur, e2);
                }
            }
            if (LOSS && valid) sl_acc += fmaxf(sqrtf(e2) - a.thres, 0.0f) * a.stab_scale;
        }
        __syncthreads();
        float* tmp = hcur; hcur = hnext; hnext = tmp;
    }
    return hcur;
}

__global__ void __launch_bounds__(NT, 1) dec_kernel(Args a) {
    extern __shared__ __align__(16) float sm[];
    const int tile = blockIdx.x, ag = blockIdx.y, tid = threadIdx.x;
    const Coord t;
    const BDecLayout D = bdec_layout(a.o, a.L);
    const int L = a.L, NP = a.n_pos, W = a.W, o = a.o, in_d = a.o + a.L;
    ChainInfo* ci = reinterpret_cast<ChainInfo*>(sm + DecSmem::CI);
    const float* Wd = a.dec + (int64_t)ag * a.dec_stride;
    stage_gru<HD>(sm + DecSmem::WF, sm + DecSmem::BIAS, Wd + D.wih, Wd + D.whh, Wd + D.bih, Wd + D.bhh);
    for (int idx = tid; idx < 16 * HD; idx += NT) {
        const int kk = idx / HD, un = idx - kk * HD;
        sm[DecSmem::LW + idx] = kk < in_d ? Wd[D.lin_w + un * in_d + kk] : 0.0f;
    }
    for (int idx = tid; idx < 8 * HD; idx += NT) sm[DecSmem::OW + idx] = idx / HD < o ? Wd[D.out_w + idx] : 0.0f;      // [o][unit]
    for (int idx = tid; idx < HD; idx += NT) sm[DecSmem::LB + idx] = Wd[D.lin_b + idx];
    for (int idx = tid; idx < 8; idx += NT) sm[DecSmem::OB + idx] = idx < o ? Wd[D.out_b + idx] : 0.0f;
    chain_setup(ci, a, tile, ag);
    const float* hist = a.hist + (int64_t)ag * a.B * a.T * a.N * a.o;
    const float* mask = a.mask + (int64_t)ag * a.B * a.T;
    const float* scale = a.scale + (int64_t)ag * NP;
    const int64_t tl = (int64_t)ag * a.tiles + tile;
    const float* lat_all = a.lat_all + tl * (NP + 1) * L * RC;
    float* dh_b = a.dh_b + tl * NP * HD * RC;
    float* dlat = a.dlat + tl * NP * L * RC;
    float* slab = a.slab + tl * W * D_ROWS * RC;
    const float ks = 1.0f / (1.0f - a.p_drop);

    // ================= forward sweep: loss and boundary states =================
    float* hcur = sm + DecSmem::HA;
    tile_zero(hcur, HD);
    __syncthreads();
    float bl = 0.0f, sl_acc = 0.0f;
    for (int j = 0; j < NP; ++j) {
        tile_s2g(dh_b + (int64_t)j * HD * RC, hcur, HD);
        hcur = dec_window<true, false>(sm, a, hist, mask, lat_all + (int64_t)j * L * RC, ci, t, j, scale[j], hcur, slab, bl, sl_acc);
    }
    bl = warp_sum(bl); sl_acc = warp_sum(sl_acc);
    if (t.lane == 0 && tid < RC) { atomicAdd(a.b_loss + ag, bl); atomicAdd(a.s_loss + ag, sl_acc); }

    // ================= backward sweep =================
    float aih[Cfg<HD>::GPT][Cfg<HD>::KPT], ahh[Cfg<HD>::GPT][Cfg<HD>::KPT];
#pragma unroll
    for (int i = 0; i < Cfg<HD>::GPT; ++i)
#pragma unroll
        for (int jx = 0; jx < Cfg<HD>::KPT; ++jx) { aih[i][jx] = 0.0f; ahh[i][jx] = 0.0f; }
    float g_bias = 0.0f;                 // thread tid: column sum of DG row tid (256 rows)
    float g_ow[2] = {0.0f, 0.0f};        // out_w[o = tid / 64 (+4)][unit = tid % 64]
    float g_ob = 0.0f;                   // tid < o
    float g_lw[4] = {0.0f, 0.0f, 0.0f, 0.0f};   // lin_w[unit = tid % 64][kk = tid / 64 + 4 m]
    float g_lb = 0.0f;                   // tid < 64
    float dh[4][4];                      // d loss / d (decoder hidden after the current step), carried
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int i = 0; i < 4; ++i) dh[c][i] = 0.0f;
    float* DG = sm + DecSmem::DG; float* us = sm + DecSmem::U; float* P = sm + DecSmem::P; float* xin = sm + DecSmem::XIN; float* dpr = sm + DecSmem::DPR;
    __syncthreads();

    for (int j = NP - 1; j >= 0; --j) {
        const float* lat_j = lat_all + (int64_t)j * L * RC;
        const float* hb_j = dh_b + (int64_t)j * HD * RC;
        hcur = sm + DecSmem::HA;
        tile_g2s(hcur, hb_j, HD);
        __syncthreads();
        float d0 = 0.0f, d1 = 0.0f;
        dec_window<false, true>(sm, a, hist, mask, lat_j, ci, t, j, scale[j], hcur, slab, d0, d1);      // ends with a barrier
        float dl0 = 0.0f, dl1 = 0.0f;    // thread: d latent_j[l = 2 (tid / 64) (+1)] of chain tid % 64
        for (int w = W - 1; w >= 0; --w) {
            const float* sl = slab + (int64_t)w * D_ROWS * RC;
            const float* hp_g = w > 0 ? slab + (int64_t)(w - 1) * D_ROWS * RC + D_H * RC : hb_j;
            // S1: d prediction, the step's input and dropped-out output tiles
            for (int idx = tid; idx < 8 * RC; idx += NT) {
                const int oo = idx >> 6, c = idx & 63;
                float v = 0.0f;
                if (oo < o && ci->gid[c] >= 0) {
                    const float e = sl[(D_P + oo) * RC + c] - hist[ci->hoff[c] + (int64_t)(j + 1 + w) * a.N * o + oo];
                    v = (e > 0.0f ? 1.0f : (e < 0.0f ? -1.0f : 0.0f)) * mask[ci->moff[c] + j + 1 + w] * scale[j];
                }
                dpr[oo * RS + c] = v;
            }
            tile_g2s(P, sl + D_Y * RC, HD);
            dec_input(xin, a, hist, lat_j, ci, j, w);
            __syncthreads();
            // S2: output-layer gradients; d hidden through tanh / dropout; gate derivatives
            {
                const int un = tid & 63, og = tid >> 6;
                g_ow[0] += row_dot(dpr + og * RS, P + un * RS);
                if (og + 4 < o) g_ow[1] += row_dot(dpr + (og + 4) * RS, P + un * RS);
                if (tid < o) g_ob += row_sum(dpr + tid * RS);
            }
            bool kp[4][4];
            keep_bits(a, ci, t, j, w, kp);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int un = unit_of(t.ug, i);
                float dy[4] = {0.0f, 0.0f, 0.0f, 0.0f}, hn[4];
                for (int oo = 0; oo < o; ++oo) {
                    float d[4]; ld4(dpr + oo * RS + t.c0, d);
                    const float wv = sm[DecSmem::OW + oo * HD + un];
#pragma unroll
                    for (int c = 0; c < 4; ++c) dy[c] = fmaf(d[c], wv, dy[c]);
                }
                ld4(sl + (D_H + un) * RC + t.c0, hn);
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float th = tanhf(hn[c]);
                    if (kp[c][i]) dh[c][i] += dy[c] * ks * (1.0f - th * th);
                }
            }
            float dhz[4][4];
            gate_derivs<HD>(DG, t, dh, sl + D_R * RC, sl + D_Z * RC, sl + D_N * RC, sl + D_GH * RC, hp_g, dhz);
            __syncthreads();
            // S3: the step's u and previous-hidden tiles
            tile_g2s(us, sl + D_U * RC, HD);
            tile_g2s(P, hp_g, HD);
            __syncthreads();
            // S4: weight gradients, data gradients
            gru_dw<HD>(DG, us, P, t, aih, ahh);
            float du[4][4], dhp[4][4];
            gru_bwd_data<HD>(sm + DecSmem::WF, DG, t, du, dhp);
            g_bias += row_sum(DG + tid * RS);
            float dli[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                float uv[4]; ld4(us + unit_of(t.ug, i) * RS + t.c0, uv);
#pragma unroll
                for (int c = 0; c < 4; ++c) { dli[i][c] = uv[c] > 0.0f ? du[c][i] : 0.0f; dh[c][i] = dhz[c][i] + dhp[c][i]; }
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < 4; ++i) st4(us + unit_of(t.ug, i) * RS + t.c0, dli[i]);
            __syncthreads();
            // S5: input-layer gradients and d latent_j
            {
                const int un = tid & 63, q = tid >> 6;
#pragma unroll
                for (int m = 0; m < 4; ++m)
                    if (q + 4 * m < in_d) g_lw[m] += row_dot(us + un * RS, xin + (q + 4 * m) * RS);
                if (tid < HD) g_lb += row_sum(us + tid * RS);
                const int c = tid & 63, l0 = 2 * q;
                float s0 = 0.0f, s1 = 0.0f;
                for (int k = 0; k < HD; ++k) {
                    const float dv = us[k * RS + c];
                    s0 = fmaf(dv, sm[DecSmem::LW + (o + l0) * HD + k], s0);
                    s1 = fmaf(dv, sm[DecSmem::LW + (o + l0 + 1) * HD + k], s1);
                }
                dl0 += s0; dl1 += s1;
            }
            __syncthreads();
        }
        {
            const int c = tid & 63, l0 = 2 * (tid >> 6);
            if (l0 < L) dlat[((int64_t)j * L + l0) * RC + c] = dl0;
            if (l0 + 1 < L) dlat[((int64_t)j * L + l0 + 1) * RC + c] = dl1;
        }
    }
    // ---- flush -----------------------------------------------------------------------------------------------------------
    float* Gd = a.g_dec + (int64_t)ag * a.dec_stride;
    flush_dw<HD>(aih, ahh, t, Gd + D.wih, Gd + D.whh);
    {
        const int blk = tid / HD, unit = col_to_unit<HD>(tid % HD);
        if (blk < 2) { atomicAdd(Gd + D.bih + blk * HD + unit, g_bias); atomicAdd(Gd + D.bhh + blk * HD + unit, g_bias); }
        else if (blk == 2) atomicAdd(Gd + D.bih + 2 * HD + unit, g_bias);
        else atomicAdd(Gd + D.bhh + 2 * HD + unit, g_bias);
        const int un = tid & 63, q = tid >> 6;
        if (q < o) atomicAdd(Gd + D.out_w + q * HD + un, g_ow[0]);
        if (q + 4 < o) atomicAdd(Gd + D.out_w + (q + 4) * HD + un, g_ow[1]);
        if (tid < o) atomicAdd(Gd + D.out_b + tid, g_ob);
#pragma unroll
        for (int m = 0; m < 4; ++m)
            if (q + 4 * m < in_d) atomicAdd(Gd + D.lin_w + un * in_d + q + 4 * m, g_lw[m]);
        if (tid < HD) atomicAdd(Gd + D.lin_b + tid, g_lb);
    }
}

static int64_t per_tile_floats(int n_pos, int L, int W) {
    return (int64_t)RC * ((int64_t)(n_pos + 1) * L + (int64_t)n_pos * L + (int64_t)(n_pos + 1) * HE + (int64_t)n_pos * HD + (int64_t)n_pos * L + (int64_t)W * D_ROWS);
}

}  // namespace blt
}  // namespace iplan

extern "C" int64_t iplan_beh_learn_tile_scratch_floats(int n_agents, int n_eps, int n_pos, int n_slots, int obs_dim, int latent_dim, int hist_len) {
    (void)obs_dim;
    const int64_t tiles = ((int64_t)n_eps * n_slots + iplan::blt::RC - 1) / iplan::blt::RC;
    return (int64_t)n_agents * tiles * iplan::blt::per_tile_floats(n_pos, latent_dim, hist_len);
}

extern "C" int iplan_beh_learn_tile(const float* enc_params, int64_t enc_stride, const float* dec_params, int64_t dec_stride,
                                    float* g_enc, float* g_dec, const float* hist, const float* mask, const float* scale, const uint8_t* keep,
                                    float* b_loss, float* s_loss, float* scratch, int64_t scratch_floats,
                                    uint64_t seed, uint64_t counter, float p_drop, float soft_coef, float thres_small_variation,
                                    int n_agents, int n_eps, int n_steps, int n_slots, int obs_dim, int latent_dim, int hist_len, void* stream) {
    using namespace iplan;
    using namespace iplan::blt;
    IPLAN_REQUIRE(enc_params && dec_params && g_enc && g_dec && hist && mask && scale && b_loss && s_loss && scratch, "beh_learn: null pointer");
    const int n_pos = n_steps - 1 - hist_len;
    IPLAN_REQUIRE(n_pos > 0, "beh_learn: episode of %d steps is shorter than the window of %d", n_steps, hist_len);
    IPLAN_REQUIRE(obs_dim > 0 && obs_dim <= 8 && latent_dim > 0 && latent_dim <= 8 && (latent_dim & 1) == 0 && n_slots > 0, "beh_learn: obs_dim <= 8 and an even latent_dim <= 8 are built (got %d, %d)", obs_dim, latent_dim);
    IPLAN_REQUIRE(n_agents > 0 && n_eps > 0 && p_drop >= 0.f && p_drop < 1.f, "beh_learn: bad arguments");
    IPLAN_REQUIRE((int64_t)n_eps * n_steps * n_slots * obs_dim < (int64_t)1 << 31, "beh_learn: history block of one agent exceeds 2^31 elements");
    const int64_t need = iplan_beh_learn_tile_scratch_floats(n_agents, n_eps, n_pos, n_slots, obs_dim, latent_dim, hist_len);
    IPLAN_REQUIRE(scratch_floats >= need, "beh_learn: scratch too small (%lld floats, need %lld)", (long long)scratch_floats, (long long)need);
    const int tiles = (int)(((int64_t)n_eps * n_slots + RC - 1) / RC);
    const int64_t nt = (int64_t)n_agents * tiles;
    Args a;
    a.enc = enc_params; a.enc_stride = enc_stride; a.dec = dec_params; a.dec_stride = dec_stride; a.g_enc = g_enc; a.g_dec = g_dec;
    a.hist = hist; a.mask = mask; a.scale = scale; a.keep = keep; a.b_loss = b_loss; a.s_loss = s_loss;
    float* p = scratch;
    a.lat_all = p; p += nt * (n_pos + 1) * latent_dim * RC;
    a.znew = p;    p += nt * n_pos * latent_dim * RC;
    a.eh_b = p;    p += nt * (n_pos + 1) * HE * RC;
    a.dh_b = p;    p += nt * n_pos * HD * RC;
    a.dlat = p;    p += nt * n_pos * latent_dim * RC;
    a.slab = p;
    a.seed = seed; a.counter = counter; a.p_drop = p_drop; a.coef = soft_coef; a.thres = thres_small_variation;
    a.stab_scale = 1.0f / ((float)n_eps * (float)hist_len * (float)n_pos);
    a.B = n_eps; a.T = n_steps; a.N = n_slots; a.o = obs_dim; a.L = latent_dim; a.W = hist_len; a.n_pos = n_pos; a.tiles = tiles;
    const size_t smem_e = sizeof(float) * (size_t)EncSmem::TOTAL, smem_d = sizeof(float) * (size_t)DecSmem::TOTAL;
    static_assert(sizeof(float) * DecSmem::TOTAL <= 227 * 1024, "decoder tile does not fit in shared memory");
    static bool configured = false;
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(dec_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_d);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(enc_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_e);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(enc_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_e);
        if (e != cudaSuccess) { set_error("beh_learn: smem attr: %s", cudaGetErrorString(e)); return (int)e; }
        configured = true;
    }
    const dim3 grid(tiles, n_agents);
    enc_fwd_kernel<<<grid, NT, smem_e, (cudaStream_t)stream>>>(a);
    dec_kernel<<<grid, NT, smem_d, (cudaStream_t)stream>>>(a);
    enc_bwd_kernel<<<grid, NT, smem_e, (cudaStream_t)stream>>>(a);
    count_launch(3);
    return check_launch("beh_learn_tile");
}
