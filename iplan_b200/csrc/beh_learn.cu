// Behavior_policy.learn — reconstruction loss and gradients of the behavioural-incentive encoder / decoder over a
// whole episode batch (reference nova/stable_behavior_policy.py:161-279; SURVEY §8f rank 3).
//
// Specified line by line by oracle/iplan_oracle.py::behavior_learn_agent (pinned to a recorded run of the reference);
// checked against that run by tools/check_beh_learn.py.
//
// Per agent-net and episode b the N slots are independent chains through the n_pos = T - 1 - W window positions:
//   pred_j, dh_{j+1} = Decoder([window_j | latent_j] ; dh_j)       W-step GRU(64), tanh, dropout, linear   (behavior_net.py:40-72)
//   eh_{j+1}, z_j    = Encoder(window_j ; eh_j)                    W-step GRU(32), softmax latent           (:17-22)
//   latent_{j+1}     = (1 - c) latent_j + c z_j                                                              (:223)
//   loss            += sum |window_{j+W} - pred_j| * mask / (sum mask + 1e-10) * o * N / n_pos               (:226-239)
// and the backward is one BPTT through all n_pos x W steps of both GRUs and the latent recursion.  Plain fp32 FFMA,
// one CTA per (episode, agent-net), one warp per slot (a warp walks its slots one after the other; lanes = hidden
// units), positions in lock step so that the weight gradients of a position are reduced by the whole CTA into a
// shared-memory accumulator (flushed with atomics once at the end).  Only the chain states at window boundaries are
// kept (global scratch); the inside of a window is recomputed in the backward sweep.
#include "common.cuh"

namespace iplan {

constexpr int BT = 256;
constexpr int BE = IPLAN_HID;            // 32 encoder hidden
constexpr int BD = IPLAN_RNN;            // 64 decoder hidden
constexpr int BE3 = 3 * BE, BD3 = 3 * BD;

struct BDecLayout { int64_t lin_w, lin_b, wih, whh, bih, bhh, out_w, out_b, total; };
__host__ __device__ inline BDecLayout bdec_layout(int o, int Ld) {
    BDecLayout L;
    int64_t off = 0;
    auto take = [&](int64_t n) { int64_t at = off; off = pad4(off + n); return at; };
    L.lin_w = take((int64_t)BD * (o + Ld)); L.lin_b = take(BD);
    L.wih = take(BD3 * BD); L.whh = take(BD3 * BD); L.bih = take(BD3); L.bhh = take(BD3);
    L.out_w = take((int64_t)o * BD); L.out_b = take(o);
    L.total = off;
    return L;
}

struct BehLearnArgs {
    const float* enc; int64_t enc_stride; const float* dec; int64_t dec_stride;
    float* g_enc; float* g_dec;
    const float* hist;        // [A][B][T][N][o]
    const float* mask;        // [A][B][T]
    const float* scale;       // [A][n_pos]  o * N / (mask elements of the next-window + 1e-10) / n_pos
    const uint8_t* keep;      // NULL (Philox) or [A][B][n_pos][N][W][64]
    float* b_loss; float* s_loss;      // [A]
    float* scratch; int64_t scratch_per_cta;
    uint64_t seed, counter; float p_drop, coef, thres, stab_scale;     // stab_scale = 1 / (B * W * n_pos)
    int B, T, N, o, L, W, n_pos;
};

__device__ __forceinline__ float bsg(float x) { return 1.0f / (1.0f + expf(-x)); }

// G[c*ldg + k] += sum_r d[r][c] * in[r][k]; gb[c] += sum_r d[r][c]   (G, gb in shared memory; one owner thread per entry)
__device__ void cta_wgrad_acc(float* G, int ldg, float* gb, const float* d, int ldd, const float* in, int ldi, int rows, int cols, int K) {
    for (int idx = threadIdx.x; idx < cols * K; idx += BT) {
        const int c = idx / K, k = idx - c * K;
        float acc = 0.0f;
        for (int r = 0; r < rows; ++r) acc = fmaf(d[(int64_t)r * ldd + c], in[(int64_t)r * ldi + k], acc);
        G[(int64_t)c * ldg + k] += acc;
    }
    for (int c = threadIdx.x; c < cols; c += BT) {
        float acc = 0.0f;
        for (int r = 0; r < rows; ++r) acc += d[(int64_t)r * ldd + c];
        gb[c] += acc;
    }
}

__global__ void __launch_bounds__(BT, 1) beh_learn_kernel(BehLearnArgs a) {
    extern __shared__ __align__(16) float sg[];                       // gradient accumulators: encoder | decoder
    const int b = blockIdx.x, ag = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int N = a.N, o = a.o, Ld = a.L, W = a.W, T = a.T, NP = a.n_pos, in_d = o + Ld;
    const float* __restrict__ We = a.enc + (int64_t)ag * a.enc_stride;
    const float* __restrict__ Wd = a.dec + (int64_t)ag * a.dec_stride;
    const BehLayout E = beh_layout(o, Ld);
    const BDecLayout D = bdec_layout(o, Ld);
    float* ge = sg;
    float* gd = sg + E.total;
    for (int idx = tid; idx < E.total + D.total; idx += BT) sg[idx] = 0.0f;
    const float* hist = a.hist + ((int64_t)ag * a.B + b) * T * N * o;          // [T][N][o]
    const float* mask = a.mask + ((int64_t)ag * a.B + b) * T;
    const float* scale = a.scale + (int64_t)ag * NP;
    const float ks = 1.0f / (1.0f - a.p_drop);

    // ---- global scratch of this CTA ------------------------------------------------------------------------------
    float* sc = a.scratch + ((int64_t)ag * a.B + b) * a.scratch_per_cta;
    float* dh_b = sc;                                         // [NP+1][N][64] decoder hidden at window boundaries
    float* eh_b = dh_b + (int64_t)(NP + 1) * N * BD;          // [NP+1][N][32]
    float* lat_b = eh_b + (int64_t)(NP + 1) * N * BE;         // [NP+1][N][L]
    float* xin = lat_b + (int64_t)(NP + 1) * N * Ld;          // [W][N][o+L]
    float* u_d = xin + (int64_t)W * N * in_d;                 // [W][N][64]
    float* h_d = u_d + (int64_t)W * N * BD;                   // [W+1][N][64]
    float* y_d = h_d + (int64_t)(W + 1) * N * BD;             // [W][N][64]
    float* prd = y_d + (int64_t)W * N * BD;                   // [W][N][o]
    float* u_e = prd + (int64_t)W * N * o;                    // [W][N][32]
    float* h_e = u_e + (int64_t)W * N * BE;                   // [W+1][N][32]
    float* nl = h_e + (int64_t)(W + 1) * N * BE;              // [N][L] new latent z_j
    float* dprd = nl + (int64_t)N * Ld;                       // [W][N][o]
    float* dgi_d = dprd + (int64_t)W * N * o;                 // [W][N][192]
    float* dgh_d = dgi_d + (int64_t)W * N * BD3;
    float* dli_d = dgh_d + (int64_t)W * N * BD3;              // [W][N][64] d (pre-ReLU decoder input layer)
    float* dgi_e = dli_d + (int64_t)W * N * BD;               // [W][N][96]
    float* dgh_e = dgi_e + (int64_t)W * N * BE3;
    float* dli_e = dgh_e + (int64_t)W * N * BE3;              // [W][N][32]
    float* dlg = dli_e + (int64_t)W * N * BE;                 // [N][L] d logits of the latent soft-max
    float* c_dh = dlg + (int64_t)N * Ld;                      // carried gradients: [N][64], [N][32], [N][L]
    float* c_eh = c_dh + (int64_t)N * BD;
    float* c_lat = c_eh + (int64_t)N * BE;

    auto kept = [&](int j, int n, int w, int c) -> bool {
        const int64_t kidx = (((((int64_t)ag * a.B + b) * NP + j) * N + n) * W + w) * BD + c;
        if (a.keep) return a.keep[kidx] != 0;
        const uint4 rnd = philox4x32(make_uint4((uint32_t)kidx, (uint32_t)(kidx >> 32), (uint32_t)a.counter, (uint32_t)(a.counter >> 32)),
                                     make_uint2((uint32_t)a.seed ^ 0x85ebca6bu, (uint32_t)(a.seed >> 32)));
        return u01(rnd.x) >= a.p_drop;
    };
    // row w of the window that ends at position j: history step j - W + 1 + w, zeros before the episode start (:140-146)
    auto win = [&](int j, int w, int n, int c) -> float {
        const int t = j - W + 1 + w;
        return t >= 0 ? hist[((int64_t)t * N + n) * o + c] : 0.0f;
    };

    // GRU cell forward for the decoder (lane owns units lane, lane + 32) and the encoder (lane owns unit lane)
    auto dec_gates = [&](const float* u, const float* hp, int c, float& r, float& z, float& nn, float& ghn) {
        float gi[3], gh[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            float ai = Wd[D.bih + q * BD + c], ah = Wd[D.bhh + q * BD + c];
            const float* wi = Wd + D.wih + (int64_t)(q * BD + c) * BD;
            const float* wh = Wd + D.whh + (int64_t)(q * BD + c) * BD;
            for (int k = 0; k < BD; ++k) { ai = fmaf(wi[k], u[k], ai); ah = fmaf(wh[k], hp[k], ah); }
            gi[q] = ai; gh[q] = ah;
        }
        r = bsg(gi[0] + gh[0]); z = bsg(gi[1] + gh[1]); ghn = gh[2]; nn = tanhf(gi[2] + r * gh[2]);
    };
    auto enc_gates = [&](const float* u, const float* hp, int c, float& r, float& z, float& nn, float& ghn) {
        float gi[3], gh[3];
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            float ai = We[E.bih + q * BE + c], ah = We[E.bhh + q * BE + c];
            const float* wi = We + E.wih + (int64_t)(q * BE + c) * BE;
            const float* wh = We + E.whh + (int64_t)(q * BE + c) * BE;
            for (int k = 0; k < BE; ++k) { ai = fmaf(wi[k], u[k], ai); ah = fmaf(wh[k], hp[k], ah); }
            gi[q] = ai; gh[q] = ah;
        }
        r = bsg(gi[0] + gh[0]); z = bsg(gi[1] + gh[1]); ghn = gh[2]; nn = tanhf(gi[2] + r * gh[2]);
    };

    // ---- forward of window position j for slot n (this warp); optionally accumulates the losses -------------------------
    float bl = 0.0f, sl = 0.0f;                                        // lane-local loss partials
    auto position_forward = [&](int j, int n, bool with_loss) {
        const float* lat = lat_b + ((int64_t)j * N + n) * Ld;
        // decoder
        for (int c = lane; c < BD; c += 32) h_d[(int64_t)n * BD + c] = dh_b[((int64_t)j * N + n) * BD + c];
        __syncwarp();
        for (int w = 0; w < W; ++w) {
            float* xr = xin + ((int64_t)w * N + n) * in_d;
            if (lane < in_d) xr[lane] = lane < o ? win(j, w, n, lane) : lat[lane - o];
            __syncwarp();
            float* ur = u_d + ((int64_t)w * N + n) * BD;
            for (int c = lane; c < BD; c += 32) {
                float acc = Wd[D.lin_b + c];
                for (int k = 0; k < in_d; ++k) acc = fmaf(Wd[D.lin_w + (int64_t)c * in_d + k], xr[k], acc);
                ur[c] = fmaxf(acc, 0.0f);
            }
            __syncwarp();
            const float* hp = h_d + ((int64_t)w * N + n) * BD;
            float* hn = h_d + ((int64_t)(w + 1) * N + n) * BD;
            float* yr = y_d + ((int64_t)w * N + n) * BD;
            for (int c = lane; c < BD; c += 32) {
                float r, z, nn, ghn;
                dec_gates(ur, hp, c, r, z, nn, ghn);
                const float hv = (1.0f - z) * nn + z * hp[c];
                hn[c] = hv;
                yr[c] = kept(j, n, w, c) ? tanhf(hv) * ks : 0.0f;
            }
            __syncwarp();
            float e2 = 0.0f;
            if (lane < o) {
                float ov = Wd[D.out_b + lane];
                for (int k = 0; k < BD; ++k) ov = fmaf(Wd[D.out_w + (int64_t)lane * BD + k], yr[k], ov);
                prd[((int64_t)w * N + n) * o + lane] = ov;
                if (with_loss) {
                    const float nx = hist[((int64_t)(j + 1 + w) * N + n) * o + lane];
                    bl += fabsf(nx - ov) * mask[j + 1 + w] * scale[j];
                    const float dcur = xr[lane] - ov;
                    e2 = dcur * dcur;
                }
            }
            if (with_loss) {                                           // stability term: clamp(|window row - prediction| - thres, 0)  (:221, :234-236)
                e2 = warp_sum(e2);
                if (lane == 0) sl += fmaxf(sqrtf(e2) - a.thres, 0.0f) * a.stab_scale;
            }
            __syncwarp();
        }
        for (int c = lane; c < BD; c += 32) dh_b[((int64_t)(j + 1) * N + n) * BD + c] = h_d[((int64_t)W * N + n) * BD + c];
        // encoder
        h_e[(int64_t)n * BE + lane] = eh_b[((int64_t)j * N + n) * BE + lane];
        __syncwarp();
        for (int w = 0; w < W; ++w) {
            const float* xr = xin + ((int64_t)w * N + n) * in_d;       // first o entries = the window row
            float* ur = u_e + ((int64_t)w * N + n) * BE;
            float acc = We[E.lin_b + lane];
            for (int k = 0; k < o; ++k) acc = fmaf(We[E.lin_w + (int64_t)lane * o + k], xr[k], acc);
            ur[lane] = fmaxf(acc, 0.0f);
            __syncwarp();
            const float* hp = h_e + ((int64_t)w * N + n) * BE;
            float r, z, nn, ghn;
            enc_gates(ur, hp, lane, r, z, nn, ghn);
            h_e[((int64_t)(w + 1) * N + n) * BE + lane] = (1.0f - z) * nn + z * hp[lane];
            __syncwarp();
        }
        const float* hl = h_e + ((int64_t)W * N + n) * BE;
        eh_b[((int64_t)(j + 1) * N + n) * BE + lane] = hl[lane];
        float lg = -INFINITY;
        if (lane < Ld) {
            lg = We[E.out_b + lane];
            for (int k = 0; k < BE; ++k) lg = fmaf(We[E.out_w + (int64_t)lane * BE + k], hl[k], lg);
        }
        const float mx = warp_max(lg);
        const float ex = lane < Ld ? expf(lg - mx) : 0.0f;
        const float den = warp_sum(ex);
        if (lane < Ld) {
            const float zl = ex / den;
            nl[(int64_t)n * Ld + lane] = zl;
            lat_b[((int64_t)(j + 1) * N + n) * Ld + lane] = (1.0f - a.coef) * lat[lane] + zl * a.coef;
        }
        __syncwarp();
    };

    // ================= forward sweep =================
    for (int n = warp; n < N; n += BT / 32) {
        for (int c = lane; c < BD; c += 32) { dh_b[(int64_t)n * BD + c] = 0.0f; c_dh[(int64_t)n * BD + c] = 0.0f; }
        eh_b[(int64_t)n * BE + lane] = 0.0f; c_eh[(int64_t)n * BE + lane] = 0.0f;
        if (lane < Ld) { lat_b[(int64_t)n * Ld + lane] = 0.0f; c_lat[(int64_t)n * Ld + lane] = 0.0f; }
        __syncwarp();
        for (int j = 0; j < NP; ++j) position_forward(j, n, true);
    }
    bl = warp_sum(bl);
    if (lane == 0) { atomicAdd(a.b_loss + ag, bl); atomicAdd(a.s_loss + ag, sl); }
    __syncthreads();

    // ================= backward sweep, positions in lock step =================
    for (int j = NP - 1; j >= 0; --j) {
        for (int n = warp; n < N; n += BT / 32) {
            position_forward(j, n, false);                             // recompute the inside of the window
            // ---- decoder BPTT ----
            float dh[2] = {c_dh[(int64_t)n * BD + lane], c_dh[(int64_t)n * BD + lane + 32]};
            float dlat = 0.0f;                                         // lanes o .. o+L-1: d latent_j from the decoder input
            for (int w = W - 1; w >= 0; --w) {
                float* dpr = dprd + ((int64_t)w * N + n) * o;
                if (lane < o) {
                    const float e = prd[((int64_t)w * N + n) * o + lane] - hist[((int64_t)(j + 1 + w) * N + n) * o + lane];
                    dpr[lane] = (e > 0.0f ? 1.0f : (e < 0.0f ? -1.0f : 0.0f)) * mask[j + 1 + w] * scale[j];
                }
                __syncwarp();
                const float* ur = u_d + ((int64_t)w * N + n) * BD;
                const float* hp = h_d + ((int64_t)w * N + n) * BD;
                const float* hn = h_d + ((int64_t)(w + 1) * N + n) * BD;
                float* dgi = dgi_d + ((int64_t)w * N + n) * BD3;
                float* dgh = dgh_d + ((int64_t)w * N + n) * BD3;
                float zz[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int c = lane + 32 * u;
                    float dy = 0.0f;
                    for (int k = 0; k < o; ++k) dy = fmaf(dpr[k], Wd[D.out_w + (int64_t)k * BD + c], dy);
                    const float th = tanhf(hn[c]);
                    if (kept(j, n, w, c)) dh[u] += dy * ks * (1.0f - th * th);
                    float r, z, nn, ghn;
                    dec_gates(ur, hp, c, r, z, nn, ghn);
                    const float dn = dh[u] * (1.0f - z), dz = dh[u] * (hp[c] - nn);
                    const float dan = dn * (1.0f - nn * nn), daz = dz * z * (1.0f - z), dar = dan * ghn * r * (1.0f - r);
                    dgi[c] = dar; dgi[BD + c] = daz; dgi[2 * BD + c] = dan;
                    dgh[c] = dar; dgh[BD + c] = daz; dgh[2 * BD + c] = dan * r;
                    zz[u] = z;
                }
                __syncwarp();
                float* dli = dli_d + ((int64_t)w * N + n) * BD;
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int c = lane + 32 * u;
                    float dhp = dh[u] * zz[u], du = 0.0f;
                    for (int g = 0; g < BD3; ++g) {
                        dhp = fmaf(dgh[g], Wd[D.whh + (int64_t)g * BD + c], dhp);
                        du = fmaf(dgi[g], Wd[D.wih + (int64_t)g * BD + c], du);
                    }
                    dli[c] = ur[c] > 0.0f ? du : 0.0f;
                    dh[u] = dhp;
                }
                __syncwarp();
                if (lane >= o && lane < in_d) {                        // the latent columns of the decoder input
                    float dx = 0.0f;
                    for (int c = 0; c < BD; ++c) dx = fmaf(dli[c], Wd[D.lin_w + (int64_t)c * in_d + lane], dx);
                    dlat += dx;
                }
            }
            c_dh[(int64_t)n * BD + lane] = dh[0]; c_dh[(int64_t)n * BD + lane + 32] = dh[1];
            // ---- latent recursion: latent_{j+1} = (1 - c) latent_j + c z_j ----
            float dnl = 0.0f;                                           // lanes 0 .. L-1: d z_j
            {
                // move the decoder's d latent (held by lanes o..o+L-1) to lanes 0..L-1
                const float dl_dec = __shfl_sync(0xffffffffu, dlat, (lane + o) & 31);
                if (lane < Ld) {
                    const float carried = c_lat[(int64_t)n * Ld + lane];
                    dnl = a.coef * carried;
                    c_lat[(int64_t)n * Ld + lane] = (1.0f - a.coef) * carried + dl_dec;
                }
            }
            // ---- encoder: soft-max latent head, then BPTT ----
            const float zl = lane < Ld ? nl[(int64_t)n * Ld + lane] : 0.0f;
            const float dot = warp_sum(zl * dnl);
            if (lane < Ld) dlg[(int64_t)n * Ld + lane] = zl * (dnl - dot);
            __syncwarp();
            float deh = c_eh[(int64_t)n * BE + lane];
            for (int l = 0; l < Ld; ++l) deh = fmaf(dlg[(int64_t)n * Ld + l], We[E.out_w + (int64_t)l * BE + lane], deh);
            for (int w = W - 1; w >= 0; --w) {
                const float* ur = u_e + ((int64_t)w * N + n) * BE;
                const float* hp = h_e + ((int64_t)w * N + n) * BE;
                float* dgi = dgi_e + ((int64_t)w * N + n) * BE3;
                float* dgh = dgh_e + ((int64_t)w * N + n) * BE3;
                float r, z, nn, ghn;
                enc_gates(ur, hp, lane, r, z, nn, ghn);
                const float dn = deh * (1.0f - z), dz = deh * (hp[lane] - nn);
                const float dan = dn * (1.0f - nn * nn), daz = dz * z * (1.0f - z), dar = dan * ghn * r * (1.0f - r);
                dgi[lane] = dar; dgi[BE + lane] = daz; dgi[2 * BE + lane] = dan;
                dgh[lane] = dar; dgh[BE + lane] = daz; dgh[2 * BE + lane] = dan * r;
                __syncwarp();
                float dhp = deh * z, du = 0.0f;
                for (int g = 0; g < BE3; ++g) {
                    dhp = fmaf(dgh[g], We[E.whh + (int64_t)g * BE + lane], dhp);
                    du = fmaf(dgi[g], We[E.wih + (int64_t)g * BE + lane], du);
                }
                dli_e[((int64_t)w * N + n) * BE + lane] = ur[lane] > 0.0f ? du : 0.0f;
                deh = dhp;
                __syncwarp();
            }
            c_eh[(int64_t)n * BE + lane] = deh;
        }
        __syncthreads();
        // ---- weight gradients of position j: outer products over the (w, n) rows, into the shared accumulators ----
        cta_wgrad_acc(gd + D.out_w, BD, gd + D.out_b, dprd, o, y_d, BD, W * N, o, BD);
        cta_wgrad_acc(gd + D.wih, BD, gd + D.bih, dgi_d, BD3, u_d, BD, W * N, BD3, BD);
        cta_wgrad_acc(gd + D.whh, BD, gd + D.bhh, dgh_d, BD3, h_d, BD, W * N, BD3, BD);
        cta_wgrad_acc(gd + D.lin_w, in_d, gd + D.lin_b, dli_d, BD, xin, in_d, W * N, BD, in_d);
        cta_wgrad_acc(ge + E.out_w, BE, ge + E.out_b, dlg, Ld, h_e + (int64_t)W * N * BE, BE, N, Ld, BE);
        cta_wgrad_acc(ge + E.wih, BE, ge + E.bih, dgi_e, BE3, u_e, BE, W * N, BE3, BE);
        cta_wgrad_acc(ge + E.whh, BE, ge + E.bhh, dgh_e, BE3, h_e, BE, W * N, BE3, BE);
        cta_wgrad_acc(ge + E.lin_w, o, ge + E.lin_b, dli_e, BE, xin, in_d, W * N, BE, o);
        __syncthreads();
    }
    float* Ge = a.g_enc + (int64_t)ag * a.enc_stride;
    float* Gd = a.g_dec + (int64_t)ag * a.dec_stride;
    for (int idx = tid; idx < E.total; idx += BT) atomicAdd(Ge + idx, ge[idx]);
    for (int idx = tid; idx < D.total; idx += BT) atomicAdd(Gd + idx, gd[idx]);
}

}  // namespace iplan

extern "C" int64_t iplan_bdec_layout(int obs_dim, int latent_dim, int64_t* offsets) {
    const iplan::BDecLayout L = iplan::bdec_layout(obs_dim, latent_dim);
    if (offsets) { const int64_t o[8] = {L.lin_w, L.lin_b, L.wih, L.whh, L.bih, L.bhh, L.out_w, L.out_b}; for (int i = 0; i < 8; ++i) offsets[i] = o[i]; }
    return L.total;
}

extern "C" int64_t iplan_beh_learn_tile_scratch_floats(int n_agents, int n_eps, int n_pos, int n_slots, int obs_dim, int latent_dim, int hist_len);
extern "C" int iplan_beh_learn_tile(const float* enc_params, int64_t enc_stride, const float* dec_params, int64_t dec_stride,
                                    float* g_enc, float* g_dec, const float* hist, const float* mask, const float* scale, const uint8_t* keep,
                                    float* b_loss, float* s_loss, float* scratch, int64_t scratch_floats,
                                    uint64_t seed, uint64_t counter, float p_drop, float soft_coef, float thres_small_variation,
                                    int n_agents, int n_eps, int n_steps, int n_slots, int obs_dim, int latent_dim, int hist_len, void* stream);

// 0 = the register-tiled kernels of beh_learn_tile.cu (default), 1 = this file's one-warp-per-chain draft (the cross-check)
static int g_beh_learn_impl = 0;
extern "C" int iplan_beh_learn_set_impl(int impl) { const int old = g_beh_learn_impl; if (impl == 0 || impl == 1) g_beh_learn_impl = impl; return old; }

static int64_t draft_scratch_floats(int n_agents, int n_eps, int n_pos, int n_slots, int obs_dim, int latent_dim, int hist_len) {
    const int64_t N = n_slots, W = hist_len, o = obs_dim, L = latent_dim, D = IPLAN_RNN, E = IPLAN_HID;
    const int64_t per = (n_pos + 1) * N * (D + E + L) + W * N * (o + L) + W * N * D + (W + 1) * N * D + W * N * D + W * N * o
                        + W * N * E + (W + 1) * N * E + N * L + W * N * o + 2 * W * N * 3 * D + W * N * D + 2 * W * N * 3 * E + W * N * E
                        + N * L + N * (D + E + L);
    return (int64_t)n_agents * n_eps * ((per + 3) & ~int64_t(3));
}

extern "C" int64_t iplan_beh_learn_scratch_floats(int n_agents, int n_eps, int n_pos, int n_slots, int obs_dim, int latent_dim, int hist_len) {
    return g_beh_learn_impl == 0 ? iplan_beh_learn_tile_scratch_floats(n_agents, n_eps, n_pos, n_slots, obs_dim, latent_dim, hist_len)
                                 : draft_scratch_floats(n_agents, n_eps, n_pos, n_slots, obs_dim, latent_dim, hist_len);
}

extern "C" int iplan_beh_learn(const float* enc_params, int64_t enc_stride, const float* dec_params, int64_t dec_stride,
                               float* g_enc, float* g_dec, const float* hist, const float* mask, const float* scale, const uint8_t* keep,
                               float* b_loss, float* s_loss, float* scratch, int64_t scratch_floats,
                               uint64_t seed, uint64_t counter, float p_drop, float soft_coef, float thres_small_variation,
                               int n_agents, int n_eps, int n_steps, int n_slots, int obs_dim, int latent_dim, int hist_len, void* stream) {
    using namespace iplan;
    if (g_beh_learn_impl == 0)
        return iplan_beh_learn_tile(enc_params, enc_stride, dec_params, dec_stride, g_enc, g_dec, hist, mask, scale, keep, b_loss, s_loss, scratch, scratch_floats,
                                    seed, counter, p_drop, soft_coef, thres_small_variation, n_agents, n_eps, n_steps, n_slots, obs_dim, latent_dim, hist_len, stream);
    IPLAN_REQUIRE(enc_params && dec_params && g_enc && g_dec && hist && mask && scale && b_loss && s_loss && scratch, "beh_learn: null pointer");
    const int n_pos = n_steps - 1 - hist_len;
    IPLAN_REQUIRE(n_pos > 0, "beh_learn: episode of %d steps is shorter than the window of %d", n_steps, hist_len);
    IPLAN_REQUIRE(obs_dim > 0 && latent_dim > 0 && obs_dim + latent_dim <= 32 && latent_dim <= 32 && n_slots > 0, "beh_learn: bad sizes");
    IPLAN_REQUIRE(n_agents > 0 && n_eps > 0 && p_drop >= 0.f && p_drop < 1.f, "beh_learn: bad arguments");
    const int64_t need = draft_scratch_floats(n_agents, n_eps, n_pos, n_slots, obs_dim, latent_dim, hist_len);
    IPLAN_REQUIRE(scratch_floats >= need, "beh_learn: scratch too small (%lld floats, need %lld)", (long long)scratch_floats, (long long)need);
    BehLearnArgs a;
    a.enc = enc_params; a.enc_stride = enc_stride; a.dec = dec_params; a.dec_stride = dec_stride; a.g_enc = g_enc; a.g_dec = g_dec;
    a.hist = hist; a.mask = mask; a.scale = scale; a.keep = keep; a.b_loss = b_loss; a.s_loss = s_loss;
    a.scratch = scratch; a.scratch_per_cta = need / ((int64_t)n_agents * n_eps);
    a.seed = seed; a.counter = counter; a.p_drop = p_drop; a.coef = soft_coef; a.thres = thres_small_variation;
    a.stab_scale = 1.0f / ((float)n_eps * (float)hist_len * (float)n_pos);
    a.B = n_eps; a.T = n_steps; a.N = n_slots; a.o = obs_dim; a.L = latent_dim; a.W = hist_len; a.n_pos = n_pos;
    const size_t smem = sizeof(float) * (size_t)(beh_layout(obs_dim, latent_dim).total + bdec_layout(obs_dim, latent_dim).total);
    IPLAN_REQUIRE(smem <= 227 * 1024, "beh_learn: %zu B of shared memory", smem);
    static size_t configured = 0;
    if (smem > configured) {
        cudaError_t e = cudaFuncSetAttribute(beh_learn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { set_error("beh_learn: smem attr %zu: %s", smem, cudaGetErrorString(e)); return (int)e; }
        configured = smem;
    }
    beh_learn_kernel<<<dim3(n_eps, n_agents), BT, smem, (cudaStream_t)stream>>>(a);
    count_launch();
    return check_launch("beh_learn");
}
