// Host-side plumbing of the C ABI: error text, launch counter, parameter layouts.
#include <stdarg.h>
#include <string.h>

#include <atomic>

#include "common.cuh"

namespace iplan {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}
DetScratch det_scratch(size_t part_floats, size_t n_counters) {
    static float* part = nullptr;
    static unsigned* count = nullptr;
    static size_t part_cap = 0, count_cap = 0;
    if (part_floats > part_cap || n_counters > count_cap) {
        cudaError_t e = cudaDeviceSynchronize();                    // earlier launches may still use the old buffers
        if (e == cudaSuccess && part_floats > part_cap) {
            cudaFree(part);
            part = nullptr; part_cap = 0;
            e = cudaMalloc(&part, part_floats * sizeof(float));
            if (e == cudaSuccess) part_cap = part_floats;
        }
        if (e == cudaSuccess && n_counters > count_cap) {
            cudaFree(count);
            count = nullptr; count_cap = 0;
            e = cudaMalloc(&count, n_counters * sizeof(unsigned));
            if (e == cudaSuccess) e = cudaMemset(count, 0, n_counters * sizeof(unsigned));
            if (e == cudaSuccess) e = cudaDeviceSynchronize();
            if (e == cudaSuccess) count_cap = n_counters;
        }
        if (e != cudaSuccess) {
            set_error("det_scratch: %zu floats, %zu counters: %s", part_floats, n_counters, cudaGetErrorString(e));
            return {nullptr, nullptr};
        }
    }
    return {part, count};
}
int sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
        n = 132;
    return n;
}

}  // namespace iplan

extern "C" int iplan_abi_version(void) { return IPLAN_ABI_VERSION; }
extern "C" const char* iplan_last_error(void) { return iplan::g_err; }
extern "C" int64_t iplan_launch_count(void) { return iplan::g_launches.load(); }

extern "C" int64_t iplan_gat_layout(int in_dim, int64_t* off) {
    const iplan::GatLayout L = iplan::gat_layout(in_dim);
    if (off) {
        const int64_t v[IPLAN_GAT_NTENSORS] = {L.enc_w, L.enc_b, L.wih_f, L.whh_f, L.bih_f, L.bhh_f, L.wih_r, L.whh_r,
                                               L.bih_r, L.bhh_r, L.he_w, L.he_b, L.q_w, L.k_w, L.v_w, L.v_b,
                                               L.c_wih, L.c_whh, L.c_bih, L.c_bhh};
        memcpy(off, v, sizeof(v));
    }
    return L.total;
}
extern "C" int64_t iplan_beh_layout(int obs_dim, int latent_dim, int64_t* off) {
    const iplan::BehLayout L = iplan::beh_layout(obs_dim, latent_dim);
    if (off) {
        const int64_t v[IPLAN_BEH_NTENSORS] = {L.lin_w, L.lin_b, L.wih, L.whh, L.bih, L.bhh, L.out_w, L.out_b};
        memcpy(off, v, sizeof(v));
    }
    return L.total;
}
static int64_t bfc_offsets(const iplan::BfcLayout& L, int64_t* off) {
    if (off) {
        const int64_t v[IPLAN_BFC_NTENSORS] = {L.w1, L.b1, L.w2, L.b2, L.w3, L.b3};
        memcpy(off, v, sizeof(v));
    }
    return L.total;
}
extern "C" int64_t iplan_bfc_layout(int in_dim, int hidden, int latent_dim, int64_t* off) {
    return bfc_offsets(iplan::bfc_layout(in_dim, hidden, latent_dim), off);
}
extern "C" int64_t iplan_bfcdec_layout(int in_dim, int latent_dim, int hidden, int64_t* off) {
    return bfc_offsets(iplan::bfc_layout(in_dim + latent_dim, hidden, in_dim), off);
}
static int64_t trunk_offsets(const iplan::TrunkLayout& L, int64_t* off, bool critic) {
    if (off) {
        const int64_t v[22] = {L.ln0_w, L.ln0_b, L.fc1_w, L.fc1_b, L.ln1_w, L.ln1_b, L.fch_w, L.fch_b, L.lnh_w, L.lnh_b,
                               L.fc2_w, L.fc2_b, L.ln2_w, L.ln2_b, L.wih, L.whh, L.bih, L.bhh, L.ln3_w, L.ln3_b,
                               L.head_w, L.head_b};
        memcpy(off, v, sizeof(v));
        if (critic) {
            int64_t o = iplan::pad4(L.head_b + 1);
            for (int i = 0; i < 4; ++i) { off[22 + i] = o; o = iplan::pad4(o + 1); }
        }
    }
    return L.total;
}
extern "C" int64_t iplan_actor_layout(int feat_dim, int n_actions, int64_t* off) {
    return trunk_offsets(iplan::trunk_layout(feat_dim, n_actions, false), off, false);
}
extern "C" int64_t iplan_critic_layout(int feat_dim, int64_t* off) {
    return trunk_offsets(iplan::trunk_layout(feat_dim, 1, true), off, true);
}
