// Launch arguments of the K1b kernel (behavior_step.cu).
#pragma once
#include "common.cuh"

namespace iplan {

struct BehArgs {
    const float* params; int64_t param_stride;
    iplan_view window, hid, lat_prev, lat_out;
    float coef;
    int n_envs, n_slots, obs_dim, latent_dim, hist_len;
    int64_t win_step;      // 0: window rows are contiguous ([hist_len][obs_dim] per node); else element stride between rows
    int win_pad;           // (win_step != 0) leading window rows that are zero padding; window.ptr = the first real row
};

}  // namespace iplan
