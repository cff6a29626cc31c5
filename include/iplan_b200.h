/*
 * iplan_b200 — C ABI of the CUDA-native iPLAN hot path (libiplan_b200.so), built for sm_90a (H100).
 *
 * The reference (wuxiyang1996/iPLAN) has no FFI layer: its operator boundary is
 * the Python object API of Prediction_policy / Behavior_policy / DcntrlMAC /
 * IPPOLearner (SURVEY.md §8b).  The host-side mirrors of those classes live in
 * iplan_b200/ (Python, same names and signatures) and bind the entry points
 * below with ctypes; every entry point names the reference function it replaces.
 *
 * Conventions
 *  - plain C: device pointers, sizes, a CUDA stream handle (void* == cudaStream_t);
 *    no torch types.  All tensors fp32 unless stated; all pointers DEVICE memory.
 *  - every call is asynchronous on `stream`; return value 0 == OK, otherwise a
 *    cudaError_t / negative argument-check code; iplan_last_error() has the text.
 *  - "view" = base pointer + element strides, so the same kernel reads either the
 *    reference's [B, A, N, *] staging layout or the packed episode store.
 */
#ifndef IPLAN_B200_H
#define IPLAN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IPLAN_ABI_VERSION 1
#define IPLAN_MAX_SLOTS 64        /* N  (max_vehicle_num) supported by the GAT kernel */
#define IPLAN_HID 32              /* GAT_hidden_dim == attention_dim == encoder_rnn_dim */
#define IPLAN_RNN 64              /* rnn_hidden_dim == mlp_hidden_dim */
#define IPLAN_MAX_ACT 8           /* n_actions upper bound */

/* element [agent][env][slot][0..dim) of a strided fp32 array */
typedef struct {
    float*  ptr;
    int64_t stride_agent;
    int64_t stride_env;
    int64_t stride_slot;
} iplan_view;

int         iplan_abi_version(void);
const char* iplan_last_error(void);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
int64_t     iplan_launch_count(void);

/* ---- flat parameter layouts ---------------------------------------------------
 * Each network's parameters are one fp32 buffer per agent: the module's
 * state_dict tensors in state_dict order, each tensor start rounded up to a
 * multiple of 4 floats.  The functions return the per-agent length and fill
 * `offsets` (one per tensor, in floats). */
#define IPLAN_GAT_NTENSORS 20     /* nova/GAT_Net.py:18-39 */
#define IPLAN_BEH_NTENSORS 8      /* nova/behavior_net.py:12-15 */
#define IPLAN_ACTOR_NTENSORS 22   /* modules/agents/ippo_actor.py:32-40 */
#define IPLAN_CRITIC_NTENSORS 26  /* modules/critics/ippo_critic.py:32-43 (+4 PopArt buffers) */
int64_t iplan_gat_layout(int in_dim, int64_t* offsets);
int64_t iplan_beh_layout(int obs_dim, int latent_dim, int64_t* offsets);
int64_t iplan_actor_layout(int feat_dim, int n_actions, int64_t* offsets);
int64_t iplan_critic_layout(int feat_dim, int64_t* offsets);

/* ---- K1: fused GAT step --------------------------------------------------------
 * replaces Prediction_policy.GAT_latent_update (nova/prediction_policy.py:92-118)
 * = per agent-net GAT_Net.forward (nova/GAT_Net.py:41-142): encode, hard attention
 * (bidirectional GRU over the N-1 neighbours, gumbel-softmax tau), soft attention,
 * GRUCell.  Two launches: the GRU chains (one CTA per (env, agent-net, direction)), then
 * attention + GRUCell (one CTA per (env, agent-net)).
 *   hist      [a][b][n][obs_dim]      history_single at time t
 *   beh_prev  [a][b][n][latent_dim]   behaviour latent of time t-1
 *   h_prev    [a][b][n][32]           attention latent of time t-1
 *   out       [a][b][n][32]           attention latent of time t (may alias nothing)
 *   gumbel    NULL -> in-kernel Philox logistic noise keyed by (seed, counter);
 *             else [A][B][N][N-1][2] gumbel pairs (parity mode, reference draw order)
 *   dbg_hard  NULL or [A][B][N][N-1] hard-attention weights (debug/parity)
 *   scratch   device buffer of >= iplan_gat_scratch_floats(...) floats handed from the first
 *             launch to the second (per-edge hard-attention logit differences) */
int64_t iplan_gat_scratch_floats(int n_envs, int n_agents, int n_slots);
int iplan_gat_step(const float* gat_params, int64_t param_stride,
                   iplan_view hist, iplan_view beh_prev, iplan_view h_prev, iplan_view out,
                   const float* gumbel, uint64_t seed, uint64_t counter,
                   float tau, float* dbg_hard, float* scratch, int64_t scratch_floats,
                   int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim,
                   void* stream);

/* iplan_gat_step with optional cudaEvent_t handles (NULL = skip) recorded on `stream` before the recurrence kernel,
 * between the two kernels and after the attention kernel: per-kernel timing of the dominant kernel inside a running
 * rollout (bench.py's roofline) without a profiler. */
int iplan_gat_step_ex(const float* gat_params, int64_t param_stride,
                      iplan_view hist, iplan_view beh_prev, iplan_view h_prev, iplan_view out,
                      const float* gumbel, uint64_t seed, uint64_t counter,
                      float tau, float* dbg_hard, float* scratch, int64_t scratch_floats,
                      int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim,
                      void* ev_begin, void* ev_mid, void* ev_end, void* stream);

/* ---- GAT_Net.forward at hidden width 128 (BASELINE.json configs[4], the synthetic GAT + GRU microbench) -----------------
 * nova/GAT_Net.py:41-142 with GAT_hidden_dim = attention_dim = 128 and 16 slots per (env, agent-net) "item".  The row x weight
 * products of the op (encode, factored input projections, q|k|v, GRUCell projections) are plain GEMMs that the host runs
 * through a library (iplan_b200/nova/gat128.py); these three kernels are the rest:
 *   iplan_gat128_recur   the bidirectional hard-attention GRU over the 15 neighbours of every ego (:57-97) on the warpgroup
 *                        tensor cores (wgmma, W_hh resident in shared memory) -> per-edge logit differences
 *       P, Q   [2 dirs][A][items][16][384]  ego / neighbour halves of W_ih [enc_i ; enc_j], rows r|z|n, pre-multiplied by the
 *              gate scales (-log2 e for r|z, 2 log2 e for n); Q additionally carries b_ih (+ b_hh for r|z), scaled alike
 *       whh    [A][2][384][128]   bhn [A][2][128] (b_hh of the n gate)   lw [A][2][128] (hard_encoding row 1 - row 0, per direction)
 *       dl     [A][items][2][15][16]  out
 *   iplan_gat128_attend  scores, gumbel hard gate, soft-max, aggregation (:99-133); qkv [A*items*16][384] (v without bias),
 *                        gumbel NULL (Philox) or [A][items][16][15][2];  x out [A*items*16][128]
 *   iplan_gat128_gates   GRUCell gate math (:140) from gi, gh [rows][384] (biases included) and h_prev -> out [rows][128] */
int iplan_gat128_recur(const float* P, const float* Q, const float* whh, const float* bhn, const float* lw, float* dl,
                       int n_agents, int64_t n_items, void* stream);
int iplan_gat128_attend(const float* qkv, const float* v_bias, const float* dl, const float* he_b, const float* gumbel,
                        uint64_t seed, uint64_t counter, float tau, float* x, int n_agents, int64_t n_items, void* stream);
int iplan_gat128_gates(const float* gi, const float* gh, const float* hprev, float* out, int64_t rows, void* stream);

/* ---- K1b: behaviour-encoder step -----------------------------------------------
 * replaces Behavior_policy.latent_update (nova/stable_behavior_policy.py:83-123)
 * = EncoderRNN.forward (nova/behavior_net.py:17-22) over the history window from the
 * carried hidden state, softmax latent, soft update (1-c)*prev + c*new.
 *   window    [a][b][n][hist_len*obs_dim]
 *   hid_io    [a][b][n][32]  GRU hidden, updated in place
 *   lat_prev  [a][b][n][latent_dim];  lat_out likewise (may alias lat_prev) */
int iplan_behavior_step(const float* beh_params, int64_t param_stride,
                        iplan_view window, iplan_view hid_io, iplan_view lat_prev, iplan_view lat_out,
                        float soft_coef,
                        int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int hist_len,
                        void* stream);

/* iplan_behavior_step reading the window rows in place from a time-strided store (no shifted copy of the window):
 *   win_stride_step == 0   as iplan_behavior_step: `window` is [a][b][n][hist_len*obs_dim], rows contiguous
 *   win_stride_step != 0   window row w (0 = oldest) of a node is at window.ptr + (w - win_pad) * win_stride_step for
 *                          w >= win_pad and all-zero for w < win_pad (observation_wrapper.py:101-119 pads in front);
 *                          e.g. the packed episode store: window.ptr -> history at time max(0, t - hist_len + 1),
 *                          win_stride_step = the store's time stride, win_pad = max(0, hist_len - 1 - t). */
int iplan_behavior_step_ex(const float* beh_params, int64_t param_stride,
                           iplan_view window, int64_t win_stride_step, int win_pad,
                           iplan_view hid_io, iplan_view lat_prev, iplan_view lat_out,
                           float soft_coef,
                           int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int hist_len,
                           void* stream);

/* ---- host-buffer entry points of the rollout step (csrc/host_api.cu) -----------------------------------------------------
 * What a binding of the reference's numpy API calls: Prediction_policy.GAT_latent_update (nova/prediction_policy.py:92-118)
 * and Behavior_policy.latent_update (nova/stable_behavior_policy.py:83-123) with HOST arrays in the reference's own layout
 * ([B][A][N][*], C order).  The env dimension is cut into n_chunks (<= 16) pieces: piece c goes host -> device on a copy stream,
 * its kernel runs on `stream` when it has landed, its result goes device -> host on a second copy stream while piece c + 1
 * computes; the call returns when host_out is complete (synchronous, like the reference).  A NULL host pointer means the
 * device buffer already holds that array (e.g. the previous call's result, still resident): nothing is uploaded for it.
 * dev_* are caller-owned device buffers of the full [B][A][N][*] size (staging for the uploaded arrays; dev_out / dev_new
 * receive the result and stay valid).  Host buffers may be pageable; page-locked ones overlap with the kernels.
 * The GAT noise counter of piece c is counter + c.  chunk_end: NULL (equal pieces) or the n_chunks increasing end indices of
 * the pieces (last = n_envs): K1 runs in waves of CTAs over the SMs, so pieces sized in whole waves with a short last piece (whose copy-out
 * nothing overlaps) cost no extra wave. */
int iplan_gat_latent_update_host(const float* gat_params, int64_t param_stride,
                                 const float* host_hist, float* dev_hist, const float* host_h, float* dev_h,
                                 const float* host_beh, float* dev_beh, float* dev_out, float* host_out,
                                 uint64_t seed, uint64_t counter, float tau, float* scratch, int64_t scratch_floats,
                                 int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int n_chunks, const int32_t* chunk_end,
                                 void* stream);
/* host_window [B][A][N][hist_len][o], host_prev / host_new [B][A][N][L], dev_hid_io [B][A][N][32] (updated in place) */
int iplan_behavior_latent_update_host(const float* beh_params, int64_t param_stride,
                                      const float* host_window, float* dev_window, const float* host_prev, float* dev_prev,
                                      float* dev_hid_io, float* dev_new, float* host_new, float soft_coef,
                                      int n_envs, int n_agents, int n_slots, int obs_dim, int latent_dim, int hist_len, int n_chunks, void* stream);
/* n device -> host copies on `stream`, then one synchronize (select_actions_ippo returns four small arrays) */
int iplan_d2h_batch(void* const* dst_host, const void* const* src_dev, const int64_t* bytes, int n, void* stream);

/* ---- K1c: controller step (actor + critic, one timestep) -------------------------
 * replaces DcntrlMAC.select_actions_ippo (controllers/dcntrl_controller.py:27-58):
 * LayerNorm(F) -> fc1 -> ReLU -> LN -> fc2 -> ReLU -> LN -> 1-step GRU -> LN ->
 * Categorical head (masked logits, sample / mode, log-prob) and value head.
 *   feat      [A][B][row_stride] controller input rows (feature order of
 *             _build_inputs, :187-213), row pitch `feat_stride_env`, agent pitch
 *             `feat_stride_agent` (floats)
 *   rnn_*_in/out  [A][B][64] with the given agent/env strides (separate for in and out)
 *   avail     NULL (all available) or uint8 [A][B][n_actions]
 *   uniforms  NULL -> Philox(seed, counter); else [A][B] in [0,1) (parity mode)
 *   greedy    1 -> mode() (test_mode=True)
 *   outputs   actions int32 [A][B], logp [A][B], values [A][B], logits [A][B][n_actions] (or NULL)
 *   next_onehot  NULL or pointer to the last-action columns of the NEXT timestep's
 *             rows (same strides as feat); the chosen action's one-hot is written there */
int iplan_controller_step(const float* actor_params, int64_t actor_stride,
                          const float* critic_params, int64_t critic_stride,
                          const float* feat, int64_t feat_stride_agent, int64_t feat_stride_env,
                          const float* rnn_a_in, const float* rnn_c_in,
                          float* rnn_a_out, float* rnn_c_out,
                          int64_t rnn_stride_agent, int64_t rnn_stride_env,
                          int64_t rnn_out_stride_agent, int64_t rnn_out_stride_env,
                          const uint8_t* avail, const float* uniforms,
                          uint64_t seed, uint64_t counter, int greedy,
                          int32_t* actions, float* logp, float* values, float* logits,
                          float* next_onehot, float* this_onehot,
                          int n_envs, int n_agents, int feat_dim, int n_actions,
                          void* stream);

/* ---- observation-history wrapper step (SURVEY §8f rank 4) ------------------------------
 * replaces observersation_state_history_wrapper.obs_history_create + obs_history_output +
 * obs_single_history_output (observation_wrapper.py:68-141) for one timestep:
 *   obs        [B][A][n_obs][obs_dim] raw observation rows, column 0 = vehicle id, all-zero rows = nothing observed
 *   slot_ids   [B][A][n_slots] int32 state: ids in first-seen order (slot = position); slot_count [B][A] (zero both to reset)
 *   window     [B][A][n_slots][hist_len][obs_dim-1] state and output: the last hist_len history rows of every slot
 *   single     [B][A][n_slots][obs_dim-1] output: the row appended this step (zeros for unobserved slots)
 *   overflow   [1] set to 1 if an agent met more than n_slots distinct ids (the reference raises IndexError) */
int iplan_obs_history_step(const float* obs, int n_envs, int n_agents, int n_obs, int obs_dim,
                           int32_t* slot_ids, int32_t* slot_count, float* window, float* single,
                           int32_t* overflow, int n_slots, int hist_len, void* stream);

/* ---- Prediction_policy.learn (SURVEY §8f rank 2; nova/prediction_policy.py:168-253) ------------------------------
 * Arithmetic specified line by line by oracle/iplan_oracle.py (prediction_learn_agent, gat_backward_manual).
 * One launch = forward, masked-L1 loss and backward of the GAT + trajectory decoder over P sampled transitions per
 * agent-net; gradients are ADDED into g_gat / g_dec (zero them first; parameter-buffer layout, iplan_gat_layout /
 * iplan_pdec_layout), the un-normalised loss sum |err| * mask into loss_sum[a].  Clip + Adam: iplan_learner_adam on the
 * two gradient buffers.
 *   x0 [A][P][N][o], lat0 [A][P][N][L], att0 [A][P][N][32], target [A][P][N][pred_len][o], mask [A][P] (0/1)
 *   gumbel NULL (Philox) or [A][P][N][N-1][2]; keep NULL (Philox) or uint8 [A][P][pred_len][N][32] dropout keep flags
 *   scale [A] = o * pred_len / (number of unmasked target elements + 1e-10)  (:230) */
#define IPLAN_PDEC_NTENSORS 8     /* nova/prediction_net.py:7-16 (DecoderRNN inside Prediction_Decoder) */
int64_t iplan_pdec_layout(int obs_dim, int64_t* offsets);
int64_t iplan_pred_learn_scratch_floats(int n_agents, int n_samples, int n_slots, int obs_dim, int pred_len);
int iplan_pred_learn(const float* gat_params, int64_t gat_stride, const float* dec_params, int64_t dec_stride,
                     float* g_gat, float* g_dec,
                     const float* x0, const float* lat0, const float* att0, const float* target, const float* mask,
                     const float* gumbel, const uint8_t* keep, const float* scale, float* loss_sum,
                     float* scratch, int64_t scratch_floats, uint64_t seed, uint64_t counter, float tau, float p_drop,
                     int n_agents, int n_samples, int n_slots, int obs_dim, int latent_dim, int pred_len, void* stream);

/* ---- Behavior_policy.learn (SURVEY §8f rank 3; nova/stable_behavior_policy.py:161-279) -----------------------------
 * Arithmetic specified line by line by oracle/iplan_oracle.py::behavior_learn_agent.
 * One call = the reconstruction loss over every window position of every episode and its gradients (one BPTT through
 * the encoder GRU, the decoder GRU and the latent recursion; three launches with the default implementation: encoder
 * forward, decoder forward + backward, encoder backward), ADDED into g_enc / g_dec (zero them first; layouts
 * iplan_beh_layout / iplan_bdec_layout).  behavior_variation_penalty = 0 only (the stability term is reported, not
 * differentiated).
 *   hist [A][B][T][N][o] (the batch without its last step), mask [A][B][T], scale [A][T-1-W] = o N / (unmasked elements
 *   of the next-window + 1e-10) / (T-1-W); keep NULL (Philox) or uint8 [A][B][T-1-W][N][W][64]; b_loss, s_loss [A] += */
#define IPLAN_BDEC_NTENSORS 8     /* nova/behavior_net.py:25-38 (DecoderRNN inside Behavior_Latent_Decoder), hidden = IPLAN_RNN */
int64_t iplan_bdec_layout(int obs_dim, int latent_dim, int64_t* offsets);
int64_t iplan_beh_learn_scratch_floats(int n_agents, int n_eps, int n_pos, int n_slots, int obs_dim, int latent_dim, int hist_len);
/* 0 (default) = three register-tiled launches (csrc/beh_learn_tile.cu: encoder forward, decoder forward + backward, encoder
 * backward; a CTA walks 64 chains in lock step), 1 = the one-warp-per-chain draft (csrc/beh_learn.cu), kept as the cross-check.
 * Returns the previous setting; iplan_beh_learn_scratch_floats answers for the active implementation.  With keep == NULL the
 * two draw different (equally distributed) Philox dropout masks. */
int iplan_beh_learn_set_impl(int impl);
int iplan_beh_learn(const float* enc_params, int64_t enc_stride, const float* dec_params, int64_t dec_stride,
                    float* g_enc, float* g_dec, const float* hist, const float* mask, const float* scale, const uint8_t* keep,
                    float* b_loss, float* s_loss, float* scratch, int64_t scratch_floats,
                    uint64_t seed, uint64_t counter, float p_drop, float soft_coef, float thres_small_variation,
                    int n_agents, int n_eps, int n_steps, int n_slots, int obs_dim, int latent_dim, int hist_len, void* stream);

/* ==== IPPO learner (IPPOLearner.train, learners/ippo_learner.py:227-317) ===============
 * All agents are processed together.  Agent a's input matrix is X_a[rows][ldx] with
 * rows = n_eps*(T+1), row (b,t) at index b*(T+1)+t — the packed EpisodeBatch layout.
 * Gradient buffers have the SAME flat layout as the parameter buffers. */

/* LayerNorm(F) statistics of every input row (parameter-free; once per train()):
 * stat [A][rows][2] = (mean, 1/sqrt(var+1e-5)).  utils/mappo_utils/mlp.py:45,51 */
int iplan_learner_row_stats(const float* X, int64_t x_stride_agent, int ldx, int feat_dim, int64_t rows,
                            int n_agents, float* stat, void* stream);

/* f16 hi / lo split of the (constant) input rows, once per train(): X = Xh + Xl to ~2^-22.
 * Xh, Xl: __half arrays with X's shape.  The two big products below stream these copies. */
int iplan_learner_x_split(const float* X, int64_t n_elems, void* Xh, void* Xl, void* stream);

/* feature LayerNorm + fc1 of actor and critic as ONE tensor-core product over X (mlp.py:50-56):
 * Z1 [A][rows][128] (actor 0..63 | critic 64..127).  Wh/Wl [A][128][ldx] __half and ws/cc [A][128]
 * are scratch (the LayerNorm-folded weights, rebuilt each call).  ldx % 32 == 0. */
int iplan_learner_fc1_forward(const float* actor, int64_t actor_stride, const float* critic, int64_t critic_stride,
                              const void* Xh, const void* Xl, int64_t x_stride_agent, int ldx, int feat_dim,
                              int64_t rows, int n_agents, const float* stat, void* Wh, void* Wl,
                              float* ws, float* cc, float* Z1, void* stream);

typedef struct {
    const float* actor; const float* critic; int64_t actor_stride, critic_stride;   /* parameters */
    float* g_actor; float* g_critic;                                                /* gradients (train) */
    int feat_dim, n_actions, n_agents, T1, n_eps, n_train_eps;
    const float* rnn_a; const float* rnn_c; int64_t rnn_stride_agent; int rnn_ld;   /* stored GRU inputs [a][row][64] */
    const int32_t* actions;        /* [A][rows] */
    const uint8_t* avail;          /* NULL or [A][rows][n_actions] */
    float* Z1; float* A1; float* Z2; float* A2; float* GI; float* GH;  /* work: [A][rows][128], 3x[A][2][rows][64], 2x[A][2][rows][192] */
    const float* stat; float* SM;  /* row stats; [A][2][128] scratch (zeroed by the caller each epoch) */
    float* logp_out; float* ent_out; float* value_out;                  /* eval outputs [A][rows] (NULL ok) */
    const float* old_logp; const float* old_value; const float* returns; const float* adv_raw; const float* alive; /* [A][rows] */
    const float* norm;             /* [A][4] from iplan_learner_adv_finalize */
    float* stats;                  /* [A][8] += policy loss, value loss, entropy, ratio, actor |g|, critic |g| */
    float clip, ent_coef, v_coef, huber_delta;
    float grad_scale;              /* power-of-two loss scale: every gradient buffer holds grad_scale * g
                                      (keeps the backward operands inside f16's normal range for the
                                      split-f16 tensor-core products); pass the same value to iplan_learner_adam */
} iplan_learner_ctx;

/* Z1 -> LN/ReLU -> fc2 -> LN/ReLU -> GRU step -> LN -> heads (R_Actor.evaluate_actions,
 * ippo_actor.py:74-102; R_Critic.forward, ippo_critic.py:47-65).
 * train == 0: writes logp_out / ent_out / value_out.
 * train != 0: K2b — fuses the PPO losses (ppo_update :185-197, cal_value_loss :128-159,
 *   entropy bonus) with their backward; leaves dZ1*rstd in Z1 and every gradient except
 *   fc1.weight / feature_norm in g_actor / g_critic. */
int iplan_learner_tail(const iplan_learner_ctx* ctx, int train, void* stream);

/* fc1.weight and feature_norm gradients from dZ1 (left in Z1 by the train tail): tensor-core
 * product G = dZ1^T X over the f16 copies.  Scratch: Dh/Dl [A][rows][128] __half (scaled split of
 * dZ1), gscale [2A] floats, G [A][128][ldx] floats. */
int iplan_learner_fc1_backward(const float* actor, int64_t actor_stride, const float* critic, int64_t critic_stride,
                               float* g_actor, float* g_critic,
                               const void* Xh, const void* Xl, int64_t x_stride_agent, int ldx, int feat_dim,
                               int64_t rows, int n_agents,
                               const float* dZ1, void* Dh, void* Dl, float* gscale,
                               const float* SM, float* G, void* stream);

/* K2a: GAE backward scan (compute_returns :344-365), raw advantages zeroed where the agent is
 * dead (:273-277) and their moments: moments [A][4] = (sum, sum of squares, count, sum of
 * alive over the training rows) in double — all-reduce them across ranks, then finalise:
 * norm [A][4] = (mean, 1/(unbiased std + 1e-5), 1/sum alive, 1/n_train_rows_global)  (:278-279) */
int iplan_learner_gae(const float* values, const float* reward, const float* alive, float gamma, float lam,
                      int T1, int n_eps, int n_train_eps, int n_agents,
                      float* returns, float* adv_raw, double* moments, void* stream);
int iplan_learner_adv_finalize(const double* moments, double n_train_rows_global, float* norm, int n_agents, void* stream);

/* clip_grad_norm_(max_norm) + torch.optim.Adam step (:205-223, :74-81) on a flat [A][total]
 * buffer; `mask` [total] is 1 where the optimiser owns the value. Adds the pre-clip norm to
 * stats[a][stat_col] when stats != NULL. */
int iplan_learner_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const float* mask,
                       float* sqnorm_scratch, int64_t stride, int64_t total, int n_agents,
                       float lr, float beta1, float beta2, float eps, int step, float max_norm,
                       float grad_scale, float* stats, int stat_col, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* IPLAN_B200_H */
