/* imb.h -- C ABI of libimb.so: the H100-native (sm_90a) GAIL/AIRL inner loop.
 *
 * The reference (HumanCompatibleAI/imitation) has no FFI/plugin registry; its boundary
 * for this path is the Python class API (SURVEY.md section 8b).  This header is the C-ABI
 * that sits directly under our Python mirror of that API (imitation_b200/): every entry
 * point below names the reference function(s) it replaces (paths relative to
 * /root/reference/src/imitation).  INTEGRATION.md shows the ctypes stub a maintainer
 * would add to the reference to call these.
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer owned by the caller
 *    (e.g. torch tensor .data_ptr()); nothing is allocated or freed inside the library;
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*), never
 *    synchronises, and is CUDA-graph capturable; per-call scalars that change from call to
 *    call live in the device-resident `imb_state` block so captured graphs can be replayed;
 *  - return value: 0 = ok, <0 = error (imb_last_error() gives the text, thread-local);
 *  - float32 arithmetic throughout; indices are int64 on the API, done masks uint8.
 *
 * Data layouts in HBM
 *  - transition TABLE (expert set, generator ring): AoS rows, row-major [capacity][tw],
 *    row = [obs(d_obs) | act(d_act; Discrete -> one-hot) | next_obs(d_obs) | done(1)],
 *    tw = 2*d_obs + d_act + 1.  Random row gathers read whole contiguous rows.
 *  - disc BATCH: SoA / feature-major [bw][ld], bw = tw + 1 (last feature row = log pi(a|s)),
 *    ld = row count rounded up to IMB_TILE_ROWS; padding columns [n, ld) are never used, so
 *    their contents do not matter (the tests fill them with NaN).  Streaming kernels read it
 *    in [feature][128-row] tiles staged into shared memory by cp.async.bulk (TMA unit).
 *  - ROLLOUT table (PPO): row-major [E*T][rw], row index = env*T + step,
 *    row = [obs(d_obs) | act(da_store) | logp | value | reward | adv | ret].
 *  - parameters: one flat fp32 vector per network in torch nn.Linear order
 *    (weight [out][in] row-major, then bias), so nn.Parameters can alias it.
 */
#ifndef IMB_H_
#define IMB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IMB_TILE_ROWS 128
#define IMB_MAX_HIDDEN 64   /* hidden widths 1..64, at most 2 hidden layers */
#define IMB_MAX_DIN 64      /* MLP input width 1..64 */
#define IMB_F_ZERO_GRAD 1    /* imb_disc_fwd_bwd: clear the gradient accumulator first */
#define IMB_F_TRAIN_NORM 2   /* imb_disc_fwd_bwd: Phi(s') uses the mid-update norm snapshot */
#define IMB_F_NO_TENSOR 4    /* imb_disc_fwd_bwd: force the fp32-FFMA kernel (A/B measurements; default = wgmma when the shape fits) */
#define IMB_RF_DETERMINISTIC 1 /* imb_rollout flags: act = mean / argmax (policy.predict(deterministic=True)) */
/* pol_act of the entry points that evaluate or plan a policy: the activation of both towers' hidden layers */
#define IMB_ACT_TANH 0       /* nn.Tanh (SB3's default, imitation's FeedForward32Policy) */
#define IMB_ACT_RELU 1       /* nn.ReLU (the reference's seals_hopper / walker / swimmer configurations) */

/* One MLP: [RunningNorm?] -> Linear(din,h1) -> act -> [Linear(h1,h2) -> act] -> Linear(h_last,n_out).
 * util/networks.py:204-283 (build_mlp).  Parameter block (at `param_off` floats into the
 * owning flat vector): W1[h1][din] b1[h1] W2[h2][h1] b2[h2] Wf[n_out][h_last] bf[n_out].  */
typedef struct imb_mlp {
  int32_t din;
  int32_t n_hidden;   /* 0, 1 or 2 */
  int32_t h1, h2;
  int32_t n_out;      /* 1 for reward/potential/value nets; d_act for the policy head */
  int32_t has_norm;   /* RunningNorm input layer (util/networks.py:98-134) */
  int32_t param_off;  /* float offset of this MLP's block in the flat parameter vector */
  int32_t norm_off;   /* float offset of [mean(din) | var(din)] in the norm-state vector */
  int32_t count_idx;  /* index of this norm's int32 count in the norm-count vector */
  float norm_eps;     /* 1e-5 */
} imb_mlp;

/* Discriminator / reward network description.
 * rewards/reward_nets.py:383-457 (BasicRewardNet), :674-736 (ShapedRewardNet),
 * :739-839 (BasicShapedRewardNet/BasicPotentialMLP); adversarial/gail.py:135-160,
 * adversarial/airl.py:67-119 (logit = r - log pi). */
typedef struct imb_disc_desc {
  int32_t d_obs, d_act;                       /* flattened widths (Discrete -> one-hot width) */
  int32_t use_state, use_action, use_next_state, use_done;
  imb_mlp base;
  int32_t shaped;                             /* 1: + gamma*(1-done)*Phi(s') - Phi(s) */
  imb_mlp potential;
  float gamma;
  int32_t subtract_logp;                      /* AIRL */
  int32_t n_params;                           /* total floats in the flat parameter vector */
} imb_disc_desc;

/* Adam hyper-parameters (torch.optim.Adam defaults: adversarial/common.py:123).  weight_decay > 0 = torch.optim.AdamW's
 * decoupled decay, param *= 1 - lr * weight_decay before the step (the reward trainer of preference comparisons,
 * algorithms/preference_comparisons.py:1182-1185); 0 = plain Adam. */
typedef struct imb_adam {
  float lr, beta1, beta2, eps, weight_decay;
} imb_adam;

/* Device-resident counters (int64 words) so that captured graphs replay correctly. */
enum {
  IMB_ST_RING_IDX = 0,    /* data/buffer.py Buffer._idx */
  IMB_ST_RING_N = 1,      /* Buffer._n_data */
  IMB_ST_EP_STEP = 2,     /* steps since the (lock-step) episode start */
  IMB_ST_EPISODE = 3,     /* episode counter (Philox reset stream) */
  IMB_ST_GLOBAL_STEP = 4, /* env steps taken per env since construction (noise stream) */
  IMB_ST_REPLAY_DRAW = 5, /* replay-sample draw counter */
  IMB_ST_EXPERT_POS = 6,  /* position inside the current expert permutation */
  IMB_ST_EXPERT_EPOCH = 7,
  IMB_ST_PPO_EPOCH = 8,   /* PPO permutation draw counter */
  IMB_ST_DISC_STEP = 9,   /* Adam step count of the discriminator */
  IMB_ST_PPO_STEP = 10,   /* Adam step count of the policy */
  IMB_ST_WORDS = 16
};

int imb_version(void);
const char* imb_last_error(void);
/* number of floats of workspace the discriminator kernels need (partials, accumulators).  The workspace must be
 * zero-filled when allocated: its launch tickets and launch record start from zero. */
int64_t imb_disc_workspace_floats(const imb_disc_desc* d);

/* ---- stage 3: discriminator ------------------------------------------------------------ */

/* RunningNorm.update_stats on a feature-major batch (util/networks.py:111-134; order of
 * operations BaseNorm.forward :79-91).  For a shaped net the potential norm is updated twice
 * (next_obs rows, then obs rows; SURVEY Appendix A.5) and the intermediate stats are kept in
 * `ws` for the forward pass.  batch: [bw][ld], rows [0,n) valid. */
int imb_disc_norm_update(const imb_disc_desc* d, const float* batch, int64_t ld, int64_t n,
                         float* norm_state, int32_t* norm_count, float* ws, void* stream);

/* RunningNorm.update_stats (util/networks.py:111-134) over `din` consecutive feature rows [row0, row0 + din) of a
 * feature-major batch, for a normaliser that is NOT the discriminator's own: the generator policy's
 * NormalizeFeaturesExtractor, which the reference updates as a side effect of `policy.evaluate_actions` on every
 * discriminator minibatch (algorithms/adversarial/common.py:606-615 with the policy left in train mode by SB3's
 * PPO.train).  defer == NULL: fold into (norm_state = [mean | var], norm_count) immediately.  defer != NULL: append the
 * batch moments to the slot list `defer` ([0] = number of slots in use, [4 + k * (2 din + 1) ...] = mean | var | n) so that
 * the update can be computed on a stream that runs beside the PPO update and applied afterwards, in order, by
 * imb_norm_fold.  The counter saturates at `defer_cap`: once the list is full, every further call overwrites the last
 * slot and leaves [0] == defer_cap, so those batches' moments are lost but a fold never reads past the list.  A caller
 * sizes the list for the most calls it makes between two folds.  `d` / `ws`: any discriminator descriptor + its
 * workspace (chunk partials live there). */
int imb_norm_batch_stats(const imb_disc_desc* d, const float* batch, int64_t ld, int64_t n, int row0, int din,
                                 float* norm_state, int32_t* norm_count, float* defer, int defer_cap, float* ws,
                                 void* stream);
int imb_norm_fold(int din, float* defer, float* norm_state, int32_t* norm_count, int n_slots /* <= 0: the list's own
                  counter, which is then reset; > 0: exactly that many slots (an all-gathered list), no reset */,
                  void* stream);
/* `train_disc` returns Mapping[str, float] (common.py:79-92): copy the n <= 15 statistics into HOST-MAPPED pinned memory
 * (16 floats) and then store the current value of state[state_idx] (the Adam step) as int32 into word 15; the host polls that
 * word -- no D2H memcpy, no event synchronisation on the critical path of the synchronous API. */
int imb_stats_publish(const float* stats_dev, int n, float* host_mapped, const int64_t* state, int state_idx, void* stream);
/* multi-GPU discriminator step (SURVEY 8e): after the [gradient | statistic sums] block at the start of the workspace
 * (n_params rounded up to 32 floats, then 5 sums) has been all-reduced over the ranks, record the GLOBAL row counts that
 * imb_disc_adam's statistics divide by (common.py:52-77 over the global 2 * minibatch rows). */
int imb_disc_set_rows(const imb_disc_desc* d, float* ws, int64_t n_rows_total, int64_t n_expert_total, void* stream);

/* Fused forward + BCE-with-logits + backward over one minibatch of n = 2*mb rows (expert rows
 * first: label 1, generator rows second: label 0), gradients ACCUMULATED into ws (scaled by
 * loss_scale = 1/(2*B), common.py:360-369).  Replaces RewardNet.forward + F.binary_cross_
 * entropy_with_logits + loss.backward() (common.py:353-369).  If grad_out != NULL the BCE is
 * skipped and grad_out[n] is used as dL/dlogit (autograd backward of RewardNet.forward).
 * logits_out[n] (optional) receives the logits.  flags: IMB_F_ZERO_GRAD clears the accumulator
 * first (common.py:346); IMB_F_TRAIN_NORM = the norm stats were just updated by
 * imb_disc_norm_update (training mode). */
int imb_disc_fwd_bwd(const imb_disc_desc* d, const float* params, const float* norm_state,
                     const float* batch, int64_t ld, int64_t n, int64_t n_expert,
                     float loss_scale, const float* grad_out, float* logits_out,
                     int flags, float* ws, void* stream);

/* Which kernel imb_disc_fwd_bwd (flags without IMB_F_NO_TENSOR) runs for the network `d` over n rows; host only, no
 * GPU needed.  <0 (imb_last_error() names the shared-memory need and limit) when imb_disc_fwd_bwd or
 * imb_reward_forward cannot run the shape at all; which of them fits does not depend on n. */
#define IMB_PLAN_TC 1          /* wgmma tensor-core kernel: unshaped 32x32 net, din <= 31, no done input, no log pi */
#define IMB_PLAN_FFMA128X2 2   /* fp32-FFMA kernel, 128-row tiles, two CTAs per SM */
#define IMB_PLAN_FFMA256 3     /* fp32-FFMA kernel, 256-row tiles, one CTA per SM (only for n > 128) */
#define IMB_PLAN_FFMA128 4     /* fp32-FFMA kernel, 128-row tiles, one CTA per SM */
int imb_disc_plan(const imb_disc_desc* d, int64_t n);

/* Finish the update: deterministic reduction of the per-CTA partials, optional copy of the
 * gradient to grad_out_flat (for external optimisers / all-reduce), optional Adam step
 * (common.py:372) and the 9 train stats of the LAST minibatch (common.py:27-92) into
 * stats_out[16] = {loss, acc, acc_expert, acc_gen, entropy, prop_expert_true,
 * prop_expert_pred, n_expert, n_generated}.  state[IMB_ST_DISC_STEP] is incremented.  The partials reduced are
 * those of the last imb_disc_fwd_bwd on the same workspace (none before the first). */
int imb_disc_reduce(const imb_disc_desc* d, float* ws, float* grad_out_flat, void* stream);
int imb_disc_adam(const imb_disc_desc* d, const imb_adam* opt, float* params, float* exp_avg,
                  float* exp_avg_sq, const float* grad_flat_or_null, float grad_div, float* ws,
                  int64_t* state, float* stats_out, void* stream);

/* Forward only (RewardNet.predict_th in eval mode, reward_nets.py:120-153; out_mode 0 = raw
 * net output, 1 = logits (AIRL subtracts log pi), 2 = GAIL reward -logsigmoid(-x),
 * gail.py:83). */
int imb_reward_forward(const imb_disc_desc* d, const float* params, const float* norm_state,
                       const float* batch, int64_t ld, int64_t n, int out_mode, float* out,
                       void* stream);

/* NormalizedRewardNet.predict_processed over T consecutive env steps of E rewards
 * (reward_nets.py:637-671): normalise step t with the running stats, THEN merge step t. */
int imb_reward_norm_scan(float* rews, int64_t n_envs, int64_t n_steps, int64_t step_stride,
                         int64_t env_stride, float* norm_state2, int32_t* norm_count, float eps,
                         int update_stats, void* stream);
/* The same scan for an output EMANorm (util/networks.py:137-201): ema_state3 = [running_mean, running_var,
 * inv_learning_rate] (float32), ema_counts2 = [count, num_batches] (int32).  Per step, after normalising with the
 * statistics from before it: inv_learning_rate += decay^num_batches (float32 powf), lr = 1 / inv_learning_rate,
 * dm = batch mean - mean, mean += lr * dm, var += lr * (batch var + (1 - lr) * dm^2 - var) (biased batch variance,
 * every operation rounded on its own), count += E, num_batches += 1.  0 < decay < 1. */
int imb_reward_ema_scan(float* rews, int64_t n_envs, int64_t n_steps, int64_t step_stride, int64_t env_stride,
                        float* ema_state3, int32_t* ema_counts2, float decay, float eps, int update_stats,
                        void* stream);

/* ---- stage 2: tables, ring buffer, sampling --------------------------------------------- */

/* Build AoS table rows from separate row-major arrays (ReplayBuffer.store, data/buffer.py:
 * 397-412, Buffer.store :147-214 with truncate_ok).  acts_f (float [n][d_act]) or acts_i
 * (int64 [n], one-hot encoded, RewardNet.preprocess reward_nets.py:88-111).  Rows are written
 * at ring positions (state[RING_IDX] + i) mod capacity for the LAST min(n,capacity) rows;
 * use_ring = 0 writes rows at i (expert table).  Ring header advanced by imb_ring_advance. */
int imb_table_store(float* table, int64_t capacity, int32_t d_obs, int32_t d_act,
                    const float* obs, const float* acts_f, const int64_t* acts_i,
                    const float* next_obs, const uint8_t* dones, int64_t n, int use_ring,
                    const int64_t* state, void* stream);
int imb_ring_advance(int64_t* state, int64_t capacity, int64_t n_stored, void* stream);

/* Index generation on device ("perf mode"; parity mode uploads host indices instead).
 * kind 0: with replacement in [0, state[RING_N]) -- Buffer.sample, buffer.py:216-232;
 * kind 1: next n entries of an endless sequence of Feistel permutations of [0,size) with
 * drop_last semantics -- make_data_loader(shuffle, drop_last) + endless_iter,
 * algorithms/base.py:272-282, util/util.py:215-241. */
int imb_sample_indices(int kind, int64_t* idx_out, int64_t n, int64_t size, uint64_t seed,
                       int64_t* state, void* stream);

/* Device sampling + gather of one discriminator minibatch in ONE launch: batch columns [0, mb) =
 * expert rows drawn like imb_sample_indices(kind 1), columns [mb, 2 mb) = generator-ring rows drawn
 * like kind 0, both at offset `start` of the update's draws (common.py:552 `sample` + :592-595
 * concatenate + the DataLoader batch of :208-216).  The draw counters advance once per update:
 * imb_sample_advance2(demo_batch_size, ...).  Bit-identical to the unfused calls. */
int imb_disc_sample_gather(const float* expert_table, int64_t n_expert, const float* ring,
                           int64_t ring_capacity, int32_t tw, int64_t mb, int64_t start,
                           uint64_t seed, const int64_t* expert_state, const int64_t* ring_state,
                           float* batch, int64_t ld, void* stream);
int imb_sample_advance2(int64_t n, int64_t n_expert, int64_t* expert_state, int64_t* ring_state,
                        void* stream);

/* Gather table rows by index into the feature-major batch at column col0 (idx == NULL ->
 * rows 0..n-1).  A warp loads 32 indices coalesced, then walks them by warp shuffle so that
 * each row is read by consecutive lanes; the 32x tw tile is transposed through shared memory
 * so batch writes are coalesced too.  Buffer.sample gather (buffer.py:231-232) + the
 * concatenate of common.py:592-595. */
int imb_gather_rows(const float* table, int64_t capacity, int32_t tw, const int64_t* idx,
                    int64_t n, float* batch, int64_t ld, int64_t col0, void* stream);

/* ---- stage 1: generator rollouts (GPU-resident VecEnv + policy + reward relabel) ---------- */

/* Actor-critic policy (SB3 ActorCriticPolicy with separate pi / vf towers;
 * imitation policies/base.py:92-104 FeedForward32Policy; optional feature RunningNorm,
 * policies/base.py:123-149).  Flat parameter vector: pi tower | vf tower | action head
 * (imb_mlp with n_hidden = 0 semantics: Linear(h, d_act)) | value head | log_std[d_act].
 * The towers' activation is not part of the descriptor: every entry point that evaluates or
 * plans the policy takes it as `pol_act` (IMB_ACT_TANH or IMB_ACT_RELU; any other value is an error). */
typedef struct imb_policy_desc {
  int32_t d_obs, d_act;     /* d_act: action dim (Box) or number of actions (Discrete) */
  int32_t discrete;
  int32_t hidden;           /* tower width (two layers of this width, activation pol_act) */
  int32_t has_norm;         /* NormalizeFeaturesExtractor */
  float norm_eps;
  int32_t off_pi_w1, off_pi_b1, off_pi_w2, off_pi_b2;
  int32_t off_vf_w1, off_vf_b1, off_vf_w2, off_vf_b2;
  int32_t off_act_w, off_act_b, off_val_w, off_val_b, off_log_std;
  int32_t n_params;
} imb_policy_desc;

/* The environment the rollout kernels step, by kind; every kind is fixed-horizon with auto-reset:
 *   IMB_ENV_SYNTH     the synthetic MuJoCo-shaped env (defined by this repo, SURVEY section 8d):
 *                     obs' = tanh(A obs + Bm u + c), reward = w.obs' - 0.1|u|^2, parameters in env_params
 *   IMB_ENV_CARTPOLE  seals/CartPole-v0: d_obs 4, Discrete(2), never terminates (DESIGN section 7e)
 *   IMB_ENV_PENDULUM  Pendulum-v1: d_obs 3, Box(-2, 2, (1,)), never terminates (DESIGN section 7e)
 * The classic-control kinds read no env_params; their observation is the whole env state. */
#define IMB_ENV_SYNTH 0
#define IMB_ENV_CARTPOLE 1
#define IMB_ENV_PENDULUM 2
typedef struct imb_env_desc {
  int32_t d_obs, d_act, discrete, horizon;
  uint64_t seed;
  int32_t env_id_offset;    /* global id of this rank's env 0 (multi-GPU sharding) */
  int32_t kind;             /* IMB_ENV_* */
} imb_env_desc;

typedef struct imb_ppo_hparams {
  float gamma, gae_lambda, clip_range, ent_coef, vf_coef, max_grad_norm, lr, adam_eps;
  int32_t n_epochs, batch_size, normalize_advantage;
} imb_ppo_hparams;

/* One generator rollout of T steps for E envs in ONE launch (thread per env): policy
 * forward + sampling (OnPolicyAlgorithm.collect_rollouts), env step with auto-reset and
 * terminal-observation handling (data/wrappers.py:69-91, data/rollout.py:120-187), learned
 * reward relabel on (old_obs, clipped act, terminal-fixed next obs, done)
 * (rewards/reward_wrapper.py:92-133 -> RewardNet.predict_processed), time-limit bootstrap,
 * rollout rows, GAE, and the flattened transition rows in reference order
 * (pop_trajectories + flatten_trajectories, wrappers.py:132-148, rollout.py:563-621) written
 * straight into the generator ring with Buffer.store truncation (buffer.py:174-192).
 * reward_mode: 0 = env reward (debug_use_ground_truth), 1 = GAIL -logsigmoid(-logit),
 * 2 = raw reward-net output (AIRL; normalise afterwards with imb_reward_norm_scan).
 * noise (optional, [T][E][d_act] normals or [T][E] uniforms) pins sampling for parity;
 * flags: IMB_RF_DETERMINISTIC for evaluation rollouts (data/rollout.py:382-506). */
int imb_rollout(const imb_env_desc* env, const float* env_params, float* env_obs,
                const imb_policy_desc* pol, int32_t pol_act, const float* pol_params, const float* pol_norm,
                const imb_disc_desc* disc, const float* disc_params, const float* disc_norm,
                int reward_mode, const imb_ppo_hparams* hp, int64_t n_envs, int64_t n_steps,
                float* rollout, float* ring, int64_t ring_capacity, float* flat_out, float* aux,
                const float* noise, int flags, const int64_t* state, void* stream);
/* floats per rollout row: d_obs + (discrete ? 1 : d_act) + 5 (logp, value, reward, adv, ret), padded
 * to a multiple of 4 (16-byte aligned rows: imb_ppo_update stages each minibatch row with one bulk copy);
 * aux needs 2*E + 2*E*T floats (V(last obs), last done, per-step time-limit bootstrap,
 * per-step ground-truth env reward). */
int imb_rollout_row_width(const imb_policy_desc* pol);
/* Rows per CTA (8, 32, 64 or 128) imb_rollout / imb_rollout_ensemble run for these shapes; host only, no GPU needed.
 * disc == NULL: reward_mode 0; n_members 1: imb_rollout, 2..16: imb_rollout_ensemble; n_sms <= 0: the current device's
 * SM count.  The preferred tile is the smallest that covers the SMs (<= 16 envs per SM: 8 rows, <= 32: 32, <= 128: 64,
 * else 128); when its shared memory exceeds what a CTA can hold, the next smaller tile that fits runs instead.  <0
 * (imb_last_error() names the shared-memory need and the limit) when not even the 8-row tile fits. */
int imb_rollout_plan(const imb_policy_desc* pol, const imb_disc_desc* disc, int32_t n_members, int64_t n_envs,
                     int32_t n_sms);
/* GAE over the rollout table once rewards are final (SB3 RolloutBuffer.compute_returns_and_
 * advantage); call BEFORE imb_rollout_advance (it needs the pre-rollout episode step). */
int imb_gae(float* rollout, int32_t rw, int32_t col_value, int64_t n_envs, int64_t n_steps,
            const float* aux, float gamma, float gae_lambda, const int64_t* state_before,
            int32_t horizon, void* stream);
/* advance EP_STEP/EPISODE/GLOBAL_STEP (+ ring header when ring_capacity > 0) after a rollout */
int imb_rollout_advance(int64_t* state, int64_t n_envs, int64_t n_steps, int32_t horizon,
                        int64_t ring_capacity, void* stream);
/* VecEnv.reset() from Philox stream IMB_STREAM_ENV_RESET keyed by seed at counter (env id, episode): env_obs[d_obs][E] =
 * 0.1 * N(0,1) for the synthetic env, the kind's uniform reset draw for the classic-control ones (DESIGN section 7e).
 * <0 when env's kind and shapes do not match. */
int imb_env_reset(float* env_obs, int64_t n_envs, const imb_env_desc* env, const int64_t* state,
                  void* stream);

/* PPO.train as ONE persistent launch of an 8-CTA thread-block cluster: n_epochs x (N/batch)
 * sequential minibatch steps (gather by permutation, evaluate_actions, clipped surrogate + value +
 * entropy loss, backward, clip_grad_norm_, Adam).  Two kernels behind this entry point: k_ppo_update for tower width <= 32
 * and batch_size <= 64 (the reference's FeedForward32Policy with SB3's default minibatch: the minibatch is resident in
 * shared memory, one lane per hidden unit), k_ppo_update_gen for tower widths up to 64 (SB3 MlpPolicy 64x64) and
 * minibatches up to 4096 rows (tuned_hps airl_seals_walker: 128, airl_seals_hopper: 512), and for every ReLU policy
 * (pol_act = IMB_ACT_RELU; k_ppo_update is tanh only).  perm == NULL -> device Feistel
 * permutations.  loss_log (optional) [n_steps_total][4] = pg_loss, value_loss, entropy_loss, total. */
int imb_ppo_update(const imb_policy_desc* pol, int32_t pol_act, float* pol_params, float* pol_norm,
                   int32_t* pol_norm_count, float* exp_avg, float* exp_avg_sq,
                   const float* rollout, int64_t n_rows, const imb_ppo_hparams* hp,
                   const int64_t* perm, uint64_t seed, float* loss_log, int64_t* state,
                   void* stream);
/* imb_ppo_update with two more SB3 PPO options and the training statistics PPO.train records (SB3 2.2.1 PPO.train as
 * restated by oracle/ppo_port.py; unpinned, like the rest of the PPO port).  imb_ppo_update is this call with
 * target_kl = clip_range_vf = 0 and stats_out = NULL, and computes the same bits as it with any stats_out.
 *  - clip_range_vf > 0: value_loss = mse(ret, old + clamp(value - old, -c, c)), old = the rollout table's value column;
 *    the gradient flows where |value - old| <= c (torch's clamp backward).  <= 0: off.
 *  - target_kl > 0: a step whose approx_kl = mean(exp(lr) - 1 - lr), lr = logp - logp_old, exceeds 1.5 target_kl takes
 *    no optimiser step and ends the call.  Its statistics are recorded and its feature RunningNorm update stays;
 *    state[IMB_ST_PPO_STEP] advances by the optimiser steps taken, state[IMB_ST_PPO_EPOCH] by the epochs begun.  <= 0: off.
 *  - stats_out (optional) [IMB_PPO_STAT_FLOATS]: entropy / policy-gradient / value loss and clip fraction = means over
 *    the steps evaluated (each step weighted equally); approx_kl = mean over the steps of the last epoch begun; loss = the
 *    total loss of the last step evaluated; explained variance 1 - var(ret - value) / var(ret) over the rollout (NaN when
 *    var(ret) = 0); std = mean exp(log_std) after the call (NaN: Discrete); n_updates = state[IMB_ST_PPO_EPOCH] after
 *    the call; the steps evaluated and epochs begun by this call; 1 when target_kl stopped it. */
#define IMB_PPO_STAT_ENTROPY_LOSS 0
#define IMB_PPO_STAT_PG_LOSS 1
#define IMB_PPO_STAT_VALUE_LOSS 2
#define IMB_PPO_STAT_APPROX_KL 3
#define IMB_PPO_STAT_CLIP_FRACTION 4
#define IMB_PPO_STAT_LOSS 5
#define IMB_PPO_STAT_EXPLAINED_VARIANCE 6
#define IMB_PPO_STAT_STD 7
#define IMB_PPO_STAT_N_UPDATES 8
#define IMB_PPO_STAT_N_STEPS 9
#define IMB_PPO_STAT_N_EPOCHS 10
#define IMB_PPO_STAT_STOPPED 11
#define IMB_PPO_STAT_FLOATS 16
int imb_ppo_update_ex(const imb_policy_desc* pol, int32_t pol_act, float* pol_params, float* pol_norm,
                      int32_t* pol_norm_count, float* exp_avg, float* exp_avg_sq,
                      const float* rollout, int64_t n_rows, const imb_ppo_hparams* hp,
                      float target_kl, float clip_range_vf, const int64_t* perm, uint64_t seed,
                      float* loss_log, float* stats_out, int64_t* state, void* stream);

/* Which kernel imb_ppo_update runs for the policy `pol` at minibatch size batch_size; host only, no GPU needed.
 * Honours IMB_PPO_FORCE_GENERAL.  <0 (imb_last_error() names the shared-memory need and limit) when no kernel can run
 * the shape.  Shapes within k_ppo_update's width and minibatch whose shared memory or parameter slice does not fit it
 * run on k_ppo_update_gen<1>. */
#define IMB_PPO_PLAN_UPDATE 1  /* k_ppo_update: tanh, tower width <= 32, minibatch <= 64 rows */
#define IMB_PPO_PLAN_GEN1 2    /* k_ppo_update_gen<1>: tower width <= 32 (every ReLU policy of that width) */
#define IMB_PPO_PLAN_GEN2 3    /* k_ppo_update_gen<2>: tower width 33 to 64 */
int imb_ppo_plan(const imb_policy_desc* pol, int32_t pol_act, int32_t batch_size);

/* Which instantiation of k_ppo_update imb_ppo_update runs for `pol` when imb_ppo_plan returns IMB_PPO_PLAN_UPDATE; host
 * only.  0: the one that reads the shape at run time (every shape without its own); 1: 17 obs / 6 actions Box with a
 * feature RunningNorm; 2: 27 / 8 Box with a feature RunningNorm; 3: 4 obs / Discrete(2) without one (all of width 32).
 * The shape-specialised instantiations compute bit for bit what the runtime-shape one computes.  Honours
 * IMB_PPO_FORCE_RUNTIME_SHAPE=1, which imb_ppo_update reads at every call and which makes it run instantiation 0. */
int imb_ppo_update_variant(const imb_policy_desc* pol);

/* Behavioural cloning: minibatches [j0, j0 + n_minibatches) of one BC.train() call (algorithms/bc.py:381-510) as ONE
 * launch of k_ppo_update_gen with the BC loss (the PPO update's persistent cluster kernel, forward / backward / slice
 * reduction / Adam shared with PPO).  Per minibatch: evaluate_actions on its rows, loss = -mean logp
 * - ent_weight * mean entropy + l2_weight * sum(w^2) / 2 (BehaviorCloningLossCalculator, bc.py:94-156) scaled by
 * minibatch_size / batch_size (bc.py:501) and accumulated; every batch_size / minibatch_size minibatches of the call
 * (bc.py:505) and after the call's last minibatch when final_flush = 1 (the incomplete batch, bc.py:507-510) one torch
 * Adam step (betas 0.9 / 0.999, lr, adam_eps; no gradient clipping).  final_flush = 2: the last minibatch ends the call
 * but its incomplete batch steps in a later flush-only launch (n_minibatches = 0, final_flush = 1, j0 = the call's
 * minibatch count), as the reference steps it after the last on_epoch_end; this launch writes the batch's metrics.  The value tower is not evaluated; its parameters get
 * only the L2 term.
 *  - table: [n_rows][imb_rollout_row_width(pol)] rollout-format rows; only obs | act (Discrete: the index) are read.
 *  - perm: int64 [epochs][n_rows], the DataLoader(shuffle=True, drop_last=True) order of the epochs the launch touches,
 *    from epoch j0 / (n_rows / minibatch_size) on; minibatch i is perm[epoch][(i % (n_rows / minibatch_size)) * mb ...].
 *  - norm_update: the policy is in training mode, so each minibatch updates the feature RunningNorm before its forward
 *    pass (evaluate_actions); 0 normalises with the statistics as they stand.
 *  - grad_carry: [n_params] floats (flat order), needed when batch_size > minibatch_size: the summed gradient of a batch
 *    a launch ends inside (j0 + n_minibatches not a multiple of batch_size / minibatch_size, final_flush 0), read back by
 *    the launch that starts inside it.
 *  - metrics (optional): [n_logged][8] = neglogp, entropy, ent_loss, prob_true_act, l2_norm, l2_loss, loss
 *    (BCTrainingMetrics of the batch's last minibatch; l2_norm at its parameters) and the batch number, one row per
 *    batch that steps in this launch whose number (bc.py:504-509) is a multiple of log_interval, in order.
 *  - state[IMB_ST_PPO_STEP]: the Adam step count, advanced per step; state[IMB_ST_PPO_EPOCH]: epochs completed.
 * A split train() computes the same bits as one launch. */
int imb_bc_train(const imb_policy_desc* pol, int32_t pol_act, float* pol_params, float* pol_norm,
                 int32_t* pol_norm_count, float* exp_avg, float* exp_avg_sq, const float* table, int64_t n_rows,
                 int32_t minibatch_size, int32_t batch_size, int64_t j0, int64_t n_minibatches, int32_t final_flush,
                 float l2_weight, float ent_weight, float lr, float adam_eps, int32_t norm_update, const int64_t* perm,
                 float* grad_carry, float* metrics, int32_t log_interval, int64_t* state, void* stream);
/* The kernel imb_bc_train runs for `pol` at minibatch_size (IMB_PPO_PLAN_GEN1 or IMB_PPO_PLAN_GEN2); host only, no GPU
 * needed.  <0 (imb_last_error() names the shared-memory need and limit) when the shape does not fit. */
int imb_bc_plan(const imb_policy_desc* pol, int32_t pol_act, int32_t minibatch_size);

/* ---- DQN (SQIL's learner; SB3 2.2 DQN.train, restated by oracle/sqil_port.py) ------------------------------------------
 * The Q-net is a policy image: the pi tower and the action head are SB3's QNetwork (Flatten -> Linear -> act -> Linear ->
 * act -> Linear(h, n_actions)), the logits its Q values.  The value tower and value head are parameters no module owns,
 * left at zero: their gradient is 0, so clip_grad_norm_ and Adam leave them at zero.  Discrete actions, no feature
 * RunningNorm.
 *
 * imb_dqn_ring_store: the T steps of E envs an imb_rollout_explore just wrote as flat rows (flat_out, [E*T][tw]) into the
 * learner ring in SB3's ReplayBuffer order: the ring is a feature-major transition table [tw][positions * n_envs]
 * (tw = 2 d_obs + n_actions + 1, one-hot actions), step t of env e goes to column ((pos + t) mod positions) * n_envs + e
 * with pos = ring_state[IMB_ST_RING_IDX]; then pos advances by n_steps (mod positions) and ring_state[IMB_ST_RING_N]
 * (positions filled) by n_steps, capped at positions.  The flat row of (e, t) is the rollout's transition order from
 * episode step env_state[IMB_ST_EP_STEP], so the call goes between the rollout and imb_rollout_advance.  One launch.
 *
 * imb_dqn_target: the TD rows of n_steps minibatches of B = n_learner + n_expert rows, in one launch of the policy
 * forward's max-over-head mode on the TARGET Q-net.  Row r = s * B + i belongs to TD step k = s0 + s of the index lists,
 * s0 = state[IMB_ST_PPO_STEP] - step_base (state NULL: s0 = 0): i < n_learner reads column ring_idx[k * n_learner + i]
 * of the learner ring, else column expert_idx[k * n_expert + i - n_learner] of the expert table (both feature-major
 * transition tables [tw][ld], one-hot actions).  rows[r] (imb_rollout_row_width floats) = obs | action index | y with
 * y = reward + ((1 - done) * gamma) * max_a Q_target(next_obs)[a], reward = reward_learner or reward_expert, each operation
 * rounded separately as torch rounds DQN.train's float32 expression.
 * imb_dqn_step: n_steps TD steps on those rows as ONE launch of k_ppo_update_gen with the DQN loss (the PPO update's
 * persistent cluster kernel): step s takes rows [s * B, (s + 1) * B), loss = F.smooth_l1_loss(Q(obs)[a], y) (beta 1,
 * mean), backward (dL/dQ_a = clamp(Q_a - y, -1, 1) / B on the taken action), clip_grad_norm_(max_grad_norm), torch Adam
 * (betas 0.9 / 0.999, lr, adam_eps; bias corrections from state[IMB_ST_PPO_STEP], which advances per step).
 * loss_log (optional): element [(k - 1 - loss_base) * 4] = the loss of the step that brings state[IMB_ST_PPO_STEP] to k.
 * state[IMB_ST_PPO_EPOCH] advances by one per call.
 * Every per-call offset is read from the counter blocks, so a learn() iteration (rollout, ring store, advance, target
 * pass, TD steps) can be captured in a CUDA graph and replayed.
 * imb_dqn_plan: the kernel imb_dqn_step runs for `pol` at batch_size (IMB_PPO_PLAN_GEN1 or GEN2); host only; <0 naming
 * the limit when the Q-net or batch does not fit. */
int imb_dqn_ring_store(const float* flat, int32_t tw, float* ring, int64_t positions, int64_t n_envs, int64_t n_steps,
                       int32_t horizon, const int64_t* env_state, int64_t* ring_state, void* stream);
int imb_dqn_target(const imb_policy_desc* pol, int32_t pol_act, const float* target_params, const float* ring,
                   int64_t ring_ld, const int64_t* ring_idx, const float* expert, int64_t expert_ld,
                   const int64_t* expert_idx, int64_t n_learner, int64_t n_expert, int64_t n_steps, float gamma,
                   float reward_learner, float reward_expert, float* rows, int64_t step_base, const int64_t* state,
                   void* stream);
int imb_dqn_step(const imb_policy_desc* pol, int32_t pol_act, float* q_params, float* exp_avg, float* exp_avg_sq,
                 const float* rows, int32_t batch_size, int64_t n_steps, float lr, float adam_eps, float max_grad_norm,
                 float* loss_log, int64_t loss_base, int64_t* state, void* stream);
int imb_dqn_plan(const imb_policy_desc* pol, int32_t pol_act, int32_t batch_size);

/* ---- SAC (SQIL's continuous-action learner; SB3 2.2 SAC.train / collect_rollouts, restated by oracle/sac_port.py) -----
 * Nets: ReLU MLPs [h, h], one flat fp32 vector each in nn.Linear order (weight [out][in], then bias):
 *   actor          latent_pi.0 (Do -> h), latent_pi.2 (h -> h), mu (h -> Da), log_std (h -> Da)
 *   critic/target  qf0.0 (Do + Da -> h), qf0.2 (h -> h), qf0.4 (h -> 1), then qf1 alike
 * Envelope: 1 <= d_obs <= 64, 1 <= d_act <= 8, 1 <= hidden <= 256, 1 <= batch_size <= 256.
 *
 * imb_sac_collect: E envs (Box actions: Pendulum-v1 or the synthetic env) for T steps in one launch.  Step t of env e
 * is a random step when random_steps[state[IMB_ST_GLOBAL_STEP] + t - g0] is 1 (random_steps NULL: none): u uniform
 * from Philox stream IMB_STREAM_SAC_RANDOM keyed by seed at counter (env id, global step + t, a / 4), the sample
 * lo + u (hi - lo); otherwise the actor's tanh(mean + std eps) (eps: normals of IMB_STREAM_SAC_ACT at counter (env id,
 * global step + t, a / 4)), or tanh(mean) with flags & IMB_SAC_DETERMINISTIC.  The buffer action is scale(sample) or
 * scale(unscale(tanh(..))), the env action unscale(buffer action), in SB3's float32 operation order; with flags &
 * IMB_SAC_PREDICT (evaluation) the env action is predict()'s unscale(tanh(..)) and the row records it instead.  Flat row
 * flat_index(e, t) of flat_out ([E*T][2 Do + Da + 1]) = obs | buffer action | next obs (terminal at the horizon) |
 * done; the env reward goes to aux[2 E + E T + e T + t] (as imb_rollout_explore).  env_obs is read and written back;
 * state is read only (imb_rollout_advance advances it).
 *
 * imb_sac_step: n_steps SAC gradient steps (ent_coef: the fixed coefficient when auto_ent is 0), four launches each (critic phase, critic reduce + Adam, actor phase, actor
 * reduce + Adam + Polyak).  Step n = state[IMB_ST_PPO_STEP] (read on the device; advanced per step) takes minibatch
 * k = n - step_base: rows b < B/2 from columns ring_idx[k * (B/2) + b] of the learner ring [tw][ring_ld], the others
 * from columns expert_idx[k * (B - B/2) + b - B/2] of the expert table [tw][expert_ld] (feature-major, tw = 2 Do + Da +
 * 1), rewards reward_learner / reward_expert.  The actor's noise on s / s' of row b: normals 0-7 / 8-15 of Philox stream
 * IMB_STREAM_SAC_STEP keyed by seed at counter (b, n, chunk).  ent (auto_ent): [log_ent_coef, its Adam m, v].  Three
 * torch Adams (betas 0.9 / 0.999, lr, adam_eps; bias corrections from n + 1); the critic targets get the Polyak update
 * with tau at step s of the call when s % target_update_interval == 0.  loss_log (optional): row k = (critic_loss,
 * actor_loss, ent_coef_loss, ent_coef).  ws: imb_sac_ws_floats floats.  Every per-step offset is read on the device, so
 * the launches replay from a CUDA graph.
 * imb_sac_plan: 0, or <0 naming the limit the shape exceeds (host only). */
#define IMB_SAC_DETERMINISTIC 1
#define IMB_SAC_PREDICT 2
int imb_sac_plan(int32_t d_obs, int32_t d_act, int32_t hidden, int32_t batch_size);
int64_t imb_sac_ws_floats(int32_t d_obs, int32_t d_act, int32_t hidden, int32_t batch_size);
int imb_sac_collect(const imb_env_desc* env, const float* env_params, float* env_obs, int32_t hidden, const float* actor,
                    int64_t n_envs, int64_t n_steps, float* flat_out, float* aux, const uint8_t* random_steps,
                    int64_t g0, int32_t flags, uint64_t seed, const int64_t* state, void* stream);
int imb_sac_step(int32_t d_obs, int32_t d_act, int32_t hidden, int32_t batch_size, float gamma, float tau, float lr,
                 float adam_eps, int32_t auto_ent, float ent_coef, float target_entropy, float reward_learner,
                 float reward_expert, int32_t target_update_interval, uint64_t seed, float* actor, float* actor_m,
                 float* actor_v, float* critic, float* critic_m, float* critic_v, float* critic_target, float* ent,
                 const float* ring, int64_t ring_ld,
                 const int64_t* ring_idx, const float* expert, int64_t expert_ld, const int64_t* expert_idx,
                 int64_t n_steps, int64_t step_base, float* loss_log, float* ws, int64_t* state, void* stream);

/* log pi(a|s) of the generator policy for the disc batch (common.py:476-519 ->
 * ActorCriticPolicy.evaluate_actions), written into the batch's last feature row. */
int imb_policy_logp(const imb_policy_desc* pol, int32_t pol_act, const float* pol_params, const float* pol_norm,
                    float* batch, int64_t ld, int64_t n, int32_t row_logp, void* stream);

/* imb_disc_reduce + imb_disc_adam in one launch (last minibatch of an update; gradient taken from
 * the workspace accumulator). */
int imb_disc_reduce_adam(const imb_disc_desc* d, const imb_adam* opt, float* params, float* exp_avg,
                         float* exp_avg_sq, float grad_div, float* ws, int64_t* state,
                         float* stats_out, void* stream);

/* ---- preference comparisons (SURVEY 8 row f1) --------------------------------------------------
 * One minibatch of P fragment pairs of L transitions each: rews[2][P][L] are the reward network's outputs for the first
 * fragments, then the second fragments (row f * L + t).  PreferenceModel.probability (algorithms/preference_comparisons.py:
 * 487-530): d = clip(sum_t discount^t (r2 - r1), -threshold, threshold), p = noise_prob / 2 + (1 - noise_prob) / (1 + e^d);
 * CrossEntropyRewardLoss (:1043-1090): loss = mean_P BCE(p, pref) with torch's log clamp at -100, accuracy = mean((p > .5)
 * == (pref > .5)).  Outputs (each optional): grad_rews[2][P][L] = grad_scale * d loss / d rews (autograd's result, incl.
 * the zero gradient of clipped pairs and torch's BCE backward denominator clamp 1e-12) -- the upstream gradient for
 * imb_disc_fwd_bwd(grad_out=...); probs_out[P]; statistics slot `stats_slot` = the four floats at stats_acc + 4 * stats_slot:
 * [0] += loss, [1] += accuracy, [2] += 1 (so the per-minibatch means of an epoch -- one slot per epoch and per quantity
 * group -- are read back once).  The reference computes this with a Python loop over the pairs (:441-454). */
int imb_pref_loss(const float* rews, int64_t n_pairs, int32_t frag_len, const float* prefs, float noise_prob,
                  float discount, float threshold, float grad_scale, float* grad_rews, float* probs_out,
                  float* stats_acc, int32_t stats_slot, void* stream);

/* Regularization of the reward model's training step (regularization/regularizers.py), on the flat parameter vector
 * params[d->n_params], one single-CTA launch per minibatch:
 *  IMB_REG_LP (LpRegularizer, coeff = lambda): adds coeff * p * sign(w) |w|^(p-1) (the gradient of
 *    lambda * sum_tensors ||w||_p^p; 0 at w = 0) to the gradient accumulator of ws, so it goes between imb_disc_fwd_bwd
 *    (which clears the accumulator with IMB_F_ZERO_GRAD) and imb_disc_reduce / imb_disc_reduce_adam (which add the
 *    minibatch's gradient to it).  Statistics slot `stats_slot` of stats_acc (optional; imb_pref_loss's layout):
 *    [0] += coeff * sum |w|^p, [2] += 1, the sum without atomics (two calls give the same bits).
 *  IMB_REG_WEIGHT_DECAY (WeightDecayRegularizer, coeff = (float)(-lambda * lr)): w = w + coeff * w, a float32
 *    multiply then a float32 add (torch's th.add(w, c * w), bit for bit); ws and stats_acc are not used.  Goes after
 *    imb_disc_fwd_bwd has read the parameters and before the optimiser step.
 * p is an integer >= 1 (ignored by weight decay).  Stream-ordered, no allocation. */
#define IMB_REG_LP 1
#define IMB_REG_WEIGHT_DECAY 2
int imb_param_regularize(const imb_disc_desc* d, int32_t kind, int32_t p, float coeff, float* params, float* ws,
                         float* stats_acc, int32_t stats_slot, void* stream);

/* Active selection of preference queries: ActiveSelectionFragmenter.__call__ + variance_estimate
 * (algorithms/preference_comparisons.py:721-778), which loops over the candidate pairs in Python and calls
 * PreferenceModel.rewards -> RewardEnsemble.predict_processed_all (rewards/reward_nets.py:926-951) -> each member's
 * predict_processed twice per pair.  Member m's raw rewards are rews[m][2C][L] (fragment f = 2 i + s is pair i's first
 * (s = 0) or second (s = 1) fragment).  A member with norm_state[m] != NULL is a NormalizedRewardNet
 * (reward_nets.py:637-671): fragment f is normalised with its output statistics as they stood before f, then f's raw
 * rewards are merged into them (RunningNorm.update_stats, util/networks.py:121-134, or EMANorm.update_stats,
 * :175-201, by norm_kind[m]), in the order f = 0, 1, ..., 2C - 1;
 * the final statistics and count are written back.  mode 0 (logit): v_m = sum_t r1 - sum_t r2 (undiscounted), score =
 * variance with ddof 1; mode 1 (probability): v_m = PreferenceModel.probability (:487-530), score = variance with ddof 0;
 * mode 2 (label): v_m = (probability > 0.5), score = q (1 - q) with q = mean_m v_m.  Outputs: scores[C] and, optional,
 * member_out[C][M] = the return difference sum r1 - sum r2 (mode 0) or the probability (modes 1, 2) per member.  No
 * atomics in the arithmetic: two calls give the same bits.  ws: imb_pref_uncertainty_ws_floats(M, C) floats, zero-filled
 * when allocated; word 0 is a ticket that every call re-arms, so one workspace serves later calls of any size up to the
 * one it was sized for.  One launch, two when a member is normalised. */
#define IMB_PU_MAX_MEMBERS 16
typedef struct imb_pref_unc_desc {
  int32_t n_members;
  const float* rews[IMB_PU_MAX_MEMBERS];
  float* norm_state[IMB_PU_MAX_MEMBERS];   /* [mean, var] of the output RunningNorm, or NULL */
  int32_t* norm_count[IMB_PU_MAX_MEMBERS];
  float norm_eps[IMB_PU_MAX_MEMBERS];
  /* 0 (zero-filled) = output RunningNorm; 1 = output EMANorm (util/networks.py:137-201): norm_state[m] =
   * [mean, var, inv_learning_rate], norm_count[m] = [count, num_batches], folded per fragment as
   * imb_reward_ema_scan folds per step, with decay norm_decay[m] (0 < decay < 1) */
  int32_t norm_kind[IMB_PU_MAX_MEMBERS];
  float norm_decay[IMB_PU_MAX_MEMBERS];
} imb_pref_unc_desc;
int64_t imb_pref_uncertainty_ws_floats(int32_t n_members, int64_t n_pairs);
int imb_pref_uncertainty(const imb_pref_unc_desc* d, int64_t n_pairs, int32_t frag_len, int32_t mode,
                         float noise_prob, float discount, float threshold, float* ws, float* scores,
                         float* member_out, void* stream);

/* ---- agent training on an ensemble reward ----------------------------------------------------------------------------
 * RewardVecEnvWrapper with reward_fn = AddSTDRewardWrapper(RewardEnsemble(members), alpha).predict_processed or
 * RewardEnsemble(members).predict_processed (rewards/reward_wrapper.py:92-133 -> rewards/reward_nets.py:1045-1080,
 * :926-989 -> each member's predict_processed, :637-671 for a NormalizedRewardNet member).
 *
 * imb_rollout_ensemble = imb_rollout with reward_mode 2 for M members of the ONE architecture `disc`: member m has its
 * own parameter vector params[m] and input-norm state norm_state[m] (both laid out as `disc` describes; NULL norm state
 * when `disc` has no input RunningNorm).  Every member is evaluated in eval mode (input norms not updated) on the same
 * (obs, clipped act, terminal-fixed next obs, done) as imb_rollout's single net, and its raw output for env e at step t
 * goes to raw[(m * T + t) * E + e] instead of the rollout table's reward column.  All M member images are resident in
 * shared memory; the call fails, naming the limit, when they do not fit. */
typedef struct imb_rollout_members {
  int32_t n_members;                            /* 2 .. IMB_PU_MAX_MEMBERS */
  const float* params[IMB_PU_MAX_MEMBERS];
  const float* norm_state[IMB_PU_MAX_MEMBERS];  /* input RunningNorm state [mean | var] per `disc`'s norm_off, or NULL */
  float* raw;                                   /* [M][T][E] raw member outputs */
} imb_rollout_members;
int imb_rollout_ensemble(const imb_env_desc* env, const float* env_params, float* env_obs,
                         const imb_policy_desc* pol, int32_t pol_act, const float* pol_params, const float* pol_norm,
                         const imb_disc_desc* disc, const imb_rollout_members* members,
                         const imb_ppo_hparams* hp, int64_t n_envs, int64_t n_steps, float* rollout, float* ring,
                         int64_t ring_capacity, float* flat_out, float* aux, const float* noise, int flags,
                         const int64_t* state, void* stream);
/* The relabel of the ensemble rollout, before imb_gae: d->rews[m] = member m's raw[T][E] from imb_rollout_ensemble.
 * Per env step t, member m with d->norm_state[m] != NULL is normalised with its output statistics from before step t,
 * then step t's E raw rewards are merged into them (RunningNorm.update_stats, util/networks.py:121-134, or
 * EMANorm.update_stats, :175-201, by norm_kind[m]), so the
 * statistics and count end as E*T separate predict_processed calls leave them; a member without one is used raw.
 * rollout[(e*T + t)*rw + col_rew] = mean_m v_m + alpha * sqrt(var_m(v_m, ddof 1)), the mean and variance two-pass in
 * member order (alpha = 0 for a bare RewardEnsemble).  No atomics in the arithmetic: two calls give the same bits.
 * ws: imb_ensemble_relabel_ws_floats(M, T) floats, zero-filled when allocated (word 0 is a ticket every call re-arms). */
int64_t imb_ensemble_relabel_ws_floats(int32_t n_members, int64_t n_steps);
int imb_ensemble_relabel(const imb_pref_unc_desc* d, float alpha, float* rollout, int32_t rw, int32_t col_rew,
                         int64_t n_envs, int64_t n_steps, float* ws, void* stream);

/* ---- exploratory rollouts of preference comparisons -------------------------------------------------------------------
 * AgentTrainer.sample's exploration phase (algorithms/preference_comparisons.py:194-205, :231-307):
 * generate_trajectories over an ExplorationWrapper (policies/exploration_wrapper.py:23-95) that switches, for the whole
 * VecEnv at once, between the wrapped policy and a random one (action_space.sample()).  The switching chain does not
 * depend on observations, so the host draws it beforehand: explore_policy[t] (uint8 [T]) is 1 when step t is a
 * random-policy step, 0 when the policy acts.
 * = imb_rollout (members == NULL) or imb_rollout_ensemble (members != NULL, reward_mode 2, disc = the member
 * architecture, disc_params = disc_norm = NULL) without a ring, except on random steps: the towers are skipped, logp
 * and value are 0, and the action is low + u (high - low) on the Box [-1, 1] or min(floor(u n), n - 1) for Discrete(n),
 * with u a uniform of Philox stream IMB_STREAM_EXPLORE keyed by explore_seed at counter (env id, explore_step0 + t,
 * a / 4) -- or, with noise != NULL, the value in the slot the policy step would read ([T][E][d_act] or [T][E]).
 * explore_step0 < 0 reads the per-call scalars from the device, so that a captured launch replays exactly: the counter
 * of step t is state[IMB_ST_GLOBAL_STEP] + t, and its entry is explore_policy[state[IMB_ST_GLOBAL_STEP] + t - g0] with
 * g0 = -1 - explore_step0 (the global step the vector starts at).
 * Policy steps follow flags (IMB_RF_DETERMINISTIC: ExplorationWrapper(deterministic_policy=True)).  The env step, reward
 * relabel, env-reward column, terminal handling and flattened rows are imb_rollout's. */
int imb_rollout_explore(const imb_env_desc* env, const float* env_params, float* env_obs,
                        const imb_policy_desc* pol, int32_t pol_act, const float* pol_params, const float* pol_norm,
                        const imb_disc_desc* disc, const float* disc_params, const float* disc_norm,
                        const imb_rollout_members* members, int reward_mode, const imb_ppo_hparams* hp,
                        int64_t n_envs, int64_t n_steps, float* rollout, float* flat_out, float* aux,
                        const float* noise, int flags, const uint8_t* explore_policy, uint64_t explore_seed,
                        int64_t explore_step0, const int64_t* state, void* stream);

/* ---- DAgger rollouts (algorithms/dagger.py) ---------------------------------------------------------------------------
 * InteractiveTrajectoryCollector under generate_trajectories(expert, deterministic_policy=True) (algorithms/dagger.py:
 * 232-287): the expert acts, and where robot_mask[t * n_envs + e] (uint8 [n_steps][n_envs]) is 1 env e executes the
 * learner's action instead (policy.predict: sampled, clipped to the Box).  The mask does not depend on observations,
 * so the host draws it beforehand.
 * = imb_rollout with the expert as the policy (flags: IMB_RF_DETERMINISTIC for its mean / argmax) and reward_mode 0,
 * without a ring, except: no value tower or bootstrap runs; each rollout row holds obs | label, the label being the
 * expert's action clipped to the Box (Discrete: its index), the other columns of the row undefined; aux's V(last obs)
 * and bootstrap entries are 0.  The learner (its own width, activation learner_act and feature RunningNorm) runs only
 * at steps where a row of a tile has its mask bit set; its Box normals / Discrete uniforms come from Philox stream
 * IMB_STREAM_DAGGER keyed by env->seed at counter (env id, global step + t, a / 4), or, with robot_noise != NULL, from
 * robot_noise laid out as noise.  The env step, env-reward column of aux, terminal handling and flattened rows are
 * imb_rollout's. */
int imb_rollout_dagger(const imb_env_desc* env, const float* env_params, float* env_obs,
                       const imb_policy_desc* expert, int32_t expert_act, const float* expert_params,
                       const float* expert_norm, const imb_policy_desc* learner, int32_t learner_act,
                       const float* learner_params, const float* learner_norm, int64_t n_envs, int64_t n_steps,
                       float* rollout, float* flat_out, float* aux, const float* noise, const float* robot_noise,
                       int flags, const uint8_t* robot_mask, const int64_t* state, void* stream);
/* Rows per CTA (8, 32, 64 or 128) imb_rollout_dagger runs for these policies over n_envs envs on n_sms SMs (<= 0: the
 * current device's), chosen as imb_rollout_plan chooses with both policy images resident; host only. */
int imb_rollout_dagger_plan(const imb_policy_desc* expert, const imb_policy_desc* learner, int64_t n_envs,
                            int32_t n_sms);

/* ---- density-based reward (algorithms/density.py) ----------------------------------------------------------------------
 * DensityAlgorithm.__call__ (:295-360), which calls sklearn KernelDensity.score once per transition:
 *   r = log( (1/N_s) sum_i K_h(x - x_i) ),  x = (features - mean) / scale,
 * over the N_s standardised demonstration rows of segment s (a stationary model has one segment, a non-stationary one a
 * segment per episode step).  The query features are columns [col0, col0 + n0) then [col1, col1 + n1) of a source row in
 * transition-table format (state: obs; state-action: obs | act; state-state: obs | next_obs).
 * Demonstrations: n_tiles = ceil(N / IMB_DENSITY_TILE) tiles of IMB_DENSITY_TILE rows, grouped by segment in order,
 * demo[tile][k][row] feature-major inside a tile (so one bulk copy stages a tile), and demo_seg[tile][row] = the row's
 * segment, -1 for the padding rows of the last tile; seg_off[n_seg + 1] = each segment's first row (and N);
 * seg_const[n_seg] = sklearn's log kernel normalisation for (h, D, kernel) minus log N_s (float64).
 * Arithmetic: fp32 direct differences sum_k (q_k - x_k)^2 (no |q|^2 + |x|^2 - 2 q.x expansion), an online log-sum-exp
 * per query in fp32, then max + log(sum) + seg_const in float64, rounded to float32.  A compact kernel counts a pair
 * when d < h (fp32), as sklearn does; a query with no pair counted scores -inf.  Exact: sklearn's tree evaluation
 * with atol = rtol = 0 is not (DESIGN.md). */
#define IMB_DENSITY_TILE 64
#define IMB_DENSITY_MAX_D 128
#define IMB_KDE_GAUSSIAN 0
#define IMB_KDE_TOPHAT 1
#define IMB_KDE_EPANECHNIKOV 2
#define IMB_KDE_EXPONENTIAL 3
#define IMB_KDE_LINEAR 4
#define IMB_KDE_COSINE 5
/* The model (arguments d .. scale):
 *  d: the feature width D, 1 .. IMB_DENSITY_MAX_D; the features of a query are its source row's columns
 *     [col0, col0 + n0) then [col1, col1 + n1), n0 + n1 = D;
 *  kernel: IMB_KDE_*; bandwidth h > 0;
 *  n_seg segments of n_demo rows in all: demo [n_tiles][D][IMB_DENSITY_TILE] floats, demo_seg [n_tiles][IMB_DENSITY_TILE],
 *  seg_off [n_seg + 1], seg_const [n_seg] as described above; mean, scale [D]: the scaler. */
/* Query segments (seg_mode):
 *  IMB_DENSITY_SEG_NONE    query q reads source row q (row_map == NULL) or row_map[q], segment 0, writes out[row * out_stride];
 *  IMB_DENSITY_SEG_STEPS   as NONE with segment steps[q] (a host-provided steps vector; queries sorted by segment run
 *                          fastest, since a query tile reads only the demonstration tiles of its segments);
 *  IMB_DENSITY_SEG_ROLLOUT the E*T steps of the rollout that started at episode step t0 = state[IMB_ST_EP_STEP] (read on
 *                          the device: the launch can be captured in a graph): query q = t * E + e reads the flattened row
 *                          flat_index(e, t, E, T, t0, horizon) of `src` (imb_rollout's flat_out), has segment
 *                          (t0 + t) mod horizon, 0 when n_seg = 1 (a caller with n_seg > 1 checks that the episode
 *                          steps stay below n_seg), and writes out[(e * T + t) * out_stride] (the rollout table's reward
 *                          column); n_query = n_envs * n_steps.
 * A query whose segment is outside [0, n_seg) scores NaN.  When there are too few query tiles to fill the GPU, each
 * tile's demonstration tiles are split over several CTAs and the last one to finish (ticket) combines the partial sums
 * in split order; the split depends only on the shapes, so two calls give bit-identical results.
 * ws: imb_density_ws_floats(n_query) floats, zero-filled when allocated (it holds launch tickets every call re-arms).
 * One launch. */
#define IMB_DENSITY_SEG_NONE 0
#define IMB_DENSITY_SEG_STEPS 1
#define IMB_DENSITY_SEG_ROLLOUT 2
int64_t imb_density_ws_floats(int64_t n_query);
int imb_density_score(int32_t d, int32_t col0, int32_t n0, int32_t col1, int32_t n1, int32_t kernel, float bandwidth,
                      int32_t n_seg, int64_t n_demo, const float* demo, const int32_t* demo_seg, const int64_t* seg_off,
                      const double* seg_const, const float* mean, const float* scale, const float* src, int32_t src_ld,
                      const int64_t* row_map, int64_t n_query, int32_t seg_mode, const int64_t* steps, const int64_t* state, int64_t n_envs,
                      int64_t n_steps, int32_t horizon, float* out, int64_t out_stride, float* ws, void* stream);

/* ---- tabular MCE IRL (algorithms/mce_irl.py) ----------------------------------------------------------------------------
 * The time sweep of one finite-horizon MDP with S states, A actions and horizon H in ONE cooperative launch, float64
 * throughout, as the reference's NumPy computes it:
 *  IMB_MCE_BACKWARD  mce_partition_fh (:38-93): Q[H-1] = r, Q[t] = r + gamma_plan * (T @ V[t+1]) for t < H - 1,
 *                    V[t] = scipy.special.logsumexp(Q[t], axis=1), pi = exp(Q - V).  reward: exactly one of `reward`
 *                    (float64) and `reward32` (float32, widened: the reward net's output).
 *  IMB_MCE_FORWARD   mce_occupancy_measures (:96-144): D[0] = initial, D[t+1] = sum_a (D[t] pi[t, :, a]) @ T[:, a, :],
 *                    Dcum = rollout.discounted_sum(D, gamma_om) (polyval's Horner from t = H; a plain sum at 1).  With
 *                    BACKWARD too, pi is the one the backward sweep computed; alone, it reads the caller's pi.
 * transition: T as [S][A][S] (row (s, a) = the next-state distribution); discounts[2] = {gamma_plan, gamma_om} (device).
 * Outputs, each optional unless stated: V [H][S], Q [H][S][A], pi [H][S][A] (an input without BACKWARD), D [H+1][S],
 * Dcum [S] (required with FORWARD).  demo_om != NULL (FORWARD; MCEIRL._train_step): weights[s] = (float)(Dcum[s] -
 * demo_om[s]) rounded to nearest, *linf = max_s |Dcum[s] - demo_om[s]| (NaN propagates).  Every sum has a fixed order
 * and no floating-point atomics: two calls give the same bits.  ws: imb_mce_plan(...) doubles.
 * imb_mce_plan is host only: the workspace in doubles (and, when grid_out != NULL, a HOST int32 pointer, the CTA count of
 * the launch), or < 0 with imb_last_error() naming the limit when the shape is outside the envelope
 * (1 <= S <= IMB_MCE_MAX_STATES, 1 <= A <= IMB_MCE_MAX_ACTIONS, 1 <= H <= IMB_MCE_MAX_HORIZON).  n_sms <= 0: the
 * current device's SMs and the kernel's occupancy (what imb_mce_sweep launches); > 0: one CTA per SM, no GPU needed. */
#define IMB_MCE_BACKWARD 1
#define IMB_MCE_FORWARD 2
#define IMB_MCE_MAX_STATES 4096
#define IMB_MCE_MAX_ACTIONS 32
#define IMB_MCE_MAX_HORIZON 1000000
int64_t imb_mce_plan(int64_t n_states, int32_t n_actions, int32_t horizon, int32_t flags, int32_t n_sms,
                     int32_t* grid_out);
int imb_mce_sweep(int64_t n_states, int32_t n_actions, int32_t horizon, int32_t flags, const double* transition,
                  const double* initial, const double* reward, const float* reward32, const double* discounts,
                  double* V, double* Q, double* pi, double* D, double* Dcum, const double* demo_om, float* weights,
                  double* linf, double* ws, int64_t ws_doubles, void* stream);

/* ---- multi-GPU: replica state around the ONE all-reduce of a round ---------------------------
 * (SURVEY.md section 8e; the reference is single-process, so there is no reference interface to
 * cite: the merge restates RunningNorm's Chan update, util/networks.py:96-134, in its additive
 * sufficient-statistics form).  avg[i] (avg_n[i] floats) are averaged over the ranks; norm i is
 * (mean[k], var[k], int32 count) and is merged exactly relative to the round-start snapshot.
 * Staging buffers are float64: buf has imb_sync_buffer_doubles() entries, start the norm part. */
#define IMB_SYNC_MAX_AVG 8
#define IMB_SYNC_MAX_NORM 4
typedef struct imb_sync_desc {
  int32_t n_avg, n_norm;
  float* avg[IMB_SYNC_MAX_AVG];
  int64_t avg_n[IMB_SYNC_MAX_AVG];
  float* mean[IMB_SYNC_MAX_NORM];
  float* var[IMB_SYNC_MAX_NORM];
  int32_t* count[IMB_SYNC_MAX_NORM];
  int32_t k[IMB_SYNC_MAX_NORM];
} imb_sync_desc;
int64_t imb_sync_buffer_doubles(const imb_sync_desc* d);
int imb_sync_snapshot(const imb_sync_desc* d, double* start, void* stream);
int imb_sync_pack(const imb_sync_desc* d, double* buf, void* stream);
int imb_sync_unpack(const imb_sync_desc* d, const double* buf, const double* start, int32_t world,
                    void* stream);

/* zero the device-resident counter block */
int imb_state_init(int64_t* state, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* IMB_H_ */
