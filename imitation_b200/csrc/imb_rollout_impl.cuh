// imb_rollout_impl.cuh -- stage 1 of the GAIL/AIRL round: generator rollouts, GPU resident.
//
// One launch runs T environment steps for E environments; a CTA owns 8 to 128 environments (= tile rows)
// and every per-step network evaluation is a shared-memory tiled GEMM over that tile
// (imb_tile.cuh), with the environment state, the policy, the reward network and the synthetic
// dynamics all resident in shared memory for the whole rollout:
//   policy forward + sampling      SB3 OnPolicyAlgorithm.collect_rollouts (restated; see
//                                  oracle/ppo_port.py -- parity unpinned by the reference)
//   env step + auto-reset          synthetic MuJoCo-shaped env (SURVEY.md section 8d), or seals/CartPole-v0 /
//                                  Pendulum-v1 stepped thread per env in float64 (DESIGN.md section 7e);
//                                  VecEnv contract of data/rollout.py:161-186
//   reward relabel                 rewards/reward_wrapper.py:92-133 -> RewardNet.predict_processed
//                                  (reward_nets.py:120-204), GAIL transform gail.py:83
//   trajectory bookkeeping         data/wrappers.py:69-148 + data/rollout.py:563-621: the flattened
//                                  transition order (finished trajectories in completion order,
//                                  then partial ones in env order) has a closed form because the
//                                  envs are fixed-horizon and run in lock-step; rows go straight
//                                  into the generator ring with Buffer.store truncation/wrap
//                                  (data/buffer.py:174-192).
// Env state is SoA [d_obs][E] in HBM (coalesced tile load/store); environments never interact inside
// a rollout because the reward net and the policy run in eval mode.
// (First version: one thread per env with register-resident MLPs -- 250 KB of unrolled SASS per variant.)
#pragma once
#include "imb_common.cuh"
#include "imb_env_step.cuh"
#include "imb_mlp.cuh"
#include "imb_tile.cuh"

namespace {

constexpr int RT = 128;              // threads per CTA
// envs (tile rows) per CTA: RR = rows_of(RPL) = 8, 32, 64 or 128 (RPL = 0: the 8-row tile, else RPL rows per lane in
// the tiled layers); rollout_plan picks the smallest tile that still fills the GPU (the kernel's time is one CTA's
// latency, so smaller tiles are faster until the SMs run out), or a smaller one when that tile's shared memory does not
// fit; tile row stride RRS = RR + 4.

struct RolloutArgs {
  imb_env_desc env;
  imb_policy_desc pol;
  imb_ppo_hparams hp;
  int reward_mode;
  int deterministic;  // 1: act = mean (Box) / argmax (Discrete), like policy.predict(deterministic=True)
  int64_t E, T;
  int rw;             // rollout row width
  int64_t ring_capacity;
  // shared-memory plan (floats)
  int HP, JP, IP, KU;          // policy width, reward-net width, obs width (padded to 32), d_obs + d_act
  int pol_off, env_off, img_off, img_sz, obsu_off, xn_off, h1_off, h2_off, nobs_off, vec_off, total;
};

// Ensemble relabel (imb_rollout_ensemble): M members of the one architecture DiscLaunch describes, member m with its own
// parameter vector and per-pass input-norm state; member m's raw output of env e at step t goes to
// raw[(m * T + t) * E + e] (step-major: a step's E rewards are contiguous, as imb_ensemble_relabel reads them).
struct RolloutMembers {
  int M;
  const float* params[IMB_PU_MAX_MEMBERS];
  const float* norm[IMB_PU_MAX_MEMBERS][MAX_PASS];  // nullptr where the pass has no input RunningNorm
  float* raw;
};

// Exploration rollout (imb_rollout_explore, policies/exploration_wrapper.py): policy[t] = 1 makes step t a random-policy
// step for every env (action_space.sample(): uniform on the Box [-1, 1], or a uniform action index), drawn from Philox
// stream IMB_STREAM_EXPLORE keyed by `seed` at counter (env id, step0 + t, a / 4); with pinned noise the uniform is read
// from the slot the policy step would read.  step0 < 0 reads both from the device, so that a captured launch replays
// exactly: the counter is state[IMB_ST_GLOBAL_STEP] + t and the step's entry is policy[state[IMB_ST_GLOBAL_STEP] + t - g0]
// with g0 = -1 - step0 (the global step the vector starts at).
struct RolloutExplore {
  const uint8_t* policy;  // [T]: 0 = the wrapped policy, 1 = random
  uint64_t seed;
  int64_t step0;
};

// DAgger rollout (imb_rollout_dagger, algorithms/dagger.py): the policy of k_rollout is the expert; a second policy image,
// the learner (its own width, activation and feature norm), sits beside it.  mask[t * E + e] = 1 makes env e execute
// the learner's action at step t (sampled from Philox stream IMB_STREAM_DAGGER at counter (env id, global step + t,
// a / 4), or read from `noise`, laid out as k_rollout's); the row records obs | the expert's action, clipped to the Box.
struct RolloutDagger {
  imb_policy_desc pol;
  int act;          // the learner's tower activation (ACT_TANH / ACT_RELU)
  int HP, img_off;  // the learner's padded width and image offset (floats), set by rollout_layout
  const float* params;
  const float* norm;
  const float* noise;
  const uint8_t* mask;
};

enum { RM_PLAIN = 0, RM_EXPLORE = 1, RM_DAGGER = 2 };

// The action head of one policy for this thread's tile row (thread per env), on the pi latent H2: Box -> mean + std * z,
// z = 0 (deterministic), the pinned noise[nidx * Da + a] or a normal of Philox stream `stream` at counter (egid, ctr,
// a / 4); Discrete -> inverse-CDF sampling with the uniform noise[nidx] or one of that stream (argmax when
// deterministic).  CTRL[a * RRS] receives the control the env sees (the action clipped to the Box [-ahi, ahi] / the
// one-hot; Discrete uses it for the logits first); rec (nullable) the recorded action: Box unclipped unless clip_rec,
// Discrete the index.
// Returns log pi(action).
__device__ __forceinline__ float action_head(const float* __restrict__ psm, const PolImg& S, int HP, int h, int Da,
                                             bool discrete, const float* __restrict__ H2, int RRS, int rt,
                                             float* __restrict__ CTRL, float* __restrict__ rec, bool clip_rec,
                                             bool deterministic, const float* __restrict__ noise, int64_t nidx,
                                             bool live, uint64_t seed, uint32_t stream, uint32_t egid, uint32_t ctr,
                                             float ahi) {
  float logp = 0.f;
  if (!discrete) {
    float z4[4] = {0.f, 0.f, 0.f, 0.f};
    for (int a = 0; a < Da; ++a) {
      float m0 = 0.f, m1 = 0.f;
      const float* wa = psm + S.wa + a * HP;
      int j = 0;
      for (; j + 2 <= h; j += 2) {
        m0 = fmaf(wa[j], H2[j * RRS + rt], m0);
        m1 = fmaf(wa[j + 1], H2[(j + 1) * RRS + rt], m1);
      }
      if (j < h) m0 = fmaf(wa[j], H2[j * RRS + rt], m0);
      const float m = psm[S.ba + a] + (m0 + m1);
      if (!deterministic && !noise && (a & 3) == 0) philox_normal4(seed, stream, egid, ctr, a >> 2, z4);
      const float z = deterministic ? 0.f : noise ? (live ? noise[nidx * Da + a] : 0.f) : ((a & 3) == 0 ? z4[0] : (a & 3) == 1 ? z4[1] : (a & 3) == 2 ? z4[2] : z4[3]);
      const float ls = psm[S.lstd + a];
      const float sd = expf(ls);
      const float act = fmaf(sd, z, m);
      const float diff = act - m;
      logp += -(diff * diff) / (2.0f * sd * sd) - ls - 0.9189385332046727f;
      const float ctl = fminf(fmaxf(act, -ahi), ahi);
      if (rec) rec[a] = clip_rec ? ctl : act;  // SB3 stores the UNCLIPPED action; predict() returns the clipped one
      CTRL[a * RRS] = ctl;                     // env and wrappers see the clipped one
    }
  } else {
    float mx = -INFINITY;
    for (int a = 0; a < Da; ++a) {
      float m0 = 0.f;
      const float* wa = psm + S.wa + a * HP;
      for (int j = 0; j < h; ++j) m0 = fmaf(wa[j], H2[j * RRS + rt], m0);
      const float m = psm[S.ba + a] + m0;
      CTRL[a * RRS] = m;  // logits, overwritten by the one-hot below
      mx = fmaxf(mx, m);
    }
    float se = 0.f;
    for (int a = 0; a < Da; ++a) se += expf(CTRL[a * RRS] - mx);
    const float lse = mx + logf(se);
    float u;
    if (noise) {
      u = live ? noise[nidx] : 0.f;
    } else {
      uint32_t k0, k1;
      philox_key(seed, stream, k0, k1);
      u = u01(philox4x32(egid, ctr, 0u, 0u, k0, k1).x);
    }
    int chosen = Da - 1;
    float cdf = 0.f;
    bool found = false;
    for (int a = 0; a < Da; ++a) {
      cdf += expf(CTRL[a * RRS] - lse);
      if (!found && !(u >= cdf)) {
        chosen = a;
        found = true;
      }
    }
    if (deterministic) {
      chosen = 0;
      for (int a = 1; a < Da; ++a)
        if (CTRL[a * RRS] > CTRL[chosen * RRS]) chosen = a;
    }
    logp = CTRL[chosen * RRS] - lse;
    for (int a = 0; a < Da; ++a) CTRL[a * RRS] = (a == chosen) ? 1.f : 0.f;
    if (rec) rec[0] = (float)chosen;
  }
  return logp;
}

// ENS: evaluate the Mb.M ensemble members (raw outputs to Mb.raw) instead of the one net at disc_params (reward column);
// the single-net variant has no member loop.  ACT: the policy towers' activation (env and reward net keep their own).
// MODE RM_EXPLORE: the exploration rollout, Xp.policy[t] picks the policy of step t (random steps skip the policy
// towers and record logp = value = 0); otherwise Xp is unused.  MODE RM_DAGGER: the DAgger rollout (Dg; LACT the
// learner's activation): no value tower, bootstrap, reward net or ring, rows obs | expert label; otherwise Dg is unused.
template <int RPL, bool ENS, int ACT, int MODE, int LACT>
__global__ void __launch_bounds__(RT, 1) k_rollout(const RolloutArgs A, const DiscLaunch L, const RolloutMembers Mb,
                                                   const float* __restrict__ env_params, float* __restrict__ env_obs,
                                                   const float* __restrict__ pol_params,
                                                   const float* __restrict__ pol_norm,
                                                   const float* __restrict__ disc_params, float* __restrict__ rollout,
                                                   float* __restrict__ ring, float* __restrict__ flat_out,
                                                   float* __restrict__ aux, const float* __restrict__ noise,
                                                   const int64_t* __restrict__ state, const RolloutExplore Xp,
                                                   const RolloutDagger Dg) {
  constexpr bool DAG = MODE == RM_DAGGER;
  constexpr int RR = rows_of(RPL), RRS = RR + TILE_PAD;
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x;
  const int rt = tid < RR ? tid : RR - 1;  // tile row of this thread in the thread-per-env parts (threads >= RR idle there)
  const bool rowthread = tid < RR;
  const int Do = A.env.d_obs, Da = A.env.d_act, h = A.pol.hidden, HP = A.HP, JP = A.JP, IP = A.IP, KU = A.KU;
  const PolImg S(Do, Da, HP);
  float* psm = smem + A.pol_off;
  float* esm = smem + A.env_off;   // ABt[KU][IP] | c[IP] | w[IP]
  float* OBSU = smem + A.obsu_off; // [KU][RRS]: obs rows, then the control (clipped action / one-hot) rows
  float* XN = smem + A.xn_off;     // [max(KP)][RRS]: normalised MLP inputs
  float* H1 = smem + A.h1_off;
  float* H2 = smem + A.h2_off;
  float* NOBS = smem + A.nobs_off; // [IP][RRS]
  float* vec = smem + A.vec_off;   // lg[RT]
  float* lg = vec;

  const int n_mem = ENS ? Mb.M : 1;
  // ---- one-time loads ------------------------------------------------------------------------------
  if (A.reward_mode != 0)
    for (int m = 0; m < n_mem; ++m)
      for (int p = 0; p < L.npass; ++p)
        load_timg(smem + A.img_off + (m * L.npass + p) * A.img_sz, L.pass[p], JP, ENS ? Mb.params[m] : disc_params,
                  ENS ? Mb.norm[m][p] : (L.pass[p].has_norm ? L.pass[p].norm : nullptr), L.pass[p].eps);
  load_policy_img(psm, S, A.pol, HP, pol_params, pol_norm);
  const PolImg LS(Do, Da, DAG ? Dg.HP : HP);
  float* lsm = smem + (DAG ? Dg.img_off : A.pol_off);
  if (DAG) load_policy_img(lsm, LS, Dg.pol, Dg.HP, Dg.params, Dg.norm);
  const int kind = A.env.kind;  // block-uniform: the env step branches on it
  const float ahi = env_act_bound(kind);
  if (kind == IMB_ENV_SYNTH) {  // the classic-control envs have no matrices (and no env_params)
    for (int i = tid; i < (KU + 2) * IP; i += RT) esm[i] = 0.f;
    __syncthreads();
    const float* eA = env_params;
    const float* eB = eA + Do * Do;
    const float* eC = eB + Do * Da;
    const float* eW = eC + Do;
    for (int i = tid; i < Do * Do; i += RT) {
      const int r = i / Do, c = i - r * Do;  // A[r][c] -> ABt[c][r]
      esm[c * IP + r] = eA[i];
    }
    for (int i = tid; i < Do * Da; i += RT) {
      const int r = i / Da, c = i - r * Da;  // B[r][c] -> ABt[Do + c][r]
      esm[(Do + c) * IP + r] = eB[i];
    }
    for (int i = tid; i < Do; i += RT) {
      esm[KU * IP + i] = eC[i];
      esm[(KU + 1) * IP + i] = eW[i];
    }
  }
  const float* ecv = esm + KU * IP;
  const float* ewv = esm + (KU + 1) * IP;
  const int64_t E = A.E, T = A.T, H = A.env.horizon;
  const int64_t e0 = (int64_t)blockIdx.x * RR;
  const int64_t e = e0 + rt;
  const bool live = rowthread && e < E;
  // The tile's environment state is SoA [d_obs][E] in HBM: one contiguous RR-float run per feature.  Full, 16-byte
  // aligned tiles are staged by the TMA unit (one cp.async.bulk per feature row, completion on an mbarrier: SASS
  // UBLKCP); ragged tail tiles take the plain coalesced loads.
  __shared__ __align__(8) uint64_t obs_bar;
  const bool bulk_tile = (e0 + RR <= E) && ((E & 3) == 0);
  if (tid == 0) {
    mbar_init(&obs_bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (bulk_tile) {
    if (tid == 0) {
      mbar_expect_tx(&obs_bar, (uint32_t)(Do * RR * 4));
      for (int k = 0; k < Do; ++k) bulk_g2s(OBSU + k * RRS, env_obs + (int64_t)k * E + e0, (uint32_t)(RR * 4), &obs_bar);
    }
    if (rowthread)
      for (int a = 0; a < Da; ++a) OBSU[(Do + a) * RRS + tid] = 0.f;
    mbar_wait(&obs_bar, 0);
  } else if (rowthread) {
    for (int k = 0; k < Do; ++k) OBSU[k * RRS + tid] = live ? env_obs[(int64_t)k * E + e] : 0.f;  // coalesced
    for (int a = 0; a < Da; ++a) OBSU[(Do + a) * RRS + tid] = 0.f;
  }
  __syncthreads();

  const int64_t t0 = state[IMB_ST_EP_STEP];
  int64_t episode = state[IMB_ST_EPISODE];
  const int64_t gstep0 = state[IMB_ST_GLOBAL_STEP];
  // exploration: the random-action counter of step 0 and the policy vector's entry of step 0 (RolloutExplore)
  const int64_t xstep0 = MODE == RM_EXPLORE ? (Xp.step0 < 0 ? gstep0 : Xp.step0) : 0;
  const int64_t xoff = MODE == RM_EXPLORE && Xp.step0 < 0 ? gstep0 - (-1 - Xp.step0) : 0;
  const uint32_t egid = (uint32_t)(A.env.env_id_offset + e);
  const int rw = A.rw;
  const int tw = 2 * Do + Da + 1;
  const int da_store = A.pol.discrete ? 1 : Da;
  const int col_logp = Do + da_store, col_val = col_logp + 1, col_rew = col_logp + 2;
  const int64_t n_total = E * T;
  const int64_t skip = (A.ring_capacity > 0 && n_total > A.ring_capacity) ? n_total - A.ring_capacity : 0;
  const int64_t ring_idx0 = state[IMB_ST_RING_IDX];

  // value head on the latent tile H2 (thread per env)
  auto value_row = [&]() {
    float v0 = 0.f, v1 = 0.f;
    int j = 0;
    for (; j + 2 <= h; j += 2) {
      v0 = fmaf(psm[S.wv + j], H2[j * RRS + rt], v0);
      v1 = fmaf(psm[S.wv + j + 1], H2[(j + 1) * RRS + rt], v1);
    }
    if (j < h) v0 = fmaf(psm[S.wv + j], H2[j * RRS + rt], v0);
    return psm[S.bv] + (v0 + v1);
  };
  // XN <- copy of a [Do][RRS] observation tile normalised by the features of policy image img
  auto norm_obs = [&](const float* __restrict__ SRC, const float* __restrict__ img, const PolImg& SI) {
    for (int i = tid; i < Do * (RR / 4); i += RT) {
      const int k = i / (RR / 4), r4 = (i - k * (RR / 4)) * 4;
      const float4 x = ld4(SRC + k * RRS + r4);
      const float m = img[SI.mean + k], is = img[SI.istd + k];
      st4(XN + k * RRS + r4, make_float4((x.x - m) * is, (x.y - m) * is, (x.z - m) * is, (x.w - m) * is));
    }
    __syncthreads();
  };
  auto value_of_obs = [&](const float* __restrict__ SRC) {
    norm_obs(SRC, psm, S);
    tile_layer<ACT, RPL>(XN, Do, psm + S.w1v, HP, psm + S.b1v, H1, HP);
    __syncthreads();
    tile_layer<ACT, RPL>(H1, h, psm + S.w2v, HP, psm + S.b2v, H2, HP);
    __syncthreads();
    const float v = value_row();
    __syncthreads();
    return v;
  };

  bool done = false;
  for (int64_t t = 0; t < T; ++t) {
    float* row = rollout + (e * T + t) * rw;
    const bool rnd = MODE == RM_EXPLORE && Xp.policy[xoff + t] != 0;  // block-uniform: one entry per step
    // ---- policy: value tower, then pi tower (H2 ends up holding the pi latent) ------------------------------
    float value = 0.f;
    if (!rnd) {
      if (DAG) norm_obs(OBSU, psm, S);
      else value = value_of_obs(OBSU);
      tile_layer<ACT, RPL>(XN, Do, psm + S.w1p, HP, psm + S.b1p, H1, HP);
      __syncthreads();
      tile_layer<ACT, RPL>(H1, h, psm + S.w2p, HP, psm + S.b2p, H2, HP);
      __syncthreads();
    }
    // ---- action head + sampling, thread per env ----------------------------------------------------------------
    float logp = 0.f;
    if (!rowthread) {
      // (threads beyond the tile's rows only take part in the tiled layers)
    } else if (rnd) {
      // random policy: action_space.sample() (exploration_wrapper.py:58-66)
      uint32_t k0, k1;
      philox_key(Xp.seed, IMB_STREAM_EXPLORE, k0, k1);
      const uint32_t ctr = (uint32_t)(xstep0 + t);
      if (!A.pol.discrete) {
        const float lo = -ahi, hi = ahi;  // the env's Box
        Philox4 r = {0u, 0u, 0u, 0u};
        for (int a = 0; a < Da; ++a) {
          if (!noise && (a & 3) == 0) r = philox4x32(egid, ctr, (uint32_t)(a >> 2), 0u, k0, k1);
          const uint32_t w = (a & 3) == 0 ? r.x : (a & 3) == 1 ? r.y : (a & 3) == 2 ? r.z : r.w;
          const float u = noise ? (live ? noise[(t * E + e) * Da + a] : 0.f) : u01(w);
          const float act = lo + u * (hi - lo);
          if (live) row[Do + a] = act;
          OBSU[(Do + a) * RRS + tid] = fminf(fmaxf(act, lo), hi);  // (a no-op unless pinned noise leaves [0, 1])
        }
      } else {
        const float u = noise ? (live ? noise[t * E + e] : 0.f) : u01(philox4x32(egid, ctr, 0u, 0u, k0, k1).x);
        const int chosen = min((int)(u * (float)Da), Da - 1);
        for (int a = 0; a < Da; ++a) OBSU[(Do + a) * RRS + tid] = (a == chosen) ? 1.f : 0.f;
        if (live) row[Do] = (float)chosen;
      }
    } else {
      logp = action_head(psm, S, HP, h, Da, A.pol.discrete, H2, RRS, rt, OBSU + Do * RRS + tid, live ? row + Do : nullptr,
                         DAG, A.deterministic, noise, t * E + e, live, A.env.seed, IMB_STREAM_ACT_NOISE, egid,
                         (uint32_t)(gstep0 + t), ahi);
    }
    if (DAG) {
      // ---- the learner acts where the mask says so; its tower runs only when some row of the tile needs it --------
      const bool robot = live && Dg.mask[t * E + e] != 0;
      if (__syncthreads_or(robot)) {
        const int lh = Dg.pol.hidden, LHP = Dg.HP;
        norm_obs(OBSU, lsm, LS);
        tile_layer<LACT, RPL>(XN, Do, lsm + LS.w1p, LHP, lsm + LS.b1p, H1, LHP);
        __syncthreads();
        tile_layer<LACT, RPL>(H1, lh, lsm + LS.w2p, LHP, lsm + LS.b2p, H2, LHP);
        __syncthreads();
        if (robot)
          action_head(lsm, LS, LHP, lh, Da, Dg.pol.discrete, H2, RRS, rt, OBSU + Do * RRS + tid, nullptr, false, false,
                      Dg.noise, t * E + e, live, A.env.seed, IMB_STREAM_DAGGER, egid, (uint32_t)(gstep0 + t), ahi);
      }
    }
    if (live) {
      for (int k = 0; k < Do; ++k) row[k] = OBSU[k * RRS + tid];
      if (!DAG) {
        row[col_logp] = logp;
        row[col_val] = value;
      }
    }
    __syncthreads();

    // ---- environment step -------------------------------------------------------------------------------------------
    float rew_env = 0.f;
    if (kind == IMB_ENV_SYNTH) {  // NOBS = tanh([obs | u] . [A | B]^T + c)
      tile_layer<ACT_TANH, RPL>(OBSU, KU, esm, IP, ecv, NOBS, IP);
      __syncthreads();
      for (int i = 0; i < Do; ++i) rew_env = fmaf(ewv[i], NOBS[i * RRS + rt], rew_env);
      if (!A.env.discrete) {
        float pen = 0.f;
        for (int a = 0; a < Da; ++a) {
          const float uu = OBSU[(Do + a) * RRS + rt];
          pen = fmaf(uu, uu, pen);
        }
        rew_env -= 0.1f * pen;
      }
    } else {  // classic control: thread per env, float64
      if (rowthread)
        rew_env = kind == IMB_ENV_CARTPOLE ? cartpole_step(OBSU + tid, OBSU + Do * RRS + tid, NOBS + tid, RRS)
                                           : pendulum_step(OBSU + tid, OBSU + Do * RRS + tid, NOBS + tid, RRS);
      __syncthreads();
    }
    done = ((t0 + t + 1) % H) == 0;
    const float donef = done ? 1.f : 0.f;

    // ---- learned reward on (obs, clipped act, terminal-fixed next obs, done); ensemble: every member in turn ---------
    float reward = rew_env;
    if (A.reward_mode != 0) {
      for (int mi = 0; mi < n_mem; ++mi) {
        for (int p = 0; p < L.npass; ++p) {
          const PassDesc& Pd = L.pass[p];
          const float* img = smem + A.img_off + (mi * L.npass + p) * A.img_sz;
          const int din = Pd.din;
          const float* mean = img + TImg::mean(din, JP);
          const float* istd = img + TImg::istd(din, JP);
          for (int i = tid; i < din * (RR / 4); i += RT) {
            const int k = i / (RR / 4), r4 = (i - k * (RR / 4)) * 4;
            const int fr = L.stage_row[Pd.in_slot[k]];  // batch feature row -> source tile row
            float4 x;
            if (fr < Do + Da) x = ld4(OBSU + fr * RRS + r4);
            else if (fr < 2 * Do + Da) x = ld4(NOBS + (fr - Do - Da) * RRS + r4);
            else x = make_float4(donef, donef, donef, donef);
            const float m = mean[k], is = istd[k];
            st4(XN + k * RRS + r4, make_float4((x.x - m) * is, (x.y - m) * is, (x.z - m) * is, (x.w - m) * is));
          }
          __syncthreads();
          const float* HL = XN;
          int hl = din;
          if (Pd.n_hidden >= 1) {
            tile_layer<ACT_RELU, RPL>(XN, din, img + TImg::w1t(din, JP), JP, img + TImg::b1(din, JP), H1, JP);
            __syncthreads();
            HL = H1;
            hl = Pd.h1;
          }
          if (Pd.n_hidden >= 2) {
            tile_layer<ACT_RELU, RPL>(H1, Pd.h1, img + TImg::w2t(din, JP), JP, img + TImg::b2(din, JP), H2, JP);
            __syncthreads();
            HL = H2;
            hl = Pd.h2;
          }
          const float* wf = img + TImg::wf(din, JP);
          float o0 = 0.f, o1 = 0.f;
          int j = 0;
          for (; j + 2 <= hl; j += 2) {
            o0 = fmaf(wf[j], HL[j * RRS + rt], o0);
            o1 = fmaf(wf[j + 1], HL[(j + 1) * RRS + rt], o1);
          }
          if (j < hl) o0 = fmaf(wf[j], HL[j * RRS + rt], o0);
          const float o = img[TImg::bf(din, JP)] + (o0 + o1);
          const float c = pass_coef(Pd.coef_kind, L.gamma, donef);
          lg[tid] = (p == 0) ? c * o : fmaf(c, o, lg[tid]);
          __syncthreads();
        }
        if (ENS && live) Mb.raw[((int64_t)mi * T + t) * E + e] = lg[tid];  // (lg[tid] is only rewritten by this thread)
      }
      reward = (A.reward_mode == 1) ? softplus_f(lg[tid]) : lg[tid];
    }
    if (live && !ENS) row[col_rew] = reward;  // ensemble: imb_ensemble_relabel writes the combined reward

    // ---- time-limit bootstrap term gamma * V(terminal obs) (added after reward normalisation) -------------------
    float boot = 0.f;
    if (!DAG && done) boot = A.hp.gamma * value_of_obs(NOBS);  // block-uniform branch (lock-step envs)
    if (live) {
      aux[2 * E + e * T + t] = boot;
      aux[2 * E + E * T + e * T + t] = rew_env;  // ground-truth env reward (BufferingWrapper records it)
      // ---- flattened transition row (reference order) -> ring / flat_out ---------------------------------------
      const int64_t f = flat_index(e, t, E, T, t0, H);
      float* dst0 = flat_out ? flat_out + f * tw : nullptr;
      float* dst1 = nullptr;
      if (ring && f >= skip) dst1 = ring + ((ring_idx0 + (f - skip)) % A.ring_capacity) * tw;
#pragma unroll 1
      for (int q = 0; q < 2; ++q) {
        float* dst = q == 0 ? dst0 : dst1;
        if (!dst) continue;
        for (int k = 0; k < Do + Da; ++k) dst[k] = OBSU[k * RRS + tid];
        for (int k = 0; k < Do; ++k) dst[Do + Da + k] = NOBS[k * RRS + tid];
        dst[2 * Do + Da] = donef;
      }
    }
    // ---- advance: on done the next observation is the reset observation ------------------------------------------
    if (done) {
      ++episode;
      if (rowthread && kind != IMB_ENV_SYNTH)
        classic_reset(kind, A.env.seed, egid, (uint32_t)episode, OBSU + tid, RRS);
      else if (rowthread)
        for (int k = 0; k < Do; ++k)
          OBSU[k * RRS + tid] = 0.1f * philox_normal(A.env.seed, IMB_STREAM_ENV_RESET, egid, (uint32_t)episode, k);
    } else if (rowthread) {
      for (int k = 0; k < Do; ++k) OBSU[k * RRS + tid] = NOBS[k * RRS + tid];
    }
    __syncthreads();
  }
  // ---- tail: state back to HBM, V(last obs) for GAE ------------------------------------------------------
  const float vlast = DAG ? 0.f : value_of_obs(OBSU);
  if (bulk_tile) {  // state tile back to HBM through the TMA unit as well (shared -> global bulk copies)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (tid == 0) {
      for (int k = 0; k < Do; ++k)
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(env_obs + (int64_t)k * E + e0),
                     "r"(smem_u32(OBSU + k * RRS)), "r"((uint32_t)(RR * 4))
                     : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
  } else if (live) {
    for (int k = 0; k < Do; ++k) env_obs[(int64_t)k * E + e] = OBSU[k * RRS + tid];
  }
  if (live) {
    aux[e] = vlast;
    aux[E + e] = done ? 1.f : 0.f;
  }
}

__global__ void k_rollout_advance(int64_t* state, int64_t n_envs, int64_t n_steps, int horizon, int64_t ring_cap) {
  const int64_t t0 = state[IMB_ST_EP_STEP];
  state[IMB_ST_EPISODE] += (t0 + n_steps) / horizon;
  state[IMB_ST_EP_STEP] = (t0 + n_steps) % horizon;
  state[IMB_ST_GLOBAL_STEP] += n_steps;
  if (ring_cap > 0) {
    const int64_t n = n_envs * n_steps;
    const int64_t kept = n < ring_cap ? n : ring_cap;
    state[IMB_ST_RING_IDX] = (state[IMB_ST_RING_IDX] + kept) % ring_cap;
    const int64_t nd = state[IMB_ST_RING_N] + kept;
    state[IMB_ST_RING_N] = nd < ring_cap ? nd : ring_cap;
  }
}

// GAE(lambda) per env over its T rows (SB3 RolloutBuffer.compute_returns_and_advantage).
// reward += bootstrap term; episode_start[t+1] == done[t] for this lock-step env, and done[t] is
// recoverable from the bootstrap bookkeeping: done at local step t <=> (t0 + t + 1) % H == 0.
__global__ void __launch_bounds__(128) k_gae(float* __restrict__ rollout, int rw, int col_val, int64_t E,
                                             int64_t T, const float* __restrict__ aux, float gamma, float lam,
                                             const int64_t* __restrict__ state_before, int horizon) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const int col_rew = col_val + 1, col_adv = col_val + 2, col_ret = col_val + 3;
  const int64_t t0 = state_before[IMB_ST_EP_STEP];
  float last = 0.f;
  float next_v = aux[e];
  float next_nonterm = 1.0f - aux[E + e];
  for (int64_t t = T - 1; t >= 0; --t) {
    float* row = rollout + (e * T + t) * rw;
    const float r = row[col_rew] + aux[2 * E + e * T + t];
    const float v = row[col_val];
    const float delta = r + gamma * next_v * next_nonterm - v;
    last = delta + gamma * lam * next_nonterm * last;
    row[col_rew] = r;
    row[col_adv] = last;
    row[col_ret] = last + v;
    next_v = v;
    // episode_start of step t  ==  done of step t-1
    next_nonterm = (t > 0 && ((t0 + t) % horizon) == 0) ? 0.f : 1.f;
  }
}

__global__ void k_env_reset(float* __restrict__ env_obs, int64_t E, int d_obs, int kind, uint64_t seed, int64_t id_off,
                            const int64_t* __restrict__ state) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint32_t ep = (uint32_t)state[IMB_ST_EPISODE];
  if (kind != IMB_ENV_SYNTH) {
    classic_reset(kind, seed, (uint32_t)(id_off + e), ep, env_obs + e, E);
    return;
  }
  for (int k = 0; k < d_obs; ++k)
    env_obs[(int64_t)k * E + e] = 0.1f * philox_normal(seed, IMB_STREAM_ENV_RESET, (uint32_t)(id_off + e), ep, k);
}

}  // namespace

// Shared-memory layout of k_rollout for a tile of rows_of(rpl) envs and n_members reward nets (A.reward_mode, A.env and
// A.pol set) and, with Dg (Dg->pol set), the DAgger learner's image: fills A's (and Dg's) widths and offsets (floats) and
// returns the bytes; n_img_floats receives the reward-net images' share.
static size_t rollout_layout(RolloutArgs& A, const DiscLaunch& L, int n_members, int rpl, size_t* n_img_floats,
                             RolloutDagger* Dg = nullptr) {
  const int RRS = rows_of(rpl) + TILE_PAD;
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const int Do = A.env.d_obs, Da = A.env.d_act;
  A.HP = A.pol.hidden <= 32 ? 32 : 64;
  A.IP = Do <= 32 ? 32 : 64;
  A.KU = Do + Da;
  const LaunchWidths lw = A.reward_mode != 0 ? launch_widths(L) : LaunchWidths{32, Do};
  A.JP = lw.JP;
  const int dmax = lw.dmax > Do ? lw.dmax : Do;
  int wmax = A.HP > A.JP ? A.HP : A.JP;
  int o = 0;
  A.pol_off = o;
  o += al(PolImg(Do, Da, A.HP).total);
  if (Dg) {
    Dg->HP = Dg->pol.hidden <= 32 ? 32 : 64;
    wmax = wmax > Dg->HP ? wmax : Dg->HP;
    Dg->img_off = o;
    o += al(PolImg(Do, Da, Dg->HP).total);
  }
  A.env_off = o;
  o += al((A.KU + 2) * A.IP);
  A.img_off = o;
  A.img_sz = al(TImg::size(dmax, A.JP));
  const int n_img = A.reward_mode != 0 ? n_members * L.npass : 0;  // every member's images stay resident
  o += n_img * A.img_sz;
  A.obsu_off = o;
  o += al(A.KU * RRS);
  A.xn_off = o;
  o += al(dmax * RRS);
  A.h1_off = o;
  o += al(wmax * RRS);
  A.h2_off = o;
  o += al(wmax * RRS);
  A.nobs_off = o;
  o += al(A.IP * RRS);
  A.vec_off = o;
  o += al(RT);
  A.total = o;
  if (n_img_floats) *n_img_floats = (size_t)n_img * A.img_sz;
  return (size_t)o * 4;
}

// The tile (rows-per-lane parameter RPL: 0, 1, 2 or 4) k_rollout runs for A.E envs on n_sms SMs, with A laid out for it.
// Preferred: the smallest tile that still covers the SMs (the kernel's duration is one CTA's latency): <= 16 envs per
// SM -> 8 rows, <= 32 -> 32 rows, <= 128 -> 64 rows, else 128 rows.  When the preferred tile's shared memory exceeds
// IMB_SMEM_MAX, the next smaller tile that fits runs instead (more CTAs, each as fast); <0 when not even the 8-row tile
// fits.
static int rollout_plan(RolloutArgs& A, const DiscLaunch& L, int n_members, int64_t n_sms, RolloutDagger* Dg = nullptr) {
  static const int order[4] = {0, 1, 2, 4};
  int i = A.E <= n_sms * 16 ? 0 : A.E <= n_sms * 32 ? 1 : A.E <= n_sms * 128 ? 2 : 3;
  size_t n_img = 0, bytes = 0;
  for (; i >= 0; --i) {
    bytes = rollout_layout(A, L, n_members, order[i], &n_img, Dg);
    if (bytes <= IMB_SMEM_MAX) return order[i];
  }
  IMB_REQUIRE(n_members <= 1,
              "rollout of a %d-member ensemble needs %zu B of shared memory at its smallest (8-row) tile (%zu B for "
              "the member images), more than the %d B limit of a CTA: use fewer or narrower members", n_members, bytes,
              n_img * 4, (int)IMB_SMEM_MAX);
  IMB_FAIL(-1, "rollout kernel needs %zu B of shared memory at its smallest (8-row) tile (%zu B for the reward-net "
           "images%s), more than the %d B limit of a CTA", bytes, n_img * 4, Dg ? ", with the learner's image" : "",
           (int)IMB_SMEM_MAX);
}

template <int RPL, bool ENS, int ACT, int MODE, int LACT = ACT>
static int launch_rollout_t(const RolloutArgs& A, const DiscLaunch& L, const RolloutMembers& Mb,
                            const float* env_params, float* env_obs, const float* pol_params, const float* pol_norm,
                            const float* disc_params, float* rollout, float* ring, float* flat_out, float* aux,
                            const float* noise, const int64_t* state, const RolloutExplore& Xp, const RolloutDagger& Dg,
                            cudaStream_t st) {
  constexpr int RR = rows_of(RPL);
  const size_t bytes = (size_t)A.total * 4;
  static size_t attr_bytes = 0;
  if (bytes > attr_bytes) {
    cudaError_t e = cudaFuncSetAttribute(k_rollout<RPL, ENS, ACT, MODE, LACT>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_bytes = bytes;
  }
  const int blocks = (int)((A.E + RR - 1) / RR);
  k_rollout<RPL, ENS, ACT, MODE, LACT><<<blocks, RT, bytes, st>>>(A, L, Mb, env_params, env_obs, pol_params, pol_norm,
                                                                  disc_params, rollout, ring, flat_out, aux, noise,
                                                                  state, Xp, Dg);
  IMB_CHECK_LAUNCH("k_rollout");
  return 0;
}

// Mb == nullptr: the single-net rollout; act: the policy towers' activation (ACT_TANH / ACT_RELU); Xp == nullptr: every
// step on the policy (no exploration variant); Dg != nullptr: the DAgger rollout (no members, no exploration)
template <int ACT>
static int launch_rollout_act(RolloutArgs A, const DiscLaunch& L, const RolloutMembers* Mb,
                              const float* env_params, float* env_obs, const float* pol_params, const float* pol_norm,
                              const float* disc_params, float* rollout, float* ring, float* flat_out, float* aux,
                              const float* noise, const int64_t* state, const RolloutExplore* Xp,
                              const RolloutDagger* Dg_in, cudaStream_t st) {
  RolloutDagger dg = Dg_in ? *Dg_in : RolloutDagger{};
  const int rpl = rollout_plan(A, L, Mb ? Mb->M : 1, imb_num_sms(), Dg_in ? &dg : nullptr);
  if (rpl < 0) return rpl;
  static const RolloutMembers no_members = {};
  static const RolloutExplore no_explore = {};
#define IMB_RL_X(R, X, XP)                                                                                             \
  return Mb ? launch_rollout_t<R, true, ACT, X>(A, L, *Mb, env_params, env_obs, pol_params, pol_norm, disc_params,    \
                                                rollout, ring, flat_out, aux, noise, state, XP, dg, st)                \
            : launch_rollout_t<R, false, ACT, X>(A, L, no_members, env_params, env_obs, pol_params, pol_norm,          \
                                                 disc_params, rollout, ring, flat_out, aux, noise, state, XP, dg, st)
#define IMB_RL_D(R, LA)                                                                                                \
  return launch_rollout_t<R, false, ACT, RM_DAGGER, LA>(A, L, no_members, env_params, env_obs, pol_params, pol_norm,  \
                                                        nullptr, rollout, nullptr, flat_out, aux, noise, state,       \
                                                        no_explore, dg, st)
#define IMB_RL(R)                                   \
  do {                                              \
    if (Dg_in && dg.act == ACT_TANH) IMB_RL_D(R, ACT_TANH); \
    if (Dg_in) IMB_RL_D(R, ACT_RELU);               \
    if (Xp) IMB_RL_X(R, RM_EXPLORE, *Xp);           \
    IMB_RL_X(R, RM_PLAIN, no_explore);              \
  } while (0)
  if (rpl == 0) IMB_RL(0);
  if (rpl == 1) IMB_RL(1);
  if (rpl == 2) IMB_RL(2);
  IMB_RL(4);
#undef IMB_RL
#undef IMB_RL_D
#undef IMB_RL_X
}

static int launch_rollout(const RolloutArgs& A, int act, const DiscLaunch& L, const RolloutMembers* Mb,
                          const float* env_params, float* env_obs, const float* pol_params, const float* pol_norm,
                          const float* disc_params, float* rollout, float* ring, float* flat_out, float* aux,
                          const float* noise, const int64_t* state, const RolloutExplore* Xp, const RolloutDagger* Dg,
                          cudaStream_t st) {
  auto go = act == ACT_TANH ? launch_rollout_act<ACT_TANH> : launch_rollout_act<ACT_RELU>;
  return go(A, L, Mb, env_params, env_obs, pol_params, pol_norm, disc_params, rollout, ring, flat_out, aux, noise,
            state, Xp, Dg, st);
}
