// imb_rollout.cu -- C-ABI entry points of stage 1 (kernels: imb_rollout_impl.cuh).
#include "imb_rollout_impl.cuh"

static_assert(IMB_ACT_TANH == ACT_TANH && IMB_ACT_RELU == ACT_RELU, "imb.h activation codes = the kernels' ACT_*");

extern "C" int imb_rollout_row_width(const imb_policy_desc* pol) {
  return imb_row_width(pol->d_obs, pol->d_act, pol->discrete != 0);
}

// the policy and reward-net shapes k_rollout accepts
static int check_shapes(const imb_policy_desc* pol, const imb_disc_desc* disc) {
  IMB_REQUIRE(pol->hidden >= 1 && pol->hidden <= 64, "policy tower width must be <= 64");
  IMB_REQUIRE(pol->d_obs >= 1 && pol->d_act >= 1 && pol->d_obs <= IMB_MAX_DIN && pol->d_act <= IMB_MAX_DIN,
              "d_obs/d_act must be in [1, %d]", IMB_MAX_DIN);
  IMB_REQUIRE(!disc || (disc->d_obs == pol->d_obs && disc->d_act == pol->d_act), "reward net / env space mismatch");
  return 0;
}

// the env kind against the shapes it steps (include/imb.h IMB_ENV_*)
static int check_env(const imb_env_desc* env) {
  IMB_REQUIRE(env != nullptr, "no env descriptor");
  switch (env->kind) {
    case IMB_ENV_SYNTH:
      return 0;
    case IMB_ENV_CARTPOLE:
      IMB_REQUIRE(env->d_obs == 4 && env->d_act == 2 && env->discrete == 1,
                  "seals/CartPole-v0 (kind %d) takes d_obs 4, d_act 2, discrete 1; got %d, %d, %d", env->kind,
                  env->d_obs, env->d_act, env->discrete);
      return 0;
    case IMB_ENV_PENDULUM:
      IMB_REQUIRE(env->d_obs == 3 && env->d_act == 1 && env->discrete == 0,
                  "Pendulum-v1 (kind %d) takes d_obs 3, d_act 1, discrete 0; got %d, %d, %d", env->kind, env->d_obs,
                  env->d_act, env->discrete);
      return 0;
    default:
      IMB_FAIL(-1, "unknown env kind %d (IMB_ENV_SYNTH, IMB_ENV_CARTPOLE or IMB_ENV_PENDULUM)", env->kind);
  }
}

extern "C" int imb_rollout_plan(const imb_policy_desc* pol, const imb_disc_desc* disc, int32_t n_members,
                                int64_t n_envs, int32_t n_sms) {
  IMB_REQUIRE(pol && n_envs >= 1, "rollout plan needs a policy and n_envs >= 1");
  IMB_REQUIRE(n_members == 1 || (disc && n_members >= 2 && n_members <= IMB_PU_MAX_MEMBERS),
              "rollout plan: %d members (1, or 2 to %d with a reward net)", n_members, IMB_PU_MAX_MEMBERS);
  if (int rc = check_shapes(pol, disc)) return rc;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.env.d_obs = pol->d_obs;
  A.env.d_act = pol->d_act;
  A.pol = *pol;
  A.reward_mode = disc ? 1 : 0;
  A.E = n_envs;
  DiscLaunch L;
  memset(&L, 0, sizeof(L));
  if (disc)
    if (int rc = build_launch(disc, nullptr, nullptr, L)) return rc;
  const int rpl = rollout_plan(A, L, n_members, n_sms > 0 ? n_sms : imb_num_sms());
  return rpl < 0 ? rpl : rows_of(rpl);
}

// members == nullptr: imb_rollout; otherwise imb_rollout_ensemble (reward_mode 2, member m's vectors from the table)
static int rollout_common(const imb_env_desc* env, const float* env_params, float* env_obs, const imb_policy_desc* pol,
                          int pol_act, const float* pol_params, const float* pol_norm, const imb_disc_desc* disc,
                          const float* disc_params, const float* disc_norm, const imb_rollout_members* members,
                          int reward_mode, const imb_ppo_hparams* hp, int64_t n_envs, int64_t n_steps, float* rollout,
                          float* ring, int64_t ring_capacity, float* flat_out, float* aux, const float* noise, int flags,
                          const int64_t* state, const RolloutExplore* Xp, const RolloutDagger* Dg, void* stream) {
  IMB_REQUIRE(n_envs >= 1 && n_steps >= 1, "rollout needs n_envs, n_steps >= 1");
  if (int rc = check_env(env)) return rc;
  IMB_REQUIRE(env->d_obs == pol->d_obs && env->d_act == pol->d_act && env->discrete == pol->discrete,
              "env / policy space mismatch");
  IMB_REQUIRE(pol_act == IMB_ACT_TANH || pol_act == IMB_ACT_RELU,
              "pol_act must be IMB_ACT_TANH (0) or IMB_ACT_RELU (1), got %d", pol_act);
  if (int rc = check_shapes(pol, reward_mode != 0 ? disc : nullptr)) return rc;
  RolloutArgs A;
  A.env = *env;
  A.pol = *pol;
  A.hp = *hp;
  A.reward_mode = reward_mode;
  A.deterministic = (flags & IMB_RF_DETERMINISTIC) ? 1 : 0;
  A.E = n_envs;
  A.T = n_steps;
  A.rw = imb_rollout_row_width(pol);
  A.ring_capacity = ring ? ring_capacity : 0;
  DiscLaunch L;
  memset(&L, 0, sizeof(L));
  if (reward_mode != 0) {
    IMB_REQUIRE(disc && (disc_params || members), "reward_mode != 0 needs a reward net");
    imb_disc_desc dd = *disc;
    dd.subtract_logp = 0;  // reward_train.predict_processed never subtracts log pi (airl.py:121-124)
    if (int rc = build_launch(&dd, members ? members->norm_state[0] : disc_norm, nullptr, L)) return rc;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (!members)
    return launch_rollout(A, pol_act, L, nullptr, env_params, env_obs, pol_params, pol_norm, disc_params, rollout, ring,
                          flat_out, aux, noise, state, Xp, Dg, st);
  const int M = members->n_members;
  IMB_REQUIRE(M >= 2 && M <= IMB_PU_MAX_MEMBERS, "imb_rollout_ensemble: %d members (2 to %d)", M, IMB_PU_MAX_MEMBERS);
  IMB_REQUIRE(members->raw != nullptr, "imb_rollout_ensemble: no raw-output buffer");
  const bool in_norm = disc->base.has_norm || (disc->shaped && disc->potential.has_norm);
  RolloutMembers Mb;
  memset(&Mb, 0, sizeof(Mb));
  Mb.M = M;
  Mb.raw = members->raw;
  for (int m = 0; m < M; ++m) {
    IMB_REQUIRE(members->params[m] != nullptr, "imb_rollout_ensemble: member %d has no parameters", m);
    IMB_REQUIRE(!in_norm || members->norm_state[m] != nullptr, "imb_rollout_ensemble: member %d has no input norm", m);
    Mb.params[m] = members->params[m];
    for (int p = 0; p < L.npass; ++p) {
      const imb_mlp& mlp = p == 0 ? disc->base : disc->potential;
      Mb.norm[m][p] = mlp.has_norm ? members->norm_state[m] + mlp.norm_off : nullptr;
    }
  }
  return launch_rollout(A, pol_act, L, &Mb, env_params, env_obs, pol_params, pol_norm, nullptr, rollout, ring, flat_out,
                        aux, noise, state, Xp, Dg, st);
}

extern "C" int imb_rollout(const imb_env_desc* env, const float* env_params, float* env_obs,
                           const imb_policy_desc* pol, int32_t pol_act, const float* pol_params, const float* pol_norm,
                           const imb_disc_desc* disc, const float* disc_params, const float* disc_norm,
                           int reward_mode, const imb_ppo_hparams* hp, int64_t n_envs, int64_t n_steps,
                           float* rollout, float* ring, int64_t ring_capacity, float* flat_out, float* aux,
                           const float* noise, int flags, const int64_t* state, void* stream) {
  return rollout_common(env, env_params, env_obs, pol, pol_act, pol_params, pol_norm, disc, disc_params, disc_norm,
                        nullptr, reward_mode, hp, n_envs, n_steps, rollout, ring, ring_capacity, flat_out, aux, noise,
                        flags, state, nullptr, nullptr, stream);
}

extern "C" int imb_rollout_ensemble(const imb_env_desc* env, const float* env_params, float* env_obs,
                                    const imb_policy_desc* pol, int32_t pol_act, const float* pol_params,
                                    const float* pol_norm, const imb_disc_desc* disc, const imb_rollout_members* members,
                                    const imb_ppo_hparams* hp, int64_t n_envs, int64_t n_steps, float* rollout,
                                    float* ring, int64_t ring_capacity, float* flat_out, float* aux, const float* noise,
                                    int flags, const int64_t* state, void* stream) {
  IMB_REQUIRE(disc && members, "imb_rollout_ensemble needs a member architecture and a member table");
  return rollout_common(env, env_params, env_obs, pol, pol_act, pol_params, pol_norm, disc, nullptr, nullptr, members, 2,
                        hp, n_envs, n_steps, rollout, ring, ring_capacity, flat_out, aux, noise, flags, state, nullptr,
                        nullptr, stream);
}

extern "C" int imb_rollout_explore(const imb_env_desc* env, const float* env_params, float* env_obs,
                                   const imb_policy_desc* pol, int32_t pol_act, const float* pol_params,
                                   const float* pol_norm, const imb_disc_desc* disc, const float* disc_params,
                                   const float* disc_norm, const imb_rollout_members* members, int reward_mode,
                                   const imb_ppo_hparams* hp, int64_t n_envs, int64_t n_steps, float* rollout,
                                   float* flat_out, float* aux, const float* noise, int flags,
                                   const uint8_t* explore_policy, uint64_t explore_seed, int64_t explore_step0,
                                   const int64_t* state, void* stream) {
  IMB_REQUIRE(explore_policy != nullptr, "imb_rollout_explore needs the per-step policy vector");
  IMB_REQUIRE(!members || (disc && reward_mode == 2 && !disc_params && !disc_norm),
              "imb_rollout_explore: a member table goes with reward_mode 2, the member architecture and no single net");
  RolloutExplore Xp;
  Xp.policy = explore_policy;
  Xp.seed = explore_seed;
  Xp.step0 = explore_step0;
  return rollout_common(env, env_params, env_obs, pol, pol_act, pol_params, pol_norm, disc, disc_params, disc_norm,
                        members, reward_mode, hp, n_envs, n_steps, rollout, nullptr, 0, flat_out, aux, noise, flags,
                        state, &Xp, nullptr, stream);
}

// the learner of a DAgger rollout against the expert it stands in for
static int check_learner(const imb_policy_desc* expert, const imb_policy_desc* learner, int learner_act) {
  IMB_REQUIRE(expert && learner, "the DAgger rollout needs an expert and a learner policy");
  IMB_REQUIRE(learner->d_obs == expert->d_obs && learner->d_act == expert->d_act &&
                  learner->discrete == expert->discrete,
              "expert / learner space mismatch");
  IMB_REQUIRE(learner_act == IMB_ACT_TANH || learner_act == IMB_ACT_RELU,
              "learner_act must be IMB_ACT_TANH (0) or IMB_ACT_RELU (1), got %d", learner_act);
  return check_shapes(learner, nullptr);
}

extern "C" int imb_rollout_dagger_plan(const imb_policy_desc* expert, const imb_policy_desc* learner, int64_t n_envs,
                                       int32_t n_sms) {
  IMB_REQUIRE(n_envs >= 1, "rollout plan needs n_envs >= 1");
  if (int rc = check_learner(expert, learner, IMB_ACT_TANH)) return rc;
  if (int rc = check_shapes(expert, nullptr)) return rc;
  RolloutArgs A;
  memset(&A, 0, sizeof(A));
  A.env.d_obs = expert->d_obs;
  A.env.d_act = expert->d_act;
  A.pol = *expert;
  A.E = n_envs;
  DiscLaunch L;
  memset(&L, 0, sizeof(L));
  RolloutDagger Dg;
  memset(&Dg, 0, sizeof(Dg));
  Dg.pol = *learner;
  const int rpl = rollout_plan(A, L, 1, n_sms > 0 ? n_sms : imb_num_sms(), &Dg);
  return rpl < 0 ? rpl : rows_of(rpl);
}

extern "C" int imb_rollout_dagger(const imb_env_desc* env, const float* env_params, float* env_obs,
                                  const imb_policy_desc* expert, int32_t expert_act, const float* expert_params,
                                  const float* expert_norm, const imb_policy_desc* learner, int32_t learner_act,
                                  const float* learner_params, const float* learner_norm, int64_t n_envs,
                                  int64_t n_steps, float* rollout, float* flat_out, float* aux, const float* noise,
                                  const float* robot_noise, int flags, const uint8_t* robot_mask,
                                  const int64_t* state, void* stream) {
  IMB_REQUIRE(robot_mask != nullptr, "imb_rollout_dagger needs the [n_steps][n_envs] robot mask");
  if (int rc = check_learner(expert, learner, learner_act)) return rc;
  RolloutDagger Dg;
  memset(&Dg, 0, sizeof(Dg));
  Dg.pol = *learner;
  Dg.act = learner_act;
  Dg.params = learner_params;
  Dg.norm = learner_norm;
  Dg.noise = robot_noise;
  Dg.mask = robot_mask;
  imb_ppo_hparams hp;
  memset(&hp, 0, sizeof(hp));
  return rollout_common(env, env_params, env_obs, expert, expert_act, expert_params, expert_norm, nullptr, nullptr,
                        nullptr, nullptr, 0, &hp, n_envs, n_steps, rollout, nullptr, 0, flat_out, aux, noise, flags,
                        state, nullptr, &Dg, stream);
}

extern "C" int imb_rollout_advance(int64_t* state, int64_t n_envs, int64_t n_steps, int32_t horizon,
                                   int64_t ring_capacity, void* stream) {
  k_rollout_advance<<<1, 1, 0, (cudaStream_t)stream>>>(state, n_envs, n_steps, horizon, ring_capacity);
  IMB_CHECK_LAUNCH("k_rollout_advance");
  return 0;
}

extern "C" int imb_gae(float* rollout, int32_t rw, int32_t col_value, int64_t n_envs, int64_t n_steps,
                       const float* aux, float gamma, float gae_lambda, const int64_t* state_before,
                       int32_t horizon, void* stream) {
  k_gae<<<(int)((n_envs + 127) / 128), 128, 0, (cudaStream_t)stream>>>(rollout, rw, col_value, n_envs, n_steps, aux,
                                                                      gamma, gae_lambda, state_before, horizon);
  IMB_CHECK_LAUNCH("k_gae");
  return 0;
}

extern "C" int imb_env_reset(float* env_obs, int64_t n_envs, const imb_env_desc* env, const int64_t* state,
                             void* stream) {
  if (int rc = check_env(env)) return rc;
  k_env_reset<<<(int)((n_envs + 127) / 128), 128, 0, (cudaStream_t)stream>>>(env_obs, n_envs, env->d_obs, env->kind,
                                                                            env->seed, env->env_id_offset, state);
  IMB_CHECK_LAUNCH("k_env_reset");
  return 0;
}
