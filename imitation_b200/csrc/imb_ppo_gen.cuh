// imb_ppo_gen.cuh -- k_ppo_update_gen: PPO.train for the shapes outside k_ppo_update's envelope
// (included by imb_ppo.cu inside its anonymous namespace; shares PpoArgs / PLay / the Adam arithmetic).
//
// k_ppo_update is built around ONE 64-row minibatch resident in shared memory and one lane per hidden unit.  The
// reference's tuned configurations also use minibatches of 128 and 512 rows (scripts/config/tuned_hps/
// airl_seals_walker / airl_seals_hopper: rl.rl_kwargs.batch_size) and scripts/ingredients/rl.py:122-194 accepts any
// policy_kwargs, e.g. SB3's MlpPolicy default net_arch 64x64.  This kernel covers those: tower width <= 64 (U = 1 or 2
// hidden units per lane), minibatch <= GEN_MAX_MB rows.  Same cluster of CL CTAs and the same parameter layout, but
//   * a minibatch is processed in passes of CL x RG = 128 rows (CTA c owns rows 16c..16c+15 of every pass); the rows are
//     read from the (L2-resident) rollout table through the step's index list, never staged as a whole;
//   * minibatch statistics (feature RunningNorm update, advantage normalisation) are computed redundantly and
//     identically by every CTA, one warp per column, before the first pass;
//   * partial gradients accumulate in the CTA's own gradient vector over the passes; the slice owners then read the CL
//     partials straight out of their peers' shared memory (DSMEM loads) between two cluster barriers, exchange the
//     squared slice norms, run clip_grad_norm_ + Adam on their slice and store the new parameters into every CTA.
// Three cluster barriers per optimiser step instead of the mbarrier-signalled exchange of k_ppo_update: simpler, and
// the barriers' cost is small against steps that carry 2-32x the arithmetic.
// ACT is the towers' activation: every ReLU policy runs here whatever its shape (k_ppo_update is tanh only).
// LK is the loss of the step: LOSS_PPO (PPO.train) or LOSS_BC (behavioural cloning, algorithms/bc.py:94-156 and
// :481-510).  A BC step is this kernel's step with
//   * the minibatch drawn from the host's per-epoch permutations in full minibatches (DataLoader drop_last=True), the
//     launch running minibatches [j0, j0 + n) of one train() call (BcArgs);
//   * only the obs | act columns of the rows read, d loss / d logp = -1 / batch_size per row, the entropy term with
//     ent_weight / batch_size, no ratio, clipping or advantage, and no value tower (no forward, backward or value loss);
//   * the feature RunningNorm updated per minibatch only when the policy is in training mode (norm_update);
//   * the reduced gradient accumulated over batch_size / minibatch_size minibatches (the gradient of an unfinished
//     batch is carried between launches in BcArgs::carry); the optimiser step adds l2_weight * w to every gradient, then
//     runs Adam without clip_grad_norm_ (no squared-norm exchange); the last, incomplete batch of a train() also steps;
//   * the BCTrainingMetrics of every logged batch's last minibatch written to BcArgs::metrics.
// A DQN step (LOSS_DQN: SB3 2.2 DQN.train, restated by oracle/sqil_port.py) is this kernel's step with
//   * minibatch gs made of table rows [gs * mb, (gs + 1) * mb) (no permutation), each row obs | act (index) | y, y the TD
//     target r + (1 - done) gamma max_a Q_target(s') that imb_dqn_target wrote before the launch;
//   * the Q values = the pi tower + action head's outputs, dL/dQ_a = clamp(Q_a - y, -1, 1) / mb on the taken action and
//     0 elsewhere (F.smooth_l1_loss, beta 1, mean); no value tower, entropy or ratio;
//   * clip_grad_norm_ and Adam as PPO's, with the Adam bias corrections from the step count (as BC's), so that steps
//     split over launches compute the same bits; loss_log[(k - 1 - B.j0) * 4] = the loss (the mean smooth L1) of the
//     step that makes the Adam step count k: the row is read from the device, so that a captured launch replays exactly;
//   * of the state words only ST_PPO_STEP advances (no epoch count), so a split leaves the state a single launch leaves.
constexpr int LOSS_PPO = 0, LOSS_BC = 1, LOSS_DQN = 2;
struct BcArgs {
  int64_t j0, n_mb;    // minibatches [j0, j0 + n_mb) of the train() call's sequence (numbered from 0 in every train())
  int k;               // minibatches per optimiser batch: batch_size / minibatch_size
  int final_flush;     // minibatch j0 + n_mb - 1 ends the train(): 1 = an incomplete batch there takes its optimiser
                       // step; 2 = that step is left to a later flush-only launch (n_mb = 0, final_flush = 1), this
                       // launch only writes the batch's metrics (the reference steps after the last on_epoch_end)
  int norm_update;     // policy.training: the feature RunningNorm is updated by every minibatch
  int log_interval;    // batches whose number is a multiple of it write their metrics
  float l2_weight;
  float inv_bs;        // 1 / batch_size
  float* carry;        // [n_params] (flat order) summed gradient of the batch the launch starts / ends inside
  float* metrics;      // [n_logged][8]: BC_M_* of each logged batch, in order
};
enum { BC_M_NEGLOGP, BC_M_ENTROPY, BC_M_ENT_LOSS, BC_M_PROB_TRUE_ACT, BC_M_L2_NORM, BC_M_L2_LOSS, BC_M_LOSS, BC_M_BATCH };
constexpr int RG = 16;             // minibatch rows per CTA and pass
constexpr int GEN_MAX_MB = 4096;   // index list of one minibatch in shared memory

struct GenLayout {
  int Pm, GP, Ms, Vs, Gs, IDX, CSM, CSI, rstat, XN, TH1, TLAT, TDZ2, TDZ1, MEAN, DM, DLS, ACT, DVAL, ADV, LPO, RET, total;
};
__host__ __device__ inline GenLayout gen_layout(int S, int HP, int KP, int Da, int mb) {
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const int DAP = (Da + 3) / 4 * 4;
  GenLayout g;
  int o = 0;
  g.Pm = o; o += al(CL * S);       // parameters, P-layout, padded to CL slices
  g.GP = o; o += al(CL * S);       // this CTA's partial gradient (all parameters), accumulated over the passes
  g.Ms = o; o += al(S);            // Adam moments of the OWNED slice
  g.Vs = o; o += al(S);
  g.Gs = o; o += al(S);            // summed gradient of the owned slice
  g.IDX = o; o += al(mb);          // rollout row of every minibatch row (int)
  g.CSM = o; o += 96;              // per-column shift (features 0..Do-1, [Do] = advantage)
  g.CSI = o; o += 96;              // per-column scale
  g.rstat = o; o += al(2 * 64 + 4);
  g.XN = o; o += KP * RG;          // normalised observations of the pass, feature-major [k][RG]
  g.TH1 = o; o += 2 * HP * RG;     // [tower][unit][RG]
  g.TLAT = o; o += 2 * HP * RG;
  g.TDZ2 = o; o += 2 * HP * RG;
  g.TDZ1 = o; o += 2 * HP * RG;
  g.MEAN = o; o += DAP * RG;       // action means / logits [a][RG]
  g.DM = o; o += DAP * RG;         // dL/d(mean|logits)
  g.DLS = o; o += DAP * RG;        // dL/d(log_std) per row
  g.ACT = o; o += DAP * RG;        // actions of the pass ([0][RG] = index for Discrete)
  g.DVAL = o; o += RG;
  g.ADV = o; o += RG;
  g.LPO = o; o += RG;
  g.RET = o; o += RG;
  g.total = al(o);
  return g;
}

__device__ __forceinline__ float dot16r(const float (&d)[16], const float* __restrict__ b) {
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = ld4(b + 4 * q);
    s0 = fmaf(d[4 * q], v.x, s0);
    s1 = fmaf(d[4 * q + 1], v.y, s1);
    s0 = fmaf(d[4 * q + 2], v.z, s0);
    s1 = fmaf(d[4 * q + 3], v.w, s1);
  }
  return s0 + s1;
}
__device__ __forceinline__ void load16(float (&d)[16], const float* __restrict__ p) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = ld4(p + 4 * q);
    d[4 * q] = v.x, d[4 * q + 1] = v.y, d[4 * q + 2] = v.z, d[4 * q + 3] = v.w;
  }
}
__device__ __forceinline__ float sum16(const float (&d)[16]) {
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    s0 += d[2 * q];
    s1 += d[2 * q + 1];
  }
  return s0 + s1;
}

// Activation of the policy towers (ACT_TANH / ACT_RELU) and its backward through the post-activation a: tanh's
// g (1 - a^2); ReLU's g where a > 0, else 0 (torch's threshold_backward: the derivative at exactly 0 is 0).
template <int ACT>
__device__ __forceinline__ float ppo_act(float z) {
  return ACT == ACT_TANH ? PPO_TANH(z) : fmaxf(z, 0.f);
}
template <int ACT>
__device__ __forceinline__ float ppo_act_grad(float g, float a) {
  return ACT == ACT_TANH ? g * (1.0f - a * a) : (a > 0.f ? g : 0.f);
}

// PACT: the towers' activation (ACT names the shared-memory action tile below); LK: the loss, LOSS_PPO, LOSS_BC or
// LOSS_DQN (`rollout` = the TD rows, perm_in unused, A.n_rows = steps x mb).  Under LOSS_BC
// `rollout` is the demonstration table, perm_in holds the permutations of the epochs from (j0 / (N / mb)) on, [epoch][N],
// A.hp.ent_coef is ent_weight, and loss_log is unused.
template <int U, int PACT, int LK = LOSS_PPO>
__global__ void __launch_bounds__(PT, 1) k_ppo_update_gen(const PpoArgs A, float* __restrict__ g_params,
                                                          float* __restrict__ g_norm, int32_t* __restrict__ g_norm_count,
                                                          float* __restrict__ g_m, float* __restrict__ g_v,
                                                          const float* __restrict__ rollout,
                                                          const int64_t* __restrict__ perm_in,
                                                          float* __restrict__ loss_log, int64_t* __restrict__ state,
                                                          const BcArgs B) {
  constexpr bool BC = LK == LOSS_BC;
  constexpr bool DQN = LK == LOSS_DQN;
  constexpr bool NOV = BC || DQN;  // no value tower
  constexpr int HP = 32 * U;
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int crank = (int)cluster.block_rank();
  extern __shared__ __align__(128) float smem[];
  __shared__ float red[32];
  __shared__ float bc[2];
  __shared__ float SSQ[CL];   // squared gradient norms of the CL slices (each written by its owner into every CTA)
  __shared__ float LOSS[32];  // [CL][3] partial loss sums (read by CTA 0)
  // training statistics (ppo_stats_fold): per-row slots of the step (summed over its passes), accumulators, the CTAs'
  // KL shares of the step (target_kl; written beside SSQ), explained-variance partials
  __shared__ float RSL[RS_N * RG];
  __shared__ float ACC[AC_N];
  __shared__ float KLS[CL];
  __shared__ double EVP[4];
  __shared__ double EVW[PT / 32];
  const imb_policy_desc& pd = A.pol;
  const int Do = pd.d_obs, Da = pd.d_act, h = pd.hidden, NP = pd.n_params, S = A.S;
  const PLay PL = make_play(pd);
  const int ldo = PL.ldo, ldh = PL.ldh;
  const int da_store = pd.discrete ? 1 : Da;
  const int col_logp = Do + da_store, col_adv = col_logp + 3, col_ret = col_logp + 4;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rw = A.rw;
  const int mb = A.hp.batch_size;
  const bool kl_on = A.target_kl > 0.f, rec = kl_on || A.stats != nullptr;  // (uniform)
  const GenLayout G = gen_layout(S, HP, A.KP, Da, mb);
  float* Pm = smem + G.Pm;
  float* GP = smem + G.GP;
  float* Ms = smem + G.Ms;
  float* Vs = smem + G.Vs;
  float* Gs = smem + G.Gs;
  int* IDX = reinterpret_cast<int*>(smem + G.IDX);
  float* CSM = smem + G.CSM;
  float* CSI = smem + G.CSI;
  float* rstat = smem + G.rstat;
  float* XN = smem + G.XN;
  float* TH1 = smem + G.TH1;
  float* TLAT = smem + G.TLAT;
  float* TDZ2 = smem + G.TDZ2;
  float* TDZ1 = smem + G.TDZ1;
  float* MEAN = smem + G.MEAN;
  float* DM = smem + G.DM;
  float* DLS = smem + G.DLS;
  float* ACT = smem + G.ACT;
  float* DVAL = smem + G.DVAL;
  float* ADV = smem + G.ADV;
  float* LPO = smem + G.LPO;
  float* RET = smem + G.RET;

  for (int i = tid; i < G.total; i += PT) smem[i] = 0.f;
  if (tid < 32) LOSS[tid] = 0.f;
  if (tid < CL) SSQ[tid] = 0.f;
  if (tid < AC_N) ACC[tid] = 0.f;
  __syncthreads();
  if (tid < 64) {
    rstat[tid] = (pd.has_norm && tid < Do) ? g_norm[tid] : 0.f;
    rstat[64 + tid] = (pd.has_norm && tid < Do) ? g_norm[Do + tid] : 1.f;
  }
  for (int p = tid; p < NP; p += PT) {
    const int q = flat_to_play(pd, PL, p);
    Pm[q] = g_params[p];
    if (q / S == crank) {
      Ms[q - crank * S] = g_m[p];
      Vs[q - crank * S] = g_v[p];
      if (BC && B.j0 % B.k != 0) Gs[q - crank * S] = B.carry[p];  // the batch began in the previous launch
    }
  }
  int32_t run_count = pd.has_norm ? *g_norm_count : 0;

  const int64_t N = A.n_rows;
  const int Ni = (int)N;
  const int64_t steps_per_epoch = BC ? N / mb : (N + mb - 1) / mb;
  const bool flush_only = BC && B.n_mb == 0;  // BC: only the optimiser step of the carried incomplete batch
  const int64_t n_steps = BC ? (flush_only ? 1 : B.n_mb) : steps_per_epoch * A.hp.n_epochs;
  int64_t adam_step = state[IMB_ST_PPO_STEP];
  const int64_t perm_draw0 = state[IMB_ST_PPO_EPOCH];
  double b1pow = pow(0.9, (double)adam_step), b2pow = pow(0.999, (double)adam_step);
  if (A.stats) ppo_ev_partial(rollout, N, rw, col_logp + 1, col_ret, crank, EVP, EVW);
  cluster.sync();  // every CTA's shared memory is initialised before any peer touches it

  int ep_now = 0, start = 0;
  int64_t kstop = 0;  // target_kl: the stopping step + 1
  int n_logged = 0;   // BC: metrics rows written
  if (BC) start = (int)(B.j0 % steps_per_epoch) * mb;
  for (int64_t gs = 0; gs < n_steps; ++gs) {
    const int nb = min(mb, Ni - start);
    const float inv_nb = 1.0f / (float)nb;
    // BC: minibatch i of the train() call ends a batch when (i + 1) * mb is a multiple of batch_size (bc.py:505) or,
    // incomplete, when it is the call's last (bc.py:507-510); that batch is number i / k, or i / k + 1 when incomplete
    bool bc_step = true, bc_log = false;
    float l2c = 0.f;  // BC: l2_weight x (the batch's minibatches so far) x mb / batch_size
    int64_t batch_num = 0;
    if (BC) {
      const int64_t i = B.j0 + gs - (flush_only ? 1 : 0);
      const bool full = (i + 1) % B.k == 0, last = B.final_flush != 0 && gs == n_steps - 1;
      bc_step = full || (last && B.final_flush == 1);
      batch_num = i / B.k + (full ? 0 : 1);
      bc_log = (bc_step || last) && !flush_only && B.metrics != nullptr && batch_num % B.log_interval == 0;
      l2c = B.l2_weight * ((float)(i % B.k + 1) / (float)B.k);
      if (bc_step) ++adam_step;
    } else {
      ++adam_step;
    }
    // ---- 0. the step's rollout rows, a clean gradient vector, Adam bias corrections ------------------------------
    for (int r = tid; r < (flush_only ? 0 : nb); r += PT) {
      int64_t idx;
      if constexpr (DQN) {
        idx = start + r;
      } else {
        if (perm_in) {
          idx = perm_in[(int64_t)ep_now * N + start + r];
        } else {
          const FeistelKey fk = feistel_key(A.seed, IMB_STREAM_PPO_PERM, (uint64_t)(perm_draw0 + ep_now), (uint64_t)N);
          idx = (int64_t)feistel_perm(fk, (uint64_t)(start + r), (uint64_t)N);
        }
      }
      IDX[r] = (int)idx;
    }
    for (int i = tid; i < CL * S; i += PT) GP[i] = 0.f;
    if (rec && tid < RS_N * RG) RSL[tid] = 0.f;
    if (tid == PT - 1) {
      if (NOV) {  // from the step count alone, so that a train() split over launches computes the same bits
        b1pow = pow(0.9, (double)adam_step);
        b2pow = pow(0.999, (double)adam_step);
      } else {
        b1pow *= 0.9;
        b2pow *= 0.999;
      }
      bc[0] = (float)((double)A.hp.lr / (1.0 - b1pow));
      bc[1] = (float)sqrt(1.0 - b2pow);
    }
    __syncthreads();
    // ---- 1. minibatch statistics, one warp per column (features: RunningNorm.update_stats + the normalisation the
    //         forward pass applies with the UPDATED statistics; last column: advantage normalisation) -----------------
    for (int c = warp; c <= Do; c += PT / 32) {
      const bool is_feat = c < Do;
      const bool need = is_feat ? (pd.has_norm != 0 && !flush_only) : (!BC && A.hp.normalize_advantage && nb > 1);
      float mean = 0.f, istd = 1.f;
      if (BC && need && !B.norm_update) {  // evaluation mode: normalise with the statistics as they stand
        mean = rstat[c];
        istd = rsqrtf(rstat[64 + c] + pd.norm_eps);
      } else if (need) {  // (warp-uniform)
        const int col = is_feat ? c : col_adv;
        float s = 0.f;
        for (int r = lane; r < nb; r += 32) s += rollout[(int64_t)IDX[r] * rw + col];
        const float bmean = warp_sum(s) * inv_nb;
        float q = 0.f;
        for (int r = lane; r < nb; r += 32) {
          const float d = rollout[(int64_t)IDX[r] * rw + col] - bmean;
          q = fmaf(d, d, q);
        }
        const float ssd = warp_sum(q);
        if (is_feat) {
          mean = rstat[c];
          float var = rstat[64 + c];
          const float bvar = ssd * inv_nb;
          const float bn = (float)nb, cn = (float)run_count, itot = rcp_fast(cn + bn), delta = bmean - mean;
          mean += delta * bn * itot;
          var *= cn;
          var += bvar * bn;
          var += delta * delta * cn * bn * itot;
          var *= itot;
          istd = rsqrtf(var + pd.norm_eps);
          __syncwarp();  // every lane has read the old statistics
          if (lane == 0) {
            rstat[c] = mean;
            rstat[64 + c] = var;
          }
        } else {
          mean = bmean;
          istd = rcp_fast(sqrt_fast(ssd / (float)(nb - 1)) + 1e-8f);
        }
      }
      if (lane == 0) {
        CSM[c] = mean;
        CSI[c] = istd;
      }
    }
    if (pd.has_norm && (!BC || (B.norm_update && !flush_only))) run_count += nb;
    __syncthreads();

    // ---- 2. passes of CL x RG rows: stage own rows -> warp-autonomous forward / loss / backward -> weight gradients ----
    float l_pg = 0.f, l_v = 0.f, l_ent = 0.f;
    const int npass = flush_only ? 0 : (nb + CL * RG - 1) / (CL * RG);
    for (int pass = 0; pass < npass; ++pass) {
      const int base = pass * (CL * RG) + crank * RG;  // first minibatch row of this CTA in this pass
      const int rws = BC ? col_logp : DQN ? col_logp + 1 : rw;  // BC reads obs | act, DQN obs | act | y
      for (int e = tid; e < RG * rws; e += PT) {
        const int i = e / rws, c = e - i * rws, r = base + i;
        const bool rl = r < nb;
        const float v = rl ? rollout[(int64_t)IDX[rl ? r : 0] * rw + c] : 0.f;
        if (c < Do) {
          XN[c * RG + i] = rl ? (v - CSM[c]) * CSI[c] : 0.f;
        } else if (c < col_logp) {
          ACT[(c - Do) * RG + i] = v;
        } else if (c == col_logp) {
          LPO[i] = v;
        } else if (c == col_adv) {
          ADV[i] = rl ? (v - CSM[Do]) * CSI[Do] : 0.f;
        } else if (c == col_ret) {
          RET[i] = v;
        }
      }
      __syncthreads();
      if (!NOV || warp < 4) {  // (BC and DQN have no value tower)
        // warp = (tower, 4 own rows), lane = hidden unit(s) lane + 32 u; only __syncwarp() between the layers
        const int cnet = warp >> 2, r0 = 4 * (warp & 3);
        const int rr = lane >> 3, la = lane & 7;  // per-row parts: lane octet rr handles row r0 + rr
        const int lrow = r0 + rr;
        const bool live = base + lrow < nb;
        float* cH1 = TH1 + cnet * HP * RG;
        float* cLAT = TLAT + cnet * HP * RG;
        float* cDZ2 = TDZ2 + cnet * HP * RG;
        float* cDZ1 = TDZ1 + cnet * HP * RG;
        const float* cW1 = Pm + (cnet ? PL.w1[1] : PL.w1[0]);
        const float* cW2 = Pm + (cnet ? PL.w2[1] : PL.w2[0]);
        const int c_b1 = cnet ? PL.b1[1] : PL.b1[0], c_b2 = cnet ? PL.b2[1] : PL.b2[0];
        int jc[U];
        bool jl[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          jl[u] = lane + 32 * u < h;
          jc[u] = jl[u] ? lane + 32 * u : 0;
        }
        float acc[U][4], h1[U][4], lat[U][4], dl[U][4];
        // layer 1
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
#pragma unroll 4
        for (int k = 0; k < Do; ++k) {
          const float4 x = ld4(XN + k * RG + r0);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const float w = cW1[jc[u] * ldo + k];
            acc[u][0] = fmaf(x.x, w, acc[u][0]);
            acc[u][1] = fmaf(x.y, w, acc[u][1]);
            acc[u][2] = fmaf(x.z, w, acc[u][2]);
            acc[u][3] = fmaf(x.w, w, acc[u][3]);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float b = Pm[c_b1 + jc[u]];
#pragma unroll
          for (int r = 0; r < 4; ++r) h1[u][r] = jl[u] ? ppo_act<PACT>(acc[u][r] + b) : 0.f;
          st4(cH1 + (lane + 32 * u) * RG + r0, make_float4(h1[u][0], h1[u][1], h1[u][2], h1[u][3]));
        }
        __syncwarp();
        // layer 2
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
#pragma unroll 4
        for (int i = 0; i < h; ++i) {
          const float4 x = ld4(cH1 + i * RG + r0);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const float w = cW2[jc[u] * ldh + i];
            acc[u][0] = fmaf(x.x, w, acc[u][0]);
            acc[u][1] = fmaf(x.y, w, acc[u][1]);
            acc[u][2] = fmaf(x.z, w, acc[u][2]);
            acc[u][3] = fmaf(x.w, w, acc[u][3]);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const float b = Pm[c_b2 + jc[u]];
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            lat[u][r] = jl[u] ? ppo_act<PACT>(acc[u][r] + b) : 0.f;
            dl[u][r] = 0.f;
          }
          st4(cLAT + (lane + 32 * u) * RG + r0, make_float4(lat[u][0], lat[u][1], lat[u][2], lat[u][3]));
        }
        auto oct_sum = [&](float v) {
          v += __shfl_xor_sync(0xffffffffu, v, 4);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          return v;
        };
        if (cnet == 1) {
          // value head: four sums over the units, transposed on the way so that octet rr ends with row r0 + rr's
          float wvj[U];
          float p0 = 0.f, p1 = 0.f, p2 = 0.f, p3 = 0.f;
#pragma unroll
          for (int u = 0; u < U; ++u) {
            wvj[u] = jl[u] ? Pm[PL.wv + jc[u]] : 0.f;
            p0 = fmaf(lat[u][0], wvj[u], p0);
            p1 = fmaf(lat[u][1], wvj[u], p1);
            p2 = fmaf(lat[u][2], wvj[u], p2);
            p3 = fmaf(lat[u][3], wvj[u], p3);
          }
          const bool up16 = (lane & 16) != 0, up8 = (lane & 8) != 0;
          float k0 = up16 ? p2 : p0, k1 = up16 ? p3 : p1;
          k0 += __shfl_xor_sync(0xffffffffu, up16 ? p0 : p2, 16);
          k1 += __shfl_xor_sync(0xffffffffu, up16 ? p1 : p3, 16);
          float kk = up8 ? k1 : k0;
          kk += __shfl_xor_sync(0xffffffffu, up8 ? k0 : k1, 8);
          const float val = oct_sum(kk) + Pm[PL.bv];
          float dv;
          bool vin = true;  // clip_range_vf: the clamp passes the gradient (torch's clamp backward: edges included)
          if (A.clip_vf > 0.f) {
            const float vold = live ? rollout[(int64_t)IDX[base + lrow] * rw + col_logp + 1] : 0.f, dvo = val - vold;
            dv = (vold + fminf(fmaxf(dvo, -A.clip_vf), A.clip_vf)) - RET[lrow];
            vin = dvo >= -A.clip_vf && dvo <= A.clip_vf;
          } else {
            dv = val - RET[lrow];
          }
          const float dval = (live && vin) ? A.hp.vf_coef * 2.0f * dv * inv_nb : 0.f;
          if (la == 0) {
            if (live) l_v += dv * dv;
            DVAL[lrow] = dval;
            if (rec && live) RSL[RS_V * RG + lrow] += dv * dv;
          }
          const float d0 = __shfl_sync(0xffffffffu, dval, 0), d1 = __shfl_sync(0xffffffffu, dval, 8);
          const float d2 = __shfl_sync(0xffffffffu, dval, 16), d3 = __shfl_sync(0xffffffffu, dval, 24);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            dl[u][0] = d0 * wvj[u];
            dl[u][1] = d1 * wvj[u];
            dl[u][2] = d2 * wvj[u];
            dl[u][3] = d3 * wvj[u];
          }
        } else {
          const float* Wa = Pm + PL.wa;
          // action means / logits from the latent tile: lane = (action ab + lane / 4, row lane % 4), a dot over the HP
          // units (pad units hold zeros)
          __syncwarp();
          {
            const int asub = lane >> 2, rrr = lane & 3;
            for (int ab = 0; ab < Da; ab += 8) {
              const int a = ab + asub, ac = a < Da ? a : 0;
              const float* wr = Wa + ac * ldh;
              const float* lr = cLAT + r0 + rrr;
              float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 8
              for (int jj = 0; jj < HP; jj += 4) {
                s0 = fmaf(wr[jj], lr[jj * RG], s0);
                s1 = fmaf(wr[jj + 1], lr[(jj + 1) * RG], s1);
                s2 = fmaf(wr[jj + 2], lr[(jj + 2) * RG], s2);
                s3 = fmaf(wr[jj + 3], lr[(jj + 3) * RG], s3);
              }
              if (a < Da) MEAN[a * RG + r0 + rrr] = ((s0 + s1) + (s2 + s3)) + Pm[PL.ba + a];
            }
          }
          __syncwarp();
          if constexpr (DQN) {
            // smooth L1 (beta 1) between Q(s)[a] and y = LPO: its gradient clamp(d, -1, 1) / mb on the taken action
            const int act = (int)ACT[lrow];
            const float y = LPO[lrow];
            for (int a = la; a < Da; a += 8) {
              float g = 0.f;
              if (live && a == act) {
                const float d = MEAN[a * RG + lrow] - y, ad = fabsf(d);
                l_pg += ad < 1.0f ? 0.5f * d * d : ad - 0.5f;
                g = fminf(fmaxf(d, -1.0f), 1.0f) * inv_nb;
              }
              DM[a * RG + lrow] = g;
              DLS[a * RG + lrow] = 0.f;
            }
          } else {
          const float adv = ADV[lrow], logp_old = LPO[lrow];
          float logp = 0.f, ent = 0.f;
          int act = 0;
          if (!pd.discrete) {
            const float* lstd = Pm + PL.ls;
            for (int a = la; a < Da; a += 8) {
              const float ls = lstd[a], ivar = __expf(-2.0f * ls);
              const float diff = ACT[a * RG + lrow] - MEAN[a * RG + lrow];
              const float d2 = diff * diff * ivar;
              logp += -0.5f * d2 - ls - 0.9189385332046727f;
              ent += 1.4189385332046727f + ls;
              DM[a * RG + lrow] = diff * ivar;   // d logp / d mean
              DLS[a * RG + lrow] = d2 - 1.0f;    // d logp / d log_std
            }
          } else {
            float mx = -INFINITY;
            for (int a = la; a < Da; a += 8) mx = fmaxf(mx, MEAN[a * RG + lrow]);
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            float se = 0.f;
            for (int a = la; a < Da; a += 8) se += expf(MEAN[a * RG + lrow] - mx);
            const float lse = mx + logf(oct_sum(se));
            act = (int)ACT[lrow];
            for (int a = la; a < Da; a += 8) {
              const float lp = MEAN[a * RG + lrow] - lse;
              if (a == act) logp = lp;
              ent -= expf(lp) * lp;
              DLS[a * RG + lrow] = lp;  // temporarily: log p_a
            }
          }
          logp = oct_sum(logp);
          ent = oct_sum(ent);
          float dl_dlogp, dent;
          if constexpr (BC) {
            // loss x mb / batch_size (bc.py:501): d / d logp = -1 / batch_size, d / d entropy = -ent_weight / batch_size;
            // l_pg, l_v, l_ent collect sum logp, sum exp(logp), sum entropy for the metrics
            dl_dlogp = live ? -B.inv_bs : 0.f;
            dent = live ? -A.hp.ent_coef * B.inv_bs : 0.f;
            if (live && la == 0) {
              l_pg += logp;
              l_v += expf(logp);
              l_ent += ent;
            }
          } else {
          const float ratio = __expf(logp - logp_old);
          const float lo = 1.0f - A.hp.clip_range, hi = 1.0f + A.hp.clip_range;
          const float pl1 = adv * ratio, pl2 = adv * fminf(fmaxf(ratio, lo), hi);
          const bool inside = (ratio >= lo) && (ratio <= hi);
          dl_dlogp = (inside || pl1 < pl2) ? -adv * ratio * inv_nb : 0.f;
          dent = -A.hp.ent_coef * inv_nb;  // d(ent_coef * ent_loss) / d(entropy)
          if (live) {
            if (la == 0) {
              l_pg += -fminf(pl1, pl2);
              l_ent += -ent;
              if (rec) {  // the row's statistics terms
                RSL[RS_PG * RG + lrow] += -fminf(pl1, pl2);
                RSL[RS_ENT * RG + lrow] += -ent;
                RSL[RS_CLIP * RG + lrow] += fabsf(ratio - 1.0f) > A.hp.clip_range ? 1.f : 0.f;
                RSL[RS_KL * RG + lrow] += (ratio - 1.0f) - (logp - logp_old);
              }
            }
          } else {
            dl_dlogp = 0.f;
            dent = 0.f;
          }
          }
          if (!pd.discrete) {
            for (int a = la; a < Da; a += 8) {
              DLS[a * RG + lrow] = live ? dl_dlogp * DLS[a * RG + lrow] + dent : 0.f;  // dH/dlog_std = 1
              DM[a * RG + lrow] = live ? dl_dlogp * DM[a * RG + lrow] : 0.f;
            }
          } else {
            for (int a = la; a < Da; a += 8) {
              const float lp = DLS[a * RG + lrow], pp = expf(lp);
              DM[a * RG + lrow] = live ? dl_dlogp * (((a == act) ? 1.f : 0.f) - pp) + dent * (-pp * (lp + ent)) : 0.f;
              DLS[a * RG + lrow] = 0.f;
            }
          }
          }
          __syncwarp();
#pragma unroll 2
          for (int a = 0; a < Da; ++a) {
            const float4 d = ld4(DM + a * RG + r0);
#pragma unroll
            for (int u = 0; u < U; ++u) {
              const float waj = Wa[a * ldh + jc[u]];
              dl[u][0] = fmaf(d.x, waj, dl[u][0]);
              dl[u][1] = fmaf(d.y, waj, dl[u][1]);
              dl[u][2] = fmaf(d.z, waj, dl[u][2]);
              dl[u][3] = fmaf(d.w, waj, dl[u][3]);
            }
          }
        }
        // dL/dz2, backward through layer 2 (lane = input unit i: dH1[i] = sum_j DZ2[j] W2[j][i]), dL/dz1
#pragma unroll
        for (int u = 0; u < U; ++u)
          st4(cDZ2 + (lane + 32 * u) * RG + r0,
              make_float4(jl[u] ? ppo_act_grad<PACT>(dl[u][0], lat[u][0]) : 0.f,
                          jl[u] ? ppo_act_grad<PACT>(dl[u][1], lat[u][1]) : 0.f,
                          jl[u] ? ppo_act_grad<PACT>(dl[u][2], lat[u][2]) : 0.f,
                          jl[u] ? ppo_act_grad<PACT>(dl[u][3], lat[u][3]) : 0.f));
        __syncwarp();
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u][0] = acc[u][1] = acc[u][2] = acc[u][3] = 0.f;
#pragma unroll 4
        for (int jj = 0; jj < h; ++jj) {
          const float4 d = ld4(cDZ2 + jj * RG + r0);
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const float w = cW2[jj * ldh + jc[u]];
            acc[u][0] = fmaf(d.x, w, acc[u][0]);
            acc[u][1] = fmaf(d.y, w, acc[u][1]);
            acc[u][2] = fmaf(d.z, w, acc[u][2]);
            acc[u][3] = fmaf(d.w, w, acc[u][3]);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
          st4(cDZ1 + (lane + 32 * u) * RG + r0,
              make_float4(jl[u] ? ppo_act_grad<PACT>(acc[u][0], h1[u][0]) : 0.f,
                          jl[u] ? ppo_act_grad<PACT>(acc[u][1], h1[u][1]) : 0.f,
                          jl[u] ? ppo_act_grad<PACT>(acc[u][2], h1[u][2]) : 0.f,
                          jl[u] ? ppo_act_grad<PACT>(acc[u][3], h1[u][3]) : 0.f));
      }
      __syncthreads();
      // weight gradients of the pass's RG rows, accumulated into GP (P-layout): thread = (tower, unit gj, every
      // NWQ-th input); the unit's dL/dz rows live in registers, the input rows are warp-uniform broadcasts
      {
        constexpr int NWQ = 128 / HP;
        const int net = tid >> 7, tt = tid & 127;
        const int gj = tt % HP, wq = tt / HP;
        const float* H1 = TH1 + net * HP * RG;
        const float* LAT = TLAT + net * HP * RG;
        const float* DZ2 = TDZ2 + net * HP * RG;
        const float* DZ1 = TDZ1 + net * HP * RG;
        const int o_w1 = net ? PL.w1[1] : PL.w1[0], o_b1 = net ? PL.b1[1] : PL.b1[0];
        const int o_w2 = net ? PL.w2[1] : PL.w2[0], o_b2 = net ? PL.b2[1] : PL.b2[0];
        float dz[16];
        if (gj < h && (!NOV || net == 0)) {
          load16(dz, DZ2 + gj * RG);
          for (int i = wq; i < h; i += NWQ) GP[o_w2 + gj * ldh + i] += dot16r(dz, H1 + i * RG);
          if (wq == 0) GP[o_b2 + gj] += sum16(dz);
          load16(dz, DZ1 + gj * RG);
          for (int k = wq; k < Do; k += NWQ) GP[o_w1 + gj * ldo + k] += dot16r(dz, XN + k * RG);
          if (wq == NWQ - 1) GP[o_b1 + gj] += sum16(dz);
          load16(dz, LAT + gj * RG);
          if (net == 0) {
            for (int a = wq; a < Da; a += NWQ) GP[PL.wa + a * ldh + gj] += dot16r(dz, DM + a * RG);
          } else if (wq == 0) {
            GP[PL.wv + gj] += dot16r(dz, DVAL);
          }
        }
        if (net == 1 && wq == NWQ - 1) {  // ba, log_std, bv: plain row sums
          for (int t = gj; t <= 2 * Da; t += HP) {
            if (t < Da) {
              load16(dz, DM + t * RG);
              GP[PL.ba + t] += sum16(dz);
            } else if (t < 2 * Da) {
              if (!pd.discrete) {
                load16(dz, DLS + (t - Da) * RG);
                GP[PL.ls + t - Da] += sum16(dz);
              }
            } else {
              load16(dz, DVAL);
              GP[PL.bv] += sum16(dz);
            }
          }
        }
      }
      __syncthreads();  // the tiles are restaged by the next pass
    }

    // ---- 3. loss terms -> CTA 0; cluster barrier: every CTA's partial gradient is complete ---------------------------
    float l2sum = 0.f;  // BC metrics: sum of w^2 at the minibatch's parameters (every CTA holds all of them)
    if (BC && bc_log && crank == 0) {
      float q = 0.f;
      for (int i = tid; i < CL * S; i += PT) q = fmaf(Pm[i], Pm[i], q);  // (pad elements are 0)
      l2sum = block_sum(q, red);
    }
    if (BC ? bc_log : loss_log != nullptr) {  // (uniform)
      const float s_pg = block_sum(l_pg, red);
      const float s_v = block_sum(l_v, red);
      const float s_ent = block_sum(l_ent, red);
      if (tid == 0) {
        float* L0 = cluster.map_shared_rank(LOSS, 0);
        L0[crank * 3 + 0] = s_pg;
        L0[crank * 3 + 1] = s_v;
        L0[crank * 3 + 2] = s_ent;
      }
    }
    if (A.stats && tid == PT - 1) ppo_stats_fold<RG>(ACC, RSL, inv_nb, start == 0);
    cluster.sync();
    if (crank == 0 && tid == 0 && loss_log) {
      float pg = 0.f, vl = 0.f, el = 0.f;
      for (int c = 0; c < CL; ++c) {
        pg += LOSS[c * 3 + 0];
        vl += LOSS[c * 3 + 1];
        el += LOSS[c * 3 + 2];
      }
      pg *= inv_nb, vl *= inv_nb, el *= inv_nb;
      const int64_t lrow = DQN ? adam_step - 1 - B.j0 : gs;
      loss_log[lrow * 4 + 0] = pg;
      loss_log[lrow * 4 + 1] = vl;
      loss_log[lrow * 4 + 2] = el;
      loss_log[lrow * 4 + 3] = pg + A.hp.ent_coef * el + A.hp.vf_coef * vl;
    }
    if constexpr (BC) {
      if (crank == 0 && tid == 0 && bc_log) {  // BCTrainingMetrics (bc.py:134-146)
        float lp = 0.f, pt = 0.f, en = 0.f;
        for (int c = 0; c < CL; ++c) {
          lp += LOSS[c * 3 + 0];
          pt += LOSS[c * 3 + 1];
          en += LOSS[c * 3 + 2];
        }
        float* o = B.metrics + (int64_t)n_logged * 8;
        const float neglogp = -(lp * inv_nb), entropy = en * inv_nb, ent_loss = -A.hp.ent_coef * entropy;
        const float l2_norm = l2sum * 0.5f, l2_loss = B.l2_weight * l2_norm;
        o[BC_M_NEGLOGP] = neglogp;
        o[BC_M_ENTROPY] = entropy;
        o[BC_M_ENT_LOSS] = ent_loss;
        o[BC_M_PROB_TRUE_ACT] = pt * inv_nb;
        o[BC_M_L2_NORM] = l2_norm;
        o[BC_M_L2_LOSS] = l2_loss;
        o[BC_M_LOSS] = neglogp + ent_loss + l2_loss;
        o[BC_M_BATCH] = (float)batch_num;
      }
      if (bc_log) ++n_logged;
    }
    // ---- 4. slice owners: sum the CL partials of the owned slice in fixed order (DSMEM loads), exchange the squared
    //         slice norms for clip_grad_norm_.  BC: add the sum to the batch's gradient so far; no norms -------------
    float ss = 0.f;
    for (int i0 = 4 * tid; i0 < S; i0 += 4 * PT) {
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int c = 0; c < CL; ++c) {  // fixed order: deterministic
        const float* rg = cluster.map_shared_rank(GP, c);
        const float4 t = ld4(rg + crank * S + i0);
        g.x += t.x, g.y += t.y, g.z += t.z, g.w += t.w;
      }
      if constexpr (BC) {  // loss.backward() accumulating into .grad (bc.py:502)
        const float4 a = ld4(Gs + i0);
        g.x = a.x + g.x, g.y = a.y + g.y, g.z = a.z + g.z, g.w = a.w + g.w;
      }
      st4(Gs + i0, g);
      if constexpr (!BC) ss += (g.x * g.x + g.y * g.y) + (g.z * g.z + g.w * g.w);
    }
    float clip = 1.0f;  // BC: no clip_grad_norm_
    if constexpr (!BC) {
      const float my_ssq = block_sum(ss, red);
      if (tid < CL) {
        cluster.map_shared_rank(SSQ, tid)[crank] = my_ssq;
        if (kl_on) cluster.map_shared_rank(KLS, tid)[crank] = ppo_kl_part<RG>(RSL, inv_nb);
      }
      cluster.sync();  // all slice norms are in place everywhere; nobody reads a peer's GP any more
      if (kl_on) {
        // target_kl (SB3: approx_kl > 1.5 target_kl): the CL shares summed in the same order everywhere, so every CTA
        // reaches the same decision; a stopping step takes no Adam step and all CTAs leave the loop here
        float kl = 0.f;
#pragma unroll
        for (int c = 0; c < CL; ++c) kl += KLS[c];
        if (kl > 1.5f * A.target_kl) {
          kstop = gs + 1;
          break;
        }
      }
      float total = 0.f;
#pragma unroll
      for (int c = 0; c < CL; ++c) total += SSQ[c];  // same order everywhere: the replicas' clip factors agree bit for bit
      total = sqrtf(total);
      clip = A.hp.max_grad_norm / (total + 1e-6f);
      clip = clip > 1.0f ? 1.0f : clip;
    }
    // ---- 5. clip_grad_norm_ + Adam on the OWNED slice; the new parameters go into every CTA's parameter vector.  BC:
    //         only a minibatch that ends a batch steps.  No CTA reads parameters between the barrier of section 3 and
    //         the one below, nor a peer's GP after it, so one barrier closes a BC minibatch ----------------------------
    if (bc_step) {
      const float step_size = bc[0], inv_bc2s = rcp_fast(bc[1]);
      auto adam1 = [&](float gg, float& m, float& v, float& pw) {
        gg *= clip;
        m = m + (gg - m) * (1.0f - 0.9f);
        v = v * 0.999f + (1.0f - 0.999f) * gg * gg;
        pw -= step_size * __fdividef(m, fmaf(sqrt_fast(v), inv_bc2s, A.hp.adam_eps));
      };
      for (int i0 = 4 * tid; i0 < S; i0 += 4 * PT) {
        float4 g = ld4(Gs + i0);
        float4 m = ld4(Ms + i0), v = ld4(Vs + i0), pw = ld4(Pm + crank * S + i0);
        if constexpr (BC) {  // + the L2 term's gradient (bc.py:138-145, every parameter); the next batch starts from 0
          g.x = fmaf(l2c, pw.x, g.x), g.y = fmaf(l2c, pw.y, g.y), g.z = fmaf(l2c, pw.z, g.z), g.w = fmaf(l2c, pw.w, g.w);
          st4(Gs + i0, make_float4(0.f, 0.f, 0.f, 0.f));
        }
        adam1(g.x, m.x, v.x, pw.x);
        adam1(g.y, m.y, v.y, pw.y);
        adam1(g.z, m.z, v.z, pw.z);
        adam1(g.w, m.w, v.w, pw.w);
        st4(Ms + i0, m);
        st4(Vs + i0, v);
#pragma unroll
        for (int c = 0; c < CL; ++c) {  // rotated start: the CL owners write to CL different CTAs at a time
          const int dstc = (crank + c) & (CL - 1);
          st4(cluster.map_shared_rank(Pm, dstc) + crank * S + i0, pw);
        }
      }
    }
    cluster.sync();  // every CTA holds all new parameter slices
    start += mb;
    if (start >= (BC ? (int)steps_per_epoch * mb : Ni)) {  // (BC: the remainder rows are dropped, drop_last=True)
      start = 0;
      ++ep_now;
    }
  }

  // ---- write back: moments by their owners, parameters / norm state / counters by CTA 0 -------------------------------
  for (int p = tid; p < NP; p += PT) {
    const int q = flat_to_play(pd, PL, p);
    if (q / S == crank) {
      g_m[p] = Ms[q - crank * S];
      g_v[p] = Vs[q - crank * S];
      if (BC && (B.j0 + B.n_mb) % B.k != 0 && B.final_flush != 1) B.carry[p] = Gs[q - crank * S];  // the batch goes on
    }
  }
  if (crank == 0) {
    for (int p = tid; p < NP; p += PT) g_params[p] = Pm[flat_to_play(pd, PL, p)];
    if (pd.has_norm) {
      if (tid < Do) {
        g_norm[tid] = rstat[tid];
        g_norm[Do + tid] = rstat[64 + tid];
      }
      if (tid == 0) *g_norm_count = run_count;
    }
    if (tid == 0) {
      state[IMB_ST_PPO_STEP] = kstop ? adam_step - 1 : adam_step;  // (the stopping step took no Adam step)
      if constexpr (BC) {  // the epochs the launch completed
        state[IMB_ST_PPO_EPOCH] = perm_draw0 + (B.j0 + B.n_mb) / steps_per_epoch - B.j0 / steps_per_epoch;
      } else if constexpr (!DQN) {  // (DQN steps draw no permutations: a launch is not an epoch)
        state[IMB_ST_PPO_EPOCH] = perm_draw0 + (kstop ? ep_now + 1 : A.hp.n_epochs);
      }
    }
  }
  if (A.stats) {
    if (tid == 0) ppo_stats_push(cluster, TH1, ACC, EVP, crank);  // (the pass tiles are free now)
    cluster.sync();
    if (crank == 0 && tid == 0) {
      float sd = __int_as_float(0x7fc00000);
      if (!pd.discrete) {
        sd = 0.f;
        for (int a = 0; a < Da; ++a) sd += expf(Pm[PL.ls + a]);
        sd /= (float)Da;
      }
      const int64_t n_eval = kstop ? kstop : n_steps;
      ppo_stats_finish(TH1, A.stats, A, n_eval, (n_eval - 1) / steps_per_epoch + 1, steps_per_epoch, sd,
                       state[IMB_ST_PPO_EPOCH], kstop != 0);
    }
  }
  cluster.sync();  // no CTA may exit while peers can still address its shared memory
}
