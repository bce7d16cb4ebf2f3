// imb_ppo.cu -- the generator update (PPO) as ONE persistent thread-block-cluster launch per round.
//
// The reference delegates this to stable-baselines3 (algorithms/adversarial/common.py:414,
// gen_algo.learn -> PPO.train); its arithmetic is restated in oracle/ppo_port.py (parity
// unpinned by the reference, SURVEY.md section 8c).  PPO.train is n_epochs x (N / batch_size)
// strictly sequential optimiser steps on 64-row minibatches: each step is ~1.3 MFLOP, far below
// launch latency, so the whole loop runs inside one kernel with parameters, gradients and Adam
// moments resident in the shared memory of an 8-CTA thread-block cluster (see k_ppo_update):
//   prefetch minibatch rows by permutation -> [feature RunningNorm update] -> advantage
//   normalisation -> warp-autonomous forward / loss / backward chain -> weight gradients ->
//   DSMEM exchange (st.async + mbarriers) -> clip_grad_norm_ -> Adam on the owned slice -> parameter all-gather.
// Also: imb_policy_logp = ActorCriticPolicy.evaluate_actions()[1] for the AIRL discriminator
// batch (common.py:476-519).
#include <cooperative_groups.h>
#include <stdlib.h>

#include "imb_common.cuh"
#include "imb_tile.cuh"

#ifdef IMB_PPO_TIMING
// phase timing: CTA 0 / thread 0 accumulates clock64() deltas per phase of the optimiser step
__device__ long long g_ppo_clk[24];
__device__ long long g_ppo_wclk[80];  // [slot][warp]: cycles since the top barrier at points of the warp chain (CTA 0)
#define PPO_TICK(i)                                  \
  do {                                               \
    if (tid == 0) {                                  \
      const long long now_ = clock64();              \
      clk_acc[i] += now_ - clk_last;                 \
      clk_last = now_;                               \
    }                                                \
  } while (0)
#define PPO_WCLK(slot)                                   \
  do {                                                   \
    if (lane == 0) wacc[slot] += clock64() - wclk0;      \
  } while (0)
#else
#define PPO_TICK(i) do {} while (0)
#define PPO_WCLK(slot) do {} while (0)
#endif
#ifndef PPO_TANH
#define PPO_TANH(x) tanh_fast(x)
#endif

namespace {

constexpr int PT = 256;   // threads per CTA: warps 0, 1 = policy chain, 2, 3 = value chain, 4-7 = statistics / prefetch
constexpr int CL = 8;     // CTAs per cluster: each owns RL rows of every minibatch and 1/CL of the gradient reduction
constexpr int RL = 8;     // minibatch rows per CTA  (CL * RL = 64 >= SB3 batch_size)
constexpr int PR = CL * RL;

struct PpoArgs {
  imb_policy_desc pol;
  imb_ppo_hparams hp;
  int64_t n_rows;
  int rw;
  uint64_t seed;
  int HP, KP, S;  // tower width / obs width padded to 32; padded-layout parameters per slice (multiple of 4)
  int RS2;        // staged row stride in shared memory: >= rw, = 4 (mod 8)
  float target_kl, clip_vf;  // SB3 PPO target_kl / clip_range_vf; <= 0: off
  float* stats;              // IMB_PPO_STAT_* of the launch, or NULL
};

// Padded parameter layout used inside the kernel ("P-layout"): W1 rows have stride ldo = d_obs|1 and W2 rows
// stride ldh = hidden|1 (odd), so that BOTH access patterns of the step -- lane = output unit (forward,
// weight gradients) and lane = input unit (backward) -- are shared-memory bank-conflict free straight from the
// parameter vector; no transposed working copies have to be rebuilt after every optimiser step.  The pad
// elements have zero value and zero gradient for ever (Adam leaves them at 0).
struct PLay {
  int w1[2], b1[2], w2[2], b2[2], wa, ba, wv, bv, ls, ldo, ldh, total;
};
__host__ __device__ inline PLay make_play(const int Do, const int Da, const int h, const bool discrete) {
  PLay L{};
  L.ldo = Do | 1;
  L.ldh = h | 1;
  int o = 0;
  for (int t = 0; t < 2; ++t) {
    L.w1[t] = o; o += h * L.ldo;
    L.b1[t] = o; o += h;
    L.w2[t] = o; o += h * L.ldh;
    L.b2[t] = o; o += h;
  }
  L.wa = o; o += Da * L.ldh;
  L.ba = o; o += Da;
  L.wv = o; o += h;
  L.bv = o; o += 1;
  L.ls = o; o += discrete ? 0 : Da;
  L.total = o;
  return L;
}
__host__ __device__ inline PLay make_play(const imb_policy_desc& pd) {
  return make_play(pd.d_obs, pd.d_act, pd.hidden, pd.discrete != 0);
}
// Launch geometry of k_ppo_update, from the shape alone (the host plans with these, a shape-specialised instantiation
// folds them into constants): obs width padded to 32 or 64; padded-layout parameters per slice, a multiple of 4 and at
// least two quads (a quad's owner is qq / (S / 4), found through the 32-bit reciprocal 2^32 / (S / 4) + 1 when S is not
// a compile-time constant, which does not fit for S / 4 = 1: policies of <= 32 padded parameters, e.g. width 1); staged
// row stride >= rw, = 4 (mod 8).
__host__ __device__ inline int ppo_kp(const int Do) { return Do <= 32 ? 32 : 64; }
__host__ __device__ inline int ppo_slice(const PLay& L) { return max(8, ((L.total + CL - 1) / CL + 3) / 4 * 4); }
__host__ __device__ inline int ppo_row_stride(const int rw) { return ((rw + 4) % 8 == 4) ? rw + 4 : rw + 8; }
// torch-flat parameter index -> P-layout index
__device__ inline int flat_to_play(const imb_policy_desc& pd, const PLay& L, int p) {
  const int Do = pd.d_obs, Da = pd.d_act, h = pd.hidden;
  auto in = [&](int off, int len) { return p >= off && p < off + len; };
  if (in(pd.off_pi_w1, h * Do)) { const int i = p - pd.off_pi_w1; return L.w1[0] + (i / Do) * L.ldo + i % Do; }
  if (in(pd.off_vf_w1, h * Do)) { const int i = p - pd.off_vf_w1; return L.w1[1] + (i / Do) * L.ldo + i % Do; }
  if (in(pd.off_pi_w2, h * h)) { const int i = p - pd.off_pi_w2; return L.w2[0] + (i / h) * L.ldh + i % h; }
  if (in(pd.off_vf_w2, h * h)) { const int i = p - pd.off_vf_w2; return L.w2[1] + (i / h) * L.ldh + i % h; }
  if (in(pd.off_pi_b1, h)) return L.b1[0] + p - pd.off_pi_b1;
  if (in(pd.off_vf_b1, h)) return L.b1[1] + p - pd.off_vf_b1;
  if (in(pd.off_pi_b2, h)) return L.b2[0] + p - pd.off_pi_b2;
  if (in(pd.off_vf_b2, h)) return L.b2[1] + p - pd.off_vf_b2;
  if (in(pd.off_act_w, Da * h)) { const int i = p - pd.off_act_w; return L.wa + (i / h) * L.ldh + i % h; }
  if (in(pd.off_act_b, Da)) return L.ba + p - pd.off_act_b;
  if (in(pd.off_val_w, h)) return L.wv + p - pd.off_val_w;
  if (p == pd.off_val_b) return L.bv;
  return L.ls + p - pd.off_log_std;
}

__device__ __forceinline__ float block_sum(float v, float* red) {
  // red: >= 16 floats of shared memory; all PT threads must call
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < PT / 32; ++w) t += red[w];
  return t;
}

// sum over the 8 lanes of an aligned lane group; ALL 32 lanes must call it convergently (a per-group member
// mask makes the compiler serialise the groups through MATCH.ANY: 40x more instructions, measured)
__device__ __forceinline__ float group8_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  return v;
}
__device__ __forceinline__ float rcp_fast(float x) { return __fdividef(1.0f, x); }
__device__ __forceinline__ float sqrt_fast(float x) {
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ float dot8r(const float (&d)[8], const float* __restrict__ b) {
  const float4 b0 = ld4(b), b1 = ld4(b + 4);
  float s0 = d[0] * b0.x, s1 = d[1] * b0.y;
  s0 = fmaf(d[2], b0.z, s0);
  s1 = fmaf(d[3], b0.w, s1);
  s0 = fmaf(d[4], b1.x, s0);
  s1 = fmaf(d[5], b1.y, s1);
  s0 = fmaf(d[6], b1.z, s0);
  s1 = fmaf(d[7], b1.w, s1);
  return s0 + s1;
}
__device__ __forceinline__ void load8(float (&d)[8], const float* __restrict__ p) {
  const float4 a = ld4(p), b = ld4(p + 4);
  d[0] = a.x, d[1] = a.y, d[2] = a.z, d[3] = a.w, d[4] = b.x, d[5] = b.y, d[6] = b.z, d[7] = b.w;
}
__device__ __forceinline__ float sum8(const float (&d)[8]) {
  return ((d[0] + d[1]) + (d[2] + d[3])) + ((d[4] + d[5]) + (d[6] + d[7]));
}
// d[i] = p[i * stride], i < N: N independent loads into a register array (compile-time indices only)
template <int N>
__device__ __forceinline__ void load_strided(float (&d)[N], const float* __restrict__ p, const int stride) {
#pragma unroll
  for (int i = 0; i < N; ++i) d[i] = p[i * stride];
}
// An empty asm that reads and writes every d[i]: the loads of d are issued before this point, and the compiler can neither
// sink them next to their uses nor load again there (with shared-memory offsets that are compile-time constants it can
// prove them independent of the stores in between, and did sink them without this)
template <int N>
__device__ __forceinline__ void pin_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i]));
}

// ---- training statistics of PPO.train (imb_ppo_update_ex: stats_out, target_kl) -----------------------------------
// Both kernels keep them in shared memory, out of the chain warps' registers.  Per step, the lanes that own a row's loss
// terms write them into per-row slots RSL[term][row] of their CTA; ONE thread per CTA folds the slots of the step, in
// row order and scaled by the step's 1 / nb, into the CTA's accumulators ACC; at the end of the launch CTA 0 sums the
// CL accumulators in rank order.  Per-row terms (dead rows 0):
enum { RS_PG = 0, RS_V, RS_ENT, RS_CLIP, RS_KL, RS_N };  // -min(surrogates), value error^2, -entropy, |r - 1| > clip, KL
// CTA accumulators: sums over the steps evaluated; the KL over the steps of the current epoch; the last step's losses
enum { AC_PG = 0, AC_V, AC_ENT, AC_CLIP, AC_KL_EPOCH, AC_LAST_PG, AC_LAST_V, AC_LAST_ENT, AC_N };

template <int NR>
__device__ __forceinline__ void ppo_stats_fold(float* __restrict__ acc, const float* __restrict__ rsl, const float inv_nb,
                                               const bool epoch_start) {
  // (one term at a time; RS_PG .. RS_CLIP share their indices with AC_PG .. AC_CLIP)
#pragma unroll 1
  for (int k = 0; k < RS_N; ++k) {
    float t = 0.f;
#pragma unroll
    for (int r = 0; r < NR; ++r) t += rsl[k * NR + r];
    t *= inv_nb;
    if (k == RS_KL) {
      acc[AC_KL_EPOCH] = epoch_start ? t : acc[AC_KL_EPOCH] + t;
    } else {
      acc[k] += t;
      if (k < RS_CLIP) acc[AC_LAST_PG + k] = t;  // the last step's losses
    }
  }
}

// k_ppo_update's fold, by one whole warp (the chain's RL = 8 rows): lane = (term lane / 8, row lane % 8) for the first
// four terms, the KL term's rows on every 8-lane group again; 8-lane butterfly sums, lane 0 updates the accumulators.
__device__ __forceinline__ void ppo_stats_fold_warp(float* __restrict__ acc, const float* __restrict__ rsl,
                                                    const float inv_nb, const bool epoch_start, const int lane) {
  static_assert(RS_CLIP == 3 && RS_KL == 4 && RL == 8, "fold layout");
  const float a = group8_sum(rsl[lane]), kl = group8_sum(rsl[RS_KL * RL + (lane & 7)]) * inv_nb;
  const float s_v = __shfl_sync(0xffffffffu, a, 8), s_ent = __shfl_sync(0xffffffffu, a, 16);
  const float s_clip = __shfl_sync(0xffffffffu, a, 24);
  if (lane == 0) {
    const float pg = a * inv_nb, v = s_v * inv_nb, ent = s_ent * inv_nb;
    acc[AC_PG] += pg;
    acc[AC_V] += v;
    acc[AC_ENT] += ent;
    acc[AC_CLIP] += s_clip * inv_nb;
    acc[AC_KL_EPOCH] = epoch_start ? kl : acc[AC_KL_EPOCH] + kl;
    acc[AC_LAST_PG] = pg;
    acc[AC_LAST_V] = v;
    acc[AC_LAST_ENT] = ent;
  }
}

// This CTA's share of the step's approx-KL (the target_kl test): its rows' KL terms in row order, times 1 / nb.
template <int NR>
__device__ __forceinline__ float ppo_kl_part(const float* __restrict__ rsl, const float inv_nb) {
  float t = 0.f;
#pragma unroll
  for (int r = 0; r < NR; ++r) t += rsl[RS_KL * NR + r];
  return t * inv_nb;
}

// Explained variance of the rollout (SB3 explained_variance(values, returns)): this CTA's sums over rows crank * PT + tid
// (stride CL * PT) of y = ret and e = ret - value (e rounded in fp32 like SB3's), both shifted by row 0's value so that a
// constant column gives a variance of exactly 0, in double; ev[4] = sum dy, sum dy^2, sum de, sum de^2 (thread 0 stores
// it).  All PT threads call it.  wred: PT / 32 doubles of shared memory.
__device__ __noinline__ void ppo_ev_partial(const float* __restrict__ rollout, const int64_t N, const int rw,
                                            const int col_val, const int col_ret, const int crank, double* ev,
                                            double* wred) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double y0 = rollout[col_ret], e0 = rollout[col_ret] - rollout[col_val];
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)crank * PT + tid; i < N; i += (int64_t)CL * PT) {
    const float y = rollout[i * rw + col_ret], e = y - rollout[i * rw + col_val];
    const double dy = (double)y - y0, de = (double)e - e0;
    s[0] += dy;
    s[1] += dy * dy;
    s[2] += de;
    s[3] += de * de;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    double v = s[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) wred[warp] = v;
    __syncthreads();
    if (tid == 0) {
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < PT / 32; ++w) t += wred[w];
      ev[k] = t;
    }
  }
}

// End of the launch, thread 0 of every CTA: its accumulators and explained-variance partials go to CTA 0's `box`
// ([CL][16] floats of shared memory no longer in use, 8-byte aligned) with remote stores; a cluster barrier follows.
template <typename Cluster>
__device__ __forceinline__ void ppo_stats_push(Cluster& cluster, float* box, const float* acc, const double* ev,
                                               const int crank) {
  float* dst = cluster.map_shared_rank(box, 0) + crank * 16;
#pragma unroll
  for (int k = 0; k < AC_N; ++k) dst[k] = acc[k];
#pragma unroll
  for (int k = 0; k < 4; ++k) reinterpret_cast<double*>(dst + 8)[k] = ev[k];
}

// CTA 0, one thread, after that barrier: the CL accumulators and explained-variance partials summed in rank order ->
// stats[IMB_PPO_STAT_*].  n_eval: optimiser steps evaluated (a target_kl stop included); n_epochs: epochs begun; spe:
// steps per epoch; std: mean exp(log_std) of the final policy (NaN: Discrete).
__device__ __noinline__ void ppo_stats_finish(const float* box, float* __restrict__ stats, const PpoArgs& A,
                                              const int64_t n_eval, const int64_t n_epochs, const int64_t spe,
                                              const float std, const int64_t n_updates, const bool stopped) {
  float acc[AC_N];
  double ev[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < AC_N; ++k) acc[k] = 0.f;
  for (int c = 0; c < CL; ++c) {  // fixed order: deterministic
    const float* a = box + c * 16;
    const double* e = reinterpret_cast<const double*>(box + c * 16 + 8);
#pragma unroll
    for (int k = 0; k < AC_N; ++k) acc[k] += a[k];
#pragma unroll
    for (int k = 0; k < 4; ++k) ev[k] += e[k];
  }
  const float ne = (float)n_eval;
  stats[IMB_PPO_STAT_ENTROPY_LOSS] = acc[AC_ENT] / ne;
  stats[IMB_PPO_STAT_PG_LOSS] = acc[AC_PG] / ne;
  stats[IMB_PPO_STAT_VALUE_LOSS] = acc[AC_V] / ne;
  stats[IMB_PPO_STAT_APPROX_KL] = acc[AC_KL_EPOCH] / (float)((n_eval - 1) % spe + 1);
  stats[IMB_PPO_STAT_CLIP_FRACTION] = acc[AC_CLIP] / ne;
  stats[IMB_PPO_STAT_LOSS] = acc[AC_LAST_PG] + A.hp.ent_coef * acc[AC_LAST_ENT] + A.hp.vf_coef * acc[AC_LAST_V];
  const double n = (double)A.n_rows;
  const double var_y = ev[1] / n - (ev[0] / n) * (ev[0] / n), var_e = ev[3] / n - (ev[2] / n) * (ev[2] / n);
  stats[IMB_PPO_STAT_EXPLAINED_VARIANCE] = var_y == 0.0 ? __int_as_float(0x7fc00000) : (float)(1.0 - var_e / var_y);
  stats[IMB_PPO_STAT_STD] = std;
  stats[IMB_PPO_STAT_N_UPDATES] = (float)n_updates;
  stats[IMB_PPO_STAT_N_STEPS] = (float)n_eval;
  stats[IMB_PPO_STAT_N_EPOCHS] = (float)n_epochs;
  stats[IMB_PPO_STAT_STOPPED] = stopped ? 1.f : 0.f;
}

// Weight gradients over the CTA's RL = 8 rows -> GP (P-layout, local shared memory), one block of one tower per routine,
// by NQ warps: thread = (unit gj = lane, every NQ-th input, wq = the warp's index among the NQ); the unit's dL/dz rows live
// in registers, the input rows are warp-uniform broadcasts, the scattered GP stores have odd lane strides (conflict free).
// Bias and head-bias gradients are plain row sums.  Every element is one dot8r / sum8 over the 8 rows in row order, so the
// thread that computes it and the time it does so do not change its bits.  The dot products of a group are all computed
// into registers BEFORE the group's stores: the compiler cannot prove that GP and the activation tiles do not alias, and
// with a store between two dots it serialises them (load latency + FMA chain per dot, ~55 cycles each; the blocks are
// latency bound).
// (the loops over inputs run from 0 with the thread's offset added inside, so that their trip counts are compile-time
// constants when the shape is)

// dW2 and b2 of a tower (operands: its H1 and dL/dz2 tiles); for the value tower also the value head's wv and bv (its
// latent tile and dL/dvalue)
template <int NQ, int HPx>
__device__ __forceinline__ void wgrad_layer2(const bool value, const int gj, const int wq, const int h, const int w2,
                                             const int b2, const int ldh, const int wv, const int bv,
                                             float* __restrict__ GP, const float* __restrict__ tH1,
                                             const float* __restrict__ tLAT, const float* __restrict__ tDZ2,
                                             const float* __restrict__ DVAL) {
  constexpr int RLc = 8;
  constexpr int T2 = (HPx + NQ - 1) / NQ;  // layer-2 inputs per thread
  float dz2[8];
  if (gj < h) {
    load8(dz2, tDZ2 + gj * RLc);
    float r[T2];  // dW2[gj][i], i = wq + NQ t
#pragma unroll
    for (int t = 0; t < T2; ++t) {
      const int i = wq + NQ * t;
      r[t] = dot8r(dz2, tH1 + (i < HPx ? i : 0) * RLc);
    }
    float rv = 0.f;
    if (value && wq == NQ - 1) {
      float lt[8];
      load8(lt, tLAT + gj * RLc);
      rv = dot8r(lt, DVAL);
    }
#pragma unroll
    for (int t = 0; t < T2; ++t) {
      const int i = wq + NQ * t;
      if (i < h) GP[w2 + gj * ldh + i] = r[t];
    }
    if (wq == 0) GP[b2 + gj] = sum8(dz2);
    if (value && wq == NQ - 1) GP[wv + gj] = rv;
  }
  if (value && wq == NQ - 1 && gj == 0) {
    load8(dz2, DVAL);
    GP[bv] = sum8(dz2);
  }
}

// dW1 and b1 of a tower (operands: its dL/dz1 tile and the normalised observations)
template <int NQ>
__device__ __forceinline__ void wgrad_layer1(const int gj, const int wq, const int h, const int Do, const int w1,
                                             const int b1, const int ldo, float* __restrict__ GP,
                                             const float* __restrict__ tDZ1, const float* __restrict__ XNc) {
  constexpr int RLc = 8;
  if (gj >= h) return;
  float dz1[8];
  load8(dz1, tDZ1 + gj * RLc);
#pragma unroll
  for (int kb = 0; kb < Do; kb += 4 * NQ) {  // dW1[gj][k], four at a time
    const int k0 = kb + wq;
    if (k0 >= Do) break;
    float r[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int k = k0 + NQ * t;
      r[t] = dot8r(dz1, XNc + (k < Do ? k : 0) * RLc);
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int k = k0 + NQ * t;
      if (k < Do) GP[w1 + gj * ldo + k] = r[t];
    }
  }
  if (wq == NQ - 1) GP[b1 + gj] = sum8(dz1);
}

// The policy's action head: Wa, ba and log_std (operands: the policy latent tile, dL/d(mean|logits), dL/dlog_std)
template <int NQ, int HPx>
__device__ __forceinline__ void wgrad_head(const int gj, const int wq, const int h, const int Da, const bool discrete,
                                           const PLay& L, float* __restrict__ GP, const float* __restrict__ tLAT,
                                           const float* __restrict__ DM, const float* __restrict__ DLS) {
  constexpr int RLc = 8;
  float d[8];
  if (gj < h) {
    load8(d, tLAT + gj * RLc);
#pragma unroll
    for (int ab = 0; ab < Da; ab += 2 * NQ) {
      const int a0 = ab + wq, a1 = a0 + NQ;
      if (a0 >= Da) break;
      const float ra = dot8r(d, DM + a0 * RLc), rb = dot8r(d, DM + (a1 < Da ? a1 : a0) * RLc);
      GP[L.wa + a0 * L.ldh + gj] = ra;
      if (a1 < Da) GP[L.wa + a1 * L.ldh + gj] = rb;
    }
  }
  if (wq == NQ - 1) {  // ba, log_std
#pragma unroll
    for (int tb = 0; tb < 2 * Da; tb += HPx) {
      const int t = tb + gj;
      if (t >= 2 * Da) break;
      if (t < Da) {
        load8(d, DM + t * RLc);
        GP[L.ba + t] = sum8(d);
      } else if (!discrete) {
        load8(d, DLS + (t - Da) * RLc);
        GP[L.ls + t - Da] = sum8(d);
      }
    }
  }
}

// Named barriers that hand a chain's tiles to the warps computing their weight gradients (0 is __syncthreads, 2 the owner
// warps' slice-norm reduction): the value tower's dL/dz2 tile, the policy head's operands (latent tile, dL/dmean,
// dL/dlog_std), the policy tower's dL/dz2 tile, the value tower's dL/dz1 tile complete.  The chain warps bar.arrive (never
// blocking the chain), the gradient warps bar.sync; the count is both together.
enum { BAR_VDZ2 = 3, BAR_PHEAD = 4, BAR_PDZ2 = 5, BAR_VDZ1 = 6 };
__device__ __forceinline__ void bar_arrive(const int id, const int n) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory");
}
__device__ __forceinline__ void bar_sync(const int id, const int n) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// PPO.train for one rollout: n_epochs x ceil(N / batch) optimiser steps, ONE cluster of CL CTAs.
// Data flow of one optimiser step (64-row minibatch, CTA c owns rows 8c..8c+7, every CTA holds all parameters):
//   * the minibatch rows are staged row-major in shared memory by asynchronous 16-byte row copies issued TWO
//     steps ahead by warps 4-7 (indices drawn on the fly, three buffers), completion on an mbarrier;
//   * minibatch statistics (feature RunningNorm update, advantage normalisation) over all 64 rows are computed
//     redundantly and identically by every CTA -- one step ahead, by warps 4-7, BESIDE the chain of warps 0-3;
//   * forward + loss + backward to dL/dz run WARP-AUTONOMOUSLY on warps 0-3: warp = (tower, 4 own rows), lane =
//     hidden unit; only __syncwarp() between layers (the two towers interact through the summed loss only), so
//     the ~8 dependent stages of the chain cost no CTA barrier, and every weight read from shared memory
//     feeds four FMAs (with 2 rows per warp on all 8 warps the chain was bound by shared-memory wavefronts);
//   * weight gradients over the CTA's 8 rows: thread = (unit, input subset) of one tower, staged in local shared
//     memory in the parameter layout.  Each block (a tower's dW2 + b2, its dW1 + b1, the action head) starts as soon
//     as the chain warps signal its operand tiles (named barriers, bar.arrive on the chain side), on warps that are
//     idle then, while warps 0, 1 finish the policy chain; only the policy tower's dW1 + b1 is left for all eight
//     warps after the step's second barrier.  The staged vector is pushed to the peer slice
//     owners through distributed shared memory with 16-byte stores; owners sum the CL partials in fixed order (their
//     own straight from the staging vector), exchange the squared slice norms, run clip_grad_norm_ + Adam on their
//     slice (the moments never leave their owner) and all-gather the new parameters into every CTA's copy (their
//     own with a local store).
// No cluster barrier inside the step loop (the exchanged data signals mbarriers at the receivers), three CTA
// barriers per optimiser step; the only global-memory traffic inside a step is the asynchronous minibatch prefetch.
// DO != 0: an instantiation for one policy shape (DO obs, DA actions, DISC discrete, NORM feature RunningNorm, tower width
// HP), whose loop bounds, layout offsets and slice geometry are compile-time constants -- the loops of the step unroll
// completely and every shared-memory address is an immediate offset, instead of unrolled blocks plus guarded remainder
// iterations that expose a shared-memory latency on the dependent FMA chain at every block boundary.  The arithmetic and
// its order are the same in every instantiation.  DO = 0: the shape is read from A.pol (every other shape).  OPT = 0:
// target_kl and clip_range_vf are off, and their code is not compiled in (the step is the one without them).
template <int HP, int DO = 0, int DA = 0, int DISC = 0, int NORM = 0, int OPT = 0>
__global__ void __launch_bounds__(PT, 1) k_ppo_update(const PpoArgs A, float* __restrict__ g_params,
                                                      float* __restrict__ g_norm, int32_t* __restrict__ g_norm_count,
                                                      float* __restrict__ g_m, float* __restrict__ g_v,
                                                      const float* __restrict__ rollout,
                                                      const int64_t* __restrict__ perm_in,
                                                      float* __restrict__ loss_log, int64_t* __restrict__ state) {
  static_assert(HP == 32, "the warp-autonomous chain maps one lane to one hidden unit");
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int crank = (int)cluster.block_rank();
  extern __shared__ __align__(128) float smem[];
  __shared__ float red[32];
  __shared__ float bc[8];
  __shared__ __align__(8) uint64_t mbar[3];  // one per staged-minibatch buffer (step s lives in buffer s % 3)
  __shared__ __align__(8) uint64_t xbar[3];  // [0]: partial gradients of the owned slice arrived; [1]: all new parameter slices; [2]: all slice norms
  __shared__ float SSQ[CL];                  // squared gradient norms of the 8 slices (each written by its owner)
  __shared__ float nred[PT / 32];            // per-warp partial sums of the owned slice's squared norm
  // training statistics (see ppo_stats_fold) and target_kl: per-row slots of the step, accumulators, the CTAs' KL shares
  // of the step (they travel with SSQ), the stopping step + 1 (0: none), explained-variance partials
  __shared__ float RSL[RS_N * RL];
  __shared__ float ACC[AC_N];
  __shared__ float KLS[CL];
  __shared__ int KSTOP;
  __shared__ double EVP[4];
  __shared__ double EVW[PT / 32];
  const imb_policy_desc& pd = A.pol;
  constexpr bool SPEC = DO != 0;
  const int Do = SPEC ? DO : pd.d_obs, Da = SPEC ? DA : pd.d_act, h = SPEC ? HP : pd.hidden, NP = pd.n_params;
  const bool discrete = SPEC ? DISC != 0 : pd.discrete != 0, has_norm = SPEC ? NORM != 0 : pd.has_norm != 0;
  const PLay PL = make_play(Do, Da, h, discrete);
  const int KP = SPEC ? ppo_kp(Do) : A.KP, S = SPEC ? ppo_slice(PL) : A.S;
  // unroll factors of the chain's loops: complete for a compile-time shape
  constexpr int U_DO = SPEC ? DO : 8, U_H = SPEC ? HP : 8, U_DA = SPEC ? DA : 4;
  // Thread t < S / 4 owns quad t of this CTA's slice, so warps 0 .. n_own_w - 1 hold owned quads.  The warps above them
  // and above the chain's warps 0-3 run the next minibatch's statistics in the TAIL of the step, beside the slice sum,
  // norm exchange and Adam, so that nothing shared-memory heavy competes with the chain for issue slots; they issue the
  // row prefetch beside the chain.  With fewer than two such warps (policies of more than 192 quads per slice) the
  // statistics stay beside the chain too, on warps 4-7.
  const int n_own_w = (S / 4 + 31) / 32;
  const bool tail_stats = n_own_w <= PT / 32 - 2;
  const int st0 = tail_stats ? 32 * max(n_own_w, 4) : 128, nst = PT - st0;  // first statistics thread, their count
  const int ldo = PL.ldo, ldh = PL.ldh;
  const int da_store = discrete ? 1 : Da;
  const int col_logp = Do + da_store, col_adv = col_logp + 3, col_ret = col_logp + 4;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // rollout row width (multiple of 4) / staged row stride (= 4 mod 8)
  const int rw = SPEC ? imb_row_width(Do, Da, discrete) : A.rw, RS2 = SPEC ? ppo_row_stride(rw) : A.RS2;
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const bool kl_on = OPT && A.target_kl > 0.f, vf_on = OPT && A.clip_vf > 0.f;  // (uniform)

  // ---- shared-memory carve-up (identical in every CTA: DSMEM addresses are rank + offset) ---------------
  int o = 0;
  float* Pm = smem + o; o += al(CL * S);        // parameters, P-layout, padded to CL slices
  float* Ms = smem + o; o += al(CL * S);        // Adam moments (P-layout indexing; only the owned slice is live)
  float* Vs = smem + o; o += al(CL * S);
  float* GP = smem + o; o += al(CL * S);        // own partial gradient (staging for the push)
  float* RECV = smem + o; o += al(CL * S);      // [source CTA][S]: partial gradients of the owned slice
  float* LOSS = smem + o; o += 32;              // [CL][3] partial loss sums (read by CTA 0)
  const int DAP = (Da + 3) / 4 * 4;
  const int rsz = al(PR * RS2);
  float* ROWS = smem + o; o += 3 * rsz;         // triple-buffered minibatch, row-major [64][RS2]
  // own-row tiles, feature-major [feature][RL]
  const int xsz = al(KP * RL);
  float* XNo = smem + o; o += 2 * xsz;          // normalised observations, double-buffered by step parity
  float* TH1 = smem + o; o += 2 * HP * RL;
  float* TLAT = smem + o; o += 2 * HP * RL;
  float* TDZ2 = smem + o; o += 2 * HP * RL;
  float* TDZ1 = smem + o; o += 2 * HP * RL;
  float* DM = smem + o; o += DAP * RL;          // dL/d(mean|logits) [a][RL]
  float* DLS = smem + o; o += DAP * RL;         // dL/d(log_std) per row [a][RL]
  float* MEAN = smem + o; o += DAP * RL;        // action means / logits [a][RL]
  float* DVAL = smem + o; o += 32;              // [RL] dL/dvalue
  float* rstat = smem + o; o += al(2 * 64 + 4); // running mean | var of the policy's feature RunningNorm

  for (int i = tid; i < CL * S; i += PT) Pm[i] = Ms[i] = Vs[i] = GP[i] = RECV[i] = 0.f;
  for (int i = tid; i < 3 * rsz; i += PT) ROWS[i] = 0.f;
  for (int i = tid; i < 2 * xsz + 8 * HP * RL + 3 * DAP * RL + 32; i += PT) XNo[i] = 0.f;  // XNo .. DVAL contiguous
  if (tid < 64) {
    rstat[tid] = (has_norm && tid < Do) ? g_norm[tid] : 0.f;
    rstat[64 + tid] = (has_norm && tid < Do) ? g_norm[Do + tid] : 1.f;
    LOSS[tid & 31] = 0.f;
  }
  if (tid < RS_N * RL) RSL[tid] = 0.f;
  if (tid < AC_N) ACC[tid] = 0.f;
  if (tid == 0) {
    KSTOP = 0;
    mbar_init(&mbar[0], nst);
    mbar_init(&mbar[1], nst);
    mbar_init(&mbar[2], nst);
    mbar_init(&xbar[0], 1);
    mbar_init(&xbar[1], 1);
    mbar_init(&xbar[2], 1);
    mbar_fence_init();
  }
  __syncthreads();
  for (int p = tid; p < NP; p += PT) {
    const int q = flat_to_play(pd, PL, p);
    Pm[q] = g_params[p];
    Ms[q] = g_m[p];
    Vs[q] = g_v[p];
  }
  int32_t run_count = has_norm ? *g_norm_count : 0;

  const int64_t N = A.n_rows;
  const int Ni = (int)N;
  const int mb = A.hp.batch_size;
  const int64_t steps_per_epoch = (N + mb - 1) / mb;
  const int64_t n_steps = steps_per_epoch * A.hp.n_epochs;
  int64_t adam_step = state[IMB_ST_PPO_STEP];
  const int64_t perm_draw0 = state[IMB_ST_PPO_EPOCH];
  double b1pow = pow(0.9, (double)adam_step), b2pow = pow(0.999, (double)adam_step);  // beta^t, kept incrementally
  const int row0 = crank * RL;        // first minibatch row owned by this CTA

  // Asynchronous row gather of one minibatch (epoch ep, first row start) into buffer `buf` by the nst statistics
  // threads: two (thread) tasks per row draw the row index and copy half of the 16-byte aligned rollout row each with
  // 16-byte cp.async (LDGSTS); completion is tracked by the buffer's mbarrier (one deferred arrival per thread).  (One
  // bulk-async copy per row and lane was tried first: the 32 per-lane UBLKCP issues serialise, ~2500 cycles per
  // warp.)  Rows are fetched at least one full optimiser step ahead (three buffers), so their latency is never waited for.
  auto issue_gather = [&](int ep, int start, int buf) {
    if (tid < st0) return;
    const int nbx = min(mb, Ni - start);
#pragma unroll
    for (int tb = 0; tb < 2 * PR; tb += nst) {
      const int t = tb + tid - st0, r = t >> 1, half = t & 1;
      if (t >= 2 * PR) break;
      if (r >= nbx) continue;
      int64_t idx;
      if (perm_in) {
        idx = perm_in[(int64_t)ep * N + start + r];
      } else {
        const FeistelKey fk = feistel_key(A.seed, IMB_STREAM_PPO_PERM, (uint64_t)(perm_draw0 + ep), (uint64_t)N);
        idx = (int64_t)feistel_perm(fk, (uint64_t)(start + r), (uint64_t)N);
      }
      const float* src = rollout + idx * rw;
      float* dst = ROWS + buf * rsz + r * RS2;
      const int nq = rw >> 2, q0 = half ? (nq + 1) >> 1 : 0, q1 = half ? nq : (nq + 1) >> 1;
#pragma unroll
      for (int qi = 0; qi < (nq + 1) >> 1; ++qi) {
        const int q = q0 + qi;
        if (q >= q1) break;
        cp_async16(dst + 4 * q, src + 4 * q);
      }
    }
    cp_async_mbar_arrive(&mbar[buf]);
  };
  // Statistics of one minibatch (step gs2, staged in buffer gs2 % 3): feature RunningNorm update + advantage
  // normalisation over all 64 rows, one 8-lane group per statistic, identically in every CTA; the group of
  // feature k also writes this CTA's own rows of it, normalised, into XNo[gs2 & 1][k][RL] (lane = row).  Run by
  // `ngrp` 8-lane groups (whole warps; group index gidx); all lanes run the same code (full-mask shuffles); idle
  // groups chew on the advantage column and discard the result.  The staged row stride RS2 = 4 (mod 8) makes
  // the 32 lanes of a warp (4 features x 8 rows) hit 32 banks.
  auto minibatch_stats = [&](int64_t gs2, int nbx, int gidx, int ngrp) {
    const int buf = (int)(gs2 % 3);
    float* R = ROWS + buf * rsz;
    float* XN = XNo + (int)(gs2 & 1) * xsz;
    const int gl = tid & 7;
    const float inv_nbx = 1.0f / (float)nbx;
    mbar_wait(&mbar[buf], (uint32_t)((gs2 / 3) & 1));  // all 64 row copies have landed
#pragma unroll
    for (int task0 = 0; task0 <= Do; task0 += ngrp) {
      const int task = task0 + gidx;
      const bool is_feat = task < Do, is_adv = task == Do;
      float* x = R + (is_feat ? task : col_adv);
      float v[8], s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[i] = (gl + 8 * i < nbx) ? x[(gl + 8 * i) * RS2] : 0.f;
        s += v[i];
      }
      const float bmean = group8_sum(s) * inv_nbx;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float d = (gl + 8 * i < nbx) ? v[i] - bmean : 0.f;
        q = fmaf(d, d, q);
      }
      const float ssd = group8_sum(q);
      if (is_feat) {
        float mean = 0.f, istd = 1.f;
        if (has_norm) {  // every lane of the group computes the update; lane 0 stores it
          mean = rstat[task];
          float var = rstat[64 + task];
          const float bvar = ssd * inv_nbx;
          const float bn = (float)nbx, c = (float)run_count, itot = rcp_fast(c + bn), delta = bmean - mean;
          mean += delta * bn * itot;
          var *= c;
          var += bvar * bn;
          var += delta * delta * c * bn * itot;
          var *= itot;
          istd = rsqrtf(var + pd.norm_eps);
          if (gl == 0) {
            if (kl_on && crank == 0 && gs2 > 0) {
              // target_kl: the statistics of step gs2 - 1 go out now -- if that step stops the training, they are the
              // result, and these are computed before the decision (the write-back skips rstat then)
              g_norm[task] = rstat[task];
              g_norm[Do + task] = rstat[64 + task];
            }
            rstat[task] = mean;
            rstat[64 + task] = var;
          }
        }
        XN[task * RL + gl] = (row0 + gl < nbx) ? (x[(row0 + gl) * RS2] - mean) * istd : 0.f;
      } else if (is_adv) {
        float am = 0.f, ais = 1.f;
        if (A.hp.normalize_advantage && nbx > 1) {
          am = bmean;
          ais = rcp_fast(sqrt_fast(ssd / (float)(nbx - 1)) + 1e-8f);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (gl + 8 * i < nbx) x[(gl + 8 * i) * RS2] = (v[i] - am) * ais;
      }
    }
  };
  __syncthreads();
  issue_gather(0, 0, 0);
  if (n_steps > 1) issue_gather(mb >= Ni ? 1 : 0, mb >= Ni ? 0 : mb, 1);
  if (A.stats) ppo_ev_partial(rollout, N, rw, col_logp + 1, col_ret, crank, EVP, EVW);  // (while the first rows land)
  minibatch_stats(0, min(mb, Ni), tid >> 3, PT / 8);
  if (has_norm) run_count += min(mb, Ni);  // (every thread keeps the count; the statistics' owners use it)
  // The gradient exchange is synchronised by the data itself: every 16-byte DSMEM store (st.async) completes
  // bytes on an mbarrier of the RECEIVING CTA, which waits until the expected byte count of the phase has
  // landed -- no cluster-wide barrier inside the step loop.  Each barrier is re-armed (one arrival + expected
  // bytes) by its owner right after the previous phase completed, which is always before a peer can send for
  // the next phase (a peer's next-phase data depends on data this CTA sends later).
  // A CTA never sends to itself: the slice sum reads its own partial from GP, the owner stores its new slice into its
  // own Pm directly, so both exchanges expect the bytes of the CL - 1 peers.
  const uint32_t xbytes = (uint32_t)((CL - 1) * S * 4);
  const unsigned qmagic = (unsigned)(0x100000000ull / (unsigned)(S / 4)) + 1u;  // exact quotient; S / 4 >= 2 (host)
  const uint32_t recv_sa = smem_u32(RECV), pm_sa = smem_u32(Pm), ssq_sa = smem_u32(SSQ);
  const uint32_t xbar0_sa = smem_u32(&xbar[0]), xbar1_sa = smem_u32(&xbar[1]), xbar2_sa = smem_u32(&xbar[2]);
  const uint32_t nbytes = (uint32_t)(CL * 4 * (kl_on ? 2 : 1));  // slice norms (+ the KL shares with target_kl)
  if (tid == 0) {
    mbar_expect_tx(&xbar[0], xbytes);
    mbar_expect_tx(&xbar[1], xbytes);
    mbar_expect_tx(&xbar[2], nbytes);
  }
  cluster.sync();

#ifdef IMB_PPO_TIMING
  long long clk_acc[16] = {0}, clk_last = clock64();
  long long wacc[10] = {0};  // per-warp chain clocks, kept in registers (a global RMW per sample stalls the chain)
#endif
  int ep_now = 0, start = 0;  // epoch and first row of the current step
  for (int64_t gs = 0; gs < n_steps; ++gs) {
    const int cur = (int)(gs & 1);
    const float* Rc = ROWS + (int)(gs % 3) * rsz;
    const float* XNc = XNo + cur * xsz;
    const int nb = min(mb, Ni - start);
    const float inv_nb = 1.0f / (float)nb;
    int ep_next = ep_now, start_next = start + mb;
    if (start_next >= Ni) {
      start_next = 0;
      ++ep_next;
    }
    ++adam_step;
    if (tid == PT - 1) {  // Adam bias corrections in double, off the critical path (double-buffered by step parity)
      b1pow *= 0.9;
      b2pow *= 0.999;
      bc[2 * cur] = (float)((double)A.hp.lr / (1.0 - b1pow));
      bc[2 * cur + 1] = (float)sqrt(1.0 - b2pow);
    }
    __syncthreads();  // the parameters written by the previous step's Adam (and XNo, the statistics) are visible
    if (kl_on && KSTOP) {
      // target_kl stopped the previous step: drain the row prefetch it issued for this step's successor, take back the
      // count this step's statistics (computed ahead) added, and leave together
      if (tid >= st0 && gs + 1 < n_steps) mbar_wait(&mbar[(int)((gs + 1) % 3)], (uint32_t)(((gs + 1) / 3) & 1));
      if (has_norm) run_count -= min(mb, Ni - start);
      break;
    }
    PPO_TICK(0);
#ifdef IMB_PPO_TIMING
    const long long wclk0 = clock64();
#endif
    float l_pg = 0.f, l_v = 0.f, l_ent = 0.f;
    // The NEXT step's minibatch statistics and own-row tile, by the statistics threads: they do not depend on the
    // parameters, and XNo[(gs + 1) & 1] and buffer (gs + 1) % 3 are not read in this step
    auto next_stats = [&]() {
      if (gs + 1 < n_steps) minibatch_stats(gs + 1, min(mb, Ni - start_next), (tid - st0) >> 3, nst / 8);
      PPO_WCLK(1);
    };
    if (warp >= 4) {
      // ---- 1b. the statistics threads, beside the chain: the statistics when they cannot go in the tail, then the row
      //          prefetch for the step after next into buffer (gs + 2) % 3 (last read by the previous step) -----------------
      if (tid >= st0) {
        if (!tail_stats) next_stats();
        if (gs + 2 < n_steps) {
          int ep2 = ep_next, start2 = start_next + mb;
          if (start2 >= Ni) {
            start2 = 0;
            ++ep2;
          }
          issue_gather(ep2, start2, (int)((gs + 2) % 3));
        }
        PPO_WCLK(3);
      }
    } else {
      // ---- 1a. warp-autonomous chain on warps 0-3: forward, loss terms, backward to dL/dz for (tower, 4 own rows).
      //          Four rows per warp: every weight fetched from shared memory feeds four FMAs (the chain was bound
      //          by shared-memory wavefronts with two rows per warp and all eight warps fetching) ---------------------
      const int cnet = warp >> 1;                // 0: policy tower (warps 0, 1), 1: value tower (warps 2, 3)
      const int j = lane, jc = lane < h ? lane : 0, r0 = 4 * (warp & 1);
      const bool jl = lane < h;
      const int rr = lane >> 3, la = lane & 7;   // per-row parts: lane octet rr handles row r0 + rr
      const int gr = row0 + r0 + rr;
      const bool live = gr < nb;
      const float* row = Rc + gr * RS2;
      float* cH1 = TH1 + cnet * HP * RL;
      float* cLAT = TLAT + cnet * HP * RL;
      float* cDZ2 = TDZ2 + cnet * HP * RL;
      float* cDZ1 = TDZ1 + cnet * HP * RL;
      const float* cW1 = Pm + (cnet ? PL.w1[1] : PL.w1[0]);
      const float* cW2 = Pm + (cnet ? PL.w2[1] : PL.w2[0]);
      const int c_b1 = cnet ? PL.b1[1] : PL.b1[0], c_b2 = cnet ? PL.b2[1] : PL.b2[0];
      // WREG: the lane's W2 row (forward, lane = output unit) and W2 column (backward, lane = input unit) come from
      // registers, each loaded as one block of 32 independent loads a phase before the loop that uses it (the row in
      // layer 1, the column in layer 2; pin_regs holds each block there), so those two loops issue only their activation
      // loads instead of a weight load beside every 16-byte activation load.  The FMAs and their order are unchanged;
      // only where a weight is read from moves (nothing writes Pm between the step's top barrier and the end of the
      // chain).  Only the shape-specialised Box instantiations: with runtime bounds the arrays would go to local memory,
      // and the Discrete one spills with them.  W1 and the action head's weights stay in shared memory: with them in
      // registers too the 17/6 instantiation spills.
      constexpr bool WREG = SPEC && !DISC;
      float w2r[WREG ? HP : 1], w2c[WREG ? HP : 1];
      if constexpr (WREG) load_strided(w2r, cW2 + jc * ldh, 1);
      // policy warps: everything the loss needs that does not depend on the forward pass is fetched now, so its
      // latency (shared-memory loads, the exponential) hides behind the layers
      const bool gfast = cnet == 0 && !discrete && Da <= 8;  // one action per lane of the octet
      float pre_adv = 0.f, pre_lpo = 0.f, pre_act = 0.f, pre_ls = 0.f, pre_ivar = 0.f;
      if (cnet == 0) {
        pre_adv = row[col_adv];
        pre_lpo = row[col_logp];
        if (gfast && la < Da) {
          pre_act = row[Do + la];
          pre_ls = Pm[PL.ls + la];
          pre_ivar = __expf(-2.0f * pre_ls);
        }
      }
      // layer 1
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      {
        const float* wp = cW1 + jc * ldo;
#pragma unroll U_DO
        for (int k = 0; k < Do; ++k) {
          const float w = wp[k];
          const float4 x = ld4(XNc + k * RL + r0);
          a0 = fmaf(x.x, w, a0);
          a1 = fmaf(x.y, w, a1);
          a2 = fmaf(x.z, w, a2);
          a3 = fmaf(x.w, w, a3);
        }
      }
      if constexpr (WREG) pin_regs(w2r);  // (loaded during layer 1)
      float b = Pm[c_b1 + jc];
      const float h10 = jl ? PPO_TANH(a0 + b) : 0.f, h11 = jl ? PPO_TANH(a1 + b) : 0.f;
      const float h12 = jl ? PPO_TANH(a2 + b) : 0.f, h13 = jl ? PPO_TANH(a3 + b) : 0.f;
      st4(cH1 + j * RL + r0, make_float4(h10, h11, h12, h13));
      __syncwarp();
      PPO_WCLK(3);
      if constexpr (WREG) load_strided(w2c, cW2 + jc, ldh);
      // layer 2
      a0 = a1 = a2 = a3 = 0.f;
      {
        const float* wp = cW2 + jc * ldh;
#pragma unroll U_H
        for (int i = 0; i < h; ++i) {
          const float w = WREG ? w2r[i] : wp[i];
          const float4 x = ld4(cH1 + i * RL + r0);
          a0 = fmaf(x.x, w, a0);
          a1 = fmaf(x.y, w, a1);
          a2 = fmaf(x.z, w, a2);
          a3 = fmaf(x.w, w, a3);
        }
      }
      if constexpr (WREG) pin_regs(w2c);  // (loaded during layer 2)
      b = Pm[c_b2 + jc];
      const float lat0 = jl ? PPO_TANH(a0 + b) : 0.f, lat1 = jl ? PPO_TANH(a1 + b) : 0.f;
      const float lat2 = jl ? PPO_TANH(a2 + b) : 0.f, lat3 = jl ? PPO_TANH(a3 + b) : 0.f;
      st4(cLAT + j * RL + r0, make_float4(lat0, lat1, lat2, lat3));
      PPO_WCLK(4);
      // heads + loss terms; dl0..dl3 = dL/dlatent of this unit for the four rows
      float dl0 = 0.f, dl1 = 0.f, dl2 = 0.f, dl3 = 0.f;
      auto oct_sum = [&](float v) {
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        return v;
      };
      if (cnet == 1) {
        // value head: four sums over the 32 units, transposed on the way so that octet rr ends with row r0 + rr's
        const float wvj = jl ? Pm[PL.wv + j] : 0.f;
        const float p0 = lat0 * wvj, p1 = lat1 * wvj, p2 = lat2 * wvj, p3 = lat3 * wvj;
        const bool up16 = (lane & 16) != 0, up8 = (lane & 8) != 0;
        float k0 = up16 ? p2 : p0, k1 = up16 ? p3 : p1;
        k0 += __shfl_xor_sync(0xffffffffu, up16 ? p0 : p2, 16);
        k1 += __shfl_xor_sync(0xffffffffu, up16 ? p1 : p3, 16);
        float kk = up8 ? k1 : k0;
        kk += __shfl_xor_sync(0xffffffffu, up8 ? k0 : k1, 8);
        const float val = oct_sum(kk) + Pm[PL.bv];
        float dv;
        bool vin = true;  // clip_range_vf: the clamp passes the gradient (torch's clamp backward: edges included)
        if (vf_on) {
          const float vold = row[col_logp + 1], dvo = val - vold;
          dv = (vold + fminf(fmaxf(dvo, -A.clip_vf), A.clip_vf)) - row[col_ret];
          vin = dvo >= -A.clip_vf && dvo <= A.clip_vf;
        } else {
          dv = val - row[col_ret];
        }
        const float dval = (live && vin) ? A.hp.vf_coef * 2.0f * dv * inv_nb : 0.f;
        if (la == 0) {
          if (live) l_v = dv * dv;
          DVAL[r0 + rr] = dval;
          RSL[RS_V * RL + r0 + rr] = live ? dv * dv : 0.f;
        }
        dl0 = __shfl_sync(0xffffffffu, dval, 0) * wvj;
        dl1 = __shfl_sync(0xffffffffu, dval, 8) * wvj;
        dl2 = __shfl_sync(0xffffffffu, dval, 16) * wvj;
        dl3 = __shfl_sync(0xffffffffu, dval, 24) * wvj;
      } else {
        const float* Wa = Pm + PL.wa;
        // action means / logits from the latent tile in shared memory: lane = (action ab + lane / 4, units q + 4 i of
        // quarter q = lane % 4): one 16-byte load brings a unit's four rows, so a weight and a latent load feed four FMAs
        // (one lane per (action, row) cost two loads per FMA: 64 loads per lane, ~700 cycles of the chain); the four
        // row sums are then reduced over the quad by a transposing butterfly (3 shuffles) that leaves row r0 + q in
        // lane q.  Pad units hold zeros; Wa rows have the odd stride ldh.
        __syncwarp();
        {
          const int asub = lane >> 2, q = lane & 3;
          const bool b0 = (lane & 1) != 0, b1 = (lane & 2) != 0;
#pragma unroll
          for (int ab = 0; ab < Da; ab += 8) {
            const int a = ab + asub, ac = a < Da ? a : 0;
            const float* wr = Wa + ac * ldh + q;
            const float* lr = cLAT + q * RL + r0;
            float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
            for (int i = 0; i < HP / 4; ++i) {
              const float w = wr[4 * i];
              const float4 l4 = ld4(lr + 4 * i * RL);
              s0 = fmaf(w, l4.x, s0);
              s1 = fmaf(w, l4.y, s1);
              s2 = fmaf(w, l4.z, s2);
              s3 = fmaf(w, l4.w, s3);
            }
            float ka = b0 ? s1 : s0, kb = b0 ? s3 : s2;
            ka += __shfl_xor_sync(0xffffffffu, b0 ? s0 : s1, 1);
            kb += __shfl_xor_sync(0xffffffffu, b0 ? s2 : s3, 1);
            float kk = b1 ? kb : ka;
            kk += __shfl_xor_sync(0xffffffffu, b1 ? ka : kb, 2);
            if (a < Da) MEAN[a * RL + r0 + q] = kk + Pm[PL.ba + a];
          }
        }
        __syncwarp();
        PPO_WCLK(5);
        const float adv = pre_adv, logp_old = pre_lpo;
        float logp = 0.f, ent = 0.f;
        float r_dm = 0.f, r_dls = 0.f;  // fast path: this lane's d logp / d mean, d logp / d log_std
        int act = 0;
        if (gfast) {
          if (la < Da) {
            const float diff = pre_act - MEAN[la * RL + r0 + rr];
            const float d2 = diff * diff * pre_ivar;
            logp = -0.5f * d2 - pre_ls - 0.9189385332046727f;
            ent = 1.4189385332046727f + pre_ls;
            r_dm = diff * pre_ivar;
            r_dls = d2 - 1.0f;
          }
        } else if (!discrete) {
          const float* lstd = Pm + PL.ls;
          for (int a = la; a < Da; a += 8) {
            const float ls = lstd[a], ivar = __expf(-2.0f * ls);
            const float diff = row[Do + a] - MEAN[a * RL + r0 + rr];
            const float d2 = diff * diff * ivar;
            logp += -0.5f * d2 - ls - 0.9189385332046727f;
            ent += 1.4189385332046727f + ls;
            DM[a * RL + r0 + rr] = diff * ivar;   // d logp / d mean
            DLS[a * RL + r0 + rr] = d2 - 1.0f;    // d logp / d log_std
          }
        } else {
          float mx = -INFINITY;
          for (int a = la; a < Da; a += 8) mx = fmaxf(mx, MEAN[a * RL + r0 + rr]);
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
          mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
          float se = 0.f;
          for (int a = la; a < Da; a += 8) se += expf(MEAN[a * RL + r0 + rr] - mx);
          const float lse = mx + logf(oct_sum(se));
          act = (int)row[Do];
          for (int a = la; a < Da; a += 8) {
            const float lp = MEAN[a * RL + r0 + rr] - lse;
            if (a == act) logp = lp;
            ent -= expf(lp) * lp;
            DLS[a * RL + r0 + rr] = lp;  // temporarily: log p_a
          }
        }
        logp = oct_sum(logp);
        PPO_WCLK(6);
        ent = oct_sum(ent);  // (Gaussian: the entropy only feeds the loss log and the statistics)
        const float ratio = __expf(logp - logp_old);
        const float lo = 1.0f - A.hp.clip_range, hi = 1.0f + A.hp.clip_range;
        const float pl1 = adv * ratio, pl2 = adv * fminf(fmaxf(ratio, lo), hi);
        const bool inside = (ratio >= lo) && (ratio <= hi);
        float dl_dlogp = (inside || pl1 < pl2) ? -adv * ratio * inv_nb : 0.f;
        float dent = -A.hp.ent_coef * inv_nb;  // d(ent_coef * ent_loss) / d(entropy)
        if (live) {
          if (la == 0) {
            l_pg = -fminf(pl1, pl2);
            l_ent = -ent;
          }
        } else {
          dl_dlogp = 0.f;
          dent = 0.f;
        }
        if (la == 0) {  // the row's statistics terms (written always: a condition here costs the chain a register)
          const int sr = r0 + rr;
          RSL[RS_PG * RL + sr] = live ? -fminf(pl1, pl2) : 0.f;
          RSL[RS_ENT * RL + sr] = live ? -ent : 0.f;
          RSL[RS_CLIP * RL + sr] = (live && fabsf(ratio - 1.0f) > A.hp.clip_range) ? 1.f : 0.f;
          RSL[RS_KL * RL + sr] = live ? (ratio - 1.0f) - (logp - logp_old) : 0.f;
        }
        if (gfast) {
          if (la < Da) {
            DLS[la * RL + r0 + rr] = dl_dlogp * r_dls + dent;  // dH/dlog_std = 1
            DM[la * RL + r0 + rr] = dl_dlogp * r_dm;
          }
        } else if (!discrete) {
          for (int a = la; a < Da; a += 8) {
            DLS[a * RL + r0 + rr] = dl_dlogp * DLS[a * RL + r0 + rr] + dent;  // dH/dlog_std = 1
            DM[a * RL + r0 + rr] = dl_dlogp * DM[a * RL + r0 + rr];
          }
        } else {
          for (int a = la; a < Da; a += 8) {
            const float lp = DLS[a * RL + r0 + rr], pp = expf(lp);
            DM[a * RL + r0 + rr] = dl_dlogp * (((a == act) ? 1.f : 0.f) - pp) + dent * (-pp * (lp + ent));
            DLS[a * RL + r0 + rr] = 0.f;
          }
        }
        __syncwarp();
        bar_arrive(BAR_PHEAD, 192);  // the head's gradients can start (warps 4-7)
        PPO_WCLK(7);
#pragma unroll U_DA
        for (int a = 0; a < Da; ++a) {
          const float waj = Wa[a * ldh + jc];
          const float4 d = ld4(DM + a * RL + r0);
          dl0 = fmaf(d.x, waj, dl0);
          dl1 = fmaf(d.y, waj, dl1);
          dl2 = fmaf(d.z, waj, dl2);
          dl3 = fmaf(d.w, waj, dl3);
        }
      }
      PPO_WCLK(2);
      // dL/dz2, backward through layer 2 (lane = input unit i: dH1[i] = sum_j DZ2[j] W2[j][i]), dL/dz1
      st4(cDZ2 + j * RL + r0,
          make_float4(jl ? dl0 * (1.0f - lat0 * lat0) : 0.f, jl ? dl1 * (1.0f - lat1 * lat1) : 0.f,
                      jl ? dl2 * (1.0f - lat2 * lat2) : 0.f, jl ? dl3 * (1.0f - lat3 * lat3) : 0.f));
      __syncwarp();
      bar_arrive(cnet ? BAR_VDZ2 : BAR_PDZ2, 192);  // the tower's layer-2 gradients can start (warps 4-7)
      a0 = a1 = a2 = a3 = 0.f;
      {
        const float* wp = cW2 + jc;
#pragma unroll U_H
        for (int jj = 0; jj < h; ++jj) {
          const float w = WREG ? w2c[jj] : wp[jj * ldh];
          const float4 d = ld4(cDZ2 + jj * RL + r0);
          a0 = fmaf(d.x, w, a0);
          a1 = fmaf(d.y, w, a1);
          a2 = fmaf(d.z, w, a2);
          a3 = fmaf(d.w, w, a3);
        }
      }
      st4(cDZ1 + j * RL + r0,
          make_float4(jl ? a0 * (1.f - h10 * h10) : 0.f, jl ? a1 * (1.f - h11 * h11) : 0.f,
                      jl ? a2 * (1.f - h12 * h12) : 0.f, jl ? a3 * (1.f - h13 * h13) : 0.f));
    }
    PPO_WCLK(0);
    // ---- 1c. weight gradients as their operands land, while warps 0, 1 are still in the policy chain: warps 4-7 (done
    //          with the prefetch, or with the statistics and the prefetch when those stay beside the chain) take the
    //          value tower's dW2 block, the policy head's and the policy tower's dW2 block, each as soon as the chain
    //          warps signal its tiles; warps 2, 3 take the value tower's dW1 block at the end of their own chain (each
    //          holds half of its rows).  Only the policy tower's dW1 block is left for after the chain.  The chain warps
    //          only arrive on these barriers, so they reach the loss log's CTA barriers below without waiting on a helper,
    //          and the tiles are not written again before the next step's top barrier. ----------------------------------------
    if (warp >= 4) {
      bar_sync(BAR_VDZ2, 192);
      wgrad_layer2<4, HP>(true, lane, warp - 4, h, PL.w2[1], PL.b2[1], ldh, PL.wv, PL.bv, GP, TH1 + HP * RL,
                          TLAT + HP * RL, TDZ2 + HP * RL, DVAL);
      PPO_WCLK(9);
      bar_sync(BAR_PHEAD, 192);
      wgrad_head<4, HP>(lane, warp - 4, h, Da, discrete, PL, GP, TLAT, DM, DLS);
      PPO_WCLK(7);
      bar_sync(BAR_PDZ2, 192);
      wgrad_layer2<4, HP>(false, lane, warp - 4, h, PL.w2[0], PL.b2[0], ldh, 0, 0, GP, TH1, TLAT, TDZ2, DVAL);
    } else if (warp >= 2) {
      bar_sync(BAR_VDZ1, 64);
      wgrad_layer1<2>(lane, warp - 2, h, Do, PL.w1[1], PL.b1[1], ldo, GP, TDZ1 + HP * RL, XNc);
      PPO_WCLK(9);
    }
    PPO_WCLK(8);
    // partial loss sums of this CTA -> CTA 0 (distributed shared memory)
    if (loss_log) {  // (uniform) loss terms are only reduced when the caller asked for the log
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
    __syncthreads();
    PPO_TICK(3);
    if (warp >= 2) PPO_WCLK(6);  // (slot 6 of the policy warps is taken by the chain)
    // ---- 2. the POLICY tower's dW1 block by all eight warps --------------------------------------------------------------
    wgrad_layer1<PT / 32>(lane, warp, h, Do, PL.w1[0], PL.b1[0], ldo, GP, TDZ1, XNc);
    __syncthreads();
    PPO_TICK(7);
    // ---- 3. push the partials to the PEER slice owners: RECV[this CTA][i], one 16-byte DSMEM store per quad ------------
    // CTA c starts with the quads owned by CTA c+1 and stops before its own slice (which its slice sum reads from GP),
    // so at any time the 8 senders target 8 different receivers
#pragma unroll
    for (int qb = 0; qb < (CL - 1) * (S / 4); qb += PT) {
      const int q = qb + tid;
      if (q >= (CL - 1) * (S / 4)) break;
      int qq = q + ((crank + 1) & (CL - 1)) * (S / 4);
      if (qq >= CL * S / 4) qq -= CL * S / 4;
      // owner = qq / (S / 4): a plain division when S is a compile-time constant
      const int p0 = 4 * qq, owner = SPEC ? qq / (S / 4) : (int)__umulhi((unsigned)qq, qmagic);
      st_async_v4(mapa_u32(recv_sa + (uint32_t)(crank * S + (p0 - owner * S)) * 4u, owner), ld4(GP + p0),
                  mapa_u32(xbar0_sa, owner));
    }
    if (loss_log) cluster.sync();  // (test / logging path only) the partial losses have landed in CTA 0
    if (crank == 0 && tid == 0 && loss_log) {
      float pg = 0.f, vl = 0.f, el = 0.f;
      for (int c = 0; c < CL; ++c) {
        pg += LOSS[c * 3 + 0];
        vl += LOSS[c * 3 + 1];
        el += LOSS[c * 3 + 2];
      }
      pg *= inv_nb, vl *= inv_nb, el *= inv_nb;
      loss_log[gs * 4 + 0] = pg;
      loss_log[gs * 4 + 1] = vl;
      loss_log[gs * 4 + 2] = el;
      loss_log[gs * 4 + 3] = pg + A.hp.ent_coef * el + A.hp.vf_coef * vl;
    }
    PPO_TICK(8);
    // the statistics fold: on warp 3 when it idles through the tail (neither slice owner nor statistics warp: small
    // policies, whose short tail the statistics warps' work nearly fills), else on the last warp
    if (A.stats && warp == ((tail_stats && n_own_w < 4) ? 3 : PT / 32 - 1))
      ppo_stats_fold_warp(ACC, RSL, rcp_fast((float)min(mb, Ni - start)), start == 0, threadIdx.x & 31);
    // (1 / nb recomputed here: keeping the step's live through the chain until the tail costs the chain a spill)
    if (tail_stats && tid >= st0) {
      // ---- 4a. the statistics threads own no slice quad: they run the next step's statistics while the owners finish
      //          the step.  They skip the exchange waits (they read none of RECV, SSQ or the new parameters before the
      //          next step's top barrier, which the owners reach only after those waits).
      next_stats();
    } else {
      // wait until the 7 peer partials of the owned slice have landed
      mbar_wait(&xbar[0], (uint32_t)(gs & 1));
      if (tid == 0) mbar_expect_tx(&xbar[0], xbytes);  // re-arm for the next step
      PPO_TICK(9);

      // ---- 4. slice owners: sum the CL partials in fixed order (one quad per thread), exchange the squared slice
      //         norms for clip_grad_norm_ (4 bytes to every CTA, same st.async + mbarrier mechanism) ------------------------
      const int i0 = 4 * tid;
      const bool own = i0 < S;  // S / 4 <= PT is checked by the launcher
      float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
      float ss = 0.f;
      if (own) {
        // CTA c's partial of the slice: RECV[c], or this CTA's own straight from GP
        auto part = [&](int c) { return ld4(c == crank ? GP + crank * S + i0 : RECV + c * S + i0); };
        g = part(0);
  #pragma unroll
        for (int c = 1; c < CL; ++c) {  // fixed order: deterministic
          const float4 t = part(c);
          g.x += t.x, g.y += t.y, g.z += t.z, g.w += t.w;
        }
        ss = (g.x * g.x + g.y * g.y) + (g.z * g.z + g.w * g.w);
      }
      // squared norm of the slice: warp sums, then the warps' in warp order, over the owner warps only (a named barrier;
      // the other warps' terms are +0.0 and are still added, so the sum is the full-CTA reduction's bit for bit)
      float my_ssq = 0.f;
      if (warp < n_own_w) {
        const float ws = warp_sum(ss);
        if (lane == 0) nred[warp] = ws;
        asm volatile("bar.sync 2, %0;" ::"r"(32 * n_own_w) : "memory");
  #pragma unroll
        for (int w = 0; w < PT / 32; ++w) my_ssq += w < n_own_w ? nred[w] : 0.f;
      }
      if (tid < CL) {
        st_async_f32(mapa_u32(ssq_sa + (uint32_t)crank * 4u, tid), my_ssq, mapa_u32(xbar2_sa, tid));
        if (kl_on)
          st_async_f32(mapa_u32(smem_u32(KLS) + (uint32_t)crank * 4u, tid), ppo_kl_part<RL>(RSL, inv_nb),
                       mapa_u32(xbar2_sa, tid));
      }
      PPO_TICK(10);
      mbar_wait(&xbar[2], (uint32_t)(gs & 1));
      if (tid == 0) mbar_expect_tx(&xbar[2], nbytes);  // re-arm for the next step
      PPO_TICK(11);
      bool stop = false;
      if (kl_on) {
        // target_kl (SB3: approx_kl > 1.5 target_kl): the CL shares summed in the same order everywhere, so every CTA
        // reaches the same decision; a stopping step takes no Adam step (nothing is all-gathered, nobody waits for
        // it), and all CTAs leave at the next step's top barrier
        float kl = 0.f;
#pragma unroll
        for (int c = 0; c < CL; ++c) kl += KLS[c];
        stop = kl > 1.5f * A.target_kl;
        if (stop && tid == 0) KSTOP = (int)gs + 1;
      }

      // ---- 5. clip_grad_norm_ + Adam on the OWNED slice (moments never leave their owner); the new parameters are
      //         all-gathered into every CTA's parameter vector ----------------------------------------------------------
      float total = 0.f;
  #pragma unroll
      for (int c = 0; c < CL; ++c) total += SSQ[c];  // same order everywhere: the replicas' clip factors agree bit for bit
      total = sqrtf(total);
      float clip = A.hp.max_grad_norm / (total + 1e-6f);
      clip = clip > 1.0f ? 1.0f : clip;
      if (own && !stop) {
        const float step_size = bc[2 * cur], inv_bc2s = rcp_fast(bc[2 * cur + 1]);
        const int q0 = crank * S + i0;
        const float4 m4 = ld4(Ms + q0), v4 = ld4(Vs + q0), p4 = ld4(Pm + q0);
        // approximate sqrt / division (~1e-7 relative on an update that is itself ~lr relative to the weights)
        auto adam1 = [&](float gg, float& m, float& v, float& pw) {
          gg *= clip;
          m = m + (gg - m) * (1.0f - 0.9f);
          v = v * 0.999f + (1.0f - 0.999f) * gg * gg;
          pw -= step_size * __fdividef(m, fmaf(sqrt_fast(v), inv_bc2s, A.hp.adam_eps));
        };
        float4 m = m4, v = v4, pw = p4;
        adam1(g.x, m.x, v.x, pw.x);
        adam1(g.y, m.y, v.y, pw.y);
        adam1(g.z, m.z, v.z, pw.z);
        adam1(g.w, m.w, v.w, pw.w);
        st4(Ms + q0, m);
        st4(Vs + q0, v);
        st4(Pm + q0, pw);
  #pragma unroll
        for (int c = 1; c < CL; ++c) {  // rotated start: the 8 owners write to 8 different CTAs at a time
          const int dstc = (crank + c) & (CL - 1);
          st_async_v4(mapa_u32(pm_sa + (uint32_t)q0 * 4u, dstc), pw, mapa_u32(xbar1_sa, dstc));
        }
      }
      if (!stop) {
        mbar_wait(&xbar[1], (uint32_t)(gs & 1));  // every CTA's new parameter slice has landed in Pm
        if (tid == 0) mbar_expect_tx(&xbar[1], xbytes);  // re-arm for the next step
      }
      PPO_TICK(12);
    }
    if (has_norm && gs + 1 < n_steps) run_count += min(mb, Ni - start_next);  // (after the statistics that read it)
    ep_now = ep_next;
    start = start_next;
    // (the barrier at the top of the next step orders these parameter writes before their first use)
  }
  __syncthreads();
#ifdef IMB_PPO_TIMING
  if (crank == 0 && tid == 0)
    for (int i = 0; i < 16; ++i) g_ppo_clk[i] = clk_acc[i];
  if (crank == 0 && lane == 0)
    for (int i = 0; i < 10; ++i) g_ppo_wclk[i * 8 + warp] = wacc[i];
#endif

  // ---- write back (CTA 0): parameters and moments in torch order, norm state, counters ------------------------------
  for (int p = tid; p < NP; p += PT) {  // moments live with their slice owner
    const int q = flat_to_play(pd, PL, p);
    if (q / S == crank) {
      g_m[p] = Ms[q];
      g_v[p] = Vs[q];
    }
  }
  // target_kl stop at step KSTOP - 1: Adam steps taken = KSTOP - 1, epochs begun = the stopped step's epoch + 1; when a
  // later step's statistics were computed ahead, rstat has moved on and g_norm already holds the stopped step's
  const int kstop = kl_on ? KSTOP : 0;
  if (crank == 0) {
    for (int p = tid; p < NP; p += PT) g_params[p] = Pm[flat_to_play(pd, PL, p)];
    if (has_norm) {
      if (tid < Do && !(kstop && kstop < n_steps)) {
        g_norm[tid] = rstat[tid];
        g_norm[Do + tid] = rstat[64 + tid];
      }
      if (tid == 0) *g_norm_count = run_count;
    }
    if (tid == 0) {
      state[IMB_ST_PPO_STEP] = kstop ? state[IMB_ST_PPO_STEP] + (kstop - 1) : adam_step;
      state[IMB_ST_PPO_EPOCH] = perm_draw0 + (kstop ? (kstop - 1) / steps_per_epoch + 1 : A.hp.n_epochs);
    }
  }
  if (A.stats) {
    if (tid == 0) ppo_stats_push(cluster, TH1, ACC, EVP, crank);  // (the chain's tiles are free now)
    cluster.sync();
    if (crank == 0 && tid == 0) {
      float sd = __int_as_float(0x7fc00000);
      if (!discrete) {
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

// ---- log pi(a|s) for the AIRL discriminator batch --------------------------------------------------------------
// The pi tower of the policy's PolImg (staged in shared memory) on the inputs x[0, Do): lat = its last hidden layer.
// ACT: the towers' activation (ACT_TANH: tanhf, ACT_RELU: fmaxf(z, 0)).
template <int HP, int ACT>
__device__ __forceinline__ void policy_tower(const float* __restrict__ smem, const PolImg& S, int Do,
                                             const float* __restrict__ x, float (&lat)[HP]) {
  const float* w1t = smem + S.w1p;
  const float* w2t = smem + S.w2p;
  float h1[HP];
#pragma unroll
  for (int j = 0; j < HP; ++j) h1[j] = smem[S.b1p + j];
  for (int k = 0; k < Do; ++k) {
    const float xv = x[k];
#pragma unroll
    for (int j = 0; j < HP; ++j) h1[j] = fmaf(w1t[k * HP + j], xv, h1[j]);
  }
#pragma unroll
  for (int j = 0; j < HP; ++j) {
    h1[j] = ACT == ACT_TANH ? tanhf(h1[j]) : fmaxf(h1[j], 0.f);
    lat[j] = smem[S.b2p + j];
  }
#pragma unroll
  for (int i = 0; i < HP; ++i) {
    const float hv = h1[i];
#pragma unroll
    for (int j = 0; j < HP; ++j) lat[j] = fmaf(w2t[i * HP + j], hv, lat[j]);
  }
#pragma unroll
  for (int j = 0; j < HP; ++j) lat[j] = ACT == ACT_TANH ? tanhf(lat[j]) : fmaxf(lat[j], 0.f);
}

// thread per batch column; obs rows [0,Do), act rows [Do, Do+Da_onehot) of the feature-major batch.  The pi tower, the
// action head and log_std come from the policy's PolImg; then xn_ld >= Do inputs per thread.
template <int HP, int ACT>
__global__ void __launch_bounds__(128) k_policy_logp(const imb_policy_desc pd, const float* __restrict__ params,
                                                    const float* __restrict__ norm, float* __restrict__ batch,
                                                    int64_t ld, int64_t n, int row_logp, int xn_off, int xn_ld) {
  extern __shared__ __align__(128) float smem[];
  const int Do = pd.d_obs, Da = pd.d_act, h = pd.hidden;
  const PolImg S(Do, Da, HP);
  const int tid = threadIdx.x;
  load_policy_img(smem, S, pd, HP, params, norm);
  __syncthreads();
  const float* wa = smem + S.wa;
  float* x = smem + xn_off + tid * xn_ld;
  for (int64_t col = (int64_t)blockIdx.x * blockDim.x + tid; col < n; col += (int64_t)gridDim.x * blockDim.x) {
    for (int k = 0; k < Do; ++k) {
      float v = batch[(int64_t)k * ld + col];
      if (pd.has_norm) v = (v - norm[k]) / sqrtf(norm[Do + k] + pd.norm_eps);
      x[k] = v;
    }
    float lat[HP];
    policy_tower<HP, ACT>(smem, S, Do, x, lat);
    float logp = 0.f;
    if (!pd.discrete) {
      for (int a = 0; a < Da; ++a) {
        float m = smem[S.ba + a];
#pragma unroll
        for (int j = 0; j < HP; ++j) m = (j < h) ? fmaf(wa[a * HP + j], lat[j], m) : m;
        const float ls = smem[S.lstd + a], sd = expf(ls);
        const float diff = batch[(int64_t)(Do + a) * ld + col] - m;
        logp += -(diff * diff) / (2.0f * sd * sd) - ls - 0.9189385332046727f;
      }
    } else {
      float mx = -INFINITY, chosen = 0.f;
      float lg[IMB_MAX_DIN];
      for (int a = 0; a < Da; ++a) {
        float m = smem[S.ba + a];
#pragma unroll
        for (int j = 0; j < HP; ++j) m = (j < h) ? fmaf(wa[a * HP + j], lat[j], m) : m;
        lg[a] = m;
        mx = fmaxf(mx, m);
        if (batch[(int64_t)(Do + a) * ld + col] > 0.5f) chosen = m;  // one-hot action rows
      }
      float se = 0.f;
      for (int a = 0; a < Da; ++a) se += expf(lg[a] - mx);
      logp = chosen - (mx + logf(se));
    }
    batch[(int64_t)row_logp * ld + col] = logp;
  }
}

// ---- DQN TD targets (imb_dqn_target) ----------------------------------------------------------------------------
// The max-over-head output mode of the policy forward above, on the target Q-net: thread per TD row r = gs * B + i of
// n_steps minibatches of B = n_l + n_e rows (learner rows first).  Row i < n_l reads column ring_idx[gs * n_l + i] of
// the feature-major learner ring, the others column exp_idx[gs * n_e + i - n_l] of the expert table (both [tw][ld]
// transition tables, Discrete actions one-hot).  y = r + ((1 - done) * gamma) * max_a Q_target(s')[a], each operation
// rounded as torch rounds DQN.train's expression; the row written is obs | action index | y (rollout-row format).
template <int HP, int ACT>
__global__ void __launch_bounds__(128) k_dqn_target(const imb_policy_desc pd, const float* __restrict__ params,
                                                   const float* __restrict__ ring, int64_t ring_ld,
                                                   const int64_t* __restrict__ ring_idx, const float* __restrict__ expert,
                                                   int64_t exp_ld, const int64_t* __restrict__ exp_idx, int64_t n_l,
                                                   int64_t n_e, int64_t n, float gamma, float rew_l, float rew_e,
                                                   float* __restrict__ out, int rw, int xn_off, int xn_ld,
                                                   int64_t step_base, const int64_t* __restrict__ state) {
  extern __shared__ __align__(128) float smem[];
  const int Do = pd.d_obs, Da = pd.d_act, h = pd.hidden;
  const PolImg S(Do, Da, HP);
  const int tid = threadIdx.x;
  load_policy_img(smem, S, pd, HP, params, nullptr);
  __syncthreads();
  const float* wa = smem + S.wa;
  float* x = smem + xn_off + tid * xn_ld;
  const int64_t B = n_l + n_e;
  const int64_t s0 = state ? state[IMB_ST_PPO_STEP] - step_base : 0;  // TD steps of the sample lists already taken
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + tid; r < n; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t gs = r / B + s0, i = r - (r / B) * B;
    const bool learner = i < n_l;
    const float* src = learner ? ring : expert;
    const int64_t ld = learner ? ring_ld : exp_ld;
    const int64_t col = learner ? ring_idx[gs * n_l + i] : exp_idx[gs * n_e + (i - n_l)];
    for (int k = 0; k < Do; ++k) x[k] = src[(int64_t)(Do + Da + k) * ld + col];
    float lat[HP];
    policy_tower<HP, ACT>(smem, S, Do, x, lat);
    float mx = -INFINITY;
    int act = 0;
    for (int a = 0; a < Da; ++a) {
      float m = smem[S.ba + a];
#pragma unroll
      for (int j = 0; j < HP; ++j) m = (j < h) ? fmaf(wa[a * HP + j], lat[j], m) : m;
      mx = fmaxf(mx, m);
      if (src[(int64_t)(Do + a) * ld + col] > 0.5f) act = a;
    }
    const float done = src[(int64_t)(2 * Do + Da) * ld + col];
    const float y = __fadd_rn(learner ? rew_l : rew_e, __fmul_rn(__fmul_rn(1.0f - done, gamma), mx));
    float* o = out + r * rw;
    for (int k = 0; k < Do; ++k) o[k] = src[(int64_t)k * ld + col];
    o[Do] = (float)act;
    o[Do + 1] = y;
  }
}

#include "imb_ppo_gen.cuh"

}  // namespace

static size_t ppo_smem_floats(const PpoArgs& A) {
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const int HP = A.HP, KP = A.KP, Da = A.pol.d_act, S = A.S;
  const int DAP = (Da + 3) / 4 * 4;
  size_t o = 0;
  o += 5 * (size_t)al(CL * S) + 32;
  o += 3 * (size_t)al(PR * A.RS2);
  o += 2 * (size_t)al(KP * RL) + (size_t)8 * HP * RL + (size_t)3 * DAP * RL + 32;
  o += al(2 * 64 + 4);
  return o;
}

// cluster launch of one of the two PPO kernels (CL CTAs of PT threads, one cluster); `extra`: k_ppo_update_gen's BcArgs
template <typename K, typename... Extra>
static int launch_cluster(K kernel, const char* name, size_t smem_bytes, size_t* attr_bytes, cudaStream_t st, const PpoArgs& A,
                          float* params, float* norm, int32_t* norm_count, float* m, float* v, const float* rollout,
                          const int64_t* perm, float* loss_log, int64_t* state, Extra... extra) {
  IMB_REQUIRE(smem_bytes <= IMB_SMEM_MAX, "%s needs %zu B of shared memory per CTA (policy / minibatch too large)", name,
              smem_bytes);
  if (smem_bytes > *attr_bytes) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute(%s): %s", name, cudaGetErrorString(e));
    *attr_bytes = smem_bytes;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(CL);
  cfg.blockDim = dim3(PT);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, A, params, norm, norm_count, m, v, rollout, perm, loss_log, state,
                                     extra...);
  if (e != cudaSuccess) IMB_FAIL(-2, "%s (cluster launch): %s", name, cudaGetErrorString(e));
  return 0;
}

extern "C" int imb_rollout_row_width(const imb_policy_desc* pol);

// The shape checks and launch geometry (rw, KP, S, RS2) every PPO kernel shares; `what` names the caller's update.
static int ppo_plan_shape(PpoArgs& A, int act, const char* what) {
  const imb_policy_desc& pd = A.pol;
  IMB_REQUIRE(act == IMB_ACT_TANH || act == IMB_ACT_RELU,
              "pol_act must be IMB_ACT_TANH (0) or IMB_ACT_RELU (1), got %d", act);
  IMB_REQUIRE(pd.hidden >= 1 && pd.hidden <= 64, "policy tower width must be <= 64");
  IMB_REQUIRE(pd.d_obs >= 1 && pd.d_obs <= IMB_MAX_DIN && pd.d_act >= 1 && pd.d_act <= IMB_MAX_DIN,
              "d_obs/d_act must be in [1, %d]", IMB_MAX_DIN);
  IMB_REQUIRE(A.hp.batch_size >= 1 && A.hp.batch_size <= GEN_MAX_MB, "%s minibatch size must be in [1, %d]", what,
              GEN_MAX_MB);
  A.rw = imb_rollout_row_width(&pd);
  IMB_REQUIRE(A.rw % 4 == 0, "rollout row width must be a multiple of 4 floats (bulk row copies)");
  A.KP = ppo_kp(pd.d_obs);
  A.S = ppo_slice(make_play(pd));
  A.RS2 = ppo_row_stride(A.rw);
  return 0;
}

// k_ppo_update_gen's plan: U = 1 or 2 hidden units per lane (IMB_PPO_PLAN_GEN1 / GEN2), HP into A, its dynamic shared
// memory into *bytes; < 0 naming the need and the limit when it does not fit.
static int gen_plan(PpoArgs& A, size_t* bytes, const char* what) {
  A.HP = A.pol.hidden <= 32 ? 32 : 64;
  *bytes = (size_t)gen_layout(A.S, A.HP, A.KP, A.pol.d_act, A.hp.batch_size).total * 4;
  IMB_REQUIRE(*bytes <= IMB_SMEM_MAX, "policy / minibatch too large for the %s update: k_ppo_update_gen<%d> needs %zu B "
              "of shared memory per CTA, the limit is %d B", what, A.HP / 32, *bytes, (int)IMB_SMEM_MAX);
  return A.HP == 32 ? IMB_PPO_PLAN_GEN1 : IMB_PPO_PLAN_GEN2;
}

// Which PPO kernel runs the policy A.pol at minibatch A.hp.batch_size (the IMB_PPO_PLAN_* codes of imb_ppo_plan), with
// the launch geometry (rw, KP, S, RS2, HP) filled into A and the dynamic shared memory into *bytes.  k_ppo_update
// (64-row minibatch resident in shared memory, one lane per hidden unit) for tower width <= 32 and minibatches <= 64
// rows when its shared memory and slice fit; else k_ppo_update_gen with U = 1 or 2 hidden units per lane.  ReLU towers
// (act = IMB_ACT_RELU) always run k_ppo_update_gen: k_ppo_update is built for the tanh policies bench.py trains.
static int ppo_plan(PpoArgs& A, int act, size_t* bytes) {
  const imb_policy_desc& pd = A.pol;
  const int rc = ppo_plan_shape(A, act, "PPO");
  if (rc != 0) return rc;
  // IMB_PPO_FORCE_GENERAL=1 (tests): run the general kernel on shapes the specialised one covers
  const char* force = getenv("IMB_PPO_FORCE_GENERAL");
  if (act == IMB_ACT_TANH && pd.hidden <= 32 && A.hp.batch_size <= PR && !(force && force[0] == '1')) {
    A.HP = 32;
    *bytes = ppo_smem_floats(A) * 4;
    if (A.S / 4 <= PT && *bytes <= IMB_SMEM_MAX) return IMB_PPO_PLAN_UPDATE;
  }
  return gen_plan(A, bytes, "PPO");
}

// The BC update runs k_ppo_update_gen<U, act, LOSS_BC> for every shape (the specialised k_ppo_update has no BC loss).
static int bc_plan(PpoArgs& A, int act, size_t* bytes) {
  const int rc = ppo_plan_shape(A, act, "BC");
  return rc != 0 ? rc : gen_plan(A, bytes, "BC");
}

extern "C" int imb_ppo_plan(const imb_policy_desc* pol, int32_t pol_act, int32_t batch_size) {
  PpoArgs A = {};
  A.pol = *pol;
  A.hp.batch_size = batch_size;
  size_t bytes;
  return ppo_plan(A, pol_act, &bytes);
}

// The policy shapes with their own instantiation of k_ppo_update (tower width 32): the policies bench.py trains.
// Entry i is instantiation i + 1 of imb_ppo_update_variant.
struct PpoShape {
  int d_obs, d_act, discrete, has_norm;
};
constexpr PpoShape kPpoShapes[] = {
    {17, 6, 0, 1},  // HalfCheetah-shaped Box with NormalizeFeaturesExtractor (GAIL and AIRL)
    {27, 8, 0, 1},  // Ant-shaped Box with NormalizeFeaturesExtractor
    {4, 2, 1, 0},   // CartPole-shaped Discrete
};
template <int I, int OPT>
constexpr auto k_ppo_update_spec =
    k_ppo_update<32, kPpoShapes[I].d_obs, kPpoShapes[I].d_act, kPpoShapes[I].discrete, kPpoShapes[I].has_norm, OPT>;
constexpr decltype(&k_ppo_update<32>) kPpoUpdateKernels[] = {k_ppo_update<32>, k_ppo_update_spec<0, 0>,
                                                            k_ppo_update_spec<1, 0>, k_ppo_update_spec<2, 0>};
// With target_kl or clip_range_vf on, every shape runs the runtime-shape instantiation with their code compiled in
// (OPT = 1): the shape-specialised ones sit at 254-255 registers, and the options' code makes the Ant-shaped one spill.
// The arithmetic is the same bit for bit in every instantiation.
constexpr auto kPpoUpdateOptKernel = k_ppo_update<32, 0, 0, 0, 0, 1>;
constexpr const char* kPpoUpdateNames[] = {"k_ppo_update", "k_ppo_update<17x6 Box, norm>", "k_ppo_update<27x8 Box, norm>",
                                           "k_ppo_update<4x2 Discrete>"};
constexpr int kNumPpoVariants = sizeof(kPpoUpdateKernels) / sizeof(kPpoUpdateKernels[0]);

// Which instantiation of k_ppo_update runs `pd` (when it runs k_ppo_update at all): 1 + its index in kPpoShapes, or 0
// for the runtime-shape one.  IMB_PPO_FORCE_RUNTIME_SHAPE=1 (tests), read at every call, forces 0.
static int ppo_variant(const imb_policy_desc& pd) {
  const char* force = getenv("IMB_PPO_FORCE_RUNTIME_SHAPE");
  if ((force && force[0] == '1') || pd.hidden != 32) return 0;
  for (int i = 0; i < kNumPpoVariants - 1; ++i) {
    const PpoShape& s = kPpoShapes[i];
    if (pd.d_obs == s.d_obs && pd.d_act == s.d_act && (pd.discrete != 0) == (s.discrete != 0) &&
        (pd.has_norm != 0) == (s.has_norm != 0))
      return i + 1;
  }
  return 0;
}

extern "C" int imb_ppo_update_variant(const imb_policy_desc* pol) { return ppo_variant(*pol); }

static int launch_ppo(const PpoArgs& A0, int act, float* params, float* norm, int32_t* norm_count, float* m, float* v,
                      const float* rollout, const int64_t* perm, float* loss_log, int64_t* state, cudaStream_t st) {
  PpoArgs A = A0;
  size_t bytes;
  const int plan = ppo_plan(A, act, &bytes);
  if (plan == IMB_PPO_PLAN_UPDATE) {
    static size_t attr_bytes[kNumPpoVariants + 1] = {};
    if (A.target_kl > 0.f || A.clip_vf > 0.f)
      return launch_cluster(kPpoUpdateOptKernel, "k_ppo_update<target_kl / clip_range_vf>", bytes,
                            &attr_bytes[kNumPpoVariants], st, A, params, norm, norm_count, m, v, rollout, perm, loss_log,
                            state);
    const int var = ppo_variant(A.pol);
    return launch_cluster(kPpoUpdateKernels[var], kPpoUpdateNames[var], bytes, &attr_bytes[var], st, A, params, norm,
                          norm_count, m, v, rollout, perm, loss_log, state);
  }
  if (plan == IMB_PPO_PLAN_GEN1 || plan == IMB_PPO_PLAN_GEN2) {
    // [U - 1][act]: k_ppo_update_gen<U, act>
    static size_t attr_bytes[2][2] = {};
    constexpr decltype(&k_ppo_update_gen<1, ACT_TANH>) kernels[2][2] = {
        {k_ppo_update_gen<1, ACT_TANH>, k_ppo_update_gen<1, ACT_RELU>},
        {k_ppo_update_gen<2, ACT_TANH>, k_ppo_update_gen<2, ACT_RELU>}};
    constexpr const char* names[2][2] = {{"k_ppo_update_gen<1>", "k_ppo_update_gen<1, relu>"},
                                         {"k_ppo_update_gen<2>", "k_ppo_update_gen<2, relu>"}};
    const int u = plan == IMB_PPO_PLAN_GEN1 ? 0 : 1;
    return launch_cluster(kernels[u][act], names[u][act], bytes, &attr_bytes[u][act], st, A, params, norm, norm_count, m,
                          v, rollout, perm, loss_log, state, BcArgs{});
  }
  return plan;
}

extern "C" int imb_ppo_update_ex(const imb_policy_desc* pol, int32_t pol_act, float* pol_params, float* pol_norm,
                                 int32_t* pol_norm_count, float* exp_avg, float* exp_avg_sq, const float* rollout,
                                 int64_t n_rows, const imb_ppo_hparams* hp, float target_kl, float clip_range_vf,
                                 const int64_t* perm, uint64_t seed, float* loss_log, float* stats_out, int64_t* state,
                                 void* stream) {
  IMB_REQUIRE(n_rows >= 1 && n_rows < (1ll << 31), "bad n_rows");
  PpoArgs A;
  A.pol = *pol;
  A.hp = *hp;
  A.n_rows = n_rows;
  A.seed = seed;
  A.target_kl = target_kl > 0.f ? target_kl : 0.f;
  A.clip_vf = clip_range_vf > 0.f ? clip_range_vf : 0.f;
  A.stats = stats_out;
  return launch_ppo(A, pol_act, pol_params, pol_norm, pol_norm_count, exp_avg, exp_avg_sq, rollout, perm, loss_log, state,
                    (cudaStream_t)stream);
}

extern "C" int imb_ppo_update(const imb_policy_desc* pol, int32_t pol_act, float* pol_params, float* pol_norm,
                              int32_t* pol_norm_count, float* exp_avg, float* exp_avg_sq, const float* rollout,
                              int64_t n_rows, const imb_ppo_hparams* hp, const int64_t* perm, uint64_t seed,
                              float* loss_log, int64_t* state, void* stream) {
  return imb_ppo_update_ex(pol, pol_act, pol_params, pol_norm, pol_norm_count, exp_avg, exp_avg_sq, rollout, n_rows, hp,
                           0.f, 0.f, perm, seed, loss_log, nullptr, state, stream);
}

extern "C" int imb_bc_plan(const imb_policy_desc* pol, int32_t pol_act, int32_t minibatch_size) {
  PpoArgs A = {};
  A.pol = *pol;
  A.hp.batch_size = minibatch_size;
  size_t bytes;
  return bc_plan(A, pol_act, &bytes);
}

extern "C" int imb_bc_train(const imb_policy_desc* pol, int32_t pol_act, float* pol_params, float* pol_norm,
                            int32_t* pol_norm_count, float* exp_avg, float* exp_avg_sq, const float* table,
                            int64_t n_rows, int32_t minibatch_size, int32_t batch_size, int64_t j0,
                            int64_t n_minibatches, int32_t final_flush, float l2_weight, float ent_weight, float lr,
                            float adam_eps, int32_t norm_update, const int64_t* perm, float* grad_carry, float* metrics,
                            int32_t log_interval, int64_t* state, void* stream) {
  IMB_REQUIRE(n_rows >= 1 && n_rows < (1ll << 31), "bad n_rows");
  IMB_REQUIRE(minibatch_size >= 1 && n_rows >= minibatch_size, "BC needs at least minibatch_size (%d) demonstration "
              "rows, got %lld", minibatch_size, (long long)n_rows);
  IMB_REQUIRE(batch_size >= minibatch_size && batch_size % minibatch_size == 0,
              "batch_size (%d) must be a multiple of minibatch_size (%d)", batch_size, minibatch_size);
  IMB_REQUIRE(j0 >= 0 && n_minibatches >= 0, "bad minibatch range");
  IMB_REQUIRE(final_flush >= 0 && final_flush <= 2, "final_flush must be 0, 1 or 2");
  IMB_REQUIRE(n_minibatches > 0 || final_flush != 1 || j0 % (batch_size / minibatch_size) != 0,
              "a flush-only launch (n_minibatches = 0) needs an incomplete batch to step");
  IMB_REQUIRE(perm != nullptr || n_minibatches == 0, "perm is required");
  IMB_REQUIRE(log_interval >= 1 || metrics == nullptr, "log_interval must be >= 1");
  const int k = batch_size / minibatch_size;
  IMB_REQUIRE(grad_carry != nullptr || (k == 1), "grad_carry is required when batch_size > minibatch_size");
  if (n_minibatches == 0 && final_flush != 1) return 0;
  PpoArgs A = {};
  A.pol = *pol;
  A.hp.batch_size = minibatch_size;
  A.hp.ent_coef = ent_weight;
  A.hp.lr = lr;
  A.hp.adam_eps = adam_eps;
  A.n_rows = n_rows;
  size_t bytes;
  const int plan = bc_plan(A, pol_act, &bytes);
  if (plan < 0) return plan;
  BcArgs B = {};
  B.j0 = j0;
  B.n_mb = n_minibatches;
  B.k = k;
  B.final_flush = final_flush;
  B.norm_update = norm_update != 0;
  B.log_interval = log_interval >= 1 ? log_interval : 1;
  B.l2_weight = l2_weight;
  B.inv_bs = 1.0f / (float)batch_size;
  B.carry = grad_carry;
  B.metrics = metrics;
  static size_t attr_bytes[2][2] = {};
  constexpr decltype(&k_ppo_update_gen<1, ACT_TANH, LOSS_BC>) kernels[2][2] = {
      {k_ppo_update_gen<1, ACT_TANH, LOSS_BC>, k_ppo_update_gen<1, ACT_RELU, LOSS_BC>},
      {k_ppo_update_gen<2, ACT_TANH, LOSS_BC>, k_ppo_update_gen<2, ACT_RELU, LOSS_BC>}};
  constexpr const char* names[2][2] = {{"k_ppo_update_gen<1, bc>", "k_ppo_update_gen<1, relu, bc>"},
                                       {"k_ppo_update_gen<2, bc>", "k_ppo_update_gen<2, relu, bc>"}};
  const int u = plan == IMB_PPO_PLAN_GEN1 ? 0 : 1;
  return launch_cluster(kernels[u][pol_act], names[u][pol_act], bytes, &attr_bytes[u][pol_act], (cudaStream_t)stream, A,
                        pol_params, pol_norm, pol_norm_count, exp_avg, exp_avg_sq, table, perm, nullptr, state, B);
}

extern "C" int imb_dqn_plan(const imb_policy_desc* pol, int32_t pol_act, int32_t batch_size) {
  IMB_REQUIRE(pol->discrete, "the DQN step runs Discrete action spaces only");
  IMB_REQUIRE(!pol->has_norm, "the DQN step runs Q-nets without a feature RunningNorm");
  PpoArgs A = {};
  A.pol = *pol;
  A.hp.batch_size = batch_size;
  size_t bytes;
  const int rc = ppo_plan_shape(A, pol_act, "DQN");
  return rc != 0 ? rc : gen_plan(A, &bytes, "DQN");
}

extern "C" int imb_dqn_step(const imb_policy_desc* pol, int32_t pol_act, float* q_params, float* exp_avg,
                            float* exp_avg_sq, const float* rows, int32_t batch_size, int64_t n_steps, float lr,
                            float adam_eps, float max_grad_norm, float* loss_log, int64_t loss_base, int64_t* state,
                            void* stream) {
  IMB_REQUIRE(n_steps >= 0 && n_steps * (int64_t)batch_size < (1ll << 31), "bad n_steps");
  if (n_steps == 0) return 0;
  PpoArgs A = {};
  A.pol = *pol;
  A.hp.batch_size = batch_size;
  A.hp.n_epochs = 1;
  A.hp.lr = lr;
  A.hp.adam_eps = adam_eps;
  A.hp.max_grad_norm = max_grad_norm;
  A.n_rows = n_steps * batch_size;
  const int plan = imb_dqn_plan(pol, pol_act, batch_size);
  if (plan < 0) return plan;
  size_t bytes;
  ppo_plan_shape(A, pol_act, "DQN");
  gen_plan(A, &bytes, "DQN");
  static size_t attr_bytes[2][2] = {};
  constexpr decltype(&k_ppo_update_gen<1, ACT_TANH, LOSS_DQN>) kernels[2][2] = {
      {k_ppo_update_gen<1, ACT_TANH, LOSS_DQN>, k_ppo_update_gen<1, ACT_RELU, LOSS_DQN>},
      {k_ppo_update_gen<2, ACT_TANH, LOSS_DQN>, k_ppo_update_gen<2, ACT_RELU, LOSS_DQN>}};
  constexpr const char* names[2][2] = {{"k_ppo_update_gen<1, dqn>", "k_ppo_update_gen<1, relu, dqn>"},
                                       {"k_ppo_update_gen<2, dqn>", "k_ppo_update_gen<2, relu, dqn>"}};
  const int u = plan == IMB_PPO_PLAN_GEN1 ? 0 : 1;
  BcArgs B = {};
  B.j0 = loss_base;
  return launch_cluster(kernels[u][pol_act], names[u][pol_act], bytes, &attr_bytes[u][pol_act], (cudaStream_t)stream, A,
                        q_params, nullptr, nullptr, exp_avg, exp_avg_sq, rows, nullptr, loss_log, state, B);
}

template <int HP, int ACT>
static int launch_dqn_target(const imb_policy_desc* pol, const float* params, const float* ring, int64_t ring_ld,
                             const int64_t* ring_idx, const float* expert, int64_t exp_ld, const int64_t* exp_idx,
                             int64_t n_l, int64_t n_e, int64_t n, float gamma, float rew_l, float rew_e, float* out,
                             int rw, int64_t step_base, const int64_t* state, cudaStream_t st) {
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const int xn_off = al(PolImg(pol->d_obs, pol->d_act, HP).total), xn_ld = pol->d_obs | 1;
  const size_t bytes = (size_t)(xn_off + al(128 * xn_ld)) * 4;
  IMB_REQUIRE(bytes <= IMB_SMEM_MAX, "policy too large");
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_dqn_target<HP, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, IMB_SMEM_MAX);
    if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute(k_dqn_target): %s", cudaGetErrorString(e));
    attr_set = true;
  }
  int64_t blocks = (n + 127) / 128;
  const int64_t cap = (int64_t)imb_num_sms() * 2;
  if (blocks > cap) blocks = cap;
  k_dqn_target<HP, ACT><<<(int)blocks, 128, bytes, st>>>(*pol, params, ring, ring_ld, ring_idx, expert, exp_ld, exp_idx,
                                                        n_l, n_e, n, gamma, rew_l, rew_e, out, rw, xn_off, xn_ld,
                                                        step_base, state);
  IMB_CHECK_LAUNCH("k_dqn_target");
  return 0;
}

extern "C" int imb_dqn_target(const imb_policy_desc* pol, int32_t pol_act, const float* target_params,
                              const float* ring, int64_t ring_ld, const int64_t* ring_idx, const float* expert,
                              int64_t expert_ld, const int64_t* expert_idx, int64_t n_learner, int64_t n_expert,
                              int64_t n_steps, float gamma, float reward_learner, float reward_expert, float* rows,
                              int64_t step_base, const int64_t* state, void* stream) {
  IMB_REQUIRE(pol_act == IMB_ACT_TANH || pol_act == IMB_ACT_RELU,
              "pol_act must be IMB_ACT_TANH (0) or IMB_ACT_RELU (1), got %d", pol_act);
  IMB_REQUIRE(pol->discrete && !pol->has_norm, "the DQN target runs Discrete Q-nets without a feature RunningNorm");
  IMB_REQUIRE(pol->hidden >= 1 && pol->hidden <= 64, "policy tower width must be <= 64");
  IMB_REQUIRE(n_learner >= 0 && n_expert >= 0 && n_steps >= 0, "bad row counts");
  IMB_REQUIRE(n_learner == 0 || (ring != nullptr && ring_idx != nullptr), "learner rows need the ring and its indices");
  IMB_REQUIRE(n_expert == 0 || (expert != nullptr && expert_idx != nullptr), "expert rows need the table and its indices");
  const int64_t n = n_steps * (n_learner + n_expert);
  if (n <= 0) return 0;
  const int rw = imb_rollout_row_width(pol);
  const cudaStream_t st = (cudaStream_t)stream;
  if (pol_act == IMB_ACT_TANH)
    return pol->hidden <= 32
               ? launch_dqn_target<32, ACT_TANH>(pol, target_params, ring, ring_ld, ring_idx, expert, expert_ld,
                                                 expert_idx, n_learner, n_expert, n, gamma, reward_learner,
                                                 reward_expert, rows, rw, step_base, state, st)
               : launch_dqn_target<64, ACT_TANH>(pol, target_params, ring, ring_ld, ring_idx, expert, expert_ld,
                                                 expert_idx, n_learner, n_expert, n, gamma, reward_learner,
                                                 reward_expert, rows, rw, step_base, state, st);
  return pol->hidden <= 32
             ? launch_dqn_target<32, ACT_RELU>(pol, target_params, ring, ring_ld, ring_idx, expert, expert_ld, expert_idx,
                                               n_learner, n_expert, n, gamma, reward_learner, reward_expert, rows, rw, step_base, state, st)
             : launch_dqn_target<64, ACT_RELU>(pol, target_params, ring, ring_ld, ring_idx, expert, expert_ld, expert_idx,
                                               n_learner, n_expert, n, gamma, reward_learner, reward_expert, rows, rw, step_base, state, st);
}

template <int HP, int ACT>
static int launch_logp(const imb_policy_desc* pol, const float* params, const float* norm, float* batch, int64_t ld,
                       int64_t n, int row_logp, cudaStream_t st) {
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const int xn_off = al(PolImg(pol->d_obs, pol->d_act, HP).total), xn_ld = pol->d_obs | 1;
  const size_t bytes = (size_t)(xn_off + al(128 * xn_ld)) * 4;
  IMB_REQUIRE(bytes <= IMB_SMEM_MAX, "policy too large");
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_policy_logp<HP, ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize, IMB_SMEM_MAX);
    if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute(k_policy_logp): %s", cudaGetErrorString(e));
    attr_set = true;
  }
  int64_t blocks = (n + 127) / 128;
  const int64_t cap = (int64_t)imb_num_sms() * 2;
  if (blocks > cap) blocks = cap;
  k_policy_logp<HP, ACT><<<(int)blocks, 128, bytes, st>>>(*pol, params, norm, batch, ld, n, row_logp, xn_off, xn_ld);
  IMB_CHECK_LAUNCH("k_policy_logp");
  return 0;
}

extern "C" int imb_policy_logp(const imb_policy_desc* pol, int32_t pol_act, const float* pol_params,
                               const float* pol_norm, float* batch, int64_t ld, int64_t n, int32_t row_logp,
                               void* stream) {
  IMB_REQUIRE(pol_act == IMB_ACT_TANH || pol_act == IMB_ACT_RELU,
              "pol_act must be IMB_ACT_TANH (0) or IMB_ACT_RELU (1), got %d", pol_act);
  if (n <= 0) return 0;
  IMB_REQUIRE(pol->hidden >= 1 && pol->hidden <= 64, "policy tower width must be <= 64");
  const cudaStream_t st = (cudaStream_t)stream;
  if (pol_act == IMB_ACT_TANH)
    return pol->hidden <= 32 ? launch_logp<32, ACT_TANH>(pol, pol_params, pol_norm, batch, ld, n, row_logp, st)
                             : launch_logp<64, ACT_TANH>(pol, pol_params, pol_norm, batch, ld, n, row_logp, st);
  return pol->hidden <= 32 ? launch_logp<32, ACT_RELU>(pol, pol_params, pol_norm, batch, ld, n, row_logp, st)
                           : launch_logp<64, ACT_RELU>(pol, pol_params, pol_norm, batch, ld, n, row_logp, st);
}

#ifdef IMB_PPO_TIMING
extern "C" __attribute__((visibility("default"))) int imb_debug_ppo_clocks(long long* out) {
  return (int)cudaMemcpyFromSymbol(out, g_ppo_clk, 16 * sizeof(long long));
}
extern "C" __attribute__((visibility("default"))) int imb_debug_ppo_warp_clocks(long long* out, int reset) {
  static const long long zero[80] = {0};
  if (reset) return (int)cudaMemcpyToSymbol(g_ppo_wclk, zero, sizeof(zero));
  return (int)cudaMemcpyFromSymbol(out, g_ppo_wclk, 80 * sizeof(long long));
}
#endif
