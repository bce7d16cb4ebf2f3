// imb_sac.cu -- SAC (SB3 2.2's SAC.train and collect_rollouts, restated by oracle/sac_port.py): the actor's collection
// in the device envs and the gradient step of the twin critics, the actor and the entropy coefficient.
//
// Nets (SB3's SACPolicy with net_arch [h, h], ReLU; torch Linear layout, each net one flat vector in nn.Linear order):
//   actor   latent_pi.0 [h][Do] [h] | latent_pi.2 [h][h] [h] | mu [Da][h] [Da] | log_std [Da][h] [Da]
//   critic  qf0.0 [h][Do+Da] [h] | qf0.2 [h][h] [h] | qf0.4 [1][h] [1] | qf1 (the same)      (critic_target alike)
//
// Every kernel here is row-tiled: a CTA of SAC_NT threads owns SAC_R rows (envs or minibatch rows) and evaluates each
// layer as "thread j computes output j for the CTA's rows", so a weight read from L2 serves the whole tile.  Weights stay
// in global memory (at h = 256 the nets do not fit in shared memory); activations of the tile live in shared memory.
//
// The gradient step is four launches per SB3 gradient step; kernel boundaries order its phases (no grid barrier):
//   k_sac_critic   (a) actor on s and s', target critics, y, twin-critic forward + backward, ent-coef terms
//   k_sac_adam     (b) critic: per-CTA partial gradients summed in CTA order + torch Adam; log_ent_coef's Adam
//   k_sac_actor    (c) critics on (s, a_pi) with the new weights, backward to the action, then the actor backward
//   k_sac_adam     (d) actor: reduce + Adam, the Polyak update of the critic targets, the step counter
// No atomics: each CTA writes its partial gradient, and the reduce sums the partials in CTA order, so a run is
// bit-reproducible.
#include "imb_common.cuh"
#include "imb_env_step.cuh"

namespace {

constexpr int SAC_NT = 256;  // threads per CTA
constexpr int SAC_R = 8;     // rows per CTA
constexpr int SAC_MAX_DO = 64, SAC_MAX_DA = 8, SAC_MAX_H = 256, SAC_MAX_B = 256;
constexpr float LOG_STD_MIN = -20.f, LOG_STD_MAX = 2.f;

// parameter offsets (floats) of the flat nets
struct SacNet {
  int Do, Da, h, din;
  // actor
  __host__ __device__ int a_w1() const { return 0; }
  __host__ __device__ int a_b1() const { return h * Do; }
  __host__ __device__ int a_w2() const { return a_b1() + h; }
  __host__ __device__ int a_b2() const { return a_w2() + h * h; }
  __host__ __device__ int a_wmu() const { return a_b2() + h; }
  __host__ __device__ int a_bmu() const { return a_wmu() + Da * h; }
  __host__ __device__ int a_wls() const { return a_bmu() + Da; }
  __host__ __device__ int a_bls() const { return a_wls() + Da * h; }
  __host__ __device__ int n_actor() const { return a_bls() + Da; }
  // one Q net; net q starts at q * n_q()
  __host__ __device__ int q_w1() const { return 0; }
  __host__ __device__ int q_b1() const { return h * din; }
  __host__ __device__ int q_w2() const { return q_b1() + h; }
  __host__ __device__ int q_b2() const { return q_w2() + h * h; }
  __host__ __device__ int q_w3() const { return q_b2() + h; }
  __host__ __device__ int q_b3() const { return q_w3() + h; }
  __host__ __device__ int n_q() const { return q_b3() + 1; }
  __host__ __device__ int n_critic() const { return 2 * n_q(); }
};
__host__ __device__ inline SacNet sac_net(int Do, int Da, int h) { return SacNet{Do, Da, h, Do + Da}; }

// ---- row-tile layers (every thread of the CTA calls them; a __syncthreads follows each) ---------------------------
// Y[r][j] = act(b[j] + sum_k W[j][k] X[r][k]), r < SAC_R, j < out: thread j, its weight row walked once for the tile
template <bool RELU>
__device__ __forceinline__ void tile_fwd(const float* __restrict__ W, const float* __restrict__ b, int in, int out,
                                         const float* X, int ldx, float* Y, int ldy) {
  for (int j = threadIdx.x; j < out; j += SAC_NT) {
    float acc[SAC_R];
#pragma unroll
    for (int r = 0; r < SAC_R; ++r) acc[r] = 0.f;
    const float* w = W + (size_t)j * in;
    for (int k = 0; k < in; ++k) {
      const float wk = __ldg(w + k);
#pragma unroll
      for (int r = 0; r < SAC_R; ++r) acc[r] = fmaf(wk, X[r * ldx + k], acc[r]);
    }
    const float bj = __ldg(b + j);
#pragma unroll
    for (int r = 0; r < SAC_R; ++r) {
      const float z = acc[r] + bj;
      Y[r * ldy + j] = RELU ? fmaxf(z, 0.f) : z;
    }
  }
}
// narrow heads (out <= 8): one warp per (row, output), lanes split k, then a warp sum
__device__ __forceinline__ void tile_head(const float* __restrict__ W, const float* __restrict__ b, int in, int out,
                                          const float* X, int ldx, float* Y, int ldy) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = warp; i < SAC_R * out; i += SAC_NT / 32) {
    const int r = i / out, j = i - r * out;
    float s = 0.f;
    for (int k = lane; k < in; k += 32) s = fmaf(__ldg(W + (size_t)j * in + k), X[r * ldx + k], s);
    s = warp_sum(s);
    if (lane == 0) Y[r * ldy + j] = s + __ldg(b + j);
  }
}
// dX[r][k] = (sum_j dY[r][j] W[j][k]) * (relu mask of A[r][k] when A), k in [k0, k1); written at dX[r * ldx + k - k0]
__device__ __forceinline__ void tile_bwd_in(const float* __restrict__ W, int in, int out, const float* dY, int ldy,
                                            int k0, int k1, const float* A, int lda, float* dX, int ldx) {
  for (int k = k0 + threadIdx.x; k < k1; k += SAC_NT) {
    float acc[SAC_R];
#pragma unroll
    for (int r = 0; r < SAC_R; ++r) acc[r] = 0.f;
    for (int j = 0; j < out; ++j) {
      const float w = W[(size_t)j * in + k];
#pragma unroll
      for (int r = 0; r < SAC_R; ++r) acc[r] = fmaf(dY[r * ldy + j], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < SAC_R; ++r) dX[r * ldx + k - k0] = (A && !(A[r * lda + k] > 0.f)) ? 0.f : acc[r];
  }
}
// this CTA's partial weight gradient: G[j][k] = sum_r dY[r][j] X[r][k], Gb[j] = sum_r dY[r][j] (rows in order)
__device__ __forceinline__ void tile_wgrad(const float* dY, int ldy, const float* X, int ldx, int in, int out,
                                           float* __restrict__ G, float* __restrict__ Gb) {
  for (int idx = threadIdx.x; idx < out * in; idx += SAC_NT) {
    const int j = idx / in, k = idx - j * in;
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < SAC_R; ++r) s = fmaf(dY[r * ldy + j], X[r * ldx + k], s);
    G[idx] = s;
  }
  for (int j = threadIdx.x; j < out; j += SAC_NT) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < SAC_R; ++r) s += dY[r * ldy + j];
    Gb[j] = s;
  }
}

// The actor's mean and clamped log_std of the tile's rows X [SAC_R][ldx]: H1, H2 [SAC_R][h] keep the latent, MU / LS
// [SAC_R][SAC_MAX_DA] the heads (LS clamped to [-20, 2]; LSM 1 where the clamp passes the gradient).
__device__ __forceinline__ void actor_forward(const float* __restrict__ P, const SacNet& N, const float* X, int ldx,
                                              float* H1, float* H2, float* MU, float* LS, float* LSM) {
  const int h = N.h;
  tile_fwd<true>(P + N.a_w1(), P + N.a_b1(), N.Do, h, X, ldx, H1, h);
  __syncthreads();
  tile_fwd<true>(P + N.a_w2(), P + N.a_b2(), h, h, H1, h, H2, h);
  __syncthreads();
  tile_head(P + N.a_wmu(), P + N.a_bmu(), h, N.Da, H2, h, MU, SAC_MAX_DA);
  tile_head(P + N.a_wls(), P + N.a_bls(), h, N.Da, H2, h, LS, SAC_MAX_DA);
  __syncthreads();
  for (int i = threadIdx.x; i < SAC_R * N.Da; i += SAC_NT) {
    const int r = i / N.Da, a = i - r * N.Da;
    const float l = LS[r * SAC_MAX_DA + a];
    LSM[r * SAC_MAX_DA + a] = (l >= LOG_STD_MIN && l <= LOG_STD_MAX) ? 1.f : 0.f;
    LS[r * SAC_MAX_DA + a] = fminf(fmaxf(l, LOG_STD_MIN), LOG_STD_MAX);
  }
  __syncthreads();
}

// SquashedDiagGaussian of row r: g = mean + std * eps, a = tanh(g) (EPS NULL: a = tanh(mean));
// log_prob = sum_a Normal(mean, std).log_prob(g) - sum_a log(1 - a^2 + 1e-6), each term in SB3's float32 order.
__device__ __forceinline__ float squash_row(int r, int Da, const float* MU, const float* LS, const float* EPS,
                                            float* ACT) {
  float s1 = 0.f, s2 = 0.f;
  for (int a = 0; a < Da; ++a) {
    const float m = MU[r * SAC_MAX_DA + a], ls = LS[r * SAC_MAX_DA + a];
    const float sd = expf(ls);
    const float g = EPS ? __fadd_rn(m, __fmul_rn(EPS[r * SAC_MAX_DA + a], sd)) : m;
    const float act = tanhf(g);
    ACT[r * SAC_MAX_DA + a] = act;
    const float d = __fsub_rn(g, m);
    s1 += __fsub_rn(__fsub_rn(-__fdiv_rn(__fmul_rn(d, d), __fmul_rn(2.f, __fmul_rn(sd, sd))), ls),
                    0.9189385332046727f);
    s2 += logf(__fadd_rn(__fsub_rn(1.f, __fmul_rn(act, act)), 1e-6f));
  }
  return s1 - s2;
}

// eps of row `row` of gradient step `n`: normals of Philox stream IMB_STREAM_SAC_STEP at counter (row, n, chunk), chunk
// 0-1 for the actor on s and 2-3 for the actor on s' (normal 4 chunk + j % 4 of oracle/philox.normals(.., 16))
// (both loops unrolled, so z stays in registers: no local-memory array)
__device__ __forceinline__ void normals_to(uint64_t seed, uint32_t stream, uint32_t a, uint32_t b, int chunk0, int Da,
                                           float* e) {
#pragma unroll
  for (int c = 0; c < SAC_MAX_DA / 4; ++c) {
    if (4 * c >= Da) break;
    float z[4];
    philox_normal4(seed, stream, a, b, chunk0 + c, z);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (4 * c + j < Da) e[4 * c + j] = z[j];
  }
}
__device__ __forceinline__ void step_eps(uint64_t seed, uint32_t row, uint32_t n, int which, int Da, float* e) {
  normals_to(seed, IMB_STREAM_SAC_STEP, row, n, which * 2, Da, e);
}

// SB3's Box scaling, in float32 and its operation order (common/policies.py scale_action / unscale_action)
__device__ __forceinline__ float box_scale(float x, float lo, float hi) {
  return __fsub_rn(__fmul_rn(2.f, __fdiv_rn(__fsub_rn(x, lo), __fsub_rn(hi, lo))), 1.f);
}
__device__ __forceinline__ float box_unscale(float x, float lo, float hi) {
  return __fadd_rn(lo, __fmul_rn(__fmul_rn(0.5f, __fadd_rn(x, 1.f)), __fsub_rn(hi, lo)));
}

// the step's hyperparameters (imb_sac_step's scalar arguments)
struct SacHp {
  int d_obs, d_act, hidden, batch_size;
  float gamma, tau, lr, adam_eps;
  int auto_ent;
  float ent_coef, target_entropy, reward_learner, reward_expert;
  int target_update_interval;
  uint64_t seed;
};

struct SacArgs {
  SacHp d;
  SacNet N;
  int64_t ring_ld, expert_ld, step_base;
  int n_blk, polyak;
};

// shared-memory plan of the step kernels (floats)
struct StepSmem {
  float *XS, *XN, *XQ, *XT, *H[8], *MU, *LS, *LSM, *EPS, *ACT, *DA, *row;  // row: [16][SAC_R] per-row scalars
};
__device__ __forceinline__ StepSmem step_smem(float* smem, int h) {
  StepSmem S;
  float* p = smem;
  S.XS = p; p += SAC_R * SAC_MAX_DO;
  S.XN = p; p += SAC_R * SAC_MAX_DO;
  S.XQ = p; p += SAC_R * (SAC_MAX_DO + SAC_MAX_DA);
  S.XT = p; p += SAC_R * (SAC_MAX_DO + SAC_MAX_DA);
  for (int i = 0; i < 8; ++i) { S.H[i] = p; p += SAC_R * h; }
  S.MU = p; p += SAC_R * SAC_MAX_DA;
  S.LS = p; p += SAC_R * SAC_MAX_DA;
  S.LSM = p; p += SAC_R * SAC_MAX_DA;
  S.EPS = p; p += SAC_R * SAC_MAX_DA;
  S.ACT = p; p += SAC_R * SAC_MAX_DA;
  S.DA = p; p += SAC_R * SAC_MAX_DA;
  S.row = p;
  return S;
}
__host__ __device__ inline size_t step_smem_bytes(int h) {
  return (size_t)4 * (SAC_R * (2 * SAC_MAX_DO + 2 * (SAC_MAX_DO + SAC_MAX_DA)) + 8 * SAC_R * h + 6 * SAC_R * SAC_MAX_DA +
                      16 * SAC_R);
}
enum { RW_REW = 0, RW_DONE, RW_VALID, RW_LOGP, RW_Y, RW_Q0, RW_Q1, RW_DQ0, RW_DQ1, RW_MINQ };

// workspace (floats): [n_blk][n_critic] critic partials | [n_blk][n_actor] actor partials | [n_blk][4] statistics
// (critic loss sum, sum (logp + target_entropy), actor loss sum, -) | [4] (alpha, step n as float bits, -, -)
__host__ __device__ inline int64_t ws_floats(const SacNet& N, int n_blk) {
  return (int64_t)n_blk * (N.n_critic() + N.n_actor() + 4) + 4;
}

// gather the tile's minibatch rows: row b < n_learner from ring column ring_idx[k][b], else expert column
// expert_idx[k][b - n_learner]; feature-major tables [tw][ld], tw = 2 Do + Da + 1
__device__ __forceinline__ void load_rows(const SacArgs& A, const float* ring, const int64_t* ring_idx,
                                          const float* expert, const int64_t* expert_idx, int64_t k, StepSmem& S,
                                          bool next) {
  const int Do = A.N.Do, Da = A.N.Da, din = A.N.din, tw = 2 * Do + Da + 1;
  const int B = A.d.batch_size, nl = B / 2, ne = B - nl;
  for (int i = threadIdx.x; i < SAC_R * tw; i += SAC_NT) {
    const int r = i / tw, c = i - r * tw;
    const int b = blockIdx.x * SAC_R + r;
    float v = 0.f;
    if (b < B) {
      const float* t = b < nl ? ring : expert;
      const int64_t ld = b < nl ? A.ring_ld : A.expert_ld;
      const int64_t col = b < nl ? ring_idx[k * nl + b] : expert_idx[k * ne + (b - nl)];
      v = t[(int64_t)c * ld + col];
    }
    if (c < Do) {
      S.XS[r * SAC_MAX_DO + c] = v;
      S.XQ[r * din + c] = v;
    } else if (c < Do + Da) {
      S.XQ[r * din + c] = v;
    } else if (c < 2 * Do + Da) {
      if (next) S.XN[r * SAC_MAX_DO + c - Do - Da] = v;
    } else {
      S.row[RW_DONE * SAC_R + r] = v;
    }
  }
  for (int r = threadIdx.x; r < SAC_R; r += SAC_NT) {
    const int b = blockIdx.x * SAC_R + r;
    S.row[RW_VALID * SAC_R + r] = b < B ? 1.f : 0.f;
    S.row[RW_REW * SAC_R + r] = b < nl ? A.d.reward_learner : A.d.reward_expert;
  }
  __syncthreads();
}

// Q net q of a twin-critic vector on XQ -> row[RW_Q0 + q]; H1, H2 keep its latents
__device__ __forceinline__ void q_forward(const float* __restrict__ C, const SacNet& N, int q, const float* XQ,
                                          float* H1, float* H2, float* out) {
  const float* P = C + (size_t)q * N.n_q();
  tile_fwd<true>(P + N.q_w1(), P + N.q_b1(), N.din, N.h, XQ, N.din, H1, N.h);
  __syncthreads();
  tile_fwd<true>(P + N.q_w2(), P + N.q_b2(), N.h, N.h, H1, N.h, H2, N.h);
  __syncthreads();
  tile_head(P + N.q_w3(), P + N.q_b3(), N.h, 1, H2, N.h, out, 1);
  __syncthreads();
}

// backward of Q net q from dQ [SAC_R] (row scalars): G2 = dQ w3 * relu'(H2), G1 = G2 W2 * relu'(H1); with G non-null
// the CTA's partial weight gradients go to G (the net's slice); with DA non-null dQ/d(action) is added into DA
__device__ __forceinline__ void q_backward(const float* __restrict__ C, const SacNet& N, int q, const float* dQ,
                                           const float* XQ, const float* H1, const float* H2, float* G2, float* G1,
                                           float* __restrict__ G, float* DA) {
  const float* P = C + (size_t)q * N.n_q();
  const int h = N.h;
  for (int i = threadIdx.x; i < SAC_R * h; i += SAC_NT) {
    const int r = i / h, j = i - r * h;
    G2[i] = H2[i] > 0.f ? dQ[r] * __ldg(P + N.q_w3() + j) : 0.f;
  }
  __syncthreads();
  if (G) {
    tile_wgrad(dQ, 1, H2, h, h, 1, G + N.q_w3(), G + N.q_b3());
    tile_wgrad(G2, h, H1, h, h, h, G + N.q_w2(), G + N.q_b2());
  }
  tile_bwd_in(P + N.q_w2(), h, h, G2, h, 0, h, H1, h, G1, h);
  __syncthreads();
  if (G) tile_wgrad(G1, h, XQ, N.din, N.din, h, G + N.q_w1(), G + N.q_b1());
  if (DA) {
    // dQ/da = G1 W1[:, Do:Do+Da]; accumulated into DA (the caller zeroed it), net 0 then net 1
    for (int i = threadIdx.x; i < SAC_R * N.Da; i += SAC_NT) {
      const int r = i / N.Da, a = i - r * N.Da;
      float s = 0.f;
      for (int j = 0; j < h; ++j) s = fmaf(G1[r * h + j], P[N.q_w1() + (size_t)j * N.din + N.Do + a], s);
      DA[r * SAC_MAX_DA + a] += s;
    }
  }
  __syncthreads();
}

// ---- (a) the critic phase --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SAC_NT, 1) k_sac_critic(const SacArgs A, const float* __restrict__ actor,
                                                       const float* __restrict__ critic,
                                                       const float* __restrict__ target, const float* __restrict__ ent,
                                                       const float* __restrict__ ring,
                                                       const int64_t* __restrict__ ring_idx,
                                                       const float* __restrict__ expert,
                                                       const int64_t* __restrict__ expert_idx,
                                                       const int64_t* __restrict__ state, float* __restrict__ ws) {
  extern __shared__ __align__(16) float smem[];
  const SacNet& N = A.N;
  StepSmem S = step_smem(smem, N.h);
  const int64_t n = state[IMB_ST_PPO_STEP], k = n - A.step_base;
  const int Da = N.Da, B = A.d.batch_size;
  const float alpha = A.d.auto_ent ? expf(ent[0]) : A.d.ent_coef;  // ent_coef, read before its own Adam step
  float* tail = ws + (int64_t)A.n_blk * (N.n_critic() + N.n_actor() + 4);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    tail[0] = alpha;
    tail[1] = __int_as_float((int)n);
  }
  load_rows(A, ring, ring_idx, expert, expert_idx, k, S, true);
  float* row = S.row;
  // actor on s' -> a', logp'
  actor_forward(actor, N, S.XN, SAC_MAX_DO, S.H[0], S.H[1], S.MU, S.LS, S.LSM);
  for (int r = threadIdx.x; r < SAC_R; r += SAC_NT) {
    step_eps(A.d.seed, (uint32_t)(blockIdx.x * SAC_R + r), (uint32_t)n, 1, Da, S.EPS + r * SAC_MAX_DA);
    row[RW_LOGP * SAC_R + r] = squash_row(r, Da, S.MU, S.LS, S.EPS, S.ACT);
  }
  __syncthreads();
  // target critics on (s', a')
  float* XT = S.XT;  // [SAC_R][din]: (s', a')
  for (int i = threadIdx.x; i < SAC_R * N.din; i += SAC_NT) {
    const int r = i / N.din, c = i - r * N.din;
    XT[i] = c < N.Do ? S.XN[r * SAC_MAX_DO + c] : S.ACT[r * SAC_MAX_DA + c - N.Do];
  }
  __syncthreads();
  q_forward(target, N, 0, XT, S.H[0], S.H[1], row + RW_Q0 * SAC_R);
  q_forward(target, N, 1, XT, S.H[0], S.H[1], row + RW_Q1 * SAC_R);
  for (int r = threadIdx.x; r < SAC_R; r += SAC_NT) {
    // y = r + (1 - d) * gamma * (min(Q1t, Q2t) - ent_coef * logp'), each operation rounded as torch rounds it
    const float mq = fminf(row[RW_Q0 * SAC_R + r], row[RW_Q1 * SAC_R + r]);
    const float nq = __fsub_rn(mq, __fmul_rn(alpha, row[RW_LOGP * SAC_R + r]));
    const float y = __fadd_rn(row[RW_REW * SAC_R + r],
                              __fmul_rn(__fmul_rn(__fsub_rn(1.f, row[RW_DONE * SAC_R + r]), A.d.gamma), nq));
    row[RW_Y * SAC_R + r] = row[RW_VALID * SAC_R + r] != 0.f ? y : 0.f;
  }
  __syncthreads();
  // actor on s -> logp (the entropy-coefficient term)
  actor_forward(actor, N, S.XS, SAC_MAX_DO, S.H[0], S.H[1], S.MU, S.LS, S.LSM);
  for (int r = threadIdx.x; r < SAC_R; r += SAC_NT) {
    step_eps(A.d.seed, (uint32_t)(blockIdx.x * SAC_R + r), (uint32_t)n, 0, Da, S.EPS + r * SAC_MAX_DA);
    row[RW_LOGP * SAC_R + r] = squash_row(r, Da, S.MU, S.LS, S.EPS, S.ACT);
  }
  __syncthreads();
  // twin critics on (s, a): forward, dL/dQ_q = (Q_q - y) / B, backward into this CTA's partial gradient
  float* part = ws + (int64_t)blockIdx.x * N.n_critic();
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    float* Qq = row + (RW_Q0 + q) * SAC_R;
    float* dQ = row + (RW_DQ0 + q) * SAC_R;
    q_forward(critic, N, q, S.XQ, S.H[2 * q], S.H[2 * q + 1], Qq);
    for (int r = threadIdx.x; r < SAC_R; r += SAC_NT)
      dQ[r] = row[RW_VALID * SAC_R + r] != 0.f ? (Qq[r] - row[RW_Y * SAC_R + r]) / (float)B : 0.f;
    __syncthreads();
    q_backward(critic, N, q, dQ, S.XQ, S.H[2 * q], S.H[2 * q + 1], S.H[4], S.H[5], part + (size_t)q * N.n_q(),
               nullptr);
  }
  if (threadIdx.x == 0) {
    float cl = 0.f, el = 0.f;
    for (int r = 0; r < SAC_R; ++r) {
      if (row[RW_VALID * SAC_R + r] == 0.f) continue;
      for (int q = 0; q < 2; ++q) {
        const float d = row[(RW_Q0 + q) * SAC_R + r] - row[RW_Y * SAC_R + r];
        cl = fmaf(d, d, cl);
      }
      el += row[RW_LOGP * SAC_R + r] + A.d.target_entropy;
    }
    float* st = ws + (int64_t)A.n_blk * (N.n_critic() + N.n_actor()) + blockIdx.x * 4;
    st[0] = cl;
    st[1] = el;
  }
}

// ---- (c) the actor phase ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SAC_NT, 1) k_sac_actor(const SacArgs A, const float* __restrict__ actor,
                                                      const float* __restrict__ critic,
                                                      const float* __restrict__ ring,
                                                      const int64_t* __restrict__ ring_idx,
                                                      const float* __restrict__ expert,
                                                      const int64_t* __restrict__ expert_idx, float* __restrict__ ws) {
  extern __shared__ __align__(16) float smem[];
  const SacNet& N = A.N;
  StepSmem S = step_smem(smem, N.h);
  const int Da = N.Da, h = N.h, B = A.d.batch_size;
  const float* tail = ws + (int64_t)A.n_blk * (N.n_critic() + N.n_actor() + 4);
  const float alpha = tail[0];
  const int64_t n = (int64_t)__float_as_int(tail[1]), k = n - A.step_base;
  load_rows(A, ring, ring_idx, expert, expert_idx, k, S, false);
  float* row = S.row;
  float* H1a = S.H[6];
  float* H2a = S.H[7];
  actor_forward(actor, N, S.XS, SAC_MAX_DO, H1a, H2a, S.MU, S.LS, S.LSM);
  for (int r = threadIdx.x; r < SAC_R; r += SAC_NT) {
    step_eps(A.d.seed, (uint32_t)(blockIdx.x * SAC_R + r), (uint32_t)n, 0, Da, S.EPS + r * SAC_MAX_DA);
    row[RW_LOGP * SAC_R + r] = squash_row(r, Da, S.MU, S.LS, S.EPS, S.ACT);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < SAC_R * N.din; i += SAC_NT) {
    const int r = i / N.din, c = i - r * N.din;
    if (c >= N.Do) S.XQ[i] = S.ACT[r * SAC_MAX_DA + c - N.Do];
  }
  for (int i = threadIdx.x; i < SAC_R * SAC_MAX_DA; i += SAC_NT) S.DA[i] = 0.f;
  __syncthreads();
  // the updated critics on (s, a_pi); the actor loss (ent_coef logp - min_q Q_q).mean() reaches the action through the
  // net that gives the minimum (torch.min's gradient; the first on a tie)
  q_forward(critic, N, 0, S.XQ, S.H[0], S.H[1], row + RW_Q0 * SAC_R);
  q_forward(critic, N, 1, S.XQ, S.H[2], S.H[3], row + RW_Q1 * SAC_R);
  for (int r = threadIdx.x; r < SAC_R; r += SAC_NT) {
    const float q0 = row[RW_Q0 * SAC_R + r], q1 = row[RW_Q1 * SAC_R + r];
    const bool valid = row[RW_VALID * SAC_R + r] != 0.f, one = q1 < q0;
    row[RW_MINQ * SAC_R + r] = one ? q1 : q0;
    row[RW_DQ0 * SAC_R + r] = valid && !one ? -1.f / (float)B : 0.f;
    row[RW_DQ1 * SAC_R + r] = valid && one ? -1.f / (float)B : 0.f;
  }
  __syncthreads();
  q_backward(critic, N, 0, row + RW_DQ0 * SAC_R, S.XQ, S.H[0], S.H[1], S.H[4], S.H[5], nullptr, S.DA);
  q_backward(critic, N, 1, row + RW_DQ1 * SAC_R, S.XQ, S.H[2], S.H[3], S.H[4], S.H[5], nullptr, S.DA);
  // squashed-Gaussian backward, per (row, action): dL/dg = alpha/B dlogp/dg + dL/da (1 - a^2),
  // dlogp/dg = 2 a (1 - a^2) / (1 - a^2 + 1e-6); dL/dmean = dL/dg; dL/dlog_std = clamp mask (-alpha/B + dL/dg std eps)
  float* DMU = S.MU;  // (overwritten in place: the forward values are no longer needed)
  float* DLS = S.LS;
  for (int i = threadIdx.x; i < SAC_R * Da; i += SAC_NT) {
    const int r = i / Da, a = i - r * Da, o = r * SAC_MAX_DA + a;
    const bool valid = row[RW_VALID * SAC_R + r] != 0.f;
    const float act = S.ACT[o], om = 1.f - act * act;
    const float dlogp = 2.f * act * om / (om + 1e-6f);
    const float dg = valid ? alpha / (float)B * dlogp + S.DA[o] * om : 0.f;
    const float sd = expf(S.LS[o]);
    DMU[o] = dg;
    DLS[o] = valid ? S.LSM[o] * (-alpha / (float)B + dg * sd * S.EPS[o]) : 0.f;
  }
  __syncthreads();
  float* part = ws + (int64_t)A.n_blk * N.n_critic() + (int64_t)blockIdx.x * N.n_actor();
  tile_wgrad(DMU, SAC_MAX_DA, H2a, h, h, Da, part + N.a_wmu(), part + N.a_bmu());
  tile_wgrad(DLS, SAC_MAX_DA, H2a, h, h, Da, part + N.a_wls(), part + N.a_bls());
  float* G2 = S.H[4];
  float* G1 = S.H[5];
  for (int i = threadIdx.x; i < SAC_R * h; i += SAC_NT) {
    const int r = i / h, j = i - r * h;
    float s = 0.f;
    for (int a = 0; a < Da; ++a) {
      s = fmaf(DMU[r * SAC_MAX_DA + a], __ldg(actor + N.a_wmu() + a * h + j), s);
      s = fmaf(DLS[r * SAC_MAX_DA + a], __ldg(actor + N.a_wls() + a * h + j), s);
    }
    G2[i] = H2a[i] > 0.f ? s : 0.f;
  }
  __syncthreads();
  tile_wgrad(G2, h, H1a, h, h, h, part + N.a_w2(), part + N.a_b2());
  tile_bwd_in(actor + N.a_w2(), h, h, G2, h, 0, h, H1a, h, G1, h);
  __syncthreads();
  tile_wgrad(G1, h, S.XS, SAC_MAX_DO, N.Do, h, part + N.a_w1(), part + N.a_b1());
  if (threadIdx.x == 0) {
    float al = 0.f;
    for (int r = 0; r < SAC_R; ++r)
      if (row[RW_VALID * SAC_R + r] != 0.f)
        al += __fsub_rn(__fmul_rn(alpha, row[RW_LOGP * SAC_R + r]), row[RW_MINQ * SAC_R + r]);
    ws[(int64_t)A.n_blk * (N.n_critic() + N.n_actor()) + blockIdx.x * 4 + 2] = al;
  }
}

// torch Adam (betas 0.9 / 0.999): m.lerp_(g, 0.1); v = 0.999 v + 0.001 g^2; p -= lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps)
__device__ __forceinline__ void adam1(float& p, float& m, float& v, float g, float step_size, float bc2_sqrt,
                                      float eps) {
  m = fmaf(0.1f, g - m, m);
  v = fmaf(0.001f, g * g, 0.999f * v);
  p -= step_size * (m / (sqrtf(v) / bc2_sqrt + eps));
}

// ---- (b) / (d): reduce + Adam of one net; which 0: the critic (+ log_ent_coef's Adam and the critic / ent-coef loss
// log), which 1: the actor (+ the Polyak update of the targets, the actor loss log, and the step counter) -------------
__global__ void __launch_bounds__(256) k_sac_adam(const SacArgs A, int which, float* __restrict__ params,
                                                  float* __restrict__ m, float* __restrict__ v,
                                                  float* __restrict__ critic, float* __restrict__ target,
                                                  float* __restrict__ ent, float* __restrict__ ws,
                                                  float* __restrict__ loss_log, int64_t* __restrict__ state) {
  const SacNet& N = A.N;
  const int n_par = which == 0 ? N.n_critic() : N.n_actor();
  const float* part = ws + (which == 0 ? 0 : (int64_t)A.n_blk * N.n_critic());
  const float* stats = ws + (int64_t)A.n_blk * (N.n_critic() + N.n_actor());
  const float* tail = stats + (int64_t)A.n_blk * 4;
  const int64_t n = (int64_t)__float_as_int(tail[1]);
  const double t = (double)(n + 1);
  const double bc1 = 1.0 - pow(0.9, t), bc2 = 1.0 - pow(0.999, t);
  const float step_size = (float)(A.d.lr / bc1), bc2_sqrt = (float)sqrt(bc2);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_par; i += stride) {
    float g = 0.f;
    for (int b = 0; b < A.n_blk; ++b) g += part[(int64_t)b * n_par + i];
    float p = params[i], mi = m[i], vi = v[i];
    adam1(p, mi, vi, g, step_size, bc2_sqrt, A.d.adam_eps);
    params[i] = p;
    m[i] = mi;
    v[i] = vi;
  }
  if (which == 1 && A.polyak) {  // polyak_update: th.mul(t, 1 - tau, out=t); th.add(t, p, alpha=tau, out=t)
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < N.n_critic(); i += stride)
      target[i] = fmaf(A.d.tau, critic[i], target[i] * (1.f - A.d.tau));
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int B = A.d.batch_size;
    float* lrow = loss_log ? loss_log + (n - A.step_base) * 4 : nullptr;
    if (which == 0) {
      float cl = 0.f, el = 0.f;
      for (int b = 0; b < A.n_blk; ++b) {
        cl += stats[b * 4];
        el += stats[b * 4 + 1];
      }
      if (lrow) {
        lrow[0] = 0.5f * (cl / (float)B);
        lrow[3] = tail[0];
      }
      if (A.d.auto_ent) {  // ent_coef_loss = -(log_ent_coef * (logp + target_entropy)).mean(), then its Adam step
        const float mean = el / (float)B;
        if (lrow) lrow[2] = -(ent[0] * mean);
        adam1(ent[0], ent[1], ent[2], -mean, step_size, bc2_sqrt, A.d.adam_eps);
      }
    } else {
      float al = 0.f;
      for (int b = 0; b < A.n_blk; ++b) al += stats[b * 4 + 2];
      if (lrow) lrow[1] = al / (float)B;
      state[IMB_ST_PPO_STEP] = n + 1;  // nothing else of this launch reads the counter (the step is in ws)
    }
  }
}

// ---- collection: E envs for T steps with the actor ---------------------------------------------------------------
struct CollectArgs {
  imb_env_desc env;
  SacNet N;
  int64_t E, T, g0;
  int flags;  // IMB_SAC_DETERMINISTIC | IMB_SAC_PREDICT
  uint64_t seed;
};

__global__ void __launch_bounds__(SAC_NT, 1) k_sac_collect(const CollectArgs C, const float* __restrict__ env_params,
                                                        float* __restrict__ env_obs, const float* __restrict__ actor,
                                                        float* __restrict__ flat_out, float* __restrict__ aux,
                                                        const uint8_t* __restrict__ random_steps,
                                                        const int64_t* __restrict__ state) {
  extern __shared__ __align__(16) float smem[];
  const SacNet& N = C.N;
  const int Do = N.Do, Da = N.Da, h = N.h, tw = 2 * Do + Da + 1;
  float* X = smem;                     // [SAC_R][SAC_MAX_DO] obs
  float* NX = X + SAC_R * SAC_MAX_DO;  // [SAC_R][SAC_MAX_DO] next obs
  float* H1 = NX + SAC_R * SAC_MAX_DO;
  float* H2 = H1 + SAC_R * h;
  float* MU = H2 + SAC_R * h;
  float* LS = MU + SAC_R * SAC_MAX_DA;
  float* LSM = LS + SAC_R * SAC_MAX_DA;
  float* EPS = LSM + SAC_R * SAC_MAX_DA;
  float* ACT = EPS + SAC_R * SAC_MAX_DA;
  float* BUF = ACT + SAC_R * SAC_MAX_DA;  // the buffer action (scaled)
  float* CTL = BUF + SAC_R * SAC_MAX_DA;  // the env action (unscaled)
  const int64_t E = C.E, T = C.T, H = C.env.horizon;
  const int kind = C.env.kind;
  const float hi = env_act_bound(kind), lo = -hi;
  const int tid = threadIdx.x;
  const bool predict = (C.flags & IMB_SAC_PREDICT) != 0;
  const int64_t e = (int64_t)blockIdx.x * SAC_R + tid;  // (thread-per-env parts: tid < SAC_R)
  const bool live = tid < SAC_R && e < E;
  const uint32_t egid = (uint32_t)(C.env.env_id_offset + e);
  for (int i = tid; i < SAC_R * SAC_MAX_DO; i += SAC_NT) {
    const int r = i / SAC_MAX_DO, c = i - r * SAC_MAX_DO;
    const int64_t er = (int64_t)blockIdx.x * SAC_R + r;
    X[i] = (c < Do && er < E) ? env_obs[(int64_t)c * E + er] : 0.f;
  }
  __syncthreads();
  const int64_t t0 = state[IMB_ST_EP_STEP], gstep0 = state[IMB_ST_GLOBAL_STEP];
  int64_t episode = state[IMB_ST_EPISODE];
  for (int64_t t = 0; t < T; ++t) {
    const uint32_t ctr = (uint32_t)(gstep0 + t);
    const bool rnd = random_steps && random_steps[gstep0 + t - C.g0] != 0;  // block-uniform
    if (!rnd) actor_forward(actor, N, X, SAC_MAX_DO, H1, H2, MU, LS, LSM);
    if (live) {
      float* bufa = BUF + tid * SAC_MAX_DA;
      if (rnd) {  // action_space.sample(): uniform in the Box, Philox stream IMB_STREAM_SAC_RANDOM (egid, step, a / 4)
        uint32_t k0, k1;
        philox_key(C.seed, IMB_STREAM_SAC_RANDOM, k0, k1);
        Philox4 w = {0u, 0u, 0u, 0u};
        for (int a = 0; a < Da; ++a) {
          if ((a & 3) == 0) w = philox4x32(egid, ctr, (uint32_t)(a >> 2), 0u, k0, k1);
          const uint32_t x = (a & 3) == 0 ? w.x : (a & 3) == 1 ? w.y : (a & 3) == 2 ? w.z : w.w;
          const float sample = __fadd_rn(lo, __fmul_rn(u01(x), __fsub_rn(hi, lo)));
          bufa[a] = box_scale(sample, lo, hi);
        }
      } else {  // the actor: tanh(mean + std eps), eps of Philox stream IMB_STREAM_SAC_ACT at (egid, step, a / 4)
        const bool det = (C.flags & IMB_SAC_DETERMINISTIC) != 0;
        if (!det) normals_to(C.seed, IMB_STREAM_SAC_ACT, egid, ctr, 0, Da, EPS + tid * SAC_MAX_DA);
        squash_row(tid, Da, MU, LS, det ? nullptr : EPS, ACT);
        for (int a = 0; a < Da; ++a) {
          const float u = box_unscale(ACT[tid * SAC_MAX_DA + a], lo, hi);  // predict()'s action
          bufa[a] = predict ? u : box_scale(u, lo, hi);
        }
      }
      // the env action: unscale(buffer action) as collect_rollouts forms it, or predict()'s action itself
      for (int a = 0; a < Da; ++a) CTL[tid * SAC_MAX_DA + a] = predict ? bufa[a] : box_unscale(bufa[a], lo, hi);
      // env step (thread per env)
      const float* ob = X + tid * SAC_MAX_DO;
      float* nob = NX + tid * SAC_MAX_DO;
      const float* ctl = CTL + tid * SAC_MAX_DA;
      const float rew = kind == IMB_ENV_PENDULUM   ? pendulum_step(ob, ctl, nob, 1)
                        : kind == IMB_ENV_CARTPOLE ? 0.f
                                                   : synth_step(env_params, Do, Da, ob, ctl, nob, 1);
      const bool done = ((t0 + t + 1) % H) == 0;
      const int64_t f = flat_index(e, t, E, T, t0, H);
      float* dst = flat_out + f * tw;
      for (int c = 0; c < Do; ++c) dst[c] = ob[c];
      for (int a = 0; a < Da; ++a) dst[Do + a] = bufa[a];
      for (int c = 0; c < Do; ++c) dst[Do + Da + c] = nob[c];
      dst[2 * Do + Da] = done ? 1.f : 0.f;
      aux[2 * E + E * T + e * T + t] = rew;  // the env reward, where imb_rollout_explore puts it
      float* xo = X + tid * SAC_MAX_DO;
      if (done) {
        if (kind != IMB_ENV_SYNTH)
          classic_reset(kind, C.env.seed, egid, (uint32_t)(episode + 1), xo, 1);
        else
          for (int c = 0; c < Do; ++c)
            xo[c] = 0.1f * philox_normal(C.env.seed, IMB_STREAM_ENV_RESET, egid, (uint32_t)(episode + 1), c);
      } else {
        for (int c = 0; c < Do; ++c) xo[c] = nob[c];
      }
    }
    if (((t0 + t + 1) % H) == 0) ++episode;
    __syncthreads();
  }
  if (live)
    for (int c = 0; c < Do; ++c) env_obs[(int64_t)c * E + e] = X[tid * SAC_MAX_DO + c];
}

static size_t collect_smem_bytes(int h) { return (size_t)4 * (2 * SAC_R * SAC_MAX_DO + 2 * SAC_R * h + 7 * SAC_R * SAC_MAX_DA); }

static int sac_check(int d_obs, int d_act, int hidden, int batch_size) {
  IMB_REQUIRE(d_obs >= 1 && d_obs <= SAC_MAX_DO, "d_obs %d: the SAC kernels run observations of 1 to %d features", d_obs,
              SAC_MAX_DO);
  IMB_REQUIRE(d_act >= 1 && d_act <= SAC_MAX_DA, "d_act %d: the SAC kernels run Box actions of 1 to %d dimensions",
              d_act, SAC_MAX_DA);
  IMB_REQUIRE(hidden >= 1 && hidden <= SAC_MAX_H, "net_arch width %d: the SAC kernels run widths 1 to %d", hidden,
              SAC_MAX_H);
  IMB_REQUIRE(batch_size >= 1 && batch_size <= SAC_MAX_B, "batch_size %d: the SAC step runs batches of 1 to %d",
              batch_size, SAC_MAX_B);
  return 0;
}

template <typename K>
static int set_smem(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
  return 0;
}

}  // namespace

extern "C" int imb_sac_plan(int32_t d_obs, int32_t d_act, int32_t hidden, int32_t batch_size) {
  return sac_check(d_obs, d_act, hidden, batch_size);
}

extern "C" int64_t imb_sac_ws_floats(int32_t d_obs, int32_t d_act, int32_t hidden, int32_t batch_size) {
  if (sac_check(d_obs, d_act, hidden, batch_size) != 0) return -1;
  return ws_floats(sac_net(d_obs, d_act, hidden), (batch_size + SAC_R - 1) / SAC_R);
}

extern "C" int imb_sac_collect(const imb_env_desc* env, const float* env_params, float* env_obs, int32_t hidden,
                               const float* actor, int64_t n_envs, int64_t n_steps, float* flat_out, float* aux,
                               const uint8_t* random_steps, int64_t g0, int32_t flags, uint64_t seed,
                               const int64_t* state, void* stream) {
  IMB_REQUIRE(!env->discrete && env->kind != IMB_ENV_CARTPOLE, "the SAC collection steps Box-action envs");
  if (sac_check(env->d_obs, env->d_act, hidden, 1) != 0) return -1;
  IMB_REQUIRE(n_envs >= 1 && n_steps >= 1 && env->horizon >= 1, "bad collection shape");
  IMB_REQUIRE(env->kind != IMB_ENV_SYNTH || env_params, "the synthetic env needs its parameters");
  CollectArgs C;
  C.env = *env;
  C.N = sac_net(env->d_obs, env->d_act, hidden);
  C.E = n_envs;
  C.T = n_steps;
  C.g0 = g0;
  C.flags = flags;
  C.seed = seed;
  const size_t bytes = collect_smem_bytes(hidden);
  static size_t attr = 0;
  if (bytes > attr) {
    if (set_smem(k_sac_collect, bytes) != 0) return -2;
    attr = bytes;
  }
  const int blocks = (int)((n_envs + SAC_R - 1) / SAC_R);
  k_sac_collect<<<blocks, SAC_NT, bytes, (cudaStream_t)stream>>>(C, env_params, env_obs, actor, flat_out, aux,
                                                                 random_steps, state);
  IMB_CHECK_LAUNCH("k_sac_collect");
  return 0;
}

extern "C" int imb_sac_step(int32_t d_obs, int32_t d_act, int32_t hidden, int32_t batch_size, float gamma, float tau,
                            float lr, float adam_eps, int32_t auto_ent, float ent_coef, float target_entropy,
                            float reward_learner, float reward_expert, int32_t target_update_interval, uint64_t seed,
                            float* actor, float* actor_m, float* actor_v, float* critic,
                            float* critic_m, float* critic_v, float* critic_target, float* ent, const float* ring,
                            int64_t ring_ld, const int64_t* ring_idx, const float* expert, int64_t expert_ld,
                            const int64_t* expert_idx, int64_t n_steps, int64_t step_base, float* loss_log, float* ws,
                            int64_t* state, void* stream) {
  const SacHp hp = {d_obs, d_act, hidden, batch_size, gamma, tau, lr, adam_eps, auto_ent, ent_coef, target_entropy,
                    reward_learner, reward_expert, target_update_interval, seed};
  const SacHp* d = &hp;
  if (sac_check(d->d_obs, d->d_act, d->hidden, d->batch_size) != 0) return -1;
  IMB_REQUIRE(!d->auto_ent || ent, "auto_ent needs the log_ent_coef vector");
  IMB_REQUIRE(d->target_update_interval >= 1, "target_update_interval must be positive");
  if (n_steps <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  SacArgs A;
  A.d = *d;
  A.N = sac_net(d->d_obs, d->d_act, d->hidden);
  A.ring_ld = ring_ld;
  A.expert_ld = expert_ld;
  A.step_base = step_base;
  A.n_blk = (d->batch_size + SAC_R - 1) / SAC_R;
  const size_t bytes = step_smem_bytes(d->hidden);
  static size_t attr = 0;
  if (bytes > attr) {
    if (set_smem(k_sac_critic, bytes) != 0 || set_smem(k_sac_actor, bytes) != 0) return -2;
    attr = bytes;
  }
  const int adam_blocks_c = (A.N.n_critic() + 255) / 256, adam_blocks_a = (A.N.n_actor() + 255) / 256;
  for (int64_t s = 0; s < n_steps; ++s) {
    A.polyak = (s % d->target_update_interval) == 0;  // SB3: gradient_step % target_update_interval inside train()
    k_sac_critic<<<A.n_blk, SAC_NT, bytes, st>>>(A, actor, critic, critic_target, ent, ring, ring_idx, expert,
                                                 expert_idx, state, ws);
    IMB_CHECK_LAUNCH("k_sac_critic");
    k_sac_adam<<<adam_blocks_c, 256, 0, st>>>(A, 0, critic, critic_m, critic_v, critic, critic_target, ent, ws,
                                               loss_log, state);
    IMB_CHECK_LAUNCH("k_sac_adam");
    k_sac_actor<<<A.n_blk, SAC_NT, bytes, st>>>(A, actor, critic, ring, ring_idx, expert, expert_idx, ws);
    IMB_CHECK_LAUNCH("k_sac_actor");
    k_sac_adam<<<adam_blocks_a > adam_blocks_c ? adam_blocks_a : adam_blocks_c, 256, 0, st>>>(
        A, 1, actor, actor_m, actor_v, critic, critic_target, ent, ws, loss_log, state);
    IMB_CHECK_LAUNCH("k_sac_adam");
  }
  return 0;
}
