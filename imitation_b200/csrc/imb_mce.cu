// imb_mce.cu -- tabular MCE IRL: the finite-horizon soft Bellman backup and the state occupancy measures of one MDP
// in one cooperative launch, float64 throughout (algorithms/mce_irl.py: mce_partition_fh :38-93,
// mce_occupancy_measures :96-144, the occupancy / weight arithmetic of MCEIRL._train_step :467-498).
//
// The grid is persistent: CTA b owns the contiguous state range [s0, s1) (and with it the rows (s, a) of T viewed as
// [S*A][S]) for the whole sweep.  One grid barrier separates consecutive time steps:
//  - backward step t: every CTA stages V[t+1] in shared memory; one warp per owned state dots the state's A rows with
//    it (per-lane strided sums, then a fixed xor-shuffle tree), Q = r + gamma * dot, V = logsumexp_a Q as scipy
//    computes it, pi = exp(Q - V).  V[t] goes to a ping-pong buffer the next step reads.
//  - forward step t: every CTA sums x[s, a] * T[(s, a), :] over its owned rows (x = D[t, s] * pi[t, s, a]) into its
//    own partial row of a double-buffered [G][S] array; after the barrier each CTA adds the G partials of ITS states'
//    columns in CTA order, which is D[t+1] for exactly the states whose rows it reads next.  No floating-point atomics,
//    and the partition depends only on the shapes and the grid, so two calls give the same bits.
//  - Dcum: each CTA runs Horner over t = H .. 0 (polyval) or a plain sum (gamma == 1) on its own states' columns.
#include <cooperative_groups.h>

#include "imb_common.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct MceArgs {
  int S, A, H, flags;
  const double* T;      // [S*A][S]
  const double* init;   // [S]
  const double* r64;    // [S] or null
  const float* r32;     // [S] or null (the reward net's float32 output)
  const double* gam;    // [2]: planning discount, occupancy discount
  double* V;            // [H][S] out, optional
  double* Q;            // [H][S][A] out, optional
  double* pi;           // [H][S][A]: out (BACKWARD) or in (FORWARD only); workspace when null
  double* D;            // [H+1][S] out, optional (workspace when null)
  double* Dcum;         // [S] out
  const double* demo;   // [S] or null: training outputs
  float* weights;       // [S]
  double* linf;         // [1]
  double* vbuf;         // [2][S] workspace: V[t+1] / V[t]
  double* part;         // [2][G][S] workspace: forward partial column sums
  double* cta_max;      // [G] workspace
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// max that keeps a NaN once it has seen one, whichever operand it arrives in (np.max propagates NaN)
__device__ __forceinline__ double nan_max(double m, double v) {
  return (isnan(m) || v <= m) ? m : v;
}

__device__ __forceinline__ double reward_of(const MceArgs& a, int s) {
  return a.r64 ? a.r64[s] : (double)a.r32[s];
}

// One backward step for the owned states: lane k < A ends holding Q[t, s, k]; V / pi / Q stores.
__device__ void backward_step(const MceArgs& a, int t, int s0, int s1, const double* __restrict__ vs, double gamma,
                              double* __restrict__ v_out, double* __restrict__ pi_buf) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int S = a.S, A = a.A;
  for (int s = s0 + warp; s < s1; s += kWarps) {
    const double r = reward_of(a, s);
    double q = r;  // this lane's action (lane < A)
    if (t < a.H - 1) {
      const double* __restrict__ row = a.T + (int64_t)s * A * S;
      for (int k = 0; k < A; ++k, row += S) {
        double acc = 0.0;
#pragma unroll 4
        for (int j = lane; j < S; j += 32) acc = fma(__ldg(row + j), vs[j], acc);
        acc = warp_sum_d(acc);
        if (lane == k) q = __dadd_rn(r, __dmul_rn(gamma, acc));  // broad_R + discount * (T @ V)
      }
    }
    // scipy.special.logsumexp: m = #(q == max), s = sum over the others of exp(q - max) in order, s /= m,
    // V = log1p(s) + log(m) + max
    double mx = lane < A ? q : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    double sum = 0.0;
    int m = 0;
    for (int k = 0; k < A; ++k) {
      const double qk = __shfl_sync(0xffffffffu, q, k);
      if (qk == mx) ++m;
      else sum += exp(qk - mx);
    }
    if (sum != 0.0) sum /= (double)m;
    const double v = (log1p(sum) + log((double)m)) + mx;
    if (lane == 0) {
      v_out[s] = v;
      if (a.V) a.V[(int64_t)t * S + s] = v;
    }
    if (lane < A) {
      const int64_t i = ((int64_t)t * S + s) * A + lane;
      if (a.Q) a.Q[i] = q;
      if (pi_buf) pi_buf[i] = exp(q - v);
    }
  }
}

__global__ void __launch_bounds__(kThreads) k_mce_sweep(MceArgs a) {
  extern __shared__ double vs[];  // [S]: V[t+1] (backward)
  __shared__ double red[kWarps];
  cg::grid_group grid = cg::this_grid();
  const int G = gridDim.x, b = blockIdx.x;
  const int S = a.S, A = a.A, H = a.H;
  const int s0 = (int)((int64_t)S * b / G), s1 = (int)((int64_t)S * (b + 1) / G);
  const bool bwd = a.flags & IMB_MCE_BACKWARD, fwd = a.flags & IMB_MCE_FORWARD;

  if (bwd) {
    const double gamma = a.gam[0];
    for (int t = H - 1; t >= 0; --t) {
      double* v_next = a.vbuf + (t & 1) * S;         // V[t] written here
      const double* v_prev = a.vbuf + ((t + 1) & 1) * S;  // V[t+1]
      if (t < H - 1) {
        for (int j = threadIdx.x; j < S; j += kThreads) vs[j] = v_prev[j];
        __syncthreads();
      }
      backward_step(a, t, s0, s1, vs, gamma, v_next, a.pi);
      grid.sync();
    }
  }
  if (!fwd) return;

  double* __restrict__ D = a.D;
  const double* __restrict__ pi = a.pi;
  for (int s = s0 + threadIdx.x; s < s1; s += kThreads) D[s] = a.init[s];
  __syncthreads();
  for (int t = 0; t < H; ++t) {
    const double* __restrict__ Dt = D + (int64_t)t * S;
    double* __restrict__ my_part = a.part + ((int64_t)(t & 1) * G + b) * S;
    for (int j = threadIdx.x; j < S; j += kThreads) {
      double acc = 0.0;
      for (int s = s0; s < s1; ++s) {
        const double d = Dt[s];
        if (d == 0.0) continue;  // adds exact zeros only (T and pi are finite)
        const double* __restrict__ row = a.T + (int64_t)s * A * S + j;
        const double* __restrict__ ps = pi + ((int64_t)t * S + s) * A;
        for (int k = 0; k < A; ++k) acc = fma(d * ps[k], __ldg(row + (int64_t)k * S), acc);
      }
      my_part[j] = acc;
    }
    grid.sync();
    const double* __restrict__ parts = a.part + (int64_t)(t & 1) * G * S;
    double* __restrict__ Dn = D + (int64_t)(t + 1) * S;
    for (int s = s0 + threadIdx.x; s < s1; s += kThreads) {
      double acc = parts[s];
      for (int c = 1; c < G; ++c) acc += parts[(int64_t)c * S + s];
      Dn[s] = acc;
    }
    __syncthreads();
  }

  // Dcum = rollout.discounted_sum(D, gamma): a plain sum over t for gamma == 1, else polyval's Horner from t = H
  const double g = a.gam[1];
  double local_max = -INFINITY;
  for (int s = s0 + threadIdx.x; s < s1; s += kThreads) {
    double c;
    if (g == 1.0) {
      c = D[s];
      for (int t = 1; t <= H; ++t) c = __dadd_rn(c, D[(int64_t)t * S + s]);
    } else {
      c = __dadd_rn(D[(int64_t)H * S + s], __dmul_rn(g, 0.0));
      for (int t = H - 1; t >= 0; --t) c = __dadd_rn(D[(int64_t)t * S + s], __dmul_rn(c, g));
    }
    a.Dcum[s] = c;
    if (a.demo) {
      const double diff = c - a.demo[s];
      a.weights[s] = __double2float_rn(diff);
      local_max = nan_max(local_max, fabs(diff));
    }
  }
  if (!a.demo) return;
  for (int o = 16; o > 0; o >>= 1) {
    local_max = nan_max(local_max, __shfl_xor_sync(0xffffffffu, local_max, o));
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local_max;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = red[0];
    for (int w = 1; w < kWarps; ++w)
      m = nan_max(m, red[w]);
    a.cta_max[b] = m;
  }
  grid.sync();
  if (b == 0 && threadIdx.x == 0) {
    double m = a.cta_max[0];
    for (int c = 1; c < G; ++c)
      m = nan_max(m, a.cta_max[c]);
    *a.linf = m;
  }
}

struct MceLayout {
  int grid;
  int64_t vbuf, pi, D, part, cta_max, total;  // offsets in doubles
};

// Grid: one CTA per kWarps states (each warp of the backward owns at least one state), capped at what can be
// co-resident on the device (occupancy API), so that cooperative grid barriers are valid.
int mce_layout(int64_t S, int32_t A, int32_t H, int32_t flags, int32_t n_sms, MceLayout* L) {
  IMB_REQUIRE(flags == IMB_MCE_BACKWARD || flags == IMB_MCE_FORWARD || flags == (IMB_MCE_BACKWARD | IMB_MCE_FORWARD),
              "imb_mce: flags must be IMB_MCE_BACKWARD, IMB_MCE_FORWARD or both, got %d", flags);
  IMB_REQUIRE(S >= 1 && S <= IMB_MCE_MAX_STATES, "imb_mce: %lld states, the kernel takes 1 .. %d (V[t+1] is staged "
              "in shared memory)", (long long)S, IMB_MCE_MAX_STATES);
  IMB_REQUIRE(A >= 1 && A <= IMB_MCE_MAX_ACTIONS, "imb_mce: %d actions, the kernel takes 1 .. %d (one warp lane per "
              "action)", A, IMB_MCE_MAX_ACTIONS);
  IMB_REQUIRE(H >= 1 && H <= IMB_MCE_MAX_HORIZON, "imb_mce: horizon %d, the kernel takes 1 .. %d", H,
              IMB_MCE_MAX_HORIZON);
  const size_t smem = (size_t)S * sizeof(double);
  int per_sm = 0;
  if (n_sms <= 0) {
    n_sms = imb_num_sms();
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_mce_sweep, kThreads, smem) != cudaSuccess)
      IMB_FAIL(-2, "imb_mce: occupancy query failed: %s", cudaGetErrorString(cudaGetLastError()));
    IMB_REQUIRE(per_sm >= 1, "imb_mce: the sweep kernel cannot be resident with %zu bytes of shared memory", smem);
  } else {
    per_sm = 1;
  }
  const int64_t want = (S + kWarps - 1) / kWarps;
  const int64_t cap = (int64_t)per_sm * n_sms;
  L->grid = (int)(want < cap ? want : cap);
  const int64_t G = L->grid;
  const bool fwd = flags & IMB_MCE_FORWARD;
  int64_t o = 0;
  L->vbuf = o;
  o += 2 * S;
  L->pi = o;
  o += fwd && (flags & IMB_MCE_BACKWARD) ? (int64_t)H * S * A : 0;
  L->D = o;
  o += fwd ? (int64_t)(H + 1) * S : 0;
  L->part = o;
  o += fwd ? 2 * G * S : 0;
  L->cta_max = o;
  o += G;
  L->total = o;
  return 0;
}

}  // namespace

extern "C" {

int64_t imb_mce_plan(int64_t n_states, int32_t n_actions, int32_t horizon, int32_t flags, int32_t n_sms,
                             int32_t* grid_out) {
  MceLayout L;
  const int rc = mce_layout(n_states, n_actions, horizon, flags, n_sms, &L);
  if (rc != 0) return rc;
  if (grid_out) *grid_out = L.grid;
  return L.total;
}

int imb_mce_sweep(int64_t n_states, int32_t n_actions, int32_t horizon, int32_t flags,
                          const double* transition, const double* initial, const double* reward,
                          const float* reward32, const double* discounts, double* V, double* Q, double* pi, double* D,
                          double* Dcum, const double* demo_om, float* weights, double* linf, double* ws,
                          int64_t ws_doubles, void* stream) {
  MceLayout L;
  const int rc = mce_layout(n_states, n_actions, horizon, flags, 0, &L);
  if (rc != 0) return rc;
  const bool bwd = flags & IMB_MCE_BACKWARD, fwd = flags & IMB_MCE_FORWARD;
  IMB_REQUIRE(ws && ws_doubles >= L.total, "imb_mce_sweep: the workspace needs %lld doubles (imb_mce_plan), got %lld",
              (long long)L.total, (long long)ws_doubles);
  IMB_REQUIRE(discounts && (!bwd || transition), "imb_mce_sweep: null discounts or transition matrix");
  IMB_REQUIRE(!bwd || ((reward != nullptr) != (reward32 != nullptr)),
              "imb_mce_sweep: the backward sweep takes exactly one of reward (float64) and reward32 (float32)");
  IMB_REQUIRE(!fwd || (transition && initial && Dcum), "imb_mce_sweep: the forward sweep needs T, the initial "
              "distribution and Dcum");
  IMB_REQUIRE(bwd || pi, "imb_mce_sweep: a forward-only sweep reads the caller's pi");
  IMB_REQUIRE(!demo_om || (fwd && weights && linf), "imb_mce_sweep: the training outputs need the forward sweep, "
              "weights and linf");
  MceArgs a;
  a.S = (int)n_states;
  a.A = n_actions;
  a.H = horizon;
  a.flags = flags;
  a.T = transition;
  a.init = initial;
  a.r64 = reward;
  a.r32 = reward32;
  a.gam = discounts;
  a.V = V;
  a.Q = Q;
  a.pi = pi ? pi : (fwd ? ws + L.pi : nullptr);
  a.D = D ? D : ws + L.D;
  a.Dcum = Dcum;
  a.demo = demo_om;
  a.weights = weights;
  a.linf = linf;
  a.vbuf = ws + L.vbuf;
  a.part = ws + L.part;
  a.cta_max = ws + L.cta_max;
  void* args[] = {&a};
  const size_t smem = (size_t)n_states * sizeof(double);
  const cudaError_t e = cudaLaunchCooperativeKernel((const void*)k_mce_sweep, dim3(L.grid), dim3(kThreads), args, smem,
                                  (cudaStream_t)stream);
  if (e != cudaSuccess) IMB_FAIL(-2, "imb_mce_sweep: %s", cudaGetErrorString(e));
  return 0;
}

}  // extern "C"
