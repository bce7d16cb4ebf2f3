// imb_disc.cu -- stage 3 of the GAIL/AIRL round: the discriminator update, fused.
//
// Replaces (reference, /root/reference/src/imitation): rewards/reward_nets.py:441-457
// (BasicRewardNet.forward), :701-736 (ShapedRewardNet.forward), util/networks.py:79-134
// (RunningNorm), algorithms/adversarial/common.py:353-372 (BCE-with-logits, backward, Adam)
// and :27-92 (compute_train_stats).
//
// Kernel plan (no spinning grid barriers -- every dependency is a kernel boundary or the
// "last block done" ticket, so a bug cannot hang the GPU):
//   k_norm_stats   per-chunk (n, mean, M2) per input feature of 1-3 normaliser updates (blockIdx.y = job);
//                  the last CTA Chan-merges each job's chunks in fixed order and folds the jobs, in order,
//                  into their running stats (RunningNorm.update_stats).
//   k_disc_fwdbwd<R>  the fp32-FFMA form (k_disc_fwdbwd_tc in imb_disc_tc.cuh is the tensor-core one):
//                  persistent CTAs of R threads over R-row tiles (R = 128 or 256) of the feature-major batch.  A
//                  tile's feature rows arrive in shared memory by cp.async.bulk on an mbarrier; the next tile's
//                  copy is issued once the last forward that reads them is done.  Per pass, the inputs are
//                  normalised into a feature-major tile and the hidden layers run as register-tiled GEMMs
//                  (tile_layer, imb_tile.cuh); the head's dot product gives each row's logit.  Per row:
//                  BCE-with-logits (or the caller's dL/dlogit) and the statistics.  Backward, last pass first
//                  (earlier passes are recomputed): dL/dz1 by gemm_acc, then the weight-gradient contractions
//                  dW = D^T . Act (wgrad_tile) into per-slice shared-memory accumulators that leave the CTA as
//                  one partial vector.  Weights stay in shared memory; activations never touch HBM.
//   k_disc_reduce  warp-per-parameter deterministic sum of the per-CTA partials (G = meta[0], written by
//                  the fwd/bwd kernel).
//   k_disc_adam    torch.optim.Adam step + the 9 train statistics.
//   k_disc_reduce_adam  both in one launch: the last block (ticket) runs the Adam step and the statistics.
#include <stdlib.h>

#include <algorithm>

#include "imb_common.cuh"
#include "imb_mlp.cuh"
#include "imb_tile.cuh"

thread_local char g_imb_err[512] = {0};

extern "C" int imb_version(void) { return 1; }
extern "C" const char* imb_last_error(void) { return g_imb_err; }

namespace {

constexpr int NORM_CHUNK = 512;       // rows per CTA in k_norm_stats
constexpr int NORM_PS = 2 * IMB_MAX_DIN + 4;  // floats per chunk record of k_norm_stats: mean | M2 | n
constexpr int MAXG = 296;             // max CTAs of k_disc_fwdbwd (2 per SM)

// ---- workspace layout (floats) -----------------------------------------------------------------
struct WsLayout {
  int64_t gacc;      // [P] accumulated gradient
  int64_t stats;     // [16] reduced sums of the last minibatch
  int64_t meta;      // [16] ints: grid of the last fwdbwd launch, n rows, n_expert
  int64_t snap;      // [2*IMB_MAX_DIN] potential-norm stats after the first (next_obs) update
  int64_t ticket;    // [16] uint tickets
  int64_t normpart;  // [MAXCHUNKS][NORM_PS]
  int64_t partial;   // [MAXG][P + 16]
  int64_t total;
};
constexpr int MAXCHUNKS = 16384;  // up to 8M rows per norm launch
__host__ __device__ inline int64_t part_stride(int P) { return (int64_t)((P + 16 + 31) / 32) * 32; }
inline WsLayout ws_layout(int P) {
  WsLayout w;
  int64_t o = 0;
  w.gacc = o;
  o += (P + 31) / 32 * 32;
  w.stats = o;
  o += 32;
  w.meta = o;
  o += 32;
  w.snap = o;
  o += 2 * IMB_MAX_DIN;
  w.ticket = o;
  o += 32;
  w.normpart = o;
  o += (int64_t)MAXCHUNKS * NORM_PS;
  w.partial = o;
  o += (int64_t)MAXG * part_stride(P);
  w.total = o;
  return w;
}

// ---- RunningNorm statistics ----------------------------------------------------------------------
// One or more RunningNorm updates over the same batch rows (AIRL: the base net's normaliser and the potential's, the
// latter updated twice: first with next_obs, then with obs -- reward_nets.py:708-710).
struct NormJob {
  int din;
  short row[IMB_MAX_DIN];  // batch feature rows
  float* rmv;              // running [mean | var] of the job's normaliser
  int32_t* cnt;
  float* snap;             // optional copy of the statistics after this job's fold
};
struct NormJobs {
  int njobs;  // 1..3
  NormJob job[3];
};

// blockIdx.y = job, blockIdx.x = chunk of chunk_rows rows; warp w handles features w, w+nw, ...: exact two-pass
// (mean, M2) inside the chunk.  The last CTA of the whole grid Chan-merges each job's chunks in index order and folds
// the jobs into their running statistics IN JOB ORDER (two jobs may share a normaliser), exactly as
// util/networks.py:111-134 does.  Deferred mode (`defer`): the batch moments go to the next free slot of `defer`
// ([0] = slot counter, slots of 2 * din + 1 floats: mean | biased variance | n) instead of into the running
// statistics; k_norm_fold applies them later, in order.  Six resident CTAs per SM hold it at 40 registers (left
// alone, ptxas spends 60 on the unrolled chunk merge).
__global__ void __launch_bounds__(256, 6) k_norm_stats(NormJobs J, const float* __restrict__ batch, int64_t ld,
                                                       int64_t n, int chunk_rows, float* __restrict__ part,
                                                       unsigned int* __restrict__ ticket, float* __restrict__ defer,
                                                       int defer_cap) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int nchunks = gridDim.x;
  const NormJob& L = J.job[blockIdx.y];
  const int64_t r0 = (int64_t)blockIdx.x * chunk_rows;
  const int cn = (int)(min(n, r0 + (int64_t)chunk_rows) - r0);
  float* my = part + ((int64_t)blockIdx.y * nchunks + blockIdx.x) * NORM_PS;
  for (int k = warp; k < L.din; k += nw) {
    float mean, m2;
    warp_moments(batch + (int64_t)L.row[k] * ld + r0, cn, lane, mean, m2);
    if (lane == 0) {
      my[k] = mean;
      my[IMB_MAX_DIN + k] = m2;
    }
  }
  if (threadIdx.x == 0) my[2 * IMB_MAX_DIN] = (float)cn;
  __threadfence();
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int jb = 0; jb < J.njobs; ++jb) {
    const NormJob& Lj = J.job[jb];
    const float* jpart = part + (int64_t)jb * nchunks * NORM_PS;
    float* slot = nullptr;
    if (defer) {
      int s = (int)defer[0];
      if (s >= defer_cap) s = defer_cap - 1;  // a full list: the last slot is overwritten (the host folds before this)
      slot = defer + 4 + (int64_t)s * (2 * Lj.din + 1);
    }
    const int32_t old_count = defer ? 0 : *Lj.cnt;
    for (int k = warp; k < Lj.din; k += nw) {
      float b_n, b_mean, b_m2;
      warp_chan_merge(jpart + 2 * IMB_MAX_DIN, jpart + k, jpart + IMB_MAX_DIN + k, NORM_PS, nchunks, lane, b_n, b_mean,
                      b_m2);
      if (lane == 0 && slot) {
        slot[k] = b_mean;
        slot[Lj.din + k] = b_m2 / b_n;
      } else if (lane == 0) {
        float mean = Lj.rmv[k], var = Lj.rmv[Lj.din + k];
        norm_fold(mean, var, (float)old_count, b_mean, b_m2 / b_n, b_n);
        Lj.rmv[k] = mean;
        Lj.rmv[Lj.din + k] = var;
        if (Lj.snap) {
          Lj.snap[k] = mean;
          Lj.snap[Lj.din + k] = var;
        }
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (slot) {
        slot[2 * Lj.din] = (float)n;
        if (defer[0] < (float)defer_cap) defer[0] += 1.0f;  // saturates at defer_cap: a fold never reads past the list
      } else {
        *Lj.cnt = old_count + (int32_t)n;
      }
    }
    __syncthreads();  // the next job may fold into the same normaliser: count and statistics are in place
  }
  if (threadIdx.x == 0) *ticket = 0u;  // re-arm for the next launch
}

// fold the deferred batch moments into the running statistics, slot by slot, with RunningNorm.update_stats'
// arithmetic (util/networks.py:121-134)
__global__ void k_norm_fold(int din, float* __restrict__ defer, float* __restrict__ run_mean_var,
                            int32_t* __restrict__ count, int k_fixed) {
  const int K = k_fixed > 0 ? k_fixed : (int)defer[0];
  const int k = threadIdx.x;
  int32_t cnt_i = *count;
  if (k < din) {
    float mean = run_mean_var[k], var = run_mean_var[din + k];
    int32_t c = cnt_i;
    for (int sidx = 0; sidx < K; ++sidx) {
      const float* slot = defer + 4 + (int64_t)sidx * (2 * din + 1);
      const float b_n = slot[2 * din];
      norm_fold(mean, var, (float)c, slot[k], slot[din + k], b_n);
      c += (int32_t)b_n;
    }
    run_mean_var[k] = mean;
    run_mean_var[din + k] = var;
  }
  __syncthreads();
  if (k == 0) {
    for (int sidx = 0; sidx < K; ++sidx) cnt_i += (int32_t)defer[4 + (int64_t)sidx * (2 * din + 1) + 2 * din];
    *count = cnt_i;
    if (k_fixed <= 0) defer[0] = 0.f;
  }
}

// ---- the fused forward / BCE / backward kernel (tiled-GEMM form, see imb_tile.cuh) ------------------
// One weight-gradient contraction over the R-row tile, by the `gthreads` threads of a contraction group (tgw = this
// thread's index in it):  dW[j][i] += sum_r D[j][r] * ACT[i][r],  db[j] += sum_r D[j][r]  for j < nj, i < ni, into
// the parameter vector's [off_w, off_w + nj * ni) and [off_b, off_b + nj).  The (JP / 32) x (IP / 32) blocks of 32 x 32
// take a warp each (wgrad_acc); when the group has threads to spare, the tile's rows are split into slices whose
// accumulators are private (slice s at AW + s * P).  MASK: D = dL/dz2 generated from H2 and the upstream g as in
// wgrad_acc, with per-j scale wf.
template <int R, bool MASK>
__device__ __forceinline__ void wgrad_tile(float* AW, int P, int nsl, int tgw, int gthreads, int JP, int IP,
                                           const float* D, const float* ACT, const float* g, const float* wf, int nj,
                                           int ni, int off_w, int off_b) {
  constexpr int RS = R + TILE_PAD;
  const int lane = threadIdx.x & 31, jl = lane & 7, il = lane >> 3;
  const int nblk = (JP / 32) * (IP / 32), ntl = nblk * 32;
  const int slices = min(gthreads / ntl, nsl);
  const int lt = tgw % ntl, sl = tgw / ntl, blk = lt >> 5;
  const int jb = (blk % (JP / 32)) * 32, ib = (blk / (JP / 32)) * 32;
  float acc[4][8], bacc[4], sj[4];
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    bacc[jj] = 0.f;
    sj[jj] = MASK ? wf[jb + jl + 8 * jj] : 0.f;
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) acc[jj][ii] = 0.f;
  }
  const int rows = R / slices;
  if (sl < slices) wgrad_acc<MASK>(acc, bacc, D, ACT, RS, jb + jl, ib + il, sl * rows, (sl + 1) * rows, g, sj);
  float* A = AW + (sl < slices ? sl : 0) * P;
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = jb + jl + 8 * jj;
    if (j < nj) {
#pragma unroll
      for (int ii = 0; ii < 8; ++ii) {
        const int i = ib + il + 4 * ii;
        if (i < ni) A[off_w + j * ni + i] += acc[jj][ii];
      }
      if (il == 0 && ib == 0) A[off_b + j] += bacc[jj];
    }
  }
}

// Dynamic shared memory (floats):
//   [image per pass][AW: 4 slices x P][stage: nstage x RS][XN: KP x RS][H1, H2, DZ1: JP x RS each]
//   [lg, gv, gp, dv, lpv: R each]
template <int R>
__global__ void __launch_bounds__(R, 256 / R) k_disc_fwdbwd(const DiscLaunch L, const float* __restrict__ params,
                                                      const float* __restrict__ batch, int64_t ld, int64_t n,
                                                      int64_t n_expert, float loss_scale,
                                                      const float* __restrict__ grad_out,
                                                      float* __restrict__ logits_out, float* __restrict__ partial,
                                                      int* __restrict__ meta, int JP, int KP, int img_sz, int aw_off, int st_off, int xn_off,
                                                      int t_off, int v_off, int nsl) {
  // one thread per tile row: R threads, warp w -> column group w % 4 (8 columns) and row half w / 4
  constexpr int RS = R + TILE_PAD;
  extern __shared__ __align__(128) float smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ float red[64];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cg = warp & 3, grp = warp >> 2, tg = tid & 127;
  float* AW = smem + aw_off;
  float* xs = smem + st_off;
  float* XN = smem + xn_off;
  float* H1 = smem + t_off;
  float* H2 = H1 + JP * RS;
  float* DZ1 = H2 + JP * RS;
  float* lg = smem + v_off;
  float* gv = lg + R;
  float* gp = gv + R;
  float* dv = gp + R;
  float* lpv = dv + R;
  const int P = L.P;

  for (int p = 0; p < L.npass; ++p)
    load_timg(smem + p * img_sz, L.pass[p], JP, params, L.pass[p].has_norm ? L.pass[p].norm : nullptr, L.pass[p].eps);
  for (int i = tid; i < nsl * P; i += R) AW[i] = 0.f;
  if (tid == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
    if (blockIdx.x == 0) {  // launch record for k_disc_reduce / k_disc_adam (stats of the LAST minibatch)
      meta[0] = (int)gridDim.x;
      meta[1] = (int)n;
      meta[2] = (int)n_expert;
      reinterpret_cast<float*>(meta)[3] = loss_scale;
    }
  }
  __syncthreads();

  const int64_t ntiles = (n + R - 1) / R;
  auto issue = [&](int64_t tile) {
    int64_t cnt = ld - tile * R;  // floats available in each feature row from this tile's start
    if (cnt > R) cnt = R;
    mbar_expect_tx(&bar, (uint32_t)(L.nstage * cnt * 4));
    for (int s = 0; s < L.nstage; ++s)
      bulk_g2s(xs + s * RS, batch + (int64_t)L.stage_row[s] * ld + tile * R, (uint32_t)(cnt * 4), &bar);
  };
  uint32_t phase = 0;
  if (tid == 0 && (int64_t)blockIdx.x < ntiles) issue(blockIdx.x);

  const int r0 = grp * 128 + lane * 4;  // this thread's row quad in the register-tiled GEMMs
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float s_loss = 0.f, s_ent = 0.f;
  int c_exp = 0, c_gen = 0, c_pred_exp = 0;

  // one MLP forward over the tile for pass `p`: builds XN, H1, H2 and returns nothing; the per-row
  // output is accumulated into lg[] (scaled by the pass coefficient) when `accumulate` is set.
  auto forward_pass = [&](int p, int nv, bool accumulate, bool first) {
    const PassDesc& Pd = L.pass[p];
    const float* img = smem + p * img_sz;
    const int din = Pd.din;
    const float* mean = img + TImg::mean(din, JP);
    const float* istd = img + TImg::istd(din, JP);
    // normalised inputs, feature-major; rows >= nv and features >= din are zero
    for (int i = tid; i < KP * (R / 4); i += R) {
      const int k = i / (R / 4), r4 = (i - k * (R / 4)) * 4;
      float4 v = zero4;
      if (k < din) {
        const float4 x = ld4(xs + Pd.in_slot[k] * RS + r4);
        const float m = mean[k], is = istd[k];
        v.x = (r4 + 0 < nv) ? (x.x - m) * is : 0.f;
        v.y = (r4 + 1 < nv) ? (x.y - m) * is : 0.f;
        v.z = (r4 + 2 < nv) ? (x.z - m) * is : 0.f;
        v.w = (r4 + 3 < nv) ? (x.w - m) * is : 0.f;
      }
      st4(XN + k * RS + r4, v);
    }
    __syncthreads();
    const float* HL = XN;
    int hl = din;
    if (Pd.n_hidden >= 1) {
      tile_layer<ACT_RELU, 4, R>(XN, din, img + TImg::w1t(din, JP), JP, img + TImg::b1(din, JP), H1, JP);
      __syncthreads();
      HL = H1;
      hl = Pd.h1;
    }
    if (Pd.n_hidden >= 2) {
      tile_layer<ACT_RELU, 4, R>(H1, Pd.h1, img + TImg::w2t(din, JP), JP, img + TImg::b2(din, JP), H2, JP);
      __syncthreads();
      HL = H2;
      hl = Pd.h2;
    }
    if (accumulate) {
      const float* wf = img + TImg::wf(din, JP);
      const float bf = img[TImg::bf(din, JP)];
      for (int r = tid; r < R; r += R) {
        float o = bf;
        for (int j = 0; j < hl; ++j) o = fmaf(wf[j], HL[j * RS + r], o);
        const float c = pass_coef(Pd.coef_kind, L.gamma, dv[r]);
        lg[r] = first ? c * o : fmaf(c, o, lg[r]);
      }
      __syncthreads();
    }
  };

  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    mbar_wait(&bar, phase);
    phase ^= 1u;
    const int nv = (int)min((int64_t)R, n - tile * R);
    for (int r = tid; r < R; r += R) {
      dv[r] = (L.done_slot >= 0 && r < nv) ? xs[L.done_slot * RS + r] : 0.f;
      lpv[r] = (L.logp_slot >= 0 && r < nv) ? xs[L.logp_slot * RS + r] : 0.f;
    }
    __syncthreads();
    // ---- logits: forward over all passes (the last pass's tiles stay valid for its backward) -------
    for (int p = 0; p < L.npass; ++p) forward_pass(p, nv, true, p == 0);
    // stage is free once the last forward that reads it is done -- unless passes are recomputed below
    const bool recompute = L.npass > 1;
    const int64_t next = tile + gridDim.x;
    if (!recompute && tid == 0 && next < ntiles) issue(next);
    // ---- dL/dlogit per row + statistics -------------------------------------------------------------
    for (int r = tid; r < R; r += R) {
      float g = 0.f;
      if (r < nv) {
        const int64_t row = tile * R + r;
        const float logit = lg[r] - lpv[r];
        if (logits_out) logits_out[row] = logit;
        if (grad_out) {
          g = grad_out[row];
        } else {
          const float y = (row < n_expert) ? 1.f : 0.f;
          const float sg = sigmoid_f(logit);
          const float sp = fmaxf(logit, 0.f) + log1pf(expf(-fabsf(logit)));
          s_loss += sp - logit * y;
          s_ent += sp - logit * sg;
          const bool pred_exp = !(logit < 0.f);
          c_pred_exp += pred_exp;
          if (y > 0.5f) c_exp += pred_exp; else c_gen += !pred_exp;
          g = (sg - y) * loss_scale;
        }
      }
      gv[r] = g;
    }
    __syncthreads();

    // ---- backward + weight gradients, pass by pass ---------------------------------------------------
    for (int pi = 0; pi < L.npass; ++pi) {
      const int p = L.npass - 1 - pi;  // last pass first: its forward tiles are still in shared memory
      if (pi > 0) forward_pass(p, nv, false, false);
      if (recompute && pi == L.npass - 1 && tid == 0 && next < ntiles) issue(next);
      const PassDesc& Pd = L.pass[p];
      const float* img = smem + p * img_sz;
      const int din = Pd.din;
      const float* wf = img + TImg::wf(din, JP);
      for (int r = tid; r < R; r += R) gp[r] = gv[r] * pass_coef(Pd.coef_kind, L.gamma, dv[r]);
      __syncthreads();
      const int h1w = Pd.h1, h2w = Pd.h2;
      const int off_w1 = Pd.param_off, off_b1 = off_w1 + h1w * din, off_w2 = off_b1 + h1w;
      const int off_b2 = off_w2 + ((Pd.n_hidden == 2) ? h2w * h1w : 0);
      const int off_wf = (Pd.n_hidden == 2) ? off_b2 + h2w : (Pd.n_hidden == 1 ? off_w2 : Pd.param_off);
      const int hl = (Pd.n_hidden == 2) ? h2w : (Pd.n_hidden == 1 ? h1w : din);
      const float* HL = (Pd.n_hidden == 2) ? H2 : (Pd.n_hidden == 1 ? H1 : XN);
      // dL/dz1 tile
      if (Pd.n_hidden == 2) {
        const float4 g = ld4(gp + r0);
        for (int jh = 0; jh < JP / 32; ++jh) {
          const int i0 = jh * 32 + cg * 8;
          float acc[4][8];
#pragma unroll
          for (int x = 0; x < 4; ++x)
#pragma unroll
            for (int t = 0; t < 8; ++t) acc[x][t] = 0.f;
          gemm_acc(acc, H2, RS, r0, img + TImg::w2(din, JP), JP, i0, h2w, g, wf);
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const float4 h = ld4(H1 + (i0 + t) * RS + r0);
            st4(DZ1 + (i0 + t) * RS + r0, make_float4(h.x > 0.f ? acc[0][t] : 0.f, h.y > 0.f ? acc[1][t] : 0.f,
                                                      h.z > 0.f ? acc[2][t] : 0.f, h.w > 0.f ? acc[3][t] : 0.f));
          }
        }
      } else if (Pd.n_hidden == 1) {
        for (int i = tid; i < JP * (R / 4); i += R) {
          const int j = i / (R / 4), r4 = (i - j * (R / 4)) * 4;
          const float4 h = ld4(H1 + j * RS + r4), g = ld4(gp + r4);
          const float w = wf[j];
          st4(DZ1 + j * RS + r4, make_float4(h.x > 0.f ? g.x * w : 0.f, h.y > 0.f ? g.y * w : 0.f,
                                             h.z > 0.f ? g.z * w : 0.f, h.w > 0.f ? g.w * w : 0.f));
        }
      }
      __syncthreads();
      // weight gradients: a group of 4 warps (128 threads) per contraction; with two groups (R = 256)
      // dW2 and dW1 run concurrently, each split into row slices with private accumulators.
      constexpr int NGRP = R / 128;
      // R = 256: two 128-thread groups run dW2 and dW1 concurrently (4 row slices each).
      // R = 128: 32-wide nets split the CTA 64/64 (dW2 | dW1, 2 slices each); otherwise sequential.
      const bool split64 = (NGRP == 1) && JP == 32 && Pd.n_hidden == 2;
      const int wg = split64 ? (tid >> 6) : grp;        // which contraction group this thread is in
      const int tgw = split64 ? (tid & 63) : tg;        // thread index inside the group
      const int gthreads = split64 ? 64 : 128;
      const bool do_w2 = Pd.n_hidden == 2 && ((NGRP == 1 && !split64) || wg == 0);
      const bool do_w1 = Pd.n_hidden >= 1 && ((NGRP == 1 && !split64) || wg == (Pd.n_hidden == 2 ? 1 : 0));
      if (do_w2) wgrad_tile<R, true>(AW, P, nsl, tgw, gthreads, JP, JP, H2, H1, gp, wf, h2w, h1w, off_w2, off_b2);
      if (do_w1) wgrad_tile<R, false>(AW, P, nsl, tgw, gthreads, JP, KP, DZ1, XN, nullptr, nullptr, h1w, din, off_w1, off_b1);
      // dwf / dbf: thread j sums its feature row against gp (slice 1 accumulators keep owners unique)
      {
        float* A = AW + 1 * P;
        for (int j = tid; j <= hl; j += R) {
          float acc = 0.f;
          if (j < hl) {
            for (int r = 0; r < R; r += 4) {
              const float4 h = ld4(HL + j * RS + r), g = ld4(gp + r);
              acc = fmaf(h.x, g.x, acc);
              acc = fmaf(h.y, g.y, acc);
              acc = fmaf(h.z, g.z, acc);
              acc = fmaf(h.w, g.w, acc);
            }
          } else {
            for (int r = 0; r < R; r += 4) {
              const float4 g = ld4(gp + r);
              acc += (g.x + g.y) + (g.z + g.w);
            }
          }
          A[off_wf + j] += acc;
        }
      }
      __syncthreads();
    }
  }

  // ---- per-CTA partials: gradients (slices summed in fixed order) + statistics ----------------------
  float* my = partial + (int64_t)blockIdx.x * part_stride(P);
  for (int i = tid; i < P; i += R) {
    float v = AW[i];
    for (int s2 = 1; s2 < nsl; ++s2) v += AW[s2 * P + i];
    my[i] = v;
  }
  s_loss = warp_sum(s_loss);
  s_ent = warp_sum(s_ent);
  c_exp = warp_sum_i(c_exp);
  c_gen = warp_sum_i(c_gen);
  c_pred_exp = warp_sum_i(c_pred_exp);
  if (lane == 0) {
    red[warp * 5 + 0] = s_loss;
    red[warp * 5 + 1] = s_ent;
    red[warp * 5 + 2] = (float)c_exp;
    red[warp * 5 + 3] = (float)c_gen;
    red[warp * 5 + 4] = (float)c_pred_exp;
  }
  __syncthreads();
  if (tid < 5) {
    float v = 0.f;
    for (int w = 0; w < R / 32; ++w) v += red[w * 5 + tid];
    my[P + tid] = v;
  }
}

}  // namespace
#include "imb_disc_tc.cuh"
namespace {

// ---- deterministic reduction of the per-CTA partials, Adam step, train statistics -------------
// The partials are those of the last fwd/bwd launch on this workspace, which records its grid size G in meta[0].

// warp per parameter (and per statistic): lanes stride over the G partial rows, shuffle-reduce.  The gradient sums are
// added to gacc (and copied to grad_out_flat), the statistic sums replace stats.
__device__ __forceinline__ void reduce_partials(int P, const int* meta, const float* partial, float* gacc, float* stats,
                                                float* grad_out_flat) {
  const int G = meta[0];
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int64_t ps = part_stride(P);
  for (int p = gw; p < P + 5; p += nwarps) {
    float acc = 0.f;
    for (int c = lane; c < G; c += 32) acc += partial[(int64_t)c * ps + p];
    acc = warp_sum(acc);
    if (lane == 0) {
      if (p < P) {
        const float v = gacc[p] + acc;
        gacc[p] = v;
        if (grad_out_flat) grad_out_flat[p] = v;
      } else {
        stats[p - P] = acc;  // statistics of the LAST minibatch only (common.py:376-381)
      }
    }
  }
}

// beta^n for an integer step count by repeated squaring (pow(double, double) costs microseconds on one thread)
__device__ __forceinline__ double dpowi(double b, int64_t n) {
  double r = 1.0;
  while (n > 0) {
    if (n & 1) r *= b;
    b *= b;
    n >>= 1;
  }
  return r;
}

// kThisLaunch: the value was written by other blocks of the same launch, so it is read past L1
template <bool kThisLaunch>
__device__ __forceinline__ float ld_sum(const float* p) {
  return kThisLaunch ? __ldcg(p) : *p;
}

// torch.optim.Adam step (AdamW's decoupled decay when weight_decay > 0) of params[0, P) by the threads of one block,
// with gradient grad / grad_div.  Thread 0 alone reads and increments the step count; the other threads take the bias
// corrections from shared memory (no race, no extra launch).
template <bool kThisLaunch>
__device__ __forceinline__ void adam_step(int P, const imb_adam& opt, float* params, float* m, float* v,
                                          const float* grad, float grad_div, int64_t* step_io) {
  // bias corrections in double like torch's Python-scalar arithmetic (torch/optim/adam.py)
  __shared__ float s_bc[2];
  if (threadIdx.x == 0) {
    const int64_t step = *step_io + 1;
    const double bc1d = 1.0 - dpowi((double)opt.beta1, step);
    const double bc2d = 1.0 - dpowi((double)opt.beta2, step);
    s_bc[0] = (float)((double)opt.lr / bc1d);
    s_bc[1] = (float)sqrt(bc2d);
    *step_io = step;
  }
  __syncthreads();
  const float step_size = s_bc[0], bc2_sqrt = s_bc[1];
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const float g = ld_sum<kThisLaunch>(grad + i) / grad_div;
    const float mi = m[i] + (g - m[i]) * (1.0f - opt.beta1);        // torch: exp_avg.lerp_(grad, 1-beta1)
    const float vi = v[i] * opt.beta2 + (1.0f - opt.beta2) * g * g;  // exp_avg_sq.mul_(b2).addcmul_(g,g,1-b2)
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + opt.eps;
    const float pw = opt.weight_decay > 0.f ? params[i] * (1.0f - opt.lr * opt.weight_decay) : params[i];  // AdamW
    params[i] = pw - step_size * (mi / denom);
  }
}

// the 9 train statistics of the last minibatch (common.py:27-92) from its sums and the row counts in meta; one thread
template <bool kThisLaunch>
__device__ __forceinline__ void train_stats(const float* stats, const int* meta, float* stats_out) {
  const float n = (float)meta[1], n_exp = (float)meta[2], n_gen = n - n_exp;
  const float loss_sum = ld_sum<kThisLaunch>(stats + 0), ent_sum = ld_sum<kThisLaunch>(stats + 1),
              c_exp = ld_sum<kThisLaunch>(stats + 2), c_gen = ld_sum<kThisLaunch>(stats + 3),
              c_pred = ld_sum<kThisLaunch>(stats + 4);
  const float nanv = __int_as_float(0x7fc00000);
  stats_out[0] = loss_sum * reinterpret_cast<const float*>(meta)[3];  // disc_loss (scaled minibatch mean)
  stats_out[1] = n > 0 ? (c_exp + c_gen) / n : nanv;                  // disc_acc
  stats_out[2] = n_exp >= 1 ? c_exp / n_exp : nanv;                   // disc_acc_expert
  stats_out[3] = c_gen / fmaxf(1.f, n_gen);                           // disc_acc_gen
  stats_out[4] = n > 0 ? ent_sum / n : nanv;                          // disc_entropy
  stats_out[5] = n > 0 ? n_exp / n : nanv;                            // disc_proportion_expert_true
  stats_out[6] = n > 0 ? c_pred / n : nanv;                           // disc_proportion_expert_pred
  stats_out[7] = n_exp;
  stats_out[8] = n_gen;
}

__global__ void __launch_bounds__(256) k_disc_reduce(int P, const int* __restrict__ meta,
                                                    const float* __restrict__ partial, float* __restrict__ gacc,
                                                    float* __restrict__ stats, float* __restrict__ grad_out_flat) {
  reduce_partials(P, meta, partial, gacc, stats, grad_out_flat);
}

// single block: P <= ~8.5k parameters = a handful of iterations per thread
__global__ void __launch_bounds__(1024) k_disc_adam(int P, imb_adam opt, float* __restrict__ params,
                                                  float* __restrict__ m, float* __restrict__ v,
                                                  const float* __restrict__ grad, float grad_div,
                                                  const float* __restrict__ stats, const int* __restrict__ meta,
                                                  int64_t* __restrict__ step_io,
                                                  float* __restrict__ stats_out) {
  adam_step<false>(P, opt, params, m, v, grad, grad_div, step_io);
  if (threadIdx.x == 0 && stats_out) train_stats<false>(stats, meta, stats_out);
}

// reduce + Adam in one launch (the last minibatch of an update): every block reduces its share of the partials
// like k_disc_reduce; the last block to finish (ticket) runs the optimiser step and the statistics.
__global__ void __launch_bounds__(256) k_disc_reduce_adam(int P, const float* __restrict__ partial,
                                                         float* __restrict__ gacc, float* __restrict__ stats,
                                                         imb_adam opt, float* __restrict__ params,
                                                         float* __restrict__ m, float* __restrict__ v, float grad_div,
                                                         const int* __restrict__ meta, int64_t* __restrict__ step_io,
                                                         float* __restrict__ stats_out,
                                                         unsigned int* __restrict__ ticket) {
  reduce_partials(P, meta, partial, gacc, stats, nullptr);
  __threadfence();
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x == 0) *ticket = 0u;  // re-arm for the next launch
  adam_step<true>(P, opt, params, m, v, gacc, grad_div, step_io);
  if (threadIdx.x == 0 && stats_out) train_stats<true>(stats, meta, stats_out);
}

// ---- regularization of the reward model's training step (imb_param_regularize) --------------------------------------
// x^k for an integer k >= 0 by repeated squaring in float32
__device__ __forceinline__ float powi_f(float x, int k) {
  float r = 1.f;
  while (k > 0) {
    if (k & 1) r *= x;
    x *= x;
    k >>= 1;
  }
  return r;
}

// Single block, like k_disc_adam.  IMB_REG_LP: gacc += coeff * p sign(w) |w|^(p-1) and, when stats is given,
// stats[0] += coeff * sum |w|^p, stats[2] += 1 -- the sum in a fixed order (per-thread strided sums, then a fixed
// shuffle tree and warp order), so two launches give the same bits.  IMB_REG_WEIGHT_DECAY: w = w + coeff * w as two
// separately rounded ops (torch's th.add(w, c * w)).
__global__ void __launch_bounds__(1024) k_param_regularize(int P, int kind, int p, float coeff,
                                                         float* __restrict__ params, float* __restrict__ gacc,
                                                         float* __restrict__ stats) {
  if (kind == IMB_REG_WEIGHT_DECAY) {
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
      const float w = params[i];
      params[i] = __fadd_rn(w, __fmul_rn(coeff, w));
    }
    return;
  }
  const float fp = (float)p;
  float s = 0.f;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const float w = params[i], a = fabsf(w);
    const float a_pm1 = powi_f(a, p - 1);  // |w|^(p-1); 1 for p = 1
    const float g = w > 0.f ? fp * a_pm1 : (w < 0.f ? -fp * a_pm1 : 0.f);  // d |w|^p / dw, 0 at w = 0
    gacc[i] = __fadd_rn(gacc[i], __fmul_rn(coeff, g));
    s += a_pm1 * a;
  }
  if (!stats) return;
  __shared__ float s_part[32];
  s = warp_sum(s);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) s_part[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_part[w];
    stats[0] += coeff * t;
    stats[2] += 1.f;
  }
}

// ---- preference comparisons: fragment returns -> Boltzmann probability -> cross entropy (+ its gradient) -------------
// PreferenceModel.probability (algorithms/preference_comparisons.py:487-530) from the (discounted) return difference
// s = sum_t g^t (r2 - r1): d = clip(s, -threshold, threshold), m = 1 / (1 + e^d), p = noise / 2 + (1 - noise) m.
// k_pref_loss also needs e^d, m and whether s was clipped for its gradient.
struct PrefProb {
  float ed, m, p;
  bool clipped;
};
__device__ __forceinline__ PrefProb pref_probability(float s, float noise_prob, float threshold) {
  PrefProb q;
  q.clipped = s < -threshold || s > threshold;
  const float d = fminf(fmaxf(s, -threshold), threshold);
  q.ed = expf(d);
  q.m = 1.0f / (1.0f + q.ed);
  q.p = noise_prob * 0.5f + (1.0f - noise_prob) * q.m;
  return q;
}

// Warp per fragment pair: lanes stride over the L time steps (coalesced: a fragment's rewards are contiguous), shuffle
// reduction of the discounted difference, lane-parallel write of the 2 L gradient entries.  The minibatch sums (loss,
// accuracy) are accumulated per CTA and added to the statistics accumulator with one atomic each; a minibatch is a few
// hundred pairs, so the order-dependent rounding of those atomics only touches the logged means (1e-7 relative).
__global__ void __launch_bounds__(256) k_pref_loss(const float* __restrict__ rews, int P, int L,
                                                  const float* __restrict__ prefs, float noise_prob, float discount,
                                                  float threshold, float grad_scale, float* __restrict__ grad_rews,
                                                  float* __restrict__ probs_out, float* __restrict__ stats_acc) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __shared__ float s_loss[8], s_acc[8];
  float w_loss = 0.f, w_acc = 0.f;
  const float inv_P = 1.0f / (float)P;
  for (int pr = blockIdx.x * nw + warp; pr < P; pr += gridDim.x * nw) {
    const float* r1 = rews + (int64_t)pr * L;
    const float* r2 = rews + ((int64_t)P + pr) * L;
    float s = 0.f;
    if (discount == 1.0f) {
      for (int t = lane; t < L; t += 32) s += r2[t] - r1[t];
    } else {
      for (int t = lane; t < L; t += 32) s = fmaf(powf(discount, (float)t), r2[t] - r1[t], s);
    }
    s = warp_sum(s);
    const PrefProb q = pref_probability(s, noise_prob, threshold);
    const bool clipped = q.clipped;  // th.clip passes the gradient on [min, max] only
    const float ed = q.ed, m = q.m, p = q.p;
    const float y = prefs[pr];
    // F.binary_cross_entropy: logs clamped at -100; backward (p - y) / max(p (1 - p), 1e-12)
    const float lp = fmaxf(logf(p), -100.0f), l1p = fmaxf(log1pf(-p), -100.0f);
    const float loss = -(y * lp + (1.0f - y) * l1p);
    const float dl_dp = (p - y) / fmaxf(p * (1.0f - p), 1e-12f) * inv_P;
    // = -(1 - noise) m (1 - m), without the cancellation in 1 - m; m (m e^d), not m m e^d: for |s| > 43.7 m m is
    // subnormal and keeps only a few bits, while m e^d = 1 - m is never small
    const float dp_dd = -(1.0f - noise_prob) * (m * (m * ed));
    const float g = clipped ? 0.f : grad_scale * dl_dp * dp_dd;  // d loss / d (returns difference)
    if (grad_rews) {
      float* g1 = grad_rews + (int64_t)pr * L;
      float* g2 = grad_rews + ((int64_t)P + pr) * L;
      for (int t = lane; t < L; t += 32) {
        const float w = discount == 1.0f ? g : g * powf(discount, (float)t);
        g1[t] = -w;
        g2[t] = w;
      }
    }
    if (lane == 0) {
      if (probs_out) probs_out[pr] = p;
      w_loss += loss;
      w_acc += ((p > 0.5f) == (y > 0.5f)) ? 1.f : 0.f;
    }
  }
  if (!stats_acc) return;
  if (lane == 0) {
    s_loss[warp] = w_loss;
    s_acc[warp] = w_acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < nw; ++w) {
      a += s_loss[w];
      b += s_acc[w];
    }
    atomicAdd(stats_acc + 0, a * inv_P);
    atomicAdd(stats_acc + 1, b * inv_P);
    if (blockIdx.x == 0) atomicAdd(stats_acc + 2, 1.0f);
  }
}

// ---- active selection of preference queries (imb_pref_uncertainty) ---------------------------------------------------
// Workspace: word 0 = the ticket, then mom[M][F][2] = each fragment's batch mean and biased variance, then aff[M][F][2] =
// the (mean, 1 / sqrt(var + eps)) each fragment is normalised with.  The ticket sits at a fixed word so that a workspace
// reused by calls with different member or candidate counts always finds it where the last call re-armed it.
__host__ __device__ __forceinline__ int64_t pu_aff_off(int M, int F) { return 1 + 2 * (int64_t)M * F; }

// NormalizedRewardNet members: a warp per (member, fragment) computes the fragment's moments; the last CTA to finish
// folds them into each member's output RunningNorm in fragment order, one thread per member.  The fold is a chain of
// F dependent updates, as in the reference, which updates the statistics once per fragment.  EMA = true is launched
// when a member has an output EMANorm (d.norm_kind[m] == 1) and folds such members with ema_fold; EMA = false is the
// RunningNorm-only kernel.
template <bool EMA>
__global__ void __launch_bounds__(256) k_pref_frag_norm(const imb_pref_unc_desc d, int F, int L, float* __restrict__ ws) {
  const int M = d.n_members;
  unsigned int* ticket = reinterpret_cast<unsigned int*>(ws);
  float* mom = ws + 1;
  float* aff = ws + pu_aff_off(M, F);
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int64_t jobs = (int64_t)M * F;
  for (int64_t j = (int64_t)blockIdx.x * nw + (threadIdx.x >> 5); j < jobs; j += (int64_t)gridDim.x * nw) {
    const int m = (int)(j / F);
    if (d.norm_state[m] == nullptr) continue;
    float mean, m2;
    warp_moments(d.rews[m] + (j - (int64_t)m * F) * L, L, lane, mean, m2);
    if (lane == 0) {
      mom[2 * j] = mean;
      mom[2 * j + 1] = m2 / (float)L;
    }
  }
  __threadfence();
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x == 0) *ticket = 0u;  // re-arm for the next call
  const int m = threadIdx.x;
  if (m >= M || d.norm_state[m] == nullptr) return;
  float* mv = d.norm_state[m];
  float mean = mv[0], var = mv[1];
  int32_t cnt = *d.norm_count[m];
  const float eps = d.norm_eps[m];
  const float* bm = mom + 2 * (int64_t)m * F;
  float* out = aff + 2 * (int64_t)m * F;
  if constexpr (EMA) {
    if (d.norm_kind[m] == 1) {
      float inv_lr = mv[2];
      int32_t nb = d.norm_count[m][1];
      const float decay = d.norm_decay[m];
      for (int f = 0; f < F; ++f) {
        out[2 * f] = mean;
        out[2 * f + 1] = 1.0f / sqrtf(var + eps);
        ema_fold(mean, var, inv_lr, nb, decay, __ldcg(bm + 2 * f), __ldcg(bm + 2 * f + 1));
        ++nb;
      }
      mv[0] = mean;
      mv[1] = var;
      mv[2] = inv_lr;
      *d.norm_count[m] = cnt + F * L;
      d.norm_count[m][1] = nb;
      return;
    }
  }
#pragma unroll 4
  for (int f = 0; f < F; ++f) {
    out[2 * f] = mean;  // normalise fragment f with the statistics from before its own update
    out[2 * f + 1] = 1.0f / sqrtf(var + eps);
    norm_fold(mean, var, (float)cnt, __ldcg(bm + 2 * f), __ldcg(bm + 2 * f + 1), (float)L);
    cnt += L;
  }
  mv[0] = mean;
  mv[1] = var;
  *d.norm_count[m] = cnt;
}

// Ensemble relabel (imb_ensemble_relabel): thread per (t, e), reading each member's raw reward of that step
// (coalesced along e) and the affine k_pref_frag_norm left for the step, with fragment = env step; two-pass mean and
// ddof-1 variance over the members in member order, as AddSTDRewardWrapper.predict_processed computes them.
__global__ void __launch_bounds__(256) k_ensemble_combine(const imb_pref_unc_desc d, int64_t E, int64_t T, float alpha,
                                                         const float* __restrict__ aff, float* __restrict__ rollout,
                                                         int rw, int col_rew) {
  const int M = d.n_members;
  const int64_t n = E * T;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = i / E, e = i - t * E;
    float v[IMB_PU_MAX_MEMBERS];
    float s = 0.f;
#pragma unroll
    for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m) {
      v[m] = 0.f;
      if (m >= M) continue;
      float x = __ldg(d.rews[m] + i);
      if (d.norm_state[m] != nullptr) {
        const float* a = aff + 2 * ((int64_t)m * T + t);
        x = (x - a[0]) * a[1];
      }
      v[m] = x;
      s += x;
    }
    const float mean = s / (float)M;
    // every product is rounded before its sum, as numpy computes var and mean + alpha * sqrt(var): no fused
    // multiply-adds
    float q = 0.f;
#pragma unroll
    for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m) {
      const float dv = v[m] - mean;
      if (m < M) q = __fadd_rn(q, __fmul_rn(dv, dv));
    }
    rollout[(e * T + t) * rw + col_rew] = mean + __fmul_rn(alpha, sqrtf(q / (float)(M - 1)));
  }
}

// Warp per candidate pair, lanes over t, one register accumulator per member (two for the logit mode's separate
// returns); each fragment's normalisation is applied as its rewards are read.  Lane 0 then takes the mode's per-member
// value and a two-pass mean / variance over the members, in member order.
__global__ void __launch_bounds__(256) k_pref_score(const imb_pref_unc_desc d, int C, int L, int mode, float noise_prob,
                                                   float discount, float threshold, const float* __restrict__ aff,
                                                   float* __restrict__ scores, float* __restrict__ member_out) {
  const int M = d.n_members, F = 2 * C;
  const int lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = blockIdx.x * nw + (threadIdx.x >> 5); i < C; i += gridDim.x * nw) {
    float v[IMB_PU_MAX_MEMBERS];
#pragma unroll
    for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m) {
      v[m] = 0.f;
      if (m >= M) continue;
      float mu1 = 0.f, is1 = 1.f, mu2 = 0.f, is2 = 1.f;
      if (d.norm_state[m] != nullptr) {
        const float* a = aff + 2 * ((int64_t)m * F + 2 * i);
        mu1 = a[0];
        is1 = a[1];
        mu2 = a[2];
        is2 = a[3];
      }
      const float* r1 = d.rews[m] + (int64_t)(2 * i) * L;
      const float* r2 = r1 + L;
      float s1 = 0.f, s2 = 0.f;
      for (int t = lane; t < L; t += 32) {
        const float x1 = (r1[t] - mu1) * is1, x2 = (r2[t] - mu2) * is2;
        if (mode == 0) {
          s1 += x1;
          s2 += x2;
        } else if (discount == 1.0f) {
          s1 += x2 - x1;
        } else {
          s1 = fmaf(powf(discount, (float)t), x2 - x1, s1);
        }
      }
      s1 = warp_sum(s1);
      if (mode == 0) {
        v[m] = s1 - warp_sum(s2);  // sum_t r1 - sum_t r2, undiscounted
      } else {
        v[m] = pref_probability(s1, noise_prob, threshold).p;
      }
    }
    if (lane != 0) continue;
    float score;
    if (mode == 2) {
      int k = 0;
#pragma unroll
      for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m) k += (m < M && v[m] > 0.5f) ? 1 : 0;
      const float q = (float)k / (float)M;
      score = q * (1.0f - q);
    } else {
      float s = 0.f;
#pragma unroll
      for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m) s += (m < M) ? v[m] : 0.f;
      const float mean = s / (float)M;
      float q = 0.f;
#pragma unroll
      for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m) {
        const float dv = v[m] - mean;
        q += (m < M) ? dv * dv : 0.f;
      }
      score = q / (float)(mode == 0 ? M - 1 : M);  // torch.var (ddof 1) for logits, np.var (ddof 0) for probabilities
    }
    scores[i] = score;
    if (member_out) {
#pragma unroll
      for (int m = 0; m < IMB_PU_MAX_MEMBERS; ++m)
        if (m < M) member_out[(int64_t)i * M + m] = v[m];
    }
  }
}

// statistics -> host-mapped pinned memory, followed by a sequence word (system-scope fence in between): the host polls
// the word instead of issuing a D2H copy and synchronising on an event (one PCIe posted write burst per update)
__global__ void k_stats_publish(const float* __restrict__ stats_dev, int n, float* host, const int64_t* __restrict__ state,
                                int state_idx) {
  const int lane = threadIdx.x;
  if (lane < n) host[lane] = stats_dev[lane];
  __threadfence_system();
  __syncwarp();
  if (lane == 0) reinterpret_cast<volatile int*>(host)[15] = (int)state[state_idx];
}

// ---- forward only (reward relabel / predict) ---------------------------------------------------
// thread per row straight from global memory (coalesced over rows for each feature); one TImg per pass, img_sz apart,
// then xn_ld >= din normalised inputs per thread.
template <int JP>
__global__ void __launch_bounds__(NT) k_reward_fwd(const DiscLaunch L, const float* __restrict__ params,
                                                   const float* __restrict__ batch, int64_t ld, int64_t n,
                                                   int out_mode, float* __restrict__ out, int img_sz, int xn_ld) {
  extern __shared__ __align__(128) float smem[];
  const int tid = threadIdx.x;
  for (int p = 0; p < L.npass; ++p) load_timg(smem + p * img_sz, L.pass[p], JP, params, L.pass[p].norm, L.pass[p].eps);
  __syncthreads();
  float* xn = smem + L.npass * img_sz + tid * xn_ld;
  for (int64_t row = (int64_t)blockIdx.x * NT + tid; row < n; row += (int64_t)gridDim.x * NT) {
    const float done = (L.done_slot >= 0) ? batch[(int64_t)L.stage_row[L.done_slot] * ld + row] : 0.f;
    float logit = 0.f;
    for (int p = 0; p < L.npass; ++p) {
      const PassDesc& P = L.pass[p];
      const float* img = smem + p * img_sz;
      const float* mean = img + TImg::mean(P.din, JP);
      const float* istd = img + TImg::istd(P.din, JP);
      for (int k = 0; k < P.din; ++k)
        xn[k] = (batch[(int64_t)L.stage_row[P.in_slot[k]] * ld + row] - mean[k]) * istd[k];
      const float o = timg_forward_row<JP>(img, P, xn);
      logit = fmaf(pass_coef(P.coef_kind, L.gamma, done), o, logit);
    }
    if (out_mode >= 1 && L.logp_slot >= 0) logit -= batch[(int64_t)L.stage_row[L.logp_slot] * ld + row];
    out[row] = (out_mode == 2) ? softplus_f(logit) : logit;
  }
}

// ---- NormalizedRewardNet.predict_processed over consecutive env steps ---------------------------
// single CTA: for t in steps: normalise the E rewards of step t with the running stats, then merge
// step t's raw rewards into the stats (reward_nets.py:637-671 + networks.py:111-134).  EMA = false: RunningNorm,
// mv = [mean, var], count = [count]; EMA = true: EMANorm (networks.py:137-201), mv = [mean, var, inv_learning_rate],
// count = [count, num_batches], and `decay` is read.
template <bool EMA>
__global__ void __launch_bounds__(1024) k_reward_norm_scan(float* __restrict__ rews, int64_t E, int64_t T,
                                                          int64_t step_stride, int64_t env_stride,
                                                          float* __restrict__ mv, int32_t* __restrict__ count,
                                                          float eps, int update, float decay) {
  __shared__ float red[64];
  __shared__ float bc[2];
  float mean = mv[0], var = mv[1];
  int32_t cnt = *count;
  float inv_lr = 0.f;
  int32_t nb = 0;
  if constexpr (EMA) {
    inv_lr = mv[2];
    nb = count[1];
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  for (int64_t t = 0; t < T; ++t) {
    float* r = rews + t * step_stride;
    const float istd = 1.0f / sqrtf(var + eps);
    float s = 0.f;
    for (int64_t e = tid; e < E; e += blockDim.x) s += r[e * env_stride];
    s = warp_sum(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (tid == 0) {
      float a = 0.f;
      for (int w = 0; w < nw; ++w) a += red[w];
      bc[0] = a / (float)E;
    }
    __syncthreads();
    const float bmean = bc[0];
    float m2 = 0.f;
    for (int64_t e = tid; e < E; e += blockDim.x) {
      const float v = r[e * env_stride];
      const float dlt = v - bmean;
      m2 = fmaf(dlt, dlt, m2);
      r[e * env_stride] = (v - mean) * istd;  // normalise with the stats BEFORE this step's update
    }
    m2 = warp_sum(m2);
    if (lane == 0) red[32 + warp] = m2;
    __syncthreads();
    if (tid == 0) {
      float a = 0.f;
      for (int w = 0; w < nw; ++w) a += red[32 + w];
      bc[1] = a / (float)E;
    }
    __syncthreads();
    if (update) {
      if constexpr (EMA) {
        ema_fold(mean, var, inv_lr, nb, decay, bmean, bc[1]);
        ++nb;
      } else {
        norm_fold(mean, var, (float)cnt, bmean, bc[1], (float)E);
      }
      cnt += (int32_t)E;
    }
    __syncthreads();
  }
  if (tid == 0 && update) {
    mv[0] = mean;
    mv[1] = var;
    *count = cnt;
    if constexpr (EMA) {
      mv[2] = inv_lr;
      count[1] = nb;
    }
  }
}

}  // namespace

extern "C" int64_t imb_disc_workspace_floats(const imb_disc_desc* d) { return ws_layout(d->n_params).total; }

// RunningNorm updates of J's jobs over rows [0, n) of the batch: one k_norm_stats launch, or one per job in job order
// when the chunk table cannot hold every job's chunks
static int norm_stats(const NormJobs& J, const float* batch, int64_t ld, int64_t n, float* ws, const WsLayout& w,
                      cudaStream_t st, float* defer = nullptr, int defer_cap = 0) {
  // chunk size: small enough to fill the GPU at the tuned batch sizes (16 384 rows -> 128 CTAs), larger for the
  // multi-million-row sweeps so the chunk table stays bounded
  const int chunk_rows = n <= (int64_t)128 * 2048 ? 128 : NORM_CHUNK;
  const int64_t chunks = (n + chunk_rows - 1) / chunk_rows;
  IMB_REQUIRE(chunks >= 1 && chunks <= MAXCHUNKS, "norm update: n=%lld out of range", (long long)n);
  if (chunks * J.njobs > MAXCHUNKS) {
    for (int j = 0; j < J.njobs; ++j)
      if (int rc = norm_stats(NormJobs{1, {J.job[j]}}, batch, ld, n, ws, w, st, defer, defer_cap)) return rc;
    return 0;
  }
  k_norm_stats<<<dim3((unsigned)chunks, J.njobs), 256, 0, st>>>(J, batch, ld, n, chunk_rows, ws + w.normpart,
                                                                 reinterpret_cast<unsigned int*>(ws + w.ticket), defer,
                                                                 defer_cap);
  IMB_CHECK_LAUNCH("k_norm_stats");
  return 0;
}

extern "C" int imb_disc_norm_update(const imb_disc_desc* d, const float* batch, int64_t ld, int64_t n,
                                    float* norm_state, int32_t* norm_count, float* ws, void* stream) {
  IMB_REQUIRE(n >= 1, "norm update needs n >= 1");
  const WsLayout w = ws_layout(d->n_params);
  DiscLaunch L;
  if (int rc = build_launch(d, norm_state, nullptr, L)) return rc;
  NormJobs J = {};
  auto add = [&](const imb_mlp& m, int pass, float* snap) {
    NormJob& job = J.job[J.njobs++];
    job.din = m.din;
    for (int k = 0; k < m.din; ++k) job.row[k] = L.stage_row[L.pass[pass].in_slot[k]];
    job.rmv = norm_state + m.norm_off;
    job.cnt = norm_count + m.count_idx;
    job.snap = snap;
  };
  if (d->base.has_norm) add(d->base, 0, nullptr);
  if (d->shaped && d->potential.has_norm) {
    // reference order: Phi(next_state) first, then Phi(state); both update the same RunningNorm
    add(d->potential, 1, ws + w.snap);
    add(d->potential, 2, nullptr);
  }
  return J.njobs ? norm_stats(J, batch, ld, n, ws, w, (cudaStream_t)stream) : 0;
}

extern "C" int imb_norm_batch_stats(const imb_disc_desc* d, const float* batch, int64_t ld, int64_t n, int row0, int din,
                                    float* norm_state, int32_t* norm_count, float* defer, int defer_cap, float* ws,
                                    void* stream) {
  IMB_REQUIRE(n >= 1 && din >= 1 && din <= IMB_MAX_DIN, "norm batch stats: bad sizes");
  IMB_REQUIRE(defer == nullptr || defer_cap >= 1, "norm batch stats: defer_cap");
  NormJobs J = {1};
  J.job[0].din = din;
  for (int k = 0; k < din; ++k) J.job[0].row[k] = (short)(row0 + k);
  J.job[0].rmv = norm_state;
  J.job[0].cnt = norm_count;
  return norm_stats(J, batch, ld, n, ws, ws_layout(d->n_params), (cudaStream_t)stream, defer, defer_cap);
}

extern "C" int imb_norm_fold(int din, float* defer, float* norm_state, int32_t* norm_count, int n_slots, void* stream) {
  IMB_REQUIRE(din >= 1 && din <= IMB_MAX_DIN, "norm fold: din");
  k_norm_fold<<<1, 64, 0, (cudaStream_t)stream>>>(din, defer, norm_state, norm_count, n_slots);
  IMB_CHECK_LAUNCH("k_norm_fold");
  return 0;
}

// multi-GPU: the statistics of the last minibatch were summed over the ranks -> the row counts k_disc_adam divides by
// are the global ones
__global__ void k_set_rows(int* meta, int64_t n, int64_t n_expert) {
  meta[1] = (int)n;
  meta[2] = (int)n_expert;
}
extern "C" int imb_disc_set_rows(const imb_disc_desc* d, float* ws, int64_t n, int64_t n_expert, void* stream) {
  const WsLayout w = ws_layout(d->n_params);
  k_set_rows<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<int*>(ws + w.meta), n, n_expert);
  IMB_CHECK_LAUNCH("k_set_rows");
  return 0;
}

extern "C" int imb_stats_publish(const float* stats_dev, int n, float* host_mapped, const int64_t* state, int state_idx,
                                 void* stream) {
  IMB_REQUIRE(n >= 1 && n <= 15 && state_idx >= 0 && state_idx < IMB_ST_WORDS, "stats publish: bad sizes");
  k_stats_publish<<<1, 32, 0, (cudaStream_t)stream>>>(stats_dev, n, host_mapped, state, state_idx);
  IMB_CHECK_LAUNCH("k_stats_publish");
  return 0;
}

struct TPlan {
  int JP, KP, img_sz, aw_off, st_off, xn_off, t_off, v_off, nsl, total;
};
static TPlan plan_tiled(const DiscLaunch& L, int R) {
  TPlan t;
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  const int RS = R + TILE_PAD;
  const LaunchWidths lw = launch_widths(L);
  t.JP = lw.JP;
  t.KP = lw.dmax <= 32 ? 32 : 64;
  t.img_sz = al(TImg::size(lw.dmax, t.JP));
  int o = L.npass * t.img_sz;
  t.nsl = (t.JP == 32 && R == 256) ? 4 : 2;  // row slices of the weight-gradient phase (>= 2: slice 1 holds dwf)
  t.aw_off = o;
  o += al(t.nsl * L.P);
  t.st_off = o;
  o += al(L.nstage * RS);
  t.xn_off = o;
  o += al(t.KP * RS);
  t.t_off = o;
  o += al(3 * t.JP * RS);
  t.v_off = o;
  o += al(5 * R);
  t.total = o;
  return t;
}

template <int R>
static int launch_fwdbwd(const DiscLaunch& L, const TPlan& t, const float* params, const float* batch, int64_t ld,
                         int64_t n, int64_t n_expert, float loss_scale, const float* grad_out, float* logits_out,
                         float* ws, const WsLayout& w, cudaStream_t st, int ctas_per_sm) {
  const size_t bytes = (size_t)t.total * 4;
  static size_t attr_bytes = 0;
  if (bytes > attr_bytes) {
    cudaError_t e = cudaFuncSetAttribute(k_disc_fwdbwd<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute(%zu): %s", bytes, cudaGetErrorString(e));
    attr_bytes = bytes;
  }
  const int64_t ntiles = (n + R - 1) / R;
  int64_t G = (int64_t)imb_num_sms() * ctas_per_sm;
  if (G > MAXG) G = MAXG;
  if (G > ntiles) G = ntiles;
  k_disc_fwdbwd<R><<<(int)G, R, bytes, st>>>(L, params, batch, ld, n, n_expert, loss_scale, grad_out, logits_out,
                                               ws + w.partial, reinterpret_cast<int*>(ws + w.meta), t.JP, t.KP, t.img_sz, t.aw_off, t.st_off, t.xn_off,
                                               t.t_off, t.v_off, t.nsl);
  IMB_CHECK_LAUNCH("k_disc_fwdbwd");
  return 0;
}

// Which k_disc_fwdbwd* kernel runs for this shape and row count (the IMB_PLAN_* codes of imb_disc_plan); the tiled
// plans are returned in t128 / t256.  Tensor cores (wgmma, 3xTF32 split) whenever the network shape fits them; else
// 128-row tiles with TWO resident CTAs per SM (independent CTAs overlap each other's barriers and epilogues); else one
// 256-row CTA; else one 128-row CTA.
static int fwdbwd_plan(const DiscLaunch& L, int64_t n, int flags, TPlan& t128, TPlan& t256) {
  if (!(flags & IMB_F_NO_TENSOR) && tc_applicable(L)) {
    const size_t bytes = (size_t)tc_plan(L).total * 4 + 128;
    IMB_REQUIRE(bytes <= IMB_SMEM_MAX, "tensor-core disc kernel: %zu B of shared memory", bytes);
    return IMB_PLAN_TC;
  }
  t256 = plan_tiled(L, 256);
  t128 = plan_tiled(L, 128);
  if (2 * ((size_t)t128.total * 4 + 1024 + 512) <= 228 * 1024) return IMB_PLAN_FFMA128X2;
  if ((size_t)t256.total * 4 <= IMB_SMEM_MAX && n > 128) return IMB_PLAN_FFMA256;
  if ((size_t)t128.total * 4 <= IMB_SMEM_MAX) return IMB_PLAN_FFMA128;
  IMB_FAIL(-1, "discriminator too large for the fused kernel: its 128-row tile needs %zu B of shared memory per CTA, "
           "the limit is %d B", (size_t)t128.total * 4, IMB_SMEM_MAX);
}

// imb_reward_forward's shared memory (floats): one TImg per pass, img_sz apart, then xn_ld normalised inputs per thread
struct FwdPlan {
  LaunchWidths lw;
  int img_sz, xn_ld, total;
};
static FwdPlan fwd_plan(const DiscLaunch& L) {
  auto al = [](int x) { return (x + 31) / 32 * 32; };
  FwdPlan f;
  f.lw = launch_widths(L);
  f.img_sz = al(TImg::size(f.lw.dmax, f.lw.JP));
  f.xn_ld = f.lw.dmax | 1;
  f.total = L.npass * f.img_sz + al(NT * f.xn_ld);
  return f;
}

extern "C" int imb_disc_plan(const imb_disc_desc* d, int64_t n) {
  IMB_REQUIRE(n >= 1, "disc plan needs n >= 1");
  DiscLaunch L;
  if (int rc = build_launch(d, nullptr, nullptr, L)) return rc;
  const size_t fb = (size_t)fwd_plan(L).total * 4;
  IMB_REQUIRE(fb <= IMB_SMEM_MAX, "reward net too large for the fused forward kernel: %zu B of shared memory, the "
              "limit is %d B", fb, IMB_SMEM_MAX);
  TPlan t128, t256;
  return fwdbwd_plan(L, n, 0, t128, t256);
}

extern "C" int imb_disc_fwd_bwd(const imb_disc_desc* d, const float* params, const float* norm_state,
                                const float* batch, int64_t ld, int64_t n, int64_t n_expert, float loss_scale,
                                const float* grad_out, float* logits_out, int flags, float* ws, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  IMB_REQUIRE(n >= 1, "fwd_bwd needs n >= 1");
  IMB_REQUIRE(ld % 4 == 0 && ld >= (n + IMB_TILE_ROWS - 1) / IMB_TILE_ROWS * IMB_TILE_ROWS,
              "batch leading dimension must cover n rounded up to %d rows", IMB_TILE_ROWS);
  const WsLayout w = ws_layout(d->n_params);
  DiscLaunch L;
  // in training mode the Phi(s') pass uses the stats snapshot taken between the two norm updates
  const bool snap = d->shaped && d->potential.has_norm && (flags & IMB_F_TRAIN_NORM);
  if (int rc = build_launch(d, norm_state, snap ? ws + w.snap : nullptr, L)) return rc;
  TPlan t128, t256;
  const int plan = fwdbwd_plan(L, n, flags, t128, t256);
  if (plan < 0) return plan;
  if (flags & IMB_F_ZERO_GRAD) {
    cudaError_t e = cudaMemsetAsync(ws + w.gacc, 0, sizeof(float) * d->n_params, st);
    if (e != cudaSuccess) IMB_FAIL(-2, "memset: %s", cudaGetErrorString(e));
  }
  if (plan == IMB_PLAN_TC) {
    const TcPlan T = tc_plan(L);
    const size_t bytes = (size_t)T.total * 4 + 128;
    static bool attr_set = false;
    if (!attr_set) {
      cudaError_t e = cudaFuncSetAttribute(k_disc_fwdbwd_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)IMB_SMEM_MAX);
      if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute(tc): %s", cudaGetErrorString(e));
      attr_set = true;
    }
    const int64_t ntiles = (n + 127) / 128;
    int64_t Gt = imb_num_sms();
    if (Gt > MAXG) Gt = MAXG;
    if (Gt > ntiles) Gt = ntiles;
    k_disc_fwdbwd_tc<<<(int)Gt, TC_THREADS, bytes, st>>>(L, T, params, batch, ld, n, n_expert, loss_scale, grad_out, logits_out,
                                                         ws + w.partial, reinterpret_cast<int*>(ws + w.meta),
                                                         part_stride(d->n_params));
    IMB_CHECK_LAUNCH("k_disc_fwdbwd_tc");
    return 0;
  }
  if (plan == IMB_PLAN_FFMA256)
    return launch_fwdbwd<256>(L, t256, params, batch, ld, n, n_expert, loss_scale, grad_out, logits_out, ws, w, st, 1);
  return launch_fwdbwd<128>(L, t128, params, batch, ld, n, n_expert, loss_scale, grad_out, logits_out, ws, w, st,
                            plan == IMB_PLAN_FFMA128X2 ? 2 : 1);
}

// warp per parameter and per statistic, at most two blocks per SM
static int reduce_blocks(int P) {
  const int blocks = ((P + 5) * 32 + 255) / 256;
  return blocks < 2 * imb_num_sms() ? blocks : 2 * imb_num_sms();
}

extern "C" int imb_disc_reduce(const imb_disc_desc* d, float* ws, float* grad_out_flat, void* stream) {
  const WsLayout w = ws_layout(d->n_params);
  k_disc_reduce<<<reduce_blocks(d->n_params), 256, 0, (cudaStream_t)stream>>>(
      d->n_params, reinterpret_cast<const int*>(ws + w.meta), ws + w.partial, ws + w.gacc, ws + w.stats, grad_out_flat);
  IMB_CHECK_LAUNCH("k_disc_reduce");
  return 0;
}

extern "C" int imb_disc_adam(const imb_disc_desc* d, const imb_adam* opt, float* params, float* exp_avg,
                             float* exp_avg_sq, const float* grad_flat_or_null, float grad_div, float* ws,
                             int64_t* state, float* stats_out, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const WsLayout w = ws_layout(d->n_params);
  const int P = d->n_params;
  const float* grad = grad_flat_or_null ? grad_flat_or_null : ws + w.gacc;
  // loss statistic: sum * loss_scale recorded by the last fwd/bwd launch (meta[3])
  k_disc_adam<<<1, 1024, 0, st>>>(P, *opt, params, exp_avg, exp_avg_sq, grad, grad_div, ws + w.stats,
                                  reinterpret_cast<const int*>(ws + w.meta), state + IMB_ST_DISC_STEP, stats_out);
  IMB_CHECK_LAUNCH("k_disc_adam");
  return 0;
}

extern "C" int imb_disc_reduce_adam(const imb_disc_desc* d, const imb_adam* opt, float* params, float* exp_avg,
                                    float* exp_avg_sq, float grad_div, float* ws, int64_t* state, float* stats_out,
                                    void* stream) {
  const WsLayout w = ws_layout(d->n_params);
  k_disc_reduce_adam<<<reduce_blocks(d->n_params), 256, 0, (cudaStream_t)stream>>>(
      d->n_params, ws + w.partial, ws + w.gacc, ws + w.stats, *opt, params, exp_avg, exp_avg_sq, grad_div,
      reinterpret_cast<const int*>(ws + w.meta), state + IMB_ST_DISC_STEP, stats_out,
      reinterpret_cast<unsigned int*>(ws + w.ticket) + 8);
  IMB_CHECK_LAUNCH("k_disc_reduce_adam");
  return 0;
}

extern "C" int imb_param_regularize(const imb_disc_desc* d, int32_t kind, int32_t p, float coeff, float* params,
                                    float* ws, float* stats_acc, int32_t stats_slot, void* stream) {
  IMB_REQUIRE(kind == IMB_REG_LP || kind == IMB_REG_WEIGHT_DECAY,
              "imb_param_regularize: kind %d (%d Lp, %d weight decay)", kind, IMB_REG_LP, IMB_REG_WEIGHT_DECAY);
  IMB_REQUIRE(kind != IMB_REG_LP || p >= 1, "imb_param_regularize: p = %d, the Lp penalty needs an integer p >= 1", p);
  IMB_REQUIRE(kind != IMB_REG_LP || ws != nullptr, "imb_param_regularize: the Lp penalty needs the workspace");
  IMB_REQUIRE(stats_slot >= 0, "imb_param_regularize: bad statistics slot");
  IMB_REQUIRE(d->n_params >= 1, "imb_param_regularize: no parameters");
  float* gacc = kind == IMB_REG_LP ? ws + ws_layout(d->n_params).gacc : nullptr;
  float* stats = kind == IMB_REG_LP && stats_acc ? stats_acc + 4 * stats_slot : nullptr;
  k_param_regularize<<<1, 1024, 0, (cudaStream_t)stream>>>(d->n_params, kind, p, coeff, params, gacc, stats);
  IMB_CHECK_LAUNCH("k_param_regularize");
  return 0;
}

template <int JP>
static int launch_fwd(const DiscLaunch& L, const FwdPlan& f, const float* params, const float* batch, int64_t ld,
                      int64_t n, int out_mode, float* out, cudaStream_t st) {
  const size_t bytes = (size_t)f.total * 4;
  IMB_REQUIRE(bytes <= IMB_SMEM_MAX, "reward net too large for the fused kernel (%zu B smem)", bytes);
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(k_reward_fwd<JP>, cudaFuncAttributeMaxDynamicSharedMemorySize, IMB_SMEM_MAX);
    if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  int64_t blocks = (n + NT - 1) / NT;
  const int64_t cap = (int64_t)imb_num_sms() * 4;
  if (blocks > cap) blocks = cap;
  k_reward_fwd<JP><<<(int)blocks, NT, bytes, st>>>(L, params, batch, ld, n, out_mode, out, f.img_sz, f.xn_ld);
  IMB_CHECK_LAUNCH("k_reward_fwd");
  return 0;
}

extern "C" int imb_reward_forward(const imb_disc_desc* d, const float* params, const float* norm_state,
                                  const float* batch, int64_t ld, int64_t n, int out_mode, float* out,
                                  void* stream) {
  if (n <= 0) return 0;
  DiscLaunch L;
  imb_disc_desc dd = *d;
  if (out_mode == 0) dd.subtract_logp = 0;
  if (int rc = build_launch(&dd, norm_state, nullptr, L)) return rc;
  const FwdPlan f = fwd_plan(L);
  return (f.lw.JP == 32) ? launch_fwd<32>(L, f, params, batch, ld, n, out_mode, out, (cudaStream_t)stream)
                         : launch_fwd<64>(L, f, params, batch, ld, n, out_mode, out, (cudaStream_t)stream);
}

template <bool EMA>
static int launch_reward_norm_scan(float* rews, int64_t n_envs, int64_t n_steps, int64_t step_stride,
                                   int64_t env_stride, float* state, int32_t* counts, float eps, int update_stats,
                                   float decay, void* stream) {
  IMB_REQUIRE(n_envs >= 1 && n_steps >= 0, "bad sizes");
  if (n_steps == 0) return 0;
  int threads = 1024;
  while (threads > 32 && threads / 2 >= n_envs) threads /= 2;
  k_reward_norm_scan<EMA><<<1, threads, 0, (cudaStream_t)stream>>>(rews, n_envs, n_steps, step_stride, env_stride,
                                                                   state, counts, eps, update_stats, decay);
  IMB_CHECK_LAUNCH("k_reward_norm_scan");
  return 0;
}

extern "C" int imb_reward_norm_scan(float* rews, int64_t n_envs, int64_t n_steps, int64_t step_stride,
                                    int64_t env_stride, float* norm_state2, int32_t* norm_count, float eps,
                                    int update_stats, void* stream) {
  return launch_reward_norm_scan<false>(rews, n_envs, n_steps, step_stride, env_stride, norm_state2, norm_count, eps,
                                        update_stats, 0.f, stream);
}

extern "C" int imb_reward_ema_scan(float* rews, int64_t n_envs, int64_t n_steps, int64_t step_stride,
                                   int64_t env_stride, float* ema_state3, int32_t* ema_counts2, float decay, float eps,
                                   int update_stats, void* stream) {
  IMB_REQUIRE(decay > 0.f && decay < 1.f, "imb_reward_ema_scan: decay %g outside (0, 1)", (double)decay);
  return launch_reward_norm_scan<true>(rews, n_envs, n_steps, step_stride, env_stride, ema_state3, ema_counts2, eps,
                                       update_stats, decay, stream);
}

extern "C" int imb_pref_loss(const float* rews, int64_t n_pairs, int32_t frag_len, const float* prefs, float noise_prob,
                             float discount, float threshold, float grad_scale, float* grad_rews, float* probs_out,
                             float* stats_acc, int32_t stats_slot, void* stream) {
  IMB_REQUIRE(n_pairs >= 1 && n_pairs < (1ll << 30) && frag_len >= 1, "imb_pref_loss: bad sizes");
  IMB_REQUIRE(stats_slot >= 0, "imb_pref_loss: bad statistics slot");
  int64_t blocks = (n_pairs + 7) / 8;
  if (blocks > 4 * imb_num_sms()) blocks = 4 * imb_num_sms();
  k_pref_loss<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(rews, (int)n_pairs, frag_len, prefs, noise_prob, discount,
                                                             threshold, grad_scale, grad_rews, probs_out,
                                                             stats_acc ? stats_acc + 4 * stats_slot : nullptr);
  IMB_CHECK_LAUNCH("k_pref_loss");
  return 0;
}

// norm_kind / norm_decay of member m of an imb_pref_unc_desc: 0 = RunningNorm, 1 = EMANorm with 0 < decay < 1
static int check_norm_kind(const imb_pref_unc_desc* d, int m, const char* who) {
  const int kind = d->norm_kind[m];
  IMB_REQUIRE(kind == 0 || kind == 1, "%s: member %d: norm kind %d (0 RunningNorm, 1 EMANorm)", who, m, kind);
  IMB_REQUIRE(kind == 0 || d->norm_state[m] == nullptr || (d->norm_decay[m] > 0.f && d->norm_decay[m] < 1.f),
              "%s: member %d: EMANorm decay %g outside (0, 1)", who, m, (double)d->norm_decay[m]);
  return 0;
}

extern "C" int64_t imb_pref_uncertainty_ws_floats(int32_t n_members, int64_t n_pairs) {
  return 1 + 4 * (int64_t)n_members * 2 * n_pairs;
}

extern "C" int imb_pref_uncertainty(const imb_pref_unc_desc* d, int64_t n_pairs, int32_t frag_len, int32_t mode,
                                    float noise_prob, float discount, float threshold, float* ws, float* scores,
                                    float* member_out, void* stream) {
  const int M = d->n_members;
  IMB_REQUIRE(M >= 2 && M <= IMB_PU_MAX_MEMBERS, "imb_pref_uncertainty: %d members (2 to %d)", M, IMB_PU_MAX_MEMBERS);
  IMB_REQUIRE(n_pairs >= 0 && n_pairs < (1ll << 28) && frag_len >= 1, "imb_pref_uncertainty: bad sizes");
  IMB_REQUIRE(mode >= 0 && mode <= 2, "imb_pref_uncertainty: mode %d (0 logit, 1 probability, 2 label)", mode);
  bool any_norm = false, any_ema = false;
  for (int m = 0; m < M; ++m) {
    IMB_REQUIRE(d->rews[m] != nullptr, "imb_pref_uncertainty: member %d has no rewards", m);
    IMB_REQUIRE((d->norm_state[m] == nullptr) == (d->norm_count[m] == nullptr),
                "imb_pref_uncertainty: member %d: norm state and count go together", m);
    if (int rc = check_norm_kind(d, m, "imb_pref_uncertainty")) return rc;
    any_norm = any_norm || d->norm_state[m] != nullptr;
    any_ema = any_ema || (d->norm_state[m] != nullptr && d->norm_kind[m] == 1);
  }
  if (n_pairs == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
  const int C = (int)n_pairs, F = 2 * C;
  const int64_t cap = 4 * (int64_t)imb_num_sms();
  if (any_norm) {
    const int64_t blocks = std::min(((int64_t)M * F + 7) / 8, cap);
    if (any_ema)
      k_pref_frag_norm<true><<<(int)blocks, 256, 0, st>>>(*d, F, frag_len, ws);
    else
      k_pref_frag_norm<false><<<(int)blocks, 256, 0, st>>>(*d, F, frag_len, ws);
    IMB_CHECK_LAUNCH("k_pref_frag_norm");
  }
  const int64_t blocks = std::min(((int64_t)C + 7) / 8, cap);
  k_pref_score<<<(int)blocks, 256, 0, st>>>(*d, C, frag_len, mode, noise_prob, discount, threshold,
                                            ws + pu_aff_off(M, F), scores, member_out);
  IMB_CHECK_LAUNCH("k_pref_score");
  return 0;
}

extern "C" int64_t imb_ensemble_relabel_ws_floats(int32_t n_members, int64_t n_steps) {
  return pu_aff_off(n_members, (int)n_steps) + 2 * (int64_t)n_members * n_steps;
}

extern "C" int imb_ensemble_relabel(const imb_pref_unc_desc* d, float alpha, float* rollout, int32_t rw, int32_t col_rew,
                                    int64_t n_envs, int64_t n_steps, float* ws, void* stream) {
  const int M = d->n_members;
  IMB_REQUIRE(M >= 2 && M <= IMB_PU_MAX_MEMBERS, "imb_ensemble_relabel: %d members (2 to %d)", M, IMB_PU_MAX_MEMBERS);
  IMB_REQUIRE(n_envs >= 1 && n_steps >= 1 && n_envs * n_steps < (1ll << 31), "imb_ensemble_relabel: bad sizes");
  IMB_REQUIRE(col_rew >= 0 && col_rew < rw, "imb_ensemble_relabel: reward column %d outside rows of %d", col_rew, rw);
  bool any_norm = false, any_ema = false;
  for (int m = 0; m < M; ++m) {
    IMB_REQUIRE(d->rews[m] != nullptr, "imb_ensemble_relabel: member %d has no rewards", m);
    IMB_REQUIRE((d->norm_state[m] == nullptr) == (d->norm_count[m] == nullptr),
                "imb_ensemble_relabel: member %d: norm state and count go together", m);
    if (int rc = check_norm_kind(d, m, "imb_ensemble_relabel")) return rc;
    any_norm = any_norm || d->norm_state[m] != nullptr;
    any_ema = any_ema || (d->norm_state[m] != nullptr && d->norm_kind[m] == 1);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  const int F = (int)n_steps, L = (int)n_envs;  // fragment = one env step of E rewards
  const int64_t cap = 4 * (int64_t)imb_num_sms();
  if (any_norm) {
    const int64_t blocks = std::min(((int64_t)M * F + 7) / 8, cap);
    if (any_ema)
      k_pref_frag_norm<true><<<(int)blocks, 256, 0, st>>>(*d, F, L, ws);
    else
      k_pref_frag_norm<false><<<(int)blocks, 256, 0, st>>>(*d, F, L, ws);
    IMB_CHECK_LAUNCH("k_pref_frag_norm");
  }
  const int64_t blocks = std::min((n_envs * n_steps + 255) / 256, 8 * (int64_t)imb_num_sms());
  k_ensemble_combine<<<(int)blocks, 256, 0, st>>>(*d, n_envs, n_steps, alpha, ws + pu_aff_off(M, F), rollout, rw,
                                                  col_rew);
  IMB_CHECK_LAUNCH("k_ensemble_combine");
  return 0;
}

extern "C" int imb_state_init(int64_t* state, void* stream) {
  cudaError_t e = cudaMemsetAsync(state, 0, sizeof(int64_t) * IMB_ST_WORDS, (cudaStream_t)stream);
  if (e != cudaSuccess) IMB_FAIL(-2, "memset: %s", cudaGetErrorString(e));
  return 0;
}
