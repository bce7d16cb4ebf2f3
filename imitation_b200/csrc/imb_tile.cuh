// imb_tile.cuh -- shared-memory tiled fp32 GEMM building blocks for the small-MLP kernels, and the shared-memory images
// of the reward net (TImg) and the policy (PolImg) that every kernel evaluating them builds.
//
// Why: a thread-per-row MLP reads one broadcast weight per FMA from shared memory; the LSU
// delivers 4 B/lane/cycle, i.e. one operand per lane per cycle per SM, while the FMA pipes want
// four -- so that form tops out at 25 % of fp32 peak, and its fully
// unrolled code (200 KB) thrashes the instruction cache.  Here every operand fetched from shared
// memory is reused from registers: each thread owns a TR x TJ output tile (2.67-4 FMAs per
// fetched float) and the reduction loops stay rolled (a few KB of code).
//
// Tiles are FEATURE-MAJOR in shared memory: element (feature f, row r) at base[f * RS + r] with
// RS = R + 4; the 4-float pad staggers consecutive feature rows by 4 banks so that the 8 lanes of
// one LDS.128 phase never collide.
#pragma once
#include "imb_common.cuh"
#include "imb_mlp.cuh"

namespace {

constexpr int TILE_PAD = 4;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }

enum { ACT_TANH = 0, ACT_RELU = 1 };

// rows per tile for a rows-per-lane parameter (RPL = 0: the 8-row tile, lane = (row, column pair))
__host__ __device__ constexpr int rows_of(int rpl) { return rpl == 0 ? 8 : 32 * rpl; }

// 8-row tile: warp -> 8-column group, lane -> (row = lane % 8, columns 2 * (lane / 8), +1): two FMAs per input and
// lane, so a layer's latency is ~K x 10 cycles and the grid covers all SMs at 1024 envs (128 CTAs)
template <int ACT>
__device__ __forceinline__ void tile_layer8(const float* __restrict__ A, int K, const float* __restrict__ Wk, int wld,
                                            const float* __restrict__ bias, float* __restrict__ OUT, int JPx) {
  constexpr int RRS = 8 + TILE_PAD;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r = lane & 7, c2 = 2 * (lane >> 3);
  for (int jh = 0; jh < JPx / 32; ++jh) {
    const int j0 = jh * 32 + warp * 8 + c2;
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;  // two accumulator pairs (even / odd k)
    int k = 0;
#pragma unroll 4
    for (; k + 2 <= K; k += 2) {
      const float x0 = A[k * RRS + r], x1 = A[(k + 1) * RRS + r];
      const float2 w0 = *reinterpret_cast<const float2*>(Wk + k * wld + j0);
      const float2 w1 = *reinterpret_cast<const float2*>(Wk + (k + 1) * wld + j0);
      a0 = fmaf(x0, w0.x, a0);
      a1 = fmaf(x0, w0.y, a1);
      b0 = fmaf(x1, w1.x, b0);
      b1 = fmaf(x1, w1.y, b1);
    }
    if (k < K) {
      const float x0 = A[k * RRS + r];
      const float2 w0 = *reinterpret_cast<const float2*>(Wk + k * wld + j0);
      a0 = fmaf(x0, w0.x, a0);
      a1 = fmaf(x0, w0.y, a1);
    }
    const float z0 = (a0 + b0) + bias[j0], z1 = (a1 + b1) + bias[j0 + 1];
    OUT[j0 * RRS + r] = ACT == ACT_TANH ? tanh_fast(z0) : fmaxf(z0, 0.f);
    OUT[(j0 + 1) * RRS + r] = ACT == ACT_TANH ? tanh_fast(z1) : fmaxf(z1, 0.f);
  }
}

// One MLP layer over a feature-major tile of ROWS rows (row stride ROWS + TILE_PAD):
//   OUT[j][r] = act(bias[j] + sum_k A[k][r] * Wk[k * wld + j])     for j < JPx (a multiple of 32)
// each element an fmaf chain over k in ascending order from 0, then + bias, then the activation.  Groups of 4 warps
// (ROWS / (32 RPL) groups, one per 128 threads) split the rows: warp -> 8-column group (warp % 4) of its group's
// 32 RPL rows (warp / 4), lane -> RPL consecutive rows.  RPL = 0 is the 8-row tile of tile_layer8.
template <int ACT, int RPL, int ROWS = rows_of(RPL)>
__device__ __forceinline__ void tile_layer(const float* __restrict__ A, int K, const float* __restrict__ Wk, int wld,
                                           const float* __restrict__ bias, float* __restrict__ OUT, int JPx) {
  if (RPL == 0) {
    tile_layer8<ACT>(A, K, Wk, wld, bias, OUT, JPx);
    return;
  }
  constexpr int RRS = ROWS + TILE_PAD;
  constexpr int NGRP = RPL > 0 ? ROWS / (32 * RPL) : 1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cg = NGRP == 1 ? warp : warp & 3;
  const int r0 = (NGRP == 1 ? 0 : (warp >> 2) * 32 * RPL) + lane * RPL;
  for (int jh = 0; jh < JPx / 32; ++jh) {
    const int j0 = jh * 32 + cg * 8;
    float acc[RPL > 0 ? RPL : 1][8];
#pragma unroll
    for (int a = 0; a < RPL; ++a)
#pragma unroll
      for (int t = 0; t < 8; ++t) acc[a][t] = 0.f;
#pragma unroll 4
    for (int k = 0; k < K; ++k) {
      float av[RPL > 0 ? RPL : 1];
      if (RPL == 4) {
        const float4 a4 = ld4(A + k * RRS + r0);
        av[0] = a4.x, av[RPL > 1 ? 1 : 0] = a4.y, av[RPL > 2 ? 2 : 0] = a4.z, av[RPL > 3 ? 3 : 0] = a4.w;
      } else if (RPL == 2) {
        const float2 a2 = *reinterpret_cast<const float2*>(A + k * RRS + r0);
        av[0] = a2.x, av[RPL > 1 ? 1 : 0] = a2.y;
      } else {
        av[0] = A[k * RRS + r0];
      }
      const float4 w0 = ld4(Wk + k * wld + j0), w1 = ld4(Wk + k * wld + j0 + 4);
      const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int x = 0; x < RPL; ++x)
#pragma unroll
        for (int t = 0; t < 8; ++t) acc[x][t] = fmaf(av[x], w[t], acc[x][t]);
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const float b = bias[j0 + t];
#pragma unroll
      for (int x = 0; x < RPL; ++x) {
        const float z = acc[x][t] + b;
        OUT[(j0 + t) * RRS + r0 + x] = ACT == ACT_TANH ? tanh_fast(z) : fmaxf(z, 0.f);
      }
    }
  }
}

// dL/dz of a ReLU layer contracted with the next layer's weights, for the 4 rows r0..r0+3 and 8 columns j0..j0+7:
//   acc[x][t] += sum_k D[k][r0 + x] * Wk[k * wld + j0 + t],   D[k][r] = (S[k][r] > 0) ? g_r * sk[k] : 0
// S: the layer's post-activation tile (feature-major, row stride RS); g: the upstream scalar of each of the 4 rows;
// sk: per-k scale; Wk: k-major weights (row stride wld, 16-byte aligned).
__device__ __forceinline__ void gemm_acc(float (&acc)[4][8], const float* __restrict__ S, int RS, int r0,
                                         const float* __restrict__ Wk, int wld, int j0, int K, const float4 g,
                                         const float* __restrict__ sk) {
#pragma unroll 2
  for (int k = 0; k < K; ++k) {
    float4 a = ld4(S + k * RS + r0);
    const float s = sk[k];
    a.x = a.x > 0.f ? g.x * s : 0.f;
    a.y = a.y > 0.f ? g.y * s : 0.f;
    a.z = a.z > 0.f ? g.z * s : 0.f;
    a.w = a.w > 0.f ? g.w * s : 0.f;
    const float4 w0 = ld4(Wk + k * wld + j0), w1 = ld4(Wk + k * wld + j0 + 4);
    const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
      for (int t = 0; t < 8; ++t) acc[x][t] = fmaf(av[x], w[t], acc[x][t]);
  }
}

// Weight-gradient contraction over tile rows [ra, rb) (multiples of 4):
//   acc[jj][ii] += sum_r D[jb + jl + 8*jj][r] * ACT[ib + il + 4*ii][r]     jj < 4, ii < 8
//   bacc[jj]    += sum_r D[jb + jl + 8*jj][r]                             (bias gradient)
// One warp (jl = lane % 8, il = lane / 8) covers a 32 x 32 block of the weight gradient; the j set
// is strided by 8 so the 8 lanes of an LDS.128 phase read 8 consecutive feature rows (conflict-free
// with the 4-bank stagger) and the ACT loads are phase-uniform broadcasts.
// MASK: D is generated on the fly as (S[j][r] > 0) ? g[r] * sj[jj] : 0.
template <bool MASK>
__device__ __forceinline__ void wgrad_acc(float (&acc)[4][8], float (&bacc)[4], const float* __restrict__ D,
                                          const float* __restrict__ ACT, int RS, int jrow0, int irow0, int ra, int rb,
                                          const float* __restrict__ gvec, const float (&sj)[4]) {
  for (int r = ra; r < rb; r += 4) {
    float4 d[4];
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) d[jj] = ld4(D + (jrow0 + 8 * jj) * RS + r);
    if (MASK) {
      const float4 g = ld4(gvec + r);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        d[jj].x = d[jj].x > 0.f ? g.x * sj[jj] : 0.f;
        d[jj].y = d[jj].y > 0.f ? g.y * sj[jj] : 0.f;
        d[jj].z = d[jj].z > 0.f ? g.z * sj[jj] : 0.f;
        d[jj].w = d[jj].w > 0.f ? g.w * sj[jj] : 0.f;
      }
    }
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) bacc[jj] += (d[jj].x + d[jj].y) + (d[jj].z + d[jj].w);
#pragma unroll
    for (int ii = 0; ii < 8; ++ii) {
      const float4 a = ld4(ACT + (irow0 + 4 * ii) * RS + r);
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        float t = acc[jj][ii];
        t = fmaf(d[jj].x, a.x, t);
        t = fmaf(d[jj].y, a.y, t);
        t = fmaf(d[jj].z, a.z, t);
        t = fmaf(d[jj].w, a.w, t);
        acc[jj][ii] = t;
      }
    }
  }
}

// Shared-memory image of one MLP, hidden widths padded to JP (32 or 64), everything zero padded:
//   W1t[din][JP] b1[JP] W2t[JP][JP] W2[JP][JP] b2[JP] wf[64] bf,pad[4] mean[64] istd[64]
struct TImg {
  __host__ __device__ static int w1t(int, int) { return 0; }
  __host__ __device__ static int b1(int din, int JP) { return din * JP; }
  __host__ __device__ static int w2t(int din, int JP) { return din * JP + JP; }
  __host__ __device__ static int w2(int din, int JP) { return din * JP + JP + JP * JP; }
  __host__ __device__ static int b2(int din, int JP) { return din * JP + JP + 2 * JP * JP; }
  __host__ __device__ static int wf(int din, int JP) { return din * JP + 2 * JP + 2 * JP * JP; }
  __host__ __device__ static int bf(int din, int JP) { return wf(din, JP) + 64; }
  __host__ __device__ static int mean(int din, int JP) { return bf(din, JP) + 4; }
  __host__ __device__ static int istd(int din, int JP) { return mean(din, JP) + 64; }
  __host__ __device__ static int size(int din, int JP) { return istd(din, JP) + 64; }
};

__device__ void load_timg(float* sm, const PassDesc& p, int JP, const float* __restrict__ params,
                          const float* __restrict__ norm, float eps) {
  const int din = p.din, tid = threadIdx.x, nt = blockDim.x;
  const float* q = params + p.param_off;
  for (int i = tid; i < TImg::mean(din, JP); i += nt) sm[i] = 0.f;
  __syncthreads();
  int off = 0, hl = din;
  // (loops unrolled so that the global loads of 8 iterations are in flight together: the image build is the
  //  whole prologue of a CTA that processes a single tile)
  if (p.n_hidden >= 1) {
#pragma unroll 8
    for (int i = tid; i < p.h1 * din; i += nt) {
      const int j = i / din, k = i - j * din;
      sm[TImg::w1t(din, JP) + k * JP + j] = q[off + i];
    }
    off += p.h1 * din;
    for (int i = tid; i < p.h1; i += nt) sm[TImg::b1(din, JP) + i] = q[off + i];
    off += p.h1;
    hl = p.h1;
  }
  if (p.n_hidden >= 2) {
#pragma unroll 8
    for (int i = tid; i < p.h2 * p.h1; i += nt) {
      const int j = i / p.h1, ii = i - j * p.h1;
      const float v = q[off + i];
      sm[TImg::w2(din, JP) + j * JP + ii] = v;
      sm[TImg::w2t(din, JP) + ii * JP + j] = v;
    }
    off += p.h2 * p.h1;
    for (int i = tid; i < p.h2; i += nt) sm[TImg::b2(din, JP) + i] = q[off + i];
    off += p.h2;
    hl = p.h2;
  }
  for (int i = tid; i < hl; i += nt) sm[TImg::wf(din, JP) + i] = q[off + i];
  off += hl;
  if (tid == 0) sm[TImg::bf(din, JP)] = q[off];
  for (int i = tid; i < din; i += nt) {
    sm[TImg::mean(din, JP) + i] = norm ? norm[i] : 0.f;
    sm[TImg::istd(din, JP) + i] = norm ? 1.0f / sqrtf(norm[din + i] + eps) : 1.f;
  }
}

// Forward of one row held by this thread through the TImg image `img` (hidden width JP): xn holds the row's
// normalised inputs (stride 1); register accumulators, one broadcast weight per FMA.
template <int JP>
__device__ __forceinline__ float timg_forward_row(const float* __restrict__ img, const PassDesc& p,
                                                  const float* __restrict__ xn) {
  const int din = p.din;
  const float* wf = img + TImg::wf(din, JP);
  const float bf = img[TImg::bf(din, JP)];
  if (p.n_hidden == 0) {
    float acc = bf;
    for (int k = 0; k < din; ++k) acc = fmaf(wf[k], xn[k], acc);
    return acc;
  }
  const float* W1t = img + TImg::w1t(din, JP);
  const float* b1 = img + TImg::b1(din, JP);
  float h1[JP], h2[JP];
#pragma unroll
  for (int j = 0; j < JP; ++j) h1[j] = b1[j];
  for (int k = 0; k < din; ++k) {
    const float xv = xn[k];
    const float4* w = reinterpret_cast<const float4*>(W1t + k * JP);
#pragma unroll
    for (int j4 = 0; j4 < JP / 4; ++j4) {
      const float4 ww = w[j4];
      h1[4 * j4 + 0] = fmaf(ww.x, xv, h1[4 * j4 + 0]);
      h1[4 * j4 + 1] = fmaf(ww.y, xv, h1[4 * j4 + 1]);
      h1[4 * j4 + 2] = fmaf(ww.z, xv, h1[4 * j4 + 2]);
      h1[4 * j4 + 3] = fmaf(ww.w, xv, h1[4 * j4 + 3]);
    }
  }
#pragma unroll
  for (int j = 0; j < JP; ++j) h1[j] = fmaxf(h1[j], 0.f);
  if (p.n_hidden == 1) {
    float acc = bf;
#pragma unroll
    for (int j = 0; j < JP; ++j) acc = fmaf(wf[j], h1[j], acc);
    return acc;
  }
  const float* W2t = img + TImg::w2t(din, JP);
  const float* b2 = img + TImg::b2(din, JP);
#pragma unroll
  for (int j = 0; j < JP; ++j) h2[j] = b2[j];
#pragma unroll
  for (int i = 0; i < JP; ++i) {
    const float hv = h1[i];
    const float4* w = reinterpret_cast<const float4*>(W2t + i * JP);
#pragma unroll
    for (int j4 = 0; j4 < JP / 4; ++j4) {
      const float4 ww = w[j4];
      h2[4 * j4 + 0] = fmaf(ww.x, hv, h2[4 * j4 + 0]);
      h2[4 * j4 + 1] = fmaf(ww.y, hv, h2[4 * j4 + 1]);
      h2[4 * j4 + 2] = fmaf(ww.z, hv, h2[4 * j4 + 2]);
      h2[4 * j4 + 3] = fmaf(ww.w, hv, h2[4 * j4 + 3]);
    }
  }
  float acc = bf;
#pragma unroll
  for (int j = 0; j < JP; ++j) acc = fmaf(wf[j], fmaxf(h2[j], 0.f), acc);
  return acc;
}

// Shared-memory image of the policy (SB3 ActorCriticPolicy, tower width padded to HP, everything zero padded):
//   piW1t[Do][HP] pib1[HP] piW2t[HP][HP] pib2[HP] vfW1t vfb1 vfW2t vfb2 Wa[Da][HP] ba[64] wv[HP] bv[4] lstd[64] mean[64] istd[64]
struct PolImg {
  int w1p, b1p, w2p, b2p, w1v, b1v, w2v, b2v, wa, ba, wv, bv, lstd, mean, istd, total;
  __host__ __device__ PolImg(int Do, int Da, int HP) {
    int o = 0;
    w1p = o; o += Do * HP;
    b1p = o; o += HP;
    w2p = o; o += HP * HP;
    b2p = o; o += HP;
    w1v = o; o += Do * HP;
    b1v = o; o += HP;
    w2v = o; o += HP * HP;
    b2v = o; o += HP;
    wa = o; o += Da * HP;
    ba = o; o += 64;
    wv = o; o += HP;
    bv = o; o += 4;
    lstd = o; o += 64;
    mean = o; o += 64;
    istd = o; o += 64;
    total = o;
  }
};

__device__ void load_policy_img(float* sm, const PolImg& S, const imb_policy_desc& pd, int HP,
                                const float* __restrict__ q, const float* __restrict__ norm) {
  const int tid = threadIdx.x, nt = blockDim.x;
  const int Do = pd.d_obs, Da = pd.d_act, h = pd.hidden;
  for (int i = tid; i < S.total; i += nt) sm[i] = 0.f;
  __syncthreads();
#pragma unroll 4
  for (int i = tid; i < h * Do; i += nt) {
    const int j = i / Do, k = i - j * Do;
    sm[S.w1p + k * HP + j] = q[pd.off_pi_w1 + i];
    sm[S.w1v + k * HP + j] = q[pd.off_vf_w1 + i];
  }
#pragma unroll 4
  for (int i = tid; i < h * h; i += nt) {
    const int j = i / h, ii = i - j * h;
    sm[S.w2p + ii * HP + j] = q[pd.off_pi_w2 + i];
    sm[S.w2v + ii * HP + j] = q[pd.off_vf_w2 + i];
  }
  for (int i = tid; i < h; i += nt) {
    sm[S.b1p + i] = q[pd.off_pi_b1 + i];
    sm[S.b2p + i] = q[pd.off_pi_b2 + i];
    sm[S.b1v + i] = q[pd.off_vf_b1 + i];
    sm[S.b2v + i] = q[pd.off_vf_b2 + i];
    sm[S.wv + i] = q[pd.off_val_w + i];
  }
  for (int i = tid; i < Da * h; i += nt) {
    const int a = i / h, ii = i - a * h;
    sm[S.wa + a * HP + ii] = q[pd.off_act_w + i];
  }
  for (int i = tid; i < Da; i += nt) {
    sm[S.ba + i] = q[pd.off_act_b + i];
    if (!pd.discrete) sm[S.lstd + i] = q[pd.off_log_std + i];
  }
  if (tid == 0) sm[S.bv] = q[pd.off_val_b];
  for (int i = tid; i < Do; i += nt) {
    sm[S.mean + i] = pd.has_norm ? norm[i] : 0.f;
    sm[S.istd + i] = pd.has_norm ? 1.0f / sqrtf(norm[Do + i] + pd.norm_eps) : 1.f;
  }
}


}  // namespace
