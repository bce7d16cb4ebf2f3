// imb_density.cu -- the kernel density reward of DensityAlgorithm (algorithms/density.py:295-360): every query row
// scored against the standardised demonstration rows of its segment (include/imb.h, imb_density_score).
//
// The reference calls sklearn KernelDensity.score once per transition in a Python loop; here one launch scores all of
// them.  A CTA owns a tile of 64 queries (standardised into shared memory once) and streams the demonstration tiles of
// the queries' segments through two shared-memory stages, each filled by cp.async.bulk on an mbarrier while the other
// is consumed.  Its 256 threads each hold 4 queries x 4 demonstration rows: per feature, two 16-byte shared loads feed
// 16 differences and 16 FMAs (the direct sum_k (q_k - x_k)^2, which keeps its accuracy at small bandwidths where the
// |q|^2 + |x|^2 - 2 q.x expansion cancels).  The log kernel values then enter a per-query online log-sum-exp (running
// max and sum), merged over the 16 threads that share a query by a fixed shuffle tree.  A pair counts only when the
// demonstration row belongs to the query's segment, so a tile may mix segments (non-stationary models, whose segments
// hold about one row per demonstration trajectory) and segments may have any sizes.  When there are too few query tiles
// to fill the GPU, the demonstration tiles of a query tile are dealt round-robin to `nsplit` CTAs and the last of them
// to finish (ticket) merges the partial (max, sum) pairs in split order.
#include <climits>

#include "imb_common.cuh"

namespace {

constexpr int DT = IMB_DENSITY_TILE;  // demonstration rows per tile = queries per query tile
constexpr int DTHREADS = 256;         // 16 x 16 threads of 4 queries x 4 demonstration rows
// The split aims at this many CTAs (two per SM of a 132-SM H100).  It is a constant, not the device's SM count, so that
// the summation order, and with it every result bit, depends only on the shapes.
constexpr int64_t SPLIT_TARGET = 264;
constexpr int64_t MAX_SPLIT = 64;

// the model: imb_density_score's arguments d .. scale (include/imb.h)
struct DensityModel {
  int d, col0, n0, col1, n1, kernel;
  float bandwidth;
  int n_seg;
  int64_t n_demo;
  const float* demo;
  const int32_t* demo_seg;
  const int64_t* seg_off;
  const double* seg_const;
  const float* mean;
  const float* scale;
};

struct DensityLaunch {
  DensityModel d;
  const float* src;
  int ld;
  const int64_t* row_map;
  int64_t n_query;
  int seg_mode;
  const int64_t* steps;
  const int64_t* state;
  int64_t E, T;
  int H;
  float* out;
  int64_t out_stride;
  unsigned int* tickets;  // [n_qtiles]
  float* partial;         // [n_qtiles][nsplit][DT][2] (max, sum)
  int nsplit;
  float h, inv_h, inv_h2, c_gauss;
};

// log of sklearn's unnormalised kernel (neighbors/_binary_tree.pxi.tp compute_log_kernel) at squared distance d2
template <int K>
__device__ __forceinline__ float log_kernel(float d2, const DensityLaunch& P) {
  if (K == IMB_KDE_GAUSSIAN) return d2 * P.c_gauss;  // -0.5 d^2 / h^2
  const float dist = sqrtf(d2);
  if (K == IMB_KDE_EXPONENTIAL) return -dist * P.inv_h;
  if (!(dist < P.h)) return -INFINITY;  // compact kernels: strict d < h
  if (K == IMB_KDE_TOPHAT) return 0.f;
  if (K == IMB_KDE_EPANECHNIKOV) return logf(1.f - d2 * P.inv_h2);
  if (K == IMB_KDE_LINEAR) return logf(1.f - dist * P.inv_h);
  return logf(cospif(0.5f * dist * P.inv_h));  // cosine: cos(pi d / (2 h))
}

// (m, s) <- the log-sum-exp pair of (m, s) and (m2, s2): exp(m) s + exp(m2) s2 = exp(m') s'
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  if (m2 == -INFINITY) return;
  if (m2 > m) {
    s = s * __expf(m - m2) + s2;
    m = m2;
  } else {
    s += s2 * __expf(m2 - m);
  }
}

__device__ __forceinline__ void finish(const DensityLaunch& P, int64_t out_row, int seg, float m, float s) {
  if (out_row < 0) return;
  double v = NAN;
  if (seg >= 0) v = (s > 0.f ? (double)m + log((double)s) : -INFINITY) + P.d.seg_const[seg];
  P.out[out_row * P.out_stride] = (float)v;
}

template <int K>
__global__ void __launch_bounds__(DTHREADS) k_density(const DensityLaunch P) {
  extern __shared__ __align__(128) float smem[];
  const int D = P.d.d;
  float* Q = smem;                                       // [D][DT] standardised queries
  float* X = smem + D * DT;                              // [2][D][DT] demonstration tile stages
  int* XS = reinterpret_cast<int*>(X + 2 * D * DT);      // [2][DT] their rows' segments
  __shared__ __align__(8) uint64_t bar[2];
  __shared__ int64_t q_src[DT], q_out[DT];
  __shared__ int q_seg[DT];
  __shared__ int seg_lo, seg_hi;
  __shared__ bool is_last;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t qt = blockIdx.x;
  const int z = blockIdx.y, nsplit = P.nsplit;

  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
    seg_lo = INT_MAX;
    seg_hi = -1;
  }
  __syncthreads();
  // ---- the tile's queries: source row, output row, segment ---------------------------------------------------------
  if (tid < DT) {
    const int64_t q = qt * DT + tid;
    int64_t src_row = -1, out_row = -1;
    int seg = -1;
    if (q < P.n_query) {
      int64_t s64 = 0;
      if (P.seg_mode == IMB_DENSITY_SEG_ROLLOUT) {
        const int64_t t0 = P.state[IMB_ST_EP_STEP];
        const int64_t t = q / P.E, e = q - t * P.E;
        src_row = flat_index(e, t, P.E, P.T, t0, P.H);
        out_row = e * P.T + t;
        s64 = P.d.n_seg == 1 ? 0 : (t0 + t) % P.H;
      } else {
        src_row = out_row = P.row_map ? P.row_map[q] : q;
        if (P.seg_mode == IMB_DENSITY_SEG_STEPS) s64 = P.steps[q];
      }
      seg = (s64 >= 0 && s64 < P.d.n_seg) ? (int)s64 : -2;  // -2: out of range, scores NaN
      if (seg >= 0) {
        atomicMin(&seg_lo, seg);
        atomicMax(&seg_hi, seg);
      }
    }
    q_src[tid] = src_row;
    q_out[tid] = out_row;
    q_seg[tid] = seg;
  }
  __syncthreads();
  for (int i = tid; i < D * DT; i += DTHREADS) {
    const int k = i / DT, r = i - k * DT;
    const int64_t row = q_src[r];
    float v = 0.f;
    if (row >= 0) {
      const int col = k < P.d.n0 ? P.d.col0 + k : P.d.col1 + (k - P.d.n0);
      v = (P.src[row * P.ld + col] - P.d.mean[k]) / P.d.scale[k];  // StandardScaler.transform
    }
    Q[i] = v;
  }
  // ---- the demonstration tiles of the queries' segments, every nsplit-th from tile b_lo + z ------------------------
  int64_t b_lo = 0, n_it = 0;
  if (seg_hi >= 0) {
    const int64_t r_lo = P.d.seg_off[seg_lo], r_hi = P.d.seg_off[seg_hi + 1];
    b_lo = r_lo / DT;
    const int64_t n_b = (r_hi + DT - 1) / DT - b_lo;
    n_it = n_b > z ? (n_b - z + nsplit - 1) / nsplit : 0;
  }
  const uint32_t tile_bytes = (uint32_t)(D * DT * 4);
  auto issue = [&](int64_t it, int st) {
    const int64_t b = b_lo + z + it * nsplit;
    mbar_expect_tx(&bar[st], tile_bytes + DT * 4);
    bulk_g2s(X + st * D * DT, P.d.demo + b * D * DT, tile_bytes, &bar[st]);
    bulk_g2s(XS + st * DT, P.d.demo_seg + b * DT, DT * 4, &bar[st]);
  };
  if (tid == 0 && n_it > 0) issue(0, 0);
  __syncthreads();  // Q complete

  int qs[4];
  float m[4], s[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    qs[r] = q_seg[ty * 4 + r];
    m[r] = -INFINITY;
    s[r] = 0.f;
  }
  for (int64_t it = 0; it < n_it; ++it) {
    const int st = (int)(it & 1);
    // stage st ^ 1 was consumed in the previous iteration, which every thread has left (barrier at its end)
    if (tid == 0 && it + 1 < n_it) issue(it + 1, st ^ 1);
    mbar_wait(&bar[st], (uint32_t)((it >> 1) & 1));
    const float* Xs = X + st * D * DT;
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
#pragma unroll 4
    for (int k = 0; k < D; ++k) {
      const float4 qv = *reinterpret_cast<const float4*>(Q + k * DT + ty * 4);
      const float4 xv = *reinterpret_cast<const float4*>(Xs + k * DT + tx * 4);
      const float qa[4] = {qv.x, qv.y, qv.z, qv.w}, xa[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float df = qa[r] - xa[c];
          acc[r][c] = fmaf(df, df, acc[r][c]);
        }
    }
    const int4 xs = *reinterpret_cast<const int4*>(XS + st * DT + tx * 4);
    const int xsa[4] = {xs.x, xs.y, xs.z, xs.w};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float lk[4], mt = -INFINITY;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        lk[c] = xsa[c] == qs[r] ? log_kernel<K>(acc[r][c], P) : -INFINITY;
        mt = fmaxf(mt, lk[c]);
      }
      if (mt != -INFINITY) {
        if (mt > m[r]) {
          s[r] *= __expf(m[r] - mt);
          m[r] = mt;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) s[r] += __expf(lk[c] - m[r]);
      }
    }
    __syncthreads();
  }
  // ---- merge over the 16 threads of a query row (fixed tree; lane tx = 0 holds the result) --------------------------
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m[r], o), s2 = __shfl_xor_sync(0xffffffffu, s[r], o);
      lse_merge(m[r], s[r], m2, s2);
    }
  if (nsplit == 1) {
    if (tx == 0)
#pragma unroll
      for (int r = 0; r < 4; ++r) finish(P, q_out[ty * 4 + r], q_seg[ty * 4 + r], m[r], s[r]);
    return;
  }
  float* part = P.partial + (qt * nsplit + z) * DT * 2;
  if (tx == 0)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      part[(ty * 4 + r) * 2] = m[r];
      part[(ty * 4 + r) * 2 + 1] = s[r];
    }
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = atomicAdd(P.tickets + qt, 1u) == (unsigned)nsplit - 1u;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (tid < DT) {
    const float* p0 = P.partial + qt * nsplit * DT * 2 + tid * 2;
    float mm = -INFINITY, ss = 0.f;
    for (int zz = 0; zz < nsplit; ++zz) lse_merge(mm, ss, __ldcg(p0 + zz * DT * 2), __ldcg(p0 + zz * DT * 2 + 1));
    finish(P, q_out[tid], q_seg[tid], mm, ss);
  }
  if (tid == 0) P.tickets[qt] = 0u;  // re-arm for the next call
}

int64_t n_qtiles_of(int64_t n_query) { return (n_query + DT - 1) / DT; }
int64_t max_split_of(int64_t n_qtiles) {
  const int64_t s = (SPLIT_TARGET + n_qtiles - 1) / n_qtiles;
  return s < 1 ? 1 : (s > MAX_SPLIT ? MAX_SPLIT : s);
}
int64_t tickets_floats(int64_t n_qtiles) { return (n_qtiles + 3) / 4 * 4; }

template <int K>
int launch_density(const DensityLaunch& P, int64_t n_qtiles, cudaStream_t st) {
  const size_t smem = (size_t)(3 * P.d.d * DT + 2 * DT) * 4;
  cudaError_t e = cudaFuncSetAttribute(k_density<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) IMB_FAIL(-2, "cudaFuncSetAttribute(k_density, %zu): %s", smem, cudaGetErrorString(e));
  k_density<K><<<dim3((unsigned)n_qtiles, (unsigned)P.nsplit), DTHREADS, smem, st>>>(P);
  IMB_CHECK_LAUNCH("k_density");
  return 0;
}

}  // namespace

extern "C" int64_t imb_density_ws_floats(int64_t n_query) {
  if (n_query <= 0) return 0;
  const int64_t nq = n_qtiles_of(n_query);
  return tickets_floats(nq) + nq * max_split_of(nq) * DT * 2;
}

extern "C" int imb_density_score(int32_t d_, int32_t col0, int32_t n0, int32_t col1, int32_t n1, int32_t kernel,
                                 float bandwidth, int32_t n_seg, int64_t n_demo, const float* demo,
                                 const int32_t* demo_seg, const int64_t* seg_off, const double* seg_const,
                                 const float* mean, const float* scale, const float* src, int32_t src_ld,
                                 const int64_t* row_map, int64_t n_query, int32_t seg_mode, const int64_t* steps,
                                 const int64_t* state, int64_t n_envs, int64_t n_steps, int32_t horizon, float* out,
                                 int64_t out_stride, float* ws, void* stream) {
  const DensityModel model{d_, col0, n0, col1, n1, kernel, bandwidth, n_seg, n_demo, demo, demo_seg, seg_off,
                           seg_const, mean, scale};
  const DensityModel* d = &model;
  IMB_REQUIRE(d->d >= 1 && d->d <= IMB_DENSITY_MAX_D, "imb_density_score: feature width %d outside [1, %d]", d->d,
              IMB_DENSITY_MAX_D);
  IMB_REQUIRE(d->n0 >= 0 && d->n1 >= 0 && d->n0 + d->n1 == d->d && d->col0 >= 0 && d->col1 >= 0,
              "imb_density_score: feature columns (%d, %d) + (%d, %d) do not give width %d", d->col0, d->n0, d->col1,
              d->n1, d->d);
  IMB_REQUIRE(src_ld >= d->col0 + d->n0 && src_ld >= d->col1 + d->n1, "imb_density_score: source rows of %d floats are "
              "narrower than the feature columns", src_ld);
  IMB_REQUIRE(d->kernel >= IMB_KDE_GAUSSIAN && d->kernel <= IMB_KDE_COSINE, "imb_density_score: unknown kernel %d",
              d->kernel);
  IMB_REQUIRE(d->bandwidth > 0.f && d->bandwidth < INFINITY, "imb_density_score: bandwidth must be positive");
  IMB_REQUIRE(d->n_seg >= 1 && d->n_demo >= 1, "imb_density_score: no demonstrations (%d segments, %lld rows)",
              d->n_seg, (long long)d->n_demo);
  IMB_REQUIRE(d->demo && d->demo_seg && d->seg_off && d->seg_const && d->mean && d->scale,
              "imb_density_score: null demonstration pointer");
  IMB_REQUIRE(seg_mode >= IMB_DENSITY_SEG_NONE && seg_mode <= IMB_DENSITY_SEG_ROLLOUT,
              "imb_density_score: unknown segment mode %d", seg_mode);
  IMB_REQUIRE(seg_mode != IMB_DENSITY_SEG_STEPS || steps, "imb_density_score: segment mode STEPS needs steps");
  if (seg_mode == IMB_DENSITY_SEG_ROLLOUT) {
    IMB_REQUIRE(state && horizon >= 1 && n_envs >= 1 && n_steps >= 1 && n_query == n_envs * n_steps,
                "imb_density_score: the rollout mode needs the state block, horizon >= 1 and n_query = n_envs * n_steps");
    IMB_REQUIRE(row_map == nullptr, "imb_density_score: the rollout mode takes no row map");
  }
  IMB_REQUIRE(n_query >= 0, "imb_density_score: negative query count");
  if (n_query == 0) return 0;
  IMB_REQUIRE(src && out && ws, "imb_density_score: null source, output or workspace");
  const int64_t nq = n_qtiles_of(n_query);
  IMB_REQUIRE(nq < (1ll << 31), "imb_density_score: too many queries");
  const int64_t n_tiles = (d->n_demo + DT - 1) / DT;
  // demonstration tiles a query tile reads: all of them (stationary), about those of one segment plus one otherwise
  const int64_t per_qtile = d->n_seg == 1 ? n_tiles : (n_tiles + d->n_seg - 1) / d->n_seg + 1;
  int64_t nsplit = nq >= SPLIT_TARGET ? 1 : max_split_of(nq);
  if (nsplit > per_qtile) nsplit = per_qtile;
  if (nsplit < 1) nsplit = 1;

  DensityLaunch P;
  P.d = *d;
  P.src = src;
  P.ld = src_ld;
  P.row_map = row_map;
  P.n_query = n_query;
  P.seg_mode = seg_mode;
  P.steps = steps;
  P.state = state;
  P.E = n_envs;
  P.T = n_steps;
  P.H = horizon;
  P.out = out;
  P.out_stride = out_stride;
  P.tickets = reinterpret_cast<unsigned int*>(ws);
  P.partial = ws + tickets_floats(nq);
  P.nsplit = (int)nsplit;
  const double h = (double)d->bandwidth;
  P.h = d->bandwidth;
  P.inv_h = (float)(1.0 / h);
  P.inv_h2 = (float)(1.0 / (h * h));
  P.c_gauss = (float)(-0.5 / (h * h));
  cudaStream_t st = (cudaStream_t)stream;
  switch (d->kernel) {
    case IMB_KDE_GAUSSIAN: return launch_density<IMB_KDE_GAUSSIAN>(P, nq, st);
    case IMB_KDE_TOPHAT: return launch_density<IMB_KDE_TOPHAT>(P, nq, st);
    case IMB_KDE_EPANECHNIKOV: return launch_density<IMB_KDE_EPANECHNIKOV>(P, nq, st);
    case IMB_KDE_EXPONENTIAL: return launch_density<IMB_KDE_EXPONENTIAL>(P, nq, st);
    case IMB_KDE_LINEAR: return launch_density<IMB_KDE_LINEAR>(P, nq, st);
    default: return launch_density<IMB_KDE_COSINE>(P, nq, st);
  }
}
