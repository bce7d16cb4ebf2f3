// imb_common.cuh -- shared device/host helpers for libimb.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "imb.h"

// opt-in dynamic shared memory ceiling: 227 KB per CTA minus room for static __shared__ data
#define IMB_SMEM_MAX (226 * 1024)

// ---- error plumbing (thread-local text, negative codes) ------------------------------------
extern thread_local char g_imb_err[512];
#define IMB_FAIL(code, ...)                                   \
  do {                                                        \
    snprintf(g_imb_err, sizeof(g_imb_err), __VA_ARGS__);      \
    return (code);                                            \
  } while (0)
#define IMB_CHECK_LAUNCH(name)                                                       \
  do {                                                                               \
    cudaError_t e__ = cudaGetLastError();                                            \
    if (e__ != cudaSuccess) IMB_FAIL(-2, "%s: %s", name, cudaGetErrorString(e__));   \
  } while (0)
#define IMB_REQUIRE(cond, ...)            \
  do {                                    \
    if (!(cond)) IMB_FAIL(-1, __VA_ARGS__); \
  } while (0)

// floats per rollout-table row: obs | action (one column when discrete) | 5 scalars, padded to a multiple of 4 floats so
// that rows are 16-byte aligned and the PPO update can stage a minibatch row with 16-byte copies
__host__ __device__ constexpr int imb_row_width(int d_obs, int d_act, bool discrete) {
  return (d_obs + (discrete ? 1 : d_act) + 5 + 3) / 4 * 4;
}

static inline int imb_num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Flattened (reference-order) index of local step t of env e in a rollout of T steps of E lock-step envs of horizon H
// that starts at episode step t0: the order pop_trajectories + flatten_trajectories give (finished trajectories in
// completion order, then the partial ones in env order; imb_rollout_impl.cuh).  The rollout writes its transition rows
// there and imb_density_score reads them back from there.
__device__ __forceinline__ int64_t flat_index(int64_t e, int64_t t, int64_t E, int64_t T, int64_t t0, int64_t H) {
  const int64_t seg = (t0 + t) / H;
  const int64_t start = seg == 0 ? 0 : seg * H - t0;
  int64_t end = (seg + 1) * H - t0;
  if (end > T) end = T;
  return E * start + e * (end - start) + (t - start);
}

// ---- warp helpers ---------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- mbarrier + 1-D bulk async copy (TMA unit; SASS: UBLKCP) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// bounded wait: a lost/never-issued copy traps (kernel error) instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spins = 0; !mbar_try_wait(bar, parity); ++spins) {
    if (spins > (1u << 22)) __trap();
  }
}
// global -> shared bulk copy, completion signalled on an mbarrier (bytes multiple of 16,
// both addresses 16-byte aligned).
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- Philox4x32-10 (bit-exact twin of oracle/philox.py) ---------------------------------------
#define IMB_STREAM_ENV_RESET 0x1001u
#define IMB_STREAM_ACT_NOISE 0x2002u
#define IMB_STREAM_REPLAY 0x3003u
#define IMB_STREAM_EXPERT 0x4004u
#define IMB_STREAM_PPO_PERM 0x5005u
#define IMB_STREAM_EXPLORE 0x7007u  // random-policy actions of the exploration rollout (0x6006: oracle expert policy)
#define IMB_STREAM_DAGGER 0x8008u   // the learner's sampled actions in the DAgger rollout
#define IMB_STREAM_SAC_ACT 0x9009u     // SAC collection: the actor's noise (imb_sac_collect)
#define IMB_STREAM_SAC_RANDOM 0xA00Au  // SAC collection: the warm-up steps' action_space.sample()
#define IMB_STREAM_SAC_STEP 0xB00Bu    // SAC gradient step: the actor's noise on s and s' (imb_sac_step)

struct Philox4 {
  uint32_t x, y, z, w;
};
__host__ __device__ __forceinline__ Philox4 philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                       uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
    uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0;
    c1 = lo1;
    c2 = n2;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
__host__ __device__ __forceinline__ void philox_key(uint64_t seed, uint32_t stream, uint32_t& k0, uint32_t& k1) {
  k0 = (uint32_t)seed;
  k1 = (uint32_t)(seed >> 32) ^ stream;
}
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * 5.9604644775390625e-08f; }
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  float u1 = u01(a), u2 = u01(b);
  float r = sqrtf(-2.0f * logf(u1));
  float th = 6.283185307179586f * u2;
  z0 = r * cosf(th);
  z1 = r * sinf(th);
}
// j-th float32 normal of counter (a, b): chunk j/4, lane j%4 (matches philox.normals()).
__device__ __forceinline__ float philox_normal(uint64_t seed, uint32_t stream, uint32_t a, uint32_t b, int j) {
  uint32_t k0, k1;
  philox_key(seed, stream, k0, k1);
  Philox4 r = philox4x32(a, b, (uint32_t)(j >> 2), 0u, k0, k1);
  float z0, z1;
  if ((j & 2) == 0)
    box_muller(r.x, r.y, z0, z1);
  else
    box_muller(r.z, r.w, z0, z1);
  return (j & 1) ? z1 : z0;
}
// the four normals of chunk c of counter (a, b): z[j % 4] == philox_normal(..., 4 c + j % 4) bit for bit, with one
// Philox call and two Box-Muller transforms instead of four of each
__device__ __forceinline__ void philox_normal4(uint64_t seed, uint32_t stream, uint32_t a, uint32_t b, int chunk,
                                               float (&z)[4]) {
  uint32_t k0, k1;
  philox_key(seed, stream, k0, k1);
  const Philox4 r = philox4x32(a, b, (uint32_t)chunk, 0u, k0, k1);
  box_muller(r.x, r.y, z[0], z[1]);
  box_muller(r.z, r.w, z[2], z[3]);
}
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7FEB352Du;
  x ^= x >> 15;
  x *= 0x846CA68Bu;
  x ^= x >> 16;
  return x;
}
// 4-byte asynchronous global -> shared copy (LDGSTS); completion via cp_async_wait_all + __syncthreads
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
}
// the mbarrier receives one arrival (counted in its expected-arrival count) once all cp.async of this thread
// issued so far have completed
__device__ __forceinline__ void cp_async_mbar_arrive(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// split cluster barrier (release / acquire): DSMEM stores before the arrive are visible after the wait
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }

// distributed shared memory: address of the same shared-memory location in CTA `rank` of the cluster, and an
// asynchronous 16-byte remote store that completes bytes on an mbarrier of the receiving CTA
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_saddr, int rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_saddr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_async_v4(uint32_t remote_saddr, const float4& v, uint32_t remote_mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(
                   remote_saddr),
               "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(remote_mbar)
               : "memory");
}

__device__ __forceinline__ void st_async_f32(uint32_t remote_saddr, float v, uint32_t remote_mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.f32 [%0], %1, [%2];" ::"r"(remote_saddr),
               "f"(v), "r"(remote_mbar)
               : "memory");
}

// tanh with ~1e-7 absolute error in a dozen instructions (tanhf's accurate path costs ~5x more and sits on
// the critical path of every layer of the latency-bound PPO step): odd polynomial below 0.1, else
// 1 - 2 / (exp(2x) + 1) with the hardware exponential; saturates correctly for large |x|.
__device__ __forceinline__ float tanh_fast(float x) {
  const float x2 = x * x;
  const float poly = x * fmaf(x2, fmaf(x2, 0.13333333f, -0.33333334f), 1.0f);
  const float t = __expf(2.0f * x);
  const float big = 1.0f - __fdividef(2.0f, t + 1.0f);
  return fabsf(x) < 0.1f ? poly : big;
}

// Feistel permutation of [0,n) with cycle walking (twin of philox.feistel_perm()).
struct FeistelKey {
  uint32_t k[4];
  int hb;
  uint32_t mask;
};
__host__ __device__ __forceinline__ FeistelKey feistel_key(uint64_t seed, uint32_t stream, uint64_t draw, uint64_t n) {
  uint32_t k0, k1;
  philox_key(seed, stream, k0, k1);
  Philox4 r = philox4x32((uint32_t)draw, (uint32_t)(draw >> 32), 0u, 0u, k0, k1);
  FeistelKey f;
  f.k[0] = r.x;
  f.k[1] = r.y;
  f.k[2] = r.z;
  f.k[3] = r.w;
  int bits = 2;
  if (n > 1) {
    bits = 0;
    uint64_t m = n - 1;
    while (m) {
      ++bits;
      m >>= 1;
    }
    if (bits < 2) bits = 2;
  }
  f.hb = (bits + 1) / 2;
  f.mask = (1u << f.hb) - 1u;
  return f;
}
__host__ __device__ __forceinline__ uint64_t feistel_perm(const FeistelKey& f, uint64_t i, uint64_t n) {
  uint64_t cur = i;
  do {
    uint32_t l = (uint32_t)(cur >> f.hb), r = (uint32_t)cur & f.mask;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint32_t fn = mix32(r ^ f.k[q]) & f.mask;
      uint32_t nl = r;
      r = (l ^ fn) & f.mask;
      l = nl;
    }
    cur = ((uint64_t)l << f.hb) | r;
  } while (cur >= n);
  return cur;
}

// ---- numerics shared by several kernels -------------------------------------------------------
__device__ __forceinline__ float softplus_f(float x) {  // -logsigmoid(-x), stable
  return fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x)));
}
__device__ __forceinline__ float sigmoid_f(float x) {
  if (x >= 0.0f) {
    float e = expf(-x);
    return 1.0f / (1.0f + e);
  }
  float e = expf(x);
  return e / (1.0f + e);
}

// RunningNorm.update_stats (util/networks.py:121-134): fold the moments of a batch of b_n rows (mean, biased variance)
// into the running (mean, var) of `cnt` rows
__device__ __forceinline__ void norm_fold(float& mean, float& var, float cnt, float b_mean, float b_var, float b_n) {
  const float tot = cnt + b_n;
  const float delta = b_mean - mean;
  mean += delta * b_n / tot;
  var *= cnt;
  var += b_var * b_n;
  var += delta * delta * cnt * b_n / tot;
  var /= tot;
}

// EMANorm.update_stats (util/networks.py:175-201): fold the moments of one batch (mean, biased variance) into the
// running (mean, var) with the learning rate 1 / inv_lr after inv_lr += decay^nb; nb counts the batches folded so
// far.  Every operation is rounded on its own, as the reference's separate float32 torch ops are: no contraction into
// fused multiply-adds.  powf is CUDA's, so decay^nb may differ from the host's in the last bit.
__device__ __forceinline__ void ema_fold(float& mean, float& var, float& inv_lr, int32_t nb, float decay, float b_mean,
                                         float b_var) {
  inv_lr = __fadd_rn(inv_lr, powf(decay, (float)nb));
  const float lr = __fdiv_rn(1.0f, inv_lr);
  const float dm = __fsub_rn(b_mean, mean);
  mean = __fadd_rn(mean, __fmul_rn(lr, dm));
  const float dv = __fsub_rn(__fadd_rn(b_var, __fmul_rn(__fsub_rn(1.0f, lr), __fmul_rn(dm, dm))), var);
  var = __fadd_rn(var, __fmul_rn(lr, dv));
}

// exact two-pass (mean, M2) of x[0, n), n >= 1, by one warp; every lane receives the result
__device__ __forceinline__ void warp_moments(const float* x, int n, int lane, float& mean, float& m2) {
  float s = 0.f;
  for (int i = lane; i < n; i += 32) s += x[i];
  mean = warp_sum(s) / (float)n;
  m2 = 0.f;
  for (int i = lane; i < n; i += 32) {
    const float dlt = x[i] - mean;
    m2 = fmaf(dlt, dlt, m2);
  }
  m2 = warp_sum(m2);
}

// Chan et al. merge of the moments (count, mean, M2) of `nchunks` chunks, chunk c's at cnt[c * stride],
// mean[c * stride] and m2[c * stride], by one warp: every lane merges its chunks (lane, lane + 32, ...) in index
// order, then the 32 lane results are merged by a fixed butterfly, so the result is deterministic and every lane
// receives it (a single thread walking all chunks cost more than the statistics themselves once the chunks became
// small enough to fill the GPU).  The chunk moments were written by other blocks of the same launch: read past L1.
__device__ __forceinline__ void warp_chan_merge(const float* cnt, const float* mean, const float* m2, int64_t stride,
                                                int nchunks, int lane, float& n_out, float& mean_out, float& m2_out) {
  float na = 0.f, ma = 0.f, m2a = 0.f;
  for (int c = lane; c < nchunks; c += 32) {
    const int64_t o = (int64_t)c * stride;
    const float nb = __ldcg(cnt + o), mb = __ldcg(mean + o), m2b = __ldcg(m2 + o);
    const float nt = na + nb;
    const float dlt = mb - ma;
    ma = ma + dlt * (nb / nt);
    m2a = m2a + m2b + dlt * dlt * (na * nb / nt);
    na = nt;
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float nb = __shfl_xor_sync(0xffffffffu, na, o), mb = __shfl_xor_sync(0xffffffffu, ma, o),
                m2b = __shfl_xor_sync(0xffffffffu, m2a, o);
    // merge (lower lane, higher lane) in that order on both sides so the pair agrees bit for bit
    const bool lowme = (lane & o) == 0;
    const float n1 = lowme ? na : nb, m1 = lowme ? ma : mb, q1 = lowme ? m2a : m2b;
    const float n2 = lowme ? nb : na, m2v = lowme ? mb : ma, q2 = lowme ? m2b : m2a;
    const float nt = n1 + n2;
    if (nt > 0.f) {
      const float dlt = m2v - m1;
      ma = m1 + dlt * (n2 / nt);
      m2a = q1 + q2 + dlt * dlt * (n1 * n2 / nt);
    }
    na = nt;
  }
  n_out = na;
  mean_out = ma;
  m2_out = m2a;
}
