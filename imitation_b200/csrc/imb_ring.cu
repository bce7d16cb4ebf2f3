// imb_ring.cu -- stage 2 of the GAIL/AIRL round: transition tables, the generator ring buffer,
// index sampling and the gather that assembles discriminator batches.
//
// Replaces (reference, /root/reference/src/imitation): data/buffer.py:147-232 (Buffer.store with
// wrap-around + truncation, Buffer.sample = np.random.randint + fancy-index gather),
// data/buffer.py:385-412 (ReplayBuffer facade), algorithms/base.py:272-282 + util/util.py:215-241
// (expert DataLoader(shuffle, drop_last) re-iterated forever) and the np.concatenate of
// algorithms/adversarial/common.py:592-595.
//
// All of these are HBM-bound byte movers: tables are AoS rows so a random gather reads whole
// contiguous rows; batches are feature-major so the consumer streams them.
#include "imb_common.cuh"

namespace {

// ---- table rows from separate row-major arrays --------------------------------------------------
// one warp per transition; lanes walk the row.  Ring placement follows Buffer.store: only the last
// min(n, capacity) rows are kept and written at (idx0 + i) mod capacity.
__global__ void __launch_bounds__(256) k_table_store(float* __restrict__ table, int64_t capacity, int d_obs,
                                                    int d_act, const float* __restrict__ obs,
                                                    const float* __restrict__ acts_f,
                                                    const int64_t* __restrict__ acts_i,
                                                    const float* __restrict__ next_obs,
                                                    const uint8_t* __restrict__ dones, int64_t n, int use_ring,
                                                    const int64_t* __restrict__ state) {
  const int tw = 2 * d_obs + d_act + 1;
  const int lane = threadIdx.x & 31;
  const int64_t gw = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t skip = (use_ring && n > capacity) ? n - capacity : 0;
  const int64_t idx0 = use_ring ? state[IMB_ST_RING_IDX] : 0;
  for (int64_t i = gw + skip; i < n; i += nwarps) {
    int64_t pos = i - skip;
    if (use_ring) pos = (idx0 + pos) % capacity;
    float* row = table + pos * tw;
    const int64_t a_idx = acts_i ? acts_i[i] : 0;
    for (int c = lane; c < tw; c += 32) {
      float v;
      if (c < d_obs)
        v = obs[i * d_obs + c];
      else if (c < d_obs + d_act)
        v = acts_f ? acts_f[i * d_act + (c - d_obs)] : ((c - d_obs) == a_idx ? 1.f : 0.f);
      else if (c < 2 * d_obs + d_act)
        v = next_obs[i * d_obs + (c - d_obs - d_act)];
      else
        v = dones[i] ? 1.f : 0.f;
      row[c] = v;
    }
  }
}

__global__ void k_ring_advance(int64_t* state, int64_t capacity, int64_t n_stored) {
  const int64_t kept = n_stored < capacity ? n_stored : capacity;
  state[IMB_ST_RING_IDX] = (state[IMB_ST_RING_IDX] + kept) % capacity;
  int64_t nd = state[IMB_ST_RING_N] + kept;
  state[IMB_ST_RING_N] = nd < capacity ? nd : capacity;
}

// ---- index generation (perf mode) -----------------------------------------------------------------
// replay draw i: Philox randint with replacement in [0, ring size)   (twin: oracle/philox.randint)
__device__ __forceinline__ int64_t replay_row(uint64_t seed, const int64_t* state, int64_t i) {
  const int64_t size = state[IMB_ST_RING_N];
  const uint64_t draw = (uint64_t)state[IMB_ST_REPLAY_DRAW];
  uint32_t k0, k1;
  philox_key(seed, IMB_STREAM_REPLAY, k0, k1);
  const Philox4 r = philox4x32((uint32_t)(i >> 2), (uint32_t)draw, (uint32_t)(draw >> 32), 0u, k0, k1);
  const uint32_t w = ((i & 3) == 0) ? r.x : ((i & 3) == 1) ? r.y : ((i & 3) == 2) ? r.z : r.w;
  return (int64_t)(((uint64_t)w * (uint64_t)size) >> 32);
}
// expert draw i of n_expert rows: endless Feistel permutations with drop_last   (twin: ExpertStreamPort in tests).
// Position `pos` inside epoch `ep`; a batch never straddles an epoch: expert_advance guarantees
// pos + batch <= n_expert - (n_expert % batch).
__device__ __forceinline__ int64_t expert_row(uint64_t seed, const int64_t* state, int64_t n_expert, int64_t i) {
  const int64_t pos = state[IMB_ST_EXPERT_POS];
  const uint64_t ep = (uint64_t)state[IMB_ST_EXPERT_EPOCH];
  const FeistelKey f = feistel_key(seed, IMB_STREAM_EXPERT, ep, (uint64_t)n_expert);
  return (int64_t)feistel_perm(f, (uint64_t)(pos + i), (uint64_t)n_expert);
}
// the expert stream after a batch of n draws
__device__ __forceinline__ void expert_advance(int64_t* state, int64_t n, int64_t n_expert) {
  int64_t pos = state[IMB_ST_EXPERT_POS] + n;
  if (pos + n > n_expert) {  // the next batch would not fit: drop the tail, start a new permutation
    pos = 0;
    state[IMB_ST_EXPERT_EPOCH] += 1;
  }
  state[IMB_ST_EXPERT_POS] = pos;
}

// kind 0: replay draws over the ring, kind 1: expert draws over size_arg rows
__global__ void __launch_bounds__(256) k_sample_indices(int kind, int64_t* __restrict__ out, int64_t n,
                                                       int64_t size_arg, uint64_t seed,
                                                       const int64_t* __restrict__ state) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (kind == 0)
    out[i] = replay_row(seed, state, i);
  else
    out[i] = expert_row(seed, state, size_arg, i);
}
__global__ void k_sample_advance(int kind, int64_t n, int64_t size, int64_t* state) {
  if (kind == 0)
    state[IMB_ST_REPLAY_DRAW] += 1;
  else
    expert_advance(state, n, size);
}

// ---- gather table rows into the feature-major batch --------------------------------------------------
// One lane per gathered row: a warp reads its 32 indices with one coalesced load, then walks the
// tw columns; in each step the 32 lanes read the same column of 32 different table rows (each
// row's 4*tw bytes are 5-6 sectors that stay in L1 across the column walk, so DRAM/L2 traffic is
// the rows themselves) and write 32 consecutive batch columns = one coalesced 128-byte store per
// feature row.  All tw loads of a lane are independent, so the whole tile costs ~one memory latency
// (the former shuffle-and-transpose form serialised 32 dependent row reads per warp).
constexpr int G_WARPS = 4;
// table row src[0, tw) -> batch column dst (feature stride ld), 8 independent loads in flight per step
__device__ __forceinline__ void row_to_column(const float* src, int tw, float* dst, int64_t ld) {
  int c = 0;
  for (; c + 8 <= tw; c += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = src[c + u];
#pragma unroll
    for (int u = 0; u < 8; ++u) dst[(int64_t)(c + u) * ld] = v[u];
  }
  for (; c < tw; ++c) dst[(int64_t)c * ld] = src[c];
}
__global__ void __launch_bounds__(G_WARPS * 32) k_gather_rows(const float* __restrict__ table, int64_t capacity,
                                                              int tw, const int64_t* __restrict__ idx, int64_t n,
                                                              float* __restrict__ batch, int64_t ld,
                                                              int64_t col0) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ngroups = (n + 31) / 32;
  for (int64_t grp = (int64_t)blockIdx.x * G_WARPS + warp; grp < ngroups; grp += (int64_t)gridDim.x * G_WARPS) {
    const int64_t mine = grp * 32 + lane;
    if (mine >= n) continue;
    int64_t r = idx ? idx[mine] : mine;
    r = r < 0 ? 0 : (r >= capacity ? capacity - 1 : r);
    row_to_column(table + r * tw, tw, batch + col0 + mine, ld);
  }
}


// ---- fused device sampling + gather of one discriminator minibatch ---------------------------------
// Batch columns [0, mb): expert rows (endless Feistel permutations with drop_last, same stream as
// k_sample_indices kind 1); columns [mb, 2 mb): generator rows (Philox randint over the ring, kind 0).  `start` is
// the minibatch's offset inside the update's demo_batch_size draws; the draw counters advance once per update
// (imb_sample_advance2).  Replaces 2 x (k_sample_indices + k_sample_advance) + 2 x k_gather_rows.
__global__ void __launch_bounds__(G_WARPS * 32) k_sample_gather(const float* __restrict__ e_table, int64_t e_n,
                                                                const float* __restrict__ g_table, int64_t g_cap,
                                                                int tw, int64_t mb, int64_t start, uint64_t seed,
                                                                const int64_t* __restrict__ e_state,
                                                                const int64_t* __restrict__ g_state,
                                                                float* __restrict__ batch, int64_t ld) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t n = 2 * mb, ngroups = (n + 31) / 32;
  for (int64_t grp = (int64_t)blockIdx.x * G_WARPS + warp; grp < ngroups; grp += (int64_t)gridDim.x * G_WARPS) {
    const int64_t mine = grp * 32 + lane;
    if (mine >= n) continue;
    const float* src;
    if (mine < mb) {
      src = e_table + expert_row(seed, e_state, e_n, start + mine) * tw;
    } else {
      int64_t r = replay_row(seed, g_state, start + (mine - mb));
      r = r < 0 ? 0 : (r >= g_cap ? g_cap - 1 : r);
      src = g_table + r * tw;
    }
    row_to_column(src, tw, batch + mine, ld);
  }
}
__global__ void k_sample_advance2(int64_t n, int64_t e_n, int64_t* e_state, int64_t* g_state) {
  g_state[IMB_ST_REPLAY_DRAW] += 1;
  expert_advance(e_state, n, e_n);
}

// ---- DQN learner ring (imb_dqn_ring_store) ---------------------------------------------------------------------
// one block: copy the T x E flat rows of a rollout into the feature-major ring [tw][P * E] at SB3's column
// ((pos + t) mod P) * E + e, pos = ring_state[RING_IDX], then advance pos by T and RING_N (= positions filled) as
// SB3's ReplayBuffer.add does T times.  flat row of (e, t): flat_index(e, t, E, T, t0, H), t0 = env_state[EP_STEP]
// (the rollout's first episode step: the call goes before imb_rollout_advance).
__global__ void __launch_bounds__(256) k_dqn_ring_store(const float* __restrict__ flat, int tw, float* __restrict__ ring,
                                                       int64_t P, int64_t E, int64_t T, int H,
                                                       const int64_t* __restrict__ env_state,
                                                       int64_t* __restrict__ ring_state) {
  const int64_t pos = ring_state[IMB_ST_RING_IDX], t0 = env_state[IMB_ST_EP_STEP], C = P * E;
  // with T > P a later step overwrites an earlier one at its position, as SB3's sequential adds do: only the last
  // min(T, P) steps are written
  const int64_t tskip = T > P ? T - P : 0, n = (T - tskip) * E * tw;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t c = i % tw, te = i / tw, t = tskip + te / E, e = te % E;
    const int64_t f = flat_index(e, t, E, T, t0, H);
    ring[c * C + ((pos + t) % P) * E + e] = flat[f * tw + c];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ring_state[IMB_ST_RING_IDX] = (pos + T) % P;
    const int64_t filled = ring_state[IMB_ST_RING_N] + T;
    ring_state[IMB_ST_RING_N] = filled < P ? filled : P;
  }
}

}  // namespace

extern "C" int imb_dqn_ring_store(const float* flat, int32_t tw, float* ring, int64_t positions, int64_t n_envs,
                                  int64_t n_steps, int32_t horizon, const int64_t* env_state, int64_t* ring_state,
                                  void* stream) {
  IMB_REQUIRE(positions >= 1 && n_envs >= 1 && n_steps >= 1 && horizon >= 1 && tw >= 1, "bad ring store shape");
  k_dqn_ring_store<<<1, 256, 0, (cudaStream_t)stream>>>(flat, tw, ring, positions, n_envs, n_steps, horizon, env_state,
                                                        ring_state);
  IMB_CHECK_LAUNCH("k_dqn_ring_store");
  return 0;
}

extern "C" int imb_table_store(float* table, int64_t capacity, int32_t d_obs, int32_t d_act, const float* obs,
                               const float* acts_f, const int64_t* acts_i, const float* next_obs,
                               const uint8_t* dones, int64_t n, int use_ring, const int64_t* state, void* stream) {
  IMB_REQUIRE(n >= 1, "Trying to store empty data.");
  IMB_REQUIRE((acts_f != nullptr) != (acts_i != nullptr), "exactly one of acts_f / acts_i must be given");
  IMB_REQUIRE(use_ring || n <= capacity, "Not enough capacity to store data.");
  int64_t warps = n < capacity ? n : capacity;
  int64_t blocks = (warps * 32 + 255) / 256;
  const int64_t cap = (int64_t)imb_num_sms() * 8;
  if (blocks > cap) blocks = cap;
  k_table_store<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(table, capacity, d_obs, d_act, obs, acts_f, acts_i,
                                                                next_obs, dones, n, use_ring, state);
  IMB_CHECK_LAUNCH("k_table_store");
  return 0;
}

extern "C" int imb_ring_advance(int64_t* state, int64_t capacity, int64_t n_stored, void* stream) {
  k_ring_advance<<<1, 1, 0, (cudaStream_t)stream>>>(state, capacity, n_stored);
  IMB_CHECK_LAUNCH("k_ring_advance");
  return 0;
}

extern "C" int imb_sample_indices(int kind, int64_t* idx_out, int64_t n, int64_t size, uint64_t seed,
                                  int64_t* state, void* stream) {
  IMB_REQUIRE(n >= 1, "n must be positive");
  if (kind == 1) IMB_REQUIRE(size >= n, "Number of transitions in `demonstrations` %lld is smaller than batch size %lld.",
                             (long long)size, (long long)n);
  k_sample_indices<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(kind, idx_out, n, size, seed, state);
  IMB_CHECK_LAUNCH("k_sample_indices");
  k_sample_advance<<<1, 1, 0, (cudaStream_t)stream>>>(kind, n, size, state);
  IMB_CHECK_LAUNCH("k_sample_advance");
  return 0;
}

extern "C" int imb_gather_rows(const float* table, int64_t capacity, int32_t tw, const int64_t* idx, int64_t n,
                               float* batch, int64_t ld, int64_t col0, void* stream) {
  if (n <= 0) return 0;
  IMB_REQUIRE(capacity >= 1 && tw >= 1, "bad table shape");
  int64_t blocks = ((n + 31) / 32 + G_WARPS - 1) / G_WARPS;
  const int64_t cap = (int64_t)imb_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  k_gather_rows<<<(int)blocks, G_WARPS * 32, 0, (cudaStream_t)stream>>>(table, capacity, tw, idx, n, batch, ld, col0);
  IMB_CHECK_LAUNCH("k_gather_rows");
  return 0;
}

extern "C" int imb_disc_sample_gather(const float* expert_table, int64_t n_expert, const float* ring,
                                      int64_t ring_capacity, int32_t tw, int64_t mb, int64_t start, uint64_t seed,
                                      const int64_t* expert_state, const int64_t* ring_state, float* batch, int64_t ld,
                                      void* stream) {
  IMB_REQUIRE(mb >= 1 && start >= 0 && tw >= 1, "bad minibatch shape");
  IMB_REQUIRE(n_expert >= mb, "Number of transitions in `demonstrations` %lld is smaller than batch size %lld.",
              (long long)n_expert, (long long)mb);
  int64_t blocks = ((2 * mb + 31) / 32 + G_WARPS - 1) / G_WARPS;
  const int64_t cap = (int64_t)imb_num_sms() * 16;
  if (blocks > cap) blocks = cap;
  k_sample_gather<<<(int)blocks, G_WARPS * 32, 0, (cudaStream_t)stream>>>(expert_table, n_expert, ring, ring_capacity, tw, mb,
                                                                        start, seed, expert_state, ring_state, batch, ld);
  IMB_CHECK_LAUNCH("k_sample_gather");
  return 0;
}

extern "C" int imb_sample_advance2(int64_t n, int64_t n_expert, int64_t* expert_state, int64_t* ring_state,
                                   void* stream) {
  k_sample_advance2<<<1, 1, 0, (cudaStream_t)stream>>>(n, n_expert, expert_state, ring_state);
  IMB_CHECK_LAUNCH("k_sample_advance2");
  return 0;
}
