// imb_mlp.cuh -- the reward net's launch descriptor (which batch rows each pass reads, and its network widths) used
// by the discriminator kernels (imb_disc.cu) and by the reward relabel inside the rollout kernel (imb_rollout.cu).
#pragma once
#include "imb_common.cuh"

namespace {

constexpr int NT = 128;               // threads per CTA in the disc fwd/bwd kernel
constexpr int XS_LD = IMB_TILE_ROWS;  // staged tile: [slot][128 rows]
constexpr int MAX_STAGE_ROWS = 200;   // 2*64 + 64 + 2 = 194
constexpr int MAX_PASS = 3;

// ---- launch descriptor passed by value to the kernels --------------------------------------------
struct PassDesc {
  int din, n_hidden, h1, h2;
  int has_norm;
  float eps;
  int param_off;     // into flat params / accumulators
  int coef_kind;     // 0: +1, 1: +gamma*(1-done), 2: -1
  const float* norm; // [mean(din) | var(din)] to use for this pass (nullptr if none)
  unsigned char in_slot[IMB_MAX_DIN];  // staged slot of MLP input k
};
struct DiscLaunch {
  int npass;
  int nstage;        // staged feature rows
  int done_slot;     // staged slot of the done row (-1 if unused)
  int logp_slot;     // staged slot of the log pi row (-1 if unused)
  int P;             // total params
  float gamma;
  short stage_row[MAX_STAGE_ROWS];  // batch feature row of each staged slot
  PassDesc pass[MAX_PASS];
};

// The widths every kernel sizes its network images by: JP, the hidden width padded to 32 or 64 columns (the widest
// hidden layer over the launch's passes), and dmax, the widest pass input.
struct LaunchWidths {
  int JP, dmax;
};
inline LaunchWidths launch_widths(const DiscLaunch& L) {
  int h = 0, dmax = 1;
  for (int p = 0; p < L.npass; ++p) {
    const PassDesc& q = L.pass[p];
    if (q.n_hidden >= 1 && q.h1 > h) h = q.h1;
    if (q.n_hidden >= 2 && q.h2 > h) h = q.h2;
    if (q.din > dmax) dmax = q.din;
  }
  return {h <= 32 ? 32 : 64, dmax};
}

// Build the launch descriptor: which batch feature rows are staged and how each pass maps its
// MLP inputs onto them.  Batch feature rows: obs [0,Do), act [Do,Do+Da), next_obs [Do+Da,2Do+Da),
// done 2Do+Da, logp 2Do+Da+1.
__host__ int build_launch(const imb_disc_desc* d, const float* norm_state, const float* snapA, DiscLaunch& L) {
  memset(&L, 0, sizeof(L));
  const int Do = d->d_obs, Da = d->d_act;
  const int row_obs = 0, row_act = Do, row_nobs = Do + Da, row_done = 2 * Do + Da, row_logp = row_done + 1;
  short slot_of[2 * IMB_MAX_DIN + IMB_MAX_DIN + 2 + 64];
  const int nrows = row_logp + 1;
  IMB_REQUIRE(nrows <= (int)(sizeof(slot_of) / sizeof(short)), "d_obs/d_act too large");
  for (int i = 0; i < nrows; ++i) slot_of[i] = -1;
  int ns = 0;
  auto need = [&](int row) {
    if (slot_of[row] < 0) {
      slot_of[row] = (short)ns;
      L.stage_row[ns++] = (short)row;
    }
    return (int)slot_of[row];
  };
  // pass 0: base net on the selected concat
  PassDesc& b = L.pass[0];
  int k = 0;
  auto push = [&](PassDesc& p, int row) -> int {
    if (k >= IMB_MAX_DIN) return -1;
    p.in_slot[k++] = (unsigned char)need(row);
    return 0;
  };
  if (d->use_state)
    for (int i = 0; i < Do; ++i)
      if (push(b, row_obs + i)) IMB_FAIL(-1, "base MLP input wider than %d", IMB_MAX_DIN);
  if (d->use_action)
    for (int i = 0; i < Da; ++i)
      if (push(b, row_act + i)) IMB_FAIL(-1, "base MLP input wider than %d", IMB_MAX_DIN);
  if (d->use_next_state)
    for (int i = 0; i < Do; ++i)
      if (push(b, row_nobs + i)) IMB_FAIL(-1, "base MLP input wider than %d", IMB_MAX_DIN);
  if (d->use_done)
    if (push(b, row_done)) IMB_FAIL(-1, "base MLP input wider than %d", IMB_MAX_DIN);
  IMB_REQUIRE(k == d->base.din, "base.din=%d does not match the selected inputs (%d)", d->base.din, k);
  auto fill = [&](PassDesc& p, const imb_mlp& m, int coef, const float* norm) {
    p.din = m.din;
    p.n_hidden = m.n_hidden;
    p.h1 = m.h1;
    p.h2 = m.h2;
    p.has_norm = m.has_norm;
    p.eps = m.norm_eps;
    p.param_off = m.param_off;
    p.coef_kind = coef;
    p.norm = m.has_norm ? norm : nullptr;
  };
  fill(b, d->base, 0, norm_state + d->base.norm_off);
  L.npass = 1;
  L.done_slot = -1;
  L.logp_slot = -1;
  if (d->shaped) {
    IMB_REQUIRE(d->potential.din == Do, "potential.din must equal d_obs");
    PassDesc& p1 = L.pass[1];  // Phi(s')   (evaluated first by the reference)
    k = 0;
    for (int i = 0; i < Do; ++i) push(p1, row_nobs + i);
    fill(p1, d->potential, 1, snapA ? snapA : norm_state + d->potential.norm_off);
    PassDesc& p2 = L.pass[2];  // Phi(s)
    k = 0;
    for (int i = 0; i < Do; ++i) push(p2, row_obs + i);
    fill(p2, d->potential, 2, norm_state + d->potential.norm_off);
    L.npass = 3;
    L.done_slot = need(row_done);
  }
  if (d->subtract_logp) L.logp_slot = need(row_logp);
  L.nstage = ns;
  L.P = d->n_params;
  L.gamma = d->gamma;
  IMB_REQUIRE(ns <= MAX_STAGE_ROWS, "too many staged rows");
  for (int p = 0; p < L.npass; ++p) {
    const PassDesc& q = L.pass[p];
    IMB_REQUIRE(q.n_hidden >= 0 && q.n_hidden <= 2, "n_hidden must be 0..2");
    IMB_REQUIRE(q.din >= 1 && q.din <= IMB_MAX_DIN, "din out of range");
    if (q.n_hidden >= 1) IMB_REQUIRE(q.h1 >= 1 && q.h1 <= IMB_MAX_HIDDEN, "h1 out of range");
    if (q.n_hidden >= 2) IMB_REQUIRE(q.h2 >= 1 && q.h2 <= IMB_MAX_HIDDEN, "h2 out of range");
  }
  return 0;
}

// coefficient of a pass's output in the logit: r + gamma*(1-done)*Phi(s') - Phi(s)
__device__ __forceinline__ float pass_coef(int kind, float gamma, float done) {
  return kind == 0 ? 1.0f : (kind == 1 ? gamma * (1.0f - done) : -1.0f);
}

}  // namespace
