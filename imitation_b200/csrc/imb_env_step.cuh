// imb_env_step.cuh -- the device envs' step and reset functions, thread per env, shared by the rollout kernel
// (imb_rollout_impl.cuh) and the SAC collection kernel (imb_sac.cu).
#pragma once
#include "imb_common.cuh"

namespace {

// ---- classic-control envs (imb_env_desc.kind; DESIGN.md section 7e) ---------------------------------------------------
// The observation is the env's whole state, so the SoA [d_obs][E] obs buffer is the only state array.  One thread steps
// one env: it reads the float32 observation obs[k * stride], computes in float64 as gymnasium does and writes the next
// observation nobs[k * stride] in float32; returns the env reward.

// the Box bound of the env's actions: Pendulum-v1's torque is in [-2, 2], the synthetic env's Box is [-1, 1] (and the
// Discrete envs have no Box)
__device__ __forceinline__ float env_act_bound(int kind) { return kind == IMB_ENV_PENDULUM ? 2.0f : 1.0f; }

// seals/CartPole-v0 (gymnasium CartPole, Euler integrator; seals' FixedHorizonCartPole reward, never terminates).
// ctl: the one-hot control, action 1 pushes the cart in +x.
__device__ __forceinline__ float cartpole_step(const float* __restrict__ obs, const float* __restrict__ ctl,
                                               float* __restrict__ nobs, int stride) {
  constexpr double g = 9.8, masspole = 0.1, total_mass = 1.0 + 0.1, length = 0.5, polemass_length = 0.1 * 0.5;
  constexpr double force_mag = 10.0, tau = 0.02, x_threshold = 2.4, theta_threshold = 12.0 * 2.0 * M_PI / 360.0;
  const double x = obs[0], x_dot = obs[stride], theta = obs[2 * stride], theta_dot = obs[3 * stride];
  const double force = ctl[stride] > 0.5f ? force_mag : -force_mag;
  double sintheta, costheta;
  sincos(theta, &sintheta, &costheta);
  const double temp = (force + polemass_length * (theta_dot * theta_dot) * sintheta) / total_mass;
  const double thetaacc =
      (g * sintheta - costheta * temp) / (length * (4.0 / 3.0 - masspole * (costheta * costheta) / total_mass));
  const double xacc = temp - polemass_length * thetaacc * costheta / total_mass;
  const double nx = x + tau * x_dot, nx_dot = x_dot + tau * xacc;
  const double ntheta = theta + tau * theta_dot, ntheta_dot = theta_dot + tau * thetaacc;
  nobs[0] = (float)nx;
  nobs[stride] = (float)nx_dot;
  nobs[2 * stride] = (float)ntheta;
  nobs[3 * stride] = (float)ntheta_dot;
  const bool inside = fabs(nx) <= x_threshold && fabs(ntheta) <= theta_threshold;
  return inside ? 1.0f : 0.0f;
}

// Pendulum-v1 (g = 10, m = l = 1, dt = 0.05, |thdot| <= 8, |u| <= 2; reward on the pre-step state).  The angle comes
// back as atan2(sin, cos) in [-pi, pi]: the dynamics see only sin(theta) and theta mod 2 pi, and angle_normalize of an
// angle in [-pi, pi] squares to its own square.  ctl: the control, already clipped to [-2, 2].
__device__ __forceinline__ float pendulum_step(const float* __restrict__ obs, const float* __restrict__ ctl,
                                               float* __restrict__ nobs, int stride) {
  constexpr double g = 10.0, dt = 0.05, max_speed = 8.0, max_torque = 2.0;
  const double th = atan2((double)obs[stride], (double)obs[0]), thdot = obs[2 * stride];
  const double u = fmin(fmax((double)ctl[0], -max_torque), max_torque);
  const double costs = th * th + 0.1 * (thdot * thdot) + 0.001 * (u * u);
  const double newthdot = fmin(fmax(thdot + (3.0 * g / 2.0 * sin(th) + 3.0 * u) * dt, -max_speed), max_speed);
  const double newth = th + newthdot * dt;
  double s, c;
  sincos(newth, &s, &c);
  nobs[0] = (float)c;
  nobs[stride] = (float)s;
  nobs[2 * stride] = (float)newthdot;
  return (float)(-costs);
}

// The reset observation of a classic env from the four uniforms of Philox stream IMB_STREAM_ENV_RESET keyed by `seed`
// at counter (env id, episode): CartPole x, x_dot, theta, theta_dot ~ U(-0.05, 0.05); Pendulum theta ~ U(-pi, pi),
// theta_dot ~ U(-1, 1), observed as (cos theta, sin theta, theta_dot).  (The same distributions as gymnasium's resets,
// not its PCG64 bits.)
__device__ __forceinline__ void classic_reset(int kind, uint64_t seed, uint32_t egid, uint32_t episode,
                                              float* __restrict__ obs, int64_t stride) {
  uint32_t k0, k1;
  philox_key(seed, IMB_STREAM_ENV_RESET, k0, k1);
  const Philox4 r = philox4x32(egid, episode, 0u, 0u, k0, k1);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  if (kind == IMB_ENV_CARTPOLE) {
    for (int k = 0; k < 4; ++k) obs[k * stride] = (float)(-0.05 + 0.1 * (double)u01(w[k]));
  } else {
    const double th = -M_PI + 2.0 * M_PI * (double)u01(w[0]), thdot = -1.0 + 2.0 * (double)u01(w[1]);
    double s, c;
    sincos(th, &s, &c);
    obs[0] = (float)c;
    obs[stride] = (float)s;
    obs[2 * stride] = (float)thdot;
  }
}

// The synthetic env (SURVEY.md section 8d) stepped by one thread: nobs[i * stride] = tanh(c_i + sum_k A[i][k] obs_k +
// sum_a Bm[i][a] ctl_a) and reward w . nobs - 0.1 |ctl|^2, with `p` the env's flat [A | Bm | c | w] and ctl already in
// the Box.  (The rollout kernel steps the same env as one tiled layer over the CTA's envs; this form sums in another
// order, so the two agree to float32 rounding, not bit for bit.)
__device__ __forceinline__ float synth_step(const float* __restrict__ p, int Do, int Da, const float* __restrict__ obs,
                                            const float* __restrict__ ctl, float* __restrict__ nobs, int stride) {
  const float* eA = p;
  const float* eB = eA + Do * Do;
  const float* eC = eB + Do * Da;
  const float* eW = eC + Do;
  float rew = 0.f;
  for (int i = 0; i < Do; ++i) {
    float z = eC[i];
    for (int k = 0; k < Do; ++k) z = fmaf(eA[i * Do + k], obs[k * stride], z);
    for (int a = 0; a < Da; ++a) z = fmaf(eB[i * Da + a], ctl[a * stride], z);
    const float n = tanhf(z);
    nobs[i * stride] = n;
    rew = fmaf(eW[i], n, rew);
  }
  float pen = 0.f;
  for (int a = 0; a < Da; ++a) pen = fmaf(ctl[a * stride], ctl[a * stride], pen);
  return rew - 0.1f * pen;
}

}  // namespace
