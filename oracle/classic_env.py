"""seals/CartPole-v0 and Pendulum-v1 as batched NumPy envs (twin of the classic-control kinds of csrc/imb_rollout_impl.cuh).

TEST INFRASTRUCTURE.  The same interface as oracle/synth_env (`ClassicEnvSpec` for `SynthEnvSpec`, `ClassicVecEnv`
for `SynthVecEnv`): a fixed horizon, then auto-reset with SB3's VecEnv contract (the returned obs is the reset obs,
infos[i]["terminal_observation"] the true last obs, infos[i]["TimeLimit.truncated"] True).

Each step starts from the float32 observation, computes in float64 with gymnasium's formulas and rounds the next
observation to float32.  The observation is the whole state: Pendulum's angle is atan2(sin, cos).  gymnasium keeps a
float64 state between steps, so a step from a recorded float32 observation lands within about one float32 ulp of the
recorded next observation (tests/test_classic_env.py holds this against the reference's expert rollouts).

Reset observations come from the uniforms of Philox stream STREAM_ENV_RESET keyed by the env seed at counter
(env id, episode): CartPole's four state variables ~ U(-0.05, 0.05); Pendulum theta ~ U(-pi, pi), theta_dot ~ U(-1, 1).
"""
import dataclasses

import numpy as np

from . import philox, synth_env

CARTPOLE, PENDULUM = "seals/CartPole-v0", "Pendulum-v1"


def uniforms(seed, stream, a, b, n):
    """`n` float32 uniforms in (0, 1) per (a, b) pair: counter = (a, b, chunk, 0), word j % 4 of chunk j // 4 (the
    device's u01 of that word).  a, b: uint32 arrays of identical shape S.  Returns float32 array S + (n,)."""
    k0, k1 = philox.key_for(seed, stream)
    a = np.asarray(a, np.uint32)
    b = np.broadcast_to(np.asarray(b, np.uint32), a.shape)
    nchunk = (n + 3) // 4
    out = np.empty(a.shape + (nchunk * 4,), np.float32)
    for j in range(nchunk):
        words = philox.philox4x32(a, b, np.uint32(j), np.uint32(0), k0, k1)
        for w in range(4):
            out[..., 4 * j + w] = philox.u01(words[w])
    return out[..., :n]


def cartpole_step(obs, acts):
    """gymnasium CartPole's Euler step and seals' FixedHorizonCartPole reward (1 inside the thresholds after the step,
    else 0; never done).  obs float32 [N, 4], acts int [N] (1 pushes +x) -> (next obs float32, reward float32)."""
    gravity, masspole, total_mass, length, force_mag, tau = 9.8, 0.1, 1.0 + 0.1, 0.5, 10.0, 0.02
    polemass_length = masspole * length
    x, x_dot, theta, theta_dot = np.asarray(obs, np.float32).astype(np.float64).T
    force = np.where(np.asarray(acts).reshape(-1) == 1, force_mag, -force_mag)
    costheta, sintheta = np.cos(theta), np.sin(theta)
    temp = (force + polemass_length * np.square(theta_dot) * sintheta) / total_mass
    thetaacc = (gravity * sintheta - costheta * temp) / (length * (4.0 / 3.0 - masspole * np.square(costheta) / total_mass))
    xacc = temp - polemass_length * thetaacc * costheta / total_mass
    x, x_dot = x + tau * x_dot, x_dot + tau * xacc
    theta, theta_dot = theta + tau * theta_dot, theta_dot + tau * thetaacc
    inside = (np.abs(x) <= 2.4) & (np.abs(theta) <= 12 * 2 * np.pi / 360)
    return np.stack([x, x_dot, theta, theta_dot], 1).astype(np.float32), inside.astype(np.float32)


def pendulum_step(obs, acts):
    """gymnasium Pendulum-v1's step (g = 10, reward on the pre-step state, never done).  obs float32 [N, 3] =
    (cos, sin, theta_dot), acts float32 [N, 1] (clipped to [-2, 2] here) -> (next obs float32, reward float32)."""
    g, m, l, dt, max_speed, max_torque = 10.0, 1.0, 1.0, 0.05, 8.0, 2.0
    obs = np.asarray(obs, np.float32).astype(np.float64)
    th, thdot = np.arctan2(obs[:, 1], obs[:, 0]), obs[:, 2]
    u = np.clip(np.asarray(acts, np.float32).reshape(-1), -max_torque, max_torque).astype(np.float64)
    costs = (((th + np.pi) % (2 * np.pi)) - np.pi) ** 2 + 0.1 * thdot ** 2 + 0.001 * u ** 2
    newthdot = np.clip(thdot + (3 * g / (2 * l) * np.sin(th) + 3.0 / (m * l ** 2) * u) * dt, -max_speed, max_speed)
    newth = th + newthdot * dt
    return np.stack([np.cos(newth), np.sin(newth), newthdot], 1).astype(np.float32), (-costs).astype(np.float32)


@dataclasses.dataclass
class ClassicEnvSpec:
    """oracle/synth_env.SynthEnvSpec's interface for one classic-control env."""
    name: str
    horizon: int = 0  # 0: the env's own (500 / 200)
    seed: int = 0

    def __post_init__(self):
        if self.name not in (CARTPOLE, PENDULUM):
            raise ValueError(f"unknown classic env {self.name!r}")
        self.discrete = self.name == CARTPOLE
        self.d_obs, self.d_act = (4, 2) if self.discrete else (3, 1)
        self.act_bound = 1.0 if self.discrete else 2.0
        if not self.horizon:
            self.horizon = 500 if self.discrete else 200

    def reset_obs(self, env_ids, episodes):
        u = uniforms(self.seed, philox.STREAM_ENV_RESET, np.asarray(env_ids, np.uint32),
                     np.asarray(episodes, np.uint32), 4).astype(np.float64)
        if self.discrete:
            return (-0.05 + 0.1 * u).astype(np.float32)
        th, thdot = -np.pi + 2.0 * np.pi * u[..., 0], -1.0 + 2.0 * u[..., 1]
        return np.stack([np.cos(th), np.sin(th), thdot], -1).astype(np.float32)

    def dynamics(self, obs, acts):
        return cartpole_step(obs, acts) if self.discrete else pendulum_step(obs, acts)


class ClassicVecEnv(synth_env.SynthVecEnv):
    """DummyVecEnv-style host env over a ClassicEnvSpec, with the env's own spaces."""

    def __init__(self, spec: ClassicEnvSpec, num_envs: int, env_id_offset: int = 0):
        super().__init__(spec, num_envs, env_id_offset)
        if not spec.discrete:
            self.action_space = synth_env._Box(-spec.act_bound, spec.act_bound, (spec.d_act,))
