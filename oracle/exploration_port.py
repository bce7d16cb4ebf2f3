"""CPU twin of the exploration rollout (csrc/imb_rollout_impl.cuh, k_rollout with EXP; imb_rollout_explore).

TEST INFRASTRUCTURE.  The reference's `ExplorationWrapper` (policies/exploration_wrapper.py:23-95) acts with the
wrapped policy or with `action_space.sample()` for the whole VecEnv at each step.  `ExplorationPolicyPort` is an
`ActorCriticPort` behind that switch, as `PPOPort.collect_rollouts` calls it once per step with the step's pinned
noise: on a random step the action is low + u (high - low) on the synthetic env's Box [-1, 1], or min(floor(u n), n - 1)
for Discrete(n), with u the step's noise (uniforms in the slots the policy step would read), and logp = value = 0
(the kernel skips the towers); other steps are the wrapped policy's, sampled or (deterministic) its mode.
"""
import numpy as np
import torch as th
from torch import nn

from . import philox

STREAM_EXPLORE = 0x7007  # csrc/imb_common.cuh IMB_STREAM_EXPLORE


class ExplorationPolicyPort(nn.Module):
    def __init__(self, policy: nn.Module, policy_steps, deterministic: bool = False):
        super().__init__()
        self.policy = policy
        self.policy_steps = np.asarray(policy_steps, np.uint8)
        self.deterministic = deterministic
        self.discrete, self.d_obs, self.d_act = policy.discrete, policy.d_obs, policy.d_act
        self.t = 0  # step of the next forward call

    def forward(self, obs, noise=None, deterministic=False):
        t = self.t
        self.t += 1
        if not self.policy_steps[t]:
            return self.policy(obs, None if self.deterministic else noise, deterministic=self.deterministic)
        u = th.as_tensor(noise, dtype=th.float32)
        n = obs.shape[0]
        if self.discrete:
            acts = th.clamp(th.floor(u * np.float32(self.d_act)).long(), max=self.d_act - 1)
        else:
            lo, hi = np.float32(-1.0), np.float32(1.0)
            acts = lo + u * (hi - lo)
        return acts, th.zeros(n, 1), th.zeros(n)

    def predict_values(self, obs):
        return self.policy.predict_values(obs)


def random_uniforms(seed: int, env_ids, step0: int, n_steps: int, d_act: int, discrete: bool) -> np.ndarray:
    """The uniforms the kernel's random steps draw without pinned noise: Philox stream STREAM_EXPLORE keyed by `seed`,
    counter (env id, step0 + t, a // 4, 0), word a % 4 (Discrete: word 0 of chunk 0) -> [T][E][d_act] or [T][E]."""
    k0, k1 = philox.key_for(seed, STREAM_EXPLORE)
    env_ids = np.asarray(env_ids, np.uint32)
    n_chunks = 1 if discrete else (d_act + 3) // 4
    out = np.empty((n_steps, len(env_ids), 4 * n_chunks), np.float32)
    for t in range(n_steps):
        for c in range(n_chunks):
            words = philox.philox4x32(env_ids, np.uint32(step0 + t), np.uint32(c), np.uint32(0), k0, k1)
            for j in range(4):
                out[t, :, 4 * c + j] = philox.u01(words[j])
    return out[:, :, 0] if discrete else out[:, :, :d_act]
