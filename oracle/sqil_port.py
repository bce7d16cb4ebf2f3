"""CPU restatement of SQIL's learner: SB3 2.2's DQN.learn loop with SQIL's replay buffer, and the DQN TD step in float64.

TEST INFRASTRUCTURE.  SB3 is not installed, so its semantics are restated from SB3 2.2.x (stable_baselines3/common/
off_policy_algorithm.py learn / collect_rollouts / _sample_action, dqn/dqn.py train / _on_step / predict,
common/buffers.py ReplayBuffer add / sample, common/utils.py get_linear_fn / polyak_update), written as that code runs:
one VecEnv step at a time.  Unpinned: re-verify wherever SB3 is available.

`LearnLoopPort.learn` walks the loop and records every global-NumPy draw and host-known event; the device DQN's host
pass (algorithms/dqn.py learn_schedule) is held to it.  The env and the Q-net are left out: actions and transitions are
supplied by the caller (`act_fn`, `step_fn`), so the same loop serves the schedule test and the whole-train test.
`td_step` is one DQN.train step in float64 NumPy with a hand-written backward, itself held to torch autograd.
"""
from typing import Callable, List, Optional

import numpy as np


def get_linear_fn(start: float, end: float, end_fraction: float):
    def func(progress_remaining: float) -> float:
        if (1 - progress_remaining) > end_fraction:
            return end
        return start + (1 - progress_remaining) * (end - start) / end_fraction
    return func


class ReplayBufferPort:
    """SB3's ReplayBuffer (optimize_memory_usage=False, handle_timeout_termination=False) storing what SQIL stores."""

    def __init__(self, buffer_size: int, n_envs: int, d_obs: int, reward: float):
        self.buffer_size = max(buffer_size // n_envs, 1)
        self.n_envs = n_envs
        self.observations = np.zeros((self.buffer_size, n_envs, d_obs), np.float32)
        self.next_observations = np.zeros((self.buffer_size, n_envs, d_obs), np.float32)
        self.actions = np.zeros((self.buffer_size, n_envs, 1), np.int64)
        self.dones = np.zeros((self.buffer_size, n_envs), np.float32)
        self.rewards = np.zeros((self.buffer_size, n_envs), np.float32)
        self.reward = reward
        self.pos, self.full = 0, False

    def add(self, obs, next_obs, action, done):
        self.observations[self.pos] = obs
        self.next_observations[self.pos] = next_obs
        self.actions[self.pos] = np.broadcast_to(np.asarray(action).reshape(-1, 1), (self.n_envs, 1))
        self.dones[self.pos] = done
        self.rewards[self.pos] = self.reward
        self.pos += 1
        if self.pos == self.buffer_size:
            self.full, self.pos = True, 0

    def sample(self, n: int):
        """(batch_inds, env_inds) in SB3's draw order."""
        upper = self.buffer_size if self.full else self.pos
        batch_inds = np.random.randint(0, upper, size=n)
        env_inds = np.random.randint(0, high=self.n_envs, size=(len(batch_inds),))
        return batch_inds, env_inds


class LearnLoopPort:
    """OffPolicyAlgorithm.learn + DQN for SQIL, over caller-supplied acting and env stepping."""

    def __init__(self, *, n_envs: int, d_obs: int, n_expert: int, buffer_size: int = 1_000_000,
                 learning_starts: int = 100, batch_size: int = 32, train_freq: int = 4, gradient_steps: int = 1,
                 target_update_interval: int = 10_000, exploration_fraction: float = 0.1,
                 exploration_initial_eps: float = 1.0, exploration_final_eps: float = 0.05):
        self.n_envs, self.learning_starts, self.batch_size = n_envs, learning_starts, batch_size
        self.train_freq, self.gradient_steps, self.target_update_interval = train_freq, gradient_steps, target_update_interval
        self.exploration_schedule = get_linear_fn(exploration_initial_eps, exploration_final_eps, exploration_fraction)
        self.buffer = ReplayBufferPort(buffer_size, n_envs, d_obs, 0.0)
        self.n_expert = n_expert
        self.exploration_rate = 0.0
        self._n_calls = 0
        self._n_updates = 0
        self.num_timesteps = 0
        # records
        self.random_steps: List[int] = []
        self.rates: List[float] = []
        self.target_update_calls: List[int] = []  # _n_calls at each polyak update
        self.samples: List[tuple] = []            # per TD step: (learner batch_inds, env_inds, expert inds)
        self.train_calls: List[int] = []          # gradient steps of each train() call

    def learn(self, total_timesteps: int, act_fn: Optional[Callable] = None, step_fn: Optional[Callable] = None,
              train_fn: Optional[Callable] = None, target_fn: Optional[Callable] = None):
        """act_fn(random: bool) -> actions; step_fn(actions) -> (obs, next_obs (terminal fixed), dones);
        train_fn(samples) runs one TD step; target_fn() one polyak update.  reset_num_timesteps=True."""
        self.num_timesteps = 0
        self._total_timesteps = total_timesteps
        while self.num_timesteps < total_timesteps:
            n_collected = 0
            while n_collected < self.train_freq:
                # _sample_action
                if self.num_timesteps < self.learning_starts:
                    random = True
                else:  # DQN.predict(deterministic=False)
                    random = bool(np.random.rand() < self.exploration_rate)
                self.random_steps.append(int(random))
                acts = act_fn(random) if act_fn else None
                obs, next_obs, dones = step_fn(acts) if step_fn else (0.0, 0.0, 0.0)
                self.num_timesteps += self.n_envs
                n_collected += 1
                self.buffer.add(obs, next_obs, acts if acts is not None else 0, dones)
                progress = 1.0 - float(self.num_timesteps) / float(self._total_timesteps)
                # DQN._on_step
                self._n_calls += 1
                if self._n_calls % max(self.target_update_interval // self.n_envs, 1) == 0:
                    self.target_update_calls.append(self._n_calls)
                    if target_fn:
                        target_fn()
                self.exploration_rate = self.exploration_schedule(progress)
                self.rates.append(self.exploration_rate)
            if self.num_timesteps > 0 and self.num_timesteps > self.learning_starts:
                gs = self.gradient_steps if self.gradient_steps >= 0 else self.train_freq * self.n_envs
                if gs > 0:
                    self.train_calls.append(gs)
                    for _ in range(gs):
                        n_l = self.batch_size // 2
                        n_e = self.batch_size - n_l
                        bi, ei = self.buffer.sample(n_l)
                        xi = np.random.randint(0, self.n_expert, size=n_e)
                        np.random.randint(0, high=1, size=(n_e,))  # the expert buffer's env index (n_envs 1)
                        self.samples.append((bi, ei, xi))
                        if train_fn:
                            train_fn(self.samples[-1])
                    self._n_updates += gs


# ---- the TD step in float64 ---------------------------------------------------------------------------------------

def _act(z, relu: bool):
    return np.maximum(z, 0.0) if relu else np.tanh(z)


def _act_grad(g, a, relu: bool):
    return np.where(a > 0, g, 0.0) if relu else g * (1.0 - a * a)


def q_forward(p, x, relu: bool = True):
    """p: dict w1 b1 w2 b2 w3 b3 (torch Linear layout) -> (h1, h2, Q)."""
    h1 = _act(x @ p["w1"].T + p["b1"], relu)
    h2 = _act(h1 @ p["w2"].T + p["b2"], relu)
    return h1, h2, h2 @ p["w3"].T + p["b3"]


def td_targets(p_target, next_obs, dones, rewards, gamma: float, relu: bool = True):
    return rewards + (1.0 - dones) * gamma * q_forward(p_target, next_obs, relu)[2].max(1)


def td_grad(p, obs, acts, y, relu: bool = True):
    """(loss, gradient dict) of F.smooth_l1_loss(Q(obs)[acts], y) (beta 1, mean)."""
    B = len(obs)
    h1, h2, q = q_forward(p, obs, relu)
    d = q[np.arange(B), acts] - y
    ad = np.abs(d)
    loss = np.mean(np.where(ad < 1.0, 0.5 * d * d, ad - 0.5))
    dq = np.zeros_like(q)
    dq[np.arange(B), acts] = np.clip(d, -1.0, 1.0) / B
    g = {"w3": dq.T @ h2, "b3": dq.sum(0)}
    dz2 = _act_grad(dq @ p["w3"], h2, relu)
    g["w2"], g["b2"] = dz2.T @ h1, dz2.sum(0)
    dz1 = _act_grad(dz2 @ p["w2"], h1, relu)
    g["w1"], g["b1"] = dz1.T @ obs, dz1.sum(0)
    return loss, g


KEYS = ("w1", "b1", "w2", "b2", "w3", "b3")


def td_step(p, m, v, step: int, obs, acts, y, lr: float, max_grad_norm: float, eps: float = 1e-8, relu: bool = True):
    """One DQN.train step: smooth L1, clip_grad_norm_, torch Adam (step = the count after this step).  Updates p, m, v
    in place; returns the loss."""
    loss, g = td_grad(p, obs, acts, y, relu)
    total = np.sqrt(sum(np.sum(g[k] ** 2) for k in KEYS))
    clip = min(max_grad_norm / (total + 1e-6), 1.0)
    bc1, bc2 = 1 - 0.9 ** step, 1 - 0.999 ** step
    for k in KEYS:
        gk = g[k] * clip
        m[k] = 0.9 * m[k] + 0.1 * gk
        v[k] = 0.999 * v[k] + 0.001 * gk * gk
        p[k] = p[k] - (lr / bc1) * m[k] / (np.sqrt(v[k]) / np.sqrt(bc2) + eps)
    return loss
