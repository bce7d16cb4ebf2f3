"""Seeded tabular MDPs for the MCE IRL tests and benchmark.  TEST INFRASTRUCTURE.

`TabularMDP` carries the attributes MCE IRL reads from a `TabularModelPOMDP` (transition_matrix [S, A, S],
observation_matrix [S, d], initial_state_dist [S], reward_matrix [S], horizon, state_dim, action_dim, state_space,
action_space, observation_space).  The builders are this repository's own:
  random_mdp       S states, A actions, each (s, a) reaching `branch` random next states with Dirichlet weights;
                   one-hot or random Gaussian observation features; `branch` random initial states.
  gridworld        an n x n slippery grid (4 moves; the intended move with probability 1 - slip, a uniformly random one
                   otherwise, walls keep the agent in place), `xy` features (row, column scaled to [0, 1]) or random
                   ones; starts uniformly in the first row.
  known_reward_mdp a small MDP with random features and a reward linear in them, so that the occupancy measure of
                   its soft-optimal policy (planned undiscounted, as MCEIRL plans) is reachable by a linear reward net:
                   the behavioural check.  Seed 0 is the one whose runs converge within the default 1000
                   iterations for a linear and a [32, 32] net at every tested discount.
"""
from dataclasses import dataclass
from typing import Optional

import numpy as np

from imitation_b200 import spaces


@dataclass
class TabularMDP:
    transition_matrix: np.ndarray
    observation_matrix: np.ndarray
    initial_state_dist: np.ndarray
    reward_matrix: np.ndarray
    horizon: Optional[int]

    @property
    def state_dim(self) -> int:
        return self.transition_matrix.shape[0]

    @property
    def action_dim(self) -> int:
        return self.transition_matrix.shape[1]

    @property
    def obs_dim(self) -> int:
        return self.observation_matrix.shape[1]

    @property
    def state_space(self):
        return spaces.Discrete(self.state_dim)

    @property
    def action_space(self):
        return spaces.Discrete(self.action_dim)

    @property
    def observation_space(self):
        return spaces.Box(-np.inf, np.inf, (self.obs_dim,), np.float32)


def _features(rng: np.random.Generator, n_states: int, obs_dim: Optional[int]) -> np.ndarray:
    if obs_dim is None:
        return np.eye(n_states)
    return rng.normal(size=(n_states, obs_dim))


def random_mdp(n_states: int, n_actions: int, branch: int, horizon: int, obs_dim: Optional[int] = None,
               seed: int = 0, reward_scale: float = 1.0) -> TabularMDP:
    """obs_dim None: one-hot features (d = S)."""
    rng = np.random.default_rng(seed)
    branch = min(branch, n_states)
    T = np.zeros((n_states, n_actions, n_states))
    for s in range(n_states):
        for a in range(n_actions):
            nxt = rng.choice(n_states, size=branch, replace=False)
            T[s, a, nxt] = rng.dirichlet(np.ones(branch))
    init = np.zeros(n_states)
    init[rng.choice(n_states, size=branch, replace=False)] = rng.dirichlet(np.ones(branch))
    obs = _features(rng, n_states, obs_dim)
    reward = reward_scale * rng.normal(size=n_states)
    return TabularMDP(T, obs, init, reward, horizon)


def gridworld(n: int, horizon: int, slip: float = 0.2, features: str = "xy", obs_dim: int = 16,
              seed: int = 0) -> TabularMDP:
    rng = np.random.default_rng(seed)
    S, moves = n * n, ((-1, 0), (1, 0), (0, -1), (0, 1))
    T = np.zeros((S, 4, S))
    for s in range(S):
        i, j = divmod(s, n)
        dest = []
        for di, dj in moves:
            ii, jj = i + di, j + dj
            dest.append(ii * n + jj if 0 <= ii < n and 0 <= jj < n else s)
        for a in range(4):
            T[s, a, dest[a]] += 1.0 - slip
            for d in dest:
                T[s, a, d] += slip / 4
    init = np.zeros(S)
    init[:n] = 1.0 / n
    if features == "xy":
        ij = np.stack(np.divmod(np.arange(S), n), axis=1)
        obs = ij / max(n - 1, 1)
    else:
        obs = rng.normal(size=(S, obs_dim))
    reward = rng.normal(size=S)
    return TabularMDP(T, obs, init, reward, horizon)


def known_reward_mdp(seed: int = 0, n_states: int = 12, n_actions: int = 3, obs_dim: int = 6,
                     horizon: int = 15) -> TabularMDP:
    mdp = random_mdp(n_states, n_actions, branch=3, horizon=horizon, obs_dim=obs_dim, seed=seed)
    w = 0.3 * np.random.default_rng(seed + 1).normal(size=obs_dim)
    mdp.reward_matrix = mdp.observation_matrix @ w
    return mdp
