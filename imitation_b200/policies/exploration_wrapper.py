"""`ExplorationWrapper` (mirror of imitation.policies.exploration_wrapper:12-95) for the device rollout.

The reference wraps a policy callable: at every step of `generate_trajectories` the current policy (the wrapped one, or
a random one calling `action_space.sample()` per env) acts for the whole VecEnv, then one `rng.random()` decides whether
to switch, and a switch draws once more to pick the new policy.  Which policy acts at a step never depends on the
observations, so the chain can be drawn on the host before the rollout: `advance(n)` draws it for n steps exactly as n
calls of the reference's `__call__` would, and returns it as the per-step vector the exploration rollout kernel reads
(`imb_rollout_explore`, via `DevicePPO.exploration_rollout`).  The random actions are drawn on the device from a Philox
stream keyed by the seed the constructor draws (the reference seeds `action_space` with it); the stream's counter is
the number of steps the chain has covered, so consecutive rollouts draw different actions and equal seeds equal ones.
There is no per-step `__call__`: the device env is stepped only by the rollout kernel.
"""
import numpy as np

from ..algorithms.preference_comparisons import make_seeds


class ExplorationWrapper:
    """Switches between `policy` and a random policy (exploration_wrapper.py:23-56): after each step the current policy
    is kept with probability 1 - switch_prob; otherwise the random policy is picked with probability random_prob.

    `policy`: the device algorithm (or its policy) whose rollout this wrapper drives; `venv`: the env it acts in, whose
    `action_space` the random policy samples (seeded with the drawn seed when it can be); `rng`: the shared generator,
    drawn from twice here (the seed, then the initial policy) and once or twice per step by `advance`."""

    def __init__(self, policy, venv, random_prob: float, switch_prob: float, rng: np.random.Generator,
                 deterministic_policy: bool = False) -> None:
        self.wrapped_policy = policy
        self.random_prob = random_prob
        self.switch_prob = switch_prob
        self.venv = venv
        self.deterministic_policy = deterministic_policy
        self.rng = rng
        self.seed = make_seeds(self.rng)
        if hasattr(venv.action_space, "seed"):
            venv.action_space.seed(self.seed)
        self.steps_taken = 0  # steps the chain has covered: the Philox counter of the next random step
        self.random_current = False
        self._switch()  # choose the initial policy at random

    def _switch(self) -> None:
        self.random_current = bool(self.rng.random() < self.random_prob)

    def advance(self, n: int) -> np.ndarray:
        """Policy of each of the next n steps (uint8 [n]: 1 = random, 0 = the wrapped policy), drawing from `rng` as n
        calls of the reference's `__call__` do (exploration_wrapper.py:75-95); the chain carries over to the next call.
        Advances `steps_taken` by n."""
        out = np.empty(n, np.uint8)
        for t in range(n):
            out[t] = self.random_current
            if self.rng.random() < self.switch_prob:
                self._switch()
        self.steps_taken += n
        return out
