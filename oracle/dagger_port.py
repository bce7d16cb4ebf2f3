"""CPU twin of the DAgger rollout (csrc/imb_rollout_impl.cuh, k_rollout in RM_DAGGER mode; imb_rollout_dagger).

TEST INFRASTRUCTURE.  The reference's `InteractiveTrajectoryCollector` under `generate_trajectories(expert, collector,
deterministic_policy=...)` (algorithms/dagger.py:232-287, data/rollout.py:382-506) on the synthetic env: at every step
the expert acts (its mean / argmax, or sampled with the step's pinned noise), the recorded label is its action as
`predict` returns it (clipped to the Box, or the index), and where mask[t][e] is set the env executes the learner's
action instead: sampled with the step's pinned robot noise, clipped.  Both policies are `ppo_port.ActorCriticPort`s
evaluated in float64 (in evaluation mode: a feature RunningNorm is applied, not updated).
"""
import copy

import numpy as np
import torch as th


def _float64(pol):
    """A float64 copy of an ActorCriticPort in evaluation mode (its features kept in float64 too)."""
    pol = copy.deepcopy(pol).double().eval()
    norm = pol.feat_norm
    pol.features = lambda obs: norm(th.flatten(obs, 1)) if norm is not None else th.flatten(obs, 1)
    return pol


def _act(pol, obs, noise, deterministic):
    with th.no_grad():
        acts, _, _ = pol(th.as_tensor(obs, dtype=th.float64), None if noise is None else
                         th.as_tensor(noise, dtype=th.float64), deterministic=deterministic)
    acts = acts.numpy()
    return acts if pol.discrete else np.clip(acts, -1.0, 1.0)


def collect(spec, expert, learner, obs0, mask, noise, robot_noise, deterministic: bool):
    """One batch of E whole episodes from episode step 0 (H = spec.horizon steps, obs0 [E][d_obs] the reset
    observations).  mask uint8 [H][E]; noise / robot_noise [H][E][d_act] normals or [H][E] uniforms (noise unused when
    deterministic).  Returns dict(obs [E][H][d_obs], labels [E][H][d_act] or [E][H], next_obs [E][H][d_obs] (the
    terminal observation last), rews [E][H])."""
    expert, learner = _float64(expert), _float64(learner)
    H = spec.horizon
    obs = np.asarray(obs0, np.float64)
    out = {k: [] for k in ("obs", "labels", "next_obs", "rews")}
    for t in range(H):
        label = _act(expert, obs, None if deterministic else noise[t], deterministic)
        executed = label.copy()
        m = np.asarray(mask[t]).astype(bool)
        if m.any():
            executed[m] = _act(learner, obs, robot_noise[t], False)[m]
        nobs, rew = spec.dynamics(obs.astype(np.float32), executed)
        out["obs"].append(obs.copy())
        out["labels"].append(label)
        out["next_obs"].append(nobs.astype(np.float64))
        out["rews"].append(rew.astype(np.float64))
        obs = nobs.astype(np.float64)
    return {k: np.swapaxes(np.stack(v), 0, 1) for k, v in out.items()}
