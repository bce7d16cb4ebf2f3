"""Tabular MCE IRL restated in float64 NumPy + torch-CPU.  TEST INFRASTRUCTURE.

Follows /root/reference/src/imitation/algorithms/mce_irl.py: `partition_fh` is mce_partition_fh (:38-93),
`occupancy` is mce_occupancy_measures (:96-144) with rollout.discounted_sum, `train_iteration` is one iteration of
MCEIRL.train (:500-556) with its _train_step (:467-498) on a torch-CPU reward net (oracle/nets_port.py) and a torch
Adam.  It is the reference the device sweep and trainer are held to at shapes the golden does not cover.
"""
from typing import Optional, Tuple

import numpy as np
import scipy.special
import torch as th


def partition_fh(T: np.ndarray, reward: np.ndarray, horizon: int, discount: float = 1.0
                 ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(V [H, S], Q [H, S, A], pi [H, S, A]) of the soft Bellman backup; T [S, A, S], reward [S]."""
    S, A = T.shape[:2]
    V = np.full((horizon, S), -np.inf)
    Q = np.zeros((horizon, S, A))
    Q[horizon - 1] = reward[:, None]
    V[horizon - 1] = scipy.special.logsumexp(Q[horizon - 1], axis=1)
    for t in reversed(range(horizon - 1)):
        Q[t] = reward[:, None] + discount * (T @ V[t + 1])
        V[t] = scipy.special.logsumexp(Q[t], axis=1)
    return V, Q, np.exp(Q - V[:, :, None])


def discounted_sum(D: np.ndarray, discount: float) -> np.ndarray:
    if discount == 1.0:
        return D.sum(axis=0)
    return np.polynomial.polynomial.polyval(discount, D)


def occupancy(T: np.ndarray, initial: np.ndarray, pi: np.ndarray, horizon: int, discount: float = 1.0
              ) -> Tuple[np.ndarray, np.ndarray]:
    """(D [H + 1, S], Dcum [S]) under the policy pi [H, S, A]."""
    S, A = T.shape[:2]
    D = np.zeros((horizon + 1, S))
    D[0] = initial
    for t in range(horizon):
        for a in range(A):
            D[t + 1] += (D[t] * pi[t, :, a]) @ T[:, a, :]
    return D, discounted_sum(D, discount)


def tensor_iter_norm(tensors) -> float:
    """util.tensor_iter_norm: the 2-norm of the per-tensor 2-norms (float32)."""
    return float(th.linalg.norm(th.as_tensor([th.norm(t.flatten(), p=2) for t in tensors])))


def train_iteration(net: th.nn.Module, opt: th.optim.Optimizer, obs: th.Tensor, T: np.ndarray, initial: np.ndarray,
                    horizon: int, demo_om: np.ndarray, discount: float) -> dict:
    """One iteration of MCEIRL.train: net in training mode on the [S, d] float32 observations (a RunningNorm input
    layer updates once), undiscounted planning, occupancy discounted by `discount`, loss = weights . r, backward, Adam.
    Returns the reward, Dcum, weights, grad, grad_norm and linf_delta of the iteration."""
    net.train()
    opt.zero_grad()
    r = net(obs, None, None, None)
    r_np = r.detach().numpy()
    _, _, pi = partition_fh(T, r_np.astype(np.float64), horizon)
    _, Dcum = occupancy(T, initial, pi, horizon, discount)
    w = th.as_tensor(Dcum - demo_om, dtype=th.float32)
    th.dot(w, r).backward()
    grads = [p.grad.detach().clone() for p in net.parameters()]
    opt.step()
    return dict(reward=r_np, Dcum=Dcum, weights=w.numpy(), grad=th.cat([g.flatten() for g in grads]).numpy(),
                grad_norm=tensor_iter_norm(grads), linf_delta=float(np.max(np.abs(demo_om - Dcum))))


def final_policy(T: np.ndarray, reward: np.ndarray, horizon: int, discount: float) -> np.ndarray:
    return partition_fh(T, np.asarray(reward, dtype=np.float64), horizon, discount)[2]


class StateOnlyNet(th.nn.Module):
    """BasicRewardNet(use_action=False) on observation rows, called as net(obs, None, None, None)."""

    def __init__(self, mlp: th.nn.Sequential):
        super().__init__()
        self.mlp = mlp

    def forward(self, state, action=None, next_state=None, done=None):
        return self.mlp(state).squeeze(1)


def port_net(d_obs: int, hid_sizes, normalize_input: bool, state_dict: Optional[dict] = None) -> StateOnlyNet:
    from oracle.nets_port import mlp_port

    net = StateOnlyNet(mlp_port(d_obs, tuple(hid_sizes), normalize_input))
    if state_dict is not None:
        net.load_state_dict({k: th.as_tensor(np.asarray(v)) for k, v in state_dict.items()})
    return net
