"""Behavioural cloning restated on torch-CPU in float64 (the reference's BC.train, algorithms/bc.py:381-510).

TEST INFRASTRUCTURE.  Needs no reference: it is pinned to tests/golden/bc.npz (recorded from the reference's own
BC.train by oracle/bc_ref.py) on the CPU, and the GPU tests hold the device kernel to it.  The policy is
oracle.ppo_port.ActorCriticPort (tanh or ReLU towers) in float64; the minibatch order is given as per-epoch index
permutations, as the reference's DataLoader(shuffle=True, drop_last=True) draws them.  The loop is the reference's:
minibatch loss (BehaviorCloningLossCalculator) x minibatch_size / batch_size, backward, an Adam step every
batch_size / minibatch_size minibatches and after an incomplete last batch, metrics of every logged batch.
"""
import types
from typing import List, Optional, Sequence

import numpy as np
import torch as th
from torch import nn

from .ppo_port import ActorCriticPort

METRICS = ("neglogp", "entropy", "ent_loss", "prob_true_act", "l2_norm", "l2_loss", "loss")


def _features(self, obs):
    """ActorCriticPort.features in the policy's own dtype (it casts to float32)."""
    x = th.flatten(obs, 1).to(self.action_net.weight.dtype)
    return self.feat_norm(x) if self.feat_norm is not None else x


def make_policy(d_obs: int, d_act: int, discrete: bool, hidden: int, normalize_features: bool, relu: bool = False,
                dtype=th.float64) -> ActorCriticPort:
    p = ActorCriticPort(d_obs, d_act, discrete=discrete, hidden=(hidden, hidden), normalize_features=normalize_features)
    p.features = types.MethodType(_features, p)
    if relu:
        for seq in (p.pi, p.vf):
            for i, m in enumerate(seq):
                if isinstance(m, nn.Tanh):
                    seq[i] = nn.ReLU()
    return p.to(dtype)


def _tensors(p: ActorCriticPort) -> List[th.Tensor]:
    """The policy's parameters in this package's flat order (imitation_b200._desc.policy_param_shapes)."""
    t = [p.pi[0].weight, p.pi[0].bias, p.pi[2].weight, p.pi[2].bias, p.vf[0].weight, p.vf[0].bias, p.vf[2].weight,
         p.vf[2].bias, p.action_net.weight, p.action_net.bias, p.value_net.weight, p.value_net.bias]
    return t + ([] if p.log_std is None else [p.log_std])


def get_flat(p: ActorCriticPort) -> np.ndarray:
    return th.cat([t.detach().reshape(-1) for t in _tensors(p)]).double().numpy()


def set_flat(p: ActorCriticPort, flat) -> None:
    flat = th.as_tensor(np.asarray(flat, dtype=np.float64))
    o = 0
    with th.no_grad():
        for t in _tensors(p):
            t.copy_(flat[o:o + t.numel()].reshape(t.shape).to(t.dtype))
            o += t.numel()
    assert o == len(flat)


def adam_state(opt: th.optim.Optimizer, p: ActorCriticPort, key: str) -> np.ndarray:
    parts = []
    for t in _tensors(p):
        st = opt.state.get(t, {})
        parts.append(st[key].detach().reshape(-1).double() if key in st else th.zeros(t.numel(), dtype=th.float64))
    return th.cat(parts).numpy()


class BCPort:
    """One BC object's training state: the policy, torch Adam (float64) and the counters a train() call reads."""

    def __init__(self, policy: ActorCriticPort, batch_size: int, minibatch_size: int, lr: float = 1e-3,
                 eps: float = 1e-8, ent_weight: float = 1e-3, l2_weight: float = 0.0):
        self.policy = policy
        self.batch_size, self.minibatch_size = batch_size, minibatch_size
        self.ent_weight, self.l2_weight = ent_weight, l2_weight
        self.opt = th.optim.Adam(policy.parameters(), lr=lr, eps=eps)

    def loss(self, obs, acts):
        p = self.policy
        _, log_prob, entropy = p.evaluate_actions(obs, acts)
        prob_true_act = th.exp(log_prob).mean()
        log_prob = log_prob.mean()
        entropy = entropy.mean()
        l2_norm = sum(th.sum(th.square(w)) for w in p.parameters()) / 2
        ent_loss = -self.ent_weight * entropy
        neglogp = -log_prob
        l2_loss = self.l2_weight * l2_norm
        loss = neglogp + ent_loss + l2_loss
        return loss, (neglogp, entropy, ent_loss, prob_true_act, l2_norm, l2_loss, loss)

    def train(self, obs: np.ndarray, acts: np.ndarray, perms: Sequence[np.ndarray], n_minibatches: int,
              log_interval: int = 500, norm_update: bool = True, grads: Optional[list] = None):
        """Minibatches 0 .. n_minibatches - 1 of one train() call, minibatch i = rows perms[i // per_epoch][...] of
        (obs, acts).  Returns [(batch_num, [7 metrics])] of the logged batches.  grads (optional): each optimiser
        batch's summed gradient (flat order), appended before its step."""
        p, mb, k = self.policy, self.minibatch_size, self.batch_size // self.minibatch_size
        per_epoch = len(obs) // mb
        p.train(norm_update)
        obs_t = th.as_tensor(np.asarray(obs, dtype=np.float64).reshape(len(obs), -1))
        acts_t = th.as_tensor(np.asarray(acts, dtype=np.float64))
        logged = []

        def step(batch_num, metrics):
            if grads is not None:
                grads.append(th.cat([(t.grad if t.grad is not None else th.zeros_like(t)).reshape(-1)
                                     for t in _tensors(p)]).numpy().copy())
            self.opt.step()
            self.opt.zero_grad()
            if batch_num % log_interval == 0:
                logged.append((batch_num, [float(m.detach()) for m in metrics]))

        self.opt.zero_grad()
        metrics = None
        for i in range(n_minibatches):
            perm = np.asarray(perms[i // per_epoch])
            idx = th.as_tensor(perm[(i % per_epoch) * mb:(i % per_epoch + 1) * mb].astype(np.int64))
            loss, metrics = self.loss(obs_t[idx], acts_t[idx])
            (loss * mb / self.batch_size).backward()
            if ((i + 1) * mb) % self.batch_size == 0:
                step(i // k, metrics)
        if n_minibatches and (n_minibatches * mb) % self.batch_size != 0:
            step((n_minibatches - 1) // k + 1, metrics)
        return logged
