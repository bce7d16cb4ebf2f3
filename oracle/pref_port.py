"""TEST INFRASTRUCTURE -- CPU restatement of the reward-model side of preference comparisons
(algorithms/preference_comparisons.py:345-530 PreferenceModel, :1043-1090 CrossEntropyRewardLoss), fragment by
fragment like the reference, on the oracle's reward-network ports.  Pinned by tests/golden/preference.npz (generated
by oracle/make_golden.py from the reference's own classes).  Only tests/ may import this module."""
from typing import Optional, Sequence, Tuple

import numpy as np
import torch as th

from . import nets_port


def fragment_transitions(frag) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """data/rollout.py:563-621 flatten_trajectories of one fragment: dones only on the last step of a terminal one."""
    obs, acts = np.asarray(frag["obs"]), np.asarray(frag["acts"])
    dones = np.zeros(len(acts), dtype=bool)
    dones[-1] = bool(frag["terminal"])
    return obs[:-1], acts, obs[1:], dones


def probability_port(rews1: th.Tensor, rews2: th.Tensor, noise_prob: float, discount_factor: float,
                     threshold: float) -> th.Tensor:
    """preference_comparisons.py:487-530 (time on axis 0; vectors for a network, matrices for an ensemble)."""
    if discount_factor == 1:
        returns_diff = (rews2 - rews1).sum(axis=0)
    else:
        discounts = discount_factor ** th.arange(len(rews1))
        if rews1.ndim == 2:
            discounts = discounts.reshape(-1, 1)
        returns_diff = (discounts * (rews2 - rews1)).sum(axis=0)
    returns_diff = th.clip(returns_diff, -threshold, threshold)
    model_probability = 1 / (1 + returns_diff.exp())
    return noise_prob * 0.5 + (1 - noise_prob) * model_probability


def preference_probs_port(net: th.nn.Module, pairs: Sequence[Tuple[dict, dict]], noise_prob=0.0, discount_factor=1.0,
                          threshold=50.0) -> Tuple[th.Tensor, Optional[th.Tensor]]:
    """PreferenceModel.forward (:411-455): one reward-network call per fragment."""
    probs, gt = [], []
    for a, b in pairs:
        r1 = net(*nets_port.preprocess_port(*fragment_transitions(a)))
        r2 = net(*nets_port.preprocess_port(*fragment_transitions(b)))
        probs.append(probability_port(r1, r2, noise_prob, discount_factor, threshold))
        gt.append(probability_port(th.as_tensor(np.asarray(a["rews"])), th.as_tensor(np.asarray(b["rews"])), noise_prob,
                                   discount_factor, threshold))
    return th.stack(probs), th.stack(gt)


def cross_entropy_loss_port(probs: th.Tensor, gt_probs: th.Tensor, preferences: np.ndarray):
    """CrossEntropyRewardLoss.forward (:1050-1090): loss, accuracy, gt_reward_loss."""
    prefs = th.as_tensor(preferences, dtype=th.float32)
    accuracy = ((probs > 0.5) == (prefs > 0.5)).float().mean()
    gt_loss = th.nn.functional.binary_cross_entropy(gt_probs, prefs)
    return th.nn.functional.binary_cross_entropy(probs, prefs), accuracy, gt_loss


def pref_loss_closed_form(rews: np.ndarray, prefs: np.ndarray, noise_prob=0.0, discount_factor=1.0, threshold=50.0,
                          grad_scale=1.0):
    """NumPy (float32) twin of the `imb_pref_loss` kernel: the closed forms the kernel evaluates for one minibatch of P
    pairs, rews[2][P][L] -> (probs[P], mean BCE loss, accuracy, grad_scale * d loss / d rews[2][P][L]).  What autograd
    computes for probability_port + binary_cross_entropy (:487-530, :1043-1090):
      d = clip(sum_t g^t (r2 - r1)),  m = 1 / (1 + e^d),  p = noise / 2 + (1 - noise) m
      d loss / d p = (p - y) / max(p (1 - p), 1e-12) / P           (torch's BCE backward, incl. its clamp)
      d p / d d    = -(1 - noise) m (m e^d)                        (= -(1 - noise) m (1 - m) without the cancellation in 1 - m,
                                                                    and without the subnormal m^2 of |d| > 43.7)
      d d / d r2_t = g^t = -d d / d r1_t, and 0 where the return difference was clipped."""
    f = np.float32
    r = np.asarray(rews, dtype=f)
    P, L = r.shape[1], r.shape[2]
    w = (f(discount_factor) ** np.arange(L, dtype=f)).astype(f)
    s = ((r[1] - r[0]) * w).sum(axis=1, dtype=f)
    clipped = (s < -threshold) | (s > threshold)
    d = np.clip(s, -threshold, threshold).astype(f)
    ed = np.exp(d, dtype=f)
    m = (f(1) / (f(1) + ed)).astype(f)
    p = (f(noise_prob) * f(0.5) + (f(1) - f(noise_prob)) * m).astype(f)
    y = np.asarray(prefs, dtype=f)
    with np.errstate(divide="ignore"):
        lp, l1p = np.maximum(np.log(p), f(-100)), np.maximum(np.log1p(-p), f(-100))
    loss = float(np.mean(-(y * lp + (f(1) - y) * l1p)))
    acc = float(np.mean((p > 0.5) == (y > 0.5)))
    g = np.where(clipped, f(0), f(grad_scale) * (p - y) / np.maximum(p * (f(1) - p), f(1e-12)) / f(P)
                 * (-(f(1) - f(noise_prob)) * (m * (m * ed)))).astype(f)
    grad = np.stack([-(g[:, None] * w[None, :]), g[:, None] * w[None, :]]).astype(f)
    return p, loss, acc, grad
