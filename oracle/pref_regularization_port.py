"""TEST INFRASTRUCTURE -- CPU restatement of preference comparisons' reward training with a regularizer
(algorithms/preference_comparisons.py:1218-1311 BasicRewardTrainer._train, :1408-1438 EnsembleTrainer._train;
regularization/regularizers.py LpRegularizer / WeightDecayRegularizer; regularization/updaters.py
IntervalParamScaler), on the oracle's reward-network ports and the preference-model port.  Pinned by
tests/golden/pref_regularization.npz (recorded from the reference's own classes).  Only tests/ may import this module."""
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch as th
from torch.utils import data as data_th

from . import pref_port


def interval_scale(lam: float, train_loss: float, val_loss: float, factor: float, lo: float, hi: float) -> float:
    """The interval rule for losses away from zero: up by (1 + factor) above [lo, hi], down by (1 - factor) below."""
    ratio = val_loss / train_loss
    if ratio > hi:
        return lam * (1 + factor)
    if ratio < lo:
        return lam * (1 - factor)
    return lam


def _minibatch(net, pairs, prefs, ids, noise_prob, discount_factor):
    probs, gt = pref_port.preference_probs_port(net, [pairs[i] for i in ids], noise_prob, discount_factor)
    return pref_port.cross_entropy_loss_port(probs, gt.float(), prefs[ids])


def train_member(net, pairs: Sequence[Tuple[dict, dict]], prefs: np.ndarray, items: List[int], seed_rng,
                 kind: str, p: int, lam: float, updater: Optional[Tuple[float, float, float]], val_split, batch_size: int,
                 minibatch_size: int, epochs: int, lr: float, noise_prob: float, discount_factor: float
                 ) -> Tuple[float, List[float], Dict[str, float]]:
    """One member's training call on dataset items `items`: -> (lambda after the call, lambda after every epoch with
    an updater, the last epoch's means of regularized_loss (Lp) and val/{loss, accuracy, gt_reward_loss})."""
    optim = th.optim.AdamW(net.parameters(), lr=lr)
    params = list(net.parameters())
    train_items, val_items = items, None
    if val_split is not None:
        n_val = int(len(items) * val_split)
        seed = int(seed_rng.integers(0, (1 << 31) - 1, (1,))[0])
        order = th.randperm(len(items), generator=th.Generator().manual_seed(seed)).tolist()
        train_items = [items[i] for i in order[:len(items) - n_val]]
        val_items = [items[i] for i in order[len(items) - n_val:]]
    lambdas, last = [], {}
    net.train()
    for _ in range(epochs):
        last, reg_sum, n_mb, scaled_sum, acc_size = {}, 0.0, 0, 0.0, 0
        optim.zero_grad()
        for ids in data_th.DataLoader(train_items, batch_size=minibatch_size, shuffle=True):
            ids = [int(i) for i in ids]
            loss, _, _ = _minibatch(net, pairs, prefs, ids, noise_prob, discount_factor)
            loss = loss * (len(ids) / batch_size)
            scaled_sum += loss.item()
            if kind == "lp":
                total = loss + lam * sum(th.linalg.vector_norm(w, ord=p).pow(p) for w in params)
                total.backward()
                reg_sum += total.item()
            else:
                loss.backward()
                for w in params:
                    w.data.add_(-lam * lr * w.data)
            n_mb += 1
            acc_size += len(ids)
            if acc_size >= batch_size:
                optim.step()
                optim.zero_grad()
                acc_size = 0
        if acc_size:
            optim.step()
        if kind == "lp":
            last["regularized_loss"] = reg_sum / n_mb
        if val_items is None:
            continue
        sums, n_v = np.zeros(3), 0
        for ids in data_th.DataLoader(val_items, batch_size=minibatch_size, shuffle=True):
            loss, acc, gt_loss = _minibatch(net, pairs, prefs, [int(i) for i in ids], noise_prob, discount_factor)
            sums += [loss.item(), acc.item(), gt_loss.item()]
            n_v += 1
        last.update({"val/loss": sums[0] / n_v, "val/accuracy": sums[1] / n_v, "val/gt_reward_loss": sums[2] / n_v})
        lam = interval_scale(lam, scaled_sum, sums[0], *updater)
        lambdas.append(lam)
    return lam, lambdas, last


def train_ensemble(nets, pairs, prefs, rng, **kw):
    """EnsembleTrainer._train: one bagging sample per member from a generator seeded by one draw of `rng`, then the
    members one after the other, sharing `rng` for their split seeds."""
    seed = int(rng.integers(0, (1 << 31) - 1, (1,))[0])
    sampler = data_th.RandomSampler(range(len(pairs)), replacement=True, num_samples=len(pairs),
                                    generator=th.Generator().manual_seed(seed))
    return [train_member(net, pairs, prefs, [int(i) for i in sampler], rng, **kw) for net in nets]
