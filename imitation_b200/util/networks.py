"""RunningNorm, EMANorm + train/eval helpers with the reference's semantics.

Mirrors imitation.util.networks: `training` / `evaluating` context managers
(util/networks.py:12-34) and `RunningNorm` (util/networks.py:47-134: in train mode update
the running statistics FIRST, then normalise with the updated ones; Chan merge with the
biased batch variance; int32 `count`).  The module is a plain nn.Module with the same buffer
names, so state_dicts are interchangeable with the reference; inside the fused reward
networks its buffers alias the flat device vectors the kernels read and write.
"""
import contextlib
import functools

import torch as th
from torch import nn


def _set_mode(m: nn.Module, mode: bool) -> None:
    # nn.Module.train() goes through Module.__setattr__ (Parameter/Module isinstance checks, ~40 us per
    # submodule); `training` is a plain instance attribute, so write it directly -- this runs around
    # every discriminator update (common.py:441-443 of the reference).
    for sub in m.modules():
        sub.__dict__["training"] = mode


@contextlib.contextmanager
def training_mode(m: nn.Module, mode: bool = False):
    old = m.training
    _set_mode(m, mode)
    try:
        yield m
    finally:
        _set_mode(m, old)


training = functools.partial(training_mode, mode=True)
evaluating = functools.partial(training_mode, mode=False)


class BaseNorm(nn.Module):
    def __init__(self, num_features: int, eps: float = 1e-5):
        super().__init__()
        self.eps = eps
        self.num_features = num_features
        self.register_buffer("running_mean", th.zeros(num_features))
        self.register_buffer("running_var", th.ones(num_features))
        self.register_buffer("count", th.zeros((), dtype=th.int))

    def reset_running_stats(self) -> None:
        self.running_mean.zero_()
        self.running_var.fill_(1)
        self.count.zero_()

    def forward(self, x: th.Tensor) -> th.Tensor:
        if self.training:
            with th.no_grad():
                self.update_stats(x)
        return (x - self.running_mean) / th.sqrt(self.running_var + self.eps)

    def update_stats(self, batch: th.Tensor) -> None:
        raise NotImplementedError


class RunningNorm(BaseNorm):
    """Stand-alone use (e.g. NormalizedRewardNet's output layer) runs these few torch ops on
    the module's device; inside fused nets the kernels update the aliased buffers instead."""

    def update_stats(self, batch: th.Tensor) -> None:
        if batch.ndim == 1:
            batch = batch.reshape(-1, 1)
        b_mean = th.mean(batch, dim=0)
        b_var = th.var(batch, dim=0, unbiased=False)
        b_n = batch.shape[0]
        delta = b_mean - self.running_mean
        tot = self.count + b_n
        self.running_mean += delta * b_n / tot
        self.running_var *= self.count
        self.running_var += b_var * b_n
        self.running_var += th.square(delta) * self.count * b_n / tot
        self.running_var /= tot
        self.count += b_n


class EMANorm(BaseNorm):
    """Exponentially weighted running statistics (util/networks.py:137-201): the k-th batch (k = num_batches, from 0)
    is folded with learning rate 1 / inv_learning_rate after inv_learning_rate += decay ** k, each line one float32
    torch op as in the reference.  Buffers, shapes and dtypes are the reference's, so state dicts load both ways.  As an
    output layer of a fused reward net the kernels update the aliased buffers instead."""

    def __init__(self, num_features: int, decay: float = 0.99, eps: float = 1e-5):
        super().__init__(num_features, eps=eps)
        if not 0 < decay < 1:
            raise ValueError("decay must be between 0 and 1")
        self.decay = decay
        self.register_buffer("inv_learning_rate", th.zeros(()))
        self.register_buffer("num_batches", th.zeros((), dtype=th.int))

    def reset_running_stats(self) -> None:
        super().reset_running_stats()
        self.inv_learning_rate.zero_()
        self.num_batches.zero_()

    def update_stats(self, batch: th.Tensor) -> None:
        if batch.ndim == 1:
            batch = batch.reshape(-1, 1)
        self.inv_learning_rate += th.pow(self.decay, self.num_batches)
        lr = 1 / self.inv_learning_rate
        delta = th.mean(batch, dim=0) - self.running_mean
        self.running_mean += lr * delta
        delta_var = th.var(batch, dim=0, unbiased=False) + (1 - lr) * th.square(delta) - self.running_var
        self.running_var += lr * delta_var
        self.count += batch.shape[0]
        self.num_batches += 1


class SqueezeLayer(nn.Module):
    def forward(self, x):
        assert x.ndim == 2 and x.shape[1] == 1
        return x.squeeze(1)
