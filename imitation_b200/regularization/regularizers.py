"""Regularizers of a network's training step (the public API of imitation.regularization.regularizers).

A regularizer is configured in two steps.  `SomeRegularizer.create(initial_lambda, lambda_updater, val_split, **kw)`
returns a `RegularizerFactory`; the trainer that owns the optimiser and the logger then calls
`factory(optimizer=..., logger=...)`.  The trainer calls `regularize_and_backward(loss)` in place of `loss.backward()`
for every minibatch and, when the regularizer has a `lambda_updater`, `update_params(train_loss, val_loss)` once per
epoch with the losses of that epoch.

`BasicRewardTrainer` runs `LpRegularizer` and `WeightDecayRegularizer` (these exact classes) inside its device-only
step with the `imb_param_regularize` kernel; subclasses and other regularizers run through its autograd path.
"""
import abc
from typing import Optional, Protocol, Union

import numpy as np
import torch as th
from torch import optim

from ..util import logger as imit_logger
from . import updaters


class RegularizerFactory(Protocol):
    """What `Regularizer.create` returns: builds the regularizer once the optimiser and the logger exist.  One factory
    may build regularizers for several networks (an ensemble's members each get their own)."""

    def __call__(self, *, optimizer: optim.Optimizer, logger: imit_logger.HierarchicalLogger) -> "Regularizer":
        ...


def _check_settings(initial_lambda, lambda_updater, val_split) -> None:
    """The constructor's validation: an updater and a validation split go together, the split lies strictly inside
    (0, 1), and a regularizer without an updater has a non-zero strength."""
    if lambda_updater is None and np.allclose(initial_lambda, 0.0):
        raise ValueError("If you do not pass a regularizer parameter updater your regularization strength must be "
                         "non-zero, as this would result in no regularization.")
    split_ok = isinstance(val_split, float) and 0 < val_split < 1 and not np.allclose(val_split, 0.0)
    if val_split is not None and not split_ok:
        raise ValueError(f"val_split = {val_split} must be a float strictly between 0 and 1.")
    if (lambda_updater is None) != (val_split is None):
        if val_split is None:
            raise ValueError("If you pass a regularizer parameter updater, you must also specify a validation split. "
                             "Otherwise the updater won't have any validation data to use for updating.")
        raise ValueError("If you pass a validation split, you must also pass a regularizer parameter updater. "
                         "Otherwise you are wasting data into the validation split that will not be used.")


class Regularizer(abc.ABC):
    """Strength `lambda_`, optionally adapted once per epoch by `lambda_updater` from the losses on the training part
    and on a validation part of `val_split` of the data.  An updater and a split go together; without an updater,
    lambda_ must be non-zero and val_split None.  The strength is recorded as `regularization_lambda` at construction
    and after every update."""

    def __init__(self, optimizer: optim.Optimizer, initial_lambda: float,
                 lambda_updater: Optional[updaters.LambdaUpdater], logger: imit_logger.HierarchicalLogger,
                 val_split: Optional[float] = None) -> None:
        _check_settings(initial_lambda, lambda_updater, val_split)
        self.optimizer, self.logger = optimizer, logger
        self.lambda_updater, self.val_split = lambda_updater, val_split
        self.lambda_ = initial_lambda
        logger.record("regularization_lambda", initial_lambda)

    @classmethod
    def create(cls, initial_lambda: float, lambda_updater: Optional[updaters.LambdaUpdater] = None,
               val_split: float = 0.0, **kwargs) -> RegularizerFactory:
        """A factory for `cls` with these settings.  The default val_split of 0.0 is rejected when the factory is
        called: pass `val_split=None` for a regularizer without an updater."""
        settings = dict(kwargs, initial_lambda=initial_lambda, lambda_updater=lambda_updater, val_split=val_split)
        return lambda *, optimizer, logger: cls(optimizer=optimizer, logger=logger, **settings)

    @abc.abstractmethod
    def regularize_and_backward(self, loss: th.Tensor):
        """Apply the regularization to one minibatch, `loss.backward()` included."""

    def update_params(self, train_loss: Union[th.Tensor, float], val_loss: Union[th.Tensor, float]) -> None:
        """lambda_ = lambda_updater(lambda_, train_loss, val_loss), recorded as `regularization_lambda`; nothing
        without an updater."""
        if self.lambda_updater is None:
            return
        self.lambda_ = self.lambda_updater(self.lambda_, train_loss, val_loss)
        self.logger.record("regularization_lambda", self.lambda_)


class LossRegularizer(Regularizer):
    """Adds `_loss_penalty(loss)` to the loss before the backward pass and records the sum as `regularized_loss`."""

    @abc.abstractmethod
    def _loss_penalty(self, loss: th.Tensor) -> Union[th.Tensor, float]:
        """The term added to the loss (not the regularized loss)."""

    def regularize_and_backward(self, loss: th.Tensor) -> th.Tensor:
        total = th.add(loss, self._loss_penalty(loss))
        total.backward()
        self.logger.record("regularized_loss", total.item())
        return total


class WeightRegularizer(Regularizer):
    """After `loss.backward()`, adds `_weight_penalty(param, group)` to every parameter the optimiser holds, in place
    (the parameters keep their storage, so views of a flat parameter vector stay views)."""

    @abc.abstractmethod
    def _weight_penalty(self, weight: th.Tensor, group: dict) -> Union[th.Tensor, float]:
        """The term added to `weight` (not the new weight)."""

    def regularize_and_backward(self, loss: th.Tensor) -> None:
        loss.backward()
        for group in self.optimizer.param_groups:
            for weight in group["params"]:
                weight.data.add_(self._weight_penalty(weight, group))


class LpRegularizer(LossRegularizer):
    """Penalty lambda_ * sum over the optimiser's parameter tensors of ||w||_p ** p, p an integer >= 1."""

    def __init__(self, optimizer: optim.Optimizer, initial_lambda: float,
                 lambda_updater: Optional[updaters.LambdaUpdater], logger: imit_logger.HierarchicalLogger, p: int,
                 val_split: Optional[float] = None) -> None:
        super().__init__(optimizer, initial_lambda, lambda_updater, logger, val_split)
        if not isinstance(p, int) or p < 1:
            raise ValueError("p must be a positive integer")
        self.p = p

    def _loss_penalty(self, loss: th.Tensor) -> th.Tensor:
        # tensor by tensor, in the optimiser's order (the summation order of the reference's penalty)
        norms = [th.linalg.vector_norm(w, ord=self.p).pow(self.p) for g in self.optimizer.param_groups
                 for w in g["params"]]
        return self.lambda_ * sum(norms)


class WeightDecayRegularizer(WeightRegularizer):
    """w <- w + (-lambda_ * lr) * w after every minibatch's backward pass, lr the parameter group's learning rate (on
    top of any decay the optimiser applies itself).  The coefficient is one Python float, multiplied into w in the
    tensor's dtype, then added: two rounded float32 operations."""

    def _weight_penalty(self, weight: th.Tensor, group: dict) -> th.Tensor:
        coeff = -self.lambda_ * group["lr"]
        return coeff * weight.data
