"""Rules that adapt a regularizer's strength lambda between epochs from the training and validation losses
(imitation.regularization.updaters).  They run on the host: the trainer hands them two Python floats per epoch."""
from typing import Protocol, Tuple, Union

import numpy as np
import torch as th

LossType = Union[th.Tensor, float]


class LambdaUpdater(Protocol):
    """`(lambda_, train_loss, val_loss) -> new lambda_`.  Implementations must be free of side effects: the trainers call
    them once per epoch and rely on the result only.  Any callable with this signature (a plain function too) will do."""

    def __call__(self, lambda_, train_loss: LossType, val_loss: LossType) -> float:
        ...


def _is_scalar(x) -> bool:
    return isinstance(x, float) or (isinstance(x, th.Tensor) and x.dim() == 0)


class IntervalParamScaler(LambdaUpdater):
    """Multiply lambda by (1 + scaling_factor) when val_loss / train_loss lies above `tolerable_interval`, by
    (1 - scaling_factor) when it lies below, and keep it inside the interval (bounds included)."""

    def __init__(self, scaling_factor: float, tolerable_interval: Tuple[float, float]):
        eps = np.finfo(float).eps
        if not eps < scaling_factor < 1 - eps:
            raise ValueError("scaling_factor must be in (0, 1) within machine precision.")
        if len(tolerable_interval) != 2:
            raise ValueError("tolerable_interval must be a tuple of length 2")
        lo, hi = tolerable_interval
        if not 0 <= lo < hi:
            raise ValueError("tolerable_interval must be a tuple whose first element is at least 0 and the second "
                             "element is greater than the first")
        self.scaling_factor = scaling_factor
        self.tolerable_interval = tolerable_interval

    def __call__(self, lambda_: float, train_loss: LossType, val_loss: LossType) -> float:
        if not _is_scalar(val_loss):
            raise ValueError("val_loss must be a scalar")
        if not _is_scalar(train_loss):
            raise ValueError("train_loss must be a scalar")
        eps = np.finfo(float).eps
        if abs(lambda_) < eps:
            raise ValueError("lambda_ must not be zero. Make sure that you're not scaling the value of lambda down too "
                             "quickly or passing an initial value of zero to the lambda parameter.")
        if lambda_ < 0:
            raise ValueError("lambda_ must be non-negative")
        if not isinstance(lambda_, float):
            raise ValueError("lambda_ must be a float")
        if train_loss < 0 or val_loss < 0:
            raise ValueError("losses must be non-negative for this updater")
        if train_loss < eps:
            # 0 / 0 leaves lambda alone; x / 0 counts as a ratio above any interval
            return lambda_ if val_loss < eps else lambda_ * (1 + self.scaling_factor)
        ratio = val_loss / train_loss
        if ratio > self.tolerable_interval[1]:
            lambda_ *= 1 + self.scaling_factor
        elif ratio < self.tolerable_interval[0]:
            lambda_ *= 1 - self.scaling_factor
        return lambda_
