"""Regularization of a network's training step: regularizers and the rules that adapt their strength."""
from .regularizers import (LossRegularizer, LpRegularizer, Regularizer, RegularizerFactory, WeightDecayRegularizer,
                           WeightRegularizer)
from .updaters import IntervalParamScaler, LambdaUpdater

__all__ = ["RegularizerFactory", "Regularizer", "LossRegularizer", "WeightRegularizer", "LpRegularizer",
           "WeightDecayRegularizer", "LambdaUpdater", "IntervalParamScaler"]
