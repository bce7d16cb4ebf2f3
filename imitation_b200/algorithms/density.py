"""Density-based reward learning (mirror of imitation.algorithms.density:24-413).

`DensityAlgorithm` fits a kernel density estimate of p(s), p(s, a) or p(s, s') on the demonstrations and rewards the
agent with its log.  The reference fits sklearn's `KernelDensity` and scores every transition with its own
`KernelDensity.score` call, in a Python loop, at every env step.  Here `train()` fits on the host in float64 (the
`StandardScaler` semantics, and sklearn's kernel normalisation constants restated by `log_kernel_norm`) and uploads the
standardised demonstration rows once; every score is then one launch of `imb_density_score` (csrc/imb_density.cu).  In
training, the rollout's reward column is overwritten by one such launch from the transition rows the rollout writes
(`RewardVecEnvWrapper.resolve` -> `reward_wrapper.DensityRelabel`, whose `finish` runs after the rollout).

Two deliberate differences from the reference:
- The device evaluates the exact estimator.  sklearn's tree evaluation with its defaults (atol = rtol = 0) is not
  exact for low-density queries: its gaussian and exponential values can differ from the exact ones well beyond
  rounding, and for the compact kernels (tophat, epanechnikov, linear) it returns finite values near -32 to -37 where
  no demonstration row lies within the bandwidth and the exact value is -inf.  Rewards of such queries therefore
  differ from the reference's (DESIGN.md section 7a).
- In a rollout, a non-stationary model scores step t of an episode with the model of episode step t; the reference's
  `RewardVecEnvWrapper` passes no steps, so its non-stationary models cannot train an agent at all.

sklearn's cosine normalisation series is reproduced as it is, including its NaN at D = 4 (the reference's rewards are
NaN there too).  sklearn is not imported: it is a test dependency only.
"""
import dataclasses
import enum
import itertools
import math
from collections.abc import Mapping
from typing import Any, Dict, Iterable, List, Optional

import numpy as np
import torch as th

from .. import _lib, spaces
from ..data import rollout, types, wrappers
from ..rewards import reward_wrapper
from . import base


class DensityType(enum.Enum):
    """Input type the density model should use."""

    STATE_DENSITY = enum.auto()
    """Density on state s."""

    STATE_ACTION_DENSITY = enum.auto()
    """Density on (s,a) pairs."""

    STATE_STATE_DENSITY = enum.auto()
    """Density on (s,s') pairs."""


def log_kernel_norm(h: float, d: int, kernel: str) -> float:
    """sklearn's log normalisation of the kernel of bandwidth h in d dimensions (neighbors/_binary_tree.pxi.tp,
    `_log_kernel_norm`), formula for formula.  The cosine series gives a negative sum at some d (d = 4 among them), and
    so NaN, exactly as sklearn does."""
    def log_vn(n):
        return 0.5 * n * math.log(math.pi) - math.lgamma(0.5 * n + 1)

    def log_sn(n):
        return math.log(2 * math.pi) + log_vn(n - 1)

    if kernel == "gaussian":
        factor = 0.5 * d * math.log(2 * math.pi)
    elif kernel == "tophat":
        factor = log_vn(d)
    elif kernel == "epanechnikov":
        factor = log_vn(d) + math.log(2.0 / (d + 2.0))
    elif kernel == "exponential":
        factor = log_sn(d - 1) + math.lgamma(d)
    elif kernel == "linear":
        factor = log_vn(d) - math.log(d + 1.0)
    elif kernel == "cosine":
        factor, tmp = 0.0, 2.0 / math.pi
        for k in range(1, d + 1, 2):
            factor += tmp
            tmp *= -(d - k) * (d - k - 1) * (2.0 / math.pi) ** 2
        factor = (math.log(factor) if factor > 0 else math.nan) + log_sn(d - 1)
    else:
        raise ValueError(f"Kernel code not recognized: {kernel!r}")
    return -factor - d * math.log(h)


class StandardScaler:
    """sklearn.preprocessing.StandardScaler(with_mean=with_std=standardise) as the reference fits it: mean, population
    standard deviation, and a scale of 1 for (near-)constant features; identity when not standardising."""

    def __init__(self, data: np.ndarray, standardise: bool):
        data = np.asarray(data, dtype=np.float64)
        n = len(data)
        self.mean_ = data.mean(axis=0) if standardise else np.zeros(data.shape[1])
        self.scale_ = np.ones(data.shape[1])
        if standardise:
            var = data.var(axis=0)
            eps = np.finfo(np.float64).eps
            constant = var <= n * eps * var + (n * self.mean_ * eps) ** 2  # sklearn's _is_constant_feature
            self.scale_ = np.where(constant, 1.0, np.sqrt(var))

    def transform(self, x: np.ndarray) -> np.ndarray:
        return (np.asarray(x, dtype=np.float64) - self.mean_) / self.scale_


@dataclasses.dataclass
class DeviceDensity:
    """The fitted model as imb_density_score reads it (include/imb.h): the feature columns of a transition-table row,
    the kernel, and the standardised demonstration rows of every segment in tiles of DENSITY_TILE rows."""

    d: int
    col0: int
    n0: int
    col1: int
    n1: int
    kernel: int
    bandwidth: float
    n_seg: int
    n_demo: int
    demo: th.Tensor       # float32 [n_tiles][d][DENSITY_TILE]
    demo_seg: th.Tensor   # int32 [n_tiles * DENSITY_TILE], -1 on padding rows
    seg_off: th.Tensor    # int64 [n_seg + 1]
    seg_const: th.Tensor  # float64 [n_seg]: log kernel normalisation - log N_s
    mean: th.Tensor       # float32 [d]
    scale: th.Tensor      # float32 [d]

    def tensors(self):
        return (self.demo, self.demo_seg, self.seg_off, self.seg_const, self.mean, self.scale)


def _first_and_rest(iterable):
    iterator = iter(iterable)
    try:
        first = next(iterator)
    except StopIteration:
        raise ValueError(f"iterable {iterable} had no elements to iterate over.")
    return first, (itertools.chain([first], iterator) if iterator is iterable else iterable)


class DensityAlgorithm(base.DemonstrationAlgorithm):
    """Learns a reward function based on density modeling: a kernel density estimate of p(s), p(s,a) or p(s,s'), and
    the reward log p.  `rl_algo` is a `DevicePPO` on a `DeviceVecEnv`."""

    def __init__(self, *, demonstrations, venv, rng: np.random.Generator,
                 density_type: DensityType = DensityType.STATE_ACTION_DENSITY, kernel: str = "gaussian",
                 kernel_bandwidth: float = 0.5, rl_algo=None, is_stationary: bool = True,
                 standardise_inputs: bool = True, custom_logger=None, allow_variable_horizon: bool = False):
        self.is_stationary = is_stationary
        self.density_type = density_type
        self.venv = venv
        self.transitions: Dict[Optional[int], np.ndarray] = dict()
        super().__init__(demonstrations=demonstrations, custom_logger=custom_logger,
                         allow_variable_horizon=allow_variable_horizon)
        self.kernel = kernel
        self.kernel_bandwidth = kernel_bandwidth
        self.standardise = standardise_inputs
        self._scaler: Optional[StandardScaler] = None
        self._model: Optional[DeviceDensity] = None
        self._ws: Optional[th.Tensor] = None  # workspace of __call__, sized for its last query count
        self.rng = rng
        self.rl_algo = rl_algo
        self.buffering_wrapper = wrappers.BufferingWrapper(self.venv)
        self.venv_wrapped = reward_wrapper.RewardVecEnvWrapper(self.buffering_wrapper, self)
        self.wrapper_callback = self.venv_wrapped.make_log_callback()

    # -- features (space_utils.flatten of Box and Discrete) ------------------------------------------------------------
    @staticmethod
    def _flat(space, x: np.ndarray, n: int) -> np.ndarray:
        """[n] space elements -> [n][flat width] float64; Discrete -> one-hot."""
        if isinstance(x, Mapping) or isinstance(space, Mapping):
            raise NotImplementedError("DensityAlgorithm on the GPU path supports Box and Discrete spaces, not Dict "
                                      "observations")
        x = np.asarray(x)
        if spaces.is_discrete(space):
            out = np.zeros((n, int(space.n)))
            out[np.arange(n), x.reshape(n).astype(np.int64) - int(getattr(space, "start", 0))] = 1.0
            return out
        return x.reshape(n, -1).astype(np.float64)

    def _widths(self):
        return spaces.flat_dim(self.venv.observation_space), spaces.flat_dim(self.venv.action_space)

    def _rows(self, obs, acts, next_obs) -> np.ndarray:
        """Transition-table rows [n][obs | act | next_obs | done] (float64; done = 0) of a batch; next_obs may be None
        when the density type does not read it."""
        n = len(obs)
        do, da = self._widths()
        rows = np.zeros((n, 2 * do + da + 1))
        rows[:, :do] = self._flat(self.venv.observation_space, obs, n)
        rows[:, do:do + da] = self._flat(self.venv.action_space, acts, n)
        if next_obs is not None:
            rows[:, do + da:2 * do + da] = self._flat(self.venv.observation_space, next_obs, n)
        return rows

    def _columns(self):
        """(col0, n0, col1, n1): the feature columns of a transition-table row for this density type."""
        do, da = self._widths()
        if self.density_type == DensityType.STATE_DENSITY:
            return 0, do, 0, 0
        if self.density_type == DensityType.STATE_ACTION_DENSITY:
            return 0, do + da, 0, 0
        if self.density_type == DensityType.STATE_STATE_DENSITY:
            return 0, do, do + da, do
        raise ValueError(f"Unknown density type {self.density_type}")

    def _features(self, rows: np.ndarray) -> np.ndarray:
        c0, n0, c1, n1 = self._columns()
        return np.concatenate([rows[:, c0:c0 + n0], rows[:, c1:c1 + n1]], axis=1)

    # -- demonstrations ----------------------------------------------------------------------------------------------
    def _get_demo_from_batch(self, obs_b, act_b, next_obs_b) -> Dict[Optional[int], List[np.ndarray]]:
        if next_obs_b is None and self.density_type == DensityType.STATE_STATE_DENSITY:
            raise ValueError("STATE_STATE_DENSITY requires next_obs_b to be provided, but it was None")
        if isinstance(obs_b, Mapping):
            raise NotImplementedError("DensityAlgorithm on the GPU path does not support Dict observations")
        act_b = np.asarray(act_b)
        obs_b = np.asarray(obs_b)
        assert act_b.shape[1:] == tuple(self.venv.action_space.shape)
        assert obs_b.shape[1:] == tuple(self.venv.observation_space.shape)
        assert len(act_b) == len(obs_b)
        if next_obs_b is not None:
            next_obs_b = np.asarray(next_obs_b)
            assert next_obs_b.shape == obs_b.shape
        return {None: list(self._features(self._rows(obs_b, act_b, next_obs_b)))}

    def set_demonstrations(self, demonstrations) -> None:
        """Sets the demonstration data: trajectories (one group per timestep), Transitions / TransitionsMinimal, or an
        iterable of transition mappings."""
        transitions: Dict[Optional[int], List[np.ndarray]] = {}
        if isinstance(demonstrations, types.TransitionsMinimal):
            transitions.update(self._get_demo_from_batch(demonstrations.obs, demonstrations.acts,
                                                         getattr(demonstrations, "next_obs", None)))
        elif isinstance(demonstrations, Iterable) and not isinstance(demonstrations, (str, bytes)):
            first, demonstrations = _first_and_rest(demonstrations)
            if isinstance(first, types.Trajectory):
                for traj in demonstrations:
                    feats = self._features(self._rows(traj.obs[:-1], traj.acts, traj.obs[1:]))
                    for i, f in enumerate(feats):
                        transitions.setdefault(i, []).append(f)
            elif isinstance(first, Mapping):
                for batch in demonstrations:
                    next_obs = batch.get("next_obs")
                    transitions.update(self._get_demo_from_batch(
                        _numpy(batch["obs"]), _numpy(batch["acts"]), None if next_obs is None else _numpy(next_obs)))
            else:
                raise TypeError(f"Unsupported demonstration type {type(demonstrations)}")
        else:
            raise TypeError(f"Unsupported demonstration type {type(demonstrations)}")

        self.transitions = {k: np.stack(v, axis=0) for k, v in transitions.items()}
        if not self.is_stationary and None in self.transitions:
            raise ValueError("Non-stationary model incompatible with non-trajectory demonstrations.")
        if self.is_stationary:
            self.transitions = {None: np.concatenate(list(self.transitions.values()), axis=0)}

    # -- fit ---------------------------------------------------------------------------------------------------------
    def train(self) -> None:
        """Fits the density model to `self.transitions` on the host (float64) and uploads it once."""
        if isinstance(self.kernel_bandwidth, str):
            raise NotImplementedError(f"bandwidth rule {self.kernel_bandwidth!r} is not supported: pass a float")
        if self.kernel not in _lib.KDE_KERNELS:
            raise ValueError(f"The 'kernel' parameter of KernelDensity must be a str among "
                             f"{sorted(_lib.KDE_KERNELS)}. Got {self.kernel!r} instead.")
        h = float(self.kernel_bandwidth)
        if not (h > 0 and math.isfinite(h)):
            raise ValueError(f"The 'bandwidth' parameter of KernelDensity must be a float in the range (0, inf). Got "
                             f"{self.kernel_bandwidth!r} instead.")
        keys = list(self.transitions)
        if not self.is_stationary:
            keys = sorted(keys)
        data = [np.asarray(self.transitions[k], dtype=np.float64) for k in keys]
        D = data[0].shape[1]
        if D > _lib.DENSITY_MAX_D:
            raise NotImplementedError(f"the density kernel scores at most {_lib.DENSITY_MAX_D} features per transition "
                                      f"(IMB_DENSITY_MAX_D), got {D}")
        self._scaler = StandardScaler(np.concatenate(data, axis=0), self.standardise)
        rows = np.concatenate([self._scaler.transform(v) for v in data], axis=0).astype(np.float32)
        sizes = np.array([len(v) for v in data], dtype=np.int64)
        N, tile = len(rows), _lib.DENSITY_TILE
        n_tiles = -(-N // tile)
        padded = np.zeros((n_tiles * tile, D), np.float32)
        padded[:N] = rows
        seg = np.full(n_tiles * tile, -1, np.int32)
        seg[:N] = np.repeat(np.arange(len(data), dtype=np.int32), sizes)
        norm = log_kernel_norm(h, D, self.kernel)
        dev = _device(self.venv)
        c0, n0, c1, n1 = self._columns()
        self._model = DeviceDensity(
            d=D, col0=c0, n0=n0, col1=c1, n1=n1, kernel=_lib.KDE_KERNELS[self.kernel], bandwidth=h, n_seg=len(data),
            n_demo=N,
            demo=th.from_numpy(np.ascontiguousarray(padded.reshape(n_tiles, tile, D).transpose(0, 2, 1))).to(dev),
            demo_seg=th.from_numpy(seg).to(dev),
            seg_off=th.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to(dev),
            seg_const=th.tensor([norm - math.log(n) for n in sizes], dtype=th.float64).to(dev),
            mean=th.from_numpy(self._scaler.mean_.astype(np.float32)).to(dev),
            scale=th.from_numpy(self._scaler.scale_.astype(np.float32)).to(dev))

    @property
    def device_model(self) -> DeviceDensity:
        if self._model is None:
            raise RuntimeError("DensityAlgorithm: call train() before scoring")
        return self._model

    # -- reward ------------------------------------------------------------------------------------------------------
    def __call__(self, state, action, next_state, done, steps=None) -> np.ndarray:
        r"""Rewards `r_t(s,a,s') = \log \hat p_t(s,a,s')` of a batch of transitions (float32, one per transition):
        one upload, one kernel launch, one read-back."""
        if not self.is_stationary and steps is None:
            raise ValueError("steps must be provided with non-stationary models")
        del done
        assert len(state) == len(action) and len(state) == len(next_state)
        model = self.device_model
        n = len(state)
        if n == 0:
            return np.zeros(0, dtype=np.float32)
        src = self._rows(state, action, next_state).astype(np.float32)
        parts = [src.reshape(-1).view(np.uint8)]
        if not self.is_stationary:
            steps = np.asarray(steps, dtype=np.int64).reshape(n)
            bad = np.flatnonzero((steps < 0) | (steps >= model.n_seg))
            if len(bad):
                raise ValueError(f"Time {steps[bad[0]]} out of range (0, {model.n_seg}], and absorbing states not "
                                 "currently supported")
            order = np.argsort(steps, kind="stable")  # queries sorted by segment: a query tile reads few demo tiles
            pad = (-parts[0].size) % 8
            parts += [np.zeros(pad, np.uint8), order.astype(np.int64).view(np.uint8), steps[order].view(np.uint8)]
        dev = model.demo.device
        buf = th.from_numpy(np.concatenate(parts)).to(dev)
        src_d = buf[:src.nbytes].view(th.float32)
        row_map = seg_steps = None
        if not self.is_stationary:
            o = src.nbytes + pad
            row_map = buf[o:o + 8 * n].view(th.int64)
            seg_steps = buf[o + 8 * n:o + 16 * n].view(th.int64)
        n_ws = _lib.density_ws_floats(n)
        if self._ws is None or self._ws.numel() != n_ws or self._ws.device != dev:
            self._ws = th.zeros(n_ws, device=dev)
        out = th.empty(n, device=dev)
        _lib.density_score(model, src_d, src.shape[1], n, out, 1, self._ws,
                           seg_mode=_lib.DENSITY_SEG_NONE if self.is_stationary else _lib.DENSITY_SEG_STEPS,
                           row_map=row_map, steps=seg_steps)
        return out.cpu().numpy()

    # -- agent -------------------------------------------------------------------------------------------------------
    def train_policy(self, n_timesteps: int = int(1e6), **kwargs: Any) -> None:
        """Train the imitation policy for a given number of timesteps (`rl_algo.learn` on the density reward)."""
        assert self.rl_algo is not None
        self.rl_algo.set_env(self.venv_wrapped)
        self.rl_algo.learn(n_timesteps, reset_num_timesteps=False, callback=self.wrapper_callback, **kwargs)
        trajs, ep_lens = self.buffering_wrapper.pop_trajectories()
        self._check_fixed_horizon(ep_lens)

    def test_policy(self, *, n_trajectories: int = 10, true_reward: bool = True):
        """Roll the current policy out and return `rollout_stats` of the trajectories; with true_reward=False their
        rewards are the density rewards, as the reference's wrapped env gives them."""
        trajs = rollout.generate_trajectories(self.rl_algo, self.venv if true_reward else self.venv_wrapped,
                                              sample_until=rollout.make_min_episodes(n_trajectories), rng=self.rng)
        if not true_reward:
            tr = types.flatten_trajectories(trajs)
            steps = np.concatenate([np.arange(len(t)) for t in trajs])
            rews = self(tr.obs, tr.acts, tr.next_obs, tr.dones, steps)
            bounds = np.cumsum([0] + [len(t) for t in trajs])
            trajs = [dataclasses.replace(t, rews=rews[a:b]) for t, a, b in zip(trajs, bounds[:-1], bounds[1:])]
        self.buffering_wrapper.pop_trajectories()
        self._check_fixed_horizon(len(traj) for traj in trajs)
        return rollout.rollout_stats(trajs)

    @property
    def policy(self):
        assert self.rl_algo is not None
        assert self.rl_algo.policy is not None
        return self.rl_algo.policy


def _numpy(x):
    if isinstance(x, Mapping):
        return x  # Dict observations: refused by _get_demo_from_batch
    return x.detach().cpu().numpy() if isinstance(x, th.Tensor) else np.asarray(x)


def _device(venv) -> th.device:
    while not hasattr(venv, "device") and hasattr(venv, "venv"):
        venv = venv.venv
    return th.device(getattr(venv, "device", "cuda"))
