"""Behavioural cloning (mirror of imitation.algorithms.bc).

`BC` has the reference's constructor, attributes, `train()` and errors (algorithms/bc.py:268-510).  Its training loop
runs on the device: each `train()` is one launch of the PPO update's persistent cluster kernel with the BC loss
(`imb_bc_train`, csrc/imb_ppo_gen.cuh), unless the host has to see the policy in between -- after each batch when
`on_batch_end` is given, at epoch ends when `on_epoch_end` is given, at logged batches when `log_rollouts_venv` is
given.  A train() split over launches computes the same bits as one launch.

The minibatch order is the reference's: every epoch iterates a torch
`DataLoader(range(N), batch_size=minibatch_size, shuffle=True, drop_last=True)` on the host, drawing from the global
torch RNG exactly as the reference's demonstration loader does; the indices are uploaded per launch.  Demonstrations
given as batch mappings keep their order every epoch.

`BehaviorCloningLossCalculator` is torch code over the policy's `evaluate_actions` (the API path; not on the hot path).
"""
import dataclasses
from typing import Any, Callable, Iterable, List, Mapping, Optional, Tuple, Union

import numpy as np
import torch as th
import torch.utils.data as th_data

from .. import _lib
from ..data import rollout, types
from ..policies import base as policy_base
from ..util import logger as imit_logger
from . import base as algo_base

# optimizer_kwargs keys that only choose torch's Adam implementation: accepted, no effect on the arithmetic
_ADAM_IMPL_KWARGS = ("foreach", "fused", "capturable", "differentiable")


@dataclasses.dataclass(frozen=True)
class BCTrainingMetrics:
    """Container for the different components of behavior cloning loss."""

    neglogp: th.Tensor
    entropy: Optional[th.Tensor]
    ent_loss: th.Tensor  # set to 0 if entropy is None
    prob_true_act: th.Tensor
    l2_norm: th.Tensor
    l2_loss: th.Tensor
    loss: th.Tensor


@dataclasses.dataclass(frozen=True)
class BehaviorCloningLossCalculator:
    """Functor to compute the loss used in Behavior Cloning (bc.py:94-156)."""

    ent_weight: float
    l2_weight: float

    def __call__(self, policy, obs, acts) -> BCTrainingMetrics:
        device = next(policy.parameters()).device
        obs = th.as_tensor(np.asarray(obs) if not isinstance(obs, th.Tensor) else obs, device=device)
        acts = th.as_tensor(np.asarray(acts) if not isinstance(acts, th.Tensor) else acts, device=device)
        _, log_prob, entropy = policy.evaluate_actions(obs, acts)
        prob_true_act = th.exp(log_prob).mean()
        log_prob = log_prob.mean()
        entropy = entropy.mean() if entropy is not None else None
        l2_norm = sum(th.sum(th.square(w)) for w in policy.parameters()) / 2
        ent_loss = -self.ent_weight * (entropy if entropy is not None else th.zeros(1))
        neglogp = -log_prob
        l2_loss = self.l2_weight * l2_norm
        loss = neglogp + ent_loss + l2_loss
        return BCTrainingMetrics(neglogp=neglogp, entropy=entropy, ent_loss=ent_loss, prob_true_act=prob_true_act,
                                 l2_norm=l2_norm, l2_loss=l2_loss, loss=loss)


@dataclasses.dataclass(frozen=True)
class RolloutStatsComputer:
    """Rollout statistics of the policy in `venv` (bc.py:170-201), through `data.rollout.generate_trajectories`."""

    venv: Optional[Any]
    n_episodes: int

    def __call__(self, policy, rng: np.random.Generator) -> Mapping[str, float]:
        if self.venv is not None and self.n_episodes > 0:
            trajs = rollout.generate_trajectories(policy, self.venv, rollout.make_min_episodes(self.n_episodes),
                                                  rng=rng)
            # the reference samples through SB3's policy.predict, which leaves the policy in evaluation mode (so later
            # minibatches no longer update a feature RunningNorm)
            policy.set_training_mode(False)
            return rollout.rollout_stats(trajs)
        return dict()


class BCLogger:
    """Utility class to help logging information relevant to Behavior Cloning (bc.py:204-247)."""

    def __init__(self, logger: imit_logger.HierarchicalLogger):
        self._logger = logger
        self._tensorboard_step = 0
        self._current_epoch = 0

    def reset_tensorboard_steps(self):
        self._tensorboard_step = 0

    def log_epoch(self, epoch_number):
        self._current_epoch = epoch_number

    def log_batch(self, batch_num: int, batch_size: int, num_samples_so_far: int, training_metrics: BCTrainingMetrics,
                  rollout_stats: Mapping[str, float]):
        self._logger.record("batch_size", batch_size)
        self._logger.record("bc/epoch", self._current_epoch)
        self._logger.record("bc/batch", batch_num)
        self._logger.record("bc/samples_so_far", num_samples_so_far)
        for k, v in training_metrics.__dict__.items():
            self._logger.record(f"bc/{k}", float(v) if v is not None else None)
        for k, v in rollout_stats.items():
            if "return" in k and "monitor" not in k:
                self._logger.record("rollout/" + k, v)
        self._logger.dump(self._tensorboard_step)
        self._tensorboard_step += 1

    def __getstate__(self):
        state = self.__dict__.copy()
        del state["_logger"]
        return state


def reconstruct_policy(policy_path: str, device: Union[th.device, str] = "auto") -> policy_base.ActorCriticPolicy:
    """Reconstruct a policy saved with `th.save` (bc.py:250-265)."""
    policy = th.load(policy_path, map_location=_device(device), weights_only=False)
    assert isinstance(policy, policy_base.ActorCriticPolicy)
    return policy


def _device(device) -> th.device:
    if isinstance(device, str) and device == "auto":
        return th.device("cuda")
    return th.device(device)


# ---- the sequence of a train() call --------------------------------------------------------------------------------
# Events, in the order the reference runs them (bc.py:447-510 with BatchIteratorWithEpochEndCallback, bc.py:35-77):
#   ("batch", i, batch_num): the optimiser step after minibatch i, then its log record and on_batch_end;
#   ("epoch", i, epoch): the end of an epoch after minibatch i (not after the last one when n_batches ends the call,
#                        islice stops before the generator resumes).
# The incomplete last batch (bc.py:507-510) steps after the loop, so after the last epoch end.

def train_events(n_minibatches: int, per_epoch: int, k: int, by_epochs: bool) -> List[Tuple[str, int, int]]:
    M, ev = n_minibatches, []
    for i in range(M):
        if (i + 1) % k == 0:
            ev.append(("batch", i, i // k))
        if (i + 1) % per_epoch == 0 and (by_epochs or i + 1 < M):
            ev.append(("epoch", i, (i + 1) // per_epoch - 1))
    if M % k:
        ev.append(("batch", M - 1, (M - 1) // k + 1))
    return ev


def plan_launches(n_minibatches: int, per_epoch: int, k: int, by_epochs: bool, log_interval: int, *,
                  on_batch_end: bool, on_epoch_end: bool, log_rollouts: bool) -> List[list]:
    """The launches and host events of one train(), in order: ["launch", j0, n, final_flush] (imb_bc_train's
    arguments) and ["batch" | "epoch", i, number].  A launch ends where the host must see the policy: before a batch
    event when on_batch_end is given, or when log_rollouts and the batch is logged; before an epoch event when
    on_epoch_end is given.  An incomplete last batch that follows such an epoch end steps in a launch of its own."""
    M = n_minibatches
    ev = train_events(M, per_epoch, k, by_epochs)
    sched: List[list] = []
    pending: List[list] = []
    j = 0  # minibatches launched so far
    last_launch: Optional[list] = None
    for idx, (kind, i, num) in enumerate(ev):
        flush = kind == "batch" and M % k != 0 and idx == len(ev) - 1
        host = ((kind == "batch" and (on_batch_end or (log_rollouts and num % log_interval == 0)))
                or (kind == "epoch" and on_epoch_end))
        if flush:
            if j < M:
                last_launch = ["launch", j, M - j, 1]
                sched.append(last_launch)
                j = M
            else:  # every minibatch has run and the host saw the last epoch end: the step has a launch of its own
                last_launch[3] = 2
                sched.append(["launch", M, 0, 1])
            sched += pending + [["batch", i, num]]
            pending = []
        elif host:
            if i + 1 > j:
                last_launch = ["launch", j, i + 1 - j, 0]
                sched.append(last_launch)
                j = i + 1
            sched += pending + [[kind, i, num]]
            pending = []
        else:
            pending.append([kind, i, num])
    if j < M:
        sched.append(["launch", j, M - j, 1])
    return sched + pending


def epoch_permutation(n: int, minibatch_size: int) -> th.Tensor:
    """One epoch's index order of the reference's demonstration loader (algorithms/base.py make_data_loader:
    DataLoader(shuffle=True, drop_last=True)), drawing from the global torch RNG as iterating that loader does."""
    loader = th_data.DataLoader(range(n), batch_size=minibatch_size, shuffle=True, drop_last=True)
    batches = list(loader)
    head = th.cat(batches) if batches else th.zeros(0, dtype=th.int64)
    # the dropped tail is never read; pad the row to n
    return th.cat([head.to(th.int64), th.zeros(n - len(head), dtype=th.int64)])


class BC(algo_base.DemonstrationAlgorithm):
    """Behavioral cloning (BC): a policy recovered by supervised learning from observation-action pairs."""

    def __init__(self, *, observation_space, action_space, rng: np.random.Generator, policy=None, demonstrations=None,
                 batch_size: int = 32, minibatch_size: Optional[int] = None, optimizer_cls=th.optim.Adam,
                 optimizer_kwargs: Optional[Mapping[str, Any]] = None, ent_weight: float = 1e-3,
                 l2_weight: float = 0.0, device: Union[str, th.device] = "auto", custom_logger=None):
        self._demo_table: Optional[th.Tensor] = None
        self._demo_n = 0
        self._shuffle = True
        self.batch_size = batch_size
        self.minibatch_size = minibatch_size or batch_size
        if self.batch_size % self.minibatch_size != 0:
            raise ValueError("Batch size must be a multiple of minibatch size.")
        self.action_space = action_space
        self.observation_space = observation_space
        # every refusal comes before the policy reaches the device
        self.lr, self.adam_eps = adam_hparams(optimizer_cls, optimizer_kwargs)
        if policy is None:
            policy = policy_base.FeedForward32Policy(observation_space=observation_space, action_space=action_space)
        check_policy(policy, self.minibatch_size)
        dev = _device(device)
        if dev.type != "cuda":
            raise NotImplementedError(f"device {device!r}: BC trains on the GPU only")
        self._dev = dev
        self._policy = policy.to(dev)
        super().__init__(demonstrations=demonstrations, custom_logger=custom_logger)
        self._bc_logger = BCLogger(self.logger)
        self.rng = rng
        assert self.policy.observation_space == self.observation_space
        assert self.policy.action_space == self.action_space
        self.loss_calculator = BehaviorCloningLossCalculator(ent_weight, l2_weight)

        n = policy.desc.n_params
        self.exp_avg = th.zeros(n, device=dev)
        self.exp_avg_sq = th.zeros(n, device=dev)
        self._grad_carry = th.zeros(n, device=dev)
        self._state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device=dev)

    @property
    def policy(self) -> policy_base.ActorCriticPolicy:
        return self._policy

    @property
    def adam_steps(self) -> int:
        """Optimiser steps taken so far (torch Adam's `step`)."""
        return int(self._state[_lib.ST_PPO_STEP])

    # -- demonstrations ---------------------------------------------------------------------------------------------
    def set_demonstrations(self, demonstrations) -> None:
        obs, acts, shuffle = self._demo_arrays(demonstrations)
        self._demo_n = len(obs)
        self._shuffle = shuffle
        self._demo_table = self.demo_table(obs, acts).to(self._dev)

    def _set_demonstration_rows(self, table: th.Tensor, n: int, loader_batch_size: int) -> None:
        """Demonstrations from the first n rows of a device table in the kernel's row format, each epoch shuffled as
        the reference's `DataLoader(transitions, loader_batch_size, shuffle=True, drop_last=True)` is (DAgger's
        dataset).  The reference's errors for a loader batch that is not minibatch_size rows and for fewer than
        minibatch_size rows."""
        if loader_batch_size != self.minibatch_size:
            raise ValueError(f"Expected batch size {self.minibatch_size} != {loader_batch_size} = len(batch['obs'])")
        if n < self.minibatch_size:
            raise ValueError(f"Number of transitions in `demonstrations` {n} is smaller than batch size "
                             f"{self.minibatch_size}.")
        if not table.is_cuda or table.shape[1] != _lib.rollout_row_width(self.policy.desc):
            raise ValueError("the demonstration table must be a device table in the kernel's row format")
        self._demo_table = table
        self._demo_n = n
        self._shuffle = True

    def _demo_arrays(self, demonstrations) -> Tuple[np.ndarray, np.ndarray, bool]:
        return demonstration_arrays(demonstrations, self.minibatch_size)

    def demo_table(self, obs, acts) -> th.Tensor:
        return demo_table(self.policy, obs, acts)

    # -- training ---------------------------------------------------------------------------------------------------
    def train(self, *, n_epochs: Optional[int] = None, n_batches: Optional[int] = None,
              on_epoch_end: Optional[Callable[[], None]] = None, on_batch_end: Optional[Callable[[], None]] = None,
              log_interval: int = 500, log_rollouts_venv=None, log_rollouts_n_episodes: int = 5,
              progress_bar: bool = True, reset_tensorboard: bool = False):
        """Train with supervised learning for n_epochs passes over the demonstrations or n_batches optimiser batches
        (bc.py:381-510).  `progress_bar` is accepted and shows nothing: the loop runs inside one kernel launch."""
        if reset_tensorboard:
            self._bc_logger.reset_tensorboard_steps()
        self._bc_logger.log_epoch(0)
        compute_rollout_stats = RolloutStatsComputer(log_rollouts_venv, log_rollouts_n_episodes)
        check_epochs_batches(n_epochs, n_batches)
        assert self._demo_table is not None
        mb, k, N = self.minibatch_size, self.batch_size // self.minibatch_size, self._demo_n
        per_epoch = N // mb
        M = n_epochs * per_epoch if n_epochs is not None else n_batches * k
        if M <= 0:
            return
        sched = plan_launches(M, per_epoch, k, n_epochs is not None, log_interval, on_batch_end=on_batch_end is not None,
                              on_epoch_end=on_epoch_end is not None,
                              log_rollouts=log_rollouts_venv is not None and log_rollouts_n_episodes > 0)
        pol = self.policy
        params, norm, norm_count = pol.flat_vectors()
        perms: List[th.Tensor] = []  # this call's epoch permutations, drawn when first needed
        rows: List[np.ndarray] = []  # metrics rows read back, consumed by the logged batches in order
        lc = self.loss_calculator
        for item in sched:
            if item[0] == "launch":
                _, j0, n, final_flush = item
                perm = None
                if n > 0:
                    e0, e1 = j0 // per_epoch, (j0 + n - 1) // per_epoch
                    while len(perms) <= e1:
                        perms.append(epoch_permutation(N, mb) if self._shuffle else th.arange(N, dtype=th.int64))
                        if perms[-1].shape != (N,):
                            raise ValueError(f"an epoch permutation must have {N} entries, got {tuple(perms[-1].shape)}")
                    perm = th.stack(perms[e0:e1 + 1]).to(self._dev)
                n_log = self._logged_in_launch(j0, n, final_flush, M, k, log_interval)
                metrics = th.empty(max(n_log, 1), _lib.BC_METRIC_FLOATS, device=self._dev) if n_log else None
                _lib.bc_train(pol.desc, params, norm if pol.normalize_features else None,
                              norm_count if pol.normalize_features else None, self.exp_avg, self.exp_avg_sq,
                              self._demo_table, N, mb, self.batch_size, j0, n, final_flush, lc.l2_weight,
                              lc.ent_weight, self.lr, self.adam_eps, pol.training, perm,
                              self._grad_carry if k > 1 else None, metrics, log_interval, self._state, act=pol.act)
                if metrics is not None:
                    rows += list(metrics[:n_log].cpu().numpy())
            elif item[0] == "batch":
                _, i, batch_num = item
                if batch_num % log_interval == 0:
                    row = rows.pop(0)
                    assert int(row[7]) == batch_num
                    m = BCTrainingMetrics(**{name: th.tensor(float(row[c])) for c, name in enumerate(_lib.BC_METRICS)})
                    self._bc_logger.log_batch(batch_num, mb, (i + 1) * mb, m, compute_rollout_stats(pol, self.rng))
                if on_batch_end is not None:
                    on_batch_end()
            else:
                self._bc_logger.log_epoch(item[2] + 1)
                if on_epoch_end is not None:
                    on_epoch_end()

    @staticmethod
    def _logged_in_launch(j0: int, n: int, final_flush: int, M: int, k: int, log_interval: int) -> int:
        """Metrics rows imb_bc_train writes for this launch: its complete batches whose number is a multiple of
        log_interval, and the call's incomplete last batch when it ends here (final_flush 1 or 2)."""
        c = sum(1 for i in range(j0, j0 + n) if (i + 1) % k == 0 and (i // k) % log_interval == 0)
        if n > 0 and final_flush and j0 + n == M and M % k and ((M - 1) // k + 1) % log_interval == 0:
            c += 1
        return c


def adam_hparams(optimizer_cls, optimizer_kwargs) -> Tuple[float, float]:
    """(lr, eps) of the torch Adam BC would build, refusing what the kernel does not run (bc.py:360-367)."""
    if optimizer_kwargs:
        if "weight_decay" in optimizer_kwargs:
            raise ValueError("Use the parameter l2_weight instead of weight_decay.")
    optimizer_kwargs = dict(optimizer_kwargs or {})
    if optimizer_cls is not th.optim.Adam:
        raise NotImplementedError(f"optimizer_cls {optimizer_cls!r}: the BC update kernel runs Adam")
    if "betas" in optimizer_kwargs and tuple(float(b) for b in optimizer_kwargs["betas"]) != (0.9, 0.999):
        raise NotImplementedError(f"betas {optimizer_kwargs['betas']!r}: the BC update kernel runs Adam with betas "
                                  "(0.9, 0.999)")
    for opt in ("amsgrad", "maximize"):
        if optimizer_kwargs.get(opt, False):
            raise NotImplementedError(f"{opt}=True: the BC update kernel runs plain Adam")
    unknown = set(optimizer_kwargs) - {"lr", "eps", "betas", "amsgrad", "maximize", *_ADAM_IMPL_KWARGS}
    if unknown:
        raise TypeError(f"Adam got unexpected keyword arguments {sorted(unknown)}")
    return float(optimizer_kwargs.get("lr", 1e-3)), float(optimizer_kwargs.get("eps", 1e-8))


def check_policy(policy, minibatch_size: int) -> None:
    """NotImplementedError unless the BC kernel can train `policy` at minibatch_size (host only)."""
    if not isinstance(policy, policy_base.ActorCriticPolicy):
        raise NotImplementedError(f"policy {type(policy).__name__}: BC trains this package's ActorCriticPolicy "
                                  "(two tanh or ReLU towers of one width <= 64, Box or Discrete actions)")
    try:
        _lib.bc_plan(policy.desc, minibatch_size, policy.act)
    except _lib.ImbError as e:
        raise NotImplementedError(f"minibatch_size {minibatch_size} with this policy: {e}") from None


def check_epochs_batches(n_epochs, n_batches) -> None:
    if (n_epochs is None) == (n_batches is None):  # BatchIteratorWithEpochEndCallback.__post_init__ (bc.py:47-57)
        raise ValueError("Must provide exactly one of `n_epochs` and `n_batches` arguments.")


def demonstration_arrays(demonstrations, minibatch_size: int) -> Tuple[np.ndarray, np.ndarray, bool]:
    """(obs, acts, shuffled) of the forms algorithms/base.py make_data_loader accepts: Transitions(Minimal), a
    sequence of trajectories (flattened), or an iterable of batch mappings of minibatch_size rows each (kept in their
    order every epoch; iterated once, here).  The reference's errors."""
    mb = minibatch_size
    if isinstance(demonstrations, Iterable) and not isinstance(demonstrations, (types.TransitionsMinimal, Mapping)):
        items = list(demonstrations)
        if items and isinstance(items[0], types.Trajectory):
            demonstrations = types.flatten_trajectories(items)
        else:
            for batch in items:
                for key in ("obs", "acts"):
                    if len(batch[key]) != mb:
                        raise ValueError(f"Expected batch size {mb} != {len(batch[key])} = len(batch['{key}'])")
            if not items:
                raise ValueError("`demonstrations` has no batches")
            return (np.concatenate([np.asarray(b["obs"]) for b in items]),
                    np.concatenate([np.asarray(b["acts"]) for b in items]), False)
    if isinstance(demonstrations, types.TransitionsMinimal):
        if len(demonstrations) < mb:
            raise ValueError(f"Number of transitions in `demonstrations` {len(demonstrations)} is smaller than "
                             f"batch size {mb}.")
        return np.asarray(demonstrations.obs), np.asarray(demonstrations.acts), True
    raise TypeError(f"`demonstrations` unexpected type {type(demonstrations)}")


def demo_table(pol, obs, acts) -> th.Tensor:
    """The demonstration rows in the rollout-table format the kernel reads: obs | act (Discrete: the index), the
    remaining columns zero.  CPU tensor."""
    n = len(obs)
    obs = th.as_tensor(np.array(obs, dtype=np.float32)).reshape(n, -1)
    if obs.shape[1] != pol.d_obs:
        raise ValueError(f"observations have {obs.shape[1]} features, the policy takes {pol.d_obs}")
    da = 1 if pol.discrete else pol.d_act
    acts = th.as_tensor(np.array(acts, dtype=np.float32)).reshape(n, -1)
    if acts.shape[1] != da:
        raise ValueError(f"actions have {acts.shape[1]} columns, the policy takes {da}")
    table = th.zeros(n, _lib.rollout_row_width(pol.desc), dtype=th.float32)
    table[:, :pol.d_obs] = obs
    table[:, pol.d_obs:pol.d_obs + da] = acts
    return table
