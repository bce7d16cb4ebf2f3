"""Reward learning from preference comparisons (SURVEY section 8f, row f1) on the fused reward networks.

Mirror of the reward-model side of imitation.algorithms.preference_comparisons: `RandomFragmenter` (:564-665),
`SyntheticGatherer` (:821-906), `PreferenceDataset` (:909-997), `PreferenceModel` (:345-530),
`CrossEntropyRewardLoss` (:1043-1090), `BasicRewardTrainer` (:1139-1323), `EnsembleTrainer` (:1326-1438) and the
`PreferenceComparisons` loop (:1482-1700) driven by a `TrajectoryDataset` (:99-124).  Same names, arguments, errors
and random-number consumption (fragment choice, bagging sampler, DataLoader shuffling), so preference datasets and
minibatch orders are identical to the reference's for the same seeds.

What is different is where the arithmetic runs.  The reference evaluates the reward network once per fragment in a
Python loop (`PreferenceModel.forward`, :441-454: 2 x pairs x members small forward passes per minibatch); here the
2 x P fragments of a minibatch are flattened into ONE batch of 2*P*L transition rows, pushed through the fused MLP
kernels (`reward_nets._FusedForward`: forward = imb_reward_forward, backward = imb_disc_fwd_bwd with the upstream
gradient of every row), and the segmented discounted return -> clipped Boltzmann probability -> BCE is a handful
of tensor ops on [P, L] device arrays.  Online RL on the learned reward (`AgentTrainer`) is out of scope of this
row (the GAIL/AIRL generator is the on-device RL path); pass a `TrajectoryDataset`.
"""
import abc
import math
import pickle
from collections import defaultdict
from typing import Any, Callable, Dict, List, Mapping, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np
import torch as th
from torch import nn
from torch.utils import data as data_th

from .. import _desc, _lib, spaces
from . import base
from ..data import rollout, types, wrappers
from ..data.types import TrajectoryWithRew
from ..regularization import regularizers
from ..rewards import reward_nets
from ..util import logger as imit_logger
from ..util.flat import views

TrajectoryWithRewPair = Tuple[TrajectoryWithRew, TrajectoryWithRew]


def make_seeds(rng: np.random.Generator, n: Optional[int] = None):
    """util/util.py:181-199."""
    seeds = rng.integers(0, (1 << 31) - 1, (n if n is not None else 1,)).tolist()
    return seeds[0] if n is None else seeds


# ------------------------------------------------------------------------------------------------
# trajectory sources
# ------------------------------------------------------------------------------------------------
class TrajectoryGenerator(abc.ABC):
    def __init__(self, custom_logger: Optional[imit_logger.HierarchicalLogger] = None):
        self.logger = custom_logger or imit_logger.configure()

    @abc.abstractmethod
    def sample(self, steps: int) -> Sequence[TrajectoryWithRew]:
        """Sample trajectories with at least `steps` transitions in total."""

    def train(self, steps: int, **kwargs: Any) -> None:
        """Train the agent, if any (no-op for fixed datasets)."""


def _get_trajectories(trajectories: Sequence[TrajectoryWithRew], steps: int) -> Sequence[TrajectoryWithRew]:
    """Prefix of `trajectories` with at least `steps` transitions (:319-342)."""
    if steps == 0:
        return []
    available = sum(len(t) for t in trajectories)
    if available < steps:
        raise RuntimeError(f"Asked for {steps} transitions but only {available} available")
    total, out = 0, []
    for t in trajectories:
        out.append(t)
        total += len(t)
        if total >= steps:
            break
    return out


class TrajectoryDataset(TrajectoryGenerator):
    """A fixed set of trajectories, shuffled at every `sample` (:99-124)."""

    def __init__(self, trajectories: Sequence[TrajectoryWithRew], rng: np.random.Generator,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None):
        super().__init__(custom_logger=custom_logger)
        self._trajectories = trajectories
        self.rng = rng

    def sample(self, steps: int) -> Sequence[TrajectoryWithRew]:
        trajectories = list(self._trajectories)
        self.rng.shuffle(trajectories)  # type: ignore[arg-type]
        return _get_trajectories(trajectories, steps)


def split_steps(steps: int, exploration_frac: float, logger=None) -> Tuple[int, int]:
    """(agent_steps, exploration_steps) of AgentTrainer.sample(steps) (:247-254), warning like the reference when a
    positive exploration_frac rounds to no exploration steps."""
    exploration_steps = int(exploration_frac * steps)
    if exploration_frac > 0 and exploration_steps == 0 and logger is not None:
        logger.warn(f"No exploration steps included: exploration_frac = {exploration_frac} > 0 but steps={steps} is "
                    "too small.")
    return steps - exploration_steps, exploration_steps


def exploration_plan(wrapper, rng: np.random.Generator, exploration_steps: int, num_envs: int, horizon: int):
    """The host side of the exploration rollout, with the reference's random-number consumption: on the lock-step
    fixed-horizon env, generate_trajectories' unbiased stop rule (data/rollout.py:382-506) rolls k = ceil(
    exploration_steps / (E H)) batches of E whole episodes, i.e. k H calls of the wrapper, then shuffles the k E
    trajectories with `rng` (the order is discarded: the BufferingWrapper's are used).  -> (k, the wrapper's policy of
    each of the k H steps)."""
    k = -(-exploration_steps // (num_envs * horizon))
    policy_steps = wrapper.advance(k * horizon)
    rng.shuffle(list(range(k * num_envs)))
    return k, policy_steps


class AgentTrainer(TrajectoryGenerator):
    """Train the device generator on a learned reward and hand its trajectories (with the ENVIRONMENT's rewards) to the
    preference pipeline (:127-316).  `algorithm` is a `DevicePPO` over a `DeviceVecEnv`; the learned reward is fused into
    the rollout kernel through `RewardVecEnvWrapper`, the `BufferingWrapper` records the ground-truth rewards."""

    def __init__(self, algorithm, reward_fn, venv, rng: np.random.Generator, exploration_frac: float = 0.0,
                 switch_prob: float = 0.5, random_prob: float = 0.5,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        from ..rewards import reward_wrapper

        self.algorithm = algorithm
        super().__init__(custom_logger)
        if isinstance(reward_fn, reward_nets.RewardNet):
            reward_fn = reward_fn.predict_processed
        self.reward_fn = reward_fn
        self.exploration_frac = exploration_frac
        self.rng = rng
        self.buffering_wrapper = wrappers.BufferingWrapper(venv)
        self.venv = self.reward_venv_wrapper = reward_wrapper.RewardVecEnvWrapper(self.buffering_wrapper,
                                                                                  reward_fn=self.reward_fn)
        self.log_callback = self.reward_venv_wrapper.make_log_callback()
        self.algorithm.set_env(self.venv)
        self.algorithm.set_logger(self.logger)
        self.exploration_wrapper = None
        if exploration_frac > 0:
            from ..policies import exploration_wrapper

            # (the reference builds it for any exploration_frac, drawing from rng twice; this one only when it is used)
            self.exploration_wrapper = exploration_wrapper.ExplorationWrapper(
                policy=self.algorithm, venv=self.algorithm.get_env(), random_prob=random_prob, switch_prob=switch_prob,
                rng=self.rng)

    def train(self, steps: int, **kwargs) -> None:
        n_transitions = self.buffering_wrapper.n_transitions
        if n_transitions:
            raise RuntimeError(f"There are {n_transitions} transitions left in the buffer. "
                               "Call AgentTrainer.sample() first to clear them.")
        self.algorithm.learn(total_timesteps=steps, reset_num_timesteps=False, callback=self.log_callback, **kwargs)

    def sample(self, steps: int) -> Sequence[TrajectoryWithRew]:
        agent_trajs, _ = self.buffering_wrapper.pop_finished_trajectories()
        agent_trajs = agent_trajs[::-1]  # the latest trajectories come from the most relevant version of the agent
        avail_steps = sum(len(t) for t in agent_trajs)
        agent_steps, exploration_steps = split_steps(steps, self.exploration_frac, self.logger)
        if avail_steps < agent_steps:
            self.logger.log(f"Requested {agent_steps} transitions but only {avail_steps} in buffer. "
                            f"Sampling {agent_steps - avail_steps} additional transitions.")
            # roll the (stochastic) policy without training until enough episodes have finished; the wrapper records them
            per = self.buffering_wrapper.num_envs * self.algorithm.n_steps
            H = self.buffering_wrapper.venv.horizon
            guard = 0
            more: List[TrajectoryWithRew] = []
            while sum(len(t) for t in more) < agent_steps - avail_steps:
                self.buffering_wrapper.before_rollout()
                self.algorithm.collect_rollouts()
                new, _ = self.buffering_wrapper.pop_finished_trajectories()
                more += list(new)
                guard += per
                if guard > 4 * (agent_steps + H * self.buffering_wrapper.num_envs) + per:
                    raise RuntimeError("could not collect enough finished trajectories")
            agent_trajs = list(agent_trajs) + more
        trajectories = list(_get_trajectories(agent_trajs, agent_steps))
        if exploration_steps > 0:
            self.logger.log(f"Sampling {exploration_steps} exploratory transitions.")
            trajectories.extend(_get_trajectories(self._exploration_trajectories(exploration_steps), exploration_steps))
        return trajectories

    def _exploration_trajectories(self, exploration_steps: int) -> List[TrajectoryWithRew]:
        """generate_trajectories(exploration_wrapper, venv, make_sample_until(min_timesteps=exploration_steps), rng) and
        the BufferingWrapper's finished trajectories afterwards (:283-301): from venv.reset(), which drops the running
        episodes, whole episodes of the E lock-step envs until they hold exploration_steps transitions, as ONE rollout
        launch with the learned reward relabelled (advancing its output normalisers) -- in completion order, with the
        environment's rewards.  The policy acts in eval mode and num_timesteps does not move (SB3's predict)."""
        bw = self.buffering_wrapper
        E, H = bw.num_envs, bw.venv.horizon
        step0 = self.exploration_wrapper.steps_taken
        k, policy_steps = exploration_plan(self.exploration_wrapper, self.rng, exploration_steps, E, H)
        self.venv.reset()  # RewardVecEnvWrapper -> BufferingWrapper.reset -> DeviceVecEnv.reset
        bw.discard()       # the running episodes' steps go with the reset (data/wrappers.py:45-61)
        flat, rews = self.algorithm.exploration_rollout(policy_steps, self.exploration_wrapper.seed, step0,
                                                        self.exploration_wrapper.deterministic_policy)
        flat, rews = flat.cpu().numpy(), rews.cpu().numpy()
        out: List[TrajectoryWithRew] = []
        for j in range(k):  # episode batch j: rows [j E H, (j + 1) E H), env-major
            out += wrappers.finished_trajectories(bw.venv, flat[j * E * H:(j + 1) * E * H],
                                                  rews[:, j * H:(j + 1) * H].reshape(-1))
        return out

    @property
    def logger(self) -> imit_logger.HierarchicalLogger:
        return self._logger

    @logger.setter
    def logger(self, value: imit_logger.HierarchicalLogger) -> None:
        self._logger = value
        self.algorithm.set_logger(value)


# ------------------------------------------------------------------------------------------------
# fragments and synthetic preferences (host side, NumPy: identical random streams to the reference)
# ------------------------------------------------------------------------------------------------
class Fragmenter(abc.ABC):
    def __init__(self, custom_logger: Optional[imit_logger.HierarchicalLogger] = None):
        self.logger = custom_logger or imit_logger.configure()

    @abc.abstractmethod
    def __call__(self, trajectories: Sequence[TrajectoryWithRew], fragment_length: int, num_pairs: int
                 ) -> Sequence[TrajectoryWithRewPair]:
        """Create fragment pairs out of a sequence of trajectories."""


class RandomFragmenter(Fragmenter):
    """Uniformly random fragments, trajectories weighted by length, with replacement (:564-665)."""

    def __init__(self, rng: np.random.Generator, warning_threshold: int = 10,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        super().__init__(custom_logger)
        self.rng = rng
        self.warning_threshold = warning_threshold

    def __call__(self, trajectories, fragment_length: int, num_pairs: int) -> Sequence[TrajectoryWithRewPair]:
        n_before = len(trajectories)
        trajectories = [t for t in trajectories if len(t) >= fragment_length]
        if len(trajectories) == 0:
            raise ValueError(f"No trajectories are long enough for the desired fragment length of {fragment_length}.")
        if n_before != len(trajectories):
            self.logger.log(f"Discarded {n_before - len(trajectories)} out of {n_before} trajectories because they "
                            f"are shorter than the desired length of {fragment_length}.")
        weights = [len(t) for t in trajectories]
        num_transitions = 2 * num_pairs * fragment_length
        if sum(weights) < num_transitions:
            self.logger.warn("Fewer transitions available than needed for desired number of fragment pairs. "
                             "Some transitions will appear multiple times.")
        elif self.warning_threshold and sum(weights) < self.warning_threshold * num_transitions:
            self.logger.warn(f"Samples will contain {num_transitions} transitions in total and only {sum(weights)} are "
                             "available. Because we sample with replacement, a significant number of transitions are "
                             "likely to appear multiple times.")
        p = np.array(weights) / sum(weights)
        fragments: List[TrajectoryWithRew] = []
        for _ in range(2 * num_pairs):  # two fragments per comparison; same draws as the reference (:645-650)
            traj = self.rng.choice(trajectories, p=p)  # type: ignore[arg-type]
            n = len(traj)
            start = self.rng.integers(0, n - fragment_length, endpoint=True)
            end = start + fragment_length
            fragments.append(TrajectoryWithRew(obs=traj.obs[start:end + 1], acts=traj.acts[start:end],
                                               infos=traj.infos[start:end] if traj.infos is not None else None,
                                               rews=traj.rews[start:end], terminal=(end == n) and traj.terminal))
        it = iter(fragments)
        return list(zip(it, it))


class PreferenceGatherer(abc.ABC):
    def __init__(self, rng: Optional[np.random.Generator] = None,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        del rng
        self.logger = custom_logger or imit_logger.configure()

    @abc.abstractmethod
    def __call__(self, fragment_pairs: Sequence[TrajectoryWithRewPair]) -> np.ndarray:
        """Probability that fragment 1 is preferred, one float32 per pair."""


class SyntheticGatherer(PreferenceGatherer):
    """Preferences from the ground-truth rewards of the fragments (:821-906)."""

    def __init__(self, temperature: float = 1, discount_factor: float = 1, sample: bool = True,
                 rng: Optional[np.random.Generator] = None, threshold: float = 50,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        super().__init__(custom_logger=custom_logger)
        self.temperature, self.discount_factor, self.sample = temperature, discount_factor, sample
        self.rng, self.threshold = rng, threshold
        if self.sample and self.rng is None:
            raise ValueError("If `sample` is True, then `rng` must be provided.")

    def __call__(self, fragment_pairs: Sequence[TrajectoryWithRewPair]) -> np.ndarray:
        returns1, returns2 = self._reward_sums(fragment_pairs)
        if self.temperature == 0:
            return (np.sign(returns1 - returns2) + 1) / 2
        returns1 /= self.temperature
        returns2 /= self.temperature
        returns_diff = np.clip(returns2 - returns1, -self.threshold, self.threshold)
        model_probs = 1 / (1 + np.exp(returns_diff))
        with np.errstate(divide="ignore", invalid="ignore"):
            xlogx = lambda q: np.where(q > 0, q * np.log(np.where(q > 0, q, 1.0)), 0.0)  # scipy.special.xlogy(q, q)
            entropy = -(xlogx(model_probs) + xlogx(1 - model_probs)).mean()
        self.logger.record("entropy", entropy)
        if self.sample:
            assert self.rng is not None
            return self.rng.binomial(n=1, p=model_probs).astype(np.float32)
        return model_probs

    def _reward_sums(self, fragment_pairs) -> Tuple[np.ndarray, np.ndarray]:
        r1, r2 = zip(*[(rollout.discounted_sum(f1.rews, self.discount_factor),
                        rollout.discounted_sum(f2.rews, self.discount_factor)) for f1, f2 in fragment_pairs])
        return np.array(r1, dtype=np.float32), np.array(r2, dtype=np.float32)


class PreferenceDataset(data_th.Dataset):
    """Fragment pairs + preference probabilities, optionally a FIFO of `max_size` (:909-997)."""

    def __init__(self, max_size: Optional[int] = None) -> None:
        self.fragments1: List[TrajectoryWithRew] = []
        self.fragments2: List[TrajectoryWithRew] = []
        self.max_size = max_size
        self.preferences: np.ndarray = np.array([])

    def push(self, fragments: Sequence[TrajectoryWithRewPair], preferences: np.ndarray) -> None:
        fragments1, fragments2 = zip(*fragments)
        if preferences.shape != (len(fragments),):
            raise ValueError(f"Unexpected preferences shape {preferences.shape}, expected {(len(fragments),)}")
        if preferences.dtype != np.float32:
            raise ValueError("preferences should have dtype float32")
        self.fragments1.extend(fragments1)
        self.fragments2.extend(fragments2)
        self.preferences = np.concatenate((self.preferences, preferences))
        if self.max_size is not None:
            extra = len(self.preferences) - self.max_size
            if extra > 0:
                self.fragments1, self.fragments2 = self.fragments1[extra:], self.fragments2[extra:]
                self.preferences = self.preferences[extra:]

    def __getitem__(self, key):
        return (self.fragments1[key], self.fragments2[key]), self.preferences[key]

    def __len__(self) -> int:
        assert len(self.fragments1) == len(self.fragments2) == len(self.preferences)
        return len(self.fragments1)

    def save(self, path) -> None:
        with open(path, "wb") as f:
            pickle.dump(self, f)

    @staticmethod
    def load(path) -> "PreferenceDataset":
        with open(path, "rb") as f:
            return pickle.load(f)


def preference_collate_fn(batch):
    fragment_pairs, preferences = zip(*batch)
    return list(fragment_pairs), np.array(preferences)


# ------------------------------------------------------------------------------------------------
# preference model and loss (device side)
# ------------------------------------------------------------------------------------------------
def get_base_model(reward_model: reward_nets.RewardNet) -> reward_nets.RewardNet:
    base = reward_model
    while hasattr(base, "base"):
        base = base.base
    return base


def _stack_fragments(frags: Sequence[TrajectoryWithRew]) -> Mapping[str, np.ndarray]:
    """Transition arrays of equal-length fragments, fragment-major: row f * L + t (what flatten_trajectories gives
    for each fragment, concatenated)."""
    L = len(frags[0])
    obs = np.stack([f.obs for f in frags])           # [F, L + 1, ...]
    acts = np.stack([f.acts for f in frags])         # [F, L, ...]
    dones = np.zeros((len(frags), L), dtype=bool)
    dones[:, -1] = [f.terminal for f in frags]
    flat = lambda a: a.reshape((a.shape[0] * a.shape[1],) + a.shape[2:])
    return dict(obs=flat(obs[:, :-1]), acts=flat(acts), next_obs=flat(obs[:, 1:]), dones=flat(dones))


class FragmentPool:
    """Device-resident transitions of every fragment a preference model has seen: fragment slot k owns rows
    [k * L, (k + 1) * L) of an AoS table [obs | act (one-hot for Discrete) | next_obs | done] (the layout of the expert / ring
    tables, imb_table_store) plus its ground-truth rewards.  A fragment is stacked on the host and uploaded ONCE, on first
    use; afterwards a minibatch of 2 P fragments is an index vector and one imb_gather_rows launch into the feature-major
    batch the reward kernels read -- the reference re-walks every fragment on the host on every use
    (preference_comparisons.py:441-454)."""

    def __init__(self, d_obs: int, d_act: int, discrete: bool, device):
        self.d_obs, self.d_act, self.discrete, self.device = d_obs, d_act, discrete, th.device(device)
        self.tw = _desc.table_width(d_obs, d_act)
        self.L: Optional[int] = None
        self.table: Optional[th.Tensor] = None
        self.rews: Optional[th.Tensor] = None
        self._slots: Dict[int, Tuple[object, int]] = {}
        self._state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device=self.device)
        self._stage_table: Optional[th.Tensor] = None
        self._stage_rews: Optional[th.Tensor] = None

    def _grow(self, n_slots: int) -> None:
        rows = n_slots * self.L
        if self.table is None:
            cap = max(rows, 256 * self.L)
            self.table = th.zeros(cap, self.tw, device=self.device)
            self.rews = th.zeros(cap, device=self.device)
        elif rows > self.table.shape[0]:
            cap = max(rows, 2 * self.table.shape[0])
            t = th.zeros(cap, self.tw, device=self.device)
            t[:self.table.shape[0]] = self.table
            r = th.zeros(cap, device=self.device)
            r[:self.rews.shape[0]] = self.rews
            self.table, self.rews = t, r

    def _upload(self, frags: Sequence[TrajectoryWithRew], table: th.Tensor, rews: th.Tensor, row0: int) -> None:
        """Stack `frags` on the host and store their L-row blocks at rows [row0, row0 + len(frags) * L) of `table`
        (and their ground-truth rewards, if any, in `rews`)."""
        tr = _stack_fragments(frags)
        n = len(tr["obs"])
        dev = self.device
        f32 = lambda x: th.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).to(dev).reshape(n, -1)
        dones = th.as_tensor(np.ascontiguousarray(tr["dones"]).astype(np.uint8)).to(dev)
        dst = table[row0:]
        if self.discrete:
            acts = th.as_tensor(np.ascontiguousarray(tr["acts"]).astype(np.int64)).to(dev).reshape(n)
            _lib.table_store(dst, n, self.d_obs, self.d_act, f32(tr["obs"]), None, acts, f32(tr["next_obs"]), dones, n,
                             False, self._state)
        else:
            _lib.table_store(dst, n, self.d_obs, self.d_act, f32(tr["obs"]), f32(tr["acts"]), None, f32(tr["next_obs"]),
                             dones, n, False, self._state)
        if isinstance(frags[0], TrajectoryWithRew):
            rews[row0:row0 + n] = th.as_tensor(np.concatenate([f.rews for f in frags]).astype(np.float32)).to(dev)

    def slots(self, frags: Sequence[TrajectoryWithRew]) -> th.Tensor:
        """Slot index of every fragment (uploading the ones not seen before), as a device int64 vector."""
        if self.L is None:
            self.L = len(frags[0])
        out, new = [], []
        for f in frags:
            ent = self._slots.get(id(f))
            if ent is None or ent[0] is not f:
                ent = (f, len(self._slots))
                self._slots[id(f)] = ent  # (keeps the fragment alive: its id cannot be reused while it is pooled)
                new.append(f)
            out.append(ent[1])
        if new:
            k0 = self._slots[id(new[0])][1]
            self._grow(len(self._slots))
            self._upload(new, self.table, self.rews, k0 * self.L)
        return th.as_tensor(np.asarray(out, dtype=np.int64)).to(self.device)

    def stage(self, frags: Sequence[TrajectoryWithRew]) -> th.Tensor:
        """Upload `frags` to the staging table (fragment j at rows [j * L, (j + 1) * L)) without registering them, and
        return that table.  Candidates of an active selection go here: only the selected ones are then `adopt`ed, so the
        rejected ones leave no rows behind.  The table is reused (and grown) across calls."""
        if self.L is None:
            self.L = len(frags[0])
        rows = len(frags) * self.L
        if self._stage_table is None or self._stage_table.shape[0] < rows:
            self._stage_table = th.zeros(rows, self.tw, device=self.device)
            self._stage_rews = th.zeros(rows, device=self.device)
        self._upload(frags, self._stage_table, self._stage_rews, 0)
        return self._stage_table

    def adopt(self, frags: Sequence[TrajectoryWithRew], staged: Sequence[int]) -> None:
        """Register `frags`, whose rows sit at staging slots `staged` since the last `stage`, as pool fragments: a
        device-to-device copy of their rows, no upload."""
        src, new = [], []
        for f, j in zip(frags, staged):
            ent = self._slots.get(id(f))
            if ent is None or ent[0] is not f:
                self._slots[id(f)] = (f, len(self._slots))
                new.append(f)
                src.append(j)
        if not new:
            return
        k0 = self._slots[id(new[0])][1]
        self._grow(len(self._slots))
        ar = th.arange(self.L, device=self.device)
        src_rows = (th.as_tensor(np.asarray(src, dtype=np.int64)).to(self.device)[:, None] * self.L + ar).reshape(-1)
        n = src_rows.numel()
        self.table[k0 * self.L:k0 * self.L + n] = self._stage_table.index_select(0, src_rows)
        self.rews[k0 * self.L:k0 * self.L + n] = self._stage_rews.index_select(0, src_rows)

    def row_index(self, slots: th.Tensor) -> th.Tensor:
        return (slots[:, None] * self.L + th.arange(self.L, device=self.device)[None, :]).reshape(-1)

    def dataset_rows(self, dataset) -> Optional[Tuple[th.Tensor, th.Tensor, th.Tensor, bool]]:
        """(R1, R2, prefs, has_gt) of a dataset of fragment pairs: R1[i] / R2[i] = the L pool rows of item i's first /
        second fragment (device int64 [N, L]), prefs = its preferences (device float32 [N]), has_gt = the fragments carry
        ground-truth rewards.  Built once per dataset state and reused by every epoch and every ensemble member; None if
        the fragments do not all have the pool's length."""
        if isinstance(dataset, PreferenceDataset):
            f1, f2, prefs = dataset.fragments1, dataset.fragments2, dataset.preferences
        else:
            items = [dataset[i] for i in range(len(dataset))]
            f1, f2 = [it[0][0] for it in items], [it[0][1] for it in items]
            prefs = np.asarray([it[1] for it in items])
        n = len(f1)
        key = (id(dataset), n, id(f1[0]), id(f1[-1]), id(f2[-1]))
        hit = self.__dict__.get("_ds_cache")
        if hit is not None and hit[0] == key:
            return hit[1]
        L = self.L if self.L is not None else len(f1[0])
        if any(len(f) != L for f in f1) or any(len(f) != L for f in f2):
            return None
        slots = self.slots(list(f1) + list(f2))
        ar = th.arange(self.L, device=self.device)[None, :]
        out = ((slots[:n, None] * self.L + ar).contiguous(), (slots[n:, None] * self.L + ar).contiguous(),
               th.as_tensor(np.ascontiguousarray(prefs, dtype=np.float32)).to(self.device),
               all(isinstance(f, TrajectoryWithRew) for f in (f1[0], f2[0], f1[-1], f2[-1])))
        self._ds_cache = (key, out)
        return out


class PreferenceModel(nn.Module):
    """Fragment rewards -> probability that the first fragment is preferred (:345-530)."""

    def __init__(self, model: reward_nets.RewardNet, noise_prob: float = 0.0, discount_factor: float = 1.0,
                 threshold: float = 50) -> None:
        super().__init__()
        self.model = model
        self.noise_prob, self.discount_factor, self.threshold = noise_prob, discount_factor, threshold
        base_model = get_base_model(model)
        self.ensemble_model = None
        if isinstance(base_model, reward_nets.RewardEnsemble):
            is_std_wrapper = isinstance(model, reward_nets.AddSTDRewardWrapper) and model.base is base_model
            if not (model is base_model or is_std_wrapper):
                raise ValueError(f"RewardEnsemble can only be wrapped by AddSTDRewardWrapper but found {type(model).__name__}.")
            self.ensemble_model = base_model
            self.member_pref_models = [PreferenceModel(m, self.noise_prob, self.discount_factor, self.threshold)
                                       for m in self.ensemble_model.members]
        # device-resident fragment pool (shared by the members of an ensemble): used when the model is a fused net,
        # possibly inside pass-through wrappers, and the fragments have equal lengths
        self.use_fragment_pool = True
        self._pool: Optional[FragmentPool] = None
        if self.ensemble_model is not None:
            for m in self.member_pref_models:
                m.__dict__["_pool_owner"] = self  # (not a submodule: a member's parameters() are its own network's only)

    _pool_owner = None

    def _fused_target(self):
        """The fused network whose forward() equals self.model's forward() (wrappers that only change predict_processed
        are transparent for the forward pass, reward_nets.py:314-322), or None."""
        m = self.model
        while isinstance(m, reward_nets.PredictProcessedWrapper):
            m = m.base
        return m if hasattr(m, "forward_batch") and hasattr(m, "_engine") else None

    def _get_pool(self, net) -> FragmentPool:
        owner = self._pool_owner or self
        if owner._pool is None:
            d = net.engine().desc
            discrete = spaces.is_discrete(net.action_space)
            owner._pool = FragmentPool(d.d_obs, d.d_act, discrete, net.engine().device())
        return owner._pool

    # -- rewards of a batch of transitions (keeps the graph for single networks) ----------------------------------
    def rewards(self, transitions) -> th.Tensor:
        tr = types.as_transition_arrays(transitions)
        state, action, next_state, done = tr["obs"], tr["acts"], tr["next_obs"], tr["dones"]
        if self.ensemble_model is not None:
            rews_np = self.ensemble_model.predict_processed_all(state, action, next_state, done)
            assert rews_np.shape == (len(state), self.ensemble_model.num_members)
            return th.as_tensor(rews_np).to(self.ensemble_model.device)
        rews = self.model(*self.model.preprocess(state, action, next_state, done))
        assert rews.shape == (len(state),)
        return rews

    def probability(self, rews1: th.Tensor, rews2: th.Tensor) -> th.Tensor:
        """Boltzmann-rational probability that fragment 1 is best; time is axis 0 (:487-530)."""
        expected_dims = 2 if self.ensemble_model is not None else 1
        assert rews1.ndim == rews2.ndim == expected_dims
        return self._probability(rews1, rews2, time_axis=0)

    def _probability(self, rews1: th.Tensor, rews2: th.Tensor, time_axis: int) -> th.Tensor:
        diff = rews2 - rews1
        if self.discount_factor == 1:
            returns_diff = diff.sum(dim=time_axis)
        else:
            L = diff.shape[time_axis]
            discounts = self.discount_factor ** th.arange(L, device=diff.device)
            shape = [1] * diff.ndim
            shape[time_axis] = L
            returns_diff = (discounts.reshape(shape) * diff).sum(dim=time_axis)
        returns_diff = th.clip(returns_diff, -self.threshold, self.threshold)  # also keeps the backward finite
        model_probability = 1 / (1 + returns_diff.exp())
        return self.noise_prob * 0.5 + (1 - self.noise_prob) * model_probability

    def forward(self, fragment_pairs: Sequence[Tuple[types.Trajectory, types.Trajectory]]
                ) -> Tuple[th.Tensor, Optional[th.Tensor]]:
        """Probabilities for all pairs: shape (P,) (single network, differentiable) or (P, members)."""
        P = len(fragment_pairs)
        frags = [p[0] for p in fragment_pairs] + [p[1] for p in fragment_pairs]
        lengths = {len(f) for f in frags}
        gt_available = isinstance(fragment_pairs[0][0], TrajectoryWithRew) and isinstance(fragment_pairs[0][1], TrajectoryWithRew)
        net = self._fused_target() if (self.use_fragment_pool and self.ensemble_model is None) else None
        pooled = None
        if len(lengths) == 1 and net is not None and net.engine().device().type == "cuda":
            # device-resident fragments: one index vector + one gather launch feed the fused kernels
            L = lengths.pop()
            pool = self._get_pool(net)
            if pool.L in (None, L):
                slots = pool.slots(frags)
                idx = pool.row_index(slots)
                e = net.engine()
                n = 2 * P * L
                batch, ld = e.new_batch(n)
                _lib.gather_rows(pool.table, pool.table.shape[0], pool.tw, idx, n, batch, ld, 0)
                rews = net.forward_batch(batch, ld, n).reshape(2, P, L)
                probs = self._probability(rews[0], rews[1], time_axis=1)
                pooled = (pool, idx)
            lengths = {L}
        if pooled is not None:
            pass
        elif len(lengths) == 1:
            # one batch of 2 * P * L rows through the fused kernels; rows f * L + t, first fragments first
            L = lengths.pop()
            rews = self.rewards(_stack_fragments(frags))
            rews = rews.reshape((2, P, L) + tuple(rews.shape[1:]))
            probs = self._probability(rews[0], rews[1], time_axis=1)
        else:  # ragged fragments: pair by pair like the reference
            probs = th.stack([self.probability(self.rewards(rollout.flatten_trajectories([a])),
                                               self.rewards(rollout.flatten_trajectories([b])))
                              for a, b in fragment_pairs])
        gt_probs = None
        if gt_available and pooled is not None:
            gr = pooled[0].rews[pooled[1]].reshape(2, P, -1)
            gt_probs = self._probability(gr[0], gr[1], time_axis=1).cpu()  # (a host tensor, like the reference's)
        elif gt_available:
            if len({len(f) for f in frags}) == 1:
                gr = th.as_tensor(np.stack([f.rews for f in frags])).reshape(2, P, -1)
                gt_probs = self._probability(gr[0], gr[1], time_axis=1)
            else:
                gt_probs = th.stack([self._probability(th.from_numpy(a.rews), th.from_numpy(b.rews), 0)
                                     for a, b in fragment_pairs])
        return probs, gt_probs

    # -- active selection: candidate scores on the device -------------------------------------------------------------
    def _scoring_members(self) -> Optional[Tuple[list, list]]:
        """(fused nets, output norms) of the members, when every member is a fused reward net on CUDA, optionally inside
        a NormalizedRewardNet, all with the same spaces and at most 16 of them; otherwise None."""
        if self.ensemble_model is None or not self.use_fragment_pool:
            return None
        members = list(self.ensemble_model.members)
        if len(members) > _lib.PU_MAX_MEMBERS:
            return None
        nets, outs = [], []
        for m in members:
            out = m if type(m) is reward_nets.NormalizedRewardNet else None
            net = m.base if out is not None else m
            if not isinstance(net, reward_nets._FusedNetMixin) or net.device.type != "cuda":
                return None
            nets.append(net)
            outs.append(out)
        d0 = nets[0].engine().desc
        if any(n.device != nets[0].device or n.engine().desc.d_obs != d0.d_obs or n.engine().desc.d_act != d0.d_act
               for n in nets):
            return None
        return nets, outs

    def uncertainty_scores(self, fragment_pairs: Sequence[TrajectoryWithRewPair], uncertainty_on: str,
                           member_values: bool = False) -> Optional[Tuple[th.Tensor, Optional[th.Tensor]]]:
        """Active-selection scores of the candidate pairs (device float32 [C]), and with `member_values` the per-member
        return differences (logit) or probabilities (probability, label) [C, M]; None when the members or fragments are
        outside the device path (see `ActiveSelectionFragmenter`).

        The candidates go to the fragment pool's staging table (slot 2 i + s = pair i, fragment s), one gather builds the
        feature-major batch, one `imb_reward_forward` per member (eval mode, as `predict_processed`) writes its raw
        rewards, and `imb_pref_uncertainty` applies the NormalizedRewardNet members' output normalisation fragment by
        fragment -- advancing their statistics as the reference's per-fragment `predict_processed` calls do -- and scores
        every pair.  `adopt_candidates` then registers the selected fragments in the pool."""
        frags = [f for pair in fragment_pairs for f in pair]
        lengths = {len(f) for f in frags}
        members = self._scoring_members()
        if len(lengths) != 1 or members is None:
            return None
        L = lengths.pop()
        nets, outs = members
        pool = self._get_pool(nets[0])
        if pool.L not in (None, L):
            return None
        table = pool.stage(frags)
        C, M, n = len(fragment_pairs), len(nets), len(frags) * L
        e0 = nets[0].engine()
        dev = e0.device()
        batch, ld = e0.new_batch(n)
        _lib.gather_rows(table, table.shape[0], pool.tw, None, n, batch, ld, 0)
        rews = th.empty(M, n, device=dev)
        for k, net in enumerate(nets):
            e = net.engine()
            _lib.reward_forward(e.desc, e.params, e.norm_state, batch, ld, n, 0, rews[k])
        norms = [None if o is None else o.output_norm_args() for o in outs]
        desc = _lib.pref_uncertainty_desc(list(rews), norms)
        ws_n = _lib.pref_uncertainty_ws_floats(M, C)
        ws = self.__dict__.get("_pu_ws")
        if ws is None or ws.numel() < ws_n or ws.device != dev:
            ws = self._pu_ws = th.zeros(ws_n, device=dev)  # (zero-filled once: the kernel re-arms its ticket)
        scores = th.empty(C, device=dev)
        member_out = th.empty(C, M, device=dev) if member_values else None
        _lib.pref_uncertainty(desc, C, L, _lib.PU_MODES[uncertainty_on], self.noise_prob, self.discount_factor,
                              self.threshold, ws, scores, member_out)
        return scores, member_out

    def adopt_candidates(self, fragment_pairs: Sequence[TrajectoryWithRewPair], chosen: Sequence[int]) -> None:
        """Register pairs `chosen` of the candidates last scored by `uncertainty_scores` in the fragment pool (a device
        row copy from the staging table), so training on them uploads nothing."""
        pool = (self._pool_owner or self)._pool
        frags = [f for i in chosen for f in fragment_pairs[i]]
        pool.adopt(frags, [2 * i + s for i in chosen for s in (0, 1)])


class ActiveSelectionFragmenter(Fragmenter):
    """Pairs the ensemble members disagree on most (:668-778): draws `fragment_sample_factor * num_pairs` candidates
    from `base_fragmenter` (the same host random draws as the reference), scores each and returns the `num_pairs` with
    the highest scores, ordered by descending score.  The score is the variance over the members of

    - `logit`: the undiscounted return difference sum_t r1 - sum_t r2 (torch.var, ddof 1; discount, threshold and noise
      are not used);
    - `probability`: `PreferenceModel.probability` (np.var, ddof 0);
    - `label`: the Bernoulli variance q (1 - q) of the labels probability > 0.5, q their mean;

    where the rewards are each member's `predict_processed` of one fragment at a time, in the order pair 0 first, pair
    0 second, pair 1 first, ...; a NormalizedRewardNet member normalises each fragment with its output statistics as
    they stood before that fragment, then merges it into them.

    Ties are ordered by descending candidate index (`np.argsort(scores, kind="stable")[::-1]`).  The reference uses
    NumPy's default sort, which is not stable and orders equal scores differently on different CPUs; the label mode has
    ties all the time.

    When every member is a fused reward net on CUDA (optionally inside a NormalizedRewardNet), there are at most 16 and
    all candidates have the fragment pool's length, the scoring runs on the device (`PreferenceModel.uncertainty_scores`)
    and the selected fragments enter the fragment pool without another upload; otherwise the reference's per-pair loop
    over `PreferenceModel.rewards` and `variance_estimate` runs."""

    def __init__(self, preference_model: PreferenceModel, base_fragmenter: Fragmenter, fragment_sample_factor: float,
                 uncertainty_on: str = "logit", custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        super().__init__(custom_logger=custom_logger)
        if preference_model.ensemble_model is None:
            raise ValueError("PreferenceModel not wrapped over an ensemble of networks.")
        self.preference_model = preference_model
        self.base_fragmenter = base_fragmenter
        self.fragment_sample_factor = fragment_sample_factor
        self._uncertainty_on = uncertainty_on
        if uncertainty_on not in ("logit", "probability", "label"):
            self.raise_uncertainty_on_not_supported()

    @property
    def uncertainty_on(self) -> str:
        return self._uncertainty_on

    def raise_uncertainty_on_not_supported(self):
        raise ValueError(f"""{self.uncertainty_on} not supported.
            `uncertainty_on` should be from `logit`, `probability`, or `label`""")

    def __call__(self, trajectories: Sequence[TrajectoryWithRew], fragment_length: int, num_pairs: int
                 ) -> Sequence[TrajectoryWithRewPair]:
        candidates = self.base_fragmenter(trajectories=trajectories, fragment_length=fragment_length,
                                          num_pairs=int(self.fragment_sample_factor * num_pairs))
        if len(candidates) == 0:
            return []
        with th.no_grad():
            dev = self.preference_model.uncertainty_scores(candidates, self.uncertainty_on)
        if dev is not None:
            # stable ascending sort, reversed: descending score, ties by descending index; one read-back
            chosen = th.argsort(dev[0], stable=True).flip(0)[:num_pairs].cpu().tolist()
            self.preference_model.adopt_candidates(candidates, chosen)
        else:
            scores = np.zeros(len(candidates))
            for i, (frag1, frag2) in enumerate(candidates):
                with th.no_grad():
                    rews1 = self.preference_model.rewards(rollout.flatten_trajectories([frag1]))
                    rews2 = self.preference_model.rewards(rollout.flatten_trajectories([frag2]))
                scores[i] = self.variance_estimate(rews1, rews2)
            chosen = np.argsort(scores, kind="stable")[::-1][:num_pairs].tolist()
        return [candidates[i] for i in chosen]

    def variance_estimate(self, rews1: th.Tensor, rews2: th.Tensor) -> float:
        """Score of one pair from the members' rewards of its fragments, [fragment_length, members] each (:749-778)."""
        if self.uncertainty_on == "logit":
            return (rews1.sum(0) - rews2.sum(0)).var().item()
        probs = self.preference_model.probability(rews1, rews2).cpu().numpy()
        assert probs.shape == (self.preference_model.model.num_members,)
        if self.uncertainty_on == "probability":
            return probs.var()
        if self.uncertainty_on == "label":
            q = (probs > 0.5).astype(np.float32).mean()
            return q * (1 - q)
        self.raise_uncertainty_on_not_supported()


class LossAndMetrics(NamedTuple):
    loss: th.Tensor
    metrics: Mapping[str, th.Tensor]


class RewardLoss(nn.Module, abc.ABC):
    @abc.abstractmethod
    def forward(self, fragment_pairs, preferences: np.ndarray, preference_model: PreferenceModel) -> LossAndMetrics:
        """Loss of the preference model on a batch of comparisons."""


class CrossEntropyRewardLoss(RewardLoss):
    """Cross entropy between the model's and the target preference probabilities (:1043-1090)."""

    def forward(self, fragment_pairs, preferences: np.ndarray, preference_model: PreferenceModel) -> LossAndMetrics:
        probs, gt_probs = preference_model(fragment_pairs)
        preferences_th = th.as_tensor(preferences, dtype=th.float32)
        predictions = probs.detach().cpu() > 0.5
        ground_truth = preferences_th > 0.5
        metrics = {"accuracy": (predictions == ground_truth).float().mean()}
        if gt_probs is not None:
            metrics["gt_reward_loss"] = th.nn.functional.binary_cross_entropy(gt_probs.cpu(), preferences_th)
        metrics = {k: v.detach().cpu() for k, v in metrics.items()}
        loss = th.nn.functional.binary_cross_entropy(probs, preferences_th.to(probs.device))
        return LossAndMetrics(loss=loss, metrics=metrics)


# ------------------------------------------------------------------------------------------------
# reward trainers
# ------------------------------------------------------------------------------------------------
class RewardTrainer(abc.ABC):
    def __init__(self, preference_model: PreferenceModel,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        self._preference_model = preference_model
        self._logger = custom_logger or imit_logger.configure()

    @property
    def logger(self) -> imit_logger.HierarchicalLogger:
        return self._logger

    @logger.setter
    def logger(self, custom_logger: imit_logger.HierarchicalLogger) -> None:
        self._logger = custom_logger

    def train(self, dataset, epoch_multiplier: float = 1.0) -> None:
        from ..util import networks

        with networks.training(self._preference_model.model):
            self._train(dataset, epoch_multiplier)

    @abc.abstractmethod
    def _train(self, dataset, epoch_multiplier: float) -> None:
        """Train the reward model."""


_PERM_FAST: Optional[bool] = None


def _epoch_permutation(n: int) -> th.Tensor:
    """The item order of ONE pass of `DataLoader(<n items>, shuffle=True)` (the reference's minibatch source,
    preference_comparisons.py:1207-1216), drawn with exactly that iterator's consumption of torch's global RNG: one
    int64 for the iterator's base seed, one for the RandomSampler's generator seed, then `randperm` on that generator.
    Producing the whole permutation at once lets an epoch upload its indices in one copy instead of collating every
    minibatch on the host.  The shortcut mirrors torch internals, so it is verified against a real DataLoader (on a
    saved / restored RNG state) the first time it is used; on any mismatch the DataLoader itself is iterated."""
    global _PERM_FAST

    def fast(k):
        th.empty((), dtype=th.int64).random_()
        g = th.Generator()
        g.manual_seed(int(th.empty((), dtype=th.int64).random_().item()))
        return th.randperm(k, generator=g)

    def slow(k):
        return th.cat([b for b in data_th.DataLoader(range(k), batch_size=max(1, min(k, 64)), shuffle=True)])

    if _PERM_FAST is None:
        state = th.get_rng_state()
        a, sa = fast(11), th.get_rng_state()
        th.set_rng_state(state)
        b, sb = slow(11), th.get_rng_state()
        th.set_rng_state(state)
        _PERM_FAST = bool(th.equal(a, b) and th.equal(sa, sb))
    return fast(n) if _PERM_FAST else slow(n)


def _resolve_subsets(dataset) -> Tuple[Any, Optional[np.ndarray]]:
    """(base dataset, item indices into it | None) of nested `Subset`s: an ensemble's bagging subsets and the
    training / validation split of a regularizer all index one shared base dataset."""
    index = None
    while isinstance(dataset, data_th.Subset):
        ind = np.asarray(dataset.indices, dtype=np.int64)
        index = ind if index is None else ind[index]
        dataset = dataset.dataset
    return dataset, index


class BasicRewardTrainer(RewardTrainer):
    """Minibatch gradient accumulation with AdamW over a `PreferenceDataset` (:1139-1323)."""

    def __init__(self, preference_model: PreferenceModel, loss: RewardLoss, rng: np.random.Generator,
                 batch_size: int = 32, minibatch_size: Optional[int] = None, epochs: int = 1, lr: float = 1e-3,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None, regularizer_factory=None) -> None:
        super().__init__(preference_model, custom_logger)
        self.loss = loss
        self.batch_size = batch_size
        self.minibatch_size = minibatch_size or batch_size
        if self.batch_size % self.minibatch_size != 0:
            raise ValueError("Batch size must be a multiple of minibatch size.")
        self.epochs = epochs
        self.optim = th.optim.AdamW(self._preference_model.parameters(), lr=lr)
        self.rng = rng
        self.regularizer: Optional[regularizers.Regularizer] = (
            regularizer_factory(optimizer=self.optim, logger=self.logger) if regularizer_factory is not None else None)
        self.last_epoch_stats: Dict[str, float] = {}
        # the regularization keys of the last epoch, recorded as reward/final/<key> (a subset of FINAL_KEYS)
        self.final_stats: Dict[str, float] = {}

    FINAL_KEYS = ("regularized_loss", "regularization_lambda", "val/loss", "val/accuracy", "val/gt_reward_loss")

    def _make_data_loader(self, dataset) -> data_th.DataLoader:
        return data_th.DataLoader(dataset, batch_size=self.minibatch_size, shuffle=True,
                                  collate_fn=preference_collate_fn)

    @property
    def requires_regularizer_update(self) -> bool:
        return self.regularizer is not None and self.regularizer.val_split is not None

    def _split(self, dataset):
        """(training part, validation part | None) of `dataset`: with a regularizer that has a validation split, the
        reference's `random_split` (:1224-1245), seeded by one `make_seeds(self.rng)` draw per call."""
        if not self.requires_regularizer_update:
            return dataset, None
        val_length = int(len(dataset) * self.regularizer.val_split)
        train_length = len(dataset) - val_length
        if val_length < 1 or train_length < 1:
            raise ValueError("Not enough data samples to split into training and validation, or the validation split "
                             "is too large/small. Make sure you've generated enough initial preference data. You can "
                             "adjust this through initial_comparison_frac in PreferenceComparisons.")
        train, val = data_th.random_split(dataset, lengths=[train_length, val_length],
                                          generator=th.Generator().manual_seed(make_seeds(self.rng)))
        return train, val

    def _skip_draws(self, dataset, epoch_multiplier: float = 1.0) -> None:
        """Make exactly the draws `train(dataset, epoch_multiplier)` makes from `self.rng` and torch's global RNG,
        without training: the split seed, then per epoch the training loader's and the validation loader's shuffles.
        A rank of a member-parallel ensemble runs this for the members it does not train."""
        train, val = self._split(dataset)
        for _ in range(round(self.epochs * epoch_multiplier)):
            _epoch_permutation(len(train))
            if val is not None:
                _epoch_permutation(len(val))

    def _record_final_stats(self, stats: Dict[str, float]) -> None:
        self.final_stats = stats
        for k, v in stats.items():
            self.logger.record(f"reward/final/{k}", v)

    # -- the fused step: a minibatch never leaves the device ------------------------------------------------------------
    use_fused_step = True

    def _fused_target(self, dataset):
        """(net, pool, base dataset, item indices | None) when the whole training step can run as kernels on the device:
        cross-entropy loss on a single fused network, every parameter trained by a plain AdamW, no regularizer or one of
        this package's `LpRegularizer` / `WeightDecayRegularizer` (exactly those classes), equal-length fragments.
        Otherwise None: the per-minibatch autograd path below covers everything else."""
        pm = self._preference_model
        if not (self.use_fused_step and type(self.loss) is CrossEntropyRewardLoss and pm.ensemble_model is None
                and pm.use_fragment_pool and type(self.optim) is th.optim.AdamW and len(self.optim.param_groups) == 1
                and type(self.regularizer) in (type(None), regularizers.LpRegularizer,
                                               regularizers.WeightDecayRegularizer)):
            return None
        g = self.optim.param_groups[0]
        if g.get("amsgrad") or g.get("maximize") or g.get("capturable") or g.get("differentiable"):
            return None
        net = pm._fused_target()
        if net is None or net.engine().device().type != "cuda":
            return None
        e = net.engine()
        plist = e._param_list()
        if ({id(p) for p in g["params"]} != {id(p) for p in plist} or not all(p.requires_grad for p in plist)
                or len(dataset) == 0):
            return None
        dataset, index = _resolve_subsets(dataset)
        pool = pm._get_pool(net)
        rows = pool.dataset_rows(dataset)
        if rows is None:
            return None
        return net, pool, rows, index

    def _fused_optimizer_state(self, e):
        """Adam moments as flat device vectors next to the flat parameter vector, ALIASED by the torch optimiser's
        per-parameter state (so `optim.state_dict()`, and the autograd path should it run later, see the same moments)."""
        plist = e._param_list()
        fo = self.__dict__.get("_fused_opt")
        if fo is None or fo["ptr"] != e.params.data_ptr():
            n, dev = e.desc.n_params, e.params.device
            m, v = th.zeros(n, device=dev), th.zeros(n, device=dev)
            shapes = [p.shape for p in plist]
            for p, pm, pv in zip(plist, views(m, shapes), views(v, shapes)):
                st = self.optim.state.get(p)
                if st:
                    pm.copy_(st["exp_avg"])
                    pv.copy_(st["exp_avg_sq"])
                self.optim.state[p] = {"step": th.tensor(float(st["step"]) if st else 0.0), "exp_avg": pm, "exp_avg_sq": pv}
            fo = dict(ptr=e.params.data_ptr(), m=m, v=v, state=th.zeros(_lib.ST_WORDS, dtype=th.int64, device=dev))
            self._fused_opt = fo
        g = self.optim.param_groups[0]
        fo["hp"] = _lib.Adam(lr=g["lr"], beta1=g["betas"][0], beta2=g["betas"][1], eps=g["eps"],
                             weight_decay=g["weight_decay"])
        fo["step"] = int(self.optim.state[plist[0]]["step"])
        fo["state"][_lib.ST_DISC_STEP] = fo["step"]
        return fo

    def _train_fused(self, target, n_items: int, epochs: int, val_index: Optional[np.ndarray] = None) -> None:
        """The reference's loop (:1218-1323) with every minibatch as device work only: row-index gather from the fragment
        pool -> imb_reward_forward -> imb_pref_loss (returns, Boltzmann probability, cross entropy, d loss / d rewards)
        -> imb_disc_fwd_bwd with that upstream gradient (accumulating over the minibatches of a batch) -> reduction +
        AdamW in one launch.  Minibatch composition is the reference's DataLoader(shuffle=True) order (same consumption of
        torch's global RNG, `_epoch_permutation`); losses and accuracies are accumulated on the device and read back once
        after the last epoch.

        With a regularizer, `imb_param_regularize` runs after every training minibatch's fwd_bwd (Lp: its gradient into
        the accumulator and its value into a statistics slot; weight decay: on the parameters, before the optimiser
        step).  With a lambda updater, the epoch's validation items (`val_index`, shuffled by their own loader's draw
        after the training loader's) go through the training-mode forward and imb_pref_loss without a gradient, and the
        epoch's statistics are read back to hand the scaled training loss and the validation loss to `update_params`;
        the new lambda applies from the next epoch."""
        net, pool, (R1, R2, prefs_all, has_gt), index = target
        pm = self._preference_model
        e = net.engine()
        e.sync()
        fo = self._fused_optimizer_state(e)
        dev, L = e.params.device, pool.L
        reg = self.regularizer
        lp = type(reg) is regularizers.LpRegularizer
        # statistics slots per epoch: 0 = model loss / accuracy / count, 1 = ground truth; with a regularizer also
        # 2 = the model statistics of a short last minibatch (so that the scaled loss sum is exact), 3 = the Lp penalty,
        # 4 / 5 = the validation model / ground truth
        S = 2 if reg is None else 6
        index_t = None if index is None else th.as_tensor(index)
        val_t = None if val_index is None else th.as_tensor(val_index)
        stats = th.zeros(4 * S * epochs, device=dev)
        train_norm = bool(net.training and e.has_norm)
        bufs: Dict[int, Tuple[th.Tensor, int, th.Tensor, th.Tensor]] = {}
        n_steps = 0

        def forward(ids):
            """Gather the minibatch's 2 P fragments, update the input norm (training mode) and evaluate the rewards."""
            P = int(ids.numel())
            idx = th.cat([R1.index_select(0, ids), R2.index_select(0, ids)]).reshape(-1)
            n = 2 * P * L
            if n not in bufs:
                b, ld = e.new_batch(n)
                bufs[n] = (b, ld, th.empty(n, device=dev), th.empty(n, device=dev))
            batch, ld, rews, grad = bufs[n]
            _lib.gather_rows(pool.table, pool.table.shape[0], pool.tw, idx, n, batch, ld, 0)
            if train_norm:
                e.norm_update(batch, ld, n)
            if train_norm and e.desc.shaped:  # the training-mode forward of a shaped net reads the mid-update snapshot
                rews = reward_nets._FusedForward._fwd_train(e, batch, ld, n)
            else:
                _lib.reward_forward(e.desc, e.params, e.norm_state, batch, ld, n, 0, rews)
            return P, idx, n, batch, ld, rews, grad, prefs_all.index_select(0, ids)

        def epoch_stats(st):
            """Host statistics of one epoch's [S, 4] slots: (loss sum, accuracy sum, minibatches) of the model."""
            model = st[0] if S == 2 else st[0] + st[2]
            return float(model[0]), float(model[1]), max(float(model[2]), 1.0)

        def scaled_loss_sum(st):
            """Sum over the epoch's training minibatches of loss * P / batch_size (the reference's train_loss)."""
            short = n_items % self.minibatch_size
            return (float(st[0, 0]) * self.minibatch_size + float(st[2, 0]) * short) / self.batch_size

        with self.logger.accumulate_means("reward"):
            for epoch_num in range(epochs):
                slot = S * epoch_num
                if reg is not None:  # lambda as it stands at the start of the epoch
                    coeff = (reg.lambda_ if lp else -reg.lambda_ * self.optim.param_groups[0]["lr"])
                    kind = _lib.REG_LP if lp else _lib.REG_WEIGHT_DECAY
                accumulated = 0
                perm = _epoch_permutation(n_items)
                perm = (perm if index_t is None else index_t[perm]).to(dev)  # the epoch's item order: one upload
                for s0 in range(0, n_items, self.minibatch_size):
                    P, idx, n, batch, ld, rews, grad, y = forward(perm[s0:s0 + self.minibatch_size])
                    mslot = slot + 2 if (reg is not None and P < self.minibatch_size) else slot
                    # (an incomplete batch gets proportionally smaller gradients: loss * len / batch_size, :1288-1291)
                    _lib.pref_loss(rews, P, L, y, pm.noise_prob, pm.discount_factor, pm.threshold, P / self.batch_size,
                                   grad, None, stats, mslot)
                    if has_gt:
                        _lib.pref_loss(pool.rews.index_select(0, idx), P, L, y, pm.noise_prob, pm.discount_factor,
                                       pm.threshold, 0.0, None, None, stats, slot + 1)
                    e.fwd_bwd(batch, ld, n, n, 0.0, grad, None, accumulated == 0, train_norm and bool(e.desc.shaped))
                    if reg is not None:
                        _lib.param_regularize(e.desc, kind, reg.p if lp else 0, coeff, e.params, e.ws, stats, slot + 3)
                    accumulated += P
                    if accumulated >= self.batch_size:
                        _lib.disc_reduce_adam(e.desc, fo["hp"], e.params, fo["m"], fo["v"], 1.0, e.ws, fo["state"], None)
                        n_steps += 1
                        accumulated = 0
                    else:
                        e.reduce(None)
                if accumulated != 0:  # an incomplete batch remains
                    _lib.disc_adam(e.desc, fo["hp"], e.params, fo["m"], fo["v"], None, 1.0, e.ws, fo["state"], None)
                    n_steps += 1
                if val_t is None:
                    continue
                vperm = val_t[_epoch_permutation(len(val_t))].to(dev)  # the validation loader's shuffle, after training's
                for s0 in range(0, len(val_t), self.minibatch_size):
                    P, idx, n, batch, ld, rews, grad, y = forward(vperm[s0:s0 + self.minibatch_size])
                    _lib.pref_loss(rews, P, L, y, pm.noise_prob, pm.discount_factor, pm.threshold, 1.0, None, None,
                                   stats, slot + 4)
                    if has_gt:
                        _lib.pref_loss(pool.rews.index_select(0, idx), P, L, y, pm.noise_prob, pm.discount_factor,
                                       pm.threshold, 0.0, None, None, stats, slot + 5)
                st = stats[4 * slot:4 * (slot + S)].cpu().numpy().reshape(S, 4)  # the epoch's one read-back
                with self.logger.add_key_prefix(f"epoch-{epoch_num}"):
                    reg.update_params(scaled_loss_sum(st), float(st[4, 0]))
            for p in e._param_list():
                self.optim.state[p]["step"] = th.tensor(float(fo["step"] + n_steps))
            st = stats.cpu().numpy().reshape(epochs, S, 4)  # (without an updater: the one read-back of the training call)
            final: Dict[str, float] = {}
            for k in range(epochs):
                loss_sum, acc_sum, nb = epoch_stats(st[k])
                self.logger.record(f"epoch-{k}/train/loss", loss_sum / nb)
                self.logger.record(f"epoch-{k}/train/accuracy", acc_sum / nb)
                if has_gt:
                    self.logger.record(f"epoch-{k}/train/gt_reward_loss", float(st[k, 1, 0]) / nb)
                final = {}
                if lp:
                    final["regularized_loss"] = (scaled_loss_sum(st[k]) + float(st[k, 3, 0])) / max(float(st[k, 3, 2]), 1.0)
                    with self.logger.add_key_prefix(f"epoch-{k}"):
                        reg.logger.record("regularized_loss", final["regularized_loss"])
                if val_t is not None:
                    nv = max(float(st[k, 4, 2]), 1.0)
                    final["val/loss"], final["val/accuracy"] = float(st[k, 4, 0]) / nv, float(st[k, 4, 1]) / nv
                    if has_gt:
                        final["val/gt_reward_loss"] = float(st[k, 5, 0]) / nv
                    for key in ("val/loss", "val/accuracy", "val/gt_reward_loss"):
                        if key in final:
                            self.logger.record(f"epoch-{k}/{key}", final[key])
            loss_sum, acc_sum, nb = epoch_stats(st[-1])
            self.last_epoch_stats = {"loss": loss_sum / nb, "accuracy": acc_sum / nb}
        for k, v in self.last_epoch_stats.items():
            self.logger.record(f"reward/final/train/{k}", v)
        self._record_final_stats(self._final_regularization_stats(final))

    def _final_regularization_stats(self, last_epoch: Dict[str, float]) -> Dict[str, float]:
        """The reward/final/ keys the reference copies from the last epoch's regularization records: the validation
        statistics, and -- when the regularizer records into this trainer's logger -- regularized_loss and lambda."""
        out = {k: v for k, v in last_epoch.items() if k.startswith("val/")}
        reg = self.regularizer
        if reg is not None and reg.logger is self.logger:
            if "regularized_loss" in last_epoch:
                out["regularized_loss"] = last_epoch["regularized_loss"]
            if self.requires_regularizer_update:
                out["regularization_lambda"] = reg.lambda_
        return {k: out[k] for k in self.FINAL_KEYS if k in out}

    def _train(self, dataset, epoch_multiplier: float = 1.0) -> None:
        dataset, val_dataset = self._split(dataset)
        epochs = round(self.epochs * epoch_multiplier)
        assert epochs > 0, "Must train for at least one epoch."
        target = self._fused_target(dataset)
        if target is not None:
            val_index = None if val_dataset is None else _resolve_subsets(val_dataset)[1]
            self._train_fused(target, len(dataset), epochs, val_index)
            return
        dataloader = self._make_data_loader(dataset)
        val_dataloader = self._make_data_loader(val_dataset) if val_dataset is not None else None
        reg = self.regularizer
        final: Dict[str, float] = {}
        with self.logger.accumulate_means("reward"):
            for epoch_num in range(epochs):
                train_loss, accumulated_size, n_batches, acc, loss_sum = 0.0, 0, 0, 0.0, 0.0
                # whatever this epoch's minibatches record as regularized_loss (any regularizer recording into this
                # logger): its mean is recovered from the running mean's value and count before and after the epoch
                reg_key = f"mean/reward/epoch-{epoch_num}/regularized_loss"
                reg_before = (self.logger.name_to_value.get(reg_key, 0.0), self.logger.name_to_count.get(reg_key, 0))
                self.optim.zero_grad()
                for fragment_pairs, preferences in dataloader:
                    out = self.loss.forward(fragment_pairs, preferences, self._preference_model)
                    self.logger.record(f"epoch-{epoch_num}/train/loss", out.loss.item())
                    for name, value in out.metrics.items():
                        self.logger.record(f"epoch-{epoch_num}/train/{name}", value.item())
                    acc += float(out.metrics["accuracy"])
                    loss_sum += out.loss.item()
                    n_batches += 1
                    # averaged over the whole batch instead of the minibatch (an incomplete batch gets smaller gradients)
                    loss = out.loss * (len(fragment_pairs) / self.batch_size)
                    train_loss += loss.item()
                    if reg is not None:
                        with self.logger.add_key_prefix(f"epoch-{epoch_num}"):
                            reg.regularize_and_backward(loss)
                    else:
                        loss.backward()
                    accumulated_size += len(fragment_pairs)
                    if accumulated_size >= self.batch_size:
                        self.optim.step()
                        self.optim.zero_grad()
                        accumulated_size = 0
                if accumulated_size != 0:
                    self.optim.step()  # an incomplete batch remains
                # `reward/final/train/loss` of the reference = mean over the last epoch's minibatches of the UNSCALED
                # minibatch loss (logger.record("loss", ...) under accumulate_means, preference_comparisons.py:1296-1323)
                self.last_epoch_stats = {"loss": loss_sum / max(n_batches, 1), "accuracy": acc / max(n_batches, 1)}
                final = {}
                n_reg = self.logger.name_to_count.get(reg_key, 0) - reg_before[1]
                if n_reg > 0:
                    v, c = self.logger.name_to_value[reg_key], self.logger.name_to_count[reg_key]
                    final["regularized_loss"] = v if n_reg == c else (v * c - reg_before[0] * reg_before[1]) / n_reg
                if val_dataloader is None:
                    continue
                # validation: the training-mode forward (an input RunningNorm updates), no backward (:1284-1296)
                val_loss, val_sums, n_val = 0.0, defaultdict(float), 0
                for fragment_pairs, preferences in val_dataloader:
                    out = self.loss.forward(fragment_pairs, preferences, self._preference_model)
                    self.logger.record(f"epoch-{epoch_num}/val/loss", out.loss.item())
                    val_sums["val/loss"] += out.loss.item()
                    for name, value in out.metrics.items():
                        self.logger.record(f"epoch-{epoch_num}/val/{name}", value.item())
                        val_sums[f"val/{name}"] += value.item()
                    val_loss += out.loss.item()
                    n_val += 1
                final.update({k: v / max(n_val, 1) for k, v in val_sums.items()})
                with self.logger.add_key_prefix(f"epoch-{epoch_num}"):
                    reg.update_params(train_loss, val_loss)
        for k, v in self.last_epoch_stats.items():
            self.logger.record(f"reward/final/train/{k}", v)
        self._record_final_stats(self._final_regularization_stats(final))


class EnsembleTrainer(BasicRewardTrainer):
    """One `BasicRewardTrainer` per ensemble member, each on its own bootstrap sample (:1326-1438)."""

    def __init__(self, preference_model: PreferenceModel, loss: RewardLoss, rng: np.random.Generator,
                 batch_size: int = 32, minibatch_size: Optional[int] = None, epochs: int = 1, lr: float = 1e-3,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None, regularizer_factory=None) -> None:
        if preference_model.ensemble_model is None:
            raise TypeError("PreferenceModel of a RewardEnsemble expected by EnsembleTrainer.")
        super().__init__(preference_model, loss=loss, batch_size=batch_size, minibatch_size=minibatch_size,
                         epochs=epochs, lr=lr, custom_logger=custom_logger, rng=rng,
                         regularizer_factory=regularizer_factory)
        self.member_trainers = [
            BasicRewardTrainer(mp, loss=loss, batch_size=batch_size, minibatch_size=minibatch_size, epochs=epochs, lr=lr,
                               custom_logger=self.logger, regularizer_factory=regularizer_factory, rng=self.rng)
            for mp in self._preference_model.member_pref_models]

    # -- members over GPUs (SURVEY 8e: "RewardEnsemble ... could place members on different GPUs"; BASELINE config 5) ----
    _dist = None

    def set_distributed(self, group=None) -> None:
        """Member-parallel training over the ranks of a `torch.distributed` group (one process per GPU, every rank
        constructed with the same seeds and fed the same dataset): member k is trained by rank k % W, on exactly the
        bagging subset and minibatch order it has in a single-process run -- every rank draws every member's subset and
        makes the draws of the members it skips (`_skip_draws`) -- and after the last member the owners broadcast their
        members' parameters, RunningNorm statistics, AdamW state, regularizer strength and final statistics.  Every rank ends with all members, bit-identical to
        the single-process result.  Additive API: the reference trains the members one after the other in one process
        (:1417-1424)."""
        import torch.distributed as dist

        self._dist = (dist.get_world_size(group), dist.get_rank(group), group)

    def _sync_members(self) -> None:
        import torch.distributed as dist

        W, rank, group = self._dist
        trainers = self.member_trainers
        states = []
        for t in trainers:
            net = t._preference_model._fused_target()
            if net is None or not t.use_fused_step:
                raise NotImplementedError("member-parallel ensemble training needs members on the device-only step "
                                          "(fused reward networks, cross-entropy loss, AdamW)")
            e = net.engine()
            e.sync()
            states.append((e, t._fused_optimizer_state(e)))  # (creates the flat moments on the ranks that skipped it)
        # per member: loss, accuracy, step count, lambda, then FINAL_KEYS (NaN: not recorded); float64 holds the Python
        # floats exactly, the all-reduce adds only zeros to the owner's row
        keys = self.FINAL_KEYS
        meta = th.zeros(len(trainers), 4 + len(keys), dtype=th.float64, device=states[0][0].params.device)
        for k, (t, (e, fo)) in enumerate(zip(trainers, states)):
            src = k % W if group is None else dist.get_global_rank(group, k % W)
            for x in (e.params, fo["m"], fo["v"]) + ((e.norm_state, e.norm_count) if e.has_norm else ()):
                dist.broadcast(x, src=src, group=group)
            if k % W == rank:
                meta[k, 0], meta[k, 1] = t.last_epoch_stats["loss"], t.last_epoch_stats["accuracy"]
                meta[k, 2] = float(t.optim.state[e._param_list()[0]]["step"])
                meta[k, 3] = float(t.regularizer.lambda_) if t.regularizer is not None else 0.0
                meta[k, 4:] = th.tensor([t.final_stats.get(key, float("nan")) for key in keys], dtype=th.float64)
        dist.all_reduce(meta, group=group)
        meta = meta.cpu()
        for k, (t, (e, fo)) in enumerate(zip(trainers, states)):
            t.last_epoch_stats = {"loss": float(meta[k, 0]), "accuracy": float(meta[k, 1])}
            for p in e._param_list():
                t.optim.state[p]["step"] = th.tensor(float(meta[k, 2]))
            if t.regularizer is not None:
                t.regularizer.lambda_ = float(meta[k, 3])
            t.final_stats = {key: float(meta[k, 4 + j]) for j, key in enumerate(keys) if not math.isnan(meta[k, 4 + j])}

    def _train(self, dataset, epoch_multiplier: float = 1.0) -> None:
        sampler = data_th.RandomSampler(dataset, replacement=True, num_samples=len(dataset),
                                        generator=th.Generator().manual_seed(make_seeds(self.rng)))
        stats = defaultdict(list)
        W, rank = (self._dist[0], self._dist[1]) if self._dist is not None else (1, 0)
        for member_idx, trainer in enumerate(self.member_trainers):
            bagging_dataset = data_th.Subset(dataset, list(sampler))
            if member_idx % W == rank:
                trainer.train(bagging_dataset, epoch_multiplier=epoch_multiplier)
            else:  # another rank's member: make the draws its training makes from self.rng and torch's global RNG
                trainer._skip_draws(bagging_dataset, epoch_multiplier)
        if W > 1:
            self._sync_members()
        final = defaultdict(list)
        for trainer in self.member_trainers:
            for k, v in trainer.last_epoch_stats.items():
                stats[k].append(v)
            for k, v in trainer.final_stats.items():
                final[k].append(v)
        self.last_epoch_stats = {k: float(np.mean(v)) for k, v in stats.items()}
        for k, v in stats.items():
            self.logger.record(f"reward/final/train/{k}", float(np.mean(v)))
            self.logger.record(f"reward/final/train/{k}_std", float(np.std(v)))
        for k, v in final.items():  # the regularization keys: member mean and standard deviation (:1426-1438)
            self.logger.record(f"reward/final/{k}", float(np.mean(v)))
            self.logger.record(f"reward/final/{k}_std", float(np.std(v)))


def _make_reward_trainer(preference_model: PreferenceModel, loss: RewardLoss, rng: np.random.Generator,
                         reward_trainer_kwargs: Optional[Mapping[str, Any]] = None) -> RewardTrainer:
    kw = dict(reward_trainer_kwargs or {})
    if preference_model.ensemble_model is not None:
        return EnsembleTrainer(preference_model, loss, rng=rng, **kw)
    return BasicRewardTrainer(preference_model, loss=loss, rng=rng, **kw)


QUERY_SCHEDULES: Dict[str, Callable[[float], float]] = {
    "constant": lambda t: 1.0,
    "hyperbolic": lambda t: 1.0 / (1.0 + t),
    "inverse_quadratic": lambda t: 1.0 / (1.0 + t ** 2),
}


class PreferenceComparisons(base.BaseImitationAlgorithm):
    """The outer loop (:1482-1760): sample trajectories -> fragments -> preferences -> train the reward model -> train the
    agent; fixed-horizon check on the sampled trajectories and one logger dump per iteration like the reference."""

    def __init__(self, trajectory_generator: TrajectoryGenerator, reward_model: reward_nets.RewardNet,
                 num_iterations: int, fragmenter: Optional[Fragmenter] = None,
                 preference_gatherer: Optional[PreferenceGatherer] = None,
                 reward_trainer: Optional[RewardTrainer] = None, comparison_queue_size: Optional[int] = None,
                 fragment_length: int = 100, transition_oversampling: float = 1,
                 initial_comparison_frac: float = 0.1, initial_epoch_multiplier: float = 200.0,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None,
                 rng: Optional[np.random.Generator] = None,
                 query_schedule: Union[str, Callable[[float], float]] = "hyperbolic",
                 allow_variable_horizon: bool = False) -> None:
        super().__init__(custom_logger=custom_logger, allow_variable_horizon=allow_variable_horizon)
        if rng is None and not (fragmenter is not None and preference_gatherer is not None and reward_trainer is not None):
            raise ValueError("If you don't provide a random state, you must provide your own "
                             "seeded fragmenter, preference gatherer, and reward_trainer. ")
        self.rng = rng
        self.model = reward_model
        self.preference_model = PreferenceModel(reward_model)
        self.reward_trainer = reward_trainer or _make_reward_trainer(self.preference_model, CrossEntropyRewardLoss(), rng)
        self.reward_trainer.logger = self.logger
        self.trajectory_generator = trajectory_generator
        self.trajectory_generator.logger = self.logger
        self.fragmenter = fragmenter or RandomFragmenter(custom_logger=self.logger, rng=rng)
        self.preference_gatherer = preference_gatherer or SyntheticGatherer(custom_logger=self.logger, rng=rng)
        self.fragment_length = fragment_length
        self.initial_comparison_frac = initial_comparison_frac
        self.initial_epoch_multiplier = initial_epoch_multiplier
        self.num_iterations = num_iterations
        self.transition_oversampling = transition_oversampling
        if callable(query_schedule):
            self.query_schedule = query_schedule
        elif query_schedule in QUERY_SCHEDULES:
            self.query_schedule = QUERY_SCHEDULES[query_schedule]
        else:
            raise ValueError(f"Unknown query schedule: {query_schedule}")
        self.dataset = PreferenceDataset(max_size=comparison_queue_size)
        self._iteration = 0

    def train(self, total_timesteps: int, total_comparisons: int,
              callback: Optional[Callable[[int], None]] = None) -> Mapping[str, Any]:
        initial_comparisons = int(total_comparisons * self.initial_comparison_frac)
        total_comparisons -= initial_comparisons
        vec = np.array([self.query_schedule(t) for t in np.linspace(0, 1, self.num_iterations)])
        shares = (vec / vec.sum() * total_comparisons)
        schedule = [initial_comparisons] + [int(x) for x in _round_keep_sum(shares)]
        timesteps_per_iteration, extra = divmod(total_timesteps, self.num_iterations)
        reward_loss = reward_accuracy = None
        for i, num_pairs in enumerate(schedule):
            num_steps = math.ceil(self.transition_oversampling * 2 * num_pairs * self.fragment_length)
            self.logger.log(f"Collecting {2 * num_pairs} fragments ({num_steps} transitions)")
            trajectories = self.trajectory_generator.sample(num_steps)
            # (assumes no fragment misses initial timesteps, allows fragments that miss terminal ones)
            self._check_fixed_horizon(len(traj) for traj in trajectories if traj.terminal)
            fragments = self.fragmenter(trajectories, self.fragment_length, num_pairs)
            with self.logger.accumulate_means("preferences"):
                preferences = self.preference_gatherer(fragments)
            self.dataset.push(fragments, np.asarray(preferences, dtype=np.float32))
            epoch_multiplier = self.initial_epoch_multiplier if i == 0 else 1.0
            self.reward_trainer.train(self.dataset, epoch_multiplier=epoch_multiplier)
            stats = getattr(self.reward_trainer, "last_epoch_stats", {})
            reward_loss, reward_accuracy = stats.get("loss"), stats.get("accuracy")
            num_steps = timesteps_per_iteration + (extra if i == self.num_iterations - 1 else 0)
            with self.logger.accumulate_means("agent"):
                self.trajectory_generator.train(steps=num_steps)
            self.logger.dump(self._iteration)
            if callback:
                callback(self._iteration)
            self._iteration += 1
        return {"reward_loss": reward_loss, "reward_accuracy": reward_accuracy}


def _round_keep_sum(x: np.ndarray) -> np.ndarray:
    """Round to integers keeping the total (util.oric, :util.py)."""
    floor = np.floor(x)
    k = int(round(x.sum() - floor.sum()))
    order = np.argsort(-(x - floor), kind="stable")
    floor[order[:k]] += 1
    return floor.astype(int)
