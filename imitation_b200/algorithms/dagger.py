"""DAgger (mirror of imitation.algorithms.dagger).

Rounds of: roll the expert in the env, where with probability 1 - beta per env and step the learner's action is
executed instead (the expert's action is always the label), then `BC.train` on every transition collected so far.

On the lock-step, fixed-horizon `DeviceVecEnv` every collection batch is E whole episodes of H steps, and the host draws
from `rng` at steps known in advance: H calls of `uniform(size=E)` for the masks, then E calls of `bytes(16)` for the
file names at the batch's last step, then one `shuffle` after the last batch.  The mask never depends on observations,
so `InteractiveTrajectoryCollector` draws a batch's mask as uint8 [H][E] before its one `imb_rollout_dagger` launch
and the UUIDs after it; `rng` ends where the reference leaves it.

The demonstrations stay on the device: the collector keeps the rows (obs | label) of every file it writes, and
`_try_load_demos` appends each round's files, in the reference's listing order, to one aggregate table BC trains from;
only files the collector did not write are read back from disk (and uploaded once).

Known differences: the learner's sampled actions (and a stochastic expert's) come from Philox, not torch's generator;
files are written in the legacy `.npz` layout (`serialize.save` of a `.npz` path), which the reference's `load` reads.
"""
import abc
import os
import pathlib
import uuid
from typing import Any, Callable, Dict, List, Mapping, Optional, Sequence, Tuple, Union

import numpy as np
import torch as th

from .. import _lib
from ..data import rollout, serialize, types
from ..util import logger as imit_logger
from . import base, bc, dqn


class BetaSchedule(abc.ABC):
    """Computes beta (% of time demonstration action used) from training round."""

    @abc.abstractmethod
    def __call__(self, round_num: int) -> float:
        """The fraction of the time to sample a demonstrator action in round `round_num`."""


class LinearBetaSchedule(BetaSchedule):
    """Linearly-decreasing schedule for beta: 1 at round 0, 0 from round `rampdown_rounds` on."""

    def __init__(self, rampdown_rounds: int) -> None:
        self.rampdown_rounds = rampdown_rounds

    def __call__(self, round_num: int) -> float:
        assert round_num >= 0
        return min(1, max(0, (self.rampdown_rounds - round_num) / self.rampdown_rounds))


class ExponentialBetaSchedule(BetaSchedule):
    """Exponentially decaying schedule for beta: decay_probability ** round_num."""

    def __init__(self, decay_probability: float):
        if not (0 < decay_probability <= 1):
            raise ValueError("decay_probability lies outside the range (0, 1].")
        self.decay_probability = decay_probability

    def __call__(self, round_num: int) -> float:
        assert round_num >= 0
        return self.decay_probability**round_num


def reconstruct_trainer(scratch_dir, venv, custom_logger: Optional[imit_logger.HierarchicalLogger] = None,
                        device: Union[th.device, str] = "auto") -> "DAggerTrainer":
    """Reconstruct a trainer from `scratch_dir/checkpoint-latest.pt` (written by `save_trainer`)."""
    custom_logger = custom_logger or imit_logger.configure()
    checkpoint_path = pathlib.Path(scratch_dir) / "checkpoint-latest.pt"
    trainer = th.load(checkpoint_path, map_location=bc._device(device), weights_only=False)
    trainer.venv = venv
    trainer._logger = custom_logger
    trainer.bc_trainer._bc_logger._logger = trainer.bc_trainer.logger  # (BCLogger does not pickle its logger)
    return trainer


def demo_file_name(trajectory_index: int, rng: np.random.Generator, prefix: str = "") -> str:
    """`_save_dagger_demo`'s file name: one `rng.bytes(16)` draw for a version-4 UUID."""
    actual_prefix = f"{prefix}-" if prefix else ""
    random_uuid = uuid.UUID(int=int.from_bytes(rng.bytes(16), "big"), version=4).hex
    return f"{actual_prefix}dagger-demo-{trajectory_index}-{random_uuid}.npz"


def _save_dagger_demo(trajectory: types.Trajectory, trajectory_index: int, save_dir, rng: np.random.Generator,
                      prefix: str = "") -> pathlib.Path:
    save_dir = pathlib.Path(save_dir)
    assert isinstance(trajectory, types.Trajectory)
    npz_path = save_dir / demo_file_name(trajectory_index, rng, prefix)
    assert not npz_path.exists(), "The following DAgger demonstration path already exists: {0}".format(npz_path)
    serialize.save(npz_path, [trajectory])
    return npz_path


def draw_robot_mask(rng: np.random.Generator, n_steps: int, n_envs: int, beta: float) -> np.ndarray:
    """uint8 [n_steps][n_envs]: 1 where the learner acts, drawn as n_steps calls of the reference's step_async draw."""
    return np.stack([rng.uniform(0, 1, size=(n_envs,)) > beta for _ in range(n_steps)]).astype(np.uint8)


class _Rows:
    """A growing device table of rows (capacity doubles): `reserve(n)` returns a view of the next n rows to fill,
    `commit(n)` keeps them."""

    def __init__(self, width: int, device):
        self.n = 0
        self.table = th.zeros(0, width, device=device)

    def reserve(self, n: int) -> th.Tensor:
        if self.n + n > len(self.table):
            grown = th.zeros(max(2 * len(self.table), self.n + n), self.table.shape[1], device=self.table.device)
            grown[:self.n] = self.table[:self.n]
            self.table = grown
        return self.table[self.n:self.n + n]

    def commit(self, n: int) -> int:
        row0 = self.n
        self.n += n
        return row0


class InteractiveTrajectoryCollector:
    """DAgger's collector on the device env (dagger.py:165-287): `generate_trajectories(expert, collector, ...)` rolls
    the expert, with the learner's action executed for each env and step with probability 1 - beta, and writes each
    finished trajectory (the expert's actions as labels, the env's rewards) to `save_dir`.

    `policy` is the learner (an `ActorCriticPolicy`) in place of the reference's `get_robot_acts` callable, which has no
    device path.  `rows` is the table the rows of written files go to, `staged` the map from file path to (first row,
    row count) in it; the trainer passes its own so that aggregation reads the rows from the device."""

    def __init__(self, venv, policy, beta: float, save_dir, rng: np.random.Generator,
                 rows: Optional[_Rows] = None, staged: Optional[Dict[str, Tuple[int, int]]] = None) -> None:
        from ..envs import synth
        from ..policies import base as policies

        if not isinstance(policy, policies.ActorCriticPolicy):
            raise NotImplementedError("InteractiveTrajectoryCollector takes the learner policy: a host callable "
                                      "(get_robot_acts) cannot act inside the device rollout")
        base_env = venv
        while not isinstance(base_env, synth.DeviceVecEnv):
            if not hasattr(base_env, "venv"):
                raise TypeError("InteractiveTrajectoryCollector needs a DeviceVecEnv")
            base_env = base_env.venv
        assert 0 <= beta <= 1
        self.venv = venv
        self.base = base_env
        self.policy = policy
        self.beta = beta
        self.save_dir = save_dir
        self.rng = rng
        self.rows = rows if rows is not None else _Rows(_lib.rollout_row_width(policy.desc), base_env.device)
        self.staged = staged if staged is not None else {}

    @property
    def num_envs(self) -> int:
        return self.base.num_envs

    @property
    def observation_space(self):
        return self.base.observation_space

    @property
    def action_space(self):
        return self.base.action_space

    def seed(self, seed: Optional[int] = None) -> List[Optional[int]]:
        self.rng = np.random.default_rng(seed=seed)
        return [None] * self.num_envs

    def reset(self) -> np.ndarray:
        return self.base.reset()

    def step_async(self, actions):
        raise NotImplementedError("the DAgger collector steps the DeviceVecEnv inside one rollout launch per batch of "
                                  "episodes: call rollout.generate_trajectories(expert, collector, ...)")

    def step_wait(self):
        raise NotImplementedError("see step_async")


    def generate_trajectories(self, expert, sample_until, rng: np.random.Generator, *, deterministic_policy: bool = False,
                              noise=None, robot_noise=None) -> Sequence[types.TrajectoryWithRew]:
        """`rollout.generate_trajectories(expert, self, ...)`: batches of E whole episodes until `sample_until` holds,
        each one launch; every finished trajectory saved in env order; then `rng.shuffle`.  noise / robot_noise (tests)
        pin the expert's and the learner's sampling of every batch ([H][E][d_act] normals or [H][E] uniforms)."""
        env, learner = self.base, self.policy
        exp = rollout._policy_of(expert)
        if isinstance(exp, dqn.DQNPolicy):  # SB3's QNetwork._predict takes the argmax whatever `deterministic` says
            deterministic_policy = True
        ep, en, _ = exp.flat_vectors()
        lp, ln, _ = learner.flat_vectors()
        E, H, Do = env.num_envs, env.horizon, env.d_obs
        rw = _lib.rollout_row_width(learner.desc)
        env.reset()
        flat = th.zeros(E * H, 2 * Do + env.d_act + 1, device=env.device)
        aux = th.zeros(2 * E + 2 * E * H, device=env.device)
        nz = None if noise is None else th.as_tensor(np.ascontiguousarray(noise)).to(env.device)
        rnz = None if robot_noise is None else th.as_tensor(np.ascontiguousarray(robot_noise)).to(env.device)
        os.makedirs(self.save_dir, exist_ok=True)
        trajectories: List[types.TrajectoryWithRew] = []
        robot_acted = False
        while True:
            mask = draw_robot_mask(self.rng, H, E, self.beta)
            robot_acted |= bool(mask.any())
            tbl = self.rows.reserve(E * H)
            _lib.rollout_dagger(env.desc, env.params, env.obs, exp.desc, ep, en, learner.desc, lp, ln, E, H, tbl, flat,
                                aux, nz, rnz, th.as_tensor(mask).to(env.device), env.state,
                                flags=_lib.IMB_RF_DETERMINISTIC if deterministic_policy else 0, expert_act=exp.act,
                                learner_act=learner.act)
            _lib.rollout_advance(env.state, E, H, H, 0)
            env.host_ep_step = 0
            row0 = self.rows.commit(E * H)
            batch = rollout.batch_trajectories(env, tbl, flat, aux)
            for e, traj in enumerate(batch):
                path = _save_dagger_demo(traj, e, self.save_dir, self.rng)
                self.staged[os.fspath(path)] = (row0 + e * H, H)
            assert rw == tbl.shape[1]
            trajectories += batch
            if sample_until(trajectories):
                break
        rng.shuffle(trajectories)
        # policy.predict leaves a policy in evaluation mode; the learner is only asked where the mask was set
        exp.set_training_mode(False)
        if robot_acted:
            learner.set_training_mode(False)
        return trajectories


class NeedsDemosException(Exception):
    """Signals demos need to be collected for current round before continuing."""


class DAggerTrainer(base.BaseImitationAlgorithm):
    """DAgger with the reference's low-level API (dagger.py:294-608): rounds of `create_trajectory_collector` +
    `generate_trajectories`, then `extend_and_update`, with demonstrations under `scratch_dir/demos/round-NNN/`."""

    DEFAULT_N_EPOCHS: int = 4

    def __init__(self, *, venv, scratch_dir, rng: np.random.Generator,
                 beta_schedule: Optional[Callable[[int], float]] = None, bc_trainer: bc.BC,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None):
        super().__init__(custom_logger=custom_logger)
        if beta_schedule is None:
            beta_schedule = LinearBetaSchedule(15)
        self.beta_schedule = beta_schedule
        self.scratch_dir = pathlib.Path(scratch_dir)
        self.venv = venv
        self.round_num = 0
        self._last_loaded_round = -1
        self.rng = rng
        if venv.observation_space != bc_trainer.observation_space:
            raise ValueError(f"Observation spaces do not match: {venv.observation_space} != "
                             f"{bc_trainer.observation_space}")
        if venv.action_space != bc_trainer.action_space:
            raise ValueError(f"Action spaces do not match: {venv.action_space} != {bc_trainer.action_space}")
        self.bc_trainer = bc_trainer
        self.bc_trainer.logger = self.logger
        width = _lib.rollout_row_width(bc_trainer.policy.desc)
        self._rows = _Rows(width, bc_trainer._dev)       # rows of every demonstration file the trainer has seen
        self._staged: Dict[str, Tuple[int, int]] = {}   # file path -> (first row, rows) in self._rows
        self._all_rows = _Rows(width, bc_trainer._dev)   # the aggregate: every loaded round's rows, in listing order

    def __getstate__(self):
        d = dict(self.__dict__)
        del d["venv"]
        del d["_logger"]
        return d

    @property
    def logger(self) -> imit_logger.HierarchicalLogger:
        return super().logger

    @logger.setter
    def logger(self, value: imit_logger.HierarchicalLogger) -> None:
        # DAgger and inner-BC logger should stay in sync
        self._logger = value
        self.bc_trainer.logger = value

    @property
    def policy(self):
        return self.bc_trainer.policy

    @property
    def batch_size(self) -> int:
        return self.bc_trainer.batch_size

    def _get_demo_paths(self, round_dir: pathlib.Path) -> List[pathlib.Path]:
        return [round_dir / f for f in sorted(os.listdir(round_dir)) if f.endswith(".npz")]

    def _demo_dir_path_for_round(self, round_num: Optional[int] = None) -> pathlib.Path:
        if round_num is None:
            round_num = self.round_num
        return self.scratch_dir / "demos" / f"round-{round_num:03d}"

    def _rows_of(self, path: pathlib.Path) -> Tuple[int, int]:
        """(first row, rows) of a demonstration file in self._rows: the collector's rows, or the file's first
        trajectory read from disk and uploaded once."""
        key = os.fspath(path)
        if key not in self._staged:
            traj = serialize.load(path)[0]
            table = bc.demo_table(self.policy, traj.obs[:-1], traj.acts)
            self._rows.reserve(len(table)).copy_(table)
            self._staged[key] = (self._rows.commit(len(table)), len(table))
        return self._staged[key]

    def _load_all_demos(self) -> List[int]:
        """Append rounds _last_loaded_round + 1 .. round_num to the aggregate table, in listing order (one gather per
        round); returns the number of files of each round."""
        num_demos_by_round = []
        for round_num in range(self._last_loaded_round + 1, self.round_num + 1):
            round_dir = self._demo_dir_path_for_round(round_num)
            demo_paths = self._get_demo_paths(round_dir)
            idx = [np.arange(r0, r0 + n) for r0, n in map(self._rows_of, demo_paths)]
            if idx:
                idx_dev = th.as_tensor(np.concatenate(idx), dtype=th.int64, device=self._rows.table.device)
                dst = self._all_rows.reserve(len(idx_dev))
                th.index_select(self._rows.table, 0, idx_dev, out=dst)
                self._all_rows.commit(len(idx_dev))
            num_demos_by_round.append(len(demo_paths))
        return num_demos_by_round

    def _try_load_demos(self) -> None:
        """Load the dataset for this round into self.bc_trainer, shuffled every epoch as the reference's DataLoader."""
        demo_dir = self._demo_dir_path_for_round()
        demo_paths = self._get_demo_paths(demo_dir) if demo_dir.is_dir() else []
        if len(demo_paths) == 0:
            raise NeedsDemosException(f"No demos found for round {self.round_num} in dir '{demo_dir}'. Maybe you need "
                                      "to collect some demos? See .create_trajectory_collector()")
        if self._last_loaded_round < self.round_num:
            self._load_all_demos()
            n = self._all_rows.n
            if n < self.batch_size:
                raise ValueError("Not enough transitions to form a single batch: "
                                 f"self.batch_size={self.batch_size} > len(transitions)={n}")
            self.bc_trainer._set_demonstration_rows(self._all_rows.table, n, self.batch_size)
            self._last_loaded_round = self.round_num

    def extend_and_update(self, bc_train_kwargs: Optional[Mapping[str, Any]] = None) -> int:
        """Load new transitions (if necessary), train BC, and advance the round counter (dagger.py:468-509)."""
        bc_train_kwargs = {} if bc_train_kwargs is None else dict(bc_train_kwargs)
        user_keys = bc_train_kwargs.keys()
        if "log_rollouts_venv" not in user_keys:
            bc_train_kwargs["log_rollouts_venv"] = self.venv
        if "n_epochs" not in user_keys and "n_batches" not in user_keys:
            bc_train_kwargs["n_epochs"] = self.DEFAULT_N_EPOCHS
        self._try_load_demos()
        self.bc_trainer.train(**bc_train_kwargs)
        self.round_num += 1
        return self.round_num

    def create_trajectory_collector(self) -> InteractiveTrajectoryCollector:
        """A collector for the current round: its beta, the learner, this round's directory, the trainer's rng."""
        return InteractiveTrajectoryCollector(venv=self.venv, policy=self.bc_trainer.policy,
                                              beta=self.beta_schedule(self.round_num),
                                              save_dir=self._demo_dir_path_for_round(), rng=self.rng,
                                              rows=self._rows, staged=self._staged)

    def save_trainer(self) -> Tuple[pathlib.Path, pathlib.Path]:
        """`th.save` the trainer (BC's optimiser state and the device tables included) to checkpoint-NNN.pt and
        checkpoint-latest.pt, and the policy to policy-NNN.pt and policy-latest.pt."""
        self.scratch_dir.mkdir(parents=True, exist_ok=True)
        checkpoint_paths = [self.scratch_dir / f"checkpoint-{self.round_num:03d}.pt",
                            self.scratch_dir / "checkpoint-latest.pt"]
        for checkpoint_path in checkpoint_paths:
            th.save(self, checkpoint_path)
        policy_paths = [self.scratch_dir / f"policy-{self.round_num:03d}.pt", self.scratch_dir / "policy-latest.pt"]
        for policy_path in policy_paths:
            th.save(self.policy, policy_path)
        return checkpoint_paths[0], policy_paths[0]


class SimpleDAggerTrainer(DAggerTrainer):
    """DAggerTrainer with synthetic feedback from `expert_policy` (dagger.py:611-694)."""

    def __init__(self, *, venv, scratch_dir, expert_policy, rng: np.random.Generator,
                 expert_trajs: Optional[Sequence[types.Trajectory]] = None, **dagger_trainer_kwargs):
        super().__init__(venv=venv, scratch_dir=scratch_dir, rng=rng, **dagger_trainer_kwargs)
        self.expert_policy = expert_policy
        if expert_policy.observation_space != self.venv.observation_space:
            raise ValueError("Mismatched observation space between expert_policy and venv")
        if expert_policy.action_space != self.venv.action_space:
            raise ValueError("Mismatched action space between expert_policy and venv")
        if expert_trajs is not None:
            for traj_index, traj in enumerate(expert_trajs):
                _save_dagger_demo(traj, traj_index, self._demo_dir_path_for_round(), self.rng, prefix="initial_data")

    def train(self, total_timesteps: int, *, rollout_round_min_episodes: int = 3,
              rollout_round_min_timesteps: int = 500, bc_train_kwargs: Optional[dict] = None) -> None:
        """Rounds of collection (rollout_round_min_* and at least batch_size timesteps) and BC until total_timesteps
        env steps have been collected."""
        total_timestep_count = 0
        round_num = 0
        while total_timestep_count < total_timesteps:
            collector = self.create_trajectory_collector()
            round_episode_count = 0
            round_timestep_count = 0
            sample_until = rollout.make_sample_until(min_timesteps=max(rollout_round_min_timesteps, self.batch_size),
                                                     min_episodes=rollout_round_min_episodes)
            trajectories = rollout.generate_trajectories(policy=self.expert_policy, venv=collector,
                                                         sample_until=sample_until, deterministic_policy=True,
                                                         rng=collector.rng)
            for traj in trajectories:
                self._logger.record_mean("dagger/mean_episode_reward", np.sum(traj.rews))
                round_timestep_count += len(traj)
                total_timestep_count += len(traj)
            round_episode_count += len(trajectories)
            self._logger.record("dagger/total_timesteps", total_timestep_count)
            self._logger.record("dagger/round_num", round_num)
            self._logger.record("dagger/round_episode_count", round_episode_count)
            self._logger.record("dagger/round_timestep_count", round_timestep_count)
            # `logger.dump` is called inside BC.train within the following fn call:
            self.extend_and_update(bc_train_kwargs)
            round_num += 1
