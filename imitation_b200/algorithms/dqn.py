"""A device DQN: SB3 2.2's `DQN` (stable_baselines3/dqn/dqn.py) as far as SQIL trains it.

SB3 is not a dependency, so its semantics are restated here, from SB3 2.2.x, as oracle/sqil_port.py restates them
(unpinned: re-verify wherever SB3 is installed):

- `learn(total_timesteps, reset_num_timesteps=True)` resets the step counts and the env, then alternates collecting
  `train_freq` VecEnv steps with `gradient_steps` TD steps (-1: as many as were collected), the latter only once
  `num_timesteps > learning_starts`.
- Per collected step: act, step, `num_timesteps += n_envs`, store the transition (the horizon's done counts as terminal,
  next_obs is the terminal observation), update the remaining progress, then `_on_step`: every
  `max(target_update_interval // n_envs, 1)` calls a polyak update with `tau`, then
  `exploration_rate = get_linear_fn(initial, final, fraction)(progress_remaining)`.
- Acting: before `learning_starts` every env takes `action_space.sample()`; after it one `np.random.rand() <
  exploration_rate` draw per step makes every env or none act at random, the others take the argmax of the Q-net.
- TD step: the replay buffer's sample, `y = r + (1 - d) gamma max_a Q_target(s')`, `F.smooth_l1_loss(Q(s)[a], y)`,
  `clip_grad_norm_(max_grad_norm)`, torch Adam (lr, eps 1e-8).

On the device, one `learn()` is one host pass that draws every global-numpy number in SB3's order (the random-step
vector, the learner and expert sample indices) and computes the target-update steps and exploration rates; then per
iteration: the exploration rollout (`imb_rollout_explore`, argmax on the policy steps), the ring store
(`imb_dqn_ring_store`, into the feature-major learner ring in SB3's (position, env) order), the target updates (a copy
of the flat vector for tau = 1, else SB3's mul / add), the TD targets (`imb_dqn_target`) and the TD steps
(`imb_dqn_step`).  Every per-iteration offset is read from a device counter, so each iteration after the first of its
kind replays from a CUDA graph.  Nothing is read back inside `learn()` but the losses, once at its end.  The random
actions come from the exploration rollout's Philox stream at the env's global step: the same distribution as
`action_space.sample()`, not its bits.
"""
from typing import NamedTuple, Optional

import numpy as np
import torch as th
from torch import nn

from .. import _desc, _lib
from ..policies import base as policy_base
from ..util import logger as imit_logger
from ..util.flat import FlatAlias


class QNetwork(nn.Module):
    """SB3's QNetwork for a flat observation: Flatten -> [Linear -> act] x 2 -> Linear(h, n_actions)."""

    def __init__(self, d_obs: int, n_actions: int, hidden: int, activation_fn):
        super().__init__()
        self.features_extractor = policy_base.FlattenExtractor()
        self.q_net = nn.Sequential(nn.Linear(d_obs, hidden), activation_fn(), nn.Linear(hidden, hidden),
                                   activation_fn(), nn.Linear(hidden, n_actions))

    def forward(self, obs):
        return self.q_net(self.features_extractor(obs))


class DQNPolicy(nn.Module):
    """SB3's DQNPolicy ("MlpPolicy") over two flat device vectors, one per Q-net.

    Each Q-net is a policy image (imb.h, imb_policy_desc): its layers are the pi tower and the action head, and the
    value tower and value head are zero tensors no module owns (their gradient is 0, so they stay 0).  The state_dict
    is SB3's: q_net.q_net.{0,2,4}.* and q_net_target.q_net.*."""

    def __init__(self, observation_space, action_space, lr_schedule=None, net_arch=None, activation_fn=nn.ReLU,
                 features_extractor_class=None, features_extractor_kwargs=None, normalize_images: bool = True,
                 optimizer_class=th.optim.Adam, optimizer_kwargs: Optional[dict] = None):
        super().__init__()
        from .. import spaces

        if not spaces.is_discrete(action_space):
            raise NotImplementedError(f"action space {action_space!r}: the device DQN runs Discrete action spaces "
                                      "(continuous-action SQIL needs SAC / TD3 / DDPG, which have no device port)")
        net_arch = [64, 64] if net_arch is None else list(net_arch)
        hidden = policy_base._tower_width(net_arch)
        if activation_fn not in policy_base._ACTIVATIONS:
            raise NotImplementedError(f"activation_fn {activation_fn!r}: the DQN step runs nn.Tanh and nn.ReLU Q-nets")
        if features_extractor_class not in (None, policy_base.FlattenExtractor) or features_extractor_kwargs:
            raise NotImplementedError("features_extractor_class: the DQN step runs Flatten features")
        if optimizer_class is not th.optim.Adam or optimizer_kwargs not in (None, {}):
            raise NotImplementedError("optimizer_class / optimizer_kwargs: the DQN step runs torch Adam with its "
                                      "defaults (eps 1e-8)")
        self.observation_space, self.action_space = observation_space, action_space
        self.d_obs, self.d_act, self.discrete, self.hidden = spaces.flat_dim(observation_space), int(action_space.n), \
            True, hidden
        self.act = policy_base._ACTIVATIONS[activation_fn]
        self.normalize_features = False
        # SB3's order: q_net, then q_net_target, then the copy (torch's default Linear init in both)
        self.q_net = QNetwork(self.d_obs, self.d_act, hidden, activation_fn)
        self.q_net_target = QNetwork(self.d_obs, self.d_act, hidden, activation_fn)
        self.q_net_target.load_state_dict(self.q_net.state_dict())
        self.q_net_target.train(False)
        self.desc = _desc.policy_desc(self.d_obs, self.d_act, True, hidden, False)

    def _aliases(self):
        al = self.__dict__.get("_flat_aliases")
        if al is None:
            al = [self._alias(self.q_net), self._alias(self.q_net_target)]
            self.__dict__["_flat_aliases"] = al
        return al

    def _alias(self, qn: QNetwork) -> FlatAlias:
        h, Do = self.hidden, self.d_obs
        holder = nn.Module()  # the value tower and head of the policy image: owned by no registered module
        for name, shape in (("w1", (h, Do)), ("b1", (h,)), ("w2", (h, h)), ("b2", (h,)), ("wv", (1, h)), ("bv", (1,))):
            holder.register_buffer(name, th.zeros(shape, device=qn.q_net[0].weight.device))
        self.__dict__.setdefault("_vf_holders", []).append(holder)
        l0, l2, l4 = qn.q_net[0], qn.q_net[2], qn.q_net[4]
        return FlatAlias([(l0, "weight"), (l0, "bias"), (l2, "weight"), (l2, "bias"), (holder, "w1"), (holder, "b1"),
                          (holder, "w2"), (holder, "b2"), (l4, "weight"), (l4, "bias"), (holder, "wv"),
                          (holder, "bv")])

    def _flat(self, i: int) -> th.Tensor:
        al = self._aliases()[i]
        dev = al.tensors()[0].device
        if dev.type != "cuda":
            raise _lib.ImbError("the device DQN runs on CUDA only (no CPU fallback)")
        flat = al.get(th.float32, dev)
        assert flat.numel() == self.desc.n_params
        return flat

    def q_flat(self) -> th.Tensor:
        """The Q-net's flat policy image (the kernels' parameter vector)."""
        return self._flat(0)

    def target_flat(self) -> th.Tensor:
        return self._flat(1)

    def flat_vectors(self):
        """(params, norm_state, norm_count) of the Q-net as a policy image, for the rollout kernels (no feature norm)."""
        flat = self.q_flat()
        ns = self.__dict__.get("_norm_state")
        if ns is None or ns.device != flat.device:
            self.__dict__["_norm_state"] = th.zeros(2, device=flat.device)
            self.__dict__["_norm_count"] = th.zeros(1, dtype=th.int32, device=flat.device)
        return flat, self._norm_state, self._norm_count

    def __getstate__(self):
        st = self.__dict__.copy()
        for k in ("_flat_aliases", "_vf_holders", "_norm_state", "_norm_count"):
            st.pop(k, None)
        return st

    def set_training_mode(self, mode: bool) -> None:
        self.q_net.train(mode)

    def forward(self, obs, deterministic: bool = True):
        return self._predict(obs, deterministic)

    def _predict(self, obs, deterministic: bool = True):
        return self.q_net(obs).argmax(dim=1).reshape(-1)

    def predict(self, observation, state=None, episode_start=None, deterministic: bool = False):
        """The argmax of the Q-net (SB3's QNetwork._predict ignores `deterministic`)."""
        obs = th.as_tensor(np.asarray(observation, np.float32)).to(self.q_net.q_net[0].weight.device)
        with th.no_grad():
            acts = self._predict(obs.reshape(-1, self.d_obs))
        return acts.cpu().numpy(), state


MlpPolicy = DQNPolicy


def linear_schedule(start: float, end: float, end_fraction: float):
    """SB3's get_linear_fn."""
    def func(progress_remaining: float) -> float:
        if (1 - progress_remaining) > end_fraction:
            return end
        return start + (1 - progress_remaining) * (end - start) / end_fraction
    return func


class LearnSchedule(NamedTuple):
    """Every draw and host-known event of one learn(), in SB3's order (see `learn_schedule`)."""
    explore: np.ndarray        # uint8 [n_iter * T]: step is a random-policy step
    rates: np.ndarray          # float64 [n_iter * T]: exploration_rate after each step's _on_step
    target_updates: np.ndarray  # int64 [n_iter]: polyak updates during the iteration's collection
    grad_steps: np.ndarray     # int64 [n_iter]: TD steps after the iteration
    learner_idx: np.ndarray    # int64 [sum grad_steps][n_l]: ring column pos * n_envs + env of each learner row
    expert_idx: np.ndarray     # int64 [sum grad_steps][n_e]
    pos: np.ndarray            # int64 [n_iter]: ring position of the iteration's first step
    n_calls: int               # _n_calls after the learn
    full: bool                 # ring full after the learn
    num_timesteps: int


def learn_schedule(total_timesteps: int, n_envs: int, train_freq: int, gradient_steps: int, learning_starts: int,
                   batch_size: int, buffer_positions: int, pos: int, full: bool, n_expert: int,
                   target_update_interval: int, n_calls: int, exploration_rate: float, rate_fn,
                   num_timesteps: int = 0, exploration_draws: bool = True) -> LearnSchedule:
    """The host pass of one learn(): every global-numpy draw in SB3's order (np.random.rand per step after
    learning_starts; per TD step the learner's randint(0, upper) and randint(0, n_envs), then the expert's randint(0,
    n_expert)), the target-update calls, the exploration rates and the ring positions.  exploration_draws False (SAC,
    which acts without epsilon-greedy draws): a step is random exactly before learning_starts, and the only draws are
    the replay indices."""
    E, T, P = n_envs, train_freq, buffer_positions
    n_l, n_e = batch_size // 2, batch_size - batch_size // 2
    every = max(target_update_interval // E, 1)
    explore, rates, tu, gsteps, lidx, eidx, poss = [], [], [], [], [], [], []
    while num_timesteps < total_timesteps:
        poss.append(pos)
        ups = 0
        for _ in range(T):
            if num_timesteps < learning_starts:
                explore.append(1)
            elif not exploration_draws:
                explore.append(0)
            else:
                explore.append(1 if np.random.rand() < exploration_rate else 0)
            num_timesteps += E
            pos += 1
            if pos == P:
                full, pos = True, 0
            progress = 1.0 - float(num_timesteps) / float(total_timesteps)
            n_calls += 1
            if n_calls % every == 0:
                ups += 1
            exploration_rate = rate_fn(progress)
            rates.append(exploration_rate)
        tu.append(ups)
        g = 0
        if num_timesteps > 0 and num_timesteps > learning_starts:
            g = gradient_steps if gradient_steps >= 0 else T * E
            for _ in range(g):
                upper = P if full else pos
                bi = np.random.randint(0, upper, size=n_l)
                ei = np.random.randint(0, E, size=(n_l,))
                lidx.append(bi.astype(np.int64) * E + ei)
                eidx.append(np.random.randint(0, n_expert, size=n_e).astype(np.int64))
        gsteps.append(g)
    cat = lambda xs, w: np.stack(xs).astype(np.int64) if xs else np.zeros((0, w), np.int64)
    return LearnSchedule(np.asarray(explore, np.uint8), np.asarray(rates, np.float64), np.asarray(tu, np.int64),
                         np.asarray(gsteps, np.int64), cat(lidx, n_l), cat(eidx, n_e), np.asarray(poss, np.int64),
                         n_calls, full, num_timesteps)


class DeviceDQN:
    """SB3 2.2's DQN constructor, defaults and learn(), on the device.  SQIL's buffer (`SQILReplayBuffer`) is the
    replay buffer it trains from: its constant rewards are what the TD-target kernel reads."""

    def __init__(self, policy, env, learning_rate=1e-4, buffer_size: int = 1_000_000, learning_starts: int = 100,
                 batch_size: int = 32, tau: float = 1.0, gamma: float = 0.99, train_freq=4, gradient_steps: int = 1,
                 replay_buffer_class=None, replay_buffer_kwargs: Optional[dict] = None,
                 optimize_memory_usage: bool = False, target_update_interval: int = 10_000,
                 exploration_fraction: float = 0.1, exploration_initial_eps: float = 1.0,
                 exploration_final_eps: float = 0.05, max_grad_norm: float = 10, stats_window_size: int = 100,
                 tensorboard_log=None, policy_kwargs: Optional[dict] = None, verbose: int = 0,
                 seed: Optional[int] = None, device="auto", _init_setup_model: bool = True):
        from ..envs import synth
        from . import sqil

        if callable(learning_rate):
            raise NotImplementedError("a callable learning_rate: the DQN step runs a constant learning rate")
        if optimize_memory_usage:
            raise NotImplementedError("optimize_memory_usage=True: the device ring stores next_obs beside obs")
        if isinstance(train_freq, tuple):
            n, unit = train_freq
            if unit != "step":
                raise NotImplementedError(f"train_freq {train_freq!r}: the device DQN collects whole VecEnv steps "
                                          "(train_freq in episodes is not supported)")
            train_freq = n
        if not isinstance(env, synth.DeviceVecEnv):
            raise NotImplementedError("the device DQN steps a DeviceVecEnv (imitation_b200.envs.make_vec_env)")
        if not env.discrete:
            raise NotImplementedError("Box action spaces: the device DQN runs Discrete action spaces")
        if replay_buffer_class is not sqil.SQILReplayBuffer:
            raise NotImplementedError(f"replay_buffer_class {replay_buffer_class!r}: the device DQN trains from "
                                      "SQILReplayBuffer (its TD targets read constant rewards)")
        self.env = env
        self.n_envs = env.num_envs
        self.learning_rate = float(learning_rate)
        self.buffer_size, self.learning_starts, self.batch_size = int(buffer_size), int(learning_starts), int(batch_size)
        self.tau, self.gamma, self.train_freq = float(tau), float(gamma), int(train_freq)
        self.gradient_steps, self.target_update_interval = int(gradient_steps), int(target_update_interval)
        self.exploration_fraction = exploration_fraction
        self.exploration_initial_eps, self.exploration_final_eps = exploration_initial_eps, exploration_final_eps
        self.max_grad_norm = float(max_grad_norm)
        self.seed = seed
        self.policy_kwargs = dict(policy_kwargs or {})
        self.exploration_schedule = linear_schedule(exploration_initial_eps, exploration_final_eps, exploration_fraction)
        self.exploration_rate = 0.0
        self.num_timesteps = 0
        self._n_calls = 0
        self._n_updates = 0
        self._episode_num = 0
        self.graph_replays = 0  # iterations replayed from a CUDA graph, and the kernels those replays ran
        self.graph_kernels = 0
        self._logger = imit_logger.configure()
        if self.seed is not None:  # BaseAlgorithm.set_random_seed, before the policy is built
            np.random.seed(self.seed)
            th.manual_seed(self.seed)
        if isinstance(policy, str):
            if policy != "MlpPolicy":
                raise NotImplementedError(f"policy {policy!r}: the device DQN runs MlpPolicy")
            policy = DQNPolicy
        if policy is not DQNPolicy:
            raise NotImplementedError(f"policy {policy!r}: the device DQN runs its MlpPolicy (DQNPolicy)")
        policy = DQNPolicy(env.observation_space, env.action_space, **self.policy_kwargs)
        try:
            _lib.dqn_plan(policy.desc, self.batch_size, policy.act)
        except _lib.ImbError as e:
            raise NotImplementedError(f"batch_size {self.batch_size} with this Q-net: {e}") from None
        if isinstance(device, str) and device == "auto":
            device = "cuda"
        self.device = th.device(device)
        if self.device.type != "cuda":
            raise NotImplementedError(f"device {device!r}: the device DQN trains on the GPU only")
        self.policy = policy.to(self.device)
        self.replay_buffer = replay_buffer_class(self.buffer_size, env.observation_space, env.action_space,
                                                 n_envs=self.n_envs, device=self.device,
                                                 **dict(replay_buffer_kwargs or {}))
        n = self.policy.desc.n_params
        self.exp_avg = th.zeros(n, device=self.device)
        self.exp_avg_sq = th.zeros(n, device=self.device)
        self._state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device=self.device)
        self.hp = _lib.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=0.2, ent_coef=0.0, vf_coef=0.5,
                                  max_grad_norm=0.5, lr=0.0, adam_eps=1e-5, n_epochs=1, batch_size=1,
                                  normalize_advantage=0)
        self.last_schedule: Optional[LearnSchedule] = None

    @property
    def q_net(self) -> QNetwork:
        return self.policy.q_net

    @property
    def q_net_target(self) -> QNetwork:
        return self.policy.q_net_target

    @property
    def logger(self):
        return self._logger

    def set_logger(self, logger) -> None:
        self._logger = logger

    def predict(self, observation, state=None, episode_start=None, deterministic: bool = False):
        """SB3's DQN.predict: with probability exploration_rate (unless deterministic) random actions, else the
        argmax (host path)."""
        if not deterministic and np.random.rand() < self.exploration_rate:
            obs = np.asarray(observation)
            n = obs.shape[0] if obs.ndim > 1 else 1
            return np.array([self.env.action_space.sample() for _ in range(n)]), state
        return self.policy.predict(observation, state, episode_start, deterministic)

    def _target_update(self) -> None:
        q, tgt = self.policy.q_flat(), self.policy.target_flat()
        if self.tau == 1.0:
            tgt.copy_(q)
        else:  # polyak_update: th.mul(t, 1 - tau, out=t); th.add(t, p, alpha=tau, out=t)
            tgt.mul_(1 - self.tau)
            tgt.add_(q, alpha=self.tau)

    def learn(self, total_timesteps: int, callback=None, log_interval: int = 4, tb_log_name: str = "DQN",
              reset_num_timesteps: bool = True, progress_bar: bool = False):
        if callback is not None:
            raise NotImplementedError("callback: the device DQN runs the collection inside the rollout kernel")
        env, buf, pol = self.env, self.replay_buffer, self.policy
        if buf.n_expert == 0:
            raise ValueError("SQIL needs demonstrations")
        if reset_num_timesteps:
            self.num_timesteps = 0
            self._episode_num = 0
            total = int(total_timesteps)
            env.reset()
        else:
            total = int(total_timesteps) + self.num_timesteps
            env.ensure_reset()
        E, T, H = self.n_envs, self.train_freq, env.horizon
        s = learn_schedule(total, E, T, self.gradient_steps, self.learning_starts, self.batch_size, buf.buffer_size,
                           buf.pos, buf.full, buf.n_expert, self.target_update_interval, self._n_calls,
                           self.exploration_rate, self.exploration_schedule, self.num_timesteps)
        self.last_schedule = s
        n_iter = len(s.grad_steps)
        if n_iter == 0:
            return self
        dev = self.device
        B = self.batch_size
        n_td = int(s.grad_steps.sum())
        # the device counters every launch reads its per-iteration offsets from: the env's global step (random-step
        # vector, Philox counter), the ring's position, the Adam step count (sample lists, loss rows)
        g0 = int(env.state[_lib.ST_GLOBAL_STEP])
        buf.sync_ring_state()
        td0 = self._n_updates
        self._state[_lib.ST_PPO_STEP] = td0
        self._x = dict(explore=th.as_tensor(s.explore).to(dev), lidx=th.as_tensor(s.learner_idx).to(dev),
                       eidx=th.as_tensor(s.expert_idx).to(dev), loss=th.zeros(max(n_td, 1), 4, device=dev),
                       g0=g0, td0=td0)
        rw = _lib.rollout_row_width(self.policy.desc)
        tw = 2 * env.d_obs + env.d_act + 1
        if getattr(self, "_tbl", None) is None or self._tbl.shape[0] != E * T:
            self._tbl = th.zeros(E * T, rw, device=dev)
            self._flat = th.zeros(E * T, tw, device=dev)
            self._aux = th.zeros(2 * E + 2 * E * T, device=dev)
        gmax = int(s.grad_steps.max())
        if getattr(self, "_td_rows", None) is None or self._td_rows.shape[0] < gmax * B:
            self._td_rows = th.zeros(max(gmax, 1) * B, rw, device=dev)
        # one graph per iteration kind (TD steps, target updates), captured at the kind's second iteration and
        # replayed from then on; the graphs bake in this learn()'s vectors, so they live for one learn()
        graphs, seen = {}, set()
        for k in range(n_iter):
            key = (int(s.grad_steps[k]), int(s.target_updates[k]))
            if key in graphs:
                graphs[key][0].replay()
                _lib.LAUNCHES["count"] += graphs[key][1]
                self.graph_replays += 1
                self.graph_kernels += graphs[key][1]
            elif key in seen:
                before = _lib.LAUNCHES["count"]
                g = th.cuda.CUDAGraph()
                with th.cuda.graph(g):
                    self._iteration(*key)
                graphs[key] = (g, _lib.LAUNCHES["count"] - before)
                _lib.LAUNCHES["count"] = before
                g.replay()
                _lib.LAUNCHES["count"] += graphs[key][1]
                self.graph_replays += 1
                self.graph_kernels += graphs[key][1]
            else:
                self._iteration(*key)
                seen.add(key)
            env.host_ep_step = (env.host_ep_step + T) % H
        loss_log = self._x["loss"]
        # host mirrors of what the device did
        self.num_timesteps = s.num_timesteps
        self._n_calls = s.n_calls
        self.exploration_rate = float(s.rates[-1])
        buf.pos = (int(s.pos[-1]) + T) % buf.buffer_size
        buf.full = s.full
        self._n_updates += n_td
        logged = {"rollout/exploration_rate": self.exploration_rate}
        if n_td:  # train/loss: the mean over the last train() call's steps, as SB3 leaves it recorded
            last = int(s.grad_steps[np.nonzero(s.grad_steps)[0][-1]])
            losses = loss_log[n_td - last:n_td, 0].cpu().numpy()
            logged.update({"train/learning_rate": self.learning_rate, "train/n_updates": self._n_updates,
                           "train/loss": float(np.mean([float(x) for x in losses]))})
        for k, v in logged.items():
            self._logger.record(k, v)
        self._last_logged = logged
        self._last_losses = loss_log[:n_td, 0]
        return self

    def _iteration(self, g: int, n_target_updates: int) -> None:
        """One iteration of learn(): collect train_freq steps, store them, the target updates, then g TD steps.  Every
        per-iteration offset is read on the device, so the same launches replay from a CUDA graph."""
        env, buf, pol, x = self.env, self.replay_buffer, self.policy, self._x
        E, T, H = self.n_envs, self.train_freq, env.horizon
        pp, pn, _ = pol.flat_vectors()
        _lib.rollout_explore(env.desc, env.params, env.obs, pol.desc, pp, pn, None, None, None, None, 0, self.hp, E, T,
                             self._tbl, self._flat, self._aux, None, x["explore"], self._explore_seed(), -1 - x["g0"],
                             env.state, flags=_lib.IMB_RF_DETERMINISTIC, act=pol.act)
        _lib.dqn_ring_store(self._flat, buf.tw, buf.ring, buf.buffer_size, E, T, H, env.state, buf.ring_state)
        _lib.rollout_advance(env.state, E, T, H, 0)
        for _ in range(n_target_updates):
            self._target_update()
        if g > 0:
            n_l, n_e = self.batch_size // 2, self.batch_size - self.batch_size // 2
            _lib.dqn_target(pol.desc, pol.target_flat(), buf.ring, buf.capacity, x["lidx"], buf.expert_table,
                            buf.n_expert, x["eidx"], n_l, n_e, g, self.gamma, 0.0, 1.0, self._td_rows,
                            step_base=x["td0"], state=self._state, act=pol.act)
            _lib.dqn_step(pol.desc, pp, self.exp_avg, self.exp_avg_sq, self._td_rows, self.batch_size, g,
                          self.learning_rate, 1e-8, self.max_grad_norm, x["loss"], self._state, loss_base=x["td0"],
                          act=pol.act)

    def _explore_seed(self) -> int:
        return (self.seed if self.seed is not None else self.env.seed) & 0xFFFFFFFFFFFFFFFF


DQN = DeviceDQN
