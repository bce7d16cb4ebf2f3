"""A device SAC: SB3 2.2's `SAC` (stable_baselines3/sac/sac.py, sac/policies.py) as far as SQIL trains it.

SB3 is not a dependency, so its semantics are restated here, from SB3 2.2.x, as oracle/sac_port.py restates them
(unpinned: re-verify wherever SB3 is installed):

- `learn(total_timesteps, reset_num_timesteps=True)` is OffPolicyAlgorithm's loop, as for DQN: collect `train_freq`
  VecEnv steps, then, once `num_timesteps > learning_starts`, one `train()` call of `gradient_steps` steps (-1: as many
  as were collected).  SAC draws nothing from the global NumPy RNG while acting, so the replay indices are its only
  global draws.
- Acting: before `learning_starts` every env takes `action_space.sample()`; after it the actor samples
  `tanh(mean + std * eps)`, with `log_std` clamped to [-20, 2].  `predict` returns `unscale_action(a)`; the buffer stores
  `scale_action(unscale_action(a))` and the env receives `unscale_action` of the buffer action, each in float32 and in
  SB3's operation order (the round trip is not the identity near 0).
- `log_prob = sum Normal(mean, std).log_prob(g) - sum log(1 - a^2 + 1e-6)` with `g = mean + std * eps`, `a = tanh(g)`.
- One gradient step, in SB3's order:
  1. `ent_coef = exp(log_ent_coef)`, read before its own Adam step (or the fixed float);
  2. `ent_coef_loss = -(log_ent_coef * (logp + target_entropy)).mean()` and its Adam step (`ent_coef="auto"` only);
  3. `y = r + (1 - d) * gamma * (min(Q1_t, Q2_t)(s', a') - ent_coef * logp')`, with a fresh sample a' on s';
  4. `critic_loss = 0.5 * sum_i mse(Q_i(s, a), y)` and the critics' Adam step;
  5. `actor_loss = (ent_coef * logp - min(Q1, Q2)(s, a_pi)).mean()` through the UPDATED critics, and the actor's
     Adam step (a_pi and logp are the sample of step 2, drawn before any update);
  6. the Polyak update of the critic targets with `tau` when `gradient_step % target_update_interval == 0`, where
     `gradient_step` is the index inside the `train()` call: with `gradient_steps=1` every step updates the targets.
  The optimisers are torch Adam (eps 1e-8), with no gradient clipping.

On the device, one `learn()` is one host pass (`dqn.learn_schedule` without the epsilon-greedy draws: the random-step
vector and the replay indices) and then per iteration: `imb_sac_collect` (the actor in the envs, writing the rollout's
flat rows), `imb_dqn_ring_store` and `imb_rollout_advance` (unchanged from DQN), and `imb_sac_step` (four launches per
gradient step).  Every per-iteration offset is read from a device counter, so each iteration after the first of its
kind replays from a CUDA graph.  The noise comes from Philox streams keyed by `seed` (else the env's): the same
distributions as SB3's `th.randn` and `action_space.sample()`, not the same bits.
"""
from typing import Optional

import numpy as np
import torch as th
from torch import nn

from .. import _lib, spaces
from ..policies import base as policy_base
from ..util import logger as imit_logger
from ..util.flat import FlatAlias
from . import dqn

LOG_STD_MIN, LOG_STD_MAX = -20, 2


def scale_action(action: np.ndarray, low, high) -> np.ndarray:
    """SB3's BasePolicy.scale_action in float32: 2 * ((action - low) / (high - low)) - 1."""
    low, high = np.float32(low), np.float32(high)
    a = np.asarray(action, np.float32)
    return (np.float32(2.0) * ((a - low) / (high - low)) - np.float32(1.0)).astype(np.float32)


def unscale_action(scaled: np.ndarray, low, high) -> np.ndarray:
    """SB3's BasePolicy.unscale_action in float32: low + 0.5 * (scaled + 1) * (high - low)."""
    low, high = np.float32(low), np.float32(high)
    a = np.asarray(scaled, np.float32)
    return (low + (np.float32(0.5) * (a + np.float32(1.0)) * (high - low))).astype(np.float32)


class Actor(nn.Module):
    """SB3's sac.policies.Actor without gSDE: latent_pi = [Linear -> ReLU] x 2, then the mu and log_std heads."""

    def __init__(self, d_obs: int, d_act: int, hidden: int):
        super().__init__()
        self.features_extractor = policy_base.FlattenExtractor()
        self.latent_pi = nn.Sequential(nn.Linear(d_obs, hidden), nn.ReLU(), nn.Linear(hidden, hidden), nn.ReLU())
        self.mu = nn.Linear(hidden, d_act)
        self.log_std = nn.Linear(hidden, d_act)

    def get_action_dist_params(self, obs):
        latent = self.latent_pi(self.features_extractor(obs))
        return self.mu(latent), th.clamp(self.log_std(latent), LOG_STD_MIN, LOG_STD_MAX)

    def forward(self, obs, deterministic: bool = False):
        mean, log_std = self.get_action_dist_params(obs)
        if deterministic:
            return th.tanh(mean)
        return th.tanh(mean + th.randn_like(mean) * log_std.exp())


class ContinuousCritic(nn.Module):
    """SB3's ContinuousCritic with n_critics 2: qf0, qf1 = [Linear -> ReLU] x 2 -> Linear(h, 1) on cat([obs, action])."""

    def __init__(self, d_obs: int, d_act: int, hidden: int):
        super().__init__()
        self.features_extractor = policy_base.FlattenExtractor()
        self.q_networks = []
        for i in range(2):
            q = nn.Sequential(nn.Linear(d_obs + d_act, hidden), nn.ReLU(), nn.Linear(hidden, hidden), nn.ReLU(),
                              nn.Linear(hidden, 1))
            self.add_module(f"qf{i}", q)
            self.q_networks.append(q)

    def forward(self, obs, actions):
        x = th.cat([self.features_extractor(obs), actions], dim=1)
        return tuple(q(x) for q in self.q_networks)


def _net_width(net_arch) -> int:
    """h of SACPolicy's net_arch when it is [h, h] for the actor and the critics alike (a list, or dict(pi=.., qf=..))."""
    if net_arch is None:
        return 256
    if isinstance(net_arch, dict):
        pi, qf = list(net_arch.get("pi", [])), list(net_arch.get("qf", []))
        if set(net_arch) - {"pi", "qf"} or pi != qf:
            raise NotImplementedError(f"net_arch {net_arch!r}: the SAC kernels run one [h, h] shared by the actor and "
                                      "the critics")
        net_arch = pi
    net_arch = list(net_arch)
    if len(net_arch) != 2 or net_arch[0] != net_arch[1] or not 1 <= int(net_arch[0]) <= 256:
        raise NotImplementedError(f"net_arch {net_arch!r}: the SAC kernels run two equal layers [h, h] with h <= 256")
    return int(net_arch[0])


class SACPolicy(nn.Module):
    """SB3's SACPolicy ("MlpPolicy"): actor, critic (qf0, qf1) and critic_target, with SB3's state_dict keys, built in
    SB3's order (torch's default Linear init, no orthogonal init).  Each net is aliased onto one flat device vector in
    nn.Linear order, through `.data`, so `state_dict()`, `th.save` and the host `predict` see the kernels' memory."""

    def __init__(self, observation_space, action_space, lr_schedule=None, net_arch=None, activation_fn=nn.ReLU,
                 n_critics: int = 2, share_features_extractor: bool = False, use_sde: bool = False,
                 features_extractor_class=None, features_extractor_kwargs=None, normalize_images: bool = True,
                 optimizer_class=th.optim.Adam, optimizer_kwargs: Optional[dict] = None):
        super().__init__()
        if not spaces.is_box(action_space):
            raise NotImplementedError(f"action space {action_space!r}: the device SAC runs Box action spaces")
        if use_sde:
            raise NotImplementedError("use_sde: the device SAC samples a squashed diagonal Gaussian (no gSDE)")
        if activation_fn is not nn.ReLU:
            raise NotImplementedError(f"activation_fn {activation_fn!r}: the SAC kernels run nn.ReLU")
        if n_critics != 2:
            raise NotImplementedError(f"n_critics {n_critics}: the SAC kernels run twin critics (n_critics=2)")
        if features_extractor_class not in (None, policy_base.FlattenExtractor) or features_extractor_kwargs:
            raise NotImplementedError("features_extractor_class: the SAC kernels run Flatten features")
        if optimizer_class is not th.optim.Adam or optimizer_kwargs not in (None, {}):
            raise NotImplementedError("optimizer_class / optimizer_kwargs: the SAC step runs torch Adam with its "
                                      "defaults (eps 1e-8)")
        hidden = _net_width(net_arch)
        self.observation_space, self.action_space = observation_space, action_space
        self.d_obs, self.d_act, self.hidden = spaces.flat_dim(observation_space), spaces.flat_dim(action_space), hidden
        self.low = np.asarray(action_space.low, np.float32).reshape(-1)
        self.high = np.asarray(action_space.high, np.float32).reshape(-1)
        # SB3's order: actor, critic, critic_target, then the copy
        self.actor = Actor(self.d_obs, self.d_act, hidden)
        self.critic = ContinuousCritic(self.d_obs, self.d_act, hidden)
        self.critic_target = ContinuousCritic(self.d_obs, self.d_act, hidden)
        self.critic_target.load_state_dict(self.critic.state_dict())
        self.critic_target.train(False)

    def _aliases(self):
        al = self.__dict__.get("_flat_aliases")
        if al is None:
            a = self.actor
            al = [FlatAlias([(a.latent_pi[0], "weight"), (a.latent_pi[0], "bias"), (a.latent_pi[2], "weight"),
                             (a.latent_pi[2], "bias"), (a.mu, "weight"), (a.mu, "bias"), (a.log_std, "weight"),
                             (a.log_std, "bias")])]
            for c in (self.critic, self.critic_target):
                al.append(FlatAlias([(q[i], w) for q in c.q_networks for i in (0, 2, 4) for w in ("weight", "bias")]))
            self.__dict__["_flat_aliases"] = al
        return al

    def _flat(self, i: int) -> th.Tensor:
        al = self._aliases()[i]
        dev = al.tensors()[0].device
        if dev.type != "cuda":
            raise _lib.ImbError("the device SAC runs on CUDA only (no CPU fallback)")
        return al.get(th.float32, dev)

    def actor_flat(self) -> th.Tensor:
        return self._flat(0)

    def critic_flat(self) -> th.Tensor:
        return self._flat(1)

    def target_flat(self) -> th.Tensor:
        return self._flat(2)

    def __getstate__(self):
        st = self.__dict__.copy()
        st.pop("_flat_aliases", None)
        return st

    def set_training_mode(self, mode: bool) -> None:
        self.actor.train(mode)
        self.critic.train(mode)

    def forward(self, obs, deterministic: bool = False):
        return self._predict(obs, deterministic)

    def _predict(self, obs, deterministic: bool = False):
        return self.actor(obs, deterministic)

    def scale_action(self, action):
        return scale_action(action, self.low, self.high)

    def unscale_action(self, scaled):
        return unscale_action(scaled, self.low, self.high)

    def predict(self, observation, state=None, episode_start=None, deterministic: bool = False):
        """SB3's BasePolicy.predict: the actor's squashed action, unscaled to the Box (host path)."""
        obs = th.as_tensor(np.asarray(observation, np.float32)).to(self.actor.mu.weight.device)
        with th.no_grad():
            acts = self._predict(obs.reshape(-1, self.d_obs), deterministic)
        return self.unscale_action(acts.cpu().numpy().reshape(-1, self.d_act)), state


MlpPolicy = SACPolicy


class SAC:
    """SB3 2.2's SAC constructor, defaults and learn(), on the device.  SQIL's buffer (`SQILReplayBuffer`) is the replay
    buffer it trains from: its constant rewards are what the step reads."""

    def __init__(self, policy, env, learning_rate=3e-4, buffer_size: int = 1_000_000, learning_starts: int = 100,
                 batch_size: int = 256, tau: float = 0.005, gamma: float = 0.99, train_freq=1, gradient_steps: int = 1,
                 action_noise=None, replay_buffer_class=None, replay_buffer_kwargs: Optional[dict] = None,
                 optimize_memory_usage: bool = False, ent_coef="auto", target_update_interval: int = 1,
                 target_entropy="auto", use_sde: bool = False, sde_sample_freq: int = -1,
                 use_sde_at_warmup: bool = False, stats_window_size: int = 100, tensorboard_log=None,
                 policy_kwargs: Optional[dict] = None, verbose: int = 0, seed: Optional[int] = None, device="auto",
                 _init_setup_model: bool = True):
        from ..envs import synth
        from . import sqil

        if callable(learning_rate):
            raise NotImplementedError("a callable learning_rate: the SAC step runs a constant learning rate")
        if use_sde or use_sde_at_warmup:
            raise NotImplementedError("use_sde: the device SAC samples a squashed diagonal Gaussian (no gSDE)")
        if action_noise is not None:
            raise NotImplementedError("action_noise: the device SAC collects without added action noise")
        if optimize_memory_usage:
            raise NotImplementedError("optimize_memory_usage=True: the device ring stores next_obs beside obs")
        if isinstance(train_freq, tuple):
            n, unit = train_freq
            if unit != "step":
                raise NotImplementedError(f"train_freq {train_freq!r}: the device SAC collects whole VecEnv steps "
                                          "(train_freq in episodes is not supported)")
            train_freq = n
        if not isinstance(env, synth.DeviceVecEnv):
            raise NotImplementedError("the device SAC steps a DeviceVecEnv (imitation_b200.envs.make_vec_env)")
        if env.discrete:
            raise NotImplementedError("Discrete action spaces: the device SAC runs Box action spaces")
        if replay_buffer_class is not sqil.SQILReplayBuffer:
            raise NotImplementedError(f"replay_buffer_class {replay_buffer_class!r}: the device SAC trains from "
                                      "SQILReplayBuffer (its step reads constant rewards)")
        self.env = env
        self.n_envs = env.num_envs
        self.learning_rate = float(learning_rate)
        self.buffer_size, self.learning_starts, self.batch_size = int(buffer_size), int(learning_starts), int(batch_size)
        self.tau, self.gamma, self.train_freq = float(tau), float(gamma), int(train_freq)
        self.gradient_steps, self.target_update_interval = int(gradient_steps), int(target_update_interval)
        self.seed = seed
        self.policy_kwargs = dict(policy_kwargs or {})
        self.num_timesteps = 0
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
                raise NotImplementedError(f"policy {policy!r}: the device SAC runs MlpPolicy")
            policy = SACPolicy
        if policy is not SACPolicy:
            raise NotImplementedError(f"policy {policy!r}: the device SAC runs its MlpPolicy (SACPolicy)")
        policy = SACPolicy(env.observation_space, env.action_space, **self.policy_kwargs)
        try:
            _lib.sac_plan(policy.d_obs, policy.d_act, policy.hidden, self.batch_size)
        except _lib.ImbError as e:
            raise NotImplementedError(str(e)) from None
        if isinstance(device, str) and device == "auto":
            device = "cuda"
        self.device = th.device(device)
        if self.device.type != "cuda":
            raise NotImplementedError(f"device {device!r}: the device SAC trains on the GPU only")
        if isinstance(target_entropy, str):
            if target_entropy != "auto":
                raise ValueError(f"target_entropy {target_entropy!r}")
            self.target_entropy = float(-np.prod(env.action_space.shape).astype(np.float32))
        else:
            self.target_entropy = float(target_entropy)
        self.ent_coef = ent_coef
        if isinstance(ent_coef, str):
            if not ent_coef.startswith("auto"):
                raise ValueError(f"ent_coef {ent_coef!r}")
            init = float(ent_coef.split("_")[1]) if "_" in ent_coef else 1.0
            if init <= 0.0:
                raise ValueError("The initial value of ent_coef must be greater than 0")
            self._auto_ent = True
            self._ent = th.zeros(3, device=self.device)  # log_ent_coef, its Adam exp_avg, exp_avg_sq
            self._ent[0] = float(th.log(th.ones(1) * init))
            self._ent_coef_value = 0.0
        else:
            self._auto_ent = False
            self._ent = th.zeros(3, device=self.device)
            self._ent_coef_value = float(ent_coef)
        self.policy = policy.to(self.device)
        self.replay_buffer = replay_buffer_class(self.buffer_size, env.observation_space, env.action_space,
                                                 n_envs=self.n_envs, device=self.device,
                                                 **dict(replay_buffer_kwargs or {}))
        self.actor_m = th.zeros_like(self.policy.actor_flat())
        self.actor_v = th.zeros_like(self.actor_m)
        self.critic_m = th.zeros_like(self.policy.critic_flat())
        self.critic_v = th.zeros_like(self.critic_m)
        self._state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device=self.device)
        self._ws = th.zeros(_lib.sac_ws_floats(policy.d_obs, policy.d_act, policy.hidden, self.batch_size),
                            device=self.device)
        self.last_schedule: Optional[dqn.LearnSchedule] = None

    @property
    def actor(self) -> Actor:
        return self.policy.actor

    @property
    def critic(self) -> ContinuousCritic:
        return self.policy.critic

    @property
    def critic_target(self) -> ContinuousCritic:
        return self.policy.critic_target

    @property
    def log_ent_coef(self) -> Optional[th.Tensor]:
        """SB3's log_ent_coef (a view of the device scalar the step updates); None for a fixed ent_coef."""
        return self._ent[0:1] if self._auto_ent else None

    @property
    def logger(self):
        return self._logger

    def set_logger(self, logger) -> None:
        self._logger = logger

    def predict(self, observation, state=None, episode_start=None, deterministic: bool = False):
        return self.policy.predict(observation, state, episode_start, deterministic)

    def _seed(self) -> int:
        return (self.seed if self.seed is not None else self.env.seed) & 0xFFFFFFFFFFFFFFFF

    def _hparams(self) -> dict:
        p = self.policy
        return dict(d_obs=p.d_obs, d_act=p.d_act, hidden=p.hidden, batch_size=self.batch_size, gamma=self.gamma,
                    tau=self.tau, lr=self.learning_rate, adam_eps=1e-8, auto_ent=self._auto_ent,
                    ent_coef=self._ent_coef_value, target_entropy=self.target_entropy, reward_learner=0.0,
                    reward_expert=1.0, target_update_interval=self.target_update_interval, seed=self._seed())

    def learn(self, total_timesteps: int, callback=None, log_interval: int = 4, tb_log_name: str = "SAC",
              reset_num_timesteps: bool = True, progress_bar: bool = False):
        if callback is not None:
            raise NotImplementedError("callback: the device SAC runs the collection inside its kernel")
        env, buf = self.env, self.replay_buffer
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
        s = dqn.learn_schedule(total, E, T, self.gradient_steps, self.learning_starts, self.batch_size,
                               buf.buffer_size, buf.pos, buf.full, buf.n_expert, 1, 0, 0.0, lambda p: 0.0,
                               self.num_timesteps, exploration_draws=False)
        self.last_schedule = s
        n_iter = len(s.grad_steps)
        if n_iter == 0:
            return self
        dev = self.device
        n_td = int(s.grad_steps.sum())
        g0 = int(env.state[_lib.ST_GLOBAL_STEP])
        buf.sync_ring_state()
        td0 = self._n_updates
        self._state[_lib.ST_PPO_STEP] = td0
        self._x = dict(explore=th.as_tensor(s.explore).to(dev), lidx=th.as_tensor(s.learner_idx).to(dev),
                       eidx=th.as_tensor(s.expert_idx).to(dev), loss=th.zeros(max(n_td, 1), 4, device=dev),
                       g0=g0, td0=td0)
        tw = 2 * env.d_obs + env.d_act + 1
        if getattr(self, "_flat", None) is None or self._flat.shape[0] != E * T:
            self._flat = th.zeros(E * T, tw, device=dev)
            self._aux = th.zeros(2 * E + 2 * E * T, device=dev)
        # one graph per iteration kind (its number of gradient steps), captured at the kind's second iteration and
        # replayed from then on; the graphs bake in this learn()'s vectors, so they live for one learn()
        graphs, seen = {}, set()
        for k in range(n_iter):
            key = int(s.grad_steps[k])
            if key in graphs:
                graphs[key][0].replay()
                _lib.LAUNCHES["count"] += graphs[key][1]
                self.graph_replays += 1
                self.graph_kernels += graphs[key][1]
            elif key in seen:
                before = _lib.LAUNCHES["count"]
                g = th.cuda.CUDAGraph()
                with th.cuda.graph(g):
                    self._iteration(key)
                graphs[key] = (g, _lib.LAUNCHES["count"] - before)
                _lib.LAUNCHES["count"] = before
                g.replay()
                _lib.LAUNCHES["count"] += graphs[key][1]
                self.graph_replays += 1
                self.graph_kernels += graphs[key][1]
            else:
                self._iteration(key)
                seen.add(key)
            env.host_ep_step = (env.host_ep_step + T) % H
        self.num_timesteps = s.num_timesteps
        buf.pos = (int(s.pos[-1]) + T) % buf.buffer_size
        buf.full = s.full
        self._n_updates += n_td
        logged = {}
        if n_td:  # the means over the last train() call's steps, as SB3 leaves them recorded
            last = int(s.grad_steps[np.nonzero(s.grad_steps)[0][-1]])
            rows = self._x["loss"][n_td - last:n_td].double().cpu().numpy()
            logged = {"train/n_updates": self._n_updates, "train/ent_coef": float(np.mean(rows[:, 3])),
                      "train/actor_loss": float(np.mean(rows[:, 1])), "train/critic_loss": float(np.mean(rows[:, 0]))}
            if self._auto_ent:
                logged["train/ent_coef_loss"] = float(np.mean(rows[:, 2]))
            logged["train/learning_rate"] = self.learning_rate
        for k, v in logged.items():
            self._logger.record(k, v)
        self._last_logged = logged
        self._last_losses = self._x["loss"][:n_td]
        return self

    def _iteration(self, g: int) -> None:
        """One iteration of learn(): collect train_freq steps, store them, then g gradient steps.  Every per-iteration
        offset is read on the device, so the same launches replay from a CUDA graph."""
        env, buf, pol, x = self.env, self.replay_buffer, self.policy, self._x
        E, T, H = self.n_envs, self.train_freq, env.horizon
        _lib.sac_collect(env.desc, env.params, env.obs, pol.hidden, pol.actor_flat(), E, T, self._flat, self._aux,
                         x["explore"], x["g0"], 0, self._seed(), env.state)
        _lib.dqn_ring_store(self._flat, buf.tw, buf.ring, buf.buffer_size, E, T, H, env.state, buf.ring_state)
        _lib.rollout_advance(env.state, E, T, H, 0)
        if g > 0:
            _lib.sac_step(self._hparams(), pol.actor_flat(), self.actor_m, self.actor_v, pol.critic_flat(),
                          self.critic_m, self.critic_v, pol.target_flat(), self._ent, buf.ring, buf.capacity,
                          x["lidx"], buf.expert_table, buf.n_expert, x["eidx"], g, x["td0"], x["loss"], self._ws,
                          self._state)
