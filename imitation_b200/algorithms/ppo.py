"""PPO generator on the GPU (`gen_algo` of the adversarial trainers).

The reference passes a stable-baselines3 `PPO` (scripts/ingredients/rl.py:122-194) and calls
`gen_algo.learn(total_timesteps, reset_num_timesteps=False, callback=...)`
(algorithms/adversarial/common.py:414).  SB3 is a host-side library; this class keeps the
constructor arguments and the attributes the trainers read (`policy`, `n_steps`, `device`,
`set_env`, `get_env`, `set_logger`, `logger`, `num_timesteps`) and runs both halves of `learn`
as kernels: one rollout launch (csrc/imb_rollout.cu) and one persistent PPO-update launch
(csrc/imb_ppo.cu).  Arithmetic follows SB3 2.2.x (oracle/ppo_port.py).

SB3's `target_kl` (early stop of `train()` on the approximate KL) and `clip_range_vf` (clipped value loss) run inside
the PPO kernel, and so do the statistics `PPO.train` records (`train/entropy_loss`, `policy_gradient_loss`,
`value_loss`, `approx_kl`, `clip_fraction`, `loss`, `explained_variance`, `std`, `n_updates`, `clip_range`,
`learning_rate`, `clip_range_vf`).  Their semantics restate SB3 2.2.1 `PPO.train` as oracle/ppo_port.py does; SB3 is not
installed here, so this parity is unpinned, like the rest of the PPO port.
"""
import math

from typing import Optional

import numpy as np
import torch as th

from .. import _lib
from ..data import wrappers
from ..policies import base as policies
from ..rewards import reward_wrapper
from ..util import logger as imit_logger


class DevicePPO:
    def __init__(self, policy, env, learning_rate: float = 3e-4, n_steps: int = 2048, batch_size: int = 64,
                 n_epochs: int = 10, gamma: float = 0.99, gae_lambda: float = 0.95, clip_range: float = 0.2,
                 normalize_advantage: bool = True, ent_coef: float = 0.0, vf_coef: float = 0.5,
                 max_grad_norm: float = 0.5, policy_kwargs: Optional[dict] = None, seed: Optional[int] = None,
                 device="cuda", sampling: str = "device", target_kl: Optional[float] = None,
                 clip_range_vf: Optional[float] = None, **unused):
        if clip_range_vf is not None and not float(clip_range_vf) > 0:  # SB3 PPO._setup_model asserts the same
            raise ValueError("`clip_range_vf` must be positive, pass `None` to deactivate vf clipping")
        if target_kl is not None and not float(target_kl) > 0:
            raise ValueError("`target_kl` must be positive, pass `None` to train every epoch")
        self.target_kl = None if target_kl is None else float(target_kl)
        self.clip_range_vf = None if clip_range_vf is None else float(clip_range_vf)
        self.learning_rate, self.clip_range = learning_rate, clip_range
        self.device = th.device(device)
        self.n_steps, self.batch_size, self.n_epochs = int(n_steps), int(batch_size), int(n_epochs)
        self._user_seed = None if seed is None else int(seed)  # SB3: the global RNGs are seeded only when a seed is given
        self.seed = 0 if seed is None else int(seed)        # the Philox streams of the kernels always need a key
        self.sampling = sampling
        self.hp = _lib.PpoHparams(gamma=gamma, gae_lambda=gae_lambda, clip_range=clip_range, ent_coef=ent_coef,
                                  vf_coef=vf_coef, max_grad_norm=max_grad_norm, lr=learning_rate, adam_eps=1e-5,
                                  n_epochs=n_epochs, batch_size=batch_size,
                                  normalize_advantage=int(normalize_advantage))
        self.env = None
        self._base_env = None
        self._logger = imit_logger.configure()
        self.num_timesteps = 0
        self.set_env(env)
        if isinstance(policy, policies.ActorCriticPolicy):
            self.policy = policy.to(self.device)
        else:
            cls = {"MlpPolicy": policies.ActorCriticPolicy, "FeedForward32Policy": policies.FeedForward32Policy}.get(
                policy, policy)
            kw = dict(policy_kwargs or {})
            if cls is policies.ActorCriticPolicy:
                kw.setdefault("net_arch", (64, 64))
            if self._user_seed is not None:
                th.manual_seed(self._user_seed)
            self.policy = cls(self._base_env.observation_space, self._base_env.action_space, **kw).to(self.device)
        try:  # refuse a policy / minibatch no PPO kernel can run now, not at the first train()
            _lib.ppo_plan(self.policy.desc, self.batch_size, act=self.policy.act)
        except _lib.ImbError as e:
            raise NotImplementedError(f"policy / minibatch not supported by the PPO update kernels: {e}") from None
        n = self.policy.desc.n_params
        self.exp_avg = th.zeros(n, device=self.device)
        self.exp_avg_sq = th.zeros(n, device=self.device)
        # training statistics of the last train() (_lib.PPO_STAT_* order), written by the PPO kernel itself
        self.train_stats = th.full((_lib.PPO_STAT_FLOATS,), math.nan, device=self.device)
        # learn() records them after its last train(), like SB3; AdversarialTrainer turns this off and records them
        # at the end of its round, so that train_gen() never waits for the PPO update
        self.record_in_learn = True
        self._tbl = None
        self._aux = None
        self._scratch = {}        # the training rollout's reward relabel buffers (reward_wrapper.Relabel)
        # buffers of exploration_rollout (table, flat rows, aux, relabel buffers): never captured
        self._x_tbl, self._x_flat, self._x_aux, self._x_scratch = None, None, None, {}
        self.loss_log = None      # optional [n_minibatch_steps][4] device tensor (parity tests)
        self.noise = None         # optional pinned sampling noise for the next rollout (parity tests)
        self.perm = None          # optional host permutations [n_epochs][N] (parity tests)
        self._capturing = False   # True while a CUDA graph of the round is being captured
        self.use_cuda_graph = True  # learn(): replay [rollout -> GAE -> advance -> PPO update] as one CUDA graph
        self._graph = None
        self._graph_key = None
        self._graph_launches = 0
        self._eager_iters = 0
        self.ev_rollout = th.cuda.Event()  # recorded after every rollout: generator samples are in the ring

    # -- SB3 surface ---------------------------------------------------------------------------------------------
    def set_env(self, env, force_reset: bool = True) -> None:
        self.env = env
        e, self._rw_wrapper, self._buffering = env, None, None
        while not hasattr(e, "desc"):
            if isinstance(e, reward_wrapper.RewardVecEnvWrapper):
                self._rw_wrapper = e
            if isinstance(e, wrappers.BufferingWrapper):
                self._buffering = e
            if not hasattr(e, "venv"):
                raise TypeError("DevicePPO needs a DeviceVecEnv (optionally wrapped); host VecEnvs have no GPU path")
            e = e.venv
        self._base_env = e

    def get_env(self):
        return self.env

    def set_logger(self, logger) -> None:
        self._logger = logger

    @property
    def logger(self):
        return self._logger

    # -- learn = collect_rollouts + train ---------------------------------------------------------------------------
    def collect_rollouts(self) -> None:
        env = self._base_env
        env.ensure_reset()
        E, T = env.num_envs, self.n_steps
        pol = self.policy
        pp, pn, pc = pol.flat_vectors()
        rw = _lib.rollout_row_width(pol.desc)
        if self._tbl is None or self._tbl.shape[0] != E * T:
            self._tbl = th.zeros(E * T, rw, device=self.device)
            self._aux = th.zeros(2 * E + 2 * E * T, device=self.device)
        flat, ring = (None, None)
        if self._buffering is not None:
            flat, ring = self._buffering.rollout_targets(T)
        t0 = env.host_ep_step
        ring_args = (ring.table if ring is not None else None, ring.capacity if ring is not None else 0)

        def launch(disc, dparams, dnorm, mode, members, flat):
            if members is None:
                _lib.rollout(env.desc, env.params, env.obs, pol.desc, pp, pn, disc, dparams, dnorm, mode, self.hp, E, T,
                             self._tbl, *ring_args, flat, self._aux, self.noise, env.state, act=pol.act)
            else:
                _lib.rollout_ensemble(env.desc, env.params, env.obs, pol.desc, pp, pn, disc, members, self.hp, E, T,
                                      self._tbl, *ring_args, flat, self._aux, self.noise, env.state, act=pol.act)

        self._relabelled_rollout(launch, self._tbl, flat, t0, E, T, self._scratch)
        da = 1 if pol.discrete else pol.d_act
        col_val = pol.d_obs + da + 1
        _lib.gae(self._tbl, rw, col_val, E, T, self._aux, self.hp.gamma, self.hp.gae_lambda, env.state, env.horizon)
        _lib.rollout_advance(env.state, E, T, env.horizon, ring.capacity if ring is not None else 0)
        if not self._capturing:
            self.after_rollout_host(t0)

    def _relabel(self) -> reward_wrapper.Relabel:
        """What fills the rollout's reward column: the RewardVecEnvWrapper's relabel, else the env reward."""
        return self._rw_wrapper.resolve() if self._rw_wrapper is not None else reward_wrapper.Relabel()

    def _relabelled_rollout(self, launch, tbl, flat, t0: int, E: int, T: int, scratch: dict) -> None:
        """Launch a rollout over the reward the RewardVecEnvWrapper describes and finish its reward column
        (rewards/reward_wrapper.py:92-133 -> predict_processed).  launch(disc, disc_params, disc_norm, reward_mode,
        members, flat) issues the rollout itself (flat: its transition rows, None when nobody reads them).  t0: the
        episode step the rollout starts at; scratch: this rollout's relabel buffers."""
        relabel = self._relabel()
        env = self._base_env
        relabel.check_steps(t0, T, env.horizon)
        if flat is None and relabel.needs_flat:  # no BufferingWrapper: the relabel reads rows of the scratch
            if scratch.get("flat") is None or scratch["flat"].shape[0] != E * T:
                scratch["flat"] = th.zeros(E * T, 2 * env.d_obs + env.d_act + 1, device=self.device)
            flat = scratch["flat"]
        disc, dparams, dnorm, members = relabel.rollout_args(scratch, E, T)
        launch(disc, dparams, dnorm, relabel.mode, members, flat)
        pol = self.policy
        col_rew = pol.d_obs + (1 if pol.discrete else pol.d_act) + 2
        relabel.finish(tbl, col_rew, flat, E, T, env.horizon, env.state, scratch)

    def exploration_rollout(self, explore_policy, seed: int, step0: int, deterministic: bool = False, noise=None):
        """The rollout of an ExplorationWrapper over this algorithm (AgentTrainer.sample's exploration phase,
        algorithms/preference_comparisons.py:283-301): len(explore_policy) steps, a whole number of episodes, from an
        episode start, step t taken by the random policy where explore_policy[t] is 1 (actions from the Philox stream
        keyed by `seed` at step step0 + t, or from `noise`) and by this policy otherwise (sampled, or its mode when
        `deterministic`).  The learned reward is relabelled as in collect_rollouts, so the output normalisers advance
        once per step.  Uses buffers of its own: the training rollout's table, ring and flat rows (which a captured
        graph bakes in) are not touched, nor is num_timesteps, and no GAE runs.  -> (flat rows [E*T][tw] in
        completion order, ground-truth env rewards [E][T]), device tensors valid until the next call."""
        env = self._base_env
        env.ensure_reset()
        E, H, T = env.num_envs, env.horizon, len(explore_policy)
        if T % H != 0 or env.host_ep_step != 0:
            raise ValueError(f"an exploration rollout covers whole episodes from an episode start: {T} steps with "
                             f"horizon {H} from episode step {env.host_ep_step}")
        pol = self.policy
        pp, pn, _ = pol.flat_vectors()
        rw = _lib.rollout_row_width(pol.desc)
        tw = 2 * env.d_obs + env.d_act + 1
        if self._x_tbl is None or self._x_tbl.shape[0] != E * T:
            self._x_tbl = th.zeros(E * T, rw, device=self.device)
            self._x_flat = th.zeros(E * T, tw, device=self.device)
            self._x_aux = th.zeros(2 * E + 2 * E * T, device=self.device)
        vec = th.as_tensor(np.ascontiguousarray(explore_policy, dtype=np.uint8)).to(self.device)
        flags = _lib.IMB_RF_DETERMINISTIC if deterministic else 0

        def launch(disc, dparams, dnorm, mode, members, flat):
            _lib.rollout_explore(env.desc, env.params, env.obs, pol.desc, pp, pn, disc, dparams, dnorm, members, mode,
                                 self.hp, E, T, self._x_tbl, flat, self._x_aux, noise, vec, seed, step0,
                                 env.state, flags=flags, act=pol.act)

        self._relabelled_rollout(launch, self._x_tbl, self._x_flat, 0, E, T, self._x_scratch)
        _lib.rollout_advance(env.state, E, T, H, 0)
        env.host_ep_step = 0
        return self._x_flat, self._x_aux[2 * E + E * T:].view(E, T)

    def after_rollout_host(self, t0: int) -> None:
        """Host-side mirrors of what the rollout kernels just did (also called per graph replay)."""
        env = self._base_env
        E, T = env.num_envs, self.n_steps
        env.host_ep_step = (t0 + T) % env.horizon
        if self._buffering is not None:
            self._buffering.after_rollout(T, t0, self._aux[2 * E + E * T:2 * E + 2 * E * T])
        self.num_timesteps += E * T

    def train(self) -> None:
        pol = self.policy
        pp, pn, pc = pol.flat_vectors()
        N = self._tbl.shape[0]
        _lib.ppo_update_ex(pol.desc, pp, pn, pc, self.exp_avg, self.exp_avg_sq, self._tbl, N, self.hp, self.perm,
                           self.seed, self.loss_log, self._base_env.state, target_kl=self.target_kl,
                           clip_range_vf=self.clip_range_vf, stats=self.train_stats, act=pol.act)

    def read_train_stats(self) -> dict:
        """The statistics of the last train() as SB3's PPO.train records them (key -> float; waits for that update)."""
        s = self.train_stats.cpu().tolist()
        out = {"train/entropy_loss": s[_lib.PPO_STAT_ENTROPY_LOSS],
               "train/policy_gradient_loss": s[_lib.PPO_STAT_PG_LOSS],
               "train/value_loss": s[_lib.PPO_STAT_VALUE_LOSS],
               "train/approx_kl": s[_lib.PPO_STAT_APPROX_KL],
               "train/clip_fraction": s[_lib.PPO_STAT_CLIP_FRACTION],
               "train/loss": s[_lib.PPO_STAT_LOSS],
               "train/explained_variance": s[_lib.PPO_STAT_EXPLAINED_VARIANCE]}
        if not self.policy.discrete:
            out["train/std"] = s[_lib.PPO_STAT_STD]
        out["train/n_updates"] = int(s[_lib.PPO_STAT_N_UPDATES])
        out["train/clip_range"] = float(self.clip_range)
        if self.clip_range_vf is not None:
            out["train/clip_range_vf"] = self.clip_range_vf
        out["train/learning_rate"] = float(self.learning_rate)
        return out

    def record_train_stats(self, logger=None) -> None:
        """Record the last train()'s statistics (read_train_stats) on `logger` (default: this algorithm's)."""
        lg = self._logger if logger is None else logger
        for k, v in self.read_train_stats().items():
            lg.record(k, v, exclude="tensorboard" if k == "train/n_updates" else None)

    def _pointer_key(self, relabel: reward_wrapper.Relabel):
        """Everything a captured graph bakes in: device pointers of the vectors the kernels touch."""
        pp, pn, pc = self.policy.flat_vectors()
        key = (pp.data_ptr(), pn.data_ptr(), pc.data_ptr(), self._tbl.data_ptr() if self._tbl is not None else 0,
               self.n_steps, id(self._rw_wrapper), id(self._buffering),
               *[t.data_ptr() for t in self._scratch.values()],
               # launch arguments of the PPO update
               self.target_kl, self.clip_range_vf, self.train_stats.data_ptr())
        if self._buffering is not None and self._buffering._ring is not None:
            key += (self._buffering._ring.table.data_ptr(),)
        return key + relabel.graph_key()

    def _iteration(self) -> None:
        """One collect_rollouts + train, replayed from a CUDA graph once it is warm (the kernels read every
        per-call scalar from the device counter block, so the captured launch sequence is exact)."""
        plain = self.noise is None and self.perm is None and self.loss_log is None
        if self._buffering is not None:
            self._buffering.before_rollout()
        if not (self.use_cuda_graph and plain) or self._eager_iters < 1 or self._tbl is None:
            self.collect_rollouts()
            if not self._capturing:
                self.ev_rollout.record()
            self.train()
            self._eager_iters += 1
            return
        relabel = self._relabel()
        key = self._pointer_key(relabel)
        if self._graph is None or key != self._graph_key:
            before = _lib.LAUNCHES["count"]
            self._capturing = True
            try:
                # two graphs with the "rollout done" event between them: the adversarial trainer's discriminator
                # stream starts from that event while the PPO update is still running
                g_roll, g_train = th.cuda.CUDAGraph(), th.cuda.CUDAGraph()
                with th.cuda.graph(g_roll):
                    self.collect_rollouts()
                with th.cuda.graph(g_train, pool=g_roll.pool()):
                    self.train()
            finally:
                self._capturing = False
            self._graph, self._graph_key = (g_roll, g_train), key
            self._graph_launches = _lib.LAUNCHES["count"] - before
            _lib.LAUNCHES["count"] = before
        t0 = self._base_env.host_ep_step
        relabel.check_steps(t0, self.n_steps, self._base_env.horizon)  # the replayed launches take no host check
        self._graph[0].replay()
        self.ev_rollout.record()
        self._graph[1].replay()
        _lib.LAUNCHES["count"] += self._graph_launches
        self.after_rollout_host(t0)

    def learn(self, total_timesteps: int, callback=None, reset_num_timesteps: bool = True, **kwargs):
        per = self._base_env.num_envs * self.n_steps
        done = 0
        if callback is not None and hasattr(callback, "init_callback"):
            callback.init_callback(self)
        while done < total_timesteps:
            if callback is not None and hasattr(callback, "on_rollout_start"):
                callback.on_rollout_start()
            self._iteration()
            done += per
        if self.record_in_learn and done > 0:
            self.record_train_stats()
        return self

    def predict(self, observation, state=None, episode_start=None, deterministic=False):
        return self.policy.predict(observation, state, episode_start, deterministic)


PPO = DevicePPO
