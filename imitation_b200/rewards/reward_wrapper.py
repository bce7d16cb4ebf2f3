"""`RewardVecEnvWrapper` (mirror of imitation.rewards.reward_wrapper:40-133).

In the reference this wrapper calls `reward_fn(old_obs, acts, terminal-fixed obs, dones)` on the
host after every env step (H2D, MLP, D2H).  Here it only DESCRIBES the relabel: the rollout
kernel evaluates the reward network in place (csrc/imb_rollout.cu), so `reward_fn` must be the
`predict_processed` of a fusable reward network.
"""
import collections

import torch as th

from .. import _lib
from . import reward_nets


class WrappedRewardCallback:
    def __init__(self, episode_rewards):
        self.episode_rewards = episode_rewards
        self.logger = None

    def init_callback(self, model):
        self.logger = model.logger

    def on_rollout_start(self):
        if len(self.episode_rewards) == 0 or self.logger is None:
            return
        self.logger.record("rollout/ep_rew_wrapped_mean", sum(self.episode_rewards) / len(self.episode_rewards))


class RewardVecEnvWrapper:
    def __init__(self, venv, reward_fn, ep_history: int = 100):
        assert not isinstance(venv, RewardVecEnvWrapper)
        self.venv = venv
        self.num_envs = venv.num_envs
        self.observation_space, self.action_space = venv.observation_space, venv.action_space
        self.episode_rewards = collections.deque(maxlen=ep_history)
        self.reward_fn = reward_fn
        self.reset()

    def make_log_callback(self) -> WrappedRewardCallback:
        return WrappedRewardCallback(self.episode_rewards)

    def reset(self):
        return self.venv.reset()

    def resolve(self) -> "Relabel":
        """The relabel of reward_fn: a `DensityRelabel`, an `EnsembleRelabel` for an ensemble reward (built once per
        wrapper and member set) or a `NetRelabel`."""
        from ..algorithms import density

        if isinstance(self.reward_fn, density.DensityAlgorithm):
            return DensityRelabel(self.reward_fn)
        net = getattr(self.reward_fn, "__self__", None)
        if not isinstance(net, reward_nets.RewardNet) or getattr(self.reward_fn, "__name__", "") != "predict_processed":
            raise NotImplementedError("RewardVecEnvWrapper on the GPU path needs reward_fn = <RewardNet>.predict_processed "
                                      "or a DensityAlgorithm")
        if isinstance(net, (reward_nets.AddSTDRewardWrapper, reward_nets.RewardEnsemble)):
            # built once per ensemble (its checks sync every member's engine); rebuilt when the members change
            ens = net.base if isinstance(net, reward_nets.AddSTDRewardWrapper) else net
            key = (id(net), tuple(id(m) for m in getattr(ens, "members", ())))
            cached = self.__dict__.get("_ensemble")
            if cached is None or cached[0] != key:
                self._ensemble = (key, EnsembleRelabel(net))
            return self._ensemble[1]
        return NetRelabel(net)


class Relabel:
    """How a rollout fills its reward column; this base is the env reward, which needs nothing.  `scratch`: one
    rollout's buffers, each kind's under names of its own."""

    mode = 0            # the rollout kernel's reward_mode: 0 env reward, 1 GAIL logit, 2 reward net
    needs_flat = False  # finish() reads the transition rows the rollout writes

    def check_steps(self, t0, n_steps, horizon):
        """Raises on the host, before any launch, if a rollout of n_steps from episode step t0 cannot be scored."""

    def rollout_args(self, scratch, n_envs, n_steps):
        """-> (disc, disc_params, disc_norm, members) of the rollout launch."""
        return None, None, None, None

    def finish(self, tbl, col_rew, flat, n_envs, n_steps, horizon, state, scratch):
        """Completes the reward column col_rew of the rollout table tbl."""

    def graph_key(self):
        """The launch arguments a captured graph bakes in, besides the scratch's buffers."""
        return ()


class NetRelabel(Relabel):
    """One fused reward net (`BasicRewardNet` / `BasicShapedRewardNet`) evaluated inside the rollout, as a GAIL logit
    (mode 1) or a reward (mode 2), then the output normalisation of an enclosing `NormalizedRewardNet` (out_norm)
    scanned over the reward column, once per env step."""

    def __init__(self, net: reward_nets.RewardNet):
        from ..algorithms.adversarial import gail

        self.mode, self.out_norm = 2, None
        if isinstance(net, gail.RewardNetFromDiscriminatorLogit):
            self.mode, net = 1, net.base
        if isinstance(net, reward_nets.NormalizedRewardNet):
            if isinstance(net.base, (reward_nets.AddSTDRewardWrapper, reward_nets.RewardNetWithVariance)):
                raise NotImplementedError("a NormalizedRewardNet around an ensemble reward is not supported (the "
                                          "reference rejects it too): normalise the members instead")
            if self.mode == 1:
                net = net.base  # GAIL bypasses the output normaliser (gail.py:82-83, SURVEY Appendix A.6)
            else:
                self.out_norm, net = net, net.base
        while isinstance(net, reward_nets.RewardNetWrapper) and not hasattr(net, "_engine"):
            net = net.base
        if not hasattr(net, "_engine"):
            raise NotImplementedError(f"reward net {type(net).__name__} has no fused sm_90a implementation")
        self.net = net

    def rollout_args(self, scratch, n_envs, n_steps):
        eng = self.net.engine()
        return eng.desc, eng.params, eng.norm_state, None

    def finish(self, tbl, col_rew, flat, n_envs, n_steps, horizon, state, scratch):
        o = self.out_norm
        if o is not None:
            rw, layer = tbl.shape[1], o.normalize_output_layer
            _lib.reward_norm_scan(tbl.view(-1)[col_rew:], n_envs, n_steps, rw, n_steps * rw, *o.output_norm_vectors(),
                                  layer.eps, True, ema_decay=layer.decay if o.output_norm_is_ema else None)

    def graph_key(self):
        return (self.mode,) + _net_key(self.net, self.out_norm)


def _net_key(net, out_norm) -> tuple:
    """The launch arguments of a fused net and of its output normaliser (vectors, eps and an EMANorm's decay)."""
    eng = net.engine()
    norm = () if out_norm is None else out_norm.output_norm_args()
    return (eng.params.data_ptr(), eng.norm_state.data_ptr(), id(out_norm)) + tuple(
        t.data_ptr() if isinstance(t, th.Tensor) else t for t in norm)


class EnsembleRelabel(Relabel):
    """An ensemble reward as the rollout evaluates it (reward_nets.py:926-989, :1045-1080): up to 16 members of one
    fused architecture, each either plain or inside a `NormalizedRewardNet` (all members alike, with output norms of one
    kind), raw rewards [M][T][E] combined per step into mean + alpha * std.  `alpha` is read from the wrapper on every
    access, so a changed `default_alpha` takes effect at the next rollout."""

    mode = 2

    def __init__(self, reward: reward_nets.RewardNet):
        self.reward = reward  # (held: the resolve() cache is keyed on its identity)
        self.wrapper = reward if isinstance(reward, reward_nets.AddSTDRewardWrapper) else None
        ensemble = reward.base if self.wrapper is not None else reward
        if not isinstance(ensemble, reward_nets.RewardEnsemble):
            raise NotImplementedError(f"AddSTDRewardWrapper around {type(ensemble).__name__}: the GPU rollout fuses "
                                      "only a RewardEnsemble's variance")
        members = list(ensemble.members)
        if len(members) > _lib.PU_MAX_MEMBERS:
            raise NotImplementedError(f"the GPU rollout evaluates at most {_lib.PU_MAX_MEMBERS} ensemble members, "
                                      f"got {len(members)}")
        self.nets, self.out_norms = [], []
        for k, m in enumerate(members):
            out_norm = m if isinstance(m, reward_nets.NormalizedRewardNet) else None
            net = m.base if out_norm is not None else m
            if not hasattr(net, "_engine"):
                raise NotImplementedError(f"ensemble member {k} ({type(net).__name__}) has no fused sm_90a "
                                          "implementation")
            self.nets.append(net)
            self.out_norms.append(out_norm)
        if len({o is None for o in self.out_norms}) > 1:
            raise NotImplementedError("ensemble members must all be NormalizedRewardNets or all plain reward nets, "
                                      "not a mix")
        if len({o.output_norm_is_ema for o in self.out_norms if o is not None}) > 1:
            raise NotImplementedError("ensemble members' output norms must all be RunningNorm or all EMANorm, not a "
                                      "mix")
        d0 = bytes(self.nets[0].engine().desc)
        for k, net in enumerate(self.nets[1:], 1):
            if bytes(net.engine().desc) != d0:
                raise NotImplementedError(f"ensemble member {k} has a different architecture from member 0: the GPU "
                                          "rollout evaluates members of one architecture")

    @property
    def alpha(self) -> float:
        return float(self.wrapper.default_alpha) if self.wrapper is not None else 0.0

    def rollout_args(self, scratch, n_envs, n_steps):
        M, n, engines = len(self.nets), n_steps * n_envs, [m.engine() for m in self.nets]
        dev, n_ws = engines[0].params.device, _lib.ensemble_relabel_ws_floats(M, n_steps)
        if scratch.get("ensemble_raw") is None or scratch["ensemble_raw"].numel() != M * n:
            scratch["ensemble_raw"] = th.empty(M * n, device=dev)  # the members' raw rewards [M][T][E]
        if scratch.get("ensemble_ws") is None or scratch["ensemble_ws"].numel() < n_ws:
            scratch["ensemble_ws"] = th.zeros(n_ws, device=dev)  # zero-filled: the relabel's ticket starts at 0
        members = _lib.rollout_members([e.params for e in engines],
                                       [e.norm_state if e.has_norm else None for e in engines], scratch["ensemble_raw"])
        return engines[0].desc, None, None, members

    def finish(self, tbl, col_rew, flat, n_envs, n_steps, horizon, state, scratch):
        norms = [None if o is None else o.output_norm_args() for o in self.out_norms]
        desc = _lib.pref_uncertainty_desc(list(scratch["ensemble_raw"].view(len(self.nets), -1)), norms)
        _lib.ensemble_relabel(desc, self.alpha, tbl, tbl.shape[1], col_rew, n_envs, n_steps, scratch["ensemble_ws"])

    def graph_key(self):
        # alpha is a launch argument of the relabel: a new default_alpha needs a new graph
        return (self.alpha,) + sum((_net_key(n, o) for n, o in zip(self.nets, self.out_norms)), ())


class DensityRelabel(Relabel):
    """A `DensityAlgorithm` reward as the rollout applies it: the rollout runs with the env reward (mode 0), then one
    `imb_density_score` launch overwrites its reward column from the terminal-fixed transition rows it wrote, before
    GAE.  A non-stationary model scores episode step t with its segment t."""

    needs_flat = True

    def __init__(self, algo):
        self.algo, self.model = algo, algo.device_model

    def check_steps(self, t0, n_steps, horizon):
        """The reference's error for the first episode step the rollout reaches that the model has no segment for."""
        n = self.model.n_seg
        if not self.algo.is_stationary and (t0 >= n or min(t0 + n_steps, horizon) > n):
            raise ValueError(f"Time {max(t0, n)} out of range (0, {n}], and absorbing states not currently supported")

    def rollout_args(self, scratch, n_envs, n_steps):
        n_ws = _lib.density_ws_floats(n_envs * n_steps)
        if scratch.get("density_ws") is None or scratch["density_ws"].numel() != n_ws:
            scratch["density_ws"] = th.zeros(n_ws, device=self.model.demo.device)  # zero-filled: tickets start at 0
        return None, None, None, None

    def finish(self, tbl, col_rew, flat, n_envs, n_steps, horizon, state, scratch):
        """tbl[(e * T + t), col_rew] = log density of the flattened row of (e, t) in flat (imb_rollout's flat_out)."""
        _lib.density_score(self.model, flat, flat.shape[1], n_envs * n_steps, tbl.view(-1)[col_rew:], tbl.shape[1],
                           scratch["density_ws"], seg_mode=_lib.DENSITY_SEG_ROLLOUT, state=state, n_envs=n_envs,
                           n_steps=n_steps, horizon=horizon)

    def graph_key(self):
        m = self.model
        return (m.d, m.col0, m.n0, m.col1, m.n1, m.kernel, m.bandwidth, m.n_seg, m.n_demo) + tuple(
            t.data_ptr() for t in m.tensors())
