"""`RewardVecEnvWrapper` (mirror of imitation.rewards.reward_wrapper:40-133).

In the reference this wrapper calls `reward_fn(old_obs, acts, terminal-fixed obs, dones)` on the
host after every env step (H2D, MLP, D2H).  Here it only DESCRIBES the relabel: the rollout
kernel evaluates the reward network in place (csrc/imb_rollout.cu), so `reward_fn` must be the
`predict_processed` of a fusable reward network.
"""
import collections

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

    def resolve(self):
        """-> (fused net with engine, reward_mode, NormalizedRewardNet or None) for the rollout kernel; for an ensemble
        reward (`AddSTDRewardWrapper(RewardEnsemble)` or a bare `RewardEnsemble`) -> (EnsembleRelabel, 2, None); for a
        `DensityAlgorithm` reward -> (DensityRelabel, 0, None)."""
        from ..algorithms import density

        if isinstance(self.reward_fn, density.DensityAlgorithm):
            return DensityRelabel(self.reward_fn), 0, None
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
            return self._ensemble[1], 2, None
        mode, out_norm = 2, None
        from ..algorithms.adversarial import gail

        if isinstance(net, gail.RewardNetFromDiscriminatorLogit):
            mode, net = 1, net.base
        if isinstance(net, reward_nets.NormalizedRewardNet):
            if isinstance(net.base, (reward_nets.AddSTDRewardWrapper, reward_nets.RewardNetWithVariance)):
                raise NotImplementedError("a NormalizedRewardNet around an ensemble reward is not supported (the "
                                          "reference rejects it too): normalise the members instead")
            if mode == 1:
                net = net.base  # GAIL bypasses the output normaliser (gail.py:82-83, SURVEY Appendix A.6)
            else:
                out_norm, net = net, net.base
        while isinstance(net, reward_nets.RewardNetWrapper) and not hasattr(net, "_engine"):
            net = net.base
        if not hasattr(net, "_engine"):
            raise NotImplementedError(f"reward net {type(net).__name__} has no fused sm_90a implementation")
        return net, mode, out_norm


class EnsembleRelabel:
    """An ensemble reward as the rollout evaluates it (reward_nets.py:926-989, :1045-1080): up to 16 members of one
    fused architecture, each either plain or inside a `NormalizedRewardNet` (all members alike, with output norms of one
    kind), combined per step into
    mean + alpha * std.  `alpha` is read from the wrapper on every access, so a changed `default_alpha` takes effect at
    the next rollout."""

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


class DensityRelabel:
    """A `DensityAlgorithm` reward as the rollout applies it: the rollout runs with the env reward (mode 0), then one
    `imb_density_score` launch overwrites its reward column from the terminal-fixed transition rows it wrote, before
    GAE.  A non-stationary model scores episode step t with its segment t."""

    def __init__(self, algo):
        self.algo = algo

    @property
    def model(self):
        return self.algo.device_model

    def check_steps(self, t0: int, n_steps: int, horizon: int) -> None:
        """The reference's error for an episode step the model has no segment for, raised on the host before the
        rollout of n_steps from episode step t0 is launched."""
        bad = self.algo.out_of_range_step(t0, n_steps, horizon)
        if bad is not None:
            raise ValueError(f"Time {bad} out of range (0, {self.model.n_seg}], and absorbing states not currently "
                             "supported")

    def relabel(self, flat, tbl, col_rew: int, n_envs: int, n_steps: int, horizon: int, ws, state) -> None:
        """tbl[(e * T + t), col_rew] = log density of the flattened row of (e, t) in flat (imb_rollout's flat_out)."""
        _lib.density_score(self.model, flat, flat.shape[1], n_envs * n_steps, tbl.view(-1)[col_rew:], tbl.shape[1],
                           ws, seg_mode=_lib.DENSITY_SEG_ROLLOUT, state=state, n_envs=n_envs, n_steps=n_steps,
                           horizon=horizon)

    def pointer_key(self) -> tuple:
        """Every launch argument of relabel() that a captured graph bakes in, besides the caller's buffers."""
        m = self.model
        return (m.d, m.col0, m.n0, m.col1, m.n1, m.kernel, m.bandwidth, m.n_seg, m.n_demo) + tuple(
            t.data_ptr() for t in m.tensors())
