"""Finite-horizon tabular Maximum Causal Entropy IRL (the reference's `imitation.algorithms.mce_irl`).

Same names, keyword arguments, defaults, logger keys, return values, warnings and errors as
/root/reference/src/imitation/algorithms/mce_irl.py.  The soft Bellman backup and the occupancy measures run as one
cooperative sm_90a launch in float64 (`imb_mce_sweep`, csrc/imb_mce.cu); the reward net's forward, backward and Adam
step run on the fused reward-net kernels (csrc/imb_disc.cu).  Per `MCEIRL.train` iteration the launch sequence is
fixed: [input RunningNorm update] -> reward forward -> sweep (undiscounted plan, occupancy discounted by `discount`,
weights and the l-infinity gap) -> forward + backward with the weights as upstream gradient -> gradient reduction ->
gradient norm -> Adam, and one read-back of (linf_delta, grad_norm) for the stopping test.

The env is any object with the attributes MCE IRL reads from a seals `TabularModelPOMDP`: transition_matrix
[S, A, S], observation_matrix [S, d], initial_state_dist, reward_matrix, horizon, state_dim, action_dim, state_space,
action_space.  The reward net must be a state-only `BasicRewardNet` the fused kernels run (at most two hidden layers of
width <= 64, d <= 64 observation features), so one-hot observations work up to 64 states.
"""
import collections
import warnings
from typing import Any, Dict, Iterable, List, Mapping, NoReturn, Optional, Tuple, Type, Union

import numpy as np
import torch as th

from .. import _lib, spaces
from ..data import types
from ..rewards import reward_nets
from ..util import logger as imit_logger
from ..util import networks
from ..util.flat import views
from . import base


def _device() -> th.device:
    return th.device("cuda", th.cuda.current_device())


class _DeviceMDP:
    """The env's T and initial-state distribution as float64 device tensors, with the sweep's workspace."""

    def __init__(self, env, flags: int):
        self.S, self.A, self.H = _dims(env, flags)
        T = _host_array("transition_matrix", env.transition_matrix, (self.S, self.A, self.S))
        init = _host_array("initial_state_dist", env.initial_state_dist, (self.S,))
        n_ws, _ = _lib.mce_plan(self.S, self.A, self.H, flags)  # this device's grid and workspace
        dev = _device()
        self.flags = flags
        self.T = th.as_tensor(T).to(dev).contiguous()
        self.init = th.as_tensor(init).to(dev).contiguous()
        self.ws = th.empty(n_ws, dtype=th.float64, device=dev)

    def discounts(self, plan: float, om: float) -> th.Tensor:
        return th.tensor([plan, om], dtype=th.float64).to(self.T.device)

    def sweep(self, flags: int, discounts: th.Tensor, **kw) -> None:
        _lib.mce_sweep(self.S, self.A, self.H, flags, self.T, self.init, kw.pop("reward", None), kw.pop("reward32", None),
                       discounts, self.ws, **kw)


def _dims(env, flags: int) -> Tuple[int, int, int]:
    """(S, A, H); ValueError for an infinite horizon, NotImplementedError (host only, before any upload) for a shape
    outside the sweep kernel's envelope."""
    if env.horizon is None:
        raise ValueError("Only finite-horizon environments are supported.")
    S, A, H = int(env.state_dim), int(env.action_dim), int(env.horizon)
    _lib.mce_plan(S, A, H, flags, n_sms=1)
    return S, A, H


def _host_array(name: str, a, shape: Tuple[int, ...]) -> np.ndarray:
    """`a` as float64, checked against the shape the sweep reads: the kernel takes raw device pointers, so an array of
    another shape would be read out of bounds instead of failing as the reference's NumPy does."""
    a = np.asarray(a, dtype=np.float64)
    if a.shape != shape:
        raise ValueError(f"{name} has shape {a.shape}, expected {shape} (S = state_dim, A = action_dim, H = horizon)")
    return a


def _reward64(env, reward: Optional[np.ndarray]) -> np.ndarray:
    return _host_array("reward", env.reward_matrix if reward is None else reward, (int(env.state_dim),))


def mce_partition_fh(env, *, reward: Optional[np.ndarray] = None, discount: float = 1.0
                     ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    r"""Soft Bellman backup for a finite-horizon MDP (Ziebart 2010, (9.1)-(9.3)) on the device.

    Returns:
        (V, Q, \pi): V[t, s], Q[t, s, a] and pi[t, s, a] as float64 arrays.

    Raises:
        ValueError: if ``env.horizon`` is None (infinite horizon).
        NotImplementedError: if the MDP is larger than the sweep kernel takes.
    """
    _dims(env, _lib.MCE_BACKWARD)
    r = _reward64(env, reward)
    m = _DeviceMDP(env, _lib.MCE_BACKWARD)
    dev = m.T.device
    V = th.empty(m.H, m.S, dtype=th.float64, device=dev)
    Q = th.empty(m.H, m.S, m.A, dtype=th.float64, device=dev)
    pi = th.empty_like(Q)
    m.sweep(_lib.MCE_BACKWARD, m.discounts(discount, 1.0), reward=th.as_tensor(r).to(dev), V=V, Q=Q, pi=pi)
    return V.cpu().numpy(), Q.cpu().numpy(), pi.cpu().numpy()


def mce_occupancy_measures(env, *, reward: Optional[np.ndarray] = None, pi: Optional[np.ndarray] = None,
                           discount: float = 1.0) -> Tuple[np.ndarray, np.ndarray]:
    """State visitation frequencies D[t, s] (shape (H + 1, S)) and their discounted sum Dcum (shape (S,)) under `pi`;
    without `pi`, under the soft-optimal policy of `reward` planned UNDISCOUNTED (as the reference plans it).

    Raises:
        ValueError: if ``env.horizon`` is None (infinite horizon).
        NotImplementedError: if the MDP is larger than the sweep kernel takes.
    """
    flags = _lib.MCE_FORWARD if pi is not None else _lib.MCE_BACKWARD | _lib.MCE_FORWARD
    S, A, H = _dims(env, flags)
    host = _host_array("pi", pi, (H, S, A)) if pi is not None else _reward64(env, reward)
    m = _DeviceMDP(env, flags)
    dev = m.T.device
    D = th.empty(m.H + 1, m.S, dtype=th.float64, device=dev)
    Dcum = th.empty(m.S, dtype=th.float64, device=dev)
    if pi is None:
        m.sweep(flags, m.discounts(1.0, discount), reward=th.as_tensor(host).to(dev), D=D, Dcum=Dcum)
    else:
        m.sweep(flags, m.discounts(1.0, discount), pi=th.as_tensor(host).to(dev), D=D, Dcum=Dcum)
    return D.cpu().numpy(), Dcum.cpu().numpy()


def squeeze_r(r_output: th.Tensor) -> th.Tensor:
    """Squeeze a reward output tensor ([n_states] or [n_states, 1]) down to [n_states]."""
    if r_output.ndim == 2:
        return th.squeeze(r_output, 1)
    assert r_output.ndim == 1
    return r_output


class TabularPolicy:
    """A tabular policy pi[t, s, a]; prediction only, on the host with the reference's draws."""

    pi: np.ndarray
    rng: np.random.Generator

    def __init__(self, state_space, action_space, pi: np.ndarray, rng: np.random.Generator) -> None:
        assert spaces.is_discrete(state_space), "state not tabular"
        assert spaces.is_discrete(action_space), "action not tabular"
        self.observation_space = state_space
        self.action_space = action_space
        self.rng = rng
        self.set_pi(pi)

    def set_pi(self, pi: np.ndarray) -> None:
        """Sets tabular policy to `pi`."""
        assert pi.ndim == 3, "expected three-dimensional policy"
        assert np.allclose(pi.sum(axis=2), 1), "policy not normalized"
        assert np.all(pi >= 0), "policy has negative probabilities"
        self.pi = pi

    def _predict(self, observation, deterministic: bool = False):
        raise NotImplementedError("Should never be called as predict overridden.")

    def forward(self, observation, deterministic: bool = False) -> NoReturn:
        raise NotImplementedError("Should never be called.")

    def _contains(self, obs) -> bool:
        n = int(self.observation_space.n)
        return np.ndim(obs) == 0 and np.issubdtype(np.asarray(obs).dtype, np.integer) and 0 <= obs < n

    def predict(self, observation, state: Optional[Tuple[np.ndarray, ...]] = None,
                episode_start: Optional[np.ndarray] = None, deterministic: bool = False
                ) -> Tuple[np.ndarray, Optional[Tuple[np.ndarray, ...]]]:
        """Actions for the MDP states `observation`; `state` = (timesteps,), reset where `episode_start`."""
        if state is None:
            timesteps = np.zeros(len(observation), dtype=int)
        else:
            assert len(state) == 1
            timesteps = state[0]
        assert len(timesteps) == len(observation), "timestep and obs batch size differ"
        if episode_start is not None:
            timesteps[episode_start] = 0
        actions: List[int] = []
        for obs, t in zip(observation, timesteps):
            assert self._contains(obs), "illegal state"
            dist = self.pi[t, obs, :]
            if deterministic:
                actions.append(int(dist.argmax()))
            else:
                actions.append(self.rng.choice(len(dist), p=dist))
        timesteps += 1
        return np.array(actions), (timesteps,)


MCEDemonstrations = Union[np.ndarray, Iterable[types.Trajectory], types.TransitionsMinimal,
                          Iterable[Mapping[str, Union[np.ndarray, th.Tensor]]]]


def _tensor_iter_norm(tensors) -> th.Tensor:
    """util.tensor_iter_norm with ord 2: the norm of the per-tensor norms (a device scalar)."""
    return th.linalg.vector_norm(th.stack([th.linalg.vector_norm(t.flatten()) for t in tensors]))


def _check_fused(reward_net, optimizer) -> None:
    """NotImplementedError for what the device trainer does not run (the reference's optimizer and net are generic)."""
    if type(optimizer) is not th.optim.Adam:
        raise NotImplementedError(f"MCEIRL trains with torch.optim.Adam on the device, got {type(optimizer).__name__}")
    g = optimizer.param_groups
    if len(g) != 1 or tuple(g[0]["betas"]) != (0.9, 0.999) or g[0]["amsgrad"] or g[0]["weight_decay"] != 0 \
            or g[0].get("maximize"):
        raise NotImplementedError("MCEIRL's device Adam takes the default betas (0.9, 0.999), no amsgrad, no "
                                  "maximize and weight_decay 0")
    if type(reward_net) is not reward_nets.BasicRewardNet or not reward_net.use_state or reward_net.use_action \
            or reward_net.use_next_state or reward_net.use_done:
        raise NotImplementedError("MCEIRL's device trainer takes a state-only BasicRewardNet (use_state=True, "
                                  "use_action=use_next_state=use_done=False)")
    if {id(p) for p in g[0]["params"]} != {id(p) for p in reward_net._engine._param_list()}:
        raise NotImplementedError("the optimizer must train exactly the reward net's parameters")


class MCEIRL(base.DemonstrationAlgorithm):
    """Tabular MCE IRL: the reward is a function of observations, the policy a function of states."""

    demo_state_om: Optional[np.ndarray]

    def __init__(self, demonstrations: Optional[MCEDemonstrations], env, reward_net: reward_nets.RewardNet,
                 rng: np.random.Generator, optimizer_cls: Type[th.optim.Optimizer] = th.optim.Adam,
                 optimizer_kwargs: Optional[Mapping[str, Any]] = None, discount: float = 1.0, linf_eps: float = 1e-3,
                 grad_l2_eps: float = 1e-4, log_interval: Optional[int] = 100, *,
                 custom_logger: Optional[imit_logger.HierarchicalLogger] = None) -> None:
        self.discount = discount
        self.env = env
        self.demo_state_om = None
        super().__init__(demonstrations=demonstrations, custom_logger=custom_logger)
        self.reward_net = reward_net
        optimizer_kwargs = optimizer_kwargs or {"lr": 1e-2}
        self.optimizer = optimizer_cls(reward_net.parameters(), **optimizer_kwargs)
        _check_fused(reward_net, self.optimizer)
        self.linf_eps = linf_eps
        self.grad_l2_eps = grad_l2_eps
        self.log_interval = log_interval
        self.rng = rng
        if self.env.horizon is None:
            raise ValueError("Only finite-horizon environments are supported.")
        ones = np.ones((self.env.horizon, self.env.state_dim, self.env.action_dim))
        self._policy = TabularPolicy(state_space=self.env.state_space, action_space=self.env.action_space,
                                     pi=ones / self.env.action_dim, rng=self.rng)

    # -- demonstrations (the reference's five forms) ---------------------------------------------------------------------
    def _set_demo_from_trajectories(self, trajs: Iterable[types.Trajectory]) -> None:
        self.demo_state_om = np.zeros((self.env.state_dim,))
        num_demos = 0
        for traj in trajs:
            cum_discount = 1.0
            for obs in traj.obs:
                self.demo_state_om[obs] += cum_discount
                cum_discount *= self.discount
            num_demos += 1
        self.demo_state_om /= num_demos

    def _set_demo_from_obs(self, obses: np.ndarray, dones: Optional[np.ndarray], next_obses: Optional[np.ndarray]) -> None:
        self.demo_state_om = np.zeros((self.env.state_dim,))
        for obs in obses:
            if isinstance(obs, th.Tensor):
                obs = obs.item()
            self.demo_state_om[obs] += 1.0
        if dones is not None and next_obses is not None:
            for done, obs in zip(dones, next_obses):
                if isinstance(done, th.Tensor):
                    done = done.item()
                    obs = obs.item()
                if done:
                    self.demo_state_om[obs] += 1.0
        else:
            warnings.warn("Training MCEIRL with transitions that lack next observation."
                          "This will result in systematically wrong occupancy measure estimates.")
        assert self.env.horizon is not None
        self.demo_state_om *= (self.env.horizon + 1) / self.demo_state_om.sum()

    def set_demonstrations(self, demonstrations: MCEDemonstrations) -> None:
        if isinstance(demonstrations, np.ndarray):
            assert demonstrations.ndim == 1
            self.demo_state_om = demonstrations
            return
        if isinstance(demonstrations, Iterable):
            it = iter(demonstrations)
            first_item = next(it)
            demonstrations_it = _chain(first_item, it)
            if isinstance(first_item, types.Trajectory):
                self._set_demo_from_trajectories(demonstrations_it)
                return
        if self.discount != 1.0:
            raise ValueError("Cannot compute discounted OM from timeless Transitions.")
        if isinstance(demonstrations, types.Transitions):
            self._set_demo_from_obs(demonstrations.obs, demonstrations.dones, demonstrations.next_obs)
        elif isinstance(demonstrations, types.TransitionsMinimal):
            self._set_demo_from_obs(demonstrations.obs, None, None)
        elif isinstance(demonstrations, Iterable):
            collated_list: Dict[str, list] = collections.defaultdict(list)
            for batch in demonstrations:
                assert isinstance(batch, Mapping)
                for k in ("obs", "dones", "next_obs"):
                    x = batch.get(k)
                    if x is not None:
                        assert isinstance(x, (np.ndarray, th.Tensor))
                        collated_list[k].append(x)
            collated = {k: np.concatenate(v) for k, v in collated_list.items()}
            assert "obs" in collated
            for k, v in collated.items():
                assert len(v) == len(collated["obs"]), k
            self._set_demo_from_obs(collated["obs"], collated.get("dones"), collated.get("next_obs"))
        else:
            raise TypeError(f"Unsupported demonstration type {type(demonstrations)}")

    # -- training ----------------------------------------------------------------------------------------------------------
    def _adam_state(self, e: reward_nets.FusedEngine) -> dict:
        """Flat Adam moments on the device, aliased by the torch optimizer's per-parameter state."""
        plist = e._param_list()
        fo = self.__dict__.get("_fused_opt")
        if fo is None or fo["ptr"] != e.params.data_ptr():
            n, dev = e.desc.n_params, e.params.device
            m, v = th.zeros(n, device=dev), th.zeros(n, device=dev)
            for p, pm, pv in zip(plist, views(m, [p.shape for p in plist]), views(v, [p.shape for p in plist])):
                st = self.optimizer.state.get(p)
                if st:
                    pm.copy_(st["exp_avg"])
                    pv.copy_(st["exp_avg_sq"])
                self.optimizer.state[p] = {"step": th.tensor(float(st["step"]) if st else 0.0), "exp_avg": pm,
                                           "exp_avg_sq": pv}
            fo = dict(ptr=e.params.data_ptr(), m=m, v=v, state=th.zeros(_lib.ST_WORDS, dtype=th.int64, device=dev))
            self._fused_opt = fo
        g = self.optimizer.param_groups[0]
        fo["hp"] = _lib.Adam(lr=g["lr"], beta1=g["betas"][0], beta2=g["betas"][1], eps=g["eps"], weight_decay=0.0)
        fo["step"] = int(self.optimizer.state[plist[0]]["step"])
        fo["state"][_lib.ST_DISC_STEP] = fo["step"]
        return fo

    def train(self, max_iter: int = 1000) -> np.ndarray:
        """Runs MCE IRL for at most `max_iter` iterations; stops early once linf_delta <= linf_eps or
        grad_norm <= grad_l2_eps.  Returns the state occupancy measure of the last iteration's reward (the reward
        before its optimiser step); `self.reward_net`, `self.optimizer` and the policy are updated in place."""
        if max_iter < 1:
            raise ValueError(f"max_iter must be at least 1, got {max_iter}")
        obs_mat = np.asarray(self.env.observation_matrix)
        assert self.demo_state_om is not None
        assert self.demo_state_om.shape == (len(obs_mat),)
        m = _DeviceMDP(self.env, _lib.MCE_BACKWARD | _lib.MCE_FORWARD)
        e = self.reward_net.engine()
        S, dev = m.S, e.params.device
        assert obs_mat.shape[1] == e.desc.d_obs, (obs_mat.shape, e.desc.d_obs)
        batch, ld = e.new_batch(S)
        batch[:e.desc.d_obs, :S] = th.as_tensor(obs_mat.T, dtype=th.float32).to(dev)
        demo = th.as_tensor(np.asarray(self.demo_state_om, dtype=np.float64)).to(dev)
        gam = m.discounts(1.0, self.discount)
        fo = self._adam_state(e)
        r32 = th.empty(S, device=dev)
        w = th.empty(S, device=dev)
        Dcum = th.empty(S, dtype=th.float64, device=dev)
        grad = th.empty(e.desc.n_params, device=dev)
        rb = th.empty(2, dtype=th.float64, device=dev)  # [linf_delta, grad_norm]: the iteration's one read-back
        plist = e._param_list()
        shapes = [p.shape for p in plist]
        flags = _lib.IMB_F_ZERO_GRAD | (_lib.IMB_F_TRAIN_NORM if e.has_norm else 0)
        n_steps = 0
        with networks.training(self.reward_net):
            for t in range(max_iter):
                e.norm_update(batch, ld, S)  # the training-mode forward's RunningNorm update (no-op without one)
                _lib.reward_forward(e.desc, e.params, e.norm_state, batch, ld, S, 0, r32)
                m.sweep(_lib.MCE_BACKWARD | _lib.MCE_FORWARD, gam, reward32=r32, Dcum=Dcum, demo_om=demo, weights=w,
                        linf=rb[0:1])
                _lib.disc_fwd_bwd(e.desc, e.params, e.norm_state, batch, ld, S, S, 0.0, w, None, flags, e.ws)
                _lib.disc_reduce(e.desc, e.ws, grad)
                rb[1] = th.linalg.vector_norm(th.stack([th.linalg.vector_norm(g) for g in views(grad, shapes)]))
                _lib.disc_adam(e.desc, fo["hp"], e.params, fo["m"], fo["v"], None, 1.0, e.ws, fo["state"], None)
                n_steps += 1
                linf_delta, grad_norm = rb.cpu().tolist()
                if self.log_interval is not None and 0 == (t % self.log_interval):
                    weight_norm = _tensor_iter_norm(self.reward_net.parameters()).item()
                    self.logger.record("iteration", t)
                    self.logger.record("linf_delta", linf_delta)
                    self.logger.record("weight_norm", weight_norm)
                    self.logger.record("grad_norm", grad_norm)
                    self.logger.dump(t)
                if linf_delta <= self.linf_eps or grad_norm <= self.grad_l2_eps:
                    break
        self._last = dict(reward=r32, weights=w, linf_delta=linf_delta, grad_norm=grad_norm, iterations=n_steps)
        for p, g in zip(plist, views(grad, shapes)):
            p.grad = g.clone()
            self.optimizer.state[p]["step"] = th.tensor(float(fo["step"] + n_steps))
        pi = th.empty(m.H, S, m.A, dtype=th.float64, device=dev)
        m.sweep(_lib.MCE_BACKWARD, m.discounts(self.discount, 1.0), reward32=r32, pi=pi)
        self._policy.set_pi(pi.cpu().numpy())
        return Dcum.cpu().numpy()

    @property
    def policy(self) -> TabularPolicy:
        return self._policy


def _chain(first, rest):
    yield first
    yield from rest
