"""`generate_trajectories` & friends on the GPU-resident VecEnv (mirror of
imitation.data.rollout: make_sample_until :226-271, generate_trajectories :382-506,
rollout_stats :509-560, flatten_trajectories[_with_rew] :563-621, generate_transitions
:624-665, discounted_sum :728-757).

The reference steps the VecEnv from Python and stops with the *unbiased* rule: once
`sample_until(trajectories)` holds, every env still finishes its current episode and is then
made inactive; finally the list is shuffled with the caller's `rng`.  On the lock-step
fixed-horizon device env every env finishes an episode at the same step, so the same rule
reduces to "roll whole episodes (one kernel launch per episode, thread per env) until the
predicate holds after a batch of E completed trajectories", appended in env order exactly as
`add_steps_and_auto_finish` would, then `rng.shuffle`.
"""
from typing import Callable, Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch as th

from .. import _lib
from . import types
from .types import flatten_trajectories, flatten_trajectories_with_rew  # noqa: F401  (re-export)

GenTrajTerminationFn = Callable[[Sequence[types.TrajectoryWithRew]], bool]


def make_min_episodes(n: int) -> GenTrajTerminationFn:
    assert n >= 1
    return lambda trajectories: len(trajectories) >= n


def make_min_timesteps(n: int) -> GenTrajTerminationFn:
    assert n >= 1
    return lambda trajectories: sum(len(t.obs) - 1 for t in trajectories) >= n


def make_sample_until(min_timesteps: Optional[int] = None, min_episodes: Optional[int] = None) -> GenTrajTerminationFn:
    if min_timesteps is None and min_episodes is None:
        raise ValueError("At least one of min_timesteps and min_episodes needs to be non-None")
    conditions = []
    if min_timesteps is not None:
        if min_timesteps <= 0:
            raise ValueError(f"min_timesteps={min_timesteps} if provided must be positive")
        conditions.append(make_min_timesteps(min_timesteps))
    if min_episodes is not None:
        if min_episodes <= 0:
            raise ValueError(f"min_episodes={min_episodes} if provided must be positive")
        conditions.append(make_min_episodes(min_episodes))
    return lambda trajs: all(c(trajs) for c in conditions)


def _policy_of(policy):
    """The device policy `policy` is or holds: an ActorCriticPolicy, a DQN's Q-net policy (which acts greedily), or a
    SAC's policy."""
    from ..algorithms import dqn, sac
    from ..policies import base as policies

    kinds = (policies.ActorCriticPolicy, dqn.DQNPolicy, sac.SACPolicy)
    if isinstance(policy, kinds):
        return policy
    inner = getattr(policy, "policy", None)
    if isinstance(inner, kinds):
        return inner
    raise TypeError("Policy must be an imitation_b200 ActorCriticPolicy or an algorithm holding one "
                    f"(host callables have no GPU path), got {type(policy)} instead")


def generate_trajectories(policy, venv, sample_until: GenTrajTerminationFn, rng: np.random.Generator, *,
                          deterministic_policy: bool = False) -> Sequence[types.TrajectoryWithRew]:
    """Roll `policy` in the device VecEnv until `sample_until` holds (unbiased, see module doc).  With a DAgger
    `InteractiveTrajectoryCollector` as `venv`, `policy` is the expert it collects demonstrations from."""
    from ..algorithms import dagger, dqn, sac
    from ..envs import synth

    if isinstance(venv, dagger.InteractiveTrajectoryCollector):
        return venv.generate_trajectories(policy, sample_until, rng, deterministic_policy=deterministic_policy)
    base = venv
    while not isinstance(base, synth.DeviceVecEnv):
        if not hasattr(base, "venv"):
            raise TypeError("generate_trajectories on the GPU path needs a DeviceVecEnv")
        base = base.venv
    pol = _policy_of(policy)
    if isinstance(pol, sac.SACPolicy):
        return _sac_trajectories(pol, base, sample_until, rng, deterministic_policy)
    if isinstance(pol, dqn.DQNPolicy):  # SB3's QNetwork._predict takes the argmax whatever `deterministic` says
        deterministic_policy = True
    pp, pn, _ = pol.flat_vectors()
    E, H, Do = base.num_envs, base.horizon, base.d_obs
    rw = _lib.rollout_row_width(pol.desc)
    hp = _lib.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                         lr=0.0, adam_eps=1e-5, n_epochs=1, batch_size=1, normalize_advantage=0)
    base.reset()  # generate_trajectories starts from venv.reset() (rollout.py:396)
    tbl = th.zeros(E * H, rw, device=base.device)
    tw = 2 * Do + base.d_act + 1
    flat = th.zeros(E * H, tw, device=base.device)  # reference-order transitions; from t0 = 0: row e*H + t
    aux = th.zeros(2 * E + 2 * E * H, device=base.device)
    trajectories = []
    while True:
        _lib.rollout(base.desc, base.params, base.obs, pol.desc, pp, pn, None, None, None, 0, hp, E, H, tbl, None, 0,
                     flat, aux, None, base.state, flags=_lib.IMB_RF_DETERMINISTIC if deterministic_policy else 0,
                     act=pol.act)
        _lib.rollout_advance(base.state, E, H, H, 0)
        base.host_ep_step = 0
        trajectories += batch_trajectories(base, tbl, flat, aux)
        if sample_until(trajectories):
            break
    rng.shuffle(trajectories)
    return trajectories


def _sac_trajectories(pol, base, sample_until, rng, deterministic: bool) -> List[types.TrajectoryWithRew]:
    """Whole episodes from reset of a SAC policy (imb_sac_collect in its predict mode, noise keyed by the env's seed):
    as in the reference's evaluation, the env steps with `predict`'s action unscale(a), and that is the recorded
    action."""
    E, H, Do, Da = base.num_envs, base.horizon, base.d_obs, base.d_act
    tw = 2 * Do + Da + 1
    base.reset()
    flat = th.zeros(E * H, tw, device=base.device)  # from t0 = 0: row e * H + t
    aux = th.zeros(2 * E + 2 * E * H, device=base.device)
    trajectories = []
    while True:
        flags = _lib.SAC_PREDICT | (_lib.SAC_DETERMINISTIC if deterministic else 0)
        _lib.sac_collect(base.desc, base.params, base.obs, pol.hidden, pol.actor_flat(), E, H, flat, aux, None, 0,
                         flags, base.seed, base.state)
        _lib.rollout_advance(base.state, E, H, H, 0)
        base.host_ep_step = 0
        rows = flat.view(E, H, tw).cpu().numpy()
        rews = aux[2 * E + E * H:].cpu().numpy().reshape(E, H)
        for e in range(E):
            obs = np.concatenate([rows[e, :, :Do], rows[e, -1:, Do + Da:2 * Do + Da]]).astype(np.float32)
            acts = rows[e, :, Do:Do + Da].astype(np.float32)
            trajectories.append(types.TrajectoryWithRew(obs=obs, acts=acts, infos=None, terminal=True,
                                                        rews=rews[e].astype(np.float32)))
        if sample_until(trajectories):
            break
    rng.shuffle(trajectories)
    return trajectories


def batch_trajectories(base, tbl, flat, aux) -> List[types.TrajectoryWithRew]:
    """The E whole episodes of one rollout launch from episode step 0 over the env's horizon H, in env order: rollout
    rows `tbl` ([E * H][rw], obs | act first), flattened rows `flat` (for the terminal observations) and `aux` (for the
    env rewards)."""
    E, H, Do, Da = base.num_envs, base.horizon, base.d_obs, base.d_act
    da = 1 if base.discrete else Da
    tw = 2 * Do + Da + 1
    rows = tbl.cpu().numpy().reshape(E, H, -1)
    term = flat.view(E, H, tw)[:, -1, Do + Da:2 * Do + Da].cpu().numpy()  # terminal observations
    rews = aux[2 * E + E * H:2 * E + 2 * E * H].cpu().numpy().reshape(E, H)
    out = []
    for e in range(E):
        obs = np.concatenate([rows[e, :, :Do], term[e:e + 1]]).astype(base.observation_space.dtype)
        if base.discrete:
            acts = rows[e, :, Do].astype(base.action_space.dtype)
        else:  # the env (and the recorded trajectory) sees the clipped action (SURVEY Appendix A.7)
            acts = np.clip(rows[e, :, Do:Do + da], base.action_space.low, base.action_space.high)
        out.append(types.TrajectoryWithRew(obs=obs, acts=acts, infos=None, terminal=True,
                                           rews=rews[e].astype(np.float32)))
    return out


def rollout_stats(trajectories: Sequence[types.TrajectoryWithRew]) -> Mapping[str, float]:
    """n_traj plus min / mean / std / max of the episode returns (`return_*`, from the trajectories' rewards), of the
    lengths (`len_*`) and -- for trajectories whose last info carries a Monitor record -- of the Monitor-captured returns
    (`monitor_return_*`, `monitor_return_len` of them); data/rollout.py:509-560."""
    assert len(trajectories) > 0
    out: Dict[str, float] = {"n_traj": len(trajectories)}
    desc = {"return": np.asarray([sum(t.rews) for t in trajectories]),
            "len": np.asarray([len(t.rews) for t in trajectories])}
    monitored = [t.infos[-1].get("episode", {}).get("r") for t in trajectories if t.infos is not None]
    monitored = [r for r in monitored if r is not None]
    if monitored:  # (possibly fewer than n_traj: trajectories without infos are skipped)
        desc["monitor_return"] = np.asarray(monitored)
        out["monitor_return_len"] = len(monitored)
    for name, vals in desc.items():
        for stat in ("min", "mean", "std", "max"):
            out[f"{name}_{stat}"] = getattr(np, stat)(vals).item()
    return out


def generate_transitions(policy, venv, n_timesteps: int, rng: np.random.Generator, *, truncate: bool = True,
                         **kwargs) -> types.TransitionsWithRew:
    traj = generate_trajectories(policy, venv, sample_until=make_min_timesteps(n_timesteps), rng=rng, **kwargs)
    tr = flatten_trajectories_with_rew(traj)
    if truncate and n_timesteps is not None:
        d = {k: v[:n_timesteps] for k, v in types.dataclass_quick_asdict(tr).items()}
        tr = types.TransitionsWithRew(**d)
    return tr


def rollout(policy, venv, sample_until, rng, *, unwrap: bool = True, exclude_infos: bool = True, verbose: bool = True,
            **kwargs):
    return generate_trajectories(policy, venv, sample_until, rng=rng, **kwargs)


def discounted_sum(arr: np.ndarray, gamma: float):
    assert arr.ndim in (1, 2)
    if gamma == 1.0:
        return arr.sum(axis=0)
    return np.polynomial.polynomial.polyval(gamma, arr)
