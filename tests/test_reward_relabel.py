"""How `DevicePPO` fills the rollout's reward column for every kind of reward a `RewardVecEnvWrapper` describes: the env
reward, one fused net (plain, inside a `NormalizedRewardNet` with RunningNorm or EMANorm, or as GAIL's logit), an
ensemble, and a `DensityAlgorithm` with and without a `BufferingWrapper`.

- the launches `collect_rollouts` and `exploration_rollout` make, by name and in order;
- one `DevicePPO` switched between kinds gives the tables and reward-model states of one that only ever used each kind,
  eagerly and replaying a captured graph;
- a changed ensemble `default_alpha`, `EMANorm` decay or re-trained density model recaptures the graph, and the run
  still equals an eager one.
"""
import copy
import functools
import types

import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu

DO, DA, E, H, T = 5, 2, 8, 8, 16  # T a whole number of episodes: every rollout ends at an episode start


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _venv():
    from imitation_b200.envs import synth

    return synth.DeviceVecEnv(DO, DA, E, horizon=H, seed=3)


def _algo(env, use_graph=True):
    from imitation_b200.algorithms import ppo

    algo = ppo.DevicePPO("FeedForward32Policy", env, n_steps=T, batch_size=32, n_epochs=1, seed=0)
    algo.use_cuda_graph = use_graph
    return algo


def _net(kind, seed=0):
    from imitation_b200.algorithms.adversarial import gail
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    th.manual_seed(seed)
    venv = _venv()
    obs, act = venv.observation_space, venv.action_space
    basic = lambda: reward_nets.BasicRewardNet(obs, act)  # noqa: E731
    if kind == "basic":
        return basic().cuda()
    if kind == "running":
        return reward_nets.NormalizedRewardNet(basic(), networks.RunningNorm).cuda()
    if kind == "ema":
        return reward_nets.NormalizedRewardNet(basic(), functools.partial(networks.EMANorm, decay=0.9)).cuda()
    if kind == "gail":
        return gail.RewardNetFromDiscriminatorLogit(basic()).cuda()
    assert kind == "ensemble"
    members = [reward_nets.NormalizedRewardNet(basic(), networks.RunningNorm) for _ in range(3)]
    return reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(obs, act, members).cuda(), default_alpha=-0.5)


def _demos(seed, n=6):
    from imitation_b200.data import types as data_types

    rng = np.random.default_rng(seed)
    return [data_types.Trajectory(obs=rng.normal(size=(H + 1, DO)).astype(np.float32),
                                  acts=rng.uniform(-1, 1, (H, DA)).astype(np.float32), infos=None, terminal=True)
            for _ in range(n)]


def _density(stationary=True):
    from imitation_b200.algorithms import density

    dens = density.DensityAlgorithm(demonstrations=_demos(1), venv=_venv(), rng=np.random.default_rng(2),
                                    density_type=density.DensityType.STATE_ACTION_DENSITY, kernel_bandwidth=0.7,
                                    is_stationary=stationary)
    dens.train()
    return dens


def _wrap(venv, reward, buffering=True):
    """venv inside a RewardVecEnvWrapper for `reward` (a reward net or a DensityAlgorithm; None: the env reward)."""
    from imitation_b200.data import wrappers
    from imitation_b200.rewards import reward_nets, reward_wrapper

    if reward is None:
        venv.reset()
        return venv
    inner = wrappers.BufferingWrapper(venv) if buffering else venv
    fn = reward.predict_processed if isinstance(reward, reward_nets.RewardNet) else reward
    return reward_wrapper.RewardVecEnvWrapper(inner, fn)


def _reward_state(reward):
    if reward is None or not isinstance(reward, th.nn.Module):
        return {}
    return {k: v.detach().clone() for k, v in reward.state_dict().items()}


def _assert_states_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert th.equal(a[k], b[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# the launch sequence of every kind
# ---------------------------------------------------------------------------------------------------------------------
ROLLOUT = {"env": [], "basic": [], "running": ["reward_norm_scan"], "ema": ["reward_norm_scan"], "gail": [],
           "ensemble": ["ensemble_relabel"], "density": ["density_score"], "density_own_rows": ["density_score"]}


@pytest.mark.parametrize("kind", list(ROLLOUT))
def test_launch_sequence(L, monkeypatch, kind):
    if kind.startswith("density"):
        reward = _density()
    else:
        reward = None if kind == "env" else _net(kind)
    algo = _algo(_wrap(_venv(), reward, buffering=kind != "density_own_rows"))
    algo.collect_rollouts()  # the env's first reset is not part of the sequence
    calls = []

    def record(name, fn):
        def call(*args, **kw):
            calls.append(name)
            return fn(*args, **kw)
        return call

    for name, fn in list(vars(L).items()):  # every entry point that launches (they all check their launch)
        if isinstance(fn, types.FunctionType) and fn.__module__ == L.__name__ and "_check" in fn.__code__.co_names:
            monkeypatch.setattr(L, name, record(name, fn))
    algo.collect_rollouts()
    members = kind == "ensemble"
    assert calls == ["rollout_ensemble" if members else "rollout", *ROLLOUT[kind], "gae", "rollout_advance"]
    del calls[:]
    algo.exploration_rollout(np.array([1, 0] * (H // 2), np.uint8), seed=5, step0=0)
    assert calls == ["rollout_explore", *ROLLOUT[kind], "rollout_advance"]
    th.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# one DevicePPO switched between kinds against DevicePPOs that only ever used one
# ---------------------------------------------------------------------------------------------------------------------
def _twin(algo, venv, reward, make_reward_copy):
    """A fresh DevicePPO on a fresh env, starting where `algo` and its env are now, with a copy of the reward."""
    other_venv = _venv()
    twin_reward = make_reward_copy(reward)
    twin = _algo(_wrap(other_venv, twin_reward), use_graph=algo.use_cuda_graph)
    other_venv.obs.copy_(venv.obs)
    other_venv.state.copy_(venv.state)
    other_venv.host_ep_step = venv.host_ep_step
    for a, b in zip(algo.policy.flat_vectors(), twin.policy.flat_vectors()):
        b.copy_(a)
    return twin, twin_reward


@pytest.mark.parametrize("use_graph", [False, True])
def test_switching_kinds_matches_one_kind_runs(L, use_graph):
    venv = _venv()
    algo = _algo(venv, use_graph)
    if use_graph:
        algo.learn(E * T)  # the one eager iteration: every kind below is captured and replayed
    dens = _density()
    kinds = [("density", dens), ("ensemble", _net("ensemble", 1)), ("ema", _net("ema", 2)), ("env", None),
             ("density", dens)]
    for name, reward in kinds:
        algo.set_env(_wrap(venv, reward))
        share = name in ("density", "env")  # no reward-model state a rollout changes
        twin, twin_reward = _twin(algo, venv, reward, (lambda r: r) if share else copy.deepcopy)
        graph = algo._graph
        for a in (algo, twin):
            if use_graph:
                a.learn(E * T)
            else:
                a.collect_rollouts()
        th.cuda.synchronize()
        if use_graph:
            assert algo._graph is not None and algo._graph is not graph, name
        assert th.equal(algo._tbl, twin._tbl), name
        if not share:
            _assert_states_equal(_reward_state(reward), _reward_state(twin_reward))


# ---------------------------------------------------------------------------------------------------------------------
# what a captured graph bakes in
# ---------------------------------------------------------------------------------------------------------------------
def _set_alpha(reward, dens):
    reward.default_alpha = 1.5


def _set_decay(reward, dens):
    reward.normalize_output_layer.decay = 0.7


def _retrain(reward, dens):
    dens.set_demonstrations(_demos(7, n=5))
    dens.train()


@pytest.mark.parametrize("kind,change", [("ensemble", _set_alpha), ("ema", _set_decay), ("density", _retrain)])
def test_changed_launch_argument_recaptures(L, kind, change):
    dens = _density(stationary=False) if kind == "density" else None
    runs = []
    for use_graph in (True, False):
        reward = dens if dens is not None else _net(kind, 4)
        venv = _venv()
        algo = _algo(_wrap(venv, reward), use_graph)
        algo.learn(2 * E * T)
        runs.append((algo, reward))
    (graph_run, graph_reward), (eager_run, eager_reward) = runs
    first = graph_run._graph
    assert first is not None
    for algo, reward in runs:
        if dens is None or algo is graph_run:  # the two runs share the density model
            change(reward, dens)
        algo.learn(2 * E * T)
    th.cuda.synchronize()
    assert graph_run._graph is not None and graph_run._graph is not first
    assert th.equal(graph_run._tbl, eager_run._tbl)
    assert th.equal(graph_run.policy.flat_vectors()[0], eager_run.policy.flat_vectors()[0])
    if dens is None:
        _assert_states_equal(_reward_state(graph_reward), _reward_state(eager_reward))
