"""`ExplorationWrapper` and the split of `AgentTrainer.sample` (reference policies/exploration_wrapper.py:23-95 and
algorithms/preference_comparisons.py:194-307), pinned to the reference on the CPU.

tests/golden/exploration.npz holds what the reference's own classes do:
    wrapper/<case>  `ExplorationWrapper` over a 3-env host env for a (switch_prob, random_prob, seed) case: the seed it
                    gives `action_space.seed`, which policy acts at each of three runs of calls (7, 13 and 5 calls), and
                    four draws of the shared generator afterwards (its state);
    sample/<case>   the reference `AgentTrainer(exploration_frac=0.5)` over `oracle.synth_env.SynthVecEnv` with a stub
                    `BaseAlgorithm` and a callable reward: after `train`, `sample(steps)` -- the lengths of its agent and
                    exploration trajectories, which wrapper calls of the exploration rollout were random, and four
                    draws of the generator afterwards.  The agent's buffer holds enough finished trajectories that no
                    top-up runs.
Re-record it where the reference sources are importable (oracle/refimport.py) with

    IMB_RECORD_REFERENCE=1 python -m pytest tests/test_exploration_reference.py -k reference_records

Where they are importable, the same test regenerates the results and compares them with the stored file.  The device
rollout that consumes the policy vector is held to a CPU twin in tests/test_exploration.py.
"""
import os

import numpy as np
import pytest

from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "exploration.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
# name: (switch_prob, random_prob, seed)
WRAPPERS = {"half": (0.5, 0.5, 0), "rare_switch": (0.1, 0.9, 1), "often_switch": (0.9, 0.2, 2),
            "never_switch": (0.0, 0.5, 3), "always_switch": (1.0, 0.5, 4)}
CALLS = (7, 13, 5)
# name: (d_obs, d_act, discrete, E, H, train steps, sample steps, exploration_frac, switch_prob, random_prob, seed)
SAMPLES = {"box": (3, 2, False, 4, 5, 160, 60, 0.5, 0.5, 0.5, 7),
           "discrete": (2, 3, True, 3, 4, 96, 50, 0.5, 0.3, 0.6, 8)}


def _reference_available() -> bool:
    from oracle import refimport

    return refimport.available()


def _fingerprint(rng):
    return rng.integers(0, 1 << 62, 4)


class _SeededSpace:
    """Gives a shim action space the `seed` method gymnasium's spaces have, recording the seeds it is given."""

    def __init__(self, space):
        self.space, self.seeds = space, []
        space.seed = self.seeds.append


def _record_policy_choices(ew_mod, log):
    """Patch the reference ExplorationWrapper.__call__ to append, per call, whether the random policy acts."""
    orig = ew_mod.ExplorationWrapper.__call__

    def call(self, observation, input_state, episode_start):
        log.append(self.current_policy == self._random_policy)
        return orig(self, observation, input_state, episode_start)

    ew_mod.ExplorationWrapper.__call__ = call
    return orig


def _record_wrapper(name):
    from imitation.policies import exploration_wrapper as ew
    from oracle import synth_env

    switch_prob, random_prob, seed = WRAPPERS[name]
    import gymnasium.spaces as shim_spaces

    venv = synth_env.SynthVecEnv(synth_env.SynthEnvSpec(2, 2, horizon=4), 3, spaces_mod=shim_spaces)
    seeded = _SeededSpace(venv.action_space)
    rng = np.random.default_rng(seed)
    policy = lambda obs, state, ep: (np.zeros((len(obs), 2), np.float32), None)  # noqa: E731
    log = []
    orig = _record_policy_choices(ew, log)
    try:
        w = ew.ExplorationWrapper(policy=policy, venv=venv, random_prob=random_prob, switch_prob=switch_prob, rng=rng)
        obs = np.zeros((3, 2), np.float32)
        for n in CALLS:
            for _ in range(n):
                w(obs, None, None)
    finally:
        ew.ExplorationWrapper.__call__ = orig
    return {f"wrapper/{name}/seed": np.array(seeded.seeds, np.int64),
            f"wrapper/{name}/random": np.array(log, np.uint8), f"wrapper/{name}/rng_after": _fingerprint(rng)}


def _record_sample(name):
    import gymnasium.spaces as shim_spaces
    from imitation.algorithms import preference_comparisons as ref_pc
    from imitation.policies import exploration_wrapper as ew
    from stable_baselines3.common import base_class

    from oracle import synth_env

    Do, Da, discrete, E, H, train_steps, steps, frac, switch_prob, random_prob, seed = SAMPLES[name]
    venv = synth_env.SynthVecEnv(synth_env.SynthEnvSpec(Do, Da, discrete=discrete, horizon=H, seed=seed), E,
                                 spaces_mod=shim_spaces)
    _SeededSpace(venv.action_space)

    class StubAlgorithm(base_class.BaseAlgorithm):
        """Steps its env with a constant action: what `learn` and `predict` do is not what is recorded."""
        num_timesteps = 0
        _obs = None
        observation_space, action_space = venv.observation_space, venv.action_space

        def predict(self, observation, state=None, episode_start=None, deterministic=False):
            n = len(observation)
            return (np.zeros(n, np.int64) if discrete else np.zeros((n, Da), np.float32)), None

        def learn(self, total_timesteps, reset_num_timesteps=False, callback=None, **kw):
            env = self.get_env()
            if self._obs is None:
                self._obs = env.reset()
            for _ in range(total_timesteps // E):
                self._obs, _, _, _ = env.step(self.predict(self._obs)[0])
                self.num_timesteps += E

    def reward_fn(obs, acts, next_obs, dones):
        return np.asarray(next_obs, np.float32).sum(1)

    rng = np.random.default_rng(seed)
    log = []
    orig = _record_policy_choices(ew, log)
    try:
        trainer = ref_pc.AgentTrainer(StubAlgorithm(), reward_fn, venv, rng, exploration_frac=frac,
                                      switch_prob=switch_prob, random_prob=random_prob)
        trainer.train(train_steps)
        n_agent_avail = trainer.buffering_wrapper.n_transitions
        log.clear()  # (training calls no wrapper; only the exploration rollout's calls are recorded)
        trajs = trainer.sample(steps)
    finally:
        ew.ExplorationWrapper.__call__ = orig
    n_expl_traj = len(log) // H * E  # k batches of E episodes
    lens = np.array([len(t) for t in trajs], np.int64)
    return {f"sample/{name}/lens": lens, f"sample/{name}/n_exploration_traj": np.int64(n_expl_traj),
            f"sample/{name}/random": np.array(log, np.uint8), f"sample/{name}/rng_after": _fingerprint(rng),
            f"sample/{name}/agent_available": np.int64(n_agent_avail)}


def _record_all():
    from oracle import refimport

    refimport.load()
    out = {}
    for name in WRAPPERS:
        out.update(_record_wrapper(name))
    for name in SAMPLES:
        out.update(_record_sample(name))
    return out


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_golden_is_what_the_reference_records():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead)."""
    out = _record_all()
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = G.load("exploration")
    assert set(z.files) == set(out)
    for k, v in out.items():
        np.testing.assert_array_equal(v, z[k], err_msg=k)


# ------------------------------------------------------------------------------------------------
# this package against the stored file
# ------------------------------------------------------------------------------------------------
class _Space:
    def __init__(self):
        self.seeds = []

    def seed(self, s):
        self.seeds.append(s)


class _Venv:
    def __init__(self):
        self.action_space = _Space()


@pytest.mark.parametrize("name", sorted(WRAPPERS))
def test_wrapper_matches_reference_golden(name):
    from imitation_b200.policies import exploration_wrapper

    z = G.load("exploration")
    switch_prob, random_prob, seed = WRAPPERS[name]
    rng = np.random.default_rng(seed)
    venv = _Venv()
    w = exploration_wrapper.ExplorationWrapper(None, venv, random_prob=random_prob, switch_prob=switch_prob, rng=rng)
    assert venv.action_space.seeds == list(z[f"wrapper/{name}/seed"]) == [w.seed]
    got, steps = [], 0
    for n in CALLS:  # the chain carries over from one call to the next
        assert w.steps_taken == steps
        v = w.advance(n)
        assert v.dtype == np.uint8 and v.shape == (n,)
        got.append(v)
        steps += n
    np.testing.assert_array_equal(np.concatenate(got), z[f"wrapper/{name}/random"])
    np.testing.assert_array_equal(_fingerprint(rng), z[f"wrapper/{name}/rng_after"])


@pytest.mark.parametrize("name", sorted(SAMPLES))
def test_sample_split_matches_reference_golden(name):
    """split_steps + exploration_plan + _get_trajectories reproduce the reference's sample(): part sizes, the random
    steps of the exploration rollout and the generator's state afterwards."""
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.policies import exploration_wrapper

    z = G.load("exploration")
    Do, Da, discrete, E, H, train_steps, steps, frac, switch_prob, random_prob, seed = SAMPLES[name]
    rng = np.random.default_rng(seed)
    w = exploration_wrapper.ExplorationWrapper(None, _Venv(), random_prob=random_prob, switch_prob=switch_prob, rng=rng)

    def episodes(n):
        return [types.TrajectoryWithRew(obs=np.zeros((H + 1, Do), np.float32), acts=np.zeros((H, Da), np.float32),
                                        infos=None, terminal=True, rews=np.zeros(H, np.float32)) for _ in range(n)]

    agent_steps, exploration_steps = pc.split_steps(steps, frac)
    avail = int(z[f"sample/{name}/agent_available"])
    assert avail >= agent_steps and avail % H == 0  # no top-up in the recorded run
    agent = pc._get_trajectories(episodes(avail // H), agent_steps)
    k, policy_steps = pc.exploration_plan(w, rng, exploration_steps, E, H)
    assert k * E == int(z[f"sample/{name}/n_exploration_traj"])
    explo = pc._get_trajectories(episodes(k * E), exploration_steps)
    np.testing.assert_array_equal([len(t) for t in list(agent) + list(explo)], z[f"sample/{name}/lens"])
    np.testing.assert_array_equal(policy_steps, z[f"sample/{name}/random"])
    np.testing.assert_array_equal(_fingerprint(rng), z[f"sample/{name}/rng_after"])


def test_split_steps_warns_when_exploration_rounds_to_zero():
    from imitation_b200.algorithms import preference_comparisons as pc

    class Log:
        def __init__(self):
            self.warnings = []

        def warn(self, msg):
            self.warnings.append(msg)

    log = Log()
    assert pc.split_steps(10, 0.05, log) == (10, 0)
    assert log.warnings == ["No exploration steps included: exploration_frac = 0.05 > 0 but steps=10 is too small."]
    assert pc.split_steps(100, 0.05, log) == (95, 5) and len(log.warnings) == 1
    assert pc.split_steps(100, 0.0, log) == (100, 0) and len(log.warnings) == 1
