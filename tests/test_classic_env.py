"""CPU: the classic-control envs' NumPy twin (oracle/classic_env.py) against the reference's recorded expert rollouts,
its reset draws and time limit, and `envs.make_vec_env`'s argument handling and seeding.

The twin steps every recorded transition of tests/golden/expert_models/{cartpole_0,pendulum_0} from its recorded float32
observation.  gymnasium carries a float64 state between steps and rounds it to float32 only for the observation, so the
recorded next observation and the twin's can differ by the float32 rounding of the state.  Each next-observation
component k is therefore held to one float32 ulp at that component's largest magnitude in the fixture,
spacing(max |next_obs[:, k]|).  Measured (CPU, NumPy float64):
  CartPole, 26 964 transitions: max errors [2.4e-7, 1.2e-7, 7.5e-9, 1.2e-7], each exactly that one ulp.
  Pendulum, 11 200 transitions: max errors [6.0e-8, 6.0e-8, 4.8e-7] against ulps [1.2e-7, 1.2e-7, 4.8e-7]; the largest
  reward error is 8.2e-7 (bound 1e-6).
The CartPole rollouts were recorded on a CartPole that ends an episode once the pole leaves the thresholds (episodes of
393 to 500 steps, reward 1 on every step), so their rewards pin the thresholds instead: seals' FixedHorizonCartPole
reward is 0 on exactly the last step of each episode that ended early and 1 on every other step.
"""
import os

import numpy as np
import pytest

from oracle import classic_env as ce
from oracle import philox

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "expert_models")


def _transitions(name):
    d = np.load(os.path.join(GOLDEN, name, "rollouts", "final.npz"), allow_pickle=True)
    obs, acts, rews = d["obs"], d["acts"], d["rews"]
    bounds = np.concatenate([[0], d["indices"], [len(acts)]])
    o, no, early_end = [], [], []
    for k, (s, e) in enumerate(zip(bounds[:-1], bounds[1:])):
        o.append(obs[s + k:e + k])  # trajectory k holds e - s + 1 observations
        no.append(obs[s + k + 1:e + k + 1])
        last = np.zeros(e - s, bool)
        last[-1] = e - s < 500
        early_end.append(last)
    return np.concatenate(o), acts, np.concatenate(no), rews, np.concatenate(early_end)


@pytest.mark.parametrize("env,fixture", [(ce.CARTPOLE, "cartpole_0"), (ce.PENDULUM, "pendulum_0")])
def test_twin_steps_every_recorded_transition(env, fixture):
    obs, acts, nobs, rews, early_end = _transitions(fixture)
    assert len(acts) == {"cartpole_0": 26964, "pendulum_0": 11200}[fixture]
    got, rew = ce.ClassicEnvSpec(env).dynamics(obs, acts)
    assert got.dtype == np.float32 and rew.dtype == np.float32
    err = np.abs(got.astype(np.float64) - nobs)
    ulp = np.spacing(np.abs(nobs).max(axis=0))
    assert (err <= ulp).all(), (err.max(axis=0), ulp)
    if env == ce.PENDULUM:
        np.testing.assert_allclose(rew, rews, rtol=0, atol=1e-6)
    else:
        assert early_end.sum() == 42
        np.testing.assert_array_equal(rew, np.where(early_end, 0.0, 1.0))


def test_twin_cartpole_thresholds_and_pendulum_clip():
    # a state that stays inside the thresholds, and one whose pole angle crosses 12 degrees in the step
    obs = np.array([[0.0, 0.0, 0.0, 0.0], [2.39, 1.0, 0.0, 0.0], [0.0, 0.0, 0.2090, 0.5]], np.float32)
    _, rew = ce.cartpole_step(obs, np.array([1, 1, 1]))
    np.testing.assert_array_equal(rew, [1.0, 0.0, 0.0])
    # Pendulum clips the torque to [-2, 2] before the step and the reward
    o = np.array([[1.0, 0.0, 0.0]] * 2, np.float32)
    a, b = ce.pendulum_step(o, np.array([[2.0], [50.0]], np.float32)), ce.pendulum_step(o, np.array([[2.0], [2.0]]))
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    # the speed clip at 8
    fast, _ = ce.pendulum_step(np.array([[0.0, 1.0, 8.0]], np.float32), np.array([[2.0]], np.float32))
    assert fast[0, 2] == 8.0


def test_uniforms_are_the_device_words():
    u = ce.uniforms(7, philox.STREAM_ENV_RESET, np.arange(5, dtype=np.uint32), np.uint32(3), 6)
    k0, k1 = philox.key_for(7, philox.STREAM_ENV_RESET)
    for j in range(6):
        w = philox.philox4x32(np.arange(5, dtype=np.uint32), np.uint32(3), np.uint32(j // 4), np.uint32(0), k0, k1)
        np.testing.assert_array_equal(u[:, j], philox.u01(w[j % 4]))


@pytest.mark.parametrize("env", [ce.CARTPOLE, ce.PENDULUM])
def test_reset_draws_lie_in_their_intervals(env):
    spec = ce.ClassicEnvSpec(env, seed=123)
    ids, eps = np.meshgrid(np.arange(4096, dtype=np.uint32), np.arange(4, dtype=np.uint32))
    o = spec.reset_obs(ids.ravel(), eps.ravel()).astype(np.float64)
    if env == ce.CARTPOLE:
        assert o.shape == (4 * 4096, 4)
        assert (np.abs(o) <= 0.05).all() and (np.abs(o).max(axis=0) > 0.0499).all()
        np.testing.assert_allclose(o.mean(axis=0), 0.0, atol=0.05 / np.sqrt(3 * o.shape[0]) * 5)
    else:
        assert o.shape == (4 * 4096, 3)
        np.testing.assert_allclose(o[:, 0] ** 2 + o[:, 1] ** 2, 1.0, atol=1e-6)
        theta = np.arctan2(o[:, 1], o[:, 0])
        counts = np.histogram(theta, bins=8, range=(-np.pi, np.pi))[0]
        assert counts.min() > 0.8 * len(theta) / 8  # ~U(-pi, pi)
        assert (np.abs(o[:, 2]) <= 1.0).all() and np.abs(o[:, 2]).max() > 0.999
    # the draw is keyed by (seed, env id, episode)
    assert not np.array_equal(spec.reset_obs([0], [0]), spec.reset_obs([0], [1]))
    assert not np.array_equal(spec.reset_obs([0], [0]), ce.ClassicEnvSpec(env, seed=124).reset_obs([0], [0]))


@pytest.mark.parametrize("env", [ce.CARTPOLE, ce.PENDULUM])
def test_done_and_terminal_observation_exactly_at_the_horizon(env):
    H = 7
    venv = ce.ClassicVecEnv(ce.ClassicEnvSpec(env, horizon=H, seed=3), 5, env_id_offset=2)
    assert ce.ClassicEnvSpec(env).horizon == (500 if env == ce.CARTPOLE else 200)
    obs = venv.reset()
    np.testing.assert_array_equal(obs, venv.spec.reset_obs(np.arange(2, 7), 0))
    rng = np.random.default_rng(0)
    for step in range(1, 2 * H + 1):
        acts = rng.integers(0, 2, 5) if env == ce.CARTPOLE else rng.uniform(-3, 3, (5, 1)).astype(np.float32)
        want, _ = venv.spec.dynamics(obs, acts)
        obs, rew, dones, infos = venv.step(acts)
        assert dones.all() == (step % H == 0) and dones.any() == dones.all()
        if step % H == 0:
            for i in range(5):
                np.testing.assert_array_equal(infos[i]["terminal_observation"], want[i])
                assert infos[i]["TimeLimit.truncated"] is True
            np.testing.assert_array_equal(obs, venv.spec.reset_obs(np.arange(2, 7), step // H))
        else:
            assert infos == [{}] * 5
            np.testing.assert_array_equal(obs, want)
    if env == ce.PENDULUM:
        np.testing.assert_array_equal(venv.action_space.low, [-2.0])


# ---- envs.make_vec_env: seeding and refusals (no device needed: the env constructor is replaced by a recorder) -----
@pytest.fixture
def recorded(monkeypatch):
    from imitation_b200.envs import classic

    made = []

    class Recorder:
        def __init__(self, env_name, num_envs, **kw):
            made.append(dict(env_name=env_name, num_envs=num_envs, **kw))

    monkeypatch.setattr(classic, "ClassicVecEnv", Recorder)
    return made


@pytest.mark.parametrize("env", ["seals/CartPole-v0", "Pendulum-v1"])
def test_make_vec_env_draws_the_reference_seeds(recorded, env):
    from imitation_b200.algorithms.preference_comparisons import make_seeds  # util.make_seeds restated
    from imitation_b200.envs import make_vec_env

    rng, ref = np.random.default_rng(42), np.random.default_rng(42)
    make_vec_env(env, rng=rng, n_envs=5, parallel=True, max_episode_steps=33)
    seeds = make_seeds(ref, 5)
    assert rng.bit_generator.state == ref.bit_generator.state
    assert recorded == [dict(env_name=env, num_envs=5, horizon=33, seed=seeds[0])]
    make_vec_env(env, rng=rng)
    make_seeds(ref, 8)
    assert rng.bit_generator.state == ref.bit_generator.state and recorded[1]["horizon"] is None


def test_make_vec_env_refuses_what_it_cannot_run(recorded):
    from imitation_b200.envs import make_vec_env

    rng = np.random.default_rng(0)
    with pytest.raises(ValueError, match="seals/CartPole-v0, Pendulum-v1"):
        make_vec_env("seals/Ant-v0", rng=rng)
    for name in ("CartPole-v1", "MountainCar-v0", "Acrobot-v1"):
        with pytest.raises(ValueError, match="terminates episodes early"):
            make_vec_env(name, rng=rng)
    with pytest.raises(NotImplementedError, match="log_dir"):
        make_vec_env("Pendulum-v1", rng=rng, log_dir="/tmp/x")
    with pytest.raises(NotImplementedError, match="post_wrappers"):
        make_vec_env("Pendulum-v1", rng=rng, post_wrappers=[lambda env, i: env])
    with pytest.raises(NotImplementedError, match="env_make_kwargs"):
        make_vec_env("Pendulum-v1", rng=rng, env_make_kwargs={"g": 9.81})
    assert recorded == []
    make_vec_env("Pendulum-v1", rng=rng, post_wrappers=[], env_make_kwargs={})  # empty ones are accepted
    assert len(recorded) == 1


def test_env_desc_carries_the_kind():
    import ctypes

    from imitation_b200 import _lib

    assert ctypes.sizeof(_lib.EnvDesc) == 32
    d = _lib.EnvDesc(d_obs=4, d_act=2, discrete=1, horizon=500, seed=9, env_id_offset=3)
    assert d.kind == _lib.ENV_SYNTH == 0  # keyword construction keeps the synthetic env
    assert (_lib.ENV_CARTPOLE, _lib.ENV_PENDULUM) == (1, 2)
