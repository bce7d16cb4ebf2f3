"""GPU: seals/CartPole-v0 and Pendulum-v1 stepped inside the rollout kernels, against their NumPy twin
(oracle/classic_env.py), plus their action bounds, every trainer that rolls out in them, and a BC policy that learns.

The comparison is teacher-forced, as in test_rollout_float64.py: every step (e, t) of a rollout is re-stepped by the
twin from the kernel's own observation row and recorded action.  Both sides compute in float64 from the same float32
observation and round once to float32, so they differ only where the device's and NumPy's float64 sin / cos / atan2
(and the compiler's FMA contraction) round a float32 boundary differently: each next observation, env reward and reset
observation is held to one float32 ulp of the twin's value, elementwise.  Done flags, the flat and ring rows against
the rollout rows, and the controls are exact.
"""
import os

import numpy as np
import pytest
import torch as th

from oracle import classic_env as ce

pytestmark = pytest.mark.gpu

ENVS = (ce.CARTPOLE, ce.PENDULUM)
# envs per tile size from the SM count (the tile the rollout plan picks; ragged and 16-byte aligned counts both occur)
TILES = {8: lambda s: 16 * s - 5, 32: lambda s: 32 * s, 64: lambda s: 128 * s - 2, 128: lambda s: 128 * s + 100}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "expert_models")
FIXTURE = {ce.CARTPOLE: "cartpole_0", ce.PENDULUM: "pendulum_0"}


def _close_ulp(got, want, what):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    tol = np.maximum(np.spacing(np.abs(want)), np.float32(2.0 ** -60))
    bad = np.abs(got.astype(np.float64) - want.astype(np.float64)) > tol
    assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} off by more than 1 ulp, e.g. {got[bad][:4]} vs {want[bad][:4]}"


def _hp():
    from imitation_b200 import _lib

    return _lib.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                           lr=0.0, adam_eps=1e-5, n_epochs=1, batch_size=1, normalize_advantage=0)


def _policy(venv, **kw):
    from imitation_b200.policies import base as policies

    th.manual_seed(11)
    return policies.FeedForward32Policy(venv.observation_space, venv.action_space, **kw).cuda()


def _demos(env):
    from imitation_b200.data import serialize

    return serialize.load(os.path.join(GOLDEN, FIXTURE[env], "rollouts", "final.npz"))


# ---------------------------------------------------------------------------------------------------------------------
# the device env against the twin
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("reward", ["env", "gail", "ensemble"])
@pytest.mark.parametrize("deterministic", [False, True], ids=["sampled", "deterministic"])
@pytest.mark.parametrize("rows", sorted(TILES))
@pytest.mark.parametrize("env", ENVS)
def test_rollout_steps_the_twin(env, rows, deterministic, reward):
    from imitation_b200 import _lib
    from imitation_b200.envs import ClassicVecEnv
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    E, H, seed, off = TILES[rows](th.cuda.get_device_properties(0).multi_processor_count), 6, 17, 9
    venv = ClassicVecEnv(env, E, horizon=H, seed=seed, env_id_offset=off)
    spec = ce.ClassicEnvSpec(env, horizon=H, seed=seed)
    pol = _policy(venv, log_std_init=0.5)
    pp, pn, _ = pol.flat_vectors()
    Do, Da, disc = venv.d_obs, venv.d_act, venv.discrete
    da, rw, tw = 1 if disc else Da, _lib.rollout_row_width(pol.desc), 2 * Do + Da + 1
    nets = []
    if reward != "env":
        th.manual_seed(3)
        nets = [reward_nets.BasicRewardNet(venv.observation_space, venv.action_space,
                                           normalize_input_layer=networks.RunningNorm).cuda()
                for _ in range(2 if reward == "ensemble" else 1)]
    engines = [n.engine() for n in nets]
    dd = engines[0].desc if engines else None
    assert _lib.rollout_plan(pol.desc, dd, max(1, len(nets)), E) == rows
    ids = np.arange(off, off + E)
    venv.reset()
    _close_ulp(venv.obs.t().cpu().numpy(), spec.reset_obs(ids, 0), "imb_env_reset")
    flags = _lib.IMB_RF_DETERMINISTIC if deterministic else 0
    for episode in range(2):
        tbl = th.zeros(E * H, rw, device="cuda")
        flat, ring = th.zeros(E * H, tw, device="cuda"), th.full((E * H, tw), -7.0, device="cuda")
        aux = th.zeros(2 * E + 2 * E * H, device="cuda")
        obs_before = venv.obs.t().cpu().numpy()
        if reward == "ensemble":
            raw = th.zeros(2 * H * E, device="cuda")
            members = _lib.rollout_members([e.params for e in engines], [e.norm_state for e in engines], raw)
            _lib.rollout_ensemble(venv.desc, None, venv.obs, pol.desc, pp, pn, dd, members, _hp(), E, H, tbl, ring,
                                  E * H, flat, aux, None, venv.state, flags=flags, act=pol.act)
            assert np.isfinite(raw.cpu().numpy()).all()
        else:
            e0 = engines[0] if engines else None
            _lib.rollout(venv.desc, None, venv.obs, pol.desc, pp, pn, dd, e0 and e0.params, e0 and e0.norm_state,
                         1 if engines else 0, _hp(), E, H, tbl, ring, E * H, flat, aux, None, venv.state, flags=flags,
                         act=pol.act)
        _lib.rollout_advance(venv.state, E, H, H, E * H)
        rows_ = tbl.cpu().numpy().reshape(E, H, rw)
        fl = flat.cpu().numpy().reshape(E, H, tw)  # from episode step 0 over one horizon: flat row e * H + t
        np.testing.assert_array_equal(ring.cpu().numpy(), flat.cpu().numpy())
        obs, act = rows_[:, :, :Do], rows_[:, :, Do:Do + da]
        # the reset observation the rollout starts from, then the observation rows follow the next observations
        np.testing.assert_array_equal(obs[:, 0], obs_before)
        if episode == 1:
            _close_ulp(obs[:, 0], spec.reset_obs(ids, 1), "auto-reset")
        np.testing.assert_array_equal(obs[:, 1:], fl[:, :-1, Do + Da:2 * Do + Da])
        # flat rows: obs | control | next obs | done
        np.testing.assert_array_equal(fl[:, :, :Do], obs)
        ctl = np.eye(Da, dtype=np.float32)[act[..., 0].astype(np.int64)] if disc else np.clip(act, -2.0, 2.0)
        np.testing.assert_array_equal(fl[:, :, Do:Do + Da], ctl)
        np.testing.assert_array_equal(fl[:, :, -1], np.broadcast_to(np.arange(H) == H - 1, (E, H)).astype(np.float32))
        want_nobs, want_rew = spec.dynamics(obs.reshape(-1, Do), act.reshape(-1) if disc else act.reshape(-1, Da))
        _close_ulp(fl[:, :, Do + Da:2 * Do + Da].reshape(-1, Do), want_nobs, "next obs")
        _close_ulp(aux[2 * E + E * H:].cpu().numpy(), want_rew, "env reward")
        assert np.isfinite(rows_).all()
        if reward == "env":
            np.testing.assert_array_equal(rows_[:, :, Do + da + 2], aux[2 * E + E * H:].cpu().numpy().reshape(E, H))
    _close_ulp(venv.obs.t().cpu().numpy(), spec.reset_obs(ids, 2), "state after the second episode")


@pytest.mark.parametrize("env", ENVS)
def test_env_reset_matches_the_twin_and_validates_the_kind(env):
    from imitation_b200 import _lib
    from imitation_b200.envs import ClassicVecEnv

    venv = ClassicVecEnv(env, 1000, seed=2 ** 31 - 2, env_id_offset=123)
    spec = ce.ClassicEnvSpec(env, seed=2 ** 31 - 2)
    for ep in range(3):
        got = venv.reset()
        assert got.shape == (1000, venv.d_obs)
        _close_ulp(got, spec.reset_obs(np.arange(123, 1123), ep), f"reset {ep}")
    bad = _lib.EnvDesc(d_obs=venv.d_obs, d_act=venv.d_act, discrete=int(not venv.discrete), horizon=10, seed=0,
                       kind=venv.kind)
    with pytest.raises(_lib.ImbError, match="takes d_obs"):
        _lib.env_reset(venv.obs, 1000, bad, venv.state)
    unknown = _lib.EnvDesc(d_obs=3, d_act=1, discrete=0, horizon=10, seed=0, kind=7)
    with pytest.raises(_lib.ImbError, match="unknown env kind 7"):
        _lib.env_reset(venv.obs, 1000, unknown, venv.state)
    pol = _policy(venv)
    pp, pn, _ = pol.flat_vectors()
    tbl, aux = th.zeros(1000 * 4, _lib.rollout_row_width(pol.desc), device="cuda"), th.zeros(2 * 1000 + 8000, device="cuda")
    with pytest.raises(_lib.ImbError, match="unknown env kind 7|takes d_obs"):
        _lib.rollout(unknown if env == ce.PENDULUM else bad, None, venv.obs, pol.desc, pp, pn, None, None, None, 0,
                     _hp(), 1000, 4, tbl, None, 0, None, aux, None, venv.state)


# ---------------------------------------------------------------------------------------------------------------------
# Pendulum's action bounds [-2, 2]
# ---------------------------------------------------------------------------------------------------------------------
def test_pendulum_action_bounds():
    from imitation_b200 import _lib
    from imitation_b200.envs import ClassicVecEnv
    from imitation_b200.rewards import reward_nets

    E, H = 512, 50
    venv = ClassicVecEnv(ce.PENDULUM, E, horizon=H, seed=4)
    spec = ce.ClassicEnvSpec(ce.PENDULUM, horizon=H, seed=4)
    pol = _policy(venv, log_std_init=1.5)  # std 4.5: most sampled torques fall outside [-2, 2]
    pp, pn, _ = pol.flat_vectors()
    rw, tw = _lib.rollout_row_width(pol.desc), 2 * 3 + 1 + 1
    th.manual_seed(5)
    net = reward_nets.BasicRewardNet(venv.observation_space, venv.action_space).cuda()
    eng = net.engine()
    venv.reset()
    tbl, flat = th.zeros(E * H, rw, device="cuda"), th.zeros(E * H, tw, device="cuda")
    aux = th.zeros(2 * E + 2 * E * H, device="cuda")
    _lib.rollout(venv.desc, None, venv.obs, pol.desc, pp, pn, eng.desc, eng.params, eng.norm_state, 2, _hp(), E, H,
                 tbl, None, 0, flat, aux, None, venv.state, act=pol.act)
    rows, fl = tbl.cpu().numpy(), flat.cpu().numpy()
    act, ctl = rows[:, 3], fl[:, 3]
    assert (act > 2).mean() > 0.2 and (act < -2).mean() > 0.2  # recorded unclipped (SB3 stores the raw sample)
    np.testing.assert_array_equal(ctl, np.clip(act, -2.0, 2.0))  # the env and the reward net see the clipped one
    assert ctl.max() == 2.0 and ctl.min() == -2.0
    nobs, rew = spec.dynamics(fl[:, :3], ctl[:, None])
    _close_ulp(fl[:, 4:7], nobs, "next obs on the clipped torque")
    # the reward net's raw output on (obs, clipped act, next obs, done), not on the unclipped action
    args = (fl[:, :3], ctl[:, None], fl[:, 4:7], fl[:, 7] > 0.5)
    np.testing.assert_allclose(rows[:, 3 + 1 + 2], net.predict(*args), rtol=1e-5, atol=1e-5)
    assert not np.allclose(rows[:, 3 + 1 + 2], net.predict(args[0], act[:, None], args[2], args[3]), atol=1e-3)

    # exploration steps: uniform on [-2, 2]
    venv2 = ClassicVecEnv(ce.PENDULUM, E, horizon=H, seed=4)
    venv2.reset()
    xt, xf = th.zeros(E * H, rw, device="cuda"), th.zeros(E * H, tw, device="cuda")
    xa = th.zeros(2 * E + 2 * E * H, device="cuda")
    _lib.rollout_explore(venv2.desc, None, venv2.obs, pol.desc, pp, pn, None, None, None, None, 0, _hp(), E, H, xt, xf,
                         xa, None, th.ones(H, dtype=th.uint8, device="cuda"), 99, 0, venv2.state, act=pol.act)
    u = xt.cpu().numpy()[:, 3]
    assert u.min() >= -2.0 and u.max() <= 2.0 and u.min() < -1.99 and u.max() > 1.99
    assert np.histogram(u, bins=8, range=(-2, 2))[0].min() > 0.8 * len(u) / 8
    np.testing.assert_array_equal(xf.cpu().numpy()[:, 3], u)

    # DAgger labels: the expert's action clipped to the Box
    venv3 = ClassicVecEnv(ce.PENDULUM, E, horizon=H, seed=4)
    venv3.reset()
    learner = _policy(venv3)
    lp, ln, _ = learner.flat_vectors()
    dt, df = th.zeros(E * H, rw, device="cuda"), th.zeros(E * H, tw, device="cuda")
    da_ = th.zeros(2 * E + 2 * E * H, device="cuda")
    mask = th.zeros(H, E, dtype=th.uint8, device="cuda")
    _lib.rollout_dagger(venv3.desc, None, venv3.obs, pol.desc, pp, pn, learner.desc, lp, ln, E, H, dt, df, da_, None,
                        None, mask, venv3.state, expert_act=pol.act, learner_act=learner.act)
    labels = dt.cpu().numpy()[:, 3]
    assert labels.min() == -2.0 and labels.max() == 2.0 and (np.abs(labels) == 2.0).mean() > 0.3
    np.testing.assert_array_equal(df.cpu().numpy()[:, 3], labels)


# ---------------------------------------------------------------------------------------------------------------------
# every trainer runs on both envs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", ENVS)
def test_make_vec_env_builds_the_device_env(env):
    from imitation_b200.algorithms.preference_comparisons import make_seeds
    from imitation_b200.envs import DeviceVecEnv, make_vec_env

    rng, ref = np.random.default_rng(3), np.random.default_rng(3)
    venv = make_vec_env(env, rng=rng, n_envs=16)
    assert isinstance(venv, DeviceVecEnv) and venv.num_envs == 16 and venv.seed == make_seeds(ref, 16)[0]
    assert venv.horizon == (500 if env == ce.CARTPOLE else 200) and venv.params is None
    assert make_vec_env(env, rng=rng, n_envs=4, max_episode_steps=20).horizon == 20
    obs = venv.reset()
    assert obs.shape == (16, venv.d_obs) and np.isfinite(obs).all()


@pytest.mark.parametrize("env", ENVS)
def test_every_trainer_runs(env, tmp_path):
    from imitation_b200.algorithms import bc, dagger, density, ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.algorithms.adversarial import airl, gail
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    H = 20
    mk = lambda n=8: make_vec_env(env, rng=np.random.default_rng(1), n_envs=n, max_episode_steps=H)  # noqa: E731
    demos = _demos(env)[:4]
    th.manual_seed(0)

    # DevicePPO.learn on the env reward
    venv = mk()
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=H, batch_size=32, n_epochs=1, seed=0)
    algo.learn(3 * 8 * H)
    assert algo.num_timesteps == 3 * 8 * H

    # generate_trajectories + rollout_stats
    trajs = rollout.generate_trajectories(algo, venv, rollout.make_min_episodes(12), np.random.default_rng(0))
    assert len(trajs) == 16 and all(len(t.acts) == H and t.obs.shape == (H + 1, venv.d_obs) for t in trajs)
    assert all(np.isfinite(t.obs).all() and np.isfinite(t.rews).all() for t in trajs)
    if env == ce.PENDULUM:
        assert all(np.abs(t.acts).max() <= 2.0 for t in trajs)
    stats = rollout.rollout_stats(trajs)
    assert stats["n_traj"] == 16 and stats["len_mean"] == H and np.isfinite(stats["return_mean"])

    # GAIL and AIRL
    for cls, net_cls in ((gail.GAIL, reward_nets.BasicRewardNet), (airl.AIRL, reward_nets.BasicShapedRewardNet)):
        venv = mk()
        gen = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=H, batch_size=32, n_epochs=1, seed=0)
        net = net_cls(venv.observation_space, venv.action_space, normalize_input_layer=networks.RunningNorm)
        tr = cls(demonstrations=demos, demo_batch_size=64, venv=venv, gen_algo=gen, reward_net=net)
        tr.train(2 * 8 * H)
        assert gen.num_timesteps == 2 * 8 * H
        assert all(th.isfinite(p).all() for p in net.parameters())

    # AgentTrainer with exploration
    venv = mk()
    reward = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space, venv.action_space),
                                             networks.RunningNorm).cuda()
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=H, batch_size=32, n_epochs=1, seed=0)
    agent = pc.AgentTrainer(algo, reward, venv, np.random.default_rng(0), exploration_frac=0.5)
    agent.train(2 * 8 * H)
    sampled = agent.sample(4 * H)
    assert len(sampled) >= 4 and all(np.isfinite(t.obs).all() and np.isfinite(t.rews).all() for t in sampled)
    if env == ce.PENDULUM:
        assert all(np.abs(t.acts).max() <= 2.0 for t in sampled)

    # SimpleDAggerTrainer, the expert a DevicePPO policy
    venv = mk()
    rng = np.random.default_rng(2)
    learner = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng, batch_size=32)
    expert = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=H, seed=1).policy
    dtr = dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp_path / "dagger", expert_policy=expert, rng=rng,
                                     bc_trainer=learner)
    dtr.train(2 * 8 * H, rollout_round_min_episodes=1, rollout_round_min_timesteps=8 * H,
              bc_train_kwargs=dict(n_epochs=1))
    assert dtr.round_num >= 1
    assert all(th.isfinite(p).all() for p in learner.policy.parameters())

    # DensityAlgorithm in rollout mode
    venv = mk()
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=H, batch_size=32, n_epochs=1, seed=0)
    dens = density.DensityAlgorithm(demonstrations=demos, venv=venv, rng=np.random.default_rng(0), rl_algo=algo,
                                    density_type=density.DensityType.STATE_ACTION_DENSITY, kernel_bandwidth=0.5)
    dens.train()
    dens.train_policy(2 * 8 * H)
    assert algo.num_timesteps == 2 * 8 * H
    stats = dens.test_policy(n_trajectories=8)
    assert stats["n_traj"] >= 8 and np.isfinite(stats["return_mean"])


# ---------------------------------------------------------------------------------------------------------------------
# something learns
# ---------------------------------------------------------------------------------------------------------------------
def test_bc_on_the_cartpole_expert_demos_balances_the_pole():
    """BC with the reference's defaults (FeedForward32Policy, batch 32, Adam at 1e-3, ent_weight 1e-3) trained for 4
    epochs on the 26 964 transitions of the cartpole_0 expert rollouts, then 64 deterministic episodes on
    make_vec_env("seals/CartPole-v0", n_envs=64).  Measured on an H100 80GB HBM3 at a 700 W power limit
    (profiles/classic_control_bench.py, same seeds): the untrained policy's return_mean is 8.0, the trained one's 499.7
    of 500."""
    from imitation_b200.algorithms import bc
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env

    rng = np.random.default_rng(0)
    th.manual_seed(0)
    venv = make_vec_env("seals/CartPole-v0", rng=rng, n_envs=64)
    trainer = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng,
                    demonstrations=_demos(ce.CARTPOLE))

    def evaluate():
        trajs = rollout.generate_trajectories(trainer.policy, venv, rollout.make_min_episodes(64),
                                              np.random.default_rng(1), deterministic_policy=True)
        return rollout.rollout_stats(trajs)["return_mean"]

    before = evaluate()
    trainer.train(n_epochs=4)
    after = evaluate()
    print(f"BC on seals/CartPole-v0: return_mean {before:.1f} untrained, {after:.1f} trained")
    assert after >= 400 and after >= 5 * before, (before, after)
