"""GPU: the device SAC -- the gradient step against the float64 SAC step of oracle/sac_port.py at every shape class it
accepts, the learner ring after a learn() against the env dynamics and the Philox streams, a whole SQIL(SAC).train
against SB3's loop replayed in float64, determinism, the reference's continuous SQIL tests with SAC, evaluation, and
learning on Pendulum-v1 from the pendulum_0 demonstrations."""
import os

import numpy as np
import pytest
import torch as th
from scipy import stats

from oracle import classic_env as ce
from oracle import philox, sac_port
from oracle import synth_env

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "expert_models")
STREAM_SAC_ACT, STREAM_SAC_RANDOM, STREAM_SAC_STEP = 0x9009, 0xA00A, 0xB00B


def _demos():
    from imitation_b200.data import serialize

    return serialize.load(os.path.join(GOLDEN, "pendulum_0", "rollouts", "final.npz"))


def _transitions():
    from imitation_b200.data import rollout

    return rollout.flatten_trajectories(_demos())


def _sqil(n_envs=1, seed=0, demos=None, venv=None, **rl_kwargs):
    from imitation_b200.algorithms import sac, sqil
    from imitation_b200.envs import make_vec_env

    if venv is None:
        venv = make_vec_env("Pendulum-v1", rng=np.random.default_rng(seed), n_envs=n_envs)
    return sqil.SQIL(venv=venv, demonstrations=_transitions() if demos is None else demos, policy="MlpPolicy",
                     rl_algo_class=sac.SAC, rl_kwargs=rl_kwargs)


def _state64(pol, log_ent_coef):
    d = (pol.d_obs, pol.d_act, pol.hidden)
    f = lambda t: t.detach().double().cpu().numpy()
    return sac_port.SACState(sac_port.actor_params(f(pol.actor_flat()), *d), sac_port.critic_params(f(pol.critic_flat()), *d),
                             sac_port.critic_params(f(pol.target_flat()), *d), log_ent_coef)


def _step_eps(seed, B, n, Da):
    z = philox.normals(seed, STREAM_SAC_STEP, np.arange(B, dtype=np.uint32), np.uint32(n), 16).astype(np.float64)
    return z[:, :Da], z[:, 8:8 + Da]


def _close_but_for_sign_flips(got, want, lr, g):
    """Adam moves each weight by about lr per step, whatever the gradient's size, so the float32 step agrees with the
    float64 one to a small part of lr * g (1e-2 of it here, far below what a wrong gradient term would give) -- except
    where a gradient component is as small as the float32 rounding of its sum, where m / sqrt(v) may take either sign
    and the two differ by up to 2 lr per step.  Those must stay rare (<= 0.2 % of the entries) and within that bound."""
    got, want = np.asarray(got).ravel(), np.asarray(want).ravel()
    d = np.abs(got - want)
    tight = 1e-2 * lr * g + 1e-6 * np.abs(want) + 1e-7
    assert np.mean(d > tight) <= 2e-3, (np.max(d), np.mean(d > tight))
    assert np.all(d <= 2 * lr * g + 1e-6 * np.abs(want) + 1e-6), np.max(d)


def _moments_close(got, want):
    """Adam moments: m = sum of 0.1 g terms, v of 0.001 g^2 terms; the float32 gradients agree with the float64 ones to
    float32 rounding of their sums, so each moment to 1e-2 relative, with an absolute floor of 1e-3 of the vector's
    largest entry for the components whose gradient is itself at rounding level."""
    got, want = np.asarray(got).ravel(), np.asarray(want).ravel()
    np.testing.assert_allclose(got, want, rtol=1e-2, atol=1e-3 * np.abs(want).max() + 1e-12)


def _flat64(dicts, keys):
    return np.concatenate([d[k].ravel() for d in dicts for k in keys])


@pytest.mark.parametrize("ent", ["auto", 0.2])
@pytest.mark.parametrize("B", [2, 33, 256])
@pytest.mark.parametrize("Do, Da", [(3, 1), (17, 6), (64, 8)])
@pytest.mark.parametrize("h", [32, 64, 96, 256])
def test_sac_step_matches_the_float64_step(h, Do, Da, B, ent):
    """g = 3 steps in one call, ent_coef "auto" (log_ent_coef 0.1) or fixed 0.2, target_update_interval 2 (Polyak at
    steps 0 and 2), targets that differ from the critics, expert actions at env scale (+-2) beside buffer actions in
    [-1, 1].  Losses agree to 1e-4 relative (plus 1e-6 absolute: a float32 sum of terms of order 1 is not resolved
    more finely than that), parameters and targets as `_close_but_for_sign_flips` says, every Adam moment as
    `_moments_close` says."""
    from imitation_b200 import _lib, spaces
    from imitation_b200.algorithms import sac

    auto = ent == "auto"
    th.manual_seed(h * 7 + Do + B)
    r = np.random.default_rng(h + Do + B)
    pol = sac.SACPolicy(spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1, 1, (Da,)), net_arch=[h, h]).cuda()
    with th.no_grad():
        for p in pol.critic_target.parameters():
            p.add_(0.05 * th.randn_like(p))
    a, c, t = pol.actor_flat(), pol.critic_flat(), pol.target_flat()
    tw, C, Ne, G = 2 * Do + Da + 1, 300, 77, 3
    ring = r.standard_normal((tw, C)).astype(np.float32)
    ring[Do:Do + Da] = r.uniform(-1, 1, (Da, C))
    ring[-1] = r.random(C) < 0.3
    expert = r.standard_normal((tw, Ne)).astype(np.float32)
    expert[Do:Do + Da] = r.uniform(-2, 2, (Da, Ne))
    expert[-1] = r.random(Ne) < 0.3
    n_l, n_e = B // 2, B - B // 2
    lidx, eidx = r.integers(0, C, (G, n_l)), r.integers(0, Ne, (G, n_e))
    st = _state64(pol, 0.1 if auto else None)
    if not auto:
        st.ent_coef = 0.2
    lr, seed = 1e-3, 1234 + h
    hp = dict(d_obs=Do, d_act=Da, hidden=h, batch_size=B, gamma=0.99, tau=0.05, lr=lr, adam_eps=1e-8, auto_ent=auto,
              ent_coef=0.0 if auto else 0.2, target_entropy=-float(Da), reward_learner=0.0, reward_expert=1.0,
              target_update_interval=2, seed=seed)
    ent_t = th.tensor([0.1 if auto else 0.0, 0.0, 0.0], device="cuda")
    am, av, cm, cv = th.zeros_like(a), th.zeros_like(a), th.zeros_like(c), th.zeros_like(c)
    state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
    loss_log = th.zeros(G, 4, device="cuda")
    ws = th.zeros(_lib.sac_ws_floats(Do, Da, h, B), device="cuda")
    _lib.sac_step(hp, a, am, av, c, cm, cv, t, ent_t, th.as_tensor(ring).cuda(), C, th.as_tensor(lidx).cuda(),
                  th.as_tensor(expert).cuda(), Ne, th.as_tensor(eidx).cuda(), G, 0, loss_log, ws, state)
    th.cuda.synchronize()
    ring64, exp64 = ring.astype(np.float64), expert.astype(np.float64)
    log = loss_log.cpu().numpy()
    for s in range(G):
        src = np.concatenate([ring64[:, lidx[s]], exp64[:, eidx[s]]], 1)
        eps, eps_n = _step_eps(seed, B, s, Da)
        want = sac_port.sac_step(st, src[:Do].T, src[Do:Do + Da].T, src[Do + Da:2 * Do + Da].T, src[-1],
                                 np.r_[np.zeros(n_l), np.ones(n_e)], eps, eps_n, gamma=0.99, tau=0.05, lr=lr,
                                 target_entropy=-float(Da), polyak=s % 2 == 0)
        for col, k in enumerate(("critic_loss", "actor_loss", "ent_coef_loss", "ent_coef")):
            if k in want:
                assert abs(log[s, col] - want[k]) <= 1e-4 * abs(want[k]) + 1e-6, (s, k, log[s, col], want[k])
    assert int(state[_lib.ST_PPO_STEP]) == G
    got = _state64(pol, None)
    for k in sac_port.ACTOR_KEYS:
        _close_but_for_sign_flips(got.actor[k], st.actor[k], lr, G)
    for i in range(2):
        for k in sac_port.Q_KEYS:
            _close_but_for_sign_flips(got.critic[i][k], st.critic[i][k], lr, G)
            _close_but_for_sign_flips(got.target[i][k], st.target[i][k], lr, G)
    _moments_close(cm.cpu().numpy(), _flat64(st.cm, sac_port.Q_KEYS))
    _moments_close(cv.cpu().numpy(), _flat64(st.cv, sac_port.Q_KEYS))
    _moments_close(am.cpu().numpy(), _flat64([st.am], sac_port.ACTOR_KEYS))
    _moments_close(av.cpu().numpy(), _flat64([st.av], sac_port.ACTOR_KEYS))
    if auto:
        assert abs(ent_t[0].item() - st.log_ent_coef) <= 1e-2 * lr * G
        assert abs(ent_t[1].item() - st.em) <= 1e-3 * abs(st.em) + 1e-7
        assert abs(ent_t[2].item() - st.ev) <= 1e-3 * abs(st.ev) + 1e-9
    else:
        assert not ent_t.any()  # a fixed coefficient: the log_ent_coef vector is not touched


def _actor_buffer_actions(pol, obs, eps, low, high):
    """scale(unscale(tanh(mean + std eps))) of the float64 actor (float32 scaling, as the device)."""
    from imitation_b200.algorithms import sac

    p = sac_port.actor_params(pol.actor_flat().double().cpu().numpy(), pol.d_obs, pol.d_act, pol.hidden)
    _, _, mean, ls, _ = sac_port.actor_forward(p, obs.astype(np.float64))
    a = np.tanh(mean + eps * np.exp(ls)).astype(np.float32)
    return sac.scale_action(sac.unscale_action(a, low, high), low, high)


@pytest.mark.parametrize("env_kind", ["pendulum", "synth"])
def test_learner_ring_after_learn_follows_the_env_and_the_streams(env_kind):
    """train_freq 3 (which does not divide the horizon), learning_starts inside the run, a ring of 128 positions that
    wraps, learning_rate 0 so the actor that acts stays fixed.  Every stored transition must be the env's step of its obs
    and env action unscale(buffer action), a random step's buffer action scale(lo + u (hi - lo)) of the Philox uniforms,
    an actor step's scale(unscale(tanh(mean + std eps))), done 1 exactly at the horizon, and obs continuous across rows
    except after a done."""
    from imitation_b200.algorithms import sac
    from imitation_b200.envs import synth

    E, T, steps, P = 2, 3, 330, 128
    if env_kind == "pendulum":
        algo = _sqil(E, learning_starts=250 * E, buffer_size=P * E, train_freq=T, learning_rate=0.0, seed=3,
                     batch_size=64, policy_kwargs=dict(net_arch=[64, 64]))
        step = lambda o, u: ce.pendulum_step(o, u)[0]
        hi = 2.0
    else:
        venv = synth.DeviceVecEnv(17, 6, E, horizon=100, seed=5)
        spec = synth_env.SynthEnvSpec(17, 6, horizon=100, seed=5)
        r = np.random.default_rng(0)
        from imitation_b200.data import types
        demos = types.Transitions(obs=r.standard_normal((300, 17)).astype(np.float32),
                                  acts=r.uniform(-1, 1, (300, 6)).astype(np.float32), infos=np.array([{}] * 300),
                                  next_obs=r.standard_normal((300, 17)).astype(np.float32), dones=np.zeros(300, bool))
        algo = _sqil(venv=venv, demos=demos, learning_starts=250 * E, buffer_size=P * E, train_freq=T,
                     learning_rate=0.0, seed=3, batch_size=64, policy_kwargs=dict(net_arch=[64, 64]))
        step = lambda o, u: spec.dynamics(o, u)[0]
        hi = 1.0
    m = algo.rl_algo
    np.random.seed(7)
    algo.train(total_timesteps=steps * E)
    assert m.graph_replays > 0
    buf = m.replay_buffer
    assert buf.full and buf.pos == (steps // T * T) % P
    Do, Da = m.env.d_obs, m.env.d_act
    obs, acts, nobs, dones = buf.observations, buf.actions, buf.next_observations, buf.dones
    ctl = sac.unscale_action(acts.reshape(-1, Da), -hi, hi)
    np.testing.assert_allclose(step(obs.reshape(-1, Do), ctl), nobs.reshape(-1, Do), rtol=0, atol=2e-5)
    explore = m.last_schedule.explore
    H = m.env.horizon
    n_steps = len(explore)
    n_rand = n_actor = 0
    for g in range(n_steps - P, n_steps):
        p = g % P
        if explore[g]:
            u = ce.uniforms(m._seed(), STREAM_SAC_RANDOM, np.arange(E), g, Da)
            want = sac.scale_action(np.float32(-hi) + u * np.float32(2 * hi), -hi, hi)
            np.testing.assert_array_equal(acts[p], want)
            n_rand += 1
        else:
            eps = philox.normals(m._seed(), STREAM_SAC_ACT, np.arange(E, dtype=np.uint32), np.uint32(g), Da)
            want = _actor_buffer_actions(m.policy, obs[p], eps.astype(np.float64), -hi, hi)
            np.testing.assert_allclose(acts[p], want, rtol=0, atol=2e-5)
            n_actor += 1
        done = (g + 1) % H == 0
        assert (dones[p] == float(done)).all()
        if g + 1 < n_steps:
            same = np.all(obs[(g + 1) % P] == nobs[p], axis=1)
            assert same.all() if not done else not same.any()
    assert n_rand > 10 and n_actor > 10


@pytest.mark.parametrize("n_envs, gradient_steps", [(1, 1), (4, 1), (1, 2), (4, 2)])
def test_sqil_sac_train_matches_the_sb3_loop_replayed_in_float64(n_envs, gradient_steps):
    """A whole SQIL(SAC).train: the oracle walks SB3's learn loop from the same NumPy seed and replays every gradient
    step in float64 on the rows of the device's buffers (the ring never wraps), with the device's step noise."""
    kw = dict(learning_starts=40, learning_rate=1e-3, batch_size=32, buffer_size=10_000, seed=11,
              gradient_steps=gradient_steps, target_update_interval=2, policy_kwargs=dict(net_arch=[32, 32]))
    total = 100 * n_envs
    algo = _sqil(n_envs, **kw)
    m = algo.rl_algo
    st = _state64(m.policy, 0.0)
    np.random.seed(123)
    algo.train(total_timesteps=total)
    buf = m.replay_buffer
    ring = buf.ring.double().cpu().numpy()
    expert = buf.expert_table.double().cpu().numpy()
    port = sac_port.SACLearnLoopPort(n_envs=n_envs, n_expert=buf.n_expert, buffer_size=kw["buffer_size"],
                                     learning_starts=kw["learning_starts"], batch_size=32,
                                     gradient_steps=gradient_steps)
    losses, n = [], [0]

    def train_fn(sample, gi):
        bi, ei, xi = sample
        src = np.concatenate([ring[:, bi * n_envs + ei], expert[:, xi]], 1)
        eps, eps_n = _step_eps(m._seed(), 32, n[0], 1)
        n[0] += 1
        losses.append(sac_port.sac_step(st, src[:3].T, src[3:4].T, src[4:7].T, src[7],
                                        np.r_[np.zeros(len(bi)), np.ones(len(xi))], eps, eps_n, gamma=0.99, tau=0.005,
                                        lr=1e-3, target_entropy=-1.0, polyak=gi % 2 == 0))

    np.random.seed(123)
    port.learn(total, train_fn=train_fn)
    assert m._n_updates == port._n_updates == len(losses) > 0
    assert m.graph_replays > 0
    np.testing.assert_array_equal(m.last_schedule.explore, port.random_steps)
    got = _state64(m.policy, None)
    g = len(losses)
    for k in sac_port.ACTOR_KEYS:
        _close_but_for_sign_flips(got.actor[k], st.actor[k], 1e-3, g)
    for i in range(2):
        for k in sac_port.Q_KEYS:
            _close_but_for_sign_flips(got.critic[i][k], st.critic[i][k], 1e-3, g)
    dev = m._last_losses.cpu().numpy()
    want = np.array([[x["critic_loss"], x["actor_loss"], x["ent_coef_loss"], x["ent_coef"]] for x in losses])
    np.testing.assert_allclose(dev, want, rtol=1e-3, atol=1e-4)
    assert m._last_logged["train/n_updates"] == g
    assert set(m._last_logged) == {"train/n_updates", "train/ent_coef", "train/actor_loss", "train/critic_loss",
                                   "train/ent_coef_loss", "train/learning_rate"}


def test_two_identical_runs_are_bit_identical():
    outs = []
    for _ in range(2):
        th.manual_seed(4)
        algo = _sqil(2, learning_starts=50, seed=4, batch_size=64, policy_kwargs=dict(net_arch=[64, 64]))
        np.random.seed(9)
        algo.train(total_timesteps=400)
        p = algo.rl_algo.policy
        outs.append([x.clone() for x in (p.actor_flat(), p.critic_flat(), p.target_flat(), algo.rl_algo._ent)])
    for a, b in zip(*outs):
        assert th.equal(a, b)


def test_sqil_no_crash_continuous():
    """The reference's test_sqil_no_crash_continuous with SAC: 500 steps on Pendulum-v1 (SB3's defaults)."""
    algo = _sqil(1)
    algo.train(total_timesteps=500)
    assert algo.rl_algo.num_timesteps == 500


def test_sqil_few_demonstrations_continuous():
    """The reference's test_sqil_few_demonstrations_continuous with SAC: 5 demonstrations, 100 steps."""
    demos = _transitions()[:5]
    algo = _sqil(1, demos=demos)
    algo.train(total_timesteps=100)
    assert algo.rl_algo.replay_buffer.n_expert == 5


@pytest.mark.parametrize("data_type", ["trajectories", "transitions"])
def test_sqil_sac_demonstration_buffer(data_type):
    from imitation_b200.algorithms import sqil

    demos = _demos() if data_type == "trajectories" else _transitions()
    model = _sqil(1, demos=demos)
    assert isinstance(model.rl_algo.replay_buffer, sqil.SQILReplayBuffer)
    eb = model.rl_algo.replay_buffer.expert_buffer
    d = _transitions()
    assert eb.actions.shape == (len(d), 1, 1)
    for i in range(0, len(d), 97):
        np.testing.assert_array_equal(eb.observations[i][0], d.obs[i])
        np.testing.assert_array_equal(eb.actions[i][0], d.acts[i])  # env scale, as recorded
        np.testing.assert_array_equal(eb.next_observations[i][0], d.next_obs[i])
        np.testing.assert_array_equal(eb.dones[i], d.dones[i])


def test_deterministic_generate_trajectories_returns_predicts_action_and_pendulum_rewards():
    from imitation_b200.algorithms import sac
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env

    algo = _sqil(1, policy_kwargs=dict(net_arch=[64, 64]), seed=2)
    env = make_vec_env("Pendulum-v1", rng=np.random.default_rng(1), n_envs=3)
    trajs = rollout.generate_trajectories(algo.rl_algo, env, rollout.make_min_episodes(3), np.random.default_rng(0),
                                          deterministic_policy=True)
    pol = algo.policy
    p = sac_port.actor_params(pol.actor_flat().double().cpu().numpy(), 3, 1, 64)
    for tr in trajs:
        assert len(tr.acts) == 200 and tr.obs.shape == (201, 3)
        _, _, mean, _, _ = sac_port.actor_forward(p, tr.obs[:-1].astype(np.float64))
        want = sac.unscale_action(np.tanh(mean).astype(np.float32), -2, 2)  # predict(deterministic=True)
        np.testing.assert_allclose(tr.acts, want, rtol=0, atol=3e-5)
        nxt, rew = ce.pendulum_step(tr.obs[:-1], tr.acts)
        np.testing.assert_allclose(nxt, tr.obs[1:], rtol=0, atol=2e-5)
        np.testing.assert_allclose(rew, tr.rews, rtol=1e-5, atol=1e-5)


def is_significant_reward_improvement(old_rewards, new_rewards, p_value: float = 0.05) -> bool:
    res = stats.permutation_test((old_rewards, new_rewards),
                                 statistic=lambda x, y, axis: np.mean(x, axis=axis) - np.mean(y, axis=axis),
                                 vectorized=True, alternative="less")
    return res.pvalue < p_value


def test_sqil_sac_learns_pendulum():
    """SQIL(SAC) on Pendulum-v1 with the pendulum_0 demonstrations, SB3's SAC defaults, seed 42, 20 000 steps; 100
    evaluation episodes of the deterministic policy before and after, the reference's permutation test."""
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env

    algo = _sqil(1, seed=42)
    eval_env = make_vec_env("Pendulum-v1", rng=np.random.default_rng(42), n_envs=100)

    def returns():
        trajs = rollout.generate_trajectories(algo.policy, eval_env, rollout.make_min_episodes(100),
                                              np.random.default_rng(42), deterministic_policy=True)
        return [float(np.sum(t.rews)) for t in trajs[:100]]

    before = returns()
    np.random.seed(42)
    algo.train(total_timesteps=20_000)
    after = returns()
    print(f"SQIL(SAC) Pendulum-v1: return {np.mean(before):.1f} -> {np.mean(after):.1f}")
    assert is_significant_reward_improvement(before, after)
