"""GPU: SQIL's device path -- the TD target pass and TD step against the float64 DQN step, the learner ring after a
learn() against the CartPole dynamics and the random-action stream, a whole SQIL.train against the SB3 learn loop of
oracle/sqil_port.py replayed in float64, the expert buffer, and the reference's test_sqil_performance_discrete."""
import os

import numpy as np
import pytest
import torch as th
from scipy import stats
from torch import nn

from imitation_b200 import _lib
from oracle import classic_env as ce
from oracle import exploration_port, sqil_port

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "expert_models")


def _demos():
    from imitation_b200.data import serialize

    return serialize.load(os.path.join(GOLDEN, "cartpole_0", "rollouts", "final.npz"))


def _transitions():
    from imitation_b200.data import rollout

    return rollout.flatten_trajectories(_demos())


def _params64(flat, pol):
    """The Q-net's layers out of a flat policy image, float64 (sqil_port's dict)."""
    d = pol.desc
    f = flat.detach().double().cpu().numpy()
    h, Do, A = pol.hidden, pol.d_obs, pol.d_act
    return {"w1": f[d.off_pi_w1:d.off_pi_w1 + h * Do].reshape(h, Do), "b1": f[d.off_pi_b1:d.off_pi_b1 + h],
            "w2": f[d.off_pi_w2:d.off_pi_w2 + h * h].reshape(h, h), "b2": f[d.off_pi_b2:d.off_pi_b2 + h],
            "w3": f[d.off_act_w:d.off_act_w + A * h].reshape(A, h), "b3": f[d.off_act_b:d.off_act_b + A]}


def _sqil(n_envs=1, seed=0, **rl_kwargs):
    from imitation_b200.algorithms import sqil
    from imitation_b200.envs import make_vec_env

    venv = make_vec_env("seals/CartPole-v0", rng=np.random.default_rng(seed), n_envs=n_envs)
    return sqil.SQIL(venv=venv, demonstrations=_transitions(), policy="MlpPolicy", rl_kwargs=rl_kwargs)


@pytest.mark.parametrize("B", [32, 220, 33])
def test_td_step_matches_the_float64_dqn_step(B):
    from imitation_b200 import _lib
    from imitation_b200.algorithms import dqn

    th.manual_seed(B)
    r = np.random.default_rng(B)
    from imitation_b200 import spaces

    pol = dqn.DQNPolicy(spaces.Box(-np.inf, np.inf, (4,)), spaces.Discrete(2)).cuda()
    with th.no_grad():  # a target that differs from the Q-net
        for p in pol.q_net_target.parameters():
            p.add_(0.1 * th.randn_like(p))
    q, tgt = pol.q_flat(), pol.target_flat()
    Do, A, tw, C, Ne = 4, 2, 11, 300, 77
    ring = th.as_tensor(r.standard_normal((tw, C)), dtype=th.float32).cuda()
    expert = th.as_tensor(r.standard_normal((tw, Ne)), dtype=th.float32).cuda()
    for t, n in ((ring, C), (expert, Ne)):
        a = r.integers(0, A, n)
        t[Do:Do + A] = 0
        t[Do + a, th.arange(n)] = 1
        t[2 * Do + A] = th.as_tensor((r.random(n) < 0.3).astype(np.float32))
    n_l, n_e, G = B // 2, B - B // 2, 3
    lidx, eidx = r.integers(0, C, (G, n_l)), r.integers(0, Ne, (G, n_e))
    rw = _lib.rollout_row_width(pol.desc)
    rows = th.zeros(G * B, rw, device="cuda")
    m, v = th.zeros_like(q), th.zeros_like(q)
    state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
    loss_log = th.zeros(G, 4, device="cuda")
    p64, pt64 = _params64(q, pol), _params64(tgt, pol)
    m64 = {k: np.zeros_like(x) for k, x in p64.items()}
    v64 = {k: np.zeros_like(x) for k, x in p64.items()}
    ring64, exp64 = ring.double().cpu().numpy(), expert.double().cpu().numpy()
    lr, mgn = 2e-3, 1.0
    # one target pass for the G steps (the target does not move inside a train() call), then G TD steps in one launch
    _lib.dqn_target(pol.desc, tgt, ring, C, th.as_tensor(lidx).cuda(), expert, Ne, th.as_tensor(eidx).cuda(), n_l, n_e,
                    G, 0.99, 0.0, 1.0, rows)
    _lib.dqn_step(pol.desc, q, m, v, rows, B, G, lr, 1e-8, mgn, loss_log, state)
    rows_h = rows.cpu().numpy()
    for s in range(G):
        src = np.concatenate([ring64[:, lidx[s]], exp64[:, eidx[s]]], 1)
        obs, acts = src[:Do].T, src[Do:Do + A].argmax(0)
        y = sqil_port.td_targets(pt64, src[Do + A:2 * Do + A].T, src[2 * Do + A], np.r_[np.zeros(n_l), np.ones(n_e)],
                                 0.99)
        got = rows_h[s * B:(s + 1) * B]
        np.testing.assert_array_equal(got[:, :Do], obs.astype(np.float32))
        np.testing.assert_array_equal(got[:, Do], acts)
        np.testing.assert_allclose(got[:, Do + 1], y, rtol=1e-5, atol=1e-5)
        loss = sqil_port.td_step(p64, m64, v64, s + 1, obs, acts, y, lr, mgn)
        assert abs(loss_log[s, 0].item() - loss) <= 1e-4 * max(1.0, abs(loss))
    got = _params64(q, pol)
    for k in sqil_port.KEYS:  # Adam moves each weight by about lr per step: the float32 step agrees to a small part of it
        np.testing.assert_allclose(got[k], p64[k], rtol=0, atol=2e-3 * lr * G + 1e-6)
    assert int(state[_lib.ST_PPO_STEP]) == G
    # the value tower of the policy image stays zero
    d = pol.desc
    assert not q[d.off_vf_w1:d.off_act_w].any() and not q[d.off_val_w:].any()


@pytest.mark.parametrize("n_envs", [1, 4])
def test_learner_ring_after_learn_follows_cartpole_the_random_stream_and_the_argmax(n_envs):
    """1 200 steps per env with train_freq 3 (which does not divide the horizon of 500, so two horizons fall inside a
    rollout), learning_starts inside the run and exploration_rate 0.5 after it, so random and greedy steps both occur, and
    a ring of 256 positions, so it wraps.  learning_rate 0 keeps the Q-net that acts fixed.  Every transition the ring
    holds must be the CartPole step of its obs and action (the terminal step at the horizon included), a random step's
    action the Philox stream's, a greedy step's the argmax of the Q-net, done 1 exactly at the horizon, and each env's
    next obs the start of its next row except after a done, where a reset observation starts the episode."""
    T, steps, P = 3, 1200, 256
    algo = _sqil(n_envs, learning_starts=300 * n_envs, buffer_size=P * n_envs, train_freq=T, learning_rate=0.0,
                 exploration_fraction=0.01, exploration_final_eps=0.5, seed=3)
    _check_learner_ring(algo, n_envs, steps, P, lambda o, a: ce.cartpole_step(o, a)[0], 2e-6)


@pytest.mark.parametrize("n_envs", [1, 4])
def test_learner_ring_after_learn_follows_the_synthetic_env_the_random_stream_and_the_argmax(n_envs):
    """The CartPole test above on envs.synth.DeviceVecEnv(17, 9, discrete=True) with a tanh [20, 20] Q-net: 399 steps
    per env, horizon 100, a ring of 128 positions.  The transitions must follow oracle.synth_env's dynamics of the
    one-hot control, and every stored action column be one-hot."""
    from imitation_b200.envs import synth
    from oracle import synth_env

    T, steps, P, H = 3, 399, 128, 100
    venv = synth.DeviceVecEnv(17, 9, n_envs, discrete=True, horizon=H, seed=5)
    spec = synth_env.SynthEnvSpec(17, 9, discrete=True, horizon=H, seed=5)
    algo = _sqil_synth(venv, learning_starts=150 * n_envs, buffer_size=P * n_envs, train_freq=T, learning_rate=0.0,
                       exploration_fraction=0.01, exploration_final_eps=0.5, seed=3,
                       policy_kwargs=dict(net_arch=[20, 20], activation_fn=nn.Tanh))
    _check_learner_ring(algo, n_envs, steps, P, lambda o, a: spec.dynamics(o, a)[0], 2e-5)
    cols = algo.rl_algo.replay_buffer._field(17, 9)
    assert set(np.unique(cols)) == {0.0, 1.0} and (cols.sum(-1) == 1).all(), "action columns not one-hot"


def _check_learner_ring(algo, n_envs, steps, P, step_fn, atol):
    dq = algo.rl_algo
    np.random.seed(7)
    algo.train(total_timesteps=steps * n_envs)
    assert dq.graph_replays > 0  # the iterations past the first of each kind ran from CUDA graphs
    buf = dq.replay_buffer
    assert buf.full and buf.pos == steps % P
    assert int(buf.ring_state[0]) == buf.pos
    Do, A = dq.env.d_obs, dq.env.d_act
    obs, acts, nobs, dones = buf.observations, buf.actions[..., 0], buf.next_observations, buf.dones
    nxt = step_fn(obs.reshape(-1, Do), acts.reshape(-1))
    np.testing.assert_allclose(nxt, nobs.reshape(-1, Do), rtol=0, atol=atol)
    explore = dq.last_schedule.explore
    u = exploration_port.random_uniforms(dq._explore_seed(), np.arange(n_envs), 0, steps, A, True)
    want_rand = np.minimum(np.floor(u * np.float32(A)).astype(np.int64), A - 1)
    relu = dq.policy.act == _lib.ACT_RELU
    q = sqil_port.q_forward(_params64(dq.policy.q_flat(), dq.policy), obs.reshape(-1, Do).astype(np.float64), relu)[2]
    q = q.reshape(P, n_envs, A)
    top2 = np.sort(q, -1)[..., -2:]
    H = dq.env.horizon
    n_rand = n_greedy = n_done = 0
    for g in range(steps - P, steps):  # the steps the ring still holds
        p = g % P
        if explore[g]:
            np.testing.assert_array_equal(acts[p], want_rand[g])
            n_rand += 1
        else:
            clear = top2[p, :, 1] - top2[p, :, 0] > 1e-4  # (a near tie may round either way in float32)
            np.testing.assert_array_equal(acts[p][clear], q[p].argmax(1)[clear])
            n_greedy += int(clear.sum())
        done = (g + 1) % H == 0
        assert (dones[p] == float(done)).all()
        n_done += done
        if g + 1 < steps:
            same = np.all(obs[(g + 1) % P] == nobs[p], axis=1)
            assert same.all() if not done else not same.any()
    assert n_rand > 20 and n_greedy > 20 and n_done >= 1
    assert dq.num_timesteps == steps * n_envs


@pytest.mark.parametrize("n_envs", [1, 4])
def test_sqil_train_matches_the_sb3_loop_replayed_in_float64(n_envs):
    """A whole SQIL.train: the oracle walks SB3's learn loop from the same NumPy seed and replays every TD step in
    float64 on the rows of the device's buffers (the ring never wraps, so a row the loop sampled is still in place),
    with the target copied at the loop's target-update calls."""
    kw = dict(learning_starts=60, learning_rate=1e-3, batch_size=33, target_update_interval=24, buffer_size=10_000,
              seed=11, exploration_fraction=0.5)
    _check_train_against_the_sb3_loop(_sqil(n_envs, **kw), kw, [240 * n_envs])


@pytest.mark.parametrize("batch_size", [33, 1])
@pytest.mark.parametrize("n_envs", [1, 4])
def test_two_sqil_trains_on_a_synthetic_env_match_the_sb3_loop_replayed_in_float64(n_envs, batch_size):
    """The test above off CartPole: envs.synth.DeviceVecEnv(17, 9, discrete=True), a tanh [20, 20] Q-net, and two
    consecutive train() calls.  The second starts at a TD step count above 0, so the Adam step count carries over, its
    loss rows are offset and k_dqn_target reads its index lists at s0 = state - step_base > 0.  batch_size 1 has no
    learner rows: every TD step is one expert row."""
    from imitation_b200.envs import synth

    kw = dict(learning_starts=60, learning_rate=1e-3, batch_size=batch_size, target_update_interval=24,
              buffer_size=10_000, seed=11, exploration_fraction=0.5,
              policy_kwargs=dict(net_arch=[20, 20], activation_fn=nn.Tanh))
    algo = _sqil_synth(synth.DeviceVecEnv(17, 9, n_envs, discrete=True, horizon=70, seed=5), **kw)
    _check_train_against_the_sb3_loop(algo, kw, [240 * n_envs, 150 * n_envs])


def _sqil_synth(venv, **rl_kwargs):
    """SQIL on a synthetic Discrete env with 300 expert transitions drawn from the env's own dynamics."""
    from imitation_b200.algorithms import sqil
    from imitation_b200.data import types
    from oracle import synth_env

    spec = synth_env.SynthEnvSpec(venv.d_obs, venv.d_act, discrete=True, horizon=venv.horizon, seed=venv.seed)
    r = np.random.default_rng(0)
    obs = r.standard_normal((300, venv.d_obs)).astype(np.float32) * 0.5
    acts = r.integers(0, venv.d_act, 300)
    demos = types.Transitions(obs=obs, acts=acts, infos=np.array([{}] * 300), next_obs=spec.dynamics(obs, acts)[0],
                              dones=r.random(300) < 0.1)
    return sqil.SQIL(venv=venv, demonstrations=demos, policy="MlpPolicy", rl_kwargs=rl_kwargs)


def _check_train_against_the_sb3_loop(algo, kw, totals):
    """Run algo.train(total) for each total, then walk SB3's loop over the same totals from the same NumPy seed,
    replaying every TD step in float64 on the rows of the device's buffers, with the target copied at the loop's
    target-update calls; the Q-net, its target and every learn()'s losses must agree."""
    dq = algo.rl_algo
    E, Do, A = dq.n_envs, dq.env.d_obs, dq.env.d_act
    relu = dq.policy.act == _lib.ACT_RELU
    p64 = _params64(dq.policy.q_flat(), dq.policy)
    np.random.seed(123)
    dev_losses, explore = [], []
    for total in totals:
        algo.train(total_timesteps=total)
        dev_losses.append(dq._last_losses.cpu().numpy())
        explore.append(dq.last_schedule.explore)
    buf = dq.replay_buffer
    ring = buf.ring.double().cpu().numpy()
    expert = buf.expert_table.double().cpu().numpy()
    B = kw["batch_size"]
    port = sqil_port.LearnLoopPort(n_envs=E, d_obs=Do, n_expert=buf.n_expert, buffer_size=kw["buffer_size"],
                                   learning_starts=kw["learning_starts"], batch_size=B,
                                   target_update_interval=kw["target_update_interval"],
                                   exploration_fraction=kw["exploration_fraction"])
    pt64 = {k: x.copy() for k, x in p64.items()}
    m64 = {k: np.zeros_like(x) for k, x in p64.items()}
    v64 = {k: np.zeros_like(x) for k, x in p64.items()}
    losses, step = [], [0]

    def train_fn(sample):
        bi, ei, xi = sample
        src = np.concatenate([ring[:, bi * E + ei], expert[:, xi]], 1)
        y = sqil_port.td_targets(pt64, src[Do + A:2 * Do + A].T, src[2 * Do + A],
                                 np.r_[np.zeros(len(bi)), np.ones(len(xi))], 0.99, relu)
        step[0] += 1
        losses[-1].append(sqil_port.td_step(p64, m64, v64, step[0], src[:Do].T, src[Do:Do + A].argmax(0), y,
                                            kw["learning_rate"], 10.0, relu=relu))

    def target_fn():
        for k in p64:
            pt64[k] = p64[k].copy()

    np.random.seed(123)
    for total in totals:
        losses.append([])
        port.learn(total, train_fn=train_fn, target_fn=target_fn)
    n = step[0]
    assert dq._n_updates == port._n_updates == n > 0 and all(losses)
    assert dq._n_calls == port._n_calls
    assert dq.exploration_rate == port.exploration_rate
    np.testing.assert_array_equal(np.concatenate(explore), port.random_steps)
    got = _params64(dq.policy.q_flat(), dq.policy)
    for k in sqil_port.KEYS:
        np.testing.assert_allclose(got[k], p64[k], rtol=0, atol=1e-3 * kw["learning_rate"] * n + 1e-6)
    got_t = _params64(dq.policy.target_flat(), dq.policy)
    for k in sqil_port.KEYS:
        np.testing.assert_allclose(got_t[k], pt64[k], rtol=0, atol=1e-3 * kw["learning_rate"] * n + 1e-6)
    for d, l in zip(dev_losses, losses):
        np.testing.assert_allclose(d, l, rtol=1e-3, atol=1e-5)
    assert dq._last_logged["train/n_updates"] == n
    assert abs(dq._last_logged["train/loss"] - losses[-1][-1]) <= 1e-3 * max(1.0, abs(losses[-1][-1]))
    assert dq._last_logged["rollout/exploration_rate"] == port.exploration_rate


@pytest.mark.parametrize("data_type", ["trajectories", "transitions"])
def test_sqil_demonstration_buffer(data_type):
    from imitation_b200.algorithms import sqil
    from imitation_b200.envs import make_vec_env

    venv = make_vec_env("seals/CartPole-v0", rng=np.random.default_rng(0), n_envs=1)
    demos = _demos() if data_type == "trajectories" else _transitions()
    model = sqil.SQIL(venv=venv, demonstrations=demos, policy="MlpPolicy")
    assert isinstance(model.rl_algo.replay_buffer, sqil.SQILReplayBuffer)
    eb = model.rl_algo.replay_buffer.expert_buffer
    d = _transitions()
    assert len(eb.observations) == len(d)
    for i in range(len(d)):
        np.testing.assert_array_equal(eb.observations[i][0], d.obs[i])
        np.testing.assert_array_equal(eb.actions[i][0], d.acts[i])
        np.testing.assert_array_equal(eb.next_observations[i][0], d.next_obs[i])
        np.testing.assert_array_equal(eb.dones[i], d.dones[i])


def is_significant_reward_improvement(old_rewards, new_rewards, p_value: float = 0.05) -> bool:
    """imitation.testing.reward_improvement.is_significant_reward_improvement: a permutation test that the old mean is
    less than the new one."""
    res = stats.permutation_test((old_rewards, new_rewards),
                                 statistic=lambda x, y, axis: np.mean(x, axis=axis) - np.mean(y, axis=axis),
                                 vectorized=True, alternative="less")
    return res.pvalue < p_value


@pytest.mark.parametrize("n_envs", [1, 4])
def test_sqil_performance_discrete(n_envs):
    """The reference's test_sqil_performance_discrete: seals/CartPole-v0, the cartpole_0 demonstrations, DQN with
    learning_starts 500, learning_rate 0.002, batch_size 220, seed 42, 1 000 steps; 100 evaluation episodes of the
    greedy policy before and after."""
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env

    algo = _sqil(n_envs, learning_starts=500, learning_rate=0.002, batch_size=220, seed=42)
    eval_env = make_vec_env("seals/CartPole-v0", rng=np.random.default_rng(42), n_envs=100)

    def returns():
        trajs = rollout.generate_trajectories(algo.policy, eval_env, rollout.make_min_episodes(100),
                                              np.random.default_rng(42))
        return [float(np.sum(t.rews)) for t in trajs[:100]]

    before = returns()
    algo.train(total_timesteps=1_000)
    after = returns()
    print(f"SQIL seals/CartPole-v0 n_envs={n_envs}: return {np.mean(before):.1f} -> {np.mean(after):.1f}")
    assert is_significant_reward_improvement(before, after)
