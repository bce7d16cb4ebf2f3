"""CPU: SQIL's and the device DQN's host side -- the constructor refusals, split_in_half, the host pass of learn()
held to a step-by-step restatement of SB3's learn loop (oracle/sqil_port.py), and the oracle's float64 TD step held
to torch autograd."""
import numpy as np
import pytest
import torch as th
from torch import nn

from imitation_b200 import spaces
from imitation_b200.algorithms import dqn, sqil
from imitation_b200.data import types
from imitation_b200.envs import classic
from oracle import sqil_port


def _transitions(n=40, d_obs=4, seed=0):
    r = np.random.default_rng(seed)
    obs = r.standard_normal((n, d_obs)).astype(np.float32)
    return types.Transitions(obs=obs, acts=r.integers(0, 2, n), infos=np.array([{}] * n),
                             next_obs=r.standard_normal((n, d_obs)).astype(np.float32),
                             dones=np.zeros(n, bool))


def _venv(name="seals/CartPole-v0", n=1):
    return classic.ClassicVecEnv(name, n, device="cpu")


@pytest.mark.parametrize("kw", ["replay_buffer_class", "replay_buffer_kwargs"])
def test_sqil_constructor_raises(kw):
    with pytest.raises(ValueError, match=f"'{kw}' not allowed"):
        sqil.SQIL(venv=_venv(), demonstrations=_transitions(), policy="MlpPolicy", rl_kwargs={kw: None})


def test_sqil_refuses_continuous_rl_algos():
    class SAC:
        pass

    with pytest.raises(NotImplementedError, match="SAC"):
        sqil.SQIL(venv=_venv("Pendulum-v1"), demonstrations=_transitions(d_obs=3), policy="MlpPolicy",
                  rl_algo_class=SAC)


@pytest.mark.parametrize("kwargs, match", [
    (dict(learning_rate=lambda p: 1e-3), "callable learning_rate"),
    (dict(optimize_memory_usage=True), "optimize_memory_usage"),
    (dict(train_freq=(1, "episode")), "episodes"),
    (dict(policy_kwargs=dict(net_arch=[64, 64, 64])), "net_arch"),
    (dict(policy_kwargs=dict(net_arch=[128, 128])), "net_arch"),
    (dict(policy_kwargs=dict(activation_fn=nn.ELU)), "activation_fn"),
])
def test_dqn_refusals_name_the_limit(kwargs, match):
    with pytest.raises(NotImplementedError, match=match):
        dqn.DQN("MlpPolicy", _venv(), replay_buffer_class=sqil.SQILReplayBuffer,
                replay_buffer_kwargs=dict(demonstrations=_transitions()), **kwargs)


def test_dqn_refuses_box_actions():
    with pytest.raises(NotImplementedError, match="Box"):
        dqn.DQN("MlpPolicy", _venv("Pendulum-v1"), replay_buffer_class=sqil.SQILReplayBuffer)


def test_unsupported_demonstrations_raise():
    with pytest.raises(NotImplementedError, match="Unsupported demonstrations type"):
        sqil.SQILReplayBuffer(100, spaces.Box(-1, 1, (4,)), spaces.Discrete(2), demonstrations=42, device="cpu")


def test_split_in_half():
    assert [sqil.split_in_half(x) for x in (0, 1, 2, 7, 32, 220, 221)] == \
        [(0, 0), (0, 1), (1, 1), (3, 4), (16, 16), (110, 110), (110, 111)]


def test_expert_buffer_holds_the_demonstrations_in_sb3_shapes():
    d = _transitions()
    buf = sqil.SQILReplayBuffer(100, spaces.Box(-1, 1, (4,)), spaces.Discrete(2), demonstrations=d, device="cpu")
    eb = buf.expert_buffer
    assert eb.observations.shape == (40, 1, 4) and eb.actions.shape == (40, 1, 1) and eb.dones.shape == (40, 1)
    for i in range(len(d)):
        np.testing.assert_array_equal(eb.observations[i][0], d.obs[i])
        np.testing.assert_array_equal(eb.actions[i][0], d.acts[i])
        np.testing.assert_array_equal(eb.next_observations[i][0], d.next_obs[i])
        np.testing.assert_array_equal(eb.dones[i], d.dones[i])
    t = buf.expert_table.numpy()
    np.testing.assert_array_equal(t[:4].T, d.obs)
    np.testing.assert_array_equal(t[4:6].argmax(0), d.acts)


SCHEDULES = [  # n_envs, learning_starts, train_freq, gradient_steps, total, buffer_size, target_update_interval
    (1, 100, 4, 1, 400, 1_000_000, 10_000),
    (1, 102, 4, 1, 400, 1_000_000, 50),    # learning_starts inside a train_freq window
    (4, 100, 4, 1, 400, 64, 12),           # n_envs 4: ring wrap, target updates every 3 calls
    (4, 98, 3, -1, 480, 40, 1),            # gradient_steps -1, every call a target update
    (1, 0, 2, 3, 90, 17, 7),               # learning_starts 0: the first draw compares with rate 0
]


@pytest.mark.parametrize("E, ls, tf, gs, total, bs, tui", SCHEDULES)
def test_learn_schedule_matches_sb3_loop(E, ls, tf, gs, total, bs, tui):
    _check_learn_schedule(E, ls, tf, gs, total, bs, tui, 33)


@pytest.mark.parametrize("E, ls, tf, gs, total, bs, tui", SCHEDULES[2:4])
def test_learn_schedule_without_learner_rows_matches_sb3_loop(E, ls, tf, gs, total, bs, tui):
    """batch_size 1: no learner rows.  SB3 still calls randint(0, upper, size=0) and randint(0, n_envs, size=(0,)),
    which return empty arrays and consume no draws; the schedule must make the same draws."""
    np.random.seed(2)
    empty = np.random.randint(0, 5, size=0), np.random.randint(0, high=4, size=(0,))
    after = np.random.rand()
    np.random.seed(2)
    assert all(e.shape == (0,) for e in empty) and np.random.rand() == after
    _check_learn_schedule(E, ls, tf, gs, total, bs, tui, 1)


def _check_learn_schedule(E, ls, tf, gs, total, bs, tui, B):
    n_exp = 57
    port = sqil_port.LearnLoopPort(n_envs=E, d_obs=1, n_expert=n_exp, buffer_size=bs, learning_starts=ls,
                                   batch_size=B, train_freq=tf, gradient_steps=gs, target_update_interval=tui,
                                   exploration_fraction=0.3)
    np.random.seed(5)
    port.learn(total)
    port.learn(total // 2)  # a second learn(): _n_calls, the rate and the buffer carry over
    next_draw = np.random.rand()
    rate_fn = dqn.linear_schedule(1.0, 0.05, 0.3)
    np.random.seed(5)
    P = max(bs // E, 1)
    s1 = dqn.learn_schedule(total, E, tf, gs, ls, B, P, 0, False, n_exp, tui, 0, 0.0, rate_fn)
    pos = (int(s1.pos[-1]) + tf) % P
    s2 = dqn.learn_schedule(total // 2, E, tf, gs, ls, B, P, pos, s1.full, n_exp, tui, s1.n_calls,
                            float(s1.rates[-1]), rate_fn)
    assert np.random.rand() == next_draw  # both consumed the same bits
    np.testing.assert_array_equal(np.concatenate([s1.explore, s2.explore]), port.random_steps)
    np.testing.assert_array_equal(np.concatenate([s1.rates, s2.rates]), port.rates)
    every = max(tui // E, 1)
    calls = np.arange(1, s2.n_calls + 1)
    assert np.concatenate([s1.target_updates, s2.target_updates]).sum() == len(port.target_update_calls)
    np.testing.assert_array_equal(calls[calls % every == 0], port.target_update_calls)
    n_td = len(port.samples)
    assert s1.learner_idx.shape[0] + s2.learner_idx.shape[0] == n_td > 0
    assert s1.learner_idx.shape[1] == B // 2 and s1.expert_idx.shape[1] == B - B // 2
    lidx = np.concatenate([s1.learner_idx, s2.learner_idx])
    eidx = np.concatenate([s1.expert_idx, s2.expert_idx])
    for k, (bi, ei, xi) in enumerate(port.samples):
        np.testing.assert_array_equal(lidx[k], bi * E + ei)
        np.testing.assert_array_equal(eidx[k], xi)
    assert [g for g in np.concatenate([s1.grad_steps, s2.grad_steps]) if g] == port.train_calls
    assert s2.full == port.buffer.full and (int(s2.pos[-1]) + tf) % P == port.buffer.pos


def test_oracle_td_step_matches_torch_autograd_float64():
    th.manual_seed(3)
    r = np.random.default_rng(3)
    d_obs, h, A, B = 4, 64, 2, 33
    net = nn.Sequential(nn.Linear(d_obs, h), nn.ReLU(), nn.Linear(h, h), nn.ReLU(), nn.Linear(h, A)).double()
    tgt = nn.Sequential(nn.Linear(d_obs, h), nn.ReLU(), nn.Linear(h, h), nn.ReLU(), nn.Linear(h, A)).double()
    opt = th.optim.Adam(net.parameters(), lr=2e-3)
    p = {k: w.detach().numpy().copy() for k, w in zip(sqil_port.KEYS, net.parameters())}
    pt = {k: w.detach().numpy().copy() for k, w in zip(sqil_port.KEYS, tgt.parameters())}
    m = {k: np.zeros_like(v) for k, v in p.items()}
    v = {k: np.zeros_like(x) for k, x in p.items()}
    for step in range(1, 4):
        obs, nobs = r.standard_normal((B, d_obs)) * 3, r.standard_normal((B, d_obs)) * 3
        acts, dones = r.integers(0, A, B), (r.random(B) < 0.2).astype(np.float64)
        rews = np.r_[np.zeros(B // 2), np.ones(B - B // 2)]
        with th.no_grad():
            nq = tgt(th.as_tensor(nobs)).max(1)[0]
            y = th.as_tensor(rews) + (1 - th.as_tensor(dones)) * 0.99 * nq
        q = th.gather(net(th.as_tensor(obs)), 1, th.as_tensor(acts)[:, None])
        loss = nn.functional.smooth_l1_loss(q, y[:, None])
        opt.zero_grad()
        loss.backward()
        nn.utils.clip_grad_norm_(net.parameters(), 0.5 if step == 2 else 10.0)
        opt.step()
        y_port = sqil_port.td_targets(pt, nobs, dones, rews, 0.99)
        np.testing.assert_allclose(y_port, y.numpy(), rtol=1e-13, atol=1e-13)
        l_port = sqil_port.td_step(p, m, v, step, obs, acts, y_port, 2e-3, 0.5 if step == 2 else 10.0)
        assert abs(l_port - loss.item()) < 1e-12
        for k, w in zip(sqil_port.KEYS, net.parameters()):
            np.testing.assert_allclose(p[k], w.detach().numpy(), rtol=1e-10, atol=1e-12)


def test_dqn_policy_state_dict_and_init_are_sb3s():
    th.manual_seed(7)
    pol = dqn.DQNPolicy(spaces.Box(-1, 1, (4,)), spaces.Discrete(2))
    keys = list(pol.state_dict())
    assert keys == [f"{net}.q_net.{i}.{w}" for net in ("q_net", "q_net_target") for i in (0, 2, 4)
                    for w in ("weight", "bias")]
    th.manual_seed(7)
    ref = nn.Sequential(nn.Linear(4, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 2))
    for a, b in zip(pol.q_net.q_net.parameters(), ref.parameters()):
        assert th.equal(a, b)
    for a, b in zip(pol.q_net_target.parameters(), pol.q_net.parameters()):
        assert th.equal(a, b)
