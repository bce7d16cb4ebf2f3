"""CPU: the device SAC's host side -- its refusals (the shape limits through imb_sac_plan), SACPolicy's SB3 state_dict and
initial weights, the host pass of learn() held to a step-by-step restatement of SB3's learn loop
(oracle/sac_port.py), the oracle's float64 SAC step held to torch autograd on SB3's own expressions, and
SQILReplayBuffer with Box actions."""
import numpy as np
import pytest
import torch as th
from torch import nn
from torch.nn import functional as F

from imitation_b200 import _lib, spaces
from imitation_b200.algorithms import dqn, sac, sqil
from imitation_b200.data import types
from imitation_b200.envs import classic, synth
from oracle import sac_port


def _transitions(n=40, d_obs=3, d_act=1, seed=0):
    r = np.random.default_rng(seed)
    return types.Transitions(obs=r.standard_normal((n, d_obs)).astype(np.float32),
                             acts=r.uniform(-2, 2, (n, d_act)).astype(np.float32), infos=np.array([{}] * n),
                             next_obs=r.standard_normal((n, d_obs)).astype(np.float32), dones=np.zeros(n, bool))


def _pendulum(n=1):
    return classic.ClassicVecEnv("Pendulum-v1", n, device="cpu")


def _sac(env=None, **kw):
    return sac.SAC("MlpPolicy", env if env is not None else _pendulum(), replay_buffer_class=sqil.SQILReplayBuffer,
                   replay_buffer_kwargs=dict(demonstrations=_transitions()), **kw)


@pytest.mark.parametrize("kwargs, match", [
    (dict(learning_rate=lambda p: 1e-3), "callable learning_rate"),
    (dict(use_sde=True), "use_sde"),
    (dict(action_noise=object()), "action_noise"),
    (dict(optimize_memory_usage=True), "optimize_memory_usage"),
    (dict(train_freq=(1, "episode")), "episodes"),
    (dict(policy_kwargs=dict(activation_fn=nn.Tanh)), "activation_fn"),
    (dict(policy_kwargs=dict(n_critics=3)), "n_critics"),
    (dict(policy_kwargs=dict(net_arch=[64, 64, 64])), "net_arch"),
    (dict(policy_kwargs=dict(net_arch=[64, 32])), "net_arch"),
    (dict(policy_kwargs=dict(net_arch=[512, 512])), "net_arch"),
    (dict(policy_kwargs=dict(net_arch=dict(pi=[64, 64], qf=[32, 32]))), "net_arch"),
    (dict(batch_size=300), "batch_size 300"),
])
def test_sac_refusals_name_the_limit(kwargs, match):
    with pytest.raises(NotImplementedError, match=match):
        _sac(**kwargs)


def test_sac_refuses_discrete_actions_and_other_buffers():
    with pytest.raises(NotImplementedError, match="Discrete"):
        sac.SAC("MlpPolicy", classic.ClassicVecEnv("seals/CartPole-v0", 1, device="cpu"),
                replay_buffer_class=sqil.SQILReplayBuffer)
    with pytest.raises(NotImplementedError, match="replay_buffer_class"):
        sac.SAC("MlpPolicy", _pendulum(), replay_buffer_class=None)


@pytest.mark.parametrize("d_obs, d_act, match", [(65, 2, "d_obs 65"), (17, 9, "d_act 9")])
def test_sac_refuses_shapes_beyond_the_kernels(d_obs, d_act, match):
    env = synth.DeviceVecEnv(d_obs, d_act, 1, device="cpu")
    with pytest.raises(NotImplementedError, match=match):
        sac.SAC("MlpPolicy", env, replay_buffer_class=sqil.SQILReplayBuffer)


def test_sac_plan_envelope():
    _lib.sac_plan(64, 8, 256, 256)
    _lib.sac_plan(1, 1, 1, 1)
    for args, match in (((65, 1, 8, 8), "d_obs"), ((3, 9, 8, 8), "d_act"), ((3, 1, 257, 8), "width 257"),
                        ((3, 1, 8, 257), "batch_size 257"), ((3, 1, 8, 0), "batch_size 0")):
        with pytest.raises(_lib.ImbError, match=match):
            _lib.sac_plan(*args)


@pytest.mark.parametrize("cls", ["TD3", "DDPG"])
def test_sqil_refuses_td3_and_ddpg(cls):
    algo = type(cls, (), {})
    with pytest.raises(NotImplementedError, match=cls):
        sqil.SQIL(venv=_pendulum(), demonstrations=_transitions(), policy="MlpPolicy", rl_algo_class=algo)


def test_sac_policy_state_dict_and_init_are_sb3s():
    th.manual_seed(3)
    pol = sac.SACPolicy(spaces.Box(-np.inf, np.inf, (3,)), spaces.Box(-2, 2, (1,)), net_arch=[32, 32])
    sd = pol.state_dict()
    want = [f"actor.latent_pi.{i}.{w}" for i in (0, 2) for w in ("weight", "bias")]
    want += [f"actor.{m}.{w}" for m in ("mu", "log_std") for w in ("weight", "bias")]
    want += [f"{c}.qf{q}.{i}.{w}" for c in ("critic", "critic_target") for q in (0, 1) for i in (0, 2, 4)
             for w in ("weight", "bias")]
    assert list(sd) == want
    assert sd["actor.latent_pi.0.weight"].shape == (32, 3) and sd["actor.mu.weight"].shape == (1, 32)
    assert sd["critic.qf0.0.weight"].shape == (32, 4) and sd["critic.qf1.4.weight"].shape == (1, 32)
    # SB3's build order: the actor's latent_pi, mu, log_std, then qf0, qf1 of the critic, then the target's (copied)
    th.manual_seed(3)
    ref = [nn.Linear(3, 32), nn.Linear(32, 32), nn.Linear(32, 1), nn.Linear(32, 1)]
    ref += [nn.Linear(4, 32), nn.Linear(32, 32), nn.Linear(32, 1), nn.Linear(4, 32), nn.Linear(32, 32),
            nn.Linear(32, 1)]
    mine = [pol.actor.latent_pi[0], pol.actor.latent_pi[2], pol.actor.mu, pol.actor.log_std]
    mine += [q[i] for q in pol.critic.q_networks for i in (0, 2, 4)]
    for a, b in zip(mine, ref):
        assert th.equal(a.weight, b.weight) and th.equal(a.bias, b.bias)
    for a, b in zip(pol.critic_target.parameters(), pol.critic.parameters()):
        assert th.equal(a, b)
    assert sac._net_width(None) == 256 and sac._net_width(dict(pi=[64, 64], qf=[64, 64])) == 64


def test_scale_round_trip_is_sb3s_float32():
    x = np.array([-1.0, -0.3, 0.0, 1e-8, 0.5, 1.0], np.float32)
    u = sac.unscale_action(x, -2.0, 2.0)
    np.testing.assert_array_equal(u, (np.float32(-2) + np.float32(0.5) * (x + np.float32(1)) * np.float32(4)))
    back = sac.scale_action(u, -2.0, 2.0)
    assert back.dtype == np.float32 and back[3] != x[3]  # not the identity near 0


SCHEDULES = [  # n_envs, learning_starts, train_freq, gradient_steps, total, buffer_size
    (1, 100, 1, 1, 400, 1_000_000),
    (1, 102, 4, 2, 400, 1_000_000),  # learning_starts inside a train_freq window
    (4, 100, 3, -1, 480, 64),        # gradient_steps -1, the ring wraps
    (4, 0, 1, 1, 200, 40),
]


@pytest.mark.parametrize("E, ls, tf, gs, total, bs", SCHEDULES)
def test_sac_learn_schedule_matches_sb3_loop(E, ls, tf, gs, total, bs):
    n_exp, B = 57, 33
    port = sac_port.SACLearnLoopPort(n_envs=E, n_expert=n_exp, buffer_size=bs, learning_starts=ls, batch_size=B,
                                     train_freq=tf, gradient_steps=gs)
    np.random.seed(5)
    port.learn(total)
    port.learn(total // 2, reset_num_timesteps=False)
    next_draw = np.random.rand()
    np.random.seed(5)
    P = max(bs // E, 1)
    s1 = dqn.learn_schedule(total, E, tf, gs, ls, B, P, 0, False, n_exp, 1, 0, 0.0, lambda p: 0.0,
                            exploration_draws=False)
    pos = (int(s1.pos[-1]) + tf) % P
    s2 = dqn.learn_schedule(total // 2 + s1.num_timesteps, E, tf, gs, ls, B, P, pos, s1.full, n_exp, 1, 0, 0.0,
                            lambda p: 0.0, s1.num_timesteps, exploration_draws=False)
    assert np.random.rand() == next_draw  # both consumed the same bits
    np.testing.assert_array_equal(np.concatenate([s1.explore, s2.explore]), port.random_steps)
    lidx = np.concatenate([s1.learner_idx, s2.learner_idx])
    eidx = np.concatenate([s1.expert_idx, s2.expert_idx])
    assert len(lidx) == len(port.samples) > 0
    for k, (bi, ei, xi) in enumerate(port.samples):
        np.testing.assert_array_equal(lidx[k], bi * E + ei)
        np.testing.assert_array_equal(eidx[k], xi)
    assert [g for g in np.concatenate([s1.grad_steps, s2.grad_steps]) if g] == port.train_calls
    assert s2.full == port.buffer.full and (int(s2.pos[-1]) + tf) % P == port.buffer.pos


def test_learn_schedule_for_dqn_is_unchanged_by_the_flag():
    np.random.seed(1)
    a = dqn.learn_schedule(300, 2, 4, 1, 50, 32, 1000, 0, False, 40, 10, 0, 0.0, dqn.linear_schedule(1, 0.05, 0.1))
    np.random.seed(1)
    b = dqn.learn_schedule(300, 2, 4, 1, 50, 32, 1000, 0, False, 40, 10, 0, 0.0, dqn.linear_schedule(1, 0.05, 0.1),
                           exploration_draws=True)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)


# ---- the oracle's float64 step against torch autograd on SB3's expressions ---------------------------------------

def _torch_sac_step(actor, critic, target, opt_a, opt_c, log_ent_coef, opt_e, ent_fixed, batch, eps, eps_n, gamma, tau,
                    target_entropy, polyak):
    """SAC.train's body for one gradient step (SB3 2.2), float64, with the actor's noise given."""
    obs, acts, nobs, dones, rews = batch

    def action_log_prob(o, e):
        latent = actor["latent"](o)
        mean, log_std = actor["mu"](latent), th.clamp(actor["ls"](latent), -20, 2)
        std = log_std.exp()
        g = mean + e * std
        a = th.tanh(g)
        lp = th.distributions.Normal(mean, std).log_prob(g).sum(1) - th.sum(th.log(1 - a ** 2 + 1e-6), dim=1)
        return a, lp

    a_pi, logp = action_log_prob(obs, eps)
    logp = logp.reshape(-1, 1)
    out = {}
    if log_ent_coef is not None:
        ent_coef = th.exp(log_ent_coef.detach())
        ent_loss = -(log_ent_coef * (logp + target_entropy).detach()).mean()
        out["ent_coef_loss"] = ent_loss.item()
        opt_e.zero_grad()
        ent_loss.backward()
        opt_e.step()
    else:
        ent_coef = th.tensor(ent_fixed, dtype=th.float64)
    out["ent_coef"] = float(ent_coef)
    with th.no_grad():
        a_n, lp_n = action_log_prob(nobs, eps_n)
        x = th.cat([nobs, a_n], 1)
        nq = th.min(th.cat([q(x) for q in target], 1), dim=1, keepdim=True)[0] - ent_coef * lp_n.reshape(-1, 1)
        y = rews + (1 - dones) * gamma * nq
    x = th.cat([obs, acts], 1)
    closs = 0.5 * sum(F.mse_loss(q(x), y) for q in critic)
    out["critic_loss"] = closs.item()
    opt_c.zero_grad()
    closs.backward()
    opt_c.step()
    x = th.cat([obs, a_pi], 1)
    minq = th.min(th.cat([q(x) for q in critic], 1), dim=1, keepdim=True)[0]
    aloss = (ent_coef * logp - minq).mean()
    out["actor_loss"] = aloss.item()
    opt_a.zero_grad()
    aloss.backward()
    opt_a.step()
    if polyak:
        with th.no_grad():
            for tq, q in zip(target, critic):
                for tp, p in zip(tq.parameters(), q.parameters()):
                    tp.mul_(1 - tau)
                    tp.add_(p, alpha=tau)
    return out


@pytest.mark.parametrize("ent, interval, g", [("auto", 1, 2), (0.2, 1, 2), ("auto", 2, 3)])
def test_oracle_sac_step_matches_torch_autograd_float64(ent, interval, g):
    Do, Da, h, B = 3, 2, 16, 12
    th.manual_seed(0)
    r = np.random.default_rng(0)
    lin = lambda i, o: nn.Linear(i, o).double()
    latent = nn.Sequential(lin(Do, h), nn.ReLU(), lin(h, h), nn.ReLU())
    mu, ls = lin(h, Da), lin(h, Da)
    with th.no_grad():  # some rows with log_std clamped at either end
        ls.bias[0] = 3.0
        ls.bias[1] = -25.0 if Da > 1 else ls.bias[1]
        ls.weight[1].mul_(50.0)
    actor = {"latent": latent, "mu": mu, "ls": ls}
    mkq = lambda: nn.Sequential(lin(Do + Da, h), nn.ReLU(), lin(h, h), nn.ReLU(), lin(h, 1))
    critic = [mkq(), mkq()]
    target = [mkq(), mkq()]
    for tq, q in zip(target, critic):
        tq.load_state_dict(q.state_dict())
    lr, gamma, tau, te = 3e-3, 0.99, 0.05, -float(Da)
    opt_a = th.optim.Adam(list(latent.parameters()) + list(mu.parameters()) + list(ls.parameters()), lr=lr)
    opt_c = th.optim.Adam([p for q in critic for p in q.parameters()], lr=lr)
    lec = th.zeros(1, dtype=th.float64, requires_grad=True) if ent == "auto" else None
    opt_e = th.optim.Adam([lec], lr=lr) if lec is not None else None
    npy = lambda m: m.weight.detach().numpy().copy()
    npb = lambda m: m.bias.detach().numpy().copy()
    qd = lambda q: {"w1": npy(q[0]), "b1": npb(q[0]), "w2": npy(q[2]), "b2": npb(q[2]), "w3": npy(q[4]),
                    "b3": npb(q[4])}
    st = sac_port.SACState({"w1": npy(latent[0]), "b1": npb(latent[0]), "w2": npy(latent[2]), "b2": npb(latent[2]),
                            "wmu": npy(mu), "bmu": npb(mu), "wls": npy(ls), "bls": npb(ls)},
                           [qd(q) for q in critic], [qd(q) for q in target], 0.0 if ent == "auto" else None,
                           0.0 if ent == "auto" else ent)
    for s in range(g):
        obs, nobs = r.standard_normal((B, Do)), r.standard_normal((B, Do))
        acts = r.uniform(-2, 2, (B, Da))
        dones = (r.random(B) < 0.3).astype(np.float64)
        rews = np.r_[np.zeros(B // 2), np.ones(B - B // 2)]
        eps, eps_n = r.standard_normal((B, Da)), r.standard_normal((B, Da))
        T = lambda x: th.as_tensor(x, dtype=th.float64)
        got = sac_port.sac_step(st, obs, acts, nobs, dones, rews, eps, eps_n, gamma=gamma, tau=tau, lr=lr,
                                target_entropy=te, polyak=s % interval == 0)
        want = _torch_sac_step(actor, critic, target, opt_a, opt_c, lec, opt_e, ent if ent != "auto" else 0.0,
                               (T(obs), T(acts), T(nobs), T(dones).reshape(-1, 1), T(rews).reshape(-1, 1)), T(eps),
                               T(eps_n), gamma, tau, te, s % interval == 0)
        for k, v in want.items():
            assert abs(got[k] - v) <= 1e-10 * max(1.0, abs(v)), k
    close = lambda a, b: np.testing.assert_allclose(a, b.detach().numpy(), rtol=1e-8, atol=1e-9)
    close(st.actor["w1"], latent[0].weight)
    close(st.actor["w2"], latent[2].weight)
    close(st.actor["wmu"], mu.weight)
    close(st.actor["wls"], ls.weight)
    close(st.actor["bls"], ls.bias)
    for i in range(2):
        for j, k in ((0, "w1"), (2, "w2"), (4, "w3")):
            close(st.critic[i][k], critic[i][j].weight)
            close(st.target[i][k], target[i][j].weight)
    if lec is not None:
        assert abs(st.log_ent_coef - lec.item()) <= 1e-12


def test_sqil_buffer_with_box_actions_keeps_sb3_shapes_and_the_unscaled_expert_actions():
    d = _transitions(d_act=2)
    buf = sqil.SQILReplayBuffer(100, spaces.Box(-np.inf, np.inf, (3,)), spaces.Box(-2, 2, (2,)), demonstrations=d,
                                device="cpu", n_envs=2)
    assert buf.tw == 2 * 3 + 2 + 1
    eb = buf.expert_buffer
    assert eb.observations.shape == (40, 1, 3) and eb.actions.shape == (40, 1, 2) and eb.actions.dtype == np.float32
    np.testing.assert_array_equal(eb.actions[:, 0], d.acts)  # as recorded, env scale (+-2), not scaled to [-1, 1]
    t = buf.expert_table.numpy()
    np.testing.assert_array_equal(t[3:5].T, d.acts)
    np.testing.assert_array_equal(t[5:8].T, d.next_obs)
    buf.add(np.ones((2, 3)), np.zeros((2, 3)), np.array([[0.5, -0.25], [1.0, -1.0]]), np.zeros(2), np.zeros(2),
            [{}, {}])
    assert buf.actions.shape == (50, 2, 2)
    np.testing.assert_array_equal(buf.actions[0], [[0.5, -0.25], [1.0, -1.0]])
    np.random.seed(0)
    smp = buf.sample(8)
    assert smp.actions.shape == (8, 2) and smp.rewards[:4].sum() == 0 and smp.rewards[4:].sum() == 4
