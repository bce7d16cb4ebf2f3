"""Exploratory rollouts of preference comparisons on the device: `imb_rollout_explore` and
`AgentTrainer(exploration_frac > 0)` (reference algorithms/preference_comparisons.py:194-307 and
policies/exploration_wrapper.py:23-95).

- the kernel with pinned noise against its CPU twin (oracle/exploration_port.py driving oracle/ppo_port.py's rollout
  over the synthetic env and the reward ports): Box and Discrete, tanh and ReLU towers, no reward net, a
  NormalizedRewardNet with a RunningNorm or an EMANorm output layer, a 5-member AddSTDRewardWrapper ensemble, and env
  counts that select each of the 8/32/64/128-row tiles;
- invariants: an all-policy vector gives imb_rollout's / imb_rollout_ensemble's bits, an all-random one gives exactly
  low + u (high - low) or floor(u n) (pinned, or from the Philox stream's twin), equal seeds give equal bits and
  consecutive calls different actions;
- `AgentTrainer.sample`: part sizes, terminal trajectories from their episode's reset observation with the synthetic
  env's closed-form rewards, num_timesteps unchanged, output statistics as step-by-step `predict_processed` leaves them,
  an empty BufferingWrapper and an env at an episode start afterwards, graph replay equal to eager execution across
  train -> sample -> train;
- `PreferenceComparisons` end to end with exploration_frac > 0, single net and ensemble with active selection.
The host side (the policy chain, the split of sample() and the generator's consumption) is pinned to the reference in
tests/test_exploration_reference.py.
"""
import copy

import numpy as np
import pytest
import torch as th
from torch import nn

pytestmark = pytest.mark.gpu

GAMMA, LAMBDA, EMA_DECAY, ALPHA = 0.97, 0.9, 0.9, -0.5


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _dev(x):
    return th.as_tensor(np.ascontiguousarray(x)).cuda().contiguous()


class _Case:
    """One exploration-rollout configuration: the oracle ports and the device inputs built from the same weights."""

    def __init__(self, L, discrete, act, reward, E, T=9, H=4, seed=11, vec_seed=0):
        from imitation_b200 import _desc
        from oracle import nets_port, ppo_port
        from tests.test_ema_norm_reference import ema_output_port
        from tests.test_gpu_kernels import _policy_flat

        self.L, self.discrete, self.reward, self.E, self.T, self.H, self.seed = L, discrete, reward, E, T, H, seed
        self.Do, self.Da = (4, 3) if discrete else (11, 3)
        Do, Da = self.Do, self.Da
        th.manual_seed(seed)
        pol = ppo_port.ActorCriticPort(Do, Da, discrete=discrete, hidden=(32, 32))
        with th.no_grad():
            for p in pol.parameters():
                p.add_(0.3 * th.randn_like(p))
        if act == "relu":
            for tower in (pol.pi, pol.vf):
                tower[1], tower[3] = nn.ReLU(), nn.ReLU()
        self.pol, self.act = pol, (L.ACT_RELU if act == "relu" else L.ACT_TANH)
        self.M = 5 if reward == "ensemble" else 1
        self.nets, self.outs = [], []
        for m in range(self.M if reward != "none" else 0):
            net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=(32, 32))
            net.eval()
            self.nets.append(net)
            batches = np.random.default_rng(m).normal(0.3 * m, 1 + m, (4, 20)).astype(np.float32)
            if reward == "ema":
                out = ema_output_port(EMA_DECAY)
                for b in batches:
                    out.norm.update_stats(th.as_tensor(b))
            else:
                out = nets_port.OutputNormPort()
                out(batches.reshape(-1))
            self.outs.append(out)
        rng = np.random.default_rng(seed + vec_seed + 1)
        vec = (rng.random(T) < 0.5).astype(np.uint8)
        vec[0], vec[1] = 0, 1  # both kinds of step
        self.vec = vec
        # pinned noise: normals (Box) / uniforms (Discrete) on policy steps, uniforms in [0, 1) on random steps
        if discrete:
            self.noise = rng.random((T, E)).astype(np.float32)
        else:
            self.noise = rng.standard_normal((T, E, Da)).astype(np.float32)
            self.noise[vec == 1] = rng.random((int(vec.sum()), E, Da)).astype(np.float32)
        # device inputs
        self.pd = _desc.policy_desc(Do, Da, discrete, 32, False)
        self.PP, self.PN = _policy_flat(pol).cuda(), th.zeros(2, device="cuda")
        self.dd = _desc.disc_desc(Do, Da) if reward != "none" else None
        self.DP = [th.cat([p.detach().reshape(-1) for p in n.mlp.parameters()]).cuda() for n in self.nets]
        self.env = L.EnvDesc(d_obs=Do, d_act=Da, discrete=int(discrete), horizon=H, seed=seed, env_id_offset=5)
        self.EP = _dev(_desc.synth_env_params(Do, Da, seed))
        self.hp = L.PpoHparams(gamma=GAMMA, gae_lambda=LAMBDA, clip_range=0.2, ent_coef=0.0, vf_coef=0.5,
                               max_grad_norm=0.5, lr=3e-4, adam_eps=1e-5, n_epochs=1, batch_size=32,
                               normalize_advantage=1)
        self.rw = L.rollout_row_width(self.pd)
        self.tw = _desc.table_width(Do, Da)
        self.c = Do + (1 if discrete else Da)  # logp column

    def out_vectors(self):
        """Device copies of the output norms' state, as the scan / relabel take them."""
        vs = []
        for o in self.outs:
            n = o.norm
            if self.reward == "ema":
                vs.append((th.tensor([float(n.running_mean), float(n.running_var), float(n.inv_learning_rate)],
                                     device="cuda"),
                           th.tensor([int(n.count), int(n.num_batches)], dtype=th.int32, device="cuda"), 1e-5,
                           EMA_DECAY))
            else:
                vs.append((th.tensor([float(n.running_mean), float(n.running_var)], device="cuda"),
                           th.tensor([int(n.count)], dtype=th.int32, device="cuda"), 1e-5))
        return vs

    def fresh_state(self):
        st = th.zeros(self.L.ST_WORDS, dtype=th.int64, device="cuda")
        obs = th.empty(self.Do, self.E, device="cuda")
        self.L.env_reset(obs, self.E, self.env, st)
        return obs, st

    def launch(self, vec, noise, obs, st, seed=123, step0=0, flags=0, explore=True):
        """One rollout (the exploration entry point, or with explore=False imb_rollout / imb_rollout_ensemble) ->
        (tbl, flat, aux, raw member outputs or None); no relabel."""
        L, E, T = self.L, self.E, self.T
        tbl = th.zeros(E * T, self.rw, device="cuda")
        flat = th.zeros(E * T, self.tw, device="cuda")
        aux = th.zeros(2 * E + 2 * E * T, device="cuda")
        raw = members = None
        if self.reward == "ensemble":
            raw = th.zeros(self.M * T * E, device="cuda")
            members = L.rollout_members(self.DP, [None] * self.M, raw)
        mode = 0 if self.reward == "none" else 2
        dparams = self.DP[0] if mode and members is None else None
        nz = None if noise is None else _dev(noise)
        args = (self.env, self.EP, obs, self.pd, self.PP, self.PN)
        if explore:
            L.rollout_explore(*args, self.dd, dparams, None, members, mode, self.hp, E, T, tbl, flat, aux, nz,
                              _dev(vec), seed, step0, st, flags=flags, act=self.act)
        elif members is None:
            L.rollout(*args, self.dd, dparams, None, mode, self.hp, E, T, tbl, None, 0, flat, aux, nz, st, flags=flags,
                      act=self.act)
        else:
            L.rollout_ensemble(*args, self.dd, members, self.hp, E, T, tbl, None, 0, flat, aux, nz, st, flags=flags,
                               act=self.act)
        return tbl, flat, aux, raw

    def relabel(self, tbl, raw, outs):
        L, E, T = self.L, self.E, self.T
        if self.reward == "ensemble":
            d = L.pref_uncertainty_desc(list(raw.view(self.M, T * E)), outs)
            ws = th.zeros(L.ensemble_relabel_ws_floats(self.M, T), device="cuda")
            L.ensemble_relabel(d, ALPHA, tbl, self.rw, self.c + 2, E, T, ws)
        elif self.reward != "none":
            o = outs[0]
            L.reward_norm_scan(tbl.view(-1)[self.c + 2:], E, T, self.rw, T * self.rw, o[0], o[1], o[2], True,
                               ema_decay=o[3] if len(o) > 3 else None)

    def twin(self, deterministic=False):
        """The CPU twin: (PPOPort buffers, reference-order flattened transitions)."""
        from oracle import data_port, exploration_port, ppo_port, synth_env
        from tests.test_ensemble_relabel_reference import ensemble_relabel_port

        spec = synth_env.SynthEnvSpec(self.Do, self.Da, discrete=self.discrete, horizon=self.H, seed=self.seed)
        buffering = data_port.BufferingPort(synth_env.SynthVecEnv(spec, self.E, env_id_offset=5))
        if self.reward == "none":
            env, last_obs = buffering, buffering.reset()
        else:
            fn = ensemble_relabel_port(list(zip(self.nets, self.outs)), ALPHA if self.reward == "ensemble" else None,
                                       self.Da if self.discrete else None)
            env = data_port.RewardRelabelPort(buffering, fn)
            last_obs = env._old_obs
        xp = exploration_port.ExplorationPolicyPort(self.pol, self.vec, deterministic=deterministic)
        gen = ppo_port.PPOPort(xp, env, n_steps=self.T, gamma=GAMMA, gae_lambda=LAMBDA,
                               noise_fn=lambda step: self.noise[step])
        gen._last_obs, gen._last_starts = last_obs, np.ones(self.E, dtype=bool)
        buf = gen.collect_rollouts()
        trajs, _ = buffering.pop_trajectories()
        return buf, data_port.flatten_port(trajs)


def _flat_order(x, T, H):
    """[E][T] per-step values -> the reference flat order (segment-major, then env, then step) from episode step 0."""
    return np.concatenate([x[:, a:min(a + H, T)].reshape(-1) for a in range(0, T, H)])


def _check_against_twin(S, tbl, flat, aux, outs, buf, want):
    E, T, H, Do, Da, c = S.E, S.T, S.H, S.Do, S.Da, S.c
    got = tbl.cpu().numpy().reshape(E, T, S.rw)
    col = lambda a: np.swapaxes(a, 0, 1)  # noqa: E731  oracle [T, E, ...] -> [E, T, ...]
    rnd = S.vec == 1
    np.testing.assert_allclose(got[:, :, :Do], col(buf["obs"]), rtol=1e-3, atol=1e-4, err_msg="obs")
    if S.discrete:
        np.testing.assert_array_equal(got[:, :, Do], col(buf["actions"]))
    else:
        np.testing.assert_allclose(got[:, :, Do:Do + Da], col(buf["actions"]), rtol=1e-3, atol=1e-4, err_msg="act")
        # random steps: the same float32 arithmetic on the same uniforms
        np.testing.assert_array_equal(got[:, rnd, Do:Do + Da], col(buf["actions"])[:, rnd])
    np.testing.assert_allclose(got[:, :, c], col(buf["log_probs"]), rtol=1e-3, atol=1e-4, err_msg="logp")
    np.testing.assert_allclose(got[:, :, c + 1], col(buf["values"]), rtol=1e-3, atol=1e-4, err_msg="value")
    assert (got[:, rnd, c] == 0).all() and (got[:, rnd, c + 1] == 0).all()
    a = aux.cpu().numpy()
    boot = a[2 * E:2 * E + E * T].reshape(E, T)
    np.testing.assert_allclose(got[:, :, c + 2] + boot, col(buf["rewards"]), rtol=1e-3, atol=2e-4, err_msg="reward")
    env_rews = a[2 * E + E * T:].reshape(E, T)
    np.testing.assert_allclose(_flat_order(env_rews, T, H), want["rews"], rtol=1e-3, atol=1e-4, err_msg="env reward")
    gf = flat.cpu().numpy()
    np.testing.assert_array_equal(gf[:, -1] > 0.5, want["dones"])
    np.testing.assert_allclose(gf[:, :Do], want["obs"], rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(gf[:, Do + Da:2 * Do + Da], want["next_obs"], rtol=1e-3, atol=1e-4)
    if S.discrete:
        np.testing.assert_array_equal(gf[:, Do:Do + Da].argmax(1), want["acts"])
    else:
        np.testing.assert_allclose(gf[:, Do:Do + Da], want["acts"], rtol=1e-3, atol=1e-4)
    for o, g in zip(S.outs, outs):  # output statistics advanced once per step, as the ports' predict_processed
        n = o.norm
        want_state = [float(n.running_mean), float(n.running_var)]
        want_count = [int(n.count)]
        if len(g) > 3:
            want_state.append(float(n.inv_learning_rate))
            want_count.append(int(n.num_batches))
        np.testing.assert_allclose(g[0].cpu().numpy(), want_state, rtol=1e-5, atol=1e-6)
        assert g[1].cpu().tolist() == want_count


# ---------------------------------------------------------------------------------------------
# the kernel against its CPU twin
# ---------------------------------------------------------------------------------------------
def _envs_for_tile(rows):
    n_sms = th.cuda.get_device_properties(0).multi_processor_count
    return {8: 37, 32: 24 * n_sms, 64: 100 * n_sms, 128: 129 * n_sms}[rows]


CASES = ([(d, a, r, 8) for d in (False, True) for a in ("tanh", "relu") for r in ("none", "running", "ema", "ensemble")]
         + [(False, "tanh", "ensemble", t) for t in (32, 64, 128)] + [(True, "relu", "running", t) for t in (32, 64, 128)])


@pytest.mark.parametrize("discrete,act,reward,tile", CASES)
def test_explore_rollout_matches_twin(L, discrete, act, reward, tile):
    S = _Case(L, discrete, act, reward, _envs_for_tile(tile))
    assert L.rollout_plan(S.pd, S.dd, S.M, S.E) == tile
    obs, st = S.fresh_state()
    outs = S.out_vectors()
    tbl, flat, aux, raw = S.launch(S.vec, S.noise, obs, st)
    S.relabel(tbl, raw, outs)
    th.cuda.synchronize()
    buf, want = S.twin()
    _check_against_twin(S, tbl, flat, aux, outs, buf, want)


@pytest.mark.parametrize("discrete", [False, True])
def test_deterministic_flag_on_policy_steps(L, discrete):
    """IMB_RF_DETERMINISTIC (ExplorationWrapper(deterministic_policy=True)): policy steps act with the mode; random
    steps still read their uniforms."""
    S = _Case(L, discrete, "tanh", "running", 37)
    obs, st = S.fresh_state()
    outs = S.out_vectors()
    tbl, flat, aux, raw = S.launch(S.vec, S.noise, obs, st, flags=L.IMB_RF_DETERMINISTIC)
    S.relabel(tbl, raw, outs)
    th.cuda.synchronize()
    buf, want = S.twin(deterministic=True)
    _check_against_twin(S, tbl, flat, aux, outs, buf, want)


# ---------------------------------------------------------------------------------------------
# invariants
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("discrete,act,reward", [(False, "tanh", "running"), (True, "relu", "ensemble"),
                                                 (False, "relu", "none"), (True, "tanh", "ema")])
def test_all_policy_vector_gives_the_plain_rollout_bits(L, discrete, act, reward):
    S = _Case(L, discrete, act, reward, 300)
    zeros = np.zeros(S.T, np.uint8)
    runs = []
    for explore in (True, False):
        for noise in (None, S.noise if discrete else np.random.default_rng(3).standard_normal(S.noise.shape)
                      .astype(np.float32)):
            obs, st = S.fresh_state()
            tbl, flat, aux, raw = S.launch(zeros, noise, obs, st, explore=explore)
            runs.append((tbl, flat, aux, raw, obs, st))
    th.cuda.synchronize()
    for a, b in ((runs[0], runs[2]), (runs[1], runs[3])):
        for x, y in zip(a, b):
            assert (x is None and y is None) or th.equal(x, y)


@pytest.mark.parametrize("discrete", [False, True])
def test_all_random_vector_gives_the_uniform_actions(L, discrete):
    from oracle import exploration_port

    S = _Case(L, discrete, "tanh", "none", 300)
    E, T, Do, Da = S.E, S.T, S.Do, S.Da
    ones = np.ones(T, np.uint8)
    u_pinned = np.random.default_rng(4).random(S.noise.shape).astype(np.float32)
    seed, step0 = 987654321, 17
    u_philox = exploration_port.random_uniforms(seed, np.arange(E) + 5, step0, T, Da, discrete)
    for noise, u in ((u_pinned, u_pinned), (None, u_philox)):
        obs, st = S.fresh_state()
        tbl, flat, aux, _ = S.launch(ones, noise, obs, st, seed=seed, step0=step0)
        th.cuda.synchronize()
        got = tbl.cpu().numpy().reshape(E, T, S.rw)
        ctrl = flat.cpu().numpy()[:, Do:Do + Da]
        if discrete:
            want = np.minimum(np.floor(u * np.float32(Da)).astype(np.int64), Da - 1)  # [T][E]
            np.testing.assert_array_equal(got[:, :, Do], want.T)
            np.testing.assert_array_equal(ctrl, np.eye(Da, dtype=np.float32)[_flat_order(want.T, T, S.H)])
        else:
            want = np.float32(-1.0) + u * (np.float32(1.0) - np.float32(-1.0))  # [T][E][Da]
            np.testing.assert_array_equal(got[:, :, Do:Do + Da], np.swapaxes(want, 0, 1))
            np.testing.assert_array_equal(ctrl, np.concatenate([np.swapaxes(want, 0, 1)[:, a:min(a + S.H, T)]
                                                                .reshape(-1, Da) for a in range(0, T, S.H)]))
        assert (got[:, :, S.c] == 0).all() and (got[:, :, S.c + 1] == 0).all()


def test_equal_seeds_equal_bits_and_consecutive_calls_differ(L):
    for discrete in (False, True):
        S = _Case(L, discrete, "tanh", "ensemble", 64)
        Do = S.Do
        runs = []
        for _ in range(2):
            obs, st = S.fresh_state()
            runs.append(S.launch(S.vec, None, obs, st, seed=5, step0=0))
            L.rollout_advance(st, S.E, S.T, S.H, 0)
            runs[-1] += (obs.clone(), st.clone())
            runs[-1] += S.launch(S.vec, None, obs, st, seed=5, step0=S.T)  # the next call continues the chain
        th.cuda.synchronize()
        for x, y in zip(*runs):
            assert (x is None and y is None) or th.equal(x, y)
        first, second = runs[0][0].cpu().numpy(), runs[0][6].cpu().numpy()
        rnd = S.vec == 1
        a1 = first.reshape(S.E, S.T, -1)[:, rnd, Do:S.c]
        a2 = second.reshape(S.E, S.T, -1)[:, rnd, Do:S.c]
        assert (a1 != a2).mean() > 0.5  # different counters, different draws


# ---------------------------------------------------------------------------------------------
# AgentTrainer.sample
# ---------------------------------------------------------------------------------------------
def _agent(use_graph, E=8, T=16, H=10, frac=0.5, reward_kind="running", seed=0):
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    venv = synth.DeviceVecEnv(11, 3, E, horizon=H, seed=3)
    th.manual_seed(seed)
    if reward_kind == "ensemble":
        members = [reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space,
                                                                              venv.action_space), networks.RunningNorm)
                   for _ in range(5)]
        reward = reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(venv.observation_space, venv.action_space,
                                                                            members).cuda(), default_alpha=ALPHA)
    else:
        reward = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space, venv.action_space),
                                                 networks.RunningNorm).cuda()
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=32, n_epochs=1, seed=0)
    algo.use_cuda_graph = use_graph
    agent = pc.AgentTrainer(algo, reward, venv, np.random.default_rng(seed), exploration_frac=frac)
    return agent, reward, algo, venv


def test_sample_parts_trajectories_and_side_effects(L):
    from imitation_b200 import _desc
    from imitation_b200.algorithms import preference_comparisons as pc
    from oracle import synth_env

    E, T, H = 8, 16, 10
    agent, reward, algo, venv = _agent(True, E, T, H)
    agent.train(steps=4 * E * T)
    steps = 150
    agent_steps, exploration_steps = pc.split_steps(steps, 0.5)
    k = -(-exploration_steps // (E * H))
    n_ts = algo.num_timesteps
    host = copy.deepcopy(reward)  # advanced step by step below, as the reference's predict_processed advances it
    trajs = agent.sample(steps)
    th.cuda.synchronize()
    assert algo.num_timesteps == n_ts
    agent_part = pc._get_trajectories(trajs, agent_steps)  # the agent part is the result's prefix
    n_agent = len(agent_part)
    explo = trajs[n_agent:]
    assert sum(len(t) for t in agent_part) >= agent_steps > sum(len(t) for t in agent_part[:-1])
    assert len(explo) == -(-exploration_steps // H) and all(len(t) == H for t in explo)
    # terminal, from the reset observation of their episode, with the env's closed-form rewards
    spec = synth_env.SynthEnvSpec(11, 3, horizon=H, seed=3)
    episode_after = int(venv.state[L.ST_EPISODE])
    for i, t in enumerate(explo):
        j, e = divmod(i, E)
        assert t.terminal
        np.testing.assert_allclose(t.obs[0], spec.reset_obs([e], [episode_after - k + j])[0], rtol=1e-6, atol=1e-7)
        nobs, rew = spec.dynamics(t.obs[:-1], t.acts)
        np.testing.assert_allclose(t.obs[1:], nobs, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(t.rews, rew, rtol=1e-4, atol=1e-5)
    # output statistics: E * k * H more, as k * H calls of predict_processed over the E transitions of each step leave
    flat = algo._x_flat.cpu().numpy().reshape(k, E, H, -1)
    for s in range(k * H):
        j, t = divmod(s, H)
        rows = flat[j, :, t]
        host.predict_processed(rows[:, :11], rows[:, 11:14], rows[:, 14:25], rows[:, 25] > 0.5)
    hn, dn = host.normalize_output_layer, reward.normalize_output_layer
    assert int(dn.count) == int(hn.count)
    np.testing.assert_allclose([float(dn.running_mean), float(dn.running_var)],
                               [float(hn.running_mean), float(hn.running_var)], rtol=1e-5, atol=1e-6)
    # the wrapper is empty and the env at an episode start
    assert agent.buffering_wrapper.n_transitions == 0 and agent.buffering_wrapper._hist == []
    assert venv.host_ep_step == 0 and int(venv.state[L.ST_EP_STEP]) == 0
    assert _desc.table_width(11, 3) == flat.shape[-1]
    # training resumes from that episode start
    agent.train(steps=E * T)
    th.cuda.synchronize()
    tbl = algo._tbl.cpu().numpy().reshape(E, T, -1)
    np.testing.assert_allclose(tbl[:, 0, :11], spec.reset_obs(np.arange(E), np.full(E, episode_after)), rtol=1e-6,
                               atol=1e-7)


@pytest.mark.parametrize("reward_kind", ["running", "ensemble"])
def test_graph_replay_equals_eager_across_train_sample_train(L, reward_kind):
    E, T, H = 8, 16, 10
    runs = {}
    for use_graph in (False, True):
        agent, reward, algo, venv = _agent(use_graph, E, T, H, reward_kind=reward_kind)
        agent.train(steps=3 * E * T)
        trajs = agent.sample(120)
        agent.train(steps=2 * E * T)
        agent.buffering_wrapper.discard()
        th.cuda.synchronize()
        runs[use_graph] = dict(tbl=algo._tbl.clone(), pol=algo.policy.flat_vectors()[0].clone(), obs=venv.obs.clone(),
                               state=venv.state.clone(), x=algo._x_tbl.clone(),
                               stats=[t.clone() for t in reward.state_dict().values()],
                               trajs=[np.concatenate([t.obs.ravel(), t.acts.ravel(), t.rews]) for t in trajs])
        if use_graph:
            assert algo._graph is not None
    a, b = runs[False], runs[True]
    for key in ("tbl", "pol", "obs", "state", "x"):
        assert th.equal(a[key], b[key]), key
    assert all(th.equal(x, y) for x, y in zip(a["stats"], b["stats"]))
    assert len(a["trajs"]) == len(b["trajs"]) and all(np.array_equal(x, y) for x, y in zip(a["trajs"], b["trajs"]))


# ---------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------
def test_quickstart_shaped_preference_comparisons_with_exploration(L):
    """The reference quickstart's shape (docs/algorithms/preference_comparisons.rst): FeedForward32Policy with
    NormalizeFeaturesExtractor, BasicRewardNet with an input RunningNorm, exploration_frac=0.05."""
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.policies import base as policies
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    E, T, H = 8, 32, 20
    venv = synth.DeviceVecEnv(11, 3, E, horizon=H, seed=5)
    rng = np.random.default_rng(0)
    th.manual_seed(0)
    reward_net = reward_nets.BasicRewardNet(venv.observation_space, venv.action_space,
                                            normalize_input_layer=networks.RunningNorm).cuda()
    fragmenter = pc.RandomFragmenter(warning_threshold=0, rng=rng)
    gatherer = pc.SyntheticGatherer(rng=rng)
    model = pc.PreferenceModel(reward_net)
    trainer = pc.BasicRewardTrainer(preference_model=model, loss=pc.CrossEntropyRewardLoss(), epochs=3, rng=rng)
    algo = ppo.DevicePPO(policies.FeedForward32Policy, venv, n_steps=T, batch_size=64, n_epochs=2, seed=0,
                         policy_kwargs=dict(features_extractor_class=policies.NormalizeFeaturesExtractor,
                                            features_extractor_kwargs=dict(normalize_class=networks.RunningNorm)))
    agent = pc.AgentTrainer(algo, reward_net, venv, rng, exploration_frac=0.05)
    pcs = pc.PreferenceComparisons(agent, reward_net, num_iterations=3, fragmenter=fragmenter,
                                   preference_gatherer=gatherer, reward_trainer=trainer, fragment_length=10,
                                   transition_oversampling=1, initial_comparison_frac=0.1,
                                   initial_epoch_multiplier=1.0, query_schedule="hyperbolic", rng=rng)
    res = pcs.train(total_timesteps=8 * E * T, total_comparisons=60)
    assert np.isfinite(res["reward_loss"]) and 0.0 <= res["reward_accuracy"] <= 1.0
    assert agent.exploration_wrapper.steps_taken > 0


def test_ensemble_with_active_selection_and_exploration(L):
    from imitation_b200.algorithms import preference_comparisons as pc

    E, T, H = 8, 16, 10
    agent, reward, algo, venv = _agent(True, E, T, H, frac=0.2, reward_kind="ensemble")
    rng = np.random.default_rng(1)
    pm = pc.PreferenceModel(reward)
    frag = pc.ActiveSelectionFragmenter(pm, pc.RandomFragmenter(warning_threshold=0, rng=rng), 2.0)
    pcs = pc.PreferenceComparisons(agent, reward, num_iterations=2, fragmenter=frag, fragment_length=5,
                                   transition_oversampling=1, initial_comparison_frac=0.5,
                                   initial_epoch_multiplier=1.0, rng=rng)
    res = pcs.train(total_timesteps=4 * E * T, total_comparisons=16)
    assert np.isfinite(res["reward_loss"]) and 0.0 <= res["reward_accuracy"] <= 1.0
    assert agent.exploration_wrapper.steps_taken > 0
