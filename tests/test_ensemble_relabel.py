"""Agent training on an ensemble reward: `imb_rollout_ensemble` + `imb_ensemble_relabel` (the relabel of
`RewardVecEnvWrapper` with reward_fn = `AddSTDRewardWrapper(RewardEnsemble(members), alpha).predict_processed`,
rewards/reward_nets.py:926-989 and :1045-1080 of the reference).

- the relabel kernel against a float64 restatement of the members' per-step output normalisation and mean + alpha * std;
- the member rollout with pinned sampling noise against the SB3 restatement (oracle/ppo_port.py) driving
  `ensemble_relabel_port` (tests/test_ensemble_relabel_reference.py, held there to what the reference's own wrappers
  record), over two rounds, Box and Discrete;
- `PreferenceComparisons` over `AgentTrainer(DevicePPO, AddSTDRewardWrapper(RewardEnsemble(...)))` end to end, graph
  replay against eager execution, and a changed `default_alpha`;
- the ensembles the fused rollout refuses, each with its message.
"""
import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _dev(x):
    return th.as_tensor(np.ascontiguousarray(x)).cuda().contiguous()


def _relabel_f64(raw, stats, alpha):
    """raw [M][T][E]; stats: per member None or (mean, var, count, eps).  Member m's step t is normalised with its
    statistics from before t, then t's E raw rewards are merged (RunningNorm.update_stats); -> reward [T][E] and the
    final statistics."""
    raw = raw.astype(np.float64)
    M, T, E = raw.shape
    v = np.empty_like(raw)
    final = []
    for m in range(M):
        if stats[m] is None:
            v[m] = raw[m]
            final.append(None)
            continue
        mean, var, cnt, eps = (float(x) for x in stats[m])
        for t in range(T):
            x = raw[m, t]
            v[m, t] = (x - mean) / np.sqrt(var + eps)
            bm, bv = x.mean(), x.var()
            tot = cnt + E
            delta = bm - mean
            mean = mean + delta * E / tot
            var = (var * cnt + bv * E + delta * delta * cnt * E / tot) / tot
            cnt = tot
        final.append((mean, var, int(cnt)))
    rew = v.mean(0) + alpha * np.sqrt(v.var(0, ddof=1))
    return rew, final


# ---------------------------------------------------------------------------------------------
# relabel kernel against the float64 restatement
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [0.0, -0.5, 1.0])
@pytest.mark.parametrize("norm", [True, False])
@pytest.mark.parametrize("T", [1, 9])
@pytest.mark.parametrize("E", [37, 1024])
@pytest.mark.parametrize("M", [2, 5, 16])
def test_relabel_kernel_matches_float64(L, M, E, T, norm, alpha):
    rng = np.random.default_rng(M * 1000 + E + T)
    raw = (rng.standard_normal((M, T, E)) * rng.uniform(0.5, 3, (M, 1, 1)) + rng.normal(0, 2, (M, 1, 1)))
    raw = raw.astype(np.float32)
    stats = [None] * M
    if norm:
        stats = [(rng.normal(0, 1), rng.uniform(0.5, 3), int(rng.integers(0, 500)), 1e-5) for _ in range(M)]
    want, final = _relabel_f64(raw, stats, alpha)
    rw, col = 12, 7
    r = _dev(raw).view(M, T * E)

    def run():
        norms = []
        for s in stats:
            if s is None:
                norms.append(None)
            else:
                norms.append((th.tensor([s[0], s[1]], dtype=th.float32, device="cuda"),
                              th.tensor([s[2]], dtype=th.int32, device="cuda"), s[3]))
        d = L.pref_uncertainty_desc(list(r), norms)
        ws = th.zeros(L.ensemble_relabel_ws_floats(M, T), device="cuda")
        tbl = th.full((E * T, rw), 7.0, device="cuda")
        L.ensemble_relabel(d, alpha, tbl, rw, col, E, T, ws)
        th.cuda.synchronize()
        assert float(ws[0]) == 0.0  # the ticket is re-armed
        return tbl, norms

    tbl, norms = run()
    got = tbl.cpu().numpy().reshape(E, T, rw)
    np.testing.assert_allclose(got[:, :, col], want.T, rtol=2e-5, atol=2e-5)
    other = np.delete(got, col, axis=2)
    assert (other == 7.0).all()  # only the reward column is written
    for m in range(M):
        if norms[m] is None:
            continue
        np.testing.assert_allclose(norms[m][0].cpu().numpy(), final[m][:2], rtol=1e-5, atol=1e-6)
        assert int(norms[m][1]) == stats[m][2] + E * T == final[m][2]
    tbl2, norms2 = run()
    assert th.equal(tbl, tbl2)
    for a, b in zip(norms, norms2):
        if a is not None:
            assert th.equal(a[0], b[0]) and th.equal(a[1], b[1])


# ---------------------------------------------------------------------------------------------
# member rollout + relabel + GAE against the SB3 restatement over two rounds
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", [
    # config 5's shape of reward: normalised members, conservative alpha
    dict(Do=11, Da=3, discrete=False, E=37, T=9, H=5, M=5, out_norm=True, in_norm=False, alpha=-0.5),
    # plain members with input RunningNorms, bare RewardEnsemble (the mean alone)
    dict(Do=4, Da=2, discrete=True, E=64, T=6, H=4, M=3, out_norm=False, in_norm=True, alpha=0.0),
])
def test_ensemble_rollout_matches_oracle(L, cfg):
    from imitation_b200 import _desc
    from oracle import data_port, nets_port, ppo_port, synth_env
    from tests.test_ensemble_relabel_reference import ensemble_relabel_port
    from tests.test_gpu_kernels import _policy_flat

    Do, Da, discrete, E, T, H, M = (cfg[k] for k in ("Do", "Da", "discrete", "E", "T", "H", "M"))
    n_rounds, seed = 2, 11
    th.manual_seed(seed)
    spec = synth_env.SynthEnvSpec(Do, Da, discrete=discrete, horizon=H, seed=seed)
    venv = synth_env.SynthVecEnv(spec, E, env_id_offset=5)
    pol = ppo_port.ActorCriticPort(Do, Da, discrete=discrete, hidden=(32, 32), normalize_features=False)
    with th.no_grad():
        for p in pol.parameters():
            p.add_(0.3 * th.randn_like(p))
    nets, out_norms = [], []
    for m in range(M):
        net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=(32, 32), normalize_input=cfg["in_norm"])
        with th.no_grad():
            if cfg["in_norm"]:
                net.mlp.normalize_input.running_mean.normal_(0, 0.2)
                net.mlp.normalize_input.running_var.uniform_(0.5, 2.0)
        net.eval()
        nets.append(net)
        if cfg["out_norm"]:  # statistics advanced beforehand
            on = nets_port.OutputNormPort()
            on(np.random.default_rng(m).normal(0.3 * m, 1 + m, 50).astype(np.float32))
            out_norms.append(on)
        else:
            out_norms.append(None)
    n_actions = Da if discrete else None
    port = ensemble_relabel_port(list(zip(nets, out_norms)), cfg["alpha"] or None, n_actions)  # 0: bare ensemble
    rng = np.random.default_rng(seed + 1)
    noise = (rng.random((n_rounds * T, E)).astype(np.float32) if discrete
             else rng.standard_normal((n_rounds * T, E, Da)).astype(np.float32))
    buffering = data_port.BufferingPort(venv)
    train_env = data_port.RewardRelabelPort(buffering, port)
    gen = ppo_port.PPOPort(pol, train_env, n_steps=T, gamma=0.97, gae_lambda=0.9, noise_fn=lambda step: noise[step])
    gen._last_obs = train_env._old_obs
    gen._last_starts = np.ones(E, dtype=bool)

    pd = _desc.policy_desc(Do, Da, discrete, 32, False)
    PP = _policy_flat(pol).cuda()
    PN = th.zeros(2, device="cuda")
    dd = _desc.disc_desc(Do, Da, normalize_input=cfg["in_norm"])
    DP = [th.cat([p.detach().reshape(-1) for p in n.mlp.parameters()]).cuda() for n in nets]
    DN = [th.cat([n.mlp.normalize_input.running_mean, n.mlp.normalize_input.running_var]).cuda() if cfg["in_norm"]
          else None for n in nets]
    ON = [None if on is None else (th.tensor([float(on.norm.running_mean), float(on.norm.running_var)],
                                             device="cuda"),
                                   th.tensor([int(on.norm.count)], dtype=th.int32, device="cuda"), 1e-5)
          for on in out_norms]
    env = L.EnvDesc(d_obs=Do, d_act=Da, discrete=int(discrete), horizon=H, seed=seed, env_id_offset=5)
    EP = _dev(_desc.synth_env_params(Do, Da, seed))
    hp = L.PpoHparams(gamma=0.97, gae_lambda=0.9, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                      lr=3e-4, adam_eps=1e-5, n_epochs=1, batch_size=32, normalize_advantage=1)
    st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
    obs = th.empty(Do, E, device="cuda")
    L.env_reset(obs, E, env, st)
    rw = L.rollout_row_width(pd)
    tw = _desc.table_width(Do, Da)
    da_store = 1 if discrete else Da
    c = Do + da_store
    raw = th.empty(M * T * E, device="cuda")
    members = L.rollout_members(DP, DN, raw)
    relabel = L.pref_uncertainty_desc(list(raw.view(M, T * E)), ON)
    ws = th.zeros(L.ensemble_relabel_ws_floats(M, T), device="cuda")
    for rnd in range(n_rounds):
        tbl = th.zeros(E * T, rw, device="cuda")
        flat = th.zeros(E * T, tw, device="cuda")
        aux = th.zeros(2 * E + 2 * E * T, device="cuda")
        nz = _dev(noise[rnd * T:(rnd + 1) * T])
        L.rollout_ensemble(env, EP, obs, pd, PP, PN, dd, members, hp, E, T, tbl, None, 0, flat, aux, nz, st)
        L.ensemble_relabel(relabel, cfg["alpha"], tbl, rw, c + 2, E, T, ws)
        L.gae(tbl, rw, c + 1, E, T, aux, 0.97, 0.9, st, H)
        L.rollout_advance(st, E, T, H, 0)
        th.cuda.synchronize()
        buf = gen.collect_rollouts()
        trajs, _ = buffering.pop_trajectories()
        want_flat = data_port.flatten_port(trajs)
        got = tbl.cpu().numpy().reshape(E, T, rw)

        def col(a):  # oracle [T, E, ...] -> [E, T, ...]
            return np.swapaxes(a, 0, 1)
        # the tolerances of test_rollout_gae_matches_oracle (closed-loop fp32 trajectories)
        np.testing.assert_allclose(got[:, :, :Do], col(buf["obs"]), rtol=1e-3, atol=1e-4, err_msg="obs")
        if discrete:
            np.testing.assert_array_equal(got[:, :, Do], col(buf["actions"]))
        else:
            np.testing.assert_allclose(got[:, :, Do:Do + Da], col(buf["actions"]), rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(got[:, :, c + 1], col(buf["values"]), rtol=1e-3, atol=1e-4, err_msg="value")
        np.testing.assert_allclose(got[:, :, c + 2], col(buf["rewards"]), rtol=1e-3, atol=2e-4, err_msg="reward")
        np.testing.assert_allclose(got[:, :, c + 3], col(buf["advantages"]), rtol=1e-3, atol=5e-4, err_msg="adv")
        np.testing.assert_allclose(got[:, :, c + 4], col(buf["returns"]), rtol=1e-3, atol=5e-4, err_msg="ret")
        gf = flat.cpu().numpy()
        np.testing.assert_array_equal(gf[:, -1] > 0.5, want_flat["dones"])
        np.testing.assert_allclose(gf[:, :Do], want_flat["obs"], rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(gf[:, Do + Da:2 * Do + Da], want_flat["next_obs"], rtol=1e-3, atol=1e-4)
        if discrete:
            np.testing.assert_array_equal(gf[:, Do:Do + Da].argmax(1), want_flat["acts"])
        for on, g in zip(out_norms, ON):
            if on is not None:
                np.testing.assert_allclose(g[0].cpu().numpy(), [float(on.norm.running_mean),
                                                                float(on.norm.running_var)], rtol=1e-5, atol=1e-6)
                assert int(g[1]) == int(on.norm.count)


# ---------------------------------------------------------------------------------------------
# the API: AgentTrainer / PreferenceComparisons on an ensemble reward
# ---------------------------------------------------------------------------------------------
def _ensemble(venv, M, normalized=True, seed=0, **kw):
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    th.manual_seed(seed)
    members = []
    for _ in range(M):
        b = reward_nets.BasicRewardNet(venv.observation_space, venv.action_space, **kw)
        members.append(reward_nets.NormalizedRewardNet(b, networks.RunningNorm) if normalized else b)
    return reward_nets.RewardEnsemble(venv.observation_space, venv.action_space, members).cuda()


def _agent(M, alpha, use_graph, E=8, T=16, H=10):
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets

    venv = synth.DeviceVecEnv(11, 3, E, horizon=H, seed=3)
    reward = reward_nets.AddSTDRewardWrapper(_ensemble(venv, M), default_alpha=alpha)
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=32, n_epochs=1, seed=0)
    algo.use_cuda_graph = use_graph
    return pc.AgentTrainer(algo, reward, venv, np.random.default_rng(0)), reward, algo


def _out_stats(reward):
    return [th.cat([m.normalize_output_layer.running_mean.reshape(1), m.normalize_output_layer.running_var.reshape(1),
                    m.normalize_output_layer.count.reshape(1).float()]).clone() for m in reward.base.members]


def test_graph_replay_equals_eager_and_alpha_takes_effect(L):
    E, T = 8, 16
    runs = {}
    for use_graph in (False, True):
        agent, reward, algo = _agent(5, -0.5, use_graph, E, T)
        counts = [int(m.normalize_output_layer.count) for m in reward.base.members]
        agent.train(steps=3 * E * T)
        agent.buffering_wrapper.discard()
        th.cuda.synchronize()
        assert [int(m.normalize_output_layer.count) for m in reward.base.members] == [c + 3 * E * T for c in counts]
        runs[use_graph] = (algo._tbl.clone(), _out_stats(reward), algo.policy.flat_vectors()[0].clone(), agent,
                           reward, algo)
    assert runs[True][5]._graph is not None  # the second run replayed a captured graph
    assert th.equal(runs[False][0], runs[True][0])
    assert all(th.equal(a, b) for a, b in zip(runs[False][1], runs[True][1]))
    assert th.equal(runs[False][2], runs[True][2])

    # a new default_alpha reaches the next (replayed) rollout: reward column = relabel(raw, stats before) + bootstrap
    _, _, _, agent, reward, algo = runs[True]
    reward.default_alpha = 1.5
    before = [s.cpu().numpy().astype(np.float64) for s in _out_stats(reward)]
    agent.train(steps=E * T)
    agent.buffering_wrapper.discard()
    th.cuda.synchronize()
    raw = algo._scratch["ensemble_raw"].view(5, T, E).cpu().numpy()
    want, final = _relabel_f64(raw, [(b[0], b[1], b[2], 1e-5) for b in before], 1.5)
    rw = algo._tbl.shape[1]
    col_rew = 11 + 3 + 2
    got = algo._tbl.cpu().numpy().reshape(E, T, rw)[:, :, col_rew]
    boot = algo._aux[2 * E:2 * E + E * T].cpu().numpy().reshape(E, T)
    np.testing.assert_allclose(got, want.T + boot, rtol=2e-5, atol=2e-5)
    for s, f in zip(_out_stats(reward), final):
        np.testing.assert_allclose(s[:2].cpu().numpy(), f[:2], rtol=1e-5, atol=1e-6)
        assert int(s[2]) == f[2]


def test_preference_comparisons_on_ensemble_reward(L):
    from imitation_b200.algorithms import preference_comparisons as pc

    E, T, H = 8, 16, 10
    agent, reward, algo = _agent(5, -0.5, True, E, T, H)
    rng = np.random.default_rng(1)
    pcs = pc.PreferenceComparisons(agent, reward, num_iterations=2, fragmenter=pc.RandomFragmenter(warning_threshold=0,
                                                                                                  rng=rng),
                                   fragment_length=5, transition_oversampling=1, initial_comparison_frac=0.5,
                                   initial_epoch_multiplier=1.0, rng=rng)
    res = pcs.train(total_timesteps=4 * E * T, total_comparisons=16)
    assert np.isfinite(res["reward_loss"]) and 0.0 <= res["reward_accuracy"] <= 1.0
    # after training: one more round advances every member's output statistics by exactly E * T
    agent.buffering_wrapper.discard()
    counts = [int(m.normalize_output_layer.count) for m in reward.base.members]
    agent.train(steps=E * T)
    th.cuda.synchronize()
    assert [int(m.normalize_output_layer.count) for m in reward.base.members] == [c + E * T for c in counts]
    assert np.isfinite(algo._tbl.cpu().numpy()).all()


# ---------------------------------------------------------------------------------------------
# what the fused rollout refuses
# ---------------------------------------------------------------------------------------------
def test_unsupported_ensembles_raise(L):
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, reward_wrapper
    from imitation_b200.util import networks

    venv = synth.DeviceVecEnv(5, 2, 4, horizon=6, seed=3)
    obs_sp, act_sp = venv.observation_space, venv.action_space

    def resolve(reward):
        return reward_wrapper.RewardVecEnvWrapper(venv, reward.predict_processed).resolve()

    def basic(**kw):
        return reward_nets.BasicRewardNet(obs_sp, act_sp, **kw).cuda()

    with pytest.raises(NotImplementedError, match="different architecture"):
        resolve(reward_nets.RewardEnsemble(obs_sp, act_sp, [basic(), basic(hid_sizes=(16, 16))]).cuda())
    with pytest.raises(NotImplementedError, match="no fused sm_90a implementation"):
        shaped = reward_nets.ShapedRewardNet(basic(), lambda s: s.sum(1), 0.99)
        resolve(reward_nets.RewardEnsemble(obs_sp, act_sp, [basic(), shaped]).cuda())
    with pytest.raises(NotImplementedError, match="not a mix"):
        mixed = [reward_nets.NormalizedRewardNet(basic(), networks.RunningNorm), basic()]
        resolve(reward_nets.RewardEnsemble(obs_sp, act_sp, mixed).cuda())
    with pytest.raises(NotImplementedError, match="at most 16 ensemble members"):
        resolve(reward_nets.RewardEnsemble(obs_sp, act_sp, [basic() for _ in range(17)]).cuda())
    with pytest.raises(NotImplementedError, match="NormalizedRewardNet around an ensemble"):
        ens = reward_nets.RewardEnsemble(obs_sp, act_sp, [basic(), basic()]).cuda()
        resolve(reward_nets.NormalizedRewardNet(ens, networks.RunningNorm))
    # accepted: both members' engines, alpha read from the wrapper
    ens = reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(obs_sp, act_sp, [basic(), basic()]).cuda(), -0.5)
    rel = resolve(ens)
    assert isinstance(rel, reward_wrapper.EnsembleRelabel) and rel.mode == 2
    assert rel.alpha == -0.5 and rel.out_norms == [None, None] and len(rel.nets) == 2
    # one wrapper resolves its ensemble once; a new default_alpha is still read at every access
    w = reward_wrapper.RewardVecEnvWrapper(venv, ens.predict_processed)
    first = w.resolve()
    ens.default_alpha = 0.25
    assert w.resolve() is first and first.alpha == 0.25


def test_member_images_that_do_not_fit_fail_with_the_limit(L):
    """16 members of 64 x 64 need more shared memory than a CTA has: the rollout names the limit."""
    from imitation_b200.algorithms import ppo
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, reward_wrapper
    from imitation_b200.data import wrappers

    venv = synth.DeviceVecEnv(11, 3, 8, horizon=10, seed=3)
    ens = _ensemble(venv, 16, normalized=False, hid_sizes=(64, 64))
    wrapped = reward_wrapper.RewardVecEnvWrapper(wrappers.BufferingWrapper(venv), ens.predict_processed)
    algo = ppo.DevicePPO("FeedForward32Policy", wrapped, n_steps=4, batch_size=32, n_epochs=1, seed=0)
    with pytest.raises(L.ImbError, match="16-member ensemble needs .* B of shared memory"):
        algo.collect_rollouts()
