"""`NormalizedRewardNet(net, EMANorm)` on the device: `imb_reward_ema_scan` (the rollout's per-step output
normalisation) and the EMA members of `k_pref_frag_norm` (active selection, ensemble relabel).

- the scan against a float64 restatement over env counts, step counts, decays and starting batch counts;
- the fragment fold with EMA members against the scan;
- whole AIRL rounds with an EMA output layer against `oracle.gail_port.AdversarialPort` whose output norm is the
  EMA restatement of tests/test_ema_norm_reference.py, and graph replay against eager rounds;
- `AgentTrainer` with one EMA-normalised net and with an ensemble of them under `AddSTDRewardWrapper`;
- active selection with EMA members, device path against the host loop;
- checkpoints, `load_reward("RewardNet_normalized")`, the reference's state dict, and the refusals.

Tolerances: rewards rtol 2e-6, statistics rtol 1e-6; variances also get atol 1e-6 x the largest variance of the case
(with E = 1 a step's batch variance is 0 and the running variance can approach 0).  CUDA's powf is not bit-identical to
the host's, and the device reduction order differs from torch's.
"""
import copy
import functools
import io

import numpy as np
import pytest
import torch as th

from tests import golden_util as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _ema_f64(raw, mean, var, ilr, cnt, nb, decay, eps):
    """raw [T][E]: step t normalised with the statistics from before it, then folded (EMANorm.update_stats) in
    float64 -> (normalised [T][E], (mean, var, inv_lr, count, num_batches))."""
    raw = raw.astype(np.float64)
    out = np.empty_like(raw)
    for t in range(raw.shape[0]):
        x = raw[t]
        out[t] = (x - mean) / np.sqrt(var + eps)
        ilr += float(np.float32(decay)) ** nb
        lr = 1.0 / ilr
        dm = x.mean() - mean
        mean += lr * dm
        var += lr * (x.var() + (1 - lr) * dm * dm - var)
        cnt += x.size
        nb += 1
    return out, (mean, var, ilr, cnt, nb)


def _ema_start(decay, nb0, rng):
    """Statistics of an EMANorm that has folded nb0 batches (inv_learning_rate = sum_k<nb0 decay^k)."""
    ilr = float(sum(np.float32(decay) ** k for k in range(nb0)))
    return float(rng.normal(0.5, 1)), float(rng.uniform(0.5, 3)), ilr, int(rng.integers(0, 1000)) + 3 * nb0, nb0


def _vectors(s):
    return (th.tensor([s[0], s[1], s[2]], dtype=th.float32, device="cuda"),
            th.tensor([s[3], s[4]], dtype=th.int32, device="cuda"))


def _check_stats(st, ct, want, vscale):
    got = st.cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(got[0], want[0], rtol=1e-6, atol=1e-6 * max(1.0, abs(want[0])))
    np.testing.assert_allclose(got[1], want[1], rtol=1e-6, atol=1e-6 * vscale)
    np.testing.assert_allclose(got[2], want[2], rtol=1e-6)
    assert ct.cpu().tolist() == [want[3], want[4]]  # counts exact


@pytest.mark.parametrize("nb0", [0, 7, 5000])
@pytest.mark.parametrize("decay", [0.5, 0.99, 0.999])
@pytest.mark.parametrize("T", [1, 9, 300])
@pytest.mark.parametrize("E", [1, 37, 1024])
def test_ema_scan_matches_float64(L, E, T, decay, nb0):
    rng = np.random.default_rng(E * 7 + T * 13 + nb0)
    raw = (rng.standard_normal((T, E)) * rng.uniform(0.5, 3) + rng.normal(0, 2)).astype(np.float32)
    s0 = _ema_start(decay, nb0, rng)
    want, final = _ema_f64(raw, *s0, decay, 1e-5)
    # the largest running variance of the case (it can approach 0 with E = 1)
    vscale = max(s0[1], final[1], float(raw.var()))

    def run(update):
        st, ct = _vectors(s0)
        r = th.as_tensor(raw).cuda().contiguous()
        L.reward_norm_scan(r, E, T, E, 1, st, ct, 1e-5, update, ema_decay=decay)
        return r, st, ct

    r, st, ct = run(True)
    np.testing.assert_allclose(r.cpu().numpy(), want, rtol=2e-6, atol=2e-6 * max(1.0, float(np.abs(want).max())))
    _check_stats(st, ct, final, vscale)
    r2, st2, ct2 = run(True)  # two calls give the same bits
    assert th.equal(r, r2) and th.equal(st, st2) and th.equal(ct, ct2)
    # update_stats = False: every step normalised with the starting statistics, which stay bit-unchanged
    r3, st3, ct3 = run(False)
    st0, ct0 = _vectors(s0)
    assert th.equal(st3, st0) and th.equal(ct3, ct0)
    np.testing.assert_allclose(r3.cpu().numpy(), (raw - s0[0]) / np.sqrt(s0[1] + 1e-5), rtol=2e-6, atol=2e-6)


def test_ema_scan_rejects_bad_decay(L):
    st, ct = _vectors((0.0, 1.0, 0.0, 0, 0))
    r = th.zeros(4, device="cuda")
    for bad in (0.0, 1.0, -0.5):
        with pytest.raises(L.ImbError, match="decay"):
            L.reward_norm_scan(r, 4, 1, 4, 1, st, ct, 1e-5, True, ema_decay=bad)


def test_fold_with_ema_members_matches_the_scan(L):
    """k_pref_frag_norm with EMA members equals the EMA scan with E = L envs and T = 2C steps (one fragment per step),
    members of both kinds in one call; two calls give the same bits."""
    gen = th.Generator().manual_seed(5)
    M, C, Lk = 4, 300, 100
    F = 2 * C
    rews = (th.randn(M, F, Lk, generator=gen) * 2.0 + 1.0).cuda()
    starts = {0: (0.3, 1.7, 3.0, 40, 3, 0.99), 2: (-0.2, 0.4, 1.9999, 3000, 400, 0.5), 3: (0.0, 1.0, 0.0, 0, 0, 0.9)}

    def call():
        norms = [None] * M
        for m, s in starts.items():
            st, ct = _vectors(s[:5])
            norms[m] = (st, ct, 1e-5, s[5])
        norms[1] = (th.tensor([0.1, 0.8], device="cuda"), th.tensor([7], dtype=th.int32, device="cuda"), 1e-5)
        ws = th.zeros(L.pref_uncertainty_ws_floats(M, C), device="cuda")
        scores, member = th.empty(C, device="cuda"), th.empty(C, M, device="cuda")
        L.pref_uncertainty(L.pref_uncertainty_desc([rews[m].reshape(-1) for m in range(M)], norms), C, Lk, 0, 0.0,
                           1.0, 50.0, ws, scores, member)
        return scores, member, norms, ws

    scores, member, norms, ws = call()
    aff = ws[1 + 2 * M * F:1 + 4 * M * F].reshape(M, F, 2)
    for m, s in starts.items():
        scan = rews[m].clone()
        st, ct = _vectors(s[:5])
        L.reward_norm_scan(scan, Lk, F, Lk, 1, st, ct, 1e-5, True, ema_decay=s[5])
        np.testing.assert_allclose(norms[m][0].cpu().numpy(), st.cpu().numpy(), rtol=1e-6, atol=1e-6)
        assert norms[m][1].cpu().tolist() == ct.cpu().tolist() == [s[3] + F * Lk, s[4] + F]
        ours = (rews[m] - aff[m, :, 0:1]) * aff[m, :, 1:2]
        np.testing.assert_allclose(ours.cpu().numpy(), scan.cpu().numpy(), rtol=1e-6, atol=1e-6)
    # the RunningNorm member of the same call: k_reward_norm_scan
    scan = rews[1].clone()
    st, ct = th.tensor([0.1, 0.8], device="cuda"), th.tensor([7], dtype=th.int32, device="cuda")
    L.reward_norm_scan(scan, Lk, F, Lk, 1, st, ct, 1e-5, True)
    np.testing.assert_allclose(norms[1][0].cpu().numpy(), st.cpu().numpy(), rtol=1e-6, atol=1e-6)
    assert int(norms[1][1]) == int(ct)
    s2, m2, n2, _ = call()
    assert th.equal(scores, s2) and th.equal(member, m2)
    assert all(th.equal(a[0], b[0]) and th.equal(a[1], b[1]) for a, b in zip(norms, n2))


# ---------------------------------------------------------------------------------------------
# whole AIRL rounds
# ---------------------------------------------------------------------------------------------
def _airl(Do, Da, E, T, H, B, cap, n_disc, seed, decay, sampling="host_compat"):
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms.adversarial import airl
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    th.manual_seed(seed)
    venv = synth.DeviceVecEnv(Do, Da, E, horizon=H, seed=seed)
    gen = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=32, n_epochs=2, seed=seed)
    net = reward_nets.BasicShapedRewardNet(venv.observation_space, venv.action_space,
                                           normalize_input_layer=networks.RunningNorm)
    net = reward_nets.NormalizedRewardNet(net, functools.partial(networks.EMANorm, decay=decay))
    rng = np.random.default_rng(seed)
    n = 4 * B
    demos = dict(obs=rng.standard_normal((n, Do)).astype(np.float32), acts=rng.uniform(-1, 1, (n, Da)).astype(np.float32),
                 next_obs=rng.standard_normal((n, Do)).astype(np.float32), dones=rng.random(n) < 0.05)
    tr = airl.AIRL(demonstrations=demos, demo_batch_size=B, venv=venv, gen_algo=gen, reward_net=net,
                   n_disc_updates_per_round=n_disc, gen_replay_buffer_capacity=cap, sampling=sampling, seed=seed)
    return tr, demos


def test_airl_rounds_match_adversarial_port(L):
    from imitation_b200.algorithms.adversarial import common
    from oracle import gail_port, nets_port, ppo_port, synth_env
    from tests.test_ema_norm_reference import EMANormPort
    from tests.test_round_parity import HP

    Do, Da, E, T, H, B, cap, n_disc, seed, n_rounds, decay = 11, 3, 16, 8, 20, 64, 96, 2, 4, 3, 0.9
    tr, demos = _airl(Do, Da, E, T, H, B, cap, n_disc, seed, decay)
    gen = tr.gen_algo
    N = E * T
    rng = np.random.default_rng(seed + 100)
    noise = rng.standard_normal((n_rounds, T, E, Da)).astype(np.float32)
    perms = np.stack([np.stack([rng.permutation(N) for _ in range(gen.n_epochs)]) for _ in range(n_rounds)])
    spec = synth_env.SynthEnvSpec(Do, Da, discrete=False, horizon=H, seed=seed)
    venv = synth_env.SynthVecEnv(spec, E)
    pol = ppo_port.ActorCriticPort(Do, Da, discrete=False, hidden=(tr.policy.hidden,) * 2, normalize_features=False)
    psd = {k: v.detach().cpu().clone() for k, v in tr.policy.state_dict().items()}
    pol.load_state_dict({"pi.0.weight": psd["mlp_extractor.policy_net.0.weight"],
                         "pi.0.bias": psd["mlp_extractor.policy_net.0.bias"],
                         "pi.2.weight": psd["mlp_extractor.policy_net.2.weight"],
                         "pi.2.bias": psd["mlp_extractor.policy_net.2.bias"],
                         "vf.0.weight": psd["mlp_extractor.value_net.0.weight"],
                         "vf.0.bias": psd["mlp_extractor.value_net.0.bias"],
                         "vf.2.weight": psd["mlp_extractor.value_net.2.weight"],
                         "vf.2.bias": psd["mlp_extractor.value_net.2.bias"],
                         "action_net.weight": psd["action_net.weight"], "action_net.bias": psd["action_net.bias"],
                         "value_net.weight": psd["value_net.weight"], "value_net.bias": psd["value_net.bias"],
                         "log_std": psd["log_std"]}, strict=False)
    flat_noise = noise.reshape((n_rounds * T,) + noise.shape[2:])
    flat_perms = perms.reshape(n_rounds * gen.n_epochs, N)
    pgen = ppo_port.PPOPort(pol, venv, n_steps=T, batch_size=gen.batch_size, n_epochs=gen.n_epochs,
                            noise_fn=lambda step: flat_noise[step], perm_fn=lambda e, n: flat_perms[e], **HP)
    net = nets_port.ShapedRewardNetPort(Do, Da, normalize_input=True)
    net.load_state_dict({G.port_key(k): v.detach().cpu().clone() for k, v in tr._reward_net.base.state_dict().items()})
    net.eval()
    expert = {k: np.asarray(v) for k, v in demos.items()}
    th.manual_seed(seed + 7)
    port = gail_port.AdversarialPort(venv=venv, expert=expert, demo_batch_size=B, gen=pgen, reward_net=net, airl=True,
                                     n_disc_updates_per_round=n_disc, gen_replay_buffer_capacity=cap,
                                     normalize_output=True)
    port.out_norm.norm = EMANormPort(1, decay).eval()
    th.manual_seed(seed + 7)
    tr._expert_compat = common._TorchCompatExpertIndices(len(expert["obs"]), B)
    want = []
    th.manual_seed(seed + 7)
    np.random.seed(seed + 11)
    for r in range(n_rounds):
        port.train(port.gen_train_timesteps)
        want.append({k: v.clone() for k, v in port.out_norm.norm.state_dict().items()})
    wnet = {k: v.detach().clone() for k, v in port.net.state_dict().items()}

    th.manual_seed(seed + 7)
    np.random.seed(seed + 11)
    layer = tr._reward_net.normalize_output_layer
    for r in range(n_rounds):
        gen.noise = th.as_tensor(noise[r]).cuda()
        gen.perm = th.as_tensor(perms[r]).cuda()
        tr.train_gen(tr.gen_train_timesteps)
        for _ in range(tr.n_disc_updates_per_round):
            tr.train_disc()
        tr.join()
        th.cuda.synchronize()
        w = want[r]
        assert int(layer.num_batches) == int(w["num_batches"]) == (r + 1) * T
        assert int(layer.count) == int(w["count"]) == (r + 1) * T * E
        # closed-loop rollouts: fp32 differences compound over steps and rounds (test_round_parity's tolerances)
        for k in ("running_mean", "running_var", "inv_learning_rate"):
            np.testing.assert_allclose(getattr(layer, k).cpu().numpy(), w[k].numpy(), rtol=2e-3, atol=2e-4,
                                       err_msg=f"round {r} {k}")
    ours = {G.port_key(k): v.detach().cpu() for k, v in tr._reward_net.base.state_dict().items()}
    for k, v in wnet.items():
        if k.endswith("count"):
            assert int(ours[k]) == int(v), k
        else:
            np.testing.assert_allclose(ours[k].numpy(), v.numpy(), rtol=2e-3, atol=2e-4, err_msg=k)


def test_airl_graph_replay_equals_eager(L):
    runs = []
    for use_graph in (False, True):
        tr, _ = _airl(11, 3, 16, 8, 20, 64, 96, 2, 6, 0.99, sampling="device")
        tr.gen_algo.use_cuda_graph = use_graph
        tr.train(3 * tr.gen_train_timesteps)
        tr.join()
        th.cuda.synchronize()
        runs.append((tr, {k: v.detach().clone() for k, v in tr._reward_net.state_dict().items()},
                     tr.policy.flat_vectors()[0].clone(), tr.gen_algo._tbl.clone()))
    assert runs[1][0].gen_algo._graph is not None  # the second run replayed a captured graph
    assert runs[0][1].keys() == runs[1][1].keys()
    for k in runs[0][1]:
        assert th.equal(runs[0][1][k], runs[1][1][k]), k
    assert th.equal(runs[0][2], runs[1][2]) and th.equal(runs[0][3], runs[1][3])
    assert int(runs[1][0]._reward_net.normalize_output_layer.num_batches) == 3 * 8


# ---------------------------------------------------------------------------------------------
# AgentTrainer: one EMA-normalised net, and an ensemble of them
# ---------------------------------------------------------------------------------------------
def _ema_stats(n):
    return (float(n.running_mean), float(n.running_var), float(n.inv_learning_rate), int(n.count),
            int(n.num_batches))


def test_agent_trainer_on_ema_ensemble_matches_restatement(L):
    """Two rollouts of AgentTrainer(DevicePPO, AddSTDRewardWrapper(RewardEnsemble(5 x NormalizedRewardNet(
    BasicRewardNet, EMANorm)), -0.5)): the reward column equals the float64 restatement on the members' raw rewards,
    and every member's statistics end where it ends."""
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    E, T, H, M, decay, alpha = 8, 16, 10, 5, 0.95, -0.5
    venv = synth.DeviceVecEnv(11, 3, E, horizon=H, seed=3)
    th.manual_seed(0)
    nets = [reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space, venv.action_space),
                                            functools.partial(networks.EMANorm, decay=decay)).cuda() for _ in range(M)]
    reward = reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(venv.observation_space, venv.action_space,
                                                                        nets), alpha)
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=32, n_epochs=1, seed=0)
    agent = pc.AgentTrainer(algo, reward, venv, np.random.default_rng(0))
    for _ in range(2):
        before = [_ema_stats(n.normalize_output_layer) for n in nets]
        agent.train(steps=E * T)
        agent.buffering_wrapper.discard()
        th.cuda.synchronize()
        raw = algo._scratch["ensemble_raw"].view(M, T, E).cpu().numpy()
        vals, finals = zip(*[_ema_f64(raw[m], *before[m], decay, 1e-5) for m in range(M)])
        v = np.stack(vals)
        want = v.mean(0) + alpha * np.sqrt(v.var(0, ddof=1))
        rw = algo._tbl.shape[1]
        got = algo._tbl.cpu().numpy().reshape(E, T, rw)[:, :, 11 + 3 + 2]
        boot = algo._aux[2 * E:2 * E + E * T].cpu().numpy().reshape(E, T)
        # the tolerance of the RunningNorm ensemble's agent test: a freshly initialised member's outputs spread little
        # around their mean, so (x - mean) / std amplifies float32 rounding of the mean
        np.testing.assert_allclose(got, want.T + boot, rtol=2e-5, atol=2e-5)
        for n, f in zip(nets, finals):
            st, ct = n.output_norm_vectors()
            _check_stats(st, ct, f, max(f[1], 1.0))


def test_agent_trainer_single_net_matches_host_predict_processed(L):
    """One EMA-normalised net: the rollout's reward column equals the host `predict_processed` (the module's own torch
    ops) called step by step on the same transitions, from a copy of the net taken before the rollout."""
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    E, T, H, decay = 8, 16, 100, 0.9  # no episode ends inside the two rollouts: next obs = the next row's obs
    venv = synth.DeviceVecEnv(11, 3, E, horizon=H, seed=3)
    th.manual_seed(0)
    net = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space, venv.action_space),
                                          functools.partial(networks.EMANorm, decay=decay)).cuda()
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=32, n_epochs=1, seed=0)
    agent = pc.AgentTrainer(algo, net, venv, np.random.default_rng(0))
    for r in range(2):
        host = copy.deepcopy(net)
        agent.train(steps=E * T)
        agent.buffering_wrapper.discard()
        th.cuda.synchronize()
        n = net.normalize_output_layer
        assert int(n.num_batches) == (r + 1) * T and int(n.count) == (r + 1) * E * T
        tbl = algo._tbl.cpu().numpy().reshape(E, T, algo._tbl.shape[1])
        obs, acts = tbl[:, :, :11], np.clip(tbl[:, :, 11:14], -1.0, 1.0)
        boot = algo._aux[2 * E:2 * E + E * T].cpu().numpy().reshape(E, T)
        want = np.stack([host.predict_processed(obs[:, t], acts[:, t], obs[:, t + 1], np.zeros(E, bool))
                         for t in range(T - 1)], 1)
        got = tbl[:, :T - 1, 11 + 3 + 2] - boot[:, :T - 1]
        np.testing.assert_allclose(got, want, rtol=2e-6, atol=2e-6 * max(1.0, float(np.abs(want).max())))


# ---------------------------------------------------------------------------------------------
# active selection with EMA members: device path against the host loop
# ---------------------------------------------------------------------------------------------
def _active(use_device):
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks
    from tests import test_active_selection as tas
    from tests.test_ema_norm_reference import ACTIVE, ACTIVE_DECAY, active_golden

    g, cands, _ = active_golden()
    Do, n_act, Da, M, hid, _, _, threshold = ACTIVE
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1.0, 1.0, (Da,))
    members = []
    for k in range(M):
        net = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs_space, act_space, hid_sizes=hid),
                                              functools.partial(networks.EMANorm, decay=ACTIVE_DECAY))
        net.load_state_dict({kk[len(f"member{k}/"):]: th.as_tensor(np.array(v)) for kk, v in g.items()
                             if kk.startswith(f"member{k}/")})
        members.append(net.cuda())
    ens = reward_nets.RewardEnsemble(obs_space, act_space, members)
    pm = pc.PreferenceModel(ens, noise_prob=tas.NOISE, discount_factor=tas.DISCOUNT, threshold=threshold)
    pm.use_fragment_pool = use_device
    pairs = [(tas._as_traj(a), tas._as_traj(b)) for a, b in cands]
    return g, ens, pm, pairs


@pytest.mark.parametrize("mode", ("logit", "probability", "label"))
def test_active_selection_device_matches_host_loop_and_golden(L, mode):
    from imitation_b200.algorithms import preference_comparisons as pc
    from tests import test_active_selection as tas
    from tests.test_ema_norm_reference import check_selection

    g, ens_d, pm_d, pairs = _active(True)
    _, ens_h, pm_h, _ = _active(False)
    scores, member = copy.deepcopy(pm_d).uncertainty_scores(pairs, mode, member_values=True)
    scores, member = scores.cpu().numpy(), member.cpu().numpy()
    tas._check_scores(g, mode, scores, diffs=member if mode == "logit" else None,
                      probs=member if mode != "logit" else None)
    frag_d = pc.ActiveSelectionFragmenter(pm_d, lambda **kw: pairs, tas.FACTOR, uncertainty_on=mode)
    frag_h = pc.ActiveSelectionFragmenter(pm_h, lambda **kw: pairs, tas.FACTOR, uncertainty_on=mode)
    got_d, got_h = frag_d(pairs, tas.L, tas.NUM_PAIRS), frag_h(pairs, tas.L, tas.NUM_PAIRS)
    sel = np.array([next(i for i, p in enumerate(pairs) if p is c) for c in got_d])
    check_selection(g, mode, scores, sel)
    if mode == "logit":  # no ties: the host loop selects the same pairs
        assert [id(p) for p in got_d] == [id(p) for p in got_h]
    assert pm_h._pool is None
    for k, (md, mh) in enumerate(zip(ens_d.members, ens_h.members)):
        a, b = md.normalize_output_layer, mh.normalize_output_layer
        sa, sb = _ema_stats(a), _ema_stats(b)
        np.testing.assert_allclose(sa[:3], sb[:3], rtol=1e-6, atol=1e-6)
        assert sa[3:] == sb[3:] == (int(g[f"{mode}/out_count{k}"]), int(g[f"{mode}/out_batches{k}"]))
        np.testing.assert_allclose(sa[:2], g[f"{mode}/out_stats{k}"], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(sa[2], g[f"{mode}/out_ema{k}"], rtol=1e-6)


# ---------------------------------------------------------------------------------------------
# checkpoints, the reference's state dict, refusals, and the AIRL config of the reference's ingredient
# ---------------------------------------------------------------------------------------------
def test_checkpoint_round_trip_and_load_reward(L, tmp_path):
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, serialize
    from imitation_b200.util import networks

    venv = synth.DeviceVecEnv(5, 2, 4, horizon=6, seed=3)
    th.manual_seed(0)
    net = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space, venv.action_space),
                                          functools.partial(networks.EMANorm, decay=0.9)).cuda()
    rng = np.random.default_rng(0)
    batch = lambda n: (rng.standard_normal((n, 5)).astype(np.float32), rng.uniform(-1, 1, (n, 2)).astype(np.float32),
                       rng.standard_normal((n, 5)).astype(np.float32), np.zeros(n, bool))
    for n in (7, 3, 11):
        net.predict_processed(*batch(n))
    st, ct = net.output_norm_vectors()  # the buffers alias the device vectors
    assert net.normalize_output_layer.inv_learning_rate.data_ptr() == st.data_ptr() + 8
    assert net.normalize_output_layer.num_batches.data_ptr() == ct.data_ptr() + 4
    assert ct.cpu().tolist() == [21, 3]
    path = tmp_path / "net.pt"
    th.save(net, path)
    back = th.load(path, weights_only=False)
    assert back.normalize_output_layer.decay == 0.9 and back.output_norm_is_ema
    for k, v in net.state_dict().items():
        assert th.equal(v, back.state_dict()[k]), k
    x = batch(9)
    np.testing.assert_array_equal(copy.deepcopy(net).predict_processed(*x), back.predict_processed(*x))
    fn = serialize.load_reward("RewardNet_normalized", str(path), venv)
    want = th.load(path, weights_only=False).predict_processed(*x, update_stats=False)
    np.testing.assert_array_equal(fn(*x), want)
    fn(*batch(6))
    np.testing.assert_array_equal(fn(*x), want)  # update_stats=False: the statistics stay where they were
    buf = io.BytesIO()
    th.save(net.state_dict(), buf)
    buf.seek(0)
    fresh = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(venv.observation_space, venv.action_space),
                                            networks.EMANorm).cuda()
    fresh.load_state_dict(th.load(buf))
    st2, ct2 = fresh.output_norm_vectors()
    assert th.equal(st, st2) and th.equal(ct, ct2)


def test_reference_state_dict_loads(L):
    """A state dict with the reference's EMANorm buffers (the golden's disc09 case, recorded from the reference's own
    module) loads, and the device scan continues from it."""
    from imitation_b200 import spaces
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    z = G.load("ema_output_norm")
    sd = {k: th.as_tensor(np.array(v)) for k, v in G.sub(z, "disc09/member_after0").items()}
    obs, act = spaces.Box(-np.inf, np.inf, (4,)), spaces.Discrete(3)
    net = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs, act),
                                          functools.partial(networks.EMANorm, decay=0.9)).cuda()
    net.load_state_dict(sd)
    st, ct = net.output_norm_vectors()
    n = net.normalize_output_layer
    assert ct.cpu().tolist() == [int(sd["normalize_output_layer.count"]), int(sd["normalize_output_layer.num_batches"])]
    np.testing.assert_array_equal(st.cpu().numpy(), [float(sd["normalize_output_layer.running_mean"]),
                                                     float(sd["normalize_output_layer.running_var"]),
                                                     float(sd["normalize_output_layer.inv_learning_rate"])])
    assert int(n.num_batches) == 150 + 9


def test_mixed_kind_ensemble_and_input_ema_raise(L):
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, reward_wrapper
    from imitation_b200.util import networks

    venv = synth.DeviceVecEnv(5, 2, 4, horizon=6, seed=3)
    obs_sp, act_sp = venv.observation_space, venv.action_space

    def basic():
        return reward_nets.BasicRewardNet(obs_sp, act_sp).cuda()

    mixed = [reward_nets.NormalizedRewardNet(basic(), networks.RunningNorm),
             reward_nets.NormalizedRewardNet(basic(), networks.EMANorm)]
    ens = reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(obs_sp, act_sp, mixed).cuda(), -0.5)
    with pytest.raises(NotImplementedError, match="output norms must all be RunningNorm or all EMANorm, not a mix"):
        reward_wrapper.RewardVecEnvWrapper(venv, ens.predict_processed).resolve()
    same = [reward_nets.NormalizedRewardNet(basic(), networks.EMANorm) for _ in range(2)]
    ens = reward_nets.RewardEnsemble(obs_sp, act_sp, same).cuda()
    rel = reward_wrapper.RewardVecEnvWrapper(venv, ens.predict_processed).resolve()
    assert all(o.output_norm_is_ema for o in rel.out_norms)
    with pytest.raises(NotImplementedError, match="normalize_input_layer must be RunningNorm or None"):
        reward_nets.BasicShapedRewardNet(obs_sp, act_sp, normalize_input_layer=networks.EMANorm)


def test_airl_with_normalize_output_ema_trains(L):
    """The reward net of the reference's `reward.normalize_output_ema` config (BasicShapedRewardNet inside
    NormalizedRewardNet(net, EMANorm), input RunningNorm) trains through AIRL.train."""
    tr, _ = _airl(17, 6, 64, 16, 50, 128, 2048, 2, 1, 0.99, sampling="device")
    tr.train(4 * tr.gen_train_timesteps)
    tr.join()
    th.cuda.synchronize()
    n = tr._reward_net.normalize_output_layer
    assert int(n.num_batches) == 4 * 16 and int(n.count) == 4 * 16 * 64
    assert np.isfinite([float(n.running_mean), float(n.running_var), float(n.inv_learning_rate)]).all()
