"""Active selection of preference queries (`ActiveSelectionFragmenter`, reference preference_comparisons.py:668-778).

The stored results in tests/golden/active_selection.npz come from the reference's own `ActiveSelectionFragmenter`,
with its `base_fragmenter` and `variance_estimate` wrapped only to record what they return and receive.  Two ensembles
(five NormalizedRewardNet members with advanced output statistics on a Box task, three BasicRewardNets with input
RunningNorms on a Discrete-action task), each scored in the three modes from the same member states.  Re-record them
where the reference sources are importable (oracle/refimport.py) with

    IMB_RECORD_REFERENCE=1 python -m pytest tests/test_active_selection.py -k reference_records

Where they are importable, the same test regenerates the results and compares them with the stored file.

The CPU restatement below (`active_selection_port`) is pinned by the same file; on the GPU the device path
(`imb_pref_uncertainty`) is held to it, and the kernel itself to a float64 restatement.
"""
import copy
import os
import tempfile

import numpy as np
import pytest
import torch as th

from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "active_selection.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
MODES = ("logit", "probability", "label")
# name: (d_obs, n_actions | None, d_act, members, hid_sizes, output norm, input norm, threshold)
CONFIGS = {
    "box": (11, None, 3, 5, (32, 32), True, False, 2.0),
    "discrete": (4, 2, 2, 3, (64, 64), False, True, 0.3),
}
L, NUM_PAIRS, FACTOR, NOISE, DISCOUNT = 25, 8, 3, 0.1, 0.9


# ------------------------------------------------------------------------------------------------
# recording (reference only)
# ------------------------------------------------------------------------------------------------
def _record_config(name, cfg, seed):
    from oracle import refimport

    refimport.load()
    from gymnasium import spaces
    from imitation.algorithms import preference_comparisons as ref_pc
    from imitation.data import types as ref_types
    from imitation.rewards import reward_nets as ref_nets
    from imitation.util import logger as ref_logger
    from imitation.util import networks as ref_networks

    Do, n_act, Da, M, hid, out_norm, in_norm, threshold = cfg
    rng = np.random.default_rng(seed)
    trajs = []
    for i in range(6):
        n = int(rng.integers(40, 80))
        acts = (rng.integers(0, n_act, n) if n_act else rng.uniform(-1, 1, (n, Da)).astype(np.float32))
        trajs.append(ref_types.TrajectoryWithRew(obs=rng.standard_normal((n + 1, Do)).astype(np.float32), acts=acts,
                                                 infos=None, terminal=bool(i % 2),
                                                 rews=rng.standard_normal(n).astype(np.float32)))
    obs_space = spaces.Box(-np.inf, np.inf, (Do,), np.float32)
    act_space = spaces.Discrete(n_act) if n_act else spaces.Box(-1.0, 1.0, (Da,), np.float32)
    th.manual_seed(seed)
    members = []
    for _ in range(M):
        kw = dict(normalize_input_layer=ref_networks.RunningNorm) if in_norm else {}
        net = ref_nets.BasicRewardNet(obs_space, act_space, hid_sizes=hid, **kw)
        if in_norm:  # non-trivial input statistics (eval mode: they stay put)
            nrm = net.mlp.normalize_input
            nrm.running_mean.copy_(th.as_tensor(0.3 * rng.standard_normal(nrm.running_mean.shape), dtype=th.float32))
            nrm.running_var.copy_(th.as_tensor(rng.uniform(0.5, 2.0, nrm.running_var.shape), dtype=th.float32))
            nrm.count.fill_(100)
        if out_norm:
            net = ref_nets.NormalizedRewardNet(net, ref_networks.RunningNorm)
            for k in range(3):  # advance the output statistics
                n = 10 + 7 * k
                net.predict_processed(rng.standard_normal((n, Do)).astype(np.float32),
                                      rng.uniform(-1, 1, (n, Da)).astype(np.float32),
                                      rng.standard_normal((n, Do)).astype(np.float32), np.zeros(n, dtype=bool))
        members.append(net)
    ens = ref_nets.RewardEnsemble(obs_space, act_space, members)
    init = [{k: v.detach().clone() for k, v in m.state_dict().items()} for m in members]
    out = {}
    for i, t in enumerate(trajs):
        out.update({f"traj{i}/{k}": np.asarray(v) for k, v in dict(obs=t.obs, acts=t.acts, rews=t.rews,
                                                                   terminal=t.terminal).items()})
    for k, m in enumerate(members):
        out.update({f"member{k}/{key}": v.numpy().copy() for key, v in init[k].items()})
    log = ref_logger.configure(tempfile.mkdtemp(prefix="imb_golden_log_active"), format_strs=[])
    for mode in MODES:
        for m, st in zip(members, init):
            m.load_state_dict(st)
        pm = ref_pc.PreferenceModel(ens, noise_prob=NOISE, discount_factor=DISCOUNT, threshold=threshold)
        base = ref_pc.RandomFragmenter(rng=np.random.default_rng(seed + 1), warning_threshold=0, custom_logger=log)
        seen = {}

        def base_fragmenter(**kw):
            seen["candidates"] = base(**kw)
            return seen["candidates"]

        frag = ref_pc.ActiveSelectionFragmenter(pm, base_fragmenter, FACTOR, uncertainty_on=mode, custom_logger=log)
        inner = frag.variance_estimate
        rec = {"scores": [], "diff": [], "probs": []}

        def variance_estimate(rews1, rews2):
            v = inner(rews1, rews2)
            rec["scores"].append(float(v))
            rec["diff"].append((rews1.sum(0) - rews2.sum(0)).numpy())
            rec["probs"].append(pm.probability(rews1, rews2).numpy())
            return v

        frag.variance_estimate = variance_estimate
        chosen = frag(trajs, L, NUM_PAIRS)
        cands = seen["candidates"]
        ids = {id(p): i for i, p in enumerate(cands)}
        out[f"{mode}/selected"] = np.array([ids[id(p)] for p in chosen])
        out[f"{mode}/scores"] = np.array(rec["scores"])
        out[f"{mode}/diff"] = np.stack(rec["diff"])
        out[f"{mode}/probs"] = np.stack(rec["probs"])
        if mode == MODES[0]:
            for i, (a, b) in enumerate(cands):
                for s, f in (("a", a), ("b", b)):
                    out.update({f"cand{i}/{s}/{k}": np.asarray(v) for k, v in dict(
                        obs=f.obs, acts=f.acts, rews=f.rews, terminal=f.terminal).items()})
        else:  # every mode draws the same candidates (same seed)
            for i, (a, b) in enumerate(cands):
                np.testing.assert_array_equal(a.obs, out[f"cand{i}/a/obs"])
        if out_norm:
            for k, m in enumerate(members):
                nrm = m.normalize_output_layer
                out[f"{mode}/out_stats{k}"] = np.array([nrm.running_mean.item(), nrm.running_var.item()], np.float32)
                out[f"{mode}/out_count{k}"] = np.array(int(nrm.count.item()))
        if mode == "probability":
            assert (np.abs(out[f"{mode}/diff"]) > threshold).any(), "no clipped pair: lower the threshold"
    return {f"{name}/{k}": v for k, v in out.items()}


def _reference_available() -> bool:
    from oracle import refimport

    return refimport.available()


def _record_all():
    rng_state = th.get_rng_state()
    try:
        out = {}
        for seed, (name, cfg) in enumerate(CONFIGS.items()):
            out.update(_record_config(name, cfg, 31 + 10 * seed))
        return out
    finally:
        th.set_rng_state(rng_state)


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_golden_is_what_the_reference_records():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead).
    Candidates, selections and counts must be identical; floats may differ in the last bits on another CPU, and the
    reference's unstable sort may order label-mode ties differently there."""
    out = _record_all()
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = G.load("active_selection")
    assert set(z.files) == set(out)
    for k, v in out.items():
        want = z[k]
        if k.endswith("label/selected"):
            scores = out[k.replace("selected", "scores")]
            np.testing.assert_array_equal(np.sort(scores[v]), np.sort(scores[want]), err_msg=k)
        elif np.issubdtype(np.asarray(v).dtype, np.floating):
            np.testing.assert_allclose(v, want, rtol=1e-6, atol=1e-7, err_msg=k)
        else:
            np.testing.assert_array_equal(v, want, err_msg=k)


# ------------------------------------------------------------------------------------------------
# golden access and the CPU restatement
# ------------------------------------------------------------------------------------------------
def _golden(name):
    z = G.load("active_selection")
    g = {k: z[k] for k in z.files if k.startswith(name + "/")}
    g = {k[len(name) + 1:]: v for k, v in g.items()}
    n = 0
    while f"cand{n}/a/obs" in g:
        n += 1
    cands = [tuple(dict(obs=g[f"cand{i}/{s}/obs"], acts=g[f"cand{i}/{s}/acts"], rews=g[f"cand{i}/{s}/rews"],
                        terminal=bool(g[f"cand{i}/{s}/terminal"])) for s in ("a", "b")) for i in range(n)]
    return g, cands


def _sub(g, prefix):
    return {k[len(prefix) + 1:]: v for k, v in g.items() if k.startswith(prefix + "/")}


def _score_tol(g, mode):
    """rtol 1e-5 and atol 1e-6 * max(1, max |return difference|)^2: the variance of near-equal numbers cancels."""
    return 1e-5, 1e-6 * max(1.0, float(np.abs(g[f"{mode}/diff"]).max())) ** 2


def active_selection_port(members, pairs, mode, num_pairs, noise_prob, discount, threshold, n_actions=None):
    """ActiveSelectionFragmenter.__call__ (:721-747) + variance_estimate (:749-778) over oracle members
    (BasicRewardNetPort, OutputNormPort | None): one predict_processed per member and fragment, pair by pair.
    Returns (selected indices under the stable tie rule, scores, per-member return differences, probabilities)."""
    from oracle import nets_port, pref_port

    def rewards(frag):
        tr = pref_port.fragment_transitions(frag)
        cols = []
        for net, out in members:
            raw = nets_port.predict_port(net, *tr, n_actions=n_actions)
            cols.append(out(raw) if out is not None else raw)
        return th.as_tensor(np.stack(cols, -1))

    scores, diffs, probs = [], [], []
    for a, b in pairs:
        r1, r2 = rewards(a), rewards(b)
        diff = r1.sum(0) - r2.sum(0)
        p = pref_port.probability_port(r1, r2, noise_prob, discount, threshold).numpy()
        if mode == "logit":
            v = diff.var().item()
        elif mode == "probability":
            v = p.var()
        else:
            q = (p > 0.5).astype(np.float32).mean()
            v = q * (1 - q)
        scores.append(v)
        diffs.append(diff.numpy())
        probs.append(p)
    scores = np.array(scores)
    return np.argsort(scores, kind="stable")[::-1][:num_pairs], scores, np.stack(diffs), np.stack(probs)


def _port_members(g, cfg):
    from oracle import nets_port

    Do, n_act, Da, M, hid, out_norm, in_norm, _ = cfg
    members = []
    for k in range(M):
        st = _sub(g, f"member{k}")
        net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=hid, normalize_input=in_norm)
        net.load_state_dict({kk.replace("_base.", ""): th.as_tensor(np.array(v)) for kk, v in st.items()
                             if not kk.startswith("normalize_output_layer.")})
        out = None
        if out_norm:
            out = nets_port.OutputNormPort()
            out.norm.running_mean.copy_(th.as_tensor(st["normalize_output_layer.running_mean"]))
            out.norm.running_var.copy_(th.as_tensor(st["normalize_output_layer.running_var"]))
            out.norm.count.fill_(int(st["normalize_output_layer.count"]))
        members.append((net, out))
    return members


def _check_scores(g, mode, scores, diffs=None, probs=None):
    rtol, atol = _score_tol(g, mode)
    want = g[f"{mode}/scores"]
    if mode == "label":  # exact, except where a member's probability sits on the 0.5 boundary
        edge = (np.abs(g[f"{mode}/probs"] - 0.5) < 1e-6).any(1)
        np.testing.assert_array_equal(np.asarray(scores, np.float32)[~edge], want.astype(np.float32)[~edge])
    else:
        np.testing.assert_allclose(scores, want, rtol=rtol, atol=atol)
    if diffs is not None:
        np.testing.assert_allclose(diffs, g[f"{mode}/diff"], rtol=1e-5, atol=1e-5)
    if probs is not None:
        np.testing.assert_allclose(probs, g[f"{mode}/probs"], rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("mode", MODES)
def test_port_matches_reference_golden(name, mode):
    cfg = CONFIGS[name]
    g, cands = _golden(name)
    members = _port_members(g, cfg)
    sel, scores, diffs, probs = active_selection_port(members, cands, mode, NUM_PAIRS, NOISE, DISCOUNT, cfg[-1],
                                                      n_actions=cfg[1])
    assert len(cands) == FACTOR * NUM_PAIRS
    _check_scores(g, mode, scores, diffs, probs)
    if cfg[5]:
        for k, (_, out) in enumerate(members):
            np.testing.assert_allclose([out.norm.running_mean.item(), out.norm.running_var.item()],
                                       g[f"{mode}/out_stats{k}"], rtol=1e-6, atol=1e-6)
            assert int(out.norm.count) == int(g[f"{mode}/out_count{k}"])
    _check_selection(g, mode, scores, sel)


def _check_selection(g, mode, scores, sel):
    """`sel` is the stable rule on `scores`, exactly, and the reference's choice up to swaps at the cutoff."""
    np.testing.assert_array_equal(sel, np.argsort(scores, kind="stable")[::-1][:NUM_PAIRS])
    want = g[f"{mode}/selected"]
    ref_scores = g[f"{mode}/scores"]
    if mode == "label":
        np.testing.assert_array_equal(np.sort(ref_scores[sel]), np.sort(ref_scores[want]))
        return
    rtol, atol = _score_tol(g, mode)
    cut = np.sort(ref_scores)[::-1][NUM_PAIRS - 1]
    near = np.abs(ref_scores - cut) <= atol + rtol * abs(cut)
    assert set(sel[~near[sel]]) == set(want[~near[want]])
    np.testing.assert_array_equal(sel[~near[sel]], want[~near[want]])


def test_tie_rule_is_descending_score_then_descending_index():
    scores = np.array([0.25, 0.0, 0.25, 0.1875, 0.25, 0.0], dtype=np.float32)
    order = np.argsort(scores, kind="stable")[::-1]
    assert order.tolist() == [4, 2, 0, 3, 5, 1]
    # the device selection (torch stable sort, reversed) gives the same order
    assert th.argsort(th.as_tensor(scores), stable=True).flip(0).tolist() == order.tolist()


def test_constructor_errors():
    from imitation_b200.algorithms import preference_comparisons as pc

    class _Single:
        ensemble_model = None

    class _Ensemble:
        ensemble_model = object()

    base = pc.RandomFragmenter(rng=np.random.default_rng(0))
    with pytest.raises(ValueError, match="PreferenceModel not wrapped over an ensemble of networks."):
        pc.ActiveSelectionFragmenter(_Single(), base, 2.0)
    with pytest.raises(ValueError, match="variance not supported"):
        pc.ActiveSelectionFragmenter(_Ensemble(), base, 2.0, uncertainty_on="variance")
    for mode in MODES:
        assert pc.ActiveSelectionFragmenter(_Ensemble(), base, 2.0, uncertainty_on=mode).uncertainty_on == mode


def test_empty_candidate_list_returns_nothing():
    from imitation_b200 import _lib
    from imitation_b200.algorithms import preference_comparisons as pc

    class _Ensemble:
        ensemble_model = object()

        def uncertainty_scores(self, *a, **k):
            raise AssertionError("nothing to score")

    n0 = _lib.LAUNCHES["count"]
    frag = pc.ActiveSelectionFragmenter(_Ensemble(), lambda **kw: [], 2.0)
    assert frag([], 10, 0) == []
    assert _lib.LAUNCHES["count"] == n0


# ------------------------------------------------------------------------------------------------
# GPU: the device path
# ------------------------------------------------------------------------------------------------
def _as_traj(d):
    from imitation_b200.data import types

    return types.TrajectoryWithRew(obs=d["obs"], acts=d["acts"], infos=None, terminal=d["terminal"], rews=d["rews"])


def _device_ensemble(g, cfg):
    from imitation_b200 import spaces
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    Do, n_act, Da, M, hid, out_norm, in_norm, _ = cfg
    obs_space = spaces.Box(-np.inf, np.inf, (Do,))
    act_space = spaces.Discrete(n_act) if n_act else spaces.Box(-1.0, 1.0, (Da,))
    members = []
    for k in range(M):
        kw = dict(normalize_input_layer=networks.RunningNorm) if in_norm else {}
        net = reward_nets.BasicRewardNet(obs_space, act_space, hid_sizes=hid, **kw)
        if out_norm:
            net = reward_nets.NormalizedRewardNet(net, networks.RunningNorm)
        net.load_state_dict({kk: th.as_tensor(np.array(v)) for kk, v in _sub(g, f"member{k}").items()})
        members.append(net.cuda())
    return reward_nets.RewardEnsemble(obs_space, act_space, members)


def _device_run(name, mode, use_device=True):
    from imitation_b200.algorithms import preference_comparisons as pc

    cfg = CONFIGS[name]
    g, cands = _golden(name)
    ens = _device_ensemble(g, cfg)
    pm = pc.PreferenceModel(ens, noise_prob=NOISE, discount_factor=DISCOUNT, threshold=cfg[-1])
    pm.use_fragment_pool = use_device
    pairs = [(_as_traj(a), _as_traj(b)) for a, b in cands]
    frag = pc.ActiveSelectionFragmenter(pm, lambda **kw: pairs, FACTOR, uncertainty_on=mode)
    return g, cfg, ens, pm, pairs, frag


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("mode", MODES)
def test_device_path_matches_reference_golden(name, mode):
    g, cfg, ens, pm, pairs, frag = _device_run(name, mode)
    # member values of the same call, from a copy of the models (the call advances the output statistics)
    pm2 = copy.deepcopy(pm)
    scores, member = pm2.uncertainty_scores(pairs, mode, member_values=True)
    chosen = frag(pairs, L, NUM_PAIRS)
    sel = np.array([next(i for i, p in enumerate(pairs) if p is c) for c in chosen])
    assert all(c is pairs[i] for c, i in zip(chosen, sel))  # the candidate objects themselves
    scores = scores.cpu().numpy()
    member = member.cpu().numpy()
    _check_scores(g, mode, scores, diffs=member if mode == "logit" else None,
                  probs=member if mode != "logit" else None)
    _check_selection(g, mode, scores, sel)
    if cfg[5]:
        for k, m in enumerate(ens.members):
            nrm = m.normalize_output_layer
            np.testing.assert_allclose([nrm.running_mean.item(), nrm.running_var.item()], g[f"{mode}/out_stats{k}"],
                                       rtol=1e-6, atol=1e-6)
            assert int(nrm.count) == int(g[f"{mode}/out_count{k}"])
    # only the selected fragments entered the fragment pool
    pool = pm._pool
    assert len(pool._slots) == 2 * NUM_PAIRS
    assert {id(f) for p in chosen for f in p} == set(pool._slots)


@pytest.mark.gpu
def test_device_and_host_loop_select_the_same_pairs():
    """The forced host loop (the reference's per-pair predict_processed calls) and the device path agree on a case
    without ties, including the output statistics they leave behind."""
    g, cfg, ens_d, pm_d, pairs, frag_d = _device_run("box", "logit")
    _, _, ens_h, pm_h, _, frag_h = _device_run("box", "logit", use_device=False)
    frag_h.base_fragmenter = lambda **kw: pairs
    got_d, got_h = frag_d(pairs, L, NUM_PAIRS), frag_h(pairs, L, NUM_PAIRS)
    assert [id(p) for p in got_d] == [id(p) for p in got_h]
    assert pm_h._pool is None
    for md, mh in zip(ens_d.members, ens_h.members):
        a, b = md.normalize_output_layer, mh.normalize_output_layer
        np.testing.assert_allclose(a.running_mean.item(), b.running_mean.item(), rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(a.running_var.item(), b.running_var.item(), rtol=1e-6, atol=1e-6)
        assert int(a.count) == int(b.count)


@pytest.mark.gpu
def test_staging_table_is_reused_and_training_uploads_nothing():
    from imitation_b200.algorithms import preference_comparisons as pc

    g, cfg, ens, pm, pairs, frag = _device_run("box", "probability")
    chosen = frag(pairs, L, NUM_PAIRS)
    pool = pm._pool
    stage = pool._stage_table
    chosen2 = frag(pairs[::-1], L, NUM_PAIRS)
    assert pool._stage_table is stage  # same size: the staging table is reused
    ids = {id(p) for p in chosen}
    items = list(chosen) + [p for p in chosen2 if id(p) not in ids]
    ds = pc.PreferenceDataset()
    ds.push(items, np.full(len(items), 0.5, dtype=np.float32))
    n_slots, table = len(pool._slots), pool.table
    # as in the reference script, the trainer shares the fragmenter's PreferenceModel
    trainer = pc.EnsembleTrainer(pm, pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(0), batch_size=4, epochs=1)
    stored = {"n": 0}
    orig = pool._upload

    def counting_upload(*a, **k):
        stored["n"] += 1
        return orig(*a, **k)

    pool._upload = counting_upload
    trainer.train(ds)
    assert stored["n"] == 0 and len(pool._slots) == n_slots and pool.table is table


@pytest.mark.gpu
def test_later_calls_with_fewer_candidates_match_the_host_loop():
    """One PreferenceModel keeps its workspace across calls; the query schedule makes later calls smaller.  Every call
    must still fold the output statistics and score from this call's moments: each call's scores, selections and
    statistics equal the reference's per-pair host loop run on the same sequence of calls."""
    from imitation_b200.data import rollout

    g, cfg, ens_d, pm_d, pairs, frag_d = _device_run("box", "logit")
    _, _, ens_h, pm_h, _, frag_h = _device_run("box", "logit", use_device=False)

    def host_scores(cands):
        out = []
        for a, b in cands:
            with th.no_grad():
                r1 = pm_h.rewards(rollout.flatten_trajectories([a]))
                r2 = pm_h.rewards(rollout.flatten_trajectories([b]))
            out.append(frag_h.variance_estimate(r1, r2))
        return np.array(out)

    def check_stats():
        for md, mh in zip(ens_d.members, ens_h.members):
            a, b = md.normalize_output_layer, mh.normalize_output_layer
            np.testing.assert_allclose([a.running_mean.item(), a.running_var.item()],
                                       [b.running_mean.item(), b.running_var.item()], rtol=1e-6, atol=1e-6)
            assert int(a.count) == int(b.count)

    for cands, n in ((pairs, NUM_PAIRS), (pairs[3:15], 5), (pairs[15:19], 2)):
        sd, _ = pm_d.uncertainty_scores(cands, "logit")
        sh = host_scores(cands)
        np.testing.assert_allclose(sd.cpu().numpy(), sh, rtol=1e-5, atol=1e-6 * max(1.0, float(np.abs(sh).max())))
        check_stats()
        frag_d.base_fragmenter = frag_h.base_fragmenter = lambda **kw: cands
        got_d, got_h = frag_d(cands, L, n), frag_h(cands, L, n)
        assert [id(p) for p in got_d] == [id(p) for p in got_h]
        check_stats()


@pytest.mark.gpu
def test_preference_comparisons_runs_with_active_selection():
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    rng = np.random.default_rng(5)
    Do, Da = 6, 2
    trajs = [types.TrajectoryWithRew(obs=rng.standard_normal((51, Do)).astype(np.float32),
                                     acts=rng.uniform(-1, 1, (50, Da)).astype(np.float32), infos=None, terminal=True,
                                     rews=rng.standard_normal(50).astype(np.float32)) for _ in range(20)]
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1.0, 1.0, (Da,))
    th.manual_seed(0)
    ens = reward_nets.RewardEnsemble(obs_space, act_space, [
        reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs_space, act_space), networks.RunningNorm).cuda()
        for _ in range(3)])
    pm = pc.PreferenceModel(ens)
    frag = pc.ActiveSelectionFragmenter(pm, pc.RandomFragmenter(rng=np.random.default_rng(1), warning_threshold=0), 2.0)
    trainer = pc.EnsembleTrainer(pm, pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(2), batch_size=8, epochs=1)
    algo = pc.PreferenceComparisons(pc.TrajectoryDataset(trajs, np.random.default_rng(3)), ens, num_iterations=2,
                                    fragmenter=frag, preference_gatherer=pc.SyntheticGatherer(rng=np.random.default_rng(4)),
                                    reward_trainer=trainer, fragment_length=10, initial_epoch_multiplier=1.0)
    out = algo.train(total_timesteps=0, total_comparisons=24)
    assert len(algo.dataset) == 24
    assert np.isfinite(out["reward_loss"])
    assert len(pm._pool._slots) == 2 * len(algo.dataset)


# ------------------------------------------------------------------------------------------------
# GPU: the kernel against a float64 restatement
# ------------------------------------------------------------------------------------------------
def _restate(rews, norms, L, mode, noise, discount, threshold):
    """float64 restatement: rews [M][2C][L] raw; norms[m] = None or (mean, var, count, eps).  Returns scores [C],
    member values [C][M], final norms."""
    rews = rews.double()
    M, F, _ = rews.shape
    C = F // 2
    proc = rews.clone()
    final = []
    for m in range(M):
        if norms[m] is None:
            final.append(None)
            continue
        mean, var, cnt, eps = norms[m]
        for f in range(F):
            x = rews[m, f]
            proc[m, f] = (x - mean) / np.sqrt(var + eps)
            bm, bv = x.mean().item(), x.var(unbiased=False).item()
            tot = cnt + L
            delta = bm - mean
            mean = mean + delta * L / tot
            var = (var * cnt + bv * L + delta * delta * cnt * L / tot) / tot
            cnt = tot
        final.append((mean, var, cnt))
    r1, r2 = proc[:, 0::2], proc[:, 1::2]  # [M][C][L]
    if mode == 0:
        v = (r1.sum(2) - r2.sum(2)).T
        return v.var(1, unbiased=True), v, final
    w = discount ** th.arange(L, dtype=th.float64)
    s = ((r2 - r1) * w).sum(2).T
    p = noise * 0.5 + (1 - noise) / (1 + th.clip(s, -threshold, threshold).exp())
    if mode == 1:
        return p.var(1, unbiased=False), p, final
    q = (p > 0.5).float().mean(1)  # q (1 - q) in float32, as np.mean / np arithmetic on the float32 labels
    return q * (1 - q), p, final


def _kernel_call(rews, norms, L, mode, noise, discount, threshold, ws=None):
    from imitation_b200 import _lib

    M, F, _ = rews.shape
    C = F // 2
    flat = [rews[m].reshape(-1).contiguous() for m in range(M)]
    dn = []
    for nm in norms:
        if nm is None:
            dn.append(None)
        else:
            st = th.tensor([nm[0], nm[1]], dtype=th.float32, device="cuda")
            ct = th.tensor([nm[2]], dtype=th.int32, device="cuda")
            dn.append((st, ct, nm[3]))
    if ws is None:
        ws = th.zeros(_lib.pref_uncertainty_ws_floats(M, C), device="cuda")
    scores, member = th.empty(C, device="cuda"), th.empty(C, M, device="cuda")
    _lib.pref_uncertainty(_lib.pref_uncertainty_desc(flat, dn), C, L, mode, noise, discount, threshold, ws, scores,
                          member)
    return scores, member, dn, ws


@pytest.mark.gpu
@pytest.mark.parametrize("M", [2, 3, 5, 8, 16])
@pytest.mark.parametrize("Lk", [1, 31, 32, 100, 1000])
def test_kernel_matches_float64_restatement(M, Lk):
    gen = th.Generator().manual_seed(M * 1000 + Lk)
    C = 37
    rews = (th.randn(M, 2 * C, Lk, generator=gen) * 0.5 + 0.2)
    rews[:, 5] = rews[:, 4]  # pair 2: identical fragments
    mixed = [None if m % 2 else (0.1 * m, 0.5 + 0.1 * m, 7 * m, 1e-5) for m in range(M)]
    for norms in (mixed, [None] * M):
        for mode in range(3):
            for discount in (1.0, 0.9):
                threshold = 0.15 * np.sqrt(Lk)  # some pairs clip
                noise = 0.0 if mode == 2 else 0.1
                scores, member, dn, _ = _kernel_call(rews.cuda(), norms, Lk, mode, noise, discount, threshold)
                want, wv, final = _restate(rews, norms, Lk, mode, noise, discount, threshold)
                scores, member = scores.cpu(), member.cpu()
                if mode == 2:
                    edge = ((wv - 0.5).abs() < 1e-5).any(1)
                    if norms[0] is None:  # identical fragments of unnormalised members: p = 0.5 exactly, label 0
                        assert scores[2].item() == 0.0 and (member[2] == 0.5).all()
                        edge[2] = False
                    np.testing.assert_array_equal(scores.numpy()[~edge.numpy()], want.float().numpy()[~edge.numpy()])
                else:
                    tol = 1e-5 * max(1.0, float(wv.abs().max())) ** 2
                    np.testing.assert_allclose(scores.numpy(), want.numpy(), rtol=1e-4, atol=tol)
                    np.testing.assert_allclose(member.numpy(), wv.numpy(), rtol=1e-4,
                                               atol=1e-5 * max(1.0, float(wv.abs().max())))
                for m in range(M):
                    if norms[m] is not None:
                        st, ct, _ = dn[m]
                        np.testing.assert_allclose(st.cpu().numpy(), final[m][:2], rtol=2e-5, atol=1e-6)
                        assert int(ct.item()) == final[m][2]


@pytest.mark.gpu
def test_workspace_reused_by_a_smaller_call():
    """A workspace sized for a large call serves a later call with fewer members and candidates: that call folds and
    scores from its own moments (the float64 restatement), and a third call on it is bit-identical to a fresh one."""
    from imitation_b200 import _lib

    gen = th.Generator().manual_seed(11)
    Lk = 40
    big = th.randn(5, 2 * 50, Lk, generator=gen) * 1.5 + 0.5
    small = th.randn(3, 2 * 20, Lk, generator=gen) * 0.7 - 0.3
    ws = th.zeros(_lib.pref_uncertainty_ws_floats(5, 50), device="cuda")
    _kernel_call(big.cuda(), [(0.2, 1.1, 9, 1e-5)] * 5, Lk, 0, 0.0, 1.0, 50.0, ws=ws)
    norms = [(0.1, 0.9, 5, 1e-5), None, (-0.4, 2.0, 30, 1e-5)]
    for mode in range(3):
        scores, member, dn, _ = _kernel_call(small.cuda(), norms, Lk, mode, 0.1, 0.9, 3.0, ws=ws)
        want, wv, final = _restate(small, norms, Lk, mode, 0.1, 0.9, 3.0)
        if mode == 2:
            edge = ((wv - 0.5).abs() < 1e-5).any(1).numpy()
            np.testing.assert_array_equal(scores.cpu().numpy()[~edge], want.float().numpy()[~edge])
        else:
            np.testing.assert_allclose(scores.cpu().numpy(), want.numpy(), rtol=1e-4,
                                       atol=1e-5 * max(1.0, float(wv.abs().max())) ** 2)
        for m in (0, 2):
            np.testing.assert_allclose(dn[m][0].cpu().numpy(), final[m][:2], rtol=2e-5, atol=1e-6)
            assert int(dn[m][1].item()) == final[m][2]
        fresh = _kernel_call(small.cuda(), norms, Lk, mode, 0.1, 0.9, 3.0)
        assert th.equal(scores, fresh[0]) and th.equal(member, fresh[1])
    assert ws[0:1].view(th.int32).item() == 0  # the ticket is re-armed


@pytest.mark.gpu
def test_fold_matches_reward_norm_scan_and_calls_are_bit_identical():
    """The per-fragment output normalisation equals k_reward_norm_scan on a copy with E = L envs and T = 2C steps (one
    fragment per step); two calls on the same inputs give the same bits."""
    from imitation_b200 import _lib

    gen = th.Generator().manual_seed(3)
    M, C, Lk = 3, 500, 100
    rews = (th.randn(M, 2 * C, Lk, generator=gen) * 2.0 + 1.0).cuda()
    norms = [(0.3, 1.7, 40, 1e-5), None, (-0.2, 0.4, 3, 1e-5)]
    scores, member, dn, ws = _kernel_call(rews, norms, Lk, 0, 0.0, 1.0, 50.0)
    F = 2 * C
    aff = ws[1 + 2 * M * F:1 + 4 * M * F].reshape(M, F, 2)  # (word 0: the ticket; then the moments)
    for m in (0, 2):
        scan = rews[m].clone()  # [T = F][E = L]
        st = th.tensor(norms[m][:2], dtype=th.float32, device="cuda")
        ct = th.tensor([norms[m][2]], dtype=th.int32, device="cuda")
        _lib.reward_norm_scan(scan, Lk, F, Lk, 1, st, ct, norms[m][3], True)
        np.testing.assert_allclose(dn[m][0].cpu().numpy(), st.cpu().numpy(), rtol=1e-6, atol=1e-6)
        assert int(dn[m][1].item()) == int(ct.item())
        ours = (rews[m] - aff[m, :, 0:1]) * aff[m, :, 1:2]
        np.testing.assert_allclose(ours.cpu().numpy(), scan.cpu().numpy(), rtol=1e-6, atol=1e-6)
    s2, m2, _, _ = _kernel_call(rews, norms, Lk, 0, 0.0, 1.0, 50.0)
    assert th.equal(scores, s2) and th.equal(member, m2)
    for mode, disc in ((1, 0.9), (2, 1.0)):
        a = _kernel_call(rews, norms, Lk, mode, 0.1, disc, 5.0)
        b = _kernel_call(rews, norms, Lk, mode, 0.1, disc, 5.0)
        assert th.equal(a[0], b[0]) and th.equal(a[1], b[1])
