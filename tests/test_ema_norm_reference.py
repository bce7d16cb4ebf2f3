"""`EMANorm` as the output layer of `NormalizedRewardNet` (reference util/networks.py:137-201 and
rewards/reward_nets.py:613-671), pinned to the reference on the CPU.

- `networks.EMANorm` against the reference's own class, bit for bit (the same float32 torch ops on the same CPU), its
  `ValueError`s, and state dicts in both directions.
- tests/golden/ema_output_norm.npz holds what the reference's own wrappers record:
    shaped      Box, `RewardVecEnvWrapper(BufferingWrapper(venv), NormalizedRewardNet(BasicShapedRewardNet, EMANorm)
                .predict_processed)` with fresh statistics;
    disc09      Discrete, `partial(EMANorm, decay=0.9)` from num_batches = 150 (decay^n ~ 1e-7: inv_learning_rate has
                almost reached 1 / (1 - decay));
    disc05      Discrete, `partial(EMANorm, decay=0.5)` from num_batches = 160 (decay^n underflows to 0 in float32);
    ensemble    Box, `AddSTDRewardWrapper(RewardEnsemble(5 x NormalizedRewardNet(BasicRewardNet, EMANorm)), -0.5)`;
    active      `ActiveSelectionFragmenter` over 3 `NormalizedRewardNet(BasicRewardNet, EMANorm)` members in the three
                modes: scores, per-member values, selections and output statistics before and after.
  Re-record it where the reference sources are importable (oracle/refimport.py) with

      IMB_RECORD_REFERENCE=1 python -m pytest tests/test_ema_norm_reference.py -k reference_records

  Where they are importable, the same test regenerates the results and compares them with the stored file.
- `EMANormPort` below is the CPU restatement, used as the `norm` of an `oracle.nets_port.OutputNormPort`; it is held
  to the stored file here, and tests/test_ema_norm.py holds the device paths to it.
"""
import contextlib
import functools
import os

import numpy as np
import pytest
import torch as th
from torch import nn

from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "ema_output_norm.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
E, T, H = 6, 9, 4
# name: (d_obs, n_actions | None, d_act (one-hot width), members (0 = a single net), shaped, decay, start num_batches,
#        alpha | None)
ROLLOUTS = {
    "shaped": (11, None, 3, 0, True, 0.99, 0, None),
    "disc09": (4, 3, 3, 0, False, 0.9, 150, None),
    "disc05": (4, 3, 3, 0, False, 0.5, 160, None),
    "ensemble": (11, None, 3, 5, False, 0.99, 3, -0.5),
}
# the active-selection case in test_active_selection's vocabulary: 3 EMA-normalised members on a Box task
ACTIVE = (11, None, 3, 3, (32, 32), True, False, 2.0)
ACTIVE_DECAY = 0.9


class EMANormPort(nn.Module):
    """EMANorm restated: normalise with the statistics as they stand; update_stats folds one batch with learning rate
    1 / inv_learning_rate after inv_learning_rate += decay ** num_batches, one float32 op per line."""

    def __init__(self, n: int = 1, decay: float = 0.99, eps: float = 1e-5):
        super().__init__()
        self.decay, self.eps = decay, eps
        self.register_buffer("running_mean", th.zeros(n))
        self.register_buffer("running_var", th.ones(n))
        self.register_buffer("count", th.zeros((), dtype=th.int))
        self.register_buffer("inv_learning_rate", th.zeros(()))
        self.register_buffer("num_batches", th.zeros((), dtype=th.int))

    @th.no_grad()
    def update_stats(self, batch: th.Tensor) -> None:
        if batch.ndim == 1:
            batch = batch[:, None]
        w = th.pow(self.decay, self.num_batches)
        self.inv_learning_rate += w
        lr = 1 / self.inv_learning_rate
        dm = batch.mean(0) - self.running_mean
        self.running_mean += lr * dm
        self.running_var += lr * (batch.var(0, unbiased=False) + (1 - lr) * dm * dm - self.running_var)
        self.count += batch.shape[0]
        self.num_batches += 1

    def forward(self, x):
        if self.training:
            self.update_stats(x)
        return (x - self.running_mean) / th.sqrt(self.running_var + self.eps)


def ema_output_port(decay, state=None):
    """NormalizedRewardNet.predict_processed with an output EMANorm: OutputNormPort whose norm is an EMANormPort,
    optionally loaded from a state dict {running_mean, running_var, count, inv_learning_rate, num_batches}."""
    from oracle import nets_port

    out = nets_port.OutputNormPort()
    out.norm = EMANormPort(1, decay).eval()
    if state is not None:
        out.norm.load_state_dict({k: th.as_tensor(np.array(v)) for k, v in state.items()})
    return out


def _out_state(st, prefix="normalize_output_layer."):
    return {k[len(prefix):]: v for k, v in st.items() if k.startswith(prefix)}


# ------------------------------------------------------------------------------------------------
# EMANorm against the reference's class
# ------------------------------------------------------------------------------------------------
def _reference_available() -> bool:
    from oracle import refimport

    return refimport.available()


def _batches(seed, n=400):
    g = th.Generator().manual_seed(seed)
    return [th.randn(int(th.randint(1, 40, (1,), generator=g)), generator=g) * 3 + 1 for _ in range(n)]


def test_ema_norm_matches_port_bit_for_bit():
    from imitation_b200.util import networks

    for decay in (0.5, 0.9, 0.99, 0.999):
        a, b = networks.EMANorm(1, decay=decay), EMANormPort(1, decay=decay)
        for x in _batches(int(decay * 1000)):
            a.update_stats(x)
            b.update_stats(x)
        assert set(a.state_dict()) == set(b.state_dict())
        for k, v in a.state_dict().items():
            assert th.equal(v, b.state_dict()[k]), (decay, k)


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_ema_norm_matches_reference_bit_for_bit():
    from oracle import refimport

    refimport.load()
    from imitation.util import networks as ref_networks

    from imitation_b200.util import networks

    for decay, nf in ((0.5, 1), (0.99, 1), (0.999, 3)):
        a, b = ref_networks.EMANorm(nf, decay=decay), networks.EMANorm(nf, decay=decay)
        for x in _batches(nf + int(decay * 1000), 300):
            x = x.reshape(-1, 1).expand(-1, nf) * th.arange(1, nf + 1) if nf > 1 else x
            a.update_stats(x)
            b.update_stats(x)
            a.train(), b.train()
            assert th.equal(a(x), b(x))  # train mode: update, then normalise with the updated statistics
        for k, v in a.state_dict().items():
            assert th.equal(v, b.state_dict()[k]), (decay, k)
        # state dicts load both ways
        c, d = networks.EMANorm(nf, decay=decay), ref_networks.EMANorm(nf, decay=decay)
        c.load_state_dict(a.state_dict())
        d.load_state_dict(b.state_dict())
        assert all(th.equal(v, c.state_dict()[k]) and th.equal(v, d.state_dict()[k]) for k, v in a.state_dict().items())


def test_ema_norm_errors_buffers_and_reset():
    from imitation_b200.util import networks

    for bad in (0.0, 1.0, -0.1, 1.5):
        with pytest.raises(ValueError, match="decay must be between 0 and 1"):
            networks.EMANorm(1, decay=bad)
    n = networks.EMANorm(4, decay=0.9, eps=1e-3)
    want = {"running_mean": ((4,), th.float32), "running_var": ((4,), th.float32), "count": ((), th.int32),
            "inv_learning_rate": ((), th.float32), "num_batches": ((), th.int32)}
    assert {k: (tuple(v.shape), v.dtype) for k, v in n.state_dict().items()} == want
    assert isinstance(n, networks.BaseNorm) and n.decay == 0.9 and n.eps == 1e-3
    n.update_stats(th.randn(5, 4))
    assert int(n.num_batches) == 1 and int(n.count) == 5 and float(n.inv_learning_rate) == 1.0
    n.reset_running_stats()
    assert int(n.num_batches) == 0 and int(n.count) == 0 and float(n.inv_learning_rate) == 0.0
    assert (n.running_mean == 0).all() and (n.running_var == 1).all()


def test_normalized_reward_net_output_layers():
    """The classes and partials NormalizedRewardNet takes, and what it still refuses."""
    from imitation_b200 import spaces
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    obs, act = spaces.Box(-1, 1, (3,)), spaces.Box(-1, 1, (2,))
    for layer, decay, eps in ((networks.EMANorm, 0.99, 1e-5), (functools.partial(networks.EMANorm, decay=0.9), 0.9, 1e-5),
                              (functools.partial(networks.EMANorm, decay=0.5, eps=1e-3), 0.5, 1e-3)):
        net = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs, act), layer)
        n = net.normalize_output_layer
        assert isinstance(n, networks.EMANorm) and net.output_norm_is_ema
        assert (n.decay, n.eps, n.num_features) == (decay, eps, 1)
    net = reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs, act), networks.RunningNorm)
    assert type(net.normalize_output_layer) is networks.RunningNorm and not net.output_norm_is_ema
    with pytest.raises(ValueError, match="decay must be between 0 and 1"):
        reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs, act), functools.partial(networks.EMANorm,
                                                                                                 decay=1.0))
    with pytest.raises(NotImplementedError, match="RunningNorm or EMANorm"):
        reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs, act), nn.BatchNorm1d)
    # input normalisation stays RunningNorm-only
    with pytest.raises(NotImplementedError, match="normalize_input_layer must be RunningNorm or None"):
        reward_nets.BasicRewardNet(obs, act, normalize_input_layer=networks.EMANorm)


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_reference_ema_class_and_state_dict_are_accepted():
    """The reference's EMANorm class (and a partial of it) builds this package's layer; state dicts of the reference's
    NormalizedRewardNet load into this package's module and back."""
    from oracle import refimport

    refimport.load()
    from gymnasium import spaces as ref_spaces
    from imitation.rewards import reward_nets as ref_nets
    from imitation.util import networks as ref_networks

    from imitation_b200 import spaces
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    th.manual_seed(0)
    ref = ref_nets.NormalizedRewardNet(ref_nets.BasicShapedRewardNet(ref_spaces.Box(-1, 1, (5,)),
                                                                     ref_spaces.Box(-1, 1, (2,))),
                                       functools.partial(ref_networks.EMANorm, decay=0.95))
    for x in _batches(3, 20):
        ref.normalize_output_layer.update_stats(x)
    ours = reward_nets.NormalizedRewardNet(reward_nets.BasicShapedRewardNet(spaces.Box(-1, 1, (5,)),
                                                                            spaces.Box(-1, 1, (2,))),
                                           functools.partial(ref_networks.EMANorm, decay=0.95))
    assert isinstance(ours.normalize_output_layer, networks.EMANorm) and ours.normalize_output_layer.decay == 0.95
    sd = ref.state_dict()
    assert set(sd) == set(ours.state_dict())
    ours.load_state_dict(sd)
    back = ref_nets.NormalizedRewardNet(ref_nets.BasicShapedRewardNet(ref_spaces.Box(-1, 1, (5,)),
                                                                      ref_spaces.Box(-1, 1, (2,))),
                                        functools.partial(ref_networks.EMANorm, decay=0.95))
    back.load_state_dict(ours.state_dict())
    for k, v in sd.items():
        assert th.equal(v, ours.state_dict()[k].cpu()) and th.equal(v, back.state_dict()[k]), k


# ------------------------------------------------------------------------------------------------
# recording (reference only)
# ------------------------------------------------------------------------------------------------
def _record_rollout(name, cfg, seed):
    from oracle import refimport, synth_env

    refimport.load()
    from gymnasium import spaces
    from imitation.data import wrappers as ref_wrappers
    from imitation.rewards import reward_nets as ref_nets
    from imitation.rewards import reward_wrapper as ref_rw
    from imitation.util import networks as ref_networks
    from stable_baselines3.common.vec_env import VecEnv

    class HostVenv(VecEnv):
        def __init__(self, inner):
            super().__init__(inner.num_envs, inner.observation_space, inner.action_space)
            self.inner = inner

        def reset(self):
            return self.inner.reset()

        def step_async(self, a):
            self.inner.step_async(a)

        def step_wait(self):
            return self.inner.step_wait()

    Do, n_act, Da, M, shaped, decay, nb0, alpha = cfg
    rng = np.random.default_rng(seed)
    th.manual_seed(seed)
    spec = synth_env.SynthEnvSpec(Do, n_act or Da, discrete=n_act is not None, horizon=H, seed=seed)
    venv = HostVenv(synth_env.SynthVecEnv(spec, E, spaces_mod=spaces))
    obs_space, act_space = venv.observation_space, venv.action_space
    layer = ref_networks.EMANorm if decay == 0.99 else functools.partial(ref_networks.EMANorm, decay=decay)
    nets = []
    for _ in range(max(M, 1)):
        base = (ref_nets.BasicShapedRewardNet if shaped else ref_nets.BasicRewardNet)(obs_space, act_space)
        net = ref_nets.NormalizedRewardNet(base, layer)
        for k in range(nb0):  # advance the output statistics to num_batches = nb0
            n = 5 + k % 7
            net.predict_processed(rng.standard_normal((n, Do)).astype(np.float32),
                                  (rng.integers(0, n_act, n) if n_act else rng.uniform(-1, 1, (n, Da)).astype(np.float32)),
                                  rng.standard_normal((n, Do)).astype(np.float32), np.zeros(n, dtype=bool))
        assert int(net.normalize_output_layer.num_batches) == nb0
        nets.append(net)
    if M:
        reward = ref_nets.AddSTDRewardWrapper(ref_nets.RewardEnsemble(obs_space, act_space, nets), default_alpha=alpha)
    else:
        reward = nets[0]
    out = {}
    for k, m in enumerate(nets):
        out.update({f"member{k}/{key}": v.detach().numpy().copy() for key, v in m.state_dict().items()})
    wrapped = ref_rw.RewardVecEnvWrapper(ref_wrappers.BufferingWrapper(venv), reward.predict_processed)
    acts, rews, obs_l, dones_l = [], [], [], []
    for _ in range(T):
        a = (rng.integers(0, n_act, E) if n_act else rng.uniform(-1.2, 1.2, (E, Da)).astype(np.float32))
        o, r, d, _infos = wrapped.step(a)
        acts.append(a), rews.append(r), obs_l.append(o), dones_l.append(d)
    assert np.stack(dones_l).any(), "no episode ended: lower the horizon"
    out.update(acts=np.stack(acts), rews=np.stack(rews), obs=np.stack(obs_l), dones=np.stack(dones_l))
    for k, m in enumerate(nets):
        out.update({f"member_after{k}/{key}": v.detach().numpy().copy() for key, v in m.state_dict().items()})
    return {f"{name}/{k}": v for k, v in out.items()}


@contextlib.contextmanager
def _reference_output_norm_is_ema():
    """test_active_selection's recorder builds its output layers as `ref_networks.RunningNorm` (its active config has no
    input norm): for the recording, that name is the reference's partial(EMANorm, decay=ACTIVE_DECAY)."""
    from imitation.util import networks as ref_networks

    old = ref_networks.RunningNorm
    ref_networks.RunningNorm = functools.partial(ref_networks.EMANorm, decay=ACTIVE_DECAY)
    try:
        yield
    finally:
        ref_networks.RunningNorm = old


def _record_active(seed):
    from oracle import refimport

    from tests import test_active_selection as tas

    refimport.load()
    from imitation.algorithms import preference_comparisons as ref_pc

    assert not ACTIVE[6]  # no input norm: the renamed class reaches the output layers only
    ema_states = {}
    orig = ref_pc.ActiveSelectionFragmenter.__call__

    def call(self, *a, **kw):  # the members' EMA buffers after each mode (the recorder keeps mean, var and count)
        r = orig(self, *a, **kw)
        for k, m in enumerate(self.preference_model.ensemble_model.members):
            ema_states[(self.uncertainty_on, k)] = (float(m.normalize_output_layer.inv_learning_rate),
                                                    int(m.normalize_output_layer.num_batches))
        return r

    with _reference_output_norm_is_ema():
        ref_pc.ActiveSelectionFragmenter.__call__ = call
        try:
            out = tas._record_config("active", ACTIVE, seed)
        finally:
            ref_pc.ActiveSelectionFragmenter.__call__ = orig
    for (mode, k), (ilr, nb) in ema_states.items():
        out[f"active/{mode}/out_ema{k}"] = np.array(ilr, np.float32)
        out[f"active/{mode}/out_batches{k}"] = np.array(nb)
    return out


def _record_all():
    rng_state = th.get_rng_state()
    try:
        out = {}
        for i, (name, cfg) in enumerate(ROLLOUTS.items()):
            out.update(_record_rollout(name, cfg, 61 + 10 * i))
        out.update(_record_active(97))
        return out
    finally:
        th.set_rng_state(rng_state)


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_golden_is_what_the_reference_records():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead).
    Observations, actions, dones, counts and selections must be identical; floats may differ in the last bits on
    another CPU."""
    out = _record_all()
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = G.load("ema_output_norm")
    assert set(z.files) == set(out)
    for k, v in out.items():
        if np.issubdtype(np.asarray(v).dtype, np.floating) and not k.endswith(("/obs", "/acts")):
            np.testing.assert_allclose(v, z[k], rtol=1e-6, atol=1e-7, err_msg=k)
        else:
            np.testing.assert_array_equal(v, z[k], err_msg=k)


# ------------------------------------------------------------------------------------------------
# the CPU restatement against the stored file
# ------------------------------------------------------------------------------------------------
def port_rollout_members(z, name, prefix="member"):
    """(net port, EMA output port) per member of rollout case `name`, from the stored states under `prefix`."""
    from oracle import nets_port

    Do, n_act, Da, M, shaped, decay, _, _ = ROLLOUTS[name]
    members = []
    for k in range(max(M, 1)):
        st = G.sub(z, f"{name}/{prefix}{k}")
        if shaped:
            net = nets_port.ShapedRewardNetPort(Do, Da)
            sd = {G.port_key(kk[len("_base."):]): v for kk, v in st.items() if kk.startswith("_base.")}
        else:
            net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=(32, 32))
            sd = {kk[len("_base."):]: v for kk, v in st.items() if kk.startswith("_base.")}
        net.load_state_dict({kk: th.as_tensor(np.array(v)) for kk, v in sd.items()})
        net.eval()
        members.append((net, ema_output_port(decay, _out_state(st))))
    return members


def rollout_reward_port(name, members):
    """reward_fn of case `name` over port members: the single net's predict_processed, or the ensemble's."""
    from oracle import nets_port

    from tests.test_ensemble_relabel_reference import ensemble_relabel_port

    Do, n_act, Da, M, shaped, decay, _, alpha = ROLLOUTS[name]
    if M:
        return ensemble_relabel_port(members, alpha, n_act)
    net, out = members[0]
    return lambda obs, acts, next_obs, dones: out(nets_port.predict_port(net, obs, acts, next_obs, dones, n_act))


def _assert_norm_close(got: dict, want: dict, vscale: float):
    np.testing.assert_allclose(got["running_mean"], want["running_mean"], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(got["running_var"], want["running_var"], rtol=1e-6, atol=1e-6 * vscale)
    np.testing.assert_allclose(got["inv_learning_rate"], want["inv_learning_rate"], rtol=1e-6)
    assert int(got["count"]) == int(want["count"]) and int(got["num_batches"]) == int(want["num_batches"])


@pytest.mark.parametrize("name", list(ROLLOUTS))
def test_port_matches_reference_golden(name):
    from oracle import data_port, synth_env

    Do, n_act, Da, M, shaped, decay, nb0, alpha = ROLLOUTS[name]
    z = G.load("ema_output_norm")
    seed = 61 + 10 * list(ROLLOUTS).index(name)
    members = port_rollout_members(z, name)
    spec = synth_env.SynthEnvSpec(Do, n_act or Da, discrete=n_act is not None, horizon=H, seed=seed)
    wrapped = data_port.RewardRelabelPort(data_port.BufferingPort(synth_env.SynthVecEnv(spec, E)),
                                          rollout_reward_port(name, members))
    assert z[f"{name}/dones"].any() and not z[f"{name}/dones"].all()
    for t in range(T):
        o, r, d, _infos = wrapped.step(z[f"{name}/acts"][t])
        np.testing.assert_array_equal(d, z[f"{name}/dones"][t])
        np.testing.assert_array_equal(o, z[f"{name}/obs"][t])
        np.testing.assert_allclose(r, z[f"{name}/rews"][t], rtol=2e-6, atol=2e-6, err_msg=f"rewards of step {t}")
    for k, (_, out) in enumerate(members):
        want = _out_state(G.sub(z, f"{name}/member_after{k}"))
        before = _out_state(G.sub(z, f"{name}/member{k}"))
        got = {kk: v.numpy() for kk, v in out.norm.state_dict().items()}
        _assert_norm_close(got, want, float(np.max(want["running_var"])))
        assert int(want["num_batches"]) == int(before["num_batches"]) + T == nb0 + T
        assert int(want["count"]) == int(before["count"]) + E * T
    if name == "disc09":  # decay^150 ~ 1.4e-7: inv_learning_rate has almost saturated at 1 / (1 - decay)
        assert abs(float(want["inv_learning_rate"]) - 10.0) < 1e-5
    if name == "disc05":  # decay^160 underflows: inv_learning_rate no longer moves
        assert float(want["inv_learning_rate"]) == float(before["inv_learning_rate"]) == 2.0


def active_golden():
    from tests import test_active_selection as tas

    z = G.load("ema_output_norm")
    g = {k[len("active/"):]: z[k] for k in z.files if k.startswith("active/")}
    n = 0
    while f"cand{n}/a/obs" in g:
        n += 1
    cands = [tuple(dict(obs=g[f"cand{i}/{s}/obs"], acts=g[f"cand{i}/{s}/acts"], rews=g[f"cand{i}/{s}/rews"],
                        terminal=bool(g[f"cand{i}/{s}/terminal"])) for s in ("a", "b")) for i in range(n)]
    return g, cands, tas


def active_port_members(g):
    from oracle import nets_port

    Do, n_act, Da, M, hid, _, _, _ = ACTIVE
    members = []
    for k in range(M):
        st = {kk[len(f"member{k}/"):]: v for kk, v in g.items() if kk.startswith(f"member{k}/")}
        net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=hid)
        net.load_state_dict({kk[len("_base."):]: th.as_tensor(np.array(v)) for kk, v in st.items()
                             if kk.startswith("_base.")})
        members.append((net, ema_output_port(ACTIVE_DECAY, _out_state(st))))
    return members


def check_selection(g, mode, scores, sel):
    """`sel` is the stable rule on `scores` exactly, and the reference's selection up to the order of equal scores
    (clipped pairs tie in the probability mode, and the reference's unstable argsort orders ties arbitrarily)."""
    from tests import test_active_selection as tas

    np.testing.assert_array_equal(sel, np.argsort(scores, kind="stable")[::-1][:tas.NUM_PAIRS])
    ref = g[f"{mode}/scores"]
    rtol, atol = tas._score_tol(g, mode)
    np.testing.assert_allclose(np.sort(ref[sel]), np.sort(ref[g[f"{mode}/selected"]]), rtol=rtol, atol=atol)


@pytest.mark.parametrize("mode", ("logit", "probability", "label"))
def test_active_selection_port_matches_reference_golden(mode):
    g, cands, tas = active_golden()
    members = active_port_members(g)
    nb0 = [int(out.norm.num_batches) for _, out in members]
    sel, scores, diffs, probs = tas.active_selection_port(members, cands, mode, tas.NUM_PAIRS, tas.NOISE, tas.DISCOUNT,
                                                          ACTIVE[-1])
    assert len(cands) == tas.FACTOR * tas.NUM_PAIRS
    tas._check_scores(g, mode, scores, diffs, probs)
    check_selection(g, mode, scores, sel)
    for k, (_, out) in enumerate(members):
        n = out.norm
        np.testing.assert_allclose([n.running_mean.item(), n.running_var.item()], g[f"{mode}/out_stats{k}"],
                                   rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(float(n.inv_learning_rate), g[f"{mode}/out_ema{k}"], rtol=1e-6)
        assert int(n.count) == int(g[f"{mode}/out_count{k}"])
        assert int(n.num_batches) == int(g[f"{mode}/out_batches{k}"]) == nb0[k] + 2 * len(cands)
