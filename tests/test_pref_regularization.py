"""Regularized reward training in preference comparisons: `imitation_b200.regularization` (LpRegularizer,
WeightDecayRegularizer, IntervalParamScaler) in `BasicRewardTrainer` / `EnsembleTrainer`, on the device-only step
(`imb_param_regularize`) and on the autograd path.

- tests/golden/pref_regularization.npz holds what the reference's own trainer does on the CPU for every case in CASES:
  initial and final state dicts (RunningNorm buffers included), lambda after every epoch, the val / train loss ratio
  the updater saw, every key and value its logger holds, and numpy's and torch's random states after the call.
  Re-record it where the reference sources are importable (oracle/refimport.py) with

      IMB_RECORD_REFERENCE=1 python -m pytest tests/test_pref_regularization.py -k reference_records

  Where they are importable, the same test regenerates the results and compares them with the stored file.
- CPU: the package against the reference's classes (errors, the updater on a grid), the CPU restatement
  (oracle/pref_regularization_port.py) against the golden, and the draws a rank makes for members it does not train.
- GPU: the kernel against float64 autograd and torch's weight decay, the device step against the autograd path and
  both against the golden.
"""
import os

import numpy as np
import pytest
import torch as th

from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "pref_regularization.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
DO, DA, L = 6, 2, 5
BASE = dict(batch_size=4, minibatch_size=2, epochs=3, lr=2e-3, lam=0.1, noise_prob=0.05, discount_factor=0.97, n=24)
# name: kind ("lp" / "wd"), p, updater (scaling factor, interval) | None, val_split, net ("basic" / "shaped"), members
# (0 = a single net), and overrides of BASE
CASES = {
    "lp2_falls": ("lp", 2, (0.1, (1.1, 1.5)), 0.2, "basic", 0, {}),
    "lp1_rises": ("lp", 1, (0.2, (0.1, 0.3)), 0.25, "basic", 0, {}),
    "lp3_fixed": ("lp", 3, None, None, "basic", 0, {}),
    "wd_fixed": ("wd", 0, None, None, "basic", 0, dict(batch_size=6, minibatch_size=3, n=20, lam=0.5)),
    "wd_updater": ("wd", 0, (0.2, (0.1, 0.3)), 0.2, "basic", 0, dict(lam=0.2)),
    "norm": ("lp", 2, (0.1, (1.1, 1.5)), 0.2, "norm", 0, {}),
    "shaped_norm": ("lp", 2, (0.1, (1.1, 1.5)), 0.2, "shaped", 0, {}),
    "ensemble": ("lp", 2, (0.1, (1.1, 1.5)), 0.2, "basic", 3, {}),
}
IGNORED_KEYS = ("reward/final/train/gt_reward_loss",)  # not recorded by this package's trainers (a known difference)
# Nets with an input RunningNorm train to other weights than the reference's on the device, with or without a
# regularizer: the reference evaluates a minibatch fragment by fragment, so each fragment is normalised with statistics
# that include it and the fragments before it, while the device evaluates the minibatch as one batch after one update.
# Their weights are held to the CPU restatement; on the device, their RunningNorm counts (training and validation rows)
# and lambdas are held to the golden.
CPU_ONLY = ("norm", "shaped_norm")
GPU_CASES = [n for n in sorted(CASES) if n not in CPU_ONLY]


def _cfg(name):
    kind, p, upd, val_split, net, members, over = CASES[name]
    return dict(BASE, **over, kind=kind, p=p, updater=upd, val_split=val_split, net=net, members=members)


def _data(name, types_mod):
    """The case's fragment pairs (TrajectoryWithRew of `types_mod`) and float32 preferences."""
    c = _cfg(name)
    rng = np.random.default_rng(sorted(CASES).index(name) + 100)

    def frag():
        return types_mod.TrajectoryWithRew(obs=rng.standard_normal((L + 1, DO)).astype(np.float32),
                                           acts=rng.uniform(-1, 1, (L, DA)).astype(np.float32), infos=None,
                                           terminal=False, rews=rng.standard_normal(L).astype(np.float32))

    pairs = [(frag(), frag()) for _ in range(c["n"])]
    return pairs, (rng.random(c["n"]) < 0.5).astype(np.float32)


def _fingerprint(rng):
    return rng.integers(0, 1 << 62, 4)


def _build(name, nets_mod, networks_mod, obs_space, act_space):
    c = _cfg(name)
    if c["net"] == "shaped":
        mk = lambda: nets_mod.BasicShapedRewardNet(obs_space, act_space, reward_hid_sizes=(32,),
                                                   potential_hid_sizes=(32, 32),
                                                   normalize_input_layer=networks_mod.RunningNorm)
    elif c["net"] == "norm":
        mk = lambda: nets_mod.BasicRewardNet(obs_space, act_space, hid_sizes=(32, 32),
                                             normalize_input_layer=networks_mod.RunningNorm)
    else:
        mk = lambda: nets_mod.BasicRewardNet(obs_space, act_space, hid_sizes=(32, 32))
    if c["members"]:
        members = [mk() for _ in range(c["members"])]
        return members, nets_mod.RewardEnsemble(obs_space, act_space, members)
    net = mk()
    return [net], net


def _run(name, pc, regs, upds, nets_mod, networks_mod, types_mod, logger_mod, spaces_mod, device="cpu", init=None,
         fused=True):
    """Train the case with one package's classes -> (member nets, trainer, logger, lambdas, ratios, rng)."""
    c = _cfg(name)
    th.manual_seed(sorted(CASES).index(name))
    members, model = _build(name, nets_mod, networks_mod, spaces_mod.Box(-np.inf, np.inf, (DO,), np.float32),
                            spaces_mod.Box(-1.0, 1.0, (DA,), np.float32))
    if init is not None:
        for i, m in enumerate(members):
            m.load_state_dict({k: th.as_tensor(v) for k, v in init[i].items()})
    members = [m.to(device) for m in members]
    model = model.to(device) if c["members"] else members[0]
    lambdas, ratios = [], []

    class Recording(upds.IntervalParamScaler):
        def __call__(self, lambda_, train_loss, val_loss):
            out = super().__call__(lambda_, train_loss, val_loss)
            lambdas.append(out)
            ratios.append(float(val_loss) / float(train_loss))
            return out

    upd = None if c["updater"] is None else Recording(c["updater"][0], c["updater"][1])
    cls = regs.LpRegularizer if c["kind"] == "lp" else regs.WeightDecayRegularizer
    kw = dict(p=c["p"]) if c["kind"] == "lp" else {}
    factory = cls.create(c["lam"], lambda_updater=upd, val_split=c["val_split"], **kw)
    logger = logger_mod.configure(None, ()) if logger_mod.__name__.startswith("imitation_b200") else \
        logger_mod.configure(os.path.join(os.environ.get("TMPDIR", "/tmp"), "imb_reg_ref_log"), ())
    rng = np.random.default_rng(7)
    pm = pc.PreferenceModel(model, noise_prob=c["noise_prob"], discount_factor=c["discount_factor"])
    args = dict(rng=rng, batch_size=c["batch_size"], minibatch_size=c["minibatch_size"], epochs=c["epochs"], lr=c["lr"],
                custom_logger=logger, regularizer_factory=factory)
    trainer = (pc.EnsembleTrainer if c["members"] else pc.BasicRewardTrainer)(pm, pc.CrossEntropyRewardLoss(), **args)
    for t in getattr(trainer, "member_trainers", [trainer]):
        t.use_fused_step = fused
    pairs, prefs = _data(name, types_mod)
    ds = pc.PreferenceDataset()
    ds.push(pairs, prefs)
    th.manual_seed(11)
    trainer.train(ds)
    return members, trainer, logger, lambdas, ratios, rng


def _reference_available():
    from oracle import refimport

    return refimport.available()


def _record_case(name):
    import gymnasium.spaces as shim_spaces
    from imitation.algorithms import preference_comparisons as ref_pc
    from imitation.data import types as ref_types
    from imitation.regularization import regularizers as ref_regs, updaters as ref_upds
    from imitation.rewards import reward_nets as ref_nets
    from imitation.util import logger as ref_logger, networks as ref_networks

    c = _cfg(name)
    th.manual_seed(sorted(CASES).index(name))
    members, _ = _build(name, ref_nets, ref_networks, shim_spaces.Box(-np.inf, np.inf, (DO,), np.float32),
                        shim_spaces.Box(-1.0, 1.0, (DA,), np.float32))
    init = [{k: v.detach().clone().numpy() for k, v in m.state_dict().items()} for m in members]
    members, trainer, logger, lambdas, ratios, rng = _run(name, ref_pc, ref_regs, ref_upds, ref_nets, ref_networks,
                                                          ref_types, ref_logger, shim_spaces, init=init)
    if c["updater"] is not None:  # no lambda decision may hinge on rounding
        lo, hi = c["updater"][1]
        for r in ratios:
            assert min(abs(r - lo) / max(lo, 1e-12), abs(r - hi) / hi) > 0.01, (name, r)
    keys = sorted(k for k in logger.name_to_value if not k.startswith("raw/"))
    out = {f"{name}/lambdas": np.array(lambdas, np.float64), f"{name}/ratios": np.array(ratios, np.float64),
           f"{name}/log_keys": np.array(keys), f"{name}/log_vals": np.array([float(logger.name_to_value[k]) for k in keys]),
           f"{name}/np_after": _fingerprint(rng), f"{name}/th_after": th.get_rng_state().numpy()}
    for i, (m, st) in enumerate(zip(members, init)):
        for k, v in st.items():
            out[f"{name}/init{i}/{k}"] = v
        for k, v in m.state_dict().items():
            out[f"{name}/final{i}/{k}"] = v.detach().numpy()
    return out


def _golden_states(z, name, which):
    out, i = [], 0
    while any(k.startswith(f"{name}/{which}{i}/") for k in z.files):
        out.append(G.sub(z, f"{name}/{which}{i}"))
        i += 1
    return out


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_reference_records_the_golden():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead)."""
    from oracle import refimport

    refimport.load()
    out = {}
    for name in CASES:
        out.update(_record_case(name))
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = np.load(STORE)
    assert sorted(z.files) == sorted(out)
    for k, v in out.items():
        if k.endswith("/log_keys"):
            assert list(z[k]) == list(v), k
        else:
            np.testing.assert_array_equal(z[k], v, err_msg=k)


# ---------------------------------------------------------------------------------------------------------------------
# the package against the reference's classes (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _both():
    from oracle import refimport

    refimport.load()
    from imitation.regularization import regularizers as ref_regs, updaters as ref_upds
    from imitation.util import logger as ref_logger

    from imitation_b200.regularization import regularizers, updaters
    from imitation_b200.util import logger

    return ((ref_regs, ref_upds, ref_logger.configure(os.path.join(os.environ.get("TMPDIR", "/tmp"), "imb_reg_err"),
                                                      ())),
            (regularizers, updaters, logger.configure()))


def _outcome(fn):
    try:
        return ("ok", fn())
    except ValueError as e:
        return ("ValueError", str(e))


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_errors_and_updater_match_the_reference():
    (rr, ru, rlog), (mr, mu, mlog) = _both()
    opt = th.optim.SGD([th.nn.Parameter(th.ones(3))], lr=0.1)
    ctor_cases = [  # (class name, initial_lambda, updater?, val_split, extra kwargs)
        ("LpRegularizer", 0.1, False, 0.0, dict(p=2)), ("LpRegularizer", 0.1, False, None, dict(p=2)),
        ("LpRegularizer", 0.0, False, None, dict(p=2)), ("LpRegularizer", 0.0, True, 0.2, dict(p=2)),
        ("LpRegularizer", 0.1, True, None, dict(p=2)), ("LpRegularizer", 0.1, False, 0.2, dict(p=2)),
        ("LpRegularizer", 0.1, True, 1.0, dict(p=2)), ("LpRegularizer", 0.1, True, 1, dict(p=2)),
        ("LpRegularizer", 0.1, True, -0.5, dict(p=2)), ("LpRegularizer", 0.1, False, None, dict(p=0)),
        ("LpRegularizer", 0.1, False, None, dict(p=2.0)), ("LpRegularizer", 0.1, True, 0.5, dict(p=3)),
        ("WeightDecayRegularizer", 0.1, False, None, {}), ("WeightDecayRegularizer", 0.1, False, 0.0, {}),
        ("WeightDecayRegularizer", 0.1, True, 0.3, {}),
    ]
    for cls, lam, with_upd, vs, kw in ctor_cases:
        got = []
        for regs, upds, log in ((rr, ru, rlog), (mr, mu, mlog)):
            upd = upds.IntervalParamScaler(0.1, (1.0, 2.0)) if with_upd else None
            res = _outcome(lambda: getattr(regs, cls).create(lam, lambda_updater=upd, val_split=vs, **kw)(
                optimizer=opt, logger=log))
            got.append((res[0], res[1] if res[0] != "ok" else (res[1].lambda_, res[1].val_split)))
        assert got[0] == got[1], (cls, lam, with_upd, vs, kw, got)
    for args in [(0.0, (1, 2)), (1.0, (1, 2)), (0.5, (1, 2, 3)), (0.5, (-1, 2)), (0.5, (2, 1)), (0.5, (1, 1)),
                 (0.5, (0, 2))]:
        a, b = _outcome(lambda: ru.IntervalParamScaler(*args) and None), _outcome(lambda: mu.IntervalParamScaler(*args)
                                                                                 and None)
        assert a == b, args
    ref_u, my_u = ru.IntervalParamScaler(0.25, (0.8, 1.3)), mu.IntervalParamScaler(0.25, (0.8, 1.3))
    grid = [0.0, 1e-17, 0.3, 0.8, 1.0, 1.04, 1.3, 2.5]
    for lam in [0.1, 1.0, 0.0, -0.5, 1, 1e-17]:
        for tl in grid + [-1.0]:
            for vl in grid + [th.tensor(0.9), th.tensor([0.9])]:
                a, b = _outcome(lambda: ref_u(lam, tl, vl)), _outcome(lambda: my_u(lam, tl, vl))
                assert a[0] == b[0] and (a[1] == b[1] or float(a[1]) == float(b[1])), (lam, tl, vl, a, b)


def test_logger_key_prefix():
    from imitation_b200.util import logger

    lg = logger.configure()
    with pytest.raises(RuntimeError):
        with lg.add_key_prefix("x"):
            pass
    with lg.accumulate_means("reward"), lg.add_key_prefix("epoch-0"), lg.add_key_prefix("val"):
        lg.record("loss", 1.0)
        lg.record("loss", 3.0)
    assert lg.name_to_value["mean/reward/epoch-0/val/loss"] == 2.0


# ---------------------------------------------------------------------------------------------------------------------
# the CPU restatement and the skipping rank's draws against the golden (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _port_nets(name, z):
    from oracle import nets_port

    c = _cfg(name)
    nets = []
    for st in _golden_states(z, name, "init"):
        if c["net"] == "shaped":
            net = nets_port.ShapedRewardNetPort(DO, DA, (32,), (32, 32), normalize_input=True)
        else:
            net = nets_port.BasicRewardNetPort(DO, DA, (32, 32), normalize_input=c["net"] == "norm")
        net.load_state_dict(G.state_to_torch(st))
        nets.append(net)
    return nets


def _as_dict(t):
    return dict(obs=t.obs, acts=t.acts, rews=t.rews, terminal=t.terminal)


def _final_key_values(z, name):
    keys, vals = list(z[f"{name}/log_keys"]), z[f"{name}/log_vals"]
    return {k: float(v) for k, v in zip(keys, vals)}


@pytest.mark.parametrize("name", sorted(CASES))
def test_cpu_port_matches_the_golden(name):
    from imitation_b200.data import types
    from oracle import pref_regularization_port as port

    z = G.load("pref_regularization")
    c = _cfg(name)
    nets = _port_nets(name, z)
    pairs, prefs = _data(name, types)
    pairs = [(_as_dict(a), _as_dict(b)) for a, b in pairs]
    kw = dict(kind=c["kind"], p=c["p"], lam=c["lam"], val_split=c["val_split"], batch_size=c["batch_size"],
              minibatch_size=c["minibatch_size"], epochs=c["epochs"], lr=c["lr"], noise_prob=c["noise_prob"],
              discount_factor=c["discount_factor"],
              updater=None if c["updater"] is None else (c["updater"][0],) + tuple(c["updater"][1]))
    rng = np.random.default_rng(7)
    th.manual_seed(11)
    if c["members"]:
        results = port.train_ensemble(nets, pairs, prefs, rng, **kw)
    else:
        results = [port.train_member(nets[0], pairs, prefs, list(range(len(pairs))), rng, **kw)]
    assert np.array_equal(np.concatenate([r[1] for r in results]) if c["updater"] else np.zeros(0),
                          z[f"{name}/lambdas"])
    np.testing.assert_array_equal(_fingerprint(rng), z[f"{name}/np_after"])
    np.testing.assert_array_equal(th.get_rng_state().numpy(), z[f"{name}/th_after"])
    for net, want in zip(nets, _golden_states(z, name, "final")):
        got = net.state_dict()
        for k, v in G.state_to_torch(want).items():
            if k.endswith("dense_final.bias"):
                continue
            np.testing.assert_allclose(got[k].numpy(), v.numpy(), rtol=2e-4, atol=2e-6, err_msg=f"{name} {k}")
    logged = _final_key_values(z, name)
    for key in ("regularized_loss", "val/loss", "val/accuracy", "val/gt_reward_loss"):
        vals = [r[2][key] for r in results if key in r[2]]
        if f"reward/final/{key}" in logged:
            np.testing.assert_allclose(np.mean(vals), logged[f"reward/final/{key}"], rtol=1e-4, atol=1e-6, err_msg=key)
        else:
            assert not vals, key


@pytest.mark.parametrize("name", sorted(CASES))
def test_skipped_members_make_the_golden_draws(name):
    """Every member skipped (a rank that trains none of them) leaves numpy's and torch's generators where training
    every member leaves them."""
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import regularizers, updaters
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import logger

    class HostNet(reward_nets.RewardNet):
        """A plain torch reward net: the draws do not depend on the network, and this one needs no CUDA library."""

        def __init__(self, obs_space, act_space):
            super().__init__(obs_space, act_space)
            self.lin = th.nn.Linear(DO + DA, 1)

        def forward(self, state, action, next_state, done):
            return self.lin(th.cat([state, action], 1)).squeeze(1)

    c = _cfg(name)
    z = G.load("pref_regularization")
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (DO,), np.float32), spaces.Box(-1.0, 1.0, (DA,), np.float32)
    members = [HostNet(obs_space, act_space) for _ in range(max(c["members"], 1))]
    model = reward_nets.RewardEnsemble(obs_space, act_space, members) if c["members"] else members[0]
    upd = None if c["updater"] is None else updaters.IntervalParamScaler(c["updater"][0], c["updater"][1])
    cls = regularizers.LpRegularizer if c["kind"] == "lp" else regularizers.WeightDecayRegularizer
    factory = cls.create(c["lam"], lambda_updater=upd, val_split=c["val_split"],
                         **(dict(p=c["p"]) if c["kind"] == "lp" else {}))
    rng = np.random.default_rng(7)
    pairs, prefs = _data(name, types)
    ds = pc.PreferenceDataset()
    ds.push(pairs, prefs)
    th.manual_seed(11)
    args = dict(rng=rng, batch_size=c["batch_size"], minibatch_size=c["minibatch_size"], epochs=c["epochs"],
                lr=c["lr"], custom_logger=logger.configure(), regularizer_factory=factory)
    if c["members"]:
        et = pc.EnsembleTrainer(pc.PreferenceModel(model), pc.CrossEntropyRewardLoss(), **args)
        et._dist = (c["members"] + 1, c["members"], None)  # the rank past the last member trains none of them
        et._sync_members = lambda: None
        et.train(ds)
    else:
        pc.BasicRewardTrainer(pc.PreferenceModel(model), pc.CrossEntropyRewardLoss(), **args)._skip_draws(ds)
    np.testing.assert_array_equal(_fingerprint(rng), z[f"{name}/np_after"])
    np.testing.assert_array_equal(th.get_rng_state().numpy(), z[f"{name}/th_after"])


def test_not_enough_data_to_split():
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import regularizers, updaters
    from imitation_b200.util import logger

    pairs, prefs = _data("lp2_falls", types)
    ds = pc.PreferenceDataset()
    ds.push(pairs[:4], prefs[:4])  # int(4 * 0.2) = 0 validation items
    t = pc.BasicRewardTrainer.__new__(pc.BasicRewardTrainer)
    t.rng = np.random.default_rng(0)
    t.regularizer = regularizers.LpRegularizer(th.optim.SGD([th.nn.Parameter(th.ones(1))], lr=1.0), 0.1,
                                               updaters.IntervalParamScaler(0.1, (1.0, 2.0)), logger.configure(), p=2,
                                               val_split=0.2)
    assert t.requires_regularizer_update
    with pytest.raises(ValueError, match="Not enough data samples to split"):
        t._split(ds)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _mine(name, fused, init):
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import regularizers, updaters
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import logger, networks

    return _run(name, pc, regularizers, updaters, reward_nets, networks, types, logger, spaces, device="cuda",
                init=init, fused=fused)


def _assert_weights_close(got, want, name):
    """Within the trainer tolerance (rtol 2e-4, atol 2e-6), except with weight decay and no Lp term: the few layer-1
    units that only 0-4 of the training rows activate flip on or off with rounding, and Adam turns a flip into a +-lr
    step, so up to an eighth of a tensor's elements may then differ by at most one step size per optimiser step of the
    call (DESIGN.md, f1 row)."""
    c = _cfg(name)
    bad = ~np.isclose(got, want, rtol=2e-4, atol=2e-6)
    if c["kind"] != "wd" or not bad.any():
        np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-6, err_msg=name)
        return
    steps = -(-int(c["n"] * (1 - (c["val_split"] or 0))) // c["batch_size"]) * c["epochs"]
    assert bad.mean() <= 0.125, (name, bad.sum(), got.shape)  # the weights and biases of a few such units
    assert np.abs(got - want).max() <= steps * c["lr"], (name, np.abs(got - want).max())


def _check_against_golden(name, z, members, trainer, lg, lambdas):
    c = _cfg(name)
    assert np.array_equal(np.array(lambdas, np.float64), z[f"{name}/lambdas"]), (name, lambdas)
    for m, want in zip(members, _golden_states(z, name, "final")):
        got = m.state_dict()
        for k, v in want.items():
            if v.dtype.kind in "iu":  # RunningNorm counts
                np.testing.assert_array_equal(got[k].cpu().numpy(), v, err_msg=f"{name} {k}")
            elif not k.endswith("dense_final.bias"):  # (cancels in r2 - r1, as in test_preference.py)
                _assert_weights_close(got[k].cpu().numpy(), v, f"{name}")
    want = _final_key_values(z, name)
    for k, v in want.items():
        if k in IGNORED_KEYS or k.startswith("reward/final/train/gt_reward_loss"):
            continue
        if c["members"] and not (k.startswith("reward/final/") or k == "regularization_lambda"):
            continue  # the reference's per-member epoch keys carry a member-k/ prefix this package does not record
        assert k in lg.name_to_value, (name, k)
        if k.endswith("regularization_lambda") or k.endswith("regularization_lambda_std"):
            assert float(lg.name_to_value[k]) == v, (name, k)
        else:
            np.testing.assert_allclose(float(lg.name_to_value[k]), v, rtol=1e-4, atol=2e-6, err_msg=f"{name} {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "autograd"])
@pytest.mark.parametrize("name", GPU_CASES)
def test_trainer_matches_the_golden(name, fused):
    z = G.load("pref_regularization")
    init = _golden_states(z, name, "init")
    members, trainer, lg, lambdas, _, rng = _mine(name, fused, init)
    trainers = getattr(trainer, "member_trainers", [trainer])
    assert all(("_fused_opt" in t.__dict__) == fused for t in trainers)
    _check_against_golden(name, z, members, trainer, lg, lambdas)
    np.testing.assert_array_equal(_fingerprint(rng), z[f"{name}/np_after"])
    np.testing.assert_array_equal(th.get_rng_state().numpy(), z[f"{name}/th_after"])
    if lambdas and not _cfg(name)["members"]:
        assert trainer.regularizer.lambda_ == lambdas[-1]


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "autograd"])
@pytest.mark.parametrize("name", CPU_ONLY)
def test_input_norm_counts_and_lambdas_match_the_golden(name, fused):
    """The validation pass runs in training mode: the input RunningNorm counts every training and validation row."""
    z = G.load("pref_regularization")
    members, _, _, lambdas, _, _ = _mine(name, fused, _golden_states(z, name, "init"))
    assert np.array_equal(np.array(lambdas, np.float64), z[f"{name}/lambdas"]), (name, lambdas)
    want = _golden_states(z, name, "final")[0]
    counts = [k for k, v in want.items() if v.dtype.kind in "iu"]
    assert counts
    for k in counts:
        np.testing.assert_array_equal(members[0].state_dict()[k].cpu().numpy(), want[k], err_msg=k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lp2_falls", "lp1_rises", "wd_fixed", "wd_updater", "norm"])
def test_fused_step_equals_the_autograd_path(name):
    """k penalty terms per step on both paths: the same weights, Adam moments and step counts, lambdas and logged keys."""
    from imitation_b200 import _lib

    z = G.load("pref_regularization")
    init = _golden_states(z, name, "init")
    runs = []
    for fused in (True, False):
        before = _lib.LAUNCHES["count"]
        runs.append(_mine(name, fused, init) + (_lib.LAUNCHES["count"] - before,))
    (ma, ta, la, lama, _, _, _), (mb, tb, lb, lamb, _, _, _) = runs
    assert lama == lamb
    for k, v in ma[0].state_dict().items():
        w = mb[0].state_dict()[k]
        if v.dtype in (th.int32, th.int64):
            assert th.equal(v, w), k
        elif not k.endswith("dense_final.bias"):
            _assert_weights_close(v.cpu().numpy(), w.cpu().numpy(), name)
    pa, pb = list(ma[0].parameters()), list(mb[0].parameters())
    for x, y in zip(pa, pb):
        assert float(ta.optim.state[x]["step"]) == float(tb.optim.state[y]["step"]) > 0
        if x.shape != pa[-1].shape or x is not pa[-1]:
            np.testing.assert_allclose(ta.optim.state[x]["exp_avg"].cpu().numpy(),
                                       tb.optim.state[y]["exp_avg"].cpu().numpy(), rtol=1e-3, atol=1e-7)
    keys = [k for k in lb.name_to_value if k.startswith("mean/") or k.startswith("reward/final/")]
    assert set(keys) - {"reward/final/train/gt_reward_loss"} <= set(la.name_to_value)
    for k in keys:
        if k in la.name_to_value:
            np.testing.assert_allclose(la.name_to_value[k], lb.name_to_value[k], rtol=1e-4, atol=2e-6, err_msg=k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["lp3_fixed", "wd_fixed"])
def test_one_extra_launch_per_training_minibatch(name):
    """A training call of the device step with a regularizer issues exactly one launch more per training minibatch than
    the same call without one (measured on a second call, after the fragments are in the pool)."""
    from imitation_b200 import _lib, spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import regularizers
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import logger

    c = _cfg(name)
    pairs, prefs = _data(name, types)
    ds = pc.PreferenceDataset()
    ds.push(pairs, prefs)
    counts = []
    for reg in (False, True):
        net = reward_nets.BasicRewardNet(spaces.Box(-np.inf, np.inf, (DO,), np.float32),
                                         spaces.Box(-1.0, 1.0, (DA,), np.float32), hid_sizes=(32, 32)).cuda()
        cls = regularizers.LpRegularizer if c["kind"] == "lp" else regularizers.WeightDecayRegularizer
        f = cls.create(c["lam"], val_split=None, **(dict(p=c["p"]) if c["kind"] == "lp" else {})) if reg else None
        tr = pc.BasicRewardTrainer(pc.PreferenceModel(net), pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(7),
                                   batch_size=c["batch_size"], minibatch_size=c["minibatch_size"], epochs=c["epochs"],
                                   lr=c["lr"], custom_logger=logger.configure(), regularizer_factory=f)
        tr.train(ds)
        before = _lib.LAUNCHES["count"]
        tr.train(ds)
        counts.append(_lib.LAUNCHES["count"] - before)
        assert "_fused_opt" in tr.__dict__
    n_mb = -(-c["n"] // c["minibatch_size"]) * c["epochs"]
    assert counts[1] == counts[0] + n_mb, (counts, n_mb)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [1, 2, 3])
def test_lp_kernel_matches_float64_autograd(p):
    """imb_param_regularize(IMB_REG_LP) against float64 autograd of lambda * sum_tensors vector_norm(w, p) ** p, with
    exact zeros (single weights and a whole zero tensor), at every reward-net shape the descriptor takes."""
    from imitation_b200 import _lib, spaces
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    lam = 0.37
    shapes = [dict(hid_sizes=(1,)), dict(hid_sizes=(64,)), dict(hid_sizes=(32, 32)), dict(hid_sizes=(64, 64)),
              dict(hid_sizes=(17, 5), normalize_input_layer=networks.RunningNorm)]
    for d_obs, kw in [(3, shapes[0]), (11, shapes[1]), (6, shapes[2]), (30, shapes[3]), (9, shapes[4])]:
        th.manual_seed(d_obs + p)
        net = reward_nets.BasicRewardNet(spaces.Box(-np.inf, np.inf, (d_obs,), np.float32),
                                         spaces.Box(-1.0, 1.0, (2,), np.float32), **kw).cuda()
        params = [q for q in net.parameters()]
        with th.no_grad():
            params[0].view(-1)[::3] = 0.0
            params[-1].zero_()  # a zero-norm tensor
        e = net.engine()
        e.sync()
        ws = e.ws
        ws.zero_()
        stats = th.zeros(8, device="cuda")
        base = th.randn(e.desc.n_params, device="cuda")
        gacc = ws[:e.desc.n_params]  # the accumulator sits at the start of the workspace (imb.h)
        gacc.copy_(base)
        _lib.param_regularize(e.desc, _lib.REG_LP, p, lam, e.params, ws, stats, 1)
        w64 = [q.detach().double().requires_grad_() for q in params]
        pen = lam * sum(th.linalg.vector_norm(w, ord=p).pow(p) for w in w64)
        grads = th.autograd.grad(pen, w64)
        want = base.double() + th.cat([g.reshape(-1) for g in grads])
        np.testing.assert_allclose(gacc.double().cpu().numpy(), want.cpu().numpy(), rtol=2e-6, atol=1e-6)
        np.testing.assert_allclose(float(stats[4]), float(pen), rtol=1e-5)
        assert float(stats[6]) == 1.0 and float(stats[0]) == 0.0
        again = th.zeros(8, device="cuda")
        _lib.param_regularize(e.desc, _lib.REG_LP, p, lam, e.params, ws, again, 1)
        assert th.equal(again[4], stats[4])  # no atomics: the same bits on every call


@pytest.mark.gpu
def test_weight_decay_kernel_is_bit_equal_to_torch():
    from imitation_b200 import _lib, spaces
    from imitation_b200.rewards import reward_nets

    net = reward_nets.BasicRewardNet(spaces.Box(-np.inf, np.inf, (11,), np.float32),
                                     spaces.Box(-1.0, 1.0, (3,), np.float32), hid_sizes=(32, 32)).cuda()
    e = net.engine()
    e.sync()
    for lam, lr in [(0.1, 1e-3), (3.7, 2e-3), (1e-3, 0.3)]:
        want = [q.detach().clone() for q in net.parameters()]
        want = [th.add(w, (-lam * lr) * w) for w in want]
        _lib.param_regularize(e.desc, _lib.REG_WEIGHT_DECAY, 0, -lam * lr, e.params, None)
        for q, w in zip(net.parameters(), want):
            assert th.equal(q.detach(), w)


@pytest.mark.gpu
def test_bad_kind_and_p_are_refused():
    from imitation_b200 import _lib, spaces
    from imitation_b200.rewards import reward_nets

    net = reward_nets.BasicRewardNet(spaces.Box(-np.inf, np.inf, (4,), np.float32),
                                     spaces.Box(-1.0, 1.0, (2,), np.float32), hid_sizes=(8,)).cuda()
    e = net.engine()
    e.sync()
    with pytest.raises(_lib.ImbError, match="kind"):
        _lib.param_regularize(e.desc, 3, 2, 0.1, e.params, e.ws)
    with pytest.raises(_lib.ImbError, match="p = 0"):
        _lib.param_regularize(e.desc, _lib.REG_LP, 0, 0.1, e.params, e.ws)


@pytest.mark.gpu
def test_user_loss_regularizer_trains_through_the_autograd_path():
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import regularizers
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import logger

    class Sum(regularizers.LossRegularizer):
        def _loss_penalty(self, loss):
            return self.lambda_ * sum(q.sum() for g in self.optimizer.param_groups for q in g["params"])

    net = reward_nets.BasicRewardNet(spaces.Box(-np.inf, np.inf, (DO,), np.float32),
                                     spaces.Box(-1.0, 1.0, (DA,), np.float32), hid_sizes=(32, 32)).cuda()
    lg = logger.configure()
    tr = pc.BasicRewardTrainer(pc.PreferenceModel(net), pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(0),
                               batch_size=4, epochs=2, custom_logger=lg,
                               regularizer_factory=Sum.create(0.5, val_split=None))
    pairs, prefs = _data("lp2_falls", types)
    ds = pc.PreferenceDataset()
    ds.push(pairs, prefs)
    assert tr._fused_target(ds) is None
    w0 = net.mlp.dense0.weight.detach().clone()
    tr.train(ds)
    assert "_fused_opt" not in tr.__dict__ and not th.equal(w0, net.mlp.dense0.weight)
    assert np.isfinite(lg.name_to_value["mean/reward/epoch-1/regularized_loss"])
    assert lg.name_to_value["reward/final/regularized_loss"] == lg.name_to_value["mean/reward/epoch-1/regularized_loss"]


@pytest.mark.gpu
def test_not_enough_data_on_the_device_step():
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import regularizers, updaters
    from imitation_b200.rewards import reward_nets

    net = reward_nets.BasicRewardNet(spaces.Box(-np.inf, np.inf, (DO,), np.float32),
                                     spaces.Box(-1.0, 1.0, (DA,), np.float32), hid_sizes=(32, 32)).cuda()
    f = regularizers.LpRegularizer.create(0.1, updaters.IntervalParamScaler(0.1, (1.0, 2.0)), val_split=0.1, p=2)
    tr = pc.BasicRewardTrainer(pc.PreferenceModel(net), pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(0),
                               batch_size=4, regularizer_factory=f)
    pairs, prefs = _data("lp2_falls", types)
    ds = pc.PreferenceDataset()
    ds.push(pairs[:9], prefs[:9])
    with pytest.raises(ValueError, match="Not enough data samples"):
        tr.train(ds)
