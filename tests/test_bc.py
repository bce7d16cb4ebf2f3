"""Behavioural cloning: `algorithms.bc.BC`, its host logic, and the BC loss of k_ppo_update_gen.

- `tests/golden/bc.npz` is recorded from the reference's own `BC.train` (oracle/bc_ref.py): Box with and without the
  feature RunningNorm, Discrete, minibatch_size < batch_size with l2_weight > 0, an incomplete last batch that is logged.
  It stores the initial parameters, the DataLoader's per-epoch index order, the trained parameters, the norm state and
  the logged metrics.  `oracle/bc_port.py` restates the loop in float64 without the reference and is pinned to it here.
- CPU: the port against the golden; errors against the reference's own classes; refusals; demonstration forms; the
  host permutation against the reference's loader (order and torch RNG consumption); the launch plan.
- GPU: the kernel against the float64 port over widths, activations, action spaces, feature norm in training and
  evaluation mode, minibatch sizes, accumulation and loss weights.  At lr = 0 the parameters stay fixed, so every
  minibatch's gradient is read out through Adam's moments (exp_avg, exp_avg_sq) and compared with float64 within
  C_GRAD of the sum of the absolute per-batch gradients (plus a floor at FLOOR of the largest); the norm state, count,
  state words and metrics are compared too.  At lr != 0 the parameters are compared after a few steps.  Then the golden
  on the device, split launches against one launch (bits), determinism, n_batches ending mid-epoch, and training on
  the expert fixtures.
"""
import math
import os

import numpy as np
import pytest
import torch as th

from imitation_b200 import _lib, spaces
from imitation_b200.algorithms import bc as bc_mod
from imitation_b200.data import types
from oracle import bc_port, refimport
from tests import golden_util as G

C_GRAD = 2e-4    # moments: relative to the beta-weighted sum of |per-batch gradient|
FLOOR = 1e-6     # ... plus this fraction of the largest such sum
C_METRIC = 1e-4  # metrics relative to their magnitude (plus C_METRIC absolute)
CASES_GOLDEN = ("box_norm", "box_plain_accum_l2", "discrete", "discrete_norm_relu_accum")


def _golden():
    return np.load(os.path.join(G.GOLDEN, "bc.npz"))


def _case(z, name):
    g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
    d_obs, d_act, discrete, hidden, norm, relu, n, bs, mb, n_epochs, log_iv = (int(x) for x in g["config"])
    lr, ent_w, l2_w = (float(x) for x in g["hparams"])
    return g, dict(d_obs=d_obs, d_act=d_act, discrete=bool(discrete), hidden=hidden, norm=bool(norm), relu=bool(relu),
                   n=n, bs=bs, mb=mb, n_epochs=n_epochs, log_interval=log_iv, lr=lr, ent_weight=ent_w, l2_weight=l2_w)


def _port_from(c, params0, norm0=None, count0=0, lr=None, eps=1e-8):
    p = bc_port.make_policy(c["d_obs"], c["d_act"], c["discrete"], c["hidden"], c["norm"], c["relu"])
    bc_port.set_flat(p, params0)
    if c["norm"] and norm0 is not None:
        d = c["d_obs"]
        p.feat_norm.running_mean.copy_(th.as_tensor(norm0[:d], dtype=th.float64))
        p.feat_norm.running_var.copy_(th.as_tensor(norm0[d:], dtype=th.float64))
        p.feat_norm.count.fill_(int(count0))
    return bc_port.BCPort(p, c["bs"], c["mb"], lr=c["lr"] if lr is None else lr, eps=eps, ent_weight=c["ent_weight"],
                          l2_weight=c["l2_weight"])


# ---- CPU --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES_GOLDEN)
def test_port_reproduces_golden(name):
    g, c = _case(_golden(), name)
    port = _port_from(c, g["params0"])
    logged = port.train(g["obs"], g["acts"], list(g["order"]), c["n_epochs"] * (c["n"] // c["mb"]), c["log_interval"])
    got = bc_port.get_flat(port.policy)
    np.testing.assert_allclose(got, g["params"], rtol=1e-4, atol=2e-5)
    assert [b for b, _ in logged] == list(g["batches"])
    np.testing.assert_allclose(np.array([m for _, m in logged]), g["metrics"], rtol=1e-4, atol=1e-5)
    if c["norm"]:
        p = port.policy.feat_norm
        np.testing.assert_allclose(np.concatenate([p.running_mean.numpy(), p.running_var.numpy()]), g["norm"],
                                   rtol=1e-5, atol=1e-6)
        assert int(p.count) == int(g["count"])


def _ref_bc():
    if not refimport.available():
        pytest.skip("needs the reference sources (oracle/refimport.py)")
    from oracle import bc_ref

    return bc_ref.load()


def _ref_policy(d_obs=3, d_act=2):
    from gymnasium import spaces as gspaces

    p = bc_port.make_policy(d_obs, d_act, False, 4, False, dtype=th.float32)
    p.observation_space = gspaces.Box(-np.inf, np.inf, (d_obs,), np.float32)
    p.action_space = gspaces.Box(-1.0, 1.0, (d_act,), np.float32)
    p.device = th.device("cpu")
    return p


def _raises(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001 -- the class and text are what is compared
        return type(e), str(e)
    return None


def test_errors_match_reference():
    rbc = _ref_bc()
    from imitation.data import types as rtypes

    pol = _ref_policy()
    kw = dict(observation_space=pol.observation_space, action_space=pol.action_space, rng=np.random.default_rng(0),
              policy=pol, device="cpu")
    ref = _raises(lambda: rbc.BC(batch_size=32, minibatch_size=5, **kw))
    assert ref == (ValueError, "Batch size must be a multiple of minibatch size.")
    ours = _raises(lambda: bc_mod.BC(observation_space=spaces.Box(-np.inf, np.inf, (3,)),
                                     action_space=spaces.Box(-1, 1, (2,)), rng=np.random.default_rng(0), batch_size=32,
                                     minibatch_size=5))
    assert ours == ref
    ref = _raises(lambda: rbc.BC(optimizer_kwargs=dict(weight_decay=0.1), **kw))
    assert ref[0] is ValueError
    assert _raises(lambda: bc_mod.adam_hparams(th.optim.Adam, dict(weight_decay=0.1))) == ref
    ref = _raises(lambda: rbc.BatchIteratorWithEpochEndCallback([], None, None, None))
    assert _raises(lambda: bc_mod.check_epochs_batches(None, None)) == ref
    assert _raises(lambda: bc_mod.check_epochs_batches(1, 2)) == ref
    obs = np.zeros((10, 3), np.float32)
    small = rtypes.TransitionsMinimal(obs=obs, acts=np.zeros((10, 2), np.float32), infos=np.array([{}] * 10))
    ref = _raises(lambda: rbc.BC(demonstrations=small, batch_size=16, **kw))
    ours_small = types.TransitionsMinimal(obs=obs, acts=np.zeros((10, 2), np.float32), infos=np.array([{}] * 10))
    assert _raises(lambda: bc_mod.demonstration_arrays(ours_small, 16)) == ref
    # an iterable of batches of the wrong size: the reference raises when the loader is iterated
    batches = [{"obs": obs[:4], "acts": np.zeros((4, 2), np.float32)}]
    trainer = rbc.BC(demonstrations=batches, batch_size=8, **kw)
    ref = _raises(lambda: trainer.train(n_epochs=1, progress_bar=False))
    assert _raises(lambda: bc_mod.demonstration_arrays(batches, 8)) == ref


def test_refusals_raise_not_implemented():
    box, act = spaces.Box(-np.inf, np.inf, (3,)), spaces.Box(-1, 1, (2,))
    kw = dict(observation_space=box, action_space=act, rng=np.random.default_rng(0))
    with pytest.raises(NotImplementedError, match="optimizer_cls"):
        bc_mod.BC(optimizer_cls=th.optim.SGD, **kw)
    with pytest.raises(NotImplementedError, match="betas"):
        bc_mod.BC(optimizer_kwargs=dict(betas=(0.8, 0.999)), **kw)
    with pytest.raises(NotImplementedError, match="amsgrad"):
        bc_mod.BC(optimizer_kwargs=dict(amsgrad=True), **kw)
    with pytest.raises(NotImplementedError, match="policy"):
        bc_mod.BC(policy=th.nn.Linear(3, 2), **kw)
    with pytest.raises(NotImplementedError, match="minibatch size must be in"):
        bc_mod.BC(batch_size=8192, **kw)
    # foreach / fused only choose torch's implementation
    assert bc_mod.adam_hparams(th.optim.Adam, dict(lr=3e-4, foreach=True, fused=False, eps=1e-6)) == (3e-4, 1e-6)


def test_demonstration_forms_map_to_table_rows():
    from imitation_b200.policies.base import ActorCriticPolicy

    rng = np.random.default_rng(1)
    obs = rng.normal(size=(12, 3)).astype(np.float32)
    acts = rng.normal(size=(12, 2)).astype(np.float32)
    tr = types.TransitionsMinimal(obs=obs, acts=acts, infos=np.array([{}] * 12))
    o, a, shuffled = bc_mod.demonstration_arrays(tr, 4)
    assert shuffled and np.array_equal(o, obs) and np.array_equal(a, acts)
    trajs = [types.Trajectory(obs=np.concatenate([obs[:6], obs[6:7]]), acts=acts[:6], infos=None, terminal=True),
             types.Trajectory(obs=np.concatenate([obs[6:12], obs[:1]]), acts=acts[6:12], infos=None, terminal=False)]
    o, a, shuffled = bc_mod.demonstration_arrays(trajs, 4)
    assert shuffled and np.array_equal(o, obs) and np.array_equal(a, acts)
    batches = [{"obs": obs[i:i + 4], "acts": acts[i:i + 4]} for i in (8, 0, 4)]
    o, a, shuffled = bc_mod.demonstration_arrays(batches, 4)
    assert not shuffled and np.array_equal(o, obs[[*range(8, 12), *range(0, 8)]])
    pol = ActorCriticPolicy(spaces.Box(-np.inf, np.inf, (3,)), spaces.Box(-1, 1, (2,)))
    t = bc_mod.demo_table(pol, obs, acts)
    assert t.shape == (12, _lib.rollout_row_width(pol.desc))
    assert th.equal(t[:, :3], th.as_tensor(obs)) and th.equal(t[:, 3:5], th.as_tensor(acts)) and not t[:, 5:].any()
    dpol = ActorCriticPolicy(spaces.Box(-np.inf, np.inf, (3,)), spaces.Discrete(4))
    idx = np.array([3, 0, 1, 2] * 3)
    t = bc_mod.demo_table(dpol, obs, idx)
    assert th.equal(t[:, 3], th.as_tensor(idx, dtype=th.float32)) and not t[:, 4:].any()


def test_host_permutation_matches_reference_loader():
    _ref_bc()
    from imitation.algorithms import base as rbase
    from imitation.data import types as rtypes

    n, mb = 37, 8
    order = []

    class Recorded(rtypes.Transitions):
        def __getitem__(self, key):
            if isinstance(key, (int, np.integer)):
                order.append(int(key))
            return super().__getitem__(key)

    obs = np.zeros((n, 2), np.float32)
    demos = Recorded(obs=obs, acts=np.zeros((n, 1), np.float32), infos=np.array([{}] * n), next_obs=obs.copy(),
                     dones=np.zeros(n, dtype=bool))
    loader = rbase.make_data_loader(demos, mb)
    for seed in (0, 5):
        th.manual_seed(seed)
        order.clear()
        for _ in range(3):  # three epochs, one iteration of the loader each
            for _ in loader:
                pass
        ref_state = th.get_rng_state()
        th.manual_seed(seed)
        ours = [bc_mod.epoch_permutation(n, mb)[:(n // mb) * mb] for _ in range(3)]
        assert th.equal(th.get_rng_state(), ref_state)
        assert np.array_equal(np.concatenate([o.numpy() for o in ours]), np.asarray(order))


def _simulate(sched, M):
    """Check a launch plan: launches cover [0, M) in order; every event comes after the launch of its minibatch."""
    done, flushed = 0, False
    for item in sched:
        if item[0] == "launch":
            _, j0, n, ff = item
            assert j0 == done and ff in (0, 1, 2)
            if n == 0:
                assert ff == 1 and j0 == M and not flushed
                flushed = True
            done = j0 + n
        else:
            assert item[1] < done
    assert done == M
    return [tuple(i) for i in sched if i[0] != "launch"]


@pytest.mark.parametrize("M,P,k,by_epochs", [(12, 4, 1, True), (15, 5, 4, True), (12, 3, 5, True), (8, 3, 2, False),
                                             (6, 6, 3, False), (9, 9, 4, True)])
def test_launch_plan_for_every_callback_combination(M, P, k, by_epochs):
    events = bc_mod.train_events(M, P, k, by_epochs)
    for ob in (False, True):
        for oe in (False, True):
            for lr_ in (False, True):
                sched = bc_mod.plan_launches(M, P, k, by_epochs, 2, on_batch_end=ob, on_epoch_end=oe, log_rollouts=lr_)
                assert _simulate(sched, M) == events
                launches = [i for i in sched if i[0] == "launch"]
                if not (ob or oe or lr_):
                    assert launches == [["launch", 0, M, 1]]
                for pos, item in enumerate(sched):  # the host sees the policy exactly where a callback needs it
                    if item[0] == "launch":
                        continue
                    need = ((item[0] == "batch" and (ob or (lr_ and item[2] % 2 == 0))) or (item[0] == "epoch" and oe))
                    if need:
                        prev = [i for i in sched[:pos] if i[0] == "launch"][-1]
                        flush = item[0] == "batch" and M % k and item is sched[-1]
                        end = M if flush else item[1] + 1
                        assert prev[1] + prev[2] == end
    # the reference's order: an incomplete last batch steps after the last epoch's end
    assert events[-2:] == ([("epoch", M - 1, M // P - 1), ("batch", M - 1, (M - 1) // k + 1)]
                           if by_epochs and M % k else events[-2:])


def test_launch_plan_splits_final_flush_after_epoch_callback():
    sched = bc_mod.plan_launches(10, 5, 4, True, 1, on_batch_end=False, on_epoch_end=True, log_rollouts=False)
    assert sched == [["launch", 0, 5, 0], ["batch", 3, 0], ["epoch", 4, 0], ["launch", 5, 5, 2], ["batch", 7, 1],
                     ["epoch", 9, 1], ["launch", 10, 0, 1], ["batch", 9, 3]]


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _policy(c):
    from imitation_b200.policies.base import ActorCriticPolicy

    act = spaces.Discrete(c["d_act"]) if c["discrete"] else spaces.Box(-1, 1, (c["d_act"],))
    return ActorCriticPolicy(spaces.Box(-np.inf, np.inf, (c["d_obs"],)), act, net_arch=[c["hidden"]] * 2,
                             activation_fn=th.nn.ReLU if c["relu"] else th.nn.Tanh, normalize_features=c["norm"])


def _device_bc(c, params0, obs, acts, norm0=None, count0=0, lr=None, train_mode=True, eps=1e-8):
    pol = _policy(c).cuda()
    flat, ns, cnt = pol.flat_vectors()
    flat.copy_(th.as_tensor(params0, dtype=th.float32))
    if c["norm"] and norm0 is not None:
        ns.copy_(th.as_tensor(norm0, dtype=th.float32))
        cnt.fill_(int(count0))
    pol.set_training_mode(train_mode)
    tr = types.TransitionsMinimal(obs=obs, acts=acts, infos=np.array([{}] * len(obs)))
    return bc_mod.BC(observation_space=pol.observation_space, action_space=pol.action_space,
                     rng=np.random.default_rng(0), policy=pol, demonstrations=tr, batch_size=c["bs"],
                     minibatch_size=c["mb"], optimizer_kwargs=dict(lr=c["lr"] if lr is None else lr, eps=eps),
                     ent_weight=c["ent_weight"], l2_weight=c["l2_weight"],
                     custom_logger=_Records())


class _Records:
    def __init__(self):
        self.rows = []
        self._cur = {}

    def record(self, key, val, exclude=None):
        self._cur[key] = val

    def dump(self, step=0):
        self.rows.append(dict(self._cur))
        self._cur = {}


def _fixed_perms(monkeypatch, perms):
    """BC draws these epoch orders instead of the DataLoader's (each padded to the N entries of a permutation row)."""
    it = iter(perms)

    def perm(n, mb):
        p = th.as_tensor(np.asarray(next(it)), dtype=th.int64)
        return th.cat([p, th.zeros(n - len(p), dtype=th.int64)])

    monkeypatch.setattr(bc_mod, "epoch_permutation", perm)


def _metrics(trainer):
    rows = trainer.logger.rows
    return [r["bc/batch"] for r in rows], np.array([[r[f"bc/{m}"] for m in bc_port.METRICS] for r in rows])


# name: (d_obs, d_act, discrete, width, norm, relu, N, batch_size, minibatch, ent_weight, l2_weight, epochs, train mode)
SWEEP = {
    "w1_box_norm": (5, 2, False, 1, True, False, 40, 8, 8, 1e-3, 0.0, 2, True),
    "w7_disc_relu_accum": (6, 3, True, 7, False, True, 70, 16, 4, 1e-2, 1e-3, 2, True),
    "w32_box_mb1": (4, 2, False, 32, True, False, 9, 4, 1, 0.0, 1e-2, 2, True),
    "w32_box_hc_mb64_eval": (17, 6, False, 32, True, False, 300, 64, 64, 1e-3, 0.0, 2, False),
    "w33_disc_norm_mb32_k4": (4, 2, True, 33, True, False, 300, 128, 32, 1e-3, 1e-4, 2, True),
    "w64_box_relu_mb128": (11, 3, False, 64, False, True, 400, 128, 128, 0.0, 0.0, 2, True),
    "w64_disc_norm_relu_eval_k4": (8, 5, True, 64, True, True, 300, 64, 16, 5e-3, 1e-3, 3, False),
    "w32_disc_mb4096": (4, 2, True, 32, False, False, 4500, 4096, 4096, 1e-3, 1e-3, 2, True),
    "w7_box_relu_mb4096_k4": (3, 2, False, 7, True, True, 4200, 4096, 1024, 0.0, 1e-2, 1, True),
}


def _sweep_case(name):
    d_obs, d_act, disc, w, norm, relu, n, bs, mb, ent_w, l2_w, epochs, train = SWEEP[name]
    c = dict(d_obs=d_obs, d_act=d_act, discrete=disc, hidden=w, norm=norm, relu=relu, n=n, bs=bs, mb=mb, n_epochs=epochs,
             log_interval=1, lr=0.0, ent_weight=ent_w, l2_weight=l2_w)
    rng = np.random.default_rng(abs(hash(name)) % 2 ** 31)
    obs = (rng.normal(size=(n, d_obs)) * 1.5 + 0.3).astype(np.float32)
    acts = (rng.integers(0, d_act, size=n) if disc else np.clip(rng.normal(size=(n, d_act)) * 0.6, -1, 1)).astype(
        np.int64 if disc else np.float32)
    th.manual_seed(1)
    pol = _policy(c)
    with th.no_grad():
        pol.action_net.weight.mul_(20.0)
        if not disc:
            pol.log_std.copy_(th.linspace(-0.4, 0.2, d_act))
    params0 = th.cat([p.detach().reshape(-1) for p in pol.parameters()]).numpy()
    norm0 = np.concatenate([rng.normal(size=d_obs) * 0.2, 1.0 + rng.random(d_obs)]).astype(np.float32) if norm else None
    count0 = 50 if norm else 0
    perms = [rng.permutation(n) for _ in range(epochs)]
    return c, obs, acts, params0, norm0, count0, perms, train


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SWEEP))
def test_kernel_matches_float64_port_at_lr0(name, monkeypatch):
    c, obs, acts, params0, norm0, count0, perms, train = _sweep_case(name)
    M = c["n_epochs"] * (c["n"] // c["mb"])
    port = _port_from(c, params0, norm0, count0, lr=0.0)
    grads = []
    logged = port.train(obs, acts, perms, M, log_interval=1, norm_update=train, grads=grads)
    _fixed_perms(monkeypatch, perms)
    trainer = _device_bc(c, params0, obs, acts, norm0, count0, lr=0.0, train_mode=train)
    trainer.train(n_epochs=c["n_epochs"], log_interval=1)
    pol = trainer.policy
    flat, ns, cnt = pol.flat_vectors()
    assert th.equal(flat.cpu(), th.as_tensor(params0, dtype=th.float32))  # lr = 0: bit-unchanged
    n_steps = len(grads)
    assert trainer.adam_steps == n_steps
    # moments = beta-weighted sums of every batch's gradient (+ l2 term, already in the port's grads)
    b1, b2 = 0.9, 0.999
    w1 = np.array([(1 - b1) * b1 ** (n_steps - 1 - s) for s in range(n_steps)])
    w2 = np.array([(1 - b2) * b2 ** (n_steps - 1 - s) for s in range(n_steps)])
    G_ = np.array(grads)
    m_ref, v_ref = w1 @ G_, w2 @ G_ ** 2
    m_abs = w1 @ np.abs(G_)
    m_dev, v_dev = trainer.exp_avg.double().cpu().numpy(), trainer.exp_avg_sq.double().cpu().numpy()
    np.testing.assert_array_less(np.abs(m_dev - m_ref), C_GRAD * m_abs + FLOOR * m_abs.max() + 1e-30)
    np.testing.assert_array_less(np.abs(v_dev - v_ref), 2 * C_GRAD * v_ref + FLOOR ** 2 * v_ref.max() + 1e-30)
    if c["norm"]:
        fn = port.policy.feat_norm
        np.testing.assert_allclose(ns.double().cpu().numpy(), np.concatenate([fn.running_mean.numpy(),
                                                                             fn.running_var.numpy()]), rtol=2e-5,
                                   atol=1e-6)
        assert int(cnt) == int(fn.count) == count0 + (M * c["mb"] if train else 0)
    batches, met = _metrics(trainer)
    assert batches == [b for b, _ in logged]
    ref = np.array([m for _, m in logged])
    np.testing.assert_allclose(met, ref, rtol=C_METRIC, atol=C_METRIC)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w7_disc_relu_accum", "w33_disc_norm_mb32_k4", "w32_box_hc_mb64_eval"])
def test_kernel_matches_float64_port_with_adam_steps(name, monkeypatch):
    c, obs, acts, params0, norm0, count0, perms, train = _sweep_case(name)
    M = c["n_epochs"] * (c["n"] // c["mb"])
    lr = 1e-3
    port = _port_from(c, params0, norm0, count0, lr=lr)
    grads = []
    port.train(obs, acts, perms, M, log_interval=1, norm_update=train, grads=grads)
    _fixed_perms(monkeypatch, perms)
    trainer = _device_bc(c, params0, obs, acts, norm0, count0, lr=lr, train_mode=train)
    trainer.train(n_epochs=c["n_epochs"], log_interval=1)
    got = trainer.policy.flat_vectors()[0].double().cpu().numpy()
    want = bc_port.get_flat(port.policy)
    # Adam moves a parameter by about lr per step whatever its gradient: where a gradient sits at fp32's noise the
    # direction may differ, so those parameters are bounded by the steps taken; every other one by a fraction of lr
    gmax = np.abs(np.array(grads)).max(axis=0)
    noisy = gmax < 1e-4 * gmax.max()
    tol = np.where(noisy, 2 * lr * len(grads), 0.02 * lr * len(grads)) + 1e-6
    np.testing.assert_array_less(np.abs(got - want), tol)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES_GOLDEN)
def test_device_reproduces_golden(name, monkeypatch):
    g, c = _case(_golden(), name)
    _fixed_perms(monkeypatch, list(g["order"]))
    # the recorded order covers the used rows of each epoch; the dropped tail is never read
    trainer = _device_bc(c, g["params0"], g["obs"], g["acts"], norm0=np.concatenate(
        [np.zeros(c["d_obs"]), np.ones(c["d_obs"])]) if c["norm"] else None)
    trainer.train(n_epochs=c["n_epochs"], log_interval=c["log_interval"])
    got = trainer.policy.flat_vectors()[0].cpu().numpy()
    np.testing.assert_allclose(got, g["params"], rtol=1e-3, atol=2e-4)
    batches, met = _metrics(trainer)
    assert batches == list(g["batches"])
    np.testing.assert_allclose(met, g["metrics"], rtol=1e-3, atol=1e-4)
    if c["norm"]:
        np.testing.assert_allclose(trainer.policy.flat_vectors()[1].cpu().numpy(), g["norm"], rtol=1e-5, atol=1e-5)


def _snapshot(trainer):
    flat, ns, cnt = trainer.policy.flat_vectors()
    return [t.clone() for t in (flat, ns, cnt, trainer.exp_avg, trainer.exp_avg_sq, trainer._state)]


@pytest.mark.gpu
def test_split_launches_and_repeats_give_the_same_bits():
    c = dict(d_obs=5, d_act=2, discrete=False, hidden=16, norm=True, relu=False, n=70, bs=24, mb=8, n_epochs=3,
             log_interval=2, lr=1e-3, ent_weight=1e-3, l2_weight=1e-3)
    rng = np.random.default_rng(3)
    obs = rng.normal(size=(70, 5)).astype(np.float32)
    acts = np.clip(rng.normal(size=(70, 2)), -1, 1).astype(np.float32)
    params0 = th.cat([p.detach().reshape(-1) for p in _policy(c).parameters()]).numpy()
    results = []
    for kwargs in (dict(), dict(), dict(on_batch_end=lambda: None), dict(on_epoch_end=lambda: None),
                   dict(on_batch_end=lambda: None, on_epoch_end=lambda: None)):
        th.manual_seed(11)
        trainer = _device_bc(c, params0, obs, acts)
        trainer.train(n_epochs=3, log_interval=2, **kwargs)
        results.append((_snapshot(trainer), _metrics(trainer)))
    for snap, (batches, met) in results[1:]:
        for a, b in zip(results[0][0], snap):
            assert th.equal(a, b)
        assert batches == results[0][1][0] and np.array_equal(met, results[0][1][1])
    # 70 // 8 = 8 minibatches per epoch, k = 3: epochs end mid-batch, the last batch (24 minibatches) is complete
    assert results[0][1][0] == [0, 2, 4, 6]


@pytest.mark.gpu
def test_n_batches_ends_mid_epoch_and_next_train_starts_fresh(monkeypatch):
    c = dict(d_obs=4, d_act=3, discrete=True, hidden=8, norm=False, relu=False, n=50, bs=16, mb=8, n_epochs=1,
             log_interval=1, lr=2e-3, ent_weight=1e-3, l2_weight=0.0)
    rng = np.random.default_rng(4)
    obs = rng.normal(size=(50, 4)).astype(np.float32)
    acts = rng.integers(0, 3, size=50)
    params0 = th.cat([p.detach().reshape(-1) for p in _policy(c).parameters()]).numpy()
    perms = [rng.permutation(50) for _ in range(3)]
    _fixed_perms(monkeypatch, perms)
    trainer = _device_bc(c, params0, obs, acts)
    trainer.train(n_batches=2)  # 4 of the 6 minibatches of epoch 0
    trainer.train(n_batches=4)  # a fresh epoch: all 6 of perms[1], then 2 of perms[2]
    port = _port_from(c, params0)
    port.train(obs, acts, perms[:1], 4)
    port.train(obs, acts, perms[1:], 8)
    got = trainer.policy.flat_vectors()[0].double().cpu().numpy()
    np.testing.assert_allclose(got, bc_port.get_flat(port.policy), rtol=1e-3, atol=2e-4)
    assert trainer.adam_steps == 6


@pytest.mark.gpu
@pytest.mark.parametrize("env", ["cartpole", "pendulum"])
def test_bc_improves_expert_log_likelihood(env):
    from imitation_b200.data import serialize

    trajs = list(serialize.load_with_rewards(os.path.join(G.GOLDEN, "expert_models", f"{env}_0", "rollouts",
                                                          "final.npz")))
    tr = types.flatten_trajectories(trajs)
    obs_space = spaces.Box(-np.inf, np.inf, tr.obs.shape[1:])
    act_space = spaces.Discrete(2) if env == "cartpole" else spaces.Box(-2.0, 2.0, tr.acts.shape[1:])
    th.manual_seed(0)
    trainer = bc_mod.BC(observation_space=obs_space, action_space=act_space, rng=np.random.default_rng(0),
                        demonstrations=trajs, batch_size=64, custom_logger=_Records())

    def neglogp():
        with th.no_grad():
            m = trainer.loss_calculator(trainer.policy, tr.obs[:4000], tr.acts[:4000])
        return float(m.neglogp)

    before = neglogp()
    trainer.train(n_epochs=2, log_interval=100)
    after = neglogp()
    assert math.isfinite(after) and after < before - 0.1, (before, after)
    assert len(trainer.logger.rows) > 0
