"""MCE IRL's host side and its float64 restatement (oracle/mce_port.py), pinned to the reference on the CPU.

tests/golden/mce_irl.npz holds what the reference's own algorithms/mce_irl.py computes over
`oracle.tabular_mdp.random_mdp(5, 3, 2, 10, one-hot, seed 42)` (the reference tests' random MDP shape):
    mdp/*                          the MDP;
    partition/<g>/{V,Q,pi}         mce_partition_fh(discount=g), g in 0, 0.5, 0.99, 1;
    occ_pi/<g>/{D,Dcum}            mce_occupancy_measures(pi=that pi, discount=g);
    occ/<g>/{D,Dcum}               mce_occupancy_measures(discount=g) (planned undiscounted);
    demo/<form>                    MCEIRL(...).demo_state_om for an ndarray, trajectories (discount 0.9 and 1),
                                   Transitions, TransitionsMinimal and an iterable of mappings; demo/warning the
                                   TransitionsMinimal warning; errors/* the reference's error messages;
    policy/*                       TabularPolicy.predict actions and timesteps over a seeded generator;
    run/<name>/*                   MCEIRL.train runs (RUNS): initial parameters, every logged record (keys / values),
                                   the stop iteration, the final parameters and Adam moments, the returned Dcum and
                                   the final pi.
The recorder asserts that every stopping test it records is at least 1 % away from its threshold at the stop
iteration and the one before, so a float32 reordering cannot move the stop.  Re-record it where the reference sources
are importable (oracle/refimport.py) with

    IMB_RECORD_REFERENCE=1 python -m pytest tests/test_mce_irl_reference.py -k reference_records

Where they are importable, the same test regenerates the results and compares them with the stored file.  The device
sweep and trainer are held to oracle/mce_port.py on the GPU in tests/test_mce_irl.py.
"""
import os
import warnings
from types import SimpleNamespace as types_ns
from typing import Any

import numpy as np
import pytest
import torch as th

from imitation_b200.algorithms import mce_irl
from imitation_b200.data import types
from imitation_b200.rewards import reward_nets
from oracle import mce_port, tabular_mdp
from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "mce_irl.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
DISCOUNTS = (0.0, 0.5, 0.99, 1.0)
# name: (hid_sizes, RunningNorm input, discount, linf_eps, grad_l2_eps, max_iter, log_interval, stop reason)
RUNS = {
    "linear_g1_max": ((), False, 1.0, 1e-3, 1e-4, 30, 10, "max_iter"),
    "mlp32_g099_linf": ((32, 32), False, 0.99, 0.1, 1e-4, 400, 4, "linf"),
    "mlp32_g099_grad": ((32, 32), False, 0.99, -1.0, 0.6, 400, 5, "grad"),
    "norm_g1_max": ((16,), True, 1.0, 1e-3, 1e-4, 25, 5, "max_iter"),
    "norm_g0_linf": ((16,), True, 0.0, 1e-3, 1e-4, 20, 1, "linf"),
}


def _mdp():
    return tabular_mdp.random_mdp(5, 3, 2, 10, obs_dim=None, seed=42)


def _trajs(n=6, seed=0, terminal=True):
    rng = np.random.default_rng(seed)
    return [(rng.integers(0, 5, 11), rng.integers(0, 3, 10), terminal) for _ in range(n)]


def _demo_seed_om(mdp):
    _, _, pi = mce_port.partition_fh(mdp.transition_matrix, mdp.reward_matrix, mdp.horizon, 1.0)
    return pi


def _demo_for(mdp, g):
    """The demonstrations of the train runs: the occupancy of the env reward's soft-optimal policy, mixed with the
    initial distribution (so that the runs have work to do)."""
    D = mce_port.occupancy(mdp.transition_matrix, mdp.initial_state_dist, _demo_seed_om(mdp), mdp.horizon, g)[1]
    return 0.8 * D + 0.2 * mdp.initial_state_dist * D.sum()


# ------------------------------------------------------------------------------------------------
# the recorder (reference sources needed)
# ------------------------------------------------------------------------------------------------
_MISSING = object()


def _reference():
    """The reference's modules, and an undo for the names added to the shared shim while they are in use."""
    from oracle import refimport

    refimport.load()
    # names the reference's module and TabularPolicy use that the names-only shim does not carry
    from gymnasium import spaces as gspaces
    from stable_baselines3.common import policies, type_aliases

    def _init(self, observation_space=None, action_space=None, **kwargs):
        th.nn.Module.__init__(self)
        self.observation_space, self.action_space = observation_space, action_space

    def _contains(self, x):
        return np.ndim(x) == 0 and np.issubdtype(np.asarray(x).dtype, np.integer) and self.start <= x < self.start + self.n

    patches = [(type_aliases, "PyTorchObs", Any), (gspaces.Discrete, "contains", _contains),
               (policies.BasePolicy, "__init__", _init)]
    saved = [(obj, name, obj.__dict__.get(name, _MISSING)) for obj, name, _ in patches]
    for obj, name, val in patches:
        setattr(obj, name, val)

    def undo():
        for obj, name, val in saved:
            if val is _MISSING:
                delattr(obj, name)
            else:
                setattr(obj, name, val)

    from imitation.algorithms import mce_irl as ref
    from imitation.data import rollout as ref_rollout
    from imitation.data import types as ref_types
    from imitation.rewards import reward_nets as ref_nets

    return (ref, ref_rollout, ref_types, ref_nets, gspaces), undo


class _RefEnv:
    """oracle.tabular_mdp's MDP with the shim's gymnasium spaces (the reference's TabularPolicy checks them)."""

    def __init__(self, mdp, gspaces):
        self.__dict__.update(transition_matrix=mdp.transition_matrix, observation_matrix=mdp.observation_matrix,
                             initial_state_dist=mdp.initial_state_dist, reward_matrix=mdp.reward_matrix,
                             horizon=mdp.horizon, state_dim=mdp.state_dim, action_dim=mdp.action_dim)
        self.state_space = gspaces.Discrete(mdp.state_dim)
        self.action_space = gspaces.Discrete(mdp.action_dim)
        self.observation_space = gspaces.Box(0.0, 1.0, (mdp.obs_dim,))


class _Log:
    def __init__(self):
        self.keys, self.values, self.dumps = [], [], []

    def record(self, key, val, exclude=None):
        self.keys.append(key)
        self.values.append(float(val))

    def dump(self, step=0):
        self.dumps.append(step)


def _margin_ok(x, eps):
    return eps < 0 or abs(x - eps) >= 0.01 * abs(eps)


def _record() -> dict:
    mods, undo = _reference()
    try:
        return _record_with(*mods)
    finally:
        undo()


def _snapshot(a) -> dict:
    """The trainer's state before an optimiser step: the net's state dict and Adam's moments and step count."""
    out = {"sd/" + k: v.detach().numpy().copy() for k, v in a.reward_net.state_dict().items()}
    for i, q in enumerate(a.reward_net.parameters()):
        st = a.optimizer.state.get(q) or {}
        zeros = np.zeros(tuple(q.shape), dtype=np.float32)
        out[f"adam/{i}/exp_avg"] = st["exp_avg"].numpy().copy() if st else zeros
        out[f"adam/{i}/exp_avg_sq"] = st["exp_avg_sq"].numpy().copy() if st else zeros
        out["adam_step"] = np.int64(float(st["step"]) if st else 0)
    return out


def _record_with(ref, ref_rollout, ref_types, ref_nets, gspaces) -> dict:
    mdp = _mdp()
    env = _RefEnv(mdp, gspaces)
    out = {"mdp/T": mdp.transition_matrix, "mdp/obs": mdp.observation_matrix, "mdp/init": mdp.initial_state_dist,
           "mdp/reward": mdp.reward_matrix, "mdp/horizon": np.int64(mdp.horizon)}
    for g in DISCOUNTS:
        V, Q, pi = ref.mce_partition_fh(env, discount=g)
        out.update({f"partition/{g}/V": V, f"partition/{g}/Q": Q, f"partition/{g}/pi": pi})
        D, Dcum = ref.mce_occupancy_measures(env, pi=pi, discount=g)
        out.update({f"occ_pi/{g}/D": D, f"occ_pi/{g}/Dcum": Dcum})
        D, Dcum = ref.mce_occupancy_measures(env, discount=g)
        out.update({f"occ/{g}/D": D, f"occ/{g}/Dcum": Dcum})

    # demonstration forms
    def algo(demo, discount=1.0):
        net = ref_nets.BasicRewardNet(env.observation_space, env.action_space, use_action=False, hid_sizes=[])
        return ref.MCEIRL(demo, env, net, np.random.default_rng(0), discount=discount)

    trajs = [ref_types.Trajectory(obs=o, acts=a, infos=None, terminal=t) for o, a, t in _trajs()]
    trans = ref_rollout.flatten_trajectories(trajs)
    out["demo/ndarray"] = algo(np.arange(5.0)).demo_state_om
    out["demo/trajs_1"] = algo(trajs).demo_state_om
    out["demo/trajs_09"] = algo(trajs, 0.9).demo_state_om
    out["demo/transitions"] = algo(trans).demo_state_om
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        out["demo/minimal"] = algo(ref_types.TransitionsMinimal(obs=trans.obs, acts=trans.acts,
                                                                infos=trans.infos)).demo_state_om
    out["demo/warning"] = np.array([str(x.message) for x in w if "MCEIRL" in str(x.message)][-1])
    batches = [{"obs": trans.obs[i:i + 16], "dones": trans.dones[i:i + 16], "next_obs": trans.next_obs[i:i + 16]}
               for i in range(0, len(trans), 16)]
    out["demo/mappings"] = algo(batches).demo_state_om
    for name, (demo, g, exc) in {"timeless": (trans, 0.9, ValueError), "type": (object(), 1.0, TypeError)}.items():
        with pytest.raises(exc) as e:
            algo(demo, g)
        out[f"errors/{name}"] = np.array(str(e.value))
    env.horizon = None
    with pytest.raises(ValueError) as e:
        ref.mce_partition_fh(env)
    out["errors/horizon"] = np.array(str(e.value))
    env.horizon = mdp.horizon

    # TabularPolicy draws
    pi = out["partition/0.99/pi"]
    pol = ref.TabularPolicy(env.state_space, env.action_space, pi, np.random.default_rng(9))
    states = np.random.default_rng(4).integers(0, 5, 40)
    acts, (ts,) = pol.predict(states)
    out["policy/states"], out["policy/acts0"], out["policy/ts0"] = states, acts, ts.copy()
    start = np.zeros(40, dtype=bool)
    start[::3] = True
    acts, (ts,) = pol.predict(states, (ts,), start)
    out["policy/start"], out["policy/acts1"], out["policy/ts1"] = start, acts, ts.copy()
    acts, _ = pol.predict(states, (ts,), None, deterministic=True)
    out["policy/acts_det"] = acts

    # train runs
    for name, (hid, norm, g, linf_eps, grad_eps, max_iter, log_interval, why) in RUNS.items():
        th.manual_seed(715298)
        kw = dict(normalize_input_layer=ref_nets.networks.RunningNorm) if norm else {}
        net = ref_nets.BasicRewardNet(env.observation_space, env.action_space, use_action=False, hid_sizes=list(hid),
                                      **kw)
        p = f"run/{name}/"
        for k, v in net.state_dict().items():
            out[p + "init/" + k] = v.numpy().copy()
        log = _Log()
        a = ref.MCEIRL(_demo_for(mdp, g), env, net, np.random.default_rng(0), discount=g, linf_eps=linf_eps,
                       grad_l2_eps=grad_eps, log_interval=log_interval)
        a._logger = log
        out[p + "demo"] = a.demo_state_om
        trace, states, vecs = [], [], []
        real_step = a._train_step

        def step(obs_mat, real_step=real_step, a=a, trace=trace, states=states, vecs=vecs):
            states.append(_snapshot(a))
            r, vis = real_step(obs_mat)
            grads = [q.grad for q in a.reward_net.parameters()]
            trace.append((float(np.max(np.abs(a.demo_state_om - vis))), float(ref.util.tensor_iter_norm(grads))))
            vecs.append((r, (vis - a.demo_state_om).astype(np.float32), vis))
            return r, vis

        a._train_step = step
        Dcum = a.train(max_iter=max_iter)
        stop = len(trace) - 1
        for linf, gn in trace[-2:]:
            assert _margin_ok(linf, linf_eps) and _margin_ok(gn, grad_eps), (name, linf, gn)
        reason = ("max_iter" if stop == max_iter - 1 and trace[-1][0] > linf_eps and trace[-1][1] > grad_eps
                  else "linf" if trace[-1][0] <= linf_eps else "grad")
        assert reason == why, (name, reason)
        out[p + "stop"] = np.int64(stop)
        # per iteration: the reward, the weights, Dcum, linf_delta and grad_norm; the state before the step at a few
        # iterations (teacher forcing: the state at k + 1, or final/ after the stop, is what step k must produce)
        out[p + "trace/reward"] = np.stack([v[0] for v in vecs])
        out[p + "trace/weights"] = np.stack([v[1] for v in vecs])
        out[p + "trace/Dcum"] = np.stack([v[2] for v in vecs])
        out[p + "trace/linf"] = np.array([t_[0] for t_ in trace])
        out[p + "trace/grad_norm"] = np.array([t_[1] for t_ in trace])
        ks = sorted({k for k in (0, 1, 2, stop // 2, stop // 2 + 1, stop - 1, stop) if 0 <= k <= stop})
        out[p + "state_iters"] = np.array(ks, dtype=np.int64)
        for k in ks:
            for key, v in states[k].items():
                out[p + f"state/{k}/{key}"] = v
        out[p + "log_keys"] = np.array(log.keys)
        out[p + "log_values"] = np.array(log.values)
        out[p + "dumps"] = np.array(log.dumps, dtype=np.int64)
        for k, v in net.state_dict().items():
            out[p + "final/" + k] = v.numpy().copy()
        for i, q in enumerate(net.parameters()):
            st = a.optimizer.state[q]
            out[p + f"adam/{i}/exp_avg"] = st["exp_avg"].numpy().copy()
            out[p + f"adam/{i}/exp_avg_sq"] = st["exp_avg_sq"].numpy().copy()
        out[p + "Dcum"] = Dcum
        out[p + "pi"] = a.policy.pi
    return out


def _reference_available() -> bool:
    from oracle import refimport

    return refimport.available()


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources")
def test_reference_records_match_golden():
    got = _record()
    if RECORD:
        np.savez_compressed(STORE, **got)
    z = np.load(STORE)
    assert sorted(z.files) == sorted(got)
    for k in z.files:
        np.testing.assert_array_equal(z[k], got[k], err_msg=k)


# ------------------------------------------------------------------------------------------------
# this package and the port against the golden (no reference needed)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(STORE)


def test_port_sweep_matches_golden(golden):
    T, init, r, H = golden["mdp/T"], golden["mdp/init"], golden["mdp/reward"], int(golden["mdp/horizon"])
    for g in DISCOUNTS:
        for got, k in zip(mce_port.partition_fh(T, r, H, g), "V Q pi".split()):
            np.testing.assert_array_equal(got, golden[f"partition/{g}/{k}"])
        for got, k in zip(mce_port.occupancy(T, init, golden[f"partition/{g}/pi"], H, g), ("D", "Dcum")):
            np.testing.assert_array_equal(got, golden[f"occ_pi/{g}/{k}"])
        _, _, pi1 = mce_port.partition_fh(T, r, H, 1.0)
        for got, k in zip(mce_port.occupancy(T, init, pi1, H, g), ("D", "Dcum")):
            np.testing.assert_array_equal(got, golden[f"occ/{g}/{k}"])


def test_mdp_builder_matches_golden(golden):
    mdp = _mdp()
    np.testing.assert_array_equal(mdp.transition_matrix, golden["mdp/T"])
    np.testing.assert_array_equal(mdp.observation_matrix, golden["mdp/obs"])


def _algo(demo, discount=1.0):
    mdp = _mdp()
    net = reward_nets.BasicRewardNet(mdp.observation_space, mdp.action_space, use_action=False, hid_sizes=[])
    return mce_irl.MCEIRL(demo, mdp, net, np.random.default_rng(0), discount=discount)


def test_demonstration_forms_match_golden(golden):
    trajs = [types.Trajectory(obs=o, acts=a, infos=None, terminal=t) for o, a, t in _trajs()]
    trans = types.flatten_trajectories(trajs)
    np.testing.assert_array_equal(_algo(np.arange(5.0)).demo_state_om, golden["demo/ndarray"])
    np.testing.assert_array_equal(_algo(trajs).demo_state_om, golden["demo/trajs_1"])
    np.testing.assert_array_equal(_algo(trajs, 0.9).demo_state_om, golden["demo/trajs_09"])
    np.testing.assert_array_equal(_algo(trans).demo_state_om, golden["demo/transitions"])
    with pytest.warns(UserWarning) as w:
        om = _algo(types.TransitionsMinimal(obs=trans.obs, acts=trans.acts, infos=trans.infos)).demo_state_om
    np.testing.assert_array_equal(om, golden["demo/minimal"])
    assert [str(x.message) for x in w if "MCEIRL" in str(x.message)] == [str(golden["demo/warning"])]
    batches = [{"obs": trans.obs[i:i + 16], "dones": trans.dones[i:i + 16], "next_obs": trans.next_obs[i:i + 16]}
               for i in range(0, len(trans), 16)]
    np.testing.assert_array_equal(_algo(batches).demo_state_om, golden["demo/mappings"])
    with pytest.raises(ValueError) as e:
        _algo(trans, 0.9)
    assert str(e.value) == str(golden["errors/timeless"])
    with pytest.raises(TypeError) as e:
        _algo(object())
    assert str(e.value) == str(golden["errors/type"]).replace("builtins.", "")  # type repr of `object`
    mdp = _mdp()
    mdp.horizon = None
    with pytest.raises(ValueError) as e:
        mce_irl.mce_partition_fh(mdp)
    assert str(e.value) == str(golden["errors/horizon"])


def test_tabular_policy_matches_golden(golden):
    mdp = _mdp()
    pol = mce_irl.TabularPolicy(mdp.state_space, mdp.action_space, golden["partition/0.99/pi"],
                                np.random.default_rng(9))
    states = golden["policy/states"]
    acts, (ts,) = pol.predict(states)
    np.testing.assert_array_equal(acts, golden["policy/acts0"])
    np.testing.assert_array_equal(ts, golden["policy/ts0"])
    acts, (ts,) = pol.predict(states, (ts,), golden["policy/start"])
    np.testing.assert_array_equal(acts, golden["policy/acts1"])
    np.testing.assert_array_equal(ts, golden["policy/ts1"])
    acts, _ = pol.predict(states, (ts,), None, deterministic=True)
    np.testing.assert_array_equal(acts, golden["policy/acts_det"])
    with pytest.raises(AssertionError, match="policy not normalized"):
        pol.set_pi(np.ones((2, 5, 3)))


@pytest.mark.parametrize("name", list(RUNS))
def test_port_train_runs_match_golden(golden, name):
    """oracle/mce_port.py's iteration, looped as MCEIRL.train loops it, replays the reference's recorded runs: the
    same stop iteration, logged keys and values, final parameters, Dcum and pi (the same torch-CPU ops)."""
    hid, norm, g, linf_eps, grad_eps, max_iter, log_interval, _ = RUNS[name]
    p = f"run/{name}/"
    mdp = _mdp()
    net = mce_port.port_net(mdp.obs_dim, hid, norm, G.sub(golden, p + "init"))
    opt = th.optim.Adam(net.parameters(), lr=1e-2)
    obs = th.as_tensor(mdp.observation_matrix, dtype=th.float32)
    keys, values = [], []
    for t in range(max_iter):
        st = mce_port.train_iteration(net, opt, obs, mdp.transition_matrix, mdp.initial_state_dist, mdp.horizon,
                                      _demo_for(mdp, g), g)
        if t % log_interval == 0:
            keys += ["iteration", "linf_delta", "weight_norm", "grad_norm"]
            values += [t, st["linf_delta"], mce_port.tensor_iter_norm([q.detach() for q in net.parameters()]),
                       st["grad_norm"]]
        if st["linf_delta"] <= linf_eps or st["grad_norm"] <= grad_eps:
            break
    assert t == int(golden[p + "stop"])
    assert keys == list(golden[p + "log_keys"])
    np.testing.assert_allclose(values, golden[p + "log_values"], rtol=1e-6, atol=1e-7)
    for k, v in net.state_dict().items():
        np.testing.assert_allclose(v.numpy(), golden[p + "final/" + k], rtol=1e-5, atol=1e-7, err_msg=k)
    np.testing.assert_allclose(st["Dcum"], golden[p + "Dcum"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(mce_port.final_policy(mdp.transition_matrix, st["reward"], mdp.horizon, g),
                               golden[p + "pi"], rtol=1e-9, atol=1e-12)


def test_refusals():
    """What the device trainer does not run raises NotImplementedError at construction, as BC's refusals do."""
    mdp = _mdp()
    demo = np.ones(5)

    def net(**kw):
        return reward_nets.BasicRewardNet(mdp.observation_space, mdp.action_space, **kw)

    rng = np.random.default_rng(0)
    lin = dict(use_action=False, hid_sizes=[])
    cases = [dict(reward_net=net(**lin), optimizer_cls=th.optim.SGD, optimizer_kwargs={"lr": 0.1}),
             dict(reward_net=net(**lin), optimizer_kwargs={"lr": 0.1, "betas": (0.8, 0.999)}),
             dict(reward_net=net(**lin), optimizer_kwargs={"lr": 0.1, "amsgrad": True}),
             dict(reward_net=net(**lin), optimizer_kwargs={"lr": 0.1, "weight_decay": 0.1}),
             dict(reward_net=net(hid_sizes=[]))]  # uses the action
    for kw in cases:
        with pytest.raises(NotImplementedError):
            mce_irl.MCEIRL(demo, mdp, rng=rng, **kw)
    with pytest.raises(NotImplementedError):  # wider than the fused kernels take
        net(use_action=False, hid_sizes=[128])
    big = types_ns(state_dim=5000, action_dim=2, horizon=3)  # rejected from its dimensions, before any array is read
    with pytest.raises(NotImplementedError, match="4096"):
        mce_irl.mce_partition_fh(big)
    with pytest.raises(NotImplementedError, match="4096"):
        mce_irl.mce_occupancy_measures(big)
    mdp.horizon = None
    with pytest.raises(ValueError, match="Only finite-horizon"):
        mce_irl.MCEIRL(None, mdp, net(**lin), rng)


def test_shape_errors_before_upload():
    """The sweep reads raw device pointers, so every array the env or the caller hands it is checked on the host first:
    a wrong shape raises ValueError (as the reference's NumPy fails) instead of being read out of bounds."""
    mdp = _mdp()
    S, A, H = 5, 3, 10
    bad_env = {"transition_matrix": np.ones((S, A, S - 1)), "initial_state_dist": np.ones(S + 1),
               "reward_matrix": np.ones((S, A))}
    for attr, val in bad_env.items():
        env = _mdp()
        setattr(env, attr, val)
        with pytest.raises(ValueError, match=attr.replace("_matrix", "") if attr == "reward_matrix" else attr):
            mce_irl.mce_partition_fh(env)
        with pytest.raises(ValueError):
            mce_irl.mce_occupancy_measures(env)
    with pytest.raises(ValueError, match="reward"):
        mce_irl.mce_partition_fh(mdp, reward=np.ones(S + 2))
    with pytest.raises(ValueError, match="reward"):
        mce_irl.mce_occupancy_measures(mdp, reward=np.ones(S - 1))
    for shape in ((H - 1, S, A), (H, S + 1, A), (H, S, A - 1)):
        with pytest.raises(ValueError, match="pi"):
            mce_irl.mce_occupancy_measures(mdp, pi=np.full(shape, 1.0 / A))


def test_train_needs_an_iteration():
    algo = _algo(np.ones(5))
    with pytest.raises(ValueError, match="max_iter"):
        algo.train(max_iter=0)
