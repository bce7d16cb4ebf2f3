"""The ensemble relabel of an agent's rollout, pinned to the reference: `RewardVecEnvWrapper(BufferingWrapper(venv),
AddSTDRewardWrapper(RewardEnsemble(members), alpha).predict_processed)` (reference rewards/reward_wrapper.py:40-133,
rewards/reward_nets.py:926-989 and :1045-1080), and the same with a bare `RewardEnsemble` (the mean alone).

tests/golden/ensemble_relabel.npz holds what the reference's own wrappers record on the host synthetic environment
(oracle/synth_env.py) with seeded actions and a horizon shorter than the rollout, so that the terminal-observation fix
is exercised: per-step rewards, observations and dones, and every member's state before and after.  Two ensembles:

    box       obs 11, act 3: five NormalizedRewardNet(BasicRewardNet) members with advanced output statistics, alpha -0.5
    discrete  obs 4, 3 actions: three BasicRewardNets with input RunningNorms, bare RewardEnsemble

Re-record them where the reference sources are importable (oracle/refimport.py) with

    IMB_RECORD_REFERENCE=1 python -m pytest tests/test_ensemble_relabel_reference.py -k reference_records

Where they are importable, the same test regenerates the results and compares them with the stored file.
`ensemble_relabel_port` below is the CPU restatement, built from the oracle's reward-net and output-norm ports; it is
held to the stored file here, and tests/test_ensemble_relabel.py holds the device rollout to it.
"""
import os

import numpy as np
import pytest
import torch as th

from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "ensemble_relabel.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
E, T, H = 6, 9, 4
# name: (d_obs, n_actions | None, d_act (one-hot width), members, output norm, input norm, alpha | None = bare ensemble)
CONFIGS = {
    "box": (11, None, 3, 5, True, False, -0.5),
    "discrete": (4, 3, 3, 3, False, True, None),
}


def ensemble_relabel_port(members, alpha, n_actions=None):
    """reward_fn(obs, acts, next_obs, dones) of AddSTDRewardWrapper(RewardEnsemble).predict_processed over oracle
    members (BasicRewardNetPort, OutputNormPort | None): every member's predict_processed in member order (a
    NormalizedRewardNet member normalises with its statistics as they stand, then merges the batch), mean over the
    members plus alpha * the ddof-1 standard deviation; alpha None = RewardEnsemble.predict_processed, the mean alone."""
    from oracle import nets_port

    def reward_fn(obs, acts, next_obs, dones):
        vals = []
        for net, out in members:
            raw = nets_port.predict_port(net, obs, acts, next_obs, dones, n_actions)
            vals.append(out(raw) if out is not None else raw)
        v = np.stack(vals, -1)
        mean = v.mean(-1)
        return mean if alpha is None else mean + alpha * np.sqrt(v.var(-1, ddof=1))

    return reward_fn


# ------------------------------------------------------------------------------------------------
# recording (reference only)
# ------------------------------------------------------------------------------------------------
def _record_config(name, cfg, seed):
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

    Do, n_act, Da, M, out_norm, in_norm, alpha = cfg
    rng = np.random.default_rng(seed)
    th.manual_seed(seed)
    spec = synth_env.SynthEnvSpec(Do, n_act or Da, discrete=n_act is not None, horizon=H, seed=seed)
    venv = HostVenv(synth_env.SynthVecEnv(spec, E, spaces_mod=spaces))
    obs_space, act_space = venv.observation_space, venv.action_space
    members = []
    for _ in range(M):
        kw = dict(normalize_input_layer=ref_networks.RunningNorm) if in_norm else {}
        net = ref_nets.BasicRewardNet(obs_space, act_space, **kw)
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
    reward = ens if alpha is None else ref_nets.AddSTDRewardWrapper(ens, default_alpha=alpha)
    out = {}
    for k, m in enumerate(members):
        out.update({f"member{k}/{key}": v.detach().numpy().copy() for key, v in m.state_dict().items()})
    wrapped = ref_rw.RewardVecEnvWrapper(ref_wrappers.BufferingWrapper(venv), reward.predict_processed)
    acts, rews, obs_l, dones_l = [], [], [], []
    for _ in range(T):
        a = (rng.integers(0, n_act, E) if n_act else rng.uniform(-1.2, 1.2, (E, Da)).astype(np.float32))
        o, r, d, _infos = wrapped.step(a)
        acts.append(a), rews.append(r), obs_l.append(o), dones_l.append(d)
    assert np.stack(dones_l).any(), "no episode ended: lower the horizon"
    out.update(acts=np.stack(acts), rews=np.stack(rews), obs=np.stack(obs_l), dones=np.stack(dones_l))
    for k, m in enumerate(members):
        out.update({f"member_after{k}/{key}": v.detach().numpy().copy() for key, v in m.state_dict().items()})
    return {f"{name}/{k}": v for k, v in out.items()}


def _reference_available() -> bool:
    from oracle import refimport

    return refimport.available()


def _record_all():
    rng_state = th.get_rng_state()
    try:
        out = {}
        for i, (name, cfg) in enumerate(CONFIGS.items()):
            out.update(_record_config(name, cfg, 41 + 10 * i))
        return out
    finally:
        th.set_rng_state(rng_state)


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_golden_is_what_the_reference_records():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead).
    Observations, actions, dones and counts must be identical; floats may differ in the last bits on another CPU."""
    out = _record_all()
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = G.load("ensemble_relabel")
    assert set(z.files) == set(out)
    for k, v in out.items():
        if np.issubdtype(np.asarray(v).dtype, np.floating) and not k.endswith(("/obs", "/acts")):
            np.testing.assert_allclose(v, z[k], rtol=1e-6, atol=1e-7, err_msg=k)
        else:
            np.testing.assert_array_equal(v, z[k], err_msg=k)


# ------------------------------------------------------------------------------------------------
# the CPU restatement against the stored file
# ------------------------------------------------------------------------------------------------
def _port_members(g, name, cfg, prefix="member"):
    from oracle import nets_port

    Do, n_act, Da, M, out_norm, in_norm, _ = cfg
    members = []
    for k in range(M):
        st = G.sub(g, f"{name}/{prefix}{k}")
        net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=(32, 32), normalize_input=in_norm)
        net.load_state_dict({kk.replace("_base.", ""): th.as_tensor(np.array(v)) for kk, v in st.items()
                             if not kk.startswith("normalize_output_layer.")})
        net.eval()
        out = None
        if out_norm:
            out = nets_port.OutputNormPort()
            out.norm.running_mean.copy_(th.as_tensor(st["normalize_output_layer.running_mean"]))
            out.norm.running_var.copy_(th.as_tensor(st["normalize_output_layer.running_var"]))
            out.norm.count.fill_(int(st["normalize_output_layer.count"]))
        members.append((net, out))
    return members


@pytest.mark.parametrize("name", list(CONFIGS))
def test_port_matches_reference_golden(name):
    from oracle import data_port, synth_env

    cfg = CONFIGS[name]
    Do, n_act, Da, M, out_norm, in_norm, alpha = cfg
    z = G.load("ensemble_relabel")
    seed = 41 + 10 * list(CONFIGS).index(name)
    members = _port_members(z, name, cfg)
    spec = synth_env.SynthEnvSpec(Do, n_act or Da, discrete=n_act is not None, horizon=H, seed=seed)
    wrapped = data_port.RewardRelabelPort(data_port.BufferingPort(synth_env.SynthVecEnv(spec, E)),
                                          ensemble_relabel_port(members, alpha, n_act))
    assert z[f"{name}/dones"].any() and not z[f"{name}/dones"].all()
    for t in range(T):
        o, r, d, _infos = wrapped.step(z[f"{name}/acts"][t])
        np.testing.assert_array_equal(d, z[f"{name}/dones"][t])
        np.testing.assert_array_equal(o, z[f"{name}/obs"][t])
        np.testing.assert_allclose(r, z[f"{name}/rews"][t], rtol=2e-6, atol=2e-6, err_msg=f"rewards of step {t}")
    # every member's state afterwards: parameters and input norms unchanged (eval mode), output statistics advanced
    # by E rewards per step
    after = _port_members(z, name, cfg, prefix="member_after")
    for (net, out), (net_a, out_a) in zip(members, after):
        for (ka, a), (_, b) in zip(net.state_dict().items(), net_a.state_dict().items()):
            np.testing.assert_array_equal(a.numpy(), b.numpy(), err_msg=ka)
        if out is not None:
            np.testing.assert_allclose([out.norm.running_mean.item(), out.norm.running_var.item()],
                                       [out_a.norm.running_mean.item(), out_a.norm.running_var.item()], rtol=1e-6)
            assert int(out.norm.count) == int(out_a.norm.count)
    if out_norm:
        before = _port_members(z, name, cfg)
        assert all(int(oa.norm.count) == int(ob.norm.count) + E * T for (_, oa), (_, ob) in zip(after, before))
