"""Import the REAL reference's `imitation.algorithms.bc` through the names-only shim (oracle/refimport.py), and record
tests/golden/bc.npz from its own BC.train.

TEST INFRASTRUCTURE; only usable where the reference sources are present.  That module needs two
names the shim does not carry: the `stable_baselines3.common.torch_layers` module (FlattenExtractor, CombinedExtractor,
BaseFeaturesExtractor; BC names them only to build its default policy, which the recorder does not use) and
`stable_baselines3.common.utils.get_device`.  `load()` attaches them to the shim's modules in this process, then
imports the reference's module.  The recorder trains oracle.ppo_port.ActorCriticPort (fp32, with the
observation_space / action_space / device attributes BC reads) and records the DataLoader's index order by wrapping the
dataset's __getitem__.

    python -m oracle.bc_ref    # rewrites tests/golden/bc.npz
"""
import os
import sys
import types

import numpy as np
import torch as th

from . import refimport

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "bc.npz")


def get_device(device="auto"):
    """stable_baselines3.common.utils.get_device: "auto" is CUDA when available (the recorder passes "cpu")."""
    if device == "auto":
        device = "cuda" if th.cuda.is_available() else "cpu"
    return th.device(device)


def load():
    refimport.load()
    import stable_baselines3.common as sb3_common
    from stable_baselines3.common import utils

    if not hasattr(sb3_common, "torch_layers"):
        tl = types.ModuleType("stable_baselines3.common.torch_layers")
        for name in ("BaseFeaturesExtractor", "FlattenExtractor", "CombinedExtractor"):
            setattr(tl, name, type(name, (th.nn.Module,), {}))
        sb3_common.torch_layers = tl
        sys.modules["stable_baselines3.common.torch_layers"] = tl
    if not hasattr(utils, "get_device"):
        utils.get_device = get_device
    from imitation.algorithms import bc

    return bc


# name: (d_obs, d_act, discrete, hidden, feature norm, relu, N, batch_size, minibatch_size, lr, ent_weight, l2_weight,
#        n_epochs, log_interval)
CASES = {
    "box_norm": (5, 3, False, 8, True, False, 100, 16, 16, 3e-3, 1e-3, 0.0, 3, 1),
    "box_plain_accum_l2": (4, 2, False, 8, False, False, 90, 32, 8, 1e-3, 1e-2, 1e-3, 3, 3),
    "discrete": (4, 3, True, 8, False, False, 70, 8, 8, 1e-3, 1e-3, 0.0, 2, 3),
    "discrete_norm_relu_accum": (3, 2, True, 6, True, True, 75, 24, 8, 2e-3, 0.0, 1e-2, 2, 1),
}


def _demos(rng, d_obs, d_act, discrete, n):
    obs = rng.normal(size=(n, d_obs)).astype(np.float32) * 2.0 + 0.5
    if discrete:
        acts = rng.integers(0, d_act, size=n).astype(np.int64)
    else:
        acts = np.clip(rng.normal(size=(n, d_act)) * 0.7, -1, 1).astype(np.float32)
    return obs, acts


def record_case(name, seed=0):
    bc = load()
    from gymnasium import spaces as gspaces
    from imitation.data import types as rtypes

    from .bc_port import get_flat, make_policy

    d_obs, d_act, discrete, hidden, norm, relu, n, bs, mb, lr, ent_w, l2_w, n_epochs, log_iv = CASES[name]
    rng = np.random.default_rng(seed)
    obs, acts = _demos(rng, d_obs, d_act, discrete, n)
    th.manual_seed(seed)
    pol = make_policy(d_obs, d_act, discrete, hidden, norm, relu, dtype=th.float32)
    if pol.log_std is not None:
        with th.no_grad():
            pol.log_std.copy_(th.linspace(-0.5, 0.3, d_act))
    with th.no_grad():  # a larger head than SB3's 0.01 gain, so that the actions' log-likelihood moves
        pol.action_net.weight.mul_(30.0)
    obs_space = gspaces.Box(-np.inf, np.inf, (d_obs,), np.float32)
    act_space = gspaces.Discrete(d_act) if discrete else gspaces.Box(-1.0, 1.0, (d_act,), np.float32)
    pol.observation_space, pol.action_space, pol.device = obs_space, act_space, th.device("cpu")
    params0 = get_flat(pol)
    order = []

    class Recorded(rtypes.Transitions):
        def __getitem__(self, key):
            if isinstance(key, (int, np.integer)):
                order.append(int(key))
            return super().__getitem__(key)

    demos = Recorded(obs=obs, acts=acts, infos=np.array([{}] * n), next_obs=obs.copy(), dones=np.zeros(n, dtype=bool))
    records = []

    class Logger:
        def record(self, key, val, exclude=None):
            records.append((key, val))

        def dump(self, step=0):
            pass

    trainer = bc.BC(observation_space=obs_space, action_space=act_space, rng=np.random.default_rng(seed), policy=pol,
                    demonstrations=demos, batch_size=bs, minibatch_size=mb, optimizer_kwargs=dict(lr=lr),
                    ent_weight=ent_w, l2_weight=l2_w, device="cpu", custom_logger=Logger())
    trainer._bc_logger = bc.BCLogger(Logger())
    order.clear()  # (set_demonstrations reads the first item)
    trainer.train(n_epochs=n_epochs, log_interval=log_iv, progress_bar=False)
    per_epoch = n // mb
    used = per_epoch * mb
    order = np.asarray(order, dtype=np.int64).reshape(n_epochs, used)
    metrics, batches = [], []
    cur = {}
    for key, val in records:
        cur[key] = val
        if key == "bc/loss":
            batches.append(cur["bc/batch"])
            metrics.append([float(cur[f"bc/{m}"]) for m in
                            ("neglogp", "entropy", "ent_loss", "prob_true_act", "l2_norm", "l2_loss", "loss")])
    out = {"config": np.asarray([d_obs, d_act, int(discrete), hidden, int(norm), int(relu), n, bs, mb, n_epochs,
                                 log_iv], dtype=np.int64),
           "hparams": np.asarray([lr, ent_w, l2_w], dtype=np.float64),
           "obs": obs, "acts": acts, "params0": params0, "order": order, "params": get_flat(pol),
           "metrics": np.asarray(metrics, dtype=np.float64).reshape(-1, 7),
           "batches": np.asarray(batches, dtype=np.int64)}
    if norm:
        out["norm"] = np.concatenate([pol.feat_norm.running_mean.numpy(), pol.feat_norm.running_var.numpy()])
        out["count"] = np.asarray(int(pol.feat_norm.count))
    return out


def record(path=GOLDEN):
    arrays = {}
    for name in CASES:
        for k, v in record_case(name).items():
            arrays[f"{name}/{k}"] = v
    np.savez_compressed(path, **arrays)
    return path


if __name__ == "__main__":
    print(record())
