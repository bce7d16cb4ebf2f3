"""Time `BC.train(n_epochs=...)` on the device against a torch-eager restatement of the same BC loop on the same GPU.

    python profiles/bc_bench.py [--epochs E] [--repeats R] [--out DIR]

Workloads (demonstrations synthetic and seeded):
  half_cheetah  the tuned bc_seals_half_cheetah configuration (scripts/config/tuned_hps): 17 obs, 6-act Box,
                FeedForward32Policy with NormalizeFeaturesExtractor(RunningNorm), batch 64, lr 0.00806,
                l2_weight 0.00573, ent_weight 1e-3; 100 000 demonstration rows
  cartpole      4 obs, Discrete(2), FeedForward32Policy, batch 32, default lr / l2 / ent; 20 000 rows
The device number is one `train(n_epochs=E)` call (one launch of k_ppo_update_gen with the BC loss), timed by a host
clock around it that ends in a device synchronise; the eager number is the reference's loop in torch ops on the same
GPU (evaluate_actions, the loss, backward, torch Adam with foreach) over the same number of minibatches.  Both report
optimiser steps/s and demonstration rows/s (rows = steps x batch size), median over --repeats after one warm-up run.
Prints one JSON line per workload with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {  # name: (d_obs, d_act, discrete, norm, batch, lr, l2_weight, rows)
    "half_cheetah": (17, 6, False, True, 64, 0.008056922426724927, 0.005728455628518169, 100_000),
    "cartpole": (4, 2, True, False, 32, 1e-3, 0.0, 20_000),
}


def _card():
    name = th.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _demos(d_obs, d_act, discrete, n, seed=0):
    from imitation_b200.data import types

    rng = np.random.default_rng(seed)
    obs = rng.normal(size=(n, d_obs)).astype(np.float32)
    acts = rng.integers(0, d_act, size=n) if discrete else np.clip(rng.normal(size=(n, d_act)), -1, 1).astype(np.float32)
    return types.TransitionsMinimal(obs=obs, acts=acts, infos=np.array([{}] * n))


def _spaces(d_obs, d_act, discrete):
    from imitation_b200 import spaces

    return spaces.Box(-np.inf, np.inf, (d_obs,)), spaces.Discrete(d_act) if discrete else spaces.Box(-1, 1, (d_act,))


def _policy(d_obs, d_act, discrete, norm):
    from imitation_b200.policies.base import FeedForward32Policy

    obs_space, act_space = _spaces(d_obs, d_act, discrete)
    return FeedForward32Policy(obs_space, act_space, normalize_features=norm).cuda()


def device_run(w, epochs):
    from imitation_b200.algorithms import bc
    from imitation_b200.util import logger

    d_obs, d_act, discrete, norm, batch, lr, l2, n = w
    th.manual_seed(0)
    obs_space, act_space = _spaces(d_obs, d_act, discrete)
    trainer = bc.BC(observation_space=obs_space, action_space=act_space, rng=np.random.default_rng(0),
                    policy=_policy(d_obs, d_act, discrete, norm), demonstrations=_demos(d_obs, d_act, discrete, n),
                    batch_size=batch, optimizer_kwargs=dict(lr=lr), l2_weight=l2, custom_logger=logger.configure())
    th.cuda.synchronize()
    t0 = time.perf_counter()
    trainer.train(n_epochs=epochs, log_interval=500)
    th.cuda.synchronize()
    return time.perf_counter() - t0, trainer.adam_steps


def eager_run(w, epochs):
    """The reference's BC.train loop (bc.py:481-510, minibatch = batch) in torch ops on the GPU."""
    d_obs, d_act, discrete, norm, batch, lr, l2, n = w
    th.manual_seed(0)
    pol = _policy(d_obs, d_act, discrete, norm)
    demos = _demos(d_obs, d_act, discrete, n)
    obs = th.as_tensor(demos.obs).cuda()
    acts = th.as_tensor(np.asarray(demos.acts, dtype=np.float32)).cuda()
    opt = th.optim.Adam(pol.parameters(), lr=lr)
    loader = th.utils.data.DataLoader(range(n), batch_size=batch, shuffle=True, drop_last=True)
    steps = 0
    th.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(epochs):
        for idx in loader:
            idx = idx.cuda(non_blocking=True)
            _, logp, ent = pol.evaluate_actions(obs[idx], acts[idx])
            l2_norm = sum(th.sum(th.square(p)) for p in pol.parameters()) / 2
            loss = -logp.mean() - 1e-3 * ent.mean() + l2 * l2_norm
            opt.zero_grad()
            loss.backward()
            opt.step()
            steps += 1
    th.cuda.synchronize()
    return time.perf_counter() - t0, steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("bc_bench needs a GPU")
    card, power = _card()
    results = []
    for name, w in WORKLOADS.items():
        batch = w[4]
        dev, eag = [], []
        device_run(w, 1)
        eager_run(w, 1)
        for _ in range(args.repeats):  # alternate the two within every repeat
            dev.append(device_run(w, args.epochs))
            eag.append(eager_run(w, args.epochs))
        dt, ds = sorted(dev)[len(dev) // 2]
        et, es = sorted(eag)[len(eag) // 2]
        r = {"workload": name, "card": card, "power_limit": power, "epochs": args.epochs, "batch": batch,
             "rows": w[7], "device_steps": ds, "device_s": round(dt, 4), "device_steps_per_s": round(ds / dt, 1),
             "device_rows_per_s": round(ds * batch / dt, 1), "eager_steps": es, "eager_s": round(et, 4),
             "eager_steps_per_s": round(es / et, 1), "eager_rows_per_s": round(es * batch / et, 1),
             "speedup": round((ds / dt) / (es / et), 2)}
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bc_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
