"""Device time of one generator round at BASELINE config 5's agent shape, tanh towers against ReLU towers: Hopper-shaped
obs 11 / act 3, MlpPolicy 64x64 with NormalizeFeaturesExtractor (RunningNorm), 8 envs x 256 steps (n_steps * E = 2048),
PPO minibatch 512, 20 epochs (the seals_hopper named config of train_preference_comparisons.py; its ReLU towers are
`activation_fn=nn.ReLU`).  Two phases, timed separately:

    rollout   DevicePPO.collect_rollouts (imb_rollout + GAE + state advance; environment reward)
    update    DevicePPO.train (imb_ppo_update: k_ppo_update_gen<2, tanh> / <2, relu>, 80 optimiser steps)

    python profiles/relu_policy_bench.py [--steps K] [--warmup W]

Each timed call is bracketed by CUDA events; tanh and ReLU alternate within every repeat so that they share the same
machine conditions.  Prints one JSON line with the median and minimum per activation and phase (ms) and the card's name
and power limit, read in the same run."""
import json
import os
import subprocess
import sys

import numpy as np
import torch as th
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Do, Da, E, T, MB, EPOCHS = 11, 3, 8, 256, 512, 20


def _card():
    name = th.cuda.get_device_name() if th.cuda.is_available() else None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _algo(activation_fn):
    from imitation_b200.algorithms import ppo
    from imitation_b200.envs import synth
    from imitation_b200.policies import base as policies
    from imitation_b200.util import networks

    th.manual_seed(0)
    venv = synth.DeviceVecEnv(Do, Da, E, horizon=1000, seed=3)
    kw = dict(net_arch=dict(pi=[64, 64], vf=[64, 64]), activation_fn=activation_fn,
              features_extractor_class=policies.NormalizeFeaturesExtractor,
              features_extractor_kwargs=dict(normalize_class=networks.RunningNorm))
    return ppo.DevicePPO("MlpPolicy", venv, n_steps=T, batch_size=MB, n_epochs=EPOCHS, seed=0, policy_kwargs=kw)


def _timed(fn):
    a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main(args):
    if not th.cuda.is_available():
        raise SystemExit("relu_policy_bench needs a CUDA device")
    from imitation_b200 import _lib

    _lib.lib()
    acts = {"tanh": nn.Tanh, "relu": nn.ReLU}
    algos = {k: _algo(a) for k, a in acts.items()}
    for _ in range(args.warmup):
        for a in algos.values():
            a.collect_rollouts()
            a.train()
    th.cuda.synchronize()
    times = {f"{k}_{ph}": [] for k in acts for ph in ("rollout", "update")}
    for _ in range(args.steps):
        for k, a in algos.items():
            times[f"{k}_rollout"].append(_timed(a.collect_rollouts))
            times[f"{k}_update"].append(_timed(a.train))
    name, power = _card()
    res = {"bench": "relu_policy", "obs": Do, "act": Da, "width": 64, "envs": E, "n_steps": T, "batch_size": MB,
           "n_epochs": EPOCHS, "repeats": args.steps, "card": name, "power_limit": power}
    for k, v in times.items():
        res[f"{k}_ms_median"] = round(float(np.median(v)), 4)
        res[f"{k}_ms_min"] = round(float(np.min(v)), 4)
    for ph in ("rollout", "update"):
        res[f"relu_over_tanh_{ph}"] = round(res[f"relu_{ph}_ms_median"] / res[f"tanh_{ph}_ms_median"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    import argparse

    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    main(p.parse_args())
