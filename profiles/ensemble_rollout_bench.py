"""Device time of one `DevicePPO.collect_rollouts` (rollout + reward relabel + GAE + state advance) at BASELINE config
5's shapes: Hopper-shaped obs 11 / act 3, 8 envs x 256 steps (`rl.batch_size` 2048), FeedForward32Policy, reward
members `BasicRewardNet` 32x32.  Three reward settings:

    single      BasicRewardNet                                          (imb_rollout, reward column written in place)
    normalized  NormalizedRewardNet(BasicRewardNet)                     (imb_rollout + imb_reward_norm_scan)
    ensemble    AddSTDRewardWrapper(RewardEnsemble(5 x NormalizedRewardNet(BasicRewardNet)), alpha = -0.5)
                                                                        (imb_rollout_ensemble + imb_ensemble_relabel)

    python profiles/ensemble_rollout_bench.py [--steps K] [--warmup W] [--envs E] [--n-steps T]

Each timed call is bracketed by CUDA events; the settings alternate within every repeat so that they share the same
machine conditions.  Prints one JSON line with the median and minimum per setting (ms) and the card's name and power
limit, read in the same run."""
import json
import os
import subprocess
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Do, Da, M, ALPHA = 11, 3, 5, -0.5


def _card():
    name = th.cuda.get_device_name() if th.cuda.is_available() else None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _setting(kind, E, T):
    from imitation_b200.algorithms import ppo
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, reward_wrapper
    from imitation_b200.util import networks

    th.manual_seed(0)
    venv = synth.DeviceVecEnv(Do, Da, E, horizon=1000, seed=3)
    obs_sp, act_sp = venv.observation_space, venv.action_space

    def basic():
        return reward_nets.BasicRewardNet(obs_sp, act_sp)

    if kind == "single":
        reward = basic()
    elif kind == "normalized":
        reward = reward_nets.NormalizedRewardNet(basic(), networks.RunningNorm)
    else:
        members = [reward_nets.NormalizedRewardNet(basic(), networks.RunningNorm) for _ in range(M)]
        reward = reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(obs_sp, act_sp, members), ALPHA)
    reward = reward.cuda()
    wrapped = reward_wrapper.RewardVecEnvWrapper(venv, reward.predict_processed)
    return ppo.DevicePPO("FeedForward32Policy", wrapped, n_steps=T, batch_size=64, n_epochs=1, seed=0)


def main(args):
    if not th.cuda.is_available():
        raise SystemExit("ensemble_rollout_bench needs a CUDA device")
    from imitation_b200 import _lib

    _lib.lib()
    kinds = ["single", "normalized", "ensemble"]
    algos = {k: _setting(k, args.envs, args.n_steps) for k in kinds}
    for _ in range(args.warmup):
        for k in kinds:
            algos[k].collect_rollouts()
    th.cuda.synchronize()
    times = {k: [] for k in kinds}
    for _ in range(args.steps):
        for k in kinds:
            a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
            a.record()
            algos[k].collect_rollouts()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    name, power = _card()
    res = {"bench": "ensemble_rollout", "envs": args.envs, "n_steps": args.n_steps, "members": M, "alpha": ALPHA,
           "repeats": args.steps, "card": name, "power_limit": power}
    for k in kinds:
        res[f"{k}_ms_median"] = round(float(np.median(times[k])), 4)
        res[f"{k}_ms_min"] = round(float(np.min(times[k])), 4)
    res["ensemble_over_single"] = round(res["ensemble_ms_median"] / res["single_ms_median"], 3)
    print(json.dumps(res))


if __name__ == "__main__":
    import argparse

    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--envs", type=int, default=8)
    p.add_argument("--n-steps", type=int, default=256)
    main(p.parse_args())
