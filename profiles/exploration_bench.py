"""Wall time of one `AgentTrainer.sample` with and without exploratory rollouts, at the shape of the reference's
preference-comparisons quickstart (docs/algorithms/preference_comparisons.rst: Pendulum, 8 envs, PPO n_steps 256,
FeedForward32Policy with NormalizeFeaturesExtractor, BasicRewardNet with an input RunningNorm, fragment length 100):
obs 3 / act 1, horizon 200, and a sample of 4000 transitions (the first iteration's 20 pairs x 2 x 100).

    python profiles/exploration_bench.py [--steps K] [--warmup W] [--sample N]

Two settings, exploration_frac 0 and 0.05 (the quickstart's); with 0.05, 200 of the 4000 transitions come from one
exploration rollout of 200 steps from reset.  Before every timed call the agent trains 3 x 8 x 256 steps so that its
buffer holds the agent part; each call is timed on the host clock between two device synchronisations (sample()
returns host trajectories).  The settings alternate within every repeat.  Prints one JSON line with the median and
minimum per setting (ms) and the card's name and power limit, read in the same run."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Do, Da, E, H, N_STEPS = 3, 1, 8, 200, 256


def _card():
    name = th.cuda.get_device_name() if th.cuda.is_available() else None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _agent(frac):
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.policies import base as policies
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    th.manual_seed(0)
    venv = synth.DeviceVecEnv(Do, Da, E, horizon=H, seed=3)
    reward = reward_nets.BasicRewardNet(venv.observation_space, venv.action_space,
                                        normalize_input_layer=networks.RunningNorm).cuda()
    algo = ppo.DevicePPO(policies.FeedForward32Policy, venv, n_steps=N_STEPS, batch_size=64, n_epochs=1, seed=0,
                         policy_kwargs=dict(features_extractor_class=policies.NormalizeFeaturesExtractor))
    return pc.AgentTrainer(algo, reward, venv, np.random.default_rng(0), exploration_frac=frac)


def main(args):
    if not th.cuda.is_available():
        raise SystemExit("exploration_bench needs a CUDA device")
    from imitation_b200 import _lib

    _lib.lib()
    fracs = [0.0, 0.05]
    agents = {f: _agent(f) for f in fracs}
    times = {f: [] for f in fracs}
    for i in range(args.warmup + args.steps):
        for f in fracs:
            agents[f].train(3 * E * N_STEPS)
            th.cuda.synchronize()
            t0 = time.perf_counter()
            agents[f].sample(args.sample)
            th.cuda.synchronize()
            if i >= args.warmup:
                times[f].append(1e3 * (time.perf_counter() - t0))
    name, power = _card()
    res = {"bench": "exploration_sample", "envs": E, "horizon": H, "sample": args.sample, "repeats": args.steps,
           "card": name, "power_limit": power}
    for f in fracs:
        res[f"frac{f}_ms_median"] = round(float(np.median(times[f])), 3)
        res[f"frac{f}_ms_min"] = round(float(np.min(times[f])), 3)
    print(json.dumps(res))


if __name__ == "__main__":
    import argparse

    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--sample", type=int, default=4000)
    main(p.parse_args())
