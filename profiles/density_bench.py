"""Time of the density reward on the device: one `DevicePPO.collect_rollouts` with a `DensityAlgorithm` reward against
the same call with a `BasicRewardNet` reward, and the `imb_density_score` launch alone.

    python profiles/density_bench.py [--steps K] [--warmup W]

Workloads (demonstrations synthetic, normal rows; the counts are what matters to the kernel):
  pendulum  8 envs x 2048 steps, obs 3 / act 1, STATE_ACTION (D = 4), N = 5 600 demonstration rows (28 Pendulum
            trajectories of 200 steps, as the reference's test_density_reward uses)
  large     16 envs x 1024 steps = 16 384 queries, obs 17 (HalfCheetah) / act 6, STATE_STATE (D = 34), N = 100 000
Both stationary, gaussian kernel, h = 0.5.  Each timing is CUDA events around the call, median over --steps repeats
after --warmup; the two rollouts alternate within every repeat.  The counts reported beside the times come from the
shapes: pairs = queries x N; per pair the kernel issues D FSUB + D FFMA (3 D flops, FFMA = 2) and one MUFU exp.  The
FP32 bound is the pair count times 2 D FP32 instructions at the data-sheet rate of 67 TFLOP/s = 33.5 T FP32
instructions/s (H100 SXM, 700 W); the kernel's share of it is that bound over the measured launch time.  Prints one
JSON line per workload with the card's name and power limit, read in the same run."""
import json
import os
import subprocess
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {  # name: (envs, steps, d_obs, d_act, demo rows, density type)
    "pendulum": (8, 2048, 3, 1, 5600, "STATE_ACTION_DENSITY"),
    "large": (16, 1024, 17, 6, 100_000, "STATE_STATE_DENSITY"),
}
FP32_INSTR_PER_S = 67e12 / 2


def _card():
    name = th.cuda.get_device_name() if th.cuda.is_available() else None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _timed(fn):
    a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def _setups(name):
    from imitation_b200.algorithms import density, ppo
    from imitation_b200.data import wrappers
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, reward_wrapper

    E, T, Do, Da, N, dtype = WORKLOADS[name]
    out = {}
    for kind in ("density", "reward_net"):
        venv = synth.DeviceVecEnv(Do, Da, E, horizon=1000, seed=3)
        algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=64, n_epochs=1, seed=0)
        if kind == "density":
            rng = np.random.default_rng(0)
            dens = density.DensityAlgorithm(demonstrations=None, venv=venv, rng=rng, rl_algo=algo,
                                            density_type=density.DensityType[dtype], kernel_bandwidth=0.5)
            D = Do + Da if dtype == "STATE_ACTION_DENSITY" else 2 * Do
            dens.transitions = {None: rng.normal(size=(N, D))}
            dens.train()
            algo.set_env(dens.venv_wrapped)
            out[kind] = (algo, dens, D)
        else:
            th.manual_seed(0)
            net = reward_nets.BasicRewardNet(venv.observation_space, venv.action_space).cuda()
            algo.set_env(reward_wrapper.RewardVecEnvWrapper(wrappers.BufferingWrapper(venv), net.predict_processed))
            out[kind] = (algo, None, None)
    return out


def bench(name, steps, warmup):
    from imitation_b200 import _lib

    E, T, Do, Da, N, dtype = WORKLOADS[name]
    s = _setups(name)
    roll = {k: [] for k in s}
    for i in range(warmup + steps):
        for k, (algo, _, _) in s.items():
            algo._buffering.discard()
            ms = _timed(algo.collect_rollouts)
            if i >= warmup:
                roll[k].append(ms)
    algo, dens, D = s["density"]
    relabel = algo._rw_wrapper.resolve()
    col_rew = Do + Da + 2
    flat = algo._buffering._flat

    def launch():
        relabel.finish(algo._tbl, col_rew, flat, E, T, algo._base_env.horizon, algo._base_env.state, algo._scratch)

    for _ in range(warmup):
        launch()
    reps = 20
    kern = [_timed(lambda: [launch() for _ in range(reps)]) / reps for _ in range(steps)]
    pairs = E * T * N
    k_ms = float(np.median(kern))
    bound_ms = 1e3 * pairs * 2 * D / FP32_INSTR_PER_S
    card, power = _card()
    return {"bench": "density", "workload": name, "queries": E * T, "demo_rows": N, "features": D,
            "density_type": dtype, "repeats": steps,
            "collect_rollouts_density_ms": round(float(np.median(roll["density"])), 3),
            "collect_rollouts_reward_net_ms": round(float(np.median(roll["reward_net"])), 3),
            "density_launch_ms": round(k_ms, 4), "pairs": pairs, "flops_per_pair": 3 * D,
            "pair_rate_per_s": float(f"{pairs / (k_ms * 1e-3):.4g}"),
            "tflops": round(pairs * 3 * D / (k_ms * 1e-3) / 1e12, 2),
            "fp32_bound_ms": round(bound_ms, 4), "fp32_bound_share": round(bound_ms / k_ms, 3),
            "launches_per_score": 1, "card": card, "power_limit": power}


def main(args):
    if not th.cuda.is_available():
        raise SystemExit("density_bench needs a CUDA device")
    from imitation_b200 import _lib

    _lib.lib()
    for name in args.workloads.split(","):
        print(json.dumps(bench(name, args.steps, args.warmup)), flush=True)


if __name__ == "__main__":
    import argparse

    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--workloads", default="pendulum,large")
    main(p.parse_args())
