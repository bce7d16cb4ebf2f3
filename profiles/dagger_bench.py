"""Time DAgger rounds on the device, split into their parts.

    python profiles/dagger_bench.py [--rounds R] [--out DIR]

Workloads (synthetic env of the same shapes; policies seeded):
  half_cheetah  the dagger_seals_half_cheetah shape: 17 obs / 6-act Box, expert MlpPolicy 64x64 (tanh), learner
                FeedForward32Policy, 8 envs, horizon 1000, ExponentialBetaSchedule(0.7), batch 16, 5 epochs,
                rollout_round_min_episodes=5 (so one collection batch of 8 episodes, 8000 steps, per round)
  cartpole      the fast_dagger_seals_cartpole shape: 4 obs / Discrete(2), expert MlpPolicy 64x64, learner
                FeedForward32Policy, 8 envs, horizon 500, the default LinearBetaSchedule(15), batch 32, the fast
                configuration's bc train_kwargs (n_batches=50), rollout_round_min_episodes=3
Each round is run through the low-level API and split into:
  collection    the `imb_rollout_dagger` launches (CUDA events around each), and env-steps/s over them;
  host          the rest of `generate_trajectories`: mask and file-name draws, trajectory assembly, file writes,
                shuffle (host clock ending in a device synchronise, minus the collection);
  aggregation   `_try_load_demos` (listing + the device gather into the aggregate table);
  bc_train      `BC.train` (`extend_and_update` once the round is loaded).
Rounds after the first run the learner where its mask bit is set (beta < 1).  Prints one JSON line per workload with
the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = {  # name: (d_obs, d_act, discrete, envs, horizon, beta schedule, batch, train kwargs, min_episodes)
    "half_cheetah": (17, 6, False, 8, 1000, ("exp", 0.7), 16, dict(n_epochs=5), 5),
    "cartpole": (4, 2, True, 8, 500, ("linear", 15), 32, dict(n_batches=50), 3),
}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def run(name, rounds, scratch):
    from imitation_b200 import _lib
    from imitation_b200.algorithms import bc, dagger
    from imitation_b200.data import rollout
    from imitation_b200.envs import synth
    from imitation_b200.policies import base as policies

    d_obs, d_act, discrete, E, H, (kind, p), batch, train_kwargs, min_episodes = WORKLOADS[name]
    venv = synth.DeviceVecEnv(d_obs, d_act, E, discrete=discrete, horizon=H, seed=0)
    th.manual_seed(0)
    expert = policies.ActorCriticPolicy(venv.observation_space, venv.action_space, net_arch=[64, 64]).cuda()
    rng = np.random.default_rng(0)
    learner = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng,
                    batch_size=batch)
    schedule = dagger.ExponentialBetaSchedule(p) if kind == "exp" else dagger.LinearBetaSchedule(p)
    tr = dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=scratch, expert_policy=expert, rng=rng, bc_trainer=learner,
                                    beta_schedule=schedule)
    events = []
    launch = _lib.rollout_dagger

    def timed(*a, **k):
        e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        e0.record()
        launch(*a, **k)
        e1.record()
        events.append((e0, e1))

    _lib.rollout_dagger = timed
    out = []
    try:
        for r in range(rounds):
            events.clear()
            collector = tr.create_trajectory_collector()
            su = rollout.make_sample_until(min_timesteps=max(500, tr.batch_size), min_episodes=min_episodes)
            th.cuda.synchronize()
            t0 = time.perf_counter()
            trajs = rollout.generate_trajectories(expert, collector, su, rng=collector.rng, deterministic_policy=True)
            th.cuda.synchronize()
            t1 = time.perf_counter()
            tr._try_load_demos()
            th.cuda.synchronize()
            t2 = time.perf_counter()
            tr.extend_and_update(dict(train_kwargs, log_rollouts_venv=None))
            th.cuda.synchronize()
            t3 = time.perf_counter()
            coll_ms = sum(a.elapsed_time(b) for a, b in events)
            steps = sum(len(t) for t in trajs)
            out.append(dict(round=r, beta=collector.beta, launches=len(events), env_steps=steps,
                            collection_ms=round(coll_ms, 3), collection_env_steps_per_s=round(steps / coll_ms * 1e3),
                            host_ms=round((t1 - t0) * 1e3 - coll_ms, 3), aggregation_ms=round((t2 - t1) * 1e3, 3),
                            bc_train_ms=round((t3 - t2) * 1e3, 3), dataset_rows=tr._all_rows.n))
    finally:
        _lib.rollout_dagger = launch
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None, help="also write the JSON lines to DIR/dagger_bench.jsonl")
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("dagger_bench needs a GPU")
    gpu = card()
    lines = []
    for name in WORKLOADS:
        with tempfile.TemporaryDirectory() as scratch:
            lines.append(json.dumps(dict(workload=name, gpu=gpu, rounds=run(name, args.rounds, scratch))))
        print(lines[-1], flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "dagger_bench.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
