"""Throughput and learning on the device classic-control envs (seals/CartPole-v0, Pendulum-v1).

    python profiles/classic_control_bench.py [--rounds R] [--total-timesteps N] [--out DIR]

Reports, with the card's name and power limit read in the same run:
  gail_round_<env>   env-steps/s of GAIL rounds (train_gen: rollout + PPO update; train_disc) on 64 envs, the generator
                     rolling out 2048 steps per round (32 steps x 64 envs); a host clock around R rounds that ends in a
                     device synchronise, after 3 warm-up rounds
  bc_cartpole        the return_mean of 64 deterministic episodes of the BC policy of
                     tests/test_classic_env_gpu.py (reference defaults, 4 epochs on the cartpole_0 demonstrations)
  gail_cartpole      GAIL on seals/CartPole-v0 from the cartpole_0 demonstrations at the reference's seals_cartpole
                     budget (total_timesteps 1.4e6, 8 envs as its default environment ingredient), with rollout_stats of
                     the generator (50 sampled episodes) before and after, and the wall time
Prints one JSON line per result; with --out, also writes them all to DIR/classic_control.json."""
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
DEMOS = os.path.join(ROOT, "tests", "golden", "expert_models", "{}", "rollouts", "final.npz")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return {"gpu": th.cuda.get_device_name(), "power_limit": power or "not measured"}


def _gail(env, n_envs, fixture, seed=0):
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms.adversarial import gail
    from imitation_b200.data import serialize
    from imitation_b200.envs import make_vec_env
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    th.manual_seed(seed)
    venv = make_vec_env(env, rng=np.random.default_rng(seed), n_envs=n_envs)
    gen = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=2048 // n_envs, batch_size=64, seed=seed)
    net = reward_nets.BasicRewardNet(venv.observation_space, venv.action_space,
                                     normalize_input_layer=networks.RunningNorm)
    demos = serialize.load(DEMOS.format(fixture))
    return gail.GAIL(demonstrations=demos, demo_batch_size=1024, venv=venv, gen_algo=gen, reward_net=net,
                     seed=seed), venv, gen


def gail_round(env, fixture, rounds):
    tr, venv, gen = _gail(env, 64, fixture)
    per = venv.num_envs * gen.n_steps
    tr.train(3 * per)
    th.cuda.synchronize()
    t = time.perf_counter()
    tr.train(rounds * per)
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    return {"env_steps_per_s": rounds * per / dt, "ms_per_round": 1e3 * dt / rounds, "rounds": rounds, "n_envs": 64}


def bc_cartpole():
    from imitation_b200.algorithms import bc
    from imitation_b200.data import rollout, serialize
    from imitation_b200.envs import make_vec_env

    rng = np.random.default_rng(0)
    th.manual_seed(0)
    venv = make_vec_env("seals/CartPole-v0", rng=rng, n_envs=64)
    trainer = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng,
                    demonstrations=serialize.load(DEMOS.format("cartpole_0")))

    def evaluate():
        trajs = rollout.generate_trajectories(trainer.policy, venv, rollout.make_min_episodes(64),
                                              np.random.default_rng(1), deterministic_policy=True)
        return rollout.rollout_stats(trajs)["return_mean"]

    before = evaluate()
    trainer.train(n_epochs=4)
    return {"return_mean_untrained": before, "return_mean_trained": evaluate()}


def gail_cartpole(total_timesteps):
    from imitation_b200.data import rollout

    tr, venv, gen = _gail("seals/CartPole-v0", 8, "cartpole_0")

    def stats():
        trajs = rollout.generate_trajectories(gen, venv, rollout.make_min_episodes(50), np.random.default_rng(0))
        s = rollout.rollout_stats(trajs)
        return {k: float(s[k]) for k in ("n_traj", "return_mean", "return_std", "return_min", "return_max")}

    before = stats()
    th.cuda.synchronize()
    t = time.perf_counter()
    tr.train(total_timesteps)
    th.cuda.synchronize()
    return {"total_timesteps": total_timesteps, "wall_s": time.perf_counter() - t, "before": before, "after": stats()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=200)
    ap.add_argument("--total-timesteps", type=int, default=int(1.4e6))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("classic_control_bench needs a GPU")
    from imitation_b200 import _build

    _build.build()
    card = _card()
    results = []
    for name, fn in (("gail_round_cartpole", lambda: gail_round("seals/CartPole-v0", "cartpole_0", args.rounds)),
                     ("gail_round_pendulum", lambda: gail_round("Pendulum-v1", "pendulum_0", args.rounds)),
                     ("bc_cartpole", bc_cartpole),
                     ("gail_cartpole", lambda: gail_cartpole(args.total_timesteps))):
        r = {"name": name, **card, **fn()}
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "classic_control.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
