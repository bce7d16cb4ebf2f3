"""SQIL throughput on seals/CartPole-v0 with the cartpole_0 demonstrations: `SQIL.train` at the tutorial's shape
(n_envs 1, SB3's DQN defaults) and at n_envs 8, against the same TD steps in torch-eager ops on the same GPU.

Prints one JSON line per result (and, with --out DIR, writes them to DIR/sqil_bench.jsonl):
  - env steps/s and gradient steps/s of SQIL.train (device-synchronised wall clock, after a warm-up call);
  - kernels per gradient step (the binding's launch counter) and host launches per gradient step (eager launches plus
    one per CUDA-graph replay);
  - two eager loops of the TD part only (target forward, smooth L1, backward, clip_grad_norm_, torch Adam), a lower
    bound on an eager DQN's step time: one sampling through SQILReplayBuffer.sample (SB3's NumPy indices), one from
    preallocated device tensors with torch.randint;
  - the greedy policy's mean return over 100 episodes before and after --return-steps env steps of training.
The card's name and power limit are read in the same run.
"""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers still print; the card is then unknown
        return {"gpu": th.cuda.get_device_name(0), "power_limit": f"unknown ({e})"}


def make(n_envs, seed=0, **kw):
    from imitation_b200.algorithms import sqil
    from imitation_b200.data import rollout, serialize
    from imitation_b200.envs import make_vec_env

    demos = serialize.load(os.path.join(ROOT, "tests", "golden", "expert_models", "cartpole_0", "rollouts", "final.npz"))
    venv = make_vec_env("seals/CartPole-v0", rng=np.random.default_rng(seed), n_envs=n_envs)
    return sqil.SQIL(venv=venv, demonstrations=rollout.flatten_trajectories(demos), policy="MlpPolicy",
                     rl_kwargs=kw)


def time_train(n_envs, steps, **kw):
    from imitation_b200 import _lib

    algo = make(n_envs, seed=1, **kw)
    algo.train(total_timesteps=100 * n_envs * 4)  # warm-up: modules loaded, buffers allocated
    th.cuda.synchronize()
    dq = algo.rl_algo
    n0, l0, r0, k0 = dq._n_updates, _lib.LAUNCHES["count"], dq.graph_replays, dq.graph_kernels
    t = time.perf_counter()
    algo.train(total_timesteps=steps)
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    g = dq._n_updates - n0
    kernels = _lib.LAUNCHES["count"] - l0
    host = kernels - (dq.graph_kernels - k0) + (dq.graph_replays - r0)  # eager launches + one per graph replay
    return {"what": "SQIL.train", "n_envs": n_envs, "env_steps": steps, "seconds": dt, "env_steps_per_s": steps / dt,
            "grad_steps_per_s": g / dt, "kernels_per_grad_step": kernels / max(g, 1),
            "host_launches_per_grad_step": host / max(g, 1)}


def time_eager(steps, batch_size=32):
    algo = make(1, seed=1, learning_starts=0)
    algo.train(total_timesteps=400)  # a filled ring to sample from
    dq, buf = algo.rl_algo, algo.rl_algo.replay_buffer
    q, tgt = dq.policy.q_net, dq.policy.q_net_target
    opt = th.optim.Adam(q.parameters(), lr=1e-4)

    def step():
        s = buf.sample(batch_size)
        with th.no_grad():
            y = s.rewards + (1 - s.dones) * 0.99 * tgt(s.next_observations).max(1, keepdim=True)[0]
        qa = th.gather(q(s.observations), 1, s.actions.long())
        loss = th.nn.functional.smooth_l1_loss(qa, y)
        opt.zero_grad()
        loss.backward()
        th.nn.utils.clip_grad_norm_(q.parameters(), 10)
        opt.step()

    for _ in range(50):
        step()
    th.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        step()
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    out = [{"what": "eager TD steps, SQILReplayBuffer.sample", "batch_size": batch_size, "grad_steps": steps,
            "seconds": dt, "grad_steps_per_s": steps / dt}]

    # the same TD step from preallocated device tensors, sampled with torch.randint on the device (no host indices)
    obs = buf.ring[:4].t().contiguous()
    acts = buf.ring[4:6].argmax(0)[:, None]
    nobs = buf.ring[6:10].t().contiguous()
    dones = buf.ring[10][:, None].contiguous()
    eobs = buf.expert_table[:4].t().contiguous()
    eacts = buf.expert_table[4:6].argmax(0)[:, None]
    enobs = buf.expert_table[6:10].t().contiguous()
    edones = buf.expert_table[10][:, None].contiguous()
    n_l, n_e, size = batch_size // 2, batch_size - batch_size // 2, buf.size() * buf.n_envs
    rews = th.cat([th.zeros(n_l, 1), th.ones(n_e, 1)]).cuda()

    def step_plain():
        li = th.randint(0, size, (n_l,), device="cuda")
        xi = th.randint(0, buf.n_expert, (n_e,), device="cuda")
        o, a = th.cat([obs[li], eobs[xi]]), th.cat([acts[li], eacts[xi]])
        no, d = th.cat([nobs[li], enobs[xi]]), th.cat([dones[li], edones[xi]])
        with th.no_grad():
            y = rews + (1 - d) * 0.99 * tgt(no).max(1, keepdim=True)[0]
        loss = th.nn.functional.smooth_l1_loss(th.gather(q(o), 1, a), y)
        opt.zero_grad()
        loss.backward()
        th.nn.utils.clip_grad_norm_(q.parameters(), 10)
        opt.step()

    for _ in range(50):
        step_plain()
    th.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        step_plain()
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    out.append({"what": "eager TD steps, preallocated device tensors + torch.randint", "batch_size": batch_size,
                "grad_steps": steps, "seconds": dt, "grad_steps_per_s": steps / dt})
    return out


def returns(n_steps, n_envs):
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env

    algo = make(n_envs, seed=2)
    ev = make_vec_env("seals/CartPole-v0", rng=np.random.default_rng(42), n_envs=100)

    def ret():
        trajs = rollout.generate_trajectories(algo.policy, ev, rollout.make_min_episodes(100), np.random.default_rng(0))
        return float(np.mean([np.sum(t.rews) for t in trajs[:100]]))

    before = ret()
    t = time.perf_counter()
    algo.train(total_timesteps=n_steps)
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    return {"what": "return", "n_envs": n_envs, "env_steps": n_steps, "return_before": before, "return_after": ret(),
            "train_seconds": dt}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40_000)
    ap.add_argument("--eager-steps", type=int, default=2_000)
    ap.add_argument("--return-steps", type=int, default=100_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)

    info = card()
    rows = [time_train(1, a.steps), time_train(8, 8 * a.steps), *time_eager(a.eager_steps),
            returns(a.return_steps, 1)]
    lines = [json.dumps({**info, **r}) for r in rows]
    for line in lines:
        print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sqil_bench.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
