"""SQIL(SAC) throughput on Pendulum-v1 with the pendulum_0 demonstrations, at SB3's SAC defaults (width 256, batch
256, train_freq 1, gradient_steps 1): `SQIL.train` at n_envs 1 and 8, the device gradient step alone, and the same SAC
gradient step in torch-eager ops on the same GPU.

Prints one JSON line per result (and, with --out DIR, writes them to DIR/sqil_sac_bench.jsonl):
  - env steps/s and gradient steps/s of SQIL.train (device-synchronised wall clock, after a warm-up call);
  - kernels per gradient step (the binding's launch counter) and host launches per gradient step (eager launches plus
    one per CUDA-graph replay);
  - the device gradient step alone (imb_sac_step, --kernel-steps steps in one call, CUDA events);
  - the SAC gradient step as SB3's train() writes it, in torch-eager ops (float32, the SACPolicy's own modules, torch
    Adam), sampling minibatches from preallocated device tensors with torch.randint (a lower bound on an eager SAC's
    step: no host indices);
  - the deterministic policy's mean return over 100 episodes before and after --return-steps env steps of training.
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
    from imitation_b200.algorithms import sac, sqil
    from imitation_b200.data import rollout, serialize
    from imitation_b200.envs import make_vec_env

    demos = serialize.load(os.path.join(ROOT, "tests", "golden", "expert_models", "pendulum_0", "rollouts", "final.npz"))
    venv = make_vec_env("Pendulum-v1", rng=np.random.default_rng(seed), n_envs=n_envs)
    return sqil.SQIL(venv=venv, demonstrations=rollout.flatten_trajectories(demos), policy="MlpPolicy",
                     rl_algo_class=sac.SAC, rl_kwargs=dict(seed=seed, **kw))


def time_train(n_envs, steps):
    from imitation_b200 import _lib

    algo = make(n_envs, seed=1)
    algo.train(total_timesteps=300 * n_envs)  # warm-up: modules loaded, buffers allocated, past learning_starts
    th.cuda.synchronize()
    m = algo.rl_algo
    n0, l0, r0, k0 = m._n_updates, _lib.LAUNCHES["count"], m.graph_replays, m.graph_kernels
    t = time.perf_counter()
    algo.train(total_timesteps=steps, reset_num_timesteps=False)
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    g = m._n_updates - n0
    kernels = _lib.LAUNCHES["count"] - l0
    host = kernels - (m.graph_kernels - k0) + (m.graph_replays - r0)  # eager launches + one per graph replay
    return {"what": "SQIL(SAC).train", "n_envs": n_envs, "env_steps": steps, "seconds": dt,
            "env_steps_per_s": steps / dt, "grad_steps_per_s": g / dt, "kernels_per_grad_step": kernels / max(g, 1),
            "host_launches_per_grad_step": host / max(g, 1)}


def time_kernel(steps):
    """imb_sac_step alone: `steps` gradient steps in one call over a filled ring, timed with CUDA events."""
    from imitation_b200 import _lib

    algo = make(1, seed=3, learning_starts=0)
    algo.train(total_timesteps=2000)
    m, buf = algo.rl_algo, algo.rl_algo.replay_buffer
    B, n_l, n_e = m.batch_size, m.batch_size // 2, m.batch_size - m.batch_size // 2
    lidx = th.randint(0, buf.size() * buf.n_envs, (steps, n_l), device="cuda")
    eidx = th.randint(0, buf.n_expert, (steps, n_e), device="cuda")
    loss = th.zeros(steps, 4, device="cuda")
    pol = m.policy
    times = []
    for _ in range(3):
        base = int(m._state[_lib.ST_PPO_STEP])
        e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        e0.record()
        _lib.sac_step(m._hparams(), pol.actor_flat(), m.actor_m, m.actor_v, pol.critic_flat(), m.critic_m, m.critic_v,
                      pol.target_flat(), m._ent, buf.ring, buf.capacity, lidx, buf.expert_table, buf.n_expert, eidx,
                      steps, base, loss, m._ws, m._state)
        e1.record()
        th.cuda.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    dt = min(times[1:])
    return {"what": "imb_sac_step", "batch_size": B, "hidden": pol.hidden, "grad_steps": steps, "seconds": dt,
            "grad_steps_per_s": steps / dt, "us_per_grad_step": 1e6 * dt / steps}


def time_eager(steps):
    """SB3's SAC.train body for one gradient step in torch-eager float32 ops (ent_coef "auto")."""
    algo = make(1, seed=4, learning_starts=0)
    algo.train(total_timesteps=2000)
    m, buf = algo.rl_algo, algo.rl_algo.replay_buffer
    pol = m.policy
    actor, critic, target = pol.actor, pol.critic, pol.critic_target
    Do, Da, B = pol.d_obs, pol.d_act, m.batch_size
    opt_a = th.optim.Adam(actor.parameters(), lr=3e-4)
    opt_c = th.optim.Adam(critic.parameters(), lr=3e-4)
    log_ent_coef = th.zeros(1, device="cuda", requires_grad=True)
    opt_e = th.optim.Adam([log_ent_coef], lr=3e-4)
    tab = lambda t, n: t[:, :n].t().contiguous()
    ring, exp = tab(buf.ring, buf.size() * buf.n_envs), buf.expert_table.t().contiguous()
    n_l, n_e = B // 2, B - B // 2
    rews = th.cat([th.zeros(n_l, 1), th.ones(n_e, 1)]).cuda()
    te = -float(Da)

    def action_log_prob(o):
        mean, log_std = actor.get_action_dist_params(o)
        std = log_std.exp()
        g = mean + th.randn_like(mean) * std
        a = th.tanh(g)
        lp = th.distributions.Normal(mean, std).log_prob(g).sum(1) - th.sum(th.log(1 - a ** 2 + 1e-6), dim=1)
        return a, lp.reshape(-1, 1)

    def step():
        li = th.randint(0, ring.shape[0], (n_l,), device="cuda")
        xi = th.randint(0, exp.shape[0], (n_e,), device="cuda")
        x = th.cat([ring[li], exp[xi]])
        obs, acts, nobs, dones = x[:, :Do], x[:, Do:Do + Da], x[:, Do + Da:2 * Do + Da], x[:, -1:]
        a_pi, logp = action_log_prob(obs)
        ent_coef = th.exp(log_ent_coef.detach())
        ent_loss = -(log_ent_coef * (logp + te).detach()).mean()
        opt_e.zero_grad()
        ent_loss.backward()
        opt_e.step()
        with th.no_grad():
            a_n, lp_n = action_log_prob(nobs)
            nq = th.min(th.cat(target(nobs, a_n), 1), dim=1, keepdim=True)[0] - ent_coef * lp_n
            y = rews + (1 - dones) * 0.99 * nq
        closs = 0.5 * sum(th.nn.functional.mse_loss(q, y) for q in critic(obs, acts))
        opt_c.zero_grad()
        closs.backward()
        opt_c.step()
        minq = th.min(th.cat(critic(obs, a_pi), 1), dim=1, keepdim=True)[0]
        aloss = (ent_coef * logp - minq).mean()
        opt_a.zero_grad()
        aloss.backward()
        opt_a.step()
        with th.no_grad():
            for tp, p in zip(target.parameters(), critic.parameters()):
                tp.mul_(1 - 0.005)
                tp.add_(p, alpha=0.005)

    for _ in range(50):
        step()
    th.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(steps):
        step()
    th.cuda.synchronize()
    dt = time.perf_counter() - t
    return {"what": "eager SAC steps, preallocated device tensors + torch.randint", "batch_size": B,
            "hidden": pol.hidden, "grad_steps": steps, "seconds": dt, "grad_steps_per_s": steps / dt,
            "us_per_grad_step": 1e6 * dt / steps}


def returns(n_steps, n_envs):
    from imitation_b200.data import rollout
    from imitation_b200.envs import make_vec_env

    algo = make(n_envs, seed=42)
    ev = make_vec_env("Pendulum-v1", rng=np.random.default_rng(42), n_envs=100)

    def ret():
        trajs = rollout.generate_trajectories(algo.policy, ev, rollout.make_min_episodes(100), np.random.default_rng(0),
                                              deterministic_policy=True)
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
    ap.add_argument("--steps", type=int, default=5_000)
    ap.add_argument("--kernel-steps", type=int, default=1_000)
    ap.add_argument("--eager-steps", type=int, default=1_000)
    ap.add_argument("--return-steps", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import __graft_entry__  # noqa: F401  (puts the repository on sys.path)

    info = card()
    rows = [time_train(1, a.steps), time_train(8, 8 * a.steps), time_kernel(a.kernel_steps), time_eager(a.eager_steps),
            returns(a.return_steps, 1)]
    lines = [json.dumps({**info, **r}) for r in rows]
    for line in lines:
        print(line, flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sqil_sac_bench.jsonl"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
