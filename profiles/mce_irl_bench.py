"""MCE IRL on the device: time per MCEIRL.train iteration and per sweep launch (imb_mce_sweep), against the reference
algorithm's per-iteration time on the host (oracle/mce_port.py's NumPy float64 sweep + torch-CPU autograd and Adam, the
reference's own arithmetic) in the same run.

Workloads:
  random5     the reference tests' random MDP shape (S = 5, A = 3, H = 10, one-hot features, linear net): overhead;
  grid32      a 32 x 32 slippery gridworld (S = 1024, A = 4, H = 100, 16 random features, [32, 32] net): T (33.5 MB)
              stays in the 50 MB L2, so the sweep's rate is reported in bytes/s, not as a share of HBM bandwidth;
  grid64      a 64 x 64 gridworld (S = 4096, A = 4, H = 100, same net): T (537 MB) streams from HBM twice per step
              pair, so the share of the 3.35 TB/s HBM3 bound is reported.
Two byte counts are reported over the sweep's kernel time.  `algo_bytes` is what the algorithm touches: 2 H S A S 8
bytes of T (one backward and one forward pass per step) plus its vectors (pi written and read back, D written and
read, V staged per step).  `read_bytes` is what the kernel actually reads: the last backward step needs no dot, and
the forward step skips the rows of states the occupancy has not reached (D[t, s] == 0, exact).  The HBM share is
computed from `read_bytes`.  `iter_ms` is the difference of two train() calls of N and 2N iterations over N, so the
once-per-call uploads (T, observations, demonstrations) and the final planning sweep are not in it.  Device times
are CUDA events after a warm-up; the card's name and power limit are read in the same run.  One JSON line per
workload.
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
# name: (builder kwargs, hidden sizes, timed iterations, host iterations)
WORKLOADS = {
    "random5": (dict(kind="random", S=5, A=3, H=10), (), 2000, 50),
    "grid32": (dict(kind="grid", n=32, H=100), (32, 32), 200, 2),
    "grid64": (dict(kind="grid", n=64, H=100), (32, 32), 20, 1),
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


def _mdp(spec):
    from oracle import tabular_mdp

    if spec["kind"] == "random":
        return tabular_mdp.random_mdp(spec["S"], spec["A"], 2, spec["H"], obs_dim=None, seed=42)
    return tabular_mdp.gridworld(spec["n"], spec["H"], features="random", obs_dim=16, seed=0)


def _timed(fn, n):
    a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def bench(name, warmup):
    from imitation_b200 import _lib
    from imitation_b200.algorithms import mce_irl
    from imitation_b200.rewards import reward_nets
    from oracle import mce_port

    spec, hid, iters, host_iters = WORKLOADS[name]
    mdp = _mdp(spec)
    S, A, H = mdp.state_dim, mdp.action_dim, mdp.horizon
    demo = mce_port.occupancy(mdp.transition_matrix, mdp.initial_state_dist,
                              mce_port.partition_fh(mdp.transition_matrix, mdp.reward_matrix, H)[2], H, 1.0)[1]
    th.manual_seed(0)
    net = reward_nets.BasicRewardNet(mdp.observation_space, mdp.action_space, use_action=False,
                                     hid_sizes=list(hid)).to("cuda")
    algo = mce_irl.MCEIRL(demo, mdp, net, np.random.default_rng(0), log_interval=None, linf_eps=-1.0,
                          grad_l2_eps=-1.0)
    algo.train(max_iter=warmup)
    th.cuda.synchronize()

    def train_ms(n):
        a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        a.record()
        algo.train(max_iter=n)
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    # per iteration, without train()'s once-per-call uploads and final sweep: the difference of two call lengths
    iter_ms = (train_ms(2 * iters) - train_ms(iters)) / iters

    # the sweep alone, as train() launches it
    m = mce_irl._DeviceMDP(mdp, _lib.MCE_BACKWARD | _lib.MCE_FORWARD)
    dev = m.T.device
    r32 = th.randn(S, device=dev)
    Dcum = th.empty(S, dtype=th.float64, device=dev)
    w = th.empty(S, device=dev)
    linf = th.empty(1, dtype=th.float64, device=dev)
    demo_d = th.as_tensor(demo).to(dev)
    gam = m.discounts(1.0, 1.0)

    def sweep():
        m.sweep(_lib.MCE_BACKWARD | _lib.MCE_FORWARD, gam, reward32=r32, Dcum=Dcum, demo_om=demo_d, weights=w, linf=linf)

    for _ in range(warmup):
        sweep()
    sweep_ms = _timed(sweep, iters)
    _, grid = _lib.mce_plan(S, A, H, _lib.MCE_BACKWARD | _lib.MCE_FORWARD)

    t_bytes = 2 * H * S * A * S * 8
    vec_bytes = 2 * H * S * A * 8 + 2 * (H + 1) * S * 8 + H * S * 8 * grid
    bytes_algo = t_bytes + vec_bytes
    # what the kernel reads of T: H - 1 backward passes (step H - 1 needs no dot) and, forward, only the rows of the
    # states with D[t, s] != 0 (the kernel skips the others; the support does not depend on the reward since pi > 0)
    D, _ = mce_irl.mce_occupancy_measures(mdp, reward=np.zeros(S))
    reached = int(np.count_nonzero(D[:H]))
    bytes_read = ((H - 1) * S + reached) * A * S * 8 + vec_bytes

    # the reference algorithm on the host: NumPy float64 sweep + torch-CPU net, autograd and Adam
    pnet = mce_port.port_net(mdp.observation_matrix.shape[1], hid, False)
    popt = th.optim.Adam(pnet.parameters(), lr=1e-2)
    obs = th.as_tensor(mdp.observation_matrix, dtype=th.float32)
    mce_port.train_iteration(pnet, popt, obs, mdp.transition_matrix, mdp.initial_state_dist, H, demo, 1.0)
    t0 = time.perf_counter()
    for _ in range(host_iters):
        mce_port.train_iteration(pnet, popt, obs, mdp.transition_matrix, mdp.initial_state_dist, H, demo, 1.0)
    host_ms = (time.perf_counter() - t0) * 1e3 / host_iters

    card, power = _card()
    out = {"workload": name, "S": S, "A": A, "H": H, "hid_sizes": list(hid), "grid_ctas": grid,
           "iter_ms": round(iter_ms, 4), "sweep_ms": round(sweep_ms, 4),
           "algo_bytes": bytes_algo, "algo_bytes_per_s": bytes_algo / (sweep_ms * 1e-3),
           "read_bytes": bytes_read, "read_bytes_per_s": bytes_read / (sweep_ms * 1e-3), "host_iter_ms": round(host_ms, 3),
           "host_iters": host_iters, "host_threads": th.get_num_threads(),
           "speedup_vs_host": round(host_ms / iter_ms, 1), "card": card, "power_limit": power}
    if name == "grid64":
        out["hbm_share_of_read_bytes"] = round(bytes_read / HBM_BYTES_PER_S / (sweep_ms * 1e-3), 3)
    return out


def main(args):
    if not th.cuda.is_available():
        raise SystemExit("mce_irl_bench needs a CUDA device")
    for name in args.workloads:
        print(json.dumps(bench(name, args.warmup)), flush=True)


if __name__ == "__main__":
    import argparse

    p = argparse.ArgumentParser()
    p.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    p.add_argument("--warmup", type=int, default=3)
    main(p.parse_args())
