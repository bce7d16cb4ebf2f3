"""Device time of one `DevicePPO.collect_rollouts` (rollout + output normalisation + GAE + state advance) at the
`airl_hc` shape of bench.py (obs 17 / act 6, 1024 envs x 8 steps, BasicShapedRewardNet with input RunningNorm inside
NormalizedRewardNet), with the two output layers:

    running  NormalizedRewardNet(net, RunningNorm)   (imb_rollout + imb_reward_norm_scan)
    ema      NormalizedRewardNet(net, EMANorm)       (imb_rollout + imb_reward_ema_scan)

    python profiles/ema_norm_bench.py [--steps K] [--warmup W]

Both settings run on one trainer, the rollout's reward function switched between calls; each timed call is bracketed
by CUDA events and the settings alternate within every repeat so that they share the same machine conditions.  Prints
one JSON line with the median and minimum per setting (ms) and the card's name and power limit, read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    import bench
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks
    from profiles.ensemble_rollout_bench import _card

    cfg = bench.CONFIGS["airl_hc"]
    tr, _ = bench.build_trainer(cfg, 0, 1, th.device("cuda"))
    gen, wrapper = tr.gen_algo, tr.venv_wrapped
    # two NormalizedRewardNets around the one shaped net; the rollout's reward function selects which one runs
    nets = {"running": tr._reward_net,
            "ema": reward_nets.NormalizedRewardNet(tr._reward_net.base, networks.EMANorm).cuda()}

    def run(kind):
        wrapper.reward_fn = nets[kind].predict_processed
        a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
        a.record()
        gen.collect_rollouts()
        b.record()
        b.synchronize()
        return a.elapsed_time(b)

    for _ in range(args.warmup):
        for kind in nets:
            run(kind)
    times = {kind: [] for kind in nets}
    for _ in range(args.steps):
        for kind in nets:
            times[kind].append(run(kind))
    name, power = _card()
    out = {"config": "airl_hc", "envs": gen._base_env.num_envs, "n_steps": gen.n_steps, "steps": args.steps,
           "gpu": name, "power_limit": power}
    for kind, ts in times.items():
        out[f"{kind}_median_ms"] = float(np.median(ts))
        out[f"{kind}_min_ms"] = float(np.min(ts))
    # every EMA call advanced the statistics by one batch per env step
    out["ema_num_batches"] = int(nets["ema"].normalize_output_layer.num_batches)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
