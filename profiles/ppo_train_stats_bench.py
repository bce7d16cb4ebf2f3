"""Cost of the PPO update's training statistics and of SB3's clip_range_vf / target_kl options.

Times one PPO-update launch (CUDA events, median of windows) on the bench.py policy shapes in five settings:
  plain      imb_ppo_update (no statistics, options off)
  stats      imb_ppo_update_ex with the statistics vector (what DevicePPO.train() launches)
  clip_vf    + clip_range_vf = 0.2
  kl_never   + target_kl = 1e30 (the KL shares travel with the slice norms every step, the stop never fires)
  both       clip_range_vf = 0.2 and target_kl = 1e30

    python profiles/ppo_train_stats_bench.py [--reps 20] [--windows 7]
"""
import argparse
import json
import os
import sys

import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from imitation_b200 import _lib  # noqa: E402
from imitation_b200.algorithms import ppo  # noqa: E402
from imitation_b200.envs import synth  # noqa: E402

# name: d_obs, d_act, discrete, feature norm, envs, n_steps, minibatch, epochs (bench.py's hc / ant / cartpole shapes)
SHAPES = {"hc": (17, 6, False, True, 16, 256, 64, 5), "ant": (27, 8, False, True, 16, 128, 16, 10),
          "cartpole": (4, 2, True, False, 16, 128, 64, 10)}
SETTINGS = {"plain": None, "stats": (None, None), "clip_vf": (None, 0.2), "kl_never": (1e30, None),
            "both": (1e30, 0.2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    out = {"gpu": th.cuda.get_device_name(), "unit": "ms per PPO-update launch (median over windows)", "shapes": {}}
    for name, (Do, Da, disc, norm, E, T, mb, ep) in SHAPES.items():
        venv = synth.DeviceVecEnv(Do, Da, E, discrete=disc, horizon=1000, seed=0)
        gen = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=mb, n_epochs=ep, seed=0,
                            policy_kwargs=dict(normalize_features=norm))
        gen.collect_rollouts()
        pol = gen.policy
        pp, pn, pc = pol.flat_vectors()
        N = gen._tbl.shape[0]

        def launch(setting):
            if setting is None:
                _lib.ppo_update(pol.desc, pp, pn, pc, gen.exp_avg, gen.exp_avg_sq, gen._tbl, N, gen.hp, None, 0, None,
                                venv.state, act=pol.act)
            else:
                _lib.ppo_update_ex(pol.desc, pp, pn, pc, gen.exp_avg, gen.exp_avg_sq, gen._tbl, N, gen.hp, None, 0, None,
                                   venv.state, target_kl=setting[0], clip_range_vf=setting[1], stats=gen.train_stats,
                                   act=pol.act)

        res = {}
        for s in SETTINGS.values():
            for _ in range(3):
                launch(s)
        th.cuda.synchronize()
        wins = {k: [] for k in SETTINGS}
        for _ in range(args.windows):  # settings interleaved window by window: clock drift hits all of them alike
            for k, s in SETTINGS.items():
                a, b = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.reps):
                    launch(s)
                b.record()
                b.synchronize()
                wins[k].append(a.elapsed_time(b) / args.reps)
        for k, w in wins.items():
            w = sorted(w)
            res[k] = {"median": w[len(w) // 2], "min": w[0], "max": w[-1]}
        res["steps_per_launch"] = ep * ((N + mb - 1) // mb)
        out["shapes"][name] = res
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
