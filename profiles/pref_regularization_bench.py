"""Cost of reward-model regularization in preference comparisons at `bench.py --config pref`'s shapes (obs 11 / act 3,
fragment length 100, 2048 pairs, 5-member RewardEnsemble of BasicRewardNet 32x32, minibatch 256 pairs, one epoch per
call): one `EnsembleTrainer.train` call with
  none      no regularizer;
  lp2       LpRegularizer(p=2), lambda 1e-3, no updater;
  wd        WeightDecayRegularizer, lambda 1e-3, no updater;
  lp2_upd   LpRegularizer(p=2) + IntervalParamScaler(0.1, (1.1, 1.5)) on a 0.2 validation split.
Each setting is timed over --calls calls (after --warmup) with a device synchronise before and after each call;
prints one JSON line with the median per setting (ms), the library launches per call and the card's name and power
limit, read in the same run.  For lp2 it also splits the cost of the extra launch: the host time of each
`_lib.param_regularize` call inside a training call (median, us) and the device time of `k_param_regularize` (CUDA events
around the replay of a CUDA graph of 200 launches on one member's parameters, us per launch)."""
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

Do, Da, L, P, M, MB = 11, 3, 100, 2048, 5, 256


def _card():
    name = th.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def _factory(setting):
    from imitation_b200.regularization import IntervalParamScaler, LpRegularizer, WeightDecayRegularizer

    return {"none": None,
            "lp2": LpRegularizer.create(1e-3, val_split=None, p=2),
            "wd": WeightDecayRegularizer.create(1e-3, val_split=None),
            "lp2_upd": LpRegularizer.create(1e-3, IntervalParamScaler(0.1, (1.1, 1.5)), val_split=0.2, p=2)}[setting]


def _time(setting, ds, calls, warmup):
    from imitation_b200 import _lib, spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.rewards import reward_nets

    th.manual_seed(0)
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1.0, 1.0, (Da,))
    members = [reward_nets.BasicRewardNet(obs_space, act_space, hid_sizes=(32, 32)).cuda() for _ in range(M)]
    ens = reward_nets.RewardEnsemble(obs_space, act_space, members)
    trainer = pc.EnsembleTrainer(pc.PreferenceModel(ens), pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(1),
                                 batch_size=MB, epochs=1, lr=1e-3, regularizer_factory=_factory(setting))
    for _ in range(warmup):
        trainer.train(ds)
    times, launches = [], []
    for _ in range(calls):
        th.cuda.synchronize()
        n0, t0 = _lib.LAUNCHES["count"], time.perf_counter()
        trainer.train(ds)
        th.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
        launches.append(_lib.LAUNCHES["count"] - n0)
    assert all("_fused_opt" in t.__dict__ for t in trainer.member_trainers), "a member left the device step"
    extra = _launch_costs(trainer, members[0], ds) if setting == "lp2" else {}
    return float(np.median(times)), int(np.median(launches)), extra


def _launch_costs(trainer, net, ds):
    from imitation_b200 import _lib

    host, orig = [], _lib.param_regularize

    def timed(*args, **kw):
        t0 = time.perf_counter()
        orig(*args, **kw)
        host.append((time.perf_counter() - t0) * 1e6)

    _lib.param_regularize = timed
    try:
        trainer.train(ds)
    finally:
        _lib.param_regularize = orig
    e = net.engine()
    n = 200
    # device time without the host in the way: the n launches captured in one CUDA graph, its replay timed by events
    # (it runs into the gradient accumulator only, which the next training minibatch clears)
    _lib.param_regularize(e.desc, _lib.REG_LP, 2, 1e-3, e.params, e.ws)
    th.cuda.synchronize()
    graph = th.cuda.CUDAGraph()
    with th.cuda.graph(graph):
        for _ in range(n):
            _lib.param_regularize(e.desc, _lib.REG_LP, 2, 1e-3, e.params, e.ws)
    graph.replay()
    start, end = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
    start.record()
    graph.replay()
    end.record()
    th.cuda.synchronize()
    return {"param_regularize_host_us": round(float(np.median(host)), 2),
            "k_param_regularize_device_us_per_launch": round(start.elapsed_time(end) * 1e3 / n, 2),
            "n_params": int(e.desc.n_params)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not th.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types

    rng = np.random.default_rng(0)
    frag = lambda: types.TrajectoryWithRew(obs=rng.standard_normal((L + 1, Do)).astype(np.float32),
                                           acts=rng.uniform(-1, 1, (L, Da)).astype(np.float32), infos=None,
                                           terminal=False, rews=rng.standard_normal(L).astype(np.float32))
    ds = pc.PreferenceDataset()
    ds.push([(frag(), frag()) for _ in range(P)], (rng.random(P) < 0.5).astype(np.float32))
    out = {}
    for setting in ("none", "lp2", "wd", "lp2_upd"):
        ms, n, extra = _time(setting, ds, a.calls, a.warmup)
        out[setting] = {"median_ms": round(ms, 3), "launches_per_call": n, **extra}
    name, power = _card()
    print(json.dumps({"bench": "pref_regularization", "calls": a.calls, "settings": out, "gpu": name,
                      "power_limit": power}))


if __name__ == "__main__":
    main()
