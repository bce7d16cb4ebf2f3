"""Active selection of preference queries at BASELINE config 5's shapes: Hopper-shaped obs 11 / act 3, fragment length
100, 2048 pairs per query round with oversampling factor 2 (4096 candidate pairs, 8192 fragments), a 5-member ensemble
of NormalizedRewardNet(BasicRewardNet 32x32) (the reference's ensemble config, scripts/ingredients/reward.py:55-64).

    python profiles/active_selection_bench.py [--steps K] [--warmup W] [--mode logit|probability|label]
                                              [--impl ours|reference] [--dump-outputs DIR]

One `ActiveSelectionFragmenter.__call__` is timed end to end (host clock; the call ends with the selection's read-back
and the timer waits for the pool's row copy), and split with CUDA events recorded around the library calls it makes:
base fragmenter (host: `RandomFragmenter`'s draws), staging upload (host stacking + copy to the staging table), member
forwards (one gather + one `imb_reward_forward` per member), scoring (`imb_pref_uncertainty`: fragment moments, output
norm fold, scores) and selection (stable sort, read-back of the selected indices, adoption into the fragment pool).  The
launch count is the library's (`_lib.LAUNCHES`); the torch sort and copies come on top.  The card's name and power
limit are read in the same run.

The reference arm runs the CPU restatement of the reference loop (one predict_processed per member and fragment) over a
bounded sample of candidates, as profiles/pref_bench.py does, and reports its per-candidate time.

`--dump-outputs DIR`: the last timed call's scores, the candidate indices of the pairs it returned (in the returned
order) and the members' output statistics, as .npy."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch as th

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

Do, Da, L, PAIRS, FACTOR, M = 11, 3, 100, 2048, 2, 5
N_TRAJ, T_LEN = 200, 1000


def _trajectories(rng):
    from imitation_b200.data import types

    return [types.TrajectoryWithRew(obs=rng.standard_normal((T_LEN + 1, Do)).astype(np.float32),
                                    acts=rng.uniform(-1, 1, (T_LEN, Da)).astype(np.float32), infos=None, terminal=True,
                                    rews=rng.standard_normal(T_LEN).astype(np.float32)) for _ in range(N_TRAJ)]


def _card():
    name = th.cuda.get_device_name() if th.cuda.is_available() else None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(th.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def reference(args):
    from oracle import nets_port, pref_port

    th.set_num_threads(min(8, os.cpu_count() or 1))
    rng = np.random.default_rng(0)
    n = 32
    pairs = []
    for _ in range(n):
        pairs.append(tuple(dict(obs=rng.standard_normal((L + 1, Do)).astype(np.float32),
                                acts=rng.uniform(-1, 1, (L, Da)).astype(np.float32), terminal=False) for _ in range(2)))
    th.manual_seed(0)
    members = [(nets_port.BasicRewardNetPort(Do, Da, hid_sizes=(32, 32)), nets_port.OutputNormPort()) for _ in range(M)]
    t0 = time.perf_counter()
    for a, b in pairs:
        r = []
        for f in (a, b):
            tr = pref_port.fragment_transitions(f)
            r.append(th.as_tensor(np.stack([out(nets_port.predict_port(net, *tr)) for net, out in members], -1)))
        (r[0].sum(0) - r[1].sum(0)).var().item()
    dt = (time.perf_counter() - t0) / n
    print(json.dumps({"impl": "reference", "metric": "active selection: ms per candidate pair", "value": dt * 1e3,
                      "unit": "ms/candidate", "higher_is_better": False, "cores": th.get_num_threads(),
                      "sample": f"{n} candidate pairs x {M} members, logit mode, CPU restatement of the reference loop",
                      "extrapolated_call_ms": dt * 1e3 * FACTOR * PAIRS}))


def main(args):
    if args.impl == "reference":
        return reference(args)
    if not th.cuda.is_available():
        raise SystemExit("the device arm needs a CUDA device")
    from imitation_b200 import _lib, spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import networks

    rng = np.random.default_rng(0)
    trajs = _trajectories(rng)
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1.0, 1.0, (Da,))
    th.manual_seed(0)
    members = [reward_nets.NormalizedRewardNet(reward_nets.BasicRewardNet(obs_space, act_space, hid_sizes=(32, 32)),
                                               networks.RunningNorm).cuda() for _ in range(M)]
    ens = reward_nets.RewardEnsemble(obs_space, act_space, members)
    pm = pc.PreferenceModel(ens)
    base = pc.RandomFragmenter(rng=np.random.default_rng(1), warning_threshold=0)
    frag = pc.ActiveSelectionFragmenter(pm, base, FACTOR, uncertainty_on=args.mode)

    # phase instrumentation: CUDA events around the library calls of one __call__
    marks = {}
    last = {}

    def ev():
        e = th.cuda.Event(enable_timing=True)
        e.record()
        return e

    def timed(phase, fn, keep=None):
        def wrapper(*a, **k):
            e0 = ev()
            out = fn(*a, **k)
            e1 = ev()
            marks.setdefault(phase, [e0, e1])[1] = e1
            if keep is not None:
                last[keep] = a
            return out
        return wrapper

    def host_base(**kw):
        t0 = time.perf_counter()
        out = base(**kw)
        marks["base_host_s"] = time.perf_counter() - t0
        marks["after_base"] = ev()
        last["candidates"] = out
        return out

    frag.base_fragmenter = host_base
    _lib.gather_rows = timed("forwards", _lib.gather_rows)
    _lib.reward_forward = timed("forwards", _lib.reward_forward)
    _lib.pref_uncertainty = timed("scoring", _lib.pref_uncertainty, keep="pu")

    def call():
        marks.clear()
        th.cuda.synchronize()
        t0 = time.perf_counter()
        out = frag(trajs, L, PAIRS)
        end = ev()
        end.synchronize()
        total = time.perf_counter() - t0
        ms = lambda a, b: a.elapsed_time(b)
        phases = {"base_fragmenter_host": marks["base_host_s"] * 1e3,
                  "staging_upload": ms(marks["after_base"], marks["forwards"][0]),
                  "member_forwards": ms(*marks["forwards"]),
                  "moments_fold_scoring": ms(*marks["scoring"]),
                  "selection_readback_adopt": ms(marks["scoring"][1], end)}
        return out, total * 1e3, phases

    for _ in range(max(1, args.warmup)):
        call()
    K = max(1, args.steps)
    totals, phases, launches = [], [], []
    for _ in range(K):
        l0 = _lib.LAUNCHES["count"]
        out, t, ph = call()
        launches.append(_lib.LAUNCHES["count"] - l0)
        totals.append(t)
        phases.append(ph)
    name, power = _card()
    med = {k: float(np.median([p[k] for p in phases])) for k in phases[0]}
    assert len(out) == PAIRS
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        a = last["pu"]
        np.save(os.path.join(args.dump_outputs, "scores.npy"), a[8].cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "output_stats.npy"),
                np.array([[m.normalize_output_layer.running_mean.item(), m.normalize_output_layer.running_var.item(),
                           float(m.normalize_output_layer.count.item())] for m in members], np.float64))
        index = {id(p): i for i, p in enumerate(last["candidates"])}  # the candidate index of every returned pair
        np.save(os.path.join(args.dump_outputs, "selected.npy"), np.array([index[id(p)] for p in out], np.int64))
    print(json.dumps({"impl": "ours", "metric": "active selection: one ActiveSelectionFragmenter call",
                      "value": float(np.median(totals)), "unit": "ms/call (median)", "higher_is_better": False,
                      "calls": K, "warmup": max(1, args.warmup), "ms_per_call_all": totals,
                      "phases_ms_median": med, "gpu_launches_per_call": launches[-1], "mode": args.mode,
                      "card": name, "power_limit": power,
                      "config": {"obs": Do, "act": Da, "fragment_length": L, "num_pairs": PAIRS, "factor": FACTOR,
                                 "candidates": FACTOR * PAIRS, "members": M,
                                 "member": "NormalizedRewardNet(BasicRewardNet 32x32, RunningNorm)",
                                 "trajectories": f"{N_TRAJ} x {T_LEN} steps"}}))


if __name__ == "__main__":
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--mode", default="logit", choices=["logit", "probability", "label"])
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    main(ap.parse_args())
