"""Worker of tests/test_pref_regularization_dist.py: one process per GPU under torch.distributed.run (NCCL).

A member-parallel `EnsembleTrainer` (`set_distributed`) with an Lp regularizer (p = 2) and an `IntervalParamScaler` on a
0.2 validation split: every rank trains member k iff k % W == rank, makes the split and shuffle draws of the members it
skips, then the owners broadcast.  On EVERY rank the members' parameters, AdamW state, step counts, regularizer
strengths and the ensemble's reward/final/* keys must equal those of the single-process training of all members,
which every rank also runs locally as its own reference (same seeds, same dataset)."""
import os
import sys

import numpy as np
import torch as th
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(distributed: bool):
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import IntervalParamScaler, LpRegularizer
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import logger, networks

    Do, Da, L, P, M = 11, 3, 20, 96, 3
    rng = np.random.default_rng(0)
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1.0, 1.0, (Da,))

    def frag():
        return types.TrajectoryWithRew(obs=rng.standard_normal((L + 1, Do)).astype(np.float32),
                                       acts=rng.uniform(-1, 1, (L, Da)).astype(np.float32), infos=None, terminal=False,
                                       rews=rng.standard_normal(L).astype(np.float32))

    ds = pc.PreferenceDataset()
    ds.push([(frag(), frag()) for _ in range(P)], (rng.random(P) < 0.5).astype(np.float32))
    th.manual_seed(3)
    members = [reward_nets.BasicRewardNet(obs_space, act_space, hid_sizes=(32, 32),
                                          normalize_input_layer=networks.RunningNorm).cuda() for _ in range(M)]
    ens = reward_nets.RewardEnsemble(obs_space, act_space, members)
    lg = logger.configure()
    factory = LpRegularizer.create(0.05, IntervalParamScaler(0.1, (1.1, 1.5)), val_split=0.2, p=2)
    et = pc.EnsembleTrainer(pc.PreferenceModel(ens), pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(1),
                            batch_size=32, minibatch_size=16, epochs=2, lr=1e-3, custom_logger=lg,
                            regularizer_factory=factory)
    if distributed:
        et.set_distributed()
    th.manual_seed(11)
    et.train(ds)
    et.train(ds, epoch_multiplier=1.5)
    th.cuda.synchronize()
    state = []
    for m, t in zip(members, et.member_trainers):
        e = m.engine()
        state.append(th.cat([e.params, e.norm_state, e.norm_count.float(), t._fused_opt["m"], t._fused_opt["v"],
                             th.tensor([float(t.optim.state[e._param_list()[0]]["step"])], device="cuda")]).clone())
    lambdas = [t.regularizer.lambda_ for t in et.member_trainers]
    final = {k: float(v) for k, v in lg.name_to_value.items() if k.startswith("reward/final/")}
    return state, lambdas, final, float(th.rand(1))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    th.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=th.device("cuda", local))
    want, want_lam, want_final, want_probe = run(distributed=False)  # every rank: all members, single-process semantics
    got, got_lam, got_final, got_probe = run(distributed=True)       # member k on rank k % W, then broadcasts
    assert len({float(w.sum()) for w in want}) == len(want), "the members did not train differently"
    assert all(lam != 0.05 for lam in want_lam), "the updater never changed lambda"
    for k, (a, b) in enumerate(zip(got, want)):
        assert th.equal(a, b), f"rank {rank}: member {k} differs from the single-process run (max |d| = {(a - b).abs().max()})"
    assert got_lam == want_lam, (rank, got_lam, want_lam)
    assert got_probe == want_probe, "torch's global RNG ended in a different state"
    for key in ("reward/final/regularized_loss", "reward/final/regularization_lambda", "reward/final/val/loss",
                "reward/final/val/accuracy", "reward/final/val/gt_reward_loss"):
        assert key in want_final and key + "_std" in want_final, key
    assert got_final == want_final, (rank, got_final, want_final)
    x = th.cat(got + [th.tensor(got_lam, dtype=th.float32, device="cuda")])
    all_x = [th.empty_like(x) for _ in range(world)]
    dist.all_gather(all_x, x)
    assert all(th.equal(all_x[0], y) for y in all_x[1:])
    dist.barrier()
    if rank == 0:
        print("DIST_PREF_REG_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
