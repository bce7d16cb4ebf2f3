"""Member-parallel ensemble training with a regularizer (`EnsembleTrainer.set_distributed`, Lp p = 2 + an
`IntervalParamScaler` on a 0.2 validation split): every rank must end bit-identical to one process, the members'
regularizer strengths and the ensemble's reward/final/* keys included.

- On 2 GPUs: tests/dist_pref_regularization_worker.py under torch.distributed.run (NCCL), the real kernels.
- On the CPU: a world-2 gloo group with the CUDA pieces replaced by the stand-ins of tests/test_host_logic.py, plus
  stand-ins for the preference loss and the regularization kernel whose statistics depend on exactly which rows each
  minibatch gathered, so the lambda decisions, the validation split and the broadcasts all shape the result."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch as th
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.skipif(th.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_regularized_ensemble_is_bit_identical_to_one_process():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29537", os.path.join(ROOT, "tests", "dist_pref_regularization_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT)
    sys.stderr.write(r.stdout[-3000:] + r.stderr[-6000:])
    assert r.returncode == 0 and "DIST_PREF_REG_OK" in r.stdout


def _install_stand_ins():
    from imitation_b200 import _lib
    from tests.test_host_logic import _install_cpu_stand_ins

    _install_cpu_stand_ins()
    gathered = {"h": 0.0}
    gather = _lib.gather_rows

    def gather_rows(table, cap, tw, idx, n, batch, ld, col0):
        gather(table, cap, tw, idx, n, batch, ld, col0)
        w = th.arange(1, idx.numel() + 1, dtype=th.float64)
        gathered["h"] = float((idx.double() * w).sum() % 7919) / 7919.0

    def pref_loss(rews, n_pairs, frag_len, prefs, noise_prob, discount, threshold, grad_scale, grad_rews, probs_out,
                  stats_acc, stats_slot=0):
        if stats_acc is not None:
            stats_acc[4 * stats_slot] += 0.2 + gathered["h"]
            stats_acc[4 * stats_slot + 1] += 0.5
            stats_acc[4 * stats_slot + 2] += 1.0

    def param_regularize(d, kind, p, coeff, params, ws, stats_acc=None, stats_slot=0):
        if kind == _lib.REG_LP:
            params.mul_(1.0 - 1e-2 * coeff)  # makes the parameters depend on every lambda
            if stats_acc is not None:
                stats_acc[4 * stats_slot] += coeff * float(params.abs().sum())
                stats_acc[4 * stats_slot + 2] += 1.0
        else:
            params.add_(coeff * params)

    _lib.gather_rows, _lib.pref_loss, _lib.param_regularize = gather_rows, pref_loss, param_regularize


def _run(distributed: bool):
    from imitation_b200 import spaces
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.data import types
    from imitation_b200.regularization import IntervalParamScaler, LpRegularizer
    from imitation_b200.rewards import reward_nets
    from imitation_b200.util import logger

    Do, Da, L, P = 5, 2, 4, 20
    rng = np.random.default_rng(0)
    obs_space, act_space = spaces.Box(-np.inf, np.inf, (Do,)), spaces.Box(-1.0, 1.0, (Da,))

    def frag():
        return types.TrajectoryWithRew(obs=rng.standard_normal((L + 1, Do)).astype(np.float32),
                                       acts=rng.uniform(-1, 1, (L, Da)).astype(np.float32), infos=None, terminal=False,
                                       rews=rng.standard_normal(L).astype(np.float32))

    ds = pc.PreferenceDataset()
    ds.push([(frag(), frag()) for _ in range(P)], (rng.random(P) < 0.5).astype(np.float32))
    th.manual_seed(3)
    members = [reward_nets.BasicRewardNet(obs_space, act_space, hid_sizes=(32, 32)) for _ in range(3)]
    ens = reward_nets.RewardEnsemble(obs_space, act_space, members)
    pm = pc.PreferenceModel(ens)
    pm._pool = pc.FragmentPool(Do, Da, False, "cpu")
    lg = logger.configure()
    factory = LpRegularizer.create(0.5, IntervalParamScaler(0.25, (0.45, 0.6)), val_split=0.2, p=2)
    et = pc.EnsembleTrainer(pm, pc.CrossEntropyRewardLoss(), rng=np.random.default_rng(1), batch_size=4,
                            minibatch_size=2, epochs=2, lr=1e-2, custom_logger=lg, regularizer_factory=factory)
    if distributed:
        et.set_distributed()
    th.manual_seed(11)
    et.train(ds)
    et.train(ds, epoch_multiplier=1.5)
    return ([m.mlp.dense0.weight.detach().clone() for m in members],
            [float(t.optim.state[m.mlp.dense0.weight]["step"]) for t, m in zip(et.member_trainers, members)],
            [t.regularizer.lambda_ for t in et.member_trainers],
            {k: float(v) for k, v in lg.name_to_value.items() if k.startswith("reward/final/")}, float(th.rand(1)))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist

    sys.path.insert(0, ROOT)
    _install_stand_ins()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out[rank] = _run(True)
    dist.destroy_process_group()


def _single(_i, out):
    sys.path.insert(0, ROOT)
    _install_stand_ins()
    out["single"] = _run(False)


def test_regularized_member_parallel_ensemble_equals_single_process_world2_gloo():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_single, args=(out,), nprocs=1, join=True)
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    w0, s0, lam0, final0, p0 = out["single"]
    assert len({float(w.sum()) for w in w0}) == 3 and all(s > 0 for s in s0)
    assert len(set(lam0)) > 1 and all(lam != 0.5 for lam in lam0), lam0  # lambda moved, differently per member
    for key in ("regularized_loss", "regularization_lambda", "val/loss", "val/accuracy", "val/gt_reward_loss"):
        assert f"reward/final/{key}" in final0 and f"reward/final/{key}_std" in final0, key
    for r in range(world):
        w, s, lam, final, p = out[r]
        assert s == s0 and lam == lam0 and p == p0, (r, s, s0, lam, lam0, p, p0)
        assert final == final0, (r, final, final0)
        for a, b in zip(w, w0):
            assert th.equal(a, b), f"rank {r}: member parameters differ from the single-process run"
