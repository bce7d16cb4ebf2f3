"""Multi-GPU plumbing: one process per GPU, `torch.distributed` (NCCL over NVLink / NVSwitch).

The path shards by environment: rank r owns envs [r*E, (r+1)*E), its rollout table, its
generator ring and its expert sampling stream; nothing on the data path crosses ranks.  The
only exchange is ONE all-reduce per round (north_star: "a single NCCL all-reduce on
discriminator and policy gradients per round"): every rank runs its round locally (PPO epochs
+ discriminator updates on its shard), then a single flat fp32 buffer

    [policy params | policy Adam m, v | disc params | disc Adam m, v | RunningNorm S0,S1,S2 ...]

is summed and turned back into the replica state: parameters and moments are averaged (the sum
of the per-rank updates of the round, i.e. local-update data parallelism), RunningNorm
statistics are merged EXACTLY through their additive sufficient statistics
(S0 = n, S1 = n*mean, S2 = n*(var + mean^2)) relative to the common round-start state.
Payload ~60 KB => latency-bound (~20-30 us on NVSwitch), independent of env count.

Works with any backend (`gloo` on CPU for the host-logic tests, `nccl` on GPUs).
"""
from typing import List, Optional, Sequence, Tuple

import torch as th
import torch.distributed as dist


def env_slice(global_envs: int, rank: int, world: int) -> Tuple[int, int]:
    """(offset, count) of rank's env slice; global_envs must divide evenly."""
    if global_envs % world != 0:
        raise ValueError(f"num_envs={global_envs} must be divisible by world size {world}")
    per = global_envs // world
    return rank * per, per


class NormStat:
    """A RunningNorm (mean, var, count) triple registered for exact cross-rank merging."""

    def __init__(self, mean: th.Tensor, var: th.Tensor, count: th.Tensor):
        self.mean, self.var, self.count = mean, var, count
        self.start: Optional[Tuple[th.Tensor, th.Tensor, th.Tensor]] = None

    def snapshot(self) -> None:
        self.start = (self.mean.clone(), self.var.clone(), self.count.clone())

    @staticmethod
    def suff(mean, var, count):
        n = count.to(th.float64)
        m = mean.to(th.float64)
        return n.reshape(1), n * m, n * (var.to(th.float64) + m * m)

    def pack(self) -> th.Tensor:
        return th.cat([t.reshape(-1) for t in self.suff(self.mean, self.var, self.count)])

    def unpack(self, summed: th.Tensor, world: int) -> None:
        k = self.mean.numel()
        s0, s1, s2 = self.suff(*self.start)
        n = summed[0:1] - (world - 1) * s0
        a = summed[1:1 + k] - (world - 1) * s1
        b = summed[1 + k:1 + 2 * k] - (world - 1) * s2
        if float(n) > 0:
            mean = a / n
            self.mean.copy_(mean.to(self.mean.dtype))
            self.var.copy_((b / n - mean * mean).clamp_min(0).to(self.var.dtype))
        self.count.copy_(n.round().to(self.count.dtype).reshape(self.count.shape))

    def numel(self) -> int:
        return 1 + 2 * self.mean.numel()


class RoundSync:
    """One all-reduce per round over [averaged tensors | norm sufficient statistics]."""

    def __init__(self, averaged: Sequence[th.Tensor], norms: Sequence[NormStat] = (), group=None):
        self.averaged = list(averaged)
        self.norms = list(norms)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        dev = self.averaged[0].device
        n_avg = sum(t.numel() for t in self.averaged)
        n_norm = sum(n.numel() for n in self.norms)
        # float64 staging keeps the sufficient statistics exact; payload is tiny (latency-bound)
        self.buf = th.zeros(n_avg + n_norm, dtype=th.float64, device=dev)
        self.n_avg = n_avg
        # CUDA tensors: pack / snapshot / unpack are one kernel each (csrc/imb_sync.cu) instead of ~60 tiny torch
        # ops and a host sync per round; CPU tensors (gloo host-logic tests) keep the torch formulation below.
        self._fused = None
        if dev.type == "cuda":
            from . import _lib
            self._fused = _lib.sync_desc(self.averaged, [(n.mean, n.var, n.count) for n in self.norms])
            assert _lib.sync_buffer_doubles(self._fused) == self.buf.numel()
            self._start = th.zeros(max(n_norm, 1), dtype=th.float64, device=dev)

    def begin_round(self) -> None:
        if self._fused is not None:
            from . import _lib
            _lib.sync_snapshot(self._fused, self._start)
            return
        for n in self.norms:
            n.snapshot()

    def broadcast_initial(self, src: int = 0) -> None:
        """Make every replica start from rank `src`'s parameters."""
        if self.world == 1:
            return
        for t in self.averaged:
            dist.broadcast(t, src, group=self.group)
        for n in self.norms:
            dist.broadcast(n.mean, src, group=self.group)
            dist.broadcast(n.var, src, group=self.group)
            dist.broadcast(n.count, src, group=self.group)

    def end_round(self) -> None:
        if self.world == 1:
            return
        if self._fused is not None:
            from . import _lib
            _lib.sync_pack(self._fused, self.buf)
            dist.all_reduce(self.buf, op=dist.ReduceOp.SUM, group=self.group)  # the single collective of the round
            _lib.sync_unpack(self._fused, self.buf, self._start, self.world)
            return
        o = 0
        for t in self.averaged:
            self.buf[o:o + t.numel()] = t.reshape(-1).to(th.float64)
            o += t.numel()
        for n in self.norms:
            self.buf[o:o + n.numel()] = n.pack()
            o += n.numel()
        dist.all_reduce(self.buf, op=dist.ReduceOp.SUM, group=self.group)  # the single collective of the round
        o = 0
        for t in self.averaged:
            t.copy_((self.buf[o:o + t.numel()] / self.world).to(t.dtype).view(t.shape))
            o += t.numel()
        for n in self.norms:
            n.unpack(self.buf[o:o + n.numel()], self.world)
            o += n.numel()


def trainer_round_sync(trainer, group=None) -> RoundSync:
    """Collect the replica state of an AdversarialTrainer (fused path) for RoundSync."""
    gen = trainer.gen_algo
    pp, pn, pc = gen.policy.flat_vectors()
    eng = trainer._fused_net.engine()
    opt = trainer._disc_opt
    # a trainer in distributed mode (`set_distributed`) keeps its discriminator replicas identical by itself: every
    # optimiser step is a global-batch step (gradient all-reduce).  Only the generator is synchronised per round then.
    disc_is_global = getattr(trainer, "_dist_world", 1) > 1
    averaged = [pp, gen.exp_avg, gen.exp_avg_sq]
    if not disc_is_global:
        averaged += [eng.params, opt.exp_avg, opt.exp_avg_sq]
    norms: List[NormStat] = []
    if gen.policy.normalize_features:
        k = gen.policy.d_obs
        norms.append(NormStat(pn[:k], pn[k:2 * k], pc[0:1]))
    off = 0
    for i, n in enumerate(eng.norms):
        k = n.running_mean.numel()
        if not disc_is_global:
            norms.append(NormStat(eng.norm_state[off:off + k], eng.norm_state[off + k:off + 2 * k],
                                  eng.norm_count[i:i + 1]))
        off += 2 * k
    return RoundSync(averaged, norms, group)
