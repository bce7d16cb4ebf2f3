"""Per-phase cycle counts of the persistent PPO update (CTA 0 / thread 0 clock64 deltas).
Build the timing variant first:
  IMB_VARIANT=_timing IMB_EXTRA_NVCC_FLAGS=-DIMB_PPO_TIMING python imitation_b200/_build.py
then run with IMB_VARIANT=_timing."""
import ctypes
import os
import sys

import torch as th

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from imitation_b200 import _desc, _lib  # noqa: E402

NAMES = ["top barrier", "-", "-", "chain + early wgrad blocks", "-", "-", "-",
         "policy dW1/b1 -> GP", "push partials (7 peers)", "barrier a wait", "slice sum + norm exchange issue", "wait: slice norms landed",
         "clip + Adam (own slice) + parameter all-gather + wait", "-"]
pd = _desc.policy_desc(17, 6, False, 32, True)
N = 4096
rw = _lib.rollout_row_width(pd)
tbl = th.randn(N, rw, device="cuda")
tbl[:, 17 + 6] = -8.0 + 0.1 * th.randn(N, device="cuda")
P = (th.rand(pd.n_params, device="cuda") - 0.5) * 0.3
PN = th.cat([th.zeros(17), th.ones(17)]).cuda()
PC = th.zeros(1, dtype=th.int32, device="cuda")
M, V = th.zeros_like(P), th.zeros_like(P)
st = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
hp = _lib.PpoHparams(gamma=0.95, gae_lambda=0.95, clip_range=0.1, ent_coef=4e-6, vf_coef=0.11, max_grad_norm=0.8,
                     lr=2.6e-4, adam_eps=1e-5, n_epochs=5, batch_size=64, normalize_advantage=1)
for _ in range(3):
    _lib.ppo_update(pd, P, PN, PC, M, V, tbl, N, hp, None, 0, None, st)
th.cuda.synchronize()
_lib.lib().imb_debug_ppo_warp_clocks(None, 1)
e0, e1 = th.cuda.Event(enable_timing=True), th.cuda.Event(enable_timing=True)
e0.record()
_lib.ppo_update(pd, P, PN, PC, M, V, tbl, N, hp, None, 0, None, st)
e1.record()
th.cuda.synchronize()
steps = 5 * N // 64
print(f"launch {e0.elapsed_time(e1):.3f} ms, {e0.elapsed_time(e1) * 1e3 / steps:.2f} us/step")
out = (ctypes.c_longlong * 16)()
rc = _lib.lib().imb_debug_ppo_clocks(out)
assert rc == 0, rc
tot = sum(out[:14])
for n, c in zip(NAMES, out):
    print(f"{n:<18s} {c / steps:9.0f} cycles/step  {100.0 * c / tot:5.1f} %")
print(f"{'total':<18s} {tot / steps:9.0f} cycles/step")

w = (ctypes.c_longlong * 80)()
assert _lib.lib().imb_debug_ppo_warp_clocks(w, 0) == 0
print("per-warp cycles/step since the top barrier (CTA 0; warps 0,1 policy tower, 2,3 value tower; warps 4-7: slot 1 = "
      "next-step stats done (in the step's tail), slot 3 = prefetch issued (beside the chain); early weight-gradient "
      "blocks: value dW2, policy head and policy dW2 on warps 4-7, value dW1 on warps 2,3).\n"
      "Each warp counts from its own read of the clock after the top barrier; the rows of warps that reach that barrier "
      "early (4-7) run ahead of the others' by about their wait there: align them on the post-chain barrier row, which "
      "thread 0 passes at the 'chain + early wgrad blocks' total above.")
for slot, name in ((1, "stats done (w4-7)"), (3, "after layer 1 | prefetch"), (4, "after layer 2"), (5, "after means (policy)"), (6, "after logp reduce"),
                   (7, "after dM/dlogstd | head wgrad (w4-7)"), (2, "after heads/loss"), (0, "chain end"),
                   (9, "value dW1 (w2,3) | value dW2 (w4-7)"), (8, "early wgrad blocks done (w2-7)"),
                   (6, "after logp reduce | post-chain barrier (w2-7)")):
    print(f"  {name:<36s}", [round(w[slot * 8 + i] / steps) for i in range(8)])
