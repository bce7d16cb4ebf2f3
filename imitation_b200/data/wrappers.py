"""`BufferingWrapper` over the GPU-resident VecEnv (mirror of imitation.data.wrappers:13-169).

The reference records every env step in per-env Python lists and rebuilds trajectories at pop
time.  Here the rollout kernel writes each transition straight to its FINAL position in the
flattened order `pop_trajectories()` + `flatten_trajectories()` would produce (finished
trajectories in completion order, then partial ones in env order -- closed form for lock-step
fixed-horizon envs, csrc/imb_rollout.cu:flat_index), and, when a ReplayBuffer is attached,
also into the generator ring.  The host API below materialises NumPy views on demand.
"""
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch as th

from .. import _desc
from . import buffer as buffer_mod
from . import types


def finished_trajectories(venv, flat: np.ndarray, rews: np.ndarray) -> List[types.TrajectoryWithRew]:
    """The E finished trajectories of one lock-step episode segment of `venv` (a DeviceVecEnv, E envs), in env order:
    flat = the segment's transition rows [E * L][tw] (env-major, the reference order) and rews their ground-truth
    rewards [E * L]."""
    E = venv.num_envs
    tr = buffer_mod.rows_to_transitions(flat, venv.d_obs, venv.d_act, venv.observation_space.shape,
                                        venv.action_space.shape, venv.observation_space.dtype, venv.action_space.dtype,
                                        venv.discrete, rews=rews.astype(np.float32))
    L = len(flat) // E
    trajs = []
    for e in range(E):
        sl = slice(e * L, (e + 1) * L)
        trajs.append(types.TrajectoryWithRew(obs=np.concatenate([tr.obs[sl], tr.next_obs[sl][-1:]]), acts=tr.acts[sl],
                                             infos=None, terminal=True, rews=tr.rews[sl]))
    return trajs


class BufferingWrapper:
    def __init__(self, venv, error_on_premature_reset: bool = True):
        self.venv = venv
        self.num_envs = venv.num_envs
        self.observation_space, self.action_space = venv.observation_space, venv.action_space
        self.error_on_premature_reset = error_on_premature_reset
        self.n_transitions: Optional[int] = None
        self._init_reset = False
        self._ring: Optional[buffer_mod.ReplayBuffer] = None
        self._flat: Optional[th.Tensor] = None      # [E*T][tw] of the last rollout, reference order
        self._env_rews: Optional[th.Tensor] = None  # [E][T] ground-truth env rewards of the last rollout
        self._last: Optional[Tuple[int, int, int]] = None  # (T, t0, H) of the last rollout
        self._ep_lens: List[int] = []
        # earlier rollouts that have not been popped yet (the reference buffers every step until pop): per-env step
        # arrays [E][T_k][tw] and rewards [E][T_k], oldest first
        self._hist: List[Tuple[np.ndarray, np.ndarray, int]] = []
        self._unsaved = False  # the device buffers hold a rollout that is not in `_hist` yet

    # -- plumbing used by DevicePPO / AdversarialTrainer ------------------------------------------------------
    @property
    def state(self):
        return self.venv.state

    @property
    def device(self):
        return self.venv.device

    def attach_ring(self, ring: buffer_mod.ReplayBuffer) -> None:
        """Generator samples go straight into `ring` (AdversarialTrainer.train_gen's
        flatten_trajectories_with_rew + ReplayBuffer.store, common.py:422-425, fused)."""
        self._ring = ring

    def rollout_targets(self, n_steps: int):
        E = self.num_envs
        tw = _desc.table_width(self.venv.d_obs, self.venv.d_act)
        if self._flat is None or self._flat.shape[0] != E * n_steps:
            self.before_rollout()
            self._flat = th.zeros(E * n_steps, tw, device=self.venv.device)
        return self._flat, self._ring

    def before_rollout(self) -> None:
        """Called before every rollout (eager or graph replay): a rollout that is still waiting to be popped is copied
        off the device buffers the next one overwrites (several PPO rollouts per `train_gen`, common.py:408-419)."""
        if self._unsaved and self.n_transitions and self._flat is not None:
            T, t0, H = self._last
            self._hist.append((self._unflatten(self._flat.cpu().numpy(), T, t0, H),
                               self._env_rews.cpu().numpy().reshape(self.num_envs, T).copy(), t0))
        self._unsaved = False

    def after_rollout(self, n_steps: int, t0: int, env_rews: th.Tensor) -> None:
        H = self.venv.horizon
        self._last = (n_steps, t0, H)
        self._env_rews = env_rews
        self.n_transitions = (self.n_transitions or 0) + self.num_envs * n_steps
        self._unsaved = True
        self._ep_lens += [H] * (self.num_envs * ((t0 + n_steps) // H))
        if self._ring is not None:
            self._ring.note_stored(self.num_envs * n_steps)

    # -- reference API -----------------------------------------------------------------------------------------------
    def reset(self, **kwargs):
        if self._init_reset and self.error_on_premature_reset and self.n_transitions:
            raise RuntimeError("BufferingWrapper reset() before samples were accessed")
        self._init_reset = True
        self.n_transitions = 0
        return self.venv.reset(**kwargs)

    @staticmethod
    def _segments_of(T: int, t0: int, H: int):
        bounds = [0] + [b for b in range(H - t0, T, H)] + [T]
        return [(bounds[i], bounds[i + 1]) for i in range(len(bounds) - 1) if bounds[i + 1] > bounds[i]]

    def _segments(self):
        return self._segments_of(*self._last)

    def _unflatten(self, flat: np.ndarray, T: int, t0: int, H: int) -> np.ndarray:
        """reference-ordered rows [segment][env][step] -> per-env step arrays [E][T][tw]"""
        E = self.num_envs
        out = np.empty((E, T, flat.shape[1]), flat.dtype)
        off = 0
        for a, b in self._segments_of(T, t0, H):
            out[:, a:b] = flat[off:off + E * (b - a)].reshape(E, b - a, -1)
            off += E * (b - a)
        return out

    def _collect(self):
        """All buffered steps since the last pop as ([E][T][tw] rows, [E][T] env rewards, T, t0): the rollouts the
        reference's wrapper would have accumulated, joined in time."""
        rows, rews = [h[0] for h in self._hist], [h[1] for h in self._hist]
        t0_all = self._hist[0][2] if self._hist else None
        if self._unsaved:  # the device buffers hold a rollout that is not in the history yet
            T, t0, H = self._last
            rows.append(self._unflatten(self._flat.cpu().numpy(), T, t0, H))
            rews.append(self._env_rews.cpu().numpy().reshape(self.num_envs, T))
            if t0_all is None:
                t0_all = t0
        rows, rews = np.concatenate(rows, 1), np.concatenate(rews, 1)
        return rows, rews, rows.shape[1], t0_all

    def pop_transitions(self) -> types.TransitionsWithRew:
        if not self.n_transitions:
            raise RuntimeError("Called pop_transitions on an empty BufferingWrapper")
        v = self.venv
        H = self.venv.horizon
        rows, rews, T, t0 = self._collect()
        segs = self._segments_of(T, t0, H)
        flat = np.concatenate([rows[:, a:b].reshape(-1, rows.shape[2]) for a, b in segs])
        frews = np.concatenate([rews[:, a:b].reshape(-1) for a, b in segs])
        out = buffer_mod.rows_to_transitions(flat, v.d_obs, v.d_act, v.observation_space.shape,
                                             v.action_space.shape, v.observation_space.dtype, v.action_space.dtype,
                                             v.discrete, rews=frews.astype(np.float32))
        assert len(out.obs) >= self.n_transitions
        self._popped = (T, t0, H)
        self.discard()
        return out

    def discard(self) -> None:
        """Forget the buffered steps (AdversarialTrainer.train_gen: they already went into the replay ring)."""
        self.n_transitions = 0
        self._ep_lens = []
        self._hist = []
        self._unsaved = False

    def pop_trajectories(self) -> Tuple[Sequence[types.TrajectoryWithRew], Sequence[int]]:
        if not self.n_transitions:
            return [], []
        ep_lens = list(self._ep_lens)
        tr = self.pop_transitions()
        T, t0, H = self._popped
        E = self.num_envs
        trajs, off = [], 0
        segs = self._segments_of(T, t0, H)
        for si, (a, b) in enumerate(segs):
            L = b - a
            terminal = (t0 + b) % H == 0
            for e in range(E):
                sl = slice(off + e * L, off + (e + 1) * L)
                obs = np.concatenate([tr.obs[sl], tr.next_obs[sl][-1:]])
                trajs.append(types.TrajectoryWithRew(obs=obs, acts=tr.acts[sl], infos=None, terminal=bool(terminal),
                                                     rews=tr.rews[sl]))
            off += E * L
        return trajs, ep_lens

    def pop_finished_trajectories(self):
        """Finished trajectories (in completion order) and their lengths; the steps of episodes that are still running
        stay buffered and are joined with later rollouts (data/wrappers.py:113-130)."""
        if not self.n_transitions:
            return [], []
        v, H, E = self.venv, self.venv.horizon, self.num_envs
        rows, rews, T, t0 = self._collect()
        segs = self._segments_of(T, t0, H)
        keep_from = T
        if (t0 + segs[-1][1]) % H != 0:  # the last segment is an unfinished episode
            keep_from = segs[-1][0]
            segs = segs[:-1]
        trajs, lens = [], []
        for a, b in segs:
            trajs += finished_trajectories(v, rows[:, a:b].reshape(-1, rows.shape[2]), rews[:, a:b].reshape(-1))
            lens += [b - a] * E
        self.discard()
        if keep_from < T:
            # (like the reference, `n_transitions` restarts at 0 while the running episodes' steps stay in the accumulator)
            self._hist = [(rows[:, keep_from:].copy(), rews[:, keep_from:].copy(), (t0 + keep_from) % H)]
        return trajs, lens
