"""ctypes binding of libimb.so (the C-ABI declared in include/imb.h).

There is NO fallback: if the shared library is missing or a call fails, this module raises.
All pointers handed to the library are device pointers of torch CUDA tensors.
"""
import ctypes as C
import os
from typing import Optional

import torch as th

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libimb" + os.environ.get("IMB_VARIANT", "") + ".so")  # IMB_VARIANT: profiling builds

IMB_TILE_ROWS = 128
IMB_MAX_HIDDEN = 64
IMB_MAX_DIN = 64
IMB_F_ZERO_GRAD = 1
IMB_F_TRAIN_NORM = 2
IMB_F_NO_TENSOR = 4   # force the fp32-FFMA discriminator kernel (A/B measurements)
IMB_RF_DETERMINISTIC = 1  # imb_rollout flags

# device-resident counter block (include/imb.h enum)
ST_RING_IDX, ST_RING_N, ST_EP_STEP, ST_EPISODE, ST_GLOBAL_STEP, ST_REPLAY_DRAW = 0, 1, 2, 3, 4, 5
ST_EXPERT_POS, ST_EXPERT_EPOCH, ST_PPO_EPOCH, ST_DISC_STEP, ST_PPO_STEP, ST_WORDS = 6, 7, 8, 9, 10, 16


class ImbError(RuntimeError):
    pass


class Mlp(C.Structure):
    _fields_ = [("din", C.c_int32), ("n_hidden", C.c_int32), ("h1", C.c_int32), ("h2", C.c_int32),
                ("n_out", C.c_int32), ("has_norm", C.c_int32), ("param_off", C.c_int32), ("norm_off", C.c_int32),
                ("count_idx", C.c_int32), ("norm_eps", C.c_float)]


class DiscDesc(C.Structure):
    _fields_ = [("d_obs", C.c_int32), ("d_act", C.c_int32), ("use_state", C.c_int32), ("use_action", C.c_int32),
                ("use_next_state", C.c_int32), ("use_done", C.c_int32), ("base", Mlp), ("shaped", C.c_int32),
                ("potential", Mlp), ("gamma", C.c_float), ("subtract_logp", C.c_int32), ("n_params", C.c_int32)]


class Adam(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float)]  # > 0: torch.optim.AdamW's decoupled decay


class PolicyDesc(C.Structure):
    _fields_ = [("d_obs", C.c_int32), ("d_act", C.c_int32), ("discrete", C.c_int32), ("hidden", C.c_int32),
                ("has_norm", C.c_int32), ("norm_eps", C.c_float),
                ("off_pi_w1", C.c_int32), ("off_pi_b1", C.c_int32), ("off_pi_w2", C.c_int32), ("off_pi_b2", C.c_int32),
                ("off_vf_w1", C.c_int32), ("off_vf_b1", C.c_int32), ("off_vf_w2", C.c_int32), ("off_vf_b2", C.c_int32),
                ("off_act_w", C.c_int32), ("off_act_b", C.c_int32), ("off_val_w", C.c_int32), ("off_val_b", C.c_int32),
                ("off_log_std", C.c_int32), ("n_params", C.c_int32)]


class EnvDesc(C.Structure):
    _fields_ = [("d_obs", C.c_int32), ("d_act", C.c_int32), ("discrete", C.c_int32), ("horizon", C.c_int32),
                ("seed", C.c_uint64), ("env_id_offset", C.c_int64)]


class PpoHparams(C.Structure):
    _fields_ = [("gamma", C.c_float), ("gae_lambda", C.c_float), ("clip_range", C.c_float), ("ent_coef", C.c_float),
                ("vf_coef", C.c_float), ("max_grad_norm", C.c_float), ("lr", C.c_float), ("adam_eps", C.c_float),
                ("n_epochs", C.c_int32), ("batch_size", C.c_int32), ("normalize_advantage", C.c_int32)]


PU_MAX_MEMBERS = 16


class PrefUncDesc(C.Structure):
    _fields_ = [("n_members", C.c_int32), ("rews", C.c_void_p * PU_MAX_MEMBERS),
                ("norm_state", C.c_void_p * PU_MAX_MEMBERS), ("norm_count", C.c_void_p * PU_MAX_MEMBERS),
                ("norm_eps", C.c_float * PU_MAX_MEMBERS), ("norm_kind", C.c_int32 * PU_MAX_MEMBERS),
                ("norm_decay", C.c_float * PU_MAX_MEMBERS)]


PU_MODES = {"logit": 0, "probability": 1, "label": 2}


class RolloutMembers(C.Structure):
    _fields_ = [("n_members", C.c_int32), ("params", C.c_void_p * PU_MAX_MEMBERS),
                ("norm_state", C.c_void_p * PU_MAX_MEMBERS), ("raw", C.c_void_p)]

SYNC_MAX_AVG, SYNC_MAX_NORM = 8, 4


class SyncDesc(C.Structure):
    _fields_ = [("n_avg", C.c_int32), ("n_norm", C.c_int32), ("avg", C.c_void_p * SYNC_MAX_AVG),
                ("avg_n", C.c_int64 * SYNC_MAX_AVG), ("mean", C.c_void_p * SYNC_MAX_NORM),
                ("var", C.c_void_p * SYNC_MAX_NORM), ("count", C.c_void_p * SYNC_MAX_NORM),
                ("k", C.c_int32 * SYNC_MAX_NORM)]


_lib: Optional[C.CDLL] = None

# every symbol include/imb.h declares (tests check the library exports each of them)
SYMBOLS = [
    "imb_version", "imb_last_error", "imb_disc_workspace_floats", "imb_disc_norm_update", "imb_disc_fwd_bwd",
    "imb_disc_reduce", "imb_disc_adam", "imb_reward_forward", "imb_reward_norm_scan", "imb_reward_ema_scan",
    "imb_table_store",
    "imb_ring_advance", "imb_sample_indices", "imb_gather_rows", "imb_rollout", "imb_rollout_row_width", "imb_gae",
    "imb_rollout_advance", "imb_env_reset", "imb_ppo_update", "imb_policy_logp", "imb_state_init",
    "imb_sync_buffer_doubles", "imb_sync_snapshot", "imb_sync_pack", "imb_sync_unpack",
    "imb_disc_sample_gather", "imb_sample_advance2", "imb_disc_reduce_adam", "imb_norm_batch_stats", "imb_norm_fold",
    "imb_disc_set_rows", "imb_stats_publish", "imb_pref_loss", "imb_pref_uncertainty_ws_floats", "imb_pref_uncertainty",
    "imb_rollout_ensemble", "imb_ensemble_relabel_ws_floats", "imb_ensemble_relabel", "imb_disc_plan", "imb_ppo_plan",
    "imb_ppo_update_variant",
]

# imb_disc_plan codes: the kernel imb_disc_fwd_bwd runs
PLAN_TC, PLAN_FFMA128X2, PLAN_FFMA256, PLAN_FFMA128 = 1, 2, 3, 4
# imb_ppo_plan codes: the kernel imb_ppo_update runs
PPO_PLAN_UPDATE, PPO_PLAN_GEN1, PPO_PLAN_GEN2 = 1, 2, 3


def lib() -> C.CDLL:
    """Load libimb.so; raise loudly (no CPU fallback) if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a). imitation_b200 has no CPU fallback.")
        _lib = C.CDLL(LIB_PATH)
        _lib.imb_last_error.restype = C.c_char_p
        _lib.imb_disc_workspace_floats.restype = C.c_int64
        _lib.imb_sync_buffer_doubles.restype = C.c_int64
        _lib.imb_pref_uncertainty_ws_floats.restype = C.c_int64
        _lib.imb_ensemble_relabel_ws_floats.restype = C.c_int64
        for name in SYMBOLS:
            getattr(_lib, name)  # AttributeError if the .so is stale
    return _lib


# kernel launches issued through this binding (bench.py reports them as `gpu_launches`)
LAUNCHES = {"count": 0}
_KERNELS_PER_CALL = {
    "imb_state_init": 0, "imb_disc_norm_update": None, "imb_disc_fwd_bwd": 1, "imb_disc_reduce": 1,
    "imb_disc_adam": 1, "imb_reward_forward": 1, "imb_reward_norm_scan": 1, "imb_reward_ema_scan": 1,
    "imb_table_store": 1,
    "imb_ring_advance": 1, "imb_sample_indices": 2, "imb_gather_rows": 1, "imb_rollout": 1, "imb_gae": 1,
    "imb_rollout_advance": 1, "imb_env_reset": 1, "imb_ppo_update": 1, "imb_policy_logp": 1,
    "imb_disc_sample_gather": 1, "imb_sample_advance2": 1, "imb_disc_reduce_adam": 1, "imb_norm_batch_stats": 1,
    "imb_norm_fold": 1, "imb_disc_set_rows": 1, "imb_stats_publish": 1, "imb_pref_loss": 1,
    "imb_pref_uncertainty": None, "imb_rollout_ensemble": 1, "imb_ensemble_relabel": None,
}


def _check(rc: int, what: str, n_kernels: Optional[int] = None):
    LAUNCHES["count"] += _KERNELS_PER_CALL.get(what, 1) if n_kernels is None else n_kernels
    if rc != 0:
        raise ImbError(f"{what}: {lib().imb_last_error().decode()} (rc={rc})")


def _p(t: Optional[th.Tensor], dtype=None):
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise ImbError("imitation_b200 kernels need CUDA tensors (no CPU path)")
    if not t.is_contiguous():
        raise ImbError("tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise ImbError(f"expected dtype {dtype}, got {t.dtype}")
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(th.cuda.current_stream().cuda_stream)


def disc_workspace_floats(d: DiscDesc) -> int:
    return int(lib().imb_disc_workspace_floats(C.byref(d)))


def sync_desc(averaged, norms) -> SyncDesc:
    """averaged: fp32 CUDA tensors; norms: (mean[k], var[k], int32 count) tensor triples (views are fine as
    long as they are contiguous)."""
    if len(averaged) > SYNC_MAX_AVG or len(norms) > SYNC_MAX_NORM:
        raise ImbError("too many tensors for one imb_sync_desc")
    d = SyncDesc()
    d.n_avg, d.n_norm = len(averaged), len(norms)
    for i, t in enumerate(averaged):
        d.avg[i], d.avg_n[i] = _p(t, th.float32).value, t.numel()
    for i, (m, v, c) in enumerate(norms):
        d.mean[i], d.var[i], d.count[i] = _p(m, th.float32).value, _p(v, th.float32).value, _p(c, th.int32).value
        d.k[i] = m.numel()
    return d


def sync_buffer_doubles(d: SyncDesc) -> int:
    return int(lib().imb_sync_buffer_doubles(C.byref(d)))


def sync_snapshot(d: SyncDesc, start):
    _check(lib().imb_sync_snapshot(C.byref(d), _p(start, th.float64), _stream()), "imb_sync_snapshot",
           1 if d.n_norm else 0)


def sync_pack(d: SyncDesc, buf):
    _check(lib().imb_sync_pack(C.byref(d), _p(buf, th.float64), _stream()), "imb_sync_pack")


def sync_unpack(d: SyncDesc, buf, start, world: int):
    _check(lib().imb_sync_unpack(C.byref(d), _p(buf, th.float64), _p(start, th.float64), C.c_int32(world), _stream()),
           "imb_sync_unpack")


def state_init(state):
    _check(lib().imb_state_init(_p(state, th.int64), _stream()), "imb_state_init")


def disc_norm_update(d, batch, ld, n, norm_state, norm_count, ws):
    _check(lib().imb_disc_norm_update(C.byref(d), _p(batch, th.float32), C.c_int64(ld), C.c_int64(n),
                                      _p(norm_state, th.float32), _p(norm_count, th.int32), _p(ws, th.float32),
                                      _stream()), "imb_disc_norm_update",
           1 if (d.shaped and d.potential.has_norm) else int(d.base.has_norm))  # shaped: one multi-job launch


def norm_batch_stats(d, batch, ld, n, row0, din, norm_state, norm_count, defer, defer_cap, ws):
    """RunningNorm update of a foreign normaliser (the policy's feature extractor) from batch rows [row0, row0 + din);
    `defer` = slot list for a later in-order `norm_fold` (None: fold immediately)."""
    _check(lib().imb_norm_batch_stats(C.byref(d), _p(batch, th.float32), C.c_int64(ld), C.c_int64(n), C.c_int(row0),
                                      C.c_int(din), _p(norm_state, th.float32), _p(norm_count, th.int32), _p(defer),
                                      C.c_int(defer_cap), _p(ws, th.float32), _stream()), "imb_norm_batch_stats")


def norm_fold(din, defer, norm_state, norm_count, n_slots=0):
    _check(lib().imb_norm_fold(C.c_int(din), _p(defer, th.float32), _p(norm_state, th.float32),
                               _p(norm_count, th.int32), C.c_int(n_slots), _stream()), "imb_norm_fold")


def stats_publish(stats_dev, n, host_pinned, state, state_idx):
    """host_pinned: a pinned (page-locked, hence device-mapped under unified addressing) float32 CPU tensor of 16 elements."""
    if host_pinned.is_cuda or not host_pinned.is_pinned() or host_pinned.numel() < 16:
        raise ImbError("stats_publish needs a pinned CPU tensor of >= 16 floats")
    _check(lib().imb_stats_publish(_p(stats_dev, th.float32), C.c_int(n), C.c_void_p(host_pinned.data_ptr()),
                                   _p(state, th.int64), C.c_int(state_idx), _stream()), "imb_stats_publish")


def disc_set_rows(d, ws, n_rows_total, n_expert_total):
    _check(lib().imb_disc_set_rows(C.byref(d), _p(ws, th.float32), C.c_int64(n_rows_total), C.c_int64(n_expert_total),
                                   _stream()), "imb_disc_set_rows")


def disc_fwd_bwd(d, params, norm_state, batch, ld, n, n_expert, loss_scale, grad_out, logits_out, flags, ws):
    _check(lib().imb_disc_fwd_bwd(C.byref(d), _p(params, th.float32), _p(norm_state, th.float32),
                                  _p(batch, th.float32), C.c_int64(ld), C.c_int64(n), C.c_int64(n_expert),
                                  C.c_float(loss_scale), _p(grad_out), _p(logits_out), C.c_int(flags),
                                  _p(ws, th.float32), _stream()), "imb_disc_fwd_bwd")


def disc_plan(d: DiscDesc, n: int) -> int:
    """PLAN_* code of the kernel `disc_fwd_bwd` runs for `d` over n rows (host only, no GPU needed); ImbError naming
    the shared-memory limit when the fused kernels cannot run the shape."""
    rc = int(lib().imb_disc_plan(C.byref(d), C.c_int64(n)))
    if rc < 0:
        raise ImbError(f"imb_disc_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def disc_reduce(d, ws, grad_out_flat=None):
    _check(lib().imb_disc_reduce(C.byref(d), _p(ws, th.float32), _p(grad_out_flat), _stream()), "imb_disc_reduce")


def disc_adam(d, opt: Adam, params, exp_avg, exp_avg_sq, grad_flat, grad_div, ws, state, stats_out):
    _check(lib().imb_disc_adam(C.byref(d), C.byref(opt), _p(params, th.float32), _p(exp_avg, th.float32),
                               _p(exp_avg_sq, th.float32), _p(grad_flat), C.c_float(grad_div), _p(ws, th.float32),
                               _p(state, th.int64), _p(stats_out), _stream()), "imb_disc_adam")


def reward_forward(d, params, norm_state, batch, ld, n, out_mode, out):
    _check(lib().imb_reward_forward(C.byref(d), _p(params, th.float32), _p(norm_state, th.float32),
                                    _p(batch, th.float32), C.c_int64(ld), C.c_int64(n), C.c_int(out_mode),
                                    _p(out, th.float32), _stream()), "imb_reward_forward")


def pref_loss(rews, n_pairs, frag_len, prefs, noise_prob, discount, threshold, grad_scale, grad_rews, probs_out, stats_acc,
              stats_slot=0):
    """Boltzmann preference probabilities + cross entropy (+ d loss / d rews) of one minibatch of fragment pairs;
    stats_acc: float32 [4 * n_slots] accumulators, slot k = (sum of minibatch losses, sum of accuracies, n minibatches, -)."""
    _check(lib().imb_pref_loss(_p(rews, th.float32), C.c_int64(n_pairs), C.c_int32(frag_len), _p(prefs, th.float32),
                               C.c_float(noise_prob), C.c_float(discount), C.c_float(threshold), C.c_float(grad_scale),
                               _p(grad_rews), _p(probs_out), _p(stats_acc), C.c_int32(stats_slot), _stream()),
           "imb_pref_loss")


def pref_uncertainty_desc(rews, norms) -> PrefUncDesc:
    """rews: one float32 CUDA tensor [2C * L] per member; norms: per member None, (state [mean, var], int32 [count],
    eps) of its output RunningNorm or (state [mean, var, inv_learning_rate], int32 [count, num_batches], eps, decay) of
    its output EMANorm."""
    if not 2 <= len(rews) <= PU_MAX_MEMBERS or len(norms) != len(rews):
        raise ImbError(f"imb_pref_uncertainty takes 2 to {PU_MAX_MEMBERS} members, got {len(rews)}")
    d = PrefUncDesc()
    d.n_members = len(rews)
    for m, (r, nm) in enumerate(zip(rews, norms)):
        d.rews[m] = _p(r, th.float32).value
        if nm is not None:
            d.norm_state[m], d.norm_count[m] = _p(nm[0], th.float32).value, _p(nm[1], th.int32).value
            d.norm_eps[m] = nm[2]
            if len(nm) > 3:
                d.norm_kind[m], d.norm_decay[m] = 1, nm[3]
    return d


def pref_uncertainty_ws_floats(n_members: int, n_pairs: int) -> int:
    return int(lib().imb_pref_uncertainty_ws_floats(C.c_int32(n_members), C.c_int64(n_pairs)))


def pref_uncertainty(d: PrefUncDesc, n_pairs, frag_len, mode, noise_prob, discount, threshold, ws, scores,
                     member_out=None):
    """Active-selection scores of n_pairs candidate pairs (mode: 0 logit, 1 probability, 2 label; PU_MODES)."""
    norm = any(d.norm_state[m] for m in range(d.n_members))
    _check(lib().imb_pref_uncertainty(C.byref(d), C.c_int64(n_pairs), C.c_int32(frag_len), C.c_int32(mode),
                                      C.c_float(noise_prob), C.c_float(discount), C.c_float(threshold),
                                      _p(ws, th.float32), _p(scores, th.float32), _p(member_out, th.float32),
                                      _stream()), "imb_pref_uncertainty", (1 + int(norm)) if n_pairs > 0 else 0)


def reward_norm_scan(rews, n_envs, n_steps, step_stride, env_stride, norm_state2, norm_count, eps, update_stats,
                     ema_decay=None):
    """NormalizedRewardNet output normalisation over n_steps env steps.  ema_decay None: RunningNorm, norm_state2
    [mean, var], norm_count [count]; otherwise EMANorm with that decay, norm_state2 [mean, var, inv_learning_rate],
    norm_count [count, num_batches]."""
    if ema_decay is None:
        _check(lib().imb_reward_norm_scan(_p(rews, th.float32), C.c_int64(n_envs), C.c_int64(n_steps),
                                          C.c_int64(step_stride), C.c_int64(env_stride), _p(norm_state2, th.float32),
                                          _p(norm_count, th.int32), C.c_float(eps), C.c_int(int(update_stats)),
                                          _stream()), "imb_reward_norm_scan")
    else:
        _check(lib().imb_reward_ema_scan(_p(rews, th.float32), C.c_int64(n_envs), C.c_int64(n_steps),
                                         C.c_int64(step_stride), C.c_int64(env_stride), _p(norm_state2, th.float32),
                                         _p(norm_count, th.int32), C.c_float(ema_decay), C.c_float(eps),
                                         C.c_int(int(update_stats)), _stream()), "imb_reward_ema_scan")


def table_store(table, capacity, d_obs, d_act, obs, acts_f, acts_i, next_obs, dones, n, use_ring, state):
    _check(lib().imb_table_store(_p(table, th.float32), C.c_int64(capacity), C.c_int32(d_obs), C.c_int32(d_act),
                                 _p(obs, th.float32), _p(acts_f), _p(acts_i), _p(next_obs, th.float32),
                                 _p(dones, th.uint8), C.c_int64(n), C.c_int(int(use_ring)), _p(state), _stream()),
           "imb_table_store")


def ring_advance(state, capacity, n_stored):
    _check(lib().imb_ring_advance(_p(state, th.int64), C.c_int64(capacity), C.c_int64(n_stored), _stream()),
           "imb_ring_advance")


def sample_indices(kind, idx_out, n, size, seed, state):
    _check(lib().imb_sample_indices(C.c_int(kind), _p(idx_out, th.int64), C.c_int64(n), C.c_int64(size),
                                    C.c_uint64(seed), _p(state, th.int64), _stream()), "imb_sample_indices")


def disc_sample_gather(e_table, e_n, ring, ring_cap, tw, mb, start, seed, e_state, g_state, batch, ld):
    _check(lib().imb_disc_sample_gather(_p(e_table, th.float32), C.c_int64(e_n), _p(ring, th.float32),
                                        C.c_int64(ring_cap), C.c_int32(tw), C.c_int64(mb), C.c_int64(start),
                                        C.c_uint64(seed), _p(e_state, th.int64), _p(g_state, th.int64),
                                        _p(batch, th.float32), C.c_int64(ld), _stream()), "imb_disc_sample_gather")


def sample_advance2(n, e_n, e_state, g_state):
    _check(lib().imb_sample_advance2(C.c_int64(n), C.c_int64(e_n), _p(e_state, th.int64), _p(g_state, th.int64),
                                     _stream()), "imb_sample_advance2")


def disc_reduce_adam(d, opt, params, exp_avg, exp_avg_sq, grad_div, ws, state, stats_out):
    _check(lib().imb_disc_reduce_adam(C.byref(d), C.byref(opt), _p(params, th.float32), _p(exp_avg, th.float32),
                                      _p(exp_avg_sq, th.float32), C.c_float(grad_div), _p(ws, th.float32),
                                      _p(state, th.int64), _p(stats_out, th.float32), _stream()),
           "imb_disc_reduce_adam")


def gather_rows(table, capacity, tw, idx, n, batch, ld, col0):
    _check(lib().imb_gather_rows(_p(table, th.float32), C.c_int64(capacity), C.c_int32(tw), _p(idx), C.c_int64(n),
                                 _p(batch, th.float32), C.c_int64(ld), C.c_int64(col0), _stream()),
           "imb_gather_rows")


def rollout_row_width(pol: PolicyDesc) -> int:
    return int(lib().imb_rollout_row_width(C.byref(pol)))


def rollout(env, env_params, env_obs, pol, pol_params, pol_norm, disc, disc_params, disc_norm, reward_mode, hp,
            n_envs, n_steps, rollout_tbl, ring, ring_capacity, flat_out, aux, noise, state, flags=0):
    _check(lib().imb_rollout(C.byref(env), _p(env_params, th.float32), _p(env_obs, th.float32), C.byref(pol),
                             _p(pol_params, th.float32), _p(pol_norm), C.byref(disc) if disc is not None else None,
                             _p(disc_params), _p(disc_norm), C.c_int(reward_mode), C.byref(hp), C.c_int64(n_envs),
                             C.c_int64(n_steps), _p(rollout_tbl, th.float32), _p(ring), C.c_int64(ring_capacity),
                             _p(flat_out), _p(aux, th.float32), _p(noise), C.c_int(flags), _p(state, th.int64),
                             _stream()),
           "imb_rollout")


def rollout_members(params, norm_states, raw) -> RolloutMembers:
    """Member table of an ensemble rollout: per member its flat parameter vector and input-norm state (None when the
    architecture has no input RunningNorm); raw: float32 [M * T * E] for the members' outputs."""
    if not 2 <= len(params) <= PU_MAX_MEMBERS or len(norm_states) != len(params):
        raise ImbError(f"imb_rollout_ensemble takes 2 to {PU_MAX_MEMBERS} members, got {len(params)}")
    d = RolloutMembers()
    d.n_members = len(params)
    for m, (pm, nm) in enumerate(zip(params, norm_states)):
        d.params[m] = _p(pm, th.float32).value
        d.norm_state[m] = _p(nm, th.float32).value if nm is not None else None
    d.raw = _p(raw, th.float32).value
    return d


def rollout_ensemble(env, env_params, env_obs, pol, pol_params, pol_norm, disc, members: RolloutMembers, hp, n_envs,
                     n_steps, rollout_tbl, ring, ring_capacity, flat_out, aux, noise, state, flags=0):
    """`rollout` with every member's raw reward written to members.raw ([M][T][E]) instead of the reward column."""
    _check(lib().imb_rollout_ensemble(C.byref(env), _p(env_params, th.float32), _p(env_obs, th.float32), C.byref(pol),
                                      _p(pol_params, th.float32), _p(pol_norm), C.byref(disc), C.byref(members),
                                      C.byref(hp), C.c_int64(n_envs), C.c_int64(n_steps), _p(rollout_tbl, th.float32),
                                      _p(ring), C.c_int64(ring_capacity), _p(flat_out), _p(aux, th.float32), _p(noise),
                                      C.c_int(flags), _p(state, th.int64), _stream()),
           "imb_rollout_ensemble")


def ensemble_relabel_ws_floats(n_members: int, n_steps: int) -> int:
    return int(lib().imb_ensemble_relabel_ws_floats(C.c_int32(n_members), C.c_int64(n_steps)))


def ensemble_relabel(d: PrefUncDesc, alpha, rollout_tbl, rw, col_rew, n_envs, n_steps, ws):
    """Per-step output normalisation of the members (d.rews[m] = member m's raw [T][E]) and mean + alpha * std into the
    rollout table's reward column."""
    norm = any(d.norm_state[m] for m in range(d.n_members))
    _check(lib().imb_ensemble_relabel(C.byref(d), C.c_float(alpha), _p(rollout_tbl, th.float32), C.c_int32(rw),
                                      C.c_int32(col_rew), C.c_int64(n_envs), C.c_int64(n_steps), _p(ws, th.float32),
                                      _stream()), "imb_ensemble_relabel", 1 + int(norm))


def gae(rollout_tbl, rw, col_value, n_envs, n_steps, aux, gamma, gae_lambda, state, horizon):
    _check(lib().imb_gae(_p(rollout_tbl, th.float32), C.c_int32(rw), C.c_int32(col_value), C.c_int64(n_envs),
                         C.c_int64(n_steps), _p(aux, th.float32), C.c_float(gamma), C.c_float(gae_lambda),
                         _p(state, th.int64), C.c_int32(horizon), _stream()), "imb_gae")


def rollout_advance(state, n_envs, n_steps, horizon, ring_capacity):
    _check(lib().imb_rollout_advance(_p(state, th.int64), C.c_int64(n_envs), C.c_int64(n_steps), C.c_int32(horizon),
                                     C.c_int64(ring_capacity), _stream()), "imb_rollout_advance")


def env_reset(env_obs, n_envs, env, state):
    _check(lib().imb_env_reset(_p(env_obs, th.float32), C.c_int64(n_envs), C.byref(env), _p(state, th.int64),
                               _stream()), "imb_env_reset")


def ppo_update(pol, params, norm, norm_count, exp_avg, exp_avg_sq, rollout_tbl, n_rows, hp, perm, seed, loss_log,
               state):
    _check(lib().imb_ppo_update(C.byref(pol), _p(params, th.float32), _p(norm), _p(norm_count),
                                _p(exp_avg, th.float32), _p(exp_avg_sq, th.float32), _p(rollout_tbl, th.float32),
                                C.c_int64(n_rows), C.byref(hp), _p(perm), C.c_uint64(seed), _p(loss_log),
                                _p(state, th.int64), _stream()), "imb_ppo_update")


def ppo_plan(pol: PolicyDesc, batch_size: int) -> int:
    """PPO_PLAN_* code of the kernel `ppo_update` runs for `pol` at minibatch size batch_size (host only, no GPU
    needed); ImbError naming the shared-memory need and limit when no PPO kernel can run the shape."""
    rc = int(lib().imb_ppo_plan(C.byref(pol), C.c_int32(batch_size)))
    if rc < 0:
        raise ImbError(f"imb_ppo_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def ppo_update_variant(pol: PolicyDesc) -> int:
    """Instantiation of k_ppo_update that `ppo_update` runs for `pol` when `ppo_plan` gives PPO_PLAN_UPDATE (host only):
    0 = the runtime-shape one, 1-3 = the shape-specialised ones (include/imb.h); IMB_PPO_FORCE_RUNTIME_SHAPE=1 forces 0."""
    return int(lib().imb_ppo_update_variant(C.byref(pol)))


def policy_logp(pol, params, norm, batch, ld, n, row_logp):
    _check(lib().imb_policy_logp(C.byref(pol), _p(params, th.float32), _p(norm), _p(batch, th.float32),
                                 C.c_int64(ld), C.c_int64(n), C.c_int32(row_logp), _stream()), "imb_policy_logp")
