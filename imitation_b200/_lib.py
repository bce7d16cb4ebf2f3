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
ENV_SYNTH, ENV_CARTPOLE, ENV_PENDULUM = 0, 1, 2  # EnvDesc.kind: the env the rollout kernels step
ACT_TANH, ACT_RELU = 0, 1  # pol_act: the policy towers' activation (imb_rollout, imb_ppo_update, imb_policy_logp, ...)

# device-resident counter block (include/imb.h enum)
ST_RING_IDX, ST_RING_N, ST_EP_STEP, ST_EPISODE, ST_GLOBAL_STEP, ST_REPLAY_DRAW = 0, 1, 2, 3, 4, 5
ST_EXPERT_POS, ST_EXPERT_EPOCH, ST_PPO_EPOCH, ST_DISC_STEP, ST_PPO_STEP, ST_WORDS = 6, 7, 8, 9, 10, 16

PU_MAX_MEMBERS = 16  # members of an imb_pref_unc_desc / imb_rollout_members
SYNC_MAX_AVG, SYNC_MAX_NORM = 8, 4  # tensors of an imb_sync_desc


class ImbError(RuntimeError):
    pass


# the C types of include/imb.h: int / int32_t, int64_t, uint64_t, float, and every data pointer and stream
_i32, _i64, _u64, _f32, _ptr = C.c_int32, C.c_int64, C.c_uint64, C.c_float, C.c_void_p


class Mlp(C.Structure):
    _fields_ = [("din", _i32), ("n_hidden", _i32), ("h1", _i32), ("h2", _i32), ("n_out", _i32), ("has_norm", _i32),
                ("param_off", _i32), ("norm_off", _i32), ("count_idx", _i32), ("norm_eps", _f32)]


class DiscDesc(C.Structure):
    _fields_ = [("d_obs", _i32), ("d_act", _i32), ("use_state", _i32), ("use_action", _i32), ("use_next_state", _i32),
                ("use_done", _i32), ("base", Mlp), ("shaped", _i32), ("potential", Mlp), ("gamma", _f32),
                ("subtract_logp", _i32), ("n_params", _i32)]


class Adam(C.Structure):
    _fields_ = [("lr", _f32), ("beta1", _f32), ("beta2", _f32), ("eps", _f32),
                ("weight_decay", _f32)]  # > 0: torch.optim.AdamW's decoupled decay


class PolicyDesc(C.Structure):
    _fields_ = [("d_obs", _i32), ("d_act", _i32), ("discrete", _i32), ("hidden", _i32), ("has_norm", _i32),
                ("norm_eps", _f32), ("off_pi_w1", _i32), ("off_pi_b1", _i32), ("off_pi_w2", _i32), ("off_pi_b2", _i32),
                ("off_vf_w1", _i32), ("off_vf_b1", _i32), ("off_vf_w2", _i32), ("off_vf_b2", _i32), ("off_act_w", _i32),
                ("off_act_b", _i32), ("off_val_w", _i32), ("off_val_b", _i32), ("off_log_std", _i32),
                ("n_params", _i32)]


class EnvDesc(C.Structure):
    _fields_ = [("d_obs", _i32), ("d_act", _i32), ("discrete", _i32), ("horizon", _i32), ("seed", _u64),
                ("env_id_offset", _i32), ("kind", _i32)]


class PpoHparams(C.Structure):
    _fields_ = [("gamma", _f32), ("gae_lambda", _f32), ("clip_range", _f32), ("ent_coef", _f32), ("vf_coef", _f32),
                ("max_grad_norm", _f32), ("lr", _f32), ("adam_eps", _f32), ("n_epochs", _i32), ("batch_size", _i32),
                ("normalize_advantage", _i32)]


class PrefUncDesc(C.Structure):
    _fields_ = [("n_members", _i32), ("rews", _ptr * PU_MAX_MEMBERS), ("norm_state", _ptr * PU_MAX_MEMBERS),
                ("norm_count", _ptr * PU_MAX_MEMBERS), ("norm_eps", _f32 * PU_MAX_MEMBERS),
                ("norm_kind", _i32 * PU_MAX_MEMBERS), ("norm_decay", _f32 * PU_MAX_MEMBERS)]


class RolloutMembers(C.Structure):
    _fields_ = [("n_members", _i32), ("params", _ptr * PU_MAX_MEMBERS), ("norm_state", _ptr * PU_MAX_MEMBERS),
                ("raw", _ptr)]


class SyncDesc(C.Structure):
    _fields_ = [("n_avg", _i32), ("n_norm", _i32), ("avg", _ptr * SYNC_MAX_AVG), ("avg_n", _i64 * SYNC_MAX_AVG),
                ("mean", _ptr * SYNC_MAX_NORM), ("var", _ptr * SYNC_MAX_NORM), ("count", _ptr * SYNC_MAX_NORM),
                ("k", _i32 * SYNC_MAX_NORM)]


# imb_disc_plan codes: the kernel imb_disc_fwd_bwd runs
PLAN_TC, PLAN_FFMA128X2, PLAN_FFMA256, PLAN_FFMA128 = 1, 2, 3, 4
# imb_ppo_plan codes: the kernel imb_ppo_update runs
PPO_PLAN_UPDATE, PPO_PLAN_GEN1, PPO_PLAN_GEN2 = 1, 2, 3
# imb_ppo_update_ex: indices of the training statistics vector (PPO_STAT_FLOATS floats)
PPO_STAT_ENTROPY_LOSS, PPO_STAT_PG_LOSS, PPO_STAT_VALUE_LOSS, PPO_STAT_APPROX_KL = 0, 1, 2, 3
PPO_STAT_CLIP_FRACTION, PPO_STAT_LOSS, PPO_STAT_EXPLAINED_VARIANCE, PPO_STAT_STD = 4, 5, 6, 7
PPO_STAT_N_UPDATES, PPO_STAT_N_STEPS, PPO_STAT_N_EPOCHS, PPO_STAT_STOPPED = 8, 9, 10, 11
PPO_STAT_FLOATS = 16
# imb_pref_uncertainty modes
PU_MODES = {"logit": 0, "probability": 1, "label": 2}
# imb_param_regularize kinds
REG_LP, REG_WEIGHT_DECAY = 1, 2
# imb_density_score: demonstration tile rows, widest feature vector, kernels (sklearn's names) and segment modes
DENSITY_TILE, DENSITY_MAX_D = 64, 128
KDE_GAUSSIAN, KDE_TOPHAT, KDE_EPANECHNIKOV, KDE_EXPONENTIAL, KDE_LINEAR, KDE_COSINE = 0, 1, 2, 3, 4, 5
KDE_KERNELS = {"gaussian": KDE_GAUSSIAN, "tophat": KDE_TOPHAT, "epanechnikov": KDE_EPANECHNIKOV,
               "exponential": KDE_EXPONENTIAL, "linear": KDE_LINEAR, "cosine": KDE_COSINE}
DENSITY_SEG_NONE, DENSITY_SEG_STEPS, DENSITY_SEG_ROLLOUT = 0, 1, 2
# imb_mce_sweep: flags and the shape envelope
MCE_BACKWARD, MCE_FORWARD = 1, 2
MCE_MAX_STATES, MCE_MAX_ACTIONS, MCE_MAX_HORIZON = 4096, 32, 1000000

_disc, _adam, _pol, _env, _hp, _pu, _members, _sync = map(C.POINTER, (
    DiscDesc, Adam, PolicyDesc, EnvDesc, PpoHparams, PrefUncDesc, RolloutMembers, SyncDesc))

# every entry point include/imb.h declares, in its order: name -> (restype, argtypes, kernels launched per call; None:
# the wrapper counts them).  tests/test_cabi_loads.py holds this table to the header.
SIGNATURES = {
    "imb_version": (_i32, [], 0),
    "imb_last_error": (C.c_char_p, [], 0),
    "imb_disc_workspace_floats": (_i64, [_disc], 0),
    "imb_disc_norm_update": (_i32, [_disc, _ptr, _i64, _i64, _ptr, _ptr, _ptr, _ptr], None),
    "imb_norm_batch_stats": (_i32, [_disc, _ptr, _i64, _i64, _i32, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr], 1),
    "imb_norm_fold": (_i32, [_i32, _ptr, _ptr, _ptr, _i32, _ptr], 1),
    "imb_stats_publish": (_i32, [_ptr, _i32, _ptr, _ptr, _i32, _ptr], 1),
    "imb_disc_set_rows": (_i32, [_disc, _ptr, _i64, _i64, _ptr], 1),
    "imb_disc_fwd_bwd": (_i32, [_disc, _ptr, _ptr, _ptr, _i64, _i64, _i64, _f32, _ptr, _ptr, _i32, _ptr, _ptr], 1),
    "imb_disc_plan": (_i32, [_disc, _i64], 0),
    "imb_disc_reduce": (_i32, [_disc, _ptr, _ptr, _ptr], 1),
    "imb_disc_adam": (_i32, [_disc, _adam, _ptr, _ptr, _ptr, _ptr, _f32, _ptr, _ptr, _ptr, _ptr], 1),
    "imb_reward_forward": (_i32, [_disc, _ptr, _ptr, _ptr, _i64, _i64, _i32, _ptr, _ptr], 1),
    "imb_reward_norm_scan": (_i32, [_ptr, _i64, _i64, _i64, _i64, _ptr, _ptr, _f32, _i32, _ptr], 1),
    "imb_reward_ema_scan": (_i32, [_ptr, _i64, _i64, _i64, _i64, _ptr, _ptr, _f32, _f32, _i32, _ptr], 1),
    "imb_table_store": (_i32, [_ptr, _i64, _i32, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _i64, _i32, _ptr, _ptr], 1),
    "imb_ring_advance": (_i32, [_ptr, _i64, _i64, _ptr], 1),
    "imb_sample_indices": (_i32, [_i32, _ptr, _i64, _i64, _u64, _ptr, _ptr], 2),
    "imb_disc_sample_gather": (_i32, [_ptr, _i64, _ptr, _i64, _i32, _i64, _i64, _u64, _ptr, _ptr, _ptr, _i64, _ptr], 1),
    "imb_sample_advance2": (_i32, [_i64, _i64, _ptr, _ptr, _ptr], 1),
    "imb_gather_rows": (_i32, [_ptr, _i64, _i32, _ptr, _i64, _ptr, _i64, _i64, _ptr], 1),
    "imb_rollout": (_i32, [_env, _ptr, _ptr, _pol, _i32, _ptr, _ptr, _disc, _ptr, _ptr, _i32, _hp, _i64, _i64, _ptr,
                           _ptr, _i64, _ptr, _ptr, _ptr, _i32, _ptr, _ptr], 1),
    "imb_rollout_row_width": (_i32, [_pol], 0),
    "imb_rollout_plan": (_i32, [_pol, _disc, _i32, _i64, _i32], 0),
    "imb_gae": (_i32, [_ptr, _i32, _i32, _i64, _i64, _ptr, _f32, _f32, _ptr, _i32, _ptr], 1),
    "imb_rollout_advance": (_i32, [_ptr, _i64, _i64, _i32, _i64, _ptr], 1),
    "imb_env_reset": (_i32, [_ptr, _i64, _env, _ptr, _ptr], 1),
    "imb_ppo_update": (_i32, [_pol, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i64, _hp, _ptr, _u64, _ptr, _ptr, _ptr],
                       1),
    "imb_ppo_update_ex": (_i32, [_pol, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i64, _hp, _f32, _f32, _ptr, _u64, _ptr,
                                 _ptr, _ptr, _ptr], 1),
    "imb_ppo_plan": (_i32, [_pol, _i32, _i32], 0),
    "imb_ppo_update_variant": (_i32, [_pol], 0),
    "imb_bc_train": (_i32, [_pol, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _i64, _i64, _i32, _f32, _f32,
                            _f32, _f32, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr], 1),
    "imb_bc_plan": (_i32, [_pol, _i32, _i32], 0),
    "imb_dqn_ring_store": (_i32, [_ptr, _i32, _ptr, _i64, _i64, _i64, _i32, _ptr, _ptr, _ptr], 1),
    "imb_dqn_target": (_i32, [_pol, _i32, _ptr, _ptr, _i64, _ptr, _ptr, _i64, _ptr, _i64, _i64, _i64, _f32, _f32, _f32,
                              _ptr, _i64, _ptr, _ptr], None),
    "imb_dqn_step": (_i32, [_pol, _i32, _ptr, _ptr, _ptr, _ptr, _i32, _i64, _f32, _f32, _f32, _ptr, _i64, _ptr, _ptr],
                     None),
    "imb_dqn_plan": (_i32, [_pol, _i32, _i32], 0),
    "imb_sac_plan": (_i32, [_i32, _i32, _i32, _i32], 0),
    "imb_sac_ws_floats": (_i64, [_i32, _i32, _i32, _i32], 0),
    "imb_sac_collect": (_i32, [_env, _ptr, _ptr, _i32, _ptr, _i64, _i64, _ptr, _ptr, _ptr, _i64, _i32, _u64, _ptr, _ptr],
                        1),
    "imb_sac_step": (_i32, [_i32, _i32, _i32, _i32, _f32, _f32, _f32, _f32, _i32, _f32, _f32, _f32, _f32, _i32, _u64, _ptr,
                            _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i64, _ptr, _ptr, _i64, _ptr, _i64, _i64, _ptr,
                            _ptr, _ptr, _ptr], None),
    "imb_policy_logp": (_i32, [_pol, _i32, _ptr, _ptr, _ptr, _i64, _i64, _i32, _ptr], 1),
    "imb_disc_reduce_adam": (_i32, [_disc, _adam, _ptr, _ptr, _ptr, _f32, _ptr, _ptr, _ptr, _ptr], 1),
    "imb_pref_loss": (_i32, [_ptr, _i64, _i32, _ptr, _f32, _f32, _f32, _f32, _ptr, _ptr, _ptr, _i32, _ptr], 1),
    "imb_param_regularize": (_i32, [_disc, _i32, _i32, _f32, _ptr, _ptr, _ptr, _i32, _ptr], 1),
    "imb_pref_uncertainty_ws_floats": (_i64, [_i32, _i64], 0),
    "imb_pref_uncertainty": (_i32, [_pu, _i64, _i32, _i32, _f32, _f32, _f32, _ptr, _ptr, _ptr, _ptr], None),
    "imb_rollout_ensemble": (_i32, [_env, _ptr, _ptr, _pol, _i32, _ptr, _ptr, _disc, _members, _hp, _i64, _i64, _ptr,
                                    _ptr, _i64, _ptr, _ptr, _ptr, _i32, _ptr, _ptr], 1),
    "imb_ensemble_relabel_ws_floats": (_i64, [_i32, _i64], 0),
    "imb_ensemble_relabel": (_i32, [_pu, _f32, _ptr, _i32, _i32, _i64, _i64, _ptr, _ptr], None),
    "imb_rollout_explore": (_i32, [_env, _ptr, _ptr, _pol, _i32, _ptr, _ptr, _disc, _ptr, _ptr, _members, _i32, _hp,
                                   _i64, _i64, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _u64, _i64, _ptr, _ptr], 1),
    "imb_rollout_dagger": (_i32, [_env, _ptr, _ptr, _pol, _i32, _ptr, _ptr, _pol, _i32, _ptr, _ptr, _i64, _i64, _ptr, _ptr,
                                  _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr], 1),
    "imb_rollout_dagger_plan": (_i32, [_pol, _pol, _i64, _i32], 0),
    "imb_density_ws_floats": (_i64, [_i64], 0),
    "imb_density_score": (_i32, [_i32, _i32, _i32, _i32, _i32, _i32, _f32, _i32, _i64, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr,
                                 _ptr, _i32, _ptr, _i64, _i32, _ptr, _ptr, _i64, _i64, _i32, _ptr, _i64, _ptr, _ptr], None),
    "imb_mce_plan": (_i64, [_i64, _i32, _i32, _i32, _i32, _ptr], 0),
    "imb_mce_sweep": (_i32, [_i64, _i32, _i32, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr,
                             _ptr, _ptr, _i64, _ptr], 1),
    "imb_sync_buffer_doubles": (_i64, [_sync], 0),
    "imb_sync_snapshot": (_i32, [_sync, _ptr, _ptr], None),
    "imb_sync_pack": (_i32, [_sync, _ptr, _ptr], 1),
    "imb_sync_unpack": (_i32, [_sync, _ptr, _ptr, _i32, _ptr], 1),
    "imb_state_init": (_i32, [_ptr, _ptr], 0),
}
SYMBOLS = list(SIGNATURES)

_lib: Optional[C.CDLL] = None


def lib() -> C.CDLL:
    """Load libimb.so; raise loudly (no CPU fallback) if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a). imitation_b200 has no CPU fallback.")
        dll = C.CDLL(LIB_PATH)
        for name, (restype, argtypes, _) in SIGNATURES.items():
            fn = getattr(dll, name)  # AttributeError if the .so is stale
            fn.restype, fn.argtypes = restype, argtypes
        _lib = dll
    return _lib


# kernel launches issued through this binding (bench.py reports them as `gpu_launches`)
LAUNCHES = {"count": 0}


def _check(rc: int, what: str, n_kernels: Optional[int] = None):
    LAUNCHES["count"] += SIGNATURES[what][2] if n_kernels is None else n_kernels
    if rc != 0:
        raise ImbError(f"{what}: {lib().imb_last_error().decode()} (rc={rc})")


def _p(t: Optional[th.Tensor], dtype=None) -> Optional[int]:
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise ImbError("imitation_b200 kernels need CUDA tensors (no CPU path)")
    if not t.is_contiguous():
        raise ImbError("tensor must be contiguous")
    if dtype is not None and t.dtype != dtype:
        raise ImbError(f"expected dtype {dtype}, got {t.dtype}")
    return t.data_ptr()


def _stream() -> int:
    return th.cuda.current_stream().cuda_stream


def disc_workspace_floats(d: DiscDesc) -> int:
    return lib().imb_disc_workspace_floats(d)


def sync_desc(averaged, norms) -> SyncDesc:
    """averaged: fp32 CUDA tensors; norms: (mean[k], var[k], int32 count) tensor triples (views are fine as
    long as they are contiguous)."""
    if len(averaged) > SYNC_MAX_AVG or len(norms) > SYNC_MAX_NORM:
        raise ImbError("too many tensors for one imb_sync_desc")
    d = SyncDesc()
    d.n_avg, d.n_norm = len(averaged), len(norms)
    for i, t in enumerate(averaged):
        d.avg[i], d.avg_n[i] = _p(t, th.float32), t.numel()
    for i, (m, v, c) in enumerate(norms):
        d.mean[i], d.var[i], d.count[i] = _p(m, th.float32), _p(v, th.float32), _p(c, th.int32)
        d.k[i] = m.numel()
    return d


def sync_buffer_doubles(d: SyncDesc) -> int:
    return lib().imb_sync_buffer_doubles(d)


def sync_snapshot(d: SyncDesc, start):
    _check(lib().imb_sync_snapshot(d, _p(start, th.float64), _stream()), "imb_sync_snapshot", 1 if d.n_norm else 0)


def sync_pack(d: SyncDesc, buf):
    _check(lib().imb_sync_pack(d, _p(buf, th.float64), _stream()), "imb_sync_pack")


def sync_unpack(d: SyncDesc, buf, start, world: int):
    _check(lib().imb_sync_unpack(d, _p(buf, th.float64), _p(start, th.float64), world, _stream()), "imb_sync_unpack")


def state_init(state):
    _check(lib().imb_state_init(_p(state, th.int64), _stream()), "imb_state_init")


def disc_norm_update(d, batch, ld, n, norm_state, norm_count, ws):
    _check(lib().imb_disc_norm_update(d, _p(batch, th.float32), ld, n, _p(norm_state, th.float32),
                                      _p(norm_count, th.int32), _p(ws, th.float32), _stream()), "imb_disc_norm_update",
           1 if (d.shaped and d.potential.has_norm) else int(d.base.has_norm))  # shaped: one multi-job launch


def norm_batch_stats(d, batch, ld, n, row0, din, norm_state, norm_count, defer, defer_cap, ws):
    """RunningNorm update of a foreign normaliser (the policy's feature extractor) from batch rows [row0, row0 + din);
    `defer` = slot list for a later in-order `norm_fold` (None: fold immediately)."""
    _check(lib().imb_norm_batch_stats(d, _p(batch, th.float32), ld, n, row0, din, _p(norm_state, th.float32),
                                      _p(norm_count, th.int32), _p(defer), defer_cap, _p(ws, th.float32), _stream()),
           "imb_norm_batch_stats")


def norm_fold(din, defer, norm_state, norm_count, n_slots=0):
    _check(lib().imb_norm_fold(din, _p(defer, th.float32), _p(norm_state, th.float32), _p(norm_count, th.int32),
                               n_slots, _stream()), "imb_norm_fold")


def stats_publish(stats_dev, n, host_pinned, state, state_idx):
    """host_pinned: a pinned (page-locked, hence device-mapped under unified addressing) float32 CPU tensor of 16 elements."""
    if host_pinned.is_cuda or not host_pinned.is_pinned() or host_pinned.numel() < 16:
        raise ImbError("stats_publish needs a pinned CPU tensor of >= 16 floats")
    _check(lib().imb_stats_publish(_p(stats_dev, th.float32), n, host_pinned.data_ptr(), _p(state, th.int64), state_idx,
                                   _stream()), "imb_stats_publish")


def disc_set_rows(d, ws, n_rows_total, n_expert_total):
    _check(lib().imb_disc_set_rows(d, _p(ws, th.float32), n_rows_total, n_expert_total, _stream()), "imb_disc_set_rows")


def disc_fwd_bwd(d, params, norm_state, batch, ld, n, n_expert, loss_scale, grad_out, logits_out, flags, ws):
    _check(lib().imb_disc_fwd_bwd(d, _p(params, th.float32), _p(norm_state, th.float32), _p(batch, th.float32), ld, n,
                                  n_expert, loss_scale, _p(grad_out), _p(logits_out), flags, _p(ws, th.float32),
                                  _stream()), "imb_disc_fwd_bwd")


def disc_plan(d: DiscDesc, n: int) -> int:
    """PLAN_* code of the kernel `disc_fwd_bwd` runs for `d` over n rows (host only, no GPU needed); ImbError naming
    the shared-memory limit when the fused kernels cannot run the shape."""
    rc = lib().imb_disc_plan(d, n)
    if rc < 0:
        raise ImbError(f"imb_disc_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def disc_reduce(d, ws, grad_out_flat=None):
    _check(lib().imb_disc_reduce(d, _p(ws, th.float32), _p(grad_out_flat), _stream()), "imb_disc_reduce")


def disc_adam(d, opt: Adam, params, exp_avg, exp_avg_sq, grad_flat, grad_div, ws, state, stats_out):
    _check(lib().imb_disc_adam(d, opt, _p(params, th.float32), _p(exp_avg, th.float32), _p(exp_avg_sq, th.float32),
                               _p(grad_flat), grad_div, _p(ws, th.float32), _p(state, th.int64), _p(stats_out),
                               _stream()), "imb_disc_adam")


def reward_forward(d, params, norm_state, batch, ld, n, out_mode, out):
    _check(lib().imb_reward_forward(d, _p(params, th.float32), _p(norm_state, th.float32), _p(batch, th.float32), ld,
                                    n, out_mode, _p(out, th.float32), _stream()), "imb_reward_forward")


def pref_loss(rews, n_pairs, frag_len, prefs, noise_prob, discount, threshold, grad_scale, grad_rews, probs_out, stats_acc,
              stats_slot=0):
    """Boltzmann preference probabilities + cross entropy (+ d loss / d rews) of one minibatch of fragment pairs;
    stats_acc: float32 [4 * n_slots] accumulators, slot k = (sum of minibatch losses, sum of accuracies, n minibatches, -)."""
    _check(lib().imb_pref_loss(_p(rews, th.float32), n_pairs, frag_len, _p(prefs, th.float32), noise_prob, discount,
                               threshold, grad_scale, _p(grad_rews), _p(probs_out), _p(stats_acc), stats_slot,
                               _stream()), "imb_pref_loss")


def param_regularize(d, kind, p, coeff, params, ws, stats_acc=None, stats_slot=0):
    """kind REG_LP: the Lp penalty's gradient (coeff = lambda) into ws's gradient accumulator, its value into statistics
    slot stats_slot of stats_acc (optional); kind REG_WEIGHT_DECAY: params += coeff * params (coeff = -lambda * lr)."""
    _check(lib().imb_param_regularize(d, kind, p, coeff, _p(params, th.float32), _p(ws, th.float32),
                                      _p(stats_acc, th.float32), stats_slot, _stream()), "imb_param_regularize")


def pref_uncertainty_desc(rews, norms) -> PrefUncDesc:
    """rews: one float32 CUDA tensor [2C * L] per member; norms: per member None, (state [mean, var], int32 [count],
    eps) of its output RunningNorm or (state [mean, var, inv_learning_rate], int32 [count, num_batches], eps, decay) of
    its output EMANorm."""
    if not 2 <= len(rews) <= PU_MAX_MEMBERS or len(norms) != len(rews):
        raise ImbError(f"imb_pref_uncertainty takes 2 to {PU_MAX_MEMBERS} members, got {len(rews)}")
    d = PrefUncDesc()
    d.n_members = len(rews)
    for m, (r, nm) in enumerate(zip(rews, norms)):
        d.rews[m] = _p(r, th.float32)
        if nm is not None:
            d.norm_state[m], d.norm_count[m] = _p(nm[0], th.float32), _p(nm[1], th.int32)
            d.norm_eps[m] = nm[2]
            if len(nm) > 3:
                d.norm_kind[m], d.norm_decay[m] = 1, nm[3]
    return d


def pref_uncertainty_ws_floats(n_members: int, n_pairs: int) -> int:
    return lib().imb_pref_uncertainty_ws_floats(n_members, n_pairs)


def pref_uncertainty(d: PrefUncDesc, n_pairs, frag_len, mode, noise_prob, discount, threshold, ws, scores,
                     member_out=None):
    """Active-selection scores of n_pairs candidate pairs (mode: 0 logit, 1 probability, 2 label; PU_MODES)."""
    norm = any(d.norm_state[m] for m in range(d.n_members))
    _check(lib().imb_pref_uncertainty(d, n_pairs, frag_len, mode, noise_prob, discount, threshold, _p(ws, th.float32),
                                      _p(scores, th.float32), _p(member_out, th.float32), _stream()),
           "imb_pref_uncertainty", (1 + int(norm)) if n_pairs > 0 else 0)


def reward_norm_scan(rews, n_envs, n_steps, step_stride, env_stride, norm_state2, norm_count, eps, update_stats,
                     ema_decay=None):
    """NormalizedRewardNet output normalisation over n_steps env steps.  ema_decay None: RunningNorm, norm_state2
    [mean, var], norm_count [count]; otherwise EMANorm with that decay, norm_state2 [mean, var, inv_learning_rate],
    norm_count [count, num_batches]."""
    if ema_decay is None:
        _check(lib().imb_reward_norm_scan(_p(rews, th.float32), n_envs, n_steps, step_stride, env_stride,
                                          _p(norm_state2, th.float32), _p(norm_count, th.int32), eps, int(update_stats),
                                          _stream()), "imb_reward_norm_scan")
    else:
        _check(lib().imb_reward_ema_scan(_p(rews, th.float32), n_envs, n_steps, step_stride, env_stride,
                                         _p(norm_state2, th.float32), _p(norm_count, th.int32), ema_decay, eps,
                                         int(update_stats), _stream()), "imb_reward_ema_scan")


def table_store(table, capacity, d_obs, d_act, obs, acts_f, acts_i, next_obs, dones, n, use_ring, state):
    _check(lib().imb_table_store(_p(table, th.float32), capacity, d_obs, d_act, _p(obs, th.float32), _p(acts_f),
                                 _p(acts_i), _p(next_obs, th.float32), _p(dones, th.uint8), n, int(use_ring), _p(state),
                                 _stream()), "imb_table_store")


def ring_advance(state, capacity, n_stored):
    _check(lib().imb_ring_advance(_p(state, th.int64), capacity, n_stored, _stream()), "imb_ring_advance")


def sample_indices(kind, idx_out, n, size, seed, state):
    _check(lib().imb_sample_indices(kind, _p(idx_out, th.int64), n, size, seed, _p(state, th.int64), _stream()),
           "imb_sample_indices")


def disc_sample_gather(e_table, e_n, ring, ring_cap, tw, mb, start, seed, e_state, g_state, batch, ld):
    _check(lib().imb_disc_sample_gather(_p(e_table, th.float32), e_n, _p(ring, th.float32), ring_cap, tw, mb, start,
                                        seed, _p(e_state, th.int64), _p(g_state, th.int64), _p(batch, th.float32), ld,
                                        _stream()), "imb_disc_sample_gather")


def sample_advance2(n, e_n, e_state, g_state):
    _check(lib().imb_sample_advance2(n, e_n, _p(e_state, th.int64), _p(g_state, th.int64), _stream()),
           "imb_sample_advance2")


def disc_reduce_adam(d, opt, params, exp_avg, exp_avg_sq, grad_div, ws, state, stats_out):
    _check(lib().imb_disc_reduce_adam(d, opt, _p(params, th.float32), _p(exp_avg, th.float32),
                                      _p(exp_avg_sq, th.float32), grad_div, _p(ws, th.float32), _p(state, th.int64),
                                      _p(stats_out, th.float32), _stream()), "imb_disc_reduce_adam")


def gather_rows(table, capacity, tw, idx, n, batch, ld, col0):
    _check(lib().imb_gather_rows(_p(table, th.float32), capacity, tw, _p(idx), n, _p(batch, th.float32), ld, col0,
                                 _stream()), "imb_gather_rows")


def rollout_row_width(pol: PolicyDesc) -> int:
    return lib().imb_rollout_row_width(pol)


def rollout_plan(pol: PolicyDesc, disc: Optional[DiscDesc], n_members: int, n_envs: int, n_sms: int = 0) -> int:
    """Rows per CTA (8, 32, 64 or 128) `rollout` (n_members 1) or `rollout_ensemble` (2 to 16) runs for these shapes
    over n_envs envs on n_sms SMs (<= 0: the current device's); disc None: reward_mode 0.  Host only, no GPU needed;
    ImbError naming the shared-memory need and limit when not even the 8-row tile fits."""
    rc = lib().imb_rollout_plan(pol, disc, n_members, n_envs, n_sms)
    if rc < 0:
        raise ImbError(f"imb_rollout_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def rollout(env, env_params, env_obs, pol, pol_params, pol_norm, disc, disc_params, disc_norm, reward_mode, hp,
            n_envs, n_steps, rollout_tbl, ring, ring_capacity, flat_out, aux, noise, state, flags=0, act=ACT_TANH):
    """act: the policy towers' activation, ACT_TANH or ACT_RELU (the same for every policy entry point below)."""
    _check(lib().imb_rollout(env, _p(env_params, th.float32), _p(env_obs, th.float32), pol, act,
                             _p(pol_params, th.float32), _p(pol_norm), disc, _p(disc_params), _p(disc_norm), reward_mode, hp, n_envs, n_steps,
                             _p(rollout_tbl, th.float32), _p(ring), ring_capacity, _p(flat_out), _p(aux, th.float32),
                             _p(noise), flags, _p(state, th.int64), _stream()), "imb_rollout")


def rollout_members(params, norm_states, raw) -> RolloutMembers:
    """Member table of an ensemble rollout: per member its flat parameter vector and input-norm state (None when the
    architecture has no input RunningNorm); raw: float32 [M * T * E] for the members' outputs."""
    if not 2 <= len(params) <= PU_MAX_MEMBERS or len(norm_states) != len(params):
        raise ImbError(f"imb_rollout_ensemble takes 2 to {PU_MAX_MEMBERS} members, got {len(params)}")
    d = RolloutMembers()
    d.n_members = len(params)
    for m, (pm, nm) in enumerate(zip(params, norm_states)):
        d.params[m], d.norm_state[m] = _p(pm, th.float32), _p(nm, th.float32)
    d.raw = _p(raw, th.float32)
    return d


def rollout_ensemble(env, env_params, env_obs, pol, pol_params, pol_norm, disc, members: RolloutMembers, hp, n_envs,
                     n_steps, rollout_tbl, ring, ring_capacity, flat_out, aux, noise, state, flags=0, act=ACT_TANH):
    """`rollout` with every member's raw reward written to members.raw ([M][T][E]) instead of the reward column."""
    _check(lib().imb_rollout_ensemble(env, _p(env_params, th.float32), _p(env_obs, th.float32), pol, act,
                                      _p(pol_params, th.float32), _p(pol_norm), disc, members, hp, n_envs, n_steps,
                                      _p(rollout_tbl, th.float32), _p(ring), ring_capacity, _p(flat_out),
                                      _p(aux, th.float32), _p(noise), flags, _p(state, th.int64), _stream()),
           "imb_rollout_ensemble")


def ensemble_relabel_ws_floats(n_members: int, n_steps: int) -> int:
    return lib().imb_ensemble_relabel_ws_floats(n_members, n_steps)


def ensemble_relabel(d: PrefUncDesc, alpha, rollout_tbl, rw, col_rew, n_envs, n_steps, ws):
    """Per-step output normalisation of the members (d.rews[m] = member m's raw [T][E]) and mean + alpha * std into the
    rollout table's reward column."""
    norm = any(d.norm_state[m] for m in range(d.n_members))
    _check(lib().imb_ensemble_relabel(d, alpha, _p(rollout_tbl, th.float32), rw, col_rew, n_envs, n_steps,
                                      _p(ws, th.float32), _stream()), "imb_ensemble_relabel", 1 + int(norm))


def rollout_explore(env, env_params, env_obs, pol, pol_params, pol_norm, disc, disc_params, disc_norm, members, reward_mode,
                    hp, n_envs, n_steps, rollout_tbl, flat_out, aux, noise, explore_policy, explore_seed, explore_step0,
                    state, flags=0, act=ACT_TANH):
    """`rollout` (members None) or `rollout_ensemble` (members: a RolloutMembers table, reward_mode 2) without a ring,
    where step t is a random-policy step when explore_policy[t] (uint8 [n_steps]) is 1: actions drawn from Philox keyed
    by explore_seed at step explore_step0 + t, or read from noise."""
    _check(lib().imb_rollout_explore(env, _p(env_params, th.float32), _p(env_obs, th.float32), pol, act,
                                     _p(pol_params, th.float32), _p(pol_norm), disc, _p(disc_params), _p(disc_norm),
                                     members, reward_mode, hp, n_envs, n_steps, _p(rollout_tbl, th.float32),
                                     _p(flat_out), _p(aux, th.float32), _p(noise), flags, _p(explore_policy, th.uint8),
                                     explore_seed, explore_step0, _p(state, th.int64), _stream()), "imb_rollout_explore")


def rollout_dagger(env, env_params, env_obs, expert, expert_params, expert_norm, learner, learner_params, learner_norm,
                   n_envs, n_steps, rollout_tbl, flat_out, aux, noise, robot_noise, robot_mask, state, flags=0,
                   expert_act=ACT_TANH, learner_act=ACT_TANH):
    """The DAgger rollout (imb_rollout_dagger): the expert acts, except where robot_mask[t][e] (uint8 [n_steps][n_envs])
    is 1, where env e executes the learner's sampled action; rows obs | the expert's clipped action (or index).
    noise / robot_noise (None: Philox) pin the expert's / the learner's sampling, laid out as `rollout`'s noise."""
    _check(lib().imb_rollout_dagger(env, _p(env_params, th.float32), _p(env_obs, th.float32), expert, expert_act,
                                    _p(expert_params, th.float32), _p(expert_norm), learner, learner_act,
                                    _p(learner_params, th.float32), _p(learner_norm), n_envs, n_steps,
                                    _p(rollout_tbl, th.float32), _p(flat_out), _p(aux, th.float32), _p(noise),
                                    _p(robot_noise), flags, _p(robot_mask, th.uint8), _p(state, th.int64), _stream()),
           "imb_rollout_dagger")


def rollout_dagger_plan(expert: PolicyDesc, learner: PolicyDesc, n_envs: int, n_sms: int = 0) -> int:
    """Rows per CTA (8, 32, 64 or 128) `rollout_dagger` runs for these policies over n_envs envs on n_sms SMs (<= 0: the
    current device's).  Host only; ImbError when not even the 8-row tile fits."""
    rc = lib().imb_rollout_dagger_plan(expert, learner, n_envs, n_sms)
    if rc < 0:
        raise ImbError(f"imb_rollout_dagger_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def density_ws_floats(n_query: int) -> int:
    return lib().imb_density_ws_floats(n_query)


def density_score(model, src, src_ld, n_query, out, out_stride, ws, seg_mode=DENSITY_SEG_NONE, row_map=None, steps=None,
                  state=None, n_envs=0, n_steps=0, horizon=0):
    """Kernel density log-likelihood of n_query source rows (imb_density_score).  model: an object with the
    imb_density_score model arguments as attributes (algorithms/density.py's DeviceDensity); out[row * out_stride]."""
    m = model
    _check(lib().imb_density_score(m.d, m.col0, m.n0, m.col1, m.n1, m.kernel, m.bandwidth, m.n_seg, m.n_demo,
                                   _p(m.demo, th.float32), _p(m.demo_seg, th.int32), _p(m.seg_off, th.int64),
                                   _p(m.seg_const, th.float64), _p(m.mean, th.float32), _p(m.scale, th.float32),
                                   _p(src, th.float32), src_ld, _p(row_map, th.int64), n_query, seg_mode,
                                   _p(steps, th.int64), _p(state, th.int64), n_envs, n_steps, horizon,
                                   _p(out, th.float32), out_stride, _p(ws, th.float32),
                                   _stream()), "imb_density_score", 1 if n_query > 0 else 0)


def mce_plan(n_states: int, n_actions: int, horizon: int, flags: int, n_sms: int = 0):
    """(workspace doubles, CTA count) of `mce_sweep` for this shape (host only; n_sms <= 0: the current device's SMs and
    the kernel's occupancy, which is what `mce_sweep` launches).  NotImplementedError naming the limit when the shape is
    outside the kernel's envelope."""
    grid = C.c_int32(0)
    rc = lib().imb_mce_plan(n_states, n_actions, horizon, flags, n_sms, C.addressof(grid))
    if rc < 0:
        raise NotImplementedError(f"imb_mce_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc, grid.value


def mce_sweep(n_states, n_actions, horizon, flags, T, initial, reward, reward32, discounts, ws, V=None, Q=None, pi=None,
              D=None, Dcum=None, demo_om=None, weights=None, linf=None):
    """The MCE IRL time sweep (imb_mce_sweep): float64 CUDA tensors except reward32 / weights (float32); `discounts`
    float64 [2] = (planning discount, occupancy discount); ws: float64 [mce_plan(...)[0]]."""
    f64 = th.float64
    _check(lib().imb_mce_sweep(n_states, n_actions, horizon, flags, _p(T, f64), _p(initial, f64), _p(reward, f64),
                               _p(reward32, th.float32), _p(discounts, f64), _p(V, f64), _p(Q, f64), _p(pi, f64),
                               _p(D, f64), _p(Dcum, f64), _p(demo_om, f64), _p(weights, th.float32), _p(linf, f64),
                               _p(ws, f64), ws.numel(), _stream()), "imb_mce_sweep")


def gae(rollout_tbl, rw, col_value, n_envs, n_steps, aux, gamma, gae_lambda, state, horizon):
    _check(lib().imb_gae(_p(rollout_tbl, th.float32), rw, col_value, n_envs, n_steps, _p(aux, th.float32), gamma,
                         gae_lambda, _p(state, th.int64), horizon, _stream()), "imb_gae")


def rollout_advance(state, n_envs, n_steps, horizon, ring_capacity):
    _check(lib().imb_rollout_advance(_p(state, th.int64), n_envs, n_steps, horizon, ring_capacity, _stream()),
           "imb_rollout_advance")


def env_reset(env_obs, n_envs, env, state):
    _check(lib().imb_env_reset(_p(env_obs, th.float32), n_envs, env, _p(state, th.int64), _stream()), "imb_env_reset")


def ppo_update(pol, params, norm, norm_count, exp_avg, exp_avg_sq, rollout_tbl, n_rows, hp, perm, seed, loss_log,
               state, act=ACT_TANH):
    _check(lib().imb_ppo_update(pol, act, _p(params, th.float32), _p(norm), _p(norm_count), _p(exp_avg, th.float32),
                                _p(exp_avg_sq, th.float32), _p(rollout_tbl, th.float32), n_rows, hp, _p(perm), seed,
                                _p(loss_log), _p(state, th.int64), _stream()), "imb_ppo_update")


def ppo_update_ex(pol, params, norm, norm_count, exp_avg, exp_avg_sq, rollout_tbl, n_rows, hp, perm, seed, loss_log,
                  state, target_kl=None, clip_range_vf=None, stats=None, act=ACT_TANH):
    """`ppo_update` with SB3's target_kl / clip_range_vf (None: off) and the training statistics written to `stats`
    (float32 [PPO_STAT_FLOATS] CUDA tensor, indices PPO_STAT_*; None: not computed)."""
    if stats is not None and stats.numel() < PPO_STAT_FLOATS:
        raise ImbError(f"the PPO statistics vector needs {PPO_STAT_FLOATS} floats")
    _check(lib().imb_ppo_update_ex(pol, act, _p(params, th.float32), _p(norm), _p(norm_count), _p(exp_avg, th.float32),
                                   _p(exp_avg_sq, th.float32), _p(rollout_tbl, th.float32), n_rows, hp,
                                   0.0 if target_kl is None else float(target_kl),
                                   0.0 if clip_range_vf is None else float(clip_range_vf), _p(perm), seed,
                                   _p(loss_log), _p(stats, th.float32), _p(state, th.int64), _stream()),
           "imb_ppo_update_ex")


def ppo_plan(pol: PolicyDesc, batch_size: int, act: int = ACT_TANH) -> int:
    """PPO_PLAN_* code of the kernel `ppo_update` runs for `pol` with activation `act` at minibatch size batch_size
    (host only, no GPU needed); ImbError naming the shared-memory need and limit when no PPO kernel can run the shape."""
    rc = lib().imb_ppo_plan(pol, act, batch_size)
    if rc < 0:
        raise ImbError(f"imb_ppo_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def ppo_update_variant(pol: PolicyDesc) -> int:
    """Instantiation of k_ppo_update that `ppo_update` runs for `pol` when `ppo_plan` gives PPO_PLAN_UPDATE (host only):
    0 = the runtime-shape one, 1-3 = the shape-specialised ones (include/imb.h); IMB_PPO_FORCE_RUNTIME_SHAPE=1 forces 0."""
    return lib().imb_ppo_update_variant(pol)


def policy_logp(pol, params, norm, batch, ld, n, row_logp, act=ACT_TANH):
    _check(lib().imb_policy_logp(pol, act, _p(params, th.float32), _p(norm), _p(batch, th.float32), ld, n, row_logp,
                                 _stream()), "imb_policy_logp")


# imb_bc_train: columns of a metrics row
BC_METRICS = ("neglogp", "entropy", "ent_loss", "prob_true_act", "l2_norm", "l2_loss", "loss")
BC_METRIC_FLOATS = 8  # the seven BCTrainingMetrics and the batch number


def bc_train(pol, params, norm, norm_count, exp_avg, exp_avg_sq, table, n_rows, minibatch_size, batch_size, j0,
             n_minibatches, final_flush, l2_weight, ent_weight, lr, adam_eps, norm_update, perm, grad_carry, metrics,
             log_interval, state, act=ACT_TANH):
    """Minibatches [j0, j0 + n_minibatches) of one BC train() call in one launch (imb_bc_train): `table` the
    demonstrations in rollout-row format, `perm` int64 [epochs][n_rows] from epoch j0 // (n_rows // minibatch_size) on,
    `metrics` float32 [n_logged][BC_METRIC_FLOATS] or None."""
    _check(lib().imb_bc_train(pol, act, _p(params, th.float32), _p(norm), _p(norm_count), _p(exp_avg, th.float32),
                              _p(exp_avg_sq, th.float32), _p(table, th.float32), n_rows, minibatch_size, batch_size, j0,
                              n_minibatches, int(final_flush), l2_weight, ent_weight, lr, adam_eps, int(norm_update),
                              _p(perm, th.int64), _p(grad_carry, th.float32), _p(metrics, th.float32), log_interval,
                              _p(state, th.int64), _stream()), "imb_bc_train", 1 if n_minibatches > 0 or final_flush == 1 else 0)


def bc_plan(pol: PolicyDesc, minibatch_size: int, act: int = ACT_TANH) -> int:
    """PPO_PLAN_GEN1 / PPO_PLAN_GEN2: the kernel `bc_train` runs for `pol` at minibatch_size (host only, no GPU needed);
    ImbError naming the shared-memory need and limit when the shape does not fit."""
    rc = lib().imb_bc_plan(pol, act, minibatch_size)
    if rc < 0:
        raise ImbError(f"imb_bc_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


def dqn_ring_store(flat, tw, ring, positions, n_envs, n_steps, horizon, env_state, ring_state):
    """Store a rollout's flat rows into the feature-major learner ring at SB3's (position, env) columns, position read
    from and advanced in ring_state (imb_dqn_ring_store)."""
    _check(lib().imb_dqn_ring_store(_p(flat, th.float32), tw, _p(ring, th.float32), positions, n_envs, n_steps, horizon,
                                    _p(env_state, th.int64), _p(ring_state, th.int64), _stream()), "imb_dqn_ring_store")


def dqn_target(pol, target_params, ring, ring_ld, ring_idx, expert, expert_ld, expert_idx, n_learner, n_expert, n_steps,
               gamma, reward_learner, reward_expert, rows, step_base=0, state=None, act=ACT_RELU):
    """TD rows obs | action index | y of n_steps minibatches (imb_dqn_target): learner rows from columns ring_idx of the
    feature-major ring [tw][ring_ld], expert rows from columns expert_idx of the feature-major expert table, from TD
    step state[ST_PPO_STEP] - step_base of the index lists on (state None: from step 0)."""
    _check(lib().imb_dqn_target(pol, act, _p(target_params, th.float32), _p(ring, th.float32), ring_ld, _p(ring_idx, th.int64),
                                _p(expert, th.float32), expert_ld, _p(expert_idx, th.int64), n_learner, n_expert, n_steps,
                                gamma, reward_learner, reward_expert, _p(rows, th.float32), step_base,
                                _p(state, th.int64), _stream()), "imb_dqn_target",
           1 if n_steps * (n_learner + n_expert) > 0 else 0)


def dqn_step(pol, q_params, exp_avg, exp_avg_sq, rows, batch_size, n_steps, lr, adam_eps, max_grad_norm, loss_log, state,
             loss_base=0, act=ACT_RELU):
    """n_steps DQN TD steps on the rows dqn_target wrote, in one launch (imb_dqn_step); loss_log float32 [rows][4] or
    None, row k - 1 - loss_base for the step that brings state[ST_PPO_STEP] to k."""
    _check(lib().imb_dqn_step(pol, act, _p(q_params, th.float32), _p(exp_avg, th.float32), _p(exp_avg_sq, th.float32),
                              _p(rows, th.float32), batch_size, n_steps, lr, adam_eps, max_grad_norm,
                              _p(loss_log, th.float32), loss_base, _p(state, th.int64), _stream()), "imb_dqn_step",
           1 if n_steps > 0 else 0)


def dqn_plan(pol: PolicyDesc, batch_size: int, act: int = ACT_RELU) -> int:
    """PPO_PLAN_GEN1 / PPO_PLAN_GEN2: the kernel `dqn_step` runs for the Q-net `pol` at batch_size (host only);
    ImbError naming the limit when the shape does not fit."""
    rc = lib().imb_dqn_plan(pol, act, batch_size)
    if rc < 0:
        raise ImbError(f"imb_dqn_plan: {lib().imb_last_error().decode()} (rc={rc})")
    return rc


SAC_STEP_LAUNCHES = 4  # kernels per SAC gradient step (imb_sac_step)
SAC_DETERMINISTIC, SAC_PREDICT = 1, 2  # imb_sac_collect flags


def sac_plan(d_obs: int, d_act: int, hidden: int, batch_size: int) -> None:
    """Host only: ImbError naming the limit when the SAC kernels cannot run the shape (imb_sac_plan)."""
    rc = lib().imb_sac_plan(d_obs, d_act, hidden, batch_size)
    if rc < 0:
        raise ImbError(f"imb_sac_plan: {lib().imb_last_error().decode()} (rc={rc})")


def sac_ws_floats(d_obs: int, d_act: int, hidden: int, batch_size: int) -> int:
    return lib().imb_sac_ws_floats(d_obs, d_act, hidden, batch_size)


def sac_collect(env, env_params, env_obs, hidden, actor, n_envs, n_steps, flat_out, aux, random_steps, g0, flags,
                seed, state):
    """n_steps steps of n_envs Box envs with the SAC actor in one launch (imb_sac_collect): flat rows obs | buffer action |
    next obs | done into flat_out, env rewards into aux; step t random when random_steps[global step + t - g0]; flags
    SAC_DETERMINISTIC | SAC_PREDICT (evaluation: the env gets predict()'s action, which the rows record)."""
    _check(lib().imb_sac_collect(env, _p(env_params), _p(env_obs, th.float32), hidden, _p(actor, th.float32), n_envs,
                                 n_steps, _p(flat_out, th.float32), _p(aux, th.float32), _p(random_steps, th.uint8), g0,
                                 int(flags), seed & 0xFFFFFFFFFFFFFFFF, _p(state, th.int64), _stream()),
           "imb_sac_collect")


def sac_step(hp: dict, actor, actor_m, actor_v, critic, critic_m, critic_v, critic_target, ent, ring, ring_ld, ring_idx,
             expert, expert_ld, expert_idx, n_steps, step_base, loss_log, ws, state):
    """n_steps SAC gradient steps (imb_sac_step).  hp: d_obs, d_act, hidden, batch_size, gamma, tau, lr, adam_eps,
    auto_ent, ent_coef, target_entropy, reward_learner, reward_expert, target_update_interval, seed."""
    _check(lib().imb_sac_step(hp["d_obs"], hp["d_act"], hp["hidden"], hp["batch_size"], hp["gamma"], hp["tau"], hp["lr"],
                              hp["adam_eps"], int(hp["auto_ent"]), hp["ent_coef"], hp["target_entropy"],
                              hp["reward_learner"], hp["reward_expert"], hp["target_update_interval"],
                              hp["seed"] & 0xFFFFFFFFFFFFFFFF, _p(actor, th.float32), _p(actor_m, th.float32),
                              _p(actor_v, th.float32), _p(critic, th.float32), _p(critic_m, th.float32),
                              _p(critic_v, th.float32), _p(critic_target, th.float32), _p(ent, th.float32),
                              _p(ring, th.float32), ring_ld, _p(ring_idx, th.int64), _p(expert, th.float32), expert_ld,
                              _p(expert_idx, th.int64), n_steps, step_base, _p(loss_log, th.float32),
                              _p(ws, th.float32), _p(state, th.int64), _stream()), "imb_sac_step",
           SAC_STEP_LAUNCHES * max(int(n_steps), 0))
