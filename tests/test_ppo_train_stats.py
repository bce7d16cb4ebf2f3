"""PPO.train's statistics, target_kl and clip_range_vf on the device (imb_ppo_update_ex, DevicePPO, the trainers).

SB3 2.2.1 PPO.train as oracle/ppo_port.py restates it (SB3 is not installed: unpinned, like the rest of the PPO port).
The float64 machinery and the cases (rows whose ratios keep MARGIN from the clip band) come from test_ppo_float64.
"""
import inspect
import math
import re
import types

import numpy as np
import pytest
import torch as th

from imitation_b200 import _lib
from tests import test_ppo_float64 as F

gpu = pytest.mark.gpu
ROOT = __file__.rsplit("/tests/", 1)[0]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_stat_layout_in_header():
    src = open(f"{ROOT}/include/imb.h").read()
    defs = {k: int(v) for k, v in re.findall(r"^#define[ \t]+IMB_PPO_STAT_(\w+)[ \t]+(\d+)", src, re.M)}
    n = defs.pop("FLOATS")
    assert n == _lib.PPO_STAT_FLOATS == 16
    assert sorted(defs.values()) == list(range(len(defs))) and len(defs) <= n
    for k, v in defs.items():
        assert getattr(_lib, "PPO_STAT_" + k) == v
    assert list(_lib.SIGNATURES).index("imb_ppo_update_ex") == list(_lib.SIGNATURES).index("imb_ppo_update") + 1


def test_device_ppo_takes_target_kl_and_clip_range_vf():
    from imitation_b200.algorithms import ppo

    params = inspect.signature(ppo.DevicePPO).parameters
    assert params["target_kl"].default is None and params["clip_range_vf"].default is None
    for bad in (0.0, -0.1):  # SB3 asserts clip_range_vf > 0; refused before anything touches the device
        with pytest.raises(ValueError, match="clip_range_vf"):
            ppo.DevicePPO("MlpPolicy", None, clip_range_vf=bad)
        with pytest.raises(ValueError, match="target_kl"):
            ppo.DevicePPO("MlpPolicy", None, target_kl=bad)


def _stand_in(discrete, clip_range_vf=None):
    from imitation_b200.algorithms import ppo

    s = th.arange(_lib.PPO_STAT_FLOATS, dtype=th.float32) / 8
    s[_lib.PPO_STAT_N_UPDATES] = 30
    g = types.SimpleNamespace(train_stats=s, policy=types.SimpleNamespace(discrete=discrete), clip_range=0.2,
                              clip_range_vf=clip_range_vf, learning_rate=3e-4, _logger=None)
    g.read_train_stats = lambda: ppo.DevicePPO.read_train_stats(g)
    g.record_train_stats = lambda logger=None: ppo.DevicePPO.record_train_stats(g, logger)
    return g


@pytest.mark.parametrize("discrete", [False, True])
def test_gen_stats_land_under_the_gen_prefix_of_the_round_dump(discrete):
    from imitation_b200.algorithms.adversarial import common
    from imitation_b200.util import logger

    lg = logger.configure()
    tr = types.SimpleNamespace(logger=lg, gen_algo=_stand_in(discrete, 0.1), _gen_stats_pending=True)
    common.AdversarialTrainer._record_gen_stats(tr)
    common.AdversarialTrainer._record_gen_stats(tr)  # (nothing pending: no second record)
    lg.dump(1)
    kv = lg.history[-1][1]
    keys = ["entropy_loss", "policy_gradient_loss", "value_loss", "approx_kl", "clip_fraction", "loss",
            "explained_variance", "n_updates", "clip_range", "clip_range_vf", "learning_rate"] + ([] if discrete else ["std"])
    assert {k for k in kv} == {f"{p}/gen/train/{k}" for k in keys for p in ("raw", "mean")}
    assert kv["raw/gen/train/approx_kl"] == _lib.PPO_STAT_APPROX_KL / 8
    assert kv["mean/gen/train/n_updates"] == 30 and kv["raw/gen/train/clip_range_vf"] == 0.1


# ---------------------------------------------------------------------------------------------------------------------
# GPU: launches
# ---------------------------------------------------------------------------------------------------------------------
def _launch(c, pd, P, norm, count, M, V, tbl, n_rows, perm, epochs, lr, step, *, ex, target_kl=None, cvf=None,
            act=_lib.ACT_TANH, mgn=1e30):
    n_steps = epochs * ((n_rows + c["mb"] - 1) // c["mb"])
    hp = _lib.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=F.CLIP, ent_coef=c["ent"], vf_coef=0.5,
                         max_grad_norm=mgn, lr=lr, adam_eps=1e-5, n_epochs=epochs, batch_size=c["mb"],
                         normalize_advantage=int(c["nadv"]))
    t = {k: th.from_numpy(np.ascontiguousarray(a)).cuda() for k, a in
         dict(params=P, exp_avg=M, exp_avg_sq=V, norm=norm).items()}
    t["count"] = th.tensor([count], dtype=th.int32, device="cuda")
    st = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
    st[_lib.ST_PPO_STEP], st[_lib.ST_PPO_EPOCH] = step, 3
    t["state"] = st
    t["log"] = th.full((n_steps, 4), float("nan"), device="cuda")
    pt = None if perm is None else th.from_numpy(np.ascontiguousarray(perm, dtype=np.int64)).cuda()
    rt = th.from_numpy(np.ascontiguousarray(tbl[:n_rows])).cuda()
    if ex:
        stats = th.full((_lib.PPO_STAT_FLOATS,), -7.0, device="cuda")
        _lib.ppo_update_ex(pd, t["params"], t["norm"], t["count"], t["exp_avg"], t["exp_avg_sq"], rt, n_rows, hp, pt,
                           c["seed"], t["log"], t["state"], target_kl=target_kl, clip_range_vf=cvf, stats=stats, act=act)
    else:
        _lib.ppo_update(pd, t["params"], t["norm"], t["count"], t["exp_avg"], t["exp_avg_sq"], rt, n_rows, hp, pt,
                        c["seed"], t["log"], t["state"], act=act)
    th.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in t.items()}
    if ex:
        out["stats"] = stats.cpu().numpy()
    return out


def _bits(a, b, what, keys=("params", "exp_avg", "exp_avg_sq", "norm", "count", "state", "log")):
    for k in keys:
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), f"{what}: {k} differs"


def _variant_env(monkeypatch, runtime):
    if runtime:
        monkeypatch.setenv("IMB_PPO_FORCE_RUNTIME_SHAPE", "1")
    else:
        monkeypatch.delenv("IMB_PPO_FORCE_RUNTIME_SHAPE", raising=False)


# 1. off path ---------------------------------------------------------------------------------------------------------
# (case, force the runtime-shape k_ppo_update, activation, expected plan, expected k_ppo_update instantiation)
OFF_CASES = [("bench_hc", False, _lib.ACT_TANH, 1, 1), ("bench_ant", False, _lib.ACT_TANH, 1, 2),
             ("bench_cartpole", False, _lib.ACT_TANH, 1, 3), ("bench_hc", True, _lib.ACT_TANH, 1, 0),
             ("u_w7_o4_d9_mb2", False, _lib.ACT_TANH, 1, 0), ("g1_w7_o33_a9_mb129", False, _lib.ACT_TANH, 2, None),
             ("g2_w40_o33_d9_mb64", False, _lib.ACT_TANH, 3, None), ("u_w20_o17_a6_mb16", False, _lib.ACT_RELU, 2, None),
             ("g2_w33_o17_a6_mb1", False, _lib.ACT_RELU, 3, None)]


@gpu
@pytest.mark.parametrize("case", OFF_CASES, ids=lambda x: f"{x[0]}-{'rt' if x[1] else 'spec'}-act{x[2]}")
def test_off_path_is_bit_exact(monkeypatch, case):
    """imb_ppo_update_ex with the options off and statistics requested computes imb_ppo_update's bits (lr != 0)."""
    name, runtime, act, plan, var = case
    _variant_env(monkeypatch, runtime)
    c = F._cfg(name)
    pd, P, norm, tbl, M, V, rng, ref, perms = F._prepare(c)
    assert _lib.ppo_plan(pd, c["mb"], act=act) == plan
    if var is not None:
        assert _lib.ppo_update_variant(pd) == var
    perm = None if c["perm"] == "device" else perms
    cnt = c["count0"] if c["norm"] else 0
    a = _launch(c, pd, P, norm, cnt, M, V, tbl, c["N"], perm, c["epochs"], 3e-4, 5, ex=False, act=act, mgn=0.5)
    b = _launch(c, pd, P, norm, cnt, M, V, tbl, c["N"], perm, c["epochs"], 3e-4, 5, ex=True, act=act, mgn=0.5)
    _bits(a, b, name)
    assert not np.array_equal(a["params"], P)
    s = b["stats"]
    assert s[_lib.PPO_STAT_STOPPED] == 0 and s[_lib.PPO_STAT_N_STEPS] == a["log"].shape[0]
    assert s[_lib.PPO_STAT_N_EPOCHS] == c["epochs"] and s[_lib.PPO_STAT_N_UPDATES] == 3 + c["epochs"]


# 2. statistics against float64 ---------------------------------------------------------------------------------------
STAT_CASES = ["u_w20_o17_a6_mb16", "u_w7_o4_d9_mb2", "bench_hc", "u_w32_o64_a6_mb16", "g1_w20_o4_d9_mb128",
              "g1_w7_o33_a9_mb129", "g2_w40_o33_d9_mb64"]


def _explained_variance(tbl, col):
    y = tbl[:, col + 4].astype(np.float64)
    e = (tbl[:, col + 4] - tbl[:, col + 1]).astype(np.float64)  # (ret - value rounded in fp32, like SB3's numpy)
    vy = y.var()
    return math.nan if vy == 0 else 1 - e.var() / vy


@gpu
@pytest.mark.parametrize("name", STAT_CASES)
def test_statistics_against_float64(name):
    c = F._cfg(name)
    pd, P, norm, tbl, M, V, rng, ref, perms = F._prepare(c)
    perm = None if c["perm"] == "device" else perms
    cnt = c["count0"] if c["norm"] else 0
    got = _launch(c, pd, P, norm, cnt, M, V, tbl, c["N"], perm, c["epochs"], 0.0, 0, ex=True)
    s, log = got["stats"], got["log"].astype(np.float64)
    st = F._state0(c, P, norm, M, V, 0)
    N, mb = c["N"], c["mb"]
    spe = (N + mb - 1) // mb
    clip, kl = [], []
    for e in range(c["epochs"]):
        for b in range(0, N, mb):
            rows = th.from_numpy(tbl[perms[e][b:b + mb]]).double()
            xn = ref.norm_update(st, rows[:, :ref.Do])
            act, lpo, adv, ret = ref.batch(rows)
            _, _, _, ratio, logp = ref.row_terms(st["P"], xn, act, lpo, adv, ret)
            lr_ = logp - lpo
            clip.append(float(((ratio - 1).abs() > ref.clip).double().mean()))
            kl.append(float((th.exp(lr_) - 1 - lr_).mean()))
    n = len(clip)
    assert s[_lib.PPO_STAT_N_STEPS] == n == log.shape[0] and s[_lib.PPO_STAT_N_EPOCHS] == c["epochs"]
    assert 0 < np.mean(clip) < 1, "the case does not clip"
    np.testing.assert_allclose(s[_lib.PPO_STAT_CLIP_FRACTION], np.mean(clip), rtol=2e-6, atol=0)
    last = kl[(n - 1) // spe * spe:]
    np.testing.assert_allclose(s[_lib.PPO_STAT_APPROX_KL], np.mean(last), rtol=1e-4, atol=1e-7)
    # the loss means and train/loss against the kernel's own loss log (fp32 summation error)
    for k, col in ((_lib.PPO_STAT_PG_LOSS, 0), (_lib.PPO_STAT_VALUE_LOSS, 1), (_lib.PPO_STAT_ENTROPY_LOSS, 2)):
        np.testing.assert_allclose(s[k], log[:, col].mean(), rtol=2e-5, atol=2e-6 * (1 + np.abs(log[:, col]).mean()))
    np.testing.assert_allclose(s[_lib.PPO_STAT_LOSS], log[-1, 3], rtol=2e-5, atol=2e-6 * (1 + abs(log[-1, 3])))
    np.testing.assert_allclose(s[_lib.PPO_STAT_EXPLAINED_VARIANCE], _explained_variance(tbl[:N], ref.col), rtol=1e-5,
                               atol=1e-6)
    if c["disc"]:
        assert math.isnan(s[_lib.PPO_STAT_STD])
    else:
        ls = P[pd.off_log_std:pd.off_log_std + c["Da"]].astype(np.float64)
        np.testing.assert_allclose(s[_lib.PPO_STAT_STD], np.exp(ls).mean(), rtol=1e-6)


@gpu
@pytest.mark.parametrize("name", ["bench_cartpole", "g1_w20_o4_d9_mb128"])
def test_explained_variance_is_nan_for_constant_returns(name):
    c = F._cfg(name)
    pd, P, norm, tbl, M, V, rng, ref, perms = F._prepare(c)
    tbl[:, ref.col + 4] = 1.25
    got = _launch(c, pd, P, norm, 0, M, V, tbl, c["N"], perms, 1, 0.0, 0, ex=True)
    assert math.isnan(got["stats"][_lib.PPO_STAT_EXPLAINED_VARIANCE])


# 3. clip_range_vf ----------------------------------------------------------------------------------------------------
class RefVf(F.Ref):
    """The float64 step with SB3's clipped value loss: mse(ret, old + clamp(value - old, -c, c))."""

    def __init__(self, c, cvf):
        super().__init__(c, c["ent"], nadv=c["nadv"])
        self.cvf = float(np.float32(cvf))

    def batch(self, rows):
        act, lpo, adv, ret = super().batch(rows)
        return act, lpo, adv, th.stack([ret, rows[:, self.col + 1]], -1)

    def row_terms(self, p, xn, act, lpo, adv, ret, padded=False):
        pg, _, el, ratio, logp = super().row_terms(p, xn, act, lpo, adv, ret[..., 0], padded)
        val = self.heads(p, xn, padded)[1]
        old = ret[..., 1]
        vpred = old + th.clamp(val - old, -self.cvf, self.cvf)
        return pg, (ret[..., 0] - vpred) ** 2, el, ratio, logp


@gpu
@pytest.mark.parametrize("name", ["bench_hc", "u_w7_o4_d9_mb2", "u_w32_o33_a17_mb64", "g1_w20_o4_d9_mb128",
                                  "g2_w64_o17_a8_mb64"])
def test_clip_range_vf_one_step_gradient(name):
    """test_ppo_float64's first measurement with the clipped value loss: old values put some rows' value predictions
    outside the band and none within the fp32 bound of an edge."""
    cvf = 0.25
    c = F._cfg(name)
    pd, P, norm, tbl, M, V, rng, ref, perms = F._prepare(c)
    idx = perms[0][:c["mb"]]
    sub = tbl[idx].copy()
    nb = len(idx)
    refv = RefVf(c, cvf)
    st = F._state0(c, P, norm, M, V, 0)
    rows = th.from_numpy(sub).double()
    xn = refv.norm_update(dict(st), rows[:, :refv.Do])
    val = refv.heads(st["P"], xn)[1].numpy()
    inside = rng.permutation(np.arange(nb) % 2 == 0)  # half of the rows (at least one) inside the band
    off = np.where(inside, rng.uniform(0.3, 0.8, nb), rng.uniform(1.3, 4.0, nb)) * cvf * rng.choice([-1, 1], nb)
    sub[:, refv.col + 1] = (val - off).astype(np.float32)  # value - old = off
    rows = th.from_numpy(sub).double()
    d = np.abs(val - sub[:, refv.col + 1].astype(np.float64))
    assert (d > cvf * 1.1).any() and (d < cvf * 0.9).any() and np.abs(d - cvf).min() > 1e-3 * cvf
    z = np.zeros_like(P)
    sub_perm = rng.permutation(nb)[None]
    perm = None if c["perm"] == "device" else sub_perm
    cnt = c["count0"] if c["norm"] else 0
    got = _launch(c, pd, P, norm, cnt, z, z, sub, nb, perm, 1, 0.0, 0, ex=True, cvf=cvf)
    plain = _launch(c, pd, P, norm, cnt, z, z, sub, nb, perm, 1, 0.0, 0, ex=True)
    assert not np.array_equal(got["exp_avg"], plain["exp_avg"]), "the value clip changed nothing"
    st = F._state0(c, P, norm, z, z, 0)
    log, tol_log, _, _ = refv.step(st, rows, 1e30, 0.0)
    F._check(got["exp_avg"], st["M"], st["tol_M"], f"{name}: exp_avg")
    F._check(got["exp_avg_sq"], st["V"], st["tol_V"], f"{name}: exp_avg_sq")
    F._check(got["log"][0], log, tol_log, f"{name}: loss log")


# 4. target_kl --------------------------------------------------------------------------------------------------------
# (d_obs, d_act, discrete, width, norm, minibatch, N, epochs, count0, ent, nadv, perm, force, plan): the specialised
# 17 x 6 Box with its feature RunningNorm (tail statistics), the runtime-shape kernel, and k_ppo_update_gen<1>
KL_CASES = {
    "kl_spec_hc": (17, 6, False, 32, True, 64, 4 * 64, 3, 10 ** 4, 0.0, True, "host", False, 1),
    "kl_rt_d9": (4, 9, True, 7, False, 16, 4 * 16 + 5, 3, 0, 0.01, True, "host", False, 1),
    "kl_gen1_hc": (17, 6, False, 32, True, 128, 4 * 128, 3, 10 ** 4, 0.0, True, "host", False, 2),
}


def _kl_cfg(name):
    Do, Da, disc, h, norm, mb, N, ep, cnt, ent, nadv, perm, force, code = KL_CASES[name]
    i = list(KL_CASES).index(name)
    return dict(name=name, Do=Do, Da=Da, disc=disc, h=h, norm=norm, mb=mb, N=N, epochs=ep, count0=cnt, ent=ent,
                nadv=nadv, perm=perm, force=force, code=code, idx=i, seed=5000 + 17 * i)


def _kl_setup(name, stop_epoch, k_first=2):
    c = _kl_cfg(name)
    pd, P, norm, tbl, M, V, rng = F._make_inputs(c)
    ref = F.Ref(c, c["ent"], nadv=c["nadv"])
    N, mb = c["N"], c["mb"]
    spe = (N + mb - 1) // mb
    perms = F._epoch_perms(c, rng)
    blocks = [perms[0][b:b + mb] for b in range(0, N, mb)]
    if stop_epoch == 0:  # every row of minibatch k_first is far from its old policy
        hot, k = set(blocks[k_first].tolist()), k_first
    else:  # one such row per full minibatch of epoch 0, all of them in the first minibatch of epoch 1
        hot, k = {int(b[0]) for b in blocks if len(b) == mb}, spe
        rest = np.array([i for i in perms[1] if i not in hot])
        perms[1] = np.concatenate([np.array(sorted(hot)), rest])
    # logp_old: ratio 4 on the hot rows, within 5 % of 1 elsewhere (float64 logp at the row's first use)
    st = F._state0(c, P, norm, M, V, 0)
    for b in blocks:
        rows = th.from_numpy(tbl[b]).double()
        xn = ref.norm_update(st, rows[:, :c["Do"]])
        act = ref.batch(rows)[0]
        logp = ref.logp_ent(st["P"], ref.heads(st["P"], xn)[0], act)[0].numpy()
        r = np.where([i in hot for i in b], 4.0, rng.uniform(0.95, 1.05, len(b)))
        tbl[b, ref.col] = (logp - np.log(r)).astype(np.float32)
    # float64 approx_kl of every step (lr ~ 0: the policy stays put) and the feature statistics after each
    st = F._state0(c, P, norm, M, V, 0)
    kls, norms = [], []
    for e in range(c["epochs"]):
        for b in range(0, N, mb):
            rows = th.from_numpy(tbl[perms[e][b:b + mb]]).double()
            xn = ref.norm_update(st, rows[:, :c["Do"]])
            act, lpo, _, _ = ref.batch(rows)
            lr_ = ref.logp_ent(st["P"], ref.heads(st["P"], xn)[0], act)[0] - lpo
            kls.append(float((th.exp(lr_) - 1 - lr_).mean()))
            norms.append((st["mean"], st["var"], st["count"]) if c["norm"] else None)
    lo, hi = max(kls[:k]), kls[k]
    assert hi > 3 * lo, (lo, hi)
    target = math.sqrt(lo * hi) / 1.5  # 1.5 target sits between with a factor >= sqrt(3) to spare on both sides
    return c, pd, P, norm, tbl, M, V, perms, kls, norms, k, spe, target


@gpu
@pytest.mark.parametrize("stop_epoch", [0, 1])
@pytest.mark.parametrize("name", list(KL_CASES))
def test_target_kl_stops_the_call(name, stop_epoch):
    """A stop at step k: parameters and moments equal a launch over the steps before k bit for bit; the state words,
    approx_kl and n_updates follow SB3.  The feature statistics of a stop in the first epoch equal a launch over k + 1
    minibatches bit for bit; for a stop in a later epoch no single shorter launch reaches the same state, so they are held
    to the float64 chain (1e-5) and the count exactly, which catches a step too many or too few."""
    c, pd, P, norm, tbl, M, V, perms, kls, norms, k, spe, target = _kl_setup(name, stop_epoch)
    N, mb, lr, step0 = c["N"], c["mb"], 1e-6, 7
    cnt = c["count0"] if c["norm"] else 0
    assert _lib.ppo_plan(pd, mb) == c["code"]
    got = _launch(c, pd, P, norm, cnt, M, V, tbl, N, perms, c["epochs"], lr, step0, ex=True, target_kl=target)
    s = got["stats"]
    ep_begun = k // spe + 1
    assert s[_lib.PPO_STAT_STOPPED] == 1 and s[_lib.PPO_STAT_N_STEPS] == k + 1 and s[_lib.PPO_STAT_N_EPOCHS] == ep_begun
    assert int(got["state"][_lib.ST_PPO_STEP]) == step0 + k
    assert int(got["state"][_lib.ST_PPO_EPOCH]) == 3 + ep_begun == s[_lib.PPO_STAT_N_UPDATES]
    np.testing.assert_allclose(s[_lib.PPO_STAT_APPROX_KL], np.mean(kls[(ep_begun - 1) * spe:k + 1]), rtol=1e-3)
    assert np.isfinite(got["log"][:k + 1]).all() and np.isnan(got["log"][k + 1:]).all()
    if stop_epoch == 0:
        # parameters and moments: those of a launch over the first k minibatches (block-shuffled epoch 0); the norm
        # state and count: those of a launch over k + 1 (the stopped step's update stays)
        a = _launch(c, pd, P, norm, cnt, M, V, tbl, k * mb, perms[:1, :k * mb], 1, lr, step0, ex=False)
        b = _launch(c, pd, P, norm, cnt, M, V, tbl, (k + 1) * mb, perms[:1, :(k + 1) * mb], 1, lr, step0, ex=False)
        _bits(a, got, name, ("params", "exp_avg", "exp_avg_sq"))
        _bits(b, got, name, ("norm", "count"))
    else:
        # stopped at the first step of epoch 1: parameters and moments of one full epoch
        a = _launch(c, pd, P, norm, cnt, M, V, tbl, N, perms[:1], 1, lr, step0, ex=False)
        _bits(a, got, name, ("params", "exp_avg", "exp_avg_sq"))
        if c["norm"]:
            mean, var, count = norms[k]
            Do = c["Do"]
            np.testing.assert_allclose(got["norm"][:Do], mean.numpy(), rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(got["norm"][Do:], var.numpy(), rtol=1e-5)
            assert int(got["count"][0]) == count
    # a target that never fires changes no bit
    never = _launch(c, pd, P, norm, cnt, M, V, tbl, N, perms, c["epochs"], lr, step0, ex=True, target_kl=1e30)
    full = _launch(c, pd, P, norm, cnt, M, V, tbl, N, perms, c["epochs"], lr, step0, ex=False)
    _bits(full, never, name)


# 5. end to end -------------------------------------------------------------------------------------------------------
TRAIN_KEYS = {"entropy_loss", "policy_gradient_loss", "value_loss", "approx_kl", "clip_fraction", "loss",
              "explained_variance", "n_updates", "clip_range", "learning_rate"}


@gpu
@pytest.mark.parametrize("algo,discrete", [("gail", False), ("airl", False), ("gail", True)])
def test_trainer_round_records_gen_stats_without_waiting_in_train_gen(algo, discrete, monkeypatch):
    from imitation_b200.algorithms import ppo
    from tests.test_gpu_api import _mk

    tr, _ = _mk(Do=4 if discrete else 17, Da=2 if discrete else 6, algo=algo, discrete=discrete, clip_range_vf=0.3)
    where = []
    inside = {"depth": 0}
    real = ppo.DevicePPO.read_train_stats

    def spy(self):
        where.append(inside["depth"])
        return real(self)

    monkeypatch.setattr(ppo.DevicePPO, "read_train_stats", spy)
    for meth in ("train_gen", "train_disc"):
        fn = getattr(tr, meth)

        def wrapped(*a, _fn=fn, **k):
            inside["depth"] += 1
            try:
                return _fn(*a, **k)
            finally:
                inside["depth"] -= 1
        monkeypatch.setattr(tr, meth, wrapped)
    tr.train(2 * tr.gen_train_timesteps)
    assert where == [0, 0], "the PPO statistics were read inside train_gen() / train_disc()"
    kv = tr.logger.history[-1][1]
    keys = TRAIN_KEYS | {"clip_range_vf"} | (set() if discrete else {"std"})
    for p in ("raw", "mean"):
        assert {k[len(p) + 11:] for k in kv if k.startswith(f"{p}/gen/train/")} == keys
    assert kv["raw/gen/train/n_updates"] == 4 and kv["raw/gen/train/clip_range_vf"] == 0.3
    assert all(np.isfinite(kv[f"raw/gen/train/{k}"]) for k in keys)


@gpu
def test_standalone_learn_records_after_train():
    from tests.test_gpu_api import _mk

    tr, _ = _mk()
    gen = tr.gen_algo
    gen.record_in_learn = True
    gen.set_logger(tr.logger)
    gen.learn(gen.n_steps * 16)
    assert tr.logger.name_to_value["train/n_updates"] == 2 and "train/std" in tr.logger.name_to_value


@gpu
def test_graph_replay_equals_eager_with_target_kl():
    """DevicePPO rounds replayed from CUDA graphs compute the eager rounds' bits with target_kl set (the statistics
    vector included); changing target_kl after capture re-captures."""
    from tests.test_gpu_api import _mk

    outs = []
    for graph in (False, True):
        tr, _ = _mk(target_kl=1e-4, seed=3)
        gen = tr.gen_algo
        gen.use_cuda_graph = graph
        gen.record_in_learn = True
        stats = []
        for r in range(4):
            if r == 3:
                gen.target_kl = 0.5
            gen.learn(gen.n_steps * 16)
            stats.append(gen.train_stats.cpu().numpy().copy())
        pp, pn, pc = gen.policy.flat_vectors()
        outs.append([t.cpu().numpy() for t in (pp, pn, pc, gen.exp_avg, gen.exp_avg_sq, gen._base_env.state)] + stats)
        if graph:
            assert gen._graph is not None and gen._graph_key[7] == 0.5  # (the key's target_kl entry)
    assert any(s[_lib.PPO_STAT_STOPPED] == 1 for s in outs[0][6:]), "target_kl never fired"
    for a, b in zip(*outs):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
