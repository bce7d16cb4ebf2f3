"""The small kernels that run every round, at every shape they accept: the preference loss, the output-norm scans, the
RunningNorm batch statistics and fold, the replica merge and the replay data path.

Every comparison is either bit equality against a NumPy twin or a bound |got - want| <= C * eps * scale with
eps = 2^-24, `want` computed in float64 from the exact float32 inputs and `scale` taken from the float64 magnitudes of
the summands.  The C of each bound is the length of the longest chain of float32 roundings the kernel applies to that
quantity, as written beside it:

  preference loss (k_pref_loss, warp per pair)
    s      C_s = ceil(L / 32) + 16 of sum_t |g^t (r2 - r1)|: a lane's ceil(L / 32) adds, 5 shuffle levels, the
           difference, the fma and CUDA's powf (<= 8 ulp).  Pairs with L = 1 have s = r2 - r1 exactly.
    p      |dp/ds| err_s + 8 eps p: expf (2 ulp), 1 + e^d, the IEEE division, the (1 - noise) product and the add.
    loss   the float64 loss over the float32 probabilities inside p's bound (rounded outwards), + 8 eps |loss|.  Near
           p = 1 the BCE on a float32 probability is ill conditioned; the bound says so instead of hiding it.
    grad   the float64 d loss / d s over the same probabilities times (1 - noise) m (1 - m) over s +- err_s, + 8 eps:
           the division, 1 / P, grad_scale and the m (m e^d) product.  Element t of a fragment's gradient is the pair's
           gradient times powf(g, t): 10 eps of it plus 2^-125 of the pair's gradient, for the t where g^t is below
           float32's normal range and powf may return 0, plus the smallest subnormal 2^-149 for products that land
           below that range (bit-equal at g = 1); fragment 1's is exactly minus fragment 2's.
    stats  the per-pair bounds / P + (ceil(P / (8 CTAs)) + 8 + CTAs + 4) eps of sum |loss| / P: a warp's pairs, the
           CTA's 8 warps and one atomic per CTA.
  output-norm scans (k_reward_norm_scan, one CTA)
    per step C = ceil(E / threads) + 48 of sum |x| (the batch moments: a thread's adds, 5 shuffle levels, up to 32
    warps, the divisions) and of the fold's summands; the bounds add up over the steps (the fold contracts errors, so
    the sum is an upper bound).  Outputs: 4 eps of (|x| + |mean|) / std and the propagated mean / variance bounds.
  RunningNorm batch statistics (k_norm_stats + k_norm_fold)
    mean   C = 2 (ceil(chunk / 32) + ceil(chunks / 32) + 12) of |mean| + std: a lane's adds, the shuffle tree, the
           lane-serial Chan merge and its butterfly.
    var    the same C of var, plus the mean's bound through (x - mean)^2: 4 std tol_mean + tol_mean^2.
    fold   8 eps of the fold's summands per slot, plus the batch bounds weighted by b_n / tot.
  replica merge (k_sync_pack / k_sync_unpack)
    averaged tensors: bit-equal to float32(sum_r x_r * (1 / world)) summed in rank order in float64.
    mean   8 eps of max |mean| over the ranks and the start (each rank's state is float32).
    var    8 eps of max (var + mean^2): var = S2 / n - mean^2 cancels, so large-offset features keep only this much.
    count  exact.
"""
import math

import numpy as np
import pytest
import torch as th

gpu = pytest.mark.gpu  # every test that launches a kernel; the checks of the float64 references run anywhere

EPS = 2.0 ** -24
F32 = np.float32


def _ceil(a, b):
    return -(-a // b)


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _sms():
    return th.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# 1. preference loss: float64 restatement of PreferenceModel.probability + F.binary_cross_entropy + its gradient
# ---------------------------------------------------------------------------------------------------------------------
def _bce(p, y):
    """torch's binary_cross_entropy per element, logs clamped at -100, in float64."""
    with np.errstate(divide="ignore"):
        lp = np.maximum(np.log(p), -100.0)
        l1p = np.maximum(np.log1p(-p), -100.0)
    return -(y * lp + (1.0 - y) * l1p)


def _dbce(p, y):
    """torch's BCE backward without the 1 / P: (p - y) / max(p (1 - p), 1e-12), increasing in p."""
    return (p - y) / np.maximum(p * (1.0 - p), 1e-12)


def _returns_diff64(rews, discount):
    """s = sum_t g^t (r2 - r1) in float64 from the float32 inputs, and the magnitude sum_t |g^t (r2 - r1)|."""
    r = np.asarray(rews, np.float64)
    Lf = r.shape[2]
    w = float(F32(discount)) ** np.arange(Lf, dtype=np.float64)
    terms = (r[1] - r[0]) * w
    return terms.sum(1), np.abs(terms).sum(1), w


def pref_loss64(rews, prefs, noise, discount, threshold, grad_scale):
    """float64 probabilities, mean BCE, accuracy and grad_scale * d loss / d rews[2][P][L] of one minibatch."""
    s, _, w = _returns_diff64(rews, discount)
    noise, thr = float(F32(noise)), float(F32(threshold))
    y = np.asarray(prefs, np.float64)
    P = len(y)
    d = np.clip(s, -thr, thr)
    e = np.exp(d)
    m = 1.0 / (1.0 + e)
    p = noise * 0.5 + (1.0 - noise) * m
    loss = _bce(p, y)
    clipped = (s < -thr) | (s > thr)
    g = np.where(clipped, 0.0, -grad_scale * _dbce(p, y) / P * (1.0 - noise) * m * (m * e))  # m e = 1 - m, uncancelled
    grad = np.stack([-g[:, None] * w[None, :], g[:, None] * w[None, :]])
    return p, float(loss.mean()), float(np.mean((p > 0.5) == (y > 0.5))), grad


def test_pref_loss64_matches_probability_port_and_autograd():
    """The float64 restatement against oracle/pref_port.probability_port + F.binary_cross_entropy + autograd, both in
    float64: clipped pairs, pairs exactly at +-threshold (th.clip passes the gradient there), s = 0, soft labels."""
    from oracle import pref_port

    rng = np.random.default_rng(0)
    # probability_port forms float32 discount powers: 0.5^t is exact there
    for noise, discount, thr in ((0.0, 1.0, 50.0), (0.1, 0.5, 1.5), (0.1, 1.0, 1.5)):
        P, Lf = 24, 7
        rews = (rng.standard_normal((2, P, Lf)) * 2).astype(F32)
        rews[:, 0, 1:] = 0
        rews[0, 0, 0], rews[1, 0, 0] = 0.25, 0.25 + thr     # s = +threshold exactly
        rews[:, 1, 1:] = 0
        rews[0, 1, 0], rews[1, 1, 0] = 0.25 + thr, 0.25     # s = -threshold exactly
        rews[1, 2] = rews[0, 2]                             # s = 0
        rews[1, 3] = rews[0, 3] + 20                        # clipped
        y = rng.random(P).astype(F32)
        y[:6] = [1, 0, 0.5, 1, 0, 1]
        p, loss, acc, grad = pref_loss64(rews, y, noise, discount, thr, 0.3)
        rt = th.tensor(rews, dtype=th.float64, requires_grad=True)
        probs = th.stack([pref_port.probability_port(rt[0, k], rt[1, k], float(F32(noise)), float(F32(discount)), thr)
                          for k in range(P)])
        lt = th.nn.functional.binary_cross_entropy(probs, th.tensor(y, dtype=th.float64))
        (0.3 * lt).backward()
        np.testing.assert_allclose(p, probs.detach().numpy(), rtol=1e-13, atol=0)
        assert abs(loss - float(lt.detach())) <= 1e-13 * abs(loss)
        np.testing.assert_allclose(grad, rt.grad.numpy(), rtol=1e-12, atol=1e-13 * np.abs(grad).max())  # p - y of soft labels cancels
        assert (grad[:, :2] != 0).all() and (grad[:, 3] == 0).all()
        assert acc == float(((probs > 0.5) == (th.tensor(y) > 0.5)).double().mean())


def _pref_bounds(rews, y, noise, discount, thr, grad_scale):
    """Per-pair float64 reference intervals [lo, hi] of p, loss and the pair's gradient (see the module docstring)."""
    s, mag, w = _returns_diff64(rews, discount)
    Lf = rews.shape[2]
    noise, thr = float(F32(noise)), float(F32(thr))
    y = y.astype(np.float64)
    P = len(y)
    err_s = (_ceil(Lf, 32) + 16) * EPS * mag
    if Lf == 1:
        err_s = np.where(np.float64(F32(s)) == s, 0.0, err_s)  # one exact difference and one exact product
    d = np.clip(s, -thr, thr)
    e = np.exp(d)
    m = 1.0 / (1.0 + e)
    p = noise * 0.5 + (1.0 - noise) * m
    k = (1.0 - noise) * m * (m * e)
    inside = np.abs(s) + err_s < thr
    outside = np.abs(s) - err_s > thr
    tol_p = np.where(outside, 0.0, k * err_s) + 8 * EPS * p
    p_lo = np.maximum(p - tol_p, 0.0).astype(F32)
    p_lo = np.where(p_lo > p - tol_p, np.nextafter(p_lo, F32(-1)), p_lo).astype(np.float64)
    p_hi = np.minimum(p + tol_p, 1.0).astype(F32)
    p_hi = np.where(p_hi < p + tol_p, np.nextafter(p_hi, F32(2)), p_hi).astype(np.float64)
    p_lo, p_hi = np.clip(p_lo, 0, 1), np.clip(p_hi, 0, 1)
    l_ends = np.stack([_bce(p_lo, y), _bce(p_hi, y)])
    l_lo = np.where((y >= p_lo) & (y <= p_hi), _bce(y, y), l_ends.min(0))
    l_hi = l_ends.max(0)
    l_mar = 8 * EPS * np.abs(l_ends).max(0)
    h_lo, h_hi = _dbce(p_lo, y), _dbce(p_hi, y)
    ks = np.exp(np.where(outside, 0.0, err_s))
    k_lo, k_hi = k / ks * (1 - 8 * EPS), k * ks * (1 + 8 * EPS)
    c = -grad_scale / P
    corners = np.stack([c * h_lo * k_lo, c * h_lo * k_hi, c * h_hi * k_lo, c * h_hi * k_hi])
    g_lo, g_hi = corners.min(0), corners.max(0)
    g_mar = 8 * EPS * np.abs(corners).max(0)
    g_lo, g_hi = np.where(inside, g_lo - g_mar, np.minimum(g_lo - g_mar, 0)), np.where(inside, g_hi + g_mar,
                                                                                       np.maximum(g_hi + g_mar, 0))
    g_lo, g_hi = np.where(outside, 0.0, g_lo), np.where(outside, 0.0, g_hi)
    return dict(s=s, p=p, tol_p=tol_p, l_lo=l_lo - l_mar, l_hi=l_hi + l_mar, g_lo=g_lo, g_hi=g_hi, w=w,
                amb=np.abs(p - 0.5) <= tol_p, y=y)


def _pref_inputs(P, Lf, discount, thr, seed):
    """rews[2][P][L] and soft labels with the special pairs in front: +-threshold exactly (L = 1), s = 0 with y = 0,
    0.5 and 1, and |s| in the band 43.7 < |s| < 50 where m^2 is subnormal."""
    g = th.Generator(device="cuda").manual_seed(seed)
    rews = th.randn(2, P, Lf, device="cuda", generator=g)
    y = th.rand(P, device="cuda", generator=g)
    y[::3] = (y[::3] > 0.5).float()
    specials = []
    if Lf == 1:
        specials += [("thr", thr, 1.0), ("thr", -thr, 0.0), ("thr", thr, 0.5), ("thr", -thr, 0.3)]
    specials += [("zero", 0.0, 0.0), ("zero", 0.0, 0.5), ("zero", 0.0, 1.0)]
    if thr > 43.7:
        specials += [("band", v, yy) for v, yy in ((44.0, 1.0), (46.5, 0.0), (49.9, 0.5), (-45.0, 0.0), (-48.0, 1.0),
                                                   (47.25, 0.2))]
    specials = specials[:P]
    for i, (kind, v, yy) in enumerate(specials):
        y[i] = yy
        if kind == "thr":
            rews[0, i, 0], rews[1, i, 0] = (0.25, 0.25 + v) if v > 0 else (0.25 - v, 0.25)
        elif kind == "zero":
            rews[1, i] = rews[0, i]
        else:
            wsum = sum(float(F32(discount)) ** t for t in range(Lf))
            rews[0, i] = 0.5
            rews[1, i] = 0.5 + v / wsum
    return rews.contiguous(), y.contiguous(), specials


PREF_CASES = [(Lf, P, disc, noise, thr) for Lf in (1, 31, 32, 33, 100, 1000) for P in (1, 8, 4225, 20000)
              for disc in (1.0, 0.9) for noise in (0.0, 0.1) for thr in (50.0, 1.5)]


@gpu
@pytest.mark.parametrize("Lf,P,discount,noise,thr", PREF_CASES)
def test_pref_loss_sweep_against_float64(L, Lf, P, discount, noise, thr):
    seed = 1000 * Lf + P + int(10 * noise) + int(thr) + int(10 * discount)
    rews, y, specials = _pref_inputs(P, Lf, discount, thr, seed)
    gs = 0.75
    grad = th.full((2 * P * Lf,), float("nan"), device="cuda")
    probs = th.full((P,), float("nan"), device="cuda")
    stats = th.zeros(12, device="cuda")
    for _ in range(2):  # two minibatches accumulate into slot 2 of a 3-slot accumulator
        L.pref_loss(rews.view(-1), P, Lf, y, noise, discount, thr, gs, grad, probs, stats, 2)
    # validation form: no gradient, no probabilities, statistics only
    stats_v = th.zeros(4, device="cuda")
    L.pref_loss(rews.view(-1), P, Lf, y, noise, discount, thr, gs, None, None, stats_v, 0)
    r, yh = rews.cpu().numpy(), y.cpu().numpy()
    B = _pref_bounds(r, yh, noise, discount, thr, gs)
    got_p = probs.cpu().numpy().astype(np.float64)
    bad = np.abs(got_p - B["p"]) > B["tol_p"]
    assert not bad.any(), f"p: {np.flatnonzero(bad)[:5]} got {got_p[bad][:5]} want {B['p'][bad][:5]}"
    gr = grad.cpu().numpy().reshape(2, P, Lf)
    np.testing.assert_array_equal(gr[0], -gr[1])
    g0 = gr[1][:, 0].astype(np.float64)
    bad = (g0 < B["g_lo"]) | (g0 > B["g_hi"])
    assert not bad.any(), (f"grad: pairs {np.flatnonzero(bad)[:5]} got {g0[bad][:5]} in [{B['g_lo'][bad][:5]}, "
                           f"{B['g_hi'][bad][:5]}] s={B['s'][bad][:5]}")
    if Lf > 1:
        want_t = g0[:, None] * B["w"][None, :]
        if discount == 1.0:
            np.testing.assert_array_equal(gr[1], np.broadcast_to(gr[1][:, :1], gr[1].shape))
        else:
            # + 2^-125 |g|: far down the fragment g^t leaves float32's normal range, where CUDA's powf may return 0;
            # + 2^-149: a product below the normal range is rounded to a multiple of the smallest subnormal
            bad = np.abs(gr[1] - want_t) > 10 * EPS * np.abs(want_t) + 2.0 ** -125 * np.abs(g0)[:, None] + 2.0 ** -149
            assert not bad.any(), (np.argwhere(bad)[:4], gr[1][bad][:4], want_t[bad][:4])
    for i, (kind, v, _) in enumerate(specials):
        if kind == "thr":  # th.clip passes the gradient at equality
            assert B["s"][i] == v and g0[i] != 0, (i, v, g0[i])
        if kind == "zero":
            assert B["s"][i] == 0 and got_p[i] == 0.5
    # statistics: [8] loss sum, [9] accuracy sum, [10] minibatch count, other slots untouched
    st = stats.cpu().numpy().astype(np.float64)
    assert (st[:8] == 0).all() and st[10] == 2.0 and st[11] == 0.0
    ctas = min(_ceil(P, 8), 4 * _sms())
    c_sum = _ceil(P, 8 * ctas) + 8 + ctas + 4
    lmag = np.maximum(np.abs(B["l_lo"]), np.abs(B["l_hi"])).sum() / P
    lo, hi = B["l_lo"].sum() / P, B["l_hi"].sum() / P
    for got, k in ((st[8], 2), (float(stats_v[0]), 1)):
        assert k * lo - 2 * c_sum * EPS * lmag <= got <= k * hi + 2 * c_sum * EPS * lmag, (got, k * lo, k * hi)
    acc_c = ((B["p"] > 0.5) == (B["y"] > 0.5)).sum()
    slack = B["amb"].sum()
    for got, k in ((st[9], 2), (float(stats_v[1]), 1)):
        n_right = got * P / k
        assert abs(n_right - acc_c) <= slack + 2 * c_sum * EPS * P, (n_right, acc_c, slack)
    assert float(stats_v[2]) == 1.0


# ---------------------------------------------------------------------------------------------------------------------
# 2. output-norm scans: NormalizedRewardNet.predict_processed over consecutive env steps, RunningNorm and EMANorm
# ---------------------------------------------------------------------------------------------------------------------
def scan64(x, mean, var, count, eps, update, ema_decay=None, inv_lr=0.0, nb=0):
    """x[T][E] float32 -> (out[T][E], mean, var, count, inv_lr, nb, tol_out[T][E], tol_mean, tol_var) in float64:
    step t is normalised with the statistics from before step t, then its batch mean and biased variance are folded
    (RunningNorm.update_stats or EMANorm.update_stats)."""
    x = np.asarray(x, np.float64)
    T, E = x.shape
    eps = float(F32(eps))
    threads = 1024
    while threads > 32 and threads // 2 >= E:
        threads //= 2
    c_loc = (_ceil(E, threads) + 48) * EPS
    out = np.empty_like(x)
    tol_out = np.empty_like(x)
    tm = tv = 0.0
    for t in range(T):
        xt = x[t]
        istd = 1.0 / math.sqrt(var + eps)
        out[t] = (xt - mean) * istd
        tol_out[t] = istd * (4 * EPS * (np.abs(xt) + abs(mean)) + tm) + np.abs(out[t]) * (tv / (2 * (var + eps)) + 4 * EPS)
        bm = xt.mean()
        bv = ((xt - bm) ** 2).mean()
        if not update:
            continue
        dm = bm - mean
        loc_m = c_loc * (np.abs(xt).mean() + abs(mean) + abs(bm))
        if ema_decay is None:
            tot = count + E
            mean = mean + dm * E / tot
            var = (var * count + bv * E + dm * dm * count * E / tot) / tot
        else:
            inv_lr = inv_lr + float(F32(ema_decay)) ** nb
            lr = 1.0 / inv_lr
            mean = mean + lr * dm
            var = var + lr * (bv + (1 - lr) * dm * dm - var)
            nb += 1
        count += E
        dm_err = tm + loc_m
        tv = tv + c_loc * (bv + var + dm * dm + np.abs(xt - bm).mean() ** 2) + 2 * abs(dm) * dm_err + dm_err ** 2 \
            + 2 * math.sqrt(bv) * loc_m + loc_m ** 2
        tm = tm + loc_m
    return out, mean, var, count, inv_lr, nb, tol_out, tm, tv


def test_scan64_matches_running_and_ema_norm():
    """The float64 scan against the reference-shaped modules in float64: oracle RunningNormPort (update, then the
    statistics of the next step) and the package's EMANorm."""
    from imitation_b200.util import networks
    from oracle import nets_port

    rng = np.random.default_rng(1)
    x = (rng.standard_normal((5, 13)) * 3 + 1).astype(F32)
    rn = nets_port.RunningNormPort(1).double()
    em = networks.EMANorm(1, decay=0.5).double()  # th.pow(decay, k) is float32: exact for 0.5
    for kind, mod in (("rn", rn), ("ema", em)):
        out = scan64(x, 0.0, 1.0, 0, 1e-5, True, None if kind == "rn" else 0.5)
        want = []
        for t in range(len(x)):
            xt = th.tensor(x[t], dtype=th.float64).reshape(-1, 1)
            want.append(((xt - mod.running_mean) / th.sqrt(mod.running_var + float(F32(1e-5)))).numpy().ravel())
            mod.update_stats(xt)
        np.testing.assert_allclose(out[0], np.stack(want), rtol=1e-13, atol=1e-13)
        assert abs(out[1] - float(mod.running_mean)) <= 1e-13 and abs(out[2] - float(mod.running_var)) <= 1e-13


SCAN_E = (1, 31, 32, 33, 1023, 1024, 1025, 4103, 65536)


@gpu
@pytest.mark.parametrize("kind", ["running", "ema"])
@pytest.mark.parametrize("E", SCAN_E)
@pytest.mark.parametrize("T", [1, 2, 300])
def test_reward_norm_scan_sweep_against_float64(L, kind, E, T):
    """Both layouts (contiguous [T][E], and the reward column of an [E][T][rw] rollout table whose other columns stay
    bit-unchanged), update_stats 0 and 1, starting counts 0 and 2^24 + 3; two calls give the same bits."""
    rng = np.random.default_rng(E * 7 + T)
    rw, col = 7, 4
    raw = (rng.standard_normal((T, E)) * 2.5 + 1.5).astype(F32)
    decay = 0.99
    g = th.Generator(device="cuda").manual_seed(E + T)
    tbl_base = th.randn(E, T, rw, device="cuda", generator=g)  # one rollout table per size, cloned per call
    tbl_base[:, :, col] = th.tensor(raw.T.copy(), device="cuda")
    other = th.ones(rw, dtype=th.bool, device="cuda")
    other[col] = False
    for cnt0, (m0, v0, ilr0, nb0) in ((0, (0.0, 1.0, 0.0, 0)), ((1 << 24) + 3, (0.3, 2.0, 37.5, 41))):
        for update in (0, 1):
            want = scan64(raw, float(F32(m0)), float(F32(v0)), cnt0, 1e-5, update,
                          None if kind == "running" else decay, float(F32(ilr0)), nb0)
            out_w, mean_w, var_w, cnt_w, ilr_w, nb_w, tol_out, tm, tv = want
            for layout in ("contig", "table"):
                runs = []
                for _ in range(2):
                    state = th.tensor([m0, v0] + ([ilr0] if kind == "ema" else []), dtype=th.float32, device="cuda")
                    cnts = th.tensor([cnt0] + ([nb0] if kind == "ema" else []), dtype=th.int32, device="cuda")
                    if layout == "contig":
                        buf = th.tensor(raw, device="cuda")
                        L.reward_norm_scan(buf, E, T, E, 1, state, cnts, 1e-5, update,
                                           None if kind == "running" else decay)
                        got = buf.cpu().numpy()
                    else:
                        tbl = tbl_base.clone()
                        L.reward_norm_scan(tbl.view(-1)[col:], E, T, rw, T * rw, state, cnts, 1e-5, update,
                                           None if kind == "running" else decay)
                        assert th.equal(tbl[:, :, other], tbl_base[:, :, other])  # bit-unchanged
                        got = tbl[:, :, col].T.cpu().numpy()
                    runs.append((got, state.cpu().numpy(), cnts.cpu().numpy()))
                for a, b in zip(runs[0], runs[1]):
                    np.testing.assert_array_equal(a, b)
                got, st, cn = runs[0]
                bad = np.abs(got - out_w) > tol_out
                assert not bad.any(), (layout, cnt0, update, np.argwhere(bad)[:3], got[bad][:3], out_w[bad][:3])
                if not update:
                    np.testing.assert_array_equal(st, np.array([m0, v0] + ([ilr0] if kind == "ema" else []), F32))
                    assert list(cn) == [cnt0] + ([nb0] if kind == "ema" else [])
                    continue
                assert abs(st[0] - mean_w) <= tm + 4 * EPS * abs(mean_w), (st[0], mean_w, tm)
                assert abs(st[1] - var_w) <= tv + 4 * EPS * var_w, (st[1], var_w, tv)
                assert int(cn[0]) == cnt_w
                if kind == "ema":
                    assert int(cn[1]) == nb_w and abs(st[2] - ilr_w) <= 4 * EPS * T * ilr_w


# ---------------------------------------------------------------------------------------------------------------------
# 3. RunningNorm batch statistics and fold (imb_norm_batch_stats / imb_norm_fold)
# ---------------------------------------------------------------------------------------------------------------------
def fold64(mean, var, count, b_mean, b_var, b_n):
    """RunningNorm.update_stats in float64 from the batch's mean and biased variance."""
    tot = count + b_n
    delta = b_mean - mean
    return mean + delta * b_n / tot, (var * count + b_var * b_n + delta * delta * count * b_n / tot) / tot, tot


def test_fold64_matches_running_norm_port():
    from oracle import nets_port

    rng = np.random.default_rng(2)
    port = nets_port.RunningNormPort(5).double()
    mean, var, cnt = np.zeros(5), np.ones(5), 0
    for n in (1, 7, 300):
        x = rng.standard_normal((n, 5)) * 3 + 1e3
        port.update_stats(th.tensor(x))
        mean, var, cnt = fold64(mean, var, cnt, x.mean(0), x.var(0), n)
    np.testing.assert_allclose(mean, port.running_mean.numpy(), rtol=1e-14)
    np.testing.assert_allclose(var, port.running_var.numpy(), rtol=1e-10)
    assert cnt == int(port.count)


def test_policy_norm_slot_list_holds_one_update():
    """The deferred policy feature-norm list of a GAIL trainer always holds one discriminator update's minibatches: with
    512 minibatches per update it has at least 512 slots (a full list would overwrite its last slot)."""
    from imitation_b200.algorithms.adversarial import common

    assert common.policy_norm_slots(512 * 128, 128) >= 512
    assert common.policy_norm_slots(65536, 128) >= 512
    assert common.policy_norm_slots(1024, 64) == 256


NORM_DIN = (1, 2, 31, 32, 33, 63, 64)
NORM_N = (1, 2, 127, 128, 129, 262144, 262145)
NORM_CASES = [(din, n) for din in NORM_DIN for n in NORM_N if n < 262144 or din in (1, 33, 64)]


def _norm_data(din, n, row0, seed, extra=8):
    """Feature-major batch [row0 + din + 2][ld]: columns [0, n + extra - 1) hold data, the rest NaN, and so do the rows
    outside [row0, row0 + din).  Features cycle through |mean| = 1e3 with std 1e-2, constants, and N(0.5, 2)."""
    ld = n + extra + 5
    g = th.Generator(device="cuda").manual_seed(seed)
    b = th.full((row0 + din + 2, ld), float("nan"), device="cuda")
    nv = n + extra - 1
    x = th.randn(din, nv, device="cuda", generator=g)
    kind = th.arange(din, device="cuda") % 3
    sign = th.where(th.arange(din, device="cuda") % 2 == 0, 1.0, -1.0)
    x = th.where((kind == 0)[:, None], sign[:, None] * 1e3 + 1e-2 * x, x)
    x = th.where((kind == 1)[:, None], (0.37 + th.arange(din, device="cuda")[:, None].float()).expand(din, nv), x)
    x = th.where((kind == 2)[:, None], 0.5 + 2 * x, x)
    b[row0:row0 + din, :nv] = x
    return b, ld, x.double().cpu().numpy()


def _moment_tols(x, chunk, nchunks):
    c = 2 * (_ceil(chunk, 32) + _ceil(nchunks, 32) + 12) * EPS
    mean, var = x.mean(1), x.var(1)
    sd = np.sqrt(var)
    tm = c * (np.abs(mean) + sd)
    return mean, var, tm, c * var + 4 * sd * tm + tm * tm


def _check_fold(got_mv, got_cnt, ref, tag):
    mean, var, cnt, tm, tv = ref
    din = len(mean)
    gm, gv = got_mv[:din].astype(np.float64), got_mv[din:2 * din].astype(np.float64)
    assert int(got_cnt) == cnt, (tag, int(got_cnt), cnt)
    bad = np.abs(gm - mean) > tm
    assert not bad.any(), (tag, "mean", np.flatnonzero(bad)[:4], gm[bad][:4], mean[bad][:4], tm[bad][:4])
    bad = np.abs(gv - var) > tv
    assert not bad.any(), (tag, "var", np.flatnonzero(bad)[:4], gv[bad][:4], var[bad][:4], tv[bad][:4])


def _fold_ref(state, batches):
    """state (mean, var, count, tol_mean, tol_var) folded with each (mean, var, n, tol_mean, tol_var) batch, float64."""
    mean, var, cnt, tm, tv = state
    for b_mean, b_var, b_n, btm, btv in batches:
        delta = b_mean - mean
        tot = cnt + b_n
        a = b_n / tot
        nm, nv, _ = fold64(mean, var, cnt, b_mean, b_var, b_n)
        dterr = tm + btm
        tv = (1 - a) * tv + a * btv + 8 * EPS * (nv + var + b_var + delta * delta) + 2 * np.abs(delta) * dterr \
            + dterr * dterr
        tm = (1 - a) * tm + a * btm + 8 * EPS * (np.abs(nm) + np.abs(delta))
        mean, var, cnt = nm, nv, tot
    return mean, var, cnt, tm, tv


@gpu
@pytest.mark.parametrize("din,n", NORM_CASES)
def test_norm_batch_stats_and_fold_sweep(L, din, n):
    """Immediate mode, deferred slots folded by count, and a fixed slot count (1, 2, 3 or 8, as after the distributed
    all-gather), at row0 0 and 3; NaN past column n and outside the feature rows never reaches a result."""
    from imitation_b200 import _desc

    d = _desc.disc_desc(2, 1, normalize_input=True)
    ws = th.zeros(L.disc_workspace_floats(d), device="cuda")
    chunk = 128 if n <= 128 * 2048 else 512
    nchunks = _ceil(n, chunk)
    k_fixed = (1, 2, 3, 8)[(NORM_DIN.index(din) + NORM_N.index(n)) % 4]
    for row0 in (0, 3):
        b, ld, x = _norm_data(din, n, row0, seed=din * 1000 + n + row0)
        flat = b.view(-1)
        mom = {}
        for off in sorted({7} | set(range(max(3, k_fixed)))):
            mean, var, tm, tv = _moment_tols(x[:, off:off + n], chunk, nchunks)
            mom[off] = (mean, var, n, tm, tv)
        rng = np.random.default_rng(din + n + row0)
        m0 = rng.standard_normal(din).astype(F32)
        v0 = (rng.random(din) + 0.5).astype(F32)
        for cnt0 in (0, 1000):
            start = (m0.astype(np.float64), v0.astype(np.float64), cnt0, np.zeros(din), np.zeros(din))
            # immediate
            ns = th.tensor(np.concatenate([m0, v0]), device="cuda")
            nc = th.tensor([cnt0], dtype=th.int32, device="cuda")
            L.norm_batch_stats(d, flat[7:], ld, n, row0, din, ns, nc, None, 0, ws)
            _check_fold(ns.cpu().numpy(), int(nc), _fold_ref(start, [mom[7]]), ("immediate", row0, cnt0))
            # deferred: three batches into a list of 8 slots, nothing changes before the fold
            cap = 8
            sw = 2 * din + 1
            defer = th.zeros(4 + cap * sw + 64, device="cuda")
            defer[4 + cap * sw:] = 12345.0  # guard past the list
            ns = th.tensor(np.concatenate([m0, v0]), device="cuda")
            nc = th.tensor([cnt0], dtype=th.int32, device="cuda")
            for off in range(3):
                L.norm_batch_stats(d, flat[off:], ld, n, row0, din, ns, nc, defer, cap, ws)
            dv = defer.cpu().numpy()
            assert dv[0] == 3.0 and (ns.cpu().numpy() == np.concatenate([m0, v0])).all() and int(nc) == cnt0
            for s in range(3):
                slot = dv[4 + s * sw:4 + (s + 1) * sw].astype(np.float64)
                mean, var, _, tm, tv = mom[s]
                assert slot[2 * din] == n
                assert (np.abs(slot[:din] - mean) <= tm).all(), ("slot mean", s, slot[:din], mean)
                assert (np.abs(slot[din:2 * din] - var) <= tv).all(), ("slot var", s, slot[din:2 * din], var)
            L.norm_fold(din, defer, ns, nc)
            _check_fold(ns.cpu().numpy(), int(nc), _fold_ref(start, [mom[s] for s in range(3)]), ("deferred", row0))
            assert float(defer[0]) == 0.0 and (defer[4 + cap * sw:] == 12345.0).all()
            # fixed slot count: the list keeps its counter
            defer.zero_()
            ns = th.tensor(np.concatenate([m0, v0]), device="cuda")
            nc = th.tensor([cnt0], dtype=th.int32, device="cuda")
            for off in range(k_fixed):
                L.norm_batch_stats(d, flat[off:], ld, n, row0, din, ns, nc, defer, cap, ws)
            L.norm_fold(din, defer, ns, nc, k_fixed)
            _check_fold(ns.cpu().numpy(), int(nc), _fold_ref(start, [mom[s] for s in range(k_fixed)]),
                        ("fixed", k_fixed, row0))
            assert float(defer[0]) == k_fixed


@gpu
def test_deferred_slot_list_saturates(L):
    """cap + 3 deferred updates into a list of cap slots: the counter stops at cap, the last slot holds the last batch,
    nothing past the list is written, and the fold applies exactly cap slots."""
    from imitation_b200 import _desc

    d = _desc.disc_desc(2, 1, normalize_input=True)
    ws = th.zeros(L.disc_workspace_floats(d), device="cuda")
    din, n, cap = 5, 300, 4
    b, ld, x = _norm_data(din, n, 0, seed=5, extra=cap + 3)
    sw = 2 * din + 1
    defer = th.zeros(4 + cap * sw + 64, device="cuda")
    defer[4 + cap * sw:] = 12345.0
    ns = th.cat([th.zeros(din), th.ones(din)]).cuda()
    nc = th.zeros(1, dtype=th.int32, device="cuda")
    for off in range(cap + 3):
        L.norm_batch_stats(d, b.view(-1)[off:], ld, n, 0, din, ns, nc, defer, cap, ws)
    th.cuda.synchronize()
    assert float(defer[0]) == cap and (defer[4 + cap * sw:] == 12345.0).all()
    L.norm_fold(din, defer, ns, nc)
    batches = []
    for off in list(range(cap - 1)) + [cap + 2]:
        mean, var, tm, tv = _moment_tols(x[:, off:off + n], 128, _ceil(n, 128))
        batches.append((mean, var, n, tm, tv))
    _check_fold(ns.cpu().numpy(), int(nc), _fold_ref((np.zeros(din), np.ones(din), 0, np.zeros(din), np.zeros(din)),
                                                     batches), "saturated")
    assert float(defer[0]) == 0.0 and int(nc) == cap * n


# ---------------------------------------------------------------------------------------------------------------------
# 4. replica merge: snapshot -> per-rank updates -> pack -> sum -> unpack, world ranks emulated in one process
# ---------------------------------------------------------------------------------------------------------------------
SYNC_CFGS = {
    "one_k1": dict(ks=(1,), avg=(40000,)),
    "two_k17_k64": dict(ks=(17, 64), avg=(40000, 3501, 1)),
    "four": dict(ks=(1, 17, 64, 17), avg=(8193, 17, 40000, 2, 1)),
}


@gpu
@pytest.mark.parametrize("cfg", sorted(SYNC_CFGS))
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_sync_merge_sweep_against_pooled_float64(L, cfg, world):
    ks, avg_sizes = SYNC_CFGS[cfg]["ks"], SYNC_CFGS[cfg]["avg"]
    rng = np.random.default_rng(world * 10 + len(ks))
    # common start: feature 0 of every norm sits at |mean| 1e3 with std 1e-2 (var = S2 / n - mean^2 cancels)
    starts = []
    for k in ks:
        m = rng.standard_normal(k) * 2
        v = rng.random(k) + 0.5
        m[0], v[0] = 1e3, 1e-4
        starts.append((m.astype(F32), v.astype(F32), int(rng.integers(0, 5000))))
    ranks = []
    for r in range(world):
        avg = [rng.standard_normal(n).astype(F32) for n in avg_sizes]
        norms = []
        for (m0, v0, c0), k in zip(starts, ks):
            nr = 0 if r == world - 1 and world > 1 else int(rng.integers(1, 700))
            rows = rng.standard_normal((nr, k)) * 1.5 + 0.3
            rows[:, 0] = 1e3 + 1e-2 * rng.standard_normal(nr)
            if nr:
                mm, vv, cc = fold64(m0.astype(np.float64), v0.astype(np.float64), c0, rows.mean(0), rows.var(0), nr)
            else:
                mm, vv, cc = m0, v0, c0
            norms.append((np.asarray(mm).astype(F32), np.asarray(vv).astype(F32), cc, rows))
        ranks.append((avg, norms))
    dev = lambda a: th.tensor(np.ascontiguousarray(a), device="cuda")
    t_start = [(dev(m), dev(v), dev(np.array([c], np.int32))) for m, v, c in starts]  # alive while the desc is used
    d_start = L.sync_desc([], t_start)
    snap = th.zeros(sum(1 + 2 * k for k in ks), dtype=th.float64, device="cuda")
    L.sync_snapshot(d_start, snap)
    total = None
    tensors = []
    for avg, norms in ranks:
        ta = [dev(a) for a in avg]
        tn = [(dev(m), dev(v), dev(np.array([c], np.int32))) for m, v, c, _ in norms]
        dsc = L.sync_desc(ta, tn)
        buf = th.zeros(L.sync_buffer_doubles(dsc), dtype=th.float64, device="cuda")
        L.sync_pack(dsc, buf)
        total = buf if total is None else total + buf
        tensors.append((dsc, ta, tn))
    dsc0, ta0, tn0 = tensors[0]
    L.sync_unpack(dsc0, total, snap, world)
    th.cuda.synchronize()
    for i in range(len(avg_sizes)):
        acc = ranks[0][0][i].astype(np.float64)
        for r in range(1, world):
            acc = acc + ranks[r][0][i].astype(np.float64)
        np.testing.assert_array_equal(ta0[i].cpu().numpy(), (acc * (1.0 / world)).astype(F32), err_msg=f"avg {i}")
    for j, k in enumerate(ks):
        m0, v0, c0 = starts[j]
        rows = np.concatenate([ranks[r][1][j][3] for r in range(world)])
        if len(rows):
            mean, var, cnt = fold64(m0.astype(np.float64), v0.astype(np.float64), c0, rows.mean(0), rows.var(0), len(rows))
        else:
            mean, var, cnt = m0.astype(np.float64), v0.astype(np.float64), c0
        mags_m = np.max([np.abs(ranks[r][1][j][0]).astype(np.float64) for r in range(world)] + [np.abs(m0)], axis=0)
        mags_v = np.max([ranks[r][1][j][1].astype(np.float64) + ranks[r][1][j][0].astype(np.float64) ** 2
                         for r in range(world)] + [v0 + m0.astype(np.float64) ** 2], axis=0)
        gm, gv, gc = (t.cpu().numpy() for t in tn0[j])
        assert int(gc[0]) == cnt, (j, int(gc[0]), cnt)
        assert (np.abs(gm - mean) <= 8 * EPS * mags_m * world).all(), (j, gm, mean)
        assert (np.abs(gv - var) <= 8 * EPS * mags_v * world).all(), (j, gv, var)


# ---------------------------------------------------------------------------------------------------------------------
# 5. data path: table store + ring, gather, index sampling, fused sample + gather; bit-exact against NumPy twins
# ---------------------------------------------------------------------------------------------------------------------
def _state():
    from imitation_b200 import _lib

    return th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")


@gpu
@pytest.mark.parametrize("discrete", [False, True])
@pytest.mark.parametrize("cap", [1, 7, 1000])
def test_table_store_ring_sweep(L, cap, discrete):
    """imb_table_store + imb_ring_advance == data_port.ReplayBufferPort.store over n = 1, cap - 1, cap, cap + 1 and
    3 cap + 5 after a first store that leaves idx0 != 0; Discrete actions land one-hot."""
    from oracle import data_port

    Do, Da = 3, 4
    tw = 2 * Do + Da + 1
    rng = np.random.default_rng(cap + discrete)
    port = data_port.ReplayBufferPort(cap, (Do,), () if discrete else (Da,), np.float32,
                                      np.int64 if discrete else np.float32)
    table = th.zeros(cap, tw, device="cuda")
    st = _state()
    for n in [max(1, cap // 2 + 1), 1, cap - 1, cap, cap + 1, 3 * cap + 5]:
        if n < 1:
            continue
        obs = rng.standard_normal((n, Do)).astype(F32)
        nobs = rng.standard_normal((n, Do)).astype(F32)
        acts = rng.integers(0, Da, n) if discrete else rng.standard_normal((n, Da)).astype(F32)
        dones = rng.random(n) < 0.3
        dv = lambda a, dt=None: th.tensor(np.ascontiguousarray(a), device="cuda", dtype=dt)
        L.table_store(table, cap, Do, Da, dv(obs), None if discrete else dv(acts), dv(acts, th.int64) if discrete else None,
                      dv(nobs), dv(dones.astype(np.uint8)), n, True, st)
        L.ring_advance(st, cap, n)
        port.store(dict(obs=obs, acts=acts, next_obs=nobs, dones=dones, infos=np.empty(n, object)))
        a = port._buffer._arrays
        pa = np.eye(Da, dtype=F32)[a["acts"]] if discrete else a["acts"]
        want = np.concatenate([a["obs"], pa, a["next_obs"], a["dones"][:, None].astype(F32)], 1)
        want[port.size():] = 0  # rows never written (the port's action 0 would be one-hot); the table started at zero
        np.testing.assert_array_equal(table.cpu().numpy(), want, err_msg=f"cap {cap} n {n}")
        assert [int(st[L.ST_RING_IDX]), int(st[L.ST_RING_N])] == [port._buffer._idx, port._buffer._n_data]


def _grid_wave_rows():
    return 16 * _sms() * 128


@gpu
@pytest.mark.parametrize("tw", [1, 7, 8, 9, 41, 129])
def test_gather_rows_sweep(L, tw):
    """Every tw % 8 of row_to_column, a gather past one grid wave of 16 x SMs x 128 rows, col0 > 0 and the clamp of
    out-of-range indices to [0, capacity - 1]; columns outside [col0, col0 + n) and rows past tw stay untouched."""
    cap = 1000
    rng = np.random.default_rng(tw)
    tab = rng.standard_normal((cap, tw)).astype(F32)
    table = th.tensor(tab, device="cuda")
    for n in (1, 33, _grid_wave_rows() + 33):
        idx = rng.integers(0, cap, n)
        idx[:: max(1, n // 7)] = -5
        idx[1:: max(2, n // 5)] = cap + 3
        col0 = 13
        ld = col0 + n + 11
        batch = th.full((tw + 1, ld), -7.0, device="cuda")
        L.gather_rows(table, cap, tw, th.tensor(idx, device="cuda"), n, batch, ld, col0)
        got = batch.cpu().numpy()
        want = np.full((tw + 1, ld), -7.0, F32)
        want[:tw, col0:col0 + n] = tab[np.clip(idx, 0, cap - 1)].T
        np.testing.assert_array_equal(got, want, err_msg=f"tw {tw} n {n}")


@gpu
@pytest.mark.parametrize("size", [1, 3, (1 << 20) + 1])
def test_replay_draws_cross_the_counter_high_word(L, size):
    """imb_sample_indices kind 0 == philox.randint with the draw counter starting at 2^32 - 2: the third draw uses the
    counter's high word.  n not a multiple of 4."""
    from oracle import philox

    seed = 4242
    st = _state()
    st[L.ST_RING_N] = size
    st[L.ST_REPLAY_DRAW] = (1 << 32) - 2
    for k, n in enumerate((7, 4099, 1, 4098)):
        idx = th.empty(n, dtype=th.int64, device="cuda")
        L.sample_indices(0, idx, n, 0, seed, st)
        want = philox.randint(seed, philox.STREAM_REPLAY, (1 << 32) - 2 + k, n, size)
        np.testing.assert_array_equal(idx.cpu().numpy(), want, err_msg=f"draw {k}")
        assert want.max() < size
    assert int(st[L.ST_REPLAY_DRAW]) == (1 << 32) + 2


@gpu
@pytest.mark.parametrize("n_expert,B", [(96, 96), (97, 96), (191, 96), (10 ** 6 + 3, 250000)])
def test_expert_stream_epochs(L, n_expert, B):
    """imb_sample_indices kind 1 == endless Feistel permutations with drop_last, over at least three epochs."""
    from oracle import philox

    seed = 77
    st = _state()
    per_epoch = n_expert // B
    perms = {}
    for k in range(3 * per_epoch + 1):
        ep, pos = divmod(k, per_epoch)
        if ep not in perms:
            perms[ep] = philox.feistel_perm(seed, philox.STREAM_EXPERT, ep, n_expert)
        idx = th.empty(B, dtype=th.int64, device="cuda")
        L.sample_indices(1, idx, B, n_expert, seed, st)
        np.testing.assert_array_equal(idx.cpu().numpy(), perms[ep][pos * B:(pos + 1) * B], err_msg=f"batch {k}")
        nk = k + 1
        assert [int(st[L.ST_EXPERT_EPOCH]), int(st[L.ST_EXPERT_POS])] == [nk // per_epoch, (nk % per_epoch) * B]


@gpu
@pytest.mark.parametrize("mb", [45, 77])
def test_disc_sample_gather_twin(L, mb):
    """imb_disc_sample_gather with mb not a multiple of 32 == the NumPy twin: expert columns from the Feistel stream,
    generator columns from Philox randint over the ring's stored prefix, over updates that roll the expert epoch."""
    from oracle import philox

    rng = np.random.default_rng(mb)
    n_e, cap, tw, seed = 200, 300, 9, 31
    B = 2 * mb
    et = rng.standard_normal((n_e, tw)).astype(F32)
    rt = rng.standard_normal((cap, tw)).astype(F32)
    e_table, ring = th.tensor(et, device="cuda"), th.tensor(rt, device="cuda")
    st_e, st_g = _state(), _state()
    st_g[L.ST_RING_N] = 251
    st_g[L.ST_REPLAY_DRAW] = (1 << 32) - 1
    ld = 2 * mb + 3
    ep, pos = 0, 0
    for upd in range(5):
        perm = philox.feistel_perm(seed, philox.STREAM_EXPERT, ep, n_e)
        draws = philox.randint(seed, philox.STREAM_REPLAY, (1 << 32) - 1 + upd, B, 251)
        for start in range(0, B, mb):
            batch = th.full((tw + 1, ld), -3.0, device="cuda")
            L.disc_sample_gather(e_table, n_e, ring, cap, tw, mb, start, seed, st_e, st_g, batch, ld)
            want = np.full((tw + 1, ld), -3.0, F32)
            want[:tw, :mb] = et[perm[pos + start:pos + start + mb]].T
            want[:tw, mb:2 * mb] = rt[draws[start:start + mb]].T
            np.testing.assert_array_equal(batch.cpu().numpy(), want, err_msg=f"update {upd} start {start}")
        L.sample_advance2(B, n_e, st_e, st_g)
        pos += B
        if pos + B > n_e:
            ep, pos = ep + 1, 0
        assert [int(st_e[L.ST_EXPERT_EPOCH]), int(st_e[L.ST_EXPERT_POS])] == [ep, pos]
    assert int(st_g[L.ST_REPLAY_DRAW]) == (1 << 32) + 4
