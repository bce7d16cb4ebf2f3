"""The generator rollout (imb_rollout / imb_rollout_ensemble) at every shape it accepts, against a float64 step.

The reference is teacher-forced: the closed loop is not replayed.  Every env step (e, t) is recomputed in float64 from
the kernel's own inputs -- the observation recorded in rollout row (e, t), the pinned noise or its Philox twin
(oracle/philox.py) when the kernel draws on the device, and the same fp32 parameters and norm statistics:

  policy   feature RunningNorm, tanh or ReLU towers, value, Box mean and act = mean + exp(log_std) z (unclipped),
           Discrete inverse-CDF draw on u, log pi
  env      next_obs = tanh(A obs + B u + c), env reward w . next_obs - 0.1 |u|^2, u = clip(act) or one-hot(act)
  reward   on (obs, u, next_obs, done): GAIL softplus (mode 1) or raw (mode 2), every pass of a shaped net, each
           ensemble member's raw output
  also     gamma V(terminal obs) on done steps, V(last obs) and the last done flag, and imb_gae on the kernel's own
           columns against float64 GAE.

The next step's recorded observation is checked against the float64 next_obs (or, on done steps, against the reset
observation 0.1 normals(seed, ENV_RESET, env id, episode), within a few ulps for the device's logf / cosf / sinf).

Tolerances follow test_disc_shape_sweep.py: each output may deviate from its float64 value by C m(y), where m(y) is the
same float64 evaluation with every weight, input and bias replaced by its absolute value (activations Lipschitz 1).  C
is not a measured fit: on an H100 80GB HBM3 (132 SMs, 700 W power limit) the largest ratio |got - want| / m(y) over
every output of every case was MAX_SEEN_RATIO = 1.39e-6 (next_obs of the 1-obs case); C = 4x that = 5.6e-6.  A Discrete draw whose u lies within DRAW_TOL of a float64 CDF
boundary may take either action; its log pi must match the action taken.

The comparator is held to the float64 step itself on the CPU (anchor: oracle/ppo_port.ActorCriticPort,
oracle/synth_env and oracle/nets_port run in float64 agree with it), and must reject a rollout simulated with each of
these mistakes: one tower weight matrix off by 0.1 %, log_std off by 1e-3, a next_obs taken from the wrong step,
Phi(s') with gamma = 1 where the net has gamma = 0.9, softplus swapped for -logsigmoid(x), the reward computed on the
unclipped action.

Exact (bitwise) checks: flat and ring rows copy the rollout rows; the flatten order equals oracle/data_port's
BufferingPort + flatten_port over a stub VecEnv whose observations encode (env, step); ring positions equal
ReplayBufferPort's with a nonzero start, wrap-around and more rows than capacity; done flags; the state words after
imb_rollout_advance; two identical launches; a single-net launch against a 2-member ensemble of the same net; and the
envs shared by 32-, 64- and 128-row launches (tile_layer sums each element in one FMA chain, in the same order at every
tile).  The 8-row tile sums two accumulator chains (tile_layer8), so it is held to the tolerance only -- every case runs
it at 16 SMs - 5 envs.
"""
import zlib

import numpy as np
import pytest
import torch as th

from imitation_b200 import _desc, _lib

MAX_SEEN_RATIO = 1.39e-6  # next_obs of the 1-obs, 1-action case (tanh_fast's absolute error on a small m)
C = 4 * MAX_SEEN_RATIO
assert C <= 1e-4
DRAW_TOL = 1e-5         # |u - CDF boundary| below which a Discrete draw may go either way (fp32 CDF of <= 64 terms)
RESET_RTOL, RESET_ATOL = 4 * 2.0 ** -23, 1e-8
SEED = 23
GAMMA, LAM = float(np.float32(0.97)), float(np.float32(0.9))

# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
# E per tile size from the SM count (test_tile_bitexact.TILES): rows8 has a ragged tail (plain loads), rows32 and
# rows128 + 100 are multiples of 4 (bulk copies), rows64 = 128 SMs - 2 is ragged again
TILES = {"rows8": lambda s: 16 * s - 5, "rows32": lambda s: 32 * s, "rows64": lambda s: 128 * s - 2,
         "rows128": lambda s: 128 * s + 100}
ALL = tuple(TILES)
N32 = dict(hid_sizes=(32, 32), normalize_input=True)
AIRL = dict(hid_sizes=(32,), potential_hid_sizes=(32, 32), shaped=True, normalize_input=True, gamma=0.9,
            subtract_logp=True)


def _case(do, da, h, *, disc=False, act="tanh", pnorm=True, mode=0, net=None, members=0, T=3, H=2, t0=1,
          noise="pinned", tiles=("rows8",), off=5, ep=3, gstep=101, big_logits=False):
    return dict(do=do, da=da, h=h, disc=disc, act=act, pnorm=pnorm, mode=mode, net=net, members=members, T=T, H=H,
                t0=t0, noise=noise, tiles=tiles, off=off, ep=ep, gstep=gstep, big_logits=big_logits)


CASES = {
    # d_obs 1 .. 64 (32- and 64-wide env tile), Box d_act 1 .. 64 (Philox chunks of 4 and ragged ones)
    "o1_a1_h1": _case(1, 1, 1, noise="philox", T=3, H=1, t0=0),
    "o4_a5_h7_relu": _case(4, 5, 7, act="relu", pnorm=False, noise="philox", tiles=ALL),
    "hc_o17_a6_h32_gail": _case(17, 6, 32, mode=1, net=N32, noise="philox", tiles=ALL),
    "o31_a9_h20_raw": _case(31, 9, 20, mode=2, net=dict(hid_sizes=(16,), use_state=False, use_next_state=True,
                                                         use_done=True),
                            T=4, H=9, t0=5),
    "o32_a6_h33_relu": _case(32, 6, 33, act="relu", mode=1, net=dict(hid_sizes=(40, 40)), tiles=ALL),
    "o33_a8_h40": _case(33, 8, 40, pnorm=False, T=5, H=2, t0=0, tiles=ALL),
    "o56_a8_h63_mode0": _case(56, 8, 63, noise="philox", T=4, H=9, t0=7),
    "o64_a64_h64_mode0": _case(64, 64, 64, noise="philox", tiles=ALL),     # Do + Da = 128
    "o64_a1_h64_relu_det": _case(64, 1, 64, act="relu", noise="det", T=3, H=1, t0=0),
    "ant_o27_a8_h64_airl": _case(27, 8, 64, mode=2, net=AIRL, noise="philox", tiles=ALL),
    "o17_a6_h32_h0_gail_tails": _case(17, 6, 32, mode=1, net=dict(hid_sizes=()), big_logits=True),
    "o11_a3_h32_n64": _case(11, 3, 32, act="relu", mode=2, net=dict(hid_sizes=(64, 64)), T=5, H=2, t0=1),
    "o5_a2_h32_det_airl": _case(5, 2, 32, mode=2, net=dict(AIRL, hid_sizes=(64,)), noise="det"),
    # Discrete: 2, 18, 64 actions (one-hot reward inputs), pinned u, device Philox u, argmax
    "cartpole_o4_d2_h32": _case(4, 2, 32, disc=True, pnorm=False, mode=1, net=dict(hid_sizes=(64, 64),
                                                                                  normalize_input=True),
                                noise="philox", tiles=ALL),
    "o8_d18_h20_relu": _case(8, 18, 20, disc=True, act="relu", mode=2, net=N32, T=4, H=9, t0=2),
    "o12_d64_h64": _case(12, 64, 64, disc=True, noise="philox", T=5, H=2, t0=0),
    "o6_d5_h32_det": _case(6, 5, 32, disc=True, noise="det", mode=1, net=N32),
    # ensembles of 2, 3 and 16 members
    "ens2_o17_a6": _case(17, 6, 32, mode=2, members=2, net=N32, noise="philox", tiles=ALL),
    "ens3_o11_a3_airl": _case(11, 3, 32, act="relu", mode=2, members=3, net=AIRL, T=4, H=9, t0=3),
    "ens16_o17_a6_nonorm": _case(17, 6, 32, mode=2, members=16, net=dict(hid_sizes=(32, 32))),
    "ens3_d4": _case(6, 4, 32, disc=True, mode=2, members=3, net=dict(hid_sizes=(16, 16), normalize_input=True),
                     noise="philox"),
    # shapes whose preferred tile does not fit into shared memory (test_rollout_plan.FALLBACK), at the env counts where
    # they run a smaller tile than preferred
    "fb_hopper_airl64": _case(11, 3, 64, mode=2, net=dict(hid_sizes=(64, 64), shaped=True,
                                                          potential_hid_sizes=(64, 64), normalize_input=True,
                                                          gamma=0.9),
                              noise="philox", tiles=("rows8", "rows128")),
    "fb_hc_ens3_64x64": _case(17, 6, 64, mode=2, members=3, net=dict(hid_sizes=(64, 64), normalize_input=True),
                              noise="philox", tiles=("rows8", "rows128")),
    "fb_ant_airl64": _case(27, 8, 64, mode=2, net=dict(hid_sizes=(64, 64), shaped=True,
                                                       potential_hid_sizes=(64, 64), normalize_input=True, gamma=0.9),
                           noise="philox", tiles=("rows8", "rows64", "rows128")),
    "fb_ens16_32x32": _case(17, 6, 32, mode=2, members=16, net=N32, noise="philox", tiles=("rows8", "rows32")),
}
FALLBACK = [n for n in CASES if n.startswith("fb_")]
RUNS = [(n, t) for n, c in CASES.items() for t in c["tiles"]]


@pytest.fixture(scope="module")
def L():
    _lib.lib()
    return _lib


def _sms():
    return th.cuda.get_device_properties(0).multi_processor_count


def _rng(*key):
    return np.random.default_rng(zlib.crc32("/".join(map(str, key)).encode()))


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _uparams(rng, shapes, wscale=1.7):
    ps = []
    for _, s in shapes:
        scale = wscale / np.sqrt(s[1]) if len(s) == 2 else 0.5
        ps.append((rng.uniform(-1, 1, int(np.prod(s))) * scale).astype(np.float32))
    return np.concatenate(ps)


def _dd(c):
    """the reward net's descriptor (None for reward mode 0); d_act is the one-hot width for Discrete"""
    if c["mode"] == 0:
        return None
    return _desc.disc_desc(c["do"], c["da"], **c["net"])


def _inputs(name):
    """fp32 numpy inputs of a case: policy parameters + norm, reward-net parameters + norms per member"""
    c = CASES[name]
    rng = _rng("inputs", name)
    Do, Da = c["do"], c["da"]
    pd = _desc.policy_desc(Do, Da, c["disc"], c["h"], c["pnorm"])
    PP = _uparams(rng, _desc.policy_param_shapes(Do, Da, c["disc"], c["h"]))
    if not c["disc"]:
        PP[pd.off_log_std:pd.off_log_std + Da] = rng.uniform(-1.5, 0.5, Da)
    PN = (np.concatenate([rng.standard_normal(Do) * 0.1, rng.uniform(0.5, 1.5, Do)]).astype(np.float32) if c["pnorm"]
          else np.zeros(2, np.float32))
    dd, DP, DN = _dd(c), [], []
    if dd is not None:
        hid = c["net"].get("hid_sizes", (32, 32))
        pot = c["net"].get("potential_hid_sizes", (32, 32))
        shapes = _desc.mlp_param_shapes(dd.base.din, hid) + (_desc.mlp_param_shapes(Do, pot) if dd.shaped else [])
        for m in range(max(1, c["members"])):
            P = _uparams(rng, shapes, wscale=60.0 if c["big_logits"] else 1.7)
            assert P.size == dd.n_params
            DP.append(P)
            nets = [dd.base.din] + ([Do] if dd.shaped else [])
            DN.append(np.concatenate([np.concatenate([rng.standard_normal(k) * 0.3, rng.uniform(0.5, 3.0, k)])
                                      for k in nets]).astype(np.float32) if dd.base.has_norm else None)
    return pd, PP, PN, dd, DP, DN


def _noise(c, E, rng):
    T, Da = c["T"], c["da"]
    if c["noise"] != "pinned":
        return None
    if c["disc"]:
        return rng.random((T, E)).astype(np.float32)
    return rng.standard_normal((T, E, Da)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# float64 step (vectorised over envs)
# ---------------------------------------------------------------------------------------------------------------------
def _t(x):
    return th.as_tensor(np.asarray(x, np.float64))


def _lin(x, mx, W, b):
    """x @ W.T + b and its magnitude |x| @ |W|.T + |b|"""
    return x @ W.T + b, mx @ W.abs().T + b.abs()


def _policy64(pd, act, PP, PN, obs, pert=None):
    """float64 policy on obs [N, Do]: pi latent, mean / logits (+ magnitudes), value (+ magnitude)"""
    P = _t(PP)
    if pert is not None:
        P = pert(P.clone())
    Do, Da, h = pd.d_obs, pd.d_act, pd.hidden
    g = lambda off, *s: P[off:off + int(np.prod(s))].reshape(*s)
    x = obs
    mx = obs.abs()
    if pd.has_norm:
        mean, var = _t(PN[:Do]), _t(PN[Do:2 * Do])
        istd = 1.0 / th.sqrt(var + float(np.float32(pd.norm_eps)))
        x, mx = (obs - mean) * istd, (obs.abs() + mean.abs()) * istd
    f = th.tanh if act == _lib.ACT_TANH else th.relu

    def tower(w1, b1, w2, b2):
        z, m = _lin(x, mx, g(w1, h, Do), g(b1, h))
        z, m = _lin(f(z), m, g(w2, h, h), g(b2, h))
        return f(z), m

    hp, mp = tower(pd.off_pi_w1, pd.off_pi_b1, pd.off_pi_w2, pd.off_pi_b2)
    hv, mv = tower(pd.off_vf_w1, pd.off_vf_b1, pd.off_vf_w2, pd.off_vf_b2)
    out, mout = _lin(hp, mp, g(pd.off_act_w, Da, h), g(pd.off_act_b, Da))
    v, mval = _lin(hv, mv, g(pd.off_val_w, 1, h), g(pd.off_val_b, 1))
    log_std = None if pd.discrete else g(pd.off_log_std, Da)
    return out, mout, v[:, 0], mval[:, 0], log_std


def _mlp64(x, mx, P, off, din, hid, norm, eps):
    if norm is not None:
        mean, var = _t(norm[:din]), _t(norm[din:2 * din])
        istd = 1.0 / th.sqrt(var + float(np.float32(eps)))
        x, mx = (x - mean) * istd, (x.abs() + mean.abs()) * istd
    for n_out, prev in [(hh, p) for hh, p in zip(hid, (din,) + tuple(hid))]:
        W = P[off:off + n_out * prev].reshape(n_out, prev)
        off += n_out * prev
        b = P[off:off + n_out]
        off += n_out
        x, mx = _lin(x, mx, W, b)
        x = th.relu(x)
    prev = hid[-1] if hid else din
    W = P[off:off + prev].reshape(1, prev)
    b = P[off + prev:off + prev + 1]
    x, mx = _lin(x, mx, W, b)
    return x[:, 0], mx[:, 0]


def _hid(m):
    return tuple(h for h, k in zip((m.h1, m.h2), range(m.n_hidden)))


def _reward64(dd, P, NS, obs, u, nobs, done, gamma=None):
    """raw reward-net output (+ magnitude) on float64 inputs, in eval mode (subtract_logp ignored)"""
    P = _t(P)
    parts = ([obs] if dd.use_state else []) + ([u] if dd.use_action else []) + \
            ([nobs] if dd.use_next_state else []) + ([done[:, None]] if dd.use_done else [])
    x = th.cat(parts, 1)
    bn = NS[dd.base.norm_off:dd.base.norm_off + 2 * dd.base.din] if dd.base.has_norm else None
    r, mr = _mlp64(x, x.abs(), P, dd.base.param_off, dd.base.din, _hid(dd.base), bn, dd.base.norm_eps)
    if dd.shaped:
        pm = dd.potential
        pn = NS[pm.norm_off:pm.norm_off + 2 * pm.din] if pm.has_norm else None
        g = float(np.float32(dd.gamma)) if gamma is None else gamma
        p1, m1 = _mlp64(nobs, nobs.abs(), P, pm.param_off, pm.din, _hid(pm), pn, pm.norm_eps)
        p0, m0 = _mlp64(obs, obs.abs(), P, pm.param_off, pm.din, _hid(pm), pn, pm.norm_eps)
        r, mr = r + g * (1 - done) * p1 - p0, mr + g * (1 - done) * m1 + m0
    return r, mr


def _softplus64(x):
    return th.clamp(x, min=0) + th.log1p(th.exp(-x.abs()))


def _env64(EP, Do, Da, obs, u):
    A, B = _t(EP[:Do * Do]).reshape(Do, Do), _t(EP[Do * Do:Do * Do + Do * Da]).reshape(Do, Da)
    c, w = _t(EP[Do * Do + Do * Da:Do * Do + Do * Da + Do]), _t(EP[Do * Do + Do * Da + Do:])
    pre = obs @ A.T + u @ B.T + c
    mpre = obs.abs() @ A.abs().T + u.abs() @ B.abs().T + c.abs()
    nobs = th.tanh(pre)
    return nobs, mpre, w, (w.abs() * mpre).sum(1)


# ---------------------------------------------------------------------------------------------------------------------
# one launch: run it, then hold every output to the float64 step
# ---------------------------------------------------------------------------------------------------------------------
def _z_and_u(c, E, noise, gstep0):
    """[T][E][Da] normals (Box) / [T][E] uniforms (Discrete) the launch uses: pinned, or the Philox twin"""
    from oracle import philox

    T = c["T"]
    if noise is not None:
        return noise.astype(np.float64)
    egid = (np.arange(E, dtype=np.int64) + c["off"]).astype(np.uint32)
    out = []
    for t in range(T):
        if c["disc"]:
            k0, k1 = philox.key_for(SEED, philox.STREAM_ACT_NOISE)
            x = philox.philox4x32(egid, np.uint32(gstep0 + t), np.uint32(0), np.uint32(0), k0, k1)[0]
            out.append(philox.u01(x))
        else:
            out.append(philox.normals(SEED, philox.STREAM_ACT_NOISE, egid, np.uint32(gstep0 + t), c["da"]))
    return np.stack(out).astype(np.float64)


def _ratio(got, want, mag, what, seen, extra=0.0):
    """max |got - want| / (C m) over the elements; records the largest |got - want| / m under `what`"""
    got, want, mag = (np.asarray(a, np.float64) for a in (got, want, mag))
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    err = np.abs(got - want) - extra
    r = np.where(mag > 0, np.maximum(err, 0) / np.where(mag > 0, mag, 1), np.where(err > 0, np.inf, 0))
    seen[what] = max(seen.get(what, 0.0), float(r.max(initial=0.0)))
    return float(r.max(initial=0.0)) / C


def _assert_within(got, want, mag, what, seen, extra=0.0):
    q = _ratio(got, want, mag, what, seen, extra)
    if q > 1:
        got, want, mag = (np.asarray(a, np.float64) for a in (got, want, mag))
        i = np.unravel_index(np.argmax(np.abs(got - want) - C * mag), got.shape)
        pytest.fail(f"{what}: {q:.3g} x the tolerance at {i}: got {got[i]!r}, float64 {want[i]!r}, m {mag[i]!r}")


def check_launch(c, pd, act, PP, PN, dd, DP, DN, EP, E, st0, obs0, noise, out, seen, flags=0):
    """Teacher-forced float64 check of one launch's outputs `out` (numpy: tbl [E][T][rw], flat [E*T][tw], aux, obs_end
    [Do][E], raw [M][T][E] for an ensemble).  Raises AssertionError (pytest's Failed) on the first output out of
    tolerance; `seen` collects the largest ratio of each output."""
    Do, Da, T, H = c["do"], c["da"], c["T"], c["H"]
    t0, ep0, g0 = int(st0[_lib.ST_EP_STEP]), int(st0[_lib.ST_EPISODE]), int(st0[_lib.ST_GLOBAL_STEP])
    det = bool(flags & _lib.IMB_RF_DETERMINISTIC)
    tbl, flat, aux = out["tbl"], out["flat"], out["aux"]
    da_store = 1 if c["disc"] else Da
    cl, cv, cr = Do + da_store, Do + da_store + 1, Do + da_store + 2
    tw = 2 * Do + Da + 1
    fmap = _flat_map(E, T, t0, H)  # flat row -> (e, t)
    finv = np.empty((E, T), np.int64)
    finv[fmap[:, 0], fmap[:, 1]] = np.arange(E * T)
    zu = None if det else _z_and_u(c, E, noise, g0)
    episode = ep0
    assert np.array_equal(tbl[:, 0, :Do], obs0.T), "obs of step 0 = the env state the launch started from"
    for t in range(T):
        obs = _t(tbl[:, t, :Do])
        out_, mout, v, mv, log_std = _policy64(pd, act, PP, PN, obs, )
        _assert_within(tbl[:, t, cv], v, mv, "value", seen)
        done = ((t0 + t + 1) % H) == 0
        if not c["disc"]:
            a_rec = tbl[:, t, Do:Do + Da].astype(np.float64)
            ls = log_std
            sd = th.exp(ls)
            z = th.zeros(E, Da, dtype=th.float64) if det else _t(zu[t])
            want = out_ + sd * z
            _assert_within(a_rec, want, mout + sd * z.abs(), "action", seen)
            diff = _t(a_rec) - out_
            lp = (-(diff * diff) / (2 * sd * sd) - ls - 0.9189385332046727).sum(1)
            mlp = (diff.abs() * mout / (sd * sd) + diff * diff / (2 * sd * sd) + ls.abs() + 0.92).sum(1)
            _assert_within(tbl[:, t, cl], lp, mlp, "logp", seen)
            u = th.clamp(_t(a_rec), -1, 1)
        else:
            k = tbl[:, t, Do].astype(np.int64)
            assert np.array_equal(tbl[:, t, Do], k.astype(np.float32)) and ((k >= 0) & (k < Da)).all()
            lse = th.logsumexp(out_, 1)
            if det:
                top = out_.max(1).values
                ok = (out_[th.arange(E), th.as_tensor(k)] >= top - C * mout.max(1).values).numpy()
            else:
                cdf = th.cumsum(th.softmax(out_, 1), 1).numpy()
                lo = np.where(k > 0, cdf[np.arange(E), np.maximum(k - 1, 0)], 0.0)
                hi = np.where(k < Da - 1, cdf[np.arange(E), k], np.inf)
                u_ = zu[t]
                ok = (u_ >= lo - DRAW_TOL) & (u_ < hi + DRAW_TOL)
            assert ok.all(), f"step {t}: Discrete action of env {np.argmin(ok)} is not the draw's"
            lp = out_[th.arange(E), th.as_tensor(k)] - lse
            mlp = mout[th.arange(E), th.as_tensor(k)] + mout.max(1).values + 1.0
            _assert_within(tbl[:, t, cl], lp, mlp, "logp", seen)
            u = th.nn.functional.one_hot(th.as_tensor(k), Da).double()
        # env step, from the recorded obs and the control the kernel applied
        nobs, mn, w, mre = _env64(EP, Do, Da, obs, u)
        rows = flat[finv[:, t]]
        nob_k = rows[:, Do + Da:2 * Do + Da]  # the next_obs the kernel fed to its reward net (terminal obs when done)
        _assert_within(nob_k, nobs, mn, "next_obs", seen)
        renv = _t(nob_k) @ w - (0.0 if c["disc"] else 0.1 * (u * u).sum(1))
        mre = _t(nob_k).abs() @ w.abs() + (0.0 if c["disc"] else 0.1 * (u * u).sum(1))
        _assert_within(aux[2 * E + E * T + np.arange(E) * T + t], renv, mre, "env_reward", seen)
        # the reward the relabel wrapper sees
        d = th.full((E,), float(done), dtype=th.float64)
        if c["mode"] == 0:
            _assert_within(tbl[:, t, cr], renv, mre, "reward", seen)
        else:
            for m in range(max(1, c["members"])):
                r, mr = _reward64(dd, DP[m], DN[m], obs, u, _t(nob_k), d)
                if c["members"]:
                    _assert_within(out["raw"][m, t], r, mr, "member_raw", seen)
                elif c["mode"] == 1:
                    sp = _softplus64(r)
                    _assert_within(tbl[:, t, cr], sp, mr + sp.abs(), "reward", seen)
                else:
                    _assert_within(tbl[:, t, cr], r, mr, "reward", seen)
        # bootstrap on done steps
        boot = aux[2 * E + np.arange(E) * T + t]
        if done:
            _, _, vt, mvt, _ = _policy64(pd, act, PP, PN, _t(nob_k))
            _assert_within(boot, GAMMA * vt, GAMMA * mvt, "bootstrap", seen)
            episode += 1
        else:
            assert (boot == 0).all(), f"step {t}: bootstrap term on a step that is not done"
        # the next observation: next_obs, or the reset observation on done
        nxt = tbl[:, t + 1, :Do] if t + 1 < T else out["obs_end"].T
        if done:
            from oracle import philox

            egid = (np.arange(E, dtype=np.int64) + c["off"]).astype(np.uint32)
            want = np.float32(0.1) * philox.normals(SEED, philox.STREAM_ENV_RESET, egid, np.uint32(episode), Do)
            np.testing.assert_allclose(nxt, want, rtol=RESET_RTOL, atol=RESET_ATOL, err_msg=f"reset obs, step {t}")
        else:
            assert np.array_equal(nxt, nob_k), f"step {t}: the next step's obs is not the next_obs of this one"
    # tail: V(last obs), last done
    _, _, vl, mvl, _ = _policy64(pd, act, PP, PN, _t(out["obs_end"].T))
    _assert_within(aux[:E], vl, mvl, "value_last", seen)
    assert (aux[E:2 * E] == float(((t0 + T) % H) == 0)).all()
    return episode


def _gae64(c, E, tbl, aux, t0, cv):
    """float64 GAE from the kernel's own value / reward / bootstrap columns (+ magnitudes)"""
    T, H = c["T"], c["H"]
    v = _t(tbl[:, :, cv])
    r = _t(tbl[:, :, cv + 1]) + _t(aux[2 * E:2 * E + E * T].reshape(E, T))
    mr = _t(tbl[:, :, cv + 1]).abs() + _t(aux[2 * E:2 * E + E * T].reshape(E, T)).abs()
    adv, madv = th.zeros(E, T, dtype=th.float64), th.zeros(E, T, dtype=th.float64)
    last, mlast = th.zeros(E, dtype=th.float64), th.zeros(E, dtype=th.float64)
    nv, nn = _t(aux[:E]), 1.0 - _t(aux[E:2 * E])
    for t in range(T - 1, -1, -1):
        delta = r[:, t] + GAMMA * nv * nn - v[:, t]
        mdelta = mr[:, t] + GAMMA * nv.abs() * nn + v[:, t].abs()
        last, mlast = delta + GAMMA * LAM * nn * last, mdelta + GAMMA * LAM * nn * mlast
        adv[:, t], madv[:, t] = last, mlast
        nv = v[:, t]
        nn = th.full((E,), 0.0 if (t > 0 and (t0 + t) % H == 0) else 1.0, dtype=th.float64)
    return r, mr, adv, madv


# ---------------------------------------------------------------------------------------------------------------------
# flatten order and ring (exact)
# ---------------------------------------------------------------------------------------------------------------------
class _TagEnv:
    """stub VecEnv whose observations are (env, local step) and whose episodes end when (t0 + step) % H == 0"""

    def __init__(self, E, t0, H):
        self.num_envs, self.t0, self.H, self.k = E, t0, H, 0
        self.observation_space = self.action_space = None

    def reset(self):
        self.k = 0
        return np.stack([np.arange(self.num_envs), np.zeros(self.num_envs)], 1)

    def step_async(self, actions):
        pass

    def step_wait(self):
        self.k += 1
        E = self.num_envs
        obs = np.stack([np.arange(E), np.full(E, self.k)], 1).astype(np.float64)
        done = (self.t0 + self.k) % self.H == 0
        infos = [{} for _ in range(E)]
        if done:  # (the reset observation carries the same tag: it is the obs of that step's rollout row)
            for i in range(E):
                infos[i]["terminal_observation"] = obs[i].copy()
        return obs, np.zeros(E), np.full(E, done), infos


_FLAT_MAPS = {}


def _flat_map(E, T, t0, H):
    """[E*T][2]: the (env, step) of each transition in the order BufferingWrapper.pop_trajectories +
    flatten_trajectories give them (oracle/data_port)"""
    from oracle import data_port

    key = (E, T, t0, H)
    if key not in _FLAT_MAPS:
        buf = data_port.BufferingPort(_TagEnv(E, t0, H))
        buf.reset()
        for _ in range(T):
            buf.step(np.zeros(E))
        trajs, _ = buf.pop_trajectories()
        fl = data_port.flatten_port(trajs)
        _FLAT_MAPS[key] = fl["obs"].astype(np.int64)
        assert np.array_equal(fl["next_obs"][:, 1], fl["obs"][:, 1] + 1)
    return _FLAT_MAPS[key]


def check_rows(c, E, st0, out):
    """flat rows copy the rollout rows, in the reference's order; done column"""
    Do, Da, T, H = c["do"], c["da"], c["T"], c["H"]
    t0 = int(st0[_lib.ST_EP_STEP])
    tbl, flat = out["tbl"], out["flat"]
    fm = _flat_map(E, T, t0, H)
    e, t = fm[:, 0], fm[:, 1]
    assert np.array_equal(flat[:, :Do], tbl[e, t, :Do]), "flat obs"
    if c["disc"]:
        assert np.array_equal(flat[:, Do:Do + Da], np.eye(Da, dtype=np.float32)[tbl[e, t, Do].astype(np.int64)])
    else:
        assert np.array_equal(flat[:, Do:Do + Da], np.clip(tbl[e, t, Do:Do + Da], -1, 1)), "flat acts = clipped acts"
    done = ((t0 + t + 1) % H) == 0
    assert np.array_equal(flat[:, -1], done.astype(np.float32)), "done column"
    nxt = np.where((t + 1 < T)[:, None], tbl[e, np.minimum(t + 1, T - 1), :Do], out["obs_end"].T[e])
    assert np.array_equal(flat[~done, Do + Da:2 * Do + Da], nxt[~done]), "flat next_obs"


def ring_port(c, cap, idx0, n0):
    from oracle import data_port

    p = data_port.ReplayBufferPort(cap, (c["do"],), (c["da"],))
    p._buffer._idx, p._buffer._n_data = idx0, n0
    return p


def check_ring(c, port, flat, ring, st):
    Do, Da = c["do"], c["da"]
    n = flat.shape[0]
    port.store(dict(obs=flat[:, :Do], acts=flat[:, Do:Do + Da], next_obs=flat[:, Do + Da:2 * Do + Da],
                    dones=flat[:, -1] > 0.5, infos=np.empty(n, object)))
    a = port._buffer._arrays
    want = np.concatenate([a["obs"], a["acts"], a["next_obs"], a["dones"][:, None].astype(np.float32)], 1)
    assert np.array_equal(ring, want), "ring rows / positions"
    assert [int(st[_lib.ST_RING_IDX]), int(st[_lib.ST_RING_N])] == [port._buffer._idx, port._buffer._n_data]


# ---------------------------------------------------------------------------------------------------------------------
# GPU launches
# ---------------------------------------------------------------------------------------------------------------------
def _hp(L):
    return L.PpoHparams(gamma=GAMMA, gae_lambda=LAM, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                        lr=3e-4, adam_eps=1e-5, n_epochs=1, batch_size=32, normalize_advantage=1)


def _launch(L, c, pd, act, PP, PN, dd, DP, DN, EP, E, st, obs, noise, ring, cap, flags=0, members=None):
    """one imb_rollout / imb_rollout_ensemble launch on device tensors; returns its outputs as numpy"""
    Do, Da, T = c["do"], c["da"], c["T"]
    rw, tw = L.rollout_row_width(pd), _desc.table_width(Do, Da)
    tbl = th.full((E * T, rw), float("nan"), device="cuda")
    flat = th.full((E * T, tw), float("nan"), device="cuda")
    aux = th.full((2 * E + 2 * E * T,), float("nan"), device="cuda")
    nz = None if noise is None else th.from_numpy(np.ascontiguousarray(noise)).cuda()
    env = L.EnvDesc(d_obs=Do, d_act=Da, discrete=int(c["disc"]), horizon=c["H"], seed=SEED, env_id_offset=c["off"])
    PPg, PNg = th.from_numpy(PP).cuda(), th.from_numpy(PN).cuda()
    out = {}
    M = len(DP) if members is None else members
    if c["members"] and M >= 2:
        raw = th.full((M * T * E,), float("nan"), device="cuda")
        DPg = [th.from_numpy(p).cuda() for p in DP[:M]]
        DNg = [None if n is None else th.from_numpy(n).cuda() for n in DN[:M]]
        L.rollout_ensemble(env, EP, obs, pd, PPg, PNg, dd, L.rollout_members(DPg, DNg, raw), _hp(L), E, T, tbl, ring,
                           cap, flat, aux, nz, st, flags=flags, act=act)
        out["raw"] = raw
    else:
        DPg = th.from_numpy(DP[0]).cuda() if dd is not None else None
        DNg = th.from_numpy(DN[0]).cuda() if dd is not None and DN[0] is not None else None
        L.rollout(env, EP, obs, pd, PPg, PNg, dd, DPg, DNg, c["mode"], _hp(L), E, T, tbl, ring, cap, flat, aux, nz,
                  st, flags=flags, act=act)
    gae = tbl.clone()
    L.gae(gae, rw, Do + (1 if c["disc"] else Da) + 1, E, T, aux, GAMMA, LAM, st, c["H"])
    th.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    if "raw" in res:
        res["raw"] = res["raw"].reshape(M, T, E)
    res.update(tbl=tbl.cpu().numpy().reshape(E, T, rw), flat=flat.cpu().numpy(), aux=aux.cpu().numpy(),
               obs_end=obs.cpu().numpy(), gae=gae.cpu().numpy().reshape(E, T, rw))
    if ring is not None:
        res["ring"] = ring.cpu().numpy()
    return res


def _setup(L, name, E):
    c = CASES[name]
    pd, PP, PN, dd, DP, DN = _inputs(name)
    act = L.ACT_RELU if c["act"] == "relu" else L.ACT_TANH
    EP = th.from_numpy(_desc.synth_env_params(c["do"], c["da"], SEED)).cuda()
    rng = _rng("state", name, E)
    obs = th.from_numpy(rng.uniform(-0.9, 0.9, (c["do"], E)).astype(np.float32)).cuda()
    st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
    st[L.ST_EP_STEP], st[L.ST_EPISODE], st[L.ST_GLOBAL_STEP] = c["t0"], c["ep"], c["gstep"]
    return c, pd, act, PP, PN, dd, DP, DN, EP, rng, obs, st


SEEN = {}


@pytest.mark.gpu
@pytest.mark.parametrize("name,tile", RUNS, ids=[f"{n}-{t}" for n, t in RUNS])
def test_rollout_matches_float64(L, name, tile):
    """two consecutive launches (the second from the advanced state, so its t0 differs), each teacher-forced against
    the float64 step; flat order, ring, GAE and the state words after each"""
    E = TILES[tile](_sms())
    c, pd, act, PP, PN, dd, DP, DN, EP, rng, obs, st = _setup(L, name, E)
    flags = L.IMB_RF_DETERMINISTIC if c["noise"] == "det" else 0
    T, H, Do = c["T"], c["H"], c["do"]
    # ring: more rows than capacity (skip + wrap) for half the cases, wrap without skip for the others
    big = zlib.crc32(name.encode()) % 2 == 0
    cap, idx0 = (E * T - 7, 5) if big else (E * T + 3, E * T - 4)
    st[L.ST_RING_IDX], st[L.ST_RING_N] = idx0, min(idx0 + 2, cap)
    ring = th.zeros(cap, _desc.table_width(Do, c["da"]), device="cuda")
    port = ring_port(c, cap, idx0, min(idx0 + 2, cap))
    seen = {}
    for launch in range(2):
        st0 = st.cpu().numpy()
        obs0 = obs.cpu().numpy()
        noise = _noise(c, E, rng)
        out = _launch(L, c, pd, act, PP, PN, dd, DP, DN, EP, E, st, obs, noise, ring, cap, flags)
        check_launch(c, pd, act, PP, PN, dd, DP, DN, EP.cpu().numpy(), E, st0, obs0, noise, out, seen, flags)
        check_rows(c, E, st0, out)
        if not c["members"]:  # (an ensemble's reward column is written by imb_ensemble_relabel)
            da_store = 1 if c["disc"] else c["da"]
            cv = Do + da_store + 1
            r, mr, adv, madv = _gae64(c, E, out["tbl"], out["aux"], int(st0[L.ST_EP_STEP]), cv)
            g = out["gae"]
            _assert_within(g[:, :, cv + 1], r, mr, "gae_reward", seen)
            _assert_within(g[:, :, cv + 2], adv, madv, "advantage", seen)
            _assert_within(g[:, :, cv + 3], adv + _t(out["tbl"][:, :, cv]), madv + _t(out["tbl"][:, :, cv]).abs(),
                           "return", seen)
        L.rollout_advance(st, E, T, H, cap)
        th.cuda.synchronize()
        s = st.cpu().numpy()
        t0 = int(st0[L.ST_EP_STEP])
        assert s[L.ST_EP_STEP] == (t0 + T) % H and s[L.ST_EPISODE] == st0[L.ST_EPISODE] + (t0 + T) // H
        assert s[L.ST_GLOBAL_STEP] == st0[L.ST_GLOBAL_STEP] + T
        check_ring(c, port, out["flat"], out["ring"], s)
    for k, v in seen.items():
        SEEN[k] = max(SEEN.get(k, 0.0), v)
    print(f"\n{name} {tile} E={E}: largest |got - want| / m: " + ", ".join(f"{k} {v:.3g}" for k, v in seen.items()))


def test_sweep_covers_every_tile():
    """rollout_plan names all four tiles over the sweep's launches (132 SMs), and the fallback cases run a smaller tile
    than the one their env count prefers"""
    tiles, fallbacks = set(), 0
    for name, tile in RUNS:
        c = CASES[name]
        pd, _, _, dd, _, _ = _inputs(name)
        E = TILES[tile](132)
        got = _lib.rollout_plan(pd, dd, max(1, c["members"]), E, 132)
        pref = 8 if E <= 16 * 132 else 32 if E <= 32 * 132 else 64 if E <= 128 * 132 else 128
        tiles.add(got)
        fallbacks += got < pref
        if name in FALLBACK and tile != "rows8":
            assert got < pref, (name, tile, got, pref)
    assert tiles == {8, 32, 64, 128} and fallbacks >= 4, (tiles, fallbacks)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hc_o17_a6_h32_gail", "cartpole_o4_d2_h32", "ens2_o17_a6"])
def test_tiles_and_repeats_give_identical_bits(L, name):
    """the envs shared by 32-, 64- and 128-row launches get the same bits (noise built for the largest E and sliced),
    and two identical launches give identical bits"""
    sms = _sms()
    Es = [TILES[k](sms) for k in ("rows32", "rows64", "rows128")]
    Emax = Es[-1]
    c, pd, act, PP, PN, dd, DP, DN, EP, rng, obs_big, st = _setup(L, name, Emax)
    noise = _noise(c, Emax, rng)
    n = Es[0]
    res = []
    for E in Es + [Es[0]]:
        obs = obs_big[:, :E].clone()  # (the launch advances its env state in place)
        nz = None if noise is None else np.ascontiguousarray(noise[:, :E])
        o = _launch(L, c, pd, act, PP, PN, dd, DP, DN, EP, E, st.clone(), obs, nz, None, 0)
        T = c["T"]
        aux = o["aux"]
        res.append(dict(tbl=o["tbl"][:n], obs_end=o["obs_end"][:, :n], vlast=aux[:n], done=aux[E:E + n],
                        boot=aux[2 * E:2 * E + n * T], renv=aux[2 * E + E * T:2 * E + E * T + n * T],
                        raw=o["raw"][:, :, :n] if "raw" in o else np.zeros(1)))
    for r, E in zip(res[1:], Es[1:] + [Es[0]]):
        for k in r:
            assert r[k].tobytes() == res[0][k].tobytes(), f"{k}: {E} envs differ from {n} envs"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ens2_o17_a6", "ens3_d4"])
def test_single_net_and_ensemble_agree(L, name):
    """imb_rollout with member 0's net (mode 2) and imb_rollout_ensemble give the same policy, env, flat and ring
    outputs, and member 0's raw output is the single net's reward column, bit for bit"""
    E = TILES["rows8"](_sms())
    c, pd, act, PP, PN, dd, DP, DN, EP, rng, obs, st = _setup(L, name, E)
    noise = _noise(c, E, rng)
    cap = E * c["T"] - 7
    outs = []
    for members in (1, len(DP)):
        ring = th.zeros(cap, _desc.table_width(c["do"], c["da"]), device="cuda")
        s = st.clone()
        s[L.ST_RING_IDX] = 5
        outs.append(_launch(L, c, pd, act, PP, PN, dd, DP, DN, EP, E, s, obs.clone(), noise, ring, cap,
                            members=members))
    one, ens = outs
    Do = c["do"]
    cr = Do + (1 if c["disc"] else c["da"]) + 2
    for k in ("flat", "ring", "obs_end", "aux"):
        assert one[k].tobytes() == ens[k].tobytes(), k
    assert one["tbl"][:, :, :cr].tobytes() == ens["tbl"][:, :, :cr].tobytes()
    assert np.array_equal(one["tbl"][:, :, cr], ens["raw"][0].T)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the float64 step against the SB3 / reference restatements, and the comparator's sensitivity
# ---------------------------------------------------------------------------------------------------------------------
def _simulate(name, E, sim=None, seed=0):
    """A rollout produced on the CPU by the float64 step (rounded to fp32 where the kernel stores), closed loop, with
    `sim`'s replacements -- the comparator's inputs for the sensitivity test.  Returns check_launch's arguments and flags."""
    from oracle import philox

    sim = sim or {}
    c = CASES[name]
    pd, PP, PN, dd, DP, DN = _inputs(name)
    act = _lib.ACT_RELU if c["act"] == "relu" else _lib.ACT_TANH
    Do, Da, T, H = c["do"], c["da"], c["T"], c["H"]
    EP = _desc.synth_env_params(Do, Da, SEED)
    rng = np.random.default_rng(seed)
    obs0 = rng.uniform(-0.9, 0.9, (Do, E)).astype(np.float32)
    st0 = np.zeros(_lib.ST_WORDS, np.int64)
    st0[_lib.ST_EP_STEP], st0[_lib.ST_EPISODE], st0[_lib.ST_GLOBAL_STEP] = c["t0"], c["ep"], c["gstep"]
    noise = _noise(c, E, rng)
    zu = _z_and_u(c, E, noise, c["gstep"])
    if c["noise"] == "det":
        zu = np.zeros_like(zu)
    t0, episode = c["t0"], c["ep"]
    rw, tw = _lib.rollout_row_width(pd), 2 * Do + Da + 1
    da_store = 1 if c["disc"] else Da
    tbl = np.zeros((E, T, rw), np.float32)
    aux = np.zeros(2 * E + 2 * E * T, np.float32)
    fm = _flat_map(E, T, t0, H)
    finv = np.empty((E, T), np.int64)
    finv[fm[:, 0], fm[:, 1]] = np.arange(E * T)
    flat = np.zeros((E * T, tw), np.float32)
    obs = obs0.T.copy()
    gfix = sim.get("potential_gamma")
    for t in range(T):
        ob = obs if "wrong_step" not in sim or t != 1 else tbl[:, 0, :Do]
        tbl[:, t, :Do] = obs
        o, _, v, _, ls = _policy64(pd, act, PP, PN, _t(obs), pert=sim.get("pert"))
        tbl[:, t, Do + da_store + 1] = v.numpy()
        if not c["disc"]:
            ls = sim["log_std"](ls) if "log_std" in sim else ls
            a = (o + th.exp(ls) * _t(zu[t])).numpy().astype(np.float32)
            tbl[:, t, Do:Do + Da] = a
            diff = _t(a) - o
            tbl[:, t, Do + da_store] = (-(diff * diff) / (2 * th.exp(2 * ls)) - ls - 0.9189385332046727).sum(1).numpy()
            u = _t(a) if sim.get("unclipped") else th.clamp(_t(a), -1, 1)
        else:
            cdf = th.cumsum(th.softmax(o, 1), 1).numpy()
            k = np.minimum((zu[t][:, None] >= cdf).sum(1), Da - 1)
            tbl[:, t, Do] = k
            tbl[:, t, Do + da_store] = (o[th.arange(E), th.as_tensor(k)] - th.logsumexp(o, 1)).numpy()
            u = th.nn.functional.one_hot(th.as_tensor(k), Da).double()
        nobs, _, w, _ = _env64(EP, Do, Da, _t(ob), u)
        nobs32 = nobs.numpy().astype(np.float32)
        done = ((t0 + t + 1) % H) == 0
        renv = _t(nobs32) @ w - (0.0 if c["disc"] else 0.1 * (u * u).sum(1))
        aux[2 * E + E * T + np.arange(E) * T + t] = renv.numpy()
        d = th.full((E,), float(done), dtype=th.float64)
        if c["mode"] == 0:
            rew = renv
        else:
            r, _ = _reward64(dd, DP[0], DN[0], _t(obs), u, _t(nobs32), d, gamma=gfix)
            sp = (lambda x: -th.nn.functional.logsigmoid(x)) if sim.get("logsigmoid") else _softplus64
            rew = sp(r) if c["mode"] == 1 else r
        tbl[:, t, Do + da_store + 2] = rew.numpy()
        rows = np.concatenate([obs, u.numpy().astype(np.float32), nobs32, np.full((E, 1), float(done), np.float32)], 1)
        flat[finv[:, t]] = rows
        if done:
            _, _, vt, _, _ = _policy64(pd, act, PP, PN, _t(nobs32))
            aux[2 * E + np.arange(E) * T + t] = (GAMMA * vt).numpy()
            episode += 1
            egid = (np.arange(E, dtype=np.int64) + c["off"]).astype(np.uint32)
            obs = np.float32(0.1) * philox.normals(SEED, philox.STREAM_ENV_RESET, egid, np.uint32(episode), Do)
        else:
            obs = nobs32
    _, _, vl, _, _ = _policy64(pd, act, PP, PN, _t(obs))
    aux[:E] = vl.numpy()
    aux[E:2 * E] = float(((t0 + T) % H) == 0)
    out = dict(tbl=tbl, flat=flat, aux=aux, obs_end=obs.T.copy())
    return (c, pd, act, PP, PN, dd, DP, DN, EP, E, st0, obs0, noise, out), (
        _lib.IMB_RF_DETERMINISTIC if c["noise"] == "det" else 0)


SENS_CASE = {"box": "hc_o17_a6_h32_gail", "airl": "o5_a2_h32_det_airl"}


def test_float64_step_matches_the_reference_restatements():
    """the float64 policy / env / reward step equals oracle/ppo_port.ActorCriticPort, oracle/synth_env.SynthEnvSpec and
    oracle/nets_port's reward nets evaluated in float64 on the same inputs"""
    from oracle import nets_port, ppo_port, synth_env

    for name in ("hc_o17_a6_h32_gail", "cartpole_o4_d2_h32", "o5_a2_h32_det_airl"):
        c = CASES[name]
        pd, PP, PN, dd, DP, DN = _inputs(name)
        Do, Da, E = c["do"], c["da"], 257
        pol = ppo_port.ActorCriticPort(Do, Da, discrete=c["disc"], hidden=(c["h"], c["h"]),
                                       normalize_features=c["pnorm"]).double()
        P = th.as_tensor(PP.astype(np.float64))
        names = [n for n, _ in _desc.policy_param_shapes(Do, Da, c["disc"], c["h"])]
        port_names = {"mlp_extractor.policy_net": "pi", "mlp_extractor.value_net": "vf"}
        sd = {}
        o = 0
        for n, s in _desc.policy_param_shapes(Do, Da, c["disc"], c["h"]):
            k = n
            for a, b in port_names.items():
                k = k.replace(a, b)
            sd[k] = P[o:o + int(np.prod(s))].reshape(s)
            o += int(np.prod(s))
        assert len(names) == len(sd)
        if c["pnorm"]:
            sd["feat_norm.running_mean"] = th.as_tensor(PN[:Do].astype(np.float64))
            sd["feat_norm.running_var"] = th.as_tensor(PN[Do:].astype(np.float64))
            pol.feat_norm.eps = float(np.float32(pd.norm_eps))
        pol.load_state_dict(sd, strict=False)
        pol.eval()
        # (ActorCriticPort.features casts the observations to float32; keep them in float64 here)
        pol.features = lambda x: pol.feat_norm(x) if pol.feat_norm is not None else x
        rng = np.random.default_rng(1)
        obs = th.as_tensor(rng.uniform(-0.9, 0.9, (E, Do)))
        noise = th.as_tensor(rng.random(E) if c["disc"] else rng.standard_normal((E, Da)))
        with th.no_grad():
            a_port, v_port, lp_port = pol(obs, noise)
        out, _, v, _, ls = _policy64(pd, _lib.ACT_TANH, PP, PN, obs)
        th.testing.assert_close(v, v_port[:, 0], rtol=1e-12, atol=1e-12)
        if c["disc"]:
            cdf = th.cumsum(th.softmax(out, 1), 1)
            k = ((noise[:, None] >= cdf).sum(1)).clamp(max=Da - 1)
            assert th.equal(k, a_port)
            th.testing.assert_close(out[th.arange(E), k] - th.logsumexp(out, 1), lp_port, rtol=1e-12, atol=1e-12)
            u = th.nn.functional.one_hot(k, Da).double()
        else:
            a = out + th.exp(ls) * noise
            th.testing.assert_close(a, a_port, rtol=1e-12, atol=1e-12)
            diff = a - out
            lp = (-(diff * diff) / (2 * th.exp(2 * ls)) - ls - 0.9189385332046727).sum(1)
            th.testing.assert_close(lp, lp_port, rtol=1e-12, atol=1e-12)
            u = th.clamp(a, -1, 1)
        spec = synth_env.SynthEnvSpec(Do, Da, discrete=c["disc"], horizon=c["H"], seed=SEED)
        EP = _desc.synth_env_params(Do, Da, SEED)
        nobs, _, w, _ = _env64(EP, Do, Da, obs, u)
        A, B = spec.A.astype(np.float64), spec.Bm.astype(np.float64)
        want = np.tanh(obs.numpy() @ A.T + u.numpy() @ B.T + spec.c.astype(np.float64))
        np.testing.assert_allclose(nobs.numpy(), want, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(w.numpy(), spec.w.astype(np.float64), rtol=0, atol=0)
        # reward net
        done = th.as_tensor((rng.random(E) < 0.3).astype(np.float64))
        kw = c["net"]
        if dd.shaped:
            net = nets_port.ShapedRewardNetPort(Do, Da, reward_hid_sizes=kw["hid_sizes"],
                                                potential_hid_sizes=kw.get("potential_hid_sizes", (32, 32)),
                                                discount_factor=float(np.float32(dd.gamma)),
                                                normalize_input=kw.get("normalize_input", False)).double()
            mods = [net.base.mlp, net.potential]
        else:
            net = nets_port.BasicRewardNetPort(Do, Da, hid_sizes=kw.get("hid_sizes", (32, 32)),
                                               normalize_input=kw.get("normalize_input", False)).double()
            mods = [net.mlp]
        o = 0
        NS = DN[0]
        for i, m in enumerate(mods):
            for lin in [x for x in m if isinstance(x, th.nn.Linear)]:
                for p in (lin.weight, lin.bias):
                    p.data = th.as_tensor(DP[0][o:o + p.numel()].astype(np.float64)).reshape(p.shape)
                    o += p.numel()
            if NS is not None:
                mlp = dd.base if i == 0 else dd.potential
                rn = m.normalize_input
                rn.running_mean = th.as_tensor(NS[mlp.norm_off:mlp.norm_off + mlp.din].astype(np.float64))
                rn.running_var = th.as_tensor(NS[mlp.norm_off + mlp.din:mlp.norm_off + 2 * mlp.din]
                                              .astype(np.float64))
                rn.eps = float(np.float32(mlp.norm_eps))
        net.eval()
        with th.no_grad():
            want = net(obs, u, nobs, done)
        r, _ = _reward64(dd, DP[0], DN[0], obs, u, nobs, done)
        th.testing.assert_close(r, want, rtol=1e-12, atol=1e-12)


def _pert_tower(P):
    pd = _inputs(SENS_CASE["box"])[0]
    n = pd.hidden * pd.d_obs
    P[pd.off_pi_w1:pd.off_pi_w1 + n] *= 1.001
    return P


MUTATIONS = {
    "tower_weight_0.1pct": ("box", dict(pert=_pert_tower)),
    "log_std_1e-3": ("box", dict(log_std=lambda ls: ls + 1e-3)),
    "next_obs_of_the_wrong_step": ("box", dict(wrong_step=True)),
    "potential_gamma_1": ("airl", dict(potential_gamma=1.0)),
    "softplus_as_minus_logsigmoid": ("box", dict(logsigmoid=True)),
    "reward_on_unclipped_action": ("box", dict(unclipped=True)),
}


def test_comparator_accepts_the_float64_rollout():
    for case in SENS_CASE.values():
        seen = {}
        args, flags = _simulate(case, 203)
        check_launch(*args, seen, flags)
        check_rows(args[0], args[9], args[10], args[13])


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_comparator_rejects(mutation):
    case, sim = MUTATIONS[mutation]
    args, flags = _simulate(SENS_CASE[case], 203, sim)
    with pytest.raises((AssertionError, pytest.fail.Exception)):
        check_launch(*args, {}, flags)
