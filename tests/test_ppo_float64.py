"""The PPO update kernels at every policy shape and minibatch they accept, against a float64 PPO step.

imb_ppo_update runs one of three kernels (imb_ppo_plan): k_ppo_update (tower width <= 32, minibatch <= 64 rows resident
in shared memory), k_ppo_update_gen<1> and k_ppo_update_gen<2> (width <= 32 / <= 64, minibatches up to 4096 rows).  The
reference below restates SB3 2.2 PPO.train (oracle/ppo_port.PPOPort.train) in float64, from the same fp32 parameters,
statistics and rollout rows: the feature RunningNorm update before normalising (train mode), tanh towers, Categorical /
diagonal Gaussian heads, ratio = exp(logp - logp_old), -min(adv r, adv clamp(r)), MSE value loss, -mean(entropy),
advantage normalisation (ddof 1, + 1e-8, skipped for one-row minibatches), clip_grad_norm_ (max / (total + 1e-6), capped
at 1) and Adam with the kernels' constants (beta 0.9f / 0.999f, bias corrections from ST_PPO_STEP).

Adam moves every weight by about lr whatever the gradient is, so comparing parameters after a run says little about the
gradient.  Three measurements avoid that amplification:

1. One step's gradient, read out through Adam's first and second moments: from exp_avg = exp_avg_sq = 0 at lr = 0 the
   kernel leaves exp_avg = (1 - 0.9f) clip g and exp_avg_sq = (1 - 0.999f) (clip g)^2; with max_grad_norm 1e30 (clip 1)
   and 0.5 (clip active, asserted).
2. Whole runs at lr = 0 over several epochs: the parameters come back bit-unchanged; every step's loss-log row, the
   feature RunningNorm after the chained minibatch updates, the final moments (the beta-weighted sums of every step's
   clipped gradient) and the state words are compared with float64.  Host and device (Feistel) permutations, ragged
   last minibatches.
3. Adam and the parameter all-gather at lr != 0, teacher-forced: the kernel is deterministic, so a launch over the
   first k minibatches of a block-shuffled permutation ends in the state a launch over k + 1 minibatches has after step
   k.  That state is the float64 start of step k + 1, and the second launch's outputs are checked against it.

Tolerances.  Each parameter's gradient is a sum over rows of per-row terms (torch.func vmap of grad).  The kernel's
gradient may deviate from float64 by C_GRAD times the sum of the absolute per-row terms, plus FLOOR times the largest
such sum: a single wrong row fails even where the sum cancels.  Each absolute per-row term is widened by how much it
changes when the tanh derivatives are padded by what fp32 cannot resolve (_PaddedTanh): 1 - tanh^2 of a nearly saturated unit
(pre-activations here reach +-30) to about 1e-7 absolute, and its change under the pre-activation's own fp32 error.
With tower weights of scale up to 15 that error is large: a first-layer pre-activation rounds to ~1e-5 absolute, which
reaches the second layer as up to ~1e-3 and moves 1 - tanh^2 there by up to ~2e-3 relative.  Beyond that the kernels'
approximations (tanh_fast's switch at |x| = 0.1, __expf, sqrt.approx, __fdividef) are about 1e-6 relative: C_GRAD =
1e-4, calibrated on an H100.  A gradient off by 1 % in one tensor, or the advantage std with ddof 0 at 64 rows (0.8 %),
stays far outside.  With clip_grad_norm_ active the clip factor carries the relative error of the total norm.  Moments
and parameters inherit these bounds through the Adam arithmetic (evaluated at the corners of the bounds), plus fp32
rounding of the recurrence; the chained RunningNorm statistics a few fp32 roundings per minibatch update.

Every case also checks that the outputs are bit-identical with and without the loss log, that two identical launches
agree bit for bit, and that imb_ppo_plan names the kernel the case expects.
"""
import math

import numpy as np
import pytest
import torch as th
from torch import func as tfunc

from imitation_b200 import _desc, _lib

pytestmark = pytest.mark.gpu

C_GRAD = 1e-4       # per-parameter gradient tolerance relative to sum_rows |per-row term|
FLOOR = 1e-7        # absolute floor, relative to the largest sum_rows |per-row term| of the step
SAT_PAD = 2e-7      # absolute error of 1 - tanh^2 in fp32 near saturation (times C_GRAD^-1 in the padded derivative)
C_LOSS = 2e-5       # loss-log terms relative to the mean magnitude of their per-row terms
MARGIN = 1e-3       # every row's ratio stays this far from the clip band's edges
B1F, B2F = float(np.float32(0.9)), float(np.float32(0.999))
U24 = 2.0 ** -24

# name: (d_obs, d_act, discrete, width, feature norm, minibatch, N, epochs, initial norm count, ent_coef,
#        normalize_advantage, permutation, force general, plan code)
#   N: an int, or "k*mb", "k*mb+1" with k minibatches; permutation "host" / "device"
CASES = {
    # ---- k_ppo_update: widths 1 / 7 / 20 / 32, d_obs across the 32 / 64 input tiles, Box d_act around the 8-lane
    #      fast path, Discrete with more than 8 actions, minibatches 1 / 2 / 16 / 48 / 63 / 64, N < mb, ragged ends
    "u_w1_o1_a1_mb1": (1, 1, False, 1, True, 1, 3, 2, 700, 0.0, True, "host", False, 1),
    "u_w7_o4_d9_mb2": (4, 9, True, 7, False, 2, "2*mb+1", 2, 0, 0.01, True, "host", False, 1),
    "u_w20_o17_a6_mb16": (17, 6, False, 20, True, 16, "3*mb", 2, 10 ** 7, 0.01, True, "device", False, 1),
    "u_w32_o31_a8_mb48": (31, 8, False, 32, True, 48, "2*mb+1", 1, 700, 0.0, False, "host", False, 1),
    "u_w32_o32_a9_mb63": (32, 9, False, 32, False, 63, "2*mb", 2, 0, 0.01, True, "host", False, 1),
    "u_w32_o33_a17_mb64": (33, 17, False, 32, True, 64, "2*mb+1", 2, 10 ** 7, 0.01, True, "host", False, 1),
    "u_w20_o60_d18_mb64": (60, 18, True, 20, True, 64, "3*mb", 2, 10 ** 7, 0.0, True, "host", False, 1),
    "u_w32_o64_a6_mb16": (64, 6, False, 32, True, 16, "3*mb+1", 1, 0, 0.01, True, "host", False, 1),
    "u_w7_o17_d2_lt_mb": (17, 2, True, 7, True, 64, 40, 3, 10 ** 7, 0.01, True, "host", False, 1),
    "u_w32_o4_d18_mb64": (4, 18, True, 32, False, 64, "8*mb", 2, 0, 0.01, False, "device", False, 1),
    "u_w1_o31_a9_mb63": (31, 9, False, 1, False, 63, "2*mb+1", 2, 0, 0.0, True, "host", False, 1),
    "u_w20_o1_a17_mb2": (1, 17, False, 20, True, 2, "4*mb", 2, 10 ** 7, 0.01, True, "host", False, 1),
    "u_w7_o64_a8_mb48": (64, 8, False, 7, False, 48, "2*mb", 2, 0, 0.0, True, "host", False, 1),
    "u_w32_o32_d9_mb1": (32, 9, True, 32, True, 1, 4, 2, 10 ** 7, 0.01, True, "host", False, 1),
    "u_w32_o64_a19_mb64": (64, 19, False, 32, True, 64, "2*mb", 2, 10 ** 7, 0.01, True, "host", False, 1),
    # ---- k_ppo_update_gen<1>: minibatches 65 / 128 / 129 / 512 / 4096, the forced-general shapes, the re-routed ones
    "g1_w32_o17_a6_mb65": (17, 6, False, 32, True, 65, "2*mb+1", 2, 10 ** 7, 0.01, True, "host", False, 2),
    "g1_w20_o4_d9_mb128": (4, 9, True, 20, False, 128, "3*mb", 2, 0, 0.01, True, "device", False, 2),
    "g1_w7_o33_a9_mb129": (33, 9, False, 7, True, 129, "2*mb+1", 2, 10 ** 7, 0.0, True, "host", False, 2),
    "g1_w32_o11_a3_mb512": (11, 3, False, 32, True, 512, "2*mb", 1, 700, 0.01, True, "host", False, 2),
    "g1_w32_o27_a8_mb4096": (27, 8, False, 32, True, 4096, "1*mb+1", 1, 0, 0.01, True, "host", False, 2),
    "g1_w1_o1_d18_lt_mb": (1, 18, True, 1, True, 512, 300, 2, 10 ** 7, 0.01, False, "host", False, 2),
    "g1_forced_w32_o17_a6": (17, 6, False, 32, True, 64, "2*mb+1", 1, 700, 0.01, True, "host", True, 2),
    "g1_forced_w20_o4_d2_mb1": (4, 2, True, 20, False, 1, 5, 2, 0, 0.01, True, "host", True, 2),
    "g1_forced_w7_o64_d18_mb16": (64, 18, True, 7, True, 16, "3*mb", 2, 10 ** 7, 0.0, True, "device", True, 2),
    "g1_reroute_o64_a20": (64, 20, False, 32, True, 64, "2*mb+1", 2, 10 ** 7, 0.01, True, "host", False, 2),
    "g1_reroute_o32_a64": (32, 64, False, 32, False, 16, "3*mb", 2, 0, 0.01, True, "host", False, 2),
    "g1_reroute_o60_d64": (60, 64, True, 32, True, 2, "4*mb+1", 2, 700, 0.01, True, "host", False, 2),
    # ---- k_ppo_update_gen<2>: widths 33 / 40 / 63 / 64, d_obs up to 64, d_act up to the plan's edge
    "g2_w33_o17_a6_mb1": (17, 6, False, 33, True, 1, 4, 2, 700, 0.01, True, "host", False, 3),
    "g2_w40_o33_d9_mb64": (33, 9, True, 40, True, 64, "2*mb+1", 2, 10 ** 7, 0.01, True, "host", False, 3),
    "g2_w63_o60_a17_mb200": (60, 17, False, 63, True, 200, "2*mb+1", 2, 10 ** 7, 0.0, True, "host", False, 3),
    "g2_w64_o64_a16_mb4096": (64, 16, False, 64, True, 4096, "1*mb+1", 1, 10 ** 7, 0.01, True, "host", False, 3),
    "g2_w64_o64_a34_mb64": (64, 34, False, 64, False, 64, "2*mb", 2, 0, 0.01, True, "host", False, 3),
    "g2_w64_o64_d35_mb1": (64, 35, True, 64, True, 1, 3, 2, 10 ** 7, 0.01, True, "host", False, 3),
    "g2_w33_o4_d18_mb200": (4, 18, True, 33, False, 200, "2*mb", 2, 0, 0.01, False, "device", False, 3),
    "g2_w64_o17_a8_mb64": (17, 8, False, 64, True, 64, "3*mb+1", 1, 700, 0.0, True, "host", False, 3),
    # ---- the three bench.py update shapes, as full runs
    "bench_hc": (17, 6, False, 32, True, 64, 4096, 5, 10 ** 7, 0.0, True, "device", False, 1),
    "bench_cartpole": (4, 2, True, 32, False, 64, 2048, 10, 0, 0.0, True, "host", False, 1),
    "bench_ant": (27, 8, False, 32, True, 16, 2048, 10, 10 ** 7, 0.01, True, "host", False, 1),
}
PREFIX_K = (0, 1, 2, 7)
START_STEP = (0, 1, 40, 10 ** 6)
CLIP = 0.2
EPS_NORM = float(np.float32(1e-5))


def _cfg(name):
    Do, Da, disc, h, norm, mb, N, ep, cnt, ent, nadv, perm, force, code = CASES[name]
    if isinstance(N, str):
        k, plus = N.split("*mb")
        N = int(k) * mb + (int(plus) if plus else 0)
    i = list(CASES).index(name)
    return dict(name=name, Do=Do, Da=Da, disc=disc, h=h, norm=norm, mb=mb, N=N, epochs=ep, count0=cnt, ent=ent,
                nadv=nadv, perm=perm, force=force, code=code, idx=i, seed=1000 + 17 * i)


@pytest.fixture(scope="module")
def L():
    _lib.lib()
    return _lib


@pytest.fixture
def force_env(monkeypatch):
    def set_force(on):
        if on:
            monkeypatch.setenv("IMB_PPO_FORCE_GENERAL", "1")
        else:
            monkeypatch.delenv("IMB_PPO_FORCE_GENERAL", raising=False)
    return set_force


# ---------------------------------------------------------------------------------------------------------------------
# the float64 PPO step
# ---------------------------------------------------------------------------------------------------------------------
class _PaddedTanh(th.autograd.Function):
    """tanh(x) whose derivative is padded by what fp32 cannot resolve: 1 - tanh^2 to SAT_PAD absolute, and its change
    2 |tanh| (1 - tanh^2) dx under the pre-activation's fp32 error dx (only used for the magnitudes of the per-row
    terms, which C_GRAD scales)."""
    generate_vmap_rule = True

    @staticmethod
    def forward(x, dx):
        return th.tanh(x)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.save_for_backward(output, inputs[1])

    @staticmethod
    def backward(ctx, g):
        y, dx = ctx.saved_tensors
        d = 1 - y * y
        return g * (d + (SAT_PAD + 2 * y.abs() * d * dx) / C_GRAD), None


class Ref:
    """Policy shape, hyper-parameters and the float64 arithmetic of one PPO optimiser step."""

    def __init__(self, c, ent_coef, vf_coef=0.5, nadv=True):
        self.c = c
        self.Do, self.Da, self.disc, self.h = c["Do"], c["Da"], c["disc"], c["h"]
        self.shapes = _desc.policy_param_shapes(self.Do, self.Da, self.disc, self.h)
        self.ent_coef, self.vf_coef, self.nadv = float(np.float32(ent_coef)), float(np.float32(vf_coef)), nadv
        self.clip = float(np.float32(CLIP))
        self.da_store = 1 if self.disc else self.Da
        self.col = self.Do + self.da_store  # logp | value | reward | adv | ret

    def unpack(self, p):
        out, o = [], 0
        for _, s in self.shapes:
            n = int(np.prod(s))
            out.append(p[o:o + n].reshape(s))
            o += n
        return out

    def heads(self, p, xn, padded=False):
        """xn [..., Do] -> action means / logits [..., Da], value [...], the value tower's latent.  padded: the towers'
        tanh is _PaddedTanh, fed with a bound of each pre-activation's fp32 error (the rounding of its dot product,
        fan_in ulps of the sum of its absolute terms, plus the error of its inputs)"""
        W = self.unpack(p)

        def layer(x, e, w, b):
            z = x @ w.T + b
            if not padded:
                return th.tanh(z), None
            dz = w.shape[1] * U24 * (x.abs() @ w.abs().T + b.abs()) + e @ w.abs().T
            y = _PaddedTanh.apply(z, dz.detach())
            return y, ((1 - y * y) * dz + SAT_PAD).detach()

        e0 = (4 * U24 * xn.abs()) if padded else None
        lat = layer(*layer(xn, e0, W[0], W[1]), W[2], W[3])[0]
        lv = layer(*layer(xn, e0, W[4], W[5]), W[6], W[7])[0]
        return lat @ W[8].T + W[9], (lv @ W[10].T)[..., 0] + W[11][0], lv, W

    def logp_ent(self, p, out, act):
        if self.disc:
            lsm = th.log_softmax(out, -1)
            return (lsm * act).sum(-1), -(lsm.exp() * lsm).sum(-1)
        ls = self.unpack(p)[12]
        d = (act - out) * th.exp(-ls)
        return (-0.5 * d * d - ls - 0.5 * math.log(2 * math.pi)).sum(-1), (0.5 + 0.5 * math.log(2 * math.pi) + ls).sum(-1)

    def row_terms(self, p, xn, act, lpo, adv, ret, padded=False):
        out, val, _, _ = self.heads(p, xn, padded)
        logp, ent = self.logp_ent(p, out, act)
        ratio = th.exp(logp - lpo)
        pg = -th.minimum(adv * ratio, adv * th.clamp(ratio, 1 - self.clip, 1 + self.clip))
        return pg, (ret - val) ** 2, -ent, ratio, logp

    def row_loss(self, p, xn, act, lpo, adv, ret, padded=False):
        pg, vl, el, _, _ = self.row_terms(p, xn, act, lpo, adv, ret, padded)
        return pg + self.ent_coef * el + self.vf_coef * vl

    def norm_update(self, st, x):
        """RunningNorm.update_stats then the train-mode normalisation with the updated statistics"""
        if not self.c["norm"]:
            return x
        nb = x.shape[0]
        bm, bv = x.mean(0), x.var(0, unbiased=False)
        delta, tot = bm - st["mean"], st["count"] + nb
        st["mean"] = st["mean"] + delta * nb / tot
        st["var"] = (st["var"] * st["count"] + bv * nb + delta * delta * st["count"] * nb / tot) / tot
        st["count"] = tot
        return (x - st["mean"]) / th.sqrt(st["var"] + EPS_NORM)

    def batch(self, rows):
        Do, c = self.Do, self.col
        act = (th.nn.functional.one_hot(rows[:, Do].long(), self.Da).double() if self.disc else rows[:, Do:Do + self.Da])
        adv = rows[:, c + 3]
        if self.nadv and rows.shape[0] > 1:
            adv = (adv - adv.mean()) / (adv.std() + 1e-8)
        return act, rows[:, c], adv, rows[:, c + 4]

    def step(self, st, rows, max_grad_norm, lr):
        """One optimiser step on state st (P, M, V, mean, var, count, t), float64 in place.  Returns the loss-log row,
        its tolerance, and the tolerance of the clipped gradient."""
        nb = rows.shape[0]
        xn = self.norm_update(st, rows[:, :self.Do])
        act, lpo, adv, ret = self.batch(rows)
        P = st["P"]
        pg, vl, el, ratio, logp = self.row_terms(P, xn, act, lpo, adv, ret)
        edge = th.minimum((ratio - (1 - self.clip)).abs(), (ratio - (1 + self.clip)).abs())
        assert float(edge.min()) >= MARGIN, f"a row's ratio lies {float(edge.min()):.2e} from the clip band's edge"
        # gradient and the magnitudes of its per-row terms
        g, A = th.zeros_like(P), th.zeros_like(P)
        grad = tfunc.vmap(tfunc.grad(self.row_loss), in_dims=(None, 0, 0, 0, 0, 0))
        grad_pad = tfunc.vmap(tfunc.grad(lambda *a: self.row_loss(*a, padded=True)),
                              in_dims=(None, 0, 0, 0, 0, 0))
        for i in range(0, nb, 512):
            s = slice(i, i + 512)
            gi = grad(P, xn[s], act[s], lpo[s], adv[s], ret[s])
            # |term| plus what the padded derivatives add to it (the pads can change a sum over units' sign pattern)
            pad = grad_pad(P, xn[s], act[s], lpo[s], adv[s], ret[s]) - gi
            g += gi.sum(0) / nb
            A += (gi.abs() + pad.abs()).sum(0) / nb
        tol_g = C_GRAD * A + FLOOR * float(A.max())
        total = float(g.norm())
        clip = min(1.0, max_grad_norm / (total + 1e-6))
        gc = clip * g
        tol_gc = clip * tol_g
        if clip < 1.0:  # the clip factor carries the total norm's relative error
            assert total / max_grad_norm > 1.001, "clip_grad_norm_ too close to its threshold for a sharp comparison"
            tol_gc = tol_gc + gc.abs() * (float((g.abs() * tol_g).sum()) / total ** 2 + 1e-6)
        # Adam with the kernel's constants
        st["t"] += 1
        M, V = st["M"], st["V"]
        Mn = B1F * M + (1 - B1F) * gc
        Vn = B2F * V + (1 - B2F) * gc * gc
        tol_M = (1 - B1F) * tol_gc + 2 * U24 * Mn.abs()
        tol_V = (1 - B2F) * (2 * gc.abs() * tol_gc + tol_gc ** 2) + 4 * U24 * Vn.abs()
        lr = float(np.float32(lr))
        bc1, bc2 = 1.0 - 0.9 ** st["t"], 1.0 - 0.999 ** st["t"]
        eps = float(np.float32(1e-5))

        def upd(m, v):
            return lr / bc1 * m / (th.sqrt(v.clamp(min=0)) / math.sqrt(bc2) + eps)

        du = upd(Mn, Vn)
        spread = th.zeros_like(P)
        for sm in (-1, 1):
            for sv in (-1, 1):
                spread = th.maximum(spread, (upd(Mn + sm * tol_M, Vn + sv * tol_V) - du).abs())
        st["tol_P"] = spread + 1e-5 * du.abs() + 4 * U24 * P.abs()
        st["P"], st["M"], st["V"] = P - du, Mn, Vn
        st["tol_M"] = B1F * st.get("tol_M", 0 * P) + tol_M
        st["tol_V"] = B2F * st.get("tol_V", 0 * P) + tol_V
        st["clip"] = clip
        # loss log and per-column tolerances from the magnitudes of the per-row terms
        out, val, lv, W = self.heads(P, xn)
        vmag = (lv * W[10][0]).abs().sum(-1) + abs(float(W[11][0])) + 1.0
        if self.disc:
            lmag = out.abs().max(-1).values
        else:
            d = (act - out) * th.exp(-W[12])
            lmag = (0.5 * d * d + W[12].abs()).sum(-1)
        mags = [(pg.abs() * (1 + logp.abs() + lmag)).mean(), (vl + 2 * vl.sqrt() * vmag).mean(),
                (el.abs() + lmag).mean()]
        log = [float(pg.mean()), float(vl.mean()), float(el.mean())]
        log.append(log[0] + self.ent_coef * log[2] + self.vf_coef * log[1])
        tol = [C_LOSS * float(m) + 1e-7 for m in mags]
        tol.append(tol[0] + self.ent_coef * tol[2] + self.vf_coef * tol[1])
        return np.array(log), np.array(tol), gc, tol_gc


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _make_inputs(c):
    """fp32 parameters (pre-activations up to about +-30, many near the tanh_fast switch at +-0.1; log_std in [-3, 1.5];
    Discrete logits spread to log-probabilities near -80), rollout rows, feature statistics near the data's."""
    rng = np.random.default_rng(c["seed"])
    Do, Da, disc, h = c["Do"], c["Da"], c["disc"], c["h"]
    parts = []
    for name, shape in _desc.policy_param_shapes(Do, Da, disc, h):
        if name.endswith("0.weight") or name.endswith("2.weight"):  # tower layers: per-unit scale 0.05 .. 15
            scale = np.geomspace(0.05, 15.0, shape[0]) if shape[0] > 1 else np.array([4.0])
            w = rng.standard_normal(shape) / np.sqrt(shape[1]) * rng.permutation(scale)[:, None]
        elif name.endswith("bias") and "mlp_extractor" in name:
            w = rng.standard_normal(shape) * 0.3
        elif name == "action_net.weight":
            w = rng.standard_normal(shape) / np.sqrt(shape[1]) * (25.0 if disc else 0.5)
        elif name == "log_std":
            w = rng.uniform(-3.0, 1.5, shape)
            w[:2] = [-3.0, 1.5][:shape[0]]
        else:
            w = rng.standard_normal(shape) * 0.5
        parts.append(w.reshape(-1))
    P = np.concatenate(parts).astype(np.float32)
    N = c["N"]
    mu, sd = rng.normal(0.2, 0.5, Do), rng.uniform(0.5, 2.0, Do)
    obs = (mu + sd * rng.standard_normal((N, Do))).astype(np.float32)
    if c["norm"]:
        norm = np.concatenate([mu + 0.05 * sd * rng.standard_normal(Do), sd ** 2 * rng.uniform(0.9, 1.1, Do)])
    else:
        norm = np.zeros(2)
    pd = _desc.policy_desc(Do, Da, disc, h, c["norm"])
    rw = _lib.rollout_row_width(pd)
    tbl = np.zeros((N, rw), np.float32)
    tbl[:, :Do] = obs
    col = Do + (1 if disc else Da)
    tbl[:, col + 1] = rng.standard_normal(N)                  # value (not read by the update)
    tbl[:, col + 3] = rng.normal(0.3, 2.0, N)                  # advantages of both signs
    tbl[:, col + 4] = rng.standard_normal(N) * 2.0             # returns
    if disc:
        tbl[:, Do] = rng.integers(0, Da, N)
    else:  # actions around the initial means (normalised with the initial statistics), 1.5 std out
        ref = Ref(c, 0.0)
        x = th.from_numpy(obs).double()
        if c["norm"]:
            x = (x - th.from_numpy(norm[:Do])) / th.sqrt(th.from_numpy(norm[Do:]) + EPS_NORM)
        out = ref.heads(th.from_numpy(P).double(), x)[0].numpy()
        ls = P[pd.off_log_std:pd.off_log_std + Da]
        tbl[:, Do:Do + Da] = out + np.exp(ls) * 1.5 * rng.standard_normal((N, Da))
    M = (rng.standard_normal(P.size) * 1e-3).astype(np.float32)
    V = (np.abs(rng.standard_normal(P.size)) * 1e-5).astype(np.float32)
    return pd, P, norm.astype(np.float32), tbl, M, V, rng


def _ratio_targets(rng, n):
    """ratio targets: inside the clip band, below it and above it (advantages carry both signs)"""
    kind = rng.integers(0, 3, n)
    inside = rng.uniform(1 - CLIP + 0.05, 1 + CLIP - 0.05, n)
    below = rng.uniform(0.3, 1 - CLIP - 0.05, n)
    above = rng.uniform(1 + CLIP + 0.05, 3.0, n)
    return np.where(kind == 0, inside, np.where(kind == 1, below, above))


def _set_logp_old(ref, tbl, rows_idx, st, P, rng):
    """logp_old of the rows of one minibatch, from their float64 logp at this step (statistics updated first)"""
    st = dict(st)
    rows = th.from_numpy(tbl[rows_idx]).double()
    xn = ref.norm_update(st, rows[:, :ref.Do])
    act, _, _, _ = ref.batch(rows)
    logp = ref.logp_ent(P, ref.heads(P, xn)[0], act)[0].numpy()
    tbl[rows_idx, ref.col] = (logp - np.log(_ratio_targets(rng, len(rows_idx)))).astype(np.float32)


def _epoch_perms(c, rng):
    """[epochs][N] minibatch order: the first epoch shuffles consecutive blocks of mb rows (its first k mb entries are a
    permutation of [0, k mb)), later epochs are full shuffles; or the device's Feistel permutations"""
    N, mb = c["N"], c["mb"]
    if c["perm"] == "device":
        from oracle import philox

        return np.stack([philox.feistel_perm(c["seed"], philox.STREAM_PPO_PERM, 3 + e, N) for e in range(c["epochs"])])
    first = np.concatenate([s + rng.permutation(min(mb, N - s)) for s in range(0, N, mb)])
    return np.stack([first] + [rng.permutation(N) for _ in range(c["epochs"] - 1)]).astype(np.int64)


def _state0(c, P, norm, M, V, step):
    Do = c["Do"]
    return dict(P=th.from_numpy(P).double(), M=th.from_numpy(M).double(), V=th.from_numpy(V).double(),
                mean=th.from_numpy(norm[:Do]).double() if c["norm"] else None,
                var=th.from_numpy(norm[Do:]).double() if c["norm"] else None,
                count=c["count0"] if c["norm"] else 0, t=step)


# ---------------------------------------------------------------------------------------------------------------------
# the kernel
# ---------------------------------------------------------------------------------------------------------------------
def _launch(L, c, pd, P, norm, count, M, V, tbl, n_rows, perm, epochs, lr, mgn, step, with_log, ent, nadv):
    n_steps = epochs * ((n_rows + c["mb"] - 1) // c["mb"])
    hp = L.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=CLIP, ent_coef=ent, vf_coef=0.5, max_grad_norm=mgn, lr=lr,
                      adam_eps=1e-5, n_epochs=epochs, batch_size=c["mb"], normalize_advantage=int(nadv))
    t = {k: th.from_numpy(np.ascontiguousarray(a)).cuda() for k, a in
         dict(params=P, exp_avg=M, exp_avg_sq=V, norm=norm).items()}
    t["count"] = th.tensor([count], dtype=th.int32, device="cuda")
    st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
    st[L.ST_PPO_STEP], st[L.ST_PPO_EPOCH] = step, 3
    st[L.ST_GLOBAL_STEP] = 12345
    t["state"] = st
    log = th.full((n_steps, 4), float("nan"), device="cuda") if with_log else None
    pt = None if perm is None else th.from_numpy(np.ascontiguousarray(perm, dtype=np.int64)).cuda()
    L.ppo_update(pd, t["params"], t["norm"], t["count"], t["exp_avg"], t["exp_avg_sq"],
                 th.from_numpy(np.ascontiguousarray(tbl[:n_rows])).cuda(), n_rows, hp, pt, c["seed"], log, t["state"])
    th.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in t.items()}
    if with_log:
        out["log"] = log.cpu().numpy()
    return out


def _same_bits(a, b, what):
    for k in a:
        if k in b:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), f"{what}: {k} differs"


def _check(got, want, tol, what):
    got, want, tol = (np.asarray(x, np.float64) for x in (got, want, tol))
    bad = np.abs(got - want) > tol
    if bad.any():
        i = np.flatnonzero(bad.ravel())
        j = i[np.argmax((np.abs(got - want) / tol).ravel()[i])]
        pytest.fail(f"{what}: {bad.sum()} of {bad.size} outside tolerance; worst at {j}: got {got.ravel()[j]!r}, "
                    f"float64 {want.ravel()[j]!r}, tolerance {tol.ravel()[j]:.3e}")
    return float(np.max(np.abs(got - want) / tol)) if got.size else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
def test_cases_cover_every_kernel(L, force_env):
    """All three kernels occur and every case runs on the kernel it names."""
    codes = set()
    for name in CASES:
        c = _cfg(name)
        force_env(c["force"])
        pd = _desc.policy_desc(c["Do"], c["Da"], c["disc"], c["h"], c["norm"])
        assert L.ppo_plan(pd, c["mb"]) == c["code"], name
        codes.add(c["code"])
    assert codes == {L.PPO_PLAN_UPDATE, L.PPO_PLAN_GEN1, L.PPO_PLAN_GEN2}


def _prepare(c):
    pd, P, norm, tbl, M, V, rng = _make_inputs(c)
    ref = Ref(c, c["ent"], nadv=c["nadv"])
    perms = _epoch_perms(c, rng)
    # logp_old from each row's float64 logp at its use in the first epoch (at lr = 0 the parameters stay put)
    st = _state0(c, P, norm, M, V, 0)
    Pd = st["P"]
    for s in range(0, c["N"], c["mb"]):
        idx = perms[0][s:s + c["mb"]]
        _set_logp_old(ref, tbl, idx, st, Pd, rng)
        ref.norm_update(st, th.from_numpy(tbl[idx, :c["Do"]]).double())
    return pd, P, norm, tbl, M, V, rng, ref, perms


@pytest.mark.parametrize("name", list(CASES))
def test_one_step_gradient_through_adam_moments(L, force_env, name):
    """Measurement 1: lr = 0 from zero moments leaves exp_avg = (1 - 0.9f) clip g, exp_avg_sq = (1 - 0.999f) (clip g)^2."""
    c = _cfg(name)
    force_env(c["force"])
    pd, P, norm, tbl, M, V, rng, ref, perms = _prepare(c)
    idx = perms[0][:c["mb"]]
    sub = tbl[idx]
    nb = len(idx)
    sub_perm = rng.permutation(nb)[None]
    z = np.zeros_like(P)
    for mgn in (1e30, 0.5):
        runs = [_launch(L, c, pd, P, norm, c["count0"] if c["norm"] else 0, z, z, sub, nb,
                        None if c["perm"] == "device" else sub_perm, 1, 0.0, mgn, 0, wl, c["ent"], c["nadv"])
                for wl in (True, False, True)]
        _same_bits(runs[0], runs[1], f"{name} mgn={mgn}: with / without the loss log")
        _same_bits(runs[0], runs[2], f"{name} mgn={mgn}: two identical launches")
        got = runs[0]
        assert np.array_equal(got["params"].view(np.uint32), P.view(np.uint32)), "lr = 0 moved a parameter"
        st = _state0(c, P, norm, z, z, 0)
        log, tol_log, gc, tol_gc = ref.step(st, th.from_numpy(sub).double(), mgn, 0.0)
        if mgn < 1:
            assert st["clip"] < 0.9, f"clip_grad_norm_ inactive (clip {st['clip']:.3f}): the case does not test it"
        else:
            assert st["clip"] == 1.0
        w = _check(got["exp_avg"], st["M"], st["tol_M"], f"{name} mgn={mgn}: exp_avg")
        w = max(w, _check(got["exp_avg_sq"], st["V"], st["tol_V"], f"{name} mgn={mgn}: exp_avg_sq"))
        w = max(w, _check(got["log"][0], log, tol_log, f"{name} mgn={mgn}: loss log"))
        print(f"{name} mgn={mgn}: worst |deviation| / tolerance {w:.3f}")


@pytest.mark.parametrize("name", list(CASES))
def test_whole_run_at_lr0(L, force_env, name):
    """Measurement 2: several epochs at lr = 0 against the chained float64 steps."""
    c = _cfg(name)
    force_env(c["force"])
    pd, P, norm, tbl, M, V, rng, ref, perms = _prepare(c)
    mgn = 0.5 if c["idx"] % 2 else 1e30
    step0 = START_STEP[c["idx"] % 4]
    cnt = c["count0"] if c["norm"] else 0
    perm = None if c["perm"] == "device" else perms
    runs = [_launch(L, c, pd, P, norm, cnt, M, V, tbl, c["N"], perm, c["epochs"], 0.0, mgn, step0, wl, c["ent"],
                    c["nadv"]) for wl in (True, False, True)]
    _same_bits(runs[0], runs[1], f"{name}: with / without the loss log")
    _same_bits(runs[0], runs[2], f"{name}: two identical launches")
    got = runs[0]
    assert np.array_equal(got["params"].view(np.uint32), P.view(np.uint32)), "lr = 0 moved a parameter"
    st = _state0(c, P, norm, M, V, step0)
    st["tol_M"] = 2 * U24 * st["M"].abs()
    st["tol_V"] = 2 * U24 * st["V"].abs()
    N, mb, w = c["N"], c["mb"], 0.0
    gs = 0
    for e in range(c["epochs"]):
        for s in range(0, N, mb):
            rows = th.from_numpy(tbl[perms[e][s:s + mb]]).double()
            log, tol_log, _, _ = ref.step(st, rows, mgn, 0.0)
            w = max(w, _check(got["log"][gs], log, tol_log, f"{name}: loss log of step {gs}"))
            gs += 1
    assert got["log"].shape[0] == gs
    w = max(w, _check(got["exp_avg"], st["M"], st["tol_M"], f"{name}: exp_avg"))
    w = max(w, _check(got["exp_avg_sq"], st["V"], st["tol_V"], f"{name}: exp_avg_sq"))
    if c["norm"]:
        Do, sd = c["Do"], th.sqrt(st["var"])
        chain = 4 * U24 * gs  # fp32 rounding of the chained statistics, a few roundings per update
        w = max(w, _check(got["norm"][:Do], st["mean"], (2e-6 + chain) * (st["mean"].abs() + sd),
                          f"{name}: RunningNorm mean"))
        w = max(w, _check(got["norm"][Do:], st["var"], (1e-6 + chain) * st["var"], f"{name}: RunningNorm var"))
        assert int(got["count"][0]) == st["count"]
    else:
        assert np.array_equal(got["norm"], norm) and int(got["count"][0]) == 0
    want_state = np.zeros(L.ST_WORDS, np.int64)
    want_state[L.ST_PPO_STEP], want_state[L.ST_PPO_EPOCH], want_state[L.ST_GLOBAL_STEP] = step0 + gs, 3 + c["epochs"], 12345
    assert np.array_equal(got["state"], want_state)
    print(f"{name}: {gs} steps, worst |deviation| / tolerance {w:.3f}")


PREFIX_CASES = [n for n in CASES if CASES[n][11] == "host"]


@pytest.mark.parametrize("name", PREFIX_CASES)
def test_adam_step_teacher_forced(L, force_env, name):
    """Measurement 3: step k + 1 at lr != 0 from the state a k-step launch leaves, against float64."""
    c = _cfg(name)
    force_env(c["force"])
    pd, P, norm, tbl, M, V, rng, ref, perms = _prepare(c)
    N, mb = c["N"], c["mb"]
    k = min(PREFIX_K[c["idx"] % 4], (N - 1) // mb)
    step0 = START_STEP[(c["idx"] // 2) % 4]
    mgn = 1e30 if c["idx"] % 3 == 0 else 0.5
    lr = 3e-4
    cnt = c["count0"] if c["norm"] else 0
    blk = perms[0]  # block-shuffled: its first k mb entries are a permutation of [0, k mb)
    if k:
        a = _launch(L, c, pd, P, norm, cnt, M, V, tbl, k * mb, blk[None, :k * mb], 1, lr, mgn, step0, True, c["ent"],
                    c["nadv"])
        start = dict(params=a["params"], exp_avg=a["exp_avg"], exp_avg_sq=a["exp_avg_sq"], norm=a["norm"],
                     count=int(a["count"][0]), step=int(a["state"][_lib.ST_PPO_STEP]))
    else:
        a, start = None, dict(params=P, exp_avg=M, exp_avg_sq=V, norm=norm, count=cnt, step=step0)
    assert start["step"] == step0 + k
    n_rows = min(N, (k + 1) * mb)
    idx = blk[k * mb:n_rows]
    c0 = dict(c, count0=start["count"])
    st = _state0(c0, start["params"], start["norm"], start["exp_avg"], start["exp_avg_sq"], start["step"])
    _set_logp_old(ref, tbl, idx, st, st["P"], rng)  # rows of step k only: the k-step launch never reads them
    b = _launch(L, c, pd, P, norm, cnt, M, V, tbl, n_rows, blk[None, :n_rows], 1, lr, mgn, step0, True, c["ent"],
                c["nadv"])
    if a is not None:
        assert np.array_equal(a["log"].view(np.uint32), b["log"][:k].view(np.uint32)), "steps before k differ"
    st["tol_M"], st["tol_V"] = 0 * st["M"], 0 * st["V"]
    log, tol_log, _, _ = ref.step(st, th.from_numpy(tbl[idx]).double(), mgn, lr)
    w = _check(b["log"][k], log, tol_log, f"{name}: loss log of step {k}")
    w = max(w, _check(b["exp_avg"], st["M"], st["tol_M"] + 2 * U24 * st["M"].abs(), f"{name}: exp_avg"))
    w = max(w, _check(b["exp_avg_sq"], st["V"], st["tol_V"] + 2 * U24 * st["V"].abs(), f"{name}: exp_avg_sq"))
    w = max(w, _check(b["params"], st["P"], st["tol_P"], f"{name}: parameters"))
    moved = np.abs(b["params"].astype(np.float64) - start["params"])
    assert np.median(moved) > 1e-5, "the step did not move the parameters"
    if c["norm"]:
        Do, sd = c["Do"], th.sqrt(st["var"])
        w = max(w, _check(b["norm"][:Do], st["mean"], (2e-6 + 4 * U24 * (k + 1)) * (st["mean"].abs() + sd),
                          f"{name}: RunningNorm mean"))
        w = max(w, _check(b["norm"][Do:], st["var"], (1e-6 + 4 * U24 * (k + 1)) * st["var"], f"{name}: RunningNorm var"))
        assert int(b["count"][0]) == st["count"]
    assert int(b["state"][_lib.ST_PPO_STEP]) == step0 + k + 1 and int(b["state"][_lib.ST_PPO_EPOCH]) == 4
    print(f"{name}: k={k} t0={step0}: worst |deviation| / tolerance {w:.3f}")


def test_device_ppo_refuses_unrunnable_shapes_at_construction(L):
    """DevicePPO asks imb_ppo_plan once the policy exists: MlpPolicy 64x64 on a 64 / 64 Box has no kernel."""
    from imitation_b200.algorithms import ppo
    from imitation_b200.envs import synth

    env = synth.DeviceVecEnv(64, 64, 8)
    with pytest.raises(NotImplementedError, match=r"k_ppo_update_gen<2> needs 257536 B of shared memory"):
        ppo.DevicePPO("MlpPolicy", env, batch_size=1)
    gen = ppo.DevicePPO("FeedForward32Policy", env, batch_size=64)  # re-routed to k_ppo_update_gen<1>
    assert L.ppo_plan(gen.policy.desc, 64) == L.PPO_PLAN_GEN1


# ---------------------------------------------------------------------------------------------------------------------
# imb_policy_logp (k_policy_logp<32> / <64>) at the same policy shapes
# ---------------------------------------------------------------------------------------------------------------------
C_LOGP = 1e-5
LOGP_SHAPES = ["u_w1_o1_a1_mb1", "u_w7_o4_d9_mb2", "u_w32_o33_a17_mb64", "u_w20_o60_d18_mb64", "g1_reroute_o32_a64",
               "g1_reroute_o60_d64", "g2_w40_o33_d9_mb64", "g2_w63_o60_a17_mb200", "g2_w64_o64_d35_mb1",
               "g2_w64_o64_a34_mb64"]


@pytest.mark.parametrize("n", [1, 127, 128, 129, (1 << 16) + 3])
@pytest.mark.parametrize("name", LOGP_SHAPES)
def test_policy_logp_against_float64(L, name, n):
    c = dict(_cfg(name), N=n)
    pd, P, norm, tbl, _, _, rng = _make_inputs(c)
    Do, Da = c["Do"], c["Da"]
    ref = Ref(c, 0.0)
    rows = th.from_numpy(tbl).double()
    x = rows[:, :Do]
    PN = th.from_numpy(norm).cuda() if c["norm"] else th.zeros(2, device="cuda")
    if c["norm"]:
        x = (x - th.from_numpy(norm[:Do]).double()) / th.sqrt(th.from_numpy(norm[Do:]).double() + EPS_NORM)
    act = ref.batch(rows)[0]
    Pd = th.from_numpy(P).double()
    out = ref.heads(Pd, x)[0]
    want = ref.logp_ent(Pd, out, act)[0].numpy()
    if c["disc"]:
        mag = (out.abs().max(-1).values + out.gather(1, act.argmax(1, keepdim=True))[:, 0].abs()).numpy()
    else:
        ls = ref.unpack(Pd)[12]
        d = (act - out) * th.exp(-ls)
        mag = (0.5 * d * d + ls.abs() + 1).sum(-1).numpy()
    bw, ld = _desc.batch_rows(Do, Da), _desc.batch_ld(n)
    batch = th.zeros(bw, ld, device="cuda")
    batch[:Do, :n] = th.from_numpy(tbl[:, :Do].T.copy()).cuda()
    batch[Do:Do + Da, :n] = act.T.float().cuda()
    L.policy_logp(pd, th.from_numpy(P).cuda(), PN, batch, ld, n, bw - 1)
    got = batch[bw - 1, :n].cpu().numpy()
    if c["disc"] and n > 1:
        assert want.min() < -40, "the logits do not spread far enough"
    w = _check(got, want, C_LOGP * (1 + np.abs(want) + mag), f"{name} n={n}: log pi")
    print(f"{name} n={n}: worst |deviation| / tolerance {w:.3f}")
