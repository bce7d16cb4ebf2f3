"""The DQN TD kernels at every Q-net shape, activation and batch they accept, against a float64 DQN step.

SQIL's discrete learner runs two kernels.  imb_dqn_target (k_dqn_target<32> for widths up to 32, <64> beyond) writes
the TD rows obs | action index | y of G minibatches of B = n_l + n_e rows, the learner rows from columns of the
feature-major ring and the expert rows from the expert table, y = r + (1 - done) gamma max_a Q_target(s'), reading
the index lists from TD step state[ST_PPO_STEP] - step_base on.  imb_dqn_step (k_ppo_update_gen<1 / 2> under
LOSS_DQN, chosen by imb_dqn_plan) runs G TD steps on those rows: F.smooth_l1_loss(Q(s)[a], y), clip_grad_norm_ and
torch Adam (eps 1e-8, bias corrections from state[ST_PPO_STEP]), the loss of the step that makes the step count k at
loss_log row k - 1 - loss_base.  The float64 reference is oracle/sqil_port.py (q_forward, td_targets, td_grad) with
tanh or ReLU towers.

Adam's first step moves every weight by lr sign(g) whatever |g| is, and Adam and an active clip are invariant to a
common scale of the gradient, so parameters after a few steps say little about the gradient (a mean over n_l rows
instead of B passes).  As in tests/test_ppo_float64.py the gradient is read through Adam's moments instead:

a. TD rows against td_targets, with non-default rewards and gamma, the index lists read from s0 = state - step_base > 0
   (the same bits as lists starting at s0 and no state), obs bit for bit, the action index exactly, y = r exactly on
   done rows.
b. G steps at lr = 0 from exp_avg = exp_avg_sq = 0: the moments are the beta-weighted sums of every step's (1 - 0.9f)
   clip g and (1 - 0.999f) (clip g)^2; at max_grad_norm 1e30 (clip 1) and at one that clips every step (asserted
   total / max_grad_norm > 1.001).  The rows' y put |Q_a - y| on both sides of 1 (asserted), so the clamped branch of
   smooth L1 carries weight.  Parameters come back bit-unchanged and the zero value tower of the image stays zero.
c. The loss log of those steps against float64, at rows addressed by loss_base with the step count starting above 0,
   rows outside left alone, and every output bit-identical without the log.
d. Adam at lr != 0, teacher-forced from start step counts 0, 1, 40 and 10^6: G steps in one launch are bit-identical to
   launches of k, 1 and G - k - 1 steps, and the 1-step launch's outputs are checked against float64 from the state
   the k-step launch left, so fp32 drift never compounds into the bound.
e. Two identical launches agree bit for bit, and dqn_target + dqn_step captured in a CUDA graph and replayed twice (the
   second replay reads its index lists and loss rows at offsets from the advanced step count) give the eager bits.

Tolerances.  The gradient constants are test_ppo_float64's, unchanged: each parameter's gradient may deviate by C_GRAD
times the sum over rows of its absolute per-row terms (torch.func vmap of grad), plus FLOOR times the largest such sum.
The per-row terms are widened where fp32 cannot resolve the derivative: tanh through test_ppo_float64._PaddedTanh, ReLU
across its kink through test_relu_policy._KinkReLU, and smooth L1's clamp(d, -1, 1) by the fp32 error bound of d
divided by C_GRAD (_PaddedHuber): clamp is 1-Lipschitz, so an error e in Q_a moves the row's dL/dQ_a by up to e.
The fp32 error bound of Q (_Ref.q) is propagated through the layers: a pre-activation errs by at most fan_in ulps of
sum |w||x| + |b| (the worst case of any summation order) plus its inputs' bounds through |w|; tanh scales that by
1 - tanh^2 and adds SAT_PAD for tanh_fast, ReLU passes it where z > -bound.  The TD target's bound is gamma (1 - done)
max_a of Q's bound (max is 1-Lipschitz) plus one rounding each of gamma mx and of the sum.  The loss log's bound is the
mean of |clamp(d)| times d's bound, plus C_LOSS (test_ppo_float64's) of the mean row magnitude.  Moments and parameters
inherit the gradient bound through the Adam arithmetic evaluated at the corners of the bounds, as test_ppo_float64.Ref.
step does.
"""
import numpy as np
import pytest
import torch as th
from torch import func as tfunc

from imitation_b200 import _desc, _lib
from oracle import sqil_port
from tests import test_ppo_float64 as F
from tests.test_relu_policy import RELU_HEAD, _KinkReLU

pytestmark = pytest.mark.gpu

C_GRAD, FLOOR, SAT_PAD, C_LOSS, U24, B1F, B2F = F.C_GRAD, F.FLOOR, F.SAT_PAD, F.C_LOSS, F.U24, F.B1F, F.B2F
EPS = 1e-8  # torch Adam's default eps, DQN's
TANH, RELU = _lib.ACT_TANH, _lib.ACT_RELU
GEN1, GEN2 = _lib.PPO_PLAN_GEN1, _lib.PPO_PLAN_GEN2
ACTIVE = "active"  # max_grad_norm half the smallest float64 gradient norm of the checked steps: clip_grad_norm_ acts
# the C ABI takes any rewards and gamma (SQIL passes 0 / 1 and 0.99): values SQIL never uses, so a swapped or hard-coded
# constant shows; the kernel receives gamma as a float32
R_L, R_E, GAMMA = 0.375, -1.25, float(np.float32(0.9))

# name: (d_obs, n_actions, width, activation, B, G steps, start step, max_grad_norm, plan)
CASES = {
    # ---- k_ppo_update_gen<1> and k_dqn_target<32>: widths 1, 7, 20, 32
    "w1_o1_a1_b1_tanh": (1, 1, 1, TANH, 1, 4, 0, 1e30, GEN1),            # B = 1: no learner rows
    "w7_o4_a2_b2_relu": (4, 2, 7, RELU, 2, 4, 1, ACTIVE, GEN1),
    "w20_o17_a9_b33_tanh": (17, 9, 20, TANH, 33, 3, 40, ACTIVE, GEN1),   # 9 actions: the lane loop's second turn
    "w32_o33_a3_b127_relu": (33, 3, 32, RELU, 127, 3, 10 ** 6, 10.0, GEN1),
    "w32_o60_a18_b128_tanh": (60, 18, 32, TANH, 128, 2, 0, ACTIVE, GEN1),  # one pass of 128 rows
    "w20_o64_a8_b129_relu": (64, 8, 20, RELU, 129, 3, 1, 1e30, GEN1),     # the first row of a second pass
    "w32_o4_a9_b4096_relu": (4, 9, 32, RELU, 4096, 2, 40, ACTIVE, GEN1),  # 32 passes
    # ---- k_ppo_update_gen<2> and k_dqn_target<64>: widths 33, 40, 63, 64
    "w33_o17_a18_b129_relu": (17, 18, 33, RELU, 129, 2, 10 ** 6, ACTIVE, GEN2),
    "w40_o33_a9_b220_tanh": (33, 9, 40, TANH, 220, 3, 0, ACTIVE, GEN2),
    "w63_o60_a3_b512_relu": (60, 3, 63, RELU, 512, 2, 1, 1e30, GEN2),
    "w64_o17_a8_b4096_tanh": (17, 8, 64, TANH, 4096, 2, 10 ** 6, ACTIVE, GEN2),
    # the largest action count imb_dqn_plan accepts at width 64, d_obs 64 (tests/test_dqn_plan.py)
    "w64_o64_a35_b1_tanh": (64, 35, 64, TANH, 1, 4, 40, 1e30, GEN2),
    "w64_o64_a35_b2_relu": (64, 35, 64, RELU, 2, 3, 1, ACTIVE, GEN2),
    # ---- SQIL's own shapes: CartPole with the default [64, 64] ReLU Q-net and SB3's batch, and a tanh [32, 32] one
    "cartpole_w64_relu_b32": (4, 2, 64, RELU, 32, 3, 0, 10.0, GEN2),
    "cartpole_w32_tanh_b220": (4, 2, 32, TANH, 220, 3, 1, 10.0, GEN1),
}


def _cfg(name):
    Do, A, h, act, B, G, t0, mgn, plan = CASES[name]
    return dict(name=name, Do=Do, A=A, h=h, act=act, B=B, G=G, t0=t0, mgn=mgn, plan=plan, n_l=B // 2, n_e=B - B // 2,
                seed=2000 + 31 * list(CASES).index(name))


# ---------------------------------------------------------------------------------------------------------------------
# the float64 DQN step
# ---------------------------------------------------------------------------------------------------------------------
class _PaddedHuber(th.autograd.Function):
    """smooth_l1 (beta 1) of d whose derivative clamp(d, -1, 1) is padded by e / C_GRAD where |d| < 1 + e: e bounds
    d's fp32 error, and clamp moves by up to e under it (only used for the magnitudes of the per-row terms, which
    C_GRAD scales)."""
    generate_vmap_rule = True

    @staticmethod
    def forward(d, e):
        return th.where(d.abs() < 1, 0.5 * d * d, d.abs() - 0.5)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.save_for_backward(*inputs)

    @staticmethod
    def backward(ctx, g):
        d, e = ctx.saved_tensors
        return g * (d.clamp(-1, 1) + (d.abs() < 1 + e).to(g.dtype) * e / C_GRAD), None


class _Ref:
    """The Q-net of a policy image (pi tower + action head; the value tower is zero) and one float64 TD step."""

    def __init__(self, c):
        self.c = c
        self.Do, self.A, self.h, self.relu = c["Do"], c["A"], c["h"], c["act"] == RELU
        self.pd = _desc.policy_desc(self.Do, self.A, True, self.h, False)
        self.rw = _lib.rollout_row_width(self.pd)

    def unpack(self, p):
        d, h, Do, A = self.pd, self.h, self.Do, self.A
        return (p[d.off_pi_w1:d.off_pi_b1].reshape(h, Do), p[d.off_pi_b1:d.off_pi_w2],
                p[d.off_pi_w2:d.off_pi_b2].reshape(h, h), p[d.off_pi_b2:d.off_pi_b2 + h],
                p[d.off_act_w:d.off_act_b].reshape(A, h), p[d.off_act_b:d.off_act_b + A])

    def value_tower(self, p):
        """the image's value tower and value head, which no DQN kernel may touch"""
        d = self.pd
        return np.concatenate([p[d.off_vf_w1:d.off_act_w], p[d.off_val_w:]])

    def dict64(self, p):
        return dict(zip(sqil_port.KEYS, (np.asarray(x, np.float64) for x in self.unpack(p))))

    def q(self, p, x, padded=False):
        """Q [..., A] of float64 torch parameters p; padded: the towers' derivatives padded, and the fp32 error bound
        of Q [..., A] (observations are exact fp32 inputs)"""
        w1, b1, w2, b2, w3, b3 = self.unpack(p)

        def layer(x, e, w, b):
            z = x @ w.T + b
            if not padded:
                return (th.relu(z) if self.relu else th.tanh(z)), None
            dz = w.shape[1] * U24 * (x.abs() @ w.abs().T + b.abs()) + e @ w.abs().T
            if self.relu:
                return _KinkReLU.apply(z, dz.detach()), (dz * (z > -dz)).detach()  # relu is 1-Lipschitz
            y = F._PaddedTanh.apply(z, dz.detach())
            return y, ((1 - y * y) * dz + SAT_PAD).detach()

        lat, e = layer(*layer(x, th.zeros_like(x) if padded else None, w1, b1), w2, b2)
        q = lat @ w3.T + b3
        if not padded:
            return q, None
        return q, (self.h * U24 * (lat.abs() @ w3.abs().T + b3.abs()) + e @ w3.abs().T).detach()

    def row_loss(self, p, x, oh, y, padded=False):
        q, eq = self.q(p, x, padded)
        qa = (q * oh).sum(-1)
        d = qa - y
        if not padded:
            return th.where(d.abs() < 1, 0.5 * d * d, d.abs() - 0.5)
        return _PaddedHuber.apply(d, ((eq * oh).sum(-1) + U24 * (qa.abs() + y.abs())).detach())

    def split(self, rows):
        rows = th.as_tensor(np.asarray(rows, np.float64))
        act = rows[:, self.Do].long()
        return rows[:, :self.Do], th.nn.functional.one_hot(act, self.A).double(), rows[:, self.Do + 1], act

    def grad(self, P, rows):
        """The float64 gradient of the mean smooth L1 over the TD rows at the fp32 parameters P, its tolerance, the
        loss, the loss's tolerance and the rows' d = Q_a - y."""
        Pd = th.as_tensor(np.asarray(P, np.float64))
        x, oh, y, act = self.split(rows)
        nb = x.shape[0]
        g, mag = th.zeros_like(Pd), th.zeros_like(Pd)
        gr = tfunc.vmap(tfunc.grad(self.row_loss), in_dims=(None, 0, 0, 0))
        grp = tfunc.vmap(tfunc.grad(lambda *a: self.row_loss(*a, padded=True)), in_dims=(None, 0, 0, 0))
        for i in range(0, nb, 512):
            s = slice(i, i + 512)
            gi = gr(Pd, x[s], oh[s], y[s])
            pad = grp(Pd, x[s], oh[s], y[s]) - gi  # (the pads can change a sum over units' sign pattern)
            g += gi.sum(0) / nb
            mag += (gi.abs() + pad.abs()).sum(0) / nb
        # the oracle's hand-written backward gives the same gradient
        loss, g_port = sqil_port.td_grad(self.dict64(P), x.numpy(), act.numpy(), y.numpy(), relu=self.relu)
        for k, a in zip(sqil_port.KEYS, self.unpack(g.numpy())):
            np.testing.assert_allclose(a, g_port[k], rtol=1e-9, atol=1e-12 * float(mag.max()))
        q, eq = self.q(Pd, x, padded=True)
        qa, ea = (q * oh).sum(-1), (eq * oh).sum(-1)
        d = qa - y
        cl = d.clamp(-1, 1).abs()
        row = th.where(d.abs() < 1, 0.5 * d * d, d.abs() - 0.5)
        tol_loss = float((cl * (ea + U24 * (qa.abs() + y.abs()))).mean() + C_LOSS * (row + cl * (qa.abs() + y.abs())).mean())
        return g, C_GRAD * mag + FLOOR * float(mag.max()), float(loss), tol_loss + 1e-7, d.numpy()

    def td_targets(self, P, nobs, done, rew):
        """y in float64 and its tolerance"""
        Pd = th.as_tensor(np.asarray(P, np.float64))
        y = sqil_port.td_targets(self.dict64(P), nobs, done, rew, GAMMA, relu=self.relu)
        q, eq = self.q(Pd, th.as_tensor(nobs), padded=True)
        mx = q.max(-1).values.numpy()
        tol = GAMMA * (1 - done) * eq.max(-1).values.numpy() + 2 * U24 * (np.abs(GAMMA * mx) + np.abs(y))
        return y, tol


def _clip(g, tol_g, mgn):
    """clip_grad_norm_ on the float64 gradient: (clip, clip g, its tolerance, total)"""
    total = float(g.norm())
    clip = min(1.0, mgn / (total + 1e-6))
    gc, tol_gc = clip * g, clip * tol_g
    if mgn < 1e30:  # the clip factor is sharp only away from the threshold
        assert abs(total / mgn - 1) > 1e-3, "clip_grad_norm_ too close to its threshold for a sharp comparison"
    if clip < 1.0:  # the clip factor carries the total norm's relative error
        tol_gc = tol_gc + gc.abs() * (float((g.abs() * tol_g).sum()) / total ** 2 + 1e-6)
    return clip, gc, tol_gc, total


def _adam(st, gc, tol_gc, lr):
    """One Adam step with the kernel's constants on the float64 state st (P, M, V, t) in place, with the moments' and
    the parameters' tolerances (test_ppo_float64.Ref.step's arithmetic)."""
    st["t"] += 1
    P, M, V = st["P"], st["M"], st["V"]
    Mn = B1F * M + (1 - B1F) * gc
    Vn = B2F * V + (1 - B2F) * gc * gc
    tol_M = (1 - B1F) * tol_gc + 2 * U24 * Mn.abs()
    tol_V = (1 - B2F) * (2 * gc.abs() * tol_gc + tol_gc ** 2) + 4 * U24 * Vn.abs()
    lr = float(np.float32(lr))
    bc1, bc2 = 1.0 - 0.9 ** st["t"], 1.0 - 0.999 ** st["t"]
    eps = float(np.float32(EPS))

    def upd(m, v):
        return lr / bc1 * m / (th.sqrt(v.clamp(min=0)) / np.sqrt(bc2) + eps)

    du = upd(Mn, Vn)
    spread = th.zeros_like(P)
    for sm in (-1, 1):
        for sv in (-1, 1):
            spread = th.maximum(spread, (upd(Mn + sm * tol_M, Vn + sv * tol_V) - du).abs())
    st["tol_P"] = spread + 1e-5 * du.abs() + 4 * U24 * P.abs()
    st["P"], st["M"], st["V"] = P - du, Mn, Vn
    st["tol_M"] = B1F * st["tol_M"] + tol_M
    st["tol_V"] = B2F * st["tol_V"] + tol_V


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _params(ref, rng):
    """An fp32 Q-net image: the tower as test_ppo_float64._make_inputs draws it (per-unit scales 0.05 .. 15, so tanh
    units saturate and sit near tanh_fast's switch), biases 0.3, the action head 0.5 / sqrt(h) (ReLU: times
    test_relu_policy.RELU_HEAD, whose latents reach the hundreds), the value tower zero."""
    d, h, Do, A = ref.pd, ref.h, ref.Do, ref.A
    P = np.zeros(d.n_params, np.float32)

    def tower(shape):
        scale = np.geomspace(0.05, 15.0, shape[0]) if shape[0] > 1 else np.array([4.0])
        return rng.standard_normal(shape) / np.sqrt(shape[1]) * rng.permutation(scale)[:, None]

    head = 0.5 * (RELU_HEAD if ref.relu else 1.0)
    for off, w in ((d.off_pi_w1, tower((h, Do))), (d.off_pi_b1, rng.standard_normal(h) * 0.3),
                   (d.off_pi_w2, tower((h, h))), (d.off_pi_b2, rng.standard_normal(h) * 0.3),
                   (d.off_act_w, rng.standard_normal((A, h)) / np.sqrt(h) * head), (d.off_act_b, rng.standard_normal(A) * 0.5)):
        P[off:off + w.size] = w.reshape(-1)
    return P


def _obs(rng, n, Do):
    """observations with per-feature offsets and spreads (test_ppo_float64._make_inputs)"""
    mu, sd = rng.normal(0.2, 0.5, Do), rng.uniform(0.5, 2.0, Do)
    return (mu + sd * rng.standard_normal((n, Do))).astype(np.float32)


def _step_rows(ref, P, rng, n):
    """n TD rows obs | action | y with y = Q_a(obs) - u: |u| in (0.05, 0.95) on even rows, (1.05, 3) on odd ones, both
    signs, so smooth L1 takes both branches in every minibatch of two rows or more (and across the steps at B = 1)"""
    obs = _obs(rng, n, ref.Do)
    act = rng.integers(0, ref.A, n)
    q = sqil_port.q_forward(ref.dict64(P), obs.astype(np.float64), relu=ref.relu)[2][np.arange(n), act]
    u = np.where(np.arange(n) % 2 == 0, rng.uniform(0.05, 0.95, n), rng.uniform(1.05, 3.0, n))
    u *= rng.choice([-1.0, 1.0], n)
    rows = np.zeros((n, ref.rw), np.float32)
    rows[:, :ref.Do], rows[:, ref.Do], rows[:, ref.Do + 1] = obs, act, q - u
    return rows


def _table(ref, rng, n):
    """a feature-major transition table [2 d_obs + n_actions + 1][n]: obs | one-hot action | next obs | done"""
    Do, A = ref.Do, ref.A
    t = np.zeros((2 * Do + A + 1, n), np.float32)
    t[:Do] = _obs(rng, n, Do).T
    t[Do + rng.integers(0, A, n), np.arange(n)] = 1.0
    t[Do + A:2 * Do + A] = _obs(rng, n, Do).T
    t[2 * Do + A] = (rng.random(n) < 0.3).astype(np.float32)
    return t


def _moments0(ref, rng):
    """nonzero starting moments (zero on the value tower, whose gradient is 0)"""
    n = ref.pd.n_params
    M = (rng.standard_normal(n) * 1e-3).astype(np.float32)
    V = (np.abs(rng.standard_normal(n)) * 1e-5).astype(np.float32)
    for a in (M, V):
        a[ref.pd.off_vf_w1:ref.pd.off_act_w] = 0
        a[ref.pd.off_val_w:] = 0
    return M, V


# ---------------------------------------------------------------------------------------------------------------------
# the kernels
# ---------------------------------------------------------------------------------------------------------------------
def _device(P, M, V, t0, n_log):
    st = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
    st[_lib.ST_PPO_STEP] = t0
    st[_lib.ST_GLOBAL_STEP] = 12345  # a word no DQN kernel may touch
    return dict(params=th.from_numpy(np.array(P)).cuda(), exp_avg=th.from_numpy(np.array(M)).cuda(),
                exp_avg_sq=th.from_numpy(np.array(V)).cuda(), state=st,
                log=th.full((max(n_log, 1), 4), float("nan"), device="cuda"))


def _step(ref, dev, rows, n_steps, lr, mgn, loss_base, with_log=True):
    c = ref.c
    _lib.dqn_step(ref.pd, dev["params"], dev["exp_avg"], dev["exp_avg_sq"], rows, c["B"], n_steps, lr, EPS, mgn,
                  dev["log"] if with_log else None, dev["state"], loss_base=loss_base, act=c["act"])


def _host(dev):
    th.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in dev.items()}


def _same_bits(a, b, what, keys=None):
    for k in keys or a:
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), f"{what}: {k} differs"


def _both_sides(d):
    ad = np.abs(d)
    return int((ad < 1).sum()), int((ad > 1).sum())


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
def test_cases_cover_both_kernels_and_activations():
    """Every case runs on the kernel it names, and both kernels run both activations."""
    seen = set()
    for name in CASES:
        c = _cfg(name)
        assert _lib.dqn_plan(_Ref(c).pd, c["B"], c["act"]) == c["plan"], name
        seen.add((c["plan"], c["act"]))
    assert seen == {(p, a) for p in (GEN1, GEN2) for a in (TANH, RELU)}


@pytest.mark.parametrize("name", list(CASES))
def test_td_rows_match_the_float64_targets(name):
    """Measurement a."""
    c = _cfg(name)
    ref, rng = _Ref(c), np.random.default_rng(c["seed"])
    Do, A, B, G, n_l, n_e = c["Do"], c["A"], c["B"], c["G"], c["n_l"], c["n_e"]
    Pt = _params(ref, rng)
    C, Ne, s0, base = 300, 77, 3, 5
    ring, expert = _table(ref, rng, C), _table(ref, rng, Ne)
    lidx, eidx = rng.integers(0, C, (s0 + G, n_l)), rng.integers(0, Ne, (s0 + G, n_e))
    cu = lambda a: th.from_numpy(np.ascontiguousarray(a)).cuda()
    state = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
    state[_lib.ST_PPO_STEP] = base + s0
    outs = []
    for st, li, ei, sb in ((state, lidx, eidx, base), (None, lidx[s0:], eidx[s0:], 0)):
        rows = th.full((G * B, ref.rw), float("nan"), device="cuda")
        _lib.dqn_target(ref.pd, cu(Pt), cu(ring), C, cu(li), cu(expert), Ne, cu(ei), n_l, n_e, G, GAMMA, R_L, R_E, rows,
                        step_base=sb, state=st, act=c["act"])
        outs.append(rows.cpu().numpy())
    _same_bits({"rows": outs[0]}, {"rows": outs[1]}, f"{name}: lists from s0 = state - step_base vs lists cut at s0")
    assert int(state[_lib.ST_PPO_STEP]) == base + s0 and not state[:_lib.ST_PPO_STEP].any()
    got = outs[0]
    assert np.isnan(got[:, Do + 2:]).all(), "the target wrote past obs | action | y"
    n_done = w = 0
    for s in range(G):
        src = np.concatenate([ring[:, lidx[s0 + s]], expert[:, eidx[s0 + s]]], 1)
        rew = np.r_[np.full(n_l, R_L), np.full(n_e, R_E)]
        done = src[2 * Do + A].astype(np.float64)
        y, tol = ref.td_targets(Pt, src[Do + A:2 * Do + A].T.astype(np.float64), done, rew)
        g = got[s * B:(s + 1) * B]
        assert np.array_equal(g[:, :Do].view(np.uint32), src[:Do].T.copy().view(np.uint32)), f"{name}: obs of step {s}"
        np.testing.assert_array_equal(g[:, Do], src[Do:Do + A].argmax(0), err_msg=f"{name}: actions of step {s}")
        dn = done == 1
        np.testing.assert_array_equal(g[dn, Do + 1], rew[dn].astype(np.float32), err_msg=f"{name}: y of done rows")
        w = max(w, F._check(g[:, Do + 1], y, tol, f"{name}: y of step {s}"))
        n_done += int(dn.sum())
    assert 0 < n_done < G * B or G * B < 16, "rows with and without done"
    print(f"{name}: worst |y deviation| / tolerance {w:.3f}")


@pytest.mark.parametrize("name", list(CASES))
def test_gradient_and_loss_through_the_adam_moments(name):
    """Measurements b and c: G steps at lr = 0 from zero moments."""
    c = _cfg(name)
    ref, rng = _Ref(c), np.random.default_rng(c["seed"] + 1)
    B, G, t0 = c["B"], c["G"], c["t0"]
    P = _params(ref, rng)
    rows = _step_rows(ref, P, rng, G * B)
    steps = [ref.grad(P, rows[s * B:(s + 1) * B]) for s in range(G)]
    sides = np.sum([_both_sides(s[4]) for s in steps], 0)
    assert sides.min() > 0, f"smooth L1's two branches: {sides} rows with |d| < 1, > 1"
    z = np.zeros_like(P)
    rows_t = th.from_numpy(rows).cuda()
    base = t0 - 2  # the log rows of this launch start at row 2: rows 0 and 1 must stay untouched
    for mgn in (1e30, 0.5 * min(float(s[0].norm()) for s in steps)):
        runs = []
        for with_log in (True, False, True):
            dev = _device(P, z, z, t0, G + 2)
            _step(ref, dev, rows_t, G, 0.0, mgn, base, with_log)
            runs.append(_host(dev))
        _same_bits(runs[0], runs[1], f"{name} mgn={mgn:g}: with / without the loss log", ["params", "exp_avg",
                                                                                             "exp_avg_sq", "state"])
        _same_bits(runs[0], runs[2], f"{name} mgn={mgn:g}: two identical launches")
        got = runs[0]
        assert np.array_equal(got["params"].view(np.uint32), P.view(np.uint32)), "lr = 0 moved a parameter"
        for k in ("exp_avg", "exp_avg_sq"):
            assert not ref.value_tower(got[k]).any(), f"{k} of the zero value tower"
        want_state = np.zeros(_lib.ST_WORDS, np.int64)
        want_state[_lib.ST_PPO_STEP], want_state[_lib.ST_GLOBAL_STEP] = t0 + G, 12345
        np.testing.assert_array_equal(got["state"], want_state)
        st = dict(P=th.from_numpy(P).double(), M=th.zeros(len(P), dtype=th.float64), V=th.zeros(len(P), dtype=th.float64),
                  t=t0, tol_M=0.0, tol_V=0.0)
        log = got["log"]
        assert np.isnan(log[:2]).all(), "a loss row below loss_base was written"
        w = 0.0
        for s, (g, tol_g, loss, tol_loss, _) in enumerate(steps):
            clip, gc, tol_gc, total = _clip(g, tol_g, mgn)
            if mgn < 1e30:
                assert total / mgn > 1.001, "clip_grad_norm_ inactive: the case does not test it"
            _adam(st, gc, tol_gc, 0.0)
            w = max(w, F._check(log[2 + s, 0], loss, tol_loss, f"{name} mgn={mgn:g}: loss of step {s}"))
        np.testing.assert_array_equal(log[2:, 1:3], 0)
        np.testing.assert_array_equal(log[2:, 3], log[2:, 0])
        w = max(w, F._check(got["exp_avg"], st["M"], st["tol_M"], f"{name} mgn={mgn:g}: exp_avg"))
        w = max(w, F._check(got["exp_avg_sq"], st["V"], st["tol_V"], f"{name} mgn={mgn:g}: exp_avg_sq"))
        print(f"{name} mgn={mgn:g}: worst |deviation| / tolerance {w:.3f}")


@pytest.mark.parametrize("name", list(CASES))
def test_adam_step_teacher_forced(name):
    """Measurement d."""
    c = _cfg(name)
    ref, rng = _Ref(c), np.random.default_rng(c["seed"] + 2)
    B, G, t0 = c["B"], c["G"], c["t0"]
    k, lr = G // 2, 1e-3
    P = _params(ref, rng)
    M, V = _moments0(ref, rng)
    rows = _step_rows(ref, P, rng, G * B)
    rows_t = th.from_numpy(rows).cuda()
    mgn = c["mgn"]
    if mgn == ACTIVE:
        mgn = 0.5 * min(float(ref.grad(P, rows[s * B:(s + 1) * B])[0].norm()) for s in range(k + 1))
    full = _device(P, M, V, t0, G)
    _step(ref, full, rows_t, G, lr, mgn, t0)
    full = _host(full)
    dev = _device(P, M, V, t0, G)
    _step(ref, dev, rows_t[:k * B], k, lr, mgn, t0)
    a = _host(dev)
    _step(ref, dev, rows_t[k * B:(k + 1) * B], 1, lr, mgn, t0)
    b = _host(dev)
    if G > k + 1:
        _step(ref, dev, rows_t[(k + 1) * B:], G - k - 1, lr, mgn, t0)
    _same_bits(full, _host(dev), f"{name}: one launch of {G} steps vs launches of {k}, 1, {G - k - 1}")
    assert int(a["state"][_lib.ST_PPO_STEP]) == t0 + k and int(b["state"][_lib.ST_PPO_STEP]) == t0 + k + 1
    # step k + 1 in float64 from the state the k-step launch left
    g, tol_g, loss, tol_loss, d = ref.grad(a["params"], rows[k * B:(k + 1) * B])
    clip, gc, tol_gc, _ = _clip(g, tol_g, mgn)
    st = dict(P=th.from_numpy(a["params"]).double(), M=th.from_numpy(a["exp_avg"]).double(),
              V=th.from_numpy(a["exp_avg_sq"]).double(), t=t0 + k, tol_M=0.0, tol_V=0.0)
    _adam(st, gc, tol_gc, lr)
    w = F._check(b["log"][k, 0], loss, tol_loss, f"{name}: loss of step {k}")
    w = max(w, F._check(b["exp_avg"], st["M"], st["tol_M"] + 2 * U24 * st["M"].abs(), f"{name}: exp_avg"))
    w = max(w, F._check(b["exp_avg_sq"], st["V"], st["tol_V"] + 2 * U24 * st["V"].abs(), f"{name}: exp_avg_sq"))
    w = max(w, F._check(b["params"], st["P"], st["tol_P"], f"{name}: parameters"))
    moved = np.abs(b["params"].astype(np.float64) - a["params"])
    assert np.median(moved[ref.pd.off_pi_w1:ref.pd.off_vf_w1]) > 1e-6, "the step did not move the parameters"
    assert not ref.value_tower(b["params"]).any(), "the zero value tower moved"
    print(f"{name}: k={k} t0={t0} clip={clip:.3f}: worst |deviation| / tolerance {w:.3f}")


@pytest.mark.parametrize("name", list(CASES))
def test_graph_replay_gives_the_eager_bits(name):
    """Measurement e: the target and the TD steps of two learn() iterations in a row, as DeviceDQN runs them (state =
    step_base = loss_base = the step count the learn() starts at, so the second iteration reads its lists and writes
    its losses at offset G), eagerly and from one captured graph replayed twice."""
    c = _cfg(name)
    ref, rng = _Ref(c), np.random.default_rng(c["seed"] + 3)
    B, G, t0, n_l, n_e = c["B"], c["G"], c["t0"], c["n_l"], c["n_e"]
    P = _params(ref, rng)
    Pt = P + (0.05 * rng.standard_normal(P.size) * (P != 0)).astype(np.float32)
    M, V = _moments0(ref, rng)
    C, Ne = 300, 77
    cu = lambda a: th.from_numpy(np.ascontiguousarray(a)).cuda()
    ring, expert, tgt = cu(_table(ref, rng, C)), cu(_table(ref, rng, Ne)), cu(Pt)
    lidx, eidx = cu(rng.integers(0, C, (2 * G, n_l))), cu(rng.integers(0, Ne, (2 * G, n_e)))
    mgn = 1.0 if c["mgn"] == ACTIVE else c["mgn"]
    dev = _device(P, M, V, t0, 2 * G)
    dev["rows"] = th.zeros(G * B, ref.rw, device="cuda")
    init = {k: v.clone() for k, v in dev.items()}

    def iteration():
        _lib.dqn_target(ref.pd, tgt, ring, C, lidx, expert, Ne, eidx, n_l, n_e, G, 0.99, 0.0, 1.0, dev["rows"],
                        step_base=t0, state=dev["state"], act=c["act"])
        _step(ref, dev, dev["rows"], G, 2e-3, mgn, t0)

    def reset():
        for k, v in init.items():
            dev[k].copy_(v)

    eager = []
    for _ in range(2):
        reset()
        iteration()
        iteration()
        eager.append(_host(dev))
    _same_bits(eager[0], eager[1], f"{name}: two identical eager runs")
    assert int(eager[0]["state"][_lib.ST_PPO_STEP]) == t0 + 2 * G and not np.isnan(eager[0]["log"]).any()
    graph = th.cuda.CUDAGraph()
    reset()
    with th.cuda.graph(graph):
        iteration()
    reset()
    graph.replay()
    graph.replay()
    _same_bits(eager[0], _host(dev), f"{name}: graph replays vs eager launches")
