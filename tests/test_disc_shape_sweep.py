"""The discriminator kernels at every network shape they accept, against a float64 evaluation of the same network.

imb_disc_fwd_bwd runs one of four kernels (imb_disc_plan): the wgmma tensor-core kernel, or the fp32-FFMA tiled kernel
with 128-row tiles and two CTAs per SM, 256-row tiles, or 128-row tiles and one CTA per SM.  Inside the FFMA kernel the
hidden width (JP = 32 / 64 columns), the input width (KP = 32 / 64), the shaped net's three passes, the done and log pi
slots and n_hidden = 0 / 1 / 2 each take their own code; imb_reward_forward has its own H = 32 / 64 kernel with a
grid-stride loop.  Every shape below is run at row counts from one row to several tiles per CTA, and checked row by row
against float64 arithmetic built from the same fp32 parameters and the same fp32 batch:

  logit = base(s, a, s', d) [+ gamma (1 - d) Phi(s') - Phi(s)] [- log pi]      (RunningNorm inputs in the nets that have it)
  loss  = loss_scale * sum_i BCE-with-logits(logit_i, y_i),  y_i = 1 for the first n_expert rows

with the gradient from float64 autograd and the statistics as the reference's compute_train_stats computes them
(oracle/disc_port.train_stats_port).  Tolerances: logits per row within north_star's 1e-5 relative, with an absolute
floor of 1e-6 of the largest |logit| for rows that cancel to ~0; gradients rtol 2e-4, atol 2e-6 max|g|, plus 3e-4 of the
sum of the absolute per-row terms for sums that cancel over many rows (at n <= 1000 one mislabelled row moves the
final bias gradient by loss_scale = 1/n, far outside that); counts exact except for rows whose float64 logit lies inside
the logit tolerance of zero, whose sign fp32 rounding decides.
"""
import zlib

import numpy as np
import pytest
import torch as th

from imitation_b200 import _desc, _lib

pytestmark = pytest.mark.gpu

LOGIT_RTOL, LOGIT_ATOL = 1e-5, 1e-6   # north_star; LOGIT_ATOL is scaled by max(1, max |logit|)
GRAD_RTOL, GRAD_ATOL = 2e-4, 2e-6     # GRAD_ATOL is scaled by max |gradient|
# a gradient summed over 10^5 rows that cancels to near zero carries the rounding of its large terms, and of the rows
# where a hidden pre-activation within rounding of zero takes the other side of its ReLU in fp32 (a few rows per 10^5):
# each parameter's gradient may also deviate by GRAD_MAG_RTOL of sum_i |w_i d logit_i / d theta| (_abs_grad).  With the
# BCE weights w_i = (sigmoid - y) / n that sum is an average over rows, so one mislabelled row (1 / n) stays far outside.
GRAD_MAG_RTOL = 3e-4
EPS32 = 2.0 ** -24

# name -> disc_desc keyword arguments (+ "onehot": the action rows hold one-hot actions)
SHAPES = {
    # tensor cores: unshaped 32x32, din <= 31, no done input, no log pi
    "tc_din1": dict(d_obs=1, d_act=0, use_action=False),
    "tc_din1_norm": dict(d_obs=1, d_act=0, use_action=False, normalize_input=True),
    "tc_din7": dict(d_obs=4, d_act=3),
    "tc_din7_norm": dict(d_obs=4, d_act=3, normalize_input=True),
    "tc_din31": dict(d_obs=20, d_act=11),
    "tc_din31_norm": dict(d_obs=20, d_act=11, normalize_input=True),
    # FFMA, JP = 32: n_hidden 0 / 1 / 2, widths that are not a multiple of 8, the done input
    "h0": dict(d_obs=17, d_act=6, hid_sizes=()),
    "h16_norm": dict(d_obs=17, d_act=6, hid_sizes=(16,), normalize_input=True),
    "h32": dict(d_obs=17, d_act=6, hid_sizes=(32,)),
    "h20x20_next_done": dict(d_obs=4, d_act=2, hid_sizes=(20, 20), use_next_state=True, use_done=True),
    "h32x32_next_done": dict(d_obs=17, d_act=6, use_next_state=True, use_done=True, normalize_input=True),
    # FFMA, JP = 64
    "cartpole_64x64": dict(d_obs=4, d_act=2, hid_sizes=(64, 64), normalize_input=True, onehot=True),
    "h40x64": dict(d_obs=11, d_act=3, hid_sizes=(40, 64)),
    # FFMA, KP = 64: the Ant shape, the widest input (din 64), and the 256-row-tile kernel
    "ant_32x32": dict(d_obs=27, d_act=8, normalize_input=True),
    "din64_next": dict(d_obs=28, d_act=8, use_next_state=True),
    "ant_16": dict(d_obs=27, d_act=8, hid_sizes=(16,), normalize_input=True),
    # shaped AIRL nets: three passes, done flags, log pi, gamma != 1
    "airl_r32_p32x32": dict(d_obs=5, d_act=2, hid_sizes=(32,), potential_hid_sizes=(32, 32), shaped=True,
                            normalize_input=True, gamma=0.9, subtract_logp=True),
    "airl_r32x32_p32": dict(d_obs=17, d_act=6, hid_sizes=(32, 32), potential_hid_sizes=(32,), shaped=True,
                            normalize_input=True, gamma=0.9, subtract_logp=True),
}
BIG = "big"  # 4 x (CTAs of the two-CTAs-per-SM grid) x 128 rows + 77: every CTA of every kernel loops >= 4 times
ROWS = [1, 127, 128, 129, 257, BIG]
LONG = {"tc_din31_norm": [1 << 18], "ant_32x32": [1 << 18]}
CASES = [(s, n) for s in SHAPES for n in ROWS + LONG.get(s, [])]


def _rows(n) -> int:
    if n == BIG:
        sms = th.cuda.get_device_properties(0).multi_processor_count
        return 4 * 2 * sms * 128 + 77
    return n


def _desc_of(name):
    kw = {k: v for k, v in SHAPES[name].items() if k != "onehot"}
    return _desc.disc_desc(**kw)


def _hid(name):
    return tuple(SHAPES[name].get("hid_sizes", (32, 32))), tuple(SHAPES[name].get("potential_hid_sizes", (32, 32)))


# ---------------------------------------------------------------------------------------------------------------------
# plan coverage (host only)
# ---------------------------------------------------------------------------------------------------------------------
def test_sweep_covers_every_kernel():
    """Every imb_disc_fwd_bwd kernel occurs in the sweep: 1 tensor cores, 2 / 3 / 4 the FFMA kernel with 128-row tiles
    at two CTAs per SM, 256-row tiles, 128-row tiles at one CTA per SM."""
    plans = {}
    for name, n in CASES:
        plans[(name, n)] = _lib.disc_plan(_desc_of(name), 135245 if n == BIG else n)
    table = "\n".join(f"  {name:20s} n={n!s:>7s} -> {p}" for (name, n), p in plans.items())
    print("\n(shape, n) -> imb_disc_plan\n" + table)
    assert set(plans.values()) == {1, 2, 3, 4}, table
    # n_hidden 0 / 1 / 2, JP 32 / 64, KP 32 / 64 each occur on an FFMA kernel
    ffma = [s for (s, _), p in plans.items() if p != 1]
    assert {len(_hid(s)[0]) for s in ffma} == {0, 1, 2}
    assert any(max(_hid(s)[0] + (0,)) > 32 for s in ffma) and any(_desc_of(s).base.din > 32 for s in ffma)


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def _layout(d):
    Do, Da = d.d_obs, d.d_act
    return dict(obs=list(range(Do)), act=list(range(Do, Do + Da)), nobs=list(range(Do + Da, 2 * Do + Da)),
                done=2 * Do + Da, logp=2 * Do + Da + 1)


def _base_rows(d):
    lay = _layout(d)
    rows = []
    rows += lay["obs"] if d.use_state else []
    rows += lay["act"] if d.use_action else []
    rows += lay["nobs"] if d.use_next_state else []
    rows += [lay["done"]] if d.use_done else []
    return rows


def _make_inputs(name, n, gen, mode="wide"):
    """fp32 parameters, feature-major batch (zero padding), norm state and counts.

    mode "wide": eval-mode statistics far from zero mean / unit variance -- feature means around +-50, std around 0.01,
    and one zero-variance feature (obs 0); "train": moderate data and statistics (the kernels' fp32 running statistics
    are then compared with float64 ones, which a mean of 50 over a std of 0.01 would turn into 5e-4 input errors);
    "plain": unnormalised standard-normal inputs."""
    kw, d = SHAPES[name], _desc_of(name)
    hid, pot = _hid(name)
    norm = bool(d.base.has_norm)
    if not norm:
        mode = "plain"
    dev = "cuda"
    lay = _layout(d)
    bw, ld = _desc.batch_rows(d.d_obs, d.d_act), _desc.batch_ld(n)

    def u(*shape):
        return th.rand(*shape, device=dev, generator=gen, dtype=th.float64) * 2 - 1

    # per batch row: generating mean / std; binary rows (one-hot actions, done) are marked
    mu, sd = th.zeros(bw, device=dev, dtype=th.float64), th.ones(bw, device=dev, dtype=th.float64)
    binary = th.zeros(bw, dtype=th.bool)
    feats = lay["obs"] + lay["act"]
    if mode == "wide":
        mu[feats] = th.sign(u(len(feats))) * 50 + u(len(feats))
        sd[feats] = 0.01 * (1 + 0.5 * u(len(feats)))
        sd[0] = 0.001
    elif mode == "train":
        mu[feats] = 3 * u(len(feats))
        sd[feats] = 1.25 + 0.75 * u(len(feats))
    mu[lay["nobs"]], sd[lay["nobs"]] = mu[lay["obs"]], sd[lay["obs"]]
    batch = th.zeros(bw, ld, device=dev)
    z = th.randn(bw, n, device=dev, generator=gen, dtype=th.float64)
    batch[:, :n] = (mu[:, None] + sd[:, None] * z).float()
    if kw.get("onehot"):
        a = th.randint(0, d.d_act, (n,), device=dev, generator=gen)
        batch[lay["act"], :n] = th.nn.functional.one_hot(a, d.d_act).T.float()
        binary[lay["act"]] = True
    batch[lay["done"], :n] = (th.rand(n, device=dev, generator=gen) < 0.3).float()
    binary[lay["done"]] = True
    batch[lay["logp"], :n] = (0.5 * th.randn(n, device=dev, generator=gen) - 1).float()

    # parameters: uniform, scaled by 1 / sqrt(fan-in) so that logits are O(1)
    shapes = _desc.mlp_param_shapes(d.base.din, hid) + (_desc.mlp_param_shapes(d.d_obs, pot) if d.shaped else [])
    ps = []
    for _, s in shapes:
        fan = s[1] if len(s) == 2 else 1
        ps.append((u(int(np.prod(s))) * (1.7 / np.sqrt(fan) if len(s) == 2 else 0.5)).float())
    P = th.cat(ps).contiguous()
    assert P.numel() == d.n_params

    # running statistics [base mean | base var | potential mean | potential var], counts [base, potential]
    def stats(rows, zero_var_row):
        m = th.empty(len(rows), device=dev, dtype=th.float64)
        v = th.empty(len(rows), device=dev, dtype=th.float64)
        for i, r in enumerate(rows):
            if binary[r]:
                m[i], v[i] = 0.5, 0.25
            else:
                m[i] = mu[r] + (0.3 if mode == "wide" else 0.5) * sd[r] * u(1)[0]
                v[i] = (sd[r] * (1.0 + 0.4 * u(1)[0])) ** 2
        if mode == "wide" and zero_var_row in rows:
            i = rows.index(zero_var_row)
            m[i], v[i] = mu[zero_var_row], 0.0
        return [m, v]

    parts = []
    if norm:
        parts += stats(_base_rows(d), 0)
        if d.shaped:
            parts += stats(lay["obs"], 0)
    NS = th.cat(parts).float().contiguous() if parts else th.zeros(2, device=dev)
    NC = th.tensor([3000, 3000 if d.shaped else 0], dtype=th.int32, device=dev)
    return d, P, batch, ld, NS, NC


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------------------------------
def _mlp64(x, P, off, hid, norm, eps, trace):
    """build_mlp in float64 on the flat parameter vector P from offset `off`: [RunningNorm] -> (Linear, ReLU)* -> Linear.
    Each Linear appends (parameter offset, fan-in, fan-out, its input, its output) to `trace`."""
    if norm is not None:
        x = (x - norm[0]) / th.sqrt(norm[1] + eps)
    h, prev = x, x.shape[1]
    for w in hid:
        z = h @ P[off:off + w * prev].view(w, prev).T + P[off + w * prev:off + w * prev + w]
        trace.append((off, prev, w, h, z))
        h = th.relu(z)
        off += w * prev + w
        prev = w
    z = h @ P[off:off + prev] + P[off + prev]
    trace.append((off, prev, 1, h, z))
    return z


def _abs_grad(trace, logit, rw, n_params):
    """per parameter: sum over rows (and passes) of |rw_i d logit_i / d theta|, the magnitude the fp32 rounding of a
    gradient summed over many rows scales with -- a gradient that cancels to near zero over 10^5 rows carries the
    rounding of its large terms"""
    ds = th.autograd.grad(logit.sum(), [t[4] for t in trace], retain_graph=True)
    A = th.zeros(n_params, dtype=th.float64, device="cuda")
    for (off, fin, fout, h, _), dz in zip(trace, ds):
        dz = dz.reshape(-1, fout).abs() * rw.abs()[:, None]
        A[off:off + fout * fin] += (dz.T @ h.detach().abs()).reshape(-1)
        A[off + fout * fin:off + fout * fin + fout] += dz.sum(0)
    return A


def _shape_combine(r, phi_next, phi_now, gamma, done):
    """ShapedRewardNet.forward: r + gamma (1 - done) Phi(s') - Phi(s)"""
    return r + gamma * (1 - done) * phi_next - phi_now


def _labels(n, n_expert):
    y = th.zeros(n, dtype=th.float64, device="cuda")
    y[:n_expert] = 1
    return y


def _row_mask(n):
    """rows the loss, its gradient and the statistics sum over"""
    return th.ones(n, dtype=th.float64, device="cuda")


def _norms64(d, NS):
    """eval-mode statistics per pass: base, Phi(s'), Phi(s) (the two potential passes share one normaliser)"""
    if not d.base.has_norm:
        return {"base": None, "pot_next": None, "pot_now": None}
    S = NS.double()
    din, Do = d.base.din, d.d_obs
    base = (S[:din], S[din:2 * din])
    pot = (S[2 * din:2 * din + Do], S[2 * din + Do:2 * din + 2 * Do]) if d.shaped else None
    return {"base": base, "pot_next": pot, "pot_now": pot}


def _ref_net(name, d, P, X, norms, trace=None):
    """float64 (raw net output, logit) over the columns X [bw, n]"""
    trace = [] if trace is None else trace
    hid, pot = _hid(name)
    lay = _layout(d)
    x = X[_base_rows(d)].T
    eps_b, eps_p = float(d.base.norm_eps), float(d.potential.norm_eps)
    raw = _mlp64(x, P, 0, hid, norms["base"], eps_b, trace)
    if d.shaped:
        off = d.potential.param_off
        phi_next = _mlp64(X[lay["nobs"]].T, P, off, pot, norms["pot_next"], eps_p, trace)
        phi_now = _mlp64(X[lay["obs"]].T, P, off, pot, norms["pot_now"], eps_p, trace)
        raw = _shape_combine(raw, phi_next, phi_now, float(d.gamma), X[lay["done"]])
    logit = raw - X[lay["logp"]] if d.subtract_logp else raw
    return raw, logit


def _softplus64(x):
    return th.clamp(x, min=0) + th.log1p(th.exp(-x.abs()))


def _ref_sums(logit, y, mask):
    """[loss sum, entropy sum, expert rows predicted expert, generator rows predicted generator, rows predicted expert]"""
    sp = _softplus64(logit)
    pe = (logit >= 0).double()
    return th.stack([(mask * (sp - logit * y)).sum(), (mask * (sp - logit * th.sigmoid(logit))).sum(),
                     (mask * y * pe).sum(), (mask * (1 - y) * (1 - pe)).sum(), (mask * pe).sum()])


# ---------------------------------------------------------------------------------------------------------------------
# kernel calls and checks
# ---------------------------------------------------------------------------------------------------------------------
def _stats_offset(d):
    """float offset of the reduced statistic sums in the workspace (ws_layout in csrc/imb_disc.cu)"""
    return (d.n_params + 31) // 32 * 32


def _ws(d):
    return th.zeros(_lib.disc_workspace_floats(d), device="cuda")


def _fwd_bwd(d, P, NS, batch, ld, n, n_exp, grad_out=None, flags=0, ws=None, zero_grad=True):
    """one imb_disc_fwd_bwd + imb_disc_reduce: (logits, accumulated gradient, the five statistic sums, workspace)"""
    ws = _ws(d) if ws is None else ws
    logits = th.full((n,), float("nan"), device="cuda")
    grad = th.full((d.n_params,), float("nan"), device="cuda")
    _lib.disc_fwd_bwd(d, P, NS, batch, ld, n, n_exp, 1.0 / n, grad_out, logits,
                      flags | (_lib.IMB_F_ZERO_GRAD if zero_grad else 0), ws)
    _lib.disc_reduce(d, ws, grad)
    o = _stats_offset(d)
    return logits, grad, ws[o:o + 5].clone(), ws


def _train_stats(d, ws, P):
    """the nine statistics imb_disc_adam reports for the last minibatch (the Adam step goes to a copy)"""
    out = th.full((16,), -1.0, device="cuda")
    st = th.zeros(_lib.ST_WORDS, dtype=th.int64, device="cuda")
    opt = _lib.Adam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)
    _lib.disc_adam(d, opt, P.clone(), th.zeros_like(P), th.zeros_like(P), None, 1.0, ws, st, out)
    return out[:9].cpu().double().numpy()


def _logit_tol(want):
    return LOGIT_RTOL * want.abs() + LOGIT_ATOL * max(1.0, float(want.abs().max()))


def _assert_rows(got, want, tol, what):
    diff = (got.double() - want).abs()
    bad = ~(diff <= tol)  # NaN fails too
    if bool(bad.any()):
        i = int(th.nonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {len(want)} rows off; first row {i}: got {float(got[i])!r}, "
                             f"want {float(want[i])!r}, tolerance {float(tol[i]):.3g}")


def _assert_grad(got, want, what, mag=None):
    """rtol 2e-4, atol 2e-6 max|g|, plus GRAD_MAG_RTOL of `mag` (_abs_grad)"""
    tol = GRAD_RTOL * want.abs() + GRAD_ATOL * float(want.abs().max())
    if mag is not None:
        tol = tol + GRAD_MAG_RTOL * mag
    _assert_rows(got, want, tol, what)


def _n_expert_values(n):
    """none, all, and one in the middle of a later tile"""
    mid = min(n - 1, 128 * max(0, (n - 1) // 128 - 1) + 61)
    return sorted({0, n, max(mid, 0)})


def _check_case(name, d, P, NS, batch, ld, n, norms, what, flags=0, ws=None, forward=True):
    from oracle.disc_port import train_stats_port

    X = batch[:, :n].double()
    Pl = P.double().requires_grad_(True)
    trace = []
    raw, lg = _ref_net(name, d, Pl, X, norms, trace)
    want_l = lg.detach()
    tol_l = _logit_tol(want_l)
    amb = want_l.abs() <= tol_l  # rows whose predicted class fp32 rounding may decide
    mask = _row_mask(n)
    for n_exp in _n_expert_values(n):
        tag = f"{what} n={n} n_expert={n_exp}"
        logits, grad, sums, w = _fwd_bwd(d, P, NS, batch, ld, n, n_exp, flags=flags, ws=ws)
        _assert_rows(logits, want_l, tol_l, f"{tag} logits")
        y = _labels(n, n_exp)
        loss = (mask * (_softplus64(lg) - lg * y)).sum() / n
        mag = _abs_grad(trace, lg, mask * (th.sigmoid(want_l) - y) / n, d.n_params)
        _assert_grad(grad, th.autograd.grad(loss, Pl, retain_graph=True)[0], f"{tag} gradient", mag)
        # the five sums: counts exact but for rows inside the logit tolerance of zero; loss and entropy within the
        # logits' own deviation (|d bce / d logit| <= 1, |d entropy / d logit| <= 1) plus fp32 rounding of each term
        # (sp and logit * y or logit * sigmoid cancel for large |logit|: a few ulp of |logit|) and of the summation
        got = sums.cpu().double().numpy()
        want = _ref_sums(want_l, y, mask).cpu().numpy()
        yb = y.bool()
        slack = np.array([float((amb & yb).sum()), float((amb & ~yb).sum()), float(amb.sum())])
        assert np.all(np.abs(got[2:] - want[2:]) <= slack), (tag, "counts", got[2:], want[2:], slack)
        dl = float((logits.double() - want_l).abs().sum())
        round_tol = 4 * EPS32 * float((want_l.abs() + 1).sum())
        for k, nm in ((0, "loss"), (1, "entropy")):
            tol = dl + round_tol + 4e-6 * abs(want[k])
            assert abs(got[k] - want[k]) <= tol, (tag, nm, got[k], want[k], tol)
        # the nine statistics: the reference's formulas (NaN accuracy without expert rows, max(1, n_gen))
        ref = train_stats_port(want_l.cpu(), y.cpu(), loss.detach().cpu())
        order = ["disc_loss", "disc_acc", "disc_acc_expert", "disc_acc_gen", "disc_entropy",
                 "disc_proportion_expert_true", "disc_proportion_expert_pred", "n_expert", "n_generated"]
        want9 = np.array([ref[k] for k in order])
        n_gen = n - n_exp
        tol9 = np.array([(dl + round_tol) / n + 4e-6 * abs(want[0]) / n, slack[2] / n, slack[0] / max(n_exp, 1),
                         slack[1] / max(n_gen, 1), (dl + round_tol) / n + 4e-6 * abs(want[1]) / n, 0, slack[2] / n,
                         0, 0]) + 1e-6 * np.abs(np.nan_to_num(want9))
        got9 = _train_stats(d, w, P)
        assert np.array_equal(np.isnan(got9), np.isnan(want9)), (tag, got9, want9)
        ok = np.isnan(want9) | (np.abs(got9 - np.nan_to_num(want9)) <= tol9)
        assert ok.all(), (tag, "statistics", [order[i] for i in np.nonzero(~ok)[0]], got9, want9)
    # grad_out (the preference-comparisons path): dL/dlogit given, weight gradients of sum grad_out * logit
    g = th.rand(n, device="cuda", generator=th.Generator(device="cuda").manual_seed(n)) * 2 - 1
    logits, grad, _, _ = _fwd_bwd(d, P, NS, batch, ld, n, n // 2, grad_out=g, flags=flags, ws=ws)
    _assert_rows(logits, want_l, tol_l, f"{what} n={n} grad_out logits")
    _assert_grad(grad, th.autograd.grad((g.double() * lg).sum(), Pl, retain_graph=True)[0], f"{what} n={n} grad_out",
                 _abs_grad(trace, lg, g.double(), d.n_params))
    if forward:
        _check_reward_forward(d, P, NS, batch, ld, n, raw.detach(), want_l, f"{what} n={n}")


def _check_reward_forward(d, P, NS, batch, ld, n, raw, logit, what):
    """imb_reward_forward, out modes 0 (raw output), 1 (logit), 2 (GAIL reward softplus(logit))"""
    for mode, want in ((0, raw), (1, logit), (2, _softplus64(logit))):
        out = th.full((n,), float("nan"), device="cuda")
        _lib.reward_forward(d, P, NS, batch, ld, n, mode, out)
        tol = _logit_tol(logit if mode else raw) + (LOGIT_RTOL * want if mode == 2 else 0)
        _assert_rows(out, want, tol, f"{what} reward_forward mode {mode}")


# ---------------------------------------------------------------------------------------------------------------------
# the sweep
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", CASES, ids=[f"{s}-{n}" for s, n in CASES])
def test_disc_kernels_match_fp64(name, n):
    """logits per row, gradients, sums and statistics for n_expert in {0, n, mid-tile}, the grad_out path and
    imb_reward_forward's three modes, on the kernel imb_disc_plan names"""
    n = _rows(n)
    gen = th.Generator(device="cuda").manual_seed(zlib.crc32(f"{name}/{n}".encode()))
    d, P, batch, ld, NS, NC = _make_inputs(name, n, gen)
    what = f"{name} (plan {_lib.disc_plan(d, n)})"
    _check_case(name, d, P, NS, batch, ld, n, _norms64(d, NS), what)
    if _lib.disc_plan(d, n) == _lib.PLAN_TC and n <= 257:  # the FFMA kernel on the same shape
        _check_case(name, d, P, NS, batch, ld, n, _norms64(d, NS), f"{name} (NO_TENSOR)", flags=_lib.IMB_F_NO_TENSOR,
                    forward=False)


def _final_layers(name, d):
    """index ranges of the final Linear layers (base, and potential when shaped) in the flat parameter vector"""
    hid, pot = _hid(name)
    out = []
    for off, din, h in ((0, d.base.din, hid),) + (((d.potential.param_off, d.d_obs, pot),) if d.shaped else ()):
        n = sum(int(np.prod(s)) for _, s in _desc.mlp_param_shapes(din, h))
        last = h[-1] if h else din
        out.append((off + n - last - 1, off + n))
    return out


@pytest.mark.parametrize("name", ["tc_din7_norm", "tc_din31", "h0", "h32", "cartpole_64x64", "ant_16",
                                  "airl_r32x32_p32"])
@pytest.mark.parametrize("n", [257, BIG])
def test_saturated_logits(name, n):
    """final layers scaled so that |logit| reaches ~80: loss, entropy and gradient where softplus and logit * y (or
    logit * sigmoid) cancel"""
    n = _rows(n)
    gen = th.Generator(device="cuda").manual_seed(7 + n)
    d, P, batch, ld, NS, NC = _make_inputs(name, n, gen)
    norms = _norms64(d, NS)
    _, lg = _ref_net(name, d, P.double(), batch[:, :n].double(), norms)
    s = 80.0 / float(lg.abs().max())
    for a, b in _final_layers(name, d):
        P[a:b] *= s
    _, lg = _ref_net(name, d, P.double(), batch[:, :n].double(), norms)
    assert float(lg.abs().max()) > 50
    _check_case(name, d, P, NS, batch, ld, n, norms, f"{name} saturated", forward=False)


# ---------------------------------------------------------------------------------------------------------------------
# padding, workspace reuse, accumulation, determinism
# ---------------------------------------------------------------------------------------------------------------------
def _bits(*ts):
    return [t.detach().cpu().clone() for t in ts]


def _assert_same_bits(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert th.equal(x.view(th.int32) if x.dtype == th.float32 else x, y.view(th.int32) if y.dtype == th.float32 else y), \
            f"{what}: output {i} differs"


@pytest.mark.parametrize("name", ["tc_din7_norm", "h20x20_next_done", "cartpole_64x64", "ant_16", "airl_r32_p32x32"])
def test_padding_reuse_accumulation_determinism(name):
    big = _rows(BIG)
    gen = th.Generator(device="cuda").manual_seed(11)
    d, P, batch, ld, NS, NC = _make_inputs(name, 300, gen)
    n, n_exp = 300, 189
    ref = _bits(*_fwd_bwd(d, P, NS, batch, ld, n, n_exp)[:3])
    # determinism: the same call on a fresh workspace gives the same bits
    _assert_same_bits(_bits(*_fwd_bwd(d, P, NS, batch, ld, n, n_exp)[:3]), ref, f"{name} repeat")

    # padding columns [n, ld) are never read: NaN there changes no logit, gradient, statistic or norm update
    nanb = batch.clone()
    nanb[:, n:] = float("nan")
    _assert_same_bits(_bits(*_fwd_bwd(d, P, NS, nanb, ld, n, n_exp)[:3]), ref, f"{name} NaN padding")
    for mode in (0, 1, 2):
        o1, o2 = th.empty(n, device="cuda"), th.empty(n, device="cuda")
        _lib.reward_forward(d, P, NS, batch, ld, n, mode, o1)
        _lib.reward_forward(d, P, NS, nanb, ld, n, mode, o2)
        _assert_same_bits(_bits(o1), _bits(o2), f"{name} NaN padding reward_forward {mode}")
    if d.base.has_norm:
        outs = []
        for b in (batch, nanb):
            ns, nc, ws = NS.clone(), NC.clone(), _ws(d)
            _lib.disc_norm_update(d, b, ld, n, ns, nc, ws)
            outs.append(_bits(ns, nc, *_fwd_bwd(d, P, ns, b, ld, n, n_exp, flags=_lib.IMB_F_TRAIN_NORM, ws=ws)[:3]))
        _assert_same_bits(outs[0], outs[1], f"{name} NaN padding, training mode")

    # one workspace, a large launch then a small one: only the last launch's partials are reduced
    gb = th.Generator(device="cuda").manual_seed(12)
    _, _, bigb, bld, _, _ = _make_inputs(name, big, gb)
    ws = _ws(d)
    _fwd_bwd(d, P, NS, bigb, bld, big, big // 3, ws=ws)
    l, g, s, ws = _fwd_bwd(d, P, NS, batch, ld, n, n_exp, ws=ws)
    _assert_same_bits(_bits(l, g, s), ref, f"{name} workspace reused after n={big}")
    assert np.array_equal(_train_stats(d, ws, P), _train_stats(d, _fwd_bwd(d, P, NS, batch, ld, n, n_exp)[3], P))

    # the tensor-core and FFMA kernels alternating on one workspace
    if _lib.disc_plan(d, n) == _lib.PLAN_TC:
        ffma = _bits(*_fwd_bwd(d, P, NS, batch, ld, n, n_exp, flags=_lib.IMB_F_NO_TENSOR)[:3])
        for k in range(4):
            fl = _lib.IMB_F_NO_TENSOR if k % 2 else 0
            got = _bits(*_fwd_bwd(d, P, NS, batch, ld, n, n_exp, flags=fl, ws=ws)[:3])
            _assert_same_bits(got, ffma if k % 2 else ref, f"{name} alternating kernels, call {k}")

    # gradient accumulation over minibatches without IMB_F_ZERO_GRAD: accumulator + this minibatch's sum, in fp32
    gm = th.Generator(device="cuda").manual_seed(13)
    _, _, b2, ld2, _, _ = _make_inputs(name, 200, gm)
    ws = _ws(d)
    _, g1, _, _ = _fwd_bwd(d, P, NS, batch, ld, n, n_exp, ws=ws)
    _, g12, _, _ = _fwd_bwd(d, P, NS, b2, ld2, 200, 100, ws=ws, zero_grad=False)
    _, g2, _, _ = _fwd_bwd(d, P, NS, b2, ld2, 200, 100)
    _assert_same_bits(_bits(g12), _bits(g1 + g2), f"{name} accumulation")
    Pl = P.double().requires_grad_(True)
    norms = _norms64(d, NS)
    loss = 0
    for bb, nn_, ne in ((batch, n, n_exp), (b2, 200, 100)):
        _, lg = _ref_net(name, d, Pl, bb[:, :nn_].double(), norms)
        loss = loss + (_softplus64(lg) - lg * _labels(nn_, ne)).sum() / nn_
    _assert_grad(g12, th.autograd.grad(loss, Pl)[0], f"{name} accumulated gradient")


# ---------------------------------------------------------------------------------------------------------------------
# training mode: RunningNorm updates, then the forward / backward with the updated statistics
# ---------------------------------------------------------------------------------------------------------------------
def _norm_update64(mean, var, count, x):
    """RunningNorm.update_stats in float64 (util/networks.py:111-134; biased batch variance, Chan merge)"""
    bm, bv, bn = x.mean(0), x.var(0, unbiased=False), x.shape[0]
    delta = bm - mean
    tot = count + bn
    return mean + delta * bn / tot, (var * count + bv * bn + delta ** 2 * count * bn / tot) / tot, tot


@pytest.mark.parametrize("name", ["tc_din7_norm", "h16_norm", "cartpole_64x64", "ant_16", "airl_r32_p32x32",
                                  "airl_r32x32_p32"])
@pytest.mark.parametrize("n", [1000, (1 << 18) + 1000])
def test_training_mode_matches_fp64(name, n):
    """imb_disc_norm_update (128-row chunks at 1 000 rows, 512-row chunks past 2^18 rows), then imb_disc_fwd_bwd with
    IMB_F_TRAIN_NORM against the float64 net in training mode: the base normaliser updated with the base inputs, the
    potential's updated with next_obs (Phi(s') uses that snapshot) and then with obs (Phi(s))."""
    gen = th.Generator(device="cuda").manual_seed(n + 5)
    d, P, batch, ld, NS, NC = _make_inputs(name, n, gen, mode="train")
    X = batch[:, :n].double()
    S = NS.double()
    din, Do = d.base.din, d.d_obs
    c0 = int(NC[0])
    bm, bv, bc = _norm_update64(S[:din], S[din:2 * din], c0, X[_base_rows(d)].T)
    want_ns, norms = [bm, bv], {"base": (bm, bv), "pot_next": None, "pot_now": None}
    if d.shaped:
        lay = _layout(d)
        pm, pv, pc = _norm_update64(S[2 * din:2 * din + Do], S[2 * din + Do:], int(NC[1]), X[lay["nobs"]].T)
        norms["pot_next"] = (pm, pv)
        pm, pv, pc = _norm_update64(pm, pv, pc, X[lay["obs"]].T)
        norms["pot_now"] = (pm, pv)
        want_ns += [pm, pv]
    ws = _ws(d)
    _lib.disc_norm_update(d, batch, ld, n, NS, NC, ws)
    want_ns = th.cat(want_ns)
    np.testing.assert_allclose(NS.cpu().numpy(), want_ns.cpu().numpy(), rtol=1e-5, atol=1e-6, err_msg=f"{name} stats")
    assert int(NC[0]) == bc and (not d.shaped or int(NC[1]) == pc)
    _check_case(name, d, P, NS, batch, ld, n, norms, f"{name} training mode", flags=_lib.IMB_F_TRAIN_NORM, ws=ws,
                forward=False)
