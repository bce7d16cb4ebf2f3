"""imb_reward_forward and imb_policy_logp held bit for bit to stored results of an earlier build.

Both are thread-per-row forwards whose arithmetic (loop order, FMA order, tanhf, the input normalisation) is fixed; a
change to how their networks sit in shared memory must leave every output bit unchanged.  The float64 tests
(test_disc_shape_sweep.py, test_ppo_float64.py) hold the same kernels to a tolerance only.  The stored results are
tests/golden/forward_bitexact.npz; re-record them (on the GPU) with

    IMB_RECORD_REFERENCE=1 python -m pytest -m gpu tests/test_forward_bitexact.py
"""
import os
import zlib

import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "forward_bitexact.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
ROWS = [1, 129, 4099]

# reward nets: disc_desc keyword arguments (+ "onehot": the action rows hold one-hot actions), the shapes of the
# discriminator shape sweep
REWARD_SHAPES = {
    "tc_din1": dict(d_obs=1, d_act=0, use_action=False),
    "tc_din1_norm": dict(d_obs=1, d_act=0, use_action=False, normalize_input=True),
    "tc_din7": dict(d_obs=4, d_act=3),
    "tc_din7_norm": dict(d_obs=4, d_act=3, normalize_input=True),
    "tc_din31": dict(d_obs=20, d_act=11),
    "tc_din31_norm": dict(d_obs=20, d_act=11, normalize_input=True),
    "h0": dict(d_obs=17, d_act=6, hid_sizes=()),
    "h16_norm": dict(d_obs=17, d_act=6, hid_sizes=(16,), normalize_input=True),
    "h32": dict(d_obs=17, d_act=6, hid_sizes=(32,)),
    "h20x20_next_done": dict(d_obs=4, d_act=2, hid_sizes=(20, 20), use_next_state=True, use_done=True),
    "h32x32_next_done": dict(d_obs=17, d_act=6, use_next_state=True, use_done=True, normalize_input=True),
    "cartpole_64x64": dict(d_obs=4, d_act=2, hid_sizes=(64, 64), normalize_input=True, onehot=True),
    "h40x64": dict(d_obs=11, d_act=3, hid_sizes=(40, 64)),
    "ant_32x32": dict(d_obs=27, d_act=8, normalize_input=True),
    "din64_next": dict(d_obs=28, d_act=8, use_next_state=True),
    "ant_16": dict(d_obs=27, d_act=8, hid_sizes=(16,), normalize_input=True),
    "airl_r32_p32x32": dict(d_obs=5, d_act=2, hid_sizes=(32,), potential_hid_sizes=(32, 32), shaped=True,
                            normalize_input=True, gamma=0.9, subtract_logp=True),
    "airl_r32x32_p32": dict(d_obs=17, d_act=6, hid_sizes=(32, 32), potential_hid_sizes=(32,), shaped=True,
                            normalize_input=True, gamma=0.9, subtract_logp=True),
}

# policies: (d_obs, d_act, discrete, hidden, feature RunningNorm), the policy shapes of the float64 log pi test
POLICY_SHAPES = {
    "u_w1_o1_a1_mb1": (1, 1, False, 1, True),
    "u_w7_o4_d9_mb2": (4, 9, True, 7, False),
    "u_w32_o33_a17_mb64": (33, 17, False, 32, True),
    "u_w20_o60_d18_mb64": (60, 18, True, 20, True),
    "g1_reroute_o32_a64": (32, 64, False, 32, False),
    "g1_reroute_o60_d64": (60, 64, True, 32, True),
    "g2_w40_o33_d9_mb64": (33, 9, True, 40, True),
    "g2_w63_o60_a17_mb200": (60, 17, False, 63, True),
    "g2_w64_o64_d35_mb1": (64, 35, True, 64, True),
    "g2_w64_o64_a34_mb64": (64, 34, False, 64, False),
}


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _rng(kind, name, n):
    return np.random.default_rng(zlib.crc32(f"{kind}/{name}".encode()) * 8 + ROWS.index(n))


def _params(rng, shapes):
    """uniform parameters scaled by 1 / sqrt(fan-in) (weights) so that pre-activations stay O(1)"""
    ps = []
    for _, s in shapes:
        scale = 1.7 / np.sqrt(s[1]) if len(s) == 2 else 0.5
        ps.append((rng.uniform(-1, 1, int(np.prod(s))) * scale).astype(np.float32))
    return np.concatenate(ps)


def _reward_outputs(L, name, n):
    from imitation_b200 import _desc

    kw = REWARD_SHAPES[name]
    d = _desc.disc_desc(**{k: v for k, v in kw.items() if k != "onehot"})
    rng = _rng("reward", name, n)
    Do, Da = d.d_obs, d.d_act
    bw, ld = _desc.batch_rows(Do, Da), _desc.batch_ld(n)
    batch = np.zeros((bw, ld), np.float32)
    batch[:, :n] = rng.standard_normal((bw, n)) * 1.5 + 0.3
    if kw.get("onehot"):
        batch[Do:Do + Da, :n] = np.eye(Da, dtype=np.float32)[rng.integers(0, Da, n)].T
    batch[2 * Do + Da, :n] = rng.random(n) < 0.3                 # done
    batch[2 * Do + Da + 1, :n] = rng.standard_normal(n) * 0.5 - 1  # log pi
    hid, pot = kw.get("hid_sizes", (32, 32)), kw.get("potential_hid_sizes", (32, 32))
    shapes = _desc.mlp_param_shapes(d.base.din, hid) + (_desc.mlp_param_shapes(Do, pot) if d.shaped else [])
    P = _params(rng, shapes)
    assert P.size == d.n_params
    if d.base.has_norm:  # [base mean | base var | potential mean | potential var]
        nets = [d.base.din] + ([Do] if d.shaped else [])
        NS = np.concatenate([np.concatenate([rng.standard_normal(k) * 0.3, rng.uniform(0.5, 3.0, k)])
                             for k in nets]).astype(np.float32)
        assert NS.size == _desc.disc_norm_floats(d)
    else:
        NS = np.zeros(2, np.float32)
    Pg, NSg, Bg = (th.from_numpy(a).cuda() for a in (P, NS, batch))
    outs = {}
    for mode in (0, 1, 2):
        out = th.full((n,), float("nan"), device="cuda")
        L.reward_forward(d, Pg, NSg, Bg, ld, n, mode, out)
        outs[f"mode{mode}"] = out
    th.cuda.synchronize()
    return {k: t.cpu().numpy() for k, t in outs.items()}


def _logp_outputs(L, name, n):
    from imitation_b200 import _desc

    Do, Da, disc, h, norm = POLICY_SHAPES[name]
    rng = _rng("logp", name, n)
    pd = _desc.policy_desc(Do, Da, disc, h, norm)
    P = _params(rng, _desc.policy_param_shapes(Do, Da, disc, h))
    assert P.size == pd.n_params
    if not disc:
        P[pd.off_log_std:pd.off_log_std + Da] = rng.uniform(-2.0, 1.0, Da)
    NS = (np.concatenate([rng.standard_normal(Do) * 0.3, rng.uniform(0.5, 3.0, Do)]).astype(np.float32) if norm
          else np.zeros(2, np.float32))
    bw, ld = _desc.batch_rows(Do, Da), _desc.batch_ld(n)
    batch = np.zeros((bw, ld), np.float32)
    batch[:Do, :n] = rng.standard_normal((Do, n)) * 1.5 + 0.3
    if disc:
        batch[Do:Do + Da, :n] = np.eye(Da, dtype=np.float32)[rng.integers(0, Da, n)].T
    else:
        batch[Do:Do + Da, :n] = rng.standard_normal((Da, n))
    B = th.from_numpy(batch).cuda()
    L.policy_logp(pd, th.from_numpy(P).cuda(), th.from_numpy(NS).cuda(), B, ld, n, bw - 1)
    th.cuda.synchronize()
    return {"logp": B[bw - 1, :n].cpu().numpy()}


def _check(got, prefix):
    if RECORD:
        stored = dict(np.load(STORE)) if os.path.exists(STORE) else {}
        stored.update({prefix + k: a for k, a in got.items()})
        np.savez_compressed(STORE, **stored)
        return
    want = np.load(STORE)
    keys = sorted(k[len(prefix):] for k in want.files if k.startswith(prefix))
    assert keys == sorted(got), (keys, sorted(got))
    for k in keys:
        w = want[prefix + k]
        assert got[k].dtype == w.dtype and got[k].shape == w.shape, k
        assert np.array_equal(got[k].view(np.uint32), w.view(np.uint32)), \
            f"{k}: {np.count_nonzero(got[k].view(np.uint32) != w.view(np.uint32))} of {got[k].size} elements differ"


@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("name", sorted(REWARD_SHAPES))
def test_reward_forward_bit_identical_to_stored(L, name, n):
    _check(_reward_outputs(L, name, n), f"reward/{name}/n{n}/")


@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("name", sorted(POLICY_SHAPES))
def test_policy_logp_bit_identical_to_stored(L, name, n):
    _check(_logp_outputs(L, name, n), f"logp/{name}/n{n}/")
