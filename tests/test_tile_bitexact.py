"""The fp32 tiled kernels held bit for bit to stored results of an earlier build: imb_disc_fwd_bwd's FFMA kernels (and
the reduce / Adam / RunningNorm launches around them) and imb_rollout / imb_rollout_ensemble at each of their four tile
sizes.

Both evaluate their MLP layers with the tiled bias + activation routine of csrc/imb_tile.cuh, whose arithmetic (FMA
order over k, bias after the sum, then the activation) is fixed; a change to how that routine is shared or laid out must
leave every output bit unchanged.  The float64 tests (test_disc_shape_sweep.py, test_gpu_kernels.py) hold the same
kernels to a tolerance only.  Arrays of more than STORE_RAW_MAX elements are stored as the SHA-256 of their bytes
(followed by their dtype and shape).  The stored results are tests/golden/tile_bitexact.npz; re-record them (on the GPU)
with

    IMB_RECORD_REFERENCE=1 python -m pytest -m gpu tests/test_tile_bitexact.py

The rollout's tile size and grid follow from the GPU's SM count, so its results hold for the SM count they were
recorded with; on another count those cases skip.
"""
import hashlib
import os
import zlib

import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tile_bitexact.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
STORE_RAW_MAX = 256
ROWS = [1, 129, 4099]

# reward nets: disc_desc keyword arguments (+ "onehot": the action rows hold one-hot actions), the shapes of the
# discriminator shape sweep
DISC_SHAPES = {
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
DISC_FLAGS = {"ffma": "IMB_F_NO_TENSOR", "default": None}

# rollout policies: (d_obs, d_act, discrete, tower width, feature RunningNorm)
POLICIES = {"box": (17, 6, False, 32, True), "discrete": (4, 3, True, 64, False)}
# rollout reward nets (disc_desc keyword arguments besides the spaces)
REWARD_NETS = {
    "n32x32_norm": dict(normalize_input=True),
    "n64x64": dict(hid_sizes=(64, 64)),
    "shaped": dict(hid_sizes=(32,), potential_hid_sizes=(32, 32), use_next_state=True, use_done=True, shaped=True,
                   normalize_input=True, gamma=0.9),
}
REWARDS = ["mode0"] + [f"mode{m}_{net}" for m in (1, 2) for net in REWARD_NETS]
# envs per tile size, from the SM count: launch_rollout's thresholds are 16, 32 and 128 envs per SM; two of the four
# leave a ragged last tile (plain loads), two are whole multiples of 4 (bulk-copy tiles)
TILES = {"rows8": lambda s: 16 * s - 5, "rows32": lambda s: 32 * s, "rows64": lambda s: 128 * s - 2,
         "rows128": lambda s: 128 * s + 100}
T_STEPS, HORIZON, ENV_SEED = 3, 2, 23


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _sms():
    return th.cuda.get_device_properties(0).multi_processor_count


def _rng(*key):
    return np.random.default_rng(zlib.crc32("/".join(map(str, key)).encode()))


def _params(rng, shapes):
    """uniform parameters scaled by 1 / sqrt(fan-in) (weights) so that pre-activations stay O(1)"""
    ps = []
    for _, s in shapes:
        scale = 1.7 / np.sqrt(s[1]) if len(s) == 2 else 0.5
        ps.append((rng.uniform(-1, 1, int(np.prod(s))) * scale).astype(np.float32))
    return np.concatenate(ps)


def _disc_params(rng, d, hid, pot):
    from imitation_b200 import _desc

    shapes = _desc.mlp_param_shapes(d.base.din, hid) + (_desc.mlp_param_shapes(d.d_obs, pot) if d.shaped else [])
    P = _params(rng, shapes)
    assert P.size == d.n_params
    return P


def _norm_state(rng, d):
    """[base mean | base var | potential mean | potential var]"""
    nets = [d.base.din] + ([d.d_obs] if d.shaped else [])
    return np.concatenate([np.concatenate([rng.standard_normal(k) * 0.3, rng.uniform(0.5, 3.0, k)])
                           for k in nets]).astype(np.float32)


def _cpu(t):
    return t.detach().cpu().numpy()


def _entries(got):
    """what is stored for each output: the array itself, or the SHA-256 of its bytes under key + '#sha256'"""
    out = {}
    for k, a in got.items():
        a = np.ascontiguousarray(a)
        if a.size > STORE_RAW_MAX:
            out[k + "#sha256"] = np.frombuffer(hashlib.sha256(a.tobytes()).digest() + a.dtype.str.encode()
                                               + str(a.shape).encode(), np.uint8)
        else:
            out[k] = a
    return out


def _check(got, prefix):
    got = _entries(got)
    if RECORD:
        stored = dict(np.load(STORE)) if os.path.exists(STORE) else {}
        stored.update({prefix + k: a for k, a in got.items()})
        np.savez_compressed(STORE, **stored)
        return
    want = np.load(STORE)
    keys = sorted(k[len(prefix):] for k in want.files if k.startswith(prefix))
    assert keys, f"no stored results under {prefix}"
    assert keys == sorted(got), (keys, sorted(got))
    bad = []
    for k in keys:
        w, g = want[prefix + k], got[k]
        if g.dtype != w.dtype or g.shape != w.shape or g.tobytes() != w.tobytes():
            detail = ""
            if not k.endswith("#sha256") and g.shape == w.shape and g.dtype == w.dtype:
                detail = f" ({np.count_nonzero(g.view(np.uint8) != w.view(np.uint8))} bytes differ)"
            bad.append(k + detail)
    assert not bad, f"{prefix}: outputs differ from the stored ones: {bad}"


# ---------------------------------------------------------------------------------------------------------------------
# imb_disc_fwd_bwd (+ reduce, Adam statistics, RunningNorm update)
# ---------------------------------------------------------------------------------------------------------------------
def _disc_inputs(name, n):
    from imitation_b200 import _desc

    kw = DISC_SHAPES[name]
    d = _desc.disc_desc(**{k: v for k, v in kw.items() if k != "onehot"})
    rng = _rng("disc", name, n)
    Do, Da = d.d_obs, d.d_act
    bw, ld = _desc.batch_rows(Do, Da), _desc.batch_ld(n)

    def batch():
        b = np.zeros((bw, ld), np.float32)
        b[:, :n] = rng.standard_normal((bw, n)) * 1.5 + 0.3
        if kw.get("onehot"):
            b[Do:Do + Da, :n] = np.eye(Da, dtype=np.float32)[rng.integers(0, Da, n)].T
        b[2 * Do + Da, :n] = rng.random(n) < 0.3                 # done
        b[2 * Do + Da + 1, :n] = rng.standard_normal(n) * 0.5 - 1  # log pi
        return th.from_numpy(b).cuda()

    P = _disc_params(rng, d, kw.get("hid_sizes", (32, 32)), kw.get("potential_hid_sizes", (32, 32)))
    NS = _norm_state(rng, d) if d.base.has_norm else np.zeros(2, np.float32)
    g = (rng.uniform(-1, 1, n)).astype(np.float32)
    return d, th.from_numpy(P).cuda(), th.from_numpy(NS).cuda(), batch(), batch(), ld, th.from_numpy(g).cuda()


def _disc_outputs(L, name, n, flags):
    d, P, NS, B1, B2, ld, g = _disc_inputs(name, n)
    ws = th.zeros(L.disc_workspace_floats(d), device="cuda")
    n_exp = n // 3
    out = {}

    def run(tag, batch, ns, grad_out=None, fl=L.IMB_F_ZERO_GRAD, n_expert=n_exp):
        lg = th.full((n,), float("nan"), device="cuda")
        gr = th.full((d.n_params,), float("nan"), device="cuda")
        L.disc_fwd_bwd(d, P, ns, batch, ld, n, n_expert, 1.0 / n, grad_out, lg, flags | fl, ws)
        L.disc_reduce(d, ws, gr)
        out[tag + "/logits"], out[tag + "/grad"] = lg, gr

    def adam(tag):
        st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
        stats, Pa = th.full((16,), -1.0, device="cuda"), P.clone()
        L.disc_adam(d, L.Adam(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8), Pa, th.zeros_like(P), th.zeros_like(P), None,
                    1.0, ws, st, stats)
        out[tag + "/stats9"], out[tag + "/adam_params"] = stats[:9], Pa

    run("bce", B1, NS)
    adam("bce")
    run("grad_out", B1, NS, grad_out=g)
    run("accum1", B1, NS)
    run("accum2", B2, NS, fl=0, n_expert=n - n_exp)  # adds to accum1's gradient
    adam("accum2")
    if d.base.has_norm:
        ns, nc = NS.clone(), th.tensor([3000, 3000 if d.shaped else 0], dtype=th.int32, device="cuda")
        L.disc_norm_update(d, B2, ld, n, ns, nc, ws)
        run("train_norm", B2, ns, fl=L.IMB_F_ZERO_GRAD | L.IMB_F_TRAIN_NORM)
        out["train_norm/norm_state"], out["train_norm/norm_count"] = ns, nc
    th.cuda.synchronize()
    return {k: _cpu(t) for k, t in out.items()}


def test_disc_cases_cover_every_ffma_plan(L):
    """plans 2 / 3 / 4 (128-row tiles at two CTAs per SM, 256-row tiles, 128-row tiles at one CTA per SM) all occur"""
    from imitation_b200 import _desc

    plans = {L.disc_plan(_desc.disc_desc(**{k: v for k, v in kw.items() if k != "onehot"}), n)
             for kw in DISC_SHAPES.values() for n in ROWS}
    assert {L.PLAN_FFMA128X2, L.PLAN_FFMA256, L.PLAN_FFMA128} <= plans, plans


@pytest.mark.parametrize("flags", sorted(DISC_FLAGS))
@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("name", sorted(DISC_SHAPES))
def test_disc_fwd_bwd_bit_identical_to_stored(L, name, n, flags):
    fl = getattr(L, DISC_FLAGS[flags]) if DISC_FLAGS[flags] else 0
    _check(_disc_outputs(L, name, n, fl), f"disc/{name}/n{n}/{flags}/")


# ---------------------------------------------------------------------------------------------------------------------
# imb_rollout / imb_rollout_ensemble
# ---------------------------------------------------------------------------------------------------------------------
def _skip_other_sm_count():
    if RECORD:
        return
    want = int(np.load(STORE)["rollout/sms"])
    if _sms() != want:
        pytest.skip(f"rollout results were recorded on a GPU with {want} SMs, this one has {_sms()}")


def _rollout_outputs(L, tile, pol, reward, members=0):
    from imitation_b200 import _desc

    Do, Da, disc, h, pnorm = POLICIES[pol]
    E, T = TILES[tile](_sms()), T_STEPS
    rng = _rng("rollout", tile, pol, reward, members)
    pd = _desc.policy_desc(Do, Da, disc, h, pnorm)
    PP = _params(rng, _desc.policy_param_shapes(Do, Da, disc, h))
    if not disc:
        PP[pd.off_log_std:pd.off_log_std + Da] = rng.uniform(-1.5, 0.5, Da)
    PN = (np.concatenate([rng.standard_normal(Do) * 0.1, rng.uniform(0.5, 1.5, Do)]).astype(np.float32) if pnorm
          else np.zeros(2, np.float32))
    mode, net = (0, None) if reward == "mode0" else (int(reward[4]), reward[6:])
    dd, DP, DN = None, None, None
    if net is not None:
        kw = REWARD_NETS[net]
        dd = _desc.disc_desc(Do, Da, **kw)
        hid, pot = kw.get("hid_sizes", (32, 32)), kw.get("potential_hid_sizes", (32, 32))
        n_nets = members or 1
        DP = [th.from_numpy(_disc_params(rng, dd, hid, pot)).cuda() for _ in range(n_nets)]
        DN = [th.from_numpy(_norm_state(rng, dd)).cuda() if dd.base.has_norm else None for _ in range(n_nets)]
    env = L.EnvDesc(d_obs=Do, d_act=Da, discrete=int(disc), horizon=HORIZON, seed=ENV_SEED, env_id_offset=5)
    EP = th.from_numpy(_desc.synth_env_params(Do, Da, ENV_SEED)).cuda()
    hp = L.PpoHparams(gamma=0.97, gae_lambda=0.9, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                      lr=3e-4, adam_eps=1e-5, n_epochs=1, batch_size=32, normalize_advantage=1)
    st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
    st[L.ST_EPISODE], st[L.ST_GLOBAL_STEP] = 3, 101
    obs = th.empty(Do, E, device="cuda")
    L.env_reset(obs, E, env, st)
    st[L.ST_EP_STEP], st[L.ST_RING_IDX] = 1, 5  # done after local steps 0 and 2
    rw, tw = L.rollout_row_width(pd), _desc.table_width(Do, Da)
    cap = E * T - 7  # the first rows are dropped and the ring wraps
    tbl = th.full((E * T, rw), float("nan"), device="cuda")
    ring = th.zeros(cap, tw, device="cuda")
    flat = th.full((E * T, tw), float("nan"), device="cuda")
    aux = th.full((2 * E + 2 * E * T,), float("nan"), device="cuda")
    PPg, PNg = th.from_numpy(PP).cuda(), th.from_numpy(PN).cuda()
    out = {}
    if members:
        raw = th.full((members * T * E,), float("nan"), device="cuda")
        L.rollout_ensemble(env, EP, obs, pd, PPg, PNg, dd, L.rollout_members(DP, DN, raw), hp, E, T, tbl, ring, cap,
                           flat, aux, None, st)
        out["raw"] = raw
    else:
        L.rollout(env, EP, obs, pd, PPg, PNg, dd, DP[0] if DP else None, DN[0] if DN else None, mode, hp, E, T, tbl,
                  ring, cap, flat, aux, None, st)
    th.cuda.synchronize()
    out.update(table=tbl, aux=aux, env_obs=obs, ring=ring, flat_out=flat)
    return {k: _cpu(t) for k, t in out.items()}


@pytest.mark.parametrize("reward", REWARDS)
@pytest.mark.parametrize("pol", sorted(POLICIES))
@pytest.mark.parametrize("tile", list(TILES))
def test_rollout_bit_identical_to_stored(L, tile, pol, reward):
    _skip_other_sm_count()
    _check(_rollout_outputs(L, tile, pol, reward), f"rollout/{tile}/{pol}/{reward}/")


@pytest.mark.parametrize("pol", sorted(POLICIES))
@pytest.mark.parametrize("tile", list(TILES))
def test_rollout_ensemble_bit_identical_to_stored(L, tile, pol):
    _skip_other_sm_count()
    _check(_rollout_outputs(L, tile, pol, "mode2_n32x32_norm", members=3), f"ensemble/{tile}/{pol}/")


def test_record_sm_count():
    """the SM count the rollout results belong to (written when recording, present otherwise)"""
    if RECORD:
        stored = dict(np.load(STORE)) if os.path.exists(STORE) else {}
        stored["rollout/sms"] = np.array(_sms())
        np.savez_compressed(STORE, **stored)
    assert "rollout/sms" in np.load(STORE).files
