"""k_ppo_update's outputs held bit for bit to stored results of an earlier build.

Changes to the persistent PPO update that only move work between threads or move data earlier (the schedule of the
optimiser step) must leave every output bit unchanged: the parameters, both Adam moments, the feature RunningNorm
state and count, the state words and the loss log.  The stored results are tests/golden/ppo_update_bitexact.npz;
re-record them (on the GPU) with

    IMB_RECORD_REFERENCE=1 python -m pytest -m gpu tests/test_ppo_bitexact.py
"""
import os

import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ppo_update_bitexact.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"

# the k_ppo_update shapes of test_ppo_update_matches_oracle, plus the hc round's update (device permutation)
CASES = {
    "hc17x6": dict(Do=17, Da=6, discrete=False, hidden=32, norm=True, N=512, mb=64, epochs=3),
    "cartpole4x2": dict(Do=4, Da=2, discrete=True, hidden=32, norm=False, N=200, mb=64, epochs=2),
    "width20": dict(Do=9, Da=3, discrete=False, hidden=20, norm=False, N=256, mb=32, epochs=2),
    "ant30x8_ragged": dict(Do=30, Da=8, discrete=False, hidden=32, norm=True, N=128, mb=48, epochs=2),
    "hc_round": dict(Do=17, Da=6, discrete=False, hidden=32, norm=True, N=4096, mb=64, epochs=5, device_perm=True),
    # 198 quads per slice: seven warps own slice quads, so the statistics run beside the chain instead of in the tail
    "wide60x4": dict(Do=60, Da=4, discrete=False, hidden=32, norm=True, N=256, mb=64, epochs=2),
}


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


def _run(L, cfg, with_log):
    from imitation_b200 import _desc

    Do, Da, discrete, N, mb, epochs = cfg["Do"], cfg["Da"], cfg["discrete"], cfg["N"], cfg["mb"], cfg["epochs"]
    rng = np.random.default_rng(2024 + Do * 100 + N)
    pd = _desc.policy_desc(Do, Da, discrete, cfg["hidden"], cfg["norm"])
    rw = L.rollout_row_width(pd)
    da_store = 1 if discrete else Da
    c = Do + da_store
    tbl = np.zeros((N, rw), np.float32)
    tbl[:, :Do] = rng.standard_normal((N, Do)) * 1.3 + 0.2
    tbl[:, Do:c] = rng.integers(0, Da, (N, 1)) if discrete else rng.standard_normal((N, Da))
    tbl[:, c] = rng.standard_normal(N) * 0.3 - (0.7 if discrete else 8.0)
    tbl[:, c + 1] = rng.standard_normal(N)
    tbl[:, c + 3] = rng.standard_normal(N) * 2
    tbl[:, c + 4] = rng.standard_normal(N)
    npar = pd.n_params
    params = (rng.random(npar, np.float32) - 0.5) * 0.6
    m = rng.standard_normal(npar).astype(np.float32) * 1e-3
    v = np.abs(rng.standard_normal(npar).astype(np.float32)) * 1e-5
    norm = (np.concatenate([rng.standard_normal(Do) * 0.1, 1.0 + rng.random(Do)]).astype(np.float32) if cfg["norm"]
            else np.zeros(2, np.float32))
    P, M, V, PN = (th.from_numpy(a).cuda() for a in (params, m, v, norm))
    PC = th.tensor([700 if cfg["norm"] else 0], dtype=th.int32, device="cuda")
    st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
    st[L.ST_PPO_STEP], st[L.ST_PPO_EPOCH] = 40, 8
    perm = None if cfg.get("device_perm") else th.from_numpy(np.stack([rng.permutation(N) for _ in range(epochs)])).cuda()
    n_steps = epochs * ((N + mb - 1) // mb)
    log = th.zeros(n_steps, 4, device="cuda") if with_log else None
    hp = L.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=0.2, ent_coef=0.01, vf_coef=0.5, max_grad_norm=0.5,
                      lr=3e-4, adam_eps=1e-5, n_epochs=epochs, batch_size=mb, normalize_advantage=1)
    L.ppo_update(pd, P, PN, PC, M, V, th.from_numpy(tbl).cuda(), N, hp, perm, 1234, log, st)
    th.cuda.synchronize()
    out = dict(params=P, exp_avg=M, exp_avg_sq=V, norm_state=PN, norm_count=PC, state=st)
    if with_log:
        out["loss_log"] = log
    return {k: t.cpu().numpy() for k, t in out.items()}


@pytest.mark.parametrize("with_log", [False, True], ids=["nolog", "log"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_ppo_update_bit_identical_to_stored(L, name, with_log):
    got = _run(L, CASES[name], with_log)
    prefix = f"{name}/{'log' if with_log else 'nolog'}/"
    if RECORD:
        stored = dict(np.load(STORE)) if os.path.exists(STORE) else {}
        stored.update({prefix + k: a for k, a in got.items()})
        np.savez_compressed(STORE, **stored)
        return
    want = np.load(STORE)
    keys = sorted(k[len(prefix):] for k in want.files if k.startswith(prefix))
    assert keys == sorted(got), (keys, sorted(got))
    for k in keys:
        assert got[k].dtype == want[prefix + k].dtype and got[k].shape == want[prefix + k].shape, k
        assert np.array_equal(got[k], want[prefix + k]), \
            f"{k}: {np.count_nonzero(got[k] != want[prefix + k])} of {got[k].size} elements differ"
