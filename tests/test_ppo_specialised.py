"""The shape-specialised instantiations of k_ppo_update against its runtime-shape instantiation, bit for bit.

imb_ppo_update runs the policies bench.py trains (17/6 Box and 27/8 Box with a feature RunningNorm, 4/2 Discrete
without one, all of width 32) on instantiations whose loop bounds and layout offsets are compile-time constants.  They
only schedule the same arithmetic differently, so every output must equal the runtime-shape instantiation's
(IMB_PPO_FORCE_RUNTIME_SHAPE=1): parameters, both Adam moments, the RunningNorm state and count, the state words and the
loss log.  The CPU test checks which instantiation imb_ppo_update_variant names for which descriptor."""
import numpy as np
import pytest

from imitation_b200 import _desc, _lib

SHAPES = {  # (d_obs, d_act, discrete, has_norm) -> instantiation
    "hc17x6": ((17, 6, False, True), 1),
    "ant27x8": ((27, 8, False, True), 2),
    "cartpole4x2": ((4, 2, True, False), 3),
}

# ragged last minibatches everywhere; minibatches of 64 and below (bench.py's ant trains with 16)
CASES = {
    "hc17x6_mb64": ("hc17x6", dict(N=300, mb=64, epochs=2)),
    "hc17x6_mb48": ("hc17x6", dict(N=250, mb=48, epochs=2)),
    "ant27x8_mb16": ("ant27x8", dict(N=200, mb=16, epochs=2)),
    "ant27x8_mb64": ("ant27x8", dict(N=150, mb=64, epochs=2)),
    "cartpole4x2_mb64": ("cartpole4x2", dict(N=200, mb=64, epochs=3)),
    "cartpole4x2_mb24": ("cartpole4x2", dict(N=100, mb=24, epochs=2)),
}


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _build

    _build.build()
    _lib.lib()
    return _lib


def test_variant_query(L, monkeypatch):
    monkeypatch.delenv("IMB_PPO_FORCE_RUNTIME_SHAPE", raising=False)
    for (Do, Da, discrete, norm), variant in SHAPES.values():
        assert L.ppo_update_variant(_desc.policy_desc(Do, Da, discrete, 32, norm)) == variant
        # any other width, norm setting or action space runs the runtime-shape instantiation
        assert L.ppo_update_variant(_desc.policy_desc(Do, Da, discrete, 20, norm)) == 0
        assert L.ppo_update_variant(_desc.policy_desc(Do, Da, discrete, 32, not norm)) == 0
        assert L.ppo_update_variant(_desc.policy_desc(Do, Da, not discrete, 32, norm)) == 0
    assert L.ppo_update_variant(_desc.policy_desc(18, 6, False, 32, True)) == 0
    assert L.ppo_update_variant(_desc.policy_desc(17, 5, False, 32, True)) == 0
    monkeypatch.setenv("IMB_PPO_FORCE_RUNTIME_SHAPE", "1")
    for (Do, Da, discrete, norm), _ in SHAPES.values():
        assert L.ppo_update_variant(_desc.policy_desc(Do, Da, discrete, 32, norm)) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("with_log", [False, True], ids=["nolog", "log"])
@pytest.mark.parametrize("perm", ["host", "device"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_specialised_matches_runtime_shape(L, monkeypatch, case, perm, with_log):
    from tests.test_ppo_bitexact import _run

    shape, run = CASES[case]
    (Do, Da, discrete, norm), variant = SHAPES[shape]
    cfg = dict(Do=Do, Da=Da, discrete=discrete, hidden=32, norm=norm, device_perm=perm == "device", **run)
    pd = _desc.policy_desc(Do, Da, discrete, 32, norm)
    assert L.ppo_plan(pd, run["mb"]) == L.PPO_PLAN_UPDATE

    monkeypatch.delenv("IMB_PPO_FORCE_RUNTIME_SHAPE", raising=False)
    assert L.ppo_update_variant(pd) == variant
    spec = _run(L, cfg, with_log)
    monkeypatch.setenv("IMB_PPO_FORCE_RUNTIME_SHAPE", "1")
    assert L.ppo_update_variant(pd) == 0
    ref = _run(L, cfg, with_log)

    assert sorted(spec) == sorted(ref)
    assert np.any(spec["params"] != 0)
    for k in ref:
        assert np.array_equal(spec[k], ref[k]), \
            f"{k}: {np.count_nonzero(spec[k] != ref[k])} of {ref[k].size} elements differ"
