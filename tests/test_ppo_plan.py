"""CPU: the envelope of the PPO update kernels, from imb_ppo_plan (host-only, no GPU).

imb_ppo_plan returns the kernel imb_ppo_update runs for a policy shape and minibatch size, or fails naming the
shared-memory need and the limit.  DevicePPO asks it at construction, so a shape no kernel can run is refused there
instead of at the first train()."""
import pytest

from imitation_b200 import _desc, _lib

UPDATE, GEN1, GEN2 = _lib.PPO_PLAN_UPDATE, _lib.PPO_PLAN_GEN1, _lib.PPO_PLAN_GEN2


@pytest.fixture(scope="module", autouse=True)
def _built():
    from imitation_b200 import _build

    _build.build()
    _lib.lib()


# (name, policy_desc arguments (d_obs, d_act, discrete, hidden, has_norm), {minibatch: expected plan code})
ACCEPTED = [
    # the reference's defaults: FeedForward32Policy, and SB3's MlpPolicy (64x64), at SB3's minibatch of 64
    ("ff32_hc", (17, 6, False, 32, True), {64: UPDATE}),
    ("ff32_cartpole", (4, 2, True, 32, False), {64: UPDATE}),
    ("mlp64_hc", (17, 6, False, 64, False), {64: GEN2}),
    ("mlp64_cartpole", (4, 2, True, 64, False), {64: GEN2}),
    # the tuned minibatches: airl_seals_walker 128, airl_seals_hopper 512
    ("ff32_walker", (17, 6, False, 32, True), {128: GEN1}),
    ("ff32_hopper", (11, 3, False, 32, True), {512: GEN1}),
    ("mlp64_walker", (17, 6, False, 64, True), {128: GEN2, 512: GEN2}),
    # bench.py: hc and airl_hc (17/6, mb 64), cartpole (Discrete 4/2, mb 64), ant (27/8, mb 16)
    ("bench_hc", (17, 6, False, 32, True), {64: UPDATE}),
    ("bench_cartpole", (4, 2, True, 32, False), {64: UPDATE}),
    ("bench_ant", (27, 8, False, 32, True), {16: UPDATE}),
    # k_ppo_update's edges: minibatch 1 and 64, width 1, d_obs 64 with the largest Box d_act that fits (19)
    ("tiny", (1, 1, False, 1, False), {1: UPDATE, 64: UPDATE, 65: GEN1, 4096: GEN1}),
    ("obs64_act19", (64, 19, False, 32, True), {1: UPDATE, 64: UPDATE, 65: GEN1}),
    # k_ppo_update_gen<2>'s edges: width 64, d_obs 64, the largest d_act at minibatch 1 and 4096
    ("mlp64_obs64_act34", (64, 34, False, 64, True), {1: GEN2, 64: GEN2}),
    ("mlp64_obs64_disc35", (64, 35, True, 64, False), {1: GEN2}),
    ("mlp64_obs64_act16", (64, 16, False, 64, True), {4096: GEN2}),
    ("width33", (33, 9, True, 33, False), {1: GEN2, 4096: GEN2}),
]

# k_ppo_update's width and minibatch but not its shared memory (or its parameter slice of <= 256 quads per CTA):
# these run on k_ppo_update_gen<1>, where they used to fail at the first launch
REROUTED = [
    ("obs64_act20", (64, 20, False, 32, True), 64),   # 234 624 B in k_ppo_update
    ("obs64_act64", (64, 64, False, 32, False), 1),
    ("obs32_act64", (32, 64, False, 32, False), 64),
    ("obs60_disc64", (60, 64, True, 32, True), 16),
]

# shapes _desc.policy_desc accepts (width <= 64, d_obs, d_act <= 64, minibatch <= 4096) that no kernel can run, with
# the shared memory k_ppo_update_gen<2> would need
REFUSED = [
    ("mlp64_obs64_act64", (64, 64, False, 64, False), 1, 257536),
    ("mlp64_obs64_act64_mb4096", (64, 64, False, 64, False), 4096, 273792),
    ("mlp64_obs64_act35", (64, 35, False, 64, True), 1, None),
    ("mlp64_obs64_act17_mb4096", (64, 17, False, 64, True), 4096, None),
    ("mlp63_obs60_disc47", (60, 47, True, 63, False), 64, None),
]


@pytest.mark.parametrize("name,args,want", ACCEPTED, ids=[c[0] for c in ACCEPTED])
def test_plan_accepts(name, args, want):
    d = _desc.policy_desc(*args)
    for mb, code in want.items():
        assert _lib.ppo_plan(d, mb) == code, (name, mb)


@pytest.mark.parametrize("name,args,mb", REROUTED, ids=[c[0] for c in REROUTED])
def test_plan_reroutes_to_general_kernel(name, args, mb):
    assert _lib.ppo_plan(_desc.policy_desc(*args), mb) == GEN1


@pytest.mark.parametrize("name,args,mb,need", REFUSED, ids=[c[0] for c in REFUSED])
def test_plan_refuses_and_names_shared_memory(name, args, mb, need):
    with pytest.raises(_lib.ImbError, match="shared memory") as e:
        _lib.ppo_plan(_desc.policy_desc(*args), mb)
    msg = str(e.value)
    assert "k_ppo_update_gen<2>" in msg and "the limit is 231424 B" in msg, msg
    if need is not None:
        assert f"needs {need} B" in msg, msg


def test_plan_honours_force_general(monkeypatch):
    d = _desc.policy_desc(17, 6, False, 32, True)
    assert _lib.ppo_plan(d, 64) == UPDATE
    monkeypatch.setenv("IMB_PPO_FORCE_GENERAL", "1")
    assert _lib.ppo_plan(d, 64) == GEN1
    assert _lib.ppo_plan(_desc.policy_desc(17, 6, False, 64, True), 64) == GEN2


def test_plan_rejects_bad_descriptions():
    d = _desc.policy_desc(17, 6, False, 32, True)
    for mb in (0, 4097):
        with pytest.raises(_lib.ImbError, match="minibatch size"):
            _lib.ppo_plan(d, mb)
    d.d_obs = 65
    with pytest.raises(_lib.ImbError, match="d_obs/d_act"):
        _lib.ppo_plan(d, 64)
    d = _desc.policy_desc(17, 6, False, 32, True)
    d.hidden = 65
    with pytest.raises(_lib.ImbError, match="tower width"):
        _lib.ppo_plan(d, 64)
