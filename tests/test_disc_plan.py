"""CPU: the envelope of the fused discriminator kernels, from imb_disc_plan (host-only, no GPU).

imb_disc_plan returns the kernel imb_disc_fwd_bwd runs for a network shape, or fails naming the shared-memory limit.
The reward nets ask it at construction, so a shape the kernels cannot run is refused there instead of at the first
discriminator update."""
import pytest

from imitation_b200 import _desc, _lib, spaces
from imitation_b200.rewards import reward_nets


@pytest.fixture(scope="module", autouse=True)
def _built():
    from imitation_b200 import _build

    _build.build()
    _lib.lib()


# (name, disc_desc kwargs, {n: expected plan code})
ACCEPTED = [
    # the reference's defaults: GAIL BasicRewardNet 32x32 and AIRL BasicShapedRewardNet (base 32, potential 32x32)
    ("gail_default_hc", dict(d_obs=17, d_act=6), {1: 1, 128: 1, 1 << 18: 1}),
    ("airl_default_hc", dict(d_obs=17, d_act=6, hid_sizes=(32,), shaped=True, subtract_logp=True), {1: 4, 4096: 4}),
    # bench.py configurations
    ("bench_hc", dict(d_obs=17, d_act=6, normalize_input=True), {16384: 1}),
    ("bench_cartpole_64x64", dict(d_obs=4, d_act=2, hid_sizes=(64, 64), normalize_input=True), {2048: 4}),
    ("bench_airl_hc", dict(d_obs=17, d_act=6, hid_sizes=(32,), shaped=True, normalize_input=True, subtract_logp=True),
     {4096: 4}),
    ("bench_ant", dict(d_obs=27, d_act=8, normalize_input=True), {64: 4}),
    # the other kernels: two CTAs per SM for small nets, 256-row tiles only for n > 128
    ("small_one_hidden", dict(d_obs=17, d_act=6, hid_sizes=(32,)), {1: 2, 1000: 2}),
    ("shaped_small_obs", dict(d_obs=5, d_act=2, hid_sizes=(32,), shaped=True, subtract_logp=True),
     {128: 4, 129: 3, 4096: 3}),
    # the widest input that fits: din 64 with next_obs
    ("din64_32x32", dict(d_obs=28, d_act=8, use_next_state=True), {257: 4}),
]

# shapes _desc.disc_desc accepts (widths <= 64, din <= 64) whose FFMA tile does not fit into one CTA's shared memory
REFUSED = [
    ("ant_64x64", dict(d_obs=27, d_act=8, hid_sizes=(64, 64))),
    ("ant_64x64_norm", dict(d_obs=27, d_act=8, hid_sizes=(64, 64), normalize_input=True)),
    ("airl_64x64_towers", dict(d_obs=17, d_act=6, hid_sizes=(64, 64), shaped=True, potential_hid_sizes=(64, 64),
                               subtract_logp=True)),
    ("airl_64x64_towers_small_obs", dict(d_obs=4, d_act=2, hid_sizes=(64, 64), shaped=True,
                                         potential_hid_sizes=(64, 64))),
    ("din64_64x64", dict(d_obs=28, d_act=8, use_next_state=True, hid_sizes=(64, 64))),
]


@pytest.mark.parametrize("name,kw,want", ACCEPTED, ids=[c[0] for c in ACCEPTED])
def test_plan_accepts(name, kw, want):
    d = _desc.disc_desc(**kw)
    for n, code in want.items():
        assert _lib.disc_plan(d, n) == code, (name, n)


@pytest.mark.parametrize("name,kw", REFUSED, ids=[c[0] for c in REFUSED])
def test_plan_refuses_and_names_shared_memory(name, kw):
    d = _desc.disc_desc(**kw)
    for n in (1, 128, 4096):
        with pytest.raises(_lib.ImbError, match="shared memory") as e:
            _lib.disc_plan(d, n)
        assert "too large" in str(e.value) and "limit" in str(e.value)


def test_plan_rejects_bad_descriptions():
    with pytest.raises(_lib.ImbError, match="n >= 1"):
        _lib.disc_plan(_desc.disc_desc(17, 6), 0)
    d = _desc.disc_desc(17, 6)
    d.base.din = 22  # does not match the selected inputs
    with pytest.raises(_lib.ImbError, match="does not match"):
        _lib.disc_plan(d, 128)


def test_reward_nets_refuse_unsupported_shapes_at_construction():
    """BasicRewardNet(obs 27, act 8, hid_sizes=(64, 64)) and AIRL nets with 64x64 towers pass _desc's width checks but
    not the kernel's shared memory: construction raises, naming the limit, instead of the first train_disc."""
    obs, act = spaces.Box(-1, 1, (27,)), spaces.Box(-1, 1, (8,))
    with pytest.raises(NotImplementedError, match="shared memory"):
        reward_nets.BasicRewardNet(obs, act, hid_sizes=(64, 64))
    with pytest.raises(NotImplementedError, match="shared memory"):
        reward_nets.BasicShapedRewardNet(spaces.Box(-1, 1, (17,)), spaces.Box(-1, 1, (6,)), reward_hid_sizes=(64, 64),
                                         potential_hid_sizes=(64, 64))
    # the shapes the kernels run are built as before
    net = reward_nets.BasicRewardNet(obs, act)
    assert _lib.disc_plan(net._engine.desc, 64) == _lib.PLAN_FFMA128
    net = reward_nets.BasicRewardNet(spaces.Box(-1, 1, (4,)), spaces.Discrete(2), hid_sizes=(64, 64))
    assert _lib.disc_plan(net._engine.desc, 2048) == _lib.PLAN_FFMA128
