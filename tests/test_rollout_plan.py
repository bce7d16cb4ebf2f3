"""CPU: the tile imb_rollout / imb_rollout_ensemble run, from imb_rollout_plan (host only, no GPU).

The rollout kernel prefers the smallest tile that still covers the SMs: up to 16 envs per SM 8 rows per CTA, up to 32
envs per SM 32 rows, up to 128 envs per SM 64 rows, beyond that 128 rows.  Every tile keeps the policy, the synthetic
env and every reward-net image resident in shared memory, and the larger tiles add per-row buffers, so wide AIRL nets
and large ensembles fit the small tiles only.  Such a shape runs on the next smaller tile that fits (more CTAs, each as
fast), instead of being refused at the env counts that prefer a larger tile; it is refused only when not even the 8-row
tile fits.  The shared memory per tile of the shapes below (KiB, of the 226 KiB a CTA can have):

    shape                                                       8     32     64    128
    Hopper 11/3, policy 64, AIRL net 64x64 / potential 64x64   163    180    204    251
    HalfCheetah 17/6, policy 64, 3 members of 64x64 nets       175    194    220    272
    Ant 27/8, policy 64, AIRL net 64x64 / potential 64x64      192    214    243    300
    17/6, policy 32, 16 members of 32x32 nets                  217    230    248    284
"""
import pytest

from imitation_b200 import _desc, _lib

SMS = 132


@pytest.fixture(scope="module", autouse=True)
def _built():
    from imitation_b200 import _build

    _build.build()
    _lib.lib()


def _pol(d_obs, d_act, hidden, discrete=False, norm=True):
    return _desc.policy_desc(d_obs, d_act, discrete, hidden, norm)


def _preferred(E, sms=SMS):
    return 8 if E <= 16 * sms else 32 if E <= 32 * sms else 64 if E <= 128 * sms else 128


# (name, policy, reward net, members, largest tile that fits)
FALLBACK = [
    ("hopper_airl64", _pol(11, 3, 64), _desc.disc_desc(11, 3, hid_sizes=(64, 64), shaped=True,
                                                       potential_hid_sizes=(64, 64), normalize_input=True), 1, 64),
    ("hc_ensemble3_64x64", _pol(17, 6, 64), _desc.disc_desc(17, 6, hid_sizes=(64, 64), normalize_input=True), 3, 64),
    ("ant_airl64", _pol(27, 8, 64), _desc.disc_desc(27, 8, hid_sizes=(64, 64), shaped=True,
                                                    potential_hid_sizes=(64, 64), normalize_input=True), 1, 32),
    ("hc_ensemble16_32x32", _pol(17, 6, 32), _desc.disc_desc(17, 6, normalize_input=True), 16, 8),
]

# the bench.py workloads: FeedForward32Policy with the reward nets of their configurations
BENCH = [
    ("hc", _pol(17, 6, 32), _desc.disc_desc(17, 6, normalize_input=True)),
    ("cartpole", _pol(4, 2, 32, discrete=True, norm=False), _desc.disc_desc(4, 2, hid_sizes=(64, 64),
                                                                             normalize_input=True)),
    ("airl_hc", _pol(17, 6, 32), _desc.disc_desc(17, 6, hid_sizes=(32,), shaped=True, normalize_input=True)),
    ("ant", _pol(27, 8, 32), _desc.disc_desc(27, 8, normalize_input=True)),
]


def _env_counts(sms=SMS):
    """1 env, and each threshold of the preferred tile with its neighbours"""
    out = [1, 1 << 20]
    for per_sm in (16, 32, 128):
        out += [per_sm * sms - 1, per_sm * sms, per_sm * sms + 1]
    return sorted(out)


@pytest.mark.parametrize("name,pol,disc,members,largest", FALLBACK, ids=[c[0] for c in FALLBACK])
def test_fallback_to_the_largest_tile_that_fits(name, pol, disc, members, largest):
    for E in _env_counts():
        want = min(_preferred(E), largest)
        assert _lib.rollout_plan(pol, disc, members, E, SMS) == want, (name, E)
    # the preferred tile does fit below the threshold where it would take the next larger one
    assert _lib.rollout_plan(pol, disc, members, {8: 16, 32: 32, 64: 128, 128: 129}[largest] * SMS, SMS) == largest


@pytest.mark.parametrize("name,pol,disc", BENCH, ids=[c[0] for c in BENCH])
def test_bench_shapes_keep_their_tile(name, pol, disc):
    for sms in (SMS, 114):
        for E in _env_counts(sms) + [64, 512, 1024]:
            assert _lib.rollout_plan(pol, disc, 1, E, sms) == _preferred(E, sms), (name, E, sms)
            assert _lib.rollout_plan(pol, None, 1, E, sms) == _preferred(E, sms), (name, "mode 0", E, sms)
    # ensembles of the hc net
    for E in _env_counts():
        assert _lib.rollout_plan(BENCH[0][1], BENCH[0][2], 3, E, SMS) == _preferred(E), E


def test_refusal_names_bytes_and_limit():
    """16 members of 64x64 nets need ~684 KiB even at the 8-row tile"""
    pol, disc = _pol(17, 6, 64), _desc.disc_desc(17, 6, hid_sizes=(64, 64), normalize_input=True)
    for E in (1, 16 * SMS, 1 << 20):
        with pytest.raises(_lib.ImbError, match=r"16-member ensemble needs \d+ B of shared memory") as e:
            _lib.rollout_plan(pol, disc, 16, E, SMS)
        assert f"{226 * 1024} B limit" in str(e.value)
    # one such net fits
    assert _lib.rollout_plan(pol, disc, 1, 1 << 20, SMS) == 128


def test_plan_rejects_bad_arguments():
    pol, disc = _pol(17, 6, 32), _desc.disc_desc(17, 6)
    with pytest.raises(_lib.ImbError, match="n_envs >= 1"):
        _lib.rollout_plan(pol, disc, 1, 0, SMS)
    with pytest.raises(_lib.ImbError, match="members"):
        _lib.rollout_plan(pol, disc, 17, 64, SMS)
    with pytest.raises(_lib.ImbError, match="members"):
        _lib.rollout_plan(pol, None, 2, 64, SMS)
    with pytest.raises(_lib.ImbError, match="space mismatch"):
        _lib.rollout_plan(pol, _desc.disc_desc(11, 3), 1, 64, SMS)


def test_default_sm_count():
    """n_sms <= 0 asks the current device (132 when none is visible); either way a valid tile"""
    assert _lib.rollout_plan(_pol(17, 6, 32), None, 1, 1000, 0) in (8, 32, 64, 128)
