"""CPU: the envelope of the DQN TD step, from imb_dqn_plan (host-only, no GPU).

imb_dqn_plan returns the kernel imb_dqn_step runs for a Q-net and batch size (k_ppo_update_gen<1> for widths up to 32,
k_ppo_update_gen<2> up to 64), or fails naming the shared memory it needs and the limit.  A DQN policy image carries a
zero value tower, so its envelope is the Discrete PPO general kernel's (tests/test_ppo_plan.py).  The edges below were
read off the plan: each accepted shape with one more action is refused.  DeviceDQN asks the plan at construction, so a
Q-net no kernel can run is refused there instead of at the first TD step."""
import numpy as np
import pytest
from torch import nn

from imitation_b200 import _desc, _lib

GEN1, GEN2 = _lib.PPO_PLAN_GEN1, _lib.PPO_PLAN_GEN2
RELU, TANH = _lib.ACT_RELU, _lib.ACT_TANH
LIMIT = "the limit is 231424 B"


@pytest.fixture(scope="module", autouse=True)
def _built():
    from imitation_b200 import _build

    _build.build()
    _lib.lib()


def _q(d_obs, n_actions, width):
    return _desc.policy_desc(d_obs, n_actions, True, width, False)


# (name, (d_obs, n_actions, width), {batch size: expected plan code}); every code holds for tanh and ReLU towers
ACCEPTED = [
    ("cartpole_mlp64", (4, 2, 64), {1: GEN2, 32: GEN2, 220: GEN2, 4096: GEN2}),
    ("cartpole_w32", (4, 2, 32), {1: GEN1, 32: GEN1, 4096: GEN1}),
    ("w1_o1_a1", (1, 1, 1), {1: GEN1, 2: GEN1, 4096: GEN1}),
    ("w7_o4_a2", (4, 2, 7), {2: GEN1, 129: GEN1}),
    ("w20_o17_a9", (17, 9, 20), {33: GEN1, 128: GEN1}),
    ("w32_o64_a64", (64, 64, 32), {1: GEN1, 64: GEN1, 4096: GEN1}),  # every shape at width <= 32 fits
    ("w33_o17_a18", (17, 18, 33), {1: GEN2, 129: GEN2}),
    ("w40_o33_a9", (33, 9, 40), {220: GEN2, 4096: GEN2}),
    ("w63_o1_a64", (1, 64, 63), {1: GEN2, 4096: GEN2}),
    ("w64_o1_a64", (1, 64, 64), {1: GEN2, 64: GEN2, 4096: GEN2}),
    # the edges at d_obs 64, width 64 / 63: the largest action count at batch 1, 64 and 4096
    ("w64_o64_a35", (64, 35, 64), {1: GEN2}),
    ("w64_o64_a34", (64, 34, 64), {1: GEN2, 64: GEN2}),
    ("w64_o64_a16", (64, 16, 64), {1: GEN2, 64: GEN2, 4096: GEN2}),
    ("w63_o64_a41", (64, 41, 63), {1: GEN2, 64: GEN2}),
    ("w63_o64_a23", (64, 23, 63), {4096: GEN2}),
]

# (name, (d_obs, n_actions, width), batch size, the shared memory k_ppo_update_gen<2> would need): one past each edge
REFUSED = [
    ("w64_o64_a36_b1", (64, 36, 64), 1, 231936),
    ("w64_o64_a35_b64", (64, 35, 64), 64, 231552),
    ("w64_o64_a17_b4096", (64, 17, 64), 4096, 232192),
    ("w63_o64_a42_b1", (64, 42, 63), 1, 231808),
    ("w63_o64_a42_b64", (64, 42, 63), 64, 231936),
    ("w63_o64_a24_b4096", (64, 24, 63), 4096, 232192),
    ("w63_o60_a47_b64", (60, 47, 63), 64, 231680),
    ("w64_o64_a64_b1", (64, 64, 64), 1, None),
]


@pytest.mark.parametrize("act", [RELU, TANH], ids=["relu", "tanh"])
@pytest.mark.parametrize("name,args,want", ACCEPTED, ids=[c[0] for c in ACCEPTED])
def test_dqn_plan_accepts(name, args, want, act):
    for B, code in want.items():
        assert _lib.dqn_plan(_q(*args), B, act) == code, (name, B)


@pytest.mark.parametrize("act", [RELU, TANH], ids=["relu", "tanh"])
@pytest.mark.parametrize("name,args,B,need", REFUSED, ids=[c[0] for c in REFUSED])
def test_dqn_plan_refuses_and_names_shared_memory(name, args, B, need, act):
    with pytest.raises(_lib.ImbError, match="shared memory") as e:
        _lib.dqn_plan(_q(*args), B, act)
    msg = str(e.value)
    assert "k_ppo_update_gen<2>" in msg and LIMIT in msg, msg
    if need is not None:
        assert f"needs {need} B" in msg, msg


def test_dqn_plan_edges_are_exact():
    """One action fewer than each refused shape is accepted: the tables above sit on the edge."""
    for _, (Do, A, h), B, _ in REFUSED[:-1]:
        assert _lib.dqn_plan(_q(Do, A - 1, h), B) == GEN2, (Do, A - 1, h, B)


def test_dqn_plan_refuses_what_the_step_cannot_run():
    with pytest.raises(_lib.ImbError, match="Discrete action spaces only"):
        _lib.dqn_plan(_desc.policy_desc(4, 2, False, 64, False), 32)
    with pytest.raises(_lib.ImbError, match="without a feature RunningNorm"):
        _lib.dqn_plan(_desc.policy_desc(4, 2, True, 64, True), 32)
    for B in (0, 4097):
        with pytest.raises(_lib.ImbError, match="minibatch size"):
            _lib.dqn_plan(_q(4, 2, 64), B)
    with pytest.raises(_lib.ImbError, match="pol_act must be IMB_ACT_TANH"):
        _lib.dqn_plan(_q(4, 2, 64), 32, 2)


def _dqn(env, **kw):
    from imitation_b200.algorithms import dqn, sqil
    from imitation_b200.data import types

    r = np.random.default_rng(0)
    n, Do = 20, env.d_obs
    demos = types.Transitions(obs=r.standard_normal((n, Do)).astype(np.float32), acts=r.integers(0, env.d_act, n),
                              infos=np.array([{}] * n), next_obs=r.standard_normal((n, Do)).astype(np.float32),
                              dones=np.zeros(n, bool))
    return dqn.DQN("MlpPolicy", env, replay_buffer_class=sqil.SQILReplayBuffer,
                   replay_buffer_kwargs=dict(demonstrations=demos), **kw)


@pytest.mark.parametrize("d_obs,n_actions,kw,need", [
    (64, 36, dict(batch_size=1), 231936),                                              # past the edge at batch 1
    (64, 35, dict(batch_size=64), 231552),                                             # the batch moves the edge
    (64, 17, dict(batch_size=4096), 232192),
    (64, 42, dict(batch_size=1, policy_kwargs=dict(net_arch=[63, 63], activation_fn=nn.Tanh)), 231808),
])
def test_device_dqn_refuses_unrunnable_q_nets_at_construction(d_obs, n_actions, kw, need):
    """A synthetic Discrete env past the edge: DeviceDQN raises NotImplementedError with the plan's text before it
    allocates anything on the device (so this runs without a GPU)."""
    from imitation_b200.envs import synth

    env = synth.DeviceVecEnv(d_obs, n_actions, 1, discrete=True, device="cpu")
    with pytest.raises(NotImplementedError, match=f"k_ppo_update_gen<2> needs {need} B of shared memory") as e:
        _dqn(env, **kw)
    assert LIMIT in str(e.value) and f"batch_size {kw['batch_size']}" in str(e.value)
