"""ReLU actor-critic generators: SB3 `policy_kwargs` as the reference's configurations pass them, and the kernels that
evaluate the policy with `activation_fn=nn.ReLU` (k_rollout<RPL, ENS, ACT_RELU>, k_ppo_update_gen<U, ACT_RELU>,
k_policy_logp<HP, ACT_RELU>).

CPU: policy construction from the reference's seals_hopper / tuned-hyper-parameter / NORMALIZE_RUNNING_POLICY_KWARGS
dicts, the kwargs refused with the limit named, state_dict and pickles, and imb_ppo_plan's routing of ReLU policies.

GPU: the PPO update against the float64 PPO step of tests/test_ppo_float64.py with its reference made ReLU (_ReluRef);
the single-net and ensemble rollouts against the SB3 restatement with ReLU towers (ActorCriticPortAct: the oracle's
ActorCriticPort with an `activation` argument); log pi against float64; DevicePPO's rollout table against the torch
policy; whole GAIL and AIRL rounds with the reference's Hopper policy_kwargs against oracle/gail_port driving the ReLU
port; and DevicePPO training inside GAIL, AIRL and PreferenceComparisons (graph replay = eager, bit for bit).

ReLU has a kink where tanh has none: a unit whose pre-activation lies within its own fp32 error bound of 0 may take
either side in the kernel.  The float64 step evaluates such units both ways (_KinkReLU: the derivative of the other
side enters the per-row magnitudes the gradient tolerance scales) and accepts either; the global tolerances of
test_ppo_float64.py are unchanged.
"""
import pickle
import warnings

import numpy as np
import pytest
import torch as th
from torch import nn

from imitation_b200 import _build, _desc, _lib, spaces
from imitation_b200.policies import base as policies
from imitation_b200.util import networks
from oracle import ppo_port

U24 = 2.0 ** -24

# the reference's policy_kwargs, literally (scripts/config/train_preference_comparisons.py seals_hopper;
# scripts/config/tuned_hps/gail_seals_hopper_best_hp_eval.json "policy" with its py/type classes resolved;
# scripts/ingredients/policy.py NORMALIZE_RUNNING_POLICY_KWARGS)
SEALS_HOPPER = dict(activation_fn=nn.ReLU, net_arch=[dict(pi=[64, 64], vf=[64, 64])])
GAIL_HOPPER_TUNED = dict(activation_fn=nn.ReLU, features_extractor_class=policies.NormalizeFeaturesExtractor,
                         features_extractor_kwargs=dict(normalize_class=networks.RunningNorm),
                         net_arch=[dict(pi=[64, 64], vf=[64, 64])])
NORMALIZE_RUNNING_POLICY_KWARGS = dict(features_extractor_class=policies.NormalizeFeaturesExtractor,
                                       features_extractor_kwargs=dict(normalize_class=networks.RunningNorm))


def _spaces(Do=11, Da=3, discrete=False):
    obs = spaces.Box(-np.inf, np.inf, (Do,), np.float32)
    act = spaces.Discrete(Da) if discrete else spaces.Box(-1.0, 1.0, (Da,), np.float32)
    return obs, act


def _policy(**kw):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return policies.ActorCriticPolicy(*_spaces(), **kw)


@pytest.fixture(scope="module")
def L():
    _build.build()
    _lib.lib()
    return _lib


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw, norm, act", [(SEALS_HOPPER, False, _lib.ACT_RELU), (GAIL_HOPPER_TUNED, True, _lib.ACT_RELU),
                                           (NORMALIZE_RUNNING_POLICY_KWARGS, True, _lib.ACT_TANH)])
def test_reference_policy_kwargs_build_the_policy(L, kw, norm, act):
    """The policy DevicePPO("MlpPolicy", policy_kwargs=kw) builds (MlpPolicy's default net_arch is 64x64)."""
    kw = {"net_arch": (64, 64), **kw}
    if isinstance(kw["net_arch"], list):  # the deprecated [dict(pi=..., vf=...)] form, unwrapped with SB3's warning
        with pytest.warns(UserWarning, match=r"net_arch=dict\(pi=\.\.\., vf=\.\.\.\)"):
            pol = policies.ActorCriticPolicy(*_spaces(), **kw)
    else:
        pol = policies.ActorCriticPolicy(*_spaces(), **kw)
    assert pol.hidden == 64 and pol.act == act and pol.normalize_features == norm
    relu = isinstance(pol.mlp_extractor.policy_net[1], nn.ReLU)
    assert relu == (act == _lib.ACT_RELU) and type(pol.mlp_extractor.value_net[3]) is type(pol.mlp_extractor.policy_net[1])
    assert isinstance(pol.features_extractor, policies.NormalizeFeaturesExtractor) == norm
    want = _lib.PPO_PLAN_GEN2
    assert L.ppo_plan(pol.desc, 512, act=pol.act) == want


def test_net_arch_forms():
    for arch in ([32, 32], (32, 32), dict(pi=[32, 32], vf=[32, 32])):
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            assert _policy(net_arch=arch).hidden == 32
    with pytest.warns(UserWarning, match=r"net_arch=\[dict\(pi=\.\.\., vf=\.\.\.\)\]"):
        assert policies.ActorCriticPolicy(*_spaces(), net_arch=[dict(pi=[40, 40], vf=[40, 40])]).hidden == 40


@pytest.mark.parametrize("kw, exc, match", [
    (dict(net_arch=dict(pi=[64, 64], vf=[32, 32])), NotImplementedError, "equal widths"),
    (dict(net_arch=[64]), NotImplementedError, r"two hidden layers of one width"),
    (dict(net_arch=[64, 64, 64]), NotImplementedError, r"two hidden layers of one width"),
    (dict(net_arch=[64, 32]), NotImplementedError, r"two hidden layers of one width"),
    (dict(net_arch=[128, 128]), NotImplementedError, r"widths 1 to 64"),
    (dict(activation_fn=nn.ELU), NotImplementedError, "nn.Tanh and nn.ReLU"),
    (dict(activation_fn=nn.LeakyReLU), NotImplementedError, "nn.Tanh and nn.ReLU"),
    (dict(activation_fn=nn.GELU), NotImplementedError, "nn.Tanh and nn.ReLU"),
    (dict(use_sde=True), NotImplementedError, "use_sde"),
    (dict(share_features_extractor=False), NotImplementedError, "share_features_extractor"),
    (dict(optimizer_class=th.optim.SGD), NotImplementedError, "optimizer_class"),
    (dict(optimizer_kwargs=dict(eps=1e-8)), NotImplementedError, "optimizer_kwargs"),
    (dict(features_extractor_class=policies.NormalizeFeaturesExtractor,
          features_extractor_kwargs=dict(normalize_class=nn.BatchNorm1d)), NotImplementedError, "normalize_class"),
    (dict(features_extractor_class=nn.Identity), NotImplementedError, "features_extractor_class"),
    (dict(features_extractor_class=policies.NormalizeFeaturesExtractor, normalize_features=False), ValueError,
     "contradicts"),
    (dict(features_extractor_class=policies.FlattenExtractor, normalize_features=True), ValueError, "contradicts"),
    (dict(no_such_kwarg=1), TypeError, "no_such_kwarg"),
])
def test_refused_policy_kwargs(kw, exc, match):
    with pytest.raises(exc, match=match):
        _policy(**kw)


def test_accepted_sb3_kwargs():
    a = _policy(net_arch=[64, 64], ortho_init=False, log_std_init=-0.5, optimizer_class=th.optim.Adam,
                optimizer_kwargs=dict(eps=1e-5), normalize_features=True,
                features_extractor_class=policies.NormalizeFeaturesExtractor)
    assert a.normalize_features and np.allclose(a.log_std.detach().numpy(), -0.5)
    assert _policy(features_extractor_class=policies.FlattenExtractor).normalize_features is False
    # NormalizeFeaturesExtractor takes the reference's signature as well as a flat width
    ext = policies.NormalizeFeaturesExtractor(_spaces(17)[0], normalize_class=networks.RunningNorm)
    assert ext.normalize.running_mean.shape == (17,)
    assert policies.NormalizeFeaturesExtractor(5).normalize.running_mean.shape == (5,)


def test_reference_classes_recognised_by_module_not_name_alone():
    """The reference's RunningNorm / NormalizeFeaturesExtractor / SB3's FlattenExtractor (named by its configurations)
    are recognised by module and name; a user's class that only shares the name is refused."""
    def cls(name, module):
        return type(name, (nn.Module,), {"__module__": module})

    norm = _policy(features_extractor_class=cls("NormalizeFeaturesExtractor", "imitation.policies.base"),
                   features_extractor_kwargs=dict(normalize_class=cls("RunningNorm", "imitation.util.networks")))
    assert norm.normalize_features
    flat = _policy(features_extractor_class=cls("FlattenExtractor", "stable_baselines3.common.torch_layers"))
    assert not flat.normalize_features
    with pytest.raises(NotImplementedError, match="normalize_class"):
        _policy(features_extractor_class=policies.NormalizeFeaturesExtractor,
                features_extractor_kwargs=dict(normalize_class=cls("RunningNorm", "my_project.norms")))
    with pytest.raises(NotImplementedError, match="features_extractor_class"):
        _policy(features_extractor_class=cls("NormalizeFeaturesExtractor", "my_project.extractors"))
    with pytest.raises(NotImplementedError, match="normalize_class"):
        policies.NormalizeFeaturesExtractor(5, normalize_class=cls("RunningNorm", "my_project.norms"))


def test_orthogonal_gains_do_not_depend_on_the_activation():
    th.manual_seed(0)
    t = _policy(net_arch=[64, 64])
    th.manual_seed(0)
    r = _policy(net_arch=[64, 64], activation_fn=nn.ReLU)
    for (k, a), (k2, b) in zip(t.state_dict().items(), r.state_dict().items()):
        assert k == k2 and th.equal(a, b), k


def test_state_dict_and_pickles():
    t = _policy(net_arch=[64, 64], normalize_features=True)
    r = _policy(net_arch=[64, 64], normalize_features=True, activation_fn=nn.ReLU)
    assert [(k, v.shape) for k, v in t.state_dict().items()] == [(k, v.shape) for k, v in r.state_dict().items()]
    assert {"mlp_extractor.policy_net.0.weight", "mlp_extractor.policy_net.2.weight", "mlp_extractor.value_net.0.weight",
            "mlp_extractor.value_net.2.weight"} <= set(r.state_dict())
    back = pickle.loads(pickle.dumps(r))
    assert back.act == _lib.ACT_RELU and isinstance(back.mlp_extractor.value_net[3], nn.ReLU)
    # a pickle written before the policy had an activation attribute loads as tanh
    old = t.__getstate__()
    del old["act"]
    fresh = policies.ActorCriticPolicy.__new__(policies.ActorCriticPolicy)
    fresh.__setstate__(old)
    assert fresh.act == _lib.ACT_TANH


def test_feed_forward32_passes_activation_through(L):
    p = policies.FeedForward32Policy(*_spaces(17, 6), activation_fn=nn.ReLU, normalize_features=True)
    assert p.hidden == 32 and p.act == _lib.ACT_RELU
    assert L.ppo_plan(p.desc, 64, act=p.act) == _lib.PPO_PLAN_GEN1  # never the tanh-only k_ppo_update


def test_ppo_plan_routes_relu_to_the_general_kernel(L, monkeypatch):
    monkeypatch.delenv("IMB_PPO_FORCE_GENERAL", raising=False)
    mbs = [1, 2, 63, 64, 65, 128, 512, 4095, 4096]
    for h in list(range(1, 65, 7)) + [32, 33, 64]:
        for Do, Da, disc, norm in ((11, 3, False, True), (4, 2, True, False)):
            d = _desc.policy_desc(Do, Da, disc, h, norm)
            for mb in mbs:
                want = _lib.PPO_PLAN_GEN1 if h <= 32 else _lib.PPO_PLAN_GEN2
                assert L.ppo_plan(d, mb, act=_lib.ACT_RELU) == want, (h, Do, mb)
                tanh = L.ppo_plan(d, mb)
                assert L.ppo_plan(d, mb, act=_lib.ACT_TANH) == tanh
                assert tanh == (_lib.PPO_PLAN_UPDATE if h <= 32 and mb <= 64 else want), (h, Do, mb)
    d = _desc.policy_desc(17, 6, False, 32, True)
    assert L.ppo_plan(d, 64) == _lib.PPO_PLAN_UPDATE and L.ppo_plan(d, 64, act=_lib.ACT_RELU) == _lib.PPO_PLAN_GEN1


def test_ppo_plan_rejects_unknown_activation(L):
    d = _desc.policy_desc(11, 3, False, 64, True)
    for act in (2, -1, 7):
        with pytest.raises(_lib.ImbError, match="pol_act must be IMB_ACT_TANH"):
            L.ppo_plan(d, 512, act=act)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the PPO update against float64 (the three measurements of tests/test_ppo_float64.py, ReLU towers)
# ---------------------------------------------------------------------------------------------------------------------
class _KinkReLU(th.autograd.Function):
    """relu(z) whose derivative, for the per-row magnitudes only, adds the other side of the kink (/ C_GRAD, which the
    tolerance multiplies back) on units whose pre-activation lies within its fp32 error bound dz of 0."""
    generate_vmap_rule = True

    @staticmethod
    def forward(z, dz):
        return th.relu(z)

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.save_for_backward(inputs[0], inputs[1])

    @staticmethod
    def backward(ctx, g):
        from tests import test_ppo_float64 as F

        z, dz = ctx.saved_tensors
        d = (z > 0).to(g.dtype)
        amb = (z.abs() <= dz).to(g.dtype)
        return g * (d + amb * (1 - 2 * d) / F.C_GRAD), None


def _relu_ref_class():
    from tests import test_ppo_float64 as F

    class _ReluRef(F.Ref):
        """test_ppo_float64.Ref with ReLU towers (forward relu; backward threshold_backward, derivative 0 at 0)."""

        def heads(self, p, xn, padded=False):
            W = self.unpack(p)

            def layer(x, e, w, b):
                z = x @ w.T + b
                if not padded:
                    return th.relu(z), None
                dz = w.shape[1] * U24 * (x.abs() @ w.abs().T + b.abs()) + e @ w.abs().T
                return _KinkReLU.apply(z, dz.detach()), (dz * (z > -dz)).detach()  # relu is 1-Lipschitz

            e0 = (4 * U24 * xn.abs()) if padded else None
            lat = layer(*layer(xn, e0, W[0], W[1]), W[2], W[3])[0]
            lv = layer(*layer(xn, e0, W[4], W[5]), W[6], W[7])[0]
            return lat @ W[8].T + W[9], (lv @ W[10].T)[..., 0] + W[11][0], lv, W

    return _ReluRef


class _ReluLib:
    """_lib with every policy entry point called for ReLU towers."""

    def __getattr__(self, name):
        return getattr(_lib, name)

    def ppo_update(self, *a, **k):
        return _lib.ppo_update(*a, act=_lib.ACT_RELU, **k)

    def ppo_plan(self, *a, **k):
        return _lib.ppo_plan(*a, act=_lib.ACT_RELU, **k)

    def policy_logp(self, *a, **k):
        return _lib.policy_logp(*a, act=_lib.ACT_RELU, **k)

    def rollout(self, *a, **k):
        return _lib.rollout(*a, act=_lib.ACT_RELU, **k)

    def rollout_ensemble(self, *a, **k):
        return _lib.rollout_ensemble(*a, act=_lib.ACT_RELU, **k)


GEN1, GEN2 = _lib.PPO_PLAN_GEN1, _lib.PPO_PLAN_GEN2
# test_ppo_float64.CASES layout: (d_obs, d_act, discrete, width, feature norm, minibatch, N, epochs, initial norm count,
#   ent_coef, normalize_advantage, permutation, force general, plan code)
RELU_CASES = {
    "relu_hopper_w64_mb512": (11, 3, False, 64, True, 512, "2*mb+1", 1, 700, 0.001, True, "host", False, GEN2),
    "relu_o17_a6_w64_mb64": (17, 6, False, 64, False, 64, "3*mb", 2, 0, 0.0, True, "device", False, GEN2),
    "relu_o4_d2_w64_mb128": (4, 2, True, 64, False, 128, "2*mb+1", 2, 0, 0.01, True, "host", False, GEN2),
    "relu_o17_a6_w32_mb64": (17, 6, False, 32, True, 64, "2*mb+1", 2, 10 ** 7, 0.01, True, "host", False, GEN1),
    "relu_o4_d9_w32_mb100": (4, 9, True, 32, True, 100, "3*mb", 2, 700, 0.01, True, "device", False, GEN1),
}


@pytest.fixture
def relu_f64(monkeypatch):
    """tests/test_ppo_float64.py with RELU_CASES and its float64 reference made ReLU, for the duration of a test."""
    from tests import test_ppo_float64 as F

    monkeypatch.setattr(F, "CASES", RELU_CASES)
    monkeypatch.setattr(F, "Ref", _relu_ref_class())
    monkeypatch.setattr(F, "_make_inputs", _relu_inputs(F._make_inputs))
    monkeypatch.delenv("IMB_PPO_FORCE_GENERAL", raising=False)
    return F


def _relu_inputs(make_inputs):
    """test_ppo_float64's inputs with the Box action head scaled down by RELU_HEAD.  Its tower weights (per-unit scales
    up to 15, which saturate tanh) leave ReLU latents in the hundreds; with log_std down to -3 the fp32 error of such
    action means alone moves the ratio by more than the gradient tolerance.  Scaled, the means have the magnitude they
    have under tanh; the actions are redrawn around them the same way."""

    def make(c):
        pd, P, norm, tbl, M, V, rng = make_inputs(c)
        if not c["disc"]:
            from tests import test_ppo_float64 as F

            Do, Da = c["Do"], c["Da"]
            P[pd.off_act_w:pd.off_act_b] *= RELU_HEAD
            x = th.from_numpy(tbl[:, :Do]).double()
            if c["norm"]:
                x = (x - th.from_numpy(norm[:Do]).double()) / th.sqrt(th.from_numpy(norm[Do:]).double() + F.EPS_NORM)
            out = F.Ref(c, 0.0).heads(th.from_numpy(P).double(), x)[0].numpy()
            ls = P[pd.off_log_std:pd.off_log_std + Da]
            tbl[:, Do:Do + Da] = out + np.exp(ls) * 1.5 * rng.standard_normal((len(tbl), Da))
        return pd, P, norm, tbl, M, V, rng

    return make


RELU_HEAD = 0.02


@pytest.mark.gpu
def test_relu_cases_run_the_general_kernels(L, relu_f64):
    for name in RELU_CASES:
        c = relu_f64._cfg(name)
        assert L.ppo_plan(_desc.policy_desc(c["Do"], c["Da"], c["disc"], c["h"], c["norm"]), c["mb"],
                          act=_lib.ACT_RELU) == c["code"], name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RELU_CASES))
def test_relu_one_step_gradient_through_adam_moments(L, relu_f64, name):
    relu_f64.test_one_step_gradient_through_adam_moments(_ReluLib(), lambda on: None, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(RELU_CASES))
def test_relu_whole_run_at_lr0(L, relu_f64, name):
    relu_f64.test_whole_run_at_lr0(_ReluLib(), lambda on: None, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in RELU_CASES if RELU_CASES[n][11] == "host"])
def test_relu_adam_step_teacher_forced(L, relu_f64, name):
    relu_f64.test_adam_step_teacher_forced(_ReluLib(), lambda on: None, name)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 129, 4099])
@pytest.mark.parametrize("name", ["relu_hopper_w64_mb512", "relu_o4_d2_w64_mb128", "relu_o17_a6_w32_mb64",
                                  "relu_o4_d9_w32_mb100"])
def test_relu_policy_logp_against_float64(L, relu_f64, name, n):
    relu_f64.test_policy_logp_against_float64(_ReluLib(), name, n)


@pytest.mark.gpu
def test_relu_and_tanh_log_pi_differ(L):
    """The activation reaches the kernel: the same parameters give a different log pi with ReLU towers."""
    pd = _desc.policy_desc(11, 3, False, 64, False)
    th.manual_seed(0)
    P = th.randn(pd.n_params, device="cuda")
    n, bw = 300, _desc.batch_rows(11, 3)
    ld = _desc.batch_ld(n)
    batch = th.randn(bw, ld, device="cuda")
    out = []
    for act in (_lib.ACT_TANH, _lib.ACT_RELU):
        b = batch.clone()
        _lib.policy_logp(pd, P, th.zeros(2, device="cuda"), b, ld, n, bw - 1, act=act)
        out.append(b[bw - 1, :n])
    assert not th.equal(out[0], out[1])


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the rollout against the SB3 restatement with ReLU towers, pinned noise
# ---------------------------------------------------------------------------------------------------------------------
class ActorCriticPortAct(ppo_port.ActorCriticPort):
    """oracle.ppo_port.ActorCriticPort (SB3's ActorCriticPolicy restated, tanh towers) with an `activation` argument:
    "tanh" (the port as it is) or "relu" (nn.ReLU after each tower layer, as SB3 builds with activation_fn=nn.ReLU)."""

    def __init__(self, *args, activation: str = "tanh", **kwargs):
        super().__init__(*args, **kwargs)
        if activation not in ("tanh", "relu"):
            raise ValueError(f"activation {activation!r}: 'tanh' or 'relu'")
        if activation == "relu":
            for tower in (self.pi, self.vf):
                for i, m in enumerate(tower):
                    if isinstance(m, nn.Tanh):
                        tower[i] = nn.ReLU()


def _relu_oracle(monkeypatch):
    """The oracle's rollout drivers in other test modules build ActorCriticPortAct(activation="relu") where they build
    the port."""
    monkeypatch.setattr(ppo_port, "ActorCriticPort", lambda *a, **k: ActorCriticPortAct(*a, activation="relu", **k))


def test_actor_critic_port_activation():
    th.manual_seed(0)
    t = ActorCriticPortAct(11, 3, hidden=(64, 64))
    th.manual_seed(0)
    r = ActorCriticPortAct(11, 3, hidden=(64, 64), activation="relu")
    assert [type(m) for m in t.pi] == [nn.Linear, nn.Tanh, nn.Linear, nn.Tanh]
    assert [type(m) for m in r.vf] == [nn.Linear, nn.ReLU, nn.Linear, nn.ReLU]
    assert all(th.equal(a, b) for a, b in zip(t.state_dict().values(), r.state_dict().values()))
    x = th.randn(5, 11)
    with th.no_grad():
        want = r.action_net(th.relu(r.pi[2](th.relu(r.pi[0](x)))))
        assert th.allclose(r._dist(x).mean, want)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [
    dict(Do=11, Da=3, discrete=False, E=37, T=9, H=5, hidden=64, norm=True, reward_mode=1),
    dict(Do=4, Da=2, discrete=True, E=64, T=6, H=4, hidden=64, norm=False, reward_mode=1),
    dict(Do=17, Da=6, discrete=False, E=33, T=4, H=1000, hidden=32, norm=False, reward_mode=0),
])
def test_relu_rollout_gae_matches_oracle(L, cfg, monkeypatch):
    """Single-net rollout (GAIL reward, env reward): tests/test_gpu_kernels.py's check (transition order, done masks and
    ring bit-exact; actions, log pi, values, rewards, GAE to its tolerances), ReLU towers in the kernel and the port."""
    from tests import test_gpu_kernels as K

    _relu_oracle(monkeypatch)
    K.test_rollout_gae_matches_oracle(_ReluLib(), cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [
    dict(Do=11, Da=3, discrete=False, E=37, T=9, H=5, M=3, out_norm=True, in_norm=False, alpha=-0.5),
    dict(Do=4, Da=2, discrete=True, E=64, T=6, H=4, M=3, out_norm=False, in_norm=True, alpha=0.0),
])
def test_relu_ensemble_rollout_matches_oracle(L, cfg, monkeypatch):
    """AddSTDRewardWrapper(RewardEnsemble(3 members)) / RewardEnsemble as the reward (k_rollout<RPL, true, ReLU>):
    tests/test_ensemble_relabel.py's check over two rounds, ReLU towers in the kernel and the port."""
    from tests import test_ensemble_relabel as R

    _relu_oracle(monkeypatch)
    R.test_ensemble_rollout_matches_oracle(_ReluLib(), cfg)


@pytest.mark.gpu
def test_relu_deterministic_generate_trajectories_match_torch_policy(L):
    """data/rollout.generate_trajectories(deterministic) with a ReLU policy: its actions are the torch policy's means."""
    from imitation_b200.data import rollout
    from imitation_b200.envs import synth

    venv = synth.DeviceVecEnv(11, 3, 8, horizon=6, seed=2)
    th.manual_seed(0)
    pol = policies.ActorCriticPolicy(venv.observation_space, venv.action_space, net_arch=[64, 64],
                                     activation_fn=nn.ReLU).cuda()
    with th.no_grad():
        for p in pol.parameters():
            p.add_(0.3 * th.randn_like(p))
    trajs = rollout.generate_trajectories(pol, venv, rollout.make_sample_until(min_episodes=8),
                                          np.random.default_rng(0), deterministic_policy=True)
    assert len(trajs) >= 8
    for tr in trajs[:8]:
        obs = th.as_tensor(tr.obs[:-1]).cuda()
        with th.no_grad():
            mean = pol.action_net(pol.mlp_extractor.policy_net(pol.features_extractor(obs))).cpu().numpy()
        np.testing.assert_allclose(tr.acts, np.clip(mean, -1, 1), rtol=1e-4, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: DevicePPO with the reference's Hopper policy_kwargs inside the trainers
# ---------------------------------------------------------------------------------------------------------------------
def _hopper_ppo(venv, **kw):
    from imitation_b200.algorithms import ppo

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return ppo.DevicePPO("MlpPolicy", venv, batch_size=512, n_epochs=20, policy_kwargs=dict(GAIL_HOPPER_TUNED),
                             seed=0, **kw)


def _trainer(algo, graph):
    from imitation_b200.algorithms.adversarial import airl, gail
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets

    th.manual_seed(0)
    venv = synth.DeviceVecEnv(11, 3, 16, horizon=40, seed=4)
    gen = _hopper_ppo(venv, n_steps=64)
    gen.use_cuda_graph = graph
    assert gen.policy.act == _lib.ACT_RELU and gen.policy.hidden == 64 and gen.policy.normalize_features
    cls = reward_nets.BasicShapedRewardNet if algo == "airl" else reward_nets.BasicRewardNet
    net = cls(venv.observation_space, venv.action_space, normalize_input_layer=networks.RunningNorm)
    rng = np.random.default_rng(0)
    n = 512
    demos = dict(obs=rng.standard_normal((n, 11)).astype(np.float32), acts=rng.uniform(-1, 1, (n, 3)).astype(np.float32),
                 next_obs=rng.standard_normal((n, 11)).astype(np.float32), dones=rng.random(n) < 0.05)
    tcls = airl.AIRL if algo == "airl" else gail.GAIL
    return tcls(demonstrations=demos, demo_batch_size=128, venv=venv, gen_algo=gen, reward_net=net,
                n_disc_updates_per_round=2, seed=0)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["gail", "airl"])
def test_hopper_policy_trains_in_adversarial_rounds(L, algo):
    """GAIL / AIRL rounds with the reference's Hopper policy: it trains, and a graph-replayed run equals an eager one."""
    runs = []
    for graph in (False, True):
        tr = _trainer(algo, graph)
        p0 = tr.policy.flat_vectors()[0].clone()
        tr.train(3 * tr.gen_train_timesteps)
        tr.join()
        th.cuda.synchronize()
        p1, pn, pc = tr.policy.flat_vectors()
        assert th.isfinite(p1).all() and not th.equal(p0, p1)
        runs.append([t.clone() for t in (p1, pn, pc)] + [t.detach().clone() for t in tr._reward_net.parameters()])
    for a, b in zip(*runs):
        assert th.equal(a, b), "graph replay differs from eager execution"


@pytest.mark.gpu
@pytest.mark.parametrize("reward", ["single", "ensemble"])
def test_device_ppo_rollout_evaluates_relu_towers(L, reward):
    """DevicePPO.collect_rollouts with a ReLU policy, a BasicRewardNet or an AddSTDRewardWrapper(RewardEnsemble)
    reward: the log pi and value columns of its rollout table are the torch policy's (eval mode) on the table's rows."""
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets, reward_wrapper

    th.manual_seed(0)
    venv = synth.DeviceVecEnv(11, 3, 16, horizon=10, seed=1)
    obs_sp, act_sp = venv.observation_space, venv.action_space
    if reward == "single":
        net = reward_nets.BasicRewardNet(obs_sp, act_sp).cuda()
    else:
        members = [reward_nets.BasicRewardNet(obs_sp, act_sp) for _ in range(3)]
        net = reward_nets.AddSTDRewardWrapper(reward_nets.RewardEnsemble(obs_sp, act_sp, members).cuda(), -0.5)
    gen = _hopper_ppo(reward_wrapper.RewardVecEnvWrapper(venv, net.predict_processed), n_steps=12)
    pol = gen.policy
    with th.no_grad():
        for p in pol.parameters():  # spread the orthogonal init so that the heads see the towers
            p.add_(0.3 * th.randn_like(p))
    gen.collect_rollouts()
    th.cuda.synchronize()
    tbl = gen._tbl
    obs, acts = tbl[:, :11], tbl[:, 11:14]
    with th.no_grad(), networks.evaluating(pol):
        values, logp, _ = pol.evaluate_actions(obs, acts)
    np.testing.assert_allclose(tbl[:, 15].cpu().numpy(), values[:, 0].cpu().numpy(), rtol=1e-4, atol=1e-5,
                               err_msg="value column")
    np.testing.assert_allclose(tbl[:, 14].cpu().numpy(), logp.cpu().numpy(), rtol=1e-4, atol=1e-4,
                               err_msg="log pi column")


def _relu_rounds(algo, seed, n_rounds, Do=11, Da=3, E=16, T=8, H=20, B=64, cap=96, n_disc=2, ppo_batch=32):
    """A GAIL / AIRL trainer whose generator is DevicePPO("MlpPolicy", policy_kwargs=<the reference's tuned Hopper
    policy_kwargs>), and oracle/gail_port.AdversarialPort on the same environment seed, demonstrations, rollout noise,
    PPO permutations and index streams, its generator ActorCriticPortAct(activation="relu") with the same weights
    (tests/test_round_parity.py's pairing, ReLU towers)."""
    from imitation_b200.algorithms import ppo
    from imitation_b200.algorithms.adversarial import airl, common, gail
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets
    from oracle import gail_port, nets_port, synth_env
    from tests import golden_util as G
    from tests.test_round_parity import HP

    th.manual_seed(seed)
    venv = synth.DeviceVecEnv(Do, Da, E, horizon=H, seed=seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # the deprecated [dict(pi=..., vf=...)] form
        gen = ppo.DevicePPO("MlpPolicy", venv, n_steps=T, batch_size=ppo_batch, n_epochs=2, seed=seed,
                            policy_kwargs=dict(GAIL_HOPPER_TUNED))
    assert gen.policy.act == _lib.ACT_RELU and gen.policy.hidden == 64 and gen.policy.normalize_features
    ncls = reward_nets.BasicShapedRewardNet if algo == "airl" else reward_nets.BasicRewardNet
    net = ncls(venv.observation_space, venv.action_space, normalize_input_layer=networks.RunningNorm)
    rng = np.random.default_rng(seed)
    n = 4 * B
    demos = dict(obs=rng.standard_normal((n, Do)).astype(np.float32), acts=rng.uniform(-1, 1, (n, Da)).astype(np.float32),
                 next_obs=rng.standard_normal((n, Do)).astype(np.float32), dones=rng.random(n) < 0.05)
    tcls = airl.AIRL if algo == "airl" else gail.GAIL
    tr = tcls(demonstrations=demos, demo_batch_size=B, venv=venv, gen_algo=gen, reward_net=net,
              n_disc_updates_per_round=n_disc, gen_replay_buffer_capacity=cap, sampling="host_compat", seed=seed)
    N = E * T
    rng = np.random.default_rng(seed + 100)
    noise = rng.standard_normal((n_rounds, T, E, Da)).astype(np.float32)
    perms = np.stack([np.stack([rng.permutation(N) for _ in range(gen.n_epochs)]) for _ in range(n_rounds)])

    pvenv = synth_env.SynthVecEnv(synth_env.SynthEnvSpec(Do, Da, discrete=False, horizon=H, seed=seed), E)
    pol = ActorCriticPortAct(Do, Da, hidden=(64, 64), normalize_features=True, activation="relu")
    psd = {k: v.detach().cpu().clone() for k, v in tr.policy.state_dict().items()}
    sd = {f"{p}.{i}.{w}": psd[f"mlp_extractor.{t}.{i}.{w}"] for p, t in (("pi", "policy_net"), ("vf", "value_net"))
          for i in (0, 2) for w in ("weight", "bias")}
    sd.update({k: psd[k] for k in ("action_net.weight", "action_net.bias", "value_net.weight", "value_net.bias",
                                   "log_std")})
    pol.load_state_dict(sd, strict=False)
    flat_noise = noise.reshape((n_rounds * T,) + noise.shape[2:])
    flat_perms = perms.reshape(n_rounds * gen.n_epochs, N)
    pgen = ppo_port.PPOPort(pol, pvenv, n_steps=T, batch_size=gen.batch_size, n_epochs=gen.n_epochs,
                            noise_fn=lambda step: flat_noise[step], perm_fn=lambda e, n: flat_perms[e], **HP)
    pcls = nets_port.ShapedRewardNetPort if algo == "airl" else nets_port.BasicRewardNetPort
    pnet = pcls(Do, Da, normalize_input=True)
    pnet.load_state_dict({G.port_key(k): v.detach().cpu().clone() for k, v in tr._reward_net.state_dict().items()})
    pnet.eval()
    expert = {k: np.asarray(v) for k, v in demos.items()}
    th.manual_seed(seed + 7)
    port = gail_port.AdversarialPort(venv=pvenv, expert=expert, demo_batch_size=B, gen=pgen, reward_net=pnet,
                                     airl=algo == "airl", n_disc_updates_per_round=n_disc,
                                     gen_replay_buffer_capacity=cap)
    th.manual_seed(seed + 7)
    tr._expert_compat = common._TorchCompatExpertIndices(len(expert["obs"]), B)
    return tr, port, noise, perms


@pytest.mark.gpu
@pytest.mark.parametrize("algo, n_rounds", [("gail", 3), ("airl", 1)])
def test_hopper_relu_rounds_match_adversarial_port(L, algo, n_rounds):
    """Whole GAIL / AIRL rounds with the reference's Hopper policy (ReLU 64x64, NormalizeFeaturesExtractor) against the
    CPU round driver with the ReLU port, at tests/test_round_parity.py's tolerances.  Every PPO minibatch step's value
    and policy loss is compared as well: it is where the towers' activation in the update shows first."""
    from imitation_b200.util import networks as nets
    from tests import golden_util as G
    from tests.test_round_parity import _run_port

    seed, Do, Da = 5, 11, 3
    tr, port, noise, perms = _relu_rounds(algo, seed, n_rounds)
    want = _run_port(port, n_rounds, seed)
    steps = tr.gen_algo.n_epochs * -(-tr.gen_train_timesteps // tr.gen_algo.batch_size)
    want_loss = np.asarray(port.gen.loss_log, np.float64).reshape(n_rounds, steps, 4)

    th.manual_seed(seed + 7)
    np.random.seed(seed + 11)
    gen = tr.gen_algo
    for r in range(n_rounds):
        gen.noise = th.as_tensor(noise[r]).cuda()
        gen.perm = th.as_tensor(perms[r]).cuda()
        gen.loss_log = th.full((steps, 4), float("nan"), device="cuda")
        tr.train_gen(tr.gen_train_timesteps)
        got_stats = []
        for _ in range(tr.n_disc_updates_per_round):
            with nets.training(tr.reward_train):
                got_stats.append(tr.train_disc())
        tr.join()
        th.cuda.synchronize()
        w = want[r]
        # PPO losses of every minibatch step: pg, value, entropy, total
        np.testing.assert_allclose(gen.loss_log.cpu().numpy(), want_loss[r], rtol=2e-3, atol=2e-4,
                                   err_msg=f"round {r} PPO loss log")
        ring = tr._gen_replay_buffer
        assert int(tr.venv.state[_lib.ST_RING_IDX]) == w["ring_idx"] == ring._idx
        assert int(tr.venv.state[_lib.ST_RING_N]) == w["ring_n"] == ring.size()
        tbl = ring.table.cpu().numpy()
        np.testing.assert_array_equal(tbl[:, -1] > 0.5, w["ring"]["dones"], err_msg=f"round {r} ring dones")
        assert th.equal(th.get_rng_state(), w["torch_rng"]), "expert DataLoader stream out of step"
        np.testing.assert_array_equal(np.random.get_state()[1], w["np_rng"], err_msg="replay index stream out of step")
        np.testing.assert_allclose(tbl[:, :Do], w["ring"]["obs"], rtol=2e-3, atol=3e-4, err_msg=f"round {r} ring obs")
        np.testing.assert_allclose(tbl[:, Do:Do + Da], w["ring"]["acts"], rtol=2e-3, atol=3e-4,
                                   err_msg=f"round {r} ring acts")
        np.testing.assert_allclose(tbl[:, Do + Da:2 * Do + Da], w["ring"]["next_obs"], rtol=2e-3, atol=3e-4)
        for k, (gs, ws) in enumerate(zip(got_stats, w["stats"])):
            for key in ws:
                np.testing.assert_allclose(gs[key], ws[key], rtol=2e-3, atol=2e-4, err_msg=f"round {r} update {k} {key}")
        ours = {G.port_key(k): v.detach().cpu() for k, v in tr._reward_net.state_dict().items()}
        for k, v in w["net"].items():
            if k.endswith("count"):
                assert int(ours[k]) == int(v), k
            else:
                np.testing.assert_allclose(ours[k].numpy(), v.numpy(), rtol=2e-3, atol=2e-4, err_msg=f"round {r} {k}")
        pp = {k: v.detach().cpu() for k, v in tr.policy.state_dict().items()}
        for t, p in (("policy_net", "pi"), ("value_net", "vf")):
            for i in (0, 2):
                np.testing.assert_allclose(pp[f"mlp_extractor.{t}.{i}.weight"].numpy(), w["pol"][f"{p}.{i}.weight"].numpy(),
                                           rtol=5e-3, atol=5e-4, err_msg=f"round {r} {p}.{i}.weight")
        for k in ("action_net.weight", "value_net.bias", "log_std"):
            np.testing.assert_allclose(pp[k].numpy(), w["pol"][k].numpy(), rtol=5e-3, atol=5e-4, err_msg=f"round {r} {k}")
        pn = tr.policy.features_extractor.normalize
        assert int(pn.count) == int(w["pol"]["feat_norm.count"]), "feature-norm count"
        np.testing.assert_allclose(pn.running_mean.cpu().numpy(), w["pol"]["feat_norm.running_mean"].numpy(),
                                   rtol=2e-3, atol=3e-4)
        np.testing.assert_allclose(pn.running_var.cpu().numpy(), w["pol"]["feat_norm.running_var"].numpy(),
                                   rtol=2e-3, atol=3e-4)


@pytest.mark.gpu
def test_hopper_policy_trains_in_preference_comparisons(L):
    """One PreferenceComparisons iteration whose AgentTrainer runs the ReLU Hopper policy on a 3-member ensemble."""
    from imitation_b200.algorithms import preference_comparisons as pc
    from imitation_b200.envs import synth
    from imitation_b200.rewards import reward_nets

    res = []
    for graph in (False, True):
        th.manual_seed(0)
        venv = synth.DeviceVecEnv(11, 3, 8, horizon=16, seed=3)
        members = [reward_nets.BasicRewardNet(venv.observation_space, venv.action_space) for _ in range(3)]
        reward = reward_nets.AddSTDRewardWrapper(
            reward_nets.RewardEnsemble(venv.observation_space, venv.action_space, members).cuda(), default_alpha=-0.5)
        algo = _hopper_ppo(venv, n_steps=64)
        algo.use_cuda_graph = graph
        agent = pc.AgentTrainer(algo, reward, venv, np.random.default_rng(0))
        rng = np.random.default_rng(1)
        pcs = pc.PreferenceComparisons(agent, reward, num_iterations=1,
                                       fragmenter=pc.RandomFragmenter(warning_threshold=0, rng=rng), fragment_length=5,
                                       transition_oversampling=1, initial_comparison_frac=0.5,
                                       initial_epoch_multiplier=1.0, rng=rng)
        p0 = algo.policy.flat_vectors()[0].clone()
        out = pcs.train(total_timesteps=2 * 8 * 64, total_comparisons=16)
        th.cuda.synchronize()
        p1 = algo.policy.flat_vectors()[0]
        assert np.isfinite(out["reward_loss"]) and th.isfinite(p1).all() and not th.equal(p0, p1)
        res.append(p1.clone())
    assert th.equal(res[0], res[1]), "graph replay differs from eager execution"
