"""Actor-critic policy with SB3's `ActorCriticPolicy` surface over a flat device vector.

Mirrors what the reference's generator uses: `imitation.policies.base.FeedForward32Policy`
(policies/base.py:92-104 = SB3 ActorCriticPolicy(net_arch=[32, 32]): separate tanh towers for
pi and vf, Linear action/value heads, state-independent log_std for Box actions, orthogonal
init with gains sqrt(2)/0.01/1) and `NormalizeFeaturesExtractor` (policies/base.py:123-149:
Flatten -> RunningNorm), and SB3's `MlpPolicy` with the `policy_kwargs` the reference's
configurations pass (scripts/config/train_preference_comparisons.py seals_hopper / walker /
swimmer, tuned_hps/{gail,airl}_seals_*: ReLU 64x64 towers, NormalizeFeaturesExtractor).
Parameter names follow SB3's state_dict so checkpoints map 1:1.
The kernels (csrc/imb_rollout.cu, csrc/imb_ppo.cu) read/write the flat vector the
nn.Parameters alias; `evaluate_actions`/`predict` below are the API-path equivalents in torch.
"""
import math
import warnings
from typing import Optional, Tuple

import numpy as np
import torch as th
from torch import nn

from .. import _desc, _lib, spaces
from ..util import networks
from ..util.flat import FlatAlias


# Where the reference's classes of the same meaning live (its configurations name them; this package imports neither
# the reference nor SB3, so they are recognised by module and name).
_REFERENCE_MODULES = {"RunningNorm": "imitation.util.networks", "NormalizeFeaturesExtractor": "imitation.policies.base",
                      "FlattenExtractor": "stable_baselines3.common.torch_layers"}


def _is_class(cls, ours: type) -> bool:
    """cls is this package's class `ours` or the reference's class of that name in its own module; a user's class that
    only shares the name is neither."""
    if cls is ours:
        return True
    return (isinstance(cls, type) and cls.__name__ == ours.__name__
            and cls.__module__ == _REFERENCE_MODULES.get(ours.__name__))


class NormalizeFeaturesExtractor(nn.Module):
    """Flatten -> RunningNorm.  Takes the reference's (observation_space, normalize_class=RunningNorm) or a flat
    observation width."""

    def __init__(self, observation_space, normalize_class=networks.RunningNorm):
        super().__init__()
        if not _is_class(normalize_class, networks.RunningNorm):
            raise NotImplementedError(f"NormalizeFeaturesExtractor: normalize_class {normalize_class!r} is not "
                                      "supported; the kernels normalise policy features with RunningNorm only")
        d_obs = observation_space if isinstance(observation_space, int) else spaces.flat_dim(observation_space)
        self.features_dim = d_obs
        self.flatten = nn.Flatten()
        self.normalize = networks.RunningNorm(d_obs)

    def forward(self, obs):
        return self.normalize(self.flatten(obs.float()))


class FlattenExtractor(nn.Module):
    def forward(self, obs):
        return th.flatten(obs.float(), 1)


# activation_fn -> the kernels' pol_act code, and back
_ACTIVATIONS = {nn.Tanh: _lib.ACT_TANH, nn.ReLU: _lib.ACT_RELU}
_ACT_MODULES = {code: cls for cls, code in _ACTIVATIONS.items()}


class _MlpExtractor(nn.Module):
    def __init__(self, d_obs, hidden, act=_lib.ACT_TANH):
        super().__init__()
        A = _ACT_MODULES[act]
        self.policy_net = nn.Sequential(nn.Linear(d_obs, hidden), A(), nn.Linear(hidden, hidden), A())
        self.value_net = nn.Sequential(nn.Linear(d_obs, hidden), A(), nn.Linear(hidden, hidden), A())


def _tower_width(net_arch) -> int:
    """The one tower width of an SB3 2.2 `net_arch` the kernels run: [h, h], dict(pi=[h, h], vf=[h, h]), or the
    deprecated [dict(pi=..., vf=...)] (unwrapped with SB3's warning); h <= 64."""
    if isinstance(net_arch, (list, tuple)) and len(net_arch) == 1 and isinstance(net_arch[0], dict):
        warnings.warn("As shared layers in the mlp_extractor are removed since SB3 v1.8.0, you should now pass directly "
                      "a dictionary and not a list (net_arch=dict(pi=..., vf=...) instead of "
                      "net_arch=[dict(pi=..., vf=...)])")
        net_arch = net_arch[0]
    if isinstance(net_arch, dict):
        pi, vf = list(net_arch.get("pi", [])), list(net_arch.get("vf", []))
        if pi != vf:
            raise NotImplementedError(f"net_arch pi={pi}, vf={vf}: the kernels run pi and vf towers of equal widths")
        layers = pi
    else:
        layers = list(net_arch)
    if len(layers) != 2 or layers[0] != layers[1]:
        raise NotImplementedError(f"net_arch {layers}: the kernels run two hidden layers of one width, [h, h]")
    h = int(layers[0])
    if not 1 <= h <= _lib.IMB_MAX_HIDDEN:
        raise NotImplementedError(f"net_arch [{h}, {h}]: the kernels run tower widths 1 to {_lib.IMB_MAX_HIDDEN}")
    return h


def _feature_norm(features_extractor_class, features_extractor_kwargs, normalize_features) -> bool:
    """Whether the features are RunningNorm-normalised, from SB3's features_extractor_class / _kwargs or this package's
    normalize_features (both may be given if they agree)."""
    kw = dict(features_extractor_kwargs or {})
    if features_extractor_class is None:
        if kw:
            raise TypeError("features_extractor_kwargs given without features_extractor_class")
        return bool(normalize_features)
    if _is_class(features_extractor_class, NormalizeFeaturesExtractor):
        cls = kw.pop("normalize_class", networks.RunningNorm)
        if kw:
            raise TypeError(f"NormalizeFeaturesExtractor got unexpected keyword arguments {sorted(kw)}")
        if not _is_class(cls, networks.RunningNorm):
            raise NotImplementedError(f"NormalizeFeaturesExtractor: normalize_class {cls!r} is not supported; the "
                                      "kernels normalise policy features with RunningNorm only")
        norm = True
    elif _is_class(features_extractor_class, FlattenExtractor):
        if kw:
            raise TypeError(f"FlattenExtractor got unexpected keyword arguments {sorted(kw)}")
        norm = False
    else:
        raise NotImplementedError(f"features_extractor_class {features_extractor_class!r}: the kernels run "
                                  "FlattenExtractor or NormalizeFeaturesExtractor(normalize_class=RunningNorm)")
    if normalize_features is not None and bool(normalize_features) != norm:
        raise ValueError(f"normalize_features={normalize_features} contradicts features_extractor_class="
                         f"{features_extractor_class.__name__}")
    return norm


class ActorCriticPolicy(nn.Module):
    """Separate pi/vf towers of two layers of one width h <= 64, tanh (SB3's default) or ReLU.

    Accepts SB3 2.2's `policy_kwargs` as far as the kernels run them: `net_arch` ([h, h], dict(pi=[h, h], vf=[h, h])
    or the deprecated [dict(...)]), `activation_fn` (nn.Tanh or nn.ReLU), `ortho_init`, `log_std_init`,
    `features_extractor_class` / `features_extractor_kwargs` (FlattenExtractor, or NormalizeFeaturesExtractor with
    RunningNorm).  SB3 options whose values the kernels cannot run raise NotImplementedError naming the option:
    use_sde=True, squash_output=True, share_features_extractor=False, an optimizer other than Adam(eps=1e-5)."""

    def __init__(self, observation_space, action_space, net_arch=(32, 32), normalize_features: Optional[bool] = None,
                 log_std_init: float = 0.0, activation_fn=nn.Tanh, ortho_init: bool = True, use_sde: bool = False,
                 full_std: bool = True, use_expln: bool = False, squash_output: bool = False,
                 features_extractor_class=None, features_extractor_kwargs: Optional[dict] = None,
                 share_features_extractor: bool = True, normalize_images: bool = True, optimizer_class=None,
                 optimizer_kwargs: Optional[dict] = None):
        super().__init__()
        hidden = _tower_width(net_arch)
        if activation_fn not in _ACTIVATIONS:
            raise NotImplementedError(f"activation_fn {activation_fn!r}: the kernels run nn.Tanh and nn.ReLU towers")
        if use_sde:
            raise NotImplementedError("use_sde=True: the kernels sample from a state-independent diagonal Gaussian")
        if squash_output:
            raise NotImplementedError("squash_output=True: the kernels do not squash actions (it needs use_sde)")
        if not share_features_extractor:
            raise NotImplementedError("share_features_extractor=False: the kernels run one features extractor for "
                                      "pi and vf (it has no parameters)")
        if optimizer_class not in (None, th.optim.Adam):
            raise NotImplementedError(f"optimizer_class {optimizer_class!r}: the PPO update kernels run Adam")
        if optimizer_kwargs not in (None, {}, {"eps": 1e-5}):
            raise NotImplementedError(f"optimizer_kwargs {optimizer_kwargs!r}: the PPO update kernels run Adam with "
                                      "SB3 PPO's eps=1e-5")
        normalize_features = _feature_norm(features_extractor_class, features_extractor_kwargs, normalize_features)
        self.observation_space, self.action_space = observation_space, action_space
        self.discrete = spaces.is_discrete(action_space)
        self.d_obs = spaces.flat_dim(observation_space)
        self.d_act = spaces.flat_dim(action_space)
        self.hidden = hidden
        self.act = _ACTIVATIONS[activation_fn]  # pol_act of every kernel that evaluates this policy
        self.normalize_features = normalize_features
        self.features_extractor = NormalizeFeaturesExtractor(self.d_obs) if normalize_features else FlattenExtractor()
        self.mlp_extractor = _MlpExtractor(self.d_obs, self.hidden, self.act)
        self.action_net = nn.Linear(self.hidden, self.d_act)
        self.value_net = nn.Linear(self.hidden, 1)
        if not self.discrete:
            self.log_std = nn.Parameter(th.ones(self.d_act) * log_std_init)
        if ortho_init:  # SB3's gains whatever the activation; False keeps torch's default nn.Linear initialisation
            for seq in (self.mlp_extractor.policy_net, self.mlp_extractor.value_net):
                for m in seq:
                    if isinstance(m, nn.Linear):
                        nn.init.orthogonal_(m.weight, gain=math.sqrt(2))
                        nn.init.zeros_(m.bias)
            nn.init.orthogonal_(self.action_net.weight, gain=0.01)
            nn.init.zeros_(self.action_net.bias)
            nn.init.orthogonal_(self.value_net.weight, gain=1.0)
            nn.init.zeros_(self.value_net.bias)
        self.desc = _desc.policy_desc(self.d_obs, self.d_act, self.discrete, self.hidden, normalize_features)
        self._flat: Optional[th.Tensor] = None

    def __getstate__(self):
        st = self.__dict__.copy()
        st["_flat"] = None
        st.pop("_aliases", None)
        st.pop("_norm_state", None)
        st.pop("_norm_count", None)
        return st

    def __setstate__(self, st):
        st.setdefault("act", _lib.ACT_TANH)  # pickles from before ReLU towers existed
        self.__dict__.update(st)
        self.desc = _desc.policy_desc(self.d_obs, self.d_act, self.discrete, self.hidden, self.normalize_features)

    # -- flat vectors for the kernels --------------------------------------------------------------------
    def flat_vectors(self) -> Tuple[th.Tensor, th.Tensor, th.Tensor]:
        """(params, norm_state[mean|var], norm_count) aliased by the module's parameters/buffers."""
        aliases = self.__dict__.get("_aliases")
        if aliases is None:
            names = [name.rpartition(".") for name, _ in
                     _desc.policy_param_shapes(self.d_obs, self.d_act, self.discrete, self.hidden)]
            aliases = [FlatAlias([(self.get_submodule(path), attr) for path, _, attr in names])]
            if self.normalize_features:
                n = self.features_extractor.normalize
                aliases += [FlatAlias([(n, "running_mean"), (n, "running_var")]), FlatAlias([(n, "count")])]
            self.__dict__["_aliases"] = aliases
        dev = aliases[0].tensors()[0].device
        if dev.type != "cuda":
            raise _lib.ImbError("imitation_b200 policies run on CUDA only (no CPU fallback)")
        flat = aliases[0].get(th.float32, dev)
        assert flat.numel() == self.desc.n_params
        if self.normalize_features:
            return flat, aliases[1].get(th.float32, dev), aliases[2].get(th.int32, dev)
        ns = self.__dict__.get("_norm_state")
        if ns is None or ns.device != dev:
            self.__dict__["_norm_state"] = th.zeros(2, device=dev)
            self.__dict__["_norm_count"] = th.zeros(1, dtype=th.int32, device=dev)
        return flat, self._norm_state, self._norm_count

    # -- SB3-compatible API (torch ops; not on the hot path) ------------------------------------------------
    def set_training_mode(self, mode: bool) -> None:
        self.train(mode)

    def _dist(self, obs):
        f = self.features_extractor(obs)
        lat_pi = self.mlp_extractor.policy_net(f)
        lat_vf = self.mlp_extractor.value_net(f)
        out = self.action_net(lat_pi)
        if self.discrete:
            dist = th.distributions.Categorical(logits=out)
        else:
            dist = th.distributions.Normal(out, th.ones_like(out) * self.log_std.exp())
        return dist, self.value_net(lat_vf)

    def forward(self, obs, deterministic: bool = False):
        dist, values = self._dist(obs)
        if self.discrete:
            actions = dist.probs.argmax(1) if deterministic else dist.sample()
            logp = dist.log_prob(actions)
        else:
            actions = dist.mean if deterministic else dist.sample()
            logp = dist.log_prob(actions).sum(1)
        return actions, values, logp

    def evaluate_actions(self, obs, actions):
        dist, values = self._dist(obs)
        if self.discrete:
            return values, dist.log_prob(actions.long().flatten()), dist.entropy()
        return values, dist.log_prob(actions).sum(1), dist.entropy().sum(1)

    def predict_values(self, obs):
        return self._dist(obs)[1]

    def predict(self, observation, state=None, episode_start=None, deterministic: bool = False):
        obs = th.as_tensor(np.asarray(observation)).to(next(self.parameters()).device)
        with th.no_grad(), networks.evaluating(self):
            actions, _, _ = self.forward(obs, deterministic)
        actions = actions.cpu().numpy()
        if not self.discrete:
            actions = np.clip(actions, self.action_space.low, self.action_space.high)
        return actions, state


class FeedForward32Policy(ActorCriticPolicy):
    """policies/base.py:92-104."""

    def __init__(self, observation_space, action_space, **kwargs):
        kwargs.pop("net_arch", None)
        super().__init__(observation_space, action_space, net_arch=(32, 32), **kwargs)
