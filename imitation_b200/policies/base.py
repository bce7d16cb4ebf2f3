"""Actor-critic policy with SB3's `ActorCriticPolicy` surface over a flat device vector.

Mirrors what the reference's generator uses: `imitation.policies.base.FeedForward32Policy`
(policies/base.py:92-104 = SB3 ActorCriticPolicy(net_arch=[32, 32]): separate tanh towers for
pi and vf, Linear action/value heads, state-independent log_std for Box actions, orthogonal
init with gains sqrt(2)/0.01/1) and `NormalizeFeaturesExtractor` (policies/base.py:123-149:
Flatten -> RunningNorm).  Parameter names follow SB3's state_dict so checkpoints map 1:1.
The kernels (csrc/imb_rollout.cu, csrc/imb_ppo.cu) read/write the flat vector the
nn.Parameters alias; `evaluate_actions`/`predict` below are the API-path equivalents in torch.
"""
import math
from typing import Optional, Tuple

import numpy as np
import torch as th
from torch import nn

from .. import _desc, _lib, spaces
from ..util import networks
from ..util.flat import FlatAlias


class NormalizeFeaturesExtractor(nn.Module):
    def __init__(self, d_obs: int):
        super().__init__()
        self.flatten = nn.Flatten()
        self.normalize = networks.RunningNorm(d_obs)

    def forward(self, obs):
        return self.normalize(self.flatten(obs.float()))


class FlattenExtractor(nn.Module):
    def forward(self, obs):
        return th.flatten(obs.float(), 1)


class _MlpExtractor(nn.Module):
    def __init__(self, d_obs, hidden):
        super().__init__()
        self.policy_net = nn.Sequential(nn.Linear(d_obs, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())
        self.value_net = nn.Sequential(nn.Linear(d_obs, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())


class ActorCriticPolicy(nn.Module):
    """`net_arch=[h, h]` separate pi/vf towers (h <= 64), tanh."""

    def __init__(self, observation_space, action_space, net_arch=(32, 32), normalize_features: bool = False,
                 log_std_init: float = 0.0):
        super().__init__()
        if len(net_arch) != 2 or net_arch[0] != net_arch[1]:
            raise NotImplementedError("fused policy supports net_arch=[h, h] (FeedForward32Policy / SB3 default)")
        self.observation_space, self.action_space = observation_space, action_space
        self.discrete = spaces.is_discrete(action_space)
        self.d_obs = spaces.flat_dim(observation_space)
        self.d_act = spaces.flat_dim(action_space)
        self.hidden = int(net_arch[0])
        self.normalize_features = normalize_features
        self.features_extractor = NormalizeFeaturesExtractor(self.d_obs) if normalize_features else FlattenExtractor()
        self.mlp_extractor = _MlpExtractor(self.d_obs, self.hidden)
        self.action_net = nn.Linear(self.hidden, self.d_act)
        self.value_net = nn.Linear(self.hidden, 1)
        if not self.discrete:
            self.log_std = nn.Parameter(th.ones(self.d_act) * log_std_init)
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
