"""AIRL (mirror of imitation.algorithms.adversarial.airl:15-132)."""
from typing import Optional

import torch as th

from ...policies import base as policies
from ...rewards import reward_nets
from . import common

STOCHASTIC_POLICIES = (policies.ActorCriticPolicy,)


class AIRL(common.AdversarialTrainer):
    _needs_logp = True

    def __init__(self, *, demonstrations, demo_batch_size: int, venv, gen_algo, reward_net, **kwargs):
        super().__init__(demonstrations=demonstrations, demo_batch_size=demo_batch_size, venv=venv,
                         gen_algo=gen_algo, reward_net=reward_net, **kwargs)
        if not isinstance(self.gen_algo.policy, STOCHASTIC_POLICIES):
            raise TypeError("AIRL needs a stochastic policy to compute the discriminator output.")
        if self._fused:
            # the fused kernels subtract log pi(a|s) inside the logit (airl.py:118-119)
            self._fused_net._engine.desc.subtract_logp = 1
            self._fused_net._engine.check_plan()  # the log pi row is one more staged batch row

    def logits_expert_is_high(self, state, action, next_state, done, log_policy_act_prob: Optional[th.Tensor] = None
                              ) -> th.Tensor:
        if log_policy_act_prob is None:
            raise TypeError("Non-None `log_policy_act_prob` is required for this method.")
        reward_output_train = self._reward_net(state, action, next_state, done)
        return reward_output_train - log_policy_act_prob

    @property
    def reward_train(self) -> reward_nets.RewardNet:
        return self._reward_net

    @property
    def reward_test(self) -> reward_nets.RewardNet:
        reward_net = self._reward_net
        while isinstance(reward_net, reward_nets.RewardNetWrapper):
            reward_net = reward_net.base
        return reward_net
