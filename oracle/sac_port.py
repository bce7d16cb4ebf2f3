"""CPU restatement of SQIL's continuous-action learner: SB3 2.2's SAC learn loop with SQIL's replay buffer, and the SAC
gradient step in float64.

TEST INFRASTRUCTURE.  SB3 is not installed, so its semantics are restated from SB3 2.2.x (stable_baselines3/common/
off_policy_algorithm.py learn / collect_rollouts / _sample_action, sac/sac.py train, sac/policies.py Actor /
SACPolicy, common/distributions.py SquashedDiagGaussianDistribution, common/policies.py ContinuousCritic /
scale_action / unscale_action, common/utils.py polyak_update), written as that code runs.  Unpinned: re-verify wherever
SB3 is available.

`SACLearnLoopPort.learn` walks the loop and records every global-NumPy draw (SAC's acting draws none: before
learning_starts it takes action_space.sample(), which has its own generator, then the actor's th.randn); the device
SAC's host pass is held to it.  `sac_step` is one SAC.train gradient step in float64 NumPy with a hand-written
backward, itself held to torch autograd; the noise eps of the actor's samples is the caller's.
"""
from typing import Callable, Dict, List, Optional

import numpy as np

from oracle.sqil_port import ReplayBufferPort

LOG_STD_MIN, LOG_STD_MAX = -20.0, 2.0
ACTOR_KEYS = ("w1", "b1", "w2", "b2", "wmu", "bmu", "wls", "bls")
Q_KEYS = ("w1", "b1", "w2", "b2", "w3", "b3")


# ---- the learn loop ------------------------------------------------------------------------------------------------

class SACLearnLoopPort:
    """OffPolicyAlgorithm.learn + SAC for SQIL: the random-step flags, the replay draws and the train() calls."""

    def __init__(self, *, n_envs: int, n_expert: int, buffer_size: int = 1_000_000, learning_starts: int = 100,
                 batch_size: int = 256, train_freq: int = 1, gradient_steps: int = 1):
        self.n_envs, self.learning_starts, self.batch_size = n_envs, learning_starts, batch_size
        self.train_freq, self.gradient_steps = train_freq, gradient_steps
        self.buffer = ReplayBufferPort(buffer_size, n_envs, 1, 0.0)
        self.n_expert = n_expert
        self._n_updates = 0
        self.num_timesteps = 0
        self.random_steps: List[int] = []
        self.samples: List[tuple] = []    # per gradient step: (learner batch_inds, env_inds, expert inds)
        self.train_calls: List[int] = []  # gradient steps of each train() call

    def learn(self, total_timesteps: int, train_fn: Optional[Callable] = None, reset_num_timesteps: bool = True):
        """train_fn(sample, gradient_step) runs one gradient step (gradient_step: its index inside the train() call)."""
        if reset_num_timesteps:
            self.num_timesteps = 0
        else:
            total_timesteps += self.num_timesteps
        while self.num_timesteps < total_timesteps:
            for _ in range(self.train_freq):
                # _sample_action: action_space.sample() before learning_starts, else the actor (no global draws)
                self.random_steps.append(int(self.num_timesteps < self.learning_starts))
                self.num_timesteps += self.n_envs
                self.buffer.add(0.0, 0.0, 0, 0.0)
            if self.num_timesteps > 0 and self.num_timesteps > self.learning_starts:
                gs = self.gradient_steps if self.gradient_steps >= 0 else self.train_freq * self.n_envs
                if gs > 0:
                    self.train_calls.append(gs)
                    for gi in range(gs):
                        n_l = self.batch_size // 2
                        n_e = self.batch_size - n_l
                        bi, ei = self.buffer.sample(n_l)
                        xi = np.random.randint(0, self.n_expert, size=n_e)
                        np.random.randint(0, high=1, size=(n_e,))  # the expert buffer's env index (n_envs 1)
                        self.samples.append((bi, ei, xi))
                        if train_fn:
                            train_fn(self.samples[-1], gi)
                    self._n_updates += gs


# ---- the nets ------------------------------------------------------------------------------------------------------

def scale_action(x, low, high):
    return 2.0 * ((x - low) / (high - low)) - 1.0


def unscale_action(x, low, high):
    return low + (0.5 * (x + 1.0) * (high - low))


def actor_params(flat: np.ndarray, d_obs: int, d_act: int, h: int) -> Dict[str, np.ndarray]:
    """The actor's flat vector (nn.Linear order) as a dict of float64 arrays."""
    shapes = {"w1": (h, d_obs), "b1": (h,), "w2": (h, h), "b2": (h,), "wmu": (d_act, h), "bmu": (d_act,),
              "wls": (d_act, h), "bls": (d_act,)}
    return _unflat(flat, shapes, ACTOR_KEYS)


def critic_params(flat: np.ndarray, d_obs: int, d_act: int, h: int) -> List[Dict[str, np.ndarray]]:
    """A twin critic's flat vector (qf0 then qf1, nn.Linear order) as two dicts."""
    shapes = {"w1": (h, d_obs + d_act), "b1": (h,), "w2": (h, h), "b2": (h,), "w3": (1, h), "b3": (1,)}
    n = sum(int(np.prod(s)) for s in shapes.values())
    flat = np.asarray(flat, np.float64)
    return [_unflat(flat[i * n:(i + 1) * n], shapes, Q_KEYS) for i in range(2)]


def _unflat(flat, shapes, keys):
    out, o = {}, 0
    flat = np.asarray(flat, np.float64)
    for k in keys:
        n = int(np.prod(shapes[k]))
        out[k] = flat[o:o + n].reshape(shapes[k]).copy()
        o += n
    return out


def actor_forward(p, obs):
    """(h1, h2, mean, clamped log_std, clamp mask)."""
    h1 = np.maximum(obs @ p["w1"].T + p["b1"], 0.0)
    h2 = np.maximum(h1 @ p["w2"].T + p["b2"], 0.0)
    mean = h2 @ p["wmu"].T + p["bmu"]
    ls = h2 @ p["wls"].T + p["bls"]
    mask = ((ls >= LOG_STD_MIN) & (ls <= LOG_STD_MAX)).astype(np.float64)
    return h1, h2, mean, np.clip(ls, LOG_STD_MIN, LOG_STD_MAX), mask


def squash(mean, log_std, eps):
    """SquashedDiagGaussian: (g, a = tanh(g), log_prob) with g = mean + std * eps (eps None: the mode)."""
    sd = np.exp(log_std)
    g = mean if eps is None else mean + eps * sd
    a = np.tanh(g)
    logp = np.sum(-((g - mean) ** 2) / (2 * sd * sd) - log_std - np.log(np.sqrt(2 * np.pi)), axis=1)
    logp = logp - np.sum(np.log(1 - a ** 2 + 1e-6), axis=1)
    return g, a, logp


def q_forward(p, x):
    h1 = np.maximum(x @ p["w1"].T + p["b1"], 0.0)
    h2 = np.maximum(h1 @ p["w2"].T + p["b2"], 0.0)
    return h1, h2, (h2 @ p["w3"].T + p["b3"])[:, 0]


def q_backward(p, x, h1, h2, dq):
    """(weight gradients, dL/dx) of one Q net from dL/dQ [B]."""
    g = {"w3": dq[None, :] @ h2, "b3": np.array([dq.sum()])}
    dz2 = (dq[:, None] * p["w3"][0][None, :]) * (h2 > 0)
    g["w2"], g["b2"] = dz2.T @ h1, dz2.sum(0)
    dz1 = (dz2 @ p["w2"]) * (h1 > 0)
    g["w1"], g["b1"] = dz1.T @ x, dz1.sum(0)
    return g, dz1 @ p["w1"]


def adam(p, m, v, g, step: int, lr: float, eps: float = 1e-8):
    """torch Adam (betas 0.9 / 0.999) on one array; step = the count after this step.  Returns (p, m, v)."""
    m = 0.9 * m + 0.1 * g
    v = 0.999 * v + 0.001 * g * g
    bc1, bc2 = 1 - 0.9 ** step, 1 - 0.999 ** step
    return p - (lr / bc1) * m / (np.sqrt(v) / np.sqrt(bc2) + eps), m, v


class SACState:
    """The float64 parameters and Adam moments of one SAC: actor (dict), critic / target (two dicts each), the entropy
    coefficient (log_ent_coef and its moments, or the fixed value)."""

    def __init__(self, actor, critic, target, log_ent_coef: Optional[float], ent_coef: float = 0.0):
        self.actor, self.critic, self.target = actor, critic, target
        self.am = {k: np.zeros_like(x) for k, x in actor.items()}
        self.av = {k: np.zeros_like(x) for k, x in actor.items()}
        self.cm = [{k: np.zeros_like(x) for k, x in q.items()} for q in critic]
        self.cv = [{k: np.zeros_like(x) for k, x in q.items()} for q in critic]
        self.log_ent_coef, self.ent_coef = log_ent_coef, ent_coef
        self.em = self.ev = 0.0
        self.step = 0


def sac_step(st: SACState, obs, acts, next_obs, dones, rewards, eps, eps_next, *, gamma: float, tau: float, lr: float,
             target_entropy: float, polyak: bool) -> Dict[str, float]:
    """One SAC.train gradient step on a minibatch (float64, in place on `st`); eps / eps_next [B][Da]: the actor's noise on
    obs / next_obs.  Returns the step's critic_loss, actor_loss, ent_coef_loss (auto) and ent_coef."""
    B = len(obs)
    st.step += 1
    a_ = st.actor
    h1, h2, mean, ls, mask = actor_forward(a_, obs)
    g, a_pi, logp = squash(mean, ls, eps)
    out = {}
    # 1-2. the entropy coefficient, read before its Adam step
    if st.log_ent_coef is not None:
        ent_coef = np.exp(st.log_ent_coef)
        mterm = np.mean(logp + target_entropy)
        out["ent_coef_loss"] = -(st.log_ent_coef * mterm)
        st.log_ent_coef, st.em, st.ev = adam(st.log_ent_coef, st.em, st.ev, -mterm, st.step, lr)
    else:
        ent_coef = st.ent_coef
    out["ent_coef"] = ent_coef
    # 3. the target
    _, _, mean_n, ls_n, _ = actor_forward(a_, next_obs)
    _, a_n, logp_n = squash(mean_n, ls_n, eps_next)
    xt = np.concatenate([next_obs, a_n], 1)
    qt = np.minimum(q_forward(st.target[0], xt)[2], q_forward(st.target[1], xt)[2])
    y = rewards + (1 - dones) * gamma * (qt - ent_coef * logp_n)
    # 4. the critics
    x = np.concatenate([obs, acts], 1)
    closs = 0.0
    for i in range(2):
        c1, c2, q = q_forward(st.critic[i], x)
        closs += 0.5 * np.mean((q - y) ** 2)
        gq, _ = q_backward(st.critic[i], x, c1, c2, (q - y) / B)
        for k in Q_KEYS:
            st.critic[i][k], st.cm[i][k], st.cv[i][k] = adam(st.critic[i][k], st.cm[i][k], st.cv[i][k], gq[k],
                                                             st.step, lr)
    out["critic_loss"] = closs
    # 5. the actor through the updated critics
    xp = np.concatenate([obs, a_pi], 1)
    fw = [q_forward(st.critic[i], xp) for i in range(2)]
    one = fw[1][2] < fw[0][2]
    minq = np.where(one, fw[1][2], fw[0][2])
    out["actor_loss"] = np.mean(ent_coef * logp - minq)
    da = np.zeros_like(a_pi)
    for i in range(2):
        dq = np.where(one == (i == 1), -1.0 / B, 0.0)
        _, dx = q_backward(st.critic[i], xp, fw[i][0], fw[i][1], dq)
        da += dx[:, obs.shape[1]:]
    om = 1 - a_pi ** 2
    dlogp = 2 * a_pi * om / (om + 1e-6)
    dg = ent_coef / B * dlogp + da * om
    dmu = dg
    dls = mask * (-ent_coef / B + dg * np.exp(ls) * eps)
    ga = {"wmu": dmu.T @ h2, "bmu": dmu.sum(0), "wls": dls.T @ h2, "bls": dls.sum(0)}
    dz2 = (dmu @ a_["wmu"] + dls @ a_["wls"]) * (h2 > 0)
    ga["w2"], ga["b2"] = dz2.T @ h1, dz2.sum(0)
    dz1 = (dz2 @ a_["w2"]) * (h1 > 0)
    ga["w1"], ga["b1"] = dz1.T @ obs, dz1.sum(0)
    for k in ACTOR_KEYS:
        a_[k], st.am[k], st.av[k] = adam(a_[k], st.am[k], st.av[k], ga[k], st.step, lr)
    # 6. Polyak
    if polyak:
        for i in range(2):
            for k in Q_KEYS:
                st.target[i][k] = st.target[i][k] * (1 - tau) + tau * st.critic[i][k]
    return out
