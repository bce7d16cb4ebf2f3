"""DAgger on the device: `imb_rollout_dagger` and `algorithms.dagger` (reference algorithms/dagger.py).

CPU: the beta schedules and their error (against the reference's own classes where its sources are importable), the
host's draws from `rng` (the masks, the file names and their listing order with E >= 11 envs, so `dagger-demo-10-...`
sorts before `dagger-demo-2-...`), and the DAgger rollout's tile plan.
GPU: the kernel against its float64 twin (oracle/dagger_port.py) over Box and Discrete, the four expert x learner
activation pairs at unequal widths, a feature RunningNorm on either policy, every tile, beta in {0, 0.5, 1} and a
deterministic or stochastic expert; beta = 1 never evaluating a NaN learner and giving the expert-only rollout's bits;
`SimpleDAggerTrainer.train` end to end (the aggregate table against the files on disk, counters, log keys, training
modes), the low-level API giving `train`'s bits, `NeedsDemosException`, and save -> reconstruct -> continue giving an
uninterrupted run's bits.
"""
import os

import numpy as np
import pytest
import torch as th
from torch import nn

from imitation_b200.algorithms import dagger


def _reference():
    from oracle import refimport

    if not refimport.available():
        return None
    try:
        refimport.load()
        from imitation.algorithms import dagger as ref_dagger
    except Exception:  # the reference's optional dependencies are not all shimmed
        return None
    return ref_dagger


# ---------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------
def test_beta_schedules_and_error():
    lin, exp = dagger.LinearBetaSchedule(15), dagger.ExponentialBetaSchedule(0.7)
    assert [lin(r) for r in (0, 1, 15, 20)] == [1, 14 / 15, 0, 0]
    assert [exp(r) for r in (0, 1, 3)] == [1, 0.7, 0.7 ** 3]
    for p in (0.0, -0.1, 1.5):
        with pytest.raises(ValueError, match=r"decay_probability lies outside the range \(0, 1\]\."):
            dagger.ExponentialBetaSchedule(p)
    ref = _reference()
    if ref is not None:
        for r in range(20):
            assert lin(r) == ref.LinearBetaSchedule(15)(r) and exp(r) == ref.ExponentialBetaSchedule(0.7)(r)
        with pytest.raises(ValueError):
            ref.ExponentialBetaSchedule(0.0)


def test_rng_draws_follow_the_reference_step_loop():
    """H steps of `uniform(size=E) > beta`, then E `bytes(16)` file names, per batch; `shuffle` at the end."""
    E, H, beta = 12, 5, 0.5
    mine, ref = np.random.default_rng(3), np.random.default_rng(3)
    names = []
    for _ in range(2):
        mask = dagger.draw_robot_mask(mine, H, E, beta)
        names += [dagger.demo_file_name(e, mine) for e in range(E)]
        want = np.stack([ref.uniform(0, 1, size=(E,)) > beta for _ in range(H)])
        np.testing.assert_array_equal(mask, want.astype(np.uint8))
        for e in range(E):
            import uuid

            u = uuid.UUID(int=int.from_bytes(ref.bytes(16), "big"), version=4).hex
            assert names[-E + e] == f"dagger-demo-{e}-{u}.npz"
    assert mine.bit_generator.state == ref.bit_generator.state
    listing = sorted(names)
    assert listing.index(next(n for n in names if n.startswith("dagger-demo-10-"))) < \
        listing.index(next(n for n in names if n.startswith("dagger-demo-2-")))
    assert dagger.demo_file_name(0, np.random.default_rng(0), "initial_data").startswith("initial_data-dagger-demo-0-")


def test_dagger_plan_falls_back_when_both_images_do_not_fit():
    from imitation_b200 import _desc, _lib

    n_sms = 132
    sizes = (37, 24 * n_sms, 100 * n_sms, 129 * n_sms)
    e, lrn = _desc.policy_desc(17, 6, False, 64, False), _desc.policy_desc(17, 6, False, 32, True)
    assert [_lib.rollout_dagger_plan(e, lrn, n, n_sms) for n in sizes] == [8, 32, 64, 128]
    wide = _desc.policy_desc(64, 8, False, 64, True)
    assert [_lib.rollout_dagger_plan(wide, wide, n, n_sms) for n in sizes] == [8, 32, 32, 32]
    with pytest.raises(_lib.ImbError, match="space mismatch"):
        _lib.rollout_dagger_plan(e, _desc.policy_desc(17, 5, False, 32, False), 8, n_sms)


# ---------------------------------------------------------------------------------------------
# GPU: the kernel against its twin
# ---------------------------------------------------------------------------------------------
def _dev(x):
    return th.as_tensor(np.ascontiguousarray(x)).cuda().contiguous()


def _port(Do, Da, discrete, width, act, norm, seed):
    from oracle import ppo_port

    th.manual_seed(seed)
    pol = ppo_port.ActorCriticPort(Do, Da, discrete=discrete, hidden=(width, width), normalize_features=norm)
    with th.no_grad():
        for p in pol.parameters():
            p.add_(0.3 * th.randn_like(p))
        if norm:
            pol.feat_norm.running_mean.normal_(0, 0.1)
            pol.feat_norm.running_var.uniform_(0.5, 1.5)
    if act == "relu":
        for tower in (pol.pi, pol.vf):
            tower[1], tower[3] = nn.ReLU(), nn.ReLU()
    return pol


def _device_policy(L, pol, width, norm):
    from imitation_b200 import _desc
    from tests.test_gpu_kernels import _policy_flat

    desc = _desc.policy_desc(pol.d_obs, pol.d_act, pol.discrete, width, norm)
    pn = (th.cat([pol.feat_norm.running_mean, pol.feat_norm.running_var]).float().cuda() if norm
          else th.zeros(2, device="cuda"))
    return desc, _policy_flat(pol).cuda(), pn


class _Case:
    def __init__(self, L, discrete, eact, lact, ew, lw, enorm, lnorm, E, H=6, seed=5):
        from imitation_b200 import _desc

        self.L, self.discrete, self.E, self.H, self.seed = L, discrete, E, H, seed
        self.Do, self.Da = (4, 3) if discrete else (11, 3)
        Do, Da = self.Do, self.Da
        self.expert = _port(Do, Da, discrete, ew, eact, enorm, seed)
        self.learner = _port(Do, Da, discrete, lw, lact, lnorm, seed + 1)
        self.eact = L.ACT_RELU if eact == "relu" else L.ACT_TANH
        self.lact = L.ACT_RELU if lact == "relu" else L.ACT_TANH
        self.ed, self.EP, self.EN = _device_policy(L, self.expert, ew, enorm)
        self.ld, self.LP, self.LN = _device_policy(L, self.learner, lw, lnorm)
        self.env = L.EnvDesc(d_obs=Do, d_act=Da, discrete=int(discrete), horizon=H, seed=seed, env_id_offset=5)
        self.envp = _dev(_desc.synth_env_params(Do, Da, seed))
        self.rw = L.rollout_row_width(self.ed)
        self.tw = _desc.table_width(Do, Da)
        rng = np.random.default_rng(seed)
        shape = (H, E) if discrete else (H, E, Da)
        draw = rng.random if discrete else rng.standard_normal
        self.noise, self.robot_noise = draw(shape).astype(np.float32), draw(shape).astype(np.float32)

    def run(self, mask, deterministic, learner_params=None, pinned=True):
        L, E, H = self.L, self.E, self.H
        st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
        obs = th.empty(self.Do, E, device="cuda")
        L.env_reset(obs, E, self.env, st)
        tbl = th.zeros(E * H, self.rw, device="cuda")
        flat = th.zeros(E * H, self.tw, device="cuda")
        aux = th.zeros(2 * E + 2 * E * H, device="cuda")
        L.rollout_dagger(self.env, self.envp, obs, self.ed, self.EP, self.EN, self.ld,
                         self.LP if learner_params is None else learner_params, self.LN, E, H, tbl, flat, aux,
                         _dev(self.noise) if pinned else None, _dev(self.robot_noise) if pinned else None, _dev(mask),
                         st, flags=L.IMB_RF_DETERMINISTIC if deterministic else 0, expert_act=self.eact,
                         learner_act=self.lact)
        th.cuda.synchronize()
        return tbl, flat, aux, obs

    def twin(self, mask, deterministic):
        from oracle import dagger_port, synth_env

        spec = synth_env.SynthEnvSpec(self.Do, self.Da, discrete=self.discrete, horizon=self.H, seed=self.seed)
        obs0 = spec.reset_obs(np.arange(self.E) + 5, np.zeros(self.E))
        return dagger_port.collect(spec, self.expert, self.learner, obs0, mask, self.noise, self.robot_noise,
                                   deterministic)

    def check(self, tbl, flat, aux, want):
        E, H, Do, Da = self.E, self.H, self.Do, self.Da
        got = tbl.cpu().numpy().reshape(E, H, self.rw)
        # float32 device arithmetic (tanh.approx towers) against float64 over H steps
        np.testing.assert_allclose(got[:, :, :Do], want["obs"], rtol=1e-3, atol=1e-3, err_msg="obs")
        if self.discrete:
            np.testing.assert_array_equal(got[:, :, Do], want["labels"])
        else:
            np.testing.assert_allclose(got[:, :, Do:Do + Da], want["labels"], rtol=1e-3, atol=1e-3, err_msg="label")
            assert np.abs(got[:, :, Do:Do + Da]).max() <= 1.0
        gf = flat.cpu().numpy().reshape(E, H, self.tw)
        np.testing.assert_allclose(gf[:, :, Do + Da:2 * Do + Da], want["next_obs"], rtol=1e-3, atol=1e-3,
                                   err_msg="next obs")
        rews = aux.cpu().numpy()[2 * E + E * H:].reshape(E, H)
        np.testing.assert_allclose(rews, want["rews"], rtol=1e-3, atol=1e-3, err_msg="env reward")


def _envs_for_tile(rows):
    n_sms = th.cuda.get_device_properties(0).multi_processor_count
    return {8: 37, 32: 24 * n_sms, 64: 100 * n_sms, 128: 129 * n_sms}[rows]


# (discrete, expert act, learner act, expert width, learner width, expert norm, learner norm, tile, beta, deterministic)
KERNEL_CASES = (
    [(d, ea, la, 64, 32, False, False, 8, 0.5, True) for d in (False, True) for ea in ("tanh", "relu")
     for la in ("tanh", "relu")]
    + [(False, "tanh", "relu", 32, 64, True, False, 8, 0.5, False), (True, "relu", "tanh", 32, 64, False, True, 8, 0.5,
                                                                        False)]
    + [(False, "relu", "tanh", 64, 32, False, True, t, b, det) for t in (32, 64, 128) for b, det in
       ((0.0, True), (0.5, False), (1.0, True))]
    + [(True, "tanh", "tanh", 64, 32, True, True, 8, b, False) for b in (0.0, 1.0)])


@pytest.fixture(scope="module")
def L():
    from imitation_b200 import _lib

    _lib.lib()
    return _lib


@pytest.mark.gpu
@pytest.mark.parametrize("discrete,eact,lact,ew,lw,enorm,lnorm,tile,beta,det", KERNEL_CASES)
def test_dagger_rollout_matches_twin(L, discrete, eact, lact, ew, lw, enorm, lnorm, tile, beta, det):
    S = _Case(L, discrete, eact, lact, ew, lw, enorm, lnorm, _envs_for_tile(tile))
    assert L.rollout_dagger_plan(S.ed, S.ld, S.E) == tile
    mask = dagger.draw_robot_mask(np.random.default_rng(1), S.H, S.E, beta)
    tbl, flat, aux, _ = S.run(mask, det)
    S.check(tbl, flat, aux, S.twin(mask, det))


@pytest.mark.gpu
@pytest.mark.parametrize("discrete", [False, True])
def test_beta_one_never_runs_the_learner_and_gives_the_expert_rollout(L, discrete):
    S = _Case(L, discrete, "relu", "tanh", 64, 32, True, False, 300)
    mask = dagger.draw_robot_mask(np.random.default_rng(2), S.H, S.E, 1.0)
    assert not mask.any()
    nan_params = th.full_like(S.LP, float("nan"))
    for det, pinned in ((True, False), (False, True), (False, False)):
        tbl, flat, aux, obs = S.run(mask, det, learner_params=nan_params, pinned=pinned)
        assert th.isfinite(tbl).all() and th.isfinite(flat).all() and th.isfinite(aux).all()
        # the expert-only rollout: imb_rollout with the same expert, sampling and env
        E, H = S.E, S.H
        st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
        obs2 = th.empty(S.Do, E, device="cuda")
        L.env_reset(obs2, E, S.env, st)
        tbl2, flat2 = th.zeros_like(tbl), th.zeros_like(flat)
        aux2 = th.zeros_like(aux)
        hp = L.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                          lr=0.0, adam_eps=1e-5, n_epochs=1, batch_size=1, normalize_advantage=0)
        L.rollout(S.env, S.envp, obs2, S.ed, S.EP, S.EN, None, None, None, 0, hp, E, H, tbl2, None, 0, flat2, aux2,
                  _dev(S.noise) if pinned else None, st, flags=L.IMB_RF_DETERMINISTIC if det else 0, act=S.eact)
        th.cuda.synchronize()
        Do, da = S.Do, 1 if discrete else S.Da
        assert th.equal(tbl[:, :Do], tbl2[:, :Do])
        want = tbl2[:, Do:Do + da] if discrete else tbl2[:, Do:Do + da].clamp(-1.0, 1.0)
        assert th.equal(tbl[:, Do:Do + da], want)
        assert th.equal(flat, flat2) and th.equal(obs, obs2)
        assert th.equal(aux[2 * E + E * H:], aux2[2 * E + E * H:])


# ---------------------------------------------------------------------------------------------
# GPU: the trainer
# ---------------------------------------------------------------------------------------------
def _trainer(tmp, E=11, H=8, seed=0, expert_trajs=True, discrete=False):
    from imitation_b200.algorithms import bc
    from imitation_b200.envs import synth
    from imitation_b200.policies import base as policies
    from imitation_b200.util import logger as imit_logger

    venv = synth.DeviceVecEnv(4, 3, E, discrete=discrete, horizon=H, seed=3)
    th.manual_seed(seed)
    expert = policies.ActorCriticPolicy(venv.observation_space, venv.action_space, net_arch=[64, 64],
                                        activation_fn=nn.ReLU).cuda()
    with th.no_grad():
        expert.action_net.weight.normal_(0, 0.5)
    rng = np.random.default_rng(seed)
    logger = imit_logger.configure()  # shared, as the reference's scripts share it: BC.train dumps DAgger's records
    learner_bc = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng,
                       batch_size=16, custom_logger=logger)
    trajs = None
    if expert_trajs:
        from imitation_b200.data import rollout

        trajs = rollout.generate_trajectories(expert, venv, rollout.make_min_episodes(2), np.random.default_rng(9),
                                              deterministic_policy=True)[:2]
    return dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp, expert_policy=expert, rng=rng, bc_trainer=learner_bc,
                                      expert_trajs=trajs, beta_schedule=dagger.ExponentialBetaSchedule(0.5),
                                      custom_logger=logger), venv


def _aggregate_from_files(tr):
    from imitation_b200.algorithms import bc
    from imitation_b200.data import serialize

    rows = []
    for r in range(tr._last_loaded_round + 1):
        for p in tr._get_demo_paths(tr._demo_dir_path_for_round(r)):
            t = serialize.load(p)[0]
            rows.append(bc.demo_table(tr.policy, t.obs[:-1], t.acts))
    return th.cat(rows)


def _snapshot(tr):
    return (tr.policy.flat_vectors()[0].clone(), tr.bc_trainer.exp_avg.clone(), tr.bc_trainer.exp_avg_sq.clone(),
            tr._all_rows.table[:tr._all_rows.n].clone(), tr.rng.bit_generator.state)


@pytest.mark.gpu
@pytest.mark.parametrize("discrete", [False, True])
def test_simple_dagger_train_end_to_end(L, tmp_path, discrete):
    th.manual_seed(0)
    tr, venv = _trainer(tmp_path, discrete=discrete)
    E, H = venv.num_envs, venv.horizon
    tr.train(3 * E * H, rollout_round_min_episodes=E, rollout_round_min_timesteps=E * H,
             bc_train_kwargs=dict(n_epochs=2, log_interval=1))
    th.cuda.synchronize()
    assert tr.round_num == 3 and tr._last_loaded_round == 2
    for r in range(3):
        names = os.listdir(tr._demo_dir_path_for_round(r))
        assert len(names) == E + (2 if r == 0 else 0)
    agg = tr._all_rows.table[:tr._all_rows.n].cpu()
    files = _aggregate_from_files(tr)
    assert tr._all_rows.n == (3 * E + 2) * H
    assert th.equal(agg[:, :venv.d_obs + (1 if discrete else 3)], files[:, :venv.d_obs + (1 if discrete else 3)])
    keys = set().union(*(kv.keys() for _, kv in tr.logger.history))
    for k in ("dagger/mean_episode_reward", "dagger/total_timesteps", "dagger/round_num", "dagger/round_episode_count",
              "dagger/round_timestep_count", "bc/loss"):
        assert k in keys
    last = [kv for _, kv in tr.logger.history if "dagger/round_num" in kv][-1]
    assert last["dagger/round_num"] == 2 and last["dagger/total_timesteps"] == 3 * E * H
    assert last["dagger/round_episode_count"] == E and last["dagger/round_timestep_count"] == E * H
    assert not tr.policy.training and not tr.expert_policy.training
    assert th.isfinite(tr.policy.flat_vectors()[0]).all()


@pytest.mark.gpu
def test_low_level_api_and_reconstruct_give_train_bits(L, tmp_path):
    from imitation_b200.data import rollout

    kw = dict(n_epochs=2, log_rollouts_venv=None)
    runs = {}
    for mode in ("train", "low", "reload"):
        th.manual_seed(1)
        tr, venv = _trainer(tmp_path / mode)
        E, H = venv.num_envs, venv.horizon
        if mode == "train":
            tr.train(3 * E * H, rollout_round_min_episodes=E, rollout_round_min_timesteps=E * H, bc_train_kwargs=kw)
        else:
            for r in range(3):
                if mode == "reload" and r == 2:
                    tr.save_trainer()
                    torch_state = th.get_rng_state()
                    tr = dagger.reconstruct_trainer(tmp_path / mode, venv)
                    th.set_rng_state(torch_state)
                collector = tr.create_trajectory_collector()
                su = rollout.make_sample_until(min_timesteps=max(E * H, tr.batch_size), min_episodes=E)
                rollout.generate_trajectories(tr.expert_policy, collector, su, rng=collector.rng,
                                              deterministic_policy=True)
                tr.extend_and_update(kw)
        th.cuda.synchronize()
        runs[mode] = _snapshot(tr)
    for mode in ("low", "reload"):
        for a, b in zip(runs["train"][:4], runs[mode][:4]):
            assert th.equal(a, b), mode
        assert runs["train"][4] == runs[mode][4]
    # an empty round directory raises
    tr, venv = _trainer(tmp_path / "empty", expert_trajs=False)
    with pytest.raises(dagger.NeedsDemosException):
        tr.extend_and_update(kw)


@pytest.mark.gpu
def test_collector_refuses_host_callables_and_host_stepping(L, tmp_path):
    tr, venv = _trainer(tmp_path, expert_trajs=False)
    with pytest.raises(NotImplementedError):
        dagger.InteractiveTrajectoryCollector(venv, lambda obs: obs, 0.5, tmp_path, np.random.default_rng(0))
    c = tr.create_trajectory_collector()
    with pytest.raises(NotImplementedError):
        c.step_async(np.zeros((venv.num_envs, 3), np.float32))
    from imitation_b200.policies import base as policies
    from imitation_b200 import spaces

    other = policies.ActorCriticPolicy(spaces.Box(-np.inf, np.inf, (5,), np.float32), venv.action_space).cuda()
    with pytest.raises(ValueError, match="Mismatched observation space"):
        dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp_path, expert_policy=other, rng=np.random.default_rng(0),
                                   bc_trainer=tr.bc_trainer)


# ---------------------------------------------------------------------------------------------
# GPU: the device trainer against the reference's recorded bookkeeping and a float64 BC
# ---------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_trainer_matches_reference_golden_and_bc_port(L, tmp_path, monkeypatch):
    """`SimpleDAggerTrainer.train` on the device env at tests/test_dagger_reference.py's recorded configuration: the
    masks, file names, listing order, dataset size, shuffles, generator state and logger records of every round are
    the reference's (tests/golden/dagger.npz), and after every round the learner's parameters and Adam moments match
    oracle/bc_port.py trained in float64 on the files' rows in listing order with the reference loader's batches."""
    from imitation_b200.algorithms import bc
    from imitation_b200.data import serialize, types
    from imitation_b200.envs import synth
    from imitation_b200.policies import base as policies
    from imitation_b200.util import logger as imit_logger
    from oracle import bc_port
    from tests import golden_util as G
    from tests import test_dagger_reference as R

    z = G.load("dagger")
    venv = synth.DeviceVecEnv(R.D_OBS, R.D_ACT, R.E, horizon=R.H, seed=R.ENV_SEED)
    th.manual_seed(0)
    expert = policies.ActorCriticPolicy(venv.observation_space, venv.action_space, net_arch=[64, 64]).cuda()

    class Log(imit_logger.HierarchicalLogger):
        def __init__(self):
            super().__init__()
            self.calls = []

        def record(self, key, val, exclude=None):
            if key.startswith("dagger/"):
                self.calls.append((f"record:{key}", float(val)))
            super().record(key, val, exclude)

        def record_mean(self, key, val, exclude=None, _direct=False):
            if key.startswith("dagger/"):
                self.calls.append((f"record_mean:{key}", float(val)))
            super().record_mean(key, val, exclude, _direct)

    log = Log()
    rng = np.random.default_rng(R.SEED)
    learner_bc = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng,
                       batch_size=R.BATCH, custom_logger=log)
    params0 = learner_bc.policy.flat_vectors()[0].detach().cpu().numpy().astype(np.float64)
    initial = [types.Trajectory(obs=o, acts=a, infos=None, terminal=True)
               for o, a in zip(z["initial/obs"], z["initial/acts"])]
    tr = dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp_path, expert_policy=expert, rng=rng,
                                    bc_trainer=learner_bc, expert_trajs=initial, custom_logger=log,
                                    beta_schedule=dagger.ExponentialBetaSchedule(R.DECAY))
    assert sorted(os.listdir(tr._demo_dir_path_for_round(0))) == sorted(z["initial/written"].tolist())

    masks, perms, rounds = [], [], []
    draw = dagger.draw_robot_mask
    monkeypatch.setattr(dagger, "draw_robot_mask", lambda *a: masks.append(draw(*a)) or masks[-1])
    perm_fn = bc.epoch_permutation
    monkeypatch.setattr(bc, "epoch_permutation", lambda n, mb: perms.append(perm_fn(n, mb)) or perms[-1])
    train = learner_bc.train

    def seeded_train(**kw):
        th.manual_seed(100 + tr.round_num)  # the recorder's stub seeds its loader likewise
        return train(**kw)

    learner_bc.train = seeded_train
    extend = tr.extend_and_update

    def recorded_extend(kw=None):
        r = tr.round_num
        written = [n for n in sorted(os.listdir(tr._demo_dir_path_for_round(r))) if not n.startswith("initial")]
        out = extend(kw)
        th.cuda.synchronize()
        rounds.append(dict(masks=np.concatenate(masks), written=written, perms=[p.numpy() for p in perms],
                           calls=list(log.calls), n=tr._all_rows.n, rng=R._fingerprint(rng),
                           params=tr.policy.flat_vectors()[0].cpu().numpy(),
                           exp_avg=tr.bc_trainer.exp_avg.cpu().numpy(), exp_avg_sq=tr.bc_trainer.exp_avg_sq.cpu().numpy()))
        masks.clear()
        perms.clear()
        log.calls.clear()
        return out

    tr.extend_and_update = recorded_extend
    tr.train(R.ROUNDS * 2 * R.E * R.H, rollout_round_min_episodes=R.MIN_EPISODES,
             rollout_round_min_timesteps=R.MIN_TIMESTEPS, bc_train_kwargs=dict(n_epochs=R.EPOCHS, log_rollouts_venv=None))
    assert len(rounds) == R.ROUNDS

    port = bc_port.BCPort(bc_port.make_policy(R.D_OBS, R.D_ACT, False, 32, False), R.BATCH, R.BATCH)
    bc_port.set_flat(port.policy, params0)
    for r, got in enumerate(rounds):
        np.testing.assert_array_equal(got["masks"], z[f"mask/{r}"])
        assert got["written"] == sorted(z[f"written/{r}"].tolist())
        assert got["n"] == int(z[f"n_rows/{r}"])
        np.testing.assert_array_equal(np.array([p[:got["n"] // R.BATCH * R.BATCH] for p in got["perms"]]),
                                      z[f"perm/{r}"])
        np.testing.assert_array_equal(got["rng"], z[f"rng_after/{r}"])
        keys = [k for k, _ in got["calls"]]
        assert keys == z[f"log/{r}/keys"].tolist()
        want_vals = dict(zip(keys, z[f"log/{r}/values"]))
        for k in ("record:dagger/total_timesteps", "record:dagger/round_num", "record:dagger/round_episode_count",
                  "record:dagger/round_timestep_count"):
            assert dict(got["calls"])[k] == want_vals[k], k
        # BC on the reference's dataset: every file so far in the reference's listing order, its recorded batches
        rows = []
        for q in range(r + 1):
            d = tr._demo_dir_path_for_round(q)
            rows += [serialize.load(d / name)[0] for name in z[f"listing/{q}"].tolist()]
        obs = np.concatenate([t.obs[:-1] for t in rows])
        acts = np.concatenate([t.acts for t in rows])
        assert len(obs) == got["n"]
        per_epoch = got["n"] // R.BATCH
        port.train(obs, acts, list(z[f"perm/{r}"]), R.EPOCHS * per_epoch, norm_update=False)
        np.testing.assert_allclose(got["params"], bc_port.get_flat(port.policy), rtol=1e-3, atol=2e-4,
                                   err_msg=f"round {r}")
        np.testing.assert_allclose(got["exp_avg"], bc_port.adam_state(port.opt, port.policy, "exp_avg"), rtol=1e-3,
                                   atol=1e-4, err_msg=f"round {r}")
    # the reference's errors
    tr2 = dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp_path / "e", expert_policy=expert,
                                     rng=np.random.default_rng(0), bc_trainer=learner_bc)
    with pytest.raises(dagger.NeedsDemosException) as e:
        tr2.extend_and_update()
    assert str(e.value).replace(str(tmp_path / "e"), "<scratch>") == str(z["errors/needs_demos"])
    big = bc.BC(observation_space=venv.observation_space, action_space=venv.action_space, rng=rng,
                batch_size=10 * R.H)
    tr3 = dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp_path / "f", expert_policy=expert,
                                     rng=np.random.default_rng(0), bc_trainer=big, expert_trajs=initial[:1])
    with pytest.raises(ValueError) as e:
        tr3.extend_and_update()
    assert str(e.value) == str(z["errors/few_transitions"])
    from imitation_b200 import spaces

    other = policies.ActorCriticPolicy(spaces.Box(-np.inf, np.inf, (R.D_OBS + 1,), np.float32), venv.action_space)
    with pytest.raises(ValueError) as e:
        dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp_path / "g", expert_policy=other.cuda(),
                                   rng=np.random.default_rng(0), bc_trainer=learner_bc)
    assert str(e.value) == str(z["errors/obs_space"])


@pytest.mark.gpu
def test_unpinned_learner_draws_its_own_philox_stream(L):
    """With no pinned noise the learner samples from IMB_STREAM_DAGGER: reproducible, not the expert's
    IMB_STREAM_ACT_NOISE draws, and distributed as N(mean, std) around the learner's mean."""
    S = _Case(L, False, "tanh", "tanh", 32, 32, False, False, 4096, H=1)
    with th.no_grad():  # actions well inside the Box, so clipping leaves the distribution alone
        S.learner.action_net.weight.mul_(0.1)
        S.learner.action_net.bias.zero_()
        S.learner.log_std.fill_(float(np.log(0.2)))
    S.ld, S.LP, S.LN = _device_policy(L, S.learner, 32, False)
    ones = np.ones((1, S.E), np.uint8)
    a1 = S.run(ones, True, pinned=False)[0].cpu().numpy()
    a2 = S.run(ones, True, pinned=False)[0].cpu().numpy()
    assert np.array_equal(a1, a2)
    # the executed learner action is next-obs' control; recover it from the twin's dynamics on the recorded obs
    from oracle import dagger_port, synth_env

    spec = synth_env.SynthEnvSpec(S.Do, S.Da, horizon=1, seed=S.seed)
    tbl, flat, _, _ = S.run(ones, True, pinned=False)
    u = flat.cpu().numpy()[:, S.Do:S.Do + S.Da]  # the control the env saw (the clipped learner action)
    obs = tbl.cpu().numpy()[:, :S.Do]
    pol = dagger_port._float64(S.learner)
    with th.no_grad():
        mean = pol._dist(pol.features(th.as_tensor(obs, dtype=th.float64))).mean.numpy()
    std = np.exp(S.learner.log_std.detach().numpy().astype(np.float64))
    inside = np.abs(u) < 0.999
    z = ((u - mean) / std)[inside]
    assert inside.mean() > 0.95 and abs(z.mean()) < 0.1 and abs(z.std() - 1) < 0.1
    # the expert's stream at the same counters: the plain rollout of the learner as the policy draws different normals
    E = S.E
    st = th.zeros(L.ST_WORDS, dtype=th.int64, device="cuda")
    o = th.empty(S.Do, E, device="cuda")
    L.env_reset(o, E, S.env, st)
    tbl2, flat2, aux2 = th.zeros(E, S.rw, device="cuda"), th.zeros(E, S.tw, device="cuda"), th.zeros(4 * E, device="cuda")
    hp = L.PpoHparams(gamma=0.99, gae_lambda=0.95, clip_range=0.2, ent_coef=0.0, vf_coef=0.5, max_grad_norm=0.5,
                      lr=0.0, adam_eps=1e-5, n_epochs=1, batch_size=1, normalize_advantage=0)
    L.rollout(S.env, S.envp, o, S.ld, S.LP, S.LN, None, None, None, 0, hp, E, 1, tbl2, None, 0, flat2, aux2, None, st,
              act=S.lact)
    th.cuda.synchronize()
    assert (flat2.cpu().numpy()[:, S.Do:S.Do + S.Da] != u).mean() > 0.9
