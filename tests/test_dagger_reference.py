"""DAgger's host bookkeeping (reference algorithms/dagger.py), pinned to the reference on the CPU.

tests/golden/dagger.npz holds what the reference's own `SimpleDAggerTrainer` and `InteractiveTrajectoryCollector` do
over `oracle.synth_env.SynthVecEnv` (E = 12 envs, horizon 4, Box actions) with a deterministic expert, two
`expert_trajs`, `ExponentialBetaSchedule(0.6)` and three rounds of two collection batches each (min_episodes 13).  The
BC trainer is a stub: its learner acts with a constant action, and its `train` iterates the reference's DataLoader
under `th.manual_seed(100 + round)`.  Per round r:
    beta/r          the collector's beta;
    mask/r          uint8 [steps][E]: where the learner's action was executed (`uniform > beta` at each step);
    written/r       the file names in the order they were written;
    listing/r       the files `_load_all_demos` read for the round, in its order;
    n_rows/r        the rows of the flattened dataset handed to BC;
    perm/r          int64 [n_epochs][N // batch_size * batch_size]: the rows of the loader's batches, in order;
    rng_after/r     four draws of a copy of the trainer's generator after the round (its state);
    log/r/keys, log/r/values   the logger calls of the round, in order (record / record_mean);
and `initial/written` (the `expert_trajs` file names), `errors/*` (the reference's error messages).  Re-record it where
the reference sources are importable (oracle/refimport.py) with

    IMB_RECORD_REFERENCE=1 python -m pytest tests/test_dagger_reference.py -k reference_records

Where they are importable, the same test regenerates the results and compares them with the stored file.  The device
collector and trainer are held to the same file on the GPU in tests/test_dagger.py.
"""
import copy
import os
import tempfile

import numpy as np
import pytest
import torch as th

from imitation_b200.algorithms import dagger
from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "dagger.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
# the recorded configuration (tests/test_dagger.py runs the device trainer at the same one)
D_OBS, D_ACT, E, H, SEED, ENV_SEED = 3, 2, 12, 4, 17, 7
DECAY, ROUNDS, MIN_EPISODES, MIN_TIMESTEPS, BATCH, EPOCHS, N_INITIAL = 0.6, 3, 13, 10, 8, 2, 2


def _fingerprint(rng):
    return copy.deepcopy(rng).integers(0, 1 << 62, 4)


def _reference_available() -> bool:
    from oracle import refimport

    return refimport.available()


# ------------------------------------------------------------------------------------------------
# the recorder (reference sources needed)
# ------------------------------------------------------------------------------------------------
class _RecRng:
    """The trainer's generator, recording every `uniform` draw."""

    def __init__(self, gen):
        self.gen, self.uniforms = gen, []

    def uniform(self, *a, **k):
        v = self.gen.uniform(*a, **k)
        self.uniforms.append(v)
        return v

    def __getattr__(self, name):
        return getattr(self.gen, name)


class _Log:
    def __init__(self):
        self.calls = []

    def record(self, key, val, exclude=None):
        self.calls.append((f"record:{key}", float(val)))

    def record_mean(self, key, val, exclude=None):
        self.calls.append((f"record_mean:{key}", float(val)))

    def dump(self, step=0):
        pass


def _record_all():
    from imitation_b200.data import serialize as our_serialize
    from imitation_b200.data import types as our_types
    from oracle import bc_ref, synth_env

    bc_ref.load()
    import gymnasium.spaces as shim_spaces
    from imitation.algorithms import dagger as ref_dagger
    from imitation.data import serialize as ref_serialize
    from imitation.data import types as ref_types

    spec = synth_env.SynthEnvSpec(D_OBS, D_ACT, horizon=H, seed=ENV_SEED)
    venv = synth_env.SynthVecEnv(spec, E, spaces_mod=shim_spaces)
    W = np.random.default_rng(0).normal(size=(D_OBS, D_ACT)).astype(np.float32)

    from stable_baselines3.common import policies as sb3_policies

    class Expert(sb3_policies.BasePolicy):
        """Deterministic: a clipped linear map of the observation."""
        observation_space, action_space = venv.observation_space, venv.action_space

        def predict(self, obs, state=None, episode_start=None, deterministic=False):
            return np.clip(np.asarray(obs) @ W, -1, 1), None

    out, written, state = {}, [], {"round": 0, "log": None}

    class Policy:
        def predict(self, obs, state=None, episode_start=None, deterministic=False):
            return np.full((len(obs), D_ACT), 0.25, np.float32), None

    class StubBC:
        observation_space, action_space, batch_size, policy = venv.observation_space, venv.action_space, BATCH, Policy()
        logger = None

        def set_demonstrations(self, loader):
            self.loader = loader

        def train(self, n_epochs, log_rollouts_venv=None, **kw):
            r = state["round"]
            obs = np.asarray(self.loader.dataset.obs, np.float64)
            where = {row.tobytes(): i for i, row in enumerate(obs)}
            assert len(where) == len(obs)
            th.manual_seed(100 + r)
            perms = []
            for _ in range(n_epochs):
                perms.append([where[row.tobytes()] for b in self.loader for row in np.asarray(b["obs"], np.float64)])
            out[f"perm/{r}"] = np.array(perms, np.int64)
            out[f"n_rows/{r}"] = np.int64(len(obs))

    def save(path, trajs):  # the legacy .npz layout, which the reference's load reads
        written.append(os.path.basename(os.fspath(path)))
        our_serialize.save(path, [our_types.TrajectoryWithRew(obs=t.obs, acts=t.acts, infos=None, terminal=t.terminal,
                                                              rews=t.rews) for t in trajs])

    orig_save, orig_load_demos = ref_serialize.save, ref_dagger.DAggerTrainer._load_all_demos
    listed = []

    def load_all(self):
        listed.clear()
        for rn in range(self._last_loaded_round + 1, self.round_num + 1):
            listed.extend(p.name for p in self._get_demo_paths(self._demo_dir_path_for_round(rn)))
        return orig_load_demos(self)

    ref_serialize.save = save
    ref_dagger.DAggerTrainer._load_all_demos = load_all
    try:
        with tempfile.TemporaryDirectory() as tmp:
            # the expert's own trajectories, from a separate env and generator
            from imitation.data import rollout as ref_rollout

            pre_env = synth_env.SynthVecEnv(spec, E, env_id_offset=100, spaces_mod=shim_spaces)
            initial = ref_rollout.generate_trajectories(Expert(), pre_env, ref_rollout.make_sample_until(min_episodes=1),
                                                        rng=np.random.default_rng(1), deterministic_policy=True)
            initial = initial[:N_INITIAL]
            out["initial/obs"] = np.stack([t.obs for t in initial])
            out["initial/acts"] = np.stack([t.acts for t in initial])
            rng = _RecRng(np.random.default_rng(SEED))
            log = _Log()
            tr = ref_dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp, expert_policy=Expert(), rng=rng,
                                                expert_trajs=initial, bc_trainer=StubBC(), custom_logger=log,
                                                beta_schedule=ref_dagger.ExponentialBetaSchedule(DECAY))
            out["initial/written"] = np.array(written)
            orig_create = tr.create_trajectory_collector

            def create():
                c = orig_create()
                r = state["round"]
                out[f"beta/{r}"] = np.float64(c.beta)
                written.clear()
                rng.uniforms.clear()
                log.calls.clear()
                return c

            tr.create_trajectory_collector = create
            orig_extend = tr.extend_and_update

            def extend(kw=None):
                r = state["round"]
                out[f"mask/{r}"] = (np.stack(rng.uniforms) > out[f"beta/{r}"]).astype(np.uint8)
                out[f"written/{r}"] = np.array(written)
                out[f"log/{r}/keys"] = np.array([k for k, _ in log.calls])
                out[f"log/{r}/values"] = np.array([v for _, v in log.calls])
                res = orig_extend(kw)
                out[f"listing/{r}"] = np.array(listed)
                out[f"rng_after/{r}"] = _fingerprint(rng.gen)
                state["round"] += 1
                return res

            tr.extend_and_update = extend
            tr.train(ROUNDS * 2 * E * H, rollout_round_min_episodes=MIN_EPISODES,
                     rollout_round_min_timesteps=MIN_TIMESTEPS, bc_train_kwargs=dict(n_epochs=EPOCHS))
            assert state["round"] == ROUNDS
        # the reference's errors
        with tempfile.TemporaryDirectory() as tmp:
            tr = ref_dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp, expert_policy=Expert(),
                                                rng=np.random.default_rng(0), bc_trainer=StubBC(), custom_logger=_Log())
            with pytest.raises(ref_dagger.NeedsDemosException) as e:
                tr.extend_and_update()
            out["errors/needs_demos"] = np.array(str(e.value).replace(tmp, "<scratch>"))
            stub = StubBC()
            stub.batch_size = 10 * H
            tr = ref_dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp, expert_policy=Expert(),
                                                rng=np.random.default_rng(0), bc_trainer=stub, custom_logger=_Log(),
                                                expert_trajs=initial[:1])
            with pytest.raises(ValueError) as e:
                tr.extend_and_update()
            out["errors/few_transitions"] = np.array(str(e.value))

            class Other(Expert):
                observation_space = shim_spaces.Box(-np.inf, np.inf, (D_OBS + 1,), np.float32)

            with pytest.raises(ValueError) as e:
                ref_dagger.SimpleDAggerTrainer(venv=venv, scratch_dir=tmp, expert_policy=Other(),
                                               rng=np.random.default_rng(0), bc_trainer=StubBC(), custom_logger=_Log())
            out["errors/obs_space"] = np.array(str(e.value))
            with pytest.raises(ValueError) as e:
                ref_dagger.ExponentialBetaSchedule(0.0)
            out["errors/decay"] = np.array(str(e.value))
        # the reference's load reads the files this package writes
        with tempfile.TemporaryDirectory() as tmp:
            p = os.path.join(tmp, "t.npz")
            t0 = our_types.TrajectoryWithRew(obs=out["initial/obs"][0], acts=out["initial/acts"][0], infos=None,
                                             terminal=True, rews=np.arange(H, dtype=np.float32))
            our_serialize.save(p, [t0])
            back = ref_serialize.load(p)[0]
            assert isinstance(back, ref_types.TrajectoryWithRew)
            np.testing.assert_array_equal(back.obs, t0.obs)
            np.testing.assert_array_equal(back.acts, t0.acts)
            np.testing.assert_array_equal(back.rews, t0.rews)
    finally:
        ref_serialize.save = orig_save
        ref_dagger.DAggerTrainer._load_all_demos = orig_load_demos
    return out


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources (oracle/refimport.py)")
def test_golden_is_what_the_reference_records():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead)."""
    out = _record_all()
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = G.load("dagger")
    assert set(z.files) == set(out)
    for k, v in out.items():
        np.testing.assert_array_equal(v, z[k], err_msg=k)


# ------------------------------------------------------------------------------------------------
# this package against the stored file
# ------------------------------------------------------------------------------------------------
def replay_host_draws(z):
    """The draws `SimpleDAggerTrainer.train` makes from its generator, restated with this package's helpers in the
    order the device collector makes them (the initial files; per round and batch, the mask of H steps before the
    launch and E file names after it; then the shuffle), for the recorded configuration."""
    rng = np.random.default_rng(SEED)
    out = {"initial/written": [dagger.demo_file_name(i, rng, "initial_data") for i in range(N_INITIAL)]}
    for r in range(ROUNDS):
        beta = dagger.ExponentialBetaSchedule(DECAY)(r)
        masks, names, n_traj = [], [], 0
        while not (n_traj >= MIN_EPISODES and n_traj * H >= max(MIN_TIMESTEPS, BATCH)):
            masks.append(dagger.draw_robot_mask(rng, H, E, beta))
            names += [dagger.demo_file_name(e, rng) for e in range(E)]
            n_traj += E
        rng.shuffle(list(range(n_traj)))
        out[f"beta/{r}"], out[f"mask/{r}"], out[f"written/{r}"] = beta, np.concatenate(masks), names
        out[f"rng_after/{r}"] = _fingerprint(rng)
    return out


def test_host_draws_match_reference_golden():
    z = G.load("dagger")
    got = replay_host_draws(z)
    for k, v in got.items():
        np.testing.assert_array_equal(np.asarray(v), z[k], err_msg=k)
    listing = sorted(z["initial/written"].tolist())
    for r in range(ROUNDS):
        # the round's files in sorted order (round 0: with the initial ones), E >= 11: "-10-" before "-2-"
        want = sorted(z[f"written/{r}"].tolist() + (listing if r == 0 else []))
        assert z[f"listing/{r}"].tolist() == want
        assert int(z[f"n_rows/{r}"]) == H * (sum(len(z[f"written/{q}"]) for q in range(r + 1)) + N_INITIAL)
        names = z[f"written/{r}"].tolist()
        assert want.index(next(n for n in names if "-demo-10-" in n)) < want.index(next(n for n in names
                                                                                       if "-demo-2-" in n))


def test_dataset_shuffle_matches_reference_golden():
    """BC's per-epoch order over DAgger's aggregate is the reference DataLoader's (same global-RNG draws)."""
    from imitation_b200.algorithms import bc

    z = G.load("dagger")
    for r in range(ROUNDS):
        n, want = int(z[f"n_rows/{r}"]), z[f"perm/{r}"]
        th.manual_seed(100 + r)
        got = [bc.epoch_permutation(n, BATCH)[:n // BATCH * BATCH].numpy() for _ in range(EPOCHS)]
        np.testing.assert_array_equal(np.array(got), want)


def test_log_records_and_errors_match_reference_golden():
    z = G.load("dagger")
    for r in range(ROUNDS):
        keys = z[f"log/{r}/keys"].tolist()
        vals = dict(zip(keys, z[f"log/{r}/values"]))
        n_traj = len(z[f"written/{r}"])
        assert keys.count("record_mean:dagger/mean_episode_reward") == n_traj
        assert keys[n_traj:] == ["record:dagger/total_timesteps", "record:dagger/round_num",
                                 "record:dagger/round_episode_count", "record:dagger/round_timestep_count"]
        assert vals["record:dagger/round_num"] == r and vals["record:dagger/round_episode_count"] == n_traj
        assert vals["record:dagger/round_timestep_count"] == n_traj * H
    with pytest.raises(ValueError) as e:
        dagger.ExponentialBetaSchedule(0.0)
    assert str(e.value) == str(z["errors/decay"])
