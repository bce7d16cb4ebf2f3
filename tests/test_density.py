"""Density-based reward learning: `algorithms.density.DensityAlgorithm` and its kernel `imb_density_score`.

- `tests/golden/density.npz` is recorded from the reference's own `DensityAlgorithm` (fitted with sklearn's
  `KernelDensity`) on the pendulum expert fixture (the first 28 trajectories as demonstrations; queries from the other
  28 and perturbed copies of them) and on CartPole (Discrete actions).  Per case it stores the queries, the reference's
  rewards, the exact float64 log density of the same standardised inputs, and the mask of queries where the two agree
  to 1e-9 relative: sklearn's tree evaluation with atol = rtol = 0 is not exact for low-density queries (and gives
  finite values where a compact kernel's exact value is -inf), while the device computes the exact estimator.
  Re-record it where the reference sources are importable (oracle/refimport.py, oracle/density_ref.py) with

      IMB_RECORD_REFERENCE=1 python -m pytest tests/test_density.py -k reference_records

  Where they are importable, the same test regenerates the results and compares them with the stored file.
- CPU: demonstration forms and segments, errors, scaler and kernel normalisation against the reference / sklearn.
- GPU: the kernel against float64 brute force over kernels, density types, widths, demonstration and query counts;
  the golden; determinism; the fused rollout relabel, GAE and graph replay; the behavioural check of the reference's
  test_density_reward; smoke runs of every demonstration form.

Tolerance: |dev - exact| <= 2e-5 (1 + |exact|), -inf where the exact value is -inf, except for queries with a pair within
1e-5 h of a compact kernel's boundary, where fp32 rounding may flip the d < h test.
"""
import dataclasses
import math
import os

import numpy as np
import pytest

from tests import golden_util as G

STORE = os.path.join(G.GOLDEN, "density.npz")
RECORD = os.environ.get("IMB_RECORD_REFERENCE") == "1"
FIXTURE = os.path.join(G.GOLDEN, "expert_models", "{}_0", "rollouts", "final.npz")
KERNELS = ("gaussian", "tophat", "epanechnikov", "exponential", "linear", "cosine")
COMPACT = ("tophat", "epanechnikov", "linear", "cosine")
TOL = 2e-5
N_IN, N_OFF = 400, 200  # queries per case: held-out transitions, perturbed copies of them


def _cases():
    """name -> (env, density type name, stationary, kernel, bandwidth, standardise)"""
    c = {}
    for t in ("STATE_DENSITY", "STATE_ACTION_DENSITY", "STATE_STATE_DENSITY"):
        c[f"pendulum_{t}"] = ("pendulum", t, True, "gaussian", 0.2, True)
    c["pendulum_STATE_DENSITY_nonstationary"] = ("pendulum", "STATE_DENSITY", False, "gaussian", 0.2, True)
    for k in KERNELS:
        for h in (0.2, 0.5):
            c[f"pendulum_{k}_{h}"] = ("pendulum", "STATE_ACTION_DENSITY", True, k, h, True)
    c["pendulum_unstandardised"] = ("pendulum", "STATE_ACTION_DENSITY", True, "gaussian", 0.5, False)
    c["cartpole_STATE_ACTION_DENSITY"] = ("cartpole", "STATE_ACTION_DENSITY", True, "gaussian", 0.5, True)
    return c


CASES = _cases()


def _trajs(env):
    from imitation_b200.data import serialize

    return list(serialize.load_with_rewards(FIXTURE.format(env)))


def _queries(env):
    """Held-out transitions (N_IN, with their episode steps) and N_OFF perturbed copies: obs, acts, next_obs, steps."""
    trajs = _trajs(env)[28:]
    rng = np.random.default_rng(7)
    obs = np.concatenate([t.obs[:-1] for t in trajs])
    nxt = np.concatenate([t.obs[1:] for t in trajs])
    acts = np.concatenate([t.acts for t in trajs])
    steps = np.concatenate([np.arange(len(t)) for t in trajs])
    i = np.sort(rng.choice(len(obs), N_IN, replace=False))
    j = np.sort(rng.choice(len(obs), N_OFF, replace=False))
    sd = obs.std(0)
    pert = lambda x: (x + rng.normal(0, 0.5, x.shape) * sd).astype(x.dtype)  # noqa: E731
    pa = acts[j] if acts.dtype.kind == "i" else (acts[j] + rng.normal(0, 0.5, acts[j].shape)).astype(acts.dtype)
    return (np.concatenate([obs[i], pert(obs[j])]), np.concatenate([acts[i], pa]), np.concatenate([nxt[i], pert(nxt[j])]),
            np.concatenate([steps[i], steps[j]]))


class _SpacesVenv:
    """The spaces of a fixture env for constructing a DensityAlgorithm (the reference's or this package's); `device`
    is where this package uploads the model."""

    def __init__(self, env, spaces_mod, device="cuda"):
        if env == "pendulum":
            self.observation_space = spaces_mod.Box(-np.inf, np.inf, (3,), np.float32)
            self.action_space = spaces_mod.Box(-2.0, 2.0, (1,), np.float32)
        else:
            self.observation_space = spaces_mod.Box(-np.inf, np.inf, (4,), np.float32)
            self.action_space = spaces_mod.Discrete(2)
        self.num_envs = 1
        self.device = device

    def reset(self, **kwargs):
        return np.zeros((1,) + tuple(self.observation_space.shape), np.float32)


def _log_kernel64(d, h, kernel):
    with np.errstate(divide="ignore", invalid="ignore"):
        if kernel == "gaussian":
            return -0.5 * d * d / (h * h)
        if kernel == "exponential":
            return -d / h
        inside = d < h
        v = {"tophat": np.zeros_like(d), "epanechnikov": np.log(1 - d * d / (h * h)), "linear": np.log(1 - d / h),
             "cosine": np.log(np.cos(0.5 * np.pi * d / h))}[kernel]
        return np.where(inside, v, -np.inf)


def _exact(queries, demo, h, kernel, log_norm, chunk=256):
    """float64 brute force log( (1/N) sum_i K_h(q - x_i) ) + log_norm, and whether each query has a pair within 1e-5 h
    of the kernel's boundary."""
    queries, demo = np.asarray(queries, np.float64), np.asarray(demo, np.float64)
    out = np.empty(len(queries))
    near = np.zeros(len(queries), bool)
    for a in range(0, len(queries), chunk):
        q = queries[a:a + chunk]
        d = np.sqrt(((q[:, None, :] - demo[None, :, :]) ** 2).sum(-1))
        lk = _log_kernel64(d, h, kernel)
        m = lk.max(1)
        with np.errstate(invalid="ignore", divide="ignore"):
            s = np.where(np.isfinite(m), np.log(np.exp(lk - np.where(np.isfinite(m), m, 0)[:, None]).sum(1)) + m, -np.inf)
        out[a:a + chunk] = s - np.log(len(demo)) + log_norm
        near[a:a + chunk] = (np.abs(d - h) <= 1e-5 * h).any(1)
    return out, near


def _check_close(dev, exact, skip=None, what=""):
    dev = np.asarray(dev, np.float64)
    keep = np.ones(len(exact), bool) if skip is None else ~skip
    ninf = np.isneginf(exact) & keep
    nan = np.isnan(exact) & keep
    fin = np.isfinite(exact) & keep
    assert np.array_equal(np.isneginf(dev[ninf]), np.ones(ninf.sum(), bool)), f"{what}: -inf expected"
    assert np.isnan(dev[nan]).all(), f"{what}: NaN expected"
    err = np.abs(dev[fin] - exact[fin]) / (1 + np.abs(exact[fin]))
    assert fin.sum() == 0 or err.max() <= TOL, f"{what}: worst |dev - exact| / (1 + |exact|) = {err.max():.3g}"


# ---------------------------------------------------------------------------------------------------------------------
# golden from the reference
# ---------------------------------------------------------------------------------------------------------------------
def _reference_available():
    try:
        import sklearn  # noqa: F401
        from oracle import refimport

        return refimport.available()
    except ImportError:
        return False


def _record_case(name):
    from imitation.algorithms import density as rd
    from gymnasium import spaces as gspaces
    from sklearn.neighbors import KernelDensity

    env, dtype, stationary, kernel, h, standardise = CASES[name]
    venv = _SpacesVenv(env, gspaces)
    algo = rd.DensityAlgorithm(demonstrations=_ref_demo("trajectories", _trajs(env)[:28]), venv=venv, rng=np.random.default_rng(0),
                               density_type=rd.DensityType[dtype], kernel=kernel, kernel_bandwidth=h,
                               is_stationary=stationary, standardise_inputs=standardise)
    algo.train()
    obs, acts, nxt, steps = _queries(env)
    with np.errstate(all="ignore"):
        ref = algo(obs, acts, nxt, np.zeros(len(obs), bool), steps)
    feats = np.stack([algo._preprocess_transition(o, a, n) for o, a, n in zip(obs, acts, nxt)])
    q = algo._scaler.transform(feats)
    exact, ref64 = np.empty(len(q)), np.empty(len(q))  # ref64: the reference's value before its float32 cast
    D = q.shape[1]
    log_norm = KernelDensity(kernel=kernel, bandwidth=h).fit(np.zeros((1, D))).score_samples(np.zeros((1, D)))[0]
    keys = [None] if stationary else sorted(algo.transitions)
    seg = np.zeros(len(q), int) if stationary else steps
    for s, k in enumerate(keys):
        sel = seg == s
        if sel.any():
            exact[sel] = _exact(q[sel], algo._scaler.transform(algo.transitions[k]), h, kernel, log_norm)[0]
            with np.errstate(all="ignore"):  # one score() per row, as the reference's __call__ makes them
                ref64[sel] = [algo._density_models[k].score(r[None]) for r in q[sel]]
    with np.errstate(invalid="ignore"):
        agree = ((ref64 == exact) | (np.isfinite(exact) & (np.abs(ref64 - exact) <= 1e-9 * np.abs(exact)))
                 | (np.isnan(ref64) & np.isnan(exact)))
    print(f"{name}: reference matches the exact estimator on {agree.sum()} of {len(agree)} queries")
    return {f"{name}/obs": obs, f"{name}/acts": acts, f"{name}/next_obs": nxt, f"{name}/steps": steps,
            f"{name}/reference": ref, f"{name}/exact": exact, f"{name}/mask": agree,
            f"{name}/scaler_mean": algo._scaler.mean_ if standardise else np.zeros(q.shape[1]),
            f"{name}/scaler_scale": algo._scaler.scale_ if standardise else np.ones(q.shape[1])}


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources and sklearn (oracle/refimport.py)")
def test_reference_records_the_golden():
    """Regenerate the stored results from the reference and compare (IMB_RECORD_REFERENCE=1: store them instead)."""
    from oracle import density_ref

    density_ref.load()
    out = {}
    for name in CASES:
        out.update(_record_case(name))
    if RECORD:
        np.savez_compressed(STORE, **out)
    z = np.load(STORE)
    assert sorted(z.files) == sorted(out)
    for k, v in out.items():
        np.testing.assert_array_equal(z[k], v, err_msg=k)


def test_golden_mask_covers_the_in_distribution_gaussian_queries():
    """The reference agrees with the exact estimator on most held-out pendulum queries; the disagreements are the
    low-density ones."""
    z = np.load(STORE)
    for name in ("pendulum_STATE_ACTION_DENSITY", "pendulum_gaussian_0.5"):
        assert z[f"{name}/mask"][:N_IN].mean() > 0.5, name


# ---------------------------------------------------------------------------------------------------------------------
# host semantics (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _ours(env="pendulum", device="cpu", **kw):
    from imitation_b200 import spaces
    from imitation_b200.algorithms import density

    kw.setdefault("rng", np.random.default_rng(0))
    return density.DensityAlgorithm(venv=_SpacesVenv(env, spaces, device), **kw)


def _theirs(env="pendulum", **kw):
    from oracle import density_ref

    density_ref.load()
    from gymnasium import spaces as gspaces
    from imitation.algorithms import density as rd

    if "density_type" in kw:
        kw["density_type"] = rd.DensityType[kw["density_type"].name]
    kw.setdefault("rng", np.random.default_rng(0))
    return rd.DensityAlgorithm(venv=_SpacesVenv(env, gspaces), **kw)


def _demo_forms(env):
    from imitation_b200.data import types

    trajs = _trajs(env)[:3]
    tr = types.flatten_trajectories(trajs)
    return {"trajectories": trajs, "transitions": tr,
            "minimal": types.TransitionsMinimal(obs=tr.obs, acts=tr.acts, infos=tr.infos),
            "mappings": [{k: v for k, v in dataclasses.asdict(tr).items()}],
            "iterator": iter(trajs)}


def _ref_demo(form, demos):
    """The same demonstrations as the reference's types (its Trajectory / Transitions classes)."""
    from oracle import density_ref

    density_ref.load()
    from imitation.data import types as rt

    if form in ("trajectories", "iterator"):
        trajs = [rt.Trajectory(obs=t.obs, acts=t.acts, infos=None, terminal=t.terminal) for t in _trajs_of(demos)]
        return trajs if form == "trajectories" else iter(trajs)
    if form == "transitions":
        return rt.Transitions(obs=demos.obs, acts=demos.acts, infos=demos.infos, next_obs=demos.next_obs,
                              dones=demos.dones)
    if form == "minimal":
        return rt.TransitionsMinimal(obs=demos.obs, acts=demos.acts, infos=demos.infos)
    return demos


def _trajs_of(demos):
    return list(demos)


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources and sklearn")
@pytest.mark.parametrize("env", ["pendulum", "cartpole"])
@pytest.mark.parametrize("dtype", ["STATE_DENSITY", "STATE_ACTION_DENSITY", "STATE_STATE_DENSITY"])
@pytest.mark.parametrize("stationary", [True, False])
@pytest.mark.parametrize("form", ["trajectories", "iterator", "transitions", "minimal", "mappings"])
def test_demonstration_forms_and_segments_match_reference(env, dtype, stationary, form):
    from imitation_b200.algorithms import density

    demos = _demo_forms(env)[form]
    ref_demos = _ref_demo(form, _trajs(env)[:3] if form in ("trajectories", "iterator") else demos)
    kw = dict(density_type=density.DensityType[dtype], is_stationary=stationary)
    outcomes = []
    for make, d in ((_theirs, ref_demos), (_ours, demos)):
        try:
            outcomes.append(make(env, demonstrations=d, **kw).transitions)
        except (ValueError, TypeError) as e:
            outcomes.append((type(e), str(e)))
    ref, got = outcomes
    if isinstance(ref, tuple):
        assert isinstance(got, tuple) and got[0] is ref[0] and got[1] == ref[1]
        return
    assert list(got) == list(ref)
    for k in ref:
        np.testing.assert_allclose(got[k], ref[k], rtol=0, atol=0, err_msg=str(k))


@pytest.mark.skipif(not _reference_available(), reason="needs the reference sources and sklearn")
def test_errors_match_reference():
    """The reference's test_density_trainer_raises, and the non-stationary errors, on both implementations."""
    from imitation_b200.algorithms import density

    for make in (_theirs, _ours):
        algo = make(demonstrations=None, density_type=density.DensityType.STATE_STATE_DENSITY)
        with pytest.raises(ValueError, match="STATE_STATE_DENSITY requires next_obs_b"):
            algo._get_demo_from_batch(np.zeros((1, 3)), np.zeros((1, 1)), None)
        with pytest.raises(TypeError, match="Unsupported demonstration type"):
            algo.set_demonstrations("foo")
        with pytest.raises(TypeError, match="Unsupported demonstration type"):
            algo.set_demonstrations(5)
        with pytest.raises(ValueError, match="Non-stationary model incompatible with non-trajectory demonstrations."):
            tr = _demo_forms("pendulum")["transitions"]
            make(demonstrations=_ref_demo("transitions", tr) if make is _theirs else tr, is_stationary=False)
        ns = make(demonstrations=None, is_stationary=False)
        with pytest.raises(ValueError, match="steps must be provided with non-stationary models"):
            ns(np.zeros((1, 3)), np.zeros((1, 1)), np.zeros((1, 3)), np.zeros(1, bool))


def test_train_refuses_what_the_kernel_does_not_support():
    from imitation_b200 import spaces
    from imitation_b200.algorithms import density

    trajs = _trajs("pendulum")[:2]
    with pytest.raises(ValueError, match="'kernel' parameter"):
        _ours(demonstrations=trajs, kernel="triangle").train()
    for rule in ("scott", "silverman"):
        with pytest.raises(NotImplementedError, match=rule):
            _ours(demonstrations=trajs, kernel_bandwidth=rule).train()
    with pytest.raises(ValueError, match="bandwidth"):
        _ours(demonstrations=trajs, kernel_bandwidth=0.0).train()
    venv = _SpacesVenv("pendulum", spaces, "cpu")
    venv.observation_space = spaces.Box(-np.inf, np.inf, (65,), np.float32)
    wide = density.DensityAlgorithm(demonstrations=None, venv=venv, rng=np.random.default_rng(0),
                                    density_type=density.DensityType.STATE_STATE_DENSITY)
    wide.transitions = {None: np.zeros((4, 130))}
    with pytest.raises(NotImplementedError, match="at most 128 features"):
        wide.train()
    dict_venv = _SpacesVenv("pendulum", spaces, "cpu")
    with pytest.raises(NotImplementedError, match="Dict"):
        density.DensityAlgorithm(demonstrations=[{"obs": {"a": np.zeros((2, 3))}, "acts": np.zeros((2, 1))}],
                                 venv=dict_venv, rng=np.random.default_rng(0))


@pytest.mark.skipif(not _reference_available(), reason="needs sklearn")
def test_scaler_matches_standard_scaler():
    from sklearn.preprocessing import StandardScaler as SkScaler

    from imitation_b200.algorithms import density

    rng = np.random.default_rng(3)
    x = rng.normal(2, 3, (500, 6))
    x[:, 2] = 1.25  # constant column: scale 1
    for standardise in (True, False):
        ours = density.StandardScaler(x, standardise)
        sk = SkScaler(with_mean=standardise, with_std=standardise).fit(x)
        np.testing.assert_allclose(ours.mean_, sk.mean_ if standardise else 0, rtol=1e-14, atol=1e-14)
        np.testing.assert_allclose(ours.scale_, sk.scale_ if standardise else 1, rtol=1e-14)
        np.testing.assert_allclose(ours.transform(x), sk.transform(x), rtol=1e-13, atol=1e-13)


@pytest.mark.skipif(not _reference_available(), reason="needs sklearn")
@pytest.mark.parametrize("kernel", KERNELS)
def test_log_kernel_norm_matches_sklearn(kernel):
    """KernelDensity fitted on one point and scored at that point gives exactly its log normalisation constant."""
    from sklearn.neighbors import KernelDensity

    from imitation_b200.algorithms import density

    for d in range(1, 9):
        for h in (0.2, 0.5, 1.7):
            want = KernelDensity(kernel=kernel, bandwidth=h).fit(np.zeros((1, d))).score_samples(np.zeros((1, d)))[0]
            got = density.log_kernel_norm(h, d, kernel)
            if math.isnan(want):
                assert math.isnan(got), (kernel, d, h)
            else:
                assert got == pytest.approx(want, rel=1e-14, abs=1e-14), (kernel, d, h)
    assert math.isnan(density.log_kernel_norm(0.5, 4, "cosine"))  # sklearn's series: NaN at D = 4


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the kernel against float64 brute force
# ---------------------------------------------------------------------------------------------------------------------
class _WidthVenv:
    def __init__(self, do, da):
        from imitation_b200 import spaces

        self.observation_space = spaces.Box(-np.inf, np.inf, (do,), np.float32)
        self.action_space = spaces.Box(-1.0, 1.0, (da,), np.float32)
        self.num_envs, self.device = 1, "cuda"

    def reset(self, **kwargs):
        return None


def _widths(dtype, D):
    """(d_obs, d_act) giving feature width D for the density type, or None."""
    if dtype == "STATE_DENSITY":
        return (D, 1)
    if dtype == "STATE_ACTION_DENSITY":
        return (D - 1, 1) if D >= 2 else None
    return (D // 2, 1) if D % 2 == 0 else None


def _sweep_case(kernel, dtype, D, seg_sizes, n_query, seed):
    """A model over segments of the given sizes and n_query queries near demonstration rows (plus some far ones);
    -> (device rewards, exact, near-boundary mask)."""
    from imitation_b200.algorithms import density

    do, da = _widths(dtype, D)
    rng = np.random.default_rng(seed)
    h = 0.5 if D <= 6 else 0.3 * math.sqrt(D)
    algo = density.DensityAlgorithm(demonstrations=None, venv=_WidthVenv(do, da), rng=rng,
                                    density_type=density.DensityType[dtype], kernel=kernel, kernel_bandwidth=h,
                                    is_stationary=len(seg_sizes) == 1)
    algo.transitions = {(None if len(seg_sizes) == 1 else s): rng.normal(0, 1, (n, D)) * rng.uniform(0.5, 2, D)
                        for s, n in enumerate(seg_sizes)}
    algo.train()
    steps = rng.integers(0, len(seg_sizes), n_query)
    # queries: a demonstration row of their segment plus noise of about the bandwidth, or (1 in 8) far away
    feats = np.empty((n_query, D))
    for i, s in enumerate(steps):
        seg = algo.transitions[None if len(seg_sizes) == 1 else s]
        feats[i] = seg[rng.integers(len(seg))] + rng.normal(0, 0.3 * h / math.sqrt(D), D) * algo._scaler.scale_
    far = rng.random(n_query) < 0.125
    feats[far] += 5 * algo._scaler.scale_
    c0, n0, c1, n1 = algo._columns()
    obs, acts, nxt = np.zeros((n_query, do)), rng.uniform(-1, 1, (n_query, da)), np.zeros((n_query, do))
    rows = np.zeros((n_query, 2 * do + da + 1))
    rows[:, c0:c0 + n0] = feats[:, :n0]
    rows[:, c1:c1 + n1] = feats[:, n0:]
    obs, acts, nxt = rows[:, :do], rows[:, do:do + da], rows[:, do + da:2 * do + da]
    got = algo(obs.astype(np.float32), acts.astype(np.float32), nxt.astype(np.float32), np.zeros(n_query, bool),
               None if algo.is_stationary else steps)
    q = algo._scaler.transform(algo._features(algo._rows(obs.astype(np.float32), acts.astype(np.float32),
                                                         nxt.astype(np.float32))))
    exact, near = np.empty(n_query), np.zeros(n_query, bool)
    norm = density.log_kernel_norm(h, D, kernel)
    for s in range(len(seg_sizes)):
        sel = (steps == s) if not algo.is_stationary else np.ones(n_query, bool)
        if sel.any():
            demo = algo._scaler.transform(algo.transitions[None if algo.is_stationary else s])
            exact[sel], near[sel] = _exact(q[sel], demo, h, kernel, norm)
    return got, exact, near if kernel in COMPACT else None


SEGMENTS = {"one_short": [37], "one_tile": [64], "tiles_remainder": [64 * 4 + 17],
            "equal": [9] * 20, "unequal": [1, 30, 7, 64, 3, 90, 12, 5]}


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 3, 4, 6, 34, 128])
@pytest.mark.parametrize("kernel", KERNELS)
def test_kernel_matches_float64(kernel, D):
    for dtype in ("STATE_DENSITY", "STATE_ACTION_DENSITY", "STATE_STATE_DENSITY"):
        if _widths(dtype, D) is None:
            continue
        for sname, sizes in SEGMENTS.items():
            for n_query in (1, 150):
                got, exact, near = _sweep_case(kernel, dtype, D, sizes, n_query, seed=D * 100 + n_query)
                _check_close(got, exact, near, f"{kernel} {dtype} D={D} {sname} n_query={n_query}")


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["gaussian", "epanechnikov"])
@pytest.mark.parametrize("sizes", [[2000], [30] * 50])
def test_kernel_more_than_one_wave_of_ctas(kernel, sizes):
    """64 * 300 + 5 queries: more query tiles than CTAs in one wave (no split of the demonstrations)."""
    got, exact, near = _sweep_case(kernel, "STATE_ACTION_DENSITY", 6, sizes, 64 * 300 + 5, seed=11)
    _check_close(got, exact, near, f"{kernel} wave")


@pytest.mark.gpu
@pytest.mark.parametrize("n_query", [5, 64 * 40 + 3])
def test_two_calls_are_bit_identical(n_query):
    from imitation_b200.algorithms import density

    rng = np.random.default_rng(5)
    algo = density.DensityAlgorithm(demonstrations=None, venv=_WidthVenv(17, 6), rng=rng)
    algo.transitions = {None: rng.normal(size=(20000, 23))}
    algo.train()
    obs, acts = rng.normal(size=(n_query, 17)).astype(np.float32), rng.normal(size=(n_query, 6)).astype(np.float32)
    a = algo(obs, acts, obs, np.zeros(n_query, bool))
    b = algo(obs, acts, obs, np.zeros(n_query, bool))
    assert a.dtype == np.float32 and np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: __call__ against the reference's golden
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_call_matches_reference_golden(name):
    from imitation_b200 import spaces
    from imitation_b200.algorithms import density

    env, dtype, stationary, kernel, h, standardise = CASES[name]
    z = np.load(STORE)
    g = {k: z[f"{name}/{k}"] for k in ("obs", "acts", "next_obs", "steps", "reference", "exact", "mask",
                                       "scaler_mean", "scaler_scale")}
    algo = density.DensityAlgorithm(demonstrations=_trajs(env)[:28], venv=_SpacesVenv(env, spaces),
                                    rng=np.random.default_rng(0), density_type=density.DensityType[dtype],
                                    kernel=kernel, kernel_bandwidth=h, is_stationary=stationary,
                                    standardise_inputs=standardise)
    algo.train()
    np.testing.assert_allclose(algo._scaler.mean_, g["scaler_mean"], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(algo._scaler.scale_, g["scaler_scale"], rtol=1e-12)
    got = algo(g["obs"], g["acts"], g["next_obs"], np.zeros(len(g["obs"]), bool), g["steps"])
    assert got.dtype == np.float32
    near = None
    if kernel in COMPACT:  # pairs within 1e-5 h of the boundary, from the float64 standardised inputs
        feats = algo._scaler.transform(algo._features(algo._rows(g["obs"], g["acts"], g["next_obs"])))
        demo = algo._scaler.transform(algo.transitions[None])
        near = _exact(feats, demo, h, kernel, 0.0)[1]
    _check_close(got, g["exact"], near, name)
    m = g["mask"] & (np.zeros(len(got), bool) if near is None else ~near)
    _check_close(got[m], g["reference"][m].astype(np.float64), None, name + " (reference, on the mask)")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the fused rollout relabel
# ---------------------------------------------------------------------------------------------------------------------
def _setup_rollout(stationary, E=8, H=12, T=16, use_buffering=True, seed=0):
    from imitation_b200.algorithms import density, ppo
    from imitation_b200.data import rollout
    from imitation_b200.envs import synth

    venv = synth.DeviceVecEnv(5, 2, E, horizon=H, seed=3)
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=T, batch_size=32, n_epochs=1, seed=seed)
    demos = rollout.generate_trajectories(algo, venv, rollout.make_min_episodes(16), np.random.default_rng(1))
    dens = density.DensityAlgorithm(demonstrations=demos, venv=venv, rng=np.random.default_rng(2), rl_algo=algo,
                                    density_type=density.DensityType.STATE_ACTION_DENSITY, kernel_bandwidth=0.5,
                                    is_stationary=stationary)
    dens.train()
    return venv, algo, dens


def _host_gae(rew, val, last_v, last_done, t0, H, gamma, lam):
    E, T = rew.shape
    adv = np.zeros((E, T))
    last = np.zeros(E)
    next_v, nnt = last_v.astype(np.float64), 1.0 - last_done
    for t in range(T - 1, -1, -1):
        delta = rew[:, t] + gamma * next_v * nnt - val[:, t]
        last = delta + gamma * lam * nnt * last
        adv[:, t] = last
        next_v = val[:, t]
        nnt = 0.0 if (t > 0 and (t0 + t) % H == 0) else 1.0
    return adv, adv + val


@pytest.mark.gpu
@pytest.mark.parametrize("stationary", [True, False])
def test_rollout_reward_column_is_the_density_of_the_popped_transitions(stationary):
    import torch as th

    E, H, T = 8, 12, 16
    venv, algo, dens = _setup_rollout(stationary, E, H, T)
    algo.set_env(dens.venv_wrapped)
    buf = dens.buffering_wrapper
    buf.reset()
    algo.n_steps = 5  # move to episode step 5
    algo.collect_rollouts()
    buf.discard()
    algo.n_steps = T
    t0 = venv.host_ep_step
    assert t0 == 5
    algo.collect_rollouts()
    th.cuda.synchronize()
    rw = algo._tbl.shape[1]
    tbl = algo._tbl.cpu().numpy().reshape(E, T, rw).astype(np.float64)
    aux = algo._aux.cpu().numpy()
    boot = aux[2 * E:2 * E + E * T].reshape(E, T)
    col_val = 5 + 2 + 1
    col_rew = col_val + 1
    trajs, _ = buf.pop_trajectories()
    segs = buf._segments_of(T, t0, H)
    for si, (a, b) in enumerate(segs):
        for e in range(E):
            tr = trajs[si * E + e]
            steps = (t0 + a + np.arange(b - a)) % H
            want = dens(tr.obs[:-1], tr.acts, tr.obs[1:], np.zeros(b - a, bool), steps)
            got = tbl[e, a:b, col_rew] - boot[e, a:b]
            np.testing.assert_allclose(got, want, rtol=1e-5, atol=2e-5 * (1 + np.abs(want).max()))
    adv, ret = _host_gae(tbl[:, :, col_rew], tbl[:, :, col_val], aux[:E], aux[E:2 * E], t0, H, algo.hp.gamma,
                         algo.hp.gae_lambda)
    np.testing.assert_allclose(tbl[:, :, col_rew + 1], adv, rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(tbl[:, :, col_rew + 2], ret, rtol=1e-4, atol=1e-4)


@pytest.mark.gpu
def test_rollout_without_buffering_wrapper_scores_rows_of_its_own():
    import torch as th

    from imitation_b200.rewards import reward_wrapper

    E, H, T = 8, 12, 16
    venv, algo, dens = _setup_rollout(True, E, H, T)
    algo.set_env(reward_wrapper.RewardVecEnvWrapper(venv, dens))
    algo.collect_rollouts()
    th.cuda.synchronize()
    assert algo._scratch.get("flat") is not None and algo._buffering is None
    rw = algo._tbl.shape[1]
    flat = algo._scratch["flat"].cpu().numpy()
    tbl = algo._tbl.cpu().numpy().reshape(E, T, rw)
    boot = algo._aux[2 * E:2 * E + E * T].cpu().numpy().reshape(E, T)
    # from t0 = 0 with T > H: rows of the first episode are env-major [e][0, H), then the partial one [e][H, T)
    for e in range(E):
        for a, b, off in ((0, H, e * H), (H, T, E * H + e * (T - H))):
            r = flat[off:off + b - a]
            want = dens(r[:, :5], r[:, 5:7], r[:, 7:12], np.zeros(b - a, bool))
            np.testing.assert_allclose(tbl[e, a:b, 9] - boot[e, a:b], want, rtol=1e-5, atol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("stationary", [True, False])
def test_graph_replay_equals_eager(stationary):
    import torch as th

    runs = []
    for use_graph in (False, True):
        venv, algo, dens = _setup_rollout(stationary, seed=4)
        algo.use_cuda_graph = use_graph
        dens.train_policy(n_timesteps=3 * 8 * 16)
        th.cuda.synchronize()
        runs.append((algo._tbl.clone(), algo.policy.flat_vectors()[0].clone(), algo))
    assert runs[1][2]._graph is not None
    assert th.equal(runs[0][0], runs[1][0]) and th.equal(runs[0][1], runs[1][1])


@pytest.mark.gpu
def test_non_stationary_model_too_short_raises_before_any_launch():
    from imitation_b200 import _lib
    from imitation_b200.algorithms import density, ppo
    from imitation_b200.data import types
    from imitation_b200.envs import synth

    venv = synth.DeviceVecEnv(5, 2, 4, horizon=12, seed=3)
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=16, batch_size=32, n_epochs=1, seed=0)
    rng = np.random.default_rng(0)
    demos = [types.Trajectory(obs=rng.normal(size=(8, 5)).astype(np.float32),
                              acts=rng.uniform(-1, 1, (7, 2)).astype(np.float32), infos=None, terminal=True)
             for _ in range(3)]
    dens = density.DensityAlgorithm(demonstrations=demos, venv=venv, rng=rng, rl_algo=algo, is_stationary=False)
    dens.train()
    with pytest.raises(ValueError, match=r"Time 7 out of range \(0, 7\], and absorbing states not currently supported"):
        dens(demos[0].obs, np.zeros((8, 2)), demos[0].obs, np.zeros(8, bool), np.arange(8))
    algo.set_env(dens.venv_wrapped)
    before = _lib.LAUNCHES["count"]
    with pytest.raises(ValueError, match=r"Time 7 out of range \(0, 7\]"):
        algo.collect_rollouts()
    assert _lib.LAUNCHES["count"] == before


@pytest.mark.gpu
@pytest.mark.parametrize("stationary", [True, False])
def test_density_reward_prefers_the_demonstrating_policy(stationary):
    """The reference's test_density_reward: held-out rollouts of the policy that gave the demonstrations score
    significantly higher under the learned reward than rollouts of a differently initialised policy."""
    from scipy import stats

    from imitation_b200.algorithms import density, ppo
    from imitation_b200.data import rollout
    from imitation_b200.envs import synth

    venv = synth.DeviceVecEnv(5, 2, 16, horizon=20, seed=3)
    expert = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=20, seed=0)
    other = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=20, seed=1)
    rng = np.random.default_rng(0)
    gen = lambda p: rollout.generate_trajectories(p, venv, rollout.make_min_episodes(32), rng,  # noqa: E731
                                                  deterministic_policy=True)
    demos, held_out, others = gen(expert), gen(expert), gen(other)
    dens = density.DensityAlgorithm(demonstrations=demos, venv=venv, rng=rng, kernel_bandwidth=0.2,
                                    is_stationary=stationary, density_type=density.DensityType.STATE_ACTION_DENSITY)
    dens.train()

    def returns(trajs):
        return [float(np.sum(dens(t.obs[:-1], t.acts, t.obs[1:], np.zeros(len(t), bool), np.arange(len(t)))))
                for t in trajs]

    ret_e, ret_o = returns(held_out), returns(others)
    assert np.mean(ret_e) > np.mean(ret_o)
    assert stats.ttest_ind(ret_e, ret_o, equal_var=False).pvalue < 0.05


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["trajectories", "transitions", "minimal", "mappings"])
def test_train_policy_and_test_policy_run_for_every_demonstration_form(form):
    """The reference's test_density_trainer_smoke and test_density_with_other_trajectory_types on the device env."""
    from imitation_b200.algorithms import density, ppo
    from imitation_b200.data import rollout, types
    from imitation_b200.envs import synth

    venv = synth.DeviceVecEnv(3, 1, 4, horizon=10, seed=3)
    algo = ppo.DevicePPO("FeedForward32Policy", venv, n_steps=10, batch_size=20, n_epochs=2, seed=0)
    trajs = rollout.generate_trajectories(algo, venv, rollout.make_min_episodes(2), np.random.default_rng(0))[:2]
    tr = types.flatten_trajectories(trajs)
    demos = {"trajectories": trajs, "transitions": tr,
             "minimal": types.TransitionsMinimal(obs=tr.obs, acts=tr.acts, infos=tr.infos),
             "mappings": [dataclasses.asdict(tr)]}[form]
    d = density.DensityAlgorithm(demonstrations=demos, venv=venv, rl_algo=algo, rng=np.random.default_rng(0))
    d.train()
    d.train_policy(n_timesteps=2)
    stats_true = d.test_policy(n_trajectories=2)
    stats_learned = d.test_policy(n_trajectories=2, true_reward=False)
    assert stats_true["n_traj"] >= 2 and stats_learned["n_traj"] >= 2
    assert np.isfinite(stats_learned["return_mean"]) and stats_learned["return_mean"] != stats_true["return_mean"]
    assert d.policy is algo.policy
