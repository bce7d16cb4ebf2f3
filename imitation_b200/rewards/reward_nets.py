"""Reward networks: the reference's `imitation.rewards.reward_nets` API over sm_90a kernels.

Same class names, constructor arguments, method names, state_dict keys and error behaviour as
/root/reference/src/imitation/rewards/reward_nets.py (RewardNet :16-224, wrappers :227-380,
BasicRewardNet :383-457, NormalizedRewardNet :613-671, ShapedRewardNet :674-736,
BasicShapedRewardNet :739-809, BasicPotentialMLP :812-839, RewardEnsemble :884-1016,
AddSTDRewardWrapper :1019-1080) for Box / Discrete spaces.  CNN variants are out of scope
(SURVEY.md section 2 row 3).

The modules are ordinary `nn.Module`s (picklable with `th.save`, parameters visible to any
`torch.optim`), but their Linear weights and RunningNorm buffers ALIAS flat device vectors that
the fused kernels (csrc/imb_disc.cu) read and write: `forward` is a custom autograd Function
around `imb_reward_forward` / `imb_disc_fwd_bwd`, and the trainers drive the same vectors
through the fully fused update.  There is no CPU path: calling a network that lives on the CPU
raises.
"""
import abc
import collections
import functools
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple, Type

import numpy as np
import torch as th
from torch import nn

from .. import _desc, _lib, spaces
from ..util import networks
from ..util.flat import FlatAlias, views


# ------------------------------------------------------------------------------------------------
# flat-vector aliasing + kernel driver shared by BasicRewardNet / BasicShapedRewardNet / potential
# ------------------------------------------------------------------------------------------------
class FusedEngine:
    """Owns the flat parameter / norm vectors of one fused discriminator and launches kernels."""

    def __init__(self, desc: _lib.DiscDesc, mlps: Sequence[nn.Sequential]):
        self.desc = desc
        self.mlps = list(mlps)  # [base mlp, (potential mlp)]
        linears = [mod for m in self.mlps for mod in m if isinstance(mod, nn.Linear)]
        self.norms = [m.normalize_input for m in self.mlps if hasattr(m, "normalize_input")]
        self._params = FlatAlias([(lin, k) for lin in linears for k in ("weight", "bias")])
        self._norm_state = self._norm_count = None
        if self.norms:
            self._norm_state = FlatAlias([(n, k) for n in self.norms for k in ("running_mean", "running_var")])
            self._norm_count = FlatAlias([(n, "count") for n in self.norms])
        self.params: Optional[th.Tensor] = None
        self.norm_state: Optional[th.Tensor] = None
        self.norm_count: Optional[th.Tensor] = None
        self.ws: Optional[th.Tensor] = None
        self.bw = _desc.batch_rows(desc.d_obs, desc.d_act)
        self.check_plan()

    def check_plan(self) -> None:
        """Raise NotImplementedError now, rather than at the first discriminator update, when the fused kernels cannot
        run this network shape (imb_disc_plan: the kernel's shared-memory need exceeds what one CTA can have)."""
        try:
            _lib.disc_plan(self.desc, _lib.IMB_TILE_ROWS)
        except _lib.ImbError as e:
            raise NotImplementedError(f"reward network shape not supported by the fused sm_90a kernels: {e}") from None

    # -- aliasing ---------------------------------------------------------------------------------
    def _param_list(self) -> List[nn.Parameter]:
        return self._params.tensors()

    def device(self) -> th.device:
        return self._param_list()[0].device

    def sync(self) -> None:
        """(Re)establish that every parameter/buffer is a view of one flat vector.  Cheap when
        nothing moved; after `.to(device)` it re-flattens.  A sub-network (e.g. the base of a
        shaped net) accepts the enclosing net's flat vector because its slice is contiguous."""
        dev = self.device()
        if dev.type != "cuda":
            raise _lib.ImbError("imitation_b200 reward nets run on CUDA only (no CPU fallback): call .to('cuda')")
        self.params = self._params.get(th.float32, dev)
        assert self.params.numel() == self.desc.n_params, (self.params.numel(), self.desc.n_params)
        if self._norm_state is not None:
            self.norm_state = self._norm_state.get(th.float32, dev)
            self.norm_count = self._norm_count.get(th.int32, dev)
        elif self.norm_state is None or self.norm_state.device != dev:
            self.norm_state = th.zeros(2, device=dev)
            self.norm_count = th.zeros(2, dtype=th.int32, device=dev)
        if self.ws is None or self.ws.device != dev:
            self.ws = th.zeros(_lib.disc_workspace_floats(self.desc), device=dev)

    @property
    def has_norm(self) -> bool:
        return bool(self.desc.base.has_norm or (self.desc.shaped and self.desc.potential.has_norm))

    # -- batches -----------------------------------------------------------------------------------
    def new_batch(self, n: int) -> Tuple[th.Tensor, int]:
        ld = _desc.batch_ld(n)
        return th.zeros(self.bw, ld, device=self.device()), ld

    def pack(self, state: th.Tensor, action: th.Tensor, next_state: th.Tensor, done: th.Tensor,
             logp: Optional[th.Tensor] = None) -> Tuple[th.Tensor, int, int]:
        """Preprocessed [N, ...] tensors -> feature-major batch (API path; a few torch copies)."""
        n = state.shape[0]
        Do, Da = self.desc.d_obs, self.desc.d_act
        batch, ld = self.new_batch(n)
        batch[:Do, :n] = state.reshape(n, -1).float().t()
        if Da:
            batch[Do:Do + Da, :n] = action.reshape(n, -1).float().t()
        batch[Do + Da:2 * Do + Da, :n] = next_state.reshape(n, -1).float().t()
        batch[2 * Do + Da, :n] = done.reshape(n).float()
        if logp is not None:
            batch[2 * Do + Da + 1, :n] = logp.reshape(n).float()
        return batch, ld, n

    # -- kernels ------------------------------------------------------------------------------------
    def forward_out(self, batch: th.Tensor, ld: int, n: int, out_mode: int) -> th.Tensor:
        out = th.empty(n, device=batch.device)
        _lib.reward_forward(self.desc, self.params, self.norm_state, batch, ld, n, out_mode, out)
        return out

    def norm_update(self, batch: th.Tensor, ld: int, n: int) -> None:
        if self.has_norm:
            _lib.disc_norm_update(self.desc, batch, ld, n, self.norm_state, self.norm_count, self.ws)

    def fwd_bwd(self, batch, ld, n, n_expert, loss_scale, grad_out, logits_out, zero_grad: bool, train_norm: bool):
        flags = (_lib.IMB_F_ZERO_GRAD if zero_grad else 0) | (_lib.IMB_F_TRAIN_NORM if train_norm else 0)
        _lib.disc_fwd_bwd(self.desc, self.params, self.norm_state, batch, ld, n, n_expert, loss_scale, grad_out,
                          logits_out, flags, self.ws)

    def reduce(self, grad_out_flat: Optional[th.Tensor] = None) -> None:
        _lib.disc_reduce(self.desc, self.ws, grad_out_flat)


class _FusedForward(th.autograd.Function):
    """logits = net(batch); backward = imb_disc_fwd_bwd(grad_out) -> per-parameter gradients."""

    @staticmethod
    def forward(ctx, engine: FusedEngine, batch, ld, n, train_norm, *params):
        ctx.engine, ctx.batch, ctx.ld, ctx.n, ctx.train_norm = engine, batch, ld, n, train_norm
        ctx.shapes = [p.shape for p in params]
        return engine.forward_out(batch, ld, n, 0) if not train_norm else _FusedForward._fwd_train(engine, batch, ld, n)

    @staticmethod
    def _fwd_train(engine, batch, ld, n):
        # training-mode forward of a shaped net must use the mid-update snapshot for Phi(s'):
        # run the fused kernel with a zero upstream gradient just to read the logits.
        logits = th.empty(n, device=batch.device)
        zero = th.zeros(n, device=batch.device)
        engine.fwd_bwd(batch, ld, n, n, 0.0, zero, logits, True, True)
        return logits

    @staticmethod
    def backward(ctx, grad_out):
        e = ctx.engine
        flat = th.empty(e.desc.n_params, device=grad_out.device)
        e.fwd_bwd(ctx.batch, ctx.ld, ctx.n, ctx.n, 0.0, grad_out.contiguous().float(), None, True, ctx.train_norm)
        e.reduce(flat)
        return (None, None, None, None, None, *views(flat, ctx.shapes))


# ------------------------------------------------------------------------------------------------
# RewardNet ABC and wrappers (API identical to the reference)
# ------------------------------------------------------------------------------------------------
def _preprocess_space(x: th.Tensor, space) -> th.Tensor:
    """SB3 preprocess_obs for non-image spaces: Box -> float, Discrete -> one-hot float."""
    if spaces.is_discrete(space):
        return nn.functional.one_hot(x.long(), num_classes=int(space.n)).float()
    return x.float()


def _to_tensor(a, device) -> th.Tensor:
    if isinstance(a, np.ndarray) and not a.flags.writeable:
        a = a.copy()
    return th.as_tensor(a).to(device)


class RewardNet(nn.Module, abc.ABC):
    def __init__(self, observation_space, action_space, normalize_images: bool = True):
        super().__init__()
        self.observation_space = observation_space
        self.action_space = action_space
        self.normalize_images = normalize_images

    @abc.abstractmethod
    def forward(self, state: th.Tensor, action: th.Tensor, next_state: th.Tensor, done: th.Tensor) -> th.Tensor:
        """Compute rewards for a batch of (preprocessed) transitions and keep gradients."""

    def preprocess(self, state: np.ndarray, action: np.ndarray, next_state: np.ndarray, done: np.ndarray
                   ) -> Tuple[th.Tensor, th.Tensor, th.Tensor, th.Tensor]:
        dev = self.device
        state_th = _preprocess_space(_to_tensor(state, dev), self.observation_space)
        action_th = _preprocess_space(_to_tensor(action, dev), self.action_space)
        next_state_th = _preprocess_space(_to_tensor(next_state, dev), self.observation_space)
        done_th = _to_tensor(done, dev).to(th.float32)
        assert state_th.shape == next_state_th.shape
        assert len(action_th) == len(state_th)
        return state_th, action_th, next_state_th, done_th

    def predict_th(self, state, action, next_state, done) -> th.Tensor:
        with networks.evaluating(self):
            s, a, ns, d = self.preprocess(state, action, next_state, done)
            with th.no_grad():
                rew_th = self(s, a, ns, d)
            assert rew_th.shape == state.shape[:1]
            return rew_th

    def predict(self, state, action, next_state, done) -> np.ndarray:
        return self.predict_th(state, action, next_state, done).detach().cpu().numpy().flatten()

    def predict_processed(self, state, action, next_state, done, **kwargs) -> np.ndarray:
        del kwargs
        return self.predict(state, action, next_state, done)

    @property
    def device(self) -> th.device:
        try:
            return next(self.parameters()).device
        except StopIteration:
            return th.device("cpu")

    @property
    def dtype(self) -> th.dtype:
        try:
            return next(self.parameters()).dtype
        except StopIteration:
            return th.get_default_dtype()


class RewardNetWrapper(RewardNet):
    def __init__(self, base: RewardNet):
        super().__init__(base.observation_space, base.action_space, base.normalize_images)
        self._base = base

    @property
    def base(self) -> RewardNet:
        return self._base

    @property
    def device(self) -> th.device:
        return self.base.device

    @property
    def dtype(self) -> th.dtype:
        return self.base.dtype

    def preprocess(self, state, action, next_state, done):
        return self.base.preprocess(state, action, next_state, done)


class ForwardWrapper(RewardNetWrapper):
    def __init__(self, base: RewardNet):
        super().__init__(base)
        if isinstance(base, PredictProcessedWrapper):
            raise ValueError("ForwardWrapper cannot be applied on top of PredictProcessedWrapper!")


class PredictProcessedWrapper(RewardNetWrapper):
    def forward(self, state, action, next_state, done) -> th.Tensor:
        return self.base.forward(state, action, next_state, done)

    @abc.abstractmethod
    def predict_processed(self, state, action, next_state, done, **kwargs) -> np.ndarray:
        """Predict processed rewards."""

    def predict(self, state, action, next_state, done) -> np.ndarray:
        return self.base.predict(state, action, next_state, done)

    def predict_th(self, state, action, next_state, done) -> th.Tensor:
        return self.base.predict_th(state, action, next_state, done)


class RewardNetWithVariance(RewardNet):
    @abc.abstractmethod
    def predict_reward_moments(self, state, action, next_state, done, **kwargs) -> Tuple[np.ndarray, np.ndarray]:
        """Mean and variance of the reward distribution."""


# ------------------------------------------------------------------------------------------------
# concrete MLP networks
# ------------------------------------------------------------------------------------------------
def _is_running_norm(cls) -> bool:
    return cls is not None and getattr(cls, "__name__", "") == "RunningNorm"


def build_mlp(in_size: int, hid_sizes: Iterable[int], out_size: int = 1, name: Optional[str] = None,
              activation: Type[nn.Module] = nn.ReLU, dropout_prob: float = 0.0, squeeze_output: bool = False,
              flatten_input: bool = False, normalize_input_layer: Optional[Type[nn.Module]] = None) -> nn.Sequential:
    """util/networks.py:204-283, restricted to what the fused kernels implement (ReLU, no dropout,
    RunningNorm input layer).  Same layer names => same state_dict keys as the reference."""
    if activation is not nn.ReLU:
        raise NotImplementedError("fused reward nets implement ReLU activations only")
    if dropout_prob > 0.0:
        raise NotImplementedError("fused reward nets do not implement dropout (not used by any reference config)")
    if normalize_input_layer is not None and not _is_running_norm(normalize_input_layer):
        raise NotImplementedError("normalize_input_layer must be RunningNorm or None (EMANorm/BatchNorm out of scope)")
    if name is not None:
        raise NotImplementedError("layer name prefixes are not supported")
    layers: Dict[str, nn.Module] = collections.OrderedDict()
    if flatten_input:
        layers["flatten"] = nn.Flatten()
    if normalize_input_layer is not None:
        layers["normalize_input"] = networks.RunningNorm(in_size)
    prev = in_size
    for i, size in enumerate(hid_sizes):
        layers[f"dense{i}"] = nn.Linear(prev, size)
        prev = size
        layers[f"act{i}"] = nn.ReLU()
    layers["dense_final"] = nn.Linear(prev, out_size)
    if squeeze_output:
        if out_size != 1:
            raise ValueError("squeeze_output is only applicable when out_size=1")
        layers["squeeze"] = networks.SqueezeLayer()
    return nn.Sequential(layers)


class _FusedNetMixin:
    """forward() through the kernels, for nets that own a FusedEngine in `self._engine`."""

    _engine: FusedEngine

    def __getstate__(self):  # th.save(module): drop device scratch, keep parameters/buffers
        state = self.__dict__.copy()
        state.pop("_engine", None)
        return state

    def __setstate__(self, state):
        self.__dict__.update(state)
        self._engine = self._make_engine()

    def engine(self) -> FusedEngine:
        self._engine.sync()
        return self._engine

    def _fused_forward(self, state, action, next_state, done) -> th.Tensor:
        e = self.engine()
        batch, ld, n = e.pack(state, action, next_state, done)
        return self.forward_batch(batch, ld, n)

    def forward_batch(self, batch: th.Tensor, ld: int, n: int) -> th.Tensor:
        """forward() on an already feature-major device batch (rows gathered from a device table: the preference
        comparisons' fragment pool, imb_gather_rows); differentiable like forward()."""
        e = self.engine()
        if n == 0:
            return th.zeros(0, device=batch.device)
        train_norm = bool(self.training and e.has_norm)
        if train_norm:
            e.norm_update(batch, ld, n)
        needs_grad = th.is_grad_enabled() and any(p.requires_grad for p in e._param_list())
        if not needs_grad:
            if train_norm and e.desc.shaped:
                return _FusedForward._fwd_train(e, batch, ld, n)
            return e.forward_out(batch, ld, n, 0)
        return _FusedForward.apply(e, batch, ld, n, train_norm and bool(e.desc.shaped), *e._param_list())


class BasicRewardNet(_FusedNetMixin, RewardNet):
    """MLP on the concatenation of the selected (state, action, next_state, done) inputs."""

    def __init__(self, observation_space, action_space, use_state: bool = True, use_action: bool = True,
                 use_next_state: bool = False, use_done: bool = False, **kwargs):
        super().__init__(observation_space, action_space)
        self.use_state, self.use_action = use_state, use_action
        self.use_next_state, self.use_done = use_next_state, use_done
        self._d_obs, self._d_act = spaces.flat_dim(observation_space), spaces.flat_dim(action_space)
        combined = (self._d_obs * use_state + self._d_act * use_action + self._d_obs * use_next_state + int(use_done))
        full = {"hid_sizes": (32, 32), **kwargs, "in_size": combined, "out_size": 1, "squeeze_output": True}
        self._hid_sizes = tuple(full["hid_sizes"])
        self._norm = full.get("normalize_input_layer") is not None
        self.mlp = build_mlp(**full)
        self._engine = self._make_engine()

    def _make_engine(self) -> FusedEngine:
        d = _desc.disc_desc(self._d_obs, self._d_act, hid_sizes=self._hid_sizes, use_state=self.use_state,
                            use_action=self.use_action, use_next_state=self.use_next_state, use_done=self.use_done,
                            normalize_input=self._norm)
        return FusedEngine(d, [self.mlp])

    def forward(self, state, action, next_state, done):
        out = self._fused_forward(state, action, next_state, done)
        assert out.shape == state.shape[:1]
        return out


class BasicPotentialMLP(nn.Module):
    """Potential Phi(s): MLP on the flattened observation (reward_nets.py:812-839)."""

    def __init__(self, observation_space, hid_sizes: Iterable[int], **kwargs):
        super().__init__()
        self._d_obs = spaces.flat_dim(observation_space)
        self._hid_sizes = tuple(hid_sizes)
        self._norm = kwargs.get("normalize_input_layer") is not None
        self._potential_net = build_mlp(in_size=self._d_obs, hid_sizes=self._hid_sizes, squeeze_output=True,
                                        flatten_input=True, **kwargs)
        self._engine = self._make_engine()

    def _make_engine(self) -> FusedEngine:
        d = _desc.disc_desc(self._d_obs, 0, hid_sizes=self._hid_sizes, use_state=True, use_action=False,
                            normalize_input=self._norm)
        return FusedEngine(d, [self._potential_net])

    __getstate__ = _FusedNetMixin.__getstate__
    __setstate__ = _FusedNetMixin.__setstate__
    engine = _FusedNetMixin.engine
    _fused_forward = _FusedNetMixin._fused_forward

    def forward(self, state: th.Tensor) -> th.Tensor:
        n = state.shape[0]
        z = th.zeros(n, device=state.device)
        return self._fused_forward(state, th.zeros(n, 0, device=state.device), state, z)


class ShapedRewardNet(ForwardWrapper):
    """base(s,a,s',d) + gamma * (1 - done) * potential(s') - potential(s)  (reward_nets.py:674-736);
    generic composition (any base / potential); see BasicShapedRewardNet for the fused form."""

    def __init__(self, base: RewardNet, potential: Callable[[th.Tensor], th.Tensor], discount_factor: float):
        super().__init__(base=base)
        self.potential = potential
        self.discount_factor = discount_factor

    def forward(self, state, action, next_state, done):
        base_out = self.base(state, action, next_state, done)
        new_shaping = self.potential(next_state).flatten()  # evaluated BEFORE potential(state), as the reference
        old_shaping = self.potential(state).flatten()
        final = base_out + self.discount_factor * (1 - done.float()) * new_shaping - old_shaping
        assert final.shape == state.shape[:1]
        return final


class BasicShapedRewardNet(_FusedNetMixin, ShapedRewardNet):
    """Shaped reward net with MLP base and MLP potential; one fused 3-pass kernel."""

    def __init__(self, observation_space, action_space, *, reward_hid_sizes: Sequence[int] = (32,),
                 potential_hid_sizes: Sequence[int] = (32, 32), use_state: bool = True, use_action: bool = True,
                 use_next_state: bool = False, use_done: bool = False, discount_factor: float = 0.99, **kwargs):
        base = BasicRewardNet(observation_space, action_space, use_state=use_state, use_action=use_action,
                              use_next_state=use_next_state, use_done=use_done, hid_sizes=reward_hid_sizes, **kwargs)
        potential = BasicPotentialMLP(observation_space, hid_sizes=potential_hid_sizes, **kwargs)
        super().__init__(base, potential, discount_factor=discount_factor)
        self._engine = self._make_engine()

    def _make_engine(self) -> FusedEngine:
        b: BasicRewardNet = self._base
        p: BasicPotentialMLP = self.potential
        d = _desc.disc_desc(b._d_obs, b._d_act, hid_sizes=b._hid_sizes, use_state=b.use_state,
                            use_action=b.use_action, use_next_state=b.use_next_state, use_done=b.use_done,
                            normalize_input=b._norm, shaped=True, potential_hid_sizes=p._hid_sizes,
                            gamma=self.discount_factor)
        if b._norm != p._norm:
            raise NotImplementedError("base and potential must both (or neither) use an input RunningNorm")
        return FusedEngine(d, [b.mlp, p._potential_net])

    def forward(self, state, action, next_state, done):
        out = self._fused_forward(state, action, next_state, done)
        assert out.shape == state.shape[:1]
        return out


_OUTPUT_NORMS = {"RunningNorm": networks.RunningNorm, "EMANorm": networks.EMANorm}


class NormalizedRewardNet(PredictProcessedWrapper):
    """Normalises `predict_processed` output with a running norm, updating it on every call
    (reward_nets.py:613-671).  `normalize_output_layer` is RunningNorm or EMANorm (this package's or the reference's
    class, matched by name), or a `functools.partial` of one carrying its keyword arguments (EMANorm's `decay`, `eps`);
    the layer is built as `normalize_output_layer(1)`, as the reference builds it."""

    def __init__(self, base: RewardNet, normalize_output_layer: Type[nn.Module]):
        super().__init__(base=base)
        layer = normalize_output_layer
        func, args, kw = ((layer.func, layer.args, layer.keywords) if isinstance(layer, functools.partial)
                          else (layer, (), {}))
        cls = _OUTPUT_NORMS.get(getattr(func, "__name__", ""))
        if cls is None:
            raise NotImplementedError("normalize_output_layer must be RunningNorm or EMANorm (or a functools.partial "
                                      f"of one), got {layer!r}")
        self.normalize_output_layer = cls(*args, 1, **kw)

    @property
    def output_norm_is_ema(self) -> bool:
        return isinstance(self.normalize_output_layer, networks.EMANorm)

    def predict_processed(self, state, action, next_state, done, update_stats: bool = True, **kwargs) -> np.ndarray:
        with networks.evaluating(self):
            rew_th = th.tensor(self.base.predict_processed(state, action, next_state, done, **kwargs),
                               device=self.device)
            rew = self.normalize_output_layer(rew_th).detach().cpu().numpy().flatten()
        if update_stats:
            with th.no_grad():
                self.normalize_output_layer.update_stats(rew_th)
        assert rew.shape == state.shape[:1]
        return rew

    def output_norm_vectors(self) -> Tuple[th.Tensor, th.Tensor]:
        """Float vector + int32 vector aliased by the norm's buffers (for the kernels): RunningNorm [mean, var] and
        [count]; EMANorm [mean, var, inv_learning_rate] and [count, num_batches]."""
        n = self.normalize_output_layer
        alias = self.__dict__.get("_out_alias")
        if alias is None or alias[0] is not n:
            ema = self.output_norm_is_ema
            fl = ["running_mean", "running_var"] + (["inv_learning_rate"] if ema else [])
            it = ["count"] + (["num_batches"] if ema else [])
            alias = (n, FlatAlias([(n, k) for k in fl]), FlatAlias([(n, k) for k in it]))
            self.__dict__["_out_alias"] = alias
        dev = self.device
        return alias[1].get(th.float32, dev), alias[2].get(th.int32, dev)

    def output_norm_args(self) -> tuple:
        """The member entry `_lib.pref_uncertainty_desc` takes: (state, count, eps), plus decay for an EMANorm."""
        n = self.normalize_output_layer
        return (*self.output_norm_vectors(), float(n.eps)) + ((float(n.decay),) if self.output_norm_is_ema else ())

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_out_alias", None)
        return state


class RewardEnsemble(RewardNetWithVariance):
    """Independent members; mean/variance over members (reward_nets.py:884-1016)."""

    members: nn.ModuleList

    def __init__(self, observation_space, action_space, members: Iterable[RewardNet]):
        super().__init__(observation_space, action_space)
        members = list(members)
        if len(members) < 2:
            raise ValueError("Must be at least 2 member in the ensemble.")
        self.members = nn.ModuleList(members)

    @property
    def num_members(self):
        return len(self.members)

    def predict_processed_all(self, state, action, next_state, done, **kwargs) -> np.ndarray:
        rewards = np.stack([m.predict_processed(state, action, next_state, done, **kwargs) for m in self.members], -1)
        assert rewards.shape == (state.shape[0], self.num_members)
        return rewards

    @th.no_grad()
    def predict_reward_moments(self, state, action, next_state, done, **kwargs):
        allr = self.predict_processed_all(state, action, next_state, done, **kwargs)
        return allr.mean(-1), allr.var(-1, ddof=1)

    def forward(self, *args) -> th.Tensor:
        raise NotImplementedError

    def predict_processed(self, state, action, next_state, done, **kwargs) -> np.ndarray:
        return self.predict(state, action, next_state, done, **kwargs)

    def predict(self, state, action, next_state, done, **kwargs):
        mean, _ = self.predict_reward_moments(state, action, next_state, done, **kwargs)
        return mean


class AddSTDRewardWrapper(PredictProcessedWrapper):
    """mean + alpha * std of a RewardNetWithVariance (reward_nets.py:1019-1080)."""

    base: RewardNetWithVariance

    def __init__(self, base: RewardNetWithVariance, default_alpha: float = 0.0):
        super().__init__(base)
        if not isinstance(base, RewardNetWithVariance):
            raise TypeError("Cannot add standard deviation to reward net that is not an instance of "
                            "RewardNetWithVariance!")
        self.default_alpha = default_alpha

    def predict_processed(self, state, action, next_state, done, alpha: Optional[float] = None, **kwargs):
        del kwargs
        if alpha is None:
            alpha = self.default_alpha
        mean, var = self.base.predict_reward_moments(state, action, next_state, done)
        return mean + alpha * np.sqrt(var)
