"""util/flat.py on CPU: module parameters and buffers kept as views of one flat vector."""
import pytest
import torch as th
from torch import nn

from imitation_b200.util import networks
from imitation_b200.util.flat import FlatAlias, contiguous_view, views

CPU = th.device("cpu")


def _mlp(seed=0):
    th.manual_seed(seed)
    return nn.Sequential(nn.Linear(3, 4), nn.ReLU(), nn.Linear(4, 2))


def _param_alias(mlp):
    return FlatAlias([(m, k) for m in mlp if isinstance(m, nn.Linear) for k in ("weight", "bias")])


def _views_of(tensors, flat):
    """Every tensor is the next slice of `flat`."""
    off = 0
    for t in tensors:
        assert t.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
        assert t.data_ptr() == flat.data_ptr() + flat.element_size() * off and t.is_contiguous()
        off += t.numel()
    assert off == flat.numel()


def _buffers(**tensors):
    m = nn.Module()
    for k, t in tensors.items():
        m.register_buffer(k, t)
    return m


def test_first_get_flattens_keeping_values_and_parameter_objects():
    mlp = _mlp()
    params = list(mlp.parameters())
    before = [p.detach().clone() for p in params]
    opt = th.optim.SGD(mlp.parameters(), lr=1.0)
    flat = _param_alias(mlp).get(th.float32, CPU)
    assert all(a is b for a, b in zip(mlp.parameters(), params))
    assert th.equal(flat, th.cat([b.reshape(-1) for b in before]))
    assert all(th.equal(p, b) for p, b in zip(params, before))
    _views_of(params, flat)
    # the module's torch forward reads the flat vector
    flat.zero_()
    flat[-2:] = th.tensor([1.0, 2.0])  # the last Linear's bias
    assert th.equal(mlp(th.randn(5, 3)), th.tensor([[1.0, 2.0]] * 5))
    # a torch optimiser holding the Parameter objects steps the flat vector
    for p in params:
        p.grad = th.ones_like(p)
    opt.step()
    assert th.equal(flat[-2:], th.tensor([0.0, 1.0])) and th.equal(flat[:-2], -th.ones(flat.numel() - 2))


def test_second_get_returns_the_same_vector():
    mlp = _mlp()
    alias = _param_alias(mlp)
    flat = alias.get(th.float32, CPU)
    ptrs = [p.data_ptr() for p in mlp.parameters()]
    again = alias.get(th.float32, CPU)
    assert again is flat and again.data_ptr() == flat.data_ptr()
    assert [p.data_ptr() for p in mlp.parameters()] == ptrs


def test_back_to_back_tensors_are_adopted_without_a_copy():
    s = th.arange(6.0)
    m = _buffers(a=s[1:3], b=s[3:6])
    flat = FlatAlias([(m, "a"), (m, "b")]).get(th.float32, CPU)
    assert flat.data_ptr() == s[1:].data_ptr() and th.equal(flat, s[1:])
    assert m.a.data_ptr() == s[1:].data_ptr() and m.b.data_ptr() == s[3:].data_ptr()
    # a sub-network adopts its slice of the enclosing network's vector (the base of a shaped reward net)
    outer, inner = _mlp(), _mlp(1)
    whole = FlatAlias([(m, k) for net in (outer, inner) for m in net if isinstance(m, nn.Linear)
                       for k in ("weight", "bias")]).get(th.float32, CPU)
    part = _param_alias(inner).get(th.float32, CPU)
    n_outer = sum(p.numel() for p in outer.parameters())
    assert part.data_ptr() == whole[n_outer:].data_ptr() and th.equal(part, whole[n_outer:])


def _wrong_dtype():
    s = th.arange(5.0, dtype=th.float64)
    return _buffers(a=s[:2], b=s[2:])


def _gap():
    s = th.arange(6.0)
    return _buffers(a=s[:2], b=s[3:])


def _two_storages():
    return _buffers(a=th.arange(2.0), b=th.arange(2.0, 5.0))


def _strided():
    s = th.arange(7.0)
    return _buffers(a=s[0:4:2], b=s[2:5])  # b starts where a would end if a were contiguous


def _re_pointed():
    m = _buffers(a=th.arange(2.0), b=th.arange(2.0, 5.0))
    FlatAlias([(m, "a"), (m, "b")]).get(th.float32, CPU)
    m.b = th.tensor([7.0, 8.0, 9.0])
    return m


@pytest.mark.parametrize("make", [_wrong_dtype, _gap, _two_storages, _strided, _re_pointed])
def test_tensors_not_back_to_back_are_re_flattened_keeping_values(make):
    m = make()
    want = th.cat([m.a.reshape(-1), m.b.reshape(-1)]).float()
    old = [m.a, m.b]
    assert contiguous_view(old, th.float32, CPU) is None
    alias = FlatAlias([(m, "a"), (m, "b")])
    flat = alias.get(th.float32, CPU)
    assert flat.dtype == th.float32 and th.equal(flat, want)
    assert all(x.untyped_storage().data_ptr() != flat.untyped_storage().data_ptr() for x in old)
    _views_of([m.a, m.b], flat)
    assert m.a.shape == old[0].shape and m.b.shape == old[1].shape
    assert alias.get(th.float32, CPU) is flat


def test_re_pointed_parameter_is_re_flattened_and_keeps_its_object():
    mlp = _mlp()
    alias = _param_alias(mlp)
    first = alias.get(th.float32, CPU)
    bias = mlp[2].bias
    bias.data = th.tensor([5.0, 6.0])
    flat = alias.get(th.float32, CPU)
    assert flat is not first and th.equal(flat[:-2], first[:-2]) and th.equal(flat[-2:], th.tensor([5.0, 6.0]))
    assert mlp[2].bias is bias
    _views_of(list(mlp.parameters()), flat)


def test_wrong_device_is_re_flattened_onto_the_requested_device():
    s = th.arange(5.0)
    m = _buffers(a=s[:2], b=s[2:])
    meta = th.device("meta")
    assert contiguous_view([m.a, m.b], th.float32, meta) is None
    flat = FlatAlias([(m, "a"), (m, "b")]).get(th.float32, meta)
    assert flat.device == meta and flat.shape == (5,)
    assert m.a.device == meta and m.a.shape == (2,) and m.b.device == meta and m.b.shape == (3,)


def test_running_norms_0d_int32_counts():
    norms = [networks.RunningNorm(3), networks.RunningNorm(2)]
    for k, n in enumerate(norms):
        n.update_stats(th.randn(4 + k, n.num_features))
    sd = [{k: v.clone() for k, v in n.state_dict().items()} for n in norms]
    state = FlatAlias([(n, k) for n in norms for k in ("running_mean", "running_var")]).get(th.float32, CPU)
    count = FlatAlias([(n, "count") for n in norms]).get(th.int32, CPU)
    assert count.tolist() == [4, 5] and state.numel() == 10
    _views_of([t for n in norms for t in (n.running_mean, n.running_var)], state)
    _views_of([n.count for n in norms], count)
    for n, want in zip(norms, sd):
        got = n.state_dict()
        assert list(got) == list(want)
        for k in want:
            assert got[k].shape == want[k].shape and got[k].dtype == want[k].dtype and th.equal(got[k], want[k]), k
    norms[1].update_stats(th.randn(3, 2))  # the module's torch update writes into the flat vectors
    assert count.tolist() == [4, 8] and th.equal(state[6:8], norms[1].running_mean)


def test_ema_norm_mixed_shapes():
    n = networks.EMANorm(1, decay=0.9)
    n.update_stats(th.randn(7))
    n.update_stats(th.randn(3))
    sd = {k: v.clone() for k, v in n.state_dict().items()}
    state = FlatAlias([(n, "running_mean"), (n, "running_var"), (n, "inv_learning_rate")]).get(th.float32, CPU)
    count = FlatAlias([(n, "count"), (n, "num_batches")]).get(th.int32, CPU)
    assert count.tolist() == [10, 2]
    assert th.equal(state, th.cat([sd["running_mean"], sd["running_var"], sd["inv_learning_rate"].reshape(1)]))
    assert n.inv_learning_rate.data_ptr() == state.data_ptr() + 8 and n.num_batches.data_ptr() == count.data_ptr() + 4
    for k, v in n.state_dict().items():
        assert v.shape == sd[k].shape and v.dtype == sd[k].dtype and th.equal(v, sd[k]), k
    n.update_stats(th.randn(4))
    assert count.tolist() == [14, 3] and float(state[2]) == float(n.inv_learning_rate)


def test_load_state_dict_writes_through():
    mlp, other = _mlp(), _mlp(1)
    norm = networks.RunningNorm(3)
    alias, count_alias = _param_alias(mlp), FlatAlias([(norm, "count")])
    flat, count = alias.get(th.float32, CPU), count_alias.get(th.int32, CPU)
    mlp.load_state_dict(other.state_dict())
    assert th.equal(flat, th.cat([p.detach().reshape(-1) for p in other.parameters()]))
    assert alias.get(th.float32, CPU) is flat
    norm.load_state_dict({"running_mean": th.ones(3), "running_var": th.ones(3), "count": th.tensor(9, dtype=th.int32)})
    assert count.tolist() == [9] and count_alias.get(th.int32, CPU) is count


def test_views_are_consecutive_slices():
    flat = th.arange(10.0)
    a, b, c = views(flat, [(2, 3), (), (3,)])
    assert a.shape == (2, 3) and b.shape == () and c.shape == (3,)
    _views_of([a, b, c], flat)
    assert th.equal(a.reshape(-1), flat[:6]) and float(b) == 6.0 and th.equal(c, flat[7:])
