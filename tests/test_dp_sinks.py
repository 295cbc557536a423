"""The gradient bucket's sinks (neuraludf_b200/dp.py) with real autograd, on the CPU.

A stand-in for a kernel-backed network's autograd.Function takes its gradient targets from ops._grad_targets (bucket views
when the handle's sink is armed, fresh tensors otherwise) and OVERWRITES them, as the library's backward kernels do after
their memset.  So these runs go through the engine's input buffers and AccumulateGrad exactly like the real networks, and
every `.grad` must equal, bit for bit, the run without a bucket (at world 1) or exactly half of it (at world 2 on torch's
fake process group, whose all_reduce leaves the local values: the mean is local * 0.5).
"""
import itertools

import pytest
import torch
import torch.distributed as dist

from neuraludf_b200 import dp, ops

D_IN, D_HID, D_OUT, N_PTS = 3, 5, 2, 7
STEPS = 3


class _Layer(torch.nn.Module):
    """weight_g [out, 1], weight_v [out, in], bias [out]: what UdfHandle reads from a weight-normed layer"""

    def __init__(self, n_in, n_out, gen):
        super().__init__()
        self.weight_v = torch.nn.Parameter(torch.randn(n_out, n_in, generator=gen))
        self.weight_g = torch.nn.Parameter(torch.rand(n_out, 1, generator=gen) + 0.5)
        self.bias = torch.nn.Parameter(torch.randn(n_out, generator=gen) * 0.1)


def _weights(m):
    vn = m.weight_v / m.weight_v.norm(dim=1, keepdim=True)
    return m.weight_g * vn, vn


class _StandIn(torch.autograd.Function):
    """y = tanh(x W0^T + b0) W1^T + b1 with W = g v / |v|; the backward in closed form, written like ops._UdfFunction's"""

    @staticmethod
    def forward(ctx, x, handle, *params):
        l0, l1 = handle.layers
        h = torch.tanh(x @ _weights(l0)[0].t() + l0.bias)
        ctx.handle = handle
        ctx.save_for_backward(x, h)
        return h @ _weights(l1)[0].t() + l1.bias

    @staticmethod
    def backward(ctx, y_bar):
        x, h = ctx.saved_tensors
        hd = ctx.handle
        l0, l1 = hd.layers
        z_bar = (y_bar @ _weights(l1)[0]) * (1.0 - h * h)
        dws = [z_bar.t() @ x, y_bar.t() @ h]
        sink, db, dgs, dvs, dbs = ops._grad_targets(hd, hd.layers)
        db.copy_(torch.cat([z_bar.sum(0), y_bar.sum(0)]))            # the ONE bias block, in layer order
        for m, dw, dg, dv in zip(hd.layers, dws, dgs, dvs):         # the weight-norm backward (unfold_grads)
            _, vn = _weights(m)
            g_hat = (dw * vn).sum(1, keepdim=True)
            dg.copy_(g_hat)
            dv.copy_(m.weight_g / m.weight_v.norm(dim=1, keepdim=True) * (dw - g_hat * vn))
        if sink is not None:
            sink.ready()
        grads = []
        for l in range(len(hd.layers)):
            grads += [dgs[l], dvs[l], dbs[l]]
        return (None, None) + tuple(grads)


class _Net(torch.nn.Module):
    """a network behind a real ops.UdfHandle, so that GradBucket arms it as it arms UDFNetwork"""

    def __init__(self, gen):
        super().__init__()
        self.lin0, self.lin1 = _Layer(D_IN, D_HID, gen), _Layer(D_HID, D_OUT, gen)
        self._handle = ops.UdfHandle([self.lin0, self.lin1], D_IN, 0, D_OUT, -1, 1.0)

    def forward(self, x):
        return _StandIn.apply(x, self._handle, *self._handle.params())


def _model():
    """a sinked network, a partially frozen one (plain path: its trainable parameters join the loose tail) and loose
    scalars, like the renderer's networks and variance / beta heads"""
    gen = torch.Generator().manual_seed(1)
    a, b = _Net(gen), _Net(gen)
    b.lin0.weight_g.requires_grad_(False)
    s = torch.nn.Parameter(torch.tensor(0.7))
    t = torch.nn.Parameter(torch.tensor([0.3, -1.1]))
    params = list(a.parameters()) + list(b.parameters()) + [s, t]
    return a, b, s, t, params


def _loss(a, b, s, t, step, k, twice):
    g = torch.Generator().manual_seed(100 * step + 10 * k)
    x = lambda: torch.randn(N_PTS, D_IN, generator=g)
    w = lambda: torch.randn(N_PTS, D_OUT, generator=g)
    ya = a(x())
    loss = s * (ya * w()).sum() + (b(x()) * w()).sum() + (t * ya.mean(0)).sum()
    if twice:                                   # the network reached a second time in the same graph (an eikonal term)
        loss = loss + (a(x()) * w()).sum()
    return loss


def _expected_offsets(net):
    """each sinked parameter's slot, from the handle's layout alone: biases first, then g / v of every layer"""
    out, off = {}, 0
    for group in net._handle.sink_layout():
        for p in group:
            out[id(p)] = off
            off += p.numel()
    return out


def _run(bucketed, overlap, set_to_none, twice, n_back, reduce=True, calls=None):
    """STEPS steps of zero_grad + n_back backward passes (+ allreduce_mean); the gradients of every step"""
    a, b, s, t, params = _model()
    opt = torch.optim.SGD(params, lr=0.0)             # for its zero_grad only
    bucket = dp.GradBucket(params, modules=[a, b], overlap=overlap) if bucketed else None
    if bucket is not None:
        assert len(bucket.regions) == 1 and a._handle.grad_sink is bucket.regions[0] and b._handle.grad_sink is None
    res = []
    for step in range(STEPS):
        opt.zero_grad(set_to_none=set_to_none)
        if calls is not None:
            calls.clear()
        for k in range(n_back):
            _loss(a, b, s, t, step, k, twice).backward()
        if bucket is not None and reduce:
            bucket.allreduce_mean()
            _assert_in_slots(a, bucket.flat)
            if calls is not None:
                _check_one_collective_each(bucket.flat, calls, dist.is_initialized())
        res.append([None if p.grad is None else p.grad.clone() for p in params])
        assert b.lin0.weight_g.grad is None
    return res, bucket, a


def _assert_in_slots(net, flat):
    """every sinked .grad IS its slot of the flat buffer: same storage, the layout's offset, the parameter's shape"""
    offsets = _expected_offsets(net)
    for p in net.parameters():
        g = p.grad
        assert g.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
        assert g.storage_offset() == flat.storage_offset() + offsets[id(p)]
        assert g.shape == p.shape and g.is_contiguous()


def _check_one_collective_each(flat, calls, distributed):
    seen = torch.zeros(flat.numel(), dtype=torch.int64)
    for x in calls:
        assert x.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr(), "a collective outside the bucket"
        lo = x.storage_offset() - flat.storage_offset()
        seen[lo:lo + x.numel()] += 1
    if distributed:
        assert bool((seen == 1).all()), "elements reduced %s times" % sorted(set(seen.tolist()))
    else:
        assert not calls


def _assert_grads(got, ref, scale):
    for step, (gs, rs) in enumerate(zip(got, ref)):
        for i, (g, r) in enumerate(zip(gs, rs)):
            if r is None:
                assert g is None, (step, i)
                continue
            assert torch.equal(g, r * scale), (step, i, float((g - r * scale).abs().max()))


@pytest.fixture(params=[1, 2], ids=["world1", "fake_world2"])
def world(request):
    if request.param == 1:
        yield 1
        return
    from torch.testing._internal.distributed.fake_pg import FakeStore
    dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=2)
    try:
        yield 2
    finally:
        dist.destroy_process_group()


@pytest.fixture
def collectives(monkeypatch):
    """every tensor handed to dist.all_reduce (the bucket's only collective)"""
    calls = []
    real = dist.all_reduce

    def spy(tensor, *args, **kw):
        calls.append(tensor)
        return real(tensor, *args, **kw)
    monkeypatch.setattr(dp.dist, "all_reduce", spy)
    return calls


CASES = list(itertools.product([True, False], [True, False], [False, True], [1, 2]))


@pytest.mark.parametrize("overlap,set_to_none,twice,n_back", CASES,
                         ids=["%s-%s-%s-%d" % ("overlap" if o else "sync", "none" if z else "zero", "twice" if t else "once",
                                               n) for o, z, t, n in CASES])
def test_sinked_gradients_match_the_run_without_bucket(world, collectives, overlap, set_to_none, twice, n_back):
    ref, _, _ = _run(False, overlap, set_to_none, twice, n_back)
    if world == 2 and overlap and (twice or n_back > 1):
        # the region went to the collective when its first invocation was done: a second one cannot be added any more
        with pytest.raises(RuntimeError, match="construct the bucket with overlap=False"):
            _run(True, overlap, set_to_none, twice, n_back, calls=collectives)
        return
    got, _, _ = _run(True, overlap, set_to_none, twice, n_back, calls=collectives)
    _assert_grads(got, ref, 1.0 if world == 1 else 0.5)


@pytest.mark.parametrize("set_to_none,twice,n_back", list(itertools.product([True, False], [False, True], [1, 2])))
def test_world1_without_allreduce(set_to_none, twice, n_back):
    """one process with no allreduce_mean() between steps (bench.py's single-GPU step): still the unbucketed gradients, and
    with one backward of a network reached once after zero_grad(set_to_none=True), the kernels wrote the slots in place"""
    ref, _, _ = _run(False, True, set_to_none, twice, n_back)
    got, bucket, a = _run(True, True, set_to_none, twice, n_back, reduce=False)
    _assert_grads(got, ref, 1.0)
    if set_to_none and not twice and n_back == 1:
        _assert_in_slots(a, bucket.flat)
