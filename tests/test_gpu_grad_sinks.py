"""The gradient bucket (neuraludf_b200/dp.py) through the real backward kernels: the UDF, colour and NeRF++ backward passes
of test_gpu_blend's render_core write their parameter gradients straight into the bucket, and autograd adopts them.

Every sinked gradient must equal, bit for bit, the same kernels' gradient without a bucket (the weight gradients are
deterministic: split-K partial sums are added in split order), lie in its slot of the flat buffer, survive
allreduce_mean(), and still pass test_gpu_blend's fp64 check.
"""
import os
import sys
import tempfile
import time
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from neuraludf_b200.synthetic import make_blend_views
from tests.golden_util import Fixtures
from tests.gpu_util import ROOT, build_modules, err_inf, report, scale_inf
from tests.test_gpu_blend import _loss

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_RAYS, S, N_OUT, N_VIEWS = 16, 32, 8, 6
# (make_blend_views seed, zero_grad(set_to_none=...), add the eikonal terms): the UDF network is reached three times in one
# backward on the eikonal steps
STEPS = ((0, True, False), (1, False, True), (2, True, True))


@pytest.fixture(scope="module")
def fx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return Fixtures("blend_outputs")


def _inputs(seed, n_rays, dev):
    """make_blend_views' rays with the fixture generator's sample depths (oracle/make_golden_blend.py)"""
    v = make_blend_views(n_rays, n_views=N_VIEWS, seed=seed)
    near, far = v["near"], v["far"]
    z = near + (far - near) * torch.linspace(0.0, 1.0, S)[None, :]
    sd = ((far - near) / S).mean().item()
    z_out = torch.linspace(1e-3, 1.0 - 1.0 / (N_OUT + 1.0), N_OUT)
    z_out = far / torch.flip(z_out, dims=[-1]) + 1.0 / S
    z_feed, _ = torch.sort(torch.cat([z, z_out], dim=-1), dim=-1)
    v = {k: t.to(dev) for k, t in v.items()}
    v.update(z=z.to(dev).contiguous(), z_feed=z_feed.to(dev).contiguous(), sd=sd)
    return v


def _shard(v, lo, hi):
    per_ray = ("rays_o", "rays_d", "near", "far", "rays_uv", "z", "z_feed")
    return {k: (t[lo:hi].contiguous() if k in per_ray else t) for k, t in v.items()}


class _Model:
    def __init__(self, golden, dev):
        from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
        self.mods = build_modules(golden, dev)
        udf, col, nerf, var, beta = self.mods
        self.ren = UDFRendererBlending(nerf, udf, var, col, beta, n_samples=S, n_importance=0, n_outside=N_OUT,
                                       up_sample_steps=0, perturb=0.0)
        self.params = [p for m in self.mods for p in m.parameters() if p.requires_grad]
        self.names = ["%s.%s" % (mn, pn) for mn, m in zip(("udf", "color", "nerf", "variance", "beta"), self.mods)
                      for pn, p in m.named_parameters() if p.requires_grad]

    def zero_grad(self, set_to_none):
        for m in self.mods:
            m.zero_grad(set_to_none=set_to_none)

    def render(self, v):
        udf, col, nerf, var, beta = self.mods
        bg = self.ren.render_core_outside(v["rays_o"], v["rays_d"], v["z_feed"], v["sd"], nerf)
        return self.ren.render_core(v["rays_o"], v["rays_d"], v["z"], v["sd"], udf, var, col, beta_network=beta,
                                    cos_anneal_ratio=0.8, background_alpha=bg["alpha"],
                                    background_sampled_color=bg["sampled_color"], flip_saturation=0.1,
                                    color_maps=v["color_maps"], w2cs=v["w2cs"], intrinsics=v["intrinsics"],
                                    query_c2w=v["query_c2w"], img_index=None, rays_uv=v["rays_uv"].clone())

    def step(self, seed, set_to_none, eikonal, loss_fn=_loss, v=None):
        """zero_grad + one backward; the parameter gradients (clones, None where there is none)"""
        self.zero_grad(set_to_none)
        v = _inputs(seed, N_RAYS, DEV) if v is None else v
        ret = self.render(v)
        loss = loss_fn(ret)
        if eikonal:                          # the UDF network twice more in the same graph: udf.gradient and udf
            udf = self.mods[0]
            g = torch.Generator().manual_seed(50 + seed)
            x = (torch.rand(256, 3, generator=g) * 1.6 - 0.8).to(DEV)
            loss = loss + 0.1 * ((udf.gradient(x).norm(dim=-1) - 1.0) ** 2).mean() + 0.01 * udf(x)[:, 0].abs().mean()
        loss.backward()
        return self.grads()

    def grads(self):
        return [None if p.grad is None else p.grad.detach().clone() for p in self.params]


def _bucket(model, overlap=True):
    from neuraludf_b200 import dp
    udf, col, nerf = model.mods[:3]
    b = dp.GradBucket(model.params, modules=(udf, col, nerf), overlap=overlap)
    assert len(b.regions) == 3
    return b


def _assert_in_slots(model, bucket):
    """every sinked parameter's .grad IS its slot of bucket.flat: the storage, the offset of the handles' layout, the shape"""
    flat, off = bucket.flat, 0
    n = 0
    for m in model.mods[:3]:
        for group in m._handle.sink_layout():
            for p in group:
                g = p.grad
                assert g is not None and g.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
                assert g.storage_offset() == flat.storage_offset() + off and g.shape == p.shape and g.is_contiguous()
                off += p.numel()
                n += 1
    assert n >= 60


def _assert_same(tag, names, got, ref, scale=1.0):
    for name, g, r in zip(names, got, ref):
        if r is None:
            assert g is None or float(g.abs().max()) == 0.0, name
            continue
        e = err_inf(g, r * scale)
        report(tag + name, err=e)
        assert torch.equal(g, r * scale), "%s: differs by %.3e (max |ref| %.3e)" % (name, e, scale_inf(r))


def _fp64_anchor(tag, model, fx):
    """test_gpu_blend's check of the parameter gradients against the fp64 fixtures"""
    from oracle.make_golden import GRAD_STRIDE
    worst, n = 0.0, 0
    for mn, m in (("udf", model.mods[0]), ("color", model.mods[1]), ("nerf", model.mods[2])):
        for pn, p in m.named_parameters():
            key = "blend_grad.%s.%s_f64" % (mn, pn)
            if key in fx.files:
                ref, new = torch.from_numpy(fx[key]), p.grad.cpu()
            elif key + "_sub" in fx.files:
                ref, new = torch.from_numpy(fx[key + "_sub"]), p.grad.reshape(-1)[::GRAD_STRIDE].cpu()
            else:
                assert p.grad is None or float(p.grad.abs().max()) == 0.0, key
                continue
            e = err_inf(new, ref) / scale_inf(ref)
            worst = max(worst, e)
            n += 1
            report(tag + "dparam.%s.%s" % (mn, pn), rel=e)
            assert e < 2e-3, (key, e)
    assert n >= 60
    report(tag + "dparam.worst_rel", rel=worst)


@pytest.fixture
def engine(request):
    from neuraludf_b200 import _lib
    L = _lib.lib()
    old = L.nudf_get_engine()
    L.nudf_set_engine(request.param)
    yield request.param
    L.nudf_set_engine(old)


@pytest.mark.parametrize("engine", [0, 1], indirect=True)
def test_sinked_gradients_match_fp64_and_the_unbucketed_kernels(golden, fx, engine):
    """three steps (different rays; zero_grad with set_to_none True / False / True; the eikonal terms on the last two) with
    allreduce_mean() between them, against a run without a bucket"""
    plain, sinked = _Model(golden, DEV), _Model(golden, DEV)
    bucket = _bucket(sinked)
    tag = "grad_sinks.e%d." % engine
    v0 = _inputs(0, N_RAYS, DEV)
    assert torch.equal(v0["z"].cpu(), torch.from_numpy(fx["blend_z"]))
    for i, (seed, set_to_none, eikonal) in enumerate(STEPS):
        ref = plain.step(seed, True, eikonal)
        got = sinked.step(seed, set_to_none, eikonal)
        if i == 0:
            _fp64_anchor(tag, sinked, fx)                   # the gradients the kernels wrote into the bucket
        bucket.allreduce_mean()
        _assert_in_slots(sinked, bucket)
        _assert_same(tag + "step%d." % i, sinked.names, got, ref)
        _assert_same(tag + "step%d.adopted." % i, sinked.names, sinked.grads(), ref)


@pytest.fixture
def fake_world2():
    from torch.testing._internal.distributed.fake_pg import FakeStore
    dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=2)
    try:
        yield
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("overlap", [True, False])
def test_sinked_gradients_fake_world2(golden, fx, fake_world2, overlap):
    """world 2 on torch's fake process group (its all_reduce leaves the local values): the mean must be exactly half of the
    unbucketed gradients.  With overlap the regions are reduced as their backward finishes, so a network reached again in
    the same backward is refused; without it the eikonal steps run too."""
    plain, sinked = _Model(golden, DEV), _Model(golden, DEV)
    bucket = _bucket(sinked, overlap=overlap)
    for i, (seed, set_to_none, eikonal) in enumerate(STEPS):
        eikonal = eikonal and not overlap
        ref = plain.step(seed, True, eikonal)
        sinked.step(seed, set_to_none, eikonal)
        bucket.allreduce_mean()
        _assert_in_slots(sinked, bucket)
        _assert_same("grad_sinks.fake2.%s.step%d." % ("overlap" if overlap else "sync", i), sinked.names, sinked.grads(),
                     ref, 0.5)
    if overlap:
        with pytest.raises(RuntimeError, match="construct the bucket with overlap=False"):
            sinked.step(3, True, True)


# ---- two real ranks --------------------------------------------------------------------------------------------------
def _ray_mean_loss(ret):
    """_loss without its mask-count normalisations: a mean over rays, so that the mean of the two halves' losses is the
    full batch's loss"""
    tgt = 0.4
    loss = (ret["color"] - tgt).abs().mean() + 0.5 * (ret["color_pixel"] - tgt).abs().mean()
    loss = loss + 0.01 * (ret["color_base"] - tgt).abs().mean() + 0.1 * ret["sparse_error"]
    pm = ret["patch_mask"].detach()
    return loss + 0.5 * ((ret["patch_colors"] - 0.4).abs().mean(dim=(1, 2)) * pm).mean()


def _rank_worker(rank, world, port, backend, engine, out_dir):
    sys.path.insert(0, ROOT)
    try:
        from neuraludf_b200 import _lib, dp
        from tests.golden_util import load_golden
        dev = torch.device("cuda", rank if torch.cuda.device_count() >= world else 0)
        torch.cuda.set_device(dev)
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        dist.init_process_group(backend, rank=rank, world_size=world)
        try:
            _lib.lib().nudf_set_engine(engine)
            model = _Model(load_golden(), dev)
            bucket = _bucket(model)
            lo, hi = dp.shard_bounds(2 * N_RAYS, rank, world)
            v = _inputs(0, 2 * N_RAYS, dev)
            sh = {k: t for k, t in zip(("rays_o", "rays_d"), dp.shard_rays(v["rays_o"], v["rays_d"], rank=rank,
                                                                              world=world))}
            model.zero_grad(True)
            ret = model.render(dict(_shard(v, lo, hi), **sh))
            _ray_mean_loss(ret).backward()
            bucket.allreduce_mean()
            _assert_in_slots(model, bucket)
            torch.save([None if g is None else g.cpu() for g in model.grads()], os.path.join(out_dir, "rank%d.pt" % rank))
        finally:
            dist.destroy_process_group()
    except Exception:
        with open(os.path.join(out_dir, "rank%d.err" % rank), "w") as f:
            f.write(traceback.format_exc())


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _spawn(backend, engine, out_dir, timeout=600.0):
    ctx = mp.spawn(_rank_worker, args=(2, _free_port(), backend, engine, out_dir), nprocs=2, join=False)
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=5.0):
            assert time.monotonic() < deadline, "the ranks did not finish in %.0f s" % timeout
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.terminate()
            p.join()


@pytest.mark.parametrize("backend,engine", [("gloo", 0), ("gloo", 1), ("nccl", 1)])
def test_two_ranks_allreduce(golden, fx, backend, engine, request):
    """two processes, each rendering its shard_rays half of one 2N-ray batch: after allreduce_mean() both hold exactly
    (g0 + g1) * 0.5 of the unbucketed half-batch gradients, and the full batch's gradient to fp32 rounding"""
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("NCCL needs a device per rank: %d visible" % torch.cuda.device_count())
    from neuraludf_b200 import _lib, dp
    L = _lib.lib()
    old = L.nudf_get_engine()
    L.nudf_set_engine(engine)
    try:
        model = _Model(golden, DEV)
        v = _inputs(0, 2 * N_RAYS, DEV)
        halves = []
        for r in range(2):
            lo, hi = dp.shard_bounds(2 * N_RAYS, r, 2)
            halves.append(model.step(None, True, False, loss_fn=_ray_mean_loss, v=_shard(v, lo, hi)))
        full = model.step(None, True, False, loss_fn=_ray_mean_loss, v=v)
    finally:
        L.nudf_set_engine(old)
    with tempfile.TemporaryDirectory() as out_dir:
        _spawn(backend, engine, out_dir)
        errs = [os.path.join(out_dir, "rank%d.err" % r) for r in range(2)]
        errs = [open(e).read() for e in errs if os.path.exists(e)]
        if errs and backend == "gloo" and "gloo" in errs[0].lower() and "cuda" in errs[0].lower():
            pytest.skip("gloo refused CUDA tensors: " + errs[0].strip().splitlines()[-1])
        assert not errs, errs[0]
        ranks = [torch.load(os.path.join(out_dir, "rank%d.pt" % r)) for r in range(2)]
    tag = "grad_sinks.%s.e%d." % (backend, engine)
    worst = 0.0
    for name, g0, g1, gf, r0, r1 in zip(model.names, halves[0], halves[1], full, ranks[0], ranks[1]):
        if g0 is None and g1 is None:
            continue
        mean = ((g0 + g1) * 0.5).cpu()
        for r, got in enumerate((r0, r1)):
            assert torch.equal(got, mean), "%s rank %d: differs from (g0 + g1) / 2 by %.3e" % (name, r, err_inf(got, mean))
        rel = err_inf(mean, gf) / scale_inf(gf)
        worst = max(worst, rel)
        report(tag + "vs_full_batch." + name, rel=rel)
        assert rel <= 1e-5, (name, rel)
    # measured worst on an H100 80GB HBM3 (700 W): 2.4e-6 on engine 0, 5.7e-7 on engine 1
    report(tag + "vs_full_batch.worst_rel", rel=worst)
