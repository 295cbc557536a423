"""Data-parallel plumbing for the ray-sharded renderer (SURVEY.md 8(e)): rays are independent, parameters are replicated,
so the only exchange per training step is the all-reduce of the parameter gradients (NCCL over NVLink/NVSwitch on the
GPU box; the same code runs on gloo/CPU tensors in the unit tests).  No kernels here.

GradBucket keeps ONE persistent flat fp32 buffer.  The networks whose backward passes are libnudf kernels (UDFNetwork,
ResidualRenderingNetwork, NeRF) get a *gradient sink*: their backward kernels write dg / dv / db straight into views of
the flat buffer and autograd adopts those views as `.grad` -- no pack / unpack copies, one collective per region.  A
region's all-reduce is issued asynchronously as soon as its backward kernels have been enqueued (the colour network's
gradients travel while the ~4 ms UDF backward still runs); `allreduce_mean()` reduces what is left and waits.
Parameters without a sink (the scalar heads) are packed into a small tail of the same buffer.

The kernels OVERWRITE their targets, so a backward invocation may only write the region when the region holds nothing
autograd still has to add to.  Otherwise (the network appears twice in one backward, two backward passes are accumulated,
or zero_grad(set_to_none=False) kept the `.grad` views) it writes fresh tensors and autograd adds them to what is there;
`allreduce_mean()` copies any gradient that does not live in its slot into it before reducing.
"""
import torch
import torch.distributed as dist


def shard_bounds(n_items, rank, world):
    """Contiguous split of n_items over `world` ranks (first ranks get the remainder): [lo, hi)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_rays(rays_o, rays_d, *more, rank=None, world=None):
    """This rank's contiguous slice of every per-ray tensor."""
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    lo, hi = shard_bounds(rays_o.shape[0], rank, world)
    return tuple(t[lo:hi] for t in (rays_o, rays_d) + more)


class _Reduced:
    """the collective handle of a region already reduced synchronously (every backend but NCCL): nothing to wait for"""

    @staticmethod
    def wait():
        return True


class _Region:
    """Contiguous slice [lo, hi) of the flat buffer holding all gradients of one kernel-backed network."""

    def __init__(self, bucket, lo):
        self.bucket, self.lo, self.hi = bucket, lo, lo
        self.offsets = {}            # id(param) -> (offset, shape)
        self.params = []
        self.work = None             # the region's collective once ready() issued it (overlap at world > 1)
        self.task = None             # the autograd graph task (one backward call) whose kernels last wrote the region

    def add(self, p):
        self.params.append(p)
        self.offsets[id(p)] = (self.hi, tuple(p.shape))
        self.hi += p.numel()

    def holds(self, p):
        """True if p.grad is the slot of p (the tensor view() hands out, adopted by autograd)"""
        flat = self.bucket.flat
        return p.grad is not None and p.grad.data_ptr() == flat.data_ptr() + self.offsets[id(p)][0] * flat.element_size()

    def block(self, params):
        """one contiguous view covering `params` (which were added consecutively), e.g. all biases of a network"""
        lo = self.offsets[id(params[0])][0]
        n = sum(p.numel() for p in params)
        return self.bucket.flat.narrow(0, lo, n)

    def view(self, p):
        """a FRESH view (own TensorImpl, so that autograd can adopt it as .grad without a copy)"""
        off, shape = self.offsets[id(p)]
        return self.bucket.flat.narrow(0, off, p.numel()).view(shape)

    def begin(self):
        """True if this backward invocation may write the region (its kernels overwrite it).  False when autograd has
        something to add the invocation's gradients to: the region was already written in this backward call (the
        network appears twice in the graph), or a parameter still holds a `.grad` (backward passes accumulated before
        allreduce_mean(), or zero_grad(set_to_none=False)), which may be a view of the region.  The invocation then
        writes fresh tensors and autograd sums them."""
        if self.work is not None:
            raise RuntimeError("GradBucket(overlap=True): a kernel-backed network ran backward again after its gradients "
                               "were handed to the collective (it appears twice in one backward, or backward passes are "
                               "accumulated before allreduce_mean()); construct the bucket with overlap=False")
        if self.task == torch._C._current_graph_task_id():
            return False
        return all(p.grad is None for p in self.params)

    def ready(self):
        """called by the backward wrapper once every kernel writing this region has been enqueued"""
        self.task = torch._C._current_graph_task_id()
        b = self.bucket
        if b.overlap and b.world() > 1:
            self.work = b._reduce(b.flat.narrow(0, self.lo, self.hi - self.lo), async_op=True)


class GradBucket:
    """Flat fp32 gradient bucket over the trainable parameters.

    GradBucket(params)                      plain mode (any tensors, any device): pack -> one all-reduce -> unpack
    GradBucket(params, modules=[udf, ...])  modules with a libnudf handle write their gradients in place (see above)
    `allreduce_mean()` leaves the mean over ranks in every `.grad` (DDP semantics: mean of the per-shard losses)."""

    def __init__(self, params, modules=(), overlap=True, group=None):
        self.params = [p for p in params if p.requires_grad]
        self.group = group
        self.overlap = overlap
        dev = self.params[0].device if self.params else torch.device("cpu")
        self.regions = []
        covered = set()
        total = 0
        for m in modules:
            h = getattr(m, "_handle", None)
            if h is None or not hasattr(h, "sink_layout"):
                continue
            groups = [[p for p in g if p.requires_grad] for g in h.sink_layout()]
            if not any(groups) or any(not p.requires_grad for g in h.sink_layout() for p in g):
                continue                       # partially frozen network: keep the plain path
            r = _Region(self, total)
            for g in groups:
                for p in g:
                    r.add(p)
                    covered.add(id(p))
            total = r.hi
            self.regions.append(r)
            h.grad_sink = r
        self.loose = [p for p in self.params if id(p) not in covered]
        self.loose_lo = total
        total += sum(p.numel() for p in self.loose)
        self.flat = torch.zeros(max(total, 1), dtype=torch.float32, device=dev)

    def world(self):
        return dist.get_world_size(self.group) if dist.is_available() and dist.is_initialized() else 1

    def _reduce(self, t, async_op=False):
        """mean over ranks, in place; with async_op a handle to wait() on (other backends than NCCL reduce at once)"""
        if dist.get_backend(self.group) == "nccl":
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group, async_op=False)
        t.mul_(1.0 / self.world())
        return _Reduced() if async_op else None

    def allreduce_replayed(self):
        """All-reduce after a CUDA-graph REPLAY of forward + backward: the kernels have written every region of the flat
        buffer, but the Python bookkeeping of the sinks (begin() / ready()) did not run, so nothing is in flight and nothing
        may be zeroed.  Packs the loose tail, ONE collective over the whole buffer, unpacks the tail.  (NCCL calls are kept
        out of captured graphs on purpose: the capture then holds only this library's and torch's kernels.)"""
        if self.world() == 1:
            return
        off = self.loose_lo
        for p in self.loose:
            n = p.numel()
            if p.grad is None:
                self.flat.narrow(0, off, n).zero_()
            else:
                self.flat.narrow(0, off, n).copy_(p.grad.reshape(-1))
            off += n
        self._reduce(self.flat)
        off = self.loose_lo
        for p in self.loose:
            n = p.numel()
            if p.grad is not None:
                p.grad.copy_(self.flat.narrow(0, off, n).view_as(p))
            off += n

    def allreduce_mean(self, group=None):
        """Afterwards every sinked parameter's `.grad` is its slot of `flat` (at world 1: every one that has a gradient)."""
        if group is not None:
            self.group = group
        world = self.world()
        for r in self.regions:
            if r.work is not None:
                continue                             # in the collective already: the gradients are the slots
            for p in r.params:
                if p.grad is None:
                    if world > 1:
                        r.view(p).zero_()            # e.g. a network outside this step's graph: it adds zero to the mean
                elif not r.holds(p):
                    r.view(p).copy_(p.grad)          # summed by autograd from fresh tensors (see _Region.begin)
        if world > 1:
            off = self.loose_lo
            for p in self.loose:
                n = p.numel()
                if p.grad is None:
                    self.flat.narrow(0, off, n).zero_()
                else:
                    self.flat.narrow(0, off, n).copy_(p.grad.reshape(-1))
                off += n
            works = [r.work for r in self.regions if r.work is not None]
            if not works:
                self._reduce(self.flat)                          # nothing in flight: one collective for everything
            else:                                                # each element enters one collective
                for r in self.regions:
                    if r.work is None:
                        self._reduce(self.flat.narrow(0, r.lo, r.hi - r.lo))
                if self.loose:
                    self._reduce(self.flat.narrow(0, self.loose_lo, self.flat.numel() - self.loose_lo))
                for w in works:
                    w.wait()
        for r in self.regions:
            for p in r.params:
                if (p.grad is not None or world > 1) and not r.holds(p):
                    p.grad = r.view(p)
            r.work, r.task = None, None
        if world == 1:
            return
        off = self.loose_lo
        for p in self.loose:
            n = p.numel()
            g = self.flat.narrow(0, off, n).view_as(p)
            if p.grad is None:
                p.grad = g.clone()
            else:
                p.grad.copy_(g)
            off += n
