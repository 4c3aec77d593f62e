"""Batch (view) sharding of the DIB-R path across the GPUs of one box.

Every view is independent in all four kernels (rasterization_cuda.cu:71-72,
dibr_soft_mask_cuda.cu:83; SURVEY.md §8e), so the forward needs no
communication: rank r renders views [start, stop).  The only exchange is an
all-gather of the per-view gradients after backward
(``torch.distributed.all_gather_into_tensor`` — NCCL over NVLink on GPUs, gloo in
the CPU tests).  One process per GPU; nothing here touches the kernels.

``ChunkedGradAllGather`` hides that exchange behind the compute: the rank's views
are rendered in a few view-chunks, and the gradients of chunk i travel (async
collective on the process group's own stream) while chunk i+1 is rasterized, so
only the last chunk's transfer is exposed (SURVEY.md §8e "chunked backward").
"""
import torch
import torch.distributed as dist

__all__ = ["shard_range", "shard_views", "all_gather_view_grads", "chunk_ranges",
           "ChunkedGradAllGather", "OverlappedGradAllGather", "pipelined_backward_all_gather",
           "PipelinedGradAllGather", "PeerGradAllGather", "make_grad_all_gather"]


def shard_range(batch, rank, world_size):
    """Contiguous shard [start, stop) of `batch` views for `rank`; the first
    ``batch % world_size`` ranks get one extra view."""
    if not (0 <= rank < world_size):
        raise ValueError(f"rank {rank} outside world of size {world_size}")
    base, extra = divmod(batch, world_size)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def shard_views(tensors, rank, world_size):
    """Slices the leading (view) dimension of every tensor for this rank."""
    out = []
    for t in tensors:
        s, e = shard_range(t.shape[0], rank, world_size)
        out.append(t[s:e])
    return out


def all_gather_view_grads(local_grads, batch, group=None):
    """All-gathers per-view gradient tensors (leading dim = local views) into
    full-batch tensors on every rank.  Equal shards use one
    ``all_gather_into_tensor`` per tensor; ragged shards are padded to the
    largest shard and trimmed."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_range(batch, r, world)[1] - shard_range(batch, r, world)[0] for r in range(world)]
    outs = []
    for g in local_grads:
        if g.shape[0] != sizes[rank]:
            raise ValueError(f"local gradient has {g.shape[0]} views, shard owns {sizes[rank]}")
        g = g.contiguous()
        if len(set(sizes)) == 1:
            full = torch.empty((batch,) + tuple(g.shape[1:]), dtype=g.dtype, device=g.device)
            dist.all_gather_into_tensor(full, g, group=group)
        else:
            m = max(sizes)
            pad = torch.zeros((m,) + tuple(g.shape[1:]), dtype=g.dtype, device=g.device)
            pad[:g.shape[0]] = g
            buf = torch.empty((world * m,) + tuple(g.shape[1:]), dtype=g.dtype, device=g.device)
            dist.all_gather_into_tensor(buf, pad, group=group)
            full = torch.cat([buf[r * m:r * m + sizes[r]] for r in range(world)], 0)
        outs.append(full)
    return outs


def chunk_ranges(views, chunks):
    """Splits `views` local views into at most `chunks` contiguous [start, stop) pieces."""
    chunks = max(1, min(int(chunks), views))
    return [shard_range(views, c, chunks) for c in range(chunks)]


class ChunkedGradAllGather:
    """All-gather of per-view gradients, one view-chunk at a time, overlapped with compute.

    Every rank owns ``local_views`` views (equal shards).  After the backward of
    local views [c0, c1) call ``submit(c0, c1, [g_fvi_chunk, g_ff_chunk, ...])``: an
    asynchronous all-gather of that chunk starts and the caller goes on with the
    next chunk.  ``finish()`` makes the current stream wait for all of them and
    returns the full tensors, rank-major: entry ``r * local_views + v`` is view v of
    rank r - the layout ``all_gather_view_grads`` produces in one call.
    """

    def __init__(self, local_views, group=None):
        self.group = group
        self.world = dist.get_world_size(group)
        self.local_views = int(local_views)
        self.full = None
        self.pending = []

    def submit(self, c0, c1, grads):
        if not (0 <= c0 < c1 <= self.local_views):
            raise ValueError(f"chunk [{c0}, {c1}) outside the {self.local_views} local views")
        grads = [g.contiguous() for g in grads]
        for g in grads:
            if g.shape[0] != c1 - c0:
                raise ValueError(f"chunk gradient has {g.shape[0]} views, chunk [{c0}, {c1}) has {c1 - c0}")
        if self.full is None:
            self.full = [torch.empty((self.world, self.local_views) + tuple(g.shape[1:]),
                                     dtype=g.dtype, device=g.device) for g in grads]
        for full, g in zip(self.full, grads):
            # one contiguous landing buffer per chunk; copied to its rank-major place in finish()
            buf = torch.empty((self.world * (c1 - c0),) + tuple(g.shape[1:]), dtype=g.dtype, device=g.device)
            work = dist.all_gather_into_tensor(buf, g, group=self.group, async_op=True)
            self.pending.append((work, full, buf, c0, c1, g))

    def finish(self):
        if self.full is None:
            raise RuntimeError("ChunkedGradAllGather.finish() before any submit()")
        for work, full, buf, c0, c1, _ in self.pending:
            work.wait()                       # the current stream waits; the host does not block on CUDA
            full[:, c0:c1].copy_(buf.view((self.world, c1 - c0) + tuple(buf.shape[1:])))
        self.pending = []
        out = [f.reshape((self.world * self.local_views,) + tuple(f.shape[2:])) for f in self.full]
        self.full = None
        return out


class OverlappedGradAllGather:
    """All-gather of the two DIB-R gradients with most of the transfer hidden behind the
    backward itself: ``grad_face_features`` (60 % of the bytes at D = 3) is final as soon
    as the rasterize branch of the fused backward has run, so its all-gather is started
    there (asynchronously, on the process group's stream) and travels while the soft-mask
    branch computes; ``grad_face_vertices_image`` follows at the end.

        feat, soft_mask, face_idx = dibr_rasterization(...)
        gather = OverlappedGradAllGather(batch).attach(soft_mask)     # this node only
        torch.autograd.backward([feat, soft_mask], [g_feat, g_mask])
        full_g_fvi, full_g_ff = gather.finish(face_vertices_image.grad)

    The hook is per call: ``attach`` stores it on the autograd node of that one
    ``dibr_rasterization`` call (other DIB-R backward passes, on this or another device
    or thread, are not affected); through the C-ABI path pass ``gather.hook`` as
    ``_host.backward(..., feature_grad_hook=gather.hook)``.  ``finish`` waits for the
    asynchronous gather, so the local gradient buffer is not touched by NCCL after it
    returns.  Equal shards only (``batch`` = world size x local views).
    """

    def __init__(self, batch, group=None):
        self.group = group
        self.world = dist.get_world_size(group)
        if batch % self.world:
            raise ValueError(f"batch {batch} is not divisible by the world size {self.world}")
        self.batch = int(batch)
        self.work = None
        self.full_ff = None
        self.local_ff = None

    def hook(self, g_ff):
        """Called by the fused backward between its two branches with the final fp32
        ``grad_face_features`` of the local views."""
        if self.work is not None:
            raise RuntimeError("OverlappedGradAllGather covers one backward call")
        if g_ff.shape[0] * self.world != self.batch:
            raise ValueError(f"local gradient has {g_ff.shape[0]} views, expected {self.batch // self.world}")
        self.local_ff = g_ff          # kept alive until finish(): NCCL reads it asynchronously
        self.full_ff = torch.empty((self.batch,) + tuple(g_ff.shape[1:]), dtype=g_ff.dtype, device=g_ff.device)
        self.work = dist.all_gather_into_tensor(self.full_ff, g_ff, group=self.group, async_op=True)

    def attach(self, output):
        """Registers the hook on the autograd node that produced ``output`` (the soft mask
        or the features of ONE ``dibr_rasterization`` call).  Returns self."""
        _dibr_node(output).feature_grad_hook = self.hook
        return self

    def finish(self, g_fvi, g_ff=None):
        """Gathers ``g_fvi`` and returns (full_g_fvi, full_g_ff).  If the backward did not go
        through the hook (e.g. only one of the two output gradients was given), pass the
        local ``g_ff`` and it is gathered here."""
        full_fvi = all_gather_view_grads([g_fvi], self.batch, self.group)[0]
        if self.work is not None:
            self.work.wait()
            full_ff = self.full_ff
        elif g_ff is not None:
            full_ff = all_gather_view_grads([g_ff], self.batch, self.group)[0]
        else:
            raise RuntimeError("no feature gradient was produced by the attached backward and none was passed")
        self.work = self.full_ff = self.local_ff = None
        return full_fvi, full_ff


def pipelined_backward_all_gather(local_views, chunks, run_chunk, g_fvi, g_ff, group=None):
    """Backward in view chunks with the gradient exchange of chunk i hidden behind chunk i+1.

    ``run_chunk(c0, c1, hook)`` must issue the backward of the local views [c0, c1) writing rows
    c0..c1-1 of the full local buffers ``g_fvi`` / ``g_ff`` (``_host.backward(..., views=(c0, c1),
    out=(g_fvi, g_ff), feature_grad_hook=hook)`` = ``dibr_b200_backward_views``) and call ``hook``
    once ``g_ff[c0:c1]`` is final (after the rasterize branch).  The all-gathers (asynchronous, on the
    process group's stream) of a chunk's ``grad_face_features`` start at its hook, those of its
    ``grad_face_vertices_image`` when the chunk is done; only the last chunk's
    ``grad_face_vertices_image`` is exposed.  Returns (full_g_fvi, full_g_ff), rank-major like
    ``all_gather_view_grads``; the current stream waits for the exchange before they are used.
    """
    world = dist.get_world_size(group)
    full_fvi = torch.empty((world, local_views) + tuple(g_fvi.shape[1:]), dtype=g_fvi.dtype, device=g_fvi.device)
    full_ff = torch.empty((world, local_views) + tuple(g_ff.shape[1:]), dtype=g_ff.dtype, device=g_ff.device)
    works = []
    for c0, c1 in chunk_ranges(local_views, chunks):
        def hook(_g_ff=None, c0=c0, c1=c1):
            works.append(dist.all_gather([full_ff[r, c0:c1] for r in range(world)], g_ff[c0:c1].contiguous(),
                                         group=group, async_op=True))
        run_chunk(c0, c1, hook)
        works.append(dist.all_gather([full_fvi[r, c0:c1] for r in range(world)], g_fvi[c0:c1].contiguous(),
                                     group=group, async_op=True))
    for w in works:
        w.wait()
    return (full_fvi.reshape((world * local_views,) + tuple(g_fvi.shape[1:])),
            full_ff.reshape((world * local_views,) + tuple(g_ff.shape[1:])))


class PipelinedGradAllGather:
    """``pipelined_backward_all_gather`` for the public API: attached to ONE ``dibr_rasterization`` call,
    it makes that call's autograd backward run in ``chunks`` view chunks (``dibr_b200_backward_views``)
    whose gradients are exchanged while the next chunk computes.

        feat, soft_mask, face_idx = dibr_rasterization(...)
        gather = PipelinedGradAllGather(chunks=2).attach(soft_mask)
        torch.autograd.backward([feat, soft_mask], [g_feat, g_mask])
        full_g_fvi, full_g_ff = gather.finish()       # rank-major, (world * local_views, F, 3, .)

    Equal shards only.  The local ``.grad`` tensors are produced as usual."""

    def __init__(self, chunks=2, group=None):
        self.chunks = int(chunks)
        self.group = group
        self.result = None

    def _run(self, local_views, run_chunk, g_fvi, g_ff):
        self.result = pipelined_backward_all_gather(local_views, self.chunks, run_chunk, g_fvi, g_ff, self.group)

    def attach(self, output):
        _dibr_node(output).view_pipeline = self._run
        return self

    def finish(self):
        if self.result is None:
            raise RuntimeError("the attached backward has not run (both output gradients are needed)")
        out, self.result = self.result, None
        return out


# ---------------------------------------------------------------------------
# All-gather by stores into peer memory (NVLink / NVSwitch)
class _PeerPool:
    """Symmetric landing buffers of one (group, gradient shapes) configuration, mapped into every
    rank of the box (``torch.distributed._symmetric_memory``: CUDA VMM allocations exchanged
    between the processes; ``buffer_ptrs[r]`` is rank r's buffer as a pointer valid HERE), two
    generations of them, plus the side streams the pushes run on.  Created once (the rendezvous is
    a collective and costs milliseconds) and reused by every step."""

    def __init__(self, group, device, local_views, shape_fvi, shape_ff, dtype, n_streams):
        import torch.distributed._symmetric_memory as symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.device = device
        self.local_views = local_views
        self.shapes = {"fvi": (local_views,) + tuple(shape_fvi), "ff": (local_views,) + tuple(shape_ff)}
        self.dtype = dtype
        esz = torch.empty((), dtype=dtype).element_size()
        self.numel = {k: int(torch.Size(v).numel()) for k, v in self.shapes.items()}
        for k, n in self.numel.items():
            if (n * esz) % 16:
                raise ValueError(f"PeerGradAllGather: the {k} shard is {n * esz} bytes, not a multiple of 16")
        # layout of one generation: [world][fvi shard] then [world][ff shard]; two generations
        self.off = {"fvi": 0, "ff": self.world * self.numel["fvi"]}
        self.gen_numel = self.world * (self.numel["fvi"] + self.numel["ff"])
        self.buf = symm_mem.empty(2 * self.gen_numel, dtype=dtype, device=device)
        self.hdl = symm_mem.rendezvous(self.buf, self.group)
        self.ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        self.ptr_array = None
        try:
            self.multicast_ptr = int(self.hdl.multicast_ptr)     # 0 when the box has no NVSwitch multicast
        except Exception:
            self.multicast_ptr = 0
        self.esz = esz
        self.streams = [torch.cuda.Stream(device, priority=-1) for _ in range(max(1, int(n_streams)))]
        self.generation = 0
        self._views = {}

    def landing(self, owner, gen, kind, src_rank=None):
        """Tensor view of rank `owner`'s landing area for `kind`: all ranks' slots, or `src_rank`'s."""
        key = (owner, gen, kind, src_rank)
        v = self._views.get(key)
        if v is None:
            n = self.numel[kind]
            off = gen * self.gen_numel + self.off[kind]
            if src_rank is None:
                v = self.hdl.get_buffer(owner, (self.world,) + self.shapes[kind], self.dtype, off)
            else:
                v = self.hdl.get_buffer(owner, self.shapes[kind], self.dtype, off + src_rank * n)
            self._views[key] = v
        return v

    def byte_offset(self, gen, kind, src_rank):
        return (gen * self.gen_numel + self.off[kind] + src_rank * self.numel[kind]) * self.esz


_peer_pools = {}


class PeerGradAllGather:
    """``OverlappedGradAllGather`` with the transfer done by STORES into the peers' memory over
    NVLink instead of an NCCL collective: every rank pushes its ``grad_face_features`` shard into
    slot `rank` of every peer's landing buffer as soon as the rasterize branch of the backward has
    produced it (``hook``), and its ``grad_face_vertices_image`` shard at the end (``finish``).

    ``engine="ce"``: one peer-to-peer ``copy_`` per destination on high-priority side streams - the
    copy engines move the bytes, no SM is taken from the soft-mask branch that runs meanwhile.
    ``engine="sm"``: ``dibr_b200_peer_push`` (csrc/peer_push.cu), one small kernel that loads each 16 B
    of the shard once and stores it to all destinations.  ``engine="mc"``:
    ``dibr_b200_peer_push_multicast``, one ``multimem.st`` per 16 B to the NVSwitch multicast mapping of
    the landing buffer - the switch replicates it to every GPU, so a rank's egress is its shard once.

    Cross-rank ordering: ``finish`` ends with the symmetric-memory barrier on the side stream (every
    rank's pushes are complete when it passes) and makes the current stream wait for it.  The
    landing buffers are persistent and double-buffered: the tensors returned by ``finish`` stay
    valid until the ``finish`` after the next one, provided they are consumed on the current stream
    (a rank starts pushing generation g+2 only after its own consumer of generation g, which
    precedes its next backward in stream order, and after every rank passed barrier g+1).
    One gather per (group, gradient shapes) is in flight at a time (``finish`` it before the next
    backward pushes).  Same interface as ``OverlappedGradAllGather`` (``hook`` / ``attach`` /
    ``finish``); equal shards, one box.  Raises at construction when symmetric memory is unavailable
    (``make_grad_all_gather`` falls back to NCCL)."""

    BARRIER_TIMEOUT_MS = 120000     # a rank that never arrives traps the barrier kernel instead of hanging the box

    def __init__(self, batch, local_fvi_shape, local_ff_shape, device, dtype=torch.float32, group=None,
                 engine="ce", streams=4, ctas=32):
        self.world = dist.get_world_size(group)
        if batch % self.world:
            raise ValueError(f"batch {batch} is not divisible by the world size {self.world}")
        if engine not in ("ce", "sm", "mc"):
            raise ValueError("engine must be 'ce', 'sm' or 'mc'")
        self.batch = int(batch)
        self.engine = engine
        self.ctas = int(ctas)
        lv = self.batch // self.world
        key = (id(group), str(device), lv, tuple(local_fvi_shape), tuple(local_ff_shape), dtype)
        pool = _peer_pools.get(key)
        if pool is None:
            pool = _PeerPool(group, device, lv, tuple(local_fvi_shape)[1:], tuple(local_ff_shape)[1:], dtype, streams)
            _peer_pools[key] = pool
        if engine == "mc" and not pool.multicast_ptr:
            raise RuntimeError("PeerGradAllGather: no NVSwitch multicast mapping for the landing buffer on this system")
        self.pool = pool
        self.gen = None          # taken at the first push: an object that is created and dropped uses no generation
        self.keep = []
        self.pushed_ff = False

    def _push(self, kind, local):
        pool = self.pool
        if tuple(local.shape) != pool.shapes[kind] or local.dtype != pool.dtype:
            raise ValueError(f"PeerGradAllGather: {kind} shard is {tuple(local.shape)} {local.dtype}, "
                             f"expected {pool.shapes[kind]} {pool.dtype}")
        if self.gen is None:
            self.gen = pool.generation
            pool.generation ^= 1
        local = local.contiguous()
        self.keep.append(local)               # alive until finish(): the side streams read it
        dev = pool.device
        ready = torch.cuda.Event()
        ready.record(torch.cuda.current_stream(dev))
        order = [(pool.rank + 1 + k) % pool.world for k in range(pool.world)]     # self last, peers rotated
        if self.engine in ("sm", "mc"):
            import ctypes
            from . import _lib
            s = pool.streams[0]
            s.wait_event(ready)
            off = pool.byte_offset(self.gen, kind, pool.rank)
            if self.engine == "mc":
                _lib.call("dibr_b200_peer_push_multicast", dev, local, local.numel() * pool.esz, pool.multicast_ptr,
                          off, self.ctas, stream=s)
                return
            if pool.ptr_array is None:
                pool.ptr_array = (ctypes.c_void_p * pool.world)(*[pool.ptrs[r] for r in order])
            _lib.call("dibr_b200_peer_push", dev, local, local.numel() * pool.esz, pool.ptr_array, pool.world, off,
                      self.ctas, stream=s)
            return
        for i, r in enumerate(order):
            s = pool.streams[i % len(pool.streams)]
            s.wait_event(ready)
            with torch.cuda.stream(s):
                pool.landing(r, self.gen, kind, pool.rank).copy_(local, non_blocking=True)

    def hook(self, g_ff):
        if self.pushed_ff:
            raise RuntimeError("PeerGradAllGather covers one backward call")
        self._push("ff", g_ff)
        self.pushed_ff = True

    def attach(self, output):
        _dibr_node(output).feature_grad_hook = self.hook
        return self

    def finish(self, g_fvi, g_ff=None):
        pool = self.pool
        if not self.pushed_ff:
            if g_ff is None:
                raise RuntimeError("no feature gradient was produced by the attached backward and none was passed")
            self._push("ff", g_ff)
        self._push("fvi", g_fvi)
        s0 = pool.streams[0]
        for s in (pool.streams[1:] if self.engine == "ce" else ()):
            e = torch.cuda.Event(); e.record(s); s0.wait_event(e)
        with torch.cuda.stream(s0):
            pool.hdl.barrier(channel=self.gen, timeout_ms=self.BARRIER_TIMEOUT_MS)
        done = torch.cuda.Event(); done.record(s0)
        torch.cuda.current_stream(pool.device).wait_event(done)
        self.keep = []
        full_fvi = pool.landing(pool.rank, self.gen, "fvi").reshape((self.batch,) + pool.shapes["fvi"][1:])
        full_ff = pool.landing(pool.rank, self.gen, "ff").reshape((self.batch,) + pool.shapes["ff"][1:])
        return full_fvi, full_ff


_DIBR_NODE = "DibrRasterizationB200"     # render/mesh/dibr.py: the node of every dtype


def _dibr_node(output):
    """The autograd node of the ``dibr_rasterization`` call (fp32 or float64) that produced ``output``."""
    is_dibr = lambda n: type(n).__name__.startswith(_DIBR_NODE)
    node = getattr(output, "grad_fn", None)
    seen = 0
    while node is not None and not is_dibr(node) and seen < 4:
        # e.g. a slice of the feature image (list/tuple face_features): step to its producer
        nxt = [fn for fn, _ in node.next_functions if fn is not None]
        node = nxt[0] if len(nxt) == 1 else None
        seen += 1
    if node is None or not is_dibr(node):
        raise ValueError("attach() needs an output of kaolin_b200.render.mesh.dibr_rasterization "
                         "that requires grad")
    return node


def make_grad_all_gather(batch, local_fvi_shape, local_ff_shape, device, transport="auto", group=None, **kw):
    """-> (gather, transport used).  ``transport``: "peer" / "peer_sm" / "peer_mc" (``PeerGradAllGather``
    with the copy-engine, store-kernel or multicast-store engine; raises if symmetric memory cannot be
    set up), "nccl" (``OverlappedGradAllGather``) or "auto" (the best peer engine every rank can set
    up, else nccl - decided collectively so that all ranks take the same path)."""
    if transport == "nccl":
        return OverlappedGradAllGather(batch, group), "nccl"
    engines = {"peer": "ce", "peer_sm": "sm", "peer_mc": "mc"}
    if transport in engines:
        return PeerGradAllGather(batch, local_fvi_shape, local_ff_shape, device, group=group,
                                 engine=engines[transport], **kw), transport
    if transport != "auto":
        raise ValueError(f"unknown transport {transport!r}")
    state = _auto_state.get(id(group))
    if state is None:
        # every rank reports what it can do: 2 = multicast stores, 1 = unicast stores, 0 = NCCL only;
        # the minimum over the ranks is what all of them use
        level = 0
        if torch.device(device).type == "cuda":
            try:
                g = PeerGradAllGather(batch, local_fvi_shape, local_ff_shape, device, group=group, engine="sm", **kw)
                level = 2 if (g.pool.multicast_ptr and AUTO_ALLOWS_MULTICAST) else 1
            except Exception as exc:          # no symmetric memory on this system / in this container
                _auto_state[("why", id(group))] = f"{type(exc).__name__}: {exc}"
        flag = torch.tensor([level], dtype=torch.int32, device=device if torch.device(device).type == "cuda" else "cpu")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        state = _auto_state[id(group)] = ("nccl", "peer_sm", "peer_mc")[int(flag.item())]
    if state == "nccl":
        return OverlappedGradAllGather(batch, group), "nccl"
    return PeerGradAllGather(batch, local_fvi_shape, local_ff_shape, device, group=group, engine=engines[state], **kw), state


# "auto" prefers the multicast engine: one store per 16 B, replicated by the NVSwitch, where the unicast
# engines send the shard once per peer
AUTO_ALLOWS_MULTICAST = True
_auto_state = {}
