"""N>1 host logic on CPU: world_size-2 gloo processes shard a batch of views and
all-gather per-view gradients; the gathered result must equal the unsharded one
(SURVEY.md §8e: "sharded result == single-GPU result")."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from kaolin_b200.multi_gpu import (pipelined_backward_all_gather, shard_range, shard_views, all_gather_view_grads, chunk_ranges,
                                   ChunkedGradAllGather, OverlappedGradAllGather)


def _fake_grads(batch, faces):
    g = torch.arange(batch * faces * 6, dtype=torch.float32).reshape(batch, faces, 3, 2)
    f = torch.arange(batch * faces * 9, dtype=torch.float32).reshape(batch, faces, 3, 3) * 0.5
    return g, f


def _worker(rank, world, batch, port, ok):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g, f = _fake_grads(batch, 7)
        lg, lf = shard_views([g, f], rank, world)
        full_g, full_f = all_gather_view_grads([lg.clone(), lf.clone()], batch)
        ok[rank] = int(torch.equal(full_g, g) and torch.equal(full_f, f))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("batch", [4, 5])
def test_two_rank_gloo_gather(batch):
    ok = mp.get_context("spawn").Array("i", [0, 0])
    port = 29500 + (os.getpid() % 2000) + batch
    mp.spawn(_worker, args=(2, batch, port, ok), nprocs=2, join=True)
    assert list(ok) == [1, 1]


def test_shard_ranges_partition_the_batch():
    for batch in (1, 7, 8, 256):
        for world in (1, 2, 3, 8):
            spans = [shard_range(batch, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == batch
            assert all(spans[i][1] == spans[i + 1][0] for i in range(world - 1))
            sizes = [e - s for s, e in spans]
            assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        shard_range(4, 2, 2)


def _chunk_worker(rank, world, batch, chunks, port, ok):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g, f = _fake_grads(batch, 5)
        lg, lf = shard_views([g, f], rank, world)
        gather = ChunkedGradAllGather(lg.shape[0])
        for c0, c1 in chunk_ranges(lg.shape[0], chunks):
            gather.submit(c0, c1, [lg[c0:c1].clone(), lf[c0:c1].clone()])
        full_g, full_f = gather.finish()
        ref_g, ref_f = all_gather_view_grads([lg.clone(), lf.clone()], batch)
        ok[rank] = int(torch.equal(full_g, g) and torch.equal(full_f, f)
                       and torch.equal(full_g, ref_g) and torch.equal(full_f, ref_f))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("batch,chunks", [(8, 4), (6, 2), (4, 8)])
def test_two_rank_gloo_chunked_gather_equals_single_gather(batch, chunks):
    ok = mp.get_context("spawn").Array("i", [0, 0])
    port = 31500 + (os.getpid() % 2000) + batch * 8 + chunks
    mp.spawn(_chunk_worker, args=(2, batch, chunks, port, ok), nprocs=2, join=True)
    assert list(ok) == [1, 1]


def test_chunk_ranges_cover_the_views():
    for views in (1, 5, 32):
        for chunks in (1, 3, 4, 64):
            spans = chunk_ranges(views, chunks)
            assert spans[0][0] == 0 and spans[-1][1] == views and len(spans) == min(chunks, views)
            assert all(e > s for s, e in spans)
            assert all(spans[i][1] == spans[i + 1][0] for i in range(len(spans) - 1))


def _overlap_worker(rank, world, batch, port, ok):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g, f = _fake_grads(batch, 5)
        lg, lf = shard_views([g, f], rank, world)
        gather = OverlappedGradAllGather(batch)
        gather.hook(lf.clone())                      # what the fused backward does between its branches
        full_g, full_f = gather.finish(lg.clone())
        # the hook never ran: the feature gradient is gathered in finish()
        gather2 = OverlappedGradAllGather(batch)
        full_g2, full_f2 = gather2.finish(lg.clone(), lf.clone())
        # attach() refuses tensors that are not outputs of dibr_rasterization
        try:
            OverlappedGradAllGather(batch).attach(torch.zeros(3, requires_grad=True) * 2)
            attached = True
        except ValueError:
            attached = False
        assert not attached
        ok[rank] = int(torch.equal(full_g, g) and torch.equal(full_f, f)
                       and torch.equal(full_g2, g) and torch.equal(full_f2, f))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_overlapped_gather():
    ok = mp.get_context("spawn").Array("i", [0, 0])
    port = 33500 + (os.getpid() % 2000)
    mp.spawn(_overlap_worker, args=(2, 6, port, ok), nprocs=2, join=True)
    assert list(ok) == [1, 1]


def _factory_worker(rank, world, batch, port, ok):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from kaolin_b200.multi_gpu import make_grad_all_gather, PeerGradAllGather
        g, f = _fake_grads(batch, 5)
        lg, lf = shard_views([g, f], rank, world)
        # on CPU tensors "auto" agrees (collectively) on the NCCL-style gather; asked twice: cached decision
        for _ in range(2):
            gather, used = make_grad_all_gather(batch, lg.shape, lf.shape, "cpu", transport="auto")
            gather.hook(lf.clone())
            full_g, full_f = gather.finish(lg.clone())
            good = used == "nccl" and torch.equal(full_g, g) and torch.equal(full_f, f)
        # an explicit peer transport without symmetric memory is an error, not a silent fallback
        try:
            PeerGradAllGather(batch, lg.shape, lf.shape, "cpu")
            raised = False
        except Exception:
            raised = True
        try:
            make_grad_all_gather(batch, lg.shape, lf.shape, "cpu", transport="carrier pigeon")
            bad = False
        except ValueError:
            bad = True
        ok[rank] = int(good and raised and bad)
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_gather_factory_falls_back_collectively():
    ok = mp.get_context("spawn").Array("i", [0, 0])
    port = 35500 + (os.getpid() % 2000)
    mp.spawn(_factory_worker, args=(2, 6, port, ok), nprocs=2, join=True)
    assert list(ok) == [1, 1]


def _pipelined_worker(rank, world, batch, chunks, port, ok):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g, f = _fake_grads(batch, 5)
        lg, lf = shard_views([g, f], rank, world)
        n = lg.shape[0]
        g_fvi, g_ff = torch.zeros_like(lg), torch.zeros_like(lf)
        order = []

        def run_chunk(c0, c1, hook):            # what _host.backward(views=(c0, c1), out=..., feature_grad_hook=hook) does
            g_ff[c0:c1] = lf[c0:c1]; order.append(("ff", c0)); hook(g_ff)
            g_fvi[c0:c1] = lg[c0:c1]; order.append(("fvi", c0))
        full_g, full_f = pipelined_backward_all_gather(n, chunks, run_chunk, g_fvi, g_ff)
        ok[rank] = int(torch.equal(full_g, g) and torch.equal(full_f, f) and len(order) == 2 * min(chunks, n))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("batch,chunks", [(8, 2), (6, 3), (4, 1)])
def test_two_rank_gloo_pipelined_backward_gather(batch, chunks):
    ok = mp.get_context("spawn").Array("i", [0, 0])
    port = 35500 + (os.getpid() % 2000) + batch * 8 + chunks
    mp.spawn(_pipelined_worker, args=(2, batch, chunks, port, ok), nprocs=2, join=True)
    assert list(ok) == [1, 1]


def test_attach_finds_the_dibr_node_through_a_slice():
    """attach() walks from an output (or a slice of it: list/tuple face_features) to the autograd node of the
    dibr_rasterization call, recognised by its class name, and stores the hook on THAT node only."""
    from kaolin_b200 import multi_gpu

    class DibrRasterizationB200(torch.autograd.Function):     # stands in for render/mesh/dibr.py's node on CPU
        @staticmethod
        def forward(ctx, x):
            return x * 2.0

        @staticmethod
        def backward(ctx, g):
            return g * 2.0

    x = torch.ones(4, 3, requires_grad=True)
    out = DibrRasterizationB200.apply(x)
    node = multi_gpu._dibr_node(out[..., :2])
    assert node is out.grad_fn
    other = DibrRasterizationB200.apply(x)
    g = object.__new__(multi_gpu.OverlappedGradAllGather)      # no process group needed for attach()
    g.hook = lambda t: None
    assert g.attach(out) is g
    assert out.grad_fn.feature_grad_hook is g.hook and not hasattr(other.grad_fn, "feature_grad_hook")
    with pytest.raises(ValueError):
        multi_gpu._dibr_node(x * 3.0)
    with pytest.raises(ValueError):
        multi_gpu._dibr_node(torch.ones(3))
