"""CPU, world_size 2, gloo: the data-parallel host logic (flat gradient arena + ONE SUM all-reduce per step) reproduces
the reference's DDP arithmetic -- loss*WORLD_SIZE followed by gradient averaging -- and keeps the replicas identical."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _net():
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.BatchNorm2d(8), torch.nn.SiLU(),
                               torch.nn.Conv2d(8, 4, 1))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from efficientteacher_b200.parallel import BnBufferSync, GradArena
    net = _net()
    # backward-completion order, like the trainer builds it
    arena = GradArena(net.parameters(), reverse=True)
    assert arena.params[0] is net[3].bias and arena.params[-1] is net[0].weight
    sync = BnBufferSync(net)
    assert net[1].running_mean.data_ptr() == sync.flat.data_ptr() and "running_var" in dict(net[1].named_buffers())
    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, nesterov=True)
    g = torch.Generator().manual_seed(10 + rank)          # per-rank shard, like init_seeds(1+RANK)
    for step in range(3):
        x = torch.randn(4, 3, 8, 8, generator=g)
        loss = net(x).square().mean()                       # per-rank mean loss, NOT multiplied by WORLD_SIZE
        loss.backward()
        assert arena.check_views()
        arena.all_reduce_sum(world)
        opt.step()
        arena.zero()
        # DDP broadcast_buffers=True: before the next forward every rank holds rank 0's running statistics
        mine = sync.flat.clone()
        sync.broadcast(world)
        both = [torch.zeros_like(sync.flat) for _ in range(world)]
        dist.all_gather(both, sync.flat)
        assert torch.equal(both[0], both[1]) and (rank == 0 or not torch.equal(mine, sync.flat))
        assert torch.equal(net[1].running_var, sync.flat[8:16])
    flat = torch.cat([p.detach().flatten() for p in net.parameters()])
    gathered = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(gathered, flat)
    if rank == 0:
        out.put([t.numpy().copy() for t in gathered])
    dist.barrier()
    dist.destroy_process_group()


def test_arena_allreduce_matches_ddp_arithmetic():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [torch.from_numpy(a) for a in q.get(timeout=120)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert torch.equal(res[0], res[1])                      # replicas bit-identical after 3 steps
    # single-process emulation of the reference: sum over ranks of the gradient of (loss_r * W) / W
    net = _net()
    opt = torch.optim.SGD(net.parameters(), lr=0.1, momentum=0.9, nesterov=True)
    gens = [torch.Generator().manual_seed(10 + r) for r in range(world)]
    for step in range(3):
        grads = None
        for r in range(world):
            net.zero_grad()
            (net(torch.randn(4, 3, 8, 8, generator=gens[r])).square().mean() * world).backward()
            cur = [p.grad.clone() / world for p in net.parameters()]
            grads = cur if grads is None else [a + b for a, b in zip(grads, cur)]
        for p, gsum in zip(net.parameters(), grads):
            p.grad = gsum
        opt.step()
    ref = torch.cat([p.detach().flatten() for p in net.parameters()])
    torch.testing.assert_close(res[0], ref, rtol=1e-5, atol=1e-6)
