"""CPU, world_size=2 gloo: the data-parallel host logic (column sharding + SUM all-reduce) reproduces the
full-batch gradients, losses and clipped update of the oracle (the N>1 path of SURVEY.md §8e)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from scalerl_b200 import parallel as par


def test_shard_bounds_cover_and_balance():
    for B in (1, 2, 7, 32, 512, 513):
        for w in (1, 2, 3, 8):
            spans = [par.shard_bounds(B, r, w) for r in range(w)]
            assert spans[0][0] == 0 and spans[-1][1] == B
            assert all(spans[i][1] == spans[i + 1][0] for i in range(w - 1))
            sizes = [b - a for a, b in spans]
            assert max(sizes) - min(sizes) <= 1
    with pytest.raises(ValueError):
        par.shard_bounds(4, 2, 2)


def _worker(rank, world, port, out_q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.set_num_threads(2)
    from oracle import impala_oracle as O
    T, B, A = 3, 6, 4
    params = O.init_params(A, seed=5)
    flat0 = torch.cat([p.reshape(-1) for p in params.values()])
    par.broadcast_params_(flat0, src=0)
    batch = O.synthetic_batch(T, B, A, seed=9, done_p=0.2)
    shard = {k: v.contiguous() for k, v in par.shard_columns(batch, rank, world).items()}
    out = O.learn_step({k: v.clone() for k, v in params.items()}, None, shard, update=False)
    flat = torch.cat([out['grads'][k].reshape(-1) for k in O.PARAM_ORDER])
    losses = torch.tensor([out['pg_loss'], out['baseline_loss'], out['entropy_loss'], out['total_loss']])
    par.allreduce_sum_(flat, losses)
    if rank == 0:      # numpy arrays travel by value: a tensor would be shared through a descriptor that this process must outlive
        out_q.put((flat.numpy(), losses.numpy()))
    dist.destroy_process_group()


def test_two_rank_gloo_matches_full_batch():
    from oracle import impala_oracle as O
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    flat, losses = (torch.from_numpy(a) for a in q.get())
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    T, B, A = 3, 6, 4
    params = O.init_params(A, seed=5)
    batch = O.synthetic_batch(T, B, A, seed=9, done_p=0.2)
    full = O.learn_step(params, None, batch, update=False)
    ref = torch.cat([full['grads'][k].reshape(-1) for k in O.PARAM_ORDER])
    assert float((flat - ref).norm() / ref.norm()) < 1e-5
    want = torch.tensor([full['pg_loss'], full['baseline_loss'], full['entropy_loss'], full['total_loss']])
    assert torch.allclose(losses, want, rtol=1e-5, atol=1e-5)
