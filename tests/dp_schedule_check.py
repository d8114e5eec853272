"""Multi-GPU check of the learning-rate schedule and RMSprop momentum in the data-parallel step (run with torchrun on >= 2 GPUs;
collected through tests/test_gpu_optim_schedule.py, not by pytest directly):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/dp_schedule_check.py

Every rank learns on its column shard with momentum 0.9 and the 'linear' schedule (RMSprop), or the schedule alone (Adam); rank 0
also runs a single-GPU learner on the FULL batch.  Both count T * B_global frames per step, so they follow the same schedule: every
step the lr must be the same bits, and the sharded weights must equal the full-batch ones up to fp32 summation order.  The
full-batch learner is then re-synchronised to the sharded state (weights and optimizer state), as in tests/dp_check.py.  At the
end the replicas must be bit-identical."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import impala_oracle as O                       # noqa: E402  (checker/input generator only)
from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams   # noqa: E402
from scalerl_b200 import parallel as par                    # noqa: E402


def main():
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    T, A, B = 6, 6, 4 * world
    params = O.init_params(A, seed=11)
    batches = [{k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=5 + i, done_p=0.1).items()} for i in range(6)]
    full_buf = {k: v.clone() for k, v in batches[0].items()}
    mine = {k: v.contiguous() for k, v in par.shard_columns(batches[0], rank, world).items()}
    total = 4 * T * B                                        # the decay ends at step 5; step 6 runs at the floor
    for optimizer, momentum in (('rmsprop', 0.9), ('adam', 0.0)):
        kw = dict(rollout_length=T, num_actions=A, optimizer=optimizer, momentum=momentum, learning_rate=2.0 ** -10, lr_schedule='linear',
                  total_frames=total, min_learning_rate=2.0 ** -14)
        shard = B200ImpalaLearner(ImpalaHParams(batch_size=B // world, **kw), init_state_dict=params)
        full = B200ImpalaLearner(ImpalaHParams(batch_size=B, **kw), init_state_dict=params, process_group=False) if rank == 0 else None
        assert shard.frames_per_step == T * B, shard.frames_per_step
        path = (f'peer memory (fused reduce+clip+optimizer kernel; {getattr(shard, "dp_path", "?")})' if shard._peers is not None
                else 'NCCL all-reduce')
        worst = 0.0
        for step, batch in enumerate(batches, start=1):
            for k, v in par.shard_columns(batch, rank, world).items():
                mine[k].copy_(v)
            s = shard.learn(mine)
            if rank == 0:
                for k, v in batch.items():
                    full_buf[k].copy_(v)
                f = full.learn(full_buf)
                assert shard.learning_rate() == full.learning_rate(), (step, shard.learning_rate(), full.learning_rate())
                rel = float((shard.flat_params - full.flat_params).norm() / full.flat_params.norm())
                worst = max(worst, rel)
                print(f'{optimizer} momentum {momentum} step {step}: lr {shard.learning_rate():.6e} | grad_norm {s["grad_norm"]:.4f} vs '
                      f'{f["grad_norm"]:.4f} | param rel-L2 {rel:.2e}', flush=True)
                assert abs(s['grad_norm'] - f['grad_norm']) <= 1e-4 * f['grad_norm'] and rel < 1e-5
                full.flat_params.copy_(shard.flat_params)                      # next step starts from identical state
                for a, b in ((full.opt_state0, shard.opt_state0), (full.opt_state1, shard.opt_state1), (full.opt_state2, shard.opt_state2)):
                    if a is not None:
                        a.copy_(b)
        assert shard.learning_rate() == 2.0 ** -14
        chk = torch.cat([shard.flat_params, shard.opt_state2 if shard.opt_state2 is not None else shard.opt_state0])
        chk = chk.view(torch.int32).to(torch.int64).sum().reshape(1)
        allc = [torch.zeros_like(chk) for _ in range(world)]
        dist.all_gather(allc, chk)
        if rank == 0:
            assert all(int(c) == int(allc[0]) for c in allc), [int(c) for c in allc]
            print(f'{optimizer} momentum {momentum}: gradient path = {path}; replicas bit-identical on {world} ranks; worst {worst:.2e}', flush=True)
        shard.release_graphs()
    if rank == 0:
        print('DP SCHEDULE CHECK OK', flush=True)
    dist.barrier(device_ids=[local])
    os._exit(0)


if __name__ == '__main__':
    main()
