"""Runs one learner step and reports what it computed: imported by tests/test_gpu_layer_exact.py, and run as a child process by
its partition sweep (SRL_WGRAD_CTAS / SRL_BWD_CTAS / SRL_PERSISTENT_CTAS / SRL_PDL are read once per process).

    python tests/layer_exact_worker.py T B A OUT_DIR

writes OUT_DIR/{bf16,fp32_split}.pt (the gradients and a SHA-1 of every debug buffer) and prints a JSON line 'RESULT {...}'."""
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import impala_oracle as O  # noqa: E402

BUFFERS = ('xs', 'a1', 'a2', 'a3', 'h', 'logits', 'baseline', 'dlogits', 'dbaseline', 'dh', 'da3', 'da2', 'da1')
LO_BUFFERS = ('a1_lo', 'a2_lo', 'a3_lo', 'dh_lo', 'da3_lo', 'da2_lo', 'da1_lo')
SEED = 11


def run_step(T, B, A, precision='bf16', fused=False, replay=False, poison=False, seed=SEED):
    """One step at seed `seed`; returns (debug buffers, gradients, batch, params), all on the CPU.
    replay: three learn() calls at learning rate 0 (eager, capture, replay) -- the buffers and gradients of the replayed graph;
    otherwise one eager forward_backward."""
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    from scalerl_b200 import _lib
    params = O.init_params(A, seed=seed)
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, precision=precision, learning_rate=0.0)
    L = B200ImpalaLearner(hp, init_state_dict=params, process_group=False)
    if fused:
        L.set_option('fused_fwd', 1)
    batch = O.synthetic_batch(T, B, A, seed=seed, done_p=0.1)
    dev = {k: v.cuda() for k, v in batch.items()}
    for _ in range(3 if replay else 1):
        if poison:
            _lib.check_hook(_lib.hooks().srl_test_poison_smem(None))
            torch.cuda.synchronize()
        if replay:
            L.learn(dev)
        else:
            L.forward_backward(dev)
    torch.cuda.synchronize()
    names = BUFFERS + (LO_BUFFERS if precision == 'fp32_split' else ())
    bufs = {n: L.debug_buffer(n).cpu() for n in names}
    grads = {k: L.grads[k].cpu().clone() for k in O.PARAM_ORDER}
    if replay:
        # learn() leaves the gradients of before clipping in L.grads: an eager forward_backward on the same (unchanged) weights gives the same bits
        flat = L.flat_grads.clone()
        L.forward_backward(dev)
        torch.cuda.synchronize()
        assert torch.equal(L.flat_grads, flat), 'grads after learn() differ from an eager forward_backward'
    L.close()
    return bufs, grads, batch, params


def digest(t):
    return hashlib.sha1(t.contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


def main():
    T, B, A, out = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
    res = {}
    for precision in ('bf16', 'fp32_split'):
        bufs, grads, _, _ = run_step(T, B, A, precision)
        hashes = {n: digest(b) for n, b in bufs.items()}
        torch.save({'grads': grads, 'hashes': hashes}, os.path.join(out, f'{precision}.pt'))
        res[precision] = len(hashes)
    print('RESULT ' + json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
