"""GPU: the conv weight and bias gradients are the per-CTA partial slices of the wgrad kernels added in CTA order and permuted to
PyTorch layout, bit for bit.  The slices are read back from the learner's workspace and summed here with a sequential fp32 loop --
the order of additions the reduce kernels promise -- so any change of order, layout or scaling shows as a mismatch."""
import os

import numpy as np
import pytest
import torch

from oracle import impala_oracle as O
from tests import layer_ref as R

pytestmark = pytest.mark.gpu

# floats per CTA slice: accumulators in the wgrad kernel's [tap-block][row][co] order, then the bias (kernels.h WSP_W*)
SLICE = {'conv3': (5 * 128 * 64, 64), 'conv2': (4 * 128 * 64, 64), 'conv1': (2 * 128 * 32, 32)}
INV255 = torch.tensor(np.float32(1.0) / np.float32(255.0))


def _cta_sum(slices):
    s = torch.zeros_like(slices[0])
    for c in range(slices.shape[0]):
        s = s + slices[c]
    return s


def _expected(part, grids):
    out, off = {}, 0
    for name in ('conv3', 'conv2', 'conv1'):
        acc, nb = SLICE[name]
        sl = part[off:off + R.WG_PART_CTAS * (acc + nb)].view(R.WG_PART_CTAS, acc + nb)[:grids[name]]
        off += R.WG_PART_CTAS * (acc + nb)
        w, b = _cta_sum(sl[:, :acc]), _cta_sum(sl[:, acc:])
        if name == 'conv3':      # rows (tap, c) -> [co][c][kh][kw]; the tenth tap block is never written
            w = w[:9 * 64 * 64].view(9, 64, 64).permute(2, 1, 0).reshape(64, 64, 3, 3)
        elif name == 'conv2':    # rows (kh, kw, c)
            w = w.view(4, 4, 32, 64).permute(3, 2, 0, 1)
        else:                    # rows (kh2, kw2, c, dy, dx), kh = 4 kh2 + dy, kw = 4 kw2 + dx; the frames entered as u8
            w = w.view(2, 2, 4, 4, 4, 32).permute(5, 2, 0, 3, 1, 4).reshape(32, 4, 8, 8) * INV255
        out[f'{name}.weight'], out[f'{name}.bias'] = w.contiguous(), b
    return out


@pytest.mark.parametrize('path', ['eager', 'graph'])
@pytest.mark.parametrize('precision', ['bf16', 'fp32_split'])
@pytest.mark.parametrize('T,B,A', [(20, 32, 6), (20, 64, 4)])
def test_conv_gradients_are_the_cta_ordered_slice_sums(T, B, A, precision, path):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, precision=precision, learning_rate=0.0)
    L = B200ImpalaLearner(hp, init_state_dict=O.init_params(A, seed=5), process_group=False)
    try:
        dev = {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=5, done_p=0.1).items()}
        for _ in range(3 if path == 'graph' else 1):       # graph: eager, capture, replay -- the gradients of the replayed step
            if path == 'graph':
                L.learn(dev)
            else:
                L.forward_backward(dev)
        torch.cuda.synchronize()
        sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        parts = R.wgrad_partitions(T * B, R.cta_counts(sm, os.environ), precision == 'fp32_split')
        want = _expected(L.debug_buffer('wgrad_part').cpu(), {k: v['grid'] for k, v in parts.items()})
        for k, w in want.items():
            got = L.grads[k].cpu()
            assert got.shape == w.shape, k
            assert torch.equal(got, w), f'{k}: {int((got != w).sum())} of {w.numel()} elements differ, max |diff| {float((got - w).abs().max()):.3e}'
    finally:
        L.close()
