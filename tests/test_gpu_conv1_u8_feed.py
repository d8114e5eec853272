"""conv1's forward fed straight from the u8 frames (RConv1Fwd::FromFrames: the window converted in shared memory, xs written from it) computes
the bits of the path it replaces, obs_s2d_kernel's space-to-depth copy into xs followed by conv1 fed from xs.  The encoder takes
the u8 path for 16-byte aligned frames in the bf16 mode and the xs path for frames that are only 4-byte aligned, so the same frames
at an offset of 4 bytes give the reference.  Compared with torch.equal: xs, a1, a2, a3, the gradients and the updated parameters.

The frame counts put the last 128-position tile partly past the frames (441 positions per frame is not a multiple of 128) and make
tiles straddle frame boundaries; 38044 frames put xs past 2^31 bytes."""
import pytest
import torch

from oracle import impala_oracle as O
from tests.test_gpu_encoder_exact import ENC_NAMES, Encoder

pytestmark = pytest.mark.gpu


def _offset_copy(t, offset):
    """a contiguous copy of t whose data starts `offset` bytes past a 256-byte aligned allocation"""
    n = t.numel() * t.element_size()
    buf = torch.empty(n + 256, dtype=torch.uint8, device=t.device)
    out = buf[offset:offset + n].view(t.dtype).view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16 == offset % 16
    return out


@pytest.mark.parametrize('T,B', [(6, 19), (20, 32), (20, 64)])
def test_learner_step_u8_feed_equals_xs_feed(T, B):
    """one captured learner step at (T+1) x B frames from aligned and from 4-byte offset frames: same activations, gradients, update"""
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    A = 6
    batch = {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=11, done_p=0.1).items()}
    got = {}
    for offset in (0, 4):
        params = O.init_params(A, seed=5)
        L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A), init_state_dict=params, process_group=False)
        try:
            b = dict(batch, obs=_offset_copy(batch['obs'], offset))
            st = L.learn(b)
            torch.cuda.synchronize()
            got[offset] = {n: L.debug_buffer(n) for n in ('xs', 'a1', 'a2', 'a3')}
            got[offset]['grads'] = L.flat_grads.clone()
            got[offset]['params'] = L.flat_params.clone()
            got[offset]['loss'] = st['total_loss']
        finally:
            L.close()
    for k in ('xs', 'a1', 'a2', 'a3', 'grads', 'params'):
        assert torch.equal(got[0][k], got[4][k]), k
    assert got[0]['loss'] == got[4]['loss']


@pytest.mark.parametrize('F', [1, 7 * 19, 21 * 32, 38044])
def test_encoder_u8_feed_equals_xs_feed(F):
    """the C-ABI encoder (frames = NF = NB) forward + backward from aligned and from 4-byte offset frames: same bits"""
    A = 6
    g = torch.Generator(device='cuda').manual_seed(F)
    params = O.init_params(A, seed=1)
    weights = [params[n].cuda().contiguous() for n in ENC_NAMES]
    obs = torch.randint(0, 256, (F, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    reward = torch.randn(F, device='cuda', generator=g)
    action = torch.randint(0, A, (F,), device='cuda', generator=g)
    dcore = torch.randn(F, 513 + A, device='cuda', generator=g)
    enc = Encoder(F, False)
    try:
        got = {}
        for offset in (0, 4):
            enc.saved.fill_(0x5A)           # each run starts from the same garbage: nothing is inherited from the first
            enc.scratch.fill_(0x5A)
            core_out = torch.empty(F, 513 + A, device='cuda')
            grads = [torch.empty_like(w) for w in weights]
            enc.forward(_offset_copy(obs, offset), reward, action, A, weights, core_out)
            enc.backward(dcore, A, grads)
            torch.cuda.synchronize()
            rows = {n: enc.row(n, torch.bfloat16)[0] for n in ('xs', 'a1', 'a2', 'a3')}
            if offset == 0:
                rows = {n: v.clone() for n, v in rows.items()}
            got[offset] = dict(rows, core_out=core_out, grads=grads)
        for k in ('xs', 'a1', 'a2', 'a3', 'core_out'):
            assert torch.equal(got[0][k], got[4][k]), k
        for n, a, b in zip(ENC_NAMES, got[0]['grads'], got[4]['grads']):
            assert torch.equal(a, b), n
    finally:
        enc.close()


def test_step_runs_the_u8_fed_conv1():
    """the default step (aligned frames, bf16 mode) runs conv1 from the frames; the fp32-split step keeps conv1 fed from xs"""
    from tests.test_gpu_step_graph import capture_variant
    for variant, from_frames in (('default', True), ('fp32_split', False)):
        G, L = capture_variant(variant)
        try:
            names = [G.labels[v] for v in G.find('conv1_fwd')]
            assert len(names) == 1 and ('FromFrames' in names[0]) == from_frames, (variant, names)
        finally:
            L.close()
