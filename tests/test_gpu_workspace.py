"""GPU: the learner context's workspace as srl_learner_debug_buffer and srl_learner_workspace_bytes report it.  Every count is
written out here from the layouts of DESIGN.md §3 (NF = (T+1)B frames, NB = TB learning frames), not read from the library."""
import pytest

pytestmark = pytest.mark.gpu

HP = 576                                    # the actor step's padded LSTM width (H = 513 + A rounded up to 64)
WPACK = (32 * 256                           # conv1, K-major
         + 64 * 512 + 4 * 32 * 256          # conv2: forward, and dgrad by output parity class
         + 2 * 64 * 576                     # conv3: forward and dgrad
         + 2 * 512 * 3136)                  # fc.weight: K-major and transposed
TWINS = ('a1', 'a2', 'a3', 'dh', 'da3', 'da2', 'da1', 'wpack')
FP32 = ('h', 'logits', 'baseline', 'dlogits', 'dbaseline')


def expected_counts(T, B, A):
    NF, NB = (T + 1) * B, T * B
    return {'xs': NF * 441 * 64, 'a1': 2 * NF * 100 * 64, 'a2': NF * 81 * 64, 'a3': NF * 49 * 64, 'a3t': NF * 64 * 49,
            'h': NF * 512, 'logits': NF * A, 'baseline': NF, 'dlogits': NB * A, 'dbaseline': NB,
            'dh': NB * 512, 'da3': NB * 81 * 64, 'da2': NB * 100 * 64, 'da1': NB * 441 * 32, 'wpack': WPACK}


@pytest.mark.parametrize('mode', ['bf16', 'fp32_split', 'lstm'])
@pytest.mark.parametrize('T,B,A', [(3, 5, 4), (20, 32, 6)])
def test_workspace_buffers(mode, T, B, A):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    use_lstm = mode == 'lstm'
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, use_lstm=use_lstm,
                       precision='fp32_split' if mode == 'fp32_split' else 'bf16')
    L = B200ImpalaLearner(hp, process_group=False)
    try:
        counts = expected_counts(T, B, A)
        if mode == 'fp32_split':
            counts.update({f'{n}_lo': counts[n] for n in TWINS})
        for name, n in counts.items():
            assert L.debug_buffer(name).numel() == n, name
        if mode != 'fp32_split':
            for name in TWINS:
                with pytest.raises(RuntimeError, match='rc=-2.*fp32-accurate'):
                    L.debug_buffer(f'{name}_lo')
        steps = {'lstm_step_xh': 2 * B * 2 * HP, 'lstm_step_w': 2 * 4 * HP * 2 * HP}
        for name, n in steps.items():
            if use_lstm:
                assert L.debug_buffer(name).numel() == n, name
                with pytest.raises(ValueError, match='unknown buffer'):
                    L.debug_buffer(name[:-1])
            else:
                with pytest.raises(ValueError, match='use_lstm'):
                    L.debug_buffer(name)
        for name in ('xs_lo', 'h_lo', 'a3t_lo', 'hpart', 'a', ''):
            with pytest.raises(ValueError, match='unknown buffer'):
                L.debug_buffer(name)
        need = sum(n * (4 if name in FP32 else 2) for name, n in counts.items())
        if use_lstm:           # core and the LSTM output [NF][H], their gradients [NB][H], f32
            need += 2 * ((T + 1) * B + T * B) * (513 + A) * 4
        assert L._L.srl_learner_workspace_bytes(L._h) >= need
    finally:
        L.close()
