"""CPU: the trainable AtariNet drop-in (scalerl_b200.algorithms.utils.atari_model.AtariNet) -- the reference's parameters and
initialisation, its constructor and input errors, and the stand-alone encoder entry points' argument checks (no GPU needed)."""
import ctypes as C

import pytest
import torch

from oracle import ref_learner
from scalerl_b200 import _lib, build as srl_build
from scalerl_b200.algorithms.utils.atari_model import AtariNet


@pytest.mark.skipif(not ref_learner.available(), reason='oracle/_ref (the reference modules) is not built')
@pytest.mark.parametrize('use_lstm', [False, True])
@pytest.mark.parametrize('A', [4, 6, 18])
def test_state_dict_and_init_match_the_reference(A, use_lstm):
    am = ref_learner._load('atari_model')
    torch.manual_seed(11)
    ref = am.AtariNet((4, 84, 84), A, use_lstm=use_lstm)
    torch.manual_seed(11)
    mine = AtariNet((4, 84, 84), A, use_lstm=use_lstm)
    rs, ms = ref.state_dict(), mine.state_dict()
    assert list(rs) == list(ms)
    for k in rs:
        assert rs[k].shape == ms[k].shape, k
        assert torch.equal(rs[k], ms[k]), k
    assert [n for n, _ in ref.named_parameters()] == [n for n, _ in mine.named_parameters()]


@pytest.mark.parametrize('kw', [dict(observation_shape=(3, 84, 84), num_actions=6), dict(observation_shape=(4, 84, 84), num_actions=0),
                                dict(observation_shape=(4, 84, 84), num_actions=32),
                                dict(observation_shape=(4, 84, 84), num_actions=6, precision='fp16')])
def test_constructor_errors(kw):
    with pytest.raises(ValueError):
        AtariNet(**kw)


def test_deepcopy_and_optimizer_work_as_on_any_module():
    import copy
    net = AtariNet((4, 84, 84), 6, use_lstm=True)
    twin = copy.deepcopy(net)
    assert twin._contexts is not net._contexts and twin._contexts.handles == {}
    for (n, p), (m, q) in zip(net.named_parameters(), twin.named_parameters()):
        assert n == m and torch.equal(p, q) and p.data_ptr() != q.data_ptr()
    torch.optim.RMSprop(net.parameters(), lr=1e-4)
    net.zero_grad(set_to_none=True)


def test_forward_on_cpu_tensors_raises():
    net = AtariNet((4, 84, 84), 6)
    T, B = 2, 3
    inputs = dict(obs=torch.zeros(T, B, 4, 84, 84, dtype=torch.uint8), reward=torch.zeros(T, B), action=torch.zeros(T, B, dtype=torch.int64),
                  done=torch.zeros(T, B, dtype=torch.bool))
    with pytest.raises(ValueError, match='CUDA'):
        net(inputs)


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


def _err(L):
    return L.srl_last_error().decode()


def test_size_query_argument_errors(lib):
    L = lib
    s, k = C.c_int64(), C.c_int64()
    for frames, prec in ((0, 0), (65537, 0), (8, 2)):
        assert L.srl_encoder_sizes(frames, prec, C.byref(s), C.byref(k)) == -1
    assert L.srl_encoder_sizes(8, 0, None, C.byref(k)) == -1 and 'NULL' in _err(L)
    assert L.srl_encoder_sizes(672, 0, C.byref(s), C.byref(k)) == 0
    # the forward keeps xs, a1, a2, a3, h and the packed weights: about 74 MB at T+1 = 21, B = 32 in the bf16 mode
    assert 74.0e6 < s.value < 75.0e6
    s1 = C.c_int64()
    assert L.srl_encoder_sizes(672, 1, C.byref(s1), C.byref(k)) == 0 and s1.value > s.value      # + the low twins


def test_entry_points_reject_bad_arguments_before_any_cuda_call(lib):
    L = lib
    h = C.c_void_p()
    assert L.srl_encoder_create(2, C.byref(h)) == -1 and 'precision' in _err(L)
    assert L.srl_encoder_create(0, None) == -1
    assert L.srl_encoder_forward(None, None, None, None, 8, 6, None, None, None, None, None) == -1 and 'NULL' in _err(L)
    assert L.srl_encoder_backward(None, None, 8, 6, None, None, None, None) == -1 and 'NULL' in _err(L)
    assert L.srl_encoder_create(0, C.byref(h)) == 0          # lanes are optional: no device needed to hold a context
    try:
        frames, A = 8, 6
        base = 1 << 40                                        # fake device addresses, far apart and 256-byte aligned
        at = lambda i: base + (i << 32)
        obs, reward, action, saved, scratch, core = at(0), at(1), at(2), at(3), at(4), at(5)
        w = (C.c_void_p * 8)(*[at(10 + i) for i in range(8)])

        def fwd(**kw):
            a = dict(obs=obs, reward=reward, action=action, frames=frames, A=A, w=w, saved=saved, scratch=scratch, core=core)
            a.update(kw)
            return L.srl_encoder_forward(h, a['obs'], a['reward'], a['action'], a['frames'], a['A'], a['w'], a['saved'], a['scratch'],
                                         a['core'], None)

        assert fwd(frames=0) == -1 and 'frames' in _err(L)
        assert fwd(frames=65537) == -1 and 'frames' in _err(L)
        assert fwd(A=32) == -1 and 'A=32' in _err(L)
        assert fwd(saved=saved + 16) == -1 and 'aligned' in _err(L)
        assert fwd(obs=obs + 1) == -1 and 'aligned' in _err(L)
        assert fwd(scratch=saved + 256) == -1 and 'overlap' in _err(L)
        assert fwd(core=obs) == -1 and 'overlap' in _err(L)
        assert fwd(core=at(16)) == -1 and 'overlap' in _err(L)                    # core_out on fc.weight
        assert fwd(w=(C.c_void_p * 8)(*([at(10)] + [None] * 7))) == -1 and 'NULL' in _err(L)
        assert fwd(w=(C.c_void_p * 8)(*([at(10) + 4] + [at(11 + i) for i in range(7)]))) == -1 and 'aligned' in _err(L)
        g = (C.c_void_p * 8)(*[at(20 + i) for i in range(8)])
        dcore = at(6)
        assert L.srl_encoder_backward(h, dcore, 0, A, saved, scratch, g, None) == -1 and 'frames' in _err(L)
        assert L.srl_encoder_backward(h, dcore, frames, A, saved, saved, g, None) == -1 and 'overlap' in _err(L)
        assert L.srl_encoder_backward(h, dcore, frames, A, saved, scratch, (C.c_void_p * 8)(*([saved] + list(g)[1:])), None) == -1
        assert 'overlap' in _err(L)
        assert L.srl_encoder_backward(h, dcore, frames, A, saved, scratch, (C.c_void_p * 8)(*([at(20)] * 8)), None) == -1
        assert 'overlap' in _err(L)
    finally:
        assert L.srl_encoder_destroy(h) == 0


def test_encoder_row_hook_argument_errors(lib):
    """srl_test_encoder_row (the test hook that names a row of the encoder's blocks) rejects what srl_encoder_sizes rejects, NULL
    arguments and unknown rows before any CUDA call"""
    H = _lib.hooks()
    err = lambda: H.srl_test_last_error().decode()
    hi, lo, n = C.c_void_p(), C.c_void_p(), C.c_int64()
    saved, scratch = 1 << 40, (1 << 40) + (1 << 36)
    row = lambda frames=8, prec=0, name=b'a1', s=saved, k=scratch, out=(C.byref(hi), C.byref(lo), C.byref(n)): \
        H.srl_test_encoder_row(frames, prec, name, s, k, *out)
    for frames in (0, -1, 65537):
        assert row(frames=frames) == -1 and f'frames={frames}' in err()
    assert row(prec=2) == -1 and 'precision=2' in err()
    assert row(name=None) == -1 and 'NULL' in err()
    assert row(s=None) == -1 and 'NULL' in err()
    assert row(k=None) == -1 and 'NULL' in err()
    assert row(out=(None, C.byref(lo), C.byref(n))) == -1 and 'NULL' in err()
    assert row(out=(C.byref(hi), C.byref(lo), None)) == -1 and 'NULL' in err()
    for bad in (b'hpart', b'', b'a1_lo', b'da0', b'logits'):
        assert row(name=bad) == -1 and 'unknown row' in err(), bad


def test_every_output_against_every_other_argument(lib):
    """each output of srl_encoder_forward / _backward placed on each other argument is rejected before any CUDA call"""
    L = lib
    h = C.c_void_p()
    assert L.srl_encoder_create(0, C.byref(h)) == 0
    try:
        at = lambda i: (1 << 40) + (i << 32)                  # fake device addresses, far apart and 256-byte aligned
        fa = dict(obs=at(0), reward=at(1), action=at(2), saved=at(3), scratch=at(4), core=at(5), **{f'w{i}': at(10 + i) for i in range(8)})
        ba = dict(dcore=at(6), saved=at(3), scratch=at(4), **{f'g{i}': at(20 + i) for i in range(8)})

        def fwd(**kw):
            a = {**fa, **kw}
            return L.srl_encoder_forward(h, a['obs'], a['reward'], a['action'], 8, 6, (C.c_void_p * 8)(*[a[f'w{i}'] for i in range(8)]),
                                         a['saved'], a['scratch'], a['core'], None)

        def bwd(**kw):
            a = {**ba, **kw}
            return L.srl_encoder_backward(h, a['dcore'], 8, 6, a['saved'], a['scratch'], (C.c_void_p * 8)(*[a[f'g{i}'] for i in range(8)]), None)

        for o in ('saved', 'scratch', 'core'):
            for other in fa:
                if other != o:
                    assert fwd(**{o: fa[other]}) == -1 and 'overlaps' in _err(L), (o, other)
        for o in ['scratch'] + [f'g{i}' for i in range(8)]:
            for other in ba:
                if other != o:
                    assert bwd(**{o: ba[other]}) == -1 and 'overlaps' in _err(L), (o, other)
        assert fwd(core=at(16)) == -1 and _err(L) == 'encoder_forward: core_out overlaps weights8[6]'
        assert bwd(g7=at(20)) == -1 and _err(L) == 'encoder_backward: grads8[7] overlaps grads8[0]'
        assert bwd(g2=at(3)) == -1 and 'grads8[2] overlaps saved' in _err(L)
    finally:
        assert L.srl_encoder_destroy(h) == 0
