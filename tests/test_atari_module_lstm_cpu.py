"""CPU: the stand-alone LSTM core entry points (srl_lstm_core_*) -- block sizes and argument checks before any CUDA call -- and the
state / done input errors of AtariNet(use_lstm=True) (no GPU needed)."""
import ctypes as C

import pytest
import torch

from scalerl_b200 import _lib, build as srl_build
from scalerl_b200.algorithms.utils.atari_model import AtariNet, lstm_block_sizes


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


def _err(L):
    return L.srl_lstm_last_error().decode()


def _al(n):
    return (n + 255) // 256 * 256


def _table_sizes(T1, B, A):
    """the row table of csrc/lstm.cu (lstm_rows) restated from shapes: (saved, scratch) bytes for a backward over all T1*B rows"""
    H = 513 + A
    Hp = (H + 63) // 64 * 64
    G, N1 = 4 * Hp, T1 * B
    layer = 2 * _al(N1 * Hp * 2) + 4 * _al(G * Hp * 2) + _al(N1 * G * 4) + _al(N1 * Hp * 4)     # hm, hbf, 4 weights, gates, c
    saved = _al(N1 * Hp * 2) + 2 * layer + _al(2 * B * Hp * 4) + _al(N1)                      # + xin0, c_init, done
    scratch = (_al(N1 * G * 4) + _al(B * G * 4) + 2 * _al(N1 * Hp * 4) + 2 * _al(N1 * G * 2) + _al(N1 * Hp * 4) + _al(G * Hp * 4)
               + 2 * _al(B * Hp * 4) + _al((N1 + 63) // 64 * G * 4))
    return saved, scratch


def test_size_query(lib):
    L = lib
    s, k = C.c_int64(), C.c_int64()
    for T1, B, A in ((0, 4, 6), (4, 0, 6), (65537, 1, 6), (257, 256, 6), (4, 4, 0), (4, 4, 32)):
        assert L.srl_lstm_core_sizes(T1, B, A, C.byref(s), C.byref(k)) == -1, (T1, B, A)
    assert 'A=32' in _err(L)
    assert L.srl_lstm_core_sizes(4, 4, 6, None, C.byref(k)) == -1 and 'NULL' in _err(L)
    for T1, B, A in ((21, 32, 6), (101, 16, 6), (1, 1, 1), (2, 130, 31), (65536, 1, 4), (1, 65536, 18)):
        assert L.srl_lstm_core_sizes(T1, B, A, C.byref(s), C.byref(k)) == 0
        assert (s.value, k.value) == _table_sizes(T1, B, A), (T1, B, A)
        assert lstm_block_sizes(T1, B, A) == (s.value, k.value)
    # about 41 MB at T+1 = 21, B = 32 (half of it the packed weights) and 0.39 GB at T+1 = 101, B = 128 (60 % gate activations)
    assert 40e6 < lstm_block_sizes(21, 32, 6)[0] < 42e6
    assert 0.38e9 < lstm_block_sizes(101, 128, 6)[0] < 0.40e9
    with pytest.raises(ValueError, match='A=0'):
        lstm_block_sizes(4, 4, 0)


BASE = 1 << 40                                   # fake device addresses, far apart and 256-byte aligned: nothing may reach CUDA


def _at(i):
    return BASE + (i << 32)


def _fwd(L, **kw):
    a = dict(core=_at(0), done=_at(1), h0=_at(2), c0=_at(3), A=6, T1=5, B=3, w=(C.c_void_p * 8)(*[_at(10 + i) for i in range(8)]),
             saved=_at(4), scratch=_at(5), out=_at(6), hT=_at(7), cT=_at(8))
    a.update(kw)
    return L.srl_lstm_core_forward(a['core'], a['done'], a['h0'], a['c0'], a['A'], a['T1'], a['B'], a['w'], a['saved'], a['scratch'],
                                   a['out'], a['hT'], a['cT'], None)


def _bwd(L, **kw):
    a = dict(dout=_at(0), dhT=_at(1), dcT=_at(2), A=6, T1=5, B=3, saved=_at(4), scratch=_at(5), g=(C.c_void_p * 8)(*[_at(20 + i) for i in range(8)]),
             dcore=_at(6), dh0=_at(7), dc0=_at(8))
    a.update(kw)
    return L.srl_lstm_core_backward(a['dout'], a['dhT'], a['dcT'], a['A'], a['T1'], a['B'], a['saved'], a['scratch'], a['g'], a['dcore'],
                                    a['dh0'], a['dc0'], None)


def _rejects(rc, L, word):
    return rc == -1 and word in _err(L)


def test_forward_rejects_bad_arguments_before_any_cuda_call(lib):
    L = lib
    for name in ('core', 'done', 'h0', 'c0', 'saved', 'scratch', 'out', 'hT', 'cT', 'w'):
        assert _rejects(_fwd(L, **{name: None}), L, 'NULL'), name
    assert _rejects(_fwd(L, w=(C.c_void_p * 8)(*([_at(10)] * 7 + [None]))), L, 'weights8[7] is NULL')
    for T1, B in ((0, 3), (5, 0), (65537, 1), (4097, 16)):
        assert _rejects(_fwd(L, T1=T1, B=B), L, 'T1*B'), (T1, B)
    assert _rejects(_fwd(L, A=0), L, 'A=0') and _rejects(_fwd(L, A=32), L, 'A=32')
    assert _rejects(_fwd(L, saved=_at(4) + 16), L, 'aligned') and _rejects(_fwd(L, scratch=_at(5) + 128), L, 'aligned')
    # every output against every other argument (inputs may share memory with each other)
    outs = ('saved', 'scratch', 'out', 'hT', 'cT')
    for o in outs:
        for other in ('core', 'done', 'h0', 'c0') + tuple(x for x in outs if x != o):
            assert _rejects(_fwd(L, **{o: _fwd_addr(other)}), L, 'overlaps'), (o, other)
        assert _rejects(_fwd(L, **{o: _at(13)}), L, 'overlaps'), o                  # on weights8[3]
    assert _rejects(_fwd(L, out=_at(0) + 4096), L, 'overlaps')                        # partly over core


def _fwd_addr(name):
    return dict(core=_at(0), done=_at(1), h0=_at(2), c0=_at(3), saved=_at(4), scratch=_at(5), out=_at(6), hT=_at(7), cT=_at(8))[name]


def _bwd_addr(name):
    return dict(dout=_at(0), dhT=_at(1), dcT=_at(2), saved=_at(4), scratch=_at(5), dcore=_at(6), dh0=_at(7), dc0=_at(8))[name]


def test_backward_rejects_bad_arguments_before_any_cuda_call(lib):
    L = lib
    for name in ('dout', 'saved', 'scratch', 'g', 'dcore'):
        assert _rejects(_bwd(L, **{name: None}), L, 'NULL'), name
    assert _rejects(_bwd(L, g=(C.c_void_p * 8)(*([None] + [_at(21 + i) for i in range(7)]))), L, 'grads8[0] is NULL')
    for T1, B in ((0, 3), (5, 0), (65537, 1)):
        assert _rejects(_bwd(L, T1=T1, B=B), L, 'T1*B'), (T1, B)
    assert _rejects(_bwd(L, A=0), L, 'A=0') and _rejects(_bwd(L, A=32), L, 'A=32')
    assert _rejects(_bwd(L, saved=_at(4) + 64), L, 'aligned') and _rejects(_bwd(L, scratch=_at(5) + 8), L, 'aligned')
    outs = ('scratch', 'dcore', 'dh0', 'dc0')
    for o in outs:
        for other in ('dout', 'dhT', 'dcT', 'saved') + tuple(x for x in outs if x != o):
            assert _rejects(_bwd(L, **{o: _bwd_addr(other)}), L, 'overlaps'), (o, other)
        assert _rejects(_bwd(L, **{o: _at(25)}), L, 'overlaps'), o                  # on grads8[5]
    g = [_at(20 + i) for i in range(8)]
    assert _rejects(_bwd(L, g=(C.c_void_p * 8)(*(g[:7] + [g[0]]))), L, 'grads8[7] overlaps grads8[0]')
    assert _rejects(_bwd(L, g=(C.c_void_p * 8)(*(g[:2] + [_at(4)] + g[3:]))), L, 'grads8[2] overlaps saved')
    assert _rejects(_bwd(L, g=(C.c_void_p * 8)(*([_at(0)] + g[1:]))), L, 'overlaps dout')


def _lookup(L, name, layer=0, T1=5, B=3, A=6, saved=_at(4), scratch=_at(5)):
    p, n = C.c_void_p(), C.c_int64()
    rc = L.srl_lstm_core_debug_buffer(T1, B, A, saved, scratch, name.encode() if name is not None else None, layer, C.byref(p), C.byref(n))
    return rc, (p.value or 0), n.value


def test_debug_buffer_rejects_bad_arguments_before_any_cuda_call(lib):
    L = lib
    assert _rejects(_lookup(L, 'gates', saved=None)[0], L, 'NULL') and _rejects(_lookup(L, None)[0], L, 'NULL')
    p, n = C.c_void_p(), C.c_int64()
    assert _rejects(L.srl_lstm_core_debug_buffer(5, 3, 6, _at(4), _at(5), b'gates', 0, None, C.byref(n)), L, 'NULL')
    assert _rejects(L.srl_lstm_debug_buffer(None, b'gates', 0, C.byref(p), C.byref(n)), L, 'NULL')
    for name in ('nope', 'gate', 'gates_lo', '', 'Hm'):
        assert _rejects(_lookup(L, name)[0], L, 'unknown buffer'), name
    for name, layer in (('gates', 2), ('gates', -1), ('hm', 7), ('xin0', 1), ('done', 1), ('dc', -1)):
        assert _rejects(_lookup(L, name, layer)[0], L, f'layer={layer}'), (name, layer)
    for T1, B, A in ((0, 3, 6), (5, 0, 6), (65537, 1, 6), (5, 3, 0), (5, 3, 32)):
        assert _rejects(_lookup(L, 'gates', T1=T1, B=B, A=A)[0], L, 'lstm_core_debug_buffer'), (T1, B, A)
    assert _rejects(_lookup(L, 'gates', saved=_at(4) + 32)[0], L, 'aligned')


@pytest.mark.parametrize('T1,B,A', [(5, 3, 6), (1, 7, 6), (2, 130, 31), (9, 128, 1), (101, 16, 6)])
def test_debug_buffer_rows_follow_the_table(lib, T1, B, A):
    """every named row: its count from the shapes, 256-byte aligned, inside the block srl_lstm_core_sizes reports, no two rows overlapping,
    and the saved / scratch split of the table"""
    from tests import lstm_ref as R
    L = lib
    H = R.hidden(A)
    Hp, N1 = R.padded(H), T1 * B
    G = 4 * Hp
    want = {'xin0': N1 * Hp, 'hm': N1 * Hp, 'hbf': N1 * Hp, 'Wih': G * Hp, 'WihT': G * Hp, 'Whh': G * Hp, 'WhhT': G * Hp, 'gates': N1 * G,
            'cseq': N1 * Hp, 'c_init': 2 * B * Hp, 'done': N1, 'gx': N1 * G, 'r': B * G, 'hseq': N1 * Hp, 'dgates': N1 * G, 'dx': N1 * Hp,
            'dwpad': G * Hp, 'dc': B * Hp, 'dhm': B * Hp, 'bias_part': (N1 + 63) // 64 * G}
    assert set(want) == set(R.LAYER_ROWS) | set(R.SHARED_ROWS)
    sb, kb = lstm_block_sizes(T1, B, A)
    spans = []
    for name in want:
        for layer in ((0, 1) if name in R.LAYER_ROWS else (0,)):
            rc, p, n = _lookup(L, name, layer, T1, B, A)
            assert rc == 0, (name, layer, _err(L))
            assert n == want[name], (name, n, want[name])
            assert p % 256 == 0, name
            base, size = (_at(4), sb) if p < _at(5) else (_at(5), kb)
            end = p + n * R.row_dtype(name).itemsize
            assert base <= p and end <= base + size, (name, layer)
            saved = name in ('xin0', 'c_init', 'done') or (name in R.LAYER_ROWS and name not in ('hseq', 'dgates'))
            assert (base == _at(4)) == saved, name
            spans.append((p, end, name, layer))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), 'rows overlap'


def test_errors_are_reported_by_srl_last_error(lib):
    """the LSTM core reports through the library's one message: srl_lstm_last_error returns what srl_last_error does"""
    L = lib
    assert L.srl_encoder_sizes(0, 0, None, None) == -1                 # another entry point's message first
    assert _fwd(L, A=32) == -1
    msg = L.srl_last_error().decode()
    assert msg.startswith('lstm_core_forward: ') and 'A=32' in msg
    assert _err(L) == msg


# ---- AtariNet(use_lstm=True): state and done errors come before the encoder (no device needed to see them)
def _inputs(T, B, A=6, done=None):
    return dict(obs=torch.zeros(T, B, 4, 84, 84, dtype=torch.uint8), reward=torch.zeros(T, B), action=torch.zeros(T, B, dtype=torch.int64),
                done=torch.zeros(T, B, dtype=torch.bool) if done is None else done)


@pytest.mark.parametrize('state,match', [
    ((), 'rnn_state must be the 2-tuple'),
    (None, 'rnn_state must be the 2-tuple'),
    ((torch.zeros(2, 3, 519),), 'rnn_state must be the 2-tuple'),
    (tuple(torch.zeros(2, 3, 519) for _ in range(3)), 'rnn_state must be the 2-tuple'),
    ((torch.zeros(2, 3, 519, dtype=torch.float64), torch.zeros(2, 3, 519)), 'rnn_state h must be float32'),
    ((torch.zeros(2, 3, 519), torch.zeros(1, 3, 519)), r'rnn_state c must be float32 \[2, 3, 519\]'),
    ((torch.zeros(2, 4, 519), torch.zeros(2, 4, 519)), r'rnn_state h must be float32 \[2, 3, 519\]'),
    ((torch.zeros(2, 3, 519), 'c'), 'rnn_state c must be float32'),
    ((torch.zeros(2, 3, 519), torch.zeros(2, 3, 519)), 'rnn_state h must be a CUDA tensor'),
])
def test_lstm_state_errors(state, match):
    net = AtariNet((4, 84, 84), 6, use_lstm=True)
    with pytest.raises(ValueError, match=match):
        net(_inputs(2, 3), state)


@pytest.mark.parametrize('done,match', [
    (torch.zeros(2, 3, dtype=torch.uint8), r"inputs\['done'\] must be bool \[2, 3\]"),
    (torch.zeros(3, 2, dtype=torch.bool), r"inputs\['done'\] must be bool \[2, 3\]"),
    (torch.zeros(2, 3), r"inputs\['done'\] must be bool"),
])
def test_lstm_done_errors(done, match):
    net = AtariNet((4, 84, 84), 6, use_lstm=True)
    state = tuple(torch.zeros(2, 3, 519) for _ in range(2))
    with pytest.raises(ValueError, match=match):
        net(_inputs(2, 3, done=done), state)


def test_lstm_missing_done_raises():
    net = AtariNet((4, 84, 84), 6, use_lstm=True)
    inputs = _inputs(2, 3)
    del inputs['done']
    with pytest.raises(ValueError, match=r"inputs\['done'\] must be bool"):
        net(inputs, tuple(torch.zeros(2, 3, 519) for _ in range(2)))
