"""The per-layer fp64 references (tests/layer_ref.py) are right before any GPU time is spent on them: the layout converters
round-trip, the chained references reproduce torch.autograd of an fp64 AtariNet, the split-operand emulation reduces to the
plain product, and the wgrad partition arithmetic mirrors res_wgrad_launch_t."""
import pytest
import torch

from oracle import impala_oracle as O
from tests import layer_ref as R


def test_converters_round_trip():
    g = torch.Generator().manual_seed(0)
    N, NFS = 3, 5
    obs = torch.randint(0, 256, (N, 4, 84, 84), generator=g, dtype=torch.uint8)
    xs = R.s2d(obs)
    assert xs.shape == (N, 21, 21, 64)
    assert torch.equal(R.xs_to_frames(xs, N), obs)
    # xs[n][Y][X][c*16 + dy*4 + dx] = obs[n][c][4Y+dy][4X+dx]   (encoder.cu obs_s2d_kernel)
    assert xs[1, 5, 7, 2 * 16 + 3 * 4 + 1] == obs[1, 2, 4 * 5 + 3, 4 * 7 + 1]
    a1 = torch.randn(N, 32, 20, 20, generator=g)
    planes = R.nchw_to_a1_planes(a1, NFS)
    assert planes.numel() == 2 * NFS * 100 * 64
    assert torch.equal(R.a1_planes_to_nchw(planes, N, NFS), a1)
    # plane hp = h & 1, row n*100 + (h>>1)*10 + (w>>1), channel (w&1)*32 + c  (res_problems.cuh)
    n, c, h, w = 2, 17, 13, 6
    assert planes[(((h & 1) * NFS + n) * 100 + (h >> 1) * 10 + (w >> 1)) * 64 + (w & 1) * 32 + c] == a1[n, c, h, w]
    assert float(planes.view(2, NFS, -1)[:, N:].abs().sum()) == 0.0
    for H in (9, 7):
        x = torch.randn(N, 64, H, H, generator=g)
        assert torch.equal(R.nhwc_to_nchw(R.nchw_to_nhwc(x), N, H), x)
    for G, V, C in ((9, 7, 64), (10, 9, 64), (21, 20, 32)):
        x = torch.randn(N, C, V, V, generator=g)
        grid = R.nchw_to_grid(x, G)
        assert grid.numel() == N * G * G * C
        back, pad = R.grid_to_nchw(grid, N, G, V, C)
        assert torch.equal(back, x) and pad.numel() == N * (G * G - V * V) * C and float(pad.abs().sum()) == 0.0
        assert grid[((1 * G + 2) * G + 3) * C + 5] == x[1, 5, 2, 3]


def _chain(params, obs, reward, action, dl, dv):
    """the per-layer references chained on their own fp64 outputs (no rounding, no low twins)"""
    P = {k: (v, None) for k, v in params.items()}
    N, NB, A = obs.shape[0], dl.shape[0], dl.shape[1]
    z1 = R.conv1_fwd(obs, P['conv1.weight'], params['conv1.bias'])
    a1 = z1.clamp_min(0)
    z2 = R.conv_fwd((a1, None), P['conv2.weight'], params['conv2.bias'], 2)
    a2 = z2.clamp_min(0)
    z3 = R.conv_fwd((a2, None), P['conv3.weight'], params['conv3.bias'], 1)
    a3 = z3.clamp_min(0)
    h = R.fc_fwd((a3, None), P['fc.weight'], params['fc.bias']).clamp_min(0)
    c = R.core(h, reward, action, A)
    logits, baseline = R.heads_fwd(c, params)
    g = R.head_grads(dl, dv, c[:NB])
    dh = R.dh_ref(dl, dv, h[:NB], params)
    g['fc.weight'], g['fc.bias'], da3 = R.fc_bwd((dh, None), (a3[:NB], None), P['fc.weight'], (a3[:NB] > 0).double())
    g['conv3.weight'], g['conv3.bias'], da2 = R.conv_bwd((a2[:NB], None), (da3, None), P['conv3.weight'], 1, (a2[:NB] > 0).double())
    g['conv2.weight'], g['conv2.bias'], da1 = R.conv_bwd((a1[:NB], None), (da2, None), P['conv2.weight'], 2, (a1[:NB] > 0).double())
    g['conv1.weight'], g['conv1.bias'], _ = R.conv_bwd((obs[:NB].double(), None), (da1, None), P['conv1.weight'], 4, None, 1.0 / 255.0)
    return logits, baseline, g, {'dh': dh, 'da3': da3, 'da2': da2, 'da1': da1}


@pytest.mark.parametrize('A', [6, 18])
def test_chained_references_equal_autograd_fp64(A):
    T1, B, NB = 2, 2, 3               # 4 frames, the first 3 learn
    batch = O.synthetic_batch(T1 - 1, B, A, seed=4)
    params = {k: v.double() for k, v in O.init_params(A, seed=3).items()}
    obs = batch['obs'].reshape(-1, 4, 84, 84)
    N = obs.shape[0]
    g = torch.Generator().manual_seed(1)
    dl, dv = torch.randn(NB, A, generator=g, dtype=torch.float64), torch.randn(NB, generator=g, dtype=torch.float64)
    ps = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    lg, bs, saved = O.atari_forward(ps, batch['obs'], batch['reward'], batch['action'], keep=True)
    for k in ('a1', 'a2', 'a3', 'h'):
        saved[k].retain_grad()
    lg, bs = lg.reshape(N, A), bs.reshape(N)
    ((lg[:NB] * dl).sum() + (bs[:NB] * dv).sum()).backward()
    logits, baseline, grads, d = _chain(params, obs, batch['reward'].reshape(-1), batch['action'].reshape(-1), dl, dv)
    assert R.rel_l2(logits, lg.detach()) < 1e-12 and R.rel_l2(baseline, bs.detach()) < 1e-12
    for k in O.PARAM_ORDER:
        assert R.rel_l2(grads[k].reshape(ps[k].shape), ps[k].grad) < 1e-12, k
    # input gradients of every layer: dh / da3 / da2 / da1 are d(loss)/d(pre-activation) = d(loss)/d(output) * (output > 0)
    for name, k in (('dh', 'h'), ('da3', 'a3'), ('da2', 'a2'), ('da1', 'a1')):
        want = (saved[k].grad * (saved[k] > 0))[:NB]
        assert R.rel_l2(d[name].reshape(want.shape), want) < 1e-12, name


def test_split_emulation():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(3, 32, 20, 20, generator=g)
    w = torch.randn(64, 32, 4, 4, generator=g)
    xh, xl = R.split(x)
    wh, wl = R.split(w)
    f = lambda a, b: torch.nn.functional.conv2d(a, b, stride=2)
    plain = f(xh.double(), wh.double())
    zero = torch.zeros_like(xl)
    # lo = 0 (or no low twin at all): exactly the plain product
    assert torch.equal(R.sp(f, R.pair(xh, zero), R.pair(wh, torch.zeros_like(wl))), plain)
    assert torch.equal(R.sp(f, R.pair(xh), R.pair(wh)), plain)
    # full split: (hi + lo)(hi + lo) - lo*lo
    full = R.sp(f, R.pair(xh, xl), R.pair(wh, wl))
    want = f(xh.double() + xl.double(), wh.double() + wl.double()) - f(xl.double(), wl.double())
    assert R.rel_l2(full, want) < 1e-13
    # the pair carries 16 significant bits: hi + lo is within 2^-16 of the fp32 value
    assert float(((xh.double() + xl.double() - x.double()).abs() / x.double().abs()).max()) < 2.0 ** -16
    assert torch.equal(R.psum(R.pair(xh, xl), (0, 2, 3)), xh.double().sum((0, 2, 3)) + xl.double().sum((0, 2, 3)))


def test_compare_stored_counts_ulps_and_ties():
    ref = torch.tensor([1.0, -2.0, 3.0, 0.5, 1e-3], dtype=torch.float64)
    hi = ref.to(torch.bfloat16)
    st = R.compare_stored(hi, None, ref)
    assert st['max_ulp'] == 0 and st['mismatch_frac'] == 0.0 and R.stored_ok(st, False)
    one = hi.clone().view(torch.int16)
    one[2] += 1
    st = R.compare_stored(one.view(torch.bfloat16), None, ref)
    assert st['max_ulp'] == 1 and st['mismatch_frac'] == 0.2 and not R.stored_ok(st, False)       # 1 of 5 > 0.5 %
    two = hi.clone().view(torch.int16)
    two[0] += 2
    assert R.compare_stored(two.view(torch.bfloat16), None, ref)['max_ulp'] == 2
    # ReLU: a unit the GPU zeroed is fine only at a tie
    pre = torch.tensor([1.0, 2.0, -1.0, 1e-9], dtype=torch.float64)
    got = torch.tensor([1.0, 2.0, 0.0, 0.0]).to(torch.bfloat16)
    st = R.compare_stored(got, None, pre.clamp_min(0), pre=pre)
    assert st['mask_flips'] == 1 and st['worst_flip_margin'] < R.TIE and R.stored_ok(st, False)
    got[1] = 0.0
    assert not R.stored_ok(R.compare_stored(got, None, pre.clamp_min(0), pre=pre), False)
    # split mode: hi + lo against the fp64 value
    v = torch.tensor([1.2345678, -3.3e-3, 7.0], dtype=torch.float64)
    h, l = R.split(v)
    assert R.stored_ok(R.compare_stored(h, l, v), True)
    assert not R.stored_ok(R.compare_stored(h, torch.zeros_like(l), v), True)


def test_wgrad_partition_mirrors_the_launch():
    # ring depths of ResWgradCfg<P, SPLIT>::STAGES (227 KB of shared memory)
    assert [R.wgrad_ring_depth(n, s) for n in ('conv3', 'conv2', 'conv1') for s in (False, True)] == [3, 2, 3, 1, 5, 3]
    ctas = R.cta_counts(132, {})
    assert ctas == {'persistent': 132, 'bwd': 118, 'side_wgrad': 64}
    p = R.wgrad_partitions(640, ctas, False)            # T=20, B=32
    assert p['conv3'] == {'chunks': 405, 'chunks_per_cta': 7, 'grid': 58, 'last_cta_chunks': 6, 'ring': 3}
    assert p['conv1'] == {'chunks': 2205, 'chunks_per_cta': 19, 'grid': 117, 'last_cta_chunks': 1, 'ring': 5}
    assert R.regimes(p['conv3'])['ring_wraps_twice'] and R.regimes(p['conv1'])['last_cta_single_chunk']
    # out-of-range overrides fall back like encoder.cu does
    assert R.cta_counts(132, {'SRL_WGRAD_CTAS': '4', 'SRL_BWD_CTAS': '8', 'SRL_PERSISTENT_CTAS': '200'}) == ctas
    assert R.cta_counts(132, {'SRL_WGRAD_CTAS': '8', 'SRL_BWD_CTAS': '16', 'SRL_PERSISTENT_CTAS': '16'}) == {'persistent': 16, 'bwd': 16, 'side_wgrad': 8}
    assert R.wgrad_partitions(640, {'side_wgrad': 8, 'bwd': 16, 'persistent': 16}, False)['conv3']['chunks_per_cta'] == 51
    assert R.wgrad_partition(81, 64) == {'chunks': 1, 'chunks_per_cta': 1, 'grid': 1, 'last_cta_chunks': 1}
