"""The stand-alone encoder (srl_encoder_forward / srl_encoder_backward, the C ABI under the Ape-X learner and actor, the q-value
forward and the AtariNet drop-in) against an fp64 evaluation of each layer on the operands the GPU itself read (tests/layer_ref.py),
at every frame count its callers use, up to the MAX_FRAMES = 65536 it accepts.  These calls run with NF = NB = frames, which no
IMPALA shape of test_gpu_layer_exact.py reaches.

The criteria are test_gpu_layer_exact.py's:
  * xs is exactly the space-to-depth copy of the frames; core_out is exactly [h, clamp(reward), one_hot(action)]; dh (and its low
    twin) is exactly the bf16 split of dcore[:, :512] * (h > 0);
  * a1, a2, a3, da3, da2, da1: layer_ref.compare_stored (ReLU ties allowed), the dgrad grids' padding bit-exactly +0;
  * h: rel-L2 <= 2e-5 and normalised max error <= 1e-4 against fp64 fc on the GPU's own a3, with its k-block sensitivity;
  * the 8 gradients, per element: |got - ref| <= c 2^-24 S, S = sum |products| (layer_ref.abs_terms) and c = 2 (n + r): n the fp32
    additions one CTA chains into an accumulator (8 k-steps of 16 positions per 128-position chunk, times the chunks per CTA, times
    the 3 products hi*hi + hi*lo + lo*hi of the fp32-split mode; fc: its k-steps over all frames), r the partials the reduce adds
    after it, and the factor 2 an fp32 addition that truncates instead of rounding.  That is the worst case of the summation, so it
    grows with the chunks per CTA.  SENSITIVITY: the share of the reference that one part of the sum carries must exceed the bound
    (in L2 norm over the tensor).  Below 1024 frames the part is test_gpu_layer_exact's, one 128-position chunk of the middle CTA
    (fc: the middle 64-frame k-block).  From 1024 frames one chunk of a sum of up to 26M positions is smaller than the worst-case
    bound, and so is one CTA's share at the largest counts (conv1 at 65536 frames, fp32-split: one of 118 CTAs moves the reference by
    0.2 x the bound), so the part is the chunks of grid / 16 consecutive CTAs from the middle one on (fc: frames / 16 consecutive
    frames from the middle k-block on).

The fp64 reference runs on the device in float64, in blocks of FRAME_BLOCK frames: forward and data gradients are per frame, the
weight gradients and their S are summed over the blocks in fp64.  Every frame is compared, on the device; only error summaries come
back to the host.  The per-tensor rms that compare_stored's tie rule uses is that of the whole tensor (a first pass over the blocks).
Measured errors, err / bound, partitions, peak device memory and wall time go to $SRL_RESULTS_DIR/encoder_exact.json."""
import ctypes as C
import os
import time

import pytest
import torch

from oracle.impala_oracle import init_params
from scalerl_b200 import _lib
from tests import layer_ref as R
from tests.exact import NTOL, RTOL, SENS, U, Checker, record

pytestmark = pytest.mark.gpu
F64 = torch.float64
FRAME_BLOCK = 1024
LARGE = 1024                 # from here on the sensitivity share is 1/16 of the wgrad CTAs (fc: of the frames)
RESULTS = 'encoder_exact.json'
ENC_NAMES = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'fc.weight', 'fc.bias')

# each frame count sits on an edge of the kernels (A = 6)
COUNTS = {
    1: 'one frame: one partial tile everywhere; conv3 wgrad in one chunk on one CTA',
    2: 'two frames',
    3: 'three frames',
    7: 'a ragged fc M tile, conv1 positions not a multiple of 128',
    8: "conv1's 400 positions per frame fill 128-position chunks exactly",
    9: 'one frame past an exact conv1 chunk count',
    127: 'one frame short of the fc M tile',
    128: "the fc M tile; exact conv1 / conv2 / conv3 forward tiles (441, 81, 49 positions per frame)",
    129: 'cdiv(frames, 128) = 2: a second fc M tile with one row',
    256: 'APEX_Q_CHUNK, the q-value forward chunk',
    257: 'one frame past APEX_Q_CHUNK',
    512: "the Ape-X learner's tested batch",
    1500: "the Ape-X actor's tested env count",
    4096: 'every wgrad ring wraps many times',
    38043: 'xs just under 2^31 bytes',
    38044: 'xs just over 2^31 bytes (56,448 bytes per frame)',
    65535: 'MAX_FRAMES - 1',
    65536: 'MAX_FRAMES',
}
A_SWEEP_FRAMES = 129
ACTIONS = (1, 6, 18, 31)     # A changes only the core width 513 + A


def _hooks():
    return _lib.hooks()


class Encoder:
    """one srl_encoder context and its two caller-owned blocks for `frames` frames"""

    def __init__(self, frames, split):
        self.lib, self.frames, self.split = _lib.lib(), frames, split
        self.E = C.c_void_p()
        _lib.check(self.lib.srl_encoder_create(int(split), C.byref(self.E)), 'encoder_create')
        sb, kb = C.c_int64(), C.c_int64()
        _lib.check(self.lib.srl_encoder_sizes(frames, int(split), C.byref(sb), C.byref(kb)), 'encoder_sizes')
        self.saved = torch.empty(sb.value, dtype=torch.uint8, device='cuda')
        self.scratch = torch.empty(kb.value, dtype=torch.uint8, device='cuda')

    @staticmethod
    def block_bytes(frames, split):
        sb, kb = C.c_int64(), C.c_int64()
        _lib.check(_lib.lib().srl_encoder_sizes(frames, int(split), C.byref(sb), C.byref(kb)), 'encoder_sizes')
        return sb.value + kb.value

    def row(self, name, dtype):
        """(hi, lo) views of a named row of the blocks (srl_test_encoder_row: the library's own carving)"""
        hi, lo, n = C.c_void_p(), C.c_void_p(), C.c_int64()
        H = _hooks()
        rc = H.srl_test_encoder_row(self.frames, int(self.split), name.encode(), self.saved.data_ptr(), self.scratch.data_ptr(),
                                    C.byref(hi), C.byref(lo), C.byref(n))
        assert rc == 0, H.srl_test_last_error().decode()
        es = torch.empty(0, dtype=dtype).element_size()

        def view(p):
            if not p:
                return None
            for blk in (self.saved, self.scratch):
                off = p - blk.data_ptr()
                if 0 <= off and off + n.value * es <= blk.numel():
                    return blk[off:off + n.value * es].view(dtype)
            raise AssertionError(f'row {name} lies outside both blocks')
        return view(hi.value), view(lo.value)

    def forward(self, obs, reward, action, A, weights, core_out):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.srl_encoder_forward(self.E, obs.data_ptr(), reward.data_ptr(), action.data_ptr(), self.frames, A,
                                                (C.c_void_p * 8)(*[t.data_ptr() for t in weights]), self.saved.data_ptr(),
                                                self.scratch.data_ptr(), core_out.data_ptr(), st), 'encoder_forward')

    def backward(self, dcore, A, grads):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(self.lib.srl_encoder_backward(self.E, dcore.data_ptr(), self.frames, A, self.saved.data_ptr(), self.scratch.data_ptr(),
                                                 (C.c_void_p * 8)(*[t.data_ptr() for t in grads]), st), 'encoder_backward')

    def close(self):
        self.lib.srl_encoder_destroy(self.E)


def _blocks(F):
    return [(k, min(F, k + FRAME_BLOCK)) for k in range(0, F, FRAME_BLOCK)]


def _share_range(F, part, G):
    """grid positions [q0, q1) of the sensitivity share of a conv wgrad launch (q = frame * G * G + position)"""
    q0 = (part['grid'] // 2) * part['chunks_per_cta'] * 128
    n = max(1, part['grid'] // 16) * part['chunks_per_cta'] * 128 if F >= LARGE else 128
    return q0, min(q0 + n, F * G * G)


def _share_mask(k0, k1, G, q0, q1):
    q = torch.arange(k0 * G * G, k1 * G * G, device='cuda')
    return ((q >= q0) & (q < q1)).to(F64).view(k1 - k0, 1, G, G)


def wgrad_bound_c(F, part, split, fc=False):
    """c of the per-element weight-gradient bound c 2^-24 S: 2 (fp32 additions of one CTA's accumulator + partials reduced after it)"""
    prods = 3 if split else 1
    if fc:
        return 2 * ((F + 15) // 16 * prods + 1)
    return 2 * (part['chunks_per_cta'] * 8 * prods + part['grid'])


class Stored:
    """compare_stored over frame blocks, merged into one summary"""

    def __init__(self):
        self.parts, self.ss_err, self.ss_ref = [], 0.0, 0.0

    def add(self, st, ref):
        self.parts.append(st)
        r2 = float(ref.pow(2).sum())
        self.ss_err += st['rel_l2'] ** 2 * r2
        self.ss_ref += r2

    def merged(self):
        p = self.parts
        out = {'n': sum(s['n'] for s in p)}
        for k in ('mask_flips', 'beyond_1ulp_cancelled', 'bad', 'beyond_pair_precision'):
            if k in p[0]:
                out[k] = sum(s[k] for s in p)
        for k in ('worst_flip_margin', 'max_ulp', 'worst_bound_frac'):
            if k in p[0]:
                out[k] = max(s[k] for s in p)
        if 'mismatch_frac' in p[0]:
            out['mismatch_frac'] = sum(s['mismatch_frac'] * s['n'] for s in p) / max(out['n'], 1)
        out['rel_l2'] = (self.ss_err / max(self.ss_ref, 1e-300)) ** 0.5
        return out


def run_case(F, A, split, seed=0):
    """one forward + backward of the C-ABI encoder on F frames and every comparison; returns (Checker, record)"""
    t_start = time.time()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_alloc = torch.cuda.memory_allocated()
    g = torch.Generator(device='cuda').manual_seed(1000 * seed + F)
    params = init_params(A, seed=seed)
    weights = [params[n].cuda().contiguous() for n in ENC_NAMES]
    obs = torch.randint(0, 256, (F, 4, 84, 84), dtype=torch.uint8, device='cuda', generator=g)
    reward = torch.randn(F, device='cuda', generator=g) * 2
    action = torch.randint(0, A, (F,), device='cuda', generator=g)
    # mostly positive: the gradient sums add up instead of cancelling, so a left-out share moves them measurably
    dcore = torch.randn(F, 513 + A, device='cuda', generator=g) + 1.0
    core_out = torch.empty(F, 513 + A, device='cuda')
    grads = [torch.empty_like(w) for w in weights]
    enc = Encoder(F, split)
    try:
        enc.forward(obs, reward, action, A, weights, core_out)
        enc.backward(dcore, A, grads)
        torch.cuda.synchronize()
        rows = {n: enc.row(n, torch.float32 if n == 'h' else torch.bfloat16) for n in ('xs', 'a1', 'a2', 'a3', 'h', 'dh', 'da3', 'da2', 'da1')}
        C_ = check(F, A, split, obs, reward, action, dcore, core_out, grads, params, rows)
    finally:
        enc.close()
    torch.cuda.synchronize()
    rec = dict(C_.res, frames=F, A=A, precision='fp32_split' if split else 'bf16', wall_s=time.time() - t_start,
               peak_device_bytes=torch.cuda.max_memory_allocated() - base_alloc,
               encoder_block_bytes=Encoder.block_bytes(F, split))
    return C_, rec


def check(F, A, split, obs, reward, action, dcore, core_out, grads, params, rows):
    ck = Checker(RESULTS)
    W = {k: tuple(None if t is None else t.cuda() for t in v) for k, v in R.weights(params, split).items()}
    bias = {k: params[k].cuda() for k in ('conv1.bias', 'conv2.bias', 'conv3.bias', 'fc.bias')}
    ctas = R.cta_counts(R.sm_count(), os.environ)
    parts = R.wgrad_partitions(F, ctas, split)
    get = lambda n: rows[n][0]
    lo = lambda n: rows[n][1] if split else None
    pl = lambda t, k0, k1, per: None if t is None else t.view(F, per)[k0:k1]

    # ---- exact outputs: xs, core_out, dh
    h_all = get('h').view(F, 512)
    xs_bad = dh_bad = 0
    for k0, k1 in _blocks(F):
        xs_bad += int((get('xs').view(F, 21, 21, 64)[k0:k1] != R.s2d(obs[k0:k1]).to(torch.bfloat16)).sum())
        v = torch.where(h_all[k0:k1] > 0, dcore[k0:k1, :512], torch.zeros((), device='cuda'))
        hi = v.to(torch.bfloat16)
        dh_bad += int((get('dh').view(F, 512)[k0:k1].view(torch.int16) != hi.view(torch.int16)).sum())
        if split:
            dh_bad += int((lo('dh').view(F, 512)[k0:k1].view(torch.int16) != (v - hi.float()).to(torch.bfloat16).view(torch.int16)).sum())
    ck.res['xs_mismatches'], ck.res['dh_mismatches'] = xs_bad, dh_bad
    if xs_bad:
        ck.fails.append(f'xs: {xs_bad} elements are not the space-to-depth copy of the frames')
    if dh_bad:
        ck.fails.append(f'dh: {dh_bad} elements are not the bf16 split of dcore * (h > 0)')
    want_core = torch.cat([h_all, reward.clamp(-1, 1).view(F, 1), torch.nn.functional.one_hot(action, A).float()], 1)
    core_bad = int((core_out.view(torch.int32) != want_core.view(torch.int32)).sum())
    ck.res['core_out_mismatches'] = core_bad
    if core_bad:
        ck.fails.append(f'core_out: {core_bad} elements are not [h, clamp(reward, -1, 1), one_hot(action)]')

    # ---- per-block references
    def a_pair(name, k0, k1, H):
        if name == 'a1':
            f = lambda t: None if t is None else R.a1_planes_to_nchw(t.view(2, F, 6400)[:, k0:k1].reshape(-1), k1 - k0)
        else:
            f = lambda t: None if t is None else R.nhwc_to_nchw(t.view(F, -1)[k0:k1], k1 - k0, H)
        return f(get(name)), f(lo(name))

    def forward_refs(k0, k1):
        n = k1 - k0
        a1 = a_pair('a1', k0, k1, 20)
        a2 = a_pair('a2', k0, k1, 9)
        a3 = a_pair('a3', k0, k1, 7)
        z1 = R.conv1_fwd(obs[k0:k1], W['conv1.weight'], bias['conv1.bias'])
        z2 = R.conv_fwd(R.pair(*a1), W['conv2.weight'], bias['conv2.bias'], 2)
        z3 = R.conv_fwd(R.pair(*a2), W['conv3.weight'], bias['conv3.bias'], 1)
        return {'a1': (a1, z1), 'a2': (a2, z2), 'a3': (a3, z3)}, (a1, a2, a3, n)

    def backward_refs(k0, k1, acts):
        a1, a2, a3, n = acts
        a1p, a2p, a3p = R.pair(*a1), R.pair(*a2), R.pair(*a3)
        dhp = R.pair(get('dh').view(F, 512)[k0:k1], None if not split else lo('dh').view(F, 512)[k0:k1])
        mask3 = (a3[0] > 0).to(F64)
        dWf, dbf, da3 = R.fc_bwd(dhp, a3p, W['fc.weight'], mask3)
        dterms = R.abs_terms(lambda d, w: d @ w, dhp, W['fc.weight']).reshape(-1, 64, 7, 7) * mask3
        out = {'fc': (dWf, dbf, dhp, a3p), 'stored': []}
        dref = da3
        layers = (('conv3', 'da3', 9, 7, 64, a2p, a2, 1, 1.0), ('conv2', 'da2', 10, 9, 64, a1p, a1, 2, 1.0),
                  ('conv1', 'da1', 21, 20, 32, (obs[k0:k1].to(F64), None), None, 4, 1.0 / 255.0))
        for name, dname, G, V, Cch, xp, xs, stride, scale in layers:
            dy_hi, pad = R.grid_to_nchw(pl(get(dname), k0, k1, G * G * Cch), n, G, V, Cch)
            dy_lo, pad_lo = (None, None) if not split else R.grid_to_nchw(pl(lo(dname), k0, k1, G * G * Cch), n, G, V, Cch)
            out['stored'].append((dname, dy_hi, dy_lo, dref, dterms, pad, pad_lo))
            dyp = R.pair(dy_hi, dy_lo)
            mask = None if xs is None else (xs[0] > 0).to(F64)
            dW, db, dx = R.conv_bwd(xp, dyp, W[f'{name}.weight'], stride, mask, scale)
            out[name] = (dW, db, dyp, xp, G, V, stride, scale)
            dref = dx
            if mask is not None:
                dterms = R.abs_terms(lambda d, w: torch.nn.grad.conv2d_input(xp[0].shape, w, d, stride=stride), dyp, W[f'{name}.weight']) * mask
        return out

    # pass 1: the rms of every stored tensor's reference and pre-activation over all frames
    ss = {}
    for k0, k1 in _blocks(F):
        fw, acts = forward_refs(k0, k1)
        for name, (_, z) in fw.items():
            ss[name + '_pre'] = ss.get(name + '_pre', 0.0) + float(z.pow(2).sum())
            ss[name] = ss.get(name, 0.0) + float(z.clamp_min(0).pow(2).sum())
        for dname, _, _, dref, _, _, _ in backward_refs(k0, k1, acts)['stored']:
            ss[dname] = ss.get(dname, 0.0) + float(dref.pow(2).sum())
    numel = {'a1': 12800, 'a2': 81 * 64, 'a3': 49 * 64, 'da3': 49 * 64, 'da2': 81 * 64, 'da1': 400 * 32}
    rms = {k: (v / (F * numel[k.replace('_pre', '')])) ** 0.5 for k, v in ss.items()}

    # pass 2: compare every block; sum the weight gradients, their S and the sensitivity shares in fp64
    stored = {n: Stored() for n in ('a1', 'a2', 'a3', 'da3', 'da2', 'da1')}
    pad_nonzero = {}
    hsum = {'err2': 0.0, 'ref2': 0.0, 'maxerr': 0.0, 'maxref': 0.0, 'sens2': 0.0}
    acc = {}
    kb = ((F + 63) // 64 // 2) * 64                                     # the middle 64-frame k-block
    ke = min(F, kb + (64 if F < LARGE else F // 16))
    share_q = {name: _share_range(F, parts[name], G) for name, G in (('conv3', 9), ('conv2', 10), ('conv1', 21))}

    def add(key, t):
        acc[key] = t.clone() if key not in acc else acc[key] + t

    for k0, k1 in _blocks(F):
        fw, acts = forward_refs(k0, k1)
        for name, ((hi, lo_), z) in fw.items():
            stored[name].add(R.compare_stored(hi, lo_, z.clamp_min(0), pre=z, rms_ref=rms[name], rms_pre=rms[name + '_pre']), z.clamp_min(0))
        # h: fp32 bounds of fc on the GPU's own a3, and the middle 64-channel k-block as its sensitivity
        a3p = R.pair(*acts[2])
        zh = R.fc_fwd(a3p, W['fc.weight'], bias['fc.bias'])
        idx = torch.arange(64, device='cuda') * 49 + 24
        kblk = R.sp(lambda a, w: a.reshape(k1 - k0, -1)[:, idx] @ w[:, idx].t(), a3p, W['fc.weight'])
        href = zh.clamp_min(0)
        d = h_all[k0:k1].to(F64) - href
        hsum['err2'] += float(d.pow(2).sum())
        hsum['ref2'] += float(href.pow(2).sum())
        hsum['maxerr'] = max(hsum['maxerr'], float(d.abs().max()))
        hsum['maxref'] = max(hsum['maxref'], float(href.abs().max()))
        hsum['sens2'] += float(((zh - kblk).clamp_min(0) - href).pow(2).sum())
        bw = backward_refs(k0, k1, acts)
        for dname, dy_hi, dy_lo, dref, dterms, pad, pad_lo in bw['stored']:
            stored[dname].add(R.compare_stored(dy_hi, dy_lo, dref, terms=dterms, rms_ref=rms[dname]), dref)
            pad_nonzero[dname] = pad_nonzero.get(dname, 0) + int((pad.contiguous().view(torch.int16) != 0).sum())
            if pad_lo is not None:
                pad_nonzero[dname + '_lo'] = pad_nonzero.get(dname + '_lo', 0) + int((pad_lo.contiguous().view(torch.int16) != 0).sum())
        # fc weight gradient, its S and its share (the frames [kb, ke))
        dWf, dbf, dhp, a3p_ = bw['fc']
        flat = tuple(None if t is None else t.reshape(t.shape[0], -1) for t in a3p_)
        add('fc.weight', dWf)
        add('fc.bias', dbf)
        add('S fc.weight', R.abs_terms(lambda dd, x: dd.t() @ x, dhp, flat))
        add('S fc.bias', R.psum((dhp[0].abs(), None if dhp[1] is None else dhp[1].abs()), 0))
        s0, s1 = max(kb, k0), min(ke, k1)
        if s0 < s1:
            sl = lambda p: tuple(None if t is None else t[s0 - k0:s1 - k0] for t in p)
            add('share fc.weight', R.sp(lambda dd, x: dd.t() @ x, sl(dhp), sl(flat)))
            add('share fc.bias', R.psum(sl(dhp), 0))
        for name in ('conv3', 'conv2', 'conv1'):
            dW, db, dyp, xp, G, V, stride, scale = bw[name]
            wshape = W[f'{name}.weight'][0].shape
            add(f'{name}.weight', dW)
            add(f'{name}.bias', db)
            ab = lambda p: (p[0].abs(), None if p[1] is None else p[1].abs())
            add(f'S {name}.weight', R.abs_terms(lambda a, dd: torch.nn.grad.conv2d_weight(a, wshape, dd, stride=stride), xp, dyp) * scale)
            add(f'S {name}.bias', R.psum(ab(dyp), (0, 2, 3)))
            q0, q1 = share_q[name]
            if q0 < k1 * G * G and q1 > k0 * G * G:
                m = _share_mask(k0, k1, G, q0, q1)[:, :, :V, :V]
                dym = (dyp[0] * m, None if dyp[1] is None else dyp[1] * m)
                pW, pb, _ = R.conv_bwd(xp, dym, W[f'{name}.weight'], stride, None, scale)
                add(f'share {name}.weight', pW)
                add(f'share {name}.bias', pb)

    # ---- verdicts
    for name, s in stored.items():
        st = s.merged()
        ck.res[name] = st
        if not R.stored_ok(st, split):
            ck.fails.append(f'{name}: {st}')
    for name, n in pad_nonzero.items():
        ck.res[name + '_padding_nonzero'] = n
        if n:
            ck.fails.append(f'{name}: {n} padding elements are not +0.0')
    he = {'rel_l2': (hsum['err2'] / max(hsum['ref2'], 1e-300)) ** 0.5, 'nerr': hsum['maxerr'] / max(hsum['maxref'], 1e-300),
          'sensitivity': (hsum['sens2'] / max(hsum['ref2'], 1e-300)) ** 0.5}
    ck.res['h'] = he
    if not (he['rel_l2'] <= RTOL and he['nerr'] <= NTOL):
        ck.fails.append(f'h: {he}')
    if he['sensitivity'] < SENS * RTOL:
        ck.fails.append(f'h: one left-out k-block moves the reference by {he["sensitivity"]:.2e} < {SENS} x {RTOL:.0e}')
    wres = {}
    for i, k in enumerate(ENC_NAMES):
        layer = k.split('.')[0]
        c = wgrad_bound_c(F, parts.get(layer), split, fc=layer == 'fc')
        ref, S, share = acc[k], acc['S ' + k], acc.get('share ' + k)
        got = grads[i].to(F64).reshape(ref.shape)
        bound = c * U * S + 1e-300
        e = (got - ref).abs()
        r = {'c': c, 'err_over_bound': float((e / bound).max()), 'rel_l2': R.rel_l2(got, ref), 'nerr': R.nerr(got, ref),
             'sensitivity': float(share.norm() / bound.norm()) if share is not None else 0.0,
             'bound_over_ref_l2': float(bound.norm() / max(float(ref.norm()), 1e-300))}
        wres[k] = r
        if not r['err_over_bound'] <= 1.0:
            ck.fails.append(f'{k}: error {r["err_over_bound"]:.3g} x the bound c 2^-24 S (c = {c})')
        if not r['sensitivity'] > 1.0:
            ck.fails.append(f'{k}: the left-out share moves the reference by only {r["sensitivity"]:.3g} x the bound (c = {c})')
    ck.res['grads'] = wres
    ck.res['partition'] = parts
    ck.res['share'] = {'fc_frames': [kb, ke], **{n: list(q) for n, q in share_q.items()}, 'kind': 'grid / 16 CTAs' if F >= LARGE else 'one chunk'}
    return ck


def _need_bytes(F, split, A=6):
    """device bytes one case allocates: the encoder's blocks, its inputs and outputs, and the fp64 reference's working set"""
    return Encoder.block_bytes(F, split) + F * (28224 + 2 * (513 + A) * 4 + 12) + (4 << 30)


def _run_and_check(F, A, split):
    need = _need_bytes(F, split, A)
    free, total = torch.cuda.mem_get_info()
    if need > free:
        record(RESULTS, f'F{F}_A{A}_{"split" if split else "bf16"}', {'skipped': True, 'need_bytes': need, 'free_bytes': free})
        pytest.skip(f'needs about {need / 2**30:.1f} GiB of device memory, {free / 2**30:.1f} GiB free')
    ck, rec = run_case(F, A, split)
    record(RESULTS, f'F{F}_A{A}_{"split" if split else "bf16"}', rec)
    print(f'F={F} A={A} split={split}: peak {rec["peak_device_bytes"] / 2**30:.2f} GiB, {rec["wall_s"]:.1f} s, '
          + ', '.join(f'{k} {v["err_over_bound"]:.3g}' for k, v in rec['grads'].items()))
    assert not ck.fails, '\n'.join(ck.fails)


@pytest.mark.parametrize('precision', ['bf16', 'fp32_split'])
@pytest.mark.parametrize('frames', list(COUNTS))
def test_encoder_exact(frames, precision):
    torch.cuda.empty_cache()
    _run_and_check(frames, 6, precision == 'fp32_split')


@pytest.mark.parametrize('precision', ['bf16', 'fp32_split'])
@pytest.mark.parametrize('A', ACTIONS)
def test_encoder_exact_core_width(A, precision):
    _run_and_check(A_SWEEP_FRAMES, A, precision == 'fp32_split')


def test_frame_counts_reach_every_partition_regime():
    """the frame-count table drives srl_encoder_backward's three wgrad launches through all four partition regimes"""
    ctas = R.cta_counts(R.sm_count(), os.environ)
    seen, table = set(), []
    for F in COUNTS:
        for split in (False, True):
            for name, p in R.wgrad_partitions(F, ctas, split).items():
                table.append({'frames': F, 'split': split, 'layer': name, **p})
                seen.update(k for k, v in R.regimes(p).items() if v)
    record(RESULTS, 'partition_regimes', {'ctas': ctas, 'table': table, 'reached': sorted(seen)})
    # below LARGE the sensitivity share is test_gpu_layer_exact's: the first chunk of the middle CTA
    for F in (f for f in COUNTS if f < LARGE):
        for name, G in (('conv3', 9), ('conv2', 10), ('conv1', 21)):
            p = R.wgrad_partitions(F, ctas, False)[name]
            n0, n1, m = R.mid_chunk_frames(F, G, p)
            q0, q1 = _share_range(F, p, G)
            assert torch.equal(_share_mask(n0, n1, G, q0, q1).cpu(), m), (F, name)
    assert seen == {'one_chunk_per_cta', 'within_ring', 'ring_wraps_twice', 'last_cta_single_chunk'}, sorted(seen)


def test_encoder_row_hook_is_the_library_carving():
    """srl_test_encoder_row names the rows where the library put them: 256-byte-aligned rows of the sizes encoder_rows gives, each
    low twin (fp32-split mode only) right after its row"""
    F = 300
    rows = (('xs', torch.bfloat16, F * 441 * 64), ('a1', torch.bfloat16, F * 400 * 32), ('a2', torch.bfloat16, F * 81 * 64),
            ('a3', torch.bfloat16, F * 49 * 64), ('h', torch.float32, F * 512), ('dh', torch.bfloat16, F * 512),
            ('da3', torch.bfloat16, F * 81 * 64), ('da2', torch.bfloat16, F * 100 * 64), ('da1', torch.bfloat16, F * 441 * 32))
    for split in (False, True):
        enc = Encoder(F, split)
        try:
            for name, dt, n in rows:
                hi, lo = enc.row(name, dt)
                assert hi.numel() == n and hi.data_ptr() % 256 == 0, name
                assert (lo is not None) == (split and name not in ('xs', 'h')), name
                if lo is not None:
                    assert lo.data_ptr() - hi.data_ptr() == (n * 2 + 255) // 256 * 256, name
        finally:
            enc.close()
