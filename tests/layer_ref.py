"""Per-layer fp64 references of the learner step, evaluated on the operands the GPU itself read (CPU only).

Every kernel of the encoder and the heads is checked on its own: the bf16 inputs a kernel read (debug buffers of the learner,
weights = the bf16 rounding of the fp32 masters, ReLU masks = (a > 0) of the GPU's own activations) go into an fp64 evaluation
of that one operation, and the result is compared with what the kernel wrote.  No rounding difference of an earlier layer
carries over, so the tolerances are those of one fp32 accumulation.

Layouts (res_problems.cuh, tma_problems.cuh, kernels.h).  NF = (T+1)B frames, NB = TB learning frames = the FIRST NB rows
(time steps 0..T-1: the logits of the last time step only bootstrap V-trace, api.cu fb_begin / column_step_kernel):
  xs    [NF][21][21][64]             space-to-depth frame, channel = (c, dy, dx)
  a1    [2][NFS][10][10][64]         row-parity planes hp = h & 1; channel = (w & 1) * 32 + c; NFS = the context's NF
  a2    [NF][9][9][64], a3 [NF][7][7][64]   NHWC
  da3g  [NB][9][9][64]               zeros outside the 7x7 outputs
  da2g  [NB][10][10][64]             zeros outside 9x9
  da1g  [NB][21][21][32]             zeros outside 20x20
  dh    [NB][512]

fp32-accurate split mode (precision = 'fp32_split'): every bf16 operand v has a low twin bf16(v - bf16(v)) and every kernel
issues hi*hi + hi*lo + lo*hi into one fp32 accumulator (igemm_res.cuh res_fwd_kernel / res_wgrad_consumer, igemm_tma.cuh
igemm_tma_kernel); the u8 frames are exact and have no low twin.  `sp` evaluates exactly those three products.
"""
import torch
import torch.nn.functional as F

F64 = torch.float64
TIE = 1e-5            # |pre-activation| < TIE * rms: a genuine tie, either side of the ReLU is right


# ------------------------------------------------------------------------------------------------ layout converters
def s2d(obs):
    """u8 / float frames [N,4,84,84] -> xs layout [N,21,21,64], channel (c,dy,dx)"""
    N = obs.shape[0]
    return obs.reshape(N, 4, 21, 4, 21, 4).permute(0, 2, 4, 1, 3, 5).reshape(N, 21, 21, 64)


def xs_to_frames(xs, N):
    return xs.reshape(N, 21, 21, 4, 4, 4).permute(0, 3, 1, 4, 2, 5).reshape(N, 4, 84, 84)


def a1_planes_to_nchw(flat, N, NFS=None):
    """a1 [hp][n][h>>1][w>>1][(w&1)*32 + c] (planes strided by NFS frames) -> [N,32,20,20]"""
    NFS = N if NFS is None else NFS
    t = flat.reshape(2, NFS, 10, 10, 2, 32)[:, :N]          # hp, n, h2, w2, wp, c
    return t.permute(1, 5, 2, 0, 3, 4).reshape(N, 32, 20, 20)


def nchw_to_a1_planes(x, NFS=None):
    N = x.shape[0]
    NFS = N if NFS is None else NFS
    out = torch.zeros(2, NFS, 10, 10, 2, 32, dtype=x.dtype)
    out[:, :N] = x.reshape(N, 32, 10, 2, 10, 2).permute(3, 0, 2, 4, 5, 1)
    return out.reshape(-1)


def nhwc_to_nchw(flat, N, H, C=64):
    return flat.reshape(N, H, H, C).permute(0, 3, 1, 2)


def nchw_to_nhwc(x):
    return x.permute(0, 2, 3, 1).reshape(-1)


def grid_to_nchw(flat, N, G, V, C=64):
    """zero-padded grid layout [N][G][G][C] -> the valid [N,C,V,V] and the padding elements (which must be exactly zero)"""
    t = flat.reshape(N, G, G, C)
    pad = torch.cat([t[:, V:, :, :].reshape(-1), t[:, :V, V:, :].reshape(-1)])
    return t[:, :V, :V, :].permute(0, 3, 1, 2), pad


def nchw_to_grid(x, G):
    N, C, V, _ = x.shape
    out = torch.zeros(N, G, G, C, dtype=x.dtype)
    out[:, :V, :V, :] = x.permute(0, 2, 3, 1)
    return out.reshape(-1)


# ------------------------------------------------------------------------------------------------ operands
def split(x):
    """fp32 value -> (hi, lo) bf16 pair as the kernels store it: hi = bf16(v), lo = bf16(v - hi)"""
    x = x.float()
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


def pair(hi, lo=None):
    return hi.to(F64), (None if lo is None else lo.to(F64))


def weights(params, split_mode):
    """the GEMM weight operands: bf16(master) (bit-equal to the packed copies), and in the split mode the low twins"""
    out = {}
    for k in ('conv1.weight', 'conv2.weight', 'conv3.weight', 'fc.weight'):
        hi, lo = split(params[k])
        out[k] = pair(hi, lo if split_mode else None)
    return out


def sp(f, a, b):
    """f(a_hi, b_hi) + f(a_hi, b_lo) + f(a_lo, b_hi): the products a kernel issues (a missing low twin contributes nothing)"""
    (ah, al), (bh, bl) = a, b
    out = f(ah, bh)
    if bl is not None:
        out = out + f(ah, bl)
    if al is not None:
        out = out + f(al, bh)
    return out


def psum(p, dims):
    hi, lo = p
    return hi.sum(dims) + (0 if lo is None else lo.sum(dims))


# ------------------------------------------------------------------------------------------------ forward (pre-activations)
def conv1_fwd(frames, W1, b1):
    """z1 = conv1(u8 frames, W1) * (1/255) + b1 (res_problems.cuh RConv1Fwd: the 1/255 is applied to the accumulator)"""
    return sp(lambda x, w: F.conv2d(x, w, stride=4), (frames.to(F64), None), W1) / 255.0 + b1.to(F64).view(1, -1, 1, 1)


def conv_fwd(x, W, b, stride):
    return sp(lambda a, w: F.conv2d(a, w, stride=stride), x, W) + b.to(F64).view(1, -1, 1, 1)


def fc_fwd(a3, Wfc, bfc):
    """z_h = a3 . Wfc^T + bfc; a3 as NCHW [N,64,7,7] -- flattened (c,h,w) = fc.weight's column order"""
    flat = tuple(None if t is None else t.reshape(t.shape[0], -1) for t in a3)
    return sp(lambda a, w: a @ w.t(), flat, Wfc) + bfc.to(F64)


def core(h, reward, action, A):
    """core = [h, clamp(reward, -1, 1), one_hot(action)] (heads.cu head_fwd_kernel)"""
    N = h.shape[0]
    return torch.cat([h.to(F64), reward.reshape(N, 1).to(F64).clamp(-1, 1),
                      F.one_hot(action.reshape(N), A).to(F64)], 1)


def heads_fwd(c, params):
    logits = c @ params['policy.weight'].to(F64).t() + params['policy.bias'].to(F64)
    baseline = c @ params['baseline.weight'].to(F64).t() + params['baseline.bias'].to(F64)
    return logits, baseline.reshape(-1)


# ------------------------------------------------------------------------------------------------ backward
def dh_ref(dlogits, dbaseline, h_nb, params):
    """head_bwd_dh_kernel / column kernel phase C: dh = (dlogits . Wp + dV Wb)[:, :512] * (h > 0)"""
    Wp, Wb = params['policy.weight'].to(F64), params['baseline.weight'].to(F64)
    d = dlogits.to(F64) @ Wp[:, :512] + dbaseline.to(F64).reshape(-1, 1) * Wb[:, :512]
    return d * (h_nb > 0)


def head_grads(dlogits, dbaseline, c_nb):
    dl, dv = dlogits.to(F64), dbaseline.to(F64).reshape(-1)
    return {'policy.weight': dl.t() @ c_nb, 'policy.bias': dl.sum(0),
            'baseline.weight': (dv @ c_nb).reshape(1, -1), 'baseline.bias': dv.sum().reshape(1)}


def fc_bwd(dh, a3_nb, Wfc, mask3):
    """fc wgrad (dh^T a3), fc bias (column sums of the dh operand), da3 = (dh . Wfc) * mask as [NB,64,7,7]"""
    flat = tuple(None if t is None else t.reshape(t.shape[0], -1) for t in a3_nb)
    dW = sp(lambda d, x: d.t() @ x, dh, flat)
    db = psum(dh, 0)
    da3 = sp(lambda d, w: d @ w, dh, Wfc).reshape(-1, 64, 7, 7) * mask3
    return dW, db, da3


def conv_bwd(x, dy, W, stride, mask_x=None, scale=1.0):
    """wgrad sum_pos x^T dy (times `scale`: conv1's 1/255), bias = column sums of the dY operand, and (mask_x given) dgrad * mask"""
    wshape = W[0].shape
    dW = sp(lambda a, d: torch.nn.grad.conv2d_weight(a, wshape, d, stride=stride), x, dy) * scale
    db = psum(dy, (0, 2, 3))
    dx = None
    if mask_x is not None:
        dx = sp(lambda d, w: torch.nn.grad.conv2d_input(x[0].shape, w, d, stride=stride), dy, W) * mask_x
    return dW, db, dx


def abs_terms(f, a, b):
    """the same products on |operands|: sum |terms|, the scale of a GEMM's fp32 accumulation error (ACC_REL times it)"""
    ab = lambda p: (p[0].abs(), None if p[1] is None else p[1].abs())
    return sp(f, ab(a), ab(b))


# ------------------------------------------------------------------------------------------------ comparisons
ACC_REL = 2.0 ** -18      # fp32 accumulation error allowance per unit of sum |terms|
MISMATCH = 5e-3           # the largest fraction of a bf16-stored output that may be one ulp from the rounding of the fp64 result


def rel_l2(a, b):
    a, b = a.to(F64), b.to(F64)
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def nerr(a, b):
    a, b = a.to(F64), b.to(F64)
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-300)) if b.numel() else 0.0


def ordered_bits(x_bf16):
    """bf16 -> integers whose difference is the distance in ulps (+0 and -0 both map to 0)"""
    i = x_bf16.contiguous().view(torch.int16).to(torch.int64)
    return torch.where(i < 0, -(i & 0x7FFF), i)


def compare_stored(got_hi, got_lo, ref, pre=None, terms=None, rms_ref=None, rms_pre=None):
    """A bf16-stored output (got_lo: the split mode's low twin) against the fp64 result `ref`.  rms_ref / rms_pre: the rms of the
    whole tensor when `ref` / `pre` is one slice of it (a tensor compared slice by slice); by default the slice's own.

    `pre` (ReLU outputs): the fp64 pre-activation; where the GPU's mask disagrees with it the unit must be a tie,
    |pre| < TIE * rms(pre), and it is left out of the value comparison.
    bf16 mode: every other element is the bf16 rounding of ref or one ulp from it, except where fp32 accumulation
    cancelled: |got - ref| <= max(TIE * rms(ref), ACC_REL * terms), terms = sum |products| where given.  Split mode:
    |hi + lo - ref| <= 2^-16 |ref| + that same accumulation allowance -- two units of the pair's last place plus the fp32 sum's
    own error, which the pair's 16 bits resolve wherever |ref| is below about rms."""
    ref = ref.to(F64).reshape(-1)
    got = got_hi.to(F64).reshape(-1) + (0 if got_lo is None else got_lo.to(F64).reshape(-1))
    keep = torch.ones_like(ref, dtype=torch.bool)
    st = {'n': ref.numel()}
    if pre is not None:
        pre = pre.to(F64).reshape(-1)
        flip = (got > 0) != (pre > 0)
        rms_z = rms_pre if rms_pre is not None else float(pre.pow(2).mean().sqrt()) if pre.numel() else 0.0
        st['mask_flips'] = int(flip.sum())
        st['worst_flip_margin'] = float(pre[flip].abs().max() / max(rms_z, 1e-300)) if bool(flip.any()) else 0.0
        keep = ~flip
    rms = rms_ref if rms_ref is not None else float(ref.pow(2).mean().sqrt()) if ref.numel() else 0.0
    err = (got - ref).abs()
    acc = torch.full_like(ref, TIE * rms)
    if terms is not None:
        acc = torch.maximum(acc, ACC_REL * terms.to(F64).reshape(-1))
    if got_lo is None:
        ulps = (ordered_bits(got_hi.reshape(-1)) - ordered_bits(ref.to(torch.bfloat16))).abs()
        cancel = err <= acc
        st['max_ulp'] = int(ulps[keep & ~cancel].max()) if bool((keep & ~cancel).any()) else 0
        st['mismatch_frac'] = float(((ulps != 0) & keep).sum()) / max(ref.numel(), 1)
        st['beyond_1ulp_cancelled'] = int(((ulps > 1) & keep & cancel).sum())
    else:
        bound = 2.0 ** -16 * ref.abs() + acc
        st['bad'] = int((keep & (err > bound)).sum())
        st['worst_bound_frac'] = float((err[keep] / bound[keep].clamp_min(1e-300)).max()) if bool(keep.any()) else 0.0
        st['beyond_pair_precision'] = int((keep & (err > 2.0 ** -16 * ref.abs())).sum())
    st['rel_l2'] = rel_l2(got[keep], ref[keep]) if bool(keep.any()) else 0.0
    return st


def stored_ok(st, split_mode):
    if 'mask_flips' in st and st['mask_flips'] and st['worst_flip_margin'] >= TIE:
        return False
    if split_mode:
        return st['bad'] == 0
    return st['max_ulp'] <= 1 and st['mismatch_frac'] <= MISMATCH


# ------------------------------------------------------------------------------------------------ wgrad partition (igemm_res.cuh)
WG_PART_CTAS = 160
_WG_IMG_BYTES = 2 * 128 * 20 * 4
# name: (WROWS, NWIN, DY_CH, A_LO, SMEM_BIAS, CWG, STAGES, SPLIT_STAGES) of RConv{3,2,1}Wgrad (res_problems.cuh)
WGRAD_PROBLEMS = {'conv3': (148, 1, 64, True, False, 3, 3, 2), 'conv2': (139, 2, 64, True, True, 2, 3, 1),
                  'conv1': (150, 1, 32, False, True, 2, 5, 3)}


def wgrad_ring_depth(name, split_mode):
    """ResWgradCfg<P, SPLIT>::STAGES"""
    wrows, nwin, dych, alo, smem_bias, cwg, stages, split_stages = WGRAD_PROBLEMS[name]
    sp_ = 1 if split_mode else 0
    win = (wrows * 128 + 1023) // 1024 * 1024
    stage = nwin * win * (1 + (1 if (sp_ and alo) else 0)) + 128 * dych * 2 * (1 + sp_)
    ones = 128 * 128 if (not smem_bias and not sp_) else 0
    fixed = ones + cwg * _WG_IMG_BYTES + 2048 + 1024 + 256
    s = split_stages if sp_ else stages
    while s > 1 and fixed + s * stage > 232448:
        s -= 1
    return s


def wgrad_partition(positions, target_ctas):
    """res_wgrad_launch_t: chunks of 128 positions, chunks_per_cta, grid, chunks of the last CTA"""
    nch = (positions + 127) // 128
    target = min(target_ctas, WG_PART_CTAS)
    cpc = (nch + target - 1) // target
    grid = (nch + cpc - 1) // cpc
    return {'chunks': nch, 'chunks_per_cta': cpc, 'grid': grid, 'last_cta_chunks': nch - (grid - 1) * cpc}


def sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def cta_counts(sm_count, env):
    """encoder.cu persistent_ctas / bwd_ctas / side_wgrad_ctas from the SRL_* overrides in `env`"""
    def _int(k):
        try:
            return int(env.get(k, ''))
        except ValueError:
            return None
    p = _int('SRL_PERSISTENT_CTAS')
    p = sm_count if p is None or p < 16 or p > sm_count else p
    b = _int('SRL_BWD_CTAS')
    b = p - p // 9 if b is None or b < 16 or b > sm_count else b
    w = _int('SRL_WGRAD_CTAS')
    w = 64 if w is None or w < 8 or w > sm_count else w
    return {'persistent': p, 'bwd': b, 'side_wgrad': w}


def wgrad_partitions(NB, ctas, split_mode):
    """the three conv wgrad launches of one step: conv3 / conv2 on the side streams, conv1 on the backward chain"""
    out = {}
    for name, grid_pos, target in (('conv3', 81, ctas['side_wgrad']), ('conv2', 100, ctas['side_wgrad']), ('conv1', 441, ctas['bwd'])):
        d = wgrad_partition(NB * grid_pos, target)
        d['ring'] = wgrad_ring_depth(name, split_mode)
        out[name] = d
    return out


def mid_chunk_frames(NB, G, part):
    """frames and position mask [n1-n0, 1, G, G] of the first chunk of the middle CTA of a wgrad launch"""
    q0 = (part['grid'] // 2) * part['chunks_per_cta'] * 128
    n0, n1 = q0 // (G * G), min(NB, (q0 + 127) // (G * G) + 1)
    m = torch.zeros((n1 - n0) * G * G, dtype=F64)
    m[q0 - n0 * G * G:q0 - n0 * G * G + 128] = 1
    return n0, n1, m.view(n1 - n0, 1, G, G)


def regimes(part):
    """which of the four partition regimes one wgrad launch is in"""
    c, r = part['chunks_per_cta'], part['ring']
    return {'one_chunk_per_cta': c == 1, 'within_ring': 2 <= c <= r, 'ring_wraps_twice': c > 2 * r,
            'last_cta_single_chunk': part['grid'] > 1 and part['last_cta_chunks'] == 1}
