"""The Ape-X Q-head kernels against an fp64 evaluation of their own operation (tests/apex_head_ref.py), element by element, on the operands
the GPU itself read: one learner step per case through B200ApexLearner, and one prioritized add per actor case through
GpuPrioritizedReplayBuffer.save_to_memory(..., priorities_from=actor).

  * Each stage is checked on the GPU's own output of the stage before it (apex_head_ref's docstring), so every bound is local.
  * Every output row the test reads is filled with NaN bytes before the step: the learner's arena starts as cudaMemset(0), so a store a
    kernel skips would otherwise read as a plausible zero.
  * Sensitivity: each case records how far the mistakes of apex_head_ref.MISTAKES move its references, in bounds, and requires >= 20x
    for the mistakes its row names.
  * Which kernel runs: launch_q_tail / launch_q_wgrad pick the kernels by head kind alone (plain: dqn_tail_kernel<false> and
    dqn_wgrad_kernel<false>; dueling: <true>; C51: cat_gemm_kernel<false> + cat_tail_kernel + cat_gemm_kernel<true>; QR: the same GEMMs
    + qr_tail_kernel; the distributional-dueling heads add dist_dueling_compose_kernel and dist_dueling_grad_kernel), and the table
    names the kind.  torch.profiler is not used to find out which kernel ran.

The worst err / bound of every check, its margin and the strongest sensitivity go to $SRL_RESULTS_DIR/apex_head_exact.json (per case,
and a summary per check)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from scalerl_b200 import _lib
from scalerl_b200.algorithms.apex import default_q_state_dict
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests import apex_cases as AC
from tests import apex_head_ref as R
from tests import exact

pytestmark = pytest.mark.gpu

RESULTS = 'apex_head_exact.json'
F64 = torch.float64


# ------------------------------------------------------------------------------------------------ the cases
# (id, head, B, A, width, edge, keywords, mistakes the case must witness).  head: apex_cases.HEADS' name, or dd_categorical / dd_quantile
# for the distributional dueling heads.  keywords: double, gamma, done_p, weights (False: weights=None), kappa, support, rewards
# ('atoms': exactly on v_min, v_max, an atom and beyond the support), precision, eps.
_W = ('wgrad_last_group', 'bias_dropped')
_CW = ('wgrad_last_kstage', 'bias_dropped', 'gemm_row0_unstored')
CASES = [
    # tail blocks / tail_loss lanes (4 warps per block, 32 lanes over the block partials)
    ('plain_B1', 'plain', 1, 6, 0, 'B=1: one warp of one block', {}, ('loss_last_block',) + _W),
    ('plain_B2', 'plain', 2, 6, 0, 'B=2: a block with 2 idle warps', {}, ('loss_last_block',)),
    ('dueling_B3', 'dueling', 3, 6, 0, 'B=3', {}, ('dueling_mean_A_minus_1', 'dueling_dcore_no_mean') + _W),
    ('plain_B5', 'plain', 5, 6, 0, 'B=5: last block with 1 warp', dict(double=True), ('loss_last_block', 'double_target_astar')),
    ('dueling_B128', 'dueling', 128, 6, 0, 'B=128: 32 blocks, one per lane', {}, ('loss_last_block',)),
    ('plain_B129', 'plain', 129, 6, 0, 'B=129: 33 blocks, lane 0 adds two', dict(weights=False), ('loss_last_block',)),
    # dqn_wgrad slabs / groups
    ('plain_B16', 'plain', 16, 6, 0, 'B=16: one full slab', {}, _W),
    ('dueling_B17', 'dueling', 17, 6, 0, 'B=17: a ragged second slab', {}, _W),
    ('plain_B512', 'plain', 512, 6, 0, 'B=512: 32 groups of one slab', {}, _W),
    ('dueling_B513', 'dueling', 513, 6, 0, 'B=513: 17 groups of two slabs', dict(double=True), _W),
    ('plain_B1024', 'plain', 1024, 6, 0, 'B=1024: 32 groups of two slabs', dict(done_p=1.0), _W),
    # cat_gemm tiles
    ('cat_B63', 'categorical', 63, 1, 63, 'B=63, R=63: one ragged tile', {}, _CW),
    ('cat_B64', 'categorical', 64, 1, 64, 'B=64, R=64: one full tile', dict(rewards='atoms', gamma=0.0), _CW + ('project_split_l_eq_u',)),
    ('cat_B65', 'categorical', 65, 5, 13, 'B=65, R=65: a 1-row second tile', dict(double=True), _CW),
    # A at the C ABI's limit
    ('plain_A31', 'plain', 129, 31, 0, 'A=31', {}, _W),
    ('dueling_A31', 'dueling', 129, 31, 0, 'A=31: R=32=DQN_MAX_A fills sd[16][32]', {}, _W + ('dueling_mean_A_minus_1',)),
    ('plain_A1', 'plain', 33, 1, 0, 'A=1', {}, _W),
    ('plain_A2', 'plain', 33, 2, 0, 'A=2', {}, _W),
    ('dueling_A1', 'dueling', 33, 1, 0, 'A=1: R=2, mean = the one advantage', {}, _W),
    ('dueling_A2', 'dueling', 33, 2, 0, 'A=2', {}, ('dueling_mean_A_minus_1',)),
    # C51 atoms, R = A K on both sides of 64, supports and rewards
    ('cat_K2', 'categorical', 37, 2, 2, 'K=2', dict(rewards='atoms'), ('project_split_l_eq_u', 'gemm_row0_unstored')),
    ('cat_K51_A31', 'categorical', 66, 31, 51, 'K=51, A=31: R=1581', dict(double=True), _CW),
    ('cat_K64_A31', 'categorical', 33, 31, 64, 'K=64=CAT_MAX_ATOMS, A=31: R=1984', dict(rewards='atoms', gamma=0.0),
     ('project_split_l_eq_u', 'wgrad_last_kstage')),
    ('cat_K63_nodone', 'categorical', 40, 3, 63, 'K=63, no dones', dict(done_p=0.0, support=(-3.0, 7.0)), _CW),
    # QR quantiles
    ('qr_N2', 'quantile', 37, 3, 2, 'N=2', {}, ('tau_i_over_N',) + _CW),
    ('qr_N31', 'quantile', 37, 3, 31, 'N=31: lane 31 idle', dict(double=True), ('tau_i_over_N', 'double_target_astar')),
    ('qr_N32', 'quantile', 37, 2, 32, 'N=32: one per lane', dict(gamma=0.0), ('tau_i_over_N',)),
    ('qr_N33', 'quantile', 37, 2, 33, 'N=33: lane 0 holds two', dict(kappa=0.5), ('tau_i_over_N',)),
    ('qr_N255', 'quantile', 20, 2, 255, 'N=255', dict(kappa=0.02), ('tau_i_over_N',)),
    ('qr_N256', 'quantile', 20, 2, 256, 'N=256=QR_MAX_QUANTILES, 8 per lane', dict(done_p=1.0), ('tau_i_over_N',)),
    ('qr_A31_N256', 'quantile', 9, 31, 256, 'A=31, N=256: R=7936', {}, ('tau_i_over_N', 'wgrad_last_kstage', 'gemm_row0_unstored')),
    ('qr_A1', 'quantile', 17, 1, 7, 'A=1', dict(weights=False), ('tau_i_over_N',)),
    # distributional dueling
    ('ddc_B65', 'dd_categorical', 65, 4, 11, 'C51 rows, A=4', {}, ('dd_grad_mean_axis', 'dd_grad_A_minus_1')),
    ('ddq_B33', 'dd_quantile', 33, 3, 9, 'QR rows, A=3', dict(double=True), ('dd_grad_mean_axis', 'dd_grad_A_minus_1')),
    ('ddc_A1', 'dd_categorical', 33, 1, 11, 'C51 rows, A=1: mean = the one advantage', {}, ('dd_grad_mean_axis',)),
    ('ddc_A2', 'dd_categorical', 33, 2, 11, 'C51 rows, A=2', {}, ('dd_grad_mean_axis', 'dd_grad_A_minus_1')),
    ('ddc_A31', 'dd_categorical', 33, 31, 11, 'C51 rows, A=31: R=341', dict(double=True), ('dd_grad_mean_axis', 'dd_grad_A_minus_1')),
    ('ddq_A1', 'dd_quantile', 33, 1, 9, 'QR rows, A=1', {}, ('dd_grad_mean_axis',)),
    ('ddq_A2', 'dd_quantile', 33, 2, 9, 'QR rows, A=2', {}, ('dd_grad_mean_axis', 'dd_grad_A_minus_1')),
    ('ddq_A31', 'dd_quantile', 33, 31, 9, 'QR rows, A=31: R=279', {}, ('dd_grad_mean_axis', 'dd_grad_A_minus_1')),
    # exact ties built into the online network (apex_cases' _tie_*: actions 1 and 4 equal and dominant): under double DQN a* is the
    # first index, 1, in the kernel and in the reference; the target network values actions 1 and 4 differently, so y shows which
    ('tie_plain', 'plain', 37, 6, 0, 'exact tie, double DQN', dict(double=True, tie=True), ()),
    ('tie_dueling', 'dueling', 37, 6, 0, 'exact tie, double DQN', dict(double=True, tie=True), ()),
    ('tie_cat', 'categorical', 37, 6, 11, 'exact tie, double DQN', dict(double=True, tie=True), ()),
    ('tie_qr', 'quantile', 37, 6, 16, 'exact tie, double DQN', dict(double=True, tie=True), ()),
    # noisy heads on their composed weights
    ('noisy_plain_B9', 'noisy_plain', 9, 5, 0, 'noisy, small', {}, ()),
    ('noisy_plain_B133', 'noisy_plain', 133, 7, 0, 'noisy, ragged', {}, ()),
    ('noisy_dueling_B9', 'noisy_dueling', 9, 5, 0, 'noisy, small', {}, ()),
    ('noisy_dueling_B133', 'noisy_dueling', 133, 7, 0, 'noisy, ragged', {}, ()),
    ('noisy_cat_B9', 'noisy_categorical', 9, 5, 11, 'noisy, small', {}, ()),
    ('noisy_cat_B133', 'noisy_categorical', 133, 7, 11, 'noisy, ragged', {}, ()),
    # fp32-split: the tail is the same code in both modes
    ('plain_split_B65', 'plain', 65, 6, 0, 'precision=fp32_split', dict(precision='fp32_split'), _W),
    # every head at large B
    *[(f'{h}_B{B}', h, B, 4, w, f'B={B}', dict(double=B == 4097), ())
      for B in (513, 4097, 65536)
      for h, w in (('plain', 0), ('dueling', 0), ('categorical', 51), ('quantile', 32), ('dd_categorical', 21), ('dd_quantile', 16))],
]


_summary = exact.summary(RESULTS)


def _ties(Ck, name, tie, B):
    """the a* tie rows (pick()'s tie set) are at most MAX_TIE_FRAC of the batch"""
    n = int(tie.sum())
    Ck.res[name] = {'tie_rows': n, 'tie_frac': n / B}
    if n > max(1, R.MAX_TIE_FRAC * B):
        Ck.fails.append(f'{name}: {n} tie rows of {B}')


def _done(Ck, case, witness=()):
    """the mistakes of `witness` each move some check of the case by >= SENS x its bound; record the case's strongest sensitivities"""
    Ck.require(case, Ck.sens, witness)
    Ck.res['sensitivity'] = {m: min(v, 1e30) for m, v in Ck.sens.items()}
    Ck.done(case)


def _nan_fill(L, names):
    """NaN bytes into the learner's device rows `names` (the C ABI's pointers, not debug_buffer's copies)"""
    lib = _lib.lib()
    for n in names:
        p, cnt = C.c_void_p(), C.c_int64()
        _lib.check(lib.srl_apex_learner_debug_buffer(L._h, n.encode(), C.byref(p), C.byref(cnt)), 'debug_buffer')
        nb = cnt.value * (8 if n == 'priorities' else 4)
        src = torch.full((nb,), 0xFF, dtype=torch.uint8, device='cuda')
        _lib.check(lib.srl_memcpy_d2d(p.value, src.data_ptr(), nb, torch.cuda.current_stream().cuda_stream), 'memcpy_d2d')
    torch.cuda.synchronize()


def _choose(alts, dev):
    """per row, the candidate (of a tie set) whose reference is nearest the device's -> index [B]"""
    err = torch.stack([(a - dev).abs().reshape(a.shape[0], -1).nan_to_num(math.inf).amax(1) for a in alts], 1)
    return err.argmin(1)


# ------------------------------------------------------------------------------------------------ one learner step
def _setup(hname, B, A, width, kw):
    dd = hname.startswith('dd_')
    kind = {'dd_categorical': 'categorical', 'dd_quantile': 'quantile'}.get(hname)
    head = AC.HEADS[kind if dd else hname]
    if width:
        head = head.but(width=width)
    if 'kappa' in kw:
        head = head.but(kappa=kw['kappa'])
    if 'support' in kw:
        head = head.but(v_min=kw['support'][0], v_max=kw['support'][1])
    if dd:
        on = default_q_state_dict(A, 2, False, width if kind == 'categorical' else 0, False, 0.5, width if kind == 'quantile' else 0, True)
        tg = default_q_state_dict(A, 3, False, width if kind == 'categorical' else 0, False, 0.5, width if kind == 'quantile' else 0, True)
    else:
        on, tg = AC.nets(head, A, seed=B % 97)
    if kw.get('tie'):
        head.tie(on, A, head.width)
    (obs, act, rew, nobs, done), w = AC.batch(B, A, seed=B + A + width, done_p=kw.get('done_p', 0.25), device='cuda')
    rew = head.scale_reward(rew)
    if kw.get('rewards') == 'atoms':
        z32, _ = AC.O.support(head.width, head.v_min, head.v_max)
        pool = torch.tensor([head.v_min - 5.0, head.v_max + 5.0, float(z32[0]), float(z32[-1]), float(z32[head.width // 2]),
                             float(z32[1])], dtype=torch.float32)
        rew = pool[torch.arange(B) % len(pool)].cuda()
    return head, dd, on, tg, (obs, act, rew, nobs, done), (None if kw.get('weights') is False else w)


def _run_case(cid, hname, B, A, width, kw, witness):
    head, dd, on, tg, bt, w = _setup(hname, B, A, width, kw)
    gamma, double, eps = kw.get('gamma', 0.97), kw.get('double', False), 1e-6
    extra = dict(distributional_dueling=True) if dd else {}
    free0 = torch.cuda.mem_get_info()[0]
    L = AC.learner(head, B, A, on, tg, double_dqn=double, gamma=gamma, priority_eps=eps, precision=kw.get('precision', 'bf16'),
                   seed=5 if head.noisy else 0, **extra)
    arena = (free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30      # the learner's device blocks (this process's change of free memory)
    try:
        _check_step(cid, head, dd, L, B, A, kw, bt, w, gamma, double, float(np.float32(eps)), witness, arena)
    finally:
        L.close()


def _check_step(cid, head, dd, L, B, A, kw, bt, w, gamma, double, eps, witness, arena):
    pre, pre_t = L.state_dict(), L.state_dict(target=True)
    dist = head.kind in ('categorical', 'quantile')
    qr = head.kind == 'quantile'
    outs = ['dcore', 'q', 'y', 'priorities', 'loss']
    if dist:
        outs += (['theta', 'theta_next_target', 'dtheta', 'target_quantiles', 'qr_loss'] if qr else
                 ['logits', 'logits_next_target', 'dlogits', 'm', 'ce'])
        if double:
            outs.append('theta_next' if qr else 'logits_next')
    if dd:
        outs += ['rows_weight_online', 'rows_bias_online', 'rows_weight_target', 'rows_bias_target', 'rows_weight_grad', 'rows_bias_grad']
    _nan_fill(L, outs)
    if not head.noisy:
        for g in L.grads.values():
            g.fill_(math.nan)
    L.learn(bt, weights=w, use_graph=False)
    torch.cuda.synchronize()
    obs, act, rew, nobs, done = bt
    act = act.long()
    dbg = lambda n: L.debug_buffer(n)
    core = lambda n: dbg(n).view(B, 514)
    h, hnt = core('core')[:, :512], core('core_next_target')[:, :512]
    hn = core('core_next')[:, :512] if double else None
    Ck = exact.Checker(RESULTS, R)
    dcore = core('dcore')
    Ck.zero('dcore_pad', dcore[:, 512:])
    g32 = float(np.float32(gamma))
    wt = None if w is None else w
    if not dist:
        a1 = _scalar(Ck, head, L, pre, pre_t, h, hn, hnt, act, rew, done, wt, g32, double, eps, B, A, dcore)
    else:
        a1 = _distributional(Ck, head, dd, L, pre, pre_t, h, hn, hnt, act, rew, done, wt, g32, double, eps, B, A, dcore)
    if kw.get('tie'):
        n = int((a1 != 1).sum())
        Ck.res['exact_tie'] = {'rows_not_first_index': n}
        if n:
            Ck.fails.append(f'exact ties: the fp64 a* is not the first index on {n} rows')
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    Ck.res['memory'] = {'learner_gib': arena, 'reference_peak_gib': peak, 'total_gib': arena + peak}
    _done(Ck, cid, witness)


def _scalar_nets(head, L, sd, net):
    if head.noisy:
        comp = AC.device_composed(L, net)
        if head.kind == 'dueling':
            return {'W': torch.cat([comp['value'][0], comp['advantage'][0]]), 'b': comp['value'][1], 'ba': comp['advantage'][1]}
        return {'W': comp['q'][0], 'b': comp['q'][1]}
    if head.kind == 'dueling':
        return {'W': torch.cat([sd['value.weight'], sd['advantage.weight']]), 'b': sd['value.bias'], 'ba': sd['advantage.bias']}
    return {'W': sd['q.weight'], 'b': sd['q.bias']}


def _scalar(Ck, head, L, pre, pre_t, h, hn, hnt, act, rew, done, w, g32, double, eps, B, A, dcore):
    kind = head.kind
    on, tg = _scalar_nets(head, L, pre, 'online'), _scalar_nets(head, L, pre_t, 'target')
    on = {k: v.cuda() for k, v in on.items()}
    tg = {k: v.cuda() for k, v in tg.items()}
    Q, SQ = R.scalar_q(kind, h, on)
    mist = {}
    if kind == 'dueling':
        mist['dueling_mean_A_minus_1'] = R.take(R.scalar_q(kind, h, on, 'dueling_mean_A_minus_1')[0], act) if A > 1 else R.take(Q, act)
    Ck.bound('q', dbg_(L, 'q'), R.take(Q, act), R.take(SQ, act), R.CHECK_C['q'], mistakes=mist)
    nx1, S1, nx2, S2, tie, a1 = R.scalar_targets(kind, hn, hnt, on, tg, double)
    y1, Sy1 = R.td_target(rew, done, g32, nx1, S1)
    y2, Sy2 = R.td_target(rew, done, g32, nx2, S2)
    ydev = dbg_(L, 'y')
    pick2 = tie & (_choose([y1, y2], ydev) == 1)
    y, Sy = torch.where(pick2, y2, y1), torch.where(pick2, Sy2, Sy1)
    _ties(Ck, 'a_star_ties', tie, B)
    mist = {}
    if double:
        nxm, Sm, *_ = R.scalar_targets(kind, hn, hnt, on, tg, double, 'double_target_astar')
        mist['double_target_astar'] = R.td_target(rew, done, g32, nxm, Sm)[0]
    Ck.bound('y', ydev, y, Sy, R.CHECK_C['y'], mistakes=mist)
    fq = R.from_qy(dbg_(L, 'q'), ydev, w, B, eps)
    Ck.bound('priority', L.debug_buffer('priorities'), fq['prio'][0], fq['prio'][1], R.CHECK_C['priority'])
    dc, Sdc = R.scalar_dcore(kind, fq['dq'], act, on)
    mist = {m: R.scalar_dcore(kind, fq['dq'], act, on, m)[0] for m in ('dueling_mean_A_minus_1', 'dueling_dcore_no_mean')
            if kind == 'dueling' and A > 1}
    Ck.bound('dcore_scalar', dcore[:, :512], dc, Sdc, R.CHECK_C['dcore_scalar'], mistakes=mist)
    lo, Sl = R.loss_ref(fq['l'], B)
    Ck.bound('loss', L.debug_buffer('loss')[:1], lo.view(1), Sl.view(1), R.CHECK_C['loss'],
             mistakes={'loss_last_block': R.loss_ref(fq['l'], B, 'loss_last_block')[0].view(1)})
    if head.noisy:
        return a1
    g, Sg = R.scalar_wgrad(kind, fq['dq'], act, h, A, B)
    mist = {m: R.scalar_wgrad(kind, fq['dq'], act, h, A, B, m)[0] for m in ('wgrad_last_group', 'bias_dropped')}
    if kind == 'dueling' and A > 1:
        mist['dueling_mean_A_minus_1'] = R.scalar_wgrad(kind, fq['dq'], act, h, A, B, 'dueling_mean_A_minus_1')[0]
    if kind == 'dueling':
        dev = torch.cat([torch.cat([L.grads['value.weight'], L.grads['value.bias'][:, None]], 1),
                         torch.cat([L.grads['advantage.weight'], L.grads['advantage.bias'][:, None]], 1)])
    else:
        dev = torch.cat([L.grads['q.weight'], L.grads['q.bias'][:, None]], 1)
    Ck.bound('head_grad', dev, g, Sg, R.CHECK_C['head_grad'], mistakes=mist)
    return a1


def dbg_(L, n):
    return L.debug_buffer(n)


def _dist_nets(head, dd, L, sd, net):
    if dd:
        return L.debug_buffer(f'rows_weight_{net}').view(-1, 512), L.debug_buffer(f'rows_bias_{net}')
    if head.noisy:
        comp = AC.device_composed(L, net)
        return comp['q'][0], comp['q'][1]
    return sd['q.weight'].cuda(), sd['q.bias'].cuda()


def _distributional(Ck, head, dd, L, pre, pre_t, h, hn, hnt, act, rew, done, w, g32, double, eps, B, A, dcore):
    qr, Kw = head.kind == 'quantile', head.width
    R_ = A * Kw
    rows = torch.arange(B, device='cuda')
    names = ('theta', 'theta_next', 'theta_next_target', 'dtheta') if qr else ('logits', 'logits_next', 'logits_next_target', 'dlogits')
    Won, bon = _dist_nets(head, dd, L, pre, 'online')
    Wtg, btg = _dist_nets(head, dd, L, pre_t, 'target')
    if dd:
        for net, sd in (('online', pre), ('target', pre_t)):
            W_, b_, SW, Sb = R.dd_compose(sd['value.weight'].cuda(), sd['value.bias'].cuda(), sd['advantage.weight'].cuda(),
                                          sd['advantage.bias'].cuda(), A)
            Ck.bound(f'rows_{net}', torch.cat([Won if net == 'online' else Wtg, (bon if net == 'online' else btg)[:, None]], 1),
                     torch.cat([W_, b_[:, None]], 1), torch.cat([SW, Sb[:, None]], 1), R.CHECK_C['rows'])
    gemm = [(names[0], h, Won, bon), (names[2], hnt, Wtg, btg)] + ([(names[1], hn, Won, bon)] if double else [])
    dev = {}
    for n, hh, W_, b_ in gemm:
        x, S = R.gemm_rows(hh, W_, b_)
        dev[n] = L.debug_buffer(n).view(B, R_)
        Ck.bound(n, dev[n], x, S, R.CHECK_C['theta' if qr else 'logits'],
                 mistakes={'gemm_row0_unstored': R.gemm_rows(hh, W_, b_, 'gemm_row0_unstored')[0]})
    xs_all = dev[names[0]].to(F64).view(B, A, Kw)
    xt = dev[names[2]].to(F64).view(B, A, Kw)
    xsel = dev[names[1]].to(F64).view(B, A, Kw) if double else xt
    Qsel, Ssel = R.qr_q(xsel) if qr else R.cat_q(xsel, AC.O.support(Kw, head.v_min, head.v_max)[0])
    a1, a2, tie = R.pick(Qsel, Ssel)
    _ties(Ck, 'a_star_ties', tie, B)
    g = g32 * (1 - done.to(F64))
    xs = xs_all[rows, act]
    wv = torch.ones(B, dtype=F64, device='cuda') if w is None else w.to(F64)
    if qr:
        T1, ST1 = R.qr_targets(xt, a1, rew, g)
        T2, ST2 = R.qr_targets(xt, a2, rew, g)
        Tdev = L.debug_buffer('target_quantiles').view(B, Kw)
        c2 = (tie & (_choose([T1, T2], Tdev) == 1))[:, None]
        mist = {}
        if double:
            am = R.pick(*R.qr_q(xt))[0]
            mist['double_target_astar'] = R.qr_targets(xt, am, rew, g)[0]
        Ck.bound('target_quantiles', Tdev, torch.where(c2, T2, T1), torch.where(c2, ST2, ST1), R.CHECK_C['target_quantiles'], mistakes=mist)
        ln, Sln, d, Sd = R.qr_loss(xs, Tdev, head.kappa, wv, B)
        lt, _, dt, _ = R.qr_loss(xs, Tdev, head.kappa, wv, B, 'tau_i_over_N')
        Ck.bound('qr_loss', L.debug_buffer('qr_loss'), ln, Sln, R.CHECK_C['qr_loss'], mistakes={'tau_i_over_N': lt})
        Ck.bound('priority', L.debug_buffer('priorities'), ln + eps, Sln, R.CHECK_C['qr_loss'])
        q, Sq = R.qr_q(xs)
        Ck.bound('q', L.debug_buffer('q'), q, Sq, R.CHECK_C['q'])
        yq, Syq = R.qr_q(Tdev.to(F64))
        Ck.bound('y', L.debug_buffer('y'), yq, Syq, R.CHECK_C['y'])
        lterm = wv * L.debug_buffer('qr_loss').to(F64)
    else:
        z32, dz32 = AC.O.support(Kw, head.v_min, head.v_max)
        lo, hi = float(np.float32(head.v_min)), float(np.float32(head.v_max))
        alts = []
        for a in (a1, a2):
            p, _, Sp, _ = R.softmax_rows(xt[rows, a])
            alts.append(R.project(p, Sp, rew, g, z32, float(dz32), lo, hi))
        mdev = L.debug_buffer('m').view(B, Kw)
        c2 = (tie & (_choose([alts[0][0], alts[1][0]], mdev) == 1))[:, None]
        m_ref, Sm = torch.where(c2, alts[1][0], alts[0][0]), torch.where(c2, alts[1][1], alts[0][1])
        p1, _, Sp1, _ = R.softmax_rows(xt[rows, a1])
        mist = {mk: R.project(p1, Sp1, rew, g, z32, float(dz32), lo, hi, mk)[0] for mk in ('project_split_l_eq_u', 'project_u_unclamped')}
        if double:
            am = R.pick(*R.cat_q(xt, z32))[0]
            pm, _, Spm, _ = R.softmax_rows(xt[rows, am])
            mist['double_target_astar'] = R.project(pm, Spm, rew, g, z32, float(dz32), lo, hi)[0]
        Ck.bound('m', mdev, m_ref, Sm, R.CHECK_C['m'], mistakes=mist)
        t = R.cat_tail(xs, mdev, z32, wv, B)
        Ck.bound('ce', L.debug_buffer('ce'), *t['ce'], R.CHECK_C['ce'])
        Ck.bound('priority', L.debug_buffer('priorities'), t['kl'][0].clamp(min=0) + eps, t['kl'][1], R.CHECK_C['kl'])
        Ck.bound('q', L.debug_buffer('q'), t['q'], t['q_S'], R.CHECK_C['q'])
        Ck.bound('y', L.debug_buffer('y'), *t['y'], R.CHECK_C['y'])
        d, Sd = t['dl']
        lterm = wv * L.debug_buffer('ce').to(F64)
    dl_dev = L.debug_buffer(names[3]).view(B, A, Kw)
    Ck.bound(names[3], dl_dev[rows, act], d, Sd, R.CHECK_C['dlogits'])
    other = dl_dev.clone()
    other[rows, act] = 0
    Ck.zero(f'{names[3]}_other_actions', other)
    dc, Sdc = R.row_dcore(dl_dev.view(B, R_), Won, Kw)
    Ck.bound('dcore', dcore[:, :512], dc, Sdc, R.CHECK_C['dcore'])
    lo_, Sl = R.loss_ref(lterm, B)
    Ck.bound('loss', L.debug_buffer('loss')[:1], lo_.view(1), Sl.view(1), R.CHECK_C['loss'],
             mistakes={'loss_last_block': R.loss_ref(lterm, B, 'loss_last_block')[0].view(1)})
    if head.noisy:
        return a1
    dlf = dl_dev.view(B, R_)
    gW, SgW = R.cat_wgrad(dlf, h, B)
    mist = {m: R.cat_wgrad(dlf, h, B, m)[0] for m in ('wgrad_last_kstage', 'bias_dropped')}
    if dd:
        gdev = torch.cat([L.debug_buffer('rows_weight_grad').view(R_, 512), L.debug_buffer('rows_bias_grad')[:, None]], 1)
    else:
        gdev = torch.cat([L.grads['q.weight'], L.grads['q.bias'][:, None]], 1)
    Ck.bound('head_grad', gdev, gW, SgW, R.CHECK_C['head_grad'], mistakes=mist)
    Ck.res['head_grad']['rel_l2'] = AC.rel_l2(gdev, gW)
    if dd:
        gv, Sv, ga, Sa = R.dd_grad(gdev[:, :512], gdev[:, 512], A, Kw)
        mv = {m: R.dd_grad(gdev[:, :512], gdev[:, 512], A, Kw, m)[2] for m in ('dd_grad_mean_axis', 'dd_grad_A_minus_1')
              if A > 1 or m == 'dd_grad_mean_axis'}
        Ck.bound('dd_grad_value', torch.cat([L.grads['value.weight'], L.grads['value.bias'][:, None]], 1), gv, Sv, R.CHECK_C['rows_sum'])
        Ck.bound('dd_grad_advantage', torch.cat([L.grads['advantage.weight'], L.grads['advantage.bias'][:, None]], 1), ga, Sa,
                 R.CHECK_C['rows'], mistakes=mv)
    return a1


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_learner_step_exact(case):
    cid, hname, B, A, width, edge, kw, witness = case
    torch.cuda.reset_peak_memory_stats()
    _run_case(cid, hname, B, A, width, kw, witness)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ the actor: q_values and priorities
ACTOR_HEADS = ['plain', 'dueling', 'categorical', 'quantile', 'dd_categorical', 'dd_quantile', 'noisy_plain', 'noisy_dueling',
               'noisy_categorical']


def _actor(hname, E, A, **kw):
    """an actor of the head on default_q_state_dict's network of seed 11 -> (head, dd, actor, state dict)"""
    dd = hname.startswith('dd_')
    head = AC.HEADS[{'dd_categorical': 'categorical', 'dd_quantile': 'quantile'}.get(hname, hname)]
    if head.width and not head.noisy:
        head = head.but(width=13 if head.kind == 'categorical' else 24)
    K = head.width if head.kind == 'categorical' else 0
    N = head.width if head.kind == 'quantile' else 0
    sd = default_q_state_dict(A, 11, head.kind == 'dueling', K, head.noisy, 0.5, N, dd)
    X = AC.actor(head, E, A, init_state_dict=sd, **(dict(distributional_dueling=True) if dd else {}), **kw)
    return head, dd, X, sd


def _actor_head(Ck, head, dd, X, sd, A):
    """the weights the actor's forwards ran on: the scalar head's {W, b, ba}, or the distributional head's rows (W, b); the
    distributional dueling rows checked against fp64 composition of the snapshot's value and advantage layers"""
    if head.noisy:
        W, b = X.debug_buffer('head_weight').view(-1, 512), X.debug_buffer('head_bias')
        if head.kind == 'dueling':
            return {'W': W, 'b': b, 'ba': X.debug_buffer('head_adv_bias')}
        return {'W': W, 'b': b} if head.kind == 'plain' else (W, b)
    if dd:
        W, b = X.debug_buffer('rows_weight').view(-1, 512), X.debug_buffer('rows_bias')
        Wr, br, SW, Sb = R.dd_compose(*(sd[n].cuda() for n in ('value.weight', 'value.bias', 'advantage.weight', 'advantage.bias')), A)
        Ck.bound('actor_rows_composed', torch.cat([W, b[:, None]], 1), torch.cat([Wr, br[:, None]], 1), torch.cat([SW, Sb[:, None]], 1),
                 R.CHECK_C['rows'])
        return W, b
    if head.kind in ('plain', 'dueling'):
        return {k: v.cuda() for k, v in _scalar_nets(head, None, sd, None).items()}
    return sd['q.weight'].cuda(), sd['q.bias'].cuda()


def _actor_rows(Ck, head, X, net, core, n):
    """the actor's logits / quantiles of its first n core rows, checked against the GEMM on them -> [n, A, width] fp64"""
    W, b = net
    x = X.debug_buffer('theta' if head.kind == 'quantile' else 'logits').view(-1, W.shape[0])[:n]
    xr, Sx = R.gemm_rows(core, W, b)
    Ck.bound('actor_head_rows', x, xr, Sx, R.CHECK_C['logits'])
    return x.to(F64).view(n, -1, head.width)


@pytest.mark.parametrize('A', [1, 2, 31])
@pytest.mark.parametrize('hname', ACTOR_HEADS)
def test_actor_q_values_exact(hname, A):
    """q_values_kernel (launch_q_values) for every head on 37 frames (not a multiple of the 4 warps of a block), its output filled with
    NaN first, against fp64 on the actor's own core rows (the scalar heads) or logits / quantiles"""
    n = 37
    head, dd, X, sd = _actor(hname, n, A)
    Ck = exact.Checker(RESULTS, R)
    try:
        obs = AC.frames(n, A, 'cuda')
        q = torch.full((n, A), math.nan, device='cuda')
        _lib.check(X._L.srl_apex_actor_q_values(X._h, obs.data_ptr(), n, q.data_ptr(), torch.cuda.current_stream().cuda_stream), 'q_values')
        torch.cuda.synchronize()
        core = X.debug_buffer('core').view(-1, 514)[:n, :512]
        net = _actor_head(Ck, head, dd, X, sd, A)
        if head.kind in ('plain', 'dueling'):
            Q, S = R.scalar_q(head.kind, core, net)
        else:
            x = _actor_rows(Ck, head, X, net, core, n)
            Q, S = R.qr_q(x) if head.kind == 'quantile' else R.cat_q(x, AC.O.support(head.width, head.v_min, head.v_max)[0])
        Ck.bound('q_values', q, Q, S, R.CHECK_C['q'], mistakes={'q_values_last_lane': R.q_values_mistake(Q, 'q_values_last_lane')})
    finally:
        X.close()
    _done(Ck, f'q_values_{hname}_A{A}', ('q_values_last_lane',))


@pytest.mark.parametrize('hname', ACTOR_HEADS)
@pytest.mark.parametrize('E', [1, 5, 4097])
def test_actor_priorities_exact(hname, E):
    """the priorities of the last of four prioritized adds (n = 3: adds at ptr 0 and E; M = E + E // 2 + 1 wraps the second mid-launch)
    against fp64 on the actor's own core rows (and logits / quantiles), the ring's n-step action, reward and done at each slot"""
    A, n, gamma, eps = 5, 3, 0.99, 1e-6
    head, dd, X, sd = _actor(hname, E, A, priority_eps=eps)
    eps = float(np.float32(eps))            # the kernels add the fp32 eps in double
    Ck = exact.Checker(RESULTS, R)
    try:
        M = E + E // 2 + 1
        mem = GpuPrioritizedReplayBuffer(M, E, alpha=1.0, n_step=n, gamma=gamma)
        gen = torch.Generator().manual_seed(E)
        for t in range(4):
            s, ns = AC.frames(E, 10 * t + E, 'cuda'), AC.frames(E, 10 * t + E + 1, 'cuda')
            a = torch.randint(0, A, (E,), generator=gen).cuda()
            r = (head.bf16_prio_reward * torch.randn(E, generator=gen)).cuda()
            d = (torch.rand(E, generator=gen) < 0.3).cuda()
            mem.save_to_memory(s, a, r, ns, d, is_vectorised=True, priorities_from=X)
        torch.cuda.synchronize()
        slots = (torch.arange(E) + E) % M
        _, ra, rr, _, rd = mem.gather(slots)
        cap = mem.sampler.capacity
        leaves = mem.sampler.trees()[0][cap + slots.cuda()]
        core = X.debug_buffer('core').view(2 * E, 514)[:, :512]
        gn = float(np.float32(gamma ** n))
        g = gn * (1 - rd.to(F64))
        act = ra.long()
        rows = torch.arange(E, device='cuda')
        net = _actor_head(Ck, head, dd, X, sd, A)
        if head.kind in ('plain', 'dueling'):
            Q, SQ = R.scalar_q(head.kind, core[:E], net)
            nx1, S1, nx2, S2, tie, _ = R.scalar_targets(head.kind, None, core[E:], net, net, False)
            q, Sq = R.take(Q, act), R.take(SQ, act)
            alts = [R.td_target(rr, rd, gn, nx, Sn) for nx, Sn in ((nx1, S1), (nx2, S2))]
            cand = [(q - y).abs() + eps for y, _ in alts]
            c2 = tie & (_choose(cand, leaves.to(F64)) == 1)
            ref = torch.where(c2, cand[1], cand[0])
            S = Sq + torch.where(c2, alts[1][1], alts[0][1]) + (ref - eps)
        else:
            x = _actor_rows(Ck, head, X, net, core, 2 * E)
            Kw = head.width
            xs, xn = x[:E][rows, act], x[E:]
            if head.kind == 'quantile':
                a1, a2, tie = R.pick(*R.qr_q(xn))
                cand, Ss = [], []
                for a in (a1, a2):
                    T, ST = R.qr_targets(xn, a, rr, g)
                    ln, Sln, _, _ = R.qr_loss(xs, T, head.kappa, None, E)
                    # T's own error moves each pair's rho by <= wt min(|u|, kappa) / kappa per unit of T_j
                    u = (T[:, None, :] - xs[:, :, None]).abs().clamp(max=head.kappa)
                    cand.append(ln + eps)
                    Ss.append(Sln + 2 * (u * ST[:, None, :]).sum((1, 2)) / (head.kappa * Kw))
            else:
                z32, dz32 = AC.O.support(Kw, head.v_min, head.v_max)
                lo, hi = float(np.float32(head.v_min)), float(np.float32(head.v_max))
                a1, a2, tie = R.pick(*R.cat_q(xn, z32))
                cand, Ss = [], []
                for a in (a1, a2):
                    p, _, Sp, _ = R.softmax_rows(xn[rows, a])
                    m, Sm = R.project(p, Sp, rr, g, z32, float(dz32), lo, hi)
                    t = R.cat_tail(xs, m, z32, None, E)
                    _, lp, _, _ = R.softmax_rows(xs)
                    lm = torch.where(m > 0, m.clamp(min=1e-300).log(), torch.zeros_like(m))
                    cand.append(t['kl'][0].clamp(min=0) + eps)
                    Ss.append(t['kl'][1] + 2 * (Sm * ((lm - lp).abs() + 1)).sum(1))
            c2 = tie & (_choose(cand, leaves.to(F64)) == 1)
            ref, S = torch.where(c2, cand[1], cand[0]), torch.where(c2, Ss[1], Ss[0])
        _ties(Ck, 'a_star_ties', tie, E)
        Ck.bound('actor_priority', leaves, ref, S, R.CHECK_C['priority'])
    finally:
        X.close()
    _done(Ck, f'actor_{hname}_E{E}')
