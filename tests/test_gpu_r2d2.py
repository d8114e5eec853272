"""GPU: the R2D2 learner step (B200R2D2Learner, srl_r2d2_learner_*) against the fp32 CPU oracle (oracle/r2d2_oracle.py), its new
kernels against fp64 on their own operands (tests/exact.py's Checker; results to $SRL_RESULTS_DIR/r2d2_exact.json), determinism, graph
replay, the sampler's leaves, the target cadence with a checkpoint round trip, and acting."""
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import r2d2_oracle as O
from scalerl_b200.algorithms.r2d2 import B200R2D2Learner, R2D2HParams, R2D2QNet, default_r2d2_state_dict
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler
from tests import exact
from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu

RESULTS = 'r2d2_exact.json'
F64 = torch.float64


def _hp(B, A, burn_in, T, n, dueling=True, rescale=True, **kw):
    return R2D2HParams(batch_size=B, num_actions=A, burn_in=burn_in, seq_len=T, n_step=n, dueling=dueling, value_rescaling=rescale, **kw)


def _batch(hp, seed, dev='cuda', done_p=0.08):
    g = torch.Generator().manual_seed(seed)
    L, B, A, H = hp.seq_rows, hp.batch_size, hp.num_actions, 513 + hp.num_actions
    frame = torch.randint(0, 256, (L, B, 4, 84, 84), generator=g, dtype=torch.uint8)
    la = torch.randint(0, A, (L, B), generator=g)
    rw = torch.randn(L, B, generator=g) * 2
    dn = torch.rand(L, B, generator=g) < done_p
    dn[0, 0] = True                                   # a done at row 0, at the burn-in boundary and on the last row
    dn[hp.burn_in, B - 1] = True
    dn[L - 1, B // 2] = True
    h0, c0 = (torch.randn(2, B, H, generator=g) * 0.3 for _ in range(2))
    w = torch.rand(B, generator=g) + 0.5
    cpu = dict(frame=frame, last_action=la, reward=rw, done=dn, state=(h0, c0))
    gpu = dict(frame=frame.to(dev), last_action=la.to(dev), reward=rw.to(dev), done=dn.to(dev), state=(h0.to(dev), c0.to(dev)))
    return cpu, gpu, w


def _target_sd(sd, seed):
    g = torch.Generator().manual_seed(seed)
    return OrderedDict((k, v + 0.02 * v.abs().mean() * torch.randn(v.shape, generator=g)) for k, v in sd.items())


def _learner(hp, seed=0, **kw):
    sd = default_r2d2_state_dict(hp.num_actions, hp.dueling, seed)
    L = B200R2D2Learner(hp, seed=seed, init_state_dict=sd, **kw)
    L.load_state_dict(_target_sd(sd, seed + 1), target=True)
    return L, sd


# ------------------------------------------------------------------------------------------------ whole-step parity with the oracle
PARITY = [  # (B, A, burn_in, T, n, dueling, rescale)
    (3, 6, 0, 5, 1, False, True),
    (8, 6, 4, 10, 3, True, False),
    (8, 6, 4, 10, 3, False, True),
    (5, 31, 2, 6, 2, True, True),
    (64, 18, 40, 80, 5, True, True),
]


@pytest.mark.parametrize('B,A,burn_in,T,n,dueling,rescale', PARITY)
def test_step_matches_oracle(B, A, burn_in, T, n, dueling, rescale):
    hp = _hp(B, A, burn_in, T, n, dueling, rescale, max_grad_norm=40.0)
    L, sd = _learner(hp)
    cpu, gpu, w = _batch(hp, 1)
    tg = L.state_dict(target=True)
    out = L.learn(gpu, weights=w.cuda(), use_graph=False)
    ref = O.learn_step(sd, tg, cpu, burn_in, n, hp.gamma, dueling, rescale=rescale, eps=hp.rescale_eps, eta=hp.priority_eta,
                       priority_eps=hp.priority_eps, weights=w, max_grad_norm=40.0, lr=hp.learning_rate, adam_eps=hp.adam_eps)
    M = T + n
    assert rel_l2(L.debug_buffer('q_online').view(M, B, A), ref['q_online']) < 1e-2
    assert rel_l2(L.debug_buffer('q_target').view(T, B, A), ref['q_target']) < 1e-2
    assert rel_l2(L.debug_buffer('y').view(T, B), ref['y']) < 2e-2
    assert rel_l2(L.debug_buffer('delta').view(T, B), ref['delta']) < 3e-2
    assert abs(out['loss'] - ref['loss']) <= 3e-2 * ref['loss']
    assert rel_l2(L.debug_buffer('priorities'), ref['priorities']) < 3e-2
    # the encoder's and the LSTM core's gradients at test_gpu_atari_module_lstm.py's tolerances (encoder 0.1, core 3e-2); the head's
    # gradients are sums over the core output of the TD errors, tighter
    errs = {k: rel_l2(L.grads[k], gw) for k, gw in ref['grads'].items()}
    tol = lambda k: 3e-2 if k.startswith('rnn_layer.') else 2e-2 if k.split('.')[0] in ('q', 'value', 'advantage') else 0.1
    assert all(e < tol(k) for k, e in errs.items()), errs
    for k, p in ref['params'].items():
        assert rel_l2(L.params[k], p) < 1e-3, k
    L.close()


# ------------------------------------------------------------------------------------------------ fp64 checks of the new kernels
EXACT = [  # (B, A, burn_in, T, n, dueling, rescale): ragged B and B T
    (3, 6, 0, 5, 1, False, True),
    (5, 31, 2, 7, 3, True, True),
    (17, 4, 1, 9, 2, True, False),
    (33, 18, 3, 13, 4, False, True),
]


def _head_rows64(p, X, dueling):
    """fp64 Q rows of X [N, H] under the head tensors p"""
    if dueling:
        v = X @ p['value.weight'].T + p['value.bias']
        adv = X @ p['advantage.weight'].T + p['advantage.bias']
        return v + adv - adv.mean(1, keepdim=True)
    return X @ p['q.weight'].T + p['q.bias']


def _row_grads64(dq, dueling):
    if not dueling:
        return dq
    s = dq.sum(1, keepdim=True)
    return torch.cat([s, dq - s / dq.shape[1]], dim=1)


@pytest.mark.parametrize('B,A,burn_in,T,n,dueling,rescale', EXACT)
def test_kernels_against_fp64(B, A, burn_in, T, n, dueling, rescale):
    hp = _hp(B, A, burn_in, T, n, dueling, rescale)
    L, _ = _learner(hp, seed=3)
    cpu, gpu, w = _batch(hp, 4, done_p=0.2)
    head = ('value.weight', 'value.bias', 'advantage.weight', 'advantage.bias') if dueling else ('q.weight', 'q.bias')
    p_on = {k: L.params[k].detach().to(F64).cpu() for k in head}
    p_tg = {k: L.target_params[k].detach().to(F64).cpu() for k in head}
    L.learn(gpu, weights=w.cuda(), use_graph=False)
    H, M = 513 + A, T + n
    db = lambda name: L.debug_buffer(name).cpu()
    ck = exact.Checker(RESULTS)
    X_on = db('out_online').view(M * B, H).to(F64)
    X_tg = db('out_target').view(hp.seq_rows, B, H)[burn_in + n:].reshape(T * B, H).to(F64)
    ck.fp32('head_fwd_online', db('q_online').to(F64), _head_rows64(p_on, X_on, dueling).reshape(-1))
    ck.fp32('head_fwd_target', db('q_target').to(F64), _head_rows64(p_tg, X_tg, dueling).reshape(-1))
    # the tail on the GPU's own Q rows
    q_on, q_tg = db('q_online').view(M, B, A).numpy(), db('q_target').view(T, B, A).numpy()
    y, delta, prio = O.tail_fp64_loop(q_on, q_tg, cpu['last_action'].numpy(), cpu['reward'].numpy(), cpu['done'].numpy(), burn_in, n,
                                      hp.gamma, rescale, hp.rescale_eps, hp.priority_eta, hp.priority_eps)
    ck.fp32('tail_y', db('y').to(F64), torch.from_numpy(y).to(F64).reshape(-1))
    ck.fp32('tail_delta', db('delta').to(F64), torch.from_numpy(delta).to(F64).reshape(-1))
    ck.fp32('tail_priorities', db('priorities'), torch.from_numpy(prio))
    act = cpu['last_action'][burn_in + 1:burn_in + T + 1].reshape(-1)
    dq_ref = torch.zeros(T * B, A, dtype=F64)
    dq_ref[torch.arange(T * B), act] = 2.0 * w.to(F64).repeat(T) * torch.from_numpy(delta).to(F64).reshape(-1) / (B * T)
    ck.fp32('tail_dq', db('dq').to(F64), dq_ref.reshape(-1))
    # the head backward on the GPU's own dQ rows
    dq = db('dq').view(T * B, A).to(F64)
    G = _row_grads64(dq, dueling)
    Wrows = torch.cat([p_on['value.weight'], p_on['advantage.weight']]) if dueling else p_on['q.weight']
    dout = db('dout').view(M * B, H)
    ck.fp32('head_dcore', dout[:T * B].to(F64), (G @ Wrows).reshape(-1))
    ck.zero('head_dcore_bootstrap_rows', dout[T * B:])
    gW = G.T @ X_on[:T * B]
    gb = G.sum(0)
    if dueling:
        ck.fp32('head_wgrad_value', L.grads['value.weight'].cpu().to(F64), gW[:1].reshape(-1))
        ck.fp32('head_wgrad_advantage', L.grads['advantage.weight'].cpu().to(F64), gW[1:].reshape(-1))
        ck.fp32('head_bgrad', torch.cat([L.grads['value.bias'], L.grads['advantage.bias']]).cpu().to(F64), gb)
    else:
        ck.fp32('head_wgrad', L.grads['q.weight'].cpu().to(F64), gW.reshape(-1))
        ck.fp32('head_bgrad', L.grads['q.bias'].cpu().to(F64), gb)
    loss_ref = float((w.to(F64).view(1, B) * torch.from_numpy(delta).to(F64) ** 2).sum() / (B * T))
    ck.fp32('loss', L.debug_buffer('loss')[:1].cpu().to(F64), torch.tensor([loss_ref], dtype=F64))
    L.close()
    ck.done(f'B{B}_A{A}_bi{burn_in}_T{T}_n{n}_{"dueling" if dueling else "plain"}_{"rescale" if rescale else "identity"}')


# ------------------------------------------------------------------------------------------------ determinism, graphs, sampler
def _state(L):
    return [t.clone() for t in (L.flat_params, L.exp_avg, L.exp_avg_sq, L.debug_buffer('priorities'))]


def test_deterministic_and_graph_replay_equals_eager():
    hp = _hp(9, 6, 3, 7, 2)
    _, gpu, w = _batch(hp, 5)
    w = w.cuda()
    runs = []
    for use_graph in (False, False, True):
        L, _ = _learner(hp, seed=7)
        for _ in range(3):
            L.learn(gpu, weights=w, use_graph=use_graph, sync_stats=False)
        torch.cuda.synchronize()
        runs.append(_state(L))
        if use_graph:
            assert len(L._graphs) == 1
        L.close()
    for a, b, c in zip(*runs):
        assert torch.equal(a, b) and torch.equal(a, c)


def test_priorities_reach_sampler_leaves():
    hp = _hp(6, 5, 2, 5, 2)
    _, gpu, w = _batch(hp, 6)
    S = GpuPrioritizedSampler(32, alpha=0.6, device='cuda')
    S.add(20)
    idxs = torch.tensor([3, 17, 0, 9, 11, 5], dtype=torch.int64, device='cuda')
    L, _ = _learner(hp)
    L.learn(gpu, weights=w.cuda(), idxs=idxs, sampler=S, use_graph=False)
    prio = L.debug_buffer('priorities')
    s, _, mp = S.trees()
    leaves = s[S.capacity + idxs]
    torch.testing.assert_close(leaves, prio ** 0.6, rtol=1e-12, atol=0)
    assert mp == pytest.approx(float(prio.max()))
    L.close()


def test_target_cadence_and_checkpoint_resume(tmp_path):
    hp = _hp(4, 6, 2, 4, 2, target_update_frequency=2)
    _, gpu, w = _batch(hp, 8)
    w = w.cuda()
    X, _ = _learner(hp, seed=11)
    X.learn(gpu, weights=w, use_graph=False)
    after1 = X.flat_params.clone()
    assert torch.equal(X.flat_target, after1)                # update 0 copies the target
    X.learn(gpu, weights=w, use_graph=False)
    assert torch.equal(X.flat_target, after1)                # update 1 does not
    X.learn(gpu, weights=w, use_graph=False)
    assert torch.equal(X.flat_target, X.flat_params)         # update 2 does
    Y, _ = _learner(hp, seed=11)
    Y.learn(gpu, weights=w, use_graph=False)
    Y.save_checkpoint(str(tmp_path / 'r2d2.pt'))
    Z, _ = _learner(hp, seed=99)
    Z.load_checkpoint(str(tmp_path / 'r2d2.pt'))
    for _ in range(2):
        Z.learn(gpu, weights=w, use_graph=False)
    for a, b in ((X.flat_params, Z.flat_params), (X.flat_target, Z.flat_target), (X.exp_avg, Z.exp_avg), (X.exp_avg_sq, Z.exp_avg_sq)):
        assert torch.equal(a, b)
    sd = Z.optimizer_state_dict()
    net = R2D2QNet(hp.num_actions, hp.dueling)
    opt = torch.optim.Adam(net.parameters(), lr=hp.learning_rate, eps=hp.adam_eps)
    opt.load_state_dict(sd)                                  # torch accepts the layout
    assert [tuple(v['exp_avg'].shape) for v in sd['state'].values()] == [tuple(p.shape) for p in net.parameters()]
    for L in (X, Y, Z):
        L.close()


# ------------------------------------------------------------------------------------------------ acting
def test_q_values_stepwise_equals_sequence_and_matches_torch():
    hp = _hp(4, 7, 2, 5, 2)
    cpu, gpu, _ = _batch(hp, 9, done_p=0.2)
    L, sd = _learner(hp)
    q_all, (hT, cT) = L.q_values(gpu['frame'], gpu['last_action'], gpu['reward'], gpu['done'], gpu['state'])
    state = gpu['state']
    rows = []
    for t in range(hp.seq_rows):
        q, state = L.q_values(gpu['frame'][t], gpu['last_action'][t], gpu['reward'][t], gpu['done'][t], state)
        rows.append(q)
    torch.testing.assert_close(torch.stack(rows), q_all, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(state[0], hT, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(state[1], cT, rtol=1e-6, atol=1e-6)
    net = R2D2QNet(hp.num_actions, hp.dueling)
    net.load_state_dict(sd)
    with torch.no_grad():
        q_ref, (h_ref, c_ref) = net(cpu['frame'], cpu['last_action'], cpu['reward'], cpu['done'], cpu['state'])
    assert rel_l2(q_all, q_ref) < 1e-2 and rel_l2(hT, h_ref) < 1e-2 and rel_l2(cT, c_ref) < 1e-2
    a, _ = L.predict(gpu['frame'][0], gpu['last_action'][0], gpu['reward'][0], gpu['done'][0], L.initial_state(hp.batch_size))
    assert a.shape == (hp.batch_size,) and a.dtype == torch.int64
    L.close()


def teardown_module():
    exact.summarize(RESULTS)
