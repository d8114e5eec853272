"""The trainable AtariNet's LSTM core on the H100 (use_lstm=True, bf16): the stand-alone core runs the learner's LSTM kernels bit for
bit; the initial-state gradients join two calls exactly where one call carries the recurrence; it matches fp32 torch; the reference's
learn() with the model, V-trace and loss imports swapped matches B200ImpalaLearner(use_lstm=True); and the autograd contract (per-call
saved state, accumulation, nothing kept without a graph, no double backward, determinism, CUDA-graph capture) holds."""
import numpy as np
import pytest
import torch

from oracle import impala_oracle as O
from oracle import ref_learner
from tests.helpers import assert_close, nerr, rel_l2
from tests.test_gpu_atari_module import ENC, _batch, _drop_ins, _hp, _learn, _learner, _net

pytestmark = pytest.mark.gpu

LSTM = tuple(f'rnn_layer.{w}_l{l}' for l in (0, 1) for w in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'))


def _case(T1, B, A, seed, done_p=0.1):
    """random core / state on the device; done rows include row 0 and two in a row"""
    H = 513 + A
    g = torch.Generator().manual_seed(seed)
    core = torch.randn(T1, B, H, generator=g) * 0.5
    done = torch.rand(T1, B, generator=g) < done_p
    done[0, 0] = True
    if T1 >= 3:
        done[1:3, B - 1] = True
    state = tuple(torch.randn(2, B, H, generator=g) * 0.3 for _ in range(2))
    return core.cuda(), done.cuda(), tuple(s.cuda() for s in state)


def _leaves(lp):
    return {k: v.detach().clone().cuda().requires_grad_(True) for k, v in lp.items()}


def _core(ws, core, done, state):
    """(out, hT, cT) of the stand-alone core under autograd"""
    from scalerl_b200.algorithms.utils.atari_model import _LstmCore
    A = core.shape[-1] - 513
    return _LstmCore.apply(A, core.contiguous(), done.contiguous().view(torch.uint8), state[0].contiguous(), state[1].contiguous(),
                           *[ws[k] for k in LSTM])


@pytest.mark.parametrize('T1,B', [(21, 32), (101, 16), (5, 3), (2, 130)])
def test_core_runs_the_learners_lstm_kernels(T1, B):
    from scalerl_b200.lstm import B200LstmCore
    A = 6
    H = 513 + A
    lp = O.init_lstm_params(A, seed=T1)
    core, done, state = _case(T1, B, A, seed=T1 * 1000 + B)
    ref = B200LstmCore(T1, B, H, state_dict=lp)
    want, (wh, wc) = ref.forward(core, done, state)
    ws = _leaves(lp)
    c = core.clone().requires_grad_(True)
    out, hT, cT = _core(ws, c, done, state)
    assert torch.equal(out, want) and torch.equal(hT, wh) and torch.equal(cT, wc)
    dout = torch.randn(T1, B, H, generator=torch.Generator().manual_seed(T1)).cuda()
    dout[-1] = 0                      # the learner's bootstrap row: no gradient, so the extra row of the core adds exact zeros
    out.backward(dout)
    ref.zero_grad()
    dcore = ref.backward(dout[:-1])
    assert torch.equal(c.grad[:-1], dcore)
    for k in LSTM:
        assert torch.equal(ws[k].grad, ref.grads[k]), (k, nerr(ws[k].grad.cpu().numpy(), ref.grads[k].cpu().numpy()))


@pytest.mark.parametrize('k', [1, 7])
def test_state_gradients_join_a_split_rollout(k):
    T1, B, A = 21, 8, 6
    H = 513 + A
    lp = O.init_lstm_params(A, seed=k)
    core, done, state = _case(T1, B, A, seed=40 + k)
    done[k, : B // 2] = True          # a done at the split row, and columns that carry the state across it
    done[k, B // 2:] = False
    w = torch.randn(T1, B, H, generator=torch.Generator().manual_seed(k)).cuda()

    def run(pieces):
        ws = _leaves(lp)
        c = core.clone().requires_grad_(True)
        h0, c0 = (s.clone().requires_grad_(True) for s in state)
        s, outs = (h0, c0), []
        for a, b in pieces:
            o, hT, cT = _core(ws, c[a:b], done[a:b], s)
            outs.append(o)
            s = (hT, cT)
        out = torch.cat(outs)
        (out * w).sum().backward()
        return out.detach(), c.grad, h0.grad, c0.grad, {n: ws[n].grad for n in LSTM}

    full, split = run([(0, T1)]), run([(0, k), (k, T1)])
    for name, a, b in zip(('out', 'dcore', 'dh0', 'dc0'), full[:4], split[:4]):
        assert torch.equal(a, b), name
    assert float(full[2].abs().max()) > 0 and float(full[3].abs().max()) > 0
    for n in LSTM:                    # the split sums two weight-gradient GEMMs and two bias reductions
        assert_close(split[4][n], full[4][n], 1e-5, n)


def test_core_against_fp32_torch():
    T1, B, A = 21, 16, 6
    lp = O.init_lstm_params(A, seed=2)
    core, done, state = _case(T1, B, A, seed=5)
    g = torch.Generator().manual_seed(6)
    dout, dhT, dcT = torch.randn(T1, B, 513 + A, generator=g), torch.randn(2, B, 513 + A, generator=g), torch.randn(2, B, 513 + A, generator=g)
    ls = {k: v.clone().requires_grad_(True) for k, v in lp.items()}
    cr = core.cpu().requires_grad_(True)
    sr = tuple(s.cpu().requires_grad_(True) for s in state)
    ref, (rh, rc) = O.lstm_core_forward(ls, cr, done.cpu(), sr)
    ((ref * dout).sum() + (rh * dhT).sum() + (rc * dcT).sum()).backward()
    ws = _leaves(lp)
    c = core.clone().requires_grad_(True)
    s = tuple(x.clone().requires_grad_(True) for x in state)
    out, hT, cT = _core(ws, c, done, s)
    ((out * dout.cuda()).sum() + (hT * dhT.cuda()).sum() + (cT * dcT.cuda()).sum()).backward()
    assert rel_l2(out, ref) < 1e-2 and rel_l2(hT, rh) < 1e-2 and rel_l2(cT, rc) < 1e-2
    assert rel_l2(c.grad, cr.grad) < 3e-2
    assert rel_l2(s[0].grad, sr[0].grad) < 3e-2 and rel_l2(s[1].grad, sr[1].grad) < 3e-2
    for k in LSTM:
        assert rel_l2(ws[k].grad, ls[k].grad) < 3e-2, k


@pytest.mark.parametrize('T,B', [(20, 32), (100, 16)])
def test_reference_learn_with_three_imports_swapped(T, B):
    A = 6
    params = {**O.init_params(A, seed=3), **O.init_lstm_params(A, seed=3)}
    batch_cpu = O.synthetic_batch(T, B, A, seed=7, done_p=0.05)
    batch = {k: v.cuda() for k, v in batch_cpu.items()}
    g = torch.Generator().manual_seed(T)
    state_cpu = tuple(torch.randn(2, B, 513 + A, generator=g) * 0.3 for _ in range(2))
    state = tuple(s.cuda() for s in state_cpu)
    L = _learner(T, B, A, use_lstm=True, params=params)
    L._set_rnn_state(state)
    L.forward_backward(batch)
    net = _net(A, use_lstm=True, state_dict=params)
    opt = torch.optim.RMSprop(net.parameters(), lr=1e-4, eps=1e-5, alpha=0.99)
    vt, lf = _drop_ins()
    got = _learn(net, vt, lf, batch, opt, _hp('abs_one'), state)
    assert sorted(got['grads']) == sorted(params)
    for k in params:
        assert_close(got['grads'][k], L.grads[k], 5e-3, k)
    if not ref_learner.available():
        return
    ref = ref_learner.ReferenceLearner(num_actions=A, use_lstm=True, state_dict=params)
    want = _learn(ref.model, ref.vtrace, ref.loss_fn, batch_cpu, ref.optimizer, _hp('abs_one'), state_cpu)
    for k in params:
        e = rel_l2(got['grads'][k], want['grads'][k])
        assert e < (0.1 if k in ENC else 1e-2), (k, e)


def _lstm_grads(net):
    return {k: p.grad.clone() for k, p in net.named_parameters() if k.startswith('rnn_layer.') and p.grad is not None}


def test_autograd_semantics():
    from scalerl_b200.algorithms.utils.atari_model import lstm_block_sizes
    T1, B, A = 6, 4, 6
    H = 513 + A
    net = _net(A, use_lstm=True)
    (c1, d1, s1), (c2, d2, s2) = _case(T1, B, A, seed=1), _case(T1, B, A, seed=2)
    w = torch.randn(T1, B, H, generator=torch.Generator().manual_seed(0)).cuda()

    def loss(core, done, state):
        out, (hT, cT) = net._lstm_core(core, done, state)
        return (out * w).sum() + hT.sum() + (cT ** 2).sum()

    net.zero_grad(set_to_none=True)
    loss(c1, d1, s1).backward()
    g1 = _lstm_grads(net)
    net.zero_grad(set_to_none=True)
    loss(c2, d2, s2).backward()
    g2 = _lstm_grads(net)
    assert sorted(g1) == sorted(LSTM)
    want = {k: g1[k] + g2[k] for k in g1}
    # two interleaved forwards, one backward of the summed loss
    net.zero_grad(set_to_none=True)
    (loss(c1, d1, s1) + loss(c2, d2, s2)).backward()
    assert all(torch.equal(_lstm_grads(net)[k], want[k]) for k in want)
    # a no_grad forward between a forward and its backward
    net.zero_grad(set_to_none=True)
    l1 = loss(c1, d1, s1)
    with torch.no_grad():
        loss(c2, d2, s2)
    l1.backward()
    assert all(torch.equal(_lstm_grads(net)[k], g1[k]) for k in g1)
    # accumulation over two backward() calls
    net.zero_grad(set_to_none=False)
    loss(c1, d1, s1).backward()
    loss(c2, d2, s2).backward()
    assert all(torch.equal(_lstm_grads(net)[k], want[k]) for k in want)
    # a differentiable call keeps its saved block; nothing is kept under no_grad or with frozen parameters and a core without grad
    saved_bytes = lstm_block_sizes(T1, B, A)[0]
    outputs = (T1 * B * H + 4 * B * H) * 4

    def held(fn):
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated()
        r = fn()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated() - m0, r

    kept, r = held(lambda: net._lstm_core(c1, d1, s1))
    assert kept >= saved_bytes + outputs
    del r
    with torch.no_grad():
        kept, r = held(lambda: net._lstm_core(c1, d1, s1))
    assert kept < outputs + 4096
    del r
    before = _lstm_grads(net)
    for p in net.rnn_layer.parameters():
        p.requires_grad_(False)
    kept, r = held(lambda: net._lstm_core(c1, d1, s1))
    assert kept < outputs + 4096 and not r[0].requires_grad
    del r
    # ... but a core that needs a gradient still gets one through the frozen parameters, which keep theirs
    cg = c1.clone().requires_grad_(True)
    out, _ = net._lstm_core(cg, d1, s1)
    (out * w).sum().backward()
    assert cg.grad is not None and all(torch.equal(_lstm_grads(net)[k], before[k]) for k in before)
    for p in net.rnn_layer.parameters():
        p.requires_grad_(True)
    # no double backward
    out, _ = net._lstm_core(c1, d1, s1)
    g = torch.autograd.grad((out ** 2).sum(), net.rnn_layer.weight_hh_l1, create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()


def _module_step(net, batch, state, w):
    out, (hT, cT) = net(batch, state)
    loss = (out['policy_logits'] ** 2).sum() + out['baseline'].sum() + (hT * w).sum() + cT.sum()
    loss.backward()


def test_determinism():
    T, B, A = 20, 32, 6
    net = _net(A, use_lstm=True).eval()
    b = _batch(T, B, A, seed=4, done_p=0.1)
    _, _, state = _case(T + 1, B, A, seed=9)
    w = torch.randn(2, B, 513 + A, generator=torch.Generator().manual_seed(1)).cuda()
    runs = []
    for _ in range(2):
        net.zero_grad(set_to_none=True)
        _module_step(net, b, state, w)
        runs.append({k: p.grad.clone() for k, p in net.named_parameters()})
    assert len(runs[0]) == 20
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_graph_capture():
    T, B, A = 5, 8, 6
    net = _net(A, use_lstm=True).eval()      # argmax actions: the captured step draws no random numbers
    static = _batch(T, B, A, seed=1, done_p=0.2)
    _, _, state = _case(T + 1, B, A, seed=3)
    w = torch.randn(2, B, 513 + A, generator=torch.Generator().manual_seed(2)).cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            net.zero_grad(set_to_none=True)
            _module_step(net, static, state, w)
    torch.cuda.current_stream().wait_stream(side)
    net.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _module_step(net, static, state, w)
    fresh = _batch(T, B, A, seed=2, done_p=0.2)
    for k in ('obs', 'reward', 'action', 'done'):
        static[k].copy_(fresh[k])
    _, _, fresh_state = _case(T + 1, B, A, seed=4)
    for s, f in zip(state, fresh_state):
        s.copy_(f)
    graph.replay()
    torch.cuda.synchronize()
    replayed = {k: p.grad.clone() for k, p in net.named_parameters()}
    assert len(replayed) == 20
    net.zero_grad(set_to_none=True)
    _module_step(net, static, state, w)
    for k, p in net.named_parameters():
        assert torch.equal(replayed[k], p.grad), k
    assert not np.isnan(float(sum(g.sum() for g in replayed.values())))
