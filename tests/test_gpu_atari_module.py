"""The trainable AtariNet drop-in on the H100: its encoder is the learner's encoder bit for bit, forward and backward; the
reference's own learn() statements run with the model, V-trace and loss imports swapped; and the autograd contract (per-call saved
state, accumulation, no double backward, determinism, CUDA-graph capture) holds."""
import pytest
import torch
from torch import nn

from oracle import impala_oracle as O
from oracle import ref_learner
from tests.helpers import assert_close, rel_l2
from tests.test_gpu_precision import _grad_tol, _mask_flips

pytestmark = pytest.mark.gpu

ENC = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'fc.weight', 'fc.bias')


def _learner(T, B, A, precision='bf16', use_lstm=False, params=None, **kw):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, precision=precision, use_lstm=use_lstm, **kw)
    return B200ImpalaLearner(hp, init_state_dict=params, process_group=False, seed=5)


def _net(A, precision='bf16', use_lstm=False, state_dict=None):
    from scalerl_b200.algorithms.utils.atari_model import AtariNet
    torch.manual_seed(0)
    net = AtariNet((4, 84, 84), A, use_lstm=use_lstm, precision=precision).cuda()
    if state_dict is not None:
        net.load_state_dict(state_dict)
    return net


def _batch(T, B, A, seed=0, done_p=0.1):
    return {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=seed, done_p=done_p).items()}


def _params(net):
    return dict(net.named_parameters())


@pytest.mark.parametrize('precision', ['bf16', 'fp32_split'])
@pytest.mark.parametrize('rows,B', [(21, 32), (2, 5)])
def test_forward_is_the_learners_forward(rows, B, precision):
    A = 6
    L = _learner(rows - 1, B, A, precision)
    net = _net(A, precision, state_dict=L.state_dict())
    batch = _batch(rows - 1, B, A, seed=rows)
    L.forward(batch)
    h = L.debug_buffer('h').view(-1, 512)[:rows * B]
    with torch.no_grad():
        core = net.encode(batch['obs'], batch['reward'], batch['action'])
    assert core.shape == (rows * B, 513 + A)
    assert torch.equal(core[:, :512], h)
    assert torch.equal(core[:, 512], batch['reward'].reshape(-1).clamp(-1, 1))
    assert torch.equal(core[:, 513:], nn.functional.one_hot(batch['action'].reshape(-1), A).float())


@pytest.mark.parametrize('T,B,A', [(20, 32, 6), (3, 5, 4)])
def test_backward_is_the_learners_backward(T, B, A):
    L = _learner(T, B, A)
    net = _net(A, state_dict=L.state_dict())
    batch = _batch(T, B, A, seed=T)
    L.forward_backward(batch)
    dh = L.debug_buffer('dh').view(-1, 512)[:T * B]
    core = net.encode(batch['obs'][:T], batch['reward'][:T], batch['action'][:T])
    dcore = torch.zeros_like(core)
    dcore[:, :512] = dh.float()
    core.backward(dcore)
    p = _params(net)
    for k in ENC:
        assert torch.equal(p[k].grad, L.grads[k]), k


def _learn(model, vtrace, loss_fn, batch, optimizer, hp, initial_rnn_state=()):
    """impala_atari.py:289-346 with the model, V-trace and loss modules passed in -> outputs, losses, pre-clip gradients, grad norm"""
    learner_outputs, _ = model(batch, initial_rnn_state)
    outputs = {k: v.detach().clone() for k, v in learner_outputs.items()}
    bootstrap_value = learner_outputs['baseline'][-1]
    batch = {key: tensor[1:] for key, tensor in batch.items()}
    learner_outputs = {key: tensor[:-1] for key, tensor in learner_outputs.items()}
    rewards = batch['reward']
    clipped_rewards = torch.clamp(rewards, -1, 1) if hp['reward_clipping'] == 'abs_one' else rewards
    discounts = (~batch['done']).float() * hp['discounting']
    vtrace_returns = vtrace.from_logits(behavior_policy_logits=batch['policy_logits'], target_policy_logits=learner_outputs['policy_logits'],
                                        actions=batch['action'], discounts=discounts, rewards=clipped_rewards,
                                        values=learner_outputs['baseline'], bootstrap_value=bootstrap_value)
    pg_loss = loss_fn.compute_policy_gradient_loss(learner_outputs['policy_logits'], batch['action'], vtrace_returns.pg_advantages)
    baseline_loss = hp['baseline_cost'] * loss_fn.compute_baseline_loss(vtrace_returns.vs - learner_outputs['baseline'])
    entropy_loss = hp['entropy_cost'] * loss_fn.compute_entropy_loss(learner_outputs['policy_logits'])
    total_loss = pg_loss + baseline_loss + entropy_loss
    optimizer.zero_grad()
    total_loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
    grad_norm = float(nn.utils.clip_grad_norm_(model.parameters(), hp['max_grad_norm']))
    optimizer.step()
    losses = [float(x) for x in (pg_loss, baseline_loss, entropy_loss, total_loss)]
    return dict(outputs=outputs, losses=losses, grads=grads, grad_norm=grad_norm)


def _hp(clip):
    return dict(reward_clipping=clip, discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, max_grad_norm=40.0)


def _drop_ins():
    from scalerl_b200.algorithms.impala import loss_fn, vtrace
    return vtrace, loss_fn


@pytest.mark.skipif(not ref_learner.available(), reason='oracle/_ref (the reference modules) is not built')
@pytest.mark.parametrize('T,B,A,seed,bseed,clip', [(3, 5, 4, 1, 10, 'none'), (20, 32, 6, 3, 7, 'abs_one')])
def test_reference_learn_with_three_imports_swapped_split_mode(T, B, A, seed, bseed, clip):
    params = O.init_params(A, seed=seed)
    batch_cpu = O.synthetic_batch(T, B, A, seed=bseed, done_p=0.05)
    ref = ref_learner.ReferenceLearner(num_actions=A, state_dict=params, reward_clipping=clip)
    want = _learn(ref.model, ref.vtrace, ref.loss_fn, batch_cpu, ref.optimizer, _hp(clip))
    net = _net(A, 'fp32_split', state_dict=params)
    before = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    opt = torch.optim.RMSprop(net.parameters(), lr=1e-4, momentum=0.0, eps=1e-5, alpha=0.99)
    vt, lf = _drop_ins()
    got = _learn(net, vt, lf, {k: v.cuda() for k, v in batch_cpu.items()}, opt, _hp(clip))
    for g, w in zip(got['losses'], want['losses']):
        assert abs(g - w) <= 1e-5 * max(1.0, abs(w)), (got['losses'], want['losses'])
    assert rel_l2(got['outputs']['policy_logits'], want['outputs']['policy_logits']) < 1e-5
    assert rel_l2(got['outputs']['baseline'], want['outputs']['baseline']) < 1e-5
    # ReLU ties: the module's forward is the learner's, so the learner's activations count the units whose mask flips against fp32
    L = _learner(T, B, A, 'fp32_split', params=params, reward_clipping=clip)
    L.forward({k: v.cuda() for k, v in batch_cpu.items()})
    flips, _, _ = _mask_flips(L, params, batch_cpu, T, B)
    tol = 2e-3 if (T, B) == (20, 32) else _grad_tol(flips)
    assert sorted(got['grads']) == sorted(want['grads'])
    for k in O.PARAM_ORDER:
        assert rel_l2(got['grads'][k], want['grads'][k]) < tol, (k, flips)
    # post-step weights: torch's clip + RMSprop on the module's gradients, against the oracle's update of the same gradients
    g_dev = {k: v.cpu().clone() for k, v in got['grads'].items()}
    O.clip_grad_norm(g_dev, 40.0)
    O.rmsprop_step(before, g_dev, O.new_opt_state(before)['square_avg'], 1e-4, 0.99, 1e-5)
    for k, v in net.state_dict().items():
        assert_close(v, before[k], 2e-6, f'post-step {k}')


def test_reference_learn_with_three_imports_swapped_bf16_against_the_learner():
    T, B, A = 20, 32, 6
    params = O.init_params(A, seed=3)
    batch = _batch(T, B, A, seed=7, done_p=0.05)
    L = _learner(T, B, A, params=params)
    L.forward_backward(batch)
    net = _net(A, state_dict=params)
    opt = torch.optim.RMSprop(net.parameters(), lr=1e-4, eps=1e-5, alpha=0.99)
    vt, lf = _drop_ins()
    got = _learn(net, vt, lf, batch, opt, _hp('abs_one'))
    for k in O.PARAM_ORDER:
        assert_close(got['grads'][k], L.grads[k], 5e-3, k)


def _core_loss(core, w):
    return (core[:, :512] * w).sum()


def _encode(net, b, rows=None):
    s = slice(None) if rows is None else slice(0, rows)
    return net.encode(b['obs'][s], b['reward'][s], b['action'][s])


def _grads(net):
    return {k: p.grad.clone() for k, p in _params(net).items() if p.grad is not None}


def test_autograd_semantics():
    T, B, A = 3, 4, 6
    net = _net(A)
    b1, b2 = _batch(T, B, A, seed=1), _batch(T, B, A, seed=2)
    w = torch.randn((T + 1) * B, 512, device='cuda', generator=torch.Generator(device='cuda').manual_seed(0))
    net.zero_grad(set_to_none=True)
    _core_loss(_encode(net, b1), w).backward()
    g1 = _grads(net)
    net.zero_grad(set_to_none=True)
    _core_loss(_encode(net, b2), w).backward()
    g2 = _grads(net)
    assert sorted(g1) == list(sorted(ENC))
    want = {k: g1[k] + g2[k] for k in g1}
    # two interleaved forwards, one backward of the summed loss
    net.zero_grad(set_to_none=True)
    c1, c2 = _encode(net, b1), _encode(net, b2)
    (_core_loss(c1, w) + _core_loss(c2, w)).backward()
    assert all(torch.equal(_grads(net)[k], want[k]) for k in want)
    # a no_grad forward between a forward and its backward
    net.zero_grad(set_to_none=True)
    c1 = _encode(net, b1)
    with torch.no_grad():
        _encode(net, b2)
    _core_loss(c1, w).backward()
    assert all(torch.equal(_grads(net)[k], g1[k]) for k in g1)
    # accumulation over two backward() calls
    net.zero_grad(set_to_none=False)
    _core_loss(_encode(net, b1), w).backward()
    _core_loss(_encode(net, b2), w).backward()
    assert all(torch.equal(_grads(net)[k], want[k]) for k in want)
    # nothing is kept after a forward with frozen encoder parameters (or under no_grad); a differentiable one keeps its block
    from scalerl_b200.algorithms.utils.atari_model import encoder_block_sizes
    saved_bytes = encoder_block_sizes((T + 1) * B)[0]
    core_bytes = (T + 1) * B * (513 + A) * 4

    def held(fn):
        torch.cuda.synchronize()
        m0 = torch.cuda.memory_allocated()
        out = fn()
        torch.cuda.synchronize()
        return torch.cuda.memory_allocated() - m0, out

    kept, c = held(lambda: _encode(net, b1))
    assert kept >= saved_bytes + core_bytes
    del c
    with torch.no_grad():
        kept, c = held(lambda: _encode(net, b1))
    assert kept < core_bytes + 1024
    del c
    for k in ENC:
        _params(net)[k].requires_grad_(False)
    kept, c = held(lambda: _encode(net, b1))
    assert kept < core_bytes + 1024 and not c.requires_grad
    del c
    for k in ENC:
        _params(net)[k].requires_grad_(True)
    # no double backward
    c = _encode(net, b1)
    g = torch.autograd.grad((c[:, :512] ** 2).sum(), net.fc.weight, create_graph=True)[0]
    with pytest.raises(RuntimeError):
        g.sum().backward()


@pytest.mark.parametrize('precision', ['bf16', 'fp32_split'])
def test_determinism(precision):
    T, B, A = 20, 32, 6
    net = _net(A, precision)
    b = _batch(T, B, A, seed=4)
    w = torch.randn((T + 1) * B, 512, device='cuda', generator=torch.Generator(device='cuda').manual_seed(1))
    runs = []
    for _ in range(2):
        net.zero_grad(set_to_none=True)
        c = _encode(net, b)
        _core_loss(c, w).backward()
        runs.append((c.detach().clone(), _grads(net)))
    assert torch.equal(runs[0][0], runs[1][0])
    for k in ENC:
        assert torch.equal(runs[0][1][k], runs[1][1][k]), k


def test_graph_capture():
    T, B, A = 5, 8, 6
    net = _net(A).eval()                  # argmax actions: the captured step draws no random numbers
    static = _batch(T, B, A, seed=1)

    def step():
        out, _ = net(static)
        loss = (out['policy_logits'] ** 2).sum() + out['baseline'].sum() + _core_loss(_encode(net, static), 1e-3)
        loss.backward()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            net.zero_grad(set_to_none=True)
            step()
    torch.cuda.current_stream().wait_stream(side)
    net.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    fresh = _batch(T, B, A, seed=2)
    for k in ('obs', 'reward', 'action'):
        static[k].copy_(fresh[k])
    graph.replay()
    torch.cuda.synchronize()
    replayed = _grads(net)
    assert sorted(replayed) == sorted(k for k, _ in net.named_parameters())
    net.zero_grad(set_to_none=True)
    step()
    eager = _grads(net)
    for k in eager:
        assert torch.equal(replayed[k], eager[k]), k


def test_lstm_module():
    T, B, A = 5, 4, 6
    L = _learner(T, B, A, use_lstm=True)
    net = _net(A, use_lstm=True, state_dict=L.state_dict())
    batch = _batch(T, B, A, seed=3, done_p=0.2)
    want, _ = L.forward(batch)
    state = tuple(s.cuda() for s in net.initial_hidden_state(B))
    with torch.no_grad():
        got, (hT, cT) = net(batch, state)
    assert hT.shape == (2, B, 513 + A) and got['action'].shape == (T + 1, B)
    assert_close(got['policy_logits'], want['policy_logits'], 1e-2, 'logits')
    assert_close(got['baseline'], want['baseline'], 1e-2, 'baseline')
    opt = torch.optim.RMSprop(net.parameters(), lr=1e-4, eps=1e-5, alpha=0.99)
    vt, lf = _drop_ins()
    r = _learn(net, vt, lf, batch, opt, _hp('abs_one'), state)
    assert all(torch.isfinite(torch.tensor(r['losses'])))
    assert len(r['grads']) == 20 == len(list(net.parameters()))
    assert all(bool(torch.isfinite(g).all()) for g in r['grads'].values())
