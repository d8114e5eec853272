"""The LSTM actor step on the GPU: B200ActorModel(use_lstm=True) over srl_learner_forward_lstm_step (csrc/lstm.cu).
Checks the step kernel against fp64 on its own bf16 operands, the actor against the learner's rollout forward (the
behaviour / target logits V-trace compares), against the fp32 CPU ActorNet, its weight and state semantics, and the trainer's
batched actor loop."""
import queue
import threading
import time

import numpy as np
import pytest
import torch

from tests.helpers import nerr, rel_l2

pytestmark = pytest.mark.gpu

A = 6
H = 513 + A
HP = 576


def _actor(N, sd=None, seed=0):
    from scalerl_b200.algorithms.impala.gpu_actor import B200ActorModel
    return B200ActorModel(N, A, init_state_dict=sd, seed=seed, use_lstm=True)


def _cpu_actor(seed):
    from scalerl_b200.algorithms.utils.atari_model import ActorNet
    return ActorNet((4, 84, 84), A, use_lstm=True, seed=seed)


def _inputs(T1, N, seed, done_p=0.0):
    g = torch.Generator().manual_seed(seed)
    return dict(obs=torch.randint(0, 256, (T1, N, 4, 84, 84), dtype=torch.uint8, generator=g), reward=torch.randn(T1, N, generator=g),
                done=torch.rand(T1, N, generator=g) < done_p, action=torch.randint(0, A, (T1, N), generator=g))


def _state(N, seed, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    return tuple(torch.randn(2, N, H, generator=g) * scale for _ in range(2))


def _dev(d):
    return {k: v.cuda() for k, v in d.items()}


def _step_order():
    """packed row -> (gate q, hidden unit j) of the interleave in csrc/lstm.cu"""
    R = np.arange(4 * HP)
    tile, r = R // 128, R % 128
    u = 8 * ((r >> 4) & 3) + (r & 7)
    return 2 * (r >> 6) + ((r >> 3) & 1), 32 * tile + u


@pytest.mark.parametrize('N', [1, 13, 64, 256, 300])
def test_step_matches_fp64_on_its_own_operands(N):
    cpu = _cpu_actor(2)
    sd = cpu.state_dict()
    gpu = _actor(N, sd)
    x = _dev(_inputs(1, N, 5, done_p=0.3))
    x['done'][0, 0] = True
    h_in, c_in = (s.cuda() for s in _state(N, 6))
    _, _, _, (h1, c1) = gpu.forward_device(x['obs'], x['reward'], x['action'], x['done'], (h_in, c_in))
    xh = gpu._ctx.debug_buffer('lstm_step_xh').view(2, N, 2 * HP).double().cpu()
    w = gpu._ctx.debug_buffer('lstm_step_w').view(2, 4 * HP, 2 * HP).double().cpu()
    q, j = _step_order()
    keep = j < H
    m = (~x['done'][0]).double().cpu().view(N, 1)
    for l in range(2):
        # the operands are what the learner path would round: bf16 weights and bf16(m . h)
        wref = torch.zeros(4 * HP, 2 * HP, dtype=torch.float64)
        wih, whh = sd[f'rnn_layer.weight_ih_l{l}'], sd[f'rnn_layer.weight_hh_l{l}']
        rows = torch.from_numpy(q[keep] * H + j[keep])
        wref[torch.from_numpy(np.nonzero(keep)[0]), :H] = wih[rows].bfloat16().double()
        wref[torch.from_numpy(np.nonzero(keep)[0]), HP:HP + H] = whh[rows].bfloat16().double()
        assert torch.equal(w[l], wref), f'packed weights of layer {l}'
        assert torch.equal(xh[l, :, HP:HP + H], (m * h_in[l].double().cpu()).float().bfloat16().double())
        assert not xh[l, :, H:HP].any() and not xh[l, :, HP + H:].any()
        # fp64 gates from the kernel's own operands, then the cell
        gp = w[l] @ xh[l].T                                          # [4Hp, N], packed row order
        gates = torch.zeros(4, HP, N, dtype=torch.float64)
        gates[torch.from_numpy(q), torch.from_numpy(j)] = gp
        b = (sd[f'rnn_layer.bias_ih_l{l}'].double() + sd[f'rnn_layer.bias_hh_l{l}'].double()).view(4, H, 1)
        i_, f_, g_, o_ = (gates[k, :H] + b[k] for k in range(4))
        c = torch.sigmoid(f_) * (m.T * c_in[l].double().cpu().T) + torch.sigmoid(i_) * torch.tanh(g_)
        h = torch.sigmoid(o_) * torch.tanh(c)
        for name, got, ref in (('h', h1[l].double().cpu().T, h), ('c', c1[l].double().cpu().T, c)):
            assert rel_l2(got, ref) < 2e-5 and nerr(got, ref) < 1e-4, (l, name, rel_l2(got, ref), nerr(got, ref))
    assert torch.equal(xh[1, :, :H], h1[0].cpu().bfloat16().double())        # layer 1 reads bf16(h') of layer 0
    # a done column starts from the zero state: the same bits as a call with a zero state
    _, _, _, (h0, c0) = gpu.forward_device(x['obs'], x['reward'], x['action'], x['done'], (torch.zeros_like(h_in), torch.zeros_like(c_in)))
    d = x['done'][0]
    assert torch.equal(h0[:, d], h1[:, d]) and torch.equal(c0[:, d], c1[:, d])
    gpu.close()


@pytest.mark.parametrize('T,B', [(20, 32), (100, 16)])
def test_actor_steps_match_the_learner_rollout(T, B):
    """the behaviour logits of T+1 actor steps and the learner's target logits of the same rollout (the pair V-trace compares)"""
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    from tests.exact import record
    sd = _cpu_actor(4).state_dict()
    x = _inputs(T + 1, B, 7, done_p=0.1)
    x['done'][0, :4] = True                       # done at row 0
    x['done'][5:7, 4:6] = True                    # two dones in a row
    x = _dev(x)
    h0, c0 = (s.cuda() for s in _state(B, 8))
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, use_lstm=True), init_state_dict=sd, process_group=False)
    ref, (hT, cT) = L.forward(x, (h0, c0))
    gpu = _actor(B, sd).eval()
    state, lg, bs = (h0, c0), [], []
    for t in range(T + 1):
        a, b, _, state = gpu.forward_device(x['obs'][t:t + 1], x['reward'][t:t + 1], x['action'][t:t + 1], x['done'][t:t + 1], state)
        lg.append(a); bs.append(b)
    err = {'logits': nerr(torch.cat(lg).cpu(), ref['policy_logits'].cpu()), 'baseline': nerr(torch.cat(bs).cpu(), ref['baseline'].cpu()),
           'hT': nerr(state[0].cpu(), hT.cpu()), 'cT': nerr(state[1].cpu(), cT.cpu())}
    record('parity_fullsize.json', f'actor_lstm_vs_learner_T{T}_B{B}', err)
    assert all(v <= 1e-3 for v in err.values()), err
    gpu.close(); L.close()


def test_actor_matches_cpu_actornet_over_episodes():
    from scalerl_b200.algorithms.utils.atari_model import SyntheticAtariEnv
    N, steps = 8, 32
    cpu = _cpu_actor(3).eval()
    gpu = _actor(N, cpu.state_dict()).eval()
    envs = [SyntheticAtariEnv((4, 84, 84), A, seed=e, episode_len=5 + e % 4) for e in range(N)]
    cat = lambda outs: {k: torch.cat([o[k] for o in outs], dim=1) for k in outs[0]}
    env_output = cat([e.reset() for e in envs])
    s_cpu, s_gpu = cpu.initial_hidden_state(N), gpu.initial_hidden_state(N)
    dones = 0
    for t in range(steps):
        ref, s_cpu = cpu(env_output, s_cpu)
        out, s_gpu = gpu(env_output, s_gpu)
        assert s_gpu[0].is_cuda and tuple(s_gpu[0].shape) == (2, N, H)
        assert rel_l2(out['policy_logits'], ref['policy_logits']) < 2e-2, t
        assert rel_l2(out['baseline'], ref['baseline']) < 2e-2, t
        env_output = cat([e.step(ref['action'][0, i]) for i, e in enumerate(envs)])
        dones += int(env_output['done'].sum())
    assert dones >= N                               # every environment ended an episode at least once
    assert rel_l2(s_gpu[1].cpu(), s_cpu[1]) < 2e-2
    # training mode: N identical columns from the zero state -> N draws of one softmax per call
    gpu.train()
    same = {k: v[:, :1].expand(-1, N, *v.shape[2:]).contiguous() for k, v in env_output.items()}
    z = gpu.initial_hidden_state(N)
    counts, draws = torch.zeros(A), 0
    for _ in range(60):
        o, _ = gpu(same, z)
        counts += torch.bincount(o['action'].view(-1), minlength=A).float()
        draws += N
    p = torch.softmax(o['policy_logits'][0, 0], -1)
    sigma = torch.sqrt(p * (1 - p) / draws)
    assert torch.all((counts / draws - p).abs() < 5 * sigma + 1e-3), (counts / draws, p)
    gpu.close()


def test_weight_refresh_and_state_semantics():
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    N = 8
    gpu = _actor(N, seed=1).eval()
    env = _inputs(1, N, 2, done_p=0.3)
    state = _state(N, 3)
    a0, _ = gpu(env, state)
    old = gpu.state_dict()
    shared = _cpu_actor(9).share_memory().eval()
    assert gpu.refresh(shared.flat_params, version=5) and gpu.weights_version == 5
    a1, _ = gpu(env, state)
    ref, _ = shared(env, state)
    assert rel_l2(a1['policy_logits'], ref['policy_logits']) < 2e-2
    # the same check is sensitive to the LSTM weights: new encoder and heads with the old LSTM weights miss by far more
    hybrid = _cpu_actor(0).eval()
    hybrid.load_state_dict({k: (old[k] if k.startswith('rnn_layer.') else v) for k, v in shared.state_dict().items()})
    stale, _ = hybrid(env, state)
    assert rel_l2(stale['policy_logits'], ref['policy_logits']) > 0.1
    assert rel_l2(a1['policy_logits'], a0['policy_logits']) > 0.1
    # sync_from a learner in the same process
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=2, batch_size=2, num_actions=A, use_lstm=True), process_group=False, seed=4)
    gpu.sync_from(L, version=6)
    net = _cpu_actor(0).eval()
    net.load_state_dict({k: v.cpu() for k, v in L.state_dict().items()})
    a2, _ = gpu(env, state)
    ref2, _ = net(env, state)
    assert rel_l2(a2['policy_logits'], ref2['policy_logits']) < 2e-2 and gpu.weights_version == 6
    # host and device input states: the same outputs; the input state is never written
    host = tuple(s.clone() for s in state)
    dev = tuple(s.cuda() for s in state)
    dev_copy = tuple(s.clone() for s in dev)
    o_h, s_h = gpu(env, host)
    o_d, s_d = gpu(env, dev)
    for k in o_h:
        assert torch.equal(o_h[k], o_d[k]), k
    assert torch.equal(s_h[0], s_d[0]) and torch.equal(s_h[1], s_d[1])
    assert all(torch.equal(a, b) for a, b in zip(host, state)) and all(torch.equal(a, b) for a, b in zip(dev, dev_copy))
    # the returned state goes back in without a copy and is itself left as it was
    keep = tuple(s.clone() for s in s_d)
    gpu(env, s_d)
    assert all(torch.equal(a, b) for a, b in zip(s_d, keep))
    gpu.close(); L.close()


def test_trainer_batched_actor_loop(tmp_path):
    """get_action_batched with the LSTM GPU actor fills the same slots and initial states as with the CPU ActorNet"""
    from scalerl_b200.algorithms.impala.impala_atari import ImpalaArguments, ImpalaTrainer
    from scalerl_b200.algorithms.utils.atari_model import SyntheticAtariEnv
    from scalerl_b200.learner import B200ImpalaLearner
    N, T = 3, 4
    sd = _cpu_actor(11).state_dict()

    def run(model_fn, sub):
        a = ImpalaArguments(num_actors=1, batch_size=N, rollout_length=T, num_buffers=2 * N, use_lstm=True, num_actions=A,
                            output_dir=str(tmp_path / sub))
        seeds = iter(range(100))
        t = ImpalaTrainer(a, env_fn=lambda: SyntheticAtariEnv((4, 84, 84), A, seed=next(seeds), episode_len=3), actor_model_fn=model_fn)
        free_q, full_q = queue.SimpleQueue(), queue.SimpleQueue()
        for m in range(2 * N):
            free_q.put(m)
        for _ in range(N):
            free_q.put(None)
        th = threading.Thread(target=t.get_action_batched, args=(0, free_q, full_q, t.actor_model, t.buffers, t.rnn_state_buffers, N))
        th.start(); th.join(timeout=300)
        assert not th.is_alive()
        assert sorted(full_q.get() for _ in range(2 * N)) == list(range(2 * N))
        return t

    def cpu_fn():
        m = _cpu_actor(0).eval()
        m.load_state_dict(sd)
        return m

    ref = run(cpu_fn, 'cpu')
    got = run(lambda: _actor(N, sd).eval(), 'gpu')
    for m in range(2 * N):
        assert rel_l2(got.buffers['policy_logits'][m], ref.buffers['policy_logits'][m]) < 2e-2, m
        for i in range(2):
            if m < N:                               # first rollout: the initial state
                assert not got.rnn_state_buffers[m][i].any()
            else:
                assert rel_l2(got.rnn_state_buffers[m][i], ref.rnn_state_buffers[m][i]) < 2e-2, (m, i)
    assert float(got.rnn_state_buffers[N][0].abs().sum()) > 0      # the second rollout starts from a carried state
    # one learner step on the first rollout of every environment
    L = B200ImpalaLearner(got.hparams(), init_state_dict=sd, process_group=False)
    slots = list(range(N))
    batch = {k: torch.stack([got.buffers[k][m] for m in slots], dim=1).cuda() for k in ('obs', 'reward', 'done', 'action', 'policy_logits', 'episode_return')}
    state = tuple(torch.cat([got.rnn_state_buffers[m][i] for m in slots], dim=1).cuda() for i in range(2))
    stats = L.learn(batch, state)
    assert all(np.isfinite(stats[k]) for k in ('total_loss', 'pg_loss', 'baseline_loss', 'entropy_loss', 'grad_norm')), stats
    got.actor_model.close(); L.close()


def test_lstm_actor_throughput_is_recorded():
    """actor steps per second at N = 256 environments per call, host tensors in and out (the state stays on the device)"""
    from tests.exact import record
    N = 256
    gpu = _actor(N)
    env = _inputs(1, N, 3, done_p=0.05)
    state = gpu.initial_hidden_state(N)
    for _ in range(5):
        _, state = gpu(env, state)
    n = 50
    t0 = time.perf_counter()
    for _ in range(n):
        _, state = gpu(env, state)
    dt = time.perf_counter() - t0
    record('parity_fullsize.json', 'gpu_actor_lstm_N256', {'calls_per_sec': n / dt, 'env_steps_per_sec': n * N / dt, 'ms_per_call': dt / n * 1e3})
    gpu.close()
