"""The Ape-X learner step on the H100 (B200ApexLearner / srl_apex_learner_*):
  1. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py): q, y, priorities and loss to 1e-5, every
     gradient to rel-L2 1e-4 when no ReLU mask differs from fp32 (2e-2 otherwise, and then every flipped unit must be a genuine tie:
     the tie accounting of test_gpu_precision.py), the weights after the step
     against the oracle's Adam on the device gradients to 2e-6;
  2. bf16: the tail against fp64 evaluated on its own operands (the core rows and the fp32 head weights);
  3. bf16: the encoder gradients equal srl_encoder_backward called directly on the tail's dcore, bit for bit;
  4. the priorities reach the sampler's trees (last occurrence of a repeated idx wins);
  5. repeated runs and graph replay give the same parameters bit for bit, with the device step count advancing;
  6. the target update is soft_target_update's arithmetic on the reference's cadence;
  7. checkpoints load into torch.optim.Adam(AtariQNet(...).parameters()), and a resumed run equals an uninterrupted one;
  8. q_values / predict against AtariQNet on the CPU.
The measured errors are written to $SRL_RESULTS_DIR/apex.json when SRL_RESULTS_DIR is set."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import apex_oracle as O
from oracle.per_oracle import PerOracle
from scalerl_b200 import _lib
from tests import layer_ref as R
from scalerl_b200.algorithms.apex import APEX_PARAM_NAMES, ApexHParams, AtariQNet, B200ApexLearner
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler

pytestmark = pytest.mark.gpu
F64 = torch.float64


def _record(name, obj):
    d = os.environ.get('SRL_RESULTS_DIR')
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, 'apex.json')
    cur = json.load(open(p)) if os.path.exists(p) else {}
    cur[name] = obj
    json.dump(cur, open(p, 'w'), indent=1)


def rel_l2(a, b):
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def nmax(a, b):
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))


def _nets(A, seed=0):
    torch.manual_seed(seed)
    on, tg = AtariQNet(A), AtariQNet(A)
    return ({k: v.detach().clone() for k, v in on.state_dict().items()}, {k: v.detach().clone() for k, v in tg.state_dict().items()})


def _batch(B, A, seed=0, done_p=0.25, device='cpu'):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    act = torch.randint(0, A, (B,), generator=g)
    rew = torch.randn(B, generator=g)
    nobs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    done = torch.rand(B, generator=g) < done_p
    w = torch.rand(B, generator=g) + 0.1
    return tuple(t.to(device) for t in (obs, act, rew, nobs, done)), w.to(device)


def _learner(B, A, on, tg, **kw):
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, **kw), init_state_dict=on)
    L.load_state_dict(tg, target=True)
    return L


def _mask_flips(L, params, obs, B):
    """test_gpu_precision.py's tie accounting on the forward over s: the learner's ReLU masks (a1, a2, a3 high parts and h, > 0) against
    fp32 pre-activations on the CPU -> (flipped units, units, worst |z| / rms of a flipped unit)"""
    import torch.nn.functional as F
    x = obs.float() / 255.0
    z1 = F.conv2d(x, params['conv1.weight'], params['conv1.bias'], stride=4)
    z2 = F.conv2d(F.relu(z1), params['conv2.weight'], params['conv2.bias'], stride=2)
    z3 = F.conv2d(F.relu(z2), params['conv3.weight'], params['conv3.bias'], stride=1)
    zh = F.linear(F.relu(z3).reshape(B, -1), params['fc.weight'], params['fc.bias'])
    g1 = R.a1_planes_to_nchw(L.debug_buffer('a1').float().cpu(), B)
    g2 = R.nhwc_to_nchw(L.debug_buffer('a2').float().cpu(), B, 9)
    g3 = R.nhwc_to_nchw(L.debug_buffer('a3').float().cpu(), B, 7)
    gh = L.debug_buffer('core').view(B, 514)[:, :512].cpu()
    flips, units, worst = 0, 0, 0.0
    for z, g in ((z1, g1), (z2, g2), (z3, g3), (zh, gh)):
        bad = (z > 0) != (g > 0)
        flips += int(bad.sum())
        units += z.numel()
        if bad.any():
            worst = max(worst, float(z[bad].abs().max() / z.pow(2).mean().sqrt()))
    return flips, units, worst


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (5, 4), (512, 18)])
def test_split_against_fp32_oracle(B, A, double, clip):
    on, tg = _nets(A, seed=B)
    (obs, act, rew, nobs, done), w = _batch(B, A, seed=B + A)
    L = _learner(B, A, on, tg, precision='fp32_split', double_dqn=double, max_grad_norm=clip, priority_eps=0.0)
    L.learn(tuple(t.cuda() for t in (obs, act, rew, nobs, done)), weights=w.cuda(), use_graph=False)
    ref = O.learn_step(on, tg, obs, act, rew, nobs, done, weights=w, gamma=0.99, double_dqn=double, max_grad_norm=clip)
    q, y, prio, loss = L.debug_buffer('q'), L.debug_buffer('y'), L.debug_buffer('priorities'), float(L.debug_buffer('loss')[0])
    err = {'q': nmax(q, ref['q']), 'y': nmax(y, ref['y']), 'priorities': nmax(prio, ref['td']),
           'loss': abs(loss - ref['loss']) / max(abs(ref['loss']), 1e-30)}
    flips, units, worst = _mask_flips(L, on, obs, B)
    gerr = {n: rel_l2(L.grads[n], ref['grads'][n]) for n in APEX_PARAM_NAMES}
    post = O.adam_on_grads(on, {n: L.grads[n] for n in APEX_PARAM_NAMES}, max_grad_norm=clip)
    perr = max(float((L.params[n].cpu() - post[n]).abs().max()) for n in APEX_PARAM_NAMES)
    _record(f'split_B{B}_A{A}_double{int(double)}_clip{clip}', dict(err, grads=gerr, relu_mask_flips=flips, relu_units=units,
                                                                         worst_flipped_margin=worst, post_step_max_abs=perr))
    for k, v in err.items():
        assert v <= 1e-5, (k, v)
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)       # only genuine ties may flip
    gtol = 1e-4 if flips == 0 else 2e-2
    for n, v in gerr.items():
        assert v <= gtol, (n, v, flips)
    assert perr <= 2e-6, perr


# ---------------------------------------------------------------------------------------------------------------- 2, 3
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (512, 18)])
def test_bf16_tail_against_fp64_and_encoder_backward(B, A, double):
    on, tg = _nets(A, seed=7)
    batch, w = _batch(B, A, seed=3, device='cuda')
    obs, act, rew, nobs, done = batch
    gamma = 0.97
    L = _learner(B, A, on, tg, double_dqn=double, gamma=gamma, priority_eps=0.0)
    pre = L.state_dict()
    L.learn(batch, weights=w, use_graph=False)
    core = L.debug_buffer('core').view(B, 514).to(F64)
    h, hnt = core[:, :512], L.debug_buffer('core_next_target').view(B, 514)[:, :512].to(F64)
    Wq, bq = pre['q.weight'].to(F64), pre['q.bias'].to(F64)
    Wt, bt = tg['q.weight'].cuda().to(F64), tg['q.bias'].cuda().to(F64)
    a = act.long()
    q_all = h @ Wq.T + bq
    q = q_all.gather(1, a[:, None]).squeeze(1)
    qt = hnt @ Wt.T + bt
    if double:
        hn = L.debug_buffer('core_next').view(B, 514)[:, :512].to(F64)
        astar = (hn @ Wq.T + bq).argmax(1)
    else:
        astar = qt.argmax(1)
    y = rew.to(F64) + gamma * qt.gather(1, astar[:, None]).squeeze(1) * (1 - done.to(F64))
    delta = q - y
    loss = (w.to(F64) * delta ** 2).mean()
    dq = 2 * w.to(F64) * delta / B
    onehot = torch.nn.functional.one_hot(a, A).to(F64) * dq[:, None]
    gW, gb = onehot.T @ h, onehot.sum(0)
    dcore = dq[:, None] * Wq[a]
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'q': (L.debug_buffer('q'), q), 'y': (L.debug_buffer('y'), y), 'delta': (L.debug_buffer('priorities'), delta.abs()),
             'q.weight': (L.grads['q.weight'], gW), 'q.bias': (L.grads['q.bias'], gb), 'dcore': (dev_dcore[:, :512], dcore)}
    err = {k: (rel_l2(u, v), nmax(u, v)) for k, (u, v) in pairs.items()}
    err['loss'] = (abs(float(L.debug_buffer('loss')[0]) - float(loss)) / float(loss),) * 2
    _record(f'bf16_tail_B{B}_A{A}_double{int(double)}', err)
    for k, (r, m) in err.items():
        assert r <= 2e-5 and m <= 1e-4, (k, r, m)
    assert not bool(dev_dcore[:, 512:].any())

    # 3: the encoder gradients of the step are srl_encoder_backward on the tail's dcore, bit for bit
    lib = _lib.lib()
    E = C.c_void_p()
    _lib.check(lib.srl_encoder_create(0, C.byref(E)), 'encoder_create')
    try:
        sb, kb = C.c_int64(), C.c_int64()
        _lib.check(lib.srl_encoder_sizes(B, 0, C.byref(sb), C.byref(kb)), 'encoder_sizes')
        saved = torch.empty(sb.value, dtype=torch.uint8, device='cuda')
        scratch = torch.empty(kb.value, dtype=torch.uint8, device='cuda')
        ws = [pre[n].cuda().contiguous() for n in APEX_PARAM_NAMES[:8]]
        gs = [torch.empty_like(t) for t in ws]
        core_out = torch.empty(B, 514, device='cuda')
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.srl_encoder_forward(E, obs.data_ptr(), rew.data_ptr(), act.data_ptr(), B, 1, (C.c_void_p * 8)(*[t.data_ptr() for t in ws]),
                                           saved.data_ptr(), scratch.data_ptr(), core_out.data_ptr(), st), 'encoder_forward')
        dc = dev_dcore.contiguous()
        _lib.check(lib.srl_encoder_backward(E, dc.data_ptr(), B, 1, saved.data_ptr(), scratch.data_ptr(),
                                            (C.c_void_p * 8)(*[t.data_ptr() for t in gs]), st), 'encoder_backward')
        torch.cuda.synchronize()
    finally:
        lib.srl_encoder_destroy(E)
    assert torch.equal(core_out, L.debug_buffer('core').view(B, 514))
    for n, g in zip(APEX_PARAM_NAMES[:8], gs):
        assert torch.equal(g, L.grads[n]), n


# ---------------------------------------------------------------------------------------------------------------- 4
def test_priorities_reach_the_trees():
    B, A, mem = 48, 6, 64
    on, tg = _nets(A)
    batch, w = _batch(B, A, seed=11, device='cuda')
    S = GpuPrioritizedSampler(mem, alpha=0.6)
    S.add(mem)
    idxs = torch.randint(0, mem, (B,), generator=torch.Generator().manual_seed(5))
    idxs[7] = idxs[2]
    idxs[B - 1] = idxs[0]                     # repeated indices: the last occurrence wins
    L = _learner(B, A, on, tg, priority_eps=1e-6)
    L.learn(batch, weights=w, idxs=idxs.cuda(), sampler=S, use_graph=False)
    prio = L.debug_buffer('priorities').cpu().numpy()
    o = PerOracle(mem, 0.6)
    o.add(mem)
    o.update_priorities(idxs.numpy(), prio)
    st, mt, mp = S.trees()
    assert mp == o.max_priority
    cap = S.capacity
    leaves = st[cap:cap + mem].cpu().numpy()
    ref = o.sum_tree.tree[cap:cap + mem]
    assert np.allclose(leaves, ref, rtol=1e-14, atol=0)
    o.set_leaves(np.nonzero(leaves != ref)[0], leaves[leaves != ref])      # adopt the GPU's rounding of p ** alpha
    assert np.array_equal(st.cpu().numpy()[1:], o.sum_tree.tree[1:])
    assert np.array_equal(mt.cpu().numpy()[1:], o.min_tree.tree[1:])


# ---------------------------------------------------------------------------------------------------------------- 5
def _run(A, on, tg, batches, use_graph, mem=64, **kw):
    """5 steps through fixed buffers (the graph replays), each writing its priorities into a sampler of its own"""
    B = batches[0][0][0].shape[0]
    L = _learner(B, A, on, tg, **kw)
    S = GpuPrioritizedSampler(mem, alpha=0.6)
    S.add(mem)
    bufs = tuple(torch.empty_like(t) for t in batches[0][0])
    wb = torch.empty_like(batches[0][1])
    ib = torch.empty(B, dtype=torch.int64, device='cuda')
    for k, (b, w) in enumerate(batches):
        for d, s in zip(bufs, b):
            d.copy_(s)
        wb.copy_(w)
        ib.copy_(torch.randint(0, mem, (B,), generator=torch.Generator().manual_seed(k)))
        L.learn(bufs, weights=wb, idxs=ib, sampler=S, use_graph=use_graph, sync_stats=False)
    torch.cuda.synchronize()
    return L, S


def test_determinism_and_graph_replay():
    B, A = 32, 6
    on, tg = _nets(A, seed=1)
    batches = [_batch(B, A, seed=s, device='cuda') for s in range(5)]
    kw = dict(double_dqn=True, max_grad_norm=10.0, target_update_frequency=2, soft_update_tau=0.5)
    (e1, s1), (e2, s2), (g, sg) = _run(A, on, tg, batches, False, **kw), _run(A, on, tg, batches, False, **kw), _run(A, on, tg, batches, True, **kw)
    assert len(g._graphs) == 1
    for t1, t2, tg_ in zip(s1.trees(), s2.trees(), sg.trees()):     # the captured priority update reaches the trees as the eager one
        assert (t1 == t2 == tg_) if isinstance(t1, float) else (torch.equal(t1, t2) and torch.equal(t1, tg_))
    for n in APEX_PARAM_NAMES:
        assert torch.equal(e1.params[n], e2.params[n]) and torch.equal(e1.params[n], g.params[n]), n
        assert torch.equal(e1.target_params[n], g.target_params[n]), n
    assert torch.equal(e1.exp_avg, g.exp_avg) and torch.equal(e1.exp_avg_sq, g.exp_avg_sq)
    assert int(g.debug_buffer('step')[0]) == int(e1.debug_buffer('step')[0]) == 5     # Adam's t advanced across the replays


# ---------------------------------------------------------------------------------------------------------------- 6
@pytest.mark.parametrize('tau', [1.0, 0.05])
def test_target_update_cadence(tau):
    B, A, freq = 16, 4, 3
    on, tg = _nets(A, seed=2)
    L = _learner(B, A, on, tg, target_update_frequency=freq, soft_update_tau=tau)
    for k in range(7):
        batch, w = _batch(B, A, seed=20 + k, device='cuda')
        before = [t.clone() for t in L.target_params.values()]
        L.learn(batch, weights=w, use_graph=False)
        if k % freq == 0:                    # dqn_agent.py:185-187, counted from 0
            O.soft_target_update(list(L.params.values()), before, tau)
        for n, e in zip(APEX_PARAM_NAMES, before):
            assert torch.equal(L.target_params[n], e), (k, n)
    assert L.target_model_update_step == 3
    if tau == 1.0:
        L.update_target(1.0)
        for n in APEX_PARAM_NAMES:
            assert torch.equal(L.target_params[n], L.params[n])


# ---------------------------------------------------------------------------------------------------------------- 7
def test_checkpoint_roundtrip_and_resume(tmp_path):
    B, A = 16, 6
    on, tg = _nets(A, seed=4)
    batches = [_batch(B, A, seed=40 + s, device='cuda') for s in range(6)]
    kw = dict(target_update_frequency=2, soft_update_tau=0.3)
    full = _learner(B, A, on, tg, **kw)
    half = _learner(B, A, on, tg, **kw)
    for b, w in batches[:3]:
        full.learn(b, weights=w)
        half.learn(b, weights=w)
    path = str(tmp_path / 'apex.pt')
    half.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {'actor_state_dict', 'actor_target_state_dict', 'optimizer_state_dict'}
    net = AtariQNet(A)
    net.load_state_dict(ck['actor_state_dict'])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck['optimizer_state_dict'])
    assert all(float(s['step']) == 3 for s in opt.state.values()) and len(opt.state) == 10
    torch.testing.assert_close(opt.state[opt.param_groups[0]['params'][8]]['exp_avg'], half.exp_avg[half._off[8]:half._off[8] + half._cnt[8]].view(A, 512).cpu(), rtol=0, atol=0)
    resumed = _learner(B, A, on, on, **kw)
    resumed.load_checkpoint(path)
    assert int(resumed.debug_buffer('step')[0]) == 3
    for b, w in batches[3:]:
        full.learn(b, weights=w)
        resumed.learn(b, weights=w)
    torch.cuda.synchronize()
    for n in APEX_PARAM_NAMES:
        assert torch.equal(full.params[n], resumed.params[n]), n
        assert torch.equal(full.target_params[n], resumed.target_params[n]), n
    assert torch.equal(full.exp_avg, resumed.exp_avg) and torch.equal(full.exp_avg_sq, resumed.exp_avg_sq)
    assert (full.learner_update_step, full.target_model_update_step) == (resumed.learner_update_step, resumed.target_model_update_step)


# ---------------------------------------------------------------------------------------------------------------- 8
@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    B, A, n = 16, 18, 37                      # n > B: the forward runs in chunks of B frames
    torch.manual_seed(9)
    net = AtariQNet(A)
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, precision=precision), init_state_dict=net.state_dict())
    obs = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8)
    q = L.q_values(obs)
    ref = net(obs).detach()
    err = rel_l2(q, ref)
    _record(f'q_values_{precision}', err)
    assert err <= tol, err
    assert torch.equal(L.predict(obs), q.argmax(-1))
    batch, w = _batch(B, A, seed=1, device='cuda')       # q_values runs on its own buffers: the step's rows stay as the step left them
    L.learn(batch, weights=w, use_graph=False)
    rows = L.debug_buffer('core_next_target')
    L.q_values(obs)
    assert torch.equal(L.debug_buffer('core_next_target'), rows)
    assert L.get_action(obs[0], eps=0.0).shape == (1,)
    a = L.get_action(obs, eps=1.0)
    assert a.shape == (n,) and int(a.min()) >= 0 and int(a.max()) < A
