"""Shared cases, helpers and checks of the Ape-X tests: the head table, the batches and frames, the error metrics, the results record,
learners, actors and their initial networks, the step and act-learn loops, the encoder-gradient bit check, and the checks every head
shares (check_*), which each head's test module runs over its own grid.

Each row of HEADS describes one Q head the way the tests build and check it: its ApexHParams / B200ApexActor keywords, its initial
networks, its AtariQNet keywords, the fp64 tail of its bf16 step, the metric of each quantity it compares with the fp32 oracle, and the
file its measured errors go to under $SRL_RESULTS_DIR.  A row's head setting (K and the support of C51, N and kappa of QR) is its
default; a test varies it with ``row.but(...)``."""
import ctypes as C
import dataclasses
import math
from typing import Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import apex_oracle as O
from oracle.per_oracle import PerOracle
from scalerl_b200 import _lib
from scalerl_b200.algorithms.apex import ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner, default_q_state_dict
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests import layer_ref as R
from tests.exact import record

F64 = torch.float64


# ---------------------------------------------------------------------------------------------------------------- inputs and metrics
def batch(B, A, seed=0, done_p=0.25, device='cpu'):
    """(obs, action, reward, next_obs, done), weights"""
    g = torch.Generator().manual_seed(seed)
    obs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    act = torch.randint(0, A, (B,), generator=g)
    rew = torch.randn(B, generator=g)
    nobs = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    done = torch.rand(B, generator=g) < done_p
    w = torch.rand(B, generator=g) + 0.1
    return tuple(t.to(device) for t in (obs, act, rew, nobs, done)), w.to(device)


def frames(n, seed, device='cpu'):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).to(device)


def rel_l2(a, b):
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def nmax(a, b):
    """max |a - b| / max |b| (tensors or arrays)"""
    a, b = torch.as_tensor(a).detach().cpu().to(F64), torch.as_tensor(b).detach().cpu().to(F64)
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))


def scaled(a, b, scale):
    """max |a - b| over the largest term size of the sums a and b are"""
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).abs().max() / max(float(scale.abs().max()), 1e-300))


def unbuilt(cls, **attrs):
    """an object with only the given host attributes: the checks before any device work"""
    o = cls.__new__(cls)
    for k, v in attrs.items():
        setattr(o, k, v)
    return o


def mask_flips(L, params, obs, B):
    """test_gpu_precision.py's tie accounting on the forward over s: the learner's ReLU masks (a1, a2, a3 high parts and h, > 0) against
    fp32 pre-activations on the CPU -> (flipped units, units, worst |z| / rms of a flipped unit)"""
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


def device_composed(L, net):
    """the learner's composed weights of `net` ('online' / 'target') as {layer: (W, b)}, the head split as the state dict"""
    W, b = L.debug_buffer(f'head_weight_{net}').view(-1, 512), L.debug_buffer(f'head_bias_{net}')
    out = {'fc': (L.debug_buffer(f'fc_weight_{net}').view(512, 3136), L.debug_buffer(f'fc_bias_{net}'))}
    if L.hp.dueling_dqn:
        out['value'], out['advantage'] = (W[:1], b), (W[1:], L.debug_buffer(f'head_adv_bias_{net}'))
    else:
        out['q'] = (W, b)
    return out


# ---------------------------------------------------------------------------------------------------------------- fp64 tails of the bf16 step
def _core(L, name, B):
    return L.debug_buffer(name).view(B, 514)[:, :512].to(F64)


def _tail_scalar(row, L, pre, tg, batch_, w, gamma, double, B, A):
    """the plain or dueling tail in fp64 on the kernel's core rows and the fp32 head weights -> (pairs, loss, extra errors)"""
    obs, act, rew, nobs, done = batch_
    h, hnt = _core(L, 'core', B), _core(L, 'core_next_target', B)
    a = act.long()
    if row.kind == 'dueling':
        def q64(h_, sd):
            Wv, bv = sd['value.weight'].cuda().to(F64), sd['value.bias'].cuda().to(F64)
            Wa, ba = sd['advantage.weight'].cuda().to(F64), sd['advantage.bias'].cuda().to(F64)
            adv = h_ @ Wa.T + ba
            return (h_ @ Wv.T + bv) + adv - adv.mean(1, keepdim=True)
    else:
        def q64(h_, sd):
            return h_ @ sd['q.weight'].cuda().to(F64).T + sd['q.bias'].cuda().to(F64)
    q = q64(h, pre).gather(1, a[:, None]).squeeze(1)
    qt = q64(hnt, tg)
    astar = (q64(_core(L, 'core_next', B), pre) if double else qt).argmax(1)
    y = rew.to(F64) + gamma * qt.gather(1, astar[:, None]).squeeze(1) * (1 - done.to(F64))
    delta = q - y
    loss = (w.to(F64) * delta ** 2).mean()
    dq = 2 * w.to(F64) * delta / B
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'q': (L.debug_buffer('q'), q), 'y': (L.debug_buffer('y'), y), 'delta': (L.debug_buffer('priorities'), delta.abs())}
    if row.kind == 'dueling':
        coef = dq[:, None] * (torch.nn.functional.one_hot(a, A).to(F64) - 1.0 / A)      # dL/dAdv
        Wv, Wa = pre['value.weight'].to(F64), pre['advantage.weight'].to(F64)
        dcore = dq[:, None] * (Wv + Wa[a] - Wa.mean(0, keepdim=True))
        pairs.update({'value.weight': (L.grads['value.weight'], (dq[:, None] * h).sum(0, keepdim=True)),
                      'value.bias': (L.grads['value.bias'], dq.sum().view(1)),
                      'advantage.weight': (L.grads['advantage.weight'], coef.T @ h), 'advantage.bias': (L.grads['advantage.bias'], coef.sum(0))})
    else:
        Wq = pre['q.weight'].to(F64)
        onehot = torch.nn.functional.one_hot(a, A).to(F64) * dq[:, None]
        dcore = dq[:, None] * Wq[a]
        pairs.update({'q.weight': (L.grads['q.weight'], onehot.T @ h), 'q.bias': (L.grads['q.bias'], onehot.sum(0))})
    pairs['dcore'] = (dev_dcore[:, :512], dcore)
    return pairs, float(loss), {}


def _tail_categorical(row, L, pre, tg, batch_, w, gamma, double, B, A):
    """the C51 tail in fp64: logits, p, m, CE, KL, dlogits, the head gradients and dcore -> (pairs, loss, extra errors)"""
    obs, act, rew, nobs, done = batch_
    K, support = row.width, (row.v_min, row.v_max)
    z32, dz32 = O.support(K, *support)
    z, lo, hi = z32.to(F64).cuda(), float(np.float32(support[0])), float(np.float32(support[1]))

    def tail64(h_, W, b):
        """logits, p, log p [B, A, K] and Q [B, A] in fp64 from core rows h and the fp32 head weights"""
        logits_ = (h_ @ W.T + b).view(-1, A, K)
        logp_ = torch.log_softmax(logits_, dim=2)
        p_ = logp_.exp()
        return logits_, p_, logp_, (p_ * z).sum(2)

    h = _core(L, 'core', B)
    Wo, bo = pre['q.weight'].cuda().to(F64), pre['q.bias'].cuda().to(F64)
    logits, p, logp, _ = tail64(h, Wo, bo)
    _, pt, _, qt = tail64(_core(L, 'core_next_target', B), tg['q.weight'].cuda().to(F64), tg['q.bias'].cuda().to(F64))
    astar = (tail64(_core(L, 'core_next', B), Wo, bo)[3] if double else qt).argmax(1)
    rows, a = torch.arange(B, device='cuda'), act.long()
    g = float(np.float32(gamma)) * (1 - done.to(F64))
    tz = (rew.to(F64)[:, None] + g[:, None] * z[None]).clamp(lo, hi)
    bj = (tz - lo) / float(dz32)
    lower, upper = bj.floor().long().clamp(0, K - 1), bj.ceil().long().clamp(0, K - 1)
    pj = pt[rows, astar]
    m = torch.zeros(B, K, dtype=F64, device='cuda')
    eq = lower == upper
    m.scatter_add_(1, lower, torch.where(eq, pj, pj * (upper.to(F64) - bj)))
    m.scatter_add_(1, upper, torch.where(eq, torch.zeros_like(pj), pj * (bj - lower.to(F64))))
    lp = logp[rows, a]
    ce = -(m * lp).sum(1)
    kl = (torch.xlogy(m, m) - m * lp).sum(1)
    dl = torch.zeros(B, A, K, dtype=F64, device='cuda')
    dl[rows, a] = (w.to(F64) / B)[:, None] * (p[rows, a] * m.sum(1, keepdim=True) - m)
    dl = dl.view(B, A * K)
    hb = torch.cat([h, torch.ones(B, 1, dtype=F64, device='cuda')], 1)
    gWb = dl.T @ hb
    dcore = dl @ Wo
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'logits': (L.debug_buffer('logits').view(B, A, K), logits), 'm': (L.debug_buffer('m').view(B, K), m),
             'ce': (L.debug_buffer('ce'), ce), 'kl': (L.debug_buffer('priorities'), kl.clamp(min=0)),
             'dlogits': (L.debug_buffer('dlogits').view(B, A * K), dl), 'q.weight': (L.grads['q.weight'], gWb[:, :512]),
             'q.bias': (L.grads['q.bias'], gWb[:, 512]), 'dcore': (dev_dcore[:, :512], dcore),
             'q': (L.debug_buffer('q'), (p[rows, a] * z).sum(1)), 'y': (L.debug_buffer('y'), (m * z).sum(1))}
    # p: the softmax of the kernel's own logits against that of the fp64 logits
    pk = torch.softmax(L.debug_buffer('logits').view(B, A, K).to(F64), dim=2)
    return pairs, float((w.to(F64) * ce).mean()), {'p': (rel_l2(pk, p), nmax(pk, p))}


def _tail_quantile(row, L, pre, tg, batch_, w, gamma, double, B, A):
    """the QR tail in fp64: theta, the target quantiles, the loss, dtheta, the head gradients and dcore -> (pairs, loss, extra errors)"""
    obs, act, rew, nobs, done = batch_
    N, kappa = row.width, row.kappa
    h = _core(L, 'core', B)
    Wo, bo = pre['q.weight'].cuda().to(F64), pre['q.bias'].cuda().to(F64)
    theta = (h @ Wo.T + bo).view(B, A, N)
    tn = (_core(L, 'core_next_target', B) @ tg['q.weight'].cuda().to(F64).T + tg['q.bias'].cuda().to(F64)).view(B, A, N)
    tno = (_core(L, 'core_next', B) @ Wo.T + bo).view(B, A, N) if double else None
    T = O.targets(tn, rew.to(F64), done, float(np.float32(gamma)), tno)
    rows, a = torch.arange(B, device='cuda'), act.long()
    ta = theta[rows, a]
    loss_n = O.quantile_loss(ta, T, kappa)
    dl = torch.zeros(B, A, N, dtype=F64, device='cuda')
    dl[rows, a] = O.dtheta_written(ta, T, kappa, w.to(F64))
    dl = dl.view(B, A * N)
    hb = torch.cat([h, torch.ones(B, 1, dtype=F64, device='cuda')], 1)
    gWb = dl.T @ hb
    dcore = dl @ Wo
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'theta': (L.debug_buffer('theta').view(B, A, N), theta), 'target_quantiles': (L.debug_buffer('target_quantiles').view(B, N), T),
             'qr_loss': (L.debug_buffer('qr_loss'), loss_n), 'priorities': (L.debug_buffer('priorities'), loss_n),
             'dtheta': (L.debug_buffer('dtheta').view(B, A * N), dl), 'q.weight': (L.grads['q.weight'], gWb[:, :512]),
             'q.bias': (L.grads['q.bias'], gWb[:, 512]), 'dcore': (dev_dcore[:, :512], dcore),
             'q': (L.debug_buffer('q'), ta.sum(1) / N), 'y': (L.debug_buffer('y'), T.sum(1) / N)}
    return pairs, float((w.to(F64) * loss_n).mean()), {}


# ---------------------------------------------------------------------------------------------------------------- the head table
# the split test's quantities: (name, learner debug buffer, oracle key, oracle key of the term size or None for normalised max)
_SCALAR = (('q', 'q', 'q', None), ('y', 'y', 'y', None), ('priorities', 'priorities', 'priorities', None))
_NOISY_SCALAR = (('q', 'q', 'q', 'q_scale'), ('y', 'y', 'y', None), ('priorities', 'priorities', 'priorities', None))
_NOISY_C51 = (('q', 'q', 'q', 'q_scale'), ('y', 'y', 'y', 'y_scale'), ('priorities', 'priorities', 'priorities', 'kl_scale'))
_C51 = (('q', 'q', 'q', 'q_scale'), ('m', 'm', 'm', None), ('ce', 'ce', 'ce', None), ('priorities', 'priorities', 'priorities', 'kl_scale'))
_QR = (('q', 'q', 'q', 'q_scale'), ('y', 'y', 'y', 'y_scale'), ('target_quantiles', 'target_quantiles', 'T', None),
       ('qr_loss', 'qr_loss', 'loss_n', None), ('priorities', 'priorities', 'priorities', None))


def _tie_scalar(sd, A, W):
    """actions 1 and 4 share their head row and the largest bias (dueling: of Adv, so of Q)"""
    layer = 'advantage' if 'advantage.weight' in sd else 'q'
    sd[f'{layer}.weight'][4] = sd[f'{layer}.weight'][1]
    sd[f'{layer}.bias'][1] = sd[f'{layer}.bias'][4] = 30.0


def _tie_categorical(sd, A, K):
    """actions 1 and 4 share their logit rows, and their top atom dominates"""
    sd['q.weight'][4 * K:5 * K] = sd['q.weight'][K:2 * K]
    sd['q.bias'][4 * K:5 * K] = sd['q.bias'][K:2 * K]
    sd['q.bias'][2 * K - 1] += 30.0
    sd['q.bias'][5 * K - 1] += 30.0


def _tie_quantile(sd, A, N):
    """actions 1 and 4 share their quantile rows, which dominate"""
    sd['q.weight'][4 * N:5 * N] = sd['q.weight'][N:2 * N]
    sd['q.bias'][N:2 * N] += 30.0
    sd['q.bias'][4 * N:5 * N] = sd['q.bias'][N:2 * N]


@dataclasses.dataclass(frozen=True)
class Head:
    """one row of the head table"""
    name: str
    kind: str                           # 'plain', 'dueling', 'categorical' or 'quantile'
    results: str                        # the file under $SRL_RESULTS_DIR
    noisy: bool = False
    width: int = 0                      # K atoms (categorical) or N quantiles (quantile)
    v_min: float = -10.0
    v_max: float = 10.0
    kappa: float = 1.0
    split_metrics: tuple = _SCALAR
    tail: object = None                 # the fp64 tail of the bf16 step
    actor_rows: Optional[str] = None    # the actor's debug buffer of head rows the learner's step also writes
    tie: object = _tie_scalar
    refusal: Optional[str] = None       # what a plain actor's sync_from names when it refuses this learner
    fp32_prio_reward: float = 1.0       # the reward scale of the fp32 actor-priority test
    bf16_prio_reward: float = 1.0       # and of the bf16 one
    trains: str = 'q.weight'            # a tensor a few steps must change
    adam_probe: str = 'q.weight'        # the tensor whose Adam state the checkpoint test compares with torch's

    def __str__(self):
        return self.name

    def but(self, **kw):
        return dataclasses.replace(self, **kw)

    @property
    def hp(self):
        """the ApexHParams / B200ApexActor keywords of the head"""
        kw = {'plain': {}, 'dueling': dict(dueling_dqn=True),
              'categorical': dict(categorical_dqn=True, num_atoms=self.width, v_min=self.v_min, v_max=self.v_max),
              'quantile': dict(quantile_dqn=True, num_quantiles=self.width, quantile_kappa=self.kappa)}[self.kind]
        return dict(kw, noisy_dqn=True) if self.noisy else kw

    @property
    def net_kw(self):
        """the AtariQNet keywords of the head"""
        kw = {'plain': {}, 'dueling': dict(dueling=True),
              'categorical': dict(categorical=True, num_atoms=self.width, v_min=self.v_min, v_max=self.v_max),
              'quantile': dict(quantile=True, num_quantiles=self.width)}[self.kind]
        return dict(kw, noisy=True) if self.noisy else kw

    @property
    def oracle(self):
        return O.Head(self.kind, self.noisy, num_atoms=self.width, v_min=self.v_min, v_max=self.v_max, num_quantiles=self.width,
                      kappa=self.kappa)

    def scale_reward(self, rew):
        """the split and bf16-tail tests' rewards: on the scale of the support for C51 (rew * (v_max - v_min) / 20, in that order), as
        drawn for the other heads"""
        return rew * (self.v_max - self.v_min) / 20 if self.kind == 'categorical' and not self.noisy else rew

    def tag(self, B, A):
        """the results key of a (B, A) case"""
        if self.noisy:
            return f'{self.kind}_B{B}_A{A}'
        return {'categorical': f'B{B}_A{A}_K{self.width}', 'quantile': f'B{B}_A{A}_N{self.width}'}.get(self.kind, f'B{B}_A{A}')

    @property
    def suffix(self):
        """the results key's head setting"""
        if self.noisy:
            return ''
        return {'categorical': f'_support{(self.v_min, self.v_max)}', 'quantile': f'_kappa{self.kappa}'}.get(self.kind, '')

    def state_dict(self, A, seed, noisy_std=0.5):
        """default_q_state_dict's initial network of seed"""
        return default_q_state_dict(A, seed, self.kind == 'dueling', self.width if self.kind == 'categorical' else 0, self.noisy,
                                    noisy_std, self.width if self.kind == 'quantile' else 0)


HEADS = {h.name: h for h in (
    Head('plain', 'plain', 'apex.json', tail=_tail_scalar),
    Head('dueling', 'dueling', 'apex_dueling.json', tail=_tail_scalar, refusal='dueling_dqn', trains='advantage.weight',
         adam_probe='advantage.weight'),
    Head('categorical', 'categorical', 'apex_categorical.json', width=51, split_metrics=_C51, tail=_tail_categorical, actor_rows='logits',
         tie=_tie_categorical, refusal='categorical_dqn', fp32_prio_reward=10.0, bf16_prio_reward=3.0),
    Head('quantile', 'quantile', 'apex_quantile.json', width=200, split_metrics=_QR, tail=_tail_quantile, actor_rows='theta',
         tie=_tie_quantile, refusal='quantile_dqn', bf16_prio_reward=3.0),
    Head('noisy_plain', 'plain', 'apex_noisy.json', noisy=True, split_metrics=_NOISY_SCALAR, trains='fc.weight_sigma',
         adam_probe='fc.weight_sigma'),
    Head('noisy_dueling', 'dueling', 'apex_noisy.json', noisy=True, split_metrics=_NOISY_SCALAR, trains='fc.weight_sigma',
         adam_probe='fc.weight_sigma'),
    Head('noisy_categorical', 'categorical', 'apex_noisy.json', noisy=True, width=11, split_metrics=_NOISY_C51, trains='fc.weight_sigma',
         adam_probe='fc.weight_sigma'),
)}


# ---------------------------------------------------------------------------------------------------------------- learners, actors, loops
def nets(head, A, seed=0, noisy_std=0.5):
    """(online, target) initial networks of a head: default_q_state_dict's of seeds 2 seed and 2 seed + 1, or (the plain head) AtariQNet's
    two in turn after torch.manual_seed(seed)"""
    if head.kind == 'plain' and not head.noisy:
        torch.manual_seed(seed)
        on, tg = AtariQNet(A), AtariQNet(A)
        return ({k: v.detach().clone() for k, v in on.state_dict().items()}, {k: v.detach().clone() for k, v in tg.state_dict().items()})
    return head.state_dict(A, 2 * seed, noisy_std), head.state_dict(A, 2 * seed + 1, noisy_std)


def learner(head, B, A, on, tg, **kw):
    """a learner of the head on (online, target); kw: ApexHParams fields and the noise seed"""
    seed = kw.pop('seed', 0)
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, **head.hp, **kw), init_state_dict=on, seed=seed)
    L.load_state_dict(tg, target=True)
    return L


def actor(head, E, A, **kw):
    return B200ApexActor(E, A, **head.hp, **kw)


def run_steps(head, A, on, tg, batches, use_graph, mem=64, **kw):
    """one learner's steps through fixed buffers (the graph replays), each writing its priorities into a sampler of its own"""
    B = batches[0][0][0].shape[0]
    L = learner(head, B, A, on, tg, **kw)
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


def act_learn_loop(head, seed, steps=60):
    """steps of act -> prioritized add of random transitions -> captured learn_from, the actor synced every 10 updates"""
    E, A, n = 16, 4, 3
    L = B200ApexLearner(ApexHParams(batch_size=32, num_actions=A, gamma=0.99 ** n, target_update_frequency=20, **head.hp), seed=seed)
    X = actor(head, E, A, seed=seed)
    X.sync_from(L)
    mem = GpuPrioritizedReplayBuffer(1024, E, n_step=n, gamma=0.99)
    torch.manual_seed(seed)
    g = torch.Generator().manual_seed(seed)
    losses = []
    for t in range(steps):
        obs, nobs = frames(E, 1000 * seed + 2 * t, 'cuda'), frames(E, 1000 * seed + 2 * t + 1, 'cuda')
        action = X.act(obs)
        reward, done = torch.randn(E, generator=g).cuda(), (torch.rand(E, generator=g) < 0.05).cuda()
        mem.save_to_memory(obs, action, reward, nobs, done, is_vectorised=True, priorities_from=X)
        if len(mem) >= 64:
            losses.append(L.learn_from(mem)['loss'])
            if len(losses) % 10 == 0:
                X.sync_from(L)
    return L, mem, losses


def assert_encoder_grads_are_srl_encoder_backward(L, pre, batch_):
    """the encoder gradients of L's step are srl_encoder_backward called directly on the tail's dcore, bit for bit (pre: the weights
    the step ran on, batch_: its batch on the device)"""
    obs, act, rew = batch_[:3]
    B = obs.shape[0]
    names = list(L.names)[:8]
    lib = _lib.lib()
    E = C.c_void_p()
    _lib.check(lib.srl_encoder_create(0, C.byref(E)), 'encoder_create')
    try:
        sb, kb = C.c_int64(), C.c_int64()
        _lib.check(lib.srl_encoder_sizes(B, 0, C.byref(sb), C.byref(kb)), 'encoder_sizes')
        saved = torch.empty(sb.value, dtype=torch.uint8, device='cuda')
        scratch = torch.empty(kb.value, dtype=torch.uint8, device='cuda')
        ws = [pre[n].cuda().contiguous() for n in names]
        gs = [torch.empty_like(t) for t in ws]
        core_out = torch.empty(B, 514, device='cuda')
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.srl_encoder_forward(E, obs.data_ptr(), rew.data_ptr(), act.data_ptr(), B, 1, (C.c_void_p * 8)(*[t.data_ptr() for t in ws]),
                                           saved.data_ptr(), scratch.data_ptr(), core_out.data_ptr(), st), 'encoder_forward')
        dc = L.debug_buffer('dcore').view(B, 514).contiguous()
        _lib.check(lib.srl_encoder_backward(E, dc.data_ptr(), B, 1, saved.data_ptr(), scratch.data_ptr(),
                                            (C.c_void_p * 8)(*[t.data_ptr() for t in gs]), st), 'encoder_backward')
        torch.cuda.synchronize()
    finally:
        lib.srl_encoder_destroy(E)
    assert torch.equal(core_out, L.debug_buffer('core').view(B, 514))
    for n, g in zip(names, gs):
        assert torch.equal(g, L.grads[n]), n


# ---------------------------------------------------------------------------------------------------------------- the checks every head shares
# each test module runs them over its own head and grid; the measured errors go to the head's results file
def check_split_against_oracle(head, B, A, double, clip):
    """fp32-accurate split operands against the fp32 CPU oracle (a noisy head's fed the device's noise): the head's quantities to 1e-5,
    every gradient to rel-L2 1e-4 (2e-2 when only genuine ReLU ties flipped), the weights after the step against the oracle's Adam to 2e-6"""
    on, tg = nets(head, A, seed=B)
    (obs, act, rew, nobs, done), w = batch(B, A, seed=B + A)
    rew = head.scale_reward(rew)
    L = learner(head, B, A, on, tg, seed=B if head.noisy else 0, precision='fp32_split', double_dqn=double, max_grad_norm=clip,
                priority_eps=0.0)
    L.learn(tuple(t.cuda() for t in (obs, act, rew, nobs, done)), weights=w.cuda(), use_graph=False)
    noise = dict(noise_online=L.debug_buffer('noise_online').cpu(), noise_target=L.debug_buffer('noise_target').cpu()) if head.noisy else {}
    ref = O.learn_step(on, tg, obs, act, rew, nobs, done, weights=w, gamma=0.99, double_dqn=double, max_grad_norm=clip, head=head.oracle,
                       **noise)
    names = list(L.names)
    assert list(ref['grads']) == names
    err = {}
    for k, buf, rk, sk in head.split_metrics:
        dev = L.debug_buffer(buf).view(ref[rk].shape)
        err[k] = scaled(dev, ref[rk], ref[sk]) if sk else nmax(dev, ref[rk])
    loss = float(L.debug_buffer('loss')[0])
    err['loss'] = abs(loss - ref['loss']) / max(abs(ref['loss']), 1e-30)
    mask_params = on
    if head.noisy:
        comp = device_composed(L, 'online')
        mask_params = dict(on, **{'fc.weight': comp['fc'][0].cpu(), 'fc.bias': comp['fc'][1].cpu()})
    flips, units, worst = mask_flips(L, mask_params, obs, B)
    gerr = {n: rel_l2(L.grads[n], ref['grads'][n]) for n in names}
    post = O.adam_on_grads(on, {n: L.grads[n] for n in names}, max_grad_norm=clip)
    perr = max(float((L.params[n].cpu() - post[n]).abs().max()) for n in names)
    record(head.results, f'split_{head.tag(B, A)}_double{int(double)}_clip{clip}{head.suffix}',
           dict(err, grads=gerr, relu_mask_flips=flips, relu_units=units, worst_flipped_margin=worst, post_step_max_abs=perr))
    for k, v in err.items():
        assert v <= 1e-5, (k, v)
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)       # only genuine ties may flip
    gtol = 1e-4 if flips == 0 else 2e-2
    for n, v in gerr.items():
        assert v <= gtol, (n, v, flips)
    assert perr <= 2e-6, perr


def check_bf16_tail_and_encoder_backward(head, B, A, double):
    """bf16: the head's tail against fp64 on its own operands (core rows, fp32 head weights); the encoder gradients equal
    srl_encoder_backward on the tail's dcore, bit for bit"""
    on, tg = nets(head, A, seed=7)
    (obs, act, rew, nobs, done), w = batch(B, A, seed=3, device='cuda')
    rew = head.scale_reward(rew)
    step_batch = (obs, act, rew, nobs, done)
    gamma = 0.97
    L = learner(head, B, A, on, tg, double_dqn=double, gamma=gamma, priority_eps=0.0)
    pre = L.state_dict()
    L.learn(step_batch, weights=w, use_graph=False)
    pairs, want_loss, extra = head.tail(head, L, pre, tg, step_batch, w, gamma, double, B, A)
    err = {k: (rel_l2(u, v), nmax(u, v)) for k, (u, v) in pairs.items()}
    err['loss'] = (abs(float(L.debug_buffer('loss')[0]) - want_loss) / want_loss,) * 2
    err.update(extra)
    record(head.results, f'bf16_tail_{head.tag(B, A)}_double{int(double)}{head.suffix}', err)
    for k, (r, m) in err.items():
        assert r <= 2e-5 and m <= 1e-4, (k, r, m)
    assert not bool(L.debug_buffer('dcore').view(B, 514)[:, 512:].any())
    assert_encoder_grads_are_srl_encoder_backward(L, pre, step_batch)


def check_actor_q_values_and_greedy_act(head, E):
    """after sync_from the actor's Q values (and head rows) are the learner's bit for bit, and act with every epsilon 0 is their first
    argmax, ties included"""
    A = 6
    L = B200ApexLearner(ApexHParams(batch_size=E if head.actor_rows else 32, num_actions=A, **head.hp), seed=3)
    X = actor(head, E, A, epsilons=np.zeros(E), seed=1)
    X.sync_from(L)
    assert X.weights_version == 1
    obs = frames(E, E, 'cuda')
    q = X.q_values(obs)
    assert torch.equal(q, L.q_values(obs))
    assert torch.equal(X.act(obs), torch.argmax(q, dim=1))
    if head.actor_rows:
        # the head rows (logits or quantiles) of the learner's step over s are the actor's over the same frames
        step_batch, _ = batch(E, A, seed=E, device='cuda')
        L.learn((obs,) + step_batch[1:], use_graph=False)
        X.act(obs)
        assert torch.equal(X.debug_buffer(head.actor_rows)[:E * A * head.width], L.debug_buffer(head.actor_rows))
        X.sync_from(L)
    # ties of Q: actions 1 and 4 get the same Q, larger than the others'; the first index wins, as in torch.argmax
    sd = L.state_dict()
    head.tie(sd, A, head.width)
    X.load_state_dict(sd)
    L.load_state_dict(sd)
    q = X.q_values(obs)
    assert torch.equal(q[:, 1], q[:, 4]) and bool((torch.argmax(q, dim=1) == 1).all())
    assert bool((X.act(obs) == 1).all())
    assert torch.equal(q, L.q_values(obs))


def check_fp32_actor_priorities(head):
    """fp32-accurate actor priorities against the oracle's initial_priorities, the trees against PerOracle"""
    E, A, gamma, M = 300, 6, 0.99, 1024
    sd = head.state_dict(A, 4)
    X = actor(head, E, A, precision='fp32_split', priority_eps=1e-6, init_state_dict=sd)
    mem = GpuPrioritizedReplayBuffer(M, E, alpha=1.0, n_step=1, gamma=gamma)       # n = 1, alpha = 1: leaf e is transition e's priority
    g = torch.Generator().manual_seed(8)
    s, ns = frames(E, 1, 'cuda'), frames(E, 2, 'cuda')
    a, r, d = torch.randint(0, A, (E,), generator=g), head.fp32_prio_reward * torch.randn(E, generator=g), torch.rand(E, generator=g) < 0.3
    mem.save_to_memory(s, a.cuda(), r.cuda(), ns, d.cuda(), is_vectorised=True, priorities_from=X)
    sum_t, min_t, mp = mem.sampler.trees()
    cap = mem.sampler.capacity
    leaves = sum_t[cap:cap + E]
    want = O.initial_priorities(sd, s.cpu(), a, r, ns.cpu(), d, float(np.float32(gamma)), 1e-6, head=head.oracle)
    err = nmax(leaves, want)
    record(head.results, 'fp32_split_actor_priorities', {'nmax': err})
    assert err <= 1e-5, err
    po = PerOracle(M, 1.0)
    po.update_priorities(list(range(E)), leaves.cpu().numpy())
    po.tree_ptr, po.size = E % M, E
    assert np.array_equal(sum_t.cpu().numpy(), po.sum_tree.tree) and np.array_equal(min_t.cpu().numpy(), po.min_tree.tree)
    assert mp == po.max_priority


def check_bf16_actor_priorities(head):
    """bf16 actor priorities are the learner's on the same weights, bit for bit"""
    E, A, n, gamma = 32, 6, 3, 0.99
    L = B200ApexLearner(ApexHParams(batch_size=E, num_actions=A, gamma=gamma ** n, double_dqn=False, priority_eps=1e-6, **head.hp), seed=2)
    X = actor(head, E, A, priority_eps=1e-6)
    X.sync_from(L)
    mem = GpuPrioritizedReplayBuffer(256, E, alpha=1.0, n_step=n, gamma=gamma)     # alpha = 1: the leaves are the priorities
    # the learner also writes its priorities into trees of its own through the same leaf update, so equal leaves mean equal priorities
    S = GpuPrioritizedSampler(256, alpha=1.0)
    S.add(256)
    g = torch.Generator().manual_seed(6)
    compared = 0
    for t in range(5):
        args = (torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(), torch.randint(0, A, (E,), generator=g).cuda(),
                (head.bf16_prio_reward * torch.randn(E, generator=g)).cuda(),
                torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(), (torch.rand(E, generator=g) < 0.3).cuda())
        ptr = (t - n + 1) * E % 256
        mem.save_to_memory(*args, is_vectorised=True, priorities_from=X)
        if t + 1 < n:
            continue
        idxs = (torch.arange(E) + ptr) % 256
        cap = mem.sampler.capacity
        leaves = mem.sampler.trees()[0][cap + idxs.cuda()]
        L.learn(mem.gather(idxs), idxs=idxs.cuda(), sampler=S, use_graph=False)
        assert torch.equal(S.trees()[0][S.capacity + idxs.cuda()], leaves), t
        if head.kind == 'plain':        # and the plain head's leaves equal its learner's fp32 priorities themselves (not so for the others)
            assert torch.equal(L.debug_buffer('priorities'), leaves), t
        X.sync_from(L)                  # the next add's weights are the learner's after this step (target == online until refreshed)
        L.update_target(1.0)
        compared += 1
    assert compared == 3


def check_determinism_and_graph_replay(head):
    """eager twice and captured: the same parameters, optimizer state, trees (and noise) bit for bit, the device step count advancing"""
    B, A = 32, 6
    on, tg = nets(head, A, seed=1)
    batches = [batch(B, A, seed=s, device='cuda') for s in range(5)]
    kw = dict(double_dqn=True, max_grad_norm=10.0, target_update_frequency=2, soft_update_tau=0.5, **(dict(seed=3) if head.noisy else {}))
    (e1, s1), (e2, s2), (g, sg) = (run_steps(head, A, on, tg, batches, False, **kw), run_steps(head, A, on, tg, batches, False, **kw),
                                   run_steps(head, A, on, tg, batches, True, **kw))
    assert len(g._graphs) == 1
    for t1, t2, tg_ in zip(s1.trees(), s2.trees(), sg.trees()):     # the captured priority update reaches the trees as the eager one
        assert (t1 == t2 == tg_) if isinstance(t1, float) else (torch.equal(t1, t2) and torch.equal(t1, tg_))
    for L in (e2, g):
        for n in e1.names:
            assert torch.equal(e1.params[n], L.params[n]) and torch.equal(e1.target_params[n], L.target_params[n]), n
        assert torch.equal(e1.flat_params, L.flat_params) and torch.equal(e1.flat_target, L.flat_target)
        assert torch.equal(e1.exp_avg, L.exp_avg) and torch.equal(e1.exp_avg_sq, L.exp_avg_sq)
        if head.noisy:
            assert torch.equal(e1.debug_buffer('noise_online'), L.debug_buffer('noise_online'))
    assert not torch.equal(e1.params[head.trains], on[head.trains].cuda())      # the head trains
    assert int(g.debug_buffer('step')[0]) == int(e1.debug_buffer('step')[0]) == 5     # Adam's t advanced across the replays
    if head.noisy:                                                                     # another noise seed gives another run
        o, _ = run_steps(head, A, on, tg, batches, False, **dict(kw, seed=4))
        assert not torch.equal(o.flat_params, e1.flat_params)


def check_captured_learn_from_loop(head):
    """two seeded act -> prioritized add -> captured learn_from loops are bit-identical"""
    L1, m1, l1 = act_learn_loop(head, 5)
    L2, m2, l2 = act_learn_loop(head, 5)
    assert len(l1) > 50 and len(L1._graphs) == 1 and all(math.isfinite(x) for x in l1)
    assert l1 == l2 and torch.equal(L1.flat_params, L2.flat_params)
    assert torch.equal(m1.sampler.trees()[0], m2.sampler.trees()[0])
    assert m1.sampler._L.srl_per_invalid_updates(m1.sampler._h, m1.sampler._stream()) == 0


def check_checkpoint_roundtrip_and_resume(head, tmp_path):
    """checkpoints load into AtariQNet and torch.optim.Adam, and a resumed run equals an uninterrupted one"""
    B, A = 16, 6
    on, tg = nets(head, A, seed=4)
    batches = [batch(B, A, seed=40 + s, device='cuda') for s in range(6)]
    kw = dict(target_update_frequency=2, soft_update_tau=0.3, **(dict(seed=7) if head.noisy else {}))
    full = learner(head, B, A, on, tg, **kw)
    half = learner(head, B, A, on, tg, **kw)
    for b, w in batches[:3]:
        full.learn(b, weights=w)
        half.learn(b, weights=w)
    path = str(tmp_path / head.results.replace('.json', '.pt'))
    half.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {'actor_state_dict', 'actor_target_state_dict', 'optimizer_state_dict'}
    assert tuple(ck['actor_state_dict']) == tuple(half.names)
    net = AtariQNet(A, **head.net_kw)
    net.load_state_dict(ck['actor_state_dict'])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck['optimizer_state_dict'])
    assert all(float(s['step']) == 3 for s in opt.state.values()) and len(opt.state) == len(half.names)
    i = half.names.index(head.adam_probe)
    torch.testing.assert_close(opt.state[opt.param_groups[0]['params'][i]]['exp_avg'],
                               half.exp_avg[half._off[i]:half._off[i] + half._cnt[i]].view(ck['actor_state_dict'][head.adam_probe].shape).cpu(),
                               rtol=0, atol=0)
    resumed = learner(head, B, A, on, on, **kw)
    resumed.load_checkpoint(path)
    assert int(resumed.debug_buffer('step')[0]) == 3
    for b, w in batches[3:]:
        full.learn(b, weights=w)
        resumed.learn(b, weights=w)
    torch.cuda.synchronize()
    if head.noisy:
        assert torch.equal(full.debug_buffer('noise_online'), resumed.debug_buffer('noise_online'))      # the noise continues
    for n in full.names:
        assert torch.equal(full.params[n], resumed.params[n]), n
        assert torch.equal(full.target_params[n], resumed.target_params[n]), n
    assert torch.equal(full.flat_params, resumed.flat_params) and torch.equal(full.flat_target, resumed.flat_target)
    assert torch.equal(full.exp_avg, resumed.exp_avg) and torch.equal(full.exp_avg_sq, resumed.exp_avg_sq)
    assert (full.learner_update_step, full.target_model_update_step) == (resumed.learner_update_step, resumed.target_model_update_step)


def check_q_values_against_cpu_network(head, precision, tol):
    """q_values / predict / get_action against AtariQNet on the CPU; q_values leaves the step's rows alone; a plain actor refuses the head"""
    B, A, n = 16, 18, 37                      # n > B: the forward runs in chunks of B frames
    torch.manual_seed(9)
    net = AtariQNet(A, **head.net_kw)
    if head.kind == 'quantile':
        with torch.no_grad():
            net.q.bias.add_(5.0)               # Q away from 0: a relative error is meaningful (C51: the (0, 200) support puts Q near 100)
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, precision=precision, **head.hp), init_state_dict=net.state_dict())
    obs = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8)
    q = L.q_values(obs)
    ref = net(obs).detach()
    err = rel_l2(q, ref)
    record(head.results, f'q_values_{precision}', err)
    assert err <= tol, err
    assert torch.equal(L.predict(obs), q.argmax(-1))
    step_batch, w = batch(B, A, seed=1, device='cuda')       # q_values runs on its own buffers: the step's rows stay as the step left them
    L.learn(step_batch, weights=w, use_graph=False)
    rows = L.debug_buffer('core_next_target')
    L.q_values(obs)
    assert torch.equal(L.debug_buffer('core_next_target'), rows)
    assert L.get_action(obs[0], eps=0.0).shape == (1,)
    a = L.get_action(obs, eps=1.0)
    assert a.shape == (n,) and int(a.min()) >= 0 and int(a.max()) < A
    if head.refusal:
        with pytest.raises(ValueError, match=head.refusal):
            B200ApexActor(4, A).sync_from(L)
