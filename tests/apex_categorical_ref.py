"""fp32 CPU oracle of the Ape-X learner step and the actor's initial priorities with the categorical (C51) Q network, for the
categorical tests.  Independent of scalerl_b200.

The reference declares ``categorical_dqn``, ``v_min``, ``v_max`` and ``num_atoms`` (DQNArguments) but builds no categorical network,
so the head restates Bellemare et al. 2017 ("A Distributional Perspective on Reinforcement Learning") on the reference's own AtariNet
layers (oracle/_ref, as oracle/apex_oracle.py's RefQNet), with q = nn.Linear(512, A K), row a K + k atom k of action a:

    p(s)[a] = softmax(logits[a K .. a K + K - 1]),  Q(s, a) = sum_k z_k p_k,  z_k = v_min + k dz,  dz = fp32((v_max - v_min) / (K - 1))

The target action is argmax_a Q_target(s') (double DQN: argmax_a Q_online(s')); the target distribution p_target(s')[a*] is projected
onto the support by Algorithm 1 (``project``; ``project_fp64_loop`` is a second, independent witness in fp64); the loss is
mean_n(w_n CE_n), CE_n = -sum_k m_k log p(s_n)[a_n, k]; the priority is max(KL(m || p(s_n)[a_n]), 0) + eps (Hessel et al. 2018).
Around it, the statements are those of oracle/apex_oracle.py (learn_step, adam_on_grads) and tests/apex_actor_ref.py
(initial_priorities): the reference's Ape-X learner update and DQNAgent's double DQN, clipping and Adam
(scalerl/algorithms/apex/worker.py:134-161, dqn/dqn_agent.py:155-182), and Actor.compute_prior (apex/worker.py:59-79)."""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet

NAMES = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'fc.weight', 'fc.bias',
         'q.weight', 'q.bias')


def support(K, v_min, v_max):
    """(z [K] fp32, dz fp32 scalar tensor): the bounds rounded to fp32, dz = (v_max - v_min) / (K - 1) rounded once, z_k = v_min + k dz"""
    lo, hi = float(np.float32(v_min)), float(np.float32(v_max))
    dz = torch.tensor((hi - lo) / (K - 1), dtype=torch.float32)
    return torch.tensor(lo, dtype=torch.float32) + torch.arange(K, dtype=torch.float32) * dz, dz


class CatRefQNet(nn.Module):
    """the reference AtariNet's conv1, conv2, conv3 and fc, then q = nn.Linear(512, A K) on the fc output"""

    def __init__(self, num_actions, num_atoms, state_dict=None):
        super().__init__()
        net = AtariNet((4, 84, 84), num_actions)
        self.A, self.K = num_actions, num_atoms
        self.conv1, self.conv2, self.conv3, self.fc = net.conv1, net.conv2, net.conv3, net.fc
        self.q = nn.Linear(512, num_actions * num_atoms)
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})

    def features(self, obs):        # atari_model.py:93-101
        x = obs.float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        x = x.view(x.shape[0], -1)
        return F.relu(self.fc(x))

    def logits(self, obs):
        return self.q(self.features(obs)).view(-1, self.A, self.K)


def dims(sd, num_atoms):
    return sd['q.bias'].numel() // num_atoms, num_atoms


def project(p, reward, done, gamma, z, dz, v_min, v_max):
    """Algorithm 1 in fp32 torch: p [N, K] the target distribution, reward / done [N] -> m [N, K], accumulated over j in order"""
    N, K = p.shape
    lo, hi = torch.tensor(float(np.float32(v_min))), torch.tensor(float(np.float32(v_max)))
    g = torch.tensor(np.float32(gamma)) * (1 - done.float())
    tz = torch.minimum(torch.maximum(reward.float()[:, None] + g[:, None] * z[None], lo), hi)
    b = (tz - lo) / dz
    lower, upper = b.floor().long().clamp(0, K - 1), b.ceil().long().clamp(0, K - 1)
    m = torch.zeros(N, K)
    for j in range(K):
        pj, l, u, bj = p[:, j], lower[:, j], upper[:, j], b[:, j]
        eq = l == u
        m.scatter_add_(1, l[:, None], torch.where(eq, pj, pj * (u.float() - bj))[:, None])
        m.scatter_add_(1, u[:, None], torch.where(eq, torch.zeros_like(pj), pj * (bj - l.float()))[:, None])
    return m


def project_fp64_loop(p, reward, done, gamma, v_min, v_max):
    """the same projection as plain loops in fp64 (numpy), the support and every product in double"""
    p, reward, done = np.asarray(p, np.float64), np.asarray(reward, np.float64), np.asarray(done, bool)
    N, K = p.shape
    dz = (v_max - v_min) / (K - 1)
    m = np.zeros((N, K))
    for n in range(N):
        for j in range(K):
            tz = min(max(reward[n] + (0.0 if done[n] else gamma) * (v_min + j * dz), v_min), v_max)
            b = (tz - v_min) / dz
            lo, up = min(max(int(np.floor(b)), 0), K - 1), min(max(int(np.ceil(b)), 0), K - 1)
            if lo == up:
                m[n, lo] += p[n, j]
            else:
                m[n, lo] += p[n, j] * (up - b)
                m[n, up] += p[n, j] * (b - lo)
    return m


def kl(m, logp):
    """sum_k m_k (log m_k - log p_k) with 0 log 0 = 0"""
    return (torch.xlogy(m, m) - m * logp).sum(-1)


def learn_step(online_sd, target_sd, obs, action, reward, next_obs, done, num_atoms, v_min, v_max, weights=None, gamma=0.99,
               double_dqn=False, max_grad_norm=None, lr=1e-3):
    """one learner update in fp32 on the CPU -> dict(q (sum z p at a), y (sum z m), m, ce, kl, loss, dlogits [N, A K] (autograd's),
    grads, params (after Adam), q_scale = sum |z| p and kl_scale = H(m) + CE: the sizes of the terms q and kl sum)"""
    A, K = dims(online_sd, num_atoms)
    z, dz = support(K, v_min, v_max)
    model, target_model = CatRefQNet(A, K, online_sd), CatRefQNet(A, K, target_sd)
    optimizer = optim.Adam(model.parameters(), lr=lr)
    obs, next_obs = obs.cpu(), next_obs.cpu()
    actions, rewards, dones = action.cpu().long(), reward.cpu().float(), done.cpu()
    weights = torch.ones_like(rewards) if weights is None else weights.cpu().float()
    rows = torch.arange(obs.shape[0])
    with torch.no_grad():                                                       # dqn_agent.py:155-163 on the expected Q
        p_next = F.softmax(target_model.logits(next_obs), dim=2)
        if double_dqn:
            a_star = (F.softmax(model.logits(next_obs), dim=2) * z).sum(2).argmax(1)
        else:
            a_star = (p_next * z).sum(2).argmax(1)
        m = project(p_next[rows, a_star], rewards, dones, gamma, z, dz, v_min, v_max)
    logits = model.logits(obs)
    logits.retain_grad()
    logp = F.log_softmax(logits, dim=2)[rows, actions]
    ce = -(m * logp).sum(1)
    loss = (weights * ce).mean()
    optimizer.zero_grad()
    loss.backward()
    grads = OrderedDict((n, p.grad.detach().clone()) for n, p in model.named_parameters())
    if max_grad_norm:                                                           # dqn_agent.py:178-181
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
    optimizer.step()
    with torch.no_grad():
        q = (logp.exp() * z).sum(1)
        # the sizes of the terms Q and KL sum (both cancel: Q on a support around 0, KL = -H(m) + CE): the scale of their fp32 errors
        q_scale = (logp.exp() * z.abs()).sum(1)
        kl_scale = (-torch.xlogy(m, m) - m * logp).sum(1).detach()
        return dict(q=q, q_scale=q_scale, kl_scale=kl_scale, y=(m * z).sum(1), m=m, ce=ce.detach(), kl=kl(m, logp.detach()), loss=float(loss.detach()),
                    dlogits=logits.grad.detach().reshape(obs.shape[0], A * K).clone(), grads=grads,
                    params=OrderedDict((n, p.detach().clone()) for n, p in model.named_parameters()))


def adam_on_grads(params_sd, grads_sd, max_grad_norm=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """the optimizer statements alone (dqn_agent.py:178-182) on given gradients: the first Adam step from zero state"""
    ps = [nn.Parameter(params_sd[n].detach().cpu().float().clone()) for n in NAMES]
    for p, n in zip(ps, NAMES):
        p.grad = grads_sd[n].detach().cpu().float().clone()
    if max_grad_norm:
        torch.nn.utils.clip_grad_norm_(ps, max_grad_norm)
    optim.Adam(ps, lr=lr, betas=betas, eps=eps).step()
    return OrderedDict((n, p.detach()) for n, p in zip(NAMES, ps))


def initial_priorities(sd, state, action, R, next_state, done, gamma_n, eps, num_atoms, v_min, v_max):
    """compute_prior's analogue on n-step transitions in fp32: one Q network (the actor's copy) is the online and the target network,
    no double DQN, pow(gamma, steps) = gamma_n; the priority is max(KL(m || p(s)[a]), 0) + eps.  -> float64 [N]"""
    A, K = dims(sd, num_atoms)
    z, dz = support(K, v_min, v_max)
    model = CatRefQNet(A, K, sd)
    rows = torch.arange(state.shape[0])
    with torch.no_grad():
        p_next = F.softmax(model.logits(next_state.cpu()), dim=2)
        a_star = (p_next * z).sum(2).argmax(1)
        m = project(p_next[rows, a_star], R.cpu().float(), done.cpu(), gamma_n, z, dz, v_min, v_max)
        logp = F.log_softmax(model.logits(state.cpu()), dim=2)[rows, action.cpu().long()]
        return kl(m, logp).clamp(min=0).double() + eps
