"""fp32 CPU oracle of the Ape-X learner step and the actor's initial priorities, for every Q head: the reference's statements around a
Q network built from the reference's own AtariNet layers (oracle/_ref, built by oracle/make_ref.py) plus the head.  Independent of
scalerl_b200.

    learner update   scalerl/algorithms/apex/worker.py:134-161 (Learner.train)
    double DQN       scalerl/algorithms/dqn/dqn_agent.py:155-167
    clip + Adam      dqn_agent.py:172-182, apex/worker.py:132
    target update    dqn_agent.py:185-190 + scalerl/utils/model_utils.py:29-32 (soft_target_update)
    initial priority Actor.compute_prior (apex/worker.py:59-79)

The reference's Actor cannot be imported (its import root scalerl.algos does not exist, and it needs gymnasium), so compute_prior's
statements are restated here.  The reference declares ``dueling_dqn``, ``categorical_dqn`` (``v_min``, ``v_max``, ``num_atoms``) and
``noisy_dqn`` / ``noisy_std`` (DQNArguments) but builds none of these networks, and no quantile network at all, so the heads restate
their papers on the AtariNet layers (``Head`` names one):

    plain        q = nn.Linear(512, A)
    dueling      V = value(h) = nn.Linear(512, 1),  Adv = advantage(h) = nn.Linear(512, A),  Q = V + Adv - Adv.mean(dim=1, keepdim=True)
                 (Wang et al. 2016, eq. 9)
    categorical  q = nn.Linear(512, A K), row a K + k atom k of action a (C51, Bellemare et al. 2017):
                 p(s)[a] = softmax(logits[a K .. a K + K - 1]),  Q(s, a) = sum_k z_k p_k,  z_k = v_min + k dz,  dz = fp32((v_max - v_min) / (K - 1));
                 the target distribution p_target(s')[a*] is projected onto the support by Algorithm 1 (``project``; ``project_fp64_loop``
                 is a second, independent witness in fp64); the loss is mean_n(w_n CE_n), CE_n = -sum_k m_k log p(s_n)[a_n, k]; the
                 priority is max(KL(m || p(s_n)[a_n]), 0) + eps (Hessel et al. 2018)
    quantile     q = nn.Linear(512, A N), row a N + i quantile i of action a at the midpoint tau_i = (2 i + 1) / (2 N) (QR-DQN, Dabney et
                 al. 2018):  Q(s, a) = (sum_i theta_{a,i}) / N,  T_j = r + gamma theta'_{a*,j} (T_j = r when done),  u_ij = T_j - theta_{a,i},
                 rho_ij = |tau_i - 1{u_ij < 0}| L_kappa(u_ij) / kappa,  loss_n = (1 / N) sum_i sum_j rho_ij,  loss = mean_n(w_n loss_n);
                 the priority is loss_n + eps

a* = argmax_a Q_target(s') (double DQN: argmax_a Q_online(s')).  A noisy head (Fortunato et al. 2018, factorised Gaussian noise) makes
fc and every head layer noisy:

    y = (mu_w + sigma_w * eps_w) x + mu_b + sigma_b * eps_b,  eps_w = outer(f(eps_out), f(eps_in)),  eps_b = f(eps_out)

with the noise given, as the f-scaled vectors of one network in the learner's layout (``split_noise``), so the oracle runs on the noise
the device drew.  Parameter names follow the learner's state_dict: conv1..3, fc (AtariNet's names), then q or value and advantage
(``weight_mu``, ``weight_sigma``, ``bias_mu``, ``bias_sigma`` for a noisy layer)."""
from collections import OrderedDict
from typing import NamedTuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet

SUFFIXES = ('weight_mu', 'weight_sigma', 'bias_mu', 'bias_sigma')


class Head(NamedTuple):
    """the Q head: kind 'plain', 'dueling', 'categorical' (num_atoms, v_min, v_max) or 'quantile' (num_quantiles, kappa), noisy or not"""
    kind: str = 'plain'
    noisy: bool = False
    num_atoms: int = 51
    v_min: float = 0.0
    v_max: float = 200.0
    num_quantiles: int = 200
    kappa: float = 1.0

    @property
    def dueling(self):
        return self.kind == 'dueling'

    @property
    def width(self):
        """head rows per action of a distributional head (K atoms or N quantiles), 0 for the scalar heads"""
        return {'categorical': self.num_atoms, 'quantile': self.num_quantiles}.get(self.kind, 0)

    def num_actions(self, sd):
        layer = 'advantage' if self.dueling else 'q'
        return sd[f'{layer}.bias_mu' if self.noisy else f'{layer}.bias'].numel() // (self.width or 1)


# ---------------------------------------------------------------------------------------------------------------- the network
def head_layers(A, dueling=False, num_atoms=0):
    """[(name, out_features)] of the head layers"""
    if dueling:
        return [('value', 1), ('advantage', A)]
    return [('q', A * num_atoms if num_atoms else A)]


def names(dueling=False):
    """the noisy network's parameter names"""
    conv = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias')
    layers = ('fc', 'value', 'advantage') if dueling else ('fc', 'q')
    return conv + tuple(f'{l}.{s}' for l in layers for s in SUFFIXES)


def split_noise(noise, A, dueling=False, num_atoms=0):
    """one network's noise vector [fc in 3136 | fc out 512 | head in 512 per head layer | head out rows] -> {layer: (eps_in, eps_out)}"""
    noise = noise.detach().cpu().float()
    out = {'fc': (noise[:3136], noise[3136:3648])}
    layers = head_layers(A, dueling, num_atoms)
    o = 3648 + 512 * len(layers)
    for i, (name, rows) in enumerate(layers):
        out[name] = (noise[3648 + 512 * i:3648 + 512 * (i + 1)], noise[o:o + rows])
        o += rows
    return out


def scale_noise(x):
    return x.sign().mul(x.abs().sqrt())


class NoisyLayer(nn.Module):
    """factorised Gaussian noisy linear layer with given noise vectors"""

    def __init__(self, in_features, out_features):
        super().__init__()
        self.weight_mu = nn.Parameter(torch.zeros(out_features, in_features))
        self.weight_sigma = nn.Parameter(torch.zeros(out_features, in_features))
        self.bias_mu = nn.Parameter(torch.zeros(out_features))
        self.bias_sigma = nn.Parameter(torch.zeros(out_features))
        self.eps_in, self.eps_out = torch.zeros(in_features), torch.zeros(out_features)

    def weights(self):
        return self.weight_mu + self.weight_sigma * torch.outer(self.eps_out, self.eps_in), self.bias_mu + self.bias_sigma * self.eps_out

    def forward(self, x):
        return F.linear(x, *self.weights())


class RefQNet(nn.Module):
    """the reference AtariNet's conv1, conv2, conv3 and fc, then the head on the fc output (by default the plain q = nn.Linear(512, A));
    with a noisy head, fc and the head layers are NoisyLayers under `noise` (one network's noise vector in the learner's layout)"""

    def __init__(self, A, state_dict=None, head=Head(), noise=None):
        super().__init__()
        net = AtariNet((4, 84, 84), A)
        self.A, self.head = A, head
        self.conv1, self.conv2, self.conv3, self.fc = net.conv1, net.conv2, net.conv3, net.fc
        if head.noisy:
            self.fc = NoisyLayer(3136, 512)
        for name, rows in head_layers(A, head.dueling, head.width):
            setattr(self, name, NoisyLayer(512, rows) if head.noisy else nn.Linear(512, rows))
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})
        if noise is not None:
            for name, (ei, eo) in split_noise(noise, A, head.dueling, head.width).items():
                getattr(self, name).eps_in, getattr(self, name).eps_out = ei.float(), eo.float()

    def features(self, obs):        # atari_model.py:93-101
        x = obs.float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        x = x.view(x.shape[0], -1)
        return F.relu(self.fc(x))

    def forward(self, obs):
        """Q [n, A] of a scalar head; the head rows [n, A, K or N] (logits or quantiles) of a distributional one"""
        h = self.features(obs)
        if self.head.width:
            return self.q(h).view(-1, self.A, self.head.width)
        if self.head.dueling:
            v, adv = self.value(h), self.advantage(h)
            return v + adv - adv.mean(dim=1, keepdim=True)
        return self.q(h)


def q_scale(model, obs, actions):
    """the size of the terms the scalar heads' Q(s, a) sums: the head on |h| with |W| and |b| (dueling: V's, Adv_a's and mean(Adv)'s
    terms added), [N]"""
    h = model.features(obs).abs()
    rows = torch.arange(obs.shape[0])
    ab = lambda layer: F.linear(h, *(t.abs() for t in layer.weights()))
    if model.head.dueling:
        adv = ab(model.advantage)
        return ab(model.value)[:, 0] + adv[rows, actions] + adv.mean(1)
    return ab(model.q)[rows, actions]


def composed(sd, noise, A, dueling=False, num_atoms=0):
    """the effective weights of every noisy layer in torch: {layer: (mu_w + sigma_w * outer(eps_out, eps_in), mu_b + sigma_b * eps_out)}"""
    out = {}
    for name, (ei, eo) in split_noise(noise, A, dueling, num_atoms).items():
        g = lambda s: sd[f'{name}.{s}'].detach().cpu().float()
        out[name] = (g('weight_mu') + g('weight_sigma') * torch.outer(eo, ei), g('bias_mu') + g('bias_sigma') * eo)
    return out


# ---------------------------------------------------------------------------------------------------------------- C51
def support(K, v_min, v_max):
    """(z [K] fp32, dz fp32 scalar tensor): the bounds rounded to fp32, dz = (v_max - v_min) / (K - 1) rounded once, z_k = v_min + k dz"""
    lo, hi = float(np.float32(v_min)), float(np.float32(v_max))
    dz = torch.tensor((hi - lo) / (K - 1), dtype=torch.float32)
    return torch.tensor(lo, dtype=torch.float32) + torch.arange(K, dtype=torch.float32) * dz, dz


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


def _c51_target(head, logits_next_t, reward, done, gamma, logits_next_online=None):
    """m [n, K]: the projected target distribution at a*, the first argmax of Q_target(s') or, with logits_next_online, of Q_online(s')"""
    z, dz = support(head.num_atoms, head.v_min, head.v_max)
    rows = torch.arange(logits_next_t.shape[0])
    p_next = F.softmax(logits_next_t, dim=2)
    a_star = ((p_next if logits_next_online is None else F.softmax(logits_next_online, dim=2)) * z).sum(2).argmax(1)
    return project(p_next[rows, a_star], reward, done, gamma, z, dz, head.v_min, head.v_max)


# ---------------------------------------------------------------------------------------------------------------- QR-DQN
def taus(N, dtype=torch.float32):
    """tau_i = (2 i + 1) / (2 N)"""
    return (2 * torch.arange(N, dtype=dtype) + 1) / torch.tensor(2 * N, dtype=dtype)


def q_of(theta):
    """Q = (sum_i theta_i) / N over the last axis"""
    return theta.sum(-1) / theta.shape[-1]


def targets(theta_next_t, reward, done, gamma, theta_next_online=None):
    """T [n, N] = r + gamma theta_t(s')[a*] (r alone when done: s' is not read), a* the first argmax of Q_target(s') or, with
    theta_next_online, of Q_online(s')"""
    n, dt = theta_next_t.shape[0], theta_next_t.dtype
    g = torch.tensor(float(np.float32(gamma)), dtype=dt)
    rows = torch.arange(n, device=theta_next_t.device)
    a_star = q_of(theta_next_t if theta_next_online is None else theta_next_online).argmax(1)
    r = reward.to(dt)[:, None].expand(n, theta_next_t.shape[2])
    nd = ~done.bool()
    T = r.clone()
    T[nd] = r[nd] + g * theta_next_t[rows, a_star][nd]
    return T


def rho(theta_a, T, kappa):
    """rho [n, N_i, N_j] of the online quantiles theta_a [n, N] against the target quantiles T [n, N]"""
    u = T[:, None, :] - theta_a[:, :, None]
    tau = taus(theta_a.shape[1], theta_a.dtype).to(u.device)[None, :, None]
    L = torch.where(u.abs() <= kappa, 0.5 * u * u, kappa * (u.abs() - 0.5 * kappa))
    return (tau - (u < 0).to(u.dtype)).abs() * L / kappa


def quantile_loss(theta_a, T, kappa):
    """loss_n = (1 / N) sum_i sum_j rho_ij  -> [n]"""
    return rho(theta_a, T, kappa).sum((1, 2)) / theta_a.shape[1]


def dtheta_written(theta_a, T, kappa, weights):
    """d mean_n(w_n loss_n) / d theta_{a,i} = -(w / (B N)) sum_j |tau_i - 1{u_ij < 0}| clamp(u_ij, -kappa, kappa) / kappa -> [n, N]"""
    B, N = theta_a.shape
    u = T[:, None, :] - theta_a[:, :, None]
    tau = taus(N, theta_a.dtype).to(u.device)[None, :, None]
    g = ((tau - (u < 0).to(u.dtype)).abs() * u.clamp(-kappa, kappa) / kappa).sum(2)
    return -(weights[:, None] / (B * N)) * g


# ---------------------------------------------------------------------------------------------------------------- the learner
def learn_step(online_sd, target_sd, obs, action, reward, next_obs, done, weights=None, gamma=0.99, double_dqn=False,
               max_grad_norm=None, lr=1e-3, head=Head(), noise_online=None, noise_target=None):
    """one learner update in fp32 on the CPU (by default with the plain head), a noisy head's networks under their given noise vectors
    (the learner's layout) -> dict(q, y, priorities (|q - y|, KL clamped at 0 or loss_n), loss, grads, params (after Adam)) and the
    head's extras:
      scalar        td (= |q - y|, the reference's td_error: the priorities)
      noisy scalar  q_scale (the size of the terms Q sums)
      categorical   m, ce, kl (unclamped), dlogits [n, A K] (autograd's), q_scale = sum |z| p, y_scale = sum |z| m and
                    kl_scale = H(m) + CE (the sizes of the terms q, y and KL sum: they cancel)
      quantile      T, theta, loss_n, dtheta [n, A N] (written out), dtheta_autograd, q_scale = mean |theta_a|, y_scale = mean |T|"""
    A = head.num_actions(online_sd)
    model, target_model = RefQNet(A, online_sd, head, noise_online), RefQNet(A, target_sd, head, noise_target)
    optimizer = optim.Adam(model.parameters(), lr=lr)
    obs, next_obs = obs.cpu(), next_obs.cpu()
    out = {}
    if not head.width:
        actions = action.cpu().long().unsqueeze(1)
        rewards = reward.cpu().float().unsqueeze(1)
        dones = done.cpu().float().unsqueeze(1)
        weights = torch.ones_like(rewards) if weights is None else weights.cpu().float().unsqueeze(1)
        with torch.no_grad():                                                       # dqn_agent.py:155-163
            if double_dqn:
                greedy_action = model(next_obs).max(dim=1, keepdim=True)[1]
                next_q_values = target_model(next_obs).gather(dim=1, index=greedy_action)
            else:
                next_q_values = target_model(next_obs).max(1, keepdim=True)[0]
        current_q_values = model(obs).gather(1, actions)                            # worker.py:148
        target_q_values = rewards + (1 - dones) * gamma * next_q_values             # worker.py:150
        td_error = torch.abs(current_q_values - target_q_values).detach()           # worker.py:152-153
        loss = (weights * (current_q_values - target_q_values.detach())**2).mean()  # worker.py:156-157
        out.update(q=current_q_values.detach().squeeze(1), y=target_q_values.detach().squeeze(1), td=td_error.squeeze(1),
                   priorities=td_error.squeeze(1))
        if head.noisy:
            with torch.no_grad():
                out.update(q_scale=q_scale(model, obs, actions.squeeze(1)))
    else:
        actions, rewards, dones = action.cpu().long(), reward.cpu().float(), done.cpu()
        weights = torch.ones_like(rewards) if weights is None else weights.cpu().float()
        B = obs.shape[0]
        rows = torch.arange(B)
        with torch.no_grad():                                                       # dqn_agent.py:155-163 on the expected Q
            nxt = model(next_obs) if double_dqn else None
            if head.kind == 'categorical':
                m = _c51_target(head, target_model(next_obs), rewards, dones, gamma, nxt)
            else:
                T = targets(target_model(next_obs), rewards, dones, gamma, nxt)
        rows_out = model(obs)
        rows_out.retain_grad()
        if head.kind == 'categorical':
            z = support(head.num_atoms, head.v_min, head.v_max)[0]
            logp = F.log_softmax(rows_out, dim=2)[rows, actions]
            ce = -(m * logp).sum(1)
            loss = (weights * ce).mean()
            with torch.no_grad():
                p = logp.exp()
                out.update(q=(p * z).sum(1), q_scale=(p * z.abs()).sum(1), y=(m * z).sum(1), y_scale=(m * z.abs()).sum(1), m=m, ce=ce.detach(),
                           kl=kl(m, logp), priorities=kl(m, logp).clamp(min=0), kl_scale=(-torch.xlogy(m, m) - m * logp).sum(1))
        else:
            theta_a = rows_out[rows, actions]
            loss_n = quantile_loss(theta_a, T, head.kappa)
            loss = (weights * loss_n).mean()
            with torch.no_grad():
                ta = theta_a.detach()
                dw = torch.zeros(B, A, head.width)
                dw[rows, actions] = dtheta_written(ta, T, head.kappa, weights)
                out.update(q=q_of(ta), q_scale=ta.abs().mean(1), y=q_of(T), y_scale=T.abs().mean(1), T=T, theta=rows_out.detach().clone(),
                           loss_n=loss_n.detach(), priorities=loss_n.detach(), dtheta=dw.reshape(B, A * head.width))
    optimizer.zero_grad()
    loss.backward()
    grads = OrderedDict((n, p.grad.detach().clone()) for n, p in model.named_parameters())
    if max_grad_norm:                                                           # dqn_agent.py:178-181
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
    optimizer.step()
    if head.width:
        dr = rows_out.grad.detach().reshape(obs.shape[0], -1).clone()
        out.update(dlogits=dr) if head.kind == 'categorical' else out.update(dtheta_autograd=dr)
    out.update(loss=float(loss.detach()), grads=grads, params=OrderedDict((n, p.detach().clone()) for n, p in model.named_parameters()))
    return out


def adam_on_grads(params_sd, grads_sd, max_grad_norm=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """the optimizer statements alone (dqn_agent.py:178-182) on given gradients: the first Adam step from zero state, in the
    state-dict order of params_sd"""
    order = list(params_sd)
    ps = [nn.Parameter(params_sd[n].detach().cpu().float().clone()) for n in order]
    for p, n in zip(ps, order):
        p.grad = grads_sd[n].detach().cpu().float().clone()
    if max_grad_norm:
        torch.nn.utils.clip_grad_norm_(ps, max_grad_norm)
    optim.Adam(ps, lr=lr, betas=betas, eps=eps).step()
    return OrderedDict((n, p.detach()) for n, p in zip(order, ps))


def initial_priorities(sd, state, action, R, next_state, done, gamma_n, eps, head=Head()):
    """compute_prior (or its analogue for a distributional head) on n-step transitions in fp32: one Q network (the actor's copy) values
    both s and s', no double DQN, mask = 1 - done, pow(gamma, steps) = gamma_n.  -> float64 priority + eps [N]: |td|, max(KL, 0) or the
    quantile Huber loss"""
    A = head.num_actions(sd)
    model = RefQNet(A, sd, head)
    state, next_state, action, done = state.cpu(), next_state.cpu(), action.cpu().long(), done.cpu()
    rows = torch.arange(state.shape[0])
    with torch.no_grad():
        if head.kind == 'categorical':
            m = _c51_target(head, model(next_state), R.cpu().float(), done, gamma_n)
            prior = kl(m, F.log_softmax(model(state), dim=2)[rows, action]).clamp(min=0)
        elif head.kind == 'quantile':
            T = targets(model(next_state), R.cpu().float(), done, gamma_n)
            prior = quantile_loss(model(state)[rows, action], T, head.kappa)
        else:
            actions = F.one_hot(action, A).float()
            rewards = R.cpu().float()
            masks = 1 - done.float()
            pred = model(state)                                                         # worker.py:69
            next_pred = model(next_state)                                               # :70
            pred_action = (pred * actions).sum(dim=1)                                   # :72
            target = rewards + masks * gamma_n * next_pred.max(1)[0]                    # :74
            td_error = pred_action - target                                             # :76
            prior = abs(td_error.detach())                                              # :77
    return prior.double() + eps


def soft_target_update(src_params, tgt_params, tau):
    """utils/model_utils.py:29-32 on lists of tensors (on any device)"""
    for src_param, tgt_param in zip(src_params, tgt_params):
        tgt_param.data.copy_(tau * src_param.data + (1.0 - tau) * tgt_param.data)
