"""fp32 CPU oracle of the Ape-X learner step and the actor's initial priorities with the quantile (QR-DQN) Q network, for the quantile
tests.  Independent of scalerl_b200.

The reference declares no quantile network, so the head restates Dabney et al. 2018 ("Distributional Reinforcement Learning with
Quantile Regression") on the reference's own AtariNet layers (oracle/_ref, as oracle/apex_oracle.py's RefQNet), with
q = nn.Linear(512, A N), row a N + i quantile i of action a at the midpoint tau_i = (2 i + 1) / (2 N):

    Q(s, a) = (sum_i theta_{a,i}) / N,  T_j = r + gamma theta'_{a*,j} (T_j = r when done),  u_ij = T_j - theta_{a,i}
    rho_ij = |tau_i - 1{u_ij < 0}| L_kappa(u_ij) / kappa,  loss_n = (1 / N) sum_i sum_j rho_ij,  loss = mean_n(w_n loss_n)

a* = argmax_a Q_target(s') (double DQN: argmax_a Q_online(s')); the priority is loss_n + eps.  Around it, the statements are those of
oracle/apex_oracle.py (learn_step, adam_on_grads) and tests/apex_actor_ref.py (initial_priorities): the reference's Ape-X learner update
and DQNAgent's double DQN, clipping and Adam (scalerl/algorithms/apex/worker.py:134-161, dqn/dqn_agent.py:155-182), and
Actor.compute_prior (apex/worker.py:59-79)."""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet

NAMES = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'fc.weight', 'fc.bias',
         'q.weight', 'q.bias')


def taus(N, dtype=torch.float32):
    """tau_i = (2 i + 1) / (2 N)"""
    return (2 * torch.arange(N, dtype=dtype) + 1) / torch.tensor(2 * N, dtype=dtype)


class QrRefQNet(nn.Module):
    """the reference AtariNet's conv1, conv2, conv3 and fc, then q = nn.Linear(512, A N) on the fc output"""

    def __init__(self, num_actions, num_quantiles, state_dict=None):
        super().__init__()
        net = AtariNet((4, 84, 84), num_actions)
        self.A, self.N = num_actions, num_quantiles
        self.conv1, self.conv2, self.conv3, self.fc = net.conv1, net.conv2, net.conv3, net.fc
        self.q = nn.Linear(512, num_actions * num_quantiles)
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})

    def features(self, obs):        # atari_model.py:93-101
        x = obs.float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        x = x.view(x.shape[0], -1)
        return F.relu(self.fc(x))

    def theta(self, obs):
        return self.q(self.features(obs)).view(-1, self.A, self.N)


def dims(sd, num_quantiles):
    return sd['q.bias'].numel() // num_quantiles, num_quantiles


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


def learn_step(online_sd, target_sd, obs, action, reward, next_obs, done, num_quantiles, kappa=1.0, weights=None, gamma=0.99,
               double_dqn=False, max_grad_norm=None, lr=1e-3):
    """one learner update in fp32 on the CPU -> dict(q, y (mean T), T, loss_n, loss, dtheta [N, A N] (written out), dtheta_autograd,
    grads, params (after Adam), q_scale = mean |theta_a|, y_scale = mean |T|: the sizes of the terms q and y sum)"""
    A, N = dims(online_sd, num_quantiles)
    model, target_model = QrRefQNet(A, N, online_sd), QrRefQNet(A, N, target_sd)
    optimizer = optim.Adam(model.parameters(), lr=lr)
    obs, next_obs = obs.cpu(), next_obs.cpu()
    actions, rewards, dones = action.cpu().long(), reward.cpu().float(), done.cpu()
    weights = torch.ones_like(rewards) if weights is None else weights.cpu().float()
    B = obs.shape[0]
    rows = torch.arange(B)
    with torch.no_grad():                                                       # dqn_agent.py:155-163 on the quantile means
        T = targets(target_model.theta(next_obs), rewards, dones, gamma, model.theta(next_obs) if double_dqn else None)
    theta = model.theta(obs)
    theta.retain_grad()
    theta_a = theta[rows, actions]
    loss_n = quantile_loss(theta_a, T, kappa)
    loss = (weights * loss_n).mean()
    optimizer.zero_grad()
    loss.backward()
    grads = OrderedDict((n, p.grad.detach().clone()) for n, p in model.named_parameters())
    if max_grad_norm:                                                           # dqn_agent.py:178-181
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
    optimizer.step()
    with torch.no_grad():
        ta = theta_a.detach()
        dw = torch.zeros(B, A, N)
        dw[rows, actions] = dtheta_written(ta, T, kappa, weights)
        return dict(q=q_of(ta), q_scale=ta.abs().mean(1), y=q_of(T), y_scale=T.abs().mean(1), T=T, theta=theta.detach().clone(),
                    loss_n=loss_n.detach(), loss=float(loss.detach()), dtheta=dw.reshape(B, A * N),
                    dtheta_autograd=theta.grad.detach().reshape(B, A * N).clone(), grads=grads,
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


def initial_priorities(sd, state, action, R, next_state, done, gamma_n, eps, num_quantiles, kappa=1.0):
    """compute_prior's analogue on n-step transitions in fp32: one Q network (the actor's copy) is the online and the target network,
    no double DQN, pow(gamma, steps) = gamma_n; the priority is the quantile Huber loss + eps.  -> float64 [N]"""
    A, N = dims(sd, num_quantiles)
    model = QrRefQNet(A, N, sd)
    rows = torch.arange(state.shape[0])
    with torch.no_grad():
        T = targets(model.theta(next_state.cpu()), R.cpu().float(), done.cpu(), gamma_n)
        theta_a = model.theta(state.cpu())[rows, action.cpu().long()]
        return quantile_loss(theta_a, T, kappa).double() + eps
