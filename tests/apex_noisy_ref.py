"""fp32 CPU oracle of the Ape-X learner step with noisy networks (Fortunato et al. 2018, factorised Gaussian noise), for the noisy tests.
Independent of scalerl_b200.

The reference declares ``noisy_dqn`` and ``noisy_std`` (DQNArguments) but builds no noisy network, so the noisy layer is restated here
on the reference's own AtariNet conv layers (oracle/_ref, as the dueling and categorical oracles):

    y = (mu_w + sigma_w * eps_w) x + mu_b + sigma_b * eps_b,  eps_w = outer(f(eps_out), f(eps_in)),  eps_b = f(eps_out)

fc and every head layer are noisy: q (plain or categorical) or value and advantage (dueling).  The noise is given, as the f-scaled
vectors of one network in the learner's layout (``split_noise``), so the oracle runs on the noise the device drew.  Around the network
the statements are those of tests/apex_dueling_ref.py (scalar heads) and tests/apex_categorical_ref.py (C51)."""
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet
from tests import apex_categorical_ref as CR

SUFFIXES = ('weight_mu', 'weight_sigma', 'bias_mu', 'bias_sigma')


def head_layers(A, dueling=False, num_atoms=0):
    """[(name, out_features)] of the noisy head layers"""
    if dueling:
        return [('value', 1), ('advantage', A)]
    return [('q', A * num_atoms if num_atoms else A)]


def names(dueling=False):
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


class NoisyRefQNet(nn.Module):
    """the reference AtariNet's conv1..3, then fc and the head as noisy layers under `noise` ({layer: (eps_in, eps_out)})"""

    def __init__(self, A, dueling=False, num_atoms=0, state_dict=None, noise=None):
        super().__init__()
        net = AtariNet((4, 84, 84), A)
        self.A, self.K, self.dueling = A, num_atoms, dueling
        self.conv1, self.conv2, self.conv3 = net.conv1, net.conv2, net.conv3
        self.fc = NoisyLayer(3136, 512)
        for name, rows in head_layers(A, dueling, num_atoms):
            setattr(self, name, NoisyLayer(512, rows))
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})
        for name, (ei, eo) in (noise or {}).items():
            getattr(self, name).eps_in, getattr(self, name).eps_out = ei.float(), eo.float()

    def features(self, obs):        # atari_model.py:93-101 with the noisy fc
        x = obs.float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        return F.relu(self.fc(x.view(x.shape[0], -1)))

    def logits(self, obs):
        return self.q(self.features(obs)).view(-1, self.A, self.K)

    def forward(self, obs):
        h = self.features(obs)
        if self.dueling:
            v, adv = self.value(h), self.advantage(h)
            return v + adv - adv.mean(dim=1, keepdim=True)
        return self.q(h)


def q_scale(model, obs, actions):
    """the size of the terms the scalar heads' Q(s, a) sums: the head on |h| with |W| and |b| (dueling: V's, Adv_a's and mean(Adv)'s
    terms added), [N]"""
    h = model.features(obs).abs()
    rows = torch.arange(obs.shape[0])
    ab = lambda layer: F.linear(h, *(t.abs() for t in layer.weights()))
    if model.dueling:
        adv = ab(model.advantage)
        return ab(model.value)[:, 0] + adv[rows, actions] + adv.mean(1)
    return ab(model.q)[rows, actions]


def learn_step(online_sd, target_sd, noise_online, noise_target, obs, action, reward, next_obs, done, dueling=False, num_atoms=0,
               v_min=0.0, v_max=200.0, weights=None, gamma=0.99, double_dqn=False, max_grad_norm=None, lr=1e-3):
    """one learner update in fp32 on the CPU, both networks under their given noise vectors (the learner's layout) -> dict(q, y,
    priorities (|q - y|, or KL for C51), q_scale (the size of the terms Q sums), loss, grads, params (after Adam)); C51 adds y_scale and
    kl_scale (apex_categorical_ref's)"""
    A = online_sd['advantage.bias_mu' if dueling else 'q.bias_mu'].numel() // (num_atoms or 1)
    model = NoisyRefQNet(A, dueling, num_atoms, online_sd, split_noise(noise_online, A, dueling, num_atoms))
    target_model = NoisyRefQNet(A, dueling, num_atoms, target_sd, split_noise(noise_target, A, dueling, num_atoms))
    optimizer = optim.Adam(model.parameters(), lr=lr)
    obs, next_obs = obs.cpu(), next_obs.cpu()
    actions, rewards, dones = action.cpu().long(), reward.cpu().float(), done.cpu()
    weights = torch.ones_like(rewards) if weights is None else weights.cpu().float()
    rows = torch.arange(obs.shape[0])
    out = {}
    if num_atoms:
        z, dz = CR.support(num_atoms, v_min, v_max)
        with torch.no_grad():
            p_next = F.softmax(target_model.logits(next_obs), dim=2)
            a_star = ((F.softmax(model.logits(next_obs), dim=2) if double_dqn else p_next) * z).sum(2).argmax(1)
            m = CR.project(p_next[rows, a_star], rewards, dones, gamma, z, dz, v_min, v_max)
        logp = F.log_softmax(model.logits(obs), dim=2)[rows, actions]
        loss = (weights * -(m * logp).sum(1)).mean()
        with torch.no_grad():
            out.update(q=(logp.exp() * z).sum(1), q_scale=(logp.exp() * z.abs()).sum(1), y=(m * z).sum(1), y_scale=(m * z.abs()).sum(1),
                       priorities=CR.kl(m, logp).clamp(min=0), kl_scale=(-torch.xlogy(m, m) - m * logp).sum(1))
    else:
        with torch.no_grad():                                                   # dqn_agent.py:155-163
            qn_t = target_model(next_obs)
            a_star = (model(next_obs) if double_dqn else qn_t).argmax(1)
            y = rewards + (1 - dones.float()) * gamma * qn_t[rows, a_star]
        q = model(obs)[rows, actions]
        loss = (weights * (q - y) ** 2).mean()
        with torch.no_grad():
            out.update(q=q.detach(), y=y, priorities=(q - y).abs().detach(), q_scale=q_scale(model, obs, actions))
    optimizer.zero_grad()
    loss.backward()
    grads = OrderedDict((n, p.grad.detach().clone()) for n, p in model.named_parameters())
    if max_grad_norm:                                                           # dqn_agent.py:178-181
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
    optimizer.step()
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


def composed(sd, noise, A, dueling=False, num_atoms=0):
    """the effective weights of every noisy layer in torch: {layer: (mu_w + sigma_w * outer(eps_out, eps_in), mu_b + sigma_b * eps_out)}"""
    out = {}
    for name, (ei, eo) in split_noise(noise, A, dueling, num_atoms).items():
        g = lambda s: sd[f'{name}.{s}'].detach().cpu().float()
        out[name] = (g('weight_mu') + g('weight_sigma') * torch.outer(eo, ei), g('bias_mu') + g('bias_sigma') * eo)
    return out
