"""fp32 CPU oracle of the Ape-X learner step: the reference's statements around a Q network built from the reference's own AtariNet
layers (oracle/_ref, built by oracle/make_ref.py) plus ``nn.Linear(512, A)``.  Independent of scalerl_b200.

    learner update   scalerl/algorithms/apex/worker.py:134-161 (Learner.train)
    double DQN       scalerl/algorithms/dqn/dqn_agent.py:155-167
    clip + Adam      dqn_agent.py:172-182, apex/worker.py:132
    target update    dqn_agent.py:185-190 + scalerl/utils/model_utils.py:29-32 (soft_target_update)

Parameter names follow the learner's state_dict: conv1..3, fc (AtariNet's names) and q."""
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet

NAMES = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'fc.weight', 'fc.bias',
         'q.weight', 'q.bias')


class RefQNet(nn.Module):
    """the reference AtariNet's conv1, conv2, conv3 and fc, then q = nn.Linear(512, A)"""

    def __init__(self, num_actions, state_dict=None):
        super().__init__()
        net = AtariNet((4, 84, 84), num_actions)
        self.conv1, self.conv2, self.conv3, self.fc = net.conv1, net.conv2, net.conv3, net.fc
        self.q = nn.Linear(512, num_actions)
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})

    def features(self, obs):        # atari_model.py:93-101
        x = obs.float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        x = x.view(x.shape[0], -1)
        return F.relu(self.fc(x))

    def forward(self, obs):
        return self.q(self.features(obs))


def learn_step(online_sd, target_sd, obs, action, reward, next_obs, done, weights=None, gamma=0.99, double_dqn=False,
               max_grad_norm=None, lr=1e-3):
    """one learner update in fp32 on the CPU -> dict(q, y, td (= |q - y|), loss, grads, params (after Adam), target_q_next)"""
    A = online_sd['q.bias'].numel()
    model, target_model = RefQNet(A, online_sd), RefQNet(A, target_sd)
    optimizer = optim.Adam(model.parameters(), lr=lr)
    obs, next_obs = obs.cpu(), next_obs.cpu()
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
    optimizer.zero_grad()
    loss.backward()
    grads = OrderedDict((n, p.grad.detach().clone()) for n, p in model.named_parameters())
    if max_grad_norm:                                                           # dqn_agent.py:178-181
        torch.nn.utils.clip_grad_norm_(model.parameters(), max_grad_norm)
    optimizer.step()
    return dict(q=current_q_values.detach().squeeze(1), y=target_q_values.detach().squeeze(1), td=td_error.squeeze(1),
                loss=float(loss.detach()), grads=grads, params=OrderedDict((n, p.detach().clone()) for n, p in model.named_parameters()))


def adam_on_grads(params_sd, grads_sd, max_grad_norm=None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8):
    """the optimizer statements alone (dqn_agent.py:178-182) on given gradients: the first Adam step from zero state"""
    ps = [nn.Parameter(params_sd[n].detach().cpu().float().clone()) for n in NAMES]
    for p, n in zip(ps, NAMES):
        p.grad = grads_sd[n].detach().cpu().float().clone()
    if max_grad_norm:
        torch.nn.utils.clip_grad_norm_(ps, max_grad_norm)
    optim.Adam(ps, lr=lr, betas=betas, eps=eps).step()
    return OrderedDict((n, p.detach()) for n, p in zip(NAMES, ps))


def soft_target_update(src_params, tgt_params, tau):
    """utils/model_utils.py:29-32 on lists of tensors (on any device)"""
    for src_param, tgt_param in zip(src_params, tgt_params):
        tgt_param.data.copy_(tau * src_param.data + (1.0 - tau) * tgt_param.data)
