"""fp32 CPU oracle of the Ape-X learner step and the actor's initial priorities with the dueling Q network, for the dueling tests.
Independent of scalerl_b200.

The reference declares ``dueling_dqn`` (DQNArguments) but builds no dueling network, so the head restates Wang et al. 2016, eq. 9, on
the reference's own AtariNet layers (oracle/_ref, as oracle/apex_oracle.py's RefQNet):

    V = value(h) = nn.Linear(512, 1),  Adv = advantage(h) = nn.Linear(512, A),  Q = V + Adv - Adv.mean(dim=1, keepdim=True)

Around it, the statements are those of oracle/apex_oracle.py (learn_step, adam_on_grads) and tests/apex_actor_ref.py
(initial_priorities): the reference's Ape-X learner update and DQNAgent's double DQN, clipping and Adam
(scalerl/algorithms/apex/worker.py:134-161, dqn/dqn_agent.py:155-182), and Actor.compute_prior (apex/worker.py:59-79)."""
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet

NAMES = ('conv1.weight', 'conv1.bias', 'conv2.weight', 'conv2.bias', 'conv3.weight', 'conv3.bias', 'fc.weight', 'fc.bias',
         'value.weight', 'value.bias', 'advantage.weight', 'advantage.bias')


def num_actions(sd):
    return sd['advantage.bias'].numel()


class DuelingRefQNet(nn.Module):
    """the reference AtariNet's conv1, conv2, conv3 and fc, then value and advantage on the fc output, Q = V + Adv - mean(Adv)"""

    def __init__(self, num_actions, state_dict=None):
        super().__init__()
        net = AtariNet((4, 84, 84), num_actions)
        self.conv1, self.conv2, self.conv3, self.fc = net.conv1, net.conv2, net.conv3, net.fc
        self.value = nn.Linear(512, 1)
        self.advantage = nn.Linear(512, num_actions)
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
        h = self.features(obs)
        v, adv = self.value(h), self.advantage(h)
        return v + adv - adv.mean(dim=1, keepdim=True)


def learn_step(online_sd, target_sd, obs, action, reward, next_obs, done, weights=None, gamma=0.99, double_dqn=False,
               max_grad_norm=None, lr=1e-3):
    """one learner update in fp32 on the CPU -> dict(q, y, td (= |q - y|), loss, grads, params (after Adam))"""
    A = num_actions(online_sd)
    model, target_model = DuelingRefQNet(A, online_sd), DuelingRefQNet(A, target_sd)
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


def initial_priorities(sd, state, action, R, next_state, done, gamma_n, eps):
    """compute_prior on n-step transitions in fp32 with the dueling network: one Q network (the actor's copy) values both s and s',
    mask = 1 - done, pow(gamma, steps) = gamma_n.  -> float64 |td| + eps [N]"""
    A = num_actions(sd)
    model = DuelingRefQNet(A, sd)
    with torch.no_grad():
        actions = F.one_hot(action.cpu().long(), A).float()
        rewards = R.cpu().float()
        masks = 1 - done.cpu().float()
        pred = model(state.cpu())                                                   # worker.py:69
        next_pred = model(next_state.cpu())                                         # :70
        pred_action = (pred * actions).sum(dim=1)                                   # :72
        target = rewards + masks * gamma_n * next_pred.max(1)[0]                    # :74
        td_error = pred_action - target                                             # :76
        prior = abs(td_error.detach())                                              # :77
    return prior.double() + eps
