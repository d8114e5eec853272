"""fp32 CPU oracle of the R2D2 learner step (Kapturowski et al. 2019, "Recurrent Experience Replay in Distributed Reinforcement
Learning"): a recurrent Q network built from the reference's own AtariNet layers (oracle/_ref, built by oracle/make_ref.py: conv1..3,
fc and the 2-layer ``rnn_layer`` of ``AtariNet(use_lstm=True)``) plus the Q head on the core output, and the sequence statements of the
paper.  Independent of scalerl_b200.

    core row      [relu(fc(conv(frame / 255))), clamp(reward, -1, 1), one_hot(last_action)], H = 513 + A (atari_model.py:91-107)
    LSTM          the state multiplied by (1 - done_t) before step t (atari_model.py:109-120)
    head          q = Linear(H, A), or dueling: Q = V + Adv - Adv.mean(1, keepdim=True) (Wang et al. 2016, eq. 9)
    burn-in       rows [0, burn_in) from the stored state without gradient (section 3); the target network runs all L rows
    target        y_t = h(sum_{k=1}^{min(n,m)} gamma^{k-1} r[t+k] + [no m] gamma^n h^-1(Q_target(s_{t+n}, argmax_a Q_online(s_{t+n}))))
                  with m the first k in 1..n with done[t+k] (section 2; h the value rescaling of Pohlen et al. 2018)
    loss          (1 / (B T)) sum_b w_b sum_t (Q_online(s_t, a_t) - y_t)^2, a_t = last_action[t+1]
    priority      eta max_t |delta_t| + (1 - eta) mean_t |delta_t| + eps (section 2)
    optimizer     clip_grad_norm_ (optional) and torch.optim.Adam

The target arithmetic (G, gamma^k, h, h^-1) is evaluated in float64 and y rounded once to fp32, as the kernel states it;
``tail_fp64_loop`` restates the tail with plain numpy loops as a second witness."""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn, optim

from oracle._ref.atari_model import AtariNet


def rescale_h(x, eps):
    """h(x) = sign(x)(sqrt(|x| + 1) - 1) + eps x"""
    return np.sign(x) * (np.sqrt(np.abs(x) + 1.0) - 1.0) + eps * x


def rescale_h_inv(x, eps):
    """h^-1(x) = sign(x)(((sqrt(1 + 4 eps (|x| + 1 + eps)) - 1) / (2 eps))^2 - 1)"""
    return np.sign(x) * (((np.sqrt(1.0 + 4.0 * eps * (np.abs(x) + 1.0 + eps)) - 1.0) / (2.0 * eps)) ** 2 - 1.0)


class RefR2D2Net(nn.Module):
    """the reference AtariNet(use_lstm=True)'s conv1..3, fc and rnn_layer, then q = Linear(H, A) or value / advantage"""

    def __init__(self, A, state_dict=None, dueling=False):
        super().__init__()
        net = AtariNet((4, 84, 84), A, use_lstm=True)
        self.A, self.dueling = A, dueling
        self.conv1, self.conv2, self.conv3, self.fc, self.rnn_layer = net.conv1, net.conv2, net.conv3, net.fc, net.rnn_layer
        H = 513 + A
        if dueling:
            self.value, self.advantage = nn.Linear(H, 1), nn.Linear(H, A)
        else:
            self.q = nn.Linear(H, A)
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})

    def core(self, frame, last_action, reward):          # atari_model.py:91-107
        T, B = frame.shape[:2]
        x = frame.reshape(T * B, 4, 84, 84).float() / 255.0
        x = F.relu(self.conv1(x))
        x = F.relu(self.conv2(x))
        x = F.relu(self.conv3(x))
        x = F.relu(self.fc(x.view(T * B, -1)))
        r = torch.clamp(reward.float(), -1, 1).view(T * B, 1)
        a = F.one_hot(last_action.long().view(T * B), self.A).float()
        return torch.cat([x, r, a], dim=-1).view(T, B, -1)

    def head(self, out):
        if self.dueling:
            v, adv = self.value(out), self.advantage(out)
            return v + adv - adv.mean(dim=-1, keepdim=True)
        return self.q(out)

    def forward(self, frame, last_action, reward, done, state):
        """-> (Q [T, B, A], (hT, cT))"""
        core = self.core(frame, last_action, reward)
        notdone = (~done.bool()).float()
        outs = []
        for t in range(core.shape[0]):                  # atari_model.py:109-120
            state = tuple(notdone[t].view(1, -1, 1) * s for s in state)
            y, state = self.rnn_layer(core[t:t + 1], state)
            outs.append(y)
        return self.head(torch.cat(outs)), state


def tail(q_on, q_tg, last_action, reward, done, burn_in, n, gamma, rescale=True, eps=1e-3):
    """the target statements, vectorised over the batch: q_on [T + n, B, A] (online Q of rows burn_in..L-1, the graph kept), q_tg
    [T, B, A] (target Q of rows burn_in+n..L-1) -> (q_taken [T, B] (differentiable), y [T, B] fp32)"""
    T = q_on.shape[0] - n
    rows = torch.arange(burn_in, burn_in + T)
    act = last_action[rows + 1].long()
    q_taken = q_on[:T].gather(2, act.unsqueeze(2)).squeeze(2)
    a_star = q_on[n:].detach().argmax(dim=2, keepdim=True)          # the first maximal index
    boot = q_tg.gather(2, a_star).squeeze(2).double().numpy()
    r, d = reward.double().numpy(), done.bool().numpy()
    G = np.zeros(q_taken.shape)
    g = np.ones(q_taken.shape)
    live = np.ones(q_taken.shape, dtype=bool)
    for k in range(1, n + 1):
        G = np.where(live, G + g * r[rows.numpy() + k], G)
        live = live & ~d[rows.numpy() + k]
        g = np.where(live, g * np.float64(np.float32(gamma)), g)
    z = G + np.where(live, g * (rescale_h_inv(boot, eps) if rescale else boot), 0.0)
    y = rescale_h(z, eps) if rescale else z
    return q_taken, torch.from_numpy(y.astype(np.float32))


def tail_fp64_loop(q_on, q_tg, last_action, reward, done, burn_in, n, gamma, rescale=True, eps=1e-3, eta=0.9, priority_eps=0.0):
    """a second, independent witness of the tail with plain loops (numpy fp64; q_taken and delta from the fp32 Q values):
    -> (y [T, B] fp32, delta [T, B] fp32, priorities [B] f64)"""
    q_on, q_tg = np.asarray(q_on, np.float32), np.asarray(q_tg, np.float32)
    la, rw, dn = np.asarray(last_action), np.asarray(reward, np.float64), np.asarray(done).astype(bool)
    T, B = q_on.shape[0] - n, q_on.shape[1]
    gamma = float(np.float32(gamma))
    h = lambda x: (np.sign(x) * (np.sqrt(abs(x) + 1.0) - 1.0) + eps * x) if rescale else x
    hinv = lambda x: (np.sign(x) * (((np.sqrt(1.0 + 4.0 * eps * (abs(x) + 1.0 + eps)) - 1.0) / (2.0 * eps)) ** 2 - 1.0)) if rescale else x
    y = np.zeros((T, B), np.float32)
    delta = np.zeros((T, B), np.float32)
    prio = np.zeros(B)
    for b in range(B):
        ad = []
        for i in range(T):
            t = burn_in + i
            q = q_on[i, b, int(la[t + 1, b])]
            a_star = int(np.argmax(q_on[i + n, b]))
            G, disc, ended = 0.0, 1.0, False
            for k in range(1, n + 1):
                G += disc * rw[t + k, b]
                if dn[t + k, b]:
                    ended = True
                    break
                disc *= gamma
            if not ended:
                G += disc * hinv(float(q_tg[i, b, a_star]))
            y[i, b] = np.float32(h(G))
            delta[i, b] = np.float32(q - y[i, b])
            ad.append(abs(float(delta[i, b])))
        prio[b] = eta * max(ad) + (1.0 - eta) * (sum(ad) / T) + priority_eps
    return y, delta, prio


def sequence_step(online, target, params, batch, burn_in, n, gamma, rescale=True, eps=1e-3, eta=0.9, priority_eps=0.0, weights=None,
                  max_grad_norm=None, lr=1e-4, betas=(0.9, 0.999), adam_eps=1e-3, adam_state=None):
    """one update: online / target map (frame, last_action, reward, done, state) -> (Q rows, state) (a RefR2D2Net, or any network of that
    signature), params the online network's named parameters (updated in place by Adam), batch = dict(frame, last_action, reward, done
    [L, B, ...], state (h0, c0)).  -> dict(q_online [T + n, B, A], q_target [T, B, A], q_taken, y, delta [T, B], priorities [B] f64,
    loss, grads (before the clip), state_burn_in)"""
    fr, la, rw, dn, st = (batch[k] for k in ('frame', 'last_action', 'reward', 'done', 'state'))
    L, B = la.shape
    T = L - burn_in - n
    w = torch.ones(B) if weights is None else weights.float()
    with torch.no_grad():
        s = st
        if burn_in:
            _, s = online(fr[:burn_in], la[:burn_in], rw[:burn_in], dn[:burn_in], st)
        q_tg_all, _ = target(fr, la, rw, dn, st)
    q_on, _ = online(fr[burn_in:], la[burn_in:], rw[burn_in:], dn[burn_in:], s)
    q_tg = q_tg_all[burn_in + n:]
    q_taken, y = tail(q_on, q_tg, la, rw, dn, burn_in, n, gamma, rescale, eps)
    delta = q_taken - y
    loss = (w.view(1, B) * delta ** 2).sum() / (B * T)
    ad = delta.detach().abs().double()
    prio = eta * ad.max(0)[0] + (1 - eta) * ad.mean(0) + priority_eps
    plist = list(params.values())
    opt = optim.Adam(plist, lr=lr, betas=betas, eps=adam_eps)
    if adam_state is not None:
        opt.load_state_dict(adam_state)
    opt.zero_grad()
    loss.backward()
    grads = OrderedDict((k, p.grad.detach().clone()) for k, p in params.items())
    if max_grad_norm:
        torch.nn.utils.clip_grad_norm_(plist, max_grad_norm)
    opt.step()
    return dict(q_online=q_on.detach(), q_target=q_tg, q_taken=q_taken.detach(), y=y, delta=delta.detach(), priorities=prio,
                loss=float(loss.detach()), grads=grads, state_burn_in=s, adam_state=opt.state_dict())


def learn_step(online_sd, target_sd, batch, burn_in, n, gamma, dueling=False, **kw):
    """sequence_step on two RefR2D2Nets loaded from state dicts -> its dict plus params (the online network after Adam)"""
    A = online_sd['q.bias' if not dueling else 'advantage.bias'].numel()
    model, target_model = RefR2D2Net(A, online_sd, dueling), RefR2D2Net(A, target_sd, dueling)
    params = OrderedDict(model.named_parameters())
    out = sequence_step(model, target_model, params, batch, burn_in, n, gamma, **kw)
    out['params'] = OrderedDict((k, p.detach().clone()) for k, p in params.items())
    return out
