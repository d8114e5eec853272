"""fp32 CPU reference of the Ape-X actor's initial priorities, for the actor tests.  Independent of scalerl_b200.

Restates Actor.compute_prior (scalerl/algorithms/apex/worker.py:59-79) on oracle.apex_oracle.RefQNet, the reference's own AtariNet layers
plus q = nn.Linear(512, A).  The reference's Actor cannot be imported (its import root scalerl.algos does not exist, and it needs
gymnasium), so its statements are restated here.  Combined with oracle/replay_oracle.py's fold, it gives the expected priority of every
transition a sequence of adds completes."""
import torch
import torch.nn.functional as F

from oracle.apex_oracle import RefQNet


def initial_priorities(sd, state, action, R, next_state, done, gamma_n, eps):
    """compute_prior on n-step transitions in fp32: one Q network (the actor's copy) values both s and s', mask = 1 - done,
    pow(gamma, steps) = gamma_n.  -> float64 |td| + eps [N]"""
    A = sd['q.bias'].numel()
    model = RefQNet(A, sd)
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
