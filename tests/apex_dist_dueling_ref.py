"""The fp32 CPU oracle of the distributional dueling head, on top of oracle/apex_oracle.py: Rainbow's dueling rows per atom or quantile
(Hessel et al. 2018) for the categorical (C51) or quantile (QR-DQN) head, W = K atoms or N quantiles per action:

    v = value(h) = nn.Linear(512, W),  adv = advantage(h) = nn.Linear(512, A W),
    rows = v.view(-1, 1, W) + adv.view(-1, A, W) - adv.view(-1, A, W).mean(1, keepdim=True)

on the reference's AtariNet conv1..3 and fc.  The rows are what the C51 or QR head's q layer gives, so the learner update and the
initial priorities are apex_oracle's own statements (learn_step, initial_priorities) on this network: ``installed()`` makes them build
it for a ``Head`` of this module, while every other head keeps apex_oracle's network.  Independent of scalerl_b200."""
import contextlib
from unittest import mock

from torch import nn

from oracle import apex_oracle as O
from oracle._ref.atari_model import AtariNet

_RefQNet = O.RefQNet


class Head(O.Head):
    """apex_oracle's Head of kind 'categorical' (num_atoms, v_min, v_max) or 'quantile' (num_quantiles, kappa), as dueling rows"""
    __slots__ = ()

    def num_actions(self, sd):
        return sd['advantage.bias_mu' if self.noisy else 'advantage.bias'].numel() // self.width


def split_noise(noise, A, W):
    """one network's noise vector [fc in 3136 | fc out 512 | value in 512 | advantage in 512 | value out W | advantage out A W] ->
    {layer: (eps_in, eps_out)}"""
    noise = noise.detach().cpu().float()
    o = 3648 + 1024
    return {'fc': (noise[:3136], noise[3136:3648]), 'value': (noise[3648:4160], noise[o:o + W]),
            'advantage': (noise[4160:4672], noise[o + W:o + W + A * W])}


class RefQNet(_RefQNet):
    """apex_oracle's RefQNet, and for a Head of this module the reference AtariNet's conv1..3 and fc, then value and advantage (noisy:
    NoisyLayers under `noise`, one network's noise vector in the learner's layout), whose forward gives the head rows [n, A, W]"""

    def __init__(self, A, state_dict=None, head=O.Head(), noise=None):
        if not isinstance(head, Head):
            super().__init__(A, state_dict, head, noise)
            return
        nn.Module.__init__(self)
        net = AtariNet((4, 84, 84), A)
        self.A, self.head = A, head
        self.conv1, self.conv2, self.conv3, self.fc = net.conv1, net.conv2, net.conv3, net.fc
        W = head.width
        layer = (lambda i, o: O.NoisyLayer(i, o)) if head.noisy else nn.Linear
        if head.noisy:
            self.fc = O.NoisyLayer(3136, 512)
        self.value, self.advantage = layer(512, W), layer(512, A * W)
        if state_dict is not None:
            self.load_state_dict({k: v.detach().cpu().float() for k, v in state_dict.items()})
        if noise is not None:
            for name, (ei, eo) in split_noise(noise, A, W).items():
                getattr(self, name).eps_in, getattr(self, name).eps_out = ei.float(), eo.float()

    def forward(self, obs):
        if not isinstance(self.head, Head):
            return super().forward(obs)
        h = self.features(obs)
        W = self.head.width
        v, adv = self.value(h).view(-1, 1, W), self.advantage(h).view(-1, self.A, W)
        return v + adv - adv.mean(1, keepdim=True)


@contextlib.contextmanager
def installed():
    """within the block apex_oracle builds its networks (learn_step, initial_priorities) as RefQNet above"""
    with mock.patch.object(O, 'RefQNet', RefQNet):
        yield
