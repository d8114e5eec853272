"""The quantile (QR-DQN) head of the Ape-X learner and actors on the H100 (ApexHParams(quantile_dqn=True),
B200ApexActor(..., quantile_dqn=True)); 1-3 and 5-6 are the checks every head shares (tests/apex_cases.py):
  1. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py): Q(s, a) and y normalised by the size of the
     terms they sum, the target quantiles, the per-transition loss, priorities and loss to 1e-5, the 10 gradients to rel-L2 1e-4 (2e-2
     when a genuine ReLU tie flipped), the weights after the step against the oracle's Adam on the device gradients to 2e-6;
  2. bf16: the quantile tail against fp64 on its own operands (core rows, fp32 head weights): theta, the target quantiles, the loss,
     dtheta, the head gradients and dcore; the encoder gradients equal srl_encoder_backward on the tail's dcore, bit for bit; done
     transitions do not read s';
  3. the actor's quantiles, Q values and eps = 0 actions are the learner's bit for bit (ties included), bf16 actor priorities are the
     learner's bit for bit, fp32-accurate actor priorities match the oracle's and the trees match PerOracle;
  4. noisy: with sigma = 0 a step is the plain quantile learner's on mu, bit for bit, and the composed head weights are torch's;
  5. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; checkpoints load into
     AtariQNet(A, quantile=True) and torch.optim.Adam, and a resumed run equals an uninterrupted one;
  6. q_values against the CPU network.
The measured errors are written to $SRL_RESULTS_DIR/apex_quantile.json when SRL_RESULTS_DIR is set."""
import math

import pytest
import torch

from oracle import apex_oracle as O
from scalerl_b200.algorithms.apex import default_q_state_dict
from tests import apex_cases as cases
from tests.apex_cases import HEADS, batch, learner

pytestmark = pytest.mark.gpu
QR = HEADS['quantile']                                 # N = 200, kappa = 1
GRID = [(32, 6, 200), (5, 4, 2), (512, 18, 51)]


def _qr(N, kappa=1.0):
    return QR.but(width=N, kappa=kappa)


def _learner(B, A, N, on, tg, **kw):
    return learner(QR.but(width=N), B, A, on, tg, **kw)


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('kappa', [1.0, 0.5])
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,N', GRID)
def test_split_against_quantile_oracle(B, A, N, double, clip, kappa):
    cases.check_split_against_oracle(_qr(N, kappa), B, A, double, clip)


# ---------------------------------------------------------------------------------------------------------------- 2
@pytest.mark.parametrize('kappa', [1.0, 0.5])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,N', [(32, 6, 200), (512, 18, 51)])
def test_bf16_quantile_tail_against_fp64_and_encoder_backward(B, A, N, double, kappa):
    cases.check_bf16_tail_and_encoder_backward(_qr(N, kappa), B, A, double)


def test_done_transitions_do_not_read_s_prime():
    """every transition done: the targets are the rewards, whatever the target network says of s' (here: inf quantiles)"""
    B, A, N = 16, 4, 32
    on, tg = (default_q_state_dict(A, s, num_quantiles=N) for s in (10, 11))
    tg['q.bias'] = torch.full_like(tg['q.bias'], math.inf)
    (obs, act, rew, nobs, done), w = batch(B, A, seed=9, device='cuda')
    L = _learner(B, A, N, on, tg, priority_eps=0.0)
    L.learn((obs, act, rew, nobs, torch.ones_like(done)), weights=w, use_graph=False)
    assert torch.equal(L.debug_buffer('target_quantiles').view(B, N), rew[:, None].expand(B, N))
    assert bool(torch.isfinite(L.debug_buffer('priorities')).all()) and math.isfinite(float(L.debug_buffer('loss')[0]))


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256])
def test_actor_quantiles_q_values_and_greedy_act_are_the_learners(E):
    cases.check_actor_q_values_and_greedy_act(QR, E)


def test_fp32_actor_priorities_against_oracle_and_trees():
    cases.check_fp32_actor_priorities(_qr(51, 0.5))


def test_bf16_actor_priorities_are_the_learners():
    cases.check_bf16_actor_priorities(QR)


# ---------------------------------------------------------------------------------------------------------------- 4
@pytest.mark.parametrize('double', [False, True])
def test_noisy_sigma_zero_is_the_plain_quantile_learner(double):
    B, A, N = 32, 6, 51
    on, tg = (default_q_state_dict(A, s, noisy=True, noisy_std=0.0, num_quantiles=N) for s in (6, 7))
    strip = lambda sd: {n.replace('_mu', ''): v for n, v in sd.items() if 'sigma' not in n}
    step_batch, w = batch(B, A, seed=4, device='cuda')
    Nz = learner(QR.but(width=N, noisy=True), B, A, on, tg, double_dqn=double)
    P = _learner(B, A, N, strip(on), strip(tg), double_dqn=double)
    Nz.learn(step_batch, weights=w, use_graph=False)
    P.learn(step_batch, weights=w, use_graph=False)
    for k in ('q', 'y', 'priorities', 'loss', 'dcore', 'theta', 'target_quantiles', 'qr_loss', 'dtheta'):
        assert torch.equal(Nz.debug_buffer(k), P.debug_buffer(k)), k
    for n, g in P.grads.items():
        m = n.replace('weight', 'weight_mu').replace('bias', 'bias_mu') if not n.startswith('conv') else n
        assert torch.equal(Nz.grads[m], g), n
        assert torch.equal(Nz.params[m], P.params[n]), n
    assert bool(Nz.grads['q.weight_sigma'].any())          # sigma learns even from 0


def test_noisy_quantile_composition_is_torchs():
    B, A, N = 16, 4, 64
    on, tg = (default_q_state_dict(A, s, noisy=True, num_quantiles=N) for s in (8, 9))
    step_batch, w = batch(B, A, seed=5, device='cuda')
    L = learner(QR.but(width=N, noisy=True), B, A, on, tg, double_dqn=True)
    L.learn(step_batch, weights=w, use_graph=False)
    for net, sd in (('online', on), ('target', tg)):
        noise = L.debug_buffer(f'noise_{net}').cpu()
        want = O.composed(sd, noise, A, False, N)
        assert torch.equal(L.debug_buffer(f'head_weight_{net}').view(-1, 512).cpu(), want['q'][0]), net
        assert torch.equal(L.debug_buffer(f'head_bias_{net}').cpu(), want['q'][1]), net
    ei, eo = O.split_noise(L.debug_buffer('noise_online'), A, False, N)['q']
    assert torch.equal(L.grads['q.weight_sigma'].cpu(), L.grads['q.weight_mu'].cpu() * torch.outer(eo, ei))


# ---------------------------------------------------------------------------------------------------------------- 5
def test_determinism_and_graph_replay():
    cases.check_determinism_and_graph_replay(QR)


def test_captured_learn_from_loop_is_deterministic():
    cases.check_captured_learn_from_loop(_qr(51))


def test_checkpoint_roundtrip_and_resume(tmp_path):
    cases.check_checkpoint_roundtrip_and_resume(QR, tmp_path)


# ---------------------------------------------------------------------------------------------------------------- 6
@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    cases.check_q_values_against_cpu_network(QR, precision, tol)
