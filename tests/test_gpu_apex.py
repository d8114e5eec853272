"""The Ape-X learner step on the H100 (B200ApexLearner / srl_apex_learner_*) with the plain head; the checks every head shares are in
tests/apex_cases.py:
  1. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py): q, y, priorities and loss to 1e-5, every
     gradient to rel-L2 1e-4 when no ReLU mask differs from fp32 (2e-2 otherwise, and then every flipped unit must be a genuine tie:
     the tie accounting of test_gpu_precision.py), the weights after the step against the oracle's Adam on the device gradients to 2e-6;
  2. bf16: the tail against fp64 evaluated on its own operands (the core rows and the fp32 head weights); the encoder gradients equal
     srl_encoder_backward called directly on the tail's dcore, bit for bit;
  3. the priorities reach the sampler's trees (last occurrence of a repeated idx wins);
  4. repeated runs and graph replay give the same parameters bit for bit, with the device step count advancing;
  5. the target update is soft_target_update's arithmetic on the reference's cadence;
  6. checkpoints load into torch.optim.Adam(AtariQNet(...).parameters()), and a resumed run equals an uninterrupted one;
  7. q_values / predict against AtariQNet on the CPU.
The measured errors are written to $SRL_RESULTS_DIR/apex.json when SRL_RESULTS_DIR is set."""
import numpy as np
import pytest
import torch

from oracle import apex_oracle as O
from oracle.per_oracle import PerOracle
from scalerl_b200.algorithms.apex import APEX_PARAM_NAMES
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler
from tests import apex_cases as cases
from tests.apex_cases import HEADS, batch, learner, nets

pytestmark = pytest.mark.gpu
PLAIN = HEADS['plain']


# ---------------------------------------------------------------------------------------------------------------- 1, 2
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (5, 4), (512, 18)])
def test_split_against_fp32_oracle(B, A, double, clip):
    cases.check_split_against_oracle(PLAIN, B, A, double, clip)


@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (512, 18)])
def test_bf16_tail_against_fp64_and_encoder_backward(B, A, double):
    cases.check_bf16_tail_and_encoder_backward(PLAIN, B, A, double)


@pytest.mark.parametrize('B', [4097, 65536])
def test_bf16_tail_and_encoder_backward_large_batch(B):
    """above B = 512: the tail's block count, the head weight-gradient slabs and the three forwards at a ragged batch and at
    MAX_FRAMES"""
    cases.check_bf16_tail_and_encoder_backward(PLAIN, B, 6, True)


# ---------------------------------------------------------------------------------------------------------------- 3
def test_priorities_reach_the_trees():
    B, mem = 48, 64
    _check_priorities(B, mem, ((2, 7), (0, B - 1)))          # repeated indices: the last occurrence wins


def test_priorities_reach_the_trees_across_launches():
    """srl_per_update_priorities writes 1024 pairs per launch: at B = 2500 (three launches) a repeated index keeps its LAST
    occurrence across launches too"""
    _check_priorities(2500, 3000, ((5, 1024), (1023, 1024), (1023, 2048), (100, 1500), (1030, 2100), (0, 2499), (2, 7)))


def _check_priorities(B, mem, repeats):
    A = 6
    on, tg = nets(PLAIN, A)
    step_batch, w = batch(B, A, seed=11, device='cuda')
    S = GpuPrioritizedSampler(mem, alpha=0.6)
    S.add(mem)
    idxs = torch.randint(0, mem, (B,), generator=torch.Generator().manual_seed(5))
    for first, later in repeats:
        idxs[later] = idxs[first]
    L = learner(PLAIN, B, A, on, tg, priority_eps=1e-6)
    L.learn(step_batch, weights=w, idxs=idxs.cuda(), sampler=S, use_graph=False)
    prio = L.debug_buffer('priorities').cpu().numpy()
    o = PerOracle(mem, 0.6)
    o.add(mem)
    o.update_priorities(idxs.numpy(), prio)
    st, mt, mp = S.trees()
    assert mp == o.max_priority
    cap = S.capacity
    leaves = st[cap:cap + mem].cpu().numpy()
    ref = o.sum_tree.tree[cap:cap + mem]
    assert np.allclose(leaves, ref, rtol=1e-14, atol=0)
    o.set_leaves(np.nonzero(leaves != ref)[0], leaves[leaves != ref])      # adopt the GPU's rounding of p ** alpha
    assert np.array_equal(st.cpu().numpy()[1:], o.sum_tree.tree[1:])
    assert np.array_equal(mt.cpu().numpy()[1:], o.min_tree.tree[1:])


# ---------------------------------------------------------------------------------------------------------------- 5
@pytest.mark.parametrize('tau', [1.0, 0.05])
def test_target_update_cadence(tau):
    B, A, freq = 16, 4, 3
    on, tg = nets(PLAIN, A, seed=2)
    L = learner(PLAIN, B, A, on, tg, target_update_frequency=freq, soft_update_tau=tau)
    for k in range(7):
        step_batch, w = batch(B, A, seed=20 + k, device='cuda')
        before = [t.clone() for t in L.target_params.values()]
        L.learn(step_batch, weights=w, use_graph=False)
        if k % freq == 0:                    # dqn_agent.py:185-187, counted from 0
            O.soft_target_update(list(L.params.values()), before, tau)
        for n, e in zip(APEX_PARAM_NAMES, before):
            assert torch.equal(L.target_params[n], e), (k, n)
    assert L.target_model_update_step == 3
    if tau == 1.0:
        L.update_target(1.0)
        for n in APEX_PARAM_NAMES:
            assert torch.equal(L.target_params[n], L.params[n])


def test_determinism_and_graph_replay():
    cases.check_determinism_and_graph_replay(PLAIN)


def test_checkpoint_roundtrip_and_resume(tmp_path):
    cases.check_checkpoint_roundtrip_and_resume(PLAIN, tmp_path)


@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    cases.check_q_values_against_cpu_network(PLAIN, precision, tol)
