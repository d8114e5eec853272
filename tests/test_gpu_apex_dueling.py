"""The dueling head of the Ape-X learner and actors on the H100 (ApexHParams(dueling_dqn=True), B200ApexActor(..., dueling_dqn=True)),
run through the checks every head shares (tests/apex_cases.py):
  1. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py): q, y, priorities and loss to 1e-5, the 12
     gradients to rel-L2 1e-4 (2e-2 when a genuine ReLU tie flipped), the weights after the step against the oracle's Adam to 2e-6;
  2. bf16: the dueling tail against fp64 on its own operands (core rows, fp32 head weights); the encoder gradients equal
     srl_encoder_backward on the tail's dcore, bit for bit;
  3. the actor's Q values are the learner's bit for bit, act with epsilon 0 is their first argmax (ties of Q included), fp32-accurate
     initial priorities match compute_prior on the dueling net and the trees PerOracle, and bf16 actor priorities are the learner's;
  4. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; checkpoints load
     into AtariQNet(A, dueling=True) and torch.optim.Adam, and a resumed run equals an uninterrupted one; q_values against the CPU net.
The measured errors are written to $SRL_RESULTS_DIR/apex_dueling.json when SRL_RESULTS_DIR is set."""
import pytest

from tests import apex_cases as cases

pytestmark = pytest.mark.gpu
DUELING = cases.HEADS['dueling']


# ---------------------------------------------------------------------------------------------------------------- 1, 2
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (5, 4), (512, 18)])
def test_split_against_dueling_oracle(B, A, double, clip):
    cases.check_split_against_oracle(DUELING, B, A, double, clip)


@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (512, 18)])
def test_bf16_dueling_tail_against_fp64_and_encoder_backward(B, A, double):
    cases.check_bf16_tail_and_encoder_backward(DUELING, B, A, double)


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256, 1500])
def test_actor_q_values_are_the_learners_and_greedy_act(E):
    cases.check_actor_q_values_and_greedy_act(DUELING, E)


def test_fp32_actor_priorities_against_compute_prior():
    cases.check_fp32_actor_priorities(DUELING)


def test_bf16_actor_priorities_are_the_learners():
    cases.check_bf16_actor_priorities(DUELING)


# ---------------------------------------------------------------------------------------------------------------- 4
def test_determinism_and_graph_replay():
    cases.check_determinism_and_graph_replay(DUELING)


def test_captured_learn_from_loop_is_deterministic():
    cases.check_captured_learn_from_loop(DUELING)


def test_checkpoint_roundtrip_and_resume(tmp_path):
    cases.check_checkpoint_roundtrip_and_resume(DUELING, tmp_path)


@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    cases.check_q_values_against_cpu_network(DUELING, precision, tol)
