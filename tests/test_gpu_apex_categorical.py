"""The categorical (C51) head of the Ape-X learner and actors on the H100 (ApexHParams(categorical_dqn=True),
B200ApexActor(..., categorical_dqn=True)), run through the checks every head shares (tests/apex_cases.py):
  1. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py): Q(s, a), m, CE, priorities and loss to 1e-5 (Q
     and the KL priorities normalised by the size of the terms they sum: Q = sum z p cancels on a support around 0, KL = CE - H(m)
     cancels when m is close to p), the 10 gradients to rel-L2 1e-4 (2e-2 when a genuine ReLU tie flipped), the weights after the step
     against the oracle's Adam on the device gradients to 2e-6;
  2. bf16: the categorical tail against fp64 on its own operands (core rows, fp32 head weights): logits, p, m, CE, KL, dlogits, the head
     gradients and dcore; the encoder gradients equal srl_encoder_backward on the tail's dcore, bit for bit;
  3. the actor's logits, Q values and eps = 0 actions are the learner's bit for bit (ties included), bf16 actor priorities are the
     learner's bit for bit, fp32-accurate actor priorities match the oracle's and the trees match PerOracle;
  4. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; checkpoints load
     into AtariQNet(A, categorical=True) and torch.optim.Adam, and a resumed run equals an uninterrupted one; q_values against the CPU net.
The measured errors are written to $SRL_RESULTS_DIR/apex_categorical.json when SRL_RESULTS_DIR is set."""
import pytest

from tests import apex_cases as cases

pytestmark = pytest.mark.gpu
CAT = cases.HEADS['categorical']                       # K = 51 on the (-10, 10) support
SUPPORTS = [(0.0, 200.0), (-10.0, 10.0)]
GRID = [(32, 6, 51), (5, 4, 2), (512, 18, 51), (64, 31, 64)]


def _cat(K, support):
    return CAT.but(width=K, v_min=support[0], v_max=support[1])


# ---------------------------------------------------------------------------------------------------------------- 1, 2
@pytest.mark.parametrize('support', SUPPORTS)
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,K', GRID)
def test_split_against_categorical_oracle(B, A, K, double, clip, support):
    cases.check_split_against_oracle(_cat(K, support), B, A, double, clip)


@pytest.mark.parametrize('support', SUPPORTS)
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,K', [(32, 6, 51), (512, 18, 51), (64, 31, 64)])
def test_bf16_categorical_tail_against_fp64_and_encoder_backward(B, A, K, double, support):
    cases.check_bf16_tail_and_encoder_backward(_cat(K, support), B, A, double)


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256, 1500])
def test_actor_logits_q_values_and_greedy_act_are_the_learners(E):
    cases.check_actor_q_values_and_greedy_act(CAT, E)


def test_fp32_actor_priorities_against_oracle_and_trees():
    cases.check_fp32_actor_priorities(_cat(51, (0.0, 200.0)))


def test_bf16_actor_priorities_are_the_learners():
    cases.check_bf16_actor_priorities(CAT)


# ---------------------------------------------------------------------------------------------------------------- 4
def test_determinism_and_graph_replay():
    cases.check_determinism_and_graph_replay(CAT)


def test_captured_learn_from_loop_is_deterministic():
    cases.check_captured_learn_from_loop(CAT)


def test_checkpoint_roundtrip_and_resume(tmp_path):
    cases.check_checkpoint_roundtrip_and_resume(CAT, tmp_path)


@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    cases.check_q_values_against_cpu_network(_cat(51, (0.0, 200.0)), precision, tol)      # Q near 100: a relative error is meaningful
