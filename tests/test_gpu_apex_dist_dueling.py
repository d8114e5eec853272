"""The distributional dueling head of the Ape-X learner and actors on the H100 (ApexHParams(distributional_dueling=True) with
categorical_dqn or quantile_dqn, B200ApexActor(..., distributional_dueling=True)): Rainbow's dueling rows per atom or quantile.  The
rows of this head are described here, as subclasses of the head table's rows (tests/apex_cases.py), and run through the checks every
head shares:
  1. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py's statements on the dueling rows of
     tests/apex_dist_dueling_ref.py) with the head's bounds (1e-5; the 12 gradients
     to rel-L2 1e-4, 2e-2 with genuine ReLU ties only; the weights after the step to 2e-6);
  2. bf16: the tail against fp64 on its own operands (core rows; the fp32 value and advantage weights composed in fp64): the rows, the
     C51 / QR quantities, dcore and the value and advantage gradients; the composed rows and the decomposed gradients element by element
     within c 2^-24 S, S the sum of the magnitudes of the terms and c the roundings; the encoder gradients equal srl_encoder_backward on
     the tail's dcore, bit for bit;
  3. the actor's rows, Q values and eps = 0 actions are the learner's bit for bit (ties included), bf16 actor priorities are the
     learner's bit for bit, fp32-accurate actor priorities match the oracle's and the trees match PerOracle;
  4. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; a target update
     between replays is seen; checkpoints load into AtariQNet(..., distributional_dueling=True) and torch.optim.Adam, and a resumed run
     equals an uninterrupted one; q_values against the CPU network; noisy variants of both heads; plain, C51 and QR actors refuse the
     learner.
The measured errors are written to $SRL_RESULTS_DIR/apex_dist_dueling.json when SRL_RESULTS_DIR is set."""
import dataclasses

import pytest
import torch

from scalerl_b200.algorithms.apex import ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner, default_q_state_dict
from tests import apex_cases as cases
from tests import apex_dist_dueling_ref as R
from tests.apex_cases import batch, learner, nmax, rel_l2
from tests.exact import record

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _oracle():
    """the shared checks' oracle statements build the dueling rows for this module's heads"""
    with R.installed():
        yield

F64 = torch.float64
RESULTS = 'apex_dist_dueling.json'
U = 2.0 ** -24


def _compose64(sd, A, W, dev='cuda'):
    """W_eff [A W, 512], b_eff [A W] in fp64 from the fp32 value and advantage layers"""
    g = lambda n: sd[n].to(dev).to(F64)
    adv, advb = g('advantage.weight').view(A, W, 512), g('advantage.bias').view(A, W)
    return ((g('value.weight')[None] + adv) - adv.mean(0, keepdim=True)).reshape(A * W, 512), \
        ((g('value.bias')[None] + advb) - advb.mean(0, keepdim=True)).reshape(A * W)


def _compose_bound(sd, A, W):
    """c 2^-24 S per element of the composed rows: S = |v| + |adv_a| + mean_a' |adv_a'|, c = A + 2 (A - 1 adds of the mean's sum, its
    division, the add and the subtraction)"""
    g = lambda n: sd[n].cuda().to(F64).abs()
    adv, advb = g('advantage.weight').view(A, W, 512), g('advantage.bias').view(A, W)
    S = (g('value.weight')[None] + adv + adv.mean(0, keepdim=True)).reshape(A * W, 512)
    Sb = (g('value.bias')[None] + advb + advb.mean(0, keepdim=True)).reshape(A * W)
    return (A + 2) * U * S, (A + 2) * U * Sb


def _decompose64(gW, gb, A, W):
    """(g_v, g_vb, g_adv, g_advb) in fp64 of the rows' gradients"""
    g, gbb = gW.to(F64).view(A, W, 512), gb.to(F64).view(A, W)
    return g.sum(0), gbb.sum(0), (g - g.mean(0, keepdim=True)).reshape(A * W, 512), (gbb - gbb.mean(0, keepdim=True)).reshape(A * W)


def _check_rows_elementwise(L, pre, A, W, key):
    """the composed rows and the decomposed gradients against fp64 on the device's own operands, element by element"""
    We, be = _compose64(pre, A, W)
    bW, bb = _compose_bound(pre, A, W)
    dW, db = L.debug_buffer('rows_weight_online').view(A * W, 512).to(F64), L.debug_buffer('rows_bias_online').to(F64)
    gW, gb = L.debug_buffer('rows_weight_grad').view(A * W, 512), L.debug_buffer('rows_bias_grad')
    gv, gvb, ga, gab = _decompose64(gW, gb, A, W)
    a = gW.to(F64).abs().view(A, W, 512)
    ab = gb.to(F64).abs().view(A, W)
    # g_v: A - 1 adds of |g|; g_adv: those over A, the division, the subtraction
    Sv, Svb = a.sum(0), ab.sum(0)
    Sa, Sab = (a + a.mean(0, keepdim=True)).reshape(A * W, 512), (ab + ab.mean(0, keepdim=True)).reshape(A * W)
    got = {'value.weight': (L.grads['value.weight'], gv, A * U * Sv), 'value.bias': (L.grads['value.bias'], gvb, A * U * Svb),
           'advantage.weight': (L.grads['advantage.weight'], ga, (A + 2) * U * Sa),
           'advantage.bias': (L.grads['advantage.bias'], gab, (A + 2) * U * Sab),
           'rows_weight': (dW, We, bW), 'rows_bias': (db, be, bb)}
    err = {}
    for k, (dev, want, bound) in got.items():
        d = (dev.to(F64) - want).abs()
        err[k] = float((d / bound.clamp(min=1e-300)).max())
        assert bool((d <= bound).all()), (k, err[k])
    record(RESULTS, f'elementwise_{key}', err)


# ---------------------------------------------------------------------------------------------------------------- the head rows
def _tail(row, L, pre, tg, batch_, w, gamma, double, B, A):
    """the C51 or QR tail in fp64 on the rows composed in fp64 from the fp32 value and advantage weights, and the value and advantage
    gradients of the fp64 rows' gradient"""
    W = row.width
    comp = lambda sd: dict(zip(('q.weight', 'q.bias'), _compose64(sd, A, W)))
    view = _RowsView(L)
    base = cases._tail_categorical if row.kind == 'categorical' else cases._tail_quantile
    pairs, loss, extra = base(row, view, comp(pre), comp(tg), batch_, w, gamma, double, B, A)
    # 'q.weight' / 'q.bias': the rows' gradients (device: rows_weight_grad) against fp64; then the decomposed ones against the fp64
    # decomposition of the fp64 rows' gradient
    gv, gvb, ga, gab = _decompose64(pairs['q.weight'][1], pairs['q.bias'][1], A, W)
    pairs.update({'value.weight': (L.grads['value.weight'], gv), 'value.bias': (L.grads['value.bias'], gvb),
                  'advantage.weight': (L.grads['advantage.weight'], ga), 'advantage.bias': (L.grads['advantage.bias'], gab)})
    pairs['rows'] = (L.debug_buffer('rows_weight_online').view(A * W, 512), comp(pre)['q.weight'])
    _check_rows_elementwise(L, pre, A, W, f'{row.tag(B, A)}_double{int(double)}{row.suffix}')
    return pairs, loss, extra


class _RowsView:
    """the learner as the C51 / QR tails of the head table read it: the rows' gradients in the places of q.weight and q.bias"""

    def __init__(self, L):
        self.L = L
        self.grads = {'q.weight': L.debug_buffer('rows_weight_grad').view(-1, 512), 'q.bias': L.debug_buffer('rows_bias_grad')}

    def debug_buffer(self, name):
        return self.L.debug_buffer(name)


def _tie_c51(sd, A, K):
    """actions 1 and 4 share their advantage rows, and their top atom dominates"""
    sd['advantage.weight'][4 * K:5 * K] = sd['advantage.weight'][K:2 * K]
    sd['advantage.bias'][2 * K - 1] += 30.0
    sd['advantage.bias'][4 * K:5 * K] = sd['advantage.bias'][K:2 * K]


def _tie_qr(sd, A, N):
    """actions 1 and 4 share their advantage rows, whose quantiles dominate"""
    sd['advantage.weight'][4 * N:5 * N] = sd['advantage.weight'][N:2 * N]
    sd['advantage.bias'][N:2 * N] += 30.0
    sd['advantage.bias'][4 * N:5 * N] = sd['advantage.bias'][N:2 * N]


@dataclasses.dataclass(frozen=True)
class DistDueling(cases.Head):
    """a row of the distributional dueling head: kind 'categorical' or 'quantile' with value and advantage layers"""

    @property
    def hp(self):
        return dict(super().hp, distributional_dueling=True)

    @property
    def net_kw(self):
        return dict(super().net_kw, distributional_dueling=True)

    @property
    def oracle(self):
        return R.Head(*super().oracle)

    def state_dict(self, A, seed, noisy_std=0.5):
        return default_q_state_dict(A, seed, False, self.width if self.kind == 'categorical' else 0, self.noisy, noisy_std,
                                    self.width if self.kind == 'quantile' else 0, dist_dueling=True)

    def tag(self, B, A):
        return f'{"noisy_" if self.noisy else ""}dd_{self.kind}_B{B}_A{A}_W{self.width}'

    @property
    def suffix(self):
        return {'categorical': f'_support{(self.v_min, self.v_max)}', 'quantile': f'_kappa{self.kappa}'}[self.kind]


C51 = DistDueling('dd_categorical', 'categorical', RESULTS, width=51, split_metrics=cases._C51, tail=_tail, actor_rows='logits', tie=_tie_c51,
                  refusal='distributional_dueling', fp32_prio_reward=10.0, bf16_prio_reward=3.0, trains='advantage.weight',
                  adam_probe='advantage.weight')
QR = DistDueling('dd_quantile', 'quantile', RESULTS, width=200, split_metrics=cases._QR, tail=_tail, actor_rows='theta', tie=_tie_qr,
                 refusal='distributional_dueling', bf16_prio_reward=3.0, trains='advantage.weight', adam_probe='advantage.weight')
NOISY_C51 = C51.but(name='noisy_dd_categorical', noisy=True, width=11, split_metrics=cases._NOISY_C51, trains='fc.weight_sigma',
                    adam_probe='fc.weight_sigma')
NOISY_QR = QR.but(name='noisy_dd_quantile', noisy=True, width=16, trains='fc.weight_sigma', adam_probe='fc.weight_sigma')
SUPPORTS = [(0.0, 200.0), (-10.0, 10.0)]


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('support', SUPPORTS)
@pytest.mark.parametrize('B,A,K', [(32, 6, 51), (5, 4, 2), (512, 18, 51), (64, 31, 64), (16, 1, 51)])
def test_split_against_oracle_c51(B, A, K, support, double, clip):
    cases.check_split_against_oracle(C51.but(width=K, v_min=support[0], v_max=support[1]), B, A, double, clip)


@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,N', [(32, 6, 200), (5, 4, 2), (512, 18, 200), (16, 1, 32)])
def test_split_against_oracle_qr(B, A, N, double, clip):
    cases.check_split_against_oracle(QR.but(width=N), B, A, double, clip)


@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head', [NOISY_C51, NOISY_QR], ids=str)
def test_noisy_split_against_oracle(head, double):
    cases.check_split_against_oracle(head, 32, 6, double, 40.0)


# ---------------------------------------------------------------------------------------------------------------- 2
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head,B,A', [(C51, 32, 6), (C51, 512, 18), (QR, 32, 6), (QR, 512, 18)], ids=str)
def test_bf16_tail_against_fp64_and_encoder_backward(head, B, A, double):
    cases.check_bf16_tail_and_encoder_backward(head, B, A, double)


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256, 1500])
@pytest.mark.parametrize('head', [C51, QR], ids=str)
def test_actor_rows_q_values_and_greedy_act_are_the_learners(head, E):
    cases.check_actor_q_values_and_greedy_act(head, E)


@pytest.mark.parametrize('head', [C51.but(width=21), QR.but(width=51, kappa=0.5)], ids=str)
def test_fp32_actor_priorities_against_oracle_and_trees(head):
    cases.check_fp32_actor_priorities(head)


@pytest.mark.parametrize('head', [C51, QR], ids=str)
def test_bf16_actor_priorities_are_the_learners(head):
    cases.check_bf16_actor_priorities(head)


def test_actor_rows_are_the_learners_composition():
    """the actor composes the snapshot as the learner composes its online network: the same rows, bit for bit"""
    A, W, E = 6, 51, 8
    L = B200ApexLearner(ApexHParams(batch_size=E, num_actions=A, **C51.hp), seed=3)
    X = cases.actor(C51, E, A)
    X.sync_from(L)
    X.q_values(cases.frames(E, 1, 'cuda'))
    L.learn(batch(E, A, seed=2, device='cuda')[0], use_graph=False)       # composes the pre-update weights, then updates them
    X_rows = X.debug_buffer('rows_weight')
    assert torch.equal(X_rows, L.debug_buffer('rows_weight_online')) and torch.equal(X.debug_buffer('rows_bias'), L.debug_buffer('rows_bias_online'))
    We, _ = _compose64(X.state_dict(), A, W)
    assert float((X_rows.view(A * W, 512).to(F64) - We).abs().max()) <= float(_compose_bound(X.state_dict(), A, W)[0].max())


# ---------------------------------------------------------------------------------------------------------------- 4
@pytest.mark.parametrize('head', [C51, QR, NOISY_C51, NOISY_QR], ids=str)
def test_determinism_and_graph_replay(head):
    cases.check_determinism_and_graph_replay(head)


@pytest.mark.parametrize('head', [C51.but(width=11), QR.but(width=51), NOISY_QR], ids=str)
def test_captured_learn_from_loop_is_deterministic(head):
    cases.check_captured_learn_from_loop(head)


@pytest.mark.parametrize('head', [C51, QR, NOISY_C51, NOISY_QR], ids=str)
def test_checkpoint_roundtrip_and_resume(head, tmp_path):
    cases.check_checkpoint_roundtrip_and_resume(head, tmp_path)


@pytest.mark.parametrize('head', [C51, QR], ids=str)
def test_target_update_between_replays_is_seen(head):
    """a target network loaded between two replays of the captured step is the one the next replay composes and reads"""
    B, A = 32, 6
    on, tg = cases.nets(head, A, seed=2)
    new_tg = head.state_dict(A, 99)
    batches = [batch(B, A, seed=s, device='cuda') for s in range(4)]
    kw = dict(target_update_frequency=1000)
    runs = []
    for graph, swap in ((True, True), (False, True), (True, False)):
        L = learner(head, B, A, on, tg, **kw)
        bufs = tuple(torch.empty_like(t) for t in batches[0][0])
        wb = torch.empty_like(batches[0][1])
        for k, (b, w) in enumerate(batches):
            if k == 3 and swap:
                L.load_state_dict(new_tg, target=True)
            for d, s in zip(bufs, b):
                d.copy_(s)
            wb.copy_(w)
            L.learn(bufs, weights=wb, use_graph=graph, sync_stats=False)
        torch.cuda.synchronize()
        assert len(L._graphs) == (1 if graph else 0)
        runs.append(L)
    g, e, stale = runs
    assert torch.equal(g.flat_params, e.flat_params) and torch.equal(g.debug_buffer('y'), e.debug_buffer('y'))
    assert torch.equal(g.debug_buffer('rows_weight_target'), e.debug_buffer('rows_weight_target'))
    We, _ = _compose64({n: v.cuda() for n, v in new_tg.items()}, A, head.width)
    assert nmax(g.debug_buffer('rows_weight_target').view(-1, 512), We) < 1e-6
    assert not torch.equal(g.debug_buffer('y'), stale.debug_buffer('y'))


@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
@pytest.mark.parametrize('head', [C51, QR], ids=str)
def test_q_values_against_cpu_network(head, precision, tol):
    """q_values / predict against AtariQNet(..., distributional_dueling=True) on the CPU; q_values leaves the step's rows alone"""
    B, A, n = 16, 18, 37                      # n > B: the forward runs in chunks of B frames
    torch.manual_seed(9)
    net = AtariQNet(A, **head.net_kw)
    if head.kind == 'quantile':
        with torch.no_grad():
            net.value.bias.add_(5.0)          # Q away from 0: a relative error is meaningful
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, precision=precision, **head.hp), init_state_dict=net.state_dict())
    obs = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8)
    q = L.q_values(obs)
    err = rel_l2(q, net(obs).detach())
    record(RESULTS, f'q_values_{head.kind}_{precision}', err)
    assert err <= tol, err
    assert torch.equal(L.predict(obs), q.argmax(-1))
    step_batch, w = batch(B, A, seed=1, device='cuda')
    L.learn(step_batch, weights=w, use_graph=False)
    rows = L.debug_buffer('rows_weight_online'), L.debug_buffer('core_next_target')
    L.q_values(obs)
    assert torch.equal(L.debug_buffer('rows_weight_online'), rows[0]) and torch.equal(L.debug_buffer('core_next_target'), rows[1])


@pytest.mark.parametrize('head', [C51, QR], ids=str)
def test_plain_c51_and_qr_actors_refuse_the_learner(head):
    L = B200ApexLearner(ApexHParams(batch_size=8, num_actions=6, **head.hp))
    others = [dict(), dict(categorical_dqn=True, num_atoms=head.width, v_min=head.v_min, v_max=head.v_max) if head.kind == 'categorical'
              else dict(quantile_dqn=True, num_quantiles=head.width), dict(categorical_dqn=True), dict(quantile_dqn=True)]
    for kw in others:
        with pytest.raises(ValueError, match='distributional_dueling=True'):
            B200ApexActor(4, 6, **kw).sync_from(L)
    X = B200ApexActor(4, 6, **head.hp)
    X.sync_from(L)
    assert torch.equal(X.flat_params, L.flat_params)
