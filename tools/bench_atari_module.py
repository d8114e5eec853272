"""Time of one learner step of the reference's learn() statements (impala_atari.py:289-346: forward, V-trace, the three losses,
zero_grad, backward, clip_grad_norm_(40), RMSprop step; the stats dict and its host reads left out) for three models:

  reference     the reference's AtariNet on cuDNN in fp32, with its own vtrace / loss_fn (oracle/_ref, built by oracle/make_ref.py;
                skipped when it is missing).  The TF32 settings of the run are printed with it.
  dropin_eager  scalerl_b200's AtariNet with the vtrace / loss_fn drop-ins (the three imports swapped), eager
  dropin_graph  the same statements captured once in a CUDA graph and replayed (RMSprop(capturable=True))
  learner       B200ImpalaLearner.learn(sync_stats=False), the whole step on the library's kernels: the floor

python tools/bench_atari_module.py [--T 20 --B 32 --A 6 --steps 50 --warmup 10 --rounds 5 --precision bf16] [--use-lstm]
--use-lstm: the same four rows with AtariNet(use_lstm=True) and B200ImpalaLearner(use_lstm=True); every model starts from the same random
initial state (h0, c0).  The drop-in runs its LSTM on the sm_90a kernels in the bf16 mode, on nn.LSTM in fp32_split.
Each round times every model over --steps steps (host clock around work that ends in a device synchronise), alternating the models;
ms per step is reported as the median and the range over the rounds.  Prints the GPU name and power limit first, then one JSON line
per model.  Needs a CUDA device; writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import impala_oracle as O          # noqa: E402  (synthetic batch and initial weights)
from oracle import ref_learner                  # noqa: E402

HP = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, max_grad_norm=40.0)


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                       capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip() or q.stderr.strip()}


def learn_statements(model, vtrace, loss_fn, batch, optimizer, initial_rnn_state=()):
    """impala_atari.py:289-346 without the stats dict"""
    learner_outputs, _ = model(batch, initial_rnn_state)
    bootstrap_value = learner_outputs['baseline'][-1]
    batch = {key: tensor[1:] for key, tensor in batch.items()}
    learner_outputs = {key: tensor[:-1] for key, tensor in learner_outputs.items()}
    clipped_rewards = torch.clamp(batch['reward'], -1, 1)
    discounts = (~batch['done']).float() * HP['discounting']
    vtrace_returns = vtrace.from_logits(behavior_policy_logits=batch['policy_logits'], target_policy_logits=learner_outputs['policy_logits'],
                                        actions=batch['action'], discounts=discounts, rewards=clipped_rewards,
                                        values=learner_outputs['baseline'], bootstrap_value=bootstrap_value)
    pg_loss = loss_fn.compute_policy_gradient_loss(learner_outputs['policy_logits'], batch['action'], vtrace_returns.pg_advantages)
    baseline_loss = HP['baseline_cost'] * loss_fn.compute_baseline_loss(vtrace_returns.vs - learner_outputs['baseline'])
    entropy_loss = HP['entropy_cost'] * loss_fn.compute_entropy_loss(learner_outputs['policy_logits'])
    total_loss = pg_loss + baseline_loss + entropy_loss
    optimizer.zero_grad()
    total_loss.backward()
    nn.utils.clip_grad_norm_(model.parameters(), HP['max_grad_norm'])
    optimizer.step()


def rmsprop(model, capturable=False):
    return torch.optim.RMSprop(model.parameters(), lr=1e-4, eps=1e-5, alpha=0.99, capturable=capturable)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--T', type=int, default=20)
    ap.add_argument('--B', type=int, default=32)
    ap.add_argument('--A', type=int, default=6)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--precision', default='bf16', choices=['bf16', 'fp32_split'])
    ap.add_argument('--use-lstm', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_atari_module.py needs a CUDA device')
    from scalerl_b200.algorithms.impala import loss_fn as lf_mine, vtrace as vt_mine
    from scalerl_b200.algorithms.utils.atari_model import AtariNet
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    print(json.dumps({'gpu': gpu_info(), 'T': a.T, 'B': a.B, 'A': a.A, 'precision': a.precision, 'use_lstm': a.use_lstm,
                      'cudnn_allow_tf32': torch.backends.cudnn.allow_tf32, 'matmul_allow_tf32': torch.backends.cuda.matmul.allow_tf32}), flush=True)
    params = O.init_params(a.A, seed=0)
    if a.use_lstm:
        params.update(O.init_lstm_params(a.A, seed=0))
    batch = {k: v.cuda() for k, v in O.synthetic_batch(a.T, a.B, a.A, seed=0, done_p=0.05).items()}
    g = torch.Generator().manual_seed(1)
    state = tuple((torch.randn(2, a.B, 513 + a.A, generator=g) * 0.3).cuda() for _ in range(2)) if a.use_lstm else ()
    steps = {}

    if ref_learner.available():
        ref = ref_learner.ReferenceLearner(num_actions=a.A, use_lstm=a.use_lstm, state_dict=params)
        ref.model.cuda()
        ref_opt = rmsprop(ref.model)
        steps['reference'] = lambda: learn_statements(ref.model, ref.vtrace, ref.loss_fn, batch, ref_opt, state)
    else:
        print(json.dumps({'model': 'reference', 'ms_per_step': 'not measured: oracle/_ref is missing (python oracle/make_ref.py)'}))

    net = AtariNet((4, 84, 84), a.A, a.use_lstm, precision=a.precision).cuda()
    net.load_state_dict(params)
    opt = rmsprop(net)
    steps['dropin_eager'] = lambda: learn_statements(net, vt_mine, lf_mine, batch, opt, state)

    gnet = AtariNet((4, 84, 84), a.A, a.use_lstm, precision=a.precision).cuda()
    gnet.load_state_dict(params)
    gopt = rmsprop(gnet, capturable=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            learn_statements(gnet, vt_mine, lf_mine, batch, gopt, state)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        learn_statements(gnet, vt_mine, lf_mine, batch, gopt, state)
    steps['dropin_graph'] = graph.replay

    if not (a.use_lstm and a.precision == 'fp32_split'):       # the learner's LSTM has bf16 operands only
        hp = ImpalaHParams(rollout_length=a.T, batch_size=a.B, num_actions=a.A, precision=a.precision, use_lstm=a.use_lstm)
        learner = B200ImpalaLearner(hp, init_state_dict=params, process_group=False)
        steps['learner'] = lambda: learner.learn(batch, state, sync_stats=False)

    for fn in steps.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k, fn in steps.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                fn()
            torch.cuda.synchronize()
            ms[k].append((time.perf_counter() - t0) * 1e3 / a.steps)
    for k, v in ms.items():
        print(json.dumps({'model': k, 'ms_per_step_median': round(statistics.median(v), 4), 'ms_per_step_min': round(min(v), 4),
                          'ms_per_step_max': round(max(v), 4), 'rounds': a.rounds, 'steps_per_round': a.steps}), flush=True)


if __name__ == '__main__':
    main()
