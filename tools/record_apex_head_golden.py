"""Record tests/golden/apex_head_digests.json: SHA-256 digests of what the Ape-X learner and actor compute with each Q head (plain,
dueling, categorical), with and without double DQN, at B=32, A=6 and at a ragged B=19, A=18 on bf16 operands, plus one fp32_split
case per head (python tools/record_apex_head_golden.py [--out PATH]).  With --noisy it records tests/golden/apex_noisy_digests.json
instead: the noisy networks (noisy_dqn=True) of each head at B=32, A=6 with double DQN and at B=19, A=18 without, on bf16 operands,
and at B=32, A=6 with double DQN on fp32_split operands.

Per case, from fixed seeds:
  * learner: the learner's q_values on 300 frames (more than one 256-frame chunk); q, y, priorities, dcore and loss after the first
    learn() (and the categorical head's logits, m, ce and dlogits); flat_params, flat_target, exp_avg and exp_avg_sq after three;
  * actor (the same online weights): two consecutive act() calls, q_values, and the tree leaves one save_to_memory(...,
    priorities_from=actor) writes;
  * noisy cases also: the learner's normals, noise and composed fc and head tensors of both networks after the first learn(), and
    the actor's noise and composed fc and head weights after each act().

tests/test_gpu_apex_head_golden.py recomputes the digests and requires them to match bit for bit: the head code may change how it
is organised, not what it computes.  The state after three steps is downstream of the encoder's conv weight gradients, which are
per-CTA partial sums added in CTA order, so its bits depend on the SM count, which is stored beside them.  Needs a CUDA device."""
import argparse
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HEADS = ('plain', 'dueling', 'categorical')
CASES = tuple(f'{head}_B{B}_A{A}_double{d}_bf16' for head in HEADS for B, A in ((32, 6), (19, 18)) for d in (0, 1)) + \
    tuple(f'{head}_B32_A6_double1_fp32_split' for head in HEADS)
NOISY_CASES = tuple(f'noisy_{head}_{c}' for head in HEADS for c in ('B32_A6_double1_bf16', 'B19_A18_double0_bf16', 'B32_A6_double1_fp32_split'))
PER_SM = 'step3.'            # digests that depend on the SM count carry this prefix
OUT = os.path.join(ROOT, 'tests', 'golden', 'apex_head_digests.json')
NOISY_OUT = os.path.join(ROOT, 'tests', 'golden', 'apex_noisy_digests.json')


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _frames(n, seed):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).cuda()


def case_digests(case):
    """{output name: sha256 of its raw bytes} of one case of CASES or NOISY_CASES"""
    from scalerl_b200.algorithms.apex import ApexHParams, B200ApexActor, B200ApexLearner, default_q_state_dict
    from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
    noisy = case.startswith('noisy_')
    head, b, a, d, precision = case[len('noisy_') if noisy else 0:].split('_', 4)
    B, A, double = int(b[1:]), int(a[1:]), d == 'double1'
    dueling, K = head == 'dueling', 51 if head == 'categorical' else 0
    kw = dict(dueling_dqn=dueling, categorical_dqn=K > 0, v_min=-10.0, v_max=10.0, num_atoms=51) | (dict(noisy_dqn=True) if noisy else {})
    on, tg = default_q_state_dict(A, 2 * B + A, dueling, K, noisy), default_q_state_dict(A, 2 * B + A + 1, dueling, K, noisy)
    out = {}

    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, double_dqn=double, precision=precision, target_update_frequency=2,
                                    **kw), init_state_dict=on)
    L.load_state_dict(tg, target=True)
    out['learner.q_values'] = _sha(L.q_values(_frames(300, 7)))
    g = torch.Generator().manual_seed(B + A)
    batch = (torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g), torch.randint(0, A, (B,), generator=g),
             torch.randn(B, generator=g) * 3, torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g),
             torch.rand(B, generator=g) < 0.25)
    batch = tuple(t.cuda() for t in batch)
    weights = (torch.rand(B, generator=g) + 0.1).cuda()
    L.learn(batch, weights=weights, use_graph=False)
    for n in ('q', 'y', 'priorities', 'dcore', 'loss') + (('logits', 'm', 'ce', 'dlogits') if K else ()):
        out[f'step1.{n}'] = _sha(L.debug_buffer(n))
    noise = ('normals', 'noise', 'fc_weight', 'fc_bias', 'head_weight', 'head_bias') + (('head_adv_bias',) if dueling else ())
    for n in (f'{n}_{net}' for n in noise for net in ('online', 'target')) if noisy else ():
        out[f'step1.{n}'] = _sha(L.debug_buffer(n))
    for _ in range(2):
        L.learn(batch, weights=weights)
    torch.cuda.synchronize()
    for n in ('flat_params', 'flat_target', 'exp_avg', 'exp_avg_sq'):
        out[PER_SM + n] = _sha(getattr(L, n))
    L.close()

    E = B
    X = B200ApexActor(E, A, seed=B + A, precision=precision, init_state_dict=on, **kw)
    obs = _frames(E, 8)
    for i in range(2):
        out[f'actor.act{i}'] = _sha(X.act(obs))
        for n in ('noise', 'fc_weight', 'head_weight') if noisy else ():
            out[f'actor.act{i}.{n}'] = _sha(X.debug_buffer(n))
    out['actor.q_values'] = _sha(X.q_values(_frames(300, 9)))
    mem = GpuPrioritizedReplayBuffer(64, E, alpha=1.0, n_step=1, gamma=0.99)      # alpha = 1: the leaves are the priorities
    mem.save_to_memory(obs, batch[1][:E], batch[2][:E], _frames(E, 10), batch[4][:E], is_vectorised=True, priorities_from=X)
    cap = mem.sampler.capacity
    out['actor.leaves'] = _sha(mem.sampler.trees()[0][cap:cap + E])
    X.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--noisy', action='store_true', help='record the noisy cases (NOISY_CASES) into NOISY_OUT')
    ap.add_argument('--out', default=None, help='default: OUT, or NOISY_OUT with --noisy')
    a = ap.parse_args()
    rec = {'sms': torch.cuda.get_device_properties(0).multi_processor_count, 'device': torch.cuda.get_device_name(),
           'cases': {c: case_digests(c) for c in (NOISY_CASES if a.noisy else CASES)}}
    with open(a.out or (NOISY_OUT if a.noisy else OUT), 'w') as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write('\n')
    print(json.dumps(rec))


if __name__ == '__main__':
    main()
